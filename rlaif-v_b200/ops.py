"""Thin tensor-level wrappers over the C ABI (shape checks + pointer extraction only).

No arithmetic happens in Python/torch here: torch provides device memory and the stream.
"""
import torch

from . import lib as _l

ACT_NONE, ACT_GELU, ACT_QUICK_GELU = 0, 1, 2
IGNORE_INDEX = -100
IMAGE_TOKEN_INDEX = -200


def _chk(t, dtype=torch.bfloat16):
    assert t.is_cuda and t.dtype == dtype, (t.device, t.dtype)
    return t


def gemm(a, b, out=None, *, a_mn=False, b_mn=False, bias=None, residual=None, act=ACT_NONE,
         accumulate=False, tile_n=0, alpha=1.0):
    """out[M,N] (+)= op(a) @ op(b)^T (+bias)(act)(+residual).

    a_mn=False: a is [M,K] (K contiguous);  a_mn=True: a is stored [K,M].
    b_mn=False: b is [N,K] (K contiguous);  b_mn=True: b is stored [K,N].
    Row strides may exceed the row length (column-block views of a wider buffer).
    """
    _chk(a), _chk(b)
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    if a_mn:
        K, M = a.shape
    else:
        M, K = a.shape
    if b_mn:
        Kb, N = b.shape
    else:
        N, Kb = b.shape
    assert K == Kb, (a.shape, b.shape, a_mn, b_mn)
    if out is None:
        assert not accumulate
        out = torch.empty((M, N), dtype=torch.bfloat16, device=a.device)
    _chk(out)
    assert out.shape == (M, N) and out.stride(1) == 1
    if residual is not None:
        _chk(residual)
        assert residual.shape == (M, N) and residual.stride(1) == 1
    if bias is not None:
        _chk(bias)
        assert bias.numel() == N and bias.is_contiguous()
    if alpha != 1.0:
        _l.call("rlaifv_gemm_bf16_scaled", _l.ptr(a), a.stride(0), int(a_mn), _l.ptr(b), b.stride(0), int(b_mn),
                _l.ptr(out), out.stride(0), M, N, K, _l.ptr(bias), _l.ptr(residual),
                residual.stride(0) if residual is not None else 0, int(act), int(accumulate), int(tile_n),
                float(alpha), _l.stream_ptr())
        return out
    _l.call("rlaifv_gemm_bf16", _l.ptr(a), a.stride(0), int(a_mn), _l.ptr(b), b.stride(0), int(b_mn),
            _l.ptr(out), out.stride(0), M, N, K, _l.ptr(bias), _l.ptr(residual),
            residual.stride(0) if residual is not None else 0, int(act), int(accumulate), int(tile_n),
            _l.stream_ptr())
    return out


def attention_fwd(q, k, v, nseq, S, n_heads, head_dim, causal, scale, out=None, lse=None, n_kv_heads=None):
    """q/k/v: [nseq*S, ld] views (column blocks allowed) sharing one row stride.
    n_kv_heads < n_heads: grouped-query attention (k/v hold n_kv_heads heads)."""
    _chk(q), _chk(k), _chk(v)
    assert q.stride(0) == k.stride(0) == v.stride(0) and q.stride(1) == 1
    M = nseq * S
    if out is None:
        out = torch.empty((M, n_heads * head_dim), dtype=torch.bfloat16, device=q.device)
    if lse is None:
        lse = torch.empty((nseq, n_heads, S), dtype=torch.float32, device=q.device)
    if n_kv_heads is not None and n_kv_heads != n_heads:
        _l.call("rlaifv_attention_fwd_gqa", _l.ptr(q), _l.ptr(k), _l.ptr(v), q.stride(0), _l.ptr(out), out.stride(0),
                _l.ptr(lse), nseq, S, n_heads, n_kv_heads, head_dim, int(causal), float(scale), _l.stream_ptr())
        return out, lse
    _l.call("rlaifv_attention_fwd", _l.ptr(q), _l.ptr(k), _l.ptr(v), q.stride(0), _l.ptr(out), out.stride(0),
            _l.ptr(lse), nseq, S, n_heads, head_dim, int(causal), float(scale), _l.stream_ptr())
    return out, lse


def attention_bwd(q, k, v, out, d_out, lse, nseq, S, n_heads, head_dim, scale, dq_f32, dk, dv, delta_ws=None,
                  n_kv_heads=None):
    """dq_f32 [M, n_heads*head_dim] fp32 must be zeroed; dk/dv bf16 views with a shared row stride."""
    _chk(q), _chk(k), _chk(v), _chk(out), _chk(d_out), _chk(dk), _chk(dv)
    _chk(dq_f32, torch.float32), _chk(lse, torch.float32)
    assert dk.stride(0) == dv.stride(0)
    if delta_ws is None:
        delta_ws = torch.empty((nseq, n_heads, S), dtype=torch.float32, device=q.device)
    if n_kv_heads is not None and n_kv_heads != n_heads:
        _l.call("rlaifv_attention_bwd_gqa", _l.ptr(q), _l.ptr(k), _l.ptr(v), q.stride(0), _l.ptr(out), out.stride(0),
                _l.ptr(d_out), d_out.stride(0), _l.ptr(lse), _l.ptr(dq_f32), _l.ptr(dk), _l.ptr(dv), dk.stride(0),
                _l.ptr(delta_ws), nseq, S, n_heads, n_kv_heads, head_dim, float(scale), _l.stream_ptr())
        return dq_f32, dk, dv
    _l.call("rlaifv_attention_bwd", _l.ptr(q), _l.ptr(k), _l.ptr(v), q.stride(0), _l.ptr(out), out.stride(0),
            _l.ptr(d_out), d_out.stride(0), _l.ptr(lse), _l.ptr(dq_f32), _l.ptr(dk), _l.ptr(dv), dk.stride(0),
            _l.ptr(delta_ws), nseq, S, n_heads, head_dim, float(scale), _l.stream_ptr())
    return dq_f32, dk, dv


def attention_bwd_split(q, k, v, out, d_out, lse, nseq, Sq, Skv, n_heads, head_dim, causal, scale, dq, dk, dv,
                        n_kv_heads=None, delta_ws=None):
    """Split backward (dK/dV kernel + dQ kernel, no atomics): dq bf16 [nseq*Sq, n_heads*head_dim] (may be the q column
    block of a fused dqkv buffer), dk/dv bf16 views sharing a row stride. Nothing needs zero-filling."""
    _chk(q), _chk(k), _chk(v), _chk(out), _chk(d_out), _chk(dq), _chk(dk), _chk(dv), _chk(lse, torch.float32)
    assert dk.stride(0) == dv.stride(0) and k.stride(0) == v.stride(0) and q.stride(1) == 1 and dq.stride(1) == 1
    if delta_ws is None:
        delta_ws = torch.empty((nseq, n_heads, Sq), dtype=torch.float32, device=q.device)
    _l.call("rlaifv_attention_bwd_split", _l.ptr(q), q.stride(0), _l.ptr(k), _l.ptr(v), k.stride(0), _l.ptr(out),
            out.stride(0), _l.ptr(d_out), d_out.stride(0), _l.ptr(lse), _l.ptr(dq), dq.stride(0), _l.ptr(dk), _l.ptr(dv),
            dk.stride(0), _l.ptr(delta_ws), nseq, Sq, Skv, n_heads, n_heads if n_kv_heads is None else n_kv_heads,
            head_dim, int(causal), float(scale), _l.stream_ptr())
    return dq, dk, dv


def attention_varlen_fwd(q, k, v, pk, n_heads, head_dim, scale, out, lse, n_kv_heads=None):
    """Causal attention of packed rows (pk: model.RowPacking): q/k/v [pk.M, ld] views sharing one row stride,
    out [pk.M, n_heads*head_dim], lse fp32 [n_heads*pk.M] (sequence s's [n_heads][len_s] block at n_heads*cu[s])."""
    _chk(q), _chk(k), _chk(v), _chk(out), _chk(lse, _f32)
    assert q.stride(0) == k.stride(0) == v.stride(0) and q.stride(1) == 1 and lse.numel() == n_heads * pk.M
    _l.call("rlaifv_attention_varlen_fwd", _l.ptr(q), _l.ptr(k), _l.ptr(v), q.stride(0), _l.ptr(out), out.stride(0),
            _l.ptr(lse), _l.ptr(pk.cu), pk.nseq, pk.max_len, pk.M, n_heads,
            n_heads if n_kv_heads is None else n_kv_heads, head_dim, float(scale), _l.stream_ptr())
    return out, lse


def attention_varlen_bwd(q, k, v, out, d_out, lse, pk, n_heads, head_dim, scale, dq, dk, dv, delta_ws,
                         n_kv_heads=None):
    """Backward of attention_varlen_fwd (split form): dq bf16 [pk.M, n_heads*head_dim] (may be the q column block of a
    fused dqkv buffer), dk/dv bf16 views sharing a row stride, delta_ws fp32 [n_heads*pk.M]. Nothing needs zeroing."""
    _chk(q), _chk(k), _chk(v), _chk(out), _chk(d_out), _chk(dq), _chk(dk), _chk(dv), _chk(lse, _f32)
    _chk(delta_ws, _f32)
    assert q.stride(0) == k.stride(0) == v.stride(0) and dk.stride(0) == dv.stride(0) and dq.stride(1) == 1
    _l.call("rlaifv_attention_varlen_bwd", _l.ptr(q), _l.ptr(k), _l.ptr(v), q.stride(0), _l.ptr(out), out.stride(0),
            _l.ptr(d_out), d_out.stride(0), _l.ptr(lse), _l.ptr(dq), dq.stride(0), _l.ptr(dk), _l.ptr(dv),
            dk.stride(0), _l.ptr(delta_ws), _l.ptr(pk.cu), pk.nseq, pk.max_len, pk.M, n_heads,
            n_heads if n_kv_heads is None else n_kv_heads, head_dim, float(scale), _l.stream_ptr())
    return dq, dk, dv


def attention_varlen_prefix_fwd(q, k, v, pk, n_heads, head_dim, scale, out, lse, n_kv_heads=None):
    """attention_varlen_fwd over a RowPacking whose borrowers read the rows below pk.pos0 from their lenders
    (pk.pos0_h / pk.partner_h, DESIGN.md §3 "Shared prompt prefixes"); LSE holds own rows only."""
    _chk(q), _chk(k), _chk(v), _chk(out), _chk(lse, _f32)
    assert q.stride(0) == k.stride(0) == v.stride(0) and q.stride(1) == 1 and lse.numel() == n_heads * pk.M
    _l.call("rlaifv_attention_varlen_prefix_fwd", _l.ptr(q), _l.ptr(k), _l.ptr(v), q.stride(0), _l.ptr(out),
            out.stride(0), _l.ptr(lse), _l.ptr(pk.cu), _l.ptr(pk.pos0_h), _l.ptr(pk.partner_h), pk.nseq, pk.max_len,
            pk.M, n_heads, n_heads if n_kv_heads is None else n_kv_heads, head_dim, float(scale), _l.stream_ptr())
    return out, lse


def attention_varlen_prefix_bwd(q, k, v, out, d_out, lse, pk, n_heads, head_dim, scale, dq, dk, dv, delta_ws,
                                n_kv_heads=None):
    """Backward of attention_varlen_prefix_fwd: a lender's rows below its borrower's pos0 receive both sequences'
    dK/dV; everything else as attention_varlen_bwd."""
    _chk(q), _chk(k), _chk(v), _chk(out), _chk(d_out), _chk(dq), _chk(dk), _chk(dv), _chk(lse, _f32)
    _chk(delta_ws, _f32)
    assert q.stride(0) == k.stride(0) == v.stride(0) and dk.stride(0) == dv.stride(0) and dq.stride(1) == 1
    _l.call("rlaifv_attention_varlen_prefix_bwd", _l.ptr(q), _l.ptr(k), _l.ptr(v), q.stride(0), _l.ptr(out),
            out.stride(0), _l.ptr(d_out), d_out.stride(0), _l.ptr(lse), _l.ptr(dq), dq.stride(0), _l.ptr(dk),
            _l.ptr(dv), dk.stride(0), _l.ptr(delta_ws), _l.ptr(pk.cu), _l.ptr(pk.pos0_h), _l.ptr(pk.partner_h),
            pk.nseq, pk.max_len, pk.M, n_heads, n_heads if n_kv_heads is None else n_kv_heads, head_dim, float(scale),
            _l.stream_ptr())
    return dq, dk, dv


def cross_attention_fwd(q, k, v, nseq, Sq, Skv, n_heads, head_dim, scale, q_shared=True, out=None, lse=None):
    """Non-causal cross-attention: q [(1 if q_shared else nseq)*Sq, ld_q], k/v [nseq*Skv, ld_kv] (column blocks of
    one buffer allowed) -> out [nseq*Sq, n_heads*head_dim], lse [nseq, n_heads, Sq]."""
    _chk(q), _chk(k), _chk(v)
    assert k.stride(0) == v.stride(0) and q.stride(1) == 1
    if out is None:
        out = torch.empty((nseq * Sq, n_heads * head_dim), dtype=torch.bfloat16, device=q.device)
    if lse is None:
        lse = torch.empty((nseq, n_heads, Sq), dtype=torch.float32, device=q.device)
    _l.call("rlaifv_cross_attention_fwd", _l.ptr(q), q.stride(0), _l.ptr(k), _l.ptr(v), k.stride(0), _l.ptr(out),
            out.stride(0), _l.ptr(lse), nseq, Sq, Skv, n_heads, head_dim, int(q_shared), float(scale), _l.stream_ptr())
    return out, lse


def cross_attention_bwd(q, k, v, out, d_out, lse, nseq, Sq, Skv, n_heads, head_dim, scale, dq_f32, dk, dv,
                        q_shared=True, delta_ws=None):
    """dq_f32 fp32 [(1 if q_shared else nseq)*Sq, n_heads*head_dim] must be zeroed (q_shared: receives the batch sum);
    dk/dv bf16 [nseq*Skv, ...] views with a shared row stride."""
    _chk(q), _chk(k), _chk(v), _chk(out), _chk(d_out), _chk(dk), _chk(dv)
    _chk(dq_f32, torch.float32), _chk(lse, torch.float32)
    assert dk.stride(0) == dv.stride(0) and k.stride(0) == v.stride(0)
    if delta_ws is None:
        delta_ws = torch.empty((nseq, n_heads, Sq), dtype=torch.float32, device=q.device)
    _l.call("rlaifv_cross_attention_bwd", _l.ptr(q), q.stride(0), _l.ptr(k), _l.ptr(v), k.stride(0), _l.ptr(out),
            out.stride(0), _l.ptr(d_out), d_out.stride(0), _l.ptr(lse), _l.ptr(dq_f32), _l.ptr(dk), _l.ptr(dv),
            dk.stride(0), _l.ptr(delta_ws), nseq, Sq, Skv, n_heads, head_dim, int(q_shared), float(scale),
            _l.stream_ptr())
    return dq_f32, dk, dv


# --------------------------------------------------------------------------------------------
# row kernels
# --------------------------------------------------------------------------------------------
_f32 = torch.float32


def rmsnorm_fwd(x, w, eps, out=None, rstd=None):
    _chk(x), _chk(w)
    M, H = x.shape
    assert x.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    _l.call("rlaifv_rmsnorm_fwd", _l.ptr(x), _l.ptr(w), _l.ptr(out), _l.ptr(rstd), M, H, float(eps),
            _l.stream_ptr())
    return out


_norm_ws = {}


def _norm_workspace(H, device):
    n = _l.load().rlaifv_rmsnorm_bwd_partials()
    key = (H, device)
    if key not in _norm_ws:
        _norm_ws[key] = torch.empty((n, H), dtype=_f32, device=device)
    return _norm_ws[key]


def rmsnorm_bwd(dy, x, w, rstd, dx, dw, dres=None, dw_accumulate=True):
    """dx = rmsnorm'(dy) (+ dres); dw (+)= sum_rows dy * xhat."""
    _chk(dy), _chk(x), _chk(w), _chk(dx), _chk(dw), _chk(rstd, _f32)
    M, H = x.shape
    ws = _norm_workspace(H, x.device)
    _l.call("rlaifv_rmsnorm_bwd", _l.ptr(dy), _l.ptr(x), _l.ptr(w), _l.ptr(rstd), _l.ptr(dres), _l.ptr(dx),
            _l.ptr(dw), int(dw_accumulate), _l.ptr(ws), M, H, _l.stream_ptr())
    return dx


def layernorm_fwd(x, w, b, eps, out=None):
    _chk(x), _chk(w), _chk(b)
    M, H = x.shape
    if out is None:
        out = torch.empty_like(x)
    _l.call("rlaifv_layernorm_fwd", _l.ptr(x), _l.ptr(w), _l.ptr(b), _l.ptr(out), M, H, float(eps),
            _l.stream_ptr())
    return out


def layernorm_bwd(dy, x, w, eps, dx, dw, db, accumulate=True):
    """dx = layernorm'(dy) (statistics recomputed from x); dw (+)= sum_rows dy*xhat; db (+)= sum_rows dy."""
    _chk(dy), _chk(x), _chk(w), _chk(dx), _chk(dw), _chk(db)
    M, H = x.shape
    ws = _norm_workspace(2 * H, x.device)
    _l.call("rlaifv_layernorm_bwd", _l.ptr(dy), _l.ptr(x), _l.ptr(w), _l.ptr(dx), _l.ptr(dw), _l.ptr(db),
            int(accumulate), _l.ptr(ws), M, H, float(eps), _l.stream_ptr())
    return dx


def add_rows_bcast(x, table, out=None):
    """out[r] = x[r] + table[r % P] (position-embedding add shared by every image of the batch)."""
    _chk(x), _chk(table)
    assert x.shape[1] == table.shape[1] and x.is_contiguous() and table.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    _l.call("rlaifv_add_rows_bcast", _l.ptr(x), _l.ptr(table), _l.ptr(out), x.shape[0], table.shape[0], x.shape[1],
            _l.stream_ptr())
    return out


def rope_fwd(qkv, cos, sin, T, n_heads, head_dim, n_kv_heads=None):
    _chk(qkv), _chk(cos), _chk(sin)
    _l.call("rlaifv_rope_fwd_gqa", _l.ptr(qkv), _l.ptr(cos), _l.ptr(sin), qkv.shape[0], T, n_heads,
            n_heads if n_kv_heads is None else n_kv_heads, head_dim, qkv.stride(0), _l.stream_ptr())
    return qkv


def rope_bwd(dqkv, dq_f32, cos, sin, T, n_heads, head_dim, n_kv_heads=None):
    """dq_f32 None: the q block of dqkv already holds dQ (bf16, split attention backward) and is rotated in place."""
    _chk(dqkv)
    if dq_f32 is not None:
        _chk(dq_f32, _f32)
    _l.call("rlaifv_rope_bwd_gqa", _l.ptr(dqkv), _l.ptr(dq_f32), _l.ptr(cos), _l.ptr(sin), dqkv.shape[0], T,
            n_heads, n_heads if n_kv_heads is None else n_kv_heads, head_dim, dqkv.stride(0), _l.stream_ptr())
    return dqkv


def rope_pos_fwd(qkv, cos, sin, pos, n_heads, head_dim, n_kv_heads=None):
    """RoPE in place on fused qkv rows whose positions are pos (int32 [M]) — the packed rows' form of rope_fwd."""
    _chk(qkv), _chk(cos), _chk(sin), _chk(pos, torch.int32)
    assert pos.numel() == qkv.shape[0]
    _l.call("rlaifv_rope_pos_fwd", _l.ptr(qkv), _l.ptr(cos), _l.ptr(sin), _l.ptr(pos), qkv.shape[0], n_heads,
            n_heads if n_kv_heads is None else n_kv_heads, head_dim, qkv.stride(0), _l.stream_ptr())
    return qkv


def rope_pos_bwd(dqkv, cos, sin, pos, n_heads, head_dim, n_kv_heads=None):
    """Inverse rotation in place of the q (bf16 dQ of the split backward) and k blocks of dqkv at positions pos."""
    _chk(dqkv), _chk(cos), _chk(sin), _chk(pos, torch.int32)
    assert pos.numel() == dqkv.shape[0]
    _l.call("rlaifv_rope_pos_bwd", _l.ptr(dqkv), _l.ptr(cos), _l.ptr(sin), _l.ptr(pos), dqkv.shape[0], n_heads,
            n_heads if n_kv_heads is None else n_kv_heads, head_dim, dqkv.stride(0), _l.stream_ptr())
    return dqkv


def swiglu_fwd(gu, out=None):
    _chk(gu)
    M, F2 = gu.shape
    if out is None:
        out = torch.empty((M, F2 // 2), dtype=torch.bfloat16, device=gu.device)
    _l.call("rlaifv_swiglu_fwd", _l.ptr(gu), _l.ptr(out), M, F2 // 2, _l.stream_ptr())
    return out


def swiglu_bwd(gu, dact, dgu=None):
    _chk(gu), _chk(dact)
    M, F2 = gu.shape
    if dgu is None:
        dgu = torch.empty_like(gu)
    _l.call("rlaifv_swiglu_bwd", _l.ptr(gu), _l.ptr(dact), _l.ptr(dgu), M, F2 // 2, _l.stream_ptr())
    return dgu


def gelu_fwd(pre, post=None):
    _chk(pre)
    if post is None:
        post = torch.empty_like(pre)
    _l.call("rlaifv_gelu_fwd", _l.ptr(pre), _l.ptr(post), pre.numel(), _l.stream_ptr())
    return post


def gelu_bwd(pre, dpost, dpre=None):
    _chk(pre), _chk(dpost)
    if dpre is None:
        dpre = torch.empty_like(pre)
    _l.call("rlaifv_gelu_bwd", _l.ptr(pre), _l.ptr(dpost), _l.ptr(dpre), pre.numel(), _l.stream_ptr())
    return dpre


def colsum(x, db, accumulate=True):
    _chk(x), _chk(db)
    M, N = x.shape
    ws = torch.empty((64, N), dtype=_f32, device=x.device)
    _l.call("rlaifv_colsum", _l.ptr(x), M, N, _l.ptr(db), int(accumulate), _l.ptr(ws), _l.stream_ptr())
    return db


def clip_im2col(images, patch, k_pad):
    _chk(images)
    N, C, S, _ = images.shape
    G = S // patch
    out = torch.empty((N * G * G, k_pad), dtype=torch.bfloat16, device=images.device)
    _l.call("rlaifv_clip_im2col", _l.ptr(images), _l.ptr(out), N, C, S, patch, k_pad, _l.stream_ptr())
    return out


def clip_embed(patch_out, cls, pos, n_img, n_patch):
    _chk(patch_out), _chk(cls), _chk(pos)
    H = patch_out.shape[1]
    x = torch.empty((n_img * (n_patch + 1), H), dtype=torch.bfloat16, device=patch_out.device)
    _l.call("rlaifv_clip_embed", _l.ptr(patch_out), _l.ptr(cls), _l.ptr(pos), _l.ptr(x), n_img, n_patch, H,
            _l.stream_ptr())
    return x


def clip_drop_cls(x, n_img, n_patch):
    _chk(x)
    H = x.shape[1]
    out = torch.empty((n_img * n_patch, H), dtype=torch.bfloat16, device=x.device)
    _l.call("rlaifv_clip_drop_cls", _l.ptr(x), _l.ptr(out), n_img, n_patch, H, _l.stream_ptr())
    return out


def splice_count(ids, n_feat_tokens, max_len):
    assert ids.dtype == torch.int64 and ids.is_cuda and ids.is_contiguous()
    nseq, L = ids.shape
    n_img = torch.empty(nseq, dtype=torch.int32, device=ids.device)
    lens = torch.empty(nseq, dtype=torch.int32, device=ids.device)
    _l.call("rlaifv_splice_count", _l.ptr(ids), nseq, L, n_feat_tokens, max_len, _l.ptr(n_img), _l.ptr(lens),
            _l.stream_ptr())
    return n_img, lens


def splice_map(ids, labels, n_img, img_index, n_feat_tokens, T, max_len):
    nseq, L = ids.shape
    src = torch.empty((nseq, T), dtype=torch.int32, device=ids.device)
    new_labels = torch.empty((nseq, T), dtype=torch.int64, device=ids.device)
    assert img_index.dtype == torch.int32 and (labels is None or labels.is_contiguous())
    _l.call("rlaifv_splice_map", _l.ptr(ids), _l.ptr(labels), _l.ptr(n_img), _l.ptr(img_index), nseq, L,
            n_feat_tokens, T, max_len, _l.ptr(src), _l.ptr(new_labels), _l.stream_ptr())
    return src, new_labels


def splice_map_inplace(input_ids, img_index, num_query, im_patch, im_start, im_end):
    """OmniLMM in-place splice: -> (src [nseq, L] int32, status int32[1])."""
    assert input_ids.dtype == torch.int64 and input_ids.is_contiguous() and img_index.dtype == torch.int32
    nseq, L = input_ids.shape
    src = torch.empty((nseq, L), dtype=torch.int32, device=input_ids.device)
    status = torch.zeros(1, dtype=torch.int32, device=input_ids.device)
    _l.call("rlaifv_splice_map_inplace", _l.ptr(input_ids), _l.ptr(img_index), nseq, L, int(num_query), int(im_patch),
            int(im_start), int(im_end), _l.ptr(src), _l.ptr(status), _l.stream_ptr())
    return src, status


def splice_gather(src, ids, embed, feat, out=None):
    _chk(embed), _chk(feat)
    nseq, T = src.shape
    H = embed.shape[1]
    if out is None:
        out = torch.empty((nseq * T, H), dtype=torch.bfloat16, device=embed.device)
    _l.call("rlaifv_splice_gather", _l.ptr(src), _l.ptr(ids), _l.ptr(embed), _l.ptr(feat), _l.ptr(out), nseq,
            ids.shape[1], T, H, _l.stream_ptr())
    return out


def splice_scatter(src, ids, dx, d_embed_f32, d_feat_f32):
    _chk(dx)
    nseq, T = src.shape
    H = dx.shape[1]
    _l.call("rlaifv_splice_scatter", _l.ptr(src), _l.ptr(ids), _l.ptr(dx), _l.ptr(d_embed_f32),
            _l.ptr(d_feat_f32), nseq, ids.shape[1], T, H, _l.stream_ptr())


def f32_to_bf16(src, dst, accumulate=False):
    _chk(src, _f32), _chk(dst)
    assert src.numel() == dst.numel()
    _l.call("rlaifv_f32_to_bf16", _l.ptr(src), _l.ptr(dst), src.numel(), int(accumulate), _l.stream_ptr())
    return dst


def f32_to_bf16_2d(src, dst, accumulate=False):
    """fp32 [rows, cols] -> bf16 [rows, cols]; either side may be a column block of a wider buffer."""
    _chk(src, _f32), _chk(dst)
    assert src.shape == dst.shape and src.dim() == 2 and src.stride(1) == 1 and dst.stride(1) == 1
    _l.call("rlaifv_f32_to_bf16_2d", _l.ptr(src), src.stride(0), _l.ptr(dst), dst.stride(0), src.shape[0], src.shape[1],
            int(accumulate), _l.stream_ptr())
    return dst


def logp_fwd(logits, labels, nseq, T, row_pos=None):
    """logits [nseq*T, V] bf16 (row stride may exceed V), or with row_pos (compact head) [n_rows, V] of the gathered
    rows; labels [nseq, T] int64 (spliced). Returns per_tok [nseq, T-1] (zeros at unsupervised positions when compact),
    lse [nseq, T] (compact: [n_rows]), logp_sum, logp_avg, count [nseq] (all fp32)."""
    _chk(logits)
    assert labels.dtype == torch.int64 and labels.is_contiguous()
    (n, V), dev = logits.shape, logits.device
    if row_pos is None:
        per_tok = torch.empty((nseq, T - 1), dtype=_f32, device=dev)
        lse = torch.zeros((nseq, T), dtype=_f32, device=dev)
    else:
        assert row_pos.numel() == n
        per_tok = torch.zeros((nseq, T - 1), dtype=_f32, device=dev)
        lse = torch.zeros(n, dtype=_f32, device=dev)
    s = torch.empty(nseq, dtype=_f32, device=dev)
    a = torch.empty(nseq, dtype=_f32, device=dev)
    c = torch.empty(nseq, dtype=_f32, device=dev)
    _l.call("rlaifv_logp_fwd", _l.ptr(logits), logits.stride(0), _l.ptr(labels), _l.ptr(row_pos), n, nseq, T, V,
            _l.ptr(per_tok), _l.ptr(lse), _l.ptr(s), _l.ptr(a), _l.ptr(c), _l.stream_ptr())
    return per_tok, lse, s, a, c


def splice_token_weight(src, token_weight, T):
    """token_weight fp32 [nseq, Lw] (text positions) -> fp32 [nseq, T-1] in spliced positions (src int32 [nseq, T])."""
    _chk(token_weight, _f32)
    assert src.dtype == torch.int32 and src.is_contiguous() and token_weight.is_contiguous() and src.shape[1] == T
    nseq, Lw = token_weight.shape
    out = torch.empty((nseq, T - 1), dtype=_f32, device=src.device)
    _l.call("rlaifv_splice_token_weight", _l.ptr(src), _l.ptr(token_weight), _l.ptr(out), nseq, Lw, T, _l.stream_ptr())
    return out


def supervised_rows(labels, cap):
    """labels [nseq, T] int64 (spliced) -> row_pos int32 [nseq*cap]: flat positions s*T+t whose NEXT token is
    supervised (the rows get_batch_logps keeps), -1 in the unused slots of each sequence's cap-sized segment."""
    _chk(labels, torch.int64)
    assert labels.is_contiguous()
    nseq, T = labels.shape
    row_pos = torch.empty(nseq * cap, dtype=torch.int32, device=labels.device)
    _l.call("rlaifv_supervised_rows", _l.ptr(labels), nseq, T, int(cap), _l.ptr(row_pos), _l.stream_ptr())
    return row_pos


def rows_gather(row_pos, x, out=None):
    _chk(x)
    assert x.is_contiguous() and row_pos.dtype == torch.int32
    n, H = row_pos.numel(), x.shape[1]
    if out is None:
        out = torch.empty((n, H), dtype=torch.bfloat16, device=x.device)
    _l.call("rlaifv_rows_gather", _l.ptr(row_pos), _l.ptr(x), _l.ptr(out), n, H, _l.stream_ptr())
    return out


def rows_scatter(row_pos, dy, dx):
    """dx[row_pos[r]] = dy[r]; dx must be zero-filled by the caller."""
    _chk(dy), _chk(dx)
    assert dy.is_contiguous() and dx.is_contiguous() and dy.shape[1] == dx.shape[1]
    _l.call("rlaifv_rows_scatter", _l.ptr(row_pos), _l.ptr(dy), _l.ptr(dx), row_pos.numel(), dy.shape[1], _l.stream_ptr())
    return dx


def logp_bwd(logits, labels, lse, d_logp, nseq, T, row_pos=None, token_weight=None, norm=None):
    """In place on the dense or (row_pos given) compact logits: logits <- d loss / d logits. token_weight [nseq, T-1]:
    token-weighted log-prob; norm [nseq] (average mode): the label count, or the weight sum when weighted."""
    _chk(logits), _chk(lse, _f32), _chk(d_logp, _f32)
    assert row_pos is None or row_pos.numel() == logits.shape[0]
    if token_weight is not None:
        _chk(token_weight, _f32)
        assert tuple(token_weight.shape) == (nseq, T - 1) and token_weight.is_contiguous()
    _l.call("rlaifv_logp_bwd", _l.ptr(logits), logits.stride(0), _l.ptr(labels), _l.ptr(row_pos), logits.shape[0],
            _l.ptr(lse), _l.ptr(d_logp), _l.ptr(token_weight), _l.ptr(norm), nseq, T, logits.shape[1], _l.stream_ptr())
    return logits


def logp_weighted_reduce(per_tok, labels, token_weight):
    """compute_weighted_logp: per_tok / token_weight fp32 [nseq, T-1], labels int64 [nseq, T] ->
    (logp_w [nseq], avg_w [nseq], wsum [nseq])."""
    _chk(per_tok, _f32), _chk(token_weight, _f32)
    assert labels.dtype == torch.int64 and labels.is_contiguous() and per_tok.is_contiguous()
    nseq, T = labels.shape
    assert tuple(per_tok.shape) == (nseq, T - 1) and tuple(token_weight.shape) == (nseq, T - 1) \
        and token_weight.is_contiguous()
    lw = torch.empty(nseq, dtype=_f32, device=per_tok.device)
    aw, ws = torch.empty_like(lw), torch.empty_like(lw)
    _l.call("rlaifv_logp_weighted_reduce", _l.ptr(per_tok), _l.ptr(labels), _l.ptr(token_weight), nseq, T, _l.ptr(lw),
            _l.ptr(aw), _l.ptr(ws), _l.stream_ptr())
    return lw, aw, ws


def dpo_loss(policy_win, policy_rej, ref_win, ref_rej, beta, dpo_weight=1.0, sft_weight=0.0, grad_scale=1.0,
             want_grad=True):
    for t in (policy_win, policy_rej, ref_win, ref_rej):
        _chk(t, _f32)
    B = policy_win.numel()
    dev = policy_win.device
    losses = torch.empty(B, dtype=_f32, device=dev)
    cr = torch.empty(B, dtype=_f32, device=dev)
    rr = torch.empty(B, dtype=_f32, device=dev)
    dpw = torch.empty(B, dtype=_f32, device=dev) if want_grad else None
    dpr = torch.empty(B, dtype=_f32, device=dev) if want_grad else None
    out9 = torch.empty(9, dtype=_f32, device=dev)
    _l.call("rlaifv_dpo_loss", _l.ptr(policy_win), _l.ptr(policy_rej), _l.ptr(ref_win), _l.ptr(ref_rej), B,
            float(beta), float(dpo_weight), float(sft_weight), float(grad_scale), _l.ptr(losses), _l.ptr(cr),
            _l.ptr(rr), _l.ptr(dpw), _l.ptr(dpr), _l.ptr(out9), _l.stream_ptr())
    return losses, cr, rr, dpw, dpr, out9


def adamw_step(master, exp_avg, exp_avg_sq, grad, param_bf16, lr, beta1, beta2, eps, weight_decay, step,
               grad_scale=1.0):
    _chk(master, _f32), _chk(exp_avg, _f32), _chk(exp_avg_sq, _f32), _chk(param_bf16)
    assert grad.dtype in (torch.bfloat16, torch.float32)
    n = master.numel()
    assert grad.numel() == n and param_bf16.numel() == n
    _l.call("rlaifv_adamw_step", _l.ptr(master), _l.ptr(exp_avg), _l.ptr(exp_avg_sq), _l.ptr(grad),
            int(grad.dtype == torch.float32), _l.ptr(param_bf16), n, float(lr), float(beta1), float(beta2),
            float(eps), float(weight_decay), int(step), float(grad_scale), _l.stream_ptr())


def adamw_offload_bucket(host_master, host_exp_avg, host_exp_avg_sq, grad, param_bf16, decay_n, ring, slot_elems, lr,
                         beta1, beta2, eps, weight_decay, step, h2d_stream, d2h_stream):
    """AdamW of one bucket whose fp32 state is in pinned host memory, streamed through the device staging `ring`
    ([n_slots, 3 * slot_elems] fp32) on h2d_stream -> the current launch stream -> d2h_stream. Elements [0, decay_n)
    get weight decay. Pinned-ness is checked by the library (a pageable tensor raises B200Error)."""
    for t in (host_master, host_exp_avg, host_exp_avg_sq):
        assert t.dtype == _f32 and t.device.type == "cpu" and t.is_contiguous()
    _chk(ring, _f32), _chk(param_bf16), _chk(grad)
    n = host_master.numel()
    assert host_exp_avg.numel() == n and host_exp_avg_sq.numel() == n and grad.numel() == n and param_bf16.numel() == n
    assert ring.dim() == 2 and ring.shape[1] == 3 * slot_elems
    _l.call("rlaifv_adamw_offload_bucket", _l.ptr(host_master), _l.ptr(host_exp_avg), _l.ptr(host_exp_avg_sq),
            _l.ptr(grad), _l.ptr(param_bf16), n, int(decay_n), _l.ptr(ring), ring.shape[0], int(slot_elems), float(lr),
            float(beta1), float(beta2), float(eps), float(weight_decay), int(step), _l.stream_ptr(),
            _l.c_void_p(h2d_stream.cuda_stream), _l.c_void_p(d2h_stream.cuda_stream))


def adamw_offload_release(ring):
    """Destroy the library's events for `ring` (call after the ring's work has completed, before freeing it)."""
    _l.call("rlaifv_adamw_offload_release", _l.ptr(ring))


def adamw8bit_step(master, code_m, code_v, absmax_m, absmax_v, grad, param_bf16, decay_n, map_m, map_v, lr, beta1,
                   beta2, eps, weight_decay, step):
    """AdamW with blockwise 8-bit moments on one slice of n elements (blocks of 256 from its first element): fp32
    master, uint8 codes [n], fp32 absmax [ceil(n / 256)], bf16 grad / param [n]. Elements [0, decay_n) get weight
    decay. map_m / map_v: the signed / unsigned dynamic maps on the device (zero2.dynamic_map)."""
    _chk(master, _f32), _chk(code_m, torch.uint8), _chk(code_v, torch.uint8), _chk(absmax_m, _f32)
    _chk(absmax_v, _f32), _chk(grad), _chk(param_bf16), _chk(map_m, _f32), _chk(map_v, _f32)
    n = master.numel()
    nb = (n + 255) // 256
    assert code_m.numel() == n and code_v.numel() == n and grad.numel() == n and param_bf16.numel() == n
    assert absmax_m.numel() == nb and absmax_v.numel() == nb and map_m.numel() == 256 and map_v.numel() == 256
    _l.call("rlaifv_adamw8bit_step", _l.ptr(master), _l.ptr(code_m), _l.ptr(code_v), _l.ptr(absmax_m),
            _l.ptr(absmax_v), _l.ptr(grad), _l.ptr(param_bf16), n, int(decay_n), _l.ptr(map_m), _l.ptr(map_v),
            float(lr), float(beta1), float(beta2), float(eps), float(weight_decay), int(step), _l.stream_ptr())


def adamw8bit_offload_bucket(host_master, host_code_m, host_code_v, host_absmax_m, host_absmax_v, grad, param_bf16,
                             decay_n, map_m, map_v, ring, slot_elems, lr, beta1, beta2, eps, weight_decay, step,
                             h2d_stream, d2h_stream):
    """adamw8bit_step of one bucket whose state is in pinned host memory, streamed through the device staging `ring`
    ([n_slots, zero2.adamw8bit_slot_bytes(slot_elems)] uint8) on h2d_stream -> the current launch stream ->
    d2h_stream. Pinned-ness is checked by the library (a pageable tensor raises B200Error)."""
    n = host_master.numel()
    nb = (n + 255) // 256
    for t, dt, k in ((host_master, _f32, n), (host_code_m, torch.uint8, n), (host_code_v, torch.uint8, n),
                     (host_absmax_m, _f32, nb), (host_absmax_v, _f32, nb)):
        assert t.dtype == dt and t.device.type == "cpu" and t.is_contiguous() and t.numel() == k
    _chk(ring, torch.uint8), _chk(param_bf16), _chk(grad), _chk(map_m, _f32), _chk(map_v, _f32)
    assert grad.numel() == n and param_bf16.numel() == n and ring.dim() == 2
    _l.call("rlaifv_adamw8bit_offload_bucket", _l.ptr(host_master), _l.ptr(host_code_m), _l.ptr(host_code_v),
            _l.ptr(host_absmax_m), _l.ptr(host_absmax_v), _l.ptr(grad), _l.ptr(param_bf16), n, int(decay_n),
            _l.ptr(map_m), _l.ptr(map_v), _l.ptr(ring), ring.shape[0], int(slot_elems), float(lr), float(beta1),
            float(beta2), float(eps), float(weight_decay), int(step), _l.stream_ptr(),
            _l.c_void_p(h2d_stream.cuda_stream), _l.c_void_p(d2h_stream.cuda_stream))


def gemm_dual(a, b, a2, b2, out, *, k2, r, n_sub=0, b_mn=False, residual=None, accumulate=False):
    """out (+)= a @ op(b)^T + a2[:, koff:koff+k2] @ op(b2)^T (+ residual), one fp32 accumulator.
    koff = (n0 // n_sub) * r per output tile when n_sub > 0, else 0."""
    _chk(a), _chk(b), _chk(a2), _chk(b2), _chk(out)
    M, K = a.shape
    N = b.shape[1] if b_mn else b.shape[0]
    assert out.shape == (M, N)
    _l.call("rlaifv_gemm_bf16_dual", _l.ptr(a), a.stride(0), 0, _l.ptr(b), b.stride(0), int(b_mn), _l.ptr(a2),
            a2.stride(0), _l.ptr(b2), b2.stride(0), int(k2), int(r), int(n_sub), _l.ptr(out), out.stride(0), M, N, K,
            _l.ptr(None), _l.ptr(residual), residual.stride(0) if residual is not None else 0, 0, int(accumulate),
            _l.stream_ptr())
    return out


def gemm_swiglu_bwd(dy, w, gu, dgu, *, b_mn=True, a2=None, b2=None):
    """dgu [M, 2F] = swiglu_bwd(gu, dy @ op(w)^T (+ a2 @ op(b2)^T)) with d(act) kept in the GEMM accumulator
    (dy [M, K], w [K, F] when b_mn else [F, K], gu = [gate | up] [M, 2F])."""
    _chk(dy), _chk(w), _chk(gu), _chk(dgu)
    M, K = dy.shape
    F = w.shape[1] if b_mn else w.shape[0]
    assert gu.shape == (M, 2 * F) and dgu.shape == (M, 2 * F) and gu.stride(1) == 1 and dgu.stride(1) == 1
    k2 = 0
    if a2 is not None:
        _chk(a2), _chk(b2)
        k2 = a2.shape[1]
    _l.call("rlaifv_gemm_bf16_swiglu_bwd", _l.ptr(dy), dy.stride(0), _l.ptr(w), w.stride(0), int(b_mn), _l.ptr(a2),
            a2.stride(0) if a2 is not None else 0, _l.ptr(b2), b2.stride(0) if b2 is not None else 0, int(k2), _l.ptr(gu),
            gu.stride(0), _l.ptr(dgu), dgu.stride(0), M, F, K, _l.stream_ptr())
    return dgu


def dropout_fwd(x, p, seed, out=None, rows=None):
    """rows (int32 [M], packed rows): row r of x [M, width] draws the mask of row rows[r] of the padded layout."""
    _chk(x)
    assert x.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    if rows is not None:
        _chk(rows, torch.int32)
        assert rows.numel() == x.shape[0]
        _l.call("rlaifv_dropout_rows_fwd", _l.ptr(x), _l.ptr(out), _l.ptr(rows), x.shape[0], x.shape[1], float(p),
                int(seed), _l.stream_ptr())
        return out
    _l.call("rlaifv_dropout_fwd", _l.ptr(x), _l.ptr(out), x.numel(), float(p), int(seed), _l.stream_ptr())
    return out


def dropout_bwd_add(dx, g, p, seed, rows=None):
    """dx += mask(seed) * g / (1 - p), the mask of dropout_fwd with the same seed (and rows)."""
    _chk(dx), _chk(g)
    assert dx.is_contiguous() and g.is_contiguous() and dx.numel() == g.numel()
    if rows is not None:
        _chk(rows, torch.int32)
        assert rows.numel() == dx.shape[0]
        _l.call("rlaifv_dropout_rows_bwd_add", _l.ptr(dx), _l.ptr(g), _l.ptr(rows), dx.shape[0], dx.shape[1], float(p),
                int(seed), _l.stream_ptr())
        return dx
    _l.call("rlaifv_dropout_bwd_add", _l.ptr(dx), _l.ptr(g), dx.numel(), float(p), int(seed), _l.stream_ptr())
    return dx


# --------------------------------------------------------------------------------------------
# FP8 (e4m3) frozen base (DESIGN.md §3 "FP8 frozen base"; the format: include/rlaifv_b200.h)
# --------------------------------------------------------------------------------------------
_E4M3 = torch.float8_e4m3fn


class Fp8Weight:
    """A frozen weight W [N, K] in e4m3: codes q [N, K], the transposed codes qt [K, N] the dgrad reads, and the
    block scales s [N/128, K/128] fp32 shared by both."""

    def __init__(self, N, K, device):
        assert N % 128 == 0 and K % 128 == 0, (N, K)
        self.N, self.K = N, K
        self.q = torch.empty((N, K), dtype=_E4M3, device=device)
        self.qt = torch.empty((K, N), dtype=_E4M3, device=device)
        self.s = torch.empty((N // 128, K // 128), dtype=_f32, device=device)

    def rows(self, n0, n):
        """(q, qt, s) views of W's rows [n0, n0 + n) (n0, n: multiples of 128), for quantizing one sub-matrix."""
        assert n0 % 128 == 0 and n % 128 == 0
        return self.q[n0:n0 + n], self.qt[:, n0:n0 + n], self.s[n0 // 128:(n0 + n) // 128]

    def nbytes(self):
        return self.q.numel() + self.qt.numel() + 4 * self.s.numel()


def fp8_scale_rows(M):
    """Row-scale leading dimension of an M-row operand: M rounded up to a multiple of 4."""
    return (M + 3) // 4 * 4


def quant_fp8_rows(x, q=None, s=None):
    """x [M, K] bf16 (row stride allowed) -> (codes [M, K] e4m3, row scales [K/128, fp8_scale_rows(M)] fp32)."""
    _chk(x)
    M, K = x.shape
    assert x.stride(1) == 1
    if q is None:
        q = torch.empty((M, K), dtype=_E4M3, device=x.device)
    if s is None:
        s = torch.empty((K // 128, fp8_scale_rows(M)), dtype=_f32, device=x.device)
    _chk(q, _E4M3), _chk(s, _f32)
    assert q.shape == (M, K) and q.stride(1) == 1 and s.shape[0] == K // 128 and s.shape[1] >= M and s.stride(1) == 1
    _l.call("rlaifv_quant_fp8_rows", _l.ptr(x), x.stride(0), _l.ptr(q), q.stride(0), _l.ptr(s), s.stride(0), M, K,
            _l.stream_ptr())
    return q, s


def quant_fp8_blocks(w, q, qt, s):
    """W [N, K] bf16 -> codes q [N, K], transposed codes qt [K, N] and block scales s [N/128, K/128] (views of a wider
    Fp8Weight allowed: Fp8Weight.rows)."""
    _chk(w), _chk(q, _E4M3), _chk(qt, _E4M3), _chk(s, _f32)
    N, K = w.shape
    assert w.stride(1) == 1 and q.shape == (N, K) and qt.shape == (K, N) and s.shape == (N // 128, K // 128)
    assert q.stride(1) == 1 and qt.stride(1) == 1 and s.stride(1) == 1
    _l.call("rlaifv_quant_fp8_blocks", _l.ptr(w), w.stride(0), _l.ptr(q), q.stride(0), _l.ptr(qt), qt.stride(0),
            _l.ptr(s), s.stride(0), N, K, _l.stream_ptr())


def gemm_fp8(aq, sa, w, out, *, dgrad=False, a2=None, b2=None, k2=0, r=0, n_sub=0, residual=None, glu=None):
    """out [M, N] = dequant(aq, sa) @ op(W)^T (+ a2[:, koff:koff+k2] @ op(b2)^T) (+ residual), W an Fp8Weight.
    Forward (dgrad=False): op(W) = W, N = W.N, b2 [N, r] K-major. dgrad: op(W) = W^T (read from w.qt), N = W.K,
    b2 [k2, N] MN-major. glu ([gate | up] [M, 2N]): out [M, 2N] receives the SwiGLU backward of the product."""
    _chk(aq, _E4M3), _chk(sa, _f32), _chk(out)
    M, K = aq.shape
    B = w.qt if dgrad else w.q
    N = B.shape[0]
    assert B.shape[1] == K and aq.stride(1) == 1 and out.stride(1) == 1 and sa.shape[0] == K // 128
    assert out.shape == ((M, 2 * N) if glu is not None else (M, N))
    if a2 is not None:
        _chk(a2), _chk(b2)
        assert k2 > 0
    if residual is not None:
        _chk(residual)
        assert residual.shape == (M, N) and residual.stride(1) == 1
    if glu is not None:
        _chk(glu)
        assert glu.shape == (M, 2 * N) and glu.stride(1) == 1
    _l.call("rlaifv_gemm_fp8", _l.ptr(aq), aq.stride(0), _l.ptr(sa), sa.stride(0), _l.ptr(B), B.stride(0), _l.ptr(w.s),
            int(dgrad), _l.ptr(a2), a2.stride(0) if a2 is not None else 0, _l.ptr(b2),
            b2.stride(0) if b2 is not None else 0, int(k2) if a2 is not None else 0, int(r), int(n_sub), _l.ptr(out),
            out.stride(0), M, N, K, _l.ptr(residual), residual.stride(0) if residual is not None else 0, _l.ptr(glu),
            glu.stride(0) if glu is not None else 0, _l.stream_ptr())
    return out

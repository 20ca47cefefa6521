"""-m gpu kernel-level parity tests through the C ABI: every row kernel, the GEMM operand forms / epilogues,
attention forward / backward, splice edge cases (bit-exact), log-prob gather, DPO loss, AdamW.
Floating-point kernels are compared with a plain fp32 torch evaluation of the same op on the same bf16
inputs (tolerances in the asserts); integer / copy work must be bit-exact."""
import math

import os

import pytest
import torch

from oracle import llava_dpo_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


@pytest.fixture(autouse=True)
def _seed():
    torch.manual_seed(0)


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
@pytest.mark.parametrize("tile_n", [128, 256, 512])
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (304, 320, 200), (1136, 768, 1000)])
def test_gemm_operand_forms(a_mn, b_mn, tile_n, M, N, K):
    from rlaifv_b200 import ops
    A = (torch.randn(K, M, device=DEV) if a_mn else torch.randn(M, K, device=DEV)).to(BF)
    B = (torch.randn(K, N, device=DEV) if b_mn else torch.randn(N, K, device=DEV)).to(BF)
    ref = (A.float().t() if a_mn else A.float()) @ (B.float() if b_mn else B.float().t())
    got = ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, tile_n=tile_n)
    assert rel(got.float(), ref) <= 6e-3          # bf16 output rounding


def test_gemm_epilogues_and_views():
    from rlaifv_b200 import ops
    M, N, K = 777, 512, 384
    x = torch.randn(M, K, device=DEV).to(BF)
    w = (torch.randn(N, K, device=DEV) * 0.05).to(BF)
    bias = torch.randn(N, device=DEV).to(BF)
    res = torch.randn(M, N, device=DEV).to(BF)
    base = x.float() @ w.float().t()
    assert rel(ops.gemm(x, w, bias=bias).float(), base + bias.float()) <= 6e-3
    g = ops.gemm(x, w, bias=bias, act=ops.ACT_GELU).float()
    assert rel(g, torch.nn.functional.gelu((base + bias.float()).to(BF).float())) <= 8e-3
    q = ops.gemm(x, w, bias=bias, act=ops.ACT_QUICK_GELU).float()
    pre = (base + bias.float()).to(BF).float()
    assert rel(q, pre * torch.sigmoid(1.702 * pre)) <= 8e-3
    r = ops.gemm(x, w, residual=res).float()
    assert rel(r, base.to(BF).float() + res.float()) <= 6e-3
    acc = torch.randn(M, N, device=DEV).to(BF)
    want = base + acc.float()
    assert rel(ops.gemm(x, w, acc.clone(), accumulate=True).float(), want) <= 6e-3
    # alpha-scaled (LoRA) + column-block output view of a wider buffer
    wide = torch.zeros(M, 3 * N, device=DEV, dtype=BF)
    ops.gemm(x, w, wide[:, N:2 * N], alpha=0.25)
    assert rel(wide[:, N:2 * N].float(), 0.25 * base) <= 6e-3
    assert float(wide[:, :N].abs().max()) == 0.0 and float(wide[:, 2 * N:].abs().max()) == 0.0



@pytest.mark.parametrize("M,F,K,k2", [(300, 512, 256, 0), (1136, 1408, 520, 0), (520, 768, 384, 16)])
def test_gemm_swiglu_bwd_epilogue_matches_two_step_path(M, F, K, k2):
    """rlaifv_gemm_bf16_swiglu_bwd: d[gate|up] from the down-projection dgrad's epilogue vs (i) the unfused kernels
    (GEMM -> bf16 d(act) -> swiglu_bwd) and (ii) fp32 torch autograd of silu(g) * u on the bf16-rounded d(act)."""
    from rlaifv_b200 import ops
    dy = (torch.randn(M, K, device=DEV) * 0.5).to(BF)
    w = (torch.randn(K, F, device=DEV) * 0.1).to(BF)                     # W_down stored [H, F]: MN-major B operand
    gu = torch.randn(M, 2 * F, device=DEV).to(BF)
    a2 = b2 = None
    if k2:
        a2 = (torch.randn(M, k2, device=DEV) * 0.5).to(BF)
        b2 = (torch.randn(k2, F, device=DEV) * 0.1).to(BF)
    dact = ops.gemm(dy, w, b_mn=True) if not k2 else ops.gemm_dual(dy, w, a2, b2, torch.empty(M, F, device=DEV, dtype=BF),
                                                                  k2=k2, r=k2, n_sub=0, b_mn=True)
    two_step = ops.swiglu_bwd(gu, dact, torch.empty(M, 2 * F, device=DEV, dtype=BF))
    fused = ops.gemm_swiglu_bwd(dy, w, gu, torch.full((M, 2 * F), float("nan"), device=DEV, dtype=BF), a2=a2, b2=b2)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(fused.float()).all())
    assert rel(fused.float(), two_step.float()) <= 8e-3 and float((fused.float() - two_step.float()).abs().mean()) <= 1e-4
    g = gu[:, :F].float().requires_grad_()
    u = gu[:, F:].float().requires_grad_()
    (torch.nn.functional.silu(g) * u).backward(dact.float())
    ref = torch.cat([g.grad, u.grad], dim=1)
    assert rel(fused.float(), ref) <= 8e-3


@pytest.mark.parametrize("a_mn,b_mn,M,N,K", [(False, True, 2100, 1024, 8320), (True, True, 1024, 2104, 8320),
                                             (False, False, 1500, 1280, 16448)])
def test_gemm_long_k_raster_and_l2_hints_do_not_change_results(a_mn, b_mn, M, N, K):
    """K >= 8192 launches of the CTA-pair kernel pick their tile raster / L2 eviction hints per shape
    (gemm.cu: l2_auto_policy). Tile order and cache hints must not change a single bit of C: the automatic policy, the
    fixed round-1 raster and hand-forced variants (n-grouped walk, every hint combination) against fp32 torch and
    against each other."""
    from rlaifv_b200 import lib, ops
    L = lib.load()
    A = (torch.randn(K, M, device=DEV) if a_mn else torch.randn(M, K, device=DEV)).to(BF)
    B = (torch.randn(K, N, device=DEV) if b_mn else torch.randn(N, K, device=DEV)).to(BF)
    ref = (A.float().t() if a_mn else A.float()) @ (B.float() if b_mn else B.float().t())
    outs = []
    try:
        for group, l2 in ((16, -1), (16, 0), (8, 0x40), (4, 0x40 | 1 | (2 << 2)), (8, 2 | (1 << 2) | (1 << 4)), (3, 0x40 | (2 << 4))):
            L.rlaifv_gemm_set_tuning(group, 0)
            L.rlaifv_gemm_set_l2(l2)
            outs.append(ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, tile_n=512).clone())
    finally:
        L.rlaifv_gemm_set_tuning(16, 0)
        L.rlaifv_gemm_set_l2(-1)
    assert rel(outs[0].float(), ref) <= 6e-3
    for o in outs[1:]:
        assert torch.equal(o, outs[0])

@pytest.mark.parametrize("M", [500, 4200])          # 4200 rows: enough tiles for the CTA-pair kernel
def test_gemm_dual_source_matches_two_products(M):
    from rlaifv_b200 import ops
    K, r, nsub = 256, 8, 2048 if M > 1000 else 256
    x = torch.randn(M, K, device=DEV).to(BF)
    W = (torch.randn(2 * nsub, K, device=DEV) * 0.05).to(BF)
    t = torch.randn(M, 2 * r, device=DEV).to(BF)
    Bc = (torch.randn(2 * nsub, r, device=DEV) * 0.1).to(BF)
    out = torch.empty(M, 2 * nsub, device=DEV, dtype=BF)
    ops.gemm_dual(x, W, t, Bc, out, k2=r, r=r, n_sub=nsub)
    ref = x.float() @ W.float().t()
    ref[:, :nsub] += t[:, :r].float() @ Bc[:nsub].float().t()
    ref[:, nsub:] += t[:, r:].float() @ Bc[nsub:].float().t()
    assert rel(out.float(), ref) <= 6e-3
    # dgrad form: dy [M,N] @ W [N,K] (MN-major) + dt [M,2r] @ A [2r,K]
    dy = torch.randn(M, 2 * nsub, device=DEV).to(BF)
    A = (torch.randn(2 * r, K, device=DEV) * 0.1).to(BF)
    dx = torch.empty(M, K, device=DEV, dtype=BF)
    ops.gemm_dual(dy, W, t, A, dx, k2=2 * r, r=r, n_sub=0, b_mn=True)
    assert rel(dx.float(), dy.float() @ W.float() + t.float() @ A.float()) <= 6e-3


# ------------------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("nseq,S,nh,D,causal", [(2, 300, 2, 128, True), (1, 1135, 2, 128, True), (2, 577, 4, 64, False),
                                                (3, 5, 2, 64, False)])
def test_attention_forward(nseq, S, nh, D, causal):
    from rlaifv_b200 import ops
    H = nh * D
    qkv = torch.randn(nseq * S, 3 * H, device=DEV).to(BF)
    scale = D ** -0.5
    out, lse = ops.attention_fwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], nseq, S, nh, D, causal, scale)

    def split(t):
        return t.float().reshape(nseq, S, nh, D).permute(0, 2, 1, 3)
    q, k, v = split(qkv[:, :H]), split(qkv[:, H:2 * H]), split(qkv[:, 2 * H:])
    s = q @ k.transpose(-1, -2) * scale
    if causal:
        s = s.masked_fill(~torch.ones(S, S, device=DEV, dtype=torch.bool).tril(), float("-inf"))
    assert rel(split(out), torch.softmax(s, -1) @ v) <= 2e-2
    assert rel(lse, torch.logsumexp(s, -1)) <= 1e-3


def test_attention_backward():
    from rlaifv_b200 import ops
    nseq, S, nh, D = 2, 687, 2, 128
    H = nh * D
    qkv = torch.randn(nseq * S, 3 * H, device=DEV).to(BF)
    scale = D ** -0.5
    out, lse = ops.attention_fwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], nseq, S, nh, D, True, scale)
    d_out = torch.randn(nseq * S, H, device=DEV).to(BF)
    dq32 = torch.zeros(nseq * S, H, device=DEV)
    dqkv = torch.zeros(nseq * S, 3 * H, device=DEV, dtype=BF)
    ops.attention_bwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], out, d_out, lse, nseq, S, nh, D, scale, dq32,
                      dqkv[:, H:2 * H], dqkv[:, 2 * H:])

    def split(t):
        return t.float().reshape(nseq, S, nh, D).permute(0, 2, 1, 3).contiguous()
    q, k, v = (split(qkv[:, i * H:(i + 1) * H]).requires_grad_() for i in range(3))
    s = (q @ k.transpose(-1, -2) * scale).masked_fill(~torch.ones(S, S, device=DEV, dtype=torch.bool).tril(), float("-inf"))
    (torch.softmax(s, -1) @ v).backward(split(d_out))
    assert rel(split(dq32), q.grad) <= 3e-2
    assert rel(split(dqkv[:, H:2 * H]), k.grad) <= 3e-2
    assert rel(split(dqkv[:, 2 * H:]), v.grad) <= 3e-2


@pytest.mark.parametrize("nseq,S,nh,nkv,causal", [(2, 687, 2, 2, True), (2, 300, 4, 2, True), (2, 1025, 2, 2, False),
                                                  (3, 70, 2, 2, False), (1, 64, 1, 1, True)])
def test_attention_backward_split_kernels(nseq, S, nh, nkv, causal):
    """dK/dV kernel + dQ kernel (no atomics): dq written as bf16 into the q block of a NaN-poisoned fused buffer."""
    from rlaifv_b200 import ops
    D = 128
    H, KV = nh * D, nkv * D
    qkv = torch.randn(nseq * S, H + 2 * KV, device=DEV).to(BF)
    scale = D ** -0.5
    q_, k_, v_ = qkv[:, :H], qkv[:, H:H + KV], qkv[:, H + KV:]
    if causal:
        out, lse = ops.attention_fwd(q_, k_, v_, nseq, S, nh, D, True, scale, n_kv_heads=nkv)
    else:
        out, lse = ops.cross_attention_fwd(q_, k_, v_, nseq, S, S, nh, D, scale, q_shared=False)
    d_out = torch.randn(nseq * S, H, device=DEV).to(BF)
    dqkv = torch.full((nseq * S, H + 2 * KV), float("nan"), device=DEV, dtype=BF)
    ops.attention_bwd_split(q_, k_, v_, out, d_out, lse, nseq, S, S, nh, D, causal, scale, dqkv[:, :H], dqkv[:, H:H + KV],
                            dqkv[:, H + KV:], n_kv_heads=nkv)

    def split(t, n):
        return t.float().reshape(nseq, S, n, D).permute(0, 2, 1, 3).contiguous()
    q, k, v = split(q_, nh).requires_grad_(), split(k_, nkv).requires_grad_(), split(v_, nkv).requires_grad_()
    g = nh // nkv
    s = q @ k.repeat_interleave(g, 1).transpose(-1, -2) * scale
    if causal:
        s = s.masked_fill(~torch.ones(S, S, device=DEV, dtype=torch.bool).tril(), float("-inf"))
    (torch.softmax(s, -1) @ v.repeat_interleave(g, 1)).backward(split(d_out, nh))
    assert torch.isfinite(dqkv.float()).all()
    assert rel(split(dqkv[:, :H], nh), q.grad) <= 3e-2
    assert rel(split(dqkv[:, H:H + KV], nkv), k.grad) <= 3e-2
    assert rel(split(dqkv[:, H + KV:], nkv), v.grad) <= 3e-2


# ------------------------------------------------------------------------------------------------ row kernels
def test_rmsnorm_forward_backward():
    from rlaifv_b200 import ops
    M, H = 333, 4096
    x = torch.randn(M, H, device=DEV).to(BF)
    w = (1 + 0.1 * torch.randn(H, device=DEV)).to(BF)
    rstd = torch.empty(M, device=DEV)
    y = ops.rmsnorm_fwd(x, w, 1e-5, rstd=rstd)
    xf = x.float().requires_grad_()
    wf = w.float().requires_grad_()
    ref = O.rms_norm(xf, wf, 1e-5)
    assert rel(y.float(), ref) <= 8e-3
    dy = torch.randn(M, H, device=DEV).to(BF)
    dres = torch.randn(M, H, device=DEV).to(BF)
    dx = torch.empty_like(x)
    dw = torch.zeros(H, device=DEV, dtype=BF)
    ops.rmsnorm_bwd(dy, x, w, rstd, dx, dw, dres=dres, dw_accumulate=False)
    ref.backward(dy.float())
    assert rel(dx.float(), xf.grad + dres.float()) <= 1e-2
    assert rel(dw.float(), wf.grad) <= 1e-2


def test_layernorm_rope_swiglu_gelu_colsum():
    from rlaifv_b200 import ops
    M, H = 577, 1024
    x = torch.randn(M, H, device=DEV).to(BF)
    w, b = torch.randn(H, device=DEV).to(BF), torch.randn(H, device=DEV).to(BF)
    assert rel(ops.layernorm_fwd(x, w, b, 1e-5).float(),
               torch.nn.functional.layer_norm(x.float(), (H,), w.float(), b.float(), 1e-5)) <= 8e-3
    # RoPE forward == oracle formula; backward == transpose
    T, nh, D = 45, 2, 128
    nseq = 3
    qkv = torch.randn(nseq * T, 3 * nh * D, device=DEV).to(BF)
    cos, sin = O.rope_cos_sin(T, D, 10000.0, BF)
    cosd, sind = cos.to(DEV).contiguous(), sin.to(DEV).contiguous()
    ref_q = qkv[:, :nh * D].float().reshape(nseq, T, nh, D)
    want = (ref_q.to(BF) * cosd[None, :, None, :] + O.rotate_half(ref_q.to(BF)) * sind[None, :, None, :])
    got = ops.rope_fwd(qkv.clone(), cosd, sind, T, nh, D)
    assert torch.equal(got[:, :nh * D].reshape(nseq, T, nh, D), want)          # same bf16 rounding order: bit-exact
    assert torch.equal(got[:, 2 * nh * D:], qkv[:, 2 * nh * D:])               # v untouched
    # SwiGLU
    F_ = 512
    gu = torch.randn(M, 2 * F_, device=DEV).to(BF)
    act = ops.swiglu_fwd(gu)
    g, u = gu[:, :F_], gu[:, F_:]
    assert rel(act.float(), (torch.nn.functional.silu(g) * u).float()) <= 8e-3      # 1 bf16 ulp (fast exp)
    dact = torch.randn(M, F_, device=DEV).to(BF)
    dgu = ops.swiglu_bwd(gu, dact)
    gf, uf = g.float().requires_grad_(), u.float().requires_grad_()
    (torch.nn.functional.silu(gf) * uf).backward(dact.float())
    assert rel(dgu[:, :F_].float(), gf.grad) <= 8e-3 and rel(dgu[:, F_:].float(), uf.grad) <= 8e-3
    # GELU fwd/bwd, column sums
    pre = torch.randn(M, H, device=DEV).to(BF)
    assert rel(ops.gelu_fwd(pre).float(), torch.nn.functional.gelu(pre.float())) <= 8e-3
    pf = pre.float().requires_grad_()
    torch.nn.functional.gelu(pf).backward(x.float())
    assert rel(ops.gelu_bwd(pre, x).float(), pf.grad) <= 8e-3
    db = torch.zeros(H, device=DEV, dtype=BF)
    ops.colsum(x, db, accumulate=False)
    assert rel(db.float(), x.float().sum(0)) <= 8e-3


# ------------------------------------------------------------------------------------------------ splice (bit-exact)
@pytest.mark.parametrize("max_len", [2048, 30])
def test_splice_index_map_and_rows_bit_exact(max_len):
    from rlaifv_b200 import ops
    P, H, V = 16, 64, 100
    ids = torch.tensor([[1, 5, -200, 7, 8, 0, 0, 0], [1, -200, 9, 10, 11, 12, 13, 2], [1, 4, 5, 6, 7, 2, 0, 0],
                        [-200, 3, 4, 5, 6, 7, 8, 9]])
    labs = torch.tensor([[-100, -100, -100, 7, 8, -100, -100, -100], [-100, -100, 9, 10, 11, 12, 13, 2],
                         [-100, 4, 5, 6, 7, 2, -100, -100], [-100, 3, 4, 5, 6, 7, 8, 9]])
    src_ref, lab_ref, T = O.splice_index_map(ids, labs, P, max_len)
    idc, labc = ids.to(DEV), labs.to(DEV)
    n_img, lens = ops.splice_count(idc, P, max_len)
    assert int(lens.max()) == T and n_img.tolist() == [1, 1, 0, 1]
    img_index = torch.arange(4, dtype=torch.int32, device=DEV)
    src, new_labels = ops.splice_map(idc, labc, n_img, img_index, P, T, max_len)
    assert torch.equal(new_labels.cpu(), lab_ref)
    assert torch.equal(src.cpu().long(), src_ref)
    embed = torch.randn(V, H, device=DEV).to(BF)
    feat = torch.randn(4 * P, H, device=DEV).to(BF)
    rows = ops.splice_gather(src, idc, embed, feat).reshape(4, T, H)
    ref = O.splice_embeds({"model.embed_tokens.weight": embed.cpu()}, ids, src_ref, feat.cpu().reshape(4, P, H))
    assert torch.equal(rows.cpu(), ref)
    # backward scatter = transpose of the gather
    dx = torch.randn(4 * T, H, device=DEV).to(BF)
    d_embed = torch.zeros(V, H, device=DEV)
    d_feat = torch.zeros(4 * P, H, device=DEV)
    ops.splice_scatter(src, idc, dx, d_embed, d_feat)
    e = embed.cpu().float().requires_grad_()
    f = feat.cpu().float().requires_grad_()
    O.splice_embeds({"model.embed_tokens.weight": e}, ids, src_ref, f.reshape(4, P, H)).backward(dx.cpu().float().reshape(4, T, H))
    assert rel(d_embed, e.grad) <= 1e-6 and rel(d_feat, f.grad) <= 1e-6


EDGE_FX = os.path.join(os.path.dirname(__file__), "golden_host", "splice_edge_cases.npz")
# two image tokens in one sequence do not occur on the DPO path (one image per sample); the case is pinned anyway
EDGE_CASES = ["truncate_max_len_20", "truncate_inside_image", "no_image_sequence", "image_first_and_last", "very_ragged",
              "two_images_one_sequence"]


@pytest.mark.parametrize("name", EDGE_CASES)
def test_splice_edge_cases_match_reference_fixture(name):
    """The splice kernels on the edge inputs whose expected labels come from the unmodified reference
    (oracle/gen_golden_splice_edges.py); index map and row copies bit-exact."""
    import numpy as np
    from rlaifv_b200 import ops
    fx = np.load(EDGE_FX)
    ids, labs = torch.from_numpy(fx[name + ":ids"]), torch.from_numpy(fx[name + ":labels"])
    max_len, P, H, V = int(fx[name + ":max_len"]), O.TINY.num_patches, 64, O.TINY.vocab_size
    nseq = ids.shape[0]
    src_ref, lab_ref, T = O.splice_index_map(ids, labs, P, max_len)
    assert np.array_equal(lab_ref.numpy(), fx[name + ":ref_labels"])
    idc, labc = ids.to(DEV).contiguous(), labs.to(DEV).contiguous()
    n_img, lens = ops.splice_count(idc, P, max_len)
    assert int(lens.max()) == T
    n_slots = int(torch.clamp(n_img, min=1).sum())
    img_index = torch.arange(n_slots, dtype=torch.int32, device=DEV)
    src, new_labels = ops.splice_map(idc, labc, n_img, img_index, P, T, max_len)
    assert np.array_equal(new_labels.cpu().numpy(), fx[name + ":ref_labels"])
    assert torch.equal(src.cpu().long(), src_ref)
    embed = torch.randn(V, H, device=DEV).to(BF)
    feat = torch.randn(n_slots * P, H, device=DEV).to(BF)
    rows = ops.splice_gather(src, idc, embed, feat).reshape(nseq, T, H)
    ref = O.splice_embeds({"model.embed_tokens.weight": embed.cpu()}, ids, src_ref, feat.cpu().reshape(n_slots, P, H))
    assert torch.equal(rows.cpu(), ref)


# ------------------------------------------------------------------------------------------------ logp / loss / optimizer
def test_logp_gather_forward_backward():
    from rlaifv_b200 import ops
    nseq, T, V = 3, 37, 32000
    logits = (torch.randn(nseq * T, V, device=DEV) * 2).to(BF)
    labels = torch.randint(0, V, (nseq, T), device=DEV)
    labels[:, :10] = -100
    labels[1, 20:] = -100
    per_tok, lse, s, a, cnt = ops.logp_fwd(logits, labels, nseq, T)
    lf = logits.float().reshape(nseq, T, V).requires_grad_()
    rp, rs, ra = O.get_batch_logps(lf, labels)
    mask = labels[:, 1:] != -100
    assert rel(per_tok[mask], rp[mask]) <= 1e-5 and rel(s, rs) <= 1e-5 and rel(a, ra) <= 1e-5
    assert torch.equal(cnt.long(), mask.sum(-1))
    g = torch.randn(nseq, device=DEV)
    (rs * g).sum().backward()
    d = ops.logp_bwd(logits.clone(), labels, lse, g, nseq, T)
    assert rel(d.float().reshape(nseq, T, V), lf.grad) <= 1e-2


def test_dpo_loss_kernel_matches_reference_formula():
    from rlaifv_b200 import ops
    B = 37
    pw, pr, rw, rr = (torch.randn(B, device=DEV) * 20 - 100 for _ in range(4))
    losses, cr, rj, dpw, dpr, out9 = ops.dpo_loss(pw, pr, rw, rr, 0.1, dpo_weight=1.0, sft_weight=0.3)
    pwf, prf = pw.clone().requires_grad_(), pr.clone().requires_grad_()
    rl, rc, rrj = O.dpo_loss(pwf, prf, rw, rr, 0.1)
    loss = rl.mean() - 0.3 * pwf.mean()
    loss.backward()
    assert rel(losses, rl.detach()) <= 1e-5 and rel(cr, rc) <= 1e-5 and rel(rj, rrj) <= 1e-5
    assert rel(dpw, pwf.grad) <= 1e-4 and rel(dpr, prf.grad) <= 1e-4
    assert abs(float(out9[0]) - float(loss)) <= 1e-4 * abs(float(loss))
    assert abs(float(out9[3]) - float((rc > rrj).float().mean())) <= 1e-6


def test_fused_adamw_matches_torch():
    from rlaifv_b200 import ops
    n = 4096 * 3
    p0 = torch.randn(n, device=DEV)
    ref_p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([ref_p], lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    master, m, v = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    pbf = torch.empty(n, device=DEV, dtype=BF)
    for step in range(1, 4):
        g = (torch.randn(n, device=DEV) * 0.1).to(BF)
        ref_p.grad = g.float()
        opt.step()
        ops.adamw_step(master, m, v, g, pbf, 1e-3, 0.9, 0.999, 1e-8, 0.01, step)
        assert rel(master, ref_p.detach()) <= 1e-5
        assert torch.equal(pbf, master.to(BF))


def test_attention_grouped_query_forward_backward():
    """GQA (4 query heads share 2 kv heads): forward and backward vs fp32 torch with repeat_interleave."""
    from rlaifv_b200 import ops
    nseq, S, nh, nkv, D = 2, 300, 4, 2, 128
    H, KV = nh * D, nkv * D
    qkv = torch.randn(nseq * S, H + 2 * KV, device=DEV).to(BF)
    q_, k_, v_ = qkv[:, :H], qkv[:, H:H + KV], qkv[:, H + KV:]
    scale = D ** -0.5
    out, lse = ops.attention_fwd(q_, k_, v_, nseq, S, nh, D, True, scale, n_kv_heads=nkv)

    def split(t, n):
        return t.float().reshape(nseq, S, n, D).permute(0, 2, 1, 3).contiguous()
    q, k, v = split(q_, nh).requires_grad_(), split(k_, nkv).requires_grad_(), split(v_, nkv).requires_grad_()
    kk, vv = k.repeat_interleave(nh // nkv, dim=1), v.repeat_interleave(nh // nkv, dim=1)
    s = (q @ kk.transpose(-1, -2) * scale).masked_fill(~torch.ones(S, S, device=DEV, dtype=torch.bool).tril(), float("-inf"))
    ref = torch.softmax(s, -1) @ vv
    assert rel(split(out, nh), ref) <= 2e-2 and rel(lse, torch.logsumexp(s, -1)) <= 1e-3
    d_out = torch.randn(nseq * S, H, device=DEV).to(BF)
    dq32 = torch.zeros(nseq * S, H, device=DEV)
    dqkv = torch.zeros(nseq * S, H + 2 * KV, device=DEV, dtype=BF)
    ops.attention_bwd(q_, k_, v_, out, d_out, lse, nseq, S, nh, D, scale, dq32, dqkv[:, H:H + KV], dqkv[:, H + KV:],
                      n_kv_heads=nkv)
    ref.backward(split(d_out, nh))
    assert rel(split(dq32, nh), q.grad) <= 3e-2
    assert rel(split(dqkv[:, H:H + KV], nkv), k.grad) <= 3e-2
    assert rel(split(dqkv[:, H + KV:], nkv), v.grad) <= 3e-2


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
def test_experimental_split_k_matches_single_pass(a_mn, b_mn):
    """rlaifv_gemm_set_split_k (off by default; measured neutral-to-slower, DESIGN.md §3): K-slice passes with C += equal
    the single pass up to one bf16 rounding per slice."""
    from rlaifv_b200 import lib, ops
    M, N, K = 520, 512, 1000                                  # ragged K: the last slice takes the tail
    a = torch.randn((K, M) if a_mn else (M, K), device=DEV).to(BF)
    b = torch.randn((K, N) if b_mn else (N, K), device=DEV).to(BF)
    ref = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn)
    L = lib.load()
    try:
        for n in (2, 3):
            L.rlaifv_gemm_set_split_k(n, 256)
            got = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn)
            assert rel(got, ref) < 2e-2
            acc = ref.clone()
            ops.gemm(a, b, acc, a_mn=a_mn, b_mn=b_mn, accumulate=True)     # C += over every slice
            assert rel(acc, 2 * ref.float()) < 2e-2
    finally:
        L.rlaifv_gemm_set_split_k(0, 0)


# --------------------------------------------------------------------------------------------
# compact lm_head (supervised positions only)
# --------------------------------------------------------------------------------------------
def test_supervised_rows_index_bit_exact():
    from rlaifv_b200 import ops
    g = torch.Generator().manual_seed(3)
    nseq, T, cap = 5, 200, 64
    labels = torch.full((nseq, T), -100, dtype=torch.int64)
    for s in range(nseq):
        n = int(torch.randint(0, cap + 1, (1,), generator=g))
        idx = torch.randperm(T - 1, generator=g)[:n] + 1           # label positions 1..T-1 (position 0 is never a target)
        labels[s, idx] = torch.randint(3, 1000, (n,), generator=g)
    labels[0, 0] = 7                                               # a label at position 0 supervises nothing
    want = torch.full((nseq, cap), -1, dtype=torch.int32)
    for s in range(nseq):
        pos = [t for t in range(T - 1) if int(labels[s, t + 1]) != -100]
        want[s, :len(pos)] = torch.tensor([s * T + t for t in pos], dtype=torch.int32)
    got = ops.supervised_rows(labels.cuda(), cap).cpu().view(nseq, cap)
    assert torch.equal(got, want)


def test_compact_head_equals_full_head():
    """forward_logps(keep_stash=True) sends only supervised rows through norm / lm_head / log-softmax: summed log-probs
    are bit-identical to the full head's, per-token values agree on the supervised positions, gradients agree."""
    from oracle import llava_dpo_oracle as O
    from rlaifv_b200 import ops
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    c = O.TINY
    dims = LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                     num_layers=c.num_layers, num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                     clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                     image_size=c.image_size, patch_size=c.patch_size)
    pol = LlavaDPOPolicy(dims, "cuda", hf_state=O.make_params(c, seed=0, scale=0.4))
    batch = O.synthetic_pair_batch(c, 3, 24, 40, seed=9, image_pos=6, ragged=True)
    ids, labels, images = batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"]
    d_logp = torch.randn(6, generator=torch.Generator().manual_seed(1)).cuda()
    grads = {}
    outs = {}
    for compact in (False, True):
        pol.compact_head = compact
        out = pol.forward_logps(ids, labels, images, keep_stash=True)
        assert ("row_pos" in pol._stash) == compact
        pol.store.grad.zero_()
        pol.backward_logps(d_logp.clone())
        pol.finalize_embed_grad()
        torch.cuda.synchronize()
        grads[compact] = pol.store.grad.float().clone()
        outs[compact] = out
    assert torch.equal(outs[True]["logp"], outs[False]["logp"]) and torch.equal(outs[True]["avg_logp"], outs[False]["avg_logp"])
    mask = outs[False]["labels"][:, 1:] != -100
    assert torch.equal(outs[True]["per_token_logps"][mask], outs[False]["per_token_logps"][mask])
    assert float(outs[True]["per_token_logps"][~mask].abs().max()) == 0.0
    a, b = grads[True], grads[False]
    assert float((a - b).norm() / b.norm()) <= 2e-3
    assert float((a - b).abs().max()) <= 2e-2 * float(b.abs().max())
    # average mode + token weights take the same compact path
    pol.compact_head = True
    out = pol.forward_logps(ids, labels, images, keep_stash=True)
    tw = (torch.rand(6, out["labels"].shape[1] - 1, generator=torch.Generator().manual_seed(2)) + 0.5).cuda()
    lw, aw, ws = ops.logp_weighted_reduce(out["per_token_logps"], out["labels"], tw)
    pol.store.grad.zero_()
    pol.backward_logps(d_logp.clone(), use_average=True, token_weight=tw, weight_sum=ws)
    pol.finalize_embed_grad()
    gc = pol.store.grad.float().clone()
    pol.compact_head = False
    pol.forward_logps(ids, labels, images, keep_stash=True)
    pol.store.grad.zero_()
    pol.backward_logps(d_logp.clone(), use_average=True, token_weight=tw, weight_sum=ws)
    pol.finalize_embed_grad()
    torch.cuda.synchronize()
    gf = pol.store.grad.float()
    assert float((gc - gf).norm() / gf.norm()) <= 2e-3

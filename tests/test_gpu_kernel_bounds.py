"""GEMM and attention kernels against fp64 references with per-element error bounds.

Every kernel result is compared with the same operation evaluated in fp64 on the same bf16 inputs. A test fails when
any single element breaks its bound. Each bound is the computation repeated on absolute values, times the rounding the
kernel does, so an error confined to one row or one tile cannot hide behind the tensor's maximum.

The inputs are built to reach the paths the kernels branch on:
  - GEMM operands have their rows (A) and columns (B) scaled by powers of two spanning 2^-6 .. 2^6 (exact in bf16):
    a value written to the wrong element is then large next to that element's bound. Shapes walk several tiles per
    CTA, use every tile form (128, 256, the 2-CTA 512), strided operands and the skinny LoRA shapes.
  - Attention scores are peaked so that the online softmax's lazy running max (attention_fwd_kernel: it moves only
    when a KV tile beats it by more than 8 log2 units) moves, and O is rescaled: "rising" moves it on nearly every
    tile, "sink" once, late, by a lot, "scaled" (q x 16 or x 8) gives near one-hot rows.
Every GPU case asserts its premise (tiles per CTA, share of steps that move the max) and prints its worst err/bound.

The tests without the gpu mark check the bounds, the replay of the kernel's softmax loop and the premises on the CPU;
they never load the library.
"""
import math

import pytest
import torch
import torch.nn.functional as F

BF = torch.bfloat16
F64 = torch.float64
DEV = "cuda"
LOG2E = 1.0 / math.log(2.0)

ATT_TILE = 128             # attention_fwd_kernel: KV tile rows
LAZY_MAX = 8.0             # ... the running max moves only when a tile's max beats it by more than this (log2 units)
ACC = 2.0 ** -14           # GEMM: fp32 accumulation over K, relative to (|A| |B|)_ij (acc_term: its floor)
ACT_SLOPE = 1.13           # max |d/dx| of GELU(erf) and of quick-GELU x * sigmoid(1.702 x)
H100_SMS = 132

# attention_fwd / bwd kernels take exp2 with ex2.approx.ftz: P below 2^-126 becomes 0. That moves a result by at most
# 2^-126 times the row sums of |dP|, |K|, |Q|, |V| these inputs reach (< 2^36): an absolute floor on every attention bound
FTZ_FLOOR = 2.0 ** -90

RISE = 32.0                # "rising": log2 units the scores climb per 128-key tile
SINK = 24.0                # "sink": natural-log units the sink key's score stands above the rest
KINDS = ["rising", "sink", "scaled"]


# ================================================================================================ rounding and bounds
def bf16(x):
    """Round to bf16 (nearest even), keep the dtype."""
    return x.to(BF).to(x.dtype)


def ulp_bf16(x):
    """Spacing of the bf16 numbers at |x| (8 significant bits); below the normal range, the spacing at 2^-126."""
    _, e = torch.frexp(x.abs().to(F64).clamp_min(2.0 ** -126))
    return torch.exp2((e - 8).to(F64))


def violations(got, ref, bound):
    """(bad, ratio): elements outside their bound (NaN counts as outside) and err / bound."""
    err = (got.to(F64) - ref.to(F64)).abs()
    return ~(err <= bound), torch.where(err == 0, 0.0, err / bound)


def within(got, ref, bound):
    return not bool(violations(got, ref, bound)[0].any())


def assert_within(name, got, ref, bound):
    bad, ratio = violations(got, ref, bound)
    worst = float(ratio.nan_to_num(nan=float("inf")).max())
    print("err/bound %-44s %.3g" % (name, worst))
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d elements outside their bound; first at %s: got %r, fp64 %r, bound %r" % (
            name, int(bad.sum()), bad.numel(), i, float(got[i]), float(ref[i]), float(bound[i])))
    return worst


# ------------------------------------------------------------------------------------------------ GEMM
def acc_term(k=0):
    """Relative error of the fp32 wgmma accumulator after a contraction of depth k, as a multiple of (|A| |B|)_ij.

    The products of two bf16 values are exact in fp32. Each 16-deep wgmma step adds 16 of them to the accumulator;
    take its error as at most two fp32 units in the last place (2^-22: the alignment of the addends and the rounding
    of the sum, either of which may truncate) of the magnitude summed so far, which (|A| |B|)_ij bounds. Over
    ceil(k / 16) steps the errors add up to ceil(k / 16) 2^-22 (|A| |B|)_ij, Higham's recursive-summation bound
    (Accuracy and Stability of Numerical Algorithms, 2nd ed., section 4.2) with one term per step. Zero-filled steps
    past K add exact zeros. That passes the fixed 2^-14 above k = 4096: at the step's deepest launch (gate|up dgrad of
    LLaVA-1.5-13B, k = 27 648) it is 1728 x 2^-22 = 2^-11.2, so the fixed term could not be shown to hold there. For
    k <= 4096 the term stays 2^-14, so the bound of every shallower case is unchanged."""
    return max(ACC, math.ceil(k / 16) * 2.0 ** -22)


def gemm_ref(a, b, a_mn, b_mn, *, a2=None, b2=None, k2=0, r=0, n_sub=0, rows=None, cols=None):
    """op(a) @ op(b)^T in fp64, and the same product of absolute values (a_mn: a stored [K, M]; b_mn: b stored
    [K, N]).

    Second source (gemm.cu GemmSecondSource): + a2[:, koff(n) : koff(n) + k2] @ op(b2)^T, a2 stored [M, *] (K-major),
    b2 in b's layout ([k2, N] when b_mn), koff(n) = (n // n_sub) * r for output column n (0 when n_sub == 0): the
    kernel's koff = (n0 / n_sub) * r is the same for every column of a tile since the tile divides n_sub. Columns of
    a2 past its extent read as zero, as TMA fills them. rows / cols (slices): only that block of the output."""
    rows = rows if rows is not None else slice(None)
    cols = cols if cols is not None else slice(None)
    x = (a.t() if a_mn else a)[rows].to(F64)
    y = (b if b_mn else b.t())[:, cols].to(F64)
    c, mag = x @ y, x.abs() @ y.abs()
    if a2 is None:
        return c, mag
    assert not a_mn, "the second source is instantiated for K-major A only"
    y2 = (b2 if b_mn else b2.t())[:, cols]
    n = torch.arange(b.shape[1] if b_mn else b.shape[0])[cols]
    koff = (n // n_sub) * r if n_sub else torch.zeros_like(n)
    for k0 in koff.unique().tolist():
        j = (koff == k0).nonzero().squeeze(1).to(y2.device)
        x2 = a2[rows, k0:k0 + k2].to(F64)
        w2 = y2[:x2.shape[1], j].to(F64)
        c[:, j] += x2 @ w2
        mag[:, j] += x2.abs() @ w2.abs()
    return c, mag


def epilogue_ref(acc, mag, *, k=0, alpha=1.0, bias=None, act=0, residual=None, old=None):
    """gemm.cu epilogue_pair in fp64, rounding to bf16 where the kernel rounds. Returns (reference, bound).

    The bound starts at the accumulation term acc_term(k) * |A||B| (k: the contraction depth, K + K2 with a second
    source) and gains one bf16 ulp at every rounding point (the kernel and the reference may round a value to
    neighbouring bf16 numbers), carried through the later steps. Without an epilogue it is ulp(C64) + acc_term(k)
    (|A||B|), the ulp taken at |C64| plus the accumulation term."""
    v, e = acc, acc_term(k) * mag

    def rnd(v, e):
        return bf16(v), e + ulp_bf16(v.abs() + e)
    if alpha != 1.0:
        v, e = rnd(v, e)
        v, e = rnd(v * alpha, e * abs(alpha))
    if bias is not None:
        v = v + bias.to(F64)
    if act:
        v, e = rnd(v, e)
        if act == 1:
            # the kernel's fp32 1 + erff(x / sqrt 2) cancels for large negative x: erff's 2 ulp near -1, times |x| / 2
            v, e = 0.5 * v * (1 + torch.erf(v / math.sqrt(2.0))), ACT_SLOPE * e + 2.0 ** -21 * v.abs()
        else:
            v, e = v * torch.sigmoid(1.702 * v), ACT_SLOPE * e
    if residual is not None:
        v, e = rnd(v, e)
        v = v + residual.to(F64)
    if old is not None:
        v = v + old.to(F64)
    return v, e + ulp_bf16(v.abs() + e)


def pow2_rows(x, gen, span=6):
    """x with each row scaled by 2^u, u uniform in [-span, span] (exact in bf16)."""
    u = torch.randint(-span, span + 1, (x.shape[0], 1), generator=gen, device=gen.device).to(x)
    return x * torch.exp2(u)


def gemm_operand(rows, k, mn, gen, pad=0, device=DEV):
    """Logical [rows, k] bf16 operand with power-of-two row scales; mn: stored transposed ([k, rows]). pad > 0: a
    column block (at column 8) of a wider buffer whose other columns are NaN, so the row stride exceeds the extent.
    The values are drawn on gen's device (a CUDA generator keeps large operands off the host)."""
    x = pow2_rows(torch.randn(rows, k, generator=gen, dtype=F64, device=gen.device), gen).to(BF)
    st = x.t().contiguous() if mn else x
    if not pad:
        return st.to(device)
    buf = torch.full((st.shape[0], st.shape[1] + pad), float("nan"), dtype=BF, device=gen.device)
    buf[:, 8:8 + st.shape[1]] = st
    return buf.to(device)[:, 8:8 + st.shape[1]]


def gemm_walk(M, N, tile_n, sms):
    """(output tiles, CTA slots launched) of one launch, by launch_gemm's formula; tile_n 512 = 2-CTA clusters of a
    256 x 256 tile, counted as one slot per cluster."""
    cl = 2 if tile_n == 512 else 1
    bn = 256 if tile_n == 512 else tile_n
    tiles = -(-M // (cl * 128)) * -(-N // bn)
    return tiles, min(tiles, sms // cl)


def lda_legal(M, a_mn):
    """M of a case, rounded up to a multiple of 8 when A is stored [K, M] (its row stride lda = M must be)."""
    return -(-M // 8) * 8 if a_mn else M


def device_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ attention
def sink_key(S, causal):
    """The key index of the "sink": the first key of the last KV tile; causal, the last tile with at least 64 queries
    at or after its first key, so that a full query tile attends to the sink."""
    return ATT_TILE * ((S - 64) // ATT_TILE if causal else (S - 1) // ATT_TILE)


def attention_inputs(kind, nq, nseq, Sq, Skv, nh, nkv, D, causal, seed):
    """bf16 (CPU) q [nq, nh, Sq, D], k / v [nseq, nkv, Skv, D], d_out [nseq, nh, Sq, D] of one generator, and the
    softmax scale D^-0.5.
      rising: q's column 0 is 2, k's column 0 grows with the key index: the score climbs RISE log2 units per tile.
      sink:   q's column 0 is 2, k's column 0 is 0 except at sink_key(), whose score stands SINK above the others.
      scaled: q x 16 (D = 128) or x 8 (D = 64)."""
    gen = torch.Generator().manual_seed(seed)
    scale = D ** -0.5
    q = torch.randn(nq, nh, Sq, D, generator=gen, dtype=F64)
    k = torch.randn(nseq, nkv, Skv, D, generator=gen, dtype=F64)
    v = torch.randn(nseq, nkv, Skv, D, generator=gen, dtype=F64)
    do = torch.randn(nseq, nh, Sq, D, generator=gen, dtype=F64)
    if kind == "rising":
        q[..., 0] = 2.0
        k[..., 0] = torch.arange(Skv, dtype=F64) * (RISE / (ATT_TILE * 2.0 * scale * LOG2E))
    elif kind == "sink":
        q[..., 0] = 2.0
        k[..., 0] = 0.0
        k[..., sink_key(Skv, causal), 0] = SINK / (2.0 * scale)
    else:
        assert kind == "scaled"
        q = q * (16.0 if D == 128 else 8.0)
    return [t.to(BF) for t in (q, k, v, do)], scale


def expand_kv(t, nh):
    """[.., nkv, S, D] -> [.., nh, S, D]: query head h reads kv head h // (nh / nkv)."""
    return t.repeat_interleave(nh // t.shape[-3], dim=-3)


def causal_mask(Sq, Skv, device):
    return torch.ones(Sq, Skv, dtype=torch.bool, device=device).triu(1)


def lazy_max_moves(q, k, scale, causal):
    """fp64 replay of attention_fwd_kernel's running-max rule (128-key tiles, threshold LAZY_MAX log2 units).

    q [.., Sq, D], k [.., Skv, D] with k's heads expanded to q's. Returns (moved, visited), bool [.., Sq, n_tiles]:
    visited marks the (row, tile) steps after the row's first tile that the kernel runs (causal: up to the tile of the
    row's query tile), moved those where the running max moves (and O is rescaled)."""
    s = (q.to(F64) @ k.to(F64).transpose(-1, -2)) * (scale * LOG2E)
    Sq, Skv = s.shape[-2:]
    nt = -(-Skv // ATT_TILE)
    if causal:
        s = s.masked_fill(causal_mask(Sq, Skv, s.device), float("-inf"))
    tmax = F.pad(s, (0, nt * ATT_TILE - Skv), value=float("-inf")).reshape(*s.shape[:-1], nt, ATT_TILE).amax(-1)
    del s
    tiles = torch.arange(nt, device=tmax.device)
    last = torch.arange(Sq, device=tmax.device) // ATT_TILE if causal else torch.full((Sq,), nt - 1, device=tmax.device)
    visited = ((tiles[None, :] >= 1) & (tiles[None, :] <= last[:, None])).expand_as(tmax)
    moved = torch.zeros(tmax.shape, dtype=torch.bool, device=tmax.device)
    m = tmax[..., 0]
    for j in range(1, nt):
        mv = torch.maximum(m, tmax[..., j]) - m > LAZY_MAX
        moved[..., j] = mv
        m = torch.where(mv, tmax[..., j], m)
    return moved & visited, visited


def moved_share(q, k, scale, causal):
    moved, visited = lazy_max_moves(q, k, scale, causal)
    return float(moved.sum()) / float(visited.sum())


# share of (row, tile) steps that move the running max, at least, per generator (the premise tests show the values)
MIN_SHARE = {"rising": 0.9, "scaled": 0.05}
MIN_SHARE_CROSS = {"rising": 0.85, "scaled": 0.05}     # Skv = 1025: the last tile holds one key and cannot rise by 8


def assert_attention_premise(kind, q, k, scale, causal, min_share):
    """The generator reaches the rescale path: enough steps move the max; for the sink, every row that sees the sink
    moves its max at the sink's tile."""
    moved, visited = lazy_max_moves(q, expand_kv(k, q.shape[-3]), scale, causal)
    share = float(moved.sum()) / float(visited.sum())
    print("premise %s: %.3f of %d (row, tile) steps move the running max" % (kind, share, int(visited.sum())))
    if kind == "sink":
        sk = sink_key(k.shape[-2], causal)
        assert bool(moved[..., sk if causal else 0:, sk // ATT_TILE].all())
    else:
        assert share >= min_share[kind], (kind, share)


def attention_ref(q, k, v, scale, causal, d_out=None):
    """fp64 attention on the bf16 inputs and the error bounds of the kernels' results.

    q [.., nh, Sq, D]; k, v [.., nh, Skv, D] (heads expanded). The bounds are per element, each plus FTZ_FLOOR:
      O:   2^-8 (P|V| + |O|)             P rounded to bf16 before PV, O rounded to bf16: each at most 2^-8 relative
                                         (bf16's unit roundoff), so this is the worst case with no margin to spare
      lse: 2^-16 (1 + |lse| + scale max_j (|q| |k|)_ij)
      dV:  2^-8 (P^T |dO|) + 2^-8 |dV|   the same two roundings
      dK:  2^-7 scale (S^T |Q|) + 2^-8 |dK|, dQ: 2^-7 scale (S |K|) + 2^-8 |dQ|, S = P o (|dP| + |delta| + sum |dO||O|):
           delta taken from the bf16 O, dS rounded to bf16, the output rounded.
    The backward terms are returned without the output-rounding part (keys *_t) so that sums over GQA groups or over
    images of shared queries can be formed before it is added."""
    q, k, v = (t.to(F64) for t in (q, k, v))
    s = (q @ k.transpose(-1, -2)) * scale
    qk = (q.abs() @ k.abs().transpose(-1, -2)) * scale
    if causal:
        m = causal_mask(s.shape[-2], s.shape[-1], s.device)
        s = s.masked_fill(m, float("-inf"))
        qk = qk.masked_fill(m, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    del s
    o = p @ v
    r = {"o": o, "o_bound": 2.0 ** -8 * (p @ v.abs() + o.abs()) + FTZ_FLOOR, "lse": lse,
         "lse_bound": 2.0 ** -16 * (1 + lse.abs() + qk.amax(-1))}
    del qk
    if d_out is None:
        return r
    do = d_out.to(F64)
    dp = do @ v.transpose(-1, -2)
    delta = (do * o).sum(-1, keepdim=True)
    shat = p * (dp.abs() + delta.abs() + (do.abs() * o.abs()).sum(-1, keepdim=True))
    ds = p * (dp - delta)
    del dp
    r["dq"] = scale * (ds @ k)
    r["dk"] = scale * (ds.transpose(-1, -2) @ q)
    r["dv"] = p.transpose(-1, -2) @ do
    r["dq_t"] = 2.0 ** -7 * scale * (shat @ k.abs())
    r["dk_t"] = 2.0 ** -7 * scale * (shat.transpose(-1, -2) @ q.abs())
    r["dv_t"] = 2.0 ** -8 * (p.transpose(-1, -2) @ do.abs())
    return r


def with_output_rounding(r, key):
    """Bound of a backward result after any group / batch sums: the product term plus 2^-8 |ref|."""
    return r[key + "_t"] + 2.0 ** -8 * r[key].abs() + FTZ_FLOOR


def group_sum(t, nkv):
    """[.., nh, S, D] -> [.., nkv, S, D]: sum over the query heads of each kv group."""
    return t.reshape(*t.shape[:-3], nkv, t.shape[-3] // nkv, *t.shape[-2:]).sum(-3)


def forward_replay(q, k, v, scale, causal, rescale=True):
    """attention_fwd_kernel's tile loop in fp32 for one head (q [Sq, D], k / v [Skv, D] bf16): S in fp32, the lazy
    running max, P rounded to bf16 before PV, O rounded to bf16. rescale=False drops `o *= alpha`."""
    c = scale * LOG2E
    s = q.float() @ k.float().t()
    if causal:
        s = s.masked_fill(causal_mask(*s.shape, s.device), float("-inf"))
    Sq, Skv = s.shape
    m = torch.full((Sq, 1), float("-inf"))
    l = torch.zeros(Sq, 1)
    o = torch.zeros(Sq, v.shape[1])
    for j in range(-(-Skv // ATT_TILE)):
        st = s[:, j * ATT_TILE:(j + 1) * ATT_TILE]
        m_new = torch.maximum(m, st.amax(-1, keepdim=True) * c)
        m_new = m_new.masked_fill(m_new == float("-inf"), 0.0)
        if j > 0:
            m_new = torch.where(m_new - m <= LAZY_MAX, m, m_new)
        alpha = torch.exp2(m - m_new)
        l = l * alpha
        if rescale:
            o = o * alpha
        p = torch.exp2(st * c - m_new)
        l = l + p.sum(-1, keepdim=True)
        o = o + bf16(p) @ v[j * ATT_TILE:(j + 1) * ATT_TILE].float()
        m = m_new
    return bf16(o / l), ((m + torch.log2(l)) / LOG2E).squeeze(-1)


def heads(t, nseq, S, n, D):
    """[nseq*S, n*D] (a column block of a fused buffer) -> [nseq, n, S, D]."""
    return t.reshape(nseq, S, n, D).permute(0, 2, 1, 3)


def rows_of(t):
    """[nseq, n, S, D] -> [nseq*S, n*D]."""
    nseq, n, S, D = t.shape
    return t.permute(0, 2, 1, 3).reshape(nseq * S, n * D)


# ================================================================================================ CPU: the bounds
def _one_row(x, r, f=2.0 ** -5):
    y = x.clone()
    y[r] = y[r] * (1 + f)
    return y


def _one_tile(x, t=64, f=2.0 ** -5):
    y = x.clone()
    y[..., t:2 * t, t:2 * t] = y[..., t:2 * t, t:2 * t] * (1 + f)
    return y


def _global_rel(a, b):
    return float((a.to(F64) - b.to(F64)).abs().max() / b.to(F64).abs().max())


@pytest.mark.parametrize("epi", [{}, {"bias": True, "act": 1}, {"bias": True, "act": 2}, {"bias": True, "residual": True},
                                 {"accumulate": True}, {"alpha": 0.3}],
                         ids=["plain", "bias_gelu", "bias_quick_gelu", "bias_residual", "accumulate", "alpha"])
def test_gemm_bound_accepts_rounded_fp64_and_rejects_one_bad_row_or_tile(epi):
    gen = torch.Generator().manual_seed(1)
    M, N, K = 300, 264, 96
    a, b = gemm_operand(M, K, False, gen, device="cpu"), gemm_operand(N, K, False, gen, device="cpu")
    acc, mag = gemm_ref(a, b, False, False)
    typical = mag / math.sqrt(K)
    kw = {"alpha": epi.get("alpha", 1.0), "act": epi.get("act", 0)}
    if epi.get("bias"):
        kw["bias"] = torch.randn(N, generator=gen, dtype=F64).to(BF)
    if epi.get("residual"):
        kw["residual"] = bf16(torch.randn(M, N, generator=gen, dtype=F64) * typical)
    if epi.get("accumulate"):
        kw["old"] = bf16(torch.randn(M, N, generator=gen, dtype=F64) * typical)
    ref, bound = epilogue_ref(acc, mag, **kw)
    assert within(bf16(ref), ref, bound)
    # the row whose values are smallest: a 2^-5 error there is invisible to a check against the tensor's maximum
    r = int(ref.abs().amax(1).argmin())
    assert not within(_one_row(bf16(ref), r), ref, bound)
    assert not within(_one_tile(bf16(ref)), ref, bound)
    if not epi:
        assert _global_rel(_one_row(bf16(ref), r), ref) < 6e-3


def test_activation_slope_bound():
    x = torch.linspace(-12, 12, 200001, dtype=F64, requires_grad=True)
    for y in (0.5 * x * (1 + torch.erf(x / math.sqrt(2.0))), x * torch.sigmoid(1.702 * x)):
        g, = torch.autograd.grad(y.sum(), x)
        assert float(g.abs().max()) <= ACT_SLOPE


@pytest.mark.parametrize("kind", KINDS)
def test_attention_bounds_accept_rounded_fp64_and_reject_one_bad_row_or_tile(kind):
    """O and lse reject a 2^-5 relative error in one row or tile. The dQ / dK / dV bounds allow more than 2^-5 of a
    row's own size where a softmax row cancels (dS = P (dP - delta) with delta from the bf16 O), so there the error is
    2^-5 of the tensor's maximum, confined to one row or tile."""
    S, D = 300, 64
    (q, k, v, do), scale = attention_inputs(kind, 1, 1, S, S, 2, 2, D, True, seed=2)
    r = attention_ref(q, k, v, scale, True, do)
    checks = [("o", r["o"], r["o_bound"]), ("dq", r["dq"], with_output_rounding(r, "dq")),
              ("dk", r["dk"], with_output_rounding(r, "dk")), ("dv", r["dv"], with_output_rounding(r, "dv"))]
    for name, ref, bound in checks:
        assert within(bf16(ref), ref, bound), name
        if name == "o":
            bad_row, bad_tile = bf16(ref), _one_tile(bf16(ref), t=32)
            bad_row[0, 0, S // 2] *= 1 + 2.0 ** -5
        else:
            err = 2.0 ** -5 * float(ref.abs().max())
            bad_row, bad_tile = bf16(ref), bf16(ref)
            bad_row[0, 0, S // 2] += err
            bad_tile[0, 0, 32:64, 32:64] -= err
        assert not within(bad_row, ref, bound), name
        assert not within(bad_tile, ref, bound), name
    lse = r["lse"].float()
    assert within(lse, r["lse"], r["lse_bound"])
    assert not within(_one_row(lse[0, 0], 5), r["lse"][0, 0], r["lse_bound"][0, 0])


@pytest.mark.parametrize("causal", [True, False])
def test_forward_replay_passes_the_o_bound_only_with_the_rescale(causal):
    """The kernel's tile loop replayed in fp32 meets the O and lse bounds; without `o *= alpha` it breaks the O bound.
    The same inputs are what the GPU cases feed the kernel."""
    S, D = 700, 128
    (q, k, v, _), scale = attention_inputs("rising", 1, 1, S, S, 1, 1, D, causal, seed=3)
    q, k, v = q[0, 0], k[0, 0], v[0, 0]
    r = attention_ref(q, k, v, scale, causal)
    o, lse = forward_replay(q, k, v, scale, causal)
    assert within(o, r["o"], r["o_bound"]) and within(lse, r["lse"], r["lse_bound"])
    o_bad, _ = forward_replay(q, k, v, scale, causal, rescale=False)
    assert not within(o_bad, r["o"], r["o_bound"])


# ================================================================================================ CPU: the premises
PERSISTENT = (4100, 2056, 520)
EPI_SHAPE = (1100, 776, 264)
STRIDED = (1000, 520, 200)


def test_gemm_premise_persistent_walk_has_more_tiles_than_slots():
    M, N, _ = PERSISTENT
    for tile_n in (128, 256, 512):
        tiles, slots = gemm_walk(M, N, tile_n, H100_SMS)
        assert tiles > slots, (tile_n, tiles, slots)
    assert gemm_walk(M, N, 128, H100_SMS) == (561, 132) and gemm_walk(M, N, 512, H100_SMS) == (153, 66)
    # the cluster corners: M <= 128 leaves the second CTA of the pair without rows
    assert gemm_walk(128, 256, 512, H100_SMS) == (1, 1)


ATT_CAUSAL = [(1135, 2, 2), (2049, 2, 2), (1135, 8, 2)]        # (S, query heads, kv heads), D = 128
ATT_NONCAUSAL = [577, 1100]                                    # D = 64, 2 sequences, 2 heads
CROSS = (3, 64, 1025, 2)                                       # nseq, Sq, Skv, heads (q shared), D = 128


def _premise_inputs(case, kind):
    if case[0] == "causal":
        S, nh, nkv = case[1]
        (q, k, _, _), scale = attention_inputs(kind, 1, 1, S, S, nh, nkv, 128, True, seed=10)
        return q, k, scale, True, MIN_SHARE
    if case[0] == "noncausal":
        S = case[1]
        (q, k, _, _), scale = attention_inputs(kind, 2, 2, S, S, 2, 2, 64, False, seed=11)
        return q, k, scale, False, MIN_SHARE
    nseq, Sq, Skv, nh = CROSS
    (q, k, _, _), scale = attention_inputs(kind, 1, nseq, Sq, Skv, nh, nh, 128, False, seed=12)
    return q, k, scale, False, MIN_SHARE_CROSS


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", [("causal", c) for c in ATT_CAUSAL] + [("noncausal", s) for s in ATT_NONCAUSAL] +
                         [("cross", CROSS)], ids=lambda c: "%s-%s" % (c[0], c[1]))
def test_attention_premise_generators_move_the_running_max(case, kind):
    q, k, scale, causal, min_share = _premise_inputs(case, kind)
    assert_attention_premise(kind, q, k, scale, causal, min_share)


def test_attention_premise_random_scores_never_move_the_max():
    """What the older kernel tests feed the kernel: randn q and k. The lazy max never moves, so O's rescale is not
    exercised by them."""
    gen = torch.Generator().manual_seed(0)
    q, k = (torch.randn(1, 2, 1135, 128, generator=gen).to(BF) for _ in range(2))
    assert moved_share(q, k, 128 ** -0.5, True) == 0.0


# ================================================================================================ GPU: GEMM
FORMS = [(False, False), (False, True), (True, True)]
FORM_IDS = ["fwd", "dgrad", "wgrad"]


def check_gemm(name, a, b, a_mn, b_mn, tile_n, *, seed=0, bias=False, act=0, residual=False, accumulate=False,
               alpha=1.0):
    """Run one GEMM into a column block of a wider buffer; compare with epilogue_ref element by element and check
    that the buffer's other columns are bitwise untouched."""
    from rlaifv_b200 import ops
    M = a.shape[1] if a_mn else a.shape[0]
    N = b.shape[1] if b_mn else b.shape[0]
    gen = torch.Generator().manual_seed(seed + 1000)
    acc, mag = gemm_ref(a, b, a_mn, b_mn)
    typical = mag / math.sqrt(a.shape[0] if a_mn else a.shape[1])
    kw = {"alpha": alpha, "act": act}
    b_t = r_t = None
    if bias:
        b_t = kw["bias"] = torch.randn(N, generator=gen).to(BF).to(DEV)
    if residual:
        rbuf = torch.randn(M, N + 16, generator=gen).to(BF).to(DEV)
        r_t = rbuf[:, 8:8 + N]
        r_t.copy_(bf16(r_t.to(F64) * typical))
        kw["residual"] = r_t
    wide = torch.randn(M, N + 24, generator=gen).to(BF).to(DEV)
    out = wide[:, 8:8 + N]
    if accumulate:
        out.copy_(bf16(out.to(F64) * typical))
        kw["old"] = out.clone()
    before = wide.clone()
    ops.gemm(a, b, out, a_mn=a_mn, b_mn=b_mn, bias=b_t, residual=r_t, act=act, accumulate=accumulate, tile_n=tile_n,
             alpha=alpha)
    torch.cuda.synchronize()
    ref, bound = epilogue_ref(acc, mag, **kw)
    worst = assert_within(name, out, ref, bound)
    assert torch.equal(wide[:, :8], before[:, :8]) and torch.equal(wide[:, 8 + N:], before[:, 8 + N:]), \
        name + ": columns outside the output block changed"
    return out, worst


@pytest.mark.gpu
@pytest.mark.parametrize("tile_n", [128, 256, 512])
@pytest.mark.parametrize("form", range(3), ids=FORM_IDS)
def test_gemm_persistent_walk(form, tile_n):
    """Several tiles per CTA (cluster): the stage / phase carry across tiles and the epilogue overlapping the next
    tile's loads."""
    M, N, K = PERSISTENT
    a_mn, b_mn = FORMS[form]
    M = lda_legal(M, a_mn)
    tiles, slots = gemm_walk(M, N, tile_n, device_sms())
    assert tiles > slots
    gen = torch.Generator().manual_seed(20 + form)
    a, b = gemm_operand(M, K, a_mn, gen), gemm_operand(N, K, b_mn, gen)
    check_gemm("walk %s tile %d" % (FORM_IDS[form], tile_n), a, b, a_mn, b_mn, tile_n)


@pytest.mark.gpu
@pytest.mark.parametrize("form", range(3), ids=FORM_IDS)
def test_gemm_tile_256_and_cluster_512_bit_identical(form):
    """The 128 x 256 tile and the 2-CTA 256 x 256 tile run the same per-element summation: identical bits."""
    from rlaifv_b200 import ops
    M, N, K = PERSISTENT
    a_mn, b_mn = FORMS[form]
    M = lda_legal(M, a_mn)
    gen = torch.Generator().manual_seed(30 + form)
    a, b = gemm_operand(M, K, a_mn, gen), gemm_operand(N, K, b_mn, gen)
    c256 = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, tile_n=256)
    c512 = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, tile_n=512)
    assert torch.equal(c256, c512)


EPILOGUES = {
    "bias_gelu": dict(bias=True, act=1),
    "bias_quick_gelu": dict(bias=True, act=2),
    "bias_residual": dict(bias=True, residual=True),
    "residual": dict(residual=True),
    "accumulate": dict(accumulate=True),
    "accumulate_wgrad": dict(accumulate=True, form=2),
    "alpha": dict(alpha=0.3),
}


@pytest.mark.gpu
@pytest.mark.parametrize("tile_n", [256, 512])
@pytest.mark.parametrize("epi", list(EPILOGUES))
def test_gemm_epilogue_bounds(epi, tile_n):
    kw = dict(EPILOGUES[epi])
    a_mn, b_mn = FORMS[kw.pop("form", 0)]
    M, N, K = EPI_SHAPE
    M = lda_legal(M, a_mn)
    gen = torch.Generator().manual_seed(40)
    a, b = gemm_operand(M, K, a_mn, gen), gemm_operand(N, K, b_mn, gen)
    check_gemm("epilogue %s tile %d" % (epi, tile_n), a, b, a_mn, b_mn, tile_n, seed=41, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("tile_n", [128, 256, 512])
@pytest.mark.parametrize("form", range(3), ids=FORM_IDS)
def test_gemm_strided_operands(form, tile_n):
    """A and B are column blocks of wider NaN-padded buffers (row stride > extent), as the LoRA slices are."""
    M, N, K = STRIDED
    a_mn, b_mn = FORMS[form]
    gen = torch.Generator().manual_seed(50 + form)
    a, b = gemm_operand(M, K, a_mn, gen, pad=40), gemm_operand(N, K, b_mn, gen, pad=40)
    assert a.stride(0) > a.shape[1] and b.stride(0) > b.shape[1]
    check_gemm("strided %s tile %d" % (FORM_IDS[form], tile_n), a, b, a_mn, b_mn, tile_n)


LORA_T, LORA_H, LORA_N = 1100, 520, 776     # tokens, in features, out features
LORA_CASES = ["x_A_n_r", "x_A_n_3r", "t_B_k_r", "dt_A_k_r", "dA_m_r", "dB_n_r"]


@pytest.mark.gpu
@pytest.mark.parametrize("r", [8, 64])
@pytest.mark.parametrize("case", LORA_CASES)
def test_gemm_lora_shapes(case, r):
    """The skinny launches of the LoRA path (model.py): N = r and N = 3r (t = s x A^T, alpha-scaled), K = r
    (t_j B^T with t_j a column block of t, and dt A), M = r (dA = dt^T x) and N = r (dB = dy^T t_j) wgrads."""
    gen = torch.Generator().manual_seed(60 + r)
    t = gemm_operand(LORA_T, 3 * r, False, gen)                  # [T, 3r]: three sub-linears' rank-r blocks
    tj = t[:, r:2 * r]                                           # column block, row stride 3r
    if case == "x_A_n_r":
        args = (gemm_operand(LORA_T, LORA_H, False, gen), gemm_operand(r, LORA_H, False, gen), False, False)
        kw = {"alpha": 0.25}
    elif case == "x_A_n_3r":
        args = (gemm_operand(LORA_T, LORA_H, False, gen), gemm_operand(3 * r, LORA_H, False, gen), False, False)
        kw = {"alpha": 0.25}
    elif case == "t_B_k_r":
        args = (tj, gemm_operand(LORA_N, r, False, gen), False, False)
        kw = {}
    elif case == "dt_A_k_r":
        args = (tj, gemm_operand(LORA_H, r, True, gen), False, True)
        kw = {}
    elif case == "dA_m_r":
        args = (tj, gemm_operand(LORA_H, LORA_T, True, gen), True, True)
        kw = {"accumulate": True}
    else:
        args = (gemm_operand(LORA_N, LORA_T, True, gen), tj, True, True)
        kw = {"accumulate": True}
    check_gemm("lora %s r=%d" % (case, r), *args, 0, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("form", range(3), ids=FORM_IDS)
@pytest.mark.parametrize("N", [256, 264, 520])
@pytest.mark.parametrize("M", [64, 128, 129, 257])
def test_gemm_cluster_corners(M, N, form):
    """The 2-CTA tile on ragged edges: M <= 128 leaves the second CTA of a pair without valid rows, N = 264 / 520
    leave one CTA's multicast half of B mostly out of bounds. The wgrad form rounds M up to a multiple of 8 (lda)."""
    K = 200
    a_mn, b_mn = FORMS[form]
    M = lda_legal(M, a_mn)
    gen = torch.Generator().manual_seed(70 + M + N)
    a, b = gemm_operand(M, K, a_mn, gen), gemm_operand(N, K, b_mn, gen)
    check_gemm("cluster corner %s M=%d N=%d" % (FORM_IDS[form], M, N), a, b, a_mn, b_mn, 512)


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["residual_pointer", "residual_odd_ldr", "bias_pointer"])
def test_gemm_rejects_misaligned_epilogue_operands(what):
    """epilogue_pair reads bias and residual as bf16 pairs: a view that breaks the 4-byte alignment is refused."""
    from rlaifv_b200 import lib, ops
    M, N, K = 256, 256, 64
    a = torch.randn(M, K, device=DEV).to(BF)
    b = torch.randn(N, K, device=DEV).to(BF)
    bias = res = None
    if what == "residual_pointer":
        res = torch.zeros(M, N + 8, device=DEV, dtype=BF)[:, 1:1 + N]
    elif what == "residual_odd_ldr":
        res = torch.zeros(M, N + 1, device=DEV, dtype=BF)[:, :N]
    else:
        bias = torch.zeros(N + 1, device=DEV, dtype=BF)[1:]
    with pytest.raises(lib.B200Error, match="aligned"):
        ops.gemm(a, b, bias=bias, residual=res)


# ================================================================================================ GPU: attention
def _attention_premise_on_device(kind, q, k, scale, causal, min_share):
    assert_attention_premise(kind, q.to(DEV), k.to(DEV), scale, causal, min_share)


def _check_forward(tag, out, lse, r, nseq, Sq, nh, D):
    assert_within(tag + " O", heads(out, nseq, Sq, nh, D), r["o"], r["o_bound"])
    assert_within(tag + " lse", lse, r["lse"], r["lse_bound"])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("S,nh,nkv", ATT_CAUSAL, ids=["S1135", "S2049", "gqa8x2-S1135"])
def test_attention_causal_d128_bounds(S, nh, nkv, kind):
    """Causal self-attention, D = 128: forward, the split backward the model runs (bf16 dQ into the fused dqkv
    buffer) and the fp32-dQ backward. 8 query heads over 2 kv heads is Mistral's group of 4."""
    from rlaifv_b200 import ops
    D, nseq = 128, 1
    (q, k, v, do), scale = attention_inputs(kind, 1, 1, S, S, nh, nkv, D, True, seed=100 + S + nh)
    _attention_premise_on_device(kind, q, k, scale, True, MIN_SHARE)
    H, KV = nh * D, nkv * D
    qkv = torch.cat([rows_of(q), rows_of(k), rows_of(v)], 1).to(DEV)
    q_, k_, v_ = qkv[:, :H], qkv[:, H:H + KV], qkv[:, H + KV:]
    d_out = rows_of(do).to(DEV)
    out, lse = ops.attention_fwd(q_, k_, v_, nseq, S, nh, D, True, scale, n_kv_heads=nkv)
    dqkv = torch.full((S, H + 2 * KV), float("nan"), device=DEV, dtype=BF)
    ops.attention_bwd_split(q_, k_, v_, out, d_out, lse, nseq, S, S, nh, D, True, scale, dqkv[:, :H],
                            dqkv[:, H:H + KV], dqkv[:, H + KV:], n_kv_heads=nkv)
    dq32 = torch.zeros(S, H, device=DEV)
    dkv = torch.full((S, 2 * KV), float("nan"), device=DEV, dtype=BF)
    ops.attention_bwd(q_, k_, v_, out, d_out, lse, nseq, S, nh, D, scale, dq32, dkv[:, :KV], dkv[:, KV:],
                      n_kv_heads=nkv)
    torch.cuda.synchronize()
    qd, kd, vd = (t.to(DEV) for t in (q, k, v))
    r = attention_ref(qd, expand_kv(kd, nh), expand_kv(vd, nh), scale, True, do.to(DEV))
    tag = "causal %s S=%d %d/%d" % (kind, S, nh, nkv)
    _check_forward(tag, out, lse, r, nseq, S, nh, D)
    dq_b = with_output_rounding(r, "dq")
    for key in ("dk", "dv"):
        r[key], r[key + "_t"] = group_sum(r[key], nkv), group_sum(r[key + "_t"], nkv)
    dk_b, dv_b = with_output_rounding(r, "dk"), with_output_rounding(r, "dv")
    assert_within(tag + " split dQ", heads(dqkv[:, :H], nseq, S, nh, D), r["dq"], dq_b)
    assert_within(tag + " split dK", heads(dqkv[:, H:H + KV], nseq, S, nkv, D), r["dk"], dk_b)
    assert_within(tag + " split dV", heads(dqkv[:, H + KV:], nseq, S, nkv, D), r["dv"], dv_b)
    assert_within(tag + " fp32 dQ", heads(dq32, nseq, S, nh, D), r["dq"], dq_b)
    assert_within(tag + " fp32-path dK", heads(dkv[:, :KV], nseq, S, nkv, D), r["dk"], dk_b)
    assert_within(tag + " fp32-path dV", heads(dkv[:, KV:], nseq, S, nkv, D), r["dv"], dv_b)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("S", ATT_NONCAUSAL)
def test_attention_noncausal_d64_forward_bounds(S, kind):
    """The CLIP tower's attention: non-causal, D = 64, ragged last KV tile."""
    from rlaifv_b200 import ops
    D, nseq, nh = 64, 2, 2
    (q, k, v, _), scale = attention_inputs(kind, nseq, nseq, S, S, nh, nh, D, False, seed=200 + S)
    _attention_premise_on_device(kind, q, k, scale, False, MIN_SHARE)
    H = nh * D
    qkv = torch.cat([rows_of(q), rows_of(k), rows_of(v)], 1).to(DEV)
    out, lse = ops.attention_fwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], nseq, S, nh, D, False, scale)
    torch.cuda.synchronize()
    r = attention_ref(q.to(DEV), k.to(DEV), v.to(DEV), scale, False)
    _check_forward("non-causal d64 %s S=%d" % (kind, S), out, lse, r, nseq, S, nh, D)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_cross_attention_shared_queries_bounds(kind):
    """The resampler's cross-attention: 64 learned queries shared by every image over 1025 keys; the backward's fp32
    dQ is the sum over the batch."""
    from rlaifv_b200 import ops
    nseq, Sq, Skv, nh = CROSS
    D = 128
    H = nh * D
    (q, k, v, do), scale = attention_inputs(kind, 1, nseq, Sq, Skv, nh, nh, D, False, seed=300)
    _attention_premise_on_device(kind, q, k, scale, False, MIN_SHARE_CROSS)
    q_ = rows_of(q).to(DEV)
    kv = torch.cat([rows_of(k), rows_of(v)], 1).to(DEV)
    d_out = rows_of(do).to(DEV)
    out, lse = ops.cross_attention_fwd(q_, kv[:, :H], kv[:, H:], nseq, Sq, Skv, nh, D, scale, q_shared=True)
    dq32 = torch.zeros(Sq, H, device=DEV)
    dkv = torch.full((nseq * Skv, 2 * H), float("nan"), device=DEV, dtype=BF)
    ops.cross_attention_bwd(q_, kv[:, :H], kv[:, H:], out, d_out, lse, nseq, Sq, Skv, nh, D, scale, dq32, dkv[:, :H],
                            dkv[:, H:], q_shared=True)
    torch.cuda.synchronize()
    r = attention_ref(q.to(DEV), k.to(DEV), v.to(DEV), scale, False, do.to(DEV))
    tag = "cross %s" % kind
    _check_forward(tag, out, lse, r, nseq, Sq, nh, D)
    r["dq"], r["dq_t"] = r["dq"].sum(0, keepdim=True), r["dq_t"].sum(0, keepdim=True)
    assert_within(tag + " dQ (batch sum)", heads(dq32, 1, Sq, nh, D), r["dq"], with_output_rounding(r, "dq"))
    assert_within(tag + " dK", heads(dkv[:, :H], nseq, Skv, nh, D), r["dk"], with_output_rounding(r, "dk"))
    assert_within(tag + " dV", heads(dkv[:, H:], nseq, Skv, nh, D), r["dv"], with_output_rounding(r, "dv"))


@pytest.mark.gpu
def test_attention_forward_and_split_backward_are_deterministic():
    """No atomics in the forward or the split backward: a second run gives the same bits."""
    from rlaifv_b200 import ops
    S, nh, D = 1135, 2, 128
    H = nh * D
    (q, k, v, do), scale = attention_inputs("rising", 1, 1, S, S, nh, nh, D, True, seed=400)
    qkv = torch.cat([rows_of(q), rows_of(k), rows_of(v)], 1).to(DEV)
    d_out = rows_of(do).to(DEV)
    runs = []
    for _ in range(2):
        out, lse = ops.attention_fwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], 1, S, nh, D, True, scale)
        dqkv = torch.full((S, 3 * H), float("nan"), device=DEV, dtype=BF)
        ops.attention_bwd_split(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], out, d_out, lse, 1, S, S, nh, D, True,
                                scale, dqkv[:, :H], dqkv[:, H:2 * H], dqkv[:, 2 * H:])
        runs.append((out, lse, dqkv))
    torch.cuda.synchronize()
    for x, y in zip(*runs):
        assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["out_pointer", "out_ld", "d_out_pointer"])
def test_attention_backward_rejects_misaligned_out_and_d_out(what):
    """The delta pass reads O and dO rows with 16-byte loads: views that break that alignment are refused before any
    launch."""
    from rlaifv_b200 import lib, ops
    S, nh, D = 128, 1, 128
    qkv = torch.randn(S, 3 * D, device=DEV).to(BF)
    out, lse = ops.attention_fwd(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], 1, S, nh, D, True, D ** -0.5)
    d_out = torch.randn(S, D, device=DEV).to(BF)
    if what == "out_pointer":
        out = torch.zeros(S, D + 8, device=DEV, dtype=BF)[:, 1:1 + D]
    elif what == "out_ld":
        out = torch.zeros(S, D + 4, device=DEV, dtype=BF)[:, :D]
    else:
        d_out = torch.zeros(S, D + 8, device=DEV, dtype=BF)[:, 1:1 + D]
    dqkv = torch.zeros(S, 3 * D, device=DEV, dtype=BF)
    with pytest.raises(lib.B200Error, match="aligned"):
        ops.attention_bwd_split(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], out, d_out, lse, 1, S, S, nh, D, True,
                                D ** -0.5, dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:])
    torch.cuda.synchronize()

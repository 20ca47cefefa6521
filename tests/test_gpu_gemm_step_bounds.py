"""Every GEMM launch of the DPO step against fp64 per element, at the shapes the step itself records.

The launches are recorded, not re-typed: one training step of a one-decoder-layer LLaVA-1.5 policy at the benchmark's
batch (tools/gemm_step_shapes.py record_step_calls), at the 7B and 13B widths, LoRA(r = 64) and full fine-tuning. Each
distinct launch (describe's signature: shapes, strides, layouts, epilogue, K2) is replayed once with crafted operands of
the same shapes and row strides, at the recorded M (9080 rows), and every output element is compared with the fp64
reference of test_gpu_kernel_bounds (gemm_ref, epilogue_ref) or, for the fused SwiGLU backward, with swiglu_bwd_ref of
test_gpu_rowop_bounds applied to the fp64 product. The accumulation term grows with the contraction depth
(acc_term: K runs to 27 648 here).

The inputs make a wrong second source visible. A, A2, B and B2 carry independent power-of-two scales per row and
column; every fourth row of A2 carries 2^BOOST more, so that there the A2 B2 term exceeds |A||B| by 2^6 and more; each
sub-linear's column block of A2 has its own scale (BLOCK_EXP), so that reading block j +- 1 moves the result far
outside its bound. Gates and ups for the SwiGLU backward span [-8, 8], every 16th gate column sits at the zero of
silu' (g = -1.2785). Each replay asserts its premise: the fp64 result without the second source, and with koff moved by
one sub-linear, breaks the bound on every 128 x 256 tile.

Edges beyond the recorded set use the same reference: gemm_dual forward over sub-linears at r = 8 .. 128 (koff not a
multiple of the 64-wide k block for r = 8, 16), with and without residual; the dgrad form with K2 = r, 2r, 3r; the
fused SwiGLU backward at ragged F with W in either layout, with and without a2. Each runs at an M for which gemm_impl's
automatic tile rule picks the 2-CTA 512 tile or the 128 tile, and writes into a column block of a wider buffer whose
other columns are checked bitwise. The rule never picks the 256 tile (test_tile_rule_never_picks_256): gemm_dual and
gemm_swiglu_bwd, which always take the automatic tile, never run it.

The tests without the gpu mark check that the bounds accept the rounded fp64 result and reject planted errors, and
restate the tile rule from gemm.cu. They never load the library.
"""
import math
import os
import re

import pytest
import torch

from test_gpu_kernel_bounds import (ACC, BF, DEV, F64, H100_SMS, _one_row, acc_term, bf16, epilogue_ref, gemm_operand,
                                    gemm_ref, violations, within)
from test_gpu_rowop_bounds import swiglu_bwd_ref

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEMM_CU = os.path.join(REPO, "rlaif-v_b200", "csrc", "gemm.cu")

BOOST = 12                   # extra power of two on every 4th row of A2
BLOCK_EXP = (0, 5, -4)       # power of two on sub-linear s's column block of A2 (s modulo 3)
SILU_ZERO = -1.2785          # silu'(g) = sg (1 + g (1 - sg)) = 0 here
PT_M, PT_N = 128, 256        # the tile of the premises and of the planted errors
REF_ELEMS = 2 ** 25          # elements of one fp64 operand block of the reference (256 MB)


# ================================================================================================ tile rule
def auto_tile(M, N, sms):
    """gemm_impl's automatic tile_n (the caller passes tile_n = 0, as gemm_dual and gemm_swiglu_bwd always do)."""
    tiles256 = -(-M // 128) * -(-N // 256)
    tiles2 = -(-M // 256) * -(-N // 256)
    if N >= 256 and tiles2 >= sms // 2:
        return 512
    return 256 if N >= 256 and tiles256 >= sms else 128


def ntile(tile_n):
    return 256 if tile_n == 512 else tile_n


# ================================================================================================ operands
def second_operand(M, width, r, gen, pad=0, device=DEV):
    """A2 [M, width] (K-major): gemm_operand's row scales, 2^BOOST more on every 4th row, column block s (width r) of
    sub-linear s scaled by 2^BLOCK_EXP[s % 3]."""
    a2 = gemm_operand(M, width, False, gen, pad=pad, device=device)
    row = torch.where(torch.arange(M, device=a2.device) % 4 == 0, 2.0 ** BOOST, 1.0)
    col = torch.exp2(torch.tensor([float(BLOCK_EXP[(j // r) % 3]) for j in range(width)], device=a2.device))
    a2.copy_((a2.to(F64) * row[:, None] * col[None, :]).to(BF))
    return a2


def glu_operand(M, F, gen, pad=0, device=DEV):
    """[gate | up] [M, 2F]: both uniform in [-8, 8]; every 16th gate column at bf16 values around the zero of silu'."""
    x = (torch.rand(M, 2 * F, generator=gen, dtype=F64, device=gen.device) * 16 - 8)
    x[:, 3:F:16] = SILU_ZERO + (torch.randint(-3, 4, x[:, 3:F:16].shape, generator=gen, device=gen.device) * 2.0 ** -7)
    x = x.to(BF)
    if not pad:
        return x.to(device)
    buf = torch.full((M, 2 * F + pad), float("nan"), dtype=BF, device=gen.device)
    buf[:, 8:8 + 2 * F] = x
    return buf.to(device)[:, 8:8 + 2 * F]


def logical(t, mn):
    return t.t() if mn else t


def typical(a, a_mn, b, b_mn, K):
    """Rank-one estimate of |C| (row norms of op(A) and op(B) over sqrt K): the scale of crafted residuals."""
    na = logical(a, a_mn).to(F64).norm(dim=1)
    nb = logical(b, b_mn).to(F64).norm(dim=1)
    return na[:, None] * nb[None, :] / math.sqrt(K)


# ================================================================================================ one launch
def spec_of(name, a, kw, r):
    """Launch description of one recorded call: every shape, row stride, layout and epilogue argument, no values."""
    s = {"fn": name}
    if name == "gemm":
        A, B = a[0], a[1]
        out = r
        s.update(a_mn=kw.get("a_mn", False), b_mn=kw.get("b_mn", False), act=kw.get("act", 0),
                 accumulate=bool(kw.get("accumulate", False)), tile_n=kw.get("tile_n", 0), alpha=kw.get("alpha", 1.0),
                 bias=kw.get("bias") is not None)
        res = kw.get("residual")
    elif name == "gemm_dual":
        A, B, A2, B2, out = a[:5]
        s.update(a_mn=False, b_mn=kw.get("b_mn", False), K2=kw["k2"], r=kw["r"], n_sub=kw.get("n_sub", 0),
                 accumulate=bool(kw.get("accumulate", False)), a2_w=A2.shape[1], lda2=A2.stride(0),
                 ldb2=B2.stride(0))
        res = kw.get("residual")
    else:
        A, B, gu, out = a[:4]
        A2 = kw.get("a2")
        s.update(a_mn=False, b_mn=kw.get("b_mn", True), ld_gu=gu.stride(0))
        if A2 is not None:
            s.update(K2=A2.shape[1], r=A2.shape[1], a2_w=A2.shape[1], lda2=A2.stride(0), ldb2=kw["b2"].stride(0))
        res = None
    M = A.shape[1] if s["a_mn"] else A.shape[0]
    K = A.shape[0] if s["a_mn"] else A.shape[1]
    N = (B.shape[1] if s["b_mn"] else B.shape[0])
    s.update(M=M, N=N, K=K, lda=A.stride(0), ldb=B.stride(0), ldc=out.stride(0))
    if res is not None:
        s["ldr"] = res.stride(0)
    return s


def _pad(ld, cols):
    p = ld - cols
    assert p == 0 or p >= 8, (ld, cols)
    return p


def build_case(spec, seed):
    """Crafted operands of a launch description on the GPU (CUDA generator seeded with `seed`), its output in a buffer
    of the description's row stride (ldc; column 8 onwards when the stride leaves room), and the launch itself."""
    from rlaifv_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(seed)
    M, N, K, a_mn, b_mn = spec["M"], spec["N"], spec["K"], spec["a_mn"], spec["b_mn"]
    glu = spec["fn"] == "gemm_swiglu_bwd"
    t = {}
    t["a"] = gemm_operand(M, K, a_mn, gen, pad=_pad(spec["lda"], M if a_mn else K))
    t["b"] = gemm_operand(N, K, b_mn, gen, pad=_pad(spec["ldb"], N if b_mn else K))
    if spec.get("K2"):
        K2 = spec["K2"]
        t["a2"] = second_operand(M, spec["a2_w"], spec["r"], gen, pad=_pad(spec["lda2"], spec["a2_w"]))
        t["b2"] = gemm_operand(N, K2, b_mn, gen, pad=_pad(spec["ldb2"], N if b_mn else K2))
    width = 2 * N if glu else N
    if glu:
        t["gu"] = glu_operand(M, N, gen, pad=_pad(spec["ld_gu"], 2 * N))
    ldc = spec["ldc"]
    off = 8 if ldc - width >= 8 else 0
    wide = torch.randn(M, ldc, generator=gen, device=DEV).to(BF)
    t["out"] = wide[:, off:off + width]
    t["wide"], t["off"] = wide, off
    if spec.get("bias"):
        t["bias"] = torch.randn(N, generator=gen, device=DEV).to(BF)
    if "ldr" in spec or spec.get("accumulate"):
        typ = typical(t["a"], a_mn, t["b"], b_mn, K)
        if "ldr" in spec:
            rb = torch.randn(M, spec["ldr"], generator=gen, device=DEV).to(BF)
            roff = 8 if spec["ldr"] - N >= 8 else 0
            t["residual"] = rb[:, roff:roff + N]
            t["residual"].copy_(bf16(t["residual"].to(F64) * typ))
        if spec.get("accumulate"):
            t["out"].copy_(bf16(t["out"].to(F64) * typ))
            t["old"] = t["out"].clone()
        del typ
    t["before"] = wide.clone()

    def launch():
        if spec["fn"] == "gemm":
            ops.gemm(t["a"], t["b"], t["out"], a_mn=a_mn, b_mn=b_mn, bias=t.get("bias"), residual=t.get("residual"),
                     act=spec.get("act", 0), accumulate=spec.get("accumulate", False), tile_n=spec.get("tile_n", 0),
                     alpha=spec.get("alpha", 1.0))
        elif spec["fn"] == "gemm_dual":
            ops.gemm_dual(t["a"], t["b"], t["a2"], t["b2"], t["out"], k2=spec["K2"], r=spec["r"], n_sub=spec["n_sub"],
                          b_mn=b_mn, residual=t.get("residual"), accumulate=spec.get("accumulate", False))
        else:
            ops.gemm_swiglu_bwd(t["a"], t["b"], t["gu"], t["out"], b_mn=b_mn, a2=t.get("a2"), b2=t.get("b2"))
    return t, launch


def shifted_blocks(a2, r, g):
    """A2 with sub-linear s's column block replaced by block s + 1 (the last by the one before it): the operand a
    kernel whose koff is one sub-linear off reads."""
    src = [s + 1 for s in range(g - 1)] + [g - 2]
    return torch.cat([a2[:, s * r:(s + 1) * r] for s in src], 1)


class TileMap:
    """Per 128 x 256 output tile: whether a planted result breaks the bound somewhere in it."""

    def __init__(self, M, N):
        self.hit = torch.zeros(-(-M // PT_M), -(-N // PT_N), dtype=torch.bool, device=DEV)

    def add(self, bad, r0, c0):
        rb, cb = bad.shape
        pr, pc = -(-rb // PT_M) * PT_M - rb, -(-cb // PT_N) * PT_N - cb
        b = torch.nn.functional.pad(bad.to(torch.uint8), (0, pc, 0, pr))
        t = b.reshape(b.shape[0] // PT_M, PT_M, b.shape[1] // PT_N, PT_N).amax(3).amax(1) > 0
        self.hit[r0 // PT_M:r0 // PT_M + t.shape[0], c0 // PT_N:c0 // PT_N + t.shape[1]] |= t

    def all(self):
        return bool(self.hit.all())


def check_case(name, spec, t):
    """Blocked fp64 reference of one launch against its output; every element within its bound, the columns outside
    the output block untouched, and the premises of a second source. Returns the worst err / bound."""
    M, N, K, a_mn, b_mn = spec["M"], spec["N"], spec["K"], spec["a_mn"], spec["b_mn"]
    glu = spec["fn"] == "gemm_swiglu_bwd"
    K2, r, n_sub = spec.get("K2", 0), spec.get("r", 0), spec.get("n_sub", 0)
    depth = 16 * (-(-K // 16) + -(-K2 // 16))
    blk = max(256, min(4096, REF_ELEMS // max(K, 1) // 256 * 256))      # columns (and B rows) per block
    rblk = min(2048, blk)                                                 # rows (and A rows) per block
    g = N // n_sub if n_sub else 0
    premises = {"second source dropped": TileMap(M, N)} if K2 else {}
    if g >= 2:
        premises["koff one sub-linear off"] = TileMap(M, N)
    dominant = 0
    a, b = t["a"], t["b"]
    a0, b0 = a[:, :0], (b[:0] if b_mn else b[:, :0])
    worst, nbad, first = 0.0, 0, None
    for r0 in range(0, M, rblk):
        rows = slice(r0, min(M, r0 + rblk))
        for c0 in range(0, N, blk):
            cols = slice(c0, min(N, c0 + blk))
            c, mag = gemm_ref(a, b, a_mn, b_mn, rows=rows, cols=cols)
            sec = {}
            if K2:
                c2, m2 = gemm_ref(a0, b0, False, b_mn, a2=t["a2"], b2=t["b2"], k2=K2, r=r, n_sub=n_sub, rows=rows,
                                  cols=cols)
                dominant += int((m2 >= 2.0 ** 6 * mag).sum())
                sec["second source dropped"] = c
                if g >= 2:
                    sec["koff one sub-linear off"] = c + gemm_ref(
                        a0, b0, False, b_mn, a2=shifted_blocks(t["a2"], r, g), b2=t["b2"], k2=K2, r=r,
                        n_sub=n_sub, rows=rows, cols=cols)[0]
                c, mag = c + c2, mag + m2
                del c2, m2
            if glu:
                _, e_d = epilogue_ref(c, mag, k=depth)
                gu = t["gu"][rows]
                gub = torch.cat([gu[:, cols], gu[:, N + cols.start:N + cols.stop]], 1)
                (dg, bdg), (du, bdu) = swiglu_bwd_ref(gub, c, e_dact=e_d, fast_div=True)
                checks = [(t["out"][rows, cols], dg, bdg, c0), (t["out"][rows, N + cols.start:N + cols.stop], du, bdu,
                                                                  N + c0)]
                for key, v in sec.items():
                    _, e_v = epilogue_ref(v, mag, k=depth)
                    (pg, _), _ = swiglu_bwd_ref(gub, v, e_dact=e_v, fast_div=True)
                    premises[key].add(~(((bf16(pg) - dg).abs()) <= bdg), r0, c0)
            else:
                kw = {"k": depth, "alpha": spec.get("alpha", 1.0), "act": spec.get("act", 0)}
                if "bias" in t:
                    kw["bias"] = t["bias"][cols]
                if "residual" in t:
                    kw["residual"] = t["residual"][rows, cols]
                if "old" in t:
                    kw["old"] = t["old"][rows, cols]
                ref, bound = epilogue_ref(c, mag, **kw)
                checks = [(t["out"][rows, cols], ref, bound, c0)]
                for key, v in sec.items():
                    pref, _ = epilogue_ref(v, mag, **kw)
                    premises[key].add(~((bf16(pref) - ref).abs() <= bound), r0, c0)
            for got, ref, bound, col0 in checks:
                bad, ratio = violations(got, ref, bound)
                worst = max(worst, float(ratio.nan_to_num(nan=float("inf")).max()))
                if bool(bad.any()):
                    nbad += int(bad.sum())
                    if first is None:
                        i, j = bad.nonzero()[0].tolist()
                        first = (r0 + i, col0 + j, float(got[i, j]), float(ref[i, j]), float(bound[i, j]))
            del c, mag, sec, checks
    print("err/bound %-60s %.3g" % (name, worst))
    assert nbad == 0, "%s: %d elements outside their bound; first at (%d, %d): got %r, fp64 %r, bound %r" % (
        (name, nbad) + first)
    w, off, width = t["wide"], t["off"], t["out"].shape[1]
    assert torch.equal(w[:, :off], t["before"][:, :off]) and torch.equal(w[:, off + width:],
                                                                          t["before"][:, off + width:]), \
        name + ": columns outside the output block changed"
    for key, tm in premises.items():
        assert tm.all(), "%s: premise: the fp64 result with the %s stays within the bound on some tile" % (name, key)
    if K2:
        assert dominant >= 0.02 * M * N, "%s: premise: A2 B2 exceeds 2^6 |A||B| on only %d elements" % (name, dominant)
    return worst


def run_case(name, spec, seed):
    t, launch = build_case(spec, seed)
    launch()
    torch.cuda.synchronize()
    return check_case(name, spec, t)


# ================================================================================================ CPU: bounds and rule
def _cpu_dual(gen, M=256, n_sub=256, g=3, K=192, r=16):
    N = g * n_sub
    a = gemm_operand(M, K, False, gen, device="cpu")
    b = gemm_operand(N, K, False, gen, device="cpu")
    a2 = second_operand(M, g * r, r, gen, device="cpu")
    b2 = gemm_operand(N, r, False, gen, device="cpu")
    return a, b, a2, b2, dict(N=N, K=K, r=r, n_sub=n_sub, g=g)


def test_dual_bound_accepts_rounded_fp64_and_rejects_planted_errors():
    gen = torch.Generator().manual_seed(11)
    a, b, a2, b2, p = _cpu_dual(gen)
    K, r, n_sub, g = p["K"], p["r"], p["n_sub"], p["g"]
    depth = K + r
    c, mag = gemm_ref(a, b, False, False, a2=a2, b2=b2, k2=r, r=r, n_sub=n_sub)
    base, _ = gemm_ref(a, b, False, False)
    shifted, _ = gemm_ref(a, b, False, False, a2=shifted_blocks(a2, r, g), b2=b2, k2=r, r=r, n_sub=n_sub)
    ref, bound = epilogue_ref(c, mag, k=depth)
    assert within(bf16(ref), ref, bound)
    tile = (slice(PT_M, 2 * PT_M), slice(PT_N, 2 * PT_N))           # second row of tiles, sub-linear 1
    for planted in (shifted, base):
        bad = bf16(ref).clone()
        bad[tile] = bf16(planted[tile])
        assert not within(bad, ref, bound)
    row = int(ref.abs().amax(1).argmin())
    assert not within(_one_row(bf16(ref), row), ref, bound)
    # the residual form rejects the same planted tiles
    res = bf16(torch.randn(c.shape, generator=gen, dtype=F64) * mag / math.sqrt(K))
    ref, bound = epilogue_ref(c, mag, k=depth, residual=res)
    assert within(bf16(ref), ref, bound)
    for planted in (shifted, base):
        bad = bf16(ref).clone()
        bad[tile] = bf16(epilogue_ref(planted, mag, k=depth, residual=res)[0][tile])
        assert not within(bad, ref, bound)


def test_dual_reference_reads_koff_per_sub_linear():
    """gemm_ref's second source against an explicit loop over output columns."""
    gen = torch.Generator().manual_seed(12)
    a, b, a2, b2, p = _cpu_dual(gen, M=40, n_sub=16, g=3, K=24, r=8)
    c, _ = gemm_ref(a, b, False, False, a2=a2, b2=b2, k2=p["r"], r=p["r"], n_sub=p["n_sub"])
    x, y, x2, y2 = (t.to(F64) for t in (a, b, a2, b2))
    for n in range(p["N"]):
        koff = (n // p["n_sub"]) * p["r"]
        col = x @ y[n] + x2[:, koff:koff + p["r"]] @ y2[n]
        assert torch.allclose(c[:, n], col, rtol=1e-12, atol=0)


def _cpu_glu(gen, M=256, F=320, K=192, k2=16):
    dy = gemm_operand(M, K, False, gen, device="cpu")
    w = gemm_operand(F, K, True, gen, device="cpu")
    a2 = second_operand(M, k2, k2, gen, device="cpu")
    b2 = gemm_operand(F, k2, True, gen, device="cpu")
    gu = glu_operand(M, F, gen, device="cpu")
    c, mag = gemm_ref(dy, w, False, True, a2=a2, b2=b2, k2=k2, r=k2)
    return c, mag, gu, K + k2


def _glu(gu, c, mag, depth):
    _, e_d = epilogue_ref(c, mag, k=depth)
    return swiglu_bwd_ref(gu, c, e_dact=e_d, fast_div=True)


def test_swiglu_bwd_bound_accepts_rounded_fp64_and_rejects_planted_errors():
    gen = torch.Generator().manual_seed(13)
    c, mag, gu, depth = _cpu_glu(gen)
    F = c.shape[1]
    (dg, bdg), (du, bdu) = _glu(gu, c, mag, depth)
    assert within(bf16(dg), dg, bdg) and within(bf16(du), du, bdu)
    sub = slice(64, 128)
    swapped = gu.clone()
    swapped[:, :F], swapped[:, F:] = gu[:, F:], gu[:, :F]
    (sg, _), (su, _) = _glu(swapped, c, mag, depth)
    neighbour = c.clone()
    neighbour[:, sub] = c[:, 128:192]
    (ng, _), (nu, _) = _glu(gu, neighbour, mag, depth)
    for pg, pu in ((sg, su), (ng, nu)):
        bad_g, bad_u = bf16(dg).clone(), bf16(du).clone()
        bad_g[:, sub], bad_u[:, sub] = bf16(pg[:, sub]), bf16(pu[:, sub])
        assert not within(bad_g, dg, bdg) and not within(bad_u, du, bdu)
    for ref, bd in ((dg, bdg), (du, bdu)):
        row = int(ref.abs().amax(1).argmin())
        assert not within(_one_row(bf16(ref), row), ref, bd)


def test_swiglu_premise_gates_reach_the_zero_of_silu_derivative():
    gen = torch.Generator().manual_seed(14)
    gu = glu_operand(64, 256, gen, device="cpu").to(F64)
    g = gu[:, :256]
    s = torch.sigmoid(g)
    d = s * (1 + g * (1 - s))
    assert float(g.min()) < -7.5 and float(g.max()) > 7.5
    assert bool(((d[:, 3::16]).abs() < 2.0 ** -6).any()) and bool((d[:, 3::16] < 0).any()) and \
        bool((d[:, 3::16] > 0).any())


def test_acc_term_keeps_the_shallow_bound_and_grows_past_k_4096():
    assert acc_term() == acc_term(520) == acc_term(4096) == ACC
    assert acc_term(4096 + 64) > ACC
    assert acc_term(27648) == 1728 * 2.0 ** -22 and acc_term(27648 + 64) == 1732 * 2.0 ** -22


def test_tile_rule_restates_gemm_cu():
    """auto_tile restates gemm_impl's rule; this reads it there, so a changed rule fails here instead of leaving the
    tile premises of the GPU cases computed from a stale copy."""
    src = open(GEMM_CU).read()
    assert re.search(r"const long long tiles256 = \(long long\)\(\(M \+ 127\) / 128\) \* \(\(N \+ 255\) / 256\);"
                     r"\s*const long long tiles2 = \(long long\)\(\(M \+ 255\) / 256\) \* \(\(N \+ 255\) / 256\);"
                     r"\s*if \(N >= 256 && tiles2 >= num_sms\(\) / 2\) bn = 512;"
                     r"\s*else bn = \(N >= 256 && tiles256 >= num_sms\(\)\) \? 256 : 128;", src)
    assert "const int ntile = bn == 512 ? 256 : bn;" in src
    assert "n_sub == 0 || n_sub % ntile == 0" in src
    for fn, tile_arg in (("rlaifv_gemm_bf16_swiglu_bwd", "nullptr, nullptr, 0, 0, 0, 0, 1.0f, stream"),
                         ("rlaifv_gemm_bf16_dual", "residual, ldr, act, accumulate, 0,")):
        body = src[src.index('extern "C" int ' + fn):]
        assert tile_arg in body[:body.index("\n}\n")], fn          # tile_n = 0: the automatic rule


def test_tile_rule_never_picks_256():
    """tiles256 <= 2 tiles2, so tiles256 >= sms implies tiles2 >= sms / 2: whenever the 256 tile qualifies, the 2-CTA
    tile is taken first. The automatic launches (every gemm_dual and gemm_swiglu_bwd) run at 512 or 128 only."""
    for sms in (132, 114, 133):
        for M in range(1, 20000, 37):
            for N in (256, 264, 512, 1088, 1216, 4096):
                assert auto_tile(M, N, sms) != 256


# the edge cases: (M, tile) pairs chosen against auto_tile at 132 SMs
DUAL_FWD = {512: (5532, 256), 128: (3000, 384)}           # tile: (M, n_sub); N = 3 n_sub, K = 1000
DUAL_DGRAD = {512: 3500, 128: 3000}                       # N = 1280, K = 1536
GLU_M = {512: 3500, 128: 3000}                            # K = 1000


def test_edge_premises_pick_the_intended_tile():
    for tile, (M, n_sub) in DUAL_FWD.items():
        assert auto_tile(M, 3 * n_sub, H100_SMS) == tile and n_sub % ntile(tile) == 0
    assert DUAL_FWD[128][1] % 256 != 0                    # the 128 tile with a sub-linear width the 256 tile refuses
    for tile, M in DUAL_DGRAD.items():
        assert auto_tile(M, 1280, H100_SMS) == tile
    for tile, M in GLU_M.items():
        for F in (1088, 1216):
            assert auto_tile(M, F, H100_SMS) == tile and F % 256 != 0 and F % 64 == 0


# ================================================================================================ GPU: recorded launches
CONFIGS = [("7b", True), ("7b", False), ("13b", True), ("13b", False)]


@pytest.fixture(scope="module", params=CONFIGS, ids=["%s-%s" % (d, "lora" if lora else "full") for d, lora in CONFIGS])
def recorded(request):
    """(dims, lora, distinct launch descriptions) of one recorded training step; asserts the 8 named frozen-base
    shapes of the decoder are among them, at the decoder's M."""
    from tools import gemm_step_shapes as gs
    dims_name, lora = request.param
    dims = gs.DIMS[dims_name]
    calls, keep = gs.record_step_calls(dims, lora=lora)
    uniq = {}
    for name, a, kw, r in calls:
        sig, d = gs.describe(name, a, kw, r)
        if sig not in uniq:
            uniq[sig] = (d, spec_of(name, a, kw, r))
    del calls, keep
    torch.cuda.empty_cache()
    launches = list(uniq.values())
    m_dec = {d["M"] for d, _ in launches if d["fn"] == "gemm_swiglu_bwd"}
    assert len(m_dec) == 1
    names = {gs.shape_name(d, dims, lora) for d, _ in launches if d["M"] in m_dec}
    want = set(gs.shape_names(dims["hidden_size"], dims["intermediate_size"], lora).values())
    assert want <= names, sorted(want - names)
    fns = {d["fn"] for d, _ in launches}
    assert fns == ({"gemm", "gemm_dual", "gemm_swiglu_bwd"} if lora else {"gemm", "gemm_swiglu_bwd"})
    print("recorded %s %s: %d distinct GEMM launches at M = %d" % (dims_name, "lora" if lora else "full",
                                                                   len(launches), m_dec.pop()))
    return dims_name, lora, launches


@pytest.mark.gpu
def test_recorded_step_launches_within_fp64_bounds(recorded):
    dims_name, lora, launches = recorded
    failures = []
    for i, (d, spec) in enumerate(launches):
        name = "%s %s %s M=%d N=%d K=%d+%d A %s B %s %s" % (dims_name, "lora" if lora else "full", d["fn"], d["M"],
                                                             d["N"], d["K"], d["K2"], d["A"], d["B"], d["epilogue"])
        if d["fn"] == "gemm":
            name += "".join(" %s" % k for k in ("alpha", "act") if spec.get(k) not in (None, 0, 1.0))
        try:
            run_case(name, spec, seed=1000 + i)
        except AssertionError as e:
            print("FAILED", e)
            failures.append(str(e).split("\n")[0])
        torch.cuda.empty_cache()
    assert not failures, "\n".join(failures)


# ================================================================================================ GPU: edges
def _edge_spec(fn, M, N, K, **kw):
    s = dict(fn=fn, M=M, N=N, K=K, a_mn=False, lda=K + 16, ldb=K, accumulate=False)
    s.update(kw)
    s["ldc"] = (2 * N if fn == "gemm_swiglu_bwd" else N) + 24
    return s


def _assert_tile(spec, tile):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert auto_tile(spec["M"], spec["N"], sms) == tile
    if spec.get("n_sub"):
        assert spec["n_sub"] % ntile(tile) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("tile", [512, 128])
@pytest.mark.parametrize("residual", [False, True], ids=["plain", "residual"])
@pytest.mark.parametrize("r", [8, 16, 64, 128])
def test_dual_forward_over_sub_linears(r, residual, tile):
    M, n_sub = DUAL_FWD[tile]
    N, K = 3 * n_sub, 1000
    spec = _edge_spec("gemm_dual", M, N, K, b_mn=False, K2=r, r=r, n_sub=n_sub, a2_w=3 * r, lda2=3 * r, ldb2=r)
    if residual:
        spec["ldr"] = N + 16
    _assert_tile(spec, tile)
    run_case("dual fwd r=%d %s tile %d" % (r, "residual" if residual else "plain", tile), spec, seed=r + tile)


@pytest.mark.gpu
@pytest.mark.parametrize("tile", [512, 128])
@pytest.mark.parametrize("mult", [1, 2, 3])
@pytest.mark.parametrize("r", [8, 64])
def test_dual_dgrad_second_source_depths(r, mult, tile):
    M, N, K = DUAL_DGRAD[tile], 1280, 1536
    k2 = mult * r
    spec = _edge_spec("gemm_dual", M, N, K, b_mn=True, ldb=N, K2=k2, r=r, n_sub=0, a2_w=k2, lda2=k2, ldb2=N)
    _assert_tile(spec, tile)
    run_case("dual dgrad K2=%d (r=%d) tile %d" % (k2, r, tile), spec, seed=100 + k2 + tile)


@pytest.mark.gpu
@pytest.mark.parametrize("tile", [512, 128])
@pytest.mark.parametrize("second", [False, True], ids=["plain", "a2"])
@pytest.mark.parametrize("b_mn", [False, True], ids=["W_K_major", "W_MN_major"])
@pytest.mark.parametrize("F", [1088, 1216])
def test_swiglu_bwd_ragged_f(F, b_mn, second, tile):
    M, K = GLU_M[tile], 1000
    spec = _edge_spec("gemm_swiglu_bwd", M, F, K, b_mn=b_mn, ldb=F if b_mn else K, ld_gu=2 * F + 40)
    if second:
        spec.update(K2=16, r=16, a2_w=16, lda2=16, ldb2=F if b_mn else 16)
    _assert_tile(spec, tile)
    run_case("swiglu_bwd F=%d W %s%s tile %d" % (F, "MN" if b_mn else "K", " a2" if second else "", tile), spec,
             seed=200 + F + tile + 2 * b_mn + second)

"""CPU reference of the FP8 frozen-base format (DESIGN.md §3 "FP8 frozen base"; include/rlaifv_b200.h).

A tile (1 x 128 of an operand row, or a 128 x 128 block of a weight) with amax = max|x| has the scale s = 2^e, e the
smallest integer with amax <= 448 * 2^e clamped to [-126, 127] (s = 1 for amax = 0), and the codes RNE_e4m3(x / s).
x / s is exact and |x / s| <= 448, so torch's float8_e4m3fn cast (round to nearest even; NaN past 448 instead of
saturating) gives every code. Also the fp64 GEMM over the dequantized operands and the fp32 scale products the
kernel promotes with.
"""
import torch

E4M3 = torch.float8_e4m3fn
E4M3_MAX = 448.0


def scale_exp(amax):
    """e of each amax (float tensor): amax = m * 2^E, m in [0.5, 1); 448 = 0.875 * 2^9."""
    m, E = torch.frexp(amax.float())
    e = torch.where(m <= 0.875, E - 9, E - 8)
    e = torch.where(amax > 0, e, torch.zeros_like(e))
    return e.clamp(-126, 127)


def _codes(x, e):
    """RNE_e4m3(x / 2^e) with e broadcast over x (x / 2^e exact in fp64, then one rounding)."""
    v = torch.ldexp(x.double(), -e.double()).float()
    assert float(v.abs().max()) <= E4M3_MAX if v.numel() else True
    return v.to(E4M3)


def quant_rows(x):
    """x [M, K] (bf16 values) -> (codes [M, K] e4m3, scales [K/128, M] fp32)."""
    M, K = x.shape
    assert K % 128 == 0
    t = x.float().view(M, K // 128, 128)
    e = scale_exp(t.abs().amax(dim=2))                       # [M, K/128]
    q = _codes(t, e[:, :, None]).view(M, K)
    return q, torch.ldexp(torch.ones_like(e, dtype=torch.float32), e.float()).t().contiguous()


def quant_blocks(w):
    """W [N, K] -> (codes [N, K], transposed codes [K, N], block scales [N/128, K/128] fp32)."""
    N, K = w.shape
    assert N % 128 == 0 and K % 128 == 0
    t = w.float().view(N // 128, 128, K // 128, 128)
    e = scale_exp(t.abs().amax(dim=(1, 3)))                  # [N/128, K/128]
    q = _codes(t, e[:, None, :, None]).view(N, K)
    return q, q.t().contiguous(), torch.ldexp(torch.ones_like(e, dtype=torch.float32), e.float())


def dequant_rows(q, s):
    """fp64 [M, K] of row codes and their scales [K/128, >= M]."""
    M, K = q.shape
    return (q.double().view(M, K // 128, 128) * s[:, :M].t().double()[:, :, None]).view(M, K)


def dequant_blocks(q, s):
    N, K = q.shape
    return (q.double().view(N // 128, 128, K // 128, 128) * s.double()[:, None, :, None]).view(N, K)


def gemm_ref(qa, sa, qw, sw, dgrad=False):
    """fp64 C of the FP8 product over the codes and scales of A and of a weight W [N_w, K_w]: forward C = A W^T
    (A [M, K_w]); dgrad C = A W (A [M, N_w]). Also returns sum |a b| of each element (fp64 over the dequantized
    operands), the magnitude the per-K-block accumulation error scales with."""
    a = dequant_rows(qa, sa)
    w = dequant_blocks(qw, sw)
    b = w.t() if dgrad else w                                # [N_out, K_contraction]
    return a @ b.t(), a.abs() @ b.abs().t()


# Error bound of one gemm_fp8 output element (tests/test_gpu_fp8_base.py), three terms:
#  - the tensor cores' FP8 accumulation inside a K-block: EPS_BLK * sum |a b|. The wgmma e4m3 accumulator's precision
#    is reduced and undocumented; on an H100 the largest error beyond the other two terms was 7.2e-4 * sum |a b|
#    (2^-10.4, at K = 1024), so EPS_BLK = 2^-9 leaves a factor of 2.7;
#  - the fp32 promotion: one FMA rounding per K-block, at most ceil(K / 128) * 2^-24 * sum |a b|; and the bf16 second
#    source's fp32 accumulation, max(2^-14, ceil(K2 / 16) * 2^-22) * sum |a2 b2| (the bf16 GEMM's acc_term);
#  - the epilogue: the bf16 rounding of the result (half an ulp, at most 2^-8 relative), after the residual add too.
EPS_BLK = 2.0 ** -9


def acc_bound(s1, K, s2=None, K2=0):
    e = (EPS_BLK + -(-K // 128) * 2.0 ** -24) * s1
    if s2 is not None:
        e = e + max(2.0 ** -14, -(-K2 // 16) * 2.0 ** -22) * s2
    return e


def epilogue_bound(ref, acc_err, residual=None):
    """Bound of |out - ref_out| for C = bf16(acc) (residual None) or bf16(bf16(acc) + residual); ref fp64."""
    e1 = acc_err + 2.0 ** -8 * (ref.abs() + acc_err)
    if residual is None:
        return e1
    return e1 + 2.0 ** -8 * ((ref + residual.double()).abs() + e1)


def swiglu_bwd_ref(d, d_err, gu):
    """fp64 d[gate | up] of the SwiGLU backward for d(act) = d (fp64) known within d_err, gate|up [M, 2F] bf16 ->
    (reference [M, 2F], bound [M, 2F]): bf16 rounding of each result, fp32 math (__expf, __fdividef) within 2^-18."""
    F = d.shape[1]
    g, u = gu[:, :F].double(), gu[:, F:].double()
    sg = torch.sigmoid(g)
    kg, ku = u * sg * (1 + g * (1 - sg)), g * sg
    ref = torch.cat([d * kg, d * ku], 1)
    dd = d.abs() + d_err
    e = torch.cat([d_err * kg.abs() + 2.0 ** -8 * (dd * kg.abs()), d_err * ku.abs() + 2.0 ** -8 * (dd * ku.abs())], 1)
    return ref, e + 2.0 ** -8 * ref.abs() + 2.0 ** -18 * torch.cat([dd * kg.abs(), dd * ku.abs()], 1)

"""Row kernels of rowops.cu against fp64 references with per-element error bounds, at the DPO step's shapes.

The norms, SwiGLU, GELU, the column sums, the log-prob head and its reductions, the DPO loss, AdamW and the fp32 ->
bf16 conversions are compared element by element with the same operation evaluated in fp64 on the same inputs. Each
bound is the fp64 computation repeated on magnitudes, times the roundings the kernel performs, plus one ulp of the
output type where the kernel rounds its output. Conventions:
  - u = 2^-24 (fp32 unit roundoff). An fp32 sum is carried as gamma_n * sum |terms|, gamma_n = n u / (1 - n u), where n
    is the most roundings any one term passes through on its way to the result: the kernel's summation tree (a thread's
    serial sum over its chunks, then the two five-level warp trees of block_sum2) bounds n far below the term count
    (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., section 4.2). With n = H instead, the LayerNorm
    bound would be loose enough to admit the one-pass variance's error on offset rows.
  - Elementary functions, from the CUDA C++ Programming Guide's accuracy tables (the build has no --use_fast_math):
    __expf(x) 2 + floor(|1.173 x|) ulp, expf / erff 2 ulp, logf / log1pf 1 ulp, rsqrtf 2 ulp; sqrtf and division are
    correctly rounded. One ulp of an fp32 result y is at most 2^-23 |y|. __expf flushes results below 2^-126 to zero
    (ex2.approx.ftz): an absolute 2^-126 where it enters.
  - Where the kernel rounds an intermediate to bf16 (RMSNorm's normalised row, SwiGLU's silu) the reference does not:
    the rounding costs one bf16 ulp of the intermediate, carried through the later steps.

Inputs reach the paths the kernels branch on: rows scaled by powers of two 2^-6 .. 2^6 (exact in bf16, so an error
confined to one small row is large next to that row's bound), LayerNorm rows whose mean is 500 times their standard
deviation, SwiGLU gates where __expf(-g) overflows, peaked and label-at-minimum log-prob rows. The CPU tests check that
every bound accepts the fp64 result rounded to the output type and rejects a 2^-5 relative error in the row with the
smallest values and in one element; they replay LayerNorm's fp32 reduction order to show that the two-pass variance
meets its bounds on offset rows and the one-pass E[x^2] - mean^2 does not; and they compute the premises (rows per
CTA, odd tail rows, chunk counts) from the launch code's grid formulas. They never load the library.
"""
import math

import numpy as np
import pytest
import torch

from test_gpu_kernel_bounds import BF, DEV, F64, H100_SMS, assert_within, bf16, pow2_rows, ulp_bf16, violations, within

F32 = torch.float32
U = 2.0 ** -24
ULP1 = 2.0 ** -23          # one fp32 ulp of y, relative to |y|, at most
FTZ = 2.0 ** -126          # __expf's flush-to-zero floor
NORM_THREADS, NORM_MAXCH = 256, 2
LOGP_THREADS = 256
BLOCK_TREE = 10            # block_sum2 and the log-prob combine: two five-level warp trees


def gam(n):
    return n * U / (1 - n * U)


def f32(v):
    """The fp32 value the kernel receives for a Python float argument, as a float."""
    return float(np.float32(v))


def ulp_f32(x):
    """Spacing of the fp32 numbers at |x|; below the normal range, the spacing at 2^-126."""
    _, e = torch.frexp(x.abs().to(F64).clamp_min(2.0 ** -126))
    return torch.exp2((e - 24).to(F64))


def rounded(ref, e, ulp=ulp_bf16):
    """Bound of a result the kernel rounds to its output type: the error carried so far plus one ulp at |ref| + e."""
    return e + ulp(ref.abs() + e)


def ceil_div(a, b):
    return -(-a // b)


# ================================================================================================ launch geometry
def norm_depth(H, cached_only=True):
    """Roundings a term passes through in a norm kernel's row sum: a thread's serial sum over its 8-element chunks
    (rmsnorm_fwd's uncached tail loop adds more chunks per thread), then block_sum2."""
    nch = H // 8
    per_thread = ceil_div(nch, NORM_THREADS)
    if cached_only:
        per_thread = min(per_thread, NORM_MAXCH)
    return 8 * per_thread + BLOCK_TREE


def rows_grid(M, sms):
    """rlaifv_rmsnorm_fwd / rlaifv_layernorm_fwd / rlaifv_logp_*: min(rows, 8 CTAs per SM)."""
    return min(M, 8 * sms)


def rmsnorm_bwd_grid(M, sms):
    return min(2 * sms, (M + 1) // 2)


def layernorm_bwd_grid(M, sms):
    return min(2 * sms, M)


def partials_depth(P):
    """reduce_partials_kernel: a thread sums partials ry, ry + 8, ... then row 0 sums the 8 lanes serially."""
    return ceil_div(P, 8) + 8


# ================================================================================================ references and bounds
def rsqrt_rel(rho):
    """|rsqrtf(v (1 + t)) / v^-1/2 - 1| for |t| <= rho: the square root of the argument's error, then rsqrtf's 2 ulp."""
    return (1 + rho / (2 * (1 - rho))) * (1 + 2 * ULP1) - 1


def layernorm_stats_ref(x, eps, H):
    """fp64 mean / rstd / xhat of bf16 rows and the error of the kernel's fp32 xhat = (x - mean) * rstd.
    mean: a sum of H exact terms (depth d) and a division: gamma_{d+1} mean|x|. The kernel's variance is one of two:
      one pass, var1 = fma(-mean_k, mean_k, sum(x^2) / H): the fma sum of exact squares and / H (gamma_{d+2} E[x^2]),
        mean_k^2 off by 2 |mean| e_mu + e_mu^2, the fma one rounding of var. The kernel keeps var1 only when
        mean_k^2 <= var1, which needs mean^2 <= 2 var (with these errors far below var): then E[x^2] <= 3 var.
        For rows with mean^2 > 2 var this term is 0.
      two pass (mean_k^2 > var1): mean((x - mean_k)^2) = var + e_mu^2, each term a subtraction, a square (fma) and the
        sum, then / H: gamma_{d+4}.
    Both are added, which covers whichever the kernel takes. var + eps rounds once more, then rsqrtf."""
    d = norm_depth(H)
    mu = x.mean(1, keepdim=True)
    xc = x - mu
    var = (xc * xc).mean(1, keepdim=True)
    r = (var + eps).rsqrt()
    xh = xc * r
    e_mu = gam(d + 1) * x.abs().mean(1, keepdim=True)
    m2 = mu * mu
    one = torch.where(m2 <= 2 * var, gam(d + 2) * (var + m2) + 2 * mu.abs() * e_mu + e_mu ** 2 + U * var,
                      torch.zeros_like(var))
    two = e_mu ** 2 + gam(d + 4) * (var + e_mu ** 2)
    rho = (one + two) / (var + eps) + U
    e_r = rsqrt_rel(rho)
    e_t1 = e_mu + U * (xc.abs() + e_mu)                                 # fl(x - mean_k)
    e_xh = r * (e_t1 * (1 + e_r) + xc.abs() * e_r + U * (xc.abs() + e_t1) * (1 + e_r))   # fl(t1 * rstd_k)
    return r, xh, e_r, e_xh


def layernorm_fwd_ref(x, w, b, eps):
    """y = bf16((x - mean) * rstd * w + b): xhat's error times |w|, then the w-multiply and b-add (fused or not:
    gamma_2 on their magnitude)."""
    x, w, b = x.to(F64), w.to(F64), b.to(F64)
    _, xh, _, e_xh = layernorm_stats_ref(x, f32(eps), x.shape[1])
    y = xh * w + b
    e = w.abs() * e_xh + gam(2) * (xh.abs() * w.abs() + b.abs() + w.abs() * e_xh)
    return y, rounded(y, e)


def param_grad_ref(terms, e_terms, mag, depth, old):
    """sum over rows of `terms` (each with error e_terms, magnitude mag), accumulated per CTA and over the partials
    (depth roundings), plus the old bf16 value when accumulating (one more rounding), rounded to bf16."""
    ref = terms.sum(0)
    e = e_terms.sum(0) + gam(depth + (old is not None)) * (mag.sum(0) + (0 if old is None else old.abs()))
    if old is not None:
        ref = ref + old
    return ref, rounded(ref, e)


def layernorm_bwd_ref(dy, x, w, eps, grid, dw_old=None, db_old=None):
    """dx = rstd (g - mean(g) - xhat mean(g xhat)), g = w dy (exact in fp32); dw = sum dy xhat; db = sum dy.
    mean(g): depth d + 1 on mean|g|. mean(g xhat): xhat's error times |g|, and the fma sum on |g| (|xhat| + e). The inner
    expression rounds twice (g - mg, then the fma), the rstd-multiply once; rstd carries e_r."""
    dy, x, w = dy.to(F64), x.to(F64), w.to(F64)
    M, H = x.shape
    d = norm_depth(H)
    r, xh, e_r, e_xh = layernorm_stats_ref(x, f32(eps), H)
    g = w * dy
    ag = g.abs()
    xm = xh.abs() + e_xh
    mg, mgx = g.mean(1, keepdim=True), (g * xh).mean(1, keepdim=True)
    e_mg = gam(d + 1) * ag.mean(1, keepdim=True)
    e_mgx = (ag * e_xh).mean(1, keepdim=True) + gam(d + 1) * (ag * xm).mean(1, keepdim=True)
    inner = g - mg - xh * mgx
    A = ag + mg.abs() + xh.abs() * mgx.abs()
    e_in = e_mg + xh.abs() * e_mgx + e_xh * (mgx.abs() + e_mgx)
    e_in = e_in + gam(2) * (A + e_in)
    dx = r * inner
    e_dx = r * (1 + e_r) * e_in + r * e_r * A + U * r * (1 + e_r) * (A + e_in)
    depth = ceil_div(M, grid) + partials_depth(grid)
    ady = dy.abs()
    dw = param_grad_ref(dy * xh, ady * e_xh, ady * xm, depth, None if dw_old is None else dw_old.to(F64))
    db = param_grad_ref(dy, torch.zeros_like(dy), ady, depth, None if db_old is None else db_old.to(F64))
    return (dx, rounded(dx, e_dx)), dw, db


def rmsnorm_fwd_ref(x, w, eps):
    """y = bf16(w * bf16(x * rstd)), rstd = rsqrtf(sum(x^2) / H + eps): the fma sum of exact squares (depth d, the tail
    loop's chunks included), / H and + eps round once each; x * rstd rounds, then to bf16 (one ulp); w * that is exact
    in fp32, rounded to bf16. Returns (y, bound), (rstd, bound)."""
    x, w = x.to(F64), w.to(F64)
    H = x.shape[1]
    eps = f32(eps)
    d = norm_depth(H, cached_only=False)
    ms = (x * x).mean(1, keepdim=True)
    r = (ms + eps).rsqrt()
    rho = gam(d + 1) * ms / (ms + eps) + U
    e_r = rsqrt_rel(rho)
    xh = x * r
    e_t = xh.abs() * (e_r + U * (1 + e_r))
    e_b = e_t + ulp_bf16(xh.abs() + e_t)
    y = w * xh
    e_y = w.abs() * e_b
    return (y, rounded(y, e_y)), (r.squeeze(1), rounded(r.squeeze(1), r.squeeze(1) * e_r, ulp_f32))


def rmsnorm_bwd_ref(dy, x, w, rstd, dres, grid, dw_old=None):
    """rstd is the forward's fp32 output, an exact input here. xhat = fl(x rstd) (u); mean(g xhat) by an fma sum of
    depth d and a division; dx = rstd * fma(-xhat, mean, g) (two roundings), + dres (one more), to bf16.
    dw = sum dy xhat: per CTA two rows per pass, then the partials."""
    dy, x, w, rstd = dy.to(F64), x.to(F64), w.to(F64), rstd.to(F64)[:, None]
    M, H = x.shape
    d = norm_depth(H)
    xh = x * rstd
    e_xh = U * xh.abs()
    g = w * dy
    ag = g.abs()
    xm = xh.abs() + e_xh
    mean = (g * xh).mean(1, keepdim=True)
    e_mean = (ag * e_xh).mean(1, keepdim=True) + gam(d + 1) * (ag * xm).mean(1, keepdim=True)
    A = ag + xh.abs() * mean.abs()
    e_in = xh.abs() * e_mean + e_xh * (mean.abs() + e_mean)
    e_in = e_in + U * (A + e_in)
    dx = rstd * (g - xh * mean)
    e = rstd * e_in + U * rstd * (A + e_in)
    if dres is not None:
        dx = dx + dres.to(F64)
        e = e + U * (rstd * A + dres.to(F64).abs() + e)
    depth = 2 * ceil_div(M, 2 * grid) + partials_depth(grid)
    ady = dy.abs()
    dw = param_grad_ref(dy * xh, ady * e_xh, ady * xm, depth, None if dw_old is None else dw_old.to(F64))
    return (dx, rounded(dx, e)), dw


def expf_fast_rel(x):
    """__expf's relative error at argument x (2 + floor(|1.173 x|) ulp)."""
    return (2 + torch.floor((1.173 * x).abs())) * ULP1


def sigmoid_err(g, fast_div=False):
    """sg = 1 / (1 + __expf(-g)): __expf's error scaled by E / (1 + E) <= 1, the add and the division (gamma_2), and
    the flush / overflow floor (for g < -88.7 __expf(-g) is inf and sg = 0, while sigmoid(g) < 2^-128). fast_div:
    the division is __fdividef (2 ulp, i.e. 4 u, instead of correctly rounded; it returns 0 for a divisor past 2^126,
    inside the same floor)."""
    s = torch.sigmoid(g)
    return s, s * (expf_fast_rel(-g) + (gam(5) if fast_div else gam(2))) * (1 + 1e-6) + FTZ


def swiglu_fwd_ref(gu):
    """act = bf16(bf16(g / (1 + __expf(-g))) * u): d(g / (1 + E))/dE = -silu / (1 + E), so the quotient carries
    |silu| (__expf's relative error + gamma_2) plus |g| 2^-126; silu rounds to bf16 (one ulp); bf16 * bf16 is exact,
    rounded to bf16."""
    gu = gu.to(F64)
    F = gu.shape[1] // 2
    g, u = gu[:, :F], gu[:, F:]
    s = g * torch.sigmoid(g)
    e_q = s.abs() * (expf_fast_rel(-g) + gam(2)) * (1 + 1e-6) + g.abs() * FTZ
    e_b = e_q + ulp_bf16(s.abs() + e_q)
    act = s * u
    return act, rounded(act, u.abs() * e_b)


def swiglu_bwd_ref(gu, dact, e_dact=None, fast_div=False):
    """sg as in sigmoid_err; du = d * fl(g sg); dg = fl(fl(d u) ... : (d u) exact, times
    fl(sg * fma(g, fl(1 - sg), 1)), each step one rounding on its magnitude.

    e_dact: the kernel's d may differ from dact by this much (the GEMM's fused form rounds its fp32 accumulator to bf16
    for d, and dact is then the fp64 product): |d| + e_dact stands for |d| in every rounding term, and e_dact times the
    computed factors (silu, u silu') is added. fast_div: sigmoid_err's __fdividef (gemm.cu swiglu_bwd_pair)."""
    gu, d = gu.to(F64), dact.to(F64)
    F = gu.shape[1] // 2
    g, u = gu[:, :F], gu[:, F:]
    s, e_s = sigmoid_err(g, fast_div)
    ag = g.abs()
    ad = d.abs() if e_dact is None else d.abs() + e_dact
    e_silu = ag * e_s + U * ag * (s + e_s)
    du = d * g * s
    e_du = ad * e_silu + U * ad * ag * (s + e_s)
    one_m = 1 - s
    e_t1 = e_s + U * (one_m + e_s)
    A2 = 1 + ag * one_m
    e_t2 = ag * e_t1 + U * (A2 + ag * e_t1)
    e_t3 = e_s * (A2 + e_t2) + s * e_t2 + U * (s + e_s) * (A2 + e_t2)
    dgu = d * u
    dg = dgu * s * (1 + g * one_m)
    e_dg = ad * u.abs() * e_t3 + U * ad * u.abs() * (s * A2 + e_t3)
    if e_dact is not None:
        e_du = e_du + e_dact * ag * (s + e_s)
        e_dg = e_dg + e_dact * u.abs() * s * A2
    return (dg, rounded(dg, e_dg)), (du, rounded(du, e_du))


SQRT1_2 = 1 / math.sqrt(2.0)


def gelu_fwd_ref(x):
    """0.5 x (1 + erff(x * 0.70710678f)): the argument carries the constant's and the product's rounding (gamma_2),
    moving erf by erf' = 2/sqrt(pi) exp(-a^2) times that; erff's 2 ulp; 1 + erff rounds; 0.5 x is exact, the product
    rounds. Large negative x cancels in 1 + erff: erff's absolute error, times |x| / 2, is the bound there."""
    x = x.to(F64)
    a = x * SQRT1_2
    er = torch.erf(a)
    e_erf = 2 / math.sqrt(math.pi) * torch.exp(-a * a) * gam(2) * a.abs() + 2 * ULP1 * er.abs()
    e_1p = e_erf + U * (1 + er.abs() + e_erf)
    y = 0.5 * x * (1 + er)
    e = 0.5 * x.abs() * e_1p + U * 0.5 * x.abs() * (1 + er + e_1p)
    return y, rounded(y, e)


def gelu_bwd_ref(x, dpost):
    """d * (cdf + x pdf), cdf = 0.5 (1 + erff(x c)) (as gelu_fwd_ref), pdf = 0.39894228f * __expf(-0.5 x x): the
    argument rounds (u |arg|), __expf's error and 2^-126, the constant and the product (gamma_2); then
    fma(x, pdf, cdf) and the d-multiply round once each."""
    x, d = x.to(F64), dpost.to(F64)
    a = x * SQRT1_2
    er = torch.erf(a)
    e_erf = 2 / math.sqrt(math.pi) * torch.exp(-a * a) * gam(2) * a.abs() + 2 * ULP1 * er.abs()
    cdf = 0.5 * (1 + er)
    e_cdf = 0.5 * (e_erf + U * (1 + er.abs() + e_erf))
    arg = -0.5 * x * x
    pdf = torch.exp(arg) / math.sqrt(2 * math.pi)
    e_pdf = pdf * (expf_fast_rel(arg) + 1.01 * U * arg.abs() + gam(2)) + FTZ
    sm = cdf + x * pdf
    A = cdf + x.abs() * pdf
    e_s = x.abs() * e_pdf + e_cdf + U * (A + x.abs() * e_pdf + e_cdf)
    o = d * sm
    e = d.abs() * e_s + U * d.abs() * (A + e_s)
    return o, rounded(o, e)


COLSUM_P = 64


def colsum_ref(x, old=None):
    """db = sum over rows: each of the 64 row-strided partial sums has ceil(M / 64) terms, then reduce_partials."""
    x = x.to(F64)
    depth = ceil_div(x.shape[0], COLSUM_P) + partials_depth(COLSUM_P)
    return param_grad_ref(x, torch.zeros_like(x), x.abs(), depth, None if old is None else old.to(F64))


def logp_depth(V):
    """(exp factors, roundings) a term of logp_fwd_kernel's online logsumexp passes through: its own __expf, one
    rescale per later chunk of its thread, one per combine level; each chunk's 8-term sum, then per later chunk a
    product and a sum, per combine level a product and a sum."""
    per_thread = ceil_div(V // 8, LOGP_THREADS)
    return per_thread + BLOCK_TREE, 8 + 2 * (per_thread + BLOCK_TREE)


def lse_ref(z):
    """fp64 logsumexp of bf16 rows and its error in the kernel. A term exp(z - M) is a product of __expf factors whose
    arguments telescope to z - M, each argument rounded (u |arg|): relative (2 NF + 2.173 (M - z)) 2^-23, plus the sum's
    gamma; __expf's flush costs at most 2^-126 per term. logf adds 1 ulp of log S, m + log S one rounding."""
    nf, dep = logp_depth(z.shape[1])
    m = z.amax(1, keepdim=True)
    t = torch.exp(z - m)
    S = t.sum(1, keepdim=True)
    e_S = (t * ((2 * nf + 2.173 * (m - z)) * ULP1 + gam(dep))).sum(1, keepdim=True) + z.shape[1] * FTZ
    dl = e_S / S
    e_log = dl / (1 - dl) + ULP1 * S.log() * (1 + dl)
    lse = (m + S.log()).squeeze(1)
    e_lse = (e_log + U * (m.abs() + S.log() + e_log)).squeeze(1)
    return lse, e_lse


def logp_rows_ref(logits, rows, labels_next):
    """per_tok and lse of the given logits rows (fp64 on the logits' device), with the errors before the output
    rounding. labels_next: the label of each row (-100 -> 0, as the kernel)."""
    z = logits[rows].to(F64)
    lse, e_lse = lse_ref(z)
    lab = labels_next.clamp_min(0)
    pt = z.gather(1, lab[:, None]).squeeze(1) - lse
    return pt, e_lse + U * (pt.abs() + e_lse), lse, e_lse


def seq_reduce_ref(pt, e_pt, mask, w, T):
    """logp_reduce_kernel: s = sum mask w pt (fma, product exact), c = sum mask w, avg = s / c. Each thread sums
    ceil((T - 1) / 256) terms, then block_sum2. Returns (sum, bound), (avg, bound), (count, bound)."""
    dep = ceil_div(T - 1, 256) + BLOCK_TREE
    mw = mask * w
    s = (pt * mw).sum(1)
    e_s = (e_pt * mw.abs()).sum(1) + gam(dep) * ((pt.abs() + e_pt) * mw.abs()).sum(1)
    c = mw.sum(1)
    e_c = gam(dep) * mw.abs().sum(1)
    avg = s / c
    e_a = (e_s + avg.abs() * e_c) / (c.abs() - e_c)
    return (s, rounded(s, e_s, ulp_f32)), (avg, rounded(avg, e_a, ulp_f32)), (c, rounded(c, e_c, ulp_f32))


def logp_bwd_rows_ref(z, lse, lab, g):
    """g (onehot(label) - __expf(z - lse)) for supervised rows: lse is the forward's fp32 output (exact input), g the
    kernel's fp32 d_logp * weight / norm (two roundings); the argument rounds (u |arg|); 1 - p rounds at the label;
    the g-multiply rounds, then to bf16."""
    a = z - lse[:, None]
    p = torch.exp(a)
    e_p = p * (expf_fast_rel(a) + 1.01 * U * a.abs()) + FTZ
    oh = torch.zeros_like(z)
    oh.scatter_(1, lab[:, None], 1.0)
    A = (oh - p).abs()
    e_A = e_p + U * (A + e_p)
    o = g[:, None] * (oh - p)
    e = g.abs()[:, None] * e_A + gam(3) * g.abs()[:, None] * (A + e_A)
    return o, rounded(o, e)


def dpo_ref(pw, pr, rw, rr, beta, dpo_w, sft_w, gs):
    """dpo_loss_kernel in fp64 from the fp32 inputs and fp32 scalars, with bounds:
      z = beta((a - b) - (c - d)): four roundings on beta(|a - b| + |c - d|)
      loss = max(-z, 0) + log1pf(expf(-|z|)) = softplus(-z): |d/dz| = sigmoid(-z), which grows at most by e^{e_z} over
             the interval; expf's 2 ulp move log1p by at most 2^-22 log1p(y); log1pf 1 ulp; the add; 2^-148 where
             expf underflows
      sig = 1 / (1 + expf(z)): sigmoid(-z) e^{e_z} - 1 from z, 2 ulp and two roundings; 2^-127 where expf overflows
      d_pw = gs (-w beta sig - sft) / B and d_pr = gs w beta sig / B: four roundings
      out9: two terms per lane then warp_sum (7 roundings), / B; accuracy counts the i whose order is ambiguous."""
    pw, pr, rw, rr = (t.to(F64) for t in (pw, pr, rw, rr))
    beta, dpo_w, sft_w, gs = f32(beta), f32(dpo_w), f32(sft_w), f32(gs)
    B = pw.numel()
    z = beta * ((pw - pr) - (rw - rr))
    e_z = gam(4) * beta * ((pw - pr).abs() + (rw - rr).abs())
    sneg = torch.sigmoid(-z)
    grow = torch.exp(e_z)
    loss = torch.nn.functional.softplus(-z)
    l1 = torch.log1p(torch.exp(-z.abs()))
    e_loss = e_z * sneg * grow + 3 * ULP1 * l1 + U * loss + 2.0 ** -148
    e_sig = sneg * ((grow - 1) + (2 * ULP1 + gam(2)) * grow) + 2.0 ** -127
    cr, rj = beta * (pw - rw), beta * (pr - rr)
    e_cr, e_rj = gam(2) * cr.abs(), gam(2) * rj.abs()
    k = abs(gs) / B
    d_pw = gs * (-dpo_w * beta * sneg - sft_w) / B
    e_dpw = k * (abs(dpo_w) * beta * e_sig + gam(4) * (abs(dpo_w) * beta * (sneg + e_sig) + abs(sft_w)))
    d_pr = gs * dpo_w * beta * sneg / B
    e_dpr = k * (abs(dpo_w) * beta * e_sig + gam(4) * abs(dpo_w) * beta * (sneg + e_sig))
    dep = ceil_div(B, 32) + 5
    t0 = dpo_w * loss - sft_w * pw
    e_t0 = abs(dpo_w) * e_loss + gam(2) * (abs(dpo_w) * loss + abs(sft_w) * pw.abs())
    ambiguous = ((cr - rj).abs() <= e_cr + e_rj).to(F64)
    cols = [
        (t0, e_t0), (cr, e_cr), (rj, e_rj), ((cr > rj).to(F64), None), (cr - rj, e_cr + e_rj + U * (cr - rj).abs()),
        (pr, 0 * pr), (pw, 0 * pw), (rr, 0 * rr), (rw, 0 * rw)]
    ref9, e9 = [], []
    for i, (v, e) in enumerate(cols):
        ref9.append(v.sum() / B)
        if e is None:
            e9.append(ambiguous.sum() / B + U)
        else:
            e9.append((e.sum() + gam(dep) * (v.abs() + e).sum()) / B + U * (v.abs().sum() + e.sum()) / B)
    ref9, e9 = torch.stack(ref9), torch.stack(e9)
    out = {
        "losses": (loss, rounded(loss, e_loss, ulp_f32)),
        "chosen_rewards": (cr, rounded(cr, e_cr, ulp_f32)),
        "rejected_rewards": (rj, rounded(rj, e_rj, ulp_f32)),
        "d_pw": (d_pw, rounded(d_pw, e_dpw, ulp_f32)),
        "d_pr": (d_pr, rounded(d_pr, e_dpr, ulp_f32)),
        "out9": (ref9, rounded(ref9, e9, ulp_f32)),
    }
    return out


def adamw_ref(p, m, v, g, lr, b1, b2, eps, wd, step, gs):
    """One AdamW step from the kernel's previous fp32 state (exact inputs) in fp64. The kernel receives beta1 / beta2
    as fp32 (fp32 0.999 makes 1 - beta2 1.29e-5 relative away from 0.001), so the reference uses the fp32 values.
      g gs (one rounding); p (1 - lr wd): three; m = fma(b1, m, (1 - b1) gj): 1 - b1 is exact (Sterbenz), gamma_3 with
      gj's; v = fma(b2, v, ((1 - b2) gj) gj): gamma_5. bc1 = 1 - powf(b1, step), bc2_sqrt = sqrtf(1 - powf(b2, step)) on
      the host: powf 1 ulp, each subtraction and sqrtf one rounding. denom = sqrtf(v) / bc2_sqrt + eps:
      |sqrt(a) - sqrt(b)| = |a - b| / (sqrt a + sqrt b), then three roundings; update (lr / bc1) (m / denom): three
      roundings plus bc1's and denom's relative errors and m's error / denom; p - update one rounding.
    Returns {name: (ref, bound)} for master, exp_avg, exp_avg_sq."""
    p, m, v, g = (t.to(F64) for t in (p, m, v, g))
    lr, b1, b2, eps, wd, gs = (f32(a) for a in (lr, b1, b2, eps, wd, gs))
    gj = g * gs
    e_gj = U * gj.abs()
    D = 1 - lr * wd
    p1 = p * D
    e_p1 = p.abs() * (gam(2) * D + U * lr * wd * (1 + U))
    m1 = b1 * m + (1 - b1) * gj
    e_m = gam(3) * (b1 * m.abs() + (1 - b1) * gj.abs())
    v1 = b2 * v + (1 - b2) * gj * gj
    e_v = gam(5) * (b2 * v + (1 - b2) * gj * gj)
    pw1, pw2 = b1 ** step, b2 ** step
    bc1, bc2 = 1 - pw1, 1 - pw2
    r1 = (ULP1 * pw1 + U * (bc1 + ULP1 * pw1)) / bc1
    r2 = 0.5 * (ULP1 * pw2 + U * (bc2 + ULP1 * pw2)) / bc2 + U
    bc2s = math.sqrt(bc2)
    sq = v1.sqrt()
    lo = (v1 - e_v).clamp_min(0).sqrt()
    e_sq = torch.where(e_v > 0, e_v / (sq + lo), torch.zeros_like(sq))
    den = sq / bc2s + eps
    e_den = (e_sq / bc2s) * (1 + r2) + (sq / bc2s) * (r2 + gam(2)) + U * den
    e_den = e_den * (1 + 1e-6)
    upd = (lr / bc1) * (m1 / den)
    rel = r1 + gam(3) + e_den / den
    e_upd = upd.abs() * rel * (1 + 1e-6) + (lr / bc1) * (e_m / den) * (1 + rel)
    p2 = p1 - upd
    e_p2 = e_p1 + e_upd
    return {"master": (p2, rounded(p2, e_p2, ulp_f32)), "exp_avg": (m1, rounded(m1, e_m, ulp_f32)),
            "exp_avg_sq": (v1, rounded(v1, e_v, ulp_f32))}


# ================================================================================================ inputs
def norm_rows(M, H, gen, device="cpu"):
    """bf16 rows: randn with power-of-two row scales 2^-6 .. 2^6; row 1 all tiny (2^-20: eps dominates)."""
    x = pow2_rows(torch.randn(M, H, generator=gen, dtype=F64), gen)
    if M > 1:
        x[1] *= 2.0 ** -20
    return x.to(BF).to(device)


def offset_rows(n, H, gen):
    """LayerNorm rows whose mean is at least 500 times their standard deviation (asserted by the premise test):
    250 + 0.4 randn in bf16 (ulp 1 there), scaled by 2^-6 .. 2^6; the last row is 100.0 with 1 in 512 elements one bf16
    ulp (0.5) higher, which the one-pass variance turns into 0."""
    x = pow2_rows(250.0 + 0.4 * torch.randn(n, H, generator=gen, dtype=F64), gen).to(BF)
    x[-1] = 100.0
    x[-1, ::512] = 100.5
    return x


def layernorm_inputs(M, H, gen, device="cpu"):
    """norm_rows with offset rows in the middle and a constant row (variance exactly 0) at M // 2 + 9."""
    x = norm_rows(M, H, gen)
    if M >= 64:
        k = min(16, M // 4)
        x[M // 2:M // 2 + k] = offset_rows(k, H, gen)
        x[M // 2 + k] = 3.0
    return x.to(device)


def ln_params(H, gen, device="cpu"):
    w = (1.0 + 0.5 * torch.randn(H, generator=gen, dtype=F64)).to(BF).to(device)
    b = (0.5 * torch.randn(H, generator=gen, dtype=F64)).to(BF).to(device)
    return w, b


def swiglu_inputs(M, F, gen, device="cpu"):
    """gate uniform in [-100, 40] (__expf(-g) overflows below -88.7), up randn with power-of-two row scales."""
    g = -100.0 + 140.0 * torch.rand(M, F, generator=gen, dtype=F64)
    u = pow2_rows(torch.randn(M, F, generator=gen, dtype=F64), gen)
    return torch.cat([g, u], 1).to(BF).to(device)


def gelu_inputs(M, N, gen, device="cpu"):
    """x uniform in [-12, 12]; every 16th row randn * 2^12 (large |x|)."""
    x = -12.0 + 24.0 * torch.rand(M, N, generator=gen, dtype=F64)
    x[::16] = torch.randn(x[::16].shape, generator=gen, dtype=F64) * 4096.0
    return x.to(BF).to(device)


def pow2_cols(M, N, gen, device="cpu"):
    x = pow2_rows(torch.randn(N, M, generator=gen, dtype=F64), gen).t().contiguous()
    return x.to(BF).to(device)


def dpo_inputs(B, gen):
    """fp32 log-probs of a few hundred nats whose margins beta 0.1 spreads across z in [-200, 200]; sample 0 has z
    exactly 0."""
    pw, pr, rw = (-300.0 * torch.rand(B, generator=gen, dtype=F64) for _ in range(3))
    rr = pr - (pw - rw) + torch.linspace(-2000.0, 2000.0, B, dtype=F64)
    pw[0], pr[0], rw[0], rr[0] = -100.0, -120.0, -105.0, -125.0
    return [t.to(F32) for t in (pw, pr, rw, rr)]


# ================================================================================================ CPU: the bounds
def _smallest_row(ref):
    return int(ref.abs().reshape(ref.shape[0], -1).amax(1).argmin())


def _assert_bound_discriminates(name, ref, bound, to):
    """The bound accepts ref rounded to the output type, and rejects a 2^-5 relative error in the row with the smallest
    values and in that row's element of median magnitude."""
    assert within(to(ref), ref, bound), name
    if ref.dim() == 1:
        ref, bound = ref[None], bound[None]
    r = _smallest_row(ref)
    bad = to(ref).clone()
    bad[r] = bad[r] * (1 + 2.0 ** -5)
    assert not within(bad, ref, bound), name + ": one row"
    row = ref[r].abs()
    j = int(row.argsort()[row.numel() // 2])
    bad = to(ref).clone()
    bad[r, j] = bad[r, j] * (1 + 2.0 ** -5)
    assert not within(bad, ref, bound), name + ": one element"


def _to_bf16(t):
    return bf16(t)


def _to_f32(t):
    return t.to(F32).to(F64)


def test_norm_bounds_accept_rounded_fp64_and_reject_one_bad_row_or_element():
    gen = torch.Generator().manual_seed(1)
    M, H = 96, 1792
    x = layernorm_inputs(M, H, gen)
    w, b = ln_params(H, gen)
    dy = norm_rows(M, H, gen)
    y, yb = layernorm_fwd_ref(x, w, b, 1e-6)
    _assert_bound_discriminates("layernorm_fwd y", y, yb, _to_bf16)
    (dx, dxb), (dw, dwb), (db, dbb) = layernorm_bwd_ref(dy, x, w, 1e-6, layernorm_bwd_grid(M, H100_SMS),
                                                        dw_old=w, db_old=b)
    _assert_bound_discriminates("layernorm_bwd dx", dx, dxb, _to_bf16)
    for name, r, bd in (("dw", dw, dwb), ("db", db, dbb)):
        assert within(bf16(r), r, bd), name
        assert not within(bf16(r) * (1 + 2.0 ** -5), r, bd), name
    H = 4096
    x = norm_rows(M, H, gen)
    w = (1.0 + 0.3 * torch.randn(H, generator=gen)).to(BF)
    dy = norm_rows(M, H, gen)
    (y, yb), (r, rb) = rmsnorm_fwd_ref(x, w, 1e-5)
    _assert_bound_discriminates("rmsnorm_fwd y", y, yb, _to_bf16)
    assert within(r.to(F32), r, rb) and not within(r.to(F32) * (1 + 2.0 ** -5), r, rb)
    rstd = r.to(F32)
    (dx, dxb), (dw, dwb) = rmsnorm_bwd_ref(dy, x, w, rstd, norm_rows(M, H, gen), rmsnorm_bwd_grid(M, H100_SMS), w)
    _assert_bound_discriminates("rmsnorm_bwd dx", dx, dxb, _to_bf16)
    assert within(bf16(dw), dw, dwb) and not within(bf16(dw) * (1 + 2.0 ** -5), dw, dwb)


def test_elementwise_bounds_accept_rounded_fp64_and_reject_one_bad_row_or_element():
    gen = torch.Generator().manual_seed(2)
    gu = swiglu_inputs(64, 512, gen)
    _assert_bound_discriminates("swiglu_fwd", *swiglu_fwd_ref(gu), _to_bf16)
    dact = pow2_rows(torch.randn(64, 512, generator=gen, dtype=F64), gen).to(BF)
    (dg, dgb), (du, dub) = swiglu_bwd_ref(gu, dact)
    _assert_bound_discriminates("swiglu_bwd dg", dg, dgb, _to_bf16)
    _assert_bound_discriminates("swiglu_bwd du", du, dub, _to_bf16)
    x = gelu_inputs(64, 512, gen)
    _assert_bound_discriminates("gelu_fwd", *gelu_fwd_ref(x), _to_bf16)
    d = pow2_rows(torch.randn(64, 512, generator=gen, dtype=F64), gen).to(BF)
    _assert_bound_discriminates("gelu_bwd", *gelu_bwd_ref(x, d), _to_bf16)
    xc = pow2_cols(300, 264, gen)
    for old in (None, (torch.randn(264, generator=gen) * 8).to(BF)):
        r, bd = colsum_ref(xc, old)
        assert within(bf16(r), r, bd)
        c = int(r.abs().argmin())
        bad = bf16(r).clone()
        bad[c] = bad[c] * (1 + 2.0 ** -5) + (2.0 ** -5 * float(r[c].abs()) == 0) * 1e-3
        assert not within(bad, r, bd)


def test_gelu_bound_covers_the_fp32_formula_where_it_cancels():
    """At x <= -8.5 the kernel's 1 + erff(x c) is exactly 0 in fp32; the bound admits that (and the true value)."""
    x = torch.tensor([[-12.0, -9.0, -8.5, -6.0, -3.0]], dtype=F64).to(BF)
    y, bd = gelu_fwd_ref(x)
    assert within(torch.zeros(1, 3, dtype=F64), y[:, :3], bd[:, :3])


def _logp_case(nseq, T, V, seed, device="cpu"):
    """logits [nseq*T, V] bf16 (sigma 1 or 4 by sequence), labels [nseq, T] with the first third at -100 (prompt), and
    the label of each row (nxt [nseq*T], -100 at t = T-1). Of the supervised rows, those at 0 mod 4 are peaked 30 above
    the rest at the label, those at 1 mod 4 have the label at the row's minimum. Generated on `device`."""
    gen = torch.Generator(device=device).manual_seed(seed)
    sig = torch.tensor([1.0 if s % 2 == 0 else 4.0 for s in range(nseq)], device=device).repeat_interleave(T)[:, None]
    z = (torch.randn(nseq * T, V, generator=gen, device=device) * sig).to(BF)
    labels = torch.randint(0, V, (nseq, T), generator=gen, device=device)
    labels[:, :T // 3] = -100

    def next_labels():
        return torch.cat([labels[:, 1:], torch.full((nseq, 1), -100, device=device)], 1).reshape(-1)
    nxt = next_labels()
    rows = torch.arange(nseq * T, device=device)
    pk = rows[(rows % 4 == 0) & (nxt >= 0)]
    z[pk, nxt[pk]] = (z[pk].float().amax(1) + 30.0).to(BF)
    mn = rows[(rows % 4 == 1) & (nxt >= 0)]
    labels.view(-1)[mn + 1] = z[mn].float().argmin(1)
    return z, labels, next_labels()


def test_logp_bounds_reject_a_wrong_label_column_and_a_nonzero_padding_row():
    gen = torch.Generator().manual_seed(3)
    nseq, T, V = 3, 40, 1000
    z, labels, nxt = _logp_case(nseq, T, V, 3)
    rows = torch.arange(nseq * T).reshape(nseq, T)[:, :T - 1].reshape(-1)
    pt, e_pt, lse, e_lse = logp_rows_ref(z, rows, nxt[rows])
    bd = rounded(pt, e_pt, ulp_f32)
    _assert_bound_discriminates("per_tok", pt.reshape(nseq, T - 1), bd.reshape(nseq, T - 1), _to_f32)
    # a wrong label column in one row: the log-prob of the label's neighbour
    sup = rows[nxt[rows] >= 0]
    r = int(sup[len(sup) // 2])
    wrong = z[r, (nxt[r] + 1) % V].to(F64) - lse[r]
    assert not within(wrong[None], pt[r:r + 1], bd[r:r + 1])
    mask = (nxt[rows] >= 0).to(F64).reshape(nseq, T - 1)
    (s, sb), (a, ab), (c, cb) = seq_reduce_ref(pt.reshape(nseq, T - 1), e_pt.reshape(nseq, T - 1), mask,
                                               torch.ones_like(mask), T)
    for name, ref, b_ in (("sum", s, sb), ("avg", a, ab)):
        _assert_bound_discriminates(name, ref, b_, _to_f32)
    assert within(c.to(F32), c, cb)
    # backward of the supervised rows; unsupervised rows and padding slots must be exactly 0
    sr = sup[:20]
    g = torch.randn(len(sr), generator=gen, dtype=F64)
    o, ob = logp_bwd_rows_ref(z[sr].to(F64), lse[sr].to(F32).to(F64), nxt[sr], g)
    _assert_bound_discriminates("logp_bwd", o, ob, _to_bf16)
    zero = torch.zeros(V, dtype=F64)
    left = zero.clone()
    left[7] = 2.0 ** -20
    assert within(zero, zero, zero) and not within(left, zero, zero)


def test_dpo_and_adamw_bounds_accept_rounded_fp64_and_reject_a_bad_element():
    gen = torch.Generator().manual_seed(4)
    pw, pr, rw, rr = dpo_inputs(37, gen)
    out = dpo_ref(pw, pr, rw, rr, 0.1, 0.75, 0.3, 0.5)
    for name, (ref, bd) in out.items():
        assert within(_to_f32(ref), ref, bd), name
        big = (ref.abs() >= bd * 64).nonzero()
        assert len(big), name
        bad = _to_f32(ref).clone()
        i = int(big[len(big) // 2])
        bad[i] = bad[i] * (1 + 2.0 ** -5)
        assert not within(bad, ref, bd), name
    n = 4096
    p = torch.randn(n, generator=gen, dtype=F64).to(F32)
    for gdt in (BF, F32):
        g = adamw_grads(n, gen, gdt)
        m = (torch.randn(n, generator=gen, dtype=F64) * 1e-3).to(F32)
        v = (torch.rand(n, generator=gen, dtype=F64) * 1e-6).to(F32)
        for step in (1, 3, 10000):
            refs = adamw_ref(p, m, v, g, 1e-3, 0.9, 0.999, 1e-8, 0.01, step, 0.125)
            for name, (ref, bd) in refs.items():
                _assert_bound_discriminates("adamw %s" % name, ref.reshape(64, -1), bd.reshape(64, -1), _to_f32)


def adamw_grads(n, gen, dtype, device="cpu"):
    """grads with magnitudes 2^-40 .. 2^4 (log-uniform), random sign; the last 8 elements 0 (with parameter 0)."""
    e = torch.randint(-40, 5, (n,), generator=gen).to(F64)
    g = torch.exp2(e) * (1 + torch.rand(n, generator=gen, dtype=F64)) * torch.sign(torch.randn(n, generator=gen))
    g[-8:] = 0
    return g.to(dtype).to(device)


# ------------------------------------------------------------------------------------------------ LayerNorm replay
def _fma32(a, b, c):
    """fp32 fma emulated in fp64 (the product of two fp32 values is exact there)."""
    return (a.astype(np.float64) * b + c).astype(np.float32)


def _block_sum(terms, fma_with=None):
    """block_sum2 after the per-thread loop of a norm kernel, replayed in fp32: terms [R, H] (fp32), thread t owning
    8-element chunks t and t + 256 (summed in that order, each left to right), then the warp and block trees. With
    fma_with, each term is terms * fma_with, accumulated by fma."""
    R, H = terms.shape
    pad = np.zeros((R, NORM_MAXCH * NORM_THREADS * 8), np.float32)
    pad[:, :H] = terms
    t = pad.reshape(R, NORM_MAXCH, NORM_THREADS, 8)
    if fma_with is not None:
        padb = np.zeros_like(pad)
        padb[:, :H] = fma_with
        tb = padb.reshape(R, NORM_MAXCH, NORM_THREADS, 8)
    s = np.zeros((R, NORM_THREADS), np.float32)
    for ci in range(NORM_MAXCH):
        for j in range(8):
            s = _fma32(t[:, ci, :, j], tb[:, ci, :, j], s) if fma_with is not None else (s + t[:, ci, :, j])
    v = s.reshape(R, NORM_THREADS // 32, 32)
    for o in (16, 8, 4, 2, 1):
        v = v[..., :o] + v[..., o:2 * o]
    w = np.zeros((R, 32), np.float32)
    w[:, :NORM_THREADS // 32] = v[..., 0]
    for o in (16, 8, 4, 2, 1):
        w = w[:, :o] + w[:, o:2 * o]
    return w[:, 0]


def layernorm_replay(x, w, b, dy, eps, two_pass):
    """layernorm_fwd_kernel / layernorm_bwd_kernel in fp32 (rsqrtf correctly rounded). The variance in one pass as
    max(fma(-mean, mean, E[x^2]), 0); with two_pass, taken again as mean((x - mean)^2) over the cached row where
    mean^2 exceeds it, as the kernel does. Returns bf16 y and dx as fp64 tensors."""
    xf = x.float().numpy()
    R, H = xf.shape
    eps = np.float32(eps)
    Hf = np.float32(H)
    mean = (_block_sum(xf) / Hf).astype(np.float32)[:, None]
    ex2 = (_block_sum(xf, fma_with=xf) / Hf).astype(np.float32)[:, None]
    var = np.maximum(_fma32(-mean, mean, ex2), np.float32(0))
    if two_pass:
        d = (xf - mean).astype(np.float32)
        again = (mean * mean).astype(np.float32) > var
        var = np.where(again, (_block_sum(d, fma_with=d) / Hf).astype(np.float32)[:, None], var)
    rstd = (1.0 / np.sqrt((var + eps).astype(np.float64))).astype(np.float32)
    xh = ((xf - mean).astype(np.float32) * rstd).astype(np.float32)
    wf, bf = w.float().numpy(), b.float().numpy()
    y = _fma32(xh, wf, bf)
    g = (wf * dy.float().numpy()).astype(np.float32)
    mg = (_block_sum(g) / Hf).astype(np.float32)[:, None]
    mgx = (_block_sum(g, fma_with=xh) / Hf).astype(np.float32)[:, None]
    dx = (rstd * _fma32(-xh, mgx, (g - mg).astype(np.float32))).astype(np.float32)
    return bf16(torch.from_numpy(y).to(F64)), bf16(torch.from_numpy(dx).to(F64))


@pytest.mark.parametrize("H", [1792, 4096])
def test_layernorm_replay_two_pass_meets_the_bounds_and_one_pass_breaks_them(H):
    """The fp32 replay of the kernel's statistics (one pass, the variance taken again in a second pass where mean^2
    exceeds it) meets the forward and backward bounds on offset rows (mean >= 500 std) and on the pow2-scaled rows
    around them; the one-pass E[x^2] - mean^2 alone breaks both on the offset rows. On every other row the two give
    the same bits: the second pass runs only where the one pass cancels."""
    gen = torch.Generator().manual_seed(5)
    M, eps = 64, 1e-6
    x = layernorm_inputs(M, H, gen)
    w, b = ln_params(H, gen)
    dy = norm_rows(M, H, gen)
    y, yb = layernorm_fwd_ref(x, w, b, eps)
    (dx, dxb), _, _ = layernorm_bwd_ref(dy, x, w, eps, layernorm_bwd_grid(M, H100_SMS))
    y2, dx2 = layernorm_replay(x, w, b, dy, eps, two_pass=True)
    assert_within("replay two-pass y H=%d" % H, y2, y, yb)
    assert_within("replay two-pass dx H=%d" % H, dx2, dx, dxb)
    y1, dx1 = layernorm_replay(x, w, b, dy, eps, two_pass=False)
    off = slice(M // 2, M // 2 + 16)
    bad_y = violations(y1[off], y[off], yb[off])[0].any(1)
    bad_dx = violations(dx1[off], dx[off], dxb[off])[0].any(1)
    print("one-pass replay H=%d: %d / 16 offset rows break the y bound, %d the dx bound" % (
        H, int(bad_y.sum()), int(bad_dx.sum())))
    assert bool(bad_y[-1]) and bool(bad_dx[-1])         # the near-constant row: variance 0, rstd eps^-1/2
    assert int(bad_y.sum()) >= 2 and int(bad_dx.sum()) >= 2
    # the rows outside the offset block are the same for both
    rest = torch.ones(M, dtype=torch.bool)
    rest[off] = False
    assert within(y1[rest], y[rest], yb[rest])
    assert torch.equal(y1[rest], y2[rest]) and torch.equal(dx1[rest], dx2[rest])


# ================================================================================================ CPU: the premises
SHAPES = {
    "rmsnorm": [(1, 4096), (2271, 4096), (18160, 4096), (2271, 5120)],
    "layernorm": [(M, H) for H in (1024, 1792, 4096) for M in (1, 64, 1154, 8200)],
    "logp_dense": (16, 1135, 32000),
    "logp_omni": (4, 301, 32008),
}


def test_premise_grids_walk_many_rows_per_cta_and_odd_tails():
    g = rows_grid(18160, H100_SMS)
    assert g == 1056 and 18160 > g
    assert 8200 > rows_grid(8200, H100_SMS)
    for M in (1154, 8200):
        assert M > layernorm_bwd_grid(M, H100_SMS)
    nseq, T, V = SHAPES["logp_dense"]
    assert nseq * (T - 1) > rows_grid(nseq * (T - 1), H100_SMS) and nseq * T > rows_grid(nseq * T, H100_SMS)
    # rmsnorm_bwd: two rows per pass; an odd M above 2 x 264 rows leaves a CTA a tail row after several passes
    M = 2271
    assert M % 2 == 1 and M > 2 * 2 * H100_SMS and rmsnorm_bwd_grid(M, H100_SMS) == 264
    assert rmsnorm_bwd_grid(18160, H100_SMS) == 264 and rmsnorm_bwd_grid(1, H100_SMS) == 1


def test_premise_chunk_counts_are_not_multiples_of_the_block():
    for n in (1792, 32000, 32008, 5120):
        assert (n // 8) % 256 != 0, n
    assert 1792 // 8 == 224 and 32008 // 8 == 4001
    # rmsnorm_fwd at H = 5120 runs the uncached tail loop: more chunks than NORM_MAXCH per thread
    assert 5120 // 8 > NORM_MAXCH * NORM_THREADS


def test_premise_offset_rows_have_mean_500_std_and_cancel_one_pass():
    gen = torch.Generator().manual_seed(6)
    x = offset_rows(16, 4096, gen).to(F64)
    ratio = x.mean(1).abs() / x.std(1, unbiased=False)
    print("offset rows: mean / std from %.0f to %.0f" % (float(ratio.min()), float(ratio.max())))
    assert bool((ratio >= 500).all())


# ================================================================================================ GPU
def _chunks(n, size):
    for s in range(0, n, size):
        yield slice(s, min(n, s + size))


class Worst:
    """Per-element check over row chunks, printing the worst err/bound of the whole case."""

    def __init__(self, name):
        self.name, self.worst = name, 0.0

    def check(self, got, ref, bound):
        bad, ratio = violations(got, ref, bound)
        self.worst = max(self.worst, float(ratio.nan_to_num(nan=float("inf")).max()))
        if bool(bad.any()):
            i = tuple(bad.nonzero()[0].tolist())
            raise AssertionError("%s: %d of %d elements outside their bound; first at %s: got %r, fp64 %r, bound %r" % (
                self.name, int(bad.sum()), bad.numel(), i, float(got[i]), float(ref[i]), float(bound[i])))

    def done(self):
        print("err/bound %-44s %.3g" % (self.name, self.worst))
        return self.worst


@pytest.mark.gpu
@pytest.mark.parametrize("M,H", SHAPES["rmsnorm"])
def test_rmsnorm_forward_backward_bounds(M, H):
    from rlaifv_b200 import ops
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    gen = torch.Generator().manual_seed(100 + M + H)
    x = norm_rows(M, H, gen, DEV)
    w = (1.0 + 0.3 * torch.randn(H, generator=gen)).to(BF).to(DEV)
    rstd = torch.empty(M, dtype=F32, device=DEV)
    y = ops.rmsnorm_fwd(x, w, 1e-5, rstd=rstd)
    torch.cuda.synchronize()
    (yr, yb), (rr, rb) = rmsnorm_fwd_ref(x, w, 1e-5)
    assert_within("rmsnorm_fwd y [%d,%d]" % (M, H), y, yr, yb)
    assert_within("rmsnorm_fwd rstd [%d,%d]" % (M, H), rstd, rr, rb)
    if H > NORM_MAXCH * NORM_THREADS * 8:
        return                                              # the backward caches the row: H <= 4096
    dy = norm_rows(M, H, gen, DEV)
    dres = norm_rows(M, H, gen, DEV)
    grid = rmsnorm_bwd_grid(M, sms)
    for use_dres, acc in ((False, False), (True, True)):
        dx = torch.full_like(x, float("nan"))
        dw = (torch.randn(H, generator=gen) * 4).to(BF).to(DEV)
        old = dw.clone()
        ops.rmsnorm_bwd(dy, x, w, rstd, dx, dw, dres=dres if use_dres else None, dw_accumulate=acc)
        torch.cuda.synchronize()
        (dxr, dxb), (dwr, dwb) = rmsnorm_bwd_ref(dy, x, w, rstd, dres if use_dres else None, grid,
                                                 old if acc else None)
        assert_within("rmsnorm_bwd dx [%d,%d] dres=%d" % (M, H, use_dres), dx, dxr, dxb)
        assert_within("rmsnorm_bwd dw [%d,%d] acc=%d" % (M, H, acc), dw, dwr, dwb)


@pytest.mark.gpu
def test_rmsnorm_bwd_rejects_zero_rows():
    from rlaifv_b200 import lib, ops
    x = torch.zeros(0, 4096, dtype=BF, device=DEV)
    w = torch.ones(4096, dtype=BF, device=DEV)
    with pytest.raises(lib.B200Error, match="rc=-1"):
        ops.rmsnorm_bwd(x, x, w, torch.zeros(1, device=DEV), x, w.clone())


@pytest.mark.gpu
def test_layernorm_fwd_rejects_rows_wider_than_the_register_cache():
    from rlaifv_b200 import lib, ops
    x = torch.zeros(4, 4104, dtype=BF, device=DEV)
    w = torch.ones(4104, dtype=BF, device=DEV)
    with pytest.raises(lib.B200Error, match="rc=-1"):
        ops.layernorm_fwd(x, w, w, 1e-5)


LN_EPS = {1024: 1e-5, 1792: 1e-6, 4096: 1e-6}


@pytest.mark.gpu
@pytest.mark.parametrize("M,H", SHAPES["layernorm"])
def test_layernorm_forward_backward_bounds(M, H):
    from rlaifv_b200 import ops
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    eps = LN_EPS[H]
    gen = torch.Generator().manual_seed(200 + M + H)
    x = layernorm_inputs(M, H, gen, DEV)
    w, b = ln_params(H, gen, DEV)
    y = ops.layernorm_fwd(x, w, b, eps)
    torch.cuda.synchronize()
    assert_within("layernorm_fwd [%d,%d]" % (M, H), y, *layernorm_fwd_ref(x, w, b, eps))
    dy = norm_rows(M, H, gen, DEV)
    grid = layernorm_bwd_grid(M, sms)
    for acc in (False, True):
        dx = torch.full_like(x, float("nan"))
        dw = (torch.randn(H, generator=gen) * 4).to(BF).to(DEV)
        db = (torch.randn(H, generator=gen) * 4).to(BF).to(DEV)
        dw0, db0 = dw.clone(), db.clone()
        ops.layernorm_bwd(dy, x, w, eps, dx, dw, db, accumulate=acc)
        torch.cuda.synchronize()
        (dxr, dxb), (dwr, dwb), (dbr, dbb) = layernorm_bwd_ref(dy, x, w, eps, grid, dw0 if acc else None,
                                                               db0 if acc else None)
        assert_within("layernorm_bwd dx [%d,%d]" % (M, H), dx, dxr, dxb)
        assert_within("layernorm_bwd dw [%d,%d] acc=%d" % (M, H, acc), dw, dwr, dwb)
        assert_within("layernorm_bwd db [%d,%d] acc=%d" % (M, H, acc), db, dbr, dbb)


@pytest.mark.gpu
@pytest.mark.parametrize("F", [11008, 14336])
def test_swiglu_bounds(F):
    from rlaifv_b200 import ops
    M = 2271
    gen = torch.Generator().manual_seed(300 + F)
    gu = swiglu_inputs(M, F, gen, DEV)
    dact = pow2_rows(torch.randn(M, F, generator=gen), gen).to(BF).to(DEV)
    act = ops.swiglu_fwd(gu)
    dgu = ops.swiglu_bwd(gu, dact)
    torch.cuda.synchronize()
    wf, wg, wu = Worst("swiglu_fwd [%d,%d]" % (M, F)), Worst("swiglu_bwd dg [%d,%d]" % (M, F)), \
        Worst("swiglu_bwd du [%d,%d]" % (M, F))
    for s in _chunks(M, 512):
        wf.check(act[s], *swiglu_fwd_ref(gu[s]))
        (dg, dgb), (du, dub) = swiglu_bwd_ref(gu[s], dact[s])
        wg.check(dgu[s, :F], dg, dgb)
        wu.check(dgu[s, F:], du, dub)
    wf.done(), wg.done(), wu.done()


@pytest.mark.gpu
@pytest.mark.parametrize("M,N", [(4608, 4096), (8200, 15360)])
def test_gelu_bounds(M, N):
    from rlaifv_b200 import ops
    gen = torch.Generator().manual_seed(400 + N)
    x = gelu_inputs(M, N, gen, DEV)
    d = pow2_rows(torch.randn(M, N, generator=gen), gen).to(BF).to(DEV)
    y = ops.gelu_fwd(x)
    dx = ops.gelu_bwd(x, d)
    torch.cuda.synchronize()
    wf, wb = Worst("gelu_fwd [%d,%d]" % (M, N)), Worst("gelu_bwd [%d,%d]" % (M, N))
    for s in _chunks(M, 1024):
        wf.check(y[s], *gelu_fwd_ref(x[s]))
        wb.check(dx[s], *gelu_bwd_ref(x[s], d[s]))
    wf.done(), wb.done()


@pytest.mark.gpu
@pytest.mark.parametrize("M,N", [(8200, 1792), (8200, 15360), (1154, 264)])
def test_colsum_bounds(M, N):
    from rlaifv_b200 import ops
    gen = torch.Generator().manual_seed(500 + N)
    x = pow2_cols(M, N, gen, DEV)
    for acc in (False, True):
        db = (torch.randn(N, generator=gen) * 16).to(BF).to(DEV)
        old = db.clone()
        ops.colsum(x, db, accumulate=acc)
        torch.cuda.synchronize()
        assert_within("colsum [%d,%d] acc=%d" % (M, N, acc), db, *colsum_ref(x, old if acc else None))


def _check_logp(name, z, labels, nxt, nseq, T, row_pos, per_tok, lse, s, a, c):
    """per_tok / lse / sums of the dense (row_pos None) or compact head against fp64, by row chunks. z: the logits the
    kernel read (compact: the gathered rows, indexed by slot)."""
    wpt, wl = Worst(name + " per_tok"), Worst(name + " lse")
    ref_pt = torch.zeros(nseq * (T - 1), dtype=F64, device=DEV)
    e_pt = torch.zeros_like(ref_pt)
    flat = torch.arange(nseq * T, device=DEV)
    if row_pos is None:
        rows = flat[flat % T != T - 1]
    else:
        rows = torch.arange(row_pos.numel(), device=DEV)[row_pos >= 0]
    pos = rows if row_pos is None else row_pos[rows].long()
    dst = (pos // T) * (T - 1) + pos % T
    got_lse = lse.reshape(-1)
    for sl in _chunks(len(rows), 2048):
        r = rows[sl]
        pt, ept, l, el = logp_rows_ref(z, r, nxt[pos[sl]])
        ref_pt[dst[sl]], e_pt[dst[sl]] = pt, ept
        lidx = pos[sl] if row_pos is None else r
        wl.check(got_lse[lidx], l, rounded(l, el, ulp_f32))
    bd = rounded(ref_pt, e_pt, ulp_f32)
    if row_pos is not None:
        covered = torch.zeros_like(ref_pt, dtype=torch.bool)
        covered[dst] = True
        bd[~covered] = 0                                    # unsupervised positions stay exactly 0
    wpt.check(per_tok.reshape(-1), ref_pt, bd)
    wpt.done(), wl.done()
    mask = (labels[:, 1:] != -100).to(F64)
    (sr, sb), (ar, ab), (cr, cb) = seq_reduce_ref(ref_pt.reshape(nseq, T - 1), e_pt.reshape(nseq, T - 1), mask,
                                                  torch.ones_like(mask), T)
    assert_within(name + " logp_sum", s, sr, sb)
    assert_within(name + " logp_avg", a, ar, ab)
    assert_within(name + " count", c, cr, cb)
    return ref_pt


def _check_logp_bwd(name, z, g_logits, nxt, nseq, T, row_pos, lse, d_logp, tw, norm):
    """g_logits: the kernel's in-place result. Supervised rows against fp64, every other row exactly 0."""
    wb = Worst(name)
    n = g_logits.shape[0]
    rows = torch.arange(n, device=DEV)
    pos = rows if row_pos is None else row_pos.long()
    valid = pos >= 0
    t = pos.clamp_min(0) % T
    b = pos.clamp_min(0) // T
    lab = torch.where(valid & (t < T - 1), nxt[pos.clamp_min(0)], torch.full_like(pos, -100))
    sup = lab >= 0
    zero = g_logits[~sup]
    assert int((zero != 0).sum()) == 0, name + ": unsupervised or padding rows not zeroed"
    g = d_logp.to(F64)[b]
    if tw is not None:
        g = g * tw.to(F64)[b, t.clamp_max(T - 2)]
    if norm is not None:
        g = g / norm.to(F64)[b]
    sr = rows[sup]
    got_lse = lse.reshape(-1)
    for sl in _chunks(len(sr), 2048):
        r = sr[sl]
        lidx = pos[r] if row_pos is None else r
        o, ob = logp_bwd_rows_ref(z[r].to(F64), got_lse[lidx].to(F64), lab[r], g[r])
        wb.check(g_logits[r], o, ob)
    return wb.done()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["dense", "compact", "omni"])
def test_logp_head_bounds(case):
    from rlaifv_b200 import ops
    nseq, T, V = SHAPES["logp_omni"] if case == "omni" else SHAPES["logp_dense"]
    z, labels, nxt = _logp_case(nseq, T, V, 600 + len(case), DEV)
    row_pos = None
    logits = z
    if case == "compact":
        cap = T - T // 3 + 8                                # -1 slots at the end of every sequence's segment
        row_pos = ops.supervised_rows(labels, cap)
        assert int((row_pos < 0).sum()) == 8 * nseq
        logits = ops.rows_gather(row_pos, z)
        del z
    per_tok, lse, s, a, c = ops.logp_fwd(logits, labels, nseq, T, row_pos=row_pos)
    torch.cuda.synchronize()
    _check_logp("logp_fwd %s" % case, logits, labels, nxt, nseq, T, row_pos, per_tok, lse, s, a, c)
    gen = torch.Generator().manual_seed(700)
    d_logp = torch.randn(nseq, generator=gen).to(DEV)
    tw = (2 * torch.rand(nseq, T - 1, generator=gen)).to(DEV)
    wsum = None
    for mode in ("sum", "average", "weighted", "weighted_average"):
        weighted = mode.startswith("weighted")
        norm = None
        if mode == "average":
            norm = c
        elif mode == "weighted_average":
            _, _, wsum = ops.logp_weighted_reduce(per_tok, labels, tw)
            norm = wsum
        g_logits = logits.clone()
        ops.logp_bwd(g_logits, labels, lse, d_logp, nseq, T, row_pos=row_pos, token_weight=tw if weighted else None,
                     norm=norm)
        torch.cuda.synchronize()
        _check_logp_bwd("logp_bwd %s %s" % (case, mode), logits, g_logits, nxt, nseq, T, row_pos, lse, d_logp,
                        tw if weighted else None, norm)
    lw, aw, ws = ops.logp_weighted_reduce(per_tok, labels, tw)
    torch.cuda.synchronize()
    mask = (labels[:, 1:] != -100).to(F64)
    (sr, sb), (ar, ab), (cr, cb) = seq_reduce_ref(per_tok.to(F64), torch.zeros_like(mask), mask, tw.to(F64), T)
    assert_within("logp_weighted_reduce %s sum" % case, lw, sr, sb)
    assert_within("logp_weighted_reduce %s avg" % case, aw, ar, ab)
    assert_within("logp_weighted_reduce %s wsum" % case, ws, cr, cb)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [8, 37])
def test_dpo_loss_bounds(B):
    from rlaifv_b200 import ops
    gen = torch.Generator().manual_seed(800 + B)
    pw, pr, rw, rr = (t.to(DEV) for t in dpo_inputs(B, gen))
    beta, dpo_w, sft_w, gs = 0.1, 0.75, 0.3, 0.5
    z = beta * ((pw.double() - pr.double()) - (rw.double() - rr.double()))
    assert float(z.min()) < -100 and float(z.max()) > 100 and float(z[0]) == 0.0
    got = dict(zip(["losses", "chosen_rewards", "rejected_rewards", "d_pw", "d_pr", "out9"],
                   ops.dpo_loss(pw, pr, rw, rr, beta, dpo_weight=dpo_w, sft_weight=sft_w, grad_scale=gs)))
    torch.cuda.synchronize()
    for name, (ref, bd) in dpo_ref(pw, pr, rw, rr, beta, dpo_w, sft_w, gs).items():
        assert_within("dpo_loss B=%d %s" % (B, name), got[name], ref, bd)


@pytest.mark.gpu
@pytest.mark.parametrize("grad_dtype", [BF, F32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_adamw_step_bounds(grad_dtype, wd):
    from rlaifv_b200 import ops
    n = 1_000_004
    gen = torch.Generator().manual_seed(900 + int(wd * 100) + (grad_dtype == F32))
    master = torch.randn(n, generator=gen).to(DEV)
    master[-8:] = 0                                         # zero parameter with zero gradient (EVA's padded columns)
    m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    pbf = torch.empty(n, dtype=BF, device=DEV)
    lr, b1, b2, eps, gs = 1e-3, 0.9, 0.999, 1e-8, 0.125
    for step in (1, 2, 3, 10000):
        g = adamw_grads(n, gen, grad_dtype, DEV)
        p0, m0, v0 = master.clone(), m.clone(), v.clone()
        ops.adamw_step(master, m, v, g, pbf, lr, b1, b2, eps, wd, step, grad_scale=gs)
        torch.cuda.synchronize()
        refs = adamw_ref(p0, m0, v0, g, lr, b1, b2, eps, wd, step, gs)
        for name, got in (("master", master), ("exp_avg", m), ("exp_avg_sq", v)):
            assert_within("adamw %s step %d wd %g %s" % (str(grad_dtype)[6:], step, wd, name), got, *refs[name])
        assert torch.equal(pbf, master.to(BF))
        assert int((master[-8:] != 0).sum()) == 0 and int((m[-8:] != 0).sum()) == 0


@pytest.mark.gpu
def test_f32_to_bf16_bit_exact():
    from rlaifv_b200 import ops
    gen = torch.Generator().manual_seed(1000)
    # dproj: the projector-output gradient [image rows, 4096]; EVA dQ [Q, E]-style 2-d blocks of a wider buffer
    for rows, cols in ((4608, 4096), (8200, 1792)):
        src = pow2_rows(torch.randn(rows, cols, generator=gen), gen).to(DEV)
        for acc in (False, True):
            dst = (torch.randn(rows, cols, generator=gen)).to(BF).to(DEV)
            old = dst.clone()
            ops.f32_to_bf16(src, dst, accumulate=acc)
            want = (old.float() + src).to(BF) if acc else src.to(BF)
            assert torch.equal(dst, want), ("f32_to_bf16", rows, cols, acc)
            wide = torch.randn(rows, cols + 24, generator=gen).to(BF).to(DEV)
            before = wide.clone()
            blk = wide[:, 8:8 + cols]
            ops.f32_to_bf16_2d(src, blk, accumulate=acc)
            want = (before[:, 8:8 + cols].float() + src).to(BF) if acc else src.to(BF)
            assert torch.equal(blk, want), ("f32_to_bf16_2d", rows, cols, acc)
            assert torch.equal(wide[:, :8], before[:, :8]) and torch.equal(wide[:, 8 + cols:], before[:, 8 + cols:])

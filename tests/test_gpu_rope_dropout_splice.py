"""RoPE, LoRA dropout, the image splice, the CLIP/EVA patch front and the compact head's row movement against exact
references at the DPO step's shapes.

These kernels of rowops.cu copy, index or round only a few times, so each result is checked bit for bit where the
reference can replay the kernel's roundings, and within a per-element fp64 bound where it cannot:
  - RoPE forward: bit-exact against the HF rounding order bf16(bf16(x cos) + bf16(rotate_half(x) sin)) on the same
    bf16 tables, and within a bound of the exact fp64 rotation. RoPE backward: within a bound of the fp64 transpose
    dx1 = dy1 c1 + dy2 s2, dx2 = dy2 c2 - dy1 s1. Both run on the HF tables and on "skew" tables whose two halves
    differ: the HF tables repeat their first half, so a kernel that swapped c1 / c2 or s1 / s2 would pass on them.
  - Dropout: a NumPy uint64 replay of the counter-based hash (splitmix64's finaliser of seed ^ (i * K)) gives the keep
    bit of every element; the kernels' outputs equal where(keep, bf16(x * fp32(1 / (1 - p))), 0) bitwise.
  - Splice: the index maps, the gather, the count and OmniLMM's in-place map equal the oracle restatements
    (oracle.llava_dpo_oracle.splice_index_map / splice_embeds, oracle.omnilmm_oracle.inplace_splice_map) exactly; the
    backward scatter's fp32 atomics are exact where a row receives at most two terms and within gamma_{n-1} sum|terms|
    of fp64 where a token id occurs n times.
  - CLIP / EVA patch front, supervised_rows, rows_gather / rows_scatter, splice_token_weight and add_rows_bcast
    (including its two in-place calls) are copies or one bf16 addition: bit-exact.

The shapes are the step's: 8 sequences of 2048 positions, LLaVA-7B (32/32 heads), LLaVA-13B (40/40) and Mistral /
OmniLMM (32/8) attention, LoRA widths 4096 - 13824 with 9081 rows, 576 image rows per block spliced at positions that
straddle the 32-token chunks of the one-warp ballot scans, V = 32000. Every GPU case prints its worst err/bound. The
RoPE bounds end in half a bf16 ulp of the result, the most a round-to-nearest can move it, so over 10^8 elements their
worst ratio comes within 10^-4 of 1: a position, half or head mix-up moves an element by many ulps.

The tests without the gpu mark show that each bound and reference tells a wrong result from the right one, check the
mask statistics of the hash replay at 18 160 rows, and compute the premises from the launch code; they never load the
library.
"""
import math
import os
import re

import numpy as np
import pytest
import torch

from oracle import llava_dpo_oracle as O
from oracle import omnilmm_oracle as OM
from test_gpu_kernel_bounds import BF, DEV, F64, H100_SMS, bf16, ulp_bf16, violations, within

F32 = torch.float32
U = 2.0 ** -24
THREADS = 256              # every grid-stride launch below: 256 threads per CTA
PAD = -2 ** 31             # SPLICE_PAD
IGNORE = -100
IMAGE = -200
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gam(n):
    return n * U / (1 - n * U)


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
        print("err/bound %-44s %.5f" % (self.name, self.worst))
        return self.worst


def same_bits(a, b):
    """Bitwise equality of two tensors of one dtype (NaN payloads and signed zeros included)."""
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    view = {BF: torch.int16, F32: torch.int32}.get(a.dtype)
    return torch.equal(a.view(view), b.view(view)) if view is not None else torch.equal(a, b)


# ================================================================================================ launch geometry
def grid_for(work, threads=THREADS, per_sm=8, sms=H100_SMS):
    """rowops.cu grid_for: one thread per work item, capped at per_sm CTAs per SM (the restatement is held to the
    source by test_premise_launch_code_is_what_the_geometry_mirrors)."""
    return max(1, min(-(-work // threads), sms * per_sm))


def full_passes(work, grid, threads=THREADS):
    """Times every thread of a grid-stride loop runs its body."""
    return work // (grid * threads)


# ================================================================================================ RoPE
T_ROPE, HD = 2048, 128
ROPE_DIMS = {"llava7b": (32, 32), "llava13b": (40, 40), "mistral": (32, 8)}
RAGGED_LENS = [2048, 1999, 1, 777, 1501, 2047, 3, 1201]          # 9577 packed rows: odd, one 1-row sequence


def rope_tables(kind, T=T_ROPE, hd=HD):
    """'hf': the HF tables (theta 10000, halves equal). 'skew': rotations of varying radius, halves different."""
    if kind == "hf":
        return O.rope_cos_sin(T, hd, 10000.0, BF)
    g = torch.Generator().manual_seed(11)
    ang = torch.rand(T, hd, generator=g, dtype=F64) * (2 * math.pi)
    r = 0.5 + torch.rand(T, hd, generator=g, dtype=F64)
    return (r * ang.cos()).to(BF), (r * ang.sin()).to(BF)


def ragged_positions(lens):
    return torch.cat([torch.arange(n) for n in lens]).to(torch.int32)


def rot_heads(buf, nh, nkv):
    """[M, nh + nkv, hd] view of the rotated (q then k) column blocks of a fused qkv row."""
    return buf[:, : (nh + nkv) * HD].reshape(buf.shape[0], nh + nkv, HD)


def rope_fwd_hf(x, c, s):
    """HF apply_rotary_pos_emb in bf16 torch: every product and the sum round to bf16, as the kernel's do."""
    return x * c + O.rotate_half(x) * s


def rope_fwd_exact(x, c, s):
    """Exact rotation in fp64 on the bf16 tables, and its bound. The kernel rounds each product to bf16 (half an ulp of
    each: the product of two bf16 values is exact in fp32), adds the two in fp32 (u of the sum of magnitudes) and
    rounds to bf16 (half an ulp of a value at most |ref| + e)."""
    x, c, s = x.to(F64), c.to(F64), s.to(F64)
    h = x.shape[-1] // 2
    x1, x2 = x[..., :h], x[..., h:]
    p = torch.cat((x1 * c[..., :h], x2 * c[..., h:]), -1)
    q = torch.cat((-x2 * s[..., :h], x1 * s[..., h:]), -1)
    ref = p + q
    e = 0.5 * ulp_bf16(p) + 0.5 * ulp_bf16(q)
    e = e + U * (p.abs() + q.abs() + e)
    return ref, e + 0.5 * ulp_bf16(ref.abs() + e)


def rope_bwd_exact(y, c, s):
    """The transpose of the rotation in fp64, dx1 = dy1 c1 + dy2 s2, dx2 = dy2 c2 - dy1 s1, and its bound. The kernel
    forms each output from two fp32 products and one fp32 sum; nvcc may contract one product into an FMA. Either way at
    most two roundings reach any term (a product of the fp32 dQ and a table entry rounds; of two bf16 values it is
    exact): gamma_2 (|a| + |b|). Then one rounding to bf16: half an ulp of a value at most |ref| + e."""
    y, c, s = y.to(F64), c.to(F64), s.to(F64)
    h = y.shape[-1] // 2
    y1, y2 = y[..., :h], y[..., h:]
    a = torch.cat((y1 * c[..., :h], y2 * c[..., h:]), -1)
    b = torch.cat((y2 * s[..., h:], -y1 * s[..., :h]), -1)
    ref = a + b
    e = gam(2) * (a.abs() + b.abs())
    return ref, e + 0.5 * ulp_bf16(ref.abs() + e)


def rope_work(M, nh, nkv):
    return M * (nh + nkv) * (HD // 16)


# ================================================================================================ dropout
K_HASH = np.uint64(0xD1B54A32D192ED03)
DROP_M, DROP_PACKED = 9081, 6007
DROP_WIDTHS = [4096, 5120, 11008, 13824]
DROP_PS = [0.0, 0.05, 0.25]


def mix32(z):
    """splitmix64's finaliser on uint64 z (wrapping arithmetic), high word: rowops.cu mix32."""
    z = z + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(32)).astype(np.uint32)


def keep_bits(seed, elems, thresh):
    """keep_bits8 for flat element indices (chunk * 8 + j): mix32(seed ^ (i * K)) >= thresh."""
    return mix32(np.uint64(seed) ^ (np.asarray(elems, dtype=np.uint64) * K_HASH)) >= np.uint32(thresh)


def dropout_threshold(p):
    """rowops.cu dropout_threshold of the fp32 p: trunc(p * 2^32) clamped to uint32."""
    t = float(np.float32(p)) * 4294967296.0
    return int(min(max(t, 0.0), 4294967295.0))


def inv_keep(p):
    """1.f / (1.f - p), both operations in fp32."""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


def lora_seed(step, fwd, layer, group, seed=7):
    """LlavaDPOPolicy._lora_seed for a LoraStore of `seed` (rng_seed = 0x5EED0000 + seed)."""
    g = ("qkv", "o", "gu", "down").index(group)
    return ((0x5EED0000 + seed) * 1000003 + step) * 4099 + (fwd * 131 + layer) * 4 + g


def sample_rows(M):
    """Rows the GPU cases replay: the first and last 64 and every 97th."""
    return sorted(set(range(64)) | set(range(M - 64, M)) | set(range(0, M, 97)))


def keep_rows(seed, rows, width, thresh):
    """Keep bits [len(rows), width] of the padded rows `rows` of a [*, width] activation."""
    r = np.asarray(rows, dtype=np.uint64)[:, None]
    return keep_bits(seed, r * np.uint64(width) + np.arange(width, dtype=np.uint64)[None, :], thresh)


def dropout_fwd_ref(x, keep, p):
    return torch.where(torch.from_numpy(keep), (x.float() * inv_keep(p)).to(BF), torch.zeros((), dtype=BF))


def dropout_bwd_ref(dx, g, keep, p):
    """dx + (keep ? fp32(g * inv) : 0) in fp32, then bf16: the kernel's select stands between its product and its
    sum, so nothing contracts."""
    t = torch.where(torch.from_numpy(keep), g.float() * inv_keep(p), torch.zeros(()))
    return (dx.float() + t).to(BF)


# ================================================================================================ LLaVA splice
P_IMG, V_TXT, MAX_LEN = 576, 32000, 2048
TRUNC_TOKEN = 31999        # occurs only in a tail the splice truncates
PAD_ID = 0                 # right padding (unk), part of each row as the collator builds it
# (padded width L, [(real length, image position or None)] for 8 sequences): chosen s and rejected s + 4 share an image
SPLICE_LAYOUTS = {
    "A": (1600, [(300, 0), (700, 31), (1000, 32), (1600, 1500), (450, 33), (1600, 35), (1200, None), (1600, 1599)]),
    "B": (900, [(900, 899), (300, 63), (640, 64), (800, None), (333, 0), (900, 31), (500, 32), (777, 35)]),
}


def splice_batch(layout, seed=0):
    """ids / labels [8, L]: text ids in [1, 31990), the first 40 % of each real prefix unsupervised, pad id 0 after it.
    Layout A puts TRUNC_TOKEN at positions 1550..1559 of sequence 5, which the splice cuts off."""
    L, seqs = SPLICE_LAYOUTS[layout]
    g = torch.Generator().manual_seed(seed)
    ids = torch.full((len(seqs), L), PAD_ID, dtype=torch.int64)
    labels = torch.full((len(seqs), L), IGNORE, dtype=torch.int64)
    for b, (n, img) in enumerate(seqs):
        ids[b, :n] = torch.randint(1, 31990, (n,), generator=g)
        labels[b, int(0.4 * n):n] = ids[b, int(0.4 * n):n]
        if img is not None:
            ids[b, img] = IMAGE
            labels[b, img] = IGNORE
    if layout == "A":
        ids[5, 1550:1560] = TRUNC_TOKEN
        labels[5, 1550:1560] = TRUNC_TOKEN
    img_index = (torch.arange(len(seqs)) % (len(seqs) // 2)).to(torch.int32)
    return ids, labels, img_index


def splice_map_ref(ids, labels, img_index, P=P_IMG, max_len=MAX_LEN):
    """The oracle map with slot k's block replaced by img_index[k] (the oracle numbers blocks by slot)."""
    src, new_labels, T = O.splice_index_map(ids, labels, P, max_len)
    r = -1 - src
    img = (src < 0) & (src != PAD)
    blk = img_index.long()[torch.where(img, r // P, 0)]
    src = torch.where(img, -1 - (blk * P + r % P), src)
    return src, new_labels, T


def token_weight_ref(src, tw):
    """splice_token_weight restated: the weight of spliced token t+1 is tw[s][j-1] when it is text token j >= 1, and 1
    otherwise."""
    nseq, T = src.shape
    Lw = tw.shape[1]
    out = torch.ones(nseq, T - 1, dtype=F32)
    s_l, w_l = src.tolist(), tw.tolist()
    for s in range(nseq):
        for t in range(T - 1):
            j = s_l[s][t + 1]
            if j >= 1 and j - 1 < Lw:
                out[s, t] = w_l[s][j - 1]
    return out


# ================================================================================================ OmniLMM in-place splice
OMNI_L, OMNI_Q = 2048, 64
OMNI_TOK = OM.OmniTokens(im_patch=32001, im_start=32002, im_end=32003)
# <im_start> positions of 8 sequences: lanes 30, 31 and 32 (= lane 0 of the next chunk) of a 32-token chunk, so the
# Q = 64 feature rows straddle two or three chunks; sequence 3 has no image, sequence 4 has two (the last ends at L-1)
OMNI_STARTS = [[30], [32 * 5 + 31], [32 * 10 + 32], [], [62, 32 * 61 + 30], [32 * 6 + 31], [32 * 20], [1000]]


def omni_batch(seed=3):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, 32000, (len(OMNI_STARTS), OMNI_L), generator=g)
    for b, starts in enumerate(OMNI_STARTS):
        for j in starts:
            ids[b, j] = OMNI_TOK.im_start
            ids[b, j + 1:j + 1 + OMNI_Q] = OMNI_TOK.im_patch
            ids[b, j + 1 + OMNI_Q] = OMNI_TOK.im_end
    n_slots = sum(len(s) for s in OMNI_STARTS)
    img_index = torch.tensor([0, 1, 2, 3, 1, 2, 3, 0][:n_slots], dtype=torch.int32)
    return ids, img_index


# ================================================================================================ CLIP / EVA front
# (images, size, patch, k_pad, width): LLaVA's CLIP-L/14-336 and OmniLMM's EVA tower (448/14, 1792)
PATCH_FRONTS = {"clip336": (9, 336, 14, 640, 1024), "eva448": (3, 448, 14, 640, 1792)}


def im2col_ref(img, patch, k_pad):
    N, C, S, _ = img.shape
    G = S // patch
    cols = img.reshape(N, C, G, patch, G, patch).permute(0, 2, 4, 1, 3, 5).reshape(N * G * G, C * patch * patch)
    return torch.cat((cols, torch.zeros(N * G * G, k_pad - cols.shape[1], dtype=img.dtype, device=img.device)), 1)


# ================================================================================================ compact head
CH_T, CH_H = 2048, 4096
CH_CAP = 1536              # cap = L, the text length of the batch


def compact_labels():
    """Spliced labels [8, 2048] with 0, 1536 (= cap, twice: mid-sequence and to the last position), a few scattered
    runs, one label at the last position, one at the first, and random densities."""
    g = torch.Generator().manual_seed(5)
    lab = torch.full((8, CH_T), IGNORE, dtype=torch.int64)
    tok = lambda n: torch.randint(1, 32000, (n,), generator=g)      # noqa: E731
    lab[1, 300:300 + CH_CAP] = tok(CH_CAP)
    for a, b in ((40, 50), (95, 97), (1000, 1400), (2040, 2048)):
        lab[2, a:b] = tok(b - a)
    lab[3, CH_T - 1] = 7
    on = torch.rand(CH_T, generator=g) < 0.3
    lab[4, on] = tok(int(on.sum()))
    lab[5, 1] = 9
    lab[6, CH_T - CH_CAP:] = tok(CH_CAP)
    on = torch.rand(CH_T, generator=g) < 0.1
    lab[7, on] = tok(int(on.sum()))
    return lab


def supervised_rows_ref(labels, cap):
    nseq, T = labels.shape
    rp = torch.full((nseq * cap,), -1, dtype=torch.int32)
    for s in range(nseq):
        t = (labels[s, 1:] != IGNORE).nonzero().flatten()
        assert t.numel() <= cap
        rp[s * cap:s * cap + t.numel()] = (s * T + t).to(torch.int32)
    return rp


# ================================================================================================ add_rows_bcast
# (rows M, table rows P, width, in place): EVA residual (P = M), resampler positions (P < M), and the two in-place
# calls as they are made: eva_tower.py d cls += (P = M = 1), resampler.py d query += (P = M = 64)
BCAST_CASES = {"eva_residual": (5 * 1025, 5 * 1025, 1792, False), "resampler_pos": (3 * 1024, 1024, 4096, False),
               "eva_cls_inplace": (1, 1, 1792, True), "resampler_query_inplace": (64, 64, 4096, True)}


def bcast_ref(x, t):
    P = t.shape[0]
    idx = torch.arange(x.shape[0], device=x.device) % P
    return (x.float() + t.float()[idx]).to(BF)


# ================================================================================================ CPU: discrimination
def _rope_cpu_case(kind, nh=4, nkv=2, T=64, seed=0):
    cos, sin = rope_tables(kind, T=T)
    g = torch.Generator().manual_seed(seed)
    M = 2 * T
    x = torch.randn(M, nh + nkv, HD, generator=g).to(BF)
    pos = torch.arange(M) % T
    return x, cos, sin, pos


def test_rope_bounds_accept_the_right_rotation_and_reject_swapped_halves_shifted_positions_and_q_heads_on_k():
    nh, nkv = 4, 2
    x, cos, sin, pos = _rope_cpu_case("skew", nh, nkv)
    c, s = cos[pos][:, None, :], sin[pos][:, None, :]
    right = rope_fwd_hf(x, c, s)
    ref, bd = rope_fwd_exact(x, c, s)
    assert within(right, ref, bd) and within(bf16(ref), ref, bd)
    h = HD // 2
    swap = lambda t: torch.cat((t[..., h:], t[..., :h]), -1)          # noqa: E731
    wrong_halves = rope_fwd_hf(x, swap(c), swap(s))
    nxt = (pos + 1).clamp(max=cos.shape[0] - 1)
    wrong_pos = rope_fwd_hf(x, cos[nxt][:, None, :], sin[nxt][:, None, :])
    wrong_heads = right.clone()
    wrong_heads[:, nh:] = rope_fwd_hf(x[:, :nkv], c, s)
    for name, wrong in (("halves", wrong_halves), ("pos+1", wrong_pos), ("k as q", wrong_heads)):
        assert not within(wrong, ref, bd), name
        assert not same_bits(wrong, right), name
    # the HF tables repeat their first half, which is why the GPU cases also run the skew tables
    hc, hs = rope_tables("hf", T=64)
    assert torch.equal(hc[:, :h], hc[:, h:]) and torch.equal(hs[:, :h], hs[:, h:])
    assert not torch.equal(cos[:, :h], cos[:, h:])

    # backward: the rounded fp64 transpose passes, the transpose with s1 / s2 swapped does not
    y = torch.randn(x.shape, generator=torch.Generator().manual_seed(1)).to(BF)
    bref, bbd = rope_bwd_exact(y, c, s)
    assert within(bf16(bref), bref, bbd)
    bad, _ = rope_bwd_exact(y, c, swap(s))
    assert not within(bf16(bad), bref, bbd)
    # an fp32 dQ: the bound also takes the kernel's fp32 arithmetic, FMA-contracted or not
    yq = torch.randn(x.shape, generator=torch.Generator().manual_seed(2), dtype=F32)
    qref, qbd = rope_bwd_exact(yq, c, s)
    y1, y2 = yq[..., :h], yq[..., h:]
    c32, s32 = c.float(), s.float()
    plain = torch.cat((y1 * c32[..., :h] + y2 * s32[..., h:], y2 * c32[..., h:] - y1 * s32[..., :h]), -1)
    assert within(plain.to(BF), qref, qbd)


def test_rope_fwd_bound_rejects_an_hf_rounding_slip():
    """The bit-exact HF comparison is the sharp check; the fp64 bound still rejects results off by a bf16 ulp in the
    smallest elements."""
    x, cos, sin, pos = _rope_cpu_case("hf")
    c, s = cos[pos][:, None, :], sin[pos][:, None, :]
    ref, bd = rope_fwd_exact(x, c, s)
    right = rope_fwd_hf(x, c, s)
    wrong = right.to(F64) + 2.0 * ulp_bf16(right.to(F64))
    assert within(right, ref, bd) and not within(wrong, ref, bd)


def test_dropout_replay_is_splitmix64_and_rejects_a_shifted_or_chunk_shared_mask():
    # splitmix64 from state 0 first returns 0xE220A8397B1DCDAF (Vigna's reference generator); mix32(0) is its high word
    assert int(mix32(np.zeros(1, dtype=np.uint64))[0]) == 0xE220A839
    p, W = 0.25, 4096
    seed = lora_seed(3, 2, 17, "gu")
    th = dropout_threshold(p)
    assert th == 1 << 30 and dropout_threshold(0.0) == 0
    keep = keep_rows(seed, [0, 5, 1023], W, th)
    x = torch.randn(3, W, generator=torch.Generator().manual_seed(0)).to(BF)
    right = dropout_fwd_ref(x, keep, p)
    shifted = dropout_fwd_ref(x, np.roll(keep, 1, axis=1), p)
    rows = np.array([0, 5, 1023], dtype=np.uint64)[:, None] * np.uint64(W)
    chunk_only = keep_bits(seed, rows + (np.arange(W, dtype=np.uint64) // np.uint64(8) * np.uint64(8))[None, :], th)
    assert not same_bits(shifted, right)
    assert not np.array_equal(chunk_only, keep)
    assert keep_bits(seed, np.arange(4096, dtype=np.uint64), dropout_threshold(0.0)).all()
    # a kept value is bf16(x * fp32(1/(1-p))); p = 0 keeps every element and multiplies by exactly 1
    assert inv_keep(0.0) == 1.0 and inv_keep(0.05) == float(np.float32(1) / np.float32(0.95))


def test_lora_seed_restatement_matches_the_policy():
    from rlaifv_b200.model import LlavaDPOPolicy

    class Stub:
        lora = type("L", (), {"rng_seed": 0x5EED0000 + 7, "step": 12})()
        _fwd_count = 3

    for i, group in ((0, "qkv"), (31, "down"), (17, "gu")):
        assert LlavaDPOPolicy._lora_seed(Stub(), i, group) == lora_seed(12, 3, i, group)
    assert lora_seed(12, 3, 5, "qkv") < 2 ** 64


@pytest.mark.parametrize("W", [4096, 11008])
def test_dropout_mask_statistics_at_the_step_shape(W):
    """18 160 x W elements (the 7B LoRA step's packed rows), p = 0.05, on the replay: the keep rate per column and per
    position j of the 8-element chunk are within 6 sigma of the binomial, and at W = 4096 so is the joint drop rate
    (p^2) under the seeds of the neighbouring linear group, layer, micro-batch forward and step."""
    M, p = 18160, 0.05
    th = dropout_threshold(p)
    q = th / 2.0 ** 32                                       # drop probability of a uniform 32-bit hash
    base = lora_seed(40, 2, 9, "qkv")
    nbrs = {"group": lora_seed(40, 2, 9, "o"), "layer": lora_seed(40, 2, 10, "qkv"),
            "forward": lora_seed(40, 3, 9, "qkv"), "step": lora_seed(41, 2, 9, "qkv")}
    assert len({base, *nbrs.values()}) == 5
    col_keep = np.zeros(W, dtype=np.int64)
    joint = dict.fromkeys(nbrs, 0)
    cols = np.arange(W, dtype=np.uint64)
    for r0 in range(0, M, 1024):
        r = np.arange(r0, min(M, r0 + 1024), dtype=np.uint64)
        el = r[:, None] * np.uint64(W) + cols[None, :]
        drop = ~keep_bits(base, el, th)
        col_keep += (~drop).sum(0)
        if W == 4096:
            for k, sd in nbrs.items():
                joint[k] += int((drop & ~keep_bits(sd, el, th)).sum())
    z = lambda got, n, pr: abs(got - n * pr) / math.sqrt(n * pr * (1 - pr))   # noqa: E731
    zc = max(z(int(k), M, 1 - q) for k in col_keep)
    zj = max(z(int(k), M * W // 8, 1 - q) for k in col_keep.reshape(-1, 8).sum(0))
    print("dropout W=%d: worst column z %.2f, worst chunk-lane z %.2f" % (W, zc, zj))
    assert zc < 6 and zj < 6
    for k, n in joint.items() if W == 4096 else ():
        zk = z(n, M * W, q * q)
        print("dropout joint drop vs %s neighbour: %.6f (p^2 = %.6f), z %.2f" % (k, n / (M * W), q * q, zk))
        assert zk < 6, k


def test_splice_references_reject_an_image_one_chunk_late_and_token_weights_off_by_one():
    """The map a kernel would write if it spliced sequence 5's image (at lane 31) one 32-token chunk late: the image's
    P rows start 32 positions later and the 32 text rows after it move up. The rows that map gathers differ from the
    reference's in that sequence only."""
    ids, labels, img_index = splice_batch("B")
    src, _, T = splice_map_ref(ids, labels, img_index)
    b, o = 5, 31
    late = src.clone()
    late[b, o:o + 32], late[b, o + 32:o + 32 + P_IMG] = src[b, o + P_IMG:o + P_IMG + 32], src[b, o:o + P_IMG]
    H = 8
    g = torch.Generator().manual_seed(4)
    params = {"model.embed_tokens.weight": torch.randn(V_TXT, H, generator=g).to(BF)}
    feat = torch.randn(ids.shape[0] // 2, P_IMG, H, generator=g).to(BF)
    right = O.splice_embeds(params, ids, src, feat)
    wrong = O.splice_embeds(params, ids, late, feat)
    assert not torch.equal(late, src) and not same_bits(wrong, right)
    assert same_bits(wrong[torch.arange(ids.shape[0]) != b], right[torch.arange(ids.shape[0]) != b])
    tw = torch.rand(ids.shape[0], ids.shape[1] - 1, generator=torch.Generator().manual_seed(1))
    right = token_weight_ref(src, tw)
    shifted = torch.cat((torch.ones(tw.shape[0], 1), tw[:, :-1]), 1)   # tw[j] read where tw[j - 1] belongs
    assert not torch.equal(token_weight_ref(src, shifted), right)


def test_scatter_bound_admits_any_order_and_rejects_a_lost_term():
    """gamma_{n-1}: zero for n <= 1 (0 + a is exact), and for n = 2 the one rounding of a + b, the same in either
    order; three or more terms leave room for the atomics' order, not for a lost term."""
    g = torch.Generator().manual_seed(0)
    terms = torch.randn(200, 16, generator=g).to(BF).to(F64)
    ref = terms.sum(0)
    bd = gam(199) * terms.abs().sum(0)
    fwd, rev = torch.zeros(16, dtype=F32), torch.zeros(16, dtype=F32)
    for t in terms.to(F32):
        fwd = fwd + t
    for t in terms.to(F32).flip(0):
        rev = rev + t
    assert within(fwd, ref, bd) and within(rev, ref, bd)
    assert not within(fwd - terms[0].to(F32), ref, bd)
    assert torch.equal(terms[0].to(F32) + terms[1].to(F32), (terms[0] + terms[1]).to(F32))


# ================================================================================================ CPU: premises
GRID_STRIDE_KERNELS = ["rope_fwd_kernel", "rope_bwd_kernel", "rope_pos_fwd_kernel", "rope_pos_bwd_kernel",
                       "dropout_fwd_kernel", "dropout_bwd_add_kernel", "dropout_rows_kernel", "im2col_patch_kernel",
                       "clip_embed_kernel", "drop_cls_kernel", "splice_gather_kernel", "splice_scatter_kernel",
                       "rows_gather_kernel", "rows_scatter_kernel", "splice_token_weight_kernel"]


def test_premise_launch_code_is_what_the_geometry_mirrors():
    """grid_for and THREADS above restate rowops.cu's launches; this reads them there, so a changed launch fails here
    instead of leaving the wrap premises below computed from stale constants."""
    src = open(os.path.join(REPO, "rlaif-v_b200", "csrc", "rowops.cu")).read()
    assert re.search(r"static inline int grid_for\(long long work_items, int threads, int max_blocks_per_sm = 8\) \{"
                     r"\s*long long blocks = \(work_items \+ threads - 1\) / threads;"
                     r"\s*long long cap = \(long long\)num_sms\(\) \* max_blocks_per_sm;", src)
    for k in GRID_STRIDE_KERNELS:
        launches = src.count(k + "<<<")
        same = re.findall(re.escape(k) + r"<<<grid_for\([^;]*?, %d\), %d, 0, ST>>>" % (THREADS, THREADS), src)
        assert launches >= 1 and len(same) == launches, k
    bcast = src[src.index("extern \"C\" int rlaifv_add_rows_bcast"):]
    bcast = bcast[:bcast.index("return 0;")]
    assert "(total + 255) / 256" in bcast and "(long long)num_sms() * 16" in bcast
    assert "add_rows_bcast_kernel<<<(int)blocks, %d, 0, ST>>>" % THREADS in bcast


def test_premise_grid_stride_loops_wrap_at_least_twice():
    sms = H100_SMS
    loops = {}
    for model, (nh, nkv) in ROPE_DIMS.items():
        loops["rope %s" % model] = rope_work(8 * T_ROPE, nh, nkv)
        loops["rope_pos %s" % model] = rope_work(sum(RAGGED_LENS), nh, nkv)
    for W in DROP_WIDTHS:
        loops["dropout %d" % W] = DROP_M * W // 8
        loops["dropout_rows %d" % W] = DROP_PACKED * W // 8
    for name, (N, S, P, k_pad, H) in PATCH_FRONTS.items():
        G = S // P
        loops["im2col %s" % name] = N * G * G * k_pad
        loops["clip_embed %s" % name] = N * (G * G + 1) * (H // 8)
        loops["drop_cls %s" % name] = N * G * G * (H // 8)
    loops["rows_gather/scatter"] = 8 * CH_CAP * (CH_H // 8)
    for name, work in loops.items():
        assert full_passes(work, grid_for(work, sms=sms)) >= 2, name
    for name, (M, P, H, inplace) in BCAST_CASES.items():
        work = M * (H // 8)
        grid = max(1, min(-(-work // THREADS), sms * 16))                  # rlaifv_add_rows_bcast: 16 CTAs per SM
        assert inplace or full_passes(work, grid) >= 2, name
    # the splice gather / scatter run one warp per spliced row: layout A's 8 x 2048 rows outnumber the warps. Two loops
    # cannot wrap at the step's shape: splice_token_weight gets a thread per position (8 x 2047 < one grid), and
    # supervised_rows is one warp per sequence, scanning its 2047 positions serially.
    rows = 8 * MAX_LEN
    assert rows > grid_for(rows * 32, sms=sms) * (THREADS // 32)


def test_premise_splice_layouts_reach_later_chunks_truncation_shared_blocks_and_repeats():
    lanes, cut_inside, cut_after = set(), 0, 0
    for layout, (L, seqs) in SPLICE_LAYOUTS.items():
        ids, labels, img_index = splice_batch(layout)
        src, _, T = splice_map_ref(ids, labels, img_index)
        for n, img in seqs:
            if img is None:
                continue
            lanes.add(img)
            end = img + P_IMG                    # spliced position after the image
            cut_inside += img < MAX_LEN < end
            cut_after += end < MAX_LEN < L - 1 + P_IMG
        assert any(img is None for _, img in seqs)
        assert 300 <= min(n for n, _ in seqs) and max(n for n, _ in seqs) <= 1600
        # two slots share a block and both splice it
        blocks = [-1 - s for s in src.flatten().tolist() if s < 0 and s != PAD]
        assert max(np.bincount(blocks)) == 2
        assert max(np.bincount(ids[ids >= 0].flatten().numpy())) >= 100
        if layout == "A":
            assert T == MAX_LEN and bool((ids == TRUNC_TOKEN).any())
            assert not bool((ids.gather(1, src.clamp(min=0)) == TRUNC_TOKEN).any())
    assert {0, 31, 32, 33, 35, 63, 64} <= lanes and 1599 in lanes and 899 in lanes     # and L - 1 of both layouts
    assert max(lanes) > 31 and cut_inside >= 1 and cut_after >= 1
    # the in-place splice: starts at lanes 30, 31 and 0 of a chunk, rows across chunk boundaries
    starts = [j for s in OMNI_STARTS for j in s]
    assert {j % 32 for j in starts} >= {30, 31, 0} and max(starts) + OMNI_Q + 1 == OMNI_L - 1


def test_premise_a_supervised_segment_is_exactly_full():
    lab = compact_labels()
    counts = (lab[:, 1:] != IGNORE).sum(1).tolist()
    assert 0 in counts and counts.count(CH_CAP) == 2 and max(counts) == CH_CAP and CH_T - 1 > CH_CAP


# ================================================================================================ GPU: RoPE
@pytest.mark.gpu
@pytest.mark.parametrize("table", ["hf", "skew"])
@pytest.mark.parametrize("model", list(ROPE_DIMS))
def test_rope_fwd_bit_exact_and_within_fp64(model, table):
    from rlaifv_b200 import ops
    nh, nkv = ROPE_DIMS[model]
    W = (nh + 2 * nkv) * HD
    cos, sin = [t.to(DEV) for t in rope_tables(table)]
    gen = torch.Generator(device=DEV).manual_seed(2 * list(ROPE_DIMS).index(model) + (table == "skew"))
    for form in ("rows", "pos"):
        if form == "rows":
            M = 8 * T_ROPE
            pos = torch.arange(M, device=DEV) % T_ROPE
        else:
            pos = ragged_positions(RAGGED_LENS).to(DEV)
            M = pos.numel()
        x0 = torch.randn(M, W, device=DEV, generator=gen).to(BF)
        qkv = x0.clone()
        if form == "rows":
            ops.rope_fwd(qkv, cos, sin, T_ROPE, nh, HD, n_kv_heads=nkv)
        else:
            ops.rope_pos_fwd(qkv, cos, sin, pos.to(torch.int32), nh, HD, n_kv_heads=nkv)
        torch.cuda.synchronize()
        w = Worst("rope_fwd %s %s %s M=%d" % (form, model, table, M))
        for r0 in range(0, M, 2048):
            sl = slice(r0, min(M, r0 + 2048))
            x = rot_heads(x0[sl], nh, nkv)
            c, s = cos[pos[sl]][:, None, :], sin[pos[sl]][:, None, :]
            got = rot_heads(qkv[sl], nh, nkv)
            assert same_bits(got, rope_fwd_hf(x, c, s)), "rope_fwd %s: not the HF bits at rows %s" % (form, sl)
            w.check(got, *rope_fwd_exact(x, c, s))
        assert same_bits(qkv[:, (nh + nkv) * HD:], x0[:, (nh + nkv) * HD:]), "v block changed"
        w.done()


@pytest.mark.gpu
@pytest.mark.parametrize("table", ["hf", "skew"])
@pytest.mark.parametrize("model", list(ROPE_DIMS))
def test_rope_bwd_within_fp64_transpose(model, table):
    """split (dQ in the q block, bf16), fp32-dQ (q block overwritten from dq_f32; GQA included) and packed rows."""
    from rlaifv_b200 import ops
    nh, nkv = ROPE_DIMS[model]
    W = (nh + 2 * nkv) * HD
    cos, sin = [t.to(DEV) for t in rope_tables(table)]
    gen = torch.Generator(device=DEV).manual_seed(7 + 2 * list(ROPE_DIMS).index(model) + (table == "skew"))
    for form in ("split", "dq_f32", "pos"):
        if form == "pos":
            pos = ragged_positions(RAGGED_LENS).to(DEV)
            M = pos.numel()
        else:
            M = 8 * T_ROPE
            pos = torch.arange(M, device=DEV) % T_ROPE
        dy0 = torch.randn(M, W, device=DEV, generator=gen).to(BF)
        d = dy0.clone()
        dq = None
        if form == "dq_f32":
            dq = torch.randn(M, nh * HD, device=DEV, generator=gen)
            d[:, :nh * HD] = float("nan")                   # the kernel must overwrite the q block from dq_f32
            ops.rope_bwd(d, dq, cos, sin, T_ROPE, nh, HD, n_kv_heads=nkv)
        elif form == "split":
            ops.rope_bwd(d, None, cos, sin, T_ROPE, nh, HD, n_kv_heads=nkv)
        else:
            ops.rope_pos_bwd(d, cos, sin, pos.to(torch.int32), nh, HD, n_kv_heads=nkv)
        torch.cuda.synchronize()
        w = Worst("rope_bwd %s %s %s M=%d" % (form, model, table, M))
        for r0 in range(0, M, 2048):
            sl = slice(r0, min(M, r0 + 2048))
            y = rot_heads(dy0[sl], nh, nkv).to(F64)
            if dq is not None:
                y[:, :nh] = dq[sl].view(-1, nh, HD).to(F64)
            c, s = cos[pos[sl]][:, None, :], sin[pos[sl]][:, None, :]
            w.check(rot_heads(d[sl], nh, nkv), *rope_bwd_exact(y, c, s))
        assert same_bits(d[:, (nh + nkv) * HD:], dy0[:, (nh + nkv) * HD:]), "v block changed"
        w.done()


# ================================================================================================ GPU: dropout
@pytest.mark.gpu
@pytest.mark.parametrize("W", DROP_WIDTHS)
def test_dropout_masks_and_values_bit_exact_against_the_hash_replay(W):
    """All four forms at M = 9081 (packed: 6007 of them), p in {0, 0.05, 0.25}, seeds of _lora_seed's formula. The
    replay covers the first and last 64 rows and every 97th row (222 padded rows, 127 packed rows); p = 0 is checked
    on every element."""
    from rlaifv_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(W)
    cpu = torch.Generator().manual_seed(W)
    M, Mp = DROP_M, DROP_PACKED
    rows = torch.randperm(M, generator=cpu)[:Mp].sort().values.to(torch.int32)
    R, Rp = sample_rows(M), sample_rows(Mp)
    rows_d = rows.to(DEV)
    for k, p in enumerate(DROP_PS):
        seed = lora_seed(100 + k, 1 + k, 31 - k, ("qkv", "gu", "down")[k])
        th = dropout_threshold(p)
        x = torch.randn(M, W, device=DEV, generator=gen).to(BF)
        x = torch.where(x == 0, torch.ones((), dtype=BF, device=DEV), x)      # a zero output is a dropped element
        out = ops.dropout_fwd(x, p, seed)
        dx0 = torch.randn(M, W, device=DEV, generator=gen).to(BF)
        g = torch.randn(M, W, device=DEV, generator=gen).to(BF)
        dx = dx0.clone()
        ops.dropout_bwd_add(dx, g, p, seed)
        xp, gp, dxp0 = x[:Mp].clone(), g[:Mp].clone(), dx0[:Mp].clone()
        outp = ops.dropout_fwd(xp, p, seed, rows=rows_d)
        dxp = dxp0.clone()
        ops.dropout_bwd_add(dxp, gp, p, seed, rows=rows_d)
        torch.cuda.synchronize()
        if p == 0:
            assert same_bits(out, x) and same_bits(outp, xp), "p = 0 is not the identity"
        keep = keep_rows(seed, R, W, th)
        keep_p = keep_rows(seed, rows[Rp].tolist(), W, th)
        xs, outs = x[R].cpu(), out[R].cpu()
        assert np.array_equal((outs != 0).numpy(), keep), "dropout_fwd W=%d p=%g: mask differs" % (W, p)
        assert same_bits(outs, dropout_fwd_ref(xs, keep, p)), "dropout_fwd W=%d p=%g: kept values differ" % (W, p)
        assert same_bits(dx[R].cpu(), dropout_bwd_ref(dx0[R].cpu(), g[R].cpu(), keep, p)), \
            "dropout_bwd_add W=%d p=%g" % (W, p)
        outps = outp[Rp].cpu()
        assert np.array_equal((outps != 0).numpy(), keep_p), "dropout_rows_fwd W=%d p=%g: mask differs" % (W, p)
        assert same_bits(outps, dropout_fwd_ref(xp[Rp].cpu(), keep_p, p)), "dropout_rows_fwd W=%d p=%g" % (W, p)
        assert same_bits(dxp[Rp].cpu(), dropout_bwd_ref(dxp0[Rp].cpu(), gp[Rp].cpu(), keep_p, p)), \
            "dropout_rows_bwd_add W=%d p=%g" % (W, p)
        print("dropout W=%d p=%g: keep rate %.5f on the replayed rows" % (W, p, keep.mean()))


# ================================================================================================ GPU: LLaVA splice
@pytest.mark.gpu
@pytest.mark.parametrize("layout,H", [("A", 4096), ("B", 5120)])
def test_llava_splice_at_step_scale(layout, H):
    from rlaifv_b200 import ops
    ids, labels, img_index = splice_batch(layout)
    src_r, lab_r, T = splice_map_ref(ids, labels, img_index)
    nseq, L = ids.shape
    ids_d, lab_d, idx_d = ids.to(DEV), labels.to(DEV), img_index.to(DEV)
    n_img, lens = ops.splice_count(ids_d, P_IMG, MAX_LEN)
    assert torch.equal(n_img.cpu(), (ids == IMAGE).sum(1).to(torch.int32))
    assert torch.equal(lens.cpu(), (src_r != PAD).sum(1).to(torch.int32))
    assert int(lens.max()) == T
    src, new_labels = ops.splice_map(ids_d, lab_d, n_img, idx_d, P_IMG, T, MAX_LEN)
    torch.cuda.synchronize()
    assert torch.equal(src.cpu().long(), src_r), "splice_map src"
    assert torch.equal(new_labels.cpu(), lab_r), "splice_map labels"

    gen = torch.Generator(device=DEV).manual_seed(H)
    embed = torch.randn(V_TXT, H, device=DEV, generator=gen).to(BF)
    n_blocks = nseq // 2
    feat = torch.randn(n_blocks * P_IMG, H, device=DEV, generator=gen).to(BF)
    out = ops.splice_gather(src, ids_d, embed, feat)
    torch.cuda.synchronize()
    ref = O.splice_embeds({"model.embed_tokens.weight": embed.cpu()}, ids, src_r, feat.cpu().view(n_blocks, P_IMG, H))
    assert same_bits(out.cpu().view(nseq, T, H), ref), "splice_gather"

    # backward: every row of dx non-zero, pad rows included (the scatter must skip them)
    dx = torch.randn(nseq * T, H, device=DEV, generator=gen).to(BF)
    d_embed = torch.zeros(V_TXT, H, device=DEV)
    d_feat = torch.zeros(n_blocks * P_IMG, H, device=DEV)
    ops.splice_scatter(src, ids_d, dx, d_embed, d_feat)
    torch.cuda.synchronize()
    flat = src_r.flatten().to(DEV)
    row_b = torch.arange(nseq * T, device=DEV) // T
    tok = flat >= 0
    tid = ids_d[row_b[tok], flat[tok]]
    img = (flat < 0) & (flat != PAD)
    fr = -1 - flat[img]
    dx64 = dx.to(F64)
    d_tok = dx64[tok]
    # feature rows: at most two terms (the pair's two sequences), each sum one fp32 rounding of exact bf16 values
    f_ref = torch.zeros(n_blocks * P_IMG, H, dtype=F64, device=DEV).index_add_(0, fr, dx64[img])
    f_cnt = torch.bincount(fr, minlength=n_blocks * P_IMG)
    assert int(f_cnt.max()) == 2 and int((f_cnt == 2).sum()) >= P_IMG
    assert same_bits(d_feat, f_ref.to(F32)), "splice_scatter d_feat"
    # token rows: n terms per id, n - 1 roundings after the exact first one
    n_tok = torch.bincount(tid, minlength=V_TXT)
    w = Worst("splice_scatter d_embed %s H=%d (max n %d)" % (layout, H, int(n_tok.max())))
    for v0 in range(0, V_TXT, 4000):
        vs = slice(v0, v0 + 4000)
        sel = (tid >= v0) & (tid < v0 + 4000)
        e_ref = torch.zeros(4000, H, dtype=F64, device=DEV).index_add_(0, tid[sel] - v0, d_tok[sel])
        e_abs = torch.zeros(4000, H, dtype=F64, device=DEV).index_add_(0, tid[sel] - v0, d_tok[sel].abs())
        nv = n_tok[vs].to(F64)
        bound = ((nv - 1).clamp(min=0) * U / (1 - (nv - 1).clamp(min=0) * U))[:, None] * e_abs
        w.check(d_embed[vs], e_ref, bound)
    if layout == "A":
        assert int(n_tok[TRUNC_TOKEN]) == 0 and not bool(d_embed[TRUNC_TOKEN].any()), "a truncated token was scattered"
    assert int(n_tok.max()) >= 100
    w.done()

    # token weights in spliced positions, text weights of length Lw = L - 1 as the collator builds them
    tw = torch.rand(nseq, L - 1, generator=torch.Generator().manual_seed(2))
    got = ops.splice_token_weight(src, tw.to(DEV), T)
    torch.cuda.synchronize()
    assert same_bits(got.cpu(), token_weight_ref(src_r, tw)), "splice_token_weight"


@pytest.mark.gpu
def test_omnilmm_inplace_splice_at_step_scale_and_status_bits():
    from rlaifv_b200 import ops
    ids, img_index = omni_batch()
    tok = OMNI_TOK
    src, status = ops.splice_map_inplace(ids.to(DEV), img_index.to(DEV), OMNI_Q, tok.im_patch, tok.im_start,
                                         tok.im_end)
    torch.cuda.synchronize()
    assert int(status) == 0
    ref = OM.inplace_splice_map(ids, tok, OMNI_Q, image_of_slot=img_index)
    assert torch.equal(src.cpu().long(), ref), "splice_map_inplace"
    # bit 0: an <im_start> without its <im_end>
    bad = ids.clone()
    j = OMNI_STARTS[1][0]
    bad[1, j + 1 + OMNI_Q] = 5
    _, status = ops.splice_map_inplace(bad.to(DEV), img_index.to(DEV), OMNI_Q, tok.im_patch, tok.im_start, tok.im_end)
    assert int(status) == 1
    with pytest.raises(ValueError):
        OM.inplace_splice_map(bad, tok, OMNI_Q, image_of_slot=img_index)
    # bit 1: the <im_end> one row late (Q + 1 patches), counts still equal
    bad = ids.clone()
    j = OMNI_STARTS[2][0]
    bad[2, j + 1 + OMNI_Q] = tok.im_patch
    bad[2, j + 2 + OMNI_Q] = tok.im_end
    _, status = ops.splice_map_inplace(bad.to(DEV), img_index.to(DEV), OMNI_Q, tok.im_patch, tok.im_start, tok.im_end)
    assert int(status) == 2
    with pytest.raises(ValueError):
        OM.inplace_splice_map(bad, tok, OMNI_Q, image_of_slot=img_index)


# ================================================================================================ GPU: patch front
@pytest.mark.gpu
@pytest.mark.parametrize("front", list(PATCH_FRONTS))
def test_clip_eva_patch_front_bit_exact(front):
    from rlaifv_b200 import ops
    N, S, P, k_pad, H = PATCH_FRONTS[front]
    G = S // P
    NP = G * G
    gen = torch.Generator(device=DEV).manual_seed(S)
    img = torch.randn(N, 3, S, S, device=DEV, generator=gen).to(BF)
    cols = ops.clip_im2col(img, P, k_pad)
    patch = torch.randn(N * NP, H, device=DEV, generator=gen).to(BF)
    cls = torch.randn(H, device=DEV, generator=gen).to(BF)
    pos = torch.randn(NP + 1, H, device=DEV, generator=gen).to(BF)
    x = ops.clip_embed(patch, cls, pos, N, NP)
    y = torch.randn(N * (NP + 1), H, device=DEV, generator=gen).to(BF)
    dropped = ops.clip_drop_cls(y, N, NP)
    torch.cuda.synchronize()
    ref = im2col_ref(img, P, k_pad)
    assert same_bits(cols, ref), "clip_im2col"
    assert not bool(cols[:, 3 * P * P:].view(torch.int16).any()), "im2col pad columns"
    emb = torch.cat((cls.view(1, 1, H).expand(N, 1, H), patch.view(N, NP, H)), 1) + pos
    assert same_bits(x.view(N, NP + 1, H), emb), "clip_embed"
    assert same_bits(dropped.view(N, NP, H), y.view(N, NP + 1, H)[:, 1:]), "clip_drop_cls"


# ================================================================================================ GPU: compact head
@pytest.mark.gpu
def test_compact_head_rows_bit_exact():
    from rlaifv_b200 import ops
    from rlaifv_b200.model import pack_rows
    lab = compact_labels()
    nseq = lab.shape[0]
    rp = ops.supervised_rows(lab.to(DEV), CH_CAP)
    torch.cuda.synchronize()
    rp_ref = supervised_rows_ref(lab, CH_CAP)
    assert torch.equal(rp.cpu(), rp_ref), "supervised_rows"
    gen = torch.Generator(device=DEV).manual_seed(9)
    x = torch.randn(nseq * CH_T, CH_H, device=DEV, generator=gen).to(BF)
    zero = torch.zeros((), dtype=BF, device=DEV)
    g_pad = ops.rows_gather(rp, x)
    ref = torch.where((rp >= 0)[:, None], x[rp.long().clamp(min=0)], zero)
    assert same_bits(g_pad, ref), "rows_gather padded"
    pk = pack_rows(lab.to(DEV))
    assert pk is not None and pk.M < nseq * CH_T
    xp = ops.rows_gather(pk.rows, x)
    assert same_bits(xp, x[pk.rows.long()]), "rows_gather packing"
    xr = pk.packed_rows(rp)
    assert same_bits(ops.rows_gather(xr, xp), ref), "rows_gather through packed_rows"
    dy = torch.randn(rp.numel(), CH_H, device=DEV, generator=gen).to(BF)
    for name, index, rows in (("padded", rp, nseq * CH_T), ("packed", xr, pk.M)):
        dx = torch.full((rows, CH_H), 0x7FC1, dtype=torch.int16, device=DEV).view(BF)      # a NaN no kernel writes
        ops.rows_scatter(index, dy, dx)
        want = torch.full((rows, CH_H), 0x7FC1, dtype=torch.int16, device=DEV).view(BF)
        on = index >= 0
        want[index[on].long()] = dy[on]
        torch.cuda.synchronize()
        assert same_bits(dx, want), "rows_scatter %s" % name


# ================================================================================================ GPU: add_rows_bcast
@pytest.mark.gpu
@pytest.mark.parametrize("case", list(BCAST_CASES))
def test_add_rows_bcast_bit_exact(case):
    from rlaifv_b200 import ops
    M, P, H, inplace = BCAST_CASES[case]
    gen = torch.Generator(device=DEV).manual_seed(M + H)
    x = torch.randn(M, H, device=DEV, generator=gen).to(BF)
    t = torch.randn(P, H, device=DEV, generator=gen).to(BF)
    ref = bcast_ref(x, t)
    if inplace:
        out = ops.add_rows_bcast(x, t, out=x)
        assert out.data_ptr() == x.data_ptr()
    else:
        out = ops.add_rows_bcast(x, t)
    torch.cuda.synchronize()
    assert same_bits(out, ref), case

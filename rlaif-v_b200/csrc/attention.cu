// Fused attention for sm_90a on wgmma: S = Q K^T and O += P V run on the warpgroup tensor cores with the S / O
// accumulators in registers; P never leaves the registers (it is the A operand of the PV wgmma). K / V (or Q / dO)
// stream through a TMA-fed two-stage shared-memory ring.
//
//   forward  (attention_fwd_kernel): one CTA per (128-row query tile, head, sequence). Causal d=128 (Llama; HF
//             llama/modeling_llama.py:199-222, attention_mask=None => pure causal, pads attended —
//             muffin/train/trainers.py:199), non-causal d=64 (CLIP; HF clip/modeling_clip.py:261-279) and d=128 (EVA
//             tower, heads padded 112 -> 128; resampler cross-attention). Softmax in fp32, P rounded to bf16 before PV.
//   backward (attention_bwd_dkv_kernel + attention_bwd_dq_kernel): dK/dV per 128-row K/V tile streaming 64-row chunks
//             of Q / dO, dQ per 128-row Q tile streaming 64-row chunks of K / V; S / dP are recomputed in each. dQ is
//             written once as bf16, or reduced into an fp32 buffer (the resampler's shared queries sum over images).
//
// Warp roles (288 threads): warpgroups 0, 1 = math, 64 rows each (thread = two rows of the wgmma accumulator layout,
// see common.cuh); warp 8 = TMA producer (one thread issues).
// Layouts: q/k/v/o are [nseq*S rows][ld] bf16 with head h at columns [h*D, h*D+D); q, k, v may be
// column blocks of one fused qkv buffer. LSE is fp32 [nseq][n_heads][S] (natural log).
#include "common.cuh"
#include "host_util.h"

namespace b200 {

constexpr int ATT_BQ = 128;
constexpr int ATT_BKV = 128;
constexpr int ATT_THREADS = 288;   // two math warpgroups + one producer warp
constexpr int ATT_STAGES = 2;
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

__device__ __forceinline__ float fast_exp2(float x) {   // MUFU.EX2, flush-to-zero (inputs are <= ~8)
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// the two rows of the 64-row block a thread holds, and its first column in every 8-column group
struct FragPos {
  int r0;   // row of d[4i], d[4i+1]; row r0 + 8 holds d[4i+2], d[4i+3]
  int c0;   // column of d[4i] is 8i + c0
};
__device__ __forceinline__ FragPos frag_pos() {
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  return FragPos{w * 16 + (lane >> 2), (lane & 3) * 2};
}

// wgmma accumulator of a 64 x (16*KS) tile -> bf16 A fragments of KS k16 steps
template <int KS>
__device__ __forceinline__ void acc_to_afrag(const float* d, uint32_t (&a)[KS][4]) {
#pragma unroll
  for (int k = 0; k < KS; ++k) {
    a[k][0] = pack_bf16(d[8 * k + 0], d[8 * k + 1]);
    a[k][1] = pack_bf16(d[8 * k + 2], d[8 * k + 3]);
    a[k][2] = pack_bf16(d[8 * k + 4], d[8 * k + 5]);
    a[k][3] = pack_bf16(d[8 * k + 6], d[8 * k + 7]);
  }
}

// S[64 x 64*NB] = A[64 rows of a K-major tile] * B[64*NB rows of a K-major tile]^T over D (both stored as D/64 atoms)
template <int D>
__device__ __forceinline__ void mma_qk_64(float (&s)[32], uint32_t a_addr, uint32_t a_atom, uint32_t b_addr,
                                          uint32_t b_atom) {
#pragma unroll
  for (int k16 = 0; k16 < D / 16; ++k16)
    wgmma_m64n64_ss<0, 0>(s, desc_kmajor(a_addr + (k16 >> 2) * a_atom, k16 & 3),
                          desc_kmajor(b_addr + (k16 >> 2) * b_atom, k16 & 3), k16 > 0);
}
template <int D>
__device__ __forceinline__ void mma_qk_128(float (&s)[64], uint32_t a_addr, uint32_t a_atom, uint32_t b_addr,
                                           uint32_t b_atom) {
#pragma unroll
  for (int k16 = 0; k16 < D / 16; ++k16)
    wgmma_m64n128_ss<0, 0>(s, desc_kmajor(a_addr + (k16 >> 2) * a_atom, k16 & 3),
                           desc_kmajor(b_addr + (k16 >> 2) * b_atom, k16 & 3), k16 > 0);
}
// O[64 x D] += P[64 x 16*KS] (registers) * V[16*KS rows][D] (MN-major B: D/64 atoms of [rows][64], atom stride given)
template <int D, int KS>
__device__ __forceinline__ void mma_pv(float (&o)[D / 2], const uint32_t (&p)[KS][4], uint32_t v_addr,
                                       uint32_t v_atom) {
#pragma unroll
  for (int k = 0; k < KS; ++k) {
    if constexpr (D == 128) wgmma_m64n128_rs<1>(o, p[k], desc_mnmajor(v_addr, k, v_atom), 1);
    else wgmma_m64n64_rs<1>(o, p[k], desc_mnmajor(v_addr, k, v_atom), 1);
  }
}

// ================================================================================================
// forward
// ================================================================================================
template <int D>
struct AttFwdCfg {
  static constexpr uint32_t Q_ATOM = ATT_BQ * 128;           // [128 rows][64 cols]
  static constexpr uint32_t KV_ATOM = ATT_BKV * 128;
  static constexpr uint32_t Q_BYTES = ATT_BQ * D * 2;
  static constexpr uint32_t KV_BYTES = ATT_BKV * D * 2;      // one of K or V
  static constexpr uint32_t OFF_K = Q_BYTES;                 // [STAGES]
  static constexpr uint32_t OFF_V = OFF_K + ATT_STAGES * KV_BYTES;
  static constexpr uint32_t OFF_BAR = OFF_V + ATT_STAGES * KV_BYTES;
  static constexpr uint32_t SMEM_BYTES = OFF_BAR + 128 + 1024;
};

template <int D, bool CAUSAL>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, bf16* __restrict__ out, long long ld_out,
                     float* __restrict__ lse_out, int Sq, int Skv, int n_heads, int kv_group, int q_shared,
                     float scale) {
  // kv_group = query heads per key/value head (1 = MHA; 4 = Mistral-7B's 32/8 GQA,
  // omnilmm/model/omnilmm.py -> HF MistralForCausalLM): K/V tiles come from head / kv_group.
  // Sq != Skv / q_shared: cross-attention of the perceiver resampler (omnilmm/model/resampler.py:149-168):
  // 64 learned queries, identical for every image (q_shared: Q is read from sequence 0), over Skv vision tokens.
  using Cfg = AttFwdCfg<D>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;                 // [STAGES]
  uint64_t* kv_empty = bars + 1 + ATT_STAGES;   // [STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int num_q_tiles = (Sq + ATT_BQ - 1) / ATT_BQ;
  const int q_tile = num_q_tiles - 1 - blockIdx.x;  // heavy (late) tiles first
  const int head = blockIdx.y, seq = blockIdx.z;
  const int q_seq = q_shared ? 0 : seq;
  const int kv_head = head / kv_group;
  const int q0 = q_tile * ATT_BQ;
  const int n_kv_all = (Skv + ATT_BKV - 1) / ATT_BKV;
  const int n_kv = CAUSAL ? min(n_kv_all, (q0 + ATT_BQ + ATT_BKV - 1) / ATT_BKV) : n_kv_all;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < ATT_STAGES; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    // ------------------------------ TMA producer ------------------------------
    if (threadIdx.x == 256) {
      tma_prefetch_desc(&tmQ);
      tma_prefetch_desc(&tmK);
      tma_prefetch_desc(&tmV);
      mbar_arrive_expect_tx(q_full, Cfg::Q_BYTES);
#pragma unroll
      for (int a = 0; a < D / 64; ++a)
        tma_load_3d(smem + a * Cfg::Q_ATOM, &tmQ, q_full, head * D + a * 64, q0, q_seq);
      for (int j = 0; j < n_kv; ++j) {
        const int s = j % ATT_STAGES;
        if (j >= ATT_STAGES) mbar_wait(&kv_empty[s], ((j / ATT_STAGES) - 1) & 1);
        mbar_arrive_expect_tx(&kv_full[s], 2 * Cfg::KV_BYTES);
#pragma unroll
        for (int a = 0; a < D / 64; ++a) {
          tma_load_3d(smem + Cfg::OFF_K + s * Cfg::KV_BYTES + a * Cfg::KV_ATOM, &tmK, &kv_full[s],
                      kv_head * D + a * 64, j * ATT_BKV, seq);
          tma_load_3d(smem + Cfg::OFF_V + s * Cfg::KV_BYTES + a * Cfg::KV_ATOM, &tmV, &kv_full[s],
                      kv_head * D + a * 64, j * ATT_BKV, seq);
        }
      }
    }
  } else {
    // ------------------------------ softmax / PV: rows [64*wg, 64*wg + 64) of the query tile ------------------------
    const FragPos fp = frag_pos();
    const int qr[2] = {q0 + wg * 64 + fp.r0, q0 + wg * 64 + fp.r0 + 8};
    const float c = scale * LOG2E;
    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    const uint32_t q_addr = smem_u32(smem) + wg * 64 * 128;
    mbar_wait(q_full, 0);
    for (int j = 0; j < n_kv; ++j) {
      const int s = j % ATT_STAGES;
      mbar_wait(&kv_full[s], (j / ATT_STAGES) & 1);
      const uint32_t k_addr = smem_u32(smem + Cfg::OFF_K + s * Cfg::KV_BYTES);
      const uint32_t v_addr = smem_u32(smem + Cfg::OFF_V + s * Cfg::KV_BYTES);
      float sv[64];
      wgmma_fence();
      mma_qk_128<D>(sv, q_addr, Cfg::Q_ATOM, k_addr, Cfg::KV_ATOM);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(sv);
      const int kv0 = j * ATT_BKV;
      if (kv0 + ATT_BKV > Skv || (CAUSAL && kv0 + ATT_BKV - 1 > q0 + wg * 64)) {
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int kv = kv0 + 8 * i + fp.c0 + (e & 1);
            if (kv >= Skv || (CAUSAL && kv > qr[e >> 1])) sv[4 * i + e] = -INFINITY;
          }
      }
      // online softmax, two rows per thread; a row's 128 columns are spread over the 4 lanes of a quad
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        mx[0] = fmaxf(mx[0], fmaxf(sv[4 * i], sv[4 * i + 1]));
        mx[1] = fmaxf(mx[1], fmaxf(sv[4 * i + 2], sv[4 * i + 3]));
      }
      float alpha[2], neg_m[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        float m_new = fmaxf(m_run[h], mx[h] * c);
        if (m_new == -INFINITY) m_new = 0.f;
        // the running max is only raised once it has grown by more than 8 (P <= 2^8 stays exact in fp32 and in the
        // bf16 exponent range): fewer O rescales, and P's bf16 rounding follows the bf16 reference more closely on long
        // sequences (DPO loss of the long tiny-model fixture: 1.7e-4 from the bf16 reference, 1.3e-3 with an eagerly
        // updated max)
        if (j > 0 && m_new - m_run[h] <= 8.0f) m_new = m_run[h];
        alpha[h] = fast_exp2(m_run[h] - m_new);      // 0 on the first tile (m_run = -inf)
        m_run[h] = m_new;
        l[h] *= alpha[h];
        neg_m[h] = -m_new;
      }
#pragma unroll
      for (int i = 0; i < D / 8; ++i) {
        o[4 * i] *= alpha[0]; o[4 * i + 1] *= alpha[0];
        o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
      }
#pragma unroll
      for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float p = fast_exp2(fmaf(sv[4 * i + e], c, neg_m[e >> 1]));   // exp2(-inf) = 0 for masked
          sv[4 * i + e] = p;
          l[e >> 1] += p;
        }
      uint32_t pa[8][4];
      acc_to_afrag<8>(sv, pa);
      reg_fence(o);
      wgmma_fence();
      mma_pv<D, 8>(o, pa, v_addr, Cfg::KV_ATOM);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(o);
      if (lane == 0) mbar_arrive(&kv_empty[s]);
    }
    // epilogue: O / l -> bf16, LSE
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
      const int q = qr[h];
      if (q >= Sq) continue;
      const float inv = 1.f / l[h];
      bf16* o_row = out + ((long long)seq * Sq + q) * ld_out + head * D + fp.c0;
#pragma unroll
      for (int i = 0; i < D / 8; ++i)
        *reinterpret_cast<uint32_t*>(o_row + 8 * i) = pack_bf16(o[4 * i + 2 * h] * inv, o[4 * i + 2 * h + 1] * inv);
      if (lse_out && fp.c0 == 0) lse_out[((long long)seq * n_heads + head) * Sq + q] = (m_run[h] + log2f(l[h])) * LN2;
    }
  }
}

// ================================================================================================
// backward (D = 128; causal self-attention, or non-causal cross-attention with Sq != Skv)
// ================================================================================================
// delta[seq][head][q] = sum_d dO * O   (fp32). HBM-bound (reads O and dO once): 16-byte loads, one (row, head) item
// per D/8 lanes, two items per lane-group in flight (the 8-byte / one-item-per-warp form ran at 38 % of the copy peak).
__global__ void attention_delta_kernel(const bf16* __restrict__ o, long long ld_o,
                                       const bf16* __restrict__ d_o, long long ld_do,
                                       float* __restrict__ delta, int nseq, int S, int n_heads, int D) {
  const int lpi = D >> 3;                                  // lanes per item (16 for D = 128, 8 for D = 64)
  const int ipw = 32 / lpi;                                // items per warp per pass
  const long long total = (long long)nseq * S * n_heads;
  const int wpb = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int sub = lane / lpi, l = lane % lpi;
  const long long stride = (long long)gridDim.x * wpb * ipw * 2;
  for (long long base = ((long long)blockIdx.x * wpb + (threadIdx.x >> 5)) * ipw * 2; base < total; base += stride) {
    float acc[2];
    long long item[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      item[u] = base + u * ipw + sub;
      acc[u] = 0.f;
      if (item[u] < total) {
        const int head = (int)(item[u] % n_heads);
        const long long row = item[u] / n_heads;
        const uint4 a = *reinterpret_cast<const uint4*>(o + row * ld_o + head * D + l * 8);
        const uint4 b = *reinterpret_cast<const uint4*>(d_o + row * ld_do + head * D + l * 8);
        const float2 a0 = unpack_bf16(a.x), a1 = unpack_bf16(a.y), a2 = unpack_bf16(a.z), a3 = unpack_bf16(a.w);
        const float2 b0 = unpack_bf16(b.x), b1 = unpack_bf16(b.y), b2 = unpack_bf16(b.z), b3 = unpack_bf16(b.w);
        acc[u] = a0.x * b0.x + a0.y * b0.y + a1.x * b1.x + a1.y * b1.y + a2.x * b2.x + a2.y * b2.y + a3.x * b3.x +
                 a3.y * b3.y;
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      for (int off = lpi >> 1; off > 0; off >>= 1) acc[u] += __shfl_xor_sync(0xffffffffu, acc[u], off);
      if (l == 0 && item[u] < total) {
        const int head = (int)(item[u] % n_heads);
        const long long row = item[u] / n_heads;
        const long long seq = row / S;
        const int q = (int)(row % S);
        delta[(seq * n_heads + head) * S + q] = acc[u];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// dK / dV: one CTA per (128-row K/V tile, kv head, sequence); math warpgroup wg owns kv rows [64*wg, 64*wg + 64).
// Two passes over every (query head of the kv group, 64-row chunk of Q / dO), streamed through a two-stage TMA ring:
//   pass 0 (dV): S^T = K Q^T, P^T = exp2(S^T*c - lse), dV += bf16(P^T) dO
//   pass 1 (dK): S^T, dP^T = V dO^T, dS^T = P^T (dP^T - delta) * scale, dK += bf16(dS^T) Q
// with the A operands straight from registers. One 64 x 128 fp32 accumulator is live at a time: dK and dV together
// with S^T and dP^T do not fit the 168 registers a thread of this CTA has; the price is one more K Q^T per chunk.
// q_shared: Q belongs to sequence 0 for every image (the resampler's learned queries).
// ------------------------------------------------------------------------------------------------
constexpr int BWD_D = 128;
constexpr int BWD_C = 64;                                      // rows per streamed chunk
struct AttBwdCfg {
  static constexpr uint32_t TILE_ATOM = 128 * 128;             // resident [128 rows][64 cols] atom
  static constexpr uint32_t TILE_BYTES = 128 * BWD_D * 2;
  static constexpr uint32_t CHUNK_ATOM = BWD_C * 128;          // streamed [64 rows][64 cols] atom
  static constexpr uint32_t CHUNK_BYTES = BWD_C * BWD_D * 2;
  static constexpr uint32_t OFF_T1 = TILE_BYTES;               // second resident tile
  static constexpr uint32_t OFF_C = 2 * TILE_BYTES;            // [STAGES][2 chunks]
  static constexpr uint32_t OFF_BAR = OFF_C + ATT_STAGES * 2 * CHUNK_BYTES;
  static constexpr uint32_t SMEM_BYTES = OFF_BAR + 128 + 1024;
};

template <bool DK>
__device__ __forceinline__ void dkv_pass(uint8_t* smem, uint64_t* c_full, uint64_t* c_empty, int it0, int n_it, int n_c,
                                         int c_first, int kv_head, int kv_group, int seq, int Sq, int n_heads,
                                         int causal, const int (&kvr)[2], uint32_t k_addr, uint32_t v_addr, float c,
                                         float scale, const float* __restrict__ lse, const float* __restrict__ delta,
                                         float (&acc)[BWD_D / 2]) {
  using Cfg = AttBwdCfg;
  const FragPos fp = frag_pos();
#pragma unroll
  for (int i = 0; i < BWD_D / 2; ++i) acc[i] = 0.f;
  for (int it = 0; it < n_it; ++it) {
    const int ii = it0 + it, s = ii % ATT_STAGES;
    const int qc0 = (c_first + it % n_c) * BWD_C;
    const int head = kv_head * kv_group + it / n_c;
    const long long base = ((long long)seq * n_heads + head) * Sq;
    const uint32_t q_addr = smem_u32(smem + Cfg::OFF_C + s * 2 * Cfg::CHUNK_BYTES);
    const uint32_t do_addr = q_addr + Cfg::CHUNK_BYTES;
    mbar_wait(&c_full[s], (ii / ATT_STAGES) & 1);
    float st[32], dpt[32];
    wgmma_fence();
    mma_qk_64<BWD_D>(st, k_addr, Cfg::TILE_ATOM, q_addr, Cfg::CHUNK_ATOM);
    if (DK) mma_qk_64<BWD_D>(dpt, v_addr, Cfg::TILE_ATOM, do_addr, Cfg::CHUNK_ATOM);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(st);
    if (DK) reg_fence(dpt);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int q = qc0 + 8 * i + fp.c0;
      // padded q: lse = +inf => P = 0
      const float l0 = q < Sq ? lse[base + q] * LOG2E : INFINITY, l1 = q + 1 < Sq ? lse[base + q + 1] * LOG2E : INFINITY;
      float d0 = 0.f, d1 = 0.f;
      if (DK) {
        d0 = q < Sq ? delta[base + q] : 0.f;
        d1 = q + 1 < Sq ? delta[base + q + 1] : 0.f;
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qq = q + (e & 1);
        const bool masked = causal && kvr[e >> 1] > qq;
        const float p = masked ? 0.f : fast_exp2(st[4 * i + e] * c - ((e & 1) ? l1 : l0));
        st[4 * i + e] = DK ? p * (dpt[4 * i + e] - ((e & 1) ? d1 : d0)) * scale : p;
      }
    }
    uint32_t fa[4][4];
    acc_to_afrag<4>(st, fa);
    reg_fence(acc);
    wgmma_fence();
    mma_pv<BWD_D, 4>(acc, fa, DK ? q_addr : do_addr, Cfg::CHUNK_ATOM);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(acc);
    if ((threadIdx.x & 31) == 0) mbar_arrive(&c_empty[s]);
  }
}

__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                         const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                         const float* __restrict__ lse, const float* __restrict__ delta, bf16* __restrict__ dk,
                         bf16* __restrict__ dv, long long ld_dkv, int Sq, int Skv, int n_heads, int kv_group,
                         int causal, int q_shared, float scale) {
  using Cfg = AttBwdCfg;
  constexpr int D = BWD_D;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* kv_full = bars;
  uint64_t* c_full = bars + 1;                  // [STAGES]
  uint64_t* c_empty = bars + 1 + ATT_STAGES;    // [STAGES]

  const int warp = threadIdx.x >> 5, wg = warp >> 2;
  const int kv0 = blockIdx.x * 128;
  const int kv_head = blockIdx.y, seq = blockIdx.z;
  const int q_seq = q_shared ? 0 : seq;
  const int n_chunks = (Sq + BWD_C - 1) / BWD_C;
  const int c_first = causal ? kv0 / BWD_C : 0;               // causal: chunks holding a q >= kv0
  const int n_c = n_chunks - c_first;
  const int n_it = n_c > 0 ? n_c * kv_group : 0;               // (query head of the group) x (q chunk), per pass

  if (threadIdx.x == 0) {
    mbar_init(kv_full, 1);
    for (int i = 0; i < ATT_STAGES; ++i) { mbar_init(&c_full[i], 1); mbar_init(&c_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    if (threadIdx.x == 256) {
      tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmDO);
      mbar_arrive_expect_tx(kv_full, 2 * Cfg::TILE_BYTES);
      for (int a = 0; a < 2; ++a) {
        tma_load_3d(smem + a * Cfg::TILE_ATOM, &tmK, kv_full, kv_head * D + a * 64, kv0, seq);
        tma_load_3d(smem + Cfg::OFF_T1 + a * Cfg::TILE_ATOM, &tmV, kv_full, kv_head * D + a * 64, kv0, seq);
      }
      for (int ii = 0; ii < 2 * n_it; ++ii) {
        const int it = ii % n_it, s = ii % ATT_STAGES;
        if (ii >= ATT_STAGES) mbar_wait(&c_empty[s], ((ii / ATT_STAGES) - 1) & 1);
        const int qc0 = (c_first + it % n_c) * BWD_C;
        const int head = kv_head * kv_group + it / n_c;
        uint8_t* dst = smem + Cfg::OFF_C + s * 2 * Cfg::CHUNK_BYTES;
        mbar_arrive_expect_tx(&c_full[s], 2 * Cfg::CHUNK_BYTES);
        for (int a = 0; a < 2; ++a) {
          tma_load_3d(dst + a * Cfg::CHUNK_ATOM, &tmQ, &c_full[s], head * D + a * 64, qc0, q_seq);
          tma_load_3d(dst + Cfg::CHUNK_BYTES + a * Cfg::CHUNK_ATOM, &tmDO, &c_full[s], head * D + a * 64, qc0, seq);
        }
      }
    }
  } else {
    const FragPos fp = frag_pos();
    const int kvr[2] = {kv0 + wg * 64 + fp.r0, kv0 + wg * 64 + fp.r0 + 8};
    const float c = scale * LOG2E;
    const uint32_t k_addr = smem_u32(smem) + wg * 64 * 128;
    const uint32_t v_addr = smem_u32(smem + Cfg::OFF_T1) + wg * 64 * 128;
    mbar_wait(kv_full, 0);
    float acc[D / 2];
#pragma unroll 1
    for (int pass = 0; pass < 2; ++pass) {
      if (pass == 0)
        dkv_pass<false>(smem, c_full, c_empty, 0, n_it, n_c, c_first, kv_head, kv_group, seq, Sq, n_heads, causal, kvr,
                        k_addr, v_addr, c, scale, lse, delta, acc);
      else
        dkv_pass<true>(smem, c_full, c_empty, n_it, n_it, n_c, c_first, kv_head, kv_group, seq, Sq, n_heads, causal, kvr,
                       k_addr, v_addr, c, scale, lse, delta, acc);
      bf16* dst = pass == 0 ? dv : dk;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int kv = kvr[h];
        if (kv >= Skv) continue;
        bf16* row = dst + ((long long)seq * Skv + kv) * ld_dkv + kv_head * D + fp.c0;
#pragma unroll
        for (int i = 0; i < D / 8; ++i)
          *reinterpret_cast<uint32_t*>(row + 8 * i) = pack_bf16(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// dQ: one CTA per (128-row Q tile, head, sequence); math warpgroup wg owns q rows [64*wg, 64*wg + 64). For every
// 64-row chunk of K / V: S = Q K^T, dP = dO V^T, dS = P (dP - delta) * scale, dQ += bf16(dS) K.
// dq_bf16 != nullptr: dQ is written once as bf16 (row stride ld_dq); else it is added into the fp32 dq_f32
// [(q_shared ? 1 : nseq) * Sq][n_heads * 128] with red.global (with q_shared the images' contributions sum up).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                        const float* __restrict__ lse, const float* __restrict__ delta, bf16* __restrict__ dq_bf16,
                        long long ld_dq, float* __restrict__ dq_f32, int Sq, int Skv, int n_heads, int kv_group,
                        int causal, int q_shared, float scale) {
  using Cfg = AttBwdCfg;
  constexpr int D = BWD_D;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* q_full = bars;
  uint64_t* c_full = bars + 1;
  uint64_t* c_empty = bars + 1 + ATT_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int num_q_tiles = (Sq + 127) / 128;
  const int q_tile = num_q_tiles - 1 - blockIdx.x;            // heavy (late) tiles first
  const int q0 = q_tile * 128;
  const int head = blockIdx.y, seq = blockIdx.z;
  const int q_seq = q_shared ? 0 : seq;
  const int kv_head = head / kv_group;
  const int n_all = (Skv + BWD_C - 1) / BWD_C;
  const int n_c = causal ? min(n_all, (q0 + 128 + BWD_C - 1) / BWD_C) : n_all;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < ATT_STAGES; ++i) { mbar_init(&c_full[i], 1); mbar_init(&c_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    if (threadIdx.x == 256) {
      tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmDO);
      mbar_arrive_expect_tx(q_full, 2 * Cfg::TILE_BYTES);
      for (int a = 0; a < 2; ++a) {
        tma_load_3d(smem + a * Cfg::TILE_ATOM, &tmQ, q_full, head * D + a * 64, q0, q_seq);
        tma_load_3d(smem + Cfg::OFF_T1 + a * Cfg::TILE_ATOM, &tmDO, q_full, head * D + a * 64, q0, seq);
      }
      for (int j = 0; j < n_c; ++j) {
        const int s = j % ATT_STAGES;
        if (j >= ATT_STAGES) mbar_wait(&c_empty[s], ((j / ATT_STAGES) - 1) & 1);
        uint8_t* dst = smem + Cfg::OFF_C + s * 2 * Cfg::CHUNK_BYTES;
        mbar_arrive_expect_tx(&c_full[s], 2 * Cfg::CHUNK_BYTES);
        for (int a = 0; a < 2; ++a) {
          tma_load_3d(dst + a * Cfg::CHUNK_ATOM, &tmK, &c_full[s], kv_head * D + a * 64, j * BWD_C, seq);
          tma_load_3d(dst + Cfg::CHUNK_BYTES + a * Cfg::CHUNK_ATOM, &tmV, &c_full[s], kv_head * D + a * 64, j * BWD_C,
                      seq);
        }
      }
    }
  } else {
    const FragPos fp = frag_pos();
    const int qr[2] = {q0 + wg * 64 + fp.r0, q0 + wg * 64 + fp.r0 + 8};
    const float c = scale * LOG2E;
    const long long base = ((long long)seq * n_heads + head) * Sq;
    float lse2[2], dl[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      lse2[h] = qr[h] < Sq ? lse[base + qr[h]] * LOG2E : INFINITY;   // padded q: P = 0
      dl[h] = qr[h] < Sq ? delta[base + qr[h]] : 0.f;
    }
    float dqacc[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) dqacc[i] = 0.f;
    const uint32_t q_addr = smem_u32(smem) + wg * 64 * 128;
    const uint32_t do_addr = smem_u32(smem + Cfg::OFF_T1) + wg * 64 * 128;
    mbar_wait(q_full, 0);
    for (int j = 0; j < n_c; ++j) {
      const int s = j % ATT_STAGES;
      const uint32_t k_addr = smem_u32(smem + Cfg::OFF_C + s * 2 * Cfg::CHUNK_BYTES);
      const uint32_t v_addr = k_addr + Cfg::CHUNK_BYTES;
      mbar_wait(&c_full[s], (j / ATT_STAGES) & 1);
      float sv[32], dp[32];
      wgmma_fence();
      mma_qk_64<D>(sv, q_addr, Cfg::TILE_ATOM, k_addr, Cfg::CHUNK_ATOM);
      mma_qk_64<D>(dp, do_addr, Cfg::TILE_ATOM, v_addr, Cfg::CHUNK_ATOM);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(sv);
      reg_fence(dp);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int kv = j * BWD_C + 8 * i + fp.c0 + (e & 1);
          const int h = e >> 1;
          const bool masked = kv >= Skv || (causal && kv > qr[h]);
          const float p = masked ? 0.f : fast_exp2(sv[4 * i + e] * c - lse2[h]);
          dp[4 * i + e] = p * (dp[4 * i + e] - dl[h]) * scale;
        }
      uint32_t da[4][4];
      acc_to_afrag<4>(dp, da);
      reg_fence(dqacc);
      wgmma_fence();
      mma_pv<D, 4>(dqacc, da, k_addr, Cfg::CHUNK_ATOM);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(dqacc);
      if (lane == 0) mbar_arrive(&c_empty[s]);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = qr[h];
      if (q >= Sq) continue;
      if (dq_bf16) {
        bf16* row = dq_bf16 + ((long long)seq * Sq + q) * ld_dq + head * D + fp.c0;
#pragma unroll
        for (int i = 0; i < D / 8; ++i)
          *reinterpret_cast<uint32_t*>(row + 8 * i) = pack_bf16(dqacc[4 * i + 2 * h], dqacc[4 * i + 2 * h + 1]);
      } else {
        float* row = dq_f32 + ((long long)q_seq * Sq + q) * ((long long)n_heads * D) + head * D + fp.c0;
#pragma unroll
        for (int i = 0; i < D / 8; ++i)
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(row + 8 * i), "f"(dqacc[4 * i + 2 * h]),
                       "f"(dqacc[4 * i + 2 * h + 1])
                       : "memory");
      }
    }
  }
}

static int make_qkv_tmap_rows(CUtensorMap* tm, const void* ptr, long long ld, int nseq, int S, int cols, int box_rows) {
  uint64_t dims[3] = {(uint64_t)cols, (uint64_t)S, (uint64_t)nseq};
  uint64_t str[2] = {(uint64_t)ld * 2, (uint64_t)S * ld * 2};
  uint32_t box[3] = {64, (uint32_t)box_rows, 1};
  return make_tmap_bf16(tm, ptr, 3, dims, str, box);
}

template <int D, bool CAUSAL>
static int launch_att_fwd(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, bf16* out,
                          long long ld_out, float* lse, int nseq, int Sq, int Skv, int n_heads, int kv_group,
                          int q_shared, float scale, cudaStream_t st) {
  using Cfg = AttFwdCfg<D>;
  auto kern = attention_fwd_kernel<D, CAUSAL>;
  B200_CHECK_CUDA(configure_smem_once((const void*)kern, (int)Cfg::SMEM_BYTES));
  dim3 grid((Sq + ATT_BQ - 1) / ATT_BQ, n_heads, nseq);
  kern<<<grid, ATT_THREADS, Cfg::SMEM_BYTES, st>>>(tq, tk, tv, out, ld_out, lse, Sq, Skv, n_heads, kv_group, q_shared,
                                                   scale);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b200

using namespace b200;

static int attention_fwd_impl(const void* q, long long ld_q, const void* k, const void* v, long long ld_kv, void* out,
                              long long ld_out, float* lse, int nseq, int Sq, int Skv, int n_heads, int n_kv_heads,
                              int head_dim, int causal, int q_shared, float scale, void* stream) {
  B200_REQUIRE(head_dim == 128 || head_dim == 64, "attention_fwd: head_dim %d not in {64,128}", head_dim);
  B200_REQUIRE(ld_q % 8 == 0 && ld_kv % 8 == 0 && ld_out % 8 == 0, "attention_fwd: ld must be a multiple of 8");
  B200_REQUIRE(n_kv_heads > 0 && n_heads % n_kv_heads == 0, "attention_fwd: n_heads %d not a multiple of n_kv_heads %d",
               n_heads, n_kv_heads);
  B200_REQUIRE(!causal || Sq == Skv, "attention_fwd: causal needs Sq == Skv (%d vs %d)", Sq, Skv);
  B200_REQUIRE(nseq > 0 && Sq > 0 && Skv > 0, "attention_fwd: empty problem");
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = make_qkv_tmap_rows(&tq, q, ld_q, q_shared ? 1 : nseq, Sq, n_heads * head_dim, ATT_BQ))) return rc;
  if ((rc = make_qkv_tmap_rows(&tk, k, ld_kv, nseq, Skv, n_kv_heads * head_dim, ATT_BKV))) return rc;
  if ((rc = make_qkv_tmap_rows(&tv, v, ld_kv, nseq, Skv, n_kv_heads * head_dim, ATT_BKV))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int g = n_heads / n_kv_heads;
  bf16* o = (bf16*)out;
  if (head_dim == 128)
    return causal ? launch_att_fwd<128, true>(tq, tk, tv, o, ld_out, lse, nseq, Sq, Skv, n_heads, g, q_shared, scale, st)
                  : launch_att_fwd<128, false>(tq, tk, tv, o, ld_out, lse, nseq, Sq, Skv, n_heads, g, q_shared, scale, st);
  return causal ? launch_att_fwd<64, true>(tq, tk, tv, o, ld_out, lse, nseq, Sq, Skv, n_heads, g, q_shared, scale, st)
                : launch_att_fwd<64, false>(tq, tk, tv, o, ld_out, lse, nseq, Sq, Skv, n_heads, g, q_shared, scale, st);
}

extern "C" int rlaifv_attention_fwd(const void* q, const void* k, const void* v, long long ld_qkv, void* out,
                                    long long ld_out, float* lse, int nseq, int S, int n_heads, int head_dim,
                                    int causal, float scale, void* stream) {
  return attention_fwd_impl(q, ld_qkv, k, v, ld_qkv, out, ld_out, lse, nseq, S, S, n_heads, n_heads, head_dim, causal, 0,
                            scale, stream);
}
// grouped-query attention: k/v hold n_kv_heads heads, query head h reads kv head h / (n_heads / n_kv_heads)
extern "C" int rlaifv_attention_fwd_gqa(const void* q, const void* k, const void* v, long long ld_qkv, void* out,
                                        long long ld_out, float* lse, int nseq, int S, int n_heads, int n_kv_heads,
                                        int head_dim, int causal, float scale, void* stream) {
  return attention_fwd_impl(q, ld_qkv, k, v, ld_qkv, out, ld_out, lse, nseq, S, S, n_heads, n_kv_heads, head_dim,
                            causal, 0, scale, stream);
}
// Cross-attention (non-causal): q [(q_shared ? 1 : nseq) * Sq rows][ld_q], k/v [nseq * Skv rows][ld_kv], out
// [nseq * Sq rows][ld_out], lse fp32 [nseq][n_heads][Sq]. Replaces nn.MultiheadAttention's core inside
// Resampler.forward (omnilmm/model/resampler.py:158-163): q_shared = the learned queries are batch-independent.
extern "C" int rlaifv_cross_attention_fwd(const void* q, long long ld_q, const void* k, const void* v, long long ld_kv,
                                          void* out, long long ld_out, float* lse, int nseq, int Sq, int Skv,
                                          int n_heads, int head_dim, int q_shared, float scale, void* stream) {
  return attention_fwd_impl(q, ld_q, k, v, ld_kv, out, ld_out, lse, nseq, Sq, Skv, n_heads, n_heads, head_dim, 0,
                            q_shared, scale, stream);
}

// delta, then the dK/dV kernel, then the dQ kernel. dq != nullptr: dQ written as bf16 [nseq*Sq rows][ld_dq];
// else added into dq_f32 (fp32 [(q_shared ? 1 : nseq) * Sq][n_heads*128], zeroed by the caller).
static int attention_bwd_impl(const void* q, long long ld_q, const void* k, const void* v, long long ld_kv,
                              const void* out, long long ld_out, const void* d_out, long long ld_dout, const float* lse,
                              void* dq, long long ld_dq, float* dq_f32, void* dk, void* dv, long long ld_dkv,
                              float* delta_ws, int nseq, int Sq, int Skv, int n_heads, int n_kv_heads, int head_dim,
                              int causal, int q_shared, float scale, void* stream) {
  B200_REQUIRE(head_dim == 128, "attention_bwd: head_dim must be 128 (got %d)", head_dim);
  B200_REQUIRE(n_kv_heads > 0 && n_heads % n_kv_heads == 0, "attention_bwd: bad head counts %d / %d", n_heads,
               n_kv_heads);
  B200_REQUIRE(!causal || Sq == Skv, "attention_bwd: causal needs Sq == Skv (%d vs %d)", Sq, Skv);
  B200_REQUIRE(nseq > 0 && Sq > 0 && Skv > 0, "attention_bwd: empty problem");
  B200_REQUIRE(ld_q % 8 == 0 && ld_kv % 8 == 0 && ld_dout % 8 == 0, "attention_bwd: ld must be a multiple of 8");
  B200_REQUIRE(dq ? (ld_dq % 2 == 0 && ((uintptr_t)dq & 3) == 0) : dq_f32 != nullptr, "attention_bwd: dq alignment");
  B200_REQUIRE(ld_dkv % 2 == 0, "attention_bwd: ld_dkv must be even");
  // attention_delta_kernel reads O and dO rows with 16-byte loads
  B200_REQUIRE(ld_out % 8 == 0 && ((uintptr_t)out & 15) == 0 && ((uintptr_t)d_out & 15) == 0,
               "attention_bwd: out / d_out must be 16-byte aligned with ld_out a multiple of 8 (ld_out %lld)", ld_out);
  const int g = n_heads / n_kv_heads;
  const int q_nseq = q_shared ? 1 : nseq;
  int rc;
  // every tensor map is built (and so validated) before the first launch
  // dK / dV: K, V resident (128-row boxes), Q / dO streamed in 64-row chunks
  CUtensorMap tq, tk, tv, tdo;
  if ((rc = make_qkv_tmap_rows(&tq, q, ld_q, q_nseq, Sq, n_heads * head_dim, BWD_C))) return rc;
  if ((rc = make_qkv_tmap_rows(&tdo, d_out, ld_dout, nseq, Sq, n_heads * head_dim, BWD_C))) return rc;
  if ((rc = make_qkv_tmap_rows(&tk, k, ld_kv, nseq, Skv, n_kv_heads * head_dim, 128))) return rc;
  if ((rc = make_qkv_tmap_rows(&tv, v, ld_kv, nseq, Skv, n_kv_heads * head_dim, 128))) return rc;
  // dQ: Q, dO resident, K / V streamed in 64-row chunks
  CUtensorMap tq2, tk2, tv2, tdo2;
  if ((rc = make_qkv_tmap_rows(&tq2, q, ld_q, q_nseq, Sq, n_heads * head_dim, 128))) return rc;
  if ((rc = make_qkv_tmap_rows(&tdo2, d_out, ld_dout, nseq, Sq, n_heads * head_dim, 128))) return rc;
  if ((rc = make_qkv_tmap_rows(&tk2, k, ld_kv, nseq, Skv, n_kv_heads * head_dim, BWD_C))) return rc;
  if ((rc = make_qkv_tmap_rows(&tv2, v, ld_kv, nseq, Skv, n_kv_heads * head_dim, BWD_C))) return rc;
  B200_CHECK_CUDA(configure_smem_once((const void*)attention_bwd_dkv_kernel, (int)AttBwdCfg::SMEM_BYTES));
  B200_CHECK_CUDA(configure_smem_once((const void*)attention_bwd_dq_kernel, (int)AttBwdCfg::SMEM_BYTES));
  cudaStream_t st = (cudaStream_t)stream;
  {
    const long long total = (long long)nseq * Sq * n_heads;
    long long blocks = (total + 7) / 8;
    if (blocks > (long long)num_sms() * 16) blocks = (long long)num_sms() * 16;
    attention_delta_kernel<<<(int)blocks, 256, 0, st>>>((const bf16*)out, ld_out, (const bf16*)d_out, ld_dout,
                                                        delta_ws, nseq, Sq, n_heads, head_dim);
    B200_CHECK_CUDA(cudaGetLastError());
  }
  {
    dim3 grid((Skv + 127) / 128, n_kv_heads, nseq);
    attention_bwd_dkv_kernel<<<grid, ATT_THREADS, AttBwdCfg::SMEM_BYTES, st>>>(
        tq, tk, tv, tdo, lse, delta_ws, (bf16*)dk, (bf16*)dv, ld_dkv, Sq, Skv, n_heads, g, causal, q_shared, scale);
    B200_CHECK_CUDA(cudaGetLastError());
  }
  {
    dim3 grid((Sq + 127) / 128, n_heads, nseq);
    attention_bwd_dq_kernel<<<grid, ATT_THREADS, AttBwdCfg::SMEM_BYTES, st>>>(
        tq2, tk2, tv2, tdo2, lse, delta_ws, (bf16*)dq, ld_dq, dq_f32, Sq, Skv, n_heads, g, causal, q_shared, scale);
    B200_CHECK_CUDA(cudaGetLastError());
  }
  return 0;
}

// Split backward for self-attention (causal or not, Sq == Skv or not; per-sequence queries): dq is written as bf16
// [nseq*Sq rows][ld_dq] (it may be the q column block of a fused dqkv buffer), dk/dv as before; no zero-fill needed.
extern "C" int rlaifv_attention_bwd_split(const void* q, long long ld_q, const void* k, const void* v, long long ld_kv,
                                          const void* out, long long ld_out, const void* d_out, long long ld_dout,
                                          const float* lse, void* dq, long long ld_dq, void* dk, void* dv,
                                          long long ld_dkv, float* delta_ws, int nseq, int Sq, int Skv, int n_heads,
                                          int n_kv_heads, int head_dim, int causal, float scale, void* stream) {
  B200_REQUIRE(dq != nullptr, "attention_bwd_split: dq missing");
  return attention_bwd_impl(q, ld_q, k, v, ld_kv, out, ld_out, d_out, ld_dout, lse, dq, ld_dq, nullptr, dk, dv, ld_dkv,
                            delta_ws, nseq, Sq, Skv, n_heads, n_kv_heads, head_dim, causal, 0, scale, stream);
}

// dq_f32 [nseq*S][n_heads*128] must be zeroed by the caller; delta_ws fp32 [nseq*n_heads*S].
extern "C" int rlaifv_attention_bwd(const void* q, const void* k, const void* v, long long ld_qkv,
                                    const void* out, long long ld_out, const void* d_out, long long ld_dout,
                                    const float* lse, float* dq_f32, void* dk, void* dv, long long ld_dkv,
                                    float* delta_ws, int nseq, int S, int n_heads, int head_dim, float scale,
                                    void* stream) {
  return attention_bwd_impl(q, ld_qkv, k, v, ld_qkv, out, ld_out, d_out, ld_dout, lse, nullptr, 0, dq_f32, dk, dv, ld_dkv, delta_ws,
                            nseq, S, S, n_heads, n_heads, head_dim, 1, 0, scale, stream);
}
// GQA: dk/dv hold n_kv_heads heads (sum over the query heads of each group is formed in registers).
extern "C" int rlaifv_attention_bwd_gqa(const void* q, const void* k, const void* v, long long ld_qkv,
                                        const void* out, long long ld_out, const void* d_out, long long ld_dout,
                                        const float* lse, float* dq_f32, void* dk, void* dv, long long ld_dkv,
                                        float* delta_ws, int nseq, int S, int n_heads, int n_kv_heads, int head_dim,
                                        float scale, void* stream) {
  return attention_bwd_impl(q, ld_qkv, k, v, ld_qkv, out, ld_out, d_out, ld_dout, lse, nullptr, 0, dq_f32, dk, dv, ld_dkv, delta_ws,
                            nseq, S, S, n_heads, n_kv_heads, head_dim, 1, 0, scale, stream);
}
// Cross-attention backward (non-causal, head_dim 128). dq_f32 fp32 [(q_shared ? 1 : nseq) * Sq][n_heads*128],
// zeroed by the caller (with q_shared it receives the sum over the batch); dk/dv bf16 [nseq * Skv rows][ld_dkv];
// delta_ws fp32 [nseq * n_heads * Sq].
extern "C" int rlaifv_cross_attention_bwd(const void* q, long long ld_q, const void* k, const void* v, long long ld_kv,
                                          const void* out, long long ld_out, const void* d_out, long long ld_dout,
                                          const float* lse, float* dq_f32, void* dk, void* dv, long long ld_dkv,
                                          float* delta_ws, int nseq, int Sq, int Skv, int n_heads, int head_dim,
                                          int q_shared, float scale, void* stream) {
  return attention_bwd_impl(q, ld_q, k, v, ld_kv, out, ld_out, d_out, ld_dout, lse, nullptr, 0, dq_f32, dk, dv, ld_dkv, delta_ws,
                            nseq, Sq, Skv, n_heads, n_heads, head_dim, 0, q_shared, scale, stream);
}

// ================================================================================================
// variable-length causal self-attention over packed rows (head_dim 128, MHA or GQA)
// ================================================================================================
// Sequence s occupies rows [cu[s], cu[s+1]) of q/k/v/out [n_rows][ld]; its row cu[s] + t is position t. LSE and the
// delta workspace are fp32 with sequence s's [n_heads][len_s] block at offset n_heads * cu[s]. Tiles are cut relative
// to cu[s], so every valid row sees the key partition, online-softmax order and chunk order of the fixed-length
// kernels above on the same sequence padded to any length: the results at rows < len_s are the same bits. A tile's
// rows past len_s are the next sequence's (or TMA zero-fill past the last row): causality hides them from valid
// queries in the forward and the dQ kernel; the dK/dV kernel, where they come after the key, masks them explicitly.
//
// Borrowed prefixes (PREFIX = true, the attention_varlen_prefix_* entry points): sequence s's own rows hold positions
// p0 = pos0[s] .. p0 + len_s - 1, and with p0 > 0 its positions below p0 are rows of its lender partner[s] (two
// sequences with identical inputs below p0 hold identical rows there, so one copy serves both). p0 is a multiple of
// 128: every own query row sees the key partition and chunk order of the fixed-length kernels on the sequence padded
// to any length, so O, LSE, dQ and the dK/dV of own rows are those kernels' bits. A lender's key tile below its
// borrower's p0 streams the lender's Q / dO chunks, then the borrower's, into one accumulator: its dK/dV is the sum
// of both copies' gradients. LSE and delta keep the [n_heads][len_s] blocks of own rows.
namespace b200 {

constexpr int PREFIX_MAX_SEQ = 64;
template <bool PREFIX>
struct PrefixMap {
  int pos0[PREFIX_MAX_SEQ];
  int partner[PREFIX_MAX_SEQ];
};
template <>
struct PrefixMap<false> {};

template <bool PREFIX>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_varlen_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                            const __grid_constant__ CUtensorMap tmV, bf16* __restrict__ out, long long ld_out,
                            float* __restrict__ lse_out, const int* __restrict__ cu, int n_heads, int kv_group,
                            float scale, const __grid_constant__ PrefixMap<PREFIX> pm) {
  constexpr int D = 128;
  using Cfg = AttFwdCfg<D>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;                 // [STAGES]
  uint64_t* kv_empty = bars + 1 + ATT_STAGES;   // [STAGES]

  const int seq = blockIdx.z;
  const int row0 = cu[seq], len = cu[seq + 1] - row0;
  const int num_q_tiles = (len + ATT_BQ - 1) / ATT_BQ;
  if ((int)blockIdx.x >= num_q_tiles) return;             // the grid is sized for the longest sequence
  int p0 = 0, lrow0 = row0;                               // first own position; the lender's row of position 0
  if constexpr (PREFIX) {
    p0 = pm.pos0[seq];
    if (p0 > 0) lrow0 = cu[pm.partner[seq]];
  }
  const int end = p0 + len;                               // one past the last position
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int q_tile = num_q_tiles - 1 - blockIdx.x;        // heavy (late) tiles first
  const int head = blockIdx.y;
  const int kv_head = head / kv_group;
  const int q0 = p0 + q_tile * ATT_BQ;
  const int n_kv = min(num_q_tiles + p0 / ATT_BKV, (q0 + ATT_BQ + ATT_BKV - 1) / ATT_BKV);

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < ATT_STAGES; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    if (threadIdx.x == 256) {
      tma_prefetch_desc(&tmQ);
      tma_prefetch_desc(&tmK);
      tma_prefetch_desc(&tmV);
      mbar_arrive_expect_tx(q_full, Cfg::Q_BYTES);
#pragma unroll
      for (int a = 0; a < D / 64; ++a)
        tma_load_2d(smem + a * Cfg::Q_ATOM, &tmQ, q_full, head * D + a * 64, row0 - p0 + q0);
      for (int j = 0; j < n_kv; ++j) {
        const int s = j % ATT_STAGES;
        if (j >= ATT_STAGES) mbar_wait(&kv_empty[s], ((j / ATT_STAGES) - 1) & 1);
        mbar_arrive_expect_tx(&kv_full[s], 2 * Cfg::KV_BYTES);
        const int kv_row = (PREFIX && j * ATT_BKV < p0 ? lrow0 : row0 - p0) + j * ATT_BKV;
#pragma unroll
        for (int a = 0; a < D / 64; ++a) {
          tma_load_2d(smem + Cfg::OFF_K + s * Cfg::KV_BYTES + a * Cfg::KV_ATOM, &tmK, &kv_full[s],
                      kv_head * D + a * 64, kv_row);
          tma_load_2d(smem + Cfg::OFF_V + s * Cfg::KV_BYTES + a * Cfg::KV_ATOM, &tmV, &kv_full[s],
                      kv_head * D + a * 64, kv_row);
        }
      }
    }
  } else {
    const FragPos fp = frag_pos();
    const int qr[2] = {q0 + wg * 64 + fp.r0, q0 + wg * 64 + fp.r0 + 8};
    const float c = scale * LOG2E;
    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    const uint32_t q_addr = smem_u32(smem) + wg * 64 * 128;
    mbar_wait(q_full, 0);
    for (int j = 0; j < n_kv; ++j) {
      const int s = j % ATT_STAGES;
      mbar_wait(&kv_full[s], (j / ATT_STAGES) & 1);
      const uint32_t k_addr = smem_u32(smem + Cfg::OFF_K + s * Cfg::KV_BYTES);
      const uint32_t v_addr = smem_u32(smem + Cfg::OFF_V + s * Cfg::KV_BYTES);
      float sv[64];
      wgmma_fence();
      mma_qk_128<D>(sv, q_addr, Cfg::Q_ATOM, k_addr, Cfg::KV_ATOM);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(sv);
      const int kv0 = j * ATT_BKV;
      if (kv0 + ATT_BKV > end || kv0 + ATT_BKV - 1 > q0 + wg * 64) {
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int kv = kv0 + 8 * i + fp.c0 + (e & 1);
            if (kv >= end || kv > qr[e >> 1]) sv[4 * i + e] = -INFINITY;
          }
      }
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        mx[0] = fmaxf(mx[0], fmaxf(sv[4 * i], sv[4 * i + 1]));
        mx[1] = fmaxf(mx[1], fmaxf(sv[4 * i + 2], sv[4 * i + 3]));
      }
      float alpha[2], neg_m[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        float m_new = fmaxf(m_run[h], mx[h] * c);
        if (m_new == -INFINITY) m_new = 0.f;
        if (j > 0 && m_new - m_run[h] <= 8.0f) m_new = m_run[h];   // lazy max, as attention_fwd_kernel
        alpha[h] = fast_exp2(m_run[h] - m_new);
        m_run[h] = m_new;
        l[h] *= alpha[h];
        neg_m[h] = -m_new;
      }
#pragma unroll
      for (int i = 0; i < D / 8; ++i) {
        o[4 * i] *= alpha[0]; o[4 * i + 1] *= alpha[0];
        o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
      }
#pragma unroll
      for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float p = fast_exp2(fmaf(sv[4 * i + e], c, neg_m[e >> 1]));
          sv[4 * i + e] = p;
          l[e >> 1] += p;
        }
      uint32_t pa[8][4];
      acc_to_afrag<8>(sv, pa);
      reg_fence(o);
      wgmma_fence();
      mma_pv<D, 8>(o, pa, v_addr, Cfg::KV_ATOM);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(o);
      if (lane == 0) mbar_arrive(&kv_empty[s]);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
      const int q = qr[h];
      if (q >= end) continue;
      const float inv = 1.f / l[h];
      bf16* o_row = out + ((long long)row0 - p0 + q) * ld_out + head * D + fp.c0;
#pragma unroll
      for (int i = 0; i < D / 8; ++i)
        *reinterpret_cast<uint32_t*>(o_row + 8 * i) = pack_bf16(o[4 * i + 2 * h] * inv, o[4 * i + 2 * h + 1] * inv);
      if (fp.c0 == 0)
        lse_out[(long long)n_heads * row0 + (long long)head * len + q - p0] = (m_run[h] + log2f(l[h])) * LN2;
    }
  }
}

// delta of attention_delta_kernel over packed rows, stored in the packed [n_heads][len_s] blocks
__global__ void attention_varlen_delta_kernel(const bf16* __restrict__ o, long long ld_o, const bf16* __restrict__ d_o,
                                              long long ld_do, float* __restrict__ delta, const int* __restrict__ cu,
                                              int nseq, long long n_rows, int n_heads, int D) {
  const int lpi = D >> 3;
  const int ipw = 32 / lpi;
  const long long total = n_rows * n_heads;
  const int wpb = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int sub = lane / lpi, l = lane % lpi;
  const long long stride = (long long)gridDim.x * wpb * ipw * 2;
  for (long long base = ((long long)blockIdx.x * wpb + (threadIdx.x >> 5)) * ipw * 2; base < total; base += stride) {
    float acc[2];
    long long item[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      item[u] = base + u * ipw + sub;
      acc[u] = 0.f;
      if (item[u] < total) {
        const int head = (int)(item[u] % n_heads);
        const long long row = item[u] / n_heads;
        const uint4 a = *reinterpret_cast<const uint4*>(o + row * ld_o + head * D + l * 8);
        const uint4 b = *reinterpret_cast<const uint4*>(d_o + row * ld_do + head * D + l * 8);
        const float2 a0 = unpack_bf16(a.x), a1 = unpack_bf16(a.y), a2 = unpack_bf16(a.z), a3 = unpack_bf16(a.w);
        const float2 b0 = unpack_bf16(b.x), b1 = unpack_bf16(b.y), b2 = unpack_bf16(b.z), b3 = unpack_bf16(b.w);
        acc[u] = a0.x * b0.x + a0.y * b0.y + a1.x * b1.x + a1.y * b1.y + a2.x * b2.x + a2.y * b2.y + a3.x * b3.x +
                 a3.y * b3.y;
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      for (int off = lpi >> 1; off > 0; off >>= 1) acc[u] += __shfl_xor_sync(0xffffffffu, acc[u], off);
      if (l == 0 && item[u] < total) {
        const int head = (int)(item[u] % n_heads);
        const int row = (int)(item[u] / n_heads);
        int lo = 0, hi = nseq - 1;                             // sequence s with cu[s] <= row < cu[s + 1]
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (cu[mid] <= row) lo = mid; else hi = mid - 1;
        }
        const int row0 = cu[lo], len = cu[lo + 1] - row0;
        delta[(long long)n_heads * row0 + (long long)head * len + (row - row0)] = acc[u];
      }
    }
  }
}

// The query chunks a dK/dV tile streams, per query head: n_own chunks of its own sequence from position c_first * 64
// (LSE / delta block at blk0, len rows from position p0), then, for a lender's tile below its borrower's first own
// position, the borrower's n_c - n_own chunks from position b_p0 (block b_blk, b_len rows).
struct DkvChunks {
  int n_own, p0, b_p0, b_len;
  long long b_blk;
};

// one pass of attention_bwd_dkv_kernel over packed rows; query positions past the sequence's end are masked
// (P = dS = 0)
template <bool DK, bool PREFIX>
__device__ __forceinline__ void varlen_dkv_pass(uint8_t* smem, uint64_t* c_full, uint64_t* c_empty, int it0, int n_it,
                                                int n_c, int c_first, int kv_head, int kv_group, long long blk0, int len,
                                                const DkvChunks& ch, const int (&kvr)[2], uint32_t k_addr,
                                                uint32_t v_addr, float c, float scale, const float* __restrict__ lse,
                                                const float* __restrict__ delta, float (&acc)[BWD_D / 2]) {
  using Cfg = AttBwdCfg;
  const FragPos fp = frag_pos();
#pragma unroll
  for (int i = 0; i < BWD_D / 2; ++i) acc[i] = 0.f;
  for (int it = 0; it < n_it; ++it) {
    const int ii = it0 + it, s = ii % ATT_STAGES;
    const int k = it % n_c;
    const int head = kv_head * kv_group + it / n_c;
    int qc0 = (c_first + k) * BWD_C;
    long long base = blk0 + (long long)head * len;        // LSE / delta of position q at base + q - p0
    int p0 = 0, len_q = len;
    if constexpr (PREFIX) {
      p0 = ch.p0;
      if (k >= ch.n_own) {
        qc0 = ch.b_p0 + (k - ch.n_own) * BWD_C;
        base = ch.b_blk + (long long)head * ch.b_len;
        p0 = ch.b_p0;
        len_q = ch.b_len;
      }
    }
    base -= p0;
    const int end = p0 + len_q;
    const uint32_t q_addr = smem_u32(smem + Cfg::OFF_C + s * 2 * Cfg::CHUNK_BYTES);
    const uint32_t do_addr = q_addr + Cfg::CHUNK_BYTES;
    mbar_wait(&c_full[s], (ii / ATT_STAGES) & 1);
    float st[32], dpt[32];
    wgmma_fence();
    mma_qk_64<BWD_D>(st, k_addr, Cfg::TILE_ATOM, q_addr, Cfg::CHUNK_ATOM);
    if (DK) mma_qk_64<BWD_D>(dpt, v_addr, Cfg::TILE_ATOM, do_addr, Cfg::CHUNK_ATOM);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(st);
    if (DK) reg_fence(dpt);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int q = qc0 + 8 * i + fp.c0;
      const float l0 = q < end ? lse[base + q] * LOG2E : INFINITY, l1 = q + 1 < end ? lse[base + q + 1] * LOG2E : INFINITY;
      float d0 = 0.f, d1 = 0.f;
      if (DK) {
        d0 = q < end ? delta[base + q] : 0.f;
        d1 = q + 1 < end ? delta[base + q + 1] : 0.f;
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qq = q + (e & 1);
        // rows past the end belong to the next sequence (causality does not hide them: they come after the key)
        const bool masked = kvr[e >> 1] > qq || qq >= end;
        const float p = masked ? 0.f : fast_exp2(st[4 * i + e] * c - ((e & 1) ? l1 : l0));
        st[4 * i + e] = masked ? 0.f : DK ? p * (dpt[4 * i + e] - ((e & 1) ? d1 : d0)) * scale : p;
      }
    }
    uint32_t fa[4][4];
    acc_to_afrag<4>(st, fa);
    reg_fence(acc);
    wgmma_fence();
    mma_pv<BWD_D, 4>(acc, fa, DK ? q_addr : do_addr, Cfg::CHUNK_ATOM);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(acc);
    if ((threadIdx.x & 31) == 0) mbar_arrive(&c_empty[s]);
  }
}

template <bool PREFIX>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_varlen_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                                const float* __restrict__ lse, const float* __restrict__ delta, bf16* __restrict__ dk,
                                bf16* __restrict__ dv, long long ld_dkv, const int* __restrict__ cu, int n_heads,
                                int kv_group, float scale, const __grid_constant__ PrefixMap<PREFIX> pm) {
  using Cfg = AttBwdCfg;
  constexpr int D = BWD_D;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* kv_full = bars;
  uint64_t* c_full = bars + 1;                  // [STAGES]
  uint64_t* c_empty = bars + 1 + ATT_STAGES;    // [STAGES]

  const int seq = blockIdx.z;
  const int row0 = cu[seq], len = cu[seq + 1] - row0;
  if ((int)blockIdx.x * 128 >= len) return;
  DkvChunks ch{0, 0, 0, 0, 0};
  int b_row0 = 0;                                             // the borrower's first own row
  if constexpr (PREFIX) ch.p0 = pm.pos0[seq];
  const int kv0 = ch.p0 + blockIdx.x * 128;
  const int warp = threadIdx.x >> 5, wg = warp >> 2;
  const int kv_head = blockIdx.y;
  const int c_first = kv0 / BWD_C;                            // chunks holding a q >= kv0
  ch.n_own = (ch.p0 + len + BWD_C - 1) / BWD_C - c_first;     // >= 1
  int n_c = ch.n_own;
  if constexpr (PREFIX) {
    const int b = pm.partner[seq];
    if (ch.p0 == 0 && b >= 0 && kv0 < pm.pos0[b]) {           // a lender's key tile below its borrower's own rows
      b_row0 = cu[b];
      ch.b_p0 = pm.pos0[b];
      ch.b_len = cu[b + 1] - b_row0;
      ch.b_blk = (long long)n_heads * b_row0;
      n_c += (ch.b_len + BWD_C - 1) / BWD_C;
    }
  }
  const int n_it = n_c * kv_group;
  const long long blk0 = (long long)n_heads * row0;

  if (threadIdx.x == 0) {
    mbar_init(kv_full, 1);
    for (int i = 0; i < ATT_STAGES; ++i) { mbar_init(&c_full[i], 1); mbar_init(&c_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    if (threadIdx.x == 256) {
      tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmDO);
      mbar_arrive_expect_tx(kv_full, 2 * Cfg::TILE_BYTES);
      for (int a = 0; a < 2; ++a) {
        tma_load_2d(smem + a * Cfg::TILE_ATOM, &tmK, kv_full, kv_head * D + a * 64, row0 - ch.p0 + kv0);
        tma_load_2d(smem + Cfg::OFF_T1 + a * Cfg::TILE_ATOM, &tmV, kv_full, kv_head * D + a * 64, row0 - ch.p0 + kv0);
      }
      for (int ii = 0; ii < 2 * n_it; ++ii) {
        const int it = ii % n_it, s = ii % ATT_STAGES;
        if (ii >= ATT_STAGES) mbar_wait(&c_empty[s], ((ii / ATT_STAGES) - 1) & 1);
        const int qc0 = (c_first + it % n_c) * BWD_C;
        const int head = kv_head * kv_group + it / n_c;
        int q_row = row0 + qc0;
        if constexpr (PREFIX) {
          const int k = it % n_c;
          q_row = k >= ch.n_own ? b_row0 + (k - ch.n_own) * BWD_C : row0 - ch.p0 + qc0;
        }
        uint8_t* dst = smem + Cfg::OFF_C + s * 2 * Cfg::CHUNK_BYTES;
        mbar_arrive_expect_tx(&c_full[s], 2 * Cfg::CHUNK_BYTES);
        for (int a = 0; a < 2; ++a) {
          tma_load_2d(dst + a * Cfg::CHUNK_ATOM, &tmQ, &c_full[s], head * D + a * 64, q_row);
          tma_load_2d(dst + Cfg::CHUNK_BYTES + a * Cfg::CHUNK_ATOM, &tmDO, &c_full[s], head * D + a * 64, q_row);
        }
      }
    }
  } else {
    const FragPos fp = frag_pos();
    const int kvr[2] = {kv0 + wg * 64 + fp.r0, kv0 + wg * 64 + fp.r0 + 8};
    const float c = scale * LOG2E;
    const uint32_t k_addr = smem_u32(smem) + wg * 64 * 128;
    const uint32_t v_addr = smem_u32(smem + Cfg::OFF_T1) + wg * 64 * 128;
    mbar_wait(kv_full, 0);
    float acc[D / 2];
#pragma unroll 1
    for (int pass = 0; pass < 2; ++pass) {
      if (pass == 0)
        varlen_dkv_pass<false, PREFIX>(smem, c_full, c_empty, 0, n_it, n_c, c_first, kv_head, kv_group, blk0, len, ch,
                                       kvr, k_addr, v_addr, c, scale, lse, delta, acc);
      else
        varlen_dkv_pass<true, PREFIX>(smem, c_full, c_empty, n_it, n_it, n_c, c_first, kv_head, kv_group, blk0, len, ch,
                                      kvr, k_addr, v_addr, c, scale, lse, delta, acc);
      bf16* dst = pass == 0 ? dv : dk;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int kv = kvr[h];
        if (kv >= ch.p0 + len) continue;
        bf16* row = dst + ((long long)row0 - ch.p0 + kv) * ld_dkv + kv_head * D + fp.c0;
#pragma unroll
        for (int i = 0; i < D / 8; ++i)
          *reinterpret_cast<uint32_t*>(row + 8 * i) = pack_bf16(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
      }
    }
  }
}

template <bool PREFIX>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_varlen_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                               const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                               const float* __restrict__ lse, const float* __restrict__ delta, bf16* __restrict__ dq,
                               long long ld_dq, const int* __restrict__ cu, int n_heads, int kv_group, float scale,
                               const __grid_constant__ PrefixMap<PREFIX> pm) {
  using Cfg = AttBwdCfg;
  constexpr int D = BWD_D;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* q_full = bars;
  uint64_t* c_full = bars + 1;
  uint64_t* c_empty = bars + 1 + ATT_STAGES;

  const int seq = blockIdx.z;
  const int row0 = cu[seq], len = cu[seq + 1] - row0;
  const int num_q_tiles = (len + 127) / 128;
  if ((int)blockIdx.x >= num_q_tiles) return;
  int p0 = 0, lrow0 = row0;                                   // first own position; the lender's row of position 0
  if constexpr (PREFIX) {
    p0 = pm.pos0[seq];
    if (p0 > 0) lrow0 = cu[pm.partner[seq]];
  }
  const int end = p0 + len;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int q_tile = num_q_tiles - 1 - blockIdx.x;            // heavy (late) tiles first
  const int q0 = p0 + q_tile * 128;
  const int head = blockIdx.y;
  const int kv_head = head / kv_group;
  const int n_c = min((end + BWD_C - 1) / BWD_C, (q0 + 128 + BWD_C - 1) / BWD_C);

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < ATT_STAGES; ++i) { mbar_init(&c_full[i], 1); mbar_init(&c_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    if (threadIdx.x == 256) {
      tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmDO);
      mbar_arrive_expect_tx(q_full, 2 * Cfg::TILE_BYTES);
      for (int a = 0; a < 2; ++a) {
        tma_load_2d(smem + a * Cfg::TILE_ATOM, &tmQ, q_full, head * D + a * 64, row0 - p0 + q0);
        tma_load_2d(smem + Cfg::OFF_T1 + a * Cfg::TILE_ATOM, &tmDO, q_full, head * D + a * 64, row0 - p0 + q0);
      }
      for (int j = 0; j < n_c; ++j) {
        const int s = j % ATT_STAGES;
        if (j >= ATT_STAGES) mbar_wait(&c_empty[s], ((j / ATT_STAGES) - 1) & 1);
        uint8_t* dst = smem + Cfg::OFF_C + s * 2 * Cfg::CHUNK_BYTES;
        mbar_arrive_expect_tx(&c_full[s], 2 * Cfg::CHUNK_BYTES);
        const int kv_row = (PREFIX && j * BWD_C < p0 ? lrow0 : row0 - p0) + j * BWD_C;
        for (int a = 0; a < 2; ++a) {
          tma_load_2d(dst + a * Cfg::CHUNK_ATOM, &tmK, &c_full[s], kv_head * D + a * 64, kv_row);
          tma_load_2d(dst + Cfg::CHUNK_BYTES + a * Cfg::CHUNK_ATOM, &tmV, &c_full[s], kv_head * D + a * 64, kv_row);
        }
      }
    }
  } else {
    const FragPos fp = frag_pos();
    const int qr[2] = {q0 + wg * 64 + fp.r0, q0 + wg * 64 + fp.r0 + 8};
    const float c = scale * LOG2E;
    const long long base = (long long)n_heads * row0 + (long long)head * len - p0;
    float lse2[2], dl[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      lse2[h] = qr[h] < end ? lse[base + qr[h]] * LOG2E : INFINITY;
      dl[h] = qr[h] < end ? delta[base + qr[h]] : 0.f;
    }
    float dqacc[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) dqacc[i] = 0.f;
    const uint32_t q_addr = smem_u32(smem) + wg * 64 * 128;
    const uint32_t do_addr = smem_u32(smem + Cfg::OFF_T1) + wg * 64 * 128;
    mbar_wait(q_full, 0);
    for (int j = 0; j < n_c; ++j) {
      const int s = j % ATT_STAGES;
      const uint32_t k_addr = smem_u32(smem + Cfg::OFF_C + s * 2 * Cfg::CHUNK_BYTES);
      const uint32_t v_addr = k_addr + Cfg::CHUNK_BYTES;
      mbar_wait(&c_full[s], (j / ATT_STAGES) & 1);
      float sv[32], dp[32];
      wgmma_fence();
      mma_qk_64<D>(sv, q_addr, Cfg::TILE_ATOM, k_addr, Cfg::CHUNK_ATOM);
      mma_qk_64<D>(dp, do_addr, Cfg::TILE_ATOM, v_addr, Cfg::CHUNK_ATOM);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(sv);
      reg_fence(dp);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int kv = j * BWD_C + 8 * i + fp.c0 + (e & 1);
          const int h = e >> 1;
          const bool masked = kv >= end || kv > qr[h];
          const float p = masked ? 0.f : fast_exp2(sv[4 * i + e] * c - lse2[h]);
          dp[4 * i + e] = p * (dp[4 * i + e] - dl[h]) * scale;
        }
      uint32_t da[4][4];
      acc_to_afrag<4>(dp, da);
      reg_fence(dqacc);
      wgmma_fence();
      mma_pv<D, 4>(dqacc, da, k_addr, Cfg::CHUNK_ATOM);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(dqacc);
      if (lane == 0) mbar_arrive(&c_empty[s]);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = qr[h];
      if (q >= end) continue;
      bf16* row = dq + ((long long)row0 - p0 + q) * ld_dq + head * D + fp.c0;
#pragma unroll
      for (int i = 0; i < D / 8; ++i)
        *reinterpret_cast<uint32_t*>(row + 8 * i) = pack_bf16(dqacc[4 * i + 2 * h], dqacc[4 * i + 2 * h + 1]);
    }
  }
}

static int make_packed_tmap(CUtensorMap* tm, const void* ptr, long long ld, long long n_rows, int cols, int box_rows) {
  uint64_t dims[2] = {(uint64_t)cols, (uint64_t)n_rows};
  uint64_t str[1] = {(uint64_t)ld * 2};
  uint32_t box[2] = {64, (uint32_t)box_rows};
  return make_tmap_bf16(tm, ptr, 2, dims, str, box);
}

static int varlen_check(const char* who, long long ld_qkv, long long ld_out, void* out, int nseq, int max_len,
                        long long n_rows, int n_heads, int n_kv_heads, int head_dim) {
  B200_REQUIRE(head_dim == 128, "%s: head_dim must be 128 (got %d)", who, head_dim);
  B200_REQUIRE(n_kv_heads > 0 && n_heads % n_kv_heads == 0, "%s: n_heads %d not a multiple of n_kv_heads %d", who,
               n_heads, n_kv_heads);
  B200_REQUIRE(nseq > 0 && max_len > 0 && n_rows > 0 && n_rows < 2147483647LL, "%s: bad shape", who);
  B200_REQUIRE(ld_qkv % 8 == 0 && ld_out % 8 == 0 && ((uintptr_t)out & 15) == 0,
               "%s: ld must be a multiple of 8 and out 16-byte aligned", who);
  return 0;
}

// a sequence either lends or borrows, never both, and lends to at most one: pos0 multiples of 128, partner links
// that pair a borrower (pos0 > 0) with a lender (pos0 == 0) both ways
static int prefix_check(const char* who, const int* pos0, const int* partner, int nseq, PrefixMap<true>* pm) {
  B200_REQUIRE(pos0 != nullptr && partner != nullptr, "%s: pos0 / partner missing", who);
  B200_REQUIRE(nseq <= PREFIX_MAX_SEQ, "%s: %d sequences (at most %d)", who, nseq, PREFIX_MAX_SEQ);
  for (int s = 0; s < nseq; ++s) {
    const int p = pos0[s], b = partner[s];
    B200_REQUIRE(p >= 0 && p % ATT_BKV == 0, "%s: pos0[%d] = %d is not a non-negative multiple of %d", who, s, p,
                 ATT_BKV);
    B200_REQUIRE(b >= -1 && b < nseq && b != s, "%s: partner[%d] = %d out of range", who, s, b);
    B200_REQUIRE(p == 0 || b >= 0, "%s: sequence %d borrows (pos0 %d) without a lender", who, s, p);
    B200_REQUIRE(b < 0 || (partner[b] == s && (p > 0) != (pos0[b] > 0)),
                 "%s: sequences %d and %d are not one lender and one borrower of each other", who, s, b);
    pm->pos0[s] = p;
    pm->partner[s] = b;
  }
  return 0;
}

template <bool PREFIX>
static int varlen_fwd(const void* q, const void* k, const void* v, long long ld_qkv, void* out, long long ld_out,
                      float* lse, const int* cu, int nseq, int max_len, long long n_rows, int n_heads, int n_kv_heads,
                      int head_dim, float scale, void* stream, const PrefixMap<PREFIX>& pm) {
  int rc;
  CUtensorMap tq, tk, tv;
  if ((rc = make_packed_tmap(&tq, q, ld_qkv, n_rows, n_heads * head_dim, ATT_BQ))) return rc;
  if ((rc = make_packed_tmap(&tk, k, ld_qkv, n_rows, n_kv_heads * head_dim, ATT_BKV))) return rc;
  if ((rc = make_packed_tmap(&tv, v, ld_qkv, n_rows, n_kv_heads * head_dim, ATT_BKV))) return rc;
  auto kern = attention_varlen_fwd_kernel<PREFIX>;
  B200_CHECK_CUDA(configure_smem_once((const void*)kern, (int)AttFwdCfg<128>::SMEM_BYTES));
  dim3 grid((max_len + ATT_BQ - 1) / ATT_BQ, n_heads, nseq);
  kern<<<grid, ATT_THREADS, AttFwdCfg<128>::SMEM_BYTES, (cudaStream_t)stream>>>(
      tq, tk, tv, (bf16*)out, ld_out, lse, cu, n_heads, n_heads / n_kv_heads, scale, pm);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

template <bool PREFIX>
static int varlen_bwd(const char* who, const void* q, const void* k, const void* v, long long ld_qkv, const void* out,
                      long long ld_out, const void* d_out, long long ld_dout, const float* lse, void* dq,
                      long long ld_dq, void* dk, void* dv, long long ld_dkv, float* delta_ws, const int* cu, int nseq,
                      int max_len, long long n_rows, int n_heads, int n_kv_heads, int head_dim, float scale,
                      void* stream, const PrefixMap<PREFIX>& pm) {
  int rc;
  B200_REQUIRE(ld_dout % 8 == 0 && ((uintptr_t)d_out & 15) == 0, "%s: d_out must be 16-byte aligned", who);
  B200_REQUIRE(dq != nullptr && ld_dq % 2 == 0 && ((uintptr_t)dq & 3) == 0 && ld_dkv % 2 == 0,
               "%s: dq / dk / dv alignment", who);
  const int g = n_heads / n_kv_heads;
  CUtensorMap tq, tk, tv, tdo, tq2, tk2, tv2, tdo2;
  if ((rc = make_packed_tmap(&tq, q, ld_qkv, n_rows, n_heads * head_dim, BWD_C))) return rc;
  if ((rc = make_packed_tmap(&tdo, d_out, ld_dout, n_rows, n_heads * head_dim, BWD_C))) return rc;
  if ((rc = make_packed_tmap(&tk, k, ld_qkv, n_rows, n_kv_heads * head_dim, 128))) return rc;
  if ((rc = make_packed_tmap(&tv, v, ld_qkv, n_rows, n_kv_heads * head_dim, 128))) return rc;
  if ((rc = make_packed_tmap(&tq2, q, ld_qkv, n_rows, n_heads * head_dim, 128))) return rc;
  if ((rc = make_packed_tmap(&tdo2, d_out, ld_dout, n_rows, n_heads * head_dim, 128))) return rc;
  if ((rc = make_packed_tmap(&tk2, k, ld_qkv, n_rows, n_kv_heads * head_dim, BWD_C))) return rc;
  if ((rc = make_packed_tmap(&tv2, v, ld_qkv, n_rows, n_kv_heads * head_dim, BWD_C))) return rc;
  auto dkv_kern = attention_varlen_bwd_dkv_kernel<PREFIX>;
  auto dq_kern = attention_varlen_bwd_dq_kernel<PREFIX>;
  B200_CHECK_CUDA(configure_smem_once((const void*)dkv_kern, (int)AttBwdCfg::SMEM_BYTES));
  B200_CHECK_CUDA(configure_smem_once((const void*)dq_kern, (int)AttBwdCfg::SMEM_BYTES));
  cudaStream_t st = (cudaStream_t)stream;
  {
    const long long total = n_rows * n_heads;
    long long blocks = (total + 7) / 8;
    if (blocks > (long long)num_sms() * 16) blocks = (long long)num_sms() * 16;
    attention_varlen_delta_kernel<<<(int)blocks, 256, 0, st>>>((const bf16*)out, ld_out, (const bf16*)d_out, ld_dout,
                                                               delta_ws, cu, nseq, n_rows, n_heads, head_dim);
    B200_CHECK_CUDA(cudaGetLastError());
  }
  {
    dim3 grid((max_len + 127) / 128, n_kv_heads, nseq);
    dkv_kern<<<grid, ATT_THREADS, AttBwdCfg::SMEM_BYTES, st>>>(tq, tk, tv, tdo, lse, delta_ws, (bf16*)dk, (bf16*)dv,
                                                               ld_dkv, cu, n_heads, g, scale, pm);
    B200_CHECK_CUDA(cudaGetLastError());
  }
  {
    dim3 grid((max_len + 127) / 128, n_heads, nseq);
    dq_kern<<<grid, ATT_THREADS, AttBwdCfg::SMEM_BYTES, st>>>(tq2, tk2, tv2, tdo2, lse, delta_ws, (bf16*)dq, ld_dq, cu,
                                                              n_heads, g, scale, pm);
    B200_CHECK_CUDA(cudaGetLastError());
  }
  return 0;
}

}  // namespace b200

// Packed causal self-attention: q/k/v/out [n_rows][ld] bf16 (q, k, v may be column blocks of one fused qkv buffer);
// cu int32 [nseq + 1] (device) cuts the rows into sequences, max_len >= the longest; lse fp32 [n_heads * n_rows].
extern "C" int rlaifv_attention_varlen_fwd(const void* q, const void* k, const void* v, long long ld_qkv, void* out,
                                           long long ld_out, float* lse, const int* cu, int nseq, int max_len,
                                           long long n_rows, int n_heads, int n_kv_heads, int head_dim, float scale,
                                           void* stream) {
  int rc;
  if ((rc = varlen_check("attention_varlen_fwd", ld_qkv, ld_out, out, nseq, max_len, n_rows, n_heads, n_kv_heads,
                         head_dim)))
    return rc;
  return varlen_fwd<false>(q, k, v, ld_qkv, out, ld_out, lse, cu, nseq, max_len, n_rows, n_heads, n_kv_heads, head_dim,
                           scale, stream, PrefixMap<false>{});
}

// Its backward: delta, the dK/dV kernel, then the dQ kernel, which writes bf16 dQ [n_rows][ld_dq] (may be the q column
// block of a fused dqkv buffer). dk/dv bf16 [n_rows][ld_dkv]; delta_ws fp32 [n_heads * n_rows]. Nothing needs zeroing.
extern "C" int rlaifv_attention_varlen_bwd(const void* q, const void* k, const void* v, long long ld_qkv,
                                           const void* out, long long ld_out, const void* d_out, long long ld_dout,
                                           const float* lse, void* dq, long long ld_dq, void* dk, void* dv,
                                           long long ld_dkv, float* delta_ws, const int* cu, int nseq, int max_len,
                                           long long n_rows, int n_heads, int n_kv_heads, int head_dim, float scale,
                                           void* stream) {
  int rc;
  if ((rc = varlen_check("attention_varlen_bwd", ld_qkv, ld_out, (void*)out, nseq, max_len, n_rows, n_heads,
                         n_kv_heads, head_dim)))
    return rc;
  return varlen_bwd<false>("attention_varlen_bwd", q, k, v, ld_qkv, out, ld_out, d_out, ld_dout, lse, dq, ld_dq, dk, dv,
                           ld_dkv, delta_ws, cu, nseq, max_len, n_rows, n_heads, n_kv_heads, head_dim, scale, stream,
                           PrefixMap<false>{});
}

// Packed causal self-attention with borrowed prefixes: the arguments of rlaifv_attention_varlen_fwd plus pos0 and
// partner, int32 [nseq] host arrays (at most 64 sequences). Sequence s's own rows [cu[s], cu[s+1]) hold positions
// pos0[s] .. pos0[s] + len_s - 1 (pos0 a multiple of 128); with pos0[s] > 0, positions t < pos0[s] are the rows
// cu[partner[s]] + t of its lender, which holds at least pos0[s] rows and has partner = s and pos0 = 0. -1 = no partner.
extern "C" int rlaifv_attention_varlen_prefix_fwd(const void* q, const void* k, const void* v, long long ld_qkv,
                                                  void* out, long long ld_out, float* lse, const int* cu,
                                                  const int* pos0, const int* partner, int nseq, int max_len,
                                                  long long n_rows, int n_heads, int n_kv_heads, int head_dim,
                                                  float scale, void* stream) {
  int rc;
  if ((rc = varlen_check("attention_varlen_prefix_fwd", ld_qkv, ld_out, out, nseq, max_len, n_rows, n_heads,
                         n_kv_heads, head_dim)))
    return rc;
  PrefixMap<true> pm;
  if ((rc = prefix_check("attention_varlen_prefix_fwd", pos0, partner, nseq, &pm))) return rc;
  return varlen_fwd<true>(q, k, v, ld_qkv, out, ld_out, lse, cu, nseq, max_len, n_rows, n_heads, n_kv_heads, head_dim,
                          scale, stream, pm);
}

// Its backward (arguments of rlaifv_attention_varlen_bwd plus pos0 / partner): dQ and dK/dV of own rows; a lender's
// rows below its borrower's pos0 receive the sum of both sequences' dK/dV.
extern "C" int rlaifv_attention_varlen_prefix_bwd(const void* q, const void* k, const void* v, long long ld_qkv,
                                                  const void* out, long long ld_out, const void* d_out,
                                                  long long ld_dout, const float* lse, void* dq, long long ld_dq,
                                                  void* dk, void* dv, long long ld_dkv, float* delta_ws,
                                                  const int* cu, const int* pos0, const int* partner, int nseq,
                                                  int max_len, long long n_rows, int n_heads, int n_kv_heads,
                                                  int head_dim, float scale, void* stream) {
  int rc;
  if ((rc = varlen_check("attention_varlen_prefix_bwd", ld_qkv, ld_out, (void*)out, nseq, max_len, n_rows, n_heads,
                         n_kv_heads, head_dim)))
    return rc;
  PrefixMap<true> pm;
  if ((rc = prefix_check("attention_varlen_prefix_bwd", pos0, partner, nseq, &pm))) return rc;
  return varlen_bwd<true>("attention_varlen_prefix_bwd", q, k, v, ld_qkv, out, ld_out, d_out, ld_dout, lse, dq, ld_dq,
                          dk, dv, ld_dkv, delta_ws, cu, nseq, max_len, n_rows, n_heads, n_kv_heads, head_dim, scale,
                          stream, pm);
}

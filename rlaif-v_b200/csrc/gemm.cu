// bf16 x bf16 -> fp32 -> bf16 GEMM for sm_90a: TMA-staged SWIZZLE_128B shared-memory tiles feeding wgmma.mma_async
// (64 x BN x 16 per warpgroup), persistent warp-specialised CTAs: one producer warpgroup issues the TMA loads of a
// multi-stage ring, two math warpgroups each own 64 rows of the 128 x BN tile and run the epilogue while the producer
// already streams the next tile's operands. The plain, residual and SwiGLU-backward epilogues write C through shared
// memory with TMA stores (epilogue_staged); the general one stores from the accumulator registers.
//
// One kernel covers the three operand forms a linear layer needs (reference call sites: every
// nn.Linear inside HF LlamaDecoderLayer / CLIPEncoderLayer / mm_projector —
// llava/model/language_model/llava_llama.py:91-102, llava/model/multimodal_projector/builder.py:39-46):
//   forward  Y[M,N]  = X[M,K]  * W[N,K]^T      A K-major,  B K-major
//   dgrad    dX[M,K] = dY[M,N] * W[N,K]        A K-major,  B MN-major
//   wgrad    dW[N,K] = dY[M,N]^T * X[M,K]      A MN-major, B MN-major
// "K-major" = contraction index contiguous in memory; "MN-major" = the tensor is stored
// [contraction][M or N] row-major. No transposes are ever materialised: wgmma reads MN-major tiles transposed.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one thread issues), warpgroups 1, 2 = MMA + epilogue of rows
// [0, 64) and [64, 128) of the tile.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

struct GemmEpilogue {
  bf16* C;
  long long ldc;
  const bf16* bias;      // [N] or nullptr
  const bf16* residual;  // [M, ldr] or nullptr
  long long ldr;
  int act;         // 0 none, 1 GELU(erf), 2 quick_gelu (x*sigmoid(1.702x))
  int accumulate;  // C = C + result (fp32 add of the old bf16 value)
  int group_m;     // raster: tiles are walked m-fastest inside groups of `group_m` row-blocks
  int debug;       // profiling only: bit0 skip the epilogue (mainloop only)
  float alpha;     // != 1: result = bf16(bf16(acc) * alpha) first (LoRA scaling, peft: lora_B(...) * scaling)
  const bf16* glu; // non-null: fused SwiGLU backward. The accumulator tile is d(act) [M, N = F]; glu = [gate | up] rows
  long long ld_glu;//   [M, 2F]; C = d[gate | up] [M, 2F]: C[:, n] = d*u*silu'(g), C[:, F + n] = d*silu(g)  (d = bf16(acc))
  int l2;          // L2 policy of the operand loads: bits 0-1 A, 2-3 B (0 normal, 1 evict first, 2 evict last);
                   // bit 6: raster groups column blocks (n-fastest inside groups of group_m)
};

// Optional second operand pair accumulated into the same accumulator tile after the first K loop:
//   C = A1 * B1^T + A2[:, koff : koff + K2] * B2^T,   koff = (n0 / n_sub) * r   (0 when n_sub == 0).
// This is how the LoRA rank-r update rides in the same CTA pass as the frozen base GEMM
// (forward: A2 = s*A(x) [M, g*r], B2 = stacked lora_B [N, r]; dgrad: A2 = s*dy*B [M, g*r], B2 = stacked lora_A).
struct GemmSecondSource {
  int K2;      // 0 = disabled
  int r;       // adapter rank (column-block width of A2 per sub-linear)
  int n_sub;   // output columns per sub-linear (forward) or 0
};

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_THREADS = 384;
constexpr uint32_t ATOM_BYTES = 64 * 128;   // one [64 rows][64 bf16] SWIZZLE_128B atom

// Epilogue forms, a template parameter of the kernel so that each launch carries only its own code:
//   EPI_PLAIN     C = bf16(acc)
//   EPI_RESIDUAL  C = bf16(bf16(acc) + residual)
//   EPI_GLU       fused SwiGLU backward (epilogue_pair_glu)
//   EPI_GENERAL   epilogue_pair: alpha, bias, activation, residual, accumulate in any combination
// PLAIN and RESIDUAL compute exactly what epilogue_pair computes for those arguments.
enum EpiKind { EPI_GENERAL, EPI_PLAIN, EPI_RESIDUAL, EPI_GLU };

// STAGED: the plain, residual and SwiGLU forms write C through SWIZZLE_128B staging atoms in the 32 KB of shared memory
// the ring leaves free (TMA stores; the residual and gate|up come in by TMA loads into the same atoms). Each math
// warpgroup owns two atoms: SLOTS staging slots of SLOT_ATOMS atoms, one subtile of 64 rows x 64 columns (SwiGLU: its
// gate and up halves) per slot. The SwiGLU form is thus single-buffered. A double-buffered one (a ring of 3 stages at
// tile 256, 5 at tile 128, to free the atoms) was 6 % slower on the LoRA step's down-projection dgrad (H100 SXM, 400 W):
// that launch waits on operand supply more than on its epilogue.
template <int BN, int EPI = EPI_GENERAL, bool STAGED = false>
struct GemmCfg {
  static constexpr int STAGES = (BN == 256) ? 4 : 6;    // 192 KB of the 227 KB a block may use
  static constexpr uint32_t A_BYTES = GEMM_BM * GEMM_BK * 2;
  static constexpr uint32_t B_BYTES = BN * GEMM_BK * 2;
  static constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int SLOT_ATOMS = EPI == EPI_GLU ? 2 : 1;
  static constexpr int SLOTS = EPI == EPI_GLU ? 1 : 2;
  static constexpr uint32_t WG_STAGING_BYTES = STAGED ? SLOTS * SLOT_ATOMS * ATOM_BYTES : 0;
  static constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES + 2 * WG_STAGING_BYTES + 256 + 1024;  // + barriers
                                                                                                   //   + alignment
  static_assert(SMEM_BYTES <= 232448, "over the 227 KB of shared memory a block may opt in to");
};

// Stall accounting, compiled in only with -DRLAIFV_GEMM_STALLS (tools/gemm_step_shapes.py builds that variant; the
// shipped library has none of it). Every CTA adds its clock64() counts to the device-wide sums below: one math thread
// per consumer warpgroup times its waits on the `full` barriers and its epilogue, the producer thread its waits on the
// `empty` barriers. Consumers waiting on `full` = operand supply (L2 / DRAM) is the limit; a producer waiting on
// `empty` while the consumers do not = the MMA issue rate is; epilogue cycles = tensor-core time lost between tiles.
enum GemmStall { ST_CTAS, ST_TILES, ST_CONS_TOTAL, ST_CONS_FULL_WAIT, ST_CONS_EPILOGUE, ST_PROD_TOTAL,
                 ST_PROD_EMPTY_WAIT, ST_FIELDS };
// The consumers' hooks keep no clock value live across the epilogue or the tile loop (next to the 128 accumulators it
// would spill, and the counters would then time a different epilogue from the shipped one): a span is added to its
// sum as -clock64() at its start and +clock64() at its end (stall_mark), a tile's `full` waits are summed in 32 bits,
// and the consumers' total is the sum of their tiles' spans (first `full` wait to the end of the epilogue).
#ifdef RLAIFV_GEMM_STALLS
__device__ unsigned long long g_gemm_stalls[ST_FIELDS];
__device__ __forceinline__ long long stall_clock() { return clock64(); }
__device__ __forceinline__ uint32_t stall_clock32() { return (uint32_t)clock(); }
__device__ __forceinline__ void stall_add(int field, long long v) {
  atomicAdd(&g_gemm_stalls[field], (unsigned long long)v);
}
__device__ __forceinline__ void stall_mark(int field, bool end) {
  const long long c = clock64();
  atomicAdd(&g_gemm_stalls[field], (unsigned long long)(end ? c : -c));
}
#else
__device__ __forceinline__ long long stall_clock() { return 0; }
__device__ __forceinline__ uint32_t stall_clock32() { return 0; }
__device__ __forceinline__ void stall_add(int, long long) {}
__device__ __forceinline__ void stall_mark(int, bool) {}
#endif

__device__ __forceinline__ void tile_coords(int t, int num_m, int num_n, int GROUP_M, int& m_blk, int& n_blk,
                                            bool n_grouped = false) {
  if (n_grouped) {            // same walk with the roles of m and n exchanged: groups of GROUP_M column blocks
    tile_coords(t, num_n, num_m, GROUP_M, n_blk, m_blk, false);
    return;
  }
  int per_group = GROUP_M * num_n;
  int g = t / per_group;
  int first_m = g * GROUP_M;
  int gsz = min(num_m - first_m, GROUP_M);
  int r = t - g * per_group;
  m_blk = first_m + r % gsz;
  n_blk = r / gsz;
}

__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == 1) return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
  if (act == 2) return v / (1.0f + __expf(-1.702f * v));
  return v;
}

// Epilogue of two adjacent accumulator columns (col, col + 1) of one output row.
__device__ __forceinline__ void epilogue_pair(float v0, float v1, long long row, int col, const GemmEpilogue& epi) {
  if (epi.alpha != 1.0f) {
    v0 = bf16_round(bf16_round(v0) * epi.alpha);
    v1 = bf16_round(bf16_round(v1) * epi.alpha);
  }
  if (epi.bias) {
    const float2 b = unpack_bf16(__ldg(reinterpret_cast<const unsigned int*>(epi.bias + col)));
    v0 += b.x;
    v1 += b.y;
  }
  if (epi.act) {
    v0 = apply_act(bf16_round(v0), epi.act);
    v1 = apply_act(bf16_round(v1), epi.act);
  }
  if (epi.residual) {
    // reference adds two bf16 tensors: round the linear output first
    const float2 q = unpack_bf16(*reinterpret_cast<const uint32_t*>(epi.residual + row * epi.ldr + col));
    v0 = bf16_round(v0) + q.x;
    v1 = bf16_round(v1) + q.y;
  }
  uint32_t* c = reinterpret_cast<uint32_t*>(epi.C + row * epi.ldc + col);
  if (epi.accumulate) {
    const float2 o = unpack_bf16(*c);
    v0 += o.x;
    v1 += o.y;
  }
  *c = pack_bf16(v0, v1);
}

// Fused SwiGLU backward (HF llama/modeling_llama.py:182-184 under autograd): the GEMM computes d(act) = dy @ W_down for
// a slice of F; instead of writing it out for a separate elementwise pass (one more launch, d(act) written and read
// back) the epilogue reads the matching gate / up values and writes d(gate) and d(up) straight into the [M, 2F]
// gradient of the fused gate|up projection. d is rounded to bf16 first (the reference materialises it); the arithmetic
// is swiglu_bwd_kernel's (rowops.cu) with an approximate reciprocal (2 ulp, far below the bf16 rounding of the result).
// g2 / u2: the bf16 pairs gate[row, col..col+1] and up[row, col..col+1]; c_row: row `row` of C.
// swiglu_bwd_pair returns the packed pairs d[gate] (dg2) and d[up] (du2).
__device__ __forceinline__ void swiglu_bwd_pair(float v0, float v1, uint32_t g2, uint32_t u2, uint32_t& dg2,
                                                uint32_t& du2) {
  const float2 g = unpack_bf16(g2), u = unpack_bf16(u2);
  const float d[2] = {bf16_round(v0), bf16_round(v1)}, gv[2] = {g.x, g.y}, uv[2] = {u.x, u.y};
  float dg[2], du[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const float sg = __fdividef(1.f, 1.f + __expf(-gv[j]));
    du[j] = d[j] * (gv[j] * sg);
    dg[j] = d[j] * uv[j] * (sg * (1.f + gv[j] * (1.f - sg)));
  }
  dg2 = pack_bf16(dg[0], dg[1]);
  du2 = pack_bf16(du[0], du[1]);
}
__device__ __forceinline__ void epilogue_pair_glu(float v0, float v1, uint32_t g2, uint32_t u2, bf16* c_row, int col,
                                                  int N) {
  uint32_t dg2, du2;
  swiglu_bwd_pair(v0, v1, g2, u2, dg2, du2);
  *reinterpret_cast<uint32_t*>(c_row + col) = dg2;
  *reinterpret_cast<uint32_t*>(c_row + N + col) = du2;
}

// One accumulator row of a thread (64 or 128 column pairs, h selects the row of the m64 fragment) in one of the
// specialised forms. The residual / gate|up values are read CH pairs at a time, all of them before the first store
// of the group: a store to C may alias them as far as the compiler knows, so loads interleaved with stores would each
// pay a full global-memory round trip in turn.
template <int EPI, int BN>
__device__ __forceinline__ void epilogue_row(const float (&acc)[BN / 2], int h, long long row, int col0, int N,
                                             const GemmEpilogue& epi) {
  constexpr int NP = BN / 8;                        // column pairs of this thread per row
  constexpr int CH = EPI == EPI_GLU ? 16 : NP;      // pairs per load group
  bf16* c_row = epi.C + row * epi.ldc;
#pragma unroll
  for (int i0 = 0; i0 < NP; i0 += CH) {
    uint32_t x[CH], y[CH];
#pragma unroll
    for (int j = 0; j < CH; ++j) {
      const int col = col0 + (i0 + j) * 8;
      if constexpr (EPI == EPI_RESIDUAL) {
        x[j] = col < N ? *reinterpret_cast<const uint32_t*>(epi.residual + row * epi.ldr + col) : 0u;
      } else if constexpr (EPI == EPI_GLU) {
        const bf16* g_row = epi.glu + row * epi.ld_glu;
        x[j] = col < N ? *reinterpret_cast<const uint32_t*>(g_row + col) : 0u;
        y[j] = col < N ? *reinterpret_cast<const uint32_t*>(g_row + N + col) : 0u;
      }
    }
#pragma unroll
    for (int j = 0; j < CH; ++j) {
      const int i = i0 + j, col = col0 + i * 8;
      if (col >= N) continue;
      float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
      if constexpr (EPI == EPI_GLU) {
        epilogue_pair_glu(v0, v1, x[j], y[j], c_row, col, N);
      } else {
        if constexpr (EPI == EPI_RESIDUAL) {
          const float2 q = unpack_bf16(x[j]);
          v0 = bf16_round(v0) + q.x;
          v1 = bf16_round(v1) + q.y;
        }
        *reinterpret_cast<uint32_t*>(c_row + col) = pack_bf16(v0, v1);
      }
    }
  }
}

// Staged epilogue (STAGED kernels) of one math warpgroup's 64 rows x BN columns, one 64 x 64 subtile per staging slot,
// slots taken round robin. Per subtile:
//   1. the slot is free. Plain: the elected thread waits until the bulk store that last used it has been read out,
//      then a named barrier (the warpgroup's 128 threads). Residual / SwiGLU: every thread waits on the slot's
//      mbarrier for the TMA load of this subtile's operands, which was issued only after the slot's previous store had
//      been read out;
//   2. every thread writes its accumulator fragment with stmatrix at the swizzled addresses (residual / SwiGLU: in
//      place, after reading its operand pairs there with ldmatrix; each warp reads and writes only its own 16 rows);
//   3. fence.proxy.async, named barrier, and the elected thread issues the TMA store(s) as one bulk group. It then
//      refills the slot with the operands of subtile j + SLOTS once the store has read it out.
// No one waits for the stores at the end of a tile: the next tile's MMAs run while the copy engine drains the slots.
// TMA clips the boxes at M and N, so M tails and the neighbouring columns of column-block views stay untouched, and a
// C that aliases the residual is read before it is written (a subtile's load lands before its store is issued). The
// values and rounding points are epilogue_row's.
// Shared-window addresses (32 bits: they stay live across the mainloop, next to the accumulators).
struct StagedEpi {
  uint32_t slots;   // this warpgroup's staging atoms
  uint32_t bar;     // one mbarrier per slot: TMA loads of the residual / gate|up subtiles
  int row0;         // first of the warpgroup's 64 rows
  int n0;           // first column of the tile (SwiGLU: in d(act), i.e. in the gate half)
  // subtiles inside N; 0 when all of the warpgroup's rows are past M (recomputed where needed: M and N are kernel
  // parameters, a register held across the mainloop is not)
  __device__ __forceinline__ int nsub(int M, int N, int BN) const {
    return row0 < M ? min(BN / 64, (N - n0 + 63) / 64) : 0;
  }
};

// TMA load of subtile j's residual (or gate and up) into its slot; elected thread only.
template <int EPI, typename Cfg>
__device__ __forceinline__ void staged_load(const StagedEpi& se, int j, const CUtensorMap* tmR, int N) {
  const int slot = j % Cfg::SLOTS;
  uint8_t* dst = smem_ptr<uint8_t>(se.slots + slot * Cfg::SLOT_ATOMS * ATOM_BYTES);
  uint64_t* bar = smem_ptr<uint64_t>(se.bar + slot * 8);
  mbar_arrive_expect_tx(bar, Cfg::SLOT_ATOMS * ATOM_BYTES);
  tma_load_2d(dst, tmR, bar, se.n0 + 64 * j, se.row0);
  if constexpr (EPI == EPI_GLU) tma_load_2d(dst + ATOM_BYTES, tmR, bar, N + se.n0 + 64 * j, se.row0);
}

// Elected thread, as the tile's mainloop starts (the loads land while its MMAs run): the first SLOTS subtiles'
// operands, once the previous tile's stores have been read out of the slots.
template <int EPI, int BN, typename Cfg>
__device__ __forceinline__ void staged_prefetch(const StagedEpi& se, const CUtensorMap* tmR, int M, int N) {
  tma_store_wait_read<0>();
  const int nsub = se.nsub(M, N, BN);
  for (int j = 0; j < Cfg::SLOTS && j < nsub; ++j) staged_load<EPI, Cfg>(se, j, tmR, N);
}

// phase: bit 1 + slot is the parity of the slot's mbarrier (bit 0 belongs to the caller).
template <int EPI, int BN, typename Cfg>
__device__ __forceinline__ void epilogue_staged(const float (&acc)[BN / 2], const StagedEpi& se, uint32_t& phase,
                                                const CUtensorMap* tmC, const CUtensorMap* tmR, int M, int N,
                                                bool leader, int bar_id) {
  const int nsub = se.nsub(M, N, BN);
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  // stmatrix / ldmatrix x4 over column pairs (i, i + 1), i = 8j + 2p: matrix q is pair i + (q >> 1), row half q & 1;
  // this lane addresses row r of matrix q
  const int q = lane >> 3, r = lane & 7;
  const uint32_t row_addr = se.slots + (16 * w + 8 * (q & 1) + r) * 128;
#pragma unroll
  for (int j = 0; j < BN / 64; ++j) {
    if (j >= nsub) break;
    const int slot = j % Cfg::SLOTS;
    const uint32_t slot_off = slot * Cfg::SLOT_ATOMS * ATOM_BYTES;
    if constexpr (EPI == EPI_PLAIN) {
      if (leader) {
        if (j == 0) tma_store_wait_read<0>();   // the previous tile's stores: long done
        else tma_store_wait_read<1>();          // subtile j - 2's store, which used this slot
      }
      named_bar_sync(bar_id, 128);
    } else {
      mbar_wait(smem_ptr<uint64_t>(se.bar + slot * 8), (phase >> (1 + slot)) & 1);
      phase ^= 2u << slot;
    }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      if constexpr (EPI == EPI_GLU) {
        // x2 halves (pair i, both row halves): gate and up in place, four registers fewer live than x4
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const uint32_t addr = row_addr + slot_off + (((2 * p + hf) ^ r) << 4);
          const int i = 8 * j + 2 * p + hf;
          uint32_t x[2], y[2];
          ldmatrix_x2(addr, x);
          ldmatrix_x2(addr + ATOM_BYTES, y);
#pragma unroll
          for (int h = 0; h < 2; ++h) swiglu_bwd_pair(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1], x[h], y[h], x[h], y[h]);
          stmatrix_x2(addr, x);
          stmatrix_x2(addr + ATOM_BYTES, y);
        }
      } else {
        const uint32_t addr = row_addr + slot_off + (((2 * p + (q >> 1)) ^ r) << 4);   // SWIZZLE_128B: chunk ^ row % 8
        uint32_t x[4];   // residual pairs, then (in place) the results
        if constexpr (EPI == EPI_RESIDUAL) ldmatrix_x4(addr, x);
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          const int i = 8 * j + 2 * p + (m >> 1), h = m & 1;
          float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
          if constexpr (EPI == EPI_RESIDUAL) {
            const float2 rv = unpack_bf16(x[m]);
            v0 = bf16_round(v0) + rv.x;
            v1 = bf16_round(v1) + rv.y;
          }
          x[m] = pack_bf16(v0, v1);
        }
        stmatrix_x4(addr, x);
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(bar_id, 128);
    if (leader) {
      const uint8_t* src = smem_ptr<uint8_t>(se.slots + slot_off);
      const int col = se.n0 + 64 * j;
      tma_store_2d(tmC, src, col, se.row0);
      if constexpr (EPI == EPI_GLU) tma_store_2d(tmC, src + ATOM_BYTES, N + col, se.row0);
      tma_store_commit();
      if constexpr (EPI != EPI_PLAIN) {
        if (j + Cfg::SLOTS < nsub) {
          tma_store_wait_read<0>();
          staged_load<EPI, Cfg>(se, j + Cfg::SLOTS, tmR, N);
        }
      }
    }
  }
}

template <bool A_MN, bool B_MN, int BN>
__device__ __forceinline__ void gemm_mma_stage(float (&acc)[BN / 2], uint32_t a_addr, uint32_t b_addr, int first) {
#pragma unroll
  for (int k16 = 0; k16 < GEMM_BK / 16; ++k16) {
    const uint64_t da = A_MN ? desc_mnmajor(a_addr, k16, ATOM_BYTES) : desc_kmajor(a_addr, k16);
    const uint64_t db = B_MN ? desc_mnmajor(b_addr, k16, ATOM_BYTES) : desc_kmajor(b_addr, k16);
    const int accum = (first && k16 == 0) ? 0 : 1;
    if constexpr (BN == 256) wgmma_m64n256_ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, accum);
    else wgmma_m64n128_ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, accum);
  }
}

// CL = 2 (tile_n = 512): a cluster of two CTAs computes a 256 x 256 tile. Each CTA stages its own 128 rows of A and
// one 128-row half of B, which TMA multicasts into the shared memory of both CTAs: per output element the pair reads B
// from L2 once instead of twice. A stage slot is refilled only after the math warps of BOTH CTAs have released it
// (they arrive on the empty barrier of each CTA), since either producer writes into both.
// tmC / tmR (STAGED only): C as {N, M} (SwiGLU: {2F, M}) and the residual (SwiGLU: gate|up) in 64 x 64 boxes.
template <bool A_MN, bool B_MN, int BN, int CL, int EPI, bool STAGED>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
                 const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR,
                 int M, int N, int K, GemmSecondSource src2, GemmEpilogue epi) {
  using Cfg = GemmCfg<BN, EPI, STAGED>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* staging = smem + STAGES * Cfg::STAGE_BYTES;     // 2 x WG_STAGING_BYTES, 1024-byte aligned
  uint64_t* full = reinterpret_cast<uint64_t*>(staging + 2 * Cfg::WG_STAGING_BYTES);
  uint64_t* empty = full + STAGES;
  uint64_t* ebar = empty + STAGES;                          // STAGED: SLOTS per math warpgroup

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const uint32_t rank = CL == 2 ? cluster_ctarank() : 0;
  const int first_tile = blockIdx.x / CL, tile_stride = gridDim.x / CL;
  const int num_m = (M + CL * GEMM_BM - 1) / (CL * GEMM_BM);
  const int num_n = (N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_k1 = (K + GEMM_BK - 1) / GEMM_BK;
  const int num_k = num_k1 + (src2.K2 + GEMM_BK - 1) / GEMM_BK;
  const bool n_grouped = (epi.l2 & 0x40) != 0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (src2.K2 > 0) {
      tma_prefetch_desc(&tmA2);
      tma_prefetch_desc(&tmB2);
    }
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8 * CL);     // lane 0 of each of the 8 math warps (of both CTAs of a pair)
    }
    if (STAGED)
      for (int i = 0; i < 2 * Cfg::SLOTS; ++i) mbar_init(&ebar[i], 1);
    fence_barrier_init();
  }
  if (CL == 2) cluster_sync_all();    // the peer's multicasts and arrives need this CTA's initialised barriers
  else __syncthreads();

  if (wg == 0) {
    // ------------------------------ TMA producer ------------------------------
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      const uint64_t pol_a = l2_policy(epi.l2 & 3), pol_b = l2_policy((epi.l2 >> 2) & 3);
      const long long clk0 = stall_clock();
      long long empty_wait = 0;
      int s = 0;
      uint32_t ph = 0;
      for (int t = first_tile; t < num_tiles; t += tile_stride) {
        int m_blk, n_blk;
        tile_coords(t, num_m, num_n, epi.group_m, m_blk, n_blk, n_grouped);
        const int m0 = (m_blk * CL + (int)rank) * GEMM_BM, n0 = n_blk * BN;
        for (int kb = 0; kb < num_k; ++kb) {
          const long long w0 = stall_clock();
          mbar_wait(&empty[s], ph ^ 1);
          empty_wait += stall_clock() - w0;
          uint8_t* a_dst = smem + s * Cfg::STAGE_BYTES;
          uint8_t* b_dst = a_dst + Cfg::A_BYTES;
          const bool second = kb >= num_k1;
          const CUtensorMap* mA = second ? &tmA2 : &tmA;
          const CUtensorMap* mB = second ? &tmB2 : &tmB;
          const int kB = (second ? kb - num_k1 : kb) * GEMM_BK;                                  // k index into B
          const int kA = second ? kB + (src2.n_sub > 0 ? (n0 / src2.n_sub) * src2.r : 0) : kB;   // into A
          mbar_arrive_expect_tx(&full[s], Cfg::STAGE_BYTES);
          if (A_MN) {
#pragma unroll
            for (int a = 0; a < GEMM_BM / 64; ++a)
              tma_load_2d_hint(a_dst + a * ATOM_BYTES, mA, &full[s], m0 + a * 64, kA, pol_a);
          } else {
            tma_load_2d_hint(a_dst, mA, &full[s], kA, m0, pol_a);
          }
          if (CL == 2) {              // this CTA's half of B, into both CTAs
            if (B_MN) {
#pragma unroll
              for (int a = 2 * (int)rank; a < 2 * (int)rank + 2; ++a)
                tma_load_2d_mc_hint(b_dst + a * ATOM_BYTES, mB, &full[s], n0 + a * 64, kB, 0x3, pol_b);
            } else {
              tma_load_2d_mc_hint(b_dst + rank * (128 * 128), mB, &full[s], kB, n0 + 128 * (int)rank, 0x3, pol_b);
            }
          } else if (B_MN) {
#pragma unroll
            for (int a = 0; a < BN / 64; ++a)
              tma_load_2d_hint(b_dst + a * ATOM_BYTES, mB, &full[s], n0 + a * 64, kB, pol_b);
          } else {
            tma_load_2d_hint(b_dst, mB, &full[s], kB, n0, pol_b);
          }
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
      stall_add(ST_CTAS, 1);
      stall_add(ST_PROD_TOTAL, stall_clock() - clk0);
      stall_add(ST_PROD_EMPTY_WAIT, empty_wait);
    }
  } else {
    // ------------------------------ MMA + epilogue: 64 rows per warpgroup ------------------------------
    setmaxnreg_inc<232>();
    const int cw = wg - 1;                                  // rows [64*cw, 64*cw + 64) of the tile
    const int g = lane >> 2, tq = lane & 3;
    float acc[BN / 2];
    int s = 0;
    uint32_t ph = 0;             // bit 0: parity of the ring's `full` barriers; STAGED: bits 1.. those of the slots
    auto release = [&](int slot) {
      mbar_arrive(&empty[slot]);
      if (CL == 2) mbar_arrive_cluster(&empty[slot], rank ^ 1);
    };
    const bool timer = (threadIdx.x & 127) == 0;   // also the warpgroup's elected thread of the staged epilogue
    StagedEpi se;
    se.slots = smem_u32(staging + cw * Cfg::WG_STAGING_BYTES);
    se.bar = smem_u32(ebar + cw * Cfg::SLOTS);
    for (int t = first_tile; t < num_tiles; t += tile_stride) {
      if (timer) stall_mark(ST_CONS_TOTAL, false);
      int m_blk, n_blk;
      tile_coords(t, num_m, num_n, epi.group_m, m_blk, n_blk, n_grouped);
      if constexpr (STAGED) {
        se.row0 = (m_blk * CL + (int)rank) * GEMM_BM + cw * 64;
        se.n0 = n_blk * BN;
        if constexpr (EPI != EPI_PLAIN) {
          if (timer && !(epi.debug & 1)) staged_prefetch<EPI, BN, Cfg>(se, &tmR, M, N);
        }
      }
      int prev = -1;
      uint32_t full_wait = 0;
      for (int kb = 0; kb < num_k; ++kb) {
        full_wait -= stall_clock32();
        mbar_wait(&full[s], ph & 1);
        full_wait += stall_clock32();
        const uint32_t a_addr = smem_u32(smem + s * Cfg::STAGE_BYTES) + cw * ATOM_BYTES;   // 64 rows / 2nd M atom
        const uint32_t b_addr = smem_u32(smem + s * Cfg::STAGE_BYTES + Cfg::A_BYTES);
        reg_fence(acc);
        wgmma_fence();
        gemm_mma_stage<A_MN, B_MN, BN>(acc, a_addr, b_addr, kb == 0);
        wgmma_commit();
        wgmma_wait<1>();              // the previous stage's MMAs are complete: hand its slot back to the producer
        reg_fence(acc);
        if (prev >= 0 && lane == 0) release(prev);
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (lane == 0) release(prev);
      if (timer) {
        stall_add(ST_TILES, 1);
        stall_add(ST_CONS_FULL_WAIT, full_wait);
      }
      if (epi.debug & 1) {
        if (timer) stall_mark(ST_CONS_TOTAL, true);
        continue;
      }
      if (timer) stall_mark(ST_CONS_EPILOGUE, false);
      if constexpr (STAGED) {
        epilogue_staged<EPI, BN, Cfg>(acc, se, ph, &tmC, &tmR, M, N, timer, 1 + cw);
      } else {
        const long long row0 = (long long)(m_blk * CL + (int)rank) * GEMM_BM + cw * 64 + (warp & 3) * 16 + g;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long row = row0 + h * 8;
          if (row >= M) continue;
          if constexpr (EPI != EPI_GENERAL) {
            epilogue_row<EPI, BN>(acc, h, row, n_blk * BN + tq * 2, N, epi);
          } else {
#pragma unroll
            for (int i = 0; i < BN / 8; ++i) {
              const int col = n_blk * BN + i * 8 + tq * 2;
              if (col >= N) continue;
              epilogue_pair(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1], row, col, epi);
            }
          }
        }
      }
      if (timer) {
        stall_mark(ST_CONS_EPILOGUE, true);
        stall_mark(ST_CONS_TOTAL, true);
      }
    }
    if (STAGED && timer) tma_store_wait_all<0>();   // the slots must outlive the bulk stores that read them
  }
  if (CL == 2) cluster_sync_all();    // the peer may still multicast into / arrive on this CTA's shared memory
}

// ------------------------------------------------------------------------------------------------------------------
// FP8 frozen-base GEMM (DESIGN.md §3 "FP8 frozen base"): C = sum_kb sa[m, kb] * sb[n / 128, kb] * (qa[m, kb] . qb[n, kb])
// over e4m3 codes in 128-deep K-blocks, then the optional bf16 second source, then the plain, residual or
// SwiGLU-backward staged epilogue. One SWIZZLE_128B row holds 128 e4m3, so an FP8 stage (128 x 128 bytes of A and of
// B) has the byte layout of a bf16 stage of 64 K and the same descriptor stepping (one k32 step = 32 bytes); the ring,
// the producer protocol and the staging atoms are those of gemm_bf16_kernel at tile 128 x 128.
// The tensor cores accumulate FP8 products at a reduced, undocumented precision, so each K-block goes into its own
// partial accumulator (scale-d = 0 on its first k32 step) and is promoted into the fp32 accumulator with one FMA by
// the exact power-of-two product of its two scales. Two 64-register accumulators per math thread.
constexpr int FP8_BK = 128;     // e4m3 per K-block: one 128-byte swizzled row, one scale per row / per weight block

struct Fp8Scales {
  const float* sa;     // row scales of A: [K / 128][ld_sa], row m of K-block kb at sa[kb * ld_sa + m]
  long long ld_sa;
  const float* sb;     // block scales of B: output block nb, K-block kb at sb[nb * sb_n + kb * sb_k]
  int sb_n, sb_k;
};

__device__ __forceinline__ void wgmma_m64n128k32_e4m3(float (&d)[64], uint64_t da, uint64_t db, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(acc));
}

// tmA / tmB: e4m3 codes as {K, rows} bytes in 128 x 128 boxes; tmA2 / tmB2: the bf16 second source as in
// gemm_bf16_kernel (B2 MN-major when B2_MN); tmC / tmR as in the staged bf16 kernel. K % 128 == 0, N % 128 == 0.
template <int EPI, bool B2_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
                const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR,
                int M, int N, int K, GemmSecondSource src2, Fp8Scales sc, GemmEpilogue epi) {
  constexpr int BN = 128;
  using Cfg = GemmCfg<BN, EPI, true>;
  constexpr int STAGES = Cfg::STAGES;
  static_assert(Cfg::A_BYTES == GEMM_BM * FP8_BK && Cfg::B_BYTES == BN * FP8_BK, "an e4m3 stage fills a bf16 slot");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* staging = smem + STAGES * Cfg::STAGE_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(staging + 2 * Cfg::WG_STAGING_BYTES);
  uint64_t* empty = full + STAGES;
  uint64_t* ebar = empty + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int num_m = (M + GEMM_BM - 1) / GEMM_BM;
  const int num_n = N / BN;
  const int num_tiles = num_m * num_n;
  const int num_k1 = K / FP8_BK;
  const int num_k = num_k1 + (src2.K2 + GEMM_BK - 1) / GEMM_BK;
  const bool n_grouped = (epi.l2 & 0x40) != 0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (src2.K2 > 0) {
      tma_prefetch_desc(&tmA2);
      tma_prefetch_desc(&tmB2);
    }
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);
    }
    for (int i = 0; i < 2 * Cfg::SLOTS; ++i) mbar_init(&ebar[i], 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------ TMA producer ------------------------------
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      const uint64_t pol_a = l2_policy(epi.l2 & 3), pol_b = l2_policy((epi.l2 >> 2) & 3);
      int s = 0;
      uint32_t ph = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int m_blk, n_blk;
        tile_coords(t, num_m, num_n, epi.group_m, m_blk, n_blk, n_grouped);
        const int m0 = m_blk * GEMM_BM, n0 = n_blk * BN;
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* a_dst = smem + s * Cfg::STAGE_BYTES;
          uint8_t* b_dst = a_dst + Cfg::A_BYTES;
          mbar_arrive_expect_tx(&full[s], Cfg::STAGE_BYTES);
          if (kb < num_k1) {
            tma_load_2d_hint(a_dst, &tmA, &full[s], kb * FP8_BK, m0, pol_a);
            tma_load_2d_hint(b_dst, &tmB, &full[s], kb * FP8_BK, n0, pol_b);
          } else {
            const int kB = (kb - num_k1) * GEMM_BK;
            const int kA = kB + (src2.n_sub > 0 ? (n0 / src2.n_sub) * src2.r : 0);
            tma_load_2d_hint(a_dst, &tmA2, &full[s], kA, m0, pol_a);
            if (B2_MN) {
#pragma unroll
              for (int a = 0; a < BN / 64; ++a)
                tma_load_2d_hint(b_dst + a * ATOM_BYTES, &tmB2, &full[s], n0 + a * 64, kB, pol_b);
            } else {
              tma_load_2d_hint(b_dst, &tmB2, &full[s], kB, n0, pol_b);
            }
          }
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------ MMA, promotion + epilogue: 64 rows per warpgroup ------------------------------
    setmaxnreg_inc<232>();
    const int cw = wg - 1;
    const int g = lane >> 2;
    float acc[BN / 2], part[BN / 2];
    int s = 0;
    uint32_t ph = 0;             // bit 0: parity of the ring's `full` barriers; bits 1.. those of the staging slots
    const bool leader = (threadIdx.x & 127) == 0;
    StagedEpi se;
    se.slots = smem_u32(staging + cw * Cfg::WG_STAGING_BYTES);
    se.bar = smem_u32(ebar + cw * Cfg::SLOTS);
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      int m_blk, n_blk;
      tile_coords(t, num_m, num_n, epi.group_m, m_blk, n_blk, n_grouped);
      se.row0 = m_blk * GEMM_BM + cw * 64;
      se.n0 = n_blk * BN;
      if constexpr (EPI != EPI_PLAIN) {
        if (leader) staged_prefetch<EPI, BN, Cfg>(se, &tmR, M, N);
      }
      const int r0 = se.row0 + (warp & 3) * 16 + g, r1 = r0 + 8;   // this thread's two accumulator rows
      const float* sa0 = sc.sa + r0;
      const float* sb = sc.sb + (long long)n_blk * sc.sb_n;
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < num_k; ++kb) {
        const bool fp8 = kb < num_k1;
        // scales first: the loads are in flight while the stage's MMAs run (rows past M have zero codes)
        float f0 = 0.f, f1 = 0.f;
        if (fp8) {
          const float b = __ldg(sb + (long long)kb * sc.sb_k);
          const long long o = (long long)kb * sc.ld_sa;
          f0 = r0 < M ? __ldg(sa0 + o) * b : 0.f;
          f1 = r1 < M ? __ldg(sa0 + o + 8) * b : 0.f;
        }
        mbar_wait(&full[s], ph & 1);
        const uint32_t a_addr = smem_u32(smem + s * Cfg::STAGE_BYTES) + cw * ATOM_BYTES;
        const uint32_t b_addr = smem_u32(smem + s * Cfg::STAGE_BYTES + Cfg::A_BYTES);
        if (fp8) {
          reg_fence(part);
          wgmma_fence();
#pragma unroll
          for (int k32 = 0; k32 < FP8_BK / 32; ++k32)
            wgmma_m64n128k32_e4m3(part, desc_kmajor(a_addr, k32), desc_kmajor(b_addr, k32), k32 > 0);
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(part);
          if (lane == 0) mbar_arrive(&empty[s]);
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] = fmaf(part[i], (i & 2) ? f1 : f0, acc[i]);
        } else {
          reg_fence(acc);
          wgmma_fence();
          gemm_mma_stage<false, B2_MN, BN>(acc, a_addr, b_addr, 0);
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(acc);
          if (lane == 0) mbar_arrive(&empty[s]);
        }
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      epilogue_staged<EPI, BN, Cfg>(acc, se, ph, &tmC, &tmR, M, N, leader, 1 + cw);
    }
    if (leader) tma_store_wait_all<0>();   // the slots must outlive the bulk stores that read them
  }
}

struct GemmLaunch {
  CUtensorMap tmA, tmB, tmA2, tmB2, tmC, tmR;
  int M, N, K;
  GemmSecondSource src2;
  GemmEpilogue epi;
  cudaStream_t stream;
};

// CTA slots of the persistent grid: the clusters of CL CTAs (each ~193 KB of shared memory, one per SM) that can be
// resident at once, asked once per kernel. num_sms() / CL would overstate it when a GPC's free SMs cannot all be
// paired, and every cluster of the grid beyond the resident ones would start its whole tile range only after another
// cluster had finished its own.
template <typename Kern>
static int resident_clusters(Kern kern, int CL, int smem_bytes) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(num_sms() / CL * CL);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = smem_bytes;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, (const void*)kern, &cfg) != cudaSuccess || n <= 0) {
    cudaGetLastError();
    n = num_sms() / CL;
  }
  return n < num_sms() / CL ? n : num_sms() / CL;
}

template <bool A_MN, bool B_MN, int BN, int CL, int EPI, bool STAGED>
static int launch_gemm(const GemmLaunch& L) {
  using Cfg = GemmCfg<BN, EPI, STAGED>;
  auto kern = gemm_bf16_kernel<A_MN, B_MN, BN, CL, EPI, STAGED>;
  B200_CHECK_CUDA(configure_smem_once((const void*)kern, (int)Cfg::SMEM_BYTES));
  static int slots_per_device[64] = {};
  int dev = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  int& slots = slots_per_device[dev & 63];
  if (slots == 0) slots = resident_clusters(kern, CL, (int)Cfg::SMEM_BYTES);
  const int num_tiles = ((L.M + CL * GEMM_BM - 1) / (CL * GEMM_BM)) * ((L.N + BN - 1) / BN);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((num_tiles < slots ? num_tiles : slots) * CL);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
  cfg.stream = L.stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  B200_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, L.tmA, L.tmB, L.tmA2, L.tmB2, L.tmC, L.tmR, L.M, L.N, L.K, L.src2,
                                     L.epi));
  return 0;
}

template <bool A_MN, bool B_MN, int EPI, bool STAGED>
static int launch_tile(int bn, const GemmLaunch& L) {
  return bn == 512 ? launch_gemm<A_MN, B_MN, 256, 2, EPI, STAGED>(L)
       : bn == 256 ? launch_gemm<A_MN, B_MN, 256, 1, EPI, STAGED>(L)
                   : launch_gemm<A_MN, B_MN, 128, 1, EPI, STAGED>(L);
}

// wgrad (A MN-major) launches have no residual or SwiGLU form: plain or general only. The general form has no staged
// kernel; the other forms have both, the register epilogue kept for the launches the staged one cannot take (gemm_impl).
template <bool A_MN, bool B_MN>
static int launch_epi(int kind, bool staged, int bn, const GemmLaunch& L) {
  if (kind == EPI_PLAIN)
    return staged ? launch_tile<A_MN, B_MN, EPI_PLAIN, true>(bn, L) : launch_tile<A_MN, B_MN, EPI_PLAIN, false>(bn, L);
  if constexpr (!A_MN) {
    if (kind == EPI_RESIDUAL)
      return staged ? launch_tile<A_MN, B_MN, EPI_RESIDUAL, true>(bn, L)
                    : launch_tile<A_MN, B_MN, EPI_RESIDUAL, false>(bn, L);
    if (kind == EPI_GLU)
      return staged ? launch_tile<A_MN, B_MN, EPI_GLU, true>(bn, L) : launch_tile<A_MN, B_MN, EPI_GLU, false>(bn, L);
  }
  return launch_tile<A_MN, B_MN, EPI_GENERAL, false>(bn, L);
}

// Build the tensor map of one operand. K-major: tensor [rows][kdim] (ld elements per row),
// box {64, box_rows}. MN-major: tensor [kdim][rows] (ld per k-row), box {64, 64}.
static int operand_tmap(CUtensorMap* tm, const void* ptr, long long ld, bool mn_major, int rows,
                        int kdim, int box_rows) {
  if (!mn_major) {
    uint64_t dims[2] = {(uint64_t)kdim, (uint64_t)rows};
    uint64_t str[1] = {(uint64_t)ld * 2};
    uint32_t box[2] = {64, (uint32_t)box_rows};
    return make_tmap_bf16(tm, ptr, 2, dims, str, box);
  } else {
    uint64_t dims[2] = {(uint64_t)rows, (uint64_t)kdim};
    uint64_t str[1] = {(uint64_t)ld * 2};
    uint32_t box[2] = {64, 64};
    return make_tmap_bf16(tm, ptr, 2, dims, str, box);
  }
}

}  // namespace b200

using namespace b200;

#ifdef RLAIFV_GEMM_STALLS
// Stall-accounting build only (not in include/rlaifv_b200.h): copy out / zero the GemmStall sums.
extern "C" int rlaifv_gemm_stalls_read(unsigned long long* host, int reset) {
  B200_CHECK_CUDA(cudaDeviceSynchronize());
  B200_CHECK_CUDA(cudaMemcpyFromSymbol(host, g_gemm_stalls, sizeof(unsigned long long) * ST_FIELDS));
  if (reset) {
    const unsigned long long zero[ST_FIELDS] = {};
    B200_CHECK_CUDA(cudaMemcpyToSymbol(g_gemm_stalls, zero, sizeof(zero)));
  }
  return ST_FIELDS;
}
#endif

static int g_group_m = 16;
static int g_debug = 0;     // bit 0: GemmEpilogue::debug; bit 1: register epilogue for every form (gemm_impl)
extern "C" int rlaifv_gemm_set_tuning(int group_m, int debug) {
  if (group_m > 0) g_group_m = group_m;
  g_debug = debug & 3;
  return 0;
}
// L2 policy of the operand loads and the tile raster (GemmEpilogue::l2; bits 4-5, the C-store hint, are accepted and
// ignored: C leaves through plain TMA stores or ordinary stores). l2 < 0 (default): chosen per launch by l2_auto_policy() below; l2 >= 0:
// the given bits for every launch.
static int g_l2 = -1;
extern "C" int rlaifv_gemm_set_l2(int l2) {
  g_l2 = l2 < 0 ? -1 : (l2 & 0x7f);
  return 0;
}
// Long-K launches (dgrad / wgrad / down projection: K = 11008 .. 22016) have operand panels of several MB per tile
// row or column; with the default raster (16 row blocks per group) the panels one wave of CTAs touches can fall out of
// the L2 before the next wave needs them again, and the launch then reads its operands from DRAM several times over.
// Grouping along the SHORTER tile dimension keeps the smaller operand's panels resident while the larger one streams:
// DRAM reads = (streamed operand) x ceil(blocks / group) + (resident operand), and the resident set (group x panel)
// has to stay well under the L2: 8 panels up to K = 16384, 4 beyond. The resident operand's TMA loads carry
// evict_last, the streamed one's evict_first. Tile order and cache hints never change a bit of the result.
static void l2_auto_policy(int M, int N, int K, int* l2, int* group) {
  if (K < 8192) return;                                    // short K: panels are small, the default raster is the best
  const bool n_grouped = N < M;
  *group = K <= 16384 ? 8 : 4;
  *l2 = n_grouped ? (0x40 | 1 | (2 << 2))                  // column blocks grouped: B resident, A streams
                  : (2 | (1 << 2));                        // row blocks grouped: A resident, B streams
}
// C ABI — see include/rlaifv_b200.h for the contract.
// EXPERIMENTAL, off by default (rlaifv_gemm_set_split_k): long-K launches without bias / activation / residual
// (dgrad, wgrad) run as `n` passes over K slices, passes 2.. with C += — each pass's operand slabs then fit the L2
// (tools/l2_raster_model.py: dgrad 2.4 -> ~0.9 GB DRAM reads at n = 2). One extra bf16 rounding per pass boundary.
static int g_split_k = 0;
static int g_split_k_min_k = 8192;
extern "C" int rlaifv_gemm_set_split_k(int n, int min_k) {
  g_split_k = n > 1 ? n : 0;
  if (min_k > 0) g_split_k_min_k = min_k;
  return 0;
}

static int gemm_impl(const void* A, long long lda, int a_mn_major, const void* B, long long ldb, int b_mn_major,
                     void* C, long long ldc, int M, int N, int K, const void* bias, const void* residual,
                     long long ldr, int act, int accumulate, int tile_n, float alpha, void* stream,
                     const void* A2 = nullptr, long long lda2 = 0, const void* B2 = nullptr, long long ldb2 = 0,
                     int K2 = 0, int r2 = 0, int n_sub = 0, const void* glu = nullptr, long long ld_glu = 0) {
  B200_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
  if (glu) {
    // the SwiGLU-backward epilogue is instantiated for K-major A only (launch_epi)
    B200_REQUIRE(!a_mn_major, "gemm (swiglu_bwd epilogue): A must be K-major");
    B200_REQUIRE(!bias && !residual && act == 0 && !accumulate && alpha == 1.0f,
                 "gemm (swiglu_bwd epilogue): no bias / residual / activation / accumulate / alpha");
    B200_REQUIRE(N % 64 == 0 && ld_glu % 8 == 0 && ld_glu >= 2LL * N && ldc >= 2LL * N,
                 "gemm (swiglu_bwd epilogue): F = %d must be a multiple of 64, gate|up rows at least 2F wide", N);
    B200_REQUIRE(((uintptr_t)glu & 15) == 0, "gemm (swiglu_bwd epilogue): gate|up not 16-byte aligned");
  }
  if (g_split_k > 1 && K2 == 0 && !bias && !residual && act == 0 && !glu && K >= g_split_k_min_k) {
    const int n = g_split_k;
    const int ks = ((K + n - 1) / n + GEMM_BK - 1) / GEMM_BK * GEMM_BK;   // slice = whole 64-wide k blocks
    g_split_k = 0;                                   // the passes themselves are ordinary launches
    int rc = 0;
    for (int s = 0; s * ks < K && rc == 0; ++s) {
      const int klen = K - s * ks < ks ? K - s * ks : ks;                 // the last slice takes the ragged tail
      const bf16* As = (const bf16*)A + (a_mn_major ? (long long)s * ks * lda : (long long)s * ks);
      const bf16* Bs = (const bf16*)B + (b_mn_major ? (long long)s * ks * ldb : (long long)s * ks);
      rc = gemm_impl(As, lda, a_mn_major, Bs, ldb, b_mn_major, C, ldc, M, N, klen, nullptr, nullptr, 0, 0,
                     s == 0 ? accumulate : 1, tile_n, alpha, stream);
    }
    g_split_k = n;
    return rc;
  }
  B200_REQUIRE(N % 8 == 0 && ldc % 8 == 0, "gemm: N (%d) and ldc (%lld) must be multiples of 8", N,
               ldc);
  B200_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "gemm: lda/ldb must be multiples of 8");
  B200_REQUIRE(!(a_mn_major && !b_mn_major), "gemm: A MN-major with B K-major is not instantiated");
  B200_REQUIRE(((uintptr_t)C & 15) == 0, "gemm: C not 16-byte aligned");
  // epilogue_pair reads bias and residual as bf16 pairs (32-bit loads at even columns)
  B200_REQUIRE(!bias || ((uintptr_t)bias & 3) == 0, "gemm: bias not 4-byte aligned");
  B200_REQUIRE(!residual || (ldr % 2 == 0 && ((uintptr_t)residual & 3) == 0),
               "gemm: residual must be 4-byte aligned with an even row stride (ldr %lld)", ldr);
  int bn = tile_n;
  if (bn == 0) {
    // the 128 x 256 tile halves the B-operand shared-memory traffic per output element of the 128 x 128 one, and the
    // CTA-pair form halves B's L2 reads again; each is taken once there are enough of its tiles to fill the SMs. Measured
    // on an H100 SXM (700 W) on the LLaVA-7B layer shapes at M = 9080: the pair is 1-3 % faster than the single-CTA
    // 128 x 256 tile on every forward, dgrad and wgrad shape, with bit-identical results.
    const long long tiles256 = (long long)((M + 127) / 128) * ((N + 255) / 256);
    const long long tiles2 = (long long)((M + 255) / 256) * ((N + 255) / 256);
    if (N >= 256 && tiles2 >= num_sms() / 2) bn = 512;
    else bn = (N >= 256 && tiles256 >= num_sms()) ? 256 : 128;
  }
  B200_REQUIRE(bn == 128 || bn == 256 || bn == 512, "gemm: tile_n must be 0, 128, 256 or 512 (2-CTA 256x256)");
  GemmSecondSource src2;
  src2.K2 = K2;
  src2.r = r2;
  src2.n_sub = n_sub;
  if (K2 > 0) {
    B200_REQUIRE(lda2 % 8 == 0 && ldb2 % 8 == 0, "gemm: lda2/ldb2 must be multiples of 8");
    const int ntile = bn == 512 ? 256 : bn;
    B200_REQUIRE(n_sub == 0 || n_sub % ntile == 0, "gemm: n_sub (%d) must be a multiple of the N tile (%d)", n_sub,
                 ntile);
  }
  CUtensorMap tmA, tmB;
  int rc = operand_tmap(&tmA, A, lda, a_mn_major != 0, M, K, GEMM_BM);
  if (rc) return rc;
  rc = operand_tmap(&tmB, B, ldb, b_mn_major != 0, N, K, bn == 512 ? 128 : bn);
  if (rc) return rc;
  CUtensorMap tmA2 = tmA, tmB2 = tmB;
  if (K2 > 0) {
    // A2 spans all sub-linears' column blocks: its contraction extent is (N / n_sub) * r (forward) or K2 (dgrad)
    const int a2_k = n_sub > 0 ? (N / n_sub) * r2 : K2;
    rc = operand_tmap(&tmA2, A2, lda2, a_mn_major != 0, M, a2_k, GEMM_BM);
    if (rc) return rc;
    rc = operand_tmap(&tmB2, B2, ldb2, b_mn_major != 0, N, K2, bn == 512 ? 128 : bn);
    if (rc) return rc;
  }
  GemmLaunch L;
  L.tmA = tmA;
  L.tmB = tmB;
  L.tmA2 = tmA2;
  L.tmB2 = tmB2;
  const bool plain = !bias && act == 0 && !accumulate && alpha == 1.0f;
  const int kind = glu ? EPI_GLU : !plain ? EPI_GENERAL : residual ? EPI_RESIDUAL : EPI_PLAIN;
  // The staged epilogue moves C, the residual and gate|up in 64 x 64 TMA boxes: a residual needs the 16-byte alignment
  // of a tensor map (C and gate|up are required to have it above).
  const bool staged = kind != EPI_GENERAL && !(g_debug & 2) &&
                      (kind != EPI_RESIDUAL || (((uintptr_t)residual & 15) == 0 && ldr % 8 == 0));
  if (staged) {
    // {columns, rows} with the real row strides: TMA clips every box at N (2F) and M
    const uint32_t box[2] = {64, 64};
    const uint64_t c_dims[2] = {(uint64_t)(glu ? 2LL * N : N), (uint64_t)M}, c_str[1] = {(uint64_t)ldc * 2};
    rc = make_tmap_bf16(&L.tmC, C, 2, c_dims, c_str, box);
    if (rc) return rc;
    L.tmR = L.tmC;
    if (kind != EPI_PLAIN) {
      const uint64_t r_dims[2] = {(uint64_t)(glu ? 2LL * N : N), (uint64_t)M};
      const uint64_t r_str[1] = {(uint64_t)(glu ? ld_glu : ldr) * 2};
      rc = make_tmap_bf16(&L.tmR, glu ? glu : residual, 2, r_dims, r_str, box);
      if (rc) return rc;
    }
  } else {
    L.tmC = L.tmR = tmA;     // not read by the register epilogue
  }
  L.M = M;
  L.N = N;
  L.K = K;
  L.src2 = src2;
  GemmEpilogue& epi = L.epi;
  epi.C = (bf16*)C;
  epi.ldc = ldc;
  epi.bias = (const bf16*)bias;
  epi.residual = (const bf16*)residual;
  epi.ldr = ldr;
  epi.act = act;
  epi.accumulate = accumulate;
  epi.alpha = alpha;
  epi.glu = (const bf16*)glu;
  epi.ld_glu = ld_glu;
  epi.group_m = g_group_m;
  epi.debug = g_debug;
  epi.l2 = 0;
  if (g_l2 < 0) l2_auto_policy(M, N, K, &epi.l2, &epi.group_m);
  else epi.l2 = g_l2 & 0x4f;
  L.stream = (cudaStream_t)stream;
  if (!a_mn_major && !b_mn_major) return launch_epi<false, false>(kind, staged, bn, L);
  if (!a_mn_major && b_mn_major) return launch_epi<false, true>(kind, staged, bn, L);
  return launch_epi<true, true>(kind, staged, bn, L);
}

extern "C" int rlaifv_gemm_max_active_clusters(int tile_n, int* clusters) {
  B200_REQUIRE(tile_n == 128 || tile_n == 256 || tile_n == 512, "gemm: tile_n must be 128, 256 or 512");
  B200_REQUIRE(clusters, "gemm_max_active_clusters: null output");
  const int cl = tile_n == 512 ? 2 : 1, bn = tile_n == 512 ? 256 : tile_n;
  // the staged plain kernel: the most shared memory any launch of this tile asks for
  const int smem = bn == 256 ? (int)GemmCfg<256, EPI_PLAIN, true>::SMEM_BYTES
                             : (int)GemmCfg<128, EPI_PLAIN, true>::SMEM_BYTES;
  if (tile_n == 512) {
    auto k = gemm_bf16_kernel<false, false, 256, 2, EPI_PLAIN, true>;
    B200_CHECK_CUDA(configure_smem_once((const void*)k, smem));
    *clusters = resident_clusters(k, cl, smem);
  } else if (bn == 256) {
    auto k = gemm_bf16_kernel<false, false, 256, 1, EPI_PLAIN, true>;
    B200_CHECK_CUDA(configure_smem_once((const void*)k, smem));
    *clusters = resident_clusters(k, cl, smem);
  } else {
    auto k = gemm_bf16_kernel<false, false, 128, 1, EPI_PLAIN, true>;
    B200_CHECK_CUDA(configure_smem_once((const void*)k, smem));
    *clusters = resident_clusters(k, cl, smem);
  }
  return 0;
}

extern "C" int rlaifv_gemm_bf16(const void* A, long long lda, int a_mn_major, const void* B, long long ldb,
                                int b_mn_major, void* C, long long ldc, int M, int N, int K, const void* bias,
                                const void* residual, long long ldr, int act, int accumulate, int tile_n,
                                void* stream) {
  return gemm_impl(A, lda, a_mn_major, B, ldb, b_mn_major, C, ldc, M, N, K, bias, residual, ldr, act, accumulate,
                   tile_n, 1.0f, stream);
}
// Same with the product scaled first: C (+)= bf16(bf16(A*B) * alpha) ... (LoRA: alpha = lora_alpha / r).
extern "C" int rlaifv_gemm_bf16_scaled(const void* A, long long lda, int a_mn_major, const void* B, long long ldb,
                                       int b_mn_major, void* C, long long ldc, int M, int N, int K,
                                       const void* bias, const void* residual, long long ldr, int act,
                                       int accumulate, int tile_n, float alpha, void* stream) {
  return gemm_impl(A, lda, a_mn_major, B, ldb, b_mn_major, C, ldc, M, N, K, bias, residual, ldr, act, accumulate,
                   tile_n, alpha, stream);
}

// C (+)= A*B^T + A2[:, koff:koff+K2] * B2^T (shared fp32 accumulator, one rounding), then bias/act/residual.
// koff = (n0 / n_sub) * r when n_sub > 0 (forward over fused sub-linears), else 0. Same operand majors as A/B.
// d[gate | up] = swiglu_bwd([gate | up], dy @ op(W)^T) in one launch — see epilogue_tile_glu. Optional second operand
// pair (K2 > 0) as in rlaifv_gemm_bf16_dual (LoRA: d(act) = dy W + (s dy B) A).
extern "C" int rlaifv_gemm_bf16_swiglu_bwd(const void* A, long long lda, const void* B, long long ldb, int b_mn_major,
                                           const void* A2, long long lda2, const void* B2, long long ldb2, int K2,
                                           const void* gu, long long ld_gu, void* dgu, long long ld_dgu, int M, int F,
                                           int K, void* stream) {
  B200_REQUIRE(gu && dgu, "gemm_swiglu_bwd: gate|up / output missing");
  return gemm_impl(A, lda, 0, B, ldb, b_mn_major, dgu, ld_dgu, M, F, K, nullptr, nullptr, 0, 0, 0, 0, 1.0f, stream, A2,
                   lda2, B2, ldb2, K2, K2, 0, gu, ld_gu);
}
extern "C" int rlaifv_gemm_bf16_dual(const void* A, long long lda, int a_mn_major, const void* B, long long ldb,
                                     int b_mn_major, const void* A2, long long lda2, const void* B2, long long ldb2,
                                     int K2, int r, int n_sub, void* C, long long ldc, int M, int N, int K,
                                     const void* bias, const void* residual, long long ldr, int act, int accumulate,
                                     void* stream) {
  B200_REQUIRE(K2 > 0 && A2 && B2, "gemm_dual: second source missing");
  return gemm_impl(A, lda, a_mn_major, B, ldb, b_mn_major, C, ldc, M, N, K, bias, residual, ldr, act, accumulate, 0,
                   1.0f, stream, A2, lda2, B2, ldb2, K2, r, n_sub);
}

template <int EPI, bool B2_MN>
static int launch_fp8(const GemmLaunch& L, const Fp8Scales& sc) {
  using Cfg = GemmCfg<128, EPI, true>;
  auto kern = gemm_fp8_kernel<EPI, B2_MN>;
  B200_CHECK_CUDA(configure_smem_once((const void*)kern, (int)Cfg::SMEM_BYTES));
  static int slots_per_device[64] = {};
  int dev = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  int& slots = slots_per_device[dev & 63];
  if (slots == 0) slots = resident_clusters(kern, 1, (int)Cfg::SMEM_BYTES);
  const int num_tiles = ((L.M + GEMM_BM - 1) / GEMM_BM) * (L.N / 128);
  kern<<<num_tiles < slots ? num_tiles : slots, GEMM_THREADS, Cfg::SMEM_BYTES, L.stream>>>(
      L.tmA, L.tmB, L.tmA2, L.tmB2, L.tmC, L.tmR, L.M, L.N, L.K, L.src2, sc, L.epi);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int rlaifv_gemm_fp8(const void* A, long long lda, const float* sa, long long ld_sa, const void* B,
                               long long ldb, const float* sb, int b_t, const void* A2, long long lda2, const void* B2,
                               long long ldb2, int K2, int r, int n_sub, void* C, long long ldc, int M, int N, int K,
                               const void* residual, long long ldr, const void* glu, long long ld_glu, void* stream) {
  B200_REQUIRE(A && B && sa && sb && C, "gemm_fp8: null operand");
  B200_REQUIRE(M > 0 && N > 0 && K > 0, "gemm_fp8: empty problem M=%d N=%d K=%d", M, N, K);
  B200_REQUIRE(N % 128 == 0 && K % 128 == 0, "gemm_fp8: N (%d) and K (%d) must be multiples of 128", N, K);
  B200_REQUIRE(lda >= K && ldb >= K && lda % 16 == 0 && ldb % 16 == 0,
               "gemm_fp8: code row strides (lda %lld, ldb %lld) must cover K and be multiples of 16 bytes", lda, ldb);
  B200_REQUIRE(ld_sa >= M && ld_sa % 4 == 0, "gemm_fp8: ld_sa (%lld) must be >= M (%d) and a multiple of 4", ld_sa, M);
  B200_REQUIRE(((uintptr_t)sa & 15) == 0 && ((uintptr_t)sb & 3) == 0, "gemm_fp8: scales misaligned");
  B200_REQUIRE(ldc % 8 == 0 && ((uintptr_t)C & 15) == 0, "gemm_fp8: C must be 16-byte aligned, ldc a multiple of 8");
  B200_REQUIRE(!(glu && residual), "gemm_fp8: a residual and a SwiGLU-backward epilogue together");
  if (residual)
    B200_REQUIRE(((uintptr_t)residual & 15) == 0 && ldr % 8 == 0 && ldr >= N,
                 "gemm_fp8: residual must be 16-byte aligned with a row stride (%lld) >= N, multiple of 8", ldr);
  if (glu)
    B200_REQUIRE(((uintptr_t)glu & 15) == 0 && ld_glu % 8 == 0 && ld_glu >= 2LL * N && ldc >= 2LL * N,
                 "gemm_fp8 (swiglu_bwd epilogue): gate|up 16-byte aligned, rows of gate|up and C at least 2F wide");
  else
    B200_REQUIRE(ldc >= N, "gemm_fp8: ldc (%lld) < N (%d)", ldc, N);
  GemmLaunch L;
  const uint32_t box8[2] = {FP8_BK, GEMM_BM};
  const uint64_t a_dims[2] = {(uint64_t)K, (uint64_t)M}, a_str[1] = {(uint64_t)lda};
  int rc = make_tmap_u8(&L.tmA, A, 2, a_dims, a_str, box8);
  if (rc) return rc;
  const uint64_t b_dims[2] = {(uint64_t)K, (uint64_t)N}, b_str[1] = {(uint64_t)ldb};
  rc = make_tmap_u8(&L.tmB, B, 2, b_dims, b_str, box8);
  if (rc) return rc;
  L.tmA2 = L.tmA;
  L.tmB2 = L.tmB;
  if (K2 > 0) {
    B200_REQUIRE(A2 && B2, "gemm_fp8: second source missing");
    B200_REQUIRE(lda2 % 8 == 0 && ldb2 % 8 == 0, "gemm_fp8: lda2/ldb2 must be multiples of 8");
    B200_REQUIRE(n_sub == 0 || (n_sub % 128 == 0 && r > 0 && N % n_sub == 0),
                 "gemm_fp8: n_sub (%d) must divide N and be a multiple of the 128-column tile", n_sub);
    rc = operand_tmap(&L.tmA2, A2, lda2, false, M, n_sub > 0 ? (N / n_sub) * r : K2, GEMM_BM);
    if (rc) return rc;
    rc = operand_tmap(&L.tmB2, B2, ldb2, b_t != 0, N, K2, 128);
    if (rc) return rc;
  }
  const uint32_t box[2] = {64, 64};
  const uint64_t c_dims[2] = {(uint64_t)(glu ? 2LL * N : N), (uint64_t)M}, c_str[1] = {(uint64_t)ldc * 2};
  rc = make_tmap_bf16(&L.tmC, C, 2, c_dims, c_str, box);
  if (rc) return rc;
  L.tmR = L.tmC;
  if (glu || residual) {
    const uint64_t r_str[1] = {(uint64_t)(glu ? ld_glu : ldr) * 2};
    rc = make_tmap_bf16(&L.tmR, glu ? glu : residual, 2, c_dims, r_str, box);
    if (rc) return rc;
  }
  L.M = M;
  L.N = N;
  L.K = K;
  L.src2.K2 = K2 > 0 ? K2 : 0;
  L.src2.r = r;
  L.src2.n_sub = n_sub;
  L.epi = GemmEpilogue{};
  L.epi.alpha = 1.0f;
  L.epi.group_m = g_group_m;
  if (g_l2 < 0) l2_auto_policy(M, N, K, &L.epi.l2, &L.epi.group_m);
  else L.epi.l2 = g_l2 & 0x4f;
  L.stream = (cudaStream_t)stream;
  Fp8Scales sc;
  sc.sa = sa;
  sc.ld_sa = ld_sa;
  sc.sb = sb;
  // block scales of W [N_w, K_w] are [N_w / 128][K_w / 128]; b_t: B is W^T, its output block indexes K_w
  sc.sb_n = b_t ? 1 : K / 128;
  sc.sb_k = b_t ? N / 128 : 1;
  const int kind = glu ? EPI_GLU : residual ? EPI_RESIDUAL : EPI_PLAIN;
  if (b_t) {
    if (kind == EPI_GLU) return launch_fp8<EPI_GLU, true>(L, sc);
    if (kind == EPI_RESIDUAL) return launch_fp8<EPI_RESIDUAL, true>(L, sc);
    return launch_fp8<EPI_PLAIN, true>(L, sc);
  }
  if (kind == EPI_GLU) return launch_fp8<EPI_GLU, false>(L, sc);
  if (kind == EPI_RESIDUAL) return launch_fp8<EPI_RESIDUAL, false>(L, sc);
  return launch_fp8<EPI_PLAIN, false>(L, sc);
}

// HBM-bound row kernels of the DPO step: RMSNorm / LayerNorm, RoPE, SwiGLU, CLIP patch im2col +
// embedding assembly, image-token splice (index map + row gather/scatter), per-token log-prob
// gather with its backward, DPO loss + gradient, fused AdamW (on-device, and streamed through a
// staging ring from pinned host memory).
// All use 128-bit global accesses and warp-shuffle reductions; bf16 storage, fp32 math, with the
// intermediate bf16 roundings of the HF eager path reproduced where they are observable.
#include "common.cuh"
#include "host_util.h"

#include <map>
#include <mutex>
#include <utility>

namespace b200 {

__device__ __forceinline__ void load8(const bf16* p, float (&v)[8]) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), c = unpack_bf16(u.z), d = unpack_bf16(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
__device__ __forceinline__ void store8(bf16* p, const float (&v)[8]) {
  uint4 u;
  u.x = pack_bf16(v[0], v[1]);
  u.y = pack_bf16(v[2], v[3]);
  u.z = pack_bf16(v[4], v[5]);
  u.w = pack_bf16(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// block-wide sum of up to 2 values; blockDim.x multiple of 32, <= 1024
__device__ __forceinline__ float2 block_sum2(float a, float b) {
  __shared__ float sa[32], sb[32];
  a = warp_sum(a);
  b = warp_sum(b);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();  // protect reuse across calls
  if (l == 0) { sa[w] = a; sb[w] = b; }
  __syncthreads();
  float x = (l < nw) ? sa[l] : 0.f, y = (l < nw) ? sb[l] : 0.f;
  x = warp_sum(x);
  y = warp_sum(y);
  return make_float2(x, y);
}

// ------------------------------------------------------------------------------------------------
// RMSNorm forward: y = bf16(w * bf16(x * rsqrt(mean(x^2)+eps)))    (HF: llama/modeling_llama.py:62-67)
// ------------------------------------------------------------------------------------------------
constexpr int NORM_THREADS = 256;
constexpr int NORM_MAXCH = 2;  // register-cached 8-element chunks per thread (H <= 4096)

__global__ void __launch_bounds__(NORM_THREADS)
rmsnorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, bf16* __restrict__ y,
                   float* __restrict__ rstd_out, int M, int H, float eps) {
  const int nch = H >> 3;
  for (long long row = blockIdx.x; row < M; row += gridDim.x) {
    const bf16* xr = x + row * H;
    float cache[NORM_MAXCH][8];
    float ss = 0.f;
#pragma unroll
    for (int ci = 0; ci < NORM_MAXCH; ++ci) {
      const int c = threadIdx.x + ci * NORM_THREADS;
      if (c < nch) {
        load8(xr + c * 8, cache[ci]);
#pragma unroll
        for (int j = 0; j < 8; ++j) ss += cache[ci][j] * cache[ci][j];
      }
    }
    for (int c = threadIdx.x + NORM_MAXCH * NORM_THREADS; c < nch; c += NORM_THREADS) {
      float v[8];
      load8(xr + c * 8, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) ss += v[j] * v[j];
    }
    const float tot = block_sum2(ss, 0.f).x;
    const float rstd = rsqrtf(tot / (float)H + eps);
    if (rstd_out && threadIdx.x == 0) rstd_out[row] = rstd;
    bf16* yr = y + row * H;
#pragma unroll
    for (int ci = 0; ci < NORM_MAXCH; ++ci) {
      const int c = threadIdx.x + ci * NORM_THREADS;
      if (c < nch) {
        float wv[8], o[8];
        load8(w + c * 8, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = wv[j] * bf16_round(cache[ci][j] * rstd);
        store8(yr + c * 8, o);
      }
    }
    for (int c = threadIdx.x + NORM_MAXCH * NORM_THREADS; c < nch; c += NORM_THREADS) {
      float v[8], wv[8];
      load8(xr + c * 8, v);
      load8(w + c * 8, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = wv[j] * bf16_round(v[j] * rstd);
      store8(yr + c * 8, v);
    }
  }
}

// RMSNorm backward. xhat = x*rstd, g = w*dy:
//   dx = rstd * (g - xhat * mean(g*xhat))  (+ dres if given);  dw[h] += sum_rows dy*xhat
// dw is accumulated per CTA in registers over its rows and written to dw_partial[grid][H] (fp32).
// NCH 8-element chunks per thread are register-cached, so H <= NORM_THREADS * 8 * NCH.
template <int NCH>
__global__ void __launch_bounds__(NORM_THREADS)
rmsnorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                   const bf16* __restrict__ w, const float* __restrict__ rstd_in,
                   const bf16* __restrict__ dres, bf16* __restrict__ dx,
                   float* __restrict__ dw_partial, int M, int H) {
  // Two rows per pass: both rows' loads are issued before the (single, two-value) block reduction, which doubles the
  // bytes in flight per CTA and halves the number of block-wide synchronisations (one row per pass ran at 45 % of the
  // copy peak: 2 CTAs/SM x 24 KB in flight, serialised by two __syncthreads per row).
  const int nch = H >> 3;
  float dwacc[NCH][8];
#pragma unroll
  for (int i = 0; i < NCH; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) dwacc[i][j] = 0.f;
  for (long long row0 = 2LL * blockIdx.x; row0 < M; row0 += 2LL * gridDim.x) {
    const bool two = row0 + 1 < M;
    const long long rows[2] = {row0, two ? row0 + 1 : row0};
    const float rstd[2] = {rstd_in[rows[0]], rstd_in[rows[1]]};
    float xh[2][NCH][8], g[2][NCH][8];
    float dot[2] = {0.f, 0.f};
#pragma unroll
    for (int ci = 0; ci < NCH; ++ci) {
      const int c = threadIdx.x + ci * NORM_THREADS;
      if (c >= nch) continue;
      float wv[8], xv[2][8], dv[2][8];
      load8(w + c * 8, wv);
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        load8(x + rows[u] * H + c * 8, xv[u]);
        load8(dy + rows[u] * H + c * 8, dv[u]);
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const float keep = (u == 0 || two) ? 1.f : 0.f;      // the duplicated tail row adds nothing to dw
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[u][ci][j] = xv[u][j] * rstd[u];
          g[u][ci][j] = wv[j] * dv[u][j];
          dot[u] += g[u][ci][j] * xh[u][ci][j];
          dwacc[ci][j] += keep * dv[u][j] * xh[u][ci][j];
        }
      }
    }
    const float2 tot = block_sum2(dot[0], dot[1]);
    const float mean[2] = {tot.x / (float)H, tot.y / (float)H};
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (u == 1 && !two) break;
#pragma unroll
      for (int ci = 0; ci < NCH; ++ci) {
        const int c = threadIdx.x + ci * NORM_THREADS;
        if (c >= nch) continue;
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd[u] * (g[u][ci][j] - xh[u][ci][j] * mean[u]);
        if (dres) {
          float rv[8];
          load8(dres + rows[u] * H + c * 8, rv);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += rv[j];
        }
        store8(dx + rows[u] * H + c * 8, o);
      }
    }
  }
#pragma unroll
  for (int ci = 0; ci < NCH; ++ci) {
    const int c = threadIdx.x + ci * NORM_THREADS;
    if (c >= nch) continue;
    float* dst = dw_partial + (long long)blockIdx.x * H + c * 8;
    *reinterpret_cast<float4*>(dst) = make_float4(dwacc[ci][0], dwacc[ci][1], dwacc[ci][2], dwacc[ci][3]);
    *reinterpret_cast<float4*>(dst + 4) = make_float4(dwacc[ci][4], dwacc[ci][5], dwacc[ci][6], dwacc[ci][7]);
  }
}

// dw[h] (bf16, accumulate or overwrite) from fp32 partials [P][H].
// Block = 32 columns x 8 row-lanes: coalesced 128-byte reads, rows strided by 8, smem tree at the end.
__global__ void __launch_bounds__(256)
reduce_partials_kernel(const float* __restrict__ part, int P, int H, bf16* __restrict__ dw, int accumulate) {
  __shared__ float sm[8][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int h = blockIdx.x * 32 + cx;
  float s = 0.f;
  if (h < H)
    for (int p = ry; p < P; p += 8) s += part[(long long)p * H + h];
  sm[ry][cx] = s;
  __syncthreads();
  if (ry == 0 && h < H) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[i][cx];
    if (accumulate) t += __bfloat162float(dw[h]);
    dw[h] = __float2bfloat16_rn(t);
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm forward (CLIP; HF clip/modeling_clip.py pre_layrnorm / layer_norm1/2): fp32 stats,
// y = bf16((x-mean)*rstd*w + b)
// ------------------------------------------------------------------------------------------------
// Mean and rstd of one register-cached row (H <= NORM_THREADS * 8 * NORM_MAXCH). One pass gives the mean and
// E[x^2] - mean^2. That difference cancels in fp32 when |mean| >> std (a row of 100.0 with 1 in 512 elements one bf16 ulp
// higher gave a variance of 0 and an rstd of eps^-1/2), so when mean^2 exceeds it the variance is taken again as the
// mean of (x - mean)^2 over the cached row. A one-pass variance that is at least mean^2 has lost at most a factor ~2 of
// the sum's rounding (E[x^2] <= 2 var), and rows of that kind get the same bits as the one-pass kernel always gave.
// The test is on block-reduced values, so the whole block takes the same branch.
__device__ __forceinline__ float2 layernorm_stats(const float (&xv)[NORM_MAXCH][8], int nch, int H, float eps) {
  float s = 0.f, ss = 0.f;
#pragma unroll
  for (int ci = 0; ci < NORM_MAXCH; ++ci)
    if (threadIdx.x + ci * NORM_THREADS < nch) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { s += xv[ci][j]; ss += xv[ci][j] * xv[ci][j]; }
    }
  const float2 tot = block_sum2(s, ss);
  const float mean = tot.x / (float)H;
  float var = fmaxf(tot.y / (float)H - mean * mean, 0.f);
  if (__fmul_rn(mean, mean) > var) {
    float dd = 0.f;
#pragma unroll
    for (int ci = 0; ci < NORM_MAXCH; ++ci)
      if (threadIdx.x + ci * NORM_THREADS < nch) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = xv[ci][j] - mean;
          dd += d * d;
        }
      }
    var = block_sum2(dd, 0.f).x / (float)H;
  }
  return make_float2(mean, rsqrtf(var + eps));
}

__global__ void __launch_bounds__(NORM_THREADS)
layernorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                     const bf16* __restrict__ b, bf16* __restrict__ y, int M, int H, float eps) {
  const int nch = H >> 3;
  for (long long row = blockIdx.x; row < M; row += gridDim.x) {
    const bf16* xr = x + row * H;
    float cache[NORM_MAXCH][8];
#pragma unroll
    for (int ci = 0; ci < NORM_MAXCH; ++ci) {
      const int c = threadIdx.x + ci * NORM_THREADS;
      if (c < nch) load8(xr + c * 8, cache[ci]);
    }
    const float2 st = layernorm_stats(cache, nch, H, eps);
    const float mean = st.x, rstd = st.y;
    bf16* yr = y + row * H;
#pragma unroll
    for (int ci = 0; ci < NORM_MAXCH; ++ci) {
      const int c = threadIdx.x + ci * NORM_THREADS;
      if (c < nch) {
        float wv[8], bv[8], o[8];
        load8(w + c * 8, wv);
        load8(b + c * 8, bv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (cache[ci][j] - mean) * rstd * wv[j] + bv[j];
        store8(yr + c * 8, o);
      }
    }
  }
}

// LayerNorm backward (trainable LayerNorms of the perceiver resampler, omnilmm/model/resampler.py:137-141).
// Statistics are recomputed from x (fp32). xhat = (x-mean)*rstd, g = w*dy:
//   dx = rstd * (g - mean(g) - xhat * mean(g*xhat));  dw[h] += sum_rows dy*xhat;  db[h] += sum_rows dy
// dw / db are accumulated per CTA in registers and written to partial[2][grid][H] (fp32).
__global__ void __launch_bounds__(NORM_THREADS)
layernorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x, const bf16* __restrict__ w,
                     bf16* __restrict__ dx, float* __restrict__ dw_partial, float* __restrict__ db_partial,
                     int M, int H, float eps) {
  const int nch = H >> 3;
  float dwacc[NORM_MAXCH][8], dbacc[NORM_MAXCH][8];
#pragma unroll
  for (int i = 0; i < NORM_MAXCH; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) { dwacc[i][j] = 0.f; dbacc[i][j] = 0.f; }
  for (long long row = blockIdx.x; row < M; row += gridDim.x) {
    const bf16* xr = x + row * H;
    const bf16* dyr = dy + row * H;
    float xv[NORM_MAXCH][8], g[NORM_MAXCH][8];
#pragma unroll
    for (int ci = 0; ci < NORM_MAXCH; ++ci) {
      const int c = threadIdx.x + ci * NORM_THREADS;
      if (c < nch) load8(xr + c * 8, xv[ci]);
    }
    const float2 st = layernorm_stats(xv, nch, H, eps);
    const float mean = st.x, rstd = st.y;
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int ci = 0; ci < NORM_MAXCH; ++ci) {
      const int c = threadIdx.x + ci * NORM_THREADS;
      if (c >= nch) continue;
      float dv[8], wv[8];
      load8(dyr + c * 8, dv);
      load8(w + c * 8, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        xv[ci][j] = (xv[ci][j] - mean) * rstd;     // xhat
        g[ci][j] = wv[j] * dv[j];
        sg += g[ci][j];
        sgx += g[ci][j] * xv[ci][j];
        dwacc[ci][j] += dv[j] * xv[ci][j];
        dbacc[ci][j] += dv[j];
      }
    }
    const float2 t2 = block_sum2(sg, sgx);
    const float mg = t2.x / (float)H, mgx = t2.y / (float)H;
#pragma unroll
    for (int ci = 0; ci < NORM_MAXCH; ++ci) {
      const int c = threadIdx.x + ci * NORM_THREADS;
      if (c >= nch) continue;
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = rstd * (g[ci][j] - mg - xv[ci][j] * mgx);
      store8(dx + row * H + c * 8, o);
    }
  }
#pragma unroll
  for (int ci = 0; ci < NORM_MAXCH; ++ci) {
    const int c = threadIdx.x + ci * NORM_THREADS;
    if (c >= nch) continue;
    float* dst = dw_partial + (long long)blockIdx.x * H + c * 8;
    *reinterpret_cast<float4*>(dst) = make_float4(dwacc[ci][0], dwacc[ci][1], dwacc[ci][2], dwacc[ci][3]);
    *reinterpret_cast<float4*>(dst + 4) = make_float4(dwacc[ci][4], dwacc[ci][5], dwacc[ci][6], dwacc[ci][7]);
    dst = db_partial + (long long)blockIdx.x * H + c * 8;
    *reinterpret_cast<float4*>(dst) = make_float4(dbacc[ci][0], dbacc[ci][1], dbacc[ci][2], dbacc[ci][3]);
    *reinterpret_cast<float4*>(dst + 4) = make_float4(dbacc[ci][4], dbacc[ci][5], dbacc[ci][6], dbacc[ci][7]);
  }
}

// y[r] = bf16(x[r] + t[r % P])  — the resampler's position-embedding adds (resampler.py:158-161): the table t
// ([P][H], frozen sin-cos embedding) is shared by every image of the batch. y may alias x: the EVA tower's cls
// gradient and the resampler's query gradient are accumulated in place (out = x), so x and y are not __restrict__.
__global__ void add_rows_bcast_kernel(const bf16* x, const bf16* __restrict__ t, bf16* y, long long M, int P, int H) {
  const int nch = H >> 3;
  const long long total = M * nch;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long row = idx / nch;
    const int c = (int)(idx % nch);
    float a[8], b[8];
    load8(x + row * H + c * 8, a);
    load8(t + (row % P) * (long long)H + c * 8, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    store8(y + row * H + c * 8, a);
  }
}

// ------------------------------------------------------------------------------------------------
// RoPE (HF llama/modeling_llama.py:124-168): cos/sin tables are bf16 [T][D];
// out = bf16(bf16(x*cos) + bf16(rotate_half(x)*sin)), applied in place to the q and k column blocks
// of the fused qkv buffer [M][3*nh*D]; token m has position m % T.
// ------------------------------------------------------------------------------------------------
__global__ void rope_fwd_kernel(bf16* __restrict__ qkv, const bf16* __restrict__ cosb,
                                const bf16* __restrict__ sinb, long long M, int T, int nrot, int D,
                                long long ld) {
  // one thread handles 8 consecutive i in [0, D/2) for one (row, rotated head); the nrot = n_heads + n_kv_heads
  // rotated heads (q block then k block) are contiguous in the fused qkv row
  const int half = D >> 1;
  const int per_head = half >> 3;
  const long long total = M * nrot * per_head;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(idx % per_head);
    long long r = idx / per_head;
    const int head = (int)(r % nrot);
    const long long row = r / nrot;
    const int pos = (int)(row % T);
    bf16* p = qkv + row * ld + (long long)head * D + c8 * 8;
    float x1[8], x2[8], c1[8], s1[8], c2[8], s2[8];
    load8(p, x1);
    load8(p + half, x2);
    load8(cosb + (long long)pos * D + c8 * 8, c1);
    load8(sinb + (long long)pos * D + c8 * 8, s1);
    load8(cosb + (long long)pos * D + half + c8 * 8, c2);
    load8(sinb + (long long)pos * D + half + c8 * 8, s2);
    float o1[8], o2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o1[j] = bf16_round(x1[j] * c1[j]) + bf16_round(-x2[j] * s1[j]);
      o2[j] = bf16_round(x2[j] * c2[j]) + bf16_round(x1[j] * s2[j]);
    }
    store8(p, o1);
    store8(p + half, o2);
  }
}

// RoPE backward + dQ fp32->bf16: dqkv[:, q block] = R^T(dq_f32), dqkv[:, k block] = R^T(dk in place).
//   dx1 = dy1*cos1 + dy2*sin2 ; dx2 = dy2*cos2 - dy1*sin1
__global__ void rope_bwd_kernel(bf16* __restrict__ dqkv, const float* __restrict__ dq_f32,
                                const bf16* __restrict__ cosb, const bf16* __restrict__ sinb,
                                long long M, int T, int nh, int nkv, int D, long long ld) {
  const int half = D >> 1;
  const int per_head = half >> 3;
  const int nrot = nh + nkv;
  const long long total = M * nrot * per_head;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(idx % per_head);
    long long r = idx / per_head;
    const int head = (int)(r % nrot);
    const long long row = r / nrot;
    const int pos = (int)(row % T);
    bf16* p = dqkv + row * ld + (long long)head * D + c8 * 8;
    float y1[8], y2[8], c1[8], s1[8], c2[8], s2[8];
    if (head < nh && dq_f32) {     // dq_f32 == nullptr: dQ already sits in the q block as bf16 (split backward)
      const float* q = dq_f32 + row * (long long)nh * D + head * D + c8 * 8;
      float4 a = *reinterpret_cast<const float4*>(q), b = *reinterpret_cast<const float4*>(q + 4);
      float4 c = *reinterpret_cast<const float4*>(q + half), d = *reinterpret_cast<const float4*>(q + half + 4);
      y1[0] = a.x; y1[1] = a.y; y1[2] = a.z; y1[3] = a.w; y1[4] = b.x; y1[5] = b.y; y1[6] = b.z; y1[7] = b.w;
      y2[0] = c.x; y2[1] = c.y; y2[2] = c.z; y2[3] = c.w; y2[4] = d.x; y2[5] = d.y; y2[6] = d.z; y2[7] = d.w;
    } else {
      load8(p, y1);
      load8(p + half, y2);
    }
    load8(cosb + (long long)pos * D + c8 * 8, c1);
    load8(sinb + (long long)pos * D + c8 * 8, s1);
    load8(cosb + (long long)pos * D + half + c8 * 8, c2);
    load8(sinb + (long long)pos * D + half + c8 * 8, s2);
    float o1[8], o2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o1[j] = y1[j] * c1[j] + y2[j] * s2[j];
      o2[j] = y2[j] * c2[j] - y1[j] * s1[j];
    }
    store8(p, o1);
    store8(p + half, o2);
  }
}

// RoPE of packed rows: rope_fwd_kernel / rope_bwd_kernel (split form: dQ already in the q block) with the position of
// row m read from pos[m] instead of m % T.
__global__ void rope_pos_fwd_kernel(bf16* __restrict__ qkv, const bf16* __restrict__ cosb, const bf16* __restrict__ sinb,
                                    const int* __restrict__ pos_of, long long M, int nrot, int D, long long ld) {
  const int half = D >> 1;
  const int per_head = half >> 3;
  const long long total = M * nrot * per_head;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(idx % per_head);
    long long r = idx / per_head;
    const int head = (int)(r % nrot);
    const long long row = r / nrot;
    const int pos = pos_of[row];
    bf16* p = qkv + row * ld + (long long)head * D + c8 * 8;
    float x1[8], x2[8], c1[8], s1[8], c2[8], s2[8];
    load8(p, x1);
    load8(p + half, x2);
    load8(cosb + (long long)pos * D + c8 * 8, c1);
    load8(sinb + (long long)pos * D + c8 * 8, s1);
    load8(cosb + (long long)pos * D + half + c8 * 8, c2);
    load8(sinb + (long long)pos * D + half + c8 * 8, s2);
    float o1[8], o2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o1[j] = bf16_round(x1[j] * c1[j]) + bf16_round(-x2[j] * s1[j]);
      o2[j] = bf16_round(x2[j] * c2[j]) + bf16_round(x1[j] * s2[j]);
    }
    store8(p, o1);
    store8(p + half, o2);
  }
}
__global__ void rope_pos_bwd_kernel(bf16* __restrict__ dqkv, const bf16* __restrict__ cosb, const bf16* __restrict__ sinb,
                                    const int* __restrict__ pos_of, long long M, int nrot, int D, long long ld) {
  const int half = D >> 1;
  const int per_head = half >> 3;
  const long long total = M * nrot * per_head;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(idx % per_head);
    long long r = idx / per_head;
    const int head = (int)(r % nrot);
    const long long row = r / nrot;
    const int pos = pos_of[row];
    bf16* p = dqkv + row * ld + (long long)head * D + c8 * 8;
    float y1[8], y2[8], c1[8], s1[8], c2[8], s2[8];
    load8(p, y1);
    load8(p + half, y2);
    load8(cosb + (long long)pos * D + c8 * 8, c1);
    load8(sinb + (long long)pos * D + c8 * 8, s1);
    load8(cosb + (long long)pos * D + half + c8 * 8, c2);
    load8(sinb + (long long)pos * D + half + c8 * 8, s2);
    float o1[8], o2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o1[j] = y1[j] * c1[j] + y2[j] * s2[j];
      o2[j] = y2[j] * c2[j] - y1[j] * s1[j];
    }
    store8(p, o1);
    store8(p + half, o2);
  }
}

// ------------------------------------------------------------------------------------------------
// SwiGLU (HF llama/modeling_llama.py:182-184): act = bf16(bf16(silu(g)) * u), gu = [g | u] per row
// ------------------------------------------------------------------------------------------------
__global__ void swiglu_fwd_kernel(const bf16* __restrict__ gu, bf16* __restrict__ act, long long M,
                                  int F) {
  // two independent 8-element chunks per thread per pass: four 16-byte loads in flight before any math
  const int nch = F >> 3;
  const long long total = M * nch;
  const long long T = (long long)gridDim.x * blockDim.x;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += 2 * T) {
    const long long idx2 = idx + T;
    const bool two = idx2 < total;
    const long long row0 = idx / nch, row1 = two ? idx2 / nch : row0;
    const int c0 = (int)(idx - row0 * nch), c1 = two ? (int)(idx2 - row1 * nch) : c0;
    float g0[8], u0[8], g1[8], u1[8], o[8];
    load8(gu + row0 * 2 * F + c0 * 8, g0);
    load8(gu + row0 * 2 * F + F + c0 * 8, u0);
    load8(gu + row1 * 2 * F + c1 * 8, g1);
    load8(gu + row1 * 2 * F + F + c1 * 8, u1);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = bf16_round(g0[j] / (1.f + __expf(-g0[j]))) * u0[j];
    store8(act + row0 * F + c0 * 8, o);
    if (two) {
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = bf16_round(g1[j] / (1.f + __expf(-g1[j]))) * u1[j];
      store8(act + row1 * F + c1 * 8, o);
    }
  }
}
__global__ void swiglu_bwd_kernel(const bf16* __restrict__ gu, const bf16* __restrict__ dact,
                                  bf16* __restrict__ dgu, long long M, int F) {
  const int nch = F >> 3;
  const long long total = M * nch;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long row = idx / nch;
    const int c = (int)(idx % nch);
    float g[8], u[8], d[8], dg[8], du[8];
    load8(gu + row * 2 * F + c * 8, g);
    load8(gu + row * 2 * F + F + c * 8, u);
    load8(dact + row * F + c * 8, d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sg = 1.f / (1.f + __expf(-g[j]));
      const float silu = g[j] * sg;
      du[j] = d[j] * silu;
      dg[j] = d[j] * u[j] * (sg * (1.f + g[j] * (1.f - sg)));
    }
    store8(dgu + row * 2 * F + c * 8, dg);
    store8(dgu + row * 2 * F + F + c * 8, du);
  }
}

// GELU(erf) backward for the mm_projector: dpre = dpost * gelu'(pre)
__global__ void gelu_bwd_kernel(const bf16* __restrict__ pre, const bf16* __restrict__ dpost,
                                bf16* __restrict__ dpre, long long n8) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n8;
       idx += (long long)gridDim.x * blockDim.x) {
    float x[8], d[8], o[8];
    load8(pre + idx * 8, x);
    load8(dpost + idx * 8, d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float cdf = 0.5f * (1.f + erff(x[j] * 0.70710678118654752f));
      const float pdf = 0.3989422804014327f * __expf(-0.5f * x[j] * x[j]);
      o[j] = d[j] * (cdf + x[j] * pdf);
    }
    store8(dpre + idx * 8, o);
  }
}

// GELU(erf) forward on a bf16 tensor (nn.GELU() between the two projector linears)
__global__ void gelu_fwd_kernel(const bf16* __restrict__ pre, bf16* __restrict__ post, long long n8) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n8;
       idx += (long long)gridDim.x * blockDim.x) {
    float x[8];
    load8(pre + idx * 8, x);
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = 0.5f * x[j] * (1.f + erff(x[j] * 0.70710678118654752f));
    store8(post + idx * 8, x);
  }
}

// column sums of a bf16 matrix [M][N] -> bias grad (fp32 accumulate, bf16 out, optional +=)
__global__ void colsum_kernel(const bf16* __restrict__ x, long long M, int N, float* __restrict__ part) {
  // grid (ceil(N/256), P); each block sums rows blockIdx.y, +P, ... for 256 columns (2 per thread)
  const int col = (blockIdx.x * blockDim.x + threadIdx.x) * 2;
  if (col >= N) return;
  float a = 0.f, b = 0.f;
  for (long long r = blockIdx.y; r < M; r += gridDim.y) {
    float2 v = unpack_bf16(*reinterpret_cast<const uint32_t*>(x + r * N + col));
    a += v.x;
    b += v.y;
  }
  part[(long long)blockIdx.y * N + col] = a;
  part[(long long)blockIdx.y * N + col + 1] = b;
}

// ------------------------------------------------------------------------------------------------
// CLIP patch embedding helpers (HF clip/modeling_clip.py:148-154,202-219)
// ------------------------------------------------------------------------------------------------
// im2col for a stride==kernel conv: out[(n*G*G + gy*G + gx)][c*P*P + py*P + px] (K padded with 0)
__global__ void im2col_patch_kernel(const bf16* __restrict__ img, bf16* __restrict__ out, int N,
                                    int C, int S, int P, int Kpad) {
  const int G = S / P;
  const long long rows = (long long)N * G * G;
  const long long total = rows * Kpad;
  const int K = C * P * P;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(idx % Kpad);
    const long long row = idx / Kpad;
    bf16 v = __float2bfloat16_rn(0.f);
    if (k < K) {
      const int c = k / (P * P);
      const int py = (k / P) % P;
      const int px = k % P;
      const int gx = (int)(row % G);
      const int gy = (int)((row / G) % G);
      const long long n = row / ((long long)G * G);
      v = img[((n * C + c) * S + gy * P + py) * (long long)S + gx * P + px];
    }
    out[idx] = v;
  }
}
// x[n][0] = bf16(cls + pos[0]); x[n][1+p] = bf16(patch[n][p] + pos[1+p])
__global__ void clip_embed_kernel(const bf16* __restrict__ patch, const bf16* __restrict__ cls,
                                  const bf16* __restrict__ pos, bf16* __restrict__ x, int N,
                                  int NP, int H) {
  const int nch = H >> 3;
  const long long total = (long long)N * (NP + 1) * nch;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % nch);
    const long long r = idx / nch;
    const int t = (int)(r % (NP + 1));
    const long long n = r / (NP + 1);
    float a[8], p[8];
    if (t == 0) load8(cls + c * 8, a);
    else load8(patch + (n * NP + (t - 1)) * (long long)H + c * 8, a);
    load8(pos + (long long)t * H + c * 8, p);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += p[j];
    store8(x + r * H + c * 8, a);
  }
}
// drop the CLS row: out[n][p] = x[n][1+p]   (clip_encoder.py:36-44 feature_select 'patch')
__global__ void drop_cls_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int N, int NP,
                                int H) {
  const int nch = H >> 3;
  const long long total = (long long)N * NP * nch;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % nch);
    const long long r = idx / nch;
    const int p = (int)(r % NP);
    const long long n = r / NP;
    *reinterpret_cast<uint4*>(out + r * H + c * 8) =
        *reinterpret_cast<const uint4*>(x + (n * (NP + 1) + 1 + p) * (long long)H + c * 8);
  }
}

// ------------------------------------------------------------------------------------------------
// Image-token splice (llava/model/llava_arch.py:231-315, attention_mask=None path).
// Index map: one warp per sequence. src[b][t] >= 0 : token position j in input_ids[b];
// src = -1-r : image-feature row r (global row in the feature matrix); src = INT_MIN : pad.
// The i-th image slot (in batch order, counting a slot-less sequence as consuming one feature
// block like the reference's cur_image_idx) takes feature block img_index[i].
// ------------------------------------------------------------------------------------------------
constexpr int SPLICE_PAD = -2147483647 - 1;
constexpr long long IMAGE_TOKEN_INDEX = -200;
constexpr long long IGNORE_INDEX = -100;

// pass 1: per-sequence image count and spliced length (before global max)
__global__ void splice_count_kernel(const long long* __restrict__ ids, int nseq, int L, int P,
                                    int max_len, int* __restrict__ n_img, int* __restrict__ len) {
  const int b = blockIdx.x;
  int cnt = 0;
  for (int j = threadIdx.x; j < L; j += 32) cnt += (ids[(long long)b * L + j] == IMAGE_TOKEN_INDEX);
  cnt = (int)warp_sum((float)cnt);
  if (threadIdx.x == 0) {
    n_img[b] = cnt;
    int t = L - cnt + cnt * P;
    len[b] = t < max_len ? t : max_len;
  }
}
// pass 2: fill src and new labels for T columns
__global__ void splice_map_kernel(const long long* __restrict__ ids,
                                  const long long* __restrict__ labels, const int* __restrict__ n_img,
                                  const int* __restrict__ img_index, int nseq, int L, int P, int T,
                                  int max_len, int* __restrict__ src, long long* __restrict__ new_labels) {
  const int b = blockIdx.x;
  // first feature-block slot of this sequence = sum over previous sequences of max(n_img,1)
  int slot0 = 0;
  for (int i = 0; i < b; ++i) slot0 += n_img[i] > 0 ? n_img[i] : 1;
  const long long* idr = ids + (long long)b * L;
  const long long* lbr = labels ? labels + (long long)b * L : nullptr;
  int* sr = src + (long long)b * T;
  long long* nl = new_labels + (long long)b * T;
  // sequential over tokens by warp-wide prefix: process 32 tokens at a time
  int out = 0, imgs_before = 0;
  for (int base = 0; base < L; base += 32) {
    const int j = base + threadIdx.x;
    const bool valid = j < L;
    const bool is_img = valid && idr[j] == IMAGE_TOKEN_INDEX;
    const unsigned img_mask = __ballot_sync(0xffffffffu, is_img);
    const int imgs_lt = __popc(img_mask & ((1u << threadIdx.x) - 1));
    // output offset of token j = out + (j-base) + imgs_lt*(P-1)
    const int o = out + threadIdx.x + imgs_lt * (P - 1);
    if (valid) {
      if (!is_img) {
        if (o < T && o < max_len) {
          sr[o] = j;
          nl[o] = lbr ? lbr[j] : IGNORE_INDEX;
        }
      } else {
        const int blk = img_index[slot0 + imgs_before + imgs_lt];
        for (int p = 0; p < P; ++p) {
          const int oo = o + p;
          if (oo < T && oo < max_len) {
            sr[oo] = -1 - (blk * P + p);
            nl[oo] = IGNORE_INDEX;
          }
        }
      }
    }
    const int nvalid = min(32, L - base);
    out += nvalid + __popc(img_mask) * (P - 1);
    imgs_before += __popc(img_mask);
  }
  const int end = out < max_len ? out : max_len;
  for (int t = end + threadIdx.x; t < T; t += 32) {
    sr[t] = SPLICE_PAD;
    nl[t] = IGNORE_INDEX;
  }
}
// In-place splice map of OmniLMM (omnilmm/model/omnilmm.py:219-258): the sequence already holds
// <im_start> <im_patch>*Q <im_end>; the Q rows after each <im_start> take the image's resampled features, every
// other row keeps its token embedding (src[b][t] = t), the length does not change. Feature blocks are consumed in
// batch order (cur_image_idx); a sequence without <im_patch> consumes none. status bit0: #<im_start> != #<im_end>,
// bit1: <im_end> not at start+Q+1 (the reference raises ValueError for both). One warp walks the whole batch.
__global__ void splice_map_inplace_kernel(const long long* __restrict__ ids, const int* __restrict__ img_index,
                                          int nseq, int L, int Q, long long im_patch, long long im_start,
                                          long long im_end, int* __restrict__ src, int* __restrict__ status) {
  const int lane = threadIdx.x;
  int slot = 0;
  for (int b = 0; b < nseq; ++b) {
    const long long* row = ids + (long long)b * L;
    int* sr = src + (long long)b * L;
    int np = 0, ns = 0, ne = 0;
    for (int j = lane; j < L; j += 32) {
      const long long t = row[j];
      np += (t == im_patch);
      ns += (t == im_start);
      ne += (t == im_end);
      sr[j] = j;
    }
    np = __reduce_add_sync(0xffffffffu, np);
    ns = __reduce_add_sync(0xffffffffu, ns);
    ne = __reduce_add_sync(0xffffffffu, ne);
    __syncwarp();
    if (np == 0) continue;
    if (ns != ne) {
      if (lane == 0) atomicOr(status, 1);
      continue;
    }
    for (int base = 0; base < L; base += 32) {
      const int j = base + lane;
      const bool is_start = j < L && row[j] == im_start;
      const unsigned mask = __ballot_sync(0xffffffffu, is_start);
      if (is_start) {
        const int k = __popc(mask & ((1u << lane) - 1));
        if (j + Q + 1 >= L || row[j + Q + 1] != im_end) {
          atomicOr(status, 2);
        } else {
          const int blk = img_index[slot + k];
          for (int q = 0; q < Q; ++q) sr[j + 1 + q] = -1 - (blk * Q + q);
        }
      }
      slot += __popc(mask);
      __syncwarp();
    }
  }
}
// row gather: out[b][t][:] = embed[ids[b][src]] | feat[-1-src] | 0     (bit-exact copies)
__global__ void splice_gather_kernel(const int* __restrict__ src, const long long* __restrict__ ids,
                                     const bf16* __restrict__ embed, const bf16* __restrict__ feat,
                                     bf16* __restrict__ out, int nseq, int L, int T, int H) {
  const int nch = H >> 3;
  const long long rows = (long long)nseq * T;
  const int wpb = blockDim.x >> 5;
  for (long long r = (long long)blockIdx.x * wpb + (threadIdx.x >> 5); r < rows;
       r += (long long)gridDim.x * wpb) {
    const int s = src[r];
    const int b = (int)(r / T);
    const bf16* sp = nullptr;
    if (s >= 0) sp = embed + ids[(long long)b * L + s] * (long long)H;
    else if (s != SPLICE_PAD) sp = feat + (long long)(-1 - s) * H;
    uint4* dst = reinterpret_cast<uint4*>(out + r * H);
    for (int c = threadIdx.x & 31; c < nch; c += 32)
      dst[c] = sp ? reinterpret_cast<const uint4*>(sp)[c] : make_uint4(0, 0, 0, 0);
  }
}
// backward scatter: d_embed[ids[b][src]] += dx (fp32 atomics), d_feat[-1-src] += dx (fp32 atomics)
__global__ void splice_scatter_kernel(const int* __restrict__ src, const long long* __restrict__ ids,
                                      const bf16* __restrict__ dx, float* __restrict__ d_embed,
                                      float* __restrict__ d_feat, int nseq, int L, int T, int H) {
  const int nch = H >> 3;
  const long long rows = (long long)nseq * T;
  const int wpb = blockDim.x >> 5;
  for (long long r = (long long)blockIdx.x * wpb + (threadIdx.x >> 5); r < rows;
       r += (long long)gridDim.x * wpb) {
    const int s = src[r];
    if (s == SPLICE_PAD) continue;
    const int b = (int)(r / T);
    float* dp = (s >= 0) ? d_embed + ids[(long long)b * L + s] * (long long)H
                         : d_feat + (long long)(-1 - s) * H;
    if ((s >= 0 && !d_embed) || (s < 0 && !d_feat)) continue;
    for (int c = threadIdx.x & 31; c < nch; c += 32) {
      float v[8];
      load8(dx + r * H + c * 8, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) atomicAdd(dp + c * 8 + j, v[j]);
    }
  }
}
__global__ void f32_to_bf16_kernel(const float* __restrict__ in, bf16* __restrict__ out, long long n8,
                                   int accumulate) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n8;
       idx += (long long)gridDim.x * blockDim.x) {
    float4 a = *reinterpret_cast<const float4*>(in + idx * 8);
    float4 b = *reinterpret_cast<const float4*>(in + idx * 8 + 4);
    float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    if (accumulate) {
      float o[8];
      load8(out + idx * 8, o);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += o[j];
    }
    store8(out + idx * 8, v);
  }
}

// strided variant: rows x cols fp32 (row stride ld_in) -> bf16 column block of a wider buffer (row stride ld_out)
__global__ void f32_to_bf16_2d_kernel(const float* __restrict__ in, long long ld_in, bf16* __restrict__ out,
                                      long long ld_out, long long rows, int cols8, int accumulate) {
  const long long total = rows * cols8;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / cols8;
    const int c = (int)(idx - r * cols8) * 8;
    const float* src = in + r * ld_in + c;
    float4 a = *reinterpret_cast<const float4*>(src);
    float4 b = *reinterpret_cast<const float4*>(src + 4);
    float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    bf16* dst = out + r * ld_out + c;
    if (accumulate) {
      float o[8];
      load8(dst, o);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += o[j];
    }
    store8(dst, v);
  }
}

// ------------------------------------------------------------------------------------------------
// Per-token log-prob gather (muffin/eval/muffin_inference_logp.py:82-115).
// Row r = (b, t), t in [0, T-1): label = labels[b][t+1]; mask = label != -100; label(-100) -> 0;
// per_tok[b][t] = logits[b][t][label] - logsumexp(logits[b][t][:]) with logits upcast to fp32
// (pinned transformers 4.35 `.float()`); lse saved for the backward.
// ------------------------------------------------------------------------------------------------
constexpr int LOGP_THREADS = 256;
__global__ void __launch_bounds__(LOGP_THREADS)
logp_fwd_kernel(const bf16* __restrict__ logits, long long ld, const long long* __restrict__ labels,
                int nseq, int T, int V, float* __restrict__ per_tok, float* __restrict__ lse_out,
                const int* __restrict__ row_pos, long long n_compact) {
  // row_pos != nullptr: COMPACT head — logits row r belongs to flat position row_pos[r] = b*T + t (t < T-1), or is a
  // padding slot (-1, skipped); lse_out is then indexed by the compact row. nullptr: dense [nseq*T] logits.
  const long long rows = row_pos ? n_compact : (long long)nseq * (T - 1);
  __shared__ float sm[32], ss[32];
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    int b, t;
    long long lrow;
    if (row_pos) {
      const int pos = row_pos[r];
      if (pos < 0) continue;          // uniform over the block
      b = pos / T;
      t = pos % T;
      lrow = r;
    } else {
      b = (int)(r / (T - 1));
      t = (int)(r % (T - 1));
      lrow = (long long)b * T + t;
    }
    const bf16* lr = logits + lrow * ld;
    float m = -INFINITY, s = 0.f;
    const int nch = V >> 3;
    for (int c = threadIdx.x; c < nch; c += LOGP_THREADS) {
      float v[8];
      load8(lr + c * 8, v);
      float cm = v[0];
#pragma unroll
      for (int j = 1; j < 8; ++j) cm = fmaxf(cm, v[j]);
      const float nm = fmaxf(m, cm);
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc += __expf(v[j] - nm);
      s = s * __expf(m - nm) + acc;
      m = nm;
    }
    // warp combine
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m, o);
      const float os = __shfl_xor_sync(0xffffffffu, s, o);
      const float nm = fmaxf(m, om);
      s = (m == -INFINITY ? 0.f : s * __expf(m - nm)) + (om == -INFINITY ? 0.f : os * __expf(om - nm));
      m = nm;
    }
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) { sm[w] = m; ss[w] = s; }
    __syncthreads();
    if (w == 0) {
      m = (l < LOGP_THREADS / 32) ? sm[l] : -INFINITY;
      s = (l < LOGP_THREADS / 32) ? ss[l] : 0.f;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, m, o);
        const float os = __shfl_xor_sync(0xffffffffu, s, o);
        const float nm = fmaxf(m, om);
        s = (m == -INFINITY ? 0.f : s * __expf(m - nm)) + (om == -INFINITY ? 0.f : os * __expf(om - nm));
        m = nm;
      }
      if (l == 0) {
        const float lse = m + logf(s);
        long long lab = labels[(long long)b * T + t + 1];
        if (lab == IGNORE_INDEX) lab = 0;
        const float z = __bfloat162float(lr[lab]);
        per_tok[(long long)b * (T - 1) + t] = z - lse;
        lse_out[row_pos ? r : lrow] = lse;
      }
    }
  }
}
// Per-sequence reductions. Token-weighted when token_weight [nseq][T-1] is given (compute_weighted_logp,
// muffin/train/trainers.py:128-137 — the `dpo_token_weighted` branch of get_beta_and_logps, :246-261), weight 1 when
// it is nullptr: mask = weight * (label != -100); logp_sum[b] = sum_t per_tok * mask; count[b] = sum_t mask;
// avg = logp_sum / count. A weight of exactly 1 rounds like the plain sum (fma(p, 1, s) == p + s).
__global__ void logp_reduce_kernel(const float* __restrict__ per_tok, const long long* __restrict__ labels,
                                   const float* __restrict__ token_weight, int nseq, int T,
                                   float* __restrict__ logp_sum, float* __restrict__ logp_avg,
                                   float* __restrict__ count_out) {
  const int b = blockIdx.x;
  float s = 0.f, c = 0.f;
  for (int t = threadIdx.x; t < T - 1; t += blockDim.x) {
    const bool mk = labels[(long long)b * T + t + 1] != IGNORE_INDEX;
    if (mk) {
      const float w = token_weight ? token_weight[(long long)b * (T - 1) + t] : 1.f;
      s += per_tok[(long long)b * (T - 1) + t] * w;
      c += w;
    }
  }
  const float2 tot = block_sum2(s, c);
  if (threadIdx.x == 0) {
    logp_sum[b] = tot.x;
    logp_avg[b] = tot.x / tot.y;
    if (count_out) count_out[b] = tot.y;
  }
}
// backward, in place: logits[b][t][v] <- g_b * w[b][t] * mask * (onehot(v==label) - softmax_v), row T-1 <- 0;
// w = token_weight (1 when nullptr); g_b = d_logp[b] (sum mode) or d_logp[b] / norm[b] (average mode, norm passed
// non-null: the label count, or the weight sum when weighted).
__global__ void __launch_bounds__(LOGP_THREADS)
logp_bwd_kernel(bf16* __restrict__ logits, long long ld, const long long* __restrict__ labels,
                const float* __restrict__ lse, const float* __restrict__ d_logp,
                const float* __restrict__ token_weight, const float* __restrict__ norm, int nseq, int T,
                int V, const int* __restrict__ row_pos, long long n_compact) {
  // row_pos: compact head (see logp_fwd_kernel) — logits row r is position row_pos[r], padding slots and unsupervised
  // rows are zeroed.
  const long long rows = row_pos ? n_compact : (long long)nseq * T;
  const int nch = V >> 3;
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    int b, t;
    if (row_pos) {
      const int pos = row_pos[r];
      b = pos < 0 ? 0 : pos / T;
      t = pos < 0 ? T - 1 : pos % T;
    } else {
      b = (int)(r / T);
      t = (int)(r % T);
    }
    bf16* lr = logits + r * ld;
    long long lab = (t < T - 1) ? labels[(long long)b * T + t + 1] : IGNORE_INDEX;
    if (lab == IGNORE_INDEX) {
      for (int c = threadIdx.x; c < nch; c += LOGP_THREADS)
        *reinterpret_cast<uint4*>(lr + c * 8) = make_uint4(0, 0, 0, 0);
      continue;
    }
    float g = d_logp[b] * (token_weight ? token_weight[(long long)b * (T - 1) + t] : 1.f);
    if (norm) g /= norm[b];
    const float l = lse[r];
    for (int c = threadIdx.x; c < nch; c += LOGP_THREADS) {
      float v[8];
      load8(lr + c * 8, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float p = __expf(v[j] - l);
        v[j] = g * (((long long)(c * 8 + j) == lab ? 1.f : 0.f) - p);
      }
      store8(lr + c * 8, v);
    }
  }
}

// Token weights through the image splice (extension: --dpo_token_weighted for LLaVA-1.5, which the reference refuses
// because its collator's weights are in TEXT positions while the log-probs are in SPLICED positions,
// muffin/train/train_muffin.py:78-81 / trainers.py:246-248). out[s][t] = weight of spliced token t+1: the text weight
// tw[s][j-1] when that token is text token j >= 1 (src >= 0), 1 for image rows / padding (masked by the labels anyway).
__global__ void splice_token_weight_kernel(const int* __restrict__ src, const float* __restrict__ tw, float* __restrict__ out,
                                           int nseq, int Lw, int T) {
  const long long total = (long long)nseq * (T - 1);
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int s = (int)(idx / (T - 1)), t = (int)(idx % (T - 1));
    const int j = src[(long long)s * T + t + 1];
    out[idx] = (j >= 1 && j - 1 < Lw) ? tw[(long long)s * Lw + j - 1] : 1.0f;
  }
}

// ------------------------------------------------------------------------------------------------
// Compact lm_head: only positions whose NEXT token carries a label contribute to get_batch_logps
// (muffin/eval/muffin_inference_logp.py:93-104: loss_mask = labels[:, 1:] != -100), i.e. 512 of the 1135 positions
// of a config-(b) sequence. row_pos[s*cap + j] = s*T + t of the j-th such position of sequence s (ascending t),
// -1 for the unused slots of the sequence's `cap`-sized segment (cap >= number of labels of a row, e.g. L).
// One warp per sequence, ballot-scan over T.
// ------------------------------------------------------------------------------------------------
__global__ void supervised_rows_kernel(const long long* __restrict__ labels, int nseq, int T, int cap,
                                       int* __restrict__ row_pos) {
  const int s = blockIdx.x;
  const int lane = threadIdx.x;
  int base = 0;
  for (int t0 = 0; t0 < T - 1; t0 += 32) {
    const int t = t0 + lane;
    const bool on = t < T - 1 && labels[(long long)s * T + t + 1] != IGNORE_INDEX;
    const unsigned m = __ballot_sync(0xffffffffu, on);
    const int idx = base + __popc(m & ((1u << lane) - 1u));
    if (on && idx < cap) row_pos[(long long)s * cap + idx] = s * T + t;
    base += __popc(m);
  }
  for (int j = min(base, cap) + lane; j < cap; j += 32) row_pos[(long long)s * cap + j] = -1;
}
// out[r] = x[row_pos[r]] (zeros for padding slots)
__global__ void rows_gather_kernel(const int* __restrict__ row_pos, const bf16* __restrict__ x, bf16* __restrict__ out,
                                   long long n_rows, int H8) {
  const long long total = n_rows * H8;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / H8;
    const int c = (int)(idx - r * H8);
    const int pos = row_pos[r];
    uint4 v = make_uint4(0, 0, 0, 0);
    if (pos >= 0) v = *reinterpret_cast<const uint4*>(x + ((long long)pos * H8 + c) * 8);
    *reinterpret_cast<uint4*>(out + idx * 8) = v;
  }
}
// dx[row_pos[r]] = dy[r] (dx zero-filled by the caller; every position appears at most once)
__global__ void rows_scatter_kernel(const int* __restrict__ row_pos, const bf16* __restrict__ dy,
                                    bf16* __restrict__ dx, long long n_rows, int H8) {
  const long long total = n_rows * H8;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / H8;
    const int c = (int)(idx - r * H8);
    const int pos = row_pos[r];
    if (pos >= 0)
      *reinterpret_cast<uint4*>(dx + ((long long)pos * H8 + c) * 8) = *reinterpret_cast<const uint4*>(dy + idx * 8);
  }
}

// ------------------------------------------------------------------------------------------------
// DPO loss + gradient (muffin/train/trainers.py:91-126, 279-311). One warp.
//   z = beta*((pw-pr)-(rw-rr)); losses = -logsigmoid(z); loss = DPO_w*mean(losses) - SFT_w*mean(pw)
//   d loss/d pw_i = (-DPO_w*beta*sigmoid(-z_i) - SFT_w)/B ;  d loss/d pr_i = DPO_w*beta*sigmoid(-z_i)/B
// out[0]=loss, metrics (local means): [1]=chosen_reward [2]=rejected_reward [3]=accuracy [4]=margin
//   [5]=logps_rejected [6]=logps_chosen [7]=ref_rejected [8]=ref_chosen
// ------------------------------------------------------------------------------------------------
__global__ void dpo_loss_kernel(const float* __restrict__ pw, const float* __restrict__ pr,
                                const float* __restrict__ rw, const float* __restrict__ rr, int B,
                                float beta, float dpo_w, float sft_w, float grad_scale,
                                float* __restrict__ losses, float* __restrict__ chosen_rewards,
                                float* __restrict__ rejected_rewards, float* __restrict__ d_pw,
                                float* __restrict__ d_pr, float* __restrict__ out9) {
  float acc[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) acc[i] = 0.f;
  for (int i = threadIdx.x; i < B; i += 32) {
    const float a = pw[i], b = pr[i], c = rw[i], d = rr[i];
    const float z = beta * ((a - b) - (c - d));
    // -logsigmoid(z) = softplus(-z) = max(-z,0) + log1p(exp(-|z|))
    const float loss = fmaxf(-z, 0.f) + log1pf(expf(-fabsf(z)));
    const float sig_neg = 1.f / (1.f + expf(z));  // sigmoid(-z)
    const float cr = beta * (a - c), rj = beta * (b - d);
    if (losses) losses[i] = loss;
    if (chosen_rewards) chosen_rewards[i] = cr;
    if (rejected_rewards) rejected_rewards[i] = rj;
    if (d_pw) d_pw[i] = grad_scale * (-dpo_w * beta * sig_neg - sft_w) / (float)B;
    if (d_pr) d_pr[i] = grad_scale * (dpo_w * beta * sig_neg) / (float)B;
    acc[0] += dpo_w * loss - sft_w * a;
    acc[1] += cr; acc[2] += rj; acc[3] += (cr > rj) ? 1.f : 0.f; acc[4] += cr - rj;
    acc[5] += b; acc[6] += a; acc[7] += d; acc[8] += c;
  }
#pragma unroll
  for (int i = 0; i < 9; ++i) acc[i] = warp_sum(acc[i]);
  if (threadIdx.x == 0 && out9) {
#pragma unroll
    for (int i = 0; i < 9; ++i) out9[i] = acc[i] / (float)B;
  }
}

// ------------------------------------------------------------------------------------------------
// Fused AdamW on a flat shard (torch.optim.AdamW semantics; fp32 master/m/v, bf16 or fp32 grads):
//   g = grad*grad_scale; p *= 1-lr*wd; m = b1 m + (1-b1) g; v = b2 v + (1-b2) g^2;
//   p -= (lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps); param_bf16 = bf16(p)
// ------------------------------------------------------------------------------------------------
// One element of the update. adamw_kernel and adamw_staged_kernel both call it, so the on-device and the offloaded
// optimizer perform the same operations in the same order and their results are bit-identical.
__device__ __forceinline__ void adamw_elem(float& p, float& m, float& v, float g, float lr, float b1, float b2,
                                           float eps, float wd, float bc1, float bc2_sqrt, float grad_scale) {
  const float gj = g * grad_scale;
  p *= (1.f - lr * wd);
  m = b1 * m + (1.f - b1) * gj;
  v = b2 * v + (1.f - b2) * gj * gj;
  const float denom = sqrtf(v) / bc2_sqrt + eps;
  p -= (lr / bc1) * (m / denom);
}

template <bool GRAD_F32>
__global__ void adamw_kernel(float* __restrict__ master, float* __restrict__ m, float* __restrict__ v,
                             const void* __restrict__ grad, bf16* __restrict__ param_out, long long n,
                             float lr, float b1, float b2, float eps, float wd, float bc1,
                             float bc2_sqrt, float grad_scale) {
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 p4 = reinterpret_cast<float4*>(master)[i];
    float4 m4 = reinterpret_cast<float4*>(m)[i];
    float4 v4 = reinterpret_cast<float4*>(v)[i];
    float g[4];
    if (GRAD_F32) {
      float4 g4 = reinterpret_cast<const float4*>(grad)[i];
      g[0] = g4.x; g[1] = g4.y; g[2] = g4.z; g[3] = g4.w;
    } else {
      uint2 u = reinterpret_cast<const uint2*>(grad)[i];
      float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y);
      g[0] = a.x; g[1] = a.y; g[2] = b.x; g[3] = b.y;
    }
    float p[4] = {p4.x, p4.y, p4.z, p4.w}, mm[4] = {m4.x, m4.y, m4.z, m4.w},
          vv[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) adamw_elem(p[j], mm[j], vv[j], g[j], lr, b1, b2, eps, wd, bc1, bc2_sqrt, grad_scale);
    reinterpret_cast<float4*>(master)[i] = make_float4(p[0], p[1], p[2], p[3]);
    reinterpret_cast<float4*>(m)[i] = make_float4(mm[0], mm[1], mm[2], mm[3]);
    reinterpret_cast<float4*>(v)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
    uint2 o;
    o.x = pack_bf16(p[0], p[1]);
    o.y = pack_bf16(p[2], p[3]);
    reinterpret_cast<uint2*>(param_out)[i] = o;
  }
}

// AdamW on one chunk of a bucket whose fp32 state was copied into a device staging slot (master | m | v, n each).
// grad / param_out point at the chunk's first element in the bucket's bf16 gradient and parameter buffers. Elements
// below decay_n get weight decay, the rest none, so a chunk that straddles the bucket's decay boundary is one launch
// (a zero wd makes 1 - lr*wd exactly 1, as in the on-device path's separate no-decay launch).
__global__ void adamw_staged_kernel(float* __restrict__ master, float* __restrict__ m, float* __restrict__ v,
                                    const bf16* __restrict__ grad, bf16* __restrict__ param_out, long long n,
                                    long long decay_n, float lr, float b1, float b2, float eps, float wd, float bc1,
                                    float bc2_sqrt) {
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 p4 = reinterpret_cast<float4*>(master)[i];
    float4 m4 = reinterpret_cast<float4*>(m)[i];
    float4 v4 = reinterpret_cast<float4*>(v)[i];
    uint2 u = reinterpret_cast<const uint2*>(grad)[i];
    float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y);
    float g[4] = {a.x, a.y, b.x, b.y};
    float p[4] = {p4.x, p4.y, p4.z, p4.w}, mm[4] = {m4.x, m4.y, m4.z, m4.w},
          vv[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j)
      adamw_elem(p[j], mm[j], vv[j], g[j], lr, b1, b2, eps, 4 * i + j < decay_n ? wd : 0.f, bc1, bc2_sqrt, 1.f);
    reinterpret_cast<float4*>(master)[i] = make_float4(p[0], p[1], p[2], p[3]);
    reinterpret_cast<float4*>(m)[i] = make_float4(mm[0], mm[1], mm[2], mm[3]);
    reinterpret_cast<float4*>(v)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
    uint2 o;
    o.x = pack_bf16(p[0], p[1]);
    o.y = pack_bf16(p[2], p[3]);
    reinterpret_cast<uint2*>(param_out)[i] = o;
  }
}

// ------------------------------------------------------------------------------------------------
// AdamW with blockwise 8-bit moments (Dettmers et al., "8-bit Optimizers via Block-wise Quantization", 2022;
// bitsandbytes AdamW8bit with percentile clipping off). State per element: the fp32 master and one uint8 code each for
// m and v; per block of 256 consecutive elements one fp32 absmax each. m = map_m[code_m] * absmax_m and
// v = map_v[code_v] * absmax_v, map_m / map_v being the signed / unsigned dynamic maps (256 strictly increasing fp32
// values each, built by zero2.dynamic_map). A block's update: dequantize, adamw_elem, absmax_m = max|m| and
// absmax_v = max v over the new fp32 moments, then store for each element the code of the map entry nearest to
// m / absmax_m (v / absmax_v), ties to the lower index; a zero absmax stores the code of 0.
// ------------------------------------------------------------------------------------------------
static constexpr int kQBlock = 256;

// Index of the entry of the sorted 256-entry map nearest to x, ties to the lower index: a binary search for the last
// entry <= x (entry 0 if there is none), then one compare with its upper neighbour.
__device__ __forceinline__ uint32_t quantize_nearest(const float* map, float x) {
  int i = 0;
#pragma unroll
  for (int step = 128; step >= 1; step >>= 1)
    if (map[i + step] <= x) i += step;
  i = min(i, kQBlock - 2);
  const float lo = map[i], hi = map[i + 1];
  return (uint32_t)(i + (hi - x < x - lo ? 1 : 0));
}

// One block of the 8-bit update, run by one whole warp: lane l owns elements [8l, 8l + 8) of the block's first `cnt`
// (a multiple of 8, at most 256). Pointers are at the block's first element (absmax_m / absmax_v at its entry);
// elements below decay_n, counted from the block's first element, get weight decay. smap: map_m | map_v in shared
// memory. adamw8bit_kernel runs it for the on-device and for the offloaded optimizer alike, so their results are
// bit-identical.
__device__ __forceinline__ void adamw8bit_block(float* __restrict__ master, uint8_t* __restrict__ qm,
                                                uint8_t* __restrict__ qv, float* __restrict__ absmax_m,
                                                float* __restrict__ absmax_v, const bf16* __restrict__ grad,
                                                bf16* __restrict__ param_out, int cnt, long long decay_n,
                                                const float* smap, float lr, float b1, float b2, float eps, float wd,
                                                float bc1, float bc2_sqrt) {
  const int lane = threadIdx.x & 31;
  const int e0 = lane * 8;
  const bool live = e0 < cnt;
  float p[8], m[8], v[8];
  float mx_m = 0.f, mx_v = 0.f;
  if (live) {
    const float4 p0 = reinterpret_cast<const float4*>(master + e0)[0];
    const float4 p1 = reinterpret_cast<const float4*>(master + e0)[1];
    const uint2 cm = *reinterpret_cast<const uint2*>(qm + e0);
    const uint2 cv = *reinterpret_cast<const uint2*>(qv + e0);
    float g[8];
    load8(grad + e0, g);
    const float am = *absmax_m, av = *absmax_v;
    p[0] = p0.x; p[1] = p0.y; p[2] = p0.z; p[3] = p0.w; p[4] = p1.x; p[5] = p1.y; p[6] = p1.z; p[7] = p1.w;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t sh = 8 * (j & 3);
      m[j] = smap[((j < 4 ? cm.x : cm.y) >> sh) & 255] * am;
      v[j] = smap[kQBlock + (((j < 4 ? cv.x : cv.y) >> sh) & 255)] * av;
      adamw_elem(p[j], m[j], v[j], g[j], lr, b1, b2, eps, e0 + j < decay_n ? wd : 0.f, bc1, bc2_sqrt, 1.f);
      mx_m = fmaxf(mx_m, fabsf(m[j]));
      mx_v = fmaxf(mx_v, v[j]);
    }
    reinterpret_cast<float4*>(master + e0)[0] = make_float4(p[0], p[1], p[2], p[3]);
    reinterpret_cast<float4*>(master + e0)[1] = make_float4(p[4], p[5], p[6], p[7]);
    store8(param_out + e0, p);
  }
  mx_m = warp_max(mx_m);
  mx_v = warp_max(mx_v);
  if (live) {
    uint2 om = make_uint2(0u, 0u), ov = make_uint2(0u, 0u);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t sh = 8 * (j & 3);
      const uint32_t c_m = quantize_nearest(smap, mx_m > 0.f ? m[j] / mx_m : 0.f);
      const uint32_t c_v = quantize_nearest(smap + kQBlock, mx_v > 0.f ? v[j] / mx_v : 0.f);
      (j < 4 ? om.x : om.y) |= c_m << sh;
      (j < 4 ? ov.x : ov.y) |= c_v << sh;
    }
    *reinterpret_cast<uint2*>(qm + e0) = om;
    *reinterpret_cast<uint2*>(qv + e0) = ov;
  }
  if (lane == 0) {
    *absmax_m = mx_m;
    *absmax_v = mx_v;
  }
}

// The 8-bit update of n elements (n % 8 == 0) whose blocks start at element 0: one warp per 256-element block, the
// last block partial when n % 256 != 0. The on-device optimizer launches it on a slice, the offloaded one on a chunk
// staged in a ring slot.
__global__ void __launch_bounds__(256) adamw8bit_kernel(float* __restrict__ master, uint8_t* __restrict__ qm,
                                                        uint8_t* __restrict__ qv, float* __restrict__ absmax_m,
                                                        float* __restrict__ absmax_v, const bf16* __restrict__ grad,
                                                        bf16* __restrict__ param_out, long long n, long long decay_n,
                                                        const float* __restrict__ map_m,
                                                        const float* __restrict__ map_v, float lr, float b1, float b2,
                                                        float eps, float wd, float bc1, float bc2_sqrt) {
  __shared__ float smap[2 * kQBlock];
  for (int i = threadIdx.x; i < 2 * kQBlock; i += blockDim.x) smap[i] = i < kQBlock ? map_m[i] : map_v[i - kQBlock];
  __syncthreads();
  const long long nblk = (n + kQBlock - 1) / kQBlock;
  const int warps = blockDim.x >> 5;
  for (long long b = (long long)blockIdx.x * warps + (threadIdx.x >> 5); b < nblk; b += (long long)gridDim.x * warps) {
    const long long e = b * kQBlock;
    const int cnt = n - e < kQBlock ? (int)(n - e) : kQBlock;
    adamw8bit_block(master + e, qm + e, qv + e, absmax_m + b, absmax_v + b, grad + e, param_out + e, cnt,
                    decay_n - e, smap, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
  }
}

// ------------------------------------------------------------------------------------------------
// Dropout for the LoRA adapter input (peft lora.Linear: lora_B(lora_A(dropout(x))), p = 0.05 in
// muffin/train/train_llava15_lora.py:115). Stateless counter-based RNG: the keep bit of element i
// is a hash of (seed, i), so the backward regenerates the mask instead of storing it.
//   fwd : out = keep ? bf16(x / (1-p)) : 0
//   bwd : dx += keep ? g / (1-p) : 0
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t mix32(uint64_t z) {   // splitmix64 finaliser, high word
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (uint32_t)(z >> 32);
}
__device__ __forceinline__ void keep_bits8(unsigned long long seed, long long chunk, uint32_t thresh, bool (&keep)[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) keep[j] = mix32(seed ^ ((unsigned long long)(chunk * 8 + j) * 0xD1B54A32D192ED03ull)) >= thresh;
}
__global__ void dropout_fwd_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, long long n8, uint32_t thresh,
                                   float inv_keep, unsigned long long seed) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n8;
       idx += (long long)gridDim.x * blockDim.x) {
    float v[8];
    bool keep[8];
    load8(x + idx * 8, v);
    keep_bits8(seed, idx, thresh, keep);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = keep[j] ? v[j] * inv_keep : 0.f;
    store8(out + idx * 8, v);
  }
}
__global__ void dropout_bwd_add_kernel(bf16* __restrict__ dx, const bf16* __restrict__ g, long long n8, uint32_t thresh,
                                       float inv_keep, unsigned long long seed) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n8;
       idx += (long long)gridDim.x * blockDim.x) {
    float a[8], b[8];
    bool keep[8];
    load8(dx + idx * 8, a);
    load8(g + idx * 8, b);
    keep_bits8(seed, idx, thresh, keep);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += keep[j] ? b[j] * inv_keep : 0.f;
    store8(dx + idx * 8, a);
  }
}
// Dropout of packed rows [n_rows][w8 * 8]: row r draws the keep bits of element (rows[r] * w8 * 8 + c), i.e. those of
// the padded row rows[r] in dropout_fwd_kernel / dropout_bwd_add_kernel. bwd: g == nullptr => forward (out = mask(x)).
__global__ void dropout_rows_kernel(const bf16* x, const bf16* __restrict__ g, bf16* out,
                                    const int* __restrict__ rows, long long n_rows, int w8, uint32_t thresh,
                                    float inv_keep, unsigned long long seed) {
  const long long n8 = n_rows * w8;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n8;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / w8;
    const long long chunk = (long long)rows[r] * w8 + (idx - r * w8);
    float a[8], b[8];
    bool keep[8];
    load8(x + idx * 8, a);
    keep_bits8(seed, chunk, thresh, keep);
    if (g) {
      load8(g + idx * 8, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += keep[j] ? b[j] * inv_keep : 0.f;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] = keep[j] ? a[j] * inv_keep : 0.f;
    }
    store8(out + idx * 8, a);
  }
}

// ---- FP8 e4m3 quantization of the frozen base's GEMM operands (DESIGN.md §3 "FP8 frozen base") ----
// A tile (1 x 128 of a row, or a 128 x 128 weight block) with amax = max|x| gets the scale s = 2^e, e the smallest
// integer with amax <= 448 * 2^e, clamped to [-126, 127] (s = 1 when amax = 0). x / s is exact and |x / s| <= 448,
// so the code RNE_e4m3(x / s) never saturates. oracle/fp8_oracle.py is the reference of every code and scale.
__device__ __forceinline__ int fp8_scale_exp(float amax) {
  if (!(amax > 0.f)) return 0;
  int E;
  const float m = frexpf(amax, &E);          // amax = m * 2^E, m in [0.5, 1); 448 = 0.875 * 2^9
  const int e = m <= 0.875f ? E - 9 : E - 8;
  return e < -126 ? -126 : (e > 127 ? 127 : e);
}
// two codes, RNE (lo in the low byte)
__device__ __forceinline__ uint32_t e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ uint2 e4m3x8(const float (&v)[8], float inv) {
  uint2 q;
  q.x = e4m3x2(v[0] * inv, v[1] * inv) | (e4m3x2(v[2] * inv, v[3] * inv) << 16);
  q.y = e4m3x2(v[4] * inv, v[5] * inv) | (e4m3x2(v[6] * inv, v[7] * inv) << 16);
  return q;
}

// One half-warp per 1 x 128 tile (16 lanes x one 16-byte load of 8 bf16); tile t = kb * M + m, so the scales of one
// K-block are written row after row. s: [K / 128][ld_s].
__global__ void __launch_bounds__(256) quant_fp8_rows_kernel(const bf16* __restrict__ x, long long ldx,
                                                             uint8_t* __restrict__ q, long long ldq,
                                                             float* __restrict__ s, long long ld_s, int M, int KB) {
  const int l = threadIdx.x & 15;
  const long long n_tiles = (long long)M * KB;
  // whole warps step together (the amax shuffle takes all 32 lanes); a half past the last tile idles
  for (long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 4; t - (threadIdx.x >> 4 & 1) < n_tiles;
       t += ((long long)gridDim.x * blockDim.x) >> 4) {
    const bool live = t < n_tiles;
    const int kb = live ? (int)(t / M) : 0, m = live ? (int)(t - (long long)kb * M) : 0;
    const long long col = (long long)kb * 128 + l * 8;
    float v[8];
    if (live) {
      load8(x + m * ldx + col, v);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.f;
    }
    float a = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) a = fmaxf(a, fabsf(v[j]));
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));
    const int e = fp8_scale_exp(a);
    if (!live) continue;
    *reinterpret_cast<uint2*>(q + m * ldq + col) = e4m3x8(v, ldexpf(1.f, -e));
    if (l == 0) s[(long long)kb * ld_s + m] = ldexpf(1.f, e);
  }
}

// One CTA per 128 x 128 block of W [N, K]: W codes, W^T codes (through shared memory) and the block's scale
// s[nb * ld_s + kb]. Runs once per matrix when the model loads.
__global__ void __launch_bounds__(256) quant_fp8_blocks_kernel(const bf16* __restrict__ w, long long ldw,
                                                               uint8_t* __restrict__ q, long long ldq,
                                                               uint8_t* __restrict__ qt, long long ldt,
                                                               float* __restrict__ s, long long ld_s) {
  __shared__ uint8_t tile[128][128 + 8];
  __shared__ float red[8];
  const int kb = blockIdx.x, nb = blockIdx.y, tid = threadIdx.x;
  const bf16* src = w + (long long)nb * 128 * ldw + kb * 128;
  float v[8][8];
  float a = 0.f;
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int idx = it * 256 + tid, row = idx >> 4, c8 = (idx & 15) * 8;
    load8(src + row * ldw + c8, v[it]);
#pragma unroll
    for (int j = 0; j < 8; ++j) a = fmaxf(a, fabsf(v[it][j]));
  }
  a = warp_max(a);
  if ((tid & 31) == 0) red[tid >> 5] = a;
  __syncthreads();
  a = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) a = fmaxf(a, red[i]);
  const int e = fp8_scale_exp(a);
  const float inv = ldexpf(1.f, -e);
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int idx = it * 256 + tid, row = idx >> 4, c8 = (idx & 15) * 8;
    const uint2 c = e4m3x8(v[it], inv);
    *reinterpret_cast<uint2*>(q + ((long long)nb * 128 + row) * ldq + kb * 128 + c8) = c;
    *reinterpret_cast<uint2*>(&tile[row][c8]) = c;
  }
  if (tid == 0) s[(long long)nb * ld_s + kb] = ldexpf(1.f, e);
  __syncthreads();
#pragma unroll
  for (int it = 0; it < 8; ++it) {        // W^T row kb*128 + k: 8 consecutive n per thread
    const int idx = it * 256 + tid, k = idx >> 4, n8 = (idx & 15) * 8;
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      lo |= (uint32_t)tile[n8 + j][k] << (8 * j);
      hi |= (uint32_t)tile[n8 + 4 + j][k] << (8 * j);
    }
    *reinterpret_cast<uint2*>(qt + ((long long)kb * 128 + k) * ldt + nb * 128 + n8) = make_uint2(lo, hi);
  }
}

static inline int grid_for(long long work_items, int threads, int max_blocks_per_sm = 8) {
  long long blocks = (work_items + threads - 1) / threads;
  long long cap = (long long)num_sms() * max_blocks_per_sm;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

}  // namespace b200

using namespace b200;
#define ST ((cudaStream_t)stream)

extern "C" int rlaifv_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int M, int H,
                                  float eps, void* stream) {
  B200_REQUIRE(H % 8 == 0 && M > 0, "rmsnorm_fwd: H %% 8 != 0 or M <= 0");
  const int grid = M < num_sms() * 8 ? M : num_sms() * 8;
  rmsnorm_fwd_kernel<<<grid, NORM_THREADS, 0, ST>>>((const bf16*)x, (const bf16*)w, (bf16*)y, rstd, M, H, eps);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// workspace: fp32 [rlaifv_rmsnorm_bwd_partials() * H]
extern "C" int rlaifv_rmsnorm_bwd_partials(void) { return num_sms() * 2; }
extern "C" int rlaifv_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd,
                                  const void* dres, void* dx, void* dw, int dw_accumulate,
                                  float* workspace, int M, int H, void* stream) {
  // Two chunks per thread cover H <= 4096 (LLaVA-1.5-7B, Mistral-7B); three cover H <= 6144 (LLaVA-1.5-13B: 5120).
  B200_REQUIRE(H % 8 == 0 && H <= NORM_THREADS * 8 * (NORM_MAXCH + 1) && M > 0,
               "rmsnorm_bwd: shape [%d,%d] unsupported", M, H);
  int grid = num_sms() * 2;
  if (grid > (M + 1) / 2) grid = (M + 1) / 2;
  if (H <= NORM_THREADS * 8 * NORM_MAXCH)
    rmsnorm_bwd_kernel<NORM_MAXCH><<<grid, NORM_THREADS, 0, ST>>>((const bf16*)dy, (const bf16*)x, (const bf16*)w,
                                                                 rstd, (const bf16*)dres, (bf16*)dx, workspace, M, H);
  else
    rmsnorm_bwd_kernel<NORM_MAXCH + 1><<<grid, NORM_THREADS, 0, ST>>>((const bf16*)dy, (const bf16*)x,
                                                                     (const bf16*)w, rstd, (const bf16*)dres,
                                                                     (bf16*)dx, workspace, M, H);
  B200_CHECK_CUDA(cudaGetLastError());
  reduce_partials_kernel<<<(H + 31) / 32, 256, 0, ST>>>(workspace, grid, H, (bf16*)dw, dw_accumulate);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int rlaifv_layernorm_fwd(const void* x, const void* w, const void* b, void* y, int M, int H,
                                    float eps, void* stream) {
  B200_REQUIRE(H % 8 == 0 && H <= NORM_THREADS * 8 * NORM_MAXCH && M > 0, "layernorm_fwd: shape [%d,%d] unsupported", M,
               H);
  const int grid = M < num_sms() * 8 ? M : num_sms() * 8;
  layernorm_fwd_kernel<<<grid, NORM_THREADS, 0, ST>>>((const bf16*)x, (const bf16*)w, (const bf16*)b,
                                                     (bf16*)y, M, H, eps);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// workspace: fp32 [2 * rlaifv_rmsnorm_bwd_partials() * H]; dw / db bf16 [H] (overwritten or accumulated)
extern "C" int rlaifv_layernorm_bwd(const void* dy, const void* x, const void* w, void* dx, void* dw, void* db,
                                    int accumulate, float* workspace, int M, int H, float eps, void* stream) {
  B200_REQUIRE(H % 8 == 0 && H <= NORM_THREADS * 8 * NORM_MAXCH && M > 0, "layernorm_bwd: shape [%d,%d] unsupported", M,
               H);
  int grid = num_sms() * 2;
  if (grid > M) grid = M;
  float* dbp = workspace + (long long)num_sms() * 2 * H;
  layernorm_bwd_kernel<<<grid, NORM_THREADS, 0, ST>>>((const bf16*)dy, (const bf16*)x, (const bf16*)w, (bf16*)dx,
                                                     workspace, dbp, M, H, eps);
  B200_CHECK_CUDA(cudaGetLastError());
  reduce_partials_kernel<<<(H + 31) / 32, 256, 0, ST>>>(workspace, grid, H, (bf16*)dw, accumulate);
  reduce_partials_kernel<<<(H + 31) / 32, 256, 0, ST>>>(dbp, grid, H, (bf16*)db, accumulate);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int rlaifv_add_rows_bcast(const void* x, const void* table, void* y, long long M, int P, int H,
                                     void* stream) {
  B200_REQUIRE(H % 8 == 0 && M > 0 && P > 0, "add_rows_bcast: bad shape");
  const long long total = M * (H / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > (long long)num_sms() * 16) blocks = (long long)num_sms() * 16;
  add_rows_bcast_kernel<<<(int)blocks, 256, 0, ST>>>((const bf16*)x, (const bf16*)table, (bf16*)y, M, P, H);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static int rope_fwd_impl(void* qkv, const void* cos_tab, const void* sin_tab, long long M, int T, int n_heads,
                         int n_kv_heads, int head_dim, long long ld, void* stream) {
  B200_REQUIRE(head_dim % 16 == 0, "rope: head_dim %% 16 != 0");
  const int nrot = n_heads + n_kv_heads;
  const long long total = M * nrot * (head_dim / 16);
  rope_fwd_kernel<<<grid_for(total, 256), 256, 0, ST>>>((bf16*)qkv, (const bf16*)cos_tab, (const bf16*)sin_tab,
                                                        M, T, nrot, head_dim, ld);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
static int rope_bwd_impl(void* dqkv, const float* dq_f32, const void* cos_tab, const void* sin_tab, long long M,
                         int T, int n_heads, int n_kv_heads, int head_dim, long long ld, void* stream) {
  B200_REQUIRE(head_dim % 16 == 0, "rope: head_dim %% 16 != 0");
  const long long total = M * (n_heads + n_kv_heads) * (head_dim / 16);
  rope_bwd_kernel<<<grid_for(total, 256), 256, 0, ST>>>((bf16*)dqkv, dq_f32, (const bf16*)cos_tab,
                                                        (const bf16*)sin_tab, M, T, n_heads, n_kv_heads, head_dim, ld);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_rope_fwd(void* qkv, const void* cos_tab, const void* sin_tab, long long M, int T,
                               int n_heads, int head_dim, long long ld, void* stream) {
  return rope_fwd_impl(qkv, cos_tab, sin_tab, M, T, n_heads, n_heads, head_dim, ld, stream);
}
extern "C" int rlaifv_rope_bwd(void* dqkv, const float* dq_f32, const void* cos_tab, const void* sin_tab,
                               long long M, int T, int n_heads, int head_dim, long long ld, void* stream) {
  return rope_bwd_impl(dqkv, dq_f32, cos_tab, sin_tab, M, T, n_heads, n_heads, head_dim, ld, stream);
}
// grouped-query layout: row = [q: n_heads*D | k: n_kv_heads*D | v: n_kv_heads*D]
extern "C" int rlaifv_rope_fwd_gqa(void* qkv, const void* cos_tab, const void* sin_tab, long long M, int T,
                                   int n_heads, int n_kv_heads, int head_dim, long long ld, void* stream) {
  return rope_fwd_impl(qkv, cos_tab, sin_tab, M, T, n_heads, n_kv_heads, head_dim, ld, stream);
}
extern "C" int rlaifv_rope_bwd_gqa(void* dqkv, const float* dq_f32, const void* cos_tab, const void* sin_tab,
                                   long long M, int T, int n_heads, int n_kv_heads, int head_dim, long long ld,
                                   void* stream) {
  return rope_bwd_impl(dqkv, dq_f32, cos_tab, sin_tab, M, T, n_heads, n_kv_heads, head_dim, ld, stream);
}

// RoPE of packed rows: the position of row m is pos[m] (int32 [M], device); backward in the split form only.
extern "C" int rlaifv_rope_pos_fwd(void* qkv, const void* cos_tab, const void* sin_tab, const int* pos, long long M,
                                   int n_heads, int n_kv_heads, int head_dim, long long ld, void* stream) {
  B200_REQUIRE(head_dim % 16 == 0 && M > 0, "rope_pos_fwd: head_dim %% 16 != 0 or M <= 0");
  const int nrot = n_heads + n_kv_heads;
  const long long total = M * nrot * (head_dim / 16);
  rope_pos_fwd_kernel<<<grid_for(total, 256), 256, 0, ST>>>((bf16*)qkv, (const bf16*)cos_tab, (const bf16*)sin_tab, pos,
                                                            M, nrot, head_dim, ld);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_rope_pos_bwd(void* dqkv, const void* cos_tab, const void* sin_tab, const int* pos, long long M,
                                   int n_heads, int n_kv_heads, int head_dim, long long ld, void* stream) {
  B200_REQUIRE(head_dim % 16 == 0 && M > 0, "rope_pos_bwd: head_dim %% 16 != 0 or M <= 0");
  const int nrot = n_heads + n_kv_heads;
  const long long total = M * nrot * (head_dim / 16);
  rope_pos_bwd_kernel<<<grid_for(total, 256), 256, 0, ST>>>((bf16*)dqkv, (const bf16*)cos_tab, (const bf16*)sin_tab, pos,
                                                            M, nrot, head_dim, ld);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int rlaifv_swiglu_fwd(const void* gu, void* act, long long M, int F, void* stream) {
  B200_REQUIRE(F % 8 == 0, "swiglu: F %% 8 != 0");
  swiglu_fwd_kernel<<<grid_for(M * (F / 8), 256), 256, 0, ST>>>((const bf16*)gu, (bf16*)act, M, F);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_swiglu_bwd(const void* gu, const void* dact, void* dgu, long long M, int F, void* stream) {
  B200_REQUIRE(F % 8 == 0, "swiglu: F %% 8 != 0");
  swiglu_bwd_kernel<<<grid_for(M * (F / 8), 256), 256, 0, ST>>>((const bf16*)gu, (const bf16*)dact, (bf16*)dgu, M, F);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_gelu_fwd(const void* pre, void* post, long long n, void* stream) {
  B200_REQUIRE(n % 8 == 0, "gelu_fwd: n %% 8 != 0");
  gelu_fwd_kernel<<<grid_for(n / 8, 256), 256, 0, ST>>>((const bf16*)pre, (bf16*)post, n / 8);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_gelu_bwd(const void* pre, const void* dpost, void* dpre, long long n, void* stream) {
  B200_REQUIRE(n % 8 == 0, "gelu_bwd: n %% 8 != 0");
  gelu_bwd_kernel<<<grid_for(n / 8, 256), 256, 0, ST>>>((const bf16*)pre, (const bf16*)dpost, (bf16*)dpre, n / 8);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
// bias gradient: db[N] (+)= column sums of x[M][N]; workspace fp32 [64*N]
extern "C" int rlaifv_colsum(const void* x, long long M, int N, void* db, int accumulate, float* workspace,
                             void* stream) {
  B200_REQUIRE(N % 2 == 0, "colsum: N odd");
  const int P = 64;
  dim3 grid((N / 2 + 127) / 128, P);
  colsum_kernel<<<grid, 128, 0, ST>>>((const bf16*)x, M, N, workspace);
  B200_CHECK_CUDA(cudaGetLastError());
  reduce_partials_kernel<<<(N + 31) / 32, 256, 0, ST>>>(workspace, P, N, (bf16*)db, accumulate);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int rlaifv_clip_im2col(const void* images, void* out, int n_img, int channels, int size, int patch,
                                  int k_pad, void* stream) {
  B200_REQUIRE(size % patch == 0 && k_pad >= channels * patch * patch, "im2col: bad geometry");
  const long long total = (long long)n_img * (size / patch) * (size / patch) * k_pad;
  im2col_patch_kernel<<<grid_for(total, 256), 256, 0, ST>>>((const bf16*)images, (bf16*)out, n_img, channels,
                                                            size, patch, k_pad);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_clip_embed(const void* patch, const void* cls, const void* pos, void* x, int n_img,
                                 int n_patch, int H, void* stream) {
  B200_REQUIRE(H % 8 == 0, "clip_embed: H %% 8 != 0");
  const long long total = (long long)n_img * (n_patch + 1) * (H / 8);
  clip_embed_kernel<<<grid_for(total, 256), 256, 0, ST>>>((const bf16*)patch, (const bf16*)cls, (const bf16*)pos,
                                                          (bf16*)x, n_img, n_patch, H);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_clip_drop_cls(const void* x, void* out, int n_img, int n_patch, int H, void* stream) {
  B200_REQUIRE(H % 8 == 0, "drop_cls: H %% 8 != 0");
  const long long total = (long long)n_img * n_patch * (H / 8);
  drop_cls_kernel<<<grid_for(total, 256), 256, 0, ST>>>((const bf16*)x, (bf16*)out, n_img, n_patch, H);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int rlaifv_splice_count(const long long* ids, int nseq, int L, int P, int max_len, int* n_img,
                                   int* len, void* stream) {
  splice_count_kernel<<<nseq, 32, 0, ST>>>(ids, nseq, L, P, max_len, n_img, len);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_splice_map(const long long* ids, const long long* labels, const int* n_img,
                                 const int* img_index, int nseq, int L, int P, int T, int max_len, int* src,
                                 long long* new_labels, void* stream) {
  splice_map_kernel<<<nseq, 32, 0, ST>>>(ids, labels, n_img, img_index, nseq, L, P, T, max_len, src, new_labels);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_splice_map_inplace(const long long* ids, const int* img_index, int nseq, int L, int num_query,
                                         long long im_patch, long long im_start, long long im_end, int* src,
                                         int* status, void* stream) {
  B200_REQUIRE(nseq > 0 && L > 0 && num_query > 0, "splice_map_inplace: bad shape");
  splice_map_inplace_kernel<<<1, 32, 0, ST>>>(ids, img_index, nseq, L, num_query, im_patch, im_start, im_end, src,
                                              status);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_splice_gather(const int* src, const long long* ids, const void* embed, const void* feat,
                                    void* out, int nseq, int L, int T, int H, void* stream) {
  B200_REQUIRE(H % 8 == 0, "splice_gather: H %% 8 != 0");
  const long long rows = (long long)nseq * T;
  splice_gather_kernel<<<grid_for(rows * 32, 256), 256, 0, ST>>>(src, ids, (const bf16*)embed, (const bf16*)feat,
                                                                 (bf16*)out, nseq, L, T, H);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_splice_scatter(const int* src, const long long* ids, const void* dx, float* d_embed,
                                     float* d_feat, int nseq, int L, int T, int H, void* stream) {
  B200_REQUIRE(H % 8 == 0, "splice_scatter: H %% 8 != 0");
  const long long rows = (long long)nseq * T;
  splice_scatter_kernel<<<grid_for(rows * 32, 256), 256, 0, ST>>>(src, ids, (const bf16*)dx, d_embed, d_feat,
                                                                  nseq, L, T, H);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_f32_to_bf16(const float* in, void* out, long long n, int accumulate, void* stream) {
  B200_REQUIRE(n % 8 == 0, "f32_to_bf16: n %% 8 != 0");
  f32_to_bf16_kernel<<<grid_for(n / 8, 256), 256, 0, ST>>>(in, (bf16*)out, n / 8, accumulate);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int rlaifv_f32_to_bf16_2d(const float* in, long long ld_in, void* out, long long ld_out, long long rows,
                                     int cols, int accumulate, void* stream) {
  B200_REQUIRE(cols % 8 == 0 && ld_in % 4 == 0 && ld_out % 8 == 0 && rows > 0, "f32_to_bf16_2d: bad shape");
  f32_to_bf16_2d_kernel<<<grid_for(rows * (cols / 8), 256), 256, 0, ST>>>(in, ld_in, (bf16*)out, ld_out, rows,
                                                                         cols / 8, accumulate);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int rlaifv_splice_token_weight(const int* src, const float* token_weight, float* out, int nseq, int Lw, int T,
                                          void* stream) {
  B200_REQUIRE(nseq > 0 && Lw > 0 && T >= 2, "splice_token_weight: bad shape");
  splice_token_weight_kernel<<<grid_for((long long)nseq * (T - 1), 256), 256, 0, ST>>>(src, token_weight, out, nseq, Lw, T);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
// ---- compact lm_head (supervised positions only) ----
extern "C" int rlaifv_supervised_rows(const long long* labels, int nseq, int T, int cap, int* row_pos, void* stream) {
  B200_REQUIRE(nseq > 0 && T >= 2 && cap > 0, "supervised_rows: bad shape");
  B200_REQUIRE((long long)nseq * T < 2147483647LL, "supervised_rows: nseq*T overflows int32");
  supervised_rows_kernel<<<nseq, 32, 0, ST>>>(labels, nseq, T, cap, row_pos);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_rows_gather(const int* row_pos, const void* x, void* out, long long n_rows, int H, void* stream) {
  B200_REQUIRE(H % 8 == 0 && n_rows > 0, "rows_gather: bad shape");
  rows_gather_kernel<<<grid_for(n_rows * (H / 8), 256), 256, 0, ST>>>(row_pos, (const bf16*)x, (bf16*)out, n_rows, H / 8);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_rows_scatter(const int* row_pos, const void* dy, void* dx, long long n_rows, int H, void* stream) {
  B200_REQUIRE(H % 8 == 0 && n_rows > 0, "rows_scatter: bad shape");
  rows_scatter_kernel<<<grid_for(n_rows * (H / 8), 256), 256, 0, ST>>>(row_pos, (const bf16*)dy, (bf16*)dx, n_rows, H / 8);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
// row_pos NULL: dense logits [nseq*T][ld], lse [nseq][T]. Otherwise the compact rows: logits [n_rows][ld], lse
// [n_rows], and per_tok [nseq][T-1] must be zero-filled by the caller (unsupervised positions stay 0).
extern "C" int rlaifv_logp_fwd(const void* logits, long long ld, const long long* labels, const int* row_pos,
                               long long n_rows, int nseq, int T, int V, float* per_tok, float* lse,
                               float* logp_sum, float* logp_avg, float* count, void* stream) {
  B200_REQUIRE(V % 8 == 0 && T >= 2, "logp_fwd: V %% 8 != 0 or T < 2");
  B200_REQUIRE(!row_pos || n_rows > 0, "logp_fwd: n_rows <= 0 with row_pos");
  const long long rows = row_pos ? n_rows : (long long)nseq * (T - 1);
  const int grid = (int)(rows < (long long)num_sms() * 8 ? rows : (long long)num_sms() * 8);
  logp_fwd_kernel<<<grid, LOGP_THREADS, 0, ST>>>((const bf16*)logits, ld, labels, nseq, T, V, per_tok, lse, row_pos,
                                                 n_rows);
  B200_CHECK_CUDA(cudaGetLastError());
  logp_reduce_kernel<<<nseq, 256, 0, ST>>>(per_tok, labels, nullptr, nseq, T, logp_sum, logp_avg, count);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
// in place: d loss / d logits, on the dense (row_pos NULL) or the compact logits. token_weight (nullable) [nseq][T-1];
// norm (nullable) [nseq] = label count (average mode) or weight sum (weighted average mode).
extern "C" int rlaifv_logp_bwd(void* logits, long long ld, const long long* labels, const int* row_pos,
                               long long n_rows, const float* lse, const float* d_logp, const float* token_weight,
                               const float* norm, int nseq, int T, int V, void* stream) {
  B200_REQUIRE(V % 8 == 0, "logp_bwd: V %% 8 != 0");
  B200_REQUIRE(!row_pos || n_rows > 0, "logp_bwd: n_rows <= 0 with row_pos");
  const long long rows = row_pos ? n_rows : (long long)nseq * T;
  const int grid = (int)(rows < (long long)num_sms() * 8 ? rows : (long long)num_sms() * 8);
  logp_bwd_kernel<<<grid, LOGP_THREADS, 0, ST>>>((bf16*)logits, ld, labels, lse, d_logp, token_weight, norm, nseq, T,
                                                 V, row_pos, n_rows);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_logp_weighted_reduce(const float* per_tok, const long long* labels, const float* token_weight,
                                           int nseq, int T, float* logp_w, float* avg_w, float* wsum_or_null,
                                           void* stream) {
  B200_REQUIRE(nseq > 0 && T >= 2, "logp_weighted_reduce: bad shape");
  logp_reduce_kernel<<<nseq, 256, 0, ST>>>(per_tok, labels, token_weight, nseq, T, logp_w, avg_w, wsum_or_null);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int rlaifv_dpo_loss(const float* policy_win, const float* policy_rej, const float* ref_win,
                               const float* ref_rej, int B, float beta, float dpo_weight, float sft_weight,
                               float grad_scale, float* losses, float* chosen_rewards, float* rejected_rewards,
                               float* d_policy_win, float* d_policy_rej, float* out9, void* stream) {
  B200_REQUIRE(B > 0, "dpo_loss: B <= 0");
  dpo_loss_kernel<<<1, 32, 0, ST>>>(policy_win, policy_rej, ref_win, ref_rej, B, beta, dpo_weight, sft_weight,
                                    grad_scale, losses, chosen_rewards, rejected_rewards, d_policy_win,
                                    d_policy_rej, out9);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int rlaifv_adamw_step(float* master, float* exp_avg, float* exp_avg_sq, const void* grad,
                                 int grad_is_f32, void* param_bf16, long long n, float lr, float beta1,
                                 float beta2, float eps, float weight_decay, int step, float grad_scale,
                                 void* stream) {
  B200_REQUIRE(n % 4 == 0 && step >= 1, "adamw: n %% 4 != 0 or step < 1");
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2_sqrt = sqrtf(1.f - powf(beta2, (float)step));
  const int grid = grid_for(n / 4, 256, 16);
  if (grad_is_f32)
    adamw_kernel<true><<<grid, 256, 0, ST>>>(master, exp_avg, exp_avg_sq, grad, (bf16*)param_bf16, n, lr, beta1,
                                             beta2, eps, weight_decay, bc1, bc2_sqrt, grad_scale);
  else
    adamw_kernel<false><<<grid, 256, 0, ST>>>(master, exp_avg, exp_avg_sq, grad, (bf16*)param_bf16, n, lr, beta1,
                                              beta2, eps, weight_decay, bc1, bc2_sqrt, grad_scale);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ---- AdamW over state streamed from pinned host memory ----------------------------------------------------------------
// Per (device, ring), one event triple per ring slot: slot s is loaded (H2D done), updated (kernel done), stored (D2H
// done). The events outlive a call, so the first load into a slot in the next call (the next bucket) waits for the last
// store out of it in this one, and the slot rotation carries on from call to call. They are created on a ring's first
// call and destroyed by rlaifv_adamw_offload_release(ring), which the owner of the ring calls before freeing it.
static constexpr int kOffloadMaxSlots = 8;
struct OffloadEvents {
  cudaEvent_t loaded[kOffloadMaxSlots] = {}, updated[kOffloadMaxSlots] = {}, stored[kOffloadMaxSlots] = {};
  int next_slot = 0;
  bool ready = false;
};
static std::mutex g_offload_mu;
static std::map<std::pair<int, const void*>, OffloadEvents> g_offload_pool;

static void destroy_offload_events(OffloadEvents& e) {
  for (int s = 0; s < kOffloadMaxSlots; ++s)
    for (cudaEvent_t* ev : {&e.loaded[s], &e.updated[s], &e.stored[s]})
      if (*ev) {
        cudaEventDestroy(*ev);
        *ev = nullptr;
      }
  e.ready = false;
}

static int offload_events(const void* ring, OffloadEvents** out) {
  int dev = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(g_offload_mu);
  OffloadEvents& e = g_offload_pool[std::make_pair(dev, ring)];
  if (!e.ready) {
    cudaError_t err = cudaSuccess;
    for (int s = 0; s < kOffloadMaxSlots && err == cudaSuccess; ++s) {
      err = cudaEventCreateWithFlags(&e.loaded[s], cudaEventDisableTiming);
      if (err == cudaSuccess) err = cudaEventCreateWithFlags(&e.updated[s], cudaEventDisableTiming);
      if (err == cudaSuccess) err = cudaEventCreateWithFlags(&e.stored[s], cudaEventDisableTiming);
    }
    if (err != cudaSuccess) {
      destroy_offload_events(e);
      g_offload_pool.erase(std::make_pair(dev, ring));
      B200_CHECK_CUDA(err);
    }
    e.ready = true;
  }
  *out = &e;
  return 0;
}

// `what` must lie in memory of type `want` over its whole [p, p + bytes) (both ends checked).
static int require_memory_type(const void* p, size_t bytes, cudaMemoryType want, const char* what) {
  const char* kind = want == cudaMemoryTypeHost ? "pinned host" : "device";
  B200_REQUIRE(p != nullptr, "adamw_offload: %s is NULL", what);
  const void* ends[2] = {p, (const char*)p + bytes - 1};
  for (const void* q : ends) {
    cudaPointerAttributes a;
    cudaError_t err = cudaPointerGetAttributes(&a, q);
    if (err != cudaSuccess) {
      cudaGetLastError();                 // clear it, so that the next launch's check does not report it
      b200::set_last_error("adamw_offload: %s %p: cudaPointerGetAttributes -> %s", what, q, cudaGetErrorString(err));
      return -1;
    }
    B200_REQUIRE(a.type == want, "adamw_offload: %s (%p, %zu bytes) must be %s memory (cudaMemoryType %d)", what, q,
                 bytes, kind, (int)a.type);
  }
  return 0;
}

// The chunk / slot / event rotation of both offloaded optimizers. [0, n) is cut into chunks of slot_elems (the last one
// shorter); chunk i takes the next slot s of the ring's rotation: load(s, off, c, h2d) enqueues its H2D copies on h2d
// after the slot's previous store, update(s, off, c) its kernel on cs once they are done, store(s, off, c, d2h) its D2H
// copies on d2h once that is done. The streams run up to n_slots chunks apart, so with 3 slots the load of chunk i+1,
// the update of chunk i and the store of chunk i-1 overlap. Each callback returns 0 or the entry point's error code.
template <class Load, class Update, class Store>
static int offload_pipeline(const void* ring, int n_slots, long long n, long long slot_elems, cudaStream_t hs,
                            cudaStream_t cs, cudaStream_t ds, Load load, Update update, Store store) {
  OffloadEvents* ev = nullptr;
  int rc;
  if ((rc = offload_events(ring, &ev)) != 0) return rc;
  for (long long off = 0; off < n; off += slot_elems) {
    const long long c = n - off < slot_elems ? n - off : slot_elems;
    const int s = ev->next_slot % n_slots;
    ev->next_slot = (s + 1) % n_slots;
    B200_CHECK_CUDA(cudaStreamWaitEvent(hs, ev->stored[s], 0));
    if ((rc = load(s, off, c, hs)) != 0) return rc;
    B200_CHECK_CUDA(cudaEventRecord(ev->loaded[s], hs));
    B200_CHECK_CUDA(cudaStreamWaitEvent(cs, ev->loaded[s], 0));
    if ((rc = update(s, off, c)) != 0) return rc;
    B200_CHECK_CUDA(cudaEventRecord(ev->updated[s], cs));
    B200_CHECK_CUDA(cudaStreamWaitEvent(ds, ev->updated[s], 0));
    if ((rc = store(s, off, c, ds)) != 0) return rc;
    B200_CHECK_CUDA(cudaEventRecord(ev->stored[s], ds));
  }
  return 0;
}

extern "C" int rlaifv_adamw_offload_bucket(float* host_master, float* host_exp_avg, float* host_exp_avg_sq,
                                           const void* grad, void* param_bf16, long long n, long long decay_n,
                                           float* ring, int n_slots, long long slot_elems, float lr, float beta1,
                                           float beta2, float eps, float weight_decay, int step, void* stream,
                                           void* h2d_stream, void* d2h_stream) {
  B200_REQUIRE(n > 0 && n % 4 == 0 && step >= 1, "adamw_offload: n <= 0, n %% 4 != 0 or step < 1");
  B200_REQUIRE(decay_n >= 0 && decay_n <= n, "adamw_offload: decay_n %lld outside [0, %lld]", decay_n, n);
  B200_REQUIRE(n_slots >= 2 && n_slots <= kOffloadMaxSlots, "adamw_offload: n_slots %d outside [2, %d]", n_slots,
               kOffloadMaxSlots);
  B200_REQUIRE(slot_elems > 0 && slot_elems % 4 == 0, "adamw_offload: slot_elems %lld not a positive multiple of 4",
               slot_elems);
  B200_REQUIRE(((uintptr_t)grad & 7) == 0 && ((uintptr_t)param_bf16 & 7) == 0 && ((uintptr_t)ring & 15) == 0,
               "adamw_offload: grad / param not 8-byte or ring not 16-byte aligned");
  const size_t state_bytes = (size_t)n * sizeof(float);
  int rc;
  if ((rc = require_memory_type(host_master, state_bytes, cudaMemoryTypeHost, "host_master")) != 0) return rc;
  if ((rc = require_memory_type(host_exp_avg, state_bytes, cudaMemoryTypeHost, "host_exp_avg")) != 0) return rc;
  if ((rc = require_memory_type(host_exp_avg_sq, state_bytes, cudaMemoryTypeHost, "host_exp_avg_sq")) != 0) return rc;
  if ((rc = require_memory_type(grad, (size_t)n * 2, cudaMemoryTypeDevice, "grad")) != 0) return rc;
  if ((rc = require_memory_type(param_bf16, (size_t)n * 2, cudaMemoryTypeDevice, "param_bf16")) != 0) return rc;
  if ((rc = require_memory_type(ring, (size_t)n_slots * 3 * slot_elems * sizeof(float), cudaMemoryTypeDevice,
                                "ring")) != 0)
    return rc;
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2_sqrt = sqrtf(1.f - powf(beta2, (float)step));
  cudaStream_t cs = (cudaStream_t)stream;
  const bf16* g = (const bf16*)grad;
  bf16* p = (bf16*)param_bf16;
  auto slot = [&](int s) { return ring + (size_t)s * 3 * slot_elems; };     // master | m | v
  auto load = [&](int s, long long off, long long c, cudaStream_t hs) -> int {
    const size_t cb = (size_t)c * sizeof(float);
    B200_CHECK_CUDA(cudaMemcpyAsync(slot(s), host_master + off, cb, cudaMemcpyHostToDevice, hs));
    B200_CHECK_CUDA(cudaMemcpyAsync(slot(s) + slot_elems, host_exp_avg + off, cb, cudaMemcpyHostToDevice, hs));
    B200_CHECK_CUDA(cudaMemcpyAsync(slot(s) + 2 * slot_elems, host_exp_avg_sq + off, cb, cudaMemcpyHostToDevice, hs));
    return 0;
  };
  auto update = [&](int s, long long off, long long c) -> int {
    long long dn = decay_n - off;
    dn = dn < 0 ? 0 : (dn > c ? c : dn);
    adamw_staged_kernel<<<grid_for(c / 4, 256, 16), 256, 0, cs>>>(slot(s), slot(s) + slot_elems,
                                                                   slot(s) + 2 * slot_elems, g + off, p + off, c, dn,
                                                                   lr, beta1, beta2, eps, weight_decay, bc1, bc2_sqrt);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
  };
  auto store = [&](int s, long long off, long long c, cudaStream_t ds) -> int {
    const size_t cb = (size_t)c * sizeof(float);
    B200_CHECK_CUDA(cudaMemcpyAsync(host_master + off, slot(s), cb, cudaMemcpyDeviceToHost, ds));
    B200_CHECK_CUDA(cudaMemcpyAsync(host_exp_avg + off, slot(s) + slot_elems, cb, cudaMemcpyDeviceToHost, ds));
    B200_CHECK_CUDA(cudaMemcpyAsync(host_exp_avg_sq + off, slot(s) + 2 * slot_elems, cb, cudaMemcpyDeviceToHost, ds));
    return 0;
  };
  return offload_pipeline(ring, n_slots, n, slot_elems, (cudaStream_t)h2d_stream, cs, (cudaStream_t)d2h_stream, load,
                          update, store);
}

// Byte size of one ring slot of the 8-bit offloaded optimizer for slot_elems (% 256 == 0) elements: master (fp32) |
// code_m | code_v (uint8) | absmax_m | absmax_v (fp32, one per 256 elements), rounded up to 256 bytes so that every
// slot starts 256-byte aligned. zero2.adamw8bit_slot_bytes sizes the ring by the same formula.
static inline size_t adamw8bit_slot_bytes(long long slot_elems) {
  const size_t raw = (size_t)slot_elems * 6 + (size_t)(slot_elems / kQBlock) * 2 * sizeof(float);
  return (raw + 255) / 256 * 256;
}

extern "C" int rlaifv_adamw8bit_step(float* master, uint8_t* code_m, uint8_t* code_v, float* absmax_m,
                                     float* absmax_v, const void* grad, void* param_bf16, long long n,
                                     long long decay_n, const float* map_m, const float* map_v, float lr, float beta1,
                                     float beta2, float eps, float weight_decay, int step, void* stream) {
  B200_REQUIRE(n > 0 && n % 8 == 0 && step >= 1, "adamw8bit: n <= 0, n %% 8 != 0 or step < 1");
  B200_REQUIRE(decay_n >= 0 && decay_n <= n, "adamw8bit: decay_n %lld outside [0, %lld]", decay_n, n);
  B200_REQUIRE(((uintptr_t)master & 15) == 0 && ((uintptr_t)grad & 15) == 0 && ((uintptr_t)param_bf16 & 15) == 0 &&
                   ((uintptr_t)code_m & 7) == 0 && ((uintptr_t)code_v & 7) == 0 && ((uintptr_t)absmax_m & 3) == 0 &&
                   ((uintptr_t)absmax_v & 3) == 0,
               "adamw8bit: master / grad / param not 16-byte, codes not 8-byte or absmax not 4-byte aligned");
  B200_REQUIRE(map_m != nullptr && map_v != nullptr, "adamw8bit: map_m / map_v is NULL");
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2_sqrt = sqrtf(1.f - powf(beta2, (float)step));
  adamw8bit_kernel<<<grid_for((n + kQBlock - 1) / kQBlock, 8, 8), 256, 0, ST>>>(
      master, code_m, code_v, absmax_m, absmax_v, (const bf16*)grad, (bf16*)param_bf16, n, decay_n, map_m, map_v, lr,
      beta1, beta2, eps, weight_decay, bc1, bc2_sqrt);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int rlaifv_adamw8bit_offload_bucket(float* host_master, uint8_t* host_code_m, uint8_t* host_code_v,
                                               float* host_absmax_m, float* host_absmax_v, const void* grad,
                                               void* param_bf16, long long n, long long decay_n, const float* map_m,
                                               const float* map_v, void* ring, int n_slots, long long slot_elems,
                                               float lr, float beta1, float beta2, float eps, float weight_decay,
                                               int step, void* stream, void* h2d_stream, void* d2h_stream) {
  B200_REQUIRE(n > 0 && n % 8 == 0 && step >= 1, "adamw8bit_offload: n <= 0, n %% 8 != 0 or step < 1");
  B200_REQUIRE(decay_n >= 0 && decay_n <= n, "adamw8bit_offload: decay_n %lld outside [0, %lld]", decay_n, n);
  B200_REQUIRE(n_slots >= 2 && n_slots <= kOffloadMaxSlots, "adamw8bit_offload: n_slots %d outside [2, %d]", n_slots,
               kOffloadMaxSlots);
  B200_REQUIRE(slot_elems > 0 && slot_elems % kQBlock == 0,
               "adamw8bit_offload: slot_elems %lld not a positive multiple of 256", slot_elems);
  B200_REQUIRE(((uintptr_t)grad & 15) == 0 && ((uintptr_t)param_bf16 & 15) == 0 && ((uintptr_t)ring & 255) == 0,
               "adamw8bit_offload: grad / param not 16-byte or ring not 256-byte aligned");
  const long long nblk = (n + kQBlock - 1) / kQBlock;
  const size_t slot_bytes = adamw8bit_slot_bytes(slot_elems);
  int rc;
  if ((rc = require_memory_type(host_master, (size_t)n * 4, cudaMemoryTypeHost, "host_master")) != 0) return rc;
  if ((rc = require_memory_type(host_code_m, (size_t)n, cudaMemoryTypeHost, "host_code_m")) != 0) return rc;
  if ((rc = require_memory_type(host_code_v, (size_t)n, cudaMemoryTypeHost, "host_code_v")) != 0) return rc;
  if ((rc = require_memory_type(host_absmax_m, (size_t)nblk * 4, cudaMemoryTypeHost, "host_absmax_m")) != 0) return rc;
  if ((rc = require_memory_type(host_absmax_v, (size_t)nblk * 4, cudaMemoryTypeHost, "host_absmax_v")) != 0) return rc;
  if ((rc = require_memory_type(grad, (size_t)n * 2, cudaMemoryTypeDevice, "grad")) != 0) return rc;
  if ((rc = require_memory_type(param_bf16, (size_t)n * 2, cudaMemoryTypeDevice, "param_bf16")) != 0) return rc;
  if ((rc = require_memory_type(map_m, kQBlock * 4, cudaMemoryTypeDevice, "map_m")) != 0) return rc;
  if ((rc = require_memory_type(map_v, kQBlock * 4, cudaMemoryTypeDevice, "map_v")) != 0) return rc;
  if ((rc = require_memory_type(ring, (size_t)n_slots * slot_bytes, cudaMemoryTypeDevice, "ring")) != 0) return rc;

  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2_sqrt = sqrtf(1.f - powf(beta2, (float)step));
  cudaStream_t cs = (cudaStream_t)stream;
  const bf16* g = (const bf16*)grad;
  bf16* p = (bf16*)param_bf16;
  // slot s: master | code_m | code_v | absmax_m | absmax_v (adamw8bit_slot_bytes). Chunks start at multiples of
  // slot_elems, so on block edges, and chunk blocks are the bucket's blocks [off / 256, off / 256 + ceil(c / 256)).
  struct Slot {
    float* master;
    uint8_t *qm, *qv;
    float *am, *av;
  };
  auto slot = [&](int s) {
    uint8_t* base = (uint8_t*)ring + (size_t)s * slot_bytes;
    Slot t;
    t.master = (float*)base;
    t.qm = base + (size_t)slot_elems * 4;
    t.qv = t.qm + slot_elems;
    t.am = (float*)(t.qv + slot_elems);
    t.av = t.am + slot_elems / kQBlock;
    return t;
  };
  auto load = [&](int s, long long off, long long c, cudaStream_t hs) -> int {
    const Slot t = slot(s);
    const long long b0 = off / kQBlock, nb = (c + kQBlock - 1) / kQBlock;
    B200_CHECK_CUDA(cudaMemcpyAsync(t.master, host_master + off, (size_t)c * 4, cudaMemcpyHostToDevice, hs));
    B200_CHECK_CUDA(cudaMemcpyAsync(t.qm, host_code_m + off, (size_t)c, cudaMemcpyHostToDevice, hs));
    B200_CHECK_CUDA(cudaMemcpyAsync(t.qv, host_code_v + off, (size_t)c, cudaMemcpyHostToDevice, hs));
    B200_CHECK_CUDA(cudaMemcpyAsync(t.am, host_absmax_m + b0, (size_t)nb * 4, cudaMemcpyHostToDevice, hs));
    B200_CHECK_CUDA(cudaMemcpyAsync(t.av, host_absmax_v + b0, (size_t)nb * 4, cudaMemcpyHostToDevice, hs));
    return 0;
  };
  auto update = [&](int s, long long off, long long c) -> int {
    const Slot t = slot(s);
    long long dn = decay_n - off;
    dn = dn < 0 ? 0 : (dn > c ? c : dn);
    adamw8bit_kernel<<<grid_for((c + kQBlock - 1) / kQBlock, 8, 8), 256, 0, cs>>>(
        t.master, t.qm, t.qv, t.am, t.av, g + off, p + off, c, dn, map_m, map_v, lr, beta1, beta2, eps, weight_decay,
        bc1, bc2_sqrt);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
  };
  auto store = [&](int s, long long off, long long c, cudaStream_t ds) -> int {
    const Slot t = slot(s);
    const long long b0 = off / kQBlock, nb = (c + kQBlock - 1) / kQBlock;
    B200_CHECK_CUDA(cudaMemcpyAsync(host_master + off, t.master, (size_t)c * 4, cudaMemcpyDeviceToHost, ds));
    B200_CHECK_CUDA(cudaMemcpyAsync(host_code_m + off, t.qm, (size_t)c, cudaMemcpyDeviceToHost, ds));
    B200_CHECK_CUDA(cudaMemcpyAsync(host_code_v + off, t.qv, (size_t)c, cudaMemcpyDeviceToHost, ds));
    B200_CHECK_CUDA(cudaMemcpyAsync(host_absmax_m + b0, t.am, (size_t)nb * 4, cudaMemcpyDeviceToHost, ds));
    B200_CHECK_CUDA(cudaMemcpyAsync(host_absmax_v + b0, t.av, (size_t)nb * 4, cudaMemcpyDeviceToHost, ds));
    return 0;
  };
  return offload_pipeline(ring, n_slots, n, slot_elems, (cudaStream_t)h2d_stream, cs, (cudaStream_t)d2h_stream, load,
                          update, store);
}

extern "C" int rlaifv_adamw_offload_release(const void* ring) {
  int dev = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(g_offload_mu);
  auto it = g_offload_pool.find(std::make_pair(dev, ring));
  if (it != g_offload_pool.end()) {
    destroy_offload_events(it->second);
    g_offload_pool.erase(it);
  }
  return 0;
}

static inline uint32_t dropout_threshold(float p) {
  double t = (double)p * 4294967296.0;
  if (t < 0) t = 0;
  if (t > 4294967295.0) t = 4294967295.0;
  return (uint32_t)t;
}
extern "C" int rlaifv_dropout_fwd(const void* x, void* out, long long n, float p, unsigned long long seed, void* stream) {
  B200_REQUIRE(n % 8 == 0 && p >= 0.f && p < 1.f, "dropout_fwd: n %% 8 != 0 or p outside [0,1)");
  dropout_fwd_kernel<<<grid_for(n / 8, 256), 256, 0, ST>>>((const bf16*)x, (bf16*)out, n / 8, dropout_threshold(p),
                                                           1.f / (1.f - p), seed);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_dropout_bwd_add(void* dx, const void* g, long long n, float p, unsigned long long seed, void* stream) {
  B200_REQUIRE(n % 8 == 0 && p >= 0.f && p < 1.f, "dropout_bwd_add: n %% 8 != 0 or p outside [0,1)");
  dropout_bwd_add_kernel<<<grid_for(n / 8, 256), 256, 0, ST>>>((bf16*)dx, (const bf16*)g, n / 8, dropout_threshold(p),
                                                               1.f / (1.f - p), seed);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_dropout_rows_fwd(const void* x, void* out, const int* rows, long long n_rows, int width, float p,
                                       unsigned long long seed, void* stream) {
  B200_REQUIRE(width % 8 == 0 && n_rows > 0 && p >= 0.f && p < 1.f, "dropout_rows_fwd: width %% 8 != 0 or bad p");
  dropout_rows_kernel<<<grid_for(n_rows * (width / 8), 256), 256, 0, ST>>>(
      (const bf16*)x, nullptr, (bf16*)out, rows, n_rows, width / 8, dropout_threshold(p), 1.f / (1.f - p), seed);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int rlaifv_dropout_rows_bwd_add(void* dx, const void* g, const int* rows, long long n_rows, int width,
                                           float p, unsigned long long seed, void* stream) {
  B200_REQUIRE(width % 8 == 0 && n_rows > 0 && p >= 0.f && p < 1.f, "dropout_rows_bwd_add: width %% 8 != 0 or bad p");
  dropout_rows_kernel<<<grid_for(n_rows * (width / 8), 256), 256, 0, ST>>>(
      (const bf16*)dx, (const bf16*)g, (bf16*)dx, rows, n_rows, width / 8, dropout_threshold(p), 1.f / (1.f - p), seed);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int rlaifv_quant_fp8_rows(const void* x, long long ldx, void* q, long long ldq, float* s, long long ld_s,
                                     int M, int K, void* stream) {
  B200_REQUIRE(x && q && s, "quant_fp8_rows: null pointer");
  B200_REQUIRE(M > 0 && K > 0 && K % 128 == 0, "quant_fp8_rows: K (%d) must be a positive multiple of 128", K);
  B200_REQUIRE(ldx >= K && ldx % 8 == 0 && ((uintptr_t)x & 15) == 0,
               "quant_fp8_rows: x must be 16-byte aligned with a row stride (%lld) >= K, multiple of 8", ldx);
  B200_REQUIRE(ldq >= K && ldq % 16 == 0 && ((uintptr_t)q & 15) == 0,
               "quant_fp8_rows: codes must be 16-byte aligned with a row stride (%lld) >= K, multiple of 16", ldq);
  B200_REQUIRE(ld_s >= M && ld_s % 4 == 0 && ((uintptr_t)s & 15) == 0,
               "quant_fp8_rows: scales need ld_s (%lld) >= M (%d), a multiple of 4, 16-byte aligned", ld_s, M);
  const long long threads = (long long)M * (K / 128) * 16;
  quant_fp8_rows_kernel<<<grid_for(threads, 256), 256, 0, ST>>>((const bf16*)x, ldx, (uint8_t*)q, ldq, s, ld_s, M,
                                                                 K / 128);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int rlaifv_quant_fp8_blocks(const void* w, long long ldw, void* q, long long ldq, void* qt, long long ldt,
                                       float* s, long long ld_s, int N, int K, void* stream) {
  B200_REQUIRE(w && q && qt && s, "quant_fp8_blocks: null pointer");
  B200_REQUIRE(N > 0 && K > 0 && N % 128 == 0 && K % 128 == 0,
               "quant_fp8_blocks: N (%d) and K (%d) must be positive multiples of 128", N, K);
  B200_REQUIRE(ldw >= K && ldw % 8 == 0 && ((uintptr_t)w & 15) == 0,
               "quant_fp8_blocks: W must be 16-byte aligned with a row stride (%lld) >= K, multiple of 8", ldw);
  B200_REQUIRE(ldq >= K && ldq % 8 == 0 && ((uintptr_t)q & 7) == 0 && ldt >= N && ldt % 8 == 0 &&
                   ((uintptr_t)qt & 7) == 0,
               "quant_fp8_blocks: code buffers must be 8-byte aligned, row strides multiples of 8 covering K / N");
  B200_REQUIRE(ld_s >= K / 128, "quant_fp8_blocks: ld_s (%lld) < K / 128", ld_s);
  quant_fp8_blocks_kernel<<<dim3(K / 128, N / 128), 256, 0, ST>>>((const bf16*)w, ldw, (uint8_t*)q, ldq,
                                                                   (uint8_t*)qt, ldt, s, ld_s);
  B200_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// Host-side helpers shared by the launchers: error reporting for the C ABI and TMA tensor-map
// construction (cuTensorMapEncodeTiled resolved at run time through the CUDA runtime so the
// library has no link-time dependency on libcuda and loads on a CPU-only box).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace b200 {

void set_last_error(const char* fmt, ...);
int num_sms();   // of the CURRENT device (cached per device)
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (device, kernel): the attribute is per device, so a
// process that drives several devices must set it on each of them
cudaError_t configure_smem_once(const void* func, int bytes);

#define B200_CHECK_CUDA(expr)                                                         \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess) {                                                          \
      b200::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,              \
                           cudaGetErrorString(_e));                                   \
      return -2;                                                                      \
    }                                                                                 \
  } while (0)

#define B200_REQUIRE(cond, ...)              \
  do {                                       \
    if (!(cond)) {                           \
      b200::set_last_error(__VA_ARGS__);     \
      return -1;                             \
    }                                        \
  } while (0)

// bf16 tensor map, SWIZZLE_128B. `rank` 2 or 3. dims/box are innermost-first, strides_bytes has
// rank-1 entries (stride of dim 1, dim 2). Returns 0 on success.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box);
// The same for one-byte elements (FP8 e4m3 codes): dims and box count bytes.
int make_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_bytes, const uint32_t* box);

}  // namespace b200

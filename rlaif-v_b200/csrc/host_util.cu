#include "host_util.h"

#include <stdarg.h>
#include <string.h>

#include <mutex>
#include <set>
#include <utility>

namespace b200 {

static thread_local char g_last_error[1024] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}
const char* get_last_error() { return g_last_error; }

int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  const int slot = (dev >= 0 && dev < 64) ? dev : 0;
  if (cached[slot] <= 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 148;
    cached[slot] = n;
  }
  return cached[slot];
}

cudaError_t configure_smem_once(const void* func, int bytes) {
  static std::mutex mu;
  static std::set<std::pair<int, const void*>> done;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(mu);
  const std::pair<int, const void*> key(dev, func);
  if (done.count(key)) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) done.insert(key);
  return e;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn resolve_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) {
    set_last_error("cuTensorMapEncodeTiled not available from the driver (%s)",
                   cudaGetErrorString(e));
    return nullptr;
  }
  fn = (EncodeTiledFn)p;
  return fn;
}

static int make_tmap(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box) {
  EncodeTiledFn fn = resolve_encode();
  if (!fn) return -3;
  cuuint64_t gdims[5];
  cuuint64_t gstr[5];
  cuuint32_t gbox[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdims[i] = dims[i];
    gbox[i] = box[i];
    estr[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  if (((uintptr_t)base & 15) != 0) {
    set_last_error("tensor map base %p not 16-byte aligned", base);
    return -1;
  }
  for (int i = 0; i + 1 < rank; ++i) {
    if (gstr[i] % 16 != 0) {
      set_last_error("tensor map stride %llu not a multiple of 16 bytes",
                     (unsigned long long)gstr[i]);
      return -1;
    }
  }
  CUresult r = fn(out, dtype, (cuuint32_t)rank, const_cast<void*>(base),
                  gdims, gstr, gbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed: CUresult %d (rank %d dims %llu,%llu box %u,%u)",
                   (int)r, rank, (unsigned long long)gdims[0], (unsigned long long)gdims[1],
                   gbox[0], gbox[1]);
    return -3;
  }
  return 0;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank, dims, strides_bytes, box);
}
int make_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, base, rank, dims, strides_bytes, box);
}

}  // namespace b200

extern "C" const char* rlaifv_last_error(void) { return b200::get_last_error(); }

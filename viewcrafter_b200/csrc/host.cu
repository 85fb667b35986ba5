// Host-side support: error text, SM count, tensor-map encoding via the driver entry point.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "common.cuh"

namespace vc {

static thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

int sm_count() {
  static std::atomic<int> cache[256];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  const int slot = dev & 255;
  int n = cache[slot].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    // VC_SM_COUNT=k (k below the real count) sizes every launch grid as if the device had k SMs: it shows that the results of
    // reproducible mode do not depend on the SM count (e.g. 114 of the PCIe H100 on a 132-SM card).  It can only shrink grids.
    const char* e = getenv("VC_SM_COUNT");
    if (e && atoi(e) > 0 && atoi(e) < n) n = atoi(e);
    cache[slot].store(n, std::memory_order_relaxed);
  }
  return n;
}

static inline int device_slot() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
  return dev & 255;
}
bool device_once_needed(DeviceOnce& o) {
  const int s = device_slot();
  return (__atomic_load_n(&o.done[s >> 6], __ATOMIC_ACQUIRE) & (1ull << (s & 63))) == 0;
}
void device_once_mark(DeviceOnce& o) {
  const int s = device_slot();
  __atomic_fetch_or(&o.done[s >> 6], 1ull << (s & 63), __ATOMIC_RELEASE);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int encode_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, int swizzle_bytes, CUtensorMapDataType dtype) {
  EncodeTiledFn fn = get_encode();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled is unavailable (no CUDA driver?)");
    return VC_ERR_CUDA;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  for (int i = 0; i + 1 < rank; ++i) {
    if (gstr[i] % 16 != 0) {
      set_error("tensor map stride %d = %llu bytes is not a multiple of 16", i, (unsigned long long)gstr[i]);
      return VC_ERR_ARG;
    }
  }
  if (reinterpret_cast<uintptr_t>(base) % 16 != 0) {
    set_error("tensor map base address is not 16-byte aligned");
    return VC_ERR_ARG;
  }
  CUresult r = fn(out, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bdim, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu,.. box %u,%u,..)", (int)r, rank,
              (unsigned long long)gdim[0], (unsigned long long)gdim[1], bdim[0], bdim[1]);
    return VC_ERR_CUDA;
  }
  return VC_OK;
}

}  // namespace vc

// Shared device/host helpers for the sm_90a kernels: mbarrier, TMA and wgmma PTX wrappers,
// wgmma descriptors, tensor-map encoding through the driver entry point (no libcuda link dependency).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define VC_OK 0
#define VC_ERR_ARG 1
#define VC_ERR_CUDA 2
#define VC_ERR_UNSUPPORTED 3

namespace vc {

// ----------------------------------------------------------------------------------------------
// error plumbing: every C-ABI entry point returns an int status; the text is kept per thread.
// ----------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
const char* last_error();

#define VC_CHECK_CUDA(expr)                                                                      \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      vc::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return VC_ERR_CUDA;                                                                        \
    }                                                                                            \
  } while (0)

#define VC_REQUIRE(cond, ...)       \
  do {                              \
    if (!(cond)) {                  \
      vc::set_error(__VA_ARGS__);   \
      return VC_ERR_ARG;            \
    }                               \
  } while (0)

// Encode a tiled fp16 tensor map (rank 2..5), zero OOB fill; swizzle_bytes: 128 (default), 64 or 0 (none).
// dims/box: innermost first, in elements.  strides_bytes: for dims 1..rank-1.  dtype: UINT8 for e4m3 weights.
int encode_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes = 128,
                    CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16);

int sm_count();   // of the CURRENT device (cached per device)

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a per-device property: launch wrappers keep one bit per device
// ordinal in a DeviceOnce and configure the kernel the first time each device is used.  Setting it twice (two threads racing)
// is harmless, so a plain atomic bit mask is enough.
struct DeviceOnce {
  unsigned long long done[4] = {0, 0, 0, 0};          // 256 device ordinals
};
bool device_once_needed(DeviceOnce& o);   // true: the caller must configure, then call device_once_mark
void device_once_mark(DeviceOnce& o);

// ----------------------------------------------------------------------------------------------
// device-side PTX wrappers
// ----------------------------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P1;\n\t.reg .b32 R1;\n\t"
      "elect.sync R1|P1, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P1;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P1;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// ---- TMA (cp.async.bulk.tensor) ----
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// TMA store (shared -> global, bulk async group): out-of-bounds parts of the box are not written
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until the bulk groups of this thread have finished READING their shared-memory source (it may be overwritten)
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// wait until the bulk groups of this thread are complete (writes performed)
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// make generic-proxy shared-memory writes visible to the async proxy (TMA) before it reads them
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma (warpgroup MMA, sm_90a) ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keep the accumulator registers live across the asynchronous MMAs (no reordering of their reads / writes around the fence)
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// named barrier over `count` threads (one id per warpgroup; id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
// signal a named barrier without waiting for it; `count` covers the arriving and the waiting (named_bar_sync) threads
__device__ __forceinline__ void named_bar_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }
// move registers between the warpgroups of a CTA (warpgroup-collective; the per-SM register file must hold the new split)
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// Shared-memory matrix descriptor, 128B swizzle, rows of 128 bytes (64 fp16) stored densely, as TMA writes them with
// CU_TENSOR_MAP_SWIZZLE_128B:
//   K-major operand  (tile [rows][64 k]):  SBO = 1024 B between 8-row groups, LBO unused (=1).
//   MN-major operand (tile [k rows][64 mn]): SBO = 1024 B between 8-row (k) groups, LBO = distance between 64-wide mn blocks.
// Advancing along K by 16 elements inside a 128-byte row adds 32 bytes to the start address (the swizzle is applied by
// the hardware on absolute address bits, so tiles must be 1024-byte aligned).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes = 16, uint32_t sbo_bytes = 1024) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;   // SWIZZLE_128B
  return d;
}

// The same for K-major e4m3 tiles of 64-byte rows (64 fp8), as TMA writes them with CU_TENSOR_MAP_SWIZZLE_64B: SBO = 512 B
// between 8-row groups; one k32 step is 32 bytes along the row (tiles 512-byte aligned).
__device__ __forceinline__ uint64_t wgmma_desc_sw64(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(512 >> 4) << 32;
  d |= (uint64_t)2 << 62;   // SWIZZLE_64B
  return d;
}

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// erf via Abramowitz-Stegun 7.1.26 (absolute error < 1.5e-7 before fp32 rounding): 1 MUFU.EX2 + 1 MUFU.RCP + 7 FMA.
// gelu_erf_fast in fp16 is within half an fp16 ulp plus 0.5 |x| (1.5e-7 + the fp32 rounding terms) of the exact GELU on every fp16
// input (tests/gelu_ref.py derives the bound).  That is not always below fp16 resolution: in the negative tail, where gelu(x) is an
// fp16 subnormal, the result is up to 2 fp16 ulps from the rounded exact value (at x = -5.53 on an H100, tests/test_misc_kernels_gpu.py,
// for gelu_erf_fast and gelu_epilogue alike).
__device__ __forceinline__ float erf_fast(float x) {
  const float ax = fabsf(x);
  const float t = __frcp_rn(fmaf(0.3275911f, ax, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float y = 1.0f - poly * t * __expf(-ax * ax);
  return copysignf(y, x);
}
__device__ __forceinline__ float gelu_erf_fast(float x) { return 0.5f * x * (1.0f + erf_fast(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

#endif  // __CUDACC__

}  // namespace vc

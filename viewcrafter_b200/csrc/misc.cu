// Small / HBM-bound kernels of the denoise step:
// nearest-2x upsample, stride-2 im2col, layout conversions, the timestep/fps embedding MLP pieces
// and the fused DDIM update.
#include <cstring>

#include "common.cuh"
#include "kernels.h"

namespace vc {

// ------------------------------------------------------------------------------------------------
// nearest 2x upsample (F.interpolate scale 2, openaimodel3d.py:101-104 / ae_modules.py:123), NHWC, 16-byte vectors
// ------------------------------------------------------------------------------------------------
__global__ void upsample2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, long long total, int H, int W, int vecs) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vecs);
    long long p = i / vecs;
    const int xo = (int)(p % (2 * W)); p /= (2 * W);
    const int yo = (int)(p % (2 * H));
    const long long n = p / (2 * H);
    out[i] = x[((n * H + (yo >> 1)) * W + (xo >> 1)) * vecs + v];
  }
}
int upsample2x_nhwc(const __half* x, __half* out, int N, int H, int W, int C, cudaStream_t stream) {
  VC_REQUIRE(x && out && C % 8 == 0, "upsample2x: bad args");
  const long long total = (long long)N * 4 * H * W * (C / 8);
  const int blocks = (int)min((long long)sm_count() * 16, (total + 255) / 256);
  upsample2x_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out), total, H, W, C / 8);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

// im2col for the stride-2 3x3 downsample conv (openaimodel3d.py:51-77): out [N*Ho*Wo, 9*C], tap-major then channel.
__global__ void im2col_s2_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, long long total, int H, int W, int vecs,
                                 int pad_lo, int Ho, int Wo) {
  const uint4 zero = make_uint4(0, 0, 0, 0);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vecs);
    long long p = i / vecs;
    const int tap = (int)(p % 9); p /= 9;
    const int xo = (int)(p % Wo); p /= Wo;
    const int yo = (int)(p % Ho);
    const long long n = p / Ho;
    const int yi = 2 * yo - pad_lo + tap / 3, xi = 2 * xo - pad_lo + tap % 3;
    out[i] = (yi >= 0 && yi < H && xi >= 0 && xi < W) ? x[((n * H + yi) * W + xi) * vecs + v] : zero;
  }
}
int im2col3x3_s2_nhwc(const __half* x, __half* out, int N, int H, int W, int C, int pad_lo, int Ho, int Wo, cudaStream_t stream) {
  VC_REQUIRE(x && out && C % 8 == 0, "im2col: bad args");
  const long long total = (long long)N * Ho * Wo * 9 * (C / 8);
  const int blocks = (int)min((long long)sm_count() * 16, (total + 255) / 256);
  im2col_s2_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out), total, H, W, C / 8,
                                               pad_lo, Ho, Wo);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

// ------------------------------------------------------------------------------------------------
// max |x| of one or two fp16 row blocks (the FP8 GEMM's activation scale).  Max is exact and order-independent, so the result
// does not depend on the launch: every CTA folds its 8-element vectors with __hmax2, then one atomicMax on the float bits
// (non-negative floats order like their bit patterns) into *amax, which the host zeroes first in stream order.
// ------------------------------------------------------------------------------------------------
__global__ void absmax_kernel(const __half* __restrict__ x1, int vec1, int ld1, const __half* __restrict__ x2, int vec2, int ld2,
                              long long rows, unsigned int* __restrict__ amax) {
  const unsigned vecs = vec1 + vec2;
  const unsigned total = (unsigned)(rows * vecs);       // < 2^31 (host check): 32-bit index arithmetic
  __half2 m = __float2half2_rn(0.f);
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const unsigned r = i / vecs;
    const int v = (int)(i - r * vecs);
    const uint4 u = v < vec1 ? __ldg(reinterpret_cast<const uint4*>(x1 + (long long)r * ld1 + v * 8))
                             : __ldg(reinterpret_cast<const uint4*>(x2 + (long long)r * ld2 + (v - vec1) * 8));
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) m = __hmax2(m, __habs2(h[e]));
  }
  float f = fmaxf(__low2float(m), __high2float(m));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) f = fmaxf(f, __shfl_xor_sync(0xffffffffu, f, o));
  __shared__ float wmax[32];
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = f;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) f = fmaxf(f, wmax[w]);
    atomicMax(amax, __float_as_uint(f));
  }
}
int absmax_f16(const __half* x1, long long rows, int cols1, int ld1, const __half* x2, int cols2, int ld2, float* amax, cudaStream_t stream) {
  VC_REQUIRE(x1 && amax && rows > 0 && cols1 > 0 && (!x2 || cols2 > 0), "absmax_f16: bad arguments");
  VC_REQUIRE(cols1 % 8 == 0 && ld1 % 8 == 0 && (reinterpret_cast<uintptr_t>(x1) & 15) == 0 &&
                 (!x2 || (cols2 % 8 == 0 && ld2 % 8 == 0 && (reinterpret_cast<uintptr_t>(x2) & 15) == 0)),
             "absmax_f16: rows must be 16-byte aligned with a multiple of 8 columns");
  const int vec2 = x2 ? cols2 / 8 : 0;
  const long long total = rows * (cols1 / 8 + vec2);
  VC_REQUIRE(total < (1ll << 31), "absmax_f16: %lld vectors out of range", total);
  const int blocks = (int)min((long long)sm_count() * 4, (total + 255) / 256);
  VC_CHECK_CUDA(cudaMemsetAsync(amax, 0, sizeof(float), stream));
  absmax_kernel<<<blocks, 256, 0, stream>>>(x1, cols1 / 8, ld1, x2, vec2, ld2, rows, reinterpret_cast<unsigned int*>(amax));
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

// ------------------------------------------------------------------------------------------------
// layout conversions at the boundary ([B,C,T,H,W] fp32 <-> [(B T) H W, C] fp16/fp32)
// ------------------------------------------------------------------------------------------------
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, __half* __restrict__ out, int B, int C, int T, long long HW,
                                    int c_off, int ldo) {
  const long long total = (long long)B * C * T * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i % HW;
    long long r = i / HW;
    const int t = (int)(r % T); r /= T;
    const int c = (int)(r % C);
    const long long b = r / C;
    out[((b * T + t) * HW + p) * ldo + c_off + c] = __float2half_rn(x[i]);
  }
}
int nchw_to_nhwc_f16(const float* x, __half* out, int B, int C, int T, long long HW, int c_off, int ldo, cudaStream_t stream) {
  VC_REQUIRE(x && out, "nchw_to_nhwc: null pointer");
  const long long total = (long long)B * C * T * HW;
  const int blocks = (int)min((long long)sm_count() * 16, (total + 255) / 256);
  nchw_to_nhwc_kernel<<<blocks, 256, 0, stream>>>(x, out, B, C, T, HW, c_off, ldo);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

__global__ void nhwc_to_ncthw_kernel(const float* __restrict__ x, int ldx, float* __restrict__ out, int B, int C, int T, long long HW) {
  const long long total = (long long)B * C * T * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i % HW;
    long long r = i / HW;
    const int t = (int)(r % T); r /= T;
    const int c = (int)(r % C);
    const long long b = r / C;
    out[i] = x[((b * T + t) * HW + p) * ldx + c];
  }
}
int nhwc_to_ncthw_f32(const float* x, int ldx, float* out, int B, int C, int T, long long HW, cudaStream_t stream) {
  VC_REQUIRE(x && out, "nhwc_to_ncthw: null pointer");
  const long long total = (long long)B * C * T * HW;
  const int blocks = (int)min((long long)sm_count() * 16, (total + 255) / 256);
  nhwc_to_ncthw_kernel<<<blocks, 256, 0, stream>>>(x, ldx, out, B, C, T, HW);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

__global__ void nhwc_to_nchw_h_kernel(const __half* __restrict__ x, int ldx, float* __restrict__ out, int N, int C, long long HW) {
  const long long total = (long long)N * C * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i % HW;
    const long long r = i / HW;
    const int c = (int)(r % C);
    const long long n = r / C;
    out[i] = __half2float(x[(n * HW + p) * ldx + c]);
  }
}
int nhwc_to_nchw_f32_from_f16(const __half* x, int ldx, float* out, int N, int C, long long HW, cudaStream_t stream) {
  VC_REQUIRE(x && out, "nhwc_to_nchw: null pointer");
  const long long total = (long long)N * C * HW;
  const int blocks = (int)min((long long)sm_count() * 16, (total + 255) / 256);
  nhwc_to_nchw_h_kernel<<<blocks, 256, 0, stream>>>(x, ldx, out, N, C, HW);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

__global__ void cast_kernel(const float* __restrict__ x, __half* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = __float2half_rn(x[i]);
}
int cast_f32_to_f16(const float* x, __half* out, long long n, cudaStream_t stream) {
  VC_REQUIRE(x && out, "cast: null pointer");
  const int blocks = (int)min((long long)sm_count() * 16, (n + 255) / 256);
  cast_kernel<<<blocks, 256, 0, stream>>>(x, out, n);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

__global__ void add_kernel(const __half2* __restrict__ a, const __half2* __restrict__ b, __half2* __restrict__ out, long long n2) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += (long long)gridDim.x * blockDim.x) {
    const float2 x = __half22float2(a[i]), y = __half22float2(b[i]);
    out[i] = __floats2half2_rn(x.x + y.x, x.y + y.y);
  }
}
// exact-erf GELU, elementwise (Resampler FeedForward, resampler.py:27-34); erf as in the GEGLU epilogue (common.cuh)
__global__ void gelu_kernel(const __half2* __restrict__ x, __half2* __restrict__ out, long long n2) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += (long long)gridDim.x * blockDim.x) {
    const float2 v = __half22float2(x[i]);
    out[i] = __floats2half2_rn(gelu_erf_fast(v.x), gelu_erf_fast(v.y));
  }
}
int gelu_rows_f16(const __half* x, __half* out, long long n, cudaStream_t stream) {
  VC_REQUIRE(x && out && n > 0 && n % 2 == 0, "gelu: bad args");
  const int blocks = (int)min((long long)sm_count() * 16, (n / 2 + 255) / 256);
  gelu_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const __half2*>(x), reinterpret_cast<__half2*>(out), n / 2);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

int add_rows_f16(const __half* a, const __half* b, __half* out, long long n, cudaStream_t stream) {
  VC_REQUIRE(a && b && out && n % 2 == 0, "add: bad args");
  const int blocks = (int)min((long long)sm_count() * 16, (n / 2 + 255) / 256);
  add_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const __half2*>(a), reinterpret_cast<const __half2*>(b),
                                         reinterpret_cast<__half2*>(out), n / 2);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

// ------------------------------------------------------------------------------------------------
// time / fps embedding pieces (utils_diffusion.py:8-28, openaimodel3d.py:549-577, :218): fp32, M is 1..B
// ------------------------------------------------------------------------------------------------
__global__ void small_linear_kernel(const float* __restrict__ x, int rows, int K, const float* __restrict__ W,
                                    const float* __restrict__ bias, int N, int act_in, float* __restrict__ out,
                                    const float* __restrict__ add) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows * N) return;
  const int r = warp / N, n = warp % N;
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) {
    float xv = x[(long long)r * K + k];
    if (act_in == 1) xv = xv / (1.0f + expf(-xv));
    acc += xv * W[(long long)n * K + k];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    float y = acc + (bias ? bias[n] : 0.f);
    if (add) y += add[(long long)r * N + n];
    out[(long long)r * N + n] = y;
  }
}
int small_linear_f32(const float* x, int rows, int K, const float* W, const float* bias, int N, int act_in, float* out,
                     const float* add, cudaStream_t stream) {
  VC_REQUIRE(x && W && out && rows > 0 && N > 0 && K > 0, "small_linear: bad args");
  const long long warps = (long long)rows * N;
  const int blocks = (int)((warps * 32 + 255) / 256);
  small_linear_kernel<<<blocks, 256, 0, stream>>>(x, rows, K, W, bias, N, act_in, out, add);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

__global__ void timestep_embedding_kernel(const long long* __restrict__ t, int n, int dim, float* __restrict__ out) {
  const int half = dim / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * half) return;
  const int r = i / half, j = i % half;
  // freqs = exp(-ln(10000) * j / half) evaluated in fp32 exactly as torch does
  const float freq = expf(-9.210340371976184f * (float)j / (float)half);
  const float arg = (float)t[r] * freq;
  out[(long long)r * dim + j] = cosf(arg);
  out[(long long)r * dim + half + j] = sinf(arg);
  if ((dim & 1) && j == 0) out[(long long)r * dim + dim - 1] = 0.f;
}
int timestep_embedding_f32(const long long* t, int n, int dim, float* out, cudaStream_t stream) {
  VC_REQUIRE(t && out && n > 0 && dim >= 2, "timestep_embedding: bad args");
  const int total = n * (dim / 2);
  timestep_embedding_kernel<<<(total + 127) / 128, 128, 0, stream>>>(t, n, dim, out);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

// ------------------------------------------------------------------------------------------------
// Fused DDIM update (ddim.py:228-281 + utils_diffusion.py:147-158), v-parameterisation, batch 1 per call.
// pass 1: double-precision sums for the two unbiased stds; pass 2: elementwise update.
// ------------------------------------------------------------------------------------------------
// CFG combine.  Two-way (ddim.py:226): u + s (c - u).  Three-way (ddim_multiplecond.py:233, vi = the "image, no text"
// branch): u + s_img (vi - u) + s (c - vi), evaluated left to right like the reference expression.
__device__ __forceinline__ float cfg_combine(float c, float u, const float* __restrict__ vi, long long i, float cfg, float cfg_img) {
  if (vi == nullptr) return u + cfg * (c - u);
  const float w = vi[i];
  return (u + cfg_img * (w - u)) + cfg * (c - w);
}
// deterministic: every block leaves its four partial sums in ws[4 + 4 * block] (fixed in-block order); ddim_apply_kernel adds the
// blocks up in index order -- no floating-point atomics, a seeded sampling run is bit-reproducible
static constexpr int DDIM_MAX_BLOCKS = 1024;
static constexpr int DDIM_REPRO_BLOCKS = 512;
__global__ void __launch_bounds__(256) ddim_stats_kernel(const float* __restrict__ vc_, const float* __restrict__ vu, const float* __restrict__ vi, long long n,
                                  float cfg, float cfg_img, double* ws) {
  __shared__ double red[8][4];
  double s1 = 0, q1 = 0, s2 = 0, q2 = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float c = vc_[i], u = vu[i];
    const float m = cfg_combine(c, u, vi, i, cfg, cfg_img);
    s1 += c; q1 += (double)c * c;
    s2 += m; q2 += (double)m * m;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o); q1 += __shfl_xor_sync(0xffffffffu, q1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o); q2 += __shfl_xor_sync(0xffffffffu, q2, o);
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { red[w][0] = s1; red[w][1] = q1; red[w][2] = s2; red[w][3] = q2; }
  __syncthreads();
  if (threadIdx.x < 4) {
    double a = 0;
    for (int i = 0; i < 8; ++i) a += red[i][threadIdx.x];
    ws[4 + 4 * blockIdx.x + threadIdx.x] = a;
  }
}
// The pieces of the DDIM apply step, shared by ddim_apply_kernel (one step for the whole input) and ddim_frames_apply_kernel (a step
// per frame), so both evaluate the same expressions in the same order.
// guidance-rescale factor std(v_cond) / std(guided v) from the statistics blocks' partial sums, added up in index order
__device__ __forceinline__ float ddim_rescale_factor(const double* ws, int stat_blocks, long long n) {
  __shared__ double tot[4];
  if (threadIdx.x < 4) {
    double a = 0;
    for (int b = 0; b < stat_blocks; ++b) a += ws[4 + 4 * b + threadIdx.x];
    tot[threadIdx.x] = a;
  }
  __syncthreads();
  const double dn = (double)n;
  const double var_t = (tot[1] - tot[0] * tot[0] / dn) / (dn - 1.0);
  const double var_c = (tot[3] - tot[2] * tot[2] / dn) / (dn - 1.0);
  return (float)sqrt(var_t > 0 ? var_t : 0.0) / (float)sqrt(var_c > 0 ? var_c : 0.0);
}
// the step's scalars and the constants derived from them
struct DdimStep {
  float sqrt_ac_t, sqrt_1mac_t, sigma_t, rescale, dir_c, sq_ap;
};
__device__ __forceinline__ DdimStep ddim_step(float sqrt_ac_t, float sqrt_1mac_t, float a_prev, float sigma_t, float scale_t,
                                              float prev_scale_t) {
  DdimStep d;
  d.sqrt_ac_t = sqrt_ac_t; d.sqrt_1mac_t = sqrt_1mac_t; d.sigma_t = sigma_t;
  d.rescale = __fdiv_rn(prev_scale_t, scale_t);
  // eta = 1 from a = 0: 1 - a' - sigma^2 is 0 in exact arithmetic, and the contracted FADD + FFMA of the fp32 step scalars lands
  // below 0 at many step counts (uniform_trailing S = 4, 7, 9, 25, ...), where an unclamped sqrtf turns every x_prev into NaN.
  // Clamped; the same bits wherever it is >= 0, and the same expression as dpm_apply_kernel (c_hist = 0 is this update bit for bit)
  d.dir_c = sqrtf(fmaxf(__fmaf_rn(-sigma_t, sigma_t, __fsub_rn(1.f, a_prev)), 0.f));
  d.sq_ap = sqrtf(a_prev);
  return d;
}
// element i: guided v, then pred_x0 and x_prev.  Every rounding is spelled out (the _rn intrinsics are never contracted), in the
// order and with the fused products ptxas chose for the contracted expressions of the original single-step kernel
// (u + s (c - u), (u + s_img (vi - u)) + s (c - vi), g (m factor) + (1 - g) m, sqrt_ac m + sqrt_1mac x, sqrt_ac x - sqrt_1mac m,
// sq_ap p0 + dir_c e_t + sigma noise): its outputs are unchanged, and a kernel that runs this code with the same step gets its bits
// whatever ptxas does around it.
__device__ __forceinline__ void ddim_element(const float* __restrict__ x, const float* __restrict__ vc_, const float* __restrict__ vu,
                                             const float* __restrict__ vi, float cfg_img, const float* __restrict__ noise,
                                             float* __restrict__ x_prev, float* __restrict__ pred_x0, long long i,
                                             const vc_ddim_scalars& s, float factor, const DdimStep& d) {
  const float c = vc_[i];
  float m = c;
  if (s.use_cfg) {
    const float u = vu[i];
    if (vi == nullptr) {
      m = __fmaf_rn(__fsub_rn(c, u), s.cfg_scale, u);
    } else {
      const float w = vi[i];
      m = __fmaf_rn(__fsub_rn(c, w), s.cfg_scale, __fmaf_rn(__fsub_rn(w, u), cfg_img, u));
    }
    if (s.guidance_rescale > 0.f)
      m = __fmaf_rn(m, __fsub_rn(1.f, s.guidance_rescale), __fmul_rn(__fmul_rn(m, factor), s.guidance_rescale));
  }
  const float xi = x[i];
  const float e_t = __fmaf_rn(m, d.sqrt_ac_t, __fmul_rn(xi, d.sqrt_1mac_t));
  float p0 = __fmaf_rn(xi, d.sqrt_ac_t, -__fmul_rn(m, d.sqrt_1mac_t));
  p0 = __fmul_rn(p0, d.rescale);
  pred_x0[i] = p0;
  x_prev[i] = __fmaf_rn(noise[i], d.sigma_t, __fmaf_rn(e_t, d.dir_c, __fmul_rn(p0, d.sq_ap)));
}
__global__ void ddim_apply_kernel(const float* __restrict__ x, const float* __restrict__ vc_, const float* __restrict__ vu,
                                  const float* __restrict__ vi, float cfg_img,
                                  const float* __restrict__ noise, float* __restrict__ x_prev, float* __restrict__ pred_x0,
                                  long long n, vc_ddim_scalars s, const double* ws, int stat_blocks) {
  float factor = 1.f;
  if (s.use_cfg && s.guidance_rescale > 0.f) factor = ddim_rescale_factor(ws, stat_blocks, n);
  const DdimStep d = ddim_step(s.sqrt_ac_t, s.sqrt_1mac_t, s.a_prev, s.sigma_t, s.scale_t, s.prev_scale_t);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    ddim_element(x, vc_, vu, vi, cfg_img, noise, x_prev, pred_x0, i, s, factor, d);
}
// per-frame step scalars, passed by value (kernel parameters: no host-to-device copy, so the launch can be captured in a CUDA graph)
struct DdimFrameTable {
  vc_ddim_frame_scalars f[VC_DDIM_MAX_FRAMES];
};
// element i of [B', C, T, HW] belongs to frame (i / HW) % T and takes that frame's step; each CTA derives the T steps once
__global__ void __launch_bounds__(256) ddim_frames_apply_kernel(const float* __restrict__ x, const float* __restrict__ vc_,
                                  const float* __restrict__ vu, const float* __restrict__ vi, float cfg_img,
                                  const float* __restrict__ noise, float* __restrict__ x_prev, float* __restrict__ pred_x0,
                                  long long n, int T, long long HW, vc_ddim_scalars s, const __grid_constant__ DdimFrameTable tab,
                                  const double* ws, int stat_blocks) {
  __shared__ DdimStep steps[VC_DDIM_MAX_FRAMES];
  for (int f = threadIdx.x; f < T; f += blockDim.x) {
    const vc_ddim_frame_scalars& q = tab.f[f];
    steps[f] = ddim_step(q.sqrt_ac_t, q.sqrt_1mac_t, q.a_prev, q.sigma_t, q.scale_t, q.prev_scale_t);
  }
  float factor = 1.f;
  if (s.use_cfg && s.guidance_rescale > 0.f) factor = ddim_rescale_factor(ws, stat_blocks, n);
  __syncthreads();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    ddim_element(x, vc_, vu, vi, cfg_img, noise, x_prev, pred_x0, i, s, factor, steps[(int)((i / HW) % T)]);
}
// the grid of the statistics and apply kernels.  Reproducible mode: a fixed number of statistics blocks, so the grid-strided order
// of the two std reductions does not depend on the SM count
static int ddim_blocks(long long n, const vc_ddim_scalars& s) {
  int blocks = (int)min(s.reproducible ? (long long)DDIM_REPRO_BLOCKS : (long long)sm_count() * 4, (n + 255) / 256);
  return blocks > DDIM_MAX_BLOCKS ? DDIM_MAX_BLOCKS : blocks;
}
int ddim_update(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img, const float* noise,
                float* x_prev, float* pred_x0, long long n, const vc_ddim_scalars& s, double* ws, cudaStream_t stream) {
  VC_REQUIRE(x && v_cond && noise && x_prev && pred_x0 && ws && n > 1, "ddim_update: bad args");
  VC_REQUIRE(!s.use_cfg || v_uncond, "ddim_update: CFG needs the unconditional output");
  VC_REQUIRE(!v_uncond_img || s.use_cfg, "ddim_update: the image-only branch is only defined with CFG on");
  const int blocks = ddim_blocks(n, s);
  if (s.use_cfg && s.guidance_rescale > 0.f) {           // ws: 4 * (1 + DDIM_MAX_BLOCKS) doubles
    ddim_stats_kernel<<<blocks, 256, 0, stream>>>(v_cond, v_uncond, v_uncond_img, n, s.cfg_scale, cfg_img, ws);
    VC_CHECK_CUDA(cudaGetLastError());
  }
  ddim_apply_kernel<<<blocks, 256, 0, stream>>>(x, v_cond, v_uncond, v_uncond_img, cfg_img, noise, x_prev, pred_x0, n, s, ws, blocks);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}
int ddim_update_frames(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img,
                       const float* noise, float* x_prev, float* pred_x0, long long n, int T, long long HW, const vc_ddim_scalars& s,
                       const vc_ddim_frame_scalars* frames, double* ws, cudaStream_t stream) {
  VC_REQUIRE(x && v_cond && noise && x_prev && pred_x0 && ws && frames, "ddim_update_frames: null pointer");
  VC_REQUIRE(T >= 1 && T <= VC_DDIM_MAX_FRAMES, "ddim_update_frames: T=%d unsupported (1..%d)", T, VC_DDIM_MAX_FRAMES);
  VC_REQUIRE(HW >= 1 && n > 1 && n % ((long long)T * HW) == 0, "ddim_update_frames: n=%lld is not a multiple of T*HW=%lld", n,
             (long long)T * HW);
  VC_REQUIRE(!s.use_cfg || v_uncond, "ddim_update_frames: CFG needs the unconditional output");
  VC_REQUIRE(!v_uncond_img || s.use_cfg, "ddim_update_frames: the image-only branch is only defined with CFG on");
  DdimFrameTable tab;
  memset(&tab, 0, sizeof(tab));
  memcpy(tab.f, frames, sizeof(vc_ddim_frame_scalars) * T);
  const int blocks = ddim_blocks(n, s);
  if (s.use_cfg && s.guidance_rescale > 0.f) {
    ddim_stats_kernel<<<blocks, 256, 0, stream>>>(v_cond, v_uncond, v_uncond_img, n, s.cfg_scale, cfg_img, ws);
    VC_CHECK_CUDA(cudaGetLastError());
  }
  ddim_frames_apply_kernel<<<blocks, 256, 0, stream>>>(x, v_cond, v_uncond, v_uncond_img, cfg_img, noise, x_prev, pred_x0, n, T, HW, s,
                                                       tab, ws, blocks);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

// ------------------------------------------------------------------------------------------------
// DPM-Solver++ multistep updates (INTEGRATION.md "Samplers"): the DDIM step above, x_ddim, plus the multistep correction
//   NH = 1, 2M:      x_prev = x_ddim + c_hist (x0 - m1)
//   NH = 2, 3M SDE:  x_prev = x_ddim + c_hist (x0 - m1) + c_hist2 (m1 - m2)
// with x0 = sqrt_ac_t x - sqrt_1mac_t v (before the dynamic rescale), m1 / m2 the x0 of the previous step / the one before.
// NH = 1: x0_hist holds m1 and is overwritten with this step's x0.  NH = 2: x0_hist holds m2 and is overwritten with this step's
// x0; x0_hist1 holds m1 and is only read.  A zero coefficient reads nothing for its term (a history may be uninitialised), and each
// non-zero one is one more __fmaf_rn: c_hist = c_hist2 = 0 is x_ddim bit for bit, c_hist2 = 0 is the NH = 1 update bit for bit.
// x_ddim is ddim_apply_kernel's expression.
// ------------------------------------------------------------------------------------------------
template <int NH>
__global__ void dpm_apply_kernel(const float* __restrict__ x, const float* __restrict__ vc_, const float* __restrict__ vu,
                                 const float* __restrict__ vi, float cfg_img,
                                 const float* __restrict__ noise, const float* __restrict__ x0_hist1, float* __restrict__ x0_hist,
                                 float* __restrict__ x_prev, float* __restrict__ pred_x0, long long n, vc_ddim_scalars s, float c_hist,
                                 float c_hist2, const double* ws, int stat_blocks) {
  static_assert(NH == 1 || NH == 2, "dpm_apply_kernel: one or two x0 histories");
  float factor = 1.f;
  if (s.use_cfg && s.guidance_rescale > 0.f) {
    __shared__ double tot[4];
    if (threadIdx.x < 4) {
      double a = 0;
      for (int b = 0; b < stat_blocks; ++b) a += ws[4 + 4 * b + threadIdx.x];
      tot[threadIdx.x] = a;
    }
    __syncthreads();
    const double dn = (double)n;
    const double var_t = (tot[1] - tot[0] * tot[0] / dn) / (dn - 1.0);
    const double var_c = (tot[3] - tot[2] * tot[2] / dn) / (dn - 1.0);
    factor = (float)sqrt(var_t > 0 ? var_t : 0.0) / (float)sqrt(var_c > 0 ? var_c : 0.0);
  }
  const float rescale = s.prev_scale_t / s.scale_t;
  // eta = 1 from a = 0: 1 - a' - sigma^2 is 0 in exact arithmetic and can round to -2e-8 (4 uniform_trailing steps); clamped as in
  // ddim_apply_kernel, the same bits wherever it is >= 0
  const float dir_c = sqrtf(fmaxf(1.f - s.a_prev - s.sigma_t * s.sigma_t, 0.f));
  const float sq_ap = sqrtf(s.a_prev);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float c = vc_[i];
    float m = c;
    if (s.use_cfg) {
      const float u = vu[i];
      m = cfg_combine(c, u, vi, i, s.cfg_scale, cfg_img);
      if (s.guidance_rescale > 0.f) m = s.guidance_rescale * (m * factor) + (1.f - s.guidance_rescale) * m;
    }
    const float xi = x[i];
    const float e_t = s.sqrt_ac_t * m + s.sqrt_1mac_t * xi;
    float p0 = s.sqrt_ac_t * xi - s.sqrt_1mac_t * m;
    const float x0 = p0;
    p0 *= rescale;
    pred_x0[i] = p0;
    const float x_ddim = sq_ap * p0 + dir_c * e_t + s.sigma_t * noise[i];
    if (NH == 1) {
      x_prev[i] = c_hist != 0.f ? __fmaf_rn(c_hist, x0 - x0_hist[i], x_ddim) : x_ddim;
    } else {
      const float m1 = (c_hist != 0.f || c_hist2 != 0.f) ? x0_hist1[i] : 0.f;
      float xp = c_hist != 0.f ? __fmaf_rn(c_hist, x0 - m1, x_ddim) : x_ddim;
      if (c_hist2 != 0.f) xp = __fmaf_rn(c_hist2, m1 - x0_hist[i], xp);
      x_prev[i] = xp;
    }
    x0_hist[i] = x0;
  }
}
// x0_hist1 == nullptr: the NH = 1 kernel (c_hist2 unused)
static int dpm_launch(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img,
                      const float* noise, const float* x0_hist1, float* x0_hist, float* x_prev, float* pred_x0, long long n,
                      const vc_ddim_scalars& s, float c_hist, float c_hist2, double* ws, cudaStream_t stream) {
  // the statistics grid of ddim_update (reproducible mode included), so every update reduces the same partial sums in the same order
  const int blocks = ddim_blocks(n, s);
  if (s.use_cfg && s.guidance_rescale > 0.f) {
    ddim_stats_kernel<<<blocks, 256, 0, stream>>>(v_cond, v_uncond, v_uncond_img, n, s.cfg_scale, cfg_img, ws);
    VC_CHECK_CUDA(cudaGetLastError());
  }
  if (x0_hist1 == nullptr)
    dpm_apply_kernel<1><<<blocks, 256, 0, stream>>>(x, v_cond, v_uncond, v_uncond_img, cfg_img, noise, nullptr, x0_hist, x_prev, pred_x0,
                                                    n, s, c_hist, 0.f, ws, blocks);
  else
    dpm_apply_kernel<2><<<blocks, 256, 0, stream>>>(x, v_cond, v_uncond, v_uncond_img, cfg_img, noise, x0_hist1, x0_hist, x_prev, pred_x0,
                                                    n, s, c_hist, c_hist2, ws, blocks);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}
int dpm_update(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img, const float* noise,
               float* x0_hist, float* x_prev, float* pred_x0, long long n, const vc_ddim_scalars& s, float c_hist, double* ws,
               cudaStream_t stream) {
  VC_REQUIRE(x && v_cond && noise && x0_hist && x_prev && pred_x0 && ws && n > 1, "dpm_update: bad args");
  VC_REQUIRE(!s.use_cfg || v_uncond, "dpm_update: CFG needs the unconditional output");
  VC_REQUIRE(!v_uncond_img || s.use_cfg, "dpm_update: the image-only branch is only defined with CFG on");
  VC_REQUIRE(x0_hist != x_prev && x0_hist != pred_x0 && x0_hist != x && x_prev != pred_x0, "dpm_update: x0_hist, x_prev and pred_x0 must not alias");
  VC_REQUIRE(isfinite(c_hist), "dpm_update: c_hist must be finite");
  return dpm_launch(x, v_cond, v_uncond, v_uncond_img, cfg_img, noise, nullptr, x0_hist, x_prev, pred_x0, n, s, c_hist, 0.f, ws, stream);
}
int dpm3_update(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img, const float* noise,
                const float* x0_hist1, float* x0_hist2, float* x_prev, float* pred_x0, long long n, const vc_ddim_scalars& s, float c1,
                float c2, double* ws, cudaStream_t stream) {
  VC_REQUIRE(x && v_cond && noise && x0_hist1 && x0_hist2 && x_prev && pred_x0 && ws && n > 1, "dpm3_update: bad args");
  VC_REQUIRE(!s.use_cfg || v_uncond, "dpm3_update: CFG needs the unconditional output");
  VC_REQUIRE(!v_uncond_img || s.use_cfg, "dpm3_update: the image-only branch is only defined with CFG on");
  VC_REQUIRE(x0_hist1 != x0_hist2 && x0_hist1 != x_prev && x0_hist1 != pred_x0 && x0_hist2 != x_prev && x0_hist2 != pred_x0 &&
             x0_hist2 != x && x_prev != pred_x0, "dpm3_update: x0_hist1, x0_hist2, x_prev and pred_x0 must not alias");
  VC_REQUIRE(isfinite(c1) && isfinite(c2), "dpm3_update: c1 and c2 must be finite");
  return dpm_launch(x, v_cond, v_uncond, v_uncond_img, cfg_img, noise, x0_hist1, x0_hist2, x_prev, pred_x0, n, s, c1, c2, ws, stream);
}

// ------------------------------------------------------------------------------------------------
// row softmax (fp32 scores -> fp16 probabilities) for the VAE's single-head d=512 AttnBlock (ae_modules.py:66-68)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ x, long long cols, float scale, __half* __restrict__ out) {
  __shared__ float red[8];
  const float* xr = x + (long long)blockIdx.x * cols;
  __half* orow = out + (long long)blockIdx.x * cols;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  float m = -INFINITY;
  for (long long i = tid; i < cols; i += 256) m = fmaxf(m, xr[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red[w] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float l = 0.f;
  for (long long i = tid; i < cols; i += 256) l += __expf((xr[i] - m) * scale);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
  if (lane == 0) red[w] = l;
  __syncthreads();
  l = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) l += red[i];
  const float inv = 1.f / l;
  for (long long i = tid; i < cols; i += 256) orow[i] = __float2half_rn(__expf((xr[i] - m) * scale) * inv);
}
int softmax_rows_f32(const float* x, long long rows, long long cols, float scale, __half* out, cudaStream_t stream) {
  VC_REQUIRE(x && out && rows > 0 && cols > 0 && scale > 0.f, "softmax_rows: bad args");
  softmax_rows_kernel<<<(unsigned)rows, 256, 0, stream>>>(x, cols, scale, out);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

}  // namespace vc

// HBM-bound normalisation kernels on channels-last fp16 activations.
//   groupnorm_nhwc : GroupNorm(32) (+SiLU) over [samples, rows, C]; C may be the concat of two tensors.
//                    pass 1 = per-CTA partial (sum, sumsq) per group (deterministic, no atomics to global),
//                    pass 2 = finalize stats in smem + normalise/affine/SiLU with 16-byte vector I/O.
//   layernorm_rows : LayerNorm over the last dim, one warp per token row, values held in registers.
// Reference semantics: lvdm/basics.py:76-87 (fp32 GroupNorm), attention.py:265,331 (eps 1e-6),
// openaimodel3d.py:256-265 (5-D GroupNorm in TemporalConvBlock), torch.nn.LayerNorm (eps 1e-5).
#include "common.cuh"
#include "kernels.h"

namespace vc {

static constexpr int GN_MAX_SPLITS = 512;

size_t groupnorm_ws_bytes(int samples) { return (size_t)samples * GN_MAX_SPLITS * 64 * sizeof(float) + (size_t)samples * sizeof(unsigned int); }

struct GnGeom {
  int C, C1, C2, vecs, ppi, cg, splits;
  long long rows, rows_per_split;
  int stat_splits;        // partial-statistics records per sample the apply pass sums
  long long stat_rows;    // rows the statistics cover (== rows, or the global row count when sharded across GPUs)
};

// Per-thread view of the rows a CTA owns: thread (pl, v) handles channel vector v (8 channels) of rows r0 + pl + k * ppi.
// Pointers are formed once and advanced by a constant stride: the loops below are pure streaming and were instruction-
// issue bound when every load recomputed a 64-bit (row * C + c) address and re-decided which of the two sources to read.
struct GnThread {
  const __half* src;      // first element this thread reads
  long long sstride;      // elements between this thread's consecutive rows in the source
  long long n;            // rows this thread handles
  long long orow0;        // first output row (sample-relative)
};
__device__ __forceinline__ GnThread gn_thread(const __half* x1, const __half* x2, const GnGeom& g, int split, int sample, int v, int pl) {
  GnThread t;
  const long long r0 = (long long)split * g.rows_per_split;
  const long long r1 = min(g.rows, r0 + g.rows_per_split);
  const long long first = r0 + pl;
  t.n = first < r1 ? (r1 - first + g.ppi - 1) / g.ppi : 0;
  t.orow0 = first;
  const int c = v * 8;
  const long long r = (long long)sample * g.rows + first;
  if (c < g.C1) { t.src = x1 + r * g.C1 + c; t.sstride = (long long)g.ppi * g.C1; }
  else { t.src = x2 + r * g.C2 + (c - g.C1); t.sstride = (long long)g.ppi * g.C2; }
  return t;
}

__device__ __forceinline__ void gn_acc8(const uint4& u, float (&s)[8], float (&ss)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 f = __half22float2(h[e]);
    s[2 * e] += f.x; ss[2 * e] = fmaf(f.x, f.x, ss[2 * e]);
    s[2 * e + 1] += f.y; ss[2 * e + 1] = fmaf(f.y, f.y, ss[2 * e + 1]);
  }
}

__device__ __forceinline__ void gn_stats_dev(const __half* __restrict__ x1, const __half* __restrict__ x2, const GnGeom& g,
                                                        float* __restrict__ partial, const int split, const int sample) {
  // red[pl][2*C]: one row of per-channel (sum | sumsq) per pixel lane, reduced in a FIXED order below -- no float atomics, so the
  // statistics (and with them the whole forward) are bit-reproducible from run to run
  extern __shared__ float red[];
  const int tid = threadIdx.x;
  const int v = tid % g.vecs, pl = tid / g.vecs;
  float s[8], ss[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) s[e] = ss[e] = 0.f;
  const GnThread t = gn_thread(x1, x2, g, split, sample, v, pl);
  const __half* p = t.src;
  long long k = 0;
  // 8 independent 16-byte loads in flight per thread (pure streaming: latency is covered by memory-level parallelism)
  for (; k + 8 <= t.n; k += 8, p += 8 * t.sstride) {
    uint4 u[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) u[i] = *reinterpret_cast<const uint4*>(p + i * t.sstride);
#pragma unroll
    for (int i = 0; i < 8; ++i) gn_acc8(u[i], s, ss);
  }
  for (; k < t.n; ++k, p += t.sstride) gn_acc8(*reinterpret_cast<const uint4*>(p), s, ss);
  float* mine = red + (long long)pl * 2 * g.C;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    mine[v * 8 + e] = s[e];
    mine[g.C + v * 8 + e] = ss[e];
  }
  __syncthreads();
  if (tid < 64) {
    const int grp = tid >> 1, which = tid & 1;
    float acc = 0.f;
    for (int q = 0; q < g.ppi; ++q) {
      const float* row = red + (long long)q * 2 * g.C + which * g.C;
      for (int c = grp * g.cg; c < (grp + 1) * g.cg; ++c) acc += row[c];
    }
    partial[((long long)sample * g.splits + split) * 64 + tid] = acc;
  }
  __syncthreads();                                  // red[] may be rewritten by the caller's next use
}

// x * sigmoid(x) = h + h * tanh(h) with h = x / 2: one MUFU.TANH + 2 FP ops per element instead of MUFU.EX2 + MUFU.RCP + 3.  The
// normalise pass issues 2 MUFU per element otherwise and is then bound by the 16-per-clock MUFU pipe rather than by HBM.  tanh.approx.f32 has a relative error of 2^-11 on tanh, i.e. an absolute error of
// <= 2.4e-4 |x| on the result -- the size of the fp16 rounding the output gets anyway.
__device__ __forceinline__ float gn_silu(float x) {
  const float h = 0.5f * x;
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
  return fmaf(h, t, h);
}

__device__ __forceinline__ uint4 gn_norm8(const uint4& u, const float (&sc)[8], const float (&sh)[8], int silu) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
  float f[8];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 t2 = __half22float2(h[e]);
    f[2 * e] = fmaf(t2.x, sc[2 * e], sh[2 * e]);
    f[2 * e + 1] = fmaf(t2.y, sc[2 * e + 1], sh[2 * e + 1]);
  }
  if (silu) {
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = gn_silu(f[e]);
  }
  uint4 o;
  o.x = pack_half2(f[0], f[1]); o.y = pack_half2(f[2], f[3]);
  o.z = pack_half2(f[4], f[5]); o.w = pack_half2(f[6], f[7]);
  return o;
}

__device__ __forceinline__ void gn_apply_dev(const __half* __restrict__ x1, const __half* __restrict__ x2, const GnGeom& g,
                                                        const float* __restrict__ partial, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float eps, int silu, __half* __restrict__ out,
                                                        const int split, const int sample) {
  __shared__ float mean_s[32], rstd_s[32];
  const int tid = threadIdx.x;
  if (tid < 32) {
    double sum = 0.0, sq = 0.0;
    const float* pp = partial + (long long)sample * g.stat_splits * 64;
    for (int sp = 0; sp < g.stat_splits; ++sp) {
      sum += pp[sp * 64 + tid * 2];
      sq += pp[sp * 64 + tid * 2 + 1];
    }
    const double n = (double)g.stat_rows * g.cg;
    const double m = sum / n;
    double var = sq / n - m * m;
    if (var < 0.0) var = 0.0;
    mean_s[tid] = (float)m;
    rstd_s[tid] = (float)(1.0 / sqrt(var + (double)eps));
  }
  __syncthreads();
  const int v = tid % g.vecs, pl = tid / g.vecs;
  float sc[8], sh[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int c = v * 8 + e;
    const int grp = c / g.cg;
    const float a = rstd_s[grp] * gamma[c];
    sc[e] = a;
    sh[e] = beta[c] - mean_s[grp] * a;
  }
  const GnThread t = gn_thread(x1, x2, g, split, sample, v, pl);
  const long long ostride = (long long)g.ppi * g.C;
  // Walk the rows BACKWARDS: in the fused kernel the statistics pass streamed them forwards, so what the L2 still
  // holds is the tail of every CTA's slice; a second forward sweep is the worst case for an LRU-like cache, the reverse sweep meets
  // the resident lines first.
  // Software pipeline: the loads of the NEXT four rows are issued before the current four are normalised and stored, so up to eight
  // 16-byte loads per thread are in flight and the DRAM latency is covered when this pass is the only one (statistics from the
  // producing GEMM: no L2-resident tail to meet).
  const long long ds = -t.sstride, dd = -ostride;
  const __half* p = t.src + (t.n - 1) * t.sstride;
  __half* o = out + ((long long)sample * g.rows + t.orow0) * g.C + v * 8 + (t.n - 1) * ostride;
  long long left = t.n;
  uint4 cur[4], nxt[4];
  int ncur = left < 4 ? (int)left : 4;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (i < ncur) cur[i] = *reinterpret_cast<const uint4*>(p + i * ds);
  left -= ncur; p += ncur * ds;
  while (ncur > 0) {
    const int nn = left < 4 ? (int)left : 4;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (i < nn) nxt[i] = *reinterpret_cast<const uint4*>(p + i * ds);
    left -= nn; p += nn * ds;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (i < ncur) *reinterpret_cast<uint4*>(o + i * dd) = gn_norm8(cur[i], sc, sh, silu);
    o += ncur * dd;
#pragma unroll
    for (int i = 0; i < 4; ++i) cur[i] = nxt[i];
    ncur = nn;
  }
}

__global__ void __launch_bounds__(512) gn_stats_kernel(const __half* __restrict__ x1, const __half* __restrict__ x2, GnGeom g,
                                                       float* __restrict__ partial) {
  gn_stats_dev(x1, x2, g, partial, blockIdx.x, blockIdx.y);
}
__global__ void __launch_bounds__(512, 2) gn_apply_kernel(const __half* __restrict__ x1, const __half* __restrict__ x2, GnGeom g,
                                                       const float* __restrict__ partial, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, float eps, int silu, __half* __restrict__ out) {
  gn_apply_dev(x1, x2, g, partial, gamma, beta, eps, silu, out, blockIdx.x, blockIdx.y);
}
// Fused single launch: statistics pass, a grid-wide rendezvous of the CTAs of one sample (all CTAs are co-resident by
// construction -- the host checks the occupancy), then the normalise pass, whose re-read of x is served by the L2 (50 MB
// on H100) when a sample fits it: HBM traffic drops from 3 passes to ~2.
__global__ void __launch_bounds__(512, 2) gn_fused_kernel(const __half* __restrict__ x1, const __half* __restrict__ x2, GnGeom g,
                                                        float* __restrict__ partial, unsigned int* __restrict__ counters,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int silu,
                                                        __half* __restrict__ out) {
  gn_stats_dev(x1, x2, g, partial, blockIdx.x, blockIdx.y);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicAdd(&counters[blockIdx.y], 1u);
    unsigned long long spins = 0;
    while (*reinterpret_cast<volatile unsigned int*>(&counters[blockIdx.y]) < (unsigned)g.splits) {
      __nanosleep(40);
      if (++spins > 200000000ull) __trap();      // cannot happen under a cooperative launch; never hang the device
    }
    __threadfence();
  }
  __syncthreads();
  gn_apply_dev(x1, x2, g, partial, gamma, beta, eps, silu, out, blockIdx.x, blockIdx.y);
}

static int gn_geometry(GnGeom& g, const __half* x1, int C1, const __half* x2, int C2, int samples, long long rows_per_sample) {
  const int C = C1 + (x2 ? C2 : 0);
  VC_REQUIRE(x1, "groupnorm: null pointer");
  VC_REQUIRE(((reinterpret_cast<uintptr_t>(x1) | reinterpret_cast<uintptr_t>(x2)) & 15) == 0,
             "groupnorm: inputs must be 16-byte aligned (rows are read as 8-channel vectors)");
  VC_REQUIRE(C % 32 == 0 && C1 % 8 == 0 && (!x2 || C2 % 8 == 0) && C <= 4096, "groupnorm: unsupported channels C1=%d C2=%d", C1, C2);
  VC_REQUIRE(samples >= 1 && rows_per_sample >= 1, "groupnorm: empty input");
  g.C = C; g.C1 = C1; g.C2 = x2 ? C2 : 0;
  g.vecs = C / 8;
  g.ppi = 512 / g.vecs > 0 ? 512 / g.vecs : 1;
  g.cg = C / 32;
  g.rows = rows_per_sample;
  int splits = (2 * sm_count() + samples - 1) / samples;
  const long long max_useful = (rows_per_sample + g.ppi - 1) / g.ppi;
  if (splits > max_useful) splits = (int)max_useful;
  if (splits > GN_MAX_SPLITS) splits = GN_MAX_SPLITS;
  if (splits < 1) splits = 1;
  g.splits = splits;
  g.rows_per_split = (rows_per_sample + splits - 1) / splits;
  g.stat_splits = splits;
  g.stat_rows = rows_per_sample;
  return VC_OK;
}

int groupnorm_nhwc(const __half* x1, int C1, const __half* x2, int C2, int samples, long long rows_per_sample,
                   const float* gamma, const float* beta, float eps, int silu, __half* out, float* partial_ws,
                   size_t ws_bytes, cudaStream_t stream) {
  VC_REQUIRE(out && gamma && beta && partial_ws, "groupnorm: null pointer");
  GnGeom g;
  int rc = gn_geometry(g, x1, C1, x2, C2, samples, rows_per_sample);
  if (rc) return rc;
  VC_REQUIRE(ws_bytes >= (size_t)samples * g.splits * 64 * sizeof(float), "groupnorm: workspace too small");
  const int threads = g.vecs * g.ppi;
  dim3 grid(g.splits, samples);
  const size_t smem = (size_t)2 * g.C * g.ppi * sizeof(float);
  // fused path: the statistics -> normalise hand-over is a grid-wide rendezvous, so every CTA must be resident at once.
  // The launch is COOPERATIVE: the driver either co-schedules the whole grid or refuses the launch -- it cannot hang when
  // other work holds SMs (the occupancy figure only sizes the grid).
  const size_t part_bytes = (size_t)samples * g.splits * 64 * sizeof(float);
  int per_sm = 0;
  VC_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gn_fused_kernel, threads, smem));
  const long long capacity = (long long)per_sm * sm_count();
  if (capacity < (long long)g.splits * samples && capacity >= samples) {   // shrink the split so that every CTA is resident
    g.splits = (int)(capacity / samples);
    g.rows_per_split = (rows_per_sample + g.splits - 1) / g.splits;
    g.stat_splits = g.splits;
    grid = dim3(g.splits, samples);
  }
  const bool fused = capacity >= (long long)g.splits * samples && ws_bytes >= part_bytes + samples * sizeof(unsigned int);
  if (fused) {
    unsigned int* counters = reinterpret_cast<unsigned int*>(reinterpret_cast<char*>(partial_ws) + part_bytes);
    VC_CHECK_CUDA(cudaMemsetAsync(counters, 0, samples * sizeof(unsigned int), stream));
    void* args[] = {(void*)&x1, (void*)&x2, (void*)&g, (void*)&partial_ws, (void*)&counters, (void*)&gamma, (void*)&beta,
                    (void*)&eps, (void*)&silu, (void*)&out};
    VC_CHECK_CUDA(cudaLaunchCooperativeKernel((const void*)gn_fused_kernel, grid, dim3(threads), args, smem, stream));
    return VC_OK;
  }
  gn_stats_kernel<<<grid, threads, smem, stream>>>(x1, x2, g, partial_ws);
  VC_CHECK_CUDA(cudaGetLastError());
  gn_apply_kernel<<<grid, threads, 0, stream>>>(x1, x2, g, partial_ws, gamma, beta, eps, silu, out);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

// Split form for statistics that span several GPUs (site-sharded 5-D GroupNorm): pass 1 leaves (sum, sumsq) per group in
// stats[samples][32][2]; the caller all-reduces that tiny buffer; pass 2 normalises with the global row count.  The per-CTA
// records are summed in fp64 and rounded once, as the single-GPU apply pass sums them: an fp32 running sum over ~260 records
// lost enough of the sum of squares to break the output bound at |mean| = 64 std.
__global__ void gn_finalize_kernel(const float* __restrict__ partial, int splits, float* __restrict__ stats) {
  const int sample = blockIdx.x, t = threadIdx.x;   // 64 threads
  double acc = 0.0;
  for (int sp = 0; sp < splits; ++sp) acc += partial[((long long)sample * splits + sp) * 64 + t];
  stats[sample * 64 + t] = (float)acc;
}

int groupnorm_stats(const __half* x1, int C1, const __half* x2, int C2, int samples, long long rows_per_sample, float* stats,
                    float* partial_ws, size_t ws_bytes, cudaStream_t stream) {
  VC_REQUIRE(stats && partial_ws, "groupnorm_stats: null pointer");
  GnGeom g;
  int rc = gn_geometry(g, x1, C1, x2, C2, samples, rows_per_sample);
  if (rc) return rc;
  VC_REQUIRE(ws_bytes >= (size_t)samples * g.splits * 64 * sizeof(float), "groupnorm: workspace too small");
  dim3 grid(g.splits, samples);
  gn_stats_kernel<<<grid, g.vecs * g.ppi, (size_t)2 * g.C * g.ppi * sizeof(float), stream>>>(x1, x2, g, partial_ws);
  VC_CHECK_CUDA(cudaGetLastError());
  gn_finalize_kernel<<<samples, 64, 0, stream>>>(partial_ws, g.splits, stats);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

// pass 1 alone: leaves splits_out records of (sum, sumsq) per group and sample in partial_ws[sample][split][64]
int groupnorm_stats_partials(const __half* x1, int C1, int samples, long long rows_per_sample, float* partial_ws, size_t ws_bytes,
                             int* splits_out, cudaStream_t stream) {
  VC_REQUIRE(partial_ws && splits_out, "groupnorm_stats_partials: null pointer");
  GnGeom g;
  int rc = gn_geometry(g, x1, C1, nullptr, 0, samples, rows_per_sample);
  if (rc) return rc;
  VC_REQUIRE(ws_bytes >= (size_t)samples * g.splits * 64 * sizeof(float), "groupnorm: workspace too small");
  dim3 grid(g.splits, samples);
  gn_stats_kernel<<<grid, g.vecs * g.ppi, (size_t)2 * g.C * g.ppi * sizeof(float), stream>>>(x1, nullptr, g, partial_ws);
  VC_CHECK_CUDA(cudaGetLastError());
  *splits_out = g.splits;
  return VC_OK;
}

int groupnorm_apply(const __half* x1, int C1, const __half* x2, int C2, int samples, long long rows_per_sample,
                    const float* stats, long long stat_rows, const float* gamma, const float* beta, float eps, int silu, __half* out,
                    cudaStream_t stream, int stat_parts) {
  VC_REQUIRE(out && gamma && beta && stats && stat_rows >= rows_per_sample && stat_parts >= 1, "groupnorm_apply: bad args");
  GnGeom g;
  int rc = gn_geometry(g, x1, C1, x2, C2, samples, rows_per_sample);
  if (rc) return rc;
  g.stat_splits = stat_parts;                   // stats = [samples][stat_parts][32][2] partial sums (1: already reduced)
  g.stat_rows = stat_rows;
  dim3 grid(g.splits, samples);
  gn_apply_kernel<<<grid, g.vecs * g.ppi, 0, stream>>>(x1, x2, g, stats, gamma, beta, eps, silu, out);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

// ------------------------------------------------------------------------------------------------
// Reproducible mode: canonical GroupNorm statistics ("leaves").  A leaf is the (sum, sumsq) per group of one block of
// rows_per_leaf contiguous rows (one chunk of a frame's pixels); one CTA computes one leaf with the thread mapping and fixed
// reduction order of gn_stats_dev, so a leaf depends only on its rows and on (rows_per_leaf, C1, C2) -- not on where the block
// sits, how many leaves the launch has or the SM count.  The frame layout and the site layout of the multi-GPU U-Net hold the
// same chunks whole, so both produce bit-identical leaves.
__global__ void __launch_bounds__(512) gn_leaves_kernel(const __half* __restrict__ x1, const __half* __restrict__ x2, GnGeom g,
                                                        float* __restrict__ leaves) {
  gn_stats_dev(x1, x2, g, leaves, 0, blockIdx.x);
}

// stats[s][64] = sum of the leaves [s * per_sample, (s + 1) * per_sample) in index order (fp64, rounded once to fp32)
__global__ void __launch_bounds__(64) gn_leaves_combine_kernel(const float* __restrict__ leaves, int per_sample, float* __restrict__ stats) {
  const int s = blockIdx.x, t = threadIdx.x;
  const float* p = leaves + (long long)s * per_sample * 64 + t;
  double acc = 0.0;
  int i = 0;
  for (; i + 8 <= per_sample; i += 8) {            // loads first, then the adds in index order
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = __ldg(p + (long long)(i + k) * 64);
#pragma unroll
    for (int k = 0; k < 8; ++k) acc += (double)v[k];
  }
  for (; i < per_sample; ++i) acc += (double)__ldg(p + (long long)i * 64);
  stats[s * 64 + t] = (float)acc;
}

int groupnorm_leaves(const __half* x1, int C1, const __half* x2, int C2, long long n_leaves, long long rows_per_leaf, float* leaves,
                     cudaStream_t stream) {
  VC_REQUIRE(leaves && n_leaves >= 1 && n_leaves <= 0x7fffffffll, "groupnorm_leaves: bad args");
  GnGeom g;
  int rc = gn_geometry(g, x1, C1, x2, C2, 1, rows_per_leaf);
  if (rc) return rc;
  g.splits = 1; g.rows_per_split = rows_per_leaf;      // one CTA per leaf: nothing below depends on the device
  g.stat_splits = 1; g.stat_rows = rows_per_leaf;
  gn_leaves_kernel<<<(unsigned)n_leaves, g.vecs * g.ppi, (size_t)2 * g.C * g.ppi * sizeof(float), stream>>>(x1, x2, g, leaves);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

int groupnorm_apply_leaves(const __half* x1, int C1, const __half* x2, int C2, int samples, long long rows_per_sample, const float* leaves,
                           int leaves_per_sample, long long stat_rows, const float* gamma, const float* beta, float eps, int silu,
                           __half* out, float* ws, size_t ws_bytes, cudaStream_t stream) {
  VC_REQUIRE(leaves && ws && samples >= 1 && leaves_per_sample >= 1, "groupnorm_apply_leaves: bad args");
  VC_REQUIRE(ws_bytes >= (size_t)samples * 64 * sizeof(float), "groupnorm_apply_leaves: workspace too small");
  gn_leaves_combine_kernel<<<samples, 64, 0, stream>>>(leaves, leaves_per_sample, ws);
  VC_CHECK_CUDA(cudaGetLastError());
  return groupnorm_apply(x1, C1, x2, C2, samples, rows_per_sample, ws, stat_rows, gamma, beta, eps, silu, out, stream, 1);
}

// ------------------------------------------------------------------------------------------------
// GroupNorm from the partial sums the producing GEMM left behind (vc_gemm_desc::gn_part, gemm_common.cuh: gn_part_accumulate):
// the statistics pass over the activation disappears -- a small kernel folds the per-(32-row block, chunk, piece) records
// (1.6 % of the activation's bytes) into per-(sample, split, group) sums in a fixed order, and gn_apply_kernel normalises in
// one read + one write.  Reference semantics as above (basics.py:76-87, openaimodel3d.py:256-265).
struct GnFin {
  const float2* part;
  int cols;               // n_chunks * 4 records per 32-row block
  int sub;
  long long rb_per_z, rb_per_sample;
  int spz;
  int cg, c_off, C_src;   // consumer group width, channel offset of this source in the concat, channels of this source
  int lanes;              // row-block lanes per CTA (blockDim.x == cols * lanes)
  int nsplit, split_off, total_splits;
};
__global__ void __launch_bounds__(1024) gn_part_finalize_kernel(GnFin f, float* __restrict__ records) {
  __shared__ float2 red[1024];
  const int tid = threadIdx.x, split = blockIdx.x, s = blockIdx.y;
  const int col = tid % f.cols, ln = tid / f.cols;
  const long long per = (f.rb_per_sample + f.nsplit - 1) / f.nsplit;
  const long long r0 = (long long)split * per, r1 = min(f.rb_per_sample, r0 + per);
  const long long base = (long long)(s / f.spz) * f.rb_per_z + (long long)(s % f.spz) * f.rb_per_sample;
  float sum = 0.f, sq = 0.f;
  const float2* p = f.part + (base + r0 + ln) * f.cols + col;
  const long long step = (long long)f.lanes * f.cols;
  long long rb = r0 + ln;
  for (; rb + 3 * f.lanes < r1; rb += 4 * f.lanes, p += 4 * step) {      // 4 independent loads in flight
    const float2 a = __ldg(p), b = __ldg(p + step), c = __ldg(p + 2 * step), d = __ldg(p + 3 * step);
    sum += a.x; sq += a.y; sum += b.x; sq += b.y; sum += c.x; sq += c.y; sum += d.x; sq += d.y;
  }
  for (; rb < r1; rb += f.lanes, p += step) {
    const float2 a = __ldg(p);
    sum += a.x; sq += a.y;
  }
  red[tid] = make_float2(sum, sq);
  __syncthreads();
  if (tid < f.cols) {
    float2 acc = red[tid];
    for (int l = 1; l < f.lanes; ++l) { const float2 o = red[l * f.cols + tid]; acc.x += o.x; acc.y += o.y; }
    red[tid] = acc;
  }
  __syncthreads();
  if (tid < 64) {
    // group `grp` of the consumer = the sub-groups [sg_lo, sg_hi) of this source; sub-group sg has one record in every chunk it touches
    // (at most two): chunk c holds it as piece sg - (32 c) / sub
    const int grp = tid >> 1, which = tid & 1;
    const int ch_lo = max(grp * f.cg - f.c_off, 0), ch_hi = min((grp + 1) * f.cg - f.c_off, f.C_src);
    float acc = 0.f;
    if (ch_hi > ch_lo) {
      const int sg_lo = ch_lo / f.sub, sg_hi = ch_hi / f.sub;
      for (int sg = sg_lo; sg < sg_hi; ++sg) {
        const int c_lo = (sg * f.sub) >> 5, c_hi = (sg * f.sub + f.sub - 1) >> 5;
        for (int c = c_lo; c <= c_hi; ++c) {
          const int k = sg - (c * 32) / f.sub;
          if (k >= 0 && k < 4) acc += which ? red[c * 4 + k].y : red[c * 4 + k].x;
        }
      }
    }
    records[((long long)s * f.total_splits + f.split_off + split) * 64 + tid] = acc;
  }
}

static constexpr int GN_PART_MAX_SPLITS = 64;          // per source
size_t groupnorm_parts_ws_bytes(int samples) { return (size_t)samples * 2 * GN_PART_MAX_SPLITS * 64 * sizeof(float); }

static int gn_part_plan(const vc_gn_part_geom& g, int C_src, int samples, GnFin& f) {
  VC_REQUIRE(g.part && g.n_chunks * 32 == C_src && (g.sub == 10 || g.sub == 8) && g.rb_per_sample >= 1 && g.samples_per_z >= 1 &&
             g.rb_per_z >= (long long)g.samples_per_z * g.rb_per_sample, "groupnorm_from_parts: bad partial-sum geometry");
  f.part = reinterpret_cast<const float2*>(g.part);
  f.cols = g.n_chunks * 4; f.sub = g.sub;
  f.rb_per_z = g.rb_per_z; f.rb_per_sample = g.rb_per_sample; f.spz = g.samples_per_z;
  f.C_src = C_src;
  VC_REQUIRE(f.cols <= 1024, "groupnorm_from_parts: too many channels");
  f.lanes = 256 / f.cols > 0 ? 256 / f.cols : 1;
  int nsplit = (2 * sm_count() + samples - 1) / samples;
  const long long max_useful = (g.rb_per_sample + 16 * f.lanes - 1) / (16 * f.lanes);     // >= 16 records per thread
  if (nsplit > max_useful) nsplit = (int)max_useful;
  if (nsplit > GN_PART_MAX_SPLITS) nsplit = GN_PART_MAX_SPLITS;
  if (nsplit < 1) nsplit = 1;
  f.nsplit = nsplit;
  return VC_OK;
}

// The finalize step alone for ONE source: partial_ws[sample][split][64] = per-group (sum, sumsq) over the sample's rows ON THIS RANK,
// from the producer's records -- the input of the cross-GPU statistics exchange (peer.cu: gn_peer_allreduce_kernel).
int groupnorm_parts_to_partials(const vc_gn_part_geom& g1, int C, int samples, float* partial_ws, size_t ws_bytes, int* splits_out,
                                cudaStream_t stream) {
  VC_REQUIRE(partial_ws && splits_out && C % 32 == 0, "groupnorm_parts_to_partials: bad args");
  GnFin f;
  int rc = gn_part_plan(g1, C, samples, f);
  if (rc) return rc;
  f.cg = C / 32; f.c_off = 0; f.split_off = 0; f.total_splits = f.nsplit;
  VC_REQUIRE(f.cg % g1.sub == 0, "groupnorm_parts_to_partials: group width %d vs sub-group width %d", f.cg, g1.sub);
  VC_REQUIRE(ws_bytes >= (size_t)samples * f.nsplit * 64 * sizeof(float), "groupnorm_parts_to_partials: workspace too small");
  gn_part_finalize_kernel<<<dim3(f.nsplit, samples), f.cols * f.lanes, 0, stream>>>(f, partial_ws);
  VC_CHECK_CUDA(cudaGetLastError());
  *splits_out = f.nsplit;
  return VC_OK;
}

int groupnorm_from_parts(const __half* x1, int C1, const vc_gn_part_geom& g1, const __half* x2, int C2, const vc_gn_part_geom& g2,
                         int samples,
                         long long rows_per_sample, const float* gamma, const float* beta, float eps, int silu, __half* out, float* ws,
                         size_t ws_bytes, cudaStream_t stream) {
  VC_REQUIRE(out && gamma && beta && ws, "groupnorm_from_parts: null pointer");
  GnGeom g;
  int rc = gn_geometry(g, x1, C1, x2, C2, samples, rows_per_sample);
  if (rc) return rc;
  VC_REQUIRE(ws_bytes >= groupnorm_parts_ws_bytes(samples), "groupnorm_from_parts: workspace too small");
  GnFin f1, f2;
  rc = gn_part_plan(g1, C1, samples, f1);
  if (rc) return rc;
  f1.cg = g.cg; f1.c_off = 0; f1.split_off = 0;
  VC_REQUIRE(g.cg % g1.sub == 0, "groupnorm_from_parts: group width %d is not a multiple of the sub-group width %d", g.cg, g1.sub);
  int total = f1.nsplit;
  if (x2) {
    rc = gn_part_plan(g2, C2, samples, f2);
    if (rc) return rc;
    VC_REQUIRE(g.cg % g2.sub == 0 && C1 % g2.sub == 0, "groupnorm_from_parts: concat boundary %d / group width %d vs sub-group width %d", C1, g.cg, g2.sub);
    f2.cg = g.cg; f2.c_off = C1; f2.split_off = f1.nsplit;
    total += f2.nsplit;
  }
  f1.total_splits = total;
  gn_part_finalize_kernel<<<dim3(f1.nsplit, samples), f1.cols * f1.lanes, 0, stream>>>(f1, ws);
  VC_CHECK_CUDA(cudaGetLastError());
  if (x2) {
    f2.total_splits = total;
    gn_part_finalize_kernel<<<dim3(f2.nsplit, samples), f2.cols * f2.lanes, 0, stream>>>(f2, ws);
    VC_CHECK_CUDA(cudaGetLastError());
  }
  g.stat_splits = total;
  g.stat_rows = rows_per_sample;
  dim3 grid(g.splits, samples);
  gn_apply_kernel<<<grid, g.vecs * g.ppi, 0, stream>>>(x1, x2, g, ws, gamma, beta, eps, silu, out);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

// ------------------------------------------------------------------------------------------------
// Persistent warps: each warp walks rows with a grid stride and keeps TWO rows in flight (all their 16-byte loads are
// issued before the first reduction) so the DRAM latency is covered by memory-level parallelism, not by block churn.
template <int MAXV>
__global__ void __launch_bounds__(256) layernorm_kernel(const __half* __restrict__ x, long long rows, int C, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float eps, __half* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  const long long gw = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int vecs = C >> 3;
  const float invC = 1.f / (float)C;
  for (long long row0 = gw * 2; row0 < rows; row0 += nwarps * 2) {
    uint4 raw[2][MAXV];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const long long row = row0 + rr;
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        const int v = lane + i * 32;
        raw[rr][i] = (row < rows && v < vecs) ? *reinterpret_cast<const uint4*>(x + row * C + v * 8) : make_uint4(0, 0, 0, 0);
      }
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const long long row = row0 + rr;
      if (row >= rows) break;                                   // warp-uniform
      float f[MAXV][8];
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        const __half2* h = reinterpret_cast<const __half2*>(&raw[rr][i]);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 t = __half22float2(h[e]);
          f[i][2 * e] = t.x; f[i][2 * e + 1] = t.y;
          sum += t.x + t.y;                                     // out-of-range vectors were loaded as zeros
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      const float mean = sum * invC;
      float sq = 0.f;
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        if (lane + i * 32 < vecs) {
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const float d = f[i][e] - mean;
            sq += d * d;
          }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
      const float rstd = rsqrtf(sq * invC + eps);
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        const int v = lane + i * 32;
        if (v < vecs) {
          const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + v * 8 + 4));
          const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + v * 8)), b1 = __ldg(reinterpret_cast<const float4*>(beta + v * 8 + 4));
          const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
          const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
          float y[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) y[e] = (f[i][e] - mean) * rstd * gg[e] + bb[e];
          uint4 o;
          o.x = pack_half2(y[0], y[1]); o.y = pack_half2(y[2], y[3]);
          o.z = pack_half2(y[4], y[5]); o.w = pack_half2(y[6], y[7]);
          *reinterpret_cast<uint4*>(out + row * C + v * 8) = o;
        }
      }
    }
  }
}

int layernorm_rows(const __half* x, long long rows, int C, const float* gamma, const float* beta, float eps, __half* out,
                   cudaStream_t stream) {
  VC_REQUIRE(x && out && gamma && beta, "layernorm: null pointer");
  VC_REQUIRE(C % 8 == 0 && C <= 2048 && rows > 0, "layernorm: unsupported C=%d rows=%lld", C, rows);
  VC_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
             "layernorm: x and out must be 16-byte aligned (rows are read and written as 8-channel vectors)");
  const int wpb = 8;
  long long blocks = (rows + 2 * wpb - 1) / (2 * wpb);
  const long long cap = (long long)sm_count() * 8;              // 8 x 256 threads = 64 warps per SM
  if (blocks > cap) blocks = cap;
  const int vecs = C / 8;
  if (vecs <= 64)
    layernorm_kernel<2><<<(unsigned)blocks, wpb * 32, 0, stream>>>(x, rows, C, gamma, beta, eps, out);
  else if (vecs <= 160)
    layernorm_kernel<5><<<(unsigned)blocks, wpb * 32, 0, stream>>>(x, rows, C, gamma, beta, eps, out);
  else
    layernorm_kernel<8><<<(unsigned)blocks, wpb * 32, 0, stream>>>(x, rows, C, gamma, beta, eps, out);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

// Statistics half of LayerNorm: stats[row] = (mean, rstd).  The normalisation itself is folded into the consuming GEMM's
// epilogue (vc_gemm_desc::ln_stats), which turns LayerNorm from a read + write pass into this read-only pass.
// One warp per group of 4 rows, every lane keeps 4 independent 16-byte loads in flight; sums are taken about a per-row
// pivot (the row's first element) so the one-pass variance does not cancel when |mean| >> std.  ~40 registers: 48+ warps
// per SM (the register-resident two-pass kernel above runs at 16 warps per SM).
__global__ void __launch_bounds__(256) ln_stats_kernel(const __half* __restrict__ x, long long rows, int C, float eps,
                                                       float2* __restrict__ stats) {
  const int lane = threadIdx.x & 31;
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  const long long gw = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int vecs = C >> 3;
  const float invC = 1.f / (float)C;
  for (long long row0 = gw * 4; row0 < rows; row0 += nwarps * 4) {
    float piv[4], s[4], q[4];
    const __half* rp[4];
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
      const long long row = min(row0 + rr, rows - 1);            // clamp: tail rows recompute the last row (not stored)
      rp[rr] = x + row * C;
      piv[rr] = __half2float(__ldg(rp[rr]));
      s[rr] = q[rr] = 0.f;
    }
    for (int v = lane; v < vecs; v += 32) {
      uint4 u[4];
#pragma unroll
      for (int rr = 0; rr < 4; ++rr) u[rr] = *reinterpret_cast<const uint4*>(rp[rr] + v * 8);
#pragma unroll
      for (int rr = 0; rr < 4; ++rr) {
        const __half2* h = reinterpret_cast<const __half2*>(&u[rr]);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(h[e]);
          const float a = f.x - piv[rr], b = f.y - piv[rr];
          s[rr] += a + b;
          q[rr] = fmaf(a, a, fmaf(b, b, q[rr]));
        }
      }
    }
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s[rr] += __shfl_xor_sync(0xffffffffu, s[rr], o);
        q[rr] += __shfl_xor_sync(0xffffffffu, q[rr], o);
      }
    }
    if (lane < 4 && row0 + lane < rows) {
      float sm = s[0], qm = q[0], pm = piv[0];
#pragma unroll
      for (int rr = 1; rr < 4; ++rr)
        if (lane == rr) { sm = s[rr]; qm = q[rr]; pm = piv[rr]; }
      const float d = sm * invC;
      const float var = fmaxf(qm * invC - d * d, 0.f);
      stats[row0 + lane] = make_float2(pm + d, rsqrtf(var + eps));
    }
  }
}

// Default for C <= 1024: the same statistics with every 16-byte load of a warp's 4 rows issued before the first conversion
// (ITERS x 4 loads in flight per lane instead of 4).  Arithmetic and rounding order per lane are those of
// ln_stats_kernel, so the results are bit-identical.
template <int ITERS>
__global__ void __launch_bounds__(256) ln_stats_unrolled_kernel(const __half* __restrict__ x, long long rows, int C, float eps,
                                                                float2* __restrict__ stats) {
  const int lane = threadIdx.x & 31;
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  const long long gw = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int vecs = C >> 3;
  const float invC = 1.f / (float)C;
  for (long long row0 = gw * 4; row0 < rows; row0 += nwarps * 4) {
    float piv[4], s[4], q[4];
    const __half* rp[4];
    uint4 u[ITERS][4];
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
      const long long row = min(row0 + rr, rows - 1);
      rp[rr] = x + row * C;
    }
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
      const int v = lane + it * 32;
#pragma unroll
      for (int rr = 0; rr < 4; ++rr) u[it][rr] = v < vecs ? *reinterpret_cast<const uint4*>(rp[rr] + v * 8) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
      piv[rr] = __half2float(__ldg(rp[rr]));
      s[rr] = q[rr] = 0.f;
    }
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
      if (lane + it * 32 < vecs) {
#pragma unroll
        for (int rr = 0; rr < 4; ++rr) {
          const __half2* h = reinterpret_cast<const __half2*>(&u[it][rr]);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(h[e]);
            const float a = f.x - piv[rr], b = f.y - piv[rr];
            s[rr] += a + b;
            q[rr] = fmaf(a, a, fmaf(b, b, q[rr]));
          }
        }
      }
    }
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s[rr] += __shfl_xor_sync(0xffffffffu, s[rr], o);
        q[rr] += __shfl_xor_sync(0xffffffffu, q[rr], o);
      }
    }
    if (lane < 4 && row0 + lane < rows) {
      float sm = s[0], qm = q[0], pm = piv[0];
#pragma unroll
      for (int rr = 1; rr < 4; ++rr)
        if (lane == rr) { sm = s[rr]; qm = q[rr]; pm = piv[rr]; }
      const float d = sm * invC;
      const float var = fmaxf(qm * invC - d * d, 0.f);
      stats[row0 + lane] = make_float2(pm + d, rsqrtf(var + eps));
    }
  }
}

// (mean, rstd) per row from the per-32-column records a producing GEMM left in parts[C/32][rows] (vc_gemm_desc::ln_part): reads
// C/32 * 8 bytes per row instead of 2 C bytes -- the LayerNorm statistics pass without re-reading the activation.  A record is
// (sum, M2 about the chunk's mean); the chunks are merged in index order with Chan's formula,
//   mean = sum_c s_c / C,   M2 = sum_c M2_c + 32 sum_c (s_c / 32 - mean)^2,
// so no term cancels when |mean| >> std.  The mean is a true division: a constant row gets its value back, and variance 0.
__global__ void __launch_bounds__(256) ln_finalize_kernel(const float2* __restrict__ parts, long long rows, int nchunks, float eps,
                                                          float2* __restrict__ stats) {
  const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= rows) return;
  const float2* p = parts + row;
  float s = 0.f;
  for (int c = 0; c < nchunks; ++c) s += __ldg(p + (long long)c * rows).x;
  const float C = 32.f * (float)nchunks;
  const float mean = s / C;
  float m2 = 0.f, between = 0.f;
  for (int c = 0; c < nchunks; ++c) {
    const float2 v = __ldg(p + (long long)c * rows);
    const float d = v.x * (1.f / 32.f) - mean;
    m2 += v.y;
    between = fmaf(d, d, between);
  }
  const float var = fmaf(32.f, between, m2) / C;
  stats[row] = make_float2(mean, rsqrtf(var + eps));
}

int layernorm_stats_from_parts(const float* parts, long long rows, int C, float eps, float* stats, cudaStream_t stream) {
  VC_REQUIRE(parts && stats && rows > 0 && C % 32 == 0, "layernorm_stats_from_parts: bad args");
  ln_finalize_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float2*>(parts), rows, C / 32, eps,
                                                                        reinterpret_cast<float2*>(stats));
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

int layernorm_stats(const __half* x, long long rows, int C, float eps, float* stats, cudaStream_t stream) {
  VC_REQUIRE(x && stats, "layernorm_stats: null pointer");
  VC_REQUIRE(C % 8 == 0 && C <= 8192 && rows > 0, "layernorm_stats: unsupported C=%d rows=%lld", C, rows);
  VC_REQUIRE((reinterpret_cast<uintptr_t>(stats) & 7) == 0, "layernorm_stats: stats must be 8-byte aligned");
  VC_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "layernorm_stats: x must be 16-byte aligned (rows are read as 8-channel vectors)");
  const int wpb = 8;
  long long blocks = (rows + 4 * wpb - 1) / (4 * wpb);
  const long long cap = (long long)sm_count() * 8;              // 8 x 256 threads = 64 warps per SM
  if (blocks > cap) blocks = cap;
  const int iters = (C / 8 + 31) / 32;
  if (iters <= 2)
    ln_stats_unrolled_kernel<2><<<(unsigned)blocks, wpb * 32, 0, stream>>>(x, rows, C, eps, reinterpret_cast<float2*>(stats));
  else if (iters <= 4)
    ln_stats_unrolled_kernel<4><<<(unsigned)blocks, wpb * 32, 0, stream>>>(x, rows, C, eps, reinterpret_cast<float2*>(stats));
  else
    ln_stats_kernel<<<(unsigned)blocks, wpb * 32, 0, stream>>>(x, rows, C, eps, reinterpret_cast<float2*>(stats));
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

}  // namespace vc

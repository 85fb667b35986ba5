// Internal C++ launch interface of the sm_90a kernels (the public boundary is include/vc_b200.h).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vc {

// Output of a GEMM scattered to the receive buffers of the ranks of a frame group (layout switch fused into the epilogue, gemm_common.cuh)
struct GemmPeerDesc {
  int mode = 0;                 // 1: frames -> sites, 2: sites -> frames
  int world = 1, rank = 0;
  int B = 1, T = 1, HW = 1;     // batch elements on this rank, frames of the clip, pixels per frame
  int f0[9] = {0};              // frame ranges of the ranks: rank q owns [f0[q], f0[q + 1])
  void* dst[8] = {nullptr};     // rank q's receive buffer of the destination layout, as mapped into this process
};

struct GemmDesc {
  // A operand: fp16, logical (K channels, X, Y, Z) with row pitch lda elements; optional second K-slab a2.
  const __half* a = nullptr; int lda = 0;
  const __half* a2 = nullptr; int lda2 = 0;
  int X = 0, Y = 1, Z = 1;        // spatial extents (linear: X = M rows)
  int bx = 128, by = 1;           // TMA box: bx*by == 128 rows per tile
  int K = 0, K1 = 0;              // reduction length per tap; K1 = part served by `a`
  const __half* w = nullptr;      // weights [num_taps*N, K] fp16, K contiguous
  int ldw = 0;                    // row pitch of w in elements (0 = K)
  int N = 0;
  int num_taps = 1;
  int tap_dx[9] = {0}; int tap_dy[9] = {0};
  __half* out = nullptr; float* out_f32 = nullptr; int ldo = 0;
  // optional output pitches (elements) along Y and Z; 0 = dense (ldo * X, ldo * X * Y).  Non-dense outputs are written by the
  // TMA-store epilogue only (fp16, N % 32 == 0): used to interleave the four parity sub-convolutions of upsample+conv.
  long long ldo_y = 0, ldo_z = 0;
  const float* bias = nullptr; int bias_z_div = 0;
  const __half* res = nullptr; int ldr = 0;
  int geglu = 0;
  // LayerNorm folded into the epilogue: the GEMM runs on the RAW rows x with weights pre-scaled by the LayerNorm gamma,
  //   out[r,n] = rstd[r] * (acc[r,n] - mean[r] * ln_colsum[n]) + bias[n]      (bias holds W.beta + linear bias)
  // ln_stats: [rows][2] fp32 (mean, rstd) from layernorm_stats; ln_colsum[n] = sum_k w[n,k] (of the fp16 weights). 1 tap only.
  const float* ln_stats = nullptr;
  const float* ln_colsum = nullptr;
  // LayerNorm statistics of the OUTPUT, gathered in the epilogue: ln_part[(n / 32) * X + row] = (sum, sumsq) over the 32 output
  // columns [n, n + 32) of the row, of the fp16-rounded values; layernorm_stats_from_parts turns them into (mean, rstd)
  float* ln_part = nullptr;
  // GroupNorm statistics of the OUTPUT, gathered in the epilogue (gemm_common.cuh: gn_part_accumulate): per 32-row block
  // rb = m_tile * 4 + quadrant (m-tiles in x, y, z order), 32-column chunk and piece,
  // gn_part[((rb * (N / 32) + chunk) * 4 + piece) * 2] = (sum, sumsq) of the fp16-rounded outputs; chunks are cut at multiples of
  // gn_sub channels (10 or 8).  groupnorm_from_parts() turns them into per-group statistics and normalises in ONE pass.
  float* gn_part = nullptr;
  int gn_sub = 0;
  const GemmPeerDesc* peer = nullptr;
  // FP8 mode: w points to e4m3 weights (ldw in elements = bytes), out[r, n] starts from acc * (s_a * w_scale[n]) with
  // s_a = *a_amax / 448 (1 if 0); A is converted to e4m3 in the kernel.  K % 16 == 0, no fp32 output, no peer scatter.
  int fp8 = 0;
  const float* w_scale = nullptr;
  const float* a_amax = nullptr;
};
int gemm_tap(const GemmDesc& d, cudaStream_t stream);
// *amax = max |x| over rows x [x1 (cols1 columns, pitch ld1) | x2 (cols2, pitch ld2)]: the FP8 GEMM's per-tensor activation scale
int absmax_f16(const __half* x1, long long rows, int cols1, int ld1, const __half* x2, int cols2, int ld2, float* amax, cudaStream_t stream);

struct AttnDesc {
  // q [B, Nq, heads, 64] (row pitch ldq), k/v [Bk, Nk, heads, 64] (pitch ldk/ldv), out [B, Nq, heads*64] (pitch ldo).
  const __half* q = nullptr; int ldq = 0;
  const __half* k = nullptr; int ldk = 0;
  const __half* v = nullptr; int ldv = 0;
  __half* out = nullptr; int ldo = 0;
  int B = 1, heads = 1, Nq = 0, Nk = 0;
  long long kv_batch_stride = 0;   // elements between K/V batches (0 = shared by all B)
  float scale = 0.125f;
  int accumulate = 0;              // out += result (second softmax branch of the image cross-attention)
};
int flash_attn_d64(const AttnDesc& d, cudaStream_t stream);

// GroupNorm(32) on NHWC fp16; x is the channel concat of (x1: C1 channels) and (x2: C2 channels, may be null).
// Statistics over `rows_per_sample` rows (pixels, or frames*pixels for the 5-D variant) x C/32 channels.
int groupnorm_nhwc(const __half* x1, int C1, const __half* x2, int C2, int samples, long long rows_per_sample,
                   const float* gamma, const float* beta, float eps, int silu, __half* out, float* partial_ws,
                   size_t ws_bytes, cudaStream_t stream);
size_t groupnorm_ws_bytes(int samples);
int groupnorm_stats(const __half* x1, int C1, const __half* x2, int C2, int samples, long long rows_per_sample, float* stats,
                    float* partial_ws, size_t ws_bytes, cudaStream_t stream);
int groupnorm_apply(const __half* x1, int C1, const __half* x2, int C2, int samples, long long rows_per_sample,
                    const float* stats, long long stat_rows, const float* gamma, const float* beta, float eps, int silu, __half* out,
                    cudaStream_t stream, int stat_parts = 1);
// Reproducible mode: leaves[n][32][2] = per-group (sum, sumsq) of the row blocks [n * rows_per_leaf, (n + 1) * rows_per_leaf), and the
// normalise step whose statistics are the sums of leaves_per_sample consecutive leaves per sample, combined in index order.
int groupnorm_leaves(const __half* x1, int C1, const __half* x2, int C2, long long n_leaves, long long rows_per_leaf, float* leaves,
                     cudaStream_t stream);
int groupnorm_apply_leaves(const __half* x1, int C1, const __half* x2, int C2, int samples, long long rows_per_sample, const float* leaves,
                           int leaves_per_sample, long long stat_rows, const float* gamma, const float* beta, float eps, int silu,
                           __half* out, float* ws, size_t ws_bytes, cudaStream_t stream);

// GroupNorm(32) (+SiLU) whose statistics come from the gn_part records of the GEMM(s) that produced x1 (and x2): no statistics pass.
struct GnPartGeom {
  const float* part = nullptr;   // [n_rb][n_chunks][4][2]
  int n_chunks = 0;              // producer N / 32
  int sub = 10;                  // sub-group width the producer cut its chunks at
  long long rb_per_z = 0;        // 32-row blocks per producer slab; sample s starts at block (s / samples_per_z) * rb_per_z + (s % samples_per_z) * rb_per_sample
  int samples_per_z = 1;
  long long rb_per_sample = 0;
};
size_t groupnorm_parts_ws_bytes(int samples);
int groupnorm_parts_to_partials(const GnPartGeom& g1, int C, int samples, float* partial_ws, size_t ws_bytes, int* splits_out,
                                cudaStream_t stream);
int groupnorm_from_parts(const __half* x1, int C1, const GnPartGeom& g1, const __half* x2, int C2, const GnPartGeom& g2, int samples,
                         long long rows_per_sample, const float* gamma, const float* beta, float eps, int silu, __half* out, float* ws,
                         size_t ws_bytes, cudaStream_t stream);

int layernorm_stats(const __half* x, long long rows, int C, float eps, float* stats, cudaStream_t stream);
int layernorm_stats_from_parts(const float* parts, long long rows, int C, float eps, float* stats, cudaStream_t stream);
int layernorm_rows(const __half* x, long long rows, int C, const float* gamma, const float* beta, float eps, __half* out,
                   cudaStream_t stream);

// Temporal self-attention over T<=32 frames per spatial site; qkv rows are [T*sites, ld] with q|k|v at column offsets.
int temporal_attn(const __half* q, const __half* k, const __half* v, int ld, __half* out, int ldo, int T, long long sites,
                  int heads, float scale, cudaStream_t stream);

int upsample2x_nhwc(const __half* x, __half* out, int N, int H, int W, int C, cudaStream_t stream);
int im2col3x3_s2_nhwc(const __half* x, __half* out, int N, int H, int W, int C, int pad_lo, int Ho, int Wo, cudaStream_t stream);
int nchw_to_nhwc_f16(const float* x, __half* out, int B, int C, int T, long long HW, int c_off, int ldo, cudaStream_t stream);
int nhwc_to_ncthw_f32(const float* x, int ldx, float* out, int B, int C, int T, long long HW, cudaStream_t stream);
int nhwc_to_nchw_f32_from_f16(const __half* x, int ldx, float* out, int N, int C, long long HW, cudaStream_t stream);
int cast_f32_to_f16(const float* x, __half* out, long long n, cudaStream_t stream);
int softmax_rows_f32(const float* x, long long rows, long long cols, float scale, __half* out, cudaStream_t stream);
int add_rows_f16(const __half* a, const __half* b, __half* out, long long n, cudaStream_t stream);
int gelu_rows_f16(const __half* x, __half* out, long long n, cudaStream_t stream);

// emb path: out[r, n] = bias[n] + sum_k act(x[r,k]) * W[n,k]   (fp32, tiny M); act: 0 none, 1 SiLU
int small_linear_f32(const float* x, int rows, int K, const float* W, const float* bias, int N, int act_in, float* out,
                     const float* add, cudaStream_t stream);
int timestep_embedding_f32(const long long* t, int n, int dim, float* out, cudaStream_t stream);

struct DdimStepScalars {
  float cfg_scale, guidance_rescale;
  float sqrt_ac_t, sqrt_1mac_t;     // model buffers gathered by timestep t (ddpm3d.py:239-251)
  float a_prev, sigma_t;            // ddim tables gathered by index
  float scale_t, prev_scale_t;      // dynamic rescale
  int use_cfg;
  int reproducible = 0;             // 1: launch grid independent of the SM count
};
// v_uncond_img != nullptr: three-way CFG of ddim_multiplecond.py:227-233 with weight cfg_img on the image-only branch
int ddim_update(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img, const float* noise,
                float* x_prev, float* pred_x0, long long n, const DdimStepScalars& s, double* ws, cudaStream_t stream);

}  // namespace vc

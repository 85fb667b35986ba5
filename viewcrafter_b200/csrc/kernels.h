// Internal C++ launch interface of the sm_90a kernels (the public boundary is include/vc_b200.h, whose descriptor structs the
// launchers take as they are).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/vc_b200.h"

namespace vc {

int gemm_tap(const vc_gemm_desc& d, cudaStream_t stream);
// *amax = max |x| over rows x [x1 (cols1 columns, pitch ld1) | x2 (cols2, pitch ld2)]: the FP8 GEMM's per-tensor activation scale
int absmax_f16(const __half* x1, long long rows, int cols1, int ld1, const __half* x2, int cols2, int ld2, float* amax, cudaStream_t stream);

int flash_attn_d64(const vc_attn_desc& d, cudaStream_t stream);

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
size_t groupnorm_parts_ws_bytes(int samples);
int groupnorm_parts_to_partials(const vc_gn_part_geom& g1, int C, int samples, float* partial_ws, size_t ws_bytes, int* splits_out,
                                cudaStream_t stream);
int groupnorm_from_parts(const __half* x1, int C1, const vc_gn_part_geom& g1, const __half* x2, int C2, const vc_gn_part_geom& g2, int samples,
                         long long rows_per_sample, const float* gamma, const float* beta, float eps, int silu, __half* out, float* ws,
                         size_t ws_bytes, cudaStream_t stream);

int layernorm_stats(const __half* x, long long rows, int C, float eps, float* stats, cudaStream_t stream);
int layernorm_stats_from_parts(const float* parts, long long rows, int C, float eps, float* stats, cudaStream_t stream);
int layernorm_rows(const __half* x, long long rows, int C, const float* gamma, const float* beta, float eps, __half* out,
                   cudaStream_t stream);

// Temporal self-attention over 1 <= T <= 128 frames per spatial site (T <= 32 and 33..128 run different kernels); qkv rows are
// [T*sites, ld] with q|k|v at column offsets.
int temporal_attn(const __half* q, const __half* k, const __half* v, int ld, __half* out, int ldo, int T, long long sites,
                  int heads, float scale, cudaStream_t stream);
// The same attention on overlapping windows of W frames with stride S, blended per frame (vc_temporal_attn_windowed); T <= W
// runs temporal_attn.
int temporal_attn_windowed(const __half* q, const __half* k, const __half* v, int ld, __half* out, int ldo, int T, long long sites,
                           int heads, int W, int S, float scale, cudaStream_t stream);

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

// v_uncond_img != nullptr: three-way CFG of ddim_multiplecond.py:227-233 with weight cfg_img on the image-only branch
int ddim_update(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img, const float* noise,
                float* x_prev, float* pred_x0, long long n, const vc_ddim_scalars& s, double* ws, cudaStream_t stream);
// ddim_update with a step per frame: element i of [B', C, T, HW] takes frames[(i / HW) % T] (host array, T <= VC_DDIM_MAX_FRAMES)
int ddim_update_frames(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img,
                       const float* noise, float* x_prev, float* pred_x0, long long n, int T, long long HW, const vc_ddim_scalars& s,
                       const vc_ddim_frame_scalars* frames, double* ws, cudaStream_t stream);
// ddim_update plus the DPM-Solver++(2M) correction x_prev += c_hist (x0 - x0_hist); x0_hist <- this step's x0 (before the dynamic rescale)
int dpm_update(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img, const float* noise,
               float* x0_hist, float* x_prev, float* pred_x0, long long n, const vc_ddim_scalars& s, float c_hist, double* ws,
               cudaStream_t stream);
// ddim_update plus the DPM-Solver++(3M) SDE correction x_prev += c1 (x0 - x0_hist1) + c2 (x0_hist1 - x0_hist2), x0_hist1 / x0_hist2 the
// previous two steps' x0; x0_hist1 is only read, x0_hist2 <- this step's x0 (before the dynamic rescale).  c2 = 0 is dpm_update bit for bit
int dpm3_update(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img, const float* noise,
                const float* x0_hist1, float* x0_hist2, float* x_prev, float* pred_x0, long long n, const vc_ddim_scalars& s, float c1,
                float c2, double* ws, cudaStream_t stream);

}  // namespace vc

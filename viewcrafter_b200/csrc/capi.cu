// extern "C" boundary of libvc_b200.so (declarations + reference citations: include/vc_b200.h).
#include <atomic>
#include <cstring>

#include "../../include/vc_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace vc {
extern std::atomic<long long> g_launches;
int pick_bn_public(int N, int geglu);
}

using namespace vc;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define H(p) reinterpret_cast<const __half*>(p)
#define HM(p) reinterpret_cast<__half*>(p)
#define COUNT(n) vc::g_launches.fetch_add(n, std::memory_order_relaxed)

extern "C" {

int vc_abi_version(void) { return VC_B200_ABI_VERSION; }
const char* vc_last_error(void) { return vc::last_error(); }
long long vc_launch_count(void) { return vc::g_launches.load(); }
void vc_reset_launch_count(void) { vc::g_launches.store(0); }

int vc_gemm_tap(const vc_gemm_desc* d, void* stream) {
  if (!d) { set_error("vc_gemm_tap: null descriptor"); return VC_ERR_ARG; }
  const int rc = gemm_tap(*d, ST(stream));
  if (rc == VC_OK) COUNT(1);                  // a descriptor refused on the host launches nothing
  return rc;
}
int vc_gemm_tile_n(int32_t N, int32_t geglu) { return vc::pick_bn_public(N, geglu); }
int vc_absmax_f16(const void* x1, int64_t rows, int32_t cols1, int32_t ld1, const void* x2, int32_t cols2, int32_t ld2, float* amax,
                  void* stream) {
  COUNT(1);
  return absmax_f16(H(x1), rows, cols1, ld1, H(x2), cols2, ld2, amax, ST(stream));
}

int vc_flash_attn_d64(const vc_attn_desc* d, void* stream) {
  if (!d) { set_error("vc_flash_attn_d64: null descriptor"); return VC_ERR_ARG; }
  COUNT(1);
  return flash_attn_d64(*d, ST(stream));
}

int vc_temporal_attn(const void* q, const void* k, const void* v, int32_t ld, void* out, int32_t ldo, int32_t T, int64_t sites,
                     int32_t heads, float scale, void* stream) {
  COUNT(1);
  return temporal_attn(H(q), H(k), H(v), ld, HM(out), ldo, T, sites, heads, scale, ST(stream));
}

int vc_temporal_attn_windowed(const void* q, const void* k, const void* v, int32_t ld, void* out, int32_t ldo, int32_t T,
                              int64_t sites, int32_t heads, int32_t W, int32_t S, float scale, void* stream) {
  COUNT(1);
  return temporal_attn_windowed(H(q), H(k), H(v), ld, HM(out), ldo, T, sites, heads, W, S, scale, ST(stream));
}

size_t vc_groupnorm_ws_bytes(int32_t samples) { return groupnorm_ws_bytes(samples); }
int vc_groupnorm_nhwc(const void* x1, int32_t C1, const void* x2, int32_t C2, int32_t samples, int64_t rows_per_sample,
                      const float* gamma, const float* beta, float eps, int32_t silu, void* out, void* ws, size_t ws_bytes,
                      void* stream) {
  COUNT(2);
  return groupnorm_nhwc(H(x1), C1, H(x2), C2, samples, rows_per_sample, gamma, beta, eps, silu, HM(out),
                        reinterpret_cast<float*>(ws), ws_bytes, ST(stream));
}
int vc_groupnorm_stats(const void* x1, int32_t C1, const void* x2, int32_t C2, int32_t samples, int64_t rows_per_sample, float* stats,
                       void* ws, size_t ws_bytes, void* stream) {
  COUNT(2);
  return groupnorm_stats(H(x1), C1, H(x2), C2, samples, rows_per_sample, stats, reinterpret_cast<float*>(ws), ws_bytes, ST(stream));
}
int vc_groupnorm_apply(const void* x1, int32_t C1, const void* x2, int32_t C2, int32_t samples, int64_t rows_per_sample,
                       const float* stats, int64_t stat_rows, const float* gamma, const float* beta, float eps, int32_t silu, void* out,
                       void* stream) {
  COUNT(1);
  return groupnorm_apply(H(x1), C1, H(x2), C2, samples, rows_per_sample, stats, stat_rows, gamma, beta, eps, silu, HM(out), ST(stream));
}
size_t vc_groupnorm_parts_ws_bytes(int32_t samples) { return groupnorm_parts_ws_bytes(samples); }
int vc_groupnorm_from_parts(const void* x1, int32_t C1, const vc_gn_part_geom* g1, const void* x2, int32_t C2, const vc_gn_part_geom* g2,
                            int32_t samples, int64_t rows_per_sample, const float* gamma, const float* beta, float eps, int32_t silu,
                            void* out, void* ws, size_t ws_bytes, void* stream) {
  if (!g1 || (x2 && !g2)) { set_error("vc_groupnorm_from_parts: null geometry"); return VC_ERR_ARG; }
  COUNT(x2 ? 3 : 2);
  return groupnorm_from_parts(H(x1), C1, *g1, H(x2), C2, x2 ? *g2 : *g1 /* not read without x2 */, samples, rows_per_sample, gamma, beta,
                              eps, silu, HM(out), reinterpret_cast<float*>(ws), ws_bytes, ST(stream));
}
int vc_groupnorm_apply_parts(const void* x1, int32_t C1, int32_t samples, int64_t rows_per_sample, const float* parts, int32_t n_parts,
                             int64_t stat_rows, const float* gamma, const float* beta, float eps, int32_t silu, void* out, void* stream) {
  COUNT(1);
  return groupnorm_apply(H(x1), C1, nullptr, 0, samples, rows_per_sample, parts, stat_rows, gamma, beta, eps, silu, HM(out), ST(stream), n_parts);
}
int vc_groupnorm_leaves(const void* x1, int32_t C1, const void* x2, int32_t C2, int64_t n_leaves, int64_t rows_per_leaf, float* leaves,
                        void* stream) {
  COUNT(1);
  return groupnorm_leaves(H(x1), C1, H(x2), C2, n_leaves, rows_per_leaf, leaves, ST(stream));
}
int vc_groupnorm_apply_leaves(const void* x1, int32_t C1, const void* x2, int32_t C2, int32_t samples, int64_t rows_per_sample,
                              const float* leaves, int32_t leaves_per_sample, int64_t stat_rows, const float* gamma, const float* beta,
                              float eps, int32_t silu, void* out, void* ws, size_t ws_bytes, void* stream) {
  COUNT(2);
  return groupnorm_apply_leaves(H(x1), C1, H(x2), C2, samples, rows_per_sample, leaves, leaves_per_sample, stat_rows, gamma, beta, eps, silu,
                                HM(out), reinterpret_cast<float*>(ws), ws_bytes, ST(stream));
}
int vc_layernorm_stats(const void* x, int64_t rows, int32_t C, float eps, float* stats, void* stream) {
  COUNT(1);
  return layernorm_stats(H(x), rows, C, eps, stats, ST(stream));
}
int vc_layernorm_stats_from_parts(const float* parts, int64_t rows, int32_t C, float eps, float* stats, void* stream) {
  COUNT(1);
  return layernorm_stats_from_parts(parts, rows, C, eps, stats, ST(stream));
}
int vc_layernorm(const void* x, int64_t rows, int32_t C, const float* gamma, const float* beta, float eps, void* out, void* stream) {
  COUNT(1);
  return layernorm_rows(H(x), rows, C, gamma, beta, eps, HM(out), ST(stream));
}

int vc_upsample2x_nhwc(const void* x, void* out, int32_t N, int32_t Hh, int32_t W, int32_t C, void* stream) {
  COUNT(1);
  return upsample2x_nhwc(H(x), HM(out), N, Hh, W, C, ST(stream));
}
int vc_im2col3x3_s2(const void* x, void* out, int32_t N, int32_t Hh, int32_t W, int32_t C, int32_t pad_lo, int32_t Ho, int32_t Wo,
                    void* stream) {
  COUNT(1);
  return im2col3x3_s2_nhwc(H(x), HM(out), N, Hh, W, C, pad_lo, Ho, Wo, ST(stream));
}
int vc_ncthw_f32_to_rows_f16(const float* x, void* out, int32_t B, int32_t C, int32_t T, int64_t HW, int32_t c_off, int32_t ldo,
                             void* stream) {
  COUNT(1);
  return nchw_to_nhwc_f16(x, HM(out), B, C, T, HW, c_off, ldo, ST(stream));
}
int vc_rows_f32_to_ncthw(const float* x, int32_t ldx, float* out, int32_t B, int32_t C, int32_t T, int64_t HW, void* stream) {
  COUNT(1);
  return nhwc_to_ncthw_f32(x, ldx, out, B, C, T, HW, ST(stream));
}
int vc_rows_f16_to_nchw_f32(const void* x, int32_t ldx, float* out, int32_t N, int32_t C, int64_t HW, void* stream) {
  COUNT(1);
  return nhwc_to_nchw_f32_from_f16(H(x), ldx, out, N, C, HW, ST(stream));
}
int vc_cast_f32_to_f16(const float* x, void* out, int64_t n, void* stream) {
  COUNT(1);
  return cast_f32_to_f16(x, HM(out), n, ST(stream));
}
int vc_add_f16(const void* a, const void* b, void* out, int64_t n, void* stream) {
  COUNT(1);
  return add_rows_f16(H(a), H(b), HM(out), n, ST(stream));
}

int vc_gelu_f16(const void* x, void* out, int64_t n, void* stream) {
  COUNT(1);
  return gelu_rows_f16(H(x), HM(out), n, ST(stream));
}

int vc_softmax_rows_f32(const float* x, int64_t rows, int64_t cols, float scale, void* out, void* stream) {
  COUNT(1);
  return softmax_rows_f32(x, rows, cols, scale, HM(out), ST(stream));
}

int vc_timestep_embedding(const int64_t* t, int32_t n, int32_t dim, float* out, void* stream) {
  COUNT(1);
  return timestep_embedding_f32(reinterpret_cast<const long long*>(t), n, dim, out, ST(stream));
}
int vc_small_linear_f32(const float* x, int32_t rows, int32_t K, const float* W, const float* bias, int32_t N, int32_t silu_in,
                        float* out, const float* add, void* stream) {
  COUNT(1);
  return small_linear_f32(x, rows, K, W, bias, N, silu_in, out, add, ST(stream));
}

int vc_ddim_update(const float* x, const float* v_cond, const float* v_uncond, const float* noise, float* x_prev, float* pred_x0,
                   int64_t n, const vc_ddim_scalars* s, void* ws, void* stream) {
  if (!s) { set_error("vc_ddim_update: null scalars"); return VC_ERR_ARG; }
  COUNT((s->use_cfg && s->guidance_rescale > 0.f) ? 2 : 1);
  return ddim_update(x, v_cond, v_uncond, nullptr, 0.f, noise, x_prev, pred_x0, n, *s, reinterpret_cast<double*>(ws), ST(stream));
}
int vc_ddim_update3(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img,
                    const float* noise, float* x_prev, float* pred_x0, int64_t n, const vc_ddim_scalars* s, void* ws, void* stream) {
  if (!s) { set_error("vc_ddim_update3: null scalars"); return VC_ERR_ARG; }
  if (!v_uncond_img) { set_error("vc_ddim_update3: null image-only branch"); return VC_ERR_ARG; }
  COUNT((s->use_cfg && s->guidance_rescale > 0.f) ? 2 : 1);
  return ddim_update(x, v_cond, v_uncond, v_uncond_img, cfg_img, noise, x_prev, pred_x0, n, *s, reinterpret_cast<double*>(ws), ST(stream));
}
int vc_ddim_update_frames(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img,
                          const float* noise, float* x_prev, float* pred_x0, int64_t n, int32_t T, int64_t HW, const vc_ddim_scalars* s,
                          const vc_ddim_frame_scalars* frames, void* ws, void* stream) {
  if (!s) { set_error("vc_ddim_update_frames: null scalars"); return VC_ERR_ARG; }
  const int rc = ddim_update_frames(x, v_cond, v_uncond, v_uncond_img, cfg_img, noise, x_prev, pred_x0, n, T, HW, *s, frames,
                                    reinterpret_cast<double*>(ws), ST(stream));
  if (rc == VC_OK) COUNT((s->use_cfg && s->guidance_rescale > 0.f) ? 2 : 1);
  return rc;
}
int vc_dpm_update(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img,
                  const float* noise, float* x0_hist, float* x_prev, float* pred_x0, int64_t n, const vc_ddim_scalars* s, float c_hist,
                  void* ws, void* stream) {
  if (!s) { set_error("vc_dpm_update: null scalars"); return VC_ERR_ARG; }
  COUNT((s->use_cfg && s->guidance_rescale > 0.f) ? 2 : 1);
  return dpm_update(x, v_cond, v_uncond, v_uncond_img, cfg_img, noise, x0_hist, x_prev, pred_x0, n, *s, c_hist,
                    reinterpret_cast<double*>(ws), ST(stream));
}
int vc_dpm3_update(const float* x, const float* v_cond, const float* v_uncond, const float* v_uncond_img, float cfg_img,
                   const float* noise, const float* x0_hist1, float* x0_hist2, float* x_prev, float* pred_x0, int64_t n,
                   const vc_ddim_scalars* s, float c1, float c2, void* ws, void* stream) {
  if (!s) { set_error("vc_dpm3_update: null scalars"); return VC_ERR_ARG; }
  COUNT((s->use_cfg && s->guidance_rescale > 0.f) ? 2 : 1);
  return dpm3_update(x, v_cond, v_uncond, v_uncond_img, cfg_img, noise, x0_hist1, x0_hist2, x_prev, pred_x0, n, *s, c1, c2,
                     reinterpret_cast<double*>(ws), ST(stream));
}

/* vc_enable_peer_access / vc_peer_exchange / vc_peer_groupnorm_stats: peer.cu */

}  // extern "C"

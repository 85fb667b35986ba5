// Tap-GEMM on wgmma: D[M,N] = sum_taps A_tap[M,K] * W_tap[N,K]^T  (fp16 in, fp32 accumulate in registers).
//
// One kernel family covers every tensor-core op on the U-Net / VAE path:
//   * nn.Linear / 1x1 conv            : 1 tap, A = [M,K] row-major
//   * 3x3 conv, stride 1, pad 1 (NHWC): 9 taps, A tile = TMA box (64ch, bw, bh, 1 frame) shifted by (dx-1, dy-1);
//                                       the zero padding is TMA out-of-bounds fill
//   * Conv3d (3,1,1), pad (1,0,0)     : 3 taps, A rows shifted by +-H*W rows of the [T*H*W, C] matrix (OOB rows = 0)
// A may come from two tensors split along K (channel concat of skip connections without materialising it).
// Epilogue (epi_tile_run): + bias[z/bias_z_div][n], GEGLU (value*gelu(gate)), + residual, fp16 / fp32 store, on the accumulator
// fragments; fp16 results go through a shared-memory output tile that the TMA stores (and the statistics) read.
//
// Persistent kernel, one CTA per SM, 128 x BN tiles, 384 threads, ping-pong schedule:
//   warpgroup 0  warp 0 is the TMA producer: it walks this CTA's tiles and their (tap, k-block) iterations through a smem
//                ring in one in-order sequence, without draining between tiles.  The warpgroup gives up registers
//                (setmaxnreg) to the two MMA warpgroups.
//   warpgroups 1, 2  own alternate tiles of the CTA's sequence (tiles 0, 2, 4, ... / 1, 3, 5, ...).  A warpgroup computes its
//                whole 128 x BN tile as two wgmma m64nBNk16 row halves (both operands from the 128B-swizzled ring, one k-block
//                in flight behind the one being issued), consumes only its own tiles' ring stages, and steps its ring
//                position past the other warpgroup's.  Then it runs the epilogue of its tile while the other warpgroup's
//                MMAs keep the tensor cores busy.  A tile's residual is TMA-loaded into the warpgroup's output tile when
//                its mainloop starts, so the epilogue finds it in shared memory.
//   The mainloops alternate strictly (an ordering barrier between the two MMA warpgroups): a warpgroup starts waiting on its
//   next tile's stages only once the other one has seen all of its own.  Besides keeping the two mainloops from sharing the
//   tensor cores, this keeps every full-barrier wait within one phase of the barrier, which the parity waits require.
// Tiles are ordered n-fastest so CTAs that run concurrently share A tiles in L2.
//
// FP8 variant (FP8 = true, vc_gemm_desc::fp8): the weights are e4m3 (per-output-channel scales w_scale), a ring stage holds
// the fp16 A tile as before and the weight tile as 64-byte rows (64B swizzle).  The MMA warpgroup reads its A fragments from
// the fp16 stage, scales them by 1 / s_a (s_a = a_amax / 448, one scale per GEMM call) and converts them to e4m3 in
// registers (round to nearest, saturating), then issues wgmma m64nBNk32 e4m3 x e4m3 with A from registers.  A stays fp16 in
// HBM: no conversion pass.  The epilogue starts from acc * (s_a * w_scale[n]) and is otherwise the fp16 one.
#include <cuda_fp8.h>

#include <type_traits>

#include "gemm_common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace vc {

template <int BN, bool FP8 = false>
struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * (FP8 ? 1 : 2);
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int OUT_BYTES = BM * BN * 2;        // one MMA warpgroup's fp16 output tile (gemm_common.cuh: epi_offset)
  static constexpr int EPI_BYTES = MMA_WGS * OUT_BYTES;
  static constexpr int BUDGET = 227 * 1024 - 1024 /*align slack*/ - 256 /*barriers*/ - EPI_BYTES;
  static constexpr int STAGES = BUDGET / STAGE_BYTES > 8 ? 8 : BUDGET / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 1024 + 256;
  static_assert(STAGES >= 4, "pipeline too shallow");
  static_assert(B_BYTES % 1024 == 0, "stages must stay 1024-byte aligned (128B swizzle atoms)");
  static_assert(BN % 32 == 0, "the output tile is made of 32-column chunks");
};

// bias / LayerNorm column sums / weight scales of columns n and n + 1 (n even, the vectors 8-byte aligned); 0 past N
__device__ __forceinline__ float2 col_pair(const float* v, int n, int N) {
  if (n + 1 < N) return __ldg(reinterpret_cast<const float2*>(v + n));
  return make_float2(n < N ? __ldg(v + n) : 0.f, 0.f);
}

// Epilogue of one 128 x BN tile, run by the MMA warpgroup that computed it, on its accumulator fragments.  Thread (warp wl,
// lane) holds rows R = 64 h + 16 wl + lane / 4 + 8 r and columns c = 8 j + 2 (lane % 4) + {0, 1} of the tile in
// acc[h][4 j + 2 r + {0, 1}].  Per element, in this order: FP8 dequantisation, folded LayerNorm, bias, residual, one rounding
// to fp16 -- or, for GEGLU, value * gelu(gate) of the column pair (c, c + BN / 2).  The residual comes from the output tile,
// where the TMA load issued at the start of the tile's mainloop left it, at the element's own position, and the fp16 result
// goes back to the same position (one owner per element: no barrier).  fp32 outputs are stored straight from the fragments.
// After one warpgroup barrier, warp wl takes rows 32 wl .. 32 wl + 31 of the tile: the statistics and the non-TMA stores read
// them one row per thread, and lane 0 issues the TMA stores of the warp's 32 x 32 boxes.
template <int BN, bool FP8>
__device__ __forceinline__ void epi_tile_run(const GemmParams& p, int tile, float (&acc)[2][BN / 2], uint8_t* otile,
                                             uint64_t* res_bar, int cw, int wl, int lane, float sa) {
  const int m_tile = fast_div(p.div_n_tiles, tile);
  const int n_tile = tile - m_tile * p.n_tiles;
  const TileCoord tc = tile_coord_m(p, m_tile);
  const int n0 = n_tile * BN;
  const bool geglu = BN == 128 && p.geglu;         // GEGLU always runs at BN = 128 (pick_bn)
  const int n_out = geglu ? p.N / 2 : p.N;
  const int col_base = geglu ? n_tile * (BN / 2) : n0;
  const float* bias = p.bias ? p.bias + (long long)(p.bias_z_div > 0 ? min(tc.z, p.Z - 1) / p.bias_z_div : 0) * p.N : nullptr;
  const uint32_t obase = smem_u32(otile);
  const int q = lane & 3;
  bool row_ok[2][2];
  long long orow[2][2];
  float2 ln[2][2];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int R = 64 * h + 16 * wl + (lane >> 2) + 8 * r;
      const int x = tc.x0 + (R & (p.bx - 1)), y = tc.y0 + (R >> p.bx_shift);
      row_ok[h][r] = x < p.X && y < p.Y && tc.z < p.Z;
      orow[h][r] = ((long long)tc.z * p.Y + y) * p.X + x;
      ln[h][r] = make_float2(0.f, 1.f);
      if (p.ln_stats && row_ok[h][r]) ln[h][r] = __ldg(reinterpret_cast<const float2*>(p.ln_stats) + orow[h][r]);
    }
  const bool res_smem = p.res && p.res_tma;
  // tile = blockIdx.x + cw * gridDim.x + 2 * gridDim.x * k: the k-th residual load of this warpgroup completes phase k & 1
  if (res_smem) mbar_wait(res_bar, ((tile - (int)blockIdx.x) / (2 * (int)gridDim.x)) & 1);
  // The common case (fp16 output, residual from the tile or none) runs a loop without per-element branches on the store path:
  // those branches cost the loop its scheduling and made it several times slower.  fp32 outputs and residuals TMA cannot load
  // take the general loop.
  auto frag_loop = [&](auto general_tag) {
    constexpr bool GENERAL = decltype(general_tag)::value;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = 8 * j + 2 * q;
      const int n = n0 + c;
      float2 ws = make_float2(1.f, 1.f), cs = make_float2(0.f, 0.f), b = make_float2(0.f, 0.f);
      if constexpr (FP8) ws = col_pair(p.w_scale, n, p.N);
      if (p.ln_stats) cs = col_pair(p.ln_colsum, n, p.N);
      if (bias) b = col_pair(bias, n, p.N);
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int R = 64 * h + 16 * wl + (lane >> 2) + 8 * r;
          const uint32_t addr = obase + epi_offset(R, c);
          float v0 = acc[h][4 * j + 2 * r], v1 = acc[h][4 * j + 2 * r + 1];
          if constexpr (FP8) { v0 *= sa * ws.x; v1 *= sa * ws.y; }
          if (p.ln_stats) {
            const float2 l = ln[h][r];
            v0 = (v0 - l.x * cs.x) * l.y;
            v1 = (v1 - l.x * cs.y) * l.y;
          }
          if (bias) { v0 += b.x; v1 += b.y; }
          if (res_smem) {
            uint32_t u;
            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(u) : "r"(addr));
            const float2 rv = __half22float2(*reinterpret_cast<const __half2*>(&u));
            v0 += rv.x; v1 += rv.y;
          } else if (GENERAL && p.res && row_ok[h][r]) {
            // residual TMA cannot address (unaligned pointer or pitch): plain loads, not __ldg -- res may alias out
            const __half* rp = p.res + orow[h][r] * p.ldr + n;
            if (n < p.N) v0 += __half2float(rp[0]);
            if (n + 1 < p.N) v1 += __half2float(rp[1]);
          }
          if (GENERAL && p.out_f32) {
            if (row_ok[h][r] && n < n_out) {
              float* op = p.out_f32 + orow[h][r] * p.ldo + n;
              if (n + 1 < n_out && p.vec_ok) {
                *reinterpret_cast<float2*>(op) = make_float2(v0, v1);
              } else {
                op[0] = v0;
                if (n + 1 < n_out) op[1] = v1;
              }
            }
          } else {
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pack_half2(v0, v1)) : "memory");
          }
        }
    }
  };
  if (!geglu) {
    if (p.out_f32 || (p.res && !p.res_tma)) frag_loop(std::true_type{});
    else frag_loop(std::false_type{});
  } else {
    // GEGLU: tile columns [0, BN/2) are values, [BN/2, BN) the matching gates (weights were interleaved per tile);
    // out[:, n_tile*BN/2 + c] = (value + bias_v) * gelu(gate + bias_g).  No residual (checked on the host).
    constexpr int HALF = BN / 2;
#pragma unroll
    for (int j = 0; j < HALF / 8; ++j) {
      const int c = 8 * j + 2 * q;
      const int n = n0 + c;
      float2 wv = make_float2(1.f, 1.f), wg = wv, cv = make_float2(0.f, 0.f), cg = cv, bv = cv, bg = cv;
      if constexpr (FP8) { wv = col_pair(p.w_scale, n, p.N); wg = col_pair(p.w_scale, n + HALF, p.N); }
      if (p.ln_stats) { cv = col_pair(p.ln_colsum, n, p.N); cg = col_pair(p.ln_colsum, n + HALF, p.N); }
      if (bias) { bv = col_pair(bias, n, p.N); bg = col_pair(bias, n + HALF, p.N); }
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int R = 64 * h + 16 * wl + (lane >> 2) + 8 * r;
          float o[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float a = acc[h][4 * j + 2 * r + e], g = acc[h][4 * (j + HALF / 8) + 2 * r + e];
            if constexpr (FP8) {
              a *= sa * (e ? wv.y : wv.x);
              g *= sa * (e ? wg.y : wg.x);
            }
            if (p.ln_stats) {
              const float2 l = ln[h][r];
              a = (a - l.x * (e ? cv.y : cv.x)) * l.y;
              g = (g - l.x * (e ? cg.y : cg.x)) * l.y;
            }
            if (bias) { a += e ? bv.y : bv.x; g += e ? bg.y : bg.x; }
            o[e] = a * gelu_epilogue(g);
          }
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(obase + epi_offset(R, c)), "r"(pack_half2(o[0], o[1])) : "memory");
        }
    }
  }
  if (p.out_f32) return;                           // no statistics on fp32 outputs (host check)
  if (p.out_tma) fence_proxy_async_smem();         // the fp16 tile is visible to the TMA stores
  named_bar_sync(1 + cw, 128);
  constexpr int CHUNKS = BN / 32;
  const int nchunks = geglu ? CHUNKS / 2 : CHUNKS;
  const EpiTile t = epi_tile(p, tile, wl, lane);
  if (p.ln_part || p.gn_part || !p.out_tma) {
    const int R = 32 * wl + lane;
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
      if (c < nchunks && col_base + 32 * c < n_out) {   // warp-uniform
        uint4 u[4];
        epi_row_load(obase + c * EPI_CHUNK_BYTES + R * 64, R, u);
        if (p.ln_part || p.gn_part) epi_stats_row32(p, t, n0 + 32 * c, u, lane);
        if (!p.out_tma) epi_store_row32(p, t, col_base + 32 * c, n_out, u);
      }
    }
  }
  if (p.out_tma && lane == 0) {
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
      if (c < nchunks && col_base + 32 * c < n_out) {
        const uint8_t* box = otile + c * EPI_CHUNK_BYTES + wl * EPI_SUB_BYTES;
        if (p.peer.mode) peer_scatter32(p, t, col_base + 32 * c, box);
        else tma_store_4d(&p.tmap_out, box, col_base + 32 * c, t.wx, t.wy, t.wz);
      }
    }
    tma_store_commit();
  }
}

// e4m3 A fragment register of wgmma k32: 4 consecutive fp16 of one row (8 bytes of the 128B-swizzled stage), each scaled by
// inv_sa in fp32 and rounded once to e4m3 (satfinite); element k in byte k
__device__ __forceinline__ uint32_t a_frag_e4m3(uint32_t addr, float inv_sa) {
  uint32_t u0, u1;
  asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(u0), "=r"(u1) : "r"(addr));
  const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&u0));
  const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&u1));
  const uint32_t q0 = __nv_cvt_float2_to_fp8x2(make_float2(lo.x * inv_sa, lo.y * inv_sa), __NV_SATFINITE, __NV_E4M3);
  const uint32_t q1 = __nv_cvt_float2_to_fp8x2(make_float2(hi.x * inv_sa, hi.y * inv_sa), __NV_SATFINITE, __NV_E4M3);
  return q0 | (q1 << 16);
}

template <int BN, bool FP8>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tap_kernel(const __grid_constant__ GemmParams p) {
  using Cfg = GemmCfg<BN, FP8>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* epi_smem = smem + STAGES * Cfg::STAGE_BYTES;          // [MMA_WGS] output tiles
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(epi_smem + Cfg::EPI_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* res_bar = empty_bar + STAGES;                         // [MMA_WGS] residual loaded into the output tile

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int kblocks = (p.K + BK - 1) / BK;
  const int iters = p.num_taps * kblocks;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmap_a);
    tma_prefetch_desc(&p.tmap_b);
    if (p.out_tma) tma_prefetch_desc(&p.tmap_out);
    if (p.res_tma) tma_prefetch_desc(&p.tmap_res);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);                  // one arrival per warp of the MMA warpgroup that owns the stage's tile
    }
    for (int w = 0; w < MMA_WGS; ++w) mbar_init(&res_bar[w], 1);
    fence_barrier_init();
  }
  __syncthreads();

  // ring positions are carried as (index, phase bit) pairs and tile coordinates come from multiply-high divisions
  if (warp < 4) {
    setmaxnreg_dec<GEMM_PRODUCER_REGS>();
    if (warp != 0) return;
    // ------------------------------ TMA producer ------------------------------
    // warp-uniform loop, ONE elected lane issues (keeps barrier / descriptor operands in uniform registers)
    int s = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const int m_tile = fast_div(p.div_n_tiles, tile);
      const TileCoord tc = tile_coord_m(p, m_tile);
      const int n0 = (tile - m_tile * p.n_tiles) * BN;
      for (int tap = 0; tap < p.num_taps; ++tap) {
        const int cx = tc.x0 + p.tap_dx[tap], cy = tc.y0 + p.tap_dy[tap];
        const int brow = tap * p.N + n0;
        for (int kb = 0; kb < kblocks; ++kb) {
          mbar_wait(&empty_bar[s], ph ^ 1);        // a fresh barrier passes the wait on the "previous" phase
          if (elect_one()) {
            uint8_t* sa = smem + s * Cfg::STAGE_BYTES;
            uint8_t* sb = sa + Cfg::A_BYTES;
            mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
            const int k = kb * BK;
            if (k < p.K1)
              tma_load_4d(sa, &p.tmap_a, &full_bar[s], k, cx, cy, tc.z);
            else
              tma_load_4d(sa, &p.tmap_a2, &full_bar[s], k - p.K1, cx, cy, tc.z);
            tma_load_2d(sb, &p.tmap_b, &full_bar[s], k, brow);
          }
          __syncwarp();
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------ MMA warpgroups + epilogue ------------------------------
    setmaxnreg_inc<GEMM_MMA_REGS>();
    const int cw = (warp >> 2) - 1;                 // tiles cw, cw + 2, cw + 4, ... of this CTA's sequence
    const int wl = warp & 3;
    uint8_t* otile = epi_smem + cw * Cfg::OUT_BYTES;
    const uint32_t ring = smem_u32(smem);
    float sa = 1.f, inv_sa = 1.f;                   // FP8: per-tensor activation scale s_a = amax / 448 (1 for an all-zero A)
    if constexpr (FP8) {
      const float amax = *p.a_amax;
      sa = amax > 0.f ? __fdiv_rn(amax, 448.f) : 1.f;
      inv_sa = __fdiv_rn(1.f, sa);
    }
    float acc[2][BN / 2];                           // rows [0, 64) and [64, 128) of the tile
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.f;
    int s = 0;
    uint32_t ph = 0;
    // step the ring position past the `iters` stages of a tile the other warpgroup consumes
    auto skip_tile = [&]() {
      s += iters;
      ph ^= (uint32_t)(s / STAGES) & 1u;
      s %= STAGES;
    };
    if (cw == 1) skip_tile();
    for (int tile = blockIdx.x + cw * gridDim.x; tile < p.total_tiles; tile += 2 * gridDim.x) {
      // this warpgroup's previous tile: its TMA stores have finished reading the output tile (each warp's lane 0 issued its own)
      if (p.out_tma && lane == 0) tma_store_wait_read();
      __syncwarp();
      // ordering barrier: the other warpgroup has waited on every stage of the tile before this one (ids 3 / 4: "cw may start").
      // It also waits for all of this warpgroup's threads, so the previous tile's epilogue is done with the output tile.
      if (tile >= (int)gridDim.x) named_bar_sync(3 + cw, 256);
      if (p.res_tma && wl == 0 && lane == 0) {
        // residual of this tile into the output tile: it lands while the mainloop runs (rows / columns outside the tensor read as 0)
        const int m_tile = fast_div(p.div_n_tiles, tile);
        const TileCoord tc = tile_coord_m(p, m_tile);
        const int n0 = (tile - m_tile * p.n_tiles) * BN;
        const int nch = min(BN, p.N - n0 + 31) / 32;
        mbar_expect_tx(&res_bar[cw], nch * EPI_CHUNK_BYTES);
        for (int c = 0; c < nch; ++c) tma_load_4d(otile + c * EPI_CHUNK_BYTES, &p.tmap_res, &res_bar[cw], n0 + 32 * c, tc.x0, tc.y0, tc.z);
      }
      __syncwarp();
      int prev = -1;
      for (int i = 0; i < iters; ++i) {
        mbar_wait(&full_bar[s], ph);
        const uint32_t a_addr = ring + s * Cfg::STAGE_BYTES;
        const uint32_t b_addr = ring + s * Cfg::STAGE_BYTES + Cfg::A_BYTES;
        if constexpr (!FP8) {
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) {
            const uint64_t db = wgmma_desc_sw128(b_addr + 32 * k);
            Wgmma<BN>::ss(acc[0], wgmma_desc_sw128(a_addr + 32 * k), db, (i > 0 || k > 0) ? 1 : 0);
            Wgmma<BN>::ss(acc[1], wgmma_desc_sw128(a_addr + 64 * BK * 2 + 32 * k), db, (i > 0 || k > 0) ? 1 : 0);
          }
          wgmma_commit();
          wgmma_wait<1>();                            // the previous k-block's MMAs have retired: its stage may be refilled
          if (prev >= 0) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
          }
        } else {
          // A fragment of wgmma k32 (8-bit): register j of thread (g = lane / 4, q = lane % 4) holds row g + 8 (j & 1) of the
          // warp's 16 rows, k = 16 (j >> 1) + 4 q .. + 3.  In the 128B-swizzled fp16 stage that is 16-byte chunk
          // c = 4 ks + 2 (j >> 1) + q / 2 of the row, stored at chunk c ^ (row & 7) = c ^ g, byte 8 (q & 1) inside it.
          // One commit group per k32 step: the conversion of the next step overlaps the MMAs of this one, and only two steps'
          // fragments (16 registers) are live at a time.
          const int g = lane >> 2, q = lane & 3;
          const uint32_t a_row = a_addr + (16 * wl + g) * (BK * 2) + (q & 1) * 8;
#pragma unroll
          for (int ks = 0; ks < BK / 32; ++ks) {
            const uint64_t db = wgmma_desc_sw64(b_addr + 32 * ks);
            uint32_t fa[2][4];
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const int c = 4 * ks + 2 * (j >> 1) + (q >> 1);
                fa[h][j] = a_frag_e4m3(a_row + (h * 64 + 8 * (j & 1)) * (BK * 2) + ((c ^ g) << 4), inv_sa);
              }
            wgmma_fence();
            WgmmaF8<BN>::rs(acc[0], fa[0], db, (i > 0 || ks > 0) ? 1 : 0);
            WgmmaF8<BN>::rs(acc[1], fa[1], db, (i > 0 || ks > 0) ? 1 : 0);
            wgmma_commit();
            wgmma_wait<1>();                          // ks = 0: the previous k-block's last step has retired
            if (ks == 0 && prev >= 0) {
              __syncwarp();
              if (lane == 0) mbar_arrive(&empty_bar[prev]);
            }
          }
        }
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      if (tile + (int)gridDim.x < p.total_tiles) named_bar_arrive(4 - cw, 256);   // the other warpgroup's next tile may start
      skip_tile();
      wgmma_wait<0>();
      wgmma_fence_regs(acc[0]);
      wgmma_fence_regs(acc[1]);
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      epi_tile_run<BN, FP8>(p, tile, acc, otile, &res_bar[cw], cw, wl, lane, sa);
    }
    if (p.out_tma && lane == 0) tma_store_wait_all();   // bulk stores must be complete before the CTA exits
  }
}

template <int BN, bool FP8 = false>
static int launch_gemm(const GemmParams& p, cudaStream_t stream) {
  using Cfg = GemmCfg<BN, FP8>;
  static DeviceOnce configured;
  if (device_once_needed(configured)) {
    VC_CHECK_CUDA(cudaFuncSetAttribute(gemm_tap_kernel<BN, FP8>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    device_once_mark(configured);
  }
  const int grid = p.total_tiles < sm_count() ? p.total_tiles : sm_count();
  gemm_tap_kernel<BN, FP8><<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(p);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

// Widest tile that divides N: the accumulator lives in registers (BN / 2 per MMA thread), so tiles stop at 160 columns.
// FP8 stops at 128: its A fragments take the registers that 160 columns would need (ptxas spills), so N = 320 runs at 64.
static int pick_bn(int N, int geglu, int fp8 = 0) {
  if (geglu) return 128;
  if (N <= 32) return 32;
  if (N <= 64) return 64;
  if (fp8 && N % 160 == 0) return N % 128 == 0 ? 128 : 64;
  if (N % 160 == 0) return 160;
  if (N % 128 == 0) return 128;
  if (N % 96 == 0 && N <= 192) return 96;
  if (N % 64 == 0 && N < 256) return 64;
  return 128;
}

int pick_bn_public(int N, int geglu) { return pick_bn(N, geglu); }

int gemm_tap(const vc_gemm_desc& d, cudaStream_t stream) {
  VC_REQUIRE(d.a && d.w && (d.out || d.out_f32), "gemm_tap: null pointer");
  VC_REQUIRE(d.num_taps >= 1 && d.num_taps <= MAX_TAPS, "gemm_tap: num_taps=%d out of range", d.num_taps);
  VC_REQUIRE(d.bx * d.by == BM && d.bx >= 1, "gemm_tap: box %dx%d must cover 128 rows", d.bx, d.by);
  VC_REQUIRE(d.by == 1 || d.bx == d.X, "gemm_tap: multi-row boxes need bx == X (X=%d bx=%d)", d.X, d.bx);
  VC_REQUIRE(d.K % 8 == 0 && d.lda % 8 == 0, "gemm_tap: K and lda must be multiples of 8 (TMA 16-byte strides)");
  VC_REQUIRE(d.K1 == d.K || (d.a2 && d.K1 % BK == 0 && d.K1 < d.K), "gemm_tap: bad K split K1=%d K=%d", d.K1, d.K);
  VC_REQUIRE(!d.geglu || (d.N % 128 == 0 && !d.res && !d.out_f32), "gemm_tap: GEGLU needs N %% 128 == 0");
  if ((reinterpret_cast<uintptr_t>(d.a) & 15) || (reinterpret_cast<uintptr_t>(d.w) & 15)) {
    set_error("gemm_tap: operands must be 16-byte aligned");
    return VC_ERR_ARG;
  }
  // the epilogue reads the bias as float4: every bias row (row z / bias_z_div starts at bias + that * N) must be 16-byte aligned
  VC_REQUIRE(!d.bias || (reinterpret_cast<uintptr_t>(d.bias) & 15) == 0, "gemm_tap: bias must be 16-byte aligned");
  VC_REQUIRE(!d.bias || d.bias_z_div <= 0 || d.N % 4 == 0, "gemm_tap: per-z bias rows (bias_z_div=%d) need N %% 4 == 0 (N=%d)",
             d.bias_z_div, d.N);
  if (d.fp8) {
    VC_REQUIRE(d.K % 16 == 0, "gemm_tap: fp8 needs K %% 16 == 0 (K=%d)", d.K);
    VC_REQUIRE(d.w_scale && d.a_amax, "gemm_tap: fp8 needs w_scale and a_amax");
    VC_REQUIRE((reinterpret_cast<uintptr_t>(d.w_scale) & 15) == 0, "gemm_tap: fp8 w_scale must be 16-byte aligned");
    VC_REQUIRE(!d.out_f32, "gemm_tap: fp8 does not support an fp32 output");
    VC_REQUIRE(!(d.peer && d.peer->mode), "gemm_tap: fp8 does not support the peer-scatter epilogue");
  }
  const void* optr = d.out_f32 ? (const void*)d.out_f32 : (const void*)d.out;
  const int esz = d.out_f32 ? 4 : 2;

  GemmParams p;
  memset(&p, 0, sizeof(p));
  const int BN = pick_bn(d.N, d.geglu, d.fp8);
  p.bx = d.bx; p.by = d.by; p.X = d.X; p.Y = d.Y; p.Z = d.Z;
  p.tiles_x = (d.X + d.bx - 1) / d.bx;
  p.tiles_y = (d.Y + d.by - 1) / d.by;
  p.n_tiles = (d.N + BN - 1) / BN;
  p.div_tiles_x = make_fastdiv(p.tiles_x);
  p.div_tiles_y = make_fastdiv(p.tiles_y);
  p.div_n_tiles = make_fastdiv(p.n_tiles);
  p.bx_shift = 0;
  while ((1 << p.bx_shift) < d.bx) ++p.bx_shift;
  VC_REQUIRE((1 << p.bx_shift) == d.bx, "gemm_tap: bx=%d must be a power of two", d.bx);
  const long long m_tiles = (long long)p.tiles_x * p.tiles_y * p.Z;

  // A: (K, X, Y, Z) with row pitch lda
  {
    uint64_t dims[4] = {(uint64_t)d.K1, (uint64_t)d.X, (uint64_t)d.Y, (uint64_t)d.Z};
    uint64_t str[3] = {(uint64_t)d.lda * 2, (uint64_t)d.lda * 2 * d.X, (uint64_t)d.lda * 2 * d.X * d.Y};
    uint32_t box[4] = {(uint32_t)BK, (uint32_t)d.bx, (uint32_t)d.by, 1};
    int rc = encode_tmap_f16(&p.tmap_a, d.a, 4, dims, str, box);
    if (rc) return rc;
    if (d.K1 != d.K) {
      uint64_t dims2[4] = {(uint64_t)(d.K - d.K1), (uint64_t)d.X, (uint64_t)d.Y, (uint64_t)d.Z};
      uint64_t str2[3] = {(uint64_t)d.lda2 * 2, (uint64_t)d.lda2 * 2 * d.X, (uint64_t)d.lda2 * 2 * d.X * d.Y};
      rc = encode_tmap_f16(&p.tmap_a2, d.a2, 4, dims2, str2, box);
      if (rc) return rc;
    } else {
      p.tmap_a2 = p.tmap_a;
    }
  }
  {
    uint64_t dims[2] = {(uint64_t)d.K, (uint64_t)d.num_taps * d.N};
    const int wbytes = d.fp8 ? 1 : 2;
    uint64_t str[1] = {(uint64_t)(d.ldw > 0 ? d.ldw : d.K) * wbytes};
    uint32_t box[2] = {(uint32_t)BK, (uint32_t)BN};
    int rc = d.fp8 ? encode_tmap_f16(&p.tmap_b, d.w, 2, dims, str, box, 64, CU_TENSOR_MAP_DATA_TYPE_UINT8)
                   : encode_tmap_f16(&p.tmap_b, d.w, 2, dims, str, box);
    if (rc) return rc;
  }
  p.N = d.N; p.K = d.K; p.K1 = d.K1;
  p.num_taps = d.num_taps;
  for (int t = 0; t < d.num_taps; ++t) { p.tap_dx[t] = d.tap_dx[t]; p.tap_dy[t] = d.tap_dy[t]; }
  p.out = static_cast<__half*>(d.out); p.out_f32 = static_cast<float*>(d.out_f32); p.ldo = d.ldo;
  p.bias = d.bias; p.bias_z_div = d.bias_z_div;
  p.res = static_cast<const __half*>(d.res); p.ldr = d.ldr;
  p.geglu = d.geglu;
  p.w_scale = d.w_scale; p.a_amax = d.a_amax;
  VC_REQUIRE((d.ln_stats == nullptr) == (d.ln_colsum == nullptr), "gemm_tap: ln_stats and ln_colsum go together");
  VC_REQUIRE(!d.ln_stats || (d.num_taps == 1 && d.N % 32 == 0 && d.Y == 1 && d.Z == 1 && !d.a2),
             "gemm_tap: folded LayerNorm needs a plain [M,K] x [N,K] GEMM with N %% 32 == 0");
  VC_REQUIRE(!d.ln_stats || ((reinterpret_cast<uintptr_t>(d.ln_stats) & 7) == 0 && (reinterpret_cast<uintptr_t>(d.ln_colsum) & 15) == 0),
             "gemm_tap: ln_stats / ln_colsum misaligned");
  p.ln_stats = d.ln_stats; p.ln_colsum = d.ln_colsum;
  VC_REQUIRE(!d.ln_part || (d.num_taps == 1 && d.N % 32 == 0 && d.Y == 1 && d.Z == 1 && !d.geglu && d.out && !d.out_f32 &&
                            (reinterpret_cast<uintptr_t>(d.ln_part) & 7) == 0),
             "gemm_tap: LayerNorm partial sums need a plain fp16 [M,N] output with N %% 32 == 0");
  p.ln_part = reinterpret_cast<float2*>(d.ln_part); p.ln_rows = d.X;
  VC_REQUIRE(!d.gn_part || ((d.gn_sub == 10 || d.gn_sub == 8) && d.N % 32 == 0 && d.N % d.gn_sub == 0 && !d.geglu && d.out && !d.out_f32 &&
                            (reinterpret_cast<uintptr_t>(d.gn_part) & 7) == 0),
             "gemm_tap: GroupNorm partial sums need an fp16 output with N %% 32 == 0 and N %% gn_sub == 0 (gn_sub 10 or 8)");
  p.gn_part = reinterpret_cast<float2*>(d.gn_part); p.gn_hp = d.gn_sub / 2; p.gn_nchunks = d.N / 32;
  // vector epilogue stores need 32-byte aligned rows (true for every activation on the U-Net / VAE path); anything
  // else (odd pitches, the 4- and 3-channel output convs) takes the predicated scalar path inside the kernel.  The output
  // and the residual are judged separately: the residual is added in registers before any store path runs.
  p.vec_ok = ((reinterpret_cast<uintptr_t>(optr) & 31) == 0) && ((long long)d.ldo * esz) % 32 == 0 ? 1 : 0;
  p.res_tma = d.res && (reinterpret_cast<uintptr_t>(d.res) & 15) == 0 && d.ldr % 8 == 0 ? 1 : 0;
  if (p.res_tma) {
    // the residual tile of 128 rows x 32 columns per box, in the output tile's layout (gemm_common.cuh: epi_offset)
    uint64_t dims[4] = {(uint64_t)d.N, (uint64_t)d.X, (uint64_t)d.Y, (uint64_t)d.Z};
    uint64_t str[3] = {(uint64_t)d.ldr * 2, (uint64_t)d.ldr * 2 * d.X, (uint64_t)d.ldr * 2 * d.X * d.Y};
    uint32_t box[4] = {32, (uint32_t)d.bx, (uint32_t)d.by, 1};
    int rc = encode_tmap_f16(&p.tmap_res, d.res, 4, dims, str, box, 64);
    if (rc) return rc;
  }
  {
    // TMA-store epilogue: fp16 output whose width is whole 32-column chunks and whose rows are 16-byte aligned
    const int n_out = d.geglu ? d.N / 2 : d.N;
    p.out_tma = (d.out && !d.out_f32 && n_out % 32 == 0 && (reinterpret_cast<uintptr_t>(d.out) & 15) == 0 && d.ldo % 8 == 0) ? 1 : 0;
    if (p.out_tma) {
      const uint32_t bw = d.bx < 32 ? d.bx : 32;
      uint64_t dims[4] = {(uint64_t)n_out, (uint64_t)d.X, (uint64_t)d.Y, (uint64_t)d.Z};
      const long long py = d.ldo_y > 0 ? d.ldo_y : (long long)d.ldo * d.X;
      const long long pz = d.ldo_z > 0 ? d.ldo_z : py * d.Y;
      uint64_t str[3] = {(uint64_t)d.ldo * 2, (uint64_t)py * 2, (uint64_t)pz * 2};
      uint32_t box[4] = {32, bw, 32 / bw, 1};
      int rc = encode_tmap_f16(&p.tmap_out, d.out, 4, dims, str, box, 64);
      if (rc) return rc;
    }
    VC_REQUIRE((d.ldo_y == 0 && d.ldo_z == 0) || (p.out_tma && !d.res && !d.ln_part),
               "gemm_tap: strided (ldo_y / ldo_z) outputs need the TMA-store epilogue (fp16, N %% 32 == 0) and no residual");
  }
  if (d.peer && d.peer->mode) {
    // layout switch fused into the epilogue: per-rank destination maps (gemm_common.cuh: GemmPeer)
    const vc_gemm_peer& q = *d.peer;
    VC_REQUIRE(q.mode == 1 || q.mode == 2, "gemm_tap: peer mode %d", q.mode);
    // before anything indexes f0[world] / dst[rank]
    VC_REQUIRE(q.world >= 2 && q.world <= GEMM_PEER_MAX && q.rank >= 0 && q.rank < q.world, "gemm_tap: peer scatter supports 2..%d ranks", GEMM_PEER_MAX);
    VC_REQUIRE(p.out_tma && !d.geglu && !d.ln_part && d.ldo_y == 0 && d.ldo_z == 0, "gemm_tap: peer scatter needs the fp16 TMA-store epilogue");
    VC_REQUIRE(q.HW % q.world == 0 && q.f0[0] == 0 && q.f0[q.world] == q.T && q.B >= 1, "gemm_tap: peer scatter: bad frame / site split");
    GemmPeer& g = p.peer;
    g.mode = q.mode; g.P = q.world; g.me = q.rank;
    g.HW = q.HW; g.HWl = q.HW / q.world; g.T = q.T;
    g.Tl_me = q.f0[q.rank + 1] - q.f0[q.rank];
    for (int r = 0; r <= q.world; ++r) g.f0[r] = q.f0[r];
    const long long rows = (long long)d.X * d.Y * d.Z;
    g.rps = q.mode == 1 ? q.HW : q.T * g.HWl;
    VC_REQUIRE(rows == (q.mode == 1 ? (long long)q.B * g.Tl_me * q.HW : (long long)q.B * q.T * g.HWl), "gemm_tap: peer scatter: %lld rows do not match the layout", rows);
    // every 32-row patch of the epilogue must be a run of consecutive rows of its slab
    const bool row_major_patches = d.Y == 1 || d.bx == d.X || (d.by == 1 && d.X % 32 == 0);
    VC_REQUIRE(row_major_patches && (d.bx >= 32 || 32 % d.bx == 0), "gemm_tap: peer scatter: tile box %dx%d of a %dx%d image is not row-contiguous", d.bx, d.by, d.X, d.Y);
    if (d.Y == 1 && d.Z == 1) { g.wrap = 1; }
    else { g.wrap = 0; VC_REQUIRE((long long)d.X * d.Y == g.rps, "gemm_tap: peer scatter: slab of %d rows expected, tile geometry has %lld", g.rps, (long long)d.X * d.Y); }
    g.div_hwl = make_fastdiv(g.HWl); g.div_rps = make_fastdiv(g.rps); g.div_tl = make_fastdiv(g.Tl_me > 0 ? g.Tl_me : 1);
    for (int r = 0; r < q.world; ++r) {
      VC_REQUIRE(q.dst[r] && (reinterpret_cast<uintptr_t>(q.dst[r]) & 15) == 0, "gemm_tap: peer scatter: destination %d missing / misaligned", r);
      const int tl_r = q.f0[r + 1] - q.f0[r];
      const __half* base = reinterpret_cast<const __half*>(q.dst[r]) + (q.mode == 2 ? (long long)q.rank * g.HWl * d.N : 0);
      uint64_t dims[3] = {(uint64_t)d.N, (uint64_t)g.HWl, (uint64_t)(q.mode == 1 ? (long long)q.B * q.T : (long long)q.B * tl_r)};
      if (dims[2] == 0) dims[2] = 1;              // a rank without frames: nothing is ever routed to it
      uint64_t str[2] = {(uint64_t)d.N * 2, (uint64_t)(q.mode == 1 ? g.HWl : q.HW) * d.N * 2};
      uint32_t box[3] = {32, 32, 1};
      int rc = encode_tmap_f16(&g.map[r], base, 3, dims, str, box, 64);
      if (rc) return rc;
    }
  }
  const long long total = m_tiles * p.n_tiles;
  VC_REQUIRE(total > 0 && total < (1ll << 31), "gemm_tap: tile count %lld out of range", total);
  p.total_tiles = (int)total;
  if (d.fp8) {
    switch (BN) {
      case 32: return launch_gemm<32, true>(p, stream);
      case 64: return launch_gemm<64, true>(p, stream);
      case 96: return launch_gemm<96, true>(p, stream);
      case 128: return launch_gemm<128, true>(p, stream);
    }
  }
  switch (BN) {
    case 32: return launch_gemm<32>(p, stream);
    case 64: return launch_gemm<64>(p, stream);
    case 96: return launch_gemm<96>(p, stream);
    case 128: return launch_gemm<128>(p, stream);
    case 160: return launch_gemm<160>(p, stream);
  }
  set_error("gemm_tap: no kernel for BN=%d", BN);
  return VC_ERR_UNSUPPORTED;
}

}  // namespace vc

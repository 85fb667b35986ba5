// Temporal self-attention over T <= 128 frames per spatial site (TemporalTransformer attn1/attn2,
// lvdm/modules/attention.py:81-126 with N = T, batch = H*W sites; the reference always takes the naive
// einsum-softmax-einsum path here, attention.py:66).
//
// T <= 32: the problem per (site, head) is a 25x25x64 attention: far below the 64-row granularity of a wgmma and
// HBM-bound (3 x T x 128 B in, T x 128 B out per pair), so it runs on warp-level mma.sync m16n8k16 tiles: one warp
// per (site, head), Q/K/V staged in shared memory with 16-byte coalesced loads, S and O accumulators in registers,
// softmax on the accumulator fragments, P re-used in registers as the A operand of P.V (no smem round trip).
// Rows live at (t * sites + site) so no layout transpose of the activations is ever needed.
#include "common.cuh"
#include "kernels.h"

namespace vc {

static constexpr int TA_PITCH = 72;                       // halves per smem row (64 + 8 pad: conflict-free ldmatrix)
static constexpr int TA_WARPS = 4;
static constexpr int TA_SMEM = TA_WARPS * 3 * 32 * TA_PITCH * 2;

__device__ __forceinline__ void ldsm_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// One warp's 32 x 32 x 64 attention tile: S = Q K^T, softmax over the first n keys (n <= 32; keys >= n are masked, so their K
// rows may hold any finite value and their V rows must be finite), O = P V.  rows.q(r) / rows.k(r) / rows.v(r) give the shared-memory
// address of row r (64 halves, 16-byte aligned).  O (unnormalised) and 1/l are left in the mma accumulator layout: thread
// (g = lane / 4, tg = lane % 4) holds rows mi * 16 + g (+ 8 for h = 1), columns ni * 8 + 2 * tg (+ 1).
template <class Rows>
__device__ __forceinline__ void ta_tile32(const Rows& rows, int n, float scale_log2, int lane, float (&o)[2][8][4], float (&inv_l)[2][2]) {
  const int tg = lane & 3;
  // ---- S = Q K^T : [32 x 32], k = 64 ----
  float s[2][4][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[mi][ni][e] = 0.f;
  const int mat = lane >> 3, mr = lane & 7;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t a[2][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
      ldsm_x4(a[mi][0], a[mi][1], a[mi][2], a[mi][3], rows.q(mi * 16 + (mat & 1) * 8 + mr) + kk * 16 + (mat >> 1) * 8);
#pragma unroll
    for (int np = 0; np < 2; ++np) {                       // two n-tiles (16 keys) per ldmatrix.x4
      uint32_t b0, b1, b2, b3;
      ldsm_x4(b0, b1, b2, b3, rows.k(np * 16 + (mat >> 1) * 8 + mr) + kk * 16 + (mat & 1) * 8);
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        mma16816(s[mi][2 * np], a[mi], b0, b1);
        mma16816(s[mi][2 * np + 1], a[mi], b2, b3);
      }
    }
  }

  // ---- softmax over the key axis (columns); each thread owns rows g / g+8 of both m-tiles ----
  uint32_t p[2][2][4];                                      // P as A fragments: [m-tile][k-step of 16 keys][4]
#pragma unroll
  for (int mi = 0; mi < 2; ++mi) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {                           // h = 0: row g, h = 1: row g + 8
      float mx = -INFINITY;
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = ni * 8 + 2 * tg + e;
          float val = s[mi][ni][2 * h + e];
          if (col >= n) val = -INFINITY;
          s[mi][ni][2 * h + e] = val;
          mx = fmaxf(mx, val);
        }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float off = mx * scale_log2;
      float l = 0.f;
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float pv = exp2f(fmaf(s[mi][ni][2 * h + e], scale_log2, -off));
          s[mi][ni][2 * h + e] = pv;
          l += pv;
        }
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      inv_l[mi][h] = 1.f / l;
    }
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      p[mi][kk][0] = pack_half2(s[mi][2 * kk][0], s[mi][2 * kk][1]);
      p[mi][kk][1] = pack_half2(s[mi][2 * kk][2], s[mi][2 * kk][3]);
      p[mi][kk][2] = pack_half2(s[mi][2 * kk + 1][0], s[mi][2 * kk + 1][1]);
      p[mi][kk][3] = pack_half2(s[mi][2 * kk + 1][2], s[mi][2 * kk + 1][3]);
    }
  }

  // ---- O = P V : [32 x 64], k = 32 keys ----
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 8; ++ni)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[mi][ni][e] = 0.f;
#pragma unroll
  for (int kk = 0; kk < 2; ++kk) {
#pragma unroll
    for (int np = 0; np < 4; ++np) {                       // two d-tiles (16 columns) per ldmatrix.x4.trans
      uint32_t b0, b1, b2, b3;
      ldsm_x4_t(b0, b1, b2, b3, rows.v(kk * 16 + (mat & 1) * 8 + mr) + np * 16 + (mat >> 1) * 8);
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        mma16816(o[mi][2 * np], p[mi][kk], b0, b1);
        mma16816(o[mi][2 * np + 1], p[mi][kk], b2, b3);
      }
    }
  }
}

// Q | K | V tiles of 32 rows each, one after the other (temporal_attn_kernel's per-warp staging).
struct TaTileRows {
  const __half *Qs, *Ks, *Vs;
  __device__ __forceinline__ const __half* q(int r) const { return Qs + r * TA_PITCH; }
  __device__ __forceinline__ const __half* k(int r) const { return Ks + r * TA_PITCH; }
  __device__ __forceinline__ const __half* v(int r) const { return Vs + r * TA_PITCH; }
};

__global__ void __launch_bounds__(TA_WARPS * 32) temporal_attn_kernel(const __half* __restrict__ q, const __half* __restrict__ k,
                                                                      const __half* __restrict__ v, int ld, __half* __restrict__ out,
                                                                      int ldo, int T, long long sites, int heads, float scale_log2) {
  extern __shared__ __align__(16) __half ta_smem[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __half* Qs = ta_smem + w * 3 * 32 * TA_PITCH;
  __half* Ks = Qs + 32 * TA_PITCH;
  __half* Vs = Ks + 32 * TA_PITCH;
  const int g = lane >> 2, tg = lane & 3;
  const int lrow = lane >> 3, lchunk = (lane & 7) * 8;       // cooperative 16-byte copies: 4 rows x 8 chunks per pass
  const long long pairs = sites * heads;

  for (long long pair = (long long)blockIdx.x * TA_WARPS + w; pair < pairs; pair += (long long)gridDim.x * TA_WARPS) {
    const long long site = pair / heads;
    const int head = (int)(pair % heads);
    __syncwarp();
    // ---- global -> smem (rows >= T are zero) ----
    uint4 rq[8], rk[8], rv[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int t = lrow + 4 * i;
      if (t < T) {
        const long long off = ((long long)t * sites + site) * ld + head * 64 + lchunk;
        rq[i] = *reinterpret_cast<const uint4*>(q + off);
        rk[i] = *reinterpret_cast<const uint4*>(k + off);
        rv[i] = *reinterpret_cast<const uint4*>(v + off);
      } else {
        rq[i] = rk[i] = rv[i] = make_uint4(0, 0, 0, 0);
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int t = lrow + 4 * i;
      *reinterpret_cast<uint4*>(Qs + t * TA_PITCH + lchunk) = rq[i];
      *reinterpret_cast<uint4*>(Ks + t * TA_PITCH + lchunk) = rk[i];
      *reinterpret_cast<uint4*>(Vs + t * TA_PITCH + lchunk) = rv[i];
    }
    __syncwarp();

    float o[2][8][4], inv_l[2][2];
    ta_tile32(TaTileRows{Qs, Ks, Vs}, T, scale_log2, lane, o, inv_l);

    // ---- O / l -> smem (reuse the Q tile) -> coalesced 16-byte row stores ----
    __syncwarp();
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 8; ++ni) {
        *reinterpret_cast<uint32_t*>(Qs + (mi * 16 + g) * TA_PITCH + ni * 8 + 2 * tg) =
            pack_half2(o[mi][ni][0] * inv_l[mi][0], o[mi][ni][1] * inv_l[mi][0]);
        *reinterpret_cast<uint32_t*>(Qs + (mi * 16 + g + 8) * TA_PITCH + ni * 8 + 2 * tg) =
            pack_half2(o[mi][ni][2] * inv_l[mi][1], o[mi][ni][3] * inv_l[mi][1]);
      }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int t = lrow + 4 * i;
      if (t < T)
        *reinterpret_cast<uint4*>(out + ((long long)t * sites + site) * ldo + head * 64 + lchunk) =
            *reinterpret_cast<const uint4*>(Qs + t * TA_PITCH + lchunk);
    }
  }
}

// ------------------------------------------------------------------------------------------------ 33 <= T <= 128
// Long clips.  One CTA of TL_WARPS warps runs one (site, head) pair at a time: Q, K and V (KT*16 rows, zero-filled past T) sit in
// shared memory, warp w computes the query tiles w, w + TL_WARPS, ... of 16 rows with the whole score row (KT*16 keys, at most 64 fp32
// per thread) in registers, so the softmax is the single max / exp / sum pass of the T <= 32 kernel and the arithmetic per element is
// the same.  The pair is HBM-bound (T/2 FLOP per byte), so the CTA keeps the next pair's Q/K/V in flight with cp.async while it
// computes the current one (TL_STAGES buffers, grid-stride over the pairs).
static constexpr int TL_WARPS = 4;
static constexpr int TL_STAGES = 2;
static constexpr int TL_MAX_T = 128;

template <int KT>
struct TlShape {
  static constexpr int ROWS = KT * 16;                                // padded frames per pair
  static constexpr int STAGE = 3 * ROWS * TA_PITCH;                   // halves: Q | K | V
  static constexpr int SMEM = TL_STAGES * STAGE * 2;                  // bytes
};

__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
  // src-size 0 zero-fills the 16 bytes without reading src: frames >= T become zero rows
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int KT>
__device__ __forceinline__ void tl_load_pair(__half* stage, const __half* __restrict__ q, const __half* __restrict__ k,
                                             const __half* __restrict__ v, int ld, int T, long long sites, int heads, long long pair) {
  constexpr int ROWS = TlShape<KT>::ROWS;
  const long long site = pair / heads;
  const int head = (int)(pair % heads);
  static_assert(TL_WARPS * 32 == 16 * 8, "one pass copies 16 rows of 8 chunks");
#pragma unroll
  for (int j = 0; j < 3 * KT; ++j) {                                 // pass j: rows 16 (j % KT) .. + 15 of tensor j / KT
    const int which = j / KT, r = 16 * (j % KT) + (threadIdx.x >> 3), c = (threadIdx.x & 7) * 8;
    const __half* src = which == 0 ? q : which == 1 ? k : v;
    const bool valid = r < T;
    const long long off = valid ? ((long long)r * sites + site) * ld + head * 64 + c : 0;
    cp_async16(stage + (which * ROWS + r) * TA_PITCH + c, src + off, valid);
  }
}

template <int KT>
__global__ void __launch_bounds__(TL_WARPS * 32, 2) temporal_attn_long_kernel(const __half* __restrict__ q, const __half* __restrict__ k,
                                                                           const __half* __restrict__ v, int ld, __half* __restrict__ out,
                                                                           int ldo, int T, long long sites, int heads, float scale_log2) {
  constexpr int ROWS = TlShape<KT>::ROWS, STAGE = TlShape<KT>::STAGE;
  extern __shared__ __align__(16) __half tl_smem[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, tg = lane & 3;
  const int mat = lane >> 3, mr = lane & 7;
  const int lrow = lane >> 3, lchunk = (lane & 7) * 8;
  const long long pairs = sites * heads;

  // prologue: the first TL_STAGES - 1 pairs of this CTA
#pragma unroll
  for (int s = 0; s < TL_STAGES - 1; ++s) {
    const long long pair = blockIdx.x + (long long)s * gridDim.x;
    if (pair < pairs) tl_load_pair<KT>(tl_smem + s * STAGE, q, k, v, ld, T, sites, heads, pair);
    cp_async_commit();
  }
  int stage = 0;
  for (long long pair = blockIdx.x; pair < pairs; pair += gridDim.x) {
    {
      const long long ahead = pair + (long long)(TL_STAGES - 1) * gridDim.x;
      if (ahead < pairs) tl_load_pair<KT>(tl_smem + ((stage + TL_STAGES - 1) % TL_STAGES) * STAGE, q, k, v, ld, T, sites, heads, ahead);
      cp_async_commit();
    }
    cp_async_wait<TL_STAGES - 1>();
    __syncthreads();
    __half* Qs = tl_smem + stage * STAGE;
    const __half* Ks = Qs + ROWS * TA_PITCH;
    const __half* Vs = Ks + ROWS * TA_PITCH;
    const long long site = pair / heads;
    const int head = (int)(pair % heads);

    for (int mt = w; mt < KT; mt += TL_WARPS) {
      // ---- S = Q K^T : [16 x ROWS], k = 64 ----
      float s[2 * KT][4];
#pragma unroll
      for (int ni = 0; ni < 2 * KT; ++ni)
#pragma unroll
        for (int e = 0; e < 4; ++e) s[ni][e] = 0.f;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        uint32_t a[4];
        ldsm_x4(a[0], a[1], a[2], a[3], Qs + (mt * 16 + (mat & 1) * 8 + mr) * TA_PITCH + kk * 16 + (mat >> 1) * 8);
#pragma unroll
        for (int np = 0; np < KT; ++np) {                      // two n-tiles (16 keys) per ldmatrix.x4
          uint32_t b0, b1, b2, b3;
          ldsm_x4(b0, b1, b2, b3, Ks + (np * 16 + (mat >> 1) * 8 + mr) * TA_PITCH + kk * 16 + (mat & 1) * 8);
          mma16816(s[2 * np], a, b0, b1);
          mma16816(s[2 * np + 1], a, b2, b3);
        }
      }

      // ---- softmax over the key axis; each thread owns rows g / g + 8 of the tile ----
      uint32_t p[KT][4];                                       // P as A fragments per k-step of 16 keys
      float inv_l[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {                            // h = 0: row g, h = 1: row g + 8
        float mx = -INFINITY;
#pragma unroll
        for (int ni = 0; ni < 2 * KT; ++ni)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = ni * 8 + 2 * tg + e;
            float val = s[ni][2 * h + e];
            if (col >= T) val = -INFINITY;
            s[ni][2 * h + e] = val;
            mx = fmaxf(mx, val);
          }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float off = mx * scale_log2;
        float l = 0.f;
#pragma unroll
        for (int ni = 0; ni < 2 * KT; ++ni)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float pv = exp2f(fmaf(s[ni][2 * h + e], scale_log2, -off));
            s[ni][2 * h + e] = pv;
            l += pv;
          }
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        inv_l[h] = 1.f / l;
      }
#pragma unroll
      for (int kk = 0; kk < KT; ++kk) {
        p[kk][0] = pack_half2(s[2 * kk][0], s[2 * kk][1]);
        p[kk][1] = pack_half2(s[2 * kk][2], s[2 * kk][3]);
        p[kk][2] = pack_half2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
        p[kk][3] = pack_half2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
      }

      // ---- O = P V : [16 x 64], k = ROWS keys (V rows >= T are zero and their P is 0) ----
      float o[8][4];
#pragma unroll
      for (int ni = 0; ni < 8; ++ni)
#pragma unroll
        for (int e = 0; e < 4; ++e) o[ni][e] = 0.f;
#pragma unroll
      for (int kk = 0; kk < KT; ++kk) {
#pragma unroll
        for (int np = 0; np < 4; ++np) {                       // two d-tiles (16 columns) per ldmatrix.x4.trans
          uint32_t b0, b1, b2, b3;
          ldsm_x4_t(b0, b1, b2, b3, Vs + (kk * 16 + (mat & 1) * 8 + mr) * TA_PITCH + np * 16 + (mat >> 1) * 8);
          mma16816(o[2 * np], p[kk], b0, b1);
          mma16816(o[2 * np + 1], p[kk], b2, b3);
        }
      }

      // ---- O / l -> this warp's own Q rows -> coalesced 16-byte row stores ----
      __syncwarp();
      __half* Os = Qs + mt * 16 * TA_PITCH;
#pragma unroll
      for (int ni = 0; ni < 8; ++ni) {
        *reinterpret_cast<uint32_t*>(Os + g * TA_PITCH + ni * 8 + 2 * tg) = pack_half2(o[ni][0] * inv_l[0], o[ni][1] * inv_l[0]);
        *reinterpret_cast<uint32_t*>(Os + (g + 8) * TA_PITCH + ni * 8 + 2 * tg) = pack_half2(o[ni][2] * inv_l[1], o[ni][3] * inv_l[1]);
      }
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = lrow + 4 * i, t = mt * 16 + r;
        if (t < T)
          *reinterpret_cast<uint4*>(out + ((long long)t * sites + site) * ldo + head * 64 + lchunk) =
              *reinterpret_cast<const uint4*>(Os + r * TA_PITCH + lchunk);
      }
    }
    __syncthreads();                                           // this stage is refilled by the next iteration's prefetch
    stage = (stage + 1) % TL_STAGES;
  }
  cp_async_wait<0>();
}

template <int KT>
static int temporal_attn_long(const __half* q, const __half* k, const __half* v, int ld, __half* out, int ldo, int T, long long sites,
                              int heads, float scale_log2, cudaStream_t stream) {
  constexpr int SMEM = TlShape<KT>::SMEM;
  static DeviceOnce configured;
  if (device_once_needed(configured)) {
    VC_CHECK_CUDA(cudaFuncSetAttribute(temporal_attn_long_kernel<KT>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    device_once_mark(configured);
  }
  int per_sm = 0;
  VC_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, temporal_attn_long_kernel<KT>, TL_WARPS * 32, SMEM));
  VC_REQUIRE(per_sm >= 1, "temporal_attn: the T=%d kernel does not fit on an SM", T);
  const long long pairs = sites * heads;
  VC_REQUIRE(pairs >= 1, "temporal_attn: sites=%lld heads=%d", sites, heads);
  long long blocks = (long long)per_sm * sm_count();                // grid-stride beyond one resident wave
  if (blocks > pairs) blocks = pairs;
  temporal_attn_long_kernel<KT><<<(unsigned)blocks, TL_WARPS * 32, SMEM, stream>>>(q, k, v, ld, out, ldo, T, sites, heads, scale_log2);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

int temporal_attn(const __half* q, const __half* k, const __half* v, int ld, __half* out, int ldo, int T, long long sites,
                  int heads, float scale, cudaStream_t stream) {
  VC_REQUIRE(T >= 1 && T <= TL_MAX_T, "temporal_attn: T=%d unsupported (1..%d)", T, TL_MAX_T);
  VC_REQUIRE(q && k && v && out, "temporal_attn: null pointer");
  VC_REQUIRE(ld % 8 == 0 && ldo % 8 == 0, "temporal_attn: pitches must be multiples of 8");
  if (T > 32) {
    const float sl2 = scale * 1.4426950408889634f;
    switch ((T + 15) / 16) {
      case 3: return temporal_attn_long<3>(q, k, v, ld, out, ldo, T, sites, heads, sl2, stream);
      case 4: return temporal_attn_long<4>(q, k, v, ld, out, ldo, T, sites, heads, sl2, stream);
      case 5: return temporal_attn_long<5>(q, k, v, ld, out, ldo, T, sites, heads, sl2, stream);
      case 6: return temporal_attn_long<6>(q, k, v, ld, out, ldo, T, sites, heads, sl2, stream);
      case 7: return temporal_attn_long<7>(q, k, v, ld, out, ldo, T, sites, heads, sl2, stream);
      default: return temporal_attn_long<8>(q, k, v, ld, out, ldo, T, sites, heads, sl2, stream);
    }
  }
  static DeviceOnce configured;
  if (device_once_needed(configured)) {
    VC_CHECK_CUDA(cudaFuncSetAttribute(temporal_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TA_SMEM));
    device_once_mark(configured);
  }
  const long long pairs = sites * heads;
  long long blocks = (pairs + TA_WARPS - 1) / TA_WARPS;
  const long long cap = (long long)sm_count() * 4;          // 4 resident blocks per SM (55 KB smem each), grid-stride beyond
  if (blocks > cap) blocks = cap;
  temporal_attn_kernel<<<(unsigned)blocks, TA_WARPS * 32, TA_SMEM, stream>>>(q, k, v, ld, out, ldo, T, sites, heads,
                                                                            scale * 1.4426950408889634f);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}


// ------------------------------------------------------------------------------------------------ windowed (FreeNoise)
// Windowed temporal attention: overlapping windows of W <= 32 frames at starts 0, S, 2S, ... (while start + W < T) and T - W; frame
// j of a window carries the weight min(j + 1, W - j) and out_t is the weighted mean of the outputs of the windows that contain t,
// summed in window order (INTEGRATION.md "Long clips: windowed temporal attention").  T > W only (T <= W is the plain kernel).
// One warp per (site, head) pair walks its windows in order; each window is ta_tile32 on shared-memory rows.  Frames stream
// through a TW_RING-frame Q/K/V ring in chunks of 16 with cp.async, up to TW_RING - W frames ahead of the window, so each input row is
// read from HBM once per pair.  The weighted fp32 sums of the open frames (at most W of them) live in a TW_ACC-row ring; a frame
// is divided by its weight sum and written out once the next window starts past it.  Shared memory is O(W), independent of T.
static constexpr int TW_WARPS = 2;
static constexpr int TW_MAX_W = 32;
static constexpr int TW_RING = 64;                                    // frames per Q/K/V ring (power of two, >= W + 16)
static constexpr int TW_CHUNK = 16;                                   // frames per cp.async group
static constexpr int TW_ACC = 32;                                     // open output rows (power of two, >= W)
static constexpr int TW_ACC_PITCH = 72;                               // floats per accumulator row (conflict-free float2 access)
static constexpr int TW_WARP_HALVES = 3 * TW_RING * TA_PITCH + TW_ACC * TW_ACC_PITCH * 2;
static constexpr int TW_SMEM = (64 + TW_WARPS * TW_WARP_HALVES) * 2; // one zero row + per-warp rings
static_assert(TW_ACC >= TW_MAX_W && TW_RING >= TW_MAX_W + TW_CHUNK, "ring sizes");

// Window i of n (T > W): i * S, the last one T - W.  n = ceil((T - W) / S) + 1.
__host__ __device__ __forceinline__ int tw_windows(int T, int W, int S) { return (T - W + S - 1) / S + 1; }
__host__ __device__ __forceinline__ int tw_start(int i, int n, int T, int W, int S) { return i == n - 1 ? T - W : i * S; }
// sum of min(j + 1, W - j) over the windows that contain frame t (j = t - start), from (t, T, W, S) alone
__host__ __device__ __forceinline__ int tw_weight_sum(int t, int T, int W, int S) {
  const int n = tw_windows(T, W, S);
  int sum = 0;
  for (int i = t < W ? 0 : (t - W) / S + 1; i < n - 1 && i * S <= t; ++i) {
    const int j = t - i * S;
    sum += min(j + 1, W - j);
  }
  if (t >= T - W) sum += min(t - (T - W) + 1, T - t);
  return sum;
}

// Q | K | V rings; window rows r >= W read the shared zero row
struct TwRingRows {
  const __half* ring;
  const __half* zero;
  int start, W;
  __device__ __forceinline__ const __half* row(int which, int r) const {
    return r < W ? ring + (which * TW_RING + ((start + r) & (TW_RING - 1))) * TA_PITCH : zero;
  }
  __device__ __forceinline__ const __half* q(int r) const { return row(0, r); }
  __device__ __forceinline__ const __half* k(int r) const { return row(1, r); }
  __device__ __forceinline__ const __half* v(int r) const { return row(2, r); }
};

// frames 16c .. 16c + 15 of one pair into the rings (frames >= T are zero-filled), one cp.async group
__device__ __forceinline__ void tw_load_chunk(__half* ring, const __half* __restrict__ q, const __half* __restrict__ k,
                                              const __half* __restrict__ v, int ld, int T, long long sites, long long site, int head,
                                              int c, int lane) {
  const int lrow = lane >> 3, lchunk = (lane & 7) * 8;
#pragma unroll
  for (int j = 0; j < 3 * TW_CHUNK / 4; ++j) {
    const int which = j / (TW_CHUNK / 4), t = c * TW_CHUNK + (j % (TW_CHUNK / 4)) * 4 + lrow;
    const __half* src = which == 0 ? q : which == 1 ? k : v;
    const bool valid = t < T;
    const long long off = valid ? ((long long)t * sites + site) * ld + head * 64 + lchunk : 0;
    cp_async16(ring + (which * TW_RING + (t & (TW_RING - 1))) * TA_PITCH + lchunk, src + off, valid);
  }
  cp_async_commit();
}

__global__ void __launch_bounds__(TW_WARPS * 32) temporal_attn_windowed_kernel(const __half* __restrict__ q, const __half* __restrict__ k,
                                                                             const __half* __restrict__ v, int ld, __half* __restrict__ out,
                                                                             int ldo, int T, long long sites, int heads, int W, int S,
                                                                             float scale_log2) {
  extern __shared__ __align__(16) __half tw_smem[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, tg = lane & 3;
  const int lrow = lane >> 3, lchunk = (lane & 7) * 8;
  const __half* zero = tw_smem;
  __half* ring = tw_smem + 64 + w * TW_WARP_HALVES;
  float* acc = reinterpret_cast<float*>(ring + 3 * TW_RING * TA_PITCH);
  if (threadIdx.x < 8) reinterpret_cast<uint4*>(tw_smem)[threadIdx.x] = make_uint4(0, 0, 0, 0);
  for (int i = lane; i < TW_ACC * TW_ACC_PITCH / 4; i += 32) reinterpret_cast<float4*>(acc)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();                                                    // the zero row is shared by the CTA's warps

  const int nwin = tw_windows(T, W, S), nchunk = (T + TW_CHUNK - 1) / TW_CHUNK;
  const long long pairs = sites * heads;
  for (long long pair = (long long)blockIdx.x * TW_WARPS + w; pair < pairs; pair += (long long)gridDim.x * TW_WARPS) {
    const long long site = pair / heads;
    const int head = (int)(pair % heads);
    int issued = 0;
    for (int wi = 0; wi < nwin; ++wi) {
      const int s0 = tw_start(wi, nwin, T, W, S);
      const int s1 = wi + 1 < nwin ? tw_start(wi + 1, nwin, T, W, S) : T;   // frames [s0, s1) are complete after this window
      // chunk c overwrites the ring rows of frames 16c - TW_RING ..: issue it once those are all below s0 (already consumed)
      __syncwarp();
      while (issued < nchunk && (issued + 1) * TW_CHUNK <= s0 + TW_RING) tw_load_chunk(ring, q, k, v, ld, T, sites, site, head, issued++, lane);
      switch (issued - (s0 + W + TW_CHUNK - 1) / TW_CHUNK) {       // groups that may stay in flight: those past this window
        case 0: cp_async_wait<0>(); break;
        case 1: cp_async_wait<1>(); break;
        case 2: cp_async_wait<2>(); break;
        default: cp_async_wait<3>(); break;
      }
      __syncwarp();

      float o[2][8][4], inv_l[2][2];
      ta_tile32(TwRingRows{ring, zero, s0, W}, W, scale_log2, lane, o, inv_l);

      // ---- acc[t] += w_j * O_j (fp32, window order) ----
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = mi * 16 + g + 8 * h;
          if (r < W) {
            const float wt = (float)min(r + 1, W - r);
            float* a = acc + ((s0 + r) & (TW_ACC - 1)) * TW_ACC_PITCH + 2 * tg;
#pragma unroll
            for (int ni = 0; ni < 8; ++ni) {
              float2 cur = *reinterpret_cast<float2*>(a + ni * 8);
              cur.x += wt * (o[mi][ni][2 * h] * inv_l[mi][h]);
              cur.y += wt * (o[mi][ni][2 * h + 1] * inv_l[mi][h]);
              *reinterpret_cast<float2*>(a + ni * 8) = cur;
            }
          }
        }
      __syncwarp();

      // ---- frames [s0, s1): / weight sum -> fp16 -> 16-byte row stores; their accumulator rows are cleared for reuse ----
      for (int t = s0 + lrow; t < s1; t += 4) {
        float4* a = reinterpret_cast<float4*>(acc + (t & (TW_ACC - 1)) * TW_ACC_PITCH + lchunk);
        const float ws = (float)tw_weight_sum(t, T, W, S);
        const float4 a0 = a[0], a1 = a[1];
        uint4 r;
        r.x = pack_half2(a0.x / ws, a0.y / ws);
        r.y = pack_half2(a0.z / ws, a0.w / ws);
        r.z = pack_half2(a1.x / ws, a1.y / ws);
        r.w = pack_half2(a1.z / ws, a1.w / ws);
        *reinterpret_cast<uint4*>(out + ((long long)t * sites + site) * ldo + head * 64 + lchunk) = r;
        a[0] = a[1] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  }
  cp_async_wait<0>();
}

int temporal_attn_windowed(const __half* q, const __half* k, const __half* v, int ld, __half* out, int ldo, int T, long long sites,
                           int heads, int W, int S, float scale, cudaStream_t stream) {
  VC_REQUIRE(T >= 1, "temporal_attn_windowed: T=%d unsupported (>= 1)", T);
  VC_REQUIRE(W >= 2 && W <= TW_MAX_W, "temporal_attn_windowed: window W=%d unsupported (2..%d)", W, TW_MAX_W);
  VC_REQUIRE(S >= 1 && S <= W, "temporal_attn_windowed: stride S=%d unsupported (1..W=%d)", S, W);
  VC_REQUIRE(q && k && v && out, "temporal_attn_windowed: null pointer");
  VC_REQUIRE(ld % 8 == 0 && ldo % 8 == 0, "temporal_attn_windowed: pitches must be multiples of 8");
  VC_REQUIRE(sites >= 1 && heads >= 1, "temporal_attn_windowed: sites=%lld heads=%d", sites, heads);
  if (T <= W) return temporal_attn(q, k, v, ld, out, ldo, T, sites, heads, scale, stream);   // one window: full attention
  static DeviceOnce configured;
  if (device_once_needed(configured)) {
    VC_CHECK_CUDA(cudaFuncSetAttribute(temporal_attn_windowed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TW_SMEM));
    device_once_mark(configured);
  }
  int per_sm = 0;
  VC_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, temporal_attn_windowed_kernel, TW_WARPS * 32, TW_SMEM));
  VC_REQUIRE(per_sm >= 1, "temporal_attn_windowed: the kernel does not fit on an SM");
  const long long pairs = sites * heads;
  long long blocks = (pairs + TW_WARPS - 1) / TW_WARPS;
  const long long cap = (long long)per_sm * sm_count();               // grid-stride beyond one resident wave
  if (blocks > cap) blocks = cap;
  temporal_attn_windowed_kernel<<<(unsigned)blocks, TW_WARPS * 32, TW_SMEM, stream>>>(q, k, v, ld, out, ldo, T, sites, heads, W, S,
                                                                                      scale * 1.4426950408889634f);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

}  // namespace vc

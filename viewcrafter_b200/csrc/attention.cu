// FlashAttention-style fused softmax(Q K^T * scale) V for head_dim 64 on wgmma (sm_90a).
//
// Used for the spatial self-attention (Nq = Nk = H*W up to 9216) and the text / image cross-attention
// (Nk = 77 / 256) of lvdm/modules/attention.py:81-144.  One CTA owns 128 query rows of one (batch, head) and streams
// BNK-key tiles of K and V through a two-stage TMA ring.  Each of the two MMA warpgroups owns 64 query rows:
//     S = Q K^T          wgmma m64nBNKk16, both operands from shared memory (128B-swizzled TMA tiles)
//     online softmax     on the accumulator fragments (two rows per thread, row max / sum over the 4-lane quad), exp2 domain
//     O += P V           wgmma with P as the register A operand (the S fragments re-packed to fp16 in place) and the V tile
//                        read MN-major (tnspB) straight from the TMA tile
// Warp roles (288 threads): warps 0..7 = two MMA / softmax warpgroups, warp 8 = TMA producer.
// Two tile widths: 64 keys (short key sequences: cross-attention, the 18x32 and 9x16 levels; smaller register and
// shared-memory footprint, two CTAs per SM) and 128 keys (long sequences: half the barrier round trips per key).
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace vc {

struct AttnParams {
  CUtensorMap tmap_q, tmap_k, tmap_v;
  __half* out;
  int ldo;
  int Nq, Nk;
  int kv_shared;       // 1: K/V batch coordinate is always 0
  float scale_log2;    // scale * log2(e)
  int accumulate;
};

static constexpr int ATT_BM = 128, ATT_D = 64;
static constexpr int ATT_THREADS = 288;
static constexpr int ATT_Q_BYTES = ATT_BM * ATT_D * 2;                 // 16 KB

template <int BNK>
struct AttnCfg {
  static constexpr int KV_BYTES = BNK * ATT_D * 2;
  static constexpr int SMEM = ATT_Q_BYTES + 4 * KV_BYTES + 1024 + 256;  // Q + 2 x (K, V) + alignment slack + barriers
  static constexpr int MIN_CTAS = BNK == 64 ? 2 : 1;
};

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int BNK>
__global__ void __launch_bounds__(ATT_THREADS, AttnCfg<BNK>::MIN_CTAS) flash_attn_d64_kernel(const __grid_constant__ AttnParams p) {
  using Cfg = AttnCfg<BNK>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + ATT_Q_BYTES;                                    // stage s: K at s * 2 KV, V at s * 2 KV + KV
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ATT_Q_BYTES + 4 * Cfg::KV_BYTES);
  uint64_t* q_full = bars + 0;
  uint64_t* kv_full = bars + 1;    // [2]  K and V tiles landed
  uint64_t* kv_empty = bars + 3;   // [2]  both warpgroups are done with the stage (one arrival per MMA warp)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * ATT_BM, head = blockIdx.y, b = blockIdx.z;
  const int bk = p.kv_shared ? 0 : b;
  const int ntiles = (p.Nk + BNK - 1) / BNK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmap_q);
    tma_prefetch_desc(&p.tmap_k);
    tma_prefetch_desc(&p.tmap_v);
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1); mbar_init(&kv_full[1], 1);
    mbar_init(&kv_empty[0], 8); mbar_init(&kv_empty[1], 8);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ------------------------------ TMA producer ------------------------------
    if (elect_one()) {
      mbar_expect_tx(q_full, ATT_Q_BYTES);
      tma_load_4d(sQ, &p.tmap_q, q_full, 0, head, q0, b);
    }
    __syncwarp();
    for (int j = 0; j < ntiles; ++j) {
      const int s = j & 1;
      uint8_t* sk = sKV + s * 2 * Cfg::KV_BYTES;
      if (j >= 2) mbar_wait(&kv_empty[s], ((j >> 1) - 1) & 1);          // tile j-2 fully consumed
      if (elect_one()) {
        mbar_expect_tx(&kv_full[s], 2 * Cfg::KV_BYTES);
        tma_load_4d(sk, &p.tmap_k, &kv_full[s], 0, head, j * BNK, bk);
        tma_load_4d(sk + Cfg::KV_BYTES, &p.tmap_v, &kv_full[s], 0, head, j * BNK, bk);
      }
      __syncwarp();
    }
    return;
  }

  // ------------------------------ MMA / softmax warpgroups ------------------------------
  const int cw = warp >> 2, wl = warp & 3;
  const uint32_t aQ = smem_u32(sQ) + cw * (64 * ATT_D * 2);
  const float sl2 = p.scale_log2;
  float o[32];                                      // O fragments: 64 rows x 64 columns per warpgroup
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // rows r0 and r0 + 8 of this thread (l: this thread's partial sum)
  mbar_wait(q_full, 0);
  for (int j = 0; j < ntiles; ++j) {
    const int s = j & 1;
    const uint32_t aK = smem_u32(sKV + s * 2 * Cfg::KV_BYTES);
    const uint32_t aV = aK + Cfg::KV_BYTES;
    mbar_wait(&kv_full[s], (j >> 1) & 1);
    float sc[BNK / 2];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < ATT_D / 16; ++k) Wgmma<BNK>::ss(sc, wgmma_desc_sw128(aQ + 32 * k), wgmma_desc_sw128(aK + 32 * k), k > 0 ? 1 : 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);

    const int valid = p.Nk - j * BNK;
    if (valid < BNK) {
#pragma unroll
      for (int i = 0; i < BNK / 2; ++i) {
        const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        if (col >= valid) sc[i] = -INFINITY;       // masked keys get probability 0
      }
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < BNK / 2; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sc[i]);
    float alpha[2], negm[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float mn = fmaxf(m[h], mx[h] * sl2);
      alpha[h] = ex2f(m[h] - mn);                   // 0 on the first tile (m = -inf)
      m[h] = mn;
      negm[h] = -mn;
      l[h] *= alpha[h];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
    // probabilities, packed to fp16 A fragments: k-slice kk covers accumulator column groups 2 kk and 2 kk + 1
    uint32_t pa[BNK / 16][4];
#pragma unroll
    for (int kk = 0; kk < BNK / 16; ++kk) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = (2 * kk + (r >> 1)) * 4 + 2 * (r & 1);   // r: (row r0, k lo), (row r0+8, k lo), (row r0, k hi), (row r0+8, k hi)
        const int h = r & 1;
        const float e0 = ex2f(fmaf(sc[i], sl2, negm[h])), e1 = ex2f(fmaf(sc[i + 1], sl2, negm[h]));
        l[h] += e0 + e1;
        pa[kk][r] = pack_half2(e0, e1);
      }
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BNK / 16; ++kk) Wgmma<64, 1>::rs(o, pa[kk], wgmma_desc_sw128(aV + kk * 16 * 128), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[s]);
  }

  // epilogue: O / l, rows r0 = 16 wl + lane / 4 and r0 + 8 of the warpgroup's 64
  float inv[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float t = l[h];
    t += __shfl_xor_sync(0xffffffffu, t, 1);
    t += __shfl_xor_sync(0xffffffffu, t, 2);
    inv[h] = 1.f / t;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = q0 + cw * 64 + 16 * wl + (lane >> 2) + 8 * h;
    if (row >= p.Nq) continue;
    __half* op = p.out + ((long long)b * p.Nq + row) * p.ldo + head * ATT_D + 2 * (lane & 3);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      float v0 = o[jj * 4 + 2 * h] * inv[h], v1 = o[jj * 4 + 2 * h + 1] * inv[h];
      __half2* dst = reinterpret_cast<__half2*>(op + 8 * jj);
      if (p.accumulate) {
        const float2 t = __half22float2(*dst);
        v0 += t.x; v1 += t.y;
      }
      *dst = __floats2half2_rn(v0, v1);
    }
  }
}

// env VC_ATTN_BN64 = 1 / 0 forces the 64- / 128-key tiles for every shape; unset: by key count
static int bn64_mode() {
  static int mode = -2;
  if (mode == -2) { const char* e = getenv("VC_ATTN_BN64"); mode = !e ? -1 : (e[0] == '1' ? 1 : 0); }
  return mode;
}

template <int BNK>
static int launch_attn(const vc_attn_desc& d, cudaStream_t stream) {
  using Cfg = AttnCfg<BNK>;
  AttnParams p;
  memset(&p, 0, sizeof(p));
  {
    uint64_t dims[4] = {64, (uint64_t)d.heads, (uint64_t)d.Nq, (uint64_t)d.B};
    uint64_t str[3] = {128, (uint64_t)d.ldq * 2, (uint64_t)d.ldq * 2 * d.Nq};
    uint32_t box[4] = {64, 1, ATT_BM, 1};
    int rc = encode_tmap_f16(&p.tmap_q, d.q, 4, dims, str, box);
    if (rc) return rc;
  }
  const int shared = d.kv_batch_stride == 0;
  {
    uint64_t dims[4] = {64, (uint64_t)d.heads, (uint64_t)d.Nk, (uint64_t)(shared ? 1 : d.B)};
    uint64_t strk[3] = {128, (uint64_t)d.ldk * 2, (uint64_t)(shared ? (long long)d.ldk * d.Nk : d.kv_batch_stride) * 2};
    uint64_t strv[3] = {128, (uint64_t)d.ldv * 2, (uint64_t)(shared ? (long long)d.ldv * d.Nk : d.kv_batch_stride) * 2};
    uint32_t box[4] = {64, 1, (uint32_t)BNK, 1};
    int rc = encode_tmap_f16(&p.tmap_k, d.k, 4, dims, strk, box);
    if (rc) return rc;
    rc = encode_tmap_f16(&p.tmap_v, d.v, 4, dims, strv, box);
    if (rc) return rc;
  }
  p.out = static_cast<__half*>(d.out); p.ldo = d.ldo; p.Nq = d.Nq; p.Nk = d.Nk; p.kv_shared = shared;
  p.scale_log2 = d.scale * 1.4426950408889634f;
  p.accumulate = d.accumulate;
  static DeviceOnce configured;
  if (device_once_needed(configured)) {
    VC_CHECK_CUDA(cudaFuncSetAttribute(flash_attn_d64_kernel<BNK>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
    device_once_mark(configured);
  }
  dim3 grid((d.Nq + ATT_BM - 1) / ATT_BM, d.heads, d.B);
  flash_attn_d64_kernel<BNK><<<grid, ATT_THREADS, Cfg::SMEM, stream>>>(p);
  VC_CHECK_CUDA(cudaGetLastError());
  return VC_OK;
}

int flash_attn_d64(const vc_attn_desc& d, cudaStream_t stream) {
  VC_REQUIRE(d.q && d.k && d.v && d.out, "flash_attn: null pointer");
  VC_REQUIRE(d.Nq > 0 && d.Nk > 0 && d.B > 0 && d.heads > 0, "flash_attn: empty problem");
  VC_REQUIRE(d.ldq % 8 == 0 && d.ldk % 8 == 0 && d.ldv % 8 == 0 && d.ldo % 8 == 0, "flash_attn: pitches must be multiples of 8");
  VC_REQUIRE(d.kv_batch_stride % 8 == 0, "flash_attn: kv batch stride must be a multiple of 8");
  const int mode = bn64_mode();
  if (mode == 1 || (mode < 0 && d.Nk <= 1024)) return launch_attn<64>(d, stream);
  return launch_attn<128>(d, stream);
}

}  // namespace vc

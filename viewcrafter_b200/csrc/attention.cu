// FlashAttention-style fused softmax(Q K^T * scale) V for head_dim 64 on wgmma (sm_90a).
//
// Used for the spatial self-attention (Nq = Nk = H*W up to 9216) and the text / image cross-attention
// (Nk = 77 / 256) of lvdm/modules/attention.py:81-144.  One CTA owns 128 (64-key tiles) or 192 (128-key tiles) query rows
// of one (batch, head) and streams BNK-key tiles of K and V through TMA rings.  Each MMA warpgroup owns 64 query rows:
//     S = Q K^T          wgmma m64nBNKk16, both operands from shared memory (128B-swizzled TMA tiles)
//     online softmax     on the accumulator fragments (two rows per thread, row max / sum over the 4-lane quad), exp2 domain
//     O += P V           wgmma with P as the register A operand (the S fragments re-packed to fp16 in place) and the V tile
//                        read MN-major (tnspB) straight from the TMA tile
// Two tile widths: 64 keys (short key sequences: cross-attention, the 18x32 and 9x16 levels; smaller register and
// shared-memory footprint, two CTAs per SM) and 128 keys (long sequences).
//
// 64 keys, serial schedule (288 threads): warps 0..7 = the two MMA / softmax warpgroups, warp 8 = TMA producer; one
// two-stage ring of (K, V) pairs.  Each warpgroup runs S, softmax, PV one after the other.
//
// 128 keys, pipelined schedule (512 threads): warpgroup 0 = TMA producer (gives its registers to the others with setmaxnreg),
// warpgroups 1..3 = MMA / softmax.  At d = 64 a score costs the tensor cores and the MUFU (one ex2) the same time, so the
// exponentials of a tile run while the tensor cores work, and three MMA warpgroups (a third warp per SM sub-partition)
// hide more of the softmax's latency than two:
//   - K and V have separate three-stage rings with their own full / empty barriers; the producer loads K(j+1) before V(j)
//     and a K stage is released when the S that read it retires, a V stage when the PV that read it retires.
//   - Inside a warpgroup: S(j+1) = Q K(j+1)^T and O += P(j) V(j) are issued back to back; the softmax of S(j+1) runs in
//     fp32 registers while PV(j) is on the tensor cores, and P(j+1) is packed to fp16 once PV(j) has retired.
//   - Between the warpgroups: a named-barrier turn (round robin) lets one warpgroup issue its MMAs while the others run
//     their exponentials.
// Both schedules compute every element with the same operations in the same order (attn_mask / attn_softmax / attn_pack /
// attn_rescale / attn_store), so their outputs are bit-identical: each tile's row max, alpha = 2^(m_old - m_new) applied
// to l before the tile's exponentials are summed and to O after the previous tile's PV retired and before this tile's PV
// accumulates, and one rounding of O / l (+ the accumulated output) at the end.
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

static constexpr int ATT_D = 64;
// pipelined schedule: register split between the producer warpgroup and the three MMA warpgroups
static constexpr int ATT_PRODUCER_REGS = 24;
static constexpr int ATT_MMA_REGS = 160;
static_assert(128 * ATT_PRODUCER_REGS + 3 * 128 * ATT_MMA_REGS <= 65536, "register split exceeds the register file");
static constexpr int ATT_BAR_TURN = 1;   // named barriers 1 + cw: "MMA warpgroup cw may issue" (0 is __syncthreads)

template <int BNK>
struct AttnCfg {
  static constexpr bool PIPELINED = BNK == 128;
  static constexpr int MMA_WGS = PIPELINED ? 3 : 2;                      // MMA warpgroups, 64 query rows each
  static constexpr int BM = 64 * MMA_WGS;                                // query rows per CTA
  static constexpr int Q_BYTES = BM * ATT_D * 2;
  static constexpr int THREADS = PIPELINED ? 128 * (1 + MMA_WGS) : 288;
  static constexpr int STAGES = PIPELINED ? 3 : 2;                       // per operand (K ring, V ring)
  static constexpr int KV_BYTES = BNK * ATT_D * 2;
  static constexpr int SMEM = Q_BYTES + 2 * STAGES * KV_BYTES + 1024 + 256;  // Q + K ring + V ring + alignment slack + barriers
  static constexpr int MIN_CTAS = BNK == 64 ? 2 : 1;
};

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Scores of keys >= valid (the tail of the last key tile) get probability 0.
template <int BNK>
__device__ __forceinline__ void attn_mask(float (&sc)[BNK / 2], int valid, int lane) {
#pragma unroll
  for (int i = 0; i < BNK / 2; ++i) {
    const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
    if (col >= valid) sc[i] = -INFINITY;
  }
}

// Online softmax of one score tile on the accumulator fragments of rows r0 and r0 + 8 (h = 0, 1) of this thread: update
// the running max m and this thread's partial sum l, return the rescale factor alpha for O and the unnormalised
// probabilities e (fp32, in the accumulator layout).
template <int BNK>
__device__ __forceinline__ void attn_softmax(const float (&sc)[BNK / 2], float sl2, float (&m)[2], float (&l)[2], float (&alpha)[2],
                                             float (&e)[BNK / 2]) {
  // Row max.  The 128-key tile splits each row into four independent chains, which shortens the latency the softmax adds
  // to a warpgroup's turn; the max is exact, so the grouping does not change it.  (The 64-key kernel runs two CTAs per SM.)
  constexpr int CH = BNK == 128 ? 4 : 1;
  float mxc[2][CH];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int c = 0; c < CH; ++c) mxc[h][c] = -INFINITY;
#pragma unroll
  for (int i = 0; i < BNK / 2; ++i) mxc[(i >> 1) & 1][(i >> 2) % CH] = fmaxf(mxc[(i >> 1) & 1][(i >> 2) % CH], sc[i]);
  float mx[2], negm[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    mx[h] = mxc[h][0];
#pragma unroll
    for (int c = 1; c < CH; ++c) mx[h] = fmaxf(mx[h], mxc[h][c]);
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    const float mn = fmaxf(m[h], mx[h] * sl2);
    alpha[h] = ex2f(m[h] - mn);                   // 0 on the first tile (m = -inf)
    m[h] = mn;
    negm[h] = -mn;
    l[h] *= alpha[h];
  }
#pragma unroll
  for (int kk = 0; kk < BNK / 16; ++kk) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = (2 * kk + (r >> 1)) * 4 + 2 * (r & 1);   // r: (row r0, k lo), (row r0+8, k lo), (row r0, k hi), (row r0+8, k hi)
      const int h = r & 1;
      e[i] = ex2f(fmaf(sc[i], sl2, negm[h]));
      e[i + 1] = ex2f(fmaf(sc[i + 1], sl2, negm[h]));
      l[h] += e[i] + e[i + 1];
    }
  }
}

// The probabilities as fp16 A fragments of the PV MMA: k-slice kk covers accumulator column groups 2 kk and 2 kk + 1.
template <int BNK>
__device__ __forceinline__ void attn_pack(const float (&e)[BNK / 2], uint32_t (&pa)[BNK / 16][4]) {
#pragma unroll
  for (int kk = 0; kk < BNK / 16; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = (2 * kk + (r >> 1)) * 4 + 2 * (r & 1);
      pa[kk][r] = pack_half2(e[i], e[i + 1]);
    }
}

__device__ __forceinline__ void attn_rescale(float (&o)[32], const float (&alpha)[2]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
}

// epilogue: O / l, rows r0 = 16 wl + lane / 4 and r0 + 8 of the 64 rows starting at row0
__device__ __forceinline__ void attn_store(const AttnParams& p, const float (&o)[32], const float (&l)[2], int row0, int wl, int lane,
                                           int head, int b) {
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
    const int row = row0 + 16 * wl + (lane >> 2) + 8 * h;
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

template <int BNK>
__global__ void __launch_bounds__(AttnCfg<BNK>::THREADS, AttnCfg<BNK>::MIN_CTAS) flash_attn_d64_kernel(const __grid_constant__ AttnParams p) {
  using Cfg = AttnCfg<BNK>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = smem + Cfg::Q_BYTES;                                    // stage s: K at s * KV
  uint8_t* sV = sK + STAGES * Cfg::KV_BYTES;                            //          V at s * KV
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + STAGES * Cfg::KV_BYTES);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;                     // [STAGES]  K tile landed (serial schedule: K and V tiles landed)
  uint64_t* k_empty = k_full + STAGES;             // [STAGES]  both warpgroups are done with the K tile (one arrival per MMA warp)
  uint64_t* v_full = k_empty + STAGES;             // [STAGES]  pipelined schedule only
  uint64_t* v_empty = v_full + STAGES;             // [STAGES]
  float* pin = reinterpret_cast<float*>(v_empty + STAGES);   // [16] pipelined schedule: written, never read (see step)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * Cfg::BM, head = blockIdx.y, b = blockIdx.z;
  const int bk = p.kv_shared ? 0 : b;
  const int ntiles = (p.Nk + BNK - 1) / BNK;
  const float sl2 = p.scale_log2;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmap_q);
    tma_prefetch_desc(&p.tmap_k);
    tma_prefetch_desc(&p.tmap_v);
    mbar_init(q_full, 1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], 4 * Cfg::MMA_WGS);
      if constexpr (Cfg::PIPELINED) { mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], 4 * Cfg::MMA_WGS); }
    }
    fence_barrier_init();
  }
  __syncthreads();

  if constexpr (!Cfg::PIPELINED) {
    if (warp == 8) {
      // ------------------------------ TMA producer ------------------------------
      if (elect_one()) {
        mbar_expect_tx(q_full, Cfg::Q_BYTES);
        tma_load_4d(sQ, &p.tmap_q, q_full, 0, head, q0, b);
      }
      __syncwarp();
      for (int j = 0; j < ntiles; ++j) {
        const int s = j & 1;
        if (j >= 2) mbar_wait(&k_empty[s], ((j >> 1) - 1) & 1);          // tile j-2 fully consumed
        if (elect_one()) {
          mbar_expect_tx(&k_full[s], 2 * Cfg::KV_BYTES);
          tma_load_4d(sK + s * Cfg::KV_BYTES, &p.tmap_k, &k_full[s], 0, head, j * BNK, bk);
          tma_load_4d(sV + s * Cfg::KV_BYTES, &p.tmap_v, &k_full[s], 0, head, j * BNK, bk);
        }
        __syncwarp();
      }
      return;
    }

    // ------------------------------ MMA / softmax warpgroups ------------------------------
    const int cw = warp >> 2, wl = warp & 3;
    const uint32_t aQ = smem_u32(sQ) + cw * (64 * ATT_D * 2);
    float o[32];                                      // O fragments: 64 rows x 64 columns per warpgroup
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // rows r0 and r0 + 8 of this thread (l: this thread's partial sum)
    mbar_wait(q_full, 0);
    for (int j = 0; j < ntiles; ++j) {
      const int s = j & 1;
      const uint32_t aK = smem_u32(sK + s * Cfg::KV_BYTES);
      const uint32_t aV = smem_u32(sV + s * Cfg::KV_BYTES);
      mbar_wait(&k_full[s], (j >> 1) & 1);
      float sc[BNK / 2];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < ATT_D / 16; ++k) Wgmma<BNK>::ss(sc, wgmma_desc_sw128(aQ + 32 * k), wgmma_desc_sw128(aK + 32 * k), k > 0 ? 1 : 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sc);

      float alpha[2];
      float e[BNK / 2];
      uint32_t pa[BNK / 16][4];
      if (p.Nk - j * BNK < BNK) attn_mask<BNK>(sc, p.Nk - j * BNK, lane);
      attn_softmax<BNK>(sc, sl2, m, l, alpha, e);
      attn_pack<BNK>(e, pa);
      attn_rescale(o, alpha);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BNK / 16; ++kk) Wgmma<64, 1>::rs(o, pa[kk], wgmma_desc_sw128(aV + kk * 16 * 128), 1);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      __syncwarp();
      if (lane == 0) mbar_arrive(&k_empty[s]);
    }
    attn_store(p, o, l, q0 + cw * 64, wl, lane, head, b);
  } else {
    if (warp < 4) {
      setmaxnreg_dec<ATT_PRODUCER_REGS>();
      if (warp != 0) return;
      // ------------------------------ TMA producer ------------------------------
      // Order K(0), K(1), V(0), K(2), V(1), ...: the MMA warpgroups issue S(j+1) before PV(j).
      if (elect_one()) {
        mbar_expect_tx(q_full, Cfg::Q_BYTES);
        tma_load_4d(sQ, &p.tmap_q, q_full, 0, head, q0, b);
      }
      __syncwarp();
      int s = 0, vs = 0;
      uint32_t ph = 0, vph = 0;
      for (int j = 0; j <= ntiles; ++j) {
        if (j < ntiles) {
          mbar_wait(&k_empty[s], ph ^ 1);            // a fresh barrier passes the wait on the "previous" phase
          if (elect_one()) {
            mbar_expect_tx(&k_full[s], Cfg::KV_BYTES);
            tma_load_4d(sK + s * Cfg::KV_BYTES, &p.tmap_k, &k_full[s], 0, head, j * BNK, bk);
          }
          __syncwarp();
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
        if (j > 0) {
          mbar_wait(&v_empty[vs], vph ^ 1);
          if (elect_one()) {
            mbar_expect_tx(&v_full[vs], Cfg::KV_BYTES);
            tma_load_4d(sV + vs * Cfg::KV_BYTES, &p.tmap_v, &v_full[vs], 0, head, (j - 1) * BNK, bk);
          }
          __syncwarp();
          if (++vs == STAGES) { vs = 0; vph ^= 1; }
        }
      }
      return;
    }

    // ------------------------------ MMA / softmax warpgroups ------------------------------
    setmaxnreg_inc<ATT_MMA_REGS>();
    const int cw = (warp >> 2) - 1, wl = warp & 3;
    const uint32_t aQ = smem_u32(sQ) + cw * (64 * ATT_D * 2);
    const uint32_t aK0 = smem_u32(sK), aV0 = smem_u32(sV);
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float alpha[2];
    uint32_t pa[BNK / 16][4];                        // P(j): written only while no PV is in flight
    int ks = 0, vs = 0;                              // ring positions of the next K tile to consume / of V(j)
    uint32_t kph = 0, vph = 0;

    // Turn-taking between the MMA warpgroups in the order 0, 1, 2, 0, ... (named barriers ATT_BAR_TURN + cw): a warpgroup
    // waits for its turn before each issue of MMAs and passes the turn to the next one after it.  Every warpgroup issues
    // ntiles + 1 times (every warpgroup runs every tile, also when its rows are all >= Nq), so the last warpgroup opens with
    // one pass to warpgroup 0 and leaves out the pass after its last issue: every barrier sees 128 waiting and 128 arriving
    // threads per generation.
    constexpr int NWG = Cfg::MMA_WGS;
    auto turn_wait = [&]() { named_bar_sync(ATT_BAR_TURN + cw, 256); };
    auto turn_pass = [&](bool last) {
      if (!(last && cw == NWG - 1)) named_bar_arrive(ATT_BAR_TURN + (cw + 1) % NWG, 256);
    };
    auto issue_s = [&](float (&sc)[BNK / 2]) {      // S = Q K^T on K stage ks; one commit group
      mbar_wait(&k_full[ks], kph);
      const uint32_t aK = aK0 + ks * Cfg::KV_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < ATT_D / 16; ++k) Wgmma<BNK>::ss(sc, wgmma_desc_sw128(aQ + 32 * k), wgmma_desc_sw128(aK + 32 * k), k > 0 ? 1 : 0);
      wgmma_commit();
    };
    auto release_k = [&]() {
      __syncwarp();
      if (lane == 0) mbar_arrive(&k_empty[ks]);
      if (++ks == STAGES) { ks = 0; kph ^= 1; }
    };
    auto issue_pv = [&]() {   // O += P V on V stage vs; one commit group
      mbar_wait(&v_full[vs], vph);
      const uint32_t aV = aV0 + vs * Cfg::KV_BYTES;
      wgmma_fence_regs(o);                           // the rescale of O is done before the MMAs start
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BNK / 16; ++kk) Wgmma<64, 1>::rs(o, pa[kk], wgmma_desc_sw128(aV + kk * 16 * 128), 1);
      wgmma_commit();
    };
    auto release_v = [&]() {
      __syncwarp();
      if (lane == 0) mbar_arrive(&v_empty[vs]);
      if (++vs == STAGES) { vs = 0; vph ^= 1; }
    };
    // Tile j < ntiles - 1, P(j) in pa: issue S(j+1) and PV(j), run the softmax of S(j+1) while PV(j) is on the tensor cores,
    // then rescale O and pack P(j+1).  Between the two waits the code has no branch (ptxas would wait for PV(j) at the join)
    // and writes no register PV(j) reads, so a partial tile j+1 is masked in its own instance (partial = true) after PV(j).
    auto step = [&](int j, bool partial) {
      float sc[BNK / 2], e[BNK / 2];
      turn_wait();
      issue_s(sc);
      issue_pv();
      turn_pass(false);
      wgmma_wait<1>();                               // groups retire in issue order: S(j+1) (issued before PV(j)) has retired
      wgmma_fence_regs(sc);
      release_k();
      if (partial) {
        wgmma_wait<0>();                             // PV(j) has retired: no MMA is in flight while the scores are masked
        attn_mask<BNK>(sc, p.Nk - (j + 1) * BNK, lane);
      }
      attn_softmax<BNK>(sc, sl2, m, l, alpha, e);
      // ptxas moves a wgmma wait up to the last instruction it must follow, which would put this wait ahead of the
      // softmax and serialise it with PV(j).  It keeps the wait behind shared-memory stores: a store of the row sums (they
      // depend on every exponential of the tile) holds it after the softmax.
      if (lane == 0) pin[warp] = l[0] + l[1];
      wgmma_wait<0>();                               // PV(j) has retired: O holds P(0..j) V and pa is free
      wgmma_fence_regs(o);
      release_v();
      attn_rescale(o, alpha);                        // alpha(j+1), before PV(j+1) accumulates into O
      attn_pack<BNK>(e, pa);
    };

    mbar_wait(q_full, 0);
    if (cw == NWG - 1) turn_pass(false);
    {
      float sc[BNK / 2], e[BNK / 2];
      turn_wait();
      issue_s(sc);                                   // S(0)
      turn_pass(false);
      wgmma_wait<0>();                               // S(0) has retired (no other group of this warpgroup is in flight)
      wgmma_fence_regs(sc);
      release_k();
      if (p.Nk < BNK) attn_mask<BNK>(sc, p.Nk, lane);
      attn_softmax<BNK>(sc, sl2, m, l, alpha, e);
      attn_rescale(o, alpha);
      attn_pack<BNK>(e, pa);
    }
    const bool partial_last = p.Nk % BNK != 0;
    for (int j = 0; j < ntiles - 2; ++j) step(j, false);
    if (ntiles >= 2) {
      if (partial_last) step(ntiles - 2, true);
      else step(ntiles - 2, false);
    }
    turn_wait();                                     // PV of the last tile
    issue_pv();
    turn_pass(true);
    wgmma_wait<0>();                                 // PV(ntiles - 1), the only group in flight, has retired
    wgmma_fence_regs(o);
    release_v();
    attn_store(p, o, l, q0 + cw * 64, wl, lane, head, b);
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
    uint32_t box[4] = {64, 1, (uint32_t)Cfg::BM, 1};
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
  dim3 grid((d.Nq + Cfg::BM - 1) / Cfg::BM, d.heads, d.B);
  flash_attn_d64_kernel<BNK><<<grid, Cfg::THREADS, Cfg::SMEM, stream>>>(p);
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

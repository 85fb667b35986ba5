// Shared pieces of the tap-GEMM kernel (gemm_tap.cu): parameter block, tile enumeration, the shared-memory output tile and
// the row passes of the epilogue over it (statistics, non-TMA stores, multi-GPU scatter).
#pragma once
#include "common.cuh"

namespace vc {

static constexpr int BM = 128;
static constexpr int BK = 64;
static constexpr int MAX_TAPS = 9;
// one producer warpgroup (TMA) + two MMA warpgroups, each owning whole 128-row tiles (alternate tiles of the CTA's sequence)
static constexpr int MMA_WGS = 2;
static constexpr int GEMM_THREADS = 128 * (1 + MMA_WGS);
// Register split (setmaxnreg): the CTA is launched with 168 registers per thread (65536 / 384, rounded down to a multiple of
// 8); the producer warpgroup hands its share to the MMA warpgroups, whose 2 x BN / 2 accumulators per thread need it.
static constexpr int GEMM_LAUNCH_REGS = 168;
static constexpr int GEMM_PRODUCER_REGS = 24;
static constexpr int GEMM_MMA_REGS = 240;
static_assert(128 * GEMM_PRODUCER_REGS + 128 * MMA_WGS * GEMM_MMA_REGS <= GEMM_LAUNCH_REGS * GEMM_THREADS, "register split exceeds the CTA's allocation");
// Output tile of an MMA warpgroup: 128 rows x BN fp16 columns in shared memory, one 8 KB block per 32-column chunk, each
// block 128 rows of 64 bytes with the 64B swizzle (16-byte unit u of row R stored at unit u ^ ((R >> 1) & 3)).  Rows 32 q ..
// 32 q + 31 of a chunk form the 2 KB box the TMA stores write (tmap_out, peer maps); a whole 8 KB block is the box of a
// residual load (tmap_res).
static constexpr int EPI_CHUNK_BYTES = BM * 32 * 2;
static constexpr int EPI_SUB_BYTES = 32 * 32 * 2;
__host__ __device__ constexpr uint32_t epi_offset(int row, int col) {   // byte offset of element (row, col) in the output tile
  return (uint32_t)((col >> 5) * EPI_CHUNK_BYTES + row * 64 + ((((col & 31) >> 3) ^ ((row >> 1) & 3)) << 4) + (col & 7) * 2);
}

// Division by a runtime constant as multiply-high + shift (valid for dividends < 2^31): the persistent kernels turn a
// linear tile index into (n-tile, x, y, z) once per tile in EVERY thread, and a generic 32-bit division is ~20 SASS
// instructions each.
struct FastDiv {
  uint32_t mul, shr, d;
};
static inline FastDiv make_fastdiv(int d) {
  FastDiv f;
  f.d = (uint32_t)d;
  if (d == 1) { f.mul = 0; f.shr = 0; return f; }
  uint32_t lg = 0;
  while ((1u << lg) < (uint32_t)d) ++lg;           // ceil(log2 d)
  const uint32_t p = 31 + lg;
  f.mul = (uint32_t)(((1ull << p) + (uint32_t)d - 1) / (uint32_t)d);
  f.shr = p - 32;
  return f;
}
#ifdef __CUDACC__
__device__ __forceinline__ int fast_div(const FastDiv& f, int n) { return f.d == 1 ? n : (int)(__umulhi((uint32_t)n, f.mul) >> f.shr); }
#endif

// Multi-GPU layout switch fused into the epilogue (frame-sharded U-Net, parallel.py): instead of writing its output locally and
// handing it to a separate exchange kernel, the GEMM that PRODUCES a tensor stores every 32-row x 32-column tile straight into the
// receive buffer of the rank that owns those rows in the other layout -- TMA stores through the NVLink peer mapping, issued tile by
// tile while the MMAs of the following tiles run.  mode 1: this rank's rows are (b, t_local, hw) ["frames"], destination
// (b, t_all, hw_local) on rank hw / HWl ["sites"]; mode 2 the reverse.  Destination tensor maps are 3-D (C, HWl, b*t) with a
// (32, 32, 1) box: a 32-row patch that runs past the end of a rank's hw range (or of a frame) is written as one clipped store per
// segment -- every segment starts or ends on a range boundary, so the rows outside it fall outside the map and are dropped.
static constexpr int GEMM_PEER_MAX = 4;
struct GemmPeer {
  int mode;              // 0: off
  int P, me;
  int wrap;              // producer rows form ONE slab-major matrix (Y == 1, Z == 1): the slab index is row / rps
  int HW, HWl, T, Tl_me;
  int rps;               // producer rows per slab (mode 1: HW, slab = b * Tl_me + t_local; mode 2: T * HWl, slab = b)
  FastDiv div_hwl, div_rps, div_tl;
  int f0[GEMM_PEER_MAX + 1];
  CUtensorMap map[GEMM_PEER_MAX];
};

struct GemmParams {
  CUtensorMap tmap_a;
  CUtensorMap tmap_a2;
  CUtensorMap tmap_b;
  CUtensorMap tmap_out;  // fp16 output as (N, X, Y, Z), box (32, min(bx,32), 32/min(bx,32), 1), 64B swizzle (out_tma only)
  CUtensorMap tmap_res;  // residual as (N, X, Y, Z), box (32, bx, by, 1), 64B swizzle (res_tma only)
  int tiles_x, tiles_y, Z;
  FastDiv div_tiles_x, div_tiles_y, div_n_tiles;
  int bx, by;
  int bx_shift;          // bx is a power of two (bx * by == 128)
  int X, Y;
  int N, K, K1;          // K1 = channels served by tmap_a (K1 == K when single source)
  int num_taps;
  int tap_dx[MAX_TAPS];
  int tap_dy[MAX_TAPS];
  int n_tiles;
  int total_tiles;       // m_tiles * n_tiles
  __half* out;
  float* out_f32;
  int ldo;
  const float* bias;
  int bias_z_div;
  const __half* res;
  int ldr;
  int geglu;
  const float* ln_stats;   // folded LayerNorm: per-row (mean, rstd); nullptr = plain
  const float* ln_colsum;  // folded LayerNorm: per-column sum of the (gamma-scaled) weights
  float2* ln_part;         // optional: per (32-column chunk, row) (sum, M2 about the chunk mean) of the fp16-rounded outputs, [N/32][ln_rows]:
  long long ln_rows;       //   the LayerNorm statistics of the tensor this GEMM writes, gathered while it is still in registers
  float2* gn_part;         // optional: GroupNorm partial (sum, sumsq) of the fp16-rounded outputs per (32-row block, 32-column chunk, piece):
  int gn_hp;               //   [m_tile * 4 + quadrant][N / 32][4]; a chunk is cut at the boundaries of gn_sub = 2 * gn_hp channel sub-groups
  int gn_nchunks;          //   (4 pieces: first partial, two whole, last partial / whole) -- see gn_part_accumulate and norm.cu: gn_part_finalize_kernel
  int out_tma;           // fp16 output written by TMA stores from the warpgroup's output tile (full-line, LSU-free)
  int vec_ok;            // output rows are 32-byte aligned: a non-TMA output is stored as 256-bit (fp16) / 64-bit (fp32) vectors
  int res_tma;           // residual 16-byte aligned with a 16-byte row pitch: loaded by TMA into the output tile while the MMAs run
  GemmPeer peer;         // output scattered to the ranks of the frame group (mode != 0: `out` itself is not written)
  // FP8 mode (gemm_tap_kernel<BN, true>): e4m3 weights, A converted to e4m3 in registers with the per-tensor scale
  // s_a = a_amax / 448; the epilogue starts from acc * (s_a * w_scale[n])
  const float* w_scale;  // [N] per-output-channel weight scales
  const float* a_amax;   // device scalar: max |A| over everything the GEMM reads (absmax_f16)
};

struct TileCoord {
  int x0, y0, z;
};

// m-tile index -> tile origin
#ifdef __CUDACC__
__device__ __forceinline__ TileCoord tile_coord_m(const GemmParams& p, int m) {
  TileCoord t;
  const int q1 = fast_div(p.div_tiles_x, m);
  const int tx = m - q1 * p.tiles_x;
  t.z = fast_div(p.div_tiles_y, q1);
  const int ty = q1 - t.z * p.tiles_y;
  t.x0 = tx << p.bx_shift;
  t.y0 = ty * p.by;
  return t;
}
#endif

#ifdef __CUDACC__
// exact-erf GELU (attention.py:415-422 uses F.gelu), erf by Abramowitz-Stegun 7.1.26 (|err| < 1.5e-7): 2 MUFU + ~12 FMA/ALU
__device__ __forceinline__ float gelu_epilogue(float x) {
  const float z = x * 0.70710678118654752440f;
  const float az = fabsf(z);
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, az, 1.0f)));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(az * az * -1.4426950408889634f));
  const float erf_abs = fmaf(-poly * t, e, 1.0f);
  const float hx = 0.5f * x;
  return fmaf(hx, copysignf(erf_abs, z), hx);
}

// ---------------------------------------------------------------------------------------------------------------
// Row passes over the fp16 output tile (statistics, non-TMA stores): one thread owns one output row and the 32 columns of a
// chunk, a warp owns 32 consecutive rows of the tile: quad = 32-row block of the 128-row tile.
// ---------------------------------------------------------------------------------------------------------------
struct EpiTile {
  long long orow;        // output row index of this thread
  int n_tile;
  int m_tile;            // linear m-tile index (x fastest, then y, then z)
  int quad;              // 32-row block of the tile owned by this warp
  int wx, wy, wz;        // (x, y, z) of the warp's first row: TMA store coordinates
  bool row_ok;
};

__device__ __forceinline__ EpiTile epi_tile(const GemmParams& p, int tile, int quad, int lane) {
  EpiTile t;
  const int mq = fast_div(p.div_n_tiles, tile);
  t.n_tile = tile - mq * p.n_tiles;
  t.m_tile = mq;
  t.quad = quad;
  const TileCoord tc = tile_coord_m(p, t.m_tile);
  const int R = quad * 32 + lane;                // tile row owned by this thread
  const int R0 = quad * 32;
  t.wx = tc.x0 + (R0 & (p.bx - 1)); t.wy = tc.y0 + (R0 >> p.bx_shift); t.wz = tc.z;
  const int x = tc.x0 + (R & (p.bx - 1)), y = tc.y0 + (R >> p.bx_shift);
  t.row_ok = x < p.X && y < p.Y && tc.z < p.Z;
  t.orow = ((long long)tc.z * p.Y + y) * p.X + x;
  return t;
}

// peer mode: the warp's 32 x 32 box of the output tile goes to the rank(s) owning its rows in the other layout (executed by one lane)
__device__ __forceinline__ void peer_scatter32(const GemmParams& p, const EpiTile& t, int col0, const uint8_t* stage) {
  const GemmPeer& g = p.peer;
  int lin = t.wy * p.X + t.wx;                 // first row of the warp's patch inside its z-slab (patches are row-contiguous: host check)
  int slab = t.wz;
  if (g.wrap) { slab = fast_div(g.div_rps, lin); lin -= slab * g.rps; }
  int rem = 32, i0 = 0;
  while (rem > 0) {
    if (lin >= g.rps) {
      if (!g.wrap) break;                      // rows past the slab are tile padding
      lin -= g.rps; ++slab;
    }
    int q, s, c2;
    if (g.mode == 1) {
      q = fast_div(g.div_hwl, lin); s = lin - q * g.HWl;
      const int b = fast_div(g.div_tl, slab);
      c2 = b * g.T + g.f0[g.me] + (slab - b * g.Tl_me);
    } else {
      const int tt = fast_div(g.div_hwl, lin); s = lin - tt * g.HWl;
      q = 0;
      while (q + 1 < g.P && tt >= g.f0[q + 1]) ++q;
      c2 = slab * (g.f0[q + 1] - g.f0[q]) + tt - g.f0[q];
    }
    const int len = min(rem, g.HWl - s);
    if (q < g.P) tma_store_3d(&g.map[q], stage, col0, s - i0, c2);
    i0 += len; lin += len; rem -= len;
  }
}

// the 32 fp16 values of this thread's row in one chunk of the output tile (row_addr: shared address of the row), in column order
__device__ __forceinline__ void epi_row_load(uint32_t row_addr, int row, uint4 (&u)[4]) {
  const int sw = (row >> 1) & 3;
#pragma unroll
  for (int h = 0; h < 4; ++h)
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(u[h].x), "=r"(u[h].y), "=r"(u[h].z), "=r"(u[h].w) : "r"(row_addr + ((h ^ sw) << 4)));
}

// fp16 output that the TMA store cannot write (unaligned pointer or pitch, ragged N): this thread's row of one chunk, copied
// from the output tile as 256-bit vectors, or by predicated scalar stores at a ragged N tail / unaligned pitch (the 320->4
// output conv).  The values were rounded once in the tile, so the output does not depend on the store path.
__device__ __forceinline__ void epi_store_row32(const GemmParams& p, const EpiTile& t, int col0, int n_out, const uint4 (&u)[4]) {
  if (!t.row_ok || col0 >= n_out) return;
  if (col0 + 32 <= n_out && p.vec_ok) {
    uint4* op = reinterpret_cast<uint4*>(p.out + t.orow * p.ldo + col0);
#pragma unroll
    for (int h = 0; h < 4; ++h) op[h] = u[h];
  } else {
    const __half* hv = reinterpret_cast<const __half*>(u);
#pragma unroll
    for (int e = 0; e < 32; ++e)
      if (col0 + e < n_out) p.out[t.orow * p.ldo + col0 + e] = hv[e];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// GroupNorm statistics of the tensor a GEMM is writing (GemmParams::gn_part), so that the consuming GroupNorm is ONE pass over
// the activation (read + write once) instead of statistics pass + normalise pass.  GroupNorm(32) groups are C/32 channels wide
// (10 / 20 / 40 in the U-Net, 30 / 60 / 80 for the skip concats) and do not line up with the 32-column chunks a thread owns,
// so each chunk is cut into 4 pieces at the boundaries of `sub`-channel sub-groups (sub = 10: every group boundary of every
// consumer is a multiple of 10; sub = 8 for power-of-two widths): with o = (first column) mod sub, the pieces are
// [0, sub-o), [sub-o, 2 sub-o), [2 sub-o, 3 sub-o), [3 sub-o, 32) -- always exactly four for sub in {8, 10}.  A thread owns one
// row: it sums its fp16-rounded values (what the consumer will read) per piece, the warp reduces the 8 numbers over its 32 rows
// with a recursive-halving exchange (9 shuffles; fixed order -> bit-reproducible) and 8 lanes store them.
// B1 = pairs in the first piece, HP = pairs per sub-group.
template <int B1, int HP>
__device__ __forceinline__ void gn_piece_sums(const float (&f)[32], bool row_ok, float (&v)[8]) {
  float s[4], q[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) s[i] = q[i] = 0.f;
#pragma unroll
  for (int e = 0; e < 16; ++e) {
    const int piece = e < B1 ? 0 : e < B1 + HP ? 1 : e < B1 + 2 * HP ? 2 : 3;
    const float2 r = __half22float2(__floats2half2_rn(f[2 * e], f[2 * e + 1]));
    s[piece] += r.x + r.y;
    q[piece] = fmaf(r.x, r.x, fmaf(r.y, r.y, q[piece]));
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[i] = row_ok ? s[i] : 0.f;
    v[4 + i] = row_ok ? q[i] : 0.f;
  }
}
__device__ __forceinline__ void gn_part_accumulate(const GemmParams& p, const EpiTile& t, int nb, const float (&f)[32], int lane) {
  float v[8];
  const int sub = 2 * p.gn_hp;
  const int o = nb % sub;                               // even: nb is a multiple of 32, sub is even
  if (p.gn_hp == 5) {
    switch (o) {
      case 0: gn_piece_sums<5, 5>(f, t.row_ok, v); break;
      case 2: gn_piece_sums<4, 5>(f, t.row_ok, v); break;
      case 4: gn_piece_sums<3, 5>(f, t.row_ok, v); break;
      case 6: gn_piece_sums<2, 5>(f, t.row_ok, v); break;
      default: gn_piece_sums<1, 5>(f, t.row_ok, v); break;
    }
  } else {
    gn_piece_sums<4, 4>(f, t.row_ok, v);                // sub = 8 divides 32: o == 0 always
  }
  // recursive halving over the 32 lanes (rows): 8 -> 4 -> 2 -> 1 values per lane, then a two-step butterfly
  {
    const bool hi = lane & 16;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float send = hi ? v[i] : v[i + 4], keep = hi ? v[i + 4] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
  }
  {
    const bool hi = lane & 8;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float send = hi ? v[i] : v[i + 2], keep = hi ? v[i + 2] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
  }
  {
    const bool hi = lane & 4;
    const float send = hi ? v[0] : v[1], keep = hi ? v[1] : v[0];
    v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  v[0] += __shfl_xor_sync(0xffffffffu, v[0], 2);
  v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
  // lane bits (4, 3, 2) select which of the 8 numbers this lane ended up with: idx = 4*b4 + 2*b3 + b2  (0..3 sums, 4..7 sums of squares)
  if ((lane & 3) == 0) {
    const int idx = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
    const long long rb = (long long)t.m_tile * 4 + t.quad;
    float* dst = reinterpret_cast<float*>(p.gn_part + (rb * p.gn_nchunks + (nb >> 5)) * 4);
    dst[(idx & 3) * 2 + (idx >> 2)] = v[0];
  }
}

// LayerNorm / GroupNorm statistics of this thread's row of one 32-column chunk (nb: its first column), from the fp16 values
// the output holds (u: epi_row_load)
__device__ __forceinline__ void epi_stats_row32(const GemmParams& p, const EpiTile& t, int nb, const uint4 (&u)[4], int lane) {
  float f[32];
  const __half2* h2 = reinterpret_cast<const __half2*>(u);
#pragma unroll
  for (int e = 0; e < 16; ++e) {
    const float2 r = __half22float2(h2[e]);
    f[2 * e] = r.x; f[2 * e + 1] = r.y;
  }
  if (p.ln_part) {                                 // LayerNorm statistics of the OUTPUT row, as stored (fp16-rounded)
    // (sum, M2): M2 is taken about the chunk's own mean, so it does not cancel when the row's |mean| >> std
    float s = 0.f;
#pragma unroll
    for (int e = 0; e < 32; e += 2) s += f[e] + f[e + 1];
    const float m = s * (1.f / 32.f);
    float q = 0.f;
#pragma unroll
    for (int e = 0; e < 32; e += 2) {
      const float a = f[e] - m, b = f[e + 1] - m;
      q = fmaf(a, a, fmaf(b, b, q));
    }
    if (t.row_ok) p.ln_part[(long long)(nb >> 5) * p.ln_rows + t.orow] = make_float2(s, q);
  }
  if (p.gn_part) gn_part_accumulate(p, t, nb, f, lane);
}
#endif  // __CUDACC__

}  // namespace vc

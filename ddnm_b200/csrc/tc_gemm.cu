// wgmma implicit-GEMM convolution for sm_90a.
//
//   out[pixel, co] = alpha * sum_k A[pixel, k] * Wt[co, k] + chanadd[image, co] + residual[pixel, co]
//
// A is never materialised: for k-block (tap, 64-channel slice) the TMA engine copies the shifted NHWC window
// [bn images x bh rows x bw cols] x 64 channels straight into 128B-swizzled shared memory; halo / padding pixels
// come from TMA out-of-bounds zero fill (no im2col, no padded copy).  Products are "fp32-grade": every fp32
// operand is pre-split into fp16 hi + lo and each k-slice issues hi*hi + hi*lo + lo*hi into one fp32 register
// accumulator (the dropped lo*lo term is ~2^-22 relative).
//
// Replaces, on the reference path, every torch.nn.Conv2d / 1x1 conv / bmm inside
//   guided_diffusion/models.py:77-189 (ResnetBlock, AttnBlock), :36-74 (Up/Downsample)
// which the reference dispatches to cuDNN / cuBLAS.
//
// CTA = 9 warps: warps 0-7 are two consumer warpgroups (wgmma m64 x BN over rows 0-63 / 64-127 of the 128-pixel tile, then the
// epilogue straight from the accumulator registers), warp 8 is the TMA producer.  Persistent over output tiles; the producer runs
// ahead across tile boundaries, so the next tile's operands are in flight while the consumers run the epilogue.
// Two orthogonal forms, chosen per layer in tc_make_launch:
//   DUAL: the B_hi and B_lo planes of a stage are adjacent in shared memory, so ONE descriptor spans both and A_hi x [B_hi; B_lo] is
//         a single m64 x 2BN instruction (accumulator columns [0, BN) = hi*hi, [BN, 2BN) = hi*lo); A_lo x B_hi follows with N = BN
//         into the first half, and the epilogue adds the halves: two instructions and one read of the A_hi rows per k-step
//         instead of three and two.
//   HALO: 3x3 stride-1 and upsample-phase (2x2) launches whose tile rows are 64-pixel runs of image rows (bw % 64 == 0, one image
//         per tile).  The three column taps dx of a (dy, 64-channel slice) read the same image rows shifted by one pixel, so the
//         producer loads them once, as a halo unit of (bw + 2) x bh pixels (bw + 1 for the upsample phases) in hi + lo, and the
//         K order becomes (dy, slice, dx).  Each dx k-block reads the unit through a descriptor whose start is shifted by 128 B
//         per pixel; wgmma applies the 128B swizzle to absolute shared-memory address bits, as TMA does when it writes the
//         1024 B-aligned unit, so the shifted start needs no base offset (the same rule that lets the K advance add 32 B).  The
//         A units have a ring of their own (HALO_UNITS, own full / empty barriers) next to a ring of 4 B stages; a unit goes back to
//         the producer once the wgmma group of its last dx k-block has completed.  Launches with a 1x1 side input keep the per-tap
//         form (see tc_make_launch).
// conv_tc_pingpong_kernel (below) runs the launches where CTAs walk several tiles: each consumer warpgroup owns a whole tile, and
// the two take turns on the tensor cores so one tile's epilogue overlaps the next tile's MMAs.  Its launches with one weight matrix
// run on clusters of two CTAs that share every weight k-block through TMA multicast (its PAIR form).
#include "tc_gemm.cuh"

#include <cstdlib>

#include "kernels.cuh"

namespace ddnm {

static constexpr int BM = 128;
static constexpr int kConsumerThreads = 256;
static constexpr int kTcThreads = kConsumerThreads + 32;
static constexpr int BK = 64;                      // fp16 elements = 128 bytes = one swizzle row
static constexpr int A_PLANE_BYTES = BM * BK * 2;  // 16 KiB

// HALO form: one A plane of a unit holds the halo rows of a tile, (bw + 2) x bh pixels of 128 B (at most 132 rows), 1024 B-aligned.
// 2 units + 4 B stages: one unit feeds 3 (2) k-blocks, so the A ring still runs as far ahead as the B ring; celeba forward (B = 16,
// CUDA graph) on an H100 SXM at 700 W: 58.2 ms, against 58.9 with 3 units + 3 B stages and 61.4 for the per-tap form.
static constexpr int HALO_PLANE_BYTES = 17 * 1024;
static constexpr int HALO_UNITS = 2;

template <int BN, bool DUAL, bool HALO = false>
struct TcCfg {
  static constexpr int B_PLANE_BYTES = BN * BK * 2;
  // without HALO one stage is {A_hi, A_lo, B_hi, B_lo}; with HALO the A units have their own ring in front of the B stages
  static constexpr int A_UNIT_BYTES = 2 * HALO_PLANE_BYTES;
  static constexpr int A_RING_BYTES = HALO ? HALO_UNITS * A_UNIT_BYTES : 0;
  static constexpr int STAGE_BYTES = (HALO ? 0 : 2 * A_PLANE_BYTES) + 2 * B_PLANE_BYTES;
  static constexpr int STAGES = (HALO || BN == 64) ? 4 : 3;
  static constexpr int RING_BYTES = A_RING_BYTES + STAGES * STAGE_BYTES;
  // GroupNorm sums of a tile: per-warp column partials (8 warps x BN x {sum, sumsq}) and the running (value, compensation) pairs
  // of up to 4 images per tile x {sum, sumsq} x BN columns
  static constexpr int PART_BYTES = 8 * BN * 8;
  static constexpr int RUN_BYTES = 4 * 2 * BN * 8;
  static constexpr int SMEM_BYTES = RING_BYTES + 1024 /*align slack*/ + 256 /*barriers*/ + PART_BYTES + RUN_BYTES;
  static constexpr int ACC = DUAL ? BN : BN / 2;     // fp32 accumulator registers per consumer thread (m64 x BN(x2) / 128 threads)
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory capacity");
};

// D[64 x N] (+)= A x B on the first N / 2 accumulator registers of d (the fragment of an m64 x N tile is a prefix of the one of a
// wider tile, so the DUAL form's A_lo x B_hi accumulates into the hi*hi half of the m64 x 2BN accumulator)
template <int N, int R>
__device__ __forceinline__ void wgmma_tile(float (&d)[R], uint64_t a, uint64_t b, uint32_t accumulate) {
  static_assert(N / 2 <= R, "accumulator too small");
  if constexpr (N == 64) wgmma_m64n64k16(*reinterpret_cast<float(*)[32]>(&d[0]), a, b, accumulate);
  else if constexpr (N == 128) wgmma_m64n128k16(*reinterpret_cast<float(*)[64]>(&d[0]), a, b, accumulate);
  else wgmma_m64n256k16(*reinterpret_cast<float(*)[128]>(&d[0]), a, b, accumulate);
}

// output tile -> (N tile, first column, first row, first image of the M tile)
__device__ __forceinline__ void tc_decode(const TcParams& p, int tile, int& n_idx, int& x0, int& y0, int& n0) {
  n_idx = tile % p.n_tiles;
  const int m = tile / p.n_tiles;
  const int tx = m % p.tiles_x;
  const int t2 = m / p.tiles_x;
  const int ty = t2 % p.tiles_y;
  const int tn = t2 / p.tiles_y;
  x0 = tx * p.bw;
  y0 = ty * p.bh;
  n0 = tn * p.bn;
}

// Barriers behind the ring: full / empty per B stage, then (HALO) full / empty per A unit, then the ping-pong kernel's MMA turns
template <int STAGES>
struct TcBars {
  uint32_t base;
  __device__ uint32_t full(int s) const { return base + 8u * s; }
  __device__ uint32_t empty(int s) const { return base + 8u * (STAGES + s); }
  __device__ uint32_t a_full(int u) const { return base + 8u * (2 * STAGES + u); }
  __device__ uint32_t a_empty(int u) const { return base + 8u * (2 * STAGES + HALO_UNITS + u); }
  __device__ uint32_t turn(int w) const { return base + 8u * (2 * STAGES + 2 * HALO_UNITS + w); }
};

// The TMA producer's position in the B-stage ring and (HALO) in the A-unit ring
struct TcRing {
  uint32_t stage = 0, phase = 0;
  uint32_t aunit = 0, aphase = 0;
};

// TMA loads of the k-blocks [kb_lo, kb_hi) of one output tile, issued by one thread: per k-block the B planes into the next stage
// and the A operand — the tap-shifted window (3x3, stride-2 phase, upsample phase), the 1x1 side input, or (HALO) one halo unit
// per (dy, channel slice) at its first dx k-block.  PAIR (the ping-pong CTA pairs): this CTA's half of the B tile, multicast into
// both CTAs of the cluster.  load_a == false (PAIR only, a ghost step): the B halves alone, in the k order of `tile`, for a peer CTA
// that has one unit more than this one.
template <class Cfg, bool PAIR, bool HALO>
__device__ __forceinline__ void tc_produce_tile(const CUtensorMap* tm_a0h, const CUtensorMap* tm_a0l, const CUtensorMap* tm_a1h,
                                                const CUtensorMap* tm_a1l, const CUtensorMap* tm_bh, const CUtensorMap* tm_bl,
                                                const TcParams& p, uint32_t smem_base, TcBars<Cfg::STAGES> bars, int tile, int kb_lo,
                                                int kb_hi, uint32_t rank, TcRing& r, bool load_a = true) {
  const int halo_r = p.mode0 == TAPS_UP2X2 ? 2 : 3;
  const int halo_w = p.bw + halo_r - 1;
  const bool lo = p.terms != 1;
  const uint32_t planes = lo ? 2u : 1u;
  // HALO: only the B planes arrive with a stage
  const uint32_t stage_tx = (HALO || !load_a) ? planes * Cfg::B_PLANE_BYTES : (uint32_t)(lo ? Cfg::STAGE_BYTES : Cfg::STAGE_BYTES / 2);
  int n_idx, x0, y0, n0;
  tc_decode(p, tile, n_idx, x0, y0, n0);
  const int bz = p.b_batched == 1 ? n0 : 0;
  for (int kb = kb_lo; kb < kb_hi; ++kb) {
    int bkb = kb;   // the weights' k-block (tap-major, see tc_make_launch)
    if constexpr (HALO) {
      // k order (dy, slice, dx); a new A unit at dx == 0
      const int ua = kb / halo_r, dx = kb - ua * halo_r, dy = ua / p.cb0, cs = ua - dy * p.cb0;
      bkb = (dy * halo_r + dx) * p.cb0 + cs;
      if (dx == 0 && load_a) {
        mbar_wait(bars.a_empty(r.aunit), r.aphase ^ 1u);
        const uint32_t ua_s = smem_base + r.aunit * Cfg::A_UNIT_BYTES;
        const uint32_t fa = bars.a_full(r.aunit);
        // halo rows y0 + dy - 1 (+ the phase row), columns from x0 - 1 (+ the phase column); borders are TMA zero fill
        const int cy = y0 + dy - 1 + p.up_py, cx = x0 - 1 + p.up_px;
        mbar_expect_tx(fa, planes * (uint32_t)(halo_w * p.bh * 128));
        tma_load_4d(ua_s, tm_a0h, fa, cs * BK, cx, cy, n0);
        if (lo) tma_load_4d(ua_s + HALO_PLANE_BYTES, tm_a0l, fa, cs * BK, cx, cy, n0);
      }
      if (dx == halo_r - 1) {
        if (++r.aunit == HALO_UNITS) {
          r.aunit = 0;
          r.aphase ^= 1u;
        }
      }
    }
    mbar_wait(bars.empty(r.stage), r.phase ^ 1u);
    const uint32_t sa = smem_base + Cfg::A_RING_BYTES + r.stage * Cfg::STAGE_BYTES;
    const uint32_t sb = HALO ? sa : sa + 2 * A_PLANE_BYTES;
    const uint32_t fb = bars.full(r.stage);
    mbar_expect_tx(fb, stage_tx);
    if (HALO || !load_a) {
    } else if (kb < p.kb0) {
      const int tap = kb / p.cb0;
      const int c = (kb - tap * p.cb0) * BK;
      int cx = x0, cy = y0, cn = n0;
      if (p.mode0 == TAPS_3X3) {
        cy += tap / 3 - 1;
        cx += tap % 3 - 1;
      } else if (p.mode0 == TAPS_UP2X2) {
        cy += tap / 2 + p.up_py - 1;
        cx += tap % 2 + p.up_px - 1;
      } else if (p.mode0 == TAPS_3X3_S2) {
        const int dy = tap / 3, dx = tap % 3;
        cy += dy >> 1;
        cx += dx >> 1;
        cn += ((dy & 1) * 2 + (dx & 1)) * p.phase_stride;
      }
      tma_load_4d(sa, tm_a0h, fb, c, cx, cy, cn);
      if (lo) tma_load_4d(sa + A_PLANE_BYTES, tm_a0l, fb, c, cx, cy, cn);
    } else {
      const int c = (kb - p.kb0) * BK;
      tma_load_4d(sa, tm_a1h, fb, c, x0, y0, n0);
      if (lo) tma_load_4d(sa + A_PLANE_BYTES, tm_a1l, fb, c, x0, y0, n0);
    }
    if (PAIR) {
      // rows [rank * BN / 2, (rank + 1) * BN / 2) of the B tile, into both CTAs (each expects the whole stage)
      constexpr int BN = Cfg::B_PLANE_BYTES / (BK * 2);
      const uint32_t half = rank * (BN / 2) * 128u;
      const int brow = n_idx * BN + (int)rank * (BN / 2);
      tma_load_3d_multicast(sb + half, tm_bh, fb, bkb * BK, brow, 0, (uint16_t)3);
      if (lo) tma_load_3d_multicast(sb + Cfg::B_PLANE_BYTES + half, tm_bl, fb, bkb * BK, brow, 0, (uint16_t)3);
    } else if (p.b_batched == 2) {
      constexpr int BN = Cfg::B_PLANE_BYTES / (BK * 2);
      tma_load_4d(sb, tm_bh, fb, kb * BK, n_idx * BN, y0, n0);
      if (lo) tma_load_4d(sb + Cfg::B_PLANE_BYTES, tm_bl, fb, kb * BK, n_idx * BN, y0, n0);
    } else {
      constexpr int BN = Cfg::B_PLANE_BYTES / (BK * 2);
      tma_load_3d(sb, tm_bh, fb, bkb * BK, n_idx * BN, bz);
      if (lo) tma_load_3d(sb + Cfg::B_PLANE_BYTES, tm_bl, fb, bkb * BK, n_idx * BN, bz);
    }
    if (++r.stage == Cfg::STAGES) {
      r.stage = 0;
      r.phase ^= 1u;
    }
  }
}

// Epilogue of one m64 accumulator fragment: rows r0 and r0 + 8 of the output tile, 2 adjacent columns per 8-column group.
// out = alpha * acc + chanadd + residual (res_mode 0 / 1 / 2), or alpha * acc into split-K partial `split_off`.  The stored values
// (0 for rows past the batch) are written back to d for the GroupNorm sums.  DUAL (dual set): the hi*lo partial sums of the same
// columns are kept BN columns further on and added first.  NTAIL (batched GEMMs whose N is not a multiple of BN): columns at or past
// p.Cout are not stored — in the attention output they belong to the next head.
template <int BN, bool DUAL, bool NTAIL, int R>
__device__ __forceinline__ void tc_epilogue_rows(const TcParams& p, float (&d)[R], bool dual, int r0, int cq, int n_idx, int x0,
                                                 int y0, int n0, int split_off) {
  const int ppi = p.bw * p.bh;
  float* orow[2];
  const float* rrow[2];
  const float* crow[2];
  bool valid[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + 8 * h;
    const int xi = r % p.bw, yi = (r / p.bw) % p.bh, ni = r / ppi;
    const int n = n0 + ni;
    valid[h] = n < p.N;
    orow[h] = p.out + (long long)n * p.out_sn + (long long)(y0 + yi) * p.out_sy + (long long)(x0 + xi) * p.out_sx + n_idx * BN +
              (long long)split_off * p.split_stride;
    rrow[h] = nullptr;
    if (p.residual) {
      // same pixel, nearest-upsampled (x_upd of ResBlock(up=True), unet.py:240) or the 2x2 average of a twice-as-large map
      // (ResBlock(down=True))
      long long rp;
      if (p.res_mode == 0) rp = ((long long)n * p.H + (y0 + yi)) * p.W + (x0 + xi);
      else if (p.res_mode == 1) rp = ((long long)n * (p.H >> 1) + ((y0 + yi) >> 1)) * (p.W >> 1) + ((x0 + xi) >> 1);
      else rp = ((long long)n * (2 * p.H) + 2 * (y0 + yi)) * (2 * p.W) + 2 * (x0 + xi);
      rrow[h] = p.residual + rp * p.ldr + n_idx * BN;
    }
    crow[h] = p.chanadd ? p.chanadd + (long long)n * p.ca_ld + n_idx * BN : nullptr;
  }
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int c = 8 * j + cq;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float a0 = d[4 * j + 2 * h], a1 = d[4 * j + 2 * h + 1];
      if constexpr (DUAL) {
        if (dual) {   // + the hi*lo partial sums of the same columns, kept BN columns further on
          a0 += d[4 * (j + BN / 8) + 2 * h];
          a1 += d[4 * (j + BN / 8) + 2 * h + 1];
        }
      }
      float v0 = p.alpha * a0, v1 = p.alpha * a1;
      if (crow[h] && valid[h]) {
        const float2 cv = __ldg(reinterpret_cast<const float2*>(crow[h] + c));
        v0 += cv.x;
        v1 += cv.y;
      }
      if (rrow[h] && valid[h]) {
        float2 rv = __ldg(reinterpret_cast<const float2*>(rrow[h] + c));
        if (p.res_mode == 2) {
          const long long r_dx = p.ldr, r_dy = (long long)2 * p.W * p.ldr;
          const float2 q1 = __ldg(reinterpret_cast<const float2*>(rrow[h] + r_dx + c));
          const float2 q2 = __ldg(reinterpret_cast<const float2*>(rrow[h] + r_dy + c));
          const float2 q3 = __ldg(reinterpret_cast<const float2*>(rrow[h] + r_dy + r_dx + c));
          rv.x = ((rv.x + q1.x) + (q2.x + q3.x)) * 0.25f;
          rv.y = ((rv.y + q1.y) + (q2.y + q3.y)) * 0.25f;
        }
        v0 += rv.x;
        v1 += rv.y;
      }
      if (!valid[h]) v0 = v1 = 0.f;
      d[4 * j + 2 * h] = v0;
      d[4 * j + 2 * h + 1] = v1;
      if (valid[h] && (!NTAIL || n_idx * BN + c < p.Cout)) *reinterpret_cast<float2*>(orow[h] + c) = make_float2(v0, v1);
    }
  }
}

// GroupNorm sums, step 1: the column sums and sums of squares of one warp's 16 rows of a fragment (after tc_epilogue_rows), reduced
// across the 8 lanes that share a column pair, into part[BN] of that 16-row group
template <int BN, int R>
__device__ __forceinline__ void tc_stats_rows(const float (&d)[R], float2* part, int lane, int cq) {
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const float a = d[4 * j + e], b = d[4 * j + 2 + e];
      float s = a + b, q = a * a + b * b;
#pragma unroll
      for (int k = 4; k <= 16; k <<= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, k);
        q += __shfl_xor_sync(0xffffffffu, q, k);
      }
      if (lane < 4) part[8 * j + cq + e] = make_float2(s, q);
    }
  }
}

template <int BN, bool DUAL, bool HALO, bool NTAIL>
__global__ void __launch_bounds__(kTcThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tm_a0h, const __grid_constant__ CUtensorMap tm_a0l,
               const __grid_constant__ CUtensorMap tm_a1h, const __grid_constant__ CUtensorMap tm_a1l,
               const __grid_constant__ CUtensorMap tm_bh, const __grid_constant__ CUtensorMap tm_bl, const TcParams p) {
  using Cfg = TcCfg<BN, DUAL, HALO>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + Cfg::RING_BYTES;
  const TcBars<STAGES> bars{bar_base};
  auto full_bar = [&](int s) { return bars.full(s); };
  auto empty_bar = [&](int s) { return bars.empty(s); };
  auto a_full_bar = [&](int u) { return bars.a_full(u); };     // HALO: A units
  auto a_empty_bar = [&](int u) { return bars.a_empty(u); };
  // HALO: k-blocks per A unit of the source-0 taps (the dx taps of one dy) and the unit's pixels per row
  const int halo_r = p.mode0 == TAPS_UP2X2 ? 2 : 3;
  const int halo_w = p.bw + halo_r - 1;
  uint8_t* stat_smem = smem_raw + (bar_base + 256u - smem_u32(smem_raw));
  float2* part = reinterpret_cast<float2*>(stat_smem);                    // [warp][BN] {sum, sumsq} over the warp's 16 rows
  float2* run = reinterpret_cast<float2*>(stat_smem + Cfg::PART_BYTES);   // [image slot][which][BN] {value, compensation}

  pdl_prologue();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int KB = p.kb0 + p.kb1;
  const int m_tiles = p.tiles_x * p.tiles_y * p.tiles_n;
  const int total_tiles = m_tiles * p.n_tiles;
  // p.deal == 0: tiles are dealt round-robin — at any moment the resident CTAs work on consecutive tiles (adjacent rows of one image).
  // p.deal == 1 (layers with one N tile and GroupNorm sums to produce): every CTA owns a CONTIGUOUS range of tiles, so its tiles lie
  // in one or two images and the epilogue's running sums are flushed to the global accumulators once or twice per CTA instead
  // of once per tile.
  // split-K (few tiles and a long K, i.e. the 8x8 level: 32-64 CTAs walking 72-144 k-blocks one after the other are
  // latency-bound): p.split_k CTAs share a tile, each accumulates its own range of k-blocks and writes alpha * acc to its own
  // partial buffer (p.out + ks * p.split_stride); splitk_reduce_kernel adds the partials in a fixed order, applies the epilogue
  // terms and accumulates the GroupNorm sums — deterministic, no floating-point atomics
  const int n_units = total_tiles * p.split_k;
  const int n_workers = (int)gridDim.x;
  const int worker = (int)blockIdx.x;
  const int unit_begin = p.deal ? (int)((long long)worker * n_units / n_workers) : worker;
  const int unit_end = p.deal ? (int)((long long)(worker + 1) * n_units / n_workers) : n_units;
  const int unit_step = p.deal ? 1 : n_workers;
  auto k_lo = [&](int u) { return (int)((long long)(u % p.split_k) * KB / p.split_k); };
  auto k_hi = [&](int u) { return (int)((long long)(u % p.split_k + 1) * KB / p.split_k); };

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tm_a0h);
    tma_prefetch_desc(&tm_a0l);
    tma_prefetch_desc(&tm_bh);
    tma_prefetch_desc(&tm_bl);
    if (p.kb1) {
      tma_prefetch_desc(&tm_a1h);
      tma_prefetch_desc(&tm_a1l);
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);    // the producer's expect_tx arrive
      mbar_init(empty_bar(s), 8);   // one arrive per consumer warp
    }
    if (HALO) {
      for (int u = 0; u < HALO_UNITS; ++u) {
        mbar_init(a_full_bar(u), 1);
        mbar_init(a_empty_bar(u), 8);
      }
    }
    mbar_fence_init();
  }
  __syncthreads();

  auto decode = [&](int tile, int& n_idx, int& x0, int& y0, int& n0) { tc_decode(p, tile, n_idx, x0, y0, n0); };

  if (warp == 8) {
    // ------------------------------------------------ TMA producer ------------------------------------------------
    if (lane == 0) {
      TcRing ring;
      for (int u = unit_begin; u < unit_end; u += unit_step)
        tc_produce_tile<Cfg, false, HALO>(&tm_a0h, &tm_a0l, &tm_a1h, &tm_a1l, &tm_bh, &tm_bl, p, smem_base, bars, u / p.split_k, k_lo(u),
                                          k_hi(u), 0u, ring);
    }
  } else {
  // ------------------------------------------------ consumers: wgmma + epilogue ------------------------------------------------
  // warpgroup wg owns tile rows [64 wg, 64 wg + 64); in the m64 accumulator fragment a thread holds, for every 8-column group j,
  // columns 8j + 2(lane % 4) + {0, 1} of rows r0 = 16 warp + lane / 4 (d[4j], d[4j+1]) and r0 + 8 (d[4j+2], d[4j+3])
  const int wg = warp >> 2;
  const uint32_t a_row_off = (uint32_t)wg * 64u * 128u;
  // HALO: the warpgroup's first pixel (yi, xi) inside the tile, as a row of the halo unit
  const uint32_t halo_row_off = (uint32_t)(((wg * 64) / p.bw) * halo_w + (wg * 64) % p.bw) * 128u;
  const int r0 = warp * 16 + (lane >> 2);
  const int cq = (lane & 3) * 2;
  const int tid = threadIdx.x;
  const int ppi = p.bw * p.bh;                // pixels (tile rows) per image
  const int wpi = ppi >= 128 ? 8 : ppi / 16;  // warps per image slot of the tile
  uint32_t stage = 0, phase = 0;
  uint32_t a_done = 0;   // HALO: A units consumed by this CTA's earlier tiles (ring slot = count % HALO_UNITS, parity = count / HALO_UNITS)
  if (p.stats) {
    for (int i = tid; i < 4 * 2 * BN; i += kConsumerThreads) run[i] = make_float2(0.f, 0.f);
  }
  float d[Cfg::ACC];
  const bool dual = DUAL && p.terms != 1;
  auto release = [&](int s) {
    if (lane == 0) mbar_arrive(empty_bar(s));
  };
  auto release_a = [&](int a) {
    if (lane == 0) mbar_arrive(a_empty_bar(a));
  };
  for (int u = unit_begin; u < unit_end; u += unit_step) {
    const int kb_lo = k_lo(u), kb_hi = k_hi(u);
    int prev = -1;
    for (int kb = kb_lo; kb < kb_hi; ++kb) {
      uint32_t a_base = smem_base + stage * Cfg::STAGE_BYTES + a_row_off;   // this warpgroup's rows of the A_hi plane
      uint32_t a_plane = A_PLANE_BYTES;                                     // A_hi -> A_lo
      uint32_t a_unit = 0;                                                  // HALO: this k-block's A unit, counted over the CTA's tiles
      bool a_first = false;                                                 //       and whether the k-block is the unit's first reader
      if constexpr (HALO) {
        // derived from kb instead of carried across iterations: at BN = 128 with DUAL the accumulator leaves no spare registers
        // HALO launches have no side input, so kb < p.kb0 always holds.  The guard and the select below only steer ptxas: written
        // without them, the BN = 128 DUAL instantiation spills 60 / 96 B (stores / loads) instead of 40 / 76
        int ua = 0, dx = 0;
        if (kb < p.kb0) {
          ua = halo_r == 3 ? (int)(__umulhi((uint32_t)kb, 0xAAAAAAABu) >> 1) : kb >> 1;
          dx = kb - ua * halo_r;
        }
        a_unit = a_done + (uint32_t)ua;
        a_first = dx == 0;
        if (a_first) mbar_wait(a_full_bar(a_unit % HALO_UNITS), (a_unit / HALO_UNITS) & 1u);
        a_base = smem_base + (a_unit % HALO_UNITS) * Cfg::A_UNIT_BYTES + (kb < p.kb0 ? halo_row_off + 128u * dx : a_row_off);
        a_plane = HALO_PLANE_BYTES;
      }
      mbar_wait(full_bar(stage), phase);
      const uint32_t sa = smem_base + Cfg::A_RING_BYTES + stage * Cfg::STAGE_BYTES;
      const uint32_t sb = HALO ? sa : sa + 2 * A_PLANE_BYTES;
      const uint64_t ah = wgmma_desc_sw128(a_base);
      const uint64_t al = wgmma_desc_sw128(a_base + a_plane);
      const uint64_t bh = wgmma_desc_sw128(sb);
      const uint64_t bl = wgmma_desc_sw128(sb + Cfg::B_PLANE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t adv = 2u * k;   // 16 fp16 = 32 bytes = 2 x 16-byte units inside the swizzle row
        const uint32_t acc = (uint32_t)(kb != kb_lo || k != 0);
        if (dual) {
          wgmma_tile<DUAL ? 2 * BN : BN>(d, ah + adv, bh + adv, acc);   // [hi*hi | hi*lo]: bh spans both adjacent planes
          wgmma_tile<BN>(d, al + adv, bh + adv, 1u);        // lo*hi into the hi*hi half
        } else {
          wgmma_tile<BN>(d, ah + adv, bh + adv, acc);
          if (p.terms != 1) {
            wgmma_tile<BN>(d, ah + adv, bl + adv, 1u);
            wgmma_tile<BN>(d, al + adv, bh + adv, 1u);
          }
        }
      }
      wgmma_commit();
      // the previous k-block's group has completed once at most this one is pending: its stage goes back to the producer
      wgmma_wait<1>();
      if (prev >= 0) release(prev);
      prev = (int)stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1u;
      }
      // and so has the previous A unit if that k-block was its last reader (this one opens a new unit)
      if (HALO && a_first && kb != kb_lo) release_a((a_unit - 1) % HALO_UNITS);
    }
    wgmma_wait<0>();
    if (prev >= 0) release(prev);
    if constexpr (HALO) {
      a_done += p.cb0 * halo_r;   // the tile's units
      release_a((a_done - 1) % HALO_UNITS);
    }

    // ---- epilogue: rows r0 and r0 + 8 of this tile, 2 adjacent columns per 8-column group ----
    int n_idx, x0, y0, n0;
    decode(u / p.split_k, n_idx, x0, y0, n0);
    tc_epilogue_rows<BN, DUAL, NTAIL>(p, d, dual, r0, cq, n_idx, x0, y0, n0, u % p.split_k);
    if (p.stats) {
      // GroupNorm statistics of the tile.  (1) per warp: the column sums over its 16 rows (one image: >= 32 pixels per image),
      // reduced across the 8 lanes that share a column pair; (2) per image slot: the warps of that image added in a fixed order
      // into running (value, compensation) pairs that persist while consecutive tiles of this CTA stay in the same image and
      // channel block (the tile -> CTA map is static, so these fp32 partial sums are the same every run); (3) flushed with one
      // order-independent fixed-point add per value otherwise, and after every tile with p.stat_per_tile
      tc_stats_rows<BN>(d, part + warp * BN, lane, cq);
      named_bar_sync(1, kConsumerThreads);
      const int nslots = 8 / wpi;
      bool flush = true;
      if (u + unit_step < unit_end) {
        int nn_idx, nx0, ny0, nn0;
        decode((u + unit_step) / p.split_k, nn_idx, nx0, ny0, nn0);
        flush = p.stat_per_tile || nslots > 1 || nn0 != n0 || nn_idx != n_idx;
      }
      for (int i = tid; i < 2 * BN; i += kConsumerThreads) {
        const int which = i / BN, col = i - which * BN;
        for (int g = 0; g < nslots; ++g) {
          float2& acc = run[(g * 2 + which) * BN + col];
          for (int w = g * wpi; w < (g + 1) * wpi; ++w) {
            const float2 pv = part[w * BN + col];
            two_sum_acc(acc.x, acc.y, which ? pv.y : pv.x);
          }
          if (flush) {
            const int n = n0 + g;
            if (n < p.N) {
              StatAcc* dst = p.stats + ((size_t)n * p.st_ld + n_idx * BN + col) * 2 + which;
              stat_add(dst, acc.x);   // integer accumulation: the total is independent of the arrival order
              stat_add(dst, acc.y);
            }
            acc = make_float2(0.f, 0.f);
          }
        }
      }
      named_bar_sync(1, kConsumerThreads);   // part[] is rewritten by the next tile
    }
  }
  }
}

// -------------------------------------------------------------------------------------------------------------------
// Ping-pong form: 3 warpgroups.  WG0 is the TMA producer (one elected thread, 40 registers per thread); WG1 and WG2 are consumers
// (232 registers) that each own a WHOLE 128-row tile as two m64 x BN fragments and take turns on the tensor cores: the units of a
// CTA alternate between them, and an ordered turn (one mbarrier per consumer) lets only one warpgroup issue wgmma at a time, in
// tile order.  A warpgroup hands the turn over right after issuing its last k-block, then waits for its MMAs, releases the stages
// and runs the epilogue while the other warpgroup's MMAs keep the tensor cores busy.  Each output element gets the products of the
// three-instruction form in the same order (hi*hi, hi*lo, lo*hi per 16-deep k-step), so the output is bit-identical to
// conv_tc_kernel without DUAL.  Used for the launches where a CTA walks at least two tiles (see tc_run).
// PAIR: clusters of two CTAs.  Each producer loads its own A and HALF of every B k-block, multicast into both CTAs, so a weight row
// crosses L2 -> SM once per two tiles; a B stage's empty barrier counts the 4 warps of consumer c in this CTA and the 4 of consumer c
// in the peer.  The tile -> worker deal is the unpaired one; the CTAs of cluster k act as workers w and w + T (T = n_tiles, see
// pp_worker), whose tiles at every step have the same N tile because the grid is a multiple of 2T.  Every warpgroup thus sees the
// same tiles in the same order as unpaired, and the output, GroupNorm sums included, is bit-identical to the unpaired launch.  When
// the deal gives the peer one unit more, this CTA walks that step as a ghost: its producer thread multicasts its B halves and
// releases each stage for this CTA's consumers, without MMAs.
// -------------------------------------------------------------------------------------------------------------------
static constexpr int kPpThreads = 384;

// PAIR: the unpaired worker whose units CTA `cta` walks.  Cluster k = cta / 2 pairs workers w and w + T (T = n_tiles) of the block
// of 2T workers it falls in; T = 1 keeps worker = cta.
__device__ __forceinline__ int pp_worker(int cta, int T) {
  const int k = cta >> 1;
  return (k / T) * 2 * T + k % T + (cta & 1) * T;
}

template <int BN, bool HALO>
struct PpCfg {
  using Ring = TcCfg<BN, false, HALO>;   // the ring layout of conv_tc_kernel (no DUAL: it only changes the accumulator)
  // GroupNorm sums, per consumer warpgroup: per-16-row-group column partials (8 groups x BN x {sum, sumsq}) and one running
  // (value, compensation) pair per {sum, sumsq} x BN column — carried across tiles only when the tile is one image (see the
  // epilogue), so one image slot suffices
  static constexpr int PART_BYTES = 8 * BN * 8;
  static constexpr int RUN_BYTES = 2 * BN * 8;
  static constexpr int STAT_BYTES = PART_BYTES + RUN_BYTES;
  static constexpr int SMEM_BYTES = Ring::RING_BYTES + 1024 /*align slack*/ + 256 /*barriers*/ + 2 * STAT_BYTES;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory capacity");
};

template <int BN, int TERMS, bool HALO, bool NTAIL, bool PAIR>
__global__ void __launch_bounds__(kPpThreads, 1)
conv_tc_pingpong_kernel(const __grid_constant__ CUtensorMap tm_a0h, const __grid_constant__ CUtensorMap tm_a0l,
                        const __grid_constant__ CUtensorMap tm_a1h, const __grid_constant__ CUtensorMap tm_a1l,
                        const __grid_constant__ CUtensorMap tm_bh, const __grid_constant__ CUtensorMap tm_bl, const TcParams p) {
  static_assert(TERMS == 1 || TERMS == 3, "1 or 3 fp16 products per MAC");
  static_assert(!PAIR || !NTAIL, "CTA pairs share one weight matrix (no batched GEMMs)");
  using Cfg = PpCfg<BN, HALO>;
  using Ring = typename Cfg::Ring;
  constexpr int STAGES = Ring::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const TcBars<STAGES> bars{smem_base + Ring::RING_BYTES};

  pdl_prologue();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int KB = p.kb0 + p.kb1;
  const int n_units = p.tiles_x * p.tiles_y * p.tiles_n * p.n_tiles * p.split_k;
  const int n_workers = (int)gridDim.x, worker = PAIR ? pp_worker((int)blockIdx.x, p.n_tiles) : (int)blockIdx.x;
  // the tile -> CTA deal of conv_tc_kernel
  const int unit_begin = p.deal ? (int)((long long)worker * n_units / n_workers) : worker;
  const int unit_end = p.deal ? (int)((long long)(worker + 1) * n_units / n_workers) : n_units;
  const int unit_step = p.deal ? 1 : n_workers;
  auto k_lo = [&](int u) { return (int)((long long)(u % p.split_k) * KB / p.split_k); };
  auto k_hi = [&](int u) { return (int)((long long)(u % p.split_k + 1) * KB / p.split_k); };
  // PAIR: units of a worker; the cluster walks max(own, peer's) steps (split_k == 1: every unit is KB k-blocks).  Only the producer
  // warpgroup uses these: at BN = 128 the consumers' main loop has no registers to spare.
  auto units_of = [&](int w) {
    return p.deal ? (int)((long long)(w + 1) * n_units / n_workers) - (int)((long long)w * n_units / n_workers)
                  : (n_units - w + n_workers - 1) / n_workers;
  };
  const int peer = worker + ((blockIdx.x & 1) ? -p.n_tiles : p.n_tiles);   // PAIR: the worker of the other CTA of the cluster

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_a0h);
    tma_prefetch_desc(&tm_a0l);
    tma_prefetch_desc(&tm_bh);
    tma_prefetch_desc(&tm_bl);
    if (p.kb1) {
      tma_prefetch_desc(&tm_a1h);
      tma_prefetch_desc(&tm_a1l);
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(bars.full(s), 1);    // the producer's expect_tx arrive
      mbar_init(bars.empty(s), PAIR ? 8 : 4);   // one arrive per warp of the consuming warpgroup (of both CTAs of a pair)
    }
    if (HALO) {
      for (int u = 0; u < HALO_UNITS; ++u) {
        mbar_init(bars.a_full(u), 1);
        mbar_init(bars.a_empty(u), 4);
      }
    }
    mbar_init(bars.turn(0), 4);   // consumer c may issue its next tile's MMAs: the 4 warps of the other one have issued theirs
    mbar_init(bars.turn(1), 4);
    mbar_fence_init();
  }
  if (PAIR) cluster_sync_all();   // the peer's barriers exist before any multicast or remote arrive can reach them
  else __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------ TMA producer ------------------------------------------------
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      TcRing ring;
      for (int u = unit_begin; u < unit_end; u += unit_step)
        tc_produce_tile<Ring, PAIR, HALO>(&tm_a0h, &tm_a0l, &tm_a1h, &tm_a1l, &tm_bh, &tm_bl, p, smem_base, bars, u / p.split_k,
                                          k_lo(u), k_hi(u), PAIR ? cluster_ctarank() : 0u, ring);
      if constexpr (PAIR) {
        const int peer_begin = p.deal ? (int)((long long)peer * n_units / n_workers) : peer;
        // ghost steps (the peer has a unit more): this thread fills each stage with its B halves (in the peer tile's k order) and
        // releases it for this CTA's consumers, one ring behind.  It issued that fill itself, after the stage's previous fill had been
        // consumed, so the full barrier is at most one phase behind the wait.
        const uint32_t g0 = (uint32_t)(units_of(worker) * KB);
        uint32_t q = g0;
        auto ghost_release = [&](uint32_t g) {
          mbar_wait(bars.full(g % STAGES), (g / STAGES) & 1u);
          for (int w = 0; w < 4; ++w) {   // the arrivals of a consumer's 4 warps, here and in the peer
            mbar_arrive(bars.empty(g % STAGES));
            mbar_arrive_cluster(bars.empty(g % STAGES), cluster_ctarank() ^ 1u);
          }
        };
        for (int j = units_of(worker); j < units_of(peer); ++j) {
          for (int kb = 0; kb < KB; ++kb, ++q) {
            if (q >= g0 + STAGES) ghost_release(q - STAGES);
            tc_produce_tile<Ring, true, HALO>(&tm_a0h, &tm_a0l, &tm_a1h, &tm_a1l, &tm_bh, &tm_bl, p, smem_base, bars,
                                              peer_begin + j * unit_step, kb, kb + 1, cluster_ctarank(), ring, false);
          }
        }
        for (uint32_t g = q >= g0 + STAGES ? q - STAGES : g0; g < q; ++g) ghost_release(g);
        // teardown: wait until the consumers of both CTAs have released the last fill of every stage.  After that no remote arrive
        // can reach this CTA, and every multicast into it has been waited for by its own consumers, so it may exit.
        for (int s = 0; s < STAGES; ++s) {
          mbar_wait(bars.empty(ring.stage), ring.phase ^ 1u);
          if (++ring.stage == STAGES) {
            ring.stage = 0;
            ring.phase ^= 1u;
          }
        }
      }
    }
    return;
  }
  // ------------------------------------------------ consumers: wgmma + epilogue ------------------------------------------------
  setmaxnreg_inc<232>();
  const int c = (warp >> 2) - 1;          // consumer warpgroup: units c, c + 2, ... of this CTA
  const int wq = warp & 3;
  const int tid = threadIdx.x - 128 * (c + 1);
  // fragment f holds tile rows [64 f, 64 f + 64); a thread holds, for every 8-column group j, columns 8j + 2(lane % 4) + {0, 1} of
  // rows 64 f + r0 (d[f][4j], d[f][4j+1]) and 64 f + r0 + 8 (d[f][4j+2], d[f][4j+3])
  const int r0 = wq * 16 + (lane >> 2);
  const int cq = (lane & 3) * 2;
  const int halo_r = p.mode0 == TAPS_UP2X2 ? 2 : 3;
  const int halo_w = p.bw + halo_r - 1;
  const int units_per_tile = p.cb0 * halo_r;   // HALO: A units per tile
  // HALO: the first pixel (yi, xi) of fragment f inside the tile, as a row of the halo unit
  uint32_t halo_row_off[2];
#pragma unroll
  for (int f = 0; f < 2; ++f) halo_row_off[f] = (uint32_t)(((f * 64) / p.bw) * halo_w + (f * 64) % p.bw) * 128u;
  const int wpi = p.bw * p.bh >= 128 ? 8 : p.bw * p.bh / 16;   // 16-row groups per image slot of the tile
  uint8_t* stat_smem = smem_raw + (bars.base + 256u - smem_u32(smem_raw)) + c * Cfg::STAT_BYTES;
  float2* part = reinterpret_cast<float2*>(stat_smem);                     // [16-row group][BN] {sum, sumsq}
  float2* run = reinterpret_cast<float2*>(stat_smem + Cfg::PART_BYTES);    // [which][BN] {value, compensation}
  if (p.stats) {
    for (int i = tid; i < 2 * BN; i += 128) run[i] = make_float2(0.f, 0.f);
  }
  auto release = [&](int s) {
    if (lane == 0) {
      mbar_arrive(bars.empty(s));
      if (PAIR) mbar_arrive_cluster(bars.empty(s), cluster_ctarank() ^ 1u);
    }
  };
  auto release_a = [&](uint32_t a) {
    if (lane == 0) mbar_arrive(bars.a_empty(a % HALO_UNITS));
  };
  // position of this warpgroup's next k-block in the B-stage ring: all k-blocks of the CTA's earlier units, both warpgroups'
  uint32_t kpos = c ? (uint32_t)(k_hi(unit_begin) - k_lo(unit_begin)) : 0u;
  float d[2][BN / 2];
  int turn = 0;
  for (int u = unit_begin + c * unit_step; u < unit_end; u += 2 * unit_step, ++turn) {
    const int kb_lo = k_lo(u), kb_hi = k_hi(u);
    if (c == 1 || turn > 0) mbar_wait(bars.turn(c), (uint32_t)(c ? turn : turn - 1) & 1u);
    uint32_t stage = kpos % STAGES, phase = (kpos / STAGES) & 1u;
    const uint32_t a_done = (uint32_t)((2 * turn + c) * units_per_tile);   // HALO: A units of the CTA's earlier tiles
    int prev = -1;
    for (int kb = kb_lo; kb < kb_hi; ++kb) {
      const uint32_t sb = smem_base + Ring::A_RING_BYTES + stage * Ring::STAGE_BYTES;
      uint32_t a_base = sb;   // fragment 0's rows of the A_hi plane
      uint32_t a_frag1 = 64u * 128u;
      uint32_t a_plane = A_PLANE_BYTES;
      uint32_t a_unit = 0;
      bool a_first = false;
      if constexpr (HALO) {
        // HALO launches have no side input: k-block kb reads unit kb / halo_r, shifted by dx pixels
        const int ua = halo_r == 3 ? (int)(__umulhi((uint32_t)kb, 0xAAAAAAABu) >> 1) : kb >> 1;
        const int dx = kb - ua * halo_r;
        a_unit = a_done + (uint32_t)ua;
        a_first = dx == 0;
        if (a_first) mbar_wait(bars.a_full(a_unit % HALO_UNITS), (a_unit / HALO_UNITS) & 1u);
        a_base = smem_base + (a_unit % HALO_UNITS) * Ring::A_UNIT_BYTES + halo_row_off[0] + 128u * dx;
        a_frag1 = halo_row_off[1] - halo_row_off[0];
        a_plane = HALO_PLANE_BYTES;
      }
      mbar_wait(bars.full(stage), phase);
      const uint32_t sbb = HALO ? sb : sb + 2 * A_PLANE_BYTES;
      const uint64_t ah0 = wgmma_desc_sw128(a_base), ah1 = wgmma_desc_sw128(a_base + a_frag1);
      const uint64_t al0 = wgmma_desc_sw128(a_base + a_plane), al1 = wgmma_desc_sw128(a_base + a_frag1 + a_plane);
      const uint64_t bh = wgmma_desc_sw128(sbb);
      const uint64_t bl = wgmma_desc_sw128(sbb + Ring::B_PLANE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t adv = 2u * k;   // 16 fp16 = 32 bytes = 2 x 16-byte units inside the swizzle row
        const uint32_t acc = (uint32_t)(kb != kb_lo || k != 0);
        wgmma_tile<BN>(d[0], ah0 + adv, bh + adv, acc);
        wgmma_tile<BN>(d[1], ah1 + adv, bh + adv, acc);
        if constexpr (TERMS == 3) {
          wgmma_tile<BN>(d[0], ah0 + adv, bl + adv, 1u);
          wgmma_tile<BN>(d[1], ah1 + adv, bl + adv, 1u);
          wgmma_tile<BN>(d[0], al0 + adv, bh + adv, 1u);
          wgmma_tile<BN>(d[1], al1 + adv, bh + adv, 1u);
        }
      }
      wgmma_commit();
      // the previous k-block's group has completed once at most this one is pending: its stage goes back to the producer
      wgmma_wait<1>();
      if (prev >= 0) release(prev);
      prev = (int)stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1u;
      }
      // and so has the previous A unit if that k-block was its last reader (this one opens a new unit)
      if (HALO && a_first && kb != kb_lo) release_a(a_unit - 1);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bars.turn(c ^ 1));   // every MMA of this tile is issued: the other warpgroup's turn
    wgmma_wait<0>();
    if (prev >= 0) release(prev);
    if (HALO) release_a(a_done + units_per_tile - 1);
    // the other warpgroup's unit (if any) lies between this one and this warpgroup's next in the ring
    kpos += (uint32_t)(kb_hi - kb_lo) + (uint32_t)(k_hi(u + unit_step) - k_lo(u + unit_step));

    // ---- epilogue ----
    int n_idx, x0, y0, n0;
    tc_decode(p, u / p.split_k, n_idx, x0, y0, n0);
#pragma unroll
    for (int f = 0; f < 2; ++f) tc_epilogue_rows<BN, false, NTAIL>(p, d[f], false, 64 * f + r0, cq, n_idx, x0, y0, n0, u % p.split_k);
    if (p.stats) {
      // GroupNorm statistics of the tile, as in conv_tc_kernel: (1) per 16-row group (warp wq of fragment f = group 4 f + wq), the
      // column sums, (2) per image slot the groups of that image in a fixed order, into a running (value, compensation) pair that
      // persists while this warpgroup's consecutive tiles stay in one image and channel block (only possible when a tile is one
      // image), (3) flushed with one fixed-point add per value otherwise
#pragma unroll
      for (int f = 0; f < 2; ++f) tc_stats_rows<BN>(d[f], part + (4 * f + wq) * BN, lane, cq);
      named_bar_sync(1 + c, 128);
      const int nslots = 8 / wpi;
      bool flush = true;
      const int un = u + 2 * unit_step;   // this warpgroup's next unit
      if (!p.stat_per_tile && un < unit_end) {
        int nn_idx, nx0, ny0, nn0;
        tc_decode(p, un / p.split_k, nn_idx, nx0, ny0, nn0);
        flush = nslots > 1 || nn0 != n0 || nn_idx != n_idx;
      }
      for (int i = tid; i < 2 * BN; i += 128) {
        const int which = i / BN, col = i - which * BN;
        for (int g = 0; g < nslots; ++g) {
          float2 acc = nslots == 1 ? run[i] : make_float2(0.f, 0.f);
          for (int w = g * wpi; w < (g + 1) * wpi; ++w) {
            const float2 pv = part[w * BN + col];
            two_sum_acc(acc.x, acc.y, which ? pv.y : pv.x);
          }
          if (flush) {
            const int n = n0 + g;
            if (n < p.N) {
              StatAcc* dst = p.stats + ((size_t)n * p.st_ld + n_idx * BN + col) * 2 + which;
              stat_add(dst, acc.x);   // integer accumulation: the total is independent of the arrival order
              stat_add(dst, acc.y);
            }
            acc = make_float2(0.f, 0.f);
          }
          if (nslots == 1) run[i] = acc;
        }
      }
      named_bar_sync(1 + c, 128);   // part[] is rewritten by this warpgroup's next tile
    }
  }
}

// -------------------------------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q));
    DDNM_CHECK(f != nullptr && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
    fn = reinterpret_cast<EncodeTiledFn>(f);
  }
  return fn;
}

// strides_elems: element strides of dims 1..rank-1 (nullptr = densely packed)
static CUtensorMap make_map_f16(const void* base, int rank, const uint64_t* dims, const uint32_t* box,
                                const uint64_t* strides_elems = nullptr) {
  CUtensorMap m;
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t b[5], es[5];
  uint64_t stride = 2;
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    b[i] = box[i];
    es[i] = 1;
    stride *= dims[i];
    if (i < rank - 1) gstr[i] = strides_elems ? strides_elems[i] * 2 : stride;
  }
  CUresult r = encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), gdim, gstr, b, es,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DDNM_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
  return m;
}

static int g_terms = 3;
void tc_set_terms(int terms) {
  DDNM_CHECK(terms == 1 || terms == 3, "terms must be 1 or 3");
  g_terms = terms;
}
int tc_get_terms() { return g_terms; }
static int g_force_bn = 0;
void tc_debug_force_bn(int bn) {
  DDNM_CHECK(bn == 0 || bn == 64 || bn == 128, "BN must be 0 (heuristic), 64 or 128");
  g_force_bn = bn;
}
static int g_dual_mode = 1;    // 1: conv_tc_kernel launches use the DUAL form (default), 0: never
void tc_debug_dual_mode(int mode) { g_dual_mode = mode; }
// HALO form wherever legal (see tc_make_launch); env DDNM_HALO=0 / tc_debug_halo(0) keep every launch on one A load per k-block
static int g_halo_enable = [] { const char* v = std::getenv("DDNM_HALO"); return v && *v ? std::atoi(v) : 1; }();
void tc_debug_halo(int on) { g_halo_enable = on; }
// ping-pong kernel for the launches where CTAs walk several tiles (see tc_run); env DDNM_PINGPONG=0 / tc_debug_pingpong(0) keep
// them on conv_tc_kernel
static int g_pingpong_enable = [] { const char* v = std::getenv("DDNM_PINGPONG"); return v && *v ? std::atoi(v) : 1; }();
void tc_debug_pingpong(int on) { g_pingpong_enable = on; }
// ping-pong launches with one N tile on CTA pairs that multicast the weights (see conv_tc_pingpong_kernel and tc_make_launch)
static int g_pp_pair_enable = [] { const char* v = std::getenv("DDNM_PP_PAIR"); return v && *v ? std::atoi(v) : 1; }();
void tc_debug_pp_pair(int on) { g_pp_pair_enable = on; }
static int g_deal = -1;
void tc_debug_deal(int mode) {
  DDNM_CHECK(mode >= -1 && mode <= 1, "deal mode must be -1 (default rule), 0 (round-robin) or 1 (contiguous ranges)");
  g_deal = mode;
}

TcLaunch tc_make_launch(const SplitView& src0, int mode0, const SplitView* src1, const __half* w_hi, const __half* w_lo,
                        int w_batches, int Cout, const View& out, const float* chanadd, int ca_ld, const float* residual,
                        int ldr, float alpha, int num_sms, int res_mode, bool invariant) {
  TcLaunch L;
  TcParams& p = L.p;
  const int taps = (mode0 == TAPS_1X1) ? 1 : (mode0 == TAPS_UP2X2 ? 4 : 9);
  DDNM_CHECK(src0.C % BK == 0, "tensor-core conv needs Cin % 64 == 0");
  DDNM_CHECK(Cout % 64 == 0, "tensor-core conv needs Cout % 64 == 0");
  p.H = out.H; p.W = out.W; p.N = out.N;
  // M tile: 128 consecutive pixels as [bn][bh][bw]
  p.bw = out.W >= 128 ? 128 : out.W;
  DDNM_CHECK(128 % p.bw == 0 && out.W % p.bw == 0, "unsupported width for the 128-pixel tile");
  p.bh = std::min(out.H, 128 / p.bw);
  DDNM_CHECK(out.H % p.bh == 0 && 128 % (p.bw * p.bh) == 0, "unsupported height for the 128-pixel tile");
  p.bn = 128 / (p.bw * p.bh);
  p.tiles_x = out.W / p.bw;
  p.tiles_y = out.H / p.bh;
  p.tiles_n = cdiv(out.N, p.bn);
  // N tile: BN = 128 halves the A-operand reads per output and the tile count; BN = 64 only where 128 would leave more than
  // half of the SMs without a tile (rounds of resident CTAs, one CTA per SM)
  {
    const int m_tiles = p.tiles_x * p.tiles_y * p.tiles_n;
    L.BN = 64;
    if (Cout % 128 == 0 && (long long)m_tiles * (Cout / 128) >= num_sms / 2) L.BN = 128;
    if (g_force_bn && Cout % g_force_bn == 0) L.BN = g_force_bn;   // tests / tuning experiments only
  }
  p.n_tiles = Cout / L.BN;
  // batch-invariant launches run the three-instruction form, which conv_tc_kernel without DUAL and the ping-pong kernel share
  // element for element, so the kernel a launch picks (tc_run: tiles per CTA) cannot change a value
  L.dual = !invariant && g_dual_mode != 0;
  L.pingpong = g_pingpong_enable != 0;
  p.mode0 = mode0;
  p.cb0 = src0.C / BK;
  p.kb0 = taps * p.cb0;
  p.kb1 = src1 ? src1->C / BK : 0;
  if (src1) DDNM_CHECK(src1->C % BK == 0 && src1->H == out.H && src1->W == out.W && src1->N == out.N, "bad 1x1 side input");
  p.phase_stride = 0;
  p.up_py = p.up_px = 0;
  p.b_batched = w_batches > 1 ? 1 : 0;
  if (p.b_batched) DDNM_CHECK(p.bn == 1 && w_batches == out.N, "batched B operand needs one image per tile");
  if (mode0 == TAPS_3X3_S2) {
    DDNM_CHECK(src0.H == out.H && src0.W == out.W && src0.N == 4 * out.N, "stride-2 source must be 4 parity phases");
    p.phase_stride = out.N;
  } else {
    DDNM_CHECK(src0.H == out.H && src0.W == out.W && src0.N == out.N, "source/output shape mismatch");
  }
  p.Cout = Cout; p.ldc = out.ld; p.out = out.p;
  p.out_sx = out.ld; p.out_sy = (long long)out.W * out.ld; p.out_sn = (long long)out.H * out.W * out.ld;
  DDNM_CHECK(out.C == Cout && out.ld % 2 == 0 && ((uintptr_t)out.p & 7) == 0, "output view misaligned (rows move as float2)");
  p.chanadd = chanadd; p.ca_ld = ca_ld; p.residual = residual; p.ldr = ldr; p.alpha = alpha; p.res_mode = res_mode;
  p.stats = out.st; p.st_ld = out.st_ld;
  p.terms = g_terms;
  p.stat_per_tile = invariant ? 1 : 0;
  if (out.st) DDNM_CHECK(p.bw * p.bh >= 32, "GroupNorm statistics need >= 32 pixels per image");
  if (residual) DDNM_CHECK(ldr % 2 == 0 && ((uintptr_t)residual & 7) == 0, "residual misaligned (rows move as float2)");
  if (chanadd) DDNM_CHECK(ca_ld % 2 == 0 && ((uintptr_t)chanadd & 7) == 0, "channel-add rows misaligned");

  const uint64_t ad[4] = {(uint64_t)src0.C, (uint64_t)src0.W, (uint64_t)src0.H, (uint64_t)src0.N};
  const uint32_t abox[4] = {(uint32_t)BK, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
  L.a0h = make_map_f16(src0.hi, 4, ad, abox);
  L.a0l = make_map_f16(src0.lo, 4, ad, abox);
  // HALO form: stride-1 taps on tiles whose warpgroups each own 64 consecutive pixels of one image row (one image per tile).  The
  // halo maps are kept next to the plain ones: a launch that is later split along K (UNetEngine::emit_tc) runs without them.
  // Not with a 1x1 side input: its k-blocks have no taps to share, and as one A unit each they left the celeba conv2 + shortcut
  // launches at 128^2 / 256^2 up to 12 % slower than the per-tap form (whole forward: 60.1 ms with them in the HALO form, 58.2 without).
  L.halo = g_halo_enable != 0 && (mode0 == TAPS_3X3 || mode0 == TAPS_UP2X2) && p.bw % 64 == 0 && p.bn == 1 && !src1;
  if (L.halo) {
    const uint32_t hbox[4] = {(uint32_t)BK, (uint32_t)(p.bw + (mode0 == TAPS_UP2X2 ? 1 : 2)), (uint32_t)p.bh, 1u};
    L.hh = make_map_f16(src0.hi, 4, ad, hbox);
    L.hl = make_map_f16(src0.lo, 4, ad, hbox);
  }
  if (src1) {
    const uint64_t ad1[4] = {(uint64_t)src1->C, (uint64_t)src1->W, (uint64_t)src1->H, (uint64_t)src1->N};
    L.a1h = make_map_f16(src1->hi, 4, ad1, abox);
    L.a1l = make_map_f16(src1->lo, 4, ad1, abox);
  } else {
    L.a1h = L.a0h;
    L.a1l = L.a0l;
  }
  const int Ktot = (p.kb0 + p.kb1) * BK;
  const uint64_t bd[3] = {(uint64_t)Ktot, (uint64_t)Cout, (uint64_t)w_batches};
  const uint32_t bbox[3] = {(uint32_t)BK, (uint32_t)L.BN, 1u};
  L.bh = make_map_f16(w_hi, 3, bd, bbox);
  L.bl = make_map_f16(w_lo, 3, bd, bbox);
  // ping-pong CTA pairs (one weight matrix; tc_run takes them when the launch runs on the ping-pong kernel unsplit).  Not for the
  // upsample phases: celeba B = 16 on an H100 SXM (700 W) ran the 128 -> 256 phases 8 % slower paired, the 256^2 / 128^2 3x3
  // launches 3-11 % faster.
  L.pp_pair = g_pp_pair_enable != 0 && w_batches == 1 && mode0 != TAPS_UP2X2;
  if (L.pp_pair) {
    const uint32_t hbox[3] = {(uint32_t)BK, (uint32_t)(L.BN / 2), 1u};
    L.bh2 = make_map_f16(w_hi, 3, bd, hbox);
    L.bl2 = make_map_f16(w_lo, 3, bd, hbox);
  }
  const int total = p.tiles_x * p.tiles_y * p.tiles_n * p.n_tiles;
  L.grid = std::min(total, num_sms);
  // contiguous tile ranges per CTA where the GroupNorm sums of the output would otherwise be flushed at every tile: one N tile
  // (so consecutive tiles of a range share their channels) and several tiles per CTA
  p.deal = g_deal >= 0 ? g_deal : (out.st != nullptr && p.n_tiles == 1 && total >= 2 * L.grid ? 1 : 0);
  if (p.n_tiles != 1) p.deal = 0;
  L.flops = 2.0 * (double)out.pixels() * Cout * Ktot;
  return L;
}

TcLaunch tc_make_up2_launch(const SplitView& src, const __half* w_hi, const __half* w_lo, int Cout, const View& out, const float* chanadd,
                            int ca_ld, int py, int px, int num_sms, bool invariant) {
  DDNM_CHECK(out.H == 2 * src.H && out.W == 2 * src.W && out.N == src.N, "upsample phase: output must be twice the source size");
  View lr = out;   // tile over the low-res pixel grid; every tile pixel (y, x) lands on output pixel (2y+py, 2x+px)
  lr.H = src.H;
  lr.W = src.W;
  TcLaunch L = tc_make_launch(src, TAPS_UP2X2, nullptr, w_hi, w_lo, 1, Cout, lr, chanadd, ca_ld, nullptr, 0, 1.0f, num_sms, 0, invariant);
  TcParams& p = L.p;
  p.up_py = py;
  p.up_px = px;
  p.out = out.p + ((size_t)py * out.W + px) * out.ld;
  p.out_sx = 2LL * out.ld;
  p.out_sy = 2LL * out.W * out.ld;
  p.out_sn = (long long)out.H * out.W * out.ld;
  return L;
}

TcConvPlan tc_plan_conv(const SplitView& src0, int mode0, const SplitView* src1, const __half* w_hi, const __half* w_lo, int Cout,
                        const View& out, const float* chanadd, int ca_ld, const float* residual, int ldr, int res_mode, int num_sms,
                        bool invariant, int split_k) {
  TcConvPlan P;
  P.out = out; P.chanadd = chanadd; P.ca_ld = ca_ld; P.residual = residual; P.ldr = ldr;
  P.L = tc_make_launch(src0, mode0, src1, w_hi, w_lo, 1, Cout, out, chanadd, ca_ld, residual, ldr, 1.0f, num_sms, res_mode, invariant);
  // split-K: few tiles walking a long K one k-block after the other (the 8x8 level: 32-64 CTAs, 72-144 k-blocks) are latency-bound;
  // 2 or 4 CTAs per tile, each over its own k-block range into its own partial buffer, then one small deterministic reduce
  const TcParams& p = P.L.p;
  const int tiles = p.tiles_x * p.tiles_y * p.tiles_n * p.n_tiles, kblocks = p.kb0 + p.kb1;
  static const bool split_on = std::getenv("DDNM_SPLITK") == nullptr || std::atoi(std::getenv("DDNM_SPLITK")) != 0;
  int S = 1;
  if (split_k > 0) {
    DDNM_CHECK(split_k == 1 || split_k == 2 || split_k == 4, "split_k must be 1, 2 or 4");
    DDNM_CHECK(split_k == 1 || (res_mode == 0 && kblocks >= split_k), "split-K needs res_mode 0 and a k-block per split");
    S = split_k;
  } else if (split_on && res_mode == 0 && kblocks >= 32) {
    // batch-invariant mode: S is part of an element's arithmetic (the k-block ranges and their fixed-order sum), so it follows the
    // per-image shape alone — 2 on the maps of at most 64 pixels, the 8x8 level where B = 16 splits by the tile count as well
    if (invariant) S = out.H * out.W <= 64 ? 2 : 1;
    else if (2 * tiles <= num_sms) S = 4 * tiles <= num_sms ? 4 : 2;
  }
  if (S == 1) return P;
  P.S = S;
  const long long stride = out.pixels() * Cout;
  P.part_elems = S * stride;
  View pv = out;   // the partial buffers: dense [pixels][Cout], no epilogue terms, no GroupNorm sums (the reduce does those)
  pv.p = nullptr; pv.ld = Cout; pv.st = nullptr; pv.st_ld = 0;
  TcLaunch Ls = tc_make_launch(src0, mode0, src1, w_hi, w_lo, 1, Cout, pv, nullptr, 0, nullptr, 0, 1.0f, num_sms, 0, invariant);
  DDNM_CHECK(Ls.BN == P.L.BN, "split-K: tile shape changed");
  Ls.p.split_k = S;
  Ls.p.split_stride = stride;
  Ls.halo = false;   // k-block ranges of a split need not be whole A units
  Ls.grid = std::min(tiles * S, num_sms);
  P.L = Ls;
  return P;
}

void tc_set_partials(TcConvPlan& P, float* part) {
  DDNM_CHECK(P.S > 1 && part != nullptr, "partial buffer for an unsplit plan");
  P.part = part;
  P.L.p.out = part;
}

void tc_run_split_reduce(const TcConvPlan& P, cudaStream_t stream) {
  DDNM_CHECK(P.S > 1 && P.part != nullptr, "split-K reduce without partial buffers");
  splitk_reduce(P.part, P.S, P.part_elems / P.S, P.out, P.chanadd, P.ca_ld, P.residual, P.ldr, stream);
}

void tc_run_conv(const TcConvPlan& P, cudaStream_t stream) {
  tc_run(P.L, stream);
  if (P.S > 1) tc_run_split_reduce(P, stream);
}

TcLaunch tc_make_gemm_launch(const GemmOperand& A, const GemmOperand& B, int M, int N, int K, int heads, int images, float* out,
                             long long out_sn, long long out_sy, long long out_sx, float alpha, int num_sms, bool invariant) {
  TcLaunch L;
  TcParams& p = L.p;
  // K and N need not fill whole 64-wide blocks: the operand maps end at K and N, so TMA zero-fills the rest of the last k-block and
  // of the last N tile, and the epilogue stores no column past N (NTAIL).  The 16-byte TMA alignment of the rows needs K % 8 == 0.
  DDNM_CHECK(M % 128 == 0 && N % 8 == 0 && K % 8 == 0, "attention GEMM: M % 128, N % 8, K % 8");
  p.H = heads; p.W = M; p.N = images;
  p.bw = 128; p.bh = 1; p.bn = 1;
  p.tiles_x = M / 128; p.tiles_y = heads; p.tiles_n = images;
  const int m_tiles = p.tiles_x * p.tiles_y * p.tiles_n;
  // as for the convolutions: BN = 128 unless it leaves most SMs idle
  L.BN = 64;
  if (N % 128 == 0 && (long long)m_tiles * (N / 128) >= num_sms / 2) L.BN = 128;
  if (g_force_bn && N % g_force_bn == 0) L.BN = g_force_bn;   // tests / tuning experiments only
  L.dual = !invariant && g_dual_mode != 0;   // as in tc_make_launch (no GroupNorm sums here)
  L.pingpong = g_pingpong_enable != 0;
  p.n_tiles = cdiv(N, L.BN);
  L.ntail = N % L.BN != 0;
  p.mode0 = TAPS_1X1;
  p.cb0 = cdiv(K, BK); p.kb0 = p.cb0; p.kb1 = 0;
  p.phase_stride = 0;
  p.up_py = p.up_px = 0;
  p.b_batched = 2;
  p.Cout = N; p.ldc = (int)out_sx; p.out = out;
  p.out_sn = out_sn; p.out_sy = out_sy; p.out_sx = out_sx;
  DDNM_CHECK(out_sx % 2 == 0 && out_sy % 2 == 0 && out_sn % 2 == 0 && ((uintptr_t)out & 7) == 0, "attention GEMM output misaligned");
  p.chanadd = nullptr; p.ca_ld = 0; p.residual = nullptr; p.ldr = 0; p.res_mode = 0; p.alpha = alpha;
  p.stats = nullptr; p.st_ld = 0;
  p.terms = g_terms;
  const uint64_t ad[4] = {(uint64_t)K, (uint64_t)M, (uint64_t)heads, (uint64_t)images};
  const uint64_t as[3] = {(uint64_t)A.s_row, (uint64_t)A.s_head, (uint64_t)A.s_img};
  const uint32_t abox[4] = {(uint32_t)BK, 128u, 1u, 1u};
  L.a0h = make_map_f16(A.hi, 4, ad, abox, as);
  L.a0l = make_map_f16(A.lo, 4, ad, abox, as);
  L.a1h = L.a0h;
  L.a1l = L.a0l;
  const uint64_t bd[4] = {(uint64_t)K, (uint64_t)N, (uint64_t)heads, (uint64_t)images};
  const uint64_t bs[3] = {(uint64_t)B.s_row, (uint64_t)B.s_head, (uint64_t)B.s_img};
  const uint32_t bbox[4] = {(uint32_t)BK, (uint32_t)L.BN, 1u, 1u};
  L.bh = make_map_f16(B.hi, 4, bd, bbox, bs);
  L.bl = make_map_f16(B.lo, 4, bd, bbox, bs);
  L.grid = std::min(m_tiles * p.n_tiles, num_sms);
  L.flops = 2.0 * (double)images * heads * M * (double)N * K;
  return L;
}

template <int BN, bool DUAL, bool HALO = false, bool NTAIL = false>
static void launch_bn(const TcLaunch& L, cudaStream_t stream) {
  using Cfg = TcCfg<BN, DUAL, HALO>;
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set))
    CUDA_CHECK(cudaFuncSetAttribute(conv_tc_kernel<BN, DUAL, HALO, NTAIL>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  launch_pdl(conv_tc_kernel<BN, DUAL, HALO, NTAIL>, dim3(L.grid), dim3(kTcThreads), (size_t)Cfg::SMEM_BYTES, stream, 1,
             HALO ? L.hh : L.a0h, HALO ? L.hl : L.a0l, L.a1h, L.a1l, L.bh, L.bl, L.p);
  CUDA_CHECK(cudaGetLastError());
}

template <int BN>
static void launch_forms(const TcLaunch& L, cudaStream_t stream) {
  if (L.ntail) {   // batched GEMMs with a partial N tile: N % 64 != 0, so BN = 64
    if constexpr (BN == 64) {
      if (L.dual) launch_bn<BN, true, false, true>(L, stream);
      else launch_bn<BN, false, false, true>(L, stream);
      return;
    }
    throw Error("partial N tiles need BN = 64");
  }
  if (L.halo && L.dual) launch_bn<BN, true, true>(L, stream);
  else if (L.halo) launch_bn<BN, false, true>(L, stream);
  else if (L.dual) launch_bn<BN, true>(L, stream);
  else launch_bn<BN, false>(L, stream);
}

template <int BN, int TERMS, bool HALO, bool NTAIL = false, bool PAIR = false>
static void launch_pingpong(const TcLaunch& L, cudaStream_t stream) {
  using Cfg = PpCfg<BN, HALO>;
  const auto kernel = conv_tc_pingpong_kernel<BN, TERMS, HALO, NTAIL, PAIR>;
  static bool attr_set[64] = {};
  static int max_clusters[64] = {};
  if (first_use_on_device(attr_set)) {
    CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    if (PAIR) {
      // a GPC with an odd number of free SMs holds fewer clusters of two than half its SMs
      cudaLaunchConfig_t cfg = {};
      cudaLaunchAttribute at;
      at.id = cudaLaunchAttributeClusterDimension;
      at.val.clusterDim.x = 2;
      at.val.clusterDim.y = 1;
      at.val.clusterDim.z = 1;
      cfg.gridDim = dim3(2);
      cfg.blockDim = dim3(kPpThreads);
      cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
      cfg.attrs = &at;
      cfg.numAttrs = 1;
      int dev = 0;
      CUDA_CHECK(cudaGetDevice(&dev));
      CUDA_CHECK(cudaOccupancyMaxActiveClusters(&max_clusters[dev & 63], kernel, &cfg));
    }
  }
  if (PAIR) {
    int dev = 0;
    CUDA_CHECK(cudaGetDevice(&dev));
    // the pairs keep the single-CTA grid: where its clusters cannot all be resident at once, the launch stays on single CTAs
    if (L.grid / 2 > max_clusters[dev & 63]) {
      launch_pingpong<BN, TERMS, HALO, NTAIL, false>(L, stream);
      return;
    }
  }
  launch_pdl(kernel, dim3(L.grid), dim3(kPpThreads), (size_t)Cfg::SMEM_BYTES, stream, PAIR ? 2 : 1, HALO ? L.hh : L.a0h,
             HALO ? L.hl : L.a0l, L.a1h, L.a1l, PAIR ? L.bh2 : L.bh, PAIR ? L.bl2 : L.bl, L.p);
  CUDA_CHECK(cudaGetLastError());
}

template <int BN, bool PAIR>
static void launch_pingpong_terms(const TcLaunch& L, cudaStream_t stream) {
  if (L.p.terms == 1) {
    if (L.halo) launch_pingpong<BN, 1, true, false, PAIR>(L, stream);
    else launch_pingpong<BN, 1, false, false, PAIR>(L, stream);
  } else {
    if (L.halo) launch_pingpong<BN, 3, true, false, PAIR>(L, stream);
    else launch_pingpong<BN, 3, false, false, PAIR>(L, stream);
  }
}

template <int BN>
static void launch_pingpong_forms(const TcLaunch& L, cudaStream_t stream) {
  if (L.ntail) {   // as in launch_forms
    if constexpr (BN == 64) {
      if (L.p.terms == 1) launch_pingpong<BN, 1, false, true>(L, stream);
      else launch_pingpong<BN, 3, false, true>(L, stream);
      return;
    }
    throw Error("partial N tiles need BN = 64");
  }
  // CTA pairs: unsplit, and a grid of whole blocks of 2 * n_tiles workers, so the two workers of a cluster (pp_worker) always have
  // the same N tile; with several N tiles the deal is round-robin (tc_make_launch)
  if (L.pp_pair && L.p.split_k == 1 && L.grid % (2 * L.p.n_tiles) == 0 && (L.p.n_tiles == 1 || L.p.deal == 0))
    launch_pingpong_terms<BN, true>(L, stream);
  else launch_pingpong_terms<BN, false>(L, stream);
}

void tc_run(const TcLaunch& L, cudaStream_t stream) {
  DDNM_CHECK(!L.halo || (L.p.split_k == 1 && L.p.kb1 == 0), "the HALO form runs unsplit launches without a 1x1 side input");
  // ping-pong needs two tiles per CTA to overlap one tile's epilogue with the next one's MMAs; a CTA with one tile (the split-K
  // launches, the 16x16 level) runs faster on two warpgroups sharing it
  const int units = L.p.tiles_x * L.p.tiles_y * L.p.tiles_n * L.p.n_tiles * L.p.split_k;
  if (L.pingpong && units > L.grid) {
    switch (L.BN) {
      case 128: launch_pingpong_forms<128>(L, stream); return;
      case 64: launch_pingpong_forms<64>(L, stream); return;
      default: throw Error("bad BN");
    }
  }
  switch (L.BN) {
    case 128: launch_forms<128>(L, stream); break;
    case 64: launch_forms<64>(L, stream); break;
    default: throw Error("bad BN");
  }
}

}  // namespace ddnm

// wgmma implicit-GEMM convolution / GEMM with 3x fp16 split ("fp32-grade" products on the
// Hopper tensor cores).  See tc_gemm.cu for the kernel; this header is the host-side launch record.
#pragma once
#include "common.cuh"

namespace ddnm {

enum TcTapMode : int {
  TAPS_3X3 = 0,     // 3x3, stride 1, zero pad 1 (pad comes from TMA out-of-bounds zero fill)
  TAPS_1X1 = 1,     // 1x1 / plain GEMM rows
  TAPS_3X3_S2 = 2,  // 3x3, stride 2, pad (0,1,0,1): source is stored as 4 parity phases (space-to-depth)
  TAPS_UP2X2 = 3,   // one output parity phase of (nearest x2 upsample -> 3x3 pad 1): a 2x2 stencil on the LOW-res source
};

struct TcParams {
  int H, W, N;                 // OUTPUT spatial size and number of images
  int bw, bh, bn;              // 128-row M tile = bn images x bh rows x bw columns
  int tiles_x, tiles_y, tiles_n;
  int n_tiles;                 // Cout / BN
  int mode0;                   // TcTapMode of source 0
  int cb0, kb0;                // source 0: 64-channel blocks per tap, total k-blocks (= taps * cb0)
  int kb1;                     // source 1 (always 1x1, e.g. the nin_shortcut input): k-blocks, 0 = absent
  int phase_stride;            // TAPS_3X3_S2: images per parity phase in the source's outer dim
  int up_py, up_px;            // TAPS_UP2X2: output parity (row, column) this launch produces
  int b_batched;               // 1: B has one matrix per image (3D map, z = image); 2: B is a 4D map sharing the A tile's
                               //    two outer coordinates (attention: y = head, n = image)
  long long out_sn, out_sy, out_sx;  // output element strides per image / row / column of the M tile's pixel grid
  int Cout, ldc;
  float* out;                  // out[pixel*ldc + co]
  const float* chanadd;        // chanadd[image*ca_ld + co] added per (image, channel): bias (+ timestep projection); may be null
  int ca_ld;                   // 0 = one row broadcast over images
  const float* residual;       // residual[pixel*ldr + co]; may be null
  int ldr;
  int res_mode;                // 0: same pixel; 1: nearest-upsampled source (H/2 x W/2); 2: 2x2 average of a (2H x 2W) source
  float alpha;                 // out = alpha*acc + chanadd + residual
  StatAcc* stats;              // optional GroupNorm sums of the OUTPUT: stats[(image*st_ld + co)*2 + {0,1}] += {sum, sumsq}
  int st_ld;
  int split_k = 1;             // > 1: this many CTAs per tile, each over its own k-block range, partial sums to out + ks * split_stride
  long long split_stride = 0;  //      (no chanadd / residual / stats: splitk_reduce applies them)
  int deal = 0;                // tile -> CTA map: 0 round-robin, 1 one contiguous range per CTA (see conv_tc_kernel)
  int terms;                   // 3: hi*hi + hi*lo + lo*hi (fp32-grade, default); 1: hi*hi only (plain fp16 inputs, fast mode)
  int stat_per_tile = 0;       // 1 (batch-invariant launches): each tile's GroupNorm partials go to `stats` on their own, never
                               //    carried into the CTA's next tile, so their grouping depends only on the tile's place in its image
};

struct TcLaunch {
  CUtensorMap a0h, a0l, a1h, a1l, bh, bl;
  CUtensorMap hh, hl;          // HALO: source 0 with a halo-row box {64, bw + 2 (up2: bw + 1), bh, 1}
  TcParams p;
  int BN = 128;
  bool dual = false;           // A_hi x [B_hi; B_lo] as one m64 x 2BN instruction, two partial accumulators
  bool halo = false;           // HALO form: one A load per (dy, channel slice) feeds the dx taps; needs split_k == 1
  bool pingpong = false;       // ping-pong kernel where the launch allows it (see tc_run); DUAL does not apply there
  bool pp_pair = false;        // the ping-pong launch may run on CTA pairs (see tc_make_launch); bh2 / bl2 have the BN/2-row box
  CUtensorMap bh2, bl2;
  bool ntail = false;          // batched GEMM whose N is not a multiple of BN: the last N tile is partial (never a convolution)
  int grid = 0;
  double flops = 0;            // algorithmic flops (2*M*N*K, counted once)
};

// Build the launch record.  src0/src1: fp16 split activations; w_hi/w_lo: [batch][Cout][Ktot] fp16 K-major with
// Ktot = taps*C0 + C1 (k index = tap*C0 + ci, then source-1 channels).
// invariant: batch-invariant launch — an output element's arithmetic depends only on its image and the layer's shape, not on
// the batch, the image's place in it or num_sms (no DUAL form, GroupNorm partials flushed per tile)
TcLaunch tc_make_launch(const SplitView& src0, int mode0, const SplitView* src1, const __half* w_hi, const __half* w_lo,
                        int w_batches, int Cout, const View& out, const float* chanadd, int ca_ld, const float* residual,
                        int ldr, float alpha, int num_sms, int res_mode = 0, bool invariant = false);
void tc_run(const TcLaunch& L, cudaStream_t stream);
// One parity phase (py, px) of conv3x3(nearest_upsample_x2(src)): src is the LOW-res split, w_* the phase's pre-summed
// [Cout][4*Cin] weights (see presum_up2_weights), out the FULL-res view; writes out[:, 2y+py, 2x+px, :].
TcLaunch tc_make_up2_launch(const SplitView& src, const __half* w_hi, const __half* w_lo, int Cout, const View& out, const float* chanadd,
                            int ca_ld, int py, int px, int num_sms, bool invariant = false);

// A convolution as it runs: one launch, or (S > 1, split-K) S CTAs per tile over disjoint k-block ranges into S partial buffers,
// then splitk_reduce (fixed-order sum + chanadd + residual + GroupNorm sums of `out`).
struct TcConvPlan {
  TcLaunch L;                   // S > 1: the partial launch, writing to `part` (see tc_set_partials)
  int S = 1;
  long long part_elems = 0;     // S > 1: floats of the partial buffer (S * pixels * Cout)
  float* part = nullptr;
  View out;
  const float* chanadd = nullptr;
  int ca_ld = 0;
  const float* residual = nullptr;
  int ldr = 0;
};
// The engine's convolution: tc_make_launch, and split-K where few tiles walk a long K (the 8x8 level).  split_k < 0: that rule
// (env DDNM_SPLITK=0 turns it off); 1, 2, 4: forced (res_mode 0 only).  A split plan needs tc_set_partials before it runs.
TcConvPlan tc_plan_conv(const SplitView& src0, int mode0, const SplitView* src1, const __half* w_hi, const __half* w_lo, int Cout,
                        const View& out, const float* chanadd, int ca_ld, const float* residual, int ldr, int res_mode, int num_sms,
                        bool invariant, int split_k = -1);
void tc_set_partials(TcConvPlan& plan, float* part);   // part: plan.part_elems floats
void tc_run_split_reduce(const TcConvPlan& plan, cudaStream_t stream);   // S > 1: the second launch of the plan
void tc_run_conv(const TcConvPlan& plan, cudaStream_t stream);           // the whole plan

// Strided fp16 (hi, lo) operand for the batched-GEMM builder: element (k, row, head, image) at
// base[k + row*s_row + head*s_head + image*s_img]; k extent = K (multiple of 8; base and strides 16-byte aligned).
struct GemmOperand {
  const __half* hi;
  const __half* lo;
  long long s_row, s_head, s_img;
};
// out[img*out_sn + head*out_sy + m*out_sx + n] = alpha * sum_k A[k, m, head, img] * B[k, n, head, img]
// (multi-head attention: QK^T and PV).  M % 128 == 0, N % 8 == 0, K % 8 == 0: a partial last k-block / N tile is zero-filled by
// TMA, and no column past N is stored.
TcLaunch tc_make_gemm_launch(const GemmOperand& A, const GemmOperand& B, int M, int N, int K, int heads, int images, float* out,
                             long long out_sn, long long out_sy, long long out_sx, float alpha, int num_sms, bool invariant = false);

// debug knobs (tests only): apply to the launches built afterwards
void tc_debug_force_bn(int bn);      // 0 (default): heuristic, 64 / 128: force the N tile where Cout (GEMM: N) allows it
void tc_debug_deal(int mode);        // -1 (default): contiguous tile ranges where they pay (one N tile + GroupNorm sums), 0 / 1: force
void tc_debug_dual_mode(int mode);   // 1 (default): DUAL form for conv_tc_kernel launches, 0: never
void tc_debug_halo(int on);          // 1 (default, env DDNM_HALO): HALO form wherever legal, 0: never
void tc_debug_pingpong(int on);      // 1 (default, env DDNM_PINGPONG): ping-pong kernel wherever it applies, 0: never
void tc_debug_pp_pair(int on);       // 1 (default, env DDNM_PP_PAIR): ping-pong launches on CTA pairs where legal, 0: single CTAs
// number of fp16 product terms used by launches built from now on (3 = parity mode, 1 = fast mode)
void tc_set_terms(int terms);
int tc_get_terms();

}  // namespace ddnm

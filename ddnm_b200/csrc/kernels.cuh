// SIMT (CUDA-core) kernels of the ddnm_b200 library: normalisation, fp16 splitting, small convolutions,
// timestep MLP, attention helpers, weight preparation.  All are HBM- or latency-bound; the FLOP-heavy
// contractions live in tc_gemm.cu.
#pragma once
#include "common.cuh"

namespace ddnm {

enum SplitMode : int { SPLIT_SAME = 0, SPLIT_S2D = 2, SPLIT_AVG2 = 3 };

// Per-channel GroupNorm sums of x into x.st (see View); only for tensors not produced by the tensor-core kernel.
void gn_stats(const View& x, cudaStream_t s);

// y = [GN affine](x) -> [SiLU] -> fp16 (hi, lo) planes.  normalise == false: raw split; true: uses x.st.
// mode SPLIT_S2D writes 4 parity phases
// (plane index = phase*N + n, phase = (y&1)*2 + (x&1)) for the stride-2 convolution, SPLIT_AVG2 writes the 2x2 average
// pool of the activated tensor (ResBlock(down=True), unet.py:237-241).  ss != nullptr: use_scale_shift_norm —
// y = GN(x) * (1 + ss[n*ss_ld + c]) + ss[n*ss_ld + C + c]   (unet.py:250-252).
void gn_apply_split(const View& x, int groups, bool normalise, const float* gamma, const float* beta, float eps,
                    bool silu, int mode, __half* hi, __half* lo, cudaStream_t s, const float* ss = nullptr, int ss_ld = 0,
                    __half* raw_hi = nullptr, __half* raw_lo = nullptr);  // raw_*: also emit the un-normalised split (SPLIT_SAME)
// same normalisation, fp32 contiguous NHWC output (feeds the small-Cout output convolution)
void gn_apply_f32(const View& x, int groups, const float* gamma, const float* beta, float eps, bool silu, float* out,
                  cudaStream_t s);

// 3x3 pad-1 convolution with tiny Cin (the network stem): x NCHW [N,Cin,H,W] fp32, w OIHW, out NHWC view.
// out = sum_k part[k] (fixed order) + chanadd + residual, with the GroupNorm sums of out (second half of a split-K convolution)
void splitk_reduce(const float* part, int S, long long stride, const View& out, const float* chanadd, int ca_ld, const float* residual, int ldr,
                   cudaStream_t s);
// network head in one pass: GroupNorm + SiLU + 3x3 convolution to Cout <= 8 channels in exact fp32 on the CUDA cores, NCHW output
bool head_conv_supported(const View& h, int Cout);
void head_conv(const View& h, int groups, const float* gamma, const float* beta, float eps, const float* w_oihw, const float* bias, int Cout,
               float* out_nchw, cudaStream_t s);
void conv3x3_small_cin(const float* x_nchw, int Cin, const float* w_oihw, const float* bias, const View& out, cudaStream_t s);
// stem of the super-resolution UNet: 3x3 pad-1 convolution of cat([x, bilinear_upsample(low_res)]) with 2C input channels.
// low_res != nullptr: x is [N,C,H,W], low_res [N,C,h,w] (h <= H, w <= W) is interpolated inside the kernel (nothing upsampled or
// concatenated is written); low_res == nullptr: x is the already concatenated [N,2C,H,W].  w OIHW [Cout,2C,3,3], out NHWC view.
void conv3x3_stem_sr(const float* x_nchw, const float* low_res_nchw, int C, int h, int w, const float* w_oihw, const float* bias,
                     const View& out, cudaStream_t s);
// out[n][o] = act_out( sum_k act_in(in[n][k]) * W[o][k] + bias[o] );  act: 0 none, 1 swish
void linear(const float* in, int N, int K, const float* W, const float* bias, int O, float* out, int ldo, int act_in,
            int act_out, cudaStream_t s);
// v[n][d] = swish(v[n][d] + table[labels[n]][d])  (UNetModel.forward: emb + label_emb(y), unet.py:651-653, then the blocks' SiLU);
// a label outside [0, num_classes) traps (nn.Embedding raises)
void add_label_swish(float* v, const float* table, const int* labels, int N, int D, int num_classes, cudaStream_t s);
// emb[n][:] = [sin(t*f) | cos(t*f)] (sin_first) or [cos | sin]; f has dim/2 entries
void sinusoid(const float* t, int N, const float* freq, int dim, bool sin_first, float* emb, cudaStream_t s);
// p[0..n) = v
void fill(float* p, int n, float v, cudaStream_t s);

// batched fp32 GEMM on CUDA cores (attention at small token counts).
//   NT: C[b][m][n] = alpha * sum_k A[b][m][k] * B[b][n][k];   NN: ... * B[b][k][n]
// Two-level batch (image, head): batch index b = outer*inner_n + inner; operand offset = outer*s? + inner*s?2.
void sgemm_batched(bool b_transposed, int outer_n, int inner_n, int M, int N, int K, float alpha, const float* A, int lda,
                   long long sa, long long sa2, const float* B, int ldb, long long sb, long long sb2, float* C, int ldc,
                   long long sc, long long sc2, cudaStream_t s);
void softmax_rows(float* x, long long rows, int cols, cudaStream_t s);
// softmax whose result is written as fp16 (hi, lo) planes (A operand of the tensor-core P.V GEMM)
void softmax_split(const float* x, long long rows, int cols, __half* hi, __half* lo, cudaStream_t s);
// per-head transposed fp16 split: dst[((img*heads + head)*ch + c)*T + t] = src[(img*T + t)*ld + head*head_stride + off + c]
void transpose_split(const float* src, int ld, int head_stride, int off, int images, int T, int heads, int ch, __half* hi,
                     __half* lo, cudaStream_t s);

// OIHW fp32 conv weight -> K-major fp16 (hi, lo) rows: dst[co*ktot + koff + tap*Cin + ci]
void split_conv_weight(const float* w_oihw, int Cout, int Cin, int taps, __half* hi, __half* lo, int ktot, int koff,
                       cudaStream_t s);

// 4 parity-phase weight matrices [4][Cout][4*Cin] (fp16 hi/lo) of conv3x3(nearest_upsample_x2(.)) from its OIHW 3x3 weight
void presum_up2_weights(const float* w_oihw, int Cout, int Cin, __half* hi, __half* lo, cudaStream_t s);

// Reference-quality direct convolution on CUDA cores (tests / validation of the tensor-core path only).
//   mode: TcTapMode; up2: input is nearest-upsampled 2x on the fly.  x, out: NHWC views; w: OIHW.
void conv_direct_ref(const View& x, const float* w_oihw, const float* bias, int taps_mode, bool up2, const View& out,
                     cudaStream_t s);

void nchw_to_nhwc(const float* src, int N, int C, int H, int W, const View& dst, cudaStream_t s);
void nhwc_to_nchw(const View& src, float* dst, cudaStream_t s);

}  // namespace ddnm

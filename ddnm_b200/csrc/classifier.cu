// UNetEncoder: launch program for guided_diffusion/unet.py::EncoderUNetModel (unet.py:684-895, the classifier of
// imagenet_256_cc.yml built by script_util.create_classifier) and for the gradient its cond_fn takes with autograd
// (diffusion.py:183-189): grad = scale * d/dx sum_b log_softmax(logits)[b, y_b].  Forward and backward are one op list.
//
// Backward structure (parameters and t get no gradient):
//   head       dlogits = onehot(y) - softmax(logits) (times GRAD_SCALE, see there); c_proj^T; attention-pool backward (only token 0's query reaches
//              the output); qkv_proj^T; the mean token's gradient spread over the pixels; out-GroupNorm + SiLU backward
//   ResBlock   conv2^T and skip^T on the tensor cores (3x3 weights flipped with Cin/Cout swapped, 1x1 transposed); GroupNorm
//              (+ scale-shift) + SiLU backward; conv1^T; GroupNorm + SiLU (+ avg-pool) backward that also adds the skip gradient
//   Attention  proj_out^T; softmax(QK^T) recomputed from the kept qkv; dV, dP, dS, dQ, dK on CUDA cores; qkv^T; GroupNorm
//              backward + the residual
//   stem       3x3, Cout -> 3 channels on CUDA cores, NCHW result
// The GroupNorm reductions are per-CTA partial sums combined in a fixed order (no floating-point atomics), so a gradient is
// bit-reproducible run to run.
#include <algorithm>
#include <cmath>

#include "engine.cuh"
#include "kernels.cuh"

namespace ddnm {

// ---------------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------------

// data-gradient weights: 3x3 w[co][ci][ky][kx] -> wt[ci][co][2-ky][2-kx]; 1x1 w[co][ci] -> wt[ci][co]
__global__ void flip_transpose_kernel(const float* __restrict__ w, int Cout, int Cin, int taps, float* __restrict__ wt) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = (long long)Cout * Cin * taps;
  if (i >= n) return;
  const int tap = (int)(i % taps);
  const long long r = i / taps;
  const int ci = (int)(r % Cin), co = (int)(r / Cin);
  wt[((long long)ci * Cout + co) * taps + (taps - 1 - tap)] = w[i];
}

// GroupNorm backward.  u = GN(x) * (1 + scale) + shift (the affine of gn_apply_kernel), z = SiLU(u) (or u), optionally
// average-pooled 2x2; g = dL/dz at z's resolution.  With g_u = dL/du and xh = (x - mean) * rstd:
//   dL/dx = rstd * (g_u*gamma' - mean_G(g_u*gamma') - xh * mean_G(g_u*gamma'*xh)),   gamma' = gamma * (1 + scale)
// The two group means come from per-(CTA, channel) partial sums (gnb_reduce_kernel) that gnb_combine_kernel adds in a fixed
// order.  A CTA walks a chunk of pixels of one image with 512 / C threads per channel (C <= 512).
struct GnbArgs {
  const float* g;
  const float* x;
  int H, W, C, ld;
  const StatAcc* st;
  int st_ld, groups;
  float eps;
  const float *gamma, *beta, *ss;
  int ss_ld, silu, pool, ppc, chunks;
};

struct GnbCoef { float mean, rstd, a, b, gp; };   // u = x * a + b, gp = gamma'

__device__ __forceinline__ GnbCoef gnb_coef(const GnbArgs& A, int n, int c) {
  const int cpg = A.C / A.groups, g0 = (c / cpg) * cpg;
  const StatAcc* s = A.st + (size_t)n * A.st_ld * 2;
  double s1 = 0, s2 = 0;
  for (int j = 0; j < cpg; ++j) {
    s1 += stat_value(s[2 * (g0 + j)]);
    s2 += stat_value(s[2 * (g0 + j) + 1]);
  }
  const double cnt = (double)A.H * A.W * cpg;
  const double mean = s1 / cnt;
  double var = s2 / cnt - mean * mean;
  var = var < 0 ? 0 : var;
  GnbCoef k;
  k.mean = (float)mean;
  k.rstd = (float)(1.0 / sqrt(var + (double)A.eps));
  float a = k.rstd * A.gamma[c], b = A.beta[c] - k.mean * a, gp = A.gamma[c];
  if (A.ss) {
    const float one_plus = 1.0f + A.ss[(size_t)n * A.ss_ld + c];
    a *= one_plus;
    b = fmaf(b, one_plus, A.ss[(size_t)n * A.ss_ld + A.C + c]);
    gp *= one_plus;
  }
  k.a = a;
  k.b = b;
  k.gp = gp;
  return k;
}

// dL/du at pixel p (full resolution) of image n, channel c; also returns xh
__device__ __forceinline__ float gnb_gu(const GnbArgs& A, const GnbCoef& k, int n, int p, int c, float& xh) {
  const float xv = A.x[((size_t)n * A.H * A.W + p) * A.ld + c];
  xh = (xv - k.mean) * k.rstd;
  float g;
  if (A.pool) {
    const int y = p / A.W, xx = p - y * A.W, Wo = A.W >> 1;
    g = 0.25f * A.g[(((size_t)n * (A.H >> 1) + (y >> 1)) * Wo + (xx >> 1)) * A.C + c];
  } else {
    g = A.g[((size_t)n * A.H * A.W + p) * A.C + c];
  }
  if (A.silu) {
    const float u = fmaf(xv, k.a, k.b);
    const float sg = 1.0f / (1.0f + expf(-u));
    g *= sg * (1.0f + u * (1.0f - sg));
  }
  return g;
}

// Threads are (channel c, pixel row r): R = blockDim.x / C threads share a channel and take every R-th pixel of the CTA's chunk;
// their partial sums are added in row order.
__global__ void gnb_reduce_kernel(GnbArgs A, double* __restrict__ part) {
  extern __shared__ double gnb_red[];   // [R][C][2]
  const int n = blockIdx.y, chunk = blockIdx.x, HW = A.H * A.W;
  const int c = threadIdx.x % A.C, r = threadIdx.x / A.C, R = blockDim.x / A.C;
  const int p0 = chunk * A.ppc, p1 = min(HW, p0 + A.ppc);
  const GnbCoef k = gnb_coef(A, n, c);
  double s1 = 0, s2 = 0;
  for (int p = p0 + r; p < p1; p += R) {
    float xh;
    const float d = gnb_gu(A, k, n, p, c, xh) * k.gp;
    s1 += d;
    s2 += (double)d * xh;
  }
  gnb_red[(r * A.C + c) * 2] = s1;
  gnb_red[(r * A.C + c) * 2 + 1] = s2;
  __syncthreads();
  if (r == 0) {
    for (int rr = 1; rr < R; ++rr) {
      s1 += gnb_red[(rr * A.C + c) * 2];
      s2 += gnb_red[(rr * A.C + c) * 2 + 1];
    }
    double* o = part + (((size_t)n * A.chunks + chunk) * A.C + c) * 2;
    o[0] = s1;
    o[1] = s2;
  }
}

// tot[n][c] = sum over the chunks' partials in chunk order (one thread per (image, channel))
__global__ void gnb_combine_kernel(const double* __restrict__ part, int chunks, int C, double* __restrict__ tot) {
  const int n = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double s1 = 0, s2 = 0;
    for (int j = 0; j < chunks; ++j) {
      const double* o = part + (((size_t)n * chunks + j) * C + c) * 2;
      s1 += o[0];
      s2 += o[1];
    }
    tot[((size_t)n * C + c) * 2] = s1;
    tot[((size_t)n * C + c) * 2 + 1] = s2;
  }
}

__global__ void gnb_apply_kernel(GnbArgs A, const double* __restrict__ tot, const float* __restrict__ add, int add_pool,
                                 float* __restrict__ dx32, __half* __restrict__ hi, __half* __restrict__ lo) {
  const int n = blockIdx.y, chunk = blockIdx.x, HW = A.H * A.W;
  const int c = threadIdx.x % A.C, r = threadIdx.x / A.C, R = blockDim.x / A.C;
  const int cpg = A.C / A.groups, g0 = (c / cpg) * cpg;
  const double cnt = (double)HW * cpg;
  double m1 = 0, m2 = 0;
  for (int j = 0; j < cpg; ++j) {
    m1 += tot[((size_t)n * A.C + g0 + j) * 2];
    m2 += tot[((size_t)n * A.C + g0 + j) * 2 + 1];
  }
  const float M1 = (float)(m1 / cnt), M2 = (float)(m2 / cnt);
  const GnbCoef k = gnb_coef(A, n, c);
  const int p0 = chunk * A.ppc, p1 = min(HW, p0 + A.ppc);
  for (int p = p0 + r; p < p1; p += R) {
    float xh;
    const float d = gnb_gu(A, k, n, p, c, xh) * k.gp;
    float v = k.rstd * (d - M1 - xh * M2);
    if (add) {
      if (add_pool) {
        const int y = p / A.W, xx = p - y * A.W, Wo = A.W >> 1;
        v += 0.25f * add[(((size_t)n * (A.H >> 1) + (y >> 1)) * Wo + (xx >> 1)) * A.C + c];
      } else {
        v += add[((size_t)n * HW + p) * A.C + c];
      }
    }
    const size_t o = ((size_t)n * HW + p) * A.C + c;
    if (dx32) dx32[o] = v;
    split_f16(v, hi[o], lo[o]);
  }
}

// Strided batched fp32 GEMM: C[m][n] (+)= alpha * sum_k A[m*am + k*ak] * B[k*bk + n*bn] (+ bias[n]), batch z = outer*inner + i
// with operand offsets outer*s?o + i*s?i.  64x64 tiles, 4x4 outputs per thread.
__global__ void __launch_bounds__(256) bgemm_kernel(int M, int N, int K, float alpha, const float* __restrict__ A, long long am, long long ak,
                                                    long long sao, long long sai, const float* __restrict__ B, long long bk, long long bn,
                                                    long long sbo, long long sbi, float* __restrict__ Cm, long long cm, long long sco,
                                                    long long sci, int inner, const float* __restrict__ bias) {
  constexpr int SK = 16;
  __shared__ float As[SK][64 + 4], Bs[SK][64 + 4];
  const int bo = blockIdx.z / inner, bi = blockIdx.z % inner;
  A += bo * sao + bi * sai;
  B += bo * sbo + bi * sbi;
  Cm += bo * sco + bi * sci;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += SK) {
    for (int i = threadIdx.x; i < 64 * SK; i += 256) {
      int mm, kk;
      if (am == 1) { mm = i % 64; kk = i / 64; } else { kk = i % SK; mm = i / SK; }
      As[kk][mm] = (m0 + mm < M && k0 + kk < K) ? A[(m0 + mm) * am + (k0 + kk) * ak] : 0.f;
      int nn, kb;
      if (bn == 1) { nn = i % 64; kb = i / 64; } else { kb = i % SK; nn = i / SK; }
      Bs[kb][nn] = (n0 + nn < N && k0 + kb < K) ? B[(k0 + kb) * bk + (n0 + nn) * bn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < SK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + j;
      if (m < M && n < N) Cm[(long long)m * cm + n] = alpha * acc[i][j] + (bias ? bias[n] : 0.f);
    }
}

static void bgemm(int outer, int inner, int M, int N, int K, float alpha, const float* A, long long am, long long ak, long long sao,
                  long long sai, const float* B, long long bk, long long bn, long long sbo, long long sbi, float* Cm, long long cm,
                  long long sco, long long sci, const float* bias, cudaStream_t s) {
  dim3 grid(cdiv(N, 64), cdiv(M, 64), outer * inner);
  DDNM_CHECK(grid.z <= 65535, "too many GEMM batches for one launch");
  bgemm_kernel<<<grid, 256, 0, s>>>(M, N, K, alpha, A, am, ak, sao, sai, B, bk, bn, sbo, sbi, Cm, cm, sco, sci, inner, bias);
  CUDA_CHECK(cudaGetLastError());
}

// dS = P * (dP - rowsum(dP * P)) in place over dP, one warp per row (softmax backward)
__global__ void softmax_bwd_kernel(const float* __restrict__ P, float* __restrict__ dP, long long rows, int cols) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* p = P + row * cols;
  float* d = dP + row * cols;
  float s = 0.f;
  for (int i = lane; i < cols; i += 32) s += p[i] * d[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  for (int i = lane; i < cols; i += 32) d[i] = p[i] * (d[i] - s);
}

// head tokens: tok[n][0][c] = mean_p hf[n][p][c] (+ pos[c][0]); tok[n][1 + p][c] = hf[n][p][c] + pos[c][1 + p] (T > 1)
__global__ void pool_tokens_kernel(const float* __restrict__ hf, int HW, int C, const float* __restrict__ pos, int T,
                                   float* __restrict__ tok) {
  const int n = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int p = 0; p < HW; ++p) {
      const float v = hf[((size_t)n * HW + p) * C + c];
      s += v;
      if (T > 1) tok[((size_t)n * T + 1 + p) * C + c] = v + pos[(size_t)c * T + 1 + p];
    }
    tok[(size_t)n * T * C + c] = s / (float)HW + (pos ? pos[(size_t)c * T] : 0.f);
  }
}

// QKVAttention (unet.py:357-393) for token 0's query only: qkv [n][t][3C] = [q | k | v], head h = columns h*ch + c of each.
// p[n][h][t] = softmax_t(alpha q0 . k_t), a0[n][h*ch + c] = sum_t p_t v_t[c]
__global__ void pool_attn_fwd_kernel(const float* __restrict__ qkv, int T, int C, int ch, float alpha, float* __restrict__ P,
                                     float* __restrict__ a0) {
  extern __shared__ float pa_sm[];   // q0[ch], p[T]
  const int n = blockIdx.x, h = blockIdx.y, heads = gridDim.y;
  float *q0 = pa_sm, *p = pa_sm + ch;
  const float* base = qkv + (size_t)n * T * 3 * C;
  for (int c = threadIdx.x; c < ch; c += blockDim.x) q0[c] = base[h * ch + c];
  __syncthreads();
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    const float* k = base + (size_t)t * 3 * C + C + h * ch;
    float s = 0.f;
    for (int c = 0; c < ch; ++c) s = fmaf(q0[c], k[c], s);
    p[t] = s * alpha;
  }
  __syncthreads();
  if (threadIdx.x == 0) {   // T <= a few hundred: one thread, fixed order
    float m = -INFINITY;
    for (int t = 0; t < T; ++t) m = fmaxf(m, p[t]);
    float s = 0.f;
    for (int t = 0; t < T; ++t) { p[t] = expf(p[t] - m); s += p[t]; }
    const float inv = 1.0f / s;
    for (int t = 0; t < T; ++t) p[t] *= inv;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < T; t += blockDim.x) P[((size_t)n * heads + h) * T + t] = p[t];
  for (int c = threadIdx.x; c < ch; c += blockDim.x) {
    float s = 0.f;
    for (int t = 0; t < T; ++t) s = fmaf(p[t], base[(size_t)t * 3 * C + 2 * C + h * ch + c], s);
    a0[(size_t)n * C + h * ch + c] = s;
  }
}

// backward of pool_attn_fwd_kernel: da0 [n][C] -> dqkv [n][t][3C] (dq is non-zero for token 0 only)
__global__ void pool_attn_bwd_kernel(const float* __restrict__ qkv, const float* __restrict__ P, const float* __restrict__ da0, int T, int C,
                                     int ch, float alpha, float* __restrict__ dqkv) {
  extern __shared__ float pb_sm[];   // q0[ch], da[ch], p[T], ds[T]
  const int n = blockIdx.x, h = blockIdx.y, heads = gridDim.y;
  float *q0 = pb_sm, *da = q0 + ch, *p = da + ch, *ds = p + T;
  __shared__ float red;
  const float* base = qkv + (size_t)n * T * 3 * C;
  float* dbase = dqkv + (size_t)n * T * 3 * C;
  for (int c = threadIdx.x; c < ch; c += blockDim.x) {
    q0[c] = base[h * ch + c];
    da[c] = da0[(size_t)n * C + h * ch + c];
  }
  for (int t = threadIdx.x; t < T; t += blockDim.x) p[t] = P[((size_t)n * heads + h) * T + t];
  __syncthreads();
  for (int t = threadIdx.x; t < T; t += blockDim.x) {   // dp_t = da . v_t
    const float* v = base + (size_t)t * 3 * C + 2 * C + h * ch;
    float s = 0.f;
    for (int c = 0; c < ch; ++c) s = fmaf(da[c], v[c], s);
    ds[t] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int t = 0; t < T; ++t) s += p[t] * ds[t];
    red = s;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < T; t += blockDim.x) ds[t] = alpha * p[t] * (ds[t] - red);
  __syncthreads();
  for (int i = threadIdx.x; i < T * ch; i += blockDim.x) {
    const int t = i / ch, c = i - t * ch;
    float* d = dbase + (size_t)t * 3 * C + h * ch + c;
    d[C] = ds[t] * q0[c];          // dk_t
    d[2 * C] = p[t] * da[c];       // dv_t
    if (t) d[0] = 0.f;
  }
  for (int c = threadIdx.x; c < ch; c += blockDim.x) {   // dq_0 = sum_t ds_t k_t
    float s = 0.f;
    for (int t = 0; t < T; ++t) s = fmaf(ds[t], base[(size_t)t * 3 * C + C + h * ch + c], s);
    dbase[h * ch + c] = s;
  }
}

// dhf[n][p][c] = dX[n][1 + p][c] (T > 1) + dX[n][0][c] / HW   (token 0 is the mean of the pixel tokens)
__global__ void pool_spread_kernel(const float* __restrict__ dX, int T, int HW, int C, float* __restrict__ dhf, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C);
  const long long r = i / C;
  const int p = (int)(r % HW), n = (int)(r / HW);
  float v = dX[(size_t)n * T * C + c] / (float)HW;
  if (T > 1) v += dX[((size_t)n * T + 1 + p) * C + c];
  dhf[i] = v;
}

// The backward pass carries GRAD_SCALE * dL/d(.) with L = sum_b log_softmax(logits)[b, y_b]: the gradients of a classifier are small
// (1e-3 .. 1e-6 per element), below the fp16 normal range (6.1e-5) where the (hi, lo) split of the data-gradient convolutions loses
// its low word.  The power-of-two factor is exact; the stem backward multiplies by scale / GRAD_SCALE.
constexpr float GRAD_SCALE = 1024.0f;

// dlogits[n][o] = GRAD_SCALE * (onehot(labels[n]) - softmax(logits[n]))   (d/dlogits of log_softmax(logits)[n, y_n])
__global__ void dlogits_kernel(const float* __restrict__ logits, const int* __restrict__ labels, int O, float* __restrict__ dl) {
  __shared__ float red[32];
  const int n = blockIdx.x;
  const float* l = logits + (size_t)n * O;
  float m = -INFINITY;
  for (int o = threadIdx.x; o < O; o += blockDim.x) m = fmaxf(m, l[o]);
  for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = -INFINITY;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m = fmaxf(m, red[w]);
  __syncthreads();
  float s = 0.f;
  for (int o = threadIdx.x; o < O; o += blockDim.x) s += expf(l[o] - m);
  for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  s = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
  const float inv = 1.0f / s;
  const int y = labels[n];
  for (int o = threadIdx.x; o < O; o += blockDim.x) dl[(size_t)n * O + o] = GRAD_SCALE * ((o == y ? 1.f : 0.f) - expf(l[o] - m) * inv);
}

// stem backward: dx[n][ci][y][x] = sum_{co,ky,kx} w[co][ci][ky][kx] * g[n][y+1-ky][x+1-kx][co]; w staged in shared memory
template <int CIN>
__global__ void __launch_bounds__(128) stem_bwd_kernel(const float* __restrict__ g, int N, int H, int W, int Co, const float* __restrict__ w,
                                                       const float* __restrict__ scale, float* __restrict__ dx) {
  extern __shared__ float sw[];   // [tap][co][ci]
  for (int i = threadIdx.x; i < Co * CIN * 9; i += blockDim.x) {
    const int tap = i % 9, ci = (i / 9) % CIN, co = i / (9 * CIN);
    sw[((size_t)tap * Co + co) * CIN + ci] = w[i];
  }
  __syncthreads();
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long long)N * H * W) return;
  const int x = (int)(pix % W), y = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
  float acc[CIN] = {};
  for (int ky = 0; ky < 3; ++ky) {
    const int yy = y + 1 - ky;
    if (yy < 0 || yy >= H) continue;
    for (int kx = 0; kx < 3; ++kx) {
      const int xx = x + 1 - kx;
      if (xx < 0 || xx >= W) continue;
      const float4* gp = reinterpret_cast<const float4*>(g + (((size_t)n * H + yy) * W + xx) * Co);
      const float* wp = sw + (size_t)(ky * 3 + kx) * Co * CIN;
      for (int c4 = 0; c4 < Co / 4; ++c4) {
        const float4 v = __ldg(gp + c4);
        const float gv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int ci = 0; ci < CIN; ++ci) acc[ci] = fmaf(wp[(c4 * 4 + j) * CIN + ci], gv[j], acc[ci]);
      }
    }
  }
  const float sc = *scale / GRAD_SCALE;
#pragma unroll
  for (int ci = 0; ci < CIN; ++ci) dx[(((size_t)n * CIN + ci) * H + y) * W + x] = acc[ci] * sc;
}

// ---------------------------------------------------------------------------------------------------------------
// program
// ---------------------------------------------------------------------------------------------------------------

UNetEncoder::UNetEncoder(const EncoderCfg& cfg, int batch)
    : UNetEngine(batch, cfg.in_channels, cfg.out_channels, cfg.image_size, cfg.groups, cfg.eps), cfg_(cfg) {
  DDNM_CHECK(cfg.pool == 0 || cfg.pool == 1, "pool must be 'adaptive' or 'attention'");
  DDNM_CHECK(cfg.in_channels == 3, "the classifier reads 3-channel images");
  DDNM_CHECK(cfg.out_channels >= 1, "bad out_channels");
}

UNetEncoder::~UNetEncoder() {
  if (ggraph_exec_) cudaGraphExecDestroy(ggraph_exec_);
  if (ggraph_) cudaGraphDestroy(ggraph_);
}

UNetEngine::TcWeights UNetEncoder::prep_weights_t(const std::string& name, int Cout, int Cin, int taps) {
  const long long n = (long long)Cout * Cin * taps;
  const float* w = P(name, n);
  float* wt = nullptr;
  CUDA_CHECK(cudaMalloc(&wt, (size_t)n * sizeof(float)));
  flip_transpose_kernel<<<(int)cdivll(n, 256), 256>>>(w, Cout, Cin, taps, wt);
  CUDA_CHECK(cudaGetLastError());
  TcWeights r;
  r.ktot = taps * Cout;
  r.hi = (__half*)arena_.alloc((size_t)n * sizeof(__half));
  r.lo = (__half*)arena_.alloc((size_t)n * sizeof(__half));
  split_conv_weight(wt, Cin, Cout, taps, r.hi, r.lo, r.ktot, 0, 0);
  CUDA_CHECK(cudaDeviceSynchronize());
  CUDA_CHECK(cudaFree(wt));
  return r;
}

// GroupNorm backward chunks per image in batch-invariant mode (256^2: 1024 pixels each; 8 images fill 4 CTAs per SM as the default does)
static constexpr int kGnbInvariantChunks = 64;

void UNetEncoder::emit_gn_backward(const std::string& name, const float* g, const View& x, const std::string& norm, const float* ss, int ss_ld,
                                   bool silu, bool pool, const float* add, bool add_pool, float* dx32, const SplitView& dst) {
  DDNM_CHECK(x.st != nullptr && x.C % groups_ == 0 && x.C <= 512, "GroupNorm backward: input without statistics / too wide");
  DDNM_CHECK((size_t)x.pixels() * x.C <= split_elems_, "split scratch too small");
  GnbArgs A;
  A.g = g; A.x = x.p; A.H = x.H; A.W = x.W; A.C = x.C; A.ld = x.ld; A.st = x.st; A.st_ld = x.st_ld; A.groups = groups_; A.eps = eps_;
  A.gamma = P(norm + ".weight", x.C);
  A.beta = P(norm + ".bias", x.C);
  A.ss = ss; A.ss_ld = ss_ld; A.silu = silu; A.pool = pool;
  const int HW = x.H * x.W;
  // pixel chunks per image: about 4 CTAs per SM over the batch; in batch-invariant mode a fixed count, since the chunks' fp64
  // partial sums (and so the gradient's last bits) follow the partition
  int chunks = std::max(1, std::min(HW, invariant_ ? kGnbInvariantChunks : cdiv(4 * num_sms_, B_)));
  A.ppc = cdiv(HW, chunks);
  A.chunks = chunks = cdiv(HW, A.ppc);
  DDNM_CHECK((size_t)B_ * (chunks + 1) * x.C * 2 <= gnb_part_elems_, "GroupNorm backward partial buffer too small");
  double* part = (double*)gnb_part_;
  double* tot = part + (size_t)B_ * chunks * x.C * 2;
  const int threads = x.C * std::max(1, 512 / x.C);
  const int Bn = B_;
  __half *hi = dst.hi, *lo = dst.lo;
  const double bytes = (double)x.pixels() * x.C * 4 * (2 + (add ? 1 : 0) + (dx32 ? 1 : 0)) + (double)x.pixels() * x.C * 4;
  add_op(name, "gn_bwd", 0, bytes, [=](cudaStream_t s) {
    gnb_reduce_kernel<<<dim3(chunks, Bn), threads, (size_t)threads * 16, s>>>(A, part);
    gnb_combine_kernel<<<Bn, A.C, 0, s>>>(part, chunks, A.C, tot);
    gnb_apply_kernel<<<dim3(chunks, Bn), threads, 0, s>>>(A, tot, add, add_pool ? 1 : 0, dx32, hi, lo);
    CUDA_CHECK(cudaGetLastError());
  });
}

// self.out (unet.py:853-871): GroupNorm + SiLU, then AttentionPool2d (unet.py:20-50) or mean + 1x1 convolution
void UNetEncoder::emit_head(const View& h) {
  const int C = h.C, HW = h.H * h.W, O = cfg_.out_channels, Bn = B_;
  const float *g = P("out.0.weight", C), *b = P("out.0.bias", C);
  const int groups = groups_;
  const float eps = eps_;
  const View hv = h;
  float *hf = hf_, *tok = tok_, *logits = out_;
  if (cfg_.pool == 1) {
    const int T = headT_, ch = cfg_.num_head_channels, heads = C / ch;
    DDNM_CHECK(C % ch == 0 && T == HW + 1, "attention pool shape");
    const float* pos = P("out.2.positional_embedding", (long long)C * T);
    const float *wq = P("out.2.qkv_proj.weight", 3LL * C * C), *bq = P("out.2.qkv_proj.bias", 3 * C);
    const float *wc = P("out.2.c_proj.weight", (long long)O * C), *bc = P("out.2.c_proj.bias", O);
    float *qkv = hqkv_, *pr = hp_, *a0 = ha0_;
    const float alpha = 1.0f / std::sqrt((float)ch);
    add_op("head.pool", "head", 2.0 * Bn * T * 3.0 * C * C + 2.0 * Bn * O * C, (double)Bn * (HW * C + 3.0 * C * C + O * C) * 4, [=](cudaStream_t s) {
      gn_apply_f32(hv, groups, g, b, eps, true, hf, s);
      pool_tokens_kernel<<<Bn, std::min(C, 512), 0, s>>>(hf, HW, C, pos, T, tok);
      CUDA_CHECK(cudaGetLastError());
      // qkv[n][t][o] = sum_c tok[n][t][c] W[o][c] + b[o]   (Conv1d weight (3C, C, 1))
      bgemm(Bn, 1, T, 3 * C, C, 1.0f, tok, C, 1, (long long)T * C, 0, wq, 1, C, 0, 0, qkv, 3 * C, (long long)T * 3 * C, 0, bq, s);
      pool_attn_fwd_kernel<<<dim3(Bn, heads), 128, (size_t)(ch + T) * 4, s>>>(qkv, T, C, ch, alpha, pr, a0);
      CUDA_CHECK(cudaGetLastError());
      linear(a0, Bn, C, wc, bc, O, logits, O, 0, 0, s);
    });
  } else {
    const float *wc = P("out.3.weight", (long long)O * C), *bc = P("out.3.bias", O);
    add_op("head.pool", "head", 2.0 * Bn * O * C, (double)Bn * (HW * C + O * C) * 4, [=](cudaStream_t s) {
      gn_apply_f32(hv, groups, g, b, eps, true, hf, s);
      pool_tokens_kernel<<<Bn, std::min(C, 512), 0, s>>>(hf, HW, C, nullptr, 1, tok);
      CUDA_CHECK(cudaGetLastError());
      linear(tok, Bn, C, wc, bc, O, logits, O, 0, 0, s);
    });
  }
}

void UNetEncoder::emit_backward(const View& stem_out, const std::vector<Layer>& layers, const View& top) {
  const int Bn = B_, O = cfg_.out_channels;
  SplitView SA{splitA_hi_, splitA_lo_}, SB{splitB_hi_, splitB_lo_};
  float* G[2] = {gx_[0], gx_[1]};
  auto with_dims = [](SplitView s, const View& v) {
    s.N = v.N; s.H = v.H; s.W = v.W; s.C = v.C;
    return s;
  };
  // ---- head ----
  {
    const int C = top.C, HW = top.H * top.W, T = cfg_.pool == 1 ? headT_ : 1;
    const float* logits = out_;
    const int* labels = labels_in_;
    float *dl = g2_, *da0 = g2_ + (size_t)Bn * O, *dX = g1_, *dhf = gqkv_, *dqkv = gx_[1];
    const float* wc = cfg_.pool == 1 ? P("out.2.c_proj.weight", (long long)O * C) : P("out.3.weight", (long long)O * C);
    const float* wq = cfg_.pool == 1 ? P("out.2.qkv_proj.weight", 3LL * C * C) : nullptr;
    float *qkv = hqkv_, *pr = hp_;
    const int ch = cfg_.num_head_channels, heads = C / ch;
    const float alpha = 1.0f / std::sqrt((float)ch);
    const int pool = cfg_.pool;
    add_op("head.bwd", "head", 2.0 * Bn * O * C + (pool ? 2.0 * Bn * T * 3.0 * C * C : 0), (double)Bn * (HW * C + 3.0 * C * C + O * C) * 4,
           [=](cudaStream_t s) {
             dlogits_kernel<<<Bn, 256, 0, s>>>(logits, labels, O, dl);
             CUDA_CHECK(cudaGetLastError());
             // da0[n][c] = sum_o dl[n][o] Wc[o][c]
             float* dtok0 = pool ? da0 : dX;
             bgemm(1, 1, Bn, C, O, 1.0f, dl, O, 1, 0, 0, wc, C, 1, 0, 0, dtok0, C, 0, 0, nullptr, s);
             if (pool) {
               pool_attn_bwd_kernel<<<dim3(Bn, heads), 128, (size_t)(2 * ch + 2 * T) * 4, s>>>(qkv, pr, da0, T, C, ch, alpha, dqkv);
               CUDA_CHECK(cudaGetLastError());
               // dX[n][t][c] = sum_o dqkv[n][t][o] Wq[o][c]
               bgemm(Bn, 1, T, C, 3 * C, 1.0f, dqkv, 3 * C, 1, (long long)T * 3 * C, 0, wq, C, 1, 0, 0, dX, C, (long long)T * C, 0, nullptr, s);
             }
             const long long total = (long long)Bn * HW * C;
             pool_spread_kernel<<<(int)cdivll(total, 256), 256, 0, s>>>(dX, T, HW, C, dhf, total);
             CUDA_CHECK(cudaGetLastError());
           });
    emit_gn_backward("head.out_norm.bwd", dhf, top, "out.0", nullptr, 0, true, false, nullptr, false, G[0], SB);
  }
  // ---- blocks, last to first; G[0] holds dL/d(block output) and SB its split ----
  for (int li = (int)layers.size() - 1; li >= 0; --li) {
    const Layer& L = layers[li];
    if (L.kind == 0) {
      const Res& r = L.r;
      const int Cin = r.x.C, Cout = r.out.C;
      const SplitView sb = with_dims(SB, r.out);
      TcWeights w2 = prep_weights_t(r.p + ".out_layers.3.weight", Cout, Cout, 9);
      emit_tc(r.p + ".conv2.dgrad", sb, TAPS_3X3, nullptr, w2, Cout, view_of(g1_, r.out.H, r.out.W, Cout), nullptr, 0, nullptr, 0);
      const float* add = G[0];
      bool add_pool = r.down;
      if (r.skip_conv) {
        TcWeights ws = prep_weights_t(r.p + ".skip_connection.weight", Cout, Cin, 1);
        emit_tc(r.p + ".skip.dgrad", sb, TAPS_1X1, nullptr, ws, Cin, view_of(g2_, r.x.H, r.x.W, Cin), nullptr, 0, nullptr, 0);
        add = g2_;
        add_pool = false;
      }
      emit_gn_backward(r.p + ".out_norm.bwd", g1_, r.h, r.p + ".out_layers.0", emb_rows(r.p), emb_ld_, true, false, nullptr,
                       false, nullptr, SA);
      TcWeights w1 = prep_weights_t(r.p + ".in_layers.2.weight", Cout, Cin, 9);
      emit_tc(r.p + ".conv1.dgrad", with_dims(SA, r.h), TAPS_3X3, nullptr, w1, Cin, view_of(g1_, r.out.H, r.out.W, Cin), nullptr, 0,
              nullptr, 0);
      emit_gn_backward(r.p + ".in_norm.bwd", g1_, r.x, r.p + ".in_layers.0", nullptr, 0, true, r.down, add, add_pool, G[1], SB);
    } else {
      const Attn& a = L.a;
      const int C = a.x.C, T = a.x.H * a.x.W, ch = cfg_.num_head_channels, heads = C / ch;
      TcWeights wp = prep_weights_t(a.p + ".proj_out.weight", C, C, 1);
      emit_tc(a.p + ".proj_out.dgrad", with_dims(SB, a.out), TAPS_1X1, nullptr, wp, C, view_of(g1_, a.x.H, a.x.W, C), nullptr, 0, nullptr, 0);
      {
        const float *qkv = a.qkv, *dA = g1_;
        float *Pm = sP_, *dP = sdP_, *dq = gqkv_;
        const float alpha = 1.0f / std::sqrt((float)ch);
        const long long q3 = 3LL * C, img = (long long)T * q3, hs = (long long)T * T;
        add_op(a.p + ".attn.bwd", "sgemm", 2.0 * Bn * heads * (double)T * T * ch * 5, (double)Bn * heads * T * T * 4 * 4, [=](cudaStream_t s) {
          // P = softmax(alpha Q K^T), recomputed from the kept qkv
          bgemm(Bn, heads, T, T, ch, alpha, qkv, q3, 1, img, 3 * ch, qkv + ch, 1, q3, img, 3 * ch, Pm, T, heads * hs, hs, nullptr, s);
          softmax_rows(Pm, (long long)Bn * heads * T, T, s);
          // dP = dA V^T
          bgemm(Bn, heads, T, T, ch, 1.0f, dA, C, 1, (long long)T * C, ch, qkv + 2 * ch, 1, q3, img, 3 * ch, dP, T, heads * hs, hs, nullptr, s);
          // dV = P^T dA
          bgemm(Bn, heads, T, ch, T, 1.0f, Pm, 1, T, heads * hs, hs, dA, C, 1, (long long)T * C, ch, dq + 2 * ch, q3, img, 3 * ch, nullptr, s);
          softmax_bwd_kernel<<<(int)cdivll((long long)Bn * heads * T * 32, 256), 256, 0, s>>>(Pm, dP, (long long)Bn * heads * T, T);
          CUDA_CHECK(cudaGetLastError());
          // dQ = alpha dS K,  dK = alpha dS^T Q
          bgemm(Bn, heads, T, ch, T, alpha, dP, T, 1, heads * hs, hs, qkv + ch, q3, 1, img, 3 * ch, dq, q3, img, 3 * ch, nullptr, s);
          bgemm(Bn, heads, T, ch, T, alpha, dP, 1, T, heads * hs, hs, qkv, q3, 1, img, 3 * ch, dq + ch, q3, img, 3 * ch, nullptr, s);
        });
      }
      View gq = view_of(gqkv_, a.x.H, a.x.W, 3 * C);
      SplitView sq = SA;
      emit_gn_split(a.p + ".dqkv.split", gq, "", false, SPLIT_SAME, sq);
      TcWeights wq = prep_weights_t(a.p + ".qkv.weight", 3 * C, C, 1);
      emit_tc(a.p + ".qkv.dgrad", sq, TAPS_1X1, nullptr, wq, C, view_of(g1_, a.x.H, a.x.W, C), nullptr, 0, nullptr, 0);
      emit_gn_backward(a.p + ".norm.bwd", g1_, a.x, a.p + ".norm", nullptr, 0, false, false, G[0], false, G[1], SB);
    }
    std::swap(G[0], G[1]);
  }
  // ---- stem ----
  {
    const float* g = G[0];
    const float* scale = scale_in_;
    const float* w = P("input_blocks.0.0.weight", (long long)stem_out.C * in_ch_ * 9);
    float* dx = grad_;
    const int H = R_, W = R_, Co = stem_out.C;
    DDNM_CHECK(Co % 4 == 0 && (size_t)Co * 3 * 9 * 4 <= 48 * 1024, "stem backward: unsupported channel count");
    add_op("stem.bwd", "stem", 2.0 * Bn * H * W * (double)Co * 3 * 9, (double)Bn * H * W * (Co + 3) * 4, [=](cudaStream_t s) {
      stem_bwd_kernel<3><<<(int)cdivll((long long)Bn * H * W, 128), 128, (size_t)Co * 3 * 9 * 4, s>>>(g, Bn, H, W, Co, w, scale, dx);
      CUDA_CHECK(cudaGetLastError());
    });
  }
}

void UNetEncoder::build_program() {
  const EncoderCfg& c = cfg_;
  const int mc = c.model_channels, R = c.image_size, L = c.n_levels;
  DDNM_CHECK(mc % 64 == 0, "model_channels must be a multiple of 64 (tensor-core K blocks)");
  DDNM_CHECK(L >= 1 && L <= 8 && R % (1 << (L - 1)) == 0, "image size not divisible by the downsampling");
  for (int lv = 0; lv < L; ++lv) {
    const int co = c.channel_mult[lv] * mc;
    DDNM_CHECK(co % 64 == 0 && co > 0, "channel counts must be multiples of 64");
  }
  const Torso t = plan_torso(R, c.in_channels, mc, c.channel_mult, L, c.num_res_blocks, c.attn_ds, c.n_attn_ds);
  // ---- sizing: widest activation (incl. qkv rows), attention score matrices, ResBlock scale|shift rows ----
  size_t act_max = (size_t)B_ * R * R * c.channel_mult[0] * mc, att_qkv = 1, att_S = 1, att_O = 1;
  std::vector<EmbProj> projs;
  auto size_block = [&](const std::string& prefix, const Block& b) {
    const int r = b.res_in;
    for (size_t j = 0; j < b.layers.size(); ++j) {
      const Block::Layer& l = b.layers[j];
      const std::string p = prefix + "." + std::to_string(j);
      if (l.kind == LAYER_ATTN) {
        const size_t T = (size_t)r * r, heads = l.cin / c.num_head_channels;
        act_max = std::max(act_max, (size_t)B_ * T * 3 * l.cin);
        att_qkv = std::max(att_qkv, (size_t)B_ * T * 3 * l.cin);
        att_S = std::max(att_S, (size_t)B_ * heads * T * T);
        att_O = std::max(att_O, (size_t)B_ * T * l.cin);
      } else {
        if (l.kind == LAYER_RES) act_max = std::max(act_max, (size_t)B_ * r * r * std::max(l.cin, l.cout));
        projs.push_back({p, p + ".emb_layers.1.weight", P(p + ".emb_layers.1.bias", 2 * l.cout), 2 * l.cout});
      }
    }
  };
  for (size_t i = 1; i < t.input.size(); ++i) size_block("input_blocks." + std::to_string(i), t.input[i]);
  size_block("middle_block", t.middle);
  headT_ = t.middle.res_in * t.middle.res_in + 1;
  alloc_common(act_max, 0);
  alloc_attention(att_qkv, att_S, att_O);
  scale_in_ = (float*)arena_.alloc(4);
  fill(scale_in_, 1, 1.0f, 0);   // the scale of an eager profile run before any grad() call
  grad_ = (float*)arena_.alloc((size_t)B_ * in_ch_ * R * R * 4);
  for (float*& g : gx_) g = (float*)arena_.alloc(act_max * 4);
  g1_ = (float*)arena_.alloc(act_max * 4);
  g2_ = (float*)arena_.alloc(std::max(act_max, (size_t)B_ * (c.out_channels + 1024)) * 4);
  gqkv_ = (float*)arena_.alloc(act_max * 4);
  sP_ = (float*)arena_.alloc(att_S * 4);
  sdP_ = (float*)arena_.alloc(att_S * 4);
  gnb_part_elems_ = (size_t)(invariant_ ? B_ * (kGnbInvariantChunks + 1) : 4 * num_sms_ + 2 * B_) * 512 * 2;
  gnb_part_ = (float*)arena_.alloc(gnb_part_elems_ * sizeof(double));

  emit_time_embed("time_embed", "time_embed.0", "time_embed.2", mc, false, nullptr, 0, projs);

  // ---- torso: every ResBlock and AttentionBlock keeps its activations for the backward pass ----
  std::vector<Layer> layers;
  View h = new_view(R, R, c.channel_mult[0] * mc);
  emit_stem("input_blocks.0.0", h);
  const View stem_out = h;
  auto run_block = [&](const std::string& prefix, const Block& b) {
    for (size_t j = 0; j < b.layers.size(); ++j) {
      const Block::Layer& l = b.layers[j];
      const std::string p = prefix + "." + std::to_string(j);
      const int ro = l.kind == LAYER_RES_DOWN ? h.H / 2 : h.H;
      View dst = new_view(ro, ro, l.cout);
      Layer rec;
      if (l.kind == LAYER_ATTN) {
        // QKVAttentionLegacy; the qkv rows in a buffer of their own
        DDNM_CHECK(h.C % c.num_head_channels == 0, "channels not divisible by num_head_channels");
        float* qkv = (float*)arena_.alloc((size_t)B_ * h.H * h.W * 3 * h.C * 4);
        emit_attention_block(p, h, dst, h.C / c.num_head_channels, false, qkv);
        rec.kind = 1;
        rec.a = Attn{p, h, dst, qkv};
      } else {
        View hv = new_view(ro, ro, l.cout);
        emit_res_block(p, h, hv, dst, l.kind);
        rec.kind = 0;
        rec.r = Res{p, h, hv, dst, l.kind == LAYER_RES_DOWN, has_param(p + ".skip_connection.weight")};
      }
      layers.push_back(rec);
      h = dst;
    }
  };
  for (size_t i = 1; i < t.input.size(); ++i) run_block("input_blocks." + std::to_string(i), t.input[i]);
  run_block("middle_block", t.middle);
  hf_ = (float*)arena_.alloc((size_t)B_ * h.H * h.W * h.C * 4);
  tok_ = (float*)arena_.alloc((size_t)B_ * headT_ * h.C * 4);
  hqkv_ = (float*)arena_.alloc((size_t)B_ * headT_ * 3 * h.C * 4);
  hp_ = (float*)arena_.alloc((size_t)B_ * (h.C / c.num_head_channels) * headT_ * 4);
  ha0_ = (float*)arena_.alloc((size_t)B_ * h.C * 4);
  DDNM_CHECK((size_t)B_ * headT_ * 3 * h.C <= act_max, "head scratch");
  emit_head(h);

  const size_t n_fwd = ops_.size();
  emit_backward(stem_out, layers, h);
  n_tail_ops_ = ops_.size() - n_fwd;
}

void UNetEncoder::check_labels(const int* labels, cudaStream_t stream) const {
  DDNM_CHECK(labels != nullptr, "null labels");
  std::vector<int> hl(B_);
  CUDA_CHECK(cudaMemcpyAsync(hl.data(), labels, (size_t)B_ * sizeof(int), cudaMemcpyDefault, stream));
  CUDA_CHECK(cudaStreamSynchronize(stream));
  for (int i = 0; i < B_; ++i)
    DDNM_CHECK(hl[i] >= 0 && hl[i] < cfg_.out_channels,
               "label " + std::to_string(hl[i]) + " outside [0, " + std::to_string(cfg_.out_channels) + ")");
}

void UNetEncoder::grad(const float* x, const float* t, const int* labels, float scale, float* grad_out, float* logits, cudaStream_t stream,
                       bool labels_checked) {
  DDNM_CHECK(finalized_, "classifier gradient before finalize");
  DDNM_CHECK(x && t && labels && grad_out, "null argument");
  if (!labels_checked) check_labels(labels, stream);
  const size_t xin = (size_t)B_ * in_ch_ * R_ * R_ * 4;
  if (x != x_in_) CUDA_CHECK(cudaMemcpyAsync(x_in_, x, xin, cudaMemcpyDeviceToDevice, stream));
  if (t != t_in_) CUDA_CHECK(cudaMemcpyAsync(t_in_, t, (size_t)B_ * 4, cudaMemcpyDeviceToDevice, stream));
  if (labels != labels_in_) CUDA_CHECK(cudaMemcpyAsync(labels_in_, labels, (size_t)B_ * sizeof(int), cudaMemcpyDeviceToDevice, stream));
  fill(scale_in_, 1, scale, stream);
  replay(stream, ops_.size(), ggraph_, ggraph_exec_);
  CUDA_CHECK(cudaMemcpyAsync(grad_out, grad_, xin, cudaMemcpyDeviceToDevice, stream));
  if (logits) CUDA_CHECK(cudaMemcpyAsync(logits, out_, out_elems() * 4, cudaMemcpyDeviceToDevice, stream));
}

}  // namespace ddnm

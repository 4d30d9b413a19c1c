// Degradation operators (functions/svd_operators.py) and the fused DDNM / DDNM+ update (functions/svd_ddnm.py:57-65,
// :114-131) as image-space CUDA kernels on NCHW fp32 images.  All kernels here are HBM-bound: algorithmic traffic of
// the fused step is xt + et + noise in, x0_t + xt_next out = 5 * 4 * C*H*W bytes per image (+ y).
#include "operators.cuh"

#include <algorithm>
#include <cmath>

#include "../../include/ddnm_b200.h"
#include "api_util.cuh"
#include "kernels.cuh"

namespace ddnm {

// ------------------------------------------------------------------------------------------------------------------
// Coefficient rules shared by every Lambda / Lambda_noise in the reference (e.g. svd_operators.py:568-604), evaluated
// per singular value with the same fp32 operation order (0-dim tensors and python floats both act as fp32 scalars).
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float lam_coeff(float s, const PlusScalars& ps) {
  const float inv = (s == 0.f) ? 0.f : __fdiv_rn(1.0f, s);
  float lam = 1.0f;
  if (ps.active) {
    const float thr = __fmul_rn(__fmul_rn(ps.a, ps.sigma_y), inv);
    if (ps.sigma_t < thr) lam = __fdiv_rn(__fdiv_rn(__fmul_rn(__fmul_rn(s, ps.sigma_t), ps.c), ps.a), ps.sigma_y);
  }
  return lam;
}
__device__ __forceinline__ void noise_coeff(float s, const PlusScalars& ps, float& d1, float& d2) {
  const float inv = (s == 0.f) ? 0.f : __fdiv_rn(1.0f, s);
  d1 = __fmul_rn(ps.sigma_t, ps.eta);
  d2 = __fmul_rn(ps.sigma_t, ps.c);
  if (ps.active) {
    const float thr = __fmul_rn(__fmul_rn(ps.a, ps.sigma_y), inv);
    float ci = (ps.sigma_t < thr) ? 1.f : 0.f;
    d1 = __fadd_rn(__fmul_rn(d1, 1.f - ci), __fmul_rn(__fmul_rn(ci, ps.sigma_t), ps.eta));
    d2 = __fmul_rn(d2, 1.f - ci);
    ci = (ps.sigma_t > thr) ? 1.f : 0.f;
    const float t1 = __fmul_rn(ps.sigma_t, ps.sigma_t);
    const float t3 = __fmul_rn(__fmul_rn(__fmul_rn(ps.a, ps.a), ps.sy2), __fmul_rn(inv, inv));
    d1 = __fadd_rn(__fmul_rn(d1, 1.f - ci), sqrtf(__fmul_rn(ci, __fsub_rn(t1, t3))));
    d2 = __fmul_rn(d2, 1.f - ci);
    ci = (s == 0.f) ? 1.f : 0.f;
    d1 = __fadd_rn(__fmul_rn(d1, 1.f - ci), __fmul_rn(__fmul_rn(ci, ps.sigma_t), ps.eta));
    d2 = __fadd_rn(__fmul_rn(d2, 1.f - ci), __fmul_rn(__fmul_rn(ci, ps.sigma_t), ps.c));
  }
}

PlusScalars make_plus(float a, float sigma_y, float sigma_t, float eta) {
  PlusScalars p;
  p.a = a; p.sigma_y = sigma_y; p.sigma_t = sigma_t; p.eta = eta;
  p.c = (float)std::sqrt(1.0 - (double)eta * (double)eta);
  p.sy2 = (float)((double)sigma_y * (double)sigma_y);
  p.active = (a != 0.f && sigma_y != 0.f) ? 1 : 0;
  return p;
}

// x0_t = (xt - et * sqrt(1-at)) / sqrt(at)      (svd_ddnm.py:57), unfused multiply / subtract / divide
__device__ __forceinline__ float x0_from(float xt, float et, const StepScalars& sc) {
  return __fdiv_rn(__fsub_rn(xt, __fmul_rn(et, sc.sqrt_1m_at)), sc.sqrt_at);
}
// xt_next = at_next.sqrt() * x0_hat + c1 * z + c2 * et      (svd_ddnm.py:65), evaluated left to right
__device__ __forceinline__ float renoise(float x0h, float z, float et, const StepScalars& sc) {
  return __fadd_rn(__fadd_rn(__fmul_rn(sc.sqrt_atn, x0h), __fmul_rn(sc.c1, z)), __fmul_rn(sc.c2, et));
}

// ------------------------------------------------------------------------------------------------------------------
// "Local group" operators: SuperResolution (group = r x r patch of one channel, svd_operators.py:479-623) and
// Colorization (group = the 3 channels of one pixel, :627-736).  A has rank 1 per group: A g = u00 * s0 * <V[:,0], g>.
// One thread owns one group; K x K basis V sits in shared memory.
// ------------------------------------------------------------------------------------------------------------------
template <int K, int MODE>  // MODE 0: SR with R = sqrt(K); MODE 1: colour (K = 3)
struct Group {
  int b;
  long long base;  // offset of element 0 inside image b
  int D, HW;
  long long yidx;
  __device__ __forceinline__ Group(long long g, int C, int Dd, long long img_elems) {
    D = Dd;
    HW = Dd * Dd;
    if (MODE == 0) {
      constexpr int R = K == 4 ? 2 : (K == 16 ? 4 : 8);
      const int yd = Dd / R;
      const int px = (int)(g % yd);
      const int py = (int)((g / yd) % yd);
      const int c = (int)((g / ((long long)yd * yd)) % C);
      b = (int)(g / ((long long)yd * yd * C));
      base = ((long long)c * Dd + (long long)py * R) * Dd + (long long)px * R;
      yidx = ((long long)b * C + c) * yd * yd + (long long)py * yd + px;
    } else {
      const int p = (int)(g % HW);
      b = (int)(g / HW);
      base = p;
      yidx = (long long)b * HW + p;
    }
  }
  __device__ __forceinline__ long long off(int k) const {
    if (MODE == 0) {
      constexpr int R = K == 4 ? 2 : (K == 16 ? 4 : 8);
      return base + (long long)(k / R) * D + (k % R);
    }
    return base + (long long)k * HW;
  }
  __device__ __forceinline__ void load(const float* p, long long img_stride, float (&v)[K]) const {
    const float* q = p + (long long)b * img_stride;
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = __ldg(q + off(k));
  }
  __device__ __forceinline__ void store(float* p, long long img_stride, const float (&v)[K]) const {
    float* q = p + (long long)b * img_stride;
#pragma unroll
    for (int k = 0; k < K; ++k) q[off(k)] = v[k];
  }
};

enum LocalFn : int { LF_A = 0, LF_PINV = 1, LF_PROJECT = 2, LF_LAMBDA = 3, LF_NOISE = 4, LF_STEP = 5 };

template <int K>
__device__ __forceinline__ float local_resid(const float (&x0)[K], const float* V, float u00, float s0, float yv, float (&resid)[K]) {
  float cval = 0.f;
#pragma unroll
  for (int k = 0; k < K; ++k) cval = fmaf(V[k * K], x0[k], cval);  // (V^T g)[0]
  const float av = __fmul_rn(u00, __fmul_rn(s0, cval));             // U (S V^T g)
  const float r = __fsub_rn(av, yv);
  const float cc = __fmul_rn(__fmul_rn(u00, r), __fdiv_rn(1.0f, s0));  // S^+ U^T r
#pragma unroll
  for (int k = 0; k < K; ++k) resid[k] = __fmul_rn(V[k * K], cc);   // V (cc, 0, ..)
  return av;
}

// The draws of one group, generated (LF_STEP with a seed).  SuperResolution: a patch row is R consecutive elements starting at
// a multiple of R, i.e. half a quad (R = 2), one quad (4) or two (8): one Philox call per 2 / 4 values, none wasted.
// Colorization: the thread owns ONE pixel in three channels, whose values lie in three different quads, so it takes noise_at
// per value (three Philox calls for three values).  Sharing the quads would need a thread per four pixels, a different kernel
// from the tape form; at ~1 % of a run's time for all step kernels together that is not worth a second kernel.
template <int K, int MODE>
__device__ __forceinline__ void local_draws(const Group<K, MODE>& G, const NoiseSrc& nz, float (&z)[K]) {
  if (MODE == 0) {
    constexpr int R = K == 4 ? 2 : (K == 16 ? 4 : 8);
#pragma unroll
    for (int kr = 0; kr < R; ++kr) {
      const long long e = G.base + (long long)kr * G.D;
      if (R == 2) {
        const float2 v = noise_pair(nz, G.b, e >> 1);
        z[kr * R] = v.x; z[kr * R + 1] = v.y;
      } else {
#pragma unroll
        for (int j = 0; j < R / 4; ++j) {
          const float4 v = noise_quad(nz, G.b, (e >> 2) + j);
          z[kr * R + 4 * j] = v.x; z[kr * R + 4 * j + 1] = v.y; z[kr * R + 4 * j + 2] = v.z; z[kr * R + 4 * j + 3] = v.w;
        }
      }
    }
  } else {
#pragma unroll
    for (int k = 0; k < K; ++k) z[k] = noise_at(nz, G.b, G.off(k));
  }
}

// GEN (LF_STEP only): in2 is null and the draws are generated in registers from gen
template <int K, int MODE, int FN, bool GEN = false>
__global__ void __launch_bounds__(128) local_kernel(const float* __restrict__ in0, const float* __restrict__ in1, long long in1_stride,
                                                    const float* __restrict__ in2, const float* __restrict__ y,
                                                    const float* __restrict__ Vg, float u00, float s0, StepScalars sc,
                                                    float* __restrict__ out0, float* __restrict__ out1, long long groups, int C,
                                                    int D, NoiseSrc gen) {
  __shared__ float V[K * K];
  for (int i = threadIdx.x; i < K * K; i += blockDim.x) V[i] = Vg[i];
  __syncthreads();
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= groups) return;
  const long long img = (long long)C * D * D;
  Group<K, MODE> G(g, C, D, img);
  const PlusScalars& ps = sc.plus;
  if (FN == LF_A) {
    float x[K];
    G.load(in0, img, x);
    float cval = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) cval = fmaf(V[k * K], x[k], cval);
    out0[G.yidx] = __fmul_rn(u00, __fmul_rn(s0, cval));
  } else if (FN == LF_PINV) {
    const float cc = __fmul_rn(__fmul_rn(u00, y[G.yidx]), __fdiv_rn(1.0f, s0));
    float o[K];
#pragma unroll
    for (int k = 0; k < K; ++k) o[k] = __fmul_rn(V[k * K], cc);
    G.store(out0, img, o);
  } else if (FN == LF_PROJECT) {
    float x[K], r[K];
    G.load(in0, img, x);
    local_resid<K>(x, V, u00, s0, y[G.yidx], r);
#pragma unroll
    for (int k = 0; k < K; ++k) x[k] = __fsub_rn(x[k], r[k]);
    G.store(out0, img, x);
  } else if (FN == LF_LAMBDA) {
    float x[K], o[K];
    G.load(in0, img, x);
#pragma unroll
    for (int k = 0; k < K; ++k) o[k] = 0.f;
#pragma unroll
    for (int j = 0; j < K; ++j) {
      float sp = 0.f;
#pragma unroll
      for (int k = 0; k < K; ++k) sp = fmaf(V[k * K + j], x[k], sp);
      sp *= lam_coeff(j == 0 ? s0 : 0.f, ps);
#pragma unroll
      for (int k = 0; k < K; ++k) o[k] = fmaf(V[k * K + j], sp, o[k]);
    }
    G.store(out0, img, o);
  } else if (FN == LF_NOISE) {
    float v[K], e[K], ov[K], oe[K];
    G.load(in0, img, v);
    G.load(in1, in1_stride, e);
#pragma unroll
    for (int k = 0; k < K; ++k) { ov[k] = 0.f; oe[k] = 0.f; }
#pragma unroll
    for (int j = 0; j < K; ++j) {
      float d1, d2;
      noise_coeff(j == 0 ? s0 : 0.f, ps, d1, d2);
      const float a = v[j] * d1, b = e[j] * d2;  // raw pixels used as spectral coordinates (svd_operators.py:581-621)
#pragma unroll
      for (int k = 0; k < K; ++k) {
        ov[k] = fmaf(V[k * K + j], a, ov[k]);
        oe[k] = fmaf(V[k * K + j], b, oe[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < K; ++k) ov[k] = __fadd_rn(ov[k], oe[k]);
    G.store(out0, img, ov);
  } else {  // LF_STEP: in0 = xt, in1 = et, in2 = noise, out0 = x0_t, out1 = xt_next
    float xt[K], et[K], z[K], x0[K], r[K];
    G.load(in0, img, xt);
    G.load(in1, in1_stride, et);
    if (GEN) local_draws<K, MODE>(G, gen, z);
    else G.load(in2, img, z);
#pragma unroll
    for (int k = 0; k < K; ++k) x0[k] = x0_from(xt[k], et[k], sc);
    G.store(out0, img, x0);
    local_resid<K>(x0, V, u00, s0, y[G.yidx], r);
    float xn[K];
    if (!sc.use_plus) {
#pragma unroll
      for (int k = 0; k < K; ++k) xn[k] = renoise(__fsub_rn(x0[k], r[k]), z[k], et[k], sc);
    } else {
      float L[K], nv[K], ne[K];
#pragma unroll
      for (int k = 0; k < K; ++k) { L[k] = 0.f; nv[k] = 0.f; ne[k] = 0.f; }
#pragma unroll
      for (int j = 0; j < K; ++j) {
        const float sj = j == 0 ? s0 : 0.f;
        float sp = 0.f;
#pragma unroll
        for (int k = 0; k < K; ++k) sp = fmaf(V[k * K + j], r[k], sp);
        sp *= lam_coeff(sj, ps);
        float d1, d2;
        noise_coeff(sj, ps, d1, d2);
        const float a = z[j] * d1, b = et[j] * d2;
#pragma unroll
        for (int k = 0; k < K; ++k) {
          L[k] = fmaf(V[k * K + j], sp, L[k]);
          nv[k] = fmaf(V[k * K + j], a, nv[k]);
          ne[k] = fmaf(V[k * K + j], b, ne[k]);
        }
      }
#pragma unroll
      for (int k = 0; k < K; ++k)
        xn[k] = __fadd_rn(__fmul_rn(sc.sqrt_atn, __fsub_rn(x0[k], L[k])), __fadd_rn(nv[k], ne[k]));
    }
    G.store(out1, img, xn);
  }
}

template <int K, int MODE>
static void local_launch(int fn, const float* in0, const float* in1, long long in1_stride, const float* in2, const float* y,
                         const float* V, float u00, float s0, const StepScalars& sc, float* out0, float* out1, long long groups,
                         int C, int D, cudaStream_t st, const NoiseSrc& noise) {
  const int grid = (int)cdivll(groups, 128);
#define LL(F, GEN) \
  local_kernel<K, MODE, F, GEN><<<grid, 128, 0, st>>>(in0, in1, in1_stride, in2, y, V, u00, s0, sc, out0, out1, groups, C, D, noise)
  switch (fn) {
    case LF_A: LL(LF_A, false); break;
    case LF_PINV: LL(LF_PINV, false); break;
    case LF_PROJECT: LL(LF_PROJECT, false); break;
    case LF_LAMBDA: LL(LF_LAMBDA, false); break;
    case LF_NOISE: LL(LF_NOISE, false); break;
    default: noise_dispatch(noise, [&](auto gen) { LL(LF_STEP, decltype(gen)::value); }); break;
  }
#undef LL
  CUDA_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------------------------
// Inpainting (svd_operators.py:324-439; mask -> indices at diffusion.py:464-471).  y holds the kept entries of the
// (pixel, channel)-interleaved image in ascending order: y[rank(p*C + c)] = x[c][p].  Pure data movement: bit-exact.
// ------------------------------------------------------------------------------------------------------------------
template <int FN, bool GEN = false>   // GEN (LF_STEP only): draws generated in registers from gen, in2 unused
__global__ void inpaint_kernel(const float* __restrict__ in0, const float* __restrict__ in1, long long in1_stride,
                               const float* __restrict__ in2, const float* __restrict__ y, const int* __restrict__ rank,
                               StepScalars sc, float* __restrict__ out0, float* __restrict__ out1, int B, int C, int HW, long long M,
                               NoiseSrc gen) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long img = (long long)C * HW;
  if (i >= (long long)B * img) return;
  const int p = (int)(i % HW);
  const int c = (int)((i / HW) % C);
  const int b = (int)(i / img);
  const int r = rank[(long long)p * C + c];
  const bool kept = r >= 0;
  const long long yi = (long long)b * M + r;
  const PlusScalars& ps = sc.plus;
  const float s = kept ? 1.f : 0.f;
  if (FN == LF_A) {
    if (kept) out0[yi] = in0[i];
  } else if (FN == LF_PINV) {
    out0[i] = kept ? y[yi] : 0.f;
  } else if (FN == LF_PROJECT) {
    const float x0 = in0[i];
    out0[i] = kept ? __fsub_rn(x0, __fsub_rn(x0, y[yi])) : __fsub_rn(x0, 0.f);
  } else if (FN == LF_LAMBDA) {
    out0[i] = __fmul_rn(in0[i], lam_coeff(s, ps));
  } else if (FN == LF_NOISE) {
    float d1, d2;
    noise_coeff(s, ps, d1, d2);
    out0[i] = __fadd_rn(__fmul_rn(in0[i], d1), __fmul_rn(in1[(long long)b * in1_stride + (i - (long long)b * img)], d2));
  } else {
    const float et = in1[(long long)b * in1_stride + (i - (long long)b * img)];
    const float z = GEN ? noise_at(gen, b, i - (long long)b * img) : in2[i];
    const float x0 = x0_from(in0[i], et, sc);
    out0[i] = x0;
    const float resid = kept ? __fsub_rn(x0, y[yi]) : 0.f;
    if (!sc.use_plus) {
      out1[i] = renoise(__fsub_rn(x0, resid), z, et, sc);
    } else {
      float d1, d2;
      noise_coeff(s, ps, d1, d2);
      const float x0h = __fsub_rn(x0, __fmul_rn(resid, lam_coeff(s, ps)));
      out1[i] = __fadd_rn(__fmul_rn(sc.sqrt_atn, x0h), __fadd_rn(__fmul_rn(z, d1), __fmul_rn(et, d2)));
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Walsh-Hadamard (svd_operators.py:211-320).  H_{D*D} = H_D (x) H_D: butterflies over the low log2(D) index bits run
// along image rows, the high bits along columns; stage order equals the reference's h = 1, 2, 4, ... loop so every
// output is produced by the same sequence of fp32 adds.  The 1/D normalisation is applied after the last stage.
// ------------------------------------------------------------------------------------------------------------------
__global__ void fwht_rows_kernel(float* __restrict__ buf, int D, long long rows) {
  extern __shared__ float sm[];
  const int rpb = blockDim.x * 2 / D;  // rows per block (each thread owns 2 elements)
  const long long row0 = (long long)blockIdx.x * rpb;
  const int lr = (threadIdx.x * 2) / D;
  const long long row = row0 + lr;
  float* s = sm + lr * D;
  const int t = threadIdx.x % (D / 2);
  if (row < rows) {
    s[t] = buf[row * D + t];
    s[t + D / 2] = buf[row * D + t + D / 2];
  }
  __syncthreads();
  for (int h = 1; h < D; h <<= 1) {
    const int i = (t / h) * 2 * h + (t % h);
    const float a = s[i], b = s[i + h];
    __syncthreads();
    s[i] = a + b;
    s[i + h] = a - b;
    __syncthreads();
  }
  if (row < rows) {
    buf[row * D + t] = s[t];
    buf[row * D + t + D / 2] = s[t + D / 2];
  }
}
// columns: block = (image, 32-column strip); smem [D][33]
__global__ void fwht_cols_kernel(float* __restrict__ buf, int D, float scale) {
  extern __shared__ float sm[];
  const long long img = blockIdx.y;
  const int c0 = blockIdx.x * 32;
  float* base = buf + img * D * D;
  const int cx = threadIdx.x % 32, ry = threadIdx.x / 32;
  const int rstep = blockDim.x / 32;
  for (int r = ry; r < D; r += rstep) sm[r * 33 + cx] = base[(long long)r * D + c0 + cx];
  __syncthreads();
  for (int h = 1; h < D; h <<= 1) {
    for (int t = ry; t < D / 2; t += rstep) {
      const int i = (t / h) * 2 * h + (t % h);
      const float a = sm[i * 33 + cx], b = sm[(i + h) * 33 + cx];
      sm[i * 33 + cx] = a + b;
      sm[(i + h) * 33 + cx] = a - b;
    }
    __syncthreads();
  }
  for (int r = ry; r < D; r += rstep) base[(long long)r * D + c0 + cx] = sm[r * 33 + cx] / scale;
}

// spectral-domain elementwise stage of the WH operator.  kept(c,q) <=> invperm[q]*C + c < M
template <int FN>
__global__ void wh_spec_kernel(const float* __restrict__ F, const float* __restrict__ F2, const float* __restrict__ y,
                               const int* __restrict__ perm, const int* __restrict__ invperm, PlusScalars ps,
                               float* __restrict__ out, int B, int C, int n2, long long M) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (FN == LF_A) {  // gather: out[b][j], j = p*C + c
    if (i >= (long long)B * M) return;
    const long long j = i % M;
    const int b = (int)(i / M);
    const int p = (int)(j / C), c = (int)(j % C);
    out[i] = F[((long long)b * C + c) * n2 + perm[p]];
    return;
  }
  if (i >= (long long)B * C * n2) return;
  const int q = (int)(i % n2);
  const int c = (int)((i / n2) % C);
  const int b = (int)(i / ((long long)C * n2));
  const long long j = (long long)invperm[q] * C + c;
  const bool kept = j < M;
  const float s = kept ? 1.f : 0.f;
  if (FN == LF_PINV) {
    out[i] = kept ? y[(long long)b * M + j] : 0.f;
  } else if (FN == LF_PROJECT) {
    out[i] = kept ? __fsub_rn(F[i], y[(long long)b * M + j]) : 0.f;
  } else if (FN == LF_LAMBDA) {
    out[i] = __fmul_rn(F[i], lam_coeff(s, ps));
  } else {  // LF_NOISE: raw pixels scaled in place of spectral coordinates
    float d1, d2;
    noise_coeff(s, ps, d1, d2);
    out[i] = __fadd_rn(__fmul_rn(F[i], d1), __fmul_rn(F2[i], d2));
  }
}

// ------------------------------------------------------------------------------------------------------------------
// elementwise helpers of the generic (non-fused) step and of the separable operators
// ------------------------------------------------------------------------------------------------------------------
__global__ void x0_kernel(const float* __restrict__ xt, const float* __restrict__ et, long long et_stride, StepScalars sc,
                          float* __restrict__ x0, float* __restrict__ et3, int B, long long img) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * img) return;
  const int b = (int)(i / img);
  const float e = et[(long long)b * et_stride + (i - (long long)b * img)];
  et3[i] = e;
  x0[i] = x0_from(xt[i], e, sc);
}
template <bool GEN>   // GEN: draws generated in registers from gen (img = elements per image), z unused
__global__ void final_ddnm_kernel(const float* __restrict__ x0, const float* __restrict__ resid, const float* __restrict__ z,
                                  const float* __restrict__ et3, StepScalars sc, float* __restrict__ xn, long long n, long long img,
                                  NoiseSrc gen) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float zi;
  if (GEN) {
    const long long b = i / img;
    zi = noise_at(gen, (int)b, i - b * img);
  } else {
    zi = z[i];
  }
  xn[i] = renoise(__fsub_rn(x0[i], resid[i]), zi, et3[i], sc);
}
__global__ void final_plus_kernel(const float* __restrict__ x0, const float* __restrict__ L, const float* __restrict__ nz,
                                  StepScalars sc, float* __restrict__ xn, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  xn[i] = __fadd_rn(__fmul_rn(sc.sqrt_atn, __fsub_rn(x0[i], L[i])), nz[i]);
}
__global__ void sub_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ o, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) o[i] = __fsub_rn(a[i], b[i]);
}
// t[b][c][pos] *= tab[(per_channel ? c : 0)][pos]
__global__ void mul_table_kernel(float* __restrict__ t, const float* __restrict__ tab, int per_channel, int C, int n2, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int pos = (int)(i % n2);
  const int c = (int)((i / n2) % C);
  t[i] = __fmul_rn(t[i], tab[(per_channel ? (long long)c * n2 : 0) + pos]);
}
// deblur Lambda tables from the un-thresholded singulars at each spectral position
template <int FN>
__global__ void deblur_coeff_kernel(const float* __restrict__ v, const float* __restrict__ e, const float* __restrict__ sorig,
                                    PlusScalars ps, float* __restrict__ out, int n2, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float s = sorig[i % n2];
  if (FN == LF_LAMBDA) {
    out[i] = __fmul_rn(v[i], lam_coeff(s, ps));
  } else {
    float d1, d2;
    noise_coeff(s, ps, d1, d2);
    out[i] = __fadd_rn(__fmul_rn(v[i], d1), __fmul_rn(e[i], d2));
  }
}

// CS (svd_operators.py:101-159): 32x32 patches <-> rows of a [B*C*y*y, 1024] matrix (row-major inside the patch)
template <bool TO_ROWS>
__global__ void cs_patch_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int D) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)B * C * D * D;
  if (i >= total) return;
  const int yd = D / 32;
  const int k = (int)(i % 1024);
  const long long pr = i / 1024;                 // (b, c, py, px)
  const int px = (int)(pr % yd), py = (int)((pr / yd) % yd);
  const long long bc = pr / ((long long)yd * yd);
  const long long img = bc * D * D + (long long)(py * 32 + k / 32) * D + (px * 32 + k % 32);
  if (TO_ROWS) dst[i] = src[img];
  else dst[img] = src[i];
}

// Denoising (svd_operators.py:442-476): A = I; Lambda / Lambda_noise are SCALAR rules of their own (not the table rule)
template <int FN, bool GEN = false>   // GEN (LF_STEP only): draws generated in registers from gen, in2 unused
__global__ void denoise_kernel(const float* __restrict__ in0, const float* __restrict__ in1, long long in1_stride,
                               const float* __restrict__ in2, const float* __restrict__ y, StepScalars sc, float* __restrict__ out0,
                               float* __restrict__ out1, int B, long long img, NoiseSrc gen) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * img) return;
  const int b = (int)(i / img);
  const PlusScalars& ps = sc.plus;
  const float asy = __fmul_rn(ps.a, ps.sigma_y);
  // Lambda (:462-467): sigma_t < a*sigma_y ? v * (sigma_t * sqrt(1-eta^2) / a / sigma_y) : v
  const float lam = (ps.sigma_t < asy) ? __fdiv_rn(__fdiv_rn(__fmul_rn(ps.sigma_t, ps.c), ps.a), ps.sigma_y) : 1.0f;
  // Lambda_noise (:469-474): sigma_t >= a*sigma_y ? v * sqrt(sigma_t^2 - a^2 sigma_y^2) : v * sigma_t * eta   (epsilon unused)
  const float t2 = __fsub_rn(__fmul_rn(ps.sigma_t, ps.sigma_t), __fmul_rn(__fmul_rn(ps.a, ps.a), ps.sy2));
  if (FN == LF_LAMBDA) {
    out0[i] = (ps.sigma_t < asy) ? __fmul_rn(in0[i], lam) : in0[i];
  } else if (FN == LF_NOISE) {
    out0[i] = (ps.sigma_t >= asy) ? __fmul_rn(in0[i], sqrtf(t2)) : __fmul_rn(__fmul_rn(in0[i], ps.sigma_t), ps.eta);
  } else {  // LF_STEP
    const float et = in1[(long long)b * in1_stride + (i - (long long)b * img)];
    const float z = GEN ? noise_at(gen, b, i - (long long)b * img) : in2[i];
    const float x0 = x0_from(in0[i], et, sc);
    out0[i] = x0;
    const float resid = __fsub_rn(x0, y[i]);
    if (!sc.use_plus) {
      out1[i] = renoise(__fsub_rn(x0, resid), z, et, sc);
    } else {
      const float L = (ps.sigma_t < asy) ? __fmul_rn(resid, lam) : resid;
      const float nz = (ps.sigma_t >= asy) ? __fmul_rn(z, sqrtf(t2)) : __fmul_rn(__fmul_rn(z, ps.sigma_t), ps.eta);
      out1[i] = __fadd_rn(__fmul_rn(sc.sqrt_atn, __fsub_rn(x0, L)), nz);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// SuperResolution, generic ratio r (K = r*r entries per patch; svd_operators.py:479-623 with r = 16 in evaluation.sh):
// patches become rows of a [B*C*y*y, K] matrix (row-major inside the patch, the reference's unfold order :510-512).  A has rank 1
// per patch, so A / A^+ / the projection / Lambda need only V[:, 0] and one dot product per row (V is orthogonal:
// V diag(l0, lz, .., lz) V^T x = lz x + (l0 - lz) <v0, x> v0); Lambda_noise multiplies RAW pixels by V (:581-621), which is a
// [rows, K] x V^T GEMM on the CUDA cores.
// ------------------------------------------------------------------------------------------------------------------
template <bool TO_ROWS>
__global__ void sr_patch_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int D, int r) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)B * C * D * D;
  if (i >= total) return;
  const int K = r * r, yd = D / r;
  const int k = (int)(i % K);
  const long long pr = i / K;                 // (b, c, py, px)
  const int px = (int)(pr % yd), py = (int)((pr / yd) % yd);
  const long long bc = pr / ((long long)yd * yd);
  const long long img = bc * D * D + (long long)(py * r + k / r) * D + (px * r + k % r);
  if (TO_ROWS) dst[i] = src[img];
  else dst[img] = src[i];
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// one warp per patch row.  P: rows [rows, K]; Q / Wv / We: further row operands; yv: [rows]
template <int FN>
__global__ void srg_rows_kernel(const float* __restrict__ P, const float* __restrict__ Q, const float* __restrict__ Wv,
                                const float* __restrict__ We, const float* __restrict__ yv, const float* __restrict__ v0, float u00,
                                float s0, PlusScalars ps, float* __restrict__ out, long long rows, int K) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* p = P ? P + row * K : nullptr;
  float dot = 0.f;
  if (FN == LF_A || FN == LF_PROJECT || FN == LF_LAMBDA) {
    for (int k = lane; k < K; k += 32) dot = fmaf(v0[k], p[k], dot);
    dot = warp_sum(dot);
  }
  if (FN == LF_A) {
    if (lane == 0) out[row] = __fmul_rn(u00, __fmul_rn(s0, dot));
  } else if (FN == LF_PINV) {
    const float cc = __fmul_rn(__fmul_rn(u00, yv[row]), __fdiv_rn(1.0f, s0));
    for (int k = lane; k < K; k += 32) out[row * K + k] = __fmul_rn(v0[k], cc);
  } else if (FN == LF_PROJECT) {
    const float r = __fsub_rn(__fmul_rn(u00, __fmul_rn(s0, dot)), yv[row]);
    const float cc = __fmul_rn(__fmul_rn(u00, r), __fdiv_rn(1.0f, s0));
    for (int k = lane; k < K; k += 32) out[row * K + k] = __fsub_rn(p[k], __fmul_rn(v0[k], cc));
  } else if (FN == LF_LAMBDA) {
    const float l0 = lam_coeff(s0, ps), lz = lam_coeff(0.f, ps);
    const float t = __fmul_rn(__fsub_rn(l0, lz), dot);
    for (int k = lane; k < K; k += 32) out[row * K + k] = fmaf(v0[k], t, __fmul_rn(lz, p[k]));
  } else {  // LF_NOISE: P = raw v rows, Q = raw eps rows, Wv = P V^T, We = Q V^T
    float d10, d20, d1z, d2z;
    noise_coeff(s0, ps, d10, d20);
    noise_coeff(0.f, ps, d1z, d2z);
    const float a0 = __fmul_rn(__fsub_rn(d10, d1z), p[0]);
    const float b0 = __fmul_rn(__fsub_rn(d20, d2z), Q[row * K]);
    for (int k = lane; k < K; k += 32) {
      const float ov = fmaf(v0[k], a0, __fmul_rn(d1z, Wv[row * K + k]));
      const float oe = fmaf(v0[k], b0, __fmul_rn(d2z, We[row * K + k]));
      out[row * K + k] = __fadd_rn(ov, oe);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Operator: the generic paths of the base class, one class per operator family, the factory
// ------------------------------------------------------------------------------------------------------------------
Scratch::~Scratch() {
  if (p_) cudaFree(p_);
}

float* Scratch::get(size_t elems) {
  if (elems_ < elems) {
    if (p_) {
      CUDA_CHECK(cudaDeviceSynchronize());
      CUDA_CHECK(cudaFree(p_));
      p_ = nullptr;
      elems_ = 0;
    }
    CUDA_CHECK(cudaMalloc(&p_, elems * sizeof(float)));
    elems_ = elems;
  }
  return p_;
}

Operator::~Operator() {
  for (void* p : owned_) cudaFree(p);
}

template <class T>
T* Operator::upload(const T* host, size_t n) {
  T* d = nullptr;
  CUDA_CHECK(cudaMalloc(&d, std::max<size_t>(n, 1) * sizeof(T)));
  owned_.push_back(d);
  CUDA_CHECK(cudaMemcpy(d, host, n * sizeof(T), cudaMemcpyHostToDevice));
  return d;
}

static inline int blocks(long long n, int t = 256) { return (int)cdivll(n, t); }

void Operator::residual(const float* x0, const float* y, int B, float* R, cudaStream_t s) {
  const long long m = (long long)B * M_;
  float* Ay = ay_.get(m);
  A(x0, B, Ay, s);
  sub_kernel<<<blocks(m), 256, 0, s>>>(Ay, y, Ay, m);
  A_pinv(Ay, B, R, s);
}

void Operator::project(const float* x0, const float* y, int B, float* out, cudaStream_t s) {
  const long long n = (long long)B * N_;
  float* R = r_.get(n);
  residual(x0, y, B, R, s);
  sub_kernel<<<blocks(n), 256, 0, s>>>(x0, R, out, n);
  CUDA_CHECK(cudaGetLastError());
}

void Operator::lambda(const float*, int, const PlusScalars&, float*, cudaStream_t) {
  throw Error(std::string(name_) + " defines no Lambda (" + src_ + "): sigma_y > 0 is unsupported" + note_ + ", as in the reference");
}

void Operator::lambda_noise(const float*, const float*, int, const PlusScalars&, float*, cudaStream_t) {
  throw Error(std::string(name_) + " defines no Lambda_noise (" + src_ + ")");
}

// the generic step: x0_t, the residual r = A^+(A x0_t - y), then the DDNM / DDNM+ update
void Operator::step(const float* xt, const float* et, long long et_stride, const NoiseSrc& nz, const float* y, int B,
                    const StepScalars& sc, float* x0_t, float* xt_next, cudaStream_t s) {
  const long long n = (long long)B * N_;
  float* et3 = et3_.get(n);
  x0_kernel<<<blocks(n), 256, 0, s>>>(xt, et, et_stride, sc, x0_t, et3, B, N_);
  float* R = r_.get(n);
  residual(x0_t, y, B, R, s);
  const float* noise = nz.tape;
  if (!sc.use_plus) {
    noise_dispatch(nz, [&](auto gen) {
      final_ddnm_kernel<decltype(gen)::value><<<blocks(n), 256, 0, s>>>(x0_t, R, noise, et3, sc, xt_next, n, N_, nz);
    });
  } else {
    if (!noise) {
      // Lambda_noise of these operators is a transform of the whole draw (a GEMM or a Walsh-Hadamard transform of the raw
      // pixels), not a map: materialise this ONE pair's draws, the same values the fused kernels make in registers
      float* Z = z_.get(n);
      noise_fill(nz, Z, B, N_, s);
      noise = Z;
    }
    lambda(R, B, sc.plus, R, s);                       // R <- Lambda(R)   (in place is safe: inputs are staged first)
    float* NZ = ay_.get(n);
    lambda_noise(noise, et3, B, sc.plus, NZ, s);
    final_plus_kernel<<<blocks(n), 256, 0, s>>>(x0_t, R, NZ, sc, xt_next, n);
  }
  CUDA_CHECK(cudaGetLastError());
}

namespace {

// the step scalars of a fused kernel's Lambda / Lambda_noise form
StepScalars with_plus(const PlusScalars& ps) {
  StepScalars sc{};
  sc.plus = ps;
  return sc;
}

std::vector<float> transpose(const float* m, int r, int c) {
  std::vector<float> t((size_t)r * c);
  for (int i = 0; i < r; ++i)
    for (int j = 0; j < c; ++j) t[(size_t)j * r + i] = m[(size_t)i * c + j];
  return t;
}

// 1/s, and 0 where s is 0 (A_pinv's factors, svd_operators.py:74-75)
std::vector<float> reciprocals(const float* s, size_t n) {
  std::vector<float> r(n);
  for (size_t i = 0; i < n; ++i) r[i] = s[i] == 0.f ? 0.f : 1.0f / s[i];
  return r;
}

// SuperResolution with r = 2, 4, 8 and Colorization: every entry, the step included, is one fused local_kernel launch
class Local final : public Operator {
 public:
  // K: elements of one group (r*r, or 3 for Colorization); V: the K x K basis; u00, s0: U_small[0], singulars[0]
  Local(int C, int D, int K, const float* V, float u00, float s0)
      : Operator((long long)C * D * D / K, (long long)C * D * D), C_(C), D_(D), K_(K), V_(upload(V, (size_t)K * K)), u00_(u00),
        s0_(s0) {}
  void A(const float* x, int B, float* y, cudaStream_t s) override {
    launch(LF_A, x, nullptr, 0, nullptr, nullptr, StepScalars{}, y, nullptr, B, s);
  }
  void A_pinv(const float* y, int B, float* x, cudaStream_t s) override {
    launch(LF_PINV, nullptr, nullptr, 0, nullptr, y, StepScalars{}, x, nullptr, B, s);
  }
  void project(const float* x0, const float* y, int B, float* out, cudaStream_t s) override {
    launch(LF_PROJECT, x0, nullptr, 0, nullptr, y, StepScalars{}, out, nullptr, B, s);
  }
  void lambda(const float* v, int B, const PlusScalars& ps, float* out, cudaStream_t s) override {
    launch(LF_LAMBDA, v, nullptr, 0, nullptr, nullptr, with_plus(ps), out, nullptr, B, s);
  }
  void lambda_noise(const float* v, const float* eps, int B, const PlusScalars& ps, float* out, cudaStream_t s) override {
    launch(LF_NOISE, v, eps, N_, nullptr, nullptr, with_plus(ps), out, nullptr, B, s);
  }
  void step(const float* xt, const float* et, long long et_stride, const NoiseSrc& nz, const float* y, int B, const StepScalars& sc,
            float* x0_t, float* xt_next, cudaStream_t s) override {
    launch(LF_STEP, xt, et, et_stride, nz.tape, y, sc, x0_t, xt_next, B, s, nz);
  }

 private:
  void launch(int fn, const float* in0, const float* in1, long long in1_stride, const float* in2, const float* y,
              const StepScalars& sc, float* out0, float* out1, int B, cudaStream_t s, const NoiseSrc& nz = NoiseSrc{}) const {
    const long long groups = (long long)B * N_ / K_;
#define LOCAL(K, MODE) local_launch<K, MODE>(fn, in0, in1, in1_stride, in2, y, V_, u00_, s0_, sc, out0, out1, groups, C_, D_, s, nz)
    switch (K_) {
      case 3: LOCAL(3, 1); break;
      case 4: LOCAL(4, 0); break;
      case 16: LOCAL(16, 0); break;
      default: LOCAL(64, 0); break;
    }
#undef LOCAL
  }
  const int C_, D_, K_;
  const float* V_;
  const float u00_, s0_;
};

// SuperResolution with any other ratio: the patch rows of sr_patch_kernel and srg_rows_kernel; the step is the generic one
class PatchRows final : public Operator {
 public:
  // V: the K x K basis; u00, s0: U_small[0], singulars[0]
  PatchRows(int C, int D, int r, const float* V, float u00, float s0)
      : Operator((long long)C * (D / r) * (D / r), (long long)C * D * D), C_(C), D_(D), ratio_(r), K_(r * r),
        V_(upload(V, (size_t)K_ * K_)), u00_(u00), s0_(s0) {
    std::vector<float> v0(K_);
    for (int k = 0; k < K_; ++k) v0[k] = V[(size_t)k * K_];
    v0_ = upload(v0.data(), (size_t)K_);
  }
  void A(const float* x, int B, float* y, cudaStream_t s) override {
    float* P = rows_.get((size_t)B * N_);
    to_rows(x, P, B, s);
    row_op<LF_A>(P, nullptr, nullptr, nullptr, nullptr, PlusScalars{}, y, B, s);
  }
  void A_pinv(const float* y, int B, float* x, cudaStream_t s) override {
    float* P = rows_.get((size_t)B * N_);
    row_op<LF_PINV>(nullptr, nullptr, nullptr, nullptr, y, PlusScalars{}, P, B, s);
    from_rows(P, x, B, s);
  }
  // fused: one pass over the rows (the step's residual still runs through A, sub and A_pinv)
  void project(const float* x0, const float* y, int B, float* out, cudaStream_t s) override {
    float* P = rows_.get((size_t)B * N_);
    float* O = rows2_.get((size_t)B * N_);
    to_rows(x0, P, B, s);
    row_op<LF_PROJECT>(P, nullptr, nullptr, nullptr, y, PlusScalars{}, O, B, s);
    from_rows(O, out, B, s);
  }
  void lambda(const float* v, int B, const PlusScalars& ps, float* out, cudaStream_t s) override {
    float* P = rows_.get((size_t)B * N_);
    float* O = rows2_.get((size_t)B * N_);
    to_rows(v, P, B, s);
    row_op<LF_LAMBDA>(P, nullptr, nullptr, nullptr, nullptr, ps, O, B, s);
    from_rows(O, out, B, s);
  }
  void lambda_noise(const float* v, const float* eps, int B, const PlusScalars& ps, float* out, cudaStream_t s) override {
    const long long n = (long long)B * N_, rows = n / K_;
    float* P = rows_.get(n);
    float* Q = rows2_.get(n);
    float* Wv = wv_.get(n);
    float* We = we_.get(n);
    to_rows(v, P, B, s);
    to_rows(eps, Q, B, s);
    // W[row][k] = sum_j V[k][j] * raw[row][j]
    sgemm_batched(true, 1, 1, (int)rows, K_, K_, 1.0f, P, K_, 0, 0, V_, K_, 0, 0, Wv, K_, 0, 0, s);
    sgemm_batched(true, 1, 1, (int)rows, K_, K_, 1.0f, Q, K_, 0, 0, V_, K_, 0, 0, We, K_, 0, 0, s);
    row_op<LF_NOISE>(P, Q, Wv, We, nullptr, ps, P, B, s);
    from_rows(P, out, B, s);
  }

 private:
  void to_rows(const float* x, float* P, int B, cudaStream_t s) const {
    sr_patch_kernel<true><<<blocks((long long)B * N_), 256, 0, s>>>(x, P, B, C_, D_, ratio_);
  }
  void from_rows(const float* P, float* x, int B, cudaStream_t s) const {
    sr_patch_kernel<false><<<blocks((long long)B * N_), 256, 0, s>>>(P, x, B, C_, D_, ratio_);
    CUDA_CHECK(cudaGetLastError());
  }
  template <int FN>
  void row_op(const float* P, const float* Q, const float* Wv, const float* We, const float* yv, const PlusScalars& ps, float* out,
              int B, cudaStream_t s) const {
    const long long rows = (long long)B * N_ / K_;
    srg_rows_kernel<FN><<<blocks(rows * 32), 256, 0, s>>>(P, Q, Wv, We, yv, v0_, u00_, s0_, ps, out, rows, K_);
    CUDA_CHECK(cudaGetLastError());
  }
  const int C_, D_, ratio_, K_;
  const float* V_;
  const float* v0_;   // V[:, 0]
  const float u00_, s0_;
  Scratch rows_;      // the input's patch rows (the Lambda_noise output in place)
  Scratch rows2_;     // the output's patch rows; in Lambda_noise the rows of eps
  Scratch wv_, we_;   // Lambda_noise: the rows of v and of eps times V^T
};

// Inpainting: every entry, the step included, is one fused inpaint_kernel launch
class Inpaint final : public Operator {
 public:
  // rank: per (pixel, channel) entry its index in y, or -1 where the mask drops it; M: the kept entries
  Inpaint(int C, int D, const std::vector<int>& rank, long long M)
      : Operator(M, (long long)C * D * D), C_(C), HW_(D * D), rank_(upload(rank.data(), rank.size())) {}
  void A(const float* x, int B, float* y, cudaStream_t s) override {
    launch<LF_A>(x, nullptr, 0, nullptr, nullptr, StepScalars{}, y, nullptr, B, s);
  }
  void A_pinv(const float* y, int B, float* x, cudaStream_t s) override {
    launch<LF_PINV>(nullptr, nullptr, 0, nullptr, y, StepScalars{}, x, nullptr, B, s);
  }
  void project(const float* x0, const float* y, int B, float* out, cudaStream_t s) override {
    launch<LF_PROJECT>(x0, nullptr, 0, nullptr, y, StepScalars{}, out, nullptr, B, s);
  }
  void lambda(const float* v, int B, const PlusScalars& ps, float* out, cudaStream_t s) override {
    launch<LF_LAMBDA>(v, nullptr, 0, nullptr, nullptr, with_plus(ps), out, nullptr, B, s);
  }
  void lambda_noise(const float* v, const float* eps, int B, const PlusScalars& ps, float* out, cudaStream_t s) override {
    launch<LF_NOISE>(v, eps, N_, nullptr, nullptr, with_plus(ps), out, nullptr, B, s);
  }
  void step(const float* xt, const float* et, long long et_stride, const NoiseSrc& nz, const float* y, int B, const StepScalars& sc,
            float* x0_t, float* xt_next, cudaStream_t s) override {
    noise_dispatch(nz, [&](auto gen) { launch<LF_STEP, decltype(gen)::value>(xt, et, et_stride, nz.tape, y, sc, x0_t, xt_next, B, s, nz); });
  }

 private:
  template <int FN, bool GEN = false>
  void launch(const float* in0, const float* in1, long long in1_stride, const float* in2, const float* y, const StepScalars& sc,
              float* out0, float* out1, int B, cudaStream_t s, const NoiseSrc& nz = NoiseSrc{}) const {
    inpaint_kernel<FN, GEN><<<blocks((long long)B * N_), 256, 0, s>>>(in0, in1, in1_stride, in2, y, rank_, sc, out0, out1, B, C_, HW_,
                                                                       M_, nz);
    CUDA_CHECK(cudaGetLastError());
  }
  const int C_, HW_;
  const int* rank_;
};

// Denoising (svd_operators.py:442-476): A = I, so the residual is x0 - y; Lambda, Lambda_noise and the step are fused
class Denoise final : public Operator {
 public:
  explicit Denoise(long long N) : Operator(N, N) {}
  void A(const float* x, int B, float* y, cudaStream_t s) override {
    CUDA_CHECK(cudaMemcpyAsync(y, x, (size_t)B * N_ * 4, cudaMemcpyDeviceToDevice, s));
  }
  void A_pinv(const float* y, int B, float* x, cudaStream_t s) override {
    CUDA_CHECK(cudaMemcpyAsync(x, y, (size_t)B * N_ * 4, cudaMemcpyDeviceToDevice, s));
  }
  void lambda(const float* v, int B, const PlusScalars& ps, float* out, cudaStream_t s) override {
    launch<LF_LAMBDA>(v, nullptr, 0, nullptr, nullptr, with_plus(ps), out, nullptr, B, s);
  }
  void lambda_noise(const float* v, const float*, int B, const PlusScalars& ps, float* out, cudaStream_t s) override {
    launch<LF_NOISE>(v, nullptr, 0, nullptr, nullptr, with_plus(ps), out, nullptr, B, s);
  }
  void step(const float* xt, const float* et, long long et_stride, const NoiseSrc& nz, const float* y, int B, const StepScalars& sc,
            float* x0_t, float* xt_next, cudaStream_t s) override {
    noise_dispatch(nz, [&](auto gen) { launch<LF_STEP, decltype(gen)::value>(xt, et, et_stride, nz.tape, y, sc, x0_t, xt_next, B, s, nz); });
  }

 protected:
  void residual(const float* x0, const float* y, int B, float* R, cudaStream_t s) override {
    const long long n = (long long)B * N_;
    sub_kernel<<<blocks(n), 256, 0, s>>>(x0, y, R, n);
  }

 private:
  template <int FN, bool GEN = false>
  void launch(const float* in0, const float* in1, long long in1_stride, const float* in2, const float* y, const StepScalars& sc,
              float* out0, float* out1, int B, cudaStream_t s, const NoiseSrc& nz = NoiseSrc{}) const {
    denoise_kernel<FN, GEN><<<blocks((long long)B * N_), 256, 0, s>>>(in0, in1, in1_stride, in2, y, sc, out0, out1, B, N_, nz);
    CUDA_CHECK(cudaGetLastError());
  }
};

// WalshHadamardCS: A keeps M of the transform's coefficients; the residual is one pass in the spectral domain
class WalshHadamard final : public Operator {
 public:
  // perm: the spectral position of each kept coefficient in order; invperm: its inverse
  WalshHadamard(int C, int D, int ratio, const std::vector<int>& perm, const std::vector<int>& invperm)
      : Operator((long long)C * D * D / ratio, (long long)C * D * D), C_(C), D_(D), perm_(upload(perm.data(), perm.size())),
        invperm_(upload(invperm.data(), invperm.size())) {}
  void A(const float* x, int B, float* y, cudaStream_t s) override {
    spec<LF_A>(spectrum(x, B, s), nullptr, nullptr, PlusScalars{}, y, B, s);
  }
  void A_pinv(const float* y, int B, float* x, cudaStream_t s) override {
    spec<LF_PINV>(nullptr, nullptr, y, PlusScalars{}, x, B, s);
    fwht(x, B, s);
  }
  void lambda(const float* v, int B, const PlusScalars& ps, float* out, cudaStream_t s) override {
    spec<LF_LAMBDA>(spectrum(v, B, s), nullptr, nullptr, ps, out, B, s);
    fwht(out, B, s);
  }
  void lambda_noise(const float* v, const float* eps, int B, const PlusScalars& ps, float* out, cudaStream_t s) override {
    spec<LF_NOISE>(v, eps, nullptr, ps, out, B, s);
    fwht(out, B, s);
  }

 protected:
  void residual(const float* x0, const float* y, int B, float* R, cudaStream_t s) override {
    spec<LF_PROJECT>(spectrum(x0, B, s), nullptr, y, PlusScalars{}, R, B, s);
    fwht(R, B, s);
  }

 private:
  // the transform of x, in scratch
  float* spectrum(const float* x, int B, cudaStream_t s) {
    const long long n = (long long)B * N_;
    float* F = spec_.get(n);
    CUDA_CHECK(cudaMemcpyAsync(F, x, n * 4, cudaMemcpyDeviceToDevice, s));
    fwht(F, B, s);
    return F;
  }
  template <int FN>
  void spec(const float* F, const float* F2, const float* y, const PlusScalars& ps, float* out, int B, cudaStream_t s) const {
    const long long n = (long long)B * (FN == LF_A ? M_ : N_);
    wh_spec_kernel<FN><<<blocks(n), 256, 0, s>>>(F, F2, y, perm_, invperm_, ps, out, B, C_, D_ * D_, M_);
    CUDA_CHECK(cudaGetLastError());
  }
  void fwht(float* buf, int B, cudaStream_t s) const {
    const long long rows = (long long)B * C_ * D_;
    const int threads = std::max(128, D_ / 2);
    const int rpb = threads * 2 / D_;
    fwht_rows_kernel<<<(int)cdivll(rows, rpb), threads, (size_t)rpb * D_ * 4, s>>>(buf, D_, rows);
    CUDA_CHECK(cudaGetLastError());
    const size_t smem = (size_t)D_ * 33 * 4;
    // the attribute is per device: set it whenever more than the default 48 KiB is needed (a cached process-wide flag would leave
    // a second GPU of the same process without it)
    if (smem > 48 * 1024) CUDA_CHECK(cudaFuncSetAttribute(fwht_cols_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(D_ / 32, B * C_);
    fwht_cols_kernel<<<grid, 256, smem, s>>>(buf, D_, (float)D_);
    CUDA_CHECK(cudaGetLastError());
  }
  const int C_, D_;
  const int *perm_, *invperm_;
  Scratch spec_;
};

// Deblurring, Deblurring2D (svd_operators.py:934-1166) and SRConv (:851-931): per image and channel, the spectrum of X is
// Vl^T X Vr (k x k), A scales it by the singular table and maps it to y = Ul S Ur^T; A_pinv is the mirror with the reciprocal
// table.  k = D for the deblurs, the low-resolution side for SRConv.  Only Deblurring defines a Lambda.
class Separable final : public Operator {
 public:
  // vl, vr: D x k; ul, ur: k x k (the same matrices on both sides unless Deblurring2D).  d: the singulars per (channel, spectral
  // position), or per position when !per_channel.  sorig: Deblurring's un-thresholded singulars per position, empty without a Lambda
  Separable(int C, int D, int k, const float* vl, const float* vr, const float* ul, const float* ur, const std::vector<float>& d,
            bool per_channel, const std::vector<float>& sorig, const char* name, const char* src, const char* note = "")
      : Operator((long long)C * k * k, (long long)C * D * D, name, src, note), C_(C), D_(D), k_(k), per_channel_(per_channel) {
    vl_ = factor(vl, D, k);
    vr_ = vr == vl ? vl_ : factor(vr, D, k);
    ul_ = factor(ul, k, k);
    ur_ = ur == ul ? ul_ : factor(ur, k, k);
    d_ = upload(d.data(), d.size());
    dinv_ = upload(reciprocals(d.data(), d.size()).data(), d.size());
    if (!sorig.empty()) sorig_ = upload(sorig.data(), sorig.size());
  }
  void A(const float* x, int B, float* y, cudaStream_t s) override {
    float *T = tmp(B), *S = spectral(B);
    sandwich(vl_.t, k_, D_, x, B, vr_.m, D_, k_, T, S, s);
    scale(S, d_, B, s);
    sandwich(ul_.m, k_, k_, S, B, ur_.t, k_, k_, T, y, s);
  }
  void A_pinv(const float* y, int B, float* x, cudaStream_t s) override {
    float *T = tmp(B), *S = spectral(B);
    sandwich(ul_.t, k_, k_, y, B, ur_.m, k_, k_, T, S, s);
    scale(S, dinv_, B, s);
    sandwich(vl_.m, D_, k_, S, B, vr_.t, k_, D_, T, x, s);
  }
  void lambda(const float* v, int B, const PlusScalars& ps, float* out, cudaStream_t s) override {
    if (!sorig_) return Operator::lambda(v, B, ps, out, s);
    const long long n = (long long)B * N_;
    float *T = tmp(B), *S = spectral(B);
    sandwich(vl_.t, D_, D_, v, B, vl_.m, D_, D_, T, S, s);
    deblur_coeff_kernel<LF_LAMBDA><<<blocks(n), 256, 0, s>>>(S, nullptr, sorig_, ps, S, D_ * D_, n);
    sandwich(vl_.m, D_, D_, S, B, vl_.t, D_, D_, T, out, s);
  }
  void lambda_noise(const float* v, const float* eps, int B, const PlusScalars& ps, float* out, cudaStream_t s) override {
    if (!sorig_) return Operator::lambda_noise(v, eps, B, ps, out, s);
    const long long n = (long long)B * N_;
    float *T = tmp(B), *S = spectral(B);
    deblur_coeff_kernel<LF_NOISE><<<blocks(n), 256, 0, s>>>(v, eps, sorig_, ps, S, D_ * D_, n);
    sandwich(vl_.m, D_, D_, S, B, vl_.t, D_, D_, T, out, s);
  }

 private:
  struct Factor {
    const float *m, *t;   // the matrix and its transpose
  };
  Factor factor(const float* host, int r, int c) {
    const std::vector<float> t = transpose(host, r, c);
    return {upload(host, (size_t)r * c), upload(t.data(), t.size())};
  }
  // a GEMM's intermediate: at most k x D per image
  float* tmp(int B) { return t_.get((size_t)B * C_ * k_ * D_); }
  // the k x k spectrum per image
  float* spectral(int B) { return s_.get((size_t)B * C_ * k_ * k_); }
  void scale(float* S, const float* table, int B, cudaStream_t s) const {
    const long long n = (long long)B * C_ * k_ * k_;
    mul_table_kernel<<<blocks(n), 256, 0, s>>>(S, table, per_channel_ ? 1 : 0, C_, k_ * k_, n);
  }
  // out[b] = L (lr x lc) * X[b] (lc x rr) * R (rr x rc), X: B*C images; T: scratch of lr*rr per image
  void sandwich(const float* L, int lr, int lc, const float* X, int B, const float* R, int rr, int rc, float* T, float* out,
                cudaStream_t s) const {
    const int nb = B * C_;
    sgemm_batched(false, nb, 1, lr, rr, lc, 1.0f, L, lc, 0, 0, X, rr, (long long)lc * rr, 0, T, rr, (long long)lr * rr, 0, s);
    sgemm_batched(false, nb, 1, lr, rc, rr, 1.0f, T, rr, (long long)lr * rr, 0, R, rc, 0, 0, out, rc, (long long)lr * rc, 0, s);
    CUDA_CHECK(cudaGetLastError());
  }
  const int C_, D_, k_;
  const bool per_channel_;
  Factor vl_, vr_, ul_, ur_;
  const float *d_, *dinv_, *sorig_ = nullptr;
  Scratch t_, s_;
};

// CS (svd_operators.py:101-159): the first cs_size coefficients of each 32 x 32 patch in the basis V
class Cs final : public Operator {
 public:
  // V: the 1024 x 1024 basis
  Cs(int C, int D, int cs_size, const float* V)
      : Operator((long long)C * (D / 32) * (D / 32) * cs_size, (long long)C * D * D, "CS", "svd_operators.py:101-159"), C_(C), D_(D),
        cs_size_(cs_size), V_(upload(V, (size_t)1024 * 1024)) {}
  void A(const float* x, int B, float* y, cudaStream_t s) override {
    const long long n = (long long)B * N_;
    float* P = patches_.get(n);
    cs_patch_kernel<true><<<blocks(n), 256, 0, s>>>(x, P, B, C_, D_);
    // first cs_size coefficients of V^T patch  ==  P [rows x 1024] . V[:, :cs]
    sgemm_batched(false, 1, 1, (int)(n / 1024), cs_size_, 1024, 1.0f, P, 1024, 0, 0, V_, 1024, 0, 0, y, cs_size_, 0, 0, s);
    CUDA_CHECK(cudaGetLastError());
  }
  void A_pinv(const float* y, int B, float* x, cudaStream_t s) override {
    const long long n = (long long)B * N_;
    float* P = patches_.get(n);
    // V (c, 0, ..)  ==  Y [rows x cs] . V[:, :cs]^T
    sgemm_batched(true, 1, 1, (int)(n / 1024), 1024, cs_size_, 1.0f, y, cs_size_, 0, 0, V_, 1024, 0, 0, P, 1024, 0, 0, s);
    cs_patch_kernel<false><<<blocks(n), 256, 0, s>>>(P, x, B, C_, D_);
    CUDA_CHECK(cudaGetLastError());
  }

 private:
  const int C_, D_, cs_size_;
  const float* V_;
  Scratch patches_;   // the patches as rows of 1024
};

// GeneralA (svd_operators.py:173-208): y = U (s * (V^T x)[:m]),  x = V add_zeros((1/s) * (U^T y))  — three small fp32 GEMMs
// over the batch
class General final : public Operator {
 public:
  // Vm: the first m columns of V (n x m), the only ones that meet a non-zero coefficient; U: m x m; sv: the m singulars
  General(long long n, int m, const std::vector<float>& Vm, const float* U, const float* sv)
      : Operator(m, n, "GeneralA", "svd_operators.py:173-208"), V_(upload(Vm.data(), Vm.size())), U_(upload(U, (size_t)m * m)),
        d_(upload(sv, (size_t)m)), dinv_(upload(reciprocals(sv, m).data(), (size_t)m)) {}
  void A(const float* x, int B, float* y, cudaStream_t s) override {
    const int n = (int)N_, m = (int)M_;
    float* T = t_.get((size_t)B * m);
    sgemm_batched(false, 1, 1, B, m, n, 1.0f, x, n, 0, 0, V_, m, 0, 0, T, m, 0, 0, s);          // T = X Vm
    mul_table_kernel<<<blocks((long long)B * m), 256, 0, s>>>(T, d_, 0, 1, m, (long long)B * m);
    sgemm_batched(true, 1, 1, B, m, m, 1.0f, T, m, 0, 0, U_, m, 0, 0, y, m, 0, 0, s);           // y[b][k] = sum_j U[k][j] T[b][j]
    CUDA_CHECK(cudaGetLastError());
  }
  void A_pinv(const float* y, int B, float* x, cudaStream_t s) override {
    const int n = (int)N_, m = (int)M_;
    float* T = t_.get((size_t)B * m);
    sgemm_batched(false, 1, 1, B, m, m, 1.0f, y, m, 0, 0, U_, m, 0, 0, T, m, 0, 0, s);          // T[b][j] = sum_k y[b][k] U[k][j]
    mul_table_kernel<<<blocks((long long)B * m), 256, 0, s>>>(T, dinv_, 0, 1, m, (long long)B * m);
    sgemm_batched(true, 1, 1, B, n, m, 1.0f, T, m, 0, 0, V_, m, 0, 0, x, n, 0, 0, s);           // x[b][i] = sum_j V[i][j] T[b][j]
    CUDA_CHECK(cudaGetLastError());
  }

 private:
  const float *V_, *U_, *d_, *dinv_;
  Scratch t_;   // the m coefficients per row
};

}  // namespace

Operator* make_operator(const ddnm_operator_desc& d) {
  const int channels = d.channels, img_dim = d.img_dim, ratio = d.ratio, n2 = img_dim * img_dim;
  const float *v_small = d.v_small, *u_small = d.u_small, *singulars = d.singulars;
  const long long* perm = d.perm;
  DDNM_CHECK(channels >= 1 && img_dim >= 2, "bad operator geometry");
  switch (d.kind) {
    case OP_SR: {
      DDNM_CHECK(ratio >= 1 && img_dim % ratio == 0, "img_dim % ratio");  // svd_operators.py:481
      DDNM_CHECK(ratio <= 64, "SuperResolution: ratio <= 64");
      DDNM_CHECK(v_small && u_small && singulars, "SuperResolution needs V_small, U_small, singulars_small");
      // 2 / 4 / 8: one thread per patch with the basis in shared memory; any other ratio (evaluation.sh runs 16x): patch rows +
      // the K x K basis as a small GEMM
      if (ratio == 2 || ratio == 4 || ratio == 8) return new Local(channels, img_dim, ratio * ratio, v_small, u_small[0], singulars[0]);
      return new PatchRows(channels, img_dim, ratio, v_small, u_small[0], singulars[0]);
    }
    case OP_COLOR:
      DDNM_CHECK(channels == 3 && v_small && u_small && singulars, "Colorization needs 3 channels and its 3x3 basis");
      return new Local(channels, img_dim, 3, v_small, u_small[0], singulars[0]);
    case OP_INPAINT: {
      DDNM_CHECK(d.mask, "Inpainting needs the mask");
      std::vector<int> rank((size_t)n2 * channels);
      int r = 0;
      for (size_t e = 0; e < rank.size(); ++e) rank[e] = d.mask[e] != 0 ? r++ : -1;
      return new Inpaint(channels, img_dim, rank, r);
    }
    case OP_WH: {
      DDNM_CHECK(perm && ratio >= 1, "WalshHadamardCS needs perm");
      DDNM_CHECK((img_dim & (img_dim - 1)) == 0 && img_dim >= 32 && img_dim <= 1024,
                 "WalshHadamardCS: img_dim must be a power of two in [32, 1024]");
      std::vector<int> p(n2), ip(n2, -1);
      for (int i = 0; i < n2; ++i) {
        DDNM_CHECK(perm[i] >= 0 && perm[i] < n2 && ip[perm[i]] < 0, "perm is not a permutation");
        p[i] = (int)perm[i];
        ip[perm[i]] = i;
      }
      return new WalshHadamard(channels, img_dim, ratio, p, ip);
    }
    case OP_DENOISE:
      return new Denoise((long long)channels * n2);
    case OP_CS:
      // ratio carries cs_size = int(32*32*cs_ratio) (svd_operators.py:111)
      DDNM_CHECK(v_small && img_dim % 32 == 0 && ratio >= 1 && ratio <= 1024, "CS needs V_small [1024,1024], img_dim % 32, 1 <= cs_size <= 1024");
      return new Cs(channels, img_dim, ratio, v_small);
    case OP_DEBLUR:
    case OP_DEBLUR2D: {
      const bool two = d.kind == OP_DEBLUR2D;   // svd_operators.py:1094-1166: different 1-D factors on the two sides, no Lambda
      if (!two) DDNM_CHECK(d.singulars_orig != nullptr, "Deblurring needs the un-thresholded singulars");
      DDNM_CHECK(v_small && u_small && singulars && perm, "Deblurring needs U, V, singular tables and perm");
      if (two) DDNM_CHECK(d.v_small2 && d.u_small2, "Deblurring2D needs the second pair of factors");
      // singulars() = _singulars.repeat(1, 3) is TILED while spectral vectors are (pos, chan)-interleaved
      // (svd_operators.py:1001 vs :984): D[c][perm[p]] = S[(C*p + c) mod n2]
      std::vector<float> tD((size_t)channels * n2), tS(two ? 0 : n2);
      for (int p = 0; p < n2; ++p) {
        const long long q = perm[p];
        DDNM_CHECK(q >= 0 && q < n2, "bad perm entry");
        for (int c = 0; c < channels; ++c) tD[(size_t)c * n2 + q] = singulars[((long long)channels * p + c) % n2];
        if (!two) tS[q] = d.singulars_orig[p];
      }
      return new Separable(channels, img_dim, img_dim, v_small, two ? d.v_small2 : v_small, u_small, two ? d.u_small2 : u_small, tD,
                           true, tS, two ? "Deblurring2D" : "Deblurring", two ? "svd_operators.py:1094-1166" : "svd_operators.py:934-1091");
    }
    case OP_SRCONV: {
      DDNM_CHECK(v_small && u_small && singulars && ratio >= 1 && img_dim % ratio == 0, "SRConv needs U_small, V_small, singulars_small");
      const int sm = img_dim / ratio;
      std::vector<float> vk((size_t)img_dim * sm), s2((size_t)sm * sm);   // vk: the first sm columns of V_small
      for (int i = 0; i < img_dim; ++i)
        for (int j = 0; j < sm; ++j) vk[(size_t)i * sm + j] = v_small[(size_t)i * img_dim + j];
      for (int i = 0; i < sm; ++i)
        for (int j = 0; j < sm; ++j) s2[(size_t)i * sm + j] = singulars[i] * singulars[j];
      return new Separable(channels, img_dim, sm, vk.data(), vk.data(), u_small, u_small, s2, false, {}, "SRConv", "svd_operators.py:851-931",
                           " for sr_bicubic");
    }
    case OP_GENERAL: {
      // dense A = U diag(s) V^T with FULL factors U [m,m], V [n,n]; only the first m columns of V ever meet a non-zero coefficient
      // (A(): temp[:, :m]; A_pinv(): add_zeros pads m..n with zeros).  x is a flat vector of n = img_dim entries per row
      DDNM_CHECK(channels == 1, "GeneralA: pass channels = 1 and img_dim = n (columns of A)");
      const long long n = img_dim;
      const int m = ratio;
      DDNM_CHECK(v_small && u_small && singulars && m >= 1 && m <= n, "GeneralA needs U [m,m], V [n,n], singulars [m] with m <= n");
      std::vector<float> vm((size_t)n * m);
      for (long long i = 0; i < n; ++i)
        for (int j = 0; j < m; ++j) vm[(size_t)i * m + j] = v_small[(size_t)i * n + j];
      return new General(n, m, vm, u_small, singulars);
    }
    default:
      throw Error("unknown operator kind");
  }
}

}  // namespace ddnm

// ------------------------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------------------------
using namespace ddnm;
extern "C" {

int ddnm_operator_create(const ddnm_operator_desc* d, void** handle) {
  DDNM_API_BEGIN
  DDNM_CHECK(d && handle, "null argument");
  *handle = make_operator(*d);
  DDNM_API_END
}
long long ddnm_operator_y_dim(void* h) { return h ? static_cast<Operator*>(h)->y_dim() : -1; }
int ddnm_operator_A(void* h, const float* x, int B, float* y, void* stream) {
  DDNM_API_BEGIN
  static_cast<Operator*>(h)->A(x, B, y, (cudaStream_t)stream);
  DDNM_API_END
}
int ddnm_operator_A_pinv(void* h, const float* y, int B, float* x, void* stream) {
  DDNM_API_BEGIN
  static_cast<Operator*>(h)->A_pinv(y, B, x, (cudaStream_t)stream);
  DDNM_API_END
}
int ddnm_operator_project(void* h, const float* x0, const float* y, int B, float* out, void* stream) {
  DDNM_API_BEGIN
  static_cast<Operator*>(h)->project(x0, y, B, out, (cudaStream_t)stream);
  DDNM_API_END
}
int ddnm_operator_lambda(void* h, const float* v, int B, float a, float sigma_y, float sigma_t, float eta, float* out, void* stream) {
  DDNM_API_BEGIN
  static_cast<Operator*>(h)->lambda(v, B, make_plus(a, sigma_y, sigma_t, eta), out, (cudaStream_t)stream);
  DDNM_API_END
}
int ddnm_operator_lambda_noise(void* h, const float* v, const float* eps, int B, float a, float sigma_y, float sigma_t, float eta,
                               float* out, void* stream) {
  DDNM_API_BEGIN
  static_cast<Operator*>(h)->lambda_noise(v, eps, B, make_plus(a, sigma_y, sigma_t, eta), out, (cudaStream_t)stream);
  DDNM_API_END
}
int ddnm_operator_destroy(void* h) {
  DDNM_API_BEGIN
  delete static_cast<Operator*>(h);
  DDNM_API_END
}

}  // extern "C"

// The "simplified" DDNM+ loop of the reference runner (guided_diffusion/diffusion.py:211-415, README quick start):
// image-space operators built from mask / colour-to-gray / average-pool (diffusion.py:244-290, helpers :27-42) and a scalar
// lambda_t / gamma_t update (:355-376).  One fused kernel per step; thread = one scale x scale patch across the 3 channels.
// The loop around the step is the SVD samplers' sample_range (sampler.cu).
#include <cmath>

#include "../../include/ddnm_b200.h"
#include "api_util.cuh"
#include "operators.cuh"

namespace ddnm {

struct SimpScalars {
  float sqrt_at, sqrt_1m_at, sqrt_atn, c1, c2, lambda_t, gamma_t;
};

enum { SF_A = 0, SF_AP = 1, SF_STEP = 2 };

// A(z) = pool(gray(z * mask)),  Ap(v) = gray2color(upsample(v)) * mask   (whichever stages are enabled)
// GEN (SF_STEP only): the draws are generated in registers from gen, z unused.  A patch row is S consecutive elements starting
// at a multiple of S, so one generator call serves min(S, 4) values: noise_at (S = 1), noise_pair (2), noise_quad (4, 8).
template <int S, int FN, bool GEN = false>
__global__ void __launch_bounds__(128) simp_kernel(const float* __restrict__ in0, const float* __restrict__ et, long long et_stride,
                                                   const float* __restrict__ z, const float* __restrict__ y, SimpDeg dg, SimpScalars sc,
                                                   float* __restrict__ out0, float* __restrict__ out1, int B, NoiseSrc gen) {
  constexpr int K = S * S;
  const int D = dg.D, yd = D / S;
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)B * yd * yd) return;
  const int px = (int)(g % yd), py = (int)((g / yd) % yd), b = (int)(g / ((long long)yd * yd));
  const long long HW = (long long)D * D, img = 3 * HW;
  const float cf = (float)(1.0 / 3.0);
  const float basef = (float)((1.0 / 3.0) * (1.0 / 3.0) + (1.0 / 3.0) * (1.0 / 3.0) + (1.0 / 3.0) * (1.0 / 3.0));
  auto off = [&](int c, int k) { return (long long)c * HW + (long long)(py * S + k / S) * D + (px * S + k % S); };
  float m[K];
#pragma unroll
  for (int k = 0; k < K; ++k) m[k] = dg.use_mask ? __ldg(dg.mask + (long long)(py * S + k / S) * D + (px * S + k % S)) : 1.f;
  const long long yo = (long long)b * 3 * yd * yd + (long long)py * yd + px;   // + c*yd*yd

  if (FN == SF_AP) {
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = y[yo + (long long)c * yd * yd];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int k = 0; k < K; ++k) {
        float w = dg.use_gray ? __fdiv_rn(__fmul_rn(v[0], cf), basef) : v[c];
        if (dg.use_mask) w = __fmul_rn(w, m[k]);
        out0[(long long)b * img + off(c, k)] = w;
      }
    return;
  }

  float x0[3][K];
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const float xv = in0[(long long)b * img + off(c, k)];
      if (FN == SF_STEP) {
        const float e = et[(long long)b * et_stride + off(c, k)];
        x0[c][k] = __fdiv_rn(__fsub_rn(xv, __fmul_rn(e, sc.sqrt_1m_at)), sc.sqrt_at);
        out0[(long long)b * img + off(c, k)] = x0[c][k];
      } else {
        x0[c][k] = xv;
      }
    }
  // A
  float a[3];
  {
    float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < K; ++k) {
      float t0 = x0[0][k], t1 = x0[1][k], t2 = x0[2][k];
      if (dg.use_mask) { t0 = __fmul_rn(t0, m[k]); t1 = __fmul_rn(t1, m[k]); t2 = __fmul_rn(t2, m[k]); }
      if (dg.use_gray) {
        const float gk = __fadd_rn(__fadd_rn(__fmul_rn(t0, cf), __fmul_rn(t1, cf)), __fmul_rn(t2, cf));
        t0 = t1 = t2 = gk;
      }
      acc[0] = __fadd_rn(acc[0], t0); acc[1] = __fadd_rn(acc[1], t1); acc[2] = __fadd_rn(acc[2], t2);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) a[c] = K > 1 ? __fdiv_rn(acc[c], (float)K) : acc[c];
  }
  if (FN == SF_A) {
#pragma unroll
    for (int c = 0; c < 3; ++c) out0[yo + (long long)c * yd * yd] = a[c];
    return;
  }
  float r[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) r[c] = __fsub_rn(a[c], y[yo + (long long)c * yd * yd]);
  constexpr int W = S >= 4 ? 4 : S;   // values per generator call
  float zg[4];
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int k = 0; k < K; ++k) {
      float w = dg.use_gray ? __fdiv_rn(__fmul_rn(r[0], cf), basef) : r[c];
      if (dg.use_mask) w = __fmul_rn(w, m[k]);
      const float x0h = __fsub_rn(x0[c][k], __fmul_rn(sc.lambda_t, w));                       // Eq. 17 (:373)
      const float e = et[(long long)b * et_stride + off(c, k)];
      if (GEN && k % W == 0) {
        if (W == 4) {
          const float4 v = noise_quad(gen, b, off(c, k) >> 2);
          zg[0] = v.x; zg[1] = v.y; zg[2] = v.z; zg[3] = v.w;
        } else if (W == 2) {
          const float2 v = noise_pair(gen, b, off(c, k) >> 1);
          zg[0] = v.x; zg[1] = v.y;
        } else {
          zg[0] = noise_at(gen, b, off(c, k));
        }
      }
      const float zz = GEN ? zg[k % W] : z[(long long)b * img + off(c, k)];
      const float nz = __fmul_rn(sc.gamma_t, __fadd_rn(__fmul_rn(sc.c1, zz), __fmul_rn(sc.c2, e)));  // (:381)
      out1[(long long)b * img + off(c, k)] = __fadd_rn(__fmul_rn(sc.sqrt_atn, x0h), nz);
    }
}

// Any other scale (evaluation.sh runs sr_averagepooling with deg_scale 16): one WARP per patch, lanes stride over the S*S pixels,
// the three channel sums meet through shuffles.  Same arithmetic per element as simp_kernel; the pooled sums are re-associated.
template <int FN, bool GEN = false>   // GEN (SF_STEP only): noise_at per value (a lane's pixels are 32 apart), z unused
__global__ void __launch_bounds__(128) simp_generic_kernel(const float* __restrict__ in0, const float* __restrict__ et, long long et_stride,
                                                           const float* __restrict__ z, const float* __restrict__ y, SimpDeg dg,
                                                           SimpScalars sc, float* __restrict__ out0, float* __restrict__ out1, int B,
                                                           NoiseSrc gen) {
  const int S = dg.scale, K = S * S;
  const int D = dg.D, yd = D / S;
  const long long g = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (g >= (long long)B * yd * yd) return;
  const int px = (int)(g % yd), py = (int)((g / yd) % yd), b = (int)(g / ((long long)yd * yd));
  const long long HW = (long long)D * D, img = 3 * HW;
  const float cf = (float)(1.0 / 3.0);
  const float basef = (float)((1.0 / 3.0) * (1.0 / 3.0) + (1.0 / 3.0) * (1.0 / 3.0) + (1.0 / 3.0) * (1.0 / 3.0));
  auto pix = [&](int k) { return (long long)(py * S + k / S) * D + (px * S + k % S); };
  const long long yo = (long long)b * 3 * yd * yd + (long long)py * yd + px;   // + c*yd*yd
  if (FN == SF_AP) {
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = y[yo + (long long)c * yd * yd];
    for (int k = lane; k < K; k += 32) {
      const float m = dg.use_mask ? __ldg(dg.mask + pix(k)) : 1.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float w = dg.use_gray ? __fdiv_rn(__fmul_rn(v[0], cf), basef) : v[c];
        if (dg.use_mask) w = __fmul_rn(w, m);
        out0[(long long)b * img + (long long)c * HW + pix(k)] = w;
      }
    }
    return;
  }
  float acc[3] = {0.f, 0.f, 0.f};
  for (int k = lane; k < K; k += 32) {
    const float m = dg.use_mask ? __ldg(dg.mask + pix(k)) : 1.f;
    float t[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const long long o = (long long)c * HW + pix(k);
      const float xv = in0[(long long)b * img + o];
      if (FN == SF_STEP) {
        const float e = et[(long long)b * et_stride + o];
        t[c] = __fdiv_rn(__fsub_rn(xv, __fmul_rn(e, sc.sqrt_1m_at)), sc.sqrt_at);
        out0[(long long)b * img + o] = t[c];
      } else {
        t[c] = xv;
      }
      if (dg.use_mask) t[c] = __fmul_rn(t[c], m);
    }
    if (dg.use_gray) {
      const float gk = __fadd_rn(__fadd_rn(__fmul_rn(t[0], cf), __fmul_rn(t[1], cf)), __fmul_rn(t[2], cf));
      t[0] = t[1] = t[2] = gk;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] = __fadd_rn(acc[c], t[c]);
  }
  float a[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v = acc[c];
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    a[c] = K > 1 ? __fdiv_rn(v, (float)K) : v;
  }
  if (FN == SF_A) {
    if (lane < 3) out0[yo + (long long)lane * yd * yd] = lane == 0 ? a[0] : (lane == 1 ? a[1] : a[2]);
    return;
  }
  float r[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) r[c] = __fsub_rn(a[c], y[yo + (long long)c * yd * yd]);
  for (int k = lane; k < K; k += 32) {
    const float m = dg.use_mask ? __ldg(dg.mask + pix(k)) : 1.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const long long o = (long long)c * HW + pix(k);
      float w = dg.use_gray ? __fdiv_rn(__fmul_rn(r[0], cf), basef) : r[c];
      if (dg.use_mask) w = __fmul_rn(w, m);
      const float x0 = out0[(long long)b * img + o];                                            // written above by this thread
      const float x0h = __fsub_rn(x0, __fmul_rn(sc.lambda_t, w));                               // Eq. 17 (:373)
      const float e = et[(long long)b * et_stride + o];
      const float zz = GEN ? noise_at(gen, b, o) : z[(long long)b * img + o];
      const float nz = __fmul_rn(sc.gamma_t, __fadd_rn(__fmul_rn(sc.c1, zz), __fmul_rn(sc.c2, e)));  // (:381)
      out1[(long long)b * img + o] = __fadd_rn(__fmul_rn(sc.sqrt_atn, x0h), nz);
    }
  }
}

template <int FN, bool GEN = false>
static void simp_launch(const SimpDeg& dg, const float* in0, const float* et, long long et_stride, const float* z, const float* y,
                        const SimpScalars& sc, float* out0, float* out1, int B, cudaStream_t st, const NoiseSrc& gen = NoiseSrc{}) {
  const int yd = dg.D / dg.scale;
  const long long groups = (long long)B * yd * yd;
  const int grid = (int)cdivll(groups, 128);
  switch (dg.scale) {
    case 1: simp_kernel<1, FN, GEN><<<grid, 128, 0, st>>>(in0, et, et_stride, z, y, dg, sc, out0, out1, B, gen); break;
    case 2: simp_kernel<2, FN, GEN><<<grid, 128, 0, st>>>(in0, et, et_stride, z, y, dg, sc, out0, out1, B, gen); break;
    case 4: simp_kernel<4, FN, GEN><<<grid, 128, 0, st>>>(in0, et, et_stride, z, y, dg, sc, out0, out1, B, gen); break;
    case 8: simp_kernel<8, FN, GEN><<<grid, 128, 0, st>>>(in0, et, et_stride, z, y, dg, sc, out0, out1, B, gen); break;
    default:   // any other scale dividing the image size
      simp_generic_kernel<FN, GEN><<<(int)cdivll(groups * 32, 128), 128, 0, st>>>(in0, et, et_stride, z, y, dg, sc, out0, out1, B, gen);
  }
  CUDA_CHECK(cudaGetLastError());
}

SimpDeg make_deg(const ddnm_simple_deg* d) {
  DDNM_CHECK(d != nullptr, "null degradation");
  DDNM_CHECK(d->channels == 3 && d->img_dim > 0 && d->scale >= 1 && d->img_dim % d->scale == 0, "bad simplified degradation");
  DDNM_CHECK(!d->use_mask || d->mask != nullptr, "mask enabled but no mask given");
  DDNM_CHECK(d->image_mask == nullptr, "per-image masks are read by the hq entry points only");
  SimpDeg g;
  g.use_mask = d->use_mask; g.use_gray = d->use_gray; g.scale = d->scale; g.D = d->img_dim; g.mask = d->mask;
  return g;
}

void simplified_step(const SimpDeg& dg, const float* xt, const float* et, long long et_stride, const NoiseSrc& noise, const float* y,
                     int B, const StepScalars& sc, float at_next, float sigma_y, float* x0t, float* xt_next, cudaStream_t st) {
  SimpScalars s{sc.sqrt_at, sc.sqrt_1m_at, sc.sqrt_atn, sc.c1, sc.c2, 0.0f, 0.0f};
  // Eq. 19 with the runner's sigma_t = sqrt(1 - at_next**2)  (diffusion.py:356, :366-371)
  const float sigma_t = std::sqrt(1.0f - at_next * at_next);
  const float asy = at_next * sigma_y;
  if (sigma_t >= asy) {
    s.lambda_t = 1.0f;
    s.gamma_t = std::sqrt(sigma_t * sigma_t - asy * asy);
  } else {
    s.lambda_t = sigma_t / asy;
    s.gamma_t = 0.0f;
  }
  noise_dispatch(noise, [&](auto gen) {
    simp_launch<SF_STEP, decltype(gen)::value>(dg, xt, et, et_stride, noise.tape, y, s, x0t, xt_next, B, st, noise);
  });
}

void simplified_A(const ddnm_simple_deg* d, const float* x, int B, float* y, cudaStream_t st) {
  SimpScalars s{};
  simp_launch<SF_A>(make_deg(d), x, nullptr, 0, nullptr, nullptr, s, y, nullptr, B, st);
}
void simplified_Ap(const ddnm_simple_deg* d, const float* y, int B, float* x, cudaStream_t st) {
  SimpScalars s{};
  simp_launch<SF_AP>(make_deg(d), nullptr, nullptr, 0, nullptr, y, s, x, nullptr, B, st);
}

}  // namespace ddnm

using namespace ddnm;
extern "C" {
int ddnm_simplified_A(const ddnm_simple_deg* d, const float* x, int B, float* y, void* stream) {
  DDNM_API_BEGIN
  simplified_A(d, x, B, y, (cudaStream_t)stream);
  DDNM_API_END
}
int ddnm_simplified_Ap(const ddnm_simple_deg* d, const float* y, int B, float* x, void* stream) {
  DDNM_API_BEGIN
  simplified_Ap(d, y, B, x, (cudaStream_t)stream);
  DDNM_API_END
}
}

// hq_demo's arbitrary-size DDNM ("mask-shift" restoration): the per-step arithmetic of
//   hq_demo/guided_diffusion/gaussian_diffusion.py:318-390 (p_mean_variance's "DDNM core": x0_t from eps, clipping, Eq. 17
//   x0_t_hat = lambda_t*Apy + x0_t - lambda_t*Ap(A(x0_t)), the mask-shift overwrite from the canvas, the posterior mean with
//   variance = gamma_t), :431-493 (p_sample, incl. the classifier's condition_mean :414-430) and :208-217 (_undo),
// plus the canvas preparation Ap(A_temp(gt)) of :651-655 for an arbitrary H x W.  The window / time loops stay on the host
// (ddnm_b200/hq.py), as in the reference; every tensor operation of a step runs here.
#include <cmath>
#include <type_traits>

#include "../../include/ddnm_b200.h"
#include "api_util.cuh"
#include "operators.cuh"

namespace ddnm {

// x0_t = clamp(sqrt_recip_alphas_cumprod*x - sqrt_recipm1_alphas_cumprod*eps, -1, 1)       (:404-411, :296-300)
__global__ void hq_x0_kernel(const float* __restrict__ x, const float* __restrict__ mo, long long mo_stride, float c_recip, float c_recipm1,
                             int clip, float* __restrict__ x0, long long img, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long b = i / img, r = i - b * img;
  float v = __fsub_rn(__fmul_rn(c_recip, x[i]), __fmul_rn(c_recipm1, mo[b * mo_stride + r]));
  if (clip) v = fminf(fmaxf(v, -1.0f), 1.0f);
  x0[i] = v;
}

struct HqRect { int dy, dx, h, w, sy, sx; };   // x0_hat[:, :, dy:dy+h, dx:dx+w] = canvas[:, :, sy:sy+h, sx:sx+w]

// the mask-shift overwrite of x0_hat element (bc, py, px); the second rectangle is applied after the first (reference order
// :363-384), so it wins where they overlap
__device__ __forceinline__ float hq_shift(float v, const float* __restrict__ canvas, int cH, int cW, const HqRect& r0, const HqRect& r1,
                                          long long bc, int py, int px) {
  if (r0.h > 0 && py >= r0.dy && py < r0.dy + r0.h && px >= r0.dx && px < r0.dx + r0.w)
    v = canvas[(bc * cH + (r0.sy + py - r0.dy)) * cW + (r0.sx + px - r0.dx)];
  if (r1.h > 0 && py >= r1.dy && py < r1.dy + r1.h && px >= r1.dx && px < r1.dx + r1.w)
    v = canvas[(bc * cH + (r1.sy + py - r1.dy)) * cW + (r1.sx + px - r1.dx)];
  return v;
}

// x0_hat = lambda*Apy + x0_t - lambda*ApA; mask-shift overwrite; mean = coef1*x0_hat + coef2*x (+ gamma*grad);
// x_next = mean + nonzero*sqrt(gamma)*noise
// GEN: the draw is generated in registers from gen, z unused
template <bool GEN>
__global__ void hq_combine_kernel(const float* __restrict__ x, const float* __restrict__ x0t, const float* __restrict__ apa,
                                  const float* __restrict__ apy, const float* __restrict__ canvas, int cH, int cW, HqRect r0, HqRect r1,
                                  const float* __restrict__ grad, const float* __restrict__ z, ddnm_hq_scalars s,
                                  float* __restrict__ x0hat, float* __restrict__ xn, int C, int D, long long n, NoiseSrc gen) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int px = (int)(i % D), py = (int)((i / D) % D);
  const long long bc = i / ((long long)D * D);
  float v = __fsub_rn(__fadd_rn(__fmul_rn(s.lambda_t, apy[i]), x0t[i]), __fmul_rn(s.lambda_t, apa[i]));
  v = hq_shift(v, canvas, cH, cW, r0, r1, bc, py, px);
  x0hat[i] = v;
  float mean = __fadd_rn(__fmul_rn(s.coef1, v), __fmul_rn(s.coef2, x[i]));
  if (grad) mean = __fadd_rn(mean, __fmul_rn(s.gamma_t, grad[i]));
  float zi;
  if (GEN) {
    const long long b = bc / C;
    zi = noise_at(gen, (int)b, i - b * C * D * D);
  } else {
    zi = z[i];
  }
  xn[i] = __fadd_rn(mean, __fmul_rn(__fmul_rn(s.nonzero, sqrtf(s.gamma_t)), zi));
}

// ---- per-image keep mask (hq_demo face256, :601-622): A(z) = pool_S(gray(z*m)), Ap(v) = gray2color(MeanUpsample_S(v))*m, with m
// the (B,3,D,D) gt_keep_mask, multiplied (not selected: PNG edge pixels are fractional).  inpainting is S = 1 without gray, so
// Ap(A(z)) = z*m*m needs no pooling; otherwise one pass pools A into y [B, G, D/S, D/S] (G = 1 with gray, else 3).
struct HqMask {
  const float* m;   // [B,3,D,D]
  int gray, S, D;
};

__device__ __forceinline__ float hq_x0_at(const float* __restrict__ x, const float* __restrict__ mo, long long mo_stride, float c_recip,
                                          float c_recipm1, int clip, long long b, long long r, long long img) {
  float v = __fsub_rn(__fmul_rn(c_recip, x[b * img + r]), __fmul_rn(c_recipm1, mo[b * mo_stride + r]));
  if (clip) v = fminf(fmaxf(v, -1.0f), 1.0f);
  return v;
}

// y[b, g, py, px] = A(z) of one S x S patch; z = x0_t from (x, eps) (X0) or `in` itself (the canvas's gt).  Pixels are summed in
// row-major order and divided once, as the simplified operators do.
template <bool X0>
__global__ void hq_mask_A_kernel(const float* __restrict__ in, const float* __restrict__ mo, long long mo_stride, ddnm_hq_scalars s,
                                 HqMask q, float* __restrict__ y, int B) {
  const int S = q.S, D = q.D, yd = D / S, G = q.gray ? 1 : 3;
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)B * G * yd * yd) return;
  const int px = (int)(g % yd), py = (int)((g / yd) % yd), ch = (int)((g / ((long long)yd * yd)) % G);
  const long long b = g / ((long long)G * yd * yd), HW = (long long)D * D, img = 3 * HW;
  const float cf = (float)(1.0 / 3.0);
  auto z = [&](int c, long long o) {
    const long long r = c * HW + o;
    const float v = X0 ? hq_x0_at(in, mo, mo_stride, s.c_recip, s.c_recipm1, s.clip, b, r, img) : in[b * img + r];
    return __fmul_rn(v, q.m[b * img + r]);
  };
  float acc = 0.f;
  for (int k = 0; k < S * S; ++k) {
    const long long o = (long long)(py * S + k / S) * D + (px * S + k % S);
    const float t = q.gray ? __fadd_rn(__fadd_rn(__fmul_rn(z(0, o), cf), __fmul_rn(z(1, o), cf)), __fmul_rn(z(2, o), cf)) : z(ch, o);
    acc = __fadd_rn(acc, t);
  }
  y[g] = S > 1 ? __fdiv_rn(acc, (float)(S * S)) : acc;
}

// Ap(A(z)) at element (b, c, py, px) = flat index i, z_i = that element of z
template <bool POOL>
__device__ __forceinline__ float hq_mask_ApA(const HqMask& q, const float* __restrict__ y, float zi, long long i, long long b, int c,
                                             int py, int px) {
  const float m = q.m[i];
  if (!POOL) return __fmul_rn(__fmul_rn(zi, m), m);
  const int yd = q.D / q.S;
  float w = y[((b * (q.gray ? 1 : 3) + (q.gray ? 0 : c)) * yd + py / q.S) * yd + px / q.S];
  if (q.gray) {
    const float cf = (float)(1.0 / 3.0);
    const float basef = (float)((1.0 / 3.0) * (1.0 / 3.0) + (1.0 / 3.0) * (1.0 / 3.0) + (1.0 / 3.0) * (1.0 / 3.0));
    w = __fdiv_rn(__fmul_rn(w, cf), basef);
  }
  return __fmul_rn(w, m);
}

// the whole step of hq_combine_kernel with x0_t and Ap(A(x0_t)) computed in place (y: the pooled A(x0_t) when POOL)
template <bool POOL, bool GEN>
__global__ void hq_mask_step_kernel(const float* __restrict__ x, const float* __restrict__ mo, long long mo_stride, HqMask q,
                                    const float* __restrict__ y, const float* __restrict__ apy, const float* __restrict__ canvas, int cH,
                                    int cW, HqRect r0, HqRect r1, const float* __restrict__ grad, const float* __restrict__ z,
                                    ddnm_hq_scalars s, float* __restrict__ x0hat, float* __restrict__ xn, long long n, NoiseSrc gen) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int D = q.D;
  const long long HW = (long long)D * D, img = 3 * HW, b = i / img, r = i - b * img, bc = i / HW;
  const int c = (int)(r / HW), py = (int)((r / D) % D), px = (int)(r % D);
  const float x0 = hq_x0_at(x, mo, mo_stride, s.c_recip, s.c_recipm1, s.clip, b, r, img);
  const float apa = hq_mask_ApA<POOL>(q, y, x0, i, b, c, py, px);
  float v = __fsub_rn(__fadd_rn(__fmul_rn(s.lambda_t, apy[i]), x0), __fmul_rn(s.lambda_t, apa));
  v = hq_shift(v, canvas, cH, cW, r0, r1, bc, py, px);
  x0hat[i] = v;
  float mean = __fadd_rn(__fmul_rn(s.coef1, v), __fmul_rn(s.coef2, x[i]));
  if (grad) mean = __fadd_rn(mean, __fmul_rn(s.gamma_t, grad[i]));
  const float zi = GEN ? noise_at(gen, (int)b, r) : z[i];
  xn[i] = __fadd_rn(mean, __fmul_rn(__fmul_rn(s.nonzero, sqrtf(s.gamma_t)), zi));
}

// canvas of a masked degradation: apy = Ap(A(gt))
template <bool POOL>
__global__ void hq_mask_canvas_kernel(const float* __restrict__ gt, HqMask q, const float* __restrict__ y, float* __restrict__ apy,
                                      long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int D = q.D;
  const long long HW = (long long)D * D, b = i / (3 * HW), r = i - b * 3 * HW;
  apy[i] = hq_mask_ApA<POOL>(q, y, gt[i], i, b, (int)(r / HW), (int)((r / D) % D), (int)(r % D));
}

// canvas preparation: Apy_temp = Ap(A_temp(gt)) for gt (B, 3, H, W): block means (optionally of the gray image) broadcast back
__global__ void hq_canvas_kernel(const float* __restrict__ gt, float* __restrict__ out, int B, int H, int W, int scale, int use_gray) {
  const int yd = H / scale, xd = W / scale;
  const long long blk = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (blk >= (long long)B * yd * xd) return;
  const int bx = (int)(blk % xd), by = (int)((blk / xd) % yd), b = (int)(blk / ((long long)xd * yd));
  const float cf = (float)(1.0 / 3.0);
  const float basef = (float)((1.0 / 3.0) * (1.0 / 3.0) + (1.0 / 3.0) * (1.0 / 3.0) + (1.0 / 3.0) * (1.0 / 3.0));
  float acc[3] = {0.f, 0.f, 0.f};
  const long long HW = (long long)H * W;
  for (int k = 0; k < scale * scale; ++k) {
    const long long o = (long long)(by * scale + k / scale) * W + (bx * scale + k % scale);
    float t0 = gt[((long long)b * 3 + 0) * HW + o], t1 = gt[((long long)b * 3 + 1) * HW + o], t2 = gt[((long long)b * 3 + 2) * HW + o];
    if (use_gray) t0 = t1 = t2 = __fadd_rn(__fadd_rn(__fmul_rn(t0, cf), __fmul_rn(t1, cf)), __fmul_rn(t2, cf));
    acc[0] = __fadd_rn(acc[0], t0); acc[1] = __fadd_rn(acc[1], t1); acc[2] = __fadd_rn(acc[2], t2);
  }
  for (int c = 0; c < 3; ++c) {
    float a = scale > 1 ? __fdiv_rn(acc[c], (float)(scale * scale)) : acc[c];
    if (use_gray) a = __fdiv_rn(__fmul_rn(scale > 1 ? __fdiv_rn(acc[0], (float)(scale * scale)) : acc[0], cf), basef);
    for (int k = 0; k < scale * scale; ++k)
      out[((long long)b * 3 + c) * HW + (long long)(by * scale + k / scale) * W + (bx * scale + k % scale)] = a;
  }
}

}  // namespace ddnm

using namespace ddnm;
static HqMask hq_mask(const ddnm_simple_deg* d) {
  DDNM_CHECK(d->channels == 3 && !d->use_mask && d->scale >= 1 && d->img_dim > 0 && d->img_dim % d->scale == 0,
             "per-image mask: 3 channels, no shared mask plane, a scale dividing the image size");
  return HqMask{d->image_mask, d->use_gray ? 1 : 0, d->scale, d->img_dim};
}

// one mask-shift step with the draw from a tape or generated (ddnm_hq_step / ddnm_hq_step_seeded)
static void hq_step(const ddnm_simple_deg* deg, const float* x, const float* model_out, int out_ch, const float* apy, const float* canvas,
                    int canvas_h, int canvas_w, const int* rects, const float* grad, const NoiseSrc& noise, const ddnm_hq_scalars* sc,
                    int B, float* x0_hat, float* x_next, float* scratch, cudaStream_t st) {
  DDNM_CHECK(deg && x && model_out && apy && canvas && rects && sc && x0_hat && x_next && scratch, "null argument");
  DDNM_CHECK(deg->channels == 3 && (out_ch == 3 || out_ch == 6), "hq step: 3-channel images, 3 or 6 model outputs");
  const int D = deg->img_dim;
  const long long img = 3LL * D * D, n = (long long)B * img;
  HqRect r0{rects[0], rects[1], rects[2], rects[3], rects[4], rects[5]}, r1{rects[6], rects[7], rects[8], rects[9], rects[10], rects[11]};
  for (const HqRect& r : {r0, r1})
    if (r.h > 0) DDNM_CHECK(r.w > 0 && r.dy >= 0 && r.dx >= 0 && r.dy + r.h <= D && r.dx + r.w <= D && r.sy >= 0 && r.sx >= 0 &&
                                r.sy + r.h <= canvas_h && r.sx + r.w <= canvas_w, "mask-shift rectangle out of range");
  if (deg->image_mask) {
    const HqMask q = hq_mask(deg);
    const bool pool = q.S > 1 || q.gray;
    const long long mo_stride = (long long)out_ch * D * D;
    const unsigned grid = (unsigned)cdivll(n, 256);
    if (pool) {
      const long long ny = (long long)B * (q.gray ? 1 : 3) * (D / q.S) * (D / q.S);
      hq_mask_A_kernel<true><<<(unsigned)cdivll(ny, 128), 128, 0, st>>>(x, model_out, mo_stride, *sc, q, scratch, B);
    }
    auto launch = [&](auto P) {
      noise_dispatch(noise, [&](auto gen) {
        hq_mask_step_kernel<decltype(P)::value, decltype(gen)::value><<<grid, 256, 0, st>>>(
            x, model_out, mo_stride, q, scratch, apy, canvas, canvas_h, canvas_w, r0, r1, grad, noise.tape, *sc, x0_hat, x_next, n, noise);
      });
    };
    if (pool) launch(std::true_type{});
    else launch(std::false_type{});
    CUDA_CHECK(cudaGetLastError());
    return;
  }
  float* x0t = scratch;          // [n]
  float* apa = scratch + n;      // [n]
  float* yb = scratch + 2 * n;   // [<= n]
  hq_x0_kernel<<<(unsigned)cdivll(n, 256), 256, 0, st>>>(x, model_out, (long long)out_ch * D * D, sc->c_recip, sc->c_recipm1, sc->clip, x0t, img, n);
  simplified_A(deg, x0t, B, yb, st);
  simplified_Ap(deg, yb, B, apa, st);
  noise_dispatch(noise, [&](auto gen) {
    hq_combine_kernel<decltype(gen)::value><<<(unsigned)cdivll(n, 256), 256, 0, st>>>(
        x, x0t, apa, apy, canvas, canvas_h, canvas_w, r0, r1, grad, noise.tape, *sc, x0_hat, x_next, 3, D, n, noise);
  });
  CUDA_CHECK(cudaGetLastError());
}

extern "C" {
int ddnm_hq_canvas(const float* gt, int B, int H, int W, int scale, int use_gray, float* apy_canvas, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(gt && apy_canvas && B >= 1 && scale >= 1 && H % scale == 0 && W % scale == 0, "bad canvas geometry");
  const long long blocks = (long long)B * (H / scale) * (W / scale);
  hq_canvas_kernel<<<(unsigned)cdivll(blocks, 128), 128, 0, (cudaStream_t)stream>>>(gt, apy_canvas, B, H, W, scale, use_gray);
  CUDA_CHECK(cudaGetLastError());
  DDNM_API_END
}

int ddnm_hq_canvas_masked(const ddnm_simple_deg* deg, const float* gt, int B, float* apy, float* scratch, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(deg && deg->image_mask && gt && apy && scratch && B >= 1, "null argument");
  const HqMask q = hq_mask(deg);
  const bool pool = q.S > 1 || q.gray;
  const cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)B * 3 * q.D * q.D;
  if (pool) {
    const long long ny = (long long)B * (q.gray ? 1 : 3) * (q.D / q.S) * (q.D / q.S);
    hq_mask_A_kernel<false><<<(unsigned)cdivll(ny, 128), 128, 0, st>>>(gt, nullptr, 0, ddnm_hq_scalars{}, q, scratch, B);
    hq_mask_canvas_kernel<true><<<(unsigned)cdivll(n, 256), 256, 0, st>>>(gt, q, scratch, apy, n);
  } else {
    hq_mask_canvas_kernel<false><<<(unsigned)cdivll(n, 256), 256, 0, st>>>(gt, q, nullptr, apy, n);
  }
  CUDA_CHECK(cudaGetLastError());
  DDNM_API_END
}

int ddnm_hq_step(const ddnm_simple_deg* deg, const float* x, const float* model_out, int out_ch, const float* apy, const float* canvas,
                 int canvas_h, int canvas_w, const int* rects, const float* grad, const float* noise, const ddnm_hq_scalars* sc, int B,
                 float* x0_hat, float* x_next, float* scratch, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(noise, "null argument");
  hq_step(deg, x, model_out, out_ch, apy, canvas, canvas_h, canvas_w, rects, grad, noise_tape(noise), sc, B, x0_hat, x_next, scratch,
          (cudaStream_t)stream);
  DDNM_API_END
}
int ddnm_hq_step_seeded(const ddnm_simple_deg* deg, const float* x, const float* model_out, int out_ch, const float* apy,
                        const float* canvas, int canvas_h, int canvas_w, const int* rects, const float* grad,
                        const ddnm_noise_seed* seed, unsigned draw, const ddnm_hq_scalars* sc, int B, float* x0_hat, float* x_next,
                        float* scratch, void* stream) {
  DDNM_API_BEGIN
  hq_step(deg, x, model_out, out_ch, apy, canvas, canvas_h, canvas_w, rects, grad, noise_seeded(seed, NZ_HQ, draw, B), sc, B, x0_hat,
          x_next, scratch, (cudaStream_t)stream);
  DDNM_API_END
}

int ddnm_hq_undo(float* x, const float* noise, float sqrt_one_minus_beta, float sqrt_beta, long long n, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(x && noise && n > 0, "null argument");
  // x = sqrt(1 - beta)*x + sqrt(beta)*noise            (:211-217)
  renoise(x, sqrt_one_minus_beta, sqrt_beta, noise_tape(noise), x, n, n, (cudaStream_t)stream);
  DDNM_API_END
}
int ddnm_hq_undo_seeded(float* x, const ddnm_noise_seed* seed, unsigned draw, float sqrt_one_minus_beta, float sqrt_beta, int B,
                        long long per_image, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(x && B >= 1 && per_image > 0, "null argument");
  renoise(x, sqrt_one_minus_beta, sqrt_beta, noise_seeded(seed, NZ_HQ, draw, B), x, (long long)B * per_image, per_image,
          (cudaStream_t)stream);
  DDNM_API_END
}
}

// The DDNM / DDNM+ reverse-diffusion loop (functions/svd_ddnm.py:19-78 and :80-164) and the runner's simplified DDNM+ loop
// (guided_diffusion/diffusion.py:325-395), enqueued on one stream with no host synchronisation: per denoising pair one UNet graph
// launch + one fused update; travel-back pairs are one elementwise kernel.  The reference instead bounces xt / x0_t through host
// memory every step (:67-68, :45).  Both loops are sample_range; they differ only in the step that follows the denoiser.
#include <cmath>
#include <memory>

#include "../../include/ddnm_b200.h"
#include "api_util.cuh"
#include "engine.cuh"
#include "operators.cuh"

namespace ddnm {

// et[b, 0..2] -= sqrt(1 - at) * grad[b]   (svd_ddnm.py:52, :113: et = et - (1 - at).sqrt()[0,0,0,0] * cls_fn(x, t, classes))
__global__ void guide_kernel(float* __restrict__ et, long long et_stride, const float* __restrict__ grad, float s1, long long img,
                             long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long b = i / img, r = i - b * img;
  float* e = et + b * et_stride + r;
  *e = __fsub_rn(*e, __fmul_rn(s1, grad[i]));
}

// Pairs [k0, k1) of the schedule on images of img elements.  State lives in the caller's buffers so that a long schedule can be
// run as several calls with a bounded noise buffer each: xt_state = current iterate (in/out), x0t = last un-projected x0_t
// (in/out, read by travel-back pairs), *have_x0 = whether x0t holds one.  noise = a tape with the draws of exactly these pairs, or
// a generated source (tape == nullptr), whose draw index is the pair's index in the whole schedule.
// step(xt, et, et_stride, z, s, at_next, x0t, xn): a denoising pair's update after the denoiser left eps in et, with the pair's
// DDIM terms in s: x0_t -> x0t, the next iterate -> xn.
template <class Step>
static void sample_range(UNetEngine* unet, long long img, const Step& step, const ddnm_schedule* sc, int k0, int k1, float* xt_state,
                         float* x0t, int* have_x0, const float* y, const NoiseSrc& noise, int B, cudaStream_t st,
                         const int* labels = nullptr, const float* grad_buf = nullptr, ddnm_guidance_fn guide = nullptr,
                         void* user = nullptr) {
  DDNM_CHECK(unet && sc && xt_state && x0t && have_x0 && y, "null argument");
  DDNM_CHECK(unet->batch() == B, "engine was built for a different batch size");   // before anything reads B elements
  DDNM_CHECK(0 <= k0 && k0 <= k1 && k1 <= sc->n_pairs, "pair range outside the schedule");
  DDNM_CHECK((labels != nullptr) == unet->class_conditional(), "class labels go with a class-conditional denoiser, and only with one");
  DDNM_CHECK((guide != nullptr) == (grad_buf != nullptr), "guidance callback and gradient buffer go together");
  const int R = unet->resolution();
  DDNM_CHECK(img == (long long)unet->in_channels() * R * R, "degradation / denoiser image size mismatch");
  DDNM_CHECK(unet->out_ch() == 3 || unet->out_ch() == 6, "denoiser must predict 3 (eps) or 6 (eps, sigma) channels");
  if (labels) unet->set_labels(labels, st);
  const long long n = (long long)B * img;
  const long long et_stride = (long long)unet->out_ch() * R * R;  // 6-channel nets: keep channels 0..2 (:54-55)
  float* xt = unet->x_in();      // the denoiser reads its input here
  float* et = unet->out_buf();   // and leaves eps here
  StreamBuf xn((size_t)n, st);
  CUDA_CHECK(cudaMemcpyAsync(xt, xt_state, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  const float eta = sc->eta;
  const float c_eta = (float)std::sqrt(1.0 - (double)eta * (double)eta);  // (1 - eta ** 2) ** 0.5 as the fp32 scalar torch sees
  for (int k = k0; k < k1; ++k) {
    const int i = sc->t_i[k], j = sc->t_j[k];
    DDNM_CHECK(i >= 0 && i < sc->num_timesteps && j >= -1 && j < sc->num_timesteps, "time index out of range");
    const float at_next = sc->abar[j + 1];
    const float s1n = std::sqrt(1.0f - at_next);
    NoiseSrc z = noise;
    if (z.tape) z.tape += (long long)(k - k0) * n;
    else z.draw = (unsigned)k;
    if (j < i) {
      const float at = sc->abar[i + 1];
      StepScalars s{};
      s.sqrt_at = std::sqrt(at);
      s.sqrt_1m_at = std::sqrt(1.0f - at);
      s.sqrt_atn = std::sqrt(at_next);
      s.c1 = s1n * eta;
      s.c2 = s1n * c_eta;
      unet->fill_t((float)i, st);
      unet->forward(xt, unet->t_in(), et, st);
      if (guide) {
        // the caller fills grad_buf (its classifier's autograd gradient) with work enqueued on this stream
        const int rc = guide(user, k, i, (void*)st);
        DDNM_CHECK(rc == 0, "classifier-guidance callback failed");
        guide_kernel<<<(int)cdivll(n, 256), 256, 0, st>>>(et, et_stride, grad_buf, s.sqrt_1m_at, img, n);
        CUDA_CHECK(cudaGetLastError());
      }
      step(xt, et, et_stride, z, s, at_next, x0t, xn.p);
      *have_x0 = 1;
    } else {
      DDNM_CHECK(*have_x0, "schedule starts with a travel-back step");
      // xt_next = at_next.sqrt() * x0_t + randn * (1 - at_next).sqrt()      (svd_ddnm.py:74)
      renoise(x0t, std::sqrt(at_next), s1n, z, xn.p, n, img, st);
    }
    CUDA_CHECK(cudaMemcpyAsync(xt, xn.p, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  CUDA_CHECK(cudaMemcpyAsync(xt_state, xt, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
}

// the whole schedule from one full-length noise tape, or from a generated source (then x_T may be null: generated, tag 1)
template <class Step>
static void sample(UNetEngine* unet, long long img, const Step& step, const ddnm_schedule* sc, const float* x_T, const float* y,
                   const NoiseSrc& noise, int B, float* out_x0, float* out_x0_pred, cudaStream_t st, const int* labels = nullptr,
                   const float* grad_buf = nullptr, ddnm_guidance_fn guide = nullptr, void* user = nullptr) {
  DDNM_CHECK(unet && sc && (x_T || !noise.tape) && y && out_x0, "null argument");
  DDNM_CHECK(unet->batch() == B, "engine was built for a different batch size");
  const long long n = (long long)B * img;
  if (!x_T) {
    DDNM_CHECK(img % 4 != 0 || reinterpret_cast<uintptr_t>(out_x0) % 16 == 0, "out_x0 must be 16-byte aligned");
    NoiseSrc xT = noise;
    xT.tag = NZ_XT;
    xT.draw = 0;
    noise_fill(xT, out_x0, B, img, st);
    x_T = out_x0;
  }
  std::unique_ptr<StreamBuf> own;
  float* x0t = out_x0_pred;
  if (!x0t) {
    own.reset(new StreamBuf((size_t)n, st));
    x0t = own->p;
  }
  if (out_x0 != x_T) CUDA_CHECK(cudaMemcpyAsync(out_x0, x_T, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  int have_x0 = 0;
  sample_range(unet, img, step, sc, 0, sc->n_pairs, out_x0, x0t, &have_x0, y, noise, B, st, labels, grad_buf, guide, user);
}

// the SVD operators' step: Operator::step with the DDNM+ scalars of svd_ddnm.py:119-131
struct SvdStep {
  Operator* op;
  const ddnm_schedule* sc;
  const float* y;
  int B;
  cudaStream_t st;
  void operator()(const float* xt, const float* et, long long et_stride, const NoiseSrc& z, StepScalars s, float at_next, float* x0t,
                  float* xn) const {
    s.use_plus = sc->plus ? 1 : 0;
    if (s.use_plus) s.plus = make_plus(s.sqrt_atn, sc->sigma_y, std::sqrt(1.0f - at_next), sc->eta);
    op->step(xt, et, et_stride, z, y, B, s, x0t, xn, st);
  }
};
static long long svd_img(const void* op) {
  DDNM_CHECK(op, "null argument");
  return static_cast<const Operator*>(op)->x_dim();
}

// the simplified loop's step: the runner's lambda_t / gamma_t update (simplified.cu)
struct SimplifiedStep {
  SimpDeg dg;
  const ddnm_schedule* sc;
  const float* y;
  int B;
  cudaStream_t st;
  void operator()(const float* xt, const float* et, long long et_stride, const NoiseSrc& z, const StepScalars& s, float at_next,
                  float* x0t, float* xn) const {
    simplified_step(dg, xt, et, et_stride, z, y, B, s, at_next, sc->sigma_y, x0t, xn, st);
  }
};

}  // namespace ddnm

using namespace ddnm;
extern "C" {
int ddnm_sample(void* unet, void* op, const ddnm_schedule* sched, const float* x_T, const float* y, const float* noise, int B,
                float* out_x0, float* out_x0_pred, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(noise, "null argument");
  const cudaStream_t st = (cudaStream_t)stream;
  sample(static_cast<UNetEngine*>(unet), svd_img(op), SvdStep{static_cast<Operator*>(op), sched, y, B, st}, sched, x_T, y,
         noise_tape(noise), B, out_x0, out_x0_pred, st);
  DDNM_API_END
}
int ddnm_sample_guided(void* unet, void* op, const ddnm_schedule* sched, const float* x_T, const float* y, const float* noise, int B,
                       const int* labels, const float* grad_buf, ddnm_guidance_fn fn, void* user, float* out_x0, float* out_x0_pred,
                       void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(noise, "null argument");
  const cudaStream_t st = (cudaStream_t)stream;
  sample(static_cast<UNetEngine*>(unet), svd_img(op), SvdStep{static_cast<Operator*>(op), sched, y, B, st}, sched, x_T, y,
         noise_tape(noise), B, out_x0, out_x0_pred, st, labels, grad_buf, fn, user);
  DDNM_API_END
}
int ddnm_sample_range(void* unet, void* op, const ddnm_schedule* sched, int k_begin, int k_end, float* xt, float* x0_pred, int* have_x0,
                      const float* y, const float* noise, int B, const int* labels, const float* grad_buf, ddnm_guidance_fn fn,
                      void* user, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(noise, "null argument");
  const cudaStream_t st = (cudaStream_t)stream;
  sample_range(static_cast<UNetEngine*>(unet), svd_img(op), SvdStep{static_cast<Operator*>(op), sched, y, B, st}, sched, k_begin, k_end,
               xt, x0_pred, have_x0, y, noise_tape(noise), B, st, labels, grad_buf, fn, user);
  DDNM_API_END
}
int ddnm_sample_range_seeded(void* unet, void* op, const ddnm_schedule* sched, int k_begin, int k_end, float* xt, float* x0_pred,
                             int* have_x0, const float* y, const ddnm_noise_seed* seed, int B, const int* labels, const float* grad_buf,
                             ddnm_guidance_fn fn, void* user, void* stream) {
  DDNM_API_BEGIN
  const cudaStream_t st = (cudaStream_t)stream;
  sample_range(static_cast<UNetEngine*>(unet), svd_img(op), SvdStep{static_cast<Operator*>(op), sched, y, B, st}, sched, k_begin, k_end,
               xt, x0_pred, have_x0, y, noise_seeded(seed, NZ_LOOP, 0, B), B, st, labels, grad_buf, fn, user);
  DDNM_API_END
}
int ddnm_sample_seeded(void* unet, void* op, const ddnm_schedule* sched, const float* x_T, const float* y, const ddnm_noise_seed* seed,
                       int B, float* out_x0, float* out_x0_pred, void* stream) {
  DDNM_API_BEGIN
  const cudaStream_t st = (cudaStream_t)stream;
  sample(static_cast<UNetEngine*>(unet), svd_img(op), SvdStep{static_cast<Operator*>(op), sched, y, B, st}, sched, x_T, y,
         noise_seeded(seed, NZ_LOOP, 0, B), B, out_x0, out_x0_pred, st);
  DDNM_API_END
}

int ddnm_sample_simplified(void* unet, const ddnm_simple_deg* d, const ddnm_schedule* sched, const float* x_T, const float* y,
                           const float* noise, int B, float* out_x0, float* out_x0_pred, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(x_T && noise, "null argument");
  const cudaStream_t st = (cudaStream_t)stream;
  const SimpDeg dg = make_deg(d);
  sample(static_cast<UNetEngine*>(unet), 3LL * dg.D * dg.D, SimplifiedStep{dg, sched, y, B, st}, sched, x_T, y, noise_tape(noise), B,
         out_x0, out_x0_pred, st);
  DDNM_API_END
}
int ddnm_sample_simplified_range(void* unet, const ddnm_simple_deg* d, const ddnm_schedule* sched, int k_begin, int k_end, float* xt,
                                 float* x0_pred, int* have_x0, const float* y, const float* noise, int B, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(noise, "null argument");
  const cudaStream_t st = (cudaStream_t)stream;
  const SimpDeg dg = make_deg(d);
  sample_range(static_cast<UNetEngine*>(unet), 3LL * dg.D * dg.D, SimplifiedStep{dg, sched, y, B, st}, sched, k_begin, k_end, xt,
               x0_pred, have_x0, y, noise_tape(noise), B, st);
  DDNM_API_END
}
int ddnm_sample_simplified_range_seeded(void* unet, const ddnm_simple_deg* d, const ddnm_schedule* sched, int k_begin, int k_end,
                                        float* xt, float* x0_pred, int* have_x0, const float* y, const ddnm_noise_seed* seed, int B,
                                        void* stream) {
  DDNM_API_BEGIN
  const cudaStream_t st = (cudaStream_t)stream;
  const SimpDeg dg = make_deg(d);
  sample_range(static_cast<UNetEngine*>(unet), 3LL * dg.D * dg.D, SimplifiedStep{dg, sched, y, B, st}, sched, k_begin, k_end, xt,
               x0_pred, have_x0, y, noise_seeded(seed, NZ_LOOP, 0, B), B, st);
  DDNM_API_END
}
}

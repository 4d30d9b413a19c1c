// The DDNM / DDNM+ reverse-diffusion loop (functions/svd_ddnm.py:19-78 and :80-164) enqueued on one stream with
// no host synchronisation: per denoising pair one UNet graph launch + one fused update; travel-back pairs are one
// elementwise kernel.  The reference instead bounces xt / x0_t through host memory every step (:67-68, :45).
#include <cmath>
#include <memory>
#include <vector>

#include "../../include/ddnm_b200.h"
#include "api_util.cuh"
#include "engine.cuh"
#include "operators.cuh"

namespace ddnm {

__global__ void fill_kernel(float* p, int n, float v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
// xt_next = at_next.sqrt() * x0_t + randn * (1 - at_next).sqrt()      (svd_ddnm.py:74)
// GEN: the draw is generated in registers from gen (img = elements per image), z unused
template <bool GEN>
__global__ void travel_back_kernel(const float* __restrict__ x0, const float* __restrict__ z, float sa, float s1, float* __restrict__ xn,
                                   long long n, long long img, NoiseSrc gen) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float zi;
  if (GEN) {
    const long long b = i / img;
    zi = noise_at(gen, (int)b, i - b * img);
  } else {
    zi = z[i];
  }
  xn[i] = __fadd_rn(__fmul_rn(sa, x0[i]), __fmul_rn(zi, s1));
}

// et[b, 0..2] -= sqrt(1 - at) * grad[b]   (svd_ddnm.py:52, :113: et = et - (1 - at).sqrt()[0,0,0,0] * cls_fn(x, t, classes))
__global__ void guide_kernel(float* __restrict__ et, long long et_stride, const float* __restrict__ grad, float s1, long long img,
                             long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long b = i / img, r = i - b * img;
  float* e = et + b * et_stride + r;
  *e = __fsub_rn(*e, __fmul_rn(s1, grad[i]));
}

// Pairs [k0, k1) of the schedule.  State lives in the caller's buffers so that a long schedule can be run as several calls
// with a bounded noise buffer each: xt_state = current iterate (in/out), x0t = last un-projected x0_t (in/out, read by
// travel-back pairs), *have_x0 = whether x0t holds one.  noise = a tape with the draws of exactly these pairs, or a generated
// source (tape == nullptr), whose draw index is the pair's index in the whole schedule.
static void sample_range(UNetEngine* unet, Operator* op, const ddnm_schedule* sc, int k0, int k1, float* xt_state, float* x0t,
                         int* have_x0, const float* y, const NoiseSrc& noise, int B, cudaStream_t st, const int* labels = nullptr,
                         const float* grad_buf = nullptr, ddnm_guidance_fn guide = nullptr, void* user = nullptr) {
  DDNM_CHECK(unet && op && sc && xt_state && x0t && have_x0 && y, "null argument");
  DDNM_CHECK(unet->batch() == B, "engine was built for a different batch size");   // before anything reads B elements
  DDNM_CHECK(0 <= k0 && k0 <= k1 && k1 <= sc->n_pairs, "pair range outside the schedule");
  DDNM_CHECK((labels != nullptr) == unet->class_conditional(), "class labels go with a class-conditional denoiser, and only with one");
  DDNM_CHECK((guide != nullptr) == (grad_buf != nullptr), "guidance callback and gradient buffer go together");
  if (labels) unet->set_labels(labels, st);
  const int R = unet->resolution();
  DDNM_CHECK(op->x_dim() == (long long)unet->in_channels() * R * R, "operator / denoiser image size mismatch");
  DDNM_CHECK(unet->out_ch() == 3 || unet->out_ch() == 6, "denoiser must predict 3 (eps) or 6 (eps, sigma) channels");
  const long long img = op->x_dim();
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
    NoiseSrc z = noise;
    if (z.tape) z.tape += (long long)(k - k0) * n;
    else z.draw = (unsigned)k;
    if (j < i) {
      const float at = sc->abar[i + 1];
      fill_kernel<<<cdiv(B, 128), 128, 0, st>>>(unet->t_in(), B, (float)i);
      unet->forward(xt, unet->t_in(), et, st);
      if (guide) {
        // the caller fills grad_buf (its classifier's autograd gradient) with work enqueued on this stream
        const int rc = guide(user, k, i, (void*)st);
        DDNM_CHECK(rc == 0, "classifier-guidance callback failed");
        guide_kernel<<<(int)cdivll(n, 256), 256, 0, st>>>(et, et_stride, grad_buf, std::sqrt(1.0f - at), img, n);
        CUDA_CHECK(cudaGetLastError());
      }
      StepScalars s{};
      s.sqrt_at = std::sqrt(at);
      s.sqrt_1m_at = std::sqrt(1.0f - at);
      s.sqrt_atn = std::sqrt(at_next);
      const float s1n = std::sqrt(1.0f - at_next);
      s.c1 = s1n * eta;
      s.c2 = s1n * c_eta;
      s.use_plus = sc->plus ? 1 : 0;
      if (s.use_plus) s.plus = Operator::make_plus(s.sqrt_atn, sc->sigma_y, s1n, eta);
      op->step(xt, et, et_stride, z, y, B, s, x0t, xn.p, st);
      *have_x0 = 1;
    } else {
      DDNM_CHECK(*have_x0, "schedule starts with a travel-back step");
      const float sa = std::sqrt(at_next), s1 = std::sqrt(1.0f - at_next);
      if (z.tape) travel_back_kernel<false><<<(int)cdivll(n, 256), 256, 0, st>>>(x0t, z.tape, sa, s1, xn.p, n, img, z);
      else travel_back_kernel<true><<<(int)cdivll(n, 256), 256, 0, st>>>(x0t, nullptr, sa, s1, xn.p, n, img, z);
      CUDA_CHECK(cudaGetLastError());
    }
    CUDA_CHECK(cudaMemcpyAsync(xt, xn.p, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  CUDA_CHECK(cudaMemcpyAsync(xt_state, xt, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
}

// the whole schedule from one full-length noise tape, or from a generated source (then x_T may be null: generated, tag 1)
static void sample(UNetEngine* unet, Operator* op, const ddnm_schedule* sc, const float* x_T, const float* y, const NoiseSrc& noise,
                   int B, float* out_x0, float* out_x0_pred, cudaStream_t st, const int* labels = nullptr,
                   const float* grad_buf = nullptr, ddnm_guidance_fn guide = nullptr, void* user = nullptr) {
  DDNM_CHECK(unet && op && sc && (x_T || !noise.tape) && y && out_x0, "null argument");
  DDNM_CHECK(unet->batch() == B, "engine was built for a different batch size");
  const long long n = (long long)B * op->x_dim();
  if (!x_T) {
    DDNM_CHECK(op->x_dim() % 4 != 0 || reinterpret_cast<uintptr_t>(out_x0) % 16 == 0, "out_x0 must be 16-byte aligned");
    NoiseSrc xT = noise;
    xT.tag = NZ_XT;
    xT.draw = 0;
    noise_fill(xT, out_x0, B, op->x_dim(), st);
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
  sample_range(unet, op, sc, 0, sc->n_pairs, out_x0, x0t, &have_x0, y, noise, B, st, labels, grad_buf, guide, user);
}

}  // namespace ddnm

using namespace ddnm;
extern "C" int ddnm_sample(void* unet, void* op, const ddnm_schedule* sched, const float* x_T, const float* y, const float* noise,
                           int B, float* out_x0, float* out_x0_pred, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(noise, "null argument");
  sample(static_cast<UNetEngine*>(unet), static_cast<Operator*>(op), sched, x_T, y, noise_tape(noise), B, out_x0, out_x0_pred,
         (cudaStream_t)stream);
  DDNM_API_END
}
extern "C" int ddnm_sample_guided(void* unet, void* op, const ddnm_schedule* sched, const float* x_T, const float* y, const float* noise,
                                  int B, const int* labels, const float* grad_buf, ddnm_guidance_fn fn, void* user, float* out_x0,
                                  float* out_x0_pred, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(noise, "null argument");
  sample(static_cast<UNetEngine*>(unet), static_cast<Operator*>(op), sched, x_T, y, noise_tape(noise), B, out_x0, out_x0_pred,
         (cudaStream_t)stream, labels, grad_buf, fn, user);
  DDNM_API_END
}
extern "C" int ddnm_sample_range(void* unet, void* op, const ddnm_schedule* sched, int k_begin, int k_end, float* xt, float* x0_pred,
                                 int* have_x0, const float* y, const float* noise, int B, const int* labels, const float* grad_buf,
                                 ddnm_guidance_fn fn, void* user, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(noise, "null argument");
  sample_range(static_cast<UNetEngine*>(unet), static_cast<Operator*>(op), sched, k_begin, k_end, xt, x0_pred, have_x0, y,
               noise_tape(noise), B, (cudaStream_t)stream, labels, grad_buf, fn, user);
  DDNM_API_END
}
extern "C" int ddnm_sample_range_seeded(void* unet, void* op, const ddnm_schedule* sched, int k_begin, int k_end, float* xt, float* x0_pred,
                                        int* have_x0, const float* y, const ddnm_noise_seed* seed, int B, const int* labels,
                                        const float* grad_buf, ddnm_guidance_fn fn, void* user, void* stream) {
  DDNM_API_BEGIN
  sample_range(static_cast<UNetEngine*>(unet), static_cast<Operator*>(op), sched, k_begin, k_end, xt, x0_pred, have_x0, y,
               noise_seeded(seed, NZ_LOOP, 0, B), B, (cudaStream_t)stream, labels, grad_buf, fn, user);
  DDNM_API_END
}
extern "C" int ddnm_sample_seeded(void* unet, void* op, const ddnm_schedule* sched, const float* x_T, const float* y,
                                  const ddnm_noise_seed* seed, int B, float* out_x0, float* out_x0_pred, void* stream) {
  DDNM_API_BEGIN
  sample(static_cast<UNetEngine*>(unet), static_cast<Operator*>(op), sched, x_T, y, noise_seeded(seed, NZ_LOOP, 0, B), B, out_x0,
         out_x0_pred, (cudaStream_t)stream);
  DDNM_API_END
}

// Degradation operators of functions/svd_operators.py as image-space CUDA kernels (no dense SVD factors are
// materialised for the structured cases; the two separable ones use small fp32 GEMMs).
#pragma once
#include <vector>

#include "../../include/ddnm_b200.h"
#include "common.cuh"
#include "noise.cuh"

namespace ddnm {

enum OpKind : int { OP_SR = 0, OP_COLOR = 1, OP_INPAINT = 2, OP_WH = 3, OP_DEBLUR = 4, OP_SRCONV = 5, OP_DENOISE = 6, OP_DEBLUR2D = 7, OP_CS = 8, OP_GENERAL = 9 };

// scalars of one DDNM+ step (svd_ddnm.py:119-131); all fp32 exactly as the reference's 0-dim tensors / casts
struct PlusScalars {
  float a, sigma_y, sigma_t, eta, c;  // c = (float)((1 - eta^2) ** 0.5)
  float sy2;                          // (float)(sigma_y ** 2)
  int active;                         // a != 0 && sigma_y != 0
};

// scalars of one sampler step (svd_ddnm.py:43-65)
struct StepScalars {
  float sqrt_at, sqrt_1m_at;          // at.sqrt(), (1 - at).sqrt()
  float sqrt_atn;                     // at_next.sqrt()
  float c1, c2;                       // DDNM: (1-at_next).sqrt()*eta, (1-at_next).sqrt()*((1-eta^2)**0.5)
  PlusScalars plus;
  int use_plus;
};

PlusScalars make_plus(float a, float sigma_y, float sigma_t, float eta);

// A device buffer of fp32 that grows on demand.  Growing waits for the device first: work queued earlier may still read the
// old allocation.
class Scratch {
 public:
  Scratch() = default;
  Scratch(const Scratch&) = delete;
  Scratch& operator=(const Scratch&) = delete;
  ~Scratch();
  float* get(size_t elems);

 private:
  float* p_ = nullptr;
  size_t elems_ = 0;
};

// One degradation operator (ddnm_operator_create builds it with make_operator).  The defaults are the generic paths: the
// projection and the step run through A, A_pinv and the Lambdas; operators whose reference class defines no Lambda refuse it.
class Operator {
 public:
  virtual ~Operator();
  Operator(const Operator&) = delete;
  Operator& operator=(const Operator&) = delete;
  long long y_dim() const { return M_; }
  long long x_dim() const { return N_; }
  virtual void A(const float* x, int B, float* y, cudaStream_t s) = 0;
  virtual void A_pinv(const float* y, int B, float* x, cudaStream_t s) = 0;
  // x0 - A^+(A x0 - y)
  virtual void project(const float* x0, const float* y, int B, float* out, cudaStream_t s);
  virtual void lambda(const float* v, int B, const PlusScalars& ps, float* out, cudaStream_t s);
  virtual void lambda_noise(const float* v, const float* eps, int B, const PlusScalars& ps, float* out, cudaStream_t s);
  // One sampler step: x0_t = (xt - et*sqrt(1-at))/sqrt(at); x0_hat by projection (and Lambda); xt_next.
  // et_stride = elements between consecutive images of et (6-channel nets keep channels 0..2).
  // noise: a tape of this pair's draws, or a generated source (noise.cuh): the fused kernels then produce the values in
  // registers, and the operators whose Lambda_noise is a transform fill one pair's worth of scratch first.
  virtual void step(const float* xt, const float* et, long long et_stride, const NoiseSrc& noise, const float* y, int B,
                    const StepScalars& sc, float* x0_t, float* xt_next, cudaStream_t s);

 protected:
  // M, N: per-image lengths of y and x.  name, src, note: the reference class and its source lines, and what the refusal of an
  // undefined Lambda adds to "sigma_y > 0 is unsupported"
  Operator(long long M, long long N, const char* name = "", const char* src = "", const char* note = "")
      : M_(M), N_(N), name_(name), src_(src), note_(note) {}
  // R = A^+(A x0 - y)
  virtual void residual(const float* x0, const float* y, int B, float* R, cudaStream_t s);
  // a device copy of n host elements, freed with the operator
  template <class T>
  T* upload(const T* host, size_t n);

  const long long M_, N_;

 private:
  const char *name_, *src_, *note_;
  std::vector<void*> owned_;
  Scratch ay_;    // A x0 - y in residual(); the step's Lambda_noise output once that is consumed
  Scratch r_;     // the residual of project() and step()
  Scratch et3_;   // step: the epsilon channels the update uses
  Scratch z_;     // step: one pair of generated draws (seeded DDNM+)
};

// validates the descriptor and builds the operator of its kind; throws Error with the reason otherwise
Operator* make_operator(const ddnm_operator_desc& d);

// simplified.cu: the runner's image-space degradations (mask / colour-to-gray / average-pool, diffusion.py:244-290) on
// (B, 3, D, D) images
struct SimpDeg {
  int use_mask, use_gray, scale, D;
  const float* mask;
};
SimpDeg make_deg(const ddnm_simple_deg* d);   // throws on a malformed degradation
void simplified_A(const ddnm_simple_deg* d, const float* x, int B, float* y, cudaStream_t st);
void simplified_Ap(const ddnm_simple_deg* d, const float* y, int B, float* x, cudaStream_t st);
// One pair of the simplified DDNM+ loop: x0_t -> x0t, the Eq. 17 / 19 update -> xt_next, with sc's DDIM terms and lambda_t, gamma_t
// derived from at_next and sigma_y (diffusion.py:355-381).  noise: a tape of this pair's draws or a generated source.
void simplified_step(const SimpDeg& dg, const float* xt, const float* et, long long et_stride, const NoiseSrc& noise, const float* y,
                     int B, const StepScalars& sc, float at_next, float sigma_y, float* x0t, float* xt_next, cudaStream_t st);

}  // namespace ddnm

// Degradation operators of functions/svd_operators.py as image-space CUDA kernels (no dense SVD factors are
// materialised for the structured cases; the two separable ones use small fp32 GEMMs).
#pragma once
#include <vector>

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

class Operator {
 public:
  Operator(int kind, int channels, int img_dim, int ratio, const float* v_small, const float* u_small, const float* singulars,
           const float* singulars_orig, const long long* perm, const long long* mask, const float* v_small2 = nullptr,
           const float* u_small2 = nullptr);
  ~Operator();
  long long y_dim() const { return M_; }
  long long x_dim() const { return N_; }
  int kind() const { return kind_; }
  void A(const float* x, int B, float* y, cudaStream_t s);
  void A_pinv(const float* y, int B, float* x, cudaStream_t s);
  void project(const float* x0, const float* y, int B, float* out, cudaStream_t s);
  void lambda(const float* v, int B, const PlusScalars& ps, float* out, cudaStream_t s);
  void lambda_noise(const float* v, const float* eps, int B, const PlusScalars& ps, float* out, cudaStream_t s);
  // One sampler step: x0_t = (xt - et*sqrt(1-at))/sqrt(at); x0_hat by projection (and Lambda); xt_next.
  // et_stride = elements between consecutive images of et (6-channel nets keep channels 0..2).
  // noise: a tape of this pair's draws, or a generated source (noise.cuh): the fused kernels then produce the values in
  // registers, and the operators whose Lambda_noise is a transform fill one pair's worth of scratch first.
  void step(const float* xt, const float* et, long long et_stride, const NoiseSrc& noise, const float* y, int B, const StepScalars& sc,
            float* x0_t, float* xt_next, cudaStream_t s);
  static PlusScalars make_plus(float a, float sigma_y, float sigma_t, float eta);

 private:
  float* scratch(int idx, size_t elems);
  void fwht(float* buf, int B, cudaStream_t s);
  void sandwich(const float* L, int lr, int lc, const float* X, int B, const float* R, int rr, int rc, float* T, float* out,
                cudaStream_t s);
  void deblur_A(const float* x, int B, float* y, cudaStream_t s);
  void deblur_Apinv(const float* y, int B, float* x, cudaStream_t s);

  void general_A(const float* x, int B, float* y, cudaStream_t s);
  void general_Apinv(const float* y, int B, float* x, cudaStream_t s);
  // SuperResolution with a ratio other than 2 / 4 / 8 (e.g. the paper's 16x): patch rows + the K x K basis as a small GEMM
  bool sr_generic_ = false;
  float* v0_ = nullptr;   // V_small[:, 0]
  void srg_A(const float* x, int B, float* y, cudaStream_t s);
  void srg_Apinv(const float* y, int B, float* x, cudaStream_t s);
  void srg_project(const float* x0, const float* y, int B, float* out, cudaStream_t s);
  void srg_lambda(const float* v, int B, const PlusScalars& ps, float* out, cudaStream_t s);
  void srg_lambda_noise(const float* v, const float* eps, int B, const PlusScalars& ps, float* out, cudaStream_t s);
  void cs_A(const float* x, int B, float* y, cudaStream_t s);
  void cs_Apinv(const float* y, int B, float* x, cudaStream_t s);
  int cs_size_ = 0;
  int kind_, C_, D_, ratio_;
  long long M_ = 0, N_ = 0;   // per-image lengths of y and x
  // device artefacts
  float *V_ = nullptr, *Vt_ = nullptr, *U_ = nullptr, *Ut_ = nullptr;
  float *Vr_ = nullptr, *Vrt_ = nullptr, *Ur_ = nullptr, *Urt_ = nullptr;   // right-hand factors (== left ones unless Deblurring2D)
  float u00_ = 1.f, s0_ = 1.f;
  float *tabD_ = nullptr, *tabDinv_ = nullptr, *tabSorig_ = nullptr;  // deblur: per (c, pos) / per pos tables; srconv: S2, S2inv
  int *rank_ = nullptr;      // inpaint: kept-rank per pixel or -1
  int *perm_ = nullptr, *invperm_ = nullptr;
  std::vector<void*> owned_;
  float* scr_[11] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  size_t scr_elems_[11] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};   // [10]: one pair of generated draws (step, seeded DDNM+)
};

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

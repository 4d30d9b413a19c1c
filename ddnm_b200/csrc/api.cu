// C ABI (include/ddnm_b200.h): denoiser handle + op-level entry points.  Operators and the sampler loop
// are exported from operators.cu / sampler.cu.
#include "../../include/ddnm_b200.h"

#include <cstring>
#include <vector>

#include "api_util.cuh"
#include "engine.cuh"
#include "kernels.cuh"
#include "tc_gemm.cuh"

using namespace ddnm;

namespace ddnm {
thread_local std::string g_last_error;
}

extern "C" {

const char* ddnm_last_error(void) { return g_last_error.c_str(); }
int ddnm_version(void) { return 100; }

int ddnm_unet_simple_create(const ddnm_simple_cfg* c, int batch, void** handle) {
  DDNM_API_BEGIN
  DDNM_CHECK(c && handle, "null argument");
  SimpleCfg cfg;
  cfg.ch = c->ch; cfg.out_ch = c->out_ch; cfg.n_levels = c->n_levels;
  DDNM_CHECK(c->n_levels >= 1 && c->n_levels <= 8 && c->n_attn_res >= 0 && c->n_attn_res <= 4, "bad config");
  for (int i = 0; i < 8; ++i) cfg.ch_mult[i] = c->ch_mult[i];
  cfg.num_res_blocks = c->num_res_blocks;
  cfg.n_attn_res = c->n_attn_res;
  for (int i = 0; i < 4; ++i) cfg.attn_res[i] = c->attn_res[i];
  cfg.in_channels = c->in_channels; cfg.resolution = c->resolution; cfg.groups = c->groups; cfg.eps = c->eps;
  *handle = static_cast<UNetEngine*>(new UNetSimple(cfg, batch));
  DDNM_API_END
}

int ddnm_unet_openai_create(const ddnm_openai_cfg* c, int batch, void** handle) {
  DDNM_API_BEGIN
  DDNM_CHECK(c && handle, "null argument");
  DDNM_CHECK(c->n_levels >= 1 && c->n_levels <= 8 && c->n_attn_ds >= 0 && c->n_attn_ds <= 4, "bad config");
  OpenAICfg cfg;
  cfg.image_size = c->image_size; cfg.model_channels = c->model_channels; cfg.num_res_blocks = c->num_res_blocks;
  cfg.n_levels = c->n_levels;
  for (int i = 0; i < 8; ++i) cfg.channel_mult[i] = c->channel_mult[i];
  cfg.n_attn_ds = c->n_attn_ds;
  for (int i = 0; i < 4; ++i) cfg.attn_ds[i] = c->attn_ds[i];
  cfg.num_head_channels = c->num_head_channels; cfg.out_channels = c->out_channels; cfg.in_channels = c->in_channels;
  cfg.groups = c->groups; cfg.eps = c->eps; cfg.num_classes = c->num_classes; cfg.low_res = c->low_res;
  cfg.num_heads = c->num_heads; cfg.num_heads_upsample = c->num_heads_upsample; cfg.new_attention_order = c->new_attention_order;
  DDNM_CHECK(c->num_classes >= 0, "bad num_classes");
  DDNM_CHECK(c->new_attention_order == 0 || c->new_attention_order == 1, "new_attention_order must be 0 or 1");
  DDNM_CHECK(c->num_head_channels > 0 || c->num_heads >= 1, "num_head_channels <= 0 needs num_heads >= 1");
  *handle = static_cast<UNetEngine*>(new UNetOpenAI(cfg, batch));
  DDNM_API_END
}

int ddnm_classifier_create(const ddnm_classifier_cfg* c, int batch, void** handle) {
  DDNM_API_BEGIN
  DDNM_CHECK(c && handle, "null argument");
  DDNM_CHECK(c->n_levels >= 1 && c->n_levels <= 8 && c->n_attn_ds >= 0 && c->n_attn_ds <= 4, "bad config");
  EncoderCfg cfg;
  cfg.image_size = c->image_size; cfg.model_channels = c->model_channels; cfg.num_res_blocks = c->num_res_blocks;
  cfg.n_levels = c->n_levels;
  for (int i = 0; i < 8; ++i) cfg.channel_mult[i] = c->channel_mult[i];
  cfg.n_attn_ds = c->n_attn_ds;
  for (int i = 0; i < 4; ++i) cfg.attn_ds[i] = c->attn_ds[i];
  cfg.num_head_channels = c->num_head_channels; cfg.out_channels = c->out_channels; cfg.in_channels = c->in_channels;
  cfg.groups = c->groups; cfg.eps = c->eps; cfg.pool = c->pool;
  *handle = static_cast<UNetEngine*>(new UNetEncoder(cfg, batch));
  DDNM_API_END
}

static UNetEncoder* as_classifier(void* h) {
  UNetEncoder* e = dynamic_cast<UNetEncoder*>(static_cast<UNetEngine*>(h));
  DDNM_CHECK(e != nullptr, "handle is not a classifier");
  return e;
}

int ddnm_classifier_forward(void* h, const float* x, const float* t, float* logits, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(x && t && logits, "null argument");
  as_classifier(h)->forward(x, t, logits, (cudaStream_t)stream);
  DDNM_API_END
}

int ddnm_classifier_grad(void* h, const float* x, const float* t, const int* labels, float scale, float* grad_out, float* logits_out,
                         void* stream) {
  DDNM_API_BEGIN
  as_classifier(h)->grad(x, t, labels, scale, grad_out, logits_out, (cudaStream_t)stream);
  DDNM_API_END
}

int ddnm_classifier_guidance_fn(void* user, int, int t, void* stream) {
  DDNM_API_BEGIN
  ddnm_classifier_guidance* g = static_cast<ddnm_classifier_guidance*>(user);
  DDNM_CHECK(g && g->classifier && g->x && g->labels && g->grad_buf, "incomplete guidance context");
  UNetEncoder* e = as_classifier(g->classifier);
  DDNM_CHECK(g->batch == e->batch(), "classifier was built for batch " + std::to_string(e->batch()) + ", the guided loop runs " +
                                         std::to_string(g->batch));
  cudaStream_t st = (cudaStream_t)stream;
  if (!g->labels_checked) {   // the loop's labels are fixed: one host read for the whole loop
    e->check_labels(g->labels, st);
    g->labels_checked = 1;
  }
  e->fill_t((float)t, st);
  e->grad(g->x, e->t_in(), g->labels, g->scale, g->grad_buf, nullptr, st, true);
  DDNM_API_END
}

int ddnm_unet_set_param(void* h, const char* name, const float* data, long long numel) {
  DDNM_API_BEGIN
  static_cast<UNetEngine*>(h)->set_param(name, data, numel);
  DDNM_API_END
}
int ddnm_unet_finalize(void* h) {
  DDNM_API_BEGIN
  static_cast<UNetEngine*>(h)->finalize();
  DDNM_API_END
}
int ddnm_unet_forward(void* h, const float* x, const float* t, float* out, void* stream) {
  DDNM_API_BEGIN
  static_cast<UNetEngine*>(h)->forward(x, t, out, (cudaStream_t)stream);
  DDNM_API_END
}
int ddnm_unet_forward_cond(void* h, const float* x, const float* t, const int* labels, float* out, void* stream) {
  DDNM_API_BEGIN
  UNetEngine* u = static_cast<UNetEngine*>(h);
  u->set_labels(labels, (cudaStream_t)stream);
  u->forward(x, t, out, (cudaStream_t)stream);
  DDNM_API_END
}
int ddnm_unet_set_low_res(void* h, const float* low_res, void* stream) {
  DDNM_API_BEGIN
  static_cast<UNetEngine*>(h)->set_low_res(low_res, (cudaStream_t)stream);
  DDNM_API_END
}
int ddnm_unet_set_precision(void* h, int fp16_terms) {
  DDNM_API_BEGIN
  static_cast<UNetEngine*>(h)->set_terms(fp16_terms);
  DDNM_API_END
}
int ddnm_unet_set_batch_invariant(void* h, int on) {
  DDNM_API_BEGIN
  static_cast<UNetEngine*>(h)->set_batch_invariant(on != 0);
  DDNM_API_END
}
int ddnm_unet_set_graph(void* h, int on) {
  DDNM_API_BEGIN
  static_cast<UNetEngine*>(h)->set_use_graph(on != 0);
  DDNM_API_END
}
int ddnm_unet_read_tap(void* h, const char* name, float* dst, long long cap, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(static_cast<UNetEngine*>(h)->read_tap(name, dst, cap, (cudaStream_t)stream), std::string("unknown tap ") + name);
  DDNM_API_END
}
int ddnm_unet_info(void* h, long long* ws, int* launches, double* flops) {
  DDNM_API_BEGIN
  UNetEngine* u = static_cast<UNetEngine*>(h);
  if (ws) *ws = (long long)u->workspace_bytes();
  if (launches) *launches = u->num_launches();
  if (flops) *flops = u->flops_per_forward();
  DDNM_API_END
}
int ddnm_unet_profile(void* h, const float* x, const float* t, float* out, void* stream, char* json, long long cap) {
  DDNM_API_BEGIN
  std::string s = static_cast<UNetEngine*>(h)->profile(x, t, out, (cudaStream_t)stream);
  DDNM_CHECK((long long)s.size() + 1 <= cap, "json buffer too small");
  std::memcpy(json, s.c_str(), s.size() + 1);
  DDNM_API_END
}
int ddnm_unet_destroy(void* h) {
  DDNM_API_BEGIN
  delete static_cast<UNetEngine*>(h);
  DDNM_API_END
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------
// op-level entry points
// ------------------------------------------------------------------------------------------------------------
namespace {
struct Tmp {
  std::vector<void*> ptrs;
  ~Tmp() {
    for (void* p : ptrs) cudaFree(p);
  }
  template <class T>
  T* get(size_t n) {
    void* p = nullptr;
    CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)));
    ptrs.push_back(p);
    return (T*)p;
  }
};
int sm_count() {
  int dev = 0, n = 0;
  CUDA_CHECK(cudaGetDevice(&dev));
  CUDA_CHECK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  return n;
}
View mkview(float* p, int N, int H, int W, int C) {
  View v;
  v.p = p; v.N = N; v.H = H; v.W = W; v.C = C; v.ld = C;
  return v;
}
// the SM count an engine built now would plan its launches for (ddnm_tc_debug_sm_count)
int planned_sm_count() {
  int dev = 0;
  CUDA_CHECK(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  CUDA_CHECK(cudaGetDeviceProperties(&prop, dev));
  return engine_sm_count(prop);
}
// the fp16 product terms of the launches built while it lives (the launch builders read the global setting)
struct TermsScope {
  int prev;
  explicit TermsScope(int t) : prev(tc_get_terms()) { tc_set_terms(t); }
  ~TermsScope() { tc_set_terms(prev); }
};
}  // namespace

extern "C" {

int ddnm_conv_tc(const float* x, int N, int H, int W, int Cin, const float* w, const float* bias, int Cout, int mode, int up2,
                 const float* side_x, int CinSide, const float* side_w, const float* residual, float* out, void* stream) {
  DDNM_API_BEGIN
  cudaStream_t s = (cudaStream_t)stream;
  Tmp tmp;
  const int taps = mode == TAPS_1X1 ? 1 : 9;
  int oH = H, oW = W;
  int smode = SPLIT_SAME;
  if (mode == TAPS_3X3_S2) { oH = H / 2; oW = W / 2; smode = SPLIT_S2D; DDNM_CHECK(!up2, "stride 2 with upsample"); }
  if (up2) { oH = 2 * H; oW = 2 * W; DDNM_CHECK(mode == TAPS_3X3 && !side_x && !residual, "upsample path: plain 3x3 only"); }
  const size_t pe = (size_t)N * H * W * Cin;
  SplitView A;
  A.hi = tmp.get<__half>(pe); A.lo = tmp.get<__half>(pe); A.C = Cin;
  if (smode == SPLIT_S2D) { A.N = 4 * N; A.H = oH; A.W = oW; } else { A.N = N; A.H = H; A.W = W; }
  View xv = mkview(const_cast<float*>(x), N, H, W, Cin);
  gn_apply_split(xv, 1, false, nullptr, nullptr, 0.f, false, smode, A.hi, A.lo, s);
  View ov = mkview(out, N, oH, oW, Cout);
  if (up2) {
    // conv3x3(nearest_upsample_x2(x)): four parity-phase 2x2 convolutions on the low-res split (the engine's path)
    const size_t per_phase = (size_t)Cout * 4 * Cin;
    __half* wh = tmp.get<__half>(4 * per_phase);
    __half* wl = tmp.get<__half>(4 * per_phase);
    presum_up2_weights(w, Cout, Cin, wh, wl, s);
    for (int ph = 0; ph < 4; ++ph) {
      TcLaunch L = tc_make_up2_launch(A, wh + ph * per_phase, wl + ph * per_phase, Cout, ov, bias, 0, ph >> 1, ph & 1, sm_count());
      tc_run(L, s);
    }
    CUDA_CHECK(cudaStreamSynchronize(s));
    return 0;
  }
  SplitView S;
  if (side_x) {
    const size_t se = (size_t)N * oH * oW * CinSide;
    S.hi = tmp.get<__half>(se); S.lo = tmp.get<__half>(se); S.N = N; S.H = oH; S.W = oW; S.C = CinSide;
    gn_apply_split(mkview(const_cast<float*>(side_x), N, oH, oW, CinSide), 1, false, nullptr, nullptr, 0.f, false, SPLIT_SAME,
                   S.hi, S.lo, s);
  }
  const int ktot = taps * Cin + (side_x ? CinSide : 0);
  __half* wh = tmp.get<__half>((size_t)Cout * ktot);
  __half* wl = tmp.get<__half>((size_t)Cout * ktot);
  split_conv_weight(w, Cout, Cin, taps, wh, wl, ktot, 0, s);
  if (side_x) split_conv_weight(side_w, Cout, CinSide, 1, wh, wl, ktot, taps * Cin, s);
  TcLaunch L = tc_make_launch(A, mode, side_x ? &S : nullptr, wh, wl, 1, Cout, ov, bias, 0, residual, Cout, 1.0f, sm_count());
  tc_run(L, s);
  CUDA_CHECK(cudaStreamSynchronize(s));
  DDNM_API_END
}

int ddnm_conv_tc_ex(const float* x, int N, int H, int W, int Cin, const float* w, const float* chanadd, int ca_ld, int Cout, int mode,
                    int up2, const float* side_x, int CinSide, const float* side_w, const float* residual, int res_mode, float* out,
                    int out_ld, int split_k, int invariant, int terms, double* stats_out, int* split_used, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(x && w && out, "null argument");
  DDNM_CHECK(mode >= TAPS_3X3 && mode <= TAPS_3X3_S2 && res_mode >= 0 && res_mode <= 2 && out_ld >= Cout && ca_ld >= 0,
             "bad mode, res_mode, out_ld or ca_ld");
  DDNM_CHECK(split_k == -1 || split_k == 1 || split_k == 2 || split_k == 4, "split_k must be -1 (the engine's rule), 1, 2 or 4");
  cudaStream_t s = (cudaStream_t)stream;
  Tmp tmp;
  const TermsScope terms_scope(terms);
  const int sms = planned_sm_count();
  const int taps = mode == TAPS_1X1 ? 1 : 9;
  int oH = H, oW = W;
  int smode = SPLIT_SAME;
  if (mode == TAPS_3X3_S2) { oH = H / 2; oW = W / 2; smode = SPLIT_S2D; DDNM_CHECK(!up2, "stride 2 with upsample"); }
  if (up2) {
    oH = 2 * H; oW = 2 * W;
    // as UNetEngine::emit_up2_conv: a plain 3x3 on the upsampled map, never split
    DDNM_CHECK(mode == TAPS_3X3 && !side_x && !residual && split_k <= 1, "upsample path: plain unsplit 3x3 only");
  }
  const size_t pe = (size_t)N * H * W * Cin;
  SplitView A;
  A.hi = tmp.get<__half>(pe); A.lo = tmp.get<__half>(pe); A.C = Cin;
  if (smode == SPLIT_S2D) { A.N = 4 * N; A.H = oH; A.W = oW; } else { A.N = N; A.H = H; A.W = W; }
  gn_apply_split(mkview(const_cast<float*>(x), N, H, W, Cin), 1, false, nullptr, nullptr, 0.f, false, smode, A.hi, A.lo, s);
  View ov = mkview(out, N, oH, oW, Cout);
  ov.ld = out_ld;
  if (stats_out) {
    ov.st = tmp.get<StatAcc>((size_t)N * Cout * 2);
    ov.st_ld = Cout;
    CUDA_CHECK(cudaMemsetAsync(ov.st, 0, (size_t)N * Cout * 2 * sizeof(StatAcc), s));
  }
  int S = 1;
  if (up2) {
    // the four parity phases add into one stats buffer, as in UNetEngine::emit_up2_conv
    const size_t per_phase = (size_t)Cout * 4 * Cin;
    __half* wh = tmp.get<__half>(4 * per_phase);
    __half* wl = tmp.get<__half>(4 * per_phase);
    presum_up2_weights(w, Cout, Cin, wh, wl, s);
    for (int ph = 0; ph < 4; ++ph)
      tc_run(tc_make_up2_launch(A, wh + ph * per_phase, wl + ph * per_phase, Cout, ov, chanadd, ca_ld, ph >> 1, ph & 1, sms, invariant != 0), s);
  } else {
    SplitView Sv;
    if (side_x) {
      const size_t se = (size_t)N * oH * oW * CinSide;
      Sv.hi = tmp.get<__half>(se); Sv.lo = tmp.get<__half>(se); Sv.N = N; Sv.H = oH; Sv.W = oW; Sv.C = CinSide;
      gn_apply_split(mkview(const_cast<float*>(side_x), N, oH, oW, CinSide), 1, false, nullptr, nullptr, 0.f, false, SPLIT_SAME,
                     Sv.hi, Sv.lo, s);
    }
    const int ktot = taps * Cin + (side_x ? CinSide : 0);
    __half* wh = tmp.get<__half>((size_t)Cout * ktot);
    __half* wl = tmp.get<__half>((size_t)Cout * ktot);
    split_conv_weight(w, Cout, Cin, taps, wh, wl, ktot, 0, s);
    if (side_x) split_conv_weight(side_w, Cout, CinSide, 1, wh, wl, ktot, taps * Cin, s);
    TcConvPlan P = tc_plan_conv(A, mode, side_x ? &Sv : nullptr, wh, wl, Cout, ov, chanadd, ca_ld, residual, Cout, res_mode, sms,
                                invariant != 0, split_k);
    if (P.S > 1) tc_set_partials(P, tmp.get<float>((size_t)P.part_elems));
    tc_run_conv(P, s);
    S = P.S;
  }
  CUDA_CHECK(cudaStreamSynchronize(s));
  if (split_used) *split_used = S;
  if (stats_out) {
    std::vector<StatAcc> h((size_t)N * Cout * 2);
    CUDA_CHECK(cudaMemcpy(h.data(), ov.st, h.size() * sizeof(StatAcc), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < h.size(); ++i) stats_out[i] = stat_value(h[i]);
  }
  DDNM_API_END
}

int ddnm_gemm_tc(const float* a, long long a_numel, long long a_off, long long a_s_row, long long a_s_head, long long a_s_img,
                 const float* b, long long b_numel, long long b_off, long long b_s_row, long long b_s_head, long long b_s_img, int M,
                 int N, int K, int heads, int images, float alpha, float* out, long long out_sn, long long out_sy, long long out_sx,
                 int invariant, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(a && b && out && M > 0 && N > 0 && K > 0 && heads > 0 && images > 0, "null or empty argument");
  cudaStream_t s = (cudaStream_t)stream;
  Tmp tmp;
  auto operand = [&](const float* src, long long numel, long long off, long long rows, long long s_row, long long s_head,
                     long long s_img) {
    DDNM_CHECK(numel % 8 == 0 && off >= 0 && s_row > 0 && s_head > 0 && s_img > 0, "GEMM operand: bad size or strides");
    DDNM_CHECK(off + (K - 1) + (rows - 1) * s_row + (heads - 1) * s_head + (images - 1) * s_img < numel,
               "GEMM operand reaches past its buffer");
    __half* hi = tmp.get<__half>((size_t)numel);
    __half* lo = tmp.get<__half>((size_t)numel);
    // the attention core's raw split (elementwise), the buffer viewed as rows of 8 channels
    gn_apply_split(mkview(const_cast<float*>(src), 1, 1, (int)(numel / 8), 8), 1, false, nullptr, nullptr, 0.f, false, SPLIT_SAME,
                   hi, lo, s);
    return GemmOperand{hi + off, lo + off, s_row, s_head, s_img};
  };
  const GemmOperand A = operand(a, a_numel, a_off, M, a_s_row, a_s_head, a_s_img);
  const GemmOperand B = operand(b, b_numel, b_off, N, b_s_row, b_s_head, b_s_img);
  tc_run(tc_make_gemm_launch(A, B, M, N, K, heads, images, out, out_sn, out_sy, out_sx, alpha, planned_sm_count(), invariant != 0), s);
  CUDA_CHECK(cudaStreamSynchronize(s));
  DDNM_API_END
}

// the super-resolution stem on its own: out (NHWC [N,H,W,Cout]) = conv3x3(cat([x, bilinear(low_res)])) + bias; low_res == NULL:
// x is the already concatenated [N,2C,H,W] (the composed form).  iters > 0: also time `iters` launches.
int ddnm_conv_stem_sr(const float* x, const float* low_res, int N, int C, int H, int W, int h, int w, const float* weight,
                      const float* bias, int Cout, float* out, int iters, float* ms_per_iter, void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(x && weight && bias && out, "null argument");
  cudaStream_t s = (cudaStream_t)stream;
  View ov = mkview(out, N, H, W, Cout);
  conv3x3_stem_sr(x, low_res, C, h, w, weight, bias, ov, s);
  if (iters > 0 && ms_per_iter) {
    cudaEvent_t e0, e1;
    CUDA_CHECK(cudaEventCreate(&e0));
    CUDA_CHECK(cudaEventCreate(&e1));
    CUDA_CHECK(cudaEventRecord(e0, s));
    for (int i = 0; i < iters; ++i) conv3x3_stem_sr(x, low_res, C, h, w, weight, bias, ov, s);
    CUDA_CHECK(cudaEventRecord(e1, s));
    CUDA_CHECK(cudaEventSynchronize(e1));
    float ms = 0;
    CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    *ms_per_iter = ms / iters;
  }
  CUDA_CHECK(cudaStreamSynchronize(s));
  DDNM_API_END
}

int ddnm_conv_direct(const float* x, int N, int H, int W, int Cin, const float* w, const float* bias, int Cout, int mode, int up2,
                     float* out, void* stream) {
  DDNM_API_BEGIN
  int oH = H, oW = W;
  if (mode == TAPS_3X3_S2) { oH = H / 2; oW = W / 2; }
  if (up2) { oH = 2 * H; oW = 2 * W; }
  conv_direct_ref(mkview(const_cast<float*>(x), N, H, W, Cin), w, bias, mode, up2 != 0, mkview(out, N, oH, oW, Cout),
                  (cudaStream_t)stream);
  DDNM_API_END
}

namespace {
__device__ __forceinline__ float bench_hash(unsigned long long i, unsigned seed) {   // uniform in [-1, 1)
  unsigned x = (unsigned)(i * 2654435761ull) ^ seed;
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return (float)(int)x * (1.0f / 2147483648.0f);
}
__global__ void bench_fill_f32(float* p, long long n, unsigned seed) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = bench_hash(i, seed);
}
__global__ void bench_fill_split(__half* hi, __half* lo, long long n, unsigned seed, float scale) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) split_f16(bench_hash(i, seed) * scale, hi[i], lo[i]);
}
}  // namespace

// iters > 0: all-zero operands (no data-dependent switching power: the kernel's clock-for-clock pace);
// iters < 0: |iters| iterations on pseudo-random operands (what the kernel sustains under the board's power cap)
int ddnm_conv_tc_bench(int N, int H, int W, int Cin, int Cout, int mode, int iters, float* ms_per_iter, double* flops) {
  DDNM_API_BEGIN
  const bool random = iters < 0;
  if (random) iters = -iters;
  // mode bits [4,8): epilogue features as the network uses them — 16: GroupNorm sums of the output, 32: residual add,
  // 64: per-(image, channel) add (bias + temb row), 128: the layer is one parity phase of an upsample convolution (2x2 taps on the
  // H x W source, strided stores into a 2H x 2W map)
  const int feat = mode >> 4;
  mode &= 15;
  const bool up2 = (feat & 8) != 0;
  Tmp tmp;
  const int taps = up2 ? 4 : (mode == TAPS_1X1 ? 1 : 9);
  const size_t pe = (size_t)N * H * W * Cin;
  SplitView A;
  A.hi = tmp.get<__half>(pe); A.lo = tmp.get<__half>(pe); A.N = N; A.H = H; A.W = W; A.C = Cin;
  float* xf = tmp.get<float>(pe);
  CUDA_CHECK(cudaMemset(xf, 0, pe * 4));
  if (random) bench_fill_f32<<<(unsigned)cdivll((long long)pe, 256), 256>>>(xf, (long long)pe, 0x1234u);
  gn_apply_split(mkview(xf, N, H, W, Cin), 1, false, nullptr, nullptr, 0.f, false, SPLIT_SAME, A.hi, A.lo, 0);
  const int ktot = taps * Cin;
  __half* wh = tmp.get<__half>((size_t)Cout * ktot);
  __half* wl = tmp.get<__half>((size_t)Cout * ktot);
  CUDA_CHECK(cudaMemset(wh, 0, (size_t)Cout * ktot * 2));
  CUDA_CHECK(cudaMemset(wl, 0, (size_t)Cout * ktot * 2));
  if (random) {
    const long long wn = (long long)Cout * ktot;
    bench_fill_split<<<(unsigned)cdivll(wn, 256), 256>>>(wh, wl, wn, 0x9876u, 1.0f / sqrtf((float)ktot));
  }
  const int oH = up2 ? 2 * H : H, oW = up2 ? 2 * W : W;
  const size_t oe = (size_t)N * oH * oW * Cout;
  float* o = tmp.get<float>(oe);
  View ov = mkview(o, N, oH, oW, Cout);
  if (feat & 1) {
    ov.st = tmp.get<StatAcc>((size_t)N * Cout * 2);
    ov.st_ld = Cout;
    CUDA_CHECK(cudaMemset(ov.st, 0, (size_t)N * Cout * 2 * sizeof(StatAcc)));
  }
  float* res = nullptr;
  if (feat & 2) {
    res = tmp.get<float>(oe);
    CUDA_CHECK(cudaMemset(res, 0, oe * 4));
    if (random) bench_fill_f32<<<(unsigned)cdivll((long long)oe, 256), 256>>>(res, (long long)oe, 0x777u);
  }
  float* ca = nullptr;
  if (feat & 4) {
    ca = tmp.get<float>((size_t)N * Cout);
    CUDA_CHECK(cudaMemset(ca, 0, (size_t)N * Cout * 4));
  }
  TcLaunch L = up2 ? tc_make_up2_launch(A, wh, wl, Cout, ov, ca, Cout, 0, 0, sm_count())
                   : tc_make_launch(A, mode, nullptr, wh, wl, 1, Cout, ov, ca, Cout, res, Cout, 1.0f, sm_count());
  for (int i = 0; i < 3; ++i) tc_run(L, 0);
  cudaEvent_t e0, e1;
  CUDA_CHECK(cudaEventCreate(&e0));
  CUDA_CHECK(cudaEventCreate(&e1));
  CUDA_CHECK(cudaEventRecord(e0, 0));
  for (int i = 0; i < iters; ++i) tc_run(L, 0);
  CUDA_CHECK(cudaEventRecord(e1, 0));
  CUDA_CHECK(cudaEventSynchronize(e1));
  float ms = 0;
  CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  *ms_per_iter = ms / iters;
  *flops = L.flops;
  DDNM_API_END
}

// Probe (tests/diag): GroupNorm+SiLU+split -> 3x3 convolution over N images, run in chunks of `chunk` images that SHARE one
// chunk-sized scratch for the fp16 planes (so the planes can stay in L2 between the pass that writes them and the convolution that
// reads them, and are overwritten in place by the next chunk).  chunk == N is the engine's current order.  ms per full pass.
int ddnm_gnconv_chunk_bench(int N, int chunk, int H, int W, int Cin, int Cout, int iters, float* ms_per_pass) {
  DDNM_API_BEGIN
  DDNM_CHECK(chunk >= 1 && N % chunk == 0, "chunk must divide N");
  Tmp tmp;
  const size_t pe = (size_t)N * H * W * Cin, ce = (size_t)chunk * H * W * Cin, oe = (size_t)N * H * W * Cout;
  float* x = tmp.get<float>(pe);
  bench_fill_f32<<<(unsigned)cdivll((long long)pe, 256), 256>>>(x, (long long)pe, 0x4321u);
  StatAcc* st = tmp.get<StatAcc>((size_t)N * Cin * 2);
  CUDA_CHECK(cudaMemset(st, 0, (size_t)N * Cin * 2 * sizeof(StatAcc)));
  View xv = mkview(x, N, H, W, Cin);
  xv.st = st; xv.st_ld = Cin;
  gn_stats(xv, 0);
  float* gamma = tmp.get<float>(Cin);
  float* beta = tmp.get<float>(Cin);
  bench_fill_f32<<<cdiv(Cin, 256), 256>>>(gamma, Cin, 0x11u);
  bench_fill_f32<<<cdiv(Cin, 256), 256>>>(beta, Cin, 0x22u);
  SplitView A;
  A.hi = tmp.get<__half>(ce); A.lo = tmp.get<__half>(ce); A.N = chunk; A.H = H; A.W = W; A.C = Cin;
  const int ktot = 9 * Cin;
  __half* wh = tmp.get<__half>((size_t)Cout * ktot);
  __half* wl = tmp.get<__half>((size_t)Cout * ktot);
  bench_fill_split<<<(unsigned)cdivll((long long)Cout * ktot, 256), 256>>>(wh, wl, (long long)Cout * ktot, 0x9876u, 1.0f / sqrtf((float)ktot));
  float* o = tmp.get<float>(oe);
  StatAcc* ost = tmp.get<StatAcc>((size_t)N * Cout * 2);
  CUDA_CHECK(cudaMemset(ost, 0, (size_t)N * Cout * 2 * sizeof(StatAcc)));
  float* ca = tmp.get<float>((size_t)N * Cout);
  CUDA_CHECK(cudaMemset(ca, 0, (size_t)N * Cout * 4));
  const int nch = N / chunk;
  std::vector<View> xs;
  std::vector<TcLaunch> Ls;
  for (int c = 0; c < nch; ++c) {
    View xc = xv;
    xc.p = x + (size_t)c * chunk * H * W * Cin; xc.N = chunk; xc.st = st + (size_t)c * chunk * Cin * 2;
    View oc = mkview(o + (size_t)c * chunk * H * W * Cout, chunk, H, W, Cout);
    oc.st = ost + (size_t)c * chunk * Cout * 2; oc.st_ld = Cout;
    xs.push_back(xc);
    Ls.push_back(tc_make_launch(A, TAPS_3X3, nullptr, wh, wl, 1, Cout, oc, ca + (size_t)c * chunk * Cout, Cout, nullptr, 0, 1.0f, sm_count()));
  }
  auto pass = [&]() {
    for (int c = 0; c < nch; ++c) {
      gn_apply_split(xs[c], 32, true, gamma, beta, 1e-6f, true, SPLIT_SAME, A.hi, A.lo, 0);
      tc_run(Ls[c], 0);
    }
  };
  for (int i = 0; i < 2; ++i) pass();
  cudaEvent_t e0, e1;
  CUDA_CHECK(cudaEventCreate(&e0));
  CUDA_CHECK(cudaEventCreate(&e1));
  CUDA_CHECK(cudaEventRecord(e0, 0));
  for (int i = 0; i < iters; ++i) pass();
  CUDA_CHECK(cudaEventRecord(e1, 0));
  CUDA_CHECK(cudaEventSynchronize(e1));
  float ms = 0;
  CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  *ms_per_pass = ms / iters;
  DDNM_API_END
}

int ddnm_groupnorm(const float* x, int N, int H, int W, int C, int groups, const float* gamma, const float* beta, float eps,
                   int silu, float* out, void* stream) {
  DDNM_API_BEGIN
  cudaStream_t s = (cudaStream_t)stream;
  Tmp tmp;
  StatAcc* st = tmp.get<StatAcc>((size_t)N * C * 2);
  CUDA_CHECK(cudaMemsetAsync(st, 0, (size_t)N * C * 2 * sizeof(StatAcc), s));
  View xv = mkview(const_cast<float*>(x), N, H, W, C);
  xv.st = st;
  xv.st_ld = C;
  gn_stats(xv, s);
  gn_apply_f32(xv, groups, gamma, beta, eps, silu != 0, out, s);
  CUDA_CHECK(cudaStreamSynchronize(s));
  DDNM_API_END
}

int ddnm_tc_debug_deal(int mode) {
  DDNM_API_BEGIN
  tc_debug_deal(mode);
  DDNM_API_END
}
int ddnm_tc_debug_dual_mode(int mode) {
  DDNM_API_BEGIN
  tc_debug_dual_mode(mode);
  DDNM_API_END
}
int ddnm_tc_debug_halo(int on) {
  DDNM_API_BEGIN
  tc_debug_halo(on);
  DDNM_API_END
}
int ddnm_tc_debug_pingpong(int on) {
  DDNM_API_BEGIN
  tc_debug_pingpong(on);
  DDNM_API_END
}
int ddnm_tc_debug_pp_pair(int on) {
  DDNM_API_BEGIN
  tc_debug_pp_pair(on);
  DDNM_API_END
}
int ddnm_tc_debug_force_bn(int bn) {
  DDNM_API_BEGIN
  tc_debug_force_bn(bn);
  DDNM_API_END
}
int ddnm_tc_debug_sm_count(int n) {
  DDNM_API_BEGIN
  engine_debug_sm_count(n);
  DDNM_API_END
}
}  // extern "C"

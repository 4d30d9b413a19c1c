// UNetEngine: what the two denoiser programs share — parameters, arena, scratch, op emitters, CUDA-graph replay.
//
// Data layout in HBM: activations fp32 NHWC; every skip tensor is born inside the channel slice of the concat
// buffer its up-path consumer will read (torch.cat at models.py:331 / unet.py:661 costs nothing); the tensor-core
// convolutions read fp16 (hi, lo) planes produced by the fused GroupNorm+SiLU+split pass.
#include "engine.cuh"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <sstream>

#include "kernels.cuh"

namespace ddnm {

Arena::~Arena() {
  for (void* b : blocks_) cudaFree(b);
}
void* Arena::alloc(size_t bytes) {
  bytes = (bytes + 1023) / 1024 * 1024;
  if (bytes == 0) bytes = 1024;
  void* p = nullptr;
  CUDA_CHECK(cudaMalloc(&p, bytes));
  blocks_.push_back(p);
  total_ += bytes;
  return p;
}

UNetEngine::UNetEngine(int batch, int in_channels, int out_ch, int resolution, int groups, float eps)
    : B_(batch), in_ch_(in_channels), out_ch_(out_ch), R_(resolution), groups_(groups), eps_(eps) {
  DDNM_CHECK(batch >= 1, "batch must be positive");
  int dev = 0;
  CUDA_CHECK(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  CUDA_CHECK(cudaGetDeviceProperties(&prop, dev));
  DDNM_CHECK(prop.major == 9 && prop.minor == 0, "ddnm_b200 kernels are built for sm_90a (H100) only");
  num_sms_ = prop.multiProcessorCount;
}

UNetEngine::~UNetEngine() {
  if (graph_exec_) cudaGraphExecDestroy(graph_exec_);
  if (graph_) cudaGraphDestroy(graph_);
  for (auto& kv : params_) cudaFree(kv.second.p);
}

void UNetEngine::set_param(const std::string& name, const float* data, long long numel) {
  DDNM_CHECK(!finalized_, "set_param after finalize");
  DDNM_CHECK(numel > 0 && data != nullptr, "empty parameter " + name);
  float* d = nullptr;
  CUDA_CHECK(cudaMalloc(&d, (size_t)numel * sizeof(float)));
  CUDA_CHECK(cudaMemcpy(d, data, (size_t)numel * sizeof(float), cudaMemcpyDefault));
  auto it = params_.find(name);
  if (it != params_.end()) cudaFree(it->second.p);
  params_[name] = Param{d, numel};
}

const float* UNetEngine::P(const std::string& name, long long expect) const {
  auto it = params_.find(name);
  DDNM_CHECK(it != params_.end(), "missing parameter '" + name + "'");
  if (expect >= 0)
    DDNM_CHECK(it->second.n == expect, "parameter '" + name + "' has " + std::to_string(it->second.n) + " elements, expected " +
                                           std::to_string(expect));
  return it->second.p;
}

View UNetEngine::new_view(int H, int W, int C) {
  View v;
  v.N = B_; v.H = H; v.W = W; v.C = C; v.ld = C;
  v.p = (float*)arena_.alloc((size_t)B_ * H * W * C * sizeof(float));
  v.st = new_stats(C);
  v.st_ld = C;
  return v;
}

// a [B][C][2] block of per-channel GroupNorm sums from the pool that one memset clears at the start of every forward
StatAcc* UNetEngine::new_stats(int C) {
  const size_t need = (size_t)B_ * C * 2;
  if (stats_chunks_.empty() || stats_chunks_.back().used + need > stats_chunks_.back().cap) {
    StatsChunk c;
    c.cap = std::max<size_t>(need, (size_t)1 << 20);   // accumulators
    c.used = 0;
    c.p = (StatAcc*)arena_.alloc(c.cap * sizeof(StatAcc));
    stats_chunks_.push_back(c);
  }
  StatsChunk& c = stats_chunks_.back();
  StatAcc* p = c.p + c.used;
  c.used += need;
  return p;
}

UNetEngine::TcWeights UNetEngine::prep_weights(const std::string& main, int Cout, int Cin, int taps, const std::string& side,
                                               int CinSide) {
  TcWeights w;
  w.ktot = taps * Cin + CinSide;
  const size_t n = (size_t)Cout * w.ktot;
  w.hi = (__half*)arena_.alloc(n * sizeof(__half));
  w.lo = (__half*)arena_.alloc(n * sizeof(__half));
  split_conv_weight(P(main, (long long)Cout * Cin * taps), Cout, Cin, taps, w.hi, w.lo, w.ktot, 0, 0);
  if (CinSide) split_conv_weight(P(side, (long long)Cout * CinSide), Cout, CinSide, 1, w.hi, w.lo, w.ktot, taps * Cin, 0);
  return w;
}

const float* UNetEngine::bias_sum(const std::string& a, const std::string& b, int C) {
  std::vector<float> ha(C), hb(C, 0.f);
  CUDA_CHECK(cudaMemcpy(ha.data(), P(a, C), C * sizeof(float), cudaMemcpyDeviceToHost));
  if (!b.empty()) CUDA_CHECK(cudaMemcpy(hb.data(), P(b, C), C * sizeof(float), cudaMemcpyDeviceToHost));
  for (int i = 0; i < C; ++i) ha[i] += hb[i];
  float* d = (float*)arena_.alloc(C * sizeof(float));
  CUDA_CHECK(cudaMemcpy(d, ha.data(), C * sizeof(float), cudaMemcpyHostToDevice));
  return d;
}

float* UNetEngine::dev_copy(const std::vector<float>& v) {
  float* d = (float*)arena_.alloc(v.size() * sizeof(float));
  CUDA_CHECK(cudaMemcpy(d, v.data(), v.size() * sizeof(float), cudaMemcpyHostToDevice));
  return d;
}

void UNetEngine::add_op(const std::string& name, const std::string& kind, double flops, double bytes,
                        std::function<void(cudaStream_t)> f) {
  ops_.push_back(OpRecord{name, kind, flops, bytes, std::move(f)});
}

// GroupNorm(+SiLU) + fp16 split of x into scratch planes dst (dims as the consuming convolution sees them)
void UNetEngine::emit_gn_split(const std::string& name, const View& x, const std::string& norm, bool silu, int mode,
                               SplitView& dst, const float* ss, int ss_ld, SplitView* raw) {
  const long long out_elems = mode == SPLIT_AVG2 ? x.pixels() * x.C / 4 : x.pixels() * x.C;
  DDNM_CHECK((size_t)out_elems <= split_elems_, "split scratch too small");
  dst.C = x.C;
  if (mode == SPLIT_SAME) { dst.N = x.N; dst.H = x.H; dst.W = x.W; }
  else if (mode == SPLIT_AVG2) { dst.N = x.N; dst.H = x.H / 2; dst.W = x.W / 2; }
  else { dst.N = 4 * x.N; dst.H = x.H / 2; dst.W = x.W / 2; }
  const double in_bytes = (double)x.pixels() * x.C * 4;
  if (!norm.empty()) {
    DDNM_CHECK(x.st != nullptr, "GroupNorm input without producer-side statistics: " + name);
    const float* g = P(norm + ".weight", x.C);
    const float* b = P(norm + ".bias", x.C);
    const int groups = groups_;
    const float eps = eps_;
    __half *hi = dst.hi, *lo = dst.lo, *rhi = nullptr, *rlo = nullptr;
    if (raw) {
      DDNM_CHECK(mode == SPLIT_SAME, "raw side output only with the plain split");
      raw->N = x.N; raw->H = x.H; raw->W = x.W; raw->C = x.C;
      rhi = raw->hi; rlo = raw->lo;
    }
    add_op(name + ".gn_split", "gn_split", 0, in_bytes + out_elems * 4.0 * (raw ? 2 : 1),
           [=](cudaStream_t s) { gn_apply_split(x, groups, true, g, b, eps, silu, mode, hi, lo, s, ss, ss_ld, rhi, rlo); });
  } else {
    __half *hi = dst.hi, *lo = dst.lo;
    add_op(name + ".split", "gn_split", 0, in_bytes + out_elems * 4.0,
           [=](cudaStream_t s) { gn_apply_split(x, 1, false, nullptr, nullptr, 0.f, silu, mode, hi, lo, s); });
  }
}

void UNetEngine::emit_tc(const std::string& name, const SplitView& a, int mode, const SplitView* side, const TcWeights& w,
                         int Cout, const View& out, const float* chanadd, int ca_ld, const float* residual, int ldr, int res_mode) {
  TcLaunch L = tc_make_launch(a, mode, side, w.hi, w.lo, 1, Cout, out, chanadd, ca_ld, residual, ldr, 1.0f, num_sms_, res_mode);
  const double bytes = (double)a.N * a.H * a.W * a.C * 4 + (side ? (double)side->N * side->H * side->W * side->C * 4 : 0) +
                       (double)Cout * w.ktot * 4 + (double)out.pixels() * Cout * 4 * (residual ? 2 : 1);
  // split-K: few tiles walking a long K one k-block after the other (the 8x8 level: 32-64 CTAs, 72-144 k-blocks) are latency-bound;
  // 2 or 4 CTAs per tile, each over its own k-block range into its own partial buffer, then one small deterministic reduce
  const int tiles = L.p.tiles_x * L.p.tiles_y * L.p.tiles_n * L.p.n_tiles, kblocks = L.p.kb0 + L.p.kb1;
  static const bool split_on = std::getenv("DDNM_SPLITK") == nullptr || std::atoi(std::getenv("DDNM_SPLITK")) != 0;
  if (split_on && !L.pair && res_mode == 0 && 2 * tiles <= num_sms_ && kblocks >= 32) {
    const int S = 4 * tiles <= num_sms_ ? 4 : 2;
    const long long stride = out.pixels() * Cout;
    float* part = (float*)arena_.alloc((size_t)S * stride * sizeof(float));
    View pv;
    pv.p = part; pv.N = out.N; pv.H = out.H; pv.W = out.W; pv.C = Cout; pv.ld = Cout;
    TcLaunch Ls = tc_make_launch(a, mode, side, w.hi, w.lo, 1, Cout, pv, nullptr, 0, nullptr, 0, 1.0f, num_sms_, 0);
    DDNM_CHECK(!Ls.pair && Ls.BN == L.BN, "split-K: tile shape changed");
    Ls.p.split_k = S;
    Ls.p.split_stride = stride;
    Ls.halo = false;   // k-block ranges of a split need not be whole A units
    Ls.grid = std::min(tiles * S, num_sms_);
    add_op(name, "tc", L.flops, bytes, [Ls](cudaStream_t s) { tc_run(Ls, s); });
    add_op(name + ".splitk_reduce", "reduce", 0, (double)(S + 1 + (residual ? 1 : 0)) * stride * 4,
           [=](cudaStream_t s) { splitk_reduce(part, S, stride, out, chanadd, ca_ld, residual, ldr, s); });
    return;
  }
  add_op(name, "tc", L.flops, bytes, [L](cudaStream_t s) { tc_run(L, s); });
}

bool UNetEngine::fused_ok(const View& x, const View* side, int Cout, const View& out) const {
  return terms_ == 3 && x.st != nullptr && tc_gn_eligible(x, side, Cout, out);
}

void UNetEngine::emit_tcgn(const std::string& name, const View& x, const std::string& norm, const float* ss, int ss_ld, const View* side,
                           const TcWeights& w, int Cout, const View& out, const float* chanadd, int ca_ld, const float* residual, int ldr) {
  GnAffine gn;
  gn.gamma = P(norm + ".weight", x.C);
  gn.beta = P(norm + ".bias", x.C);
  gn.eps = eps_;
  gn.groups = groups_;
  gn.silu = true;
  gn.ss = ss;
  gn.ss_ld = ss_ld;
  TcLaunch L = tc_make_gn_launch(x, gn, side, w.hi, w.lo, Cout, out, chanadd, ca_ld, residual, ldr, num_sms_);
  // algorithmic HBM bytes: the fp32 activation(s) in, the weights, the fp32 output (+ residual) — no fp16 planes
  const double bytes = (double)x.pixels() * x.C * 4 + (side ? (double)side->pixels() * side->C * 4 : 0) + (double)Cout * w.ktot * 4 +
                       (double)out.pixels() * Cout * 4 * (residual ? 2 : 1);
  add_op(name, "tc", L.flops, bytes, [L](cudaStream_t s) { tc_run(L, s); });
}

// scratch every program needs; split planes are shared by all convolutions of a forward (stream order serialises them)
void UNetEngine::alloc_common(size_t split_elems, size_t hbuf_elems) {
  split_elems_ = split_elems;
  hbuf_elems_ = hbuf_elems;
  splitA_hi_ = (__half*)arena_.alloc(split_elems * 2);
  splitA_lo_ = (__half*)arena_.alloc(split_elems * 2);
  splitB_hi_ = (__half*)arena_.alloc(split_elems * 2);
  splitB_lo_ = (__half*)arena_.alloc(split_elems * 2);
  hbuf_ = (float*)arena_.alloc(hbuf_elems * 4);
  x_in_ = (float*)arena_.alloc((size_t)B_ * in_ch_ * R_ * R_ * 4);
  t_in_ = (float*)arena_.alloc((size_t)B_ * 4);
  labels_in_ = (int*)arena_.alloc((size_t)B_ * 4);
  CUDA_CHECK(cudaMemset(labels_in_, 0, (size_t)B_ * 4));
  out_ = (float*)arena_.alloc((size_t)B_ * out_ch_ * R_ * R_ * 4);
}

void UNetEngine::emit_up2_conv(const std::string& name, const SplitView& a, const std::string& wname, int Cout, const View& out,
                               const float* chanadd, int ca_ld) {
  const int Cin = a.C;
  const size_t per_phase = (size_t)Cout * 4 * Cin;
  __half* wh = (__half*)arena_.alloc(4 * per_phase * sizeof(__half));
  __half* wl = (__half*)arena_.alloc(4 * per_phase * sizeof(__half));
  presum_up2_weights(P(wname, (long long)Cout * Cin * 9), Cout, Cin, wh, wl, 0);
  for (int ph = 0; ph < 4; ++ph) {
    TcLaunch L = tc_make_up2_launch(a, wh + ph * per_phase, wl + ph * per_phase, Cout, out, chanadd, ca_ld, ph >> 1, ph & 1, num_sms_);
    const double bytes = (double)a.N * a.H * a.W * Cin * 4 + (double)per_phase * 4 + (double)a.N * a.H * a.W * Cout * 4;
    add_op(name + ".ph" + std::to_string(ph), "tc", L.flops, bytes, [L](cudaStream_t s) { tc_run(L, s); });
  }
}

void UNetEngine::alloc_attention(size_t qkv_elems, size_t s_elems, size_t o_elems) {
  qkv_ = (float*)arena_.alloc(qkv_elems * 4);
  attS_ = (float*)arena_.alloc(s_elems * 4);
  attO_ = (float*)arena_.alloc(o_elems * 4);
  qkvh_ = (__half*)arena_.alloc(qkv_elems * 2);
  qkvl_ = (__half*)arena_.alloc(qkv_elems * 2);
  ph_ = (__half*)arena_.alloc(s_elems * 2);
  pl_ = (__half*)arena_.alloc(s_elems * 2);
  vth_ = (__half*)arena_.alloc(o_elems * 2);
  vtl_ = (__half*)arena_.alloc(o_elems * 2);
}

void UNetEngine::emit_attention_core(const std::string& name, int T, int heads, int ch, int qkv_ld, int head_stride, int q_off,
                                     int k_off, int v_off, float alpha) {
  float *q = qkv_, *S = attS_, *O = attO_;
  const int Bn = B_, C = heads * ch;
  const long long img = (long long)T * qkv_ld;
  const double fl = 2.0 * Bn * heads * (double)T * T * ch;
  const double sbytes = (double)Bn * heads * T * T * 4;
  if (T % 128 == 0 && ch % 64 == 0) {
    // tensor cores: raw fp16 split of q|k|v, S = alpha Q K^T, softmax -> fp16 P, V^T planes, O = P V
    __half *qh = qkvh_, *ql = qkvl_, *ph = ph_, *pl = pl_, *vh = vth_, *vl = vtl_;
    // the raw split is elementwise, so the [token][qkv_ld] buffer is viewed as rows of C = heads*ch channels (<= MAX_C)
    DDNM_CHECK(qkv_ld % C == 0, "qkv row is not a multiple of the attention width");
    View qv;
    qv.p = qkv_; qv.N = B_; qv.H = 1; qv.W = T * (qkv_ld / C); qv.C = C; qv.ld = C;
    add_op(name + ".qkv_split", "gn_split", 0, (double)Bn * T * qkv_ld * 8,
           [=](cudaStream_t s) { gn_apply_split(qv, 1, false, nullptr, nullptr, 0.f, false, SPLIT_SAME, qh, ql, s); });
    const long long hs = head_stride ? head_stride : qkv_ld;   // extent-1 dims still need a legal (non-zero) TMA stride
    GemmOperand A{qh + q_off, ql + q_off, qkv_ld, hs, img};
    GemmOperand Bk{qh + k_off, ql + k_off, qkv_ld, hs, img};
    TcLaunch L1 = tc_make_gemm_launch(A, Bk, T, T, ch, heads, Bn, S, (long long)heads * T * T, (long long)T * T, T, alpha, num_sms_);
    add_op(name + ".qk", "tc", L1.flops, (double)Bn * T * qkv_ld * 4 + sbytes, [L1](cudaStream_t s) { tc_run(L1, s); });
    add_op(name + ".softmax", "softmax", 0, sbytes * 2, [=](cudaStream_t s) { softmax_split(S, (long long)Bn * heads * T, T, ph, pl, s); });
    add_op(name + ".v_transpose", "gn_split", 0, (double)Bn * T * C * 8,
           [=](cudaStream_t s) { transpose_split(q, qkv_ld, head_stride, v_off, Bn, T, heads, ch, vh, vl, s); });
    GemmOperand P{ph, pl, T, (long long)T * T, (long long)heads * T * T};
    GemmOperand Vt{vh, vl, T, (long long)ch * T, (long long)heads * ch * T};
    TcLaunch L2 = tc_make_gemm_launch(P, Vt, T, ch, T, heads, Bn, O, (long long)T * C, ch, C, 1.0f, num_sms_);
    add_op(name + ".pv", "tc", L2.flops, sbytes + (double)Bn * T * C * 8, [L2](cudaStream_t s) { tc_run(L2, s); });
  } else {
    add_op(name + ".qk", "sgemm", fl, (double)Bn * heads * T * (2.0 * ch + T) * 4, [=](cudaStream_t s) {
      sgemm_batched(true, Bn, heads, T, T, ch, alpha, q + q_off, qkv_ld, img, head_stride, q + k_off, qkv_ld, img, head_stride, S, T,
                    (long long)heads * T * T, (long long)T * T, s);
    });
    add_op(name + ".softmax", "softmax", 0, sbytes * 2, [=](cudaStream_t s) { softmax_rows(S, (long long)Bn * heads * T, T, s); });
    add_op(name + ".pv", "sgemm", fl, (double)Bn * heads * T * (2.0 * ch + T) * 4, [=](cudaStream_t s) {
      sgemm_batched(false, Bn, heads, T, ch, T, 1.0f, S, T, (long long)heads * T * T, (long long)T * T, q + v_off, qkv_ld, img, head_stride, O,
                    C, (long long)T * C, ch, s);
    });
  }
}

// network stem: 3x3 conv on the caller's NCHW tensor -> NHWC view
void UNetEngine::emit_stem(const std::string& wname, const View& out) {
  const float* xin = x_in_;
  const float *w = P(wname + ".weight", (long long)out.C * in_ch_ * 9), *b = P(wname + ".bias", out.C);
  const int cin = in_ch_;
  add_op("stem", "stem", 2.0 * B_ * R_ * R_ * (double)out.C * cin * 9, (double)B_ * R_ * R_ * (cin + out.C) * 4,
         [=](cudaStream_t s) { conv3x3_small_cin(xin, cin, w, b, out, s); });
  // (the GroupNorm sums of the stem output are accumulated by the stem kernel itself: out.st)
}

// network head: GroupNorm + SiLU + 3x3 conv to out_ch (3 or 6), NCHW result.  The convolution runs on the tensor cores with
// the output channels zero-padded to one 64-wide N tile (10-20x redundant columns still beat a CUDA-core kernel ~2x), then
// the out_ch real channels are copied out as NCHW.
void UNetEngine::emit_head(const std::string& norm, const std::string& conv, const View& fh) {
  DDNM_CHECK(fh.st != nullptr, "head input without statistics");
  DDNM_CHECK(out_ch_ <= 64, "head convolution: out_ch <= 64");
  if (head_conv_supported(fh, out_ch_) && std::getenv("DDNM_HEAD_TC") == nullptr) {
    // one kernel: the activation is read once, normalised on the way into shared memory, convolved in exact fp32 (3 or 6 output
    // channels are too few for the tensor cores: the padded-N form below streams the A operand for 0.6 ms + a 0.2 ms GroupNorm pass)
    const float *g = P(norm + ".weight", fh.C), *b = P(norm + ".bias", fh.C);
    const float *w = P(conv + ".weight", (long long)out_ch_ * fh.C * 9), *cb = P(conv + ".bias", out_ch_);
    const int groups = groups_, oc = out_ch_;
    const float eps = eps_;
    float* o = out_;
    add_op("head.conv", "head", 2.0 * fh.pixels() * (double)oc * fh.C * 9, (double)fh.pixels() * (fh.C + oc) * 4,
           [=](cudaStream_t s) { head_conv(fh, groups, g, b, eps, w, cb, oc, o, s); });
    return;
  }
  SplitView A{splitA_hi_, splitA_lo_};
  emit_gn_split("head", fh, norm, true, SPLIT_SAME, A);
  const int ktot = 9 * fh.C;
  TcWeights w;
  w.ktot = ktot;
  w.hi = (__half*)arena_.alloc((size_t)64 * ktot * sizeof(__half));
  w.lo = (__half*)arena_.alloc((size_t)64 * ktot * sizeof(__half));
  CUDA_CHECK(cudaMemset(w.hi, 0, (size_t)64 * ktot * sizeof(__half)));
  CUDA_CHECK(cudaMemset(w.lo, 0, (size_t)64 * ktot * sizeof(__half)));
  split_conv_weight(P(conv + ".weight", (long long)out_ch_ * fh.C * 9), out_ch_, fh.C, 9, w.hi, w.lo, ktot, 0, 0);
  std::vector<float> hb(64, 0.f);
  CUDA_CHECK(cudaMemcpy(hb.data(), P(conv + ".bias", out_ch_), out_ch_ * sizeof(float), cudaMemcpyDeviceToHost));
  float* bias64 = dev_copy(hb);
  View o64;
  o64.N = B_; o64.H = fh.H; o64.W = fh.W; o64.C = 64; o64.ld = 64;
  o64.p = (float*)arena_.alloc((size_t)B_ * fh.H * fh.W * 64 * sizeof(float));
  emit_tc("head.conv", A, TAPS_3X3, nullptr, w, 64, o64, bias64, 0, nullptr, 0);
  float* o = out_;
  const View real = o64.slice(0, out_ch_);
  add_op("head.to_nchw", "head", 0, (double)fh.pixels() * (64 + out_ch_) * 4, [=](cudaStream_t s) { nhwc_to_nchw(real, o, s); });
}

void UNetEngine::set_terms(int t) {
  DDNM_CHECK(!finalized_, "precision must be chosen before finalize");
  DDNM_CHECK(t == 1 || t == 3, "terms must be 1 (fast fp16) or 3 (fp32-grade)");
  terms_ = t;
}

void UNetEngine::finalize() {
  DDNM_CHECK(!finalized_, "finalize called twice");
  const int prev = tc_get_terms();
  tc_set_terms(terms_);
  try {
    build_program();
  } catch (...) {
    tc_set_terms(prev);
    throw;
  }
  tc_set_terms(prev);
  // every GroupNorm sum is accumulated with (integer, order-independent) atomics during the forward: clear the pool first
  std::vector<OpRecord> zero;
  for (const StatsChunk& c : stats_chunks_) {
    StatAcc* sb = c.p;
    const size_t sbytes = c.used * sizeof(StatAcc);
    zero.push_back(OpRecord{"stats.zero", "memset", 0, (double)sbytes,
                            [=](cudaStream_t s) { CUDA_CHECK(cudaMemsetAsync(sb, 0, sbytes, s)); }});
  }
  ops_.insert(ops_.begin(), zero.begin(), zero.end());
  CUDA_CHECK(cudaDeviceSynchronize());
  finalized_ = true;
}

void UNetEngine::run_ops(cudaStream_t s, size_t n) {
  for (size_t i = 0; i < n && i < ops_.size(); ++i) ops_[i].run(s);
}

void UNetEngine::set_labels(const int* labels_dev, cudaStream_t stream) {
  DDNM_CHECK(class_cond_, "set_labels on a network without a label embedding");
  DDNM_CHECK(labels_dev != nullptr, "null labels");
  if (labels_dev != labels_in_) CUDA_CHECK(cudaMemcpyAsync(labels_in_, labels_dev, (size_t)B_ * sizeof(int), cudaMemcpyDeviceToDevice, stream));
}

void UNetEngine::forward(const float* x, const float* t, float* out, cudaStream_t stream) {
  DDNM_CHECK(finalized_, "forward before finalize");
  const size_t xin = (size_t)B_ * in_ch_ * R_ * R_ * 4;
  if (x != x_in_) CUDA_CHECK(cudaMemcpyAsync(x_in_, x, xin, cudaMemcpyDeviceToDevice, stream));
  if (t != t_in_) CUDA_CHECK(cudaMemcpyAsync(t_in_, t, (size_t)B_ * 4, cudaMemcpyDeviceToDevice, stream));
  replay(stream, ops_.size() - n_tail_ops_, graph_, graph_exec_);
  if (out != out_) CUDA_CHECK(cudaMemcpyAsync(out, out_, out_elems() * 4, cudaMemcpyDeviceToDevice, stream));
}

// runs ops_[0, n) on `stream`: eagerly, or as a CUDA graph captured on first use into (g, exec)
void UNetEngine::replay(cudaStream_t stream, size_t n, cudaGraph_t& g, cudaGraphExec_t& exec) {
  if (!use_graph_) {
    run_ops(stream, n);
    return;
  }
  if (!exec) {
    // Capture once on a private stream (the caller's may be the legacy default stream, which cannot capture).
    // A warm-up pass runs first: one-time cudaFuncSetAttribute calls are not capturable.
    cudaStream_t cs = nullptr;
    CUDA_CHECK(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
    CUDA_CHECK(cudaStreamSynchronize(stream));
    run_ops(cs, n);
    CUDA_CHECK(cudaStreamSynchronize(cs));
    CUDA_CHECK(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
    try {
      run_ops(cs, n);
    } catch (...) {
      cudaGraph_t gg = nullptr;
      cudaStreamEndCapture(cs, &gg);
      if (gg) cudaGraphDestroy(gg);
      cudaStreamDestroy(cs);
      throw;
    }
    CUDA_CHECK(cudaStreamEndCapture(cs, &g));
    CUDA_CHECK(cudaGraphInstantiate(&exec, g, 0));
    CUDA_CHECK(cudaStreamDestroy(cs));
  }
  CUDA_CHECK(cudaGraphLaunch(exec, stream));
}

bool UNetEngine::read_tap(const std::string& name, float* dst, long long capacity, cudaStream_t stream) {
  auto it = taps_.find(name);
  if (it == taps_.end()) return false;
  const View& v = it->second;
  DDNM_CHECK(capacity >= v.pixels() * v.C, "tap buffer too small");
  nhwc_to_nchw(v, dst, stream);
  return true;
}

double UNetEngine::flops_per_forward() const {
  double f = 0;
  for (auto& op : ops_) f += op.flops;
  return f;
}

std::string UNetEngine::profile(const float* x, const float* t, float* out, cudaStream_t stream) {
  const bool g = use_graph_;
  use_graph_ = false;
  forward(x, t, out, stream);  // warm
  CUDA_CHECK(cudaStreamSynchronize(stream));
  std::vector<cudaEvent_t> ev(ops_.size() + 1);
  for (auto& e : ev) CUDA_CHECK(cudaEventCreate(&e));
  CUDA_CHECK(cudaEventRecord(ev[0], stream));
  for (size_t i = 0; i < ops_.size(); ++i) {
    ops_[i].run(stream);
    CUDA_CHECK(cudaEventRecord(ev[i + 1], stream));
  }
  CUDA_CHECK(cudaStreamSynchronize(stream));
  std::ostringstream js;
  js << "[";
  for (size_t i = 0; i < ops_.size(); ++i) {
    float ms = 0;
    CUDA_CHECK(cudaEventElapsedTime(&ms, ev[i], ev[i + 1]));
    if (i) js << ",";
    js << "{\"name\":\"" << ops_[i].name << "\",\"kind\":\"" << ops_[i].kind << "\",\"ms\":" << ms << ",\"flops\":" << ops_[i].flops
       << ",\"bytes\":" << ops_[i].bytes << "}";
  }
  js << "]";
  for (auto& e : ev) cudaEventDestroy(e);
  use_graph_ = g;
  return js.str();
}

}  // namespace ddnm

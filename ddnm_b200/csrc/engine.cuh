// The engines: static launch programs for the three networks on the reference's hot path
//   UNetSimple   <- guided_diffusion/models.py::Model             (celeba_hq.yml, model.type == "simple")
//   UNetOpenAI   <- guided_diffusion/unet.py::UNetModel           (imagenet_256.yml, model.type == "openai")
//   UNetEncoder  <- guided_diffusion/unet.py::EncoderUNetModel    (the classifier of imagenet_256_cc.yml)
// built once per (config, batch) and replayed as a CUDA graph.  UNetEngine holds everything they share.
#pragma once
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "common.cuh"
#include "tc_gemm.cuh"

namespace ddnm {

struct SimpleCfg {
  int ch = 128, out_ch = 3, n_levels = 6;
  int ch_mult[8] = {1, 1, 2, 2, 4, 4, 0, 0};
  int num_res_blocks = 2;
  int n_attn_res = 1;
  int attn_res[4] = {16, 0, 0, 0};
  int in_channels = 3, resolution = 256, groups = 32;
  float eps = 1e-6f;
};

class Arena {
 public:
  ~Arena();
  void* alloc(size_t bytes);
  size_t used() const { return total_; }

 private:
  std::vector<void*> blocks_;
  size_t total_ = 0;
};

struct OpRecord {
  std::string name;
  std::string kind;   // "tc", "gn_stats", "gn_apply", ...
  double flops = 0;   // algorithmic
  double bytes = 0;   // algorithmic HBM bytes (in + out)
  std::function<void(cudaStream_t)> run;
};

struct OpenAICfg {
  int image_size = 256, model_channels = 256, num_res_blocks = 2, n_levels = 6;
  int channel_mult[8] = {1, 1, 2, 2, 4, 4, 0, 0};
  int n_attn_ds = 3;
  int attn_ds[4] = {8, 16, 32, 0};   // downsample rates at which attention runs (image_size // resolution)
  int num_head_channels = 64;
  int out_channels = 6, in_channels = 3, groups = 32;
  float eps = 1e-5f;
  int num_classes = 0;   // > 0: class-conditional (label_emb [num_classes, 4*model_channels], unet.py:478-479)
  int low_res = 0;       // > 0: SuperResModel (unet.py:667-681): the stem convolves cat([x, bilinear(low_res)]), low_res [B,3,s,s]
  // heads per attention block when num_head_channels <= 0 (unet.py:277-283): num_heads in the input and middle blocks,
  // num_heads_upsample (<= 0: num_heads, unet.py:452-453) in the output blocks
  int num_heads = 1, num_heads_upsample = -1;
  int new_attention_order = 0;   // 1: QKVAttention (q, k, v split before the heads, unet.py:361-389); 0: QKVAttentionLegacy
};

// tests: engines built after the call size their grids and launch policy for min(n, the device's count) SMs (0 = the device's count)
void engine_debug_sm_count(int n);
int engine_sm_count(const cudaDeviceProp& prop);   // the SM count launches are planned for on that device

class UNetEngine {
 public:
  UNetEngine(int batch, int in_channels, int out_ch, int resolution, int groups, float eps);
  virtual ~UNetEngine();
  void set_param(const std::string& name, const float* data, long long numel);
  void finalize();
  // x: [B,3,R,R] NCHW fp32, t: [B] fp32 (device), out: [B,out_ch,R,R] NCHW fp32 (device)
  void forward(const float* x, const float* t, float* out, cudaStream_t stream);
  // tests: copy an internal activation (by oracle tap name) as NCHW fp32
  bool read_tap(const std::string& name, float* dst_nchw, long long capacity, cudaStream_t stream);
  // per-op timing of one eager (non-graph) forward; returns JSON
  std::string profile(const float* x, const float* t, float* out, cudaStream_t stream);
  int batch() const { return B_; }
  int out_ch() const { return out_ch_; }
  int in_channels() const { return in_ch_; }
  int resolution() const { return R_; }
  float* x_in() const { return x_in_; }
  float* t_in() const { return t_in_; }
  // t_in() = t for every image, on the device
  void fill_t(float t, cudaStream_t stream);
  // class labels of the next forward (device int32 [B]); only meaningful for class-conditional networks
  int* labels_in() const { return labels_in_; }
  bool class_conditional() const { return class_cond_; }
  void set_labels(const int* labels_dev, cudaStream_t stream);
  // super-resolution networks: the conditioning image [B, in_channels, s, s] (s = low_res_size()) every following forward reads
  int low_res_size() const { return lowres_; }
  void set_low_res(const float* low_res_dev, cudaStream_t stream);
  float* out_buf() const { return out_; }
  void set_use_graph(bool on) { use_graph_ = on; }
  // 3 = fp32-grade products (parity mode, default); 1 = single fp16 product per MAC (fast, NOT parity-grade). Before finalize.
  void set_terms(int t);
  // batch-invariant mode (see tc_make_launch): every image's result depends on that image and the layer shapes alone, not on the
  // batch size, the image's row, padding rows or the SM count.  Before finalize.
  void set_batch_invariant(bool on);
  size_t workspace_bytes() const { return arena_.used(); }
  int num_launches() const { return (int)ops_.size(); }
  double flops_per_forward() const;

 protected:
  struct Param { float* p; long long n; };
  const float* P(const std::string& name, long long expect = -1) const;
  View new_view(int H, int W, int C);
  // [B_][H][W][C] over existing memory, no statistics
  View view_of(float* p, int H, int W, int C) const;
  StatAcc* new_stats(int C);
  struct TcWeights { __half *hi, *lo; int ktot; };
  // main / side: full parameter names of the OIHW weight tensors ("" = absent)
  TcWeights prep_weights(const std::string& main, int Cout, int Cin, int taps, const std::string& side, int CinSide);
  const float* bias_sum(const std::string& a, const std::string& b, int C);
  float* dev_copy(const std::vector<float>& v);
  bool has_param(const std::string& name) const { return params_.count(name) != 0; }

  void add_op(const std::string& name, const std::string& kind, double flops, double bytes, std::function<void(cudaStream_t)> f);
  // norm: parameter prefix of the GroupNorm ("" = raw split); ss: optional per-(image, channel) scale/shift rows
  // [scale(C) | shift(C)] with row pitch ss_ld (use_scale_shift_norm, unet.py:250-252)
  // raw: optional second destination receiving the un-normalised split of x in the same pass (1x1 shortcut input)
  void emit_gn_split(const std::string& name, const View& x, const std::string& norm, bool silu, int mode, SplitView& dst,
                     const float* ss = nullptr, int ss_ld = 0, SplitView* raw = nullptr);
  void emit_tc(const std::string& name, const SplitView& a, int mode, const SplitView* side, const TcWeights& w, int Cout,
               const View& out, const float* chanadd, int ca_ld, const float* residual, int ldr, int res_mode = 0);
  // softmax(alpha * Q K^T) V for `heads` heads of width ch over T tokens; q/k/v live in the fp32 buffer qkv
  // ([token][qkv_ld], head h at column h*head_stride + {q_off, k_off, v_off}); result -> attO_ [token][heads*ch].
  // T % 128 == 0 and ch % 8 == 0 run both contractions on the tensor cores (a head width that is not a multiple of 64 ends in a
  // zero-filled partial k-block / N tile), otherwise (8x8 maps) on CUDA cores.
  void emit_attention_core(const std::string& name, float* qkv, int T, int heads, int ch, int qkv_ld, int head_stride, int q_off,
                           int k_off, int v_off, float alpha);
  void alloc_attention(size_t qkv_elems, size_t s_elems, size_t o_elems);
  // conv3x3(nearest_upsample_x2(a)) + bias as 4 parity-phase 2x2 convolutions on the low-res split `a` (4/9 of the MACs,
  // no upsampled copy); wname: OIHW 3x3 weight parameter
  void emit_up2_conv(const std::string& name, const SplitView& a, const std::string& wname, int Cout, const View& out,
                     const float* chanadd, int ca_ld);
  void emit_stem(const std::string& wname, const View& out);
  void emit_head(const std::string& norm, const std::string& conv, const View& h);

  // one block's projection of the timestep embedding: `rows` rows of the stacked matrix, from the [rows, 4 ch] parameter `weight`
  struct EmbProj { std::string block, weight; const float* bias; int rows; };
  // timestep embedding: sinusoid(t) over ch channels ([sin | cos] if sin_first), layer0 -> SiLU -> layer1 (+ label_emb[labels_in_]
  // if label_emb) -> SiLU, then every projection in `projs` as one stacked Linear into [B][emb_ld_] rows (emb_rows)
  void emit_time_embed(const std::string& name, const std::string& layer0, const std::string& layer1, int ch, bool sin_first,
                       const float* label_emb, int num_classes, const std::vector<EmbProj>& projs);
  const float* emb_rows(const std::string& block) const { return emb_all_ + emb_off_.at(block); }

  // guided_diffusion/unet.py's module lists as data: a block is one TimestepEmbedSequential, its layers run in order
  enum LayerKind { LAYER_CONV, LAYER_RES, LAYER_RES_DOWN, LAYER_RES_UP, LAYER_ATTN };
  struct Block {
    struct Layer { int kind, cin, cout; };
    std::vector<Layer> layers;
    int res_in, res_out, cout;
  };
  struct Torso { std::vector<Block> input; Block middle; };
  // input_blocks (input[0] is the stem convolution) and middle_block of UNetModel / EncoderUNetModel (unet.py:482-565, :740-823)
  static Torso plan_torso(int image_size, int in_channels, int model_channels, const int* channel_mult, int n_levels,
                          int num_res_blocks, const int* attn_ds, int n_attn_ds);
  // ResBlock._forward (unet.py:236-256), use_scale_shift_norm = True; kind LAYER_RES, LAYER_RES_DOWN or LAYER_RES_UP.
  // h: where in_layers' convolution writes (out's shape), with the statistics out_layers' GroupNorm reads
  void emit_res_block(const std::string& p, const View& x, const View& h, const View& out, int kind);
  // AttentionBlock._forward (unet.py:299-305); qkv: [B][T][3C] destination of the qkv convolution
  void emit_attention_block(const std::string& p, const View& x, const View& out, int heads, bool new_order, float* qkv);

  // hbuf_elems == 0: no resblock intermediate
  void alloc_common(size_t split_elems, size_t hbuf_elems);
  virtual void build_program() = 0;
  // elements of the result forward() copies out: [B, out_ch, R, R] for the denoisers
  virtual size_t out_elems() const { return (size_t)B_ * out_ch_ * R_ * R_; }
  void run_ops(cudaStream_t s, size_t n = (size_t)-1);
  void replay(cudaStream_t stream, size_t n, cudaGraph_t& g, cudaGraphExec_t& exec);

  int B_, in_ch_, out_ch_, R_, groups_;
  float eps_;
  int num_sms_ = 132;
  bool finalized_ = false, use_graph_ = true;
  int terms_ = 3;
  bool invariant_ = false;
  Arena arena_;
  std::map<std::string, Param> params_;
  std::vector<OpRecord> ops_;
  size_t n_tail_ops_ = 0;   // ops at the end of ops_ that forward() leaves out (the classifier's backward pass)
  std::map<std::string, View> taps_;
  // fixed I/O staging (graph replays need stable addresses)
  float *x_in_ = nullptr, *t_in_ = nullptr, *out_ = nullptr;
  int* labels_in_ = nullptr;
  bool class_cond_ = false;
  float* lowres_in_ = nullptr;   // [B][in_ch_][lowres_][lowres_] when lowres_ > 0
  int lowres_ = 0;
  bool lowres_set_ = false;
  // scratch
  __half *splitA_hi_ = nullptr, *splitA_lo_ = nullptr, *splitB_hi_ = nullptr, *splitB_lo_ = nullptr;
  size_t split_elems_ = 0;
  float* hbuf_ = nullptr;      // resblock intermediate
  size_t hbuf_elems_ = 0;
  float *qkv_ = nullptr, *attS_ = nullptr, *attO_ = nullptr;
  __half *qkvh_ = nullptr, *qkvl_ = nullptr, *ph_ = nullptr, *pl_ = nullptr, *vth_ = nullptr, *vtl_ = nullptr;
  struct StatsChunk { StatAcc* p; size_t cap, used; };
  std::vector<StatsChunk> stats_chunks_;
  float* emb_all_ = nullptr;   // [B][emb_ld_] every block's projection of the timestep embedding
  int emb_ld_ = 0;
  std::map<std::string, int> emb_off_;
  cudaGraph_t graph_ = nullptr;
  cudaGraphExec_t graph_exec_ = nullptr;
};

class UNetSimple : public UNetEngine {
 public:
  UNetSimple(const SimpleCfg& cfg, int batch);

 private:
  void build_program() override;
  void emit_resblock(const std::string& p, const View& x, const View& out);
  void emit_attn(const std::string& p, const View& x, const View& out);
  void emit_downsample(const std::string& p, const View& x, const View& out);
  void emit_upsample(const std::string& p, const View& x, const View& out);
  SimpleCfg cfg_;
};

class UNetOpenAI : public UNetEngine {
 public:
  UNetOpenAI(const OpenAICfg& cfg, int batch);

 private:
  void build_program() override;
  // heads of an attention block over C channels; upsample: the block belongs to the output blocks
  int attn_heads(int C, bool upsample) const;
  OpenAICfg cfg_;
};

// guided_diffusion/unet.py::EncoderUNetModel (the classifier of imagenet_256_cc.yml): use_scale_shift_norm, resblock_updown,
// legacy attention in the blocks, pool "attention" (AttentionPool2d) or "adaptive".  Besides the logits it computes
//   grad = scale * d/dx sum_b log_softmax(classifier(x, t))[b, labels[b]]       (cond_fn, diffusion.py:183-189)
// with a hand-written backward pass in the same op list: the forward keeps every GroupNorm input (with its statistics), each
// attention block's qkv and the head's tokens in dedicated buffers; the convolution data gradients run on the tensor-core
// kernel with flipped / transposed weights.
struct EncoderCfg {
  int image_size = 256, model_channels = 128, num_res_blocks = 2, n_levels = 6;
  int channel_mult[8] = {1, 1, 2, 2, 4, 4, 0, 0};
  int n_attn_ds = 3;
  int attn_ds[4] = {8, 16, 32, 0};
  int num_head_channels = 64;
  int out_channels = 1000, in_channels = 3, groups = 32;
  float eps = 1e-5f;
  int pool = 1;   // 0 adaptive, 1 attention
};

class UNetEncoder : public UNetEngine {
 public:
  UNetEncoder(const EncoderCfg& cfg, int batch);
  ~UNetEncoder() override;
  // logits [B, out_channels] (may be null) and grad [B, in_channels, R, R] (NCHW fp32, device); labels: device int32 [B]
  // labels_checked: the caller already ran check_labels on these labels (a guided loop checks its fixed labels once)
  void grad(const float* x, const float* t, const int* labels, float scale, float* grad_out, float* logits, cudaStream_t stream,
            bool labels_checked = false);
  // throws unless every label is in [0, out_channels); reads them to the host (synchronises `stream`)
  void check_labels(const int* labels, cudaStream_t stream) const;
  int num_classes() const { return cfg_.out_channels; }

 private:
  void build_program() override;
  size_t out_elems() const override { return (size_t)B_ * cfg_.out_channels; }
  struct Res { std::string p; View x, h, out; bool down, skip_conv; };
  struct Attn { std::string p; View x, out; float* qkv; };
  struct Layer { int kind; Res r; Attn a; };   // kind 0 ResBlock, 1 AttentionBlock
  void emit_head(const View& h);
  void emit_backward(const View& stem_out, const std::vector<Layer>& layers, const View& top);
  // GroupNorm (+ scale-shift) (+ SiLU) (+ 2x2 average pool) backward: g = gradient of the block's activation, x = the
  // GroupNorm input; writes dx (+ add) as fp32 (dx32, may be null) and as the fp16 split `dst` of the next data-gradient convolution
  void emit_gn_backward(const std::string& name, const float* g, const View& x, const std::string& norm, const float* ss, int ss_ld,
                        bool silu, bool pool, const float* add, bool add_pool, float* dx32, const SplitView& dst);
  TcWeights prep_weights_t(const std::string& w, int Cout, int Cin, int taps);
  EncoderCfg cfg_;
  // head (attention pool): tokens X [B][T][C], qkv [B][T][3C], probabilities [B][heads][T], pooled a0 [B][C]
  int headT_ = 0;
  float *hf_ = nullptr, *tok_ = nullptr, *hqkv_ = nullptr, *hp_ = nullptr, *ha0_ = nullptr;
  // backward scratch
  float *scale_in_ = nullptr, *grad_ = nullptr, *gx_[2] = {nullptr, nullptr}, *g1_ = nullptr, *g2_ = nullptr, *gqkv_ = nullptr;
  float *sP_ = nullptr, *sdP_ = nullptr, *gnb_part_ = nullptr;
  size_t gnb_part_elems_ = 0;
  cudaGraph_t ggraph_ = nullptr;
  cudaGraphExec_t ggraph_exec_ = nullptr;
};

}  // namespace ddnm

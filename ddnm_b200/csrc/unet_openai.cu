// UNetOpenAI: launch program for guided_diffusion/unet.py::UNetModel as configured by imagenet_256.yml and the rest of the
// guided-diffusion ImageNet family (use_scale_shift_norm, resblock_updown; legacy or new attention order, heads of num_head_channels
// channels or a fixed count per block; learn_sigma -> 6 outputs).
// Everything is computed with fp32-grade arithmetic (the reference's fp32 mode); its optional fp16 torso
// (unet.py:619-625) is a lower-precision variant of the same maths.
#include <algorithm>
#include <cmath>

#include "engine.cuh"
#include "kernels.cuh"

namespace ddnm {

UNetOpenAI::UNetOpenAI(const OpenAICfg& cfg, int batch)
    : UNetEngine(batch, cfg.in_channels, cfg.out_channels, cfg.image_size, cfg.groups, cfg.eps), cfg_(cfg) {
  class_cond_ = cfg.num_classes > 0;
  DDNM_CHECK(cfg.low_res >= 0 && cfg.low_res <= cfg.image_size, "low_res size must be in [0, image_size]");
  lowres_ = cfg.low_res;
}

// ResBlock._forward (unet.py:236-256), use_scale_shift_norm = True.
//   kind DOWN: h = avg_pool(SiLU(GN(x))), x = avg_pool(x);  kind UP: nearest x2 of both (h_upd / x_upd, :170-177)
void UNetOpenAI::emit_resblock(const std::string& p, const View& x, const View& out, int kind) {
  const int Cin = x.C, Cout = out.C;
  DDNM_CHECK((size_t)(out.pixels() * Cout) <= hbuf_elems_, "hbuf too small");
  if (kind != RES_PLAIN) DDNM_CHECK(Cin == Cout, "up/down ResBlocks keep the channel count");
  SplitView A{splitA_hi_, splitA_lo_}, Bs{splitB_hi_, splitB_lo_};
  const int mode1 = kind == RES_DOWN ? SPLIT_AVG2 : SPLIT_SAME;
  const bool has_skip_conv = has_param(p + ".skip_connection.weight");
  View h;
  h.p = hbuf_; h.N = B_; h.H = out.H; h.W = out.W; h.C = Cout; h.ld = Cout;
  h.st = new_stats(Cout); h.st_ld = Cout;   // conv1's epilogue accumulates the sums out_layers.0 needs
  emit_gn_split(p + ".in", x, p + ".in_layers.0", true, mode1, A, nullptr, 0, has_skip_conv ? &Bs : nullptr);
  if (kind == RES_UP) {
    // in_conv(nearest_up(SiLU(GN(x)))) as four 2x2 parity-phase convolutions on the low-res activation
    emit_up2_conv(p + ".conv1", A, p + ".in_layers.2.weight", Cout, h, P(p + ".in_layers.2.bias", Cout), 0);
  } else {
    TcWeights w1 = prep_weights(p + ".in_layers.2.weight", Cout, Cin, 9, "", 0);
    emit_tc(p + ".conv1", A, TAPS_3X3, nullptr, w1, Cout, h, P(p + ".in_layers.2.bias", Cout), 0, nullptr, 0);
  }
  // out_norm(h) * (1 + scale) + shift -> SiLU -> conv  (:250-253); scale|shift = emb_layers(emb) computed once per forward
  emit_gn_split(p + ".out", h, p + ".out_layers.0", true, SPLIT_SAME, A, ss_all_ + ss_off_.at(p), ss_total_);
  if (has_skip_conv) {
    DDNM_CHECK(kind == RES_PLAIN, "skip convolution on an up/down block");
    TcWeights w2 = prep_weights(p + ".out_layers.3.weight", Cout, Cout, 9, p + ".skip_connection.weight", Cin);
    emit_tc(p + ".conv2+skip", A, TAPS_3X3, &Bs, w2, Cout, out, bias_sum(p + ".out_layers.3.bias", p + ".skip_connection.bias", Cout), 0,
            nullptr, 0);
  } else {
    DDNM_CHECK(Cin == Cout, "identity skip needs equal channels");
    TcWeights w2 = prep_weights(p + ".out_layers.3.weight", Cout, Cout, 9, "", 0);
    emit_tc(p + ".conv2", A, TAPS_3X3, nullptr, w2, Cout, out, P(p + ".out_layers.3.bias", Cout), 0, x.p, x.ld,
            kind == RES_UP ? 1 : (kind == RES_DOWN ? 2 : 0));
  }
}

// AttentionBlock.__init__ (unet.py:277-283, 452-453): num_head_channels-wide heads, else a fixed count per block
int UNetOpenAI::attn_heads(int C, bool upsample) const {
  int heads = cfg_.num_heads;
  if (cfg_.num_head_channels > 0) heads = C / cfg_.num_head_channels;
  else if (upsample && cfg_.num_heads_upsample > 0) heads = cfg_.num_heads_upsample;
  DDNM_CHECK(heads >= 1 && C % heads == 0 && (cfg_.num_head_channels <= 0 || C % cfg_.num_head_channels == 0),
             "attention channels " + std::to_string(C) + " do not split into equal heads");
  return heads;
}

// AttentionBlock._forward (unet.py:299-305); weight = softmax((q*s)^T (k*s)), s = ch^-1/4; a = weight . v; head h of a is channels
// [h*ch, (h+1)*ch) in both orders.  The qkv channels of head h are
//   QKVAttentionLegacy (:337-354): [q | k | v] at h*3ch + {0, ch, 2ch}   (heads split before q, k, v)
//   QKVAttention (:361-389):       h*ch + {0, C, 2C}                    (q, k, v split before the heads)
void UNetOpenAI::emit_attn(const std::string& p, const View& x, const View& out, int heads) {
  const int C = x.C, T = x.H * x.W, ch = C / heads;
  SplitView A{splitA_hi_, splitA_lo_};
  emit_gn_split(p + ".norm", x, p + ".norm", false, SPLIT_SAME, A);
  TcWeights wqkv = prep_weights(p + ".qkv.weight", 3 * C, C, 1, "", 0);
  View qkv;
  qkv.p = qkv_; qkv.N = B_; qkv.H = x.H; qkv.W = x.W; qkv.C = 3 * C; qkv.ld = 3 * C;
  emit_tc(p + ".qkv", A, TAPS_1X1, nullptr, wqkv, 3 * C, qkv, P(p + ".qkv.bias", 3 * C), 0, nullptr, 0);
  const float alpha = 1.0f / std::sqrt((float)ch);   // (ch^-1/4)^2
  if (cfg_.new_attention_order) emit_attention_core(p, T, heads, ch, 3 * C, ch, 0, C, 2 * C, alpha);
  else emit_attention_core(p, T, heads, ch, 3 * C, 3 * ch, 0, ch, 2 * ch, alpha);
  View ov;
  ov.p = attO_; ov.N = B_; ov.H = x.H; ov.W = x.W; ov.C = C; ov.ld = C;
  emit_gn_split(p + ".proj_in", ov, "", false, SPLIT_SAME, A);
  TcWeights wp = prep_weights(p + ".proj_out.weight", C, C, 1, "", 0);
  emit_tc(p + ".proj_out", A, TAPS_1X1, nullptr, wp, C, out, P(p + ".proj_out.bias", C), 0, x.p, x.ld);
}

void UNetOpenAI::build_program() {
  const OpenAICfg& c = cfg_;
  const int mc = c.model_channels, R = c.image_size, nrb = c.num_res_blocks, L = c.n_levels;
  DDNM_CHECK(mc % 64 == 0, "model_channels must be a multiple of 64 (tensor-core K blocks)");
  auto attn_at = [&](int ds) {
    for (int i = 0; i < c.n_attn_ds; ++i)
      if (c.attn_ds[i] == ds) return true;
    return false;
  };
  // ---- the module list of UNetModel.__init__ (unet.py:479-611) as data ----
  struct Layer { int kind; int cin, cout; };  // kind: 0 conv, 1 res, 2 res_down, 3 res_up, 4 attn
  struct Block { std::vector<Layer> layers; int res_in, res_out, cout; };
  std::vector<Block> inp, outb;
  std::vector<int> chans, chan_res;
  int ch = c.channel_mult[0] * mc, ds = 1, res = R;
  inp.push_back({{{0, c.in_channels, ch}}, res, res, ch});
  chans.push_back(ch);
  chan_res.push_back(res);
  for (int lv = 0; lv < L; ++lv) {
    for (int i = 0; i < nrb; ++i) {
      Block b{{}, res, res, c.channel_mult[lv] * mc};
      b.layers.push_back({1, ch, c.channel_mult[lv] * mc});
      ch = c.channel_mult[lv] * mc;
      if (attn_at(ds)) b.layers.push_back({4, ch, ch});
      inp.push_back(b);
      chans.push_back(ch);
      chan_res.push_back(res);
    }
    if (lv != L - 1) {
      inp.push_back({{{2, ch, ch}}, res, res / 2, ch});
      res /= 2;
      ds *= 2;
      chans.push_back(ch);
      chan_res.push_back(res);
    }
  }
  const int mid_ch = ch, mid_res = res;
  {
    std::vector<int> cs = chans, rs = chan_res;
    for (int lv = L - 1; lv >= 0; --lv) {
      for (int i = 0; i <= nrb; ++i) {
        const int ich = cs.back();
        DDNM_CHECK(rs.back() == res, "skip resolution mismatch");
        cs.pop_back();
        rs.pop_back();
        Block b{{}, res, res, c.channel_mult[lv] * mc};
        b.layers.push_back({1, ch + ich, c.channel_mult[lv] * mc});
        ch = c.channel_mult[lv] * mc;
        if (attn_at(ds)) b.layers.push_back({4, ch, ch});
        if (lv && i == nrb) {
          b.layers.push_back({3, ch, ch});
          b.res_out = res * 2;
          res *= 2;
          ds /= 2;
        }
        outb.push_back(b);
      }
    }
  }
  const int n_out = (int)outb.size();
  DDNM_CHECK(n_out == (int)inp.size(), "input / output block count mismatch");

  // ---- scratch sizing + per-ResBlock scale|shift rows ----
  size_t split_max = 0, hbuf_max = 0, att_qkv = 0, att_S = 0, att_O = 0;
  int n_gn = 1;
  std::vector<std::string> rb_names;
  std::vector<int> rb_cout;
  auto plan_layers = [&](const std::string& prefix, const std::vector<Layer>& layers, int r) {
    for (size_t j = 0; j < layers.size(); ++j) {
      const Layer& l = layers[j];
      const std::string p = prefix + "." + std::to_string(j);
      if (l.kind == 1 || l.kind == 2 || l.kind == 3) {
        const int ro = l.kind == 2 ? r / 2 : (l.kind == 3 ? r * 2 : r);
        split_max = std::max(split_max, (size_t)B_ * ro * ro * std::max(l.cin, l.cout));
        split_max = std::max(split_max, (size_t)B_ * r * r * l.cin);
        hbuf_max = std::max(hbuf_max, (size_t)B_ * ro * ro * l.cout);
        n_gn += 2;
        rb_names.push_back(p);
        rb_cout.push_back(l.cout);
        r = ro;
      } else if (l.kind == 4) {
        const size_t T = (size_t)r * r, heads = attn_heads(l.cin, prefix.rfind("output_blocks", 0) == 0);
        split_max = std::max(split_max, (size_t)B_ * T * l.cin);
        att_qkv = std::max(att_qkv, (size_t)B_ * T * 3 * l.cin);
        att_S = std::max(att_S, (size_t)B_ * heads * T * T);
        att_O = std::max(att_O, (size_t)B_ * T * l.cin);
        n_gn += 1;
      }
    }
  };
  for (size_t i = 0; i < inp.size(); ++i) plan_layers("input_blocks." + std::to_string(i), inp[i].layers, inp[i].res_in);
  std::vector<Layer> mid = {{1, mid_ch, mid_ch}, {4, mid_ch, mid_ch}, {1, mid_ch, mid_ch}};
  plan_layers("middle_block", mid, mid_res);
  for (int i = 0; i < n_out; ++i) plan_layers("output_blocks." + std::to_string(i), outb[i].layers, outb[i].res_in);
  alloc_common(split_max, hbuf_max);
  alloc_attention(att_qkv, att_S, att_O);

  // ---- timestep embedding (nn.py:103-121, unet.py:472-476,649) and every emb_layers Linear as one matrix (unet.py:188-194) ----
  const int tdim = mc * 4;
  emb_ = (float*)arena_.alloc((size_t)B_ * mc * 4);
  temb0_ = (float*)arena_.alloc((size_t)B_ * tdim * 4);
  temb_ = (float*)arena_.alloc((size_t)B_ * tdim * 4);
  freq_ = (float*)arena_.alloc((size_t)(mc / 2) * 4);
  CUDA_CHECK(cudaMemcpy(freq_, P("__freq", mc / 2), (mc / 2) * 4, cudaMemcpyDeviceToDevice));
  ss_total_ = 0;
  for (size_t i = 0; i < rb_names.size(); ++i) {
    ss_off_[rb_names[i]] = ss_total_;
    ss_total_ += 2 * rb_cout[i];
  }
  embW_all_ = (float*)arena_.alloc((size_t)ss_total_ * tdim * 4);
  embB_all_ = (float*)arena_.alloc((size_t)ss_total_ * 4);
  ss_all_ = (float*)arena_.alloc((size_t)B_ * ss_total_ * 4);
  for (size_t i = 0; i < rb_names.size(); ++i) {
    const int off = ss_off_[rb_names[i]], n2 = 2 * rb_cout[i];
    CUDA_CHECK(cudaMemcpy(embW_all_ + (size_t)off * tdim, P(rb_names[i] + ".emb_layers.1.weight", (long long)n2 * tdim), (size_t)n2 * tdim * 4,
                          cudaMemcpyDeviceToDevice));
    CUDA_CHECK(cudaMemcpy(embB_all_ + off, P(rb_names[i] + ".emb_layers.1.bias", n2), (size_t)n2 * 4, cudaMemcpyDeviceToDevice));
  }
  {
    float *t = t_in_, *emb = emb_, *t0 = temb0_, *t1 = temb_, *fr = freq_, *ss = ss_all_, *W = embW_all_, *Bv = embB_all_;
    const float *w0 = P("time_embed.0.weight", (long long)tdim * mc), *b0 = P("time_embed.0.bias", tdim);
    const float *w1 = P("time_embed.2.weight", (long long)tdim * tdim), *b1 = P("time_embed.2.bias", tdim);
    const int Bn = B_, mcn = mc, tot = ss_total_, ncls = cfg_.num_classes;
    // class-conditional (imagenet_256_cc.yml): emb = time_embed(t) + label_emb(y) (unet.py:651-653) before the blocks' SiLU
    const float* lab = ncls > 0 ? P("label_emb.weight", (long long)ncls * tdim) : nullptr;
    const int* labels = labels_in_;
    add_op("time_embed", "temb", 0, 0, [=](cudaStream_t s) {
      sinusoid(t, Bn, fr, mcn, false, emb, s);               // [cos | sin]
      linear(emb, Bn, mcn, w0, b0, tdim, t0, tdim, 0, 1, s);  // SiLU between the two Linears, applied at the producer
      if (lab) {
        linear(t0, Bn, tdim, w1, b1, tdim, t1, tdim, 0, 0, s);
        add_label_swish(t1, lab, labels, Bn, tdim, ncls, s);  // t1 = SiLU(emb + label_emb[y])
      } else {
        linear(t0, Bn, tdim, w1, b1, tdim, t1, tdim, 0, 1, s);  // emb is only consumed through emb_layers' SiLU
      }
      linear(t1, Bn, tdim, W, Bv, tot, ss, tot, 0, 0, s);     // emb_layers Linear for all blocks at once
    });
  }

  // ---- concat buffers: output block u reads cat[u] = [h (Ch) | skip (Cs)]; skip i lives in cat[n_out-1-i] ----
  std::vector<View> cat(n_out);
  std::vector<int> catCh(n_out);
  {
    int hch = mid_ch;
    for (int u = 0; u < n_out; ++u) {
      const int total = outb[u].layers[0].cin;
      catCh[u] = hch;
      cat[u] = new_view(outb[u].res_in, outb[u].res_in, total);
      DDNM_CHECK(total - hch == chans[n_out - 1 - u], "skip channel bookkeeping");
      hch = outb[u].cout;
    }
  }
  auto hs_slot = [&](int i) {
    const int u = n_out - 1 - i;
    return cat[u].slice(catCh[u], cat[u].C - catCh[u]);
  };
  auto run_layers = [&](const std::string& prefix, const std::vector<Layer>& layers, View cur, const View& final_dst) {
    for (size_t j = 0; j < layers.size(); ++j) {
      const Layer& l = layers[j];
      const std::string p = prefix + "." + std::to_string(j);
      const bool last = j + 1 == layers.size();
      int ro = cur.H;
      if (l.kind == 2) ro = cur.H / 2;
      if (l.kind == 3) ro = cur.H * 2;
      View dst = last ? final_dst : new_view(ro, ro, l.cout);
      DDNM_CHECK(dst.H == ro && dst.C == l.cout, "layer destination shape");
      if (l.kind == 4) emit_attn(p, cur, dst, attn_heads(cur.C, prefix.rfind("output_blocks", 0) == 0));
      else emit_resblock(p, cur, dst, l.kind == 2 ? RES_DOWN : (l.kind == 3 ? RES_UP : RES_PLAIN));
      cur = dst;
    }
    return cur;
  };

  View h = hs_slot(0);
  emit_stem("input_blocks.0.0", h);
  taps_["in.0"] = h;
  for (size_t i = 1; i < inp.size(); ++i) {
    View slot = hs_slot((int)i);
    h = run_layers("input_blocks." + std::to_string(i), inp[i].layers, h, slot);
    taps_["in." + std::to_string(i)] = h;
  }
  h = run_layers("middle_block", mid, h, cat[0].slice(0, catCh[0]));
  taps_["mid"] = h;
  for (int u = 0; u < n_out; ++u) {
    View dst = u + 1 < n_out ? cat[u + 1].slice(0, catCh[u + 1]) : new_view(outb[u].res_out, outb[u].res_out, outb[u].cout);
    h = run_layers("output_blocks." + std::to_string(u), outb[u].layers, cat[u], dst);
    taps_["out." + std::to_string(u)] = h;
  }
  emit_head("out.0", "out.2", h);
}

}  // namespace ddnm

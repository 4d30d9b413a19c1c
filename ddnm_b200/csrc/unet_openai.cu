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

// AttentionBlock.__init__ (unet.py:277-283, 452-453): num_head_channels-wide heads, else a fixed count per block
int UNetOpenAI::attn_heads(int C, bool upsample) const {
  int heads = cfg_.num_heads;
  if (cfg_.num_head_channels > 0) heads = C / cfg_.num_head_channels;
  else if (upsample && cfg_.num_heads_upsample > 0) heads = cfg_.num_heads_upsample;
  DDNM_CHECK(heads >= 1 && C % heads == 0 && (cfg_.num_head_channels <= 0 || C % cfg_.num_head_channels == 0),
             "attention channels " + std::to_string(C) + " do not split into equal heads");
  return heads;
}

void UNetOpenAI::build_program() {
  const OpenAICfg& c = cfg_;
  const int mc = c.model_channels, R = c.image_size, nrb = c.num_res_blocks, L = c.n_levels;
  DDNM_CHECK(mc % 64 == 0, "model_channels must be a multiple of 64 (tensor-core K blocks)");
  const Torso t = plan_torso(R, c.in_channels, mc, c.channel_mult, L, nrb, c.attn_ds, c.n_attn_ds);
  const std::vector<Block>& inp = t.input;
  // ---- the output blocks of UNetModel.__init__ (unet.py:567-611) as data; each pops the skip of one input block ----
  std::vector<Block> outb;
  {
    int ch = t.middle.cout, res = t.middle.res_out, ds = 1 << (L - 1);
    size_t n_skip = inp.size();
    for (int lv = L - 1; lv >= 0; --lv) {
      const int co = c.channel_mult[lv] * mc;
      for (int i = 0; i <= nrb; ++i) {
        const Block& skip = inp[--n_skip];
        DDNM_CHECK(skip.res_out == res, "skip resolution mismatch");
        Block b{{{LAYER_RES, ch + skip.cout, co}}, res, res, co};
        ch = co;
        if (std::find(c.attn_ds, c.attn_ds + c.n_attn_ds, ds) != c.attn_ds + c.n_attn_ds) b.layers.push_back({LAYER_ATTN, ch, ch});
        if (lv && i == nrb) {
          b.layers.push_back({LAYER_RES_UP, ch, ch});
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
  std::vector<EmbProj> projs;
  auto plan_block = [&](const std::string& prefix, const Block& b) {
    int r = b.res_in;
    for (size_t j = 0; j < b.layers.size(); ++j) {
      const Block::Layer& l = b.layers[j];
      const std::string p = prefix + "." + std::to_string(j);
      if (l.kind == LAYER_RES || l.kind == LAYER_RES_DOWN || l.kind == LAYER_RES_UP) {
        const int ro = l.kind == LAYER_RES_DOWN ? r / 2 : (l.kind == LAYER_RES_UP ? r * 2 : r);
        split_max = std::max(split_max, (size_t)B_ * ro * ro * std::max(l.cin, l.cout));
        split_max = std::max(split_max, (size_t)B_ * r * r * l.cin);
        hbuf_max = std::max(hbuf_max, (size_t)B_ * ro * ro * l.cout);
        projs.push_back({p, p + ".emb_layers.1.weight", P(p + ".emb_layers.1.bias", 2 * l.cout), 2 * l.cout});
        r = ro;
      } else if (l.kind == LAYER_ATTN) {
        const size_t T = (size_t)r * r, heads = attn_heads(l.cin, prefix.rfind("output_blocks", 0) == 0);
        split_max = std::max(split_max, (size_t)B_ * T * l.cin);
        att_qkv = std::max(att_qkv, (size_t)B_ * T * 3 * l.cin);
        att_S = std::max(att_S, (size_t)B_ * heads * T * T);
        att_O = std::max(att_O, (size_t)B_ * T * l.cin);
      }
    }
  };
  for (size_t i = 0; i < inp.size(); ++i) plan_block("input_blocks." + std::to_string(i), inp[i]);
  plan_block("middle_block", t.middle);
  for (int i = 0; i < n_out; ++i) plan_block("output_blocks." + std::to_string(i), outb[i]);
  alloc_common(split_max, hbuf_max);
  alloc_attention(att_qkv, att_S, att_O);

  // class-conditional (imagenet_256_cc.yml): emb = time_embed(t) + label_emb(y) (unet.py:651-653) before the blocks' SiLU
  const float* label_emb = c.num_classes > 0 ? P("label_emb.weight", (long long)c.num_classes * mc * 4) : nullptr;
  emit_time_embed("time_embed", "time_embed.0", "time_embed.2", mc, false, label_emb, c.num_classes, projs);

  // ---- concat buffers: output block u reads cat[u] = [h (Ch) | skip (Cs)]; skip i lives in cat[n_out-1-i] ----
  std::vector<View> cat(n_out);
  std::vector<int> catCh(n_out);
  {
    int hch = t.middle.cout;
    for (int u = 0; u < n_out; ++u) {
      const int total = outb[u].layers[0].cin;
      catCh[u] = hch;
      cat[u] = new_view(outb[u].res_in, outb[u].res_in, total);
      DDNM_CHECK(total - hch == inp[n_out - 1 - u].cout, "skip channel bookkeeping");
      hch = outb[u].cout;
    }
  }
  auto hs_slot = [&](int i) {
    const int u = n_out - 1 - i;
    return cat[u].slice(catCh[u], cat[u].C - catCh[u]);
  };
  auto run_block = [&](const std::string& prefix, const Block& b, View cur, const View& final_dst) {
    for (size_t j = 0; j < b.layers.size(); ++j) {
      const Block::Layer& l = b.layers[j];
      const std::string p = prefix + "." + std::to_string(j);
      const bool last = j + 1 == b.layers.size();
      int ro = cur.H;
      if (l.kind == LAYER_RES_DOWN) ro = cur.H / 2;
      if (l.kind == LAYER_RES_UP) ro = cur.H * 2;
      View dst = last ? final_dst : new_view(ro, ro, l.cout);
      DDNM_CHECK(dst.H == ro && dst.C == l.cout, "layer destination shape");
      if (l.kind == LAYER_ATTN) {
        emit_attention_block(p, cur, dst, attn_heads(cur.C, prefix.rfind("output_blocks", 0) == 0), c.new_attention_order, qkv_);
      } else {
        DDNM_CHECK((size_t)(dst.pixels() * l.cout) <= hbuf_elems_, "hbuf too small");
        View hv = view_of(hbuf_, ro, ro, l.cout);
        hv.st = new_stats(l.cout); hv.st_ld = l.cout;   // conv1's epilogue accumulates the sums out_layers.0 needs
        emit_res_block(p, cur, hv, dst, l.kind);
      }
      cur = dst;
    }
    return cur;
  };

  View h = hs_slot(0);
  emit_stem("input_blocks.0.0", h);
  taps_["in.0"] = h;
  for (size_t i = 1; i < inp.size(); ++i) {
    View slot = hs_slot((int)i);
    h = run_block("input_blocks." + std::to_string(i), inp[i], h, slot);
    taps_["in." + std::to_string(i)] = h;
  }
  h = run_block("middle_block", t.middle, h, cat[0].slice(0, catCh[0]));
  taps_["mid"] = h;
  for (int u = 0; u < n_out; ++u) {
    View dst = u + 1 < n_out ? cat[u + 1].slice(0, catCh[u + 1]) : new_view(outb[u].res_out, outb[u].res_out, outb[u].cout);
    h = run_block("output_blocks." + std::to_string(u), outb[u], cat[u], dst);
    taps_["out." + std::to_string(u)] = h;
  }
  emit_head("out.0", "out.2", h);
}

}  // namespace ddnm

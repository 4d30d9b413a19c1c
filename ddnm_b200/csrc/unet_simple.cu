// UNetSimple: launch program for guided_diffusion/models.py::Model (the celeba_hq.yml denoiser).
#include <algorithm>
#include <cmath>

#include "engine.cuh"
#include "kernels.cuh"

namespace ddnm {

UNetSimple::UNetSimple(const SimpleCfg& cfg, int batch)
    : UNetEngine(batch, cfg.in_channels, cfg.out_ch, cfg.resolution, cfg.groups, cfg.eps), cfg_(cfg) {}

// ResnetBlock (models.py:115-134)
void UNetSimple::emit_resblock(const std::string& p, const View& x, const View& out) {
  const int Cin = x.C, Cout = out.C;
  DDNM_CHECK((size_t)(x.pixels() * Cout) <= hbuf_elems_, "hbuf too small");
  SplitView A{splitA_hi_, splitA_lo_}, Bs{splitB_hi_, splitB_lo_};
  View h = view_of(hbuf_, x.H, x.W, Cout);
  h.st = new_stats(Cout); h.st_ld = Cout;   // conv1's epilogue accumulates the sums norm2 needs
  // blocks with a 1x1 shortcut also need the raw split of x: produced by the same pass that normalises it
  emit_gn_split(p + ".norm1", x, p + ".norm1", true, SPLIT_SAME, A, nullptr, 0, Cin != Cout ? &Bs : nullptr);
  TcWeights w1 = prep_weights(p + ".conv1.weight", Cout, Cin, 9, "", 0);
  emit_tc(p + ".conv1", A, TAPS_3X3, nullptr, w1, Cout, h, emb_rows(p), emb_ld_, nullptr, 0);
  emit_gn_split(p + ".norm2", h, p + ".norm2", true, SPLIT_SAME, A);
  if (Cin != Cout) {
    // nin_shortcut (1x1 on the raw block input) rides along as extra K blocks of conv2's GEMM
    TcWeights w2 = prep_weights(p + ".conv2.weight", Cout, Cout, 9, p + ".nin_shortcut.weight", Cin);
    emit_tc(p + ".conv2+nin", A, TAPS_3X3, &Bs, w2, Cout, out, bias_sum(p + ".conv2.bias", p + ".nin_shortcut.bias", Cout), 0,
            nullptr, 0);
  } else {
    TcWeights w2 = prep_weights(p + ".conv2.weight", Cout, Cout, 9, "", 0);
    emit_tc(p + ".conv2", A, TAPS_3X3, nullptr, w2, Cout, out, P(p + ".conv2.bias", Cout), 0, x.p, x.ld);
  }
}

// AttnBlock (models.py:164-189): single head over T = H*W tokens, head dim = C
void UNetSimple::emit_attn(const std::string& p, const View& x, const View& out) {
  const int C = x.C, T = x.H * x.W;
  SplitView A{splitA_hi_, splitA_lo_};
  emit_gn_split(p + ".norm", x, p + ".norm", false, SPLIT_SAME, A);
  // q, k, v 1x1 convolutions as one GEMM with stacked weights [q; k; v]
  TcWeights wqkv;
  wqkv.ktot = C;
  wqkv.hi = (__half*)arena_.alloc((size_t)3 * C * C * sizeof(__half));
  wqkv.lo = (__half*)arena_.alloc((size_t)3 * C * C * sizeof(__half));
  std::vector<float> hb(3 * C);
  const char* nm[3] = {".q", ".k", ".v"};
  for (int i = 0; i < 3; ++i) {
    split_conv_weight(P(p + nm[i] + ".weight", (long long)C * C), C, C, 1, wqkv.hi + (size_t)i * C * C, wqkv.lo + (size_t)i * C * C, C, 0, 0);
    CUDA_CHECK(cudaMemcpy(hb.data() + i * C, P(p + nm[i] + ".bias", C), C * sizeof(float), cudaMemcpyDeviceToHost));
  }
  float* bqkv = dev_copy(hb);
  emit_tc(p + ".qkv", A, TAPS_1X1, nullptr, wqkv, 3 * C, view_of(qkv_, x.H, x.W, 3 * C), bqkv, 0, nullptr, 0);
  // one head of width C; w_ = bmm(q, k) * int(c) ** (-0.5)
  emit_attention_core(p, qkv_, T, 1, C, 3 * C, 0, 0, C, 2 * C, 1.0f / sqrtf((float)C));
  emit_gn_split(p + ".proj_in", view_of(attO_, x.H, x.W, C), "", false, SPLIT_SAME, A);
  TcWeights wp = prep_weights(p + ".proj_out.weight", C, C, 1, "", 0);
  emit_tc(p + ".proj_out", A, TAPS_1X1, nullptr, wp, C, out, P(p + ".proj_out.bias", C), 0, x.p, x.ld);
}

// Downsample (models.py:67-71): pad (0,1,0,1) + 3x3 stride 2
void UNetSimple::emit_downsample(const std::string& p, const View& x, const View& out) {
  SplitView A{splitA_hi_, splitA_lo_};
  emit_gn_split(p + ".s2d", x, "", false, SPLIT_S2D, A);
  TcWeights w = prep_weights(p + ".conv.weight", x.C, x.C, 9, "", 0);
  emit_tc(p + ".conv", A, TAPS_3X3_S2, nullptr, w, x.C, out, P(p + ".conv.bias", x.C), 0, nullptr, 0);
}

// Upsample (models.py:47-52): nearest x2 + 3x3
void UNetSimple::emit_upsample(const std::string& p, const View& x, const View& out) {
  SplitView A{splitA_hi_, splitA_lo_};
  emit_gn_split(p + ".split", x, "", false, SPLIT_SAME, A);
  emit_up2_conv(p + ".conv", A, p + ".conv.weight", x.C, out, P(p + ".conv.bias", x.C), 0);
}

void UNetSimple::build_program() {
  const SimpleCfg& c = cfg_;
  const int L = c.n_levels, R = c.resolution, nrb = c.num_res_blocks;
  DDNM_CHECK(c.ch % 64 == 0, "base channel count must be a multiple of 64 (tensor-core K blocks)");
  auto has_attn = [&](int res) {
    for (int i = 0; i < c.n_attn_res; ++i)
      if (c.attn_res[i] == res) return true;
    return false;
  };
  auto mult = [&](int lv) { return c.ch * c.ch_mult[lv]; };
  auto in_mult = [&](int lv) { return lv == 0 ? c.ch : c.ch * c.ch_mult[lv - 1]; };

  // ---- plan shapes: the hs stack (models.py:311-319) and the up-path concat buffers (:328-335) ----
  struct HS { int res, C; };
  std::vector<HS> hs_shape;
  hs_shape.push_back({R, c.ch});
  {
    int res = R;
    for (int lv = 0; lv < L; ++lv) {
      for (int ib = 0; ib < nrb; ++ib) hs_shape.push_back({res, mult(lv)});
      if (lv != L - 1) {
        res /= 2;
        hs_shape.push_back({res, mult(lv)});
      }
    }
  }
  const int n_up = L * (nrb + 1);
  DDNM_CHECK((int)hs_shape.size() == n_up, "skip stack / up-block count mismatch");
  struct UpB { int lv, ib, res, Ch, Cs, Cout; };
  std::vector<UpB> upb;
  {
    int res = R >> (L - 1);
    int block_in = mult(L - 1);
    for (int lv = L - 1; lv >= 0; --lv) {
      for (int ib = 0; ib <= nrb; ++ib) {
        const int skip = (ib == nrb) ? in_mult(lv) : mult(lv);
        upb.push_back({lv, ib, res, block_in, skip, mult(lv)});
        block_in = mult(lv);
      }
      if (lv != 0) res *= 2;
    }
    for (int u = 0; u < n_up; ++u) {
      const HS& h = hs_shape[n_up - 1 - u];
      DDNM_CHECK(h.res == upb[u].res && h.C == upb[u].Cs, "skip shape does not match its up block");
    }
  }

  // ---- scratch sizing ----
  size_t split_max = 0, hbuf_max = 0, att_tok = 0, att_c = 0, att_T = 0;
  int n_gn = 0;
  std::vector<EmbProj> projs;
  auto plan_conv_in = [&](int res, int Cin, bool up2) {
    split_max = std::max(split_max, (size_t)B_ * res * res * Cin * (up2 ? 4 : 1));
  };
  auto plan_rb = [&](const std::string& p, int res, int Cin, int Cout) {
    plan_conv_in(res, Cin, false);
    plan_conv_in(res, Cout, false);
    hbuf_max = std::max(hbuf_max, (size_t)B_ * res * res * Cout);
    n_gn += 2;
    // conv1.bias joins the projection bias: both are added to every pixel of conv1's output (models.py:119,121)
    projs.push_back({p, p + ".temb_proj.weight", bias_sum(p + ".temb_proj.bias", p + ".conv1.bias", Cout), Cout});
  };
  auto plan_attn = [&](int res, int C) {
    plan_conv_in(res, C, false);
    att_tok = std::max(att_tok, (size_t)res * res);
    att_c = std::max(att_c, (size_t)C);
    att_T = std::max(att_T, (size_t)res * res);
    n_gn += 1;
  };
  {
    int res = R;
    for (int lv = 0; lv < L; ++lv) {
      int cin = in_mult(lv);
      for (int ib = 0; ib < nrb; ++ib) {
        plan_rb("down." + std::to_string(lv) + ".block." + std::to_string(ib), res, cin, mult(lv));
        cin = mult(lv);
        if (has_attn(res)) plan_attn(res, cin);
      }
      if (lv != L - 1) {
        plan_conv_in(res, cin, false);
        res /= 2;
      }
    }
    plan_rb("mid.block_1", res, mult(L - 1), mult(L - 1));
    plan_attn(res, mult(L - 1));
    plan_rb("mid.block_2", res, mult(L - 1), mult(L - 1));
    for (const UpB& u : upb) {
      plan_rb("up." + std::to_string(u.lv) + ".block." + std::to_string(u.ib), u.res, u.Ch + u.Cs, u.Cout);
      if (has_attn(u.res)) plan_attn(u.res, u.Cout);
      if (u.ib == nrb && u.lv != 0) plan_conv_in(u.res, u.Cout, true);
    }
    n_gn += 1;  // norm_out
  }
  alloc_common(split_max, hbuf_max);
  alloc_attention((size_t)B_ * att_tok * 3 * att_c, (size_t)B_ * att_T * att_T, (size_t)B_ * att_tok * att_c);

  // ---- program ----
  emit_time_embed("temb", "temb.dense.0", "temb.dense.1", c.ch, true, nullptr, 0, projs);
  // concat buffers for the up path; hs[i] lives in cat[n_up-1-i].slice(Ch, Cs)
  std::vector<View> cat(n_up);
  for (int u = 0; u < n_up; ++u) cat[u] = new_view(upb[u].res, upb[u].res, upb[u].Ch + upb[u].Cs);
  auto hs_slot = [&](int i) {
    const int u = n_up - 1 - i;
    return cat[u].slice(upb[u].Ch, upb[u].Cs);
  };
  std::vector<View> hs;
  {
    View v0 = hs_slot(0);
    emit_stem("conv_in", v0);
    hs.push_back(v0);
    taps_["conv_in"] = v0;
  }
  int res = R;
  for (int lv = 0; lv < L; ++lv) {
    for (int ib = 0; ib < nrb; ++ib) {
      const std::string p = "down." + std::to_string(lv) + ".block." + std::to_string(ib);
      View slot = hs_slot((int)hs.size());
      if (has_attn(res)) {
        View tmp = new_view(res, res, mult(lv));
        emit_resblock(p, hs.back(), tmp);
        emit_attn("down." + std::to_string(lv) + ".attn." + std::to_string(ib), tmp, slot);
      } else {
        emit_resblock(p, hs.back(), slot);
      }
      hs.push_back(slot);
      taps_["down." + std::to_string(lv) + "." + std::to_string(ib)] = slot;
    }
    if (lv != L - 1) {
      View slot = hs_slot((int)hs.size());
      emit_downsample("down." + std::to_string(lv) + ".downsample", hs.back(), slot);
      hs.push_back(slot);
      taps_["down." + std::to_string(lv) + ".ds"] = slot;
      res /= 2;
    }
  }
  {
    const int C = mult(L - 1);
    View m1 = new_view(res, res, C), m2 = new_view(res, res, C);
    emit_resblock("mid.block_1", hs.back(), m1);
    taps_["mid.block_1"] = m1;
    emit_attn("mid.attn_1", m1, m2);
    taps_["mid.attn_1"] = m2;
    View dst = cat[0].slice(0, upb[0].Ch);
    emit_resblock("mid.block_2", m2, dst);
    taps_["mid.block_2"] = dst;
  }
  View final_h;
  for (int u = 0; u < n_up; ++u) {
    const UpB& ub = upb[u];
    const std::string p = "up." + std::to_string(ub.lv) + ".block." + std::to_string(ub.ib);
    const bool attn = has_attn(ub.res);
    const bool last_in_level = ub.ib == nrb;
    const bool upsample_next = last_in_level && ub.lv != 0;
    View dest;
    if (u == n_up - 1) dest = new_view(ub.res, ub.res, ub.Cout);
    else if (upsample_next) dest = new_view(ub.res, ub.res, ub.Cout);
    else dest = cat[u + 1].slice(0, upb[u + 1].Ch);
    if (attn) {
      View tmp = new_view(ub.res, ub.res, ub.Cout);
      emit_resblock(p, cat[u], tmp);
      emit_attn("up." + std::to_string(ub.lv) + ".attn." + std::to_string(ub.ib), tmp, dest);
    } else {
      emit_resblock(p, cat[u], dest);
    }
    taps_["up." + std::to_string(ub.lv) + "." + std::to_string(ub.ib)] = dest;
    if (upsample_next) {
      View d2 = cat[u + 1].slice(0, upb[u + 1].Ch);
      emit_upsample("up." + std::to_string(ub.lv) + ".upsample", dest, d2);
      taps_["up." + std::to_string(ub.lv) + ".us"] = d2;
    }
    if (u == n_up - 1) final_h = dest;
  }
  emit_head("norm_out", "conv_out", final_h);
}

}  // namespace ddnm

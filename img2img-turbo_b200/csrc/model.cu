// The model graph of the hot path, appended op by op to a Plan (static shapes => one CUDA graph).
//
// Mirrors, layer for layer, what the reference executes through diffusers 0.25.1:
//   VAE encoder  : my_vae_encoder_fwd        src/model.py:14-27   (+ quant_conv, posterior sample)
//   UNet         : UNet2DConditionModel call src/pix2pix_turbo.py:199 (SD-Turbo config, t == 999)
//   DDPM step    : sched.step                src/pix2pix_turbo.py:200 (closed form)
//   VAE decoder  : my_vae_decoder_fwd        src/model.py:30-54   (skip convs, gamma)
// with LoRA folded into the weights, the time embedding folded into conv1 biases, TwinConv blended, and
// NHWC activations so that [B,H,W,C] == [B, HW, C] tokens (no permutes around the transformer blocks).
#include "engine.cuh"

namespace i2it {

static inline int ceil_div_i(long long a, long long b) { return static_cast<int>((a + b - 1) / b); }

#define DISPATCH_T(dt, ...)                                   \
  do {                                                        \
    if ((dt) == DT_BF16) { using T = __nv_bfloat16; __VA_ARGS__; } \
    else { using T = __half; __VA_ARGS__; }                   \
  } while (0)

// ------------------------------------------------------------------------------------------ VAE
Act Engine::vae_resnet(Plan& P, const std::string& p, const Act& x, const Act* skip, const PW* skip_w, bool gn_next) {
  Act h = group_norm(P, x, norm(p + ".norm1"), 1e-6f, true);
  mark_layer(P, p + ".norm1", h);
  ConvOpts o1; o1.gn_out = true;                     // conv1 feeds norm2: its epilogue takes the GroupNorm statistics
  h = conv(P, h, prep(p + ".conv1", {p + ".conv1"}), o1);
  mark_layer(P, p + ".conv1", h);
  h = group_norm(P, h, norm(p + ".norm2"), 1e-6f, true);
  mark_layer(P, p + ".norm2", h);
  ConvOpts o;
  o.gn_out = gn_next;                                // the block's output feeds another GroupNorm (norm1 / attention / conv_norm_out)
  if (has(p + ".conv_shortcut.weight")) {
    // x + conv2(h) with a 1x1 shortcut: the shortcut is one more K-slab of the SAME GEMM (second A tensor), its bias is
    // pre-added to conv2's, so there is no separate launch and no residual read
    I2IT_CHECK(skip == nullptr, "vae_resnet: shortcut and skip source at once");
    PW wsc = prep(p + ".conv_shortcut", {p + ".conv_shortcut"});
    PW w2 = prep(p + ".conv2+sc", {p + ".conv2"}, false, false, p + ".conv_shortcut.bias");
    o.x2 = &x; o.w2 = &wsc;
    Act y = conv(P, h, w2, o);
    mark_layer(P, p + ".conv2", y);
    return y;
  }
  o.res = &x;
  if (skip) { o.x2 = skip; o.w2 = skip_w; }        // decoder: the next block's  + skip_conv(skip*gamma)  folded in here
  Act y = conv(P, h, prep(p + ".conv2", {p + ".conv2"}), o);
  mark_layer(P, p + ".conv2", y);
  return y;
}

Act Engine::vae_attn(Plan& P, const std::string& p, const Act& x) {
  // diffusers Attention (1 head, d = C) with residual; tokens are the NHWC pixels
  const int C = x.C, B = x.N, N = x.H * x.W;
  Act t = group_norm(P, x, norm(p + ".group_norm"), 1e-6f, false);
  mark_layer(P, p + ".group_norm", t);
  Act qk = linear(P, t, prep(p + ".qk", {p + ".to_q", p + ".to_k"}));
  mark_layer(P, p + ".qk", qk);
  Act vt = vt_proj(P, t, B, N, prep(p + ".to_v", {p + ".to_v"}));
  mark_layer(P, p + ".to_v", vt);
  Act a = attention(P, qk.slice(0, C), qk.slice(C, C), vt, B, N, N, 1, C, B);
  a.N = x.N; a.H = x.H; a.W = x.W;
  mark_layer(P, p, a);
  Act y = linear(P, a, prep(p + ".to_out.0", {p + ".to_out.0"}), &x, TG_ACT_NONE, true);   // -> mid_block.resnets.1.norm1
  mark_layer(P, p + ".to_out.0", y);
  return y;
}

Act Engine::build_vae_encoder(Plan& P, const std::string& vp, int B_out, int H, int W, std::vector<Act>& skips,
                              const U8View* u8_in, bool shared_input) {
  const std::string e = vp + "encoder";
  // a variations forward encodes its one input image once: everything up to the moments (and the skips) at batch 1, the
  // posterior sample at batch B_out
  const int B = shared_input ? 1 : B_out;
  // conv_in (3 -> C0, 3x3): the NCHW boundary tensor is packed straight into im2col rows [B,H,W,32] (27 taps*channels + 5
  // zeros), so the conv is ONE K=32 GEMM tap with 64-byte TMA rows instead of nine taps of 16-byte rows
  Act xcol = alloc_act(P, B, H, W, 32);
  {
    const long long total = static_cast<long long>(H) * W * B;
    uint16_t* yp = xcol.p;
    Plan* plan = &P;
    const int dt = dtype, hh = H, ww = W;
    if (u8_in) {
      const U8View src = *u8_in;
      add_op(P, [=](cudaStream_t st) {
        DISPATCH_T(dt, (launch_k(pack_input_im2col_u8_kernel<T>, dim3(ceil_div_i(total, 128)), dim3(128), 0, st, 0,
                           src.get(), src.img, src.w, reinterpret_cast<T*>(yp), hh, ww, total, plan->io.in_mode)));
      }, "pack_im2col_u8", 0, 1.0 * total * (3 + 64));
    } else {
      add_op(P, [=](cudaStream_t st) {
        DISPATCH_T(dt, (launch_k(pack_input_im2col_kernel<T>, dim3(ceil_div_i(total, 128)), dim3(128), 0, st, 0,
                           reinterpret_cast<const T*>(plan->io.x), reinterpret_cast<T*>(yp), hh, ww, total)));
      }, "pack_im2col", 0, 2.0 * total * (3 + 32));
    }
  }
  mark_layer(P, e + ".conv_in.im2col", xcol);
  ConvOpts oin; oin.ksize = 1; oin.gn_out = true;
  Act s = conv(P, xcol, prep_im2col3(e + ".conv_in"), oin);
  mark_layer(P, e + ".conv_in", s);
  xcol = Act();
  for (int i = 0; i < 4; ++i) {
    skips.push_back(s);                                   // model.py:18-20: the INPUT of each down block
    mark(P, "skip" + std::to_string(i), s);
    for (int j = 0; j < 2; ++j)      // the last resnet before a downsampler feeds a conv, not a GroupNorm
      s = vae_resnet(P, e + ".down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), s, nullptr, nullptr,
                     !(j == 1 && i < 3));
    if (i < 3) {
      ConvOpts o; o.stride = 2; o.asym = true; o.gn_out = true;
      const std::string d = e + ".down_blocks." + std::to_string(i) + ".downsamplers.0.conv";
      s = conv(P, s, prep(d, {d}), o);
      mark_layer(P, d, s);
    }
  }
  s = vae_resnet(P, e + ".mid_block.resnets.0", s);
  s = vae_attn(P, e + ".mid_block.attentions.0", s);
  s = vae_resnet(P, e + ".mid_block.resnets.1", s);
  mark(P, "enc_mid", s);
  s = group_norm(P, s, norm(e + ".conv_norm_out"), 1e-6f, true);
  mark_layer(P, e + ".conv_norm_out", s);
  s = conv(P, s, prep(e + ".conv_out", {e + ".conv_out"}), ConvOpts());
  mark_layer(P, e + ".conv_out", s);
  ConvOpts o1; o1.ksize = 1;
  Act mom = conv(P, s, prep(vp + "quant_conv", {vp + "quant_conv"}), o1);
  mark(P, "moments", mom);
  Act z = alloc_act(P, B_out, H / 8, W / 8, 8, 8, true);
  {
    const long long HW = static_cast<long long>(H / 8) * (W / 8), total = HW * B_out, mom_img = shared_input ? 0 : HW;
    const uint16_t* mp = mom.p;
    const int ldm = mom.ld, dt = dtype;
    uint16_t* zp = z.p;
    Plan* plan = &P;
    const float sf = cfg.scaling_factor;
    P.keep.push_back(mom.hold);
    add_op(P, [=](cudaStream_t st) {
      DISPATCH_T(dt, (launch_k(latent_sample_kernel<T>, dim3(ceil_div_i(total, 128)), dim3(128), 0, st, 0,
                         reinterpret_cast<const T*>(mp), ldm, mom_img, reinterpret_cast<const T*>(plan->io.eps),
                         reinterpret_cast<const T*>(plan->io.noise), plan->io.r, sf, reinterpret_cast<T*>(zp), HW, total)));
    });
  }
  mark(P, "latent", z);
  return z;
}

void Engine::build_vae_decoder(Plan& P, const std::string& vp, const Act& dec_in, std::vector<Act>& skips) {
  const std::string d = vp + "decoder";
  ConvOpts o1; o1.ksize = 1;
  Act s = conv(P, dec_in, prep(vp + "post_quant_conv", {vp + "post_quant_conv"}), o1);
  mark_layer(P, vp + "post_quant_conv", s);
  { ConvOpts oc; oc.gn_out = true; s = conv(P, s, prep(d + ".conv_in", {d + ".conv_in"}), oc); }
  mark_layer(P, d + ".conv_in", s);
  // `sample = sample + skip_conv_i(skip_i * gamma)` (src/model.py:40-42) is folded into whichever conv PRODUCES `sample`
  // for up-block i: mid_block.resnets.1.conv2 for i = 0, the previous block's upsampler conv for i >= 1.  gamma is folded
  // into the bias-free 1x1 weights.
  auto skip_w = [&](int i) { const std::string sk = d + ".skip_conv_" + std::to_string(i + 1); return prep(sk, {sk}, false, true); };
  // the skip that skip_conv_(k+1) reads.  A variations forward encoded one image: its batch-1 skip is replicated to the
  // decoder's batch right before the block that reads it, so a batch-n copy lives for one layer, not across the UNet
  auto skip_in = [&](int i, int k) {
    if (skips[i].N == dec_in.N) return skips[i];
    Act rep = replicate_image(P, skips[i], dec_in.N);
    mark_layer(P, d + ".skip_conv_" + std::to_string(k + 1) + ".replica", rep);
    return rep;
  };
  s = vae_resnet(P, d + ".mid_block.resnets.0", s);
  s = vae_attn(P, d + ".mid_block.attentions.0", s);
  {
    PW w0 = skip_w(0);
    const Act sk = skip_in(3, 0);
    skips[3] = Act();
    s = vae_resnet(P, d + ".mid_block.resnets.1", s, &sk, &w0);
  }
  mark(P, "dec_mid", s);
  for (int i = 0; i < 4; ++i) {
    for (int j = 0; j < 3; ++j)      // resnets.2 feeds the upsampler conv (i < 3) or conv_norm_out (i == 3)
      s = vae_resnet(P, d + ".up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), s, nullptr, nullptr,
                     !(j == 2 && i < 3));
    if (i < 3) {
      // Upsample2D: nearest-2x + conv3x3, as four parity-phase 2x2 convs on the low-res tensor (2.25x fewer FLOPs, the
      // upsampled tensor never exists); the next block's skip conv rides along as a second source at output resolution
      const std::string u = d + ".up_blocks." + std::to_string(i) + ".upsamplers.0.conv";
      PW wn = skip_w(i + 1);
      const Act sk = skip_in(2 - i, i + 1);
      skips[2 - i] = Act();
      s = conv_up2x(P, s, prep_subpixel(u), &sk, &wn, true);
      mark_layer(P, u, s);
    }
    mark(P, "dec_up" + std::to_string(i), s);
  }
  s = group_norm(P, s, norm(d + ".conv_norm_out"), 1e-6f, true);
  mark_layer(P, d + ".conv_norm_out", s);
  if (cfg.keep_stages) {   // tests compare the PRE-clamp image (BASELINE.md section 5): one extra launch, test mode only
    Act pre = conv(P, s, prep(d + ".conv_out", {d + ".conv_out"}), ConvOpts());
    mark(P, "pre_clamp", pre);
  }
  ConvOpts oo; oo.act = TG_ACT_CLAMP1; oo.to_io_out_nchw = true;
  conv(P, s, prep(d + ".conv_out", {d + ".conv_out"}), oo);
}

// ------------------------------------------------------------------------------------------ UNet
Act Engine::unet_resnet(Plan& P, const std::string& p, const Act& x, bool gn_next, const Act* out) {
  Act h = group_norm(P, x, norm(p + ".norm1"), 1e-5f, true);
  mark_layer(P, p + ".norm1", h);
  // t == 999 always: time_emb_proj(silu(emb)) is a per-channel constant -> part of conv1's bias
  ConvOpts o1; o1.gn_out = true;
  h = conv(P, h, prep(p + ".conv1", {p + ".conv1"}, false, false, temb_bias(p)), o1);
  mark_layer(P, p + ".conv1", h);
  h = group_norm(P, h, norm(p + ".norm2"), 1e-5f, true);
  mark_layer(P, p + ".norm2", h);
  ConvOpts o;
  o.gn_out = gn_next;
  o.out = out;
  if (has(p + ".conv_shortcut.weight")) {
    PW wsc = prep(p + ".conv_shortcut", {p + ".conv_shortcut"});
    PW w2 = prep(p + ".conv2+sc", {p + ".conv2"}, false, false, p + ".conv_shortcut.bias");
    o.x2 = &x; o.w2 = &wsc;
    Act y = conv(P, h, w2, o);
    mark_layer(P, p + ".conv2", y);
    return y;
  }
  o.res = &x;
  Act y = conv(P, h, prep(p + ".conv2", {p + ".conv2"}), o);
  mark_layer(P, p + ".conv2", y);
  return y;
}

Act Engine::unet_xformer(Plan& P, const std::string& p, const Act& x, int heads, int text_batch, bool gn_next, const Act* out) {
  const int C = x.C, B = x.N, N = x.H * x.W, d = C / heads;
  const std::string b = p + ".transformer_blocks.0";
  Act t = group_norm(P, x, norm(p + ".norm"), 1e-6f, false);
  mark_layer(P, p + ".norm", t);
  t = linear(P, t, prep(p + ".proj_in", {p + ".proj_in"}));
  mark_layer(P, p + ".proj_in", t);
  {  // self-attention
    Act n = layer_norm(P, t, norm(b + ".norm1"));
    mark_layer(P, b + ".norm1", n);
    Act qk = linear(P, n, prep(b + ".attn1.qk", {b + ".attn1.to_q", b + ".attn1.to_k"}));
    mark_layer(P, b + ".attn1.qk", qk);
    Act vt = vt_proj(P, n, B, N, prep(b + ".attn1.to_v", {b + ".attn1.to_v"}));
    mark_layer(P, b + ".attn1.to_v", vt);
    Act a = attention(P, qk.slice(0, C), qk.slice(C, C), vt, B, N, N, heads, d, B);
    a.N = x.N; a.H = x.H; a.W = x.W;
    mark_layer(P, b + ".attn1", a);
    t = linear(P, a, prep(b + ".attn1.to_out.0", {b + ".attn1.to_out.0"}), &t);
    mark_layer(P, b + ".attn1.to_out.0", t);
  }
  {  // cross-attention over the 77 text tokens
    Act n = layer_norm(P, t, norm(b + ".norm2"));
    mark_layer(P, b + ".norm2", n);
    Act q = linear(P, n, prep(b + ".attn2.to_q", {b + ".attn2.to_q"}));
    mark_layer(P, b + ".attn2.to_q", q);
    Act k2, v2t;
    if (text_kv_) {                                   // computed once per prompt by i2it_set_text
      auto it = text_kv_->kv.find(b);
      I2IT_CHECK(it != text_kv_->kv.end(), "no cached text K/V for " + b);
      k2 = it->second.first; v2t = it->second.second;
    } else {
      k2 = linear(P, text_, prep(b + ".attn2.to_k", {b + ".attn2.to_k"}));
      v2t = vt_proj(P, text_, text_batch, 77, prep(b + ".attn2.to_v", {b + ".attn2.to_v"}));
    }
    mark_layer(P, b + ".attn2.to_k", k2);            // inline or cached: the audit checks both against this block's weights
    mark_layer(P, b + ".attn2.to_v", v2t);
    Act a = attention(P, q, k2, v2t, B, N, 77, heads, d, text_batch);
    a.N = x.N; a.H = x.H; a.W = x.W;
    mark_layer(P, b + ".attn2", a);
    t = linear(P, a, prep(b + ".attn2.to_out.0", {b + ".attn2.to_out.0"}), &t);
    mark_layer(P, b + ".attn2.to_out.0", t);
  }
  {  // GEGLU feed-forward: h * gelu(g) fused into the first projection's epilogue (weight rows interleaved)
    Act n = layer_norm(P, t, norm(b + ".norm3"));
    mark_layer(P, b + ".norm3", n);
    Act g = linear(P, n, prep(b + ".ff.net.0.proj", {b + ".ff.net.0.proj"}, true), nullptr, TG_ACT_GEGLU);
    mark_layer(P, b + ".ff.net.0.proj", g);
    t = linear(P, g, prep(b + ".ff.net.2", {b + ".ff.net.2"}), &t);
    mark_layer(P, b + ".ff.net.2", t);
  }
  Act y = linear(P, t, prep(p + ".proj_out", {p + ".proj_out"}), &x, TG_ACT_NONE, gn_next, out);
  mark_layer(P, p + ".proj_out", y);
  return y;
}

// every transformer block of the UNet, in execution-independent fixed order (the cross-attention K/V^T cache is keyed by it)
std::vector<std::string> Engine::xformer_prefixes() const {
  std::vector<std::string> v;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 2; ++j) v.push_back("unet.down_blocks." + std::to_string(i) + ".attentions." + std::to_string(j));
  v.push_back("unet.mid_block.attentions.0");
  for (int i = 1; i < 4; ++i)
    for (int j = 0; j < 3; ++j) v.push_back("unet.up_blocks." + std::to_string(i) + ".attentions." + std::to_string(j));
  return v;
}

// K = to_k(text), V^T = (to_v(text))^T of every cross-attention layer: 2 launches per block, run only when the prompt changes
void Engine::build_text_kv(TextKV& T) {
  Plan& P = T.plan;
  T.text = alloc_act(P, T.text_batch, 1, 77, cfg.cross_dim);
  {
    uint16_t* tp = T.text.p;
    const size_t bytes = static_cast<size_t>(T.text_batch) * 77 * cfg.cross_dim * 2;
    Plan* plan = &P;
    add_op(P, [=](cudaStream_t st) {
      cudaMemcpyAsync(tp, plan->io.text, bytes, cudaMemcpyDeviceToDevice, st);
      g_pdl.prev_is_kernel = false;
    });
  }
  for (const auto& p : xformer_prefixes()) {
    const std::string b = p + ".transformer_blocks.0";
    Act k2 = linear(P, T.text, prep(b + ".attn2.to_k", {b + ".attn2.to_k"}));
    Act v2t = vt_proj(P, T.text, T.text_batch, 77, prep(b + ".attn2.to_v", {b + ".attn2.to_v"}));
    T.kv[b] = std::make_pair(k2, v2t);
  }
  flush_prep();
  I2IT_CUDA(cudaDeviceSynchronize());
}

Act Engine::build_unet(Plan& P, const Act& z, int text_batch, bool text_cached) {
  const std::string u = "unet";
  const int* ch = cfg.unet_channels;
  const int* heads = cfg.unet_heads;
  text_kv_ = nullptr;
  if (text_cached) {
    auto it = textkv_.find(text_batch);
    I2IT_CHECK(it != textkv_.end(), "text_emb == NULL but i2it_set_text has not been called for this text_batch since the last "
                                    "i2it_finalize_weights");
    text_kv_ = it->second.get();
  } else {
    // stage the text embedding: its projections are TMA operands, whose maps need a fixed base address
    text_ = alloc_act(P, text_batch, 1, 77, cfg.cross_dim);
    P.keep.push_back(text_.hold);
    uint16_t* tp = text_.p;
    const size_t bytes = static_cast<size_t>(text_batch) * 77 * cfg.cross_dim * 2;
    Plan* plan = &P;
    add_op(P, [=](cudaStream_t st) {
      cudaMemcpyAsync(tp, plan->io.text, bytes, cudaMemcpyDeviceToDevice, st);
      g_pdl.prev_is_kernel = false;   // a copy node: the next kernel takes a full dependency
    });
  }
  // torch.cat([h, skip], dim=1) without copies: every skip connection is produced straight into the upper channel slice of
  // the concat buffer its up-block resnet will read, and the running `h` into the lower slice (I2IT_NO_CATFUSE=1: copy kernels).
  // Consumer q (pop order, 3 per up block) needs sC(q) channels of `h` in front of the skip.
  struct SkipSlot { Act cat, skip; int sC; };
  std::vector<SkipSlot> res;
  const int rch[4] = {ch[3], ch[2], ch[1], ch[0]};
  const int total_pushes = 12;                       // conv_in + 4 x 2 block outputs + 3 downsamplers
  int pushes = 0;
  const bool fuse = use_catfuse;
  auto make_slot = [&](int N, int H, int W, int skipC) {
    const int q = total_pushes - 1 - pushes++, i = q / 3, j = q % 3;
    SkipSlot t;
    t.sC = (j == 0) ? (i == 0 ? ch[3] : rch[i - 1]) : rch[i];
    if (fuse) { t.cat = alloc_act(P, N, H, W, t.sC + skipC); t.skip = t.cat.slice(t.sC, skipC); }
    return t;
  };
  auto push = [&](SkipSlot& t, const Act& produced) { t.skip = produced; res.push_back(t); };   // keeps the producer's GN partials
  auto h_target = [&]() { return res.back().cat.slice(0, res.back().sC); };                      // where the next `h` goes

  Act s;
  {
    SkipSlot t = make_slot(z.N, z.H, z.W, ch[0]);
    ConvOpts oc; oc.gn_out = true;
    if (fuse) oc.out = &t.skip;
    if (has(u + ".conv_in.conv_in_pretrained.weight"))
      s = conv(P, z, prep_twin(u + ".conv_in.conv_in_pretrained", u + ".conv_in.conv_in_curr"), oc);
    else
      s = conv(P, z, prep(u + ".conv_in", {u + ".conv_in"}), oc);
    mark_layer(P, u + ".conv_in", s);
    push(t, s);
  }
  for (int i = 0; i < 4; ++i) {
    const std::string blk = u + ".down_blocks." + std::to_string(i);
    for (int j = 0; j < 2; ++j) {
      // who consumes the output decides whether the producing GEMM takes GroupNorm statistics: the transformer's GroupNorm
      // (i < 3), the next resnet's norm1 (j == 0, or the mid block after the last down block) — not the downsampler conv
      SkipSlot t = make_slot(s.N, s.H, s.W, ch[i]);
      const Act* ov = fuse ? &t.skip : nullptr;
      s = unet_resnet(P, blk + ".resnets." + std::to_string(j), s, true, i < 3 ? nullptr : ov);
      if (i < 3) s = unet_xformer(P, blk + ".attentions." + std::to_string(j), s, heads[i], text_batch, j == 0, ov);
      push(t, s);
    }
    if (i < 3) {
      SkipSlot t = make_slot(s.N, (s.H + 1) / 2, (s.W + 1) / 2, ch[i]);
      ConvOpts o; o.stride = 2; o.gn_out = true;
      if (fuse) o.out = &t.skip;
      s = conv(P, s, prep(blk + ".downsamplers.0.conv", {blk + ".downsamplers.0.conv"}), o);
      mark_layer(P, blk + ".downsamplers.0.conv", s);
      push(t, s);
    }
  }
  I2IT_CHECK(pushes == total_pushes, "unet: unexpected number of skip connections");
  s = unet_resnet(P, u + ".mid_block.resnets.0", s, true);
  s = unet_xformer(P, u + ".mid_block.attentions.0", s, heads[3], text_batch, true);
  {
    Act tgt;
    if (fuse) tgt = h_target();
    s = unet_resnet(P, u + ".mid_block.resnets.1", s, false, fuse ? &tgt : nullptr);   // -> concat (GroupNorm over the concatenation)
  }
  mark(P, "unet_mid", s);
  for (int i = 0; i < 4; ++i) {
    const std::string blk = u + ".up_blocks." + std::to_string(i);
    const int hcount = heads[3 - i];
    for (int j = 0; j < 3; ++j) {
      SkipSlot t = res.back();
      res.pop_back();
      Act cat;
      if (fuse) {
        I2IT_CHECK(s.C == t.sC && s.p == t.cat.p && s.H == t.cat.H && s.W == t.cat.W, "unet: concat slot mismatch");
        cat = t.cat;                                                   // both halves were written in place
      } else {
        cat = alloc_act(P, s.N, s.H, s.W, s.C + t.skip.C);             // torch.cat([h, skip], dim=1)
        copy_channels(P, s, cat.slice(0, s.C));
        copy_channels(P, t.skip, cat.slice(s.C, t.skip.C));
      }
      t = SkipSlot();
      mark_layer(P, blk + ".resnets." + std::to_string(j) + ".concat", cat);   // torch.cat([h, skip], dim=1)
      const bool last = (i == 3 && j == 2);                            // the very last block feeds conv_norm_out directly
      // the block's output is the next concat's `h` unless an upsampler (j == 2, i < 3) or conv_norm_out (last) follows
      Act tgt;
      const bool to_cat = fuse && j < 2;
      if (to_cat) tgt = h_target();
      const Act* ov = to_cat ? &tgt : nullptr;
      s = unet_resnet(P, blk + ".resnets." + std::to_string(j), cat, i > 0, i > 0 ? nullptr : ov);
      if (i > 0) s = unet_xformer(P, blk + ".attentions." + std::to_string(j), s, hcount, text_batch, last, ov);
    }
    if (i < 3) {
      // Upsample2D: 2x nearest, or — when the latent is not a multiple of 8 (UNet2DConditionModel.forward: forward_upsample_size)
      // — nearest to the spatial size of the next skip connection (e.g. 14 -> 27 columns for a 560x840 image)
      const SkipSlot& nxt = res.back();
      s = upsample_to(P, s, nxt.skip.H, nxt.skip.W);
      mark_layer(P, blk + ".upsamplers.0.nearest", s);
      Act tgt;
      ConvOpts oc;
      if (fuse) { tgt = h_target(); oc.out = &tgt; }
      s = conv(P, s, prep(blk + ".upsamplers.0.conv", {blk + ".upsamplers.0.conv"}), oc);
      mark_layer(P, blk + ".upsamplers.0.conv", s);
    }
  }
  I2IT_CHECK(res.empty(), "unet: residual stack not consumed");
  (void)ch;
  s = group_norm(P, s, norm(u + ".conv_norm_out"), 1e-5f, true);
  mark_layer(P, u + ".conv_norm_out", s);
  s = conv(P, s, prep(u + ".conv_out", {u + ".conv_out"}), ConvOpts());
  text_ = Act();
  text_kv_ = nullptr;
  return s;
}

// ------------------------------------------------------------------------------------------ whole path
void Engine::resample_fixed(Plan& P, const U8View& src, int B, int inH, int inW, int rsH, int rsW, int y0, int x0, int H, int W,
                            const U8View& dst) {
  const bool need_h = inW != rsW, need_v = inH != rsH;
  I2IT_CHECK(need_h || need_v, "resample_fixed: the size does not change");
  I2IT_CHECK(y0 >= 0 && x0 >= 0 && y0 + H <= rsH && x0 + W <= rsW, "resample_fixed: window outside the resized image");
  // a caller's images are offsets from the pointer each launch reads (one graph per IO set); a plan buffer's are addresses
  auto addr = [](const U8View& v) { return v.slot ? 0 : reinterpret_cast<uintptr_t>(v.get()); };
  RsImage m{addr(src), addr(dst), 0, inH, inW, rsH, rsW, y0, x0, H, W};
  if (need_h && need_v) {
    const std::pair<int, int> rr = rs_rows(m, rs_tables_);
    auto mid = alloc_raw(P, static_cast<size_t>(B) * (rr.second - rr.first) * W * 3);
    P.keep.push_back(mid);
    m.mid = reinterpret_cast<uintptr_t>(mid.get());
  }
  std::vector<RsPass> d, v;
  std::vector<int> tab;
  double bytes[2] = {0, 0};
  rs_add_images(m, B, src.img, dst.img, /*skip_identity=*/true, rs_tables_, d, v, tab, bytes);
  const size_t nh = d.size();
  d.insert(d.end(), v.begin(), v.end());
  // [descriptors | tables] on the device, written once here: a fresh block, never recycled by later ops of the plan
  const size_t dbytes = d.size() * sizeof(RsPass);
  char* dev = static_cast<char*>(P.pool.get_fresh(dbytes + tab.size() * sizeof(int)));
  I2IT_CUDA(cudaMemcpy(dev, d.data(), dbytes, cudaMemcpyHostToDevice));
  I2IT_CUDA(cudaMemcpy(dev + dbytes, tab.data(), tab.size() * sizeof(int), cudaMemcpyHostToDevice));
  const RsPass* dd = reinterpret_cast<const RsPass*>(dev);
  const int* dtab = reinterpret_cast<const int*>(dev + dbytes);
  const std::string geo = std::to_string(B) + "x" + std::to_string(inH) + "x" + std::to_string(inW) + "->" + std::to_string(rsH) +
                          "x" + std::to_string(rsW) + "@" + std::to_string(y0) + "," + std::to_string(x0) + ":" +
                          std::to_string(H) + "x" + std::to_string(W);
  // one block per output row: the rows are known here, and no block strides or exits early
  if (need_h) resample_pass(P, false, dd, B, dtab, src, need_v ? U8View() : dst, B * d[0].rows, "resample_h", bytes[0], geo);
  if (need_v) resample_pass(P, true, dd + nh, B, dtab, need_h ? U8View() : src, dst, B * H, "resample_v", bytes[1], geo);
}

void Engine::resample_pass(Plan& P, bool vertical, const RsPass* d, int n, const int* tab, const U8View& src, const U8View& dst,
                           int grid, const char* kind, double bytes, const std::string& shape) {
  add_op(P, [=](cudaStream_t st) {
    auto base = [](const U8View& v) { return v.slot ? reinterpret_cast<uintptr_t>(v.get()) : uintptr_t(0); };
    launch_k(vertical ? resample_v_kernel : resample_h_kernel, dim3(grid), dim3(256), 0, st, 0, d, n, tab, base(src), base(dst));
  }, kind, 0, bytes, shape);
}

void Engine::resample_ragged(Plan& P, int B, int first, int slot) {
  const RsPass* d = reinterpret_cast<const RsPass*>(P.rg.dev) + first;
  const int* tab = P.rg.tab();
  // the grid depends on the device alone: its blocks stride over whatever rows the call has, so a captured launch serves any mix
  const int grid = num_sms * 8;
  const std::string shape = std::to_string(B) + " images, max_side " + std::to_string(P.rg.max_side);
  P.rg.ops[slot] = P.ops.size();
  resample_pass(P, false, d, B, tab, U8View(), U8View(), grid, "resample_h_ragged", 0, shape);
  P.rg.ops[slot + 1] = P.ops.size();
  resample_pass(P, true, d + B, B, tab, U8View(), U8View(), grid, "resample_v_ragged", 0, shape);
}

void Engine::resize_ragged_op(Plan& P, const void* const* x, const int* hw_in, void* const* out, const int* hw_out, int n,
                              int max_side) {
  I2IT_CHECK(n >= 1, "i2it_op_resize_u8_ragged: n must be >= 1");
  I2IT_CHECK(max_side > 0, "i2it_op_resize_u8_ragged: max_side must be positive");
  I2IT_CHECK(x && out && hw_in && hw_out, "i2it_op_resize_u8_ragged: null array");
  std::vector<RsImage> im(n);
  std::vector<size_t> mid_off(n);
  size_t mid_bytes = 0;
  for (int i = 0; i < n; ++i) {
    const std::string at = " (image " + std::to_string(i) + ")";
    const int H = hw_in[2 * i], W = hw_in[2 * i + 1], H2 = hw_out[2 * i], W2 = hw_out[2 * i + 1];
    I2IT_CHECK(H > 0 && W > 0 && H2 > 0 && W2 > 0, "i2it_op_resize_u8_ragged: sizes must be positive" + at);
    I2IT_CHECK(H <= max_side && W <= max_side && H2 <= max_side && W2 <= max_side,
               "i2it_op_resize_u8_ragged: a dimension exceeds max_side (" + std::to_string(max_side) + ")" + at);
    I2IT_CHECK(x[i] && out[i], "i2it_op_resize_u8_ragged: null image pointer" + at);
    im[i] = RsImage{reinterpret_cast<uintptr_t>(x[i]), reinterpret_cast<uintptr_t>(out[i]), 0, H, W, H2, W2, 0, 0, H2, W2};
    const std::pair<int, int> rr = rs_rows(im[i], rs_tables_);
    mid_off[i] = mid_bytes;
    mid_bytes += static_cast<size_t>(rr.second - rr.first) * W2 * 3;
  }
  auto mid = alloc_raw(P, mid_bytes);
  P.keep.push_back(mid);
  RsCall c;
  std::vector<RsPass> v;
  for (int i = 0; i < n; ++i) {
    im[i].mid = reinterpret_cast<uintptr_t>(mid.get()) + mid_off[i];
    rs_add_images(im[i], 1, 0, 0, /*skip_identity=*/false, rs_tables_, c.d, v, c.tab, c.bytes);
  }
  c.d.insert(c.d.end(), v.begin(), v.end());
  const size_t dbytes = c.d.size() * sizeof(RsPass);
  P.rg.max_side = max_side;
  P.rg.descs = 2 * n;
  P.rg.dev_bytes = dbytes + c.tab.size() * sizeof(int);
  P.rg.dev = static_cast<char*>(P.pool.get_fresh(P.rg.dev_bytes));
  I2IT_CUDA(cudaMemcpy(P.rg.dev, c.d.data(), dbytes, cudaMemcpyHostToDevice));
  I2IT_CUDA(cudaMemcpy(P.rg.dev + dbytes, c.tab.data(), c.tab.size() * sizeof(int), cudaMemcpyHostToDevice));
  resample_ragged(P, n, 0, 0);
  P.meta[P.rg.ops[0]].bytes = c.bytes[0];
  P.meta[P.rg.ops[1]].bytes = c.bytes[1];
}

void rs_check_geometry(const i2it_resize_desc& d, int H, int W, const std::string& at) {
  I2IT_CHECK(d.in_H > 0 && d.in_W > 0 && d.resize_H > 0 && d.resize_W > 0 && d.out_H > 0 && d.out_W > 0,
             "resize geometry: sizes must be positive" + at);
  I2IT_CHECK(d.crop_y >= 0 && d.crop_x >= 0 && d.crop_y + H <= d.resize_H && d.crop_x + W <= d.resize_W,
             "resize geometry: the H x W crop window lies outside the resized image" + at);
}

void rs_check_ragged(const i2it_resize_desc* g, int n, int H, int W, int max_side) {
  I2IT_CHECK(max_side > 0, "ragged forward: max_side must be positive");
  I2IT_CHECK(g != nullptr && n > 0, "ragged forward: no geometry");
  for (int i = 0; i < n; ++i) {
    const i2it_resize_desc& d = g[i];
    const std::string at = " (image " + std::to_string(i) + ")";
    rs_check_geometry(d, H, W, at);
    I2IT_CHECK(d.in_H <= max_side && d.in_W <= max_side && d.resize_H <= max_side && d.resize_W <= max_side &&
               d.out_H <= max_side && d.out_W <= max_side,
               "resize geometry: a dimension exceeds max_side (" + std::to_string(max_side) + ")" + at);
  }
}

static uintptr_t rs_at(const void* p, long long off = 0) { return p ? reinterpret_cast<uintptr_t>(p) + off : 0; }

RsCall rs_forward_call(const i2it_resize_desc* g, int n, int H, int W, int max_side, RsTableCache& cache, const void* const* x,
                       void* const* out, const RaggedBufs* rg) {
  RsCall c;
  std::vector<RsPass> d[4];
  const long long net = 3ll * H * W;
  for (int i = 0; i < n; ++i) {
    const i2it_resize_desc& e = g[i];
    const RsImage in{x ? rs_at(x[i]) : 0, rg ? rs_at(rg->in_net, i * net) : 0, rg ? rs_at(rg->in_mid, i * 3ll * max_side * W) : 0,
                     e.in_H, e.in_W, e.resize_H, e.resize_W, e.crop_y, e.crop_x, H, W};
    const RsImage o{rg ? rs_at(rg->out_net, i * net) : 0, out ? rs_at(out[i]) : 0, rg ? rs_at(rg->out_mid, i * 3ll * H * max_side) : 0,
                    H, W, e.out_H, e.out_W, 0, 0, e.out_H, e.out_W};
    rs_add_images(in, 1, 0, 0, /*skip_identity=*/false, cache, d[0], d[1], c.tab, c.bytes);
    rs_add_images(o, 1, 0, 0, /*skip_identity=*/false, cache, d[2], d[3], c.tab, c.bytes + 2);
  }
  for (auto& v : d) c.d.insert(c.d.end(), v.begin(), v.end());
  I2IT_CHECK(static_cast<long long>(c.tab.size()) <= rs_forward_bound(n, H, W, max_side),
             "ragged resize: the call's tables exceed the plan's bound");
  return c;
}

Plan* Engine::plan_for(int B, int H, int W, int direction, int text_batch, bool text_cached, int io_mode,
                       const i2it_resize_desc* g, bool evict, int max_side) {
  std::vector<int> key{B, H, W, direction, text_batch, text_cached ? 1 : 0, io_mode};
  if (g) key.insert(key.end(), {g->in_H, g->in_W, g->resize_H, g->resize_W, g->crop_y, g->crop_x, g->out_H, g->out_W});
  const bool ragged = (io_mode & IO_RAGGED) != 0;
  if (ragged) key.push_back(max_side);
  auto it = plans_.find(key);
  if (it != plans_.end()) return it->second.get();
  I2IT_CHECK(finalized_, "i2it_finalize_weights must be called before a forward");
  std::string vp = "vae.";
  if (cfg.model_kind == I2IT_CYCLEGAN && direction == I2IT_B2A) vp = "vae_b2a.";
  const bool mixed = direction == DIR_MIXED;     // Engine::forward has run check_mixed
  std::unique_ptr<Plan> up(new Plan());
  Plan& P = *up;
  P.key = key;
  // a mixed plan builds the VAE from the vae. weights paired with their vae_b2a. twins (prep / norm do the pairing while
  // mixed_dir_ is set); its launches read the image's direction from P.dir, which every call rewrites before the first launch
  struct MixedBuild {
    const int*& slot;
    ~MixedBuild() { slot = nullptr; }
  } mixed_build{mixed_dir_};
  if (mixed) {
    P.dir = static_cast<int*>(P.pool.get_fresh(static_cast<size_t>(B) * sizeof(int)));
    I2IT_CUDA(cudaMemset(P.dir, 0, static_cast<size_t>(B) * sizeof(int)));
    mixed_dir_ = P.dir;
  }
  P.pool.arena = &arena_;      // transient buffers alias those of the handle's other forward plans
  // a build that throws must not leave engine members pointing into the dying plan's pool (text_ holds a pool block):
  // declared after `up`, so it runs before the plan is destroyed
  struct BuildGuard {
    Engine* e; bool ok = false;
    ~BuildGuard() { if (!ok) { e->text_ = Act(); e->text_kv_ = nullptr; } }
  } guard{this};
  std::vector<Act> skips;
  const bool shared_input = (io_mode & IO_SHARED_IN) != 0;
  const int B_in = shared_input ? 1 : B;      // images the input side (resize_in, packing, VAE encoder) runs on
  if (io_mode & IO_U8_OUT) {
    // allocated FIRST and held for the plan's lifetime: pool liveness follows build order, and the last conv writes here
    auto tmp = alloc_raw(P, static_cast<size_t>(B) * 3 * H * W * 2);
    P.keep.push_back(tmp);
    P.u8_out_tmp = tmp.get();
  }
  // what the first kernel reads: the caller's [B, H, W, 3] image, or with a geometry the H x W network window of its resize
  U8View net_in;
  net_in.slot = &P.io.x_u8; net_in.img = 3ll * H * W; net_in.w = W;
  if (ragged) {
    // capacity buffers: every call's images fit them (rs_check_ragged), so the plan and its graph serve any mix of sizes
    I2IT_CHECK(max_side > 0, "ragged plan: max_side must be positive");
    P.rg.max_side = max_side;
    P.rg.descs = 4 * B;
    P.rg.dev_bytes = 4 * static_cast<size_t>(B) * sizeof(RsPass) + rs_forward_bound(B, H, W, max_side) * sizeof(int);
    P.rg.dev = static_cast<char*>(P.pool.get_fresh(P.rg.dev_bytes));
    auto mid = alloc_raw(P, static_cast<size_t>(B) * max_side * W * 3);
    auto img = alloc_raw(P, static_cast<size_t>(B) * H * W * 3);
    P.keep.push_back(mid);
    P.keep.push_back(img);
    P.rg.in_mid = static_cast<uint8_t*>(mid.get());
    P.rg.in_net = static_cast<uint8_t*>(img.get());
    P.ranges.emplace_back(P.ops.size(), "resize_in");
    resample_ragged(P, B, 0, 0);
    net_in = U8View();
    net_in.p = P.rg.in_net; net_in.img = 3ll * H * W; net_in.w = W;
  } else if (g) {
    net_in.img = 3ll * g->in_H * g->in_W; net_in.w = g->in_W;
    if (g->in_H == g->resize_H && g->in_W == g->resize_W) {
      net_in.off = 3 * (static_cast<long long>(g->crop_y) * g->in_W + g->crop_x);   // a crop of the input itself: no pass
    } else {
      auto buf = alloc_raw(P, static_cast<size_t>(B_in) * H * W * 3);
      P.keep.push_back(buf);
      U8View d;
      d.p = static_cast<uint8_t*>(buf.get()); d.img = 3ll * H * W; d.w = W;
      P.ranges.emplace_back(P.ops.size(), "resize_in");
      resample_fixed(P, net_in, B_in, g->in_H, g->in_W, g->resize_H, g->resize_W, g->crop_y, g->crop_x, H, W, d);
      net_in = d;
    }
  }
  P.ranges.emplace_back(P.ops.size(), "vae_encode");
  Act z = build_vae_encoder(P, vp, B, H, W, skips, (io_mode & IO_U8_IN) ? &net_in : nullptr, shared_input);
  P.ranges.emplace_back(P.ops.size(), "unet");
  Act pred = build_unet(P, z, text_batch, text_cached);
  mark(P, "model_pred", pred);
  P.ranges.emplace_back(P.ops.size(), "ddpm_step");
  Act dec_in = alloc_act(P, B, H / 8, W / 8, 8, 8, true);
  {
    // alpha_bar_999 of the scaled-linear schedule (fp32 cumprod, as diffusers computes it): 0.0046600951
    const float sa = 0.06826488673686981f, s1 = 0.9976672530174255f, inv_sf = 1.0f / cfg.scaling_factor;
    const long long HW = static_cast<long long>(H / 8) * (W / 8), total = HW * B;
    const uint16_t* zp = z.p;
    const uint16_t* pp = pred.p;
    uint16_t* dp = dec_in.p;
    const int ldp = pred.ld, dt = dtype;
    // the two wrappers call DDPMScheduler.step with different timestep shapes => different rounding (kernels.cuh)
    const int three_round = (cfg.model_kind == I2IT_CYCLEGAN) ? 1 : 0;
    Plan* plan = &P;
    P.keep.push_back(z.hold);
    P.keep.push_back(pred.hold);
    add_op(P, [=](cudaStream_t st) {
      DISPATCH_T(dt, (launch_k(ddpm_step_kernel<T>, dim3(ceil_div_i(total, 128)), dim3(128), 0, st, 0,
                         reinterpret_cast<const T*>(zp), reinterpret_cast<const T*>(pp), ldp, s1, sa, inv_sf,
                         reinterpret_cast<T*>(dp), reinterpret_cast<T*>(plan->io.out_latent), HW, total, three_round)));
    });
  }
  mark(P, "dec_in", dec_in);
  P.ranges.emplace_back(P.ops.size(), "vae_decode");
  build_vae_decoder(P, vp, dec_in, skips);
  if (io_mode & IO_U8_OUT) {
    // the last conv wrote NCHW into an internal buffer (forward() points io.out at it); convert to uint8 HWC for the caller,
    // or with an output size into an internal [B, H, W, 3] image that the resize passes read
    const long long HW = static_cast<long long>(H) * W, total = HW * B;
    const int dt = dtype;
    Plan* plan = &P;
    U8View out;
    out.slot = &P.io.out_u8; out.img = 3 * HW; out.w = W;
    const bool resize_out = ragged || (g && (g->out_H != H || g->out_W != W));
    U8View net_out = out;
    if (resize_out) {
      auto buf = alloc_raw(P, static_cast<size_t>(total) * 3);
      P.keep.push_back(buf);
      net_out = U8View();
      net_out.p = static_cast<uint8_t*>(buf.get()); net_out.img = 3 * HW; net_out.w = W;
    }
    add_op(P, [=](cudaStream_t st) {
      DISPATCH_T(dt, (launch_k(nchw_to_u8hwc_kernel<T>, dim3(ceil_div_i(total, 256)), dim3(256), 0, st, 0,
                         reinterpret_cast<const T*>(plan->io.out), net_out.get(), HW, total)));
    }, "unpack_u8", 0, 1.0 * total * (6 + 3));
    if (ragged) {
      auto mid = alloc_raw(P, static_cast<size_t>(B) * H * max_side * 3);
      P.keep.push_back(mid);
      P.rg.out_net = net_out.p;
      P.rg.out_mid = static_cast<uint8_t*>(mid.get());
      P.ranges.emplace_back(P.ops.size(), "resize_out");
      resample_ragged(P, B, 2 * B, 2);
    } else if (resize_out) {
      out.img = 3ll * g->out_H * g->out_W; out.w = g->out_W;
      P.ranges.emplace_back(P.ops.size(), "resize_out");
      resample_fixed(P, net_out, B, H, W, g->out_H, g->out_W, 0, 0, g->out_H, g->out_W, out);
    }
  }
  flush_prep();                             // every weight of the plan: one fold/re-layout launch (+ the time-embedding GEMVs)
  I2IT_CUDA(cudaDeviceSynchronize());       // weight preparation ran on the default stream
  I2IT_CUDA(cudaGetLastError());
  // back the plan's transient bytes before it can run; a failed mapping throws here, before the plan is inserted, and
  // leaves the arena and the resident plans as they were
  arena_.grow(P.pool.transient());
  P.last_run = ++tick_;
  Plan* raw_plan = up.get();
  plans_[key] = std::move(up);
  guard.ok = true;
  ++plan_builds_;
  if (evict) evict_lru(raw_plan);
  return raw_plan;
}

}  // namespace i2it

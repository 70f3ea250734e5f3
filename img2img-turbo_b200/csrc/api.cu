// extern "C" boundary of libi2it (see include/i2it.h).  Nothing throws across it.
#include "engine.cuh"

using namespace i2it;

struct i2it_handle {
  Engine* eng = nullptr;
  std::vector<OpMeta> op_meta;     // launch list of the last diagnostic op call (i2it_op_launches)
};
static thread_local std::string g_create_error;

#define API_BEGIN(h)                                            \
  if (!(h) || !(h)->eng) return 1;                              \
  Engine& E = *(h)->eng;                                        \
  try {                                                         \
    I2IT_CUDA(cudaSetDevice(E.cfg.device));
#define API_END                                                 \
    return 0;                                                   \
  } catch (const std::exception& ex) {                          \
    E.last_error = ex.what();                                   \
    cudaGetLastError();                                         \
    return 2;                                                   \
  } catch (...) {                                               \
    E.last_error = "unknown C++ exception";                     \
    return 3;                                                   \
  }

extern "C" {

int i2it_default_config(i2it_config* c) {
  if (!c) return 1;
  std::memset(c, 0, sizeof *c);
  c->dtype = I2IT_BF16;
  c->model_kind = I2IT_PIX2PIX;
  c->device = 0;
  const int uc[4] = {320, 640, 1280, 1280}, uh[4] = {5, 10, 20, 20}, vc[4] = {128, 256, 512, 512};
  for (int i = 0; i < 4; ++i) { c->unet_channels[i] = uc[i]; c->unet_heads[i] = uh[i]; c->vae_channels[i] = vc[i]; }
  c->cross_dim = 1024;
  c->temb_dim = 1280;
  c->scaling_factor = 0.18215f;
  c->keep_stages = 0;
  c->use_cuda_graph = 1;
  c->text_heads = 16;
  c->text_act = 0;
  return 0;
}

int i2it_create(const i2it_config* cfg, i2it_handle** out) {
  if (!cfg || !out) return 1;
  try {
    i2it_handle* h = new i2it_handle();
    h->eng = new Engine(*cfg);
    *out = h;
    return 0;
  } catch (const std::exception& ex) {
    g_create_error = ex.what();
    cudaGetLastError();
    return 2;
  }
}

void i2it_destroy(i2it_handle* h) {
  if (!h) return;
  try { delete h->eng; } catch (...) {}
  delete h;
}

const char* i2it_last_error(const i2it_handle* h) {
  if (!h || !h->eng) return g_create_error.c_str();
  return h->eng->last_error.c_str();
}

int i2it_set_weight(i2it_handle* h, const char* key, const void* data, const int64_t* shape, int ndim, int dtype,
                    int is_device) {
  API_BEGIN(h)
  I2IT_CHECK(key && data && shape && ndim > 0 && ndim <= 4, "i2it_set_weight: bad arguments");
  E.set_weight(key, data, shape, ndim, dtype, is_device != 0);
  API_END
}

int i2it_set_adapter_scale(i2it_handle* h, const char* adapter, float s) {
  API_BEGIN(h)
  I2IT_CHECK(adapter != nullptr, "null adapter name");
  E.set_adapter_scale(adapter, s);
  API_END
}

int i2it_finalize_weights(i2it_handle* h, float lw_unet, float lw_vae, float skip_gamma, float twin_r) {
  API_BEGIN(h)
  E.finalize(lw_unet, lw_vae, skip_gamma, twin_r);
  API_END
}

int i2it_refold_weights(i2it_handle* h, float lw_unet, float lw_vae, float skip_gamma, float twin_r) {
  API_BEGIN(h)
  E.refold(lw_unet, lw_vae, skip_gamma, twin_r);
  API_END
}

int i2it_workspace_bytes(i2it_handle* h, int batch, int H, int W, size_t* bytes) {
  API_BEGIN(h)
  I2IT_CHECK(bytes != nullptr, "null out pointer");
  // the plan the last forward ran when it has this shape (whatever its text / io mode): building a second plan of a
  // 12 MP image only to measure it would hold two workspaces
  Plan* P = E.last_plan();
  const bool match = P && P->key.size() >= 3 && P->key[0] == batch && P->key[1] == H && P->key[2] == W;
  if (!match) P = E.plan_for(batch, H, W, I2IT_A2B, 1);
  *bytes = P->pool.total;
  API_END
}

int i2it_set_max_plans(i2it_handle* h, int max_plans) {
  API_BEGIN(h)
  E.set_max_plans(max_plans);
  API_END
}

int i2it_release_plans(i2it_handle* h) {
  API_BEGIN(h)
  E.release_plans();
  API_END
}

int i2it_memory_stats_get(i2it_handle* h, i2it_memory_stats* s) {
  API_BEGIN(h)
  I2IT_CHECK(s != nullptr, "null out pointer");
  *s = E.memory_stats();
  API_END
}

int i2it_debug_poison_workspace(i2it_handle* h, int value) {
  API_BEGIN(h)
  E.poison_workspace(value);
  API_END
}

int i2it_forward(i2it_handle* h, const i2it_forward_desc* d, void* stream) {
  API_BEGIN(h)
  I2IT_CHECK(d != nullptr, "i2it_forward: null request");
  E.check_device_error();
  E.forward(*d, static_cast<cudaStream_t>(stream));
  API_END
}

int i2it_set_text(i2it_handle* h, const void* text_emb, int text_batch, void* stream) {
  API_BEGIN(h)
  E.check_device_error();
  E.set_text(text_emb, text_batch, static_cast<cudaStream_t>(stream));
  API_END
}

int i2it_encode_text(i2it_handle* h, const int32_t* tokens, int batch, void* out, void* stream) {
  API_BEGIN(h)
  E.check_device_error();
  E.encode_text(reinterpret_cast<const int*>(tokens), batch, out, static_cast<cudaStream_t>(stream));
  API_END
}

int i2it_mixed_size_check(int H, int W, char* msg, size_t cap) {
  const std::string why = i2it::mixed_size_rule(H, W);
  if (msg && cap > 0) {
    const size_t n = std::min(cap - 1, why.size());
    std::memcpy(msg, why.data(), n);
    msg[n] = 0;
  }
  return why.empty() ? 0 : 1;
}

int i2it_debug_ragged_tables(const i2it_resize_desc* g, int n, int H, int W, int max_side, long long* used, long long* bound) {
  try {
    i2it::rs_check_ragged(g, n, H, W, max_side);
    i2it::RsTableCache cache;
    const i2it::RsCall c = i2it::rs_forward_call(g, n, H, W, max_side, cache, nullptr, nullptr, nullptr);   // what the forward uploads
    if (used) *used = static_cast<long long>(c.tab.size());
    if (bound) *bound = i2it::rs_forward_bound(n, H, W, max_side);
    return 0;
  } catch (...) {
    return -1;
  }
}

int i2it_debug_graph_captures(i2it_handle* h, int* captures) {
  API_BEGIN(h)
  I2IT_CHECK(captures != nullptr, "null out pointer");
  *captures = E.graph_captures;
  API_END
}

int i2it_debug_resample_coeffs(int in_size, int out_size, int* bounds, int* coeffs, int cap) {
  try {
    const i2it::ResampleTable t = i2it::lanczos_table(in_size, out_size);   // the host function the plans upload from
    if (coeffs && static_cast<size_t>(cap) < t.coeffs.size()) return -1;
    if (bounds) std::memcpy(bounds, t.bounds.data(), t.bounds.size() * sizeof(int));
    if (coeffs) std::memcpy(coeffs, t.coeffs.data(), t.coeffs.size() * sizeof(int));
    return t.ksize;
  } catch (...) {
    return -1;
  }
}

long long i2it_debug_fast_div(long long max_dividend, int d, int x) {
  const uint32_t m = i2it::make_magic(max_dividend, d);              // the host function launch_gemm uses
  if (m == 0) return -1;
  if (d == 1) return x;                                              // fast_div selects x for d == 1
  return static_cast<long long>((static_cast<unsigned long long>(static_cast<uint32_t>(x)) * m) >> 32);   // == __umulhi(x, m)
}

int i2it_prep_launch_count(i2it_handle* h, int* launches) {
  API_BEGIN(h)
  I2IT_CHECK(launches != nullptr, "null out pointer");
  *launches = E.prep_launches_;
  API_END
}

int i2it_launch_count(i2it_handle* h, int batch, int H, int W, int direction, int* launches) {
  API_BEGIN(h)
  I2IT_CHECK(launches != nullptr, "null out pointer");
  Plan* P = E.last_plan();
  const bool match = P && P->key.size() >= 4 && P->key[0] == batch && P->key[1] == H && P->key[2] == W && P->key[3] == direction;
  if (!match) P = E.plan_for(batch, H, W, direction, 1);
  *launches = static_cast<int>(P->ops.size());
  API_END
}

int i2it_profile(i2it_handle* h, int reps, char* json, size_t cap, void* stream) {
  API_BEGIN(h)
  I2IT_CHECK(json != nullptr && cap > 2 && reps > 0, "i2it_profile: bad arguments");
  const std::string js = E.profile_json(reps, static_cast<cudaStream_t>(stream));
  I2IT_CHECK(js.size() + 1 <= cap, "i2it_profile: buffer too small (" + std::to_string(js.size() + 1) + " bytes needed)");
  std::memcpy(json, js.c_str(), js.size() + 1);
  API_END
}

int i2it_read_stage(i2it_handle* h, const char* name, float* dst, size_t dst_elems, int dims[4]) {
  API_BEGIN(h)
  E.read_stage(name, dst, dst_elems, dims);
  API_END
}

static void copy_json(const std::string& js, char* json, size_t cap, const char* what) {
  I2IT_CHECK(json != nullptr && cap > 2, std::string(what) + ": bad arguments");
  I2IT_CHECK(js.size() + 1 <= cap, std::string(what) + ": buffer too small (" + std::to_string(js.size() + 1) + " bytes needed)");
  std::memcpy(json, js.c_str(), js.size() + 1);
}

int i2it_stage_names(i2it_handle* h, char* json, size_t cap) {
  API_BEGIN(h)
  copy_json(E.stage_names_json(), json, cap, "i2it_stage_names");
  API_END
}

int i2it_text_stage_names(i2it_handle* h, char* json, size_t cap) {
  API_BEGIN(h)
  copy_json(E.stage_names_json(/*text=*/true), json, cap, "i2it_text_stage_names");
  API_END
}

int i2it_prepared_keys(i2it_handle* h, char* json, size_t cap) {
  API_BEGIN(h)
  copy_json(E.prepared_keys_json(), json, cap, "i2it_prepared_keys");
  API_END
}

int i2it_read_prepared(i2it_handle* h, const char* key, void* w, size_t w_elems, float* bias, size_t b_elems, int dims[4]) {
  API_BEGIN(h)
  I2IT_CHECK(key != nullptr && dims != nullptr, "i2it_read_prepared: null argument");
  E.read_prepared(key, w, w_elems, bias, b_elems, dims);
  API_END
}

int i2it_debug_refold_info(i2it_handle* h, char* json, size_t cap) {
  API_BEGIN(h)
  copy_json(E.refold_info_json(), json, cap, "i2it_debug_refold_info");
  API_END
}

// ------------------------------------------------------------------------------------------------
// diagnostic single-op entry points
// ------------------------------------------------------------------------------------------------
static void run_plan(i2it_handle* h, Plan& P, cudaStream_t st) {
  Engine& E = *h->eng;
  h->op_meta = P.meta;
  E.flush_prep();
  I2IT_CUDA(cudaDeviceSynchronize());
  for (auto& op : P.ops) op(st);
  cudaError_t e = cudaStreamSynchronize(st);
  E.check_device_error();
  I2IT_CUDA(e);
  I2IT_CUDA(cudaGetLastError());
}

static Act view(const void* p, int N, int H, int W, int C, int ld) {
  Act a;
  a.p = reinterpret_cast<uint16_t*>(const_cast<void*>(p));
  a.N = N; a.H = H; a.W = W; a.C = C; a.ld = ld;
  return a;
}

// the b2a weight set and directions of i2it_op_conv2d_sel
struct OpSel { const float* w; const float* bias; const float* w2; const int* dirs; };

static int op_conv(i2it_handle* h, const i2it_conv_desc* d, const OpSel* sel, void* stream) {
  API_BEGIN(h)
  I2IT_CHECK(d && d->x && d->w && d->out, "i2it_op_conv2d_ex: null operand");
  const int stride = d->stride > 0 ? d->stride : 1, k = d->ksize, oc = (d->act == TG_ACT_GEGLU) ? d->Cout / 2 : d->Cout;
  I2IT_CHECK(!d->asym_pad || ((d->H | d->W) & 1) == 0, "i2it_op_conv2d_ex: asymmetric padding needs an even map");
  I2IT_CHECK(!d->up2x || (k == 3 && stride == 1 && d->bias && !d->residual && !d->out_fp32 && d->act == TG_ACT_NONE),
             "i2it_op_conv2d_ex: up2x is a biased 3x3 stride-1 conv without residual, activation or fp32 output");
  I2IT_CHECK(!d->tokens || (k == 1 && !d->up2x), "i2it_op_conv2d_ex: token rows need a 1x1 conv");
  I2IT_CHECK(!d->gn_y || (d->gn_gamma && d->gn_beta && !d->out_fp32), "i2it_op_conv2d_ex: GroupNorm needs gamma, beta, 16-bit out");
  const int64_t wshape[4] = {d->Cout, d->Cin, k, k};
  E.set_weight("__op.conv.weight", d->w, wshape, 4, I2IT_F32, true);
  if (d->bias) { const int64_t bshape[1] = {d->Cout}; E.set_weight("__op.conv.bias", d->bias, bshape, 1, I2IT_F32, true); }
  if (d->x2) {
    I2IT_CHECK(d->w2 != nullptr, "i2it_op_conv2d_ex: x2 without w2");
    const int64_t w2shape[4] = {d->Cout, d->C2, 1, 1};
    E.set_weight("__op.conv2.weight", d->w2, w2shape, 4, I2IT_F32, true);
  }
  if (sel) {
    I2IT_CHECK(sel->w && !sel->bias == !d->bias, "i2it_op_conv2d_sel: w_alt is required, and bias_alt iff bias");
    I2IT_CHECK(sel->dirs, "i2it_op_conv2d_sel: null direction array");
    for (int i = 0; i < d->N; ++i)
      I2IT_CHECK(sel->dirs[i] == 0 || sel->dirs[i] == 1, "i2it_op_conv2d_sel: direction " + std::to_string(sel->dirs[i]) +
                                                             " of image " + std::to_string(i) + " is neither 0 nor 1");
    E.set_weight("__op.convb.weight", sel->w, wshape, 4, I2IT_F32, true);
    if (d->bias) { const int64_t bshape[1] = {d->Cout}; E.set_weight("__op.convb.bias", sel->bias, bshape, 1, I2IT_F32, true); }
    if (d->x2 && sel->w2) {
      const int64_t w2shape[4] = {d->Cout, d->C2, 1, 1};
      E.set_weight("__op.conv2b.weight", sel->w2, w2shape, 4, I2IT_F32, true);
    }
  }
  E.finalize(1.f, 1.f, 1.f, -1.f);
  {
    Plan P;
    P.debug_tapgemm = true;
    if (sel) {
      P.dir = static_cast<int*>(P.pool.get_fresh(static_cast<size_t>(d->N) * sizeof(int)));
      I2IT_CUDA(cudaMemcpy(P.dir, sel->dirs, static_cast<size_t>(d->N) * sizeof(int), cudaMemcpyHostToDevice));
    }
    // the selecting op: each weight carries its b2a twin and the directions (a shared second-source weight without w2_alt)
    auto paired = [&](PW a, const PW& b) {
      if (!sel) return a;
      a.w_alt = b.w; a.bias_alt = b.bias; a.dir = P.dir;
      return a;
    };
    // Ho = ceil(H / stride): Engine::conv pads an odd map to even before a stride-2 conv
    const int Ho = d->up2x ? 2 * d->H : (d->H + stride - 1) / stride, Wo = d->up2x ? 2 * d->W : (d->W + stride - 1) / stride;
    Act xin = view(d->x, d->N, d->H, d->W, d->Cin, d->ldx);
    Act res = view(d->residual, d->N, Ho, Wo, oc, d->ldr);
    Act ov = view(d->out, d->N, Ho, Wo, oc, d->ldo);
    Act x2 = view(d->x2, d->N, Ho, Wo, d->C2, d->ld2);
    PW pw2;
    if (d->x2) pw2 = E.prep("__op.conv2", {"__op.conv2"});
    if (d->x2 && sel && sel->w2) pw2 = paired(pw2, E.prep("__op.conv2b", {"__op.conv2b"}));
    Act y;
    if (d->up2x) {
      const PW pw = paired(E.prep_subpixel("__op.conv"), sel ? E.prep_subpixel("__op.convb") : PW());
      y = E.conv_up2x(P, xin, pw, d->x2 ? &x2 : nullptr, d->x2 ? &pw2 : nullptr, d->gn_y != nullptr);
      E.copy_channels(P, y, ov);
    } else {
      const PW pw = paired(E.prep("__op.conv", {"__op.conv"}, d->act == TG_ACT_GEGLU),
                           sel ? E.prep("__op.convb", {"__op.convb"}, d->act == TG_ACT_GEGLU) : PW());
      ConvOpts o;
      o.ksize = k; o.stride = stride; o.asym = d->asym_pad != 0; o.act = d->act; o.out_fp32 = d->out_fp32 != 0;
      o.gn_out = d->gn_y != nullptr;
      if (d->tokens) {
        o.gn_rows_per_image = 1ll * d->H * d->W;
        xin = xin.as_rows(); res = res.as_rows(); ov = ov.as_rows(); x2 = x2.as_rows();
      }
      if (d->residual) o.res = &res;
      if (d->x2) { o.x2 = &x2; o.w2 = &pw2; }
      o.out = &ov;
      y = E.conv(P, xin, pw, o);
      y.N = d->N; y.H = Ho; y.W = Wo;
    }
    if (d->gn_y) {
      NormW nw; nw.g = d->gn_gamma; nw.b = d->gn_beta; nw.C = oc;
      const Act g = E.group_norm(P, y, nw, d->gn_eps, d->gn_silu != 0);
      E.copy_channels(P, g, view(d->gn_y, d->N, Ho, Wo, oc, d->ldg));
    }
    run_plan(h, P, static_cast<cudaStream_t>(stream));
  }
  API_END
}

int i2it_op_conv2d_ex(i2it_handle* h, const i2it_conv_desc* d, void* stream) { return op_conv(h, d, nullptr, stream); }

int i2it_op_conv2d_sel(i2it_handle* h, const i2it_conv_desc* d, const float* w_alt, const float* bias_alt, const float* w2_alt,
                       const int* directions, void* stream) {
  const OpSel sel{w_alt, bias_alt, w2_alt, directions};
  return op_conv(h, d, &sel, stream);
}

int i2it_op_conv2d(i2it_handle* h, const void* x, int N, int H, int W, int Cin, int ldx, const float* w,
                   const float* bias, int Cout, int ksize, int stride, int asym_pad, const void* residual, int ldr,
                   int act, void* out, int ldo, int out_fp32, void* stream) {
  i2it_conv_desc d;
  std::memset(&d, 0, sizeof d);
  d.x = x; d.N = N; d.H = H; d.W = W; d.Cin = Cin; d.ldx = ldx; d.w = w; d.bias = bias; d.Cout = Cout; d.ksize = ksize;
  d.stride = stride; d.asym_pad = asym_pad; d.residual = residual; d.ldr = ldr; d.act = act; d.out = out; d.ldo = ldo;
  d.out_fp32 = out_fp32;
  return i2it_op_conv2d_ex(h, &d, stream);
}

int i2it_op_launches(i2it_handle* h, char* json, size_t cap) {
  API_BEGIN(h)
  I2IT_CHECK(json != nullptr && cap > 2, "i2it_op_launches: bad arguments");
  std::string js = "[";
  for (size_t i = 0; i < h->op_meta.size(); ++i)
    js += std::string(i ? "," : "") + "{\"kind\":\"" + h->op_meta[i].kind + "\",\"shape\":\"" + h->op_meta[i].shape + "\"}";
  js += "]";
  I2IT_CHECK(js.size() + 1 <= cap, "i2it_op_launches: buffer too small");
  std::memcpy(json, js.c_str(), js.size() + 1);
  API_END
}

int i2it_op_group_norm(i2it_handle* h, const void* x, int N, int HW, int C, int ldx, const float* gamma,
                       const float* beta, float eps, int silu, void* out, int ldo, void* stream) {
  API_BEGIN(h)
  {
    Plan P;
    NormW nw; nw.g = gamma; nw.b = beta; nw.C = C;
    Act y = E.group_norm(P, view(x, N, 1, HW, C, ldx), nw, eps, silu != 0);
    E.copy_channels(P, y, view(out, N, 1, HW, C, ldo));
    run_plan(h, P, static_cast<cudaStream_t>(stream));
  }
  API_END
}

int i2it_op_layer_norm(i2it_handle* h, const void* x, int rows, int C, int ldx, const float* gamma, const float* beta,
                       float eps, void* out, int ldo, void* stream) {
  API_BEGIN(h)
  (void)eps;
  {
    Plan P;
    NormW nw; nw.g = gamma; nw.b = beta; nw.C = C;
    Act y = E.layer_norm(P, view(x, 1, 1, rows, C, ldx), nw);
    E.copy_channels(P, y, view(out, 1, 1, rows, C, ldo));
    run_plan(h, P, static_cast<cudaStream_t>(stream));
  }
  API_END
}

int i2it_op_attention(i2it_handle* h, const void* q, int ldq, const void* k, int ldk, const void* vt, int ldv, int B,
                      int Nq, int Nk, int heads, int d, int kv_batch, int causal, void* out, int ldo, void* stream) {
  API_BEGIN(h)
  I2IT_CHECK(!causal || (d == FA_D && E.use_flash), "i2it_op_attention: causal attention runs on the flash path (d = 64)");
  {
    Plan P;
    P.debug_tapgemm = true;
    const int C = heads * d;
    const Act qa = view(q, B, 1, Nq, C, ldq), ka = view(k, kv_batch, 1, Nk, C, ldk), va = view(vt, kv_batch, 1, C, ldv, ldv);
    Act o = causal ? E.flash_attention(P, qa, ka, va, B, Nq, Nk, heads, kv_batch, true)
                   : E.attention(P, qa, ka, va, B, Nq, Nk, heads, d, kv_batch);
    E.copy_channels(P, o, view(out, B, 1, Nq, C, ldo));
    run_plan(h, P, static_cast<cudaStream_t>(stream));
  }
  API_END
}

int i2it_op_vt_proj(i2it_handle* h, const void* x, int B, int ntok, int Cin, int ldx, const float* w, const float* bias, int Cout,
                    void* out, void* stream) {
  API_BEGIN(h)
  const int64_t wshape[2] = {Cout, Cin};
  E.set_weight("__op.vt.weight", w, wshape, 2, I2IT_F32, true);
  if (bias) { const int64_t bshape[1] = {Cout}; E.set_weight("__op.vt.bias", bias, bshape, 1, I2IT_F32, true); }
  E.finalize(1.f, 1.f, 1.f, -1.f);
  {
    Plan P;
    P.debug_tapgemm = true;
    const PW pw = E.prep("__op.vt", {"__op.vt"});
    const Act vt = E.vt_proj(P, view(x, 1, 1, B * ntok, Cin, ldx), B, ntok, pw);
    E.copy_channels(P, vt, view(out, B, 1, Cout, vt.C, vt.C));
    run_plan(h, P, static_cast<cudaStream_t>(stream));
  }
  API_END
}

int i2it_op_upsample2x(i2it_handle* h, const void* x, int N, int H, int W, int C, void* out, void* stream) {
  API_BEGIN(h)
  {
    Plan P;
    Act y = E.upsample2x(P, view(x, N, H, W, C, C));
    E.copy_channels(P, y, view(out, N, 2 * H, 2 * W, C, C));
    run_plan(h, P, static_cast<cudaStream_t>(stream));
  }
  API_END
}

int i2it_op_upsample_to(i2it_handle* h, const void* x, int N, int H, int W, int C, int Ho, int Wo, void* out, void* stream) {
  API_BEGIN(h)
  {
    Plan P;
    Act y = E.upsample_to(P, view(x, N, H, W, C, C), Ho, Wo);
    E.copy_channels(P, y, view(out, N, Ho, Wo, C, C));
    run_plan(h, P, static_cast<cudaStream_t>(stream));
  }
  API_END
}

int i2it_debug_tapgemm_override(i2it_handle* h, int bn, int stages, int grid) {
  API_BEGIN(h)
  I2IT_CHECK(bn >= 0 && stages >= 0 && grid >= 0, "i2it_debug_tapgemm_override: values must be >= 0 (0: the engine's choice)");
  E.dbg_bn = bn; E.dbg_stages = stages; E.dbg_grid = grid;
  API_END
}

int i2it_op_resize_u8_ragged(i2it_handle* h, const void* const* x, const int* hw_in, void* const* out, const int* hw_out,
                             int n, int max_side, void* stream) {
  API_BEGIN(h)
  {
    Plan P;
    E.resize_ragged_op(P, x, hw_in, out, hw_out, n, max_side);
    run_plan(h, P, static_cast<cudaStream_t>(stream));
  }
  API_END
}

int i2it_op_resize_u8(i2it_handle* h, const void* x, int B, int H, int W, void* out, int H2, int W2, void* stream) {
  API_BEGIN(h)
  I2IT_CHECK(B > 0 && H > 0 && W > 0 && H2 > 0 && W2 > 0, "i2it_op_resize_u8: sizes must be positive");
  I2IT_CHECK(x && out, "i2it_op_resize_u8: null image pointer");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (H == H2 && W == W2) {   // PIL returns a copy
    h->op_meta.clear();
    I2IT_CUDA(cudaMemcpyAsync(out, x, static_cast<size_t>(B) * H * W * 3, cudaMemcpyDeviceToDevice, st));
    I2IT_CUDA(cudaStreamSynchronize(st));
  } else {
    Plan P;
    P.io.x_u8 = x; P.io.out_u8 = out;
    U8View s, d;
    s.slot = &P.io.x_u8; s.img = 3ll * H * W; s.w = W;
    d.slot = &P.io.out_u8; d.img = 3ll * H2 * W2; d.w = W2;
    E.resample_fixed(P, s, B, H, W, H2, W2, 0, 0, H2, W2, d);
    run_plan(h, P, st);
  }
  API_END
}

}  // extern "C"

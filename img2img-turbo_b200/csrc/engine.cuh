// Engine: weight store, load-time fold, plan builder (the model graph) and executor behind the C ABI.
#pragma once
#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/i2it.h"
#include "kernels.cuh"
#include "prep.cuh"
#include "tapgemm.cuh"
#include "flash.cuh"
#include "resample.cuh"

namespace i2it {

// ---------------------------------------------------------------------------------------------
// TMA tensor-map encoding (driver entry point fetched through the runtime: no libcuda link dependency)
// ---------------------------------------------------------------------------------------------
struct TmapSpec {
  const void* base = nullptr;
  uint64_t dim[5] = {1, 1, 1, 1, 1};
  uint64_t stride[4] = {16, 16, 16, 16};   // bytes, dims 1..4
  uint32_t box[5] = {1, 1, 1, 1, 1};
  TmapSpec() = default;
  // A view of a 16-bit tensor, innermost dimension first; dimensions left out have extent 1 (box 1).  stride[i] is the step of
  // dimension i + 1 in elements.  A dimension of extent 1 keeps its stride when that is a whole multiple of 16 bytes and
  // otherwise takes the 16-byte placeholder TMA accepts; any other stride must be a multiple of 8 elements, or an Error
  // naming the operand `what` is thrown (TMA cannot express such a pitch).
  TmapSpec(const char* what, const void* base, std::initializer_list<long long> dims,
           std::initializer_list<long long> strides, std::initializer_list<int> boxes);
};
CUtensorMap encode_tmap(const TmapSpec& s, int dtype);

// ---------------------------------------------------------------------------------------------
// workspace arena: one reserved virtual address range per handle whose head is backed by physical memory (CUDA virtual memory
// management).  Physical memory is mapped and unmapped at the tail only, so an address, once handed out, never moves: tensor
// maps and captured graphs stay valid while the arena grows and shrinks.
// ---------------------------------------------------------------------------------------------
struct Arena {
  int device = 0;
  CUdeviceptr base = 0;
  size_t reserved = 0, gran = 0, mapped = 0;
  struct Chunk { size_t off, size; CUmemGenericAllocationHandle h; };
  std::vector<Chunk> chunks;                 // physical allocations mapped back to back from `base`
  ~Arena();
  char* ptr();                               // base address (the range is reserved on first use)
  size_t round(size_t bytes) const { return (bytes + gran - 1) / gran * gran; }
  void grow(size_t bytes);                   // map [mapped, round(bytes)); throws with the old mapping intact
  // unmap down to round(bytes); the first `keep` bytes keep their contents (a chunk straddling the new end is re-created
  // smaller only when none of its bytes lie below `keep`).  Callers synchronise the device first.
  void shrink(size_t bytes, size_t keep);
  void fill(int value);                      // memset every mapped byte (synchronous)
};

// ---------------------------------------------------------------------------------------------
// workspace pool (plan-build time only; execution never allocates)
// ---------------------------------------------------------------------------------------------
struct Pool {
  std::vector<std::pair<void*, size_t>> blocks;   // cudaMalloc'd blocks, freed with the pool
  std::multimap<size_t, void*> free_;
  size_t total = 0;                // transient + persistent bytes
  size_t persistent = 0;           // get_fresh bytes
  // Transient blocks (get) are recycled by build-order liveness and written by every forward before it reads them.  With an
  // arena they are offsets from its base, shared with every other plan of the handle (whose forwards never overlap); the
  // arena maps them when the plan is complete (Engine::plan_for).  Without one, each is its own cudaMalloc.
  Arena* arena = nullptr;
  ~Pool();
  void* get(size_t bytes, size_t* actual);
  // never recycled and never in the arena: state written at build time or kept between replays (zero-padded small-channel
  // tensors, GroupNorm tickets, resample tables)
  void* get_fresh(size_t bytes);
  void put(void* p, size_t bytes) { free_.emplace(bytes, p); }
  size_t transient() const { return total - persistent; }
};

// GroupNorm partial statistics written by the epilogue of the GEMM that PRODUCED a tensor (see TapGemmParams::gn_part):
// [phases][images][slots_per_image][C / red] x (sum, sum of squares), fp32
struct GnPart {
  std::shared_ptr<void> hold;
  float* buf = nullptr;
  int red = 2, slots_per_image = 0, C = 0, phases = 1, images = 0;
};

struct Act {                       // NHWC view, 2-byte elements
  std::shared_ptr<void> hold;
  uint16_t* p = nullptr;
  int N = 0, H = 0, W = 0, C = 0, ld = 0;
  std::shared_ptr<GnPart> gn;      // statistics of this (whole) tensor, if its producer computed them
  long long img() const { return static_cast<long long>(H) * W * ld; }
  long long rows() const { return static_cast<long long>(N) * H * W; }
  Act as_rows() const { Act a = *this; a.W = static_cast<int>(rows()); a.N = 1; a.H = 1; return a; }
  Act slice(int c0, int c) const { Act a = *this; a.p = p + c0; a.C = c; a.gn = nullptr; return a; }
};

struct PW {                        // prepared (folded, re-laid-out) weight: [taps][rows][cin_pad] + fp32 bias
  uint16_t* w = nullptr;
  float* bias = nullptr;
  int rows = 0, cin = 0, cin_pad = 0, taps = 1;
  // a mixed-direction plan's VAE weight: the b2a twin (same shape), taken by the images whose dir[] entry is 1
  uint16_t* w_alt = nullptr;
  float* bias_alt = nullptr;
  const int* dir = nullptr;        // non-null: the launches that use this weight select per image
};
// ---- kernel launch for plan ops: programmatic dependent launch (see pdl_sync in common.cuh) when the previous op of the
// plan was also a kernel; `cluster` > 0 adds a (cluster,1,1) cluster dimension.  Executor state, one engine call per thread.
struct PdlState { bool enabled = true; bool prev_is_kernel = false; };
extern thread_local PdlState g_pdl;
template <typename... KA, typename... A>
inline void launch_k(void (*kern)(KA...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster, A&&... args) {
  cudaLaunchConfig_t cfg;
  std::memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[2];
  unsigned n = 0;
  if (cluster > 0) {
    at[n].id = cudaLaunchAttributeClusterDimension;
    at[n].val.clusterDim.x = cluster; at[n].val.clusterDim.y = 1; at[n].val.clusterDim.z = 1;
    ++n;
  }
  if (g_pdl.enabled && g_pdl.prev_is_kernel) {
    at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = at; cfg.numAttrs = n;
  cudaLaunchKernelEx(&cfg, kern, std::forward<A>(args)...);
  g_pdl.prev_is_kernel = true;
}

struct NormW {
  const float* g = nullptr; const float* b = nullptr; int C = 0;
  const float* g_alt = nullptr; const float* b_alt = nullptr; const int* dir = nullptr;   // as PW's alternative set
};

struct IO {
  const void* x = nullptr; const void* text = nullptr; const void* eps = nullptr; const void* noise = nullptr;
  float r = 1.f; void* out = nullptr; void* out_latent = nullptr;
  const void* x_u8 = nullptr; void* out_u8 = nullptr;   // uint8 HWC boundary (x_u8 / out_u8 requests): out then points at an internal buffer
  int in_mode = 0;                                      // u8 input transform (see pack_input_im2col_u8_kernel)
  int pad_ = 0;
  bool operator==(const IO& o) const { return std::memcmp(this, &o, sizeof(IO)) == 0; }
};
// IO_SHARED_IN: a variations forward, one input image for the whole batch (its encoder runs at batch 1)
// IO_RAGGED: uint8 images of their own sizes, each resized to and from the one network size (x_u8_list requests)
enum IoMode : int { IO_U8_IN = 1, IO_U8_OUT = 2, IO_SHARED_IN = 4, IO_RAGGED = 8 };
// the plan-key direction of a mixed-direction CycleGAN plan (I2IT_A2B = 0 and I2IT_B2A = 1 are the single-direction ones)
constexpr int DIR_MIXED = 2;
// the 128-row tile box (tw x th pixels of tn images) Engine::conv picks for an Ho x Wo output; nchw: the final image's launch
void conv_box(bool stride1, int Ho, int Wo, bool nchw, int& tw, int& th, int& tn);

// uint8 HWC images [B][img bytes][w pixels per row][3] an op reads or writes: a caller pointer read from the plan's IO at
// launch time (slot), or a plan-internal buffer (p); off selects a window's first pixel
struct U8View {
  const void* const* slot = nullptr;
  uint8_t* p = nullptr;
  long long off = 0, img = 0;
  int w = 0;
  uint8_t* get() const { return (slot ? static_cast<uint8_t*>(const_cast<void*>(*slot)) : p) + off; }
};

// Capacity buffers of a ragged plan (or a ragged resize op).  The descriptors and tables live in `dev`: [descs RsPass][tables],
// rewritten by every call; the horizontal passes write the intermediates, the input side's vertical pass the network image
// the packing kernel reads, and the output conversion the network image the output side's passes read.
struct RaggedBufs {
  int max_side = 0, descs = 0;
  char* dev = nullptr;
  size_t dev_bytes = 0;
  uint8_t* in_mid = nullptr;       // [B][max_side][W][3]
  uint8_t* in_net = nullptr;       // [B][H][W][3]
  uint8_t* out_net = nullptr;      // [B][H][W][3]
  uint8_t* out_mid = nullptr;      // [B][H][max_side][3]
  size_t ops[4] = {0, 0, 0, 0};    // plan indices of the input side's h / v and the output side's h / v launches
  const int* tab() const { return reinterpret_cast<const int*>(dev + descs * sizeof(RsPass)); }
};

// The sizes a mixed-direction forward accepts: every tile of every VAE launch must hold rows of one image (conv boxes of one
// image: Engine::conv's box picker gives tn == 1; the attention's token launches: (H/8)(W/8) a multiple of 128).  Returns
// "" when H x W is accepted, else the reason.  Host only.
std::string mixed_size_rule(int H, int W);

// descriptors and tables of one ragged call, built on the host; bytes: algorithmic bytes of the four launches
struct RsCall {
  std::vector<RsPass> d;
  std::vector<int> tab;
  double bytes[4] = {0, 0, 0, 0};
};
// Rejects, with a message ending in `at`, a resize geometry with a non-positive size or an H x W crop window outside its
// resized image.  Host only.
void rs_check_geometry(const i2it_resize_desc& d, int H, int W, const std::string& at = "");
// Rejects, with a message, a ragged forward geometry: rs_check_geometry's rejections of each image, a dimension above
// max_side.  Host only.
void rs_check_ragged(const i2it_resize_desc* g, int n, int H, int W, int max_side);
// The call's descriptors (input h, input v, output h, output v; n each) and tables.  x / out / rg may be null (host-only
// sizing: the descriptors then carry null pointers).
RsCall rs_forward_call(const i2it_resize_desc* g, int n, int H, int W, int max_side, RsTableCache& cache, const void* const* x,
                       void* const* out, const RaggedBufs* rg);

struct OpMeta {                  // bookkeeping for i2it_profile / bench roofline accounting
  std::string kind;              // "tapgemm:conv3x3", "gn_apply", ...
  double flops = 0, bytes = 0;   // ALGORITHMIC work of the launch (2*M*N*K; unique bytes in + out + weights)
  std::string shape;
};

struct Plan {
  Pool pool;                                           // declared first: destroyed last
  std::vector<std::function<void(cudaStream_t)>> ops;  // one kernel launch each
  std::vector<OpMeta> meta;                            // parallel to ops
  std::map<std::string, Act> stages;
  std::vector<std::string> stage_order;                // stage names in build order (i2it_stage_names)
  struct Trace { unsigned long long* buf; int grid; std::string what; };
  std::vector<Trace> traces;                           // I2IT_TRACE=1 only
  std::vector<std::shared_ptr<void>> keep;
  std::vector<int> key;                                // (B, H, W, direction, text_batch, text_cached, io_mode[, resize geometry | max_side])
  unsigned long long last_run = 0;                     // engine tick of the last forward (or the build): LRU eviction order
  void* u8_out_tmp = nullptr;                          // NCHW image the last conv writes when the caller wants uint8 HWC
  int* gn_counter = nullptr;                           // per-image tickets of the GroupNorm last-block reductions (zero between launches)
  std::vector<std::pair<size_t, const char*>> ranges;  // (first op index, name): NVTX stage ranges of the eager path
  bool debug_tapgemm = false;                          // a diagnostic op plan: its tapgemm launches take the engine's dbg_* override
  RaggedBufs rg;                                       // IO_RAGGED plans and ragged resize ops
  int* dir = nullptr;                                  // mixed-direction plans: [B] directions, written before every run
  IO io;
  std::vector<std::pair<IO, cudaGraphExec_t>> graphs;  // small cache: one instantiated graph per distinct IO pointer set
  ~Plan() { for (auto& g : graphs) cudaGraphExecDestroy(g.second); }
};

struct ConvOpts {
  int ksize = 3, stride = 1;
  bool asym = false;             // VAE Downsample2D: F.pad(0,1,0,1) then pad-0 stride-2 conv
  const Act* res = nullptr;
  int act = TG_ACT_NONE;
  const Act* out = nullptr;      // write into this view instead of allocating
  bool out_fp32 = false;
  float alpha = 1.f;
  bool to_io_out_nchw = false;   // final image: write NCHW straight into IO.out
  int bias_mode = -1;            // -1: column bias iff the weight has one
  // second source folded into the same accumulator: out = conv(x) + conv1x1(x2)   (resnet conv_shortcut, decoder skip convs)
  const Act* x2 = nullptr;
  const PW* w2 = nullptr;
  bool x2_identity = false;      // x2/w2 is the residual x identity trick: not algorithmic work (excluded from flop counts)
  int subpixel_phase = -1;       // >=0: this launch is parity phase (py*2+px) of a fused nearest-2x-upsample + 3x3 conv
  bool gn_out = false;           // the consumer of the output is a GroupNorm: take its statistics in this GEMM's epilogue
  std::shared_ptr<GnPart> gn_share;   // sub-pixel phases 1..3 add to the partial buffer phase 0 created
  long long gn_rows_per_image = 0;    // linear(): rows per image of the flattened token matrix (0: spatial conv)
};

struct WT {                      // raw fp32 tensor of the state dict, on device
  float* d = nullptr;
  std::vector<int64_t> shape;
  long long numel = 0;
};

// The fold inputs a prepared weight's coefficients read (Recipe::uses)
enum FoldInput : unsigned { FOLD_LW_UNET = 1, FOLD_LW_VAE = 2, FOLD_GAMMA = 4, FOLD_TWIN_R = 8, FOLD_ADAPTER_SCALE = 16 };

// How a prepared weight was made, so Engine::refold can push its jobs again into the same buffers: `emit` is the prep_*
// or temb_bias call that made it (with its arguments), and reads the engine's fold inputs when it runs.  uses / reads /
// after are recorded by each run.
struct Recipe {
  std::string key;                   // its prepared_ / prepared_f32_ key
  std::function<void()> emit;
  unsigned uses = 0;                 // FoldInput bits
  std::vector<std::string> reads;    // master tensors its jobs read
  std::vector<std::string> after;    // recipes whose outputs its jobs read (a UNet conv1 bias reads its time-embedding GEMV)
};

// cached cross-attention operands of one prompt batch: K [tb*77, C] and V^T [tb][C][80] per transformer block
struct TextKV {
  Plan plan;                                   // declared first: its pool outlives the Acts below
  Act text;
  std::map<std::string, std::pair<Act, Act>> kv;   // transformer-block prefix -> (K, V^T)
  int text_batch = 0;
  bool filled = false;
};

class Engine {
 public:
  explicit Engine(const i2it_config& c);
  ~Engine();
  i2it_config cfg;
  int dtype, num_sms;
  std::string last_error;

  void set_weight(const std::string& key, const void* data, const int64_t* shape, int ndim, int dt, bool is_dev);
  void set_adapter_scale(const std::string& a, float s) { adapter_scale_[a] = s; }
  void finalize(float lw_unet, float lw_vae, float skip_gamma, float twin_r);
  // i2it_refold_weights: rewrite, in place, the prepared weights whose fold inputs changed since the last fold
  void refold(float lw_unet, float lw_vae, float skip_gamma, float twin_r);
  std::string refold_info_json() const;                               // i2it_debug_refold_info
  // g: LANCZOS resize geometry of a uint8 forward; part of the plan key
  // evict: enforce the plan limit once the plan is in (forward() does it itself after the plan becomes the last-run one)
  // max_side: the capacity of an IO_RAGGED plan (part of its key)
  Plan* plan_for(int B, int H, int W, int direction, int text_batch, bool text_cached = false, int io_mode = 0,
                 const i2it_resize_desc* g = nullptr, bool evict = true, int max_side = 0);
  // one image forward (i2it_forward): refuses every request include/i2it.h does not list, then runs check_mixed (a mixed
  // request), check_forward and the operand checks, all before a plan is built
  void forward(const i2it_forward_desc& d, cudaStream_t st);
  // rejects, with a message, what a mixed forward refuses before building anything: a pix2pix handle, a direction other
  // than 0 / 1, and a size whose VAE tiles would hold rows of two images
  void check_mixed(const int* dirs, int B, int H, int W) const;
  // the checks every image forward starts with (network size, text batch, a cached text when text is null); returns
  // whether the text is the cached one
  bool check_forward(int B, int H, int W, int text_batch, const void* text) const;
  // cross-attention K / V^T of the prompt, computed once per prompt (i2it_set_text) instead of once per forward
  void set_text(const void* text, int text_batch, cudaStream_t st);
  // CLIP text tower (SURVEY 8f #1): tokens [batch, 77] int32 -> last_hidden_state [batch, 77, hidden] in the handle dtype
  void encode_text(const int* tokens, int batch, void* out, cudaStream_t st);
  bool has_text_encoder() const { return has("text_encoder.text_model.embeddings.token_embedding.weight"); }
  Plan* last_plan() const { return last_plan_; }
  // ---- image-forward plan cache: transient buffers of every plan share one arena; plans are evicted least recently run ----
  void set_max_plans(int n);                                          // 0: no limit
  void release_plans();                                               // drop every image-forward plan, unmap the arena
  i2it_memory_stats memory_stats() const;
  void poison_workspace(int value);                                   // memset every mapped arena byte (tests)
  void read_stage(const std::string& name, float* dst, size_t dst_elems, int dims[4]);
  std::string stage_names_json(bool text = false) const;             // last forward's (text: last encode_text's) stages
  std::string prepared_keys_json() const;                            // every prepared-weight cache key, sorted
  // a prepared weight exactly as the kernels read it: [taps][rows][cin_pad] 16-bit + fp32 bias; dims = taps, rows, cin_pad, has_bias
  void read_prepared(const std::string& key, void* w, size_t w_elems, float* bias, size_t b_elems, int dims[4]);

  // ---- op builders (append launches to a plan) ----
  Act alloc_act(Plan& P, int N, int H, int W, int C, int ld = 0, bool zero_persistent = false);
  std::shared_ptr<void> alloc_raw(Plan& P, size_t bytes);
  Act conv(Plan& P, const Act& x, const PW& w, const ConvOpts& o);
  Act linear(Plan& P, const Act& x, const PW& w, const Act* res = nullptr, int act = TG_ACT_NONE, bool gn_out = false,
             const Act* out = nullptr);
  Act group_norm(Plan& P, const Act& x, const NormW& nw, float eps, bool silu);
  int* gn_counters(Plan& P, int images);
  Act layer_norm(Plan& P, const Act& x, const NormW& nw, bool to_io_out = false);
  Act upsample2x(Plan& P, const Act& x) { return upsample_to(P, x, 2 * x.H, 2 * x.W); }
  Act upsample_to(Plan& P, const Act& x, int Ho, int Wo);          // F.interpolate(size=(Ho,Wo), mode="nearest")
  Act pad_even(Plan& P, const Act& x);                               // zero-padded copy with even H and W
  // PIL LANCZOS resize of src [B, inH, inW, 3] to rsH x rsW, window [y0, y0+H) x [x0, x0+W) written densely to dst
  // [B, H, W, 3]: the horizontal pass if the width changes, then the vertical pass if the height changes (at least one must).
  // Descriptors and tables are uploaded here, once.
  void resample_fixed(Plan& P, const U8View& src, int B, int inH, int inW, int rsH, int rsW, int y0, int x0, int H, int W,
                      const U8View& dst);
  // one resize launch of `grid` blocks over descriptors d[0, n); a caller's view (slot) is the base its side's descriptor
  // addresses are relative to, read at launch; a plan buffer's or an empty view's base is 0
  void resample_pass(Plan& P, bool vertical, const RsPass* d, int n, const int* tab, const U8View& src, const U8View& dst,
                     int grid, const char* kind, double bytes, const std::string& shape);
  // the ragged resize launches (horizontal, vertical) over descriptors [first, first + B) and [first + B, first + 2B) of P.rg;
  // ops slot: where their plan indices go in P.rg.ops
  void resample_ragged(Plan& P, int B, int first, int slot);
  // i2it_op_resize_u8_ragged: x[i] [hw_in] -> out[i] [hw_out], with tables and intermediates sized by this call
  void resize_ragged_op(Plan& P, const void* const* x, const int* hw_in, void* const* out, const int* hw_out, int n, int max_side);
  void copy_channels(Plan& P, const Act& src, const Act& dst_slice);
  Act replicate_image(Plan& P, const Act& src, int n);               // [1,H,W,C] -> [n,H,W,C], every image a copy of src
  // V^T[b] = Wv X[b]^T (+ row bias): returns [B][C][ldv] as an Act with N=B,H=1,W=C,ld=ldv (C field = Ntok)
  Act vt_proj(Plan& P, const Act& x_tokens, int B, int ntok, const PW& wv);
  // attention core on projected operands; q/k are column slices of token matrices; returns [B*Nq, heads*d]
  Act attention(Plan& P, const Act& q, const Act& k, const Act& vt, int B, int Nq, int Nk, int heads, int d,
                int kv_batch);
  Act flash_attention(Plan& P, const Act& q, const Act& k, const Act& vt, int B, int Nq, int Nk, int heads, int kv_batch,
                      bool causal = false);
  Act flash_attention512(Plan& P, const Act& q, const Act& k, const Act& vt, int B, int Nq, int Nk, int kv_batch);
  bool use_flash = true;

  // ---- weights ----
  bool has(const std::string& key) const;
  const WT& raw(const std::string& name, const char* what) const;   // accepts X.what or X.base_layer.what
  // skip_scale: scaled by the skip-conv gamma; bias_add: key of an fp32 vector added to the bias (a master tensor, or a
  // temb_bias output)
  PW prep(const std::string& cache_key, const std::vector<std::string>& names, bool geglu = false,
          bool skip_scale = false, const std::string& bias_add = "");
  PW prep_twin(const std::string& pre, const std::string& cur);     // blended at the fold's twin_r
  PW prep_im2col3(const std::string& name);
  PW prep_identity(int n);                                          // [n][n] identity as a 1x1 'weight'
  PW prep_subpixel(const std::string& name);                       // 16 pre-summed 2x2 taps for upsample2x+conv3x3
  Act conv_up2x(Plan& P, const Act& x, const PW& wsub, const Act* x2, const PW* w2, bool gn_out = false);                        // 3x3 conv over 3 channels as a K=32 single-tap GEMM
  NormW norm(const std::string& name);
  std::string temb_bias(const std::string& resnet_prefix);          // time_emb_proj(silu(emb)) at t=999: its prepared_f32_ key
  void free_prepared();
  void flush_prep();                                                // run all pending preparation jobs (4-5 launches)
  int prep_launches_ = 0;

  // ---- model graph ----
  // shared_input: the encoder runs on one image and the posterior sample at batch B from its moments
  Act build_vae_encoder(Plan& P, const std::string& vp, int B, int H, int W, std::vector<Act>& skips,
                        const U8View* u8_in = nullptr, bool shared_input = false);
  Act build_unet(Plan& P, const Act& z, int text_batch, bool text_cached);
  void build_text_kv(struct TextKV& T);
  std::vector<std::string> xformer_prefixes() const;
  void build_vae_decoder(Plan& P, const std::string& vp, const Act& dec_in, std::vector<Act>& skips);
  Act vae_resnet(Plan& P, const std::string& p, const Act& x, const Act* skip = nullptr, const PW* skip_w = nullptr,
                 bool gn_next = true);
  Act vae_attn(Plan& P, const std::string& p, const Act& x);
  // `out`: write the block's output into this view (a channel slice of a pre-allocated concat buffer) instead of a new tensor
  Act unet_resnet(Plan& P, const std::string& p, const Act& x, bool gn_next = false, const Act* out = nullptr);
  Act unet_xformer(Plan& P, const std::string& p, const Act& x, int heads, int text_batch, bool gn_next = false,
                   const Act* out = nullptr);
  // keep_stages >= 1: the named checkpoints (skip0, latent, model_pred, ...); keep_stages >= 2 also every layer output under its
  // state-dict prefix (mark_layer), for the per-layer audit of tests/layer_audit.py.  Marks hold tensors; they add no launches.
  void mark(Plan& P, const std::string& name, const Act& a) { if (cfg.keep_stages) keep_stage(P, name, a); }
  void mark_layer(Plan& P, const std::string& name, const Act& a) { if (cfg.keep_stages >= 2) keep_stage(P, name, a); }
  void keep_stage(Plan& P, const std::string& name, const Act& a) {
    if (!P.stages.count(name)) P.stage_order.push_back(name);
    P.stages[name] = a;
  }

  template <typename F> void add_op(Plan& P, F&& f, const char* kind = "misc", double flops = 0, double bytes = 0,
                                    const std::string& shape = "") {
    P.ops.emplace_back(std::forward<F>(f));
    OpMeta m; m.kind = kind; m.flops = flops; m.bytes = bytes; m.shape = shape;
    P.meta.push_back(m);
  }
  // encodes the tensor maps and appends the launch
  // sel: a selecting launch (tapgemm_sel_kernel: tapgemm_kernel's body with each tile's weight set chosen by its image); x / x2
  // are the alternative maps of B and the second source's B (of A when sel->sel_a), and sel's dir / bias / dim / div are set
  // by the caller
  struct SelSpec { TmapSpec x, x2; TapGemmSel s; };
  void launch_gemm(Plan& P, const TmapSpec& sa, TmapSpec sb, const TapGemmParams& p, bool out_from_io, const char* kind,
                   double k_valid, double bytes, const TmapSpec* sa2 = nullptr, const TmapSpec* sb2 = nullptr,
                   const SelSpec* sel = nullptr);
  // launch_gemm for a single-tap GEMM over 128-row tiles of [batch][heads][M] rows (V^T projection, attention QK and PV):
  // fills p's tile space, N, BN (bn 0: plan_bn's choice), n_tiles, kchunks (K-wide), ocol, err and sb's 64 x BN box.  A's
  // head and image coordinates advance by a_step per tile, B's by b_head and b_img (0: one operand for every head / image).
  // p brings the output, its strides, out_fp32, alpha and the bias.
  void launch_rows(Plan& P, const TmapSpec& sa, TmapSpec sb, TapGemmParams p, int M, int heads, int batch, int a_step,
                   int b_head, int b_img, int N, int K, int bn, const char* kind, double k_valid, double bytes,
                   const SelSpec* sel = nullptr);
  bool use_idres = true, use_pdl = false, trace_on = false, use_tmaout = true, use_gnepi = true, use_splitk = true, use_catfuse = true, use_ostg2 = true, use_lean = true, sync_each = false;
  bool tma_eligible(const TapGemmParams& p, bool out_from_io) const;
  std::string profile_json(int reps, cudaStream_t st);
  void dump_trace(Plan& P, cudaStream_t st);
  int pick_bn(long long m_tiles, int N, int step) const;   // step 64 / 128: BN restricted to multiples (TMA-store rounds)
  // pick_bn, or the forced width of i2it_debug_tapgemm_override in a diagnostic op plan
  int plan_bn(const Plan& P, long long m_tiles, int N, int step) const;
  int dbg_bn = 0, dbg_stages = 0, dbg_grid = 0;            // i2it_debug_tapgemm_override (0: the engine's choice)

  int* d_err = nullptr;      // device alias of a mapped host word written by the tapgemm watchdog
  int* err_host_ = nullptr;
  cudaStream_t gstream_ = nullptr;          // graphs are captured/replayed here (capture is illegal on the legacy stream)
  cudaEvent_t ev_in_ = nullptr, ev_out_ = nullptr;
  void check_device_error();
  int graph_captures = 0;                   // CUDA graphs captured since create (i2it_debug_graph_captures)

 private:
  std::unordered_map<std::string, WT> w_;
  std::unordered_map<std::string, float> adapter_scale_;
  float lw_unet_ = 1.f, lw_vae_ = 1.f, skip_gamma_ = 1.f, twin_r_ = -1.f;
  bool finalized_ = false;
  bool folded_ = false;                                     // finalized at least once
  std::unordered_map<std::string, PW> prepared_;
  std::unordered_map<std::string, float*> prepared_f32_;
  std::vector<void*> prep_allocs_;
  float* emb_act_ = nullptr;
  std::vector<PrepJob> pending_jobs_;
  std::vector<GemvJob> pending_gemv_[3];
  long long pending_blocks_ = 0;
  // device job tables of flush_prep (three GEMV stages, the preparation jobs): reused, grown when a flush needs more
  struct JobTable { void* p = nullptr; size_t cap = 0; };
  JobTable job_tables_[4];
  void* upload_jobs(int table, const void* jobs, size_t bytes);
  // ---- refold state ----
  std::vector<Recipe> recipes_;                             // every prepared weight's recipe, in creation order
  long long recording_ = -1;                                // index of the recipe being run: fill_fold & co. record into it
  std::set<std::string> dirty_w_;                           // masters registered since the last fold
  std::map<std::string, std::vector<int64_t>> fold_shapes_; // every master's shape at the last fold
  std::unordered_map<std::string, float> fold_adapter_scale_;
  std::vector<void*> retired_;                              // replaced masters plans may still read: freed by finalize
  std::vector<std::string> refold_touched_;                 // the last refold's rebuilt recipes
  long long refold_jobs_ = 0, refold_gemv_jobs_ = 0;
  double refold_bytes_ = 0;
  void add_recipe(const std::string& key, std::function<void()> emit);
  void run_recipe(size_t i);
  const WT& src(const std::string& name, const char* what);   // raw() that records the read in the running recipe
  const float* f32_input(const std::string& key);             // a master tensor or a prepared fp32 vector, recorded
  float fold_input(FoldInput which);                          // a fold scalar, recorded
  void snapshot_fold();
  void fill_fold(PrepJob& j, const std::string& name, float c0 = 1.f, const std::string& other = "", float c1 = 0.f);
  void push_job(PrepJob& j);
  void push_bias_job(float* out, const float* b, const float* add, int cout, int row_off, int half, float c0 = 1.f,
                     const float* b1 = nullptr, float c1 = 0.f);
  std::map<int, std::unique_ptr<struct TextKV>> textkv_;   // by text_batch
  std::map<int, std::unique_ptr<Plan>> textenc_;            // CLIP text tower plans, by batch
  Arena arena_;                                             // declared before plans_: outlives them
  int max_plans_ = 0;
  unsigned long long tick_ = 0;
  int plan_builds_ = 0, plan_evictions_ = 0;
  void sync_plans();                                        // gstream_ and the device: before a plan dies or memory unmaps
  // down to max_plans_, never the last-run plan; keep_last: the last forward's workspace bytes keep their contents
  void evict_lru(const Plan* also_keep = nullptr, bool keep_last = true);
  void trim_arena(bool keep_last);                          // unmap what no resident plan needs
  std::map<std::vector<int>, std::unique_ptr<Plan>> plans_;
  // run a forward plan on `st`: replay (or capture) its graph, or launch its ops; `before` is enqueued ahead of the first
  // launch on the stream they run on
  void run(Plan* P, const IO& io, cudaStream_t st, const std::function<void(cudaStream_t)>& before = nullptr);
  // ragged calls: host tables, and the pinned blob one async copy per call moves into the plan's descriptor buffer; the blob
  // is rewritten only after rs_ev_ says the previous copy has read it
  RsTableCache rs_tables_;
  char* rs_blob_ = nullptr;
  size_t rs_blob_cap_ = 0;
  cudaEvent_t rs_ev_ = nullptr;
  size_t stage_ragged(const RsCall& c, size_t cap);     // fills the blob; returns its byte count
  // mixed-direction forwards: the pinned copy of the call's directions one async copy moves into Plan::dir (dir_ev_ says
  // the previous copy has read it); mixed_dir_ is the plan's array while a mixed plan is being built (prep / norm pair the
  // vae. weights with their vae_b2a. twins then)
  int* dir_blob_ = nullptr;
  int dir_blob_cap_ = 0;
  cudaEvent_t dir_ev_ = nullptr;
  const int* mixed_dir_ = nullptr;
  std::function<void(cudaStream_t)> stage_dirs(Plan* P, const int* dirs, int B);
  Plan* last_plan_ = nullptr;
  Plan* last_text_plan_ = nullptr;   // the plan of the last encode_text (its stages: i2it_text_stage_names)
  Act text_;                     // staged text embedding while a UNet plan is being built
  TextKV* text_kv_ = nullptr;    // ... or the cached cross-attention operands (text_emb == NULL forwards)

  float adapter_weight(const std::string& name, const std::string& adapter);
  void* dmalloc(size_t bytes);
};

}  // namespace i2it

/* libi2it — C ABI of the H100-native one-step image-translation path
 *
 *     VAE.encode -> one SD-Turbo UNet step (t = 999) -> DDPM closed form -> VAE.decode
 *
 * This is the boundary the reference's Python wrappers would bind (via ctypes; see INTEGRATION.md) in
 * place of the four diffusers calls at
 *     src/pix2pix_turbo.py:198-203   (deterministic)   and :204-218 (stochastic)
 *     src/cyclegan_turbo.py:199-207  (forward_with_networks)
 * i.e.  vae.encode(x).latent_dist.sample()*sf ; unet(z, 999, text).sample ; sched.step(...).prev_sample ;
 *       vae.decode(x0/sf).sample.clamp(-1,1)
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross this header.
 *   - every function returns 0 on success, non-zero on failure; i2it_last_error() gives the message.
 *     Nothing throws across the ABI.
 *   - the caller owns inputs, outputs and the CUDA stream; the library owns folded weights + workspace.
 *   - a handle is NOT thread-safe: one handle per (device, stream).  Work is enqueued asynchronously on
 *     the caller's stream (the caller synchronises), except where noted.
 *   - activations at the boundary are NCHW contiguous in the handle's dtype (fp16 or bf16), exactly what
 *     the reference passes to / receives from vae.encode / vae.decode after `.half()`.
 */
#ifndef I2IT_H
#define I2IT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct i2it_handle i2it_handle;

enum { I2IT_F16 = 0, I2IT_BF16 = 1, I2IT_F32 = 2 };
enum { I2IT_PIX2PIX = 0, I2IT_CYCLEGAN = 1 };
enum { I2IT_A2B = 0, I2IT_B2A = 1 };
/* uint8 input transforms of a uint8 forward (what the reference CLIs do on the host before the forward) */
enum { I2IT_IN_UNIT = 0,        /* F.to_tensor(img): u8/255                       src/inference_paired.py:50      */
       I2IT_IN_NORMALIZE = 1,   /* ToTensor + Normalize([0.5],[0.5])              src/inference_unpaired.py:45-47 */
       I2IT_IN_SKETCH = 2 };    /* (F.to_tensor(img) < 0.5).float()               src/inference_paired.py:56-57   */

/* Network hyper-parameters (HF config.json of stabilityai/sd-turbo; i2it_default_config fills them in). */
typedef struct i2it_config {
  int dtype;                 /* I2IT_F16 | I2IT_BF16 : activation + weight dtype, fp32 accumulation        */
  int model_kind;            /* I2IT_PIX2PIX | I2IT_CYCLEGAN                                               */
  int device;                /* CUDA device ordinal                                                        */
  int unet_channels[4];      /* 320, 640, 1280, 1280                                                       */
  int unet_heads[4];         /* 5, 10, 20, 20 (head_dim is 64 everywhere)                                  */
  int cross_dim;             /* 1024                                                                       */
  int temb_dim;              /* 1280                                                                       */
  int vae_channels[4];       /* 128, 256, 512, 512                                                         */
  float scaling_factor;      /* 0.18215                                                                    */
  int keep_stages;           /* 1: keep named intermediate tensors readable via i2it_read_stage (tests);   */
                             /* 2: also every layer output (per-layer audit; needs memory for all of them) */
  int use_cuda_graph;        /* 1: replay the forward as one CUDA graph when shapes and pointers repeat    */
  int text_heads;            /* CLIP text tower: attention heads (16; head_dim must be 64); 0 = hidden/64  */
  int text_act;              /* CLIP text tower MLP activation: 0 = gelu (SD-Turbo), 1 = quick_gelu        */
} i2it_config;

/* Fill `cfg` with the SD-Turbo configuration. */
int i2it_default_config(i2it_config* cfg);

/* Create / destroy an engine.  Replaces AutoencoderKL/UNet2DConditionModel construction
 * (src/pix2pix_turbo.py:36-45; cyclegan_turbo.py:115-124). */
int i2it_create(const i2it_config* cfg, i2it_handle** out);
void i2it_destroy(i2it_handle* h);
const char* i2it_last_error(const i2it_handle* h);   /* h may be NULL: last error of a failed create */

/* Register one tensor of the state dict.  `key` is "<model>.<diffusers key>" with model in
 * {unet, vae, vae_b2a}; peft spellings ("X.base_layer.weight", "X.lora_A.<adapter>.weight",
 * "X.lora_B.<adapter>.weight") are accepted as-is.  `data` may be a host or device pointer
 * (is_device); dtype is I2IT_F32/F16/BF16.  The engine keeps an fp32 device copy (synchronous).  A key registered again
 * with the same shape is copied into its existing copy after the handle's work drains (plans read some tensors, such as
 * the norm scales, directly), so i2it_refold_weights can fold it in place.  A key registered again with another shape gets
 * a new copy; the old one stays allocated until the next i2it_finalize_weights or i2it_destroy, because resident plans may
 * still read it.
 * Replaces load_state_dict at src/pix2pix_turbo.py:66-78, cyclegan_turbo.py:162-190. */
int i2it_set_weight(i2it_handle* h, const char* key, const void* data, const int64_t* shape, int ndim,
                    int dtype, int is_device);

/* LoRA scale (lora_alpha / r) of an adapter name ("default", "vae_skip", "default_encoder", ...);
 * replaces peft LoraConfig scaling (src/pix2pix_turbo.py:141-151, cyclegan_turbo.py:66-72). */
int i2it_set_adapter_scale(i2it_handle* h, const char* adapter, float alpha_over_r);

/* Fold LoRA into the base weights (W' = W + s*w*B@A in fp32, one rounding), blend TwinConv
 * (W = (1-r) W_pre + r W_cur), scale the skip convs by gamma, fold the t=999 time embedding into
 * conv1 biases, re-lay out for the kernels.  Callable again when the runtime weights change
 * (stochastic mode: unet.set_adapters(["default"],[r]), set_weights_and_activate_adapters(vae,...,[r]),
 * decoder.gamma = r, conv_in.r = r  — src/pix2pix_turbo.py:206-217).
 * lora_weight_* multiply the adapter scales of the UNet / VAE adapters; twin_r < 0 means "no TwinConv blend
 * requested" (error if the state dict has a TwinConv). */
int i2it_finalize_weights(i2it_handle* h, float lora_weight_unet, float lora_weight_vae, float skip_gamma,
                          float twin_r);

/* Fold again with new scalars, or after i2it_set_weight re-registered tensors of an unchanged shape, writing the prepared
 * weights in place.  Synchronous: it waits for the handle's work, rebuilds only the prepared weights whose fold inputs
 * changed (a scalar they read, or a tensor re-registered since the last fold) in one preparation launch plus at most three
 * time-embedding GEMV launches, and waits for them.  Every prepared weight is then bit-identical to what
 * i2it_finalize_weights with the same arguments would write.
 * Kept: every forward plan and its CUDA graphs, the workspace arena, the text-tower plans.  Dropped: the i2it_set_text
 * cache (the projections carry the LoRA scale), with the same error as after i2it_finalize_weights.
 * Refused, with nothing changed, when the handle was never finalized, when twin_r < 0 differs from twin_r < 0 at the last
 * fold, or when a tensor was added, or re-registered with another shape, since the last fold: those need
 * i2it_finalize_weights. */
int i2it_refold_weights(i2it_handle* h, float lora_weight_unet, float lora_weight_vae, float skip_gamma, float twin_r);

/* Bytes of device workspace the engine holds for a (batch, H, W) forward: the last forward's plan when it has this shape,
 * else the plan is built.  Every buffer grows linearly in H*W (the VAE attention runs fused above 8192 tokens).
 * The count is the plan's own need, transient plus persistent bytes: its transient part lives in the arena the handle's
 * forward plans share (i2it_memory_stats_get).  Building a plan here never evicts the last forward's plan. */
int i2it_workspace_bytes(i2it_handle* h, int batch, int H, int W, size_t* bytes);

/* Keep at most max_plans image-forward plans (0 = no limit, the default); the least recently run plan is evicted first and
 * rebuilt, bit-identically, when its key returns.  The plan of the last forward is never evicted.  Evicting synchronises
 * the device. */
int i2it_set_max_plans(i2it_handle* h, int max_plans);

/* Drop every image-forward plan and its graphs and unmap the shared workspace.  Prepared weights, the i2it_set_text cache and
 * the text-tower plans are kept.  Synchronous. */
int i2it_release_plans(i2it_handle* h);

typedef struct i2it_memory_stats {
  size_t arena_bytes;        /* physical bytes mapped for the transient workspace shared by all forward plans */
  size_t plan_bytes;         /* persistent per-plan bytes, summed over resident plans */
  int plans;                 /* resident image-forward plans */
  int plan_builds, plan_evictions;   /* counters since create */
} i2it_memory_stats;
int i2it_memory_stats_get(i2it_handle* h, i2it_memory_stats* s);

/* Test hook: memset every mapped arena byte to `value` (synchronous).  A forward must not read transient workspace it did not
 * write itself, so poisoning between forwards must leave every output unchanged. */
int i2it_debug_poison_workspace(i2it_handle* h, int value);

/* LANCZOS resize geometry of a uint8 forward (i2it_forward_desc.geometry): what the reference CLIs do with PIL on the host
 * around the forward (src/inference_unpaired.py:40-45,53; src/inference_paired.py:38-41), bit-exact with
 * Image.resize(size, Image.LANCZOS).  The caller's image [batch, in_H, in_W, 3] is resized to resize_H x resize_W; the network
 * runs on the H x W window at (crop_y, crop_x) of it (transforms.CenterCrop); its output image is resized to out_H x out_W.
 * All sizes are rows x columns. */
typedef struct i2it_resize_desc {
  int in_H, in_W;
  int resize_H, resize_W;
  int crop_y, crop_x;
  int out_H, out_W;
} i2it_resize_desc;

/* One image forward (i2it_forward).  Plain fields; zero (or NULL) means unused.  The accepted requests, by which input,
 * geometry, shared_input and directions they set (the output pointer matches the input: out, out_u8 or out_u8_list):
 *
 *   request              input              geometry                 shared_input   directions
 *   plain                x                  NULL                     0              NULL
 *   uint8                x_u8               NULL                     0              NULL
 *   uint8 resize         x_u8               one                      0              NULL
 *   variations           x [1]              NULL                     1              NULL
 *   uint8 variations     x_u8 [1]           one or NULL              1              NULL
 *   ragged               x_u8_list          batch, with max_side     0              NULL
 *   mixed                x                  NULL                     0              host array, no noise_map
 *   ragged mixed         x_u8_list          batch, with max_side     0              host array, no noise_map
 *
 * Every other combination is rejected before any launch and without building a plan: two inputs or outputs of different
 * kinds, a geometry on the NCHW x, shared_input with x_u8_list or with directions, directions with x_u8, and a noise_map
 * with directions.
 *
 * Plain.  All pointers are DEVICE pointers in the handle dtype, NCHW contiguous:
 *   x        [batch, 3, H, W]          control image / input image (fed to the VAE as is)
 *   text_emb [text_batch, 77, cross]   CLIP hidden states (text_batch is 1 or batch)
 *   eps      [batch, 4, H/8, W/8]      the posterior noise of latent_dist.sample()
 *   noise_map[batch, 4, H/8, W/8]      nullable; non-NULL selects the stochastic blend with r
 *   out      [batch, 3, H, W]          clamp(-1,1) image
 *   out_latent [batch, 4, H/8, W/8]    nullable; x_denoised (the "output latents")
 * direction selects vae (A2B) or vae_b2a (B2A) for I2IT_CYCLEGAN; ignored for I2IT_PIX2PIX.
 * text_emb may be NULL: the cross-attention K / V^T cached by the last i2it_set_text(…, text_batch) are used (one prompt,
 * many images: the reference re-projects the 77 text tokens in all 16 cross-attention layers on every forward).
 * The DDPM step follows the wrapper the handle was created for: fp32 with one rounding for I2IT_PIX2PIX
 * (src/pix2pix_turbo.py:162,200-201: 1-D timesteps), three activation-dtype roundings for I2IT_CYCLEGAN
 * (src/cyclegan_turbo.py:205: 0-dim timestep).
 * H and W must be multiples of 8.  4032x3024 (12 MP) at batch 1 runs on one 80 GB H100 (measured workspace and time
 * in DESIGN section 8).  Each forward key (batch, H, W, direction, text mode, io mode, resize geometry) has its own plan.
 * The transient workspace of all of a handle's forward plans is one shared arena, sized by the largest resident plan;
 * each plan also holds a few small persistent buffers of its own.  Plans stay until i2it_finalize_weights,
 * i2it_release_plans or an eviction under i2it_set_max_plans; an evicted plan is rebuilt, bit-identically, when its key
 * returns.
 *
 * uint8.  The plain forward with a uint8 HWC boundary: x_u8 [batch, H, W, 3] and out_u8 [batch, H, W, 3] are device
 * pointers.  Input transform `in_mode` (I2IT_IN_*) and the output `ToPILImage()(out*0.5+0.5)` (src/inference_paired.py:72,
 * src/inference_unpaired.py:53; three activation-dtype roundings then truncation to uint8) are fused into the first /
 * a trailing kernel, so a caller moves 3 bytes per pixel each way instead of 2 x 3 x sizeof(half).
 *
 * uint8 resize.  The uint8 forward with a resize geometry: x_u8 [batch, in_H, in_W, 3] -> out_u8 [batch, out_H, out_W, 3]
 * (device pointers); eps / noise_map / out_latent have the network size H x W (multiples of 8).  Each resize is one or two
 * launches (horizontal pass if the width changes, then vertical if the height changes; none for an unchanged size), captured
 * in the same CUDA graph; the coefficient tables are computed on the host once per plan.  The geometry is part of the plan
 * key.  Rejected before any launch: non-positive sizes, or a crop window outside the resized image.
 *
 * Variations.  n = batch variations of ONE image in one forward: the plain forward with x [1, 3, H, W] and every other
 * operand at batch n (eps [n, 4, H/8, W/8], noise_map [n, 4, H/8, W/8] or NULL, out [n, 3, H, W], out_latent [n, 4, H/8, W/8]
 * or NULL, text_emb [text_batch, 77, cross] with text_batch 1 or n, or NULL for the i2it_set_text cache).  The VAE encoder
 * runs once, at batch 1: its moments feed every image's posterior sample (each with its own eps and noise_map rows), and
 * each of its four skips is replicated to batch n right before the decoder conv that reads it.  Output image i is
 * bit-identical to image i of the plain forward on the image repeated n times (and to a batch-1 forward of it with eps[i],
 * noise_map[i]): the encoder of a batch computes each image alone.  A variations key is its own plan (n = 1 is the plain
 * batch-1 plan).  Rejected before any launch: n < 1, text_batch not 1 or n, and whatever the plain forward rejects.
 * Replaces the one-forward-per-seed loop of gradio_sketch2image.py.
 *
 * uint8 variations.  Variations with the uint8 HWC boundary of the uint8 / uint8 resize forwards: x_u8 [1, in_H, in_W, 3]
 * -> out_u8 [n, out_H, out_W, 3].  geometry is one resize geometry or NULL (then in_H = out_H = H, in_W = out_W = W); the
 * input resize passes and packing run at batch 1, the output conversion and resize at batch n.  Rejected before any launch:
 * what the variations and uint8 resize forwards reject.
 *
 * Ragged.  n = batch uint8 images of their own sizes through one forward at batch n on an H x W network:
 *   x_u8_list[i]   [geometry[i].in_H, geometry[i].in_W, 3]    device pointers, one per image
 *   out_u8_list[i] [geometry[i].out_H, geometry[i].out_W, 3]  device pointers, one per image
 *   geometry[i]    image i's resize geometry (its crop window is H x W)
 *   eps / noise_map / out_latent [n, 4, H/8, W/8], text_emb [text_batch, 77, cross] or NULL, as in the uint8 forward.
 * Each image goes through exactly the passes of the uint8 resize forward, so output i is byte-equal to a batch-1
 * uint8 resize forward of image i with eps[i] and noise_map[i].  A dimension that does not change is an identity pass,
 * so every call makes two resize launches per side.
 * The plan is keyed by (n, H, W, direction, text mode, max_side) and by no image size: max_side is a capacity that
 * every in_*, resize_* and out_* size of the call must not exceed, and its buffers are sized by it.  Each call
 * builds its descriptors and coefficient tables on the host (tables cached per size pair) and copies them to the plan with
 * one asynchronous copy ahead of the first launch.  The image pointers live in those descriptors, not in the captured
 * graph, so any mix of sizes and pointers replays one graph.
 * Rejected before any launch: n < 1, a NULL array or image pointer, non-positive sizes, a crop window outside its resized
 * image, a dimension above max_side (or max_side <= 0), and whatever the uint8 forward rejects.
 *
 * Mixed.  A CycleGAN batch that mixes both directions in one forward: image i goes through vae (directions[i] == I2IT_A2B)
 * or vae_b2a (I2IT_B2A).  directions is a HOST array of batch values; every other operand is the plain forward's (there is
 * no noise_map: CycleGAN has none), with text_batch 1 or batch and text_emb NULL for the i2it_set_text cache.  The UNet, the
 * DDPM step and the latent sampling are the same for both directions; every VAE launch that reads weights (the convs,
 * quant_conv / post_quant_conv, the attention's projections and the GroupNorm applies) takes each 128-row tile's or each
 * image's weights from its direction, in the same accumulation order, so output image i is byte-equal to image i of a
 * single-direction forward in directions[i] (same x, eps, text).  One plan per (batch, H, W, text mode) serves every
 * mix: the directions are copied to the plan ahead of the first launch, and its CUDA graph reads them there.  It has the
 * launch count and tile geometry of the single-direction plan.
 * Accepted sizes: those whose every VAE tile holds rows of one image (i2it_mixed_size_check), e.g. 256x256, 512x512,
 * 512x768 and 1024x1024; 1280x720 is refused (its (H/8)(W/8) = 14400 latent pixels are not a multiple of 128).
 * Rejected before any launch, and without building a plan: a pix2pix handle, a NULL directions array, a value other
 * than 0 or 1, a refused size, and whatever the plain forward rejects.
 *
 * Ragged mixed.  The ragged forward with a direction per image (host array of n values, as the mixed forward): uploads of
 * any size and both directions through one plan.  Output i is byte-equal to the batch-1 uint8 resize forward of upload i in
 * directions[i].  Rejected before any launch: what the ragged and mixed forwards reject. */
typedef struct i2it_forward_desc {
  int batch, H, W;
  int direction;                       /* I2IT_A2B | I2IT_B2A (other values are refused); unused with directions */
  const int* directions;               /* host array of batch directions (mixed requests), or NULL */
  int shared_input;                    /* 1: variations of one input image */
  const void* x;                       /* NCHW input in the handle dtype */
  const void* x_u8;                    /* uint8 HWC input */
  const void* const* x_u8_list;        /* batch uint8 HWC inputs (ragged requests) */
  int in_mode;                         /* I2IT_IN_* of a uint8 input */
  const i2it_resize_desc* geometry;    /* NULL, one geometry, or batch geometries (ragged requests) */
  int max_side;                        /* capacity of a ragged plan */
  const void* text_emb; int text_batch;
  const void* eps; const void* noise_map; float r;
  void* out;                           /* NCHW output in the handle dtype */
  void* out_u8;                        /* uint8 HWC output */
  void* const* out_u8_list;            /* batch uint8 HWC outputs (ragged requests) */
  void* out_latent;
} i2it_forward_desc;

/* The fused hot path: run the forward `d` describes on `stream` (a cudaStream_t). */
int i2it_forward(i2it_handle* h, const i2it_forward_desc* d, void* stream);

/* Project and cache the cross-attention operands of a prompt: K = to_k(text_emb), V^T = to_v(text_emb)^T for every
 * transformer block (32 small launches, enqueued on `stream`).  text_emb [text_batch, 77, cross] device pointer in the
 * handle dtype; it is consumed before the call returns control to the stream order (the caller may reuse the buffer after
 * the stream reaches this point).  Must be called again after i2it_finalize_weights or i2it_refold_weights (the projections carry the LoRA
 * scale).
 * Replaces the per-forward `attn2.to_k / attn2.to_v` calls under unet(...) at src/pix2pix_turbo.py:199. */
int i2it_set_text(i2it_handle* h, const void* text_emb, int text_batch, void* stream);

/* The CLIP text tower on the engine (SURVEY.md section 8f #1): tokens [batch, 77] int32 (device) -> last_hidden_state
 * [batch, 77, hidden] (device, handle dtype), i.e. `self.text_encoder(tokens)[0]` of src/pix2pix_turbo.py:190-196
 * and cyclegan_turbo.py:251-253.  Needs the "text_encoder.<transformers CLIPTextModel key>" tensors registered with
 * i2it_set_weight.  Enqueued on `stream` (no CUDA graph: a prompt is encoded once and cached by the caller).
 * The kernels read batch * 77 ids and write batch * 77 rows: the caller owns both sizes, and every id must lie in
 * [0, vocab) (the Python binding checks both before the launch). */
int i2it_encode_text(i2it_handle* h, const int32_t* tokens, int batch, void* out, void* stream);

/* Whether a mixed-direction forward accepts the network size H x W: 0 if it does, 1 if not, with the reason (naming the
 * rule) in msg (cap bytes, NUL-terminated; msg may be NULL).  The rule: (H/8)(W/8) is a multiple of 128 (the VAE
 * attention's token launches), and on every VAE map level H/2^k x W/2^k the conv's 128-row tile box covers pixels of one
 * image.  No GPU needed. */
int i2it_mixed_size_check(int H, int W, char* msg, size_t cap);

/* Number of kernel launches one forward of this shape issues (for bench accounting): the plan the last forward used if it
 * has this shape, else the plan with the text embedding passed inline. */
int i2it_launch_count(i2it_handle* h, int batch, int H, int W, int direction, int* launches);

/* Kernel launches spent on weight preparation (LoRA fold / TwinConv / re-layout / time embedding) since the handle was
 * created: a job table makes this 4-5 per finalize+plan instead of one to four per tensor. */
int i2it_prep_launch_count(i2it_handle* h, int* launches);

/* Host-side check of the division-free tile decode the GEMM kernels use (csrc/tapgemm.cuh: make_magic / fast_div): returns the
 * quotient the device computes for x / d (magic made for dividends <= max_dividend, 32-bit high multiply), or -1 when the host
 * would refuse that tile space.  No GPU needed: lets the CPU test suite pin the index arithmetic bit for bit. */
long long i2it_debug_fast_div(long long max_dividend, int d, int x);

/* Host-side tables of one LANCZOS resize pass from in_size to out_size samples, exactly as the resample kernels get them:
 * bounds [out_size][2] = (first input index, number of taps), coeffs [out_size][ksize] 22-bit fixed-point weights (zero past
 * the taps).  Either pointer may be NULL; coeffs must hold `cap` ints.  Returns ksize, or -1 for bad sizes or a short buffer.
 * No GPU needed. */
int i2it_debug_resample_coeffs(int in_size, int out_size, int* bounds, int* coeffs, int cap);

/* Host-side sizing of a ragged forward (i2it_forward_desc) on n geometries: *used = coefficient-table ints the call
 * uploads, *bound = the ints its plan reserves for any call with this n, H, W and max_side.  Returns -1 for a geometry the
 * forward would reject.  No GPU needed. */
int i2it_debug_ragged_tables(const i2it_resize_desc* g, int n, int H, int W, int max_side, long long* used, long long* bound);

/* CUDA graphs the handle has captured since create (a replay captures none). */
int i2it_debug_graph_captures(i2it_handle* h, int* captures);

/* What the last i2it_refold_weights rebuilt, as JSON: {"recipes": [prepared-weight keys, in fold order], "jobs": preparation
 * jobs, "gemv_jobs": time-embedding GEMV jobs, "bytes": algorithmic bytes those jobs read and write}. */
int i2it_debug_refold_info(i2it_handle* h, char* json, size_t cap);

/* Per-launch device timing of the plan the LAST forward used: runs it `reps` more times with CUDA events around
 * every launch and writes a JSON array [{"i","kind","ms","flops","bytes","shape"}...] (algorithmic flops/bytes per
 * launch) into `json`.  Synchronous.  This is what bench.py's roofline numbers are computed from. */
int i2it_profile(i2it_handle* h, int reps, char* json, size_t cap, void* stream);

/* Named intermediate tensors of the LAST forward (needs cfg.keep_stages): copies the stage as fp32 NCHW
 * into dst (device pointer) and reports its dims.  Synchronous.  Names: "skip0".."skip3", "moments",
 * "latent", "model_pred", "dec_in", "pre_out"... (see DESIGN.md). */
int i2it_read_stage(i2it_handle* h, const char* name, float* dst, size_t dst_elems, int dims[4]);

/* Every stage of the LAST forward in build order, as JSON [{"name","dims":[N,C,H,W]}...].  With cfg.keep_stages = 2
 * the forward also keeps every layer output under its state-dict prefix ("unet.down_blocks.0.resnets.0.conv1", ...;
 * DESIGN.md section 6 lists the names); the output image is bit-identical to keep_stages = 0.  Synchronous. */
int i2it_stage_names(i2it_handle* h, char* json, size_t cap);

/* Every stage of the LAST i2it_encode_text, in the format of i2it_stage_names.  With cfg.keep_stages = 2 the text tower
 * keeps every layer output under its transformers state-dict prefix ("text_encoder.text_model.embeddings",
 * "text_encoder.text_model.encoder.layers.0.self_attn.qk", ...; DESIGN.md section 6); i2it_read_stage reads a
 * "text_encoder."-prefixed name from this plan.  The encoded output is bit-identical to keep_stages = 0.  Synchronous. */
int i2it_text_stage_names(i2it_handle* h, char* json, size_t cap);

/* Cache keys of every prepared (folded, re-laid-out) weight, as a sorted JSON array of strings.  Synchronous. */
int i2it_prepared_keys(i2it_handle* h, char* json, size_t cap);

/* Copies the prepared weight `key` exactly as the kernels read it: w = [taps][rows][cin_pad] 16-bit elements of the
 * handle dtype, bias = [rows] fp32 (when the weight has one).  dims = {taps, rows, cin_pad, has_bias}.  w / bias may be
 * NULL to query dims only; host or device pointers.  Synchronous. */
int i2it_read_prepared(i2it_handle* h, const char* key, void* w, size_t w_elems, float* bias, size_t b_elems, int dims[4]);

/* ---- diagnostic single-op entry points (used by tests/ to check each kernel against the oracle) ----
 * Activations NHWC with pixel stride ld (elements); weights fp32 device pointers in PyTorch layout.
 * Every pitch an op loads through TMA must be a multiple of 8 elements (16 bytes): ldx and ld2 of the conv ops,
 * ldq / ldk / ldv of i2it_op_attention and ldx of i2it_op_vt_proj.  Any other pitch is refused before anything is launched.
 * All are synchronous on `stream`. */
/* The output is [N, Ho, Wo, Cout] (Cout/2 for GEGLU) with Ho = ceil(H / stride): an odd map is zero-padded to even
 * (as F.conv2d(stride=2, padding=1) does).  The asymmetric VAE padding needs even H and W. */
int i2it_op_conv2d(i2it_handle* h, const void* x, int N, int H, int W, int Cin, int ldx, const float* w,
                   const float* bias, int Cout, int ksize, int stride, int asym_pad, const void* residual,
                   int ldr, int act, void* out, int ldo, int out_fp32, void* stream);
/* act values of the conv ops (csrc/tapgemm.cuh TgAct) */
enum { I2IT_ACT_NONE = 0, I2IT_ACT_CLAMP1 = 1, I2IT_ACT_GEGLU = 2, I2IT_ACT_GELU = 3, I2IT_ACT_QUICKGELU = 4 };
/* Every variant of the GEMM-backed conv: i2it_op_conv2d's fields plus the ones below.  Zero-initialise unused fields.
 * LoRA adapters of the op weight are registered as "__op.conv.lora_{A,B}.<adapter>.weight" (scale: i2it_set_adapter_scale). */
typedef struct i2it_conv_desc {
  const void* x; int N, H, W, Cin, ldx;
  const float* w; const float* bias; int Cout, ksize, stride, asym_pad;
  const void* residual; int ldr;
  int act;
  void* out; int ldo, out_fp32;
  /* second source folded into the same accumulator: out += conv1x1(x2, w2); x2 [N, Ho, Wo, C2] (pixel stride ld2),
   * w2 [Cout, C2, 1, 1] fp32 */
  const void* x2; int C2, ld2; const float* w2;
  int up2x;              /* nearest-2x upsample then the 3x3 conv (sub-pixel: four parity launches); x2 at output size */
  int tokens;            /* 1x1 only: N images of H*W token rows each (GroupNorm statistics per 128-row tile) */
  /* gn_y != NULL: GroupNorm(32 groups, gn_eps, gn_gamma/gn_beta, optional SiLU) of the output into gn_y (pixel stride ldg),
   * with the statistics taken in the conv epilogue where the launch qualifies */
  void* gn_y; int ldg, gn_silu; float gn_eps; const float* gn_gamma; const float* gn_beta;
} i2it_conv_desc;
int i2it_op_conv2d_ex(i2it_handle* h, const i2it_conv_desc* d, void* stream);
/* i2it_op_conv2d_ex with a second weight set chosen per image, as a mixed-direction plan's VAE convs run: image n uses
 * (w_alt, bias_alt, w2_alt) where directions[n] == 1 (host array of d->N values, each 0 or 1) and d's weights where it is
 * 0.  bias_alt is required iff d->bias is; w2_alt NULL shares d->w2.  A GroupNorm (d->gn_y) uses d's gamma / beta for
 * every image.  Refused: a tile that would hold rows of two images (tokens: H*W not a multiple of 128). */
int i2it_op_conv2d_sel(i2it_handle* h, const i2it_conv_desc* d, const float* w_alt, const float* bias_alt, const float* w2_alt,
                       const int* directions, void* stream);
/* Launch list of the last op call, as a JSON array [{"kind","shape"}...] (GEMM shape strings carry BN, tma/tma2, gn;
 * softmax launches carry their variant 32 / 128 / long). */
int i2it_op_launches(i2it_handle* h, char* json, size_t cap);
int i2it_op_group_norm(i2it_handle* h, const void* x, int N, int HW, int C, int ldx, const float* gamma,
                       const float* beta, float eps, int silu, void* out, int ldo, void* stream);
int i2it_op_layer_norm(i2it_handle* h, const void* x, int rows, int C, int ldx, const float* gamma,
                       const float* beta, float eps, void* out, int ldo, void* stream);
/* q [B,Nq,heads*d] (ldq), k [B,Nk,heads*d] (ldk), vt [B, heads*d, ldv] (V transposed), out [B,Nq,heads*d];
 * causal (flash path, d = 64 only): query i attends keys 0..i */
int i2it_op_attention(i2it_handle* h, const void* q, int ldq, const void* k, int ldk, const void* vt, int ldv,
                      int B, int Nq, int Nk, int heads, int d, int kv_batch, int causal, void* out, int ldo,
                      void* stream);
/* V^T projection: x [B*ntok, Cin] (ldx), w [Cout, Cin] fp32, bias [Cout] (nullable) -> out [B][Cout][round_up(ntok, 8)] */
int i2it_op_vt_proj(i2it_handle* h, const void* x, int B, int ntok, int Cin, int ldx, const float* w, const float* bias,
                    int Cout, void* out, void* stream);
int i2it_op_upsample2x(i2it_handle* h, const void* x, int N, int H, int W, int C, void* out, void* stream);
/* F.interpolate(size=(Ho, Wo), mode="nearest") */
int i2it_op_upsample_to(i2it_handle* h, const void* x, int N, int H, int W, int C, int Ho, int Wo, void* out,
                        void* stream);
/* LANCZOS resize of uint8 HWC images, bit-exact with PIL: x [B, H, W, 3] -> out [B, H2, W2, 3] (device pointers).
 * The same passes as a uint8 resize forward; an unchanged size is a device copy (no launch). */
int i2it_op_resize_u8(i2it_handle* h, const void* x, int B, int H, int W, void* out, int H2, int W2, void* stream);
/* Ragged LANCZOS resize, bit-exact with PIL per image: x[i] [hw_in[2i], hw_in[2i+1], 3] -> out[i] [hw_out[2i],
 * hw_out[2i+1], 3] (device pointers).  Two launches, the passes of a ragged forward; every dimension must be <= max_side.
 * Rejected before any launch: n < 1, NULL pointers, non-positive sizes, a dimension above max_side. */
int i2it_op_resize_u8_ragged(i2it_handle* h, const void* const* x, const int* hw_in, void* const* out, const int* hw_out,
                             int n, int max_side, void* stream);
/* Test hook: force tapgemm's tile width, ring depth and persistent grid in the plans of the i2it_op_* calls made after it
 * (forward, encode_text and set_text plans never read it).  0 keeps the engine's choice.  bn replaces pick_bn's width (one of
 * 16, 32, 48, 64, 80, 96, 112, 128, 160, 192, 224, 256, at most round_up(N, 16)); launches that fix their width themselves
 * (split-K: 256, the P V GEMM: the head dim) keep it.  stages: 2 .. the ring depth the launch would get; grid: 1 .. min(tiles,
 * SMs).  Each applies to every tapgemm launch of the op; an op whose launch cannot take a value fails with the legal range. */
int i2it_debug_tapgemm_override(i2it_handle* h, int bn, int stages, int grid);

#ifdef __cplusplus
}
#endif
#endif /* I2IT_H */

// Engine implementation: weight store + load-time fold, op builders, executor.  The model graph lives in model.cu.
#include "engine.cuh"

#include <algorithm>
#include <cstdlib>

#include <nvtx3/nvToolsExt.h>   // header-only: ranges show up under Nsight tools, no-ops otherwise

namespace i2it {

static inline int ceil_div(long long a, long long b) { return static_cast<int>((a + b - 1) / b); }
static inline int round_up(int a, int b) { return (a + b - 1) / b * b; }
static inline int pow2ceil(int v) { int p = 1; while (p < v) p <<= 1; return p; }

#define DISPATCH_T(dt, ...)                                   \
  do {                                                        \
    if ((dt) == DT_BF16) { using T = __nv_bfloat16; __VA_ARGS__; } \
    else { using T = __half; __VA_ARGS__; }                   \
  } while (0)

// ---------------------------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

TmapSpec::TmapSpec(const char* what, const void* b, std::initializer_list<long long> dims,
                   std::initializer_list<long long> strides, std::initializer_list<int> boxes) : base(b) {
  std::copy(dims.begin(), dims.end(), dim);
  std::copy(boxes.begin(), boxes.end(), box);
  int i = 0;
  for (const long long s : strides) {
    const uint64_t bytes = 2ull * s;
    if (dim[i + 1] > 1 && bytes % 16 != 0)
      throw Error(std::string(what) + ": pitch " + std::to_string(s) + " elements (dimension " + std::to_string(i + 1) +
                  ") is not a multiple of 8");
    if (bytes != 0 && bytes % 16 == 0) stride[i] = bytes;
    ++i;
  }
}

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    I2IT_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    I2IT_CHECK(q == cudaDriverEntryPointSuccess && p != nullptr, "cuTensorMapEncodeTiled unavailable in this driver");
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

CUtensorMap encode_tmap(const TmapSpec& s, int dtype) {
  CUtensorMap m;
  cuuint64_t dims[5], strides[4];
  cuuint32_t box[5], es[5] = {1, 1, 1, 1, 1};
  for (int i = 0; i < 5; ++i) { dims[i] = s.dim[i]; box[i] = s.box[i]; }
  for (int i = 0; i < 4; ++i) strides[i] = s.stride[i];
  const CUtensorMapDataType dt = (dtype == DT_BF16) ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUresult r = encode_fn()(&m, dt, 5, const_cast<void*>(s.base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[512];
    snprintf(buf, sizeof buf,
             "cuTensorMapEncodeTiled failed (%d): base=%p dim=(%llu,%llu,%llu,%llu,%llu) stride=(%llu,%llu,%llu,%llu) "
             "box=(%u,%u,%u,%u,%u)", static_cast<int>(r), s.base, (unsigned long long)dims[0], (unsigned long long)dims[1],
             (unsigned long long)dims[2], (unsigned long long)dims[3], (unsigned long long)dims[4],
             (unsigned long long)strides[0], (unsigned long long)strides[1], (unsigned long long)strides[2],
             (unsigned long long)strides[3], box[0], box[1], box[2], box[3], box[4]);
    throw Error(buf);
  }
  return m;
}

// ---------------------------------------------------------------------------------------------
// workspace arena (virtual memory management entry points fetched like cuTensorMapEncodeTiled)
// ---------------------------------------------------------------------------------------------
template <typename F> static F driver_fn(const char* name) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  I2IT_CUDA(cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q));
  I2IT_CHECK(q == cudaDriverEntryPointSuccess && p != nullptr, std::string(name) + " unavailable in this driver");
  return reinterpret_cast<F>(p);
}

struct Vmm {
  decltype(&cuMemAddressReserve) reserve = driver_fn<decltype(&cuMemAddressReserve)>("cuMemAddressReserve");
  decltype(&cuMemAddressFree) free = driver_fn<decltype(&cuMemAddressFree)>("cuMemAddressFree");
  decltype(&cuMemGetAllocationGranularity) granularity =
      driver_fn<decltype(&cuMemGetAllocationGranularity)>("cuMemGetAllocationGranularity");
  decltype(&cuMemCreate) create = driver_fn<decltype(&cuMemCreate)>("cuMemCreate");
  decltype(&cuMemRelease) release = driver_fn<decltype(&cuMemRelease)>("cuMemRelease");
  decltype(&cuMemMap) map = driver_fn<decltype(&cuMemMap)>("cuMemMap");
  decltype(&cuMemUnmap) unmap = driver_fn<decltype(&cuMemUnmap)>("cuMemUnmap");
  decltype(&cuMemSetAccess) set_access = driver_fn<decltype(&cuMemSetAccess)>("cuMemSetAccess");
};
static const Vmm& vmm() {
  static const Vmm v;
  return v;
}

static void cu_check(CUresult r, const char* what, size_t bytes) {
  if (r != CUDA_SUCCESS)
    throw Error(std::string("workspace arena: ") + what + " of " + std::to_string(bytes) + " bytes failed (CUresult " +
                std::to_string(static_cast<int>(r)) + ")");
}

static CUmemAllocationProp arena_prop(int device) {
  CUmemAllocationProp prop;
  std::memset(&prop, 0, sizeof prop);
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  return prop;
}

char* Arena::ptr() {
  if (!base) {
    const Vmm& v = vmm();
    const CUmemAllocationProp prop = arena_prop(device);
    cu_check(v.granularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM), "cuMemGetAllocationGranularity", 0);
    size_t free_b = 0, total_b = 0;
    I2IT_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const size_t size = round(total_b);     // no plan can need more than the device holds
    cu_check(v.reserve(&base, size, 0, 0, 0), "cuMemAddressReserve", size);
    reserved = size;
  }
  return reinterpret_cast<char*>(base);
}

void Arena::grow(size_t bytes) {
  ptr();
  const size_t target = round(bytes);
  if (target <= mapped) return;
  I2IT_CHECK(target <= reserved, "workspace arena: " + std::to_string(target) + " bytes exceed the device's memory");
  const Vmm& v = vmm();
  const size_t size = target - mapped;
  const CUmemAllocationProp prop = arena_prop(device);
  CUmemGenericAllocationHandle h;
  cu_check(v.create(&h, size, &prop, 0), "cuMemCreate", size);
  CUresult r = v.map(base + mapped, size, 0, h, 0);
  if (r != CUDA_SUCCESS) { v.release(h); cu_check(r, "cuMemMap", size); }
  CUmemAccessDesc acc;
  std::memset(&acc, 0, sizeof acc);
  acc.location = prop.location;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  r = v.set_access(base + mapped, size, &acc, 1);
  if (r != CUDA_SUCCESS) { v.unmap(base + mapped, size); v.release(h); cu_check(r, "cuMemSetAccess", size); }
  chunks.push_back({mapped, size, h});
  mapped = target;
}

void Arena::shrink(size_t bytes, size_t keep) {
  if (!base) return;
  const Vmm& v = vmm();
  const size_t target = round(bytes);
  auto drop_last = [&]() {
    const Chunk c = chunks.back();
    chunks.pop_back();
    mapped = c.off;
    cu_check(v.unmap(base + c.off, c.size), "cuMemUnmap", c.size);
    cu_check(v.release(c.h), "cuMemRelease", c.size);
  };
  while (!chunks.empty() && chunks.back().off >= target) drop_last();
  if (mapped > target && chunks.back().off >= keep) {   // re-create the straddling chunk at the new size
    drop_last();
    grow(target);
  }
}

void Arena::fill(int value) {
  if (!mapped) return;
  I2IT_CUDA(cudaMemset(reinterpret_cast<void*>(base), value, mapped));
  I2IT_CUDA(cudaDeviceSynchronize());
}

Arena::~Arena() {
  if (!base) return;
  try {
    const Vmm& v = vmm();
    for (auto it = chunks.rbegin(); it != chunks.rend(); ++it) {
      v.unmap(base + it->off, it->size);
      v.release(it->h);
    }
    v.free(base, reserved);
  } catch (...) {}
}

// ---------------------------------------------------------------------------------------------
// pool
// ---------------------------------------------------------------------------------------------
Pool::~Pool() {
  for (auto& b : blocks) cudaFree(b.first);
}
void* Pool::get(size_t bytes, size_t* actual) {
  bytes = (bytes + 511) / 512 * 512;
  auto it = free_.lower_bound(bytes);
  if (it != free_.end() && it->first <= bytes + bytes / 2 + (1u << 20)) {
    void* p = it->second;
    *actual = it->first;
    free_.erase(it);
    return p;
  }
  void* p = nullptr;
  if (arena) {
    p = arena->ptr() + transient();      // the plan's new transient blocks tile [0, transient()) of the arena
  } else {
    I2IT_CUDA(cudaMalloc(&p, bytes));
    blocks.emplace_back(p, bytes);
  }
  total += bytes;
  *actual = bytes;
  return p;
}

void* Pool::get_fresh(size_t bytes) {
  bytes = (bytes + 511) / 512 * 512;
  void* p = nullptr;
  I2IT_CUDA(cudaMalloc(&p, bytes));
  blocks.emplace_back(p, bytes);
  total += bytes;
  persistent += bytes;
  return p;
}

// ---------------------------------------------------------------------------------------------
// engine basics
// ---------------------------------------------------------------------------------------------
__global__ void cvt16_to_f32_kernel(const uint16_t* s, float* d, long long n, int is_bf16) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (is_bf16) d[i] = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(s)[i]);
  else d[i] = __half2float(reinterpret_cast<const __half*>(s)[i]);
}

thread_local PdlState g_pdl;

// tapgemm instantiations: the MMA of a k16 step is one wgmma of the tile's full width, so BN is a template parameter.  The
// LEAN variant only runs TMA-store launches (whole 64-column rounds); the full variant takes every BN pick_bn can choose.
// Callers that set BN themselves must use one of these widths: attn_pv's BN = min(head dim, 256) covers head dims 16, 32, ..., 160,
// 192, 224 and >= 256 (the model's are 64 and 512); 176, 208 and 240 are refused at plan time.
#define TG_BN_LEAN(X) X(64) X(128) X(192) X(256)
#define TG_BN_FULL(X) X(16) X(32) X(48) X(64) X(80) X(96) X(112) X(128) X(160) X(192) X(224) X(256)
// the plain and the selecting kernel of one instantiation (both nullptr: no such instantiation)
template <typename T> struct TgKernels {
  void (*plain)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, TapGemmParams) = nullptr;
  void (*sel)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, TapGemmParams, CUtensorMap, CUtensorMap,
              TapGemmSel) = nullptr;
};
template <typename T> static TgKernels<T> tapgemm_for(bool lean, int bn) {
#define TG_CASE_LEAN(n) if (lean && bn == n) return {tapgemm_kernel<T, true, n>, tapgemm_sel_kernel<T, true, n>};
#define TG_CASE_FULL(n) if (!lean && bn == n) return {tapgemm_kernel<T, false, n>, tapgemm_sel_kernel<T, false, n>};
  TG_BN_LEAN(TG_CASE_LEAN)
  TG_BN_FULL(TG_CASE_FULL)
#undef TG_CASE_LEAN
#undef TG_CASE_FULL
  return {};
}

Engine::Engine(const i2it_config& c) : cfg(c), dtype(c.dtype) {
  I2IT_CHECK(c.dtype == DT_F16 || c.dtype == DT_BF16, "dtype must be I2IT_F16 or I2IT_BF16");
  I2IT_CUDA(cudaSetDevice(c.device));
  cudaDeviceProp prop;
  I2IT_CUDA(cudaGetDeviceProperties(&prop, c.device));
  I2IT_CHECK(prop.major == 9 && prop.minor == 0, "libi2it is built for sm_90a (H100) only; found compute capability " +
                                                  std::to_string(prop.major) + "." + std::to_string(prop.minor));
  num_sms = prop.multiProcessorCount;
  auto tg_smem = [](auto k) { if (k) I2IT_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, TG_SMEM)); };
  for (int lean = 0; lean < 2; ++lean)
    for (int bn = 16; bn <= 256; bn += 16) {
      const auto h = tapgemm_for<__half>(lean, bn);
      const auto b = tapgemm_for<__nv_bfloat16>(lean, bn);
      tg_smem(h.plain); tg_smem(h.sel); tg_smem(b.plain); tg_smem(b.sel);
    }
  I2IT_CUDA(cudaFuncSetAttribute(flash_attn_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, FA_SMEM));
  I2IT_CUDA(cudaFuncSetAttribute(flash_attn_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, FA_SMEM));
  I2IT_CUDA(cudaFuncSetAttribute(flash_attn512_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, FA5_SMEM));
  I2IT_CUDA(cudaFuncSetAttribute(flash_attn512_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, FA5_SMEM));
  use_flash = std::getenv("I2IT_NO_FLASH") == nullptr;     // both flash kernels (d = 64, and d = 512 above 8192 keys)
  use_pdl = std::getenv("I2IT_PDL") != nullptr;     // programmatic dependent launch: measured neutral (1 CTA/SM kernels cannot co-reside), opt-in
#ifdef I2IT_TRACE_BUILD
  trace_on = std::getenv("I2IT_TRACE") != nullptr;
#endif
  use_tmaout = std::getenv("I2IT_NO_TMAOUT") == nullptr;   // TMA-store epilogue (per-thread stores otherwise)
  use_ostg2 = std::getenv("I2IT_NO_OSTG2") == nullptr;     // second TMA-store box per epilogue warp where the operand ring can spare 32 KB
  sync_each = std::getenv("I2IT_SYNC_EACH") != nullptr;    // eager path: synchronise after every launch and name the one that faults
  use_lean = std::getenv("I2IT_NO_LEAN") == nullptr;       // compile-time-stripped epilogue for the plain (no activation) TMA-store launches
  use_gnepi = std::getenv("I2IT_NO_GNEPI") == nullptr;     // GroupNorm statistics in the producing GEMM's epilogue
  use_splitk = std::getenv("I2IT_NO_SPLITK") == nullptr;   // split-K for the 8x8 1280-channel convs
  use_catfuse = std::getenv("I2IT_NO_CATFUSE") == nullptr; // UNet skip concatenations written in place (no copy kernels)
  // identity residual as a K-slab (opt-in): the coalesced residual through the store box is the default
  use_idres = std::getenv("I2IT_IDRES") != nullptr && std::getenv("I2IT_NO_IDRES") == nullptr;
  int* h = nullptr;
  I2IT_CUDA(cudaHostAlloc(&h, sizeof(int), cudaHostAllocMapped));
  *h = 0;
  I2IT_CUDA(cudaHostGetDevicePointer(&d_err, h, 0));
  err_host_ = h;
  I2IT_CUDA(cudaStreamCreateWithFlags(&gstream_, cudaStreamNonBlocking));
  I2IT_CUDA(cudaEventCreateWithFlags(&ev_in_, cudaEventDisableTiming));
  I2IT_CUDA(cudaEventCreateWithFlags(&ev_out_, cudaEventDisableTiming));
  I2IT_CUDA(cudaEventCreateWithFlags(&rs_ev_, cudaEventDisableTiming));
  I2IT_CUDA(cudaEventCreateWithFlags(&dir_ev_, cudaEventDisableTiming));
  encode_fn();
  arena_.device = c.device;
}

Engine::~Engine() {
  cudaSetDevice(cfg.device);
  cudaDeviceSynchronize();          // graphs and the arena's mappings go below; neither waits for the device by itself
  plans_.clear();
  textkv_.clear();
  textenc_.clear();
  free_prepared();
  for (auto& kv : w_) cudaFree(kv.second.d);
  for (void* p : retired_) cudaFree(p);
  for (auto& t : job_tables_) cudaFree(t.p);
  if (err_host_) cudaFreeHost(err_host_);
  if (gstream_) cudaStreamDestroy(gstream_);
  if (ev_in_) cudaEventDestroy(ev_in_);
  if (ev_out_) cudaEventDestroy(ev_out_);
  if (rs_ev_) cudaEventDestroy(rs_ev_);
  if (rs_blob_) cudaFreeHost(rs_blob_);
  if (dir_ev_) cudaEventDestroy(dir_ev_);
  if (dir_blob_) cudaFreeHost(dir_blob_);
}

void Engine::check_device_error() {
  if (err_host_ && *err_host_ != 0) {
    const int code = *err_host_;
    throw Error("tapgemm watchdog tripped (pipeline stage code " + std::to_string(code) +
                ": 1=producer/empty 2=producer/epilogue-done 3=consumer/full)");
  }
}

// ---------------------------------------------------------------------------------------------
// image-forward plan cache
// ---------------------------------------------------------------------------------------------
void Engine::sync_plans() {
  I2IT_CUDA(cudaStreamSynchronize(gstream_));   // graph replays
  I2IT_CUDA(cudaDeviceSynchronize());           // eager forwards on the caller's stream
}

void Engine::trim_arena(bool keep_last) {
  size_t need = 0;
  for (const auto& kv : plans_) need = std::max(need, kv.second->pool.transient());
  // the last forward's stages (i2it_read_stage) live in the arena: those bytes keep their contents unless a forward is about
  // to overwrite them anyway
  const size_t keep = (keep_last && last_plan_) ? last_plan_->pool.transient() : 0;
  try {
    arena_.shrink(need, keep);
  } catch (...) {                               // the arena may now be smaller than the resident plans: drop them
    plans_.clear();
    last_plan_ = nullptr;
    throw;
  }
}

void Engine::evict_lru(const Plan* also_keep, bool keep_last) {
  if (max_plans_ <= 0) return;
  bool evicted = false;
  while (static_cast<int>(plans_.size()) > max_plans_) {
    auto victim = plans_.end();
    for (auto it = plans_.begin(); it != plans_.end(); ++it) {
      const Plan* p = it->second.get();
      if (p == last_plan_ || p == also_keep) continue;
      if (victim == plans_.end() || p->last_run < victim->second->last_run) victim = it;
    }
    if (victim == plans_.end()) break;
    if (!evicted) sync_plans();
    evicted = true;
    plans_.erase(victim);
    ++plan_evictions_;
  }
  if (evicted) trim_arena(keep_last);
}

void Engine::set_max_plans(int n) {
  I2IT_CHECK(n >= 0, "max_plans must be >= 0 (0: no limit)");
  max_plans_ = n;
  evict_lru();
}

void Engine::release_plans() {
  sync_plans();
  plans_.clear();
  last_plan_ = nullptr;
  arena_.shrink(0, 0);
}

i2it_memory_stats Engine::memory_stats() const {
  i2it_memory_stats s;
  std::memset(&s, 0, sizeof s);
  s.arena_bytes = arena_.mapped;
  for (const auto& kv : plans_) s.plan_bytes += kv.second->pool.persistent;
  s.plans = static_cast<int>(plans_.size());
  s.plan_builds = plan_builds_;
  s.plan_evictions = plan_evictions_;
  return s;
}

void Engine::poison_workspace(int value) {
  sync_plans();
  arena_.fill(value);
}

void* Engine::dmalloc(size_t bytes) {
  void* p = nullptr;
  I2IT_CUDA(cudaMalloc(&p, std::max<size_t>(bytes, 16)));
  prep_allocs_.push_back(p);
  return p;
}

void Engine::free_prepared() {
  for (void* p : prep_allocs_) cudaFree(p);
  prep_allocs_.clear();
  prepared_.clear();
  prepared_f32_.clear();
  recipes_.clear();
  emb_act_ = nullptr;
  pending_jobs_.clear();
  pending_blocks_ = 0;
  for (auto& g : pending_gemv_) g.clear();
}

void Engine::set_weight(const std::string& key_in, const void* data, const int64_t* shape, int ndim, int dt, bool is_dev) {
  std::string key = key_in;
  const std::string bl = ".base_layer.";
  const size_t pos = key.find(bl);
  if (pos != std::string::npos) key = key.substr(0, pos) + "." + key.substr(pos + bl.size());
  std::vector<int64_t> shp(shape, shape + ndim);
  long long numel = 1;
  for (int i = 0; i < ndim; ++i) numel *= shape[i];
  I2IT_CHECK(numel > 0, "empty tensor for key " + key);
  I2IT_CHECK(dt == DT_F32 || dt == DT_F16 || dt == DT_BF16, "unsupported weight dtype");
  auto it = w_.find(key);
  // the same shape: copy into the existing master, whose address the prepared weights' recipes and the plans (norm scales,
  // text embeddings) hold; no forward may be reading it meanwhile
  const bool in_place = it != w_.end() && it->second.shape == shp;
  float* dst = nullptr;
  if (in_place) {
    sync_plans();
    dst = it->second.d;
  } else {
    I2IT_CUDA(cudaMalloc(&dst, numel * sizeof(float)));
  }
  if (dt == DT_F32) {
    I2IT_CUDA(cudaMemcpy(dst, data, numel * sizeof(float), is_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
  } else {
    uint16_t* tmp = nullptr;
    I2IT_CUDA(cudaMalloc(&tmp, numel * 2));
    I2IT_CUDA(cudaMemcpy(tmp, data, numel * 2, is_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
    cvt16_to_f32_kernel<<<ceil_div(numel, 256), 256>>>(tmp, dst, numel, dt == DT_BF16);
    I2IT_CUDA(cudaDeviceSynchronize());
    cudaFree(tmp);
  }
  if (!in_place) {
    // resident plans may still read the old master (a norm scale): it lives until the next finalize drops them
    if (it != w_.end()) { retired_.push_back(it->second.d); w_.erase(it); }
    WT t;
    t.d = dst; t.shape = shp; t.numel = numel;
    w_.emplace(key, std::move(t));
  }
  dirty_w_.insert(key);
  finalized_ = false;
}

bool Engine::has(const std::string& key) const { return w_.count(key) != 0; }

const WT& Engine::raw(const std::string& name, const char* what) const {
  auto it = w_.find(name + "." + what);
  I2IT_CHECK(it != w_.end(), "missing weight '" + name + "." + what + "'");
  return it->second;
}

const WT& Engine::src(const std::string& name, const char* what) {
  const WT& w = raw(name, what);
  if (recording_ >= 0) recipes_[recording_].reads.push_back(name + "." + what);
  return w;
}

const float* Engine::f32_input(const std::string& key) {
  auto it = prepared_f32_.find(key);
  if (it != prepared_f32_.end()) {
    if (recording_ >= 0) recipes_[recording_].after.push_back(key);
    return it->second;
  }
  auto w = w_.find(key);
  I2IT_CHECK(w != w_.end(), "missing weight '" + key + "'");
  if (recording_ >= 0) recipes_[recording_].reads.push_back(key);
  return w->second.d;
}

float Engine::fold_input(FoldInput which) {
  I2IT_CHECK(which == FOLD_GAMMA || which == FOLD_TWIN_R, "fold_input: the LoRA weights are read through adapter_weight");
  if (recording_ >= 0) recipes_[recording_].uses |= which;
  return which == FOLD_GAMMA ? skip_gamma_ : twin_r_;
}

float Engine::adapter_weight(const std::string& name, const std::string& adapter) {
  auto it = adapter_scale_.find(adapter);
  I2IT_CHECK(it != adapter_scale_.end(), "no scale registered for LoRA adapter '" + adapter + "' (layer " + name + ")");
  const bool is_unet = name.rfind("unet.", 0) == 0;
  if (recording_ >= 0) recipes_[recording_].uses |= (is_unet ? FOLD_LW_UNET : FOLD_LW_VAE) | FOLD_ADAPTER_SCALE;
  return it->second * (is_unet ? lw_unet_ : lw_vae_);
}

void Engine::add_recipe(const std::string& key, std::function<void()> emit) {
  Recipe r;
  r.key = key;
  r.emit = std::move(emit);
  recipes_.push_back(std::move(r));
  try {
    run_recipe(recipes_.size() - 1);
  } catch (...) {
    recipes_.pop_back();
    throw;
  }
}

void Engine::run_recipe(size_t i) {
  Recipe& r = recipes_[i];
  // a run that throws pushes no launch: its buffers keep the last fold, and so must what the recipe says that fold read
  const unsigned uses = r.uses;
  std::vector<std::string> reads = std::move(r.reads), after = std::move(r.after);
  r.uses = 0;
  r.reads.clear();
  r.after.clear();
  recording_ = static_cast<long long>(i);
  try {
    r.emit();
  } catch (...) {
    recording_ = -1;
    r.uses = uses;
    r.reads = std::move(reads);
    r.after = std::move(after);
    throw;
  }
  recording_ = -1;
}

void Engine::snapshot_fold() {
  fold_shapes_.clear();
  for (const auto& kv : w_) fold_shapes_[kv.first] = kv.second.shape;
  fold_adapter_scale_ = adapter_scale_;
  dirty_w_.clear();
}

void Engine::finalize(float lw_unet, float lw_vae, float skip_gamma, float twin_r) {
  sync_plans();
  lw_unet_ = lw_unet; lw_vae_ = lw_vae; skip_gamma_ = skip_gamma; twin_r_ = twin_r;
  plans_.clear();                  // the arena stays mapped: the plans rebuilt with the new weights need the same bytes
  textkv_.clear();                 // cached cross-attention operands were projected with the old (LoRA-scaled) weights
  textenc_.clear();
  last_plan_ = nullptr;
  last_text_plan_ = nullptr;
  free_prepared();
  for (void* p : retired_) cudaFree(p);
  retired_.clear();
  snapshot_fold();
  finalized_ = true;
  folded_ = true;
}

// algorithmic bytes a preparation job reads and writes (each source element once)
static double prep_job_bytes(const PrepJob& j) {
  if (j.mode == PREP_IDENTITY) return 2.0 * j.n;
  if (j.mode == PREP_BIAS) return 4.0 * j.cout * (1 + (j.bias != nullptr) + (j.w1 != nullptr) + (j.bias_add != nullptr));
  const double inner = 1.0 * j.cin * j.taps;
  double b = 4.0 * j.cout * inner * (j.w1 ? 2 : 1) + 2.0 * j.n;
  for (int a = 0; a < j.n_adapters; ++a) b += 4.0 * j.rank[a] * (inner + j.cout);
  return b;
}

static double gemv_job_bytes(const GemvJob& j) {
  double b = 4.0 * (1.0 * j.out * j.in + j.in + j.out * (j.b ? 2 : 1));
  for (int a = 0; a < j.n_adapters; ++a) b += 4.0 * j.rank[a] * (1.0 * j.in + j.out);
  return b;
}

void Engine::refold(float lw_unet, float lw_vae, float skip_gamma, float twin_r) {
  sync_plans();
  I2IT_CHECK(folded_, "i2it_refold_weights: the weights were never folded; call i2it_finalize_weights first");
  I2IT_CHECK((twin_r < 0.f) == (twin_r_ < 0.f),
             std::string("i2it_refold_weights: twin_r ") + (twin_r < 0.f ? "< 0 turns the TwinConv blend off" : ">= 0 turns the TwinConv blend on") +
             " since the last fold; call i2it_finalize_weights");
  // every master a recipe or a plan reads keeps its address and shape (set_weight copies same-shape tensors in place)
  for (const auto& kv : w_) {
    auto it = fold_shapes_.find(kv.first);
    I2IT_CHECK(it != fold_shapes_.end(), "i2it_refold_weights: tensor '" + kv.first + "' was added since the last fold; "
                                         "call i2it_finalize_weights");
    I2IT_CHECK(it->second == kv.second.shape, "i2it_refold_weights: tensor '" + kv.first + "' changed shape since the last "
                                              "fold; call i2it_finalize_weights");
  }
  I2IT_CHECK(w_.size() == fold_shapes_.size(), "i2it_refold_weights: a tensor has gone since the last fold; call i2it_finalize_weights");
  float* cur[4] = {&lw_unet_, &lw_vae_, &skip_gamma_, &twin_r_};
  const float next[4] = {lw_unet, lw_vae, skip_gamma, twin_r};
  const unsigned bit[4] = {FOLD_LW_UNET, FOLD_LW_VAE, FOLD_GAMMA, FOLD_TWIN_R};
  float prev[4];
  unsigned changed = adapter_scale_ != fold_adapter_scale_ ? FOLD_ADAPTER_SCALE : 0u;
  for (int i = 0; i < 4; ++i) {
    prev[i] = *cur[i];
    if (std::memcmp(&next[i], cur[i], sizeof(float)) != 0) changed |= bit[i];   // bitwise: 0 and -0 fold to different bits
    *cur[i] = next[i];
  }
  // the recipes in creation order: a recipe runs after those whose outputs it reads, and its jobs are the ones a fresh
  // finalize would push for it
  std::vector<std::string> touched;
  std::set<std::string> rebuilt;
  try {
    for (size_t i = 0; i < recipes_.size(); ++i) {
      const Recipe& r = recipes_[i];
      bool dirty = (r.uses & changed) != 0;
      for (const auto& k : r.reads) dirty = dirty || dirty_w_.count(k) != 0;
      for (const auto& k : r.after) dirty = dirty || rebuilt.count(k) != 0;
      if (!dirty) continue;
      run_recipe(i);
      rebuilt.insert(recipes_[i].key);
      touched.push_back(recipes_[i].key);
    }
  } catch (...) {
    for (int i = 0; i < 4; ++i) *cur[i] = prev[i];
    pending_jobs_.clear();
    pending_blocks_ = 0;
    for (auto& g : pending_gemv_) g.clear();
    throw;
  }
  refold_touched_ = std::move(touched);
  refold_jobs_ = static_cast<long long>(pending_jobs_.size());
  refold_gemv_jobs_ = 0;
  refold_bytes_ = 0;
  for (const auto& j : pending_jobs_) refold_bytes_ += prep_job_bytes(j);
  for (const auto& g : pending_gemv_) {
    refold_gemv_jobs_ += static_cast<long long>(g.size());
    for (const auto& j : g) refold_bytes_ += gemv_job_bytes(j);
  }
  flush_prep();
  I2IT_CUDA(cudaDeviceSynchronize());
  I2IT_CUDA(cudaGetLastError());
  // cached cross-attention operands were projected with the old weights; their buffers stay (cached-text plans read them)
  for (auto& kv : textkv_) kv.second->filled = false;
  snapshot_fold();
  finalized_ = true;
}

std::string Engine::refold_info_json() const {
  std::string js = "{\"recipes\":[";
  for (size_t i = 0; i < refold_touched_.size(); ++i) js += std::string(i ? "," : "") + "\"" + refold_touched_[i] + "\"";
  return js + "],\"jobs\":" + std::to_string(refold_jobs_) + ",\"gemv_jobs\":" + std::to_string(refold_gemv_jobs_) +
         ",\"bytes\":" + std::to_string(static_cast<long long>(refold_bytes_)) + "}";
}

// Fold recipe of a layer: c0*W (+ c1*W_other) + sum_adapters s_a * B_a @ A_a — filled into a job, evaluated on device
void Engine::fill_fold(PrepJob& j, const std::string& name, float c0, const std::string& other, float c1) {
  const WT& w = src(name, "weight");
  j.w0 = w.d; j.c0 = c0; j.w1 = nullptr; j.c1 = 0.f; j.n_adapters = 0;
  if (!other.empty()) {
    const WT& o = src(other, "weight");
    I2IT_CHECK(o.numel == w.numel, "TwinConv shapes differ");
    j.w1 = o.d; j.c1 = c1;
  }
  const std::string pre = name + ".lora_A.";
  std::vector<std::string> adapters;
  for (const auto& kv : w_)
    if (kv.first.compare(0, pre.size(), pre) == 0) {
      const std::string rest = kv.first.substr(pre.size());            // "<adapter>.weight"
      adapters.push_back(rest.substr(0, rest.rfind('.')));
    }
  std::sort(adapters.begin(), adapters.end());                          // fixed summation order
  for (const auto& adapter : adapters) {
    const float s = adapter_weight(name, adapter);
    if (s == 0.f) continue;
    const WT& A = src(name + ".lora_A." + adapter, "weight");
    I2IT_CHECK(has(name + ".lora_B." + adapter + ".weight"), "lora_A without lora_B for " + name);
    const WT& Bm = src(name + ".lora_B." + adapter, "weight");
    const int rank = static_cast<int>(A.shape[0]);
    const long long inner = A.numel / rank;
    I2IT_CHECK(Bm.shape[0] * inner == w.numel && Bm.shape[1] == rank, "LoRA shape mismatch at " + name);
    I2IT_CHECK(j.n_adapters < PREP_MAX_ADAPTERS, "too many LoRA adapters on " + name);
    j.A[j.n_adapters] = A.d; j.B[j.n_adapters] = Bm.d; j.s[j.n_adapters] = s; j.rank[j.n_adapters] = rank;
    ++j.n_adapters;
  }
}

void Engine::push_job(PrepJob& j) {
  if (j.n <= 0) return;
  j.block0 = pending_blocks_;
  pending_blocks_ += (j.n + PREP_ELEMS_PER_BLOCK - 1) / PREP_ELEMS_PER_BLOCK;
  pending_jobs_.push_back(j);
}

void Engine::push_bias_job(float* out, const float* b, const float* add, int cout, int row_off, int half, float c0,
                           const float* b1, float c1) {
  PrepJob j;
  std::memset(&j, 0, sizeof j);
  j.mode = PREP_BIAS; j.out = out; j.bias = b; j.bias_add = add; j.cout = cout; j.row_off = row_off; j.interleave_half = half;
  j.c0 = c0; j.w1 = b1; j.c1 = c1;
  j.n = cout;
  push_job(j);
}

void* Engine::upload_jobs(int table, const void* jobs, size_t bytes) {
  JobTable& t = job_tables_[table];
  if (t.cap < bytes) {
    I2IT_CUDA(cudaDeviceSynchronize());   // an earlier flush's launch may still read the old table
    cudaFree(t.p);
    t.p = nullptr;
    t.cap = 0;
    I2IT_CUDA(cudaMalloc(&t.p, bytes));
    t.cap = bytes;
  }
  // on the default stream, as the launches that read the table: ordered after the previous flush's launch
  I2IT_CUDA(cudaMemcpy(t.p, jobs, bytes, cudaMemcpyHostToDevice));
  return t.p;
}

// Runs every pending preparation job: <= 3 GEMV launches (time embedding chain) + ONE fold/re-layout launch.
void Engine::flush_prep() {
  for (int st = 0; st < 3; ++st) {
    auto& g = pending_gemv_[st];
    if (g.empty()) continue;
    int warps = 0;
    for (auto& j : g) { j.warp0 = warps; warps += j.out; }
    GemvJob* d = static_cast<GemvJob*>(upload_jobs(st, g.data(), g.size() * sizeof(GemvJob)));
    gemv_jobs_kernel<<<ceil_div(warps * 32ll, 256), 256>>>(d, static_cast<int>(g.size()));
    I2IT_CUDA(cudaGetLastError());
    prep_launches_ += 1;
    g.clear();
  }
  if (!pending_jobs_.empty()) {
    PrepJob* d = static_cast<PrepJob*>(upload_jobs(3, pending_jobs_.data(), pending_jobs_.size() * sizeof(PrepJob)));
    I2IT_CHECK(pending_blocks_ < (1ll << 31), "weight preparation: too many blocks for one launch");
    DISPATCH_T(dtype, (prep_jobs_kernel<T><<<static_cast<unsigned>(pending_blocks_), 256>>>(d, static_cast<int>(pending_jobs_.size()))));
    I2IT_CUDA(cudaGetLastError());
    prep_launches_ += 1;
    pending_jobs_.clear();
    pending_blocks_ = 0;
  }
}

// Mixed-direction plans: a vae. weight is prepared (through its usual cache key) together with its vae_b2a. twin, and the
// pair goes to the launch, which selects per image.  While the twins are prepared the pairing is paused.
static bool is_a2b_vae(const std::string& key) { return key.compare(0, 4, "vae.") == 0; }
static std::string b2a_key(const std::string& key) { return is_a2b_vae(key) ? "vae_b2a." + key.substr(4) : key; }
struct MixedPause {
  const int*& slot;
  const int* dir;
  explicit MixedPause(const int*& s) : slot(s), dir(s) { slot = nullptr; }
  ~MixedPause() { slot = dir; }
};
static PW pair_pw(PW a, const PW& b, const int* dir, const std::string& key) {
  I2IT_CHECK(a.rows == b.rows && a.cin == b.cin && a.cin_pad == b.cin_pad && a.taps == b.taps && !a.bias == !b.bias,
             "mixed-direction plan: " + key + " and its vae_b2a twin differ in shape");
  a.w_alt = b.w; a.bias_alt = b.bias; a.dir = dir;
  return a;
}

PW Engine::prep(const std::string& cache_key, const std::vector<std::string>& names, bool geglu, bool skip_scale,
                const std::string& bias_add) {
  if (mixed_dir_ && is_a2b_vae(cache_key)) {
    MixedPause pause(mixed_dir_);
    std::vector<std::string> nb;
    for (const auto& n : names) nb.push_back(b2a_key(n));
    const PW a = prep(cache_key, names, geglu, skip_scale, bias_add);
    return pair_pw(a, prep(b2a_key(cache_key), nb, geglu, skip_scale, b2a_key(bias_add)), pause.dir, cache_key);
  }
  auto it = prepared_.find(cache_key);
  if (it != prepared_.end()) return it->second;
  I2IT_CHECK(finalized_, "i2it_finalize_weights must be called before a forward");
  PW pw;
  const WT& w0 = raw(names[0], "weight");
  pw.cin = static_cast<int>(w0.shape[1]);
  pw.taps = (w0.shape.size() == 4) ? static_cast<int>(w0.shape[2] * w0.shape[3]) : 1;
  pw.cin_pad = round_up(pw.cin, 8);
  bool any_bias = !bias_add.empty();
  for (const auto& n : names) {
    const WT& w = raw(n, "weight");
    I2IT_CHECK(static_cast<int>(w.shape[1]) == pw.cin, "fused projection with different input widths: " + n);
    pw.rows += static_cast<int>(w.shape[0]);
    any_bias = any_bias || has(n + ".bias");
  }
  I2IT_CHECK(!geglu || names.size() == 1, "GEGLU interleave applies to a single projection");
  const size_t wbytes = static_cast<size_t>(pw.taps) * pw.rows * pw.cin_pad * 2;
  pw.w = static_cast<uint16_t*>(dmalloc(wbytes));
  if (any_bias) pw.bias = static_cast<float*>(dmalloc(pw.rows * sizeof(float)));
  add_recipe(cache_key, [this, pw, names, geglu, skip_scale, bias_add]() {
    const float scale = skip_scale ? fold_input(FOLD_GAMMA) : 1.f;
    const float* add = bias_add.empty() ? nullptr : f32_input(bias_add);
    int row_off = 0;
    for (const auto& n : names) {
      const int cout = static_cast<int>(raw(n, "weight").shape[0]);
      const int half = geglu ? cout / 2 : 0;
      PrepJob j;
      std::memset(&j, 0, sizeof j);
      fill_fold(j, n);
      j.mode = PREP_STORE; j.out = pw.w; j.cout = cout; j.cin = pw.cin; j.taps = pw.taps; j.cin_pad = pw.cin_pad;
      j.rows_total = pw.rows; j.row_off = row_off; j.interleave_half = half; j.scale = scale;
      j.n = static_cast<long long>(cout) * pw.cin_pad * pw.taps;
      push_job(j);
      if (pw.bias) push_bias_job(pw.bias, has(n + ".bias") ? src(n, "bias").d : nullptr, add, cout, row_off, half);
      row_off += cout;
    }
  });
  prepared_[cache_key] = pw;
  return pw;
}

PW Engine::prep_twin(const std::string& pre, const std::string& cur) {
  const std::string key = pre + "|twin";
  auto it = prepared_.find(key);
  if (it != prepared_.end()) return it->second;
  I2IT_CHECK(twin_r_ >= 0.f, "the state dict has a TwinConv conv_in but no blend ratio r was given (deterministic forward on a "
                             "sketch_to_image_stochastic model is undefined in the reference too)");
  PW pw;
  const WT& w0 = raw(pre, "weight");
  pw.rows = static_cast<int>(w0.shape[0]);
  pw.cin = static_cast<int>(w0.shape[1]);
  pw.taps = static_cast<int>(w0.shape[2] * w0.shape[3]);
  pw.cin_pad = round_up(pw.cin, 8);
  pw.w = static_cast<uint16_t*>(dmalloc(static_cast<size_t>(pw.taps) * pw.rows * pw.cin_pad * 2));
  pw.bias = static_cast<float*>(dmalloc(pw.rows * sizeof(float)));
  add_recipe(key, [this, pw, pre, cur]() {
    const float r = fold_input(FOLD_TWIN_R);
    PrepJob j;
    std::memset(&j, 0, sizeof j);
    fill_fold(j, pre, 1.f - r, cur, r);                       // W = (1-r) W_pre + r W_cur   (pix2pix_turbo.py:23-26)
    j.mode = PREP_STORE; j.out = pw.w; j.cout = pw.rows; j.cin = pw.cin; j.taps = pw.taps; j.cin_pad = pw.cin_pad;
    j.rows_total = pw.rows; j.scale = 1.f;
    j.n = static_cast<long long>(pw.rows) * pw.cin_pad * pw.taps;
    push_job(j);
    push_bias_job(pw.bias, src(pre, "bias").d, nullptr, pw.rows, 0, 0, 1.f - r, src(cur, "bias").d, r);   // (1-r) b_pre + r b_cur
  });
  prepared_[key] = pw;
  return pw;
}

PW Engine::prep_im2col3(const std::string& name) {
  if (mixed_dir_ && is_a2b_vae(name)) {
    MixedPause pause(mixed_dir_);
    const PW a = prep_im2col3(name);
    return pair_pw(a, prep_im2col3(b2a_key(name)), pause.dir, name);
  }
  const std::string key = name + "|im2col";
  auto it = prepared_.find(key);
  if (it != prepared_.end()) return it->second;
  const WT& w0 = raw(name, "weight");
  I2IT_CHECK(w0.shape.size() == 4 && w0.shape[1] == 3 && w0.shape[2] == 3 && w0.shape[3] == 3, "prep_im2col3: expects [Cout,3,3,3]");
  PW pw;
  pw.rows = static_cast<int>(w0.shape[0]); pw.cin = 32; pw.cin_pad = 32; pw.taps = 1;
  pw.w = static_cast<uint16_t*>(dmalloc(static_cast<size_t>(pw.rows) * 32 * 2));
  pw.bias = static_cast<float*>(dmalloc(pw.rows * sizeof(float)));
  add_recipe(key, [this, pw, name]() {
    PrepJob j;
    std::memset(&j, 0, sizeof j);
    fill_fold(j, name);
    j.mode = PREP_IM2COL3; j.out = pw.w; j.cout = pw.rows; j.cin = 3; j.taps = 9; j.scale = 1.f;
    j.n = static_cast<long long>(pw.rows) * 32;
    push_job(j);
    push_bias_job(pw.bias, src(name, "bias").d, nullptr, pw.rows, 0, 0);
  });
  prepared_[key] = pw;
  return pw;
}

PW Engine::prep_identity(int n) {
  const std::string key = "identity|" + std::to_string(n);
  auto it = prepared_.find(key);
  if (it != prepared_.end()) return it->second;
  PW pw;
  pw.rows = n; pw.cin = n; pw.cin_pad = n; pw.taps = 1;
  pw.w = static_cast<uint16_t*>(dmalloc(static_cast<size_t>(n) * n * 2));
  add_recipe(key, [this, pw, n]() {
    PrepJob j;
    std::memset(&j, 0, sizeof j);
    j.mode = PREP_IDENTITY; j.out = pw.w; j.cout = n; j.n = static_cast<long long>(n) * n;
    push_job(j);
  });
  prepared_[key] = pw;
  return pw;
}

PW Engine::prep_subpixel(const std::string& name) {
  if (mixed_dir_ && is_a2b_vae(name)) {
    MixedPause pause(mixed_dir_);
    const PW a = prep_subpixel(name);
    return pair_pw(a, prep_subpixel(b2a_key(name)), pause.dir, name);
  }
  const std::string key = name + "|subpixel";
  auto it = prepared_.find(key);
  if (it != prepared_.end()) return it->second;
  const WT& w0 = raw(name, "weight");
  I2IT_CHECK(w0.shape.size() == 4 && w0.shape[2] == 3 && w0.shape[3] == 3, "prep_subpixel: expects a 3x3 conv");
  PW pw;
  pw.rows = static_cast<int>(w0.shape[0]); pw.cin = static_cast<int>(w0.shape[1]); pw.cin_pad = round_up(pw.cin, 8); pw.taps = 16;
  const long long total = 16ll * pw.rows * pw.cin_pad;
  pw.w = static_cast<uint16_t*>(dmalloc(static_cast<size_t>(total) * 2));
  pw.bias = static_cast<float*>(dmalloc(pw.rows * sizeof(float)));
  add_recipe(key, [this, pw, name, total]() {
    PrepJob j;
    std::memset(&j, 0, sizeof j);
    fill_fold(j, name);
    j.mode = PREP_SUBPIXEL; j.out = pw.w; j.cout = pw.rows; j.cin = pw.cin; j.taps = 9; j.cin_pad = pw.cin_pad; j.scale = 1.f;
    j.n = total;
    push_job(j);
    push_bias_job(pw.bias, src(name, "bias").d, nullptr, pw.rows, 0, 0);
  });
  prepared_[key] = pw;
  return pw;
}

// nearest-2x upsample + conv3x3 (+ optional folded 1x1 second source at output resolution) as four parity-phase launches
Act Engine::conv_up2x(Plan& P, const Act& x, const PW& wsub, const Act* x2, const PW* w2, bool gn_out) {
  Act out = alloc_act(P, x.N, 2 * x.H, 2 * x.W, wsub.rows);
  for (int ph = 0; ph < 4; ++ph) {
    ConvOpts o;
    o.subpixel_phase = ph;
    o.out = &out;
    o.x2 = x2; o.w2 = w2;
    o.gn_out = gn_out;
    o.gn_share = out.gn;                 // phase 0 creates the partial buffer, phases 1..3 fill their slot ranges
    Act y = conv(P, x, wsub, o);
    out.gn = y.gn;
  }
  return out;
}

NormW Engine::norm(const std::string& name) {
  NormW n;
  const WT& g = raw(name, "weight");
  n.g = g.d;
  n.b = raw(name, "bias").d;
  n.C = static_cast<int>(g.numel);
  if (mixed_dir_ && is_a2b_vae(name)) {
    const WT& g2 = raw(b2a_key(name), "weight");
    I2IT_CHECK(g2.numel == g.numel, "mixed-direction plan: " + name + " and its vae_b2a twin differ in shape");
    n.g_alt = g2.d;
    n.b_alt = raw(b2a_key(name), "bias").d;
    n.dir = mixed_dir_;
  }
  return n;
}

std::string Engine::temb_bias(const std::string& p) {
  const std::string key = p + "|temb";
  if (prepared_f32_.count(key)) return key;
  const int T = cfg.temb_dim, C0 = cfg.unet_channels[0];
  auto gemv = [this](int stage, const std::string& name, const float* x, float* y, int out, int in, int silu) {
    PrepJob f;
    std::memset(&f, 0, sizeof f);
    fill_fold(f, name);
    GemvJob g;
    std::memset(&g, 0, sizeof g);
    g.w = f.w0; g.b = src(name, "bias").d; g.x = x; g.y = y; g.out = out; g.in = in; g.silu_out = silu;
    g.n_adapters = f.n_adapters;
    for (int a = 0; a < f.n_adapters; ++a) { g.A[a] = f.A[a]; g.B[a] = f.B[a]; g.s[a] = f.s[a]; g.rank[a] = f.rank[a]; }
    pending_gemv_[stage].push_back(g);
  };
  static const std::string emb = "unet.time_embedding|emb";   // the shared embedding: a recipe of its own, in no cache
  if (!emb_act_) {
    // Timesteps(flip_sin_to_cos=True, freq_shift=0) at t = 999, then TimestepEmbedding, then the SiLU every resnet applies
    std::vector<float> te(C0);
    const int half = C0 / 2;
    for (int i = 0; i < half; ++i) {
      const float f = expf(-logf(10000.f) * static_cast<float>(i) / static_cast<float>(half));
      te[i] = cosf(999.f * f);
      te[half + i] = sinf(999.f * f);
    }
    float* d_te = static_cast<float*>(dmalloc(C0 * sizeof(float)));
    float* d_h = static_cast<float*>(dmalloc(T * sizeof(float)));
    float* e = static_cast<float*>(dmalloc(T * sizeof(float)));
    I2IT_CUDA(cudaMemcpy(d_te, te.data(), C0 * sizeof(float), cudaMemcpyHostToDevice));
    add_recipe(emb, [=]() {
      gemv(0, "unet.time_embedding.linear_1", d_te, d_h, T, C0, 1);
      gemv(1, "unet.time_embedding.linear_2", d_h, e, T, T, 1);
    });
    emb_act_ = e;
  }
  const WT& w = raw(p + ".time_emb_proj", "weight");
  const int cout = static_cast<int>(w.shape[0]);
  float* out = static_cast<float*>(dmalloc(cout * sizeof(float)));
  float* e = emb_act_;
  add_recipe(key, [=]() {
    recipes_[recording_].after.push_back(emb);
    gemv(2, p + ".time_emb_proj", e, out, cout, T, 0);
  });
  prepared_f32_[key] = out;
  return key;
}

// ---------------------------------------------------------------------------------------------
// op builders
// ---------------------------------------------------------------------------------------------
std::shared_ptr<void> Engine::alloc_raw(Plan& P, size_t bytes) {
  size_t actual = 0;
  void* p = P.pool.get(bytes, &actual);
  Pool* pool = &P.pool;
  return std::shared_ptr<void>(p, [pool, actual](void* q) { pool->put(q, actual); });
}

Act Engine::alloc_act(Plan& P, int N, int H, int W, int C, int ld, bool zero_persistent) {
  Act a;
  a.N = N; a.H = H; a.W = W; a.C = C; a.ld = ld ? ld : C;
  const size_t bytes = static_cast<size_t>(N) * H * W * a.ld * 2;
  if (zero_persistent) {
    // A recycled block would be dirtied at RUN time by the earlier ops that used it (the memset below runs once, at
    // build time), so padded small-channel tensors get their own allocation for the plan's lifetime.
    void* p = P.pool.get_fresh(bytes);
    I2IT_CUDA(cudaMemset(p, 0, bytes));
    a.hold = std::shared_ptr<void>(p, [](void*) {});
    a.p = static_cast<uint16_t*>(p);
    return a;
  }
  a.hold = alloc_raw(P, bytes);
  a.p = static_cast<uint16_t*>(a.hold.get());
  return a;
}

int Engine::pick_bn(long long m_tiles, int N, int step) const {
  if (N <= 16) return 16;
  static const int cand_any[] = {256, 224, 192, 160, 128, 112, 96, 80, 64, 48, 32, 16};   // = TG_BN_FULL
  static const int cand_64[] = {256, 192, 128, 64};
  static const int cand_128[] = {256, 128};
  const int* cand = step == 128 ? cand_128 : (step == 64 ? cand_64 : cand_any);
  const int ncand = step == 128 ? 2 : (step == 64 ? 4 : 12);
  int best = cand[ncand - 1];
  double best_cost = 1e30;
  for (int i = 0; i < ncand; ++i) {
    const int bn = cand[i];
    if (bn > round_up(N, step > 0 ? step : 16)) continue;
    const long long tiles = m_tiles * ceil_div(N, bn);
    const long long waves = (tiles + num_sms - 1) / num_sms;
    // a tile's time is bounded by its L2->SMEM traffic (A 128 rows + B bn rows per k-step) as much as by the MMA (bn)
    const double cost = static_cast<double>(waves) * (128 + bn);
    if (cost < best_cost - 1e-9) { best_cost = cost; best = bn; }
  }
  return best;
}

int Engine::plan_bn(const Plan& P, long long m_tiles, int N, int step) const {
  if (!P.debug_tapgemm || dbg_bn == 0) return pick_bn(m_tiles, N, step);
  const int hi = round_up(N, 16);
  if (tapgemm_for<__half>(false, dbg_bn).plain == nullptr || dbg_bn > hi) {
    std::string legal;
#define TG_LIST(n) if (n <= hi) legal += (legal.empty() ? "" : ", ") + std::to_string(n);
    TG_BN_FULL(TG_LIST)
#undef TG_LIST
    throw Error("tapgemm override: BN=" + std::to_string(dbg_bn) + " is illegal for N=" + std::to_string(N) + "; legal: " + legal);
  }
  return dbg_bn;
}

// The TMA-store epilogue handles 16-bit row-major outputs whose channel count and tile width are whole 64-column rounds (128
// accumulator columns for GEGLU) with 16-byte aligned rows; everything else keeps per-thread stores.
bool Engine::tma_eligible(const TapGemmParams& p, bool out_from_io) const {
  if (!use_tmaout || out_from_io || p.out_fp32 || p.ocol != 1 || p.bias_mode == TG_BIAS_ROW || p.out == nullptr) return false;
  const int acols = (p.act == TG_ACT_GEGLU) ? 128 : 64;
  if (p.N % acols != 0 || p.BN % acols != 0) return false;
  if (reinterpret_cast<uintptr_t>(p.out) % 16 != 0) return false;
  for (int d = 0; d < 4; ++d)
    if (p.ext[d] > 1 && (p.ostride[d] * 2) % 16 != 0) return false;
  if (p.res) {
    if (p.rcol != 1 || reinterpret_cast<uintptr_t>(p.res) % 16 != 0 || p.act == TG_ACT_GEGLU) return false;
    for (int d = 0; d < 4; ++d)
      if (p.ext[d] > 1 && (p.rstride[d] * 2) % 16 != 0) return false;
  }
  return true;
}

void conv_box(bool stride1, int Ho, int Wo, bool nchw, int& tw, int& th, int& tn) {
  if (stride1) tw = (Ho == 1) ? std::min(128, pow2ceil(Wo)) : std::min(nchw ? 32 : 16, pow2ceil(Wo));
  else tw = std::min(16, pow2ceil(Wo));
  th = std::min(128 / tw, pow2ceil(Ho));
  tn = 128 / (tw * th);
}

void Engine::launch_gemm(Plan& P, const TmapSpec& sa, TmapSpec sb, const TapGemmParams& p_in, bool out_from_io,
                         const char* kind, double k_valid, double bytes, const TmapSpec* sa2p, const TmapSpec* sb2p,
                         const SelSpec* sel) {
  TapGemmParams p = p_in;
  for (int t = 0; t < p.num_taps; ++t)
    if (p.tap_kc[t] == 0) p.tap_kc[t] = p.kchunks;          // single-source callers only set kchunks
  if (p.nprim == 0) p.nprim = p.num_taps;
  const long long m_tiles = 1ll * p.tdim[0] * p.tdim[1] * p.tdim[2] * p.tdim[3];
  const long long total_tiles = m_tiles * p.n_tiles * (p.ksplit > 1 ? p.ksplit : 1);
  I2IT_CHECK(p.BN % 16 == 0 && p.BN <= 256, "tapgemm: BN must be a multiple of 16 up to 256");
  const TmapSpec sb2 = sb2p ? *sb2p : sb;
  p.tma_out = tma_eligible(p, out_from_io) ? 1 : 0;
  {  // smem ring geometry: B stage = the real tile rounded to the 1024-byte swizzle atom, as many stages as fit
    p.b_stage = (p.BN * TG_BK * 2 + 1023) / 1024 * 1024;
    int budget = TG_STAGES * (TG_A_STAGE + TG_B_STAGE);
    const int per = TG_A_STAGE + p.b_stage;
    // a second store box per epilogue warp out of the ring's last 32 KB when at least 4 stages remain and the tile's mainloop
    // is short (<= 48 k-steps, i.e. <= 96 * BN tensor cycles): those launches wait on TMA-store drain, not on operands; the
    // long-K launches hide their epilogue anyway and keep the deeper ring
    int ksteps = 0;
    for (int t = 0; t < p.num_taps; ++t) ksteps += p.tap_kc[t];
    p.ostg2 = (use_ostg2 && p.tma_out && ksteps <= 48 && (budget - TG_OSTG_BYTES) / per >= 4) ? 1 : 0;
    if (p.ostg2) budget -= TG_OSTG_BYTES;
    p.stages = std::max(2, std::min(TG_MAX_STAGES, budget / per));
    if (P.debug_tapgemm && dbg_stages) {
      I2IT_CHECK(dbg_stages >= 2 && dbg_stages <= p.stages, "tapgemm override: stages=" + std::to_string(dbg_stages) +
                                                               " is illegal for " + kind + " BN=" + std::to_string(p.BN) +
                                                               "; legal: 2.." + std::to_string(p.stages));
      p.stages = dbg_stages;
    }
  }
  const CUtensorMap ta = encode_tmap(sa, dtype), tb = encode_tmap(sb, dtype);
  const CUtensorMap ta2 = sa2p ? encode_tmap(*sa2p, dtype) : ta, tb2 = sb2p ? encode_tmap(sb2, dtype) : tb;
  const int dt = dtype;
  Plan* plan = &P;
  const double m_valid = 1.0 * p.ext[0] * p.ext[1] * p.ext[2] * p.ext[3];
  const int max_grid = static_cast<int>(std::min<long long>(total_tiles, num_sms));
  int grid = max_grid;
  if (P.debug_tapgemm && dbg_grid) {
    I2IT_CHECK(dbg_grid <= max_grid, "tapgemm override: grid=" + std::to_string(dbg_grid) + " is illegal for " + kind + " with " +
                                         std::to_string(total_tiles) + " tiles; legal: 1.." + std::to_string(max_grid));
    grid = dbg_grid;
  }
  const bool lean = use_lean && p.tma_out && p.act == TG_ACT_NONE;      // the epilogue variant without activation / direct-store code
  char shp[168];
  snprintf(shp, sizeof shp, "M=%.0f N=%d K=%.0f taps=%d BN=%d tiles=%lld grid=%d st=%d%s%s%s%s", m_valid, p.N, k_valid, p.num_taps,
           p.BN, total_tiles, grid, p.stages, p.tma_out ? (p.ostg2 ? " tma2" : " tma") : "",
           (p.gn_part && p.tma_out) ? " gn" : "", lean ? " lean" : "", sel ? " sel" : "");
  // TMA-store epilogue: the output tensor map has the tile's row dims (extents = logical extents, so ragged edges are clipped
  // by the hardware) and a box of 64 columns x the 32 rows one epilogue warp owns
  if (!p.tma_out) p.gn_part = nullptr;
  CUtensorMap to = ta;
  if (p.tma_out) {
    int left = 32, bx[4], ex[4];
    for (int d = 0; d < 4; ++d) {
      ex[d] = std::max(1, p.ext[d]);
      bx[d] = std::min(p.box[d], left);
      left /= bx[d];
    }
    I2IT_CHECK(left == 1, "TMA-store box: the tile's row box does not factor into 32-row warp boxes");
    to = encode_tmap(TmapSpec("TMA-store output", p.out, {(p.act == TG_ACT_GEGLU) ? p.N / 2 : p.N, ex[0], ex[1], ex[2], ex[3]},
                              {p.ostride[0], p.ostride[1], p.ostride[2], p.ostride[3]}, {64, bx[0], bx[1], bx[2], bx[3]}),
                     dtype);
  }
  p.trace = nullptr;
  if (trace_on) {   // diagnostic timeline (I2IT_TRACE=1): 16 clock64 stamps per CTA, dumped to stderr after each forward
    p.trace = static_cast<unsigned long long*>(dmalloc(static_cast<size_t>(grid) * 16 * sizeof(unsigned long long)));
    I2IT_CUDA(cudaMemset(p.trace, 0, static_cast<size_t>(grid) * 16 * sizeof(unsigned long long)));
    P.traces.push_back({p.trace, grid, std::string(kind) + " " + shp});
  }
  {  // division-free tile decode (see fast_div): dividends are tile indices
    const long long maxd = std::max<long long>(total_tiles, m_tiles) + grid;
    p.magic[0] = make_magic(maxd, p.n_tiles);
    for (int d = 0; d < 4; ++d) p.magic[d + 1] = make_magic(maxd, p.tdim[d]);
    for (int d = 0; d < 5; ++d) I2IT_CHECK(p.magic[d] != 0, "tapgemm: tile space too large for the division-free tile decode");
    p.gn_shift = 0;
    while ((1 << p.gn_shift) < p.gn_red) ++p.gn_shift;
  }
  I2IT_CHECK(tapgemm_for<__half>(lean, p.BN).plain != nullptr, "tapgemm: no kernel instantiated for BN=" + std::to_string(p.BN));
  // a selecting launch (tapgemm_sel_kernel) also takes the alternative maps and TapGemmSel
  CUtensorMap tx = tb, tx2 = tb2;
  TapGemmSel s{};
  if (sel) {
    // the alternative maps have the geometry (and boxes) of the ones they replace; only the base differs
    I2IT_CHECK(p.ksplit <= 1, "tapgemm: a selecting launch cannot split K");
    I2IT_CHECK(sel->s.dir && (sel->s.dim == 0 || sel->s.dim == 2 || sel->s.dim == 3) && sel->s.div >= 1 &&
               (!sel->s.bias == !p.bias), "tapgemm: bad selecting launch");
    tx = encode_tmap(sel->x, dtype);
    tx2 = sb2p ? encode_tmap(sel->x2, dtype) : tx;
    s = sel->s;
    s.magic = make_magic(static_cast<long long>(p.tdim[s.dim]) + 1, s.div);
    I2IT_CHECK(s.magic != 0, "tapgemm: tile space too large for the division-free image decode");
  }
  const bool selecting = sel != nullptr;
  add_op(P, [ta, tb, ta2, tb2, to, p, grid, dt, out_from_io, plan, lean, selecting, tx, tx2, s](cudaStream_t st) {
    TapGemmParams q = p;
    if (out_from_io) q.out = plan->io.out;
    DISPATCH_T(dt, {
      const auto k = tapgemm_for<T>(lean, q.BN);
      if (selecting) launch_k(k.sel, dim3(grid), dim3(TG_THREADS), TG_SMEM, st, 0, ta, tb, ta2, tb2, to, q, tx, tx2, s);
      else launch_k(k.plain, dim3(grid), dim3(TG_THREADS), TG_SMEM, st, 0, ta, tb, ta2, tb2, to, q);
    });
  }, kind, 2.0 * m_valid * p.N * k_valid, bytes, shp);
}

void Engine::launch_rows(Plan& P, const TmapSpec& sa, TmapSpec sb, TapGemmParams p, int M, int heads, int batch, int a_step,
                         int b_head, int b_img, int N, int K, int bn, const char* kind, double k_valid, double bytes,
                         const SelSpec* sel) {
  p.tdim[0] = ceil_div(M, 128); p.tdim[1] = heads; p.tdim[2] = batch; p.tdim[3] = 1;
  p.box[0] = 128; p.box[1] = 1; p.box[2] = 1; p.box[3] = 1;
  p.ext[0] = M; p.ext[1] = heads; p.ext[2] = batch; p.ext[3] = 1;
  p.a_mul[0] = 128; p.a_mul[1] = a_step; p.a_mul[2] = a_step;
  p.b_mul[0] = b_head; p.b_mul[1] = b_img; p.b_mul[2] = 0;
  p.N = N;
  p.BN = bn ? bn : plan_bn(P, 1ll * p.tdim[0] * heads * batch, N, 0);
  p.n_tiles = ceil_div(N, p.BN);
  sb.box[0] = 64; sb.box[1] = p.BN;
  p.num_taps = 1;
  p.kchunks = ceil_div(K, 64);
  p.ocol = 1;
  p.err = d_err;
  launch_gemm(P, sa, sb, p, false, kind, k_valid, bytes, nullptr, nullptr, sel);
}

// ---- TMA views of the GEMM operands that more than one launch describes ----
// NHWC activation as (channel, x, y, image); phase >= 0: every other pixel and row, from parity (phase >> 1, phase & 1)
static TmapSpec act_view(const char* what, const Act& x, int phase, std::initializer_list<int> box) {
  const int s = phase >= 0 ? 2 : 1;
  const long long ld = x.ld, img = x.img();
  const uint16_t* base = phase >= 0 ? x.p + (static_cast<long long>(phase >> 1) * x.W + (phase & 1)) * ld : x.p;
  return TmapSpec(what, base, {x.C, x.W / s, x.H / s, x.N}, {s * ld, s * x.W * ld, img, img}, box);
}

// prepared weight [taps][rows][cin_pad] as (k, row, tap), boxes of 64 x box_rows
static TmapSpec pw_view(const char* what, const PW& w, int box_rows) {
  const long long tap = 1ll * w.rows * w.cin_pad, all = tap * w.taps;
  return TmapSpec(what, w.w, {w.cin_pad, w.rows, w.taps}, {w.cin_pad, tap, all, all}, {64, box_rows});
}

// head-split Q or K: rows [batch][n][heads * d] with pitch t.ld as (channel, token, head, image)
static TmapSpec heads_view(const char* what, const Act& t, int d, int n, int heads, int batch, std::initializer_list<int> box) {
  const long long img = 1ll * n * t.ld;
  return TmapSpec(what, t.p, {d, n, heads, batch}, {t.ld, d, img, img}, box);
}

// V^T [kv_batch][heads * d][vt.ld] as (key, channel, head, image)
static TmapSpec vt_view(const Act& vt, int nk, int d, int heads, int kv_batch, std::initializer_list<int> box) {
  const long long ld = vt.ld, img = 1ll * heads * d * ld;
  return TmapSpec("attention V^T", vt.p, {nk, d, heads, kv_batch}, {ld, d * ld, img, img}, box);
}

Act Engine::conv(Plan& P, const Act& x, const PW& w, const ConvOpts& o_in) {
  // A 3x3 conv's identity residual becomes one more K-slab (second source x identity weights): exact (bf16 * 1.0 accumulated
  // in fp32) and it rides the TMA pipeline instead of latency-bound epilogue loads (+1/9 MMA work; r01: 0.85 -> see profiles)
  if (use_idres && o_in.res && !o_in.x2 && o_in.ksize == 3 && o_in.stride == 1 && o_in.subpixel_phase < 0 && !o_in.out_fp32 &&
      o_in.act != TG_ACT_GEGLU && o_in.res->C == w.rows && w.rows % 8 == 0 && w.rows <= 256 /* wider layers are MMA-bound */ && o_in.res->N == x.N && o_in.res->H == x.H &&
      o_in.res->W == x.W) {
    ConvOpts o2 = o_in;
    const PW ident = prep_identity(w.rows);
    o2.x2 = o_in.res; o2.w2 = &ident; o2.res = nullptr; o2.x2_identity = true;
    return conv(P, x, w, o2);
  }
  if (o_in.stride == 2 && ((x.H | x.W) & 1)) {
    // odd-sized map (latent of an image that is a multiple of 8 but not of 64): the right / bottom zero padding is materialised
    // once so that the 5-D parity view stays a plain box; Ho = ceil(H/2) as F.conv2d(stride=2, padding=1) gives
    return conv(P, pad_even(P, x), w, o_in);
  }
  const ConvOpts& o = o_in;
  const bool sub = o.subpixel_phase >= 0;
  const int k = o.ksize, taps = sub ? 4 : k * k;
  I2IT_CHECK(sub ? (w.taps == 16 && k == 3 && o.stride == 1 && o.out && !o.res && !o.to_io_out_nchw) : (w.taps == taps),
             "conv: weight taps mismatch");
  I2IT_CHECK(x.C == w.cin || x.C == w.cin_pad, "conv: input channels " + std::to_string(x.C) + " vs weight " +
                                                  std::to_string(w.cin));
  I2IT_CHECK(x.ld % 8 == 0, "conv: pixel stride must be a multiple of 8 elements");
  const int Ho = x.H / o.stride, Wo = x.W / o.stride;
  const int gemm_n = w.rows;
  const int outc = (o.act == TG_ACT_GEGLU) ? gemm_n / 2 : gemm_n;

  Act out;
  if (o.out) {
    out = *o.out;
  } else if (!o.to_io_out_nchw) {
    I2IT_CHECK(!o.out_fp32, "conv: fp32 output needs an explicit out view");
    const int ld = round_up(outc, 8);
    const bool small = (outc % 8) != 0;
    out = alloc_act(P, x.N, Ho, Wo, small ? ld : outc, ld, small);
  }

  TmapSpec sa;
  TapGemmParams p;
  std::memset(&p, 0, sizeof p);
  int tw, th, tn;
  const long long ldo = o.to_io_out_nchw ? 0 : out.ld;
  if (o.stride == 1) {
    conv_box(true, x.H, x.W, o.to_io_out_nchw, tw, th, tn);
    sa = act_view("conv x", x, -1, {64, tw, th, tn});
    p.tdim[0] = ceil_div(x.W, tw); p.tdim[1] = ceil_div(x.H, th); p.tdim[2] = ceil_div(x.N, tn); p.tdim[3] = 1;
    p.box[0] = tw; p.box[1] = th; p.box[2] = tn; p.box[3] = 1;
    p.ext[0] = Wo; p.ext[1] = Ho; p.ext[2] = x.N; p.ext[3] = 1;
    p.a_mul[0] = tw; p.a_mul[1] = th; p.a_mul[2] = tn; p.a_mul[3] = 0;
    const int pad = k / 2;
    if (sub) {
      // output parity (py,px): 2x2 taps at low-res offsets (ty-1+py, tx-1+px); output pixel (2y+py, 2x+px)
      const int py = o.subpixel_phase >> 1, px = o.subpixel_phase & 1;
      for (int ty = 0; ty < 2; ++ty)
        for (int tx = 0; tx < 2; ++tx) {
          const int t = ty * 2 + tx;
          p.tap_a[t][0] = 0; p.tap_a[t][1] = tx - 1 + px; p.tap_a[t][2] = ty - 1 + py; p.tap_a[t][3] = 0; p.tap_a[t][4] = 0;
          p.tap_b[t][0] = 0; p.tap_b[t][1] = o.subpixel_phase * 4 + t; p.tap_b[t][2] = 0; p.tap_b[t][3] = 0;
        }
      p.ostride[0] = 2 * ldo; p.ostride[1] = 2ll * (2 * Wo) * ldo;
      p.ostride[2] = 4ll * Ho * Wo * ldo; p.ostride[3] = 0;
    } else {
      for (int ky = 0; ky < k; ++ky)
        for (int kx = 0; kx < k; ++kx) {
          const int t = ky * k + kx;
          p.tap_a[t][0] = 0; p.tap_a[t][1] = kx - pad; p.tap_a[t][2] = ky - pad; p.tap_a[t][3] = 0; p.tap_a[t][4] = 0;
          p.tap_b[t][0] = 0; p.tap_b[t][1] = t; p.tap_b[t][2] = 0; p.tap_b[t][3] = 0;
        }
      p.ostride[0] = ldo; p.ostride[1] = static_cast<long long>(Wo) * ldo;
      p.ostride[2] = static_cast<long long>(Ho) * Wo * ldo; p.ostride[3] = 0;
    }
    p.kchunks = ceil_div(x.C, 64);
  } else {
    I2IT_CHECK(o.stride == 2 && k == 3, "conv: only 3x3 stride-2 is on the path");
    I2IT_CHECK(x.ld % 8 == 0 && x.C % 64 == 0 && x.H % 2 == 0 && x.W % 2 == 0, "conv s2: needs NHWC with ld%8==0, C%64==0, even H/W");
    conv_box(false, Ho, Wo, false, tw, th, tn);
    const long long LD = x.ld;
    // 5-D view (px*ld + c, xo, py, yo, n) of the NHWC input (pixel pitch ld >= C: the input may be a channel slice of a concat
    // buffer): a stride-2 tap is a plain box in this view.  dim 0 spans the C channels of the even pixel, the gap, and the C
    // channels of the odd pixel; boxes only ever start at c or ld + c with c + 64 <= C.
    sa = TmapSpec("conv x", x.p, {LD + x.C, Wo, 2, Ho, x.N}, {2 * LD, x.W * LD, 2 * x.W * LD, 1ll * x.H * x.W * LD},
                  {64, tw, 1, th, tn});
    p.tdim[0] = ceil_div(Wo, tw); p.tdim[1] = 1; p.tdim[2] = ceil_div(Ho, th); p.tdim[3] = ceil_div(x.N, tn);
    p.box[0] = tw; p.box[1] = 1; p.box[2] = th; p.box[3] = tn;
    p.ext[0] = Wo; p.ext[1] = 1; p.ext[2] = Ho; p.ext[3] = x.N;
    p.a_mul[0] = tw; p.a_mul[1] = 0; p.a_mul[2] = th; p.a_mul[3] = tn;
    const int padl = o.asym ? 0 : 1;
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx) {
        const int t = ky * 3 + kx;
        const int ex = kx - padl, ey = ky - padl;
        const int px = ex & 1, py = ey & 1;
        const int ox = (ex - px) / 2, oy = (ey - py) / 2;
        p.tap_a[t][0] = px * x.ld; p.tap_a[t][1] = ox; p.tap_a[t][2] = py; p.tap_a[t][3] = oy; p.tap_a[t][4] = 0;
        p.tap_b[t][0] = 0; p.tap_b[t][1] = t; p.tap_b[t][2] = 0; p.tap_b[t][3] = 0;
      }
    p.ostride[0] = ldo; p.ostride[1] = 0; p.ostride[2] = static_cast<long long>(Wo) * ldo;
    p.ostride[3] = static_cast<long long>(Ho) * Wo * ldo;
    p.kchunks = x.C / 64;
  }

  const long long m_tiles = 1ll * p.tdim[0] * p.tdim[1] * p.tdim[2] * p.tdim[3];
  p.N = gemm_n;
  {
    // whole 64-column store rounds (128 accumulator columns for GEGLU) when the output can take the TMA-store epilogue
    const int acols = (o.act == TG_ACT_GEGLU) ? 128 : 64;
    const bool rounds = use_tmaout && !o.to_io_out_nchw && !o.out_fp32 && gemm_n % acols == 0 && (ldo % 8) == 0;
    p.BN = plan_bn(P, m_tiles, gemm_n, rounds ? acols : 0);
  }
  p.n_tiles = ceil_div(gemm_n, p.BN);
  TmapSpec sb = pw_view("conv weight", w, p.BN);
  p.num_taps = taps;
  p.nprim = taps;
  p.ocol = 1;
  p.out_fp32 = o.out_fp32 ? 1 : 0;
  if (o.to_io_out_nchw) {
    p.out = nullptr;                                   // patched from IO at launch
    const long long hw = static_cast<long long>(Ho) * Wo;
    p.ostride[0] = 1; p.ostride[1] = Wo; p.ostride[2] = hw * outc; p.ostride[3] = 0;
    p.ocol = hw;
  } else if (sub) {
    const int py = o.subpixel_phase >> 1, px = o.subpixel_phase & 1;
    p.out = out.p + (static_cast<long long>(py) * (2 * Wo) + px) * ldo;
  } else {
    p.out = out.p;
  }
  if (o.res) {
    I2IT_CHECK(o.stride == 1, "conv: residual only on stride-1 convs");
    p.res = o.res->p;
    const long long ldr = o.res->ld;
    p.rstride[0] = ldr; p.rstride[1] = static_cast<long long>(Wo) * ldr; p.rstride[2] = static_cast<long long>(Ho) * Wo * ldr;
    p.rcol = 1;
  }
  p.bias = w.bias;
  p.bias_mode = (o.bias_mode >= 0) ? o.bias_mode : (w.bias ? TG_BIAS_COL : TG_BIAS_NONE);
  if (!w.bias) p.bias_mode = TG_BIAS_NONE;
  p.alpha = o.alpha;
  p.act = o.act;
  p.err = d_err;

  // GroupNorm statistics of the output in this GEMM's epilogue (the consumer is a GroupNorm): needs the TMA-store path, a
  // 32-group channel count, and m-tiles that never straddle two images (so a 32-row slot belongs to one image)
  if ((o.gn_out || o.gn_share) && use_gnepi && outc % 64 == 0 && tma_eligible(p, o.to_io_out_nchw) && o.act != TG_ACT_GEGLU) {
    long long mt_img = 0;                 // m-tiles per image
    int images = x.N;
    if (o.gn_rows_per_image > 0) {        // flattened token matrix: 128-row tiles
      if (o.gn_rows_per_image % 128 == 0 && x.rows() % o.gn_rows_per_image == 0) {
        mt_img = o.gn_rows_per_image / 128;
        images = static_cast<int>(x.rows() / o.gn_rows_per_image);
      }
    } else if (tn == 1) {
      mt_img = (o.stride == 1) ? 1ll * p.tdim[0] * p.tdim[1] : 1ll * p.tdim[0] * p.tdim[2];
    }
    if (mt_img > 0) {
      const int cgrp = outc / 32;
      const int red = (cgrp == 4 || cgrp == 8 || cgrp == 16) ? cgrp : 2;
      std::shared_ptr<GnPart> g = o.gn_share;
      if (!g) {
        g = std::make_shared<GnPart>();
        g->red = red; g->C = outc; g->images = images; g->phases = sub ? 4 : 1;
        g->slots_per_image = static_cast<int>(mt_img * 4);
        g->hold = alloc_raw(P, static_cast<size_t>(g->phases) * images * g->slots_per_image * (outc / red) * 2 * sizeof(float));
        g->buf = static_cast<float*>(g->hold.get());
      }
      I2IT_CHECK(g->C == outc && g->slots_per_image == mt_img * 4 && g->images == images, "conv: shared GroupNorm partials mismatch");
      p.gn_part = g->buf;
      p.gn_red = g->red;
      p.gn_slot0 = sub ? o.subpixel_phase * images * g->slots_per_image : 0;
      p.gn_mtiles = static_cast<int>(mt_img * images);
      out.gn = g;
    }
  }

  // split-K for the 8x8 / 1280-channel convs (M = 64 rows per image): with K = 11.5k..23k and 4 m-tiles per batch of 8 the
  // launch had 80-108 weight-bandwidth-bound CTAs; five K ranges per tile write fp32 partials that splitk_reduce sums in a fixed
  // order.  The decision and the ranges depend on the layer only (never on the batch): batch-invariant bits.
  const bool splitk = use_splitk && !sub && k == 3 && o.stride == 1 && !o.to_io_out_nchw && !o.out_fp32 && o.act == TG_ACT_NONE &&
                      x.H * x.W <= 64 && p.kchunks * taps >= 180 && p.kchunks % 5 == 0 && gemm_n >= 640 && gemm_n % 8 == 0;
  std::shared_ptr<void> sk_hold;
  const Act* sk_res = nullptr;
  const float* sk_bias = nullptr;
  if (splitk) {
    const int S = 5;                      // kchunks is 20 or 40 here: equal shares
    const long long Mrows = 1ll * x.N * Ho * Wo;
    sk_hold = alloc_raw(P, static_cast<size_t>(S) * Mrows * gemm_n * sizeof(float));
    p.ksplit = S;
    p.kc_per = ceil_div(p.kchunks, S);
    p.split_ostride = Mrows * gemm_n;
    p.out = sk_hold.get();
    p.out_fp32 = 1;
    p.ostride[0] = gemm_n; p.ostride[1] = 1ll * Wo * gemm_n; p.ostride[2] = 1ll * Ho * Wo * gemm_n; p.ostride[3] = 0;
    sk_res = o.res; sk_bias = (p.bias_mode == TG_BIAS_COL) ? p.bias : nullptr;
    p.res = nullptr; p.bias = nullptr; p.bias_mode = TG_BIAS_NONE;
    p.gn_part = nullptr; out.gn = nullptr;
    p.BN = 256;
    p.n_tiles = ceil_div(gemm_n, p.BN);
    sb.box[1] = p.BN;
  }

  TmapSpec sa2, sb2;
  double k2 = 0;
  if (o.x2) {
    // extra 1x1 "tap" over a second activation tensor with the same spatial geometry as the output
    I2IT_CHECK(o.w2 && o.stride == 1 && o.w2->taps == 1 && o.w2->rows == w.rows, "conv: bad second source");
    const int sm = sub ? 2 : 1;     // sub-pixel: the second source lives at OUTPUT resolution, sampled at this parity
    I2IT_CHECK(o.x2->N == x.N && o.x2->H == sm * Ho && o.x2->W == sm * Wo && (o.x2->C == o.w2->cin || o.x2->C == o.w2->cin_pad),
               "conv: second source shape mismatch");
    I2IT_CHECK(taps + 1 <= TG_MAX_TAPS, "conv: too many taps");
    sa2 = act_view("conv x2", *o.x2, o.subpixel_phase, {64, tw, th, tn});
    sb2 = pw_view("conv w2", *o.w2, p.BN);
    for (int t = 0; t < taps; ++t) { p.tap_src[t] = 0; p.tap_kc[t] = p.kchunks; }
    const int t2 = taps;
    for (int d = 0; d < 5; ++d) p.tap_a[t2][d] = 0;
    for (int d = 0; d < 4; ++d) p.tap_b[t2][d] = 0;
    p.tap_src[t2] = 1;
    p.tap_kc[t2] = ceil_div(o.x2->C, 64);
    p.num_taps = taps + 1;
    k2 = o.x2_identity ? 0 : o.w2->cin;
  }
  SelSpec sel{};
  if (w.dir) {
    // mixed-direction plan: each tile takes its image's weight set, so no tile may hold rows of two images
    const std::string why = " would hold rows of two images (mixed-direction forwards need one image per tile)";
    sel.x = sb; sel.x.base = w.w_alt;
    sel.s.dir = w.dir; sel.s.bias = (p.bias_mode == TG_BIAS_NONE) ? nullptr : w.bias_alt; sel.s.div = 1;
    if (p.bias_mode == TG_BIAS_NONE) p.bias = nullptr;
    if (o.gn_rows_per_image > 0) {                 // flattened token rows: image = 128-row tile / (tiles per image)
      I2IT_CHECK(o.gn_rows_per_image % 128 == 0 && tw == 128 && x.rows() % o.gn_rows_per_image == 0,
                 "conv: a token tile of " + std::to_string(o.gn_rows_per_image) + " rows per image" + why);
      sel.s.dim = 0; sel.s.div = static_cast<int>(o.gn_rows_per_image / 128);
    } else {
      I2IT_CHECK(tn == 1, "conv: a " + std::to_string(x.H) + "x" + std::to_string(x.W) + " tile box" + why);
      sel.s.dim = (o.stride == 1) ? 2 : 3;
    }
    if (o.x2) { sel.x2 = sb2; if (o.w2->w_alt) sel.x2.base = o.w2->w_alt; }   // an identity second source is shared
  }
  {
    const double m_valid = 1.0 * x.N * Ho * Wo, k_valid = 1.0 * taps * w.cin + k2;
    const double bytes = 2.0 * (1.0 * x.N * x.H * x.W * w.cin + m_valid * outc * (o.out_fp32 ? 2 : 1) + 1.0 * gemm_n * k_valid +
                                (o.res ? m_valid * outc : 0) + m_valid * k2);
    const char* kind = sub ? "tapgemm:conv_up2x" : (k == 3) ? (o.stride == 2 ? "tapgemm:conv3x3s2" : "tapgemm:conv3x3") : "tapgemm:linear";
    launch_gemm(P, sa, sb, p, o.to_io_out_nchw, kind, k_valid, bytes, o.x2 ? &sa2 : nullptr, o.x2 ? &sb2 : nullptr,
                w.dir ? &sel : nullptr);
  }
  if (splitk) {
    const float* part = static_cast<const float*>(sk_hold.get());
    const long long Mrows = 1ll * x.N * Ho * Wo, total = Mrows * (gemm_n / 8), sstride = p.split_ostride;
    const uint16_t* rp = sk_res ? sk_res->p : nullptr;
    uint16_t* op = out.p;
    const int ldr = sk_res ? sk_res->ld : 0, ldo2 = out.ld, S = p.ksplit, dt = dtype, Nn = gemm_n;
    const float* bb = sk_bias;
    add_op(P, [=](cudaStream_t st) {
      DISPATCH_T(dt, (launch_k(splitk_reduce_kernel<T>, dim3(ceil_div(total, 256)), dim3(256), 0, st, 0, part, S, sstride, bb,
                               reinterpret_cast<const T*>(rp), ldr, reinterpret_cast<T*>(op), ldo2, Nn, total)));
    }, "splitk_reduce", 0, 4.0 * S * Mrows * gemm_n + 4.0 * Mrows * gemm_n);
  }
  return out;
}

Act Engine::linear(Plan& P, const Act& x, const PW& w, const Act* res, int act, bool gn_out, const Act* out) {
  ConvOpts o;
  o.ksize = 1;
  o.act = act;
  o.gn_out = gn_out;
  o.gn_rows_per_image = static_cast<long long>(x.H) * x.W;
  Act xr = x.as_rows(), rr, orows;
  if (res) { rr = res->as_rows(); o.res = &rr; }
  if (out) { orows = out->as_rows(); o.out = &orows; }
  Act y = conv(P, xr, w, o);
  y.N = x.N; y.H = x.H; y.W = x.W;
  return y;
}

// One ticket counter per image, shared by every GroupNorm launch of a plan: launches are stream-ordered and each one leaves
// the counters at zero (the block that draws the last ticket re-arms it), so graph replays start clean.
int* Engine::gn_counters(Plan& P, int images) {
  I2IT_CHECK(images <= 4096, "group_norm: batch too large for the ticket array");
  if (!P.gn_counter) {
    P.gn_counter = static_cast<int*>(P.pool.get_fresh(4096 * sizeof(int)));
    I2IT_CUDA(cudaMemset(P.gn_counter, 0, 4096 * sizeof(int)));
  }
  return P.gn_counter;
}

Act Engine::group_norm(Plan& P, const Act& x, const NormW& nw, float eps, bool silu) {
  I2IT_CHECK(x.C == nw.C && x.C % 32 == 0 && x.C % 8 == 0, "group_norm: bad channel count " + std::to_string(x.C));
  const int C = x.C, HW = x.H * x.W, cg = C / 32, vecs = C / 8;
  I2IT_CHECK(vecs <= 1024, "group_norm: too many channels");
  // tuning knobs (plan-build time): threads per CTA and CTAs per image
  static const int env_thr = std::getenv("I2IT_GN_THREADS") ? atoi(std::getenv("I2IT_GN_THREADS")) : 128;   // measured best (r01 sweep)
  static const int env_chunks = std::getenv("I2IT_GN_CHUNKS") ? atoi(std::getenv("I2IT_GN_CHUNKS")) : 512;
  const int rows = std::max(1, std::min(1024, env_thr) / vecs), threads = vecs * rows;
  const int chunks = std::max(1, std::min(env_chunks, ceil_div(HW, rows * 4)));
  // statistics pass over the tensor (no epilogue partials available): at most 64 chunk partials per image
  const int schunks = std::min(chunks, 64), spix = ceil_div(HW, schunks);
  const int pix = ceil_div(HW, chunks);
  I2IT_CHECK(chunks <= 1024, "group_norm: too many chunks");
  auto partial = alloc_raw(P, static_cast<size_t>(x.N) * 64 * 32 * sizeof(double) * 2);   // [N][<=64 chunks][32] double2 (or float2)
  auto stats = alloc_raw(P, static_cast<size_t>(x.N) * 64 * sizeof(float));
  Act y = alloc_act(P, x.N, x.H, x.W, C);
  float* d_part = static_cast<float*>(partial.get());
  float* d_stats = static_cast<float*>(stats.get());
  int* d_counter = gn_counters(P, x.N);                // zeroed once at build time; every launch leaves it at zero again
  const uint16_t* xp = x.p;
  uint16_t* yp = y.p;
  const long long ximg = x.img(), yimg = y.img();
  const int ldx = x.ld, ldy = y.ld, N = x.N, dt = dtype, isilu = silu ? 1 : 0;
  const float* g = nw.g;
  const float* b = nw.b;
  const double inv_count = 1.0 / (static_cast<double>(HW) * cg);
  if (x.gn && use_gnepi && x.gn->C == C && x.gn->images == N) {
    // the producer's epilogue already summed the tensor: reduce its per-slot partials (no pass over the tensor itself)
    const GnPart gp = *x.gn;
    const float* pb = gp.buf;
    const int per_row = C / gp.red, epg = cg / gp.red;
    I2IT_CHECK(per_row <= 640, "group_norm: too many partial entries per slot");
    const int nch = std::max(1, std::min(64, gp.slots_per_image / 16));
    const int e_lanes = std::min(256, pow2ceil(per_row));
    double2* p2 = reinterpret_cast<double2*>(d_part);
    add_op(P, [=](cudaStream_t st) {
      launch_k(gn_part_reduce_kernel, dim3(nch, N), dim3(256), 0, st, 0, pb, gp.phases, gp.images, gp.slots_per_image, per_row, epg,
               e_lanes, p2, d_counter, inv_count, eps, d_stats);
    }, "gn_final_part", 0, 8.0 * gp.phases * N * gp.slots_per_image * per_row);
  } else {
    add_op(P, [=](cudaStream_t st) {
      DISPATCH_T(dt, (launch_k(gn_stats_kernel<T>, dim3(schunks, N), dim3(threads), static_cast<size_t>(rows) * 2 * C * sizeof(float), st, 0,
                               reinterpret_cast<const T*>(xp), ximg, ldx, C, HW, cg, spix, d_part, d_counter, inv_count, eps, d_stats)));
    }, "gn_stats", 0, 2.0 * N * HW * C);
  }
  if (nw.dir) {   // mixed-direction plan: image n takes its direction's gamma / beta
    const int* dir = nw.dir;
    const float* g2 = nw.g_alt;
    const float* b2 = nw.b_alt;
    add_op(P, [=](cudaStream_t st) {
      DISPATCH_T(dt, (launch_k(gn_apply_sel_kernel<T>, dim3(chunks, N), dim3(threads), 0, st, 0,
                         reinterpret_cast<const T*>(xp), ximg, ldx, reinterpret_cast<T*>(yp), yimg, ldy, C, HW, cg, pix,
                         d_stats, g, b, isilu, dir, g2, b2)));
    }, "gn_apply_sel", 0, 4.0 * N * HW * C);
    return y;
  }
  add_op(P, [=](cudaStream_t st) {
    DISPATCH_T(dt, (launch_k(gn_apply_kernel<T>, dim3(chunks, N), dim3(threads), 0, st, 0,
                       reinterpret_cast<const T*>(xp), ximg, ldx, reinterpret_cast<T*>(yp), yimg, ldy, C, HW, cg, pix,
                       d_stats, g, b, isilu)));
  }, "gn_apply", 0, 4.0 * N * HW * C);
  return y;     // (y carries no statistics: it is a different tensor)
}

Act Engine::layer_norm(Plan& P, const Act& x, const NormW& nw, bool to_io_out) {
  I2IT_CHECK(x.C == nw.C && x.C % 8 == 0 && x.C <= 1280, "layer_norm: C must be a multiple of 8 and <= 1280");
  Act y = to_io_out ? x : alloc_act(P, x.N, x.H, x.W, x.C);       // to_io_out: dense rows straight into the caller's buffer
  const long long rows = x.rows();
  const uint16_t* xp = x.p;
  uint16_t* yp = to_io_out ? nullptr : y.p;
  const int ldx = x.ld, ldy = to_io_out ? x.C : y.ld, C = x.C, dt = dtype;
  const float* g = nw.g;
  const float* b = nw.b;
  Plan* plan = &P;
  add_op(P, [=](cudaStream_t st) {
    uint16_t* dst = yp ? yp : static_cast<uint16_t*>(plan->io.out);
    DISPATCH_T(dt, (launch_k(layernorm_kernel<T>, dim3(ceil_div(rows * 32, 256)), dim3(256), 0, st, 0,
                       reinterpret_cast<const T*>(xp), ldx, reinterpret_cast<T*>(dst), ldy, static_cast<int>(rows), C, g, b,
                       1e-5f)));
  }, "layernorm", 0, 4.0 * rows * C);
  return y;
}

Act Engine::upsample_to(Plan& P, const Act& x, int Ho, int Wo) {
  Act y = alloc_act(P, x.N, Ho, Wo, x.C);
  const long long total = static_cast<long long>(x.N) * Ho * Wo * (x.C / 8);
  const uint16_t* xp = x.p;
  uint16_t* yp = y.p;
  const int ldx = x.ld, ldy = y.ld, H = x.H, W = x.W, C = x.C, dt = dtype;
  const float sh = static_cast<float>(H) / static_cast<float>(Ho), sw = static_cast<float>(W) / static_cast<float>(Wo);
  const double N_ = x.N;
  add_op(P, [=](cudaStream_t st) {
    DISPATCH_T(dt, (launch_k(upsample_nearest_kernel<T>, dim3(ceil_div(total, 256)), dim3(256), 0, st, 0, reinterpret_cast<const T*>(xp),
                             ldx, reinterpret_cast<T*>(yp), ldy, H, W, Ho, Wo, sh, sw, C, total)));
  }, "upsample_nearest", 0, 2.0 * N_ * C * (1.0 * H * W + 1.0 * Ho * Wo));
  return y;
}

Act Engine::pad_even(Plan& P, const Act& x) {
  const int H2 = x.H + (x.H & 1), W2 = x.W + (x.W & 1);
  if (H2 == x.H && W2 == x.W && x.ld == x.C) return x;
  Act y = alloc_act(P, x.N, H2, W2, x.C);
  const long long total = static_cast<long long>(x.N) * H2 * W2 * (x.C / 8);
  const uint16_t* xp = x.p;
  uint16_t* yp = y.p;
  const int ldx = x.ld, H = x.H, W = x.W, C = x.C, dt = dtype;
  add_op(P, [=](cudaStream_t st) {
    DISPATCH_T(dt, (launch_k(pad_copy_kernel<T>, dim3(ceil_div(total, 256)), dim3(256), 0, st, 0, reinterpret_cast<const T*>(xp), ldx,
                             reinterpret_cast<T*>(yp), H, W, H2, W2, C, total)));
  }, "pad_even", 0, 4.0 * total * 8);
  return y;
}

void Engine::copy_channels(Plan& P, const Act& src, const Act& dst) {
  I2IT_CHECK(src.C == dst.C && src.rows() == dst.rows() && src.C % 8 == 0, "copy_channels: shape mismatch");
  const long long total = src.rows() * (src.C / 8);
  const uint16_t* xp = src.p;
  uint16_t* yp = dst.p;
  const int ldx = src.ld, ldy = dst.ld, C = src.C, dt = dtype;
  add_op(P, [=](cudaStream_t st) {
    DISPATCH_T(dt, (launch_k(copy2d_kernel<T>, dim3(ceil_div(total, 256)), dim3(256), 0, st, 0, reinterpret_cast<const T*>(xp), ldx,
                                                                         reinterpret_cast<T*>(yp), ldy, C, total)));
  }, "concat_copy", 0, 4.0 * total * 8);
}

Act Engine::replicate_image(Plan& P, const Act& src, int n) {
  I2IT_CHECK(src.N == 1 && src.C % 8 == 0 && n >= 1, "replicate_image: needs one image with C % 8 == 0");
  Act y = alloc_act(P, n, src.H, src.W, src.C);
  const long long rows = src.rows(), total = rows * n * (src.C / 8);
  const uint16_t* xp = src.p;
  uint16_t* yp = y.p;
  const int ldx = src.ld, C = src.C, dt = dtype;
  const std::string shape = std::to_string(n) + "x" + std::to_string(src.H) + "x" + std::to_string(src.W) + "x" + std::to_string(C);
  add_op(P, [=](cudaStream_t st) {
    DISPATCH_T(dt, (launch_k(replicate_image_kernel<T>, dim3(ceil_div(total, 256)), dim3(256), 0, st, 0,
                             reinterpret_cast<const T*>(xp), ldx, reinterpret_cast<T*>(yp), C, C, rows, total)));
  }, "replicate", 0, 2.0 * rows * C * (n + 1), shape);
  return y;
}

Act Engine::vt_proj(Plan& P, const Act& x, int B, int ntok, const PW& wv) {
  I2IT_CHECK(x.rows() == static_cast<long long>(B) * ntok, "vt_proj: token count mismatch");
  I2IT_CHECK(x.C == wv.cin || x.C == wv.cin_pad, "vt_proj: width mismatch");
  const int C = wv.rows, ldv = round_up(ntok, 8);
  Act vt = alloc_act(P, B, 1, C, ldv, ldv);      // [B][C rows][ldv]; "C" field carries the padded token count
  Act tokens = x;                                 // as [B, 1, ntok, C]
  tokens.N = B; tokens.H = 1; tokens.W = ntok;
  const TmapSpec sa = pw_view("vt_proj weight", wv, 128), sb = act_view("vt_proj x", tokens, -1, {});
  TapGemmParams p;
  std::memset(&p, 0, sizeof p);
  p.out = vt.p;
  p.ostride[0] = ldv; p.ostride[1] = 0; p.ostride[2] = static_cast<long long>(C) * ldv; p.ostride[3] = 0;
  p.bias = wv.bias;
  p.bias_mode = wv.bias ? TG_BIAS_ROW : TG_BIAS_NONE;
  p.alpha = 1.f;
  SelSpec sel{};
  if (wv.dir) {   // mixed-direction plan: the weight is the row operand, so the selection takes A and the row bias; t[2] = image
    sel.x = sa; sel.x.base = wv.w_alt;
    sel.s.dir = wv.dir; sel.s.bias = wv.bias_alt; sel.s.dim = 2; sel.s.div = 1; sel.s.sel_a = 1;
  }
  launch_rows(P, sa, sb, p, C, 1, B, 0, 0, 1, ntok, x.C, 0, "tapgemm:vt", wv.cin,
              2.0 * (1.0 * C * wv.cin + 1.0 * B * ntok * wv.cin + 1.0 * B * C * ntok), wv.dir ? &sel : nullptr);
  return vt;
}

Act Engine::attention(Plan& P, const Act& q, const Act& k, const Act& vt, int B, int Nq, int Nk, int heads, int d,
                      int kv_batch) {
  if (d == FA_D && use_flash) return flash_attention(P, q, k, vt, B, Nq, Nk, heads, kv_batch);
  // The VAE attention (one head of 512) goes fused only where the unfused S + P buffers grow large (N*N*6 bytes per image:
  // 0.4 GB at Nk = 8192, 100 GB at 4K).  The rule reads the per-image shape only, so every image of a batch takes the same
  // path as its batch-1 call.  At and below 8192 keys (every 512^2 forward) the unfused path is kept as it was.
  if (d == FA5_D && heads == 1 && Nk > 8192 && use_flash) return flash_attention512(P, q, k, vt, B, Nq, Nk, kv_batch);
  I2IT_CHECK(d % 64 == 0 && (d <= 256 || d % 256 == 0), "attention: head dim must be a multiple of 64");

  I2IT_CHECK(kv_batch == B || kv_batch == 1, "attention: kv batch must be 1 or B");
  const int C = heads * d, lds = round_up(Nk, 8);
  const long long rows = static_cast<long long>(B) * heads * Nq;
  auto sbuf = alloc_raw(P, static_cast<size_t>(rows) * lds * sizeof(float));
  auto pbuf = alloc_raw(P, static_cast<size_t>(rows) * lds * 2);
  float* S = static_cast<float*>(sbuf.get());
  uint16_t* Pm = static_cast<uint16_t*>(pbuf.get());
  Act out = alloc_act(P, B, 1, Nq, C);
  const int kvb = (kv_batch == B) ? 1 : 0;

  {  // S = alpha * Q K^T   (fp32 logits)
    const TmapSpec sa = heads_view("attention Q", q, d, Nq, heads, B, {64, 128}),
                   sb = heads_view("attention K", k, d, Nk, heads, kv_batch, {});
    TapGemmParams p;
    std::memset(&p, 0, sizeof p);
    p.out = S;
    p.out_fp32 = 1;
    p.ostride[0] = lds; p.ostride[1] = static_cast<long long>(Nq) * lds; p.ostride[2] = static_cast<long long>(heads) * Nq * lds;
    p.alpha = 1.0f / sqrtf(static_cast<float>(d));
    launch_rows(P, sa, sb, p, Nq, heads, B, 1, 1, kvb, Nk, d, 0, "tapgemm:attn_qk", d,
                2.0 * B * heads * (1.0 * Nq * d + 1.0 * Nk * d) + 4.0 * rows * Nk);
  }
  {  // P = softmax(S)
    const int dt = dtype;
    if (Nk > 4096) {
      add_op(P, [=](cudaStream_t st) {
        DISPATCH_T(dt, (launch_k(softmax_long_kernel<T>, dim3(static_cast<unsigned>(rows)), dim3(256), 0, st, 0, S, lds, reinterpret_cast<T*>(Pm),
                                                                                          lds, Nk, lds)));
      }, "softmax", 0, 6.0 * rows * Nk, "long");
    } else if (Nk > 1024) {
      add_op(P, [=](cudaStream_t st) {
        DISPATCH_T(dt, (launch_k(softmax_kernel<T, 128>, dim3(static_cast<unsigned>(rows)), dim3(128), 0, st, 0, S, lds, reinterpret_cast<T*>(Pm), lds,
                                                                                          rows, Nk, lds)));
      }, "softmax", 0, 6.0 * rows * Nk, "128");
    } else {
      add_op(P, [=](cudaStream_t st) {
        DISPATCH_T(dt, (launch_k(softmax_kernel<T, 32>, dim3(static_cast<unsigned>((rows + 3) / 4)), dim3(128), 0, st, 0,
                           S, lds, reinterpret_cast<T*>(Pm), lds, rows, Nk, lds)));
      }, "softmax", 0, 6.0 * rows * Nk, "32");
    }
  }
  {  // O = P V   (V given transposed: [kvB][C][ldv])
    const long long plane = 1ll * Nq * lds, img = plane * heads;
    const TmapSpec sa("attention P", Pm, {Nk, Nq, heads, B}, {lds, plane, img, img}, {64, 128}),
                   sb = vt_view(vt, Nk, d, heads, kv_batch, {});
    TapGemmParams p;
    std::memset(&p, 0, sizeof p);
    p.out = out.p;
    p.ostride[0] = out.ld; p.ostride[1] = d; p.ostride[2] = static_cast<long long>(Nq) * out.ld;
    p.alpha = 1.f;
    launch_rows(P, sa, sb, p, Nq, heads, B, 1, 1, kvb, d, Nk, std::min(d, 256), "tapgemm:attn_pv", Nk,
                2.0 * (1.0 * rows * Nk + 1.0 * B * heads * Nk * d + 1.0 * rows * d));
  }
  return out;
}

// the FlashParams both fused attentions fill: query tiles of bm rows, out [B * Nq][out.ld]
static FlashParams flash_params(const Act& out, int B, int Nq, int Nk, int heads, int kv_batch, int d, int bm, int* err) {
  I2IT_CHECK(kv_batch == B || kv_batch == 1, "attention: kv batch must be 1 or B");
  FlashParams fp;
  std::memset(&fp, 0, sizeof fp);
  fp.Nq = Nq; fp.Nk = Nk; fp.heads = heads; fp.B = B;
  fp.q_tiles = ceil_div(Nq, bm);
  fp.kv_bmul = (kv_batch == B) ? 1 : 0;
  fp.scale_log2e = (1.0f / sqrtf(static_cast<float>(d))) * 1.4426950408889634f;
  fp.out = out.p;
  fp.ldo = out.ld;
  fp.err = err;
  return fp;
}

Act Engine::flash_attention(Plan& P, const Act& q, const Act& k, const Act& vt, int B, int Nq, int Nk, int heads, int kv_batch,
                            bool causal) {
  const int d = FA_D, C = heads * d;
  Act out = alloc_act(P, B, 1, Nq, C);
  FlashParams fp = flash_params(out, B, Nq, Nk, heads, kv_batch, d, FA_BM, d_err);
  fp.causal = causal ? 1 : 0;
  const CUtensorMap tq = encode_tmap(heads_view("attention Q", q, d, Nq, heads, B, {64, FA_BM}), dtype),
                    tk = encode_tmap(heads_view("attention K", k, d, Nk, heads, kv_batch, {64, FA_BN}), dtype),
                    tv = encode_tmap(vt_view(vt, Nk, d, heads, kv_batch, {FA_BN, d}), dtype);
  const int grid = fp.q_tiles * heads * B, dt = dtype;
  char shp[96];
  snprintf(shp, sizeof shp, "B=%d h=%d Nq=%d Nk=%d d=%d", B, heads, Nq, Nk, d);
  add_op(P, [=](cudaStream_t st) {
    DISPATCH_T(dt, (launch_k(flash_attn_kernel<T>, dim3(grid), dim3(FA_THREADS), FA_SMEM, st, 0, tq, tk, tv, fp)));
  }, "flash_attn", 4.0 * B * heads * Nq * Nk * d, 2.0 * (2.0 * B * Nq * C + 2.0 * kv_batch * Nk * C), shp);
  return out;
}

Act Engine::flash_attention512(Plan& P, const Act& q, const Act& k, const Act& vt, int B, int Nq, int Nk, int kv_batch) {
  const int d = FA5_D;
  Act out = alloc_act(P, B, 1, Nq, d);
  const FlashParams fp = flash_params(out, B, Nq, Nk, 1, kv_batch, d, FA5_BM, d_err);
  // 3-D maps: the kernel addresses (channel or key, token or channel, image)
  const CUtensorMap tq = encode_tmap(TmapSpec("attention Q", q.p, {d, Nq, B}, {q.ld, 1ll * Nq * q.ld}, {64, FA5_BM}), dtype),
                    tk = encode_tmap(TmapSpec("attention K", k.p, {d, Nk, kv_batch}, {k.ld, 1ll * Nk * k.ld}, {64, FA5_BN}), dtype),
                    tv = encode_tmap(TmapSpec("attention V^T", vt.p, {Nk, d, kv_batch}, {vt.ld, 1ll * d * vt.ld}, {FA5_BN, 64}),
                                     dtype);
  const long long grid = 2ll * fp.q_tiles * B;
  I2IT_CHECK(grid < (1ll << 31), "attention: too many query tiles");
  const int dt = dtype;
  char shp[96];
  snprintf(shp, sizeof shp, "B=%d h=1 Nq=%d Nk=%d d=%d", B, Nq, Nk, d);
  add_op(P, [=](cudaStream_t st) {
    DISPATCH_T(dt, (launch_k(flash_attn512_kernel<T>, dim3(static_cast<unsigned>(grid)), dim3(FA5_THREADS), FA5_SMEM, st, 0,
                             tq, tk, tv, fp)));
  }, "flash_attn512", 4.0 * B * Nq * Nk * d, 2.0 * (2.0 * B * Nq * d + 2.0 * kv_batch * Nk * d), shp);
  return out;
}

// ---------------------------------------------------------------------------------------------
// executor
// ---------------------------------------------------------------------------------------------
void Engine::set_text(const void* text, int text_batch, cudaStream_t st) {
  I2IT_CHECK(finalized_, "i2it_finalize_weights must be called before i2it_set_text");
  I2IT_CHECK(text != nullptr && text_batch > 0, "i2it_set_text: null text embedding");
  auto& slot = textkv_[text_batch];
  if (!slot) {
    slot.reset(new TextKV());
    slot->text_batch = text_batch;
    build_text_kv(*slot);
  }
  TextKV& T = *slot;
  T.plan.io.text = text;
  nvtxRangePushA("i2it:text_kv");
  g_pdl.enabled = false; g_pdl.prev_is_kernel = false;
  for (auto& op : T.plan.ops) op(st);
  nvtxRangePop();
  I2IT_CUDA(cudaGetLastError());
  T.filled = true;
}

// CLIP text tower on the engine (SURVEY 8f #1; transformers models/clip/modeling_clip.py CLIPTextTransformer.forward): token +
// position embeddings, pre-LN transformer layers with CAUSAL self-attention (16 heads x 64 for SD-Turbo's OpenCLIP-H tower) and a
// GELU MLP, final LayerNorm -> last_hidden_state, i.e. `text_encoder(tokens)[0]` of src/pix2pix_turbo.py:190-196.
// Same kernels as the image path: tapgemm (fused q|k projection, V^T projection with row bias, GELU in the fc1 epilogue, residual
// adds in the out_proj / fc2 epilogues), flash_attn with the causal flag, layernorm.
void Engine::encode_text(const int* tokens, int batch, void* out, cudaStream_t st) {
  I2IT_CHECK(finalized_, "i2it_finalize_weights must be called before i2it_encode_text");
  I2IT_CHECK(tokens && out && batch > 0, "i2it_encode_text: bad arguments");
  I2IT_CHECK(has_text_encoder(), "no text_encoder.* weights were registered (i2it_set_weight)");
  auto& slot = textenc_[batch];
  if (!slot) {
    slot.reset(new Plan());
    Plan& P = *slot;
    const std::string te = "text_encoder.text_model";
    const WT& tok = raw(te + ".embeddings.token_embedding", "weight");
    const WT& pos = raw(te + ".embeddings.position_embedding", "weight");
    const int C = static_cast<int>(tok.shape[1]), vocab = static_cast<int>(tok.shape[0]), ntok = static_cast<int>(pos.shape[0]);
    I2IT_CHECK(C % 64 == 0 && C <= 1280, "text encoder width must be a multiple of 64 (64-wide heads) and <= 1280");
    const int heads = cfg.text_heads > 0 ? cfg.text_heads : C / 64;
    I2IT_CHECK(heads * 64 == C, "text encoder: head_dim must be 64");
    const int act = cfg.text_act == 1 ? TG_ACT_QUICKGELU : TG_ACT_GELU;
    int layers = 0;
    while (has(te + ".encoder.layers." + std::to_string(layers) + ".layer_norm1.weight")) ++layers;
    I2IT_CHECK(layers > 0, "text encoder: no layers found");
    Act x = alloc_act(P, batch, 1, ntok, C);
    {
      const long long total = static_cast<long long>(batch) * ntok * (C / 8);
      uint16_t* xp = x.p;
      const float* tp = tok.d;
      const float* pp = pos.d;
      const int dt = dtype;
      Plan* plan = &P;
      add_op(P, [=](cudaStream_t s2) {
        DISPATCH_T(dt, (launch_k(clip_embed_kernel<T>, dim3(ceil_div(total, 256)), dim3(256), 0, s2, 0,
                           reinterpret_cast<const int*>(plan->io.x), tp, pp, reinterpret_cast<T*>(xp), C, ntok, vocab, total)));
      }, "clip_embed", 0, 2.0 * total * 8 * 3);
    }
    // keep_stages >= 2: every layer output under its transformers state-dict prefix (tests/text_audit.py); no launches added
    mark_layer(P, te + ".embeddings", x);
    for (int l = 0; l < layers; ++l) {
      const std::string L = te + ".encoder.layers." + std::to_string(l);
      Act n = layer_norm(P, x, norm(L + ".layer_norm1"));
      mark_layer(P, L + ".layer_norm1", n);
      Act qk = linear(P, n, prep(L + ".qk", {L + ".self_attn.q_proj", L + ".self_attn.k_proj"}));
      mark_layer(P, L + ".self_attn.qk", qk);
      Act vt = vt_proj(P, n, batch, ntok, prep(L + ".self_attn.v_proj", {L + ".self_attn.v_proj"}));
      mark_layer(P, L + ".self_attn.v_proj", vt);
      Act a = flash_attention(P, qk.slice(0, C), qk.slice(C, C), vt, batch, ntok, ntok, heads, batch, /*causal=*/true);
      a.N = batch; a.H = 1; a.W = ntok;
      mark_layer(P, L + ".self_attn", a);
      x = linear(P, a, prep(L + ".self_attn.out_proj", {L + ".self_attn.out_proj"}), &x);
      mark_layer(P, L + ".self_attn.out_proj", x);
      Act m = layer_norm(P, x, norm(L + ".layer_norm2"));
      mark_layer(P, L + ".layer_norm2", m);
      Act h = linear(P, m, prep(L + ".mlp.fc1", {L + ".mlp.fc1"}), nullptr, act);
      mark_layer(P, L + ".mlp.fc1", h);
      x = linear(P, h, prep(L + ".mlp.fc2", {L + ".mlp.fc2"}), &x);
      mark_layer(P, L + ".mlp.fc2", x);
    }
    layer_norm(P, x, norm(te + ".final_layer_norm"), /*to_io_out=*/true);
    P.keep.push_back(x.hold);
    flush_prep();
    I2IT_CUDA(cudaDeviceSynchronize());
  }
  Plan& P = *slot;
  P.io.x = tokens;
  P.io.out = out;
  last_text_plan_ = &P;
  nvtxRangePushA("i2it:clip_text_encoder");
  g_pdl.enabled = false; g_pdl.prev_is_kernel = false;
  for (auto& op : P.ops) op(st);
  nvtxRangePop();
  I2IT_CUDA(cudaGetLastError());
}

bool Engine::check_forward(int B, int H, int W, int text_batch, const void* text) const {
  I2IT_CHECK(H % 8 == 0 && W % 8 == 0 && H > 0 && W > 0, "H and W must be positive multiples of 8 (as the reference CLIs crop them)");
  I2IT_CHECK(B > 0 && (text_batch == 1 || text_batch == B), "text_batch must be 1 or batch");
  if (text) return false;
  auto it = textkv_.find(text_batch);
  I2IT_CHECK(it != textkv_.end() && it->second->filled,
             "text_emb == NULL: call i2it_set_text first (and again after every i2it_finalize_weights or i2it_refold_weights)");
  return true;
}

void Engine::forward(const i2it_forward_desc& d, cudaStream_t st) {
  const int B = d.batch, H = d.H, W = d.W;
  const i2it_resize_desc* g = d.geometry;
  const bool u8 = d.x_u8 || d.out_u8, ragged = d.x_u8_list || d.out_u8_list, mixed = d.directions != nullptr;
  // the requests include/i2it.h lists; every other combination is refused before its operands are looked at
  I2IT_CHECK((d.x || d.out) + u8 + ragged <= 1,
             "i2it_forward: one image boundary per request: x / out, x_u8 / out_u8 or x_u8_list / out_u8_list");
  I2IT_CHECK(!g || u8 || ragged, "i2it_forward: a resize geometry needs a uint8 input (x_u8 or x_u8_list), not the NCHW x");
  I2IT_CHECK(!(d.shared_input && ragged), "i2it_forward: shared_input (variations of one image) with a ragged x_u8_list");
  I2IT_CHECK(!(mixed && d.shared_input), "mixed-direction forward: directions with shared_input (variations of one image)");
  I2IT_CHECK(!(mixed && u8), "mixed-direction forward: directions with the uint8 x_u8 (a mixed uint8 batch is a ragged x_u8_list)");
  I2IT_CHECK(!(mixed && d.noise_map), "mixed-direction forward: directions with a noise_map (CycleGAN has none)");
  I2IT_CHECK(mixed || d.direction == I2IT_A2B || d.direction == I2IT_B2A,
             "i2it_forward: direction " + std::to_string(d.direction) + " is neither I2IT_A2B (0) nor I2IT_B2A (1)");
  I2IT_CHECK(B >= 1, "i2it_forward: batch size n must be >= 1");
  if (u8 || ragged)
    I2IT_CHECK(d.in_mode >= 0 && d.in_mode <= 2, "i2it_forward: in_mode must be I2IT_IN_UNIT, I2IT_IN_NORMALIZE or I2IT_IN_SKETCH");
  int direction = d.direction;
  if (mixed) { check_mixed(d.directions, B, H, W); direction = DIR_MIXED; }
  const bool text_cached = check_forward(B, H, W, d.text_batch, d.text_emb);
  IO io;
  std::memset(&io, 0, sizeof io);
  io.text = d.text_emb; io.eps = d.eps; io.noise = d.noise_map; io.r = d.r; io.out_latent = d.out_latent;
  if (u8 || ragged) io.in_mode = d.in_mode;
  if (!ragged) {
    io.x = d.x; io.x_u8 = d.x_u8; io.out = d.out; io.out_u8 = d.out_u8;
    I2IT_CHECK((io.x || io.x_u8) && io.eps && (io.out || io.out_u8), "null input/output pointer");
    if (g) {
      rs_check_geometry(*g, H, W);
      // nothing to resize or crop: the plan (and its key) of the plain uint8 forward
      if (g->in_H == H && g->in_W == W && g->resize_H == H && g->resize_W == W && g->out_H == H && g->out_W == W) g = nullptr;
    }
    // one variation of one image is the plain batch-1 forward: same plan, same output
    const int io_mode = (u8 ? IO_U8_IN | IO_U8_OUT : 0) | (d.shared_input && B > 1 ? IO_SHARED_IN : 0);
    Plan* P = plan_for(B, H, W, direction, d.text_batch, text_cached, io_mode, g, /*evict=*/false);
    if (u8) io.out = P->u8_out_tmp;
    run(P, io, st, mixed ? stage_dirs(P, d.directions, B) : nullptr);
    return;
  }
  const void* const* x = d.x_u8_list;
  void* const* out = d.out_u8_list;
  I2IT_CHECK(x && out && g, "ragged forward: null image or geometry array");
  rs_check_ragged(g, B, H, W, d.max_side);    // before the pointers: an empty output (a zero size) has a null one
  for (int i = 0; i < B; ++i)
    I2IT_CHECK(x[i] && out[i], "ragged forward: null image pointer (image " + std::to_string(i) + ")");
  I2IT_CHECK(io.eps, "null input/output pointer");
  // the tables first: a size pair the table builder refuses fails here, before a plan is built or anything is enqueued
  for (int i = 0; i < B; ++i) {
    const int pairs[4][2] = {{g[i].in_H, g[i].resize_H}, {g[i].in_W, g[i].resize_W}, {H, g[i].out_H}, {W, g[i].out_W}};
    for (const auto& pr : pairs)
      if (pr[0] != pr[1]) rs_tables_.get(pr[0], pr[1]);
  }
  // the images live in the descriptors, not in the launches: the graph cache key holds no image pointer
  Plan* P = plan_for(B, H, W, direction, d.text_batch, text_cached, IO_U8_IN | IO_U8_OUT | IO_RAGGED, nullptr, /*evict=*/false,
                     d.max_side);
  io.out = P->u8_out_tmp;
  const RsCall c = rs_forward_call(g, B, H, W, d.max_side, rs_tables_, x, out, &P->rg);
  for (int k = 0; k < 4; ++k) P->meta[P->rg.ops[k]].bytes = c.bytes[k];   // i2it_profile: this call's geometries
  const size_t bytes = stage_ragged(c, P->rg.dev_bytes);
  char* dev = P->rg.dev;
  const char* blob = rs_blob_;
  const std::function<void(cudaStream_t)> dir_copy = mixed ? stage_dirs(P, d.directions, B) : nullptr;
  run(P, io, st, [=](cudaStream_t s) {
    I2IT_CUDA(cudaMemcpyAsync(dev, blob, bytes, cudaMemcpyHostToDevice, s));
    I2IT_CUDA(cudaEventRecord(rs_ev_, s));
    if (dir_copy) dir_copy(s);
  });
}

std::string mixed_size_rule(int H, int W) {
  const std::string hw = std::to_string(H) + "x" + std::to_string(W);
  if (H <= 0 || W <= 0 || H % 8 || W % 8) return "H and W must be positive multiples of 8";
  const long long tok = 1ll * (H / 8) * (W / 8);
  if (tok % 128 != 0)
    return hw + " is refused: the VAE attention's token launches need (H/8)*(W/8) = " + std::to_string(tok) +
           " latent pixels per image to be a multiple of 128, so that no 128-row tile holds rows of two images";
  // the VAE's convs: stride 1 on every level H/2^k x W/2^k (k = 0..3; the final image's launch on level 0), stride 2 into
  // levels 1..3.  The box shrinks with the map, but every level is checked as the picker sees it.
  for (int k = 0; k < 4; ++k) {
    const int h = H >> k, w = W >> k;
    int tw, th, tn;
    const bool kinds[3][2] = {{true, false}, {true, k == 0}, {false, false}};
    for (int i = 0; i < 3; ++i) {
      if (i == 2 && k == 0) continue;       // no stride-2 conv writes level 0
      conv_box(kinds[i][0], h, w, kinds[i][1], tw, th, tn);
      if (tn != 1)
        return hw + " is refused: a VAE conv on its " + std::to_string(h) + "x" + std::to_string(w) + " map has a " +
               std::to_string(tw) + "x" + std::to_string(th) + "-pixel tile box that spans " + std::to_string(tn) +
               " images (one image per 128-row tile needs the box to fill 128 pixels of one image)";
    }
  }
  return "";
}

void Engine::check_mixed(const int* dirs, int B, int H, int W) const {
  I2IT_CHECK(cfg.model_kind == I2IT_CYCLEGAN, "mixed-direction forward: a pix2pix handle has one VAE; directions are CycleGAN's");
  for (int i = 0; i < B; ++i)
    I2IT_CHECK(dirs[i] == I2IT_A2B || dirs[i] == I2IT_B2A, "mixed-direction forward: direction " + std::to_string(dirs[i]) +
                                                                " of image " + std::to_string(i) + " is neither I2IT_A2B (0) nor I2IT_B2A (1)");
  const std::string why = mixed_size_rule(H, W);
  I2IT_CHECK(why.empty(), "mixed-direction forward: " + why);
}

std::function<void(cudaStream_t)> Engine::stage_dirs(Plan* P, const int* dirs, int B) {
  I2IT_CHECK(P->dir != nullptr, "mixed-direction forward: the plan has no direction array");
  I2IT_CUDA(cudaEventSynchronize(dir_ev_));     // the previous call's copy has read the blob
  if (B > dir_blob_cap_) {
    if (dir_blob_) I2IT_CUDA(cudaFreeHost(dir_blob_));
    dir_blob_ = nullptr;
    dir_blob_cap_ = 0;
    I2IT_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&dir_blob_), static_cast<size_t>(B) * sizeof(int), cudaHostAllocDefault));
    dir_blob_cap_ = B;
  }
  std::memcpy(dir_blob_, dirs, static_cast<size_t>(B) * sizeof(int));
  int* dev = P->dir;
  const int* blob = dir_blob_;
  cudaEvent_t ev = dir_ev_;
  return [=](cudaStream_t s) {
    I2IT_CUDA(cudaMemcpyAsync(dev, blob, static_cast<size_t>(B) * sizeof(int), cudaMemcpyHostToDevice, s));
    I2IT_CUDA(cudaEventRecord(ev, s));
  };
}

size_t Engine::stage_ragged(const RsCall& c, size_t cap) {
  const size_t dbytes = c.d.size() * sizeof(RsPass), bytes = dbytes + c.tab.size() * sizeof(int);
  I2IT_CHECK(bytes <= cap, "ragged resize: the call's tables exceed the plan's bound");
  I2IT_CUDA(cudaEventSynchronize(rs_ev_));      // the previous call's copy has read the blob
  if (bytes > rs_blob_cap_) {
    if (rs_blob_) I2IT_CUDA(cudaFreeHost(rs_blob_));
    rs_blob_ = nullptr;
    rs_blob_cap_ = 0;
    I2IT_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&rs_blob_), bytes, cudaHostAllocDefault));
    rs_blob_cap_ = bytes;
  }
  std::memcpy(rs_blob_, c.d.data(), dbytes);
  std::memcpy(rs_blob_ + dbytes, c.tab.data(), c.tab.size() * sizeof(int));
  return bytes;
}

void Engine::run(Plan* P, const IO& io, cudaStream_t st, const std::function<void(cudaStream_t)>& before) {
  P->io = io;
  last_plan_ = P;
  P->last_run = ++tick_;
  evict_lru(nullptr, /*keep_last=*/false);   // this forward rewrites the workspace: no byte of it needs to survive
  if (cfg.use_cuda_graph) {
    // replay on the engine's own stream, ordered after/before the caller's stream with events
    I2IT_CUDA(cudaEventRecord(ev_in_, st));
    I2IT_CUDA(cudaStreamWaitEvent(gstream_, ev_in_, 0));
    if (before) before(gstream_);
    cudaGraphExec_t ge = nullptr;
    for (auto& g : P->graphs) if (g.first == io) ge = g.second;
    if (!ge) {
      // pointers are baked into the captured launches: one graph per distinct IO set (the torch allocator recycles blocks,
      // so a steady-state loop hits this cache)
      if (P->graphs.size() >= 8) { cudaGraphExecDestroy(P->graphs.front().second); P->graphs.erase(P->graphs.begin()); }
      cudaGraph_t g = nullptr;
      I2IT_CUDA(cudaStreamBeginCapture(gstream_, cudaStreamCaptureModeThreadLocal));
      g_pdl.enabled = use_pdl; g_pdl.prev_is_kernel = false;
      for (auto& op : P->ops) op(gstream_);
      I2IT_CUDA(cudaStreamEndCapture(gstream_, &g));
      I2IT_CUDA(cudaGraphInstantiate(&ge, g, 0));
      cudaGraphDestroy(g);
      P->graphs.emplace_back(io, ge);
      ++graph_captures;
    }
    nvtxRangePushA("i2it:forward(graph)");
    I2IT_CUDA(cudaGraphLaunch(ge, gstream_));
    nvtxRangePop();
    I2IT_CUDA(cudaEventRecord(ev_out_, gstream_));
    I2IT_CUDA(cudaStreamWaitEvent(st, ev_out_, 0));
  } else {
    if (before) before(st);
    g_pdl.enabled = use_pdl; g_pdl.prev_is_kernel = false;
    size_t next_range = 0;
    bool open = false;
    for (size_t i = 0; i < P->ops.size(); ++i) {
      if (next_range < P->ranges.size() && P->ranges[next_range].first == i) {   // NVTX: vae_encode / unet / ddpm_step / vae_decode
        if (open) nvtxRangePop();
        nvtxRangePushA((std::string("i2it:") + P->ranges[next_range].second).c_str());
        open = true;
        ++next_range;
      }
      P->ops[i](st);
      if (sync_each) {   // I2IT_SYNC_EACH=1 (debugging): attribute an asynchronous fault to the launch that caused it
        const cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess)
          throw Error("launch " + std::to_string(i) + " (" + P->meta[i].kind + " " + P->meta[i].shape + "): " + cudaGetErrorString(e));
      }
    }
    if (open) nvtxRangePop();
    I2IT_CUDA(cudaGetLastError());
  }
  if (trace_on) dump_trace(*P, st);
}

// I2IT_TRACE=1: per GEMM launch, the median over CTAs of each phase stamp relative to the CTA's entry stamp (SM cycles).
// slots: 1 prologue done | 2 first tile's loads issued | 3 all loads issued | 4 first operands landed | 5 first tile's MMAs
// complete | 7 first bias slice staged | 8 first accumulator ready | 9 first tile stored | 10 all tiles
// stored | 11 CTA joined
void Engine::dump_trace(Plan& P, cudaStream_t st) {
  I2IT_CUDA(cudaStreamSynchronize(st));
  I2IT_CUDA(cudaStreamSynchronize(gstream_));
  int idx = 0;
  for (auto& t : P.traces) {
    std::vector<unsigned long long> h(static_cast<size_t>(t.grid) * 16);
    I2IT_CUDA(cudaMemcpy(h.data(), t.buf, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    std::string line = "TRACE " + std::to_string(idx++) + " " + t.what + " |";
    for (int sl = 1; sl <= 12; ++sl) {
      std::vector<long long> d;
      for (int c = 0; c < t.grid; ++c)
        if (h[c * 16 + sl] && h[c * 16]) d.push_back(static_cast<long long>(h[c * 16 + sl] - h[c * 16]));
      if (d.empty()) { line += " -"; continue; }
      std::sort(d.begin(), d.end());
      line += " " + std::to_string(d[d.size() / 2]);
      if (sl == 12) line += " max " + std::to_string(d.back());
    }
    fprintf(stderr, "%s\n", line.c_str());
  }
}

// Per-launch device timing of the last forward's plan (CUDA events around every op, `reps` passes, averaged).
std::string Engine::profile_json(int reps, cudaStream_t st) {
  I2IT_CHECK(last_plan_ != nullptr, "profile: run a forward first");
  Plan& P = *last_plan_;
  const size_t n = P.ops.size();
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) I2IT_CUDA(cudaEventCreate(&e));
  std::vector<double> ms(n, 0.0);
  for (int r = 0; r < reps; ++r) {
    I2IT_CUDA(cudaEventRecord(ev[0], st));
    g_pdl.enabled = false;   // per-launch timing: full serialisation between kernels
    for (size_t i = 0; i < n; ++i) { P.ops[i](st); I2IT_CUDA(cudaEventRecord(ev[i + 1], st)); }
    I2IT_CUDA(cudaStreamSynchronize(st));
    for (size_t i = 0; i < n; ++i) { float t = 0; I2IT_CUDA(cudaEventElapsedTime(&t, ev[i], ev[i + 1])); ms[i] += t / reps; }
  }
  for (auto& e : ev) cudaEventDestroy(e);
  std::string js = "[";
  char buf[512];
  for (size_t i = 0; i < n; ++i) {
    const OpMeta& m = P.meta[i];
    snprintf(buf, sizeof buf, "%s{\"i\":%zu,\"kind\":\"%s\",\"ms\":%.6f,\"flops\":%.6g,\"bytes\":%.6g,\"shape\":\"%s\"}", i ? "," : "", i,
             m.kind.c_str(), ms[i], m.flops, m.bytes, m.shape.c_str());
    js += buf;
  }
  return js + "]";
}

__global__ void stage_to_nchw_f32_kernel(const uint16_t* x, int ld, int C, long long HW, long long total, float* out,
                                         int is_bf16) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;   // over N*C*HW (NCHW order)
  if (i >= total) return;
  const long long p = i % HW;
  const long long r = i / HW;
  const int c = static_cast<int>(r % C);
  const long long n = r / C;
  const uint16_t v = x[(n * HW + p) * ld + c];
  out[i] = is_bf16 ? __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(&v))
                   : __half2float(*reinterpret_cast<const __half*>(&v));
}

void Engine::read_stage(const std::string& name_in, float* dst, size_t dst_elems, int dims[4]) {
  // "text_encoder.*" names are stages of the last encode_text, every other name one of the last forward
  const bool text = name_in.rfind("text_encoder.", 0) == 0;
  const Plan* plan = text ? last_text_plan_ : last_plan_;
  I2IT_CHECK(plan != nullptr, text ? "no encode_text has run yet" : "no forward has run yet");
  // "name@i" selects image i of the stage (large-batch stages do not fit a test's scratch buffer)
  std::string name = name_in;
  int pick = -1;
  const size_t at = name.find('@');
  if (at != std::string::npos) { pick = atoi(name.c_str() + at + 1); name = name.substr(0, at); }
  auto it = plan->stages.find(name);
  I2IT_CHECK(it != plan->stages.end(), "unknown stage '" + name + "' (was keep_stages set?)");
  const Act& a = it->second;
  I2IT_CHECK(pick < a.N, "read_stage: image index out of range");
  const int n = pick >= 0 ? 1 : a.N;
  dims[0] = n; dims[1] = a.C; dims[2] = a.H; dims[3] = a.W;
  const long long HW = static_cast<long long>(a.H) * a.W, total = HW * a.C * n;
  I2IT_CHECK(static_cast<size_t>(total) <= dst_elems, "read_stage: destination too small");
  I2IT_CUDA(cudaDeviceSynchronize());
  const uint16_t* src = a.p + (pick >= 0 ? static_cast<long long>(pick) * a.img() : 0);
  stage_to_nchw_f32_kernel<<<ceil_div(total, 256), 256>>>(src, a.ld, a.C, HW, total, dst, dtype == DT_BF16);
  I2IT_CUDA(cudaDeviceSynchronize());
}

std::string Engine::stage_names_json(bool text) const {
  const Plan* plan = text ? last_text_plan_ : last_plan_;
  I2IT_CHECK(plan != nullptr, text ? "no encode_text has run yet" : "no forward has run yet");
  std::string js = "[";
  for (size_t i = 0; i < plan->stage_order.size(); ++i) {
    const std::string& n = plan->stage_order[i];
    const Act& a = plan->stages.at(n);
    js += std::string(i ? "," : "") + "{\"name\":\"" + n + "\",\"dims\":[" + std::to_string(a.N) + "," + std::to_string(a.C) + "," +
          std::to_string(a.H) + "," + std::to_string(a.W) + "]}";
  }
  return js + "]";
}

std::string Engine::prepared_keys_json() const {
  std::vector<std::string> keys;
  for (const auto& kv : prepared_) keys.push_back(kv.first);
  std::sort(keys.begin(), keys.end());
  std::string js = "[";
  for (size_t i = 0; i < keys.size(); ++i) js += std::string(i ? "," : "") + "\"" + keys[i] + "\"";
  return js + "]";
}

void Engine::read_prepared(const std::string& key, void* w, size_t w_elems, float* bias, size_t b_elems, int dims[4]) {
  auto it = prepared_.find(key);
  I2IT_CHECK(it != prepared_.end(), "unknown prepared weight '" + key + "'");
  const PW& pw = it->second;
  dims[0] = pw.taps; dims[1] = pw.rows; dims[2] = pw.cin_pad; dims[3] = pw.bias ? 1 : 0;
  const size_t n = static_cast<size_t>(pw.taps) * pw.rows * pw.cin_pad;
  I2IT_CUDA(cudaDeviceSynchronize());                     // preparation runs on the default stream
  if (w) {
    I2IT_CHECK(n <= w_elems, "read_prepared: weight destination too small");
    I2IT_CUDA(cudaMemcpy(w, pw.w, n * 2, cudaMemcpyDefault));
  }
  if (bias && pw.bias) {
    I2IT_CHECK(static_cast<size_t>(pw.rows) <= b_elems, "read_prepared: bias destination too small");
    I2IT_CUDA(cudaMemcpy(bias, pw.bias, pw.rows * sizeof(float), cudaMemcpyDefault));
  }
}

}  // namespace i2it

// tapgemm: the one tensor-core kernel of the path.
//
//   D[m, n] = act( alpha * sum_{tap t} sum_k A_t[m, k] * B_t[n, k]  + bias ) + residual
//
// A_t is a TMA *box* of the activation tensor shifted by the tap's spatial offset, so a 3x3 /
// stride-2 / 1x1 convolution, a linear layer and the attention GEMMs (Q K^T, P V, V^T = W X^T)
// are all the same implicit GEMM.  Zero padding, ragged edges and channel padding come from TMA
// out-of-bounds zero fill, never from materialised copies.
//
// sm_90a structure (one persistent CTA per SM, 384 threads):
//   warp 8        : TMA producer   cp.async.bulk.tensor.5d -> 128B-swizzled smem ring (4 stages at BN = 256)
//   warps 0..7    : two consumer warpgroups; warpgroup g owns tile rows [64g, 64g+64):
//                   mainloop  one wgmma.mma_async m64nBNk16 per k16 step (BN is a template parameter, so the chain has
//                             no run-time predicates), fp32 accumulators in registers, defined anew by each tile's first MMA
//                   epilogue  TMA-store launches: from the wgmma fragments -> bias/residual/GEGLU/clamp -> swizzled store boxes
//                             -> TMA stores (the ring is not touched, so the producer loads the next tile meanwhile);
//                             direct-store launches: fp32 staging tile in smem (aliases the operand ring) -> one accumulator ROW
//                             per thread -> per-thread stores
//   mbarriers     : full/empty per smem stage; epi_done holds the producer off the ring while it is a staging tile
//
// Replaces every nn.Conv2d / nn.Linear / SDPA matmul under vae.encode / unet(...) / vae.decode of the reference
// pipeline, which dispatch to cuDNN implicit GEMM, cuBLAS and flash/mem-efficient SDPA in the reference stack.
#pragma once
#include <type_traits>
#include "common.cuh"

namespace i2it {

constexpr int TG_BM = 128;             // rows per tile (two m64 warpgroup slabs)
constexpr int TG_BK = 64;              // K elements per stage (= 128 B = one swizzle atom)
constexpr int TG_STAGES = 4;            // stages when the B tile is the full 32 KiB; smaller tiles get more (<= TG_MAX_STAGES)
constexpr int TG_MAX_STAGES = 16;       // small B tiles (BN <= 128) need more stages for the same lookahead in TIME
constexpr int TG_MAX_TAPS = 16;
constexpr int TG_A_STAGE = TG_BM * TG_BK * 2;    // 16 KiB
constexpr int TG_B_STAGE = 256 * TG_BK * 2;      // 32 KiB (BN <= 256)
constexpr int TG_EPI_WARPS = 8;                  // the two consumer warpgroups
constexpr int TG_EPI_GROUPS = TG_EPI_WARPS / 4;  // warps per 32-row quarter: they take the 32-column rounds in turn
constexpr int TG_EPI_RPW = 8 / TG_EPI_GROUPS;    // rounds per warp at BN = 256
constexpr int TG_BAR_BYTES = 512;
constexpr int TG_BIAS_BYTES = 2 * 256 * 4;       // per-tile bias slice, double-buffered across tiles
// Epilogue store boxes: each epilogue warp owns ONE TMA box = 32 rows x 64 output columns (128-byte rows, SWIZZLE_128B: the
// 16-byte chunk c of row r lives at r*128 + ((c ^ (r & 7)) << 4)).  The two warps that hold a 32-row quarter's fragments write
// their column pairs into it with conflict-free 32-bit st.shared and ONE lane hands the 4 KB box to the TMA unit, which writes
// full lines and clips ragged edges.  The residual takes the same road in reverse: coalesced 16-byte global loads (4 rows x
// 128 B per instruction) into the box, added in place.
constexpr int TG_OSTG_WARP = 32 * 128;
constexpr int TG_OSTG_BYTES = TG_EPI_WARPS * TG_OSTG_WARP;
// manual 1024-byte alignment slack of the dynamic smem base: 512 B are budgeted (a full 1 KB would put the CTA over the
// 227 KB limit) and the kernels trap with an error word if the runtime base needs more (it is 1 KB aligned in practice).
constexpr int TG_ALIGN_PAD = 512;
constexpr int TG_SMEM = TG_STAGES * (TG_A_STAGE + TG_B_STAGE) + TG_BAR_BYTES + TG_BIAS_BYTES + TG_OSTG_BYTES + TG_ALIGN_PAD;
// + one producer warpgroup (warp 8 issues the TMA loads, warps 9..11 idle).  Registers are allocated per warpgroup, so the
// producer warpgroup gives its registers to the consumers (setmaxnreg): 128 x 40 + 256 x 232 <= 64 K.  ptxas honours the
// two setmaxnreg with each inside its own role's branch (see the role split in tapgemm_body).  The kernel is still register-
// allocated within the launch's 168 per thread: ptxas needs the launch bound to honour setmaxnreg (without it: C7508).
constexpr int TG_THREADS = (TG_EPI_WARPS + 4) * 32;
constexpr int TG_REGS_PRODUCER = 40, TG_REGS_CONSUMER = 232;
// fp32 accumulator staging: 128 rows x (BN + 4) floats.  BN is a multiple of 16, so the row pitch is 4 mod 8 words and eight
// consecutive rows hit eight different 16-byte bank groups (conflict-free row reads).  It lives at the start of the operand ring
// and must stay clear of the second set of store boxes, which takes the ring's last 32 KB.
constexpr int TG_STG_BYTES = TG_BM * (256 + 4) * 4;
static_assert(TG_STG_BYTES <= TG_STAGES * (TG_A_STAGE + TG_B_STAGE) - TG_OSTG_BYTES, "accumulator staging must fit the ring");

enum TgAct : int { TG_ACT_NONE = 0, TG_ACT_CLAMP1 = 1, TG_ACT_GEGLU = 2, TG_ACT_GELU = 3, TG_ACT_QUICKGELU = 4 };   // 3, 4: CLIP MLP
enum TgBias : int { TG_BIAS_NONE = 0, TG_BIAS_COL = 1, TG_BIAS_ROW = 2 };

struct TapGemmParams {
  // ---- tile space: 4 "row" dims d1..d4 of the A tensor map (d0 is K) ----
  int tdim[4];     // tiles per dim
  int box[4];      // A box extent per dim, prod == 128; row r of a tile = j1 + box0*(j2 + box1*(j3 + box2*j4))
  int ext[4];      // logical extent per dim: row valid iff t*box + j < ext
  int a_mul[4];    // A coordinate(d) = t_d * a_mul[d] + tap_a[tap][d+1]
  int b_mul[3];    // B coordinate(2..4) = t_{2..4} * b_mul + tap_b[tap][1..3]
  int n_tiles, BN, N;
  int num_taps, kchunks;   // kchunks: default K chunks per tap (tap_kc overrides per tap)
  int tap_src[TG_MAX_TAPS]; // 0: (tmA, tmB)   1: (tmA2, tmB2) — a second activation tensor folded into the same accumulator
  int tap_kc[TG_MAX_TAPS];  // K chunks (of 64) for this tap
  int nprim;                // the first nprim taps share kchunks and are walked k-chunk-outer / tap-inner (same
                            // accumulation order in every kernel variant => bit-identical results); the rest follow
  int stages, b_stage;      // smem ring: number of stages and bytes per B stage (sized to the actual tile, <= TG_MAX_STAGES)
  int layout_pad0;          // unused; see layout_pad1
  int tap_a[TG_MAX_TAPS][5];
  int tap_b[TG_MAX_TAPS][4];
  uint32_t layout_pad1;     // unused.  Removing these two words moves every later field by 8 bytes, and with it ptxas's
                            // register allocation of the (spilling) tapgemm_kernel: -36 % images/s, measured A/B on one H100
  // ---- epilogue ----
  void* out;
  long long ostride[4];   // elements
  long long ocol;         // element stride between consecutive output columns (1 = contiguous)
  int out_fp32;
  const void* res;        // optional residual, element type == activation type
  long long rstride[4];
  long long rcol;
  const float* bias;
  int bias_mode;
  float alpha;
  int act;
  int* err;               // device error word (watchdog)
  int tma_out;            // 1: 64-column rounds are staged in smem and stored by TMA (I2IT_NO_TMAOUT=1 -> 0: per-thread stores)
  int ostg2;              // 1: every epilogue warp alternates between TWO store boxes (the second set lives in the last 32 KB of the
                          // operand ring, which the host then sizes 32 KB smaller): a round no longer waits for the TMA store of
                          // the previous round to drain its box (I2IT_NO_OSTG2=1 -> 0)
  // GroupNorm statistics of the OUTPUT tensor, taken from the staged (rounded) tile: per 32-row slot and per `gn_red` columns,
  // (sum, sum of squares) -> gn_part[(slot0 + m_tile*4 + quarter) * (N/gn_red) + col/gn_red][2]; nullptr = off
  float* gn_part;
  // split-K: the primary taps' k-chunks are divided over `ksplit` tiles that write fp32 partials
  // `split_ostride` elements apart (splitk_reduce_kernel sums them in a fixed order); secondary taps go with split 0
  int ksplit, kc_per;
  long long split_ostride;
  int gn_red, gn_slot0, gn_mtiles;   // gn_mtiles: m-tiles of the launch
  int gn_shift;                      // log2(gn_red)
  // tile decode without integer division: magic[i] = floor(2^32 / d_i) + 1 for d = (n_tiles, tdim[0..3]); exact while
  // tile * d < 2^32 (the host refuses larger tile spaces)
  uint32_t magic[5];
  unsigned long long* trace;   // optional (I2IT_TRACE=1): 16 %clock64 stamps per CTA at the phase boundaries, else nullptr
};

// Operands of a selecting launch (tapgemm_sel_kernel), kept out of TapGemmParams so that no field of the plain kernels moves
// (see layout_pad1).  Every 128-row tile belongs to one image; dir[image] picks that tile's weight set: 0 = the launch's own
// maps and bias, 1 = the alternative maps (tmX for B, tmX2 for the second source's B; tmX for A when sel_a) and `bias`.
struct TapGemmSel {
  const int* dir;          // [images], 0 or 1, device memory (rewritten before each forward; the graph reads it)
  const float* bias;       // the alternative column bias (row bias when sel_a), nullptr iff p.bias is
  int dim;                 // the tile coordinate that holds the image: image = t[dim] / div  (dim 0, 2 or 3)
  int div;                 // 1, or the m-tiles per image of a flattened-token launch
  uint32_t magic;          // make_magic(., div)
  int sel_a;               // 1: the weight is the row operand (V^T projection): the selection replaces A, not B
};

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// Bounded wait: a protocol bug must surface as a trapped launch with an error word, never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int* err, int code) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3ff) == 0 && globaltimer_ns() - t0 > 4000000000ull) {
      if (err) atomicExch(err, code);
      __threadfence_system();
      __trap();
    }
  }
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1,
                                            int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
// TMA store of one box from shared memory (async proxy): the writer threads fence (fence.proxy.async) and sync first
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* tm, uint32_t src, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(tm)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// one lane of a fully converged warp (warp-uniform control flow keeps descriptors/addresses in uniform registers)
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
// ---- Hopper warpgroup MMA (all four warps of a warpgroup execute these together) ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T for the tile's whole width N (BN) in one instruction, both operands K-major in
// 128B-swizzled smem.  ACC = false is the first k16 step of a tile: scale-d = 0 and output-only operands, so D is overwritten
// (an exact -0 sum stays -0) and the accumulators carry nothing from the previous tile.
// Fragment of D: register 4*g + e of thread (warp w, lane l) is row 16w + l/4 + 8*(e >> 1), column 8g + 2*(l % 4) + (e & 1).
#define TG_D4(C, i) C(d[i]), C(d[i + 1]), C(d[i + 2]), C(d[i + 3])
#define TG_D8(C, i) TG_D4(C, i), TG_D4(C, i + 4)
#define TG_D32(C, i) TG_D8(C, i), TG_D8(C, i + 8), TG_D8(C, i + 16), TG_D8(C, i + 24)
#define TG_WGMMA_N16(TY, C) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n16k16.f32." TY "." TY " {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}" \
    : TG_D8(C, 0) : "l"(a), "l"(b), "r"(scale_d))
#define TG_WGMMA_N32(TY, C) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n32k16.f32." TY "." TY " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}" \
    : TG_D8(C, 0), TG_D8(C, 8) : "l"(a), "l"(b), "r"(scale_d))
#define TG_WGMMA_N48(TY, C) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n48k16.f32." TY "." TY " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1, 0, 0;\n\t}" \
    : TG_D8(C, 0), TG_D8(C, 8), TG_D8(C, 16) : "l"(a), "l"(b), "r"(scale_d))
#define TG_WGMMA_N64(TY, C) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}" \
    : TG_D32(C, 0) : "l"(a), "l"(b), "r"(scale_d))
#define TG_WGMMA_N80(TY, C) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n80k16.f32." TY "." TY " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}, %40, %41, p, 1, 1, 0, 0;\n\t}" \
    : TG_D32(C, 0), TG_D8(C, 32) : "l"(a), "l"(b), "r"(scale_d))
#define TG_WGMMA_N96(TY, C) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n96k16.f32." TY "." TY " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, %48, %49, p, 1, 1, 0, 0;\n\t}" \
    : TG_D32(C, 0), TG_D8(C, 32), TG_D8(C, 40) : "l"(a), "l"(b), "r"(scale_d))
#define TG_WGMMA_N112(TY, C) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %58, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n112k16.f32." TY "." TY " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55}, %56, %57, p, 1, 1, 0, 0;\n\t}" \
    : TG_D32(C, 0), TG_D8(C, 32), TG_D8(C, 40), TG_D8(C, 48) : "l"(a), "l"(b), "r"(scale_d))
#define TG_WGMMA_N128(TY, C) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}" \
    : TG_D32(C, 0), TG_D32(C, 32) : "l"(a), "l"(b), "r"(scale_d))
#define TG_WGMMA_N160(TY, C) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %82, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n160k16.f32." TY "." TY " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79}, %80, %81, p, 1, 1, 0, 0;\n\t}" \
    : TG_D32(C, 0), TG_D32(C, 32), TG_D8(C, 64), TG_D8(C, 72) : "l"(a), "l"(b), "r"(scale_d))
#define TG_WGMMA_N192(TY, C) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n192k16.f32." TY "." TY " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95}, %96, %97, p, 1, 1, 0, 0;\n\t}" \
    : TG_D32(C, 0), TG_D32(C, 32), TG_D32(C, 64) : "l"(a), "l"(b), "r"(scale_d))
#define TG_WGMMA_N224(TY, C) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %114, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n224k16.f32." TY "." TY " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111}, %112, %113, p, 1, 1, 0, 0;\n\t}" \
    : TG_D32(C, 0), TG_D32(C, 32), TG_D32(C, 64), TG_D8(C, 96), TG_D8(C, 104) : "l"(a), "l"(b), "r"(scale_d))
#define TG_WGMMA_N256(TY, C) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n256k16.f32." TY "." TY " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, 0, 0;\n\t}" \
    : TG_D32(C, 0), TG_D32(C, 32), TG_D32(C, 64), TG_D32(C, 96) : "l"(a), "l"(b), "r"(scale_d))

#define TG_WGMMA_CASE(n, C)                                                                \
  else if constexpr (N == n) { if constexpr (F16) TG_WGMMA_N##n("f16", C); else TG_WGMMA_N##n("bf16", C); }
#define TG_WGMMA_SWITCH(C)                                                                                          \
  if constexpr (N == 0) {}                                                                                          \
  TG_WGMMA_CASE(16, C) TG_WGMMA_CASE(32, C) TG_WGMMA_CASE(48, C) TG_WGMMA_CASE(64, C) TG_WGMMA_CASE(80, C)          \
  TG_WGMMA_CASE(96, C) TG_WGMMA_CASE(112, C) TG_WGMMA_CASE(128, C) TG_WGMMA_CASE(160, C) TG_WGMMA_CASE(192, C)     \
  TG_WGMMA_CASE(224, C) TG_WGMMA_CASE(256, C)                                                                       \
  else static_assert(N == 0, "no wgmma wrapper for this N");
// scale_d == 0 overwrites D (the flash kernels' form, with a run-time flag)
template <int N, typename T> __device__ __forceinline__ void wgmma_ss(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
  constexpr bool F16 = std::is_same<T, __half>::value;
  TG_WGMMA_SWITCH("+f")
}
template <int N, bool ACC, typename T> __device__ __forceinline__ void wgmma_ss(float* d, uint64_t a, uint64_t b) {
  if constexpr (ACC) {
    wgmma_ss<N, T>(d, a, b, 1u);
  } else {
    constexpr bool F16 = std::is_same<T, __half>::value;
    const uint32_t scale_d = 0u;
    TG_WGMMA_SWITCH("=f")
  }
}
#undef TG_WGMMA_SWITCH
#undef TG_WGMMA_CASE
#undef TG_WGMMA_N16
#undef TG_WGMMA_N32
#undef TG_WGMMA_N48
#undef TG_WGMMA_N64
#undef TG_WGMMA_N80
#undef TG_WGMMA_N96
#undef TG_WGMMA_N112
#undef TG_WGMMA_N128
#undef TG_WGMMA_N160
#undef TG_WGMMA_N192
#undef TG_WGMMA_N224
#undef TG_WGMMA_N256
#undef TG_D32
#undef TG_D8
#undef TG_D4
// K-major, 128B-swizzled operand tile for wgmma: rows of 128 B, 8-row groups 1024 B apart (SBO), start address advanced by
// 32 B (+2 in the descriptor) per K = 16 step inside the swizzle atom.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
  uint64_t d = static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;           // leading byte offset (unused for swizzled K-major)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;   // stride byte offset between 8-row core-matrix groups
  d |= static_cast<uint64_t>(1) << 62;           // SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void sts16(uint32_t saddr, const uint4& u) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(saddr), "r"(u.x), "r"(u.y), "r"(u.z), "r"(u.w) : "memory");
}
__device__ __forceinline__ uint4 lds16(uint32_t saddr) {
  uint4 u;
  asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "r"(saddr) : "memory");
  return u;
}

// timeline stamp for the diagnostic trace (build with `make TRACE=1`, run with I2IT_TRACE=1; one thread per role writes;
// cycles are per-SM, compare within a CTA only)
__device__ __forceinline__ void tg_stamp(const TapGemmParams& p, int slot) {
#ifdef I2IT_TRACE_BUILD   // `make TRACE=1`: even a never-taken stamp in the issue loops costs ~2 % of a step, so it is compiled out by default
  if (p.trace) p.trace[blockIdx.x * 16 + slot] = static_cast<unsigned long long>(clock64());
#endif
}

struct TileCoord {
  int nt, t[4], split;
};
// x / d with the host's magic number (one IMAD.HI instead of ~20 instructions; the tile loops of all three roles decode a tile
// per iteration and the r02g profile charged 137 of the epilogue's 1460 instructions per tile to these divisions)
__device__ __forceinline__ int fast_div(int x, int d, uint32_t magic) {
  const int q = static_cast<int>(__umulhi(static_cast<uint32_t>(x), magic));      // branch-free: one IMAD.HI + one select
  return d == 1 ? x : q;
}
__device__ __forceinline__ TileCoord decode_tile(const TapGemmParams& p, int tile) {
  TileCoord c;
  int r = fast_div(tile, p.n_tiles, p.magic[0]), q;
  c.nt = tile - r * p.n_tiles;
  q = fast_div(r, p.tdim[0], p.magic[1]); c.t[0] = r - q * p.tdim[0]; r = q;
  q = fast_div(r, p.tdim[1], p.magic[2]); c.t[1] = r - q * p.tdim[1]; r = q;
  q = fast_div(r, p.tdim[2], p.magic[3]); c.t[2] = r - q * p.tdim[2]; r = q;
  q = fast_div(r, p.tdim[3], p.magic[4]); c.t[3] = r - q * p.tdim[3];
  c.split = q;                                   // 0 unless ksplit > 1 (slowest index)
  return c;
}
inline uint32_t make_magic(long long max_dividend, int d) {   // host; 0 = the tile space is too large for the 32-bit magic (caller raises)
  if (d <= 1) return 1u;                                        // unused (fast_div selects x for d == 1)
  if (max_dividend * d >= (1ll << 32)) return 0u;
  return static_cast<uint32_t>((1ull << 32) / static_cast<unsigned>(d)) + 1u;
}

// One 16-column chunk of one accumulator row: alpha, bias, (GEGLU), residual, clamp, single rounding, store.
template <typename T>
__device__ __forceinline__ void epilogue_chunk(const TapGemmParams& p, const uint32_t (&raw)[16], int col0, long long obase,
                                               long long rbase, float rbias, const float* sbias, bool rfast, const uint4& r0,
                                               const uint4& r1) {
  float v[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = __uint_as_float(raw[i]) * p.alpha;
  if (p.bias_mode == TG_BIAS_COL) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] += sbias[i];   // smem broadcast; columns >= N hold 0 (staged once per tile)
  } else if (p.bias_mode == TG_BIAS_ROW) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] += rbias;
  }
  const bool full = (col0 + 16 <= p.N);
  if (p.act == TG_ACT_GEGLU) {
    // interleaved columns (2j, 2j+1) = (h_j, gate_j) -> out column j = h * gelu(gate)
    float o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = v[2 * i] * gelu_erf_f(v[2 * i + 1]);
    T* optr = reinterpret_cast<T*>(p.out) + obase + (col0 >> 1);
    if (p.res) {
      const T* rptr = reinterpret_cast<const T*>(p.res) + rbase + (col0 >> 1);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] += Elem<T>::to_f(rptr[i]);
    }
    if (full && ((reinterpret_cast<uintptr_t>(optr) & 15) == 0)) {
      uint4 u;
      u.x = Elem<T>::pack(o[0], o[1]); u.y = Elem<T>::pack(o[2], o[3]);
      u.z = Elem<T>::pack(o[4], o[5]); u.w = Elem<T>::pack(o[6], o[7]);
      st16(optr, u);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) if (col0 + 2 * i + 1 < p.N) optr[i] = Elem<T>::from_f(o[i]);
    }
    return;
  }
  if (p.act == TG_ACT_GELU) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = gelu_erf_f(v[i]);
  } else if (p.act == TG_ACT_QUICKGELU) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = quick_gelu_f(v[i]);
  }
  if (p.res) {
    if (rfast) {
      const uint32_t ru[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float2 f = Elem<T>::unpack(ru[i]);
        v[2 * i] += f.x; v[2 * i + 1] += f.y;
      }
    } else {
      const T* rptr = reinterpret_cast<const T*>(p.res) + rbase + col0 * p.rcol;
#pragma unroll
      for (int i = 0; i < 16; ++i) if (col0 + i < p.N) v[i] += Elem<T>::to_f(rptr[i * p.rcol]);
    }
  }
  if (p.act == TG_ACT_CLAMP1) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = fminf(fmaxf(v[i], -1.0f), 1.0f);
  }
  if (p.out_fp32) {
    float* optr = reinterpret_cast<float*>(p.out) + obase + col0 * p.ocol;
    if (full && p.ocol == 1 && ((reinterpret_cast<uintptr_t>(optr) & 15) == 0)) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
        *reinterpret_cast<float4*>(optr + 4 * i) = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
    } else {
#pragma unroll
      for (int i = 0; i < 16; ++i) if (col0 + i < p.N) optr[i * p.ocol] = v[i];
    }
  } else {
    T* optr = reinterpret_cast<T*>(p.out) + obase + col0 * p.ocol;
    if (full && p.ocol == 1 && ((reinterpret_cast<uintptr_t>(optr) & 15) == 0)) {
      uint4 u0, u1;
      u0.x = Elem<T>::pack(v[0], v[1]);   u0.y = Elem<T>::pack(v[2], v[3]);
      u0.z = Elem<T>::pack(v[4], v[5]);   u0.w = Elem<T>::pack(v[6], v[7]);
      u1.x = Elem<T>::pack(v[8], v[9]);   u1.y = Elem<T>::pack(v[10], v[11]);
      u1.z = Elem<T>::pack(v[12], v[13]); u1.w = Elem<T>::pack(v[14], v[15]);
      st16(optr, u0);
      st16(optr + 8, u1);
    } else {
#pragma unroll
      for (int i = 0; i < 16; ++i) if (col0 + i < p.N) optr[i * p.ocol] = Elem<T>::from_f(v[i]);
    }
  }
}

// Row coordinates of tile row (j1..j4) in tile c: g1..g4, whether the row lies inside the tensor, and its residual offset.
struct RowCoord {
  int g1, g2, g3, g4, ok;
  long long rbase;
};
__device__ __forceinline__ RowCoord row_coord(const TapGemmParams& p, const TileCoord& c, int j1, int j2, int j3, int j4) {
  RowCoord r;
  r.g1 = c.t[0] * p.box[0] + j1; r.g2 = c.t[1] * p.box[1] + j2; r.g3 = c.t[2] * p.box[2] + j3; r.g4 = c.t[3] * p.box[3] + j4;
  r.ok = (r.g1 < p.ext[0]) && (r.g2 < p.ext[1]) && (r.g3 < p.ext[2]) && (r.g4 < p.ext[3]);
  r.rbase = p.res ? r.g1 * p.rstride[0] + r.g2 * p.rstride[1] + r.g3 * p.rstride[2] + r.g4 * p.rstride[3] : 0;
  return r;
}

// Stage this tile's column-bias slice in smem (zeros where there is none, so the epilogue adds unconditionally); all 256
// epilogue threads take part.  The slice is double-buffered across tiles (acc = iter & 1).  The bias is p.bias, or with SEL
// `sel_bias`, the bias of the tile's image's weight set (tapgemm_sel_kernel).
template <bool SEL>
__device__ __forceinline__ void stage_bias(const TapGemmParams& p, const float* sel_bias, float* sb, int n0, int warp) {
  for (int cc = warp * 32 + (threadIdx.x & 31); cc < p.BN; cc += TG_EPI_WARPS * 32)
    sb[cc] = (p.bias_mode == TG_BIAS_COL && n0 + cc < p.N) ? (SEL ? sel_bias : p.bias)[n0 + cc] : 0.f;
  asm volatile("bar.sync 1, %0;" ::"n"(TG_EPI_WARPS * 32) : "memory");   // the epilogue warps only
}

// TMA-store epilogue, straight from the wgmma fragments (every tma_out launch: no staging tile, so the operand ring stays with
// the producer, which loads the next tile while this runs).  Rounds of 64 OUTPUT columns (128 accumulator columns for GEGLU)
// go through swizzled 32 x 64 store boxes (see TG_OSTG_WARP).  The tile's 32-row quarter q = warp >> 1 comes from the two
// warps 2q, 2q+1 of one warpgroup (fragment rows 16 (warp & 1) + [0, 16) each); they share the boxes of warps 2q and 2q+1
// (and the second set with ostg2) and meet at named barrier 2 + q (64 threads).  Box slot s = rsel & (ostg2 ? 3 : 1) of a
// round belongs to warp 2q + (s & 1): its lane 0 issues the TMA store and it takes the GroupNorm statistics from the box.
// Lane L of both warps describes tile row 32q + L (rc).  The arithmetic per element is that of every other epilogue:
// fmaf(acc, alpha, bias), activation, residual, clamp, one rounding.
template <typename T, bool LEAN, int BN>
__device__ __forceinline__ void epilogue_frag(const TapGemmParams& p, const CUtensorMap* tmO, const TileCoord& c, int m_tile,
                                              const float (&accum)[BN / 2], int warp, const RowCoord& rc, const float* sb,
                                              uint32_t ostg, uint32_t ostg2, int& rsel, bool stamp) {
  const int lane = threadIdx.x & 31, q = warp >> 1, half = warp & 1;
  const int n0 = c.nt * BN;
  const bool geglu = !LEAN && p.act == TG_ACT_GEGLU;
  const bool res_on = p.res != nullptr && !geglu;
  const int lrow = lane >> 3, lch = lane & 7;
  const int fr0 = 16 * half + (lane >> 2);                    // this thread's fragment rows in the quarter: fr0, fr0 + 8
  const int sw = lane >> 2;                                   // == fr0 & 7 == (fr0 + 8) & 7
  const int ok0 = __shfl_sync(0xffffffffu, rc.ok, fr0), ok1 = __shfl_sync(0xffffffffu, rc.ok, fr0 + 8);
  const int cq = 2 * (lane & 3);                              // column pair inside an 8-column fragment group
  // Residual: this warp's 16 rows of the box, 4 rows x 128 B per instruction; one round ahead of the math.
  uint4 rq[4];
  auto load_res = [&](int r) {
    const int colg = n0 + 64 * r;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int src_row = 16 * half + 4 * i + lrow;
      const long long rb = __shfl_sync(0xffffffffu, rc.rbase, src_row);
      const int ok = __shfl_sync(0xffffffffu, rc.ok, src_row);
      rq[i] = make_uint4(0u, 0u, 0u, 0u);
      if (ok && colg < p.N) rq[i] = ld_nc16(reinterpret_cast<const T*>(p.res) + rb + colg + lch * 8);
    }
  };
  if (res_on) load_res(0);
  if (stamp) tg_stamp(p, 8);

  // one round: take a free box, (residual in), the caller's fragment writes, TMA store + statistics by the box's owner
  auto round = [&](int r, int c0, auto&& write_box) {
    const int s = rsel & (p.ostg2 ? 3 : 1);
    ++rsel;
    const bool owner = (s & 1) == half;                       // warp-uniform
    const uint32_t box = (s >= 2 ? ostg2 : ostg) + (2 * q + (s & 1)) * TG_OSTG_WARP;
    // the owner's previous TMA store out of this box must have finished READING it (two box sets: the store before that)
    if (owner && lane == 0) { if (p.ostg2) bulk_wait_read1(); else bulk_wait_read0(); }
    asm volatile("bar.sync %0, 64;" ::"r"(2 + q) : "memory");
    if (res_on) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int rr = 16 * half + 4 * i + lrow;
        sts16(box + rr * 128 + ((lch ^ (rr & 7)) << 4), rq[i]);
      }
      __syncwarp();                                           // a thread reads back only rows of its own warp
      if (r + 1 < BN / 64) load_res(r + 1);
    }
    write_box(box);
    fence_async_smem();                                       // generic-proxy writes -> visible to the TMA unit
    asm volatile("bar.sync %0, 64;" ::"r"(2 + q) : "memory");
    if (!owner) return;
    const int ocol0 = geglu ? ((n0 + c0) >> 1) : (n0 + c0);
    if (lane == 0) {                                          // lane 0 describes row 32q, the box origin
      tma_store_5d(tmO, box, ocol0, rc.g1, rc.g2, rc.g3, rc.g4);
      bulk_commit();
    }
    if (p.gn_part) {
      // GroupNorm statistics of the tensor just produced, from the ROUNDED values in the box (what the next layer's GroupNorm
      // sees; rows outside the tensor were written as zeros).  Lane (rg, ch) = (lane >> 3, lane & 7) reads the 16-byte chunk
      // ch (8 output columns) of rows rg, rg+4, ..., rg+28: eight independent conflict-free ld.shared.v4 (a quarter warp
      // covers one 128-byte row), per-column-pair sums in registers, then the four row groups are combined by two shuffle
      // steps and lanes 0..7 write one (sum, sum of squares) entry per gn_red columns.  Fixed order, no atomics.
      const int rg = lane >> 3, ch = lane & 7;
      uint4 w[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int rr = 4 * i + rg;
        w[i] = lds16(box + rr * 128 + ((ch ^ (rr & 7)) << 4));
      }
      float s2[4] = {0.f, 0.f, 0.f, 0.f}, q2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t ww[4] = {w[i].x, w[i].y, w[i].z, w[i].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = Elem<T>::unpack(ww[j]);
          s2[j] += f.x + f.y;
          q2[j] = fmaf(f.x, f.x, fmaf(f.y, f.y, q2[j]));
        }
      }
      const int red = p.gn_red;                              // 2, 4, 8 or 16 columns per entry (warp-uniform)
      if (red >= 4) { s2[0] += s2[1]; q2[0] += q2[1]; s2[2] += s2[3]; q2[2] += q2[3]; }
      if (red >= 8) { s2[0] += s2[2]; q2[0] += q2[2]; }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if ((red >= 4 && (j & 1)) || (red >= 8 && j)) continue;   // folded above
        s2[j] += __shfl_xor_sync(0xffffffffu, s2[j], 8);  q2[j] += __shfl_xor_sync(0xffffffffu, q2[j], 8);
        s2[j] += __shfl_xor_sync(0xffffffffu, s2[j], 16); q2[j] += __shfl_xor_sync(0xffffffffu, q2[j], 16);
      }
      if (red == 16) { s2[0] += __shfl_xor_sync(0xffffffffu, s2[0], 1); q2[0] += __shfl_xor_sync(0xffffffffu, q2[0], 1); }
      if (rg == 0 && m_tile < p.gn_mtiles) {                 // slots without a valid row still get their zeros
        const int per_row = p.N >> p.gn_shift;
        const long long slot = p.gn_slot0 + static_cast<long long>(m_tile) * 4 + q;
        float2* dst = reinterpret_cast<float2*>(p.gn_part) + slot * per_row + ((ocol0 + 8 * ch) >> p.gn_shift);
        if (red == 2) {
          reinterpret_cast<float4*>(dst)[0] = make_float4(s2[0], q2[0], s2[1], q2[1]);
          reinterpret_cast<float4*>(dst)[1] = make_float4(s2[2], q2[2], s2[3], q2[3]);
        } else if (red == 4) {
          *reinterpret_cast<float4*>(dst) = make_float4(s2[0], q2[0], s2[2], q2[2]);
        } else if (red == 8 || (ch & 1) == 0) {
          *dst = make_float2(s2[0], q2[0]);
        }
      }
    }
  };

  if (geglu) {
    // interleaved accumulator columns (2j, 2j+1) = (h_j, gate_j) sit in one thread -> output column j = h * gelu(gate)
#pragma unroll
    for (int r = 0; r < BN / 128; ++r) {
      const int c0 = 128 * r;
      if (n0 + c0 >= p.N) break;                               // whole round beyond N (last n-tile): nothing to store
      round(r, c0, [&](uint32_t box) {
#pragma unroll
        for (int gg = 0; gg < 16; ++gg) {                     // accumulator columns c0 + 8 gg + cq, +1 -> output column 4 gg + cq / 2
          const int G = 16 * r + gg, col = c0 + 8 * gg + cq;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float hv = accum[4 * G + 2 * e] * p.alpha + sb[col];
            const float gv = accum[4 * G + 2 * e + 1] * p.alpha + sb[col + 1];
            const uint32_t u = Elem<T>::pack(hv * gelu_erf_f(gv), 0.f);
            const uint32_t a = box + (fr0 + 8 * e) * 128 + (((gg >> 1) ^ sw) << 4) + 8 * (gg & 1) + cq;
            asm volatile("st.shared.b16 [%0], %1;" ::"r"(a), "h"(static_cast<unsigned short>(u & 0xffffu)) : "memory");
          }
        }
      });
    }
    return;
  }
#pragma unroll
  for (int r = 0; r < BN / 64; ++r) {
    const int c0 = 64 * r;
    if (n0 + c0 >= p.N) break;                                 // whole round beyond N (last n-tile): nothing to store
    round(r, c0, [&](uint32_t box) {
#pragma unroll
      for (int gg = 0; gg < 8; ++gg) {                        // accumulator / output columns c0 + 8 gg + cq, +1
        const int G = 8 * r + gg, col = c0 + 8 * gg + cq;
        const float2 bq = *reinterpret_cast<const float2*>(sb + col);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float v0 = fmaf(accum[4 * G + 2 * e], p.alpha, bq.x), v1 = fmaf(accum[4 * G + 2 * e + 1], p.alpha, bq.y);
          if (!LEAN) {
            if (p.act == TG_ACT_GELU) { v0 = gelu_erf_f(v0); v1 = gelu_erf_f(v1); }
            else if (p.act == TG_ACT_QUICKGELU) { v0 = quick_gelu_f(v0); v1 = quick_gelu_f(v1); }
          }
          const uint32_t a = box + (fr0 + 8 * e) * 128 + ((gg ^ sw) << 4) + 2 * cq;
          if (res_on) {
            uint32_t ru;
            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(ru) : "r"(a) : "memory");
            const float2 f = Elem<T>::unpack(ru);
            v0 += f.x; v1 += f.y;
          }
          if (!LEAN && p.act == TG_ACT_CLAMP1) { v0 = fminf(fmaxf(v0, -1.0f), 1.0f); v1 = fminf(fmaxf(v1, -1.0f), 1.0f); }
          uint32_t u = Elem<T>::pack(v0, v1);
          if (p.gn_part && !(e ? ok1 : ok0)) u = 0u;          // clipped by the TMA store; keeps the statistics clean
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(u) : "memory");
        }
      }
    });
  }
}

// Direct-store epilogue of one output tile for one thread (= one accumulator row, read from the fp32 staging tile at `arow`):
// the launches whose output does not fit whole TMA-store rounds (fp32 logits, NCHW image, row-bias V^T, split-K partials,
// channel counts that are not multiples of 64).  The row's warp pair takes the 32-column rounds in turn (grp = warp & 1).
template <typename T, bool SEL = false>
__device__ __forceinline__ void epilogue_direct(const TapGemmParams& p, const TileCoord& c, const RowCoord& rc, int warp,
                                                uint32_t arow, const float* sb, bool stamp, const float* sel_bias = nullptr) {
  const int g1 = rc.g1, g2 = rc.g2, g3 = rc.g3, g4 = rc.g4;
  const bool row_ok = rc.ok;
  const long long rbase = rc.rbase;
  const int grp = warp & 1;
  const int n0 = c.nt * p.BN;
  const bool geglu = p.act == TG_ACT_GEGLU;
  auto acc_ld16 = [&](int col, uint32_t (&r)[16]) {          // accumulator columns [col, col+16) of this thread's row
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint4 u = lds16(arow + (col + 4 * i) * 4);
      r[4 * i] = u.x; r[4 * i + 1] = u.y; r[4 * i + 2] = u.z; r[4 * i + 3] = u.w;
    }
  };
  const long long obase = g1 * p.ostride[0] + g2 * p.ostride[1] + g3 * p.ostride[2] + g4 * p.ostride[3] + c.split * p.split_ostride;
  const float rbias = (p.bias_mode == TG_BIAS_ROW && row_ok) ? (SEL ? sel_bias : p.bias)[g1] : 0.0f;
  // This thread's WHOLE residual slice (its row x the 32-column rounds r = grp, grp+2, ...; <= 256 B) is requested up front,
  // so the global loads are in flight together.
  const int nrounds = (p.BN + 31) >> 5;
  const bool res_on = p.res != nullptr && row_ok && p.rcol == 1 && !geglu;
  uint4 rq[TG_EPI_RPW][4];
  bool fast[TG_EPI_RPW];
#pragma unroll
  for (int i = 0; i < TG_EPI_RPW; ++i) {
    const int r = grp + TG_EPI_GROUPS * i;
    fast[i] = false;
    if (res_on && r < nrounds) {
      const int colg = n0 + 32 * r;
      const int nch = min(2, (p.BN - 32 * r) >> 4);
      const T* rgrp = reinterpret_cast<const T*>(p.res) + rbase + colg;
      if (colg + 16 * nch <= p.N && (reinterpret_cast<uintptr_t>(rgrp) & 15) == 0) {
        rq[i][0] = ld_nc16(rgrp); rq[i][1] = ld_nc16(rgrp + 8);
        if (nch == 2) { rq[i][2] = ld_nc16(rgrp + 16); rq[i][3] = ld_nc16(rgrp + 24); }
        fast[i] = true;
      }
    }
  }

  if (stamp) tg_stamp(p, 8);

#pragma unroll
  for (int i = 0; i < TG_EPI_RPW; ++i) {
    const int r = grp + TG_EPI_GROUPS * i;
    if (r >= nrounds) break;                     // warp-uniform
    const int c0 = 32 * r;
    const int nch = min(2, (p.BN - c0) >> 4);
    uint32_t raw0[16], raw1[16];
    acc_ld16(c0, raw0);
    if (nch == 2) acc_ld16(c0 + 16, raw1);
    const int col0 = n0 + c0;
    if (row_ok) {
      if (col0 < p.N) epilogue_chunk<T>(p, raw0, col0, obase, rbase, rbias, sb + c0, fast[i], rq[i][0], rq[i][1]);
      if (nch == 2 && col0 + 16 < p.N)
        epilogue_chunk<T>(p, raw1, col0 + 16, obase, rbase, rbias, sb + c0 + 16, fast[i], rq[i][2], rq[i][3]);
    }
  }
}


// the weight set of tile c of a selecting launch: 0 (the launch's own) or 1 (the alternative)
__device__ __forceinline__ int sel_dir(const TapGemmSel& s, const TileCoord& c) {
  const int v = s.dim == 0 ? c.t[0] : (s.dim == 2 ? c.t[2] : c.t[3]);
  return s.dir[fast_div(v, s.div, s.magic)];
}

// The body of tapgemm_kernel and tapgemm_sel_kernel.  SEL (a weight set chosen per tile by the tile's image: mixed-direction
// CycleGAN batches, see TapGemmSel) changes three things, each under `if constexpr (SEL)`: the prefetch of the two
// alternative maps, the map the producer loads each tile's weight stages from, and the bias slice the epilogue stages for the
// tile.  The ring, the MMA chain, the accumulation order, the GroupNorm slots and the stores are the same.  One body, so an
// edit to the mainloop, the producer or the epilogue reaches both kernels.  ptxas's allocation of tapgemm_kernel is fragile
// (see layout_pad1), so the body was checked against the two separate kernels it replaced: `cuobjdump -sass` of every
// tapgemm_sel_kernel instantiation is identical, and every tapgemm_kernel instantiation differs only in the order of two
// `UMOV URx, URZ` of the prologue, with the same registers, stack and spills under -Xptxas -v.  Even small changes move
// that code: a bias pointer argument for the plain path in stage_bias rewrote the LEAN kernels, hence its SEL form.
// tmX / tmX2 / sel: the selecting launch's operands, nullptr when !SEL.
template <typename T, bool LEAN, int BN, bool SEL>
__device__ __forceinline__ void tapgemm_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmA2,
                                             const CUtensorMap& tmB2, const CUtensorMap& tmO, const TapGemmParams& p,
                                             const CUtensorMap* tmX, const CUtensorMap* tmX2, const TapGemmSel* sel) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  if (TG_ALIGN_PAD < 1024 && base - smem_u32(smem_raw) > static_cast<uint32_t>(TG_ALIGN_PAD)) {
    if (threadIdx.x == 0 && p.err) { atomicExch(p.err, 90); __threadfence_system(); }
    __trap();
  }
  const int NS = p.stages;
  const uint32_t BST = static_cast<uint32_t>(p.b_stage);
  const uint32_t sA = base;
  const uint32_t sB = base + NS * TG_A_STAGE;
  const uint32_t ostg = base + TG_STAGES * (TG_A_STAGE + TG_B_STAGE);   // epilogue store boxes (1024-byte aligned)
  const uint32_t ostg2 = ostg - TG_OSTG_BYTES;                          // optional second set: the ring's last 32 KB (p.ostg2)
  const uint32_t bars = ostg + TG_OSTG_BYTES;
  auto full_bar = [&](int s) { return bars + 8u * s; };
  auto empty_bar = [&](int s) { return bars + 8u * (TG_MAX_STAGES + s); };
  const uint32_t epi_done = bars + 8u * (2 * TG_MAX_STAGES);
  float* const s_bias = reinterpret_cast<float*>(smem_raw + (bars - smem_u32(smem_raw)) + TG_BAR_BYTES);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) tg_stamp(p, 0);
  const int nsplit = p.ksplit > 1 ? p.ksplit : 1;
  const int total_tiles = p.n_tiles * p.tdim[0] * p.tdim[1] * p.tdim[2] * p.tdim[3] * nsplit;
  int steps = 0, sec_steps = 0;
  for (int t = 0; t < p.num_taps; ++t) steps += p.tap_kc[t];
  for (int t = p.nprim; t < p.num_taps; ++t) sec_steps += p.tap_kc[t];

  if (warp == TG_EPI_WARPS && lane == 0) {
    for (int s = 0; s < NS; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), TG_EPI_WARPS); }
    mbar_init(epi_done, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA2)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB2)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmO)) : "memory");
    if constexpr (SEL) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmX)) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmX2)) : "memory");
    }
  }
  __syncthreads();
  pdl_sync();   // prologue (barriers, descriptor prefetch) overlaps the previous kernel's tail; no global access before here
  if (threadIdx.x == 0) tg_stamp(p, 1);

  // setmaxnreg inside each role's branch: issued by all warps before the role branches, both were ignored (C7507)
  if (warp >= TG_EPI_WARPS) {
    reg_dec<TG_REGS_PRODUCER>();
    if (warp == TG_EPI_WARPS) {             // warps 9..11 only hand their registers to the consumers
      // ================================ TMA producer (whole warp runs the loop, one elected lane issues) ==========
      int stage = 0, phase = 0, iter = 0;
      const uint32_t tx_bytes = TG_A_STAGE + static_cast<uint32_t>(p.BN) * (TG_BK * 2);
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++iter) {
        const TileCoord c = decode_tile(p, tile);
        const int a1 = c.t[0] * p.a_mul[0], a2 = c.t[1] * p.a_mul[1], a3 = c.t[2] * p.a_mul[2],
                  a4 = c.t[3] * p.a_mul[3];
        const int b2 = c.t[1] * p.b_mul[0], b3 = c.t[2] * p.b_mul[1], b4 = c.t[3] * p.b_mul[2];
        const int n0 = c.nt * p.BN;
        // direct-store launches: the ring doubles as the previous tile's accumulator staging tile until its epilogue has read it
        if (iter > 0 && !p.tma_out) mbar_wait(epi_done, (iter - 1) & 1, p.err, 2);
        bool alt = false;
        if constexpr (SEL) alt = sel_dir(*sel, c) != 0;
        auto load_step = [&](int t, int kc) {
          const CUtensorMap* ta = p.tap_src[t] ? &tmA2 : &tmA;
          const CUtensorMap* tb = p.tap_src[t] ? &tmB2 : &tmB;
          if constexpr (SEL) {
            if (alt && sel->sel_a) ta = tmX;
            else if (alt) tb = p.tap_src[t] ? tmX2 : tmX;
          }
          mbar_wait(empty_bar(stage), phase ^ 1, p.err, 1);
          if (elect_one()) {
            mbar_expect_tx(full_bar(stage), tx_bytes);
            tma_load_5d(sA + stage * TG_A_STAGE, ta, full_bar(stage), kc * TG_BK + p.tap_a[t][0],
                        a1 + p.tap_a[t][1], a2 + p.tap_a[t][2], a3 + p.tap_a[t][3], a4 + p.tap_a[t][4]);
            tma_load_5d(sB + stage * BST, tb, full_bar(stage), kc * TG_BK + p.tap_b[t][0], n0,
                        b2 + p.tap_b[t][1], b3 + p.tap_b[t][2], b4 + p.tap_b[t][3]);
          }
          __syncwarp();
          if (++stage == NS) { stage = 0; phase ^= 1; }
        };
        const int kc0 = nsplit > 1 ? c.split * p.kc_per : 0, kc1 = nsplit > 1 ? min(p.kchunks, kc0 + p.kc_per) : p.kchunks;
        for (int kc = kc0; kc < kc1; ++kc)
          for (int t = 0; t < p.nprim; ++t) load_step(t, kc);
        if (c.split == 0)
          for (int t = p.nprim; t < p.num_taps; ++t)
            for (int kc = 0; kc < p.tap_kc[t]; ++kc) load_step(t, kc);
        if (tile == static_cast<int>(blockIdx.x) && lane == 0) tg_stamp(p, 2);   // first tile's loads all issued
      }
      if (lane == 0) tg_stamp(p, 3);
    }
  } else {
    reg_inc<TG_REGS_CONSUMER>();
    // ============================ consumers: wgmma mainloop + epilogue (warps 0..7) ============================
    const int wg = warp >> 2;                    // warpgroup: tile rows [64 wg, 64 wg + 64) in the mainloop
    const int row = 32 * (warp >> 1) + lane;     // epilogue: tile row described by this lane (quarter warp >> 1)
    int rr = row;
    const int j1 = rr % p.box[0]; rr /= p.box[0];
    const int j2 = rr % p.box[1]; rr /= p.box[1];
    const int j3 = rr % p.box[2];
    const int j4 = rr / p.box[2];
    constexpr int spitch = BN + 4;               // staging row pitch in floats
    const uint32_t arow = base + static_cast<uint32_t>(row * spitch * 4);
    // one k-step (one ring stage): four k16 MMAs of the tile's full width; the first of a tile overwrites the accumulators
    auto mma_stage = [&](float (&accum)[BN / 2], int stage, auto first) {
      wgmma_fence();
      const uint32_t a0 = sA + stage * TG_A_STAGE + wg * (64 * 128), b0 = sB + stage * BST;
#pragma unroll
      for (int k = 0; k < TG_BK / 16; ++k) {
        const uint64_t adesc = wgmma_desc_sw128(a0) + 2 * k, bdesc = wgmma_desc_sw128(b0) + 2 * k;
        if (decltype(first)::value && k == 0) wgmma_ss<BN, false, T>(accum, adesc, bdesc);
        else wgmma_ss<BN, true, T>(accum, adesc, bdesc);
      }
      wgmma_commit();
    };
    int stage = 0, phase = 0, iter = 0, rsel = 0;   // rsel: store-box rounds so far (epilogue_frag)
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++iter) {
      int tsteps = steps;
      if (nsplit > 1) {                                                         // this tile's share of the K loop
        const int split = tile / (total_tiles / nsplit);
        const int kc0 = split * p.kc_per, kc1 = min(p.kchunks, kc0 + p.kc_per);
        tsteps = (kc1 - kc0) * p.nprim + (split == 0 ? sec_steps : 0);
      }
      float accum[BN / 2];                         // live from the tile's first MMA to the staging store only
      mbar_wait(full_bar(stage), phase, p.err, 3);
      if (iter == 0 && threadIdx.x == 0) tg_stamp(p, 4);                         // first operands landed
      mma_stage(accum, stage, std::true_type());
      int prev = stage;
      if (++stage == NS) { stage = 0; phase ^= 1; }
      for (int s = 1; s < tsteps; ++s) {
        mbar_wait(full_bar(stage), phase, p.err, 3);
        mma_stage(accum, stage, std::false_type());
        wgmma_wait<1>();                                   // the previous step's MMAs have read their stage
        if (lane == 0) mbar_arrive(empty_bar(prev));
        prev = stage;
        if (++stage == NS) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(empty_bar(prev));
      if (iter == 0 && threadIdx.x == 0) tg_stamp(p, 5);                        // first tile's MMAs complete

      const TileCoord c = decode_tile(p, tile);
      const RowCoord rc = row_coord(p, c, j1, j2, j3, j4);
      float* const sb = s_bias + (iter & 1) * 256;
      // a launch with a single n-tile stages its one slice into both buffers during the first two tiles and then skips this and
      // its barrier (110 tiles per CTA in the 512x512 convs)
      const float* sel_bias = nullptr;
      if constexpr (SEL) {
        sel_bias = sel_dir(*sel, c) ? sel->bias : p.bias;
        stage_bias<SEL>(p, sel_bias, sb, c.nt * BN, warp);   // every tile: the slice changes with the tile's image
      } else if (p.n_tiles > 1 || iter < 2) {
        stage_bias<SEL>(p, nullptr, sb, c.nt * BN, warp);
      }
      if (iter == 0 && threadIdx.x == 0) tg_stamp(p, 7);
      if (LEAN || p.tma_out) {
        epilogue_frag<T, LEAN, BN>(p, &tmO, c, fast_div(tile, p.n_tiles, p.magic[0]), accum, warp, rc, sb, ostg, ostg2, rsel,
                                   iter == 0 && threadIdx.x == 0);
      } else if constexpr (!LEAN) {
        // accumulators -> fp32 staging tile (the producer is parked on epi_done, so no load writes the ring meanwhile); the
        // barrier first: the other warpgroup's last MMAs may still be reading the ring stages the staging tile overlays
        asm volatile("bar.sync 1, %0;" ::"n"(TG_EPI_WARPS * 32) : "memory");
        {
          const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
          for (int g = 0; g < BN / 8; ++g) {
            const uint32_t a = base + static_cast<uint32_t>((r0 * spitch + 8 * g + c0) * 4);
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(accum[4 * g]), "f"(accum[4 * g + 1]) : "memory");
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a + 8 * spitch * 4), "f"(accum[4 * g + 2]),
                         "f"(accum[4 * g + 3]) : "memory");
          }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(TG_EPI_WARPS * 32) : "memory");
        epilogue_direct<T, SEL>(p, c, rc, warp, arow, sb, iter == 0 && threadIdx.x == 0, sel_bias);
        // staging tile consumed: the ring goes back to the producer (generic reads ordered before the TMA's async writes)
        fence_async_smem();
        asm volatile("bar.sync 1, %0;" ::"n"(TG_EPI_WARPS * 32) : "memory");
        if (threadIdx.x == 0) mbar_arrive(epi_done);
      }
      if (iter == 0 && threadIdx.x == 0) tg_stamp(p, 9);                        // first tile stored
    }
    if (p.tma_out && lane == 0) bulk_wait_all();      // the store boxes live in this CTA's shared memory
    if (threadIdx.x == 0) tg_stamp(p, 10);
  }
  __syncthreads();
  if (threadIdx.x == 0) tg_stamp(p, 11);
}

template <typename T, bool LEAN, int BN>
__global__ void __launch_bounds__(TG_THREADS, 1)
tapgemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
               const __grid_constant__ CUtensorMap tmO, const __grid_constant__ TapGemmParams p) {
  tapgemm_body<T, LEAN, BN, false>(tmA, tmB, tmA2, tmB2, tmO, p, nullptr, nullptr, nullptr);
}

// tapgemm with the weight set of each tile chosen by the tile's image (see TapGemmSel): the extra maps and TapGemmSel follow
// the plain kernel's parameters, so none of those moves
template <typename T, bool LEAN, int BN>
__global__ void __launch_bounds__(TG_THREADS, 1)
tapgemm_sel_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
                   const __grid_constant__ CUtensorMap tmO, const __grid_constant__ TapGemmParams p,
                   const __grid_constant__ CUtensorMap tmXm, const __grid_constant__ CUtensorMap tmX2m,
                   const __grid_constant__ TapGemmSel selm) {
  tapgemm_body<T, LEAN, BN, true>(tmA, tmB, tmA2, tmB2, tmO, p, &tmXm, &tmX2m, &selm);
}

}  // namespace i2it

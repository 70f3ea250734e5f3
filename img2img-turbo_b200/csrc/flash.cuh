// flash_attn_kernel: fused softmax(Q K^T * scale) V for head_dim 64 (all UNet self/cross attention and the CLIP text tower).
//
// Replaces, per attention layer, the three launches  S = QK^T (fp32 logits to HBM) -> softmax -> O = PV  — i.e. what the
// reference gets from F.scaled_dot_product_attention / xformers FMHA (diffusers AttnProcessor2_0).
//
// One CTA = one 128-row Q tile of one (batch, head); 288 threads:
//   warp 8        : TMA producer   Q once; (K_j [64 keys x 64], V^T_j [64 d x 64 keys]) through a 3-stage ring
//   warps 0..7    : two consumer warpgroups, warpgroup g owns Q rows [64g, 64g+64):
//                   S_j = Q K_j^T      4 x wgmma m64n64k16 (both operands in smem) -> fp32 registers
//                   online softmax in fp32 on the accumulator fragments (a row lives in 4 lanes of a quad)
//                   O += P_j V_j       4 x wgmma m64n64k16 with P_j as the REGISTER A operand: the accumulator fragment of
//                                      S converts to the A fragment of P in place (16-bit pack), P never touches smem
//                   the row sum l is taken over the ROUNDED probabilities, the same values the numerator uses
// 2 CTAs per SM (65 KB smem each) so one CTA's MMAs overlap the other's exponentials.
#pragma once
#include "tapgemm.cuh"

namespace i2it {

constexpr int FA_BM = 128, FA_BN = 64, FA_D = 64, FA_STAGES = 3;
constexpr int FA_Q_BYTES = FA_BM * FA_D * 2;            // 16 KiB
constexpr int FA_KV_STAGE = 2 * FA_BN * FA_D * 2;       // K 8 KiB + V^T 8 KiB
constexpr int FA_SMEM = FA_Q_BYTES + FA_STAGES * FA_KV_STAGE + 256 + 1024;
constexpr int FA_THREADS = 288;

struct FlashParams {
  int Nq, Nk, heads, B, q_tiles, kv_bmul;   // kv_bmul: 1 if K/V are per batch item, 0 if one K/V set is shared (text)
  float scale_log2e;                        // softmax scale * log2(e)
  void* out;                                // [B*Nq, ldo] tokens, head h at columns [64h, 64h+64)
  long long ldo;
  int causal;                               // 1: key j attends only to queries i >= j (CLIP text tower); KV tiles past the diagonal are skipped
  int* err;
};

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// D[64 x 64] += A[64 x 16] (registers, the m64k16 A fragment) * B[64 x 16]^T (K-major 128B-swizzled smem)
template <typename T> __device__ __forceinline__ void wgmma_rs64(float* d, const uint32_t (&a)[4], uint64_t b);
template <> __device__ __forceinline__ void wgmma_rs64<__half>(float* d, const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32, %33, %34, %35}, %36, 1, 1, 1, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_rs64<__nv_bfloat16>(float* d, const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32, %33, %34, %35}, %36, 1, 1, 1, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}

template <typename T>
__global__ void __launch_bounds__(FA_THREADS, 2)
flash_attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                  const __grid_constant__ CUtensorMap tmVt, const __grid_constant__ FlashParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base;
  const uint32_t sKV = base + FA_Q_BYTES;
  const uint32_t bars = sKV + FA_STAGES * FA_KV_STAGE;
  const uint32_t q_full = bars;
  auto kv_full = [&](int s) { return bars + 8u * (1 + s); };
  auto kv_empty = [&](int s) { return bars + 8u * (1 + FA_STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x % p.q_tiles;
  const int h = (blockIdx.x / p.q_tiles) % p.heads;
  const int b = blockIdx.x / (p.q_tiles * p.heads);
  int nkv = (p.Nk + FA_BN - 1) / FA_BN;
  if (p.causal) nkv = min(nkv, (qt * FA_BM + FA_BM + FA_BN - 1) / FA_BN);   // same value in both roles

  if (warp == 8 && lane == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < FA_STAGES; ++s) { mbar_init(kv_full(s), 1); mbar_init(kv_empty(s), 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmQ)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmK)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmVt)) : "memory");
  }
  __syncthreads();
  pdl_sync();   // prologue (barriers, descriptor prefetch) overlaps the previous kernel's tail; no global access before here

  if (warp == 8) {
    // producer: warp-uniform loop, one elected lane issues the TMA
    if (elect_one()) {
      mbar_expect_tx(q_full, FA_Q_BYTES);
      tma_load_5d(sQ, &tmQ, q_full, 0, qt * FA_BM, h, b, 0);
    }
    __syncwarp();
    for (int j = 0; j < nkv; ++j) {
      const int s = j % FA_STAGES;
      mbar_wait(kv_empty(s), ((j / FA_STAGES) & 1) ^ 1, p.err, 11);
      if (elect_one()) {
        mbar_expect_tx(kv_full(s), FA_KV_STAGE);
        tma_load_5d(sKV + s * FA_KV_STAGE, &tmK, kv_full(s), 0, j * FA_BN, h, b * p.kv_bmul, 0);
        tma_load_5d(sKV + s * FA_KV_STAGE + FA_BN * FA_D * 2, &tmVt, kv_full(s), j * FA_BN, 0, h, b * p.kv_bmul, 0);
      }
      __syncwarp();
    }
  } else {
    // ---------------- consumers: thread (warp w, lane l) holds rows r and r + 8, r = 16 (w % 4) + l / 4 of its warpgroup ----
    const int wg = warp >> 2;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int q0 = qt * FA_BM + r0, q1 = q0 + 8;
    const int klim0 = p.causal ? min(p.Nk, q0 + 1) : p.Nk;     // keys [0, klim) are visible to the row
    const int klim1 = p.causal ? min(p.Nk, q1 + 1) : p.Nk;
    const float sc = p.scale_log2e;
    const int ccol = 2 * (lane & 3);
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // running maxima (raw logit units) and row sums
    mbar_wait(q_full, 0, p.err, 12);
    const uint64_t qdesc = wgmma_desc_sw128(sQ + wg * (64 * 128));
    for (int j = 0; j < nkv; ++j) {
      const int s = j % FA_STAGES;
      mbar_wait(kv_full(s), (j / FA_STAGES) & 1, p.err, 13);
      const uint32_t sK = sKV + s * FA_KV_STAGE, sV = sK + FA_BN * FA_D * 2;
      float sacc[32];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < FA_D / 16; ++k) wgmma_ss<64, T>(sacc, qdesc + 2 * k, wgmma_desc_sw128(sK) + 2 * k, k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      const int kbase = j * FA_BN;
      // element-wise masking only where needed: the last KV tile, or causal tiles that reach this warp's diagonal
      const bool ragged = (kbase + FA_BN > p.Nk) || (p.causal && kbase + FA_BN - 1 > qt * FA_BM + wg * 64 + (warp & 3) * 16);
      if (ragged) {
#pragma unroll
        for (int g = 0; g < 8; ++g)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (kbase + 8 * g + ccol + (e & 1) >= (e < 2 ? klim0 : klim1)) sacc[4 * g + e] = -INFINITY;
      }
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        mx0 = fmaxf(mx0, fmaxf(sacc[4 * g], sacc[4 * g + 1]));
        mx1 = fmaxf(mx1, fmaxf(sacc[4 * g + 2], sacc[4 * g + 3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
      // a row with no visible key yet keeps m = -inf: factor 1 on its (zero) state, and every p below is exp2(-inf) = 0
      const float f0 = (mn0 == -INFINITY) ? 1.f : fast_exp2((m0 - mn0) * sc);
      const float f1 = (mn1 == -INFINITY) ? 1.f : fast_exp2((m1 - mn1) * sc);
      const float ng0 = (mn0 == -INFINITY) ? 0.f : -mn0 * sc, ng1 = (mn1 == -INFINITY) ? 0.f : -mn1 * sc;
      m0 = mn0; m1 = mn1;
      // p = exp2(s*scale - m*scale), packed to 16 bit: pk[2g] is row r (keys 8g + ccol, +1), pk[2g+1] row r + 8
      uint32_t pk[16];
      float ls0 = 0.f, ls1 = 0.f;
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        pk[2 * g] = Elem<T>::pack(fast_exp2(fmaf(sacc[4 * g], sc, ng0)), fast_exp2(fmaf(sacc[4 * g + 1], sc, ng0)));
        pk[2 * g + 1] = Elem<T>::pack(fast_exp2(fmaf(sacc[4 * g + 2], sc, ng1)), fast_exp2(fmaf(sacc[4 * g + 3], sc, ng1)));
        const float2 a = Elem<T>::unpack(pk[2 * g]), c = Elem<T>::unpack(pk[2 * g + 1]);
        ls0 += a.x + a.y;
        ls1 += c.x + c.y;
      }
      ls0 += __shfl_xor_sync(0xffffffffu, ls0, 1); ls0 += __shfl_xor_sync(0xffffffffu, ls0, 2);
      ls1 += __shfl_xor_sync(0xffffffffu, ls1, 1); ls1 += __shfl_xor_sync(0xffffffffu, ls1, 2);
      l0 = l0 * f0 + ls0;
      l1 = l1 * f1 + ls1;
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        o[4 * g] *= f0; o[4 * g + 1] *= f0;
        o[4 * g + 2] *= f1; o[4 * g + 3] *= f1;
      }
      // O += P V: keys [16kk, 16kk+16) of P are the A fragment {row r k, row r+8 k, row r k+8, row r+8 k+8}
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < FA_BN / 16; ++kk) {
        const uint32_t a[4] = {pk[4 * kk], pk[4 * kk + 1], pk[4 * kk + 2], pk[4 * kk + 3]};
        wgmma_rs64<T>(o, a, wgmma_desc_sw128(sV) + 2 * kk);
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(kv_empty(s));                 // K_j and V_j have been read by this warp's MMAs
    }
    const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
    T* const obase = reinterpret_cast<T*>(p.out) + static_cast<long long>(b) * p.Nq * p.ldo + h * FA_D + ccol;
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      if (q0 < p.Nq)
        *reinterpret_cast<uint32_t*>(obase + q0 * p.ldo + 8 * g) = Elem<T>::pack(o[4 * g] * inv0, o[4 * g + 1] * inv0);
      if (q1 < p.Nq)
        *reinterpret_cast<uint32_t*>(obase + q1 * p.ldo + 8 * g) = Elem<T>::pack(o[4 * g + 2] * inv1, o[4 * g + 3] * inv1);
    }
  }
}

// flash_attn512_kernel: fused softmax(Q K^T / sqrt(512)) V for ONE head of 512 (the VAE mid-block attention), used where
// the unfused path's fp32 logits (B * N * N * 6 bytes for S and P) would not fit: a 4K frame needs 100 GB of them.
//
// A 64-row x 512 fp32 O tile is 256 registers per thread, so each CTA owns one 64-row Q tile and one HALF (256 columns) of
// d_v; grid = 2 x q_tiles x B, the two halves of a Q tile adjacent in launch order so K / V^T come from L2 the second time.
// S is recomputed by both halves (1.5x the minimal MMA work) to keep the d = 64 kernel's structure: S and O in registers,
// P fed back as the register A operand.  One consumer warpgroup per CTA: O (128) + S (32) + P (16) registers per thread
// need more than the 168 a 9-warp CTA can have (three warps share an SM sub-partition's 16K registers; ptxas did not honour
// setmaxnreg for a second warpgroup), while 5 warps get up to 255.  160 threads, 1 CTA per SM:
//   warp 4      : TMA producer  Q once (8 boxes of 64 rows x 64 d, 64 KB, resident); per KV tile j twelve 64 x 64
//                 128B-swizzled boxes, K_j's 8 d-chunks then V^T_j's 4 column blocks of this half, through a 20-slot ring
//   warps 0..3  : S_j = Q K_j^T    8 chunks x 4 wgmma m64n64k16 (smem x smem); the K slots are released when S is complete
//                 online softmax exactly as flash_attn_kernel (fp32 logits, ex2.approx, row sum over the ROUNDED P)
//                 O[:, 64c..] += P_j V_j   4 column blocks x 4 wgmma m64n64k16, P as the register A operand
// Shared memory: Q 64 KB + ring 20 x 8 KB = 224 KB: the producer runs up to 1.6 KV tiles ahead.  Numerics per element do not
// depend on B or on the tile's position: image i of a batch is bit for bit its batch-1 result.
constexpr int FA5_BM = 64, FA5_BN = 64, FA5_D = 512, FA5_DV = 256;    // FA5_DV: the d_v half one CTA produces
constexpr int FA5_KCH = FA5_D / 64, FA5_VCH = FA5_DV / 64;            // 8 K boxes + 4 V^T boxes per KV tile
constexpr int FA5_SLOTS = 20;
constexpr int FA5_BOX = 64 * 64 * 2;                                   // 8 KiB; a Q box (64 rows x 64 d) is the same size
constexpr int FA5_Q_BYTES = FA5_KCH * FA5_BOX;                         // 64 KiB
constexpr int FA5_SMEM = FA5_Q_BYTES + FA5_SLOTS * FA5_BOX + 512 + 1024;
constexpr int FA5_THREADS = 160;

template <typename T>
__global__ void __launch_bounds__(FA5_THREADS, 1)
flash_attn512_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmVt, const __grid_constant__ FlashParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base;
  const uint32_t sR = base + FA5_Q_BYTES;
  const uint32_t bars = sR + FA5_SLOTS * FA5_BOX;
  const uint32_t q_full = bars;
  auto full = [&](int i) { return bars + 8u * (1 + i); };
  auto empty = [&](int i) { return bars + 8u * (1 + FA5_SLOTS + i); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int half = blockIdx.x & 1;
  const int qt = (blockIdx.x >> 1) % p.q_tiles;
  const int b = (blockIdx.x >> 1) / p.q_tiles;
  const int nkv = (p.Nk + FA5_BN - 1) / FA5_BN;

  if (warp == 4 && lane == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < FA5_SLOTS; ++i) { mbar_init(full(i), 1); mbar_init(empty(i), 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmQ)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmK)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmVt)) : "memory");
  }
  __syncthreads();
  pdl_sync();

  if (warp == 4) {
    if (elect_one()) {
      mbar_expect_tx(q_full, FA5_Q_BYTES);
      for (int c = 0; c < FA5_KCH; ++c) tma_load_5d(sQ + c * FA5_BOX, &tmQ, q_full, 64 * c, qt * FA5_BM, b, 0, 0);
    }
    __syncwarp();
    const int kb = b * p.kv_bmul;
    int slot = 0, ph = 0;
    for (int j = 0; j < nkv; ++j) {
      for (int i = 0; i < FA5_KCH + FA5_VCH; ++i) {
        mbar_wait(empty(slot), ph ^ 1, p.err, 21);
        if (elect_one()) {
          const uint32_t dst = sR + slot * FA5_BOX;
          mbar_expect_tx(full(slot), FA5_BOX);
          if (i < FA5_KCH) tma_load_5d(dst, &tmK, full(slot), 64 * i, j * FA5_BN, kb, 0, 0);
          else tma_load_5d(dst, &tmVt, full(slot), j * FA5_BN, half * FA5_DV + 64 * (i - FA5_KCH), kb, 0, 0);
        }
        __syncwarp();
        if (++slot == FA5_SLOTS) { slot = 0; ph ^= 1; }
      }
    }
  } else {
    // thread (warp w, lane l) holds rows r and r + 8, r = 16 w + l / 4
    const int q0 = qt * FA5_BM + warp * 16 + (lane >> 2), q1 = q0 + 8;
    const float sc = p.scale_log2e;
    const int ccol = 2 * (lane & 3);
    float o[FA5_VCH][32];
#pragma unroll
    for (int c = 0; c < FA5_VCH; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    mbar_wait(q_full, 0, p.err, 22);
    int slot = 0, ph = 0;       // ring position of the tile's first box
    for (int j = 0; j < nkv; ++j) {
      int sl[FA5_KCH + FA5_VCH], pp[FA5_KCH + FA5_VCH];
#pragma unroll
      for (int i = 0; i < FA5_KCH + FA5_VCH; ++i) {
        sl[i] = slot; pp[i] = ph;
        if (++slot == FA5_SLOTS) { slot = 0; ph ^= 1; }
      }
      float sacc[32];
      // every wait precedes the MMA chain: a (divergent) spin between two wgmmas makes ptxas serialise them
      for (int c = 0; c < FA5_KCH; ++c) mbar_wait(full(sl[c]), pp[c], p.err, 23);
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < FA5_KCH; ++c) {
        const uint64_t qd = wgmma_desc_sw128(sQ + c * FA5_BOX), kd = wgmma_desc_sw128(sR + sl[c] * FA5_BOX);
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss<64, T>(sacc, qd + 2 * k, kd + 2 * k, (c | k) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0)
        for (int c = 0; c < FA5_KCH; ++c) mbar_arrive(empty(sl[c]));
      const int kbase = j * FA5_BN;
      if (kbase + FA5_BN > p.Nk) {
#pragma unroll
        for (int g = 0; g < 8; ++g)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (kbase + 8 * g + ccol + (e & 1) >= p.Nk) sacc[4 * g + e] = -INFINITY;
      }
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        mx0 = fmaxf(mx0, fmaxf(sacc[4 * g], sacc[4 * g + 1]));
        mx1 = fmaxf(mx1, fmaxf(sacc[4 * g + 2], sacc[4 * g + 3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
      const float f0 = (mn0 == -INFINITY) ? 1.f : fast_exp2((m0 - mn0) * sc);
      const float f1 = (mn1 == -INFINITY) ? 1.f : fast_exp2((m1 - mn1) * sc);
      const float ng0 = (mn0 == -INFINITY) ? 0.f : -mn0 * sc, ng1 = (mn1 == -INFINITY) ? 0.f : -mn1 * sc;
      m0 = mn0; m1 = mn1;
      uint32_t pk[16];
      float ls0 = 0.f, ls1 = 0.f;
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        pk[2 * g] = Elem<T>::pack(fast_exp2(fmaf(sacc[4 * g], sc, ng0)), fast_exp2(fmaf(sacc[4 * g + 1], sc, ng0)));
        pk[2 * g + 1] = Elem<T>::pack(fast_exp2(fmaf(sacc[4 * g + 2], sc, ng1)), fast_exp2(fmaf(sacc[4 * g + 3], sc, ng1)));
        const float2 a = Elem<T>::unpack(pk[2 * g]), c = Elem<T>::unpack(pk[2 * g + 1]);
        ls0 += a.x + a.y;
        ls1 += c.x + c.y;
      }
      ls0 += __shfl_xor_sync(0xffffffffu, ls0, 1); ls0 += __shfl_xor_sync(0xffffffffu, ls0, 2);
      ls1 += __shfl_xor_sync(0xffffffffu, ls1, 1); ls1 += __shfl_xor_sync(0xffffffffu, ls1, 2);
      l0 = l0 * f0 + ls0;
      l1 = l1 * f1 + ls1;
#pragma unroll
      for (int c = 0; c < FA5_VCH; ++c)
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          o[c][4 * g] *= f0; o[c][4 * g + 1] *= f0;
          o[c][4 * g + 2] *= f1; o[c][4 * g + 3] *= f1;
        }
      for (int c = 0; c < FA5_VCH; ++c) mbar_wait(full(sl[FA5_KCH + c]), pp[FA5_KCH + c], p.err, 24);
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < FA5_VCH; ++c) {
        const uint64_t vd = wgmma_desc_sw128(sR + sl[FA5_KCH + c] * FA5_BOX);
#pragma unroll
        for (int kk = 0; kk < FA5_BN / 16; ++kk) {
          const uint32_t a[4] = {pk[4 * kk], pk[4 * kk + 1], pk[4 * kk + 2], pk[4 * kk + 3]};
          wgmma_rs64<T>(o[c], a, vd + 2 * kk);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0)
        for (int c = 0; c < FA5_VCH; ++c) mbar_arrive(empty(sl[FA5_KCH + c]));
    }
    const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
    T* const obase = reinterpret_cast<T*>(p.out) + static_cast<long long>(b) * p.Nq * p.ldo + half * FA5_DV + ccol;
#pragma unroll
    for (int c = 0; c < FA5_VCH; ++c)
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        if (q0 < p.Nq)
          *reinterpret_cast<uint32_t*>(obase + q0 * p.ldo + 64 * c + 8 * g) = Elem<T>::pack(o[c][4 * g] * inv0, o[c][4 * g + 1] * inv0);
        if (q1 < p.Nq)
          *reinterpret_cast<uint32_t*>(obase + q1 * p.ldo + 64 * c + 8 * g) =
              Elem<T>::pack(o[c][4 * g + 2] * inv1, o[c][4 * g + 3] * inv1);
      }
  }
}

}  // namespace i2it

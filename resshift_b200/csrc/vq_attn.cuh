// Fused single-head attention over all T positions of an image, O = softmax(Q K^T C^-1/2) V, for the VQ-GAN bottleneck
// at sizes where the T x T score matrix cannot be materialised (vq.inc takes this kernel for H*W > 8192).
//
// reference: AttnBlock.forward (ldm/modules/diffusionmodules/model.py:180-199; the MemoryEfficientAttnBlock path at
// :205-268 computes the same).  q, k, v, out: fp16 [N][T][C] (row stride ld); one launch, grid (T / 64, N).
//
// A launch may cover a range of query rows [row_begin, row_end) (multiples of 64) instead of all T: grid
// ((row_end - row_begin) / 64, N), CTA x takes query tile row_begin / 64 + x; K and V are always all T keys, and rows
// outside the range are neither read as queries nor written.  A row's result depends only on its query and the full K, V
// walked in the same order, so any partition of the rows over several launches (or GPUs) is bit-identical to one launch.
//
// A CTA owns 64 queries and walks the T keys in blocks of BK keys (vq_attn_bk: 32, or 16 at C = 512), in a fixed order,
// with an online softmax (running row max and row sum in fp32), so memory is O(T C) and the result is bit-reproducible and
// per image.  Warp 8 is the TMA producer: the Q tile once, then per key block the K block and the V block, each behind its
// own mbarrier, in a four-stage ring.  The two consumer warpgroups split the channels: warpgroup g owns channel half g.
// The producer is a whole (third) warpgroup so that setmaxnreg can hand its registers to the consumers.  ptxas still
// allocates the consumer code within the 168 registers of a 384-thread CTA, so at C = 512, where a consumer thread holds
// 128 fp32 output accumulators, the key block is 16 keys (8 score registers) instead of 32: with 32 it spills.
//
//     S_g [64 x BK]   = Q[:, half g] . K[:, half g]^T        (SS wgmma m64nBKk16, both K-major)
//     S               = S_0 + S_1                            (exchanged through shared memory behind a named barrier; fp32
//                                                             addition commutes, so both warpgroups hold bit-identical S
//                                                             and run the same softmax)
//     P               = exp2(S C^-1/2 log2e - m)             (fp16, kept in registers as the next wgmma's A operand)
//     O_g [64 x C/2] = O_g * exp2(m_old - m) + P . V[:, half g]   (RS wgmma m64n(C/2)k16, V MN-major: imm-trans-b = 1)
//
// (a warp skips the rescale of O when none of its 16 rows got a new maximum: multiplying by exactly 1 changes nothing)
//
// At the end O_g / l is rounded to fp16, staged in the dead Q tile (swizzled like a TMA load) and written by TMA stores.
//
// Shared memory at C = 512: Q 64 KB + 4 stages x (K 16 KB + V 16 KB) + 2 x 2 x 4 KB score exchange = 208 KB (+ barriers
// and the 1 KB alignment slack), under the 227 KB an H100 CTA may use; 192 KB at C = 256, 112 KB at C = 128.  The exchange is double-buffered, so one named
// barrier per key block suffices: a warpgroup can only overwrite its buffer of block j after the other passed the barrier
// of block j + 1, i.e. after it read block j.
#pragma once

#include "common.cuh"
#include "conv_gemm.cuh"

namespace rs {

constexpr int kVqAttnBM = 64;                    // queries per CTA
constexpr int kVqAttnStages = 4;
// keys per block (see the header)
__host__ __device__ constexpr int vq_attn_bk(int C) { return C == 512 ? 16 : 32; }
constexpr int kVqAttnThreads = 384;         // two consumer warpgroups + the producer warpgroup (warp 8 issues the loads)
constexpr int kVqAttnTmaWarp = 8;
constexpr int kVqAttnProducerRegs = 24;      // setmaxnreg budgets: 128 x 24 + 256 x 240 <= 64 K registers
constexpr int kVqAttnConsumerRegs = 240;

struct VqAttnParams {
  CUtensorMap tmQ, tmK, tmV, tmO;    // {C, T, 1, N}, boxes {64, 64 | BK, 1, 1}, 128-byte swizzle
  int T;
  int q_tile0;                       // first query tile (row_begin / 64) of the launch's row range
  float scale_log2;                  // C^-1/2 * log2(e)
};

template <int C>
struct VqAttnSmem {
  static constexpr int kBK = vq_attn_bk(C);
  static constexpr int kQTile = kVqAttnBM * 128;            // [64 queries x 64 channels] fp16
  static constexpr int kKvTile = kBK * 128;                 // [BK keys x 64 channels] fp16
  static constexpr int q = 0;
  static constexpr int k = q + (C / 64) * kQTile;           // [stage][C / 64 tiles]
  static constexpr int v = k + kVqAttnStages * (C / 64) * kKvTile;
  static constexpr int xch = v + kVqAttnStages * (C / 64) * kKvTile;   // [2 buffers][2 warpgroups][BK / 2 regs][128 threads] fp32
  static constexpr int bars = xch + 2 * 2 * (kBK / 2) * 128 * 4;
  static constexpr int total = bars + 64;
  static constexpr int launch_bytes = total + 1024;         // + alignment slack of the dynamic shared memory base
};

#ifdef __CUDACC__

// Shared-memory matrix descriptor of an MN-major operand with the 128-byte swizzle: 64-element rows (128 B) along MN, one
// row per K index, 8-row (K) groups 1024 B apart (SBO), consecutive 64-wide MN blocks `lbo` bytes apart (LBO).  Advancing
// 16 along K is +2048 B on the start address.
__device__ __forceinline__ uint64_t wgmma_desc_sw128_mn(uint32_t smem_addr, uint32_t lbo) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;            // SWIZZLE_128B
  return d;
}

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

template <int C>
__global__ void __launch_bounds__(kVqAttnThreads, 1) vq_attn_sm90_kernel(const __grid_constant__ VqAttnParams p) {
  static_assert(C == 128 || C == 256 || C == 512, "vq_attn: C in {128, 256, 512}");
  using L = VqAttnSmem<C>;
  constexpr int kBK = L::kBK;
  constexpr int kHalf = C / 2;                     // channels per warpgroup
  constexpr int kTilesHalf = kHalf / 64;           // 64-channel tiles per warpgroup
  constexpr int kSRegs = kBK / 2;            // S accumulator registers per thread
  constexpr uint32_t kQBytes = (uint32_t)(C / 64) * L::kQTile;
  constexpr uint32_t kKvBytes = (uint32_t)(C / 64) * L::kKvTile;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* k_full = reinterpret_cast<uint64_t*>(smem + L::bars);
  uint64_t* v_full = k_full + kVqAttnStages;
  uint64_t* empty = v_full + kVqAttnStages;
  uint64_t* q_full = empty + kVqAttnStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = (p.q_tile0 + (int)blockIdx.x) * kVqAttnBM, img = (int)blockIdx.y;
  const int nblk = p.T / kBK;

  if (warp == kVqAttnTmaWarp && lane == 0) {
    tma_prefetch_desc(&p.tmQ); tma_prefetch_desc(&p.tmK); tma_prefetch_desc(&p.tmV); tma_prefetch_desc(&p.tmO);
    for (int s = 0; s < kVqAttnStages; ++s) { mbar_init(&k_full[s], 1); mbar_init(&v_full[s], 1); mbar_init(&empty[s], 8); }
    mbar_init(q_full, 1);
    mbar_fence_init();
  }
  __syncthreads();
  pdl_trigger();
  pdl_wait();

  if (warp >= kVqAttnTmaWarp) {
    // ===================== TMA producer: Q once, then K_j and V_j of every key block =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kVqAttnProducerRegs));
    if (warp != kVqAttnTmaWarp) return;
    const bool el = elect_one();
    if (el) {
      mbar_arrive_expect_tx(q_full, kQBytes);
      for (int t = 0; t < C / 64; ++t) tma_load_4d(smem + L::q + t * L::kQTile, &p.tmQ, q_full, t * 64, q0, 0, img);
    }
    int stage = 0; uint32_t phase = 0;
    for (int j = 0; j < nblk; ++j) {
      mbar_wait(&empty[stage], phase ^ 1);
      if (el) {
        uint8_t* sk = smem + L::k + stage * (C / 64) * L::kKvTile;
        uint8_t* sv = smem + L::v + stage * (C / 64) * L::kKvTile;
        mbar_arrive_expect_tx(&k_full[stage], kKvBytes);
        for (int t = 0; t < C / 64; ++t) tma_load_4d(sk + t * L::kKvTile, &p.tmK, &k_full[stage], t * 64, j * kBK, 0, img);
        mbar_arrive_expect_tx(&v_full[stage], kKvBytes);
        for (int t = 0; t < C / 64; ++t) tma_load_4d(sv + t * L::kKvTile, &p.tmV, &v_full[stage], t * 64, j * kBK, 0, img);
      }
      if (++stage == kVqAttnStages) { stage = 0; phase ^= 1; }
    }
    return;
  }

  // ===================== consumers: warpgroup wg owns channels [wg * C/2, (wg + 1) * C/2) =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kVqAttnConsumerRegs));
  const int wg = warp >> 2;
  const int tid = threadIdx.x & 127;
  const uint32_t sQ0 = smem_u32(smem + L::q), sK0 = smem_u32(smem + L::k), sV0 = smem_u32(smem + L::v);
  float* xch = reinterpret_cast<float*>(smem + L::xch);

  float o[kHalf / 2];
#pragma unroll
  for (int i = 0; i < kHalf / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // rows rA, rB of this thread

  mbar_wait(q_full, 0);
  int stage = 0; uint32_t phase = 0;
  for (int j = 0; j < nblk; ++j) {
    // ---- S_wg = Q[:, half] . K_j[:, half]^T ----
    float s[kSRegs];
#pragma unroll
    for (int i = 0; i < kSRegs; ++i) s[i] = 0.f;
    mbar_wait(&k_full[stage], phase);
    wgmma_fence();
#pragma unroll
    for (int t = 0; t < kTilesHalf; ++t) {
      const int tc = wg * kTilesHalf + t;
      const uint64_t adesc = wgmma_desc_sw128(sQ0 + (uint32_t)(tc * L::kQTile));
      const uint64_t bdesc = wgmma_desc_sw128(sK0 + (uint32_t)((stage * (C / 64) + tc) * L::kKvTile));
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) Wgmma<kBK>::mma(s, adesc + 2 * kk, bdesc + 2 * kk);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);

    // ---- exchange the partial scores: both warpgroups form S_0 + S_1 ----
    float* mine = xch + ((size_t)((j & 1) * 2 + wg) * kSRegs) * 128;
    const float* other = xch + ((size_t)((j & 1) * 2 + (wg ^ 1)) * kSRegs) * 128;
#pragma unroll
    for (int i = 0; i < kSRegs; ++i) mine[i * 128 + tid] = s[i];
    named_bar_sync(1, 256);
#pragma unroll
    for (int i = 0; i < kSRegs; ++i) s[i] += other[i * 128 + tid];

    // ---- online softmax: register i holds row (i / 2) % 2 (rA / rB), column 8 (i / 4) + 2 (lane % 4) + i % 2 ----
    float corr[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < kSRegs; ++i)
        if (((i >> 1) & 1) == h) { s[i] *= p.scale_log2; mx = fmaxf(mx, s[i]); }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx);
      corr[h] = exp2f(m_run[h] - m_new);
      m_run[h] = m_new;
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < kSRegs; ++i)
        if (((i >> 1) & 1) == h) { s[i] = exp2f(s[i] - m_new); sum += s[i]; }
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      l_run[h] = l_run[h] * corr[h] + sum;
    }
    if (__any_sync(0xffffffffu, corr[0] != 1.f || corr[1] != 1.f)) {
#pragma unroll
      for (int i = 0; i < kHalf / 2; ++i) o[i] *= corr[(i >> 1) & 1];
    }
    // P as the A operand: k-step kk covers columns 16 kk .. 16 kk + 15 = accumulator registers 8 kk .. 8 kk + 7
    uint32_t pa[kBK / 16][4];
#pragma unroll
    for (int kk = 0; kk < kBK / 16; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) pa[kk][r] = pack_half2(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);

    // ---- O_wg += P . V_j[:, half] ----
    mbar_wait(&v_full[stage], phase);
    wgmma_fence();
    const uint32_t vbase = sV0 + (uint32_t)((stage * (C / 64) + wg * kTilesHalf) * L::kKvTile);
#pragma unroll
    for (int kk = 0; kk < kBK / 16; ++kk)
      WgmmaRsTB<kHalf>::mma(o, pa[kk], wgmma_desc_sw128_mn(vbase + (uint32_t)(kk * 16 * 128), (uint32_t)L::kKvTile));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    if (lane == 0) mbar_arrive(&empty[stage]);
    if (++stage == kVqAttnStages) { stage = 0; phase ^= 1; }
  }

  // ---- epilogue: O / l -> fp16, staged in the Q tile (dead once both warpgroups' last wgmma retired), TMA store ----
  named_bar_sync(1, 256);
  const float inv[2] = {1.f / l_run[0], 1.f / l_run[1]};
  const int rA = 16 * (warp & 3) + (lane >> 2);
  uint8_t* stg = smem + L::q;
#pragma unroll
  for (int i = 0; i < kHalf / 8; ++i) {
    const int c = wg * kHalf + 8 * i + 2 * (lane & 3);
    uint8_t* tile = stg + (c >> 6) * L::kQTile + 4 * (lane & 3);
    const int u = (c & 63) >> 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = rA + 8 * h;
      *reinterpret_cast<uint32_t*>(tile + r * 128 + ((u ^ (r & 7)) << 4)) =
          pack_half2(o[4 * i + 2 * h] * inv[h], o[4 * i + 2 * h + 1] * inv[h]);
    }
  }
  fence_proxy_async_smem();
  named_bar_sync(1, 256);
  if (threadIdx.x == 0) {
    for (int t = 0; t < C / 64; ++t) tma_store_4d(&p.tmO, stg + t * L::kQTile, t * 64, q0, 0, img);
    tma_store_commit();
    tma_store_wait_read();
  }
}

#endif
}  // namespace rs

// Multi-head attention over all T = H * W positions of a level, O = softmax(Q K^T D^-1/2) V per (image, head), for the
// AttentionBlocks of UNetModel (reference models/unet.py:224-344: QKVAttentionLegacy / QKVAttention, einsum path).
//
// q, k and v are channel slices of the qkv 1x1 conv's NHWC fp16 output [N * T][3C], read in place; head h of width D
// starts at column
//     legacy order (QKVAttentionLegacy): q 3Dh, k 3Dh + D, v 3Dh + 2D
//     new order (QKVAttention):          q Dh,  k C + Dh,  v 2C + Dh
// and its output goes to column Dh of [N * T][C] (the proj_out input).  One launch covers every head of every image:
// grid (ceil(T / 128), heads, N).
//
// A CTA owns 128 queries of one (image, head): consumer warpgroup w (0, 1) owns the 64-query tile w, with all D channels.
// Warp 8 is the TMA producer: the two Q tiles once, then per block of 64 keys the K block and the V block, each behind its
// own mbarrier, in a four-stage ring shared by both consumers.  The tensor map is 3-D per image ({3C, T, N}), so rows
// past T load as zeros; keys past T are masked to -inf before the row max and queries past T are not stored, so any
// T >= 1 runs.  Keys are walked in one fixed order, so results are bit-reproducible and per image (an image's output
// does not depend on the batch around it).
//
//     S [64 x 64]  = Q_w . K_j^T                        (SS wgmma m64n64k16, both K-major, 128-byte swizzle)
//     P            = exp2(S D^-1/2 log2e - m)           (fp16, kept in registers as the A operand of the next wgmma)
//     O [64 x DV]  = O * exp2(m_old - m) + P . V_j      (RS wgmma m64nDVk16, V MN-major)
//
// Loads are 64 channels wide (one 128-byte swizzle row).  At D = 32 the box holds the head's 32 channels and 32 of the
// neighbouring columns: Q K^T runs over the first two k16 steps only, and P V computes 64 output columns of which the
// first 32 are stored (DV = 64; the other 32 cost tensor time the exp2 rate hides: at D = 32 the kernel is bound by one
// MUFU exp2 per 128 tensor FLOPs).  At D = 128 there are two 64-channel tiles per row block.
//
// Shared memory: Q 2 x (D / 64) x 8 KB + 4 stages x (K + V) (D / 64) x 8 KB: 80 KB at D <= 64, 160 KB at D = 128.
#pragma once

#include "common.cuh"
#include "conv_gemm.cuh"
#include "vq_attn.cuh"

namespace rs {

constexpr int kUnetAttnBM = 64;              // queries per consumer warpgroup
constexpr int kUnetAttnCtaRows = 128;        // queries per CTA
constexpr int kUnetAttnBK = 64;              // keys per block
constexpr int kUnetAttnStages = 4;
constexpr int kUnetAttnThreads = 384;        // two consumer warpgroups + the producer warpgroup (warp 8 issues the loads)
constexpr int kUnetAttnTmaWarp = 8;

struct UnetAttnParams {
  CUtensorMap tm;                    // qkv {3C, T, 1, N}, box {64, 64, 1, 1}, 128-byte swizzle
  __half* out; long long out_sN; int out_ld;   // output rows of image n: out + n * out_sN + t * out_ld, head h at column D h
  int T;
  int head_stride;                   // column step between heads of q (and of k, v): 3D (legacy) or D (new order)
  int k_col0, v_col0;                // columns of head 0's k and v: D, 2D (legacy) or C, 2C (new order)
  float scale_log2;                  // D^-1/2 * log2(e)
};

template <int D>
struct UnetAttnSmem {
  static constexpr int kTiles = D <= 64 ? 1 : D / 64;       // 64-channel tiles per row block
  static constexpr int kTile = 64 * 128;                    // [64 rows x 64 channels] fp16
  static constexpr int q = 0;                               // [2 warpgroups][kTiles]
  static constexpr int k = q + 2 * kTiles * kTile;          // [stage][kTiles]
  static constexpr int v = k + kUnetAttnStages * kTiles * kTile;
  static constexpr int bars = v + kUnetAttnStages * kTiles * kTile;
  static constexpr int total = bars + 128;
  static constexpr int launch_bytes = total + 1024;         // + alignment slack of the dynamic shared memory base
};

#ifdef __CUDACC__

template <int D>
__global__ void __launch_bounds__(kUnetAttnThreads, 1) unet_attn_sm90_kernel(const __grid_constant__ UnetAttnParams p) {
  static_assert(D == 32 || D == 64 || D == 128, "unet_attn: head dim in {32, 64, 128}");
  using L = UnetAttnSmem<D>;
  constexpr int kTiles = L::kTiles;
  constexpr int kDV = D < 64 ? 64 : D;             // output columns computed per row (D = 32: 64, half of them stored)
  constexpr int kKSteps = D < 64 ? 2 : 4;          // k16 steps of Q K^T per 64-channel tile
  constexpr uint32_t kQBytes = 2u * kTiles * L::kTile;
  constexpr uint32_t kKvBytes = (uint32_t)kTiles * L::kTile;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* k_full = reinterpret_cast<uint64_t*>(smem + L::bars);
  uint64_t* v_full = k_full + kUnetAttnStages;
  uint64_t* empty = v_full + kUnetAttnStages;
  uint64_t* q_full = empty + kUnetAttnStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = (int)blockIdx.x * kUnetAttnCtaRows, head = (int)blockIdx.y, img = (int)blockIdx.z;
  const int nblk = (p.T + kUnetAttnBK - 1) / kUnetAttnBK;

  if (warp == kUnetAttnTmaWarp && lane == 0) {
    tma_prefetch_desc(&p.tm);
    for (int s = 0; s < kUnetAttnStages; ++s) { mbar_init(&k_full[s], 1); mbar_init(&v_full[s], 1); mbar_init(&empty[s], 8); }
    mbar_init(q_full, 1);
    mbar_fence_init();
  }
  __syncthreads();
  pdl_trigger();
  pdl_wait();

  if (warp >= kUnetAttnTmaWarp) {
    // ===================== TMA producer: both Q tiles once, then K_j and V_j of every key block =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kVqAttnProducerRegs));
    if (warp != kUnetAttnTmaWarp) return;
    const bool el = elect_one();
    const int qc = head * p.head_stride, kc = p.k_col0 + qc, vc = p.v_col0 + qc;
    if (el) {
      mbar_arrive_expect_tx(q_full, kQBytes);
      for (int w = 0; w < 2; ++w)
        for (int t = 0; t < kTiles; ++t)
          tma_load_4d(smem + L::q + (w * kTiles + t) * L::kTile, &p.tm, q_full, qc + 64 * t, q0 + kUnetAttnBM * w, 0, img);
    }
    int stage = 0; uint32_t phase = 0;
    for (int j = 0; j < nblk; ++j) {
      mbar_wait(&empty[stage], phase ^ 1);
      if (el) {
        uint8_t* sk = smem + L::k + stage * kTiles * L::kTile;
        uint8_t* sv = smem + L::v + stage * kTiles * L::kTile;
        mbar_arrive_expect_tx(&k_full[stage], kKvBytes);
        for (int t = 0; t < kTiles; ++t) tma_load_4d(sk + t * L::kTile, &p.tm, &k_full[stage], kc + 64 * t, j * kUnetAttnBK, 0, img);
        mbar_arrive_expect_tx(&v_full[stage], kKvBytes);
        for (int t = 0; t < kTiles; ++t) tma_load_4d(sv + t * L::kTile, &p.tm, &v_full[stage], vc + 64 * t, j * kUnetAttnBK, 0, img);
      }
      if (++stage == kUnetAttnStages) { stage = 0; phase ^= 1; }
    }
    return;
  }

  // ===================== consumers: warpgroup wg owns queries [q0 + 64 wg, q0 + 64 wg + 64) =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kVqAttnConsumerRegs));
  const int wg = warp >> 2;
  const uint32_t sQ = smem_u32(smem + L::q) + (uint32_t)(wg * kTiles * L::kTile);
  const uint32_t sK0 = smem_u32(smem + L::k), sV0 = smem_u32(smem + L::v);

  float o[kDV / 2];
#pragma unroll
  for (int i = 0; i < kDV / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // rows rA, rB of this thread

  mbar_wait(q_full, 0);
  int stage = 0; uint32_t phase = 0;
  for (int j = 0; j < nblk; ++j) {
    // ---- S = Q . K_j^T ----
    float s[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = 0.f;
    mbar_wait(&k_full[stage], phase);
    wgmma_fence();
#pragma unroll
    for (int t = 0; t < kTiles; ++t) {
      const uint64_t adesc = wgmma_desc_sw128(sQ + (uint32_t)(t * L::kTile));
      const uint64_t bdesc = wgmma_desc_sw128(sK0 + (uint32_t)((stage * kTiles + t) * L::kTile));
#pragma unroll
      for (int kk = 0; kk < kKSteps; ++kk) Wgmma<64>::mma(s, adesc + 2 * kk, bdesc + 2 * kk);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);

    // ---- online softmax: register i holds row (i / 2) % 2 (rA / rB), key 64 j + 8 (i / 4) + 2 (lane % 4) + i % 2 ----
    const int kv_left = p.T - j * kUnetAttnBK;      // valid keys in this block (>= 1)
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      s[i] *= p.scale_log2;
      if (kv_left < kUnetAttnBK && 8 * (i >> 2) + 2 * (lane & 3) + (i & 1) >= kv_left) s[i] = -INFINITY;
    }
    float corr[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (((i >> 1) & 1) == h) mx = fmaxf(mx, s[i]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx);
      corr[h] = exp2f(m_run[h] - m_new);
      m_run[h] = m_new;
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (((i >> 1) & 1) == h) { s[i] = exp2f(s[i] - m_new); sum += s[i]; }
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      l_run[h] = l_run[h] * corr[h] + sum;
    }
    if (__any_sync(0xffffffffu, corr[0] != 1.f || corr[1] != 1.f)) {
#pragma unroll
      for (int i = 0; i < kDV / 2; ++i) o[i] *= corr[(i >> 1) & 1];
    }
    // P as the A operand: k-step kk covers keys 16 kk .. 16 kk + 15 = accumulator registers 8 kk .. 8 kk + 7
    uint32_t pa[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) pa[kk][r] = pack_half2(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);

    // ---- O += P . V_j ----
    mbar_wait(&v_full[stage], phase);
    wgmma_fence();
    const uint32_t vbase = sV0 + (uint32_t)(stage * kTiles * L::kTile);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      WgmmaRsTB<kDV>::mma(o, pa[kk], wgmma_desc_sw128_mn(vbase + (uint32_t)(kk * 16 * 128), (uint32_t)L::kTile));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    if (lane == 0) mbar_arrive(&empty[stage]);
    if (++stage == kUnetAttnStages) { stage = 0; phase ^= 1; }
  }

  // ---- epilogue: O / l -> fp16, straight to the rows of this warpgroup's tile that lie inside T ----
  const float inv[2] = {1.f / l_run[0], 1.f / l_run[1]};
  const int rA = q0 + kUnetAttnBM * wg + 16 * (warp & 3) + (lane >> 2);
  __half* obase = p.out + (long long)img * p.out_sN + head * D;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = rA + 8 * h;
    if (r >= p.T) continue;
    __half* orow = obase + (long long)r * p.out_ld;
#pragma unroll
    for (int i = 0; i < kDV / 8; ++i) {
      const int c = 8 * i + 2 * (lane & 3);
      if (c < D)
        *reinterpret_cast<uint32_t*>(orow + c) = pack_half2(o[4 * i + 2 * h] * inv[h], o[4 * i + 2 * h + 1] * inv[h]);
    }
  }
}

#endif
}  // namespace rs

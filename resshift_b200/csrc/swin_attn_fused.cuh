// The attention half of a Swin block as ONE kernel:
//
//     y = x + proj( window_attention( qkv( norm1(x) ) ) )            (+ GroupNorm statistics of y for norm2)
//
// reference: SwinTransformerBlock.forward, models/swin_transformer.py:246-275 (norm1 = GroupNorm32, torch.roll,
// window_partition, WindowAttention.forward :114-145 incl. qkv / relative-position bias / shift mask / softmax / proj,
// window_reverse, roll back, residual).  Unfused this is four launches (gn_apply, qkv GEMM, window_attn, proj GEMM) and a
// [pixels, 3E] fp16 round trip through HBM / L2 (150 MB per block at batch 16, 64x64); here a CTA owns TWO 8x8 windows
// (128 tokens) and nothing but x and y touches global memory.  Warpgroup g owns window g of the pair (64 token rows);
// warp 8 is the TMA producer of the weights.  The two warpgroups share nothing but the weight ring, so they synchronise
// only through its mbarriers and their own named barriers.
//
//   * the 64 token rows of a window are gathered with cp.async (the cyclic shift and the window partition are address
//     arithmetic: wrapped windows do not map onto TMA boxes) straight into the 128-byte-swizzled K-major layout a TMA
//     load would produce, then normalised in place (per-image affine from the producers' (mean, M2) pairs, gn_stats.cuh);
//   * per head pair (2j, 2j + 1): the q, k and v rows of W_qkv are three contiguous 64-row ranges, loaded as three TMA
//     boxes into one [192 x 64] ring slot per 64-channel k-block; one wgmma m64n192 chain gives [q | k | v] of both heads
//     for the window's 64 tokens (96 fp32 per thread), stored + bias as fp16 like the unfused path stores qkv: q and k
//     K-major, v transposed (dims x tokens) so that P . V_h is a register-A wgmma with a K-major B operand;
//   * per head: S = Q_h K_h^T (wgmma m64n64, two k16 steps inside the 64-wide swizzled block), + relative-position bias,
//     + shift mask, softmax in fp32 registers (same arithmetic as window_attn_kernel), P kept in registers as the A
//     operand of O_h = P . V_h (wgmma m64n32), O_h / rowsum stored as fp16 into the swizzled O tile;
//   * y = O . W_proj^T + b + x with W_proj streamed through the same ring, raw x re-fetched into the (dead) X tile while
//     the attention and the projection run, results staged in the (dead) O tile and written as full token rows;
//   * (mean, M2) of y per (image, window, channel) for the norm2 that follows (slots = windows per image, 64 tokens each).
//
// The producer runs ahead over the CTA's whole (persistent, contiguous) pair range; weights do not depend on the previous
// kernel, so it never waits for it (PDL) and the first slots land while that kernel drains.
#pragma once

#include "common.cuh"
#include "gn_stats.cuh"
#include "window_attn.cuh"
#include "wgmma.cuh"

namespace rs {

struct SwinAttnParams {
  CUtensorMap tmWqkv, tmWproj;          // {wqkv_ld, 3E} / {wproj_ld, E} fp16, boxes {64, 64}, 128-byte swizzle
  const __half* x; int x_ld;            // [N*H*W, E] view (row stride x_ld)
  __half* y; int y_ld;                  // output view (may alias x: every token row is read before it is written)
  int N, H, W, heads;
  int shift;                            // 0 or 4
  float scale;                          // head_dim^-0.5
  // norm1: the producers' (mean, M2) pairs gn_part[N][gn_slots][E][2]
  const float* gn_part; int gn_slots;
  const float* gamma; const float* beta; float eps;
  const __half* wqkv; int wqkv_ld;      // [3E][E] fp16, row stride wqkv_ld
  const float* bqkv;                    // [3E]
  const float* relbias;                 // [heads][64][64] fp32
  const __half* wproj; int wproj_ld;    // [E][E]
  const float* bproj;                   // [E]
  GnSink sink[2];                       // statistics of y (slots = windows per image, 64 values each)
  int total_windows;                    // N * (H/8) * (W/8)
};

constexpr int kSwinThreads = 288;       // two consumer warpgroups (window 0 / 1 of the pair) + the TMA producer warp
constexpr int kSwinTmaWarp = 8;
constexpr int kSwinRing = 3;            // weight ring slots of [192 rows x 64] fp16

// shared-memory layout (offsets from the 1024-aligned base); every operand tile is [rows x 64] fp16 with the 128-byte
// swizzle, rows 128 B apart; a [128 x 64] tile holds window 0 in rows 0..63 and window 1 in rows 64..127
template <int kE>
struct SwinSmem {
  static constexpr int kKb = kE / 64;                       // 64-channel k-blocks
  static constexpr int kTile = 128 * 128;                   // [128 rows x 64]
  static constexpr int kWin = 64 * 128;                     // one window's rows of a tile; also one [64 x 64] block
  static constexpr int kSlot = 192 * 128;
  static constexpr int x = 0;                               // kKb tiles: normalised X, then the raw x rows (residual)
  static constexpr int o = x + kKb * kTile;                 // kKb tiles: attention output, then the staged y rows
  static constexpr int qkv = o + kKb * kTile;               // [2 windows][q | k | v^T] blocks; also per-window scratch
  static constexpr int ring = qkv + 2 * 3 * kWin;
  static constexpr int ab = ring + kSwinRing * kSlot;       // [2 windows][kE][2] norm1 affine
  static constexpr int mr = ab + 2 * kE * 2 * 4;            // [2 windows][32][2] group (mean, rstd)
  static constexpr int pix = mr + 2 * 32 * 2 * 4;           // [2 windows][64] token -> pixel row, or -1
  static constexpr int bias = pix + 2 * 64 * 4;             // [3E] qkv bias, then [E] proj bias (fp32)
  static constexpr int bars = bias + 4 * kE * 4;
  static constexpr int total = bars + 2 * kSwinRing * 8;
  static constexpr int launch_bytes = total + 1024;         // + alignment slack of the dynamic shared memory base
};

#ifdef __CUDACC__

template <int kE>
__global__ void __launch_bounds__(kSwinThreads, 1) swin_attn_fused_kernel(const __grid_constant__ SwinAttnParams p) {
  static_assert(kE == 64 || kE == 192, "fused Swin attention: E in {64, 192}");
  using L = SwinSmem<kE>;
  constexpr int kKb = L::kKb;
  constexpr int kHeadPairs = kE / 64;
  constexpr int kPieces = kE / 8;                           // 16-byte pieces per token row
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + L::bars);
  uint64_t* empty = full + kSwinRing;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_pairs = (p.total_windows + 1) >> 1;
  const int per_cta = (num_pairs + gridDim.x - 1) / gridDim.x;
  const int pair_begin = blockIdx.x * per_cta;
  const int pair_end = min(pair_begin + per_cta, num_pairs);

  if (warp == kSwinTmaWarp && lane == 0) {
    tma_prefetch_desc(&p.tmWqkv); tma_prefetch_desc(&p.tmWproj);
    for (int s = 0; s < kSwinRing; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    mbar_fence_init();
  }
  __syncthreads();
  pdl_trigger();

  if (warp == kSwinTmaWarp) {
    // ===================== TMA producer: per pair, the qkv slots of every head pair, then the proj slots =============
    const bool el = elect_one();
    int stage = 0; uint32_t phase = 0;
    for (int pair = pair_begin; pair < pair_end; ++pair) {
      for (int j = 0; j < kHeadPairs; ++j)
        for (int kb = 0; kb < kKb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          if (el) {
            uint8_t* dst = smem + L::ring + stage * L::kSlot;
            mbar_arrive_expect_tx(&full[stage], 3 * L::kWin);
            for (int w = 0; w < 3; ++w) tma_load_2d(dst + w * L::kWin, &p.tmWqkv, &full[stage], kb * 64, w * kE + j * 64);
          }
          if (++stage == kSwinRing) { stage = 0; phase ^= 1; }
        }
      for (int kb = 0; kb < kKb; ++kb) {
        mbar_wait(&empty[stage], phase ^ 1);
        if (el) {
          uint8_t* dst = smem + L::ring + stage * L::kSlot;
          mbar_arrive_expect_tx(&full[stage], kE * 128);
          for (int r = 0; r < kE / 64; ++r) tma_load_2d(dst + r * L::kWin, &p.tmWproj, &full[stage], kb * 64, r * 64);
        }
        if (++stage == kSwinRing) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup wg owns window 2 * pair + wg =====================
  const int wg = warp >> 2;
  const int wt = threadIdx.x & 127;
  const int g = lane >> 2, t = lane & 3;
  const int r0 = 16 * (warp & 3) + g;                       // this thread's token rows in the window: r0 and r0 + 8
  uint8_t* sX = smem + L::x + wg * L::kWin;                 // k-block kb at + kb * kTile
  uint8_t* sO = smem + L::o + wg * L::kWin;
  uint8_t* sQ = smem + L::qkv + wg * 3 * L::kWin;           // [64 tokens x 64 (2 heads x 32)]
  uint8_t* sK = sQ + L::kWin;                               // [64 tokens x 64]
  uint8_t* sVt = sK + L::kWin;                              // [64 (2 heads x 32 dims) x 64 tokens]
  float* sScr = reinterpret_cast<float*>(sQ);               // norm1 per-channel pairs, then the statistics of y
  float* sAB = reinterpret_cast<float*>(smem + L::ab) + wg * kE * 2;
  float* sMR = reinterpret_cast<float*>(smem + L::mr) + wg * 64;
  int* sPix = reinterpret_cast<int*>(smem + L::pix) + wg * 64;
  const float* sBqkv = reinterpret_cast<const float*>(smem + L::bias);
  const float* sBproj = sBqkv + 3 * kE;
  const uint32_t sX0 = smem_u32(sX), sO0 = smem_u32(sO), ring0 = smem_u32(smem + L::ring);
  const int nWx = p.W >> 3, nWy = p.H >> 3, nW = nWx * nWy;
  const int HW = p.H * p.W;
  auto wg_sync = [&]() { named_bar_sync(1 + wg, 128); };
  // byte offset of (row r, channels c .. c + 1) in a swizzled [rows x 64] block
  auto swz = [](int r, int c) { return r * 128 + ((((c >> 3) ^ r) & 7) << 4) + (c & 7) * 2; };

  int stage = 0; uint32_t phase = 0;
  auto release = [&](int s) { if (s >= 0 && lane == 0) mbar_arrive(&empty[s]); };
  int cur_img = -1;
  // the biases are read from shared memory: the epilogues then only wait for shared-memory loads
  for (int i = threadIdx.x; i < 4 * kE; i += 256)
    reinterpret_cast<float*>(smem + L::bias)[i] = i < 3 * kE ? __ldg(p.bqkv + i) : __ldg(p.bproj + i - 3 * kE);
  named_bar_sync(3, 256);
  pdl_wait();

  for (int pair = pair_begin; pair < pair_end; ++pair) {
    // ---- geometry of the window ----
    const int w = 2 * pair + wg;
    const bool wvalid = w < p.total_windows;
    const int wc = min(w, p.total_windows - 1);
    const int n_img = wc / nW, wy = (wc % nW) / nWx;
    if (wt < 64) {
      int pix = -1;
      if (wvalid) {
        const int wx = (wc % nW) % nWx;
        const int yy = (wy * 8 + (wt >> 3) + p.shift) % p.H, xx = (wx * 8 + (wt & 7) + p.shift) % p.W;
        pix = (n_img * p.H + yy) * p.W + xx;
      }
      sPix[wt] = pix;
    }
    wg_sync();
    // ---- gather the 64 token rows (raw x) into the swizzled X blocks ----
    for (int i = wt; i < 64 * kPieces; i += 128) {
      const int r = i / kPieces, u = i - r * kPieces;
      uint8_t* dst = sX + (u >> 3) * L::kTile + swz(r, u * 8);
      const int pix = sPix[r];
      if (pix >= 0) cp_async_16(dst, p.x + (long long)pix * p.x_ld + u * 8);
      else *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
    }
    cp_async_commit();
    // ---- norm1 affine of the window's image (recomputed only when the image changes) ----
    if (n_img != cur_img) {                                 // uniform over the warpgroup
      constexpr int cpg = kE / 32;
      const float ns = (float)HW / (float)p.gn_slots;
      for (int c = wt; c < kE; c += 128) {
        const float2 mq = gn_channel_from_pairs(p.gn_part + (size_t)n_img * p.gn_slots * kE * 2 + (size_t)c * 2, p.gn_slots, kE, ns);
        sScr[c * 2] = mq.x; sScr[c * 2 + 1] = mq.y;
      }
      wg_sync();
      if (wt < 32) {
        float chp[2 * cpg];
#pragma unroll
        for (int k = 0; k < cpg; ++k) { chp[2 * k] = sScr[(wt * cpg + k) * 2]; chp[2 * k + 1] = sScr[(wt * cpg + k) * 2 + 1]; }
        const float2 mr = gn_group_from_channels(chp, cpg, (float)HW, p.eps);
        sMR[wt * 2] = mr.x; sMR[wt * 2 + 1] = mr.y;
      }
      wg_sync();
      for (int c = wt; c < kE; c += 128) {
        const int gg = c / cpg;
        const float a = sMR[gg * 2 + 1] * __ldg(p.gamma + c);
        const float b = __ldg(p.beta + c) - sMR[gg * 2] * a;
        sAB[c * 2] = a; sAB[c * 2 + 1] = b;
      }
      cur_img = n_img;
    }
    // ---- wait for x, normalise in place ----
    cp_async_wait<0>();
    wg_sync();
    for (int i = wt; i < 64 * kPieces; i += 128) {
      const int u = i >> 6, r = i & 63;                     // a warp: one 8-channel piece of 32 rows (affine broadcast)
      const float* ab = sAB + u * 8 * 2;
      uint4* ptr = reinterpret_cast<uint4*>(sX + (u >> 3) * L::kTile + swz(r, u * 8));
      uint4 raw = *ptr;
      __half2* hh = reinterpret_cast<__half2*>(&raw);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float2 f = __half22float2(hh[k]);
        f.x = fmaf(f.x, ab[(2 * k) * 2], ab[(2 * k) * 2 + 1]);
        f.y = fmaf(f.y, ab[(2 * k + 1) * 2], ab[(2 * k + 1) * 2 + 1]);
        hh[k] = __floats2half2_rn(f.x, f.y);
      }
      *ptr = raw;
    }
    fence_proxy_async_smem();                               // the tensor core reads X through the async proxy
    wg_sync();

    const int la = p.shift ? swin_label(wy, r0 & 7, p.H, p.shift) : 0;       // (r0 + 8) & 7 == r0 & 7

    // ================= head pairs =================
    for (int j = 0; j < kHeadPairs; ++j) {
      // ---- [q | k | v] of heads 2j, 2j + 1 (64 tokens x 192) = Xn . W_j^T ----
      float acc[96];
#pragma unroll
      for (int i = 0; i < 96; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < kKb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint64_t adesc = wgmma_desc_sw128(sX0 + (uint32_t)(kb * L::kTile));
        const uint64_t bdesc = wgmma_desc_sw128(ring0 + (uint32_t)(stage * L::kSlot));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) Wgmma<192>::mma(acc, adesc + 2 * k, bdesc + 2 * k);
        wgmma_commit();
        wgmma_wait<1>();
        release(prev);
        prev = stage;
        if (++stage == kSwinRing) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      release(prev);
      wg_sync();                                            // every warp's reads of the previous head pair's q / k / v^T retired
      // + bias, round to fp16 (as the unfused path stores qkv): q and k K-major, v transposed
#pragma unroll
      for (int i = 0; i < 24; ++i) {
        const int c = 8 * i + 2 * t, which = i >> 3, cc = c & 63;
        const float2 bb = *reinterpret_cast<const float2*>(sBqkv + which * kE + 64 * j + cc);
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int r = r0 + 8 * hr;
          const float v0 = acc[4 * i + 2 * hr] + bb.x, v1 = acc[4 * i + 2 * hr + 1] + bb.y;
          if (which < 2) {
            *reinterpret_cast<__half2*>(sQ + which * L::kWin + swz(r, cc)) = __floats2half2_rn(v0, v1);
          } else {
            *reinterpret_cast<__half*>(sVt + swz(cc, r)) = __float2half_rn(v0);
            *reinterpret_cast<__half*>(sVt + swz(cc + 1, r)) = __float2half_rn(v1);
          }
        }
      }
      fence_proxy_async_smem();
      wg_sync();                                            // q, k, v^T of all 64 tokens in place
      if (j == kHeadPairs - 1) {
        // the normalised X rows are dead (every warp's last qkv wgmma retired before the barrier above): fetch the RAW
        // rows (residual) into them; they land while the attention and the projection run
        for (int i = wt; i < 64 * kPieces; i += 128) {
          const int r = i / kPieces, u = i - r * kPieces;
          const int pix = sPix[r];
          if (pix >= 0) cp_async_16(sX + (u >> 3) * L::kTile + swz(r, u * 8), p.x + (long long)pix * p.x_ld + u * 8);
        }
        cp_async_commit();
      }
      // ---- attention core of heads 2j, 2j + 1 (same arithmetic as window_attn_kernel) ----
#pragma unroll 1
      for (int hh = 0; hh < 2; ++hh) {
        const int h = 2 * j + hh;
        // this thread's relative-position-bias values (independent of everything staged): issue early
        const float* bias = p.relbias + (size_t)h * 64 * 64;
        float2 bv0[8], bv1[8];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          bv0[nt] = __ldg(reinterpret_cast<const float2*>(bias + r0 * 64 + nt * 8 + 2 * t));
          bv1[nt] = __ldg(reinterpret_cast<const float2*>(bias + (r0 + 8) * 64 + nt * 8 + 2 * t));
        }
        // S = Q_h . K_h^T: register 4 nt + e holds row r0 + 8 (e >> 1), key 8 nt + 2 t + (e & 1)
        float s[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) s[i] = 0.f;
        const uint64_t qdesc = wgmma_desc_sw128(smem_u32(sQ)) + 4 * hh;       // + 32 channels = 64 B
        const uint64_t kdesc = wgmma_desc_sw128(smem_u32(sK)) + 4 * hh;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) Wgmma<64>::mma(s, qdesc + 2 * kk, kdesc + 2 * kk);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(s);
        float mx0 = -1e30f, mx1 = -1e30f;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          const int col = nt * 8 + 2 * t;
          const float2 b0 = bv0[nt], b1 = bv1[nt];
          float m0 = 0.f, m1 = 0.f;
          if (p.shift) {
            if (swin_label(wy, col & 7, p.H, p.shift) != la) m0 = -100.0f;
            if (swin_label(wy, (col + 1) & 7, p.H, p.shift) != la) m1 = -100.0f;
          }
          s[4 * nt + 0] = s[4 * nt + 0] * p.scale + b0.x + m0;
          s[4 * nt + 1] = s[4 * nt + 1] * p.scale + b0.y + m1;
          s[4 * nt + 2] = s[4 * nt + 2] * p.scale + b1.x + m0;
          s[4 * nt + 3] = s[4 * nt + 3] * p.scale + b1.y + m1;
          mx0 = fmaxf(mx0, fmaxf(s[4 * nt + 0], s[4 * nt + 1]));
          mx1 = fmaxf(mx1, fmaxf(s[4 * nt + 2], s[4 * nt + 3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            s[4 * nt + e] = __expf(s[4 * nt + e] - mx0); sum0 += s[4 * nt + e];
            s[4 * nt + 2 + e] = __expf(s[4 * nt + 2 + e] - mx1); sum1 += s[4 * nt + 2 + e];
          }
        }
        sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1); sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
        sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1); sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
        // O_h = P . V_h: P (fp16) as the A operand, k-step kk = keys 16 kk .. 16 kk + 15 = registers 8 kk .. 8 kk + 7
        uint32_t pa[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
          for (int rr = 0; rr < 4; ++rr) pa[kk][rr] = pack_h2(s[8 * kk + 2 * rr], s[8 * kk + 2 * rr + 1]);
        float o[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) o[i] = 0.f;
        const uint64_t vdesc = wgmma_desc_sw128(smem_u32(sVt) + (uint32_t)(hh * 32 * 128));
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) WgmmaRs<32>::mma(o, pa[kk], vdesc + 2 * kk);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int cc = hh * 32 + 8 * i + 2 * t;
          *reinterpret_cast<__half2*>(sO + j * L::kTile + swz(r0, cc)) = __floats2half2_rn(o[4 * i] * inv0, o[4 * i + 1] * inv0);
          *reinterpret_cast<__half2*>(sO + j * L::kTile + swz(r0 + 8, cc)) = __floats2half2_rn(o[4 * i + 2] * inv1, o[4 * i + 3] * inv1);
        }
      }
    }

    // ================= projection: y = O . W_proj^T + b + x =================
    fence_proxy_async_smem();
    wg_sync();                                              // O of all heads and tokens in place
    float acc2[kE / 2];
#pragma unroll
    for (int i = 0; i < kE / 2; ++i) acc2[i] = 0.f;
    {
      int prev = -1;
      for (int kb = 0; kb < kKb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint64_t adesc = wgmma_desc_sw128(sO0 + (uint32_t)(kb * L::kTile));
        const uint64_t bdesc = wgmma_desc_sw128(ring0 + (uint32_t)(stage * L::kSlot));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) Wgmma<kE>::mma(acc2, adesc + 2 * k, bdesc + 2 * k);
        wgmma_commit();
        wgmma_wait<1>();
        release(prev);
        prev = stage;
        if (++stage == kSwinRing) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc2);
      release(prev);
    }
    cp_async_wait<0>();                                     // this thread's raw x rows
    wg_sync();                                              // everyone's; and every warp's proj wgmma retired (O is free)
    // ---- epilogue: + bias + raw x -> fp16 (one rounding), staged in O, statistics, row stores ----
    float* sStat = sScr;                                    // [4 warps][kE][2] = (mean, M2) over the warp's 16 rows
    const bool want_stats = p.sink[0].part != nullptr;
#pragma unroll
    for (int i = 0; i < kE / 8; ++i) {
      const int c = 8 * i + 2 * t;
      const int off0 = (c >> 6) * L::kTile + swz(r0, c & 63), off1 = (c >> 6) * L::kTile + swz(r0 + 8, c & 63);
      const float2 bb = *reinterpret_cast<const float2*>(sBproj + c);
      const float2 x0 = __half22float2(*reinterpret_cast<const __half2*>(sX + off0));
      const float2 x1 = __half22float2(*reinterpret_cast<const __half2*>(sX + off1));
      const __half2 y0 = __floats2half2_rn(acc2[4 * i] + bb.x + x0.x, acc2[4 * i + 1] + bb.y + x0.y);
      const __half2 y1 = __floats2half2_rn(acc2[4 * i + 2] + bb.x + x1.x, acc2[4 * i + 3] + bb.y + x1.y);
      *reinterpret_cast<__half2*>(sO + off0) = y0;
      *reinterpret_cast<__half2*>(sO + off1) = y1;
      if (want_stats) {
        // column sums over the 16 rows of the warp (values as stored): the rows live in the 8 lane groups g, fixed tree
        const float2 f0 = __half22float2(y0), f1 = __half22float2(y1);
        float sx = f0.x + f1.x, sy = f0.y + f1.y;
        float qx = fmaf(f0.x, f0.x, f1.x * f1.x), qy = fmaf(f0.y, f0.y, f1.y * f1.y);
#pragma unroll
        for (int off = 4; off <= 16; off <<= 1) {
          sx += __shfl_xor_sync(0xffffffffu, sx, off); sy += __shfl_xor_sync(0xffffffffu, sy, off);
          qx += __shfl_xor_sync(0xffffffffu, qx, off); qy += __shfl_xor_sync(0xffffffffu, qy, off);
        }
        if (g == 0) {
          const float m0 = sx * (1.0f / 16.0f), m1 = sy * (1.0f / 16.0f);
          float* dst = sStat + ((size_t)(warp & 3) * kE + c) * 2;
          dst[0] = m0; dst[1] = fmaxf(qx - sx * m0, 0.f);
          dst[2] = m1; dst[3] = fmaxf(qy - sy * m1, 0.f);
        }
      }
    }
    wg_sync();                                              // staged rows and per-warp statistics complete
    if (wvalid) {
      // full token rows to global
      for (int i = wt; i < 64 * kPieces; i += 128) {
        const int r = i / kPieces, u = i - r * kPieces;
        *reinterpret_cast<uint4*>(p.y + (long long)sPix[r] * p.y_ld + u * 8) =
            *reinterpret_cast<const uint4*>(sO + (u >> 3) * L::kTile + swz(r, u * 8));
      }
      if (want_stats) {
        // merge the four 16-row warps of the window (Chan et al., equal counts) and deliver the window's pairs
        const int slot = w % nW;
        for (int c = wt; c < kE; c += 128) {
          float m[4], q[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) { m[k] = sStat[((size_t)k * kE + c) * 2]; q[k] = sStat[((size_t)k * kE + c) * 2 + 1]; }
          float ma, qa, mb, qb, mm, qq;
          chan_merge_equal(16.f, m[0], q[0], m[1], q[1], ma, qa);
          chan_merge_equal(16.f, m[2], q[2], m[3], q[3], mb, qb);
          chan_merge_equal(32.f, ma, qa, mb, qb, mm, qq);
#pragma unroll
          for (int d = 0; d < 2; ++d) {
            const GnSink& sk = p.sink[d];
            if (!sk.part) continue;
            float* dst = sk.part + (((size_t)n_img * nW + slot) * sk.cstride + sk.coff + c) * 2;
            dst[0] = mm; dst[1] = qq;
          }
        }
      }
    }
    wg_sync();                                              // this window's shared memory is free for the next pair
  }
}

#endif  // __CUDACC__
}  // namespace rs

// Fused Swin MLP:  out = residual + fc2( GELU( fc1(x) ) )  in ONE kernel on wgmma, hidden activations never leave the SM.
//
// reference: Mlp.forward (models/swin_transformer.py:27-33: 1x1 conv E -> 4E, exact-erf GELU, 1x1 conv 4E -> E) and the
// residual add around it in SwinTransformerBlock.forward (:279).  Unfused this is two GEMMs with a [pixels, 4E] fp16
// intermediate written to and re-read from HBM; here a CTA owns a 128-pixel tile and walks the hidden dimension in
// chunks of 64 (with the accumulators of both GEMMs in registers, a wider chunk would spill).  Each of the two consumer
// warpgroups owns 64 rows of the tile:
//
//     acc1[64 x 64]   = X[64 x E] . W1_j^T            (wgmma, registers)
//     H_j             = GELU(acc1 + b1_j) -> fp16, written to shared memory as the next wgmma's A operand
//                                           (K-major, 128-byte swizzle: what a TMA load would have produced)
//     acc2[64 x E]   += H_j . W2_j^T                   (wgmma, registers, accumulates over all chunks)
//
// then the staged epilogue of conv_gemm.cuh (+ b2, + residual through a TMA load, fp16, TMA store, GroupNorm partials).
// Warp 8 is the TMA producer: X once, then per chunk the fc1 weight tiles followed by the fc2 weight tiles, through one
// ring of slots in the order the consumers use them.  The Swin block's norm2 runs in front of this kernel (gn_apply_kernel).
#pragma once

#include "common.cuh"
#include "conv_gemm.cuh"

namespace rs {

constexpr int kMlpHc = 64;                  // hidden columns per chunk (one 128-byte swizzled K tile of GEMM 2)
constexpr int kMlpThreads = kConvThreads;   // two consumer warpgroups + the TMA producer warp
constexpr int kMlpTmaWarp = kConvTmaWarp;

struct MlpParams {
  CUtensorMap tmX, tmW1, tmW2, tmOut, tmRes;
  const float* bias1;                // [Hd]
  const float* bias2;                // [E]
  int E, Hd;                         // E in {64, 128, 192, 256};  Hd % 64 == 0
  int ring;                          // weight ring depth (slots of max(64, E) rows x 64 fp16)
  int bw, bh, bn, tiles_w, tiles_h;
  int Wout, Hout, Nimg;
  int has_res;
  GnSink sink[2]; int gn_slots;      // fused GroupNorm statistics of the output (gn_stats.cuh)
};

// shared-memory layout (offsets from the 1024-aligned base)
struct MlpSmem {
  int x, h, ring, bars, b1, b2, total;
  __host__ __device__ MlpSmem(int E, int Hd, int ring_depth) {
    const int slot = (E > kMlpHc ? E : kMlpHc) * kConvBK * 2;
    x = 0;                                          // E/64 tiles of [128 rows x 64] (the staging area at the end)
    h = x + (E / 64) * kConvBM * kConvBK * 2;       // [128 rows x 64]: one hidden chunk
    ring = h + (kMlpHc / 64) * kConvBM * kConvBK * 2;
    bars = ring + ring_depth * slot;
    b1 = bars + 1024;
    b2 = b1 + Hd * 4;
    total = b2 + E * 4;
  }
};

#ifdef __CUDACC__

template <int E>
__global__ void __launch_bounds__(kMlpThreads, 1) mlp_fused_sm90_kernel(const __grid_constant__ MlpParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int kx = E / 64;                       // k-blocks of the first GEMM
  constexpr int kTile = kConvBM * kConvBK * 2;     // 16 KB: 128 rows x 64 fp16
  constexpr int kW1 = kMlpHc * kConvBK * 2;        // fc1 weight tile: 64 hidden rows x 64 fp16
  constexpr int kW2 = E * kConvBK * 2;             // fc2 weight tile: E rows x 64 fp16
  constexpr int kSlot = kW1 > kW2 ? kW1 : kW2;
  const MlpSmem L(E, p.Hd, p.ring);
  uint8_t* sX = smem + L.x;
  uint8_t* sH = smem + L.h;
  uint8_t* sRing = smem + L.ring;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L.bars);
  uint64_t* empty_bar = full_bar + p.ring;
  uint64_t* x_full = empty_bar + p.ring;
  uint64_t* res_bar = x_full + 1;
  float* s_b1 = reinterpret_cast<float*>(smem + L.b1);
  float* s_b2 = reinterpret_cast<float*>(smem + L.b2);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunks = p.Hd / kMlpHc;
  int mt = (int)blockIdx.x;
  const int tw = mt % p.tiles_w; mt /= p.tiles_w;
  const int th = mt % p.tiles_h; mt /= p.tiles_h;
  const int w0 = tw * p.bw, h0 = th * p.bh, n0 = mt * p.bn;

  if (warp == kMlpTmaWarp && lane == 0) {
    tma_prefetch_desc(&p.tmX); tma_prefetch_desc(&p.tmW1); tma_prefetch_desc(&p.tmW2);
    tma_prefetch_desc(&p.tmOut); if (p.has_res) tma_prefetch_desc(&p.tmRes);
    for (int s = 0; s < p.ring; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConvEpiWarps); }
    mbar_init(x_full, 1); mbar_init(res_bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  pdl_trigger();
  pdl_wait();

  if (warp == kMlpTmaWarp) {
    // ===================== TMA producer: X once, then per chunk kx fc1 tiles and one fc2 tile =====================
    const bool el = elect_one();
    if (el) {
      mbar_arrive_expect_tx(x_full, (uint32_t)(kx * kTile));
      for (int kb = 0; kb < kx; ++kb) tma_load_4d(sX + (size_t)kb * kTile, &p.tmX, x_full, kb * kConvBK, w0, h0, n0);
    }
    int stage = 0; uint32_t phase = 0;
    auto next = [&]() { if (++stage == p.ring) { stage = 0; phase ^= 1; } };
    for (int j = 0; j < chunks; ++j) {
      for (int kb = 0; kb < kx; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (el) {
          mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)kW1);
          tma_load_2d(sRing + (size_t)stage * kSlot, &p.tmW1, &full_bar[stage], kb * kConvBK, j * kMlpHc);
        }
        next();
      }
      for (int t = 0; t < kMlpHc / kConvBK; ++t) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (el) {
          mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)kW2);
          tma_load_2d(sRing + (size_t)stage * kSlot, &p.tmW2, &full_bar[stage], j * kMlpHc + t * kConvBK, 0);
        }
        next();
      }
    }
    return;
  }

  // ===================== consumers (8 warps, warpgroup wg owns rows 64 wg .. 64 wg + 63) =====================
  const int wg = warp >> 2;
  const int rA = 64 * wg + 16 * (warp & 3) + (lane >> 2), rB = rA + 8;
  const int etid = threadIdx.x;
  constexpr int kCons = 32 * kConvEpiWarps;
  for (int i = etid; i < p.Hd; i += kCons) s_b1[i] = __ldg(p.bias1 + i);
  for (int i = etid; i < E; i += kCons) s_b2[i] = __ldg(p.bias2 + i);
  mbar_wait(x_full, 0);
  named_bar_sync(1, kCons);                                       // biases visible

  const uint32_t sX0 = smem_u32(sX), sH0 = smem_u32(sH), sR0 = smem_u32(sRing);
  int stage = 0; uint32_t phase = 0;
  auto release = [&](int s) { if (s >= 0 && lane == 0) mbar_arrive(&empty_bar[s]); };
  float acc2[E / 2];
#pragma unroll
  for (int i = 0; i < E / 2; ++i) acc2[i] = 0.f;
  for (int j = 0; j < chunks; ++j) {
    // ---- GEMM 1: acc1 = X . W1_j^T ----
    float acc1[kMlpHc / 2];
#pragma unroll
    for (int i = 0; i < kMlpHc / 2; ++i) acc1[i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < kx; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint64_t adesc = wgmma_desc_sw128(sX0 + (uint32_t)(kb * kTile + wg * (64 * 128)));
      const uint64_t bdesc = wgmma_desc_sw128(sR0 + (uint32_t)(stage * kSlot));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kConvBK / 16; ++k) Wgmma<kMlpHc>::mma(acc1, adesc + 2 * k, bdesc + 2 * k);
      wgmma_commit();
      wgmma_wait<1>();
      release(prev);
      prev = stage;
      if (++stage == p.ring) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc1);
    release(prev);
    // ---- H_j = GELU(acc1 + b1) -> fp16 rows of this warpgroup (GEMM 2 of chunk j - 1 has retired: H is free) ----
    const float* b1 = s_b1 + j * kMlpHc;
#pragma unroll
    for (int i = 0; i < kMlpHc / 8; ++i) {
      const int c = 8 * i + 2 * (lane & 3);
      const float2 bb = *reinterpret_cast<const float2*>(b1 + c);
      uint8_t* tile = sH + (size_t)(c >> 6) * kTile + 4 * (lane & 3);
      const int u = (c & 63) >> 3;
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int r = hr ? rB : rA;
        *reinterpret_cast<__half2*>(tile + r * 128 + ((u ^ (r & 7)) << 4)) =
            __floats2half2_rn(gelu_erf_f(acc1[4 * i + 2 * hr] + bb.x), gelu_erf_f(acc1[4 * i + 2 * hr + 1] + bb.y));
      }
    }
    fence_proxy_async_smem();                                     // H_j is read by the tensor core through the async proxy
    named_bar_sync(2 + wg, 128);                                  // the warpgroup's 64 rows of H_j are complete
    // ---- GEMM 2: acc2 += H_j . W2_j^T ----
    prev = -1;
    for (int t = 0; t < kMlpHc / kConvBK; ++t) {
      mbar_wait(&full_bar[stage], phase);
      const uint64_t adesc = wgmma_desc_sw128(sH0 + (uint32_t)(t * kTile + wg * (64 * 128)));
      const uint64_t bdesc = wgmma_desc_sw128(sR0 + (uint32_t)(stage * kSlot));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kConvBK / 16; ++k) Wgmma<E>::mma(acc2, adesc + 2 * k, bdesc + 2 * k);
      wgmma_commit();
      wgmma_wait<1>();
      release(prev);
      prev = stage;
      if (++stage == p.ring) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc2);
    release(prev);
  }

  // ---- epilogue: acc2 + b2 (+ residual) -> fp16 -> TMA store, GroupNorm partials ----
  named_bar_sync(1, kCons);                                       // X and H are dead: every MMA of both warpgroups retired
  uint8_t* sblk = sX;                                             // kx staging blocks of [128 rows x 64 columns]
  float* wsum = reinterpret_cast<float*>(sH);                     // [4 quads][E][2]
  if (p.has_res) {
    if (etid == 0) {
      mbar_arrive_expect_tx(res_bar, (uint32_t)(kx * kTile));
      for (int bq = 0; bq < kx; ++bq) tma_load_4d(sblk + (size_t)bq * kTile, &p.tmRes, res_bar, bq * 64, w0, h0, n0);
    }
    mbar_wait(res_bar, 0);
  }
#pragma unroll
  for (int i = 0; i < E / 8; ++i) {
    const int c = 8 * i + 2 * (lane & 3);
    const float2 bb = *reinterpret_cast<const float2*>(s_b2 + c);
    uint8_t* tile = sblk + (size_t)(c >> 6) * kTile + 4 * (lane & 3);
    const int u = (c & 63) >> 3;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int r = hr ? rB : rA;
      __half2* dst = reinterpret_cast<__half2*>(tile + r * 128 + ((u ^ (r & 7)) << 4));
      float f0 = acc2[4 * i + 2 * hr] + bb.x, f1 = acc2[4 * i + 2 * hr + 1] + bb.y;
      if (p.has_res) { const float2 x = __half22float2(*dst); f0 += x.x; f1 += x.y; }
      *dst = __floats2half2_rn(f0, f1);
    }
  }
  named_bar_sync(1, kCons);                                       // the staged tile is complete
  const bool want_stats = p.sink[0].part != nullptr;
  if (want_stats) {
    // statistics of the values as stored: warp (quad, column parity) reads back 32 rows x 16 columns (gn_stats.cuh)
    const int quad = warp & 3, cpar = warp >> 2;
    const int r = quad * 32 + lane;
    for (int c = cpar * 16; c < E; c += 32) {
      const uint8_t* brow = sblk + (size_t)(c >> 6) * kTile + r * 128;
      const int u0 = (c & 63) >> 3;
      const uint4 o0 = *reinterpret_cast<const uint4*>(brow + (((u0) ^ (r & 7)) << 4));
      const uint4 o1 = *reinterpret_cast<const uint4*>(brow + (((u0 + 1) ^ (r & 7)) << 4));
      warp_chunk_stats(o0, o1, lane, wsum + ((size_t)quad * E + c) * 2);
    }
  }
  fence_proxy_async_smem();
  named_bar_sync(1, kCons);
  if (etid == 0) {
    for (int bq = 0; bq < kx; ++bq) tma_store_4d(&p.tmOut, sblk + (size_t)bq * kTile, bq * 64, w0, h0, n0);
    tma_store_commit();
  }
  if (want_stats) {
    const int slot = th * p.tiles_w + tw;
    if (n0 < p.Nimg)
      write_quad_pairs(wsum, E, E, 0, p.bn, n0, p.Nimg, slot, p.gn_slots, p.sink[0], p.sink[1], etid, kCons);
    // (no plan gives an MLP sink group statistics; without this branch ptxas spills loop state of the <128> / <192>
    // instances in the main loop, so it stays)
    if (p.sink[0].gstat || p.sink[1].gstat) {
      int* s_flag = reinterpret_cast<int*>(wsum + 8 * E);
      const GnSink* const sk[4] = {&p.sink[0], &p.sink[0], p.sink[1].part ? &p.sink[1] : nullptr, p.sink[1].part ? &p.sink[1] : nullptr};
      const int n1 = (p.bn == 2 && n0 + 1 < p.Nimg) ? n0 + 1 : -1;
      const int im[4] = {n0 < p.Nimg ? n0 : -1, n0 < p.Nimg ? n1 : -1, n0 < p.Nimg ? n0 : -1, n0 < p.Nimg ? n1 : -1};
      const unsigned int ad[4] = {(unsigned)E, (unsigned)E, (unsigned)E, (unsigned)E};
      gn_arrive<4>(sk, im, ad, p.gn_slots, 128.0f / (float)p.bn, etid, kCons, 1, s_flag);
    }
  }
  if (etid == 0) tma_store_wait_read();
}

#endif
}  // namespace rs

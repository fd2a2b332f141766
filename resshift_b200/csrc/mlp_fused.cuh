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
// Warp 8 is the TMA producer: X once, then per chunk one slot with the E/64 fc1 weight tiles followed by one slot with
// the fc2 weight tile (both E x 128 bytes), through one ring of slots in the order the consumers use them.
//
// The two warpgroups take turns on the tensor core (ping-pong): a warpgroup issues GEMM 2 of chunk j - 1 and GEMM 1 of
// chunk j back to back, hands the turn to the other warpgroup, and runs GELU(j) while the other's MMAs execute.  A pair
// of named barriers passes the turn, so the GELU of one warpgroup overlaps the MMAs of the other instead of both
// warpgroups alternating GEMM and GELU in lockstep.  Each row's arithmetic is the same as in a lockstep loop: the same
// wgmma sequence builds acc1 per chunk, and acc2 adds the chunks in order.  The Swin block's norm2 runs in front of this
// kernel (gn_apply_kernel).
//
// On maps with few tiles (p.split > 1) a cluster of `split` CTAs shares one tile: CTA rank r loads the same X and runs
// the r-th contiguous range of Hd / 64 / split hidden chunks.  The ranks > 0 then leave their fp32 acc2 in their dead
// weight ring, and rank 0 adds them to its own through distributed shared memory in rank order (the same sum on every
// run) before the epilogue.  This fixes the fc2 summation order per launch shape: the split rule (mlp_finalize) reads
// only the shape and the SM count.
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
  int ring;                          // weight ring depth (slots of E x 128 bytes)
  int bw, bh, bn, tiles_w, tiles_h;
  int Wout, Hout, Nimg;
  int has_res;
  int split;                         // CTAs (one cluster) that share a tile's hidden chunks; 1: one CTA per tile
  GnSink sink[2]; int gn_slots;      // fused GroupNorm statistics of the output (gn_stats.cuh)
};

// shared-memory layout (offsets from the 1024-aligned base)
struct MlpSmem {
  int x, h, ring, bars, b1, b2, total;
  __host__ __device__ MlpSmem(int E, int Hd, int ring_depth) {
    const int slot = E * kConvBK * 2;               // E/64 fc1 tiles of [64 x 64], or one fc2 tile of [E x 64]
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
  constexpr int kSlot = kx * kW1;                  // a chunk's fc1 tiles, or its fc2 tile
  static_assert(kSlot == kW2 && kMlpHc == kConvBK, "one fc1 slot and one fc2 slot per hidden chunk");
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
  const int split = p.split;
  const int rank = (int)blockIdx.x % split;        // the cluster rank: clusters are `split` consecutive CTAs along x
  const int chunks = p.Hd / kMlpHc / split;        // this CTA's hidden chunks, j0 .. j0 + chunks - 1
  const int j0 = rank * chunks;
  int mt = (int)blockIdx.x / split;
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
    // ===================== TMA producer: X once, then per chunk one slot of kx fc1 tiles and one fc2 slot =============
    const bool el = elect_one();
    if (el) {
      mbar_arrive_expect_tx(x_full, (uint32_t)(kx * kTile));
      for (int kb = 0; kb < kx; ++kb) tma_load_4d(sX + (size_t)kb * kTile, &p.tmX, x_full, kb * kConvBK, w0, h0, n0);
    }
    int stage = 0; uint32_t phase = 0;
    auto next = [&]() { if (++stage == p.ring) { stage = 0; phase ^= 1; } };
    for (int j = j0; j < j0 + chunks; ++j) {
      mbar_wait(&empty_bar[stage], phase ^ 1);
      if (el) {
        mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)(kx * kW1));
        for (int kb = 0; kb < kx; ++kb)
          tma_load_2d(sRing + (size_t)stage * kSlot + (size_t)kb * kW1, &p.tmW1, &full_bar[stage], kb * kConvBK, j * kMlpHc);
      }
      next();
      mbar_wait(&empty_bar[stage], phase ^ 1);
      if (el) {
        mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)kW2);
        tma_load_2d(sRing + (size_t)stage * kSlot, &p.tmW2, &full_bar[stage], j * kMlpHc, 0);
      }
      next();
    }
    __syncwarp();
    if (split > 1) { cluster_sync_all(); cluster_sync_all(); }    // the two cluster barriers of the reduction below
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
  auto take = [&]() { mbar_wait(&full_bar[stage], phase); const int s = stage; if (++stage == p.ring) { stage = 0; phase ^= 1; } return s; };
  auto release = [&](int s) { if (s >= 0 && lane == 0) mbar_arrive(&empty_bar[s]); };
  // turn barriers: warpgroup wg waits on kTurn + wg for the other warpgroup to have issued its MMAs.  Warpgroup 0 opens
  // the first turn and warpgroup 1 takes the last, so every bar.sync has exactly one matching bar.arrive.
  constexpr int kTurn = 2;
  float acc2[E / 2];
#pragma unroll
  for (int i = 0; i < E / 2; ++i) acc2[i] = 0.f;
  // ---- GEMM 2 of chunk j: acc2 += H_j . W2_j^T ----
  auto gemm2 = [&]() {
    const int s = take();
    const uint64_t adesc = wgmma_desc_sw128(sH0 + (uint32_t)(wg * (64 * 128)));
    const uint64_t bdesc = wgmma_desc_sw128(sR0 + (uint32_t)(s * kSlot));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kConvBK / 16; ++k) Wgmma<E>::mma(acc2, adesc + 2 * k, bdesc + 2 * k);
    wgmma_commit();
    return s;
  };
  for (int j = 0; j < chunks; ++j) {
    float acc1[kMlpHc / 2];
#pragma unroll
    for (int i = 0; i < kMlpHc / 2; ++i) acc1[i] = 0.f;
    // The turn's bar.sync also covers all 128 threads of this warpgroup: their H_{j-1} stores (and the proxy fence each
    // thread made after them) are ordered before GEMM 2 reads H.
    if (wg == 1 || j > 0) named_bar_sync(kTurn + wg, 256);
    const int s2 = j > 0 ? gemm2() : -1;
    // ---- GEMM 1: acc1 = X . W1_j^T ----
    const int s1 = take();
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < kx; ++kb) {
      const uint64_t adesc = wgmma_desc_sw128(sX0 + (uint32_t)(kb * kTile + wg * (64 * 128)));
      const uint64_t bdesc = wgmma_desc_sw128(sR0 + (uint32_t)(s1 * kSlot + kb * kW1));
#pragma unroll
      for (int k = 0; k < kConvBK / 16; ++k) Wgmma<kMlpHc>::mma(acc1, adesc + 2 * k, bdesc + 2 * k);
    }
    wgmma_commit();
    named_bar_arrive(kTurn + 1 - wg, 256);
    wgmma_wait<0>();
    wgmma_fence_regs(acc1);
    wgmma_fence_regs(acc2);
    release(s2);
    release(s1);
    // ---- H_j = GELU(acc1 + b1) -> fp16 rows of this warpgroup (GEMM 2 of chunk j - 1 has retired: H is free) ----
    const float* b1 = s_b1 + (j0 + j) * kMlpHc;
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
  }
  named_bar_sync(kTurn + wg, 256);
  const int s2 = gemm2();
  if (wg == 0) named_bar_arrive(kTurn + 1, 256);
  wgmma_wait<0>();
  wgmma_fence_regs(acc2);
  release(s2);

  named_bar_sync(1, kCons);                                       // X, H and the ring are dead: every MMA retired
  if (split > 1) {
    // ---- cluster: rank 0 adds the partial acc2 of ranks 1 .. split - 1, in rank order ----
    // [E/4][kCons] float2: each thread's partial, read back by the same thread index of rank 0 (mlp_finalize checks
    // that the ring holds 128 x E floats)
    const uint32_t red = sR0 + (uint32_t)etid * 8u;
    if (rank != 0) {
      float2* mine = reinterpret_cast<float2*>(sRing) + etid;
#pragma unroll
      for (int i = 0; i < E / 4; ++i) mine[i * kCons] = make_float2(acc2[2 * i], acc2[2 * i + 1]);
    }
    cluster_sync_all();                                           // the partials are visible across the cluster
    if (rank == 0) {
      for (int r = 1; r < split; ++r) {
        const uint32_t base = mapa_u32(red, (uint32_t)r);
#pragma unroll
        for (int i = 0; i < E / 4; ++i) {
          const float2 v = ld_dsmem_f32x2(base + (uint32_t)(i * kCons * 8));
          acc2[2 * i] += v.x;
          acc2[2 * i + 1] += v.y;
        }
      }
    }
    cluster_sync_all();                                           // rank 0 has read them: the other CTAs may exit
    if (rank != 0) return;
  }

  // ---- epilogue: acc2 + b2 (+ residual) -> fp16 -> TMA store, GroupNorm partials ----
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

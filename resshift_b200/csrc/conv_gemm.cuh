// Implicit-GEMM convolution / linear layer on the sm_90a tensor cores (wgmma + TMA + mbarrier pipeline).
//
//   D[M = N*H*W pixels, Cout] = sum over taps, channels  A[pixel + tap offset, c] * Wt[cout, tap, c]
//
// * activations are NHWC fp16 *views* (channel count C, row stride ld >= C): a 4-D TMA tensor map
//   {C, W, H, N} per source.  One CTA computes a 128-pixel x BN-channel output tile; the 128 pixels
//   are a (bw x bh x bn) box in (W, H, N), so the tile of a 3x3 tap is the same box shifted by
//   (dw, dh) — TMA's out-of-bounds zero fill implements the conv padding, and the box lands in
//   shared memory exactly as the K-major, 128-byte-swizzled operand wgmma expects.
// * stride-2 convs read the four (row, column)-parity sub-grids of the input through four strided
//   tensor maps over the same buffer (no copy); each tap names its map.
// * weights are [Cout][tap][Cin_pad] fp16 (K-major), one 2-D tensor map.
// * warp roles: warps 0..7 = two consumer warpgroups (warpgroup g issues the wgmma of rows 64g..64g+63 of every
//   128-pixel sub-tile, accumulates in registers and runs the epilogue of those rows), warp 8 = TMA producer.
// * covers reference call sites: every nn.Conv2d / nn.Linear inside UNetModelSwin.forward
//   (reference models/unet.py:147,173,184,707,862,69,99-101; models/swin_transformer.py:22-24,105-107,480,515).
#pragma once

#include "common.cuh"
#include "gn_stats.cuh"
#include "wgmma.cuh"

namespace rs {

constexpr int kConvBM = 128;      // pixels per tile (two warpgroups x wgmma M = 64)
constexpr int kConvBK = 64;       // channels per k-block (128 B rows, SWIZZLE_128B)
constexpr int kConvEpiWarps = 8;  // the two consumer warpgroups
constexpr int kConvThreads = 32 * kConvEpiWarps + 32;
constexpr int kConvTmaWarp = kConvEpiWarps;        // warp 8
constexpr int kMaxTaps = 9;
constexpr int kMaxSrc = 4;
// channel-tile widths with a compiled kernel (wgmma takes N as an immediate; scripts/gen_wgmma.py writes the wrappers)
constexpr int kConvBNs[] = {16, 32, 48, 64, 80, 96, 128, 160, 192, 256};
constexpr bool conv_bn_supported(int bn) {
  for (int v : kConvBNs) if (v == bn) return true;
  return false;
}

enum ConvAct : int { ACT_NONE = 0, ACT_GELU = 1, ACT_SILU = 2 };

struct ConvParams {
  CUtensorMap tmA[kMaxSrc];
  CUtensorMap tmB;
  int num_taps;
  int tap_src[kMaxTaps];
  int tap_dh[kMaxTaps];
  int tap_dw[kMaxTaps];
  int kchunks;           // ceil(Cin / 64); the channels of a partial last chunk beyond Cin arrive zero-filled from TMA
  int w_tap_stride;      // K offset between consecutive taps in the weight matrix (= Cin_pad)
  int bw, bh, bn;        // pixel box of a tile, bw*bh*bn == 128
  int tiles_w, tiles_h, tiles_n;
  int Wout, Hout, Nimg;
  int BN, n_tiles, Cout;
  int stages;
  int epi_off;           // byte offset of the epilogue staging area (0: it reuses the operand ring once the MMAs are done)
  int bar_off;           // byte offset of the barriers (the bias tile follows 256 B later)
  int cg;                // 1: one CTA per tile;  2: CTA pair (cluster of 2) on two neighbouring 128-pixel tiles that share
                         //    every weight tile: each CTA loads half of it and multicasts that half to both
  int splitk;            // > 1: the K loop is cut into `splitk` ranges, one CTA (or pair) each; the epilogue then only
                         //      stores fp32 partial accumulators to `partial` and splitk_reduce_kernel finishes the layer
  float* partial;        // [splitk][Nimg*Hout*Wout pixels][Cout] fp32
  int msub;              // 128-pixel sub-tiles per CTA (1 or 2): two sub-tiles share every weight tile (fewer operand bytes per MMA)
  // epilogue
  const float* bias;                 // [Cout] fp32 or nullptr; with bias_sN > 0 one row per image
  int bias_sN;                       // elements between the bias rows of consecutive images (0: one row for all)
  const __half* residual;           // optional, same pixel grid as the output
  long long res_sN, res_sH, res_sW;  // strides in elements
  __half* out;                       // NHWC fp16 view (may be nullptr when out_f32 is set)
  long long out_sN, out_sH, out_sW;
  float* out_f32_nchw;               // optional fp32 NCHW output [Nimg, Cout, Hout, Wout]
  int act;
  unsigned long long* dbg;           // optional per-CTA timeline (8 x u64 per CTA, globaltimer ns), profiling aid
  // staged epilogue: results go to shared memory (128B-swizzled 64-column blocks) and leave through TMA stores;
  // the residual tile arrives the same way through a TMA load
  CUtensorMap tmOut, tmRes;
  int tma_out;                       // 1: staged epilogue (fp16 NHWC output); 0: direct per-thread stores
  int tma_res;
  int epi_bc;                        // staging block width in columns: 64 / 32 / 16 (swizzle 128B / 64B / 32B),
                                     // the largest that divides BN so a block never spills into the next channel tile
  // fused GroupNorm statistics of the OUTPUT for up to two consumers (gn_stats.cuh): per image / 128-pixel tile slot /
  // channel the pair (mean, M2) of the stored fp16 values
  GnSink sink[2];
  int gn_slots;
  // persistent mode: CTAs (pairs) walk work units u = worker, worker + #workers, ...; the producer loads the next
  // unit's operands while the consumers run the epilogue of the current one (staging area outside the ring)
  int persist;
  int num_units;         // (pixel tiles or tile pairs) x channel tiles
  // second, activated output (ResBlockConv reads every block output raw and through SiLU): silu_out = SiLU(v) of the
  // fp16 value v stored to `out`, an NHWC fp16 view of its own (staged epilogue: through tmSilu from the same tile).
  // Only the EX instances of the wgmma kernel (and the SIMT / split-K kernels) read silu_out and film.
  __half* silu_out;
  long long silu_sN, silu_sH, silu_sW;
  CUtensorMap tmSilu;
  // FiLM after the activation (ResBlockConv with scale-shift norm): v = fp16(act(acc + bias)), stored as
  // fp16(v * (1 + film[n][c]) + film[n][Cout + c]) (the reference's autocast forward rounds there too); rows film_sN apart
  // (0: one row for all images); no residual, one sub-tile.  Applied after the accumulators are dead.
  const float* film;
  int film_sN;
};

#ifdef __CUDACC__

// Every (BN, MS) instance has the same structure; BN and the sub-tile count are template parameters because the
// accumulators live in registers (BN / 2 floats per thread and sub-tile).  EX instances (one sub-tile) also have the
// epilogue's FiLM and SiLU-output passes; the others compile without them, so the convs that use neither run the same code.
template <int BN, int MS, bool EX = false>
__global__ void __launch_bounds__(kConvThreads, (BN * MS <= 128) ? 2 : 1) conv_gemm_sm90_kernel(const __grid_constant__ ConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [stages][MS x A 16 KB | B BN*128 B] (+ staging area when persistent), then barriers, then the bias tile
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int a_bytes = kConvBM * kConvBK * 2;             // one sub-tile of A
  constexpr int b_bytes = BN * kConvBK * 2;
  constexpr int stage_bytes = MS * a_bytes + b_bytes;
  constexpr int kAcc = BN / 2;                               // accumulator registers per thread and sub-tile
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + p.bar_off);
  uint64_t* empty_bar = full_bar + p.stages;
  uint64_t* res_bar = empty_bar + p.stages;
  float* s_bias = reinterpret_cast<float*>(smem + p.bar_off + 256);   // [BN] bias of the current channel tile
  uint8_t* sepi = smem + p.epi_off;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  unsigned long long* dbg = p.dbg ? p.dbg + (size_t)blockIdx.x * 8 : nullptr;
  if (dbg && threadIdx.x == 0) {
    uint32_t smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    dbg[0] = global_timer_ns(); dbg[7] = smid;
  }

  // pair mode: the cluster is one CTA pair, cluster rank = rank inside the pair
  const int cg = p.cg;
  const uint32_t crank = cg == 2 ? cluster_ctarank() : 0;
  const uint32_t rank = crank & 1;
  const uint32_t peer = crank ^ 1u;
  const uint16_t pair_mask = (uint16_t)(3u << (crank & ~1u));    // multicast mask of this pair
  int unit0 = cg == 2 ? (blockIdx.x >> 1) : blockIdx.x;         // work unit: a CTA, or a CTA pair
  const int split = unit0 % p.splitk;                            // which K range (fastest index: splits of a tile run together)
  unit0 /= p.splitk;
  const int unit_step = p.persist ? (int)gridDim.x / cg : 1;
  const int unit_end = p.persist ? p.num_units : unit0 + 1;
  const int total_kb = p.num_taps * p.kchunks;
  const int kb_begin = (int)((long long)total_kb * split / p.splitk);
  const int kb_end = (int)((long long)total_kb * (split + 1) / p.splitk);
  const int num_kb = kb_end - kb_begin;
  auto tile_origin = [&](int mt, int& tw_, int& th_, int& w0_, int& h0_, int& n0_) {
    tw_ = mt % p.tiles_w; mt /= p.tiles_w;
    th_ = mt % p.tiles_h; mt /= p.tiles_h;
    w0_ = tw_ * p.bw; h0_ = th_ * p.bh; n0_ = mt * p.bn;
  };
  // first 128-pixel tile of a unit (sub-tiles follow) and its channel tile
  auto unit_tiles = [&](int unit, int& n_tile_, int& mt0_) {
    n_tile_ = unit % p.n_tiles;
    mt0_ = cg == 2 ? (unit / p.n_tiles) * 2 + (int)rank : (unit / p.n_tiles) * MS;
  };

  if (warp == kConvTmaWarp && lane == 0) {
    for (int s = 0; s < kMaxSrc; ++s) tma_prefetch_desc(&p.tmA[s]);
    tma_prefetch_desc(&p.tmB);
    if (p.tma_out) tma_prefetch_desc(&p.tmOut);
    if (p.tma_res) tma_prefetch_desc(&p.tmRes);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConvEpiWarps * cg);      // every consumer warp of every CTA that reads the slot's weights
    }
    mbar_init(res_bar, 1);
    mbar_fence_init();
  }
  if (cg == 2) cluster_sync_all(); else __syncthreads();     // peer barriers must be initialised before remote arrivals
  // everything above (barrier init, descriptor prefetch) overlaps the previous kernel's tail
  pdl_trigger();
  pdl_wait();
  if (dbg && threadIdx.x == 0) dbg[1] = global_timer_ns();

  if (warp == kConvTmaWarp) {
    // ===================== TMA producer =====================
    // (warp-uniform loop, only the asynchronous instructions are issued by one elected lane)
    const bool el = elect_one();
    int stage = 0;
    uint32_t phase = 0;
    for (int unit = unit0; unit < unit_end; unit += unit_step) {
      int n_tile, mt0;
      unit_tiles(unit, n_tile, mt0);
      int tws[MS], ths[MS], w0s[MS], h0s[MS], n0s[MS];
#pragma unroll
      for (int sub = 0; sub < MS; ++sub) tile_origin(mt0 + sub, tws[sub], ths[sub], w0s[sub], h0s[sub], n0s[sub]);
      int tap = kb_begin / p.kchunks;
      int kc = kb_begin - tap * p.kchunks;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + (size_t)stage * stage_bytes;
        uint8_t* sb = sa + MS * a_bytes;
        const CUtensorMap* ma = &p.tmA[p.tap_src[tap]];
        const int dw = p.tap_dw[tap], dh = p.tap_dh[tap];
        const int kcol = kc * kConvBK, wcol = tap * p.w_tap_stride + kc * kConvBK;
        if (el) {
          mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)stage_bytes);
#pragma unroll
          for (int sub = 0; sub < MS; ++sub)
            tma_load_4d(sa + sub * a_bytes, ma, &full_bar[stage], kcol, w0s[sub] + dw, h0s[sub] + dh, n0s[sub]);
          if (cg == 2)   // this CTA's half of the weight tile, to both CTAs of the pair
            tma_load_2d_mc(sb + rank * (b_bytes / 2), &p.tmB, &full_bar[stage], wcol, n_tile * BN + (int)rank * (BN / 2), pair_mask);
          else
            tma_load_2d(sb, &p.tmB, &full_bar[stage], wcol, n_tile * BN);
        }
        if (++kc == p.kchunks) { kc = 0; ++tap; }
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ===================== consumers: wgmma main loop + epilogue (8 warps) =====================
    const int wg = warp >> 2;                        // warpgroup: rows 64 wg .. 64 wg + 63 of every sub-tile
    const int rA = 64 * wg + 16 * (warp & 3) + (lane >> 2);   // the two rows of this thread's accumulator fragments
    const int rB = rA + 8;
    const int etid = threadIdx.x;                    // 0..255 among consumer threads
    const uint32_t smem0 = smem_u32(smem);
    int stage = 0;
    uint32_t phase = 0;
    int iter = 0;
    for (int unit = unit0; unit < unit_end; unit += unit_step, ++iter) {
      int n_tile, mt0;
      unit_tiles(unit, n_tile, mt0);
      const int col0 = n_tile * BN;
      float acc[MS][kAcc];
#pragma unroll
      for (int sub = 0; sub < MS; ++sub)
#pragma unroll
        for (int i = 0; i < kAcc; ++i) acc[sub][i] = 0.f;
      int prev_stage = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        if (dbg && etid == 0 && kb == 0) dbg[2] = global_timer_ns();
        const uint32_t sa = smem0 + (uint32_t)stage * (uint32_t)stage_bytes;
        const uint64_t bdesc = wgmma_desc_sw128(sa + MS * a_bytes);
        wgmma_fence();
#pragma unroll
        for (int sub = 0; sub < MS; ++sub) {
          const uint64_t adesc = wgmma_desc_sw128(sa + sub * a_bytes + wg * (64 * 128));
#pragma unroll
          for (int k = 0; k < kConvBK / 16; ++k) Wgmma<BN>::mma(acc[sub], adesc + 2 * k, bdesc + 2 * k);
        }
        wgmma_commit();
        // the previous k-block's MMAs have retired: its slot may be refilled (in pair mode the slot's weights were also
        // written by the peer, which must hear from this CTA's consumers too)
        wgmma_wait<1>();
        if (prev_stage >= 0 && lane == 0) {
          mbar_arrive(&empty_bar[prev_stage]);
          if (cg == 2) mbar_arrive_remote(mapa_u32(smem_u32(&empty_bar[prev_stage]), peer));
        }
        prev_stage = stage;
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int sub = 0; sub < MS; ++sub) wgmma_fence_regs(acc[sub]);
      if (prev_stage >= 0 && lane == 0) {
        mbar_arrive(&empty_bar[prev_stage]);
        if (cg == 2) mbar_arrive_remote(mapa_u32(smem_u32(&empty_bar[prev_stage]), peer));
      }
      if (dbg && etid == 0) dbg[4] = global_timer_ns();
      // every MMA of both warpgroups has retired (the ring may be reused as staging), and the previous unit's epilogue is
      // complete (its staged tile has been read by the TMA store)
      named_bar_sync(1, 32 * kConvEpiWarps);

      if (p.splitk > 1) {
        // ---------- split-K: raw fp32 partial sums, finished by splitk_reduce_kernel ----------
        int tw, th, w0, h0, n0;
        tile_origin(mt0, tw, th, w0, h0, n0);
        const long long npix = (long long)p.Nimg * p.Hout * p.Wout;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int r = hr ? rB : rA;
          const int w = w0 + r % p.bw, h = h0 + (r / p.bw) % p.bh, n = n0 + r / (p.bw * p.bh);
          if (w >= p.Wout || h >= p.Hout || n >= p.Nimg) continue;
          const long long pix = ((long long)n * p.Hout + h) * p.Wout + w;
          float* prow = p.partial + ((long long)split * npix + pix) * p.Cout;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int col = col0 + 8 * j + 2 * (lane & 3);
            if (col < p.Cout) *reinterpret_cast<float2*>(prow + col) = make_float2(acc[0][4 * j + 2 * hr], acc[0][4 * j + 2 * hr + 1]);
          }
        }
      } else if (p.tma_out) {
        // ---------- staged epilogue ----------
        // Per sub-tile: BN/bc blocks of [128 rows x bc columns] fp16, swizzled like the TMA box — first the residual
        // tile lands there (TMA load), then the finished outputs are written in place, then one TMA store per block.
        // After the blocks of all sub-tiles: per-warp GroupNorm partials [MS][4 quads][BN][2].
        const int bc = p.epi_bc;                       // columns per staging block
        const int nblk = BN / bc;
        const int blk_bytes = kConvBM * bc * 2;
        const int sub_bytes = nblk * blk_bytes;
        const int bshift = (bc == 64) ? 6 : (bc == 32 ? 5 : 4);
        // Swizzle<B,4,3>: the 16-byte unit index is XORed with address bits [7, 7+B); row pitch is 2*bc bytes
        auto swz_of = [&](int r) { return (bc == 64) ? (r & 7) : (bc == 32 ? ((r >> 1) & 3) : ((r >> 2) & 1)); };
        float* wsum_all = reinterpret_cast<float*>(sepi + (size_t)MS * sub_bytes);
        // per-image bias (one sub-tile per CTA only: conv_finalize never pairs it with msub = 2): s_bias holds [bn][BN],
        // one row per image of the tile; with tiles of at most 8 images, rows rA and rB = rA + 8 share an image
        const bool bias_rows = MS == 1 && p.bias_sN != 0;
        if (!bias_rows) {
          for (int i = etid; i < BN; i += 32 * kConvEpiWarps)
            s_bias[i] = (p.bias && col0 + i < p.Cout) ? __ldg(p.bias + col0 + i) : 0.f;
        } else {
          const int nb = mt0 / (p.tiles_w * p.tiles_h) * p.bn;     // first image of the tile
          for (int il = 0; il < p.bn; ++il) {
            const int n = nb + il;
            for (int c = etid; c < BN; c += 32 * kConvEpiWarps)
              s_bias[il * BN + c] = (col0 + c < p.Cout && n < p.Nimg) ? __ldg(p.bias + n * p.bias_sN + col0 + c) : 0.f;
          }
        }
        const float* s_bias_row = s_bias + (bias_rows ? (rA / (p.bw * p.bh)) * BN : 0);
        if (p.tma_res && etid == 0) {
          mbar_arrive_expect_tx(res_bar, (uint32_t)(MS * sub_bytes));
          for (int sub = 0; sub < MS; ++sub) {
            int tw, th, w0, h0, n0;
            tile_origin(mt0 + sub, tw, th, w0, h0, n0);
            for (int b = 0; b < nblk; ++b)
              tma_load_4d(sepi + (size_t)sub * sub_bytes + (size_t)b * blk_bytes, &p.tmRes, res_bar, col0 + b * bc, w0, h0, n0);
          }
        }
        named_bar_sync(1, 32 * kConvEpiWarps);         // bias tile visible
        if (p.tma_res) mbar_wait(res_bar, (uint32_t)(iter & 1));
        const int swA = swz_of(rA), swB = swz_of(rB);
#pragma unroll
        for (int sub = 0; sub < MS; ++sub) {
          uint8_t* sblk = sepi + (size_t)sub * sub_bytes;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int c = 8 * j + 2 * (lane & 3);
            const float2 b2 = *reinterpret_cast<const float2*>(s_bias_row + c);
            uint8_t* blk = sblk + (size_t)(c >> bshift) * blk_bytes + 4 * (lane & 3);
            const int u = (c & (bc - 1)) >> 3;         // 16-byte unit of columns 8j..8j+7 inside the block
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
              const int r = hr ? rB : rA;
              __half2* dst = reinterpret_cast<__half2*>(blk + r * (2 * bc) + ((u ^ (hr ? swB : swA)) << 4));
              float f0 = acc[sub][4 * j + 2 * hr] + b2.x, f1 = acc[sub][4 * j + 2 * hr + 1] + b2.y;
              if (p.act == ACT_GELU) { f0 = gelu_erf_f(f0); f1 = gelu_erf_f(f1); }
              else if (p.act == ACT_SILU) { f0 = silu_f(f0); f1 = silu_f(f1); }
              if (p.tma_res) { const float2 x = __half22float2(*dst); f0 += x.x; f1 += x.y; }
              *dst = __floats2half2_rn(f0, f1);
            }
          }
        }
        named_bar_sync(1, 32 * kConvEpiWarps);         // the staged tile is complete
        if (EX && MS == 1 && p.film) {
          // FiLM on the staged fp16 values, in place once the accumulators are dead (conv_finalize: no residual, one
          // sub-tile); every 16-byte unit reads its image's scale and shift rows
          const int nb = mt0 / (p.tiles_w * p.tiles_h) * p.bn;     // first image of the tile
          const int upr = bc / 8;                                  // 16-byte units per row of a block
          for (int i = etid; i < nblk * kConvBM * upr; i += 32 * kConvEpiWarps) {
            const int b = i / (kConvBM * upr), r = (i / upr) % kConvBM, up = i % upr;
            const int c = col0 + b * bc + ((up ^ swz_of(r)) << 3), n = nb + r / (p.bw * p.bh);
            if (c >= p.Cout || n >= p.Nimg) continue;                // (columns / images the stores clip)
            uint4* unit = reinterpret_cast<uint4*>(sepi + (size_t)b * blk_bytes + r * (2 * bc) + (up << 4));
            const float* row = p.film + (long long)n * p.film_sN + c;
            uint4 v = *unit;
            __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float2 f = __half22float2(h[k]);
              h[k] = __floats2half2_rn(fmaf(f.x, 1.f + __ldg(row + 2 * k), __ldg(row + p.Cout + 2 * k)),
                                       fmaf(f.y, 1.f + __ldg(row + 2 * k + 1), __ldg(row + p.Cout + 2 * k + 1)));
            }
            *unit = v;
          }
          named_bar_sync(1, 32 * kConvEpiWarps);
        }
        const bool want_stats = p.sink[0].part != nullptr;
        if (want_stats) {
          // statistics of the values as stored (gn_stats.cuh): warp (quad, column parity) reads back 32 rows x 16 columns
          const int quad = warp & 3, cpar = warp >> 2;
          const int r = quad * 32 + lane, swz = swz_of(r);
          for (int sub = 0; sub < MS; ++sub) {
            const uint8_t* sblk = sepi + (size_t)sub * sub_bytes;
            for (int c = cpar * 16; c < BN; c += 32) {
              const uint8_t* brow = sblk + (size_t)(c >> bshift) * blk_bytes + r * (2 * bc);
              const int u0 = (c & (bc - 1)) >> 3;
              const uint4 o0 = *reinterpret_cast<const uint4*>(brow + (((u0) ^ swz) << 4));
              const uint4 o1 = *reinterpret_cast<const uint4*>(brow + (((u0 + 1) ^ swz) << 4));
              warp_chunk_stats(o0, o1, lane, wsum_all + ((size_t)(sub * 4 + quad) * BN + c) * 2);
            }
          }
        }
        fence_proxy_async_smem();
        named_bar_sync(1, 32 * kConvEpiWarps);
        if (dbg && etid == 0) dbg[6] = global_timer_ns();
        if (etid == 0) {
          for (int sub = 0; sub < MS; ++sub) {
            int tw, th, w0, h0, n0;
            tile_origin(mt0 + sub, tw, th, w0, h0, n0);
            for (int b = 0; b < nblk; ++b)
              if (col0 + b * bc < p.Cout)
                tma_store_4d(&p.tmOut, sepi + (size_t)sub * sub_bytes + (size_t)b * blk_bytes, col0 + b * bc, w0, h0, n0);
          }
          tma_store_commit();
        }
        if (want_stats) {
          for (int sub = 0; sub < MS; ++sub) {
            int tw, th, w0, h0, n0;
            tile_origin(mt0 + sub, tw, th, w0, h0, n0);
            const int ncols = min(BN, p.Cout - col0);
            const int slot = th * p.tiles_w + tw;
            if (n0 < p.Nimg)                                           // (else: padding tile of an odd pair)
              write_quad_pairs(wsum_all + (size_t)sub * 8 * BN, BN, ncols, col0, p.bn, n0, p.Nimg, slot, p.gn_slots, p.sink[0], p.sink[1],
                               etid, 32 * kConvEpiWarps);
          }
        }
        if (EX && p.silu_out) {
          // the second output from the same staged tile: once the store above has read it, SiLU of every stored fp16
          // value in place (the staging layout is elementwise), then the same boxes through tmSilu
          if (etid == 0) tma_store_wait_read();
          named_bar_sync(1, 32 * kConvEpiWarps);
          uint4* sv = reinterpret_cast<uint4*>(sepi);
          for (int i = etid; i < MS * sub_bytes / 16; i += 32 * kConvEpiWarps) {
            uint4 v = sv[i];
            __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float2 f = __half22float2(h[k]);
              h[k] = __floats2half2_rn(silu_f(f.x), silu_f(f.y));
            }
            sv[i] = v;
          }
          fence_proxy_async_smem();
          named_bar_sync(1, 32 * kConvEpiWarps);
          if (etid == 0) {
            for (int sub = 0; sub < MS; ++sub) {
              int tw, th, w0, h0, n0;
              tile_origin(mt0 + sub, tw, th, w0, h0, n0);
              for (int b = 0; b < nblk; ++b)
                if (col0 + b * bc < p.Cout)
                  tma_store_4d(&p.tmSilu, sepi + (size_t)sub * sub_bytes + (size_t)b * blk_bytes, col0 + b * bc, w0, h0, n0);
            }
            tma_store_commit();
          }
        }
        if (etid == 0) tma_store_wait_read();
      } else {
        // ---------- direct epilogue (fp32 NCHW model head, or RS_CONV_EPI=direct) ----------
#pragma unroll
        for (int sub = 0; sub < MS; ++sub) {
          int tw, th, w0, h0, n0;
          tile_origin(mt0 + sub, tw, th, w0, h0, n0);
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int r = hr ? rB : rA;
            const int w = w0 + r % p.bw, h = h0 + (r / p.bw) % p.bh, n = n0 + r / (p.bw * p.bh);
            if (w >= p.Wout || h >= p.Hout || n >= p.Nimg) continue;
            __half* orow = p.out ? p.out + n * p.out_sN + h * p.out_sH + w * p.out_sW : nullptr;
            const __half* rrow = p.residual ? p.residual + n * p.res_sN + h * p.res_sH + w * p.res_sW : nullptr;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int col = col0 + 8 * j + 2 * (lane & 3) + e;
                if (col >= p.Cout) continue;
                float f = acc[sub][4 * j + 2 * hr + e];
                if (p.bias) f += __ldg(p.bias + n * p.bias_sN + col);
                if (p.act == ACT_GELU) f = gelu_erf_f(f);
                else if (p.act == ACT_SILU) f = silu_f(f);
                if (rrow) f += __half2float(rrow[col]);
                if (p.out_f32_nchw) p.out_f32_nchw[(((long long)n * p.Cout + col) * p.Hout + h) * p.Wout + w] = f;
                if (orow) orow[col] = __float2half_rn(f);
              }
            }
          }
        }
      }
    }
  }

  if (dbg && threadIdx.x == 0) dbg[5] = global_timer_ns();
  // pair: neither CTA may retire while the other can still arrive on its barriers or read its shared memory
  if (cg == 2) cluster_sync_all();
}

// kernel instance of a (channel-tile width, sub-tiles per CTA) configuration, nullptr if none is compiled
using ConvKernelFn = void (*)(const ConvParams);
template <int BN>
inline ConvKernelFn conv_kernel_ms(int msub, bool ex) {
  if (ex) return msub == 1 ? conv_gemm_sm90_kernel<BN, 1, true> : nullptr;
  if (msub == 1) return conv_gemm_sm90_kernel<BN, 1>;
  if constexpr (BN <= 128) { if (msub == 2) return conv_gemm_sm90_kernel<BN, 2>; }
  return nullptr;
}
// ex: the conv writes a SiLU output or applies FiLM rows (one sub-tile only)
inline ConvKernelFn conv_kernel_for(int bn, int msub, bool ex = false) {
  switch (bn) {
    case 16: return conv_kernel_ms<16>(msub, ex);
    case 32: return conv_kernel_ms<32>(msub, ex);
    case 48: return conv_kernel_ms<48>(msub, ex);
    case 64: return conv_kernel_ms<64>(msub, ex);
    case 80: return conv_kernel_ms<80>(msub, ex);
    case 96: return conv_kernel_ms<96>(msub, ex);
    case 128: return conv_kernel_ms<128>(msub, ex);
    case 160: return conv_kernel_ms<160>(msub, ex);
    case 192: return conv_kernel_ms<192>(msub, ex);
    case 256: return conv_kernel_ms<256>(msub, ex);
    default: return nullptr;
  }
}

// ------------------------------------------------------------------------------------------------
// Plain SIMT implementation of the same operator (debug / cross-check path, selected with
// RS_CONV_IMPL=simt).  Same ConvParams epilogue fields; sources passed as raw views.
// ------------------------------------------------------------------------------------------------
struct ConvSimtSrc {
  const __half* ptr[kMaxSrc];
  long long sN[kMaxSrc], sH[kMaxSrc], sW[kMaxSrc];
  int H[kMaxSrc], W[kMaxSrc];
  int C;
  const __half* wt;     // [Cout][taps][w_tap_stride]
};

__global__ void conv_simt_kernel(const __grid_constant__ ConvParams p, const __grid_constant__ ConvSimtSrc s) {
  pdl_trigger();
  pdl_wait();
  // one warp per output pixel, lanes stride over output channels
  const long long pix = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const long long npix = (long long)p.Nimg * p.Hout * p.Wout;
  if (pix >= npix) return;
  const int w = (int)(pix % p.Wout);
  const int h = (int)((pix / p.Wout) % p.Hout);
  const int n = (int)(pix / ((long long)p.Wout * p.Hout));
  const int ktot = p.num_taps * p.w_tap_stride;
  for (int co = lane; co < p.Cout; co += 32) {
    float acc = 0.f;
    for (int t = 0; t < p.num_taps; ++t) {
      const int src = p.tap_src[t];
      const int hh = h + p.tap_dh[t], ww = w + p.tap_dw[t];
      if (hh < 0 || ww < 0 || hh >= s.H[src] || ww >= s.W[src]) continue;
      const __half* a = s.ptr[src] + n * s.sN[src] + hh * s.sH[src] + ww * s.sW[src];
      const __half* wr = s.wt + (long long)co * ktot + t * p.w_tap_stride;
      for (int c = 0; c < s.C; c += 2) {
        const float2 av = __half22float2(*reinterpret_cast<const __half2*>(a + c));
        const float2 wv = __half22float2(*reinterpret_cast<const __half2*>(wr + c));
        acc = fmaf(av.x, wv.x, acc);
        acc = fmaf(av.y, wv.y, acc);
      }
    }
    if (p.bias) acc += p.bias[n * p.bias_sN + co];
    if (p.act == ACT_GELU) acc = gelu_erf_f(acc);
    else if (p.act == ACT_SILU) acc = silu_f(acc);
    if (p.residual) acc += __half2float(p.residual[n * p.res_sN + h * p.res_sH + w * p.res_sW + co]);
    if (p.out_f32_nchw) p.out_f32_nchw[(((long long)n * p.Cout + co) * p.Hout + h) * p.Wout + w] = acc;
    __half v = __float2half_rn(acc);
    if (p.film)      // on the fp16 value, as the wgmma kernel's epilogues do
      v = __float2half_rn(fmaf(__half2float(v), 1.f + p.film[(long long)n * p.film_sN + co], p.film[(long long)n * p.film_sN + p.Cout + co]));
    if (p.out) p.out[n * p.out_sN + h * p.out_sH + w * p.out_sW + co] = v;
    if (p.silu_out) p.silu_out[n * p.silu_sN + h * p.silu_sH + w * p.silu_sW + co] = __float2half_rn(silu_f(__half2float(v)));
  }
}

#endif  // __CUDACC__

}  // namespace rs

// The attention half of a Swin block as ONE kernel:
//
//     y = x + proj( window_attention( qkv( norm1(x) ) ) )            (+ GroupNorm statistics of y for norm2)
//
// reference: SwinTransformerBlock.forward, models/swin_transformer.py:246-275 (norm1 = GroupNorm32, torch.roll,
// window_partition, WindowAttention.forward :114-145 incl. qkv / relative-position bias / shift mask / softmax / proj,
// window_reverse, roll back, residual).  Unfused this is four launches (gn_apply, qkv GEMM, window_attn, proj GEMM) and a
// [pixels, 3E] fp16 round trip through HBM / L2 (150 MB per block at batch 16, 64x64); here a CTA owns TWO 8x8 windows
// (128 tokens) and nothing but x and y touches global memory:
//
//   * the 128 token rows are gathered with cp.async (the cyclic shift and the window partition are address arithmetic),
//     normalised in place in shared memory (per-image affine from the producers' (mean, M2) pairs, gn_stats.cuh);
//   * per head: [q_h | k_h | v_h] = Xn . W_h^T on mma.sync m16n8k16 (A / B fragments by ldmatrix; the 96 weight rows of
//     the head stream through a double-buffered cp.async ring), stored as fp16 like the unfused path stores qkv;
//     then the tested attention core (QK^T, + bias, + mask, softmax in fp32, PV) on the same tensor-core path;
//   * y = O . W_proj^T + b + x with the weight rows streamed through the same ring, raw x re-fetched into the (dead)
//     operand rows while the last head computes, results staged in shared memory and written as full token rows;
//   * (mean, M2) of y per (image, window, channel) for the norm2 that follows (slots = windows per image, 64 tokens each).
//
// 8 warps: warp w owns token rows [16w, 16w + 16) = rows [(w & 3) * 16, ...) of window (w >> 2).  mma.sync: the
// shifted-window gather does not map onto TMA boxes (wrapped windows split into partial boxes), and the whole attention
// half is 25 % of the model's FLOPs — what matters here is that qkv / P / O never leave the SM and that three launches
// disappear from the dependency chain of every Swin block.
#pragma once

#include "common.cuh"
#include "gn_stats.cuh"
#include "window_attn.cuh"

namespace rs {

struct SwinAttnParams {
  const __half* x; int x_ld;            // [N*H*W, E] view (row stride x_ld)
  __half* y; int y_ld;                  // output view (may alias x: every token row is read before it is written)
  int N, H, W, heads;
  int shift;                            // 0 or 4
  float scale;                          // head_dim^-0.5
  // norm1: producers' pairs (gn_part, gn_slots) or finalised group statistics (gn_gstat)
  const float* gn_part; int gn_slots; const float* gn_gstat;
  const float* gamma; const float* beta; float eps;
  const __half* wqkv; int wqkv_ld;      // [3E][E] fp16, row stride wqkv_ld
  const float* bqkv;                    // [3E]
  const float* relbias;                 // [heads][64][64] fp32
  const __half* wproj; int wproj_ld;    // [E][E]
  const float* bproj;                   // [E]
  GnSink sink[2];                       // statistics of y (slots = windows per image, 64 values each)
  int total_windows;                    // N * (H/8) * (W/8)
};

#ifdef __CUDACC__

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* row_addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(row_addr)));
}

constexpr int kSwinThreads = 256;

template <int kE>
struct SwinSmem {
  static constexpr int PE = kE + 8;                         // halves per row of X / O / W (conflict-free ldmatrix rows)
  static constexpr int kChunkRows = 96;                     // weight rows per streamed chunk (q_h | k_h | v_h of one head)
  static constexpr size_t x_bytes = (size_t)128 * PE * 2;
  static constexpr size_t o_bytes = (size_t)128 * PE * 2;
  static constexpr size_t qkv_bytes = (size_t)2 * 3 * 64 * kAttnPad * 2;      // also the statistics scratch (8 warps x kE x 2 floats)
  static constexpr size_t w_bytes = (size_t)2 * kChunkRows * PE * 2;
  static constexpr size_t ab_bytes = (size_t)2 * kE * 2 * sizeof(float) + (size_t)2 * kE * 2 * sizeof(float) + 2 * 32 * 2 * sizeof(float);
  static constexpr size_t pix_bytes = 128 * sizeof(int);
  static constexpr size_t total = x_bytes + o_bytes + (qkv_bytes > (size_t)8 * kE * 2 * 4 ? qkv_bytes : (size_t)8 * kE * 2 * 4) + w_bytes + ab_bytes + pix_bytes + 64;
};

template <int kE>
__global__ void __launch_bounds__(kSwinThreads, 1) swin_attn_fused_kernel(const __grid_constant__ SwinAttnParams p) {
  using S = SwinSmem<kE>;
  constexpr int PE = S::PE;
  constexpr int kHeads = kE / 32;
  constexpr int kNT = kE / 8;                               // 8-column tiles of the proj output per warp
  constexpr int kProjChunks = (kE + S::kChunkRows - 1) / S::kChunkRows;
  constexpr int kChunks = kHeads + kProjChunks;             // weight chunks per window pair
  extern __shared__ __align__(16) uint8_t swin_smem[];
  __half* sX = reinterpret_cast<__half*>(swin_smem);
  __half* sO = reinterpret_cast<__half*>(swin_smem + S::x_bytes);
  uint8_t* qkv_raw = swin_smem + S::x_bytes + S::o_bytes;
  __half* sQKV = reinterpret_cast<__half*>(qkv_raw);        // [2 windows][q | k | v][64][kAttnPad]
  constexpr size_t qkv_sz = (S::qkv_bytes > (size_t)8 * kE * 2 * 4 ? S::qkv_bytes : (size_t)8 * kE * 2 * 4);
  __half* sW = reinterpret_cast<__half*>(qkv_raw + qkv_sz);
  float* sAB = reinterpret_cast<float*>(qkv_raw + qkv_sz + S::w_bytes);       // [2 windows][kE][2] affine of norm1
  float* sCh = sAB + 2 * kE * 2;                                              // [2][kE][2] per-channel (mean, M2) scratch
  float* sMR = sCh + 2 * kE * 2;                                              // [2][32][2] group (mean, rstd)
  int* sPix = reinterpret_cast<int*>(sMR + 2 * 32 * 2);                       // [128] token -> pixel row, or -1

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int wi = warp >> 2;                                  // which window of the pair
  const int row0 = warp * 16;                                // first token row of this warp inside the 128-row tile
  const int nWx = p.W >> 3, nWy = p.H >> 3, nW = nWx * nWy;
  const int HW = p.H * p.W;
  const int num_pairs = (p.total_windows + 1) >> 1;
  const int per_cta = (num_pairs + gridDim.x - 1) / gridDim.x;
  const int pair_begin = blockIdx.x * per_cta;
  const int pair_end = min(pair_begin + per_cta, num_pairs);

  pdl_trigger();

  // weight chunk c of the stream: c < kHeads: rows {q_c, k_c, v_c} of W_qkv (96 rows); else 96-row chunks of W_proj
  auto stage_chunk = [&](int c, int buf) {
    __half* dst = sW + (size_t)buf * S::kChunkRows * PE;
    constexpr int cpr = kE / 8;                              // 16-byte pieces per row
    for (int i = tid; i < S::kChunkRows * cpr; i += kSwinThreads) {
      const int r = i / cpr, piece = i - r * cpr;
      const __half* src;
      if (c < kHeads) {
        const int which = r >> 5, d = r & 31;
        src = p.wqkv + (size_t)(which * kE + c * 32 + d) * p.wqkv_ld + piece * 8;
      } else {
        const int pr = (c - kHeads) * S::kChunkRows + r;
        if (pr >= kE) continue;
        src = p.wproj + (size_t)pr * p.wproj_ld + piece * 8;
      }
      cp_async_16(dst + (size_t)r * PE + piece * 8, src);
    }
    cp_async_commit();
  };

  int cur_img[2] = {-1, -1};
  // weights do not depend on the producing kernel: the first chunk streams in while it drains
  if (pair_begin < pair_end) stage_chunk(0, 0);
  pdl_wait();

  for (int pair = pair_begin; pair < pair_end; ++pair) {
    // ---- geometry of the two windows ----
    const int wg = 2 * pair + wi;
    const bool wvalid = wg < p.total_windows;
    int n_img[2], wy_[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int w2 = min(2 * pair + k, p.total_windows - 1);
      n_img[k] = w2 / nW;
      wy_[k] = (w2 % nW) / nWx;
    }
    if (tid < 128) {
      const int k = tid >> 6, tok = tid & 63;
      const int w2 = 2 * pair + k;
      int pix = -1;
      if (w2 < p.total_windows) {
        const int n = w2 / nW, rem = w2 % nW, wy = rem / nWx, wx = rem % nWx;
        const int yy = (wy * 8 + (tok >> 3) + p.shift) % p.H, xx = (wx * 8 + (tok & 7) + p.shift) % p.W;
        pix = (n * p.H + yy) * p.W + xx;
      }
      sPix[tid] = pix;
    }
    __syncthreads();
    if (pair != pair_begin) stage_chunk(0, 0);               // chunk 0 of this pair (the first pair's is already in flight)
    // ---- gather the 128 token rows (raw x) ----
    {
      constexpr int cpr = kE / 8;
      for (int i = tid; i < 128 * cpr; i += kSwinThreads) {
        const int r = i / cpr, piece = i - r * cpr;
        const int pix = sPix[r];
        __half* dst = sX + (size_t)r * PE + piece * 8;
        if (pix >= 0) cp_async_16(dst, p.x + (long long)pix * p.x_ld + piece * 8);
        else *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
      }
      cp_async_commit();
    }
    // ---- norm1 affine of the windows' images (recomputed only when the image changes) ----
    const bool need_ab = (n_img[0] != cur_img[0]) || (n_img[1] != cur_img[1]);     // uniform
    if (need_ab) {
      constexpr int cpg = kE / 32;
      if (p.gn_gstat) {
        if (tid < 64) {
          const int k = tid >> 5, gg = tid & 31;
          const float2 mr = ldcg_f2(p.gn_gstat + ((size_t)n_img[k] * 32 + gg) * 2);
          sMR[(k * 32 + gg) * 2] = mr.x; sMR[(k * 32 + gg) * 2 + 1] = mr.y;
        }
      } else {
        const float ns = (float)HW / (float)p.gn_slots;
        for (int idx = tid; idx < 2 * kE; idx += kSwinThreads) {
          const int k = idx / kE, c = idx - k * kE;
          const float2 mq = gn_channel_from_pairs(p.gn_part + (size_t)n_img[k] * p.gn_slots * kE * 2 + (size_t)c * 2, p.gn_slots, kE, ns);
          sCh[(k * kE + c) * 2] = mq.x; sCh[(k * kE + c) * 2 + 1] = mq.y;
        }
        __syncthreads();
        if (tid < 64) {
          const int k = tid >> 5, gg = tid & 31;
          float chp[2 * cpg];
#pragma unroll
          for (int j = 0; j < cpg; ++j) { chp[2 * j] = sCh[(k * kE + gg * cpg + j) * 2]; chp[2 * j + 1] = sCh[(k * kE + gg * cpg + j) * 2 + 1]; }
          const float2 mr = gn_group_from_channels(chp, cpg, (float)HW, p.eps);
          sMR[(k * 32 + gg) * 2] = mr.x; sMR[(k * 32 + gg) * 2 + 1] = mr.y;
        }
      }
      __syncthreads();
      for (int idx = tid; idx < 2 * kE; idx += kSwinThreads) {
        const int k = idx / kE, c = idx - k * kE, gg = c / cpg;
        const float a = sMR[(k * 32 + gg) * 2 + 1] * __ldg(p.gamma + c);
        const float b = __ldg(p.beta + c) - sMR[(k * 32 + gg) * 2] * a;
        sAB[(k * kE + c) * 2] = a; sAB[(k * kE + c) * 2 + 1] = b;
      }
      cur_img[0] = n_img[0]; cur_img[1] = n_img[1];
    }
    // ---- wait for x (the group committed last), normalise in place ----
    cp_async_wait<0>();                                      // x tile and weight chunk 0 have landed (this thread's copies)
    __syncthreads();
    {
      constexpr int cpr = kE / 8;
      for (int i = tid; i < 128 * cpr; i += kSwinThreads) {
        const int r = i / cpr, piece = i - r * cpr;
        const float* ab = sAB + ((size_t)(r >> 6) * kE + piece * 8) * 2;
        uint4* ptr = reinterpret_cast<uint4*>(sX + (size_t)r * PE + piece * 8);
        uint4 raw = *ptr;
        __half2* hh = reinterpret_cast<__half2*>(&raw);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 f = __half22float2(hh[j]);
          f.x = fmaf(f.x, ab[(2 * j) * 2], ab[(2 * j) * 2 + 1]);
          f.y = fmaf(f.y, ab[(2 * j + 1) * 2], ab[(2 * j + 1) * 2 + 1]);
          hh[j] = __floats2half2_rn(f.x, f.y);
        }
        *ptr = raw;
      }
    }
    __syncthreads();

    const int la = p.shift ? swin_label(wy_[wi], (row0 + g) & 7, p.H, p.shift) : 0;       // (row + 8) & 7 == row & 7
    const int lrow0 = (warp & 3) * 16 + g;                   // this lane's rows inside its window: lrow0 and lrow0 + 8

    // ================= heads =================
    for (int h = 0; h < kHeads; ++h) {
      const int buf = h & 1;
      // prefetch the next chunk of the weight stream (next head, or the first proj chunk) into the other buffer: it was
      // last read two chunks ago, and every warp has passed a barrier since
      stage_chunk(h + 1, buf ^ 1);
      // this lane's relative-position-bias values for head h (independent of everything staged): issue early
      const float* bias = p.relbias + (size_t)h * 64 * 64;
      float2 bv0[8], bv1[8];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        bv0[nt] = __ldg(reinterpret_cast<const float2*>(bias + lrow0 * 64 + nt * 8 + 2 * t));
        bv1[nt] = __ldg(reinterpret_cast<const float2*>(bias + (lrow0 + 8) * 64 + nt * 8 + 2 * t));
      }
      cp_async_wait<1>();                                    // chunk h has landed (this thread's copies)
      __syncthreads();                                       // ... everybody's; and every warp finished head h-1's attention
      // ---- [q_h | k_h | v_h] (16 rows x 96) = Xn rows . W_h^T ----
      const __half* wbuf = sW + (size_t)buf * S::kChunkRows * PE;
      float acc[12][4];
#pragma unroll
      for (int nt = 0; nt < 12; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll 2
      for (int ks = 0; ks < kE / 16; ++ks) {
        uint32_t a[4];
        ldmatrix_x4(a, sX + (size_t)(row0 + (lane & 7) + ((lane >> 3) & 1) * 8) * PE + ks * 16 + (lane >> 4) * 8);
#pragma unroll
        for (int np = 0; np < 6; ++np) {
          uint32_t b[4];
          ldmatrix_x4(b, wbuf + (size_t)(np * 16 + (lane & 7) + (lane >> 4) * 8) * PE + ks * 16 + ((lane >> 3) & 1) * 8);
          const uint32_t b0[2] = {b[0], b[1]}, b1[2] = {b[2], b[3]};
          mma_16816(acc[2 * np], a, b0);
          mma_16816(acc[2 * np + 1], a, b1);
        }
      }
      // + bias, round to fp16 (as the unfused path stores qkv), into the per-window q / k / v tiles
      {
        __half* qkvw = sQKV + (size_t)wi * 3 * 64 * kAttnPad;
#pragma unroll
        for (int nt = 0; nt < 12; ++nt) {
          const int which = nt >> 2, d = (nt & 3) * 8 + 2 * t;
          const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bqkv + which * kE + h * 32 + d));
          __half* dst = qkvw + (size_t)which * 64 * kAttnPad;
          *reinterpret_cast<__half2*>(dst + lrow0 * kAttnPad + d) = __floats2half2_rn(acc[nt][0] + bb.x, acc[nt][1] + bb.y);
          *reinterpret_cast<__half2*>(dst + (lrow0 + 8) * kAttnPad + d) = __floats2half2_rn(acc[nt][2] + bb.x, acc[nt][3] + bb.y);
        }
      }
      if (h == kHeads - 1) {
        // the normalised x rows of this warp are dead now: fetch the RAW rows (residual) into them; they land while the
        // last head's attention and the projection run
        constexpr int cpr = kE / 8;
        __syncwarp();                                        // every lane's last ldmatrix of these rows has been issued
        for (int i = lane; i < 16 * cpr; i += 32) {
          const int r = row0 + i / cpr, piece = i % cpr;
          const int pix = sPix[r];
          if (pix >= 0) cp_async_16(sX + (size_t)r * PE + piece * 8, p.x + (long long)pix * p.x_ld + piece * 8);
        }
      }
      __syncthreads();                                       // K and V rows of all four warps of a window are in place
      // ---- attention core of head h for this warp's 16 query rows (same arithmetic as window_attn_kernel) ----
      {
        const __half* sQ = sQKV + (size_t)wi * 3 * 64 * kAttnPad;
        const __half* sK = sQ + 64 * kAttnPad;
        const __half* sV = sK + 64 * kAttnPad;
        uint32_t qa[2][4];
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
          const int d = ks * 16 + 2 * t;
          qa[ks][0] = *reinterpret_cast<const uint32_t*>(&sQ[lrow0 * kAttnPad + d]);
          qa[ks][1] = *reinterpret_cast<const uint32_t*>(&sQ[(lrow0 + 8) * kAttnPad + d]);
          qa[ks][2] = *reinterpret_cast<const uint32_t*>(&sQ[lrow0 * kAttnPad + d + 8]);
          qa[ks][3] = *reinterpret_cast<const uint32_t*>(&sQ[(lrow0 + 8) * kAttnPad + d + 8]);
        }
        float s[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
          for (int ks = 0; ks < 2; ++ks) {
            const int key = nt * 8 + g, d = ks * 16 + 2 * t;
            uint32_t kb[2];
            kb[0] = *reinterpret_cast<const uint32_t*>(&sK[key * kAttnPad + d]);
            kb[1] = *reinterpret_cast<const uint32_t*>(&sK[key * kAttnPad + d + 8]);
            mma_16816(s[nt], qa[ks], kb);
          }
        }
        float mx0 = -1e30f, mx1 = -1e30f;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          const int col = nt * 8 + 2 * t;
          const float2 b0 = bv0[nt], b1 = bv1[nt];
          float m0 = 0.f, m1 = 0.f;
          if (p.shift) {
            if (swin_label(wy_[wi], col & 7, p.H, p.shift) != la) m0 = -100.0f;
            if (swin_label(wy_[wi], (col + 1) & 7, p.H, p.shift) != la) m1 = -100.0f;
          }
          s[nt][0] = s[nt][0] * p.scale + b0.x + m0;
          s[nt][1] = s[nt][1] * p.scale + b0.y + m1;
          s[nt][2] = s[nt][2] * p.scale + b1.x + m0;
          s[nt][3] = s[nt][3] * p.scale + b1.y + m1;
          mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
          mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            s[nt][e] = __expf(s[nt][e] - mx0); sum0 += s[nt][e];
            s[nt][2 + e] = __expf(s[nt][2 + e] - mx1); sum1 += s[nt][2 + e];
          }
        }
        sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1); sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
        sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1); sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
        float o[4][4];
#pragma unroll
        for (int dt = 0; dt < 4; ++dt) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          uint32_t pa[4];
          pa[0] = pack_h2(s[2 * kk][0], s[2 * kk][1]);
          pa[1] = pack_h2(s[2 * kk][2], s[2 * kk][3]);
          pa[2] = pack_h2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
          pa[3] = pack_h2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
          for (int dt = 0; dt < 4; ++dt) {
            uint32_t vb[2];
            ldmatrix_x2_trans(vb, &sV[(kk * 16 + (lane & 15)) * kAttnPad + dt * 8]);
            mma_16816(o[dt], pa, vb);
          }
        }
        const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;
#pragma unroll
        for (int dt = 0; dt < 4; ++dt) {
          const int d = h * 32 + dt * 8 + 2 * t;
          *reinterpret_cast<__half2*>(&sO[(size_t)(row0 + g) * PE + d]) = __floats2half2_rn(o[dt][0] * inv0, o[dt][1] * inv0);
          *reinterpret_cast<__half2*>(&sO[(size_t)(row0 + g + 8) * PE + d]) = __floats2half2_rn(o[dt][2] * inv1, o[dt][3] * inv1);
        }
      }
    }

    // ================= projection: y = O . W_proj^T + b + x =================
    cp_async_commit();                                       // (group of the raw-x rows issued during the last head)
    float acc2[kNT][4];
#pragma unroll
    for (int nt = 0; nt < kNT; ++nt) acc2[nt][0] = acc2[nt][1] = acc2[nt][2] = acc2[nt][3] = 0.f;
#pragma unroll
    for (int pc = 0; pc < kProjChunks; ++pc) {
      const int c = kHeads + pc, buf = c & 1;
      if (pc + 1 < kProjChunks) { stage_chunk(c + 1, buf ^ 1); cp_async_wait<1>(); }     // (buffer last read by chunk c-1: barrier below precedes)
      else cp_async_wait<0>();
      __syncthreads();
      const __half* wbuf = sW + (size_t)buf * S::kChunkRows * PE;
      constexpr int rows_here_max = S::kChunkRows;
      const int rows_here = min(rows_here_max, kE - pc * S::kChunkRows);
#pragma unroll 2
      for (int ks = 0; ks < kE / 16; ++ks) {
        uint32_t a[4];
        ldmatrix_x4(a, sO + (size_t)(row0 + (lane & 7) + ((lane >> 3) & 1) * 8) * PE + ks * 16 + (lane >> 4) * 8);
#pragma unroll
        for (int np = 0; np < S::kChunkRows / 16; ++np) {
          if (np * 16 < rows_here) {
            uint32_t b[4];
            ldmatrix_x4(b, wbuf + (size_t)(np * 16 + (lane & 7) + (lane >> 4) * 8) * PE + ks * 16 + ((lane >> 3) & 1) * 8);
            const uint32_t b0[2] = {b[0], b[1]}, b1[2] = {b[2], b[3]};
            const int nt = pc * (S::kChunkRows / 8) + 2 * np;
            if (nt < kNT) mma_16816(acc2[nt], a, b0);
            if (nt + 1 < kNT) mma_16816(acc2[nt + 1], a, b1);
          }
        }
      }
      if (pc + 1 < kProjChunks) __syncthreads();             // the buffer of chunk c may be refilled after everyone read it
    }
    // ---- epilogue: + bias + raw x -> fp16 (one rounding), staged in this warp's (dead) O rows, statistics, row stores ----
    __syncthreads();                                         // every warp is done with the weight ring: it becomes the statistics scratch
    float* sStat = reinterpret_cast<float*>(sW);             // [8 warps][kE][2] = (mean, M2) over the warp's 16 rows
    const bool want_stats = p.sink[0].part != nullptr;
#pragma unroll
    for (int nt = 0; nt < kNT; ++nt) {
      const int c = nt * 8 + 2 * t;
      const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bproj + c));
      const float2 x0 = __half22float2(*reinterpret_cast<const __half2*>(&sX[(size_t)(row0 + g) * PE + c]));
      const float2 x1 = __half22float2(*reinterpret_cast<const __half2*>(&sX[(size_t)(row0 + g + 8) * PE + c]));
      const __half2 y0 = __floats2half2_rn(acc2[nt][0] + bb.x + x0.x, acc2[nt][1] + bb.y + x0.y);
      const __half2 y1 = __floats2half2_rn(acc2[nt][2] + bb.x + x1.x, acc2[nt][3] + bb.y + x1.y);
      *reinterpret_cast<__half2*>(&sO[(size_t)(row0 + g) * PE + c]) = y0;
      *reinterpret_cast<__half2*>(&sO[(size_t)(row0 + g + 8) * PE + c]) = y1;
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
          float* dst = sStat + ((size_t)warp * kE + c) * 2;
          dst[0] = m0; dst[1] = fmaxf(qx - sx * m0, 0.f);
          dst[2] = m1; dst[3] = fmaxf(qy - sy * m1, 0.f);
        }
      }
    }
    __syncwarp();
    // full token rows to global (this warp's 16 rows)
    if (wvalid) {
      constexpr int cpr = kE / 8;
      for (int i = lane; i < 16 * cpr; i += 32) {
        const int r = row0 + i / cpr, piece = i % cpr;
        *reinterpret_cast<uint4*>(p.y + (long long)sPix[r] * p.y_ld + piece * 8) = *reinterpret_cast<const uint4*>(sO + (size_t)r * PE + piece * 8);
      }
    }
    if (want_stats) {
      __syncthreads();
      // merge the four 16-row warps of each window (Chan et al., equal counts) and deliver the window's pairs
      for (int idx = tid; idx < 2 * kE; idx += kSwinThreads) {
        const int k = idx / kE, c = idx - k * kE;
        const int w2 = 2 * pair + k;
        if (w2 >= p.total_windows) continue;
        float m[4], q[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) { m[j] = sStat[((size_t)(k * 4 + j) * kE + c) * 2]; q[j] = sStat[((size_t)(k * 4 + j) * kE + c) * 2 + 1]; }
        float ma, qa2, mb, qb, mm, qq;
        chan_merge_equal(16.f, m[0], q[0], m[1], q[1], ma, qa2);
        chan_merge_equal(16.f, m[2], q[2], m[3], q[3], mb, qb);
        chan_merge_equal(32.f, ma, qa2, mb, qb, mm, qq);
        const int n = w2 / nW, slot = w2 % nW;
#pragma unroll
        for (int d = 0; d < 2; ++d) {
          const GnSink& sk = p.sink[d];
          if (!sk.part) continue;
          float* dst = sk.part + (((size_t)n * nW + slot) * sk.cstride + sk.coff + c) * 2;
          dst[0] = mm; dst[1] = qq;
        }
      }
    }
    __syncthreads();                                         // this pair's shared memory is free for the next pair
  }
}

#endif  // __CUDACC__
}  // namespace rs

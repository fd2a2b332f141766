// GroupNorm(32 groups, eps 1e-5, fp32 statistics) + FiLM + SiLU on NHWC fp16 views.
//
// reference: GroupNorm32 (models/basic_ops.py:15-17,89-96), its uses in ResBlock
// (models/unet.py:144-148,168-175,198-202: GN -> SiLU, and GN*(1+scale)+shift -> SiLU) and in
// SwinTransformerBlock (models/swin_transformer.py:248,279: plain GN), final head (unet.py:859-863).
//
// Statistics (gn_stats.cuh): every producer tile delivers (mean, M2) pairs per (image, slot, channel); the last producer
// CTA of an image reduces them to gstat[image][group] = (mean, rstd).  Producers are
//   * the epilogue of the conv / GEMM / MLP kernel that wrote the tensor (one slot per 128-pixel tile), or
//   * gn_stats_kernel below (one slot per CTA) for tensors that have no fusable producer.
// gn_apply_kernel folds (mean, rstd, gamma, beta, FiLM) into a per-(image, channel) affine a*x+b in shared memory,
// then streams x -> y = act(a*x+b) with 128-bit accesses.
#pragma once

#include "common.cuh"
#include "gn_stats.cuh"

namespace rs {

struct GnStatsParams {
  const __half* x;          // view [N][HW][C], row stride ld
  long long sN;             // image stride (elements)
  int ld, C, HW, N;
  GnSink sink;              // part [N][slots][C][2], gstat, counter, expected = slots * C
  int slots;
  int rows_per_slot;        // divides HW: every slot holds the same number of rows
};

struct GnApplyParams {
  const __half* x; long long x_sN; int x_ld;
  __half* y; long long y_sN; int y_ld;
  int C, HW, N;
  const float* gstat;       // [N][32][2] = (group mean, group rstd) finalised by the producer, or nullptr: combine here
  const float* part;        // [N][slots][C][2] (mean, M2) pairs (used when gstat == nullptr)
  int slots;
  float eps;
  const float* gamma;       // [C]
  const float* beta;        // [C]
  const float* film;        // optional [N or 1][2*C] : scale = film[0:C], shift = film[C:2C]
  long long film_sN;        // 0 when the same timestep embedding is shared by the whole batch
  int silu;
  int rows_per_cta;
  int Cs;                   // channels per CTA (blockIdx.z selects the slice; a multiple of 8 and of C/32): small tensors
                            // are split over channels as well as rows so that every SM gets a CTA
};

#ifdef __CUDACC__

// One CTA per (slot, image).  Each thread owns one 8-channel vector column and walks rows (4 loads in flight), keeping
// pivot-shifted sums; row-lanes are merged through shared memory in lane order (Chan et al.).
__global__ void __launch_bounds__(256) gn_stats_kernel(const __grid_constant__ GnStatsParams p) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float s_red[];   // [lanes][C][3] = (rows, mean, M2); + flags
  const int vecs = p.C >> 3;
  const int lanes = blockDim.x / vecs;
  const int n = blockIdx.y, slot = blockIdx.x;
  const int vec = threadIdx.x % vecs;
  const int rl = threadIdx.x / vecs;
  if (rl < lanes) {
    float pv[8], s1[8], s2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { pv[j] = 0.f; s1[j] = 0.f; s2[j] = 0.f; }
    int cnt = 0;
    const int r0 = slot * p.rows_per_slot;
    const int r1 = min(r0 + p.rows_per_slot, p.HW);
    const __half* base = p.x + n * p.sN + vec * 8;
    auto acc = [&](const uint4& raw) {
      const __half2* h = reinterpret_cast<const __half2*>(&raw);
      float st[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h[j]); st[2 * j] = f.x; st[2 * j + 1] = f.y; }
      if (cnt == 0) {
#pragma unroll
        for (int j = 0; j < 8; ++j) pv[j] = st[j];
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float d = st[j] - pv[j]; s1[j] += d; s2[j] = fmaf(d, d, s2[j]); }
      }
      ++cnt;
    };
    int r = r0 + rl;
    for (; r + 3 * lanes < r1; r += 4 * lanes) {
      uint4 raw[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) raw[u] = *reinterpret_cast<const uint4*>(base + (long long)(r + u * lanes) * p.ld);
#pragma unroll
      for (int u = 0; u < 4; ++u) acc(raw[u]);
    }
    for (; r < r1; r += lanes) acc(*reinterpret_cast<const uint4*>(base + (long long)r * p.ld));
    float* dst = s_red + ((size_t)rl * p.C + vec * 8) * 3;
    const float inv = cnt ? 1.0f / (float)cnt : 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      dst[3 * j] = (float)cnt;
      dst[3 * j + 1] = pv[j] + s1[j] * inv;
      dst[3 * j + 2] = fmaxf(s2[j] - s1[j] * s1[j] * inv, 0.f);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < p.C; i += blockDim.x) {
    float cn = 0.f, mean = 0.f, m2 = 0.f;
    for (int l = 0; l < lanes; ++l) {
      const float* e = s_red + ((size_t)l * p.C + i) * 3;
      const float nb = e[0];
      if (nb == 0.f) continue;
      const float tot = cn + nb, d = e[1] - mean;
      mean += d * (nb / tot);
      m2 += e[2] + d * d * (cn * nb / tot);
      cn = tot;
    }
    float* dst = p.sink.part + (((size_t)n * p.slots + slot) * p.C + i) * 2;
    dst[0] = mean; dst[1] = m2;
  }
  if (!p.sink.gstat) return;
  int* s_flag = reinterpret_cast<int*>(s_red + (size_t)lanes * p.C * 3);
  const GnSink* const sk[1] = {&p.sink};
  const int im[1] = {n};
  const unsigned int ad[1] = {(unsigned)p.C};
  gn_arrive<1>(sk, im, ad, p.slots, (float)p.rows_per_slot, threadIdx.x, blockDim.x, 1, s_flag);
}

// Group statistics from the producers' pairs as a small kernel of its own: one CTA per (group, image), the K = slots * cpg
// items of the group strided over 256 threads (4 loads in flight each), common pivot = item 0, fixed reduction order.
// For tensors with hundreds of tile slots per image (the VQ-GAN's 128x128 / 256x256 maps) it avoids both alternatives:
// every consumer CTA re-reading slots x C pairs, and the last producer CTA reducing them on the tail of a persistent conv
// kernel (one CTA ends up last for every image).
struct GnFinalizeParams {
  const float* part;        // [N][slots][C][2]
  float* gstat;             // [N][32][2] = (mean, rstd)
  int slots, C;
  float ns, eps;            // values per item (rows per slot)
};

__global__ void __launch_bounds__(256) gn_finalize_kernel(const GnFinalizeParams p) {
  pdl_trigger();
  pdl_wait();
  __shared__ float s_w[8][2];
  const int g = blockIdx.x, n = blockIdx.y;
  const int cpg = p.C >> 5;
  const int K = p.slots * cpg;
  const float* base = p.part + (size_t)n * p.slots * p.C * 2 + (size_t)g * cpg * 2;
  const float pivot = ldcg_f2(base).x;
  float s1 = 0.f, s2 = 0.f;
  auto item = [&](int i) -> float2 {
    const int sl = i / cpg, c = i - sl * cpg;
    return ldcg_f2(base + ((size_t)sl * p.C + c) * 2);
  };
  int i = threadIdx.x;
  for (; i + 3 * 256 < K; i += 4 * 256) {
    float2 e[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) e[u] = item(i + u * 256);
#pragma unroll
    for (int u = 0; u < 4; ++u) { const float d = e[u].x - pivot; s1 += d; s2 += fmaf(p.ns * d, d, e[u].y); }
  }
  for (; i < K; i += 256) { const float2 e = item(i); const float d = e.x - pivot; s1 += d; s2 += fmaf(p.ns * d, d, e.y); }
#pragma unroll
  for (int off = 16; off; off >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, off);
    s2 += __shfl_xor_sync(0xffffffffu, s2, off);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { s_w[warp][0] = s1; s_w[warp][1] = s2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) { a += s_w[w][0]; b += s_w[w][1]; }
    const float invK = 1.0f / (float)K;
    const float dm = a * invK;
    const float m2 = fmaxf(b - p.ns * (float)K * dm * dm, 0.f);
    p.gstat[((size_t)n * 32 + g) * 2] = pivot + dm;
    p.gstat[((size_t)n * 32 + g) * 2 + 1] = rsqrtf(m2 * invK / p.ns + p.eps);
  }
}

__global__ void __launch_bounds__(256, 4) gn_apply_kernel(const GnApplyParams p) {
  pdl_trigger();
  extern __shared__ float s_ab[];    // a[Cs], b[Cs], gamma[Cs], beta[Cs], mean[32], rstd[32]  (this CTA's channel slice)
  const int Cs = p.Cs;
  const int c0 = blockIdx.z * Cs;    // first channel of the slice (group aligned)
  float* s_a = s_ab;
  float* s_b = s_ab + Cs;
  float* s_g = s_ab + 2 * Cs;
  float* s_be = s_ab + 3 * Cs;
  float* s_mean = s_ab + 4 * Cs;
  float* s_rstd = s_mean + 32;
  const int n = blockIdx.y;
  const int cpg = p.C / 32;
  // layer parameters do not depend on the producing kernel: fetch them while it drains
  for (int c = threadIdx.x; c < Cs; c += blockDim.x) { s_g[c] = __ldg(p.gamma + c0 + c); s_be[c] = __ldg(p.beta + c0 + c); }
  pdl_wait();
  // the first rows of x do not depend on the statistics: put their loads in flight before the (latency-bound) statistics
  // prologue below, so that its L2 round trips and barriers overlap the first data round trip
  const int vecs = Cs >> 3;
  const int lanes = blockDim.x / vecs;
  const int vec = threadIdx.x % vecs, rl = threadIdx.x / vecs;
  const bool active = rl < lanes;
  const int c = vec * 8;
  const int r0 = blockIdx.x * p.rows_per_cta;
  const int r1 = min(r0 + p.rows_per_cta, p.HW);
  const __half* xb = p.x + n * p.x_sN + c0 + c;
  __half* yb = p.y + n * p.y_sN + c0 + c;
  int r = r0 + rl;
  constexpr int kPre = 4;
  uint4 pre[kPre];
#pragma unroll
  for (int u = 0; u < kPre; ++u)
    if (active && r + u * lanes < r1) pre[u] = *reinterpret_cast<const uint4*>(xb + (long long)(r + u * lanes) * p.x_ld);
  if (p.gstat) {
    // the image's 32 (mean, rstd) pairs were finalised by the producer side / gn_finalize_kernel: one small read
    if (threadIdx.x < Cs / cpg) {
      const float2 mr = ldcg_f2(p.gstat + ((size_t)n * 32 + c0 / cpg + threadIdx.x) * 2);
      s_mean[threadIdx.x] = mr.x; s_rstd[threadIdx.x] = mr.y;
    }
  } else {
    // combine the producers' (mean, M2) pairs here (small tensors: a few slots): per channel over the slots, then per
    // group over its channels — Chan's formula around pivots at both levels, fixed order
    const float ns = (float)p.HW / (float)p.slots;
    const float* part = p.part + (size_t)n * p.slots * p.C * 2 + (size_t)c0 * 2;
    for (int cc = threadIdx.x; cc < Cs; cc += blockDim.x) {
      const float2 mq = gn_channel_from_pairs(part + (size_t)cc * 2, p.slots, p.C, ns);
      s_a[cc] = mq.x; s_b[cc] = mq.y;
    }
    __syncthreads();
    if (threadIdx.x < Cs / cpg) {
      const int g = threadIdx.x;
      float chp[2 * 64];                                            // cpg <= 64 (C <= 2048)
      for (int j = 0; j < cpg; ++j) { chp[2 * j] = s_a[g * cpg + j]; chp[2 * j + 1] = s_b[g * cpg + j]; }
      const float2 mr = gn_group_from_channels(chp, cpg, (float)p.HW, p.eps);
      s_mean[g] = mr.x; s_rstd[g] = mr.y;
    }
  }
  __syncthreads();
  {
    const float* f = p.film ? p.film + n * p.film_sN + c0 : nullptr;
    for (int cc = threadIdx.x; cc < Cs; cc += blockDim.x) {
      const int g = cc / cpg;
      float a = s_rstd[g] * s_g[cc];
      float b = s_be[cc] - s_mean[g] * a;
      if (f) { const float sc = 1.0f + f[cc]; a *= sc; b = b * sc + f[p.C + cc]; }
      s_a[cc] = a; s_b[cc] = b;
    }
  }
  __syncthreads();
  if (!active) return;
  float a[8], b[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { a[j] = s_a[c + j]; b[j] = s_b[c + j]; }
  auto one = [&](const uint4& raw) {
    const __half2* h = reinterpret_cast<const __half2*>(&raw);
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 f = __half22float2(h[j]);
      f.x = fmaf(f.x, a[2 * j], b[2 * j]);
      f.y = fmaf(f.y, a[2 * j + 1], b[2 * j + 1]);
      if (p.silu) { f.x = silu_f(f.x); f.y = silu_f(f.y); }
      oh[j] = __floats2half2_rn(f.x, f.y);
    }
    return o;
  };
#pragma unroll
  for (int u = 0; u < kPre; ++u)
    if (r + u * lanes < r1) *reinterpret_cast<uint4*>(yb + (long long)(r + u * lanes) * p.y_ld) = one(pre[u]);
  r += kPre * lanes;
  for (; r + 7 * lanes < r1; r += 8 * lanes) {
    uint4 raw[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) raw[u] = *reinterpret_cast<const uint4*>(xb + (long long)(r + u * lanes) * p.x_ld);
#pragma unroll
    for (int u = 0; u < 8; ++u) *reinterpret_cast<uint4*>(yb + (long long)(r + u * lanes) * p.y_ld) = one(raw[u]);
  }
  for (; r + 3 * lanes < r1; r += 4 * lanes) {
    uint4 raw[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) raw[u] = *reinterpret_cast<const uint4*>(xb + (long long)(r + u * lanes) * p.x_ld);
#pragma unroll
    for (int u = 0; u < 4; ++u) *reinterpret_cast<uint4*>(yb + (long long)(r + u * lanes) * p.y_ld) = one(raw[u]);
  }
  for (; r < r1; r += lanes) {
    const uint4 raw = *reinterpret_cast<const uint4*>(xb + (long long)r * p.x_ld);
    *reinterpret_cast<uint4*>(yb + (long long)r * p.y_ld) = one(raw);
  }
}

#endif
}  // namespace rs

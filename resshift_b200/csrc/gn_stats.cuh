// GroupNorm statistics plumbing shared by every kernel that PRODUCES a tensor a GroupNorm will read.
//
// reference: GroupNorm32 = F.group_norm(x.float(), 32 groups, eps) (models/basic_ops.py:15-17; eps 1e-5 in the UNet,
// 1e-6 in the VQ-GAN: ldm/modules/diffusionmodules/model.py:47).  The reduction spans a whole image, so it cannot be a
// pure epilogue of one output tile.  Three stages, all deterministic (fixed summation order, no floating-point atomics):
//
//   1. every producer tile writes, per (image, tile slot, channel), the pair (mean, M2) of the fp16 values it STORED
//      (M2 = sum of squared deviations from that local mean).  Local sums are taken around a pivot (the first row of the
//      tile), so a channel with |mean| >> std loses nothing to cancellation (E[x^2] - mean^2 in fp32 does).
//   2. the pairs of each of the 32 groups are combined — Chan et al.'s parallel variance formula, again around a pivot —
//      into gstat[image][group] = (mean, rstd): by every consumer CTA itself on small maps (few tile slots), or on maps
//      with many slots by gn_finalize_kernel, a small launch in front of the consumer, or by the last CTA of
//      gn_stats_kernel to finish an image (an integer arrival counter per (GroupNorm, image) decides who that is; the
//      arithmetic does not depend on who) when no producer epilogue delivers the pairs.
//   3. consumers (gn_apply_kernel, the fused MLP's and the qkv GEMM's in-shared-memory operand transform) read the 32
//      pairs of their image and fold gamma / beta (/ FiLM) into a per-channel affine.
//
// Compared with round 1 (every consumer CTA re-reducing slots x C raw sums: 41 KB per CTA at 64x64, 0.5 MB at 256x256)
// the consumers' preamble is one 256-byte read, and the statistics are robust.
#pragma once

#include "common.cuh"

namespace rs {

// what a producer needs to know about ONE consuming GroupNorm (up to two per producer: a skip tensor feeds the next
// encoder block and, later, the decoder's concat GroupNorm)
struct GnSink {
  float* part;            // [N][slots][cstride][2] = (mean, M2) per image / tile slot / channel; nullptr: no statistics
  float* gstat;           // [N][32][2] = (group mean, group rstd), written by the last-arriving gn_stats_kernel CTA
  unsigned int* counter;  // [N] channel-slots delivered so far (zeroed before every forward)
  int cstride;            // channel count of the consumer's tensor (this producer may cover only a slice of it)
  int coff;               // first channel of this producer's slice
  unsigned int expected;  // slots * cstride: the image is complete when the counter reaches it
  float eps;
};

#ifdef __CUDACC__

__device__ __forceinline__ float2 ldcg_f2(const float* p) {
  float2 v;
  asm volatile("ld.global.cg.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p) : "memory");
  return v;
}

// counter += v with acquire-release semantics at GPU scope, by ONE thread after a CTA barrier: the barrier orders the
// other threads' pair stores before it (causality is cumulative over bar.sync), the release half publishes them, and —
// if this turns out to be the last arrival — the acquire half orders the finaliser's reads after every earlier arrival.
// (Each thread issuing __threadfence() instead would cost a GPU-scope fence per thread and tile.)
__device__ __forceinline__ unsigned int atom_add_acq_rel_gpu(unsigned int* p, unsigned int v) {
  unsigned int old;
  asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}

// Combine two (count, mean, M2) triples with equal counts n each (Chan et al.): used for the two 64-row halves of a tile.
__device__ __forceinline__ void chan_merge_equal(float n, float m0, float q0, float m1, float q1, float& m, float& q) {
  m = 0.5f * (m0 + m1);
  const float d0 = m0 - m, d1 = m1 - m;
  q = q0 + q1 + n * (d0 * d0 + d1 * d1);
}

// Group statistics of image `n` from the per-(slot, channel) pairs: ONE warp (all 32 lanes) reduces kG groups at once
// (g0, g0 + gstep, ...) so that kG x 4 independent L2 loads are in flight per lane — the finaliser sits on the tail of a
// producer kernel and is pure load latency.  Per group: K = slots * cpg items of `ns` values each, single pass around
// the pivot item 0; lanes take items lane, lane + 32, ...; lane partials are combined with a fixed shuffle tree.
template <int kG>
__device__ __forceinline__ void gn_finalize_groups(const float* part, int n, int slots, int C, int g0, int gstep, int cpg, float ns,
                                                   float eps, float* gstat, int lane) {
  const float* base = part + (size_t)n * slots * C * 2;
  const int K = slots * cpg;
  float pivot[kG], s1[kG], s2[kG];
#pragma unroll
  for (int q = 0; q < kG; ++q) {
    const int g = g0 + q * gstep;
    pivot[q] = g < 32 ? ldcg_f2(base + (size_t)(g * cpg) * 2).x : 0.f;
    s1[q] = 0.f; s2[q] = 0.f;
  }
  for (int i0 = 0; i0 < K; i0 += 128) {
    float2 e[kG][4];
#pragma unroll
    for (int q = 0; q < kG; ++q) {
      const int g = g0 + q * gstep;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * 32 + lane;
        if (g < 32 && i < K) {
          const int sl = i / cpg, c = i - sl * cpg;
          e[q][u] = ldcg_f2(base + ((size_t)sl * C + g * cpg + c) * 2);
        } else {
          e[q][u] = make_float2(pivot[q], 0.f);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < kG; ++q)
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float d = e[q][u].x - pivot[q];
        s1[q] += d;
        s2[q] += fmaf(ns * d, d, e[q][u].y);
      }
  }
#pragma unroll
  for (int q = 0; q < kG; ++q) {
    float a = s1[q], b = s2[q];
#pragma unroll
    for (int off = 16; off; off >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, off);
      b += __shfl_xor_sync(0xffffffffu, b, off);
    }
    const int g = g0 + q * gstep;
    const float invK = 1.0f / (float)K;
    const float dm = a * invK;                    // group mean - pivot
    const float m2 = fmaxf(b - ns * (float)K * dm * dm, 0.f);
    const float var = m2 * invK / ns;
    if (lane == 0 && g < 32) {
      gstat[((size_t)n * 32 + g) * 2] = pivot[q] + dm;
      gstat[((size_t)n * 32 + g) * 2 + 1] = rsqrtf(var + eps);
    }
  }
}

// Arrival protocol, called by ALL `nthreads` threads of a producer's epilogue group (named barrier `bar_id`) AFTER they
// have written their (mean, M2) pairs for up to kMax (sink, image) pairs.  `img[i] < 0` = nothing delivered for entry i.
//   add[i]  = channels this CTA delivered for (sink[i], img[i]) in this tile slot
// The last arriver of an image reduces the image's 32 groups (warp w takes groups w, w + #warps, ... four at a time).
template <int kMax>
__device__ __forceinline__ void gn_arrive(const GnSink* const (&sink)[kMax], const int (&img)[kMax], const unsigned int (&add)[kMax],
                                          int slots, float ns, int tid, int nthreads, int bar_id, int* s_flag /* [kMax] shared */) {
  named_bar_sync(bar_id, nthreads);               // every thread's pair stores happen-before the arrival below
  if (tid < kMax) {
    int last = 0;
    if (sink[tid] != nullptr && img[tid] >= 0 && sink[tid]->gstat != nullptr) {
      const unsigned int old = atom_add_acq_rel_gpu(sink[tid]->counter + img[tid], add[tid]);
      last = (old + add[tid] == sink[tid]->expected) ? 1 : 0;
    }
    s_flag[tid] = last;
  }
  named_bar_sync(bar_id, nthreads);               // ... and the acquiring arrival happens-before the finaliser's reads
  const int warp = tid >> 5, lane = tid & 31, nwarps = nthreads >> 5;
#pragma unroll
  for (int i = 0; i < kMax; ++i) {
    if (!s_flag[i]) continue;                     // uniform across the group
    const GnSink& s = *sink[i];                   // (pairs are read with ld.global.cg: L2, never a stale L1 line)
    const int cpg = s.cstride / 32;
    for (int g = warp; g < 32; g += 4 * nwarps) gn_finalize_groups<4>(s.part, img[i], slots, s.cstride, g, nwarps, cpg, ns, s.eps, s.gstat, lane);
  }
  named_bar_sync(bar_id, nthreads);               // s_flag may be rewritten by the next tile
}

// (mean, M2) of the `rows` fp16 values x[r * pitch_h] (r = 0 .. rows-1) read through `ld(r)` -> float2 (two adjacent
// columns), around the pivot ld(0).  Returns mean / M2 per column.
template <typename Ld>
__device__ __forceinline__ void pivot_stats2(Ld ld, int rows, float2& mean, float2& m2) {
  const float2 p = ld(0);
  float2 s1 = make_float2(0.f, 0.f), s2 = make_float2(0.f, 0.f);
  for (int r = 1; r < rows; ++r) {
    const float2 v = ld(r);
    const float dx = v.x - p.x, dy = v.y - p.y;
    s1.x += dx; s1.y += dy;
    s2.x = fmaf(dx, dx, s2.x); s2.y = fmaf(dy, dy, s2.y);
  }
  const float inv = 1.0f / (float)rows;
  mean = make_float2(p.x + s1.x * inv, p.y + s1.y * inv);
  m2 = make_float2(fmaxf(s2.x - s1.x * s1.x * inv, 0.f), fmaxf(s2.y - s1.y * s1.y * inv, 0.f));
}

// One step of warp_chunk_stats' transpose-reduce: lanes that differ in bit 2 * kHalf exchange halves of their first
// 2 * kHalf columns.  The step width is a template argument so that every sv / sq index is a compile-time constant:
// written as one loop over (half >>= 1, bit >>= 1), nvcc kept a run-time index and put sv / sq in local memory, which
// in the MMA kernels (most of L1 carved out as shared memory) went to L2 and cost about 10 us per 128-row tile of the
// fused MLP at E = 192.
template <int kHalf>
__device__ __forceinline__ void warp_xor_step(float (&sv)[16], float (&sq)[16], int lane) {
  constexpr int bit = 2 * kHalf;
  const bool upper = (lane & bit) != 0;
#pragma unroll
  for (int j = 0; j < kHalf; ++j) {
    const float send_s = upper ? sv[j] : sv[j + kHalf];
    const float keep_s = upper ? sv[j + kHalf] : sv[j];
    sv[j] = keep_s + __shfl_xor_sync(0xffffffffu, send_s, bit);
    const float send_q = upper ? sq[j] : sq[j + kHalf];
    const float keep_q = upper ? sq[j + kHalf] : sq[j];
    sq[j] = keep_q + __shfl_xor_sync(0xffffffffu, send_q, bit);
  }
}

// Statistics of one epilogue chunk while the accumulator tile drains: this warp's 32 rows x 16 columns, the values
// exactly as stored (o0 / o1 = the two 16-byte units of fp16 the lane writes).  Transpose-reduce over the 32 lanes
// (16 shuffles per moment, fixed tree), then (sum, sum of squares) -> (mean, M2) right here: over 32 fp16 values the
// subtraction q - s^2/32 is benign (relative error ~1e-3 of M2 even for |mean| = 60 std), and every later combination
// is Chan's formula on (mean, M2) pairs, so nothing down the line cancels.  dst = &wq[(quad * BN + c) * 2].
__device__ __forceinline__ void warp_chunk_stats(const uint4& o0, const uint4& o1, int lane, float* dst) {
  float sv[16], sq[16];
  const __half2* q0 = reinterpret_cast<const __half2*>(&o0);
  const __half2* q1 = reinterpret_cast<const __half2*>(&o1);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 x0 = __half22float2(q0[j]);
    const float2 x1 = __half22float2(q1[j]);
    sv[2 * j] = x0.x; sv[2 * j + 1] = x0.y; sv[8 + 2 * j] = x1.x; sv[8 + 2 * j + 1] = x1.y;
  }
#pragma unroll
  for (int j = 0; j < 16; ++j) sq[j] = sv[j] * sv[j];
  warp_xor_step<8>(sv, sq, lane);
  warp_xor_step<4>(sv, sq, lane);
  warp_xor_step<2>(sv, sq, lane);
  warp_xor_step<1>(sv, sq, lane);
  sv[0] += __shfl_xor_sync(0xffffffffu, sv[0], 1);
  sq[0] += __shfl_xor_sync(0xffffffffu, sq[0], 1);
  if ((lane & 1) == 0) {
    const int cidx = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
    const float mean = sv[0] * (1.0f / 32.0f);
    dst[cidx * 2] = mean;
    dst[cidx * 2 + 1] = fmaxf(sq[0] - sv[0] * mean, 0.f);
  }
}

// Final write of one tile's pairs from wq[4 quads][BN][2] (32 rows each, as produced above) into up to two sinks.
// bn = images per tile (1: the four quads belong to image n0, ns = 128; 2: quads 0,1 -> n0 and 2,3 -> n0 + 1, ns = 64).
__device__ __forceinline__ void write_quad_pairs(const float* wq, int BN, int ncols, int col0, int bn, int n0, int Nimg, int slot,
                                                 int slots, const GnSink& s0, const GnSink& s1, int tid, int nthreads) {
  for (int cc = tid; cc < ncols; cc += nthreads) {
    float m[4], q[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { m[k] = wq[((size_t)k * BN + cc) * 2]; q[k] = wq[((size_t)k * BN + cc) * 2 + 1]; }
    float ma, qa, mb, qb;
    chan_merge_equal(32.f, m[0], q[0], m[1], q[1], ma, qa);
    chan_merge_equal(32.f, m[2], q[2], m[3], q[3], mb, qb);
#pragma unroll
    for (int d = 0; d < 2; ++d) {
      const GnSink& s = d == 0 ? s0 : s1;
      if (!s.part) continue;
      const size_t ch = (size_t)s.coff + col0 + cc;
      float* dst = s.part + (((size_t)n0 * slots + slot) * s.cstride + ch) * 2;
      if (bn == 1) {
        float mm, qq;
        chan_merge_equal(64.f, ma, qa, mb, qb, mm, qq);
        dst[0] = mm; dst[1] = qq;
      } else {
        dst[0] = ma; dst[1] = qa;
        if (n0 + 1 < Nimg) {
          float* dst1 = s.part + (((size_t)(n0 + 1) * slots + slot) * s.cstride + ch) * 2;
          dst1[0] = mb; dst1[1] = qb;
        }
      }
    }
  }
}

// Consumer-side combine (GroupNorms whose producers do not finalise: the small UNet levels): (mean, M2) of ONE channel of
// image n over all slots, single pass around the first slot's mean, 16 independent loads in flight.  Returns the
// channel's mean and M2 over slots * ns values.
__device__ __forceinline__ float2 gn_channel_from_pairs(const float* part_nc /* &part[n][0][c][0] */, int slots, int C, float ns) {
  const float pivot = reinterpret_cast<const float2*>(part_nc)->x;
  float s1 = 0.f, s2 = 0.f;
  int sl = 0;
  for (; sl + 16 <= slots; sl += 16) {
    float2 e[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) e[u] = *reinterpret_cast<const float2*>(part_nc + (size_t)(sl + u) * C * 2);
#pragma unroll
    for (int u = 0; u < 16; ++u) { const float d = e[u].x - pivot; s1 += d; s2 += fmaf(ns * d, d, e[u].y); }
  }
  for (; sl + 4 <= slots; sl += 4) {
    float2 e[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) e[u] = *reinterpret_cast<const float2*>(part_nc + (size_t)(sl + u) * C * 2);
#pragma unroll
    for (int u = 0; u < 4; ++u) { const float d = e[u].x - pivot; s1 += d; s2 += fmaf(ns * d, d, e[u].y); }
  }
  for (; sl < slots; ++sl) {
    const float2 e = *reinterpret_cast<const float2*>(part_nc + (size_t)sl * C * 2);
    const float d = e.x - pivot; s1 += d; s2 += fmaf(ns * d, d, e.y);
  }
  const float dm = s1 / (float)slots;
  return make_float2(pivot + dm, fmaxf(s2 - ns * (float)slots * dm * dm, 0.f));
}
// ... and one group from its cpg channels' (mean, M2) (each over cnt values), sequential in channel order
__device__ __forceinline__ float2 gn_group_from_channels(const float* ch_pairs /* [cpg][2] */, int cpg, float cnt, float eps) {
  const float pivot = ch_pairs[0];
  float s1 = 0.f, s2 = 0.f;
  for (int j = 0; j < cpg; ++j) { const float d = ch_pairs[2 * j] - pivot; s1 += d; s2 += fmaf(cnt * d, d, ch_pairs[2 * j + 1]); }
  const float dm = s1 / (float)cpg;
  const float m2 = fmaxf(s2 - cnt * (float)cpg * dm * dm, 0.f);
  return make_float2(pivot + dm, rsqrtf(m2 / (cnt * (float)cpg) + eps));
}

#endif  // __CUDACC__
}  // namespace rs

// Small kernels of the VQ-GAN bookends and the image I/O edges (everything that is not a conv / GroupNorm / GEMM):
// row softmax of the single-head attention, nearest-codebook quantisation, the two tiny 1x1 convs around the quantiser
// (and around the KL first stage's posterior),
// torch-compatible bicubic upsampling, uint8 <-> [-1, 1] conversion with mask blending, overlap-average tile scatter.
#pragma once

#include "common.cuh"

namespace rs {

#ifdef __CUDACC__

// ------------------------------------------------------------------------------------------------
// softmax over the rows of S [rows][cols] fp16 (row stride ld), in place:  P = softmax(scale * S)
// reference: AttnBlock.forward, ldm/modules/diffusionmodules/model.py:190-192 (w_ * c^-0.5, softmax over keys).
// One CTA per row; each thread keeps its (at most 32) elements in registers between the passes.
// ------------------------------------------------------------------------------------------------
constexpr int kSoftmaxMaxCols = 8192;             // the longest row: 256 threads x 4 vectors x 8 halves
struct SoftmaxParams {
  __half* s; long long ld; int rows, cols; float scale;
};
// What the kernel computes correctly: rows that fit in its registers, read and written as 16-byte vectors from a
// 16-byte aligned start.  Anything else would be silently wrong (columns dropped or misaligned), so both the plan and
// the single-operator entry refuse it here.
inline int softmax_rows_check(const SoftmaxParams& p) {
  RS_CHECK(p.s != nullptr && (reinterpret_cast<uintptr_t>(p.s) & 15) == 0, "row softmax: S must be 16-byte aligned");
  RS_CHECK(p.rows >= 1, "row softmax: rows >= 1");
  RS_CHECK(p.cols >= 8 && p.cols <= kSoftmaxMaxCols && p.cols % 8 == 0,
           "row softmax: cols must be a multiple of 8 in [8, 8192], got " + std::to_string(p.cols));
  RS_CHECK(p.ld >= p.cols && p.ld % 8 == 0, "row softmax: row stride ld >= cols and a multiple of 8, got " + std::to_string(p.ld));
  return 0;
}
__global__ void __launch_bounds__(256) softmax_rows_kernel(const SoftmaxParams p) {
  pdl_trigger();
  pdl_wait();
  __shared__ float s_red[8];
  __half* row = p.s + (long long)blockIdx.x * p.ld;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int kMaxVec = kSoftmaxMaxCols / (256 * 8);   // 4 x 8 halves per thread
  uint4 raw[kMaxVec];
  float v[kMaxVec][8];
  const int nvec = p.cols >> 3;
  float mx = -3.0e38f;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int u = tid + i * 256;
    if (u < nvec) {
      raw[i] = *reinterpret_cast<const uint4*>(row + (long long)u * 8);
      const __half2* h = reinterpret_cast<const __half2*>(&raw[i]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]);
        v[i][2 * j] = f.x * p.scale; v[i][2 * j + 1] = f.y * p.scale;
        mx = fmaxf(mx, fmaxf(v[i][2 * j], v[i][2 * j + 1]));
      }
    }
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  if (lane == 0) s_red[warp] = mx;
  __syncthreads();
  mx = s_red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) mx = fmaxf(mx, s_red[w]);
  __syncthreads();
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int u = tid + i * 256;
    if (u < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { v[i][j] = __expf(v[i][j] - mx); sum += v[i][j]; }
    }
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
  if (lane == 0) s_red[warp] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) sum += s_red[w];          // fixed order
  const float inv = 1.0f / sum;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int u = tid + i * 256;
    if (u < nvec) {
      uint4 o;
      __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) oh[j] = __floats2half2_rn(v[i][2 * j] * inv, v[i][2 * j + 1] * inv);
      *reinterpret_cast<uint4*>(row + (long long)u * 8) = o;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// y[n, co, hw] = b[co] + sum_ci w[co, ci] * x[n, ci, hw]   (fp32 NCHW in and out, C <= 8): quant_conv of the encoder
// reference: VQModelTorch.encode, ldm/models/autoencoder.py:28-31 (Conv2d(z_channels, embed_dim, 1)).
// ------------------------------------------------------------------------------------------------
struct PointwiseParams {
  const float* x; float* y; const __half* w; int w_ld; const float* b; int Cin, Cout, N, HW;
};
__global__ void pointwise_conv_f32_kernel(const PointwiseParams p) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)p.N * p.HW) return;
  const int n = (int)(i / p.HW), hw = (int)(i % p.HW);
  float xin[8];
  for (int c = 0; c < p.Cin; ++c) xin[c] = p.x[((long long)n * p.Cin + c) * p.HW + hw];
  for (int co = 0; co < p.Cout; ++co) {
    float acc = p.b[co];
    for (int c = 0; c < p.Cin; ++c) acc = fmaf(__half2float(p.w[co * p.w_ld + c]), xin[c], acc);
    p.y[((long long)n * p.Cout + co) * p.HW + hw] = acc;
  }
}

// ------------------------------------------------------------------------------------------------
// quant_conv and DiagonalGaussianDistribution of the KL first stage in one pass (reference
// ldm/models/autoencoder.py:65-72, ldm/modules/distributions/distributions.py:24-37,61-62):
//   moments = quant_conv(h)                        [N, 2E, HW]  (same fp32 accumulation as pointwise_conv_f32_kernel)
//   mean, logvar = moments[:, :E], clamp(moments[:, E:], -30, 20);  std = exp(0.5 logvar)
//   z = mean + std * noise   (noise given: sample())        z = mean   (noise == nullptr: mode())
// The product and the sum are rounded separately, as torch evaluates `self.mean + self.std * randn`.
// ------------------------------------------------------------------------------------------------
struct KlPosteriorParams {
  const float* h;            // [N, Cin, HW] fp32: the encoder's output (2 z_channels)
  const __half* w; int w_ld; const float* b; int Cin, E;   // quant_conv [2E][Cin] (fp16, row stride w_ld), bias [2E]
  const float* noise;        // [N, E, HW] fp32 or nullptr
  float* z;                  // [N, E, HW]
  float* moments;            // [N, 2E, HW] or nullptr
  int N, HW;
};
__global__ void kl_posterior_kernel(const KlPosteriorParams p) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)p.N * p.HW) return;
  const int n = (int)(i / p.HW), hw = (int)(i % p.HW);
  float xin[16], m[16];
  for (int c = 0; c < p.Cin; ++c) xin[c] = p.h[((long long)n * p.Cin + c) * p.HW + hw];
  for (int co = 0; co < 2 * p.E; ++co) {
    float acc = p.b[co];
    for (int c = 0; c < p.Cin; ++c) acc = fmaf(__half2float(p.w[co * p.w_ld + c]), xin[c], acc);
    m[co] = acc;
    if (p.moments) p.moments[((long long)n * 2 * p.E + co) * p.HW + hw] = acc;
  }
  for (int c = 0; c < p.E; ++c) {
    const long long o = ((long long)n * p.E + c) * p.HW + hw;
    float zc = m[c];
    if (p.noise) {
      const float logvar = fminf(fmaxf(m[p.E + c], -30.0f), 20.0f);
      zc = __fadd_rn(zc, __fmul_rn(expf(0.5f * logvar), p.noise[o]));
    }
    p.z[o] = zc;
  }
}

// ------------------------------------------------------------------------------------------------
// Wide forms of the two kernels above, for latents of 16 to 64 channels (LDM's kl-f16 / kl-f32, 16-channel f8 KL
// autoencoders): a CTA stages a tile of kWideTile positions of one image (NCHW fp32, read coalesced along HW) and the
// whole fp16 weight matrix in shared memory, so nothing is held in per-thread arrays.  Warp w computes output rows
// w, w + 8, ... of the tile, lane = position.  Same arithmetic as the narrow kernels: fp32 input times fp16 weight,
// fmaf from the bias in ascending input-channel order; the KL form computes the mean and logvar rows of channel c in
// the same pass, clamps logvar to [-30, 20] and rounds mean + std * noise as two operations.
// The weight rows are moved as 16-byte vectors: w 16-byte aligned, w_ld a multiple of 8 (the arena's packed rows are).
// ------------------------------------------------------------------------------------------------
constexpr int kWideTile = 32;                      // positions per CTA (one per lane)
constexpr int kWidePointwiseMaxCin = 64, kWidePointwiseMaxCout = 64;
constexpr int kWideKlMaxCin = 128, kWideKlMaxE = 64;
__host__ __device__ constexpr int wide_ldw(int cin) { return (cin + 7) / 8 * 8; }
// dynamic shared memory of a wide launch: the weight rows [rows][ldw] fp16, then the tile [Cin][kWideTile] fp32
__host__ __device__ constexpr size_t wide_1x1_smem(int cin, int rows) {
  return (size_t)rows * wide_ldw(cin) * 2 + (size_t)cin * kWideTile * 4;
}

// stage weight rows [0, rows) and positions [hw0, hw0 + kWideTile) of x (one image, [Cin][HW]); positions past HW read 0
__device__ __forceinline__ void wide_1x1_stage(const float* x, int Cin, int HW, int hw0, const __half* w, int w_ld, int rows,
                                               __half* s_w, float* s_x) {
  const int ldw = wide_ldw(Cin), vrow = ldw / 8;
  for (int v = threadIdx.x; v < rows * vrow; v += blockDim.x) {
    const int r = v / vrow, k = v % vrow;
    reinterpret_cast<uint4*>(s_w)[v] = *reinterpret_cast<const uint4*>(w + (long long)r * w_ld + 8 * k);
  }
  for (int v = threadIdx.x; v < Cin * kWideTile; v += blockDim.x) {
    const int c = v / kWideTile, t = v % kWideTile;
    s_x[v] = hw0 + t < HW ? x[(long long)c * HW + hw0 + t] : 0.f;
  }
  __syncthreads();
}

// pointwise_conv_f32_kernel for 9 <= Cin <= 64 (Cout <= 64); grid (ceil(HW / kWideTile), N), 256 threads
__global__ void __launch_bounds__(256) pointwise_conv_wide_kernel(const PointwiseParams p) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) unsigned char s_raw[];
  __half* s_w = reinterpret_cast<__half*>(s_raw);
  float* s_x = reinterpret_cast<float*>(s_raw + (size_t)p.Cout * wide_ldw(p.Cin) * 2);
  const int n = blockIdx.y, hw0 = blockIdx.x * kWideTile;
  wide_1x1_stage(p.x + (long long)n * p.Cin * p.HW, p.Cin, p.HW, hw0, p.w, p.w_ld, p.Cout, s_w, s_x);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, ldw = wide_ldw(p.Cin);
  if (hw0 + lane >= p.HW) return;
  for (int co = warp; co < p.Cout; co += blockDim.x / 32) {
    const __half* wr = s_w + co * ldw;                         // broadcast reads
    float acc = p.b[co];
    for (int c = 0; c < p.Cin; ++c) acc = fmaf(__half2float(wr[c]), s_x[c * kWideTile + lane], acc);
    p.y[((long long)n * p.Cout + co) * p.HW + hw0 + lane] = acc;
  }
}

// kl_posterior_kernel for Cin > 16 or 2E > 16 (Cin <= 128, E <= 64); grid (ceil(HW / kWideTile), N), 256 threads
__global__ void __launch_bounds__(256) kl_posterior_wide_kernel(const KlPosteriorParams p) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) unsigned char s_raw[];
  __half* s_w = reinterpret_cast<__half*>(s_raw);
  float* s_x = reinterpret_cast<float*>(s_raw + (size_t)2 * p.E * wide_ldw(p.Cin) * 2);
  const int n = blockIdx.y, hw0 = blockIdx.x * kWideTile;
  wide_1x1_stage(p.h + (long long)n * p.Cin * p.HW, p.Cin, p.HW, hw0, p.w, p.w_ld, 2 * p.E, s_w, s_x);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, ldw = wide_ldw(p.Cin);
  const int hw = hw0 + lane;
  if (hw >= p.HW) return;
  for (int c = warp; c < p.E; c += blockDim.x / 32) {
    const __half* wm = s_w + c * ldw;                          // mean row c and logvar row E + c, broadcast reads
    const __half* wl = s_w + (p.E + c) * ldw;
    float am = p.b[c], al = p.b[p.E + c];
    for (int k = 0; k < p.Cin; ++k) {
      const float xv = s_x[k * kWideTile + lane];
      am = fmaf(__half2float(wm[k]), xv, am);
      al = fmaf(__half2float(wl[k]), xv, al);
    }
    if (p.moments) {
      p.moments[((long long)n * 2 * p.E + c) * p.HW + hw] = am;
      p.moments[((long long)n * 2 * p.E + p.E + c) * p.HW + hw] = al;
    }
    const long long o = ((long long)n * p.E + c) * p.HW + hw;
    float zc = am;
    if (p.noise) {
      const float logvar = fminf(fmaxf(al, -30.0f), 20.0f);
      zc = __fadd_rn(zc, __fmul_rn(expf(0.5f * logvar), p.noise[o]));
    }
    p.z[o] = zc;
  }
}

// ------------------------------------------------------------------------------------------------
// VectorQuantizer2.forward (reference ldm/modules/vqvae/quantize.py:271-284) fused with post_quant_conv
// (ldm/models/autoencoder.py:33-38) and the layout change the decoder's first conv wants:
//   idx = argmin_j ( |z|^2 + |e_j|^2 - 2 z.e_j )   (first minimum, fp32)
//   out[pix, :] = post_quant_conv(e_idx)  as NHWC fp16 padded to Cpad channels.
// One thread per latent position; the codebook streams through shared memory in chunks read by the whole CTA.
// With idx_in (VQModelTorch.decode_code, autoencoder.py:42-45) the codes are given: e_idx is gathered from the codebook
// (an index outside [0, n_e) gives NaN at that position) and z is not read.
// ------------------------------------------------------------------------------------------------
struct QuantizeParams {
  const float* z;            // [N, E, HW] fp32
  const float* codebook;     // [n_e, E] fp32
  int n_e, E, N, HW;
  int quantize;              // 0: force_not_quantize (z passes through)
  const __half* pw; int pw_ld; const float* pb; int Cz;   // post_quant_conv [Cz][E] (fp16, row stride pw_ld), bias [Cz]
  __half* out; int Cpad;     // [N*HW, Cpad]
  int* idx_out;              // optional [N, HW]
  const int* idx_in;         // optional [N, HW]: given codes (then quantize must be 0 and z may be null)
};
__global__ void __launch_bounds__(256) vq_quantize_kernel(const QuantizeParams p) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float s_code[];               // [chunk][E + 1]: code, |e|^2
  constexpr int kChunk = 1024;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < (long long)p.N * p.HW;
  const int n = live ? (int)(i / p.HW) : 0, hw = live ? (int)(i % p.HW) : 0;
  float zv[8];
  float zz = 0.f;
  for (int c = 0; c < p.E; ++c) { zv[c] = live && !p.idx_in ? p.z[((long long)n * p.E + c) * p.HW + hw] : 0.f; }
  for (int c = 0; c < p.E; ++c) zz += zv[c] * zv[c];          // torch.sum(z ** 2, dim=1): sequential over E
  int best = 0;
  if (p.quantize) {
    float bestd = 3.0e38f;
    const int stride = p.E + 1;
    for (int j0 = 0; j0 < p.n_e; j0 += kChunk) {
      const int cnt = min(kChunk, p.n_e - j0);
      __syncthreads();
      for (int t = threadIdx.x; t < cnt; t += blockDim.x) {
        float ee = 0.f;
        for (int c = 0; c < p.E; ++c) { const float e = p.codebook[(long long)(j0 + t) * p.E + c]; s_code[t * stride + c] = e; ee += e * e; }
        s_code[t * stride + p.E] = ee;
      }
      __syncthreads();
      for (int t = 0; t < cnt; ++t) {
        const float* e = s_code + t * stride;                  // broadcast reads
        float dot = 0.f;
        for (int c = 0; c < p.E; ++c) dot = fmaf(zv[c], e[c], dot);
        const float d = (zz + e[p.E]) - 2.0f * dot;
        if (d < bestd) { bestd = d; best = j0 + t; }           // strict <: the first minimum wins, like torch.argmin
      }
    }
  }
  if (!live) return;
  float q[8];
  if (p.idx_in) {
    const int code = p.idx_in[i];
    for (int c = 0; c < p.E; ++c) q[c] = code >= 0 && code < p.n_e ? p.codebook[(long long)code * p.E + c] : __int_as_float(0x7fc00000);
  } else {
    for (int c = 0; c < p.E; ++c) q[c] = p.quantize ? p.codebook[(long long)best * p.E + c] : zv[c];
  }
  if (p.idx_out) p.idx_out[i] = p.quantize ? best : -1;
  __half* o = p.out + i * p.Cpad;
  int co = 0;
  for (; co < p.Cz; ++co) {
    float acc = p.pb[co];
    for (int c = 0; c < p.E; ++c) acc = fmaf(__half2float(p.pw[co * p.pw_ld + c]), q[c], acc);
    o[co] = __float2half_rn(acc);
  }
  for (; co < p.Cpad; ++co) o[co] = __float2half_rn(0.f);
}

// ------------------------------------------------------------------------------------------------
// vq_quantize_kernel for E = 16, 24, .., 64 (compile-time, so z stays in registers), Cz <= 64, Cpad = round_up(Cz, 8):
// the same nearest code ((|z|^2 + |e|^2) - 2 z.e in fp32, the first minimum wins), the same decode_code gather (NaN for
// an index outside [0, n_e)), the same post_quant_conv arithmetic (fmaf from the bias in ascending e order), the output
// row written as 16-byte stores.  The codebook streams through shared memory in chunks of kQuantWideChunk<E> codes
// (rows padded to E + 4 floats, |e|^2 beside them: 32 KB), post_quant_conv's rows [Cz][E] fp16 are staged once.
// One thread per latent position, 256 per CTA.  codebook, pw and out must be 16-byte aligned, pw_ld a multiple of 8.
// ------------------------------------------------------------------------------------------------
constexpr int kQuantWideMaxCz = 64;
template <int E>
constexpr int kQuantWideChunk = (32 * 1024 / (4 * (E + 5))) / 32 * 32;
template <int E>
__global__ void __launch_bounds__(256) vq_quantize_wide_kernel(const QuantizeParams p) {
  static_assert(E % 8 == 0 && E >= 16 && E <= 64, "wide quantiser: E a multiple of 8 in [16, 64]");
  constexpr int kChunk = kQuantWideChunk<E>, kLd = E + 4, kV = E / 4;
  __shared__ __align__(16) float s_code[kChunk * kLd];
  __shared__ float s_ee[kChunk];
  __shared__ __align__(16) __half s_w[kQuantWideMaxCz * E];
  __shared__ float s_b[kQuantWideMaxCz];
  pdl_trigger();
  pdl_wait();
  const int cpad = p.Cpad;
  for (int v = threadIdx.x; v < cpad * (E / 8); v += blockDim.x) {      // rows past Cz are zero
    const int r = v / (E / 8), k = v % (E / 8);
    reinterpret_cast<uint4*>(s_w)[v] = r < p.Cz ? *reinterpret_cast<const uint4*>(p.pw + (long long)r * p.pw_ld + 8 * k)
                                                : make_uint4(0u, 0u, 0u, 0u);
  }
  for (int r = threadIdx.x; r < cpad; r += blockDim.x) s_b[r] = r < p.Cz ? p.pb[r] : 0.f;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < (long long)p.N * p.HW;
  const int n = live ? (int)(i / p.HW) : 0, hw = live ? (int)(i % p.HW) : 0;
  float zv[E];
  float zz = 0.f;
#pragma unroll
  for (int c = 0; c < E; ++c) zv[c] = live && !p.idx_in ? p.z[((long long)n * E + c) * p.HW + hw] : 0.f;
#pragma unroll
  for (int c = 0; c < E; ++c) zz += zv[c] * zv[c];           // torch.sum(z ** 2, dim=1): sequential over E
  int best = 0;
  if (p.quantize) {
    float bestd = 3.0e38f;
    for (int j0 = 0; j0 < p.n_e; j0 += kChunk) {
      const int cnt = min(kChunk, p.n_e - j0);
      __syncthreads();
      const float4* src = reinterpret_cast<const float4*>(p.codebook + (long long)j0 * E);
      for (int v = threadIdx.x; v < cnt * kV; v += blockDim.x)                 // coalesced 16-byte reads
        *reinterpret_cast<float4*>(s_code + (v / kV) * kLd + 4 * (v % kV)) = src[v];
      __syncthreads();
      for (int t = threadIdx.x; t < cnt; t += blockDim.x) {
        const float* e = s_code + t * kLd;
        float ee = 0.f;
#pragma unroll
        for (int c = 0; c < E; ++c) ee += e[c] * e[c];
        s_ee[t] = ee;
      }
      __syncthreads();
      for (int t = 0; t < cnt; ++t) {
        const float4* e4 = reinterpret_cast<const float4*>(s_code + t * kLd);   // broadcast reads
        float dot = 0.f;
#pragma unroll
        for (int v = 0; v < kV; ++v) {
          const float4 e = e4[v];
          dot = fmaf(zv[4 * v], e.x, dot); dot = fmaf(zv[4 * v + 1], e.y, dot);
          dot = fmaf(zv[4 * v + 2], e.z, dot); dot = fmaf(zv[4 * v + 3], e.w, dot);
        }
        const float d = (zz + s_ee[t]) - 2.0f * dot;
        if (d < bestd) { bestd = d; best = j0 + t; }           // strict <: the first minimum wins, like torch.argmin
      }
    }
  }
  __syncthreads();                                             // s_w / s_b staged (no chunk loop without quantize)
  if (!live) return;
  // q overwrites z in registers: the code row, the given code's row (NaN when out of range) or z itself
  if (p.idx_in) {
    const int code = p.idx_in[i];
    const bool ok = code >= 0 && code < p.n_e;
#pragma unroll
    for (int c = 0; c < E; ++c) zv[c] = ok ? p.codebook[(long long)code * E + c] : __int_as_float(0x7fc00000);
  } else if (p.quantize) {
#pragma unroll
    for (int c = 0; c < E; ++c) zv[c] = p.codebook[(long long)best * E + c];
  }
  if (p.idx_out) p.idx_out[i] = p.quantize ? best : -1;
  uint4* o = reinterpret_cast<uint4*>(p.out + i * cpad);
  for (int co0 = 0; co0 < cpad; co0 += 8) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = s_b[co0 + j];
#pragma unroll
    for (int c = 0; c < E; ++c) {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaf(__half2float(s_w[(co0 + j) * E + c]), zv[c], acc[j]);
    }
    uint4 u;
    __half* h = reinterpret_cast<__half*>(&u);
#pragma unroll
    for (int j = 0; j < 8; ++j) h[j] = __float2half_rn(co0 + j < p.Cz ? acc[j] : 0.f);
    o[co0 / 8] = u;
  }
}

// ------------------------------------------------------------------------------------------------
// Bicubic upsampling by an integer factor, fp32 NCHW, identical to F.interpolate(mode='bicubic', align_corners=False)
// (A = -0.75, source index (dst + 0.5) / sf - 0.5, border pixels clamped) — the pre-upsample of encode_first_stage
// (reference models/gaussian_diffusion.py:503-504).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cubic_weights(float t, float (&w)[4]) {
  const float A = -0.75f;
  // same polynomial forms as ATen's cubic_convolution1 / cubic_convolution2 (UpSample.h)
  auto c1 = [&](float x) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; };
  auto c2 = [&](float x) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; };
  w[0] = c2(t + 1.f); w[1] = c1(t); w[2] = c1(1.f - t); w[3] = c2(2.f - t);
}
struct BicubicParams { const float* x; float* y; int NC, H, W, sf; };
__global__ void bicubic_upsample_kernel(const BicubicParams p) {
  pdl_trigger();
  pdl_wait();
  const int OW = p.W * p.sf, OH = p.H * p.sf;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)p.NC * OH * OW) return;
  const int ox = (int)(i % OW), oy = (int)((i / OW) % OH);
  const long long nc = i / ((long long)OW * OH);
  const float scale = 1.0f / (float)p.sf;
  const float sx = scale * ((float)ox + 0.5f) - 0.5f, sy = scale * ((float)oy + 0.5f) - 0.5f;
  const float fx = floorf(sx), fy = floorf(sy);
  const int ix = (int)fx, iy = (int)fy;
  float wx[4], wy[4];
  cubic_weights(sx - fx, wx);
  cubic_weights(sy - fy, wy);
  const float* src = p.x + nc * (long long)p.H * p.W;
  float acc = 0.f;
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int yy = min(max(iy - 1 + a, 0), p.H - 1);
    float r = 0.f;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int xx = min(max(ix - 1 + b, 0), p.W - 1);
      r += src[(long long)yy * p.W + xx] * wx[b];
    }
    acc += r * wy[a];
  }
  p.y[i] = acc;
}

__global__ void zero_u32_kernel(unsigned int* ptr, int n) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ptr[i] = 0u;
}

// ------------------------------------------------------------------------------------------------
// Image I/O edges (reference sampler.py:218-223,286 + utils/util_image.py:216-273 tensor2img / imwrite):
//   ingest:  uint8 HWC (RGB, 1 or 3 channels) -> fp32 NCHW in [-1, 1]      ((v / 255 - 0.5) / 0.5)
//   emit:    fp32 NCHW in [-1, 1] -> clamp -> * 0.5 + 0.5 -> optional mask-back blend with the LQ image -> uint8 HWC
//            (round(v * 255), as tensor2img does: (x * 255).round() of the [0, 1]-clamped value), RGB or BGR order
// ------------------------------------------------------------------------------------------------
struct IngestParams { const uint8_t* src; float* dst; int N, H, W, C; };
__global__ void ingest_u8_kernel(const IngestParams p) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // over N*H*W pixels
  if (i >= (long long)p.N * p.H * p.W) return;
  const long long n = i / ((long long)p.H * p.W), hw = i % ((long long)p.H * p.W);
  for (int c = 0; c < p.C; ++c) {
    const float v = (float)p.src[i * p.C + c] / 255.0f;
    p.dst[(n * p.C + c) * (long long)p.H * p.W + hw] = (v - 0.5f) / 0.5f;
  }
}
struct EmitParams {
  const float* sr;           // [N, 3, H, W] in [-1, 1] (un-clamped)
  const float* lq;           // optional [N, 3, H, W] in [-1, 1]: mask-back source
  const float* mask;         // optional [N, 1, H, W] in [-1, 1] (1 = unknown area: keep the model output there)
  uint8_t* dst;              // [N, H, W, 3]
  int N, H, W, bgr;
};
__global__ void emit_u8_kernel(const EmitParams p) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long HW = (long long)p.H * p.W;
  if (i >= (long long)p.N * HW) return;
  const long long n = i / HW, hw = i % HW;
  const float m = p.mask ? p.mask[n * HW + hw] * 0.5f + 0.5f : 1.0f;
  for (int c = 0; c < 3; ++c) {
    float v = fminf(fmaxf(p.sr[(n * 3 + c) * HW + hw], -1.0f), 1.0f) * 0.5f + 0.5f;
    if (p.mask) v = v * m + (p.lq[(n * 3 + c) * HW + hw] * 0.5f + 0.5f) * (1.0f - m);
    v = fminf(fmaxf(v, 0.0f), 1.0f);
    p.dst[i * 3 + (p.bgr ? 2 - c : c)] = (uint8_t)__float2int_rn(v * 255.0f);
  }
}

// ------------------------------------------------------------------------------------------------
// Overlap-average of tiled results (reference ImageSpliterTh.update / gather, utils/util_image.py:962-979): every output
// pixel is the mean of the tiles that cover it.  Gather form (no atomics, deterministic): one thread per output pixel
// walks the tile grid; tiles are [T, N, C, th, tw] with tile t = ty * ntx + tx at (ys[ty], xs[tx]) in output pixels.
// ------------------------------------------------------------------------------------------------
struct TileGatherParams {
  const float* tiles; float* out;
  int N, C, H, W;            // output
  int th, tw, nty, ntx;
  const int* ys; const int* xs;   // [nty], [ntx] tile origins (output pixels), ascending
};
__global__ void tile_gather_kernel(const TileGatherParams p) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long HW = (long long)p.H * p.W;
  if (i >= (long long)p.N * p.C * HW) return;
  const int x = (int)(i % p.W), y = (int)((i / p.W) % p.H);
  const long long nc = i / HW;
  const long long tstride = (long long)p.N * p.C * p.th * p.tw;
  float acc = 0.f;
  int cnt = 0;
  for (int ty = 0; ty < p.nty; ++ty) {
    const int ly = y - p.ys[ty];
    if (ly < 0 || ly >= p.th) continue;
    for (int tx = 0; tx < p.ntx; ++tx) {
      const int lx = x - p.xs[tx];
      if (lx < 0 || lx >= p.tw) continue;
      acc += p.tiles[(long long)(ty * p.ntx + tx) * tstride + (nc * p.th + ly) * p.tw + lx];
      ++cnt;
    }
  }
  p.out[i] = acc / (float)cnt;
}

#endif
}  // namespace rs

// Small HBM/latency-bound kernels around the GEMMs: input packing, nearest upsample, timestep
// embedding MLP, the residual-shift sampling update, and weight repacking.
#pragma once

#include "common.cuh"
#include "gn_stats.cuh"

namespace rs {

#ifdef __CUDACC__

// ------------------------------------------------------------------------------------------------
// UNet input: cat([x * in_scale, lq], dim=1) in NCHW fp32  ->  NHWC fp16 with channels padded to Cpad.
// reference: _scale_input (models/gaussian_diffusion.py:598-603) + th.cat (models/unet.py:882).
// The LQ part is either raw NCHW fp32 (realsr: feature_extractor is Identity, unet.py:689-691) or an
// NHWC fp16 feature map produced by the feature extractor.
// ------------------------------------------------------------------------------------------------
struct PackInputParams {
  const float* x; int Cx;             // [N, Cx, H, W] fp32
  const float* scale_tab; int scale_idx;   // optional per-step table; value 1/sqrt(eta*kappa^2+1)
  const float* lq_nchw; int Cl;       // [N, Cl, H, W] fp32 or nullptr
  const float* mask_nchw;             // [N, 1, H, W] fp32 after lq_nchw (cond_mask without feature extractor) or nullptr
  const __half* lq_nhwc; int lq_ld;   // [N*H*W, Cl] fp16 or nullptr
  __half* out; int Cpad;              // [N*H*W, Cpad]
  int N, HW;
  int lq_unshuffle, W;                // 1: lq_nchw is [N, Cl / 4, 2H, 2W], packed as F.pixel_unshuffle(lq, 2) (channel 4c + 2dy + dx)
  unsigned int* zero_ptr; int zero_n; // GroupNorm arrival counters of the forward that follows (gn_stats.cuh): reset here
};

__global__ void pack_input_kernel(const PackInputParams p) {
  pdl_trigger();
  pdl_wait();
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix < p.zero_n) p.zero_ptr[pix] = 0u;
  const long long total = (long long)p.N * p.HW;
  if (pix >= total) return;
  const int n = (int)(pix / p.HW);
  const int hw = (int)(pix % p.HW);
  const float sc = p.scale_tab ? p.scale_tab[p.scale_idx] : 1.0f;
  __half* o = p.out + pix * p.Cpad;
  int c = 0;
  for (; c < p.Cx; ++c) o[c] = __float2half_rn(p.x[((long long)n * p.Cx + c) * p.HW + hw] * sc);
  if (p.lq_nchw && p.lq_unshuffle) {
    const int y = hw / p.W, xx = hw % p.W;
    const long long W2 = 2LL * p.W, plane = 4LL * p.HW;
    for (int j = 0; j < p.Cl; ++j, ++c)
      o[c] = __float2half_rn(p.lq_nchw[((long long)n * (p.Cl / 4) + j / 4) * plane + (2 * y + ((j >> 1) & 1)) * W2 + 2 * xx + (j & 1)]);
  } else if (p.lq_nchw) {
    for (int j = 0; j < p.Cl; ++j, ++c) o[c] = __float2half_rn(p.lq_nchw[((long long)n * p.Cl + j) * p.HW + hw]);
    if (p.mask_nchw) o[c++] = __float2half_rn(p.mask_nchw[(long long)n * p.HW + hw]);
  } else if (p.lq_nhwc) {
    for (int j = 0; j < p.Cl; ++j, ++c) o[c] = p.lq_nhwc[pix * p.lq_ld + j];
  }
  for (; c < p.Cpad; ++c) o[c] = __float2half_rn(0.f);
}

// NCHW fp32 image (+ optional mask) -> NHWC fp16, channels padded: input of the feature extractor
// (reference models/unet.py:876-881: th.cat([lq, mask], dim=1)).
struct PackImageParams {
  const float* a; int Ca;
  const float* b; int Cb;
  __half* out; int Cpad;
  int N, HW;
};
__global__ void pack_image_kernel(const PackImageParams p) {
  pdl_trigger();
  pdl_wait();
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long long)p.N * p.HW) return;
  const int n = (int)(pix / p.HW);
  const int hw = (int)(pix % p.HW);
  __half* o = p.out + pix * p.Cpad;
  int c = 0;
  for (int j = 0; j < p.Ca; ++j, ++c) o[c] = __float2half_rn(p.a[((long long)n * p.Ca + j) * p.HW + hw]);
  for (int j = 0; j < p.Cb; ++j, ++c) o[c] = __float2half_rn(p.b[((long long)n * p.Cb + j) * p.HW + hw]);
  for (; c < p.Cpad; ++c) o[c] = __float2half_rn(0.f);
}

// ------------------------------------------------------------------------------------------------
// 2x resampling, NHWC fp16 views, 16-byte vectors: nearest x2 upsample (reference Upsample.forward,
// models/unet.py:71-81) and 2x2 average pool (Downsample without conv, avg_pool2d, :83-108)
// ------------------------------------------------------------------------------------------------
struct UpsampleParams {
  const __half* x; long long x_sN; int x_ld;   // [N, H, W, C] view (the input, for both directions)
  __half* y; long long y_sN; int y_ld;         // [N, 2H, 2W, C] (upsample) or [N, H/2, W/2, C] (pool) view
  int N, H, W, C;
  __half* s; long long s_sN; int s_ld;         // optional second output on y's grid: SiLU of every fp16 value stored to y
};
__device__ __forceinline__ uint4 silu_h8(uint4 v) {
  __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
  for (int k = 0; k < 4; ++k) { const float2 f = __half22float2(h[k]); h[k] = __floats2half2_rn(silu_f(f.x), silu_f(f.y)); }
  return v;
}
__global__ void avgpool2x2_kernel(const UpsampleParams p) {
  pdl_trigger();
  pdl_wait();
  const int vecs = p.C >> 3, Ho = p.H / 2, Wo = p.W / 2;
  const long long total = (long long)p.N * Ho * Wo * vecs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vecs);
    long long q = i / vecs;
    const int ox = (int)(q % Wo); q /= Wo;
    const int oy = (int)(q % Ho); q /= Ho;
    const int n = (int)q;
    const __half* src = p.x + n * p.x_sN + ((long long)(2 * oy) * p.W + 2 * ox) * p.x_ld + v * 8;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint4 raw = *reinterpret_cast<const uint4*>(src + ((long long)(k >> 1) * p.W + (k & 1)) * p.x_ld);
      const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
      for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h[j]); acc[2 * j] += f.x; acc[2 * j + 1] += f.y; }
    }
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) oh[j] = __floats2half2_rn(0.25f * acc[2 * j], 0.25f * acc[2 * j + 1]);
    *reinterpret_cast<uint4*>(p.y + n * p.y_sN + ((long long)oy * Wo + ox) * p.y_ld + v * 8) = o;
    if (p.s) *reinterpret_cast<uint4*>(p.s + n * p.s_sN + ((long long)oy * Wo + ox) * p.s_ld + v * 8) = silu_h8(o);
  }
}
__global__ void upsample2x_kernel(const UpsampleParams p) {
  pdl_trigger();
  pdl_wait();
  const int vecs = p.C >> 3;
  const long long total = (long long)p.N * (2 * p.H) * (2 * p.W) * vecs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vecs);
    long long q = i / vecs;
    const int ox = (int)(q % (2 * p.W)); q /= 2 * p.W;
    const int oy = (int)(q % (2 * p.H)); q /= 2 * p.H;
    const int n = (int)q;
    const uint4 raw = *reinterpret_cast<const uint4*>(p.x + n * p.x_sN + ((long long)(oy >> 1) * p.W + (ox >> 1)) * p.x_ld + v * 8);
    *reinterpret_cast<uint4*>(p.y + n * p.y_sN + ((long long)oy * 2 * p.W + ox) * p.y_ld + v * 8) = raw;
    if (p.s) *reinterpret_cast<uint4*>(p.s + n * p.s_sN + ((long long)oy * 2 * p.W + ox) * p.s_ld + v * 8) = silu_h8(raw);
  }
}

// ------------------------------------------------------------------------------------------------
// Timestep path (reference timestep_embedding, models/basic_ops.py:99-117; time_embed, models/unet.py:683-687;
// ResBlock.emb_layers = SiLU -> Linear, models/unet.py:161-167).  Tiny: one warp per output element.
// ------------------------------------------------------------------------------------------------
__global__ void timestep_embedding_kernel(const float* __restrict__ t, float* __restrict__ out, int B, int dim) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int half_dim = dim / 2;
  if (i >= B * half_dim) return;
  const int b = i / half_dim, k = i % half_dim;
  const float freq = expf(-logf(10000.0f) * (float)k / (float)half_dim);
  const float a = t[b] * freq;
  out[(long long)b * dim + k] = cosf(a);
  out[(long long)b * dim + half_dim + k] = sinf(a);
  if ((dim & 1) && k == 0) out[(long long)b * dim + dim - 1] = 0.f;
}

// out = a + b (fp32, load time: the folded bias of a ResBlock without scale-shift norm)
__global__ void add_f32_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int n) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i] + b[i];
}

// out[b, o] = bias[o] + sum_k act(x[b, k]) * W[o, k];  W fp16 row-major [O, K], x/out fp32.
__global__ void linear_small_kernel(const float* __restrict__ x, const __half* __restrict__ W,
                                    const float* __restrict__ bias, float* __restrict__ out, int B, int K, int O,
                                    int silu_in, int silu_out) {
  pdl_trigger();
  pdl_wait();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= B * O) return;
  const int b = warp / O, o = warp % O;
  const float* xr = x + (long long)b * K;
  const __half* wr = W + (long long)o * K;
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) {
    float xv = xr[k];
    if (silu_in) xv = silu_f(xv);
    acc = fmaf(xv, __half2float(wr[k]), acc);
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (lane == 0) {
    acc += bias[o];
    if (silu_out) acc = silu_f(acc);
    out[(long long)b * O + o] = acc;
  }
}

// ------------------------------------------------------------------------------------------------
// The sampler's step: one kernel family for the four processes the loop runs, fp32 NCHW in/out.  Every instance
// resets the next forward's GroupNorm arrival counters, turns the model output into x0 by its mean type, applies the
// process's update, writes x_next and, when `next_in` is set (the host leaves it NULL on a process's last step),
// emits the NEXT denoiser input x_next (times in_scale[t-1] for ResShift) as NHWC fp16 in channels [0, C).
//
// ResShift (reference p_sample, models/gaussian_diffusion.py:332-365, with q_posterior_mean_variance :210-232):
//     x_{t-1} = coef1[t] * x_t + coef2[t] * x0 + [t != 0] * std[t] * noise
// x0 by the parameterisation MT (reference p_mean_variance :277-292 and _predict_xstart_from_* :308-324), op by op in
// the reference's order with no FMA contraction:
//     xstart        x0 = out
//     residual      x0 = y - out
//     epsilon       x0 = ((x_t - eps_coef[t] * out) - eta[t] * y) / one_minus_eta[t]
//     epsilon_scale x0 = ((x_t - out) - eta[t] * y) / one_minus_eta[t]
// with eps_coef = fp32(fp32(sqrt_eta) * kappa), eta = fp32(eta), one_minus_eta = fp32(1 - eta) (_extract_into_tensor
// tables), so x0 is bit for bit the reference's fp32 expression.  The xstart instance writes no x0 (it is `out`).
//
// GaussianDiffusionDDPM (reference models/gaussian_diffusion.py:742-1066); the denoiser sees x_t unscaled
// (_scale_input is the identity, :1213-1214):
//   x0       = sqrt_recip_acp[t] x_t - sqrt_recipm1_acp[t] eps (_predict_xstart_from_eps :838-843), or the model
//              output itself for x0 prediction; clamped to [-1, 1] with clip (process_xstart :803-808)
//   ancestral  mean = coef1[t] x0 + coef2[t] x_t (q_posterior_mean_variance :726-729);
//              x_{t-1} = mean + [t != 0] exp(0.5 log_variance[t]) noise (p_sample :887-891)
//   DDIM       eps' = (sqrt_recip_acp[t] x_t - x0) / sqrt_recipm1_acp[t] (_predict_eps_from_xstart :855-859);
//              sigma = eta sqrt((1 - acp_prev) / (1 - acp)) sqrt(1 - acp / acp_prev);
//              x_{t-1} = x0 sqrt(acp_prev) + sqrt(1 - acp_prev - sigma^2) eps' + [t != 0] sigma noise (ddim_sample
//              :1010-1027)
//   inversion  eps' as DDIM; x_{t+1} = x0 sqrt(acp_next[t]) + sqrt(1 - acp_next[t]) eps' (ddim_reverse_sample
//              :1054-1064), t walking 0 .. T-1 upward; acp_next[T-1] is 0, so the last step returns eps'; nothing is drawn
// Every operation is the reference's fp32 tensor operation on the fp32 table values (_extract_into_tensor), in its
// order and rounded on its own (no FMA contraction); the [t != 0] factor multiplies as the reference's nonzero_mask does.
//
// A learned-variance model (learn_sigma: LEARNED / LEARNED_RANGE, p_mean_variance :772-786) outputs 2C channels: the
// mean half [0, C) is read as above, at the image stride out_sN, and the ancestral step takes its log variance from the
// variance half v = out[C + c] instead of the kDdLogVar row:
//   LEARNED        log_var = v
//   LEARNED_RANGE  frac = (v + 1) / 2;  log_var = frac * log(betas)[t] + (1 - frac) * posterior_log_variance_clipped[t]
// DDIM and inversion never read the variance half.  The fixed instances (VAR = kVarFixed) read a [N, C, HW] output at i.
// ------------------------------------------------------------------------------------------------
enum MeanType : int { kMeanXstart = 0, kMeanEpsilon = 1, kMeanEpsilonScale = 2, kMeanResidual = 3 };
enum StepProcess : int { kStepResShift = 0, kStepAncestral = 1, kStepDdim = 2, kStepInversion = 3 };
// the model output's layout and, for the ancestral step, where its log variance comes from; DDIM and inversion run
// every 2C-output model as kVarLearned (they read the mean half only)
enum StepVar : int { kVarFixed = 0, kVarLearned = 1, kVarLearnedRange = 2 };

// The step's [T] fp32 tables, by process: row[r] is the table the plan's table region holds at r * 1024.  kDdLogVar
// holds the fixed log variance, or LEARNED_RANGE's min_log (posterior_log_variance_clipped); kDdLogBetas (its max_log)
// is read by LEARNED_RANGE only.
enum ResShiftRow : int { kRsCoef1 = 0, kRsCoef2, kRsStd, kRsInScale, kRsEpsCoef, kRsEta, kRsOneMinusEta, kRsRows };
enum DdpmRow : int {
  kDdSqrtRecipAcp = 0, kDdSqrtRecipm1Acp, kDdCoef1, kDdCoef2, kDdLogVar, kDdAcp, kDdAcpPrev, kDdLogBetas, kDdRows
};
enum InversionRow : int { kInvSqrtRecipAcp = 0, kInvSqrtRecipm1Acp, kInvAcpNext, kInvRows };
constexpr int kStepRows = 8;

struct StepParams {
  const float* x_t;       // [N, C, HW]
  const float* out;       // [N, C, HW] (kVarFixed), or [N, >= 2C, HW] at image stride out_sN: the model output
  const float* y;         // [N, C, HW] z_y: read by the ResShift residual and epsilon types
  const float* noise;     // [N, C, HW]: not read by inversion
  float* x_next;          // [N, C, HW]
  float* x0_out;          // optional [N, C, HW]: x0 (not written by the ResShift xstart instance)
  const float* row[kStepRows];        // [T] fp32 tables, indexed by the process's row enum
  float eta;              // DDIM
  int clip;               // DDPM processes: clamp x0 to [-1, 1]
  int t;                  // schedule index of THIS step
  int N, C, HW;
  __half* next_in; int next_cpad;     // optional: [N*HW, next_cpad]; channels [0, C) are written here
  unsigned int* zero_ptr; int zero_n; // GroupNorm arrival counters of the NEXT denoiser forward: reset here
  long long out_sN;       // the model output's image stride in elements: C * HW, or 2C * HW for a learned variance
  int var_mode;           // StepVar of the ancestral step (launch_step picks the instance by it and out_sN)
};

template <int MT>
__device__ __forceinline__ float predict_xstart(const StepParams& p, long long i, float xt) {
  if constexpr (MT == kMeanResidual) {
    return __fsub_rn(p.y[i], p.out[i]);
  } else if constexpr (MT == kMeanEpsilon) {
    const float num = __fsub_rn(__fsub_rn(xt, __fmul_rn(p.row[kRsEpsCoef][p.t], p.out[i])), __fmul_rn(p.row[kRsEta][p.t], p.y[i]));
    return __fdiv_rn(num, p.row[kRsOneMinusEta][p.t]);
  } else {
    static_assert(MT == kMeanEpsilonScale, "unknown mean type");
    const float num = __fsub_rn(__fsub_rn(xt, p.out[i]), __fmul_rn(p.row[kRsEta][p.t], p.y[i]));
    return __fdiv_rn(num, p.row[kRsOneMinusEta][p.t]);
  }
}

template <int PROCESS, int MT, int VAR = kVarFixed>
__global__ void step_kernel(const StepParams p) {
  static_assert(VAR == kVarFixed || PROCESS != kStepResShift, "the ResShift process has no learned variance");
  static_assert(VAR != kVarLearnedRange || PROCESS == kStepAncestral, "only the ancestral step reads the variance half");
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < p.zero_n) p.zero_ptr[i] = 0u;
  const long long total = (long long)p.N * p.C * p.HW;
  if (i >= total) return;
  const int t = p.t;
  const float xt = p.x_t[i];
  // where element i's mean value sits in the model output: i itself, or the same (c, hw) of image n at stride out_sN
  long long io = i;
  if constexpr (VAR != kVarFixed) {
    const long long img = (long long)p.C * p.HW;
    io = i + (i / img) * (p.out_sN - img);
  }
  // x0 (eps prediction) and eps' (DDIM, inversion) factors of the DDPM processes, read once ahead of the x0_out store
  const float sra = p.row[kDdSqrtRecipAcp][t], srm1 = p.row[kDdSqrtRecipm1Acp][t];
  float x0;
  if constexpr (PROCESS == kStepResShift) {
    if constexpr (MT == kMeanXstart) x0 = p.out[i];
    else x0 = predict_xstart<MT>(p, i, xt);
  } else {
    static_assert(MT == kMeanEpsilon || MT == kMeanXstart, "DDPM steps predict eps or x0");
    if constexpr (MT == kMeanEpsilon)
      x0 = __fsub_rn(__fmul_rn(sra, xt), __fmul_rn(srm1, p.out[io]));
    else x0 = p.out[io];
    if (p.clip) x0 = x0 < -1.0f ? -1.0f : (x0 > 1.0f ? 1.0f : x0);     // clamp(-1, 1): NaN stays NaN
  }
  if constexpr (PROCESS != kStepResShift || MT != kMeanXstart) {
    if (p.x0_out) p.x0_out[i] = x0;
  }
  float v;
  if constexpr (PROCESS == kStepResShift) {
    const float c1 = p.row[kRsCoef1][t], c2 = p.row[kRsCoef2][t];
    v = c1 * xt + c2 * x0;
    if (t != 0) v += p.row[kRsStd][t] * p.noise[i];
  } else if constexpr (PROCESS == kStepAncestral) {
    const float nonzero = t != 0 ? 1.0f : 0.0f;
    const float mean = __fadd_rn(__fmul_rn(p.row[kDdCoef1][t], x0), __fmul_rn(p.row[kDdCoef2][t], xt));
    float log_var;
    if constexpr (VAR == kVarFixed) {
      log_var = p.row[kDdLogVar][t];
    } else {
      const float v = p.out[io + (long long)p.C * p.HW];          // the variance half
      if constexpr (VAR == kVarLearned) {
        log_var = v;
      } else {
        // (v + 1) / 2: halving is exact, so the product by 0.5 is the reference's division bit for bit
        const float frac = __fmul_rn(__fadd_rn(v, 1.0f), 0.5f);
        log_var = __fadd_rn(__fmul_rn(frac, p.row[kDdLogBetas][t]), __fmul_rn(__fsub_rn(1.0f, frac), p.row[kDdLogVar][t]));
      }
    }
    const float sd = expf(__fmul_rn(0.5f, log_var));
    v = __fadd_rn(mean, __fmul_rn(__fmul_rn(nonzero, sd), p.noise[i]));
  } else {
    static_assert((int)kDdSqrtRecipAcp == (int)kInvSqrtRecipAcp && (int)kDdSqrtRecipm1Acp == (int)kInvSqrtRecipm1Acp,
                  "DDIM and inversion keep the eps' rows in the same place");
    const float eps = __fdiv_rn(__fsub_rn(__fmul_rn(sra, xt), x0), srm1);
    if constexpr (PROCESS == kStepDdim) {
      const float nonzero = t != 0 ? 1.0f : 0.0f;
      const float ab = p.row[kDdAcp][t], abp = p.row[kDdAcpPrev][t];
      const float sigma = __fmul_rn(__fmul_rn(p.eta, __fsqrt_rn(__fdiv_rn(__fsub_rn(1.0f, abp), __fsub_rn(1.0f, ab)))),
                                    __fsqrt_rn(__fsub_rn(1.0f, __fdiv_rn(ab, abp))));
      const float mean = __fadd_rn(__fmul_rn(x0, __fsqrt_rn(abp)),
                                   __fmul_rn(__fsqrt_rn(__fsub_rn(__fsub_rn(1.0f, abp), __fmul_rn(sigma, sigma))), eps));
      v = __fadd_rn(mean, __fmul_rn(__fmul_rn(nonzero, sigma), p.noise[i]));
    } else {
      static_assert(PROCESS == kStepInversion, "unknown step process");
      const float an = p.row[kInvAcpNext][t];
      v = __fadd_rn(__fmul_rn(x0, __fsqrt_rn(an)), __fmul_rn(__fsqrt_rn(__fsub_rn(1.0f, an)), eps));
    }
  }
  p.x_next[i] = v;
  if (p.next_in) {
    const float vin = PROCESS == kStepResShift ? v * p.row[kRsInScale][t - 1] : v;
    const int hw = (int)(i % p.HW);
    const int c = (int)((i / p.HW) % p.C);
    const int n = (int)(i / ((long long)p.HW * p.C));
    p.next_in[((long long)n * p.HW + hw) * p.next_cpad + c] = __float2half_rn(vin);
  }
}

// prior_sample (reference models/gaussian_diffusion.py:517-529): x_T = z_y + kappa*sqrt_eta_T * noise
__global__ void prior_sample_kernel(const float* __restrict__ zy, const float* __restrict__ noise,
                                    float* __restrict__ out, float coef, long long total) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) out[i] = zy[i] + coef * noise[i];
}

// ------------------------------------------------------------------------------------------------
// Split-K finish: out = act(sum_s partial[s] + bias) + residual, fp16 NHWC view (or fp32 NCHW), plus the
// GroupNorm partial statistics of the result.  One CTA per (128-pixel slot, image) — the same slots the
// conv epilogue would have produced; splits are summed in a fixed order, statistics reduced in a fixed tree.
// ------------------------------------------------------------------------------------------------
struct SplitKReduceParams {
  const float* partial;     // [S][N*HW][C]
  int S, N, HW, C;
  const float* bias; int bias_sN;         // bias_sN > 0: one bias row per image
  const __half* residual; long long res_sN; int res_ld;
  __half* out; long long out_sN; int out_ld;
  int act;
  int rows_per_slot, slots;
  int cols_per_cta;         // multiple of 8; grid.z = ceil(C / cols_per_cta)
  GnSink sink[2];           // fused GroupNorm statistics of the result (gn_stats.cuh)
  __half* silu_out; long long silu_sN; int silu_ld;   // optional: SiLU of the stored fp16 result (ConvParams::silu_out)
  const float* film; int film_sN;                     // optional FiLM after the activation (ConvParams::film)
};

__global__ void __launch_bounds__(256) splitk_reduce_kernel(const __grid_constant__ SplitKReduceParams p) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float s_red[];       // [lanes][cols_per_cta][3] = (rows, mean, M2) per row-lane and column
  const int c_begin = blockIdx.z * p.cols_per_cta;
  const int ccols = min(p.cols_per_cta, p.C - c_begin);
  const int vecs = ccols >> 3;
  const int lanes = blockDim.x / vecs;
  const int n = blockIdx.y, slot = blockIdx.x;
  const int vec = threadIdx.x % vecs, rl = threadIdx.x / vecs;
  const long long npix = (long long)p.N * p.HW;
  const bool want_stats = p.sink[0].part != nullptr;
  if (rl < lanes) {
    // statistics of the stored values around a pivot (this thread's first row): no cancellation for |mean| >> std
    float pv[8], s1[8], s2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { pv[j] = 0.f; s1[j] = 0.f; s2[j] = 0.f; }
    int cnt = 0;
    const int r0 = slot * p.rows_per_slot, r1 = min(r0 + p.rows_per_slot, p.HW);
    const int c = c_begin + vec * 8;
    float bs[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) bs[j] = p.bias ? p.bias[n * p.bias_sN + c + j] : 0.f;
    for (int r = r0 + rl; r < r1; r += lanes) {
      const long long pix = (long long)n * p.HW + r;
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
      for (int s = 0; s < p.S; ++s) {
        const float4* src = reinterpret_cast<const float4*>(p.partial + ((long long)s * npix + pix) * p.C + c);
        const float4 a = src[0], b = src[1];
        acc[0] += a.x; acc[1] += a.y; acc[2] += a.z; acc[3] += a.w;
        acc[4] += b.x; acc[5] += b.y; acc[6] += b.z; acc[7] += b.w;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float v = acc[j] + bs[j];
        if (p.act == 1) v = gelu_erf_f(v); else if (p.act == 2) v = silu_f(v);
        acc[j] = v;
      }
      if (p.residual) {
        const uint4 raw = *reinterpret_cast<const uint4*>(p.residual + n * p.res_sN + (long long)r * p.res_ld + c);
        const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h[j]); acc[2 * j] += f.x; acc[2 * j + 1] += f.y; }
      }
      uint4 o;
      __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) oh[j] = __floats2half2_rn(acc[2 * j], acc[2 * j + 1]);
      *reinterpret_cast<uint4*>(p.out + n * p.out_sN + (long long)r * p.out_ld + c) = o;
      if (want_stats) {
        float st[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(oh[j]); st[2 * j] = f.x; st[2 * j + 1] = f.y; }
        if (cnt == 0) {
#pragma unroll
          for (int j = 0; j < 8; ++j) pv[j] = st[j];
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) { const float d = st[j] - pv[j]; s1[j] += d; s2[j] = fmaf(d, d, s2[j]); }
        }
        ++cnt;
      }
    }
    if (p.film || p.silu_out) {
      // FiLM on the stored fp16 values and their SiLU, in a pass of their own over this thread's rows (as the conv
      // epilogue does; conv_finalize gives FiLM neither a residual nor statistics sinks)
      float fs[8], fh[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        fs[j] = p.film ? 1.f + p.film[(long long)n * p.film_sN + c + j] : 1.f;
        fh[j] = p.film ? p.film[(long long)n * p.film_sN + p.C + c + j] : 0.f;
      }
      for (int r = r0 + rl; r < r1; r += lanes) {
        uint4* dst = reinterpret_cast<uint4*>(p.out + n * p.out_sN + (long long)r * p.out_ld + c);
        uint4 o = *dst;
        if (p.film) {
          __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(oh[j]);
            oh[j] = __floats2half2_rn(fmaf(f.x, fs[2 * j], fh[2 * j]), fmaf(f.y, fs[2 * j + 1], fh[2 * j + 1]));
          }
          *dst = o;
        }
        if (p.silu_out) *reinterpret_cast<uint4*>(p.silu_out + n * p.silu_sN + (long long)r * p.silu_ld + c) = silu_h8(o);
      }
    }
    if (want_stats) {
      float* dst = s_red + ((size_t)rl * ccols + vec * 8) * 3;
      const float inv = cnt ? 1.0f / (float)cnt : 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        dst[3 * j] = (float)cnt;
        dst[3 * j + 1] = pv[j] + s1[j] * inv;
        dst[3 * j + 2] = fmaxf(s2[j] - s1[j] * s1[j] * inv, 0.f);
      }
    }
  }
  if (!want_stats) return;
  __syncthreads();
  // merge the row-lanes of each column in lane order (Chan et al.), then deliver the slot's pair to the sinks
  for (int i = threadIdx.x; i < ccols; i += blockDim.x) {
    float cn = 0.f, mean = 0.f, m2 = 0.f;
    for (int l = 0; l < lanes; ++l) {
      const float* e = s_red + ((size_t)l * ccols + i) * 3;
      const float nb = e[0];
      if (nb == 0.f) continue;
      const float tot = cn + nb, d = e[1] - mean;
      mean += d * (nb / tot);
      m2 += e[2] + d * d * (cn * nb / tot);
      cn = tot;
    }
    const int ch = c_begin + i;
#pragma unroll
    for (int d = 0; d < 2; ++d)
      if (p.sink[d].part) {
        float* dst = p.sink[d].part + (((size_t)n * p.slots + slot) * p.sink[d].cstride + p.sink[d].coff + ch) * 2;
        dst[0] = mean; dst[1] = m2;
      }
  }
}

// ------------------------------------------------------------------------------------------------
// Weight repacking (load time): fp32 OIHW -> fp16 [O][kh][kw][Ipad]; fp32 [O, I] -> fp16 [O][Ipad]
// ------------------------------------------------------------------------------------------------
__global__ void pack_conv_weight_kernel(const float* __restrict__ src, __half* __restrict__ dst, int O, int I,
                                        int KH, int KW, int Ipad) {
  pdl_trigger();
  pdl_wait();
  const long long total = (long long)O * KH * KW * Ipad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % Ipad);
    long long q = i / Ipad;
    const int kw = (int)(q % KW); q /= KW;
    const int kh = (int)(q % KH); q /= KH;
    const int o = (int)q;
    float v = 0.f;
    if (c < I) v = src[(((long long)o * I + c) * KH + kh) * KW + kw];
    dst[i] = __float2half_rn(v);
  }
}

// relative_position_bias_table [(2w-1)^2, heads] -> dense [heads][w*w][w*w] fp32
// (reference models/swin_transformer.py:93-103 for the index, :127-130 for the gather)
__global__ void expand_relpos_kernel(const float* __restrict__ table, float* __restrict__ dst, int heads, int w) {
  pdl_trigger();
  pdl_wait();
  const int T = w * w;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= heads * T * T) return;
  const int h = i / (T * T), r = (i / T) % T, c = i % T;
  const int dy = r / w - c / w + w - 1, dx = r % w - c % w + w - 1;
  dst[i] = table[(dy * (2 * w - 1) + dx) * heads + h];
}

__global__ void copy_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, long long n) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[i];
}

// the decoder's fp32 output stage with tanh_out (reference model.py:658-659)
__global__ void copy_tanh_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, long long n) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = tanhf(src[i]);
}

#endif
}  // namespace rs

// Host-side launch helpers: TMA descriptor encoding and one launcher per kernel family.
#pragma once

#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <mutex>
#include <utility>
#include <vector>

#include "common.cuh"
#include "conv_gemm.cuh"
#include "elementwise.cuh"
#include "mlp_fused.cuh"
#include "norm_act.cuh"
#include "window_attn.cuh"
#include "swin_attn_fused.cuh"
#include "vq_attn.cuh"
#include "unet_attn.cuh"

namespace rs {

// ---- driver entry point for cuTensorMapEncodeTiled (the .so does not link libcuda) --------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_tiled() {
  static std::atomic<PFN_encodeTiled> fn{nullptr};     // plans may be bound from several host threads at once
  PFN_encodeTiled f = fn.load(std::memory_order_acquire);
  if (!f) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      f = reinterpret_cast<PFN_encodeTiled>(p);
      fn.store(f, std::memory_order_release);
    }
  }
  return f;
}

// NHWC fp16 view descriptor used by the host code.
struct View {
  __half* ptr = nullptr;   // resolved at bind time
  int tens = -1;           // owning workspace tensor
  long long off = 0;       // element offset inside the tensor (channel slice + batch slice)
  int c0 = 0, n0 = 0;      // bookkeeping of the same slice: first channel / first image inside the owning tensor
  int N = 0, H = 0, W = 0, C = 0, ld = 0;
  long long sW() const { return ld; }
  long long sH() const { return (long long)W * ld; }
  long long sN() const { return (long long)H * W * ld; }
};

// 4-D activation map {C, W, H, N} with explicit element strides; box {64, bw, bh, bn}, 128B swizzle.
inline int encode_act_map(CUtensorMap* m, const __half* base, int C, int W, int H, int N, long long sW,
                          long long sH, long long sN, int bw, int bh, int bn, int box_c = kConvBK) {
  PFN_encodeTiled enc = get_encode_tiled();
  RS_CHECK(enc != nullptr, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)sW * 2, (cuuint64_t)sH * 2, (cuuint64_t)sN * 2};
  cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bn};
  const CUtensorMapSwizzle swz = box_c == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : (box_c == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  RS_CHECK(box_c == 64 || box_c == 32 || box_c == 16, "activation box width");
  cuuint32_t estr[4] = {1, 1, 1, 1};
  RS_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0, "activation base must be 16-byte aligned");
  RS_CHECK(sW % 8 == 0 && sH % 8 == 0 && sN % 8 == 0, "activation strides must be multiples of 16 bytes");
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<__half*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(activation) failed with CUresult " + std::to_string((int)r));
  return 0;
}
// 2-D weight map {Ktot, Cout}, box {64, BN}.
inline int encode_weight_map(CUtensorMap* m, const __half* base, int Ktot, int Cout, int BN) {
  PFN_encodeTiled enc = get_encode_tiled();
  RS_CHECK(enc != nullptr, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  cuuint64_t dims[2] = {(cuuint64_t)Ktot, (cuuint64_t)Cout};
  cuuint64_t strides[1] = {(cuuint64_t)Ktot * 2};
  cuuint32_t box[2] = {(cuuint32_t)kConvBK, (cuuint32_t)BN};
  cuuint32_t estr[2] = {1, 1};
  RS_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0 && Ktot % 8 == 0, "weight matrix must be 16-byte aligned");
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(weights) failed with CUresult " + std::to_string((int)r));
  return 0;
}

// The kernel-choice overrides of the environment (INTEGRATION.md): test hooks and tuning aids, none set in production.
// A plan reads them once, when it is created, and every later decision of that plan (layout, tile configurations at
// bind, the kernels it launches) follows that snapshot; a single-operator entry point reads them per call.
struct Overrides {
  bool conv_simt = false;     // RS_CONV_IMPL=simt: the SIMT cross-check conv kernel (no fused MLP / Swin attention / statistics)
  bool attn_simt = false;     // RS_ATTN_IMPL=simt: the SIMT cross-check window-attention kernel (no fused Swin attention)
  bool conv_direct = false;   // RS_CONV_EPI=direct: per-thread stores instead of the staged TMA epilogue
  // RS_CONV_{BN,CG,OCC,MSUB,SPLITK}: forced tile configuration (0: the cost model's pick); RS_CONV_PERSIST 0 / 1
  // disables / forces the persistent kernel (-1: the cost model)
  int conv_bn = 0, conv_cg = 0, conv_occ = 0, conv_msub = 0, conv_splitk = 0, conv_persist = -1;
  bool no_reuse = false;      // RS_NO_REUSE=1: no workspace aliasing, every block output stays readable (rs_plan_probe)
  // RS_SWIN_FUSE_MIN_PAIRS: a Swin level with fewer pairs of 8x8 windows keeps the four-launch attention half.  A level with
  // few window pairs is one long serial tile per CTA on a handful of SMs; below this many pairs the four small launches,
  // whose prologues overlap through PDL, are used instead.  At the benchmark shape (batch 16, the 64x64 and 32x32 levels
  // fused) the default measured 127.7 ms per 15-step loop against 134.8 ms with every level on four launches (H100 80GB
  // HBM3 SXM, 700 W).  With an earlier build of the wgmma kernel, thresholds 96 / 32 / 8 / 1 (also fusing the 16x16 and
  // 8x8 levels) measured 135.3 / 134.1 / 135.3 / 135.6 ms, one run each: within the run-to-run spread, so 96 stays
  // (H100 80GB HBM3 SXM, 400 W)
  int swin_fuse_min_pairs = 96;
};
inline Overrides read_overrides() {
  auto var = [](const char* name) { return std::getenv(name); };
  auto num = [&](const char* name, int dflt) { const char* v = var(name); return v ? std::atoi(v) : dflt; };
  auto is = [&](const char* name, const char* val) { const char* v = var(name); return v && std::strcmp(v, val) == 0; };
  Overrides o;
  o.conv_simt = is("RS_CONV_IMPL", "simt");
  o.attn_simt = is("RS_ATTN_IMPL", "simt");
  o.conv_direct = is("RS_CONV_EPI", "direct");
  o.conv_bn = num("RS_CONV_BN", 0); o.conv_cg = num("RS_CONV_CG", 0); o.conv_occ = num("RS_CONV_OCC", 0);
  o.conv_msub = num("RS_CONV_MSUB", 0); o.conv_splitk = num("RS_CONV_SPLITK", 0); o.conv_persist = num("RS_CONV_PERSIST", -1);
  o.no_reuse = num("RS_NO_REUSE", 0) != 0;
  o.swin_fuse_min_pairs = num("RS_SWIN_FUSE_MIN_PAIRS", o.swin_fuse_min_pairs);
  return o;
}

// All kernels go through this launcher: cudaLaunchKernelEx with the programmatic-stream-serialization
// attribute (PDL), so kernel N+1's prologue overlaps kernel N's tail, also inside captured graphs.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kc(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                             int cluster_x, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  int n = 1;
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x; attr[n].val.clusterDim.y = 1; attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = attr; cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                            Args&&... args) {
  return launch_kc(kernel, grid, block, smem, st, 1, std::forward<Args>(args)...);
}

// per-device state of the library is indexed by the CUDA device ordinal
constexpr int kMaxDevices = 64;

// streaming multiprocessors of the current device (grid sizes of persistent kernels, the wave model of the cost
// estimates), read once per device; host-only previews without a device assume an H100 SXM (132).  Threads driving
// different devices may ask at the same time: every slot is written with the same value, atomically.
inline int num_sms() {
  static std::atomic<int> cache[kMaxDevices] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) { (void)cudaGetLastError(); return 132; }
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) { (void)cudaGetLastError(); n = 132; }
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

// shared memory of the conv epilogue's staging area: msub output tiles + per-warp GroupNorm partials
inline size_t conv_epi_bytes(int BN, int msub) {
  return (size_t)msub * ((size_t)BN * kConvBM * 2 + (size_t)4 * BN * 2 * sizeof(float));
}
// what a persistent conv CTA needs beyond its operand ring: staging area, barriers, bias tile, alignment slack
inline size_t conv_persist_extra_bytes(int BN) { return (conv_epi_bytes(BN, 1) + 1023) / 1024 * 1024 + 256 + 1024 + 1024; }

inline int pow2_floor_div(int x, int cap) {   // largest power of two dividing x, capped
  int p = 1;
  while (p * 2 <= cap && x % (p * 2) == 0) p *= 2;
  return p;
}

// Host description of one conv / linear layer instance.
struct ConvDesc {
  View in;                 // input view (for stride 2: the full-resolution input)
  int ksize = 1, stride = 1;
  int pad_lo = 1;          // stride-2 convs: 1 = symmetric padding 1 (UNet Downsample, reference models/unet.py:99-108);
                           // 0 = pad (0,1,0,1) then a padding-free conv (VQ-GAN Downsample, ldm/.../model.py:78-87)
  const __half* wt = nullptr;   // [Cout][taps][ipad]
  int ipad = 0;
  const float* bias = nullptr;
  bool bias_per_image = false;    // the bias is a per-image row set per launch (prm.bias / prm.bias_sN): size its tile
  int Cout = 0;
  View out;               // NHWC fp16 output view (ptr may be null when out_f32 is used)
  bool has_out = true;
  View res; bool has_res = false;
  View silu_out; bool has_silu = false;   // second output: SiLU of the stored fp16 output (same grid and channels)
  bool film = false;      // FiLM rows after the activation, set per launch (prm.film / red.film)
  float* out_f32 = nullptr;
  int act = ACT_NONE;
  int bn_override = 0;
  int msub_request = 0;           // sub-tiles per CTA asked for (0: RS_CONV_MSUB, else the cost model)
  unsigned long long* dbg = nullptr;
  float* partial = nullptr;       // split-K scratch [S][pixels][Cout] fp32 (caller-provided when the plan chose S > 1)
  bool allow_split = false;
  SplitKReduceParams red;         // filled by finalize() when S > 1
  int red_grid_x = 0, red_grid_z = 1; size_t red_smem = 0;
  // fused GroupNorm statistics of the output (up to two consumers; gn_stats.cuh).  `expected` is filled by finalize()
  // (slots * cstride) unless the caller set it (a statistics buffer only partly covered by this producer: unit tests)
  GnSink sink[2] = {};
  // filled by finalize()
  ConvParams prm;
  ConvSimtSrc simt;
  bool simt_kernel = false;       // launch the SIMT cross-check kernel (RS_CONV_IMPL=simt) instead of the wgmma one
  int grid = 0; size_t smem = 0;
};

struct TileConfig { int BN = 0, msub = 1, stages = 2, occ = 1, cg = 1, splitk = 1, persist = 0; double est_cycles = 1e30; };

// Cost model that ranks tile configurations (its constants come from the throughput figures of the H100 SXM and have not
// been calibrated against timelines).  Per 64-channel k-block and 128-pixel tile the tensor pipe needs 4*BN cycles
// (dense fp16 wgmma: 4096 flop/clk/SM); every operand byte crosses shared memory (TMA write, 128 B/clk per SM) and is
// read by wgmma (A once, B once per warpgroup); a CTA pair (cg = 2) fetches only half of B from L2 per CTA (TMA
// multicast).  Shallow rings are additionally latency-bound (~3000 cycles per load).  The epilogue (~18 cycles per
// column + set-up) hides under a co-resident CTA; whole waves are counted.
inline TileConfig pick_tile_config(const Overrides& o, int m_tiles, int cout16, int num_kb, int f_bn, bool allow_split = false,
                                   bool allow_persist = false, bool allow_msub2 = true, int msub_request = 0) {
  const int f_msub = msub_request ? msub_request : o.conv_msub, f_occ = o.conv_occ, f_cg = o.conv_cg;
  TileConfig best, bestp;      // best one-tile-per-CTA configuration (ranking model below), best persistent one
  double best_real = 1e30;     // realistic estimate of `best` (see the end of the function)
  for (int cand = std::min(cout16, 256); cand >= 16; cand -= 16) {
    if (f_bn ? (cand != std::min(f_bn, std::min(cout16, 256))) : (cout16 % cand != 0)) continue;
    if (!conv_bn_supported(cand)) continue;
    const int n_tiles = (cout16 + cand - 1) / cand;
    // msub = 2 only on request (RS_CONV_MSUB=2 or the descriptor), and then wherever the layer can take it (one CTA per
    // tile, an even tile count, a channel tile with that instance); otherwise one sub-tile
    const bool ms2_cand = f_msub == 2 && allow_msub2 && m_tiles % 2 == 0 && conv_kernel_for(cand, 2);
    for (int cg = 1; cg <= 2; ++cg) {
      if (f_cg && cg != f_cg && !(f_cg == 2 && m_tiles < 2)) continue;   // a single tile cannot form a pair
      if (cg == 2 && ms2_cand && f_cg != 2) continue;
      if (cg == 2 && (cand % 16 != 0 || m_tiles < 2)) continue;
      // persistent mode: one CTA (pair) per SM walks ceil(units / workers) tiles; the producer fetches the next tile's
      // operands while the consumers run the epilogue, so a tile costs about max(main loop, epilogue) and set-up / first
      // round trip are paid once
      if (allow_persist) {
        const long long units_p = (long long)((m_tiles + cg - 1) / cg) * n_tiles;
        const int workers = cg == 2 ? num_sms() / 2 : num_sms();
        const int sbytes_p = kConvBM * kConvBK * 2 + cand * kConvBK * 2;
        const size_t extra = conv_persist_extra_bytes(cand);
        const int st_p = (int)std::min<size_t>(8, ((size_t)227 * 1024 - extra) / (size_t)sbytes_p);
        // (only layers with at least two PIXEL tiles per worker; getting there through many narrow channel tiles would
        // re-read the A operand once per channel tile)
        if ((m_tiles + cg - 1) / cg >= 2 * workers && st_p >= 2) {
          const double kb_p = std::max(std::max(4.0 * cand, 2.0 * sbytes_p / 128.0), 2600.0 / st_p);
          const double epi_p = 5000.0 + 3.0 * cand;
          const double rounds = std::ceil((double)units_p / workers);
          const double total = rounds * std::max(num_kb * kb_p, epi_p) + epi_p + 3000.0;
          if (total < bestp.est_cycles) {
            bestp.est_cycles = total; bestp.BN = cand; bestp.msub = 1; bestp.stages = std::min(st_p, std::max(2, num_kb));
            bestp.occ = 1; bestp.cg = cg; bestp.splitk = 1; bestp.persist = 1;
          }
        }
      }
      const bool ms2 = ms2_cand && cg == 1;
      for (int ms = 1; ms <= 2; ++ms) {
        if (ms == 2 ? !ms2 : ms2) continue;
        const int sbytes = ms * kConvBM * kConvBK * 2 + cand * kConvBK * 2;
        for (int occ = 1; occ <= 2; ++occ) {
          if (f_occ && occ != f_occ) continue;
          if (occ == 2 && ms * cand > 128) continue;                       // registers: accumulators of two CTAs per SM
          const int budget = (occ == 2 ? 111 : 222) * 1024 - 2048;
          int st = std::min(std::min(8, std::max(2, num_kb)), budget / sbytes);
          // the staged epilogue (output tile + statistics scratch) reuses the ring: it must be at least that large
          // (short-K layers with wide channel tiles in pair mode: 2 stages x (16 KB + BN/2 x 128 B) < BN x 288 B)
          {
            const int st_need = (int)((conv_epi_bytes(cand, ms) + sbytes - 1) / sbytes);
            if (st_need > budget / sbytes) continue;
            st = std::max(st, st_need);
          }
          if (st < 2 || (size_t)st * sbytes + 2304 > (size_t)(occ == 2 ? 113 : 227) * 1024) continue;
          const double smem_cycles = (sbytes + ms * kConvBM * kConvBK * 2.0 + 2.0 * cand * kConvBK * 2.0) / 128.0;
          // SM time for every resident CTA to advance one k-block: tensor / smem work of each, or the load latency
          // amortised over the ring depth
          // load latency: assumed ~3000 cycles when many tiles share each weight tile (L2 hits), ~7500 when the layer has so
          // few pixel tiles that every weight tile is a fresh HBM read for a handful of CTAs
          const double load_lat = m_tiles >= 64 ? 3000.0 : 7500.0;
          const double kb_cycles = std::max(occ * std::max(ms * 4.0 * cand, smem_cycles), load_lat / st);
          const double epi = 18.0 * cand * ms + 3000.0 + (cg == 2 ? 2500.0 : 0.0);  // + pipeline fill / set-up (+ cluster syncs)
          const long long units = (long long)((m_tiles + cg * ms - 1) / (cg * ms)) * n_tiles;   // CTAs or CTA pairs
          const double slots = (cg == 2 ? num_sms() / 2 : num_sms()) * (double)occ;
          // split-K: S CTAs (pairs) share one output tile's K loop; costs an fp32 round trip + a small reduce kernel
          const int f_split = o.conv_splitk;
          const int kSplits[6] = {1, 2, 3, 4, 6, 8};
          for (int si = 0; si < 6; ++si) {
            const int S = kSplits[si];
            if (S > 1 && (!allow_split || ms != 1 || num_kb / S < 6)) continue;
            if (f_split && allow_split && ms == 1 && num_kb / f_split >= 6 && S != f_split) continue;
            const double waves = std::ceil((double)units * S / slots);
            const double kbs = std::ceil((double)num_kb / S);
            const double round = kbs * kb_cycles + (occ == 2 ? 0.5 * epi : epi);
            // fp32 partials written once by the conv epilogue and read once by the reduce kernel (assumed ~2 KB/clk
            // chip-wide each way), plus a second kernel launch / drain (a fixed cost for the pair)
            const double part_bytes = 4.0 * m_tiles * 128.0 * cout16 * S;
            const double total = waves * round + (S == 1 ? 0.0 : 19000.0 + 2.0 * part_bytes / 2048.0);
            if (total < best.est_cycles) {
              best.est_cycles = total; best.BN = cand; best.msub = ms;
              best.stages = std::max(std::min(st, (int)std::max(2.0, kbs)), std::min(st, (int)((conv_epi_bytes(cand, ms) + sbytes - 1) / sbytes)));
              best.occ = occ; best.cg = cg; best.splitk = S; best.persist = 0;
              // what a wave really costs (timelines r1_s25): co-resident CTAs run in lockstep, so set-up, the first
              // operand round trip and the whole epilogue are exposed once per wave
              best_real = waves * (kbs * kb_cycles + epi + 5000.0) + (S == 1 ? 0.0 : 19000.0 + 2.0 * part_bytes / 2048.0);
            }
          }
        }
      }
    }
  }
  // the ranking model above is optimistic in absolute terms (set-up, first round trip and epilogue are exposed once per
  // wave); compare the persistent estimate with that realistic figure, ties going to the persistent mode
  if (bestp.BN && 0.85 * bestp.est_cycles < best_real) return bestp;
  return best;
}

// geometry-only preview of the configuration conv_finalize() will choose (used at plan time to size split-K scratch)
inline TileConfig conv_preview_config(const Overrides& o, int N, int Hin, int Win, int Cin, int Cout, int ksize, int stride,
                                      bool allow_split) {
  const int Hout = Hin / stride, Wout = Win / stride;
  const int bw = pow2_floor_div(Wout, kConvBM);
  const int bh = pow2_floor_div(Hout, kConvBM / bw);
  const int bn = kConvBM / (bw * bh);
  const int m_tiles = (Wout / bw) * (Hout / bh) * ((N + bn - 1) / bn);
  const bool contiguous = (bw == Wout) || (bh == 1);
  const int num_kb = ksize * ksize * ((Cin + kConvBK - 1) / kConvBK);
  const bool sp = allow_split && contiguous && bn <= 2;
  return pick_tile_config(o, m_tiles, (Cout + 15) / 16 * 16, num_kb, o.conv_bn, sp);
}

// The statistics sinks a producer's kernel receives: the set ones of `sink` first; an unset `expected` becomes slots (the
// producer's pair slots per image) x cstride, an unset eps GroupNorm32's 1e-5
inline void compact_sinks(const GnSink (&sink)[2], int slots, GnSink (&out)[2]) {
  out[0] = GnSink{}; out[1] = GnSink{};
  int k = 0;
  for (const GnSink& s : sink) {
    if (!s.part) continue;
    out[k] = s;
    if (out[k].expected == 0) out[k].expected = (unsigned)(slots * s.cstride);
    if (out[k].eps == 0.f) out[k].eps = 1e-5f;
    ++k;
  }
}

inline int conv_finalize(ConvDesc& d, const Overrides& o) {
  ConvParams& p = d.prm;
  std::memset(&p, 0, sizeof(p));
  const int Hin = d.in.H, Win = d.in.W;
  RS_CHECK(d.ksize == 1 || d.ksize == 3, "kernel size must be 1 or 3");
  RS_CHECK(d.stride == 1 || (d.stride == 2 && d.ksize == 3 && Hin % 2 == 0 && Win % 2 == 0), "unsupported stride");
  const int Hout = Hin / d.stride, Wout = Win / d.stride, N = d.in.N;
  p.Hout = Hout; p.Wout = Wout; p.Nimg = N; p.Cout = d.Cout;
  p.num_taps = d.ksize * d.ksize;
  p.kchunks = (d.in.C + kConvBK - 1) / kConvBK;
  p.w_tap_stride = d.ipad;
  RS_CHECK(d.ipad % 8 == 0 && d.ipad >= d.in.C, "weight channel padding");
  // pixel box
  p.bw = pow2_floor_div(Wout, kConvBM);
  p.bh = pow2_floor_div(Hout, kConvBM / p.bw);
  p.bn = kConvBM / (p.bw * p.bh);
  p.tiles_w = Wout / p.bw; p.tiles_h = Hout / p.bh; p.tiles_n = (N + p.bn - 1) / p.bn;
  const int m_tiles = p.tiles_w * p.tiles_h * p.tiles_n;
  // ---- tile configuration: channel tile BN, sub-tiles per CTA (msub), CTAs per SM (occ), ring depth (stages) ----
  // Chosen by the cost model of pick_tile_config: the main loop is bound by the bytes of TMA loads in flight per SM
  // (ring capacity / ~3000-cycle load latency) unless the tensor pipe is slower (4*BN cycles per 64-channel k-block per
  // 128-pixel sub-tile); the epilogue hides under the other resident CTA when two fit; whole waves of CTAs are counted.
  const int cout16 = (d.Cout + 15) / 16 * 16;
  const int num_kb = p.num_taps * p.kchunks;
  const bool contiguous_tiles = (p.bw == Wout) || (p.bh == 1);
  // (the SIMT cross-check kernel computes whole outputs, bias / residual / activation included: it never splits K)
  const bool simt = o.conv_simt;
  d.simt_kernel = simt;
  const bool can_split = d.allow_split && d.partial != nullptr && contiguous_tiles && p.bn <= 2 && d.has_out && !d.out_f32 && !simt;
  const int want_persist = o.conv_persist;                           // 0 / 1 disables / forces the persistent kernel
  // per-image bias rows of a box of more than 8 images (maps of fewer than 16 pixels per 128-pixel box): the direct
  // epilogue, which reads them per element (the staged one holds one row per 16 accumulator rows)
  const bool bias_direct = d.bias_per_image && p.bn > 8;
  RS_CHECK(!bias_direct || (!d.has_silu && !d.film), "per-image bias on boxes of more than 8 images cannot take silu_out or FiLM");
  const bool persist_ok = d.has_out && !d.out_f32 && want_persist != 0 && !o.conv_direct && !simt && !bias_direct &&
                          (d.msub_request ? d.msub_request : o.conv_msub) != 2;
  const TileConfig tc = pick_tile_config(o, m_tiles, cout16, num_kb, d.bn_override ? d.bn_override : o.conv_bn, can_split,
                                         persist_ok && want_persist != 1, !d.bias_per_image && !d.film && !d.has_silu, d.msub_request);
  const int BN = tc.BN, msub = tc.msub, stages = tc.stages, cg = tc.cg;
  p.cg = cg;
  p.splitk = tc.splitk; p.partial = d.partial;
  RS_CHECK(conv_kernel_for(BN, msub, d.has_silu || d.film) != nullptr, "no valid tile configuration");
  p.BN = BN; p.n_tiles = (cout16 + BN - 1) / BN;
  p.msub = msub;
  const int stage_bytes = msub * kConvBM * kConvBK * 2 + BN * kConvBK * 2;
  p.stages = stages;
  p.epi_off = 0;
  p.bar_off = stages * stage_bytes;
  // bias tile: [BN] floats, or [bn][BN] when every image has its own bias row
  RS_CHECK(!d.bias_per_image || msub == 1, "per-image bias needs one sub-tile per CTA");
  RS_CHECK(!d.film || (msub == 1 && d.Cout % 8 == 0), "FiLM rows need one sub-tile per CTA and Cout % 8 == 0");
  RS_CHECK(!d.film || (!d.has_res && d.has_out && !d.out_f32 && !d.sink[0].part && !d.sink[1].part),
           "FiLM rows need an fp16 output and no residual or statistics sinks");
  const size_t bias_tile = d.bias_per_image && !bias_direct ? std::max<size_t>(1024, (size_t)p.bn * BN * sizeof(float)) : 1024;
  d.smem = (size_t)stages * stage_bytes + 1024 + 256 + bias_tile;   // ring + alignment slack + barriers + bias tile
  RS_CHECK(d.smem <= 227 * 1024, "shared memory budget exceeded");
  d.grid = (cg == 2 ? ((m_tiles + 1) / 2) * p.n_tiles * 2 : (m_tiles / msub) * p.n_tiles) * p.splitk;
  // taps
  if (d.stride == 1) {
    int t = 0;
    for (int ky = 0; ky < d.ksize; ++ky)
      for (int kx = 0; kx < d.ksize; ++kx, ++t) {
        p.tap_src[t] = 0; p.tap_dh[t] = ky - d.ksize / 2; p.tap_dw[t] = kx - d.ksize / 2;
      }
  } else {
    int t = 0;
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx, ++t) {
        if (d.pad_lo == 1) {        // input row 2i + ky - 1: parity (ky != 1), one step back for ky = 0
          const int hp = (ky == 1) ? 0 : 1, wp = (kx == 1) ? 0 : 1;
          p.tap_src[t] = hp * 2 + wp; p.tap_dh[t] = (ky == 0) ? -1 : 0; p.tap_dw[t] = (kx == 0) ? -1 : 0;
        } else {                    // input row 2i + ky: parity (ky == 1), one step forward for ky = 2 (TMA zero fill = the pad)
          const int hp = (ky == 1) ? 1 : 0, wp = (kx == 1) ? 1 : 0;
          p.tap_src[t] = hp * 2 + wp; p.tap_dh[t] = (ky == 2) ? 1 : 0; p.tap_dw[t] = (kx == 2) ? 1 : 0;
        }
      }
  }
  // epilogue
  p.bias = d.bias; p.bias_sN = 0; p.act = d.act;
  if (d.has_res) {
    RS_CHECK(d.res.H == Hout && d.res.W == Wout && d.res.N == N && d.res.C >= d.Cout, "residual geometry");
    p.residual = d.res.ptr; p.res_sN = d.res.sN(); p.res_sH = d.res.sH(); p.res_sW = d.res.sW();
  }
  if (d.has_out) {
    RS_CHECK(d.out.H == Hout && d.out.W == Wout && d.out.N == N, "output geometry");
    p.out = d.out.ptr; p.out_sN = d.out.sN(); p.out_sH = d.out.sH(); p.out_sW = d.out.sW();
    RS_CHECK(d.out.ld % 8 == 0 && (reinterpret_cast<uintptr_t>(d.out.ptr) & 15) == 0, "output alignment");
  }
  if (d.has_silu) {
    RS_CHECK(d.has_out && !d.out_f32 && d.Cout % 8 == 0, "the SiLU output needs an fp16 output and Cout % 8 == 0");
    RS_CHECK(d.silu_out.H == Hout && d.silu_out.W == Wout && d.silu_out.N == N, "SiLU output geometry");
    RS_CHECK(d.silu_out.ld % 8 == 0 && (reinterpret_cast<uintptr_t>(d.silu_out.ptr) & 15) == 0, "SiLU output alignment");
    p.silu_out = d.silu_out.ptr; p.silu_sN = d.silu_out.sN(); p.silu_sH = d.silu_out.sH(); p.silu_sW = d.silu_out.sW();
  }
  p.out_f32_nchw = d.out_f32;
  p.dbg = d.dbg;
  // staged epilogue (TMA store / TMA residual load) for fp16 NHWC outputs
  // (the direct epilogue has no SiLU output or FiLM: such convs keep the staged epilogue under RS_CONV_EPI=direct)
  p.tma_out = (d.has_out && !d.out_f32 && p.splitk == 1 && (!o.conv_direct || d.has_silu || d.film) && !simt && !bias_direct) ? 1 : 0;
  p.tma_res = (p.tma_out && d.has_res) ? 1 : 0;
  p.epi_bc = (BN % 64 == 0) ? 64 : (BN % 32 == 0 ? 32 : 16);
  if (p.tma_out) {
    int rc = encode_act_map(&p.tmOut, d.out.ptr, d.Cout, Wout, Hout, N, d.out.sW(), d.out.sH(), d.out.sN(), p.bw, p.bh, p.bn, p.epi_bc);
    if (rc) return rc;
    if (p.tma_res) {
      rc = encode_act_map(&p.tmRes, d.res.ptr, d.Cout, Wout, Hout, N, d.res.sW(), d.res.sH(), d.res.sN(), p.bw, p.bh, p.bn, p.epi_bc);
      if (rc) return rc;
    }
    if (d.has_silu) {
      rc = encode_act_map(&p.tmSilu, d.silu_out.ptr, d.Cout, Wout, Hout, N, d.silu_out.sW(), d.silu_out.sH(), d.silu_out.sN(),
                          p.bw, p.bh, p.bn, p.epi_bc);
      if (rc) return rc;
    }
    // the staging area (column blocks + per-warp GN partials) must fit in the operand ring
    // (the persistent kernel stages in buffers of its own, sized below)
    RS_CHECK(tc.persist || conv_epi_bytes(BN, msub) <= (size_t)stages * stage_bytes, "epilogue staging does not fit in the pipeline shared memory");
  }
  // persistent variant (conv_persist.cuh) when the cost model chose it (every SM / pair gets at least two tiles), or
  // when RS_CONV_PERSIST = 1 forces it for any eligible layer
  {
    const int units = (cg == 2 ? (m_tiles + 1) / 2 : m_tiles) * p.n_tiles;
    const int workers = cg == 2 ? num_sms() / 2 : num_sms();
    const bool eligible = persist_ok && p.tma_out && p.splitk == 1 && msub == 1;
    p.persist = (eligible && (tc.persist || want_persist == 1)) ? 1 : 0;
    RS_CHECK(!tc.persist || p.persist, "persistent configuration chosen for an ineligible layer");
    p.num_units = units;
    if (p.persist) {
      // the staging area (output tile + statistics scratch) follows the ring: the producer refills the ring while the
      // consumers drain the previous tile
      const size_t extra = conv_persist_extra_bytes(BN);
      const int st = (int)std::min<size_t>(8, ((size_t)227 * 1024 - extra - (bias_tile - 1024)) / (size_t)stage_bytes);
      RS_CHECK(st >= 2, "persistent conv: shared memory budget");
      p.stages = std::min(st, std::max(2, num_kb));
      p.epi_off = p.stages * stage_bytes;
      p.bar_off = p.epi_off + (int)conv_epi_bytes(BN, 1);
      d.smem = (size_t)p.bar_off + 256 + bias_tile + 1024;
      RS_CHECK(d.smem <= 227 * 1024, "persistent conv: shared memory budget");
      d.grid = cg * std::min(units, workers);
    }
  }
  p.gn_slots = p.tiles_w * p.tiles_h;
  RS_CHECK(!(d.sink[0].part || d.sink[1].part) || p.bn <= 2, "fused GroupNorm statistics need tiles of at most two images");
  if (p.tma_out) compact_sinks(d.sink, p.gn_slots, p.sink);
  if (p.splitk > 1) {
    // the conv kernel only produces fp32 partial sums; bias / activation / residual / fp16 store / GroupNorm statistics
    // happen in the reduce kernel, one CTA per (128-pixel slot, image)
    SplitKReduceParams& r = d.red;
    std::memset(&r, 0, sizeof(r));
    r.partial = d.partial; r.S = p.splitk; r.N = N; r.HW = Hout * Wout; r.C = d.Cout;
    r.bias = d.bias; r.act = d.act;
    if (d.has_res) { r.residual = d.res.ptr; r.res_sN = d.res.sN(); r.res_ld = d.res.ld; }
    r.out = d.out.ptr; r.out_sN = d.out.sN(); r.out_ld = d.out.ld;
    r.rows_per_slot = p.bw * p.bh; r.slots = p.tiles_w * p.tiles_h;
    compact_sinks(d.sink, p.gn_slots, r.sink);
    if (d.has_silu) { r.silu_out = d.silu_out.ptr; r.silu_sN = d.silu_out.sN(); r.silu_ld = d.silu_out.ld; }
    RS_CHECK(d.Cout % 8 == 0 && d.Cout <= 2048, "split-K reduce needs Cout % 8 == 0");
    p.bias = nullptr; p.residual = nullptr; p.act = ACT_NONE; p.sink[0] = GnSink{}; p.sink[1] = GnSink{};
    p.silu_out = nullptr;
    d.red_grid_x = r.slots;
    // column blocks so that the reduce kernel fills the machine even with one slot per image
    int cpc = d.Cout;
    while (cpc > 64 && cpc % 16 == 0 && (long long)r.slots * N * (d.Cout / cpc) < 2 * num_sms()) cpc /= 2;
    r.cols_per_cta = cpc;
    d.red_grid_z = (d.Cout + cpc - 1) / cpc;
    const int lanes = 256 / std::max(1, cpc / 8);
    d.red_smem = (size_t)std::max(1, lanes) * cpc * 3 * sizeof(float);
  }
  // tensor maps + SIMT mirrors
  ConvSimtSrc& s = d.simt;
  std::memset(&s, 0, sizeof(s));
  s.C = d.in.C; s.wt = d.wt;
  const int nsrc = d.stride == 1 ? 1 : 4;
  for (int i = 0; i < kMaxSrc; ++i) {
    const int j = i < nsrc ? i : 0;
    const int hp = d.stride == 2 ? (j >> 1) : 0, wp = d.stride == 2 ? (j & 1) : 0;
    const __half* base = d.in.ptr + (long long)hp * d.in.sH() + (long long)wp * d.in.sW();
    const long long sW = d.in.sW() * d.stride, sH = d.in.sH() * d.stride, sN = d.in.sN();
    s.ptr[i] = base; s.sN[i] = sN; s.sH[i] = sH; s.sW[i] = sW; s.H[i] = Hout; s.W[i] = Wout;
    if (!simt) {
      int rc = encode_act_map(&p.tmA[i], base, d.in.C, Wout, Hout, N, sW, sH, sN, p.bw, p.bh, p.bn);
      if (rc) return rc;
    }
  }
  if (!simt) {
    int rc = encode_weight_map(&p.tmB, d.wt, p.num_taps * d.ipad, d.Cout, BN / cg);   // pair mode: each CTA loads half
    if (rc) return rc;
  }
  return 0;
}

// Raises the dynamic shared-memory limit of every large kernel.  The runtime keeps function attributes per device, so
// this runs once on every device the library launches on (the current one), outside any stream capture; host threads
// driving different devices may call it at the same time.
inline int conv_init() {
  static std::atomic<bool> attr_set[kMaxDevices] = {};
  static std::mutex mu;
  int dev = 0;
  RS_CUDA_OK(cudaGetDevice(&dev));
  RS_CHECK(dev >= 0 && dev < kMaxDevices, "device ordinal out of range");
  if (attr_set[dev].load(std::memory_order_acquire)) return 0;
  std::lock_guard<std::mutex> lock(mu);
  if (!attr_set[dev].load(std::memory_order_relaxed)) {
    for (int bn : kConvBNs)
      for (int ms = 1; ms <= 2; ++ms)
        for (bool ex : {false, true})
          if (ConvKernelFn k = conv_kernel_for(bn, ms, ex))
            RS_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    RS_CUDA_OK(cudaFuncSetAttribute(window_attn_kernel<8, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnMaxSmem));
    RS_CUDA_OK(cudaFuncSetAttribute(window_attn_kernel<8, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnMaxSmem));
    RS_CUDA_OK(cudaFuncSetAttribute(window_attn_kernel<16, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnMaxSmem));
    RS_CUDA_OK(cudaFuncSetAttribute(window_attn_kernel<16, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnMaxSmem));
    RS_CUDA_OK(cudaFuncSetAttribute(mlp_fused_sm90_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    RS_CUDA_OK(cudaFuncSetAttribute(mlp_fused_sm90_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    RS_CUDA_OK(cudaFuncSetAttribute(mlp_fused_sm90_kernel<192>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    RS_CUDA_OK(cudaFuncSetAttribute(mlp_fused_sm90_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    RS_CUDA_OK(cudaFuncSetAttribute(swin_attn_fused_kernel<192>, cudaFuncAttributeMaxDynamicSharedMemorySize, SwinSmem<192>::launch_bytes));
    RS_CUDA_OK(cudaFuncSetAttribute(swin_attn_fused_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, SwinSmem<64>::launch_bytes));
    RS_CUDA_OK(cudaFuncSetAttribute(vq_attn_sm90_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, VqAttnSmem<128>::launch_bytes));
    RS_CUDA_OK(cudaFuncSetAttribute(vq_attn_sm90_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, VqAttnSmem<256>::launch_bytes));
    RS_CUDA_OK(cudaFuncSetAttribute(vq_attn_sm90_kernel<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, VqAttnSmem<512>::launch_bytes));
    RS_CUDA_OK(cudaFuncSetAttribute(unet_attn_sm90_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, UnetAttnSmem<32>::launch_bytes));
    RS_CUDA_OK(cudaFuncSetAttribute(unet_attn_sm90_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, UnetAttnSmem<64>::launch_bytes));
    RS_CUDA_OK(cudaFuncSetAttribute(unet_attn_sm90_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, UnetAttnSmem<128>::launch_bytes));
    attr_set[dev].store(true, std::memory_order_release);
  }
  return 0;
}

inline int conv_launch(const ConvDesc& d, cudaStream_t st) {
  if (d.simt_kernel) {
    const long long npix = (long long)d.prm.Nimg * d.prm.Hout * d.prm.Wout;
    const int warps = 8;
    (void)launch_k(conv_simt_kernel, dim3((unsigned)((npix + warps - 1) / warps)), dim3(warps * 32), (size_t)(0), st, d.prm, d.simt);
  } else {
    const ConvKernelFn k = conv_kernel_for(d.prm.BN, d.prm.msub, d.has_silu || d.film);
    RS_CHECK(k != nullptr, "no conv kernel for this channel tile");
    (void)launch_kc(k, dim3(d.grid), dim3(kConvThreads), (size_t)(d.smem), st, d.prm.cg, d.prm);
    if (d.prm.splitk > 1)
      (void)launch_k(splitk_reduce_kernel, dim3(d.red_grid_x, d.prm.Nimg, d.red_grid_z), dim3(256), d.red_smem, st, d.red);
  }
  RS_CUDA_OK(cudaGetLastError());
  return 0;
}

// ---- GroupNorm -------------------------------------------------------------------------------
// number of 128-pixel tile slots per image the conv kernel uses for an H x W output (and whether its epilogue can
// produce per-image statistics: tiles must not span more than two images)
inline int conv_tile_slots(int H, int W, bool* fusable = nullptr) {
  const int bw = pow2_floor_div(W, kConvBM);
  const int bh = pow2_floor_div(H, kConvBM / bw);
  if (fusable) *fusable = (kConvBM / (bw * bh)) <= 2;
  return (W / bw) * (H / bh);
}

struct GnDesc {
  View in, out;
  const float* gamma = nullptr; const float* beta = nullptr;
  const float* film = nullptr; long long film_sN = 0;   // resolved per launch for FiLM layers
  int film_off = -1;      // offset of this layer's [2C] slice inside an embedding row, or -1
  int silu = 0;
  float* part = nullptr;  // [N][slots][C][2] (mean, M2) pairs
  float* gstat = nullptr; // [N][32][2] (mean, rstd), finalised by gn_finalize_kernel or the last gn_stats_kernel CTA
  unsigned int* counter = nullptr;   // [N]
  float eps = 1e-5f;
  int slots = 0;
  bool fused = false;     // statistics already delivered by the producing kernels' epilogues
  bool finalize_kernel = false;   // fused statistics with many slots: reduce part -> gstat with gn_finalize_kernel first
};

inline void gn_chunks(int HW, int N, int* chunks, int* rows) {
  // enough CTAs to fill the machine, at least 32 rows each, and every chunk with the SAME number of rows (the
  // statistics combine assumes equal counts per slot): the largest divisor of HW not above the target
  int c = std::max(1, std::min((HW + 31) / 32, (num_sms() * 4 + N - 1) / N));
  while (c > 1 && HW % c != 0) --c;
  *chunks = c; *rows = HW / c;
}

// The launch geometry of one GroupNorm (host only; gn_launch launches exactly this)
struct GnGeometry {
  int slots = 0;          // pair slots per image (the producers', or gn_stats_kernel's CTAs per image)
  int rows_per_slot = 0;
  int stats_ctas = 0;     // gn_stats_kernel CTAs per image (0: the producers delivered the pairs)
  bool finalize = false;  // gn_finalize_kernel runs in front of the apply
  int apply_ctas = 0;     // gn_apply_kernel grid.x (row blocks per image)
  int apply_rows = 0;     // rows per apply CTA
  int csplit = 1;         // gn_apply_kernel grid.z (channel slices)
};

inline GnGeometry gn_geometry(const GnDesc& g) {
  const int C = g.in.C, HW = g.in.H * g.in.W, N = g.in.N;
  GnGeometry r;
  r.slots = g.slots;
  if (!g.fused) {         // gn_stats_kernel: the caller's slot count, or enough CTAs to fill the machine
    int chunks, rows;
    gn_chunks(HW, N, &chunks, &rows);
    if (r.slots <= 0) r.slots = chunks;
    r.stats_ctas = r.slots;
  }
  r.rows_per_slot = r.slots > 0 ? HW / r.slots : 0;
  r.finalize = g.fused && g.finalize_kernel;
  // apply: ~4 CTAs per SM in total, all resident at once (each CTA re-derives the per-channel affine from the
  // partials — a latency, not a bandwidth cost), at least 16 rows each
  int actas = std::max(1, std::min((HW + 15) / 16, (num_sms() * 4 + N - 1) / N));
  r.apply_rows = (HW + actas - 1) / actas;
  r.apply_ctas = (HW + r.apply_rows - 1) / r.apply_rows;
  // small tensors: split the channels too (slices aligned to GroupNorm groups and to 8-channel vectors) until there
  // are ~1.5 CTAs per SM — a 8x8 C=640 layer would otherwise run on 64 CTAs
  const int cpg = C / 32;
  int unit = cpg; while (unit % 8) unit += cpg;                     // lcm(8, channels per group)
  for (int cs = 2; r.apply_ctas * N * r.csplit < num_sms() * 3 / 2 && cs <= C / unit; ++cs)
    if (C % cs == 0 && (C / cs) % unit == 0) r.csplit = cs;
  return r;
}

inline int gn_launch(const GnDesc& g, cudaStream_t st) {
  const int C = g.in.C, HW = g.in.H * g.in.W, N = g.in.N;
  RS_CHECK(C % 32 == 0 && C % 8 == 0 && C <= 2048, "GroupNorm channel count");
  RS_CHECK(g.in.ld % 8 == 0 && g.out.ld % 8 == 0, "GroupNorm view alignment");
  RS_CHECK(g.gstat != nullptr || g.part != nullptr, "GroupNorm needs a statistics buffer");
  const GnGeometry geo = gn_geometry(g);
  const int slots = geo.slots;
  if (!g.fused) {
    const int lanes = 256 / (C / 8);
    RS_CHECK(g.part != nullptr && (g.gstat == nullptr || g.counter != nullptr), "GroupNorm statistics buffers");
    RS_CHECK(HW % slots == 0, "GroupNorm statistics slots must divide H*W");
    GnStatsParams sp{};
    sp.x = g.in.ptr; sp.sN = g.in.sN(); sp.ld = g.in.ld; sp.C = C; sp.HW = HW; sp.N = N;
    sp.sink.part = g.part; sp.sink.gstat = g.gstat; sp.sink.counter = g.counter; sp.sink.cstride = C; sp.sink.coff = 0;
    sp.sink.expected = (unsigned)(slots * C); sp.sink.eps = g.eps;
    sp.slots = slots; sp.rows_per_slot = geo.rows_per_slot;
    (void)launch_k(gn_stats_kernel, dim3(geo.stats_ctas, N), dim3(256), (size_t)lanes * C * 3 * sizeof(float) + 16, st, sp);
    RS_CUDA_OK(cudaGetLastError());
  }
  if (geo.finalize) {
    RS_CHECK(g.part != nullptr && g.gstat != nullptr && slots > 0 && HW % slots == 0, "GroupNorm finalisation buffers");
    GnFinalizeParams fp{g.part, g.gstat, slots, C, (float)geo.rows_per_slot, g.eps};
    (void)launch_k(gn_finalize_kernel, dim3(32, N), dim3(256), (size_t)0, st, fp);
    RS_CUDA_OK(cudaGetLastError());
  }
  GnApplyParams ap{g.in.ptr, g.in.sN(), g.in.ld, g.out.ptr, g.out.sN(), g.out.ld, C, HW, N, g.gstat, g.part, slots, g.eps,
                   g.gamma, g.beta, g.film, g.film_sN, g.silu, geo.apply_rows, C / geo.csplit};
  (void)launch_k(gn_apply_kernel, dim3(geo.apply_ctas, N, geo.csplit), dim3(256),
                 (size_t)(4 * (C / geo.csplit) + 64) * sizeof(float), st, ap);
  RS_CUDA_OK(cudaGetLastError());
  return 0;
}

// ---- fused Swin MLP (mlp_fused.cuh) ---------------------------------------------------------------
struct MlpDesc {
  View in, out, res;
  bool has_res = true;
  const __half* w1 = nullptr; const float* b1 = nullptr;    // fc1: [Hd][E] fp16
  const __half* w2 = nullptr; const float* b2 = nullptr;    // fc2: [E][Hd] fp16
  int E = 0, Hd = 0;
  GnSink sink[2] = {};
  MlpParams prm;
  int grid = 0; size_t smem = 0;
};

inline bool mlp_supported(int E, int Hd, int H, int W, int N) {
  (void)N;
  bool fus = false;
  conv_tile_slots(H, W, &fus);
  return (E == 64 || E == 128 || E == 192 || E == 256) && Hd % kMlpHc == 0 && fus;
}

inline int mlp_finalize(MlpDesc& d) {
  MlpParams& p = d.prm;
  std::memset(&p, 0, sizeof(p));
  const int H = d.in.H, W = d.in.W, N = d.in.N;
  RS_CHECK(mlp_supported(d.E, d.Hd, H, W, N), "fused MLP: unsupported shape (E in {64, 128, 192, 256}, hidden % 64)");
  RS_CHECK(d.in.C == d.E && d.out.C == d.E, "fused MLP: channel mismatch");
  p.E = d.E; p.Hd = d.Hd; p.bias1 = d.b1; p.bias2 = d.b2;
  p.bw = pow2_floor_div(W, kConvBM);
  p.bh = pow2_floor_div(H, kConvBM / p.bw);
  p.bn = kConvBM / (p.bw * p.bh);
  p.tiles_w = W / p.bw; p.tiles_h = H / p.bh;
  const int tiles_n = (N + p.bn - 1) / p.bn;
  p.Wout = W; p.Hout = H; p.Nimg = N;
  // ring slots for the weight tiles: as many as fit next to X, one hidden chunk and the bias tables
  const int slot = std::max(kMlpHc, d.E) * kConvBK * 2;
  const int fixed = MlpSmem(d.E, d.Hd, 0).total + 1024;     // + alignment slack
  p.ring = std::min(8, (227 * 1024 - fixed) / slot);
  RS_CHECK(p.ring >= 2, "fused MLP: not enough shared memory for the weight ring");
  d.smem = (size_t)MlpSmem(d.E, d.Hd, p.ring).total + 1024;
  RS_CHECK(d.smem <= 227 * 1024, "fused MLP: shared memory budget exceeded");
  p.has_res = d.has_res ? 1 : 0;
  // Few tiles leave most SMs idle (batch 16: 32 tiles at 16x16, 8 at 8x8): split each tile's hidden chunks over a
  // cluster of p.split CTAs, the smallest divisor of the chunk count that brings the grid to half the SMs, else the
  // largest, and at most 4.  Measured at batch 16, E = 192, hidden 768 (DESIGN.md §7), us per launch for S = 1 / 2 / 3
  // / 4 / 6: 8x8 38.4 / 31.0 / 29.0 / 28.7 / 30.1, 16x16 38.7 / 31.4 / 29.9 / 44.8 / 49.6; 32x32 (128 tiles) is
  // fastest unsplit.  The reduction needs the ring to hold a 128 x E fp32 partial.
  const int tiles = p.tiles_w * p.tiles_h * tiles_n, chunks = d.Hd / kMlpHc;
  p.split = 1;
  if (p.ring * slot >= kConvBM * d.E * 4)
    for (int s = 2; s <= 4 && tiles * p.split < num_sms() / 2; ++s)
      if (chunks % s == 0) p.split = s;
  d.grid = tiles * p.split;
  int rc = encode_act_map(&p.tmX, d.in.ptr, d.E, W, H, N, d.in.sW(), d.in.sH(), d.in.sN(), p.bw, p.bh, p.bn, 64);
  if (rc) return rc;
  rc = encode_weight_map(&p.tmW1, d.w1, d.E, d.Hd, kMlpHc); if (rc) return rc;
  rc = encode_weight_map(&p.tmW2, d.w2, d.Hd, d.E, d.E); if (rc) return rc;
  rc = encode_act_map(&p.tmOut, d.out.ptr, d.E, W, H, N, d.out.sW(), d.out.sH(), d.out.sN(), p.bw, p.bh, p.bn, 64);
  if (rc) return rc;
  if (d.has_res) {
    rc = encode_act_map(&p.tmRes, d.res.ptr, d.E, W, H, N, d.res.sW(), d.res.sH(), d.res.sN(), p.bw, p.bh, p.bn, 64);
    if (rc) return rc;
  }
  p.gn_slots = p.tiles_w * p.tiles_h;
  compact_sinks(d.sink, p.gn_slots, p.sink);
  return 0;
}

inline int mlp_launch(const MlpDesc& d, cudaStream_t st) {
  switch (d.E) {
    case 64: (void)launch_kc(mlp_fused_sm90_kernel<64>, dim3(d.grid), dim3(kMlpThreads), d.smem, st, d.prm.split, d.prm); break;
    case 128: (void)launch_kc(mlp_fused_sm90_kernel<128>, dim3(d.grid), dim3(kMlpThreads), d.smem, st, d.prm.split, d.prm); break;
    case 192: (void)launch_kc(mlp_fused_sm90_kernel<192>, dim3(d.grid), dim3(kMlpThreads), d.smem, st, d.prm.split, d.prm); break;
    case 256: (void)launch_kc(mlp_fused_sm90_kernel<256>, dim3(d.grid), dim3(kMlpThreads), d.smem, st, d.prm.split, d.prm); break;
    default: RS_CHECK(false, "fused MLP: embedding width");
  }
  RS_CUDA_OK(cudaGetLastError());
  return 0;
}

// ---- fused attention half of a Swin block (swin_attn_fused.cuh) -----------------
struct SwinAttnDesc {
  View x, y;                               // input / output token tensors [N, H, W, E] (y may alias x)
  int heads = 0, shift = 0;
  const float* gn_part = nullptr; int gn_slots = 0;
  const float* gamma = nullptr; const float* beta = nullptr;
  const __half* wqkv = nullptr; int wqkv_ld = 0; const float* bqkv = nullptr;
  const float* relbias = nullptr;
  const __half* wproj = nullptr; int wproj_ld = 0; const float* bproj = nullptr;
  GnSink sink[2] = {};                     // window pairs of y only: the consumer combines them
  SwinAttnParams prm;
  int grid = 0;                            // persistent CTAs: swin_attn_finalize sets min(pairs, SMs)
};
// (8x8 windows and 32-wide heads only: every other level takes the four-launch form around window_attn_kernel)
inline bool swin_attn_supported(int E, int heads, int H, int W, int window) {
  return window == 8 && (E == 192 || E == 64) && heads * 32 == E && H % 8 == 0 && W % 8 == 0;
}
inline int swin_attn_finalize(SwinAttnDesc& d) {
  SwinAttnParams& p = d.prm;
  std::memset(&p, 0, sizeof(p));
  const int E = d.x.C;
  RS_CHECK(swin_attn_supported(E, d.heads, d.x.H, d.x.W, 8), "fused Swin attention: E in {64, 192}, head_dim 32, H and W multiples of 8");
  RS_CHECK(d.y.C == E && d.y.H == d.x.H && d.y.W == d.x.W && d.y.N == d.x.N, "fused Swin attention: output geometry");
  RS_CHECK(d.x.ld % 8 == 0 && d.y.ld % 8 == 0 && d.wqkv_ld % 8 == 0 && d.wproj_ld % 8 == 0, "fused Swin attention: 16-byte rows");
  RS_CHECK(d.gn_part && d.gn_slots > 0, "fused Swin attention: norm1 statistics");
  RS_CHECK(d.x.H * d.x.W % d.gn_slots == 0,
           "fused Swin attention: norm1 slots must divide H*W = " + std::to_string(d.x.H * d.x.W) + ", got " + std::to_string(d.gn_slots));
  int rc = encode_weight_map(&p.tmWqkv, d.wqkv, d.wqkv_ld, 3 * E, 64); if (rc) return rc;
  rc = encode_weight_map(&p.tmWproj, d.wproj, d.wproj_ld, E, 64); if (rc) return rc;
  p.x = d.x.ptr; p.x_ld = d.x.ld; p.y = d.y.ptr; p.y_ld = d.y.ld;
  p.N = d.x.N; p.H = d.x.H; p.W = d.x.W; p.heads = d.heads; p.shift = d.shift; p.scale = 0.17677669529663687f;
  p.gn_part = d.gn_part; p.gn_slots = d.gn_slots; p.gamma = d.gamma; p.beta = d.beta; p.eps = 1e-5f;
  p.wqkv = d.wqkv; p.wqkv_ld = d.wqkv_ld; p.bqkv = d.bqkv; p.relbias = d.relbias;
  p.wproj = d.wproj; p.wproj_ld = d.wproj_ld; p.bproj = d.bproj;
  p.total_windows = d.x.N * (d.x.H / 8) * (d.x.W / 8);
  // the kernel's epilogue writes one (mean, M2) pair per 8x8 window of 64 tokens, not per 128-pixel conv tile: its
  // slots are windows
  const int nW = (d.x.H / 8) * (d.x.W / 8);
  compact_sinks(d.sink, nW, p.sink);
  const int pairs = (p.total_windows + 1) / 2;
  d.grid = std::min(pairs, num_sms());
  return 0;
}
inline int swin_attn_launch(const SwinAttnDesc& d, cudaStream_t st) {
  if (d.x.C == 192) (void)launch_k(swin_attn_fused_kernel<192>, dim3(d.grid), dim3(kSwinThreads), (size_t)SwinSmem<192>::launch_bytes, st, d.prm);
  else (void)launch_k(swin_attn_fused_kernel<64>, dim3(d.grid), dim3(kSwinThreads), (size_t)SwinSmem<64>::launch_bytes, st, d.prm);
  RS_CUDA_OK(cudaGetLastError());
  return 0;
}

// ---- fused VQ-GAN attention over all positions of an image (vq_attn.cuh) -----------------
struct VqAttnDesc {
  View q, k, v, out;                       // [N, H, W, C]; T = H * W positions per image
  int row_begin = 0, row_end = -1;         // query rows [row_begin, row_end) of every image (-1: T); empty: no launch
  VqAttnParams prm;
};
// sets the query-row range of a (finalized or not) descriptor: multiples of 64 inside [0, T]; an empty range only if
// allow_empty (a plan then skips the launch)
inline int vq_attn_set_rows(VqAttnDesc& d, long long row_begin, long long row_end, bool allow_empty) {
  const long long T = (long long)d.q.H * d.q.W;
  RS_CHECK(row_begin >= 0 && row_begin <= row_end && row_end <= T,
           "fused VQ-GAN attention: rows [" + std::to_string(row_begin) + ", " + std::to_string(row_end) + ") outside [0, T = " + std::to_string(T) + ")");
  RS_CHECK(row_begin % kVqAttnBM == 0 && row_end % kVqAttnBM == 0, "fused VQ-GAN attention: row range bounds must be multiples of 64");
  RS_CHECK(allow_empty || row_end > row_begin, "fused VQ-GAN attention: empty row range");
  d.row_begin = (int)row_begin; d.row_end = (int)row_end;
  d.prm.q_tile0 = (int)(row_begin / kVqAttnBM);
  return 0;
}
inline int vq_attn_finalize(VqAttnDesc& d) {
  VqAttnParams& p = d.prm;
  std::memset(&p, 0, sizeof(p));
  const int N = d.q.N, C = d.q.C;
  const long long T = (long long)d.q.H * d.q.W;
  RS_CHECK(C == 128 || C == 256 || C == 512, "fused VQ-GAN attention: C in {128, 256, 512}, got " + std::to_string(C));
  RS_CHECK(T > 0 && T % kVqAttnBM == 0 && T <= (1LL << 30), "fused VQ-GAN attention: T = H * W must be a positive multiple of 64, got " + std::to_string(T));
  RS_CHECK(N >= 1 && N <= 65535, "fused VQ-GAN attention: batch in [1, 65535]");
  const View* vs[4] = {&d.q, &d.k, &d.v, &d.out};
  for (const View* v : vs) {
    RS_CHECK(v->N == N && (long long)v->H * v->W == T && v->C == C, "fused VQ-GAN attention: q, k, v, out must all be [N, T, C]");
    RS_CHECK(v->ptr != nullptr && v->ld >= C && v->ld % 8 == 0, "fused VQ-GAN attention: rows of >= C elements, 16-byte aligned");
  }
  p.T = (int)T;
  { int rc = vq_attn_set_rows(d, d.row_begin, d.row_end < 0 ? T : d.row_end, true); if (rc) return rc; }
  p.scale_log2 = (float)(1.4426950408889634 / std::sqrt((double)C));
  CUtensorMap* maps[4] = {&p.tmQ, &p.tmK, &p.tmV, &p.tmO};
  const int rows[4] = {kVqAttnBM, vq_attn_bk(C), vq_attn_bk(C), kVqAttnBM};
  for (int i = 0; i < 4; ++i) {
    const View& v = *vs[i];
    int rc = encode_act_map(maps[i], v.ptr, C, (int)T, 1, N, v.ld, T * v.ld, v.sN(), rows[i], 1, 1, 64);
    if (rc) return rc;
  }
  return 0;
}
inline int vq_attn_launch(const VqAttnDesc& d, cudaStream_t st) {
  if (d.row_end == d.row_begin) return 0;
  const dim3 grid((unsigned)((d.row_end - d.row_begin) / kVqAttnBM), (unsigned)d.q.N);
  switch (d.q.C) {
    case 128: (void)launch_k(vq_attn_sm90_kernel<128>, grid, dim3(kVqAttnThreads), (size_t)VqAttnSmem<128>::launch_bytes, st, d.prm); break;
    case 256: (void)launch_k(vq_attn_sm90_kernel<256>, grid, dim3(kVqAttnThreads), (size_t)VqAttnSmem<256>::launch_bytes, st, d.prm); break;
    case 512: (void)launch_k(vq_attn_sm90_kernel<512>, grid, dim3(kVqAttnThreads), (size_t)VqAttnSmem<512>::launch_bytes, st, d.prm); break;
    default: RS_CHECK(false, "fused VQ-GAN attention: C in {128, 256, 512}");
  }
  RS_CUDA_OK(cudaGetLastError());
  return 0;
}

// ---- multi-head attention over all positions of a level (unet_attn.cuh): UNetModel's AttentionBlock -----------------
struct UnetAttnDesc {
  View qkv, out;                           // [N, H, W, 3C] (the qkv conv's output), [N, H, W, C]
  int heads = 1;
  bool new_order = false;                  // QKVAttention (split qkv, then heads) instead of QKVAttentionLegacy
  UnetAttnParams prm;
};
inline bool unet_attn_head_dim_ok(int D) { return D == 32 || D == 64 || D == 128; }
inline int unet_attn_finalize(UnetAttnDesc& d) {
  UnetAttnParams& p = d.prm;
  std::memset(&p, 0, sizeof(p));
  const int N = d.qkv.N, C = d.out.C;
  const long long T = (long long)d.qkv.H * d.qkv.W;
  RS_CHECK(d.heads > 0 && C % d.heads == 0 && unet_attn_head_dim_ok(C / d.heads),
           "UNetModel attention: head dim (channels / heads) must be 32, 64 or 128");
  const int D = C / d.heads;
  RS_CHECK(d.qkv.C == 3 * C && d.out.N == N && (long long)d.out.H * d.out.W == T, "UNetModel attention: qkv [N, T, 3C] -> out [N, T, C]");
  RS_CHECK(T >= 1 && T <= (1LL << 30) && N >= 1 && N <= 65535 && d.heads <= 65535, "UNetModel attention: T >= 1, batch and heads <= 65535");
  RS_CHECK(d.qkv.ptr && d.out.ptr && d.qkv.ld % 8 == 0 && d.out.ld % 2 == 0 && d.out.ld >= C, "UNetModel attention: views");
  p.out = d.out.ptr; p.out_sN = d.out.sN(); p.out_ld = d.out.ld;
  p.T = (int)T;
  p.head_stride = d.new_order ? D : 3 * D;
  p.k_col0 = d.new_order ? C : D;
  p.v_col0 = d.new_order ? 2 * C : 2 * D;
  p.scale_log2 = (float)(1.4426950408889634 / std::sqrt((double)D));
  return encode_act_map(&p.tm, d.qkv.ptr, 3 * C, (int)T, 1, N, d.qkv.ld, T * d.qkv.ld, d.qkv.sN(), kUnetAttnBK, 1, 1, 64);
}
inline int unet_attn_launch(const UnetAttnDesc& d, cudaStream_t st) {
  const long long T = (long long)d.qkv.H * d.qkv.W;
  const dim3 grid((unsigned)((T + kUnetAttnCtaRows - 1) / kUnetAttnCtaRows), (unsigned)d.heads, (unsigned)d.qkv.N);
  switch (d.out.C / d.heads) {
    case 32: (void)launch_k(unet_attn_sm90_kernel<32>, grid, dim3(kUnetAttnThreads), (size_t)UnetAttnSmem<32>::launch_bytes, st, d.prm); break;
    case 64: (void)launch_k(unet_attn_sm90_kernel<64>, grid, dim3(kUnetAttnThreads), (size_t)UnetAttnSmem<64>::launch_bytes, st, d.prm); break;
    case 128: (void)launch_k(unet_attn_sm90_kernel<128>, grid, dim3(kUnetAttnThreads), (size_t)UnetAttnSmem<128>::launch_bytes, st, d.prm); break;
    default: RS_CHECK(false, "UNetModel attention: head dim 32, 64 or 128");
  }
  RS_CUDA_OK(cudaGetLastError());
  return 0;
}

// heads per CTA of window_attn_kernel when the caller does not ask for a count: all of them when there are plenty of
// windows, fewer (more CTAs) otherwise
inline int attn_default_hpc(int heads, long long windows) {
  int hpc = heads;
  while (hpc > 1 && windows * (heads / hpc) < 4 * num_sms() && hpc % 2 == 0) hpc /= 2;
  if (hpc > 1 && windows * (heads / hpc) < 4 * num_sms() && heads % hpc == 0) hpc = 1;
  return hpc;
}

// what one launch of the window-attention core runs: the SIMT cross-check (one head per CTA) or the instance of
// window_attn_kernel with hpc heads per CTA
struct AttnLaunch { bool simt; int hpc; dim3 grid; size_t smem; };

// one launch of the window-attention core: the instance of window_attn_kernel for (window side, head width), or with
// simt the SIMT cross-check (RS_ATTN_IMPL=simt).  hpc = heads per CTA (0: attn_default_hpc); *info = what was launched
template <int WS, int HD>
inline int attn_launch_instance(WinAttnParams& p, int windows, int hpc, AttnLaunch* info, cudaStream_t st) {
  const int heads = p.heads;
  p.hpc = hpc ? hpc : attn_default_hpc(heads, windows);
  // (at WS = 8 sized for the output channels of all heads: an upper bound of what hpc heads stage)
  const size_t smem = window_attn_smem_bytes<WS, HD>(WS == 8 ? heads : p.hpc);
  RS_CHECK(smem <= (size_t)kAttnMaxSmem, "attention tile does not fit in shared memory");   // limit raised in conv_init()
  const dim3 grid(windows, heads / p.hpc);
  if (info) *info = AttnLaunch{false, p.hpc, grid, smem};
  (void)launch_k(window_attn_kernel<WS, HD>, grid, dim3(WS == 8 ? 128 : 256), smem, st, p);
  return 0;
}

inline int attn_launch(const View& qkv, const View& out, const float* bias, int heads, int E, int window, int shift,
                       bool simt, cudaStream_t st, int hpc = 0, AttnLaunch* info = nullptr) {
  RS_CHECK(window == 8 || window == 16, "window attention kernels: window_size 8 or 16, got " + std::to_string(window));
  RS_CHECK(heads > 0 && E % heads == 0 && (E / heads == 32 || E / heads == 64),
           "window attention kernels: head_dim 32 or 64");
  RS_CHECK(qkv.H % window == 0 && qkv.W % window == 0,
           "window attention needs H, W multiples of the window (" + std::to_string(window) + ")");
  RS_CHECK(shift == 0 || shift == window / 2, "window attention: shift is 0 or half the window");
  RS_CHECK(hpc >= 0 && (hpc == 0 || heads % hpc == 0),
           "window attention: hpc must divide heads = " + std::to_string(heads) + ", got " + std::to_string(hpc));
  RS_CHECK(!simt || hpc <= 1, "window attention: hpc must be 0 or 1 for the SIMT kernel (one head per CTA)");
  const int hd = E / heads;
  const int windows = qkv.N * (qkv.H / window) * (qkv.W / window);
  WinAttnParams p{qkv.ptr, qkv.ld, out.ptr, out.ld, bias, qkv.N, qkv.H, qkv.W, heads, E, shift,
                  hd == 32 ? 0.17677669529663687f : 0.125f, heads, window, hd};
  int rc = 0;
  if (simt) {
    if (info) *info = AttnLaunch{true, 1, dim3(windows, heads), 0};
    (void)launch_k(window_attn_simt_kernel, dim3(windows, heads), dim3(window * window), (size_t)0, st, p);
  } else if (window == 8) {
    rc = hd == 32 ? attn_launch_instance<8, 32>(p, windows, hpc, info, st) : attn_launch_instance<8, 64>(p, windows, hpc, info, st);
  } else {
    rc = hd == 32 ? attn_launch_instance<16, 32>(p, windows, hpc, info, st) : attn_launch_instance<16, 64>(p, windows, hpc, info, st);
  }
  if (rc) return rc;
  RS_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace rs

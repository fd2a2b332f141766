// Fused (shifted-)window multi-head self-attention core: windows of WS x WS tokens (WS = 8 or 16), heads HD wide
// (HD = 32 or 64); T = WS * WS tokens per window.
//
// reference: WindowAttention.forward (models/swin_transformer.py:114-145) together with the
// data movement around it in SwinTransformerBlock.forward (:251-275): torch.roll(-s), window_partition,
// q*scale, q@k^T, + relative-position bias, + shift mask, softmax, @v, window_reverse, torch.roll(+s).
// All of the movement is address arithmetic here: token (r, c) of window (wy, wx) of image n lives at
// pixel ((wy*WS + r + s) % H, (wx*WS + c + s) % W) of the un-shifted NHWC tensor, for reads and writes.
//
//   qkv : [N*H*W, 3*E] fp16, channel = which*E + head*HD + d      (output of the qkv GEMM, bias included)
//   out : [N*H*W, E]   fp16, channel = head*HD + d                (input of the proj GEMM)
//   bias: [heads][T][T] fp32, relative_position_bias_table gathered by relative_position_index
//   mask: generated on the fly; reproduces the reference's calculate_mask (:214-236) including its
//         axis quirks (see resshift_b200/arch.py::shifted_window_mask): label(token) = region(wy*WS + c).
//
// window_attn_kernel<WS, HD>: one CTA per window, looping over its heads.
//   WS = 8: 4 warps x 16 query rows and a double-buffered cp.async pipeline (head h+1 streams in while head h is
//   computed).  QK^T and PV run on mma.sync m16n8k16 with the score tile kept in registers (the C fragment of QK^T is
//   the A fragment of PV); V is read through ldmatrix.trans; the 64 x E output tile is staged in shared memory and
//   written as full 2*E-byte rows.
//   WS = 16: 256 queries against 256 keys per head on wgmma.  Two warpgroups, each taking two chunks of 64 query rows:
//   S = Q K^T is one m64n256 accumulator (128 fp32 registers per thread), so the softmax is a plain row softmax in
//   registers and P is the register A operand of P V, with V stored transposed as swin_attn_fused.cuh does.  q, k and
//   v^T of one head sit in 128-byte-swizzled K-major tiles; a chunk's output rows replace its (dead) q rows and leave
//   as HD-wide row segments.  The heads are not pipelined: q / k / v^T of the next head load after the last chunk.
// window_attn_simt_kernel is a plain fp32 version for every (WS, HD), kept as a cross-check (RS_ATTN_IMPL=simt).
#pragma once

#include "common.cuh"
#include "wgmma.cuh"

namespace rs {

struct WinAttnParams {
  const __half* qkv; int qkv_ld;
  __half* out; int out_ld;
  const float* bias;        // [heads][WS*WS][WS*WS]
  int N, H, W, heads, E;
  int shift;                // 0 or WS / 2
  float scale;              // head_dim^-0.5
  int hpc;                  // heads per CTA (grid.y = heads / hpc): fewer heads per CTA when there are few windows
  int ws, hd;               // window side, head width: the instance of window_attn_kernel; read by the SIMT cross-check
};

#ifdef __CUDACC__

__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ void cp_async_16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// two 8x8 b16 matrices, transposed on load: the B fragment (k x n, "col") of m16n8k16 from a row-major [k][n] tile
__device__ __forceinline__ void ldmatrix_x2_trans(uint32_t (&r)[2], const void* row_addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];"
               : "=r"(r[0]), "=r"(r[1])
               : "r"(smem_u32(row_addr)));
}

// region label of a token for the shifted-window mask (reference quirk: depends on wy and the token COLUMN)
__device__ __forceinline__ int swin_label(int wy, int c, int H, int shift, int ws = 8) {
  const int y = wy * ws + c;
  return (y < H - ws) ? 0 : ((y < H - shift) ? 1 : 2);
}

// shared memory of one CTA.  WS = 8: [2 buffers][q | k | v][64][HD + 8] halves (8 halves of padding: conflict-free
// fragment reads and ldmatrix rows), the output tile [64][hpc * HD + 8] halves, the pixel table.  WS = 16: q and k as
// [256][64] halves in rows of 128 bytes (HD = 32 fills half of each row), v^T as four [HD][64 keys] blocks, the pixel
// table, and the slack that aligns the tiles to the 1024 bytes of the swizzle pattern.
constexpr int kAttnMaxSmem = 160 * 1024;     // dynamic shared memory every instance may ask for
template <int WS, int HD>
constexpr size_t window_attn_smem_bytes(int hpc) {
  return WS == 8 ? (size_t)2 * 3 * 64 * (HD + 8) * 2 + (size_t)64 * (hpc * HD + 8) * 2 + 64 * sizeof(int)
                 : (size_t)2 * 256 * 128 + (size_t)4 * HD * 128 + 256 * sizeof(int) + 1024;
}

template <int WS, int HD>
__global__ void __launch_bounds__(WS == 8 ? 128 : 256) window_attn_kernel(const WinAttnParams p) {
  static_assert((WS == 8 || WS == 16) && (HD == 32 || HD == 64), "window attention: windows of 8 or 16, heads of 32 or 64");
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) uint8_t attn_smem[];
  constexpr int T = WS * WS;
  const int head0 = blockIdx.y * p.hpc;
  const int nWx = p.W / WS, nWy = p.H / WS;
  int win = blockIdx.x;
  const int wx = win % nWx; win /= nWx;
  const int wy = win % nWy; win /= nWy;
  const int n = win;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;

  if constexpr (WS == 8) {
    constexpr int kPad = HD + 8;             // halves per smem row
    constexpr int kParts = HD / 8;           // 16-byte pieces of a head's row
    __half* sbuf = reinterpret_cast<__half*>(attn_smem);
    const int buf_halves = 3 * 64 * kPad;
    const int opitch = p.hpc * HD + 8;
    __half* sOut = sbuf + 2 * buf_halves;
    int* sPix = reinterpret_cast<int*>(sOut + 64 * opitch);

    if (threadIdx.x < 64) {
      const int r = threadIdx.x >> 3, c = threadIdx.x & 7;
      const int y = (wy * 8 + r + p.shift) % p.H;
      const int x = (wx * 8 + c + p.shift) % p.W;
      sPix[threadIdx.x] = (n * p.H + y) * p.W + x;
    }
    __syncthreads();

    auto stage_head = [&](int head, int buf) {
      __half* dst = sbuf + buf * buf_halves;
      for (int i = threadIdx.x; i < 64 * 3 * kParts; i += 128) {
        const int tok = i / (3 * kParts), rem = i - tok * 3 * kParts, which = rem / kParts, part = rem % kParts;
        const __half* src = p.qkv + (long long)sPix[tok] * p.qkv_ld + which * p.E + head * HD + part * 8;
        cp_async_16(dst + which * 64 * kPad + tok * kPad + part * 8, src);
      }
      cp_async_commit();
    };

    const int row0 = warp * 16 + g;          // this lane's rows: row0 and row0 + 8
    const int la = p.shift ? swin_label(wy, row0 & 7, p.H, p.shift) : 0;     // (row0 + 8) & 7 == row0 & 7

    stage_head(head0, 0);
    for (int hi = 0; hi < p.hpc; ++hi) {
      const int head = head0 + hi;
      const int buf = hi & 1;
      // this lane's 32 relative-position-bias values (a load-time table, independent of the staged q/k/v): issued before
      // waiting for the tile so the L2 round trip hides under the cp.async wait and the QK^T MMAs
      const float* bias = p.bias + (long long)head * 64 * 64;
      float2 bv0[8], bv1[8];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        bv0[nt] = __ldg(reinterpret_cast<const float2*>(bias + row0 * 64 + nt * 8 + 2 * t));
        bv1[nt] = __ldg(reinterpret_cast<const float2*>(bias + (row0 + 8) * 64 + nt * 8 + 2 * t));
      }
      if (hi + 1 < p.hpc) { stage_head(head + 1, buf ^ 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
      __syncthreads();
      const __half* sQ = sbuf + buf * buf_halves;
      const __half* sK = sQ + 64 * kPad;
      const __half* sV = sK + 64 * kPad;

      // S = Q K^T : Q fragments for the HD / 16 k-steps
      uint32_t qa[HD / 16][4];
#pragma unroll
      for (int ks = 0; ks < HD / 16; ++ks) {
        const int d = ks * 16 + 2 * t;
        qa[ks][0] = *reinterpret_cast<const uint32_t*>(&sQ[row0 * kPad + d]);
        qa[ks][1] = *reinterpret_cast<const uint32_t*>(&sQ[(row0 + 8) * kPad + d]);
        qa[ks][2] = *reinterpret_cast<const uint32_t*>(&sQ[row0 * kPad + d + 8]);
        qa[ks][3] = *reinterpret_cast<const uint32_t*>(&sQ[(row0 + 8) * kPad + d + 8]);
      }
      float s[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
        for (int ks = 0; ks < HD / 16; ++ks) {
          const int key = nt * 8 + g, d = ks * 16 + 2 * t;
          uint32_t kb[2];
          kb[0] = *reinterpret_cast<const uint32_t*>(&sK[key * kPad + d]);
          kb[1] = *reinterpret_cast<const uint32_t*>(&sK[key * kPad + d + 8]);
          mma_16816(s[nt], qa[ks], kb);
        }
      }
      // scale, bias, mask; row-wise softmax (each row is spread over the 4 lanes of a quad)
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

      // O = P V : k = keys (4 steps of 16), n = d (HD / 8 tiles of 8); V[key][d] row-major, read transposed
      float o[HD / 8][4];
#pragma unroll
      for (int dt = 0; dt < HD / 8; ++dt) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        uint32_t pa[4];
        pa[0] = pack_h2(s[2 * kk][0], s[2 * kk][1]);
        pa[1] = pack_h2(s[2 * kk][2], s[2 * kk][3]);
        pa[2] = pack_h2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
        pa[3] = pack_h2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
        for (int dt = 0; dt < HD / 8; ++dt) {
          // lanes 0..15 name the 16 key rows of this k-step (lanes 16..31 are ignored by .x2 but must be valid)
          uint32_t vb[2];
          ldmatrix_x2_trans(vb, &sV[(kk * 16 + (lane & 15)) * kPad + dt * 8]);
          mma_16816(o[dt], pa, vb);
        }
      }
      const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;
#pragma unroll
      for (int dt = 0; dt < HD / 8; ++dt) {
        const int d = hi * HD + dt * 8 + 2 * t;
        *reinterpret_cast<__half2*>(&sOut[row0 * opitch + d]) = __floats2half2_rn(o[dt][0] * inv0, o[dt][1] * inv0);
        *reinterpret_cast<__half2*>(&sOut[(row0 + 8) * opitch + d]) = __floats2half2_rn(o[dt][2] * inv1, o[dt][3] * inv1);
      }
      __syncthreads();      // everyone done with this head's buffer before it is refilled two iterations later
    }
    // write this CTA's 64 x (hpc*HD) slice as contiguous row segments
    const int units = p.hpc * kParts;
    for (int i = threadIdx.x; i < 64 * units; i += 128) {
      const int tok = i / units, u = i - tok * units;
      *reinterpret_cast<uint4*>(p.out + (long long)sPix[tok] * p.out_ld + head0 * HD + u * 8) =
          *reinterpret_cast<const uint4*>(&sOut[tok * opitch + u * 8]);
    }
  } else {
    constexpr int kParts = HD / 8;
    constexpr int kBlk = T * 128;                                        // q or k: [256 tokens][128 B]
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(attn_smem) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + kBlk;
    uint8_t* sVt = sK + kBlk;                                            // [4 blocks of 64 keys][HD][128 B]
    int* sPix = reinterpret_cast<int*>(sVt + 4 * HD * 128);
    // byte offset of (row r, halves c .. c + 1) in a swizzled block of 128-byte rows
    auto swz = [](int r, int c) { return r * 128 + ((((c >> 3) ^ r) & 7) << 4) + (c & 7) * 2; };

    {
      const int r = threadIdx.x >> 4, c = threadIdx.x & 15;
      const int y = (wy * 16 + r + p.shift) % p.H;
      const int x = (wx * 16 + c + p.shift) % p.W;
      sPix[threadIdx.x] = (n * p.H + y) * p.W + x;
    }
    __syncthreads();

    const int wg = warp >> 2, wt = threadIdx.x & 127;
    for (int hi = 0; hi < p.hpc; ++hi) {
      const int head = head0 + hi;
      // ---- q and k rows by cp.async; v through registers, transposed ----
      for (int i = threadIdx.x; i < 2 * T * kParts; i += 256) {
        const int which = i / (T * kParts), rem = i - which * T * kParts, tok = rem / kParts, part = rem % kParts;
        cp_async_16(sQ + which * kBlk + swz(tok, part * 8),
                    p.qkv + (long long)sPix[tok] * p.qkv_ld + which * p.E + head * HD + part * 8);
      }
      cp_async_commit();
      {
        const int key = threadIdx.x;                                     // a warp: 32 keys of one row of v^T per store
        const uint4* src = reinterpret_cast<const uint4*>(p.qkv + (long long)sPix[key] * p.qkv_ld + 2 * p.E + head * HD);
        uint4 v[kParts];
#pragma unroll
        for (int part = 0; part < kParts; ++part) v[part] = __ldg(src + part);
        uint8_t* blk = sVt + (key >> 6) * HD * 128;
#pragma unroll
        for (int part = 0; part < kParts; ++part) {
          const __half* hv = reinterpret_cast<const __half*>(&v[part]);
#pragma unroll
          for (int e = 0; e < 8; ++e) *reinterpret_cast<__half*>(blk + swz(part * 8 + e, key & 63)) = hv[e];
        }
      }
      cp_async_wait<0>();
      fence_proxy_async_smem();                                          // the tensor core reads through the async proxy
      __syncthreads();

      const float* bias = p.bias + (long long)head * T * T;
#pragma unroll 1
      for (int chunk = 0; chunk < 2; ++chunk) {
        const int base = (2 * wg + chunk) * 64;                          // this warpgroup's 64 query rows
        const int r0 = base + 16 * (warp & 3) + g;                       // this thread's rows: r0 and r0 + 8
        // S = Q K^T: register 4 nt + e holds row r0 + 8 (e >> 1), key 8 nt + 2 t + (e & 1)
        float s[128];
#pragma unroll
        for (int i = 0; i < 128; ++i) s[i] = 0.f;
        const uint64_t qdesc = wgmma_desc_sw128(smem_u32(sQ) + (uint32_t)(base * 128));
        const uint64_t kdesc = wgmma_desc_sw128(smem_u32(sK));
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < HD / 16; ++kk) Wgmma<256>::mma(s, qdesc + 2 * kk, kdesc + 2 * kk);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(s);
        // scale, bias, mask (the label of a token depends on its column r & 15: rows r0 and r0 + 8 differ)
        const int la0 = p.shift ? swin_label(wy, r0 & 15, p.H, p.shift, 16) : 0;
        const int la1 = p.shift ? swin_label(wy, (r0 + 8) & 15, p.H, p.shift, 16) : 0;
        float mx0 = -1e30f, mx1 = -1e30f;
#pragma unroll
        for (int nt = 0; nt < 32; ++nt) {
          const int col = nt * 8 + 2 * t;
          const float2 b0 = __ldg(reinterpret_cast<const float2*>(bias + r0 * T + col));
          const float2 b1 = __ldg(reinterpret_cast<const float2*>(bias + (r0 + 8) * T + col));
          float m00 = 0.f, m01 = 0.f, m10 = 0.f, m11 = 0.f;
          if (p.shift) {
            const int l0 = swin_label(wy, col & 15, p.H, p.shift, 16), l1 = swin_label(wy, (col + 1) & 15, p.H, p.shift, 16);
            if (l0 != la0) m00 = -100.0f;
            if (l1 != la0) m01 = -100.0f;
            if (l0 != la1) m10 = -100.0f;
            if (l1 != la1) m11 = -100.0f;
          }
          s[4 * nt + 0] = s[4 * nt + 0] * p.scale + b0.x + m00;
          s[4 * nt + 1] = s[4 * nt + 1] * p.scale + b0.y + m01;
          s[4 * nt + 2] = s[4 * nt + 2] * p.scale + b1.x + m10;
          s[4 * nt + 3] = s[4 * nt + 3] * p.scale + b1.y + m11;
          mx0 = fmaxf(mx0, fmaxf(s[4 * nt + 0], s[4 * nt + 1]));
          mx1 = fmaxf(mx1, fmaxf(s[4 * nt + 2], s[4 * nt + 3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
        for (int nt = 0; nt < 32; ++nt) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            s[4 * nt + e] = __expf(s[4 * nt + e] - mx0); sum0 += s[4 * nt + e];
            s[4 * nt + 2 + e] = __expf(s[4 * nt + 2 + e] - mx1); sum1 += s[4 * nt + 2 + e];
          }
        }
        sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1); sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
        sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1); sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
        // O = P V: P (fp16) as the A operand, k-step kk = keys 16 kk .. 16 kk + 15 = registers 8 kk .. 8 kk + 7
        uint32_t pa[16][4];
#pragma unroll
        for (int kk = 0; kk < 16; ++kk)
#pragma unroll
          for (int rr = 0; rr < 4; ++rr) pa[kk][rr] = pack_h2(s[8 * kk + 2 * rr], s[8 * kk + 2 * rr + 1]);
        float o[HD / 2];
#pragma unroll
        for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 16; ++kk)
          WgmmaRs<HD>::mma(o, pa[kk], wgmma_desc_sw128(smem_u32(sVt) + (uint32_t)((kk >> 2) * HD * 128)) + 2 * (kk & 3));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        // the chunk's q rows are dead (the warpgroup's QK^T retired): its output rows replace them, then leave as
        // HD-wide row segments
        named_bar_sync(1 + wg, 128);
        const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;
#pragma unroll
        for (int i = 0; i < HD / 8; ++i) {
          const int cc = 8 * i + 2 * t;
          *reinterpret_cast<__half2*>(sQ + swz(r0, cc)) = __floats2half2_rn(o[4 * i] * inv0, o[4 * i + 1] * inv0);
          *reinterpret_cast<__half2*>(sQ + swz(r0 + 8, cc)) = __floats2half2_rn(o[4 * i + 2] * inv1, o[4 * i + 3] * inv1);
        }
        named_bar_sync(1 + wg, 128);
        for (int i = wt; i < 64 * kParts; i += 128) {
          const int r = base + i / kParts, u = i % kParts;
          *reinterpret_cast<uint4*>(p.out + (long long)sPix[r] * p.out_ld + head * HD + u * 8) =
              *reinterpret_cast<const uint4*>(sQ + swz(r, u * 8));
        }
      }
      __syncthreads();      // every read of this head's q (output rows), k and v^T retired before the next head lands
    }
  }
}

// Plain fp32 cross-check for any window side p.ws <= 16 and head width p.hd <= 64: one CTA of ws * ws threads per
// (window, head), one thread per query row, k and v read from global memory.
__global__ void __launch_bounds__(256) window_attn_simt_kernel(const WinAttnParams p) {
  pdl_trigger();
  pdl_wait();
  const int ws = p.ws, hd = p.hd, T = ws * ws;
  const int head = blockIdx.y;
  const int nWx = p.W / ws, nWy = p.H / ws;
  int win = blockIdx.x;
  const int wx = win % nWx; win /= nWx;
  const int wy = win % nWy; win /= nWy;
  const int n = win;
  auto pixel = [&](int tok) {
    const int y = (wy * ws + tok / ws + p.shift) % p.H, x = (wx * ws + tok % ws + p.shift) % p.W;
    return ((long long)n * p.H + y) * p.W + x;
  };
  const int i = threadIdx.x;
  const long long pix = pixel(i);
  const __half* row = p.qkv + pix * p.qkv_ld + head * hd;
  float q[64];
  for (int d = 0; d < hd; ++d) q[d] = __half2float(row[d]) * p.scale;
  const float* bias = p.bias + (long long)head * T * T;
  const int li = p.shift ? swin_label(wy, i % ws, p.H, p.shift, ws) : 0;
  float sc[256];
  float mx = -1e30f;
  for (int j = 0; j < T; ++j) {
    const __half* kr = p.qkv + pixel(j) * p.qkv_ld + p.E + head * hd;
    float s = 0.f;
    for (int d = 0; d < hd; ++d) s = fmaf(q[d], __half2float(kr[d]), s);
    s += bias[i * T + j];
    if (p.shift && swin_label(wy, j % ws, p.H, p.shift, ws) != li) s += -100.0f;
    sc[j] = s; mx = fmaxf(mx, s);
  }
  float sum = 0.f;
  for (int j = 0; j < T; ++j) { sc[j] = __expf(sc[j] - mx); sum += sc[j]; }
  const float inv = 1.0f / sum;
  __half* dst = p.out + pix * p.out_ld + head * hd;
  for (int d = 0; d < hd; ++d) {
    float o = 0.f;
    for (int j = 0; j < T; ++j) o = fmaf(sc[j], __half2float(p.qkv[pixel(j) * p.qkv_ld + 2 * p.E + head * hd + d]), o);
    dst[d] = __float2half_rn(o * inv);
  }
}

#endif
}  // namespace rs

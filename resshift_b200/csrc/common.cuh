// Common device/host helpers for the ResShift H100 (sm_90a) kernels.
// Raw PTX wrappers for mbarrier / TMA / clusters / wgmma (no CUTLASS dependency).
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <string>

namespace rs {

// ----------------------------------------------------------------------------------------
// Error plumbing: every C-ABI entry point returns 0 or a negative code; the message is kept
// in a thread-local string readable through rs_last_error().
// ----------------------------------------------------------------------------------------
void set_error(const std::string& msg);
int fail(int code, const std::string& msg);

#define RS_CUDA_OK(expr)                                                                       \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      (void)cudaGetLastError(); /* clear the error so later calls report their own */            \
      return ::rs::fail(-2, std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " (" + \
                                __FILE__ + ":" + std::to_string(__LINE__) + ")");              \
    }                                                                                          \
  } while (0)

#define RS_CHECK(cond, msg)                                                              \
  do {                                                                                   \
    if (!(cond)) {                                                                       \
      return ::rs::fail(-1, std::string("check failed: ") + #cond + " — " + (msg) + " (" + \
                                __FILE__ + ":" + std::to_string(__LINE__) + ")");        \
    }                                                                                    \
  } while (0)

#ifdef __CUDACC__

// ----------------------------------------------------------------------------------------
// small device utilities
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// Programmatic dependent launch: `pdl_trigger` lets the next kernel in the stream start its prologue
// early; `pdl_wait` blocks until every prerequisite grid has completed and its writes are visible.
// Every kernel of this library calls pdl_wait() before its first access to global memory.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// x * sigmoid(x): ex2 + approximate reciprocal (2 ulp), no IEEE-division fix-up sequence (the GroupNorm pass that
// applies it is bound by instruction issue / MUFU, not by memory)
__device__ __forceinline__ float silu_f(float v) { return __fdividef(v, 1.0f + __expf(-v)); }
// exact-erf GELU (nn.GELU default, reference models/swin_transformer.py:18):  0.5 x (1 + erf(x / sqrt 2)).
// erf(z) = sign(z) (1 - 2^P(|z|)) with P a degree-7 minimax-style fit of log2(erfc) on [0, 4] (clamped beyond):
// |erf error| <= 4.3e-6, |GELU error| <= 6.4e-7 over all x — three orders below the fp16 rounding of the stored
// result — for one MUFU (ex2) and nine FMAs (the epilogues that apply it are instruction-bound).
__device__ __forceinline__ float gelu_erf_f(float v) {
  const float z = fminf(fabsf(v) * 0.70710678118654752f, 4.0f);
  float pz = fmaf(z, -2.177763781e-05f, 5.068330793e-04f);
  pz = fmaf(z, pz, -5.339398049e-03f);
  pz = fmaf(z, pz, 3.423144668e-02f);
  pz = fmaf(z, pz, -1.528908461e-01f);
  pz = fmaf(z, pz, -9.167589545e-01f);
  pz = fmaf(z, pz, -1.628154397e+00f);
  pz = fmaf(z, pz, 6.178960575e-06f);
  float ex;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ex) : "f"(pz));
  // 0.5 v (1 + sign(v) (1 - ex))  =  h + |h| - |h| ex   with h = v / 2
  const float h = 0.5f * v;
  return h + fmaf(-fabsf(h), ex, fabsf(h));
}

// ----------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Arrive on a barrier that lives in another CTA of the cluster (address from mapa_u32) with the default CTA-scope
// release.  The cluster-scope form (mbarrier.arrive.release.cluster) fences at cluster scope and is not needed when the
// remote waiter only needs the count: the consumer warps arrive after wgmma.wait_group shows their reads of the slot
// retired, so the peer's next TMA write into it cannot overtake them.
__device__ __forceinline__ void mbar_arrive_remote(uint32_t bar_cluster_addr) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(bar_cluster_addr) : "memory");
}
// Bounded spin: a pipeline bug must not hang the GPU; after ~2 s of polling the kernel traps instead, which surfaces
// as a launch failure on the host.
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = global_timer_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0xFFu) == 0 && global_timer_ns() - t0 > 2000000000ull) __trap();   // (no printf: a call here
                                                                                        // would serialise the wgmma pipeline)
  }
}

// ----------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor), tile mode, completion on an mbarrier
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ---- clusters: rank, cluster-wide barrier, distributed shared memory, TMA multicast ----
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cta address -> shared::cluster address of the same offset in CTA `rank`
__device__ __forceinline__ uint32_t mapa_u32(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
// 16-byte load from the shared memory of another CTA of the cluster (address from mapa_u32)
__device__ __forceinline__ float4 ld_shared_cluster_f4(uint32_t cluster_addr) {
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(cluster_addr)
               : "memory");
  return v;
}
// 2-D tile load written to the same shared-memory offset of every CTA in `cta_mask`; each destination CTA's barrier at
// the offset of `bar` receives the bytes that landed there
__device__ __forceinline__ void tma_load_2d_mc(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}

// smem -> global tile store (bulk async group), coordinates clip out-of-bounds elements
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the staged shared memory has been READ by every committed store (it may be reused / the CTA may exit); the global
// writes themselves complete asynchronously, at the latest at kernel completion
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// same, but the most recent committed store may still be reading (double-buffered staging)
__device__ __forceinline__ void tma_store_wait_read_keep1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
// generic-proxy smem writes -> visible to the async proxy (TMA store reads them)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ----------------------------------------------------------------------------------------
// wgmma (Hopper warpgroup MMA, accumulators in registers; the instruction wrappers are in wgmma.cuh)
// ----------------------------------------------------------------------------------------
// registers and shared memory written before this point are ordered before the warpgroup's next wgmma
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// at most kPending committed groups of this warpgroup are still in flight (their operands may still be read)
template <int kPending>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory"); }
// keeps the accumulator registers live across the wait: no use of them is scheduled before it
template <int kRegs>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[kRegs]) {
#pragma unroll
  for (int i = 0; i < kRegs; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor, K-major operand, 128-byte swizzle (sm_90 layout):
//   rows are 128 B (64 fp16) apart, 8-row groups 1024 B apart (SBO).  Bit layout follows the PTX ISA "matrix
//   descriptor" of wgmma (start addr [0,14), LBO [16,30), SBO [32,46), base offset [49,52), swizzle [62,64) with
//   SWIZZLE_128B = 1).  Advancing 16 fp16 (32 B) along K inside the swizzled row is +2 on the address field.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;            // LBO (ignored for swizzled K-major); 16 B
  d |= static_cast<uint64_t>(1024 >> 4) << 32;    // SBO = 1024 B
  d |= static_cast<uint64_t>(1) << 62;            // SWIZZLE_128B
  return d;
}

#endif  // __CUDACC__

}  // namespace rs

// Common device/host helpers for the sm_90a kernels: error plumbing for the C-ABI,
// and thin inline-PTX wrappers for mbarrier, TMA (cp.async.bulk.tensor) and
// wgmma (descriptors / fence / commit / wait).  No CUTLASS: everything is spelled out.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/yolob200.h"

namespace yb {

// ----------------------------------------------------------------------------------
// host-side error plumbing
// ----------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define YB_CUDA(call)                                                        \
  do {                                                                       \
    cudaError_t _e = (call);                                                 \
    if (_e != cudaSuccess) return yb::cuda_fail(_e, #call, __FILE__, __LINE__); \
  } while (0)

#define YB_REQUIRE(cond, ...)                \
  do {                                       \
    if (!(cond)) {                           \
      yb::set_error(__VA_ARGS__);            \
      return YB_ERR_INVALID_ARGUMENT;        \
    }                                        \
  } while (0)

static inline int ceil_div(long a, long b) { return (int)((a + b - 1) / b); }
int num_sms();
// runtime switches (csrc/capi.cu): "" when unset
const char* opt(const char* key);
int opt_int(const char* key, int dflt);
struct DeviceOnce { unsigned long long mask = 0; };
int ensure_smem_attr(DeviceOnce& once, const void* kernel, int bytes);

// ----------------------------------------------------------------------------------
// storage dtype helpers (activations/weights are fp16 or bf16; math is fp32)
// ----------------------------------------------------------------------------------
template <typename T> struct Pack2;
template <> struct Pack2<__half> {
  static __device__ __forceinline__ uint32_t pack(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  static __device__ __forceinline__ float2 unpack(uint32_t u) {
    return __half22float2(*reinterpret_cast<__half2*>(&u));
  }
};
template <> struct Pack2<__nv_bfloat16> {
  static __device__ __forceinline__ uint32_t pack(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  static __device__ __forceinline__ float2 unpack(uint32_t u) {
    return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
  }
};

__device__ __forceinline__ float leaky01(float v) { return v > 0.f ? v : 0.1f * v; }

// e4m3 storage (the fp8 inference plan): cvt.rn.satfinite rounds to nearest even and saturates to +-448.
// a -> the low byte (the lower address), b -> the high byte.
__device__ __forceinline__ uint32_t e4m3x2_pack(float a, float b) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(b), "f"(a));
  return r;
}
// 16 values times `mul` -> 16 e4m3 codes in memory order
__device__ __forceinline__ uint4 e4m3x16_pack(const float (&v)[16], float mul) {
  uint32_t w[4];
#pragma unroll
  for (int j = 0; j < 4; ++j)
    w[j] = e4m3x2_pack(v[4 * j] * mul, v[4 * j + 1] * mul) | (e4m3x2_pack(v[4 * j + 2] * mul, v[4 * j + 3] * mul) << 16);
  return make_uint4(w[0], w[1], w[2], w[3]);
}
// v[j] += code_j * scale for the 16 e4m3 codes of u (the e4m3 -> f16 conversion is exact)
__device__ __forceinline__ void e4m3x16_unpack_fma(const uint4 u, float scale, float (&v)[16]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    uint32_t h2;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"((uint16_t)(w[j >> 1] >> (16 * (j & 1)))));
    const float2 f = __half22float2(*reinterpret_cast<__half2*>(&h2));
    v[2 * j] = fmaf(f.x, scale, v[2 * j]);
    v[2 * j + 1] = fmaf(f.y, scale, v[2 * j + 1]);
  }
}

#ifdef __CUDACC__
// ----------------------------------------------------------------------------------
// PTX wrappers
// ----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .b32 %%rx;\n"
      ".reg .pred %%px;\n"
      "     elect.sync %%rx|%%px, %1;\n"
      "@%%px mov.s32 %0, 1;\n"
      "}\n"
      : "+r"(pred)
      : "r"(0xffffffffu));
  return pred != 0;
}

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
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
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must trap (kernel fault) instead of hanging the GPU.  (No printf here: a function call
// inside a wgmma main loop makes ptxas serialise every wgmma of the kernel.)
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}

// ---- TMA ----
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// im2col mode, NHWC tensor seen as {C, W, H, N}; (w,h) = base pixel, (ow,oh) = filter-tap offsets
__device__ __forceinline__ void tma_load_im2col_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c, int w,
                                                   int h, int n, uint16_t ow, uint16_t oh) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h),
      "r"(n), "h"(ow), "h"(oh)
      : "memory");
}

// TMA store: a [box] tile of (swizzled) shared memory -> global, rows/cols past the tensor bounds are clipped.
// Bulk-group completion: commit, then wait_group(.read) before the shared-memory tile is reused / the CTA exits.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() {   // at most N most-recent groups still READING shared memory
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_group() {        // at most N most-recent groups not yet complete
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---- stmatrix / ldmatrix: four 8x8 matrices of 16-bit elements between registers and shared memory ----
// Lane l gives the address of row l & 7 (16 bytes) of matrix l >> 3; register i of lane l holds row l >> 2, columns
// 2 (l & 3) and + 1 of matrix i, which is the layout of a wgmma accumulator fragment packed to 16 bits.
__device__ __forceinline__ void stmatrix_x4(uint32_t saddr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(r0), "r"(r1), "r"(r2),
               "r"(r3)
               : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t saddr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(saddr)
               : "memory");
}

// ---- clusters: TMA multicast, cluster-wide barrier, remote mbarrier arrive ----
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {   // every thread of every CTA of the cluster
  __syncwarp();
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// Arrive on the barrier at the same shared-memory offset in CTA `cta` of the cluster, with the default .release.cta
// semantics.  The consumers' stage release only has to follow their own wgmma reads (already retired by
// wgmma.wait_group); a .cluster-scope release compiles to MEMBAR.ALL.GPU + ERRBAR per arrive, which in the conv main
// loop stalls every k-block (DESIGN.md §5).
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n"
      ".reg .b32 ra;\n"
      "mapa.shared::cluster.u32 ra, %0, %1;\n"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(cta)
      : "memory");
}
// the box lands at the same shared-memory offset in every CTA of `mask`; each destination's bytes are credited to the
// barrier at the same offset in that CTA
__device__ __forceinline__ void tma_load_2d_multicast(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                      uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5}], [%2], %3;"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "h"(mask), "r"(c0), "r"(c1)
      : "memory");
}
// im2col-mode load (tma_load_im2col_4d) multicast like tma_load_2d_multicast
__device__ __forceinline__ void tma_load_im2col_4d_multicast(void* dst, const CUtensorMap* m, uint64_t* bar, int c, int w,
                                                             int h, int n, uint16_t ow, uint16_t oh, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5, %6, %7}], [%2], {%8, %9}, %3;"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "h"(mask), "r"(c), "r"(w), "r"(h),
      "r"(n), "h"(ow), "h"(oh)
      : "memory");
}

// ---- wgmma (warpgroup MMA, operands in shared memory, fp32 accumulators in registers) ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {   // at most N most-recent wgmma groups of this thread still pending
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across a wgmma fence or wait
template <int K>
__device__ __forceinline__ void wgmma_fence_operand(float (&d)[K]) {
#pragma unroll
  for (int i = 0; i < K; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// named barrier over the 128 threads of one warpgroup (ids 1.. : 0 is __syncthreads)
__device__ __forceinline__ void warpgroup_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
// named barrier over `n` threads: wait (sync) / signal without waiting (arrive)
__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }


// wgmma shared-memory matrix descriptor (PTX ISA "matrix descriptor format"): [0,14) addr>>4, [16,30) LBO>>4,
// [32,46) SBO>>4, [62,64) layout (1 = 128B, 2 = 64B swizzle).  The swizzle is a function of the shared-memory address
// bits, so a descriptor may start at any 16-byte-aligned row of a tile the TMA wrote with the same swizzle.
// K-major tiles whose rows are one swizzle span wide: SBO = bytes between 8-row groups (LBO unused).
// MN-major tiles: LBO = bytes between 64 / 32-element MN blocks, SBO = bytes between 8-row K groups.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t swizzle_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)(swizzle_bytes == 128 ? 1 : 2) << 62;
  return d;
}
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t saddr, uint32_t sbo_bytes, uint32_t swizzle_bytes) {
  return make_smem_desc(saddr, 16, sbo_bytes, swizzle_bytes);
}
#endif  // __CUDACC__

}  // namespace yb

// Shared device/host helpers for the dwm_b200 sm_90a kernels.
//
// Everything here is raw PTX for Hopper (wgmma / TMA / mbarrier).
// No CUTLASS/CuTe is included; the bit layout of the wgmma shared-memory
// descriptor follows the PTX ISA tables.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <stdint.h>
#include <stdio.h>

namespace dwm {

// ---------------------------------------------------------------------------
// error plumbing (host)
// ---------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);

#define DWM_CHECK_CUDA(expr)                                                   \
  do {                                                                         \
    cudaError_t _e = (expr);                                                   \
    if (_e != cudaSuccess) {                                                   \
      ::dwm::set_last_error("%s failed: %s (%s:%d)", #expr,                    \
                            cudaGetErrorString(_e), __FILE__, __LINE__);       \
      return -2;                                                               \
    }                                                                          \
  } while (0)

#define DWM_REQUIRE(cond, ...)                                                 \
  do {                                                                         \
    if (!(cond)) {                                                             \
      ::dwm::set_last_error(__VA_ARGS__);                                      \
      return -1;                                                               \
    }                                                                          \
  } while (0)

// Encodes a 2-D row-major tensor map (inner dim contiguous), 128B swizzle.
// rows x cols elements of `elem_bytes`; row pitch `ld` elements.
int make_tmap_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols,
                 uint64_t ld, uint32_t box_rows, uint32_t box_cols, int elem_bytes);

// The same for items x rows x cols with item pitch `item_ld` elements; a box is one item deep.
int make_tmap_3d(CUtensorMap* map, const void* base, uint64_t items, uint64_t rows, uint64_t cols,
                 uint64_t ld, uint64_t item_ld, uint32_t box_rows, uint32_t box_cols, int elem_bytes);

int make_tmap_nd(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_bytes, const uint32_t* box, int elem_bytes);

int sm_count();

// true if p (which may be null) is a multiple of `bytes`, a power of two
inline bool is_aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

#ifdef __CUDACC__
// ---------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------
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

// ---- mbarrier -------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
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
// Spin on a phase parity.  With -DDWM_BOUNDED_WAIT the spin traps after a
// very large number of polls so a pipeline bug surfaces as a CUDA error
// instead of a hung GPU box.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#ifdef DWM_BOUNDED_WAIT
  for (uint32_t it = 0; it < (1u << 26); ++it) {
    if (mbar_try_wait(bar, parity)) return;
  }
  printf("dwm_b200: mbarrier wait timed out (block %d thread %d)\n", blockIdx.x, threadIdx.x);
  __trap();
#else
  while (!mbar_try_wait(bar, parity)) {
  }
#endif
}

// ---- TMA ------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tile load global -> shared, completion on an mbarrier (tx bytes).
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* smem,
                                            int32_t c0, int32_t c1, uint64_t cache_hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      :
      : "r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
        "r"(c1), "l"(cache_hint)
      : "memory");
}
// L2 eviction-priority descriptors (createpolicy encodings, as used by CUTLASS).
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;
// L2 prefetch of a tensor-map box (no shared-memory destination, no completion tracking).
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* m, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_prefetch_5d(const CUtensorMap* m, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.prefetch.tensor.5d.L2.global.tile [%0, {%1, %2, %3, %4, %5}];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
// 5-D box load (implicit-GEMM convolution taps; gathered attention sequences).
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* m, uint64_t* bar, void* smem, int c0,
                                            int c1, int c2, int c3, int c4, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2], %8;"
      :
      : "r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "r"(c2), "r"(c3), "r"(c4), "l"(hint)
      : "memory");
}

// 3-D box store shared -> global, tracked by this thread's bulk async-groups; the parts of the
// box outside the tensor map are not written.
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* smem, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the shared-memory sources of all committed bulk stores of this thread have been read
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// all committed bulk stores of this thread are complete
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// named barrier over `n` threads (barrier 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int n) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}
// four 8x8 16-bit matrices to shared memory: lanes 8i..8i+7 give the row addresses of matrix i,
// register i of lane l holds row l/4, columns 2(l%4), 2(l%4)+1 of matrix i (the mma fragment)
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1),
               "r"(r2), "r"(r3)
               : "memory");
}

// ---- clusters of two CTAs ----------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_u32(uint32_t smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
  return r;
}
// Arrive on an mbarrier of another CTA of the cluster, without cluster-scope release semantics.
// The only use is a consumer telling the peer's producer that this CTA has finished READING a
// stage, so the peer's next multicast may overwrite it.  Those reads were made by wgmma and are
// complete once wgmma.wait_group returns; no write of this thread has to become visible to the
// peer.  ".release.cluster" would make ptxas put MEMBAR.ALL.GPU in front of the arrive, which
// waits for every earlier store of the warp (the previous tile's epilogue) inside the k-loop.
// The plain form (default .release.cta) is a bare SYNCS.ARRIVE.TRANS64.RED.
__device__ __forceinline__ void mbar_arrive_remote(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
// 2-D tile load written to the same shared-memory offset of every CTA in `mask`; each
// destination's mbarrier at the offset of `bar` receives the transaction bytes
__device__ __forceinline__ void tma_load_2d_mc(const CUtensorMap* m, uint64_t* bar, void* smem, int32_t c0,
                                               int32_t c1, uint16_t mask, uint64_t cache_hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      ".L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5, %6;"
      :
      : "r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "h"(mask), "l"(cache_hint)
      : "memory");
}

// ---- wgmma (Hopper warpgroup MMA) -----------------------------------------------
// Shared-memory matrix descriptor for a K-major operand tile written by TMA with 128-byte
// swizzle: rows are 128 B apart, 8-row groups 1024 B apart.
//   [0,14)  start address >> 4        [16,30) leading byte offset >> 4 (unused for SW128 K-major)
//   [32,46) stride byte offset >> 4   [49,52) base offset (0: tiles are 1024-byte aligned)
//   [62,64) layout type (1 = SWIZZLE_128B)
// Advancing 16 elements (32 B) along K inside the swizzle atom adds 2 to the start field.
// The 128-byte swizzle phase follows the absolute shared-memory address bits [7:9], exactly as
// TMA wrote the tile, so a row-shifted view (start k x 128 B past a 1024-byte boundary) needs
// no base offset: the field stays 0.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// Orders register accesses of the accumulators before the next wgmma of this warpgroup.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving accumulator reads / writes across wgmma_fence / wgmma_wait.
template <int N>
__device__ __forceinline__ void fence_operands(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Register re-partition between warpgroups (whole warpgroup executes).
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// ---- numerics ---------------------------------------------------------------
__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
// tanh-GELU in its sigmoid form: 0.5*x*(1+tanh(u)) == x * sigmoid(2u); one ex2 + one
// rcp on the SFU instead of the ~30-instruction precise tanhf (which made the FF1
// epilogue, 256 activations per thread per tile, slower than the tile's MMAs).
__device__ __forceinline__ float gelu_tanh(float x) {
  const float k2 = 2.0f * 0.7978845608028654f;
  const float u2 = k2 * (x + 0.044715f * x * x * x);
  return __fdividef(x, 1.0f + __expf(-u2));
}
__device__ __forceinline__ float silu(float x) { return x / (1.0f + __expf(-x)); }

template <typename T>
struct Cvt;
template <>
struct Cvt<__nv_bfloat16> {
  __device__ static __forceinline__ uint32_t pack2(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  }
  __device__ static __forceinline__ float2 unpack2(uint32_t u) {
    __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
    return __bfloat1622float2(v);
  }
  __device__ static __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  __device__ static __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};
template <>
struct Cvt<__half> {
  __device__ static __forceinline__ uint32_t pack2(float a, float b) {
    __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  }
  __device__ static __forceinline__ float2 unpack2(uint32_t u) {
    __half2 v = *reinterpret_cast<__half2*>(&u);
    return __half22float2(v);
  }
  __device__ static __forceinline__ float to_f(__half v) { return __half2float(v); }
  __device__ static __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- E4M3 row quantization ------------------------------------------------------
// One recipe everywhere (GEMM operands and weights): amax == 0 -> scale 1, q = 0; otherwise
// inv = 448 / amax, q = cvt.rn.satfinite.e4m3(x * inv), scale = amax / 448, IEEE divisions.
constexpr float kE4M3Max = 448.f;
__device__ __forceinline__ float e4m3_inv(float amax) { return amax > 0.f ? __fdiv_rn(kE4M3Max, amax) : 0.f; }
__device__ __forceinline__ float e4m3_scale(float amax) { return amax > 0.f ? __fdiv_rn(amax, kE4M3Max) : 1.f; }
// four values * inv -> four E4M3 bytes, the first in the lowest byte
__device__ __forceinline__ uint32_t e4m3x4(float a, float b, float c, float d, float inv) {
  uint16_t lo, hi;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(__fmul_rn(b, inv)), "f"(__fmul_rn(a, inv)));
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(__fmul_rn(d, inv)), "f"(__fmul_rn(c, inv)));
  return static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
}
#endif  // __CUDACC__

}  // namespace dwm

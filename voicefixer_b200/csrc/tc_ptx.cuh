// PTX wrappers of the Hopper tensor-core path (conv_gemm_tc.cu, resstack_pair.cu): TMA tile loads and stores, cp.async operand
// staging with zero fill, the generic -> async proxy fence, mbarriers, named barriers, setmaxnreg, wgmma fences / groups,
// ldmatrix and the shared-memory matrix descriptor; on the host, the SM count and the tensor-map encoder their launches use.
#pragma once
#include <atomic>
#include <cuda.h>      // CUtensorMap and the types of its encoder; the encoder itself is looked up at run time
#include "vfx_common.cuh"

namespace vfx {
namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// 16-byte global -> shared copy; ok == false writes 16 zero bytes (convolution padding, K / N tails)
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool ok) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// wgmma reads shared memory through the async proxy: make this thread's (generic-proxy) cp.async data visible to it
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// mbarrier stage hand-off (arrive: release, try_wait: acquire, both at CTA scope)
__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done)
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(bar), "r"(parity) : "memory");
}
// TMA operand staging: one thread arms the stage's full barrier with the bytes to come, then issues the tile loads.  Each
// load writes its whole box (elements outside the tensor as zeros) through the async proxy, in the swizzle of the tensor
// map, and completes that many bytes on the barrier; wgmma reads through the same proxy, so no fence lies between them.
// `map` is the address of a CUtensorMap in a __grid_constant__ kernel parameter; coordinates are innermost first.
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
               ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
// TMA tile store: one thread writes a box of shared memory (in the map's swizzle) to the tensor, clipping whatever lies
// outside it.  The writers of the box fence_proxy_async() and synchronise before it is issued; the stores of one
// commit_group form a bulk group, and wait_read<N> returns once all but the newest N groups have read shared memory.
__device__ __forceinline__ void tma_store_4d(const void* map, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// named barriers over a subset of the CTA's warps (id 0 is __syncthreads)
__device__ __forceinline__ void named_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ bool named_sync_or(int id, int nthreads, bool v) {
  uint32_t r;
  asm volatile("{\n\t.reg .pred p, q;\n\tsetp.ne.u32 p, %1, 0;\n\tbar.red.or.pred q, %2, %3, p;\n\tselp.u32 %0, 1, 0, q;\n\t}"
               : "=r"(r) : "r"((uint32_t)v), "r"(id), "r"(nthreads) : "memory");
  return r != 0;
}
// per-warpgroup register budget of a warp-specialised kernel
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// register dependence on a wgmma accumulator: the compiler may not move its reads or writes across this point
template <int N> __device__ __forceinline__ void wgmma_fence_operand(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
// ... and on a register A fragment, which the tensor core reads until its group has retired
template <int N> __device__ __forceinline__ void wgmma_fence_operand(uint32_t (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(r[i])::"memory");
}
// four 8 x 8 b16 matrices from shared memory: lanes 8i ... 8i + 7 give the addresses of matrix i's rows (16 bytes each),
// and lane l receives bytes 4 (l % 4) ... + 3 of row l / 4 of matrix i in r[i]
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}

// K-major operand tile with 128-byte rows in the 128-byte swizzle (16-byte chunk c of row r stored at chunk c ^ (r & 7)),
// 1024-byte aligned.  Descriptor: [0,14) start >> 4, [16,30) leading offset >> 4 (unused for this layout: 1),
// [32,46) stride between 8-row groups >> 4 (1024 B), [62,64) layout = 1 (128-byte swizzle).  Adding k >> 4 to the
// descriptor selects the K slice starting k bytes into each row (the swizzle is applied on absolute address bits).
__device__ __forceinline__ uint64_t sw128_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ uint32_t sw128_offset(int row, int chunk) { return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4)); }

// ---- host: what a persistent launch sizes its grid by, and the encoder of its tensor maps
inline int sm_count(int dev) {
  static std::atomic<int> sms[64];                    // per device, queried once (host threads may drive several devices)
  if (dev < 64) {
    const int n = sms[dev].load(std::memory_order_relaxed);
    if (n) return n;
  }
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 0;
  if (dev < 64) sms[dev].store(n, std::memory_order_relaxed);
  return n;
}

// cuTensorMapEncodeTiled, through the runtime (the library calls nothing else of the driver API)
using EncodeTiled = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                 const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiled tensor_map_encoder() {
  static const EncodeTiled fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &p, 12000, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiled>(p);
  }();
  return fn;
}

}  // namespace
}  // namespace vfx

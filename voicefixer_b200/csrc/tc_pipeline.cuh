// The pipeline of the persistent, warp-specialised wgmma kernels (conv_gemm_tc.cu, resstack_pair.cu): their launch
// shape, the ring of operand stages and its hand-off, the consumers' K loop, and the host side of their launches.
//
// A CTA has three warpgroups.  Warpgroup 0 produces: for every K slice (128 bytes of K) it brings a 128-row A tile and
// the slice's weight rows into the next stage of a ring of 128-byte-swizzled K-major tiles.  Warpgroups 1 and 2 consume,
// 64 rows each (k_loop).  Slice k of a CTA's sequence goes into stage k % STAGES, and two mbarriers per stage hand it
// over: `full` once the slice has landed, `empty` once every consumer warp's wgmma group has read it.  The producer feeds
// the ring in one of two ways:
//  - TMA: one thread arms the stage's full barrier with the bytes to come (mbar_expect_tx) and issues the tensor-map
//    loads, which complete the barrier themselves.
//  - cp.async: every thread of the warpgroup stages 16-byte chunks, then (Ring::cp_async_handoff) waits for its own
//    copies of an earlier slice, fences them against the tensor core's async-proxy reads and arrives on that slice's
//    full barrier.
// The ring is filled for the next tile while the consumers run the epilogue of this one.
#pragma once
#include "tc_ptx.cuh"
#include "wgmma_ptx.cuh"

namespace vfx {
namespace {

// operand kind (0 tf32, 1 bf16, 2 fp16) -> element type and size
template <int KIND> struct OpT;
template <> struct OpT<0> { using T = tf32_t; static constexpr int ESZ = 4; };
template <> struct OpT<1> { using T = __nv_bfloat16; static constexpr int ESZ = 2; };
template <> struct OpT<2> { using T = __half; static constexpr int ESZ = 2; };

constexpr int BM = 128, NT = 384;                  // rows of an A tile; warpgroup 0 produces, warpgroups 1 and 2 consume
constexpr int A_BYTES = BM * 128;                  // one A tile of a stage; the weight rows follow it
constexpr int SMEM_MAX = 227 * 1024;               // dynamic shared memory of one sm_90 CTA
constexpr int PROD_REGS = 56, CONS_REGS = 224;     // 128 x 56 + 256 x 224 <= 384 x 168 (the launch allocation)

// The ring of a kernel whose stages take STAGE bytes each and whose own shared memory takes FIXED bytes.  Shared memory:
// up to 1024 bytes to align the ring, the STAGES stages, the kernel's FIXED bytes, then the full and the empty mbarriers.
// As many stages as fit, at most 8; fewer than MIN does not compile.
template <int STAGE_, int FIXED_, int MIN> struct RingPlan {
  static constexpr int STAGE = STAGE_, FIXED = FIXED_;
  static constexpr int FIT = (SMEM_MAX - 1024 - FIXED) / (STAGE + 16);
  static constexpr int STAGES = FIT < 8 ? FIT : 8;
  // cp.async: the producer signals slice k full after issuing slice k + AHEAD (cp.async.wait_group AHEAD).  It must wait
  // for an empty slot before issuing, and the consumers free slot k - 1 only once slice k is full, so AHEAD <= STAGES - 2:
  // with more, the producer waits for a slot the consumers can only free after a signal it has not sent yet.
  // TMA has no such rule: a slice's full barrier is completed by its loads, whatever the issuing thread does next, so
  // that thread may block on the empty barrier of the oldest stage with every other stage in flight.
  static constexpr int AHEAD = STAGES - 2;
  static constexpr int SMEM = 1024 + FIXED + STAGES * (STAGE + 16);
  static_assert(STAGES >= MIN && SMEM <= SMEM_MAX, "tc_pipeline: shared-memory plan");
};

// The ring of plan P in shared memory, stage 0 at the 1024-byte aligned `base`; the kernel's FIXED bytes start at
// base + STAGES * STAGE.  k counts the CTA's K slices.
template <class P> struct Ring {
  static constexpr int S = P::STAGES;
  uint32_t base;

  __device__ __forceinline__ uint32_t stage(uint32_t k) const { return base + k % S * P::STAGE; }
  __device__ __forceinline__ uint32_t full(uint32_t k) const { return base + S * P::STAGE + P::FIXED + 8 * (k % S); }
  __device__ __forceinline__ uint32_t empty(uint32_t k) const { return full(k) + 8 * S; }

  // one thread, before the CTA's first barrier.  full: the TMA thread's expect_tx plus the bytes of the stage's loads, or
  // every cp.async producer thread after its own copies of the stage have landed; empty: every consumer warp, after its
  // wgmma group has read the stage
  __device__ __forceinline__ void init(bool tma) const {
    for (int s = 0; s < S; ++s) {
      mbar_init(full(s), tma ? 1 : 128);
      mbar_init(empty(s), 8);
    }
  }
  // producer: wait until slice k's stage has been read by the consumers of slice k - S
  __device__ __forceinline__ void acquire(uint32_t k) const {
    if (k >= (uint32_t)S) mbar_wait(empty(k), ((k / S) & 1) ^ 1);
  }
  // cp.async producer thread, after issuing its copies of slice k: they form one group, and slice k - AHEAD is signalled
  __device__ __forceinline__ void cp_async_handoff(uint32_t k) const {
    cp_async_commit();
    if (k >= (uint32_t)P::AHEAD) {
      cp_async_wait<P::AHEAD>();                  // this thread's chunks of slice k - AHEAD have landed
      fence_proxy_async();                        // ... and are visible to the tensor core's (async-proxy) reads
      mbar_arrive(full(k - P::AHEAD));
    }
  }
  // cp.async producer thread, after its last slice (k slices issued in all): signal the slices still outstanding
  __device__ __forceinline__ void cp_async_drain(uint32_t k) const {
    cp_async_wait<0>();
    fence_proxy_async();
    for (uint32_t j = k > (uint32_t)P::AHEAD ? k - P::AHEAD : 0; j < k; ++j) mbar_arrive(full(j));
  }
  // consumer: wait for slice k; and, once the wgmma group of this warp has read it, hand its stage back (lane l)
  __device__ __forceinline__ void wait_full(uint32_t k) const { mbar_wait(full(k), (k / S) & 1); }
  __device__ __forceinline__ void release(uint32_t k, int l) const {
    __syncwarp();
    if (l == 0) mbar_arrive(empty(k));
  }
};

// The consumers' K loop of one tile, for consumer warpgroup cw: acc = the sum of the tile's niter K slices, which the
// feed f describes.  Slice it is 4 m64nBN wgmma (32 bytes of K each) into a zeroed partial: the tensor core's accumulator
// adds truncate, so the partials are added to acc in slice order with round-to-nearest fp32 adds, and the error of long
// reductions (9 taps x 768 channels) does not build up as a bias.  One group is in flight: slice it goes into partial
// it & 1 while slice it - 1 is added.
// The feed: wait(it) before slice it is read; b(it), the address of its BN weight rows (K-major, 128-byte swizzle);
// its A operand, either (REG_A false) a(it), the address of its 128-row A tile, of which warpgroup cw reads rows
// cw * 64 on by descriptor, or (REG_A true) a_frag(it, fr), which loads this warp's 16 x (32 bytes of K) register
// fragment of each of the 4 wgmma; release(it) once slice it's wgmma group has retired, before its partial is added.
// The register fragments of the group in flight are not overwritten before its wgmma_wait: two sets alternate.
// niter is a runtime value on purpose: with a compile-time count, ptxas peels the loop and serialises its wgmma groups
// (C7514), and a fully unrolled loop spills.
template <int BN, int KIND, class Feed>
__device__ __forceinline__ void k_loop(float (&acc)[BN / 2], int niter, int cw, const Feed& f) {
  float p0[BN / 2], p1[BN / 2];
  uint32_t f0[4][4], f1[4][4];                    // register A fragments (Feed::REG_A only)
  auto issue = [&](float (&p)[BN / 2], uint32_t (&fr)[4][4], int it) {
    f.wait(it);
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) p[i] = 0.f;
    const uint64_t db = sw128_desc(f.b(it));
    if constexpr (Feed::REG_A) {
      f.a_frag(it, fr);
      wgmma_fence();
#pragma unroll
      for (int q = 0; q < 4; ++q) Wgmma<BN, KIND>::mma(p, fr[q], db + 2 * q);
    } else {
      const uint64_t da = sw128_desc(f.a(it) + cw * 64 * 128);
      wgmma_fence();
#pragma unroll
      for (int q = 0; q < 4; ++q) Wgmma<BN, KIND>::mma(p, da + 2 * q, db + 2 * q);
    }
    wgmma_commit();
  };
  auto retire = [&](float (&p)[BN / 2], uint32_t (&fr)[4][4], int it) {
    wgmma_fence_operand(p);                       // the reads of p below stay after the wgmma_wait that precedes
    if constexpr (Feed::REG_A) {
#pragma unroll
      for (int q = 0; q < 4; ++q) wgmma_fence_operand(fr[q]);   // fr stays allocated until its group has retired
    }
    f.release(it);
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] += p[i];
    wgmma_fence_operand(acc);                     // the adds stay here, before the next slice is issued: p is reused
  };
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  issue(p0, f0, 0);
  int it = 1;
#pragma unroll 1
  for (; it + 1 < niter; it += 2) {
    issue(p1, f1, it);
    wgmma_wait<1>();
    retire(p0, f0, it - 1);
    issue(p0, f0, it + 1);
    wgmma_wait<1>();
    retire(p1, f1, it);
  }
  if (it < niter) {
    issue(p1, f1, it);
    wgmma_wait<1>();
    retire(p0, f0, it - 1);
    wgmma_wait<0>();
    retire(p1, f1, it);
  } else {
    wgmma_wait<0>();
    retire(p0, f0, it - 1);
  }
}

// The feed of K slices k0, k0 + 1, ... of a ring: slice it's A tile is a_tile(it, stage address), its weight rows
// b_tile(it, stage address); its stage is handed back by lane l's warp once read, then released(it) runs.
template <class P, class ATile, class BTile, class Released> struct RingFeed {
  static constexpr bool REG_A = false;
  const Ring<P>& ring;
  uint32_t k0;
  int l;
  ATile a_tile;
  BTile b_tile;
  Released released;
  __device__ __forceinline__ void wait(int it) const { ring.wait_full(k0 + it); }
  __device__ __forceinline__ uint32_t a(int it) const { return a_tile(it, ring.stage(k0 + it)); }
  __device__ __forceinline__ uint32_t b(int it) const { return b_tile(it, ring.stage(k0 + it)); }
  __device__ __forceinline__ void release(int it) const {
    ring.release(k0 + it, l);
    released(it);
  }
};
template <class P, class ATile, class BTile, class Released>
__device__ __forceinline__ RingFeed<P, ATile, BTile, Released> ring_feed(const Ring<P>& ring, uint32_t k0, int l,
                                                                         ATile a_tile, BTile b_tile, Released released) {
  return {ring, k0, l, a_tile, b_tile, released};
}
// the weight rows of a stage that carries them: they follow its A tile
struct StageB {
  __device__ __forceinline__ uint32_t operator()(int, uint32_t sa) const { return sa + A_BYTES; }
};

// ---- host

// the tensor-map element type of an operand precision
inline CUtensorMapDataType map_dtype(int precision) {
  return precision == VFX_PREC_TF32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
         : precision == VFX_PREC_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                      : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
}

// Launches KERNEL persistently over `tiles` tiles: grid = min(tiles, SMs), NT threads, smem bytes of dynamic shared
// memory.  The kernel's shared-memory limit is raised once per device; the bit mask is a static of this instantiation,
// so each kernel has its own.  `who` names the kernel in errors.
template <auto KERNEL, class... Args>
int launch_persistent(const char* who, int smem, long long tiles, cudaStream_t st, const Args&... args) {
  static unsigned long long attr_set = 0;      // devices on which KERNEL's shared-memory limit has been raised
  int dev = 0;
  VFX_CUDA_CHECK(cudaGetDevice(&dev));
  if (dev >= 64 || !(attr_set >> dev & 1)) {
    VFX_CUDA_CHECK(cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    if (dev < 64) attr_set |= 1ull << dev;
  }
  const int sms = sm_count(dev);
  VFX_REQUIRE(sms > 0, "%s: cannot read the SM count of device %d", who, dev);
  const int grid = (int)(tiles < sms ? tiles : sms);
  if (tiles + grid >= (1LL << 31)) return VFX_ERR_UNSUPPORTED;      // the tile walk t += gridDim.x stays inside int
  KERNEL<<<grid, NT, smem, st>>>(args...);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

}  // namespace
}  // namespace vfx

// ResStack pair x' = x + conv2_{k3,d=1}(lrelu_0.01(conv1_{k3,dilation}(a) + b1)) + b2 (include/vfx_b200.h,
// vfx_resstack_pair), ResStack.forward voicefixer/vocoder/model/modules.py:592-595.
//
// Fused form (VFX_PAIR_FUSED; the engine's fused pairs): a persistent, warp-specialised kernel on the pipeline of
// tc_pipeline.cuh (ring, feed and K loop).  grid = min(tiles, SMs); a tile is 126 output rows of one item, and each CTA
// walks a static stride over the (item, row block) tiles with the row block fastest, so that neighbouring CTAs work on
// neighbouring rows and the dilation halo comes from L2.
//  - Weights.  At C = 64 W1 and W2 are loaded once per CTA (96 KB tf32, 48 KB 16-bit) and stay resident; the ring
//    carries A tiles only.  At C = 128 (192 KB in 16-bit) they stream through the ring beside each A tile.
//  - Producer: per tile, conv1's 3 x NKS K slices (the 128 a rows [r0 - 1, r0 + 127) shifted by the tap, and at C = 128
//    the tap's W1 rows), then at C = 128 conv2's 3 x NKS slices (W2 rows only).  It runs ahead into the next tile's
//    conv1 while the consumers finish conv2 and the epilogue of this one.  Two forms:
//      TMA (launches without lens): a box of the (C, L, B) operand map at row r0 - 1 + (tap - 1) * dilation and a box of
//      the [3][C][C] weight map per weight slice; the out-of-bounds fill is conv1's zero padding.
//      cp.async (ragged batches): zero fill beyond the item's own length.
//  - Consumers: conv1's K loop; its epilogue writes lrelu(h + b1) in the operand format into shared memory (rows outside
//    [0, L) are zero: conv2's padding), and conv2's tap t reads h shifted by t rows.  At C = 64 h is one buffer of 130
//    rows, written once, and conv2 takes A from registers: per 32 bytes of K each warp loads its 16-row fragment with one
//    ldmatrix at rows + t.  At C = 128 the accumulator and two partials leave no registers for fragments, so h is
//    written three times, copy t shifted up by t rows, and conv2's tap t reads copy t by descriptor.  A named barrier
//    keeps the next tile's h writes behind this tile's last conv2 read.  conv2's epilogue adds b2 and the residual and
//    writes x' / act(x').
//  - Nothing global in the epilogues' critical path: b1 and b2 are staged in shared memory once per CTA.  In tf32 the
//    residual (the encoded stream, a == x) is rows 1 ... 126 of conv1's centre-tap A tiles, which are kept out of the
//    ring for that, read into registers in the h epilogue and then released to the producer (one mbarrier).  In the
//    16-bit modes x is a separate fp32 tensor: at C = 64 the residual is loaded into registers before conv2's K loop,
//    at C = 128 (no registers to spare beside the accumulator and two partials) it is prefetched into L2 then and
//    loaded after the K loop.
// h never leaves the SM: HBM traffic is a (with a halo), the residual (16-bit modes) and the outputs.  Shared memory
// (PairCfg): tf32 C = 64 weights 96 KB, centre tiles 32 KB, h 32.5 KB, 4 ring stages of 16 KB; 16-bit C = 64 weights
// 48 KB, h 16.25 KB, 8 stages of 16 KB; 16-bit C = 128 h copies 96 KB, 4 stages of 16 KB of a + 16 KB of weights.
// Every sum is in the order of the blocked form: per K slice 4 wgmma into a zeroed partial, partials added in (tap,
// channel slice) order with round-to-nearest fp32 adds, then (acc + b) + residual.  Register A fragments hold the same
// operand values the descriptor form reads (h is rounded to the operand format when it is written).
//
// Blocked form (VFX_PAIR_BLOCKED, the tests' reference): two conv_gemm_tc launches per row block, h in a scratch.
#include <string.h>
#include "tc_pipeline.cuh"

namespace vfx {

namespace {
constexpr size_t PAIR_SCRATCH_BYTES = 32u << 20;

constexpr int P_ROWS = 126;                       // output rows of a tile (of the 128 rows of its A tiles)

// Shared memory beside the ring: the resident weights, the tf32 centre tiles, h, b1 / b2, and the mbarriers of the centre
// tiles and of the weights.  Everything read by descriptor or written by TMA comes first, 1024-byte aligned.
// RES (C = 64): W1 and W2 stay in shared memory for the CTA's life, the ring carries A tiles only, and h is one buffer
// of 130 rows that conv2 reads through registers.  At C = 128 the weights (192 KB in 16-bit) do not fit, and the
// accumulator and two partials take 192 of the consumers' 224 registers, leaving none for two register A fragment
// sets: the weights stream through the ring beside each A tile and h is kept as three shifted copies that conv2 reads by
// descriptor.
template <int C, int KIND> struct PairCfg {
  static constexpr int ESZ = OpT<KIND>::ESZ, NKS = C * ESZ / 128, NITER = 3 * NKS;   // K slices per convolution
  static constexpr bool RES = C == 64;
  static constexpr int WS = C * 128;                              // the weight rows of one K slice
  static constexpr int W = RES ? 2 * NITER * WS : 0;              // resident W1, W2
  static constexpr int COPIES = RES ? 1 : 3;                      // of h
  // an h slice: 128 rows read by descriptor, 1024-byte aligned for the swizzle; 130 rows read by ldmatrix, which applies
  // no swizzle of its own and needs 16-byte rows only (the 1 536 bytes this saves in tf32 make the fourth stage fit)
  static constexpr int HS = (RES ? 130 : 128) * 128;
  static constexpr int H = COPIES * NKS * HS;
  static constexpr int CTR = KIND == 0 ? NKS * 16384 : 0;         // tf32: conv1's centre-tap A tiles (the residual)
  static constexpr int PT = RES ? NITER : 2 * NITER;              // ring slices per tile
  using Plan = RingPlan<A_BYTES + (RES ? 0 : WS), W + H + CTR + 2 * C * 4 + 16, 3>;
  // 4 stages of 16 KB, 231 504 B in tf32; 8 stages, 198 544 B at 16-bit C = 64; 4 stages of 32 KB, 231 504 B at C = 128
  static_assert(Plan::SMEM == (KIND == 0 ? 231504 : C == 64 ? 198544 : 231504), "resstack_pair: shared-memory plan");
};

// What a TMA launch carries beside the descriptor: the operand (C, L, B), box (128 bytes, 128 rows, 1), and the two
// weight arrays (C, C, 3), box (128 bytes, C rows, 1)
struct PairMaps { CUtensorMap a, w1, w2; };

// element n of row j of h (K-major, 128-byte slices of HS bytes, 128-byte swizzle); also, at HS = 16 KB, the layout of
// conv1's centre-tap A tiles
template <int ESZ, int HS> __device__ __forceinline__ uint32_t h_offset(int j, int n) {
  const int kb = n * ESZ;
  return (uint32_t)((kb >> 7) * HS + j * 128 + ((((kb & 127) >> 4) ^ (j & 7)) << 4) + (kb & 15));
}

// conv2's K slices at RES: A from the h buffer through registers, tap t at h rows shifted by t, and W2 resident.  Lane l
// of warp w in consumer warpgroup cw gives ldmatrix the address of A row cw * 64 + 16 w + l % 8 + 8 (l / 8 % 2), 16-byte
// chunk l / 16 of each 32 bytes of K.  The 128-byte swizzle keeps the eight rows of each ldmatrix phase on distinct
// banks at every shift.
template <int C, int KIND> struct HFeed {
  using G = PairCfg<C, KIND>;
  static constexpr bool REG_A = true;
  uint32_t hbase, w2;
  int row, hi;
  __device__ __forceinline__ void wait(int) const {}
  __device__ __forceinline__ void release(int) const {}
  __device__ __forceinline__ uint32_t b(int it) const { return w2 + (uint32_t)it * G::WS; }
  __device__ __forceinline__ void a_frag(int it, uint32_t (&fr)[4][4]) const {
    const int tap = it / G::NKS, ks = it - tap * G::NKS, j = row + tap;
    const uint32_t base = hbase + (uint32_t)(ks * G::HS + j * 128);
#pragma unroll
    for (int q = 0; q < 4; ++q) ldmatrix_x4(fr[q], base + (uint32_t)(((2 * q + hi) ^ (j & 7)) << 4));
  }
};

// tile t -> item b, its first output row r0 and the item's length L; false where the tile holds no row of its item (a
// ragged batch's rows at or beyond lens[b]).  The producer and the consumers skip tiles by this function alone.
__device__ __forceinline__ bool pair_tile(const vfx_pair_desc& d, int nrb, int t, int& b, int& r0, int& L) {
  b = t / nrb;
  r0 = (t - b * nrb) * P_ROWS;
  L = d.lens ? d.lens[b] : d.L;
  return r0 < L;
}

template <int C, int KIND, bool TMA>
__global__ void __launch_bounds__(NT, 1) pair_fused_kernel(const __grid_constant__ vfx_pair_desc d,
                                                             const __grid_constant__ PairMaps m, const int niter) {
  using T = typename OpT<KIND>::T;
  using G = PairCfg<C, KIND>;
  constexpr int ESZ = G::ESZ, AL = 16 / ESZ, BK = 128 / ESZ, NKS = G::NKS, NITER = G::NITER;
  constexpr int S = G::Plan::STAGES, STAGE = G::Plan::STAGE;
  constexpr bool EARLY = KIND != 0 && C == 64;    // 16-bit C = 64: the residual goes to registers before conv2
  extern __shared__ uint8_t smem_raw[];
  const Ring<typename G::Plan> ring{(smem_u32(smem_raw) + 1023u) & ~1023u};
  uint8_t* const gbase = smem_raw + (ring.base - smem_u32(smem_raw));
  const uint32_t wbase = ring.base + S * STAGE, cbase = wbase + G::W, hbase = cbase + G::CTR;
  const uint32_t cempty = hbase + G::H + 2 * C * 4, wfull = cempty + 8;
  const uint8_t* const cgen = gbase + S * STAGE + G::W;
  uint8_t* const hgen = gbase + S * STAGE + G::W + G::CTR;
  float* const bias = reinterpret_cast<float*>(hgen + G::H);                   // b1[C], b2[C]

  const int tid = threadIdx.x;
  if (tid == 0) {
    ring.init(TMA);
    mbar_init(cempty, 8);                           // every consumer warp, after it has read its residual rows
    if (G::RES) mbar_init(wfull, TMA ? 1 : 128);    // the weights have landed
  }
  for (int i = tid; i < 2 * C; i += NT) bias[i] = i < C ? d.b1[i] : d.b2[i - C];
  // h rows 128 and 129 feed only output rows 126 and 127, which are never stored, and are never written: zero them so
  // that they hold no NaN
  if constexpr (G::RES)
    for (int i = tid; i < NKS * 64; i += NT) reinterpret_cast<uint32_t*>(hgen + i / 64 * G::HS + 128 * 128)[i % 64] = 0u;
  __syncthreads();
  // derived after each role's setmaxnreg, so that nothing stays live across it
#define VFX_PAIR_WALK const int nrb = (d.L + P_ROWS - 1) / P_ROWS, ntiles = d.B * nrb;

  if (tid < 128) {
    // ================================================================ producer
    setmaxnreg_dec<PROD_REGS>();
    VFX_PAIR_WALK
    uint32_t k = 0, u = 0;                          // K slices issued, tiles staged by this CTA
    if constexpr (TMA) {
      if (tid != 0) return;
      if constexpr (G::RES) {
        mbar_expect_tx(wfull, G::W);
        for (int s = 0; s < 2 * NITER; ++s) {
          const int tap = s % NITER / NKS, ks = s % NKS;
          tma_load_3d(wbase + s * G::WS, s < NITER ? &m.w1 : &m.w2, wfull, ks * BK, 0, tap);
        }
      }
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++u) {
        int b, r0, L;
        pair_tile(d, nrb, t, b, r0, L);
        for (int it = 0; it < G::PT; ++it, ++k) {
          ring.acquire(k);
          const bool p2 = it >= NITER;
          const int kk = p2 ? it - NITER : it, tap = kk / NKS, ks = kk - tap * NKS;
          const uint32_t sa = ring.stage(k), full = ring.full(k);
          if (!p2) {
            const bool ctr = KIND == 0 && tap == 1;
            if (ctr && ks == 0 && u > 0) mbar_wait(cempty, (u - 1) & 1);   // the last tile's residual has been read
            mbar_expect_tx(full, A_BYTES + (G::RES ? 0 : G::WS));
            tma_load_3d(ctr ? cbase + ks * 16384 : sa, &m.a, full, ks * BK, r0 - 1 + (tap - 1) * d.dilation, b);
          } else {
            mbar_expect_tx(full, G::WS);
          }
          if (!G::RES) tma_load_3d(sa + A_BYTES, p2 ? &m.w2 : &m.w1, full, ks * BK, 0, tap);
        }
      }
      return;
    }
    // this thread's staging work: chunk `chunk` of a rows lrow + 16 i and of weight rows lrow + 16 i
    const int chunk = tid & 7, lrow = tid >> 3;
    // weight rows lrow + 16 i of a K slice at W, into the slice's shared memory at dst
    const auto stage_w = [&](uint32_t dst, const char* W) {
#pragma unroll
      for (int i = 0; i < C / 16; ++i) {
        const int n = lrow + 16 * i;
        cp_async16(dst + sw128_offset(n, chunk), W + (long long)n * C * ESZ, true);
      }
    };
    if constexpr (G::RES) {
#pragma unroll 1
      for (int s = 0; s < 2 * NITER; ++s) {
        const int tap = s % NITER / NKS, ks = s % NKS;
        stage_w(wbase + s * G::WS, static_cast<const char*>(s < NITER ? d.w1 : d.w2) +
                                       ((long long)tap * C * C + ks * BK + chunk * AL) * ESZ);
      }
      cp_async_commit();
      cp_async_wait<0>();
      fence_proxy_async();
      mbar_arrive(wfull);
    }
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
      int b, r0, L;
      if (!pair_tile(d, nrb, t, b, r0, L)) continue;
      const char* A = static_cast<const char*>(d.a) + (long long)b * d.L * C * ESZ;
      for (int it = 0; it < G::PT; ++it, ++k) {
        ring.acquire(k);
        const bool p2 = it >= NITER;
        const int kk = p2 ? it - NITER : it, tap = kk / NKS, ks = kk - tap * NKS, c = ks * BK + chunk * AL;
        const uint32_t sa = ring.stage(k);
        if (!p2) {
          const bool ctr = KIND == 0 && tap == 1;
          if (ctr && ks == 0 && u > 0) mbar_wait(cempty, (u - 1) & 1);
          const uint32_t dst = ctr ? cbase + ks * 16384 : sa;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int r = lrow + 16 * i, g = r0 - 1 + r + (tap - 1) * d.dilation;
            const bool ok = g >= 0 && g < L;
            cp_async16(dst + sw128_offset(r, chunk), ok ? A + ((long long)g * C + c) * ESZ : A, ok);
          }
        }
        if (!G::RES) stage_w(sa + A_BYTES, static_cast<const char*>(p2 ? d.w2 : d.w1) + ((long long)tap * C * C + c) * ESZ);
        ring.cp_async_handoff(k);
      }
      ++u;
    }
    ring.cp_async_drain(k);
    return;
  }

  // ================================================================== consumers
  setmaxnreg_inc<CONS_REGS>();
  VFX_PAIR_WALK
#undef VFX_PAIR_WALK
  const int ct = tid - 128, cw = ct >> 7, w = (ct >> 5) & 3, l = tid & 31;
  float* const dst = d.x_out ? d.x_out : d.x;
  T* const out_act = reinterpret_cast<T*>(d.out_act);
  const float* const b1 = bias;
  const float* const b2 = bias + C;
  float acc[C / 2], xr[C / 2];
  // the A tile of K slice it (of the niter = NITER slices, a kernel argument: see k_loop): conv1's come from the ring,
  // except in tf32 the centre tap's, which are the centre tiles; at C = 128 conv2's are the h copies.  The weight rows
  // are resident (RES) or follow the stage's A tile.
  const auto conv1_a = [=](int it, uint32_t sa) {
    return KIND == 0 && it / NKS == 1 ? cbase + (uint32_t)(it - NKS) * 16384 : sa;
  };
  const auto conv1_b = [=](int it, uint32_t sa) { return G::RES ? wbase + (uint32_t)it * G::WS : sa + A_BYTES; };
  const auto conv2_a = [=](int it, uint32_t) { return hbase + (uint32_t)it * 16384; };
  const auto none = [](int) {};
  // accumulator element (j, h, e) of lane l in warp w of consumer warpgroup cw is row cw*64 + w*16 + l/4 + 8h,
  // column 8j + 2(l%4) + e
  const int row0 = cw * 64 + w * 16 + (l >> 2);
  if constexpr (G::RES) mbar_wait(wfull, 0);

  uint32_t k = 0;                                   // K slices consumed by this CTA
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    int b, r0, L;
    if (!pair_tile(d, nrb, t, b, r0, L)) continue;
    const long long item = (long long)b * d.L * C;
    // the 16-bit modes' residual rows of this thread (x, fp32), all loaded before any is used
    auto load_res = [&] {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = row0 + 8 * h, g = r0 + i;
        const bool live = i < P_ROWS && g < L;
        const float* xrow = d.x + item + (long long)g * C;
#pragma unroll
        for (int j = 0; j < C / 8; ++j) {
          const float2 r = live ? *reinterpret_cast<const float2*>(xrow + 8 * j + 2 * (l & 3)) : make_float2(0.f, 0.f);
          xr[4 * j + 2 * h] = r.x;
          xr[4 * j + 2 * h + 1] = r.y;
        }
      }
    };

    // ---- conv1 -> h
    k_loop<C, KIND>(acc, niter, cw, ring_feed(ring, k, l, conv1_a, conv1_b, none));
    k += NITER;
    named_sync(1, 256);                             // every consumer's conv2 of the last tile has read h
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i = row0 + 8 * h, g = r0 - 1 + i;
      const bool inside = g >= 0 && g < L;
#pragma unroll
      for (int j = 0; j < C / 8; ++j) {
        const int n = 8 * j + 2 * (l & 3);
        float v0 = acc[4 * j + 2 * h] + b1[n], v1 = acc[4 * j + 2 * h + 1] + b1[n + 1];
        v0 = inside ? (v0 > 0.f ? v0 : 0.01f * v0) : 0.f;
        v1 = inside ? (v1 > 0.f ? v1 : 0.01f * v1) : 0.f;
#pragma unroll
        for (int c = 0; c < G::COPIES; ++c) {
          const int jr = i - c;
          if (jr < 0) continue;
          uint8_t* p = hgen + c * NKS * G::HS + h_offset<ESZ, G::HS>(jr, n);
          if (ESZ == 2) {
            *reinterpret_cast<uint32_t*>(p) = pack16<KIND == 2>(v0, v1);
          } else {
            *reinterpret_cast<float2*>(p) = make_float2(round_tf32(v0), round_tf32(v1));
          }
        }
      }
    }
    if constexpr (KIND == 0) {
      // output row i is row i + 1 of the centre-tap tiles (a == x): its residual, bit for bit as it lies in x
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = row0 + 8 * h;
#pragma unroll
        for (int j = 0; j < C / 8; ++j) {
          const float2 r = i < P_ROWS ? *reinterpret_cast<const float2*>(cgen + h_offset<4, 16384>(i + 1, 8 * j + 2 * (l & 3)))
                                      : make_float2(0.f, 0.f);
          xr[4 * j + 2 * h] = r.x;
          xr[4 * j + 2 * h + 1] = r.y;
        }
      }
      __syncwarp();
      if (l == 0) mbar_arrive(cempty);
    } else if constexpr (EARLY) {
      load_res();
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = row0 + 8 * h, g = r0 + i;
        if (i < P_ROWS && g < L)
          asm volatile("prefetch.global.L2 [%0];" ::"l"(d.x + item + (long long)g * C + 32 * (l & 3)));
      }
    }
    if constexpr (!G::RES) fence_proxy_async();     // the h copies are visible to conv2's descriptor reads
    named_sync(1, 256);

    // ---- conv2 from h, residual, outputs
    if constexpr (G::RES) {
      k_loop<C, KIND>(acc, niter, cw, HFeed<C, KIND>{hbase, wbase + NITER * G::WS, cw * 64 + w * 16 + (l & 15), l >> 4});
    } else {
      k_loop<C, KIND>(acc, niter, cw, ring_feed(ring, k, l, conv2_a, StageB{}, none));
      k += NITER;
    }
    if constexpr (KIND != 0 && !EARLY) load_res();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i = row0 + 8 * h, g = r0 + i;
      if (i >= P_ROWS || g >= L) continue;
      const long long row = item + (long long)g * C;
      // the thread's two adjacent columns n, n + 1 go out as one 8-byte (raw, tf32 operand) or 4-byte (16-bit) store
#pragma unroll
      for (int j = 0; j < C / 8; ++j) {
        const int n = 8 * j + 2 * (l & 3);
        float v[2], y[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float r = xr[4 * j + 2 * h + e];
          v[e] = (acc[4 * j + 2 * h + e] + b2[n + e]) + (KIND == 0 ? stream_dec(r, 100.0f) : r);
          y[e] = apply_act(v[e], d.act, d.act_param);
          if (KIND == 0 && d.stream_enc_out) v[e] = stream_enc(v[e], 0.01f);
        }
        if (d.write_raw) *reinterpret_cast<float2*>(dst + row + n) = make_float2(v[0], v[1]);
        if (out_act) {
          if (ESZ == 4)
            *reinterpret_cast<float2*>(out_act + row + n) = make_float2(round_tf32(y[0]), round_tf32(y[1]));
          else
            *reinterpret_cast<uint32_t*>(out_act + row + n) = pack16<KIND == 2>(y[0], y[1]);
        }
      }
    }
  }
}

// the launch's tensor maps (no lens: every item spans the whole tensor)
int pair_maps(const vfx_pair_desc& d, PairMaps& m) {
  const long long esz = (long long)prec_esz(d.precision), C = d.C;
  const EncodeTiled encode = tensor_map_encoder();
  VFX_REQUIRE(encode, "resstack_pair: this CUDA driver has no cuTensorMapEncodeTiled");
  const CUtensorMapDataType dt = map_dtype(d.precision);
  const cuuint32_t bk = (cuuint32_t)(128 / esz), ones[3] = {1, 1, 1};
  const cuuint64_t adim[3] = {(cuuint64_t)C, (cuuint64_t)d.L, (cuuint64_t)d.B};
  const cuuint64_t astr[2] = {(cuuint64_t)(C * esz), (cuuint64_t)(d.L * C * esz)};
  const cuuint32_t abox[3] = {bk, 128, 1};
  const cuuint64_t wdim[3] = {(cuuint64_t)C, (cuuint64_t)C, 3};
  const cuuint64_t wstr[2] = {(cuuint64_t)(C * esz), (cuuint64_t)(C * C * esz)};
  const cuuint32_t wbox[3] = {bk, (cuuint32_t)C, 1};
  CUresult r = encode(&m.a, dt, 3, const_cast<void*>(d.a), adim, astr, abox, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  VFX_REQUIRE(r == CUDA_SUCCESS, "resstack_pair: operand tensor map refused (CUresult %d)", (int)r);
  const void* ws[2] = {d.w1, d.w2};
  CUtensorMap* wm[2] = {&m.w1, &m.w2};
  for (int i = 0; i < 2; ++i) {
    r = encode(wm[i], dt, 3, const_cast<void*>(ws[i]), wdim, wstr, wbox, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    VFX_REQUIRE(r == CUDA_SUCCESS, "resstack_pair: weight tensor map refused (CUresult %d)", (int)r);
  }
  return VFX_OK;
}

template <int C, int KIND, bool TMA>
int launch_pair(const vfx_pair_desc& d, const PairMaps& m, cudaStream_t st) {
  return launch_persistent<pair_fused_kernel<C, KIND, TMA>>("resstack_pair", PairCfg<C, KIND>::Plan::SMEM,
                                                            (long long)d.B * ceil_div(d.L, P_ROWS), st, d, m,
                                                            PairCfg<C, KIND>::NITER);
}

// launches without per-item lengths are fed by TMA, ragged ones by cp.async
template <int C, int KIND>
int launch_fused(const vfx_pair_desc& d, cudaStream_t st) {
  PairMaps m;
  memset(&m, 0, sizeof(m));
  if (d.lens) return launch_pair<C, KIND, false>(d, m, st);
  const int r = pair_maps(d, m);
  return r != VFX_OK ? r : launch_pair<C, KIND, true>(d, m, st);
}

}  // namespace

size_t resstack_pair_scratch_bytes() { return PAIR_SCRATCH_BYTES; }

static int pair_blocked(const vfx_pair_desc& d, int prec, cudaStream_t st) {
  VFX_REQUIRE(d.scratch && d.scratch_bytes >= PAIR_SCRATCH_BYTES && ((uintptr_t)d.scratch & 127) == 0,
              "resstack_pair: needs a 128-byte aligned scratch of vfx_resstack_pair_scratch_bytes() bytes");
  const int C = d.C, L = d.L;
  const long long item = (long long)L * C;
  const long long rows = (long long)(PAIR_SCRATCH_BYTES / (prec_esz(prec) * C)) / d.B - 2;   // output rows per block
  VFX_REQUIRE(rows >= 1, "resstack_pair: batch of %d does not fit the scratch", d.B);
  float* dst = d.x_out ? d.x_out : d.x;
  for (long long r0 = 0; r0 < L; r0 += rows) {
    const int nr = (int)(L - r0 < rows ? L - r0 : rows);
    const int h0 = r0 > 0 ? (int)r0 - 1 : 0;
    const int h1 = r0 + nr + 1 < L ? (int)r0 + nr + 1 : L;
    const int nh = h1 - h0;
    vfx_conv_desc c1;
    memset(&c1, 0, sizeof(c1));
    c1.a = d.a; c1.B = d.B; c1.H = 1; c1.W = L; c1.Cin = C;
    c1.a_sW = C; c1.a_sH = item; c1.a_sB = item;
    c1.w = d.w1; c1.ntaps = 3;
    for (int k = 0; k < 3; ++k) { c1.dw[k] = (k - 1) * d.dilation + h0; c1.w_off[k] = (long long)k * C * C; }
    c1.Hq = 1; c1.Wq = nh; c1.N = C; c1.sh = 1; c1.sw = 1; c1.OH = 1; c1.OW = nh;
    c1.bias = d.b1; c1.bias_mod = C;
    c1.out_act = d.scratch; c1.oa_sW = C; c1.oa_sH = (long long)nh * C; c1.oa_sB = (long long)nh * C;
    c1.act = VFX_ACT_LRELU; c1.act_param = 0.01f;
    int r = conv_gemm_tc(prec, c1, st);
    if (r != VFX_OK) return r;

    vfx_conv_desc c2;
    memset(&c2, 0, sizeof(c2));
    c2.a = d.scratch; c2.B = d.B; c2.H = 1; c2.W = nh; c2.Cin = C;
    c2.a_sW = C; c2.a_sH = (long long)nh * C; c2.a_sB = (long long)nh * C;
    c2.w = d.w2; c2.ntaps = 3;
    for (int k = 0; k < 3; ++k) { c2.dw[k] = k - 1 + (int)(r0 - h0); c2.w_off[k] = (long long)k * C * C; }
    c2.Hq = 1; c2.Wq = nr; c2.N = C; c2.sh = 1; c2.sw = 1; c2.OH = 1; c2.OW = nr;
    c2.bias = d.b2; c2.bias_mod = C;
    c2.residual = d.x + r0 * C; c2.r_sW = C; c2.r_sH = item; c2.r_sB = item;
    c2.res_enc = d.stream_enc ? 1 : 0; c2.enc_slope = 0.01f;
    if (d.write_raw) {
      c2.out_raw = dst + r0 * C; c2.o_sW = C; c2.o_sH = item; c2.o_sB = item;
      c2.raw_enc = d.stream_enc && d.stream_enc_out ? 1 : 0;
    }
    if (d.out_act) {
      c2.out_act = (char*)d.out_act + r0 * C * (long long)prec_esz(prec); c2.oa_sW = C; c2.oa_sH = item; c2.oa_sB = item;
      c2.act = d.act; c2.act_param = d.act_param;
    }
    r = conv_gemm_tc(prec, c2, st);
    if (r != VFX_OK) return r;
  }
  return VFX_OK;
}

bool pair_supported(int prec, int C, bool stream_enc) {
  return prec == VFX_PREC_TF32 ? C == 64 && stream_enc
                               : (prec == VFX_PREC_BF16 || prec == VFX_PREC_FP16) && (C == 64 || C == 128) && !stream_enc;
}

int resstack_pair(const vfx_pair_desc& d, cudaStream_t st) {
  VFX_REQUIRE(d.form == VFX_PAIR_FUSED || d.form == VFX_PAIR_BLOCKED, "resstack_pair: form %d is not a vfx_pair_form", d.form);
  const int prec = d.precision;
  if (!pair_supported(prec, d.C, d.stream_enc != 0) || (d.stream_enc && !d.x_out)) return VFX_ERR_UNSUPPORTED;
  VFX_REQUIRE(d.a && d.x && d.w1 && d.w2 && d.b1 && d.b2 && d.B > 0 && d.L > 0 && d.dilation > 0, "resstack_pair: bad arguments");
  if (d.form == VFX_PAIR_BLOCKED) return d.lens ? VFX_ERR_UNSUPPORTED : pair_blocked(d, prec, st);
  if (((uintptr_t)d.a & 15) || ((uintptr_t)d.w1 & 15) || ((uintptr_t)d.w2 & 15)) return VFX_ERR_UNSUPPORTED;
  // the fused kernel reads and writes each thread's two adjacent columns with one access
  if (((uintptr_t)d.x & 7) || ((uintptr_t)d.x_out & 7) || ((uintptr_t)d.out_act & (2 * prec_esz(prec) - 1)))
    return VFX_ERR_UNSUPPORTED;
  if (prec == VFX_PREC_TF32) return launch_fused<64, 0>(d, st);
  if (prec == VFX_PREC_BF16) return d.C == 64 ? launch_fused<64, 1>(d, st) : launch_fused<128, 1>(d, st);
  return d.C == 64 ? launch_fused<64, 2>(d, st) : launch_fused<128, 2>(d, st);
}

}  // namespace vfx

// Channels-last shifted-window convolution GEMM on the Hopper tensor cores (wgmma), the bf16 / fp16 / tf32 path of
// every Conv1d / Conv2d / ConvTranspose / Linear (field semantics: include/vfx_b200.h, vfx_conv_desc).
//
//   out[b, oh, ow, n] = bias[n % bias_mod] + residual + sum_{tap} sum_{c} W[tap][n][c] * A[b, qh+dh, qw+dw, c]
//
// Persistent, warp-specialised kernel on the pipeline of tc_pipeline.cuh (ring, feed and K loop): grid = min(tiles,
// SMs), each CTA walks a static stride over the 128 x BN output tiles in N-fastest order (the N tiles of one M tile run
// together, so their A rows come from HBM about once).
//  - Producer: the K slices are (tap, 128-byte channel slice), tap outer; a slice is the shifted input rows and the tap's
//    weight rows.  Whatever lies outside the input (convolution padding), beyond Cin or beyond N arrives as zeros, so any
//    tap offset, stride and edge is handled without a separate padded tensor.  Two forms (TMA below):
//      TMA: two tensor-map loads per slice, a box of the [B][H][W][Cin] input at the tile's origin plus the tap's offset
//      and a box of the weights; the out-of-bounds fill of the maps supplies the zeros.  A box is a rectangle of one
//      tensor, so an M tile is a rectangle of the output grid (TmaPlan) and not 128 consecutive rows of the flattened one.
//      cp.async: zero-fill copies from a per-tile row table.  It serves the launches a tensor map cannot express: ragged
//      batches, whose zeros depend on the item, and operands whose strides or weight offsets the maps do not take
//      (tma_plan).
//  - Epilogue, in one of two forms chosen on the host (tma_store_plan), each element in the same order: bias, fp32
//    residual, raw output, eval-BN affine, activation, operand for the next layer.
//      TMA store (TMA launches whose residual and outputs tensor maps can express): the producer thread loads the tile's
//      residual into the dense, swizzled epilogue buffer during the K loop, as soon as the previous tile's stores have
//      read it; the consumers combine their accumulator fragments with it in registers, write each output into the
//      buffer and one thread stores it with TMA stores, which run while the next tile's K loop does.  The maps' clipping
//      drops what the launch does not store.  Raw and operand outputs share the buffer: the operand is written once the
//      raw output's stores have read it.
//      Row loop (the others): the tile goes through a padded shared fp32 buffer and is processed row by row, with 16-byte
//      accesses where the host found every pointer, stride and column offset aligned.  A thread's column parameters are
//      read once per tile and all its residual rows are loaded before its first store.
// kind tf32 reads fp32 operands and ignores their low 13 mantissa bits: producers round tf32 operands to nearest, and the
// encoded stream of vfx_conv_desc.res_enc / raw_enc is read as round-to-nearest(lrelu(x)) by construction.
// Ragged batches (seq_in / seq_out): each item's extent on the sequence axis acts as that item's own edge, so every row
// inside it is computed from the same operands as with the item alone; a tile none of whose rows is stored is skipped.
//
// What still stands between this kernel and the roof: the A halo of the taps is re-read from L2 for every tap, every
// CTA reads its own copy of the weights from L2, the ring is 5 stages deep at BN = 128 (the fp32 epilogue buffer takes
// the rest of shared memory), the per-slice sum costs BN / 2 FADDs per slice in the consumers, and the consumers still
// spend the epilogue's arithmetic and shared-memory passes with the tensor cores idle (one buffer: a launch with both a
// raw and an operand output also waits for the raw stores to read it).
#include "tc_pipeline.cuh"

namespace vfx {

namespace {

// epilogue offsets of one tile row (ok == 0: the row is not stored)
struct OutRow { long long raw, act, res; int ok; };

// What a TMA launch carries beside the descriptor.  An M tile is the box of tw x th x tb output-grid positions
// (qw, qh, b) at a multiple of the box: a whole number of lines, or a piece of one line, of one item, or whole items,
// so that its input rows are one box of the input tensor.  Tile row r is position (r % tw, r / tw % th, r / (tw th));
// rows from tw th tb on do not exist (their shared memory is not written and their results are not stored).
// With the TMA-store epilogue (tma_store_plan) the residual and the outputs have maps of their own over the output grid
// (N, Wq', Hq', B), Wq' / Hq' the positions q with q s + r inside OW / OH: the tile's boxes at (n0, w0, h0, b0) are then
// its rows, and the maps' clipping drops the rows and columns the row-loop epilogue does not store.
struct TmaPlan {
  CUtensorMap a;           // input  (Cin, W, H, B),    box (128 bytes, tw, th, tb)
  CUtensorMap w;           // weights (Cin, N, groups), box (128 bytes, BN, 1): tap t is group wtap[t]
  CUtensorMap r, o, oa;    // residual, raw and operand output, box (128 bytes or BN columns, tw, th, tb)
  int tw, th, tb;
  int ntw, nth, mtiles;    // boxes per line, per item's lines, in all
  int wtap[9];
};

// The staged tile of the TMA-store epilogue: column boxes of ob = min(BN * esz, 128) bytes by BM rows, dense, each in the
// swizzle of its map (16-byte chunk c of row r at c ^ (r & 7) in 128-byte rows, c ^ (r / 2 & 3) in 64-byte ones).
// Byte offset of column c of row r in elements of esz bytes:
template <int BN, int ESZ> __device__ __forceinline__ uint32_t st_offset(int r, int c) {
  constexpr int OB = BN * ESZ < 128 ? BN * ESZ : 128, CPB = OB / ESZ;
  const uint32_t o = (uint32_t)(r * OB + c % CPB * ESZ);
  return (uint32_t)(c / CPB * (BM * OB)) + (o ^ ((o >> 7) & (OB / 16 - 1)) << 4);
}

// TST: the TMA-store epilogue (TMA producer only); without it, the row-loop epilogue and its row table.  Shared memory
// beside the ring: the epilogue buffer, then the row tables (TST: the buffer's two mbarriers).
template <int BN, bool TMA, bool TST> struct Cfg {
  static constexpr int EPI_LD = TST ? BN : BN + 8; // fp32 words per epilogue row; +8 keeps the fragment stores conflict-free
  static constexpr int EPI = BM * EPI_LD * 4;
  static constexpr int PROWS = TMA ? 0 : BM * 24;  // the cp.async producer's row table
  static constexpr int ROWS = TST ? 16 : PROWS + BM * (int)sizeof(OutRow);   // + the epilogue's
  using Plan = RingPlan<A_BYTES + BN * 128, EPI + ROWS, TST ? 5 : 3>;   // 4 stages at BN = 128 (TST: 5), 7 at 64, 8 at 32
};

// output-grid row m -> item b and grid position (qh, qw); false beyond the problem (M < 2^31: 32-bit divisions)
__device__ __forceinline__ bool grid_row(const vfx_conv_desc& d, int M, int m, int& b, int& qh, int& qw) {
  if (m >= M) return false;
  qw = m % d.Wq;
  const int r = m / d.Wq;
  qh = r % d.Hq; b = r / d.Hq;
  return true;
}
// row r of M tile mt -> item b and grid position (qh, qw); false where the tile has no such row
template <bool TMA>
__device__ __forceinline__ bool tile_row(const vfx_conv_desc& d, const TmaPlan& tp, int M, int mt, int r, int& b, int& qh, int& qw) {
  if (!TMA) return grid_row(d, M, mt * BM + r, b, qh, qw);
  const int j = r / tp.tw, u = mt / tp.ntw;
  qw = mt % tp.ntw * tp.tw + r % tp.tw;
  qh = u % tp.nth * tp.th + j % tp.th;
  b = u / tp.nth * tp.tb + j / tp.th;
  return j / tp.th < tp.tb && qw < d.Wq && qh < d.Hq && b < d.B;
}
// whether grid position (b, qh, qw) is stored: inside the output and, in a ragged batch, inside its item's extent.
// The producer and the consumers both decide a tile's skip from this function alone, so they walk the same tiles.
template <bool SEQ> __device__ __forceinline__ bool row_stored(const vfx_conv_desc& d, int b, int qh, int qw) {
  const int oh = qh * d.sh + d.rh, ow = qw * d.sw + d.rw;
  return oh < d.OH && ow < d.OW && (!SEQ || !d.seq_out || (d.seq_axis ? ow : oh) < d.seq_out[b]);
}

// one output element, in the order every path keeps: bias (bv = bias[n % bias_mod]), then the residual (rv, decoded
// when encoded), then the raw output (encoded when asked), then the BN affine (sc, sf = act_scale[n], act_shift[n]) and
// the activation of the operand
__device__ __forceinline__ float add_in(const vfx_conv_desc& d, float v, float bv, float rv) {
  if (d.bias) v += bv;
  if (d.residual) v += d.res_enc ? stream_dec(rv, 1.0f / d.enc_slope) : rv;
  return v;
}
__device__ __forceinline__ float raw_out(const vfx_conv_desc& d, float v) { return d.raw_enc ? stream_enc(v, d.enc_slope) : v; }
__device__ __forceinline__ float act_out(const vfx_conv_desc& d, float v, float sc, float sf) {
  const float va = d.act_scale ? fmaf(v, sc, sf) : v;
  return apply_act(va, d.act, d.act_param);
}

// TMA: the operands arrive through the tensor maps of `tp` and the M tiles are its boxes; otherwise through cp.async
// with 128 consecutive rows of the flattened output grid per M tile, `tp` unused, and the per-item extents
// (seq_in / seq_out) honoured where the descriptor carries them.
// vec: every output / residual pointer, stride and column offset allows 4-column vector accesses (row-loop epilogue).
// TST: the tile leaves through TMA stores of tp.o / tp.oa, and its residual arrives through tp.r during its K loop.
template <int BN, int KIND, bool TMA, bool TST>
__global__ void __launch_bounds__(NT, 1) conv_gemm_wgmma_kernel(const __grid_constant__ vfx_conv_desc d,
                                                                 const __grid_constant__ TmaPlan tp, const int nkc,
                                                                 const int vec) {
  static_assert(TMA || !TST, "conv_gemm_tc: the TMA-store epilogue needs the TMA producer's tile boxes");
  using T = typename OpT<KIND>::T;
  using C = Cfg<BN, TMA, TST>;
  constexpr bool SEQ = !TMA;
  constexpr int ESZ = OpT<KIND>::ESZ, AL = 16 / ESZ, BK = 128 / ESZ;   // elements per 16-byte chunk / per K slice
  constexpr int S = C::Plan::STAGES, STAGE = C::Plan::STAGE;
  extern __shared__ uint8_t smem_raw[];
  const Ring<typename C::Plan> ring{(smem_u32(smem_raw) + 1023u) & ~1023u};
  uint8_t* const gbase = smem_raw + (ring.base - smem_u32(smem_raw));
  float* const epi = reinterpret_cast<float*>(gbase + S * STAGE);
  int4* const prow = reinterpret_cast<int4*>(gbase + S * STAGE + C::EPI);        // (cp.async producer only)
  long long* const pbase = reinterpret_cast<long long*>(prow + BM);
  OutRow* const crow = reinterpret_cast<OutRow*>(gbase + S * STAGE + C::EPI + C::PROWS);   // (row-loop epilogue only)
  // TMA-store epilogue: the staged tile, and its two mbarriers (full: the buffer is free and the tile's residual has
  // landed; empty: the stores of the tile before have read the buffer)
  const uint32_t epi_s = ring.base + S * STAGE, efull = epi_s + C::EPI, eempty = efull + 8;

  const int tid = threadIdx.x;
  if (tid == 0) {
    ring.init(TMA);
    if (TST) {
      mbar_init(efull, 1);              // the producer thread's arrival (with the residual's bytes)
      mbar_init(eempty, 1);             // the consumer thread that issues the stores
    }
  }
  __syncthreads();

  // derived after each role's setmaxnreg, so that nothing stays live across it
#define VFX_TILE_WALK                                                                                              \
  const int M = d.B * d.Hq * d.Wq;                 /* < 2^31, and so is the tile count (conv_gemm_tc) */           \
  const int ntn = (d.N + BN - 1) / BN, ntiles = (TMA ? tp.mtiles : (M + BM - 1) / BM) * ntn, niter = d.ntaps * nkc; \
  const bool skips = SEQ && d.seq_out;

  if (tid < 128) {
    // ================================================================ producer
    setmaxnreg_dec<PROD_REGS>();
    VFX_TILE_WALK
    if constexpr (TMA) {
      if (tid != 0) return;
      const uint32_t bytes = (uint32_t)(tp.tw * tp.th * tp.tb * 128 + BN * 128);   // of one stage: whole boxes, zeros included
      const uint32_t rbytes = d.residual ? (uint32_t)(tp.tw * tp.th * tp.tb * BN * 4) : 0u;   // of a tile's residual
      // TST: tile i's residual goes into the epilogue buffer once the stores of tile i - 1 have read it.  That is signalled
      // after the consumers' slice min(2, slices - 1) of tile i, so the wait comes after slice S >= 5 of the tile has been
      // issued (or after its last): by then slices 0 to 3 are in the ring, and the ring stays full up to that point.
      const int rl = niter < S ? niter : S;
      auto epi_load = [&](int i, int n0, int w0, int h0, int b0) {
        if (i > 0) mbar_wait(eempty, (i - 1) & 1);
        if (!rbytes) { mbar_arrive(efull); return; }
        mbar_expect_tx(efull, rbytes);
#pragma unroll
        for (int bx = 0; bx < BN / 32; ++bx) tma_load_4d(epi_s + bx * BM * 128, &tp.r, efull, n0 + 32 * bx, w0, h0, b0);
      };
      uint32_t k = 0;                                 // K slices issued by this CTA
      int i = 0;                                      // tiles begun by this CTA
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++i) {
        const int mt = t / ntn, u = mt / tp.ntw;
        const int n0 = t % ntn * BN;
        const int w0 = mt % tp.ntw * tp.tw, h0 = u % tp.nth * tp.th, b0 = u / tp.nth * tp.tb;
        for (int it = 0; it < niter; ++it, ++k) {
          if (TST && it == rl) epi_load(i, n0, w0, h0, b0);
          ring.acquire(k);
          const int tap = it / nkc;
          const int c = (it - tap * nkc) * BK;
          const uint32_t sa = ring.stage(k), full = ring.full(k);
          mbar_expect_tx(full, bytes);
          tma_load_4d(sa, &tp.a, full, c, w0 + d.dw[tap], h0 + d.dh[tap], b0);
          tma_load_3d(sa + A_BYTES, &tp.w, full, c, n0, tp.wtap[tap]);
        }
        if (TST && rl == niter) epi_load(i, n0, w0, h0, b0);
      }
      return;
    }
    // this thread's staging work: chunk `chunk` of A rows lrow + 16 i and of B rows lrow + 16 i
    const int chunk = tid & 7, lrow = tid >> 3;
    uint32_t k = 0;                                   // K slices issued by this CTA
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
      const int m0 = t / ntn * BM;
      const int n0 = t % ntn * BN;
      named_sync(1, 128);                             // the previous tile's row table is no longer read
      // row tid: its element offset in A and its valid input ranges ih in [0, hlim), iw in [0, wlim), relative to the
      // row (the input edges and, in a ragged batch, its item's extent vfx_conv_desc.seq_in); none beyond M
      int4 q = make_int4(0, 0, 0, 0);
      long long base = 0;
      bool live = false;
      int b, qh, qw;
      if (grid_row(d, M, m0 + tid, b, qh, qw)) {
        const int rlim = SEQ && d.seq_in ? d.seq_in[b] : 0x7fffffff;
        const int hl = SEQ && d.seq_axis == 0 && rlim < d.H ? rlim : d.H, wl = SEQ && d.seq_axis == 1 && rlim < d.W ? rlim : d.W;
        q = make_int4(qh, hl > 0 ? hl : 0, qw, wl > 0 ? wl : 0);
        base = (long long)b * d.a_sB + (long long)qh * d.a_sH + (long long)qw * d.a_sW;
        live = row_stored<SEQ>(d, b, qh, qw);
      }
      prow[tid] = q;
      pbase[tid] = base;
      if (skips) {
        if (!named_sync_or(1, 128, live)) continue;   // ragged batch: no row of this tile is stored
      } else {
        named_sync(1, 128);
      }
      for (int it = 0; it < niter; ++it, ++k) {
        ring.acquire(k);
        const int tap = it / nkc;
        const int c = (it - tap * nkc) * BK + chunk * AL;
        const bool c_ok = c < d.Cin;
        const uint32_t sa = ring.stage(k), sb = sa + A_BYTES;
        const int dh = d.dh[tap], dw = d.dw[tap];
        const long long toff = (long long)dh * d.a_sH + (long long)dw * d.a_sW + c;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int r = lrow + 16 * i;
          const int4 p = prow[r];
          const bool ok = c_ok && (unsigned)(p.x + dh) < (unsigned)p.y && (unsigned)(p.z + dw) < (unsigned)p.w;
          const char* src = static_cast<const char*>(d.a) + (ok ? (pbase[r] + toff) * ESZ : 0);
          cp_async16(sa + sw128_offset(r, chunk), src, ok);
        }
#pragma unroll 4
        for (int i = 0; i < BN / 16; ++i) {
          const int n = lrow + 16 * i;
          const bool ok = c_ok && n0 + n < d.N;
          const char* src = static_cast<const char*>(d.w) + (ok ? (d.w_off[tap] + (long long)(n0 + n) * d.Cin + c) * ESZ : 0);
          cp_async16(sb + sw128_offset(n, chunk), src, ok);
        }
        ring.cp_async_handoff(k);
      }
    }
    ring.cp_async_drain(k);
    return;
  }

  // ================================================================== consumers
  setmaxnreg_inc<CONS_REGS>();
  VFX_TILE_WALK
#undef VFX_TILE_WALK
  const int ct = tid - 128, cw = ct >> 7, w = (ct >> 5) & 3, l = tid & 31;
  T* out_act = reinterpret_cast<T*>(d.out_act);
  float acc[BN / 2];
  uint32_t k = 0;                                     // K slices consumed by this CTA
  int ti = 0;                                         // tiles begun by this CTA
  const int rel = niter > 3 ? 2 : niter - 1;          // (the producer waits for it after slice S > rel + 1)
  // TST: after the tile's slice `rel`, the thread that issued the previous tile's stores hands the buffer back to the
  // producer once they have read it, early enough for the residual load to hide behind the rest of the K loop and late
  // enough for the stores to have read it (waiting stalls that thread's warpgroup)
  auto released = [&](int it) {
    if (TST && ct == 0 && it == rel && ti > 0) {
      bulk_wait_read<0>();
      mbar_arrive(eempty);
    }
  };

  for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++ti) {
    const int mt = t / ntn;
    const int n0 = t % ntn * BN;
    if (skips) {
      int b, qh, qw;
      const bool live = tile_row<TMA>(d, tp, M, mt, ct & 127, b, qh, qw) && row_stored<SEQ>(d, b, qh, qw);
      if (!named_sync_or(2, 256, live)) continue;
    }
    k_loop<BN, KIND>(acc, niter, cw, ring_feed(ring, k, l, [](int, uint32_t sa) { return sa; }, StageB{}, released));
    k += niter;

    // ---- epilogue: accumulator element (j, h, e) of lane l in warp w of consumer warpgroup cw is
    //      row cw*64 + w*16 + l/4 + 8h, column 8j + 2(l%4) + e
    if constexpr (TST) {
      // Each thread combines its own fragments with bias and the staged residual, in registers, then writes each output
      // into the buffer in its map's layout; one thread stores the boxes.  The element order is the row-loop epilogue's.
      const int u = mt / tp.ntw;
      const int w0 = mt % tp.ntw * tp.tw, h0 = u % tp.nth * tp.th, b0 = u / tp.nth * tp.tb;
      const int rq = cw * 64 + w * 16 + (l >> 2);
      uint8_t* const eb = reinterpret_cast<uint8_t*>(epi);
      mbar_wait(efull, ti & 1);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + 2 * (l & 3);
        float bv[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int n = n0 + c + e;                   // columns from N on are clipped by the stores
          bv[e] = d.bias && n < d.N ? d.bias[n < d.bias_mod ? n : n % d.bias_mod] : 0.f;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float* const v = acc + 4 * j + 2 * h;
          const float2 rv = d.residual ? *reinterpret_cast<const float2*>(eb + st_offset<BN, 4>(rq + 8 * h, c)) : make_float2(0.f, 0.f);
          v[0] = add_in(d, v[0], bv[0], rv.x);
          v[1] = add_in(d, v[1], bv[1], rv.y);
        }
      }
      // the buffer's generic writes -> the async proxy, then one thread stores its column boxes of ob bytes (cpb columns)
      auto store = [&](const CUtensorMap* map, int ob, int cpb) {
        fence_proxy_async();
        named_sync(2, 256);
        if (ct == 0) {
          for (int bx = 0; bx < BN / cpb; ++bx) tma_store_4d(map, epi_s + bx * BM * ob, n0 + bx * cpb, w0, h0, b0);
          bulk_commit();
        }
      };
      // fragment pair q = 2 j + h of this thread: its fp32 slot in the buffer (the residual's and the raw output's layout)
      auto slot = [&](int q) { return eb + st_offset<BN, 4>(rq + 8 * (q & 1), 8 * (q >> 1) + 2 * (l & 3)); };
      if (d.out_raw) {
#pragma unroll
        for (int q = 0; q < BN / 4; ++q)
          *reinterpret_cast<float2*>(slot(q)) = make_float2(raw_out(d, acc[2 * q]), raw_out(d, acc[2 * q + 1]));
        store(&tp.o, 128, 32);
      }
      if (out_act) {
        // one buffer: the operand overwrites the raw output once its stores have read it
        if (d.out_raw) {
          if (ct == 0) bulk_wait_read<0>();
          named_sync(2, 256);
        }
        // Leaky ReLU (or none) is applied in registers.  The other activations run as a loop over the thread's own slots
        // (unrolled, their code per element overflows the instruction cache).  A tf32 operand goes into the slot, a
        // 16-bit pair into the slot's first word.
        const bool cheap = d.act == VFX_ACT_LRELU || d.act == VFX_ACT_NONE;
        if (cheap) {
#pragma unroll
          for (int q = 0; q < BN / 4; ++q) {
            const int n = n0 + 8 * (q >> 1) + 2 * (l & 3);
            const bool in0 = d.act_scale && n < d.N, in1 = d.act_scale && n + 1 < d.N;
            float y0 = d.act_scale ? fmaf(acc[2 * q], in0 ? d.act_scale[n] : 1.f, in0 ? d.act_shift[n] : 0.f) : acc[2 * q];
            float y1 = d.act_scale ? fmaf(acc[2 * q + 1], in1 ? d.act_scale[n + 1] : 1.f, in1 ? d.act_shift[n + 1] : 0.f) : acc[2 * q + 1];
            if (d.act == VFX_ACT_LRELU) {
              y0 = y0 > 0.f ? y0 : y0 * d.act_param;
              y1 = y1 > 0.f ? y1 : y1 * d.act_param;
            }
            if (ESZ == 4)
              *reinterpret_cast<float2*>(slot(q)) = make_float2(round_tf32(y0), round_tf32(y1));
            else
              *reinterpret_cast<uint32_t*>(slot(q)) = pack16<KIND == 2>(y0, y1);
          }
        } else {
#pragma unroll
          for (int q = 0; q < BN / 4; ++q) *reinterpret_cast<float2*>(slot(q)) = make_float2(acc[2 * q], acc[2 * q + 1]);
        }
#pragma unroll 2
        for (int q = 0; q < (cheap ? 0 : BN / 4); ++q) {
          const int n = n0 + 8 * (q >> 1) + 2 * (l & 3);
          const bool in0 = d.act_scale && n < d.N, in1 = d.act_scale && n + 1 < d.N;
          float2* const p = reinterpret_cast<float2*>(slot(q));
          const float2 v = *p;
          const float y0 = act_out(d, v.x, in0 ? d.act_scale[n] : 1.f, in0 ? d.act_shift[n] : 0.f);
          const float y1 = act_out(d, v.y, in1 ? d.act_scale[n + 1] : 1.f, in1 ? d.act_shift[n + 1] : 0.f);
          if (ESZ == 4)
            *p = make_float2(round_tf32(y0), round_tf32(y1));
          else
            *reinterpret_cast<uint32_t*>(p) = pack16<KIND == 2>(y0, y1);
        }
        constexpr int OB = BN * ESZ < 128 ? BN * ESZ : 128;
        if (ESZ == 2) {
          // into the 16-bit layout, which overlaps other threads' slots: all are read before any is overwritten
          uint32_t y[BN / 4];
#pragma unroll
          for (int q = 0; q < BN / 4; ++q) y[q] = *reinterpret_cast<const uint32_t*>(slot(q));
          named_sync(2, 256);
#pragma unroll
          for (int q = 0; q < BN / 4; ++q)
            *reinterpret_cast<uint32_t*>(eb + st_offset<BN, ESZ>(rq + 8 * (q & 1), 8 * (q >> 1) + 2 * (l & 3))) = y[q];
        }
        store(&tp.oa, OB, OB / ESZ);
      }
      continue;
    }
    named_sync(2, 256);                               // the previous tile's epilogue has finished reading epi / crow
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = cw * 64 + w * 16 + (l >> 2) + 8 * h;
        *reinterpret_cast<float2*>(epi + row * C::EPI_LD + 8 * j + 2 * (l & 3)) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
    if (ct < BM) {
      OutRow o{0, 0, 0, 0};
      int b, qh, qw;
      if (tile_row<TMA>(d, tp, M, mt, ct, b, qh, qw) && row_stored<SEQ>(d, b, qh, qw)) {
        const int oh = qh * d.sh + d.rh, ow = qw * d.sw + d.rw;
        o.raw = (long long)b * d.o_sB + (long long)oh * d.o_sH + (long long)ow * d.o_sW + d.o_col;
        o.act = (long long)b * d.oa_sB + (long long)oh * d.oa_sH + (long long)ow * d.oa_sW + d.oa_col;
        o.res = (long long)b * d.r_sB + (long long)oh * d.r_sH + (long long)ow * d.r_sW + d.r_col;
        o.ok = 1;
      }
      crow[ct] = o;
    }
    named_sync(2, 256);

    // row by row: BN / 4 threads per row, 4 consecutive columns each, rows r0 + RPP i
    constexpr int TPR = BN / 4, RPP = 256 / TPR, RPT = BM / RPP;
    const int c4 = (ct % TPR) * 4, n = n0 + c4, r0 = ct / TPR;
    if (n >= d.N) continue;
    const int ncol = d.N - n < 4 ? d.N - n : 4;
    const bool full = vec && ncol == 4;
    // The thread's columns are the same in every row: their parameters are read once per tile.
    float bv[4], sc[4], sf[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int ne = e < ncol ? n + e : n;            // columns from N on are not stored
      bv[e] = d.bias ? d.bias[ne % d.bias_mod] : 0.f;
      sc[e] = d.act_scale ? d.act_scale[ne] : 1.f;
      sf[e] = d.act_scale ? d.act_shift[ne] : 0.f;
    }
    if (d.residual) {
      // All of the thread's residual rows are loaded before any is used and before its first store, so the tile waits
      // for memory once and not once per row (the compiler cannot move a load above a store it may alias: the tf32
      // ResStack writes the encoded stream in place over its residual).  That is safe because each residual element is
      // read by the thread that writes the same element of out_raw, and by no other: the residual's element (row, n) is
      // the output's (row, n) or lies outside it.  Bias and residual are then added into the staged tile, so that the
      // unrolled part stays small; the row pass below is a loop (unrolled with its stores, it overflows the
      // instruction cache).
      float4 rv[RPT];
#pragma unroll
      for (int i = 0; i < RPT; ++i) {
        const OutRow& o = crow[r0 + RPP * i];
        rv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (o.ok) {
          const float* p = d.residual + o.res + n;
          if (full) {
            rv[i] = *reinterpret_cast<const float4*>(p);
          } else {
            rv[i].x = p[0];
            if (ncol > 1) rv[i].y = p[1];
            if (ncol > 2) rv[i].z = p[2];
            if (ncol > 3) rv[i].w = p[3];
          }
        }
      }
#pragma unroll
      for (int i = 0; i < RPT; ++i) {
        const int r = r0 + RPP * i;
        if (!crow[r].ok) continue;
        float4* q = reinterpret_cast<float4*>(epi + r * C::EPI_LD + c4);
        const float4 v = *q;
        *q = make_float4(add_in(d, v.x, bv[0], rv[i].x), add_in(d, v.y, bv[1], rv[i].y), add_in(d, v.z, bv[2], rv[i].z),
                         add_in(d, v.w, bv[3], rv[i].w));
      }
    }
    for (int r = r0; r < BM; r += RPP) {
      const OutRow o = crow[r];
      if (!o.ok) continue;
      float4 v = *reinterpret_cast<const float4*>(epi + r * C::EPI_LD + c4);
      if (!d.residual)
        v = make_float4(add_in(d, v.x, bv[0], 0.f), add_in(d, v.y, bv[1], 0.f), add_in(d, v.z, bv[2], 0.f), add_in(d, v.w, bv[3], 0.f));
      if (full) {
        if (d.out_raw)
          *reinterpret_cast<float4*>(d.out_raw + o.raw + n) = make_float4(raw_out(d, v.x), raw_out(d, v.y), raw_out(d, v.z), raw_out(d, v.w));
        if (out_act) {
          const float y0 = act_out(d, v.x, sc[0], sf[0]), y1 = act_out(d, v.y, sc[1], sf[1]);
          const float y2 = act_out(d, v.z, sc[2], sf[2]), y3 = act_out(d, v.w, sc[3], sf[3]);
          if (ESZ == 4)
            *reinterpret_cast<float4*>(out_act + o.act + n) = make_float4(round_tf32(y0), round_tf32(y1), round_tf32(y2), round_tf32(y3));
          else
            *reinterpret_cast<uint2*>(out_act + o.act + n) = make_uint2(pack16<KIND == 2>(y0, y1), pack16<KIND == 2>(y2, y3));
        }
      } else {
        const float ve[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (e >= ncol) break;
          if (d.out_raw) d.out_raw[o.raw + n + e] = raw_out(d, ve[e]);
          if (out_act) out_act[o.act + n + e] = from_f<T>(act_out(d, ve[e], sc[e], sf[e]));
        }
      }
    }
  }
  if (TST && ct == 0) bulk_wait<0>();                // the last tile's stores, before the CTA's shared memory goes
}

// The tile boxes and the two tensor maps of a launch without per-item extents.  Returns 1 with `tp` filled, 0 where a
// tensor map cannot express the operands (the launch then takes the cp.async producer), or an error.
// Input: dimensions (Cin, W, H, B) with the descriptor's strides; the out-of-bounds fill of a box at the tile's origin
// plus the tap's offset is the zero padding on every side, at any dilation (coordinates are 32-bit and may lie wholly
// outside), the Cin tail of the last channel slice and the rows of a partial tile.
// Weights: the taps' [N][Cin] matrices start at arbitrary offsets (the ConvTranspose phase groups use some taps of a
// larger array), so the third dimension counts in units of the greatest common divisor of the offsets' differences,
// from the lowest offset.  Rows n >= N of a box are then zeros, not the next matrix.
int tma_plan(int precision, const vfx_conv_desc& d, int bn, TmaPlan& tp) {
  const long long esz = (long long)prec_esz(precision), LIM = 1LL << 40;          // tensor-map strides are below 2^40 bytes
  if (d.W <= 0 || d.H <= 0) return 0;
  // ---- tiles: a piece of a line, else whole lines of an item, else whole items
  tp.tw = d.Wq < BM ? d.Wq : BM;
  tp.th = tp.tw < d.Wq ? 1 : (d.Hq < BM / tp.tw ? d.Hq : BM / tp.tw);
  tp.tb = tp.th < d.Hq || tp.tw < d.Wq ? 1 : (d.B < BM / (tp.tw * tp.th) ? d.B : BM / (tp.tw * tp.th));
  tp.ntw = ceil_div(d.Wq, tp.tw);
  tp.nth = ceil_div(d.Hq, tp.th);
  const long long mtiles = (long long)tp.ntw * tp.nth * ceil_div(d.B, tp.tb);
  if (mtiles >= (1LL << 31) / BM) return 0;
  tp.mtiles = (int)mtiles;
  // ---- input map; the stride of a dimension of size 1 is never used: it takes the dense one, whatever the descriptor says
  const cuuint64_t adim[4] = {(cuuint64_t)d.Cin, (cuuint64_t)d.W, (cuuint64_t)d.H, (cuuint64_t)d.B};
  const long long asrc[3] = {d.a_sW, d.a_sH, d.a_sB};
  cuuint64_t astr[3];
  long long dense = d.Cin * esz;
  for (int i = 0; i < 3; ++i) {
    const long long s = adim[i + 1] > 1 ? asrc[i] * esz : dense;
    if (s <= 0 || s >= LIM || s % 16) return 0;
    astr[i] = (cuuint64_t)s;
    dense = s < LIM / (long long)adim[i + 1] ? s * (long long)adim[i + 1] : LIM;
  }
  // ---- weight map
  long long lo = d.w_off[0], g = 0;
  for (int t = 1; t < d.ntaps; ++t) lo = d.w_off[t] < lo ? d.w_off[t] : lo;
  for (int t = 0; t < d.ntaps; ++t)
    for (long long a = d.w_off[t] - lo; a;) { const long long r = g % a; g = a; a = r; }
  const long long mat = (long long)d.N * d.Cin;
  if (g == 0) g = mat;                              // one matrix
  if (lo < 0 || g < mat || g * esz >= LIM) return 0;   // matrices that overlap are left to cp.async
  long long groups = 1;
  for (int t = 0; t < d.ntaps; ++t) {
    tp.wtap[t] = (int)((d.w_off[t] - lo) / g);
    groups = tp.wtap[t] + 1 > groups ? tp.wtap[t] + 1 : groups;
  }
  const cuuint64_t wdim[3] = {(cuuint64_t)d.Cin, (cuuint64_t)d.N, (cuuint64_t)groups};
  const cuuint64_t wstr[2] = {(cuuint64_t)(d.Cin * esz), (cuuint64_t)(g * esz)};
  // ---- encode
  const EncodeTiled encode = tensor_map_encoder();
  VFX_REQUIRE(encode, "conv_gemm_tc: this CUDA driver has no cuTensorMapEncodeTiled");
  const CUtensorMapDataType dt = map_dtype(precision);
  const cuuint32_t bk = (cuuint32_t)(128 / esz), ones[4] = {1, 1, 1, 1};
  const cuuint32_t abox[4] = {bk, (cuuint32_t)tp.tw, (cuuint32_t)tp.th, (cuuint32_t)tp.tb}, wbox[3] = {bk, (cuuint32_t)bn, 1};
  CUresult r = encode(&tp.a, dt, 4, const_cast<void*>(d.a), adim, astr, abox, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  VFX_REQUIRE(r == CUDA_SUCCESS, "conv_gemm_tc: input tensor map refused (CUresult %d)", (int)r);
  r = encode(&tp.w, dt, 3, const_cast<char*>(static_cast<const char*>(d.w)) + lo * esz, wdim, wstr, wbox, ones,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  VFX_REQUIRE(r == CUDA_SUCCESS, "conv_gemm_tc: weight tensor map refused (CUresult %d)", (int)r);
  return 1;
}

// A map of the output grid, dimensions (N, Wq', Hq', B), over the tensor at p (elements of esz bytes from column col,
// strides sB / sH / sW): base p + col + rh sH + rw sW, strides (sw sW, sh sH, sB), box (cols, tw, th, tb) in the 128- or
// 64-byte swizzle of a cols * esz byte row.  Returns 1, 0 where a map cannot express it, or an error.
int grid_map(CUtensorMap& m, CUtensorMapDataType dt, long long esz, const void* p, int col, long long sB, long long sH,
             long long sW, int cols, const vfx_conv_desc& d, const TmaPlan& tp) {
  const long long LIM = 1LL << 40;
  const int wq = d.Wq < ceil_div(d.OW - d.rw, d.sw) ? d.Wq : ceil_div(d.OW - d.rw, d.sw);
  const int hq = d.Hq < ceil_div(d.OH - d.rh, d.sh) ? d.Hq : ceil_div(d.OH - d.rh, d.sh);
  if (wq <= 0 || hq <= 0) return 0;                 // nothing is stored (the row-loop epilogue tests each row)
  const char* base = static_cast<const char*>(p) + (col + d.rh * sH + d.rw * sW) * esz;
  if ((uintptr_t)base & 15) return 0;
  const cuuint64_t dim[4] = {(cuuint64_t)d.N, (cuuint64_t)wq, (cuuint64_t)hq, (cuuint64_t)d.B};
  const long long src[3] = {d.sw * sW, d.sh * sH, sB};
  cuuint64_t str[3];
  long long dense = d.N * esz;
  for (int i = 0; i < 3; ++i) {
    const long long s = dim[i + 1] > 1 ? src[i] * esz : dense;
    if (s <= 0 || s >= LIM || s % 16) return 0;
    str[i] = (cuuint64_t)s;
    dense = s < LIM / (long long)dim[i + 1] ? s * (long long)dim[i + 1] : LIM;
  }
  const cuuint32_t box[4] = {(cuuint32_t)cols, (cuuint32_t)tp.tw, (cuuint32_t)tp.th, (cuuint32_t)tp.tb}, ones[4] = {1, 1, 1, 1};
  const EncodeTiled encode = tensor_map_encoder();
  VFX_REQUIRE(encode, "conv_gemm_tc: this CUDA driver has no cuTensorMapEncodeTiled");
  const CUresult r = encode(&m, dt, 4, const_cast<char*>(base), dim, str, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            cols * esz == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  VFX_REQUIRE(r == CUDA_SUCCESS, "conv_gemm_tc: output-grid tensor map refused (CUresult %d)", (int)r);
  return 1;
}

// The residual and output maps of the TMA-store epilogue, for a launch tma_plan has planned.  Returns 1 with them in
// `tp`, 0 where one of them cannot be expressed (a base not 16-byte aligned, such as an odd column, or a stride not a
// multiple of 16 bytes: the launch keeps the row-loop epilogue), or an error.
int tma_store_plan(int precision, const vfx_conv_desc& d, int bn, TmaPlan& tp) {
  const long long esz = (long long)prec_esz(precision);
  const int acols = bn * esz < 128 ? bn : (int)(128 / esz);      // operand columns per 128-byte (or BN-wide) box
  int ok = 1;
  if (d.residual)
    ok = grid_map(tp.r, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, d.residual, d.r_col, d.r_sB, d.r_sH, d.r_sW, 32, d, tp);
  if (d.out_raw && ok == 1)
    ok = grid_map(tp.o, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, d.out_raw, d.o_col, d.o_sB, d.o_sH, d.o_sW, 32, d, tp);
  if (d.out_act && ok == 1)
    ok = grid_map(tp.oa, map_dtype(precision), esz, d.out_act, d.oa_col, d.oa_sB, d.oa_sH, d.oa_sW, acols, d, tp);
  return ok;
}

template <int BN, int KIND, bool TMA, bool TST>
int launch(const vfx_conv_desc& d, const TmaPlan& tp, int vec, cudaStream_t st) {
  const int nkc = ceil_div(d.Cin, 128 / OpT<KIND>::ESZ);
  const long long mtiles = TMA ? tp.mtiles : ((long long)d.B * d.Hq * d.Wq + BM - 1) / BM;
  const int r = launch_persistent<conv_gemm_wgmma_kernel<BN, KIND, TMA, TST>>(
      "conv_gemm_tc", Cfg<BN, TMA, TST>::Plan::SMEM, mtiles * ceil_div(d.N, BN), st, d, tp, nkc, vec);
  if (r == VFX_OK && TMA) ++g_conv_tma_launches;
  if (r == VFX_OK && TST) ++g_conv_tma_store_launches;
  return r;
}

// Launches without per-item extents go through TMA where tma_plan can express them, and among those, the ones whose
// residual and outputs tma_store_plan can express leave through TMA stores.  The cp.async instantiation reads the extents
// only where the descriptor has them, so it also runs the others.
template <int BN, int KIND>
int launch_bn(int precision, const vfx_conv_desc& d, int vec, cudaStream_t st) {
  TmaPlan tp{};
  int tma = 0;
  if (!d.seq_in && !d.seq_out && (tma = tma_plan(precision, d, BN, tp)) < 0) return tma;
  if (!tma) return launch<BN, KIND, false, false>(d, tp, vec, st);
  const int tst = tma_store_plan(precision, d, BN, tp);
  if (tst < 0) return tst;
  return tst ? launch<BN, KIND, true, true>(d, tp, vec, st) : launch<BN, KIND, true, false>(d, tp, vec, st);
}

template <int KIND>
int launch_kind(int precision, const vfx_conv_desc& d, int vec, cudaStream_t st) {
  if (d.N <= 32) return launch_bn<32, KIND>(precision, d, vec, st);
  if (d.N <= 64) return launch_bn<64, KIND>(precision, d, vec, st);
  return launch_bn<128, KIND>(precision, d, vec, st);
}

// 4 consecutive columns of every output row start 4 * esz-aligned (16 B for fp32)
bool vec_ok(const void* p, int esz, long long sB, long long sH, long long sW, int col) {
  return !p || (((uintptr_t)p & (4 * esz - 1)) == 0 && (sB | sH | sW | col) % 4 == 0);
}

}  // namespace

int conv_gemm_tc(int precision, const vfx_conv_desc& d, cudaStream_t st) {
  // ---- shapes this kernel covers; everything else returns UNSUPPORTED (the engine then runs the SIMT kernel)
  if (precision != VFX_PREC_BF16 && precision != VFX_PREC_TF32 && precision != VFX_PREC_FP16) return VFX_ERR_UNSUPPORTED;
  VFX_REQUIRE(d.ntaps >= 1 && d.ntaps <= 9, "conv_gemm: ntaps %d out of range", d.ntaps);
  VFX_REQUIRE(d.B > 0 && d.Hq > 0 && d.Wq > 0 && d.N > 0 && d.Cin > 0, "conv_gemm: empty problem");
  VFX_REQUIRE(d.a && d.w, "conv_gemm: null operand");
  VFX_REQUIRE(!d.bias || d.bias_mod > 0, "conv_gemm: bias_mod must be > 0");
  if ((d.res_enc && d.residual) || (d.raw_enc && d.out_raw))
    VFX_REQUIRE(d.enc_slope > 0.f, "conv_gemm_tc: enc_slope must be positive");
  const int esz = (int)prec_esz(precision);
  const int al = 16 / esz;                          // 16-byte cp.async chunks of operand rows
  if (d.Cin % al || d.a_sW % al || d.a_sH % al || d.a_sB % al || ((uintptr_t)d.a & 15) || ((uintptr_t)d.w & 15))
    return VFX_ERR_UNSUPPORTED;
  for (int t = 0; t < d.ntaps; ++t) if (d.w_off[t] % al) return VFX_ERR_UNSUPPORTED;
  const long long M = (long long)d.B * d.Hq * d.Wq;
  if (M + BM - 1 >= (1LL << 31)) return VFX_ERR_UNSUPPORTED;       // rows and tile row ends (m0 + 127) stay inside int
  // the ConvT phase groups and the concat buffers start rows at arbitrary columns: vector epilogue only when aligned
  const int vec = vec_ok(d.out_raw, 4, d.o_sB, d.o_sH, d.o_sW, d.o_col) &&
                  vec_ok(d.out_act, esz, d.oa_sB, d.oa_sH, d.oa_sW, d.oa_col) &&
                  vec_ok(d.residual, 4, d.r_sB, d.r_sH, d.r_sW, d.r_col);
  if (precision == VFX_PREC_TF32) return launch_kind<0>(precision, d, vec, st);
  if (precision == VFX_PREC_BF16) return launch_kind<1>(precision, d, vec, st);
  return launch_kind<2>(precision, d, vec, st);
}

}  // namespace vfx

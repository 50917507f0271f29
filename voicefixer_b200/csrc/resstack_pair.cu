// ResStack pair x' = x + conv2_{k3,d=1}(lrelu_0.01(conv1_{k3,dilation}(a) + b1)) + b2 (include/vfx_b200.h,
// vfx_resstack_pair), ResStack.forward voicefixer/vocoder/model/modules.py:592-595.
//
// Fused form (VFX_PAIR_FUSED; the engine's fused pairs): one CTA per 126 output rows of one item, two warpgroups.
// conv1 computes h for the 128 rows [r0 - 1, r0 + 127) with wgmma (a staged by cp.async into 128-byte-swizzled tiles,
// W1 streamed through the same 3-stage ring); its epilogue writes lrelu(h + b1) in the operand format into shared
// memory three times, copy t shifted up by t rows, so that conv2's tap t reads copy t as an ordinary K-major A tile
// (rows outside [0, L) are zero: conv2's padding).  conv2 streams W2 through the ring, accumulates in registers and its
// epilogue adds b2 and the residual and writes x' / act(x').  h never leaves the SM: HBM traffic is a (with a halo),
// the residual and the outputs.  Shared memory: 3 copies of h (48 KB bf16 C = 64, 96 KB tf32 C = 64 or 16-bit C = 128)
// + 3 stages of (16 KB of a + C x 128 B of weights).
//
// Ragged batches (vfx_pair_desc.lens): item b is computed as if its length were lens[b]; tiles starting beyond it exit.
//
// Blocked form (VFX_PAIR_BLOCKED, the tests' reference): conv_gemm_tc.cu's two convolutions per row block, h in a scratch.
#include <string.h>
#include "tc_ptx.cuh"
#include "wgmma_ptx.cuh"

namespace vfx {

namespace {
constexpr size_t PAIR_SCRATCH_BYTES = 32u << 20;

template <int KIND> struct PairT;
template <> struct PairT<0> { using T = tf32_t; static constexpr int ESZ = 4; };
template <> struct PairT<1> { using T = __nv_bfloat16; static constexpr int ESZ = 2; };
template <> struct PairT<2> { using T = __half; static constexpr int ESZ = 2; };

constexpr int P_ROWS = 126, P_STAGES = 3, P_A_BYTES = 128 * 128;

template <int C, int KIND> constexpr int pair_nks() { return C * PairT<KIND>::ESZ / 128; }
template <int C, int KIND> constexpr int pair_smem() {
  return P_STAGES * (P_A_BYTES + C * 128) + 3 * pair_nks<C, KIND>() * 16384 + 1024;
}

// element n of row j of an h copy (K-major, 128-byte slices of 16 KB, 128-byte swizzle)
template <int ESZ> __device__ __forceinline__ uint32_t h_offset(int j, int n) {
  const int kb = n * ESZ;
  return (uint32_t)((kb >> 7) * 16384 + j * 128 + ((((kb & 127) >> 4) ^ (j & 7)) << 4) + (kb & 15));
}

template <int C, int KIND>
__global__ void __launch_bounds__(256) pair_fused_kernel(const __grid_constant__ vfx_pair_desc d) {
  using T = typename PairT<KIND>::T;
  constexpr int ESZ = PairT<KIND>::ESZ, AL = 16 / ESZ, BK = 128 / ESZ, NKS = pair_nks<C, KIND>();
  constexpr int STAGE = P_A_BYTES + C * 128, NITER = 3 * NKS;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t hbase = sbase + P_STAGES * STAGE;
  uint8_t* const hgen = smem_raw + (hbase - smem_u32(smem_raw));

  const int tid = threadIdx.x, chunk = tid & 7, lrow = tid >> 3, wg = tid >> 7, w = (tid >> 5) & 3, l = tid & 31;
  const int b = blockIdx.y, r0 = blockIdx.x * P_ROWS;
  const long long item = (long long)b * d.L * C;
  const int L = d.lens ? d.lens[b] : d.L;         // this item's length (ragged batch): its rows beyond are padding
  if (r0 >= L) return;
  const char* __restrict__ A = reinterpret_cast<const char*>(d.a) + item * ESZ;
  const char* __restrict__ W1 = reinterpret_cast<const char*>(d.w1);
  const char* __restrict__ W2 = reinterpret_cast<const char*>(d.w2);

  // phase 1 (it < NITER): a rows + W1; phase 2: W2 only (a comes from the h copies)
  auto load = [&](int it, int s) {
    const bool p2 = it >= NITER;
    const int k = p2 ? it - NITER : it, tap = k / NKS, c = (k % NKS) * BK + chunk * AL;
    const uint32_t sa = sbase + s * STAGE, sb = sa + P_A_BYTES;
    if (!p2) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = lrow + 32 * i, g = r0 - 1 + r + (tap - 1) * d.dilation;
        const bool ok = g >= 0 && g < L;
        cp_async16(sa + sw128_offset(r, chunk), ok ? A + ((long long)g * C + c) * ESZ : A, ok);
      }
    }
    const char* Wt = p2 ? W2 : W1;
#pragma unroll
    for (int i = 0; i < C / 32; ++i) {
      const int n = lrow + 32 * i;
      cp_async16(sb + sw128_offset(n, chunk), Wt + ((long long)tap * C * C + (long long)n * C + c) * ESZ, true);
    }
  };

  float acc[C / 2];
  auto run = [&](int it0) {            // NITER K slices starting at global iteration it0 (stage = it % P_STAGES)
#pragma unroll
    for (int i = 0; i < C / 2; ++i) acc[i] = 0.f;
#pragma unroll
    for (int s = 0; s < P_STAGES - 1; ++s) {
      load(it0 + s, (it0 + s) % P_STAGES);
      cp_async_commit();
    }
    for (int k = 0; k < NITER; ++k) {
      const int it = it0 + k;
      cp_async_wait<P_STAGES - 2>();
      fence_proxy_async();
      __syncthreads();
      if (k + P_STAGES - 1 < NITER) load(it + P_STAGES - 1, (it + P_STAGES - 1) % P_STAGES);
      cp_async_commit();
      const uint32_t sa = sbase + (it % P_STAGES) * STAGE;
      const uint32_t a_tile = it < NITER ? sa + wg * 64 * 128 : hbase + (uint32_t)k * 16384 + wg * 64 * 128;
      const uint64_t da = sw128_desc(a_tile), db = sw128_desc(sa + P_A_BYTES);
      float part[C / 2];
#pragma unroll
      for (int i = 0; i < C / 2; ++i) part[i] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) Wgmma<C, KIND>::mma(part, da + 2 * kk, db + 2 * kk);
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < C / 2; ++i) acc[i] += part[i];     // round-to-nearest sum of the slices (conv_gemm_tc.cu)
    }
    cp_async_wait<0>();
    __syncthreads();
  };

  // ---- conv1 -> h copies
  run(0);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int i = wg * 64 + w * 16 + (l >> 2) + 8 * h, g = r0 - 1 + i;
    const bool inside = g >= 0 && g < L;
#pragma unroll
    for (int j = 0; j < C / 8; ++j) {
      const int n = 8 * j + 2 * (l & 3);
      float v0 = acc[4 * j + 2 * h] + d.b1[n], v1 = acc[4 * j + 2 * h + 1] + d.b1[n + 1];
      v0 = inside ? (v0 > 0.f ? v0 : 0.01f * v0) : 0.f;
      v1 = inside ? (v1 > 0.f ? v1 : 0.01f * v1) : 0.f;
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        const int jr = i - t;
        if (jr < 0) continue;
        uint8_t* dst = hgen + t * NKS * 16384 + h_offset<ESZ>(jr, n);
        if (ESZ == 2) {
          *reinterpret_cast<uint32_t*>(dst) = pack16<KIND == 2>(v0, v1);
        } else {
          *reinterpret_cast<float2*>(dst) = make_float2(round_tf32(v0), round_tf32(v1));
        }
      }
    }
  }
  fence_proxy_async();
  __syncthreads();

  // ---- conv2 from the h copies, residual, outputs
  run(NITER);
  float* dst = d.x_out ? d.x_out : d.x;
  T* out_act = reinterpret_cast<T*>(d.out_act);
  // acc + b2 and every residual element of the thread are loaded before the first store, so the stores (which may
  // overwrite x in place) do not serialise the loads; each element is read and written by this thread alone.
  float xr[C / 2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int i = wg * 64 + w * 16 + (l >> 2) + 8 * h, g = r0 + i;
    const bool live = i < P_ROWS && g < L;
    const long long row = item + (long long)g * C;
#pragma unroll
    for (int j = 0; j < C / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = 8 * j + 2 * (l & 3) + e;
        acc[4 * j + 2 * h + e] += d.b2[n];
        xr[4 * j + 2 * h + e] = live ? d.x[row + n] : 0.f;
      }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int i = wg * 64 + w * 16 + (l >> 2) + 8 * h, g = r0 + i;
    if (i >= P_ROWS || g >= L) continue;
    const long long row = item + (long long)g * C;
#pragma unroll
    for (int j = 0; j < C / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = 8 * j + 2 * (l & 3) + e;
        const float r = xr[4 * j + 2 * h + e];
        const float v = acc[4 * j + 2 * h + e] + (d.stream_enc ? stream_dec(r, 100.0f) : r);
        if (d.write_raw) dst[row + n] = (d.stream_enc && d.stream_enc_out) ? stream_enc(v, 0.01f) : v;
        if (out_act) out_act[row + n] = from_f<T>(apply_act(v, d.act, d.act_param));
      }
  }
}

template <int C, int KIND>
int launch_fused(const vfx_pair_desc& d, cudaStream_t st) {
  constexpr int smem = pair_smem<C, KIND>();
  static unsigned long long attr_set = 0;      // devices on which the shared-memory limit has been raised
  int dev = 0;
  VFX_CUDA_CHECK(cudaGetDevice(&dev));
  if (dev >= 64 || !(attr_set >> dev & 1)) {
    VFX_CUDA_CHECK(cudaFuncSetAttribute(pair_fused_kernel<C, KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    if (dev < 64) attr_set |= 1ull << dev;
  }
  dim3 grid(ceil_div(d.L, P_ROWS), d.B);
  pair_fused_kernel<C, KIND><<<grid, 256, smem, st>>>(d);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
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
  if (prec == VFX_PREC_TF32) return launch_fused<64, 0>(d, st);
  if (prec == VFX_PREC_BF16) return d.C == 64 ? launch_fused<64, 1>(d, st) : launch_fused<128, 1>(d, st);
  return d.C == 64 ? launch_fused<64, 2>(d, st) : launch_fused<128, 2>(d, st);
}

}  // namespace vfx

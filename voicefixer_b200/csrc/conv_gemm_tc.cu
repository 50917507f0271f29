// Channels-last shifted-window convolution GEMM on the Hopper tensor cores (wgmma), the bf16 / fp16 / tf32 path of
// every Conv1d / Conv2d / ConvTranspose / Linear (field semantics: include/vfx_b200.h, vfx_conv_desc).
//
//   out[b, oh, ow, n] = bias[n % bias_mod] + residual + sum_{tap} sum_{c} W[tap][n][c] * A[b, qh+dh, qw+dw, c]
//
// A CTA computes a 128 x BN output tile with two warpgroups (64 rows each, one m64nBN wgmma accumulator in
// registers).  The K loop runs over (tap, 128-byte channel slice): every thread stages 16-byte chunks of the
// shifted input rows and of the tap's weight rows with cp.async into a 4-stage ring of 128-byte-swizzled K-major
// tiles; chunks outside the input (convolution padding), beyond Cin or beyond N are zero-filled by the copy itself,
// so any tap offset, stride and edge is handled without a separate padded tensor.  kind tf32 reads fp32 operands and
// ignores their low 13 mantissa bits: producers round tf32 operands to nearest, and the encoded stream of
// vfx_conv_desc.res_enc / raw_enc is read as round-to-nearest(lrelu(x)) by construction.  The epilogue (bias, fp32
// residual, eval-BN affine, activation, operand for the next layer) works on the accumulator registers directly.
// Ragged batches (seq_in / seq_out): each item's extent on the sequence axis acts as that item's own edge, so every row
// inside it is computed from the same operands as with the item alone.
#include "tc_ptx.cuh"
#include "wgmma_ptx.cuh"

namespace vfx {

namespace {

constexpr int BM = 128, NT = 256, STAGES = 4;
constexpr int A_BYTES = BM * 128;

template <int KIND> struct OpT;
template <> struct OpT<0> { using T = tf32_t; static constexpr int ESZ = 4; };
template <> struct OpT<1> { using T = __nv_bfloat16; static constexpr int ESZ = 2; };
template <> struct OpT<2> { using T = __half; static constexpr int ESZ = 2; };

template <int BN> constexpr int smem_bytes() { return STAGES * (A_BYTES + BN * 128) + 1024; }

// SEQ: the descriptor carries per-item extents (seq_in / seq_out); without them the kernel is compiled without the checks
template <int BN, int KIND, bool SEQ>
__global__ void __launch_bounds__(NT) conv_gemm_wgmma_kernel(const __grid_constant__ vfx_conv_desc d, const int nkc) {
  using T = typename OpT<KIND>::T;
  constexpr int ESZ = OpT<KIND>::ESZ, AL = 16 / ESZ, BK = 128 / ESZ;   // elements per 16-byte chunk / per K slice
  constexpr int STAGE = A_BYTES + BN * 128;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;

  const int tid = threadIdx.x;
  const long long M = (long long)d.B * d.Hq * d.Wq;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const char* __restrict__ A = reinterpret_cast<const char*>(d.a);
  const char* __restrict__ Wt = reinterpret_cast<const char*>(d.w);

  // ---- this thread's staging work: chunk `chunk` of A rows lrow + 32 i and of B rows lrow + 32 i
  const int chunk = tid & 7, lrow = tid >> 3;
  int rb[4], rh[4], rw[4], rlim[4];     // rlim: the item's extent on the sequence axis (vfx_conv_desc.seq_in)
  bool live = false;                    // some row of this thread is stored (checked only with seq_out)
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + lrow + 32 * i;
    if (m < M) {
      rw[i] = (int)(m % d.Wq);
      const long long r = m / d.Wq;
      rh[i] = (int)(r % d.Hq); rb[i] = (int)(r / d.Hq);
      rlim[i] = SEQ && d.seq_in ? d.seq_in[rb[i]] : 0x7fffffff;
      if (SEQ && d.seq_out) {
        const int oh = rh[i] * d.sh + d.rh, ow = rw[i] * d.sw + d.rw;
        live |= oh < d.OH && ow < d.OW && (d.seq_axis ? ow : oh) < d.seq_out[rb[i]];
      }
    } else {
      rb[i] = -1; rh[i] = 0; rw[i] = 0; rlim[i] = 0;
    }
  }
  // ragged batch: a tile whose 128 rows all lie beyond their items' extents has nothing to store
  if (SEQ && d.seq_out && !__syncthreads_or(live)) return;
  const int niter = d.ntaps * nkc;
  auto load_stage = [&](int it, int s) {
    const int tap = it / nkc;
    const int c = (it - tap * nkc) * BK + chunk * AL;
    const bool c_ok = c < d.Cin;
    const uint32_t sa = sbase + s * STAGE, sb = sa + A_BYTES;
    const int dh = d.dh[tap], dw = d.dw[tap];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = lrow + 32 * i;
      const int ih = rh[i] + dh, iw = rw[i] + dw;
      const bool ok = c_ok && rb[i] >= 0 && ih >= 0 && ih < d.H && iw >= 0 && iw < d.W && (!SEQ || (d.seq_axis ? iw : ih) < rlim[i]);
      const char* src = ok ? A + ((long long)rb[i] * d.a_sB + (long long)ih * d.a_sH + (long long)iw * d.a_sW + c) * ESZ : A;
      cp_async16(sa + sw128_offset(r, chunk), src, ok);
    }
#pragma unroll
    for (int i = 0; i < BN / 32; ++i) {
      const int n = lrow + 32 * i;
      const bool ok = c_ok && n0 + n < d.N;
      const char* src = ok ? Wt + (d.w_off[tap] + (long long)(n0 + n) * d.Cin + c) * ESZ : Wt;
      cp_async16(sb + sw128_offset(n, chunk), src, ok);
    }
  };

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  const int wg = tid >> 7;

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < niter) load_stage(s, s);
    cp_async_commit();
  }
  for (int it = 0; it < niter; ++it) {
    cp_async_wait<STAGES - 2>();          // this thread's chunks of stage `it` have landed
    fence_proxy_async();
    __syncthreads();                      // ... everyone's, and stage it-1 is no longer read by either warpgroup
    if (it + STAGES - 1 < niter) load_stage(it + STAGES - 1, (it + STAGES - 1) % STAGES);
    cp_async_commit();
    const uint32_t sa = sbase + (it % STAGES) * STAGE;
    const uint64_t da = sw128_desc(sa + wg * 64 * 128), db = sw128_desc(sa + A_BYTES);
    float part[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) part[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) Wgmma<BN, KIND>::mma(part, da + 2 * kk, db + 2 * kk);   // 32 bytes of K each
    wgmma_commit();
    wgmma_wait<0>();
    // the tensor core's accumulator adds truncate; summing the K slices here rounds to nearest, so the error of
    // long reductions (9 taps x 768 channels) does not build up as a bias
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
  }
  cp_async_wait<0>();

  // ---- epilogue: accumulator element (j, h, e) of lane l in warp w of warpgroup wg is
  //      row wg*64 + w*16 + l/4 + 8h, column 8j + 2(l%4) + e
  const int w = (tid >> 5) & 3, l = tid & 31;
  T* out_act = reinterpret_cast<T*>(d.out_act);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const long long m = m0 + wg * 64 + w * 16 + (l >> 2) + 8 * h;
    if (m >= M) continue;
    const int qw = (int)(m % d.Wq);
    const long long r = m / d.Wq;
    const int qh = (int)(r % d.Hq), b = (int)(r / d.Hq);
    const int oh = qh * d.sh + d.rh, ow = qw * d.sw + d.rw;
    if (oh >= d.OH || ow >= d.OW) continue;
    if (SEQ && d.seq_out && (d.seq_axis ? ow : oh) >= d.seq_out[b]) continue;
    const long long o_raw = (long long)b * d.o_sB + (long long)oh * d.o_sH + (long long)ow * d.o_sW + d.o_col;
    const long long o_act = (long long)b * d.oa_sB + (long long)oh * d.oa_sH + (long long)ow * d.oa_sW + d.oa_col;
    const long long o_res = (long long)b * d.r_sB + (long long)oh * d.r_sH + (long long)ow * d.r_sW + d.r_col;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = n0 + 8 * j + 2 * (l & 3) + e;
        if (n >= d.N) continue;
        float v = acc[4 * j + 2 * h + e];
        if (d.bias) v += d.bias[n % d.bias_mod];
        if (d.residual) {
          const float rv = d.residual[o_res + n];
          v += d.res_enc ? stream_dec(rv, 1.0f / d.enc_slope) : rv;
        }
        if (d.out_raw) d.out_raw[o_raw + n] = d.raw_enc ? stream_enc(v, d.enc_slope) : v;
        if (out_act) {
          const float va = d.act_scale ? fmaf(v, d.act_scale[n], d.act_shift[n]) : v;
          out_act[o_act + n] = from_f<T>(apply_act(va, d.act, d.act_param));
        }
      }
  }
}

template <int BN, int KIND, bool SEQ>
int launch(const vfx_conv_desc& d, cudaStream_t st) {
  constexpr int smem = smem_bytes<BN>();
  static unsigned long long attr_set = 0;      // devices on which the shared-memory limit has been raised
  int dev = 0;
  VFX_CUDA_CHECK(cudaGetDevice(&dev));
  if (dev >= 64 || !(attr_set >> dev & 1)) {
    VFX_CUDA_CHECK(cudaFuncSetAttribute(conv_gemm_wgmma_kernel<BN, KIND, SEQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    if (dev < 64) attr_set |= 1ull << dev;
  }
  const long long M = (long long)d.B * d.Hq * d.Wq;
  const int nkc = ceil_div(d.Cin, 128 / OpT<KIND>::ESZ);
  dim3 grid(ceil_div(M, BM), ceil_div(d.N, BN));
  conv_gemm_wgmma_kernel<BN, KIND, SEQ><<<grid, NT, smem, st>>>(d, nkc);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

template <int KIND, bool SEQ>
int launch_n(const vfx_conv_desc& d, cudaStream_t st) {
  if (d.N <= 32) return launch<32, KIND, SEQ>(d, st);
  if (d.N <= 64) return launch<64, KIND, SEQ>(d, st);
  return launch<128, KIND, SEQ>(d, st);
}

template <int KIND>
int launch_kind(const vfx_conv_desc& d, cudaStream_t st) {
  return (d.seq_in || d.seq_out) ? launch_n<KIND, true>(d, st) : launch_n<KIND, false>(d, st);
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
  const int al = 16 / (int)prec_esz(precision);     // 16-byte cp.async chunks of operand rows
  if (d.Cin % al || d.a_sW % al || d.a_sH % al || d.a_sB % al || ((uintptr_t)d.a & 15) || ((uintptr_t)d.w & 15))
    return VFX_ERR_UNSUPPORTED;
  for (int t = 0; t < d.ntaps; ++t) if (d.w_off[t] % al) return VFX_ERR_UNSUPPORTED;
  if (ceil_div((long long)d.B * d.Hq * d.Wq, BM) >= (1LL << 31)) return VFX_ERR_UNSUPPORTED;
  if (precision == VFX_PREC_TF32) return launch_kind<0>(d, st);
  if (precision == VFX_PREC_BF16) return launch_kind<1>(d, st);
  return launch_kind<2>(d, st);
}

}  // namespace vfx

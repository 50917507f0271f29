// Generic channels-last shifted-window convolution GEMM, SIMT fp32-FMA implementation.
//
//   out[b, oh, ow, n] = bias[n] + residual + sum_{tap} sum_{c} W[tap][n][c] * A[b, qh+dh, qw+dw, c]
//
// This is the validation-precision path (VFX_PREC_FP32: fp32 operands, fp32 FMA, fixed summation
// order => deterministic) behind every Conv1d / Conv2d / ConvTranspose / Linear of the reference:
//   Conv2d 3x3            voicefixer/restorer/modules.py:19-41,70-71
//   Conv2d 1x1 shortcut   voicefixer/restorer/modules.py:46-53,73-74
//   ConvTranspose2d       voicefixer/restorer/modules.py:113-122,150 (4 output-parity phases)
//   Linear / GRU W_ih     voicefixer/restorer/model.py:71-98,35-42
//   Conv1d k3/k7 dilated  voicefixer/vocoder/model/generator.py:33-54,75,96; modules.py:550-576
//   ConvTranspose1d       voicefixer/vocoder/model/modules.py:451-459 (u output phases, 2 taps each)
// With bf16 (or tf32-rounded) operands it reproduces the tensor-core path's arithmetic (the products are
// exact in fp32) and is used by tests to cross-check the wgmma kernel.
#include "vfx_common.cuh"

namespace vfx {

namespace {

constexpr int BM = 128, BN = 64, BK = 16, NT = 256;

template <typename T> struct Vec8;   // 8 consecutive operand elements
template <> struct Vec8<float> {
  float v[8];
  __device__ void load(const float* p) {
    float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
};
// tf32 operands: what the tf32 tensor-core instructions do with an fp32 word -- the low 13 mantissa bits are ignored
// (tools/probe_tf32_rounding.py).  Pre-rounded operands pass through unchanged; an encoded stream (res_enc / raw_enc)
// comes out as round-to-nearest(lrelu(x)), exactly as on the tensor core.
template <> struct Vec8<tf32_t> {
  float v[8];
  __device__ void load(const tf32_t* p) {
    const uint4 a = *reinterpret_cast<const uint4*>(p), b = *reinterpret_cast<const uint4*>(p + 4);
    const uint32_t u[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = __uint_as_float(u[i] & 0xFFFFE000u);
  }
};
template <> struct Vec8<__half> {
  float v[8];
  __device__ void load(const __half* p) {
    uint4 r = *reinterpret_cast<const uint4*>(p);
    const __half2* h = reinterpret_cast<const __half2*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = __half22float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
  }
};
template <> struct Vec8<__nv_bfloat16> {
  float v[8];
  __device__ void load(const __nv_bfloat16* p) {
    uint4 r = *reinterpret_cast<const uint4*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = __bfloat1622float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
  }
};

template <typename T>
__global__ void __launch_bounds__(NT) conv_gemm_simt_kernel(const vfx_conv_desc d, const bool vec_ok) {
  __shared__ __align__(16) float As[BK][BM];
  __shared__ __align__(16) float Bs[BK][BN];
  __shared__ int row_b[BM], row_h[BM], row_w[BM], row_lim[BM];

  const int tid = threadIdx.x;
  const long long M = (long long)d.B * d.Hq * d.Wq;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const T* __restrict__ A = reinterpret_cast<const T*>(d.a);
  const T* __restrict__ Wt = reinterpret_cast<const T*>(d.w);

  if (tid < BM) {
    long long m = m0 + tid;
    if (m < M) {
      int qw = (int)(m % d.Wq);
      long long r = m / d.Wq;
      row_w[tid] = qw; row_h[tid] = (int)(r % d.Hq); row_b[tid] = (int)(r / d.Hq);
      row_lim[tid] = d.seq_in ? d.seq_in[row_b[tid]] : 0x7fffffff;     // the item's extent (vfx_conv_desc.seq_in)
    } else {
      row_b[tid] = -1; row_h[tid] = 0; row_w[tid] = 0; row_lim[tid] = 0;
    }
  }
  if (d.seq_out) {     // ragged batch: a tile whose rows all lie beyond their items' extents has nothing to store
    bool live = false;
    if (tid < BM && row_b[tid] >= 0) {
      const int oh = row_h[tid] * d.sh + d.rh, ow = row_w[tid] * d.sw + d.rw;
      live = oh < d.OH && ow < d.OW && (d.seq_axis ? ow : oh) < d.seq_out[row_b[tid]];
    }
    if (!__syncthreads_or(live)) return;
  }
  __syncthreads();

  const int tx = tid & 15, ty = tid >> 4;
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int a_row = tid >> 1, a_k = (tid & 1) * 8;     // A loader: 128 rows x 2 halves of 8
  const int b_row = tid >> 2, b_k = (tid & 3) * 4;     // B loader: 64 rows x 4 quarters of 4
  const int ab = row_b[a_row], ah = row_h[a_row], aw = row_w[a_row], alim = row_lim[a_row];
  const int bn = n0 + b_row;

  for (int tap = 0; tap < d.ntaps; ++tap) {
    const int ih = ah + d.dh[tap], iw = aw + d.dw[tap];
    const bool inb = (ab >= 0) && ih >= 0 && ih < d.H && iw >= 0 && iw < d.W && (d.seq_axis ? iw : ih) < alim;
    const T* ap = A + (long long)(ab < 0 ? 0 : ab) * d.a_sB + (long long)ih * d.a_sH + (long long)iw * d.a_sW;
    const T* wp = Wt + d.w_off[tap] + (long long)bn * d.Cin;
    for (int c0 = 0; c0 < d.Cin; c0 += BK) {
      // ---- load A (8 channels of one row)
      float av[8];
      if (inb && vec_ok) {
        Vec8<T> v; v.load(ap + c0 + a_k);
#pragma unroll
        for (int j = 0; j < 8; ++j) av[j] = v.v[j];
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          int c = c0 + a_k + j;
          av[j] = (inb && c < d.Cin) ? to_f(ap[c]) : 0.f;
        }
      }
      float bv[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int c = c0 + b_k + j;
        bv[j] = (bn < d.N && c < d.Cin) ? to_f(wp[c]) : 0.f;
      }
      __syncthreads();   // previous tile fully consumed
#pragma unroll
      for (int j = 0; j < 8; ++j) As[a_k + j][a_row] = av[j];
#pragma unroll
      for (int j = 0; j < 4; ++j) Bs[b_k + j][b_row] = bv[j];
      __syncthreads();
#pragma unroll
      for (int k = 0; k < BK; ++k) {
        float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 8]);
        float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * 8 + 4]);
        float4 b0 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
        float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        float b[4] = {b0.x, b0.y, b0.z, b0.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
    }
  }

  // ---- epilogue
  T* out_act = reinterpret_cast<T*>(d.out_act);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = ty * 8 + i;
    const int b = row_b[r];
    if (b < 0) continue;
    const int oh = row_h[r] * d.sh + d.rh, ow = row_w[r] * d.sw + d.rw;
    if (oh >= d.OH || ow >= d.OW) continue;
    if (d.seq_out && (d.seq_axis ? ow : oh) >= d.seq_out[b]) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= d.N) continue;
      float v = acc[i][j];
      if (d.bias) v += d.bias[n % d.bias_mod];
      if (d.residual) {
        const float r = d.residual[(long long)b * d.r_sB + (long long)oh * d.r_sH + (long long)ow * d.r_sW + d.r_col + n];
        v += d.res_enc ? stream_dec(r, 1.0f / d.enc_slope) : r;
      }
      if (d.out_raw)
        d.out_raw[(long long)b * d.o_sB + (long long)oh * d.o_sH + (long long)ow * d.o_sW + d.o_col + n] =
            d.raw_enc ? stream_enc(v, d.enc_slope) : v;
      if (out_act) {
        const float va = d.act_scale ? fmaf(v, d.act_scale[n], d.act_shift[n]) : v;
        out_act[(long long)b * d.oa_sB + (long long)oh * d.oa_sH + (long long)ow * d.oa_sW + d.oa_col + n] =
            from_f<T>(apply_act(va, d.act, d.act_param));
      }
    }
  }
}

}  // namespace

int conv_gemm_simt(int precision, const vfx_conv_desc& d, cudaStream_t st) {
  VFX_REQUIRE(d.ntaps >= 1 && d.ntaps <= 9, "conv_gemm: ntaps %d out of range", d.ntaps);
  VFX_REQUIRE(d.B > 0 && d.Hq > 0 && d.Wq > 0 && d.N > 0 && d.Cin > 0, "conv_gemm: empty problem");
  VFX_REQUIRE(d.a && d.w, "conv_gemm: null operand");
  VFX_REQUIRE(!d.bias || d.bias_mod > 0, "conv_gemm: bias_mod must be > 0");
  const long long M = (long long)d.B * d.Hq * d.Wq;
  dim3 grid(ceil_div(M, BM), ceil_div(d.N, BN));
  const int esz = (int)prec_esz(precision);
  const int al = 16 / esz;   // elements per 16 bytes
  bool vec_ok = (d.Cin % BK == 0) && (d.a_sB % al == 0) && (d.a_sH % al == 0) && (d.a_sW % al == 0) &&
                ((uintptr_t)d.a % 16 == 0);
  if (precision == VFX_PREC_BF16)
    conv_gemm_simt_kernel<__nv_bfloat16><<<grid, NT, 0, st>>>(d, vec_ok);
  else if (precision == VFX_PREC_FP16)
    conv_gemm_simt_kernel<__half><<<grid, NT, 0, st>>>(d, vec_ok);
  else if (precision == VFX_PREC_TF32)     // fp32 FMA on tf32-rounded operands (products exact): same arithmetic as wgmma tf32
    conv_gemm_simt_kernel<tf32_t><<<grid, NT, 0, st>>>(d, vec_ok);
  else
    conv_gemm_simt_kernel<float><<<grid, NT, 0, st>>>(d, vec_ok);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

}  // namespace vfx

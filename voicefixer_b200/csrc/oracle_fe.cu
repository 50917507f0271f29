// Front end of Vocoder.oracle (voicefixer/vocoder/base.py:61-73) on the device, item by item of a ragged batch:
// peak-normalise, |librosa.stft| (n_fft 2048, hop 441, periodic Hann, center, librosa 0.10's pad_mode="constant"),
// the Slaney-normalised HTK mel basis, 20 log10(max(1e-5, mel)) - 20, normalise and clip to [-4, 4], then the -4 tail
// pad of pre() (vocoder/model/util.py).  The restore front end (frontend.cu) differs in nearly every step: reflection
// padding, no peak scaling, the 1e-8 magnitude clamp, the checkpoint's own mel filterbank and a linear-mel output.
#include <algorithm>
#include "vfx_common.cuh"
#include "fft.cuh"

namespace vfx {

namespace {

// peak[b] = max |x| over item b's own samples.  The non-negative floats' bit patterns order like their values, so an
// atomicMax on the bits is an exact maximum whatever the block partition.  frames[b] (optional) = 1 + L_b / 441.
__global__ void __launch_bounds__(256) oracle_peak_kernel(const float* __restrict__ wav, int L_cap,
                                                          const int* __restrict__ lens, unsigned int* __restrict__ peak_bits,
                                                          int* __restrict__ frames) {
  const int b = blockIdx.y, tid = threadIdx.x;
  const int Lb = lens ? min(max(lens[b], 1), L_cap) : L_cap;
  if (frames && blockIdx.x == 0 && tid == 0) frames[b] = 1 + Lb / 441;
  const float* x = wav + (long long)b * L_cap;
  float m = 0.f;
  for (long long i = (long long)blockIdx.x * 256 + tid; i < Lb; i += (long long)gridDim.x * 256) m = fmaxf(m, fabsf(x[i]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ float wm[8];
  if ((tid & 31) == 0) wm[tid >> 5] = m;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < 8; ++w) m = fmaxf(m, wm[w]);
    atomicMax(peak_bits + b, __float_as_uint(m));
  }
}

// One block per (conditioning row t, item b).  Row t < T_b is STFT frame t: samples t * 441 - 1024 + n, zero outside
// [0, L_b), each divided by the item's peak (IEEE division, numpy's float32 wav / max), times the periodic Hann in double
// (librosa's stft takes a float64 window from get_window and multiplies the float32 frames by it without a cast; a
// float32 window product moves a full-scale tone's output by up to 1e-3), packed into a 1024-point complex FFT in double
// (numpy's rfft computes in float64; a float32 transform of a pure tone is off by up to 1e-3 in the normalised output,
// where the tone's packed mirror bin cancels) and untangled; rounded to complex64 and |X| in float32
// without a clamp (np.abs), the banded mel basis, and the dB / normalise epilogue in double as numpy evaluates it (the
// float64 min_level promotes it), rounded to fp32 and then to the operand format.
template <typename T>
__global__ void __launch_bounds__(256) oracle_mel_kernel(const float* __restrict__ wav, int L_cap, int Tc_cap,
                                                         const int* __restrict__ lens,
                                                         const unsigned int* __restrict__ peak_bits,
                                                         const float* __restrict__ basis, const int* __restrict__ b_start,
                                                         const int* __restrict__ b_len, T* __restrict__ cond_op,
                                                         float* __restrict__ cond_f32) {
  __shared__ double2 bufA[1024], bufB[1024], tw[1024];     // 48 KB; the magnitudes reuse the FFT's free buffer
  const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int Lb = lens ? min(max(lens[b], 1), L_cap) : L_cap;
  const int Tb = 1 + Lb / 441, Tcb = Tb + Tb % 2 + 4;
  const long long row = ((long long)b * Tc_cap + t) * 128;
  if (t >= Tb) {                                   // the -4 tail of pre(); past Tc_b, rows no kernel reads
    if (tid < 128) {
      if (cond_op) cond_op[row + tid] = from_f<T>(-4.0f);
      if (cond_f32) cond_f32[row + tid] = t < Tcb ? -4.0f : 0.0f;
    }
    return;
  }
  const float peak = __uint_as_float(peak_bits[b]);
  const float* x = wav + (long long)b * L_cap;
  const int base = t * 441 - 1024;
  for (int k = tid; k < 1024; k += 256) {
    double s, c;
    sincospi(-k / 1024.0, &s, &c);                            // exp(-2 pi i k / 2048)
    tw[k] = make_double2(c, s);
  }
  for (int n = tid; n < 1024; n += 256) {
    double v[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = 2 * n + h, i = base + j;
      const float s = (i >= 0 && i < Lb) ? __fdiv_rn(x[i], peak) : 0.0f;
      v[h] = (double)s * (0.5 - 0.5 * cospi(j / 1024.0));      // 0.5 - 0.5 cos(2 pi j / 2048)
    }
    bufA[n] = make_double2(v[0], v[1]);
  }
  __syncthreads();
  const double2* Z = fft1024(bufA, bufB, tw, tid);
  float* mag = reinterpret_cast<float*>(Z == bufA ? bufB : bufA);
  for (int k = tid; k <= 1024; k += 256) {
    const double2 X = rfft_untangle(Z, tw, k);
    const float re = (float)X.x, im = (float)X.y;
    mag[k] = sqrtf(re * re + im * im);
  }
  __syncthreads();
  if (tid < 128) {
    const int s = b_start[tid], n = b_len[tid];
    const float* f = basis + (long long)tid * 1025 + s;
    float acc = 0.f;
    for (int j = 0; j < n; ++j) acc = fmaf(mag[s + j], f[j], acc);
    const double min_level = exp(-100.0 / 20.0 * log(10.0));
    double S = 20.0 * log10(fmax(min_level, fabs((double)acc))) - 20.0;
    S = fmin(fmax(8.0 * ((S + 115.0) / 115.0) - 4.0, -4.0), 4.0);
    const float c = (float)S;
    if (cond_op) cond_op[row + tid] = from_f<T>(c);
    if (cond_f32) cond_f32[row + tid] = c;
  }
}

}  // namespace

int oracle_frontend(const float* wav, int B, int L_cap, const int* lens, const float* basis, const int* b_start,
                    const int* b_len, unsigned int* peak_bits, int* frames, void* cond_op, int precision, float* cond_f32, cudaStream_t st) {
  VFX_REQUIRE(wav && B > 0 && L_cap > 0 && peak_bits && (cond_op || cond_f32), "oracle_frontend: bad arguments");
  const int T = 1 + L_cap / 441, Tc = T + T % 2 + 4;
  VFX_CUDA_CHECK(cudaMemsetAsync(peak_bits, 0, sizeof(unsigned int) * B, st));
  dim3 pgrid((unsigned)std::min<long long>(ceil_div(L_cap, 256 * 16), 256), B);
  oracle_peak_kernel<<<pgrid, 256, 0, st>>>(wav, L_cap, lens, peak_bits, frames);
  VFX_LAUNCH_CHECK();
  dim3 grid(Tc, B);
#define VFX_ORACLE_LAUNCH(TY)                                                                                     \
  oracle_mel_kernel<TY><<<grid, 256, 0, st>>>(wav, L_cap, Tc, lens, peak_bits, basis, b_start, b_len, \
                                              reinterpret_cast<TY*>(cond_op), cond_f32)
  if (cond_op && precision == VFX_PREC_BF16) VFX_ORACLE_LAUNCH(__nv_bfloat16);
  else if (cond_op && precision == VFX_PREC_FP16) VFX_ORACLE_LAUNCH(__half);
  else if (cond_op && precision == VFX_PREC_TF32) VFX_ORACLE_LAUNCH(tf32_t);
  else VFX_ORACLE_LAUNCH(float);
#undef VFX_ORACLE_LAUNCH
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

}  // namespace vfx

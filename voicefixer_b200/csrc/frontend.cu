// Framed real FFT (2048, hop 441, periodic Hann, reflect pad) -> magnitude -> 128-bin mel.
// Replaces the reference's DFT-matrix conv1d STFT (torchlibrosa STFT built at
// voicefixer/tools/modules/fDomainHelper.py:23-31, used by spectrogram_phase :81-86 with
// eps = 1e-8 from wav_to_spectrogram_phase :88) and MelScale.forward
// (voicefixer/tools/mel_scale.py:63-77), as called by VoiceFixer._pre voicefixer/base.py:78-85.
// The unused cos/sin phase outputs (SURVEY D8) are not computed.
#include "vfx_common.cuh"
#include "fft.cuh"

namespace vfx {

namespace {

__global__ void __launch_bounds__(256) stft_mel_kernel(const float* __restrict__ wav, int L, int T,
                                                       const int* __restrict__ ext_len, const int* __restrict__ ext_frames,
                                                       const float* __restrict__ window,
                                                       const float2* __restrict__ tw,
                                                       const float* __restrict__ fbT,
                                                       const int* __restrict__ fb_start,
                                                       const int* __restrict__ fb_len,
                                                       float* __restrict__ mel, float* __restrict__ sp) {
  __shared__ float2 bufA[1024], bufB[1024];
  __shared__ float mag[1025];
  const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const float* x = wav + (long long)b * L;
  // ragged batch: item b has its own length Lb <= L (the row stride) and frames t < 1 + Lb / 441; it is reflected at Lb
  const int Lb = ext_len ? ext_len[b] : L;
  if (ext_frames && t >= ext_frames[b]) return;
  const int base = t * 441 - 1024;
  // z[n] = xw[2n] + i*xw[2n+1], reflect padding at both ends (F.pad(..., mode='reflect'))
  for (int n = tid; n < 1024; n += 256) {
    float v[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int i = base + 2 * n + h;
      if (i < 0) i = -i;
      if (i >= Lb) i = 2 * (Lb - 1) - i;
      v[h] = x[i] * window[2 * n + h];
    }
    bufA[n] = make_float2(v[0], v[1]);
  }
  __syncthreads();
  const float2* Z = fft1024(bufA, bufB, tw, tid);
  // untangle the packed real transform, magnitude with the reference's clamp (eps 1e-8)
  for (int k = tid; k <= 1024; k += 256) {
    const float2 X = rfft_untangle(Z, tw, k);
    const float m = sqrtf(fmaxf(X.x * X.x + X.y * X.y, 1e-8f));
    mag[k] = m;
    if (sp) sp[((long long)b * T + t) * 1025 + k] = m;
  }
  __syncthreads();
  if (tid < 128) {
    const int s = fb_start[tid], n = fb_len[tid];
    const float* f = fbT + (long long)tid * 1025 + s;
    float acc = 0.f;
    for (int j = 0; j < n; ++j) acc = fmaf(mag[s + j], f[j], acc);
    mel[((long long)b * T + t) * 128 + tid] = acc;
  }
}

}  // namespace

int stft_mel(const float* wav, int B, int L, int T, const int* ext_len, const int* ext_frames, const float* window,
             const float2* tw, const float* fbT, const int* fb_start, const int* fb_len, float* mel, float* sp,
             cudaStream_t st) {
  VFX_REQUIRE(L > 1024, "frontend: L=%d must exceed 1024 (reflect padding of n_fft/2)", L);
  VFX_REQUIRE(T == 1 + L / 441, "frontend: T=%d inconsistent with L=%d", T, L);
  dim3 grid(T, B);
  stft_mel_kernel<<<grid, 256, 0, st>>>(wav, L, T, ext_len, ext_frames, window, tw, fbT, fb_start, fb_len, mel, sp);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

}  // namespace vfx

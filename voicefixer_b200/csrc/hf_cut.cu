// Mode-1 pre-filter on the device: VoiceFixer.remove_higher_frequency (voicefixer/base.py:87-104)
// with librosa 0.10.1's (Dockerfile:9) stft/istft defaults restated: n_fft 2048, hop 512, periodic
// Hann, center=True with ZERO padding, istft length 512*(frames-1), window-sum-square normalised.
//   pass 1  per frame: rFFT -> S (kept), feature = max(log10(|S|+1e-8), 0) summed per bin
//   pass 2  per item : threshold = ratio * sum(energy); cut i = first bin where the running sum
//                      reaches it (loop semantics of base.py:96-99, bins >= i are zeroed)
//   pass 3  per frame: S' = |S| * S/(|S|+1e-8) for bins < i -> inverse rFFT -> * window
//   pass 4  per sample: overlap-add gather of the (<= 4) covering frames / window-sum-square
#include "vfx_common.cuh"
#include "fft.cuh"

namespace vfx {

namespace {

constexpr int NF = 2048, HOP = 512, NB = 1025;

// Per-item lengths (ragged batch, `lens` non-NULL): item b is L_b = clamp(lens[b], HOP, L) samples long in a row of L
// (= L_cap) samples and is processed as if it were alone: nfr_b = 1 + L_b / HOP frames, samples at or after L_b read as
// zero (librosa's constant padding at the item's own end), istft length out_len_b = HOP * (nfr_b - 1).
__device__ __forceinline__ int item_len(const int* lens, int b, int L) { return lens ? min(max(lens[b], HOP), L) : L; }

__global__ void __launch_bounds__(256) hf_fwd_kernel(const float* __restrict__ wav, int L, int nfr,
                                                     const int* __restrict__ lens,
                                                     const float* __restrict__ window,
                                                     const float2* __restrict__ tw, float2* __restrict__ S,
                                                     double* __restrict__ energy) {
  __shared__ float2 bufA[1024], bufB[1024];
  const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int Lb = item_len(lens, b, L);
  if (t >= 1 + Lb / HOP) return;                 // past the item's last frame: no spectrum, no energy
  const float* x = wav + (long long)b * L;
  const int base = t * HOP - NF / 2;
  for (int n = tid; n < 1024; n += 256) {
    float v[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i = base + 2 * n + h;
      v[h] = (i >= 0 && i < Lb) ? x[i] * window[2 * n + h] : 0.f;
    }
    bufA[n] = make_float2(v[0], v[1]);
  }
  __syncthreads();
  const float2* Z = fft1024(bufA, bufB, tw, tid);
  float2* Sp = S + ((long long)b * nfr + t) * NB;
  for (int k = tid; k <= 1024; k += 256) {
    const float2 X = rfft_untangle(Z, tw, k);
    Sp[k] = X;
    const float f = log10f(sqrtf(X.x * X.x + X.y * X.y) + 1e-8f);
    if (f > 0.f) atomicAdd(&energy[(long long)b * NB + k], (double)f);
  }
}

__global__ void hf_cut_index_kernel(const double* __restrict__ energy, float ratio, int* __restrict__ cut,
                                    const int* __restrict__ lens, int L, int* __restrict__ lens_out) {
  const int b = blockIdx.x;
  if (threadIdx.x != 0) return;
  if (lens_out) lens_out[b] = HOP * (item_len(lens, b, L) / HOP);      // the item's filtered length out_len_b
  const double* e = energy + (long long)b * NB;
  double total = 0.0;
  for (int k = 0; k < NB; ++k) total += e[k];
  const double thr = total * (double)ratio;
  double cur = e[0];
  int i = 0;
  // base.py:96-99 (the reference would raise IndexError at i == 1024; unreachable for ratio < 1)
  while (i < NB - 1 && cur < thr) { cur += e[i + 1]; ++i; }
  cut[b] = i;
}

__global__ void __launch_bounds__(256) hf_inv_kernel(const float2* __restrict__ S, int nfr, int L,
                                                     const int* __restrict__ lens,
                                                     const int* __restrict__ cut,
                                                     const float* __restrict__ window,
                                                     const float2* __restrict__ tw, float* __restrict__ frames) {
  __shared__ float2 X[NB];
  __shared__ float2 bufA[1024], bufB[1024];
  const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  if (t >= 1 + item_len(lens, b, L) / HOP) return;
  const float2* Sp = S + ((long long)b * nfr + t) * NB;
  const int ci = cut[b];
  for (int k = tid; k <= 1024; k += 256) {
    float2 v = make_float2(0.f, 0.f);
    if (k < ci) {
      const float2 s = Sp[k];
      const float mag = sqrtf(s.x * s.x + s.y * s.y);
      const float g = mag / (mag + 1e-8f);           // spec*cos + j*spec*sin, base.py:91,103
      v = make_float2(s.x * g, s.y * g);
    }
    X[k] = v;
  }
  __syncthreads();
  // pack the half spectrum back into the 1024-point complex transform of z[n] = x[2n] + i x[2n+1]:
  // Z[k] = E[k] + i O[k], E = (X[k] + conj X[1024-k])/2, O = conj(w^k) (X[k] - conj X[1024-k])/2;
  // inverse FFT through the forward routine: ifft(Z) = conj(fft(conj Z)) / 1024
  for (int k = tid; k < 1024; k += 256) {
    const float2 xk = X[k], xn = X[1024 - k];
    const float2 e = make_float2(0.5f * (xk.x + xn.x), 0.5f * (xk.y - xn.y));
    const float2 d = make_float2(0.5f * (xk.x - xn.x), 0.5f * (xk.y + xn.y));
    const float2 w = make_float2(tw[k].x, -tw[k].y);                    // exp(+2 pi i k / 2048)
    const float2 o = cmul(w, d);
    const float2 z = make_float2(e.x - o.y, e.y + o.x);                  // E + i O
    bufA[k] = make_float2(z.x, -z.y);                                    // conj
  }
  __syncthreads();
  const float2* zt = fft1024(bufA, bufB, tw, tid);
  float* fp = frames + ((long long)b * nfr + t) * NF;
  const float sc = 1.0f / 1024.0f;
  for (int n = tid; n < 1024; n += 256) {
    const float2 z = zt[n];
    fp[2 * n] = z.x * sc * window[2 * n];
    fp[2 * n + 1] = -z.y * sc * window[2 * n + 1];
  }
}

// out_len: row stride of `out` (HOP * (nfr - 1); L_cap on a ragged batch, whose item b fills out_len_b samples of its
// row from its own frames and zeros the rest)
__global__ void hf_ola_kernel(const float* __restrict__ frames, int nfr, int out_len, int L,
                              const int* __restrict__ lens, const float* __restrict__ window, float* __restrict__ out) {
  const int b = blockIdx.y;
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= out_len) return;
  const int nfr_b = lens ? 1 + item_len(lens, b, L) / HOP : nfr;
  if (n >= HOP * (nfr_b - 1)) { out[(long long)b * out_len + n] = 0.f; return; }
  const int p = n + NF / 2;                      // position in the un-trimmed overlap-add buffer
  const int t_hi = min(p / HOP, nfr_b - 1);
  const int t_lo = p >= NF ? (p - NF) / HOP + 1 : 0;   // first frame with p - t * HOP < NF (floor, not truncation)
  float acc = 0.f, wss = 0.f;
  for (int t = t_lo; t <= t_hi; ++t) {
    const int j = p - t * HOP;
    if (j >= 0 && j < NF) {
      acc += frames[((long long)b * nfr + t) * NF + j];
      const float w = window[j];
      wss += w * w;
    }
  }
  out[(long long)b * out_len + n] = wss > 1.17549435e-38f ? acc / wss : acc;
}

}  // namespace

size_t hf_cut_workspace(int B, int L) {
  const size_t nfr = 1 + (size_t)L / HOP;
  return (size_t)B * nfr * NB * sizeof(float2) + (size_t)B * nfr * NF * sizeof(float) + (size_t)B * NB * sizeof(double) +
         (size_t)B * 4 + 4096;
}

int hf_cut(const float* wav, int B, int L, const int* lens, float ratio, const float* window, const float2* tw, float* out,
           int* lens_out, int* cut_bins, void* ws, size_t ws_bytes, cudaStream_t st) {
  VFX_REQUIRE(wav && out && ws && B > 0 && L >= HOP, "hf_cut: bad arguments (L=%d)", L);
  const int nfr = 1 + L / HOP;
  const int out_len = lens ? L : HOP * (nfr - 1);
  if (ws_bytes < hf_cut_workspace(B, L)) {
    set_error("hf_cut: workspace too small: need %zu bytes", hf_cut_workspace(B, L));
    return VFX_ERR_WORKSPACE;
  }
  char* p = reinterpret_cast<char*>(ws);
  double* energy = reinterpret_cast<double*>(p); p += (((size_t)B * NB * sizeof(double)) + 255) & ~(size_t)255;
  float2* S = reinterpret_cast<float2*>(p); p += (((size_t)B * nfr * NB * sizeof(float2)) + 255) & ~(size_t)255;
  float* frames = reinterpret_cast<float*>(p); p += (((size_t)B * nfr * NF * sizeof(float)) + 255) & ~(size_t)255;
  int* cut = cut_bins ? cut_bins : reinterpret_cast<int*>(p);
  VFX_CUDA_CHECK(cudaMemsetAsync(energy, 0, (size_t)B * NB * sizeof(double), st));
  hf_fwd_kernel<<<dim3(nfr, B), 256, 0, st>>>(wav, L, nfr, lens, window, tw, S, energy);
  VFX_LAUNCH_CHECK();
  hf_cut_index_kernel<<<B, 32, 0, st>>>(energy, ratio, cut, lens, L, lens ? lens_out : nullptr);
  VFX_LAUNCH_CHECK();
  hf_inv_kernel<<<dim3(nfr, B), 256, 0, st>>>(S, nfr, L, lens, cut, window, tw, frames);
  VFX_LAUNCH_CHECK();
  hf_ola_kernel<<<dim3(ceil_div(out_len, 256), B), 256, 0, st>>>(frames, nfr, out_len, L, lens, window, out);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

}  // namespace vfx

// 1024-point complex FFT in shared memory + the packed real-FFT (2048) untangle helpers, in float2 (the restore front end
// and the mode-1 pre-filter) or double2 (Vocoder.oracle's front end, whose reference computes the FFT in float64).
#pragma once
#include <cuda_runtime.h>

namespace vfx {

static __device__ __forceinline__ float2 cplx(float x, float y) { return make_float2(x, y); }
static __device__ __forceinline__ double2 cplx(double x, double y) { return make_double2(x, y); }

template <typename C>
static __device__ __forceinline__ C cmul(C a, C b) {
  return cplx(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// In-place-in-shared-memory complex FFT of 1024 points (radix-2 Stockham autosort, 10 passes,
// 256 threads, two butterflies per thread per pass).  tw[i] = exp(-2*pi*i*I/2048), i < 1024.
// Returns the buffer holding the result.
template <typename C>
static __device__ __forceinline__ C* fft1024(C* a, C* b, const C* __restrict__ tw, int tid) {
  C* src = a; C* dst = b;
#pragma unroll 1
  for (int Ns = 1; Ns < 1024; Ns <<= 1) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int j = tid + q * 256;          // butterfly index 0..511
      const int k = j & (Ns - 1);
      const C w = tw[k * (1024 / Ns)];
      const C u = src[j];
      const C v = cmul(w, src[j + 512]);
      const int j0 = ((j - k) << 1) + k;
      dst[j0] = cplx(u.x + v.x, u.y + v.y);
      dst[j0 + Ns] = cplx(u.x - v.x, u.y - v.y);
    }
    __syncthreads();
    C* t = src; src = dst; dst = t;
  }
  return src;
}


// X[k], k in [0,1024], of the 2048-point real transform whose even/odd samples were packed as
// z[n] = x[2n] + i x[2n+1] and transformed into Z (1024 complex).  tw[k] = exp(-2 pi i k / 2048).
template <typename C>
static __device__ __forceinline__ C rfft_untangle(const C* Z, const C* __restrict__ tw, int k) {
  using R = decltype(C().x);
  if (k == 1024) return cplx(Z[0].x - Z[0].y, R(0));
  const C zk = Z[k], zn = Z[(1024 - k) & 1023];
  const C e = cplx(R(0.5) * (zk.x + zn.x), R(0.5) * (zk.y - zn.y));
  const C o = cplx(R(0.5) * (zk.y + zn.y), R(-0.5) * (zk.x - zn.x));   // -i/2 (zk - conj zn)
  const C wo = cmul(tw[k], o);
  return cplx(e.x + wo.x, e.y + wo.y);
}

}  // namespace vfx

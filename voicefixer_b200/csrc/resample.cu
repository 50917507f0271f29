// Polyphase sample-rate conversion to 44.1 kHz (vfx_resample, vfx_resample_src): scipy.signal.resample_poly(x, up, down)
// on float32 input, restated bit for bit, for a ragged batch of items of mixed rates.  The arithmetic contract
// (voicefixer_b200/resample.py): output j of an item's 44.1 kHz stream is
//   p = (j + rem) * down;  y[j] = sum over i = max(0, ceil((p - h_len + 1) / up)) .. min(n_in - 1, floor(p / up)),
//   ascending, of x[i] * h'[p - i * up]
// summed in float32 from 0 with a separate multiply and add per tap, as scipy's upfirdn loop does (a fused multiply-add
// changes about 40 % of the samples).  Every index is 64-bit: at 48 kHz, p passes 2^31 after about 304 s.
#include "vfx_common.cuh"

namespace vfx {

namespace {

// Where recording sample i of an item lives.  WindowSrc: a staged window, xw[i - first] (vfx_resample);
// StridedSrc: the caller's whole recording in place, src[i * stride] (vfx_resample_src).
struct WindowSrc {
  const float* xw; long long first;
  __device__ __forceinline__ float operator()(long long i) const { return __ldg(xw + (i - first)); }
};
struct StridedSrc {
  const float* src; long long stride;
  __device__ __forceinline__ float operator()(long long i) const { return __ldg(src + i * stride); }
};

// The body both kernels share: one thread per output sample j < L_cap of row b.  The 20 (16 / 48 kHz) to 44 (96 kHz)
// taps an output reads lie one `up` apart in h'; a ratio's taps (at most 36 KB at the common rates) stay in L1 and are
// read through the read-only path.
template <typename Item, typename Src>
__device__ __forceinline__ void resample_row(const Item& it, Src x, const float* __restrict__ h, int b, long long j,
                                             int L_cap, float* __restrict__ y, int* __restrict__ lens_out) {
  if (lens_out && j == 0) lens_out[b] = it.y_len;
  if (j >= L_cap) return;
  float acc = 0.f;
  if (j < it.y_len) {
    const long long J = it.y_first + j;                    // index in the item's 44.1 kHz stream
    if (it.up == 1 && it.down == 1) {
      acc = x(J);
    } else {
      const long long up = it.up;
      const long long p = (J + it.rem) * (long long)it.down;
      const long long num = p - it.h_len + 1;
      long long i = num <= 0 ? 0 : (num + up - 1) / up;
      const long long last = min(it.n_in - 1, p / up);
      const float* tap = h + it.h_off + (p - i * up);
      for (; i <= last; ++i, tap -= up) acc = __fadd_rn(acc, __fmul_rn(x(i), __ldg(tap)));
    }
  }
  y[(long long)b * L_cap + j] = acc;
}

__global__ void __launch_bounds__(256) resample_kernel(const float* __restrict__ x, const float* __restrict__ h,
                                                       const vfx_resample_item* __restrict__ items, int L_cap,
                                                       float* __restrict__ y, int* __restrict__ lens_out) {
  const int b = blockIdx.y;
  const vfx_resample_item it = items[b];
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  resample_row(it, WindowSrc{x + it.x_off, it.x_first}, h, b, j, L_cap, y, lens_out);
}

__global__ void __launch_bounds__(256) resample_src_kernel(const float* __restrict__ h,
                                                           const vfx_resample_src_item* __restrict__ items, int L_cap,
                                                           float* __restrict__ y, int* __restrict__ lens_out) {
  const int b = blockIdx.y;
  const vfx_resample_src_item it = items[b];
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  resample_row(it, StridedSrc{it.src, it.stride}, h, b, j, L_cap, y, lens_out);
}

}  // namespace

int resample(const float* x, const float* h, const vfx_resample_item* items, int B, int L_cap, float* y, int* lens_out,
             cudaStream_t st) {
  VFX_REQUIRE(items && y && B > 0 && B <= 65535 && L_cap > 0, "resample: bad arguments");
  dim3 grid((unsigned)ceil_div(L_cap, 256), B);
  resample_kernel<<<grid, 256, 0, st>>>(x, h, items, L_cap, y, lens_out);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int resample_src(const float* h, const vfx_resample_src_item* items, int B, int L_cap, float* y, int* lens_out,
                 cudaStream_t st) {
  VFX_REQUIRE(items && y && B > 0 && B <= 65535 && L_cap > 0, "resample_src: bad arguments");
  dim3 grid((unsigned)ceil_div(L_cap, 256), B);
  resample_src_kernel<<<grid, 256, 0, st>>>(h, items, L_cap, y, lens_out);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

}  // namespace vfx

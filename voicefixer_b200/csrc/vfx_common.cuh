// Shared declarations of the vfx_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include "../../include/vfx_b200.h"

namespace vfx {

void set_error(const char* fmt, ...);

#define VFX_CUDA_CHECK(expr)                                                          \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess) {                                                          \
      vfx::set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr,           \
                     cudaGetErrorString(_e));                                         \
      return VFX_ERR_CUDA;                                                            \
    }                                                                                 \
  } while (0)

extern unsigned long long g_launches;   // kernels launched by this library (bench.py's gpu_launches)
extern unsigned long long g_conv_tma_launches;   // those of them that were conv_gemm_tc launches fed by TMA
extern unsigned long long g_conv_tma_store_launches;   // ... and of those, the ones whose epilogue stored through TMA
#define VFX_LAUNCH_CHECK()                                                            \
  do { ++vfx::g_launches; VFX_CUDA_CHECK(cudaGetLastError()); } while (0)

#define VFX_REQUIRE(cond, ...)                                                        \
  do {                                                                                \
    if (!(cond)) {                                                                    \
      vfx::set_error(__VA_ARGS__);                                                    \
      return VFX_ERR_INVALID;                                                         \
    }                                                                                 \
  } while (0)

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// ------------------------------------------------------------------ device helpers
__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) {
  return __float2bfloat16_rn(v);
}
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }
// VFX_PREC_TF32 operand element: fp32 storage holding a value already rounded to tf32 (10-bit mantissa,
// round-to-nearest) by its producer, so that the tensor core's truncation of the low 13 bits is exact.
// (Un-rounded operands make the tf32 tensor core truncate: a CPU simulation of the whole path gave 1.4e-2 waveform
// rel-RMS with truncation against 1.7e-3 with round-to-nearest, tools/sim_precision.py.)
struct tf32_t { float v; };
__device__ __forceinline__ float round_tf32(float v) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
  return __uint_as_float(u);
}
__device__ __forceinline__ float to_f(tf32_t v) { return __uint_as_float(__float_as_uint(v.v) & 0xFFFFE000u); }   // as the tensor core reads it
template <> __device__ __forceinline__ tf32_t from_f<tf32_t>(float v) { return tf32_t{round_tf32(v)}; }

// Encoded tf32 stream (vfx_conv_desc.res_enc / raw_enc): S = bits(lrelu(x)) + 0x1000 -- see include/vfx_b200.h.
// (lrelu and its inverse as max / min with the scaled value: two instructions, the same result for 0 < slope < 1)
__device__ __forceinline__ float stream_enc(float x, float slope) {
  const float y = fmaxf(x, x * slope);
  return __uint_as_float(__float_as_uint(y) + 0x1000u);
}
__device__ __forceinline__ float stream_dec(float s, float inv_slope) {
  const float y = __uint_as_float(__float_as_uint(s) - 0x1000u);
  return fminf(y, y * inv_slope);
}

// element size of a GEMM operand / weight in the given vfx_precision
static inline size_t prec_esz(int precision) { return (precision == VFX_PREC_BF16 || precision == VFX_PREC_FP16) ? 2 : 4; }
// two fp32 -> one packed pair of 16-bit operands (bf16 or fp16), round-to-nearest
template <bool FP16> __device__ __forceinline__ uint32_t pack16(float lo, float hi) {
  if (FP16) { __half2 h = __floats2half2_rn(lo, hi); return *reinterpret_cast<uint32_t*>(&h); }
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

__device__ __forceinline__ float apply_act(float v, int act, float p) {
  switch (act) {
    case VFX_ACT_LRELU: return v > 0.f ? v : v * p;
    case VFX_ACT_ELU: return v > 0.f ? v : expm1f(v);
    case VFX_ACT_LRELU_XSINX: {
      float u = v > 0.f ? v : v * p;
      return u + sinf(u);
    }
    case VFX_ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    default: return v;
  }
}

// ------------------------------------------------------------------ kernels (host launchers)
int conv_gemm_simt(int precision, const vfx_conv_desc& d, cudaStream_t st);
int resstack_pair(const vfx_pair_desc& d, cudaStream_t st);        // ResStack pair, fused or blocked form (vfx_pair_desc.form)
size_t resstack_pair_scratch_bytes();
// the pairs resstack_pair runs: bf16 / fp16 at C = 64 or 128 without stream encoding, tf32 at C = 64 on the encoded stream
bool pair_supported(int prec, int C, bool stream_enc);
int conv_gemm_tc(int precision, const vfx_conv_desc& d, cudaStream_t st);   // wgmma: bf16 / fp16 (f16 kinds) or tf32

// y = act(scale[b][c]*x + shift[b][c]); x fp32 [B][P][C] (row pitch ldx), y operand type.
// bn_C == 1: single-channel BN (scale[b][0]).  stat_sB: element stride between items (0 = shared).
int bn_act(int precision, const float* x, long long x_sB, long long ldx, int B, long long P, int C,
           const float* scale, const float* shift, int bn_C, int stat_sB, int act, float act_param,
           void* y, long long y_sB, long long ldy, cudaStream_t st);
// per-item biased batch statistics -> scale/shift [B][C] (train-mode BN, eps 1e-5)
// acc: scratch of 2*B*bn_C doubles.  seq (ragged batch, NULL = all P positions): item b's statistics cover its first
// min(seq[b] * per_row, P) positions only (per_row = W of a [B][H][W][C] map, 1 for a [B][T][C] plane).
int bn_stats(const float* x, long long x_sB, long long ldx, int B, long long P, int C, int bn_C,
             const float* gamma, const float* beta, float* scale, float* shift, double* acc,
             const int* seq, int per_row, cudaStream_t st);
int dropout_apply(float* x, const uint8_t* keep, long long n, cudaStream_t st);
// seeded dropout in place on x fp32 [B][T][512] at denoiser dropout `layer` (0 or 1), item b keyed by keys[b] (device)
int dropout_seeded(float* x, int B, int T, const vfx_drop_key* keys, int layer, cudaStream_t st);
int avgpool2x2(const float* x, long long x_sB, long long x_sH, long long x_sW, int B, int H, int W,
               int C, float* y, cudaStream_t st);
// Ragged batches: the kernels below that take `ext_*` / `lens` pointers (device int32 [B], NULL = every item spans the
// whole tensor) read each item's own extent at that stage from the table ragged_extents() fills.
enum {
  EXT_SAMPLES = 0,          // L_b
  EXT_FRAMES = 1,           // T_b = 1 + L_b / 441
  EXT_UNET0 = 2,            // EXT_UNET0 + k, k = 0..6: Tp_b >> k, Tp_b = 64 * ceil(T_b / 64)
  EXT_COND = 9,             // Tc_b = T_b + T_b % 2 + 4
  EXT_COND_PAD = 10,        // Tc_b + 6 (reflect-padded condnet output)
  EXT_UP0 = 11,             // EXT_UP0 + j, j = 0..3: up-sampler j's output length Tc_b * (7, 49, 147, 441)
  EXT_LEVELS = 15
};
// lens[B] -> ext[EXT_LEVELS][B]; every length is clamped into [1025, L_cap] first
int ragged_extents(const int* lens, int B, int L_cap, int* ext, cudaStream_t st);
// the same table for the vocoder alone, from mel frame counts frames[B] (clamped into [1, T_cap]): samples = S_b =
// Tc_b * 441 (the untrimmed generated length), frames = T_b, the conditioning and up-sampler rows as above
int frame_extents(const int* frames, int B, int T_cap, int* ext, cudaStream_t st);
// Vocoder.oracle's front end (oracle_fe.cu).  wav[B][L_cap], item b = its first L_b = clamp(lens[b], 1, L_cap) samples
// (lens NULL: L_cap each); peak_bits: B uint32 of workspace; frames (optional) receives T_b = 1 + L_b / 441.
// Writes the normalised conditions [B][Tc_cap][128] in the operand format `precision` to cond_op and / or in fp32 to
// cond_f32 (either may be NULL): rows T_b .. Tc_b - 1 are -4; rows from Tc_b on are -4 in cond_op and 0 in cond_f32.
// basis / b_start / b_len: the Slaney HTK mel basis [128][1025] fp32 and its band of non-zero bins per row.
int oracle_frontend(const float* wav, int B, int L_cap, const int* lens, const float* basis, const int* b_start,
                    const int* b_len, unsigned int* peak_bits, int* frames, void* cond_op, int precision, float* cond_f32,
                    cudaStream_t st);
int stft_mel(const float* wav, int B, int L, int T, const int* ext_len, const int* ext_frames, const float* window,
             const float2* tw, const float* fbT, const int* fb_start, const int* fb_len, float* mel, float* sp,
             cudaStream_t st);
int gru_layer(const float* gi, const float* whh_t, const float* bhh, int B, int T, const int* lens, float* out,
              cudaStream_t st);
// denoiser tail: clean = sigmoid(lin)*mel ; x = log10(clip(clean)); unet_in[b][t][f<127][2]
// (zero rows for ext_frames[b] <= t < Tp)
int mask_log_pack(const float* lin_sig, const float* mel, int B, int T, int Tp, const int* ext_frames, float* xlog,
                  float* unet_in, cudaStream_t st);
// unet head: out[b][t][f] = (f<127 ? bias + sum_c w[c]*x[b][t][f][c] : 0) + xlog[b][t][f]
int unet_head(const float* x, int B, int T, int Tp, const float* w, const float* bias,
              const float* xlog, float* out, cudaStream_t st);
// vocoder conditions: (from_log) / weight, dB, normalise, tail pad of -4 -> cond [B][Tc][128]
// tab = mel_weight[128] ++ [min_level] (fp32, computed by the host exactly as the reference does)
// (ragged: frames t < ext_frames[b] are converted, the rest of the rows is the -4 tail)
int voc_normalize(const float* mel, int B, int T, int Tc, const int* ext_frames, int input_is_log, const float* tab,
                  void* cond, int precision, cudaStream_t st);
int cast_rows(const float* x, long long n, void* y, int precision, cudaStream_t st);
// rows [0,3) and [3+L, L+6) of a [B][L+6][C] operand buffer <- reflection of the interior (ragged: L_b = ext_len[b])
int reflect_pad3(void* buf, int B, int L, int C, const int* ext_len, int precision, cudaStream_t st);
// final conv: lrelu0.2 -> reflect pad 3 -> conv k7 (64->1) -> tanh -> trim -> *scale
// ragged (ext_gen, ext_len non-NULL): item b reflects at S_b = ext_gen[b], trims to L_b = ext_len[b] centred
// (lo_b = (S_b - L_b) / 2) and writes zeros from L_b to out_len
int voc_post(const float* x, int B, int L, const float* w, const float* bias, int lo, int out_len,
             const int* ext_gen, const int* ext_len, float scale, float* out, cudaStream_t st);
// lens (ragged batch, NULL = every item has L samples): L is the capacity and the row stride of wav and out; item b is
// filtered as if alone with clamp(lens[b], 512, L) samples, out holds its 512 * (L_b / 512) samples and zeros after, and
// lens_out[b] (optional) receives that length
int hf_cut(const float* wav, int B, int L, const int* lens, float ratio, const float* window, const float2* tw,
           float* out, int* lens_out, int* cut_bins, void* ws, size_t ws_bytes, cudaStream_t st);
size_t hf_cut_workspace(int B, int L);
// polyphase rate conversion (resample.cu): row b of y[B][L_cap] <- items[b]'s output samples (items: the device copy of
// a table vfx_resample has validated), then zeros; lens_out[b] (optional) <- y_len
int resample(const float* x, const float* h, const vfx_resample_item* items, int B, int L_cap, float* y, int* lens_out,
             cudaStream_t st);
// the same arithmetic on items that read their recordings in place (vfx_resample_src)
int resample_src(const float* h, const vfx_resample_src_item* items, int B, int L_cap, float* y, int* lens_out,
                 cudaStream_t st);
// row b of x[B][ldx] -> items[b]'s destination (items: the device copy of a table vfx_scatter_rows has validated);
// max_len: the longest item
int scatter_rows(const float* x, int B, long long ldx, const vfx_scatter_item* items, int max_len, cudaStream_t st);
// vfx_pack_pcm16's two launches (items: the device copy of a table vfx_pack_pcm16 has validated; vmax[B]: scratch for
// the per-file maxima); max_n: the most frames (n) of any item
int pack_pcm16(const vfx_pcm16_item* items, int B, long long max_n, unsigned* vmax, short* y, cudaStream_t st);

}  // namespace vfx

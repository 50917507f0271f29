// HBM-bound elementwise / reduction kernels of the path (all channels-last).
#include "vfx_common.cuh"
#include "philox.cuh"

namespace vfx {

namespace {

// ------------------------------------------------------------------ bn_act
// y = act(scale*x + shift).  Reference: F.leaky_relu_(bn(x)) voicefixer/restorer/modules.py:70-71,
// F.relu_(bn1(x)) modules.py:150, BatchNorm2d(1)/ReLU members of the denoiser restorer/model.py:69-99.
template <typename T>
__global__ void bn_act_kernel(const float* __restrict__ x, long long x_sB, long long ldx, int B,
                              long long P, int C, const float* __restrict__ scale,
                              const float* __restrict__ shift, int bn_C, int stat_sB, int act,
                              float act_param, T* __restrict__ y, long long y_sB, long long ldy) {
  const int C4 = C >> 2;
  const long long total = (long long)B * P * C4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    const long long r = i / C4;
    const long long p = r % P;
    const int b = (int)(r / P);
    const float4 v = *reinterpret_cast<const float4*>(x + b * x_sB + p * ldx + c);
    float in[4] = {v.x, v.y, v.z, v.w}, o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int sc = b * stat_sB + (bn_C == 1 ? 0 : c + j);
      const float s = scale ? scale[sc] : 1.f, t = shift ? shift[sc] : 0.f;
      o[j] = apply_act(fmaf(in[j], s, t), act, act_param);
    }
    T* yp = y + b * y_sB + p * ldy + c;
#pragma unroll
    for (int j = 0; j < 4; ++j) yp[j] = from_f<T>(o[j]);
  }
}

template <typename T>
__global__ void bn_act_scalar_kernel(const float* __restrict__ x, long long x_sB, long long ldx, int B,
                                     long long P, int C, const float* __restrict__ scale,
                                     const float* __restrict__ shift, int bn_C, int stat_sB, int act,
                                     float act_param, T* __restrict__ y, long long y_sB, long long ldy) {
  const long long total = (long long)B * P * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long r = i / C;
    const long long p = r % P;
    const int b = (int)(r / P);
    const int sc = b * stat_sB + (bn_C == 1 ? 0 : c);
    const float s = scale ? scale[sc] : 1.f, t = shift ? shift[sc] : 0.f;
    y[b * y_sB + p * ldy + c] = from_f<T>(apply_act(fmaf(x[b * x_sB + p * ldx + c], s, t), act, act_param));
  }
}

// ------------------------------------------------------------------ bn_stats (mode 2)
// Biased batch statistics per item (reference batch is 1: SURVEY D5), F.batch_norm training=True.
// Ragged batch (seq non-NULL): item b's positions are its first seq[b] * per_row; the blocks past them exit, and the
// blocks inside see exactly the rows (and row partition) they would see on the item alone.
__device__ __forceinline__ long long stat_positions(const int* seq, int per_row, int b, long long P) {
  return seq ? min(P, (long long)seq[b] * per_row) : P;
}

__global__ void bn_stats_accum_kernel(const float* __restrict__ x, long long x_sB, long long ldx,
                                      long long P, int C, int bn_C, long long rows_per_block,
                                      const int* __restrict__ seq, int per_row,
                                      double* __restrict__ acc /*[B][bn_C][2]*/) {
  const int b = blockIdx.z;
  const int c = blockIdx.y * 32 + threadIdx.x;
  const long long Pb = stat_positions(seq, per_row, b, P);
  const long long p0 = (long long)blockIdx.x * rows_per_block;
  if (p0 >= Pb) return;                          // uniform over the block
  const long long p1 = min(Pb, p0 + rows_per_block);
  double s = 0.0, s2 = 0.0;
  if (c < C) {
    const float* xp = x + b * x_sB + c;
    for (long long p = p0 + threadIdx.y; p < p1; p += blockDim.y) {
      const float v = xp[p * ldx];
      s += v; s2 += (double)v * v;
    }
  }
  __shared__ double sh[2][8][33];
  sh[0][threadIdx.y][threadIdx.x] = s;
  sh[1][threadIdx.y][threadIdx.x] = s2;
  __syncthreads();
  if (threadIdx.y == 0) {
    for (int j = 1; j < 8; ++j) { s += sh[0][j][threadIdx.x]; s2 += sh[1][j][threadIdx.x]; }
    if (bn_C == 1) {
      for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_down_sync(0xffffffffu, s, o);
        s2 += __shfl_down_sync(0xffffffffu, s2, o);
      }
      if (threadIdx.x == 0) { atomicAdd(&acc[(long long)b * 2], s); atomicAdd(&acc[(long long)b * 2 + 1], s2); }
    } else if (c < C) {
      atomicAdd(&acc[((long long)b * C + c) * 2], s);
      atomicAdd(&acc[((long long)b * C + c) * 2 + 1], s2);
    }
  }
}

// count: values per statistic, positions x C for the single-channel (bn_C == 1) norms, positions otherwise
__global__ void bn_stats_final_kernel(const double* __restrict__ acc, int B, int bn_C, long long P, int C,
                                      const int* __restrict__ seq, int per_row,
                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                      float* __restrict__ scale, float* __restrict__ shift) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * bn_C) return;
  const int c = i % bn_C;
  const long long Pb = stat_positions(seq, per_row, i / bn_C, P);
  const double count = bn_C == 1 ? (double)Pb * C : (double)Pb;
  const double mean = acc[2 * i] / count;
  double var = acc[2 * i + 1] / count - mean * mean;
  if (var < 0) var = 0;
  const float inv = (float)(1.0 / sqrt(var + 1e-5));
  const float s = gamma[c] * inv;
  scale[i] = s;
  shift[i] = beta[c] - (float)mean * s;
}

__global__ void dropout_kernel(float* __restrict__ x, const uint8_t* __restrict__ keep, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    x[i] = keep[i] ? x[i] * 2.0f : 0.f;     // nn.Dropout(0.5): scale 1/(1-p)
}

// Seeded dropout (DESIGN.md §3): the keep bit of unit j of frame t of item b at `layer` is bit (j % 32) of word
// (j % 128) / 32 of Philox4x32-10(counter (t, 4 layer + j / 128, stream lo, stream hi), key (seed lo, seed hi)),
// (seed, stream) = keys[b].  One warp per frame row of 512 units: lane l serves 128-unit group g = l / 8 and computes its
// Philox call (8 lanes share one); for word i it takes units 128 g + 32 i + 4 (l % 8) .. + 3, i.e. bits 4 (l % 8) .. + 3,
// as one 16-byte access, so each warp access covers four whole 128-byte lines.  Rows t >= T_b are treated like the
// others: nothing reads them.
constexpr int DROP_ROWS = 8;                 // frame rows (warps) per block

__global__ void __launch_bounds__(32 * DROP_ROWS) dropout_seeded_kernel(float* __restrict__ x, int T,
                                                                        const vfx_drop_key* __restrict__ keys,
                                                                        int layer) {
  const int b = blockIdx.y;
  const int t = blockIdx.x * DROP_ROWS + (threadIdx.x >> 5);
  if (t >= T) return;
  const int lane = threadIdx.x & 31, g = lane >> 3, s = lane & 7;
  const unsigned long long seed = keys[b].seed, stream = keys[b].stream;
  const philox4 r = philox4x32_10((uint32_t)t, (uint32_t)(4 * layer + g), (uint32_t)stream, (uint32_t)(stream >> 32),
                                  (uint32_t)seed, (uint32_t)(seed >> 32));
  float4* p = reinterpret_cast<float4*>(x + ((long long)b * T + t) * 512 + 128 * g + 4 * s);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t bits = r.w[i] >> (4 * s);
    float4 v = p[8 * i];
    v.x = (bits & 1u) ? v.x * 2.0f : 0.f;
    v.y = (bits & 2u) ? v.y * 2.0f : 0.f;
    v.z = (bits & 4u) ? v.z * 2.0f : 0.f;
    v.w = (bits & 8u) ? v.w * 2.0f : 0.f;
    p[8 * i] = v;
  }
}

// F.avg_pool2d(x, (2,2)) voicefixer/restorer/modules.py:103 (floor: odd last column dropped)
__global__ void avgpool_kernel(const float* __restrict__ x, long long x_sB, long long x_sH,
                               long long x_sW, int B, int Ho, int Wo, int C, float* __restrict__ y) {
  const int C4 = C >> 2;
  const long long total = (long long)B * Ho * Wo * C4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    long long r = i / C4;
    const int w = (int)(r % Wo); r /= Wo;
    const int h = (int)(r % Ho);
    const int b = (int)(r / Ho);
    const float* p = x + b * x_sB + (2LL * h) * x_sH + (2LL * w) * x_sW + c;
    const float4 a = *reinterpret_cast<const float4*>(p), bq = *reinterpret_cast<const float4*>(p + x_sW);
    const float4 cq = *reinterpret_cast<const float4*>(p + x_sH),
                 dq = *reinterpret_cast<const float4*>(p + x_sH + x_sW);
    float4 o;
    o.x = (a.x + bq.x + cq.x + dq.x) * 0.25f; o.y = (a.y + bq.y + cq.y + dq.y) * 0.25f;
    o.z = (a.z + bq.z + cq.z + dq.z) * 0.25f; o.w = (a.w + bq.w + cq.w + dq.w) * 0.25f;
    *reinterpret_cast<float4*>(y + (((long long)b * Ho + h) * Wo + w) * C + c) = o;
  }
}

// restorer Generator.forward voicefixer/restorer/model.py:105-109 + UNet input pad/crop
// restorer/model_kqq_bn.py:144-151: clean = sigmoid(lin)*mel; x = to_log(clean);
// unet_in[b][t][f][0..1] = (to_log(mel), x) for f < 127, zero rows for T <= t < Tp.
__global__ void mask_log_pack_kernel(const float* __restrict__ lin, const float* __restrict__ mel,
                                     int B, int T, int Tp, const int* __restrict__ ext_frames,
                                     float* __restrict__ xlog, float* __restrict__ unet_in) {
  const long long total = (long long)B * Tp * 128;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int f = (int)(i & 127);
    const long long r = i >> 7;
    const int t = (int)(r % Tp);
    const int b = (int)(r / Tp);
    float lm = 0.f, lx = 0.f;
    if (t < (ext_frames ? ext_frames[b] : T)) {
      const long long src = ((long long)b * T + t) * 128 + f;
      const float m = mel[src];
      const float s = 1.f / (1.f + expf(-lin[src]));
      lx = log10f(fmaxf(s * m, 1e-8f));
      lm = log10f(fmaxf(m, 1e-8f));
      xlog[src] = lx;
    }
    if (f < 127) {
      float2 o; o.x = lm; o.y = lx;
      *reinterpret_cast<float2*>(unet_in + (((long long)b * Tp + t) * 127 + f) * 2) = o;
    }
  }
}

// after_conv2 (1x1, 32->1, bias) + F.pad(0,1) + crop + residual: restorer/model_kqq_bn.py:174-178,
// restorer/model.py:113.
__global__ void unet_head_kernel(const float* __restrict__ x, int B, int T, int Tp,
                                 const float* __restrict__ w, const float* __restrict__ bias,
                                 const float* __restrict__ xlog, float* __restrict__ out) {
  const long long total = (long long)B * T * 128;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int f = (int)(i & 127);
    const long long r = i >> 7;
    const int t = (int)(r % T);
    const int b = (int)(r / T);
    float v = 0.f;
    if (f < 127) {
      const float4* xp = reinterpret_cast<const float4*>(x + (((long long)b * Tp + t) * 127 + f) * 32);
      v = bias[0];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 a = xp[q];
        v = fmaf(a.x, w[4 * q], v); v = fmaf(a.y, w[4 * q + 1], v);
        v = fmaf(a.z, w[4 * q + 2], v); v = fmaf(a.w, w[4 * q + 3], v);
      }
    }
    out[i] = v + xlog[i];
  }
}

// from_log tools/pytorch_util.py:25-27; Vocoder.forward vocoder/base.py:51-54; tr_amp_to_db,
// tr_normalize, tr_pre vocoder/model/util.py:8-36,69-80.  tab = mel_weight[128] ++ [min_level].
template <typename T>
__global__ void voc_normalize_kernel(const float* __restrict__ mel, int B, int Tn, int Tc,
                                     const int* __restrict__ ext_frames, int input_is_log, const float* __restrict__ tab,
                                     T* __restrict__ cond) {
  const long long total = (long long)B * Tc * 128;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i & 127);
    const long long r = i >> 7;
    const int t = (int)(r % Tc);
    const int b = (int)(r / Tc);
    float c = -4.0f;
    if (t < (ext_frames ? ext_frames[b] : Tn)) {
      float v = mel[((long long)b * Tn + t) * 128 + k];
      if (input_is_log) v = exp10f(fminf(v, 5.0f));
      v = v / tab[k];
      const float S = 20.0f * log10f(fmaxf(tab[128], fabsf(v))) - 20.0f;
      c = fminf(fmaxf(8.0f * ((S + 115.0f) / 115.0f) - 4.0f, -4.0f), 4.0f);
    }
    cond[i] = from_f<T>(c);
  }
}

template <typename T>
__global__ void cast_kernel(const float* __restrict__ x, long long n, T* __restrict__ y) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    y[i] = from_f<T>(x[i]);
}

// nn.ReflectionPad1d(3) voicefixer/vocoder/model/generator.py:74,94 on a [B][L+6][C] buffer
template <typename T>
__global__ void reflect_pad3_kernel(T* __restrict__ buf, int B, int Lmax, int C, const int* __restrict__ ext_len) {
  const long long total = (long long)B * 6 * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int j = (int)((i / C) % 6);
    const int b = (int)(i / (6LL * C));
    T* base = buf + (long long)b * (Lmax + 6) * C;
    const int L = ext_len ? ext_len[b] : Lmax;    // ragged batch: the item's own length, padded at its own end
    const int dst = j < 3 ? j : L + j;            // rows 0,1,2 and L+3,L+4,L+5
    const int src = j < 3 ? 6 - j : L + 4 - j;    // x[3-j] at row 6-j ; x[L-2-(j-3)] at row L+4-j
    base[(long long)dst * C + c] = base[(long long)src * C + c];
  }
}

// generator[14..17]: LeakyReLU(0.2) -> ReflectionPad1d(3) -> Conv1d(64,1,7) -> Tanh
// (voicefixer/vocoder/model/generator.py:93-99) fused with _trim_center (voicefixer/base.py:63-76).
//
// A 64 -> 1 channel reduction over 7 taps: 448 MACs per output sample on a tensor that is read once (HBM-bound when done
// right).  16 lanes share an output: lane q owns channels [4q, 4q+4) and its 7 x 4 weights in registers; a group walks a
// run of 64 consecutive outputs, loading each input row ONCE as one coalesced 256-byte request (16 lanes x float4) and
// feeding it to the 7 outputs it contributes to (7 rotating accumulators, statically indexed by unrolling the row loop
// by 7); a finished output is summed across the 16 lanes by a 4-step butterfly.  No shared memory.  (The previous
// version staged rows in shared memory and issued two LDS per FMA: 2.0 ms for 3.6 GB = 28 % of HBM.)
constexpr int POST_RUN = 64;                 // outputs per 16-lane group (70 input rows = 10 x 7)
constexpr int POST_GROUPS = 16;              // groups per block (256 threads)

__device__ __forceinline__ float4 post_load_row(const float* __restrict__ xb, int t, int L, int q) {
  if (t < 0) t = -t;                         // ReflectionPad1d(3)
  if (t >= L) t = 2 * (L - 1) - t;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (t >= 0 && t < L) v = __ldcs(reinterpret_cast<const float4*>(xb + (long long)t * 64) + q);
  v.x = v.x > 0.f ? v.x : 0.2f * v.x; v.y = v.y > 0.f ? v.y : 0.2f * v.y;
  v.z = v.z > 0.f ? v.z : 0.2f * v.z; v.w = v.w > 0.f ? v.w : 0.2f * v.w;
  return v;
}

__global__ void __launch_bounds__(16 * POST_GROUPS) voc_post_kernel(const float* __restrict__ x, int Lmax,
                                                                     const float* __restrict__ w,
                                                                     const float* __restrict__ bias, int lo,
                                                                     int out_len, const int* __restrict__ ext_gen,
                                                                     const int* __restrict__ ext_len, float scale,
                                                                     float* __restrict__ out) {
  const int q = threadIdx.x & 15, g = threadIdx.x >> 4;
  const int b = blockIdx.y;
  const int o0 = (blockIdx.x * POST_GROUPS + g) * POST_RUN;       // first output of this group's run (may be >= out_len)
  const float* xb = x + (long long)b * Lmax * 64;
  // ragged batch: the item's generated length L and its own centred trim; outputs from `valid` to out_len are zeros
  const int L = ext_gen ? ext_gen[b] : Lmax;
  const int valid = ext_gen ? ext_len[b] : out_len;
  if (ext_gen) lo = (L - valid) / 2;
  float4 wk[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) wk[k] = *reinterpret_cast<const float4*>(w + k * 64 + 4 * q);
  const float bv = bias[0];
  float acc[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) acc[k] = 0.f;
  const int t0 = lo + o0 - 3;                                     // input position of row 0 of the run
  float4 cur[7], nxt[7];
#pragma unroll
  for (int j = 0; j < 7; ++j) cur[j] = post_load_row(xb, t0 + j, L, q);
  float res = 0.f;
#pragma unroll 1
  for (int it = 0; it < (POST_RUN + 6) / 7; ++it) {
    if (it + 1 < (POST_RUN + 6) / 7) {
#pragma unroll
      for (int j = 0; j < 7; ++j) nxt[j] = post_load_row(xb, t0 + 7 * (it + 1) + j, L, q);   // in flight during this block of rows
    }
#pragma unroll
    for (int j = 0; j < 7; ++j) {
      const float4 xv = cur[j];                                   // row r = 7 it + j feeds outputs r - k, k = 0..6
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        float a = acc[(j - k + 7) % 7];
        a = fmaf(xv.x, wk[k].x, a); a = fmaf(xv.y, wk[k].y, a); a = fmaf(xv.z, wk[k].z, a); a = fmaf(xv.w, wk[k].w, a);
        acc[(j - k + 7) % 7] = a;
      }
      // output o = r - 6 is complete: its slot is (j + 1) % 7
      float sum = acc[(j + 1) % 7];
      acc[(j + 1) % 7] = 0.f;
      sum += __shfl_xor_sync(0xffffffffu, sum, 8);
      sum += __shfl_xor_sync(0xffffffffu, sum, 4);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      const int o = 7 * it + j - 6;
      if ((o & 15) == q) res = sum;                               // lane q keeps outputs o = q (mod 16)
      if (o >= 0 && (o & 15) == 15) {                             // 16 outputs gathered: one coalesced 64-byte store
        const int oo = o0 + o - 15 + q;
        if (oo < out_len) out[(long long)b * out_len + oo] = oo < valid ? tanhf(res + bv) * scale : 0.f;
      }
    }
#pragma unroll
    for (int j = 0; j < 7; ++j) cur[j] = nxt[j];
  }
}

// Per-item extents of a ragged batch at every stage of restore() (vfx_common.cuh, EXT_*): the shapes each item would
// have if it were restored alone.  Lengths are clamped into [1025, L_cap] so that no kernel can leave the tensors.
__global__ void ragged_extents_kernel(const int* __restrict__ lens, int B, int L_cap, int* __restrict__ ext) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int L = min(max(lens[b], 1025), L_cap);
  const int T = 1 + L / 441;
  const int Tp = (T + 63) / 64 * 64;
  const int Tc = T + T % 2 + 4;
  ext[EXT_SAMPLES * B + b] = L;
  ext[EXT_FRAMES * B + b] = T;
  for (int k = 0; k < 7; ++k) ext[(EXT_UNET0 + k) * B + b] = Tp >> k;
  ext[EXT_COND * B + b] = Tc;
  ext[EXT_COND_PAD * B + b] = Tc + 6;
  ext[(EXT_UP0 + 0) * B + b] = Tc * 7;
  ext[(EXT_UP0 + 1) * B + b] = Tc * 49;
  ext[(EXT_UP0 + 2) * B + b] = Tc * 147;
  ext[(EXT_UP0 + 3) * B + b] = Tc * 441;
}

// The same table for the vocoder alone, from per-item mel frame counts (frames clamped into [1, T_cap]).  The samples
// row is the generated length S_b, so voc_post's centred trim is lo = 0 and item b's output is untrimmed, as
// Vocoder.forward returns it.  The UNet rows are unused by the vocoder; they hold the values restore() would use.
__global__ void frame_extents_kernel(const int* __restrict__ frames, int B, int T_cap, int* __restrict__ ext) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int T = min(max(frames[b], 1), T_cap);
  const int Tp = (T + 63) / 64 * 64;
  const int Tc = T + T % 2 + 4;
  ext[EXT_SAMPLES * B + b] = Tc * 441;
  ext[EXT_FRAMES * B + b] = T;
  for (int k = 0; k < 7; ++k) ext[(EXT_UNET0 + k) * B + b] = Tp >> k;
  ext[EXT_COND * B + b] = Tc;
  ext[EXT_COND_PAD * B + b] = Tc + 6;
  ext[(EXT_UP0 + 0) * B + b] = Tc * 7;
  ext[(EXT_UP0 + 1) * B + b] = Tc * 49;
  ext[(EXT_UP0 + 2) * B + b] = Tc * 147;
  ext[(EXT_UP0 + 3) * B + b] = Tc * 441;
}

// Row b of a (B, ldx) batch, from column src_off -> items[b].dst[dst_off, dst_off + len) (vfx_scatter_rows): one
// thread per sample.
__global__ void __launch_bounds__(256) scatter_rows_kernel(const float* __restrict__ x, long long ldx,
                                                           const vfx_scatter_item* __restrict__ items) {
  const int b = blockIdx.y;
  const vfx_scatter_item it = items[b];
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < it.len) it.dst[it.dst_off + j] = __ldg(x + (long long)b * ldx + it.src_off + j);
}

// vfx_pack_pcm16.  A float's key orders as the float does (NaN above +inf), so that one atomicMax per warp gives a
// file's np.max: the key of a NaN is the largest, and a NaN anywhere makes the maximum NaN.  Key 0 is below every float.
__device__ __forceinline__ unsigned pcm16_key(float v) {
  const unsigned u = __float_as_uint(v);
  return isnan(v) ? 0xFFFFFFFFu : (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// vmax[b] <- the key of file b's maximum over its n * C samples (vmax zeroed before); grid (x, B), frames grid-strided
__global__ void __launch_bounds__(256) pcm16_max_kernel(const vfx_pcm16_item* __restrict__ items,
                                                        unsigned* __restrict__ vmax) {
  const vfx_pcm16_item& it = items[blockIdx.y];
  unsigned m = 0;
  for (int c = 0; c < it.C; ++c)
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < it.n; t += (long long)gridDim.x * blockDim.x)
      m = max(m, pcm16_key(__ldg(it.rows[c] + t)));
  m = __reduce_max_sync(0xFFFFFFFFu, m);
  if ((threadIdx.x & 31) == 0 && m != 0) atomicMax(vmax + blockIdx.y, m);
}

// numpy's float32 -> int16 cast on x86: truncation toward zero to int32 (cvttss2si, whose out-of-range result
// 0x80000000 covers NaN and +-inf), then the low 16 bits.  cvt.rzi.s32.f32 saturates instead, so that range is explicit.
__device__ __forceinline__ short pcm16_of(float v) {
  if (!(v >= -2147483648.f && v < 2147483648.f)) return 0;
  return (short)(unsigned short)((unsigned)__float2int_rz(v) & 0xFFFFu);
}

// file b's interleaved y[dst_off + t * C + c] <- its rows[c][t], scaled by 32768 iff its maximum is <= 1
__global__ void __launch_bounds__(256) pcm16_pack_kernel(const vfx_pcm16_item* __restrict__ items,
                                                         const unsigned* __restrict__ vmax, short* __restrict__ y) {
  const vfx_pcm16_item& it = items[blockIdx.y];
  const bool scale = vmax[blockIdx.y] <= pcm16_key(1.0f);
  short* out = y + it.dst_off;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < it.n; t += (long long)gridDim.x * blockDim.x)
    for (int c = 0; c < it.C; ++c) {
      const float v = __ldg(it.rows[c] + t);
      out[t * it.C + c] = pcm16_of(scale ? v * 32768.f : v);
    }
}

inline int grid_for(long long total, int block = 256) {
  long long g = (total + block - 1) / block;
  if (g > 132LL * 32) g = 132LL * 32;      // 32 blocks per SM of an H100 SXM
  if (g < 1) g = 1;
  return (int)g;
}

inline bool valid_prec(int precision) { return precision >= VFX_PREC_FP32 && precision <= VFX_PREC_FP16; }
inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

// The launchers refuse a bad call before any launch: they also serve the C ABI's per-kernel test entry points, whose
// arguments come from outside the library.

int bn_act(int precision, const float* x, long long x_sB, long long ldx, int B, long long P, int C,
           const float* scale, const float* shift, int bn_C, int stat_sB, int act, float act_param,
           void* y, long long y_sB, long long ldy, cudaStream_t st) {
  VFX_REQUIRE(x && y && B > 0 && P > 0 && C > 0 && ldx >= C && ldy >= C && x_sB >= 0 && y_sB >= 0,
              "bn_act: bad arguments (B %d, P %lld, C %d, ldx %lld, ldy %lld)", B, P, C, ldx, ldy);
  VFX_REQUIRE((bn_C == 1 || bn_C == C) && stat_sB >= 0 && valid_prec(precision),
              "bn_act: bad statistics layout or precision (bn_C %d, C %d, stat_sB %d, precision %d)", bn_C, C, stat_sB,
              precision);
  const bool vec = (C % 4 == 0) && (ldx % 4 == 0) && (x_sB % 4 == 0) && ((uintptr_t)x % 16 == 0);
  const long long total = (long long)B * P * (vec ? C / 4 : C);
  const int g = grid_for(total);
#define VFX_BN_LAUNCH(K, T)                                                                      \
  K<T><<<g, 256, 0, st>>>(x, x_sB, ldx, B, P, C, scale, shift, bn_C, stat_sB, act, act_param,   \
                          reinterpret_cast<T*>(y), y_sB, ldy)
  if (precision == VFX_PREC_BF16) {
    if (vec) VFX_BN_LAUNCH(bn_act_kernel, __nv_bfloat16); else VFX_BN_LAUNCH(bn_act_scalar_kernel, __nv_bfloat16);
  } else if (precision == VFX_PREC_FP16) {
    if (vec) VFX_BN_LAUNCH(bn_act_kernel, __half); else VFX_BN_LAUNCH(bn_act_scalar_kernel, __half);
  } else if (precision == VFX_PREC_TF32) {
    if (vec) VFX_BN_LAUNCH(bn_act_kernel, tf32_t); else VFX_BN_LAUNCH(bn_act_scalar_kernel, tf32_t);
  } else {
    if (vec) VFX_BN_LAUNCH(bn_act_kernel, float); else VFX_BN_LAUNCH(bn_act_scalar_kernel, float);
  }
#undef VFX_BN_LAUNCH
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int bn_stats(const float* x, long long x_sB, long long ldx, int B, long long P, int C, int bn_C,
             const float* gamma, const float* beta, float* scale, float* shift, double* acc,
             const int* seq, int per_row, cudaStream_t st) {
  VFX_REQUIRE(x && gamma && beta && scale && shift && acc, "bn_stats: null pointer");
  VFX_REQUIRE(B > 0 && B <= 65535 && P > 0 && C > 0 && ldx >= C && x_sB >= 0 && (bn_C == 1 || bn_C == C),
              "bn_stats: bad shape (B %d, P %lld, C %d, bn_C %d, ldx %lld; B <= 65535)", B, P, C, bn_C, ldx);
  VFX_REQUIRE(!seq || per_row > 0, "bn_stats: per_row %d must be positive with seq", per_row);
  VFX_CUDA_CHECK(cudaMemsetAsync(acc, 0, sizeof(double) * 2 * B * bn_C, st));
  const long long rows_per_block = 256;
  dim3 grid(ceil_div(P, rows_per_block), ceil_div(C, 32), B), block(32, 8);
  bn_stats_accum_kernel<<<grid, block, 0, st>>>(x, x_sB, ldx, P, C, bn_C, rows_per_block, seq, per_row, acc);
  VFX_LAUNCH_CHECK();
  bn_stats_final_kernel<<<ceil_div(B * bn_C, 128), 128, 0, st>>>(acc, B, bn_C, P, C, seq, per_row, gamma, beta, scale,
                                                                  shift);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int dropout_apply(float* x, const uint8_t* keep, long long n, cudaStream_t st) {
  VFX_REQUIRE(x && keep && n > 0, "dropout_apply: bad arguments (n %lld)", n);
  dropout_kernel<<<grid_for(n), 256, 0, st>>>(x, keep, n);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int dropout_seeded(float* x, int B, int T, const vfx_drop_key* keys, int layer, cudaStream_t st) {
  VFX_REQUIRE(x && keys && B > 0 && B <= 65535 && T > 0 && (layer == 0 || layer == 1),
              "dropout_seeded: bad arguments (B %d, T %d, layer %d; B <= 65535, layer 0 or 1)", B, T, layer);
  VFX_REQUIRE(aligned16(x) && ((uintptr_t)keys & 7) == 0,
              "dropout_seeded: x must be 16-byte aligned and keys 8-byte aligned");
  dim3 grid(ceil_div(T, DROP_ROWS), B);
  dropout_seeded_kernel<<<grid, 32 * DROP_ROWS, 0, st>>>(x, T, keys, layer);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int avgpool2x2(const float* x, long long x_sB, long long x_sH, long long x_sW, int B, int H, int W,
               int C, float* y, cudaStream_t st) {
  VFX_REQUIRE(x && y && B > 0 && H > 0 && W > 0 && C > 0, "avgpool: bad arguments (B %d, H %d, W %d, C %d)", B, H, W, C);
  VFX_REQUIRE(aligned16(x) && aligned16(y), "avgpool: x and y must be 16-byte aligned");
  VFX_REQUIRE(C % 4 == 0 && x_sW % 4 == 0 && x_sH % 4 == 0 && x_sB % 4 == 0, "avgpool: C/strides must be multiples of 4");
  const int Ho = H / 2, Wo = W / 2;
  avgpool_kernel<<<grid_for((long long)B * Ho * Wo * C / 4), 256, 0, st>>>(x, x_sB, x_sH, x_sW, B, Ho, Wo, C, y);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int mask_log_pack(const float* lin, const float* mel, int B, int T, int Tp, const int* ext_frames, float* xlog,
                  float* unet_in, cudaStream_t st) {
  VFX_REQUIRE(lin && mel && xlog && unet_in && B > 0 && T > 0 && Tp >= T,
              "mask_log_pack: bad arguments (B %d, T %d, Tp %d)", B, T, Tp);
  VFX_REQUIRE(((uintptr_t)unet_in & 7) == 0, "mask_log_pack: unet_in must be 8-byte aligned");
  mask_log_pack_kernel<<<grid_for((long long)B * Tp * 128), 256, 0, st>>>(lin, mel, B, T, Tp, ext_frames, xlog, unet_in);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int unet_head(const float* x, int B, int T, int Tp, const float* w, const float* bias,
              const float* xlog, float* out, cudaStream_t st) {
  VFX_REQUIRE(x && w && bias && xlog && out && B > 0 && T > 0 && Tp >= T,
              "unet_head: bad arguments (B %d, T %d, Tp %d)", B, T, Tp);
  VFX_REQUIRE(aligned16(x), "unet_head: x must be 16-byte aligned");
  unet_head_kernel<<<grid_for((long long)B * T * 128), 256, 0, st>>>(x, B, T, Tp, w, bias, xlog, out);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int voc_normalize(const float* mel, int B, int T, int Tc, const int* ext_frames, int input_is_log, const float* tab,
                  void* cond, int precision, cudaStream_t st) {
  VFX_REQUIRE(mel && tab && cond && B > 0 && T > 0 && Tc > 0 && valid_prec(precision),
              "voc_normalize: bad arguments (B %d, T %d, Tc %d, precision %d)", B, T, Tc, precision);
  const int g = grid_for((long long)B * Tc * 128);
  if (precision == VFX_PREC_BF16)
    voc_normalize_kernel<__nv_bfloat16><<<g, 256, 0, st>>>(mel, B, T, Tc, ext_frames, input_is_log, tab,
                                                           reinterpret_cast<__nv_bfloat16*>(cond));
  else if (precision == VFX_PREC_FP16)
    voc_normalize_kernel<__half><<<g, 256, 0, st>>>(mel, B, T, Tc, ext_frames, input_is_log, tab, reinterpret_cast<__half*>(cond));
  else if (precision == VFX_PREC_TF32)
    voc_normalize_kernel<tf32_t><<<g, 256, 0, st>>>(mel, B, T, Tc, ext_frames, input_is_log, tab, reinterpret_cast<tf32_t*>(cond));
  else
    voc_normalize_kernel<float><<<g, 256, 0, st>>>(mel, B, T, Tc, ext_frames, input_is_log, tab,
                                                   reinterpret_cast<float*>(cond));
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int ragged_extents(const int* lens, int B, int L_cap, int* ext, cudaStream_t st) {
  VFX_REQUIRE(lens && ext && B > 0 && L_cap > 1024, "ragged_extents: bad arguments");
  ragged_extents_kernel<<<ceil_div(B, 128), 128, 0, st>>>(lens, B, L_cap, ext);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int frame_extents(const int* frames, int B, int T_cap, int* ext, cudaStream_t st) {
  VFX_REQUIRE(frames && ext && B > 0 && T_cap > 0, "frame_extents: bad arguments");
  frame_extents_kernel<<<ceil_div(B, 128), 128, 0, st>>>(frames, B, T_cap, ext);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int cast_rows(const float* x, long long n, void* y, int precision, cudaStream_t st) {
  VFX_REQUIRE(x && y && n > 0 && valid_prec(precision), "cast_rows: bad arguments (n %lld, precision %d)", n, precision);
  if (precision == VFX_PREC_BF16)
    cast_kernel<__nv_bfloat16><<<grid_for(n), 256, 0, st>>>(x, n, reinterpret_cast<__nv_bfloat16*>(y));
  else if (precision == VFX_PREC_FP16)
    cast_kernel<__half><<<grid_for(n), 256, 0, st>>>(x, n, reinterpret_cast<__half*>(y));
  else if (precision == VFX_PREC_TF32)
    cast_kernel<tf32_t><<<grid_for(n), 256, 0, st>>>(x, n, reinterpret_cast<tf32_t*>(y));
  else
    cast_kernel<float><<<grid_for(n), 256, 0, st>>>(x, n, reinterpret_cast<float*>(y));
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int reflect_pad3(void* buf, int B, int L, int C, const int* ext_len, int precision, cudaStream_t st) {
  VFX_REQUIRE(buf && B > 0 && C > 0 && valid_prec(precision), "reflect_pad3: bad arguments (B %d, C %d, precision %d)",
              B, C, precision);
  VFX_REQUIRE(L >= 4, "reflect_pad3: length %d too short for reflection pad 3", L);
  const int g = grid_for((long long)B * 6 * C);
  if (precision == VFX_PREC_BF16 || precision == VFX_PREC_FP16)      // a 2-byte copy either way
    reflect_pad3_kernel<__nv_bfloat16><<<g, 256, 0, st>>>(reinterpret_cast<__nv_bfloat16*>(buf), B, L, C, ext_len);
  else
    reflect_pad3_kernel<float><<<g, 256, 0, st>>>(reinterpret_cast<float*>(buf), B, L, C, ext_len);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int voc_post(const float* x, int B, int L, const float* w, const float* bias, int lo, int out_len,
             const int* ext_gen, const int* ext_len, float scale, float* out, cudaStream_t st) {
  VFX_REQUIRE(x && w && bias && out && B > 0 && B <= 65535 && L > 0 && out_len > 0,
              "voc_post: bad arguments (B %d, L %d, out_len %d; B <= 65535)", B, L, out_len);
  VFX_REQUIRE(!ext_gen == !ext_len, "voc_post: ext_gen and ext_len go together");
  VFX_REQUIRE(ext_gen || (lo >= 0 && (long long)lo + out_len <= L),
              "voc_post: trim [%d, %lld) outside the generated length %d", lo, (long long)lo + out_len, L);
  VFX_REQUIRE(((uintptr_t)x & 15) == 0 && ((uintptr_t)w & 15) == 0, "voc_post: x and w must be 16-byte aligned");
  dim3 grid(ceil_div(out_len, POST_RUN * POST_GROUPS), B);
  voc_post_kernel<<<grid, 16 * POST_GROUPS, 0, st>>>(x, L, w, bias, lo, out_len, ext_gen, ext_len, scale, out);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int scatter_rows(const float* x, int B, long long ldx, const vfx_scatter_item* items, int max_len, cudaStream_t st) {
  VFX_REQUIRE(x && items && B > 0 && B <= 65535 && max_len > 0 && max_len <= ldx,
              "scatter_rows: bad arguments (B %d, ldx %lld, max_len %d; B <= 65535)", B, ldx, max_len);
  dim3 grid(ceil_div(max_len, 256), B);
  scatter_rows_kernel<<<grid, 256, 0, st>>>(x, ldx, items);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

int pack_pcm16(const vfx_pcm16_item* items, int B, long long max_n, unsigned* vmax, short* y, cudaStream_t st) {
  VFX_REQUIRE(items && vmax && y && B > 0 && B <= 65535 && max_n > 0,
              "pack_pcm16: bad arguments (B %d, max_n %lld; B <= 65535)", B, max_n);
  VFX_CUDA_CHECK(cudaMemsetAsync(vmax, 0, sizeof(unsigned) * B, st));
  dim3 grid(ceil_div(std::min(max_n, 1024LL * 256), 256), B);
  pcm16_max_kernel<<<grid, 256, 0, st>>>(items, vmax);
  VFX_LAUNCH_CHECK();
  pcm16_pack_kernel<<<grid, 256, 0, st>>>(items, vmax, y);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

}  // namespace vfx

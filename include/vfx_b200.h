/* vfx_b200.h — C ABI of the H100-native VoiceFixer restore() hot path.
 *
 * The reference (haoheliu/voicefixer, pure Python/PyTorch) has no FFI; its boundary for this path
 * is five nn.Module.forward seams (SURVEY 8b).  Each entry point below replaces one of them and
 * cites it (paths relative to the reference checkout).  Conventions:
 *   - extern "C", plain pointers and sizes, no torch types; all data pointers are DEVICE pointers
 *     unless the name ends in _host; `stream` is a cudaStream_t passed as void*.
 *   - every function returns 0 (VFX_OK) or a negative vfx_status; vfx_last_error() gives the text.
 *   - no allocation inside compute calls: the caller passes a workspace obtained from
 *     vfx_workspace_bytes().  Weights are registered once by name (device pointers owned by caller).
 *   - tensors are fp32 unless stated; activations inside the engine are channels-last.
 */
#ifndef VFX_B200_H
#define VFX_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vfx_engine vfx_engine;

enum vfx_status {
  VFX_OK = 0,
  VFX_ERR_INVALID = -1,     /* bad argument / shape (mirrors the reference's AssertionError/ValueError) */
  VFX_ERR_MISSING_WEIGHT = -2,
  VFX_ERR_WORKSPACE = -3,   /* workspace too small */
  VFX_ERR_CUDA = -4,
  VFX_ERR_UNSUPPORTED = -5
};

/* Arithmetic of the convolution GEMMs.
 *   FP32: SIMT fp32 FMA (validation path, bit-for-bit deterministic).
 *   BF16: wgmma tensor-core MMA, bf16 operands and weights, fp32 accumulation.
 *   TF32: wgmma tensor-core MMA (tf32), fp32 storage with operands and weights rounded to tf32
 *         (round-to-nearest) by their producers, fp32 accumulation -- the arithmetic of the reference's own
 *         CUDA path (torch.backends.cudnn.allow_tf32 defaults to True; the reference's test/test.py:27-35
 *         compares that path with its CPU path).  Weights are registered in the FP32 layout.
 *   FP16: wgmma on fp16 operands and weights, fp32 accumulation: the SAME 10-bit mantissa as tf32 (so the same
 *         waveform parity) in 2-byte storage, i.e. the BF16 mode's memory traffic and kernels -- at fp16's exponent
 *         range (|x| < 65504; smaller than 6e-5 loses relative precision).  Everything outside the GEMM operands stays fp32. */
enum vfx_precision { VFX_PREC_FP32 = 0, VFX_PREC_BF16 = 1, VFX_PREC_TF32 = 2, VFX_PREC_FP16 = 3 };

/* restore() modes, voicefixer/base.py:110-115. mode 1's pre-filter is vfx_hf_cut(). */
enum vfx_mode { VFX_MODE_EVAL = 0, VFX_MODE_TRAIN_BN = 2 };

/* Seeded dropout key of one item (vfx_restore_seeded, vfx_analysis_seeded, vfx_dropout_seeded; DESIGN.md §3).  Mode 2's
 * keep bit of unit j in [0, 512) of frame t at dropout layer l (0: after dn.lin4, restorer/model.py:75; 1: after
 * dn.lin11, model.py:94) is bit j % 32 of word (j % 128) / 32 of Philox4x32-10 with counter (t, 4 l + j / 128,
 * stream & 0xffffffff, stream >> 32) and key (seed & 0xffffffff, seed >> 32); kept units are doubled, the others zeroed.
 * The mask is a pure function of the key and the position: no mask tensor exists.  16 bytes, 8-byte aligned. */
typedef struct vfx_drop_key {
  unsigned long long seed, stream;
} vfx_drop_key;

const char* vfx_last_error(void);
int vfx_version(void);

/* ---- engine lifetime ------------------------------------------------------------------ */
/* device >= 0: an engine on that sm_90a device.  device == -1: a planning-only engine that makes no
 * CUDA call -- vfx_engine_set_tensor / vfx_engine_finalize validate a weight set (names and byte sizes)
 * and vfx_workspace_bytes* size the workspace on a host without a GPU; every launching entry point
 * refuses it with VFX_ERR_INVALID. */
int vfx_engine_create(vfx_engine** out, int device, int precision);
int vfx_engine_destroy(vfx_engine* e);

/* Register one weight tensor (device pointer stays owned by the caller; `bytes` is checked
 * against what the engine expects when it is first used).  Names and layouts: DESIGN.md §3.
 * Replaces torch.load + load_state_dict: voicefixer/base.py:15-30, voicefixer/vocoder/base.py:24-32. */
int vfx_engine_set_tensor(vfx_engine* e, const char* name, const void* dev_ptr, size_t bytes);
/* Engine options: "use_tc" (BF16 / FP16 / TF32; 1 = wgmma kernel [default], 0 = SIMT cross-check on the same operands),
 * "profile" (0/1/2, see vfx_profile_report; 2 = one tag per shape / dilation),
 * "tf32_stream" (TF32: vocoder residual streams as one encoded tensor, vfx_conv_desc.res_enc / raw_enc, default 1),
 * "fuse_pairs" (1 [default] = every ResStack pair vfx_resstack_pair supports runs as one fused kernel, 0 = every pair as
 *  its two convolutions; the switch that compares the fused kernel against the two-launch path). */
int vfx_engine_set_option(vfx_engine* e, const char* key, int value);
/* Number of CUDA kernels this library has launched in this process (bench.py's gpu_launches). */
unsigned long long vfx_launch_count(void);
/* How many of them were tensor-core convolutions whose operands were staged by TMA (launches without per-item extents
 * whose operands a tensor map can express, DESIGN.md §4.1); the others were staged with cp.async. */
unsigned long long vfx_conv_tma_launch_count(void);
/* How many of those TMA-fed launches also loaded their residual and stored their outputs through tensor maps (the
 * others -- a residual or output base not 16-byte aligned, or a stride not a multiple of 16 bytes -- ran the row-loop
 * epilogue, DESIGN.md §4.1). */
unsigned long long vfx_conv_tma_store_launch_count(void);
/* With option "profile" = 1 every launch group is bracketed by CUDA events on the call's stream;
 * this synchronises, writes one line per tag "tag count total_ms flops bytes" and clears the log. */
int vfx_profile_report(vfx_engine* e, char* buf, size_t cap);
/* Resolve every name the engine needs; returns VFX_ERR_MISSING_WEIGHT and lists them otherwise.
 * Two weight sets are complete: analysis + vocoder (VoiceFixer, voicefixer/base.py:11-30), or the
 * vocoder alone -- nothing but "voc." tensors registered, all present (the reference's stand-alone
 * Vocoder class, voicefixer/vocoder/base.py:10-40).  On a vocoder-only engine vfx_frontend_mel,
 * vfx_analysis and vfx_restore return VFX_ERR_INVALID and vfx_workspace_bytes returns 0. */
int vfx_engine_finalize(vfx_engine* e);

/* Bytes of workspace needed by vfx_restore()/vfx_analysis()/vfx_vocoder() for a batch of B
 * segments of L samples each (T = 1 + L/441 frames). */
size_t vfx_workspace_bytes(const vfx_engine* e, int B, int L);
size_t vfx_workspace_bytes_frames(const vfx_engine* e, int B, int T);

/* ---- the five seams -------------------------------------------------------------------- */

/* wav[B][L] -> mel[B][T][128], T = 1 + L/441 (requires L > 1024: reflect pad).
 * Replaces FDomainHelper.wav_to_spectrogram_phase (voicefixer/tools/modules/fDomainHelper.py:88-110,
 * torchlibrosa STFT n_fft 2048 / hop 441 / periodic Hann / reflect) + MelScale.forward
 * (voicefixer/tools/mel_scale.py:63-77) as called from VoiceFixer._pre (voicefixer/base.py:78-85).
 * sp_out (optional, may be NULL): magnitude spectrogram [B][T][1025]. */
int vfx_frontend_mel(vfx_engine* e, const float* wav, int B, int L, float* mel, float* sp_out,
                     void* stream);

/* mel[B][T][128] (linear) -> mel_log[B][T][128] (log10 domain).
 * Replaces restorer Generator.forward (voicefixer/restorer/model.py:103-120): denoiser
 * (:69-99), to_log (tools/pytorch_util.py:18-22), UNetResComplex_100Mb.forward
 * (restorer/model_kqq_bn.py:130-181).  mode: vfx_mode.  drop_masks (mode 2 only, may be NULL =
 * no dropout): two keep-masks uint8 [2][B][T][512] for the Dropout(0.5)s at model.py:75,94. */
int vfx_analysis(vfx_engine* e, const float* mel, int B, int T, int mode,
                 const uint8_t* drop_masks, float* mel_log_out, void* workspace,
                 size_t workspace_bytes, void* stream);
/* vfx_analysis in mode 2 with seeded dropout: item b's masks come from keys[b] (device, B of them; vfx_drop_key)
 * instead of a mask tensor.  Bit-identical to vfx_analysis(mode 2) with the masks the keys define.  B <= 65535; same
 * workspace as vfx_analysis. */
int vfx_analysis_seeded(vfx_engine* e, const float* mel, int B, int T, const vfx_drop_key* keys, float* mel_log_out,
                        void* workspace, size_t workspace_bytes, void* stream);

/* mel[B][T][128] -> wav[B][out_len].
 * Replaces Vocoder.forward (voicefixer/vocoder/base.py:42-56: de-weight, dB, normalise, tr_pre)
 * + vocoder Generator.forward (voicefixer/vocoder/model/generator.py:127-145).
 * input_is_log != 0: input is the analysis stage's log10 mel and from_log
 * (tools/pytorch_util.py:25-27) is applied first.  The generator emits S = (T + T%2 + 4)*441
 * samples; trim_len < 0: write all S (out_len = S); else _trim_center (voicefixer/base.py:63-76)
 * to trim_len samples (out_len = trim_len).  scale multiplies the output (oracle(): 2^15). */
int vfx_vocoder(vfx_engine* e, const float* mel, int B, int T, int input_is_log, float* wav_out,
                int trim_len, float scale, void* workspace, size_t workspace_bytes, void* stream);

/* Vocoder Generator alone on normalised conditions cond[B][Tc][128] (channels-last view of the
 * reference's (B,128,Tc)) -> wav[B][Tc*441]*scale.  Used by Vocoder.oracle (vocoder/base.py:74-77). */
int vfx_vocoder_cond(vfx_engine* e, const float* cond, int B, int Tc, float* wav_out, int trim_len,
                     float scale, void* workspace, size_t workspace_bytes, void* stream);

/* vfx_vocoder (trim_len = -1) for B mels of DIFFERENT lengths, Vocoder.forward (voicefixer/vocoder/base.py:42-56) item by
 * item: mel[B][T_cap][128] holds item b in its first frames[b] rows (device int32, clamped into [1, T_cap]; the other rows
 * are never read).  wav_out[B][Tc_cap*441], Tc_cap = T_cap + T_cap%2 + 4: row b is bit-identical to vfx_vocoder on item b
 * alone, its (T_b + T_b%2 + 4)*441 samples untrimmed, followed by zeros.  A small kernel turns frames into per-item extents
 * that the kernels read on the device, so one captured graph of shape (B, T_cap) serves any lengths.
 * Workspace: vfx_workspace_bytes_frames(e, B, T_cap). */
int vfx_vocoder_ragged(vfx_engine* e, const float* mel, int B, int T_cap, const int* frames, int input_is_log,
                       float* wav_out, float scale, void* workspace, size_t workspace_bytes, void* stream);

/* Front end of Vocoder.oracle (voicefixer/vocoder/base.py:61-73; the counterpart of vfx_frontend_mel) on the device:
 * wav[B][L_cap] holds item b in its first lens[b] samples (device int32, clamped into [1, L_cap]; lens NULL = every item
 * is L_cap long).  Per item: peak-normalise (wav / max|wav|, IEEE division), |STFT| (n_fft 2048, hop 441, periodic Hann,
 * center with librosa 0.10's zero padding, no clamp), the Slaney-normalised HTK mel basis, 20 log10(max(1e-5, mel)) - 20,
 * normalise and clip to [-4, 4], and pre()'s -4 tail.  cond_out: fp32 [B][Tc_cap][128], Tc_cap = T_cap + T_cap%2 + 4,
 * T_cap = 1 + L_cap/441; item b fills rows < Tc_b (rows T_b .. Tc_b - 1 are -4, T_b = 1 + L_b/441) and zeros after.
 * An all-zero item divides by a zero peak, as the reference does.  Workspace: 4*B bytes (the per-item peaks). */
int vfx_oracle_cond(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, float* cond_out, void* workspace,
                    size_t workspace_bytes, void* stream);

/* Vocoder.oracle (voicefixer/vocoder/base.py:58-77) up to the file write: the front end of vfx_oracle_cond into the
 * workspace in the operand format, then the Generator on the frame-based extents.  wav_out[B][Tc_cap*441]: row b holds
 * item b's (T_b + T_b%2 + 4)*441 samples times scale (oracle(): 2^15), then zeros; bit-identical to the same call on
 * item b alone (B = 1, L_cap = L_b). */
int vfx_oracle(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, float scale, float* wav_out,
               void* workspace, size_t workspace_bytes, void* stream);
/* Workspace of vfx_oracle for (B, L_cap): the vfx_oracle pass run dry (works on a planning-only
 * engine); 0 for B <= 0 or L_cap <= 0. */
size_t vfx_oracle_workspace_bytes(const vfx_engine* e, int B, int L_cap);

/* Whole restore_inmem loop body (voicefixer/base.py:120-135) for B equal-length segments (vfx_restore_ragged below for
 * segments of different lengths):
 * wav[B][L] -> wav_out[B][L].  Equivalent to frontend -> analysis -> vocoder(trim_len = L). */
int vfx_restore(vfx_engine* e, const float* wav, int B, int L, int mode, const uint8_t* drop_masks,
                float* wav_out, void* workspace, size_t workspace_bytes, void* stream);

/* vfx_restore (mode 0; vfx_restore_ragged_mode below for mode 2) for B segments of DIFFERENT lengths: wav[B][L_cap] holds item b in its first lens[b] samples
 * (the rest is never read), lens[B] is a device int32 array.  wav_out[B][L_cap] receives item b's restoration in its
 * first lens[b] samples -- bit-identical to vfx_restore on that item alone -- and zeros after them.  A small kernel turns
 * lens into per-item extents at every stage (frames, UNet levels, vocoder rates) that the kernels read on the device, so
 * one launch sequence (or one captured CUDA graph) of shape (B, L_cap) serves any lengths; lengths are clamped into
 * [1025, L_cap].  Workspace: vfx_workspace_bytes(e, B, L_cap). */
int vfx_restore_ragged(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, float* wav_out,
                       void* workspace, size_t workspace_bytes, void* stream);

/* vfx_restore_ragged in either mode: vfx_restore_ragged is the mode-0 call (mode = VFX_MODE_EVAL, drop_masks = NULL).
 * mode VFX_MODE_TRAIN_BN: every train-mode BatchNorm takes item b's statistics over its own rows only (its T_b frames in
 * the denoiser, its Tp_b >> k rows of UNet level k), so row b is bit-identical to vfx_restore(mode 2) on item b alone
 * with the masks drop_masks[:, b, :T_b].  drop_masks (optional): keep-masks uint8 [2][B][T_cap][512], T_cap =
 * 1 + L_cap/441; rows t >= T_b are never read.  Precondition of mode 2 (the caller enforces it): every item has
 * 1 + lens[b]/441 > 64 frames, because the reference refuses a 1 x 1 UNet centre in train mode; an item that breaks it
 * gets finite, unspecified samples.  Workspace: vfx_workspace_bytes(e, B, L_cap). */
int vfx_restore_ragged_mode(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, int mode,
                            const uint8_t* drop_masks, float* wav_out, void* workspace, size_t workspace_bytes,
                            void* stream);

/* Mode 2 with seeded dropout: lens NULL = B equal-length segments (vfx_restore), else a ragged batch as
 * vfx_restore_ragged_mode, with its frame precondition.  Item b's masks come from keys[b] (device, B of them;
 * vfx_drop_key), so row b depends on item b's samples and key only: bit-identical to the same call on item b alone,
 * and to vfx_restore / vfx_restore_ragged_mode(mode 2) with the masks the keys define.  B <= 65535; same workspace as
 * vfx_restore. */
int vfx_restore_seeded(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, const vfx_drop_key* keys,
                       float* wav_out, void* workspace, size_t workspace_bytes, void* stream);

/* The analysis half of vfx_restore_ragged_mode / vfx_restore_seeded (the denoised mel that restore_inmem hands
 * your_vocoder_func, voicefixer/base.py:126-129, before from_log): wav[B][L_cap] holds item b in its first lens[b]
 * samples (device int32, required; clamped into [1025, L_cap]), L_cap > 1024.  The per-item extents of lens, the front
 * end and the analysis write mel_log_out[B][T_cap][128], T_cap = 1 + L_cap/441: its first T_b = 1 + L_b/441 rows of
 * item b are bit-identical to vfx_frontend_mel + vfx_analysis on item b alone; rows t >= T_b are unspecified.
 * mode: VFX_MODE_EVAL or VFX_MODE_TRAIN_BN (mode 1 is vfx_hf_cut_ragged first, then mode 0).  In mode 2 the dropout
 * comes from drop_masks (uint8 [2][B][T_cap][512], rows t >= T_b never read) or from keys (device, B of them, B <= 65535;
 * vfx_drop_key), never both, or neither (no dropout); keys are refused outside mode 2, masks are ignored in mode 0.
 * Precondition of mode 2 (the caller enforces it): every item has T_b > 64 frames, as for vfx_restore_ragged_mode.
 * Every argument is checked before the first launch.  Workspace: vfx_analysis_workspace_bytes(e, B, L_cap). */
int vfx_analysis_ragged(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, int mode,
                        const uint8_t* drop_masks, const vfx_drop_key* keys, float* mel_log_out,
                        void* workspace, size_t workspace_bytes, void* stream);
/* Workspace of vfx_analysis_ragged for (B, L_cap) in either mode: that call run dry in mode 2 (works on a planning-only
 * engine; at most vfx_workspace_bytes(e, B, L_cap), which also sizes the vocoder); 0 for B <= 0, L_cap <= 1024 (a
 * shape vfx_analysis_ragged refuses, as vfx_workspace_bytes does) or a vocoder-only engine. */
size_t vfx_analysis_workspace_bytes(const vfx_engine* e, int B, int L_cap);

/* mode 1 pre-filter, VoiceFixer.remove_higher_frequency (voicefixer/base.py:87-104) with the
 * librosa 0.10.1 stft/istft defaults (n_fft 2048, hop 512, Hann, center, zero pad):
 * wav[B][L] -> wav_out[B][512*(L/512)].  Returns the per-item cut bin in cut_bins[B] (optional).
 * Workspace: vfx_hf_cut_workspace_bytes(B, L). */
int vfx_hf_cut(vfx_engine* e, const float* wav, int B, int L, float ratio, float* wav_out,
               int* cut_bins, void* workspace, size_t workspace_bytes, void* stream);
/* Workspace of vfx_hf_cut for (B, L) and of vfx_hf_cut_ragged for (B, L_cap); needs no engine.  0 for a negative B or L. */
size_t vfx_hf_cut_workspace_bytes(int B, int L);

/* vfx_hf_cut for B items of DIFFERENT lengths: wav[B][L_cap] holds item b in its first lens[b] samples (device int32;
 * clamped into [512, L_cap]; the rest of the row is never read).  Item b is filtered as if it were alone: its own
 * 1 + L_b/512 frames set its cut bin, and wav_out[B][L_cap] receives its 512*(L_b/512) filtered samples followed by
 * zeros.  lens_out[B] (device int32, optional) receives those lengths, so the result can feed vfx_restore_ragged(_mode)
 * without a host round trip (mode 1 of a ragged batch).  Workspace: vfx_hf_cut_workspace_bytes(B, L_cap). */
int vfx_hf_cut_ragged(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, float ratio, float* wav_out,
                      int* lens_out, int* cut_bins, void* workspace, size_t workspace_bytes, void* stream);

/* ---- sample-rate conversion ------------------------------------------------------------ */

/* One item of vfx_resample: output samples [y_first, y_first + y_len) of one recording's 44.1 kHz stream, computed from
 * a window of its samples.  The recording has n_in samples; x[x_off .. x_off + x_len) holds its samples
 * [x_first, x_first + x_len).  up / down: 44100 / rate in lowest terms (1 / 1 = a copy).  h[h_off .. h_off + h_len) holds
 * the ratio's taps h', pre-padded with zeros and scaled by up, and rem is their output offset (a copy needs neither). */
typedef struct vfx_resample_item {
  long long x_off, x_first, n_in;
  long long y_first;
  long long h_off;
  int x_len, y_len;
  int up, down, rem, h_len;
} vfx_resample_item;

/* Resampling as librosa.load(path, sr=44100) does it in this project: scipy.signal.resample_poly(x, up, down) on float32
 * input (the host loader, wavio._resample), bit for bit, for B items of mixed rates in one launch.  Output j of an
 * item's stream is the sum, in float32 from 0 with a separate multiply and add per tap, over ascending inputs
 * i = max(0, ceil((p - h_len + 1) / up)) .. min(n_in - 1, floor(p / up)), p = (j + rem) * down, of x[i] * h'[p - i*up].
 * voicefixer_b200/resample.py builds the taps and the windows.
 * y[B][L_cap]: row b receives item b's y_len samples, then zeros.  lens_out[B] (device int32, optional) receives y_len,
 * ready for vfx_restore_ragged_mode / vfx_hf_cut_ragged / vfx_oracle.  items_host is a host array; the library
 * validates every item before any launch: up, down >= 1; the window lies inside x[0, x_elems) and inside the recording;
 * the taps lie inside h[0, h_elems); 0 <= y_len <= L_cap; the outputs lie inside the stream's ceil(n_in * up / down)
 * samples; and the window holds every input those outputs read.  A bad item returns VFX_ERR_INVALID naming it, and
 * nothing is launched or written.  The table is staged into the workspace: vfx_resample_workspace_bytes(B) bytes
 * (needs no engine; 0 for B <= 0).  B <= 65535. */
int vfx_resample(vfx_engine* e, const float* x, long long x_elems, const float* h, long long h_elems,
                 const vfx_resample_item* items_host, int B, float* y, int L_cap, int* lens_out,
                 void* workspace, size_t workspace_bytes, void* stream);
size_t vfx_resample_workspace_bytes(int B);

/* One item of vfx_resample_src: output samples [y_first, y_first + y_len) of one recording's 44.1 kHz stream, read
 * from the whole recording where it lies: its n_in samples are src[0], src[stride], ..., src[(n_in - 1) * stride]
 * (a device pointer; stride >= 1 elements, e.g. one channel of an interleaved tensor).  up, down, rem, h_off, h_len:
 * as in vfx_resample_item. */
typedef struct vfx_resample_src_item {
  const float* src;
  long long stride;
  long long n_in, y_first, h_off;
  int y_len, up, down, rem, h_len;
} vfx_resample_src_item;

/* vfx_resample with every item reading its recording in place (device-resident input: no staged windows).  Same
 * arithmetic, bit for bit, in the same kernel body; up = down = 1 is the copy that fills a row at 44.1 kHz, so one
 * launch builds the rows of a batch at every rate.  y[B][L_cap]: row b receives item b's y_len samples, then zeros;
 * lens_out[B] (device int32, optional) receives y_len.  The library validates every item before any launch: a non-null
 * src; 1 <= stride and (n_in - 1) * stride within 2^62; up, down >= 1; the taps lie inside h[0, h_elems) (a copy needs
 * none); 0 <= y_len <= L_cap; the outputs lie inside the stream's ceil(n_in * up / down) samples.  A bad item returns
 * VFX_ERR_INVALID naming it, and nothing is launched or written.  The table is staged into the workspace:
 * vfx_resample_src_workspace_bytes(B) bytes (needs no engine; 0 for B <= 0).  B <= 65535. */
int vfx_resample_src(vfx_engine* e, const float* h, long long h_elems, const vfx_resample_src_item* items_host, int B,
                     float* y, int L_cap, int* lens_out, void* workspace, size_t workspace_bytes, void* stream);
size_t vfx_resample_src_workspace_bytes(int B);

/* One item of vfx_scatter_rows: samples [src_off, src_off + len) of row b go to dst[dst_off, dst_off + len), dst a
 * device buffer of dst_elems floats.  src_off = 0 copies the row's first len samples (a zero-initialised item does);
 * a live stream's window gives only its kept span, which starts src_off samples into the row.  src_off sits in what
 * was the struct's tail padding: sizeof stays 32. */
typedef struct vfx_scatter_item {
  float* dst;
  long long dst_elems, dst_off;
  int len;
  int src_off;
} vfx_scatter_item;

/* Row b of x[B][ldx] (device) -> items_host[b]'s destination, one launch for the batch: the rows of a ragged batch back
 * into per-recording outputs (a restored segment at its offset in its recording, a generated waveform into its own
 * buffer, a window's kept span into a block of its own).  The library validates every item before any launch: a
 * non-null dst; 0 <= len <= ldx; 0 <= src_off and src_off + len <= ldx; 0 <= dst_off and dst_off + len <= dst_elems; and no two items' destination ranges overlap.  A bad item returns
 * VFX_ERR_INVALID naming it, and nothing is launched or written.  Items of length 0 write nothing (a table of them
 * launches nothing).  The table is staged into the workspace: vfx_scatter_rows_workspace_bytes(B) bytes (0 for B <= 0).
 * B <= 65535. */
int vfx_scatter_rows(const float* x, int B, long long ldx, const vfx_scatter_item* items_host, void* workspace,
                     size_t workspace_bytes, void* stream);
size_t vfx_scatter_rows_workspace_bytes(int B);

/* The most channels one file of vfx_pack_pcm16 may have (also the most a FLAC stream holds). */
#define VFX_PCM16_MAX_CHANNELS 8

/* One file of vfx_pack_pcm16: its C channels are the float32 device rows rows[0 .. C), n samples each; its interleaved
 * int16 samples [n][C] go to y[dst_off .. dst_off + n * C). */
typedef struct vfx_pcm16_item {
  const float* rows[VFX_PCM16_MAX_CHANNELS];
  long long n, dst_off;
  int C;
} vfx_pcm16_item;

/* 16-bit PCM of B files in two launches (a per-file maximum, then the packing), with the arithmetic of the host
 * quantiser (wavio.pcm16, tools/wav.py's save_wave) bit for bit: a file whose maximum over all its samples is <= 1 is
 * scaled by 32768 (a NaN anywhere makes the maximum NaN, and the file is not scaled); each value is truncated toward
 * zero to int32 and its low 16 bits kept, a value outside int32's range, +-inf and NaN giving 0 (what the x86 C cast
 * numpy uses gives).  y: a device buffer of y_elems int16.  The library validates every item before any launch: C in
 * [1, VFX_PCM16_MAX_CHANNELS]; rows[0 .. C) non-null; n >= 1; 0 <= dst_off and dst_off + n * C <= y_elems; and no two
 * items' destination ranges overlap.  A bad item returns VFX_ERR_INVALID naming it, and nothing is launched or
 * written.  The table and the per-file maxima are staged into the workspace: vfx_pack_pcm16_workspace_bytes(B) bytes
 * (0 for B <= 0).  B <= 65535. */
int vfx_pack_pcm16(const vfx_pcm16_item* items_host, int B, short* y, long long y_elems, void* workspace,
                   size_t workspace_bytes, void* stream);
size_t vfx_pack_pcm16_workspace_bytes(int B);

/* ---- per-kernel test entry points (tests/ call the kernels through these) --------------- */

/* Generic channels-last "shifted-window" convolution GEMM; the one kernel family behind every
 * Conv1d/Conv2d/ConvTranspose/Linear on the path.  See DESIGN.md §4 for the field semantics. */
typedef struct vfx_conv_desc {
  const void* a;            /* operand activations [B][H][W][Cin], element type per `precision` */
  int B, H, W, Cin;
  long long a_sB, a_sH, a_sW;   /* element strides (channels contiguous) */
  const void* w;            /* weights [*][N][Cin] K-major, element type per `precision` */
  int ntaps;
  int dh[9], dw[9];         /* input offset of each tap relative to the output grid position */
  long long w_off[9];       /* element offset of each tap's [N][Cin] matrix inside w */
  int Hq, Wq;               /* output grid (GEMM M = B*Hq*Wq) */
  int N;                    /* output channels of this GEMM */
  int sh, rh, sw, rw;       /* output coordinate = (qh*sh+rh, qw*sw+rw) (transposed-conv phases) */
  int OH, OW;               /* outputs outside [0,OH)x[0,OW) are dropped */
  float* out_raw;           /* fp32 result (+bias +residual), may be NULL */
  long long o_sB, o_sH, o_sW; int o_col;
  void* out_act;            /* act(result) as next operand (element type per precision), may be NULL */
  long long oa_sB, oa_sH, oa_sW; int oa_col;
  const float* bias; int bias_mod;          /* bias[n % bias_mod], NULL = none */
  const float* residual;    /* fp32, added before activation, NULL = none */
  long long r_sB, r_sH, r_sW; int r_col;
  int act;                  /* vfx_act applied to out_act */
  float act_param;          /* leaky slope */
  const float* act_scale;   /* optional per-channel affine before the activation of out_act:          */
  const float* act_shift;   /* out_act = act(result * act_scale[n] + act_shift[n]) (fused eval-mode BN) */
  /* TF32 "encoded stream" (vocoder ResStacks in VFX_PREC_TF32): ONE fp32 tensor S serves both as the next convolution's
   * tf32 operand and as the lossless carrier of the fp32 residual stream:  S = bits(lrelu(x, enc_slope)) + 0x1000.
   * The tf32 tensor core ignores the low 13 mantissa bits of an operand, so reading S as an operand yields exactly
   * round-to-nearest-tf32(lrelu(x)); subtracting 0x1000 from the bits and inverting the (bijective) leaky ReLU gives x back.
   * res_enc: `residual` holds S, it is decoded before the add.  raw_enc: `out_raw` receives S of the result. */
  int res_enc, raw_enc;
  float enc_slope;
  /* Per-item extents along one sequence axis (ragged batches, vfx_restore_ragged); NULL = the whole tensor.
   * seq_axis 0 = H (the UNet's [B][T][F][C]), 1 = W (the 1-D [B][1][L][C] layouts).  An input coordinate on that axis
   * >= seq_in[b] reads as zero (like one outside [0, H) x [0, W)); an output whose coordinate on that axis, in the
   * output space (q*s + r, the space of OH / OW), is >= seq_out[b] is not stored.  A 128-row tile whose rows all lie
   * beyond seq_out exits before its K loop. */
  const int* seq_in;
  const int* seq_out;
  int seq_axis;
} vfx_conv_desc;

enum vfx_act { VFX_ACT_NONE = 0, VFX_ACT_LRELU = 1, VFX_ACT_ELU = 2,
               VFX_ACT_LRELU_XSINX = 3 /* v = lrelu(x, p); v + sin v */, VFX_ACT_SIGMOID = 4 };

/* impl: 0 = SIMT, 1 = wgmma tensor cores (BF16, TF32 or FP16). */
int vfx_conv_gemm(int precision, int impl, const vfx_conv_desc* d, void* stream);

/* Fused ResStack pair on the wgmma tensor cores:
 *   x' = x + conv2_{k3,d=1}( lrelu_0.01( conv1_{k3,dilation}( a ) + b1 ) ) + b2
 * ResStack.forward voicefixer/vocoder/model/modules.py:592-595 (layers :550-576).
 * form: VFX_PAIR_FUSED = one persistent kernel (a CTA per SM walking blocks of rows), the intermediate h kept in shared
 * memory (no scratch); it needs a, w1, w2 16-byte aligned, x / x_out 8-byte aligned and out_act aligned to two elements
 * (VFX_ERR_UNSUPPORTED otherwise);
 * VFX_PAIR_BLOCKED = the two convolutions of vfx_conv_gemm per block of rows with h in `scratch` (required:
 * vfx_resstack_pair_scratch_bytes() bytes, 128-byte aligned), the reference the fused form is tested against.  Any other
 * form returns VFX_ERR_INVALID.
 *   VFX_PREC_BF16 / VFX_PREC_FP16, C = 64 or 128: a = lrelu_0.01(x) in the operand format [B][L][C]; x fp32 is read as the residual
 *     and, if write_raw, overwritten with x' (or written to x_out); out_act (optional, operand format, must not alias a) receives act(x').
 *   VFX_PREC_TF32, C = 64, stream_enc = 1: a == x == the encoded stream S (vfx_conv_desc.raw_enc), fp32 [B][L][C];
 *     the result goes to x_out (required, aliasing neither input) as S' (stream_enc_out = 1) or as plain x' (0).
 * w1 / w2: [3][C][C] in the operand format, tap-major.  Other precisions (VFX_PREC_FP32) and shapes return
 * VFX_ERR_UNSUPPORTED. */
enum vfx_pair_form { VFX_PAIR_FUSED = 0, VFX_PAIR_BLOCKED = 1 };
typedef struct vfx_pair_desc {
  const void* a;
  float* x;
  const void* w1; const float* b1; int dilation;
  const void* w2; const float* b2;
  int B, L, C;
  int write_raw;
  void* out_act; int act; float act_param;
  int precision;            /* vfx_precision: VFX_PREC_BF16, VFX_PREC_FP16 or VFX_PREC_TF32 */
  int form;                 /* vfx_pair_form; 0 (a zeroed descriptor) is the fused kernel */
  float* x_out;             /* NULL = in place over x (16-bit modes only) */
  int stream_enc, stream_enc_out;
  void* scratch;            /* VFX_PAIR_BLOCKED: device scratch of vfx_resstack_pair_scratch_bytes() bytes, 128-byte aligned: holds h */
  size_t scratch_bytes;
  const int* lens;          /* optional per-item length (<= L; L stays the item stride): rows >= lens[b] read as zero and are not
                             * written, as if item b had length lens[b].  NULL = every item has length L.  VFX_PAIR_BLOCKED
                             * refuses it with VFX_ERR_UNSUPPORTED. */
} vfx_pair_desc;
size_t vfx_resstack_pair_scratch_bytes(void);
int vfx_resstack_pair(const vfx_pair_desc* d, void* stream);

/* One direction-pair GRU layer recurrence: gi[B][T][2][768] (x W_ih^T + b_ih, fwd|bwd),
 * whh_t[2][256][768] (W_hh transposed), bhh[2][768] -> out[B][T][512] (fwd 256 | bwd 256).
 * torch.nn.GRU gate order r,z,n (voicefixer/restorer/model.py:35-42,61). */
int vfx_gru_layer(const float* gi, const float* whh_t, const float* bhh, int B, int T, float* out,
                  void* stream);
/* The same with a per-item sequence length lens[B] (device int32, 1 <= lens[b] <= T): item b's backward direction starts
 * at lens[b] - 1, as if the item were run alone with T = lens[b].  out[b][t] for t >= lens[b] is undefined. */
int vfx_gru_layer_ragged(const float* gi, const float* whh_t, const float* bhh, int B, int T, const int* lens,
                         float* out, void* stream);

/* The element-wise, batch-statistics and waveform-output kernels (elementwise.cu), each as the engine launches it.  A bad
 * call (null pointer, non-positive size, misaligned vector access, B beyond a grid dimension) returns VFX_ERR_INVALID
 * before any launch.  Per-item tables (seq, ext_*, lens, frames) are device int32 [B]; NULL = every item spans the tensor. */
/* Train-mode BatchNorm statistics, F.batch_norm(training=True) (restorer/modules.py:70, restorer/model.py:69-99): x fp32
 * [B][P][C] (pitch ldx) -> scale / shift [B][bn_C] = gamma / sqrt(var + 1e-5), beta - mean * scale; bn_C = 1 pools all
 * P x C values, bn_C = C is per channel; acc: caller scratch of 16 * B * bn_C bytes; seq: item b covers its first
 * min(seq[b] * per_row, P) positions.  B <= 65535. */
int vfx_bn_stats(const float* x, long long x_sB, long long ldx, int B, long long P, int C, int bn_C, const float* gamma,
                 const float* beta, float* scale, float* shift, double* acc, const int* seq, int per_row, void* stream);
/* y = act(x * scale + shift) in the operand format, F.leaky_relu_(bn(x)) (restorer/modules.py:70-71); scale / shift
 * [b * stat_sB + (bn_C == 1 ? 0 : c)], NULL = 1 / 0; columns >= C of y are not written. */
int vfx_bn_act(int precision, const float* x, long long x_sB, long long ldx, int B, long long P, int C,
               const float* scale, const float* shift, int bn_C, int stat_sB, int act, float act_param, void* y,
               long long y_sB, long long ldy, void* stream);
/* nn.Dropout(0.5) in train mode (restorer/model.py:75,94) in place: x[i] = keep[i] ? 2 x[i] : 0. */
int vfx_dropout_apply(float* x, const uint8_t* keep, long long n, void* stream);
/* Seeded dropout as the engine launches it in mode 2: x [B][T][512] in place (16-byte aligned), row b * T + t being
 * frame t of item b, keys[b] (device, 8-byte aligned) its vfx_drop_key, layer 0 or 1.  B <= 65535. */
int vfx_dropout_seeded(float* x, int B, int T, const vfx_drop_key* keys, int layer, void* stream);
/* F.avg_pool2d(x, (2, 2)) (restorer/modules.py:103): x [B][H][W][C] (element strides, multiples of 4; x and y 16-byte
 * aligned, C % 4 == 0) -> dense y [B][H/2][W/2][C]. */
int vfx_avgpool2x2(const float* x, long long x_sB, long long x_sH, long long x_sW, int B, int H, int W, int C, float* y,
                   void* stream);
/* Generator.forward's mask and to_log (restorer/model.py:105-109) + the UNet input pad (restorer/model_kqq_bn.py:144-151):
 * xlog[B][T][128] = log10(max(sigmoid(lin) mel, 1e-8)); unet_in[B][Tp][127][2] = (log10(max(mel, 1e-8)), xlog) for
 * t < T_b = ext_frames[b], zeros for T_b <= t < Tp. */
int vfx_mask_log_pack(const float* lin, const float* mel, int B, int T, int Tp, const int* ext_frames, float* xlog,
                      float* unet_in, void* stream);
/* after_conv2 (1x1, 32 -> 1) + F.pad + crop + residual (restorer/model_kqq_bn.py:174-178, restorer/model.py:113):
 * out[B][T][128] = (f < 127 ? bias + sum_c w[c] x[b][t][f][c] : 0) + xlog; x [B][Tp][127][32], 16-byte aligned. */
int vfx_unet_head(const float* x, int B, int T, int Tp, const float* w, const float* bias, const float* xlog, float* out,
                  void* stream);
/* Vocoder.forward's conditions (vocoder/base.py:51-54, vocoder/model/util.py:8-36,69-80): from_log (input_is_log),
 * / mel_weight, dB, normalise and clip to [-4, 4], pre()'s -4 tail: mel [B][T][128] -> cond [B][Tc][128] in the operand
 * format; tab = mel_weight[128] ++ [min_level]. */
int vfx_voc_normalize(const float* mel, int B, int T, int Tc, const int* ext_frames, int input_is_log, const float* tab,
                      void* cond, int precision, void* stream);
/* nn.ReflectionPad1d(3) (vocoder/model/generator.py:74,94) in place on buf [B][L + 6][C]: rows 0..2 and L_b + 3..L_b + 5
 * from the interior rows 3..L_b + 2 (L_b = ext_len[b], else L >= 4); 2-byte elements in bf16 / fp16, 4 otherwise. */
int vfx_reflect_pad3(void* buf, int B, int L, int C, const int* ext_len, int precision, void* stream);
/* generator[14..17] + _trim_center (vocoder/model/generator.py:93-99, base.py:63-76): x [B][L][64] fp32, w [7][64],
 * out[B][out_len] = tanh(conv1d(reflect_pad3(lrelu_0.2(x)), w) + bias)[lo + j] * scale; ext_gen / ext_len (both or
 * neither): item b has S_b = ext_gen[b] rows, lo_b = (S_b - L_b) / 2, L_b = ext_len[b], zeros from L_b on.  B <= 65535. */
int vfx_voc_post(const float* x, int B, int L, const float* w, const float* bias, int lo, int out_len, const int* ext_gen,
                 const int* ext_len, float scale, float* out, void* stream);
/* fp32 -> the operand format (bf16 / fp16 round to nearest even, tf32 ties away from zero) over n elements. */
int vfx_cast_rows(const float* x, long long n, void* y, int precision, void* stream);
/* The per-item extent table of a ragged restore (DESIGN.md §3): lens[B] clamped into [1025, L_cap] -> ext[15][B]. */
int vfx_ragged_extents(const int* lens, int B, int L_cap, int* ext, void* stream);
/* The same table for the vocoder alone (DESIGN.md §3): frames[B] clamped into [1, T_cap] -> ext[15][B]. */
int vfx_frame_extents(const int* frames, int B, int T_cap, int* ext, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VFX_B200_H */

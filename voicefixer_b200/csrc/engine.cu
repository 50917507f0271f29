// vfx_b200 engine: weight registry, workspace planning and the launch sequence of the restore()
// hot path behind the C ABI of include/vfx_b200.h.  One engine per process/GPU; all device memory
// (weights, workspace, inputs, outputs) is owned by the caller; only small constant tables (Hann window, FFT twiddles,
// the oracle's Slaney mel basis) are allocated here at create time.
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <mutex>
#include <unordered_map>
#include <vector>
#include "vfx_common.cuh"

namespace vfx {

static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

unsigned long long g_launches = 0;
unsigned long long g_conv_tma_launches = 0;
unsigned long long g_conv_tma_store_launches = 0;

struct Tensor { const void* p; size_t bytes; };

// per-tag CUDA-event timing of the launch sequence (option "profile")
struct ProfRec { std::string tag; cudaEvent_t a, b; double flops, bytes; };

}  // namespace vfx

enum { VFX_PART_ANALYSIS = 1, VFX_PART_VOCODER = 2 };   // analysis = front end + denoiser + UNet ("fe.", "dn.", "unet.")

struct vfx_engine {
  int device = 0;   // -1: planning-only engine (no CUDA calls; finalize and workspace queries only)
  int precision = VFX_PREC_FP32;
  bool finalized = false;
  int use_tc = 1;   // BF16 / FP16 / TF32: wgmma tensor-core kernel where the shape allows (0 = SIMT cross-check on the same operands)
  std::unordered_map<std::string, vfx::Tensor> tensors;
  float* d_window = nullptr;    // periodic Hann, 2048
  float2* d_tw = nullptr;       // exp(-2 pi i k / 2048), k < 1024
  float* d_obasis = nullptr;    // Vocoder.oracle's Slaney HTK mel basis [128][1025] (a constant, not a checkpoint weight)
  int* d_oband = nullptr;       // its band of non-zero bins per row: start[128] ++ len[128]
  std::vector<std::string> missing;
  int parts = 0;    // VFX_PART_* bits of the weight sets found complete by vfx_engine_finalize
  int tf32_stream = 1;  // TF32: vocoder residual streams are kept as ONE encoded fp32 tensor (operand + residual carrier)
  int fuse_pairs = 1;   // ResStack pairs that pair_supported() accepts run as ONE fused kernel (resstack_pair.cu)
  int profile = 0;
  std::vector<vfx::ProfRec> prof;
  std::string prof_report;
  size_t esz() const { return vfx::prec_esz(precision); }
  bool tensor_core() const { return precision != VFX_PREC_FP32; }   // operands are a tensor-core format (bf16 / tf32)
};

namespace vfx {

namespace {

constexpr int UNET_C[7] = {2, 32, 64, 128, 256, 384, 384};       // channels per level (0 = input)
constexpr int VOC_CIN[4] = {1024, 512, 256, 128};
constexpr int VOC_COUT[4] = {512, 256, 128, 64};
constexpr int VOC_U[4] = {7, 7, 3, 3};

// ------------------------------------------------------------------ workspace bump allocator
struct Bump {
  char* base; size_t cap; size_t off = 0; size_t peak = 0; bool overflow = false;
  Bump(void* b, size_t c) : base((char*)b), cap(c) {}
  void* raw(size_t bytes) {
    off = (off + 255) & ~(size_t)255;
    size_t o = off;
    off += bytes;
    if (off > peak) peak = off;
    if (base == nullptr) return (void*)(uintptr_t)(256 + o);   // dry run: fake non-null pointer
    if (off > cap) { overflow = true; return base; }
    return base + o;
  }
  template <typename T> T* alloc(size_t n) { return (T*)raw(n * sizeof(T)); }
  size_t mark() const { return off; }
  void reset(size_t m) { off = m; }
};

struct Ctx {
  vfx_engine* e; cudaStream_t st; Bump* ws; bool dry; int mode; int rc = VFX_OK;
  const int* ext = nullptr;   // ragged batch: per-item extents ext[EXT_LEVELS][B] on the device (NULL = equal lengths)
  int ext_B = 0;
  bool train() const { return mode == VFX_MODE_TRAIN_BN; }
  int prec() const { return e->precision; }
  const int* ext_at(int level) const { return ext ? ext + (size_t)level * ext_B : nullptr; }
};

// workspace of the ragged path's extent table (taken from the planner's slack, see dry_run)
size_t ext_table_bytes(int B) { return ((size_t)EXT_LEVELS * B * sizeof(int) + 255) & ~(size_t)255; }

// Sets a convolution's per-item extents (vfx_conv_desc.seq_in / seq_out; NULL on an equal-length batch)
void set_seq(vfx_conv_desc& d, const int* seq_in, const int* seq_out, int axis) {
  d.seq_in = seq_in; d.seq_out = seq_out; d.seq_axis = axis;
}

struct ProfScope {
  Ctx& c; bool on;
  ProfScope(Ctx& c_, const char* tag, double flops, double bytes) : c(c_), on(false) {
    if (c.dry || !c.e->profile) return;
    ProfRec r; r.tag = tag; r.flops = flops; r.bytes = bytes;
    if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return;
    cudaEventRecord(r.a, c.st);
    c.e->prof.push_back(r);
    on = true;
  }
  ~ProfScope() { if (on) cudaEventRecord(c.e->prof.back().b, c.st); }
};

double conv_flops(const vfx_conv_desc& d) {
  return 2.0 * d.B * d.Hq * d.Wq * (double)d.N * d.Cin * d.ntaps;
}
// algorithmic HBM bytes of one conv launch: the input tensor once (taps re-read from L2), fp32 residual in,
// fp32 raw out, operand out (weights are negligible and stay in L2)
double conv_bytes(const vfx_conv_desc& d, int prec) {
  const double esz = (double)prec_esz(prec);
  const double M = (double)d.B * d.Hq * d.Wq;
  return (double)d.B * d.H * d.W * d.Cin * esz + M * d.N * ((d.residual ? 4.0 : 0.0) + (d.out_raw ? 4.0 : 0.0) + (d.out_act ? esz : 0.0));
}

#define VFX_TRY(expr) do { int _r = (expr); if (_r != VFX_OK) return _r; } while (0)

const void* get(Ctx& c, const std::string& name, size_t bytes) {
  auto it = c.e->tensors.find(name);
  if (it == c.e->tensors.end()) {
    c.e->missing.push_back(name);
    set_error("weight tensor '%s' not registered", name.c_str());
    c.rc = VFX_ERR_MISSING_WEIGHT;
    return nullptr;
  }
  if (it->second.bytes != bytes) {
    set_error("weight tensor '%s' has %zu bytes, engine expects %zu", name.c_str(), it->second.bytes, bytes);
    c.rc = VFX_ERR_INVALID;
    return nullptr;
  }
  return it->second.p;
}
const float* getf(Ctx& c, const std::string& name, size_t n) { return (const float*)get(c, name, n * 4); }
const void* getw(Ctx& c, const std::string& name, size_t n, int prec) {
  return get(c, name, n * prec_esz(prec));
}

int run_conv(Ctx& c, int prec, const vfx_conv_desc& d, const char* tag = "conv") {
  if (c.dry) return VFX_OK;
  if (c.rc != VFX_OK) return c.rc;
  ProfScope ps(c, tag, conv_flops(d), conv_bytes(d, prec));
  if (prec != VFX_PREC_FP32 && c.e->use_tc) {
    int r = conv_gemm_tc(prec, d, c.st);
    if (r != VFX_ERR_UNSUPPORTED) return r;
  }
  return conv_gemm_simt(prec, d, c.st);
}

vfx_conv_desc conv_base(const void* a, int B, int H, int W, int Cin, const void* w, int N) {
  vfx_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.a = a; d.B = B; d.H = H; d.W = W; d.Cin = Cin;
  d.a_sW = Cin; d.a_sH = (long long)W * Cin; d.a_sB = (long long)H * W * Cin;
  d.w = w; d.N = N; d.Hq = H; d.Wq = W; d.sh = 1; d.sw = 1; d.OH = H; d.OW = W;
  d.bias_mod = N;
  return d;
}
void set_raw(vfx_conv_desc& d, float* p, long long ld, int col) {
  d.out_raw = p; d.o_sW = ld; d.o_sH = (long long)d.OW * ld; d.o_sB = (long long)d.OH * d.OW * ld; d.o_col = col;
}
void set_act(vfx_conv_desc& d, void* p, long long ld, int col, int act, float param) {
  d.out_act = p; d.oa_sW = ld; d.oa_sH = (long long)d.OW * ld; d.oa_sB = (long long)d.OH * d.OW * ld;
  d.oa_col = col; d.act = act; d.act_param = param;
}
void set_res(vfx_conv_desc& d, const float* p, long long ld, int col) {
  d.residual = p; d.r_sW = ld; d.r_sH = (long long)d.OW * ld; d.r_sB = (long long)d.OH * d.OW * ld; d.r_col = col;
}
void taps3x3(vfx_conv_desc& d, long long mat) {
  d.ntaps = 9;
  for (int kh = 0; kh < 3; ++kh)
    for (int kw = 0; kw < 3; ++kw) {
      int t = kh * 3 + kw;
      d.dh[t] = kh - 1; d.dw[t] = kw - 1; d.w_off[t] = (long long)t * mat;
    }
}

// ------------------------------------------------------------------ BN handling
struct BnRef { const float* scale; const float* shift; int stat_sB; };

// Eval: the folded running-stat affine registered by the host ("<name>.scale/.shift").
// Train (mode 2): per-item biased batch statistics of `x` (SURVEY D5/a19).  seq / per_row: the items' extents at this
// level (ragged batch; NULL = all P positions): item b's statistics cover its first seq[b] * per_row positions.
int bn_resolve(Ctx& c, const std::string& name, int bn_C, const float* x, long long x_sB, long long ldx,
               int B, long long P, int C, const int* seq, int per_row, BnRef* out) {
  if (!c.train()) {
    out->scale = getf(c, name + ".scale", bn_C);
    out->shift = getf(c, name + ".shift", bn_C);
    out->stat_sB = 0;
    return c.rc;
  }
  const float* gamma = getf(c, name + ".gamma", bn_C);
  const float* beta = getf(c, name + ".beta", bn_C);
  float* sc = c.ws->alloc<float>((size_t)B * bn_C);
  float* sh = c.ws->alloc<float>((size_t)B * bn_C);
  double* acc = c.ws->alloc<double>((size_t)2 * B * bn_C);
  out->scale = sc; out->shift = sh; out->stat_sB = bn_C;
  if (c.dry || c.rc != VFX_OK) return c.rc;
  return bn_stats(x, x_sB, ldx, B, P, C, bn_C, gamma, beta, sc, sh, acc, seq, per_row, c.st);
}

// operand = act(bn(x)); x raw fp32 [B][P][C] (pitch ldx) -> dense operand [B][P][C]
int bn_act_op(Ctx& c, int prec, const std::string& bn, int bn_C, const float* x, long long x_sB,
              long long ldx, int B, long long P, int C, const int* seq, int per_row, int act, float slope, void* y) {
  BnRef r;
  VFX_TRY(bn_resolve(c, bn, bn_C, x, x_sB, ldx, B, P, C, seq, per_row, &r));
  if (c.dry) return VFX_OK;
  ProfScope ps(c, "bn_act", 0.0, (double)B * P * C * (4 + prec_esz(prec)));
  return bn_act(prec, x, x_sB, ldx, B, P, C, r.scale, r.shift, bn_C, r.stat_sB, act, slope, y,
                (long long)P * C, C, c.st);
}

// ------------------------------------------------------------------ UNet
// ConvBlockRes.forward voicefixer/restorer/modules.py:68-76 on a channels-last raw tensor.
// in: raw fp32 [B][H][W][Cin] with pitch ld_in; out: raw fp32 with pitch ld_out (+col), may alias in.
struct BlockScratch { void* opA; float* rawH; void* opH; float* rawS; void* opX; };

// Eval-mode fusion hooks of a block (ignored in mode 2, which needs batch statistics between the ops):
//   opA_ready : s.opA already holds lrelu(bn1(in)) -- written by the previous conv's epilogue
//   next_bn   : BatchNorm whose eval affine + activation conv2's epilogue applies to produce the NEXT
//               consumer's operand in s.opA (next_slope: 0.01 LeakyReLU for ConvBlockRes.bn1, 0 = ReLU for
//               DecoderBlockRes.bn1)
struct BlockFuse { bool opA_ready = false; const char* next_bn = nullptr; float next_slope = 0.01f; };

// seq: the items' extents along H at this level (ragged batch; NULL = all H rows).  The eval BatchNorms (bn_act) are
// pointwise, so rows beyond an item's extent only carry values that the convolutions never read; the train-mode
// statistics cover each item's own rows (seq[b] * W positions).
int conv_block(Ctx& c, const std::string& p, const float* in, long long ld_in, int B, int H, int W,
               int Cin, int Cout, float* out, long long ld_out, const BlockScratch& s, const int* seq,
               const BlockFuse& fz = BlockFuse()) {
  const int prec = c.prec();
  const long long P = (long long)H * W;
  const bool fuse = !c.train();
  // bf16 / tf32 modes: a 2-channel input (first encoder block) is zero-padded to 32 operand channels so the block
  // runs on the tensor-core kernel; the host packs conv1 / shortcut weights as [..][Cout][32] accordingly.
  const int Cop = (prec != VFX_PREC_FP32 && Cin < 32) ? 32 : Cin;
  if (Cop != Cin && !c.dry) {
    VFX_CUDA_CHECK(cudaMemsetAsync(s.opA, 0, (size_t)B * P * Cop * prec_esz(prec), c.st));
    VFX_CUDA_CHECK(cudaMemsetAsync(s.opX, 0, (size_t)B * P * Cop * prec_esz(prec), c.st));
  }
  if (!(fuse && fz.opA_ready)) {
    BnRef r;
    VFX_TRY(bn_resolve(c, p + ".bn1", Cin, in, P * ld_in, ld_in, B, P, Cin, seq, W, &r));
    if (!c.dry) {
      ProfScope ps(c, "bn_act", 0.0, (double)B * P * Cin * (4 + prec_esz(prec)));
      VFX_TRY(bn_act(prec, in, P * ld_in, ld_in, B, P, Cin, r.scale, r.shift, Cin, r.stat_sB, VFX_ACT_LRELU, 0.01f, s.opA,
                     P * Cop, Cop, c.st));
    }
  }
  char tg[64];
  if (fuse) {     // conv1 with bn2 folded in: h = lrelu(conv1f(a) + b) straight into the operand buffer
    vfx_conv_desc d = conv_base(s.opA, B, H, W, Cop, getw(c, p + ".conv1f.w", (size_t)9 * Cout * Cop, prec), Cout);
    taps3x3(d, (long long)Cout * Cop);
    set_seq(d, seq, seq, 0);
    d.bias = getf(c, p + ".conv1f.b", Cout);
    set_act(d, s.opH, Cout, 0, VFX_ACT_LRELU, 0.01f);
    snprintf(tg, sizeof(tg), "unet.conv3x3.W%d.%dto%d", W, Cin, Cout);
    VFX_TRY(run_conv(c, prec, d, c.e->profile > 1 ? tg : "unet.conv3x3"));
  } else {
    vfx_conv_desc d = conv_base(s.opA, B, H, W, Cop, getw(c, p + ".conv1.w", (size_t)9 * Cout * Cop, prec), Cout);
    taps3x3(d, (long long)Cout * Cop);
    set_seq(d, seq, seq, 0);
    set_raw(d, s.rawH, Cout, 0);
    snprintf(tg, sizeof(tg), "unet.conv3x3.W%d.%dto%d", W, Cin, Cout);
    VFX_TRY(run_conv(c, prec, d, c.e->profile > 1 ? tg : "unet.conv3x3"));
    VFX_TRY(bn_act_op(c, prec, p + ".bn2", Cout, s.rawH, P * Cout, Cout, B, P, Cout, seq, W, VFX_ACT_LRELU, 0.01f, s.opH));
  }
  const float* res = in; long long ld_res = ld_in;
  if (Cin != Cout) {
    const void* xin = in;
    if (prec != VFX_PREC_FP32 || ld_in != Cin) {   // shortcut consumes raw x as a dense operand
      if (!c.dry) VFX_TRY(bn_act(prec, in, P * ld_in, ld_in, B, P, Cin, nullptr, nullptr, Cin, 0, VFX_ACT_NONE, 0.f,
                                 s.opX, P * Cop, Cop, c.st));
      xin = s.opX;
    }
    vfx_conv_desc d = conv_base(xin, B, H, W, Cop, getw(c, p + ".sc.w", (size_t)Cout * Cop, prec), Cout);
    d.ntaps = 1;
    set_seq(d, seq, seq, 0);
    d.bias = getf(c, p + ".sc.b", Cout);
    set_raw(d, s.rawS, Cout, 0);
    VFX_TRY(run_conv(c, prec, d, "unet.shortcut"));
    res = s.rawS; ld_res = Cout;
  }
  {
    vfx_conv_desc d = conv_base(s.opH, B, H, W, Cout, getw(c, p + ".conv2.w", (size_t)9 * Cout * Cout, prec), Cout);
    taps3x3(d, (long long)Cout * Cout);
    set_seq(d, seq, seq, 0);
    set_res(d, res, ld_res, 0);
    set_raw(d, out, ld_out, 0);
    if (fuse && fz.next_bn) {   // the consumer's eval BatchNorm + activation, fused: s.opA = act(bn(out))
      const std::string nb(fz.next_bn);
      d.act_scale = getf(c, nb + ".scale", Cout);
      d.act_shift = getf(c, nb + ".shift", Cout);
      set_act(d, s.opA, Cout, 0, VFX_ACT_LRELU, fz.next_slope);
    }
    snprintf(tg, sizeof(tg), "unet.conv3x3.W%d.%dto%d.res", W, Cout, Cout);
    VFX_TRY(run_conv(c, prec, d, c.e->profile > 1 ? tg : "unet.conv3x3"));
  }
  return c.rc;
}

// UNetResComplex_100Mb.forward voicefixer/restorer/model_kqq_bn.py:130-181.
// unet_in raw [B][Tp][127][2]; returns pointer to the last feature map raw [B][Tp][127][32].
int unet_forward(Ctx& c, const float* unet_in, int B, int Tp, float** feat_out) {
  const int prec = c.prec();
  int Hl[7], Wl[7];
  Hl[0] = Tp; Wl[0] = 127;                       // level l (1..6) works at Hl[l-1] x Wl[l-1]
  for (int l = 1; l < 7; ++l) { Hl[l] = Hl[l - 1] / 2; Wl[l] = Wl[l - 1] / 2; }
  const size_t esz = c.e->esz();
  const size_t P1 = (size_t)B * Tp * 127;
  BlockScratch s;
  s.opA = c.ws->raw(P1 * 64 * esz);
  s.rawH = c.ws->alloc<float>(P1 * 32);
  s.opH = c.ws->raw(P1 * 32 * esz);
  s.rawS = c.ws->alloc<float>(P1 * 32);
  s.opX = c.ws->raw(P1 * 64 * esz);
  float* cat[7]; float* pool[7];
  for (int l = 1; l <= 6; ++l) {
    const size_t P = (size_t)B * Hl[l - 1] * Wl[l - 1];
    cat[l] = c.ws->alloc<float>(P * 2 * UNET_C[l]);
    pool[l] = c.ws->alloc<float>((size_t)B * Hl[l] * Wl[l] * UNET_C[l]);
  }
  char name[96];
  // ---- encoder: level l output lives in the second half of the decoder's concat buffer
  const float* x = unet_in; int Cx = 2;
  for (int l = 1; l <= 6; ++l) {
    const int H = Hl[l - 1], W = Wl[l - 1], C = UNET_C[l];
    float* skip = cat[l] + C;                     // pitch 2C
    char nbn[4][96];
    for (int j = 1; j <= 4; ++j) {
      snprintf(name, sizeof(name), "unet.enc%d.b%d", l, j);
      BlockFuse fz;
      fz.opA_ready = j > 1;                               // produced by block j-1's conv2 epilogue
      if (j < 4) { snprintf(nbn[j], sizeof(nbn[j]), "unet.enc%d.b%d.bn1", l, j + 1); fz.next_bn = nbn[j]; }
      if (j == 1) VFX_TRY(conv_block(c, name, x, Cx, B, H, W, Cx, C, skip, 2 * C, s, c.ext_at(EXT_UNET0 + l - 1), fz));
      else VFX_TRY(conv_block(c, name, skip, 2 * C, B, H, W, C, C, skip, 2 * C, s, c.ext_at(EXT_UNET0 + l - 1), fz));
    }
    // (every extent is a multiple of 64 >> (l - 1): the 2 x 2 windows of an item's rows never straddle its end)
    ProfScope ps(c, "unet.pool", 0.0, (double)B * H * W * C * 5.0);
    if (!c.dry) VFX_TRY(avgpool2x2(skip, (long long)H * W * 2 * C, (long long)W * 2 * C, 2 * C, B, H, W, C, pool[l], c.st));
    x = pool[l]; Cx = C;
  }
  // ---- centre block (in place on pool[6]): conv_block7
  {
    BlockFuse fz; fz.next_bn = "unet.dec1.bn1"; fz.next_slope = 0.0f;      // relu(bn1(x)) before the first ConvTranspose
    VFX_TRY(conv_block(c, "unet.center", pool[6], 384, B, Hl[6], Wl[6], 384, 384, pool[6], 384, s, c.ext_at(EXT_UNET0 + 6), fz));
  }
  float* xd = pool[6];
  int Cd = 384;
  const bool fuse = !c.train();
  // ---- decoder i = 1..6 at level l = 7 - i  (DecoderBlockRes.forward restorer/modules.py:149-157)
  for (int i = 1; i <= 6; ++i) {
    const int l = 7 - i;
    const int H = Hl[l], W = Wl[l];               // input grid
    const int OH = Hl[l - 1], OW = Wl[l - 1];     // output grid (= 2H, 2W+1)
    const int Cout = UNET_C[l];
    snprintf(name, sizeof(name), "unet.dec%d", i);
    const std::string p(name);
    const long long Pin = (long long)H * W;
    if (!fuse)   // eval: relu(bn1(x)) was written into s.opA by the producing conv2's epilogue
      VFX_TRY(bn_act_op(c, prec, p + ".bn1", Cd, xd, Pin * Cd, Cd, B, Pin, Cd, c.ext_at(EXT_UNET0 + l), W, VFX_ACT_LRELU,
                        0.0f, s.opA));
    const void* wt = getw(c, p + ".up.w", (size_t)9 * Cout * Cd, prec);
    for (int rh = 0; rh < 2; ++rh)
      for (int rw = 0; rw < 2; ++rw) {
        vfx_conv_desc d = conv_base(s.opA, B, H, W, Cd, wt, Cout);
        d.Hq = H; d.Wq = W + 1; d.sh = 2; d.sw = 2; d.rh = rh; d.rw = rw; d.OH = OH; d.OW = OW;
        int n = 0;
        for (int kh = (rh ? 1 : 0); kh < 3; kh += 2)
          for (int kw = (rw ? 1 : 0); kw < 3; kw += 2) {
            d.dh[n] = kh == 2 ? -1 : 0; d.dw[n] = kw == 2 ? -1 : 0;
            d.w_off[n] = (long long)(kh * 3 + kw) * Cout * Cd;
            ++n;
          }
        d.ntaps = n;
        set_seq(d, c.ext_at(EXT_UNET0 + l), c.ext_at(EXT_UNET0 + l - 1), 0);
        set_raw(d, cat[l], 2 * Cout, 0);
        VFX_TRY(run_conv(c, prec, d, "unet.convT"));
      }
    // conv_block2..5: first consumes the concat tensor (2C -> C, with shortcut)
    float* dl = pool[l];                          // dense [B][OH][OW][Cout]: reuse? sizes differ -> own buffer
    dl = c.ws->alloc<float>((size_t)B * OH * OW * Cout);
    char nbn[96];
    for (int j = 2; j <= 5; ++j) {
      snprintf(name, sizeof(name), "unet.dec%d.b%d", i, j);
      BlockFuse fz;
      fz.opA_ready = j > 2;
      if (j < 5) { snprintf(nbn, sizeof(nbn), "unet.dec%d.b%d.bn1", i, j + 1); fz.next_bn = nbn; }
      else if (i < 6) { snprintf(nbn, sizeof(nbn), "unet.dec%d.bn1", i + 1); fz.next_bn = nbn; fz.next_slope = 0.0f; }
      else { snprintf(nbn, sizeof(nbn), "unet.after.bn1"); fz.next_bn = nbn; }
      if (j == 2) VFX_TRY(conv_block(c, name, cat[l], 2 * Cout, B, OH, OW, 2 * Cout, Cout, dl, Cout, s, c.ext_at(EXT_UNET0 + l - 1), fz));
      else VFX_TRY(conv_block(c, name, dl, Cout, B, OH, OW, Cout, Cout, dl, Cout, s, c.ext_at(EXT_UNET0 + l - 1), fz));
    }
    xd = dl; Cd = Cout;
  }
  {
    BlockFuse fz; fz.opA_ready = true;                   // dec6.b5 produced lrelu(after.bn1(x))
    VFX_TRY(conv_block(c, "unet.after", xd, 32, B, Tp, 127, 32, 32, xd, 32, s, c.ext_at(EXT_UNET0), fz));
  }
  *feat_out = xd;
  return c.rc;
}

// ------------------------------------------------------------------ denoiser
// nn.Sequential voicefixer/restorer/model.py:69-99 (always fp32 SIMT: 1 % of the path's FLOPs,
// recurrent part is precision-sensitive).  mel [B][T][128] -> lin15 raw [B*T][128].
// Denoiser GEMMs: fp32 SIMT in fp32 mode; in bf16 mode the same tensor-core kernel as the convolutions
// (bf16 operands, fp32 accumulate / bias / outputs).  The GRU recurrence itself is always fp32.
int linear(Ctx& c, const void* a, long long M, int K, const std::string& p, int N, float* out_raw,
           void* out_act, int act, const char* tag = "dn.linear") {
  const int prec = c.prec();
  vfx_conv_desc d = conv_base(a, 1, 1, (int)M, K, getw(c, p + ".w", (size_t)N * K, prec), N);
  d.ntaps = 1;
  d.bias = getf(c, p + ".b", N);
  if (out_raw) set_raw(d, out_raw, N, 0);
  if (out_act) set_act(d, out_act, N, 0, act, 0.f);
  return run_conv(c, prec, d, tag);
}

// fp32 tensor -> dense GEMM operand: the tensor itself in fp32 mode, a bf16 copy in bf16 mode
const void* dn_operand(Ctx& c, const float* x, long long M, int C, void* scratch, int* rc) {
  *rc = VFX_OK;
  if (c.prec() == VFX_PREC_FP32) return x;      // bf16: a bf16 copy; tf32: a copy rounded to tf32
  if (!c.dry) *rc = bn_act(c.prec(), x, M * C, C, 1, M, C, nullptr, nullptr, 1, 0, VFX_ACT_NONE, 0.f, scratch, M * C, C, c.st);
  return scratch;
}

int bn_gru(Ctx& c, const std::string& p, const float* x, int B, int T, void* op, float* gi,
           float* y0, float* y1) {
  const long long M = (long long)B * T;
  const int prec = c.prec();
  // BN2d(1) over the (T,512) plane of each item
  VFX_TRY(bn_act_op(c, prec, p + ".bn", 1, x, (long long)T * 512, 512, B, T, 512, c.ext_at(EXT_FRAMES), 1, VFX_ACT_NONE,
                    0.f, op));
  const void* in = op;
  float* outs[2] = {y0, y1};
  for (int layer = 0; layer < 2; ++layer) {
    char nm[64];
    snprintf(nm, sizeof(nm), "%s.l%d", p.c_str(), layer);
    const std::string q(nm);
    vfx_conv_desc d = conv_base(in, 1, 1, (int)M, 512, getw(c, q + ".wih", (size_t)1536 * 512, prec), 1536);
    d.ntaps = 1;
    d.bias = getf(c, q + ".bih", 1536);
    set_raw(d, gi, 1536, 0);
    const float* whh = getf(c, q + ".whh_t", (size_t)2 * 256 * 768);
    const float* bhh = getf(c, q + ".bhh", 2 * 768);
    VFX_TRY(run_conv(c, prec, d, "dn.gru_in"));
    if (!c.dry && c.rc == VFX_OK) {
      ProfScope ps(c, "dn.gru", 2.0 * M * 2 * 768 * 256, 0.0);
      VFX_TRY(gru_layer(gi, whh, bhh, B, T, c.ext_at(EXT_FRAMES), outs[layer], c.st));
    }
    if (layer == 0) { int rc; in = dn_operand(c, y0, M, 512, op, &rc); VFX_TRY(rc); }
  }
  return c.rc;
}

int relu_inplace(Ctx& c, float* x, int B, int T, int C) {
  if (c.dry) return VFX_OK;
  return bn_act(VFX_PREC_FP32, x, (long long)T * C, C, B, T, C, nullptr, nullptr, 1, 0, VFX_ACT_LRELU, 0.f, x,
                (long long)T * C, C, c.st);
}

// Mode 2's dropout masks: explicit keep-masks uint8 [2][B][T][512], or one seeded key per item (both NULL: no dropout).
// Either way the caller owns the memory, so the workspace does not depend on the choice.
struct DropSrc {
  const uint8_t* masks = nullptr;
  const vfx_drop_key* keys = nullptr;
};

// Dropout `layer` (0: after lin4, 1: after lin11) in place on x [B][T][512]
int dropout(Ctx& c, float* x, int B, int T, const DropSrc& drop, int layer) {
  if (!c.train() || c.dry) return VFX_OK;
  const long long n = (long long)B * T * 512;
  if (drop.keys) return dropout_seeded(x, B, T, drop.keys, layer, c.st);
  if (drop.masks) return dropout_apply(x, drop.masks + layer * n, n, c.st);
  return VFX_OK;
}

// Ragged batch: every op but the GRU recurrence and the train-mode statistics is per frame (Linear GEMMs over B*T rows,
// BatchNorm and ReLU via bn_act, dropout), so frames beyond an item's end only produce values that no later kernel reads;
// the GRU and the statistics take the items' frame counts (EXT_FRAMES).
int denoiser_forward(Ctx& c, const float* mel, int B, int T, const DropSrc& drop, float* lin_out) {
  const long long M = (long long)B * T;
  const int prec = c.prec();
  void* a = c.ws->alloc<float>(M * 512);          // operand scratch (fp32-sized)
  float* b = c.ws->alloc<float>(M * 512);
  float* y0 = c.ws->alloc<float>(M * 512);
  float* gi = c.ws->alloc<float>(M * 1536);
  const std::string p = "dn.";
  const int* fr = c.ext_at(EXT_FRAMES);
  VFX_TRY(bn_act_op(c, prec, p + "bn0", 1, mel, (long long)T * 128, 128, B, T, 128, fr, 1, VFX_ACT_NONE, 0.f, a));
  VFX_TRY(linear(c, a, M, 128, p + "lin1", 256, b, nullptr, 0));
  VFX_TRY(relu_inplace(c, b, B, T, 256));
  VFX_TRY(bn_act_op(c, prec, p + "bn3", 1, b, (long long)T * 256, 256, B, T, 256, fr, 1, VFX_ACT_NONE, 0.f, a));
  VFX_TRY(linear(c, a, M, 256, p + "lin4", 512, b, nullptr, 0));
  VFX_TRY(dropout(c, b, B, T, drop, 0));
  VFX_TRY(relu_inplace(c, b, B, T, 512));
  VFX_TRY(bn_gru(c, p + "g7", b, B, T, a, gi, y0, b));       // result in b
  VFX_TRY(bn_gru(c, p + "g8", b, B, T, a, gi, y0, b));
  VFX_TRY(bn_act_op(c, prec, p + "bn9", 1, b, (long long)T * 512, 512, B, T, 512, fr, 1, VFX_ACT_LRELU, 0.f, a));
  VFX_TRY(linear(c, a, M, 512, p + "lin11", 512, b, nullptr, 0));
  VFX_TRY(dropout(c, b, B, T, drop, 1));
  VFX_TRY(bn_act_op(c, prec, p + "bn13", 1, b, (long long)T * 512, 512, B, T, 512, fr, 1, VFX_ACT_LRELU, 0.f, a));
  VFX_TRY(linear(c, a, M, 512, p + "lin15", 128, lin_out, nullptr, 0));
  return c.rc;
}

int analysis_forward(Ctx& c, const float* mel, int B, int T, const DropSrc& drop, float* mel_log_out) {
  const int Tp = (T + 63) / 64 * 64;
  // mode 2: the reference's train-mode BatchNorm raises "Expected more than 1 value per channel when training"
  // when the UNet centre is 1x1, i.e. for segments of at most 64 frames (checked on the capacity; a ragged item that
  // breaks it gets finite, unspecified samples: its 1 x 1 centre statistics have zero variance)
  if (c.train() && !c.dry) VFX_REQUIRE(Tp > 64, "mode 2 needs more than 64 frames per segment (got T=%d): Expected more than 1 value per channel when training", T);
  const size_t m0 = c.ws->mark();
  float* xlog = c.ws->alloc<float>((size_t)B * T * 128);
  float* unet_in = c.ws->alloc<float>((size_t)B * Tp * 127 * 2);
  float* lin = c.ws->alloc<float>((size_t)B * T * 128);
  {
    const size_t m1 = c.ws->mark();
    VFX_TRY(denoiser_forward(c, mel, B, T, drop, lin));
    c.ws->reset(m1);
  }
  if (!c.dry) VFX_TRY(mask_log_pack(lin, mel, B, T, Tp, c.ext_at(EXT_FRAMES), xlog, unet_in, c.st));
  float* feat = nullptr;
  VFX_TRY(unet_forward(c, unet_in, B, Tp, &feat));
  const float* hw = getf(c, "unet.head.w", 32);
  const float* hb = getf(c, "unet.head.b", 1);
  if (!c.dry && c.rc == VFX_OK) VFX_TRY(unet_head(feat, B, T, Tp, hw, hb, xlog, mel_log_out, c.st));
  c.ws->reset(m0);
  return c.rc;
}

// ------------------------------------------------------------------ vocoder
// The inputs and outputs of fused pair i of stack j (last: i == 7, last_stack: j == 3).  A pair reads its operand with a
// halo that neighbouring tiles would overwrite in place, so the operand ping-pongs from cur to nxt: the tf32 encoded stream
// between X and A0 (fused at C = 64 only, the last stack, whose 8 pairs end in X), the 16-bit operand between A0 and Hh.
void pair_io(vfx_pair_desc& pd, bool enc, bool last, bool last_stack, void* cur, void* nxt, float* X, void* U) {
  pd.a = cur;
  if (enc) {
    pd.x = (float*)cur; pd.x_out = (float*)nxt; pd.write_raw = 1;
    pd.stream_enc = 1; pd.stream_enc_out = last ? 0 : 1;    // the last pair hands plain x' to the final convolution
    return;
  }
  pd.x = X;
  pd.write_raw = (!last || last_stack) ? 1 : 0;             // the next up-sampler consumes the operand only
  if (!last) { pd.out_act = nxt; pd.act = VFX_ACT_LRELU; pd.act_param = 0.01f; }
  else if (!last_stack) { pd.out_act = U; pd.act = VFX_ACT_LRELU_XSINX; pd.act_param = 0.2f; }
}

// ResStack j: 8 x (x + conv_k3_d1(lrelu(conv_k3_d3^i(lrelu(x))))), modules.py:550-576,592-595, width C, L rows (ext: the
// items' lengths), x (or, enc, the encoded stream) in X.  A pair that pair_supported() accepts is one fused kernel (h stays
// on chip), the others two convolutions with h in Hh.  The last stack ends with x' in X, the others with the next operand in U.
int resstack(Ctx& c, int j, int B, long long L, int C, const int* ext, bool enc, float* X, void* A0, void* Hh, void* U) {
  const int prec = c.prec();
  const bool fused = c.e->use_tc && c.e->fuse_pairs && pair_supported(prec, C, enc);
  void* cur = enc ? (void*)X : A0; void* nxt = enc ? A0 : Hh;
  const std::string rs = "voc.rs" + std::to_string(j);
  for (int i = 0, dil = 1; i < 8; ++i, dil *= 3) {
    const std::string p = rs + ".l" + std::to_string(i);
    const std::string per_dil = c.e->profile > 1 ? ".d" + std::to_string(dil) : "";   // profile 2: a tag per dilation
    const void* w1 = getw(c, p + ".c1.w", (size_t)3 * C * C, prec); const float* b1 = getf(c, p + ".c1.b", C);
    const void* w2 = getw(c, p + ".c2.w", (size_t)3 * C * C, prec); const float* b2 = getf(c, p + ".c2.b", C);
    if (fused) {
      vfx_pair_desc pd;
      memset(&pd, 0, sizeof(pd));
      pd.precision = prec; pd.dilation = dil; pd.B = B; pd.L = (int)L; pd.C = C; pd.lens = ext;
      pd.w1 = w1; pd.b1 = b1; pd.w2 = w2; pd.b2 = b2;
      pair_io(pd, enc, i == 7, j == 3, cur, nxt, X, U);
      if (!c.dry && c.rc == VFX_OK) {
        const double els = (double)B * L * C;
        // algorithmic bytes of a pair (SURVEY 8d): x in + x' out, fp32
        ProfScope ps(c, (rs + ".pair" + per_dil).c_str(), 2.0 * 2.0 * 3.0 * C * els, 8.0 * els);
        VFX_TRY(resstack_pair(pd, c.st));
      }
      std::swap(cur, nxt);
    } else {
      vfx_conv_desc d1 = conv_base(enc ? (const void*)X : (const void*)A0, B, 1, (int)L, C, w1, C);
      d1.ntaps = 3;
      for (int k = 0; k < 3; ++k) { d1.dw[k] = (k - 1) * dil; d1.w_off[k] = (long long)k * C * C; }
      set_seq(d1, ext, ext, 1);
      d1.bias = b1;
      set_act(d1, Hh, C, 0, VFX_ACT_LRELU, 0.01f);
      VFX_TRY(run_conv(c, prec, d1, (rs + ".c1" + per_dil).c_str()));
      vfx_conv_desc d2 = conv_base(Hh, B, 1, (int)L, C, w2, C);
      d2.ntaps = 3;
      for (int k = 0; k < 3; ++k) { d2.dw[k] = k - 1; d2.w_off[k] = (long long)k * C * C; }
      set_seq(d2, ext, ext, 1);
      d2.bias = b2;
      set_res(d2, X, C, 0);
      if (enc) {
        d2.res_enc = 1; d2.enc_slope = 0.01f;
        if (i < 7) { set_raw(d2, X, C, 0); d2.raw_enc = 1; }              // S' in place
        else if (j == 3) set_raw(d2, X, C, 0);                           // last stack: plain x' for the final conv
        else set_act(d2, U, C, 0, VFX_ACT_LRELU_XSINX, 0.2f);            // next UpsampleNet's operand only
      } else {
        set_raw(d2, X, C, 0);
        if (i < 7) set_act(d2, A0, C, 0, VFX_ACT_LRELU, 0.01f);
        else if (j < 3) set_act(d2, U, C, 0, VFX_ACT_LRELU_XSINX, 0.2f);  // act + next UpsampleNet's x+sin x
      }
      VFX_TRY(run_conv(c, prec, d2, (rs + ".c2").c_str()));
    }
  }
  return VFX_OK;     // a missing weight stays in c.rc: the dry pass goes on listing the others
}

// vocoder Generator.forward voicefixer/vocoder/model/generator.py:127-145 on cond [B][Tc][128]
// (operand precision), then the fused post conv / tanh / trim.
int vocoder_generator(Ctx& c, const void* cond, int B, int Tc, float* wav_out, int trim_len, float scale) {
  const int prec = c.prec();
  const size_t esz = c.e->esz();
  const size_t m0 = c.ws->mark();
  const long long S = (long long)Tc * 441;
  // condnet buffers
  void* c0 = c.ws->raw((size_t)B * (Tc + 6) * 512 * esz);
  void* c1 = c.ws->raw((size_t)B * (Tc + 6) * 512 * esz);
  // full-rate buffers: X raw fp32, A0 / Hh / U operands
  const size_t maxel = (size_t)B * S * 64;
  float* X = c.ws->alloc<float>(maxel);
  void* A0 = c.ws->raw(maxel * esz);
  void* Hh = c.ws->raw(maxel * esz);
  void* U = c.ws->raw(maxel * esz);
  char name[96];
  // ---- condnet: 5 x (Conv1d k3 p1 + ELU), generator.py:33-54
  const void* in = cond; int Cin = 128;
  void* pp[2] = {c0, c1};
  for (int i = 0; i < 5; ++i) {
    snprintf(name, sizeof(name), "voc.cond%d", i);
    const std::string p(name);
    vfx_conv_desc d = conv_base(in, B, 1, Tc, Cin, getw(c, p + ".w", (size_t)3 * 512 * Cin, prec), 512);
    d.ntaps = 3;
    for (int k = 0; k < 3; ++k) { d.dw[k] = k - 1; d.w_off[k] = (long long)k * 512 * Cin; }
    set_seq(d, c.ext_at(EXT_COND), c.ext_at(EXT_COND), 1);
    d.bias = getf(c, p + ".b", 512);
    void* out = pp[i & 1];
    if (i == 4) {   // last ELU output goes to rows 3..Tc+2 of the reflect-padded buffer
      set_act(d, (char*)out + (size_t)3 * 512 * esz, 512, 0, VFX_ACT_ELU, 0.f);
      d.oa_sB = (long long)(Tc + 6) * 512;
    } else {
      set_act(d, out, 512, 0, VFX_ACT_ELU, 0.f);
    }
    VFX_TRY(run_conv(c, prec, d, "voc.condnet"));
    in = out; Cin = 512;
  }
  if (!c.dry) VFX_TRY(reflect_pad3((void*)in, B, Tc, 512, c.ext_at(EXT_COND), prec, c.st));
  // ---- ReflectionPad1d(3) + Conv1d(512,1024,k7) + LeakyReLU(0.2); the x + sin x of the first
  //      UpsampleNet (modules.py:504) is applied in the same epilogue.
  {
    vfx_conv_desc d = conv_base(in, B, 1, Tc + 6, 512, getw(c, "voc.pre.w", (size_t)7 * 1024 * 512, prec), 1024);
    d.ntaps = 7; d.Wq = Tc; d.OW = Tc;
    for (int k = 0; k < 7; ++k) { d.dw[k] = k; d.w_off[k] = (long long)k * 1024 * 512; }
    set_seq(d, c.ext_at(EXT_COND_PAD), c.ext_at(EXT_COND), 1);
    d.bias = getf(c, "voc.pre.b", 1024);
    set_act(d, U, 1024, 0, VFX_ACT_LRELU_XSINX, 0.2f);
    VFX_TRY(run_conv(c, prec, d, "voc.pre"));
  }
  // TF32 "encoded stream" (vfx_conv_desc.res_enc / raw_enc): X holds S = bits(lrelu(x)) + 0x1000, which conv1 reads as
  // its tf32 operand and conv2 decodes as the fp32 residual -- no separate activated copy (24 -> 20 bytes per element and pair)
  const bool enc = prec == VFX_PREC_TF32 && c.e->use_tc && c.e->tf32_stream;
  long long Lin = Tc;
  for (int j = 0; j < 4; ++j) {
    const int Ci = VOC_CIN[j], Co = VOC_COUT[j], u = VOC_U[j];
    const long long Lout = Lin * u;
    // ragged batch: items' lengths at this up-sampler's input (= rows of its reshaped output view) and output rate
    const int* ext_in = c.ext_at(j == 0 ? EXT_COND : EXT_UP0 + j - 1);
    const int* ext_out = c.ext_at(EXT_UP0 + j);
    char up_tag[32];
    snprintf(up_tag, sizeof(up_tag), "voc.up%d", j);
    // ---- UpsampleNet: ConvTranspose1d(k=2u, s=u, p, op) as two phase-group GEMMs (modules.py:451-459)
    snprintf(name, sizeof(name), "voc.up%d", j);
    {
      const std::string p(name);
      const void* w = getw(c, p + ".w", (size_t)2 * u * Co * Ci, prec);
      const float* bias = getf(c, p + ".b", Co);
      const int pad = u / 2 + u % 2, nA = u - pad;
      const long long mat = (long long)Co * Ci;
      for (int grp = 0; grp < 2; ++grp) {
        const int nph = grp == 0 ? nA : u - nA;
        // Output described as the reshaped view [B][Lin][u*Co] (row q holds output samples q*u .. q*u+u-1):
        // the phase group is then a plain stride-1 GEMM writing columns [r0*Co, (r0+nph)*Co) of row q.
        vfx_conv_desc d = conv_base(U, B, 1, (int)Lin, Ci, w, nph * Co);
        d.ntaps = 2;
        int r0;
        if (grp == 0) { d.dw[0] = 0; d.w_off[0] = pad * mat; d.dw[1] = -1; d.w_off[1] = (pad + u) * mat; r0 = 0; }
        else          { d.dw[0] = 1; d.w_off[0] = 0;         d.dw[1] = 0;  d.w_off[1] = u * mat;         r0 = nA; }
        d.bias = bias; d.bias_mod = Co;
        set_seq(d, ext_in, ext_in, 1);
        set_raw(d, X, (long long)u * Co, r0 * Co);
        if (enc) { d.raw_enc = 1; d.enc_slope = 0.01f; }
        else set_act(d, A0, (long long)u * Co, r0 * Co, VFX_ACT_LRELU, 0.01f);
        VFX_TRY(run_conv(c, prec, d, up_tag));
      }
    }
    VFX_TRY(resstack(c, j, B, Lout, Co, ext_out, enc, X, A0, Hh, U));
    Lin = Lout;
  }
  // ---- LeakyReLU(0.2) + ReflectionPad1d(3) + Conv1d(64,1,7) + Tanh + _trim_center
  int lo = 0; long long out_len = S;
  if (trim_len >= 0) {
    VFX_REQUIRE(trim_len <= S, "vocoder: trim_len %d exceeds generated length %lld", trim_len, S);
    const long long diff = S - trim_len;
    lo = (int)(diff / 2); out_len = trim_len;
    VFX_REQUIRE(diff == 0 || diff / 2 >= 1, "vocoder: _trim_center is degenerate for a length difference of 1");
  }
  const float* pw = getf(c, "voc.post.w", 7 * 64);
  const float* pb = getf(c, "voc.post.b", 1);
  ProfScope ps(c, "voc.post", 2.0 * B * out_len * 7 * 64, (double)B * S * 64 * 4);
  if (!c.dry && c.rc == VFX_OK) VFX_TRY(voc_post(X, B, (int)S, pw, pb, lo, (int)out_len, c.ext_at(EXT_UP0 + 3),
                                                         c.ext_at(EXT_SAMPLES), scale, wav_out, c.st));
  c.ws->reset(m0);
  return c.rc;
}

int vocoder_forward(Ctx& c, const float* mel, int B, int T, int input_is_log, float* wav_out, int trim_len,
                    float scale) {
  const int Tc = T + T % 2 + 4;
  const size_t m0 = c.ws->mark();
  void* cond = c.ws->raw((size_t)B * Tc * 128 * c.e->esz());
  const float* tab = getf(c, "voc.mel_tab", 129);
  if (!c.dry && c.rc == VFX_OK) VFX_TRY(voc_normalize(mel, B, T, Tc, c.ext_at(EXT_FRAMES), input_is_log, tab, cond, c.prec(), c.st));
  VFX_TRY(vocoder_generator(c, cond, B, Tc, wav_out, trim_len, scale));
  c.ws->reset(m0);
  return c.rc;
}

// the Generator on fp32 conditions cond[B][Tc][128], cast into the operand format in the workspace first
int vocoder_cond_forward(Ctx& c, const float* cond, int B, int Tc, float* wav_out, int trim_len, float scale) {
  void* op = c.ws->raw((size_t)B * Tc * 128 * c.e->esz());
  if (!c.dry) VFX_TRY(cast_rows(cond, (long long)B * Tc * 128, op, c.prec(), c.st));
  return vocoder_generator(c, op, B, Tc, wav_out, trim_len, scale);
}

int frontend_forward(Ctx& c, const float* wav, int B, int L, float* mel, float* sp) {
  const int T = 1 + L / 441;
  const float* fbT = getf(c, "fe.fbT", (size_t)128 * 1025);
  const int* fs = (const int*)get(c, "fe.fb_start", 128 * 4);
  const int* fl = (const int*)get(c, "fe.fb_len", 128 * 4);
  if (c.dry || c.rc != VFX_OK) return c.rc;
  ProfScope ps(c, "fe.stft_mel", (double)B * T * (5.0 * 1024 * 10 + 2.0 * 2050), (double)B * L * 4);
  return stft_mel(wav, B, L, T, c.ext_at(EXT_SAMPLES), c.ext_at(EXT_FRAMES), c.e->d_window, c.e->d_tw, fbT, fs, fl, mel,
                  sp, c.st);
}

// Vocoder.forward on a ragged batch of mels: item b is the first frames[b] rows of mel[B][T_cap][128]; the frame-based
// extent table gives every vocoder kernel the item's own lengths, and voc_post writes its S_b samples untrimmed, then zeros.
int vocoder_ragged_forward(Ctx& c, const float* mel, int B, int T_cap, const int* frames, int input_is_log,
                           float* wav_out, float scale) {
  int* ext = c.ws->alloc<int>((size_t)EXT_LEVELS * B);
  if (!c.dry) VFX_TRY(frame_extents(frames, B, T_cap, ext, c.st));
  c.ext = ext; c.ext_B = B;
  return vocoder_forward(c, mel, B, T_cap, input_is_log, wav_out, -1, scale);
}

// Vocoder.oracle (vocoder/base.py:58-77 up to the file write) on wav[B][L_cap]: the device front end writes the
// conditions in the operand format straight into the workspace, and the generator consumes them.  lens (ragged batch,
// NULL = L_cap each): the front end also writes each item's frame count, from which the frame-based extent table is built.
// The table is allocated either way, so that one dry pass sizes both forms.
int oracle_forward(Ctx& c, const float* wav, int B, int L_cap, const int* lens, float scale, float* wav_out) {
  const int T = 1 + L_cap / 441, Tc = T + T % 2 + 4;
  unsigned int* peak = c.ws->alloc<unsigned int>(B);
  int* frames = c.ws->alloc<int>(B);
  int* ext = c.ws->alloc<int>((size_t)EXT_LEVELS * B);
  void* cond = c.ws->raw((size_t)B * Tc * 128 * c.e->esz());
  if (!c.dry) {
    VFX_TRY(oracle_frontend(wav, B, L_cap, lens, c.e->d_obasis, c.e->d_oband,
                            c.e->d_oband + 128, peak, lens ? frames : nullptr, cond, c.prec(), nullptr, c.st));
    if (lens) VFX_TRY(frame_extents(frames, B, T, ext, c.st));
  }
  if (lens) { c.ext = ext; c.ext_B = B; }
  return vocoder_generator(c, cond, B, Tc, wav_out, -1, scale);
}

// the front end of oracle_forward alone, into fp32 conditions [B][Tc_cap][128]
int oracle_cond_forward(Ctx& c, const float* wav, int B, int L_cap, const int* lens, float* cond_out) {
  unsigned int* peak = c.ws->alloc<unsigned int>(B);
  if (c.dry) return VFX_OK;
  return oracle_frontend(wav, B, L_cap, lens, c.e->d_obasis, c.e->d_oband, c.e->d_oband + 128,
                         peak, nullptr, nullptr, c.prec(), cond_out, c.st);
}

// vfx_resample: the item table is staged into the workspace, then one launch
int resample_forward(Ctx& c, const float* x, const float* h, const vfx_resample_item* items_host, int B, int L_cap,
                     float* y, int* lens_out) {
  vfx_resample_item* items = c.ws->alloc<vfx_resample_item>(B);
  if (c.dry) return VFX_OK;
  VFX_CUDA_CHECK(cudaMemcpyAsync(items, items_host, sizeof(vfx_resample_item) * B, cudaMemcpyHostToDevice, c.st));
  return resample(x, h, items, B, L_cap, y, lens_out, c.st);
}

// One item of vfx_resample against the buffers (include/vfx_b200.h): VFX_ERR_INVALID with a message naming item b.
int check_resample_item(const vfx_resample_item& it, int b, long long x_elems, long long h_elems, int L_cap) {
  VFX_REQUIRE(it.up >= 1 && it.down >= 1 && it.up <= (1 << 20), "resample: item %d: ratio %d/%d (up must lie in [1, 2^20], "
              "down >= 1)", b, it.up, it.down);
  VFX_REQUIRE(it.n_in >= 0 && it.n_in <= (1LL << 40), "resample: item %d: recording length %lld", b, it.n_in);
  VFX_REQUIRE(it.x_off >= 0 && it.x_len >= 0 && it.x_off + it.x_len <= x_elems, "resample: item %d: window "
              "x[%lld, %lld) is not inside the %lld staged samples", b, it.x_off, it.x_off + it.x_len, x_elems);
  VFX_REQUIRE(it.x_first >= 0 && it.x_first + it.x_len <= it.n_in, "resample: item %d: window [%lld, %lld) is not inside "
              "its recording of %lld samples", b, it.x_first, it.x_first + it.x_len, it.n_in);
  const bool copy = it.up == 1 && it.down == 1;
  if (!copy)
    VFX_REQUIRE(it.h_off >= 0 && it.h_len >= 1 && it.h_off + it.h_len <= h_elems && it.rem >= 0, "resample: item %d: "
                "taps h[%lld, %lld) (rem %d) are not inside the %lld given", b, it.h_off, it.h_off + it.h_len, it.rem,
                h_elems);
  const long long n_out = (it.n_in * it.up + it.down - 1) / it.down;
  VFX_REQUIRE(it.y_len >= 0 && it.y_len <= L_cap, "resample: item %d: y_len %d is not in [0, L_cap = %d]", b, it.y_len,
              L_cap);
  VFX_REQUIRE(it.y_first >= 0 && it.y_first + it.y_len <= n_out, "resample: item %d: outputs [%lld, %lld) are not inside "
              "the stream's %lld samples", b, it.y_first, it.y_first + it.y_len, n_out);
  if (it.y_len == 0) return VFX_OK;
  long long lo = it.y_first, hi = it.y_first + it.y_len - 1;           // the inputs the outputs read (a copy: the same)
  if (!copy) {
    const long long num = (it.y_first + it.rem) * it.down - it.h_len + 1;
    lo = num <= 0 ? 0 : (num + it.up - 1) / it.up;
    hi = std::min(it.n_in - 1, (hi + it.rem) * it.down / it.up);
  }
  if (lo <= hi)
    VFX_REQUIRE(it.x_first <= lo && hi < it.x_first + it.x_len, "resample: item %d: outputs [%lld, %lld) read inputs "
                "[%lld, %lld); the window holds [%lld, %lld)", b, it.y_first, it.y_first + it.y_len, lo, hi + 1, it.x_first,
                it.x_first + it.x_len);
  return VFX_OK;
}

// vfx_resample_src: the item table is staged into the workspace, then one launch
int resample_src_forward(Ctx& c, const float* h, const vfx_resample_src_item* items_host, int B, int L_cap, float* y,
                         int* lens_out) {
  vfx_resample_src_item* items = c.ws->alloc<vfx_resample_src_item>(B);
  if (c.dry) return VFX_OK;
  VFX_CUDA_CHECK(cudaMemcpyAsync(items, items_host, sizeof(vfx_resample_src_item) * B, cudaMemcpyHostToDevice, c.st));
  return resample_src(h, items, B, L_cap, y, lens_out, c.st);
}

// One item of vfx_resample_src against the buffers (include/vfx_b200.h): VFX_ERR_INVALID with a message naming item b.
int check_resample_src_item(const vfx_resample_src_item& it, int b, long long h_elems, int L_cap) {
  VFX_REQUIRE(it.src, "resample_src: item %d: src is null", b);
  VFX_REQUIRE(it.up >= 1 && it.down >= 1 && it.up <= (1 << 20), "resample_src: item %d: ratio %d/%d (up must lie in "
              "[1, 2^20], down >= 1)", b, it.up, it.down);
  VFX_REQUIRE(it.n_in >= 0 && it.n_in <= (1LL << 40), "resample_src: item %d: recording length %lld", b, it.n_in);
  VFX_REQUIRE(it.stride >= 1 && (it.n_in <= 1 || it.stride <= (1LL << 62) / (it.n_in - 1)), "resample_src: item %d: "
              "stride %lld (must be >= 1, and (n_in - 1) * stride within 2^62)", b, it.stride);
  if (!(it.up == 1 && it.down == 1))
    VFX_REQUIRE(it.h_off >= 0 && it.h_len >= 1 && it.h_off + it.h_len <= h_elems && it.rem >= 0, "resample_src: item "
                "%d: taps h[%lld, %lld) (rem %d) are not inside the %lld given", b, it.h_off, it.h_off + it.h_len, it.rem,
                h_elems);
  const long long n_out = (it.n_in * it.up + it.down - 1) / it.down;
  VFX_REQUIRE(it.y_len >= 0 && it.y_len <= L_cap, "resample_src: item %d: y_len %d is not in [0, L_cap = %d]", b,
              it.y_len, L_cap);
  VFX_REQUIRE(it.y_first >= 0 && it.y_first <= n_out - it.y_len, "resample_src: item %d: outputs [%lld, %lld) are not "
              "inside the stream's %lld samples", b, it.y_first, it.y_first + it.y_len, n_out);
  return VFX_OK;
}

// vfx_scatter_rows: the item table is staged into the workspace, then one launch
static_assert(sizeof(vfx_scatter_item) == 32, "vfx_scatter_item: src_off must fit the tail padding");
int scatter_rows_forward(Ctx& c, const float* x, int B, long long ldx, const vfx_scatter_item* items_host,
                         int max_len) {
  vfx_scatter_item* items = c.ws->alloc<vfx_scatter_item>(B);
  if (c.dry) return VFX_OK;
  VFX_CUDA_CHECK(cudaMemcpyAsync(items, items_host, sizeof(vfx_scatter_item) * B, cudaMemcpyHostToDevice, c.st));
  return scatter_rows(x, B, ldx, items, max_len, c.st);
}

// The items of vfx_scatter_rows (include/vfx_b200.h): each on its own, then no two destination ranges overlapping.
// Sets *max_len to the longest item.
int check_scatter_items(const vfx_scatter_item* items, int B, long long ldx, int* max_len) {
  std::vector<std::pair<uintptr_t, int>> ranges;        // (first byte, item) of each non-empty destination range
  *max_len = 0;
  for (int b = 0; b < B; ++b) {
    const vfx_scatter_item& it = items[b];
    VFX_REQUIRE(it.dst, "scatter_rows: item %d: dst is null", b);
    VFX_REQUIRE(it.len >= 0 && it.len <= ldx, "scatter_rows: item %d: len %d is not in [0, ldx = %lld]", b, it.len, ldx);
    VFX_REQUIRE(it.src_off >= 0 && it.src_off <= ldx - it.len, "scatter_rows: item %d: source columns [%d, %lld) are "
                "not inside its row of ldx = %lld", b, it.src_off, (long long)it.src_off + it.len, ldx);
    VFX_REQUIRE(it.dst_off >= 0 && it.dst_elems >= 0 && it.dst_off <= it.dst_elems - it.len, "scatter_rows: item %d: "
                "destination [%lld, %lld) is not inside its %lld elements", b, it.dst_off, it.dst_off + it.len,
                it.dst_elems);
    if (it.len > 0) ranges.push_back({(uintptr_t)(it.dst + it.dst_off), b});
    *max_len = std::max(*max_len, it.len);
  }
  std::sort(ranges.begin(), ranges.end());
  for (size_t k = 1; k < ranges.size(); ++k) {
    const vfx_scatter_item& p = items[ranges[k - 1].second];
    VFX_REQUIRE(ranges[k - 1].first + sizeof(float) * p.len <= ranges[k].first, "scatter_rows: item %d: its destination "
                "overlaps item %d's", ranges[k].second, ranges[k - 1].second);
  }
  return VFX_OK;
}

// vfx_pack_pcm16: the item table and the per-file maxima are staged into the workspace, then two launches
int pack_pcm16_forward(Ctx& c, const vfx_pcm16_item* items_host, int B, short* y, long long max_n) {
  vfx_pcm16_item* items = c.ws->alloc<vfx_pcm16_item>(B);
  unsigned* vmax = c.ws->alloc<unsigned>(B);
  if (c.dry) return VFX_OK;
  VFX_CUDA_CHECK(cudaMemcpyAsync(items, items_host, sizeof(vfx_pcm16_item) * B, cudaMemcpyHostToDevice, c.st));
  return pack_pcm16(items, B, max_n, vmax, y, c.st);
}

// The items of vfx_pack_pcm16 (include/vfx_b200.h): each on its own, then no two destination ranges overlapping.
// Sets *max_n to the longest item.
int check_pcm16_items(const vfx_pcm16_item* items, int B, long long y_elems, long long* max_n) {
  std::vector<std::pair<long long, int>> ranges;        // (first element, item) of each destination range
  *max_n = 0;
  for (int b = 0; b < B; ++b) {
    const vfx_pcm16_item& it = items[b];
    VFX_REQUIRE(it.C >= 1 && it.C <= VFX_PCM16_MAX_CHANNELS, "pack_pcm16: item %d: %d channels (1 .. %d are packed)", b,
                it.C, VFX_PCM16_MAX_CHANNELS);
    for (int ch = 0; ch < it.C; ++ch) VFX_REQUIRE(it.rows[ch], "pack_pcm16: item %d: channel %d's row is null", b, ch);
    VFX_REQUIRE(it.n >= 1 && it.n <= (1LL << 40), "pack_pcm16: item %d: length %lld is not in [1, 2^40]", b, it.n);
    VFX_REQUIRE(it.dst_off >= 0 && it.dst_off <= y_elems - it.n * it.C, "pack_pcm16: item %d: destination [%lld, %lld) "
                "is not inside the %lld given", b, it.dst_off, it.dst_off + it.n * it.C, y_elems);
    ranges.push_back({it.dst_off, b});
    *max_n = std::max(*max_n, it.n);
  }
  std::sort(ranges.begin(), ranges.end());
  for (size_t k = 1; k < ranges.size(); ++k) {
    const vfx_pcm16_item& p = items[ranges[k - 1].second];
    VFX_REQUIRE(ranges[k - 1].first + p.n * p.C <= ranges[k].first, "pack_pcm16: item %d: its destination overlaps "
                "item %d's", ranges[k].second, ranges[k - 1].second);
  }
  return VFX_OK;
}

// Vocoder.oracle's mel basis: librosa.filters.mel(sr=44100, n_fft=2048, n_mels=128, fmin=0, fmax=22050, htk=True) with
// its default norm="slaney" (vocoder/model/util.py:115-123), built in float64 as librosa builds it and cast to float32
// (wavio.slaney_htk_mel_basis is the same formula on the host).  band: start[128] ++ len[128] of each row's non-zeros.
void slaney_htk_mel_basis(std::vector<float>& basis, std::vector<int>& band) {
  const int n_mels = 128, nbin = 1025;
  double mel_f[130];
  const double mmax = 2595.0 * log10(1.0 + 22050.0 / 700.0), step = mmax / 129.0;
  for (int i = 0; i < 130; ++i) {
    const double m = i == 129 ? mmax : i * step;                     // np.linspace(0, mmax, 130)
    mel_f[i] = 700.0 * (pow(10.0, m / 2595.0) - 1.0);
  }
  basis.assign((size_t)n_mels * nbin, 0.f);
  band.assign(2 * n_mels, 0);
  for (int i = 0; i < n_mels; ++i) {
    const double enorm = 2.0 / (mel_f[i + 2] - mel_f[i]);
    int lo = -1, hi = -1;
    for (int k = 0; k < nbin; ++k) {
      const double f = k * (22050.0 / 1024.0);                       // np.linspace(0, sr / 2, 1025): exact steps
      const double lower = -(mel_f[i] - f) / (mel_f[i + 1] - mel_f[i]);
      const double upper = (mel_f[i + 2] - f) / (mel_f[i + 2] - mel_f[i + 1]);
      const float w = (float)(std::max(0.0, std::min(lower, upper)) * enorm);
      basis[(size_t)i * nbin + k] = w;
      if (w != 0.f) { if (lo < 0) lo = k; hi = k; }
    }
    band[i] = lo < 0 ? 0 : lo;
    band[n_mels + i] = lo < 0 ? 0 : hi - lo + 1;
  }
}

// lens (ragged batch): per-item lengths on the device; L is then the capacity (row stride of wav / wav_out)
int restore_forward(Ctx& c, const float* wav, int B, int L, const DropSrc& drop, const int* lens, float* wav_out) {
  const int T = 1 + L / 441;
  if (lens) {
    int* ext = c.ws->alloc<int>((size_t)EXT_LEVELS * B);
    if (!c.dry) VFX_TRY(ragged_extents(lens, B, L, ext, c.st));
    c.ext = ext; c.ext_B = B;
  }
  float* mel = c.ws->alloc<float>((size_t)B * T * 128);
  float* mel_log = c.ws->alloc<float>((size_t)B * T * 128);
  VFX_TRY(frontend_forward(c, wav, B, L, mel, nullptr));
  VFX_TRY(analysis_forward(c, mel, B, T, drop, mel_log));
  VFX_TRY(vocoder_forward(c, mel_log, B, T, 1, wav_out, L, 1.0f));
  return c.rc;
}

// restore_forward on a ragged batch without the vocoder: the extents of lens, the front end, and analysis_forward into
// mel_log_out[B][T_cap][128].  The extent table is allocated in the dry pass too, so that pass sizes the whole call.
int analysis_ragged_forward(Ctx& c, const float* wav, int B, int L_cap, const int* lens, const DropSrc& drop,
                            float* mel_log_out) {
  const int T = 1 + L_cap / 441;
  int* ext = c.ws->alloc<int>((size_t)EXT_LEVELS * B);
  if (!c.dry) VFX_TRY(ragged_extents(lens, B, L_cap, ext, c.st));
  c.ext = ext; c.ext_B = B;
  float* mel = c.ws->alloc<float>((size_t)B * T * 128);
  VFX_TRY(frontend_forward(c, wav, B, L_cap, mel, nullptr));
  return analysis_forward(c, mel, B, T, drop, mel_log_out);
}

// The planner: runs fwd(Ctx&) on a null allocator, which makes no CUDA call, and returns the peak of its workspace.
// *rc receives fwd's status.
template <typename F>
size_t dry_peak(vfx_engine* e, int mode, F&& fwd, int* rc) {
  Bump ws(nullptr, 0);
  Ctx c{e, nullptr, &ws, true, mode};
  const int r = fwd(c);
  *rc = r != VFX_OK ? r : c.rc;
  return ws.peak;
}

// One launching call: fwd(Ctx&) runs dry first, so that a workspace below its peak is refused before the first launch (a
// bump allocator that overflows mid-sequence would alias buffers), then the same fwd runs live.  Because one callable
// serves both passes, the size the call checks is the size its launches use.
template <typename F>
int planned_call(vfx_engine* e, int mode, void* workspace, size_t workspace_bytes, void* stream, F&& fwd) {
  int r;
  const size_t need = dry_peak(e, mode, fwd, &r);
  if (r != VFX_OK) return r;
  if (need > workspace_bytes) {
    set_error("workspace too small: %zu bytes given, this call needs %zu", workspace_bytes, need);
    return VFX_ERR_WORKSPACE;
  }
  Bump ws(workspace, workspace_bytes);
  Ctx c{e, (cudaStream_t)stream, &ws, false, mode};
  VFX_TRY(fwd(c));
  if (ws.overflow) { set_error("workspace too small: need %zu bytes", ws.peak); return VFX_ERR_WORKSPACE; }
  return c.rc;
}

}  // namespace
}  // namespace vfx

// ====================================================================== C ABI
using namespace vfx;

extern "C" {

const char* vfx_last_error(void) { return vfx::g_err; }
int vfx_version(void) { return 100; }

int vfx_engine_create(vfx_engine** out, int device, int precision) {
  VFX_REQUIRE(out != nullptr, "engine_create: out is null");
  VFX_REQUIRE(precision == VFX_PREC_FP32 || precision == VFX_PREC_BF16 || precision == VFX_PREC_TF32 || precision == VFX_PREC_FP16,
              "engine_create: bad precision %d", precision);
  if (device == -1) {   // planning-only: weight-set validation and workspace sizing on a host without a GPU
    vfx_engine* e = new vfx_engine();
    e->device = -1; e->precision = precision;
    *out = e;
    return VFX_OK;
  }
  int ndev = 0;
  VFX_CUDA_CHECK(cudaGetDeviceCount(&ndev));
  VFX_REQUIRE(device >= 0 && device < ndev, "engine_create: device %d not present (%d devices)", device, ndev);
  VFX_CUDA_CHECK(cudaSetDevice(device));
  cudaDeviceProp prop;
  VFX_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("vfx_b200 is built for sm_90a only; device %d is sm_%d%d", device, prop.major, prop.minor);
    return VFX_ERR_UNSUPPORTED;
  }
  vfx_engine* e = new vfx_engine();
  e->device = device; e->precision = precision;
  std::vector<float> win(2048);
  std::vector<float2> tw(1024);
  for (int n = 0; n < 2048; ++n) win[n] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * n / 2048.0));
  for (int k = 0; k < 1024; ++k) {
    tw[k].x = (float)cos(-2.0 * M_PI * k / 2048.0);
    tw[k].y = (float)sin(-2.0 * M_PI * k / 2048.0);
  }
  VFX_CUDA_CHECK(cudaMalloc(&e->d_window, 2048 * sizeof(float)));
  VFX_CUDA_CHECK(cudaMalloc(&e->d_tw, 1024 * sizeof(float2)));
  VFX_CUDA_CHECK(cudaMemcpy(e->d_window, win.data(), 2048 * sizeof(float), cudaMemcpyHostToDevice));
  VFX_CUDA_CHECK(cudaMemcpy(e->d_tw, tw.data(), 1024 * sizeof(float2), cudaMemcpyHostToDevice));
  std::vector<float> basis;
  std::vector<int> band;
  slaney_htk_mel_basis(basis, band);
  VFX_CUDA_CHECK(cudaMalloc(&e->d_obasis, basis.size() * sizeof(float)));
  VFX_CUDA_CHECK(cudaMalloc(&e->d_oband, band.size() * sizeof(int)));
  VFX_CUDA_CHECK(cudaMemcpy(e->d_obasis, basis.data(), basis.size() * sizeof(float), cudaMemcpyHostToDevice));
  VFX_CUDA_CHECK(cudaMemcpy(e->d_oband, band.data(), band.size() * sizeof(int), cudaMemcpyHostToDevice));
  *out = e;
  return VFX_OK;
}

int vfx_engine_destroy(vfx_engine* e) {
  if (!e) return VFX_OK;
  if (e->device >= 0) {
    cudaFree(e->d_window);
    cudaFree(e->d_tw);
    cudaFree(e->d_obasis);
    cudaFree(e->d_oband);
  }
  delete e;
  return VFX_OK;
}

unsigned long long vfx_launch_count(void) { return vfx::g_launches; }
unsigned long long vfx_conv_tma_launch_count(void) { return vfx::g_conv_tma_launches; }
unsigned long long vfx_conv_tma_store_launch_count(void) { return vfx::g_conv_tma_store_launches; }

int vfx_profile_report(vfx_engine* e, char* buf, size_t cap) {
  VFX_REQUIRE(e && buf && cap > 0, "profile_report: bad arguments");
  VFX_REQUIRE(e->device >= 0, "profile_report: planning-only engine");
  VFX_CUDA_CHECK(cudaSetDevice(e->device));
  VFX_CUDA_CHECK(cudaDeviceSynchronize());
  struct Agg { double ms = 0, flops = 0, bytes = 0; long n = 0; };
  std::vector<std::pair<std::string, Agg>> agg;
  for (auto& r : e->prof) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, r.a, r.b);
    cudaEventDestroy(r.a); cudaEventDestroy(r.b);
    size_t i = 0;
    for (; i < agg.size(); ++i) if (agg[i].first == r.tag) break;
    if (i == agg.size()) agg.push_back({r.tag, Agg()});
    agg[i].second.ms += ms; agg[i].second.flops += r.flops; agg[i].second.bytes += r.bytes; agg[i].second.n++;
  }
  e->prof.clear();
  std::string out;
  char line[256];
  for (auto& a : agg) {
    snprintf(line, sizeof(line), "%s %ld %.6f %.6e %.6e\n", a.first.c_str(), a.second.n, a.second.ms, a.second.flops,
             a.second.bytes);
    out += line;
  }
  snprintf(buf, cap, "%s", out.c_str());
  return VFX_OK;
}

int vfx_engine_set_option(vfx_engine* e, const char* key, int value) {
  VFX_REQUIRE(e && key, "set_option: null argument");
  if (!strcmp(key, "use_tc")) { e->use_tc = value; return VFX_OK; }
  if (!strcmp(key, "profile")) { e->profile = value; return VFX_OK; }
  if (!strcmp(key, "fuse_pairs")) { e->fuse_pairs = value; return VFX_OK; }
  if (!strcmp(key, "tf32_stream")) { e->tf32_stream = value; return VFX_OK; }
  set_error("set_option: unknown key '%s'", key);
  return VFX_ERR_INVALID;
}

int vfx_engine_set_tensor(vfx_engine* e, const char* name, const void* dev_ptr, size_t bytes) {
  VFX_REQUIRE(e && name && dev_ptr, "set_tensor: null argument");
  e->tensors[name] = vfx::Tensor{dev_ptr, bytes};
  e->finalized = false;
  return VFX_OK;
}

// The restore planner (L > 0) or the frames planner (B items of T frames: analysis + vocoder, or the vocoder alone on a
// vocoder-only engine), in mode 2, whose batch statistics take the most workspace.  The slack also holds
// vfx_restore_ragged's extent table, so one workspace size serves both entry points.
static size_t dry_run(vfx_engine* e, int B, int T, int L, int* rc) {
  const size_t peak = dry_peak(e, VFX_MODE_TRAIN_BN, [&](Ctx& c) {
    if (L > 0) return restore_forward(c, nullptr, B, L, DropSrc(), nullptr, nullptr);
    float* mel = c.ws->alloc<float>((size_t)B * T * 128);
    const bool voc_only = e->finalized && !(e->parts & VFX_PART_ANALYSIS);
    const int r = voc_only ? VFX_OK : analysis_forward(c, mel, B, T, DropSrc(), mel);
    return r != VFX_OK ? r : vocoder_forward(c, mel, B, T, 1, nullptr, -1, 1.f);
  }, rc);
  return peak + std::max<size_t>(4096, ext_table_bytes(B));
}

int vfx_engine_finalize(vfx_engine* e) {
  VFX_REQUIRE(e, "finalize: null engine");
  e->missing.clear();
  int r, r2;
  dry_run(e, 1, 64, 0, &r);
  // also the front-end tables
  dry_peak(e, VFX_MODE_EVAL, [](Ctx& c) { return frontend_forward(c, nullptr, 1, 44100, nullptr, nullptr); }, &r2);
  if (r == VFX_OK) r = r2;
  if (!e->missing.empty()) {
    // The reference's stand-alone Vocoder class (voicefixer/vocoder/base.py:10-40) loads the synthesis checkpoint only.
    // An engine that holds nothing but "voc." tensors, all of them present, is complete for vfx_vocoder /
    // vfx_vocoder_cond; the analysis-side entry points refuse it.
    bool voc_only = !e->tensors.empty();
    for (auto& kv : e->tensors) if (kv.first.rfind("voc.", 0) != 0) voc_only = false;
    if (voc_only) {
      std::vector<std::string> analysis_missing;
      analysis_missing.swap(e->missing);
      int rv;
      dry_peak(e, VFX_MODE_EVAL, [](Ctx& c) {
        float* mel = c.ws->alloc<float>((size_t)64 * 128);
        return vocoder_forward(c, mel, 1, 64, 1, nullptr, -1, 1.f);
      }, &rv);
      if (rv == VFX_OK && e->missing.empty()) {
        e->parts = VFX_PART_VOCODER;
        e->finalized = true;
        return VFX_OK;
      }
      if (e->missing.empty()) return rv;     // e.g. a tensor of the wrong size: message already set
    }
    std::string s = "missing weight tensors:";
    for (size_t i = 0; i < e->missing.size() && i < 12; ++i) s += " " + e->missing[i];
    if (e->missing.size() > 12) s += " ...";
    set_error("%s (%zu total)", s.c_str(), e->missing.size());
    return VFX_ERR_MISSING_WEIGHT;
  }
  if (r != VFX_OK) return r;
  e->parts = VFX_PART_ANALYSIS | VFX_PART_VOCODER;
  e->finalized = true;
  return VFX_OK;
}

size_t vfx_workspace_bytes(const vfx_engine* e, int B, int L) {
  if (!e || B <= 0 || L <= 1024) return 0;
  if (e->finalized && !(e->parts & VFX_PART_ANALYSIS)) return 0;   // restore() needs the analysis weights
  int rc;
  return dry_run(const_cast<vfx_engine*>(e), B, 0, L, &rc);
}

size_t vfx_workspace_bytes_frames(const vfx_engine* e, int B, int T) {
  if (!e || B <= 0 || T <= 0) return 0;
  int rc;
  return dry_run(const_cast<vfx_engine*>(e), B, T, 0, &rc);
}

// oracle(): the planner is the dry pass of the whole call (front end, frame table, generator)
size_t vfx_oracle_workspace_bytes(const vfx_engine* e, int B, int L_cap) {
  if (!e || B <= 0 || L_cap <= 0 || (long long)(1 + L_cap / 441 + 5) * 441 > 0x7fffffffLL) return 0;
  int rc;
  const size_t peak = dry_peak(const_cast<vfx_engine*>(e), VFX_MODE_EVAL,
                               [&](Ctx& c) { return oracle_forward(c, nullptr, B, L_cap, nullptr, 1.f, nullptr); }, &rc);
  return rc == VFX_OK ? peak : 0;
}

#define VFX_ENTER(e)                                                                     \
  VFX_REQUIRE((e) != nullptr, "null engine");                                            \
  VFX_REQUIRE((e)->finalized, "engine not finalized (call vfx_engine_finalize)");        \
  VFX_REQUIRE((e)->device >= 0, "planning-only engine (device -1) cannot launch work");  \
  VFX_CUDA_CHECK(cudaSetDevice((e)->device))

#define VFX_NEED_ANALYSIS(e)                                                              \
  VFX_REQUIRE((e)->parts & VFX_PART_ANALYSIS,                                            \
              "this engine holds the vocoder weights only (stand-alone Vocoder); the analysis module is not loaded")

int vfx_frontend_mel(vfx_engine* e, const float* wav, int B, int L, float* mel, float* sp_out, void* stream) {
  VFX_ENTER(e);
  VFX_NEED_ANALYSIS(e);
  VFX_REQUIRE(wav && mel && B > 0, "frontend: bad arguments");
  // no workspace: an allocation the front end might make is refused by the dry pass
  return planned_call(e, VFX_MODE_EVAL, nullptr, 0, stream,
                      [&](Ctx& c) { return frontend_forward(c, wav, B, L, mel, sp_out); });
}

int vfx_analysis(vfx_engine* e, const float* mel, int B, int T, int mode, const uint8_t* drop_masks,
                 float* mel_log_out, void* workspace, size_t workspace_bytes, void* stream) {
  VFX_ENTER(e);
  VFX_NEED_ANALYSIS(e);
  VFX_REQUIRE(mel && mel_log_out && B > 0 && T > 0 && workspace, "analysis: bad arguments");
  VFX_REQUIRE(mode == VFX_MODE_EVAL || mode == VFX_MODE_TRAIN_BN, "analysis: bad mode %d", mode);
  DropSrc drop;
  drop.masks = drop_masks;
  return planned_call(e, mode, workspace, workspace_bytes, stream,
                      [&](Ctx& c) { return analysis_forward(c, mel, B, T, drop, mel_log_out); });
}

// The key table of a seeded call: checked before any launch, since the dropout kernel's grid holds B in y
#define VFX_DROP_KEYS(what)                                                                                          \
  VFX_REQUIRE(keys && ((uintptr_t)keys & 7) == 0, what ": keys must be a non-null, 8-byte aligned device pointer");   \
  VFX_REQUIRE(B <= 65535, what ": B=%d exceeds 65535", B)

int vfx_analysis_seeded(vfx_engine* e, const float* mel, int B, int T, const vfx_drop_key* keys, float* mel_log_out,
                        void* workspace, size_t workspace_bytes, void* stream) {
  VFX_DROP_KEYS("analysis_seeded");
  VFX_ENTER(e);
  VFX_NEED_ANALYSIS(e);
  VFX_REQUIRE(mel && mel_log_out && B > 0 && T > 0 && workspace, "analysis_seeded: bad arguments");
  DropSrc drop;
  drop.keys = keys;
  return planned_call(e, VFX_MODE_TRAIN_BN, workspace, workspace_bytes, stream,
                      [&](Ctx& c) { return analysis_forward(c, mel, B, T, drop, mel_log_out); });
}

int vfx_vocoder(vfx_engine* e, const float* mel, int B, int T, int input_is_log, float* wav_out, int trim_len,
                float scale, void* workspace, size_t workspace_bytes, void* stream) {
  VFX_ENTER(e);
  VFX_REQUIRE(mel && wav_out && B > 0 && T > 0 && workspace, "vocoder: bad arguments");
  return planned_call(e, VFX_MODE_EVAL, workspace, workspace_bytes, stream,
                      [&](Ctx& c) { return vocoder_forward(c, mel, B, T, input_is_log, wav_out, trim_len, scale); });
}

int vfx_vocoder_cond(vfx_engine* e, const float* cond, int B, int Tc, float* wav_out, int trim_len, float scale,
                     void* workspace, size_t workspace_bytes, void* stream) {
  VFX_ENTER(e);
  VFX_REQUIRE(cond && wav_out && B > 0 && Tc >= 4 && workspace, "vocoder_cond: bad arguments");
  return planned_call(e, VFX_MODE_EVAL, workspace, workspace_bytes, stream,
                      [&](Ctx& c) { return vocoder_cond_forward(c, cond, B, Tc, wav_out, trim_len, scale); });
}

int vfx_vocoder_ragged(vfx_engine* e, const float* mel, int B, int T_cap, const int* frames, int input_is_log,
                       float* wav_out, float scale, void* workspace, size_t workspace_bytes, void* stream) {
  VFX_ENTER(e);
  VFX_REQUIRE(mel && frames && wav_out && B > 0 && T_cap > 0 && workspace, "vocoder_ragged: bad arguments");
  return planned_call(e, VFX_MODE_EVAL, workspace, workspace_bytes, stream, [&](Ctx& c) {
    return vocoder_ragged_forward(c, mel, B, T_cap, frames, input_is_log, wav_out, scale);
  });
}

#define VFX_ORACLE_ARGS(what)                                                                                       \
  VFX_REQUIRE(wav && B > 0 && L_cap > 0 && workspace, what ": bad arguments");                                       \
  VFX_REQUIRE((long long)(1 + L_cap / 441 + 5) * 441 <= 0x7fffffffLL, what ": L_cap=%d is too long", L_cap)

int vfx_oracle_cond(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, float* cond_out, void* workspace,
                    size_t workspace_bytes, void* stream) {
  VFX_ENTER(e);
  VFX_ORACLE_ARGS("oracle_cond");
  VFX_REQUIRE(cond_out, "oracle_cond: cond_out is null");
  return planned_call(e, VFX_MODE_EVAL, workspace, workspace_bytes, stream,
                      [&](Ctx& c) { return oracle_cond_forward(c, wav, B, L_cap, lens, cond_out); });
}

int vfx_oracle(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, float scale, float* wav_out,
               void* workspace, size_t workspace_bytes, void* stream) {
  VFX_ENTER(e);
  VFX_ORACLE_ARGS("oracle");
  VFX_REQUIRE(wav_out, "oracle: wav_out is null");
  return planned_call(e, VFX_MODE_EVAL, workspace, workspace_bytes, stream,
                      [&](Ctx& c) { return oracle_forward(c, wav, B, L_cap, lens, scale, wav_out); });
}

static int restore_entry(vfx_engine* e, const float* wav, int B, int L, int mode, const DropSrc& drop,
                         const int* lens, float* wav_out, void* workspace, size_t workspace_bytes, void* stream) {
  VFX_ENTER(e);
  VFX_NEED_ANALYSIS(e);
  VFX_REQUIRE(wav && wav_out && B > 0 && workspace, "restore: bad arguments");
  VFX_REQUIRE(mode == VFX_MODE_EVAL || mode == VFX_MODE_TRAIN_BN, "restore: bad mode %d", mode);
  VFX_REQUIRE(L > 1024, "restore: L=%d must exceed 1024 samples", L);
  return planned_call(e, mode, workspace, workspace_bytes, stream,
                      [&](Ctx& c) { return restore_forward(c, wav, B, L, drop, lens, wav_out); });
}

int vfx_restore(vfx_engine* e, const float* wav, int B, int L, int mode, const uint8_t* drop_masks,
                float* wav_out, void* workspace, size_t workspace_bytes, void* stream) {
  DropSrc drop;
  drop.masks = drop_masks;
  return restore_entry(e, wav, B, L, mode, drop, nullptr, wav_out, workspace, workspace_bytes, stream);
}

int vfx_restore_ragged_mode(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, int mode,
                            const uint8_t* drop_masks, float* wav_out, void* workspace, size_t workspace_bytes,
                            void* stream) {
  VFX_REQUIRE(lens, "restore_ragged: lens is null");
  DropSrc drop;
  drop.masks = drop_masks;
  return restore_entry(e, wav, B, L_cap, mode, drop, lens, wav_out, workspace, workspace_bytes, stream);
}

int vfx_restore_seeded(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, const vfx_drop_key* keys,
                       float* wav_out, void* workspace, size_t workspace_bytes, void* stream) {
  VFX_DROP_KEYS("restore_seeded");
  DropSrc drop;
  drop.keys = keys;
  return restore_entry(e, wav, B, L_cap, VFX_MODE_TRAIN_BN, drop, lens, wav_out, workspace, workspace_bytes, stream);
}

int vfx_restore_ragged(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, float* wav_out,
                       void* workspace, size_t workspace_bytes, void* stream) {
  return vfx_restore_ragged_mode(e, wav, B, L_cap, lens, VFX_MODE_EVAL, nullptr, wav_out, workspace, workspace_bytes,
                                 stream);
}

// the analysis half of a ragged restore: the dry pass in mode 2, whose batch statistics take the most workspace; 0 for a
// shape vfx_analysis_ragged refuses, as vfx_workspace_bytes
size_t vfx_analysis_workspace_bytes(const vfx_engine* e, int B, int L_cap) {
  if (!e || B <= 0 || L_cap <= 1024) return 0;
  if (e->finalized && !(e->parts & VFX_PART_ANALYSIS)) return 0;
  int rc;
  const size_t peak = dry_peak(const_cast<vfx_engine*>(e), VFX_MODE_TRAIN_BN, [&](Ctx& c) {
    return analysis_ragged_forward(c, nullptr, B, L_cap, nullptr, DropSrc(), nullptr);
  }, &rc);
  return rc == VFX_OK ? peak : 0;
}

int vfx_analysis_ragged(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, int mode,
                        const uint8_t* drop_masks, const vfx_drop_key* keys, float* mel_log_out, void* workspace,
                        size_t workspace_bytes, void* stream) {
  VFX_REQUIRE(wav && lens && mel_log_out && B > 0 && workspace, "analysis_ragged: bad arguments");
  VFX_REQUIRE(mode == VFX_MODE_EVAL || mode == VFX_MODE_TRAIN_BN, "analysis_ragged: bad mode %d (mode 1 is "
              "vfx_hf_cut_ragged, then mode 0)", mode);
  VFX_REQUIRE(L_cap > 1024, "analysis_ragged: L_cap=%d must exceed 1024 samples", L_cap);
  VFX_REQUIRE(!(drop_masks && keys), "analysis_ragged: drop_masks and keys are two sources of the same masks: give one "
              "of them");
  if (keys) {
    VFX_REQUIRE(mode == VFX_MODE_TRAIN_BN, "analysis_ragged: keys are mode 2's dropout; mode is %d", mode);
    VFX_DROP_KEYS("analysis_ragged");
  }
  VFX_ENTER(e);
  VFX_NEED_ANALYSIS(e);
  DropSrc drop;
  drop.masks = drop_masks;
  drop.keys = keys;
  return planned_call(e, mode, workspace, workspace_bytes, stream, [&](Ctx& c) {
    return analysis_ragged_forward(c, wav, B, L_cap, lens, drop, mel_log_out);
  });
}

size_t vfx_hf_cut_workspace_bytes(int B, int L) { return B < 0 || L < 0 ? 0 : hf_cut_workspace(B, L); }

int vfx_hf_cut(vfx_engine* e, const float* wav, int B, int L, float ratio, float* wav_out, int* cut_bins,
               void* workspace, size_t workspace_bytes, void* stream) {
  VFX_ENTER(e);
  return hf_cut(wav, B, L, nullptr, ratio, e->d_window, e->d_tw, wav_out, nullptr, cut_bins, workspace, workspace_bytes,
                (cudaStream_t)stream);
}

int vfx_hf_cut_ragged(vfx_engine* e, const float* wav, int B, int L_cap, const int* lens, float ratio, float* wav_out,
                      int* lens_out, int* cut_bins, void* workspace, size_t workspace_bytes, void* stream) {
  VFX_ENTER(e);
  VFX_REQUIRE(lens, "hf_cut_ragged: lens is null");
  return hf_cut(wav, B, L_cap, lens, ratio, e->d_window, e->d_tw, wav_out, lens_out, cut_bins, workspace,
                workspace_bytes, (cudaStream_t)stream);
}

size_t vfx_resample_workspace_bytes(int B) {
  if (B <= 0) return 0;
  int rc;
  const size_t peak = dry_peak(nullptr, VFX_MODE_EVAL, [&](Ctx& c) {
    return resample_forward(c, nullptr, nullptr, nullptr, B, 1, nullptr, nullptr);
  }, &rc);
  return rc == VFX_OK ? peak : 0;
}

int vfx_resample(vfx_engine* e, const float* x, long long x_elems, const float* h, long long h_elems,
                 const vfx_resample_item* items_host, int B, float* y, int L_cap, int* lens_out,
                 void* workspace, size_t workspace_bytes, void* stream) {
  VFX_ENTER(e);
  VFX_REQUIRE(items_host && y && B > 0 && B <= 65535 && L_cap > 0 && workspace && x_elems >= 0 && h_elems >= 0,
              "resample: bad arguments");
  VFX_REQUIRE(x || x_elems == 0, "resample: x is null");
  VFX_REQUIRE(h || h_elems == 0, "resample: h is null");
  for (int b = 0; b < B; ++b) VFX_TRY(check_resample_item(items_host[b], b, x_elems, h_elems, L_cap));
  return planned_call(e, VFX_MODE_EVAL, workspace, workspace_bytes, stream,
                      [&](Ctx& c) { return resample_forward(c, x, h, items_host, B, L_cap, y, lens_out); });
}

size_t vfx_resample_src_workspace_bytes(int B) {
  if (B <= 0) return 0;
  int rc;
  const size_t peak = dry_peak(nullptr, VFX_MODE_EVAL, [&](Ctx& c) {
    return resample_src_forward(c, nullptr, nullptr, B, 1, nullptr, nullptr);
  }, &rc);
  return rc == VFX_OK ? peak : 0;
}

int vfx_resample_src(vfx_engine* e, const float* h, long long h_elems, const vfx_resample_src_item* items_host, int B,
                     float* y, int L_cap, int* lens_out, void* workspace, size_t workspace_bytes, void* stream) {
  VFX_ENTER(e);
  VFX_REQUIRE(items_host && y && B > 0 && B <= 65535 && L_cap > 0 && workspace && h_elems >= 0,
              "resample_src: bad arguments");
  VFX_REQUIRE(h || h_elems == 0, "resample_src: h is null");
  for (int b = 0; b < B; ++b) VFX_TRY(check_resample_src_item(items_host[b], b, h_elems, L_cap));
  return planned_call(e, VFX_MODE_EVAL, workspace, workspace_bytes, stream,
                      [&](Ctx& c) { return resample_src_forward(c, h, items_host, B, L_cap, y, lens_out); });
}

size_t vfx_scatter_rows_workspace_bytes(int B) {
  if (B <= 0) return 0;
  int rc;
  const size_t peak = dry_peak(nullptr, VFX_MODE_EVAL, [&](Ctx& c) {
    return scatter_rows_forward(c, nullptr, B, 1, nullptr, 1);
  }, &rc);
  return rc == VFX_OK ? peak : 0;
}

int vfx_scatter_rows(const float* x, int B, long long ldx, const vfx_scatter_item* items_host, void* workspace,
                     size_t workspace_bytes, void* stream) {
  VFX_REQUIRE(x && items_host && B > 0 && B <= 65535 && ldx > 0 && workspace, "scatter_rows: bad arguments");
  int max_len;
  VFX_TRY(check_scatter_items(items_host, B, ldx, &max_len));
  if (max_len == 0) return VFX_OK;
  return planned_call(nullptr, VFX_MODE_EVAL, workspace, workspace_bytes, stream,
                      [&](Ctx& c) { return scatter_rows_forward(c, x, B, ldx, items_host, max_len); });
}

size_t vfx_pack_pcm16_workspace_bytes(int B) {
  if (B <= 0) return 0;
  int rc;
  const size_t peak = dry_peak(nullptr, VFX_MODE_EVAL, [&](Ctx& c) {
    return pack_pcm16_forward(c, nullptr, B, nullptr, 1);
  }, &rc);
  return rc == VFX_OK ? peak : 0;
}

int vfx_pack_pcm16(const vfx_pcm16_item* items_host, int B, short* y, long long y_elems, void* workspace,
                   size_t workspace_bytes, void* stream) {
  VFX_REQUIRE(items_host && y && B > 0 && B <= 65535 && y_elems > 0 && workspace, "pack_pcm16: bad arguments");
  long long max_n;
  VFX_TRY(check_pcm16_items(items_host, B, y_elems, &max_n));
  return planned_call(nullptr, VFX_MODE_EVAL, workspace, workspace_bytes, stream,
                      [&](Ctx& c) { return pack_pcm16_forward(c, items_host, B, y, max_n); });
}

int vfx_conv_gemm(int precision, int impl, const vfx_conv_desc* d, void* stream) {
  VFX_REQUIRE(d, "conv_gemm: null descriptor");
  if (impl == 1) {
    VFX_REQUIRE(precision == VFX_PREC_BF16 || precision == VFX_PREC_TF32 || precision == VFX_PREC_FP16,
                "conv_gemm: the tensor-core implementation takes bf16, fp16 or tf32 operands");
    return conv_gemm_tc(precision, *d, (cudaStream_t)stream);
  }
  return conv_gemm_simt(precision, *d, (cudaStream_t)stream);
}

size_t vfx_resstack_pair_scratch_bytes(void) { return resstack_pair_scratch_bytes(); }

int vfx_resstack_pair(const vfx_pair_desc* d, void* stream) {
  VFX_REQUIRE(d, "resstack_pair: null descriptor");
  const int r = resstack_pair(*d, (cudaStream_t)stream);
  if (r == VFX_ERR_UNSUPPORTED)
    set_error("resstack_pair: unsupported (bf16 / fp16: C = 64 or 128; tf32: C = 64 with stream_enc and x_out; "
              "16-byte aligned tensors; the blocked form takes no lens)");
  return r;
}

int vfx_gru_layer(const float* gi, const float* whh_t, const float* bhh, int B, int T, float* out, void* stream) {
  return gru_layer(gi, whh_t, bhh, B, T, nullptr, out, (cudaStream_t)stream);
}

int vfx_gru_layer_ragged(const float* gi, const float* whh_t, const float* bhh, int B, int T, const int* lens,
                         float* out, void* stream) {
  VFX_REQUIRE(lens, "gru_layer_ragged: lens is null");
  return gru_layer(gi, whh_t, bhh, B, T, lens, out, (cudaStream_t)stream);
}

int vfx_bn_stats(const float* x, long long x_sB, long long ldx, int B, long long P, int C, int bn_C, const float* gamma,
                 const float* beta, float* scale, float* shift, double* acc, const int* seq, int per_row, void* stream) {
  return bn_stats(x, x_sB, ldx, B, P, C, bn_C, gamma, beta, scale, shift, acc, seq, per_row, (cudaStream_t)stream);
}

int vfx_bn_act(int precision, const float* x, long long x_sB, long long ldx, int B, long long P, int C,
               const float* scale, const float* shift, int bn_C, int stat_sB, int act, float act_param, void* y,
               long long y_sB, long long ldy, void* stream) {
  return bn_act(precision, x, x_sB, ldx, B, P, C, scale, shift, bn_C, stat_sB, act, act_param, y, y_sB, ldy,
                (cudaStream_t)stream);
}

int vfx_dropout_apply(float* x, const uint8_t* keep, long long n, void* stream) {
  return dropout_apply(x, keep, n, (cudaStream_t)stream);
}

int vfx_dropout_seeded(float* x, int B, int T, const vfx_drop_key* keys, int layer, void* stream) {
  return dropout_seeded(x, B, T, keys, layer, (cudaStream_t)stream);
}

int vfx_avgpool2x2(const float* x, long long x_sB, long long x_sH, long long x_sW, int B, int H, int W, int C, float* y,
                   void* stream) {
  return avgpool2x2(x, x_sB, x_sH, x_sW, B, H, W, C, y, (cudaStream_t)stream);
}

int vfx_mask_log_pack(const float* lin, const float* mel, int B, int T, int Tp, const int* ext_frames, float* xlog,
                      float* unet_in, void* stream) {
  return mask_log_pack(lin, mel, B, T, Tp, ext_frames, xlog, unet_in, (cudaStream_t)stream);
}

int vfx_unet_head(const float* x, int B, int T, int Tp, const float* w, const float* bias, const float* xlog, float* out,
                  void* stream) {
  return unet_head(x, B, T, Tp, w, bias, xlog, out, (cudaStream_t)stream);
}

int vfx_voc_normalize(const float* mel, int B, int T, int Tc, const int* ext_frames, int input_is_log, const float* tab,
                      void* cond, int precision, void* stream) {
  return voc_normalize(mel, B, T, Tc, ext_frames, input_is_log, tab, cond, precision, (cudaStream_t)stream);
}

int vfx_reflect_pad3(void* buf, int B, int L, int C, const int* ext_len, int precision, void* stream) {
  return reflect_pad3(buf, B, L, C, ext_len, precision, (cudaStream_t)stream);
}

int vfx_voc_post(const float* x, int B, int L, const float* w, const float* bias, int lo, int out_len, const int* ext_gen,
                 const int* ext_len, float scale, float* out, void* stream) {
  return voc_post(x, B, L, w, bias, lo, out_len, ext_gen, ext_len, scale, out, (cudaStream_t)stream);
}

int vfx_cast_rows(const float* x, long long n, void* y, int precision, void* stream) {
  return cast_rows(x, n, y, precision, (cudaStream_t)stream);
}

int vfx_ragged_extents(const int* lens, int B, int L_cap, int* ext, void* stream) {
  return ragged_extents(lens, B, L_cap, ext, (cudaStream_t)stream);
}

int vfx_frame_extents(const int* frames, int B, int T_cap, int* ext, void* stream) {
  return frame_extents(frames, B, T_cap, ext, (cudaStream_t)stream);
}

}  // extern "C"

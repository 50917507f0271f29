"""CPU oracle for the VoiceFixer restore()/Vocoder path.  TEST INFRASTRUCTURE ONLY.

A plain PyTorch-fp32 (CPU) restatement of the reference algorithm, function by function,
each citing the reference file:line it follows (paths relative to /root/reference).  Only
`tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` leg may
import this module; the product path (`voicefixer_b200`) never does and fails loudly when its
CUDA extension is missing.

Parity pin: this restatement is checked against the UNMODIFIED reference nn.Modules imported
from /root/reference (tests/golden/make_golden.py, run in the build container) and against the
committed outputs of those modules (tests/golden/*.npz).  The reference's own FLAC golden files
(test/utterance/target/*.flac) need the Zenodo checkpoints, which are not available offline;
they pin only the length arithmetic here (tests/test_oracle.py::test_fixture_lengths).

All functions take flat state dicts in the reference checkpoint layout:
  ana: keys of vf.ckpt           ("generator.denoiser.*", "generator.unet.*", "mel.fb",
                                  "f_helper.stft.conv_real.weight", ...)
  voc: keys of ckpt["generator"] ("condnet.0.bias", "...parametrizations.weight.original0/1"
                                  or old-style "...weight_g/weight_v")

Arithmetic follows the dtype and device of the state dicts: given float64 copies of the checkpoints (on any device),
every function computes in float64 there, on the float32 samples it is given.  Constants the reference defines in
float32 (the vocoder's mel weights and min_level, the Slaney basis, the checkpoint's STFT kernels) keep their float32
values, converted exactly.  With float32 state dicts the results are the fp32 oracle's, bit for bit.

Operand rounding (`operand_rounding`): a model of the engine's tensor-core precisions.  Inside the context, the
operands of every dense contraction the engine runs on the tensor cores are rounded to tf32 / fp16 / bf16 where the
engine rounds them (csrc/engine.cu, weights.py); accumulation stays in the state dicts' dtype.  Rounded:
  - every Conv1d / Conv2d / ConvTranspose input and weight of the UNet and the vocoder (the operand buffers A0 / Hh /
    U / opA / opH / opX and the conditions, cast by their producers' epilogues), including the shortcut convs' raw x;
  - the denoiser's Linear inputs act(bn(x)) and weights;
  - the GRU input projections: bn(x) and layer 0's output y0 (dn_operand), and the w_ih weights;
  - in eval mode, UNet ConvBlockRes.conv1 with bn2 folded into it: the engine rounds round(w1 * bn2.scale) and adds
    bn2.shift in fp32 (weights._conv_block's conv1f), so the model does the same.
Not rounded: the STFT front end (an fp32 FFT), the GRU recurrence, the UNet head after_conv2 (unet.head.w is fp32),
the vocoder post conv generator.16 (voc.post.w is fp32 and reads plain x'), BatchNorm statistics, residual adds,
the denoiser mask and the log.  Tensors the engine keeps in fp32 between contractions pass through
`OperandRounding.stored` (identity here), so that a test can model a wiring fault that would store one in the
operand format.
"""
import contextlib
import math
import numpy as np
import torch
import torch.nn.functional as F

SR = 44100
N_FFT = 2048
HOP = 441
N_MEL = 128
SEG_LEN = SR * 30                      # voicefixer/base.py:116
UPSAMPLE_SCALES = (7, 7, 3, 3)         # voicefixer/vocoder/config.py:20
MEL_W_A, MEL_W_B = 18.8927416350036, 0.0269863588184314   # vocoder/config.py:301,310
BN_EPS = 1e-5                          # nn.BatchNorm2d default, every BatchNorm of the analysis model


# --------------------------------------------------------------------------- operand rounding
def round_tf32(x):
    """Nearest tf32 value, ties away from zero (PTX cvt.rna.tf32.f32), in x's dtype (float32 or float64)."""
    if x.dtype == torch.float64:
        i = x.contiguous().view(torch.int64)
        return ((i + (1 << 41)) & ~((1 << 42) - 1)).view(torch.float64)
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def trunc_tf32(x):
    """Truncation to tf32: what the tensor core does to an fp32 operand that was not rounded."""
    if x.dtype == torch.float64:
        i = x.contiguous().view(torch.int64)
        return (i & ~((1 << 42) - 1)).view(torch.float64)
    i = x.contiguous().view(torch.int32)
    return (i & ~0x1FFF).view(torch.float32)


def _via(dtype):
    return lambda x: x.to(dtype).to(x.dtype)


ROUNDINGS = {"tf32": round_tf32, "tf32-trunc": trunc_tf32, "fp16": _via(torch.float16), "bf16": _via(torch.bfloat16)}


class OperandRounding:
    """The operand format of one engine precision: `operand` rounds a contraction's input or weight, `stored` is
    applied to the tensors the engine keeps in fp32 between contractions ("vocoder.residual": the ResStack stream x
    after the up-sampler and after each pair; "unet.block": each ConvBlockRes output).  Subclass to model faults.

    `where` names the rounding point of `operand`:
      "denoiser.input" / "denoiser.weight"  the denoiser's Linear layers
      "gru.input" / "gru.weight"            the GRU input projections: bn(x) or layer 0's output, and w_ih
      "unet.bn_act"    act(bn(x)) read by a UNet conv: ConvBlockRes.conv1 and the decoders' ConvTranspose, and in
                       train mode ConvBlockRes.conv2 (written by bn_act; in eval mode by the producing conv's epilogue)
      "unet.act"       ConvBlockRes.conv2's input in eval mode (conv1's epilogue, bn2 folded)
      "unet.shortcut"  the shortcut conv's raw x
      "unet.weight"    every UNet conv weight (the folded conv1 weight in eval mode)
      "vocoder.cond"   the conditions read by condnet.0 (voc_normalize, or the oracle front end)
      "vocoder.act"    every other vocoder conv input
      "vocoder.weight" every vocoder conv weight"""

    def __init__(self, fmt):
        if fmt not in ROUNDINGS:
            raise ValueError(f"unknown operand format '{fmt}' (one of {sorted(ROUNDINGS)})")
        self.fmt = fmt
        self.round = ROUNDINGS[fmt]

    def operand(self, x, where):
        return self.round(x)

    def stored(self, x, where):
        return x


_rounding = None


@contextlib.contextmanager
def operand_rounding(model):
    """Runs the oracle with the operand rounding `model` (an OperandRounding or a format name) inside the block."""
    global _rounding
    saved = _rounding
    _rounding = OperandRounding(model) if isinstance(model, str) else model
    try:
        yield _rounding
    finally:
        _rounding = saved


def _op(x, where):
    return x if _rounding is None else _rounding.operand(x, where)


def _stored(x, where):
    return x if _rounding is None else _rounding.stored(x, where)


# --------------------------------------------------------------------------- front end
def stft_mag(wav, ana):
    """wav (B, L) -> sp (B, 1, T, 1025).
    torchlibrosa.stft.STFT.forward as built at tools/modules/fDomainHelper.py:23-31 (DFT-matrix
    conv1d, stride 441, reflect pad 1024) and spectrogram_phase fDomainHelper.py:81-86 with
    eps=1e-8 (wav_to_spectrogram_phase :88)."""
    kr = ana["f_helper.stft.conv_real.weight"]
    x = wav.to(dtype=kr.dtype, device=kr.device)[:, None, :]
    x = F.pad(x, (N_FFT // 2, N_FFT // 2), mode="reflect")
    real = F.conv1d(x, kr, stride=HOP)
    imag = F.conv1d(x, ana["f_helper.stft.conv_imag.weight"], stride=HOP)
    real = real[:, None].transpose(2, 3)
    imag = imag[:, None].transpose(2, 3)
    return torch.clamp(real ** 2 + imag ** 2, 1e-8, np.inf) ** 0.5


def mel_scale(sp, ana):
    """sp (B,1,T,1025) -> mel (B,1,T,128): tools/mel_scale.py:63-77 through base.py:83."""
    return torch.matmul(sp, ana["mel.fb"])


def frontend(wav, ana):
    """VoiceFixer._pre, base.py:78-85."""
    sp = stft_mag(wav, ana)
    return sp, mel_scale(sp, ana)


# --------------------------------------------------------------------------- denoiser
def _bn1(x, ana, prefix, train):
    """nn.BatchNorm2d(1) on (B,1,T,F); eval: running stats; train: biased batch stats over
    (N,H,W).  restorer/model.py:69-99 (BatchNorm2d(1) members)."""
    w, b = ana[prefix + ".weight"], ana[prefix + ".bias"]
    if train:
        return F.batch_norm(x, None, None, w, b, True, 0.0, BN_EPS)
    return F.batch_norm(x, ana[prefix + ".running_mean"], ana[prefix + ".running_var"], w, b,
                        False, 0.0, BN_EPS)


def gru_layer_dir(x, w_ih, w_hh, b_ih, b_hh, reverse):
    """One direction of one torch.nn.GRU layer, batch_first.  x (B,T,I) -> (B,T,H).
    Gate order r,z,n; n = tanh(W_in x + b_in + r*(W_hn h + b_hn)); h' = (1-z)*n + z*h."""
    B, T, _ = x.shape
    H = w_hh.shape[1]
    gi = _op(x, "gru.input") @ _op(w_ih, "gru.weight").t() + b_ih
    h = x.new_zeros(B, H)
    out = x.new_zeros(B, T, H)
    steps = range(T - 1, -1, -1) if reverse else range(T)
    for t in steps:
        gh = h @ w_hh.t() + b_hh
        i_r, i_z, i_n = gi[:, t].chunk(3, 1)
        h_r, h_z, h_n = gh.chunk(3, 1)
        r = torch.sigmoid(i_r + h_r)
        z = torch.sigmoid(i_z + h_z)
        n = torch.tanh(i_n + r * h_n)
        h = (1 - z) * n + z * h
        out[:, t] = h
    return out


def bn_gru(x, ana, prefix, train):
    """BN_GRU.forward restorer/model.py:56-62: BN2d(1) -> 2-layer bidirectional GRU(512->256)."""
    x = _bn1(x, ana, prefix + ".bn", train).squeeze(1)
    for layer in (0, 1):
        outs = []
        for suffix, rev in (("", False), ("_reverse", True)):
            g = prefix + ".gru."
            outs.append(gru_layer_dir(x, ana[g + f"weight_ih_l{layer}{suffix}"],
                                      ana[g + f"weight_hh_l{layer}{suffix}"],
                                      ana[g + f"bias_ih_l{layer}{suffix}"],
                                      ana[g + f"bias_hh_l{layer}{suffix}"], rev))
        x = torch.cat(outs, -1)
    return x.unsqueeze(1)


def denoiser(mel, ana, train=False, drop_masks=None):
    """nn.Sequential at restorer/model.py:69-99.  drop_masks: in train mode (mode 2) the two
    Dropout(0.5) keep-masks (bool, shapes (B,1,T,512)); None -> no dropout (p forced to 0,
    SURVEY 8c hygiene note: torch RNG-stream parity is not attainable)."""
    p = "generator.denoiser."
    x = _bn1(mel, ana, p + "0", train)
    x = F.relu(_linear(x, ana, p + "1"))
    x = _bn1(x, ana, p + "3", train)
    x = _linear(x, ana, p + "4")
    if train and drop_masks is not None:
        x = x * drop_masks[0].to(x) * 2.0
    x = F.relu(x)
    x = bn_gru(x, ana, p + "7", train)
    x = bn_gru(x, ana, p + "8", train)
    x = F.relu(_bn1(x, ana, p + "9", train))
    x = _linear(x, ana, p + "11")
    if train and drop_masks is not None:
        x = x * drop_masks[1].to(x) * 2.0
    x = F.relu(_bn1(x, ana, p + "13", train))
    x = _linear(x, ana, p + "15")
    return torch.sigmoid(x)


def _linear(x, ana, p):
    return F.linear(_op(x, "denoiser.input"), _op(ana[p + ".weight"], "denoiser.weight"), ana[p + ".bias"])


# --------------------------------------------------------------------------- UNet
def _bn2d(x, ana, prefix, train):
    w, b = ana[prefix + ".weight"], ana[prefix + ".bias"]
    if train:
        return F.batch_norm(x, None, None, w, b, True, 0.0, BN_EPS)
    return F.batch_norm(x, ana[prefix + ".running_mean"], ana[prefix + ".running_var"], w, b,
                        False, 0.0, BN_EPS)


def _conv1_bn2(a, ana, p, train):
    """bn2(conv1(a)).  Under operand rounding in eval mode, the engine's form: bn2 folded into conv1, the folded
    weight rounded, the shift added after the contraction (weights._conv_block, engine.cu conv_block)."""
    w1 = ana[p + ".conv1.weight"]
    if _rounding is None or train:
        return _bn2d(F.conv2d(_op(a, "unet.bn_act"), _op(w1, "unet.weight"), padding=1), ana, p + ".bn2", train)
    q = p + ".bn2"
    scale = ana[q + ".weight"] / torch.sqrt(ana[q + ".running_var"] + BN_EPS)
    shift = ana[q + ".bias"] - ana[q + ".running_mean"] * scale
    return F.conv2d(_op(a, "unet.bn_act"), _op(w1 * scale[:, None, None, None], "unet.weight"), shift, padding=1)


def conv_block_res(x, ana, p, train):
    """ConvBlockRes.forward restorer/modules.py:68-76 (pre-activation, lrelu 0.01)."""
    origin = x
    x = _conv1_bn2(F.leaky_relu(_bn2d(x, ana, p + ".bn1", train), 0.01), ana, p, train)
    x = F.conv2d(_op(F.leaky_relu(x, 0.01), "unet.bn_act" if train else "unet.act"), _op(ana[p + ".conv2.weight"],
                                                                                          "unet.weight"), padding=1)
    if (p + ".shortcut.weight") in ana:
        return _stored(F.conv2d(_op(origin, "unet.shortcut"), _op(ana[p + ".shortcut.weight"], "unet.weight"),
                                ana[p + ".shortcut.bias"]) + x, "unet.block")
    return _stored(origin + x, "unet.block")


def encoder_block(x, ana, p, train):
    """EncoderBlockRes.forward restorer/modules.py:97-104."""
    for i in (1, 2, 3, 4):
        x = conv_block_res(x, ana, f"{p}.conv_block{i}", train)
    return F.avg_pool2d(x, (2, 2)), x


def decoder_block(x, skip, ana, p, train):
    """DecoderBlockRes.forward restorer/modules.py:149-157 (relu(bn1) -> ConvT 3x3 s2 ->
    prune last time row -> cat -> 4 ConvBlockRes)."""
    x = F.conv_transpose2d(_op(F.relu(_bn2d(x, ana, p + ".bn1", train)), "unet.bn_act"),
                           _op(ana[p + ".conv1.weight"], "unet.weight"), stride=2)
    x = x[:, :, 0:-1, :]
    x = torch.cat((x, skip), 1)
    for i in (2, 3, 4, 5):
        x = conv_block_res(x, ana, f"{p}.conv_block{i}", train)
    return x


def unet(x, ana, train=False):
    """UNetResComplex_100Mb.forward restorer/model_kqq_bn.py:130-181.  x (B,2,T,128)."""
    u = "generator.unet."
    origin_len = x.shape[2]
    pad_len = int(np.ceil(origin_len / 64)) * 64 - origin_len
    x = F.pad(x, (0, 0, 0, pad_len))
    x = x[..., 0:x.shape[-1] - 1]
    skips = []
    for i in range(1, 7):
        x, s = encoder_block(x, ana, f"{u}encoder_block{i}", train)
        skips.append(s)
    x = conv_block_res(x, ana, u + "conv_block7", train)
    for i in range(1, 7):
        x = decoder_block(x, skips[6 - i], ana, f"{u}decoder_block{i}", train)
    x = conv_block_res(x, ana, u + "after_conv_block1", train)
    x = F.conv2d(x, ana[u + "after_conv2.weight"], ana[u + "after_conv2.bias"])      # fp32 in the engine too
    x = F.pad(x, (0, 1))
    return x[:, :, 0:origin_len, :]


def to_log(x):
    """tools/pytorch_util.py:18-22."""
    assert torch.sum(x < 0) == 0
    return torch.log10(torch.clip(x, min=1e-8))


def from_log(x):
    """tools/pytorch_util.py:25-27."""
    return 10 ** torch.clip(x, max=5)


def analysis(mel, ana, train=False, drop_masks=None):
    """restorer Generator.forward restorer/model.py:103-120 -> out['mel'] (log10 domain)."""
    clean = denoiser(mel.clone(), ana, train, drop_masks) * mel
    x = to_log(clean)
    unet_in = torch.cat([to_log(mel), x], 1)
    return unet(unet_in, ana, train) + x


# --------------------------------------------------------------------------- vocoder
def _wn(voc, prefix):
    """torch weight_norm (dim=0): w = v * g/||v|| over all dims but 0 (SURVEY D6/a17).
    Accepts the parametrizations layout and the old weight_g/weight_v layout."""
    if prefix + ".parametrizations.weight.original0" in voc:
        g, v = voc[prefix + ".parametrizations.weight.original0"], voc[prefix + ".parametrizations.weight.original1"]
    elif prefix + ".weight_g" in voc:
        g, v = voc[prefix + ".weight_g"], voc[prefix + ".weight_v"]
    else:
        return voc[prefix + ".weight"]
    return torch._weight_norm(v, g, 0)


def mel_weight():
    """Config.get_mel_weight_torch vocoder/config.py:296-316: a*exp(b*k), k = 1..128."""
    k = torch.linspace(1, N_MEL, N_MEL)
    return MEL_W_A * torch.exp(MEL_W_B * k)


def vocoder_normalize(mel):
    """Vocoder.forward vocoder/base.py:51-54 + tr_amp_to_db/tr_normalize/tr_pre
    vocoder/model/util.py:8-36,69-80.  mel (B,1,T,128) linear -> cond (B,128,T + T%2 + 4)."""
    assert mel.size()[-1] == 128
    mel = mel / mel_weight()[None, None, None, :].to(mel)
    min_level = torch.exp(torch.tensor(-100.0) / 20 * torch.log(torch.tensor(10.0))).to(mel)
    S = 20 * torch.log10(torch.maximum(min_level, torch.abs(mel))) - 20.0
    S = torch.clip(8.0 * ((S + 115.0) / 115.0) - 4.0, -4.0, 4.0)
    c = S[:, 0].transpose(1, 2)
    pad_tail = c.size(-1) % 2 + 4
    return torch.cat([c, torch.zeros(c.size(0), N_MEL, pad_tail, dtype=c.dtype, device=c.device) - 4.0], -1)


def res_stack(x, voc, p):
    """ResStack.forward modules.py:592-595 over the Sequentials built at :550-576."""
    x = _stored(x, "vocoder.residual")
    for i in range(8):
        d = 3 ** i
        h = F.conv1d(_op(F.leaky_relu(x, 0.01), "vocoder.act"), _op(_wn(voc, f"{p}.layers.{i}.1"), "vocoder.weight"),
                     voc[f"{p}.layers.{i}.1.bias"], dilation=d, padding=d)
        h = F.conv1d(_op(F.leaky_relu(h, 0.01), "vocoder.act"), _op(_wn(voc, f"{p}.layers.{i}.3"), "vocoder.weight"),
                     voc[f"{p}.layers.{i}.3.bias"], padding=1)
        x = _stored(x + h, "vocoder.residual")
    return x


def upsample_net(x, voc, p, u):
    """UpsampleNet.forward modules.py:501-517 with org=False, no_skip=True: x + sin x, then
    weight-normed ConvTranspose1d(k=2u, s=u, p=u//2+u%2, output_padding=u%2).  The skip_conv
    result is discarded by the reference (SURVEY D7) and is not computed here."""
    x = x + torch.sin(x)
    return F.conv_transpose1d(_op(x, "vocoder.act"), _op(_wn(voc, p + ".layer"), "vocoder.weight"),
                              voc[p + ".layer.bias"], stride=u, padding=u // 2 + u % 2, output_padding=u % 2)


def vocoder_generator(cond, voc):
    """vocoder Generator.forward generator.py:127-145 (condnet :33-54, generator :73-100)."""
    x = cond
    for i in (0, 2, 4, 6, 8):
        x = F.elu(F.conv1d(_op(x, "vocoder.cond" if i == 0 else "vocoder.act"),
                           _op(_wn(voc, f"condnet.{i}"), "vocoder.weight"), voc[f"condnet.{i}.bias"], padding=1))
    x = F.conv1d(_op(F.pad(x, (3, 3), mode="reflect"), "vocoder.act"), _op(_wn(voc, "generator.1"), "vocoder.weight"),
                 voc["generator.1.bias"])
    x = F.leaky_relu(x, 0.2)
    for j, u in enumerate(UPSAMPLE_SCALES):
        x = upsample_net(x, voc, f"generator.{3 + 3 * j}", u)
        x = res_stack(x, voc, f"generator.{4 + 3 * j}")
        x = F.leaky_relu(x, 0.2)
    # fp32 in the engine too: voc.post.w is fp32 and reads plain x'
    x = F.conv1d(F.pad(x, (3, 3), mode="reflect"), _wn(voc, "generator.16"), voc["generator.16.bias"])
    return torch.tanh(x)


def vocoder_forward(mel, voc):
    """Vocoder.forward vocoder/base.py:42-56: (B,1,T,128) linear mel -> (B,1,(T+T%2+4)*441)."""
    return vocoder_generator(vocoder_normalize(mel), voc)


# --------------------------------------------------------------------------- restore
def trim_center(est, ref_len):
    """VoiceFixer._trim_center base.py:63-76 (est longer than ref on this path)."""
    n = est.shape[-1]
    diff = abs(n - ref_len)
    if n == ref_len:
        return est
    assert n > ref_len
    est = est[..., int(diff // 2): -int(diff // 2)]
    return est[..., :min(n, ref_len)]


def remove_higher_frequency(wav, ratio=0.95, dtype=np.float32, return_cut=False):
    """VoiceFixer.remove_higher_frequency base.py:87-104 (mode 1) with librosa 0.10.1
    (Dockerfile:9) defaults restated: stft(n_fft=2048, hop=512, hann periodic, center=True,
    pad_mode='constant'), istft(length=None -> 512*(frames-1), window-sumsquare normalised).
    dtype: np.float32 (the reference's arithmetic) or np.float64.  return_cut: also return the first
    zeroed bin."""
    wav = np.asarray(wav, dtype=dtype)
    cdt = np.result_type(dtype, np.complex64)
    n_fft, hop = 2048, 512
    win = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n_fft) / n_fft)).astype(dtype)
    x = np.pad(wav, (n_fft // 2, n_fft // 2), mode="constant")
    nfr = 1 + (len(x) - n_fft) // hop
    idx = np.arange(n_fft)[None, :] + hop * np.arange(nfr)[:, None]
    stft = np.fft.rfft(x[idx] * win[None, :], axis=1).T.astype(cdt)     # (1025, T)
    real, img = np.real(stft), np.imag(stft)
    mag = (real ** 2 + img ** 2) ** 0.5
    cos, sin = real / (mag + 1e-8), img / (mag + 1e-8)
    spec = np.abs(stft)
    feature = np.log10(spec + 1e-8)
    feature[feature < 0] = 0
    energy_level = np.sum(feature, axis=1)
    threshold = np.sum(energy_level) * ratio
    curent_level, i = energy_level[0], 0
    while i < energy_level.shape[0] and curent_level < threshold:
        curent_level += energy_level[i + 1, ...]
        i += 1
    spec[i:, ...] = 0
    stft = spec * cos + 1j * spec * sin
    frames = np.fft.irfft(stft.T, n=n_fft, axis=1).astype(dtype) * win[None, :]
    out_len = n_fft + hop * (nfr - 1)
    y = np.zeros(out_len, dtype=dtype)
    wss = np.zeros(out_len, dtype=dtype)
    wsq = win ** 2
    for t in range(nfr):
        y[t * hop:t * hop + n_fft] += frames[t]
        wss[t * hop:t * hop + n_fft] += wsq
    nz = wss > np.finfo(np.float32).tiny
    y[nz] /= wss[nz]
    y = y[n_fft // 2: n_fft // 2 + hop * (nfr - 1)]
    return (y, i) if return_cut else y


def _np_dtype(t):
    return torch.empty(0, dtype=t.dtype).numpy().dtype


def restore_inmem(wav, ana, voc, mode=0, drop_masks_fn=None):
    """VoiceFixer.restore_inmem base.py:106-139: np (L,) -> np (1, N) in the state dicts' dtype (float32 for the
    checkpoints as stored).  30 s segments, independent, concatenated (SURVEY D4).  mode 2 = train-mode BN (+ dropout
    if masks given).  The samples are read as float32, as the reference reads them."""
    like = ana["mel.fb"]
    dt = _np_dtype(like)
    wav = np.asarray(np.asarray(wav, dtype=np.float32), dtype=dt)
    train = (mode == 2)
    res = []
    break_point = SEG_LEN
    while break_point < wav.shape[0] + SEG_LEN:
        segment = wav[break_point - SEG_LEN: break_point]
        if mode == 1:
            segment = remove_higher_frequency(segment, dtype=dt)
        _, mel = frontend(torch.from_numpy(np.ascontiguousarray(segment))[None].to(like.device), ana)
        masks = drop_masks_fn(mel.shape[2]) if (train and drop_masks_fn) else None
        out_mel = analysis(mel, ana, train, masks)
        out = vocoder_forward(from_log(out_mel), voc)
        out = trim_center(out, segment.shape[-1])
        res.append(out)
        break_point += SEG_LEN
    return torch.cat(res, -1).squeeze(0).cpu().numpy()


# --------------------------------------------------------------------------- oracle() front end
def slaney_htk_mel_basis():
    """librosa.filters.mel(sr=44100, n_fft=2048, htk=True, n_mels=128, fmin=0, fmax=22050),
    norm='slaney' default, built in float64 then cast to float32 (vocoder/model/util.py:115-123)."""
    n_mels, fmax = 128, 22050.0
    fftfreqs = np.linspace(0, SR / 2.0, 1 + N_FFT // 2)
    mmax = 2595.0 * np.log10(1.0 + fmax / 700.0)
    mels = np.linspace(0.0, mmax, n_mels + 2)
    mel_f = 700.0 * (10.0 ** (mels / 2595.0) - 1.0)
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    weights = np.zeros((n_mels, 1 + N_FFT // 2))
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, np.newaxis]
    return weights.astype(np.float32)


def oracle_cond(wav, dtype=torch.float32):
    """Vocoder.oracle front end vocoder/base.py:61-73: peak-normalise, |librosa.stft|
    (n_fft 2048, hop 441, hann, center, pad_mode='constant' per librosa 0.10.1), Slaney mel,
    dB-20, normalise, pre() -> cond (1,128,T+T%2+4).  librosa's stft multiplies the float32 frames by
    get_window's float64 window without a cast: the windowed frames are float64.
    dtype: torch.float32 (the reference's arithmetic and result) or torch.float64 (float64 throughout, on the
    float32 samples and the float32 Slaney basis)."""
    f64 = dtype == torch.float64
    wav = np.asarray(np.asarray(wav, dtype=np.float32), dtype=np.float64 if f64 else np.float32)
    wav = wav / np.max(np.abs(wav))
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N_FFT) / N_FFT)
    x = np.pad(wav, (N_FFT // 2, N_FFT // 2), mode="constant")
    nfr = 1 + (len(x) - N_FFT) // HOP
    idx = np.arange(N_FFT)[None, :] + HOP * np.arange(nfr)[:, None]
    stft = np.fft.rfft(x[idx] * win[None, :], axis=1).T
    stft = np.abs(stft if f64 else stft.astype(np.complex64))
    basis = slaney_htk_mel_basis()
    mel = np.dot(basis.astype(np.float64) if f64 else basis, stft)
    min_level = np.exp(-100 / 20 * np.log(10))
    S = 20 * np.log10(np.maximum(min_level, np.abs(mel))) - 20
    S = np.clip(8.0 * ((S + 115.0) / 115.0) - 4.0, -4.0, 4.0)
    c = torch.from_numpy(np.ascontiguousarray(np.transpose(S, (1, 0)))).to(dtype).unsqueeze(0).transpose(1, 2)
    pad_tail = c.size(-1) % 2 + 4
    return torch.cat([c, torch.zeros(1, N_MEL, pad_tail, dtype=dtype) - 4.0], -1)


def oracle_wave(wav, voc):
    """Vocoder.oracle vocoder/base.py:58-77 up to (not including) the file write:
    returns float wav_re * 2**15 as np (1, 1, S), in the dtype and on the device of voc."""
    like = voc["condnet.0.bias"]
    cond = oracle_cond(wav, like.dtype).to(like.device)
    return (vocoder_generator(cond, voc) * 2 ** 15).cpu().numpy()

"""Checkpoint -> kernel-native weight tensors.

Reads the reference checkpoint layout (SURVEY 3.1), folds weight-norm once (the reference
recomputes g*v/||v|| on every forward, SURVEY D6), turns eval-mode BatchNorm running stats into
per-channel scale/shift, and re-lays every convolution as [taps][Cout][Cin] (K-major) for the
channels-last shifted-window GEMM kernels.  Names are the ones csrc/engine.cu looks up.
"""
import numpy as np
import torch

BN_EPS = 1e-5


def round_tf32(t):
    """fp32 -> nearest tf32 value (10-bit mantissa, ties away from zero = PTX cvt.rna.tf32.f32), kept in fp32 storage.
    The tensor core truncates the low 13 mantissa bits of a tf32 operand; pre-rounded weights make that exact."""
    i = t.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


class _Wdt:
    """Weight element format of a vfx_precision: storage dtype + rounding + whether tiny Cin is padded for the MMA."""

    def __init__(self, precision):
        if precision not in ("fp32", "bf16", "tf32", "fp16"):
            raise ValueError(f"unknown precision '{precision}'")
        self.precision = precision
        self.tensor_core = precision != "fp32"

    def __call__(self, t):
        if self.precision == "bf16":
            return t.to(torch.bfloat16)
        if self.precision == "tf32":
            return round_tf32(t)
        if self.precision == "fp16":
            if float(t.abs().max()) > 6.0e4:
                raise ValueError("a weight exceeds fp16's range (65504): use precision tf32 or bf16 for this checkpoint")
            return t.to(torch.float16)
        return t.float()


def _bn(out, name, sd, prefix):
    g, b = sd[prefix + ".weight"].double(), sd[prefix + ".bias"].double()
    m, v = sd[prefix + ".running_mean"].double(), sd[prefix + ".running_var"].double()
    scale = g / torch.sqrt(v + BN_EPS)
    out[name + ".scale"] = scale.float()
    out[name + ".shift"] = (b - m * scale).float()
    out[name + ".gamma"] = g.float()
    out[name + ".beta"] = b.float()


def _weight_norm(sd, prefix):
    """w = g * v / ||v|| over all dims but 0 (torch weight_norm dim=0); both key layouts."""
    if prefix + ".parametrizations.weight.original0" in sd:
        g = sd[prefix + ".parametrizations.weight.original0"]
        v = sd[prefix + ".parametrizations.weight.original1"]
    elif prefix + ".weight_g" in sd:
        g, v = sd[prefix + ".weight_g"], sd[prefix + ".weight_v"]
    elif prefix + ".weight" in sd:
        return sd[prefix + ".weight"].float()
    else:
        raise KeyError(f"vocoder checkpoint has no weight for '{prefix}'")
    return torch._weight_norm(v.float(), g.float(), 0)


def check_stft_kernels(sd):
    """The engine computes the STFT with an FFT + analytic periodic Hann window.  vf.ckpt also
    stores the reference's DFT-conv kernels (base.py:23-29 loads them over the constructed ones);
    refuse checkpoints whose kernels are not the Hann-windowed DFT."""
    key = "f_helper.stft.conv_real.weight"
    if key not in sd:
        return
    w = sd[key].double()[:, 0, :]                       # (1025, 2048)
    if tuple(w.shape) != (1025, 2048):
        raise ValueError(f"{key} has shape {tuple(sd[key].shape)}, expected (1025, 1, 2048)")
    n = torch.arange(2048, dtype=torch.float64)
    win = 0.5 - 0.5 * torch.cos(2 * np.pi * n / 2048)
    for k in (0, 1, 7, 512, 1024):
        ref = torch.cos(2 * np.pi * ((n * k) % 2048) / 2048) * win
        if (w[k] - ref).abs().max() > 1e-4:
            raise ValueError("checkpoint STFT kernels are not a periodic-Hann DFT; unsupported")


def _conv_block(out, name, sd, p, wdt):
    _bn(out, name + ".bn1", sd, p + ".bn1")
    _bn(out, name + ".bn2", sd, p + ".bn2")
    w1, w2 = sd[p + ".conv1.weight"].float(), sd[p + ".conv2.weight"].float()
    pad_cin = wdt.tensor_core and w1.shape[1] < 32            # tensor-core paths: zero-pad tiny Cin to 32 operand channels
    if pad_cin:
        w1 = torch.nn.functional.pad(w1, (0, 0, 0, 0, 0, 32 - w1.shape[1]))
    out[name + ".conv1.w"] = wdt(w1.permute(2, 3, 0, 1).reshape(9, w1.shape[0], w1.shape[1]).contiguous())
    out[name + ".conv2.w"] = wdt(w2.permute(2, 3, 0, 1).reshape(9, w2.shape[0], w2.shape[1]).contiguous())
    # eval mode: bn2 folds into conv1 (scale rows, shift as bias) -> conv1f; its epilogue applies the LeakyReLU
    sc2, sh2 = out[name + ".bn2.scale"], out[name + ".bn2.shift"]
    w1f = w1 * sc2[:, None, None, None]
    out[name + ".conv1f.w"] = wdt(w1f.permute(2, 3, 0, 1).reshape(9, w1f.shape[0], w1f.shape[1]).contiguous())
    out[name + ".conv1f.b"] = sh2.clone()
    if p + ".shortcut.weight" in sd:
        ws = sd[p + ".shortcut.weight"].float()[:, :, 0, 0]
        if pad_cin:
            ws = torch.nn.functional.pad(ws, (0, 32 - ws.shape[1]))
        out[name + ".sc.w"] = wdt(ws.contiguous())
        out[name + ".sc.b"] = sd[p + ".shortcut.bias"].float()


def pack_analysis(sd, precision="fp32"):
    """vf.ckpt flat state dict -> {engine name: CPU tensor}."""
    wdt = _Wdt(precision)
    check_stft_kernels(sd)
    out = {}
    fb = sd["mel.fb"].float()                           # (1025, 128)
    if tuple(fb.shape) != (1025, 128):
        raise ValueError(f"mel.fb has shape {tuple(fb.shape)}, expected (1025, 128)")
    fbT = fb.t().contiguous()
    nz = fbT != 0
    start = torch.zeros(128, dtype=torch.int32)
    length = torch.zeros(128, dtype=torch.int32)
    for m in range(128):
        idx = torch.nonzero(nz[m]).flatten()
        if idx.numel():
            start[m] = int(idx[0]); length[m] = int(idx[-1]) - int(idx[0]) + 1
    out["fe.fbT"], out["fe.fb_start"], out["fe.fb_len"] = fbT, start, length
    # ---- denoiser (GEMM weights in the operand precision; GRU recurrence weights always fp32)
    d = "generator.denoiser."
    for ref, name in (("0", "bn0"), ("3", "bn3"), ("7.bn", "g7.bn"), ("8.bn", "g8.bn"), ("9", "bn9"), ("13", "bn13")):
        _bn(out, "dn." + name, sd, d + ref)
    for ref, name in (("1", "lin1"), ("4", "lin4"), ("11", "lin11"), ("15", "lin15")):
        out[f"dn.{name}.w"] = wdt(sd[d + ref + ".weight"].float().contiguous())
        out[f"dn.{name}.b"] = sd[d + ref + ".bias"].float()
    for g in ("7", "8"):
        for layer in (0, 1):
            p = f"{d}{g}.gru."
            sfx = [f"_l{layer}", f"_l{layer}_reverse"]
            out[f"dn.g{g}.l{layer}.wih"] = wdt(torch.cat([sd[p + "weight_ih" + s].float() for s in sfx], 0).contiguous())
            out[f"dn.g{g}.l{layer}.bih"] = torch.cat([sd[p + "bias_ih" + s].float() for s in sfx], 0).contiguous()
            out[f"dn.g{g}.l{layer}.whh_t"] = torch.stack([sd[p + "weight_hh" + s].float().t() for s in sfx], 0).contiguous()
            out[f"dn.g{g}.l{layer}.bhh"] = torch.stack([sd[p + "bias_hh" + s].float() for s in sfx], 0).contiguous()
    # ---- UNet
    u = "generator.unet."
    for i in range(1, 7):
        for j in range(1, 5):
            _conv_block(out, f"unet.enc{i}.b{j}", sd, f"{u}encoder_block{i}.conv_block{j}", wdt)
    _conv_block(out, "unet.center", sd, u + "conv_block7", wdt)
    for i in range(1, 7):
        p = f"{u}decoder_block{i}"
        _bn(out, f"unet.dec{i}.bn1", sd, p + ".bn1")
        wt = sd[p + ".conv1.weight"].float()             # ConvTranspose2d (Cin, Cout, 3, 3)
        out[f"unet.dec{i}.up.w"] = wdt(wt.permute(2, 3, 1, 0).reshape(9, wt.shape[1], wt.shape[0]).contiguous())
        for j in range(2, 6):
            _conv_block(out, f"unet.dec{i}.b{j}", sd, f"{p}.conv_block{j}", wdt)
    _conv_block(out, "unet.after", sd, u + "after_conv_block1", wdt)
    out["unet.head.w"] = sd[u + "after_conv2.weight"].float().reshape(32).contiguous()
    out["unet.head.b"] = sd[u + "after_conv2.bias"].float().reshape(1)
    return out


def pack_vocoder(sd, precision="fp32"):
    """ckpt['generator'] state dict -> {engine name: CPU tensor}."""
    wdt = _Wdt(precision)
    out = {}
    # Config.get_mel_weight_torch (vocoder/config.py:296-316) and tr_amp_to_db's min_level
    # (vocoder/model/util.py:33-36), computed with the same fp32 torch ops as the reference
    k = torch.linspace(1, 128, 128)
    w = 18.8927416350036 * torch.exp(0.0269863588184314 * k)
    min_level = torch.exp(torch.tensor(-100.0) / 20 * torch.log(torch.tensor(10.0)))
    out["voc.mel_tab"] = torch.cat([w, min_level.reshape(1)]).float()
    for n, i in enumerate((0, 2, 4, 6, 8)):
        out[f"voc.cond{n}.w"] = wdt(_weight_norm(sd, f"condnet.{i}").permute(2, 0, 1).contiguous())
        out[f"voc.cond{n}.b"] = sd[f"condnet.{i}.bias"].float()
    out["voc.pre.w"] = wdt(_weight_norm(sd, "generator.1").permute(2, 0, 1).contiguous())
    out["voc.pre.b"] = sd["generator.1.bias"].float()
    for j in range(4):
        p = f"generator.{3 + 3 * j}.layer"
        wt = _weight_norm(sd, p)                         # ConvTranspose1d (Cin, Cout, 2u)
        out[f"voc.up{j}.w"] = wdt(wt.permute(2, 1, 0).contiguous())
        out[f"voc.up{j}.b"] = sd[p + ".bias"].float()
        r = f"generator.{4 + 3 * j}"
        for i in range(8):
            for k_ref, k_name in ((1, "c1"), (3, "c2")):
                q = f"{r}.layers.{i}.{k_ref}"
                out[f"voc.rs{j}.l{i}.{k_name}.w"] = wdt(_weight_norm(sd, q).permute(2, 0, 1).contiguous())
                out[f"voc.rs{j}.l{i}.{k_name}.b"] = sd[q + ".bias"].float()
    out["voc.post.w"] = _weight_norm(sd, "generator.16")[0].t().contiguous().float()   # (7, 64)
    out["voc.post.b"] = sd["generator.16.bias"].float().reshape(1)
    return out

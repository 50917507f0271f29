"""GPU tests of the individual kernels through the C ABI against plain PyTorch fp32 ops."""
import ctypes
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from conftest import golden, rel_rms

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda:0")


def _rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(_dev())


@pytest.mark.parametrize("C,L,dil,B", [(64, 700, 1, 2), (64, 300, 27, 1), (128, 257, 243, 2), (32, 100, 2187, 1)])
def test_conv1d_dilated_fp32(C, L, dil, B):
    from gpu_util import conv_gemm
    torch.backends.cudnn.allow_tf32 = False
    x, w, b = _rnd(B, C, L, seed=1), _rnd(C, C, 3, seed=2, scale=0.1), _rnd(C, seed=3)
    ref = F.conv1d(x, w, b, dilation=dil, padding=dil)
    a = x.permute(0, 2, 1).contiguous()[:, None]                   # (B,1,L,C)
    wp = w.permute(2, 0, 1).contiguous()
    raw, act = conv_gemm(a, wp, [(0, -dil), (0, 0), (0, dil)], bias=b, want_act=True, act="lrelu", act_param=0.01)
    assert rel_rms(raw[:, 0].permute(0, 2, 1).cpu(), ref.cpu()) < 1e-5
    assert rel_rms(act[:, 0].permute(0, 2, 1).cpu(), F.leaky_relu(ref, 0.01).cpu()) < 1e-5


@pytest.mark.parametrize("Cin,Cout,H,W", [(2, 32, 64, 127), (32, 32, 16, 15), (64, 32, 8, 7), (384, 384, 2, 1)])
def test_conv2d_3x3_residual_fp32(Cin, Cout, H, W):
    from gpu_util import conv_gemm
    torch.backends.cudnn.allow_tf32 = False
    x, w = _rnd(2, Cin, H, W, seed=4), _rnd(Cout, Cin, 3, 3, seed=5, scale=0.1)
    res = _rnd(2, Cout, H, W, seed=6)
    ref = F.conv2d(x, w, padding=1) + res
    a = x.permute(0, 2, 3, 1).contiguous()
    wp = w.permute(2, 3, 0, 1).reshape(9, Cout, Cin).contiguous()
    taps = [(kh - 1, kw - 1) for kh in range(3) for kw in range(3)]
    raw, _ = conv_gemm(a, wp, taps, residual=res.permute(0, 2, 3, 1).contiguous())
    assert rel_rms(raw.permute(0, 3, 1, 2).cpu(), ref.cpu()) < 1e-5


@pytest.mark.parametrize("u,Cin,Cout,L", [(7, 64, 32, 50), (3, 32, 64, 33)])
def test_conv_transpose1d_phase_groups_fp32(u, Cin, Cout, L):
    """ConvTranspose1d(k=2u, s=u, p=u//2+u%2, output_padding=u%2) as two phase-group GEMMs."""
    from gpu_util import conv_gemm
    x, w, b = _rnd(2, Cin, L, seed=7), _rnd(Cin, Cout, 2 * u, seed=8, scale=0.1), _rnd(Cout, seed=9)
    pad = u // 2 + u % 2
    ref = F.conv_transpose1d(x, w, b, stride=u, padding=pad, output_padding=u % 2)
    assert ref.shape[-1] == u * L
    a = x.permute(0, 2, 1).contiguous()[:, None]
    wp = w.permute(2, 1, 0).contiguous()                           # (2u, Cout, Cin)
    mat = Cout * Cin
    nA = u - pad
    out = torch.zeros(2, 1, u * L, Cout, device=_dev())
    conv_gemm(a, wp, [(0, 0), (0, -1)], N=nA * Cout, w_off=[pad * mat, (pad + u) * mat], bias=b, bias_mod=Cout,
              sw=u, rw=0, OW=u * L, out_ld=Cout, out_raw=out)
    conv_gemm(a, wp, [(0, 1), (0, 0)], N=(u - nA) * Cout, w_off=[0, u * mat], bias=b, bias_mod=Cout,
              sw=u, rw=nA, OW=u * L, out_ld=Cout, out_raw=out)
    assert rel_rms(out[:, 0].permute(0, 2, 1).cpu(), ref.cpu()) < 1e-5


def test_conv_transpose2d_phases_fp32():
    """ConvTranspose2d(k3, s2, p0) + prune of the last time row, as 4 output-parity GEMMs."""
    from gpu_util import conv_gemm
    Cin, Cout, H, W = 64, 32, 5, 3
    x, w = _rnd(2, Cin, H, W, seed=10), _rnd(Cin, Cout, 3, 3, seed=11, scale=0.1)
    ref = F.conv_transpose2d(x, w, stride=2)[:, :, :-1, :]
    OH, OW = 2 * H, 2 * W + 1
    a = x.permute(0, 2, 3, 1).contiguous()
    wp = w.permute(2, 3, 1, 0).reshape(9, Cout, Cin).contiguous()
    out = torch.zeros(2, OH, OW, Cout, device=_dev())
    for rh in range(2):
        for rw in range(2):
            taps, offs = [], []
            for kh in ([1] if rh else [0, 2]):
                for kw in ([1] if rw else [0, 2]):
                    taps.append((-1 if kh == 2 else 0, -1 if kw == 2 else 0))
                    offs.append((kh * 3 + kw) * Cout * Cin)
            conv_gemm(a, wp, taps, Hq=H, Wq=W + 1, N=Cout, w_off=offs, sh=2, rh=rh, sw=2, rw=rw, OH=OH, OW=OW,
                      out_raw=out)
    assert rel_rms(out.permute(0, 3, 1, 2).cpu(), ref.cpu()) < 1e-5


def test_conv_bf16_operands_simt_is_exact_to_rounding():
    """bf16 operands, fp32 accumulate: equals an fp32 conv of the bf16-rounded inputs."""
    from gpu_util import conv_gemm
    C, L = 64, 400
    x, w = _rnd(1, C, L, seed=12).bfloat16(), _rnd(C, C, 3, seed=13, scale=0.1).bfloat16()
    ref = F.conv1d(x.float(), w.float(), padding=1)
    a = x.permute(0, 2, 1).contiguous()[:, None]
    raw, _ = conv_gemm(a, w.permute(2, 0, 1).contiguous(), [(0, -1), (0, 0), (0, 1)], precision="bf16")
    assert rel_rms(raw[:, 0].permute(0, 2, 1).cpu(), ref.cpu()) < 1e-5


def test_gru_layer_matches_torch_gru():
    from voicefixer_b200 import _lib
    lib = _lib.load()
    B, T = 5, 37
    torch.backends.cudnn.allow_tf32 = False          # the cuDNN GRU reference would run TF32 otherwise
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    gru = torch.nn.GRU(512, 256, num_layers=1, bidirectional=True, batch_first=True).to(_dev())
    x = _rnd(B, T, 512, seed=14)
    with torch.no_grad():
        ref, _ = gru(x)
        wih = torch.cat([gru.weight_ih_l0, gru.weight_ih_l0_reverse], 0)
        bih = torch.cat([gru.bias_ih_l0, gru.bias_ih_l0_reverse], 0)
        gi = (x @ wih.t() + bih).contiguous()                       # (B,T,1536) = [B][T][2][768]
        whh_t = torch.stack([gru.weight_hh_l0.t(), gru.weight_hh_l0_reverse.t()], 0).contiguous()
        bhh = torch.stack([gru.bias_hh_l0, gru.bias_hh_l0_reverse], 0).contiguous()
    out = torch.empty(B, T, 512, device=_dev())
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    _lib.check(lib.vfx_gru_layer(p(gi), p(whh_t), p(bhh), B, T, p(out), None), "vfx_gru_layer")
    torch.cuda.synchronize()
    assert rel_rms(out.cpu(), ref.cpu()) < 1e-5


def test_frontend_fft_mel_vs_reference_golden(engine):
    g = golden("frontend")
    mel, sp = engine.frontend(g["wav"], return_sp=True)
    assert rel_rms(mel.cpu().numpy(), g["mel"][:, 0]) < 2e-5        # stated tolerance: rFFT vs DFT-conv, fp32
    assert rel_rms(sp.cpu().numpy()[:, :4], g["sp_slice"][:, 0]) < 2e-5


def test_frontend_rejects_short_input(engine):
    from voicefixer_b200._lib import VfxError
    with pytest.raises(VfxError, match="1024"):
        engine.frontend(np.zeros((1, 1000), np.float32))


def test_hf_cut_mode1_prefilter_vs_oracle(engine):
    """vfx_hf_cut vs the oracle's restatement of remove_higher_frequency (base.py:87-104)."""
    from voicefixer_b200 import synthetic
    from oracle import vf_oracle as O
    wav = synthetic.make_utterances(2, seconds=0.8, seed=41)
    out, cut = engine.hf_cut(wav)
    for b in range(2):
        ref = O.remove_higher_frequency(wav[b])
        assert out.shape[1] == ref.shape[0] == 512 * (wav.shape[1] // 512)
        assert rel_rms(out[b].cpu().numpy(), ref) < 5e-7       # measured 1.4e-7 on an H100 (700 W)
    assert all(0 < int(c) < 1025 for c in cut.cpu())


def test_restore_mode1_vs_oracle(engine, states):
    """mode 1 end to end through the API semantics: pre-filter, shorter output (132300 -> 132096 style)."""
    from voicefixer_b200 import synthetic
    from oracle import vf_oracle as O
    wav = synthetic.make_utterances(1, seconds=0.6, seed=43)[0]
    ref = O.restore_inmem(wav, states[0], states[1], mode=1)
    x, _ = engine.hf_cut(wav[None])
    out = engine.restore(x).cpu().numpy()
    assert out.shape == ref.shape == (1, 512 * (wav.shape[0] // 512))
    assert rel_rms(out, ref) < 2e-4

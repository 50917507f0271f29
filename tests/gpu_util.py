"""Helpers for the GPU tests: build vfx_conv_desc structs from torch tensors."""
import ctypes
import torch
from voicefixer_b200 import _lib


def conv_gemm(a, w, taps, Hq=None, Wq=None, N=None, w_off=None, bias=None, bias_mod=None, residual=None,
              act="none", act_param=0.0, want_raw=True, want_act=False, sh=1, rh=0, sw=1, rw=0, OH=None, OW=None,
              out_ld=None, out_col=0, precision="fp32", impl=0, out_raw=None, out_act=None, res_enc=0, raw_enc=0,
              enc_slope=0.0, act_scale=None, act_shift=None, act_ld=None, act_col=None, act_sB=None):
    """a: (B,H,W,Cin) cuda (fp32 or bf16); w: flat weight tensor; taps: [(dh,dw)].
    act_scale / act_shift: per-channel affine applied before the activation of out_act (both or neither);
    act_ld / act_col: row pitch and first column of out_act when they differ from the raw output's (out_ld / out_col);
    act_sB: item stride of out_act in elements, in place of the dense OH * OW * pitch (e.g. a padded buffer)."""
    lib = _lib.load()
    B, H, W, Cin = a.shape
    d = _lib.ConvDesc()
    d.a = a.data_ptr(); d.B, d.H, d.W, d.Cin = B, H, W, Cin
    d.a_sW, d.a_sH, d.a_sB = a.stride(2), a.stride(1), a.stride(0)
    d.w = w.data_ptr(); d.ntaps = len(taps)
    N = N if N is not None else w.shape[-2]
    for i, (dh, dw) in enumerate(taps):
        d.dh[i], d.dw[i] = dh, dw
        d.w_off[i] = w_off[i] if w_off is not None else i * N * Cin
    d.Hq, d.Wq, d.N = Hq or H, Wq or W, N
    d.sh, d.rh, d.sw, d.rw = sh, rh, sw, rw
    d.OH, d.OW = OH or d.Hq, OW or d.Wq
    ld = out_ld or N
    dt = {"bf16": torch.bfloat16, "fp16": torch.float16}.get(precision, torch.float32)      # tf32: fp32 storage
    if want_raw:
        if out_raw is None:
            out_raw = torch.zeros(B, d.OH, d.OW, ld, device=a.device)
        d.out_raw = out_raw.data_ptr()
        d.o_sW, d.o_sH, d.o_sB, d.o_col = ld, d.OW * ld, d.OH * d.OW * ld, out_col
    if want_act:
        ald = act_ld or ld
        if out_act is None:
            out_act = torch.zeros(B, d.OH, d.OW, ald, device=a.device, dtype=dt)
        d.out_act = out_act.data_ptr()
        d.oa_sW, d.oa_sH, d.oa_sB = ald, d.OW * ald, d.OH * d.OW * ald
        d.oa_col = out_col if act_col is None else act_col
        if act_sB is not None:
            d.oa_sB = act_sB
    if (act_scale is None) != (act_shift is None):
        raise ValueError("act_scale and act_shift go together")
    if act_scale is not None:
        d.act_scale, d.act_shift = act_scale.data_ptr(), act_shift.data_ptr()
    if bias is not None:
        d.bias = bias.data_ptr(); d.bias_mod = bias_mod or bias.numel()
    if residual is not None:
        d.residual = residual.data_ptr()
        d.r_sW, d.r_sH, d.r_sB, d.r_col = residual.stride(2), residual.stride(1), residual.stride(0), 0
    d.act = _lib.ACT[act]; d.act_param = act_param
    d.res_enc, d.raw_enc, d.enc_slope = res_enc, raw_enc, enc_slope
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.vfx_conv_gemm(_lib.PREC[precision], impl, ctypes.byref(d), st), "vfx_conv_gemm")
    torch.cuda.synchronize()
    return out_raw, out_act

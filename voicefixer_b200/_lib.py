"""ctypes binding of libvfx_b200.so (the C ABI declared in include/vfx_b200.h).

There is no CPU or PyTorch fallback: if the shared library is missing or fails to load, importing
the product path raises.  Build it with `python -m voicefixer_b200.build` (nvcc, sm_90a)."""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libvfx_b200.so")

VFX_OK = 0
PREC = {"fp32": 0, "bf16": 1, "tf32": 2, "fp16": 3}
ACT = {"none": 0, "lrelu": 1, "elu": 2, "lrelu_xsinx": 3, "sigmoid": 4}
PAIR_FORM = {"fused": 0, "blocked": 1}
PCM16_MAX_CHANNELS = 8                 # VFX_PCM16_MAX_CHANNELS

_c = ctypes
_vp, _i, _f, _sz, _ll = _c.c_void_p, _c.c_int, _c.c_float, _c.c_size_t, _c.c_longlong


class ConvDesc(ctypes.Structure):
    """struct vfx_conv_desc (include/vfx_b200.h)."""
    _fields_ = [
        ("a", _vp), ("B", _i), ("H", _i), ("W", _i), ("Cin", _i),
        ("a_sB", _ll), ("a_sH", _ll), ("a_sW", _ll),
        ("w", _vp), ("ntaps", _i), ("dh", _i * 9), ("dw", _i * 9), ("w_off", _ll * 9),
        ("Hq", _i), ("Wq", _i), ("N", _i), ("sh", _i), ("rh", _i), ("sw", _i), ("rw", _i),
        ("OH", _i), ("OW", _i),
        ("out_raw", _vp), ("o_sB", _ll), ("o_sH", _ll), ("o_sW", _ll), ("o_col", _i),
        ("out_act", _vp), ("oa_sB", _ll), ("oa_sH", _ll), ("oa_sW", _ll), ("oa_col", _i),
        ("bias", _vp), ("bias_mod", _i),
        ("residual", _vp), ("r_sB", _ll), ("r_sH", _ll), ("r_sW", _ll), ("r_col", _i),
        ("act", _i), ("act_param", _f), ("act_scale", _vp), ("act_shift", _vp),
        ("res_enc", _i), ("raw_enc", _i), ("enc_slope", _f),
        ("seq_in", _vp), ("seq_out", _vp), ("seq_axis", _i),
    ]


class PairDesc(ctypes.Structure):
    """struct vfx_pair_desc (include/vfx_b200.h)."""
    _fields_ = [("a", _vp), ("x", _vp), ("w1", _vp), ("b1", _vp), ("dilation", _i), ("w2", _vp), ("b2", _vp),
                ("B", _i), ("L", _i), ("C", _i), ("write_raw", _i), ("out_act", _vp), ("act", _i), ("act_param", _f),
                ("precision", _i), ("form", _i), ("x_out", _vp), ("stream_enc", _i), ("stream_enc_out", _i),
                ("scratch", _vp), ("scratch_bytes", _sz), ("lens", _vp)]


class ResampleItem(ctypes.Structure):
    """struct vfx_resample_item (include/vfx_b200.h)."""
    _fields_ = [("x_off", _ll), ("x_first", _ll), ("n_in", _ll), ("y_first", _ll), ("h_off", _ll),
                ("x_len", _i), ("y_len", _i), ("up", _i), ("down", _i), ("rem", _i), ("h_len", _i)]


class ResampleSrcItem(ctypes.Structure):
    """struct vfx_resample_src_item (include/vfx_b200.h)."""
    _fields_ = [("src", _vp), ("stride", _ll), ("n_in", _ll), ("y_first", _ll), ("h_off", _ll),
                ("y_len", _i), ("up", _i), ("down", _i), ("rem", _i), ("h_len", _i)]


class ScatterItem(ctypes.Structure):
    """struct vfx_scatter_item (include/vfx_b200.h)."""
    _fields_ = [("dst", _vp), ("dst_elems", _ll), ("dst_off", _ll), ("len", _i), ("src_off", _i)]


class Pcm16Item(ctypes.Structure):
    """struct vfx_pcm16_item (include/vfx_b200.h)."""
    _fields_ = [("rows", _vp * PCM16_MAX_CHANNELS), ("n", _ll), ("dst_off", _ll), ("C", _i)]


# name -> (restype, argtypes); must list every symbol include/vfx_b200.h declares
SIGNATURES = {
    "vfx_last_error": (_c.c_char_p, []),
    "vfx_version": (_i, []),
    "vfx_engine_create": (_i, [_c.POINTER(_vp), _i, _i]),
    "vfx_engine_destroy": (_i, [_vp]),
    "vfx_engine_set_tensor": (_i, [_vp, _c.c_char_p, _vp, _sz]),
    "vfx_engine_set_option": (_i, [_vp, _c.c_char_p, _i]),
    "vfx_engine_finalize": (_i, [_vp]),
    "vfx_launch_count": (_c.c_ulonglong, []),
    "vfx_conv_tma_launch_count": (_c.c_ulonglong, []),
    "vfx_conv_tma_store_launch_count": (_c.c_ulonglong, []),
    "vfx_profile_report": (_i, [_vp, _c.c_char_p, _sz]),
    "vfx_workspace_bytes": (_sz, [_vp, _i, _i]),
    "vfx_workspace_bytes_frames": (_sz, [_vp, _i, _i]),
    "vfx_frontend_mel": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp]),
    "vfx_analysis": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "vfx_analysis_seeded": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "vfx_vocoder": (_i, [_vp, _vp, _i, _i, _i, _vp, _i, _f, _vp, _sz, _vp]),
    "vfx_vocoder_cond": (_i, [_vp, _vp, _i, _i, _vp, _i, _f, _vp, _sz, _vp]),
    "vfx_restore": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "vfx_hf_cut": (_i, [_vp, _vp, _i, _i, _f, _vp, _vp, _vp, _sz, _vp]),
    "vfx_hf_cut_workspace_bytes": (_sz, [_i, _i]),
    "vfx_conv_gemm": (_i, [_i, _i, _c.POINTER(ConvDesc), _vp]),
    "vfx_resstack_pair": (_i, [_c.POINTER(PairDesc), _vp]),
    "vfx_resstack_pair_scratch_bytes": (_sz, []),
    "vfx_gru_layer": (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp]),
    "vfx_gru_layer_ragged": (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "vfx_restore_ragged": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "vfx_restore_ragged_mode": (_i, [_vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
    "vfx_restore_seeded": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "vfx_analysis_ragged": (_i, [_vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "vfx_analysis_workspace_bytes": (_sz, [_vp, _i, _i]),
    "vfx_hf_cut_ragged": (_i, [_vp, _vp, _i, _i, _vp, _f, _vp, _vp, _vp, _vp, _sz, _vp]),
    "vfx_vocoder_ragged": (_i, [_vp, _vp, _i, _i, _vp, _i, _vp, _f, _vp, _sz, _vp]),
    "vfx_oracle_cond": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "vfx_oracle": (_i, [_vp, _vp, _i, _i, _vp, _f, _vp, _vp, _sz, _vp]),
    "vfx_oracle_workspace_bytes": (_sz, [_vp, _i, _i]),
    "vfx_resample": (_i, [_vp, _vp, _ll, _vp, _ll, _c.POINTER(ResampleItem), _i, _vp, _i, _vp, _vp, _sz, _vp]),
    "vfx_resample_workspace_bytes": (_sz, [_i]),
    "vfx_resample_src": (_i, [_vp, _vp, _ll, _c.POINTER(ResampleSrcItem), _i, _vp, _i, _vp, _vp, _sz, _vp]),
    "vfx_resample_src_workspace_bytes": (_sz, [_i]),
    "vfx_scatter_rows": (_i, [_vp, _i, _ll, _c.POINTER(ScatterItem), _vp, _sz, _vp]),
    "vfx_scatter_rows_workspace_bytes": (_sz, [_i]),
    "vfx_pack_pcm16": (_i, [_c.POINTER(Pcm16Item), _i, _vp, _ll, _vp, _sz, _vp]),
    "vfx_pack_pcm16_workspace_bytes": (_sz, [_i]),
    "vfx_bn_stats": (_i, [_vp, _ll, _ll, _i, _ll, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    "vfx_bn_act": (_i, [_i, _vp, _ll, _ll, _i, _ll, _i, _vp, _vp, _i, _i, _i, _f, _vp, _ll, _ll, _vp]),
    "vfx_dropout_apply": (_i, [_vp, _vp, _ll, _vp]),
    "vfx_dropout_seeded": (_i, [_vp, _i, _i, _vp, _i, _vp]),
    "vfx_avgpool2x2": (_i, [_vp, _ll, _ll, _ll, _i, _i, _i, _i, _vp, _vp]),
    "vfx_mask_log_pack": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "vfx_unet_head": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "vfx_voc_normalize": (_i, [_vp, _i, _i, _i, _vp, _i, _vp, _vp, _i, _vp]),
    "vfx_reflect_pad3": (_i, [_vp, _i, _i, _i, _vp, _i, _vp]),
    "vfx_voc_post": (_i, [_vp, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _f, _vp, _vp]),
    "vfx_cast_rows": (_i, [_vp, _ll, _vp, _i, _vp]),
    "vfx_ragged_extents": (_i, [_vp, _i, _i, _vp, _vp]),
    "vfx_frame_extents": (_i, [_vp, _i, _i, _vp, _vp]),
}

_lib = None


class VfxError(RuntimeError):
    pass


def load():
    """Loads the CUDA library; raises (never falls back) when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise VfxError(
            f"{LIB_PATH} not found: the vfx_b200 CUDA extension is not built. "
            "Run `python -m voicefixer_b200.build` (needs nvcc). There is no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != VFX_OK:
        msg = load().vfx_last_error().decode("utf-8", "replace")
        codes = {-1: "invalid argument", -2: "missing weight", -3: "workspace too small",
                 -4: "CUDA error", -5: "unsupported"}
        raise VfxError(f"{what} failed ({codes.get(rc, rc)}): {msg}")

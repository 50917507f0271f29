"""The kernel-level entry points of elementwise.cu without a GPU: their bindings match the header, and every argument
check returns VFX_ERR_INVALID with a message before any CUDA call (so these calls launch nothing on any host)."""
import os
import re
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ["vfx_bn_stats", "vfx_bn_act", "vfx_dropout_apply", "vfx_avgpool2x2", "vfx_mask_log_pack", "vfx_unet_head",
           "vfx_voc_normalize", "vfx_reflect_pad3", "vfx_voc_post", "vfx_cast_rows", "vfx_ragged_extents",
           "vfx_frame_extents"]


def _header_args(name):
    hdr = open(os.path.join(ROOT, "include", "vfx_b200.h")).read()
    m = re.search(r"\b" + name + r"\((.*?)\);", hdr, flags=re.S)
    assert m, name
    return [a.strip() for a in m.group(1).split(",")]


@pytest.mark.parametrize("name", ENTRIES)
def test_entry_bound_like_the_header(name):
    from voicefixer_b200 import _lib
    assert name in _lib.SIGNATURES
    assert hasattr(_lib.load(), name)
    args = _header_args(name)
    types = _lib.SIGNATURES[name][1]
    assert len(types) == len(args)
    assert [i for i, a in enumerate(args) if a.startswith("float ")] == [i for i, t in enumerate(types) if t is _lib._f]
    assert [i for i, a in enumerate(args) if a.startswith("long long ")] == \
        [i for i, t in enumerate(types) if t is _lib._ll]
    assert [i for i, a in enumerate(args) if a.startswith("int ")] == [i for i, t in enumerate(types) if t is _lib._i]
    assert args[-1] == "void* stream"


# Device pointers are never dereferenced by a refused call: fake, 256-byte-aligned addresses stand in for them.
P, Q, R, S, U = 0x1000, 0x2000, 0x3000, 0x4000, 0x5000
MIS4 = 0x1004                         # 4-byte aligned, not 16
FP32, BF16, TF32 = 0, 1, 2


def _bn_stats(**kw):
    a = dict(x=P, x_sB=64 * 32, ldx=32, B=2, P=64, C=32, bn_C=32, gamma=Q, beta=R, scale=S, shift=U, acc=0x6000,
             seq=None, per_row=1)
    a.update(kw)
    return ("vfx_bn_stats", list(a.values()))


def _bn_act(**kw):
    a = dict(prec=FP32, x=P, x_sB=64 * 32, ldx=32, B=2, P=64, C=32, scale=Q, shift=R, bn_C=32, stat_sB=32, act=1,
             p=0.01, y=S, y_sB=64 * 32, ldy=32)
    a.update(kw)
    return ("vfx_bn_act", list(a.values()))


def _avgpool(**kw):
    a = dict(x=P, sB=8 * 8 * 64, sH=8 * 64, sW=64, B=2, H=8, W=8, C=32, y=Q)
    a.update(kw)
    return ("vfx_avgpool2x2", list(a.values()))


def _mlp(**kw):
    a = dict(lin=P, mel=Q, B=2, T=100, Tp=128, ext=None, xlog=R, unet_in=S)
    a.update(kw)
    return ("vfx_mask_log_pack", list(a.values()))


def _head(**kw):
    a = dict(x=P, B=2, T=100, Tp=128, w=Q, bias=R, xlog=S, out=U)
    a.update(kw)
    return ("vfx_unet_head", list(a.values()))


def _norm(**kw):
    a = dict(mel=P, B=2, T=100, Tc=104, ext=None, is_log=1, tab=Q, cond=R, prec=FP32)
    a.update(kw)
    return ("vfx_voc_normalize", list(a.values()))


def _pad(**kw):
    a = dict(buf=P, B=2, L=100, C=512, ext=None, prec=BF16)
    a.update(kw)
    return ("vfx_reflect_pad3", list(a.values()))


def _post(**kw):
    a = dict(x=P, B=2, L=4410, w=Q, bias=R, lo=0, out_len=4410, ext_gen=None, ext_len=None, scale=1.0, out=S)
    a.update(kw)
    return ("vfx_voc_post", list(a.values()))


CASES = {
    "bn_stats_null_x": (_bn_stats(x=None), "bn_stats: null pointer"),
    "bn_stats_null_acc": (_bn_stats(acc=None), "bn_stats: null pointer"),
    "bn_stats_B0": (_bn_stats(B=0), "bn_stats: bad shape"),
    "bn_stats_B_grid_z": (_bn_stats(B=65536), "B <= 65535"),
    "bn_stats_P0": (_bn_stats(P=0), "bn_stats: bad shape"),
    "bn_stats_C0": (_bn_stats(C=0, bn_C=1), "bn_stats: bad shape"),
    "bn_stats_bn_C": (_bn_stats(bn_C=3), "bn_stats: bad shape"),
    "bn_stats_per_row": (_bn_stats(seq=Q, per_row=0), "per_row 0 must be positive"),
    "bn_act_null_x": (_bn_act(x=None), "bn_act: bad arguments"),
    "bn_act_null_y": (_bn_act(y=None), "bn_act: bad arguments"),
    "bn_act_B0": (_bn_act(B=0), "bn_act: bad arguments"),
    "bn_act_P0": (_bn_act(P=0), "bn_act: bad arguments"),
    "bn_act_C0": (_bn_act(C=0, bn_C=1), "bn_act: bad arguments"),
    "bn_act_ldy": (_bn_act(ldy=16), "bn_act: bad arguments"),
    "bn_act_bn_C": (_bn_act(bn_C=2), "bn_act: bad statistics layout"),
    "bn_act_precision": (_bn_act(prec=4), "precision 4"),
    "dropout_n0": (("vfx_dropout_apply", [P, Q, 0]), "dropout_apply: bad arguments"),
    "dropout_null_keep": (("vfx_dropout_apply", [P, None, 100]), "dropout_apply: bad arguments"),
    "avgpool_x_align": (_avgpool(x=MIS4), "x and y must be 16-byte aligned"),
    "avgpool_y_align": (_avgpool(y=MIS4), "x and y must be 16-byte aligned"),
    "avgpool_C": (_avgpool(C=6), "C/strides must be multiples of 4"),
    "avgpool_stride": (_avgpool(sW=66), "C/strides must be multiples of 4"),
    "avgpool_B0": (_avgpool(B=0), "avgpool: bad arguments"),
    "avgpool_null_y": (_avgpool(y=None), "avgpool: bad arguments"),
    "mask_log_pack_Tp": (_mlp(Tp=64), "mask_log_pack: bad arguments"),
    "mask_log_pack_T0": (_mlp(T=0), "mask_log_pack: bad arguments"),
    "mask_log_pack_null": (_mlp(mel=None), "mask_log_pack: bad arguments"),
    "mask_log_pack_align": (_mlp(unet_in=MIS4), "unet_in must be 8-byte aligned"),
    "unet_head_align": (_head(x=MIS4), "x must be 16-byte aligned"),
    "unet_head_T0": (_head(T=0), "unet_head: bad arguments"),
    "unet_head_null_bias": (_head(bias=None), "unet_head: bad arguments"),
    "voc_normalize_Tc0": (_norm(Tc=0), "voc_normalize: bad arguments"),
    "voc_normalize_B0": (_norm(B=0), "voc_normalize: bad arguments"),
    "voc_normalize_null_tab": (_norm(tab=None), "voc_normalize: bad arguments"),
    "voc_normalize_precision": (_norm(prec=-1), "precision -1"),
    "reflect_pad3_L3": (_pad(L=3), "too short for reflection pad 3"),
    "reflect_pad3_B0": (_pad(B=0), "reflect_pad3: bad arguments"),
    "reflect_pad3_null": (_pad(buf=None), "reflect_pad3: bad arguments"),
    "voc_post_ext_gen_alone": (_post(ext_gen=Q + 64), "ext_gen and ext_len go together"),
    "voc_post_ext_len_alone": (_post(ext_len=Q + 64), "ext_gen and ext_len go together"),
    "voc_post_B_grid_y": (_post(B=65536), "B <= 65535"),
    "voc_post_out_len0": (_post(out_len=0), "voc_post: bad arguments"),
    "voc_post_L0": (_post(L=0), "voc_post: bad arguments"),
    "voc_post_null_bias": (_post(bias=None), "voc_post: bad arguments"),
    "voc_post_trim": (_post(lo=1), "outside the generated length"),
    "voc_post_align": (_post(x=MIS4), "16-byte aligned"),
    "cast_rows_n0": (("vfx_cast_rows", [P, 0, Q, TF32]), "cast_rows: bad arguments"),
    "cast_rows_null": (("vfx_cast_rows", [None, 100, Q, TF32]), "cast_rows: bad arguments"),
    "cast_rows_precision": (("vfx_cast_rows", [P, 100, Q, 9]), "precision 9"),
    "ragged_extents_L_cap": (("vfx_ragged_extents", [P, 2, 1024, Q]), "ragged_extents: bad arguments"),
    "ragged_extents_B0": (("vfx_ragged_extents", [P, 0, 44100, Q]), "ragged_extents: bad arguments"),
    "frame_extents_T_cap": (("vfx_frame_extents", [P, 2, 0, Q]), "frame_extents: bad arguments"),
    "frame_extents_null": (("vfx_frame_extents", [None, 2, 100, Q]), "frame_extents: bad arguments"),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_bad_call_refused_before_any_launch(case):
    from voicefixer_b200 import _lib
    lib = _lib.load()
    (name, args), match = CASES[case]
    n0 = lib.vfx_launch_count()
    rc = getattr(lib, name)(*args, None)
    assert rc == -1, f"{name} returned {rc}"
    assert re.search(match, lib.vfx_last_error().decode())
    assert lib.vfx_launch_count() == n0

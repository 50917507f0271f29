"""The fused ResStack pair's host-side switches without a GPU: the engine's one pair option, and the pair descriptor's
form and precision checks, which refuse a descriptor before anything reads its pointers."""
import ctypes
import pytest

VFX_ERR_INVALID, VFX_ERR_UNSUPPORTED = -1, -5


def _engine(lib, prec):
    from voicefixer_b200 import _lib
    h = ctypes.c_void_p()
    _lib.check(lib.vfx_engine_create(ctypes.byref(h), -1, _lib.PREC[prec]), "vfx_engine_create")
    return h


@pytest.mark.parametrize("prec", ["tf32", "bf16", "fp16", "fp32"])
def test_engine_has_one_pair_option(prec):
    from voicefixer_b200 import _lib
    lib = _lib.load()
    h = _engine(lib, prec)
    try:
        for v in (0, 1):
            assert lib.vfx_engine_set_option(h, b"fuse_pairs", v) == 0
        for key in (b"fuse_pair", b"fuse_pair2", b"fuse_pair3"):
            assert lib.vfx_engine_set_option(h, key, 1) == VFX_ERR_INVALID
            assert b"unknown key" in lib.vfx_last_error()
    finally:
        lib.vfx_engine_destroy(h)


def _desc(**kw):
    """A C = 64 bf16 pair whose pointers are non-null but never dereferenced: every call below is refused first."""
    from voicefixer_b200 import _lib
    d = _lib.PairDesc()
    d.a, d.x, d.w1, d.b1, d.w2, d.b2 = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000
    d.dilation, d.B, d.L, d.C, d.write_raw = 1, 1, 300, 64, 1
    d.precision, d.form = _lib.PREC["bf16"], _lib.PAIR_FORM["fused"]
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("form", [2, -1])
def test_pair_refuses_unknown_form(form):
    from voicefixer_b200 import _lib
    lib = _lib.load()
    assert lib.vfx_resstack_pair(ctypes.byref(_desc(form=form)), None) == VFX_ERR_INVALID
    assert f"form {form}".encode() in lib.vfx_last_error()


@pytest.mark.parametrize("form", ["fused", "blocked"])
def test_pair_refuses_fp32(form):
    from voicefixer_b200 import _lib
    lib = _lib.load()
    d = _desc(precision=_lib.PREC["fp32"], form=_lib.PAIR_FORM[form])
    assert lib.vfx_resstack_pair(ctypes.byref(d), None) == VFX_ERR_UNSUPPORTED

"""GPU parity tests proper: the CUDA path through the C ABI against (a) the committed outputs of
the unmodified reference (tests/golden) and (b) the oracle on fresh seeded inputs.

Stated tolerances (relative RMS on fp32 values, precision "fp32" = SIMT fp32-FMA convolutions):
  stage outputs (mel, log-mel)   1e-4
  waveforms                      2e-4   (reference's own acceptance: mean-abs 1e-2, test/test.py:35)
"""
import numpy as np
import pytest
import torch
from conftest import golden, rel_rms

pytestmark = pytest.mark.gpu
TOL_STAGE, TOL_WAV = 1e-4, 2e-4


@pytest.mark.parametrize("T", [1, 63, 65, 130])
def test_analysis_vs_reference_golden(engine, T):
    g = golden(f"analysis_T{T}")
    out = engine.analysis(g["mel"][:, 0])
    assert rel_rms(out.cpu().numpy(), g["out"][:, 0]) < TOL_STAGE


def test_analysis_mode2_vs_reference_golden(engine):
    g = golden("analysis_mode2")
    T = g["mel"].shape[2]
    masks = torch.stack([torch.from_numpy(np.unpackbits(g[k])[: T * 512].reshape(1, T, 512)) for k in ("mask0", "mask1")])
    out = engine.analysis(g["mel"][:, 0], mode=2, drop_masks=masks)
    assert rel_rms(out.cpu().numpy(), g["out"][:, 0]) < 2e-4


@pytest.mark.parametrize("T", [3, 20])
def test_vocoder_vs_reference_golden(engine, T):
    g = golden(f"vocoder_T{T}")
    out = engine.vocoder(g["mel"][:, 0])
    assert out.shape[-1] == (T + T % 2 + 4) * 441
    assert rel_rms(out.cpu().numpy(), g["out"][:, 0]) < TOL_WAV


def test_restore_mode0_vs_reference_golden(engine):
    g = golden("restore_mode0")
    out = engine.restore(g["wav"][None])
    assert out.shape == (1, g["wav"].shape[0])
    assert rel_rms(out.cpu().numpy(), g["out"]) < TOL_WAV


def test_restore_batch_items_are_independent(engine, states):
    """Batched items give the same result as single items (reference batch is always 1)."""
    from voicefixer_b200 import synthetic
    wav = synthetic.make_utterances(3, seconds=0.4, seed=5)
    yb = engine.restore(wav).cpu().numpy()
    y1 = engine.restore(wav[1:2]).cpu().numpy()
    assert rel_rms(yb[1:2], y1) < 1e-6


def test_restore_vs_oracle_fresh_input(engine, states):
    from voicefixer_b200 import synthetic
    from oracle import vf_oracle as O
    wav = synthetic.make_utterances(1, seconds=0.7, seed=77)[0]
    ref = O.restore_inmem(wav, states[0], states[1], mode=0)
    out = engine.restore(wav[None]).cpu().numpy()
    assert rel_rms(out, ref) < TOL_WAV


def test_api_dropin_restore_inmem_and_segmentation(tmp_path, monkeypatch, states):
    """VoiceFixer().restore_inmem through the mirrored API with checkpoints in the reference
    layout; 30.3 s input -> two independent segments concatenated (base.py:116-138)."""
    from voicefixer_b200 import synthetic, api
    monkeypatch.setenv("HOME", str(tmp_path))
    synthetic.write_checkpoints(str(tmp_path), seed=0)
    vf = api.VoiceFixer(precision="fp32")
    g = golden("restore_mode0")
    out = vf.restore_inmem(g["wav"], cuda=True, mode=0)
    assert out.dtype == np.float32 and out.shape == g["out"].shape
    assert rel_rms(out, g["out"]) < TOL_WAV
    gs = golden("restore_segmented")
    wav = synthetic.make_utterances(1, seconds=float(gs["seconds"]), seed=int(gs["wav_seed"]))[0]
    out = vf.restore_inmem(wav, cuda=True, mode=0)
    assert out.shape == (1, wav.shape[0])
    got = np.concatenate([out[0, a:b] for a, b in gs["slices"]])
    assert rel_rms(got, gs["out_slices"]) < TOL_WAV
    assert abs(float(np.mean(np.abs(out))) - float(gs["mean_abs"])) < 1e-4
    # file API + Vocoder.forward
    from voicefixer_b200 import wavio
    wavio.save_wave(g["wav"][None], str(tmp_path / "in.wav"))
    vf.restore(str(tmp_path / "in.wav"), str(tmp_path / "out.wav"), cuda=True, mode=0)
    y = wavio.load_mono(str(tmp_path / "out.wav"))
    assert y.shape[0] == g["wav"].shape[0]
    gv = golden("vocoder_T3")
    w = vf._model.vocoder(torch.from_numpy(gv["mel"]), cuda=True)
    assert rel_rms(w.cpu().numpy(), gv["out"]) < TOL_WAV


# ---------------------------------------------------------------------------- BASELINE sizes, asserting
# One 10 s utterance (T = 1001 frames, BASELINE configs[2] item size) and one 30 s segment (T = 3001, the segment
# size of restore_inmem, voicefixer/base.py:116) against the CPU oracle on the same input and checkpoints, in every
# precision (CPU prediction of the operand-rounding error alone, tools/sim_precision.py: tf32 1.7e-3, bf16 1.3e-2
# relative RMS):
#   fp32   rel-RMS 2e-4
#   tf32   rel-RMS 2e-3, mean-abs 1e-3      (SURVEY 8d's figure; measured 1.65e-3 / 3.5e-4 on the 10 s utterance)
#   fp16   as tf32: the same 10-bit mantissa (CPU prediction 1.64e-3), 2-byte operands, fp16's exponent range
#   bf16   rel-RMS 3e-2,   mean-abs 5e-3    (reference's own CPU<->GPU acceptance bar: mean-abs 1e-2, test/test.py:35)
FULL_TOL = {"fp32": (2e-4, 1e-4), "tf32": (2e-3, 1e-3), "fp16": (2e-3, 1e-3), "bf16": (3e-2, 5e-3)}


@pytest.fixture(scope="module")
def oracle_10s(states):
    from voicefixer_b200 import synthetic
    from oracle import vf_oracle as O
    wav = synthetic.make_utterances(1, seconds=10.0, seed=1234)[0]
    return wav, O.restore_inmem(wav, states[0], states[1], mode=0)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("prec", ["fp32", "tf32", "fp16", "bf16"])
def test_restore_10s_vs_oracle(states, oracle_10s, prec):
    from voicefixer_b200.engine import Engine
    wav, ref = oracle_10s
    assert 1 + wav.shape[0] // 441 == 1001
    out = Engine(states[0], states[1], precision=prec).restore(wav[None]).cpu().numpy()
    tol_rms, tol_mae = FULL_TOL[prec]
    assert out.shape == ref.shape
    assert rel_rms(out, ref) < tol_rms
    assert float(np.mean(np.abs(out - ref))) < tol_mae


@pytest.mark.timeout(900)
def test_restore_30s_segment_vs_oracle(states):
    """T = 3001: one full restore_inmem segment, tensor-core precisions."""
    from voicefixer_b200 import synthetic
    from voicefixer_b200.engine import Engine
    from oracle import vf_oracle as O
    wav = synthetic.make_utterances(1, seconds=30.0, seed=4321)[0]
    assert 1 + wav.shape[0] // 441 == 3001
    ref = O.restore_inmem(wav, states[0], states[1], mode=0)
    for prec in ("tf32", "fp16", "bf16"):
        out = Engine(states[0], states[1], precision=prec).restore(wav[None]).cpu().numpy()
        tol_rms, tol_mae = FULL_TOL[prec]
        assert rel_rms(out, ref) < tol_rms, prec
        assert float(np.mean(np.abs(out - ref))) < tol_mae, prec


def test_full_size_properties(engine):
    """BASELINE config sizes (10 s items): output length, finiteness, |y| <= 1, batch
    permutation equivariance (a size-independent property of independent items)."""
    from voicefixer_b200 import synthetic
    wav = torch.from_numpy(synthetic.make_utterances(2, seconds=10.0, seed=9)).cuda()
    y = engine.restore(wav)
    assert y.shape == wav.shape and bool(torch.isfinite(y).all()) and float(y.abs().max()) <= 1.0
    y2 = engine.restore(wav.flip(0))
    assert rel_rms(y2.flip(0).cpu().numpy(), y.cpu().numpy()) < 1e-6


# ---------------------------------------------------------------------------- bf16 tensor-core path
# Stated tolerances for precision "bf16" (wgmma: bf16 operands, fp32 accumulation, fp32 bias / residual stream /
# activations), with margin over the error of bf16 rounding against the reference goldens.
TOL_BF16_STAGE, TOL_BF16_WAV, TOL_BF16_MAE = 1.5e-2, 3e-2, 5e-3      # reference's own bar: mean-abs 1e-2


@pytest.fixture(scope="module")
def engine_bf16(states):
    from voicefixer_b200.engine import Engine
    return Engine(states[0], states[1], precision="bf16")


@pytest.mark.parametrize("T", [1, 65, 130])
def test_bf16_analysis_vs_reference_golden(engine_bf16, T):
    g = golden(f"analysis_T{T}")
    assert rel_rms(engine_bf16.analysis(g["mel"][:, 0]).cpu().numpy(), g["out"][:, 0]) < TOL_BF16_STAGE


@pytest.mark.parametrize("T", [3, 20])
def test_bf16_vocoder_vs_reference_golden(engine_bf16, T):
    g = golden(f"vocoder_T{T}")
    out = engine_bf16.vocoder(g["mel"][:, 0]).cpu().numpy()
    assert rel_rms(out, g["out"][:, 0]) < TOL_BF16_WAV
    assert float(np.mean(np.abs(out - g["out"][:, 0]))) < TOL_BF16_MAE


def test_bf16_restore_vs_reference_golden(engine_bf16):
    g = golden("restore_mode0")
    out = engine_bf16.restore(g["wav"][None]).cpu().numpy()
    assert rel_rms(out, g["out"]) < TOL_BF16_WAV
    assert float(np.mean(np.abs(out - g["out"]))) < TOL_BF16_MAE


def test_bf16_tensor_core_path_equals_simt_bf16(engine_bf16, states):
    """Same bf16 operands through the SIMT kernel.  Accumulation order, fast-math activations and
    bf16 rounding ties differ, and through ~200 layers two bf16 pipelines decorrelate to the bf16
    noise floor (the same ~1e-2 both show against the fp32 reference)."""
    from voicefixer_b200 import synthetic
    wav = synthetic.make_utterances(2, seconds=0.5, seed=13)
    y_tc = engine_bf16.restore(wav).cpu().numpy()
    engine_bf16.set_option("use_tc", 0)
    y_simt = engine_bf16.restore(wav).cpu().numpy()
    engine_bf16.set_option("use_tc", 1)
    assert rel_rms(y_tc, y_simt) < TOL_BF16_WAV


def test_bf16_mode2_vs_reference_golden(engine_bf16):
    g = golden("analysis_mode2")
    T = g["mel"].shape[2]
    masks = torch.stack([torch.from_numpy(np.unpackbits(g[k])[: T * 512].reshape(1, T, 512)) for k in ("mask0", "mask1")])
    out = engine_bf16.analysis(g["mel"][:, 0], mode=2, drop_masks=masks)
    assert rel_rms(out.cpu().numpy(), g["out"][:, 0]) < 3e-2


# ---------------------------------------------------------------------------- tf32 tensor-core path
# precision "tf32": wgmma tf32 on fp32 storage, every operand rounded to tf32 by its producer, fp32
# accumulation -- the arithmetic class of the reference's own CUDA path (cuDNN TF32 convolutions, SURVEY D10).
TOL_TF32_STAGE, TOL_TF32_WAV, TOL_TF32_MAE = 1e-3, 2e-3, 1e-3


@pytest.fixture(scope="module")
def engine_tf32(states):
    from voicefixer_b200.engine import Engine
    return Engine(states[0], states[1], precision="tf32")


@pytest.mark.parametrize("T", [1, 63, 65, 130])
def test_tf32_analysis_vs_reference_golden(engine_tf32, T):
    g = golden(f"analysis_T{T}")
    assert rel_rms(engine_tf32.analysis(g["mel"][:, 0]).cpu().numpy(), g["out"][:, 0]) < TOL_TF32_STAGE


@pytest.mark.parametrize("T", [3, 20])
def test_tf32_vocoder_vs_reference_golden(engine_tf32, T):
    g = golden(f"vocoder_T{T}")
    out = engine_tf32.vocoder(g["mel"][:, 0]).cpu().numpy()
    assert rel_rms(out, g["out"][:, 0]) < TOL_TF32_WAV
    assert float(np.mean(np.abs(out - g["out"][:, 0]))) < TOL_TF32_MAE


def test_tf32_restore_vs_reference_golden(engine_tf32):
    g = golden("restore_mode0")
    out = engine_tf32.restore(g["wav"][None]).cpu().numpy()
    assert rel_rms(out, g["out"]) < TOL_TF32_WAV
    assert float(np.mean(np.abs(out - g["out"]))) < TOL_TF32_MAE


def test_tf32_tensor_core_path_equals_simt_on_same_operands(engine_tf32):
    """tf32 x tf32 products are exact in fp32: the SIMT kernel on the same rounded operands differs from the wgmma
    kernel only by accumulation order, far below the tf32 rounding noise."""
    from voicefixer_b200 import synthetic
    wav = synthetic.make_utterances(2, seconds=0.5, seed=13)
    y_tc = engine_tf32.restore(wav).cpu().numpy()
    engine_tf32.set_option("use_tc", 0)
    y_simt = engine_tf32.restore(wav).cpu().numpy()
    engine_tf32.set_option("use_tc", 1)
    assert rel_rms(y_tc, y_simt) < TOL_TF32_WAV


def test_tf32_mode2_vs_reference_golden(engine_tf32):
    g = golden("analysis_mode2")
    T = g["mel"].shape[2]
    masks = torch.stack([torch.from_numpy(np.unpackbits(g[k])[: T * 512].reshape(1, T, 512)) for k in ("mask0", "mask1")])
    out = engine_tf32.analysis(g["mel"][:, 0], mode=2, drop_masks=masks)
    assert rel_rms(out.cpu().numpy(), g["out"][:, 0]) < 4e-3


def test_tf32_encoded_stream_engine_path(states, oracle_10s):
    """tf32 with the encoded vocoder stream (one fp32 tensor as operand + residual carrier): same tolerance as plain tf32,
    and within rounding noise of it."""
    from voicefixer_b200.engine import Engine
    wav, ref = oracle_10s
    eng = Engine(states[0], states[1], precision="tf32")
    eng.set_option("tf32_stream", 0)
    y0 = eng.restore(wav[None]).cpu().numpy()
    eng.set_option("tf32_stream", 1)
    y1 = eng.restore(wav[None]).cpu().numpy()
    assert rel_rms(y1, ref) < FULL_TOL["tf32"][0] and float(np.mean(np.abs(y1 - ref))) < FULL_TOL["tf32"][1]
    assert rel_rms(y1, y0) < FULL_TOL["tf32"][0]


@pytest.mark.parametrize("prec", ["tf32", "fp16", "bf16"])
def test_fused_pairs_engine_path(states, oracle_10s, prec):
    """fuse_pairs: every ResStack pair the fused kernel supports (tf32: C = 64 on the encoded stream; 16-bit: C = 64 and
    128) as one kernel (1, the default) or as its two convolution launches (0).  The fused kernel adds the same slices in
    the same order as the convolution: the two runs give the same bits, and both meet the mode's tolerance."""
    from voicefixer_b200.engine import Engine
    wav, ref = oracle_10s
    eng = Engine(states[0], states[1], precision=prec)
    eng.set_option("fuse_pairs", 0)
    y0 = eng.restore(wav[None]).cpu().numpy()
    eng.set_option("fuse_pairs", 1)
    y1 = eng.restore(wav[None]).cpu().numpy()
    for y in (y0, y1):
        assert rel_rms(y, ref) < FULL_TOL[prec][0] and float(np.mean(np.abs(y - ref))) < FULL_TOL[prec][1]
    assert np.array_equal(y1, y0), f"max |fused - unfused| {np.max(np.abs(y1 - y0)):.3e}, rel-rms {rel_rms(y1, y0):.3e}"


# ---------------------------------------------------------------------------- fp16 tensor-core path
# precision "fp16": the bf16 mode's kernels (fused ResStack pairs included) with the other 16-bit operand format.  fp16
# carries tf32's 10-bit mantissa, so the tolerances are tf32's.
@pytest.fixture(scope="module")
def engine_fp16(states):
    from voicefixer_b200.engine import Engine
    return Engine(states[0], states[1], precision="fp16")


@pytest.mark.parametrize("T", [1, 65, 130])
def test_fp16_analysis_vs_reference_golden(engine_fp16, T):
    g = golden(f"analysis_T{T}")
    assert rel_rms(engine_fp16.analysis(g["mel"][:, 0]).cpu().numpy(), g["out"][:, 0]) < TOL_TF32_STAGE


@pytest.mark.parametrize("T", [3, 20])
def test_fp16_vocoder_vs_reference_golden(engine_fp16, T):
    g = golden(f"vocoder_T{T}")
    out = engine_fp16.vocoder(g["mel"][:, 0]).cpu().numpy()
    assert rel_rms(out, g["out"][:, 0]) < TOL_TF32_WAV
    assert float(np.mean(np.abs(out - g["out"][:, 0]))) < TOL_TF32_MAE


def test_fp16_restore_and_simt_cross_check(engine_fp16):
    g = golden("restore_mode0")
    out = engine_fp16.restore(g["wav"][None]).cpu().numpy()
    assert rel_rms(out, g["out"]) < TOL_TF32_WAV
    engine_fp16.set_option("use_tc", 0)
    y_simt = engine_fp16.restore(g["wav"][None]).cpu().numpy()
    engine_fp16.set_option("use_tc", 1)
    assert rel_rms(out, y_simt) < TOL_TF32_WAV


def test_cuda_graph_replay_matches_direct_launch(engine_bf16):
    """Engine.make_graph: the captured launch sequence reproduces the direct run bit for bit."""
    from voicefixer_b200 import synthetic
    wav = torch.from_numpy(synthetic.make_utterances(2, seconds=0.5, seed=17)).cuda()
    ref = engine_bf16.restore(wav).clone()
    out = torch.empty_like(wav)
    g = engine_bf16.make_graph(wav, out)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


@pytest.mark.timeout(240)
def test_api_modes_1_2_and_vocoder_oracle(tmp_path, monkeypatch, states):
    """restore_inmem modes 1 / 2 and Vocoder.oracle through the mirrored API, against the oracle."""
    from voicefixer_b200 import synthetic, api, wavio
    from oracle import vf_oracle as O
    monkeypatch.setenv("HOME", str(tmp_path))
    synthetic.write_checkpoints(str(tmp_path), seed=0)
    vf = api.VoiceFixer(precision="fp32")
    wav = synthetic.make_utterances(1, seconds=0.6, seed=51)[0]
    out1 = vf.restore_inmem(wav, cuda=True, mode=1)                         # mode 1: pre-filter, shorter output
    ref1 = O.restore_inmem(wav, states[0], states[1], mode=1)
    assert out1.shape == ref1.shape == (1, 512 * (wav.shape[0] // 512))
    # mode 1: measured 3.7e-6 on an H100 (700 W).  The pre-filter agrees with the oracle's to 1.4e-7; when its
    # overlap-add left frame 0 out of samples 513..1023 this was 2.6e-4.
    assert rel_rms(out1, ref1) < 2e-5
    # mode 2 (train-mode BN, no dropout masks): <= 64 frames is an error in the reference too (1x1 UNet centre)
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        vf.restore_inmem(wav, cuda=True, mode=2)
    wav2 = synthetic.make_utterances(1, seconds=1.6, seed=53)[0]
    out2 = vf.restore_inmem(wav2, cuda=True, mode=2, drop_masks_fn=False)   # train-mode BN only: deterministic
    ref2 = O.restore_inmem(wav2, states[0], states[1], mode=2)
    assert out2.shape == (1, wav2.shape[0]) and rel_rms(out2, ref2) < 5e-4
    # explicit masks through the API == the oracle with the same masks; the default draws them from torch's RNG
    T2 = 1 + wav2.shape[0] // 441
    keep = torch.rand(2, 1, T2, 512, generator=torch.Generator().manual_seed(5)) >= 0.5
    out2m = vf.restore_inmem(wav2, cuda=True, mode=2, drop_masks_fn=lambda B, T: keep)
    ref2m = O.restore_inmem(wav2, states[0], states[1], mode=2, drop_masks_fn=lambda T: keep[:, :1])
    assert rel_rms(out2m, ref2m) < 5e-4 and rel_rms(out2m, out2) > 1e-2
    torch.manual_seed(11)
    out2r = vf.restore_inmem(wav2, cuda=True, mode=2)                        # reference default: random dropout
    assert out2r.shape == out2.shape and np.isfinite(out2r).all() and rel_rms(out2r, out2) > 1e-2
    with pytest.raises(ValueError, match="dropout masks must have shape"):
        vf.restore_inmem(wav2, cuda=True, mode=2, drop_masks_fn=lambda B, T: keep[:, :, :-1])
    with pytest.raises(ValueError):
        vf.restore_inmem(wav, cuda=True, mode=3)
    # Vocoder.oracle: wav file -> |STFT| -> Slaney mel -> Generator -> int16 wav file (vocoder/base.py:58-77)
    src = synthetic.make_utterances(1, seconds=0.4, seed=52)[0]
    wavio.save_wave(src[None], str(tmp_path / "src.wav"))
    voc = api.Vocoder(44100, _engine=vf._engine)
    voc.oracle(str(tmp_path / "src.wav"), str(tmp_path / "orc.wav"), cuda=True)
    got = wavio.load_mono(str(tmp_path / "orc.wav"))
    x16 = wavio.load_mono(str(tmp_path / "src.wav"))                         # what oracle() actually read (int16 round trip)
    ref = O.oracle_wave(x16, states[1])[0, 0] / 2 ** 15
    assert got.shape == ref.shape and float(np.mean(np.abs(got - ref))) < 2e-4

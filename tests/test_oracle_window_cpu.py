"""The host front end of Vocoder.oracle (api.oracle_conditions) and the CPU oracle's (vf_oracle.oracle_cond) window
the frames as librosa 0.10.1's stft does: get_window returns the periodic Hann in float64, and stft multiplies the
float32 frames by it without a cast, so the windowed frames are float64.  A float32 window product moves the
conditions of a full-scale 1 kHz tone by about 1e-3 (the far mel bands sit at the product's rounding floor)."""
import numpy as np

SR = 44100


def _cond(wav, window_dtype):
    """librosa's arithmetic written out, with the window (and hence the product) in `window_dtype`"""
    from voicefixer_b200 import wavio
    w = np.asarray(wav, np.float32)
    w = w / np.max(np.abs(w))
    win = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(2048) / 2048)).astype(window_dtype)
    x = np.pad(w, (1024, 1024))
    T = 1 + (len(x) - 2048) // 441
    idx = np.arange(2048)[None, :] + 441 * np.arange(T)[:, None]
    mag = np.abs(np.fft.rfft(x[idx] * win[None, :], axis=1).astype(np.complex64))
    mel = mag.astype(np.float64) @ wavio.slaney_htk_mel_basis().astype(np.float64).T
    S = 20 * np.log10(np.maximum(np.exp(-100 / 20 * np.log(10)), np.abs(mel))) - 20
    S = np.clip(8.0 * ((S + 115.0) / 115.0) - 4.0, -4.0, 4.0)
    return np.concatenate([S, np.full((T % 2 + 4, 128), -4.0)])


def _tone_1k():
    t = np.arange(2 * SR) / SR
    return np.sin(2 * np.pi * 1000.0 * t).astype(np.float32)


def test_oracle_conditions_window_product_is_float64():
    from voicefixer_b200.api import oracle_conditions
    from oracle import vf_oracle as O
    wav = _tone_1k()
    ref = _cond(wav, np.float64)
    host = oracle_conditions(wav)[0]
    cpu_oracle = O.oracle_cond(wav).numpy()[0].T
    assert host.shape == cpu_oracle.shape == ref.shape
    assert np.max(np.abs(host - ref)) <= 1e-6
    assert np.max(np.abs(cpu_oracle - ref)) <= 1e-6
    # the same restatement with a float32 window product is far off: the bound above can tell the two apart
    assert np.max(np.abs(_cond(wav, np.float32) - ref)) > 1e-4

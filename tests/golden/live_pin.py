"""Live pin of the oracle against the UNMODIFIED reference on inputs that are NOT in the committed fixtures.

    python tests/golden/live_pin.py [seed] [--save]   # needs the reference checkout; prints one JSON line

--save writes tests/golden/live_pin.npz: the seed, the dropout masks the reference drew, and each case's reference output
as a fixed seeded sample of 512 elements, which tests/test_oracle.py checks the oracle against without the reference.

Same loading recipe as make_golden.py (stub-loader + seeded synthetic checkpoints under a temporary HOME, loaded by
the reference's own VoiceFixer() / Vocoder(44100)).  Cases: analysis at T in {2, 64, 128, 257} (pad/crop edges of the
64-frame UNet grid), Vocoder.forward at odd and even T, restore_inmem mode 0 on 1.3 s, restore_inmem mode 2
(train-mode BN + the dropout masks the reference actually drew, captured by forward hooks), and the
your_vocoder_func hook (base.py:126-129)."""
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)


SAMPLE = 512


def cases(seed, ana, voc, ref_fns, masks=None):
    """name -> output for every case; ref_fns: the reference's callables, or None for the oracle's (with `masks`)."""
    import torch
    from voicefixer_b200 import synthetic
    from oracle import vf_oracle as O
    out = {}
    for T in (2, 64, 128, 257):
        m = torch.rand(1, 1, T, 128, generator=torch.Generator().manual_seed(seed + T)) ** 4 * 30.0
        out[f"analysis_T{T}"] = ref_fns["analysis"](m) if ref_fns else O.analysis(m, ana)
    for T in (5, 12):
        m = torch.rand(1, 1, T, 128, generator=torch.Generator().manual_seed(seed + 500 + T)) ** 4 * 30.0
        out[f"vocoder_T{T}"] = ref_fns["vocoder"](m) if ref_fns else O.vocoder_forward(m, voc)
    wav = synthetic.make_utterances(1, seconds=1.3, seed=seed + 1)[0]
    out["restore_mode0_1.3s"] = ref_fns["restore0"](wav) if ref_fns else O.restore_inmem(wav, ana, voc, mode=0)
    wav2 = synthetic.make_utterances(1, seconds=1.6, seed=seed + 2)[0]
    out["restore_mode2_1.6s"] = (ref_fns["restore2"](wav2) if ref_fns else
                                 O.restore_inmem(wav2, ana, voc, mode=2, drop_masks_fn=lambda T: masks))
    if ref_fns:
        out["hook_mel"], out["hook_out"] = ref_fns["hook"](wav)
    else:
        _, mel = O.frontend(torch.from_numpy(wav)[None], ana)
        o_mel = O.from_log(O.analysis(mel, ana))
        out["hook_mel"] = o_mel
        out["hook_out"] = O.trim_center(O.vocoder_forward(o_mel, voc) * 0.5, wav.shape[0]).squeeze(0).numpy()
    return {k: np.asarray(v, np.float32) for k, v in out.items()}


def main(seed, save=False):
    os.environ["HOME"] = tempfile.mkdtemp(prefix="vfx_home_")
    import torch
    torch.set_num_threads(8)
    from voicefixer_b200 import synthetic
    from oracle import vf_oracle as O
    synthetic.write_checkpoints(os.environ["HOME"], seed=0)
    ana, voc = synthetic.make_analysis_state(0), synthetic.make_vocoder_state(1)
    import ref_loader
    ref_loader.install()
    from voicefixer.base import VoiceFixer as RefVoiceFixer          # unmodified reference
    from voicefixer.vocoder.base import Vocoder as RefVocoder
    ref, ref_voc = RefVoiceFixer(), RefVocoder(44100)
    model = ref._model

    def rel(a, b):
        a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
        assert a.shape == b.shape, (a.shape, b.shape)
        return float(np.sqrt(np.mean((a - b) ** 2)) / (np.sqrt(np.mean(b ** 2)) + 1e-30))

    def restore2(wav2):
        # mode 2 end to end: capture the masks the reference's two Dropout(0.5) drew (x2 scaling: kept <=> out != 0)
        hooks = []
        for mod in model.generator.denoiser:
            if isinstance(mod, torch.nn.Dropout):
                hooks.append(mod.register_forward_hook(lambda _m, inp, outp: masks.append((outp != 0) | (inp[0] == 0))))
        torch.manual_seed(seed + 3)
        out2 = ref.restore_inmem(wav2, cuda=False, mode=2)
        for h in hooks:
            h.remove()
        return out2

    def hook(wav):
        # the your_vocoder_func hook: the reference hands the callback a linear mel [1, 1, T, 128]
        seen = {}

        def my_vocoder(mel):
            seen["mel"] = mel.clone()
            return ref_voc.forward(mel, cuda=False) * 0.5
        ref2 = RefVoiceFixer()                                           # fresh module (mode 2 above moved BN running stats)
        out3 = ref2.restore_inmem(wav, cuda=False, mode=0, your_vocoder_func=my_vocoder)
        return seen["mel"], out3

    masks = []
    fns = {"analysis": lambda m: model(None, m)["mel"], "vocoder": lambda m: ref_voc.forward(m, cuda=False),
           "restore0": lambda w: ref.restore_inmem(w, cuda=False, mode=0), "restore2": restore2, "hook": hook}
    with torch.no_grad():
        got_ref = cases(seed, ana, voc, fns)
        got = cases(seed, ana, voc, None, masks)
    rep = {k: rel(got[k], got_ref[k]) for k in got}
    if save:
        rng = np.random.default_rng(seed)
        arrs = {"seed": np.array(seed)}
        for i, mk in enumerate(masks):
            arrs[f"mask{i}"] = np.packbits(mk.numpy().astype(np.uint8))
            arrs[f"mask{i}_shape"] = np.array(mk.shape)
        for k, v in got_ref.items():
            idx = np.sort(rng.choice(v.size, min(v.size, SAMPLE), replace=False))
            arrs[k + ".shape"], arrs[k + ".idx"], arrs[k + ".ref"] = np.array(v.shape), idx.astype(np.int32), v.ravel()[idx]
        np.savez_compressed(os.path.join(HERE, "live_pin.npz"), **arrs)
    print(json.dumps(rep))


if __name__ == "__main__":
    args = [a for a in sys.argv[1:] if a != "--save"]
    main(int(args[0]) if args else 9000, save="--save" in sys.argv)

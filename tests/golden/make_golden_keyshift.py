"""Generates tests/golden/keyshift.npz by EXECUTING THE UNMODIFIED reference MelSpectrogram (modules/rmvpe/spec.py) on CPU
through oracle/refshim.py for keyshift in {-5 .. +5}, plus one fractional shift, one speed != 1 and one center=False case.  The
binarizer's pitch augmentation (preprocessing/me_binarizer.py:235-247) draws from key_shift_range, [-12, 12] in both shipped
configs; make_golden_keyshift_wide.py covers the shifts beyond +-5.  Build container only; outputs are committed.

    python tests/golden/make_golden_keyshift.py
"""
import pathlib
import sys

import numpy as np
import torch

HERE = pathlib.Path(__file__).resolve().parent
REPO = HERE.parent.parent
sys.path.insert(0, str(REPO))

from oracle import refshim  # noqa: E402
from some_b200 import synth  # noqa: E402


def main():
    torch.set_num_threads(1)
    refshim.load_reference()
    import modules.rmvpe as ref_rmvpe
    mel = ref_rmvpe.MelSpectrogram(n_mel_channels=80, sampling_rate=44100, win_length=2048, hop_length=512,
                                   mel_fmin=40, mel_fmax=8000)
    wave = synth.synth_waveform(4242, seconds=1.2)
    audio = torch.from_numpy(wave).unsqueeze(0)
    out = {'seed': np.int64(4242), 'seconds': np.float64(1.2)}
    with torch.no_grad():
        for ks in range(-5, 6):
            out[f'ks_{ks}'] = mel(audio, keyshift=ks)[0].numpy()
        out['ks_frac_2.37'] = mel(audio, keyshift=2.37)[0].numpy()            # non-integer shift (round_midi: false)
        out['speed_1.25'] = mel(audio, keyshift=0, speed=1.25)[0].numpy()
        out['nocenter_ks3'] = mel(audio, keyshift=3, center=False)[0].numpy()
    np.savez_compressed(HERE / 'keyshift.npz', **out)
    print({k: v.shape for k, v in out.items() if hasattr(v, 'shape') and v.ndim == 2})


if __name__ == '__main__':
    main()

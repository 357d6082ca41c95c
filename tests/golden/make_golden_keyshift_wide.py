"""Generates tests/golden/keyshift_wide.npz by EXECUTING THE UNMODIFIED reference MelSpectrogram (modules/rmvpe/spec.py) on CPU
through oracle/refshim.py, across the key shifts both shipped configs draw from (key_shift_range: [-12, 12], configs/continuous.yaml
and configs/discrete.yaml; fractional when round_midi is off, preprocessing/me_binarizer.py:235-247): every integer shift in
[-12, -6] and [6, 12] (keyshift.npz has -5..5), the fractional shifts +-0.5, 7.3, -11.9 and 11.99, center=False at +-12 and
speed 0.8 and 2.0 at +12, each on two signals (mel_f64.wide_signals), plus the shortest audio torch.stft accepts at +12
(center=False, 4096 samples = n_fft').  The archive is written with fixed zip timestamps, so rerunning this script
reproduces the committed file byte for byte.  Build container only; outputs are committed.

    python tests/golden/make_golden_keyshift_wide.py [OUT.npz]
"""
import io
import pathlib
import sys
import zipfile

import numpy as np
import torch

HERE = pathlib.Path(__file__).resolve().parent
REPO = HERE.parent.parent
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(HERE))

from mel_f64 import SR, WIDE_CASES, WIDE_SECONDS, loud_over_quiet, wide_signals  # noqa: E402
from oracle import refshim  # noqa: E402

SHORTEST_KS12 = 4096   # n + pad_total == n_fft' at +12 with center=False


def save_npz(path, arrays):
    """np.savez_compressed with every member dated 1980-01-01, so the bytes depend on the arrays only"""
    with zipfile.ZipFile(path, 'w', compression=zipfile.ZIP_DEFLATED) as z:
        for name, a in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(a), allow_pickle=False)
            info = zipfile.ZipInfo(name + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def compute():
    torch.set_num_threads(1)
    refshim.load_reference()
    import modules.rmvpe as ref_rmvpe
    mel = ref_rmvpe.MelSpectrogram(n_mel_channels=80, sampling_rate=SR, win_length=2048, hop_length=512,
                                   mel_fmin=40, mel_fmax=8000)
    out = {'seconds': np.float64(WIDE_SECONDS)}
    with torch.no_grad():
        for sig, wave in wide_signals().items():
            audio = torch.from_numpy(wave).unsqueeze(0)
            for key, kw in WIDE_CASES:
                out[f'{sig}/{key}'] = mel(audio, **kw)[0].numpy()              # [80, T]
        short = torch.from_numpy(loud_over_quiet(SHORTEST_KS12)).unsqueeze(0)
        out['shortest_ks12'] = mel(short, keyshift=12, center=False)[0].numpy()
    return out


def main(path):
    out = compute()
    save_npz(path, out)
    print({k: v.shape for k, v in out.items() if v.ndim == 2})


if __name__ == '__main__':
    main(pathlib.Path(sys.argv[1]) if len(sys.argv) > 1 else HERE / 'keyshift_wide.npz')

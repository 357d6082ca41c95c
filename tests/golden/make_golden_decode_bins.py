"""Generates tests/golden/decode_bins.npz by EXECUTING THE UNMODIFIED REFERENCE decode (utils/infer_utils.py) through
oracle/refshim.py (build container only): decode_gaussian_blurred_probs, decode_bounds_to_alignment and
decode_note_sequence on the order-independent probes of decode_bins_cases.py, for every head width in WIDTHS.  The
probes are regenerated in the tests from the same seeds.

    python tests/golden/make_golden_decode_bins.py
"""
import pathlib
import sys

import numpy as np
import torch

HERE = pathlib.Path(__file__).resolve().parent
REPO = HERE.parent.parent
sys.path.insert(0, str(REPO))

from oracle import refshim  # noqa: E402
sys.path.insert(0, str(HERE))
from decode_bins_cases import DEVIATION, THRESHOLD, WIDTHS, make_probe  # noqa: E402


def main():
    torch.set_num_threads(1)
    refshim.load_reference()
    import utils.infer_utils as ref_decode
    out = {}
    for n, vmin, vmax in WIDTHS:
        probs, bounds = make_probe(n, vmin, vmax)
        values, rest = ref_decode.decode_gaussian_blurred_probs(torch.from_numpy(probs)[None], vmin=vmin, vmax=vmax,
                                                                deviation=DEVIATION, threshold=THRESHOLD)
        f2i = ref_decode.decode_bounds_to_alignment(torch.from_numpy(bounds)[None])
        nm, nd, nk = ref_decode.decode_note_sequence(f2i, values, ~rest)
        key = f'n{n}_{vmin}_{vmax}'
        out[f'{key}_probs_checksum'] = np.float64(probs.astype(np.float64).sum())
        out[f'{key}_values'] = values[0].numpy()
        out[f'{key}_rest'] = rest[0].numpy()
        out[f'{key}_frame2item'] = f2i[0].numpy()
        out[f'{key}_note_midi'] = nm[0].numpy()
        out[f'{key}_note_dur'] = nd[0].numpy()
        out[f'{key}_note_mask'] = nk[0].numpy()
        print(key, probs.shape, 'notes', int(f2i.max()), 'rest frames', int(rest.sum()))
    np.savez_compressed(HERE / 'decode_bins.npz', **out)


if __name__ == '__main__':
    main()

"""Probe inputs of tests/golden/decode_bins.npz (make_golden_decode_bins.py): head widths other than the shipped 128 / 129,
fed to the reference's decode_gaussian_blurred_probs and decode_note_sequence.

Every probe gives a result that does not depend on the order in which the reference sums: a frame's window around its
argmax holds at most two non-zero weights (one-hot frames, whose value is the bin value when the weight is 1; two-hot
frames, whose value is the midpoint of two bins of equal weight; all-zero frames; maxima tied with a bin outside the
window), and the frames a note averages are either identical or at most two.  So the oracle and the kernel must give the
reference's bits exactly.  Bounds are 1 on the first frame of a note and 0 elsewhere, so every note is a known run of
frames.  Regenerated in the tests from the seeds below.
"""
import numpy as np

WIDTHS = [(200, 21, 108), (256, 0, 127), (64, 40, 103), (2, 0, 127)]
DEVIATION, THRESHOLD = 1.0, 0.1


def width_of(n, vmin, vmax):
    """infer_utils.py:11-12."""
    return int(3 * DEVIATION / ((vmax - vmin) / (n - 1)))


def make_probe(n, vmin, vmax):
    """(probs float32 [T, n], bounds float32 [T]) of the width's probes, seeded by the width."""
    rng = np.random.default_rng(1000 + n + vmin)
    w = width_of(n, vmin, vmax)
    notes = []

    def row(*hot):
        r = np.zeros(n, dtype=np.float32)
        for j, v in hot:
            r[j] = v
        return r

    zero = row()
    # every bin one-hot at weight 1 (value = the bin value), 1-3 identical frames per note
    for j in range(n):
        notes.append([row((j, 1.0))] * (1 + j % 3))
    # one-hot at random weights, above and below the rest threshold (values fl(fl(w v) / w))
    for j in rng.integers(0, n, 24):
        notes.append([row((j, np.float32(rng.uniform(0.1, 1.0))))])
        notes.append([row((j, np.float32(rng.uniform(0.01, 0.1))))])
    # two-hot of equal weight inside the window (midpoints), and of unequal weight
    for j in rng.integers(0, n - 1, 24):
        d = int(rng.integers(1, w + 1)) if w > 0 else 1
        k = min(j + d, n - 1)
        a = np.float32(rng.choice([1.0, 0.5, 0.75, rng.uniform(0.1, 1.0)]))
        notes.append([row((j, a), (k, a))] * int(rng.integers(1, 3)))
        notes.append([row((j, a), (k, np.float32(rng.uniform(0.1, 1.0))))])
    # tied maxima with bins outside the window, across lanes j / j + 32 of the kernel's warp, and three-way
    for j in range(0, n - 1, max(1, n // 16)):
        for k in (j + w + 1, j + 32, n - 1):
            if j < k < n:
                notes.append([row((j, 1.0), (k, 1.0))])
                notes.append([row((k, 1.0), (j, 0.5))])
        if j + 2 * w + 2 < n:
            notes.append([row((j, 0.5), (j + w + 1, 0.5), (j + 2 * w + 2, 0.5))])
    # all-zero frames (weight sum 0, rest): a note with no voiced frame
    notes.append([zero, zero])
    # exactly half of a note voiced (unmasked / dur = 0.5 -> not a rest), and less than half
    for j in rng.integers(0, n, 6):
        notes.append([zero, row((j, 1.0)), zero, row((j, 1.0))])
        notes.append([zero, row((j, 1.0)), zero])
    # histogram-mode ties: the first maximal rounded bin wins although the other bin comes first in the note
    idx = np.arange(n, dtype=np.float32) * np.float32((vmax - vmin) / (n - 1)) + np.float32(vmin)
    for j in rng.integers(0, n, 12):
        far = np.nonzero(np.abs(idx - idx[j]) > 1.0)[0]
        if far.size:
            k = int(rng.choice(far))
            lo, hi = (j, k) if np.rint(idx[j]) < np.rint(idx[k]) else (k, j)
            notes.append([row((hi, 1.0)), row((hi, 1.0)), row((lo, 1.0)), row((lo, 1.0))])
    # values exactly on center +- 0.5 (integer bin values: the midpoint of two neighbouring bins), on both sides
    if idx.size > 1 and idx[1] - idx[0] == 1.0:
        for j in rng.integers(0, n - 1, 8):
            mid = row((j, 1.0), (j + 1, 1.0))
            notes.append([row((j, 1.0)), mid, row((j, 1.0))])
            notes.append([row((j + 1, 1.0)), mid, row((j + 1, 1.0))])
    order = rng.permutation(len(notes))
    probs, bounds = [], []
    for i in order:
        probs += notes[i]
        bounds += [1.0] + [0.0] * (len(notes[i]) - 1)
    return np.stack(probs).astype(np.float32), np.asarray(bounds, dtype=np.float32)

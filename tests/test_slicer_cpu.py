"""CPU tests of the slicer row (SURVEY.md §8f-1): the oracle restatement against the golden vectors produced by the
unmodified reference (tests/golden/make_golden_slicer.py), and the native slicer's decisions (some_slicer_ranges,
csrc/slicer.cu: run-based, on the host) against the oracle's frame-by-frame walk.  The RMS kernel itself is tested on the
GPU (tests/test_gpu_slicer.py), the incremental slicer in tests/test_stream_cpu.py."""
import pathlib
import sys

import numpy as np
import pytest

HERE = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / 'golden'))

from oracle import slicer as osl  # noqa: E402
from slicer_cases import CASES, make_case  # noqa: E402
from some_b200 import _lib  # noqa: E402
from some_b200 import slicer as psl  # noqa: E402

GOLD = np.load(HERE / 'golden' / 'slicer.npz')
SLICER_DEFAULTS = dict(threshold=-40., min_length=5000, min_interval=300, hop_size=20, max_sil_kept=5000)


def both(sr, **kw):
    """(the oracle's parameters, the native frame counts) for the same Slicer constructor arguments."""
    full = dict(SLICER_DEFAULTS, **kw)
    return osl.SlicerParams(sr, **full), psl.slicer_frames(sr, psl.slicer_params(**full))


def oracle_ranges(rms, p, n):
    return osl.chunk_ranges(osl.silence_tags(rms, p), rms.shape[0], p.hop_size, n)


@pytest.mark.parametrize('name', list(CASES))
def test_oracle_matches_reference_golden(name):
    wave = make_case(name)
    p = osl.SlicerParams(44100, **CASES[name]['slicer'])
    got = np.asarray(osl.slice_ranges(wave, p), dtype=np.int64).reshape(-1, 2)
    np.testing.assert_array_equal(got, GOLD[f'{name}__ranges'])
    np.testing.assert_array_equal(got[:, 0] / 44100, GOLD[f'{name}__offsets'])     # chunk['offset'] (slicer2.py:64)
    if f'{name}__rms' in GOLD:
        rms = osl.rms_frames(wave, p.win_size, p.hop_size)
        assert rms.shape[0] == int(GOLD[f'{name}__rms_len'])
        ref = GOLD[f'{name}__rms']
        np.testing.assert_array_equal(rms if ref.shape[0] == rms.shape[0] else rms[::7], ref)   # bit-exact
        assert float(rms.astype(np.float64).sum()) == float(GOLD[f'{name}__rms_sum'])


@pytest.mark.parametrize('name', [n for n in CASES if n not in ('short3',)])
def test_native_ranges_equal_frame_walk_on_golden_cases(name):
    wave = make_case(name)
    kw = CASES[name]['slicer']
    p, s = osl.SlicerParams(44100, **kw), psl.Slicer(44100, **kw)
    rms = osl.rms_frames(wave, p.win_size, p.hop_size)
    [got] = psl.cut_ranges(s, [len(wave)], lambda _: [rms])          # the frame counts come from the Slicer's attributes
    assert got == oracle_ranges(rms, p, len(wave))
    np.testing.assert_array_equal(np.asarray(got, dtype=np.int64).reshape(-1, 2), GOLD[f'{name}__ranges'])


def test_native_ranges_equal_frame_walk_random():
    """Random RMS lists with silent runs of every length class (<= keep, <= 2 keep, > 2 keep, leading, trailing, ties)."""
    rng = np.random.default_rng(4242)
    for trial in range(300):
        kw = dict(threshold=-40., min_length=int(rng.integers(300, 3000)), min_interval=int(rng.integers(40, 300)),
                  hop_size=int(rng.integers(5, 40)), max_sil_kept=int(rng.integers(40, 800)))
        if not kw['min_length'] >= kw['min_interval'] >= kw['hop_size'] or kw['max_sil_kept'] < kw['hop_size']:
            continue
        p, f = both(16000, **kw)
        total = int(rng.integers(50, 1500))
        rms = (0.05 + 0.05 * rng.random(total)).astype(np.float32)
        pos = 0 if rng.random() < 0.3 else int(rng.integers(1, 40))
        while pos < total:
            ln = int(rng.integers(1, 120))
            quiet = (0.009 * rng.random(ln)).astype(np.float32)
            if rng.random() < 0.3:
                quiet[:] = np.float32(0.0)                                  # exact ties: first-index argmin must win
            rms[pos:pos + ln] = quiet[:max(0, min(ln, total - pos))]
            pos += ln + int(rng.integers(1, 200))
        n = (total - 1) * p.hop_size + int(rng.integers(0, p.hop_size))
        assert psl.slicer_ranges(rms, n, f) == oracle_ranges(rms, p, n), (trial, kw)


def test_slicer_parameters_and_errors():
    for kw in (dict(), dict(max_sil_kept=1000), dict(threshold=-30., min_length=2000, min_interval=200, hop_size=10, max_sil_kept=300)):
        p, s = osl.SlicerParams(44100, **kw), psl.Slicer(44100, **kw)
        for k in ('sr', 'threshold', 'hop_size', 'win_size', 'min_length', 'min_interval', 'max_sil_kept'):
            assert getattr(p, k) == getattr(s, k), k
    assert psl.Slicer(44100, max_sil_kept=1000).win_size == 3528 and psl.Slicer(44100).hop_size == 882
    with pytest.raises(ValueError):
        psl.Slicer(44100, min_length=100, min_interval=300)
    with pytest.raises(ValueError):
        psl.Slicer(44100, max_sil_kept=10)


def test_short_waveform_is_one_chunk_without_gpu():
    s = psl.Slicer(44100, max_sil_kept=1000)
    w = make_case('short3')
    chunks = s.slice(w)                  # below min_length: the reference returns the input untouched (slicer2.py:79-80)
    assert len(chunks) == 1 and chunks[0]['offset'] == 0 and chunks[0]['waveform'] is w


# ---------------------------------------------------------------------------------------------- native slicer vs the oracle
@pytest.mark.parametrize('name', list(CASES))
def test_golden_slicer_waveforms(name):
    wave = make_case(name)
    kw = CASES[name]['slicer']
    p, f = both(44100, **kw)
    rms = osl.rms_frames(wave, p.win_size, p.hop_size)
    assert psl.slicer_ranges(rms, len(wave), f) == oracle_ranges(rms, p, len(wave))


def test_random_rms_lists():
    rng = np.random.default_rng(5151)
    checked = 0
    for trial in range(400):
        kw = dict(threshold=-40., min_length=int(rng.integers(300, 3000)), min_interval=int(rng.integers(40, 300)),
                  hop_size=int(rng.integers(5, 40)), max_sil_kept=int(rng.integers(40, 800)))
        if not kw['min_length'] >= kw['min_interval'] >= kw['hop_size'] or kw['max_sil_kept'] < kw['hop_size']:
            continue
        p, f = both(16000, **kw)
        total = int(rng.integers(1, 1500))
        rms = (0.05 + 0.05 * rng.random(total)).astype(np.float32)
        pos = 0 if rng.random() < 0.3 else int(rng.integers(1, 40))
        while pos < total:
            ln = int(rng.integers(1, 160))
            quiet = (0.009 * rng.random(ln)).astype(np.float32)
            if rng.random() < 0.3:
                quiet[:] = np.float32(0.0)                          # ties: the first index of the minimum wins
            rms[pos:pos + ln] = quiet[:max(0, min(ln, total - pos))]
            pos += ln + int(rng.integers(1, 200))
        n = (total - 1) * p.hop_size + int(rng.integers(0, p.hop_size))
        assert psl.slicer_ranges(rms, n, f) == oracle_ranges(rms, p, n), (trial, kw)
        checked += 1
    assert checked > 100


def test_threshold_compares_in_float32():
    p, f = both(44100, max_sil_kept=1000)
    t = np.float32(p.threshold)
    assert np.float32(f.threshold) == t
    below, above = np.nextafter(t, np.float32(0)), np.nextafter(t, np.float32(1))
    for v in (below, t, above):
        rms = np.full(2000, 0.2, dtype=np.float32)
        rms[600:900] = v                                        # a 300-frame run at the threshold
        rms[1500:1560] = v
        n = 1999 * p.hop_size + 5
        got, want = psl.slicer_ranges(rms, n, f), oracle_ranges(rms, p, n)
        assert got == want, v
        assert (len(got) > 1) == bool(v < t)


def test_leading_trailing_and_silent_runs():
    p, f = both(44100, max_sil_kept=1000)
    keep = p.max_sil_kept
    rng = np.random.default_rng(3)

    def run(layout):
        rms = np.concatenate([np.full(ln, 0.001 if quiet else 0.2, dtype=np.float32) * (1 + 0.1 * rng.random(ln)).astype(np.float32)
                              for ln, quiet in layout])
        n = (rms.shape[0] - 1) * p.hop_size + 7
        got, want = psl.slicer_ranges(rms, n, f), oracle_ranges(rms, p, n)
        assert got == want, layout
        return got

    run([(keep + 30, True), (800, False)])                                   # leading silence longer than keep
    run([(20, True), (800, False)])                                          # short leading silence
    run([(800, False), (keep + 100, True)])                                  # trailing silence
    run([(800, False), (10, True)])                                          # short trailing run
    run([(3000, True)])                                                      # all silent
    for span in (keep, keep + 1, 2 * keep, 2 * keep + 1, keep - 1):          # the three branches and their edges
        run([(700, False), (span, True), (700, False), (span, True), (400, False)])
        run([(span, True), (700, False)])
    zeros = np.zeros(3000, dtype=np.float32)                                 # all zero: no chunk at all
    assert psl.slicer_ranges(zeros, 3000 * p.hop_size, f) == oracle_ranges(zeros, p, 3000 * p.hop_size)


def test_slicer_refusals():
    with pytest.raises(_lib.SomeB200Error, match='min_length >= min_interval'):
        psl.slicer_frames(44100, psl.slicer_params(min_length=100, min_interval=300))
    with pytest.raises(_lib.SomeB200Error, match='max_sil_kept >= hop_size'):
        psl.slicer_frames(44100, psl.slicer_params(max_sil_kept=10))
    with pytest.raises(_lib.SomeB200Error, match='do not fit'):
        p, f = both(44100, max_sil_kept=1000)
        rms = np.tile(np.array([0.2] * 400 + [0.0] * 300, dtype=np.float32), 20)
        lib = _lib.load()
        out = np.zeros(2, dtype=np.int64)
        import ctypes as C
        cnt = C.c_int()
        _lib.check(lib.some_slicer_ranges(rms.ctypes.data, rms.shape[0], rms.shape[0] * p.hop_size, C.byref(f), out.ctypes.data,
                                          1, C.byref(cnt)), 'some_slicer_ranges')

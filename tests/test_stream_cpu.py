"""CPU tests of the streaming slicer (some_slicer_stream_*, csrc/slicer.cu): fed the RMS list in any pieces, its ranges,
concatenated, equal some_slicer_ranges on the whole list (itself checked against the oracle in test_slicer_cpu.py),
each range comes back no later than the delivery bound, and the state it keeps stays O(max_sil_kept).  The device half of
streaming is tested in tests/test_gpu_stream.py."""
import ctypes as C
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

DEFAULTS = dict(threshold=-40., min_length=5000, min_interval=300, hop_size=20, max_sil_kept=1000)


def frames_for(sr, **kw):
    return psl.slicer_frames(sr, psl.slicer_params(**dict(DEFAULTS, **kw)))


def reach(f):
    """Samples that complete frame k: k * hop + reach(f)."""
    return f.win_size - f.win_size // 2


def offline(rms, n, f):
    """transcribe_sliced's ranges: the short-recording rule, then some_slicer_ranges."""
    if (n + f.hop_size - 1) // f.hop_size <= f.min_length:
        return [(0, n)]
    return psl.slicer_ranges(rms, n, f)


def streamed(rms, n, f, blocks, log=None):
    """Feeds rms in blocks of the given sizes (the frames the n samples complete; the rest at finish).  log collects
    (frames fed, ranges returned, keep_from()) per call.  Every range a call returns lies where keep_from() said before it."""
    st = psl.SlicerStream(f)

    def kept(out, before):
        keep, head, _ = before
        for a, b in out:
            assert a >= keep or b <= head, (a, b, before)
        return out

    try:
        within = 0 if n < reach(f) else min(rms.shape[0], (n - reach(f)) // f.hop_size + 1)
        got, k, b = [], 0, 0
        while k < within:
            m = min(blocks[b % len(blocks)], within - k)
            b += 1
            fixed = min(n, (k + m - 1) * f.hop_size + reach(f))
            before = st.keep_from()
            out = kept(st.feed(rms[k:k + m], fixed), before)
            k += m
            got += out
            if log is not None:
                log.append((k, out, st.keep_from()))
        before = st.keep_from()
        got += kept(st.finish(rms[k:], n), before)
        return got
    finally:
        st.close()


def check_all_feeds(rms, n, f, rng):
    want = offline(rms, n, f)
    assert streamed(rms, n, f, [1]) == want
    assert streamed(rms, n, f, [1 << 30]) == want
    assert streamed(rms, n, f, list(rng.integers(1, 200, 16))) == want
    return want


def length_for(total, f, rng):
    """A sample count whose RMS list has `total` frames."""
    return (total - 1) * f.hop_size + int(rng.integers(1, f.hop_size))


def test_random_rms_lists():
    rng = np.random.default_rng(6262)
    checked = 0
    for trial in range(250):
        kw = dict(threshold=-40., min_length=int(rng.integers(300, 3000)), min_interval=int(rng.integers(40, 300)),
                  hop_size=int(rng.integers(5, 40)), max_sil_kept=int(rng.integers(40, 800)))
        if not kw['min_length'] >= kw['min_interval'] >= kw['hop_size'] or kw['max_sil_kept'] < kw['hop_size']:
            continue
        f = frames_for(16000, **kw)
        total = int(rng.integers(1, 1500))
        rms = (0.05 + 0.05 * rng.random(total)).astype(np.float32)
        pos = 0 if rng.random() < 0.3 else int(rng.integers(1, 40))
        while pos < total:
            ln = int(rng.integers(1, 160))
            quiet = (0.009 * rng.random(ln)).astype(np.float32)
            if rng.random() < 0.3:
                quiet[:] = np.float32(0.0)
            rms[pos:pos + ln] = quiet[:max(0, min(ln, total - pos))]
            pos += ln + int(rng.integers(1, 200))
        check_all_feeds(rms, length_for(total, f, rng), f, rng)
        checked += 1
    assert checked > 60


@pytest.mark.parametrize('name', list(CASES))
def test_golden_slicer_waveforms(name):
    wave = make_case(name)
    f = frames_for(44100, **dict(DEFAULTS, **CASES[name]['slicer']))
    rms = osl.rms_frames(wave, f.win_size, f.hop_size)
    check_all_feeds(rms, len(wave), f, np.random.default_rng(7))


def layout(spec, rng):
    return np.concatenate([np.full(ln, 0.001 if quiet else 0.2, dtype=np.float32) * (1 + 0.1 * rng.random(ln)).astype(np.float32)
                           for ln, quiet in spec])


@pytest.mark.parametrize('kw', [dict(), dict(max_sil_kept=250, min_interval=300),          # max_sil_kept < min_interval
                                dict(hop_size=20, min_interval=20, min_length=600)],       # win_size / 2 < hop_size
                         ids=['default', 'keep_lt_interval', 'half_window_lt_hop'])
def test_silent_runs(kw):
    rng = np.random.default_rng(11)
    f = frames_for(44100, **kw)
    keep, mi, ml = f.max_sil_kept, f.min_interval, f.min_length
    if kw.get('min_interval') == 20:
        assert f.win_size // 2 < f.hop_size
    specs = [[(keep + 30, True), (ml + 50, False)],                       # leading silence longer than keep
             [(20, True), (ml + 50, False), (10, True)],                  # short leading, short trailing run
             [(ml + 10, False), (keep + 100, True)],                      # trailing silence
             [(ml + 10, False), (max(1, mi - 1), True)],                  # trailing run shorter than min_interval
             [(ml + 10, False), (mi, True)],
             [(3000, True)],                                              # all silent
             [(ml + 5, False), (4000, True), (ml + 5, False), (4000, True)],   # long runs
             [(ml // 3, False), (3 * keep, True), (ml, False), (2 * keep + 1, True), (20, False)]]  # a phrase shorter than min_length
    for span in (keep - 1, keep, keep + 1, 2 * keep, 2 * keep + 1, mi - 1, mi):
        specs.append([(ml + 7, False), (max(1, span), True), (ml + 3, False), (max(1, span), True), (400, False)])
        specs.append([(max(1, span), True), (ml + 3, False)])
    for spec in specs:
        rms = layout(spec, rng)
        rms[rng.random(rms.shape[0]) < 0.02] = np.float32(0.0)       # ties of the minimum
        check_all_feeds(rms, length_for(rms.shape[0], f, rng), f, rng)
    zeros = np.zeros(3000, dtype=np.float32)
    check_all_feeds(zeros, length_for(3000, f, rng), f, rng)
    short = layout([(ml // 3, False), (ml // 3, True), (ml // 4, False)], rng)   # no longer than min_length: one chunk
    n = length_for(short.shape[0], f, rng)
    assert check_all_feeds(short, n, f, rng) == [(0, n)]


@pytest.mark.parametrize('silence_s, then_voice', [(0.5, True), (2.0, True), (3.0, True), (0.5, False), (2.0, False),
                                                  (3.0, False)])
def test_delivery_bound(silence_s, then_voice):
    """A phrase of at least min_length, a silence, then a phrase or the end: the chunk comes back by the feed that makes
    known the voiced frame after the silence or frame max(ss + 2 keep, ss + min_interval - 1, begin + min_length - 1)."""
    rng = np.random.default_rng(int(silence_s * 10) + then_voice)
    f = frames_for(44100)
    assert (f.hop_size, f.max_sil_kept, f.min_interval, f.min_length) == (882, 50, 15, 250)
    ss = 300
    sil = int(round(silence_s * 1000 / 20))
    rms = layout([(ss, False), (sil, True)] + ([(400, False)] if then_voice else []), rng)
    n = length_for(rms.shape[0], f, rng)
    log = []
    got = streamed(rms, n, f, [1], log)
    assert got == offline(rms, n, f)
    first = got[0]
    assert first[0] == 0 and ss - 1 <= first[1] // f.hop_size <= ss + f.max_sil_kept
    bound = max(ss + 2 * f.max_sil_kept, ss + f.min_interval - 1, f.min_length - 1)
    if then_voice:
        bound = min(bound, ss + sil)
    if not then_voice and ss + sil <= bound:                      # the recording ends first: finish delivers the chunk
        assert not any(out for _, out, _ in log) and len(got) == 1
        return
    delivered = next(k for k, out, _ in log if out)
    assert delivered <= bound + 1                                 # frames [0, delivered) known when it came back
    if silence_s == 3.0:
        assert delivered - ss == 2 * f.max_sil_kept + 1           # 100 frames of 20 ms into the silence


def test_memory_stays_bounded_in_long_silence():
    rng = np.random.default_rng(5)
    f = frames_for(44100)
    keep = f.max_sil_kept
    rms = layout([(400, False), (20000, True), (300, False), (9000, True)], rng)
    n = length_for(rms.shape[0], f, rng)
    log = []
    assert streamed(rms, n, f, [1, 7, 33], log) == offline(rms, n, f)
    held = [h for _, _, (_, _, h) in log]
    assert max(held) <= 3 * keep + 70
    for k, _, (keep_from, head, _) in log:
        if 400 + 2 * keep + 5 < k < 20400:                        # well inside the first long silence, after delivery
            assert keep_from >= (k - keep) * f.hop_size and head == 0


@pytest.mark.parametrize('kw', [dict(), dict(max_sil_kept=250, min_interval=300)], ids=['default', 'keep_lt_interval'])
@pytest.mark.parametrize('then', ['voice', 'end'])
def test_memory_stays_bounded_in_leading_silence(kw, then):
    """A stream opened before the singer starts: during the leading silence only the first and the last max_sil_kept frames
    are needed (the all-silent recording's cut lies in the first, a leading cut's right end in the last)."""
    rng = np.random.default_rng(6)
    f = frames_for(44100, **kw)
    keep = f.max_sil_kept
    rms = layout([(20000, True)] + ([(400, False), (20000, True)] if then == 'voice' else []), rng)
    n = length_for(rms.shape[0], f, rng)
    log = []
    got = streamed(rms, n, f, [1, 9, 40], log)
    assert got == offline(rms, n, f)
    if then == 'end':
        assert len(got) == 1 and got[0][0] == 0 and got[0][1] <= keep * f.hop_size     # the all-silent recording's cut
    checked = 0
    for k, _, (keep_from, head, held) in log:
        assert held <= 3 * keep + 70
        if f.min_length + 5 < k < 20000 and k > max(keep, f.min_interval) + 5:
            assert keep_from >= (k - keep) * f.hop_size and head == keep * f.hop_size
            checked += 1
        elif k > 20001:
            assert head == 0
    assert checked > 1000


def test_refusals():
    lib = _lib.load()
    f = frames_for(44100)
    h = C.c_void_p()
    with pytest.raises(_lib.SomeB200Error, match='null pointer'):
        _lib.check(lib.some_slicer_stream_create(None, C.byref(h)), 'some_slicer_stream_create')
    st = psl.SlicerStream(f)
    ptr, cnt = C.c_void_p(), C.c_int()
    with pytest.raises(_lib.SomeB200Error, match='bad arguments'):
        _lib.check(lib.some_slicer_stream_feed(st.handle, None, 5, 10 ** 6, C.byref(ptr), C.byref(cnt)))
    with pytest.raises(_lib.SomeB200Error, match='complete'):
        st.feed(np.full(10, 0.2, np.float32), 5 * f.hop_size)         # frames the fixed samples do not complete
    st.feed(np.full(3, 0.2, np.float32), 3 * f.hop_size + reach(f))
    with pytest.raises(_lib.SomeB200Error, match='went back'):
        st.feed(np.zeros(0, np.float32), 10)
    with pytest.raises(_lib.SomeB200Error, match='frames of'):
        st.finish(np.zeros(0, np.float32), 10 ** 6)                    # not long enough for the short rule, frames missing
    st.close()
    st = psl.SlicerStream(f)
    assert st.finish(np.zeros(0, np.float32), 100) == [(0, 100)]
    with pytest.raises(_lib.SomeB200Error, match='has finished'):
        st.feed(np.zeros(0, np.float32), 100)
    with pytest.raises(_lib.SomeB200Error, match='has finished'):
        st.finish(np.zeros(0, np.float32), 100)
    st.close()
    with pytest.raises(_lib.SomeB200Error, match='min_length >= min_interval'):
        psl.slicer_frames(44100, psl.slicer_params(min_length=100, min_interval=300))
    with pytest.raises(_lib.SomeB200Error, match='max_sil_kept >= hop_size'):
        psl.slicer_frames(44100, psl.slicer_params(max_sil_kept=10))

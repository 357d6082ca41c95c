"""CPU tests of stream peeks (some_stream_peek*, csrc/session.cu): the argument refusals that need no session, and the
properties of the open region [a, b) a peek transcribes, on the streaming slicer alone (a = some_slicer_stream_keep_from's
sample, b = the fixed samples): a never decreases, is never before the end of a delivered chunk, and every later chunk begins
at or after it, except the all-silent recording's one chunk [0, e), e <= max_sil_kept hops, after a long leading silence.
The same properties through the session are tested in tests/test_gpu_stream_peek.py."""
import ctypes as C

import numpy as np
import pytest

from some_b200 import _lib
from some_b200 import slicer as psl

DEFAULTS = dict(threshold=-40., min_length=5000, min_interval=300, hop_size=20, max_sil_kept=1000)


def frames_for(sr, **kw):
    return psl.slicer_frames(sr, psl.slicer_params(**dict(DEFAULTS, **kw)))


def test_refusals_without_a_session():
    lib = _lib.load()
    with pytest.raises(_lib.SomeB200Error, match='some_stream_peek: bad arguments'):
        _lib.check(lib.some_stream_peek(None, None))
    notes = (C.c_void_p * 1)()
    streams = (C.c_void_p * 1)()
    with pytest.raises(_lib.SomeB200Error, match='some_stream_peek_many: bad arguments'):
        _lib.check(lib.some_stream_peek_many(None, 1, notes))
    with pytest.raises(_lib.SomeB200Error, match='some_stream_peek_many: bad arguments'):
        _lib.check(lib.some_stream_peek_many(streams, 1, None))
    with pytest.raises(_lib.SomeB200Error, match='some_stream_peek_many: bad arguments'):
        _lib.check(lib.some_stream_peek_many(streams, -1, notes))
    with pytest.raises(_lib.SomeB200Error, match='stream 0 is NULL'):
        _lib.check(lib.some_stream_peek_many(streams, 1, notes))
    assert lib.some_stream_peek_many(streams, 0, notes) == 0


def events(rms, n, f, blocks):
    """Feeds rms in blocks (the frames the n samples complete; the rest at finish) and records, in order, a peek before
    every feed and before the finish (('peek', a, b, head)) and every range delivered (('chunk', a, b))."""
    st = psl.SlicerStream(f)
    reach = f.win_size - f.win_size // 2
    try:
        within = 0 if n < reach else min(rms.shape[0], (n - reach) // f.hop_size + 1)
        log, k, b, fixed = [], 0, 0, 0
        while k < within:
            a, head, _ = st.keep_from()
            log.append(('peek', a, fixed, head))
            m = min(blocks[b % len(blocks)], within - k)
            b += 1
            fixed = min(n, (k + m - 1) * f.hop_size + reach)
            log += [('chunk', *r) for r in st.feed(rms[k:k + m], fixed)]
            k += m
        a, head, _ = st.keep_from()
        log.append(('peek', a, fixed, head))
        log += [('chunk', *r) for r in st.finish(rms[k:], n)]
        return log
    finally:
        st.close()


def check_region(log, f):
    peeks = [e for e in log if e[0] == 'peek']
    chunks = [e for e in log if e[0] == 'chunk']
    assert all(0 <= a <= b for _, a, b, _ in peeks)
    assert all(p[1] <= q[1] for p, q in zip(peeks, peeks[1:])), 'a went back'
    a_max, end_max, exceptions = 0, 0, 0
    for e in log:
        if e[0] == 'peek':
            assert e[1] >= end_max, ('a before a delivered chunk', e, end_max)
            a_max = max(a_max, e[1])
        else:
            if e[1] < a_max:
                # the all-silent recording after a leading silence longer than max_sil_kept: its one chunk lies in [0, head)
                assert chunks == [e] and e[1] == 0 and e[2] <= f.max_sil_kept * f.hop_size, (e, a_max)
                assert all(h > 0 for _, a, _, h in peeks if a > 0)
                exceptions += 1
            end_max = max(end_max, e[2])
    return exceptions


def test_region_properties_on_random_rms_lists():
    rng = np.random.default_rng(4242)
    f = frames_for(16000, min_length=1000, min_interval=100, hop_size=10, max_sil_kept=300)
    keep, ml = f.max_sil_kept, f.min_length
    checked = 0
    for trial in range(200):
        total = int(rng.integers(1, 1200))
        rms = (0.05 + 0.05 * rng.random(total)).astype(np.float32)
        pos = 0 if rng.random() < 0.3 else int(rng.integers(1, 40))
        while pos < total:
            ln = int(rng.integers(1, 3 * keep))
            rms[pos:pos + ln] = (0.009 * rng.random(min(ln, total - pos))).astype(np.float32)
            pos += ln + int(rng.integers(1, 200))
        n = (total - 1) * f.hop_size + int(rng.integers(1, f.hop_size))
        for blocks in ([1], [7], list(rng.integers(1, 120, 8))):
            check_region(events(rms, n, f, blocks), f)
        checked += 1
    assert checked == 200
    # the cases the properties single out: a leading silence longer than max_sil_kept, then voice or the end; a silence long
    # enough for early delivery; a recording no longer than min_length hops
    quiet, loud = np.float32(0.001), np.float32(0.2)
    lead = np.concatenate([np.full(keep + 40, quiet), np.full(ml + 20, loud)])
    gap = np.concatenate([np.full(ml + 20, loud), np.full(3 * keep, quiet), np.full(ml, loud)])
    silent = np.full(ml + 3 * keep, quiet)
    silent[keep // 2] = np.float32(0.0005)                  # where the trailing rule cuts the all-silent recording
    short = np.concatenate([np.full(ml // 3, loud), np.full(ml // 3, quiet), np.full(ml // 4, loud)])
    for rms, exceptions in ((lead, 0), (gap, 0), (silent, 1), (short, 0)):
        n = (rms.shape[0] - 1) * f.hop_size + 1
        assert check_region(events(rms, n, f, [5]), f) == exceptions

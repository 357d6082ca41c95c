"""CPU tests of a session on several devices (csrc/session.cu): some_session_open_devices refuses bad arguments before it
reads the model file, and a bad model file before any CUDA call, with some_session_open's message; some_shard_clips, the
host-only rule that assigns a call's chunks to the replicas, equals the pure-Python LPT assignment some_b200.dist used, here
restated.  The device path is tested in tests/test_gpu_session_devices.py."""
import ctypes as C
import heapq
import os

import numpy as np
import pytest

from some_b200 import _lib, dist, export
from some_b200 import session as nsess


@pytest.fixture(scope='module')
def model_file(tmp_path_factory):
    """A well-formed model file (lay 0, outdim 128, zero weights) written by the exporter's writer."""
    path = tmp_path_factory.mktemp('model') / 'tiny.somemodel'
    tensors = {name: np.zeros(shape, dtype=dt) for name, dt, shape in export.tensor_specs(0, 128)}
    scalars = dict(lay=0, outdim=128, quantized=False, audio_sample_rate=44100, hop_size=512, win_size=2048, midi_min=0,
                   midi_max=127, midi_prob_deviation=1.0, rest_threshold=0.1, bias_corrected=True)
    export.write_model_file(path, scalars, tensors)
    return path


def open_raw(path, devices, n=None):
    """some_session_open_devices through ctypes (devices None: a NULL list) -> (rc, message); closes what it opened."""
    lib = _lib.load()
    arr = None if devices is None else (C.c_int * max(len(devices), 1))(*devices)
    h = C.c_void_p()
    rc = lib.some_session_open_devices(os.fsencode(os.fspath(path)), arr, len(devices or []) if n is None else n, C.byref(h))
    msg = lib.some_last_error().decode()
    if rc == 0:
        lib.some_session_close(h)
    return rc, msg


def open_error(path, device):
    try:
        s = nsess.Session(path, device)
    except _lib.SomeB200Error as e:
        return str(e)
    s.close()
    return None


def test_argument_refusals_come_before_the_file(tmp_path):
    absent = tmp_path / 'absent.somemodel'           # the file is not read: the arguments are refused first
    for devices, n, expect in [(None, 1, 'the device list is NULL'), ([0], 0, '0 devices (1 to 64)'),
                               ([0] * 65, None, '65 devices (1 to 64)'), ([0, -1], None, 'devices[1] is -1'),
                               ([-3], None, 'devices[0] is -3')]:
        rc, msg = open_raw(absent, devices, n)
        assert rc != 0 and msg == f'some_session_open_devices: {expect}', msg
    rc, msg = open_raw(absent, [0, 0])
    assert rc != 0 and 'cannot open the model file' in msg


def test_bad_file_gives_the_message_of_some_session_open(model_file, tmp_path):
    data = model_file.read_bytes()
    cases = {'magic': b'NOTMODEL' + data[8:], 'size': data + b'\0' * 256, 'cut': data[:-512]}
    for name, blob in cases.items():
        p = tmp_path / f'{name}.somemodel'
        p.write_bytes(blob)
        one = open_error(p, 0)
        assert one is not None and str(p) in one
        # a device that cannot exist: the file is refused before any device is looked at
        for devices in ([0], [0, 0], [999, 0]):
            many = open_error(p, devices)
            assert many.split(': ', 1)[1] == one.split(': ', 1)[1], (one, many)
            assert many.startswith('some_session_open_devices failed')


def test_devices_are_checked_after_the_file(model_file):
    """A valid file: validation passes, then the list is checked entry by entry and a refusal names the index (without a GPU
    the first device is refused; with one, device 999 is)."""
    msg = open_error(model_file, [0, 999])
    assert msg is not None and 'some_session_open_devices: devices[' in msg and 'no CUDA device' in msg, msg
    one = open_error(model_file, 999)
    assert one is not None and 'some_session_open: no CUDA device 999' in one and 'devices[' not in one


def python_lpt(lengths, world):
    """The assignment dist._shard_clips made in pure Python: LPT over clip_cost, clips in order of (-cost, index), each to
    the least loaded rank, ties to the lowest."""
    cost = [t * (103.31e6 + 16384.0 * t) for t in (1 + n // 512 for n in lengths)]
    order = sorted(range(len(lengths)), key=lambda i: (-cost[i], i))
    heap = [(0.0, r) for r in range(world)]
    owner = [0] * len(lengths)
    for i in order:
        load, r = heapq.heappop(heap)
        owner[i] = r
        heapq.heappush(heap, (load + cost[i], r))
    return owner


def shards_of(owner, world):
    return tuple(tuple(i for i, o in enumerate(owner) if o == r) for r in range(world))


def test_shard_clips_equals_python_lpt():
    rng = np.random.default_rng(7)
    for trial in range(200):
        n = int(rng.integers(0, 80))
        world = int(rng.integers(1, 10))
        scale = [2048, 44100 * 20, 44100 * 600][trial % 3]
        lengths = [int(x) for x in rng.integers(0, scale, size=n)]
        want = python_lpt(lengths, world)
        assert nsess.shard_clips(lengths, world) == want, (lengths, world)
        assert dist._shard_clips(tuple(lengths), world) == shards_of(want, world)


@pytest.mark.parametrize('lengths, world', [
    ([], 1), ([], 4),                                        # no clips
    ([1000], 3), ([5 * 44100, 44100], 8),                    # fewer clips than replicas
    ([512 * 10] * 9, 4), ([0, 511, 100, 7] * 3, 2),         # equal costs (the same frame count): index order, lowest replica
    ([44100 * s for s in (3, 30, 7, 12, 0)], 1),             # one replica
    ([2 ** 40, 3, 2 ** 33, 2 ** 40], 3),                     # very long clips
])
def test_shard_clips_edges(lengths, world):
    want = python_lpt(lengths, world)
    got = nsess.shard_clips(lengths, world)
    assert got == want
    assert dist.shard_clips(lengths, world) == [list(s) for s in shards_of(want, world)]
    if len(lengths) >= world:
        assert set(got) == set(range(world))                # every replica gets a clip


def test_shard_clips_refusals():
    lib = _lib.load()
    owner = np.zeros(2, np.int32)
    lens = np.array([10, -1], np.int64)
    assert lib.some_shard_clips(lens.ctypes.data, 2, 2, owner.ctypes.data) != 0
    assert 'clip 1 has a negative length' in lib.some_last_error().decode()
    assert lib.some_shard_clips(lens.ctypes.data, 1, 0, owner.ctypes.data) != 0
    assert 'bad arguments' in lib.some_last_error().decode()
    assert lib.some_shard_clips(None, 0, 1, None) == 0

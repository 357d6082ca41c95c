"""Audio already on the GPU, host side (no GPU needed): the C layout of some_device_audio and some_downmix_item, a numpy
restatement of the two orders K-downmix follows (csrc/downmix.cuh) held bit for bit against np.mean(y, axis=0) on
adversarial float32 values, and the mapping from a tensor's shape and strides to the descriptor, with its refusals."""
import ctypes as C
import os
import pathlib
import shutil
import subprocess

import numpy as np
import pytest
import torch

from some_b200 import _lib, audio

REPO = pathlib.Path(__file__).resolve().parent.parent


# --------------------------------------------------------------------------- C ABI
def test_device_structs_match_the_c_compiler(tmp_path):
    if shutil.which('gcc') is None:
        pytest.skip('gcc not available')
    pairs = [('some_device_audio', _lib.DeviceAudio), ('some_downmix_item', _lib.DownmixItem)]
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "some_b200.h"\nint main(void){\n'
    for name, cls in pairs:
        src += f'  printf("%zu\\n", sizeof({name}));\n'
        for field, _ in cls._fields_:
            src += f'  printf("%zu\\n", offsetof({name}, {field}));\n'
    src += '  printf("%d %d %d\\n", SOME_DOWNMIX_MONO, SOME_DOWNMIX_PLANAR, SOME_DOWNMIX_INTERLEAVED);\n  return 0;\n}\n'
    (tmp_path / 't.c').write_text(src)
    subprocess.check_call(['gcc', '-I', os.path.join(REPO, 'include'), str(tmp_path / 't.c'), '-o', str(tmp_path / 't')])
    out = [int(v) for v in subprocess.check_output([str(tmp_path / 't')], text=True).split()]
    k = 0
    for name, cls in pairs:
        assert out[k] == C.sizeof(cls), name
        k += 1
        for field, _ in cls._fields_:
            assert out[k] == getattr(cls, field).offset, (name, field)
            k += 1
    assert out[k:] == [_lib.DOWNMIX_MONO, _lib.DOWNMIX_PLANAR, _lib.DOWNMIX_INTERLEAVED]


# --------------------------------------------------------------------------- numpy's orders
def planar_mean(y: np.ndarray) -> np.ndarray:
    """mono_mean_planar: the rows added one after another into +0.0, then / channels."""
    s = np.zeros(y.shape[1], np.float32)
    for row in y:
        s = s + row
    return s / np.float32(y.shape[0])


def pairwise_mean(y: np.ndarray) -> np.ndarray:
    """mono_mean: a left-to-right sum below 8 channels; from 8 up, eight running sums combined as a tree, then the rest;
    +0.0 added, then / channels."""
    ch = y.shape[0]
    if ch < 8:
        s = y[0].copy()
        for c in range(1, ch):
            s = s + y[c]
    else:
        r = [y[j].copy() for j in range(8)]
        i = 8
        while i + 8 <= ch:
            for j in range(8):
                r[j] = r[j] + y[i + j]
            i += 8
        s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for c in range(i, ch):
            s = s + y[c]
    return (np.float32(0.0) + s) / np.float32(ch)


def adversarial(rng, ch: int, n: int) -> np.ndarray:
    """float32 [ch, n]: magnitudes from 1e-38 to 1e38 mixed, cancelling pairs, all -0.0 frames and subnormals."""
    y = (rng.standard_normal((ch, n)) * 10.0 ** rng.integers(-38, 38, (ch, n))).astype(np.float32)
    if n < 16:
        y[:, 0] = -0.0
        return y
    y[:, : n // 8] = rng.standard_normal((ch, 1)).astype(np.float32) * np.float32(1e30)       # big values that cancel
    if ch > 1:
        y[-1, : n // 8] = -y[: -1, : n // 8].sum(axis=0, dtype=np.float32)
    y[:, n // 8: n // 8 + 5] = -0.0
    y[:, n // 8 + 5: n // 8 + 9] = np.float32(1e-45) * rng.integers(-3, 4, (ch, 4))
    return y


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


@pytest.mark.parametrize('ch', list(range(1, 10)) + [16, 17, 128])
@pytest.mark.parametrize('n', [2, 3, 1000, 8192 + 77])
def test_numpy_orders_are_restated_bit_for_bit(ch, n):
    rng = np.random.default_rng(1000 * ch + n)
    y = adversarial(rng, ch, n)
    np.testing.assert_array_equal(bits(planar_mean(y)), bits(np.mean(y, axis=0)))               # C-contiguous [C, n]
    wide = np.zeros((ch, n + 13), np.float32)
    wide[:, 5:5 + n] = y
    np.testing.assert_array_equal(bits(planar_mean(y)), bits(np.mean(wide[:, 5:5 + n], axis=0)))   # larger channel stride
    inter = np.ascontiguousarray(y.T).T                                                     # [C, n] view of [n, C]
    np.testing.assert_array_equal(bits(pairwise_mean(y)), bits(np.mean(inter, axis=0)))
    # an all -0.0 frame gives +0.0 in both orders
    z = 0 if n < 16 else n // 8 + 1
    assert not np.signbit(planar_mean(y)[z]) and not np.signbit(pairwise_mean(y)[z])


@pytest.mark.parametrize('ch', [2, 9, 33])
def test_one_frame_takes_the_pairwise_order_whatever_its_stride(ch):
    rng = np.random.default_rng(ch)
    y = adversarial(rng, ch, 64)[:, 3:4]
    wide = np.zeros((ch, 7), np.float32)
    wide[:, 2:3] = y
    for view in (np.ascontiguousarray(y), wide[:, 2:3]):
        np.testing.assert_array_equal(bits(pairwise_mean(y)), bits(np.mean(view, axis=0)))


def test_orders_differ_from_eight_channels():
    rng = np.random.default_rng(7)
    for ch, differ in ((7, False), (8, True), (16, True)):
        y = (rng.standard_normal((ch, 20000)) * 10.0 ** rng.integers(-4, 5, (ch, 20000))).astype(np.float32)
        assert (not np.array_equal(bits(planar_mean(y)), bits(pairwise_mean(y)))) == differ, ch


# --------------------------------------------------------------------------- tensor -> descriptor
def test_layout_from_shape_and_stride():
    lib = _lib.load()
    t = torch.zeros(2, 1000)
    assert audio.device_layout(t, 0, 'w') == (2, 1000, 1000, 1, _lib.DOWNMIX_PLANAR)
    assert audio.device_layout(torch.zeros(1000, 2).t(), 0, 'w') == (2, 1000, 1, 2, _lib.DOWNMIX_INTERLEAVED)
    assert audio.device_layout(torch.zeros(1000), 0, 'w') == (1, 1000, 0, 1, _lib.DOWNMIX_MONO)
    assert audio.device_layout(torch.zeros(1, 1000), 0, 'w') == (1, 1000, 1000, 1, _lib.DOWNMIX_PLANAR)
    assert audio.device_layout(torch.zeros(6, 1200)[:, 100:1100], 0, 'w') == (6, 1000, 1200, 1, _lib.DOWNMIX_PLANAR)
    big = torch.zeros(4, 3000)
    assert audio.device_layout(big[1:3, 7:1007], 0, 'w') == (2, 1000, 3000, 1, _lib.DOWNMIX_PLANAR)
    assert audio.device_layout(torch.zeros(5, 1), 0, 'w')[4] == _lib.DOWNMIX_INTERLEAVED          # one frame: pairwise
    assert audio.device_layout(torch.zeros(5, 9)[:, 4:5], 0, 'w')[4] == _lib.DOWNMIX_INTERLEAVED
    assert audio.device_layout(torch.zeros(0), 0, 'w')[4] == _lib.DOWNMIX_MONO
    assert audio.device_layout(torch.zeros(128, 10), 0, 'w')[:2] == (128, 10)
    layout = C.c_int()
    assert lib.some_downmix_layout(2, 10, 1, 2, C.byref(layout)) == 0 and layout.value == _lib.DOWNMIX_INTERLEAVED


@pytest.mark.parametrize('make, what', [
    (lambda: torch.zeros(2, 100, dtype=torch.float64), 'float32'),
    (lambda: torch.zeros(2, 100, dtype=torch.float16), 'float32'),
    (lambda: torch.zeros(2, 3, 100), 'shape'),
    (lambda: torch.zeros(()), 'shape'),
    (lambda: np.zeros(100, np.float32), 'torch tensor'),
    (lambda: torch.zeros(129, 100), '129 channels'),
    (lambda: torch.zeros(0, 100), '0 channels'),
    (lambda: torch.zeros(200)[::2], 'none of the down-mix layouts'),
    (lambda: torch.zeros(2, 200)[:, ::2], 'none of the down-mix layouts'),
    (lambda: torch.zeros(100, 3).t()[:2], 'none of the down-mix layouts'),      # interleaved with a frame stride > channels
    (lambda: torch.zeros(1, 100).expand(2, 100), 'none of the down-mix layouts'),
    (lambda: torch.zeros(100, 2).as_strided((2, 100), (50, 1)), 'none of the down-mix layouts'),   # overlapping rows
])
def test_wrapper_refusals_name_the_index(make, what):
    with pytest.raises(ValueError, match=f'w: item 3: .*{what}'):
        audio.device_layout(make(), 3, 'w')


def test_device_audio_refuses_cpu_tensors():
    with pytest.raises(ValueError, match='transcribe_device: item 1: a CUDA tensor expected'):
        audio.device_audio(torch.zeros(2, 100), 1, 'transcribe_device', 44100)


def test_pack_refuses_bad_items():
    lib = _lib.load()
    desc = np.zeros(int(lib.some_downmix_bytes(2)), np.uint8)
    good = _lib.DownmixItem(16, 100, 2, _lib.DOWNMIX_PLANAR, 100, 16)
    for bad, msg in ((_lib.DownmixItem(16, 100, 2, _lib.DOWNMIX_PLANAR, 99, 16), 'planar channel stride'),
                     (_lib.DownmixItem(16, 100, 2, _lib.DOWNMIX_MONO, 0, 16), 'mono with 2 channels'),
                     (_lib.DownmixItem(16, 100, 129, _lib.DOWNMIX_PLANAR, 100, 16), '129 channels'),
                     (_lib.DownmixItem(None, 100, 2, _lib.DOWNMIX_PLANAR, 100, 16), 'null pointer'),
                     (_lib.DownmixItem(16, 100, 2, 7, 100, 16), 'unknown layout')):
        arr = (_lib.DownmixItem * 2)(good, bad)
        assert lib.some_downmix_pack(arr, 2, desc.ctypes.data) != 0
        err = lib.some_last_error().decode()
        assert 'item 1' in err and msg in err, err
    arr = (_lib.DownmixItem * 2)(good, _lib.DownmixItem(16, 20000, 2, _lib.DOWNMIX_INTERLEAVED, 1, 16))
    assert lib.some_downmix_pack(arr, 2, desc.ctypes.data) == 0
    tiles = np.frombuffer(desc[:32].tobytes(), np.int64)
    assert tiles[0] == 2 and tiles[1] == 1 + 5        # 100 planar frames: one tile; 20000 stereo frames at 4096 per tile

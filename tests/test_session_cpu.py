"""CPU tests of the native session's host parts: the frame counts some_slicer_derive gives the session's slicer against
some_b200.slicer.Slicer's attributes (the slicer's decisions are tested in test_slicer_cpu.py), and some_session_open's
validation of model files (csrc/session.cu), which runs before any CUDA call.  The device path is tested in
tests/test_gpu_session.py."""
import struct

import numpy as np
import pytest

from some_b200 import _lib, export
from some_b200 import session as nsess
from some_b200 import slicer as psl

SLICER_DEFAULTS = dict(threshold=-40., min_length=5000, min_interval=300, hop_size=20, max_sil_kept=5000)


def both(sr, **kw):
    """(some_b200.slicer.Slicer, the native frame counts) for the same constructor arguments."""
    full = dict(SLICER_DEFAULTS, **kw)
    return psl.Slicer(sr, **full), psl.slicer_frames(sr, psl.slicer_params(**full))


def test_derived_frame_counts_equal_slicer():
    for sr, kw in [(44100, dict()), (44100, dict(max_sil_kept=1000)), (16000, dict(min_interval=30, min_length=250,
                                                                                   max_sil_kept=50, hop_size=20)),
                   (16000, dict(min_interval=50, min_length=330, max_sil_kept=70)), (44100, dict(hop_size=5, min_interval=5)),
                   (22050, dict(threshold=-33.3, min_length=1234.5, min_interval=250.5, hop_size=12.5, max_sil_kept=777)),
                   (48000, dict(threshold=-60.))]:
        s, f = both(sr, **kw)
        assert (f.hop_size, f.win_size, f.min_length, f.min_interval, f.max_sil_kept) == \
            (s.hop_size, s.win_size, s.min_length, s.min_interval, s.max_sil_kept), (sr, kw)
        assert np.float32(f.threshold) == np.float32(s.threshold)


def test_rounding_ties_go_to_even():
    """Parameters whose derived counts are exact .5 ties: Python's round goes to the even neighbour, and so must the C side."""
    cases = [(16000, dict(min_interval=30, min_length=250, max_sil_kept=50)),     # 1.5 -> 2, 12.5 -> 12, 2.5 -> 2
             (16000, dict(min_interval=50, min_length=330, max_sil_kept=70)),     # 2.5 -> 2, 16.5 -> 16, 3.5 -> 4
             (44100, dict(hop_size=5, min_interval=5, min_length=5))]             # hop 220.5 -> 220
    ties = 0
    for sr, kw in cases:
        full = dict(SLICER_DEFAULTS, **kw)
        hop = round(sr * full['hop_size'] / 1000)
        raw = [sr * full['hop_size'] / 1000, sr * full['min_interval'] / 1000 / hop, sr * full['min_length'] / 1000 / hop,
               sr * full['max_sil_kept'] / 1000 / hop]
        ties += sum(1 for x in raw if x % 1 == 0.5)
        s, f = both(sr, **kw)
        assert (f.hop_size, f.min_length, f.min_interval, f.max_sil_kept) == (s.hop_size, s.min_length, s.min_interval,
                                                                              s.max_sil_kept)
    assert ties >= 6


# ---------------------------------------------------------------------------------------------- model file validation
@pytest.fixture(scope='module')
def model_file(tmp_path_factory):
    """A well-formed model file (lay 0, outdim 128, zero weights) written by the exporter's writer, and its directory."""
    path = tmp_path_factory.mktemp('model') / 'tiny.somemodel'
    tensors = {name: np.zeros(shape, dtype=dt) for name, dt, shape in export.tensor_specs(0, 128)}
    scalars = dict(lay=0, outdim=128, quantized=False, audio_sample_rate=44100, hop_size=512, win_size=2048, midi_min=0,
                   midi_max=127,
                   midi_prob_deviation=1.0, rest_threshold=0.1, bias_corrected=True)
    entries = export.write_model_file(path, scalars, tensors)
    return path, path.read_bytes(), {e['name']: e for e in entries}


def open_error(path):
    try:
        s = nsess.Session(path)
    except _lib.SomeB200Error as e:
        return str(e)
    s.close()
    return None


def test_well_formed_file_passes_validation(model_file):
    path, data, _ = model_file
    assert data[:8] == b'SOMEB200' and len(data) % 256 == 0
    msg = open_error(path)
    # without a GPU the first CUDA call fails: validation has passed; with an H100 the file opens
    assert msg is None or 'device' in msg, msg


def _patched(data, offset, fmt, *values):
    b = bytearray(data)
    struct.pack_into(fmt, b, offset, *values)
    return bytes(b)


def test_open_refuses_bad_files(model_file, tmp_path):
    path, data, entries = model_file
    head = entries['w_head']
    cases = {
        'bad magic': _patched(data, 0, '8s', b'NOTMODEL'),
        'unsupported format version 2': _patched(data, 8, '<I', 2),
        'written for ABI 201': _patched(data, 12, '<I', 201),
        'truncated directory': _patched(data, 32, '<I', 1_000_000),
        "tensor 'w_in.0' lies outside the data section": _patched(data, entries['w_in.0']['entry_offset'] + 104, '<Q', len(data)),
        "missing tensor 'w_head'": _patched(data, head['entry_offset'], '64s', b'w_hexd'),
        "tensor 'w_head' is bf16 [64, 1024]": _patched(data, head['entry_offset'] + 72, '<QQ', 64, 1024),
        'does not match the': data + b'\0' * 256,
    }
    msgs = set()
    for i, (expect, blob) in enumerate(cases.items()):
        p = tmp_path / f'bad{i}.somemodel'
        p.write_bytes(blob)
        msg = open_error(p)
        assert msg is not None and expect in msg and str(p) in msg, (expect, msg)
        assert 'device' not in msg.split(str(p))[-1], msg
        msgs.add(msg)
    assert len(msgs) == len(cases)
    tail = tmp_path / 'cut.somemodel'
    tail.write_bytes(data[:-512])                            # a truncated data section is a file-size mismatch
    assert 'does not match the' in open_error(tail)
    assert 'cannot open' in open_error(tmp_path / 'absent.somemodel')


def test_writer_refuses_wrong_tensors(tmp_path):
    tensors = {name: np.zeros(shape, dtype=dt) for name, dt, shape in export.tensor_specs(0, 129)}
    scalars = dict(lay=0, outdim=129, quantized=True, audio_sample_rate=44100, hop_size=512, win_size=2048, midi_min=0,
                   midi_max=127,
                   midi_prob_deviation=1.0, rest_threshold=0.1, bias_corrected=True)
    assert tensors['b_head'].shape == (160,)
    bad = dict(tensors, w_head=np.zeros((128, 512), np.uint16))
    with pytest.raises(ValueError, match='w_head'):
        export.write_model_file(tmp_path / 'x', scalars, bad)
    with pytest.raises(ValueError, match='hop_size'):
        export.write_model_file(tmp_path / 'z', dict(scalars, hop_size=256), tensors)
    del tensors['kaiser_best']
    with pytest.raises(ValueError, match='kaiser_best'):
        export.write_model_file(tmp_path / 'y', scalars, tensors)

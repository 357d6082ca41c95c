"""The fp32 model file (export --precision fp32) without a GPU: the fp32 tensor table of weights.py and its C mirror in
csrc/session.cu agree name by name, dtype and shape (the reader accepts exactly what the writer writes, for every layer count
and head width), a file written from a seeded checkpoint parses, some_session_open refuses malformed fp32 files before any
CUDA call, and a bf16 file keeps the header it had."""
import struct

import numpy as np
import pytest
import torch

from some_b200 import _lib, export, synth, weights
from some_b200 import session as nsess

SCALARS = dict(quantized=False, audio_sample_rate=44100, hop_size=512, win_size=2048, midi_min=0, midi_max=127,
               midi_prob_deviation=1.0, rest_threshold=0.1, bias_corrected=False)
OLD_HEADER = struct.Struct('<8sIIQQIiiiiiiffffiQ40x')      # the header before the precision field


def open_error(path):
    try:
        s = nsess.Session(path)
    except _lib.SomeB200Error as e:
        return str(e)
    s.close()
    return None


def zero_file(path, lay, outdim, precision='fp32'):
    tensors = {n: np.zeros(shape, dtype=dt) for n, dt, shape in export.tensor_specs(lay, outdim, precision)}
    entries = export.write_model_file(path, dict(SCALARS, lay=lay, outdim=outdim, precision=precision), tensors)
    return {e['name']: e for e in entries}


def passed_validation(msg):
    # without a GPU the first CUDA call fails after validation has passed; with an H100 the file opens
    return msg is None or 'device' in msg


def test_f32_table_is_the_bf16_table_in_f32():
    for lay in (0, 1, 3, 8):
        b, f = weights.model_tensors(lay), weights.model_tensors_f32(lay)
        assert [(t.key, t.field, t.index, t.block) for t in b] == [(t.key, t.field, t.index, t.block) for t in f]
        assert all(t.dtype == weights.F32 for t in f)
        assert [t.shape for t in f] == [('outdim',) if t.field == 'b_head' else t.shape for t in b]


@pytest.mark.parametrize('lay,outdim', [(0, 128), (1, 129), (3, 128)])
def test_reader_takes_exactly_the_f32_table(lay, outdim, tmp_path):
    path = tmp_path / 'zero.somemodel'
    entries = zero_file(path, lay, outdim)
    assert passed_validation(open_error(path)), open_error(path)
    with open(path, 'r+b') as f:
        for name, e in entries.items():
            if lay == 3 and name.startswith(('blk', 'glu')) and not name.startswith(('blk7.', 'glu5.')):
                continue                # the other rows are the ones lay 1 checks; each open reads the whole file
            f.seek(e['entry_offset'])
            f.write(('x' + name).encode('ascii'))
            f.flush()
            msg = open_error(path)
            assert msg is not None and f"missing tensor '{name}'" in msg, (name, msg)
            f.seek(e['entry_offset'])
            f.write(name.encode('ascii') + b'\0')
        f.flush()
    assert passed_validation(open_error(path))


def test_seeded_checkpoint_f32_file_parses(tmp_path):
    config = synth.named_config('two_head')
    sd = synth.fabricate_state_dict(config, seed=1234)
    ck = weights.checkpoint_f32(sd, config)
    lay = config['midi_extractor_args']['lay']
    tensors = {}
    for t in weights.model_tensors_f32(lay):
        v = weights.packed_tensor(ck, t)
        tensors[t.key] = np.array([v], '<f4') if isinstance(v, float) else v.detach().to(torch.float32).contiguous().numpy()
    for n, dt, shape in export.FRONT_END:
        tensors[n] = np.zeros(shape, dtype=dt)
    path = tmp_path / 'seeded.somemodel'
    export.write_model_file(path, dict(SCALARS, lay=lay, outdim=128, precision='fp32'), tensors)
    assert passed_validation(open_error(path)), open_error(path)
    data = path.read_bytes()
    assert struct.unpack_from('<i', data, 88)[0] == 1
    e = {x['name']: x for x in export.write_model_file(tmp_path / 'again', dict(SCALARS, lay=lay, outdim=128, precision='fp32'),
                                                         tensors)}
    w = e['blk0.ffn_w1.0']
    np.testing.assert_array_equal(np.frombuffer(data, '<f4', w['nbytes'] // 4, w['offset']),
                                  tensors['blk0.ffn_w1.0'].reshape(-1))


def test_open_refuses_bad_f32_files(tmp_path):
    path = tmp_path / 'ok.somemodel'
    entries = zero_file(path, 1, 128)
    data = path.read_bytes()
    w = entries['blk0.ffn_w1.0']
    b = bytearray(data)
    struct.pack_into('<I', b, w['entry_offset'] + 64, 2)                  # dtype bf16 ...
    struct.pack_into('<Q', b, w['entry_offset'] + 112, w['nbytes'] // 2)  # ... with a bf16 tensor's byte count
    cases = {
        "tensor 'blk0.ffn_w1.0' is bf16 [2048, 512], an fp32 model": bytes(b),
        'does not match the': data[:-512],
        'unknown precision 7': data[:88] + struct.pack('<i', 7) + data[92:],
    }
    for i, (expect, blob) in enumerate(cases.items()):
        p = tmp_path / f'bad{i}.somemodel'
        p.write_bytes(blob)
        msg = open_error(p)
        assert msg is not None and expect in msg and str(p) in msg, (expect, msg)
        assert 'device' not in msg.split(str(p))[-1], msg
    # a bf16 file whose header says fp32: its bf16 tensors are refused by name
    bf = tmp_path / 'bf16.somemodel'
    zero_file(bf, 0, 128, 'bf16')
    raw = bf.read_bytes()
    p = tmp_path / 'mislabelled.somemodel'
    p.write_bytes(raw[:88] + struct.pack('<i', 1) + raw[92:])
    msg = open_error(p)
    assert msg is not None and "tensor 'w_in.0' is bf16" in msg and 'an fp32 model' in msg, msg
    with pytest.raises(ValueError):
        export.write_model_file(tmp_path / 'x', dict(SCALARS, lay=0, outdim=128, precision='fp16'), {})


def test_bf16_file_is_unchanged(tmp_path):
    """A bf16 file has the header of the format before fp32 files: the same fields, the precision bytes zero."""
    path = tmp_path / 'bf16.somemodel'
    entries = zero_file(path, 1, 129, 'bf16')
    data = path.read_bytes()
    n = len(entries)
    data_off = (128 + 128 * n + 255) // 256 * 256
    want = OLD_HEADER.pack(b'SOMEB200', 1, 202, len(data), 128, n, 1, 129, 0, 44100, 512, 2048, 0.0, 127.0, 1.0, 0.1, 0,
                           data_off)
    assert data[:128] == want
    assert [(k, e['offset']) for k, e in entries.items()] == \
           [(k, e['offset']) for k, e in zip([s[0] for s in export.tensor_specs(1, 129)], entries.values())]
    assert export.tensor_specs(1, 129) == export.tensor_specs(1, 129, 'bf16')

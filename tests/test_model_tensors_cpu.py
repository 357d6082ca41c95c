"""The packed model's tensors against tests/golden/model_tensors.json (tests/golden/make_golden_model_tensors.py): the model
file's format (export.tensor_specs), the device pointers of the C mirror (build_c_model) and of the fp32 validation model
(build_f32_model), and the native reader (some_session_open, csrc/session.cu) against the writer."""
import ctypes as C
import json
import pathlib
import sys

import numpy as np
import pytest
import torch

HERE = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / 'golden'))

from make_golden_model_tensors import attribute_paths, struct_fields  # noqa: E402
from some_b200 import _lib, export, synth, weights  # noqa: E402
from some_b200 import session as nsess  # noqa: E402

GOLDEN = json.loads((HERE / 'golden' / 'model_tensors.json').read_text())


@pytest.mark.parametrize('lay', [0, 1, 8])
@pytest.mark.parametrize('outdim', [128, 129])
def test_tensor_specs_match_the_recorded_format(lay, outdim):
    got = [[n, dt.str, list(shape)] for n, dt, shape in export.tensor_specs(lay, outdim)]
    assert got == GOLDEN['tensor_specs'][f'{lay}/{outdim}']


@pytest.mark.parametrize('lay', [0, 1])
def test_c_model_points_at_the_recorded_tensors(lay):
    """Every field build_c_model sets holds the data_ptr of the ModelWeights tensor recorded for it, with either launch
    sequence; nothing else is set."""
    config = synth.named_config('two_head', lay=lay)
    w = weights.ModelWeights(synth.fabricate_state_dict(config, seed=7), config, 'cpu')
    tensors = dict(attribute_paths(w))
    for fold in (False, True):
        m, _keep = weights.build_c_model(w, fold)
        assert (m.lay, m.outdim, m.ln_fold) == (lay, 128, int(fold))
        fields = dict(struct_fields(m, lay))
        want = GOLDEN['c_model'][f'{lay}/{int(fold)}']
        assert list(fields) == list(want)
        for field, path in want.items():
            if field == 'b_cut':
                assert fields[field] == np.float32(w.b_cut)
            else:
                assert fields[field] == tensors[path].data_ptr(), (field, path)
        if lay == 0:
            assert m.glu_w[0] is None and m.glu_b[0] is None


def checkpoint_transforms(sd, lay):
    """field -> what the fp32 validation path runs: the checkpoint's own tensors, to_q | to_kv concatenated, the 1x1
    convolutions squeezed, BatchNorm folded into the depthwise taps in float64 and the taps transposed to [K][C]."""
    out = {}
    for s, n in enumerate(('inln', 'inln1')):
        out[f'w_in[{s}]'], out[f'b_in[{s}]'] = sd[f'model.{n}.weight'], sd[f'model.{n}.bias']
    prefixes = [f'model.cf_lay.{i}.att{s}' for i in range(lay) for s in (1, 2)] + ['model.att1', 'model.att2']
    for j, p in enumerate(prefixes):
        b = f'blocks[{j}].'
        for k in range(5):
            out[f'{b}ln_g[{k}]'], out[f'{b}ln_b[{k}]'] = sd[f'{p}.norm{k + 1}.weight'], sd[f'{p}.norm{k + 1}.bias']
        for k in range(2):
            for n in (1, 2):
                out[f'{b}ffn_w{n}[{k}]'] = sd[f'{p}.ffn{k + 1}.ln{n}.weight']
                out[f'{b}ffn_b{n}[{k}]'] = sd[f'{p}.ffn{k + 1}.ln{n}.bias']
        out[b + 'w_qkv'] = torch.cat([sd[f'{p}.att.to_q.weight'], sd[f'{p}.att.to_kv.weight']])
        out[b + 'w_out'], out[b + 'b_out'] = sd[f'{p}.att.to_out.0.weight'], sd[f'{p}.att.to_out.0.bias']
        for n in (1, 2):
            out[f'{b}w_pw{n}'] = sd[f'{p}.conv.pointwise_conv{n}.weight'][:, :, 0]
            out[f'{b}b_pw{n}'] = sd[f'{p}.conv.pointwise_conv{n}.bias']
        bn = {k: sd[f'{p}.conv.norm.{k}'].double() for k in ('weight', 'bias', 'running_mean', 'running_var')}
        g = bn['weight'] / torch.sqrt(bn['running_var'] + 1e-5)
        out[b + 'w_dw'] = (sd[f'{p}.conv.depthwise_conv.weight'][:, 0, :].double() * g[:, None]).t()
        out[b + 'b_dw'] = (sd[f'{p}.conv.depthwise_conv.bias'].double() - bn['running_mean']) * g + bn['bias']
    for j in range(2 * lay):
        out[f'glu_w[{j}]'] = sd[f'model.cf_lay.{j // 2}.glu{j % 2 + 1}.0.weight']
        out[f'glu_b[{j}]'] = sd[f'model.cf_lay.{j // 2}.glu{j % 2 + 1}.0.bias']
    out['w_head'], out['b_head'] = sd['model.outln.weight'], sd['model.outln.bias']
    out['w_cut'] = sd['model.cutheard.weight'][0]
    return out


def test_f32_model_is_the_checkpoint_transforms():
    """Every field of the fp32 validation model (build_f32_model) points at its checkpoint transform, bit for bit."""
    config = synth.named_config('two_head', lay=1)
    sd = synth.fabricate_state_dict(config, seed=7)
    m, _keep = weights.build_f32_model(sd, config, 'cpu')
    fields = dict(struct_fields(m, 1))
    shapes = GOLDEN['f32_model']['1']
    assert list(fields) == list(shapes) and (m.lay, m.outdim) == (1, 128)
    assert fields.pop('b_cut') == np.float32(sd['model.cutheard.bias'][0])
    want = checkpoint_transforms(sd, 1)
    assert sorted(want) == sorted(fields)
    for field, ptr in fields.items():
        expected = want[field].float().contiguous().numpy()
        assert list(expected.shape) == shapes[field], field
        got = np.ctypeslib.as_array((C.c_float * expected.size).from_address(ptr)).reshape(expected.shape)
        assert np.array_equal(got.view(np.uint32), expected.view(np.uint32)), field


def open_error(path):
    try:
        s = nsess.Session(path)
    except _lib.SomeB200Error as e:
        return str(e)
    s.close()
    return None


@pytest.mark.parametrize('lay', [0, 1, 3])
def test_reader_takes_every_tensor_the_writer_writes(lay, tmp_path):
    """A zero model file written from tensor_specs passes the reader's validation (without a GPU the first CUDA call then
    fails); with any one tensor renamed, the reader names that tensor as missing: every row of its table is a tensor of
    the format."""
    path = tmp_path / 'zero.somemodel'
    tensors = {name: np.zeros(shape, dtype=dt) for name, dt, shape in export.tensor_specs(lay, 129)}
    scalars = dict(lay=lay, outdim=129, quantized=True, audio_sample_rate=44100, hop_size=512, win_size=2048, midi_min=0,
                   midi_max=127, midi_prob_deviation=1.0, rest_threshold=0.1, bias_corrected=True)
    entries = export.write_model_file(path, scalars, tensors)
    msg = open_error(path)
    assert msg is None or 'device' in msg, msg
    last = (f'blk{2 * lay + 1}.', f'glu{2 * lay - 1}.')
    with open(path, 'r+b') as f:
        for e in entries:
            if lay == 3 and e['name'].startswith(('blk', 'glu')) and not e['name'].startswith(last):
                continue                # the rows lay 1 renames already; each open reads the whole 100 MB file
            f.seek(e['entry_offset'])
            f.write(('x' + e['name']).encode('ascii'))
            f.flush()
            msg = open_error(path)
            assert msg is not None and f"missing tensor '{e['name']}'" in msg, (e['name'], msg)
            f.seek(e['entry_offset'])
            f.write(e['name'].encode('ascii') + b'\0')
        f.flush()
    msg = open_error(path)
    assert msg is None or 'device' in msg, msg

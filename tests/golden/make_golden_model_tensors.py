"""Generates tests/golden/model_tensors.json: what the packed model looks like from outside, so that a change to how the
packing code is organised can be checked against it.

* ``tensor_specs``: the model file's tensors (export.tensor_specs: name, dtype, shape, in file order) for lay 0 / 1 / 8 and
  outdim 128 / 129;
* ``c_model``: for lay 0 and 1 and both ln_fold settings, every field build_c_model sets in some_model / some_block_weights
  -> the attribute path (below ModelWeights) of the tensor it points to (``b_cut``: the value);
* ``f32_model``: for lay 1, every field build_f32_model sets in some_model_f32 / some_block_weights_f32 -> the shape of the
  tensor it points to.

    python tests/golden/make_golden_model_tensors.py
"""
import ctypes as C
import json
import pathlib
import re
import sys

HERE = pathlib.Path(__file__).resolve().parent
REPO = HERE.parent.parent
sys.path.insert(0, str(REPO))

import torch  # noqa: E402

from some_b200 import export, synth, weights  # noqa: E402


def attribute_paths(obj, name=''):
    """(path, tensor) of every tensor ModelWeights holds (the rounding registry aside), e.g. blocks[1][0].ffn[1]['w1']."""
    if isinstance(obj, torch.Tensor):
        yield name, obj
    elif isinstance(obj, (list, tuple)):
        for i, v in enumerate(obj):
            yield from attribute_paths(v, f'{name}[{i}]')
    elif isinstance(obj, dict):
        for k, v in obj.items():
            yield from attribute_paths(v, f'{name}[{k!r}]')
    elif hasattr(obj, '__dict__') and not isinstance(obj, weights.RoundingRegistry):
        for k, v in vars(obj).items():
            yield from attribute_paths(v, f'{name}.{k}' if name else k)


def struct_fields(s, lay, prefix=''):
    """(field path, value) of every pointer field of a model struct, and of b_cut; blocks and GLU arrays followed."""
    for name, ctype in s._fields_:
        v = getattr(s, name)
        if name == 'b_cut':
            yield prefix + name, float(v)
        elif ctype is C.c_void_p:
            yield prefix + name, v
        elif issubclass(ctype, C.Array):
            yield from ((f'{prefix}{name}[{i}]', x) for i, x in enumerate(v))
        elif name == 'blocks':
            for j in range(2 * (lay + 1)):
                yield from struct_fields(v[j], lay, f'{prefix}{name}[{j}].')
        elif name in ('glu_w', 'glu_b'):
            yield from ((f'{prefix}{name}[{j}]', v[j]) for j in range(2 * lay))


def main():
    out = {'tensor_specs': {}, 'c_model': {}, 'f32_model': {}}
    for lay in (0, 1, 8):
        for outdim in (128, 129):
            out['tensor_specs'][f'{lay}/{outdim}'] = [[n, dt.str, list(shape)]
                                                      for n, dt, shape in export.tensor_specs(lay, outdim)]
    for lay in (0, 1):
        config = synth.named_config('two_head', lay=lay)
        w = weights.ModelWeights(synth.fabricate_state_dict(config, seed=5), config, 'cpu')
        by_ptr = {}
        for path, t in attribute_paths(w):
            assert t.data_ptr() not in by_ptr, (path, by_ptr[t.data_ptr()])
            by_ptr[t.data_ptr()] = path
        for fold in (False, True):
            m, _keep = weights.build_c_model(w, fold)
            out['c_model'][f'{lay}/{int(fold)}'] = {f: 'b_cut' if f == 'b_cut' else by_ptr[v]
                                                    for f, v in struct_fields(m, lay)}
    config = synth.named_config('two_head', lay=1)
    m, (keep, *_) = weights.build_f32_model(synth.fabricate_state_dict(config, seed=5), config, 'cpu')
    shapes = {t.data_ptr(): list(t.shape) for t in keep}
    out['f32_model']['1'] = {f: None if f == 'b_cut' else shapes[v] for f, v in struct_fields(m, 1)}
    text = json.dumps(out, indent=1)
    for _ in range(2):      # innermost lists on one line: a shape, then a whole tensor_specs row
        text = re.sub(r'\[\s+((?:[^\[\]{}]|\[[^\[\]{}\n]*\])*?)\s+\]', lambda m: '[' + ' '.join(m.group(1).split()) + ']',
                      text)
    (HERE / 'model_tensors.json').write_text(text + '\n')


if __name__ == '__main__':
    main()

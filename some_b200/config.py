"""Configuration and checkpoint-schema helpers for the SOME inference hot path.

* ``flatten_config`` restates the ``base_config`` inheritance of
  the reference's utils/config_utils.py:11-41 (read_full_config / override_dict) so the
  stock ``configs/*.yaml`` chain can be flattened into the ``config.yaml`` the reference
  writes beside a checkpoint (train.py:42-43) and that infer.py:21 reads back.
* ``model_param_shapes`` is the strict ``state_dict`` schema of
  ``modules.model.Gmidi_conform.midi_conforms`` (Gmidi_conform.py:22-28,
  Gconform.py:92-116): the plugin validates checkpoints against it the way
  ``load_state_dict(strict=True)`` does in base_infer.py:27-33.
"""
from __future__ import annotations

import pathlib
from collections import OrderedDict
from typing import Dict, Tuple

import yaml

# The model geometry the sm_90a kernels are specialised for (every shipped config uses it:
# configs/{two_head_model,quant_two_head_model,midi_conformer,continuous,discrete}.yaml).
DIM = 512
HEADS = 8
HEAD_DIM = 64
KERNEL_SIZE = 31
UNITS_DIM = 80
FFN_DIM = 4 * DIM
MAX_OUTDIM = 256


def override_dict(old: dict, new: dict) -> None:
    for k, v in new.items():
        if isinstance(v, dict) and k in old:
            override_dict(old[k], new[k])
        else:
            old[k] = v


def flatten_config(config_path, root=None) -> dict:
    """Resolve ``base_config`` chains.  ``root`` = directory that relative ``base_config``
    entries (e.g. ``configs/base.yaml``) are resolved against (the reference resolves them
    against the process CWD, i.e. its repository root)."""
    config_path = pathlib.Path(config_path)
    root = pathlib.Path(root) if root is not None else config_path.resolve().parent.parent
    with open(config_path, 'r', encoding='utf8') as f:
        config = yaml.safe_load(f)
    if 'base_config' not in config:
        return config
    bases = config['base_config']
    if not isinstance(bases, list):
        bases = [bases]
    squashed: dict = {}
    for base in bases:
        base_path = pathlib.Path(base)
        if not base_path.is_absolute():
            base_path = root / base_path
        override_dict(squashed, flatten_config(base_path, root))
    override_dict(squashed, config)
    squashed.pop('base_config')
    return squashed


def check_supported(config: dict) -> dict:
    """Validates the geometry and returns the extractor args."""
    args = dict(config['midi_extractor_args'])
    problems = []
    if args.get('dim') != DIM:
        problems.append(f"dim={args.get('dim')} (kernels are built for {DIM})")
    if args.get('attention_heads', 4) != HEADS or args.get('attention_heads_dim', 64) != HEAD_DIM:
        problems.append(f"attention {args.get('attention_heads')}x{args.get('attention_heads_dim')} "
                        f"(kernels are built for {HEADS}x{HEAD_DIM})")
    if args.get('kernel_size', 31) != KERNEL_SIZE:
        problems.append(f"kernel_size={args.get('kernel_size')} (kernels are built for {KERNEL_SIZE})")
    if config['units_dim'] != UNITS_DIM:
        problems.append(f"units_dim={config['units_dim']} (mel front end emits {UNITS_DIM})")
    if not (1 <= config['midi_num_bins'] <= MAX_OUTDIM):
        problems.append(f"midi_num_bins={config['midi_num_bins']} (max {MAX_OUTDIM})")
    if config.get('win_size', 2048) != 2048 or config.get('hop_size', 512) != 512:
        problems.append('win_size/hop_size must be 2048/512 (fused STFT kernel)')
    if problems:
        raise NotImplementedError('some_b200: unsupported model geometry: ' + '; '.join(problems))
    return args


def _block_shapes(prefix: str, dim: int, k: int) -> 'OrderedDict[str, Tuple[int, ...]]':
    s: 'OrderedDict[str, Tuple[int, ...]]' = OrderedDict()
    for ffn in ('ffn1', 'ffn2'):
        s[f'{prefix}.{ffn}.ln1.weight'] = (4 * dim, dim)
        s[f'{prefix}.{ffn}.ln1.bias'] = (4 * dim,)
        s[f'{prefix}.{ffn}.ln2.weight'] = (dim, 4 * dim)
        s[f'{prefix}.{ffn}.ln2.bias'] = (dim,)
    s[f'{prefix}.att.to_q.weight'] = (HEADS * HEAD_DIM, dim)
    s[f'{prefix}.att.to_kv.weight'] = (2 * HEADS * HEAD_DIM, dim)
    s[f'{prefix}.att.to_out.0.weight'] = (dim, HEADS * HEAD_DIM)
    s[f'{prefix}.att.to_out.0.bias'] = (dim,)
    s[f'{prefix}.conv.pointwise_conv1.weight'] = (2 * dim, dim, 1)
    s[f'{prefix}.conv.pointwise_conv1.bias'] = (2 * dim,)
    s[f'{prefix}.conv.depthwise_conv.weight'] = (dim, 1, k)
    s[f'{prefix}.conv.depthwise_conv.bias'] = (dim,)
    s[f'{prefix}.conv.norm.weight'] = (dim,)
    s[f'{prefix}.conv.norm.bias'] = (dim,)
    s[f'{prefix}.conv.norm.running_mean'] = (dim,)
    s[f'{prefix}.conv.norm.running_var'] = (dim,)
    s[f'{prefix}.conv.norm.num_batches_tracked'] = ()
    s[f'{prefix}.conv.pointwise_conv2.weight'] = (dim, dim, 1)
    s[f'{prefix}.conv.pointwise_conv2.bias'] = (dim,)
    for i in range(1, 6):
        s[f'{prefix}.norm{i}.weight'] = (dim,)
        s[f'{prefix}.norm{i}.bias'] = (dim,)
    return s


def model_param_shapes(config: dict) -> 'OrderedDict[str, Tuple[int, ...]]':
    """Ordered ``state_dict`` schema (names without the checkpoint's ``model.`` prefix)."""
    args = config['midi_extractor_args']
    dim, lay, k = args['dim'], args['lay'], args.get('kernel_size', 31)
    indim, outdim = config['units_dim'], config['midi_num_bins']
    s: 'OrderedDict[str, Tuple[int, ...]]' = OrderedDict()
    s['model.inln.weight'] = (dim, indim)
    s['model.inln.bias'] = (dim,)
    s['model.inln1.weight'] = (dim, indim)
    s['model.inln1.bias'] = (dim,)
    s['model.outln.weight'] = (outdim, dim)
    s['model.outln.bias'] = (outdim,)
    s['model.cutheard.weight'] = (1, dim)
    s['model.cutheard.bias'] = (1,)
    for i in range(lay):
        s.update(_block_shapes(f'model.cf_lay.{i}.att1', dim, k))
        s.update(_block_shapes(f'model.cf_lay.{i}.att2', dim, k))
        for g in ('glu1', 'glu2'):
            s[f'model.cf_lay.{i}.{g}.0.weight'] = (2 * dim, dim)
            s[f'model.cf_lay.{i}.{g}.0.bias'] = (2 * dim,)
    s.update(_block_shapes('model.att1', dim, k))
    s.update(_block_shapes('model.att2', dim, k))
    return s


def load_state_dict_strict(model_path, config: dict, map_location='cpu') -> Dict[str, 'object']:
    """``torch.load(path)['state_dict']``, keep ``model.``-prefixed keys, strip the prefix,
    and enforce exactly the reference schema (base_infer.py:27-33, strict=True)."""
    import torch

    ckpt = torch.load(model_path, map_location=map_location, weights_only=False)
    raw = ckpt['state_dict']
    prefix = 'model.'
    sd = OrderedDict((k[len(prefix):], v) for k, v in raw.items() if k.startswith(prefix))
    schema = model_param_shapes(config)
    missing = [k for k in schema if k not in sd]
    unexpected = [k for k in sd if k not in schema]
    mismatched = [f'{k}: checkpoint {tuple(sd[k].shape)} vs model {schema[k]}'
                  for k in schema if k in sd and tuple(sd[k].shape) != tuple(schema[k])]
    if missing or unexpected or mismatched:
        msg = ['Error(s) in loading state_dict for midi_conforms:']
        if missing:
            msg.append('Missing key(s) in state_dict: ' + ', '.join(f'"{k}"' for k in missing) + '.')
        if unexpected:
            msg.append('Unexpected key(s) in state_dict: ' + ', '.join(f'"{k}"' for k in unexpected) + '.')
        if mismatched:
            msg.append('size mismatch for ' + '; '.join(mismatched))
        raise RuntimeError('\n\t'.join(msg))
    return sd

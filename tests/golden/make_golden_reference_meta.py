"""Generates tests/golden/reference_configs.json (the reference's named configs, flattened through their base_config
chains) and tests/golden/reference_state_dict_shapes.json (parameter names and shapes of the reference's
midi_conforms for the two_head config) from the UNMODIFIED reference (SOME_REFERENCE_ROOT).

    python tests/golden/make_golden_reference_meta.py
"""
import json
import pathlib
import sys

HERE = pathlib.Path(__file__).resolve().parent
REPO = HERE.parent.parent
sys.path.insert(0, str(REPO))

from oracle import refshim  # noqa: E402
from some_b200 import config as sconfig  # noqa: E402
from some_b200 import synth  # noqa: E402


def main():
    root = refshim.REFERENCE_ROOT
    configs = {name: sconfig.flatten_config(f'{root}/configs/{name}.yaml', root=root)
               for name in ('two_head_model', 'midi_conformer', 'quant_two_head_model')}
    (HERE / 'reference_configs.json').write_text(json.dumps(configs, sort_keys=True, indent=1) + '\n')
    sys.path.insert(0, root)
    from modules.model.Gmidi_conform import midi_conforms
    cfg = synth.named_config('two_head')
    ref = midi_conforms({'midi_extractor_args': dict(cfg['midi_extractor_args']), 'units_dim': 80,
                         'midi_num_bins': 128}).state_dict()
    shapes = {k: list(v.shape) for k, v in ref.items()}
    (HERE / 'reference_state_dict_shapes.json').write_text(json.dumps(shapes, indent=0) + '\n')


if __name__ == '__main__':
    main()

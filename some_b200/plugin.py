"""H100-native drop-in for the reference's ``inference`` plugin package
(the reference's inference/{base_infer,me_infer,me_quant_infer}.py, registry __init__.py:5-8).

Same class names, constructor signature, attributes and method contracts, so that infer.py:24-37,
batch_infer.py:26-34,54 and webui.py:28-54 run unchanged when this repo precedes the reference on
``sys.path`` (the top-level ``inference`` package of this repo re-exports these classes).

All compute goes through libsome_b200.so (hand-written sm_90a kernels).  ``infer()`` runs the whole
list of clips as ONE var-len batch (mel -> trunk -> decode) instead of the reference's serial
batch-1 loop; the per-clip methods ``preprocess / forward_model / postprocess`` keep the reference's
tensor contracts and also run on the GPU kernels.  There is no CPU fallback.
"""
from __future__ import annotations

import pathlib
import threading
from typing import Dict, List

import numpy as np
import torch

from . import _lib
from .config import load_state_dict_strict
from .engine import Engine, frames_of


class BaseInference:
    """inference/base_infer.py:13-53."""

    def __init__(self, config: dict, model_path: pathlib.Path, device=None):
        if device is None:
            device = 'cuda' if torch.cuda.is_available() else 'cpu'      # base_infer.py:15-16
        self.config = config
        self.model_path = model_path
        self.device = device
        if torch.device(device).type != 'cuda':
            raise _lib.SomeB200Error(
                f"some_b200 plugin needs a CUDA (sm_90a) device, got device='{device}'. "
                "It has no CPU path; use the reference implementation on CPU.")
        self.timestep = self.config['hop_size'] / self.config['audio_sample_rate']   # base_infer.py:20
        self._lock = threading.Lock()     # webui.py:104 runs up to 10 concurrent callers on one instance
        self.model: Engine = self.build_model()

    def build_model(self) -> Engine:
        """base_infer.py:23-35: load ``state_dict`` (keys prefixed ``model.``), strict."""
        state_dict = load_state_dict_strict(self.model_path, self.config, map_location='cpu')
        engine = Engine(self.config, state_dict, self.device)
        print(f'| load \'model\' from \'{self.model_path}\'.')
        return engine

    def preprocess(self, waveform: np.ndarray) -> Dict[str, torch.Tensor]:
        raise NotImplementedError()

    def forward_model(self, sample: Dict[str, torch.Tensor]):
        raise NotImplementedError()

    def postprocess(self, results: Dict[str, torch.Tensor]) -> List[Dict[str, np.ndarray]]:
        raise NotImplementedError()

    def infer(self, waveforms: List[np.ndarray]) -> List[Dict[str, np.ndarray]]:
        raise NotImplementedError()


class MIDIExtractionInference(BaseInference):
    """inference/me_infer.py:15-97."""
    quantized = False
    head = 'sigmoid'

    def __init__(self, config: dict, model_path: pathlib.Path, device=None):
        super().__init__(config, model_path, device=device)
        self.midi_min = self.config['midi_min']
        self.midi_max = self.config['midi_max']
        # the stock quantized config chain lacks these two keys (SURVEY.md discrepancy 6); the
        # quantized decode does not use them, so read them leniently
        self.midi_deviation = self.config.get('midi_prob_deviation', 1.0)
        self.rest_threshold = self.config.get('rest_threshold', 0.1)

    # ---- per-clip API (reference tensor contracts) -------------------------------------------
    def _tables(self, n: int):
        dev = self.model.device
        t = frames_of(n)
        start = torch.zeros(1, dtype=torch.int64, device=dev)
        length = torch.full((1,), n, dtype=torch.int64, device=dev)
        cu = torch.tensor([0, t], dtype=torch.int32, device=dev)
        return start, length, cu, t

    def preprocess(self, waveform: np.ndarray) -> Dict[str, torch.Tensor]:
        """me_infer.py:29-63: units [1, T, 80] (log-mel, K-mel kernel), pitch zeros [1, T], masks ones."""
        eng = self.model
        with self._lock, torch.cuda.device(eng.device):
            wav = torch.from_numpy(np.ascontiguousarray(waveform, dtype=np.float32)).to(eng.device)
            if wav.numel() == 0:
                wav = torch.zeros(4, dtype=torch.float32, device=eng.device)
            start, length, cu, t = self._tables(int(waveform.shape[0]))
            mel = torch.empty((t, 80), dtype=torch.float32, device=eng.device)
            eng.run_mel(wav, start, length, cu, 1, t, mel, None)
        units = mel.unsqueeze(0)
        pitch = torch.zeros(units.shape[:2], dtype=torch.float32, device=eng.device)
        return {'units': units, 'pitch': pitch, 'masks': torch.ones_like(pitch, dtype=torch.bool)}

    @torch.no_grad()
    def forward_model(self, sample: Dict[str, torch.Tensor]):
        """me_infer.py:65-76: probs [1, T, N] (sigmoid / softmax applied), bounds [1, T]."""
        eng = self.model
        units = sample['units']
        assert units.dim() == 3 and units.shape[0] == 1, 'per-clip API: units [1, T, 80]; use infer() for batches'
        t = units.shape[1]
        with self._lock, torch.cuda.device(eng.device):
            ws = eng.workspace(t)
            ws.units[:t].copy_(units[0])
            cu = torch.tensor([0, t], dtype=torch.int32, device=eng.device)
            eng.run_trunk(ws, t, 1, cu, t, self.head)
            probs = ws.probs[:t].clone().unsqueeze(0)
            bounds = ws.bounds[:t].clone().unsqueeze(0)
        return {'probs': probs, 'bounds': bounds, 'masks': sample['masks']}

    def postprocess(self, results: Dict[str, torch.Tensor]) -> Dict[str, np.ndarray]:
        """me_infer.py:78-97 / me_quant_infer.py:21-38 for one clip (K-decode kernel)."""
        eng = self.model
        probs, bounds, masks = results['probs'], results['bounds'], results['masks']
        probs *= masks[..., None]                                                   # me_infer.py:82-83 (in place)
        bounds *= masks
        t = probs.shape[1]
        with self._lock, torch.cuda.device(eng.device):
            ws = eng.workspace(t)
            cu = torch.tensor([0, t], dtype=torch.int32, device=eng.device)
            nc = torch.empty(1, dtype=torch.int32, device=eng.device)
            eng.run_decode(ws, t, 1, cu, nc, self.quantized, probs=probs[0].contiguous(), bounds=bounds[0].contiguous())
            n = int(nc.item())
            return {
                'note_midi': ws.note_midi[:n].cpu().numpy(),
                'note_dur': ws.note_dur[:n].cpu().numpy().astype(np.int64) * self.timestep,
                'note_rest': ws.note_rest[:n].cpu().numpy().astype(bool),
            }

    # ---- batched fast path ---------------------------------------------------------------------
    def infer(self, waveforms: List[np.ndarray]) -> List[Dict[str, np.ndarray]]:
        """base_infer.py:46-53, batched: same order as the input, one dict per waveform."""
        with self._lock:
            return self.model.infer(list(waveforms), quantized=self.quantized)


class QuantizedMIDIExtractionInference(MIDIExtractionInference):
    """inference/me_quant_infer.py:10-38: softmax head, argmax decode, rest = bin 128."""
    quantized = True
    head = 'softmax'


task_inference_mapping = {                                                           # inference/__init__.py:5-8
    'training.MIDIExtractionTask': 'inference.MIDIExtractionInference',
    'training.QuantizedMIDIExtractionTask': 'inference.QuantizedMIDIExtractionInference',
}

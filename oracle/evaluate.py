"""CPU restatement of the validation losses and MIDI accuracy of the training tasks, for one item (batch of one, as the
validation loader serves them):

- targets of the collaters: MIDIExtractionDataset.collater (training/me_task.py:26-49, gaussian-blurred bins zeroed on
  rests, gathered by unit2note) and QuantizedMIDIExtractionDataset.collater (training/me_quant_task.py:14-26, midi_idx);
  bounds = diff(unit2note, prepend 0) > 0;
- losses with torch.nn.functional on the CPU: BCEWithLogitsLoss / CrossEntropyLoss(ignore_index=-1), and BinaryEMDLoss
  (modules/losses/bound_loss.py:6-19);
- MIDIAccuracy(tolerance=0.5).update (modules/metrics/midi_acc.py:16-35) on the validation step's decode
  (me_task.py:115-154 / me_quant_task.py:78-120).  torchmetrics and lightning are not installed here, so the metric's two
  counters are restated rather than imported; the gaussian-blurred decode is oracle/decode.py's restatement.

The label arrays (``unit2note``, ``note_midi``, ``note_rest``) are the caller's: tests take them from
tests/golden/eval_*.npz, which the unmodified reference produced (tests/golden/make_golden_eval.py).

TEST INFRASTRUCTURE — see oracle/__init__.py.
"""
import math

import torch
import torch.nn.functional as F

from . import decode as odecode


def targets(labels: dict, config: dict, quantized: bool) -> dict:
    """Collater targets of one item: 'probs' [T, N] (continuous) or 'midi_idx' [T] (quantized), and 'bounds' [T]."""
    u = torch.as_tensor(labels['unit2note']).long()
    out = {'bounds': (torch.diff(u, prepend=u.new_zeros(1)) > 0).float()}
    if quantized:
        out['midi_idx'] = F.pad(torch.as_tensor(labels['note_midi']).long(), [1, 0], value=-1)[u]
        return out
    n_bins = config['midi_num_bins']
    interval = (config['midi_max'] - config['midi_min']) / (n_bins - 1)
    sigma = config['midi_prob_deviation'] / interval
    miu = ((torch.as_tensor(labels['note_midi']).float() - config['midi_min']) / interval)[:, None]
    x = torch.arange(n_bins).float()[None, :]
    probs = ((x - miu) / sigma).pow(2).div(-2).exp()
    probs *= ~torch.as_tensor(labels['note_rest']).bool()[:, None]
    out['probs'] = F.pad(probs, [0, 0, 1, 0])[u]
    return out


def losses(logits, bounds, labels: dict, config: dict, quantized: bool) -> dict:
    """{'midi_loss', 'bound_loss'} of one item from the raw head ``logits`` [T, N] and the sigmoid ``bounds`` [T]."""
    logits, bounds = torch.as_tensor(logits).float(), torch.as_tensor(bounds).float()
    tg = targets(labels, config, quantized)
    if quantized:
        midi = F.cross_entropy(logits[None].transpose(1, 2), tg['midi_idx'][None], ignore_index=-1)
    else:
        midi = F.binary_cross_entropy_with_logits(logits, tg['probs'])
    scale = math.sqrt(bounds.shape[0])
    bound = F.l1_loss(bounds.cumsum(dim=0) / scale, tg['bounds'].cumsum(dim=0) / scale)
    return {'midi_loss': float(midi), 'bound_loss': float(bound)}


def accuracy_counts(logits, labels: dict, config: dict, quantized: bool, probs=None):
    """(correct, total) that MIDIAccuracy(tolerance=0.5).update adds for one item.  ``probs``: the activated head to
    decode instead of the sigmoid / softmax of ``logits`` (a kernel's own activations, which may differ from torch's in
    the last ulp)."""
    logits = torch.as_tensor(logits).float()
    u = torch.as_tensor(labels['unit2note']).long()
    if probs is not None:
        probs = torch.as_tensor(probs).float()
    if quantized:
        probs = torch.softmax(logits, dim=-1) if probs is None else probs
        midi_pred = probs.argmax(dim=-1)
        rest_pred = midi_pred == 128
        midi_pred = midi_pred.float()
        note_midi_gt = torch.as_tensor(labels['note_midi']).float()
        note_midi_gt[torch.as_tensor(labels['note_midi']) == 128] = -torch.inf
    else:
        probs = torch.sigmoid(logits) if probs is None else probs
        values, rest = odecode.decode_gaussian_blurred_probs_vec(
            probs.numpy(), config['midi_min'], config['midi_max'], config['midi_prob_deviation'], config['rest_threshold'])
        midi_pred, rest_pred = torch.from_numpy(values), torch.from_numpy(rest)
        note_midi_gt = torch.as_tensor(labels['note_midi']).float().clone()
        note_midi_gt[torch.as_tensor(labels['note_rest']).bool()] = -torch.inf
    midi_pred = midi_pred.clone()
    midi_pred[rest_pred] = -torch.inf
    midi_gt = F.pad(note_midi_gt, [1, 0], value=-torch.inf)[u]
    rest_gt = midi_gt < 0
    mask = u > 0
    close = ~rest_pred & ~rest_gt & (torch.abs(midi_pred - midi_gt) <= 0.5)
    overall = close & (rest_pred == rest_gt) & mask
    return int(overall.sum()), int(mask.sum())

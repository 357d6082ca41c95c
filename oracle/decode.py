"""CPU restatement of the note decoding (utils/infer_utils.py:9-76) and of the plugin's
pre/post-processing (inference/me_infer.py:29-97, inference/me_quant_infer.py:11-38,
inference/base_infer.py:46-53).

Written with explicit numpy loops per clip (not the reference's batched scatter_add form) so it is
an independent restatement; arithmetic order follows what the torch CPU kernels do:
  * ``cumsum`` on float32 accumulates in float64 and rounds each prefix to float32
    (ATen cpu_cum_base_kernel uses acc_type<float, /*is_cuda=*/false> = double);
  * ``round`` is half-to-even;
  * ``scatter_add`` on CPU adds in frame order in the tensor's own dtype (float32 / int64).

TEST INFRASTRUCTURE — see oracle/__init__.py.
"""
import numpy as np
import torch

from . import model as omodel


def decode_bounds_to_alignment(bounds: np.ndarray) -> np.ndarray:
    """infer_utils.py:27-39 (use_diff=True).  bounds float32 [T] -> int64 [T], 1-based, non-decreasing."""
    bounds = np.asarray(bounds, dtype=np.float32)
    csum = np.cumsum(bounds.astype(np.float64)).astype(np.float32)     # :28 cumsum (double accumulator)
    step = np.rint(csum).astype(np.int64)                              # :28 round().long()
    prev = np.concatenate([np.array([-1], dtype=np.int64), step[:-1]])  # :30-35 diff(prepend=-1) > 0
    inc = (step - prev) > 0
    return np.cumsum(inc.astype(np.int64))                             # :38


def bin_values(n: int, interval: float, vmin) -> np.ndarray:
    """infer_utils.py:13-14, ``idx * interval + vmin`` with ``idx`` an int64 tensor: torch computes it in float32, the
    python scalars rounded to float32 and the product rounded before the sum.  (In float64 with one final rounding, 58 of
    the 200 bins of N = 200 over [21, 108] would differ.)"""
    return np.arange(n).astype(np.float32) * np.float32(interval) + np.float32(vmin)


def decode_gaussian_blurred_probs(probs: np.ndarray, vmin, vmax, deviation, threshold):
    """infer_utils.py:9-24.  probs float32 [T, N] -> (values float32 [T], rest bool [T])."""
    probs = np.asarray(probs, dtype=np.float32)
    t, n = probs.shape
    interval = (vmax - vmin) / (n - 1)                                 # :11
    width = int(3 * deviation / interval)                              # :12
    idx_values = bin_values(n, interval, vmin)                         # :13-14
    values = np.zeros(t, dtype=np.float32)
    rest = np.zeros(t, dtype=bool)
    for i in range(t):
        c = int(np.argmax(probs[i]))                                   # :15 (first maximal index)
        lo, hi = max(c - width, 0), min(c + width + 1, n)              # :16-17
        w = probs[i, lo:hi]                                            # :18-19
        product_sum = np.float32(0)
        weight_sum = np.float32(0)
        for j in range(hi - lo):                                       # :20-21 (fp32 sums; <= 7 non-zero terms)
            product_sum = np.float32(product_sum + np.float32(w[j] * idx_values[lo + j]))
            weight_sum = np.float32(weight_sum + w[j])
        values[i] = product_sum / (weight_sum + np.float32(weight_sum == 0))   # :22
        rest[i] = probs[i].max() < np.float32(threshold)               # :23
    return values, rest


def decode_note_sequence(frame2item: np.ndarray, values: np.ndarray, masks: np.ndarray, threshold=0.5):
    """infer_utils.py:42-76 for one clip.  frame2item int64 [T] (0 = padding), values float32 or
    int64 [T], masks bool [T] -> (item_values float32 [N], item_dur int64 [N], item_masks bool [N]),
    N = max(frame2item) (index 0 dropped, :54,57,65,72-74)."""
    frame2item = np.asarray(frame2item, dtype=np.int64)
    masks = np.asarray(masks, dtype=bool)
    n_items = int(frame2item.max()) if frame2item.size else 0          # :52 space - 1
    integer_values = np.issubdtype(np.asarray(values).dtype, np.integer)
    item_dur = np.zeros(n_items + 1, dtype=np.int64)
    item_unmasked = np.zeros(n_items + 1, dtype=np.int64)
    hist = np.zeros((n_items + 1, 128), dtype=np.int64)
    vq = np.rint(values).astype(np.int64)                              # :61
    for f in range(frame2item.shape[0]):
        it = frame2item[f]
        item_dur[it] += 1                                              # :54-56
        item_unmasked[it] += int(masks[f])                             # :57-59
        hist[it, vq[f]] += int(masks[f])                               # :62-64
    with np.errstate(divide='ignore', invalid='ignore'):
        item_masks = (item_unmasked[1:] / item_dur[1:]) >= threshold   # :60 (0/0 = nan -> False)
    center = hist.argmax(axis=1).astype(np.float32 if not integer_values else np.int64)   # :65 first maximal bin
    center[0] = 0                                                      # :66 F.pad(.., [1, 0])
    item_valid = np.zeros(n_items + 1, dtype=np.int64)
    acc_dtype = np.int64 if integer_values else np.float32
    item_sum = np.zeros(n_items + 1, dtype=acc_dtype)
    for f in range(frame2item.shape[0]):
        it = frame2item[f]
        c = center[it]
        near = bool(masks[f]) and (values[f] >= c - 0.5) and (values[f] <= c + 0.5)   # :67
        item_valid[it] += int(near)                                    # :68-70
        if near:
            item_sum[it] = acc_dtype(item_sum[it] + values[f])         # :71-73 (sequential, own dtype)
    denom = item_valid[1:] + (item_valid[1:] == 0)
    if integer_values:
        item_values = (torch.from_numpy(item_sum[1:]) / torch.from_numpy(denom)).numpy()  # int64/int64 -> float32 (:74)
    else:
        item_values = (item_sum[1:] / denom.astype(np.float32)).astype(np.float32)
    return item_values.astype(np.float32), item_dur[1:], item_masks


# --------------------------------------------------------------------------- vectorised forms (CPU baseline timing)
# The loop forms above are the readable specification; they cost ~35 ms per 30 s clip in pure Python, which would inflate
# the CPU baseline that bench.py reports.  These numpy forms do the same arithmetic in the same order (tests/
# test_oracle_golden.py::test_vectorised_decode_equals_loops) at the speed of the reference's own torch ops.
def decode_gaussian_blurred_probs_vec(probs: np.ndarray, vmin, vmax, deviation, threshold):
    """infer_utils.py:9-24, one gather of the <= 2 * width + 1 bins around the argmax per frame."""
    probs = np.asarray(probs, dtype=np.float32)
    t, n = probs.shape
    interval = (vmax - vmin) / (n - 1)                                 # :11
    width = int(3 * deviation / interval)                              # :12
    idx_values = bin_values(n, interval, vmin)                         # :13-14
    center = probs.argmax(axis=1)                                      # :15
    win = center[:, None] + np.arange(-width, width + 1)[None, :]      # :16-18 as a window of bin indices
    ok = (win >= 0) & (win < n)
    win = np.clip(win, 0, n - 1)
    w = np.where(ok, np.take_along_axis(probs, win, axis=1), np.float32(0))
    prod = (w * idx_values[win]).astype(np.float32)
    product_sum = np.zeros(t, dtype=np.float32)
    weight_sum = np.zeros(t, dtype=np.float32)
    for j in range(win.shape[1]):                                      # ascending bins, fp32, like the loop form
        product_sum = (product_sum + prod[:, j]).astype(np.float32)
        weight_sum = (weight_sum + w[:, j]).astype(np.float32)
    values = product_sum / (weight_sum + (weight_sum == 0).astype(np.float32))   # :22
    rest = probs.max(axis=1) < np.float32(threshold)                   # :23
    return values.astype(np.float32), rest


def decode_note_sequence_vec(frame2item: np.ndarray, values: np.ndarray, masks: np.ndarray, threshold=0.5):
    """infer_utils.py:42-76 for one clip with bincount / add.at instead of per-frame Python loops."""
    frame2item = np.asarray(frame2item, dtype=np.int64)
    masks = np.asarray(masks, dtype=bool)
    values = np.asarray(values)
    n_items = int(frame2item.max()) if frame2item.size else 0
    integer_values = np.issubdtype(values.dtype, np.integer)
    space = n_items + 1
    item_dur = np.bincount(frame2item, minlength=space).astype(np.int64)                  # :54-56
    item_unmasked = np.bincount(frame2item, weights=masks, minlength=space).astype(np.int64)   # :57-59
    with np.errstate(divide='ignore', invalid='ignore'):
        item_masks = (item_unmasked[1:] / item_dur[1:]) >= threshold                       # :60
    vq = np.rint(values).astype(np.int64)                                                  # :61
    hist = np.bincount(frame2item * 128 + vq, weights=masks, minlength=space * 128).reshape(space, 128)   # :62-64
    center = hist.argmax(axis=1).astype(np.int64 if integer_values else np.float32)        # :65
    center[0] = 0                                                                          # :66
    c = center[frame2item]
    near = masks & (values >= c - 0.5) & (values <= c + 0.5)                               # :67
    item_valid = np.bincount(frame2item, weights=near, minlength=space).astype(np.int64)   # :68-70
    acc_dtype = np.int64 if integer_values else np.float32
    item_sum = np.zeros(space, dtype=acc_dtype)
    np.add.at(item_sum, frame2item[near], values[near].astype(acc_dtype))                  # :71-73 frame order, own dtype
    denom = item_valid[1:] + (item_valid[1:] == 0)
    if integer_values:
        item_values = (torch.from_numpy(item_sum[1:]) / torch.from_numpy(denom)).numpy()   # int64 / int64 -> float32 (:74)
    else:
        item_values = (item_sum[1:] / denom.astype(np.float32)).astype(np.float32)
    return item_values.astype(np.float32), item_dur[1:], item_masks


# --------------------------------------------------------------------------- plugin restatement
def infer_clip(sd, config, waveform: np.ndarray, quantized: bool = False, return_intermediates=False, fast=False):
    """One iteration of BaseInference.infer (base_infer.py:48-52): preprocess (me_infer.py:29-63),
    forward_model (:65-76 / me_quant_infer.py:11-19), postprocess (:78-97 / :21-38)."""
    timestep = config['hop_size'] / config['audio_sample_rate']        # base_infer.py:20
    wav = torch.from_numpy(np.ascontiguousarray(waveform, dtype=np.float32)).unsqueeze(0)
    with torch.no_grad():
        mel = omodel.log_mel(wav, config['audio_sample_rate'], config['win_size'], config['hop_size'],
                             config['units_dim'], config['fmin'], config['fmax'])
        units = mel.transpose(1, 2)                                    # me_infer.py:31
        probs, bounds = omodel.model_forward(sd, config, units, mask=torch.ones(units.shape[:2], dtype=torch.bool),
                                             sig=not quantized, softmax=quantized)
    probs_np = probs[0].numpy()
    bounds_np = bounds[0].numpy()
    t = probs_np.shape[0]
    masks = np.ones(t, dtype=bool)                                     # me_infer.py:62 (mask-mul is a no-op)
    frame2item = decode_bounds_to_alignment(bounds_np) * masks         # :84
    if quantized:
        midi = probs_np.argmax(axis=-1).astype(np.int64)               # me_quant_infer.py:28
        rest = midi == 128                                             # :29
        values = np.clip(midi, 0, 127)                                 # :31
    else:
        blur = decode_gaussian_blurred_probs_vec if fast else decode_gaussian_blurred_probs
        values, rest = blur(probs_np, config['midi_min'], config['midi_max'],                   # me_infer.py:85-88
                            config['midi_prob_deviation'], config['rest_threshold'])
    notes = decode_note_sequence_vec if fast else decode_note_sequence
    note_midi, note_dur, note_mask = notes(frame2item, values, ~rest & masks)                   # :89-91
    out = {
        'note_midi': note_midi,                                        # :94
        'note_dur': note_dur * timestep,                               # :95 int64 * python float -> float64
        'note_rest': ~note_mask,                                       # :92,96
    }
    if return_intermediates:
        out.update(mel=mel[0].numpy(), probs=probs_np, bounds=bounds_np, frame2item=frame2item,
                   values=np.asarray(values), rest=rest)
    return out


def infer(sd, config, waveforms, quantized=False, fast=False):
    """BaseInference.infer, base_infer.py:46-53 (serial batch-1 loop).  ``fast`` = the vectorised decode forms (same
    results, the speed of the reference's torch ops): what bench.py times as the CPU baseline."""
    return [infer_clip(sd, config, w, quantized, fast=fast) for w in waveforms]

"""some_decode_notes (csrc/decode.cu) against the oracle, bit for bit, where a decode goes wrong quietly.

The kernel and oracle/decode.py do the same sequential float32 operations, so every output must be identical:
frame2item, rest and values per frame, and note_count, note_dur, note_rest and note_midi per note.  The inputs cover
  * clips longer than one 2048-frame chunk of the alignment scan, which carries the double prefix of the bounds, the
    previous rounded step and the note count from chunk to chunk (1 to 10 337 frames, and clips of no frame);
  * prefixes exactly half-way between two integers (bounds 0.5 and 0.25) on both sides of frame 2048, and bounds within a
    few ulp of 0.5;
  * 5000 one-frame notes in one clip (many passes of the per-note grid-stride);
  * saturated heads: maxima tied across the lanes of a warp (bins j, j + 32, ..., and bin 128 of the quantized head),
    all-zero frames, values exactly on a note's center +- 0.5, histogram-mode ties, notes with no valid frame and notes
    exactly half voiced;
  * head widths 2, 64, 200 and 256, also against the unmodified reference's outputs (tests/golden/decode_bins.npz);
  * the oracle's own 30 s probabilities and bounds, whose notes must come out exactly.
"""
import pathlib
import sys
import types

import numpy as np
import pytest
import torch

from oracle import decode as od
from some_b200 import _lib, synth
from some_b200.engine import Engine

sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent / 'golden'))
from decode_bins_cases import DEVIATION, THRESHOLD, WIDTHS, make_probe  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = 'cuda'
CHUNK = 2048                 # DEC_CHUNK of decode.cu
EDGE_LENGTHS = [1, 2047, 2048, 2049, 4096, 4097, 6143, 10337]


# --------------------------------------------------------------------------- inputs (CPU, seeded)
def _random_probs(rng, t, n):
    return (rng.random((t, n), dtype=np.float32) ** 6).astype(np.float32)


def _saturated_probs(rng, t, n):
    """Sigmoid heads saturate at exactly 1.0, often in several bins of one frame: 1-6 tied maxima per frame at random
    bins or at bins 32 apart (one lane of the kernel's warp), some all-zero frames."""
    p = (rng.random((t, n), dtype=np.float32) ** 6 * 0.9).astype(np.float32)
    for i in range(t):
        kind = i % 4
        if kind == 0:
            p[i, rng.choice(n, min(n, int(rng.integers(1, 7))), replace=False)] = 1.0
        elif kind == 1:
            p[i, int(rng.integers(0, min(32, n)))::32] = 1.0
        elif kind == 2:
            p[i, int(rng.integers(0, n))] = 1.0
            p[i, int(rng.integers(0, n))] = 1.0
        elif rng.random() < 0.5:
            p[i] = 0.0
    return p


def _bounds(rng, t, kind):
    if kind == 'cube':
        return (rng.random(t, dtype=np.float32) ** 3).astype(np.float32)
    if kind == 'half':        # within a few ulp of 0.5: prefixes land on and next to k + 0.5
        return (np.float32(0.5) + rng.integers(-4, 5, t).astype(np.float32) * np.float32(2 ** -24)).astype(np.float32)
    if kind == 'carry':
        # the prefix of the first chunk is 2046.5 + 2^-14, which float32 rounds (half-even) to 2046.5; frame 2048 adds
        # 2^-14 more.  From the double prefix the sum is 2046.5 + 2^-13 (step 2047, a new note at frame 2048); from a
        # prefix carried in float32 it would round back to 2046.5 (step 2046, no new note).
        head = np.array([1.0] * (CHUNK - 2) + [0.5, 2 ** -14, 2 ** -14], dtype=np.float32)
        return np.concatenate([head, _bounds(rng, t - len(head), 'cube')])
    raise ValueError(kind)


def sigmoid_clips():
    """(name, probs [T, 128], bounds [T]) of the one 128-bin launch: 68 clips."""
    rng = np.random.default_rng(2048)
    n = 128
    clips = [('empty0', np.zeros((0, n), np.float32), np.zeros(0, np.float32))]
    for t in EDGE_LENGTHS:
        clips.append((f'len{t}', _random_probs(rng, t, n), _bounds(rng, t, 'cube')))
    for k in range(20):       # the carry of the double prefix over chunk boundaries
        t = int(rng.integers(6000, 12001))
        clips.append((f'long{k}', _random_probs(rng, t, n), _bounds(rng, t, 'cube' if k % 2 == 0 else 'half')))
    clips.append(('carry', _random_probs(rng, 4500, n), _bounds(rng, 4500, 'carry')))
    clips.append(('ones5000', _random_probs(rng, 5000, n), np.ones(5000, np.float32)))
    for b in (0.5, 0.25):
        clips.append((f'exact{b}', _random_probs(rng, 4100, n), np.full(4100, b, np.float32)))
    clips.append(('empty1', np.zeros((0, n), np.float32), np.zeros(0, np.float32)))
    probs, bounds = make_probe(n, 0, 127)            # integer bin values: midpoints sit on center +- 0.5
    clips.append(('probe', probs, bounds))
    clips.append(('probe_cube', np.tile(probs, (6, 1)), _bounds(rng, 6 * len(probs), 'cube')))
    for k in range(8):
        t = int(rng.integers(1500, 7000))
        clips.append((f'saturated{k}', _saturated_probs(rng, t, n), _bounds(rng, t, ('cube', 'half')[k % 2])))
    clips.append(('zeros', np.zeros((3000, n), np.float32), _bounds(rng, 3000, 'cube')))
    while len(clips) < 68:    # short clips between the long ones
        t = int(rng.integers(1, 700))
        clips.append((f'short{len(clips)}', _random_probs(rng, t, n), _bounds(rng, t, 'cube')))
    return clips


def quantized_clips():
    """(name, probs [T, 129], bounds [T]) of the quantized launch: softmax outputs with bin 128 (rest) tied to others."""
    rng = np.random.default_rng(129)
    n = 129

    def softmax(t, rest_bias):
        x = rng.standard_normal((t, n)).astype(np.float32) * 2.0
        x[:, 128] += rest_bias
        return torch.softmax(torch.from_numpy(x), -1).numpy()

    def tied(t):
        p = softmax(t, 0.0) * np.float32(0.5)
        for i in range(t):
            top = np.float32(0.9)
            kind = i % 3
            if kind == 0:     # bin 128 tied with a bin of another lane, or of lane 0 (0, 32, 64, 96)
                p[i, [128, int(rng.integers(0, 128))]] = top
            elif kind == 1:
                p[i, [128, 32 * int(rng.integers(0, 4))]] = top
            else:
                p[i, rng.choice(n, int(rng.integers(2, 6)), replace=False)] = top
        return p

    clips = [('empty0', np.zeros((0, n), np.float32), np.zeros(0, np.float32))]
    for t in EDGE_LENGTHS:
        clips.append((f'len{t}', softmax(t, 1.0), _bounds(rng, t, 'cube')))
    for k in range(4):
        t = int(rng.integers(6000, 12001))
        clips.append((f'long{k}', softmax(t, 1.0), _bounds(rng, t, ('cube', 'half')[k % 2])))
    clips.append(('carry', softmax(4500, 1.0), _bounds(rng, 4500, 'carry')))
    clips.append(('ones5000', softmax(5000, 0.0), np.ones(5000, np.float32)))
    clips.append(('tied', tied(4500), _bounds(rng, 4500, 'cube')))
    clips.append(('uniform', np.full((2500, n), 1 / 129, np.float32), _bounds(rng, 2500, 'half')))
    probs, bounds = make_probe(n, 0, 128)
    clips.append(('probe', probs, bounds))
    return clips


# --------------------------------------------------------------------------- kernel and oracle
@pytest.fixture(scope='module')
def lib():
    return _lib.load()


def _decode(lib, clips, n, quantized, vmin=0, vmax=127):
    """some_decode_notes over all ``clips`` in one launch, through Engine.run_decode -> per clip dict of outputs."""
    eng = Engine.__new__(Engine)
    eng.lib, eng.device, eng.outdim, eng.launches, eng.prof = lib, torch.device(DEV), n, 0, None
    eng.config = dict(midi_min=vmin, midi_max=vmax, midi_prob_deviation=DEVIATION, rest_threshold=THRESHOLD)
    frames = [len(b) for _, _, b in clips]
    cu = np.zeros(len(clips) + 1, dtype=np.int32)
    np.cumsum(frames, out=cu[1:])
    m = int(cu[-1])
    probs = torch.from_numpy(np.concatenate([p for _, p, _ in clips]).reshape(m, n)).to(DEV)
    bounds = torch.from_numpy(np.concatenate([b for _, _, b in clips])).to(DEV)
    ws = types.SimpleNamespace(
        scratch=torch.empty(int(lib.some_decode_scratch_bytes(m)), dtype=torch.uint8, device=DEV),
        note_midi=torch.full((m,), float('nan'), device=DEV),
        note_dur=torch.full((m,), -1, dtype=torch.int32, device=DEV),
        note_rest=torch.full((m,), 7, dtype=torch.uint8, device=DEV))
    nc = torch.full((len(clips),), -1, dtype=torch.int32, device=DEV)
    dbg = {}
    eng.run_decode(ws, m, len(clips), torch.from_numpy(cu).to(DEV), nc, quantized, dbg, probs=probs, bounds=bounds)
    torch.cuda.synchronize()
    host = {k: v.cpu().numpy() for k, v in dbg.items()}
    nd, nm, nr, nc = ws.note_dur.cpu().numpy(), ws.note_midi.cpu().numpy(), ws.note_rest.cpu().numpy(), nc.cpu().numpy()
    out = []
    for i in range(len(clips)):
        r0, r1 = int(cu[i]), int(cu[i + 1])
        k = int(nc[i])
        out.append({'frame2item': host['frame2item'][r0:r1], 'values': host['values'][r0:r1],
                    'rest': host['rest'][r0:r1].astype(bool), 'note_count': k, 'note_dur': nd[r0:r0 + k],
                    'note_midi': nm[r0:r0 + k], 'note_rest': nr[r0:r0 + k].astype(bool)})
    return out


def _oracle(probs, bounds, quantized, vmin=0, vmax=127):
    f2i = od.decode_bounds_to_alignment(bounds)
    if quantized:
        midi = probs.argmax(-1).astype(np.int64)
        rest, vals = midi == 128, np.clip(midi, 0, 127)
    else:
        vals, rest = od.decode_gaussian_blurred_probs_vec(probs, vmin, vmax, DEVIATION, THRESHOLD)
    nm, nd, nk = od.decode_note_sequence_vec(f2i, vals, ~rest)
    return {'frame2item': f2i, 'values': vals.astype(np.float32), 'rest': rest, 'note_count': len(nd), 'note_dur': nd,
            'note_midi': nm, 'note_rest': ~nk}


def _assert_equal(name, got, ref):
    assert got['note_count'] == ref['note_count'], (name, got['note_count'], ref['note_count'])
    for k in ('frame2item', 'rest', 'values', 'note_dur', 'note_rest', 'note_midi'):
        g, r = got[k], ref[k]
        bad = np.nonzero(g != r)[0] if g.shape == r.shape else []
        assert g.shape == r.shape and len(bad) == 0, \
            f'{name}: {k} differs at {len(bad)} places, first {bad[:5]}: {g[bad[:5]]} vs {r[bad[:5]]}'


# --------------------------------------------------------------------------- tests
def test_sigmoid_head_chunks_ties_and_zeros_bit_exact(lib):
    clips = sigmoid_clips()
    assert len(clips) >= 64
    got = _decode(lib, clips, 128, False)
    for (name, p, b), g in zip(clips, got):
        _assert_equal(name, g, _oracle(p, b, False))
    by_name = dict(zip([c[0] for c in clips], got))
    assert by_name['empty0']['note_count'] == by_name['empty1']['note_count'] == 0
    assert by_name['ones5000']['note_count'] == 5000
    assert by_name['exact0.5']['note_count'] == 2051         # round-half-even: steps 0, 1, 2, 2, 2, 3, 4, 4, 4, ...
    f2i = by_name['carry']['frame2item']
    assert f2i[CHUNK] == f2i[CHUNK - 1] + 1


def test_quantized_head_chunks_and_rest_ties_bit_exact(lib):
    clips = quantized_clips()
    got = _decode(lib, clips, 129, True)
    for (name, p, b), g in zip(clips, got):
        _assert_equal(name, g, _oracle(p, b, True))
    by_name = dict(zip([c[0] for c in clips], got))
    assert not by_name['tied']['rest'].any()                # bin 128 tied with any other bin: the other bin wins
    assert by_name['len10337']['rest'].any()


@pytest.mark.parametrize('n,vmin,vmax', WIDTHS)
def test_head_widths_match_reference_and_oracle(lib, golden_dir, n, vmin, vmax):
    g = np.load(golden_dir / 'decode_bins.npz')
    key = f'n{n}_{vmin}_{vmax}'
    rng = np.random.default_rng(n)
    probs, bounds = make_probe(n, vmin, vmax)
    clips = [('probe', probs, bounds),
             ('probe_cube', np.tile(probs, (4, 1)), _bounds(rng, 4 * len(probs), 'cube')),
             ('random', _random_probs(rng, 4500, n), _bounds(rng, 4500, 'cube')),
             ('saturated', _saturated_probs(rng, 2100, n), _bounds(rng, 2100, 'half'))]
    got = _decode(lib, clips, n, False, vmin, vmax)
    for (name, p, b), r in zip(clips, got):
        _assert_equal(f'{key} {name}', r, _oracle(p, b, False, vmin, vmax))
    ref = {'frame2item': g[f'{key}_frame2item'], 'values': g[f'{key}_values'], 'rest': g[f'{key}_rest'],
           'note_count': len(g[f'{key}_note_dur']), 'note_dur': g[f'{key}_note_dur'],
           'note_midi': g[f'{key}_note_midi'], 'note_rest': ~g[f'{key}_note_mask']}
    _assert_equal(f'{key} reference', got[0], ref)


@pytest.mark.parametrize('cfg', ['two_head', 'quant_two_head'])
def test_oracle_distribution_30s_notes_exact(lib, cfg):
    """The probabilities and bounds a model produces (the oracle's forward on a 30 s clip, 2584 frames) decode to the
    oracle's notes exactly."""
    config = synth.named_config(cfg)
    quantized = cfg.startswith('quant')
    sd = synth.fabricate_state_dict(config, seed=1234)
    out = od.infer_clip(sd, config, synth.synth_waveform(31, seconds=30.0), quantized=quantized,
                        return_intermediates=True, fast=True)
    assert out['probs'].shape[0] > CHUNK
    got = _decode(lib, [(cfg, out['probs'], out['bounds'])], config['midi_num_bins'], quantized)[0]
    _assert_equal(cfg, got, _oracle(out['probs'], out['bounds'], quantized))
    np.testing.assert_array_equal(got['note_midi'], out['note_midi'])
    np.testing.assert_array_equal(got['note_dur'] * (512 / 44100), out['note_dur'])
    np.testing.assert_array_equal(got['note_rest'], out['note_rest'])

"""GPU tests of some_eval_clips (csrc/evaluate.cu) and the evaluator (some_b200/evaluate.py) against
tests/golden/eval_*.npz, which the unmodified reference produced (tests/golden/make_golden_eval.py): losses within
relative 1e-5 and accuracy counts exactly equal, for the golden logits and for the fp32 driver on the fixture's audio;
launch-independence; predicted notes equal to infer()'s; FLAC / 48 kHz inputs; and the measured bf16 vs fp32 gap."""
import numpy as np
import pytest
import torch

from oracle import evaluate as oeval
from oracle import flac as of
from some_b200 import _lib, audio, evaluate, plugin, synth

pytestmark = pytest.mark.gpu

TIMESTEP = 512 / 44100
CFGS = ['two_head', 'quant_two_head']


def _instance(cfg, tmp_path):
    config = synth.named_config(cfg)
    ckpt = synth.write_checkpoint(tmp_path / 'ckpt', config, seed=1234)
    cls = plugin.QuantizedMIDIExtractionInference if cfg.startswith('quant') else plugin.MIDIExtractionInference
    return cls(config=config, model_path=ckpt, device='cuda:0'), config


def _golden(golden_dir, cfg, tmp_path):
    """(npz, dataset dir, per-item label arrays) of the fixture, the dataset rewritten from the generator's seeds."""
    g = np.load(golden_dir / f'eval_{cfg}.npz')
    quantized = cfg.startswith('quant')
    items = [(f'item{s}',) + synth.synth_labelled(int(s), float(t)) for s, t in zip(g['seeds'], g['seconds'])]
    data = synth.write_labelled_dataset(tmp_path / 'data', items)
    labs = evaluate.load_labels(data, synth.named_config(cfg), quantized)
    arrs = [evaluate.item_labels(it, g[f'item{i}_unit2note'].shape[0], TIMESTEP, quantized) for i, it in enumerate(labs)]
    return g, data, arrs


class _FakeEngine:
    """Just what evaluate.eval_clips reads from an engine."""

    def __init__(self, config):
        self.config = config
        self.outdim = config['midi_num_bins']
        self.lib = _lib.load()
        self.prof = None
        self.launches = 0

    @property
    def _stream(self):
        import ctypes
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def _mark(self, name, work):
        import contextlib
        return contextlib.nullcontext()


def _kernel(config, quantized, logits, bounds, arrs, head=_lib.EVAL_HEAD_F32):
    """some_eval_clips over the given clips in one launch -> (midi sums, bound sums, correct, probs)."""
    dev = torch.device('cuda', 0)
    cu = np.concatenate([[0], np.cumsum([len(b) for b in bounds])]).astype(np.int32)
    lg = torch.from_numpy(np.concatenate(logits)).to(dev)
    bd = torch.from_numpy(np.concatenate(bounds)).to(dev)
    cu_d = torch.from_numpy(cu).to(dev)
    lab = evaluate._Labels(arrs, dev)
    probs = torch.empty_like(lg)
    evaluate.eval_clips(_FakeEngine(config), lg, bd, cu_d, lab, 0, len(arrs), 0, int(cu[-1]), quantized, head, probs=probs)
    torch.cuda.synchronize()
    return lab.midi_loss.cpu().numpy(), lab.bound_loss.cpu().numpy(), lab.correct.cpu().numpy(), probs.cpu().numpy(), cu


def _per_item(sums, t, n, quantized):
    return sums / t if quantized else sums / (t * n)


@pytest.mark.parametrize('cfg', CFGS)
def test_kernel_on_golden_logits(cfg, golden_dir, tmp_path):
    g, _, arrs = _golden(golden_dir, cfg, tmp_path)
    config = synth.named_config(cfg)
    quantized = cfg.startswith('quant')
    for pre in ('', 'lean_'):
        k = len(arrs)
        logits = [g[f'item{i}_{pre}logits'] for i in range(k)]
        bounds = [g[f'item{i}_{pre}bounds'] for i in range(k)]
        ms, bs, cor, probs, cu = _kernel(config, quantized, logits, bounds, arrs)
        for i in range(k):
            t = len(bounds[i])
            np.testing.assert_allclose(_per_item(ms[i], t, config['midi_num_bins'], quantized), g[f'item{i}_{pre}midi_loss'],
                                       rtol=1e-5)
            np.testing.assert_allclose(bs[i] / t, g[f'item{i}_{pre}bound_loss'], rtol=1e-5)
            assert cor[i] == g[f'item{i}_{pre}correct'], (pre, i)
            ref = torch.softmax(torch.from_numpy(logits[i]), -1) if quantized else torch.sigmoid(torch.from_numpy(logits[i]))
            np.testing.assert_allclose(probs[cu[i]:cu[i + 1]], ref.numpy(), rtol=1e-5, atol=1e-7)
    assert g['item0_lean_correct'] > 0


def _spanning_clip(rng, t, config, quantized):
    """(logits [t, N], bounds [t], label arrays) of a clip whose notes (20-400 frames, some rests) span every multiple of
    2048, the chunk of the kernel's bound-loss scan.  Most frames of a pitched note lean towards its pitch, so the
    accuracy counts are far from 0."""
    n = config['midi_num_bins']
    starts = [0]
    while starts[-1] < t:
        s = starts[-1] + int(rng.integers(20, 400))
        if any(s - 60 <= c <= s + 60 for c in range(2048, t, 2048)):
            s += 150                                                     # no note starts right at a chunk boundary
        starts.append(s)
    durs = np.diff(np.minimum(starts, t))
    durs = durs[durs > 0]
    k = len(durs)
    unit2note = np.repeat(np.arange(1, k + 1, dtype=np.int64), durs)
    rest = rng.random(k) < 0.15
    if quantized:
        note_midi = np.where(rest, 128, rng.integers(0, 128, k)).astype(np.int64)
        target = note_midi[unit2note - 1]
        logits = rng.standard_normal((t, n)).astype(np.float32) * 2.0
        lean = rng.random(t) < 0.7
        logits[np.nonzero(lean)[0], target[lean]] += 6.0
    else:
        vmin, vmax = config['midi_min'], config['midi_max']
        note_midi = rng.uniform(vmin + 1, vmax - 1, k).astype(np.float32)
        interval = (vmax - vmin) / (n - 1)
        miu = (note_midi[unit2note - 1] - vmin) / interval
        bump = np.exp(-((np.arange(n)[None, :] - miu[:, None]) * interval / config['midi_prob_deviation']) ** 2 / 2)
        lean = (rng.random(t) < 0.7) & ~rest[unit2note - 1]
        logits = (rng.standard_normal((t, n)) * 1.5 - 3.0 + 9.0 * bump * lean[:, None]).astype(np.float32)
    bounds = rng.random(t) ** 8 * 0.1                                    # a bound head: high where a note starts
    bounds[np.cumsum(durs)[:-1]] = rng.uniform(0.6, 1.0, k - 1)
    bounds = bounds.astype(np.float32)
    labels = {'unit2note': unit2note, 'note_midi': note_midi, 'note_rest': rest if not quantized else note_midi == 128}
    for c in range(2048, t, 2048):
        assert unit2note[c - 1] == unit2note[c]
    return logits, bounds, labels


@pytest.mark.parametrize('head', [_lib.EVAL_HEAD_TC, _lib.EVAL_HEAD_F32])
@pytest.mark.parametrize('cfg,bins,vmin,vmax', [('two_head', 128, 0, 127), ('two_head', 200, 21, 108),
                                                ('quant_two_head', 129, 0, 127)])
def test_kernel_past_one_chunk(cfg, bins, vmin, vmax, head):
    """Clips of 2047 to 9000 frames, so the bound-loss scan carries its double prefix, note count and previous note across
    2048-frame chunks: losses against the oracle on the logits, and the accuracy counts exactly against the oracle's on the
    kernel's own activations (CUDA's exp and torch's can differ by an ulp, which may move a value across +- 0.5)."""
    config = dict(synth.named_config(cfg), midi_num_bins=bins, midi_min=vmin, midi_max=vmax)
    quantized = cfg.startswith('quant')
    rng = np.random.default_rng(bins + head)
    clips = [_spanning_clip(rng, t, config, quantized) for t in (2047, 2048, 2049, 5000, 9000)]
    logits, bounds, arrs = (list(x) for x in zip(*clips))
    ms, bs, cor, probs, cu = _kernel(config, quantized, logits, bounds, arrs, head=head)
    for i, t in enumerate(len(b) for b in bounds):
        ref = oeval.losses(logits[i], bounds[i], arrs[i], config, quantized)
        np.testing.assert_allclose(_per_item(ms[i], t, bins, quantized), ref['midi_loss'], rtol=1e-5)
        np.testing.assert_allclose(bs[i] / t, ref['bound_loss'], rtol=1e-5)
        p = probs[cu[i]:cu[i + 1]]
        act = torch.softmax(torch.from_numpy(logits[i]), -1) if quantized else torch.sigmoid(torch.from_numpy(logits[i]))
        np.testing.assert_allclose(p, act.numpy(), rtol=1e-5, atol=1e-7)
        correct, total = oeval.accuracy_counts(logits[i], arrs[i], config, quantized, probs=p)
        assert total == t and cor[i] == correct, (i, cor[i], correct)
        assert correct > t // 8, correct


@pytest.mark.parametrize('cfg', CFGS)
def test_mixed_launch_equals_one_at_a_time(cfg, golden_dir, tmp_path):
    """Per-clip results are bitwise independent of which other clips share the launch (and of the launch count)."""
    g, _, arrs = _golden(golden_dir, cfg, tmp_path)
    config = synth.named_config(cfg)
    quantized = cfg.startswith('quant')
    rng = np.random.default_rng(5)
    order = rng.permutation(np.repeat(np.arange(len(arrs)), 9))           # 18 clips, both fixtures items, mixed
    pres = ['', 'lean_']
    logits = [g[f'item{i % 2}_{pres[j % 2]}logits'] for j, i in enumerate(order)]
    bounds = [g[f'item{i % 2}_{pres[j % 2]}bounds'] for j, i in enumerate(order)]
    many = _kernel(config, quantized, logits, bounds, [arrs[i] for i in order], head=_lib.EVAL_HEAD_TC)
    for j, i in enumerate(order):
        one = _kernel(config, quantized, [logits[j]], [bounds[j]], [arrs[i]], head=_lib.EVAL_HEAD_TC)
        assert many[0][j] == one[0][0] and many[1][j] == one[1][0] and many[2][j] == one[2][0], j
        np.testing.assert_array_equal(many[3][many[4][j]:many[4][j + 1]], one[3])


@pytest.mark.parametrize('cfg', CFGS)
def test_fp32_driver_matches_reference(cfg, golden_dir, tmp_path):
    g, data, _ = _golden(golden_dir, cfg, tmp_path)
    ins, config = _instance(cfg, tmp_path)
    rep = evaluate.evaluate_dataset(ins, data, config, precision='fp32')
    quantized = cfg.startswith('quant')
    assert [it.name for it in rep.items] == [str(g[f'item{i}_name']) for i in range(len(rep.items))]
    for i, it in enumerate(rep.items):
        assert it.frames == it.total == g[f'item{i}_unit2note'].shape[0]
        np.testing.assert_allclose(it.midi_loss, g[f'item{i}_midi_loss'], rtol=1e-5)
        np.testing.assert_allclose(it.bound_loss, g[f'item{i}_bound_loss'], rtol=1e-5)
        assert it.correct == g[f'item{i}_correct']
    # the predicted notes are infer_accurate()'s
    waves = [audio.load_native(data / 'wavs' / f'item{s}.wav')[0] for s in g['seeds']]
    acc = ins.model.infer_accurate(waves, quantized)
    for it, r in zip(rep.items, acc):
        for k in ('note_midi', 'note_dur', 'note_rest'):
            np.testing.assert_array_equal(getattr(it, k), r[k])


@pytest.mark.parametrize('cfg', CFGS)
def test_bf16_notes_equal_infer_and_batching(cfg, tmp_path):
    """bf16 driver: predicted notes equal infer()'s exactly; a batch of many items equals the items one at a time."""
    ins, config = _instance(cfg, tmp_path)
    items = [(f's{k}',) + synth.synth_labelled(700 + k, 3.0 + 2.1 * k) for k in range(6)]
    data = synth.write_labelled_dataset(tmp_path / 'data', items)
    rep = evaluate.evaluate_dataset(ins, data, config)
    waves = [audio.load_native(data / 'wavs' / f'{n}.wav')[0] for n, *_ in items]
    ref = ins.infer(waves)
    for it, r in zip(rep.items, ref):
        for k in ('note_midi', 'note_dur', 'note_rest'):
            np.testing.assert_array_equal(getattr(it, k), r[k])
    small = evaluate.evaluate_dataset(ins, data, config, max_frames_per_batch=1)         # one item per batch
    for a, b in zip(rep.items, small.items):
        assert (a.midi_loss, a.bound_loss, a.correct, a.total) == (b.midi_loss, b.bound_loss, b.correct, b.total)
    assert rep.summary == small.summary
    assert set(rep.summary) == {'midi_loss', 'bound_loss', 'total_loss', 'midi_acc'}


def test_flac_and_48k_inputs(tmp_path):
    ins, config = _instance('two_head', tmp_path)
    w, lab = synth.synth_labelled(901, 4.0)
    base = synth.write_labelled_dataset(tmp_path / 'wav', [('a', w, lab)])
    # FLAC of the same 16-bit samples, under the .wav name (the loader sniffs the content)
    ints = np.round(audio.load_native(base / 'wavs' / 'a.wav')[0].astype(np.float64) * 32768).astype(np.int64)
    flac = synth.write_labelled_dataset(tmp_path / 'flac', [('a', w, lab)])
    (flac / 'wavs' / 'a.wav').write_bytes(of.encode(ints[:, None], rate=44100, bps=16))
    r_wav = evaluate.evaluate_dataset(ins, base, config)
    r_flac = evaluate.evaluate_dataset(ins, flac, config, load_audio=audio.read_encoded)
    # 48 kHz WAV: the same report as the 44.1 kHz samples librosa.load would resample it to
    w48 = synth.write_labelled_dataset(tmp_path / 'w48', [('a', w, lab)], sr=48000)
    y48, _ = audio.load_native(w48 / 'wavs' / 'a.wav')
    y = audio.resample(y48, 48000, 44100)
    r48 = evaluate.evaluate_dataset(ins, w48, config)
    arr = evaluate.item_labels(evaluate.load_labels(w48, config)[0], 1 + len(y) // 512, TIMESTEP)
    ms, bs, c, t, notes = evaluate.evaluate_recordings(ins, [y], [arr])[0]
    assert (r48.items[0].midi_loss, r48.items[0].bound_loss, r48.items[0].correct) == (ms / (t * 128), bs / t, c)
    np.testing.assert_array_equal(r48.items[0].note_midi, notes['note_midi'])
    a, b = r_wav.items[0], r_flac.items[0]
    assert (a.midi_loss, a.bound_loss, a.correct, a.total) == (b.midi_loss, b.bound_loss, b.correct, b.total)
    np.testing.assert_array_equal(a.note_midi, b.note_midi)


# bf16 vs fp32 on seeded random weights and labelled synthetic audio (12 items of 6-20 s).  Relative gaps of the summary
# losses measured on an H100 (BASELINE.md): midi_loss 2.3e-5 / 1.1e-5, bound_loss 1.5e-4 / 6.0e-4, total_loss 1.4e-4 / 2.7e-4
# (two_head / quant_two_head).  The bounds are 5-10x the largest of them: operand rounding passes, a change in what the
# bf16 trunk computes does not.  With random weights no frame is a hit on either path (midi_acc = 0 on both), so the
# accuracy bound (an absolute 2 % of the frames) is not yet tied to a measurement on a trained checkpoint.
GAP = {'midi_loss': 2e-4, 'bound_loss': 3e-3, 'total_loss': 2e-3, 'midi_acc': 2e-2}


@pytest.mark.parametrize('cfg', CFGS)
def test_bf16_vs_fp32_gap(cfg, tmp_path):
    ins, config = _instance(cfg, tmp_path)
    items = [(f'g{k}',) + synth.synth_labelled(800 + k, 6.0 + 1.3 * k) for k in range(12)]
    data = synth.write_labelled_dataset(tmp_path / 'data', items)
    b = evaluate.evaluate_dataset(ins, data, config)
    f = evaluate.evaluate_dataset(ins, data, config, precision='fp32')
    gaps = {}
    for k in GAP:
        gaps[k] = abs(b.summary[k] - f.summary[k]) / (abs(f.summary[k]) if k != 'midi_acc' else 1.0)
    print(f'{cfg}: bf16 {b.summary} fp32 {f.summary} gap {gaps}')
    for k, tol in GAP.items():
        assert gaps[k] <= tol, (k, gaps[k])

"""The tiled fp32 trunk (some_forward_f32_tiled, csrc/accurate.cu) against the fp32 checker (some_forward_f32): every
workspace buffer bit for bit, for every model kind and head, on var-len batches whose clip lengths sit on and around every
tile edge of the three tiled kernels (GEMM rows 128, attention queries 64 and keys 32, depthwise-conv rows 32); clips are
independent of their batch; and the layers above it: Engine.infer / infer_sliced with precision='fp32', the plugin's
`infer_precision: fp32` and the batched fp32 evaluation, each against the checker's one-clip-at-a-time drivers."""
import ctypes as C

import numpy as np
import pytest
import torch

from some_b200 import _lib, evaluate, plugin, synth
from some_b200.config import DIM, FFN_DIM
from some_b200.slicer import Slicer

pytestmark = pytest.mark.gpu

HOP = 512
# 1 .. 2584 frames (a 30 s clip); 31-33 / 63-65 / 127-129 straddle the 32-row, 64-query and 128-row tiles
FRAMES = [1, 2, 31, 32, 33, 63, 64, 65, 95, 97, 127, 128, 129, 191, 862, 2584]
HEADS = {'sigmoid': _lib.EPI_SIGMOID_F32, 'softmax': _lib.EPI_SOFTMAX_F32, 'logits': _lib.EPI_BIAS_F32}
BUFFERS = ('x', 'a', 'h', 'qkv', 'g', 'y', 'probs', 'bounds')


def _instance(cfg, tmp_path, **overrides):
    config = synth.named_config(cfg)
    config.update(overrides)
    ckpt = synth.write_checkpoint(tmp_path / 'ckpt', config, seed=1234)
    cls = plugin.QuantizedMIDIExtractionInference if cfg.startswith('quant') else plugin.MIDIExtractionInference
    return cls(config=config, model_path=ckpt, device='cuda:0'), config


def _waves(frames, seed):
    """One synthetic clip per entry with exactly that many frames (T = 1 + len // 512)."""
    rng = np.random.default_rng(seed)
    return [synth.synth_waveform(seed + i, num_samples=(t - 1) * HOP + int(rng.integers(0, HOP)))
            for i, t in enumerate(frames)]


class _Ws:
    """An fp32 workspace of torch tensors, every buffer pre-filled with the same NaN pattern."""

    def __init__(self, m, outdim):
        f = lambda *shape: torch.full(shape, float('nan'), dtype=torch.float32, device='cuda')
        self.t = {'x': f(2, m, DIM), 'a': f(2, m, DIM), 'h': f(2, m, FFN_DIM), 'qkv': f(2, m, 3 * DIM), 'g': f(2, m, DIM),
                  'y': f(2, m, 2 * DIM), 'units': f(m, 80), 'probs': f(m, outdim), 'bounds': f(m)}
        c = self.c = _lib.WorkspaceF32C()
        for s in range(2):
            for k in ('x', 'a', 'h', 'qkv', 'g', 'y'):
                getattr(c, k)[s] = self.t[k][s].data_ptr()
        c.units, c.probs, c.bounds = self.t['units'].data_ptr(), self.t['probs'].data_ptr(), self.t['bounds'].data_ptr()


def _mel(eng, waves):
    host, tables, cu = eng.pack(waves)
    m = int(cu[-1])
    units = torch.empty((m, 80), dtype=torch.float32, device='cuda')
    tab = tables.cuda()
    cu_d = torch.from_numpy(cu).cuda()
    eng.run_mel(host.cuda(), tab[:len(waves)], tab[len(waves):], cu_d, len(waves), int(np.diff(cu).max()), units, None)
    return units, cu


def _run(eng, fn, units, cu, head):
    m, b = int(cu[-1]), len(cu) - 1
    ws = _Ws(m, eng.outdim)
    ws.t['units'].copy_(units)
    cu_d = torch.from_numpy(cu.astype(np.int32)).cuda()
    _lib.check(fn(C.byref(eng.model_f32()), C.byref(ws.c), m, b, cu_d.data_ptr(), int(np.diff(cu).max()), HEADS[head],
                  eng._stream), fn.__name__)
    torch.cuda.synchronize()
    return ws.t


@pytest.mark.parametrize('cfg', ['two_head', 'quant_two_head', 'midi_conformer'])
def test_every_buffer_equals_checker(cfg, tmp_path):
    ins, _ = _instance(cfg, tmp_path)
    eng = ins.model
    units, cu = _mel(eng, _waves(FRAMES, 11))
    m = int(cu[-1])
    assert m % 128 and m % 64 and m % 32, m          # the last row tile of every kernel is partial
    for head in HEADS:
        want = _run(eng, eng.lib.some_forward_f32, units, cu, head)
        got = _run(eng, eng.lib.some_forward_f32_tiled, units, cu, head)
        for k in BUFFERS:
            assert torch.equal(got[k], want[k]), (cfg, head, k)
        assert not torch.isnan(got['probs']).any() and not torch.isnan(got['bounds']).any()


def test_clip_rows_do_not_depend_on_the_batch(tmp_path):
    ins, _ = _instance('two_head', tmp_path)
    eng = ins.model
    frames = [33, 1, 129, 862, 64, 2]
    waves = _waves(frames, 23)
    units, cu = _mel(eng, waves)
    batch = _run(eng, eng.lib.some_forward_f32_tiled, units, cu, 'sigmoid')
    for i, t in enumerate(frames):
        alone = _run(eng, eng.lib.some_forward_f32_tiled, units[cu[i]:cu[i + 1]], np.array([0, t]), 'sigmoid')
        for k in ('x', 'a', 'h', 'qkv', 'g', 'y'):
            assert torch.equal(batch[k][:, cu[i]:cu[i + 1]], alone[k]), (t, k)
        for k in ('probs', 'bounds'):
            assert torch.equal(batch[k][cu[i]:cu[i + 1]], alone[k]), (t, k)


def test_workspace_f32_carve():
    lib = _lib.load()
    for m, n in ((1, 128), (1000, 129), (4097, 128)):
        nbytes = int(lib.some_workspace_f32_bytes(m, n))
        block = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
        c = _lib.WorkspaceF32C()
        _lib.check(lib.some_workspace_f32_carve(block.data_ptr(), nbytes, m, n, C.byref(c)), 'carve')
        ptrs = [c.x[0], c.x[1], c.a[0], c.a[1], c.h[0], c.h[1], c.qkv[0], c.qkv[1], c.g[0], c.g[1], c.y[0], c.y[1],
                c.units, c.probs, c.bounds]
        sizes = [4 * m * w for w in (DIM,) * 4 + (FFN_DIM,) * 2 + (3 * DIM,) * 2 + (DIM,) * 2 + (2 * DIM,) * 2 + (80, n, 1)]
        assert all(p % 256 == 0 for p in ptrs)
        assert all(p + s <= q for p, s, q in zip(ptrs, sizes, ptrs[1:]))
        assert ptrs[-1] + sizes[-1] <= block.data_ptr() + nbytes
        assert lib.some_workspace_f32_carve(block.data_ptr(), nbytes - 1, m, n, C.byref(c)) < 0
        assert b'too small' in lib.some_last_error()


@pytest.mark.parametrize('cfg', ['two_head', 'quant_two_head'])
def test_engine_fp32_equals_infer_accurate(cfg, tmp_path):
    ins, _ = _instance(cfg, tmp_path)
    eng = ins.model
    q = cfg.startswith('quant')
    waves = _waves([2584] * 13 + [1, 65, 862, 300], 41)        # > 2 x 16384 frames: three pipeline chunks
    _, cu, _ = eng.pack(waves)
    assert len(eng._chunks(cu)) > 1
    got = eng.infer(waves, q, precision='fp32')
    inter = eng.infer(waves[-4:], q, return_intermediates=True, precision='fp32')
    want = eng.infer_accurate(waves, q)
    for g, w in zip(got, want):
        for k in ('note_midi', 'note_dur', 'note_rest'):
            np.testing.assert_array_equal(g[k], w[k])
    for g, w in zip(inter, want[-4:]):
        for k in ('note_midi', 'note_dur', 'note_rest', 'mel', 'probs', 'bounds'):
            np.testing.assert_array_equal(g[k], w[k])
    with pytest.raises(ValueError):
        eng.infer(waves[:1], q, precision='fp16')


@pytest.mark.parametrize('cfg', ['two_head', 'quant_two_head'])
def test_plugin_infer_precision(cfg, tmp_path):
    ins, _ = _instance(cfg, tmp_path, infer_precision='fp32')
    assert ins.precision == 'fp32'
    waves = _waves([400, 1, 129], 61)
    got = ins.infer(waves)
    want = ins.model.infer_accurate(waves, ins.quantized)
    for g, w in zip(got, want):
        for k in ('note_midi', 'note_dur', 'note_rest'):
            np.testing.assert_array_equal(g[k], w[k])
    # a long recording: slicer chunks through the fp32 trunk, each the checker's notes on that chunk
    rec = np.concatenate([synth.synth_waveform(71, seconds=9.0), np.zeros(44100, np.float32),
                          synth.synth_waveform(72, seconds=7.0)])
    slicer = Slicer(sr=44100, max_sil_kept=1000)
    offs, notes = ins.model.infer_sliced(rec, slicer, ins.quantized, precision='fp32')
    chunks = slicer.slice(rec)
    assert len(chunks) > 1 and offs == [c['offset'] for c in chunks]
    for n, w in zip(notes, ins.model.infer_accurate([c['waveform'] for c in chunks], ins.quantized)):
        for k in ('note_midi', 'note_dur', 'note_rest'):
            np.testing.assert_array_equal(n[k], w[k])


@pytest.mark.parametrize('cfg', ['two_head', 'quant_two_head'])
def test_batched_fp32_evaluation_equals_per_item(cfg, tmp_path):
    ins, config = _instance(cfg, tmp_path)
    items = [(f'e{k}',) + synth.synth_labelled(900 + k, 2.0 + 1.7 * k) for k in range(7)]
    data = synth.write_labelled_dataset(tmp_path / 'data', items)
    batched = evaluate.evaluate_dataset(ins, data, config, precision='fp32')
    per_item = evaluate.evaluate_dataset(ins, data, config, precision='fp32', per_item=True)
    assert len(batched.items) == len(per_item.items) == 7
    for a, b in zip(batched.items, per_item.items):
        assert (a.name, a.frames, a.midi_loss, a.bound_loss, a.correct, a.total) == \
               (b.name, b.frames, b.midi_loss, b.bound_loss, b.correct, b.total)
        for k in ('note_midi', 'note_dur', 'note_rest'):
            np.testing.assert_array_equal(getattr(a, k), getattr(b, k))
    assert batched.summary == per_item.summary and batched.precision == 'fp32'
    with pytest.raises(ValueError):
        evaluate.evaluate_dataset(ins, data, config, per_item=True)

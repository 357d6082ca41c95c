"""End-to-end GPU parity: the plugin (waveform -> notes through libsome_b200.so) against the golden
vectors produced by the unmodified reference (tests/golden) and against the oracle restatement.

Tolerances (BASELINE.json north_star: 1e-2 on bf16 outputs): probabilities / bounds within 1e-2 of the
fp32 reference; decoded notes are discontinuous functions of those (cumsum().round()), so note
agreement is reported as a rate and asserted loosely, while the decode itself is tested bit-exactly in
test_gpu_kernels.py::test_decode_matches_oracle."""
import numpy as np
import pytest
import torch

from some_b200 import synth

pytestmark = pytest.mark.gpu


def _plugin(cfg_name, tmp_path):
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    from some_b200 import plugin
    config = synth.named_config(cfg_name)
    ckpt = synth.write_checkpoint(tmp_path, config, seed=1234)
    cls = plugin.QuantizedMIDIExtractionInference if cfg_name.startswith('quant') else plugin.MIDIExtractionInference
    return cls(config=config, model_path=ckpt), config


def _golden_waves(g, cfg_name):
    secs = float(g['seconds'])
    waves = [synth.synth_waveform(int(s), seconds=secs + 0.37 * i) for i, s in enumerate(g['seeds'])]
    if cfg_name == 'two_head':
        waves += [synth.edge_case_waveforms()['ragged'], synth.edge_case_waveforms()['short']]
    return waves


def _note_agreement(a, b):
    """fraction of frames whose (rounded pitch, rest) label agrees between two note lists"""
    def expand(r, hop=512 / 44100):
        d = np.rint(np.asarray(r['note_dur']) / hop).astype(int)
        lab = np.where(r['note_rest'], -1, np.rint(r['note_midi']).astype(int))
        return np.repeat(lab, d)
    ea, eb = expand(a), expand(b)
    n = min(len(ea), len(eb))
    return float((ea[:n] == eb[:n]).mean()) if n else 1.0


@pytest.mark.parametrize('cfg_name', ['two_head', 'quant_two_head', 'midi_conformer'])
def test_plugin_matches_reference_golden(cfg_name, tmp_path, golden_dir):
    ins, config = _plugin(cfg_name, tmp_path)
    g = np.load(golden_dir / f'plugin_{cfg_name}.npz')
    waves = _golden_waves(g, cfg_name)
    # per-clip API: preprocess -> forward_model (probabilities, like the reference returns them)
    worst_p = worst_b = 0.0
    for i, w in enumerate(waves):
        sample = ins.preprocess(w)
        assert sample['units'].shape == (1, synth.frames_of(len(w)), 80)
        res = ins.forward_model(sample)
        probs, bounds = res['probs'][0].cpu().numpy(), res['bounds'][0].cpu().numpy()
        assert probs.shape == g[f'clip{i}_probs'].shape
        worst_p = max(worst_p, float(np.abs(probs - g[f'clip{i}_probs']).max()))
        worst_b = max(worst_b, float(np.abs(bounds - g[f'clip{i}_bounds']).max()))
        notes = ins.postprocess(res)
        assert notes['note_midi'].dtype == np.float32 and notes['note_dur'].dtype == np.float64
        assert notes['note_rest'].dtype == np.bool_
    print(f'{cfg_name}: max |probs - ref| = {worst_p:.3e}, max |bounds - ref| = {worst_b:.3e}')
    assert worst_p < 1e-2 and worst_b < 1e-2          # bf16 tolerance of the north star
    # batched public entry point == per-clip path, and close to the reference's notes
    batch = ins.infer(waves)
    assert len(batch) == len(waves)
    rates = []
    for i, (w, r) in enumerate(zip(waves, batch)):
        ref = {k: g[f'clip{i}_{k}'] for k in ('note_midi', 'note_dur', 'note_rest')}
        assert abs(r['note_dur'].sum() - ref['note_dur'].sum()) < 1e-9     # durations tile the clip exactly
        rates.append(_note_agreement(r, ref))
    print(f'{cfg_name}: frame-level note agreement with the reference: {rates}')
    assert min(rates) > 0.85


def test_batched_equals_per_clip(tmp_path):
    """Var-len batching must be exactly equivalent to independent clips (no cross-clip leakage)."""
    ins, config = _plugin('two_head', tmp_path)
    waves = [synth.synth_waveform(300 + i, seconds=s) for i, s in enumerate([1.0, 2.5, 0.2, 3.1])]
    waves.append(np.zeros(0, dtype=np.float32))
    waves.append(synth.edge_case_waveforms()['one_frame'])
    batch = ins.model.infer(waves, return_intermediates=True)
    for w, rb in zip(waves, batch):
        single = ins.model.infer([w], return_intermediates=True)[0]
        np.testing.assert_array_equal(rb['mel'], single['mel'])
        np.testing.assert_array_equal(rb['probs'], single['probs'])
        np.testing.assert_array_equal(rb['bounds'], single['bounds'])
        for k in ('note_midi', 'note_dur', 'note_rest'):
            np.testing.assert_array_equal(rb[k], single[k])


def test_ln_fold_matches_standalone_layernorm(tmp_path):
    """some_forward with norm1..norm4 folded into the GEMMs (SOME_B200_LN_FOLD=1) against the same sequencer with stand-alone
    LayerNorm launches (the product default): same function up to bf16 operand rounding (bf16(x) . W*gamma vs bf16(LN(x)) . W), and the native
    profiler sees the expected launch counts (15 + 12 lay folded, 18 + 16 lay unfolded)."""
    ins, _ = _plugin('two_head', tmp_path)
    eng = ins.model
    frames = [300, 41, 129, 1]
    m, b = sum(frames), len(frames)
    cu_host = np.cumsum([0] + frames)
    cu = torch.tensor(cu_host, dtype=torch.int32, device=eng.device)
    ws = eng.workspace(m)
    torch.manual_seed(0)
    ws.units[:m].copy_(torch.randn(m, 80, device=eng.device) * 3 - 4)
    out, launches = {}, {}
    for fold in (True, False):
        eng.set_ln_fold(fold)
        ws.probs.fill_(float('nan'))
        ws.bounds.fill_(float('nan'))
        eng.start_profile(cu_host)
        eng.run_trunk(ws, m, b, cu, max(frames), 'sigmoid')
        prof = eng.stop_profile()
        launches[fold] = sum(v['launches'] for v in prof.values())
        assert launches[fold] == eng.trunk_launches
        out[fold] = (ws.probs[:m].clone(), ws.bounds[:m].clone())
        assert not torch.isnan(out[fold][0]).any() and not torch.isnan(out[fold][1]).any()
    eng.set_ln_fold(False)                     # the product default
    lay = eng.w.lay
    assert launches[True] == 15 + 12 * lay and launches[False] == 18 + 16 * lay
    # two bf16 evaluations of the same fp32 function: each is within ~2.5e-3 of it (tests/test_gpu_parity_long.py)
    assert float((out[True][0] - out[False][0]).abs().max()) < 6e-3
    assert float((out[True][1] - out[False][1]).abs().max()) < 6e-3


def test_programmatic_dependent_launch_is_bit_identical(tmp_path):
    """some_set_pdl: the trunk kernels launched with the programmatic-serialization attribute (each one may start its prologue
    while its predecessor is still running and blocks in griddepcontrol.wait before touching activations) compute exactly what
    the fully serialised launches compute -- eagerly and when the chunk replays as a CUDA graph (the small-batch path)."""
    ins, _ = _plugin('two_head', tmp_path)
    eng = ins.model
    frames = [300, 41, 129, 1]
    m, b = sum(frames), len(frames)
    cu = torch.tensor(np.cumsum([0] + frames), dtype=torch.int32, device=eng.device)
    ws = eng.workspace(m)
    torch.manual_seed(1)
    ws.units[:m].copy_(torch.randn(m, 80, device=eng.device) * 3 - 4)
    out = {}
    for on in (0, 1):
        ws.probs.fill_(float('nan'))
        ws.bounds.fill_(float('nan'))
        was = eng.lib.some_set_pdl(on)
        try:
            for _ in range(3):                       # back to back: the overlap window is between consecutive kernels
                eng.run_trunk(ws, m, b, cu, max(frames), 'sigmoid')
        finally:
            assert eng.lib.some_set_pdl(was) == on
        torch.cuda.synchronize()
        out[on] = (ws.probs[:m].clone(), ws.bounds[:m].clone())
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    assert not torch.isnan(out[1][0]).any()
    # end to end through the graph-replayed small-chunk path (one ~10 s clip), PDL on (default 'small') vs off
    clip = [synth.synth_waveform(321, seconds=9.0)]
    notes = {}
    for mode in ('off', 'small'):
        eng.pdl = mode
        for _ in range(3):                           # eager, capture, replay
            notes[mode] = ins.infer(clip)
    eng.pdl = 'small'
    for k in ('note_midi', 'note_dur', 'note_rest'):
        np.testing.assert_array_equal(notes['off'][0][k], notes['small'][0][k])


def test_chunked_pipeline_equals_single_chunk(tmp_path):
    """infer() cuts big batches into pipeline chunks (staging / H2D overlap); results must not depend on it."""
    ins, _ = _plugin('two_head', tmp_path)
    waves = [synth.synth_waveform(500 + i, seconds=s) for i, s in enumerate([1.3, 0.7, 2.2, 0.4, 1.9, 1.1, 0.9])]
    whole = ins.infer(waves)
    ins.model.MIN_CHUNK_FRAMES = 64           # force several chunks
    assert len(ins.model._chunks(np.cumsum([0] + [synth.frames_of(len(w)) for w in waves]).astype(np.int32))) >= 2
    chunked = ins.infer(waves)
    for a, b in zip(whole, chunked):
        for k in ('note_midi', 'note_dur', 'note_rest'):
            np.testing.assert_array_equal(a[k], b[k])


def test_pinned_inputs_skip_staging_same_results(tmp_path):
    """Clips handed over in page-locked memory are copied H2D from the caller's buffer (no staging memcpy); mixed
    pinned / pageable batches and chunking must give the same notes as the all-pageable path."""
    from some_b200.engine import pinned_array
    ins, _ = _plugin('two_head', tmp_path)
    waves = [synth.synth_waveform(700 + i, seconds=s) for i, s in enumerate([1.3, 0.7, 2.2, 0.4, 1.9])]
    ref = ins.infer(waves)
    pinned = []
    for w in waves:
        a = pinned_array(len(w))
        a[:] = w
        pinned.append(a)
    assert torch.from_numpy(pinned[0]).is_pinned()
    mixed = [pinned[0], waves[1], pinned[2], waves[3], pinned[4]]
    ins.model.MIN_CHUNK_FRAMES = 64
    for batch in (pinned, mixed):
        got = ins.infer(batch)
        for a, b in zip(ref, got):
            for k in ('note_midi', 'note_dur', 'note_rest'):
                np.testing.assert_array_equal(a[k], b[k])


def test_silence_is_log_clamp(tmp_path):
    ins, _ = _plugin('two_head', tmp_path)
    units = ins.preprocess(np.zeros(44100, dtype=np.float32))['units']
    assert torch.all(units == float(np.log(np.float32(1e-5))))


def test_two_engines_on_two_devices_in_one_process(tmp_path):
    """ADVICE r01 (medium): function attributes (dynamic shared-memory opt-in, carveout) and the SM count are per device; the
    library keeps them per device ordinal, so a second engine on cuda:1 in the same process must work and agree with cuda:0."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two CUDA devices in one process')
    from some_b200 import plugin
    config = synth.named_config('two_head')
    ckpt = synth.write_checkpoint(tmp_path, config, seed=1234)
    waves = [synth.synth_waveform(800 + i, seconds=s) for i, s in enumerate([1.1, 2.3])]
    outs = []
    for dev in ('cuda:0', 'cuda:1'):
        ins = plugin.MIDIExtractionInference(config=config, model_path=ckpt, device=dev)
        outs.append(ins.infer(waves))
    for a, b in zip(*outs):
        for k in ('note_midi', 'note_dur', 'note_rest'):
            np.testing.assert_array_equal(a[k], b[k])

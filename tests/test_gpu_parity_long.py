"""GPU parity AT THE BENCHMARKED SHAPES (VERDICT r01 "weak 1"): a 30 s two_head clip, a 30 s quant clip and a 10 s
midi_conformer (lay 8) clip, each inside a batch large enough to be cut into >= 2 pipeline chunks at the engine's DEFAULT
MIN_CHUNK_FRAMES, compared on every frame with the oracle (which tests/test_oracle_golden.py pins to the unmodified
reference at exactly these lengths) and with the reference's own committed outputs (tests/golden/long_*.npz).

Tolerance: 1e-2 on probabilities / bounds (north_star, bf16 operands).  The decoded notes are a discontinuous function of
those (cumsum().round()): frame-level agreement and exact-boundary agreement with the fp32 reference are reported and
asserted at the measured level."""
import numpy as np
import pytest
import torch

from some_b200 import synth
from oracle.metrics import note_agreement

pytestmark = pytest.mark.gpu

CASES = {   # cfg: (batch clips, min frame agreement, min exact-boundary agreement) — thresholds = measured - margin
    # thresholds sit below the agreement measured with the load-time bias correction on.  With seeded random weights
    # `bounds` hovers around 0.5 on every frame (a boundary every 2-3 frames), the worst case for cumsum().round(): a residual
    # mean error of +-1e-4 (input dependent) is a drift of up to 0.3 over 2584 frames and moves boundaries by one frame.
    # The fp32 validation mode decodes exactly the oracle's notes (tests/test_gpu_accurate.py).
    # Exact-boundary agreement is reported and only floored (it swings 0.30-0.93 between clips for the reason above);
    # the frame-level agreement is the asserted figure.
    'two_head': (14, 0.93, 0.25),
    'quant_two_head': (14, 0.98, 0.25),
    'midi_conformer': (40, 0.91, 0.25),
}


def _plugin(cfg_name, tmp_path):
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    from some_b200 import plugin
    config = synth.named_config(cfg_name)
    ckpt = synth.write_checkpoint(tmp_path, config, seed=1234)
    cls = plugin.QuantizedMIDIExtractionInference if cfg_name.startswith('quant') else plugin.MIDIExtractionInference
    return cls(config=config, model_path=ckpt), config


@pytest.mark.parametrize('cfg_name', list(CASES))
def test_benchmark_shape_matches_oracle_and_reference(cfg_name, tmp_path, golden_dir):
    from oracle import decode as odecode
    n_clips, min_frames, min_bounds = CASES[cfg_name]
    ins, config = _plugin(cfg_name, tmp_path)
    eng = ins.model
    g = np.load(golden_dir / f'long_{cfg_name}.npz')
    secs = float(g['seconds'])
    golden_wave = synth.synth_waveform(int(g['seed']), seconds=secs)
    other = synth.synth_waveform(900, seconds=secs)
    # the golden clip sits in the LAST pipeline chunk, a second checked clip in the first one
    waves = [np.ascontiguousarray(np.roll(other, 911 * i) * np.float32(1 - 0.02 * (i % 5))) for i in range(n_clips - 1)]
    waves.append(golden_wave)
    cu = np.concatenate([[0], np.cumsum([synth.frames_of(len(w)) for w in waves])]).astype(np.int32)
    chunks = eng._chunks(cu)
    assert len(chunks) >= 2, f'batch of {cu[-1]} frames was not cut into pipeline chunks (MIN_CHUNK_FRAMES={eng.MIN_CHUNK_FRAMES})'
    quant = cfg_name.startswith('quant')
    product = ins.infer(waves)                                       # the multi-chunk product path
    single = eng.infer(waves, quantized=quant, return_intermediates=True)   # one chunk, with probs / bounds
    for a, b in zip(product, single):
        for k in ('note_midi', 'note_dur', 'note_rest'):
            np.testing.assert_array_equal(a[k], b[k])                # chunking must not change a single note
    sd = synth.fabricate_state_dict(config, seed=1234)
    report = []
    for idx in (0, n_clips - 1):
        ref = odecode.infer_clip(sd, config, waves[idx], quantized=quant, return_intermediates=True)
        got = single[idx]
        dp = float(np.abs(got['probs'] - ref['probs']).max())
        db = float(np.abs(got['bounds'] - ref['bounds']).max())
        dm = float(np.abs(got['mel'] - ref['mel'].T).max())
        fr, bd = note_agreement(ref, product[idx])
        report.append((idx, dm, dp, db, fr, bd, len(ref['note_midi']), len(product[idx]['note_midi'])))
        print(f'{cfg_name}: clip {idx}: max|mel|={dm:.2e} max|probs|={dp:.2e} max|bounds|={db:.2e} '
              f'mean(bounds err)={float((got["bounds"].astype(np.float64) - ref["bounds"]).mean()):+.2e} '
              f'frame agreement={fr:.4f} exact boundaries={bd:.4f} notes {len(product[idx]["note_midi"])} '
              f'(fp32 oracle {len(ref["note_midi"])})')
        assert dp < 1e-2 and db < 1e-2, (cfg_name, idx, dp, db)      # north_star bf16 tolerance
        assert dm < 1e-3
        assert abs(product[idx]['note_dur'].sum() - ref['note_dur'].sum()) < 1e-9   # durations tile the clip exactly
        assert fr > min_frames and bd > min_bounds, (cfg_name, idx, fr, bd)
    # the reference's own committed outputs for the golden clip
    got = single[-1]
    assert float(np.abs(got['bounds'] - g['bounds']).max()) < 1e-2
    assert float(np.abs(got['probs'][g['rows']] - g['probs_rows']).max()) < 1e-2
    assert float(np.abs(got['probs'].max(1) - g['probs_max']).max()) < 1e-2
    fr, bd = note_agreement({k: g[k] for k in ('note_midi', 'note_dur', 'note_rest')}, product[-1])
    assert fr > min_frames and bd > min_bounds, (cfg_name, 'reference golden', fr, bd)
    print(f'{cfg_name}: vs reference golden: frame agreement={fr:.4f} exact boundaries={bd:.4f}; chunks={chunks}')

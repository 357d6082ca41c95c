"""Pins oracle/ (the CPU restatement) against the golden vectors produced by the unmodified
reference (tests/golden/make_golden.py) and the SURVEY.md §4 known answers.  CPU only."""
import pathlib
import sys

import numpy as np
import pytest
import torch

from oracle import decode as odecode
from oracle import melbank
from oracle import model as omodel
from oracle.metrics import note_agreement
from some_b200 import synth

sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent / 'golden'))
from decode_bins_cases import DEVIATION, THRESHOLD, WIDTHS, make_probe  # noqa: E402


def test_melbank_known_answers(golden_dir):
    w = melbank.mel_filterbank(44100, 2048, 80, 40, 8000)
    assert w.shape == (80, 1025) and w.dtype == np.float32
    assert abs(float(w.sum()) - 3.716216) < 1e-5
    assert abs(float(w.max()) - 0.041265) < 1e-6
    assert int((w != 0).sum()) == 727
    nz = np.nonzero(w.sum(0))[0]
    assert (nz[0], nz[-1]) == (2, 371)
    assert int((w != 0).sum(0).max()) == 2
    ref = np.load(golden_dir / 'mel.npz')['mel_basis']     # buffer of the reference's MelSpectrogram
    assert np.array_equal(w, ref)
    import torchaudio
    ta = torchaudio.functional.melscale_fbanks(1025, 40, 8000, 80, 44100, norm='slaney', mel_scale='htk').T.numpy()
    assert np.abs(w - ta).max() < 2e-7                      # independent implementation


def _assert_log_mel_close(got, ref, key, log_atol, floor):
    """Round-off of an fp32 FFT is absolute: about eps times the frame's energy in every bin, so a band far below the
    frame's largest one can carry a large relative error, and how large depends on the FFT code the CPU runs.  Between
    MKL's AVX-512, AVX2 and SSE4.2 paths the oracle differs from the reference's fp32 bands by up to 3.6e-7 of the
    frame's largest band (and the reference's own bands differ from a float64 STFT by up to 5.5e-3 in the log domain, on
    the quietest bands of a pure tone).  So every band is compared in the linear domain relative to the largest band of
    its frame (2e-6), and in the log domain where it is at least ``floor`` of that band (``log_atol``)."""
    glin, rlin = np.exp(got.astype(np.float64)), np.exp(ref.astype(np.float64))
    scale = rlin.max(axis=0, keepdims=True)                     # [1, T]: the frame's largest band
    lin_err = float((np.abs(glin - rlin) / scale).max()) if ref.size else 0.0
    assert lin_err < 2e-6, (key, lin_err)
    big = rlin >= floor * scale
    log_err = float(np.abs(got - ref)[big].max()) if big.any() else 0.0
    assert log_err < log_atol, (key, log_err)


def test_log_mel_matches_reference(golden_dir):
    g = np.load(golden_dir / 'mel.npz')
    clips = synth.edge_case_waveforms()
    clips['sung3s'] = synth.synth_waveform(101, seconds=3.0)
    for name, w in clips.items():
        ref = g['mel_' + name]
        got = omodel.log_mel(torch.from_numpy(w).unsqueeze(0))[0].numpy()
        assert got.shape == ref.shape == (80, synth.frames_of(len(w))), name
        _assert_log_mel_close(got, ref, name, log_atol=2e-4, floor=1e-2)
    assert np.all(g['mel_zeros'] == np.float32(np.log(np.float32(1e-5))))   # silence -> log(clamp)


def test_decode_known_answers(golden_dir):
    g = np.load(golden_dir / 'decode_kat.npz')
    for b in range(2):
        f2i, vals = g['ex_frame2item'][b], g['ex_values'][b]
        iv, idur, im = odecode.decode_note_sequence(f2i, vals, f2i > 0)
        n = int(f2i.max())
        np.testing.assert_array_equal(iv, g['ex_item_values'][b][:n])
        np.testing.assert_array_equal(idur, g['ex_item_dur'][b][:n])
        np.testing.assert_array_equal(im, g['ex_item_masks'][b][:n])
    # the published expectations themselves (SURVEY.md §4)
    np.testing.assert_array_equal(g['ex_item_values'], [[60.25, 57, 50, 0], [50.25, 53, 47, 38]])
    np.testing.assert_array_equal(g['ex_item_dur'], [[4, 2, 3, 0], [3, 1, 5, 2]])
    np.testing.assert_array_equal(odecode.decode_bounds_to_alignment(g['kat_bounds'][0]), g['kat_frame2item'][0])
    np.testing.assert_array_equal(g['kat_frame2item'][0], [1, 1, 1, 2, 2, 2, 2, 3, 4, 4])
    v, r = odecode.decode_gaussian_blurred_probs(g['kat_probs'][0], 0, 127, 1.0, 0.1)
    np.testing.assert_allclose(v, g['kat_values'][0], rtol=0, atol=1e-5)
    np.testing.assert_array_equal(r, g['kat_rest'][0])


def test_decode_random_matches_reference(golden_dir):
    g = np.load(golden_dir / 'decode_kat.npz')
    gen = torch.Generator().manual_seed(99)
    rb = (torch.rand(4, 700, generator=gen) ** 3).numpy()
    rp = (torch.rand(4, 700, 128, generator=gen) ** 6).numpy()
    assert abs(rb.astype(np.float64).sum() - float(g['rnd_bounds_checksum'])) < 1e-6
    assert abs(rp.astype(np.float64).sum() - float(g['rnd_probs_checksum'])) < 1e-4
    for i in range(4):
        f2i = odecode.decode_bounds_to_alignment(rb[i])
        np.testing.assert_array_equal(f2i, g['rnd_frame2item'][i])
        v, r = odecode.decode_gaussian_blurred_probs(rp[i], 0, 127, 1.0, 0.1)
        # float32 sums of <= 7 terms in a different association order: a few ulp at |v| <= 127
        np.testing.assert_allclose(v, g['rnd_values'][i], rtol=0, atol=1e-4)
        np.testing.assert_array_equal(r, g['rnd_rest'][i])
        # feed the reference's own values so the segmented decode is compared exactly
        nm, nd, nk = odecode.decode_note_sequence(g['rnd_frame2item'][i], g['rnd_values'][i], ~g['rnd_rest'][i])
        np.testing.assert_array_equal(nd, g[f'rnd_note_dur_{i}'])
        np.testing.assert_array_equal(nk, g[f'rnd_note_mask_{i}'])
        np.testing.assert_allclose(nm, g[f'rnd_note_midi_{i}'], rtol=0, atol=1e-4)


@pytest.mark.parametrize('cfg_name', ['two_head', 'quant_two_head', 'midi_conformer'])
def test_plugin_restatement_matches_reference(golden_dir, cfg_name):
    torch.set_num_threads(max(1, torch.get_num_threads()))
    g = np.load(golden_dir / f'plugin_{cfg_name}.npz')
    config = synth.named_config(cfg_name)
    sd = synth.fabricate_state_dict(config, seed=1234)
    secs = float(g['seconds'])
    waves = [synth.synth_waveform(int(s), seconds=secs + 0.37 * i) for i, s in enumerate(g['seeds'])]
    if cfg_name == 'two_head':
        waves += [synth.edge_case_waveforms()['ragged'], synth.edge_case_waveforms()['short']]
    quant = cfg_name.startswith('quant')
    for i, w in enumerate(waves):
        assert len(w) == int(g[f'clip{i}_num_samples'])
        out = odecode.infer_clip(sd, config, w, quantized=quant, return_intermediates=True)
        np.testing.assert_allclose(out['probs'], g[f'clip{i}_probs'], rtol=0, atol=2e-5)
        np.testing.assert_allclose(out['bounds'], g[f'clip{i}_bounds'], rtol=0, atol=2e-5)
        # decode restated on the reference's exact probabilities must agree exactly
        probs, bounds = g[f'clip{i}_probs'], g[f'clip{i}_bounds']
        f2i = odecode.decode_bounds_to_alignment(bounds)
        if quant:
            midi = probs.argmax(-1).astype(np.int64)
            vals, rest = np.clip(midi, 0, 127), midi == 128
        else:
            vals, rest = odecode.decode_gaussian_blurred_probs(probs, 0, 127, 1.0, 0.1)
        nm, nd, nk = odecode.decode_note_sequence(f2i, vals, ~rest)
        assert nm.dtype == g[f'clip{i}_note_midi'].dtype == np.float32
        np.testing.assert_array_equal(nd * (512 / 44100), g[f'clip{i}_note_dur'])
        np.testing.assert_array_equal(~nk, g[f'clip{i}_note_rest'])
        np.testing.assert_allclose(nm, g[f'clip{i}_note_midi'], rtol=0, atol=1e-4)


# --------------------------------------------------------------------------- the benchmarked shapes (round 2)
@pytest.mark.parametrize('cfg_name', ['two_head', 'quant_two_head', 'midi_conformer'])
def test_oracle_matches_reference_at_benchmark_lengths(golden_dir, cfg_name):
    """30 s two_head / quant clips (T = 2584) and a 10 s lay-8 clip: the oracle against outputs of the unmodified reference
    (tests/golden/make_golden_long.py).  fp32 vs fp32, different thread counts / reduction orders: 2e-5 like the short
    clips; the decoded notes must be the reference's."""
    g = np.load(golden_dir / f'long_{cfg_name}.npz')
    config = synth.named_config(cfg_name)
    sd = synth.fabricate_state_dict(config, seed=1234)
    w = synth.synth_waveform(int(g['seed']), seconds=float(g['seconds']))
    assert len(w) == int(g['num_samples'])
    quant = cfg_name.startswith('quant')
    out = odecode.infer_clip(sd, config, w, quantized=quant, return_intermediates=True)
    assert out['probs'].shape[0] == synth.frames_of(len(w)) == g['bounds'].shape[0]
    np.testing.assert_allclose(out['bounds'], g['bounds'], rtol=0, atol=5e-5)
    np.testing.assert_allclose(out['probs'][g['rows']], g['probs_rows'], rtol=0, atol=5e-5)
    np.testing.assert_allclose(out['probs'].max(1), g['probs_max'], rtol=0, atol=5e-5)
    ref = {k: g[k] for k in ('note_midi', 'note_dur', 'note_rest')}
    frames, bounds = note_agreement(ref, out)
    # cumsum().round() is discontinuous: a 1e-5 difference can move a boundary that sits on a rounding edge
    assert frames > 0.995 and bounds > 0.995, (frames, bounds)
    # decode restated on the reference's exact bounds must give the reference's note durations
    f2i = odecode.decode_bounds_to_alignment(g['bounds'])
    assert int(f2i.max()) == len(g['note_dur'])
    np.testing.assert_array_equal(np.bincount(f2i)[1:] * (512 / 44100), g['note_dur'])


def test_vectorised_decode_equals_loops():
    """bench.py times the vectorised decode forms; they must be the loop specification, bit for bit."""
    gen = torch.Generator().manual_seed(5)
    for t in (1, 37, 700, 2584):
        probs = (torch.rand(t, 128, generator=gen) ** 6).numpy()
        bounds = (torch.rand(t, generator=gen) ** 3).numpy()
        v0, r0 = odecode.decode_gaussian_blurred_probs(probs, 0, 127, 1.0, 0.1)
        v1, r1 = odecode.decode_gaussian_blurred_probs_vec(probs, 0, 127, 1.0, 0.1)
        np.testing.assert_array_equal(v0, v1)
        np.testing.assert_array_equal(r0, r1)
        f2i = odecode.decode_bounds_to_alignment(bounds)
        for vals in (v0, np.clip(probs.argmax(1), 0, 127).astype(np.int64)):
            a = odecode.decode_note_sequence(f2i, vals, ~r0)
            b = odecode.decode_note_sequence_vec(f2i, vals, ~r0)
            for x, y in zip(a, b):
                assert x.dtype == y.dtype
                np.testing.assert_array_equal(x, y)


@pytest.mark.parametrize('n,vmin,vmax', WIDTHS)
def test_decode_head_widths_match_reference_exactly(golden_dir, n, vmin, vmax):
    """Head widths other than 128 (tests/golden/make_golden_decode_bins.py): the bin values are float32 arithmetic in the
    reference, so on probes whose sums do not depend on their order the oracle must give the reference's bits."""
    g = np.load(golden_dir / 'decode_bins.npz')
    key = f'n{n}_{vmin}_{vmax}'
    probs, bounds = make_probe(n, vmin, vmax)
    assert probs.astype(np.float64).sum() == g[f'{key}_probs_checksum']
    f2i = odecode.decode_bounds_to_alignment(bounds)
    np.testing.assert_array_equal(f2i, g[f'{key}_frame2item'])
    for blur, notes in ((odecode.decode_gaussian_blurred_probs, odecode.decode_note_sequence),
                        (odecode.decode_gaussian_blurred_probs_vec, odecode.decode_note_sequence_vec)):
        v, r = blur(probs, vmin, vmax, DEVIATION, THRESHOLD)
        np.testing.assert_array_equal(v, g[f'{key}_values'])
        np.testing.assert_array_equal(r, g[f'{key}_rest'])
        nm, nd, nk = notes(f2i, v, ~r)
        np.testing.assert_array_equal(nm, g[f'{key}_note_midi'])
        np.testing.assert_array_equal(nd, g[f'{key}_note_dur'])
        np.testing.assert_array_equal(nk, g[f'{key}_note_mask'])
    # the probes reach what they are for: every bin value, rests, notes with and without valid frames
    one_hot = (probs == 1.0).sum(1) == (probs != 0).sum(1)
    assert set(probs[one_hot].argmax(1)) == set(range(n))
    assert g[f'{key}_rest'].any() and (~g[f'{key}_note_mask']).any() and g[f'{key}_note_mask'].any()


def test_quantised_decode_matches_reference(golden_dir):
    """inference/me_quant_infer.py:21-38 on random 129-bin probabilities: the oracle's quantised decode against the
    reference's own postprocess outputs (decode_quant_kat.npz), exactly."""
    g = np.load(golden_dir / 'decode_quant_kat.npz')
    gen = torch.Generator().manual_seed(77)
    for i, t in enumerate((700, 700, 1, 37)):
        logits = torch.randn(1, t, 129, generator=gen) * 2.0
        logits[..., 128] += 1.0
        probs = torch.softmax(logits, dim=-1)
        bounds = torch.rand(1, t, generator=gen) ** 3
        assert abs(probs.double().sum().item() + bounds.double().sum().item() - float(g[f'q{i}_checksum'])) < 1e-6
        midi = probs[0].numpy().argmax(-1).astype(np.int64)
        f2i = odecode.decode_bounds_to_alignment(bounds[0].numpy())
        for fn in (odecode.decode_note_sequence, odecode.decode_note_sequence_vec):
            nm, nd, nk = fn(f2i, np.clip(midi, 0, 127), midi != 128)
            np.testing.assert_array_equal(nm, g[f'q{i}_note_midi'])
            np.testing.assert_array_equal(nd * (512 / 44100), g[f'q{i}_note_dur'])
            np.testing.assert_array_equal(~nk, g[f'q{i}_note_rest'])


def test_oracle_keyshift_mel_matches_reference(golden_dir):
    """oracle.model.log_mel with keyshift / speed / center (modules/rmvpe/spec.py:39-46,63-68) against the unmodified
    reference MelSpectrogram (tests/golden/make_golden_keyshift.py)."""
    import torch
    from oracle import model as omodel
    from some_b200 import synth
    g = np.load(golden_dir / 'keyshift.npz')
    audio = torch.from_numpy(synth.synth_waveform(int(g['seed']), seconds=float(g['seconds']))).unsqueeze(0)
    cases = [(f'ks_{k}', dict(keyshift=k)) for k in range(-5, 6)]
    cases += [('ks_frac_2.37', dict(keyshift=2.37)), ('speed_1.25', dict(speed=1.25)), ('nocenter_ks3', dict(keyshift=3, center=False))]
    for key, kw in cases:
        got = omodel.log_mel(audio, fmin=40, fmax=8000, **kw)[0].numpy()
        assert got.shape == g[key].shape, key
        _assert_log_mel_close(got, g[key], key, log_atol=2e-5, floor=0.1)   # same torch.stft: round-off only

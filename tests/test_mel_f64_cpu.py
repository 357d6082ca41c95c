"""The float64 log-mel of tests/golden/mel_f64.py and the error bounds it gives the mel kernels (csrc/mel.cu), without a GPU:

* mel64 agrees with the unmodified reference's fp32 outputs (mel.npz, keyshift.npz, keyshift_wide.npz) at an fp32 FFT's level;
* the key-shift bound, a probabilistic one, holds for a numpy emulation of the direct-DFT kernel's arithmetic at n' = 4096;
* the bounds have power: each planted defect of the STFT (a frame one sample off, the symmetric window, a shifted pad,
  a neighbour's samples in the padding, the filterbank one bin off, the magnitude scale dropped, n' rounded down) moves
  the result by more than twice the bound, so a kernel with that defect fails the GPU tests (tests/test_gpu_mel_f64.py);
  tables of reduced precision (an fp16 window or twiddle table) fail the bound on impulses in the register FFT, and move
  the sung-note signal's log-mel by far more than the key-shift test's every-band tolerance."""
import pathlib
import subprocess
import sys

import numpy as np
import pytest

HERE = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / 'golden'))

from mel_f64 import (BASIS, C_FFT, CLAMP, SR, SUNG_LOG_TOL, WIDE_CASES, bound_ratios, c_dft, fft_signals,  # noqa: E402
                     hann32, loud_over_quiet, mel64, shift_lengths, wide_signals)
from oracle import refshim  # noqa: E402
from some_b200 import synth  # noqa: E402

GOLDEN = HERE / 'golden'
REF_LOG_TOL = 5e-4   # the reference's fp32 torch.stft against float64, where a band is far above its round-off


def check_reference(name, golden_t80, ref):
    """the reference's fp32 log-mel against mel64: within an fp32 FFT's bound (the register FFT's C_FFT) in both domains,
    and within REF_LOG_TOL in the log wherever the band is 1000 x above that bound"""
    lin, log, err = bound_ratios(golden_t80, ref, C_FFT)
    assert lin <= 1.0 and log <= 1.0, (name, lin, log)
    assert err <= REF_LOG_TOL, (name, err)


def test_reference_matches_mel_golden():
    g = np.load(GOLDEN / 'mel.npz')
    assert np.array_equal(g['mel_basis'].astype(np.float64), BASIS)
    clips = synth.edge_case_waveforms()
    clips['sung3s'] = synth.synth_waveform(101, seconds=3.0)
    for name, w in clips.items():
        check_reference(name, g['mel_' + name].T, mel64(w))


def test_reference_matches_keyshift_golden():
    g = np.load(GOLDEN / 'keyshift.npz')
    audio = synth.synth_waveform(int(g['seed']), seconds=float(g['seconds']))
    cases = [(f'ks_{k}', dict(keyshift=k)) for k in range(-5, 6)]
    cases += [('ks_frac_2.37', dict(keyshift=2.37)), ('speed_1.25', dict(speed=1.25)),
              ('nocenter_ks3', dict(keyshift=3, center=False))]
    for key, kw in cases:
        check_reference(key, g[key].T, mel64(audio, **kw))


def test_reference_matches_keyshift_wide_golden():
    g = np.load(GOLDEN / 'keyshift_wide.npz')
    sigs = wide_signals()
    assert float(g['seconds']) * SR == len(sigs['sung'])
    for sig, wave in sigs.items():
        for key, kw in WIDE_CASES:
            ref = mel64(wave, **kw)
            check_reference(f'{sig}/{key}', g[f'{sig}/{key}'].T, ref)
            if sig == 'sung':   # no band of the sung signal is near the fp32 round-off: every band is within 2e-4
                err = float(np.abs(g[f'{sig}/{key}'].T - ref.log).max())
                assert err <= SUNG_LOG_TOL / 5, (key, err)
    check_reference('shortest_ks12', g['shortest_ks12'].T, mel64(loud_over_quiet(4096), keyshift=12, center=False))
    with pytest.raises(RuntimeError):   # one sample shorter: torch.stft refuses it, and so does the restatement
        mel64(loud_over_quiet(4095), keyshift=12, center=False)


@pytest.mark.skipif(not refshim.reference_available(), reason='needs the reference source tree')
def test_keyshift_wide_golden_regenerates(tmp_path):
    """make_golden_keyshift_wide.py reproduces the committed archive byte for byte.  It runs in a process of its own:
    loading the reference replaces modules and installs import stubs, which must not leak into this session."""
    out = tmp_path / 'k.npz'
    subprocess.run([sys.executable, str(GOLDEN / 'make_golden_keyshift_wide.py'), str(out)], check=True,
                   cwd=HERE.parent, stdout=subprocess.DEVNULL)
    assert out.read_bytes() == (GOLDEN / 'keyshift_wide.npz').read_bytes()


# ------------------------------------------------------------------------------------ the key-shift kernel's arithmetic
def emulate_dft_kernel(audio, keyshift, frames):
    """some_mel_logmel_keyshift's arithmetic in numpy for the given frames (center=True, speed 1): fp32 v = x w, one
    sequential fmaf chain per bin over all n' samples with the fp32 twiddle table exp(-2 pi i (k n mod n') / n') (fmaf
    approximated as the float64 sum of the exact product, rounded to fp32), |X| scaled by 2048 / n', bins the shorter FFT
    lacks zero, the filterbank as an fmaf chain over each filter's bins, logf(max(., clamp)).  [len(frames), 80]"""
    n_fft, win, hop = shift_lengths(keyshift)
    pl = win // 2
    ang = -2.0 * np.pi * np.arange(n_fft) / n_fft
    twr, twi = np.cos(ang).astype(np.float32).astype(np.float64), np.sin(ang).astype(np.float32).astype(np.float64)
    w = hann32(win).astype(np.float32)
    x = np.asarray(audio, dtype=np.float32)
    xp = np.concatenate([np.zeros(pl, np.float32), x, np.zeros(n_fft, np.float32)])
    xs = np.stack([xp[f * hop:f * hop + n_fft] for f in frames])          # [F, n']
    v = (xs * w[None, :]).astype(np.float32).astype(np.float64)          # rounded products
    k = np.arange(372)
    re = np.zeros((len(frames), 372), np.float64)
    im = np.zeros((len(frames), 372), np.float64)
    for j in range(n_fft):
        idx = (k * j) % n_fft
        re = (v[:, j:j + 1] * twr[idx][None] + re).astype(np.float32).astype(np.float64)
        im = (v[:, j:j + 1] * twi[idx][None] + im).astype(np.float32).astype(np.float64)
    re, im = re.astype(np.float32), im.astype(np.float32)
    mag = (np.sqrt(re * re + im * im) * np.float32(2048 / win)).astype(np.float32)
    mag[:, k >= n_fft // 2 + 1] = 0
    b32 = BASIS.astype(np.float32)
    acc = np.zeros((len(frames), 80), np.float32)
    for m in range(80):
        for b in np.nonzero(b32[m])[0]:
            acc[:, m] = (np.float64(b32[m, b]) * mag[:, b].astype(np.float64) + acc[:, m]).astype(np.float32)
    return np.log(np.maximum(acc, np.float32(CLAMP))).astype(np.float32)


@pytest.mark.parametrize('keyshift', [12, -12])
def test_dft_bound_holds_for_emulated_kernel(keyshift):
    """the probabilistic key-shift bound c_dft(n') holds for the emulated chain at n' = 4096 and 1024, on the signal
    with the widest dynamic range (a full-scale tone over -100 dB noise) and on the sung-note signal"""
    for name, wave in wide_signals().items():
        ref = mel64(wave, keyshift=keyshift)
        frames = list(range(0, ref.log.shape[0], 3))
        got = emulate_dft_kernel(wave, keyshift, frames)
        sub = type(ref)(ref.log[frames], ref.lin[frames], ref.S[frames], ref.scale, ref.n_fft)
        lin, log, err = bound_ratios(got, sub, c_dft(ref.n_fft))
        print(f'emulated direct DFT, {name} at {keyshift:+d} (n\' = {ref.n_fft}): error / bound {max(lin, log):.3f}, '
              f'largest log error where compared {err:.2e}')
        assert lin <= 1.0 and log <= 1.0, (name, keyshift, lin, log)


# ------------------------------------------------------------------------------------------------------- test power
NEIGHBOUR = np.random.default_rng(1).standard_normal(4096)
DEFECTS = {
    'frame start one sample late': (0, dict(start_shift=1)),
    'symmetric Hann window': (0, dict(periodic=False)),
    'left pad one sample longer': (0, dict(pad_left_delta=1)),
    'left pad one sample longer at +12': (12, dict(pad_left_delta=1)),
    'edge frame reads the previous clip': (0, dict(left_neighbour=NEIGHBOUR)),
    'filterbank reads bin k + 1': (0, dict(bin_offset=1)),
    'magnitude scale 2048 / win\' dropped at +12': (12, dict(drop_scale=True)),
    'magnitude scale 2048 / win\' dropped at -12': (-12, dict(drop_scale=True)),
    'n_fft\' rounded down at 11.99': (11.99, dict(rounding=np.floor)),
    'n_fft\' rounded down at -11.9': (-11.9, dict(rounding=np.floor)),
}


@pytest.mark.parametrize('defect', list(DEFECTS))
def test_planted_defect_breaks_the_bound(defect):
    """a kernel with the defect computes (the defective STFT) + (its rounding, <= tau); it is caught when the defect alone
    moves some band by more than 2 tau.  Required on each of three signals, of different kinds"""
    keyshift, kw = DEFECTS[defect]
    n = 8 * 512 + 1
    sigs = fft_signals(n)
    sigs = {'sung': wide_signals()['sung'][:n], 'loud_over_quiet': sigs['loud_over_quiet'], 'impulses': sigs['impulses']}
    for name, x in sigs.items():
        clean = mel64(x, keyshift=keyshift)
        bad = mel64(x, keyshift=keyshift, **kw)
        c = C_FFT if keyshift == 0 else c_dft(clean.n_fft)
        lin, log, _ = bound_ratios(bad.log, clean, 2.0 * c)
        assert max(lin, log) > 1.0, (defect, name, lin, log)


@pytest.mark.parametrize('table', ['window', 'twiddle'])
def test_fp16_table_is_caught(table):
    """an fp16 window or twiddle table: at keyshift 0 it breaks twice the register-FFT bound on the impulses signal, which
    the register-FFT test runs at every clip length; at +-12 it stays inside the key-shift bound (whose slack is in
    |s_j| <= S_t) but moves some band of the sung-note signal by more than twice SUNG_LOG_TOL, the tolerance the key-shift
    test holds every band of that signal to"""
    kw = {f'{table}_dtype': np.float16}
    x = fft_signals(8 * 512 + 1)['impulses']
    clean = mel64(x)
    lin, log, _ = bound_ratios(mel64(x, **kw).log, clean, 2.0 * C_FFT)
    assert max(lin, log) > 1.0, (table, lin, log)
    sung = wide_signals()['sung']
    for keyshift in (12, -12):
        moved = float(np.abs(mel64(sung, keyshift=keyshift, **kw).log - mel64(sung, keyshift=keyshift).log).max())
        assert moved > 2.0 * SUNG_LOG_TOL, (table, keyshift, moved)

"""Float64 restatement of the reference log-mel (modules/rmvpe/spec.py:38-72) and the error bounds the two fp32 mel kernels
of csrc/mel.cu are held to, plus the test signals.  Used by tests/test_mel_f64_cpu.py, tests/test_gpu_mel_f64.py and
make_golden_keyshift_wide.py.  It runs on the CPU: numpy for the arithmetic, torch only for the reference's fp32 Hann
window and some_b200.synth for the sung-note signal, so it imports and runs without a GPU.

mel64 takes the reference's two fp32 parameter tensors as they are, promoted to float64: the mel basis (tests/golden/mel.npz)
and the periodic Hann window of torch.hann_window(win', float32).  The window matters: fp32 rounding of 1 - cos(2 pi n / N)
puts a 1 % relative error on w[1], and the kernels use the reference's fp32 window, not an exact one.  Every operation after
those parameters is float64.

Error bound.  Every |X_k| of frame t is at most S_t = sum_n |x_n w_n|, and every partial sum an FFT or DFT forms of that frame
is a sum of a subset of the x_n w_n times unit-modulus twiddles, so it is at most S_t too.  A rounding in a stage of an
FFT is relative to the value it rounds; the values of one stage that reach an output bin are partial DFTs over disjoint
subsets of the samples, so their moduli add up to at most S_t and each stage contributes at most (its constant) u S_t to
every bin (u = 2^-24, round to nearest).  The filterbank multiplies each bin's error by W[m, b] >= 0, so band m of frame t
is off by at most

    tau[t, m] = c * 2^-24 * S_t * scale * sum_b W[m, b]

(scale = 2048 / win' on the key-shift path, 1 otherwise).  c per kernel is derived below, to first order in u."""
from __future__ import annotations

import pathlib
from dataclasses import dataclass

import numpy as np

HERE = pathlib.Path(__file__).resolve().parent
SR, N_FFT, HOP, N_MELS, CLAMP = 44100, 2048, 512, 80, 1e-5
MEL_BINS = 372   # bins 0..371 carry every non-zero weight of the basis (some_b200.weights.mel_tables checks it)
U = 2.0 ** -24
# every band of the sung-note signal against the reference's fp32 output or float64: the reference's own torch.stft is
# within 2e-4 of float64 there, the key-shift kernel's n'-term chains within 3e-4 on an H100
SUNG_LOG_TOL = 1e-3
BASIS = np.load(HERE / 'mel.npz')['mel_basis'].astype(np.float64)   # [80, 1025], the reference's fp32 basis
W_SUM = BASIS.sum(axis=1)                                           # [80]

# Register FFT (some_mel_logmel), per bin, in units of u S_t.  A complex add or subtract rounds each component: u |result|.
# A twiddle multiply re = fma(x, wr, -(y wi)), im = fma(y, wr, x wi) (or the compiler's contraction of x wr - y wi) is
# off by at most 2 sqrt2 u |d| per component, 4 u |d| in modulus, plus u |d| for the fp32 twiddle table: 5 u |d|.
#   window product x w (rounded, not fused)                              1
#   one 32-point pass: 5 radix-2 stages x (subtract 1 + twiddle 5)      30
#   inter-pass twiddle W_1024^(n2 k1)                                     5
#   second 32-point pass                                                 30
#   -> 66 per complex bin Z_k of the 1024-point transform of z_n = x_2n w_2n + i x_2n+1 w_2n+1, sum |z_n| <= S_t.
#   The real-FFT unpack X_k = (Z_k + conj Z_N-k) / 2 - i W_2048^k (Z_k - conj Z_N-k) / 2 takes each of Z_k, Z_N-k with a
#   coefficient of modulus <= 1:                                       2 x 66 = 132
#   its own roundings: E 1, O 1, W O 5, E + W O 1 (|E|, |O| <= S_t)       8
#   |X| = sqrtf(re^2 + im^2): the sum of squares 2 u relative, halved by the root, plus the root's own rounding  2
#   filterbank: an fmaf chain of <= 24 non-negative terms, gamma_24 on sum_b W |X_b| <= S_t sum_b W    24
C_FFT = 1 + 132 + 8 + 2 + 24   # = 167


# Direct DFT (some_mel_logmel_keyshift): bin k is one sequential chain acc = fmaf(v_j, tw_j, acc) over all n' samples
# (re and im separately).  Worst case that is gamma_n' = n' u: 4096 at n' = 4096, a vacuous bound.  Instead the standard
# probabilistic model (Higham & Mary, SIAM J. Sci. Comput. 41(5), 2019): the roundings delta_j of the chain are independent,
# mean zero and |delta_j| <= u, so by Hoeffding's inequality the chain's error sum_j delta_j s_j (s_j the partial sums,
# |s_j| <= S_t) exceeds lam u sqrt(sum_j s_j^2) <= lam u sqrt(n') S_t with probability at most 2 exp(-lam^2 / 2).  lam = 6
# puts that at 3e-8 per chain, below one expected failure in all the chains (2 per bin, 372 bins, every frame) the tests run.
# re and im together: sqrt2 lam u sqrt(n') S_t.  The rest, in units of u S_t:
#   window product v = x w 1, fp32 twiddle table sqrt2 -> 2, |X| 2, the fp32 scale 2048 / win' and its product 2,
#   filterbank chain <= 24 terms 24                                                                          30
# Checked against a numpy emulation of the chain's arithmetic at n' = 4096 and 1024 on a loud tone over quiet noise and on
# a sung-note signal (tests/test_mel_f64_cpu.py::test_dft_bound_holds_for_emulated_kernel): the emulation reaches 2 % of
# the bound, the kernel on an H100 under 5 %.  The slack is in |s_j| <= S_t, which is not tightened: the partial sums of
# the bin a strong component sits in (DC in bin 0, a tone on a bin centre) do grow to S_t.
LAM = 6.0


def c_dft(n_fft: int) -> float:
    return np.sqrt(2.0) * LAM * np.sqrt(n_fft) + 30.0


def shift_lengths(keyshift=0, speed=1, rounding=np.round):
    """(n_fft', win', hop') of spec.py:39-42"""
    factor = 2 ** (keyshift / 12)
    return int(rounding(N_FFT * factor)), int(rounding(N_FFT * factor)), int(np.round(HOP * speed))


def hann32(n: int, periodic: bool = True) -> np.ndarray:
    """torch.hann_window(n, float32) (spec.py:45), the reference's fp32 values promoted to float64"""
    import torch
    return torch.hann_window(n, periodic=periodic, dtype=torch.float32).double().numpy()


@dataclass
class Mel64:
    log: np.ndarray     # [T, 80] log(max(mel, clamp))
    lin: np.ndarray     # [T, 80] mel before the clamp
    S: np.ndarray       # [T] sum_n |x_n w_n| of each frame
    scale: float        # the magnitude scale 2048 / win' (1 without a key shift)
    n_fft: int

    def tau(self, c: float) -> np.ndarray:
        """the linear-domain bound c 2^-24 S_t scale sum_b W[m, b], [T, 80]"""
        return c * U * self.S[:, None] * self.scale * W_SUM[None, :]


def mel64(audio, keyshift=0, speed=1, center=True, *, start_shift=0, periodic=True, pad_left_delta=0, left_neighbour=None,
          bin_offset=0, drop_scale=False, rounding=np.round, window_dtype=None, twiddle_dtype=None) -> Mel64:
    """spec.py:38-72 in float64 for one clip.  The keyword-only arguments plant a defect (the sensitivity tests use them):
    start_shift moves every frame's start by that many samples, periodic=False takes the symmetric Hann window,
    pad_left_delta moves the left zero pad (the right one keeps the total), left_neighbour fills the left pad with those
    samples instead of zeros, bin_offset makes the filterbank read bin k + offset, drop_scale leaves out the 2048 / win'
    of spec.py:68, rounding replaces np.round in the n_fft' of spec.py:40, window_dtype rounds the window to that type and
    twiddle_dtype takes the bins the filterbank reads as a direct DFT with exp(-2 pi i m / n') rounded to that type."""
    x = np.asarray(audio, dtype=np.float64)
    n_fft, win, hop = shift_lengths(keyshift, speed, rounding)
    pl, pr = (win // 2, (win + 1) // 2) if center else (0, 0)
    pl, pr = pl + pad_left_delta, pr - pad_left_delta
    left = np.zeros(pl)
    if left_neighbour is not None and pl > 0:
        nb = np.asarray(left_neighbour, dtype=np.float64)[-pl:]
        left[pl - len(nb):] = nb
    xp = np.concatenate([left, x, np.zeros(pr)])
    if len(xp) < n_fft:
        raise RuntimeError(f'{len(x)} samples are shorter than one window of {n_fft}')   # torch.stft refuses these
    t = 1 + (len(xp) - n_fft) // hop
    assert start_shift >= 0
    xp = np.concatenate([xp, np.zeros(start_shift)])
    frames = xp[(np.arange(t) * hop + start_shift)[:, None] + np.arange(n_fft)[None, :]]   # [T, n_fft]
    window = hann32(win, periodic)
    if window_dtype is not None:
        window = window.astype(window_dtype).astype(np.float64)
    xw = frames * window[None, :]
    mag = np.abs(np.fft.rfft(xw, axis=1))                                       # [T, n_fft // 2 + 1]
    if twiddle_dtype is not None:
        kb = min(MEL_BINS, mag.shape[1])
        ang = -2.0 * np.pi * ((np.arange(n_fft)[:, None] * np.arange(kb)[None, :]) % n_fft) / n_fft
        rnd = lambda a: a.astype(twiddle_dtype).astype(np.float64)   # noqa: E731
        mag[:, :kb] = np.abs(xw @ (rnd(np.cos(ang)) + 1j * rnd(np.sin(ang))))
    scale = 1.0
    if keyshift != 0:
        size = N_FFT // 2 + 1
        if mag.shape[1] < size:
            mag = np.pad(mag, ((0, 0), (0, size - mag.shape[1])))
        mag = mag[:, :size]
        scale = 1.0 if drop_scale else N_FFT / win
        mag = mag * scale
    if bin_offset:
        mag = np.concatenate([mag[:, bin_offset:], np.zeros((t, bin_offset))], axis=1)
    lin = mag @ BASIS.T
    return Mel64(np.log(np.maximum(lin, CLAMP)), lin, np.abs(xw).sum(axis=1), N_FFT / win if keyshift != 0 else 1.0, n_fft)


def log_rounding(v: np.ndarray) -> np.ndarray:
    """absolute error of an fp32 logf(v) result: logf's 1 ulp plus the rounding of the stored value, 2 ulp of |log v|"""
    return 2.0 * np.spacing(np.abs(np.log(v)).astype(np.float32)).astype(np.float64)


def bound_ratios(got_log, ref: Mel64, c: float):
    """Largest error / bound of fp32 log-mel `got_log` [T, 80] against ref:
    linear: |exp(got) - max(mel64, clamp)| <= tau + max(mel64, clamp) * (the log's own rounding);
    log:    |got - log mel64| <= tau / mel64 + (the log's rounding), only where mel64 >= 1000 tau.
    Returns (linear ratio, log ratio, largest log error where the log comparison applies)."""
    g = np.asarray(got_log, dtype=np.float64)
    assert g.shape == ref.log.shape, (g.shape, ref.log.shape)
    tau = ref.tau(c)
    want = np.maximum(ref.lin, CLAMP)
    lin_ratio = float((np.abs(np.exp(g) - want) / (tau + want * log_rounding(want))).max())
    big = (ref.lin >= 1000.0 * tau) & (ref.lin > 0)
    if not big.any():
        return lin_ratio, 0.0, 0.0
    err = np.abs(g - np.log(want))[big]
    log_ratio = float((err / (tau[big] / ref.lin[big] + log_rounding(want[big]))).max())
    return lin_ratio, log_ratio, float(err.max())


# ------------------------------------------------------------------------------------------------ test signals
def loud_over_quiet(n: int, seed: int = 3) -> np.ndarray:
    """a full-scale 1 kHz tone over white noise at -100 dBFS: quiet bands next to a loud one"""
    t = np.arange(n) / SR
    rng = np.random.default_rng(seed)
    return (0.99 * np.sin(2 * np.pi * 1000.3 * t) + 1e-5 * rng.standard_normal(n)).astype(np.float32)


def impulses(n: int) -> np.ndarray:
    """unit impulses at the first and last sample and at +-1 of frame window edges (frame f reads [512 f - 1024,
    512 f + 1024)): each of those samples sits where the window is 0, tiny, or the zero padding starts"""
    x = np.zeros(n, dtype=np.float32)
    for i in (0, n - 1, 511, 513, 1535, 1537, 4095, 4096 + 1023, 4096 + 1025):
        if 0 <= i < n:
            x[i] = 1.0
    return x


def fft_signals(n: int) -> dict:
    """the register-FFT test signals of one clip length"""
    t = np.arange(n) / SR
    rng = np.random.default_rng(n)
    tone = lambda f: np.sin(2 * np.pi * f * t + 0.3).astype(np.float32)   # noqa: E731
    return {
        'silence': np.zeros(n, dtype=np.float32),
        'dc': np.full(n, 0.5, dtype=np.float32),
        'square': np.where(np.sin(2 * np.pi * 441.0 * t + 0.1) >= 0, 1.0, -1.0).astype(np.float32),
        'tone_bin': tone(100 * SR / N_FFT),
        'tone_half_bin': tone(100.5 * SR / N_FFT),
        'tone_40hz': tone(40.0),
        'tone_8khz': tone(8000.0),
        'loud_over_quiet': loud_over_quiet(n),
        'impulses': impulses(n),
        'noise_1e-4': (1e-4 * rng.standard_normal(n)).astype(np.float32),
        'noise_1': np.clip(rng.standard_normal(n), -1, 1).astype(np.float32),
    }


# key-shift golden (make_golden_keyshift_wide.py): cases as (name, kwargs of forward)
WIDE_SECONDS = 0.5
WIDE_CASES = ([(f'ks_{k}', dict(keyshift=k)) for k in list(range(-12, -5)) + list(range(6, 13))]
              + [(f'ks_frac_{k}', dict(keyshift=k)) for k in (-0.5, 0.5, 7.3, -11.9, 11.99)]
              + [('nocenter_ks12', dict(keyshift=12, center=False)), ('nocenter_ks-12', dict(keyshift=-12, center=False)),
                 ('speed_0.8_ks12', dict(keyshift=12, speed=0.8)), ('speed_2.0_ks12', dict(keyshift=12, speed=2.0))])


def wide_signals() -> dict:
    """the two signals of keyshift_wide.npz: the sung-note signal of keyshift.npz (seed 4242) and a loud tone over quiet"""
    from some_b200 import synth
    n = int(round(WIDE_SECONDS * SR))
    return {'sung': synth.synth_waveform(4242, num_samples=n), 'loud': loud_over_quiet(n)}

"""Both log-mel kernels of csrc/mel.cu against the float64 restatement of the reference (tests/golden/mel_f64.py), held to
error bounds derived from each kernel's arithmetic:

* the register FFT (some_mel_logmel, through the C ABI) on clip lengths on and around the zero-padded edges, the 8-frame
  warp and 64-frame CTA tiles and a 30 s clip, packed var-len once 16-byte aligned (interior frames load straight from the
  waveform) and once at odd float offsets (every frame is staged), with NaN between the clips; silence, DC, a full-scale
  square wave, tones on and between bins and at the basis edges, a loud tone over -100 dB noise, impulses at the clip and
  frame edges and white noise;
* the key-shift direct DFT (some_mel_logmel_keyshift, through some_b200.spec.MelSpectrogram) across the shipped configs'
  key_shift_range [-12, 12], fractional shifts, speed and center=False, against tests/golden/keyshift_wide.npz and float64,
  at frame counts around its 8-frame tile, n' below 742 (bins past n' / 2 are zero) and its refusals.

Each test prints its largest error / bound per case group."""
import ctypes as C
import pathlib
import sys

import numpy as np
import pytest
import torch

HERE = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / 'golden'))

from mel_f64 import (BASIS, C_FFT, CLAMP, HOP, SR, SUNG_LOG_TOL, WIDE_CASES, bound_ratios, c_dft,  # noqa: E402
                     fft_signals, loud_over_quiet, mel64, wide_signals)
from some_b200 import _lib, synth  # noqa: E402
from some_b200.weights import mel_tables  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = 'cuda'
# the first interior frame is f = 2 and needs L >= 2048; the last is floor((L - 1024) / 512); T = 1 + L // 512 crosses the
# 8-frame warp and 64-frame CTA tiles at 8 * 512 and 64 * 512
LENGTHS = [1, 511, 512, 513, 1023, 1024, 1025, 1535, 1536, 2047, 2048, 2049, 8 * 512 - 1, 8 * 512 + 1, 64 * 512 - 1,
           64 * 512 + 1, 65 * 512, 30 * SR]
GOLDEN_LOG_TOL = 1e-3   # the tolerance of test_gpu_kernels.py::test_keyshift_mel_matches_reference_golden (shifts -5..5)
KS_FR = 8   # frames per CTA of the key-shift kernel


@pytest.fixture(scope='module')
def lib():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    return _lib.load()


@pytest.fixture(scope='module')
def tables():
    tab = mel_tables(synth.named_config('two_head'), DEV)
    assert np.array_equal(tab['bank'].astype(np.float64), BASIS)
    return tab


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def bits(t):
    return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int16)


@pytest.fixture(scope='module')
def fft_cases():
    """(signal, length, samples, mel64) for every signal at every length"""
    cases = []
    for n in LENGTHS:
        for name, x in fft_signals(n).items():
            cases.append((name, n, x, mel64(x)))
    return cases


def pack(cases, odd):
    """all clips in one buffer with NaN between them; starts 16-byte aligned, or at odd float offsets"""
    starts, pos = [], 0
    for _, n, _, _ in cases:
        pos += 4
        pos = (pos + 3) // 4 * 4 + (1 + 2 * (len(starts) % 2) if odd else 0)
        starts.append(pos)
        pos += n
    wave = np.full(pos + 4, np.nan, dtype=np.float32)
    for s, (_, n, x, _) in zip(starts, cases):
        wave[s:s + n] = x
    return torch.from_numpy(wave).to(DEV), starts


def run_mel(lib, tab, wave, starts, lens, frames, guard=8):
    """some_mel_logmel with both outputs into NaN-filled buffers of M + guard rows"""
    cu = np.zeros(len(frames) + 1, dtype=np.int32)
    np.cumsum(frames, out=cu[1:])
    m = int(cu[-1])
    f32 = torch.full((m + guard, 80), float('nan'), device=DEV)
    bf16 = torch.full((m + guard, 80), float('nan'), device=DEV, dtype=torch.bfloat16)
    st = torch.tensor(starts, dtype=torch.int64, device=DEV)
    ln = torch.tensor(lens, dtype=torch.int64, device=DEV)
    cu_d = torch.from_numpy(cu).to(DEV)
    _lib.check(lib.some_mel_logmel(wave.data_ptr(), st.data_ptr(), ln.data_ptr(), cu_d.data_ptr(), len(frames), max(frames),
                                   tab['mel_start'].data_ptr(), tab['mel_count'].data_ptr(), tab['mel_weights'].data_ptr(),
                                   tab['twiddle'].data_ptr(), tab['window'].data_ptr(), f32.data_ptr(), bf16.data_ptr(),
                                   CLAMP, stream()), 'some_mel_logmel')
    torch.cuda.synchronize()
    return f32, bf16, cu


def print_table(title, worst):
    print(f'\n{title}: largest error / bound (linear, log) and largest log error where the log is compared')
    for key, (lin, log, err) in worst.items():
        print(f'  {key:<36} {lin:8.4f} {log:8.4f}   {err:.2e}')


def merge(worst, key, r):
    old = worst.get(key, (0.0, 0.0, 0.0))
    worst[key] = tuple(max(a, b) for a, b in zip(old, r))


@pytest.mark.parametrize('odd', [False, True], ids=['aligned', 'odd_offsets'])
def test_register_fft_against_float64(lib, tables, fft_cases, odd):
    wave, starts = pack(fft_cases, odd)
    lens = [n for _, n, _, _ in fft_cases]
    frames = [1 + n // HOP for n in lens]
    f32, bf16, cu = run_mel(lib, tables, wave, starts, lens, frames)
    m = int(cu[-1])
    assert torch.isnan(f32[m:]).all() and torch.isnan(bf16[m:].float()).all(), 'a guard row after M was written'
    assert torch.equal(bits(bf16[:m]), bits(f32[:m].to(torch.bfloat16))), 'out_bf16 is not bf16_rn(out_f32)'
    got_all = f32[:m].cpu().numpy()
    silent = np.float32(np.log(np.float32(CLAMP)))
    worst = {}
    for i, (name, n, _, ref) in enumerate(fft_cases):
        got = got_all[cu[i]:cu[i + 1]]
        assert np.isfinite(got).all(), (name, n)
        # frames whose samples are all zero (silence, the padding, impulses far away) are exactly the clamp's log: the
        # same bits everywhere, within 1 ulp of log(1e-5f)
        zero = ref.S == 0
        if zero.any():
            z = got[zero].view(np.int32)
            assert (z == z.flat[0]).all(), (name, n)
            assert abs(int(z.flat[0]) - int(silent.view(np.int32))) <= 1, (name, n, got[zero].flat[0])
        r = bound_ratios(got, ref, C_FFT)
        assert r[0] <= 1.0 and r[1] <= 1.0, (name, n, odd, r)
        merge(worst, name, r)
    print_table(f'register FFT, {"odd offsets" if odd else "16-byte aligned"}', worst)


# ------------------------------------------------------------------------------------------------- key-shift DFT
@pytest.fixture(scope='module')
def spec_mel():
    from some_b200.spec import MelSpectrogram
    mel = MelSpectrogram(80, SR, 2048, 512, mel_fmin=40, mel_fmax=8000)
    assert np.array_equal(mel.mel_basis.numpy().astype(np.float64), BASIS)
    return mel


def ks_run(mel, x, **kw):
    """[T, 80] fp32 log-mel of one clip"""
    return mel(torch.from_numpy(np.asarray(x, np.float32)).to(DEV)[None], **kw)[0].t().cpu().numpy()


def ks_check(worst, group, got, ref, name):
    r = bound_ratios(got, ref, c_dft(ref.n_fft))
    assert r[0] <= 1.0 and r[1] <= 1.0, (name, r)
    merge(worst, group, r)
    return r


def test_keyshift_against_golden_and_float64(spec_mel):
    """every case of keyshift_wide.npz within the bound of float64, and within 1e-3 of the reference's log:
    * on the sung-note signal in every band, as for shifts -5..5 (the reference's fp32 output is within 2e-4 of float64 in
      every band there);
    * on the loud tone over -100 dB noise only where the band is 1000 x above the bound: in its quiet bands the reference's
      own fp32 output is off float64 by up to 0.04 in the log (fp32 round-off of the loud bins, |X| <= S_t), so no fp32
      implementation can match it there; the linear comparison with float64 covers those bands."""
    g = np.load(HERE / 'golden' / 'keyshift_wide.npz')
    worst, worst_ks12 = {}, {}
    cases = [(sig, wave, key, kw) for sig, wave in wide_signals().items() for key, kw in WIDE_CASES]
    cases.append(('shortest', loud_over_quiet(4096), 'shortest_ks12', dict(keyshift=12, center=False)))
    for sig, wave, key, kw in cases:
        name = key if sig == 'shortest' else f'{sig}/{key}'
        got = ks_run(spec_mel, wave, **kw)
        want = g[name].T
        assert got.shape == want.shape, (name, got.shape, want.shape)
        ref = mel64(wave, **kw)
        kind = 'fractional' if 'frac' in key else 'speed' if 'speed' in key else 'center=False' if 'nocenter' in key else 'integer'
        ks_check(worst, f'{sig} {kind}', got, ref, name)
        tau = ref.tau(c_dft(ref.n_fft))
        compared = np.ones_like(ref.lin, dtype=bool) if sig == 'sung' else ref.lin >= 1000.0 * tau
        err = float(np.abs(got - want)[compared].max()) if compared.any() else 0.0
        assert err < GOLDEN_LOG_TOL, (name, err)
        if abs(kw.get('keyshift', 0)) == 12:
            big = ref.lin >= 1000.0 * tau
            now = (float(np.abs(got - ref.log)[big].max()) if big.any() else 0.0, float(np.abs(got - ref.log).max()))
            worst_ks12[sig] = tuple(max(a, b) for a, b in zip(worst_ks12.get(sig, (0.0, 0.0)), now))
    print_table('key-shift DFT, keyshift_wide.npz cases against float64', worst)
    for sig, (above, every) in worst_ks12.items():
        print(f'  {sig} at +-12: largest |log-mel - float64| {above:.2e} where the band is 1000 x above the bound, '
              f'{every:.2e} over every band')


@pytest.mark.parametrize('keyshift', [12, -12, -18, -24])
def test_keyshift_tiles_and_short_ffts(spec_mel, keyshift):
    """frame counts on and around multiples of the 8-frame tile; at -18 (n' = 724) and -24 (n' = 512) the bins past n' / 2
    do not exist and must be zero, as the reference pads them.  The sung-note signal is also held to SUNG_LOG_TOL in every
    band, which an fp16 window or twiddle table breaks (tests/test_mel_f64_cpu.py::test_fp16_table_is_caught)"""
    worst = {}
    for t in (1, 7, 8, 9, 15, 16, 17, 63, 64, 65):
        n = (t - 1) * HOP + 100
        for name, x in (('loud', loud_over_quiet(n)), ('sung', synth.synth_waveform(4242, num_samples=n))):
            got = ks_run(spec_mel, x, keyshift=keyshift)
            assert got.shape == (t, 80)
            ref = mel64(x, keyshift=keyshift)
            ks_check(worst, f'{keyshift:+d} {name}', got, ref, (keyshift, t, name))
            if name == 'sung':   # every band, as against the golden
                err = float(np.abs(got - ref.log).max())
                assert err < SUNG_LOG_TOL, (keyshift, t, err)
                merge(worst, f'{keyshift:+d} sung, every band', (0.0, 0.0, err))
    print_table(f'key-shift DFT at {keyshift:+d}, T around multiples of {KS_FR}', worst)


def test_keyshift_batch_equals_alone(spec_mel):
    n = 37 * HOP + 11
    clips = [loud_over_quiet(n), synth.synth_waveform(4242, num_samples=n),
             np.clip(np.random.default_rng(5).standard_normal(n), -1, 1).astype(np.float32)]
    for kw in (dict(keyshift=12), dict(keyshift=-11.9), dict(keyshift=12, speed=2.0, center=False)):
        both = spec_mel(torch.from_numpy(np.stack(clips)).to(DEV), **kw)
        for i, x in enumerate(clips):
            alone = spec_mel(torch.from_numpy(x).to(DEV)[None], **kw)[0]
            assert torch.equal(bits(both[i]), bits(alone)), (kw, i)


def test_keyshift_refusals(lib, tables, spec_mel):
    """what the key-shift kernel refuses is refused on the host, with its message, before anything is launched"""
    x = loud_over_quiet(8 * HOP)
    # n' < 372 (a shift below about -29): the reference computes it, the kernel does not keep enough bins
    assert np.isfinite(mel64(x, keyshift=-30).log).all()
    with pytest.raises(_lib.SomeB200Error, match=r'n_fft 362 / hop 512 / pad 181 out of range'):
        spec_mel(torch.from_numpy(x).to(DEV)[None], keyshift=-30)
    with pytest.raises(_lib.SomeB200Error, match=r'n_fft 8679 / hop 512 / pad 4339 out of range'):
        spec_mel(torch.from_numpy(x).to(DEV)[None], keyshift=25)
    with pytest.raises(_lib.SomeB200Error, match=r'n_fft 8192 with hop 4096 needs 257664 B of shared memory'):
        spec_mel(torch.from_numpy(x).to(DEV)[None], keyshift=24, speed=8)
    # one sample shorter than the shortest audio torch.stft accepts at +12 (center=False: n = n' = 4096)
    with pytest.raises(RuntimeError, match='shorter than one STFT window'):
        spec_mel(torch.from_numpy(loud_over_quiet(4095)).to(DEV)[None], keyshift=12, center=False)
    # the refused calls through the C ABI leave their output untouched
    wave = torch.from_numpy(x).to(DEV)
    st = torch.zeros(1, dtype=torch.int64, device=DEV)
    ln = torch.full((1,), len(x), dtype=torch.int64, device=DEV)
    cu = torch.tensor([0, 9], dtype=torch.int32, device=DEV)
    out = torch.full((9, 80), float('nan'), device=DEV)
    tw = torch.zeros((8192, 2), device=DEV)
    win = torch.zeros(8192, device=DEV)
    for n_fft, hop in ((362, 512), (8679, 512), (8192, 4096)):
        rc = lib.some_mel_logmel_keyshift(wave.data_ptr(), st.data_ptr(), ln.data_ptr(), cu.data_ptr(), 1, 9, n_fft, hop,
                                          n_fft // 2, 1.0, tables['mel_start'].data_ptr(), tables['mel_count'].data_ptr(),
                                          tables['mel_weights'].data_ptr(), tw.data_ptr(), win.data_ptr(), out.data_ptr(),
                                          None, CLAMP, stream())
        assert rc != 0 and b'some_mel_logmel_keyshift' in lib.some_last_error()
    torch.cuda.synchronize()
    assert torch.isnan(out).all()

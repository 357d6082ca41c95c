"""Bit-exact self-consistency of the log-mel, LayerNorm and depthwise-conv kernels (through the C ABI): no kernel mixes
clips or groups, so the rows of a clip must come out the same bits whether the clip runs alone or batched with others,
at any alignment of its samples and in either group.  A tiling that leaks across a clip, tile or CTA edge shows up here."""
import ctypes as C

import numpy as np
import pytest
import torch

from some_b200 import _lib, synth
from some_b200.weights import mel_tables

pytestmark = pytest.mark.gpu

DEV = 'cuda'
# clip lengths in frames: around the 16-row LayerNorm CTAs, 8-frame mel warps, 64-frame mel CTAs and 128-row dwconv tiles, and a 30 s clip
FRAMES = [1, 31, 32, 33, 127, 128, 129, 157, 159, 2584]


@pytest.fixture(scope='module')
def lib():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    return _lib.load()


@pytest.fixture(scope='module')
def tables():
    return mel_tables(synth.named_config('two_head'), DEV)


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _cu(frames):
    cu = np.zeros(len(frames) + 1, dtype=np.int32)
    np.cumsum(frames, out=cu[1:])
    return torch.from_numpy(cu).to(DEV)


def samples_for(frames):
    """a clip length in samples that gives `frames` frames (T = 1 + n // 512), with a ragged tail"""
    return (frames - 1) * _lib.HOP + 37


def run_mel(lib, tab, wave, starts, lens, frames):
    cu = _cu(frames)
    m = int(cu[-1])
    f32 = torch.full((m, _lib.N_MELS), float('nan'), device=DEV)
    bf16 = torch.full((m, _lib.N_MELS), float('nan'), device=DEV, dtype=torch.bfloat16)
    st = torch.tensor(starts, dtype=torch.int64, device=DEV)
    ln = torch.tensor(lens, dtype=torch.int64, device=DEV)
    _lib.check(lib.some_mel_logmel(wave.data_ptr(), st.data_ptr(), ln.data_ptr(), cu.data_ptr(), len(frames), max(frames),
                                   tab['mel_start'].data_ptr(), tab['mel_count'].data_ptr(), tab['mel_weights'].data_ptr(),
                                   tab['twiddle'].data_ptr(), tab['window'].data_ptr(), f32.data_ptr(), bf16.data_ptr(),
                                   1e-5, stream()), 'some_mel_logmel')
    torch.cuda.synchronize()
    return f32, bf16


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32 if a.dtype == torch.float32 else torch.int16),
                       b.contiguous().view(torch.int32 if b.dtype == torch.float32 else torch.int16))


def test_mel_batched_equals_alone(lib, tables):
    lens = [samples_for(f) for f in FRAMES]
    # clips laid end to end with a 2-sample gap so that every other clip starts 8-byte aligned
    starts, pos = [], 0
    for n in lens:
        starts.append(pos)
        pos += n + 2
    wave = torch.zeros(pos, dtype=torch.float32)
    for i, (s, n) in enumerate(zip(starts, lens)):
        wave[s:s + n] = torch.from_numpy(synth.synth_waveform(900 + i, num_samples=n))
    wave_gap = wave.to(DEV)
    f32_all, bf16_all = run_mel(lib, tables, wave_gap, starts, lens, FRAMES)
    r0 = 0
    for s, n, t in zip(starts, lens, FRAMES):
        f32_one, bf16_one = run_mel(lib, tables, wave_gap, [s], [n], [t])
        assert same_bits(f32_all[r0:r0 + t], f32_one), f'mel f32 of the {t}-frame clip differs batched vs alone'
        assert same_bits(bf16_all[r0:r0 + t], bf16_one), f'mel bf16 of the {t}-frame clip differs batched vs alone'
        r0 += t
    assert torch.isfinite(f32_all).all()


@pytest.mark.parametrize('frames', [33, 129, 2584])
def test_mel_aligned_equals_misaligned(lib, tables, frames):
    """the same samples at an 8-byte-aligned start (interior frames load float2 directly) and at a 4-byte offset (every
    frame is staged through the warp's tile) give the same bits"""
    n = samples_for(frames)
    x = torch.from_numpy(synth.synth_waveform(77 + frames, num_samples=n)).to(DEV)
    buf = torch.zeros(n + 8, device=DEV)
    buf[2:2 + n] = x
    a32, a16 = run_mel(lib, tables, buf, [2], [n], [frames])
    buf2 = torch.zeros(n + 8, device=DEV)
    buf2[3:3 + n] = x
    b32, b16 = run_mel(lib, tables, buf2, [3], [n], [frames])
    assert buf.data_ptr() % 8 == 0 and buf2.data_ptr() % 8 == 0
    assert same_bits(a32, b32) and same_bits(a16, b16)


def run_ln(lib, xs, gammas, betas, with_f32=True):
    m = xs[0].shape[0]
    ob = [torch.full((m, 512), float('nan'), device=DEV, dtype=torch.bfloat16) for _ in xs]
    of = [torch.full((m, 512), float('nan'), device=DEV) for _ in xs]
    a = _lib.LnArgs()
    a.x, a.gamma, a.beta = _lib.pair(*xs), _lib.pair(*gammas), _lib.pair(*betas)
    a.out_bf16 = _lib.pair(*ob)
    a.out_f32 = _lib.pair(*of) if with_f32 else (C.c_void_p * 2)()
    a.groups, a.M = len(xs), m
    _lib.check(lib.some_layernorm(C.byref(a), stream()), 'some_layernorm')
    torch.cuda.synchronize()
    return ob, of


@pytest.mark.parametrize('m', [1, 17, 1003, sum(FRAMES)])
def test_layernorm_rows_groups_and_outputs(lib, m):
    """each row's bits depend on that row only: the whole batch equals every clip's rows run alone, groups = 2 equals
    groups = 1 for each group, and the bf16 output does not depend on whether the f32 one is written"""
    torch.manual_seed(m)
    x = [torch.randn(m, 512, device=DEV) * 3 + 1.5 for _ in range(2)]
    g = [torch.rand(512, device=DEV) + 0.5 for _ in range(2)]
    b = [torch.randn(512, device=DEV) * 0.1 for _ in range(2)]
    ob2, of2 = run_ln(lib, x, g, b)
    for i in range(2):
        ob1, of1 = run_ln(lib, [x[i]], [g[i]], [b[i]])
        assert same_bits(ob1[0], ob2[i]) and same_bits(of1[0], of2[i])
        obn, _ = run_ln(lib, [x[i]], [g[i]], [b[i]], with_f32=False)
        assert same_bits(obn[0], ob2[i])
    if m == sum(FRAMES):
        r0 = 0
        for t in FRAMES:
            ob1, of1 = run_ln(lib, [x[0][r0:r0 + t].contiguous()], [g[0]], [b[0]])
            assert same_bits(ob1[0], ob2[0][r0:r0 + t]) and same_bits(of1[0], of2[0][r0:r0 + t])
            r0 += t


def run_dw(lib, xs, ws, bs, frames):
    cu = _cu(frames)
    m = int(cu[-1])
    out = [torch.full((m, 512), float('nan'), device=DEV, dtype=torch.bfloat16) for _ in xs]
    a = _lib.DwconvArgs()
    a.x, a.w, a.b, a.out = _lib.pair(*xs), _lib.pair(*ws), _lib.pair(*bs), _lib.pair(*out)
    a.groups, a.B, a.cu_frames, a.max_frames = len(xs), len(frames), cu.data_ptr(), max(frames)
    _lib.check(lib.some_dwconv_bn_silu(C.byref(a), stream()), 'some_dwconv_bn_silu')
    torch.cuda.synchronize()
    return out


def test_dwconv_batched_equals_alone_and_groups(lib):
    torch.manual_seed(11)
    m = sum(FRAMES)
    x = [torch.randn(m, 512, device=DEV).to(torch.bfloat16) for _ in range(2)]
    w = [torch.randn(31, 512, device=DEV) * 0.2 for _ in range(2)]
    b = [torch.randn(512, device=DEV) * 0.1 for _ in range(2)]
    both = run_dw(lib, x, w, b, FRAMES)
    for i in range(2):
        one_group = run_dw(lib, [x[i]], [w[i]], [b[i]], FRAMES)[0]
        assert same_bits(one_group, both[i]), f'group {i}: groups = 1 and groups = 2 differ'
        r0 = 0
        for t in FRAMES:
            alone = run_dw(lib, [x[i][r0:r0 + t].contiguous()], [w[i]], [b[i]], [t])[0]
            assert same_bits(alone, both[i][r0:r0 + t]), f'group {i}: the {t}-frame clip differs batched vs alone'
            r0 += t
    assert all(torch.isfinite(o.float()).all() for o in both)

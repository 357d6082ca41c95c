"""The row-wise trunk kernels of csrc/rowwise.cu, through the C ABI, against the float64 models and references of
tests/golden/rowwise_f64.py, computed on the device:

* some_layernorm: every output within ln_bound of kernel64 and within that plus the eps32 gap of exact64, at M around the
  16-row CTAs and at the benchmark's 165 376 rows per group, groups 1 and 2 with different data and parameters, out_f32
  null and not; the bf16 output is RNE of the same launch's fp32 output bit for bit and does not depend on out_f32;
  constant rows with at most 15 significant bits give beta exactly;
* some_bound_head: within head_bound at M around the 8-row CTA and at 165 376 rows, z across +-40;
* some_row_stats: slot 0 within the sum bounds, slots 1.. untouched, the bf16 copy RNE(x);
* some_dwconv_bn_silu: every in-clip row within dw_bound of kernel64 (the exact bf16 gap) and within that plus the fold
  bound of exact64 (Conv1d + BatchNorm1d from the unfolded parameters), for clip lengths around the 128-frame tiles and
  16-frame warps, at 64 x 2584 frames (84 tiles per persistent CTA on 132 SMs), with runs of empty tiles and a larger
  max_frames; one group and two give the same bits;
* fences: inputs are views with NaN rows behind them, outputs buffers whose rows past M (or cu_frames[B]) and the unused
  ln_stats slots hold a NaN payload that must keep its bits.

Run with -s to see max and rms err / bound per kernel, regime and group."""
import ctypes as C
import pathlib
import sys
import zlib

import numpy as np
import pytest
import torch

HERE = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / 'golden'))

import rowwise_f64 as rf  # noqa: E402
from rowwise_f64 import DIM, DW_REGIMES, HEAD_REGIMES, K, ROW_REGIMES, abs_ratio, gap_ratio  # noqa: E402
from some_b200 import _lib  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = 'cuda'
BF16 = torch.bfloat16
GUARD = 3
NAN32, NAN16 = 0x7fc0dead, 0x7fa5           # NaN payloads no kernel computes
LN_M = [1, 2, 15, 16, 17, 31, 33, 1003, 64 * 2584]
HEAD_M = [1, 7, 8, 9, 16, 17, 1003, 64 * 2584]
STATS_M = [1, 2, 15, 16, 17, 33, 1003, 64 * 2584]
DW_FRAMES = [1, 2, 14, 15, 16, 17, 30, 31, 32, 112, 113, 127, 128, 129, 143, 144, 255, 256, 257, 300, 2584]


@pytest.fixture(scope='module')
def lib():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    return _lib.load()


def seeded(*key):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def nan_f32(*shape):
    return torch.full(shape, NAN32, dtype=torch.int32, device=DEV).view(torch.float32)


def nan_bf16(*shape):
    return torch.full(shape, NAN16, dtype=torch.int16, device=DEV).view(BF16)


def fenced(x):
    """x [m, 512] fp32 in a buffer with GUARD NaN rows behind it"""
    buf = torch.full((x.shape[0] + GUARD, x.shape[1]), float('nan'), device=DEV, dtype=x.dtype)
    buf[:x.shape[0]] = x
    return buf


def untouched(label, t, payload):
    bits = t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)
    assert bool((bits == payload).all()), f'{label}: a store landed outside the rows or slots the kernel owns'


def report(label, r):
    """r <= 1 elementwise; prints and returns max and rms"""
    mx, rms = r.max().item(), r.square().mean().sqrt().item()
    print(f'{label}: err/bound max {mx:.3g} rms {rms:.3g}', flush=True)
    assert mx <= 1.0, f'{label}: error {mx:.3g} x its bound at {np.unravel_index(int(r.argmax()), tuple(r.shape))}'
    return mx, rms


def same_bits(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


# ------------------------------------------------------------------------------------------------------------ LayerNorm
def run_ln(lib, xs, gammas, betas, with_f32=True):
    """one launch, groups = len(xs); returns each group's (bf16 [M, 512], fp32 [M, 512] or None)"""
    m = xs[0].shape[0]
    xb = [fenced(x) for x in xs]
    ob = [nan_bf16(m + GUARD, DIM) for _ in xs]
    of = [nan_f32(m + GUARD, DIM) for _ in xs]
    a = _lib.LnArgs()
    a.x, a.gamma, a.beta = _lib.pair(*xb), _lib.pair(*gammas), _lib.pair(*betas)
    a.out_bf16 = _lib.pair(*ob)
    a.out_f32 = _lib.pair(*of) if with_f32 else (C.c_void_p * 2)()
    a.groups, a.M = len(xs), m
    _lib.check(lib.some_layernorm(C.byref(a), stream()), 'some_layernorm')
    torch.cuda.synchronize()
    for i in range(len(xs)):
        untouched(f'layernorm group {i} bf16 rows past M', ob[i][m:], NAN16)
        untouched(f'layernorm group {i} fp32', of[i][m:] if with_f32 else of[i], NAN32)
    return [(ob[i][:m], of[i][:m] if with_f32 else None) for i in range(len(xs))]


@pytest.mark.parametrize('m', LN_M)
def test_layernorm(lib, m):
    for name in ROW_REGIMES:
        x = [rf.rows(name, m, seeded('ln', name, m, g), DEV) for g in range(2)]
        par = [rf.ln_params(seeded('ln params', name, g), DEV) for g in range(2)]
        both = run_ln(lib, x, [p[0] for p in par], [p[1] for p in par])
        for g in range(2):
            ob, of = both[g]
            gamma, beta = par[g]
            ref, e = rf.ln_bound(x[g], gamma, beta)
            report(f'layernorm M={m} {name} group {g} fp32', abs_ratio(of, ref, e))
            report(f'layernorm M={m} {name} group {g} fp32 vs exact64',
                   abs_ratio(of, rf.ln_exact64(x[g], gamma, beta), e + rf.ln_eps_gap(x[g], gamma)))
            assert same_bits(ob, of.to(BF16)), f'{name} group {g}: the bf16 output is not RNE of the fp32 output'
            report(f'layernorm M={m} {name} group {g} bf16 gap', gap_ratio(ob, ref, e))
            if name == 'const15':
                assert torch.equal(of, beta.expand(m, DIM)), f'group {g}: constant rows do not give beta exactly'
            alone, = run_ln(lib, [x[g]], [gamma], [beta], with_f32=False)
            assert same_bits(alone[0], ob), f'{name} group {g}: groups = 1 without out_f32 changes the bf16 output'
            del ref, e


# ------------------------------------------------------------------------------------------------------------ bound head
@pytest.mark.parametrize('m', HEAD_M)
def test_bound_head(lib, m):
    for name in HEAD_REGIMES:
        x = rf.rows(name, m, seeded('head', name, m), DEV)
        gamma, beta = rf.ln_params(seeded('head params', name), DEV)
        w, bias = rf.head_params(name, seeded('head w', name), DEV)
        out = nan_f32(m + GUARD)
        _lib.check(lib.some_bound_head(fenced(x).data_ptr(), gamma.data_ptr(), beta.data_ptr(), w.data_ptr(), bias, m,
                                       out.data_ptr(), stream()), 'some_bound_head')
        torch.cuda.synchronize()
        untouched(f'bound head {name} rows past M', out[m:], NAN32)
        ref, e = rf.head_bound(x, gamma, beta, w, bias)
        report(f'bound head M={m} {name}', abs_ratio(out[:m], ref, e))
        report(f'bound head M={m} {name} vs exact64',
               abs_ratio(out[:m], rf.head_exact64(x, gamma, beta, w, bias), e + rf.head_eps_gap(x, gamma, w)))


# ------------------------------------------------------------------------------------------------------------ row stats
@pytest.mark.parametrize('m', STATS_M)
def test_row_stats(lib, m):
    for name in ROW_REGIMES:
        x = [rf.rows(name, m, seeded('stats', name, m, g), DEV) for g in range(2)]
        xb = [nan_bf16(m + GUARD, DIM) for _ in range(2)]
        st = [nan_f32(m + GUARD, _lib.LN_SLOTS, 2) for _ in range(2)]
        a = _lib.RowStatsArgs()
        a.x, a.out_bf16, a.ln_stats = _lib.pair(*[fenced(v) for v in x]), _lib.pair(*xb), _lib.pair(*st)
        a.groups, a.M = 2, m
        _lib.check(lib.some_row_stats(C.byref(a), stream()), 'some_row_stats')
        torch.cuda.synchronize()
        for g in range(2):
            untouched(f'row stats {name} group {g} slots 1..', st[g][:, 1:], NAN32)
            untouched(f'row stats {name} group {g} rows past M', st[g][m:], NAN32)
            untouched(f'row stats {name} group {g} bf16 rows past M', xb[g][m:], NAN16)
            assert same_bits(xb[g][:m], x[g].to(BF16)), f'{name} group {g}: the bf16 copy is not RNE(x)'
            s, q = rf.stats_exact64(x[g])
            es, eq = rf.stats_bound(x[g])
            report(f'row stats M={m} {name} group {g} sum', abs_ratio(st[g][:m, 0, 0], s, es))
            report(f'row stats M={m} {name} group {g} sum of squares', abs_ratio(st[g][:m, 0, 1], q, eq))


# ------------------------------------------------------------------------------------------------------------ dwconv
def pack_fold(p):
    """the BatchNorm fold the project ships (some_pack_dwconv_bn, the C twin of weights.checkpoint_block): fp32 taps
    [31, 512] and bias [512] on the device"""
    args = [p[k].cpu().contiguous().numpy() for k in ('weight', 'bias', 'bn_weight', 'bn_bias', 'bn_mean', 'bn_var')]
    taps, bias = np.zeros((K, DIM), np.float32), np.zeros(DIM, np.float32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    assert _lib.load().some_pack_dwconv_bn(*[ptr(a) for a in args], DIM, K, ptr(taps), ptr(bias)) == 0
    return torch.from_numpy(taps).to(DEV), torch.from_numpy(bias).to(DEV)


def dw_data(name, frames, key):
    gen = seeded('dw', name, key)
    x = torch.cat([rf.dw_clip(name, t, i, gen, DEV) for i, t in enumerate(frames)])
    p = rf.dw_regime_params(name, gen, DEV)
    return x, p, *pack_fold(p)


def run_dw(lib, xs, taps, biases, frames, max_frames=None):
    cu = [0] + [int(v) for v in np.cumsum(frames)]
    m = cu[-1]
    cu_d = torch.tensor(cu, dtype=torch.int32, device=DEV)
    out = [nan_bf16(m + GUARD, DIM) for _ in xs]
    a = _lib.DwconvArgs()
    a.x = _lib.pair(*[fenced(x.to(BF16)) for x in xs])
    a.w, a.b, a.out = _lib.pair(*taps), _lib.pair(*biases), _lib.pair(*out)
    a.groups, a.B, a.cu_frames, a.max_frames = len(xs), len(frames), cu_d.data_ptr(), max_frames or max(frames)
    _lib.check(lib.some_dwconv_bn_silu(C.byref(a), stream()), 'some_dwconv_bn_silu')
    torch.cuda.synchronize()
    for i in range(len(xs)):
        untouched(f'dwconv group {i} rows past cu_frames[B]', out[i][m:], NAN16)
    return [o[:m] for o in out], cu


def check_dw(label, out, x, cu, p, taps, bias):
    ref, e = rf.dw_bound(x, cu, taps, bias)
    r = report(label, gap_ratio(out, ref, e))
    report(label + ' vs exact64', gap_ratio(out, rf.dw_exact64(x, cu, p), e + rf.dw_fold_bound(x, cu, taps, bias)))
    return r


@pytest.mark.parametrize('name', DW_REGIMES)
def test_dwconv_every_clip_length(lib, name):
    """one var-len launch of DW_FRAMES in two groups of different data and parameters; one group and a larger max_frames
    give the same bits"""
    d = [dw_data(name, DW_FRAMES, g) for g in range(2)]
    outs, cu = run_dw(lib, [v[0] for v in d], [v[2] for v in d], [v[3] for v in d], DW_FRAMES)
    for g in range(2):
        x, p, taps, bias = d[g]
        check_dw(f'dwconv {name} group {g}', outs[g], x, cu, p, taps, bias)
        one, _ = run_dw(lib, [x], [taps], [bias], DW_FRAMES, max_frames=max(DW_FRAMES) + 300)
        assert same_bits(one[0], outs[g]), f'{name} group {g}: one group with a larger max_frames changes the bits'


@pytest.mark.parametrize('groups', [2, 1])
def test_dwconv_benchmark_scale(lib, groups):
    """64 x 2584 frames: 21 tiles per clip, 1344 per (channel block, group), so each persistent CTA walks many tiles and
    its double buffer swaps"""
    frames = [2584] * 64
    names = ['iid_synthetic', 'iid_trained'][:groups]
    d = [dw_data(name, frames, 'scale') for name in names]
    outs, cu = run_dw(lib, [v[0] for v in d], [v[2] for v in d], [v[3] for v in d], frames)
    for g, name in enumerate(names):
        check_dw(f'dwconv 64 x 2584 groups={groups} {name}', outs[g], *d[g][:1], cu, *d[g][1:])


def test_dwconv_runs_of_empty_tiles(lib):
    """one 2584-frame clip then 200 one-frame clips: 21 tiles per clip, 20 of them empty for all but the first clip"""
    frames = [2584] + [1] * 200
    d = [dw_data(name, frames, 'empty') for name in ('edges', 'iid_trained')]
    outs, cu = run_dw(lib, [v[0] for v in d], [v[2] for v in d], [v[3] for v in d], frames)
    for g, name in enumerate(('edges', 'iid_trained')):
        check_dw(f'dwconv 2584 + 200 x 1 {name}', outs[g], *d[g][:1], cu, *d[g][1:])

"""The float64 references, models and bounds of tests/golden/rowwise_f64.py, without a GPU:

* each exact64 is the float64 torch.nn module it restates: LayerNorm, Linear + sigmoid, Conv1d + BatchNorm1d.eval() + SiLU;
* each bound holds for an fp32 emulation of its kernel (csrc/rowwise.cu) written below, on every data regime, under every
  combination of: the per-lane order and the butterfly order forward, reversed or shuffled (the conv's tap order likewise),
  rsqrtf and expf moved by -2, 0 or +2 ulp, tanh.approx moved by -2^-10.987, 0 or +2^-10.987 relative, every fp32 operation
  rounded to nearest (fmaf rounded once);
* kernel64 of the depthwise conv, from the project's folds (weights.checkpoint_block and some_pack_dwconv_bn), lies within
  the fold bound of exact64 for the synthetic and the trained-like BatchNorm statistics;
* the bounds have power: each planted defect of an emulation exceeds twice its bound on at least one regime.

Run with -s to see the ratios."""
import ctypes as C
import itertools
import pathlib
import sys
import zlib

import numpy as np
import pytest
import torch

HERE = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / 'golden'))

import rowwise_f64 as rf  # noqa: E402
from rowwise_f64 import (DIM, DW_REGIMES, HEAD_REGIMES, K, ROW_REGIMES, TANH_REL, abs_ratio, gap_ratio,  # noqa: E402
                         ln_bound, ln_exact64, rows)

F32, F64 = np.float32, np.float64


def gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


# ------------------------------------------------------------------------------------------------ fp32 building blocks
def fma32(a, b, c):
    """fmaf(a, b, c) on float32 arrays, rounded once to nearest even: a b is exact in float64, the float64 sum's own
    rounding error (TwoSum) breaks a float64 result that sits exactly on an fp32 midpoint"""
    p = a.astype(F64) * b.astype(F64)
    c = c.astype(F64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    mant, _ = np.frexp(s)
    t = np.ldexp(mant, 25)
    mid = (t == np.floor(t)) & (np.fmod(np.abs(t), 2) == 1) & (err != 0)
    s = np.where(mid, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def move_ulps(r, k):
    """float32 r moved by k ulp"""
    for _ in range(abs(k)):
        r = np.nextafter(r, np.where(np.full_like(r, k > 0, dtype=bool), F32(np.inf), F32(-np.inf))).astype(F32)
    return r


def rsqrt32(a, ulps):
    with np.errstate(invalid='ignore'):             # a negative variance (a planted defect) gives NaN, as rsqrtf does
        return move_ulps((1.0 / np.sqrt(a.astype(F64))).astype(F32), ulps)


def exp32(a, ulps):
    return move_ulps(np.exp(a.astype(F64)).astype(F32), ulps)


def bf16_tz(x):
    """float32 -> bf16 toward zero (as float32)"""
    return (np.ascontiguousarray(x, F32).view(np.uint32) & np.uint32(0xffff0000)).view(F32)


def bf16_rne(x):
    return torch.from_numpy(np.ascontiguousarray(x, F32)).to(torch.bfloat16).float().numpy()


ORDERS = ('fwd', 'rev', 'rand')


def perm(order, n, seed=0):
    return {'fwd': list(range(n)), 'rev': list(range(n - 1, -1, -1)),
            'rand': torch.randperm(n, generator=gen('perm', n, seed)).tolist()}[order]


def lanes(x):
    """[M, 512] -> [M, 32 lanes, 16 slots]: lane l slot 4 i + j holds column 128 i + 4 l + j"""
    return np.ascontiguousarray(x.reshape(x.shape[0], 4, 32, 4).transpose(0, 2, 1, 3).reshape(x.shape[0], 32, 16))


def unlanes(y):
    return np.ascontiguousarray(y.reshape(y.shape[0], 32, 4, 4).transpose(0, 2, 1, 3).reshape(y.shape[0], DIM))


def butterfly(v, order):
    """xor butterfly over the 32 lanes of v [M, 32]: every lane ends with the same value whatever the level order"""
    for o in [16, 8, 4, 2, 1][::-1 if order == 'rev' else 1] if order != 'rand' else [4, 16, 1, 8, 2]:
        v = (v + v[:, np.arange(32) ^ o]).astype(F32)
    return v[:, 0]


# ------------------------------------------------------------------------------------------------ the kernels in fp32
def emulate_ln(x, gamma, beta, lane_order='fwd', fly='fwd', rsqrt_ulps=0, defect=None):
    """ln_normalise in fp32: x [M, 512], gamma, beta [512] float32 -> y [M, 512] float32 (before any store)"""
    v = lanes(x.astype(F32))
    p16 = perm(lane_order, 16)
    s = np.zeros(v.shape[:2], F32)
    for i in p16:
        s = (s + v[:, :, i]).astype(F32)
    if defect == 'lane dropped from the mean':
        s[:, 5] = 0
    mean = (butterfly(s, fly) * F32(1 / 512))[:, None]
    if defect == 'one-pass variance':
        q = np.zeros(v.shape[:2], F32)
        for i in p16:
            q = fma32(v[:, :, i], v[:, :, i], q)
        var = (butterfly(q, fly) * F32(1 / 512) - mean[:, 0] * mean[:, 0]).astype(F32)
    else:
        q = np.zeros(v.shape[:2], F32)
        for i in p16:
            d = (v[:, :, i] - mean).astype(F32)
            q = fma32(d, d, q)
        var = (butterfly(q, fly) * F32(1 / 511 if defect == '/511' else 1 / 512)).astype(F32)
    eps = F32(1e-6 if defect == 'eps 1e-6' else 1e-5)
    if defect == 'eps outside the root':
        rstd = (F32(1) / (np.sqrt(var).astype(F32) + eps)).astype(F32)
    else:
        rstd = rsqrt32((var + eps).astype(F32), rsqrt_ulps)
    gl, bl = lanes(gamma[None].astype(F32))[0], lanes(beta[None].astype(F32))[0]
    if defect == 'gamma/beta permuted in a lane':
        pi = [1, 2, 3, 0] + list(range(4, 16))       # the first float4 of every lane rotated
        gl, bl = gl[:, pi], bl[:, pi]
    prod = ((v - mean[:, :, None]).astype(F32) * rstd[:, None, None]).astype(F32)
    return unlanes(fma32(prod, gl[None], bl[None]))


def emulate_head(x, gamma, beta, w, bias, lane_order='fwd', fly='fwd', rsqrt_ulps=0, exp_ulps=0, defect=None):
    """bound_head_kernel in fp32 -> [M] float32"""
    y = lanes(emulate_ln(x, gamma, beta, lane_order, fly, rsqrt_ulps))
    wl = lanes(w[None].astype(F32))[0]
    dot = np.zeros(y.shape[:2], F32)
    for i in perm(lane_order, 16, 1):
        dot = fma32(y[:, :, i], np.broadcast_to(wl[:, i], dot.shape), dot)
    z = butterfly(dot, fly)
    if defect != 'bias dropped':
        z = (z + F32(bias)).astype(F32)
    if defect == 'sigmoid(-z)':
        z = -z
    e = exp32(-z, exp_ulps)
    return (F32(1) / (F32(1) + e).astype(F32)).astype(F32)


def emulate_stats(x, lane_order='fwd', fly='fwd', defect=None):
    """row_stats_kernel's (s, q) in fp32"""
    v = lanes(x.astype(F32))
    if defect == 'q of centred values':
        v2 = lanes((x.astype(F64) - x.astype(F64).mean(1, keepdims=True)).astype(F32))
    else:
        v2 = v
    s = np.zeros(v.shape[:2], F32)
    q = np.zeros(v.shape[:2], F32)
    for i in perm(lane_order, 16):
        s = (s + v[:, :, i]).astype(F32)
        q = fma32(v2[:, :, i], v2[:, :, i], q)
    if defect == 'lane dropped':
        s[:, 9] = 0
        q[:, 9] = 0
    return butterfly(s, fly), butterfly(q, fly)


def emulate_dw(x, cu, taps, bias, tap_order='fwd', tanh_rel=0.0, defect=None, pad_rows=None):
    """dwconv_kernel in fp32: x [M, 512] bf16 values, taps [31, 512], bias [512] float32 -> bf16 out [M, 512] (float32).
    pad_rows: for the defect that reads the neighbouring clips' rows instead of zeros, the rows around the batch"""
    m = x.shape[0]
    out = np.zeros((m, DIM), F32)
    taps = taps[::-1] if defect == 'flipped taps' else taps
    shift = {'halo 14': -1, 'halo 16': 1}.get(defect, 0)
    seed = bias * 0 if defect == 'bias dropped' else bias
    full = np.concatenate([pad_rows[0], x, pad_rows[1]]) if pad_rows is not None else None
    npad = pad_rows[0].shape[0] if pad_rows is not None else 0
    for b in range(len(cu) - 1):
        t0, t1 = cu[b], cu[b + 1]
        t = t1 - t0
        # row j of win is clip row j - 16: output row i, tap k reads clip row i + k - 15 (+ shift) = win row i + k + 1 (+ shift)
        if defect == 'neighbour rows as padding':
            win = full[npad + t0 - rf.HALO - 1:npad + t1 + rf.HALO + 1]
        else:
            win = np.zeros((t + 2 * rf.HALO + 2, DIM), F32)
            win[rf.HALO + 1:rf.HALO + 1 + t] = x[t0:t1]
        a = np.broadcast_to(seed, (t, DIM)).astype(F32)
        for k in perm(tap_order, K, 2):
            j = k + 1 + shift
            a = fma32(np.broadcast_to(taps[k], (t, DIM)), win[j:j + t], a)
        h = (a * F32(0.5)).astype(F32)
        th = (np.tanh(h.astype(F64)) * (1 + tanh_rel)).astype(F32)
        y = fma32(h, th, h)
        out[t0:t1] = bf16_tz(y) if defect == 'bf16 truncation' else bf16_rne(y)
    return out


# ------------------------------------------------------------------------------------------------ data
M_ROWS = 512            # the outlier sweeps all 512 columns


def ln_data(name, m=M_ROWS, seed=0):
    x = rows(name, m, gen('rows', name, m, seed))
    g, b = rf.ln_params(gen('ln', name, seed))
    return x, g, b


def dw_data(name, frames, seed=0):
    """(x, cu, unfolded params, fp32 taps, fp32 bias, pad rows (+-2^14) around the batch)"""
    gg = gen('dw', name, seed)
    x = torch.cat([rf.dw_clip(name, t, i, gg) for i, t in enumerate(frames)])
    cu = [0] + list(np.cumsum(frames))
    p = rf.dw_regime_params(name, gg)
    taps, bias = pack_fold(p)
    pad = torch.sign(torch.randn(2, rf.HALO + 1, DIM, generator=gg)) * rf.EDGE
    return x, cu, p, taps, bias, (pad[0].numpy(), pad[1].numpy())


def pack_fold(p, defect=None):
    """some_pack_dwconv_bn (the C fold) of unfolded parameters: fp32 taps [31, 512] and bias [512]"""
    from some_b200 import _lib
    lib = _lib.load()
    var = p['bn_var'] - (1e-5 if defect == 'fold without eps' else 0.0)
    mean = torch.zeros_like(p['bn_mean']) if defect == 'fold without the mean' else p['bn_mean']
    args = [p['weight'], p['bias'], p['bn_weight'], p['bn_bias'], mean, var.float()]
    args = [a.contiguous().numpy() for a in args]
    taps, bias = np.zeros((K, DIM), F32), np.zeros(DIM, F32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    assert lib.some_pack_dwconv_bn(*[ptr(a) for a in args], DIM, K, ptr(taps), ptr(bias)) == 0
    return taps, bias


DW_FRAMES = [1, 2, 16, 31, 40]


# ------------------------------------------------------------------------------------------------ restatements
def test_exact64_restates_the_torch_modules():
    torch.manual_seed(0)
    x, g, b = ln_data('iid', 64)
    ln = torch.nn.LayerNorm(DIM, eps=1e-5).double()
    with torch.no_grad():
        ln.weight.copy_(g.double()), ln.bias.copy_(b.double())
        torch.testing.assert_close(ln_exact64(x, g, b), ln(x.double()), atol=1e-13, rtol=1e-13)
        w, bias = rf.head_params('saturate', gen('head'))
        lin = torch.nn.Linear(DIM, 1).double()
        lin.weight.copy_(w.double()[None]), lin.bias.fill_(bias)
        torch.testing.assert_close(rf.head_exact64(x, g, b, w, bias), torch.sigmoid(lin(ln(x.double())))[:, 0],
                                   atol=1e-13, rtol=1e-12)
        s, q = rf.stats_exact64(x)
        torch.testing.assert_close(s, x.double().sum(1), atol=0, rtol=1e-14)
        for name in ('iid_synthetic', 'iid_trained'):
            xx, cu, p, _, _, _ = dw_data(name, DW_FRAMES)
            conv = torch.nn.Conv1d(DIM, DIM, K, padding=rf.HALO, groups=DIM).double()
            conv.weight.copy_(p['weight'].double()[:, None]), conv.bias.copy_(p['bias'].double())
            bn = torch.nn.BatchNorm1d(DIM, eps=1e-5).double().eval()
            bn.weight.copy_(p['bn_weight'].double()), bn.bias.copy_(p['bn_bias'].double())
            bn.running_mean.copy_(p['bn_mean'].double()), bn.running_var.copy_(p['bn_var'].double())
            ex = rf.dw_exact64(xx, cu, p)
            for i in range(len(cu) - 1):
                clip = xx[cu[i]:cu[i + 1]].double().t()[None]
                ref = torch.nn.SiLU()(bn(conv(clip)))[0].t()
                torch.testing.assert_close(ex[cu[i]:cu[i + 1]], ref, atol=1e-12, rtol=1e-12)


@pytest.mark.parametrize('stats', ['synthetic', 'trained'])
def test_dw_kernel64_from_the_project_folds_within_the_fold_bound(stats):
    """the C fold and weights.checkpoint_block give the same fp32 operands, and kernel64 on them is within
    dw_fold_bound of exact64 (the unfolded BatchNorm); the bound is not loose by orders of magnitude"""
    from some_b200 import synth, weights
    name = 'iid_synthetic' if stats == 'synthetic' else 'iid_trained'
    x, cu, p, taps, bias, _ = dw_data(name, DW_FRAMES)
    sd = synth.fabricate_state_dict(synth.named_config('two_head'))
    pre = 'model.cf_lay.0.att1'
    sd[f'{pre}.conv.depthwise_conv.weight'] = p['weight'][:, None]
    sd[f'{pre}.conv.depthwise_conv.bias'] = p['bias']
    for k, v in (('weight', 'bn_weight'), ('bias', 'bn_bias'), ('running_mean', 'bn_mean'), ('running_var', 'bn_var')):
        sd[f'{pre}.conv.norm.{k}'] = p[v]
    blk = weights.checkpoint_block(sd, pre)
    assert np.array_equal(blk.w_dw.float().numpy(), taps) and np.array_equal(blk.b_dw.float().numpy(), bias)
    _, y = rf.dw_kernel64(x, cu, torch.from_numpy(taps), torch.from_numpy(bias))
    r = abs_ratio(y, rf.dw_exact64(x, cu, p), rf.dw_fold_bound(x, cu, torch.from_numpy(taps), torch.from_numpy(bias)))
    print(f'dwconv fold ({stats} BatchNorm statistics): kernel64 vs exact64 err/fold bound max {float(r.max()):.3g}')
    assert float(r.max()) <= 1.0 and float(r.max()) > 1e-3


def test_regimes_are_what_they_claim():
    x = rows('dc', 64, gen('check'))
    assert float((x.double().mean(1).abs() / x.double().std(1)).min()) > 2 ** 15
    x = rows('outlier', 512, gen('check'))
    assert sorted(int(i) for i in (x == rf.OUTLIER).nonzero()[:, 1]) == list(range(DIM))
    x = rows('const15', 64, gen('check'))
    k = x[:, 0].double() / torch.exp2(torch.floor(torch.log2(x[:, 0].double().abs().clamp_min(1e-30))) - 14)
    assert bool((k == k.round()).all())
    x, g, b = ln_data('saturate', 256)
    w, bias = rf.head_params('saturate', gen('ln', 'saturate', 0))
    z = ln_exact64(x, g, b) @ w.double() + bias
    assert float(z.min()) < -40 and float(z.max()) > 40
    x, cu, p, taps, bias, _ = dw_data('span', [200])
    a, _ = rf.dw_kernel64(x, cu, torch.from_numpy(taps), torch.from_numpy(bias))
    assert float(a.min()) < -19 and float(a.max()) > 19 and float((a < -8.6).double().mean()) > 0.2
    x, cu, p, taps, bias, _ = dw_data('huge', [200])
    a, _ = rf.dw_kernel64(x, cu, torch.from_numpy(taps), torch.from_numpy(bias))
    assert float(a.abs().max()) > 2 ** 19
    x, cu, *_ = dw_data('ramp', [200])
    assert bool((x[1:] != x[:-1]).all())


# ------------------------------------------------------------------------------------------------ the bounds hold
LN_VARIANTS = list(itertools.product(ORDERS, ORDERS, (-2, 0, 2)))


def test_layernorm_bound_holds_for_emulated_kernel():
    worst = worst16 = 0.0
    for name in ROW_REGIMES:
        x, g, b = ln_data(name)
        ref, e = ln_bound(x, g, b)
        for lo, fo, ru in LN_VARIANTS:
            y = emulate_ln(x.numpy(), g.numpy(), b.numpy(), lo, fo, ru)
            r = float(abs_ratio(torch.from_numpy(y), ref, e).max())
            rb = float(gap_ratio(torch.from_numpy(bf16_rne(y)), ref, e).max())
            assert r <= 1.0 and rb <= 1.0, (name, lo, fo, ru, r, rb)
            if name == 'const15':
                assert np.array_equal(y, np.broadcast_to(b.numpy(), y.shape)), 'constant rows: output is not beta'
            worst, worst16 = max(worst, r), max(worst16, rb)
        print(f'layernorm {name}: largest emulated err/bound so far {worst:.3g} (fp32), {worst16:.3g} (bf16 gap)')
    print(f'== layernorm: largest emulated err/bound {worst:.3g} (fp32), {worst16:.3g} (bf16 gap) over {len(LN_VARIANTS)} variants')


def test_bound_head_bound_holds_for_emulated_kernel():
    worst = 0.0
    for name in HEAD_REGIMES:
        x, g, b = ln_data(name)
        w, bias = rf.head_params(name, gen('ln', name, 0))
        ref, e = rf.head_bound(x, g, b, w, bias)
        for (lo, fo, ru), eu in itertools.product(LN_VARIANTS[::2], (-2, 0, 2)):
            s = emulate_head(x.numpy(), g.numpy(), b.numpy(), w.numpy(), bias, lo, fo, ru, eu)
            r = float(abs_ratio(torch.from_numpy(s), ref, e).max())
            assert r <= 1.0, (name, lo, fo, ru, eu, r)
            worst = max(worst, r)
    print(f'== bound head: largest emulated err/bound {worst:.3g}')


def test_row_stats_bound_holds_for_emulated_kernel():
    worst = 0.0
    for name in ROW_REGIMES:
        x, _, _ = ln_data(name)
        s64, q64 = rf.stats_exact64(x)
        es, eq = rf.stats_bound(x)
        for lo, fo in itertools.product(ORDERS, ORDERS):
            s, q = emulate_stats(x.numpy(), lo, fo)
            r = max(float(abs_ratio(torch.from_numpy(s), s64, es).max()), float(abs_ratio(torch.from_numpy(q), q64, eq).max()))
            assert r <= 1.0, (name, lo, fo, r)
            worst = max(worst, r)
    print(f'== row stats: largest emulated err/bound {worst:.3g}')


def test_dwconv_bound_holds_for_emulated_kernel():
    worst = 0.0
    for name in DW_REGIMES:
        x, cu, p, taps, bias, _ = dw_data(name, DW_FRAMES)
        tt, bt = torch.from_numpy(taps), torch.from_numpy(bias)
        ref, e = rf.dw_bound(x, cu, tt, bt)
        ex = rf.dw_exact64(x, cu, p)
        ef = rf.dw_fold_bound(x, cu, tt, bt)
        for order, tr in itertools.product(ORDERS, (-TANH_REL, 0.0, TANH_REL)):
            y = torch.from_numpy(emulate_dw(x.numpy(), cu, taps, bias, order, tr))
            r = float(gap_ratio(y, ref, e).max())
            rx = float(gap_ratio(y, ex, e + ef).max())
            assert r <= 1.0 and rx <= 1.0, (name, order, tr, r, rx)
            worst = max(worst, r, rx)
        print(f'dwconv {name}: largest emulated err/bound so far {worst:.3g}')
    print(f'== dwconv: largest emulated err/bound {worst:.3g}')


# ------------------------------------------------------------------------------------------------ power
LN_DEFECTS = ['one-pass variance', '/511', 'eps outside the root', 'eps 1e-6', 'lane dropped from the mean',
              'gamma/beta permuted in a lane']


@pytest.mark.parametrize('defect', LN_DEFECTS)
def test_layernorm_planted_defect_breaks_the_bound(defect):
    best = (0.0, None)
    for name in ROW_REGIMES:
        x, g, b = ln_data(name)
        ref, e = ln_bound(x, g, b)
        y = emulate_ln(x.numpy(), g.numpy(), b.numpy(), defect=defect)
        r = float(abs_ratio(torch.from_numpy(y), ref, e).max())
        best = max(best, (r, name))
    print(f'layernorm defect {defect}: err/bound {best[0]:.3g} ({best[1]})')
    assert best[0] > 2.0, (defect, best)


@pytest.mark.parametrize('defect', ['sigmoid(-z)', 'bias dropped'])
def test_bound_head_planted_defect_breaks_the_bound(defect):
    best = (0.0, None)
    for name in HEAD_REGIMES:
        x, g, b = ln_data(name)
        w, bias = rf.head_params(name, gen('ln', name, 0))
        ref, e = rf.head_bound(x, g, b, w, bias)
        s = emulate_head(x.numpy(), g.numpy(), b.numpy(), w.numpy(), bias, defect=defect)
        best = max(best, (float(abs_ratio(torch.from_numpy(s), ref, e).max()), name))
    print(f'bound head defect {defect}: err/bound {best[0]:.3g} ({best[1]})')
    assert best[0] > 2.0, (defect, best)


@pytest.mark.parametrize('defect', ['q of centred values', 'lane dropped'])
def test_row_stats_planted_defect_breaks_the_bound(defect):
    best = (0.0, None)
    for name in ROW_REGIMES:
        x, _, _ = ln_data(name)
        s64, q64 = rf.stats_exact64(x)
        es, eq = rf.stats_bound(x)
        s, q = emulate_stats(x.numpy(), defect=defect)
        r = max(float(abs_ratio(torch.from_numpy(s), s64, es).max()), float(abs_ratio(torch.from_numpy(q), q64, eq).max()))
        best = max(best, (r, name))
    print(f'row stats defect {defect}: err/bound {best[0]:.3g} ({best[1]})')
    assert best[0] > 2.0, (defect, best)


DW_DEFECTS = ['flipped taps', 'halo 14', 'halo 16', 'neighbour rows as padding', 'fold without eps', 'fold without the mean',
              'bias dropped', 'bf16 truncation']


@pytest.mark.parametrize('defect', DW_DEFECTS)
def test_dwconv_planted_defect_breaks_the_bound(defect):
    """against exact64 within the kernel bound plus the fold bound, as tests/test_gpu_rowwise_f64.py checks the kernel"""
    best = (0.0, None)
    for name in DW_REGIMES:
        x, cu, p, taps, bias, pad = dw_data(name, DW_FRAMES)
        tt, bt = torch.from_numpy(taps), torch.from_numpy(bias)
        _, e = rf.dw_bound(x, cu, tt, bt)
        e = e + rf.dw_fold_bound(x, cu, tt, bt)
        if defect.startswith('fold'):
            taps, bias = pack_fold(p, defect)
        y = torch.from_numpy(emulate_dw(x.numpy(), cu, taps, bias, defect=defect, pad_rows=pad))
        best = max(best, (float(gap_ratio(y, rf.dw_exact64(x, cu, p), e).max()), name))
    print(f'dwconv defect {defect}: err/bound {best[0]:.3g} ({best[1]})')
    assert best[0] > 2.0, (defect, best)

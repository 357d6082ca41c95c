"""The float64 attention model and bound of tests/golden/attention_f64.py, without a GPU:

* exact64 is F.scaled_dot_product_attention in float64, and kernel64 lies within the loose bound of it;
* the bound holds for an fp32 emulation of some_attention_varlen's arithmetic (csrc/attention_tc.cu) written below, on every
  data regime and clip lengths up to 2584, with the summation order of S and P.V forward, reversed or shuffled, the
  accumulations rounding to nearest or truncating, and ex2 perturbed by +-2^-22;
* the bound has power: each planted defect of the emulation (the last key masked, a key of the next clip read, a tile
  short, O or l not rescaled, P truncated, the tile maximum over half the keys, one quad lane's l lost, V one column off)
  moves some output by more than twice the bound, so a kernel with it fails tests/test_gpu_attention_f64.py.  Each
  defect also reports whether the 2e-2 tolerance against fp32 SDPA, the kernel's only check before these tests, caught it.

Run with -s to see the ratios."""
import pathlib
import sys
import zlib

import numpy as np
import pytest
import torch

HERE = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / 'golden'))

from attention_f64 import (BN, C, DH, OUTLIER_K, REGIMES, bf16_rn, bound, exact64, heads, kernel64,  # noqa: E402
                           loose_bound, model_heads, outlier_keys, regime)


def gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def clip_data(name, t, seed=0):
    """qkv of one clip of a regime and the first row of the clip after it (a different draw of the same regime)"""
    qkv = regime(name, t, gen(name, t, seed))
    nxt = regime(name, max(t, 1), gen(name, t, seed, 'next'))[:1]
    return qkv, nxt


# ------------------------------------------------------------------------------------------------ the kernel in fp32
def r32(x, trunc=False):
    """float64 -> the nearest fp32 (or the fp32 toward zero), as float64"""
    f = x.float().double()
    if trunc:
        over = f.abs() > x.abs()
        f = torch.where(over, torch.nextafter(f.float(), torch.zeros_like(f.float())).double(), f)
    return f


def bf16_tz(x):
    """non-negative float64 x rounded down to a bf16 value"""
    _, e = torch.frexp(x)
    sp = torch.ldexp(torch.ones_like(x), e.clamp_min(-125) - 8)
    return torch.floor(x / sp) * sp


def ex2(x, rel):
    """ex2.approx.ftz: the fp32 of 2^x, moved by rel, results below 2^-126 flushed to zero"""
    y = r32(r32(torch.exp2(x)) * (1 + rel))
    return torch.where(y < 2.0 ** -126, torch.zeros_like(y), y)


def emulate(q, k, v, order='fwd', trunc=False, ex2_rel=0.0, defect=None, nxt=None, seed=0):
    """some_attention_varlen on one head in fp32: q [R, 64] (any R of the clip's query rows), k, v [T, 64], float64 of bf16
    values -> bf16 output [R, 64] (float64).
    order: 'fwd', 'rev' or 'rand', the order of the 64 terms of each score and of each tile's 64 P v products; trunc: those
    accumulations and the lane sums truncate instead of rounding to nearest.  nxt = (k, v) [1, 64] of the next clip's first
    row and the next head's v [T, 1], for the defects that read them."""
    r, t = q.shape[0], k.shape[0]
    perm = {'fwd': list(range(DH)), 'rev': list(range(DH - 1, -1, -1)),
            'rand': torch.randperm(DH, generator=gen('order', seed)).tolist()}[order]
    keys_k, keys_v = k, v
    if defect == 'next clip key':
        keys_k, keys_v = torch.cat([k, nxt[0]]), torch.cat([v, nxt[1]])
    if defect == 'V one column off':
        keys_v = torch.cat([v[:, 1:], nxt[2]], 1)
    s = torch.zeros(r, keys_k.shape[0], dtype=torch.float64)
    for c in perm:
        s = r32(s + q[:, c:c + 1] * keys_k[:, c][None, :], trunc)
    nt = -(-t // BN)
    if defect == 'tile short':
        nt -= 1
    m = torch.full((r, 1), -np.inf, dtype=torch.float64)
    lanes = torch.zeros(r, 4, dtype=torch.float64)
    o = torch.zeros(r, DH, dtype=torch.float64)
    for j in range(nt):
        valid = min(BN, t - j * BN) - (defect == 'last key masked' and j == nt - 1)
        if defect == 'next clip key' and j == nt - 1:
            valid += 1
        sc = torch.full((r, BN), -np.inf, dtype=torch.float64)
        sc[:, :valid] = s[:, j * BN:j * BN + valid]
        mx = sc[:, :BN // 2].amax(1, keepdim=True) if defect == 'half tile max' else sc.amax(1, keepdim=True)
        m_new = torch.maximum(m, mx)
        alpha = ex2(r32(r32(m - m_new) * C), ex2_rel)
        alpha = torch.where(torch.isnan(alpha), torch.zeros_like(alpha), alpha)    # -inf - finite on the first tile
        mc = r32(m_new * C)
        p = ex2(r32(sc * C - mc), ex2_rel)                   # fmaf: one rounding of the exact s c - mc
        p = torch.where(sc == -np.inf, torch.zeros_like(p), p)
        pair = p.view(r, 8, 4, 2)                            # key 8 jj + 2 lane + e
        ts = torch.zeros(r, 4, dtype=torch.float64)
        for jj in range(8):
            ts = r32(ts + r32(pair[:, jj, :, 0] + pair[:, jj, :, 1], trunc), trunc)
        lanes = r32(ts + (lanes if defect == 'l not rescaled' else lanes * alpha))
        if not (defect == 'O not rescaled' and j == 1):
            o = r32(o * alpha)
        P = bf16_tz(p) if defect == 'P toward zero' else bf16_rn(p)
        vt = keys_v[j * BN:j * BN + valid]
        for i in perm:
            if i < valid:
                o = r32(o + P[:, i:i + 1] * vt[i][None, :], trunc)
        m = m_new
    if defect == 'quad lane lost':
        lt = r32(r32(lanes[:, 0] + lanes[:, 1]) + lanes[:, 2])
    else:
        lt = r32(r32(lanes[:, 0] + lanes[:, 1]) + r32(lanes[:, 2] + lanes[:, 3]))
    inv = r32(1.0 / lt)
    return bf16_rn(r32(o * inv[:, None]))


def ratios(got, want, b):
    """(max, rms) of |got - want| / b"""
    err = (got - want).abs()
    r = torch.nan_to_num(torch.where(err == 0, torch.zeros_like(err), err / b), nan=np.inf)
    return float(r.max()), float(r.square().mean().sqrt())


def sdpa32_caught(got, q, k, v):
    """does the 2e-2 tolerance against fp32 SDPA (the kernel's only check before these tests) reject got?"""
    ref = torch.nn.functional.scaled_dot_product_attention(q.float()[None], k.float()[None], v.float()[None])[0]
    return not torch.allclose(got.float(), ref, atol=2e-2, rtol=2e-2)


# ------------------------------------------------------------------------------------------------ restatement and model
@pytest.mark.parametrize('t', [1, 2, 65, 200, 1100])
def test_exact64_is_sdpa_and_kernel64_within_loose_bound(t):
    for name in REGIMES:
        qkv, _ = clip_data(name, t)
        cu = [0, t]
        ex = exact64(qkv, cu)
        q, k, v = heads(qkv)
        ref = torch.nn.functional.scaled_dot_product_attention(q[None], k[None], v[None])[0]
        torch.testing.assert_close(ex, ref.transpose(0, 1).reshape(t, -1), atol=1e-12, rtol=1e-12)
        md, = kernel64(qkv, cu)
        mx, rms = ratios(md.out(), ex, loose_bound(md))
        print(f'T={t} {name}: kernel64 vs exact64 err/loose bound max {mx:.3g} rms {rms:.3g}')
        assert mx <= 1.0, (name, t, mx)


def test_regimes_are_what_they_claim():
    """the outlier key sits at every key % 8, outside the first tile, more than 127 above every other score in the
    exponent; the ramp moves every row's maximum by more than 2^4 in the exponent on every whole tile; equal and zero_q
    give p = 1 exactly"""
    t = 1100
    pos = outlier_keys(t)
    assert sorted(i % 8 for i in pos) == list(range(8)) and min(pos) >= BN
    q, k, v = heads(regime('outlier', t, gen('check')))
    md = model_heads(q, k, v)
    for h, i in enumerate(pos):
        others = torch.cat([md.s[h, :, :i], md.s[h, :, i + 1:]], 1).amax(1)
        assert bool(((md.s[h, :, i] - others) * C > 127).all()) and bool((k[h, i] == OUTLIER_K).all())
    md = model_heads(*heads(regime('ramp', 17 * BN, gen('check'))))   # whole tiles: a short last one may not move it
    assert bool(((md.m[..., 1:] - md.m[..., :-1]) * C > 4).all()), 'the ramp regime does not move the maximum on every tile'
    for name in ('equal', 'zero_q'):
        md = model_heads(*heads(regime(name, 200, gen('check'))))
        assert bool((md.p == 1).all()), name


# ------------------------------------------------------------------------------------------------ the bound holds
VARIANTS = [dict(order='fwd'), dict(order='rev', trunc=True, ex2_rel=2.0 ** -22),
            dict(order='rand', ex2_rel=-2.0 ** -22), dict(order='rand', trunc=True, ex2_rel=2.0 ** -22)]


@pytest.mark.parametrize('t', [1, 2, 63, 64, 65, 129, 200, 1100, 2584])
def test_bound_holds_for_emulated_kernel(t):
    """every regime, one head each (a different head per regime), all variants up to T = 200; above that a quarter (T = 1100)
    or an eighth (T = 2584) of the query rows, and two variants or one, so the file stays quick"""
    rows = torch.arange(0, t, 1 if t <= 200 else 4 if t <= 1100 else 8)
    worst = 0.0
    for n, name in enumerate(REGIMES):
        qkv, _ = clip_data(name, t)
        q, k, v = heads(qkv)
        h = n % 8
        md = model_heads(q[h:h + 1], k[h:h + 1], v[h:h + 1])
        b = merge_rows(bound(md), rows)
        want = md.o[0][rows]
        variants = VARIANTS if t <= 200 else VARIANTS[n % 2::2] if t <= 1100 else [VARIANTS[n % 4]]
        for i, var in enumerate(variants):
            got = emulate(q[h][rows], k[h], v[h], seed=i, **var)
            mx, rms = ratios(got, want, b)
            print(f'T={t} {name} head {h} {var}: emulation err/bound max {mx:.3g} rms {rms:.3g}')
            assert mx <= 1.0, (t, name, var, mx)
            worst = max(worst, mx)
    print(f'T={t}: largest emulation err/bound {worst:.3g}')


def merge_rows(b, rows):
    return b[rows][:, :DH]


# ------------------------------------------------------------------------------------------------ power
DEFECTS = ['last key masked', 'next clip key', 'tile short', 'O not rescaled', 'l not rescaled', 'P toward zero',
           'half tile max', 'quad lane lost', 'V one column off']


@pytest.mark.parametrize('defect', DEFECTS)
def test_planted_defect_breaks_the_bound(defect):
    """a kernel with the defect computes the defective result plus its rounding; it is caught where the defect moves an
    output by more than twice the bound.  Required on at least one regime at T = 65, 128 or 200 (128 for a tile short,
    which needs T % 64 == 0; 65 and 200 for the next clip's key, which needs T % 64 != 0)"""
    lengths = {'tile short': [128], 'next clip key': [65, 200]}.get(defect, [65, 128, 200])
    best = (0.0, None, None)
    caught = {}
    for t in lengths:
        for name in REGIMES:
            qkv, nxt = clip_data(name, t)
            q, k, v = heads(qkv)
            _, kn, vn = heads(nxt)
            md = model_heads(q[:1], k[:1], v[:1])
            got = emulate(q[0], k[0], v[0], defect=defect, nxt=(kn[0], vn[0], v[1][:, :1]))
            mx, _ = ratios(got, md.o[0], bound(md)[:, :DH])
            if mx > best[0]:
                best = (mx, name, t)
            caught.setdefault(name, []).append(sdpa32_caught(got, q[0], k[0], v[0]))
    today = [n for n, c in caught.items() if any(c)]
    print(f'{defect}: err/bound {best[0]:.3g} ({best[1]}, T={best[2]}); the 2e-2 check against fp32 SDPA catches it on '
          f'{today or "no regime"}, on the peaky data it ran on: {any(caught["peaky"])}')
    assert best[0] > 2.0, (defect, best)

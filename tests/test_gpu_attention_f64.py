"""some_attention_varlen (csrc/attention_tc.cu), through the C ABI, against the float64 model of its arithmetic and the
float64 attention of tests/golden/attention_f64.py, computed on the device:

* bound: every output within bound() of kernel64 and within bound() + loose_bound() of exact64, for one var-len launch of
  clips straddling the 64-key tiles, the 128-query CTAs and the 64-row consumer warpgroups, two groups of different data,
  every data regime;
* bits: each clip alone equals its rows of the batch, groups = 1 equals each group of groups = 2, a larger max_frames
  changes nothing, and filler rows in front (another row alignment of every tile) leave the bits as they are;
* fences: qkv is a view with NaN rows after M, so a read past M shows up as NaN through 0 * NaN in P.V; rows inside M that
  no clip owns hold 2^14, which would swamp any score they took part in (the last key tile of the last clip loads them
  and masks them, so they must be finite); out is prefilled with a sentinel that every out-of-clip row keeps;
* benchmark scale: 64 clips of 2584 frames in two groups, many CTA waves.

Run with -s to see max and rms err / bound per case."""
import ctypes as C
import pathlib
import sys
import zlib

import numpy as np
import pytest
import torch

HERE = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / 'golden'))

from attention_f64 import REGIMES, bound, exact64, heads, loose_bound, model_heads, regime  # noqa: E402
from some_b200 import _lib  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = 'cuda'
BF16 = torch.bfloat16
FRAMES = [1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 1100, 2584]
GUARD = 3                      # sentinel rows behind out, NaN rows behind qkv
LOOSE = 3                      # rows of qkv / out inside M that no clip owns
LOOSE_VALUE = 2.0 ** 14        # what those rows of qkv hold
SENTINEL = -3072.0             # exact in bf16
NAN = float('nan')


@pytest.fixture(scope='module')
def lib():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    return _lib.load()


def seeded(*key):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


def cumsum(frames, start=0):
    return [start] + list(np.cumsum(frames) + start)


def batch(name, frames, gen):
    """qkv of clips of one regime, end to end, float32 on the device"""
    return torch.cat([regime(name, t, gen, DEV) for t in frames])


def fenced_qkv(x, loose=0):
    """bf16 view [rows + loose] of x with `loose` rows of LOOSE_VALUE after it and GUARD NaN rows behind the view"""
    buf = torch.full((x.shape[0] + loose + GUARD, 1536), NAN, dtype=BF16, device=DEV)
    buf[:x.shape[0]] = x
    buf[x.shape[0]:x.shape[0] + loose] = LOOSE_VALUE
    return buf[:x.shape[0] + loose]


def attention(lib, qkv, cu, max_frames=None):
    """one launch, groups = len(qkv), qkv views of M rows; returns each group's out [M, 512], taken from a sentinel buffer
    of M + GUARD rows whose out-of-clip rows are checked to be untouched"""
    m = qkv[0].shape[0]
    bufs = [torch.full((m + GUARD, 512), SENTINEL, dtype=BF16, device=DEV) for _ in qkv]
    outs = [b[:m] for b in bufs]
    cu_d = torch.tensor(cu, dtype=torch.int32, device=DEV)
    a = _lib.AttnArgs()
    a.qkv, a.out = _lib.pair(*qkv), _lib.pair(*outs)
    a.groups, a.B, a.M = len(qkv), len(cu) - 1, m
    a.cu_frames, a.max_frames = cu_d.data_ptr(), max_frames or int(np.diff(cu).max())
    _lib.check(lib.some_attention_varlen(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
               'some_attention_varlen')
    torch.cuda.synchronize()
    for i, buf in enumerate(bufs):
        kept = torch.ones(buf.shape[0], dtype=torch.bool, device=DEV)
        for b in range(len(cu) - 1):
            kept[cu[b]:cu[b + 1]] = False
        assert bool((buf[kept] == SENTINEL).all()), f'group {i}: a store landed outside the clips\' rows'
        assert not bool(torch.isnan(buf[~kept].float()).any()), f'group {i}: NaN in a clip\'s rows'
    return outs


def check_bound(label, err, b):
    """err <= b elementwise; prints and returns max and rms of err / b"""
    r = torch.where(err == 0, torch.zeros_like(err), err / b)
    mx, rms = r.max().item(), r.square().mean().sqrt().item()
    print(f'{label}: err/bound max {mx:.3g} rms {rms:.3g}', flush=True)
    assert mx <= 1.0, f'{label}: error {mx:.3g} x its bound at {np.unravel_index(int(r.argmax()), tuple(r.shape))}'
    return mx, rms


def check_clip(label, out, qkv_clip):
    """the kernel's rows of one clip against kernel64 (bound) and exact64 (bound + loose bound)"""
    md = model_heads(*heads(qkv_clip))
    got = out.double()
    b = bound(md)
    r = check_bound(label, (got - md.out()).abs(), b)
    check_bound(label + ' vs exact64', (got - exact64(qkv_clip, [0, qkv_clip.shape[0]])).abs(), b + loose_bound(md))
    return r


def bits(t):
    return t.view(torch.int16)


def assert_bitwise(label, got, want):
    bad = bits(got) != bits(want)
    assert not bool(bad.any()), (f'{label}: {int(bad.sum())} of {bad.numel()} elements differ, first at '
                                 f'{tuple(int(i) for i in bad.nonzero()[0])}')


# ------------------------------------------------------------------------------------------------------------ bound
@pytest.mark.parametrize('name', REGIMES)
def test_bound_every_clip_length(lib, name):
    """one var-len launch of FRAMES, two groups of different draws, LOOSE rows inside M that no clip owns"""
    cu = cumsum(FRAMES)
    x = [batch(name, FRAMES, seeded('bound', name, g)) for g in range(2)]
    outs = attention(lib, [fenced_qkv(xi, LOOSE) for xi in x], cu)
    worst = {}
    for g in range(2):
        for b, t in enumerate(FRAMES):
            r = check_clip(f'{name} group {g} T={t}', outs[g][cu[b]:cu[b + 1]], x[g][cu[b]:cu[b + 1]])
            worst[g] = tuple(max(u, w) for u, w in zip(worst.get(g, (0.0, 0.0)), r))
    for g, (mx, rms) in worst.items():
        print(f'== {name} group {g}: largest err/bound max {mx:.3g}, largest rms {rms:.3g} over {len(FRAMES)} clips')


# ------------------------------------------------------------------------------------------------------------ bits
def test_bits_alone_groups_max_frames_and_filler(lib):
    cu = cumsum(FRAMES)
    x = [batch(name, FRAMES, seeded('bits', name)) for name in ('spread', 'peaky')]
    q = [fenced_qkv(xi) for xi in x]
    ref = attention(lib, q, cu)
    for b, t in enumerate(FRAMES):
        alone = attention(lib, [fenced_qkv(xi[cu[b]:cu[b + 1]]) for xi in x], [0, t])
        for g in range(2):
            assert_bitwise(f'clip {b} (T={t}) group {g} alone', alone[g], ref[g][cu[b]:cu[b + 1]])
    for g in range(2):
        assert_bitwise(f'group {g} in a one-group launch', attention(lib, [q[g]], cu)[0], ref[g])
    wide = attention(lib, q, cu, max_frames=max(FRAMES) + 300)
    for g in range(2):
        assert_bitwise(f'group {g} with max_frames {max(FRAMES) + 300}', wide[g], ref[g])
    for r0 in (1, 7, 64, 127):
        filler = [fenced_qkv(torch.cat([regime('peaky', r0, seeded('filler', r0, g), DEV), xi])) for g, xi in enumerate(x)]
        moved = attention(lib, filler, [0] + cumsum(FRAMES, r0))
        for g in range(2):
            assert_bitwise(f'group {g} behind {r0} filler rows', moved[g][r0:], ref[g])


# ------------------------------------------------------------------------------------------------------------ scale
def test_benchmark_scale(lib):
    """64 clips x 2584 frames (the benchmark's 30 s chunk) in two groups: the first, a middle and the last clip of each
    group against the bound, every row finite"""
    frames = [2584] * 64
    cu = cumsum(frames)
    x = [batch(name, frames, seeded('scale', name)) for name in ('spread', 'peaky')]
    outs = attention(lib, [fenced_qkv(xi, LOOSE) for xi in x], cu)
    for g in range(2):
        assert bool(torch.isfinite(outs[g][:cu[-1]].float()).all()), f'group {g}: a non-finite output'
        for b in (0, 31, 63):
            check_clip(f'64 x 2584 group {g} clip {b}', outs[g][cu[b]:cu[b + 1]], x[g][cu[b]:cu[b + 1]])

"""Every epilogue of some_gemm (csrc/gemm.cu) against the kernel's own fp32 accumulator, and that accumulator against float64.

The *twin* of an epilogue is SOME_EPI_BIAS_F32 run on the same A, W and bias with ld_out = N.  Its direct stores give
v = acc + bias exactly as every epilogue sees it before its activation: the mainloop and the bias loop of epilogue_tile are
shared by all instantiations.  The relations below therefore hold whatever the tensor cores' accumulation order or
rounding is, provided the mainloop gives the same fp32 accumulator for a row and column whatever the epilogue, tile
position or launch; the width test checks that across columns, rows and groups.

* the twin against float64: a worst-case bound valid for any summation order, and an rms bound;
* every epilogue against its twin: bit for bit where the epilogue rounds once (bf16 stores, the residual fmaf, the
  LayerNorm producers' bf16 copy), within bounds built from the documented errors of tanh.approx, ex2.approx and rsqrtf
  where it approximates;
* every call shape of csrc/forward.cu in both launch sequences, two groups of different data, M in {1, 63, 64, 65, 129}
  and one M with at least three tiles per SM;
* fences: outputs prefilled with NaN, A and W passed as views with NaN rows behind them, sentinel rows (and columns)
  around every output, head bias padded with NaN in one run and +1e30 in another.

Every tolerance-based check prints the max and rms of err / bound (run with -s to see them)."""
import ctypes as C
import math
import zlib

import numpy as np
import pytest
import torch

from some_b200 import _lib

pytestmark = pytest.mark.gpu

DEV = 'cuda'
U = 2.0 ** -24                 # fp32 unit roundoff (round to nearest)
EPS_TANH = 2.0 ** -10.987      # tanh.approx.f32: maximum relative error (PTX ISA)
EPS_EX2 = 2.0 ** -22           # ex2.approx.f32: maximum relative error (PTX ISA)
GUARD = 3                      # sentinel rows behind every output
SENTINEL = -3072.0             # exact in bf16 and fp32
NAN = float('nan')
BF16, F32 = torch.bfloat16, torch.float32

E = _lib
GLU_EPIS = (E.EPI_GLU_BF16, E.EPI_GLU_RESID_F32, E.EPI_GLU_RESID_F32_LN, E.EPI_LN_GLU_BF16)
RESID_EPIS = (E.EPI_RESID_F32, E.EPI_RESID_F32_LN, E.EPI_GLU_RESID_F32, E.EPI_GLU_RESID_F32_LN)
LN_CONSUMERS = (E.EPI_LN_STORE_BF16, E.EPI_LN_SILU_BF16, E.EPI_LN_GLU_BF16)
LN_PRODUCERS = (E.EPI_RESID_F32_LN, E.EPI_GLU_RESID_F32_LN)
HEADS = (E.EPI_BIAS_F32, E.EPI_SIGMOID_F32, E.EPI_SOFTMAX_F32)


@pytest.fixture(scope='module')
def lib():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    return _lib.load()


def seeded(*key):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


# ------------------------------------------------------------------------------------------------------------ launching
def gemm(lib, epi, A, W, out, bias=None, resid=None, alpha=1.0, ln_s=None, stats=None, parts=0, out_bf16=None):
    """One some_gemm launch.  A, W, out and the optional per-group arguments are lists with one tensor per group; M, K and
    lda come from A[0], N from W[0], ld_out from out[0]."""
    none = (C.c_void_p * 2)()
    g = _lib.GemmArgs()
    g.A, g.W, g.out = _lib.pair(*A), _lib.pair(*W), _lib.pair(*out)
    g.bias = _lib.pair(*bias) if bias is not None else none
    g.resid = _lib.pair(*resid) if resid is not None else none
    g.ln_s = _lib.pair(*ln_s) if ln_s is not None else none
    g.ln_stats = _lib.pair(*stats) if stats is not None else none
    g.out_bf16 = _lib.pair(*out_bf16) if out_bf16 is not None else none
    g.groups, (g.M, g.K), g.N = len(A), A[0].shape, W[0].shape[0]
    g.lda, g.ld_out = A[0].stride(0), out[0].stride(0)
    g.epilogue, g.alpha, g.ln_parts = epi, alpha, parts
    _lib.check(lib.some_gemm(C.byref(g), C.c_void_p(torch.cuda.current_stream().cuda_stream)), 'some_gemm')
    torch.cuda.synchronize()


def operand(t, ld=None):
    """bf16 view of t [rows, K] inside a buffer with NaN rows behind it (and NaN columns past K when ld > K): the tensor
    maps must zero-fill the rows past M (A) or N (W), not read them."""
    rows, k = t.shape
    buf = torch.full((rows + 5, ld or k), NAN, dtype=BF16, device=DEV)
    buf[:rows, :k] = t
    return buf[:rows, :k]


def fenced(rows, cols, dtype, fill, ld=None):
    """(buffer, view): the view [:rows, :cols] holds fill; GUARD rows behind it and the columns past cols (ld > cols) hold
    SENTINEL."""
    buf = torch.full((rows + GUARD, ld or cols), SENTINEL, dtype=dtype, device=DEV)
    buf[:rows, :cols] = fill
    return buf, buf[:rows, :cols]


def assert_fenced(buf, view, what):
    rows, cols = view.shape
    rest = buf.clone()
    rest[:rows, :cols] = SENTINEL
    assert bool((rest == SENTINEL).all()), f'{what}: a store landed outside [:M, :out_cols]'
    assert not bool(torch.isnan(view).any()), f'{what}: NaN left in [:M, :out_cols] (an element was never stored)'


def padded_bias(b, pad_value):
    """head bias: padded to a multiple of 32 floats (include/some_b200.h) with pad_value"""
    return torch.cat([b, b.new_full(((-b.numel()) % 32,), pad_value)])


def twin(lib, A, W, bias):
    """SOME_EPI_BIAS_F32 on the same operands with ld_out = N: v = acc + bias of every group (bias None: v = acc)."""
    m, n = A[0].shape[0], W[0].shape[0]
    outs = [fenced(m, n, F32, NAN) for _ in A]
    gemm(lib, E.EPI_BIAS_F32, A, W, [o for _, o in outs], bias=bias)
    for i, (buf, o) in enumerate(outs):
        assert_fenced(buf, o, f'twin group {i}')
    return [o.clone() for _, o in outs]


def glu_unpack(y):
    """inverse of weights.glu_pack_rows on the columns: packed [M, 2C] (32-column groups of 16 out | 16 gate) -> (out
    [M, C], gate [M, C])"""
    m, n = y.shape
    y = y.reshape(m, n // 32, 2, 16)
    return y[:, :, 0].reshape(m, n // 2), y[:, :, 1].reshape(m, n // 2)


def many_rows(n, groups=2):
    """an M whose launch has at least three tiles per SM (the last m-block ragged): every CTA runs several tiles, so the
    slab counters, ring phases and residual-load parities wrap inside a CTA"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    num_m = -(-3 * sms // (groups * -(-n // 256)))
    return 128 * (num_m - 1) + 91


# ------------------------------------------------------------------------------------------------------------ bounds
def check_bound(label, err, bound):
    """err <= bound elementwise; prints max and rms of err / bound"""
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    mx, rms = r.max().item(), r.square().mean().sqrt().item()
    print(f'{label}: err/bound max {mx:.3g} rms {rms:.3g}', flush=True)
    assert mx <= 1.0, f'{label}: error {mx:.3g} x its bound at {np.unravel_index(int(r.argmax()), tuple(r.shape))}'
    return rms


def assert_bitwise(label, got, want):
    bad = got != want
    assert not bool(bad.any()), (f'{label}: {int(bad.sum())} of {bad.numel()} elements differ, first at '
                                 f'{tuple(int(i) for i in bad.nonzero()[0])}')


def check_against_float64(label, v, A, W, b):
    """The accumulator is a sum of K exact products (bf16 x bf16 fits in fp32) plus the bias, K + 1 terms.  In any order,
    each term passes through at most K additions, and an fp32 addition that rounds to nearest or truncates is off by
    at most 2^-23 of its result, which is at most the sum S of the magnitudes of all terms.  So
    |v - y| <= ((1 + 2^-23)^K - 1) S <= (K + 1) 2^-23 S  (K 2^-23 < 2^-11 here).
    rms: if the K roundings were independent and centred, each at most 2^-24 S, their sum would have an rms of at most
    sqrt(K + 1) 2^-24 S, i.e. err / bound ~ 1 / (2 sqrt(K + 1)).  Allowed: 8 times that.  Not rigorous, but at K = 2048
    a dropped k-block or a single dropped product lands far above it while the worst case is loose."""
    k = A.shape[1]
    a, w = A.double(), W.double()
    y, s = a @ w.t(), a.abs() @ w.abs().t()
    if b is not None:
        bb = b[:W.shape[0]].double()
        y, s = y + bb, s + bb.abs()
    rms = check_bound(label + ' twin vs float64', (v.double() - y).abs(), (k + 1) * 2.0 ** -23 * s)
    assert rms <= 8 / (2 * math.sqrt(k + 1)), f'{label}: rms err/bound {rms:.3g} over 8x the random-walk estimate'


def half_ulp_bf16(x):
    """half the bf16 spacing at magnitude |x| (a bf16 store that rounds to nearest moves any |z| <= |x| by at most this)"""
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x), e - 9)


def bf16_bound(ref, e):
    """bound on |bf16(z) - ref| for any fp32 z with |z - ref| <= e"""
    return e + half_ulp_bf16(ref.abs() + e)


def silu_err(v):
    """SiLU through tanh.approx (silu_fast: h = v/2, fmaf(h, tanh(h), h)): |h| |tanh h| eps_tanh, doubled for margin.  Absolute:
    for large negative v the output is tiny and this error is not."""
    h = v.abs() / 2
    return h * torch.tanh(h) * 2 * EPS_TANH


def sigmoid_err(g):
    """sigmoid_fast = fmaf(0.5, tanh(g/2), 0.5): 0.5 |tanh(g/2)| eps_tanh, doubled for margin"""
    return 0.5 * torch.tanh(g.abs() / 2) * 2 * EPS_TANH


def expf_rel(x):
    """relative error of __expf(x) = ex2.approx(x * log2e_f32): ex2.approx (EPS_EX2, doubled for margin) plus the move of the
    exponent: the fp32 product rounds (U) and log2e_f32 is 1.34e-8 relative below log2(e), so e^x gains a factor
    e^(x d) with |d| < 7.3e-8 < 2^-23"""
    return 2 * EPS_EX2 + x.abs() * 2.0 ** -23


def fma32(a, alpha, c):
    """fp32 fmaf(a, alpha, c) for fp32 tensors a, c: one rounding of the exact value.  a * alpha is exact in float64; the
    float64 sum is rounded to fp32 by torch, and the one case where that is not the rounding of the exact value -- the
    float64 sum sits on an fp32 tie while the exact one does not -- is decided by the TwoSum error of the float64 sum."""
    p, c = a.double() * float(np.float32(alpha)), c.double()
    s = p + c
    bp = s - p
    err = (p - (s - bp)) + (c - bp)
    f = s.float()
    other = torch.nextafter(f, torch.where(s > f.double(), torch.full_like(f, math.inf), torch.full_like(f, -math.inf)))
    tie = ((f.double() + other.double()) / 2 == s) & (err != 0)
    up = torch.maximum(f, other)
    down = torch.minimum(f, other)
    return torch.where(tie, torch.where(err > 0, up, down), f)


def check_ln_stats(label, st, x, parts):
    """LayerNorm producers: slot j of ln_stats holds (sum x, sum x^2) of the row over its n = out_cols / parts columns of the
    kernel's own fp32 out.  Each term passes through at most n - 1 fp32 additions (the x^2 products are exact inside fmaf),
    so each sum is within n 2^-23 of the sum of its terms' magnitudes.  Slots past parts and rows past M stay NaN."""
    m, c = x.shape
    n = c // parts
    cols = x.double().reshape(m, parts, n)
    s, q = cols.sum(-1), (cols * cols).sum(-1)
    got = st[:m, :parts].double()
    check_bound(label + ' ln_stats sum x', (got[..., 0] - s).abs(), n * 2.0 ** -23 * cols.abs().sum(-1))
    check_bound(label + ' ln_stats sum x^2', (got[..., 1] - q).abs(), n * 2.0 ** -23 * q)
    assert bool(torch.isnan(st[:m, parts:]).all()) and bool(torch.isnan(st[m:]).all()), f'{label}: ln_stats written out of range'


def ln_folded(acc, st, parts, s_n, bias, k):
    """LayerNorm-folded consumers: float64 value of fmaf(fmaf(s_n, -mean, acc), rstd, b') from the kernel's own mean and rstd
    of the stats the test supplies, and the bound delta on how far the kernel's fp32 evaluation may lie from it.
    mean: the fp32 slot sums in the kernel's order, times 1/K (exact for K = 512).  The inner and the outer fmaf round once
    each (U); rstd: rsqrtf is within 2 ulp (2^-22 relative, CUDA programming guide), and the fmaf of the variance and the
    + eps round once each (2 U in the argument, U in the root), under 2^-21 together."""
    s, q = st[:, 0, 0], st[:, 0, 1]
    for i in range(1, parts):
        s, q = s + st[:, i, 0], q + st[:, i, 1]
    inv_k = float(np.float32(1.0) / np.float32(k))
    mean = (s * inv_k).double()
    var = (q.double() * inv_k - mean * mean).clamp_min(0.0)
    rstd = (var + float(np.float32(1e-5))).rsqrt()
    inner = acc.double() - s_n.double()[None, :] * mean[:, None]
    y = inner * rstd[:, None] + bias.double()[None, :]
    delta = 2 * U * y.abs() + inner.abs() * rstd[:, None] * (2.0 ** -21 + 2 * U)
    return y, delta


def check_glu(label, out, yo, yg, do=0.0, dg=0.0, resid=None):
    """out = bf16(yo * sigmoid_fast(yg)) (resid None) or fp32 resid + yo * sigmoid_fast(yg), with yo, yg known within do, dg.
    The sigmoid moves by at most dg / 4, and fp32 rounds twice in the product (sigmoid's fmaf and the multiply), once more
    in the residual add."""
    sg = torch.sigmoid(yg)
    ref = yo * sg
    e = do * (sg + dg / 4) + yo.abs() * dg / 4 + (yo.abs() + do) * (sigmoid_err(yg.abs() + dg) + 4 * U * (sg + dg / 4))
    if resid is None:
        check_bound(label, (out.double() - ref).abs(), bf16_bound(ref, e))
    else:
        ref = resid.double() + ref
        check_bound(label, (out.double() - ref).abs(), e + 2 * U * ref.abs())


def check_sigmoid_head(label, out, v):
    """1 / (1 + __expf(-v)): the exponential's relative error r moves sigmoid by sigma (1 - sigma) r, the add and the
    IEEE division round once each; 1 % for second-order terms"""
    v = v.double()
    s = torch.sigmoid(v)
    check_bound(label, (out.double() - s).abs(), 1.01 * (s * (1 - s) * expf_rel(v) + 2 * U * s) + 2.0 ** -126)


def check_softmax_head(label, out, v):
    """__expf(v - max) per column (the subtraction rounds: U |d| more in the exponent), an fp32 sum of n positive terms
    (relative (n - 1) U), one IEEE division and one multiply: out_i is within p_i (r_i + sum_j p_j r_j + (n + 1) U) of the
    exact p_i; 1 % for second-order terms, and 2^-126 for exponentials flushed to zero"""
    v = v.double()
    n = v.shape[1]
    p = torch.softmax(v, -1)
    r = expf_rel(v - v.max(-1, keepdim=True).values) + (v - v.max(-1, keepdim=True).values).abs() * U
    rel = r + (p * r).sum(-1, keepdim=True) + (n + 1) * U
    check_bound(label, (out.double() - p).abs(), 1.01 * p * rel + 2.0 ** -126)


# ------------------------------------------------------------------------------------------------------------ twin
@pytest.mark.parametrize('n', list(range(1, 257)) + [512])
def test_twin_against_float64_columns_rows_groups_and_heads(lib, n):
    """The twin at every head width and at N = 512: against float64; its first N columns against a launch at a wider N
    whose extra W rows are zeros; its rows against launches with r0 filler rows in front (another tile row, consumer
    warpgroup and swizzle phase); each group of the two-group launch against a one-group launch.  Then the sigmoid and
    softmax heads at the same N, their bias padded with NaN and with +1e30: the padding must not reach an output."""
    m, k = 200, 512
    gen = seeded('width', n)
    A0 = [torch.randn(m, k, device=DEV, generator=gen).to(BF16) for _ in range(2)]
    W0 = [(torch.randn(n, k, device=DEV, generator=gen) / k ** 0.5).to(BF16) for _ in range(2)]
    b0 = [torch.randn(n, device=DEV, generator=gen) for _ in range(2)]
    A, W = [operand(a) for a in A0], [operand(w) for w in W0]
    bias = [padded_bias(b, NAN) for b in b0]
    v = twin(lib, A, W, bias)
    for i in range(2):
        check_against_float64(f'N={n} K={k} group {i}', v[i], A0[i], W0[i], b0[i])

    wide = 256 * (-(-n // 256) + 1)
    Ww = [operand(torch.cat([w, w.new_zeros(wide - n, k)])) for w in W0]
    vw = twin(lib, A, Ww, [torch.cat([b, b.new_zeros(wide - n)]) for b in b0])
    for i in range(2):
        assert_bitwise(f'N={n} group {i}: columns of a launch at N={wide}', vw[i][:, :n], v[i])

    for r0 in (1, 7, 64, 127):
        filler = [operand(torch.cat([torch.randn(r0, k, device=DEV, generator=gen).to(BF16), a])) for a in A0]
        vs = twin(lib, filler, W, bias)
        for i in range(2):
            assert_bitwise(f'N={n} group {i}: rows behind {r0} filler rows', vs[i][r0:], v[i])

    for i in range(2):
        assert_bitwise(f'N={n}: group {i} alone', twin(lib, [A[i]], [W[i]], [bias[i]])[0], v[i])

    if n > 256:
        return
    for epi, check in ((E.EPI_SIGMOID_F32, check_sigmoid_head), (E.EPI_SOFTMAX_F32, check_softmax_head)):
        runs = []
        for pad in (NAN, 1e30):
            outs = [fenced(m, n, F32, NAN) for _ in range(2)]
            gemm(lib, epi, A, W, [o for _, o in outs], bias=[padded_bias(b, pad) for b in b0])
            for i, (buf, o) in enumerate(outs):
                assert_fenced(buf, o, f'N={n} epilogue {epi} group {i}')
            runs.append([o for _, o in outs])
        for i in range(2):
            assert_bitwise(f'N={n} epilogue {epi} group {i}: bias padding NaN vs +1e30', runs[1][i], runs[0][i])
            check(f'N={n} epilogue {epi} group {i}', runs[0][i], v[i])


# ------------------------------------------------------------------------------------------------------------ epilogues
# (id, epilogue, N, K, alpha, ln_parts): every some_gemm call of csrc/forward.cu, in both launch sequences, plus the
# residual epilogue at an alpha whose product with v is not exact (the ABI takes any alpha)
CASES = [
    ('in_proj', E.EPI_BIAS_F32, 512, 80, 1.0, 0),
    ('qkv', E.EPI_STORE_BF16, 1536, 512, 1.0, 0),
    ('ffn_w1', E.EPI_SILU_BF16, 2048, 512, 1.0, 0),
    ('out_proj', E.EPI_RESID_F32, 512, 512, 1.0, 0),
    ('ffn_w2', E.EPI_RESID_F32, 512, 2048, 0.5, 0),
    ('resid_alpha_0.3', E.EPI_RESID_F32, 512, 512, 0.3, 0),
    ('pw1', E.EPI_GLU_BF16, 1024, 512, 1.0, 0),
    ('glu_mix', E.EPI_GLU_RESID_F32, 1024, 512, 1.0, 0),
    ('out_proj_ln', E.EPI_RESID_F32_LN, 512, 512, 1.0, 0),
    ('ffn_w2_ln', E.EPI_RESID_F32_LN, 512, 2048, 0.5, 0),
    ('glu_mix_ln', E.EPI_GLU_RESID_F32_LN, 1024, 512, 1.0, 0),
    *[(f'qkv_ln{p}', E.EPI_LN_STORE_BF16, 1536, 512, 1.0, p) for p in (1, 4, 8)],
    *[(f'ffn_w1_ln{p}', E.EPI_LN_SILU_BF16, 2048, 512, 1.0, p) for p in (1, 4, 8)],
    *[(f'pw1_ln{p}', E.EPI_LN_GLU_BF16, 1024, 512, 1.0, p) for p in (1, 4, 8)],
    *[(f'head_{name}{n}', epi, n, 512, 1.0, 0) for n in (128, 129)
      for name, epi in (('logits', E.EPI_BIAS_F32), ('sigmoid', E.EPI_SIGMOID_F32), ('softmax', E.EPI_SOFTMAX_F32))],
]


def run_case(lib, case, m, gen, lda=None, ld_extra=0):
    """Runs one epilogue on two groups of different data with every fence in place and checks it against its twin."""
    name, epi, n, k, alpha, parts = case
    glu = epi in GLU_EPIS
    out_cols = n // 2 if glu else n
    ld = out_cols + ld_extra
    label = f'{name} M={m} N={n} K={k}'
    if epi in LN_CONSUMERS:
        x = [torch.randn(m, k, device=DEV, generator=gen) * 1.7 + 0.4 for _ in range(2)]
        A0 = [t.to(BF16) for t in x]
    else:
        A0 = [torch.randn(m, k, device=DEV, generator=gen).to(BF16) for _ in range(2)]
    W0 = [(torch.randn(n, k, device=DEV, generator=gen) / k ** 0.5).to(BF16) for _ in range(2)]
    b0 = [torch.randn(n, device=DEV, generator=gen) for _ in range(2)]
    A, W = [operand(a, lda) for a in A0], [operand(w) for w in W0]
    bias = [padded_bias(b, NAN) for b in b0]

    # the twin: acc + bias, or acc alone for the LayerNorm consumers (they apply the bias after the normalisation)
    v = twin(lib, A, W, None if epi in LN_CONSUMERS else bias)
    for i in range(2):
        check_against_float64(f'{label} group {i}', v[i], A0[i], W0[i], None if epi in LN_CONSUMERS else b0[i])
    if epi == E.EPI_BIAS_F32 and ld_extra == 0:
        return   # the twin itself (at its shape, with the fences above)

    kw = {}
    if epi in RESID_EPIS:
        r = [torch.randn(m, out_cols, device=DEV, generator=gen) * 2 + 0.5 for _ in range(2)]
        # group 0 in place (resid is out), group 1 out of place
        outs = [fenced(m, out_cols, F32, r[0], ld), fenced(m, out_cols, F32, NAN, ld)]
        _, rview = fenced(m, out_cols, F32, r[1], ld)
        kw['resid'] = [outs[0][1], rview]
        kw['alpha'] = alpha
    else:
        outs = [fenced(m, out_cols, F32 if epi in HEADS else BF16, NAN, ld) for _ in range(2)]
    if epi in LN_PRODUCERS:
        xb = [fenced(m, out_cols, BF16, NAN, ld) for _ in range(2)]
        stats = [torch.full((m + GUARD, _lib.LN_SLOTS, 2), NAN, device=DEV) for _ in range(2)]
        kw.update(out_bf16=[o for _, o in xb], stats=stats)
    if epi in LN_CONSUMERS:
        stats, s_n, bp = [], [], []
        for i in range(2):
            st = torch.full((m + GUARD, _lib.LN_SLOTS, 2), NAN, device=DEV)
            cols = x[i].reshape(m, parts, k // parts)
            st[:m, :parts, 0], st[:m, :parts, 1] = cols.sum(-1), (cols * cols).sum(-1)
            stats.append(st)
            s_n.append(W0[i].double().sum(1).float())
            bp.append(b0[i])
        kw.update(stats=stats, ln_s=s_n, parts=parts)
    gemm(lib, epi, A, W, [o for _, o in outs], bias=bias, **kw)
    for i, (buf, o) in enumerate(outs):
        assert_fenced(buf, o, f'{label} group {i}')
    if epi in LN_PRODUCERS:
        for i, (buf, o) in enumerate(xb):
            assert_fenced(buf, o, f'{label} out_bf16 group {i}')

    for i in range(2):
        lab, out = f'{label} group {i}', outs[i][1]
        if epi == E.EPI_STORE_BF16:
            assert_bitwise(lab + ': out vs bf16(v)', out, v[i].to(BF16))
        elif epi == E.EPI_SILU_BF16:
            ref = torch.nn.functional.silu(v[i].double())
            check_bound(lab + ' silu', (out.double() - ref).abs(), bf16_bound(ref, silu_err(v[i].double()) + 2 * U * ref.abs()))
        elif epi == E.EPI_GLU_BF16:
            vo, vg = glu_unpack(v[i].double())
            check_glu(lab + ' glu', out, vo, vg)
        elif epi in (E.EPI_RESID_F32, E.EPI_RESID_F32_LN):
            assert_bitwise(lab + ': out vs fmaf(v, alpha, resid)', out, fma32(v[i], alpha, r[i]))
        elif epi in (E.EPI_GLU_RESID_F32, E.EPI_GLU_RESID_F32_LN):
            vo, vg = glu_unpack(v[i].double())
            check_glu(lab + ' glu + resid', out, vo, vg, resid=r[i])
        elif epi in LN_CONSUMERS:
            y, d = ln_folded(v[i], stats[i][:m], parts, s_n[i], bp[i], k)
            if epi == E.EPI_LN_STORE_BF16:
                check_bound(lab + ' LayerNorm fold', (out.double() - y).abs(), bf16_bound(y, d))
            elif epi == E.EPI_LN_SILU_BF16:
                ref = torch.nn.functional.silu(y)
                e = 1.1 * d + silu_err(y.abs() + d) + 2 * U * ref.abs()     # |silu'| < 1.1
                check_bound(lab + ' LayerNorm fold + silu', (out.double() - ref).abs(), bf16_bound(ref, e))
            else:
                (yo, yg), (do, dg) = glu_unpack(y), glu_unpack(d)
                check_glu(lab + ' LayerNorm fold + glu', out, yo, yg, do, dg)
        elif epi == E.EPI_BIAS_F32:
            assert_bitwise(lab + ': strided logits vs the twin', out, v[i])
        elif epi == E.EPI_SIGMOID_F32:
            check_sigmoid_head(lab + ' sigmoid', out, v[i])
        else:
            check_softmax_head(lab + ' softmax', out, v[i])
        if epi in LN_PRODUCERS:
            assert_bitwise(lab + ': out_bf16 vs bf16(out)', xb[i][1], out.to(BF16))
            check_ln_stats(lab, stats[i], out, 8 if glu else n // 128)

    if epi in (E.EPI_SIGMOID_F32, E.EPI_SOFTMAX_F32):
        # the same launch with the bias padding at +1e30: a padded column taking part anywhere changes the result
        again = [fenced(m, out_cols, F32, NAN, ld) for _ in range(2)]
        gemm(lib, epi, A, W, [o for _, o in again], bias=[padded_bias(b, 1e30) for b in b0])
        for i in range(2):
            assert_bitwise(f'{label} group {i}: bias padding NaN vs +1e30', again[i][1], outs[i][1])


@pytest.mark.parametrize('m', [1, 63, 64, 65, 129, 'many'])
@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_epilogue_against_its_twin(lib, case, m):
    m = many_rows(case[2]) if m == 'many' else m
    run_case(lib, case, m, seeded('epilogue', case[0], m))


@pytest.mark.parametrize('case', [c for c in CASES if c[0] in ('qkv', 'out_proj_ln', 'glu_mix', 'head_softmax129',
                                                             'head_logits129')], ids=lambda c: c[0])
def test_strided_operands_and_outputs(lib, case):
    """lda > K (A's columns past K are NaN) and ld_out > out_cols (the columns between hold a sentinel): the tensor maps
    and the head stores must use the pitches, not the widths."""
    run_case(lib, case, 300, seeded('strided', case[0]), lda=case[3] + 64, ld_extra=64 if case[1] not in HEADS else 3)


# ------------------------------------------------------------------------------------------------------------ activations
def test_activations_across_the_range(lib):
    """A = 0, so the accumulator is exactly 0 and every epilogue sees v = bias: SiLU, the GLU gate and the sigmoid and softmax
    heads over pre-activations from -40 to +40, against the same bounds.  Prints the error in bf16 ulps of the exact
    output, split at v = -4, where tanh.approx's absolute error stops being small against the output."""
    m, k, n = 64, 64, 2048
    A = [operand(torch.zeros(m, k, device=DEV, dtype=BF16))] * 2
    W = [operand(torch.zeros(n, k, device=DEV, dtype=BF16))] * 2
    sweep = [torch.linspace(-40, 8, n, device=DEV), torch.linspace(-6, 6, n, device=DEV)]

    def ulps(label, out, ref, v):
        e = (out.double() - ref).abs() / (2 * half_ulp_bf16(ref))
        for part, sel in (('v < -4', v < -4), ('v >= -4', v >= -4)):
            if bool(sel.any()):
                print(f'{label} {part}: max |out - exact| {e[:, sel].max().item():.3g} bf16 ulps of the exact output')
        over = (e > 1).any(0)
        if bool(over.any()):
            print(f'{label}: over one bf16 ulp of the exact output for v <= {v[over].max().item():.3g}')

    outs = [fenced(m, n, BF16, NAN) for _ in range(2)]
    gemm(lib, E.EPI_SILU_BF16, A, W, [o for _, o in outs], bias=sweep)
    for i in range(2):
        v = sweep[i].double()[None, :].expand(m, n)
        ref = torch.nn.functional.silu(v)
        check_bound(f'silu sweep {i}', (outs[i][1].double() - ref).abs(), bf16_bound(ref, silu_err(v) + 2 * U * ref.abs()))
        ulps(f'silu sweep {i}', outs[i][1], ref, sweep[i])

    # GLU: out half of every packed group = 1, gate half = the sweep, so out = sigmoid_fast(gate)
    gates = [s[::2].contiguous() for s in sweep]
    packed = [torch.stack([torch.ones(n // 32, 16, device=DEV), g.reshape(n // 32, 16)], 1).reshape(n) for g in gates]
    outs = [fenced(m, n // 2, BF16, NAN) for _ in range(2)]
    gemm(lib, E.EPI_GLU_BF16, A, W, [o for _, o in outs], bias=packed)
    for i in range(2):
        g = gates[i].double()[None, :].expand(m, n // 2)
        check_glu(f'glu gate sweep {i}', outs[i][1], torch.ones_like(g), g)
        ulps(f'glu gate sweep {i}', outs[i][1], torch.sigmoid(g), gates[i])

    wide = [torch.linspace(-40, 40, n, device=DEV), torch.linspace(-3, 3, n, device=DEV)]
    outs = [fenced(m, n, F32, NAN) for _ in range(2)]
    gemm(lib, E.EPI_SIGMOID_F32, A, W, [o for _, o in outs], bias=wide)
    for i in range(2):
        check_sigmoid_head(f'sigmoid head sweep {i}', outs[i][1], wide[i][None, :].expand(m, n))

    soft = [torch.linspace(-60, 10, 256, device=DEV), torch.linspace(-1, 1, 256, device=DEV)]
    outs = [fenced(m, 256, F32, NAN) for _ in range(2)]
    gemm(lib, E.EPI_SOFTMAX_F32, A, [w[:256] for w in W], [o for _, o in outs], bias=soft)
    for i in range(2):
        check_softmax_head(f'softmax head sweep {i}', outs[i][1], soft[i][None, :].expand(m, 256))

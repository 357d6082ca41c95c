"""Float64 restatements of the row-wise trunk kernels of csrc/rowwise.cu, float64 models of what each kernel computes, the
error bound that holds each kernel to its model, and the test data.  Used by tests/test_rowwise_f64_cpu.py and
tests/test_gpu_rowwise_f64.py.  Pure torch: every function runs on the tensors' device, the CPU or a GPU.

Kernels and references (rows of 512 fp32 values unless said otherwise):
  some_layernorm       nn.LayerNorm(512, eps 1e-5); fp32 and/or bf16 out
  some_bound_head      sigmoid(Linear(512, 1)(LayerNorm(x))) = norm5 -> cutheard -> sigmoid; fp32 out
  some_row_stats       (sum x, sum x^2) per row in slot 0 of ln_stats, and bf16(x)
  some_dwconv_bn_silu  SiLU(BatchNorm1d_eval(Conv1d(512, 512, 31, padding=15, groups=512)(x))) per clip, zero padding at
                       each clip's ends; bf16 x and out, the BatchNorm folded into fp32 taps w' and bias b' on the host

exact64 is the module's float64 semantics (eps 1e-5 in float64, the BatchNorm from its unfolded parameters).  kernel64 is
the same arithmetic in float64 on the operands the kernel receives: the LayerNorm's eps is 1e-5f (EPS32, not 1e-5), the
depthwise conv gets the fp32 folded taps and bias.  The bounds below hold a kernel's output to kernel64; u = 2^-24 and
g_n = n u / (1 - n u) (Higham, Accuracy and Stability of Numerical Algorithms, §3.1).  Every sum bound holds for ANY order
of fp32 additions that rounds to nearest, so it holds whatever order the compiler or the warp shuffles pick.

LayerNorm (ln_bound; rowwise.cu ln_normalise).  Lane l holds columns 128 i + 4 l + j (i, j < 4).
* Mean.  Each lane adds its 16 values in a chain (the first add to 0 is exact), then a 5-level xor butterfly adds the lanes:
  every value passes at most 20 roundings, so |S^ - S| <= g21 sum |x|.  The scale 1/512 is exact, so
  |dm| = |m^ - m| <= g21 sum |x| / 512.
* Deviations.  d^_i = fl(x_i - m^) = (d_i - dm)(1 + e), |e| <= u, d_i = x_i - m.  Since sum d_i = 0,
  sum (d_i - dm)^2 = V + 512 dm^2 with V = sum d_i^2.
* Variance.  The fmaf chain d^ d^ + q (16 roundings per lane) and the butterfly (5) give Q^ within g21 of sum d^^2, so
  Q^ / 512 lies in [(1 - g21)(1 - u)^2 V, (1 + g21)(1 + u)^2 (V + 512 dm^2)] / 512.  Adding eps32 rounds once (nvcc may
  contract the scale and the add into one fmaf: one rounding fewer).  Relative to A = V / 512 + eps32 that is rho_A.
* rsqrtf.  2 ulp maximum error (CUDA C++ Programming Guide, single-precision functions; the library is built without
  fast-math, csrc/Makefile), i.e. at most 2^-22 relative; the bound allows E_RSQRT = 3 2^-23, which also covers an
  emulation that moves the correctly rounded value by 2 ulp.  rstd^ / rstd = (A / A^)^(1/2) (1 +- E_RSQRT) -> rho.
* Output.  p = fl(d^ rstd^) = (d - dm) rstd (1 + e)(1 + e')(1 + rho) so |p - d rstd| <= E_p = |dm| rstd (1 + u)^2 (1 + rho)
  + |d| rstd ((1 + u)^2 (1 + rho) - 1); y^ = fmaf(p, g, b) rounds once: |y^ - y| <= |g| E_p + u (|y| + |g| E_p).
* Range.  512 dm^2, V and Q^ below FLT_MAX (|x - mean| < 2^59 or so), and V / 512 + eps32 not subnormal (it is >= eps32).
  Constant rows whose value has at most 15 significant bits have exact partial sums (k c needs 15 + 9 bits for k <= 512):
  the mean is exact, every d is 0 and the output is beta bit for bit.
* bf16 store.  The bf16 output is RNE of the fp32 one, so it lies in [bf16_rn(y - e), bf16_rn(y + e)] (rounding to nearest
  is monotone): the exact bf16 gap (gap_ratio), so that a truncating store, off by up to one bf16 ulp, stays visible.

Bound head (head_bound; rowwise.cu bound_head_kernel).  y^ is the LayerNorm above (before any store) with its bound e.
* Dot product.  16 fmaf per lane and the butterfly: 21 roundings per term, |dot^ - y^ . w| <= g21 |y^| . |w|, and
  |y^ - y| . |w| <= e . |w|.  The bias add rounds once: e_z.
* Sigmoid.  expf(-z) has 2 ulp (the bound allows E_EXP = 3 2^-23 relative); 1 + E and the IEEE reciprocal round once
  each, so sigma^ = sigma(z^)(1 + eta) with 1 + eta <= (1 + u) / ((1 - E_EXP)(1 - u)).  sigma is 1/4-Lipschitz:
  |sigma^ - sigma(z)| <= e_z / 4 + eta (sigma(z) + e_z / 4) + TINY (a subnormal expf result, |z| > 87, is absolute).

Row statistics (stats_bound; rowwise.cu row_stats_kernel).  s: the same chain and butterfly as the mean, g21 sum |x|.
q: fmaf chain x x + q and butterfly, 21 roundings of non-negative terms: g21 sum x^2.  The bf16 copy is RNE(x) exactly.

Depthwise conv (dw_bound, dw_fold_bound; rowwise.cu dwconv_kernel).
* Pre-activation.  a = b' + sum_k w'_k x_{t+k-15} as a 31-deep fmaf chain seeded with b' (zero rows outside the clip):
  |a^ - a| <= e_a = g31 (|b'| + sum |w' x|).
* silu_fast (sm90_ptx.cuh): h = 0.5 a^ (exact), t = tanh.approx(h), out = fmaf(h, t, h).  tanh.approx.f32 has maximum
  relative error 2^-10.987 (PTX ISA, tanh); the bound allows E_TANH = 2^-10.987 + 2^-23, which covers an emulation that
  rounds the perturbed value to fp32.  out = (silu(a^) + h tanh(h) e_t)(1 + e_f).  SiLU is Lipschitz with constant
  SILU_LIP = 1.0998 (max of |silu'|, at x ~ 2.4), so |out - silu(a)| <= 1.0998 e_a + |h| |tanh h| E_TANH + u |out| + TINY,
  |h| <= (|a| + e_a) / 2.  Subnormals: the PTX ISA lists subnormal inputs as supported by tanh.approx.f32; were a subnormal
  h flushed to zero, out = h instead of h + h tanh h, a difference below |h|^2 < 2^-250, inside TINY, so the bound holds
  either way.  Below a = -8.6 this error is larger than a bf16 ulp of the output; where tanh(h) is -1, out is exactly 0.
* Fold (dw_fold_bound).  w'_k = fp32(w_k g / sqrt(var + eps)), b' = fp32((b - mean) g / sqrt(var + eps) + beta), each
  computed in float64 and rounded once: |w'32 - w'64| <= u |w'64|, so |a_kernel64 - a_exact64| <= u (|b'| + sum |w' x|)
  and the outputs differ by at most 1.0998 times that (times 1 + 2^-20 for the float64 arithmetic of the fold).
* bf16 store: the exact bf16 gap, as for the LayerNorm.

Data (the regimes below) cover the existing fp32-torch parity data of tests/test_gpu_kernels.py as the 'iid' and
'centred' LayerNorm / row-statistics regimes and the 'legacy' depthwise regime."""
from __future__ import annotations

import math

import numpy as np
import torch

DIM, K, HALO = 512, 31, 15
U = 2.0 ** -24


def g(n: int) -> float:
    return n * U / (1 - n * U)


G21, G31 = g(21), g(31)
EPS32 = float(np.float32(1e-5))                       # the LayerNorm's eps as the kernel holds it (1e-5f)
BN_EPS = 1e-5
E_RSQRT = 3 * 2.0 ** -23                              # rsqrtf: 2 ulp (CUDA guide); 3 ulp allowed
E_EXP = 3 * 2.0 ** -23                                # expf: 2 ulp (CUDA guide); 3 ulp allowed
TANH_REL = 2.0 ** -10.987                             # tanh.approx.f32 maximum relative error (PTX ISA)
E_TANH = TANH_REL + 2.0 ** -23
SILU_LIP = 1.0998                                     # max |d/dx x sigmoid(x)| = 1.09984 at x = 2.3994
TINY = 2.0 ** -140                                    # absolute allowance for subnormal intermediates


# ------------------------------------------------------------------------------------------------------------ bf16
def bf16_rn(x: torch.Tensor) -> torch.Tensor:
    """float64 x rounded to the nearest bf16 value (ties to even), one rounding, subnormals included"""
    _, e = torch.frexp(x)
    sp = torch.ldexp(torch.ones_like(x), e.clamp_min(-125) - 8)
    return torch.round(x / sp) * sp


def bf16_next(v: torch.Tensor, up: bool) -> torch.Tensor:
    """the bf16 neighbour of the bf16 values v toward +inf (up) or -inf, as float64"""
    b = v.float().to(torch.bfloat16).view(torch.int16).int() & 0xffff
    sign, mag = b >= 0x8000, b & 0x7fff
    grow = sign ^ up                                       # the magnitude grows
    cross = ~grow & (mag == 0)                             # from a zero to the smallest subnormal of the other sign
    sign = torch.where(cross, ~sign, sign)
    mag = torch.where(cross, torch.ones_like(mag), torch.where(grow, mag + 1, mag - 1))
    bits = (sign.int() << 15) | mag
    return (bits - 65536 * (bits >= 32768).int()).short().view(torch.bfloat16).double()


def gap_ratio(got: torch.Tensor, ref: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """the smallest s for which the bf16 value got is RNE of some value in [ref - s e, ref + s e] (the exact bf16 gap):
    for got above ref, ref + s e must reach the midpoint between got and its lower neighbour, and likewise below.  So the
    ratio is <= 1 exactly when got is an allowed store, 0 when got is RNE(ref) itself, and a truncating store that lands
    one bf16 value low shows as a ratio far above 1 wherever e is small against a bf16 ulp"""
    got, ref = got.double(), ref.double()
    err = got - ref
    mid_dn = (got + bf16_next(got, up=False)) / 2
    mid_up = (got + bf16_next(got, up=True)) / 2
    s = torch.where(err > 0, mid_dn - ref, ref - mid_up).clamp_min(0) / (e * (1 + 2.0 ** -40))
    return torch.where(err == 0, torch.zeros_like(err), torch.nan_to_num(s, nan=math.inf))


def abs_ratio(got: torch.Tensor, ref: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """|got - ref| / e (0 where equal, inf for a NaN)"""
    err = (got.double() - ref.double()).abs()
    return torch.nan_to_num(torch.where(err == 0, torch.zeros_like(err), err / e), nan=math.inf)


# ------------------------------------------------------------------------------------------------------------ LayerNorm
def layernorm64(x, gamma, beta, eps):
    x = x.double()
    d = x - x.mean(-1, keepdim=True)
    rstd = ((d * d).mean(-1, keepdim=True) + eps).rsqrt()
    return d * rstd * gamma.double() + beta.double()


def ln_exact64(x, gamma, beta):
    """nn.LayerNorm(512, eps=1e-5) in float64"""
    return layernorm64(x, gamma, beta, BN_EPS)


def ln_kernel64(x, gamma, beta):
    """the LayerNorm with the kernel's eps32"""
    return layernorm64(x, gamma, beta, EPS32)


def ln_bound(x, gamma, beta):
    """(ln_kernel64, e): the bound on |fp32 output - ln_kernel64| (module docstring)"""
    x, ga = x.double(), gamma.double().abs()
    n = x.shape[-1]
    m = x.mean(-1, keepdim=True)
    d = x - m
    V = (d * d).sum(-1, keepdim=True)
    dm = G21 * x.abs().sum(-1, keepdim=True) / n
    A = V / n + EPS32
    a_hi = ((1 + G21) * (1 + U) ** 2 * (V + n * dm * dm) / n + EPS32) * (1 + U) + TINY
    a_lo = ((1 - G21) * (1 - U) ** 2 * V / n + EPS32) * (1 - U)
    rho = torch.maximum((A / a_lo).sqrt() * (1 + E_RSQRT) - 1, 1 - (A / a_hi).sqrt() * (1 - E_RSQRT))
    rstd = A.rsqrt()
    grow = (1 + U) ** 2 * (1 + rho)
    e_p = dm * rstd * grow + d.abs() * rstd * (grow - 1)
    y = d * rstd * gamma.double() + beta.double()
    e = ga * e_p
    return y, e + U * (y.abs() + e)


def ln_eps_gap(x, gamma):
    """bound on |ln_kernel64 - ln_exact64|: the two eps give rstd's that differ by |A32^-1/2 - A^-1/2|"""
    x = x.double()
    d = x - x.mean(-1, keepdim=True)
    v = (d * d).mean(-1, keepdim=True)
    return (1 + 2.0 ** -30) * d.abs() * gamma.double().abs() * ((v + EPS32).rsqrt() - (v + BN_EPS).rsqrt()).abs()


# ------------------------------------------------------------------------------------------------------------ bound head
def head_exact64(x, gamma, beta, w, bias):
    """norm5 -> Linear(512, 1) -> sigmoid in float64"""
    return torch.sigmoid(ln_exact64(x, gamma, beta) @ w.double() + bias)


def head_bound(x, gamma, beta, w, bias):
    """(head kernel64, e): the bound on |bounds - kernel64| (module docstring)"""
    y, e = ln_bound(x, gamma, beta)
    aw = w.double().abs()
    z = y @ w.double() + bias
    e_dot = e @ aw + G21 * ((y.abs() + e) @ aw)
    e_z = e_dot + U * (z.abs() + e_dot)
    s = torch.sigmoid(z)
    eta = (1 + U) / ((1 - E_EXP) * (1 - U)) - 1
    return s, e_z / 4 + eta * (s + e_z / 4) + TINY


def head_eps_gap(x, gamma, w):
    return 0.25 * ln_eps_gap(x, gamma) @ w.double().abs()


# ------------------------------------------------------------------------------------------------------------ row stats
def stats_exact64(x):
    """(sum x, sum x^2) per row in float64"""
    x = x.double()
    return x.sum(-1), (x * x).sum(-1)


def stats_bound(x):
    x = x.double()
    return G21 * x.abs().sum(-1) + TINY, G21 * (x * x).sum(-1) + TINY


# ------------------------------------------------------------------------------------------------------------ depthwise conv
def clip_ids(cu, device):
    """per row of [cu[0], cu[-1]): its clip's first row and end row"""
    cu_t = torch.as_tensor(np.asarray(cu, dtype=np.int64), device=device)
    lens = cu_t[1:] - cu_t[:-1]
    return torch.repeat_interleave(cu_t[:-1], lens), torch.repeat_interleave(cu_t[1:], lens)


def conv31(x, cu, taps, absolute=False):
    """sum_k taps[k] x[t + k - 15] per clip with zero rows outside the clip, as 31 shifted multiply-adds in float64:
    x [M, 512], taps [31, 512]; absolute: sum |taps[k] x| (the bound's magnitude sum)"""
    x, taps = x.double(), taps.double()
    if absolute:
        x, taps = x.abs(), taps.abs()
    m = x.shape[0]
    start, end = clip_ids(cu, x.device)
    rows = torch.arange(m, device=x.device)
    acc = torch.zeros_like(x)
    xp = torch.nn.functional.pad(x, (0, 0, HALO, HALO))
    for k in range(K):
        src = rows + (k - HALO)
        ok = ((src >= start) & (src < end)).double()[:, None]
        acc += taps[k] * xp[k:k + m] * ok
    return acc


def dw_fold64(p):
    """(taps [31, 512], bias [512]) of the BatchNorm fold in float64 from unfolded parameters p (see dw_params)"""
    scale = p['bn_weight'].double() / (p['bn_var'].double() + BN_EPS).sqrt()
    return (p['weight'].double() * scale[:, None]).t(), (p['bias'].double() - p['bn_mean'].double()) * scale + p['bn_bias'].double()


def dw_exact64(x, cu, p):
    """Conv1d(512, 512, 31, padding=15, groups=512) -> BatchNorm1d(eval, eps 1e-5) -> SiLU in float64 from the unfolded
    parameters, per clip"""
    conv = conv31(x, cu, p['weight'].double().t()) + p['bias'].double()
    bn = (conv - p['bn_mean'].double()) / (p['bn_var'].double() + BN_EPS).sqrt() * p['bn_weight'].double() + p['bn_bias'].double()
    return torch.nn.functional.silu(bn)


def dw_kernel64(x, cu, taps, bias):
    """(pre-activation, SiLU of it) in float64 from the fp32 folded taps [31, 512] and bias [512] the kernel receives"""
    a = conv31(x, cu, taps) + bias.double()
    return a, torch.nn.functional.silu(a)


def dw_magnitude(x, cu, taps, bias):
    return conv31(x, cu, taps, absolute=True) + bias.double().abs()


def dw_bound(x, cu, taps, bias):
    """(kernel64 output, e): the bound on |fp32 SiLU output - kernel64| before the bf16 store (module docstring)"""
    a, y = dw_kernel64(x, cu, taps, bias)
    e_a = G31 * dw_magnitude(x, cu, taps, bias)
    h = (a.abs() + e_a) / 2
    e_t = h * torch.tanh(h) * E_TANH
    e = SILU_LIP * e_a + e_t
    return y, e + U * (y.abs() + e) + TINY


def dw_fold_bound(x, cu, taps, bias):
    """bound on |SiLU(kernel64) - exact64| from the fold's rounding to fp32"""
    return SILU_LIP * U * (1 + 2.0 ** -20) * dw_magnitude(x, cu, taps, bias)


# ------------------------------------------------------------------------------------------------------------ data
ROW_REGIMES = ('iid', 'centred', 'dc', 'const15', 'const', 'outlier', 'scaled')
HEAD_REGIMES = ROW_REGIMES + ('saturate',)
DW_REGIMES = ('legacy', 'iid_synthetic', 'iid_trained', 'ramp', 'edges', 'span', 'zeros', 'huge')
OUTLIER = 2.0 ** 8
EDGE = 2.0 ** 14


def rows(name: str, m: int, gen: torch.Generator, device='cpu') -> torch.Tensor:
    """x [m, 512] fp32 of a row regime:
    iid       N(1.5, 3^2) (the LayerNorm / bound head data of the fp32 parity test this replaces)
    centred   N(-0.3, 2^2) (the row-statistics data of that test)
    dc        mean 2^12, std 2^-4: |mean| / std = 2^16, a residual stream with a large DC offset
    const15   constant rows whose value has at most 15 significant bits: every partial sum exact, output beta bit for bit
    const     constant rows of arbitrary fp32 value
    outlier   N(0, 1) with one 2^8 entry per row at column (row mod 512): every lane and each of its 16 slots
    scaled    iid rows scaled by 2^-20 .. 2^20 (the exponent steps by 1 per row): eps dominates at the small end
    saturate  iid rows (for the bound head with a large w, see head_params)"""
    f = lambda *s: torch.randn(*s, generator=gen, device=device)
    if name in ('iid', 'saturate'):
        return f(m, DIM) * 3 + 1.5
    if name == 'centred':
        return f(m, DIM) * 2 - 0.3
    if name == 'dc':
        return (f(m, DIM) * 2.0 ** -4 + 2.0 ** 12).float()
    if name == 'const15':
        k = torch.randint(-2 ** 15 + 1, 2 ** 15, (m, 1), generator=gen, device=device).double()
        e = torch.randint(-20, 10, (m, 1), generator=gen, device=device).double()
        return (k * torch.exp2(e)).float().expand(m, DIM).contiguous()
    if name == 'const':
        return (f(m, 1) * 10).expand(m, DIM).contiguous()
    if name == 'outlier':
        x = f(m, DIM)
        x[torch.arange(m, device=device), torch.arange(m, device=device) % DIM] = OUTLIER
        return x
    if name == 'scaled':
        s = torch.exp2(torch.arange(m, device=device) % 41 - 20.0)
        return (f(m, DIM) * 3 + 1.5) * s[:, None]
    raise ValueError(name)


def ln_params(gen: torch.Generator, device='cpu'):
    """gamma ~ U(0.5, 1.5), beta ~ N(0, 0.1^2): distinct per column, so a column permutation shows"""
    return (torch.rand(DIM, generator=gen, device=device) + 0.5, torch.randn(DIM, generator=gen, device=device) * 0.1)


def head_params(name: str, gen: torch.Generator, device='cpu'):
    """(w [512], bias): w ~ N(0, 1/512) (the old parity test's), or for 'saturate' 20 times that, so that z spans about
    +-40 (and beyond) over the rows and the sigmoid saturates both ways"""
    w = torch.randn(DIM, generator=gen, device=device) / DIM ** 0.5
    return (w * 20 if name == 'saturate' else w), 0.3


def dw_params(stats: str, gen: torch.Generator, device='cpu', beta_span=False):
    """unfolded fp32 parameters: Conv1d weight [512, 31] and bias, BatchNorm1d weight, bias, running mean and var.
    identity   w ~ N(0, 0.2^2), b ~ N(0, 0.1^2) with gamma 1, beta 0, mean 0, var 1 (the old parity test's taps)
    synthetic  as synth.fabricate_state_dict: U(+-1/sqrt(31)) conv, gamma U(0.8, 1.2), beta N(0, 0.05^2), mean N(0, 0.1^2),
               var U(0.5, 1.5)
    trained    var log-uniform in [1e-4, 1e-2] and mean U(-1, 1): eps and the mean's placement matter
    beta_span: beta from -20 to 20 over the channels (pre-activations across [-20, 20])"""
    r = lambda *s: torch.rand(*s, generator=gen, device=device)
    n = lambda *s: torch.randn(*s, generator=gen, device=device)
    if stats == 'identity':
        p = dict(weight=n(DIM, K) * 0.2, bias=n(DIM) * 0.1, bn_weight=torch.ones(DIM, device=device),
                 bn_bias=torch.zeros(DIM, device=device), bn_mean=torch.zeros(DIM, device=device),
                 bn_var=torch.ones(DIM, device=device))
    else:
        lim = 1 / K ** 0.5
        p = dict(weight=(r(DIM, K) * 2 - 1) * lim, bias=(r(DIM) * 2 - 1) * lim, bn_weight=r(DIM) * 0.4 + 0.8,
                 bn_bias=n(DIM) * 0.05)
        if stats == 'synthetic':
            p.update(bn_mean=n(DIM) * 0.1, bn_var=r(DIM) + 0.5)
        elif stats == 'trained':
            p.update(bn_mean=r(DIM) * 2 - 1, bn_var=torch.exp2(r(DIM) * math.log2(100) + math.log2(1e-4)))
        else:
            raise ValueError(stats)
    if beta_span:
        p['bn_bias'] = torch.linspace(-20, 20, DIM, device=device)
    return {k: v.float().contiguous() for k, v in p.items()}


DW_STATS = {'legacy': 'identity', 'iid_trained': 'trained'}


def dw_regime_params(name: str, gen: torch.Generator, device='cpu'):
    return dw_params(DW_STATS.get(name, 'synthetic'), gen, device, beta_span=name in ('span', 'zeros'))


def dw_clip(name: str, t: int, index: int, gen: torch.Generator, device='cpu') -> torch.Tensor:
    """x [t, 512] (bf16 values as fp32) of clip `index` of a depthwise regime:
    legacy, iid_*  N(0, 1)
    ramp           x[t, c] = ((t + 7 c + 3 index) mod 509 - 254) / 64: every frame's value differs from its neighbours', so a
                   one-frame shift, flipped taps or a 14- or 16-row halo shows
    edges          N(0, 1) in even clips, +-2^14 in odd ones: a read across a clip edge shows
    span           N(0, 1) with beta from -20 to 20 over the channels: pre-activations across [-20, 20]
    zeros          exact zeros (out = silu_fast(b'))
    huge           N(0, 1) 2^18: |pre-activation| up to about 2^20"""
    x = torch.randn(t, DIM, generator=gen, device=device)
    if name == 'ramp':
        tt = torch.arange(t, device=device)[:, None] + 7 * torch.arange(DIM, device=device)[None, :] + 3 * index
        x = ((tt % 509) - 254).float() / 64
    elif name == 'edges' and index % 2 == 1:
        x = torch.sign(x) * EDGE
    elif name == 'zeros':
        x = torch.zeros_like(x)
    elif name == 'huge':
        x = x * 2.0 ** 18
    elif name not in ('legacy', 'iid_synthetic', 'iid_trained', 'span', 'edges'):
        raise ValueError(name)
    return x.to(torch.bfloat16).float()

"""Float64 restatement of the reference attention (base_attention.py:34-45: softmax(q k^T / 8) v per clip and head, no mask),
a float64 model of what the bf16 attention kernel some_attention_varlen (csrc/attention_tc.cu) computes, the error bound
that holds the kernel to that model, and the test data.  Used by tests/test_attention_f64_cpu.py and
tests/test_gpu_attention_f64.py.  Pure torch: every function runs on the tensors' device, the CPU or a GPU.

Layout.  qkv [M, 1536] holds bf16 values: q of head h at columns 64 h, k at 512 + 64 h, v at 1024 + 64 h; clip b owns rows
[cu[b], cu[b + 1]).  The output is [M, 512] = 'b t (h c)'.

The kernel, per query row and head.  s_i = q . k_i accumulates 64 exact bf16 products in fp32 on the tensor cores.  Keys run
in 64-key tiles counted from the clip start; keys past the clip end are masked (p = 0).  Per tile j: m_j = max(m_{j-1}, the
tile's largest score), alpha_j = ex2((m_{j-1} - m_j) c) (0 on the first tile), mc = fp32(m_j c),
p_i = ex2(fmaf(s_i, c, -mc)) with ex2 = ex2.approx.ftz and c = fp32(log2 e) * 0.125, P_i = bf16_rn(p_i),
l = fmaf(l, alpha, sum of the lane's 16 p) per lane of the row's quad, O = O alpha + sum_i P_i v_i (64 products on the
tensor cores).  At the end the quad's four l are added in two steps, and out = bf16_rn(O * (1 / l)).

The model (kernel64).  The same steps in float64 from the exact scores s_i: m_j the exact running maximum, p_i =
2^((s_i - m_j(i)) c), P_i = bf16_rn(p_i), a_j = 2^((m_j - m_last) c), and

    o_bar = sum_i a_j(i) P_i v_i / sum_i a_j(i) p_i.

Write W_i = a_j P_i and Lam_i = a_j p_i = 2^((s_i - m_last) c) (so L = sum Lam >= 1: the key at the maximum has Lam = 1).

The bound (bound()) on |out - o_bar| holds for any fp32 summation order, rounding to nearest or truncating, in the tensor-core
accumulations and the lane sums; u = 2^-24 for the operations the kernel spells out (fmaf, multiplies, the IEEE division).

* S.  64 exact products in any order: |s^_i - s_i| <= 65 2^-23 sigma_i, sigma_i = sum |q k_i| (the bound of
  check_against_float64 in tests/test_gpu_gemm_epilogues.py).  The kernel's running maximum m^_j is a maximum of s^ over
  the same keys, so |m^_j - m_j| <= dm_j, the largest score error in tiles <= j.
* Exponents.  p^_i = ex2(fmaf(s^_i, c, -mu_j)) with mu_j = fp32(m^_j c) = m^_j c + d_mu, |d_mu| <= u |m^_j c|, and the fmaf
  rounds once, u of its result |arg_i| <= (m_j - s_i) c + (65 2^-23 sigma_i + dm_j) c + u |m^_j c|.  ex2.approx is within
  EPS_EX2 = 2^-22 relative (PTX ISA); the bound allows twice that.  alpha^_j = ex2(fp32(fp32(m^_{j-1} - m^_j) c)): the
  subtraction and the product round once each, so its exponent is (m^_{j-1} - m^_j) c + d2_j, |d2_j| <= 2^-23 (1 + u)
  |m^_{j-1} - m^_j| c, which is 0 where the maximum does not move.  The rescale factors after tile j multiply to
  A_j = 2^((m^_j - m^_last) c + D_j) (1 + e)^(tiles after j), D_j = sum of d2 over the later tiles: they telescope, and
  are not exactly consistent with the two rounded m c the p's used; D_j carries that.
  With the common factor K = 2^((m_last - m^_last) c), which cancels between numerator and denominator:
      A_j p^_i / (K Lam_i) = 2^((s^_i - s_i) c + D_j - d_mu + d_fma) (1 + e)^(1 + tiles after j)  ->  relative lambda_i
      A_j / (K a_j)         = 2^((m^_j - m_j) c + D_j) (1 + e)^(tiles after j)                    ->  relative omega_j
  The maximum's error cancels in the denominator's terms, not in the numerator's: P is snapped to a bf16 value.
* Flips of P.  p^_i is within rho_i p_i of p_i, rho_i from 2^((65 2^-23 sigma_i + dm_j) c + u |m^_j c| + u |arg_i|) and one
  ex2.  Rounding to nearest is monotone, so bf16(p^_i) lies between bf16_rn(p_i (1 - rho_i)) and bf16_rn(p_i (1 + rho_i)):
  it equals P_i unless p_i is within rho_i p_i of a rounding midpoint, and then it is one bf16 ulp away.  The bound allows
  exactly that gap, so a defect that moves the output by about one output ulp stays visible.
* FTZ and underflow.  ex2.approx.ftz flushes results below 2^-126 to zero (alpha^ of a maximum that jumps by more than 126 in
  the exponent, p of keys far below the maximum).  Every such key has Lam_i < 2^-100: for those, the bound allows any
  weight in [0, 2^-99] in the numerator and the denominator.
* O.  Per tile, O alpha^ rounds (u), then 64 exact products P v join it in any order: 65 2^-23 of the tile's partial
  magnitude sum, which holds every key of that tile and the tiles before it.  Summed over tiles, key i counts
  (tiles - j(i)) times: E_O <= (65 2^-23 + u) sum_i |W^_i v_i| (tiles - j(i)).
* l.  Positive terms: 16 per lane per tile summed in any order (15 2^-23 relative), one fmaf per tile (u each, at most
  `tiles` of them after a key's tile), two quad adds (2 u): relative nu = 15 2^-23 + (tiles + 2) u of the sum of the
  kernel's weights, on top of their lambda.
* Output.  |O/l - o_bar| <= (sum_i |W^_i - W_i| |v_i| + E_O + |o_bar| sum_i |Lam^_i - Lam_i|) / (L - sum_i |Lam^_i - Lam_i|);
  1 / l and O * inv round once each (2 u relative); the bf16 store is bf16_bound (as in the GEMM test).  The first-order
  sum is multiplied by 1.01: every relative term is below 1e-2 here, so their products are below 1 % of the sum.

The loose bound (loose_bound()) of o_bar against exact64: o_bar rounds P to bf16 in the numerator only, at most 2^-8
relative per key (bf16 keeps 8 significant bits), and its weights 2^((s - m_last) c) differ from e^((s - m) / 8) by the
rounding of log2 e to fp32 in c (relative c - 1 / (8 ln 2), times |s - m_last|).  So |o_bar - exact| <= 2^-8 sum w~ |v| + 2 eta sum w |v|, with w the exact
softmax weights, w~ = Lam / L and eta the weights' largest relative change."""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

HEADS, DH, DIM = 8, 64, 512
BN = 64                                                               # keys per tile
C = float(np.float32(np.float32(1.4426950408889634) * np.float32(0.125)))   # the kernel's c, exactly
C_EXACT = 1.0 / (8.0 * math.log(2.0))                                 # log2(e) / 8
U = 2.0 ** -24
EPS_EX2 = 2.0 ** -22                                                  # ex2.approx.f32: maximum relative error (PTX ISA)
E_EX2 = 2 * EPS_EX2                                                   # allowed by the bound
S_ERR = 65 * 2.0 ** -23                                               # 64 products + 1, any order (times sigma)
TINY = 2.0 ** -100                                                    # keys below this weight: absolute allowance 2 TINY
OUTLIER_K = 48.0                                                      # the outlier key's value (see regime 'outlier')


# ------------------------------------------------------------------------------------------------------------ bf16
def bf16_rn(x: torch.Tensor) -> torch.Tensor:
    """float64 x rounded to the nearest bf16 value (ties to even), one rounding, subnormals included"""
    _, e = torch.frexp(x)
    sp = torch.ldexp(torch.ones_like(x), e.clamp_min(-125) - 8)       # the bf16 spacing at |x|
    return torch.round(x / sp) * sp


def half_ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """half the bf16 spacing at magnitude |x| (a bf16 store that rounds to nearest moves any |z| <= |x| by at most this)"""
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x), e - 9)


def bf16_bound(ref: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """bound on |bf16(z) - ref| for any fp32 z with |z - ref| <= e"""
    return e + half_ulp_bf16(ref.abs() + e)


# ------------------------------------------------------------------------------------------------------------ layout
def heads(qkv_clip: torch.Tensor):
    """[T, 1536] -> q, k, v as float64 [8, T, 64]"""
    z = qkv_clip.double()
    t = z.shape[0]
    return tuple(z[:, j * DIM:(j + 1) * DIM].reshape(t, HEADS, DH).transpose(0, 1) for j in range(3))


def merge(o: torch.Tensor) -> torch.Tensor:
    """[H, T, 64] -> [T, H * 64] ('b h t c -> b t (h c)')"""
    return o.transpose(0, 1).reshape(o.shape[1], -1)


def exact64(qkv: torch.Tensor, cu) -> torch.Tensor:
    """base_attention.py:34-45 in float64, per clip: [cu[-1], 512] (rows of clip b at cu[b] .. cu[b + 1])"""
    outs = []
    for b in range(len(cu) - 1):
        q, k, v = heads(qkv[int(cu[b]):int(cu[b + 1])])
        outs.append(merge(torch.softmax(q @ k.transpose(1, 2) * 0.125, -1) @ v))
    return torch.cat(outs)


# ------------------------------------------------------------------------------------------------------------ model
@dataclass
class Model:
    """kernel64 of one clip, every head at once; per-key tensors are [H, T, T] (query, key), per-tile ones [H, T, tiles]"""
    o: torch.Tensor       # [H, T, 64] o_bar
    v: torch.Tensor       # [H, T, 64]
    s: torch.Tensor       # scores q . k (float64)
    sigma: torch.Tensor   # sum_c |q_c k_c|
    tile: torch.Tensor    # [T] key tile index
    m: torch.Tensor       # [H, T, tiles] exact running maximum
    p: torch.Tensor       # 2^((s - m_j) c)
    P: torch.Tensor       # bf16_rn(p)
    a: torch.Tensor       # [H, T, tiles] 2^((m_j - m_last) c)
    L: torch.Tensor       # [H, T] sum a p

    @property
    def tiles(self) -> int:
        return self.m.shape[-1]

    def out(self) -> torch.Tensor:
        """o_bar as [T, H * 64]"""
        return merge(self.o)


def model_heads(q, k, v) -> Model:
    """the kernel's arithmetic in float64 on one clip: q, k, v [H, T, 64] float64"""
    h, t, _ = q.shape
    nt = -(-t // BN)
    s = q @ k.transpose(1, 2)
    sigma = q.abs() @ k.abs().transpose(1, 2)
    tile = torch.arange(t, device=q.device) // BN
    sp = torch.nn.functional.pad(s, (0, nt * BN - t), value=-math.inf).view(h, t, nt, BN)
    m = sp.amax(-1).cummax(-1).values
    p = torch.exp2((s - m[..., tile]) * C)
    P = bf16_rn(p)
    a = torch.exp2((m - m[..., -1:]) * C)
    ak = a[..., tile]
    L = (ak * p).sum(-1)
    o = (ak * P) @ v / L[..., None]
    return Model(o, v, s, sigma, tile, m, p, P, a, L)


def kernel64(qkv: torch.Tensor, cu) -> list:
    """model_heads of every clip of a var-len batch: one Model per clip"""
    return [model_heads(*heads(qkv[int(cu[b]):int(cu[b + 1])])) for b in range(len(cu) - 1)]


def bound(md: Model) -> torch.Tensor:
    """[T, H * 64] bound on |kernel output - o_bar| (module docstring)"""
    h, t, nt = md.m.shape
    tile = md.tile
    err_s = S_ERR * md.sigma                                                       # |s^ - s|
    dm = torch.nn.functional.pad(err_s, (0, nt * BN - t)).view(h, t, nt, BN).amax(-1).cummax(-1).values   # |m^_j - m_j|
    mk, dmk = md.m[..., tile], dm[..., tile]
    mc_err = U * (mk.abs() + dmk) * C                                              # fp32(m^ c)
    arg = (mk - md.s) * C + (err_s + dmk) * C + mc_err                            # |fmaf result|
    # rescale exponents d2_j (tile j >= 1) and their sums over the later tiles D_j
    move = torch.zeros_like(md.m)
    move[..., 1:] = (md.m[..., 1:] - md.m[..., :-1]) + dm[..., 1:] + dm[..., :-1]
    d2 = 2.0 ** -23 * (1 + U) * move * C
    D = d2.flip(-1).cumsum(-1).flip(-1) - d2
    after = (nt - 1 - torch.arange(nt, device=md.m.device)).double()             # tiles after j
    omega = torch.exp2(dm * C + D) * (1 + E_EX2) ** after - 1                       # [H, T, nt]
    om_k = omega[..., tile]
    lam = torch.exp2(err_s * C + mc_err + U * arg + D[..., tile]) * (1 + E_EX2) ** (1 + after[tile]) - 1
    rho = torch.exp2((err_s + dmk) * C + mc_err + U * arg) * (1 + E_EX2) - 1 + 2.0 ** -40
    gap = bf16_rn(md.p * (1 + rho)) - bf16_rn(md.p * (1 - rho))                   # 0 unless P may flip
    ak = md.a[..., tile]
    W, Lam = ak * md.P, ak * md.p
    tiny = (Lam < TINY).double()
    keep = 1 - tiny
    av = md.v.abs()
    w_err = keep * (om_k * W + (1 + om_k) * ak * gap) + tiny * 2 * TINY              # |W^ - W|
    w_hat = keep * ((1 + om_k) * (W + ak * gap)) + tiny * 2 * TINY                  # |W^|
    e_o = (65 * 2.0 ** -23 + U) * ((w_hat * (nt - tile).double()) @ av) + nt * 2.0 ** -120
    nu = 15 * 2.0 ** -23 + (nt + 2) * U
    l_err = (keep * (lam + nu * (1 + lam)) * Lam + tiny * 2 * TINY).sum(-1, keepdim=True)   # |L^ - L|
    num = w_err @ av + e_o
    ob = md.o.abs()
    e1 = 1.01 * (num + ob * l_err) / (md.L[..., None] - l_err)
    e2 = e1 + 1.01 * (ob + e1) * 2 * U
    return merge(bf16_bound(md.o, e2))


def loose_bound(md: Model) -> torch.Tensor:
    """[T, H * 64] bound on |o_bar - exact64| (module docstring)"""
    w = torch.softmax(md.s * 0.125, -1)
    ak = md.a[..., md.tile]
    wt = ak * md.p / md.L[..., None]
    eta = float(torch.exp2((md.m[..., -1:] - md.s).amax() * abs(C - C_EXACT)) - 1)
    av = md.v.abs()
    t = md.s.shape[-1]
    return merge(1.01 * (2.0 ** -8 * (wt @ av) + 2 * eta * (w @ av)) + t * 2.0 ** -120 * av.amax(1, keepdim=True))


# ------------------------------------------------------------------------------------------------------------ data
REGIMES = ('spread', 'peaky', 'ramp', 'outlier', 'equal', 'zero_q', 'big_v')


def outlier_keys(t: int) -> list:
    """the key position of head h's outlier: key % 8 == h, in a tile other than the first when the clip has one"""
    if t <= 8:
        return [h % t for h in range(HEADS)]
    if t < BN + 8:
        return [8 * ((t - 1 - h) // 8) + h for h in range(HEADS)]
    return [BN + 8 * (((t - BN - 8) * (h + 1) // HEADS) // 8) + h for h in range(HEADS)]


def regime(name: str, t: int, gen: torch.Generator, device='cpu') -> torch.Tensor:
    """qkv [t, 1536] (bf16 values, as float32) of one clip:
    spread   q, k, v ~ N(0, 0.5^2): attention spread over many keys, |o| ~ 0.01-0.03 at t = 2584
    peaky    N(0, 1.5^2): a few keys carry each row
    ramp     k grows with the key index (t / 64 per channel, q aligned with it): every row's maximum jumps by more than
             2^4 (about 2^8) in the exponent from one whole 64-key tile to the next, so O and l are rescaled on every tile
    outlier  q > 0 and one key of each head at +48 in every channel (outlier_keys): its score is more than 127 above every
             other in the exponent, so the earlier tiles' rescale underflows to 0; positions cover every key % 8
    equal    every key of a head the same vector: all scores equal, p = 1 exactly
    zero_q   q = 0: o = the mean of v
    big_v    spread, with one channel per head at +-2^10 (sign per key in even heads, +2^10 throughout in odd ones)"""
    z = torch.randn(t, 3 * DIM, generator=gen, device=device) * (1.5 if name == 'peaky' else 0.5)
    if name == 'ramp':
        sgn = torch.sign(torch.randn(1, DIM, generator=gen, device=device))
        z[:, DIM:2 * DIM] += (torch.arange(t, device=device, dtype=torch.float32) / 64.0)[:, None] * sgn
        z[:, :DIM] = z[:, :DIM].abs() * sgn * 2.0
    elif name == 'outlier':
        z[:, :DIM] = z[:, :DIM].abs()
        for h, i in enumerate(outlier_keys(t)):
            z[i, DIM + DH * h:DIM + DH * (h + 1)] = OUTLIER_K
    elif name == 'equal':
        z[:, DIM:2 * DIM] = z[:1, DIM:2 * DIM]
    elif name == 'zero_q':
        z[:, :DIM] = 0.0
    elif name == 'big_v':
        for h in range(HEADS):
            col = 2 * DIM + DH * h + (11 * h + 5) % DH
            if h % 2 == 0:
                z[:, col] = torch.sign(torch.randn(t, generator=gen, device=device)) * 2.0 ** 10
            else:
                z[:, col] = 2.0 ** 10
    elif name not in ('spread', 'peaky'):
        raise ValueError(name)
    return z.to(torch.bfloat16).float()

"""Host-side packing of a reference checkpoint (``state_dict`` of
``modules.model.Gmidi_conform.midi_conforms``) into the device layouts the sm_90a kernels consume:

* every nn.Linear / 1x1 Conv1d weight -> bf16 [N, K] (K-major, exactly nn.Linear's own layout);
* to_q | to_kv concatenated to one [1536, 512] matrix (base_attention.py:31-32: q, then k, then v);
* GLU producers (pointwise_conv1, glu1, glu2) row-interleaved in groups of 16 so an output channel
  and its gate land in the same 32-column chunk of the GEMM epilogue;
* BatchNorm1d (eval, eps 1e-5) folded into the depthwise taps: w' = w * g / sqrt(var + eps),
  b' = (b - mean) * g / sqrt(var + eps) + beta  (base_conv.py:66-67);
* LayerNorm folding (norm1..norm4 of every conform_blocke, Gconform.py:57-62): for the Linear behind each of them
  W' = bf16(W * gamma), s = row sums of W', b' = bias + W . beta, so that  LN(x) . W^T + bias = rstd * (bf16(x) . W'^T -
  mean * s) + b'  is evaluated in the consumer GEMM's epilogue (csrc/gemm.cu, SOME_EPI_LN_*);
* mel filterbank (librosa htk / slaney, spec.py:22-28) as per-filter contiguous bin ranges, periodic
  Hann window and double-precision FFT twiddles.
"""
from __future__ import annotations

from typing import Dict, List

import numpy as np
import torch

from . import _lib
from .config import DIM

BN_EPS = 1e-5


# --------------------------------------------------------------------------- mel front-end tables
def mel_filterbank_htk_slaney(sr: int, n_fft: int, n_mels: int, fmin: float, fmax: float) -> np.ndarray:
    """librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax, htk=True) with the default Slaney area
    normalisation (librosa 0.9.x), as called at modules/rmvpe/spec.py:22-28.  float32 [n_mels, 1 + n_fft/2]."""
    if fmax is None:
        fmax = sr / 2.0
    n_bins = 1 + n_fft // 2
    fft_freqs = np.linspace(0.0, sr / 2.0, n_bins)
    to_mel = lambda f: 2595.0 * np.log10(1.0 + f / 700.0)
    edges_mel = np.linspace(to_mel(float(fmin)), to_mel(float(fmax)), n_mels + 2)
    edges_hz = 700.0 * (10.0 ** (edges_mel / 2595.0) - 1.0)
    width = np.diff(edges_hz)
    bank = np.zeros((n_mels, n_bins), dtype=np.float32)
    for m in range(n_mels):
        rising = (fft_freqs - edges_hz[m]) / width[m]
        falling = (edges_hz[m + 2] - fft_freqs) / width[m + 1]
        bank[m] = np.maximum(0.0, np.minimum(rising, falling))
    bank *= (2.0 / (edges_hz[2:] - edges_hz[:-2]))[:, None]
    return bank


def mel_tables(config: dict, device) -> Dict[str, torch.Tensor]:
    sr, n_fft = config['audio_sample_rate'], config['win_size']
    bank = mel_filterbank_htk_slaney(sr, n_fft, config['units_dim'], config['fmin'], config['fmax'])
    nz = bank != 0
    start = np.zeros(bank.shape[0], dtype=np.int32)
    count = np.zeros(bank.shape[0], dtype=np.int32)
    weights = np.zeros((bank.shape[0], _lib.MEL_MAXW), dtype=np.float32)
    for m in range(bank.shape[0]):
        idx = np.nonzero(nz[m])[0]
        if idx.size == 0:
            continue
        lo, hi = int(idx[0]), int(idx[-1])
        if hi >= _lib.MEL_BINS or hi - lo + 1 > _lib.MEL_MAXW:
            raise NotImplementedError(
                f'mel filter {m} spans bins {lo}..{hi}: outside what the fused kernel keeps '
                f'({_lib.MEL_BINS} bins, {_lib.MEL_MAXW} per filter); fmin/fmax/sr differ from the shipped configs')
        start[m], count[m] = lo, hi - lo + 1
        weights[m, :hi - lo + 1] = bank[m, lo:hi + 1]
    # twiddles of the 32 x 32 register FFT (mel.cu): W_1024^(n2 k1) at [k1 * 32 + n2] (between the two 32-point passes),
    # then W_2048^k for the real-FFT unpack of bins k < 372; computed in double
    k1, n2 = np.meshgrid(np.arange(32, dtype=np.float64), np.arange(32, dtype=np.float64), indexing='ij')
    ang = -2.0 * np.pi * (k1 * n2).reshape(-1) / 1024.0
    parts = [np.stack([np.cos(ang), np.sin(ang)], axis=1)]
    ang = -2.0 * np.pi * np.arange(_lib.MEL_BINS, dtype=np.float64) / 2048.0
    parts.append(np.stack([np.cos(ang), np.sin(ang)], axis=1))
    tw = np.concatenate(parts, axis=0).astype(np.float32)
    assert tw.shape == (_lib.MEL_TW, 2)
    window = torch.hann_window(n_fft, periodic=True, dtype=torch.float32)    # spec.py:45 torch.hann_window
    return {
        'mel_start': torch.from_numpy(start).to(device),
        'mel_count': torch.from_numpy(count).to(device),
        'mel_weights': torch.from_numpy(weights).to(device),
        'twiddle': torch.from_numpy(tw).to(device),
        'window': window.to(device),
        'bank': bank,
    }


# --------------------------------------------------------------------------- trunk weights
def glu_pack_rows(w: torch.Tensor) -> torch.Tensor:
    """[2C, ...] (rows 0..C-1 = out, C..2C-1 = gate) -> groups of 32 rows: 16 out rows then their 16 gates."""
    c = w.shape[0] // 2
    assert c % 16 == 0
    out = w[:c].reshape(c // 16, 16, *w.shape[1:])
    gate = w[c:].reshape(c // 16, 16, *w.shape[1:])
    return torch.cat([out, gate], dim=1).reshape(w.shape)


def _pad32(v: torch.Tensor) -> torch.Tensor:
    n = v.shape[0]
    pad = (-n) % 32
    return torch.cat([v, v.new_zeros(pad)]) if pad else v


class RoundingRegistry:
    """bf16 weight tensor (by device pointer) -> (fp32 master of exactly what was rounded, the bias tensor of that layer).
    Filled while the checkpoint is packed, consumed once by Engine.calibrate() (bias correction for the weight rounding:
    bias += (W - bf16(W)) . E[a]), then dropped."""

    def __init__(self, device):
        self.device = device
        self.entries: Dict[int, tuple] = {}

    def round(self, master: torch.Tensor, bias=None) -> torch.Tensor:
        master = master.to(device=self.device, dtype=torch.float32).contiguous()
        w = master.to(torch.bfloat16).contiguous()
        self.entries[w.data_ptr()] = (master, w, bias)
        return w

    def attach_bias(self, w: torch.Tensor, bias: torch.Tensor):
        m, ww, _ = self.entries[w.data_ptr()]
        self.entries[w.data_ptr()] = (m, ww, bias)


class BlockWeights:
    """Device tensors of one conform_blocke (Gconform.py:37-63)."""

    def __init__(self, sd, p: str, device, reg: 'RoundingRegistry'):
        f32 = lambda t: t.to(device=device, dtype=torch.float32).contiguous()

        def bf(t, bias=None):
            return reg.round(t, bias)

        self.ln_g = [f32(sd[f'{p}.norm{i}.weight']) for i in range(1, 6)]
        self.ln_b = [f32(sd[f'{p}.norm{i}.bias']) for i in range(1, 6)]
        self.ffn = []
        for name in ('ffn1', 'ffn2'):
            b1, b2 = f32(sd[f'{p}.{name}.ln1.bias']), f32(sd[f'{p}.{name}.ln2.bias'])
            self.ffn.append(dict(w1=bf(sd[f'{p}.{name}.ln1.weight'], b1), b1=b1, w2=bf(sd[f'{p}.{name}.ln2.weight'], b2), b2=b2))
        self.w_qkv = bf(torch.cat([sd[f'{p}.att.to_q.weight'], sd[f'{p}.att.to_kv.weight']], dim=0))   # no bias to correct
        self.b_out = f32(sd[f'{p}.att.to_out.0.bias'])
        self.w_out = bf(sd[f'{p}.att.to_out.0.weight'], self.b_out)
        self.b_pw1 = f32(glu_pack_rows(sd[f'{p}.conv.pointwise_conv1.bias']))
        self.w_pw1 = bf(glu_pack_rows(sd[f'{p}.conv.pointwise_conv1.weight'][:, :, 0]), self.b_pw1)
        scale = sd[f'{p}.conv.norm.weight'].double() / torch.sqrt(sd[f'{p}.conv.norm.running_var'].double() + BN_EPS)
        dw = sd[f'{p}.conv.depthwise_conv.weight'][:, 0, :].double()            # [C, K]
        self.w_dw = f32((dw * scale[:, None]).t())                              # [K, C]
        self.b_dw = f32((sd[f'{p}.conv.depthwise_conv.bias'].double() - sd[f'{p}.conv.norm.running_mean'].double())
                        * scale + sd[f'{p}.conv.norm.bias'].double())
        self.b_pw2 = f32(sd[f'{p}.conv.pointwise_conv2.bias'])
        self.w_pw2 = bf(sd[f'{p}.conv.pointwise_conv2.weight'][:, :, 0], self.b_pw2)

        # ---- LayerNorm-folded consumers: (norm index, weight [N, 512], bias or None) -> (W' bf16, s f32, b' f32)
        def fold(i, w, b, pack=lambda t: t):
            g64, b64 = sd[f'{p}.norm{i}.weight'].double(), sd[f'{p}.norm{i}.bias'].double()
            w64 = w.double()
            bias = f32(pack((w64 @ b64 + (b.double() if b is not None else 0.0)).float()))
            wf = bf(pack((w64 * g64[None, :]).float()), bias)
            s_col = wf.double().sum(dim=1)                           # sums of the ROUNDED operand the tensor core sees
            return wf, f32(s_col), bias

        self.ffn_fold = [fold(1, sd[f'{p}.ffn1.ln1.weight'], sd[f'{p}.ffn1.ln1.bias']),
                         fold(4, sd[f'{p}.ffn2.ln1.weight'], sd[f'{p}.ffn2.ln1.bias'])]
        self.qkv_fold = fold(2, torch.cat([sd[f'{p}.att.to_q.weight'], sd[f'{p}.att.to_kv.weight']], dim=0), None)
        self.pw1_fold = fold(3, sd[f'{p}.conv.pointwise_conv1.weight'][:, :, 0], sd[f'{p}.conv.pointwise_conv1.bias'],
                             pack=glu_pack_rows)


class ModelWeights:
    """All device tensors of Gmidi_conform (Gconform.py:92-140); index 0 = midi stream (att1), 1 = bound (att2)."""

    def __init__(self, sd, config: dict, device):
        args = config['midi_extractor_args']
        self.lay = args['lay']
        self.outdim = config['midi_num_bins']
        self.rounding = reg = RoundingRegistry(device)      # dropped by Engine.calibrate()
        bf = reg.round
        f32 = lambda t: t.to(device=device, dtype=torch.float32).contiguous()
        self.b_in = [f32(sd['model.inln.bias']), f32(sd['model.inln1.bias'])]
        self.w_in = [bf(sd['model.inln.weight'], self.b_in[0]), bf(sd['model.inln1.weight'], self.b_in[1])]
        self.blocks: List[List[BlockWeights]] = []      # [lay + 1][2]
        self.glu_w, self.glu_b = [], []                 # [lay][2]: index 0 = glu1 (fed by midi), 1 = glu2 (fed by bound)
        for i in range(self.lay):
            p = f'model.cf_lay.{i}'
            self.blocks.append([BlockWeights(sd, p + '.att1', device, reg), BlockWeights(sd, p + '.att2', device, reg)])
            self.glu_b.append([f32(glu_pack_rows(sd[p + '.glu1.0.bias'])), f32(glu_pack_rows(sd[p + '.glu2.0.bias']))])
            self.glu_w.append([bf(glu_pack_rows(sd[p + '.glu1.0.weight']), self.glu_b[-1][0]),
                               bf(glu_pack_rows(sd[p + '.glu2.0.weight']), self.glu_b[-1][1])])
        self.blocks.append([BlockWeights(sd, 'model.att1', device, reg), BlockWeights(sd, 'model.att2', device, reg)])
        self.b_head = f32(_pad32(sd['model.outln.bias']))
        self.w_head = bf(sd['model.outln.weight'], self.b_head)          # [outdim, 512]
        self.w_cut = f32(sd['model.cutheard.weight'][0])                 # [512]
        self.b_cut = float(sd['model.cutheard.bias'][0])
        assert self.w_in[0].shape == (DIM, config['units_dim'])


def build_c_model(w: ModelWeights, ln_fold: bool = True):
    """ctypes mirror (include/some_b200.h: some_model) of the packed weights for the native launch sequencer
    some_forward.  Returns (ModelC, keepalive): the struct only holds raw pointers, `keepalive` owns the arrays."""
    import ctypes as C
    nblk = (w.lay + 1) * 2
    blocks = (_lib.BlockWeightsC * nblk)()
    for i, pair in enumerate(w.blocks):
        for s, bw in enumerate(pair):
            b = blocks[2 * i + s]
            for k in range(5):
                b.ln_g[k], b.ln_b[k] = bw.ln_g[k].data_ptr(), bw.ln_b[k].data_ptr()
            for k in range(2):
                f = bw.ffn[k]
                b.ffn_w1[k], b.ffn_b1[k] = f['w1'].data_ptr(), f['b1'].data_ptr()
                b.ffn_w2[k], b.ffn_b2[k] = f['w2'].data_ptr(), f['b2'].data_ptr()
            b.w_qkv, b.w_out, b.b_out = bw.w_qkv.data_ptr(), bw.w_out.data_ptr(), bw.b_out.data_ptr()
            b.w_pw1, b.b_pw1 = bw.w_pw1.data_ptr(), bw.b_pw1.data_ptr()
            b.w_dw, b.b_dw = bw.w_dw.data_ptr(), bw.b_dw.data_ptr()
            b.w_pw2, b.b_pw2 = bw.w_pw2.data_ptr(), bw.b_pw2.data_ptr()
            for k in range(2):
                b.ffn_w1f[k], b.ffn_s1[k], b.ffn_b1f[k] = (t.data_ptr() for t in bw.ffn_fold[k])
            b.w_qkvf, b.s_qkv, b.b_qkvf = (t.data_ptr() for t in bw.qkv_fold)
            b.w_pw1f, b.s_pw1, b.b_pw1f = (t.data_ptr() for t in bw.pw1_fold)
    n_glu = max(w.lay * 2, 1)
    glu_w = (C.c_void_p * n_glu)()
    glu_b = (C.c_void_p * n_glu)()
    for i in range(w.lay):
        for s in range(2):
            glu_w[2 * i + s] = w.glu_w[i][s].data_ptr()
            glu_b[2 * i + s] = w.glu_b[i][s].data_ptr()
    m = _lib.ModelC()
    m.lay, m.outdim = w.lay, w.outdim
    for s in range(2):
        m.w_in[s], m.b_in[s] = w.w_in[s].data_ptr(), w.b_in[s].data_ptr()
    m.blocks = C.cast(blocks, C.POINTER(_lib.BlockWeightsC))
    m.glu_w = C.cast(glu_w, C.POINTER(C.c_void_p))
    m.glu_b = C.cast(glu_b, C.POINTER(C.c_void_p))
    m.w_head, m.b_head, m.w_cut, m.b_cut = w.w_head.data_ptr(), w.b_head.data_ptr(), w.w_cut.data_ptr(), w.b_cut
    m.ln_fold = int(bool(ln_fold))
    return m, (blocks, glu_w, glu_b)


def build_f32_model(sd, config: dict, device):
    """fp32 weights of the validation path (some_forward_f32, csrc/accurate.cu): the checkpoint's own tensors in nn.Linear
    layout, to_q | to_kv concatenated, BatchNorm folded into the depthwise taps (in double), nothing rounded or packed.
    Returns (ModelF32C, keepalive)."""
    import ctypes as C
    f32 = lambda t: t.to(device=device, dtype=torch.float32).contiguous()
    keep = []

    def ptr(t):
        t = f32(t)
        keep.append(t)
        return t.data_ptr()

    lay, outdim = config['midi_extractor_args']['lay'], config['midi_num_bins']
    prefixes = [f'model.cf_lay.{i}.att{s}' for i in range(lay) for s in (1, 2)] + ['model.att1', 'model.att2']
    blocks = (_lib.BlockWeightsF32C * len(prefixes))()
    for b, p in zip(blocks, prefixes):
        for k in range(5):
            b.ln_g[k], b.ln_b[k] = ptr(sd[f'{p}.norm{k + 1}.weight']), ptr(sd[f'{p}.norm{k + 1}.bias'])
        for k, name in enumerate(('ffn1', 'ffn2')):
            b.ffn_w1[k], b.ffn_b1[k] = ptr(sd[f'{p}.{name}.ln1.weight']), ptr(sd[f'{p}.{name}.ln1.bias'])
            b.ffn_w2[k], b.ffn_b2[k] = ptr(sd[f'{p}.{name}.ln2.weight']), ptr(sd[f'{p}.{name}.ln2.bias'])
        b.w_qkv = ptr(torch.cat([sd[f'{p}.att.to_q.weight'], sd[f'{p}.att.to_kv.weight']], dim=0))
        b.w_out, b.b_out = ptr(sd[f'{p}.att.to_out.0.weight']), ptr(sd[f'{p}.att.to_out.0.bias'])
        b.w_pw1, b.b_pw1 = ptr(sd[f'{p}.conv.pointwise_conv1.weight'][:, :, 0]), ptr(sd[f'{p}.conv.pointwise_conv1.bias'])
        scale = sd[f'{p}.conv.norm.weight'].double() / torch.sqrt(sd[f'{p}.conv.norm.running_var'].double() + BN_EPS)
        dw = sd[f'{p}.conv.depthwise_conv.weight'][:, 0, :].double()
        b.w_dw = ptr((dw * scale[:, None]).t())
        b.b_dw = ptr((sd[f'{p}.conv.depthwise_conv.bias'].double() - sd[f'{p}.conv.norm.running_mean'].double()) * scale
                     + sd[f'{p}.conv.norm.bias'].double())
        b.w_pw2, b.b_pw2 = ptr(sd[f'{p}.conv.pointwise_conv2.weight'][:, :, 0]), ptr(sd[f'{p}.conv.pointwise_conv2.bias'])
    n_glu = max(2 * lay, 1)
    glu_w, glu_b = (C.c_void_p * n_glu)(), (C.c_void_p * n_glu)()
    for i in range(lay):
        for s in range(2):
            glu_w[2 * i + s] = ptr(sd[f'model.cf_lay.{i}.glu{s + 1}.0.weight'])
            glu_b[2 * i + s] = ptr(sd[f'model.cf_lay.{i}.glu{s + 1}.0.bias'])
    m = _lib.ModelF32C()
    m.lay, m.outdim = lay, outdim
    m.w_in[0], m.w_in[1] = ptr(sd['model.inln.weight']), ptr(sd['model.inln1.weight'])
    m.b_in[0], m.b_in[1] = ptr(sd['model.inln.bias']), ptr(sd['model.inln1.bias'])
    m.blocks = C.cast(blocks, C.POINTER(_lib.BlockWeightsF32C))
    m.glu_w, m.glu_b = C.cast(glu_w, C.POINTER(C.c_void_p)), C.cast(glu_b, C.POINTER(C.c_void_p))
    m.w_head, m.b_head = ptr(sd['model.outln.weight']), ptr(sd['model.outln.bias'])
    m.w_cut, m.b_cut = ptr(sd['model.cutheard.weight'][0]), float(sd['model.cutheard.bias'][0])
    return m, (keep, blocks, glu_w, glu_b)

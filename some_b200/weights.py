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

import itertools
from collections import namedtuple
from types import SimpleNamespace
from typing import Dict, List

import numpy as np
import torch

from . import _lib
from .config import DIM, FFN_DIM

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


def checkpoint_block(sd, p: str) -> SimpleNamespace:
    """The checkpoint tensors of one conform_blocke under BlockWeights' names: to_q | to_kv concatenated, 1x1 convolutions
    squeezed to [N, K], BatchNorm folded into the depthwise taps in float64, taps transposed to [K][C].  Neither rounded nor
    GLU-packed: the fp32 validation path runs them as they are, BlockWeights packs them."""
    d = lambda n: sd[f'{p}.{n}'].double()
    scale = d('conv.norm.weight') / torch.sqrt(d('conv.norm.running_var') + BN_EPS)
    return SimpleNamespace(
        ln_g=[sd[f'{p}.norm{i}.weight'] for i in range(1, 6)], ln_b=[sd[f'{p}.norm{i}.bias'] for i in range(1, 6)],
        ffn=[dict(w1=sd[f'{p}.{f}.ln1.weight'], b1=sd[f'{p}.{f}.ln1.bias'], w2=sd[f'{p}.{f}.ln2.weight'],
                  b2=sd[f'{p}.{f}.ln2.bias']) for f in ('ffn1', 'ffn2')],
        w_qkv=torch.cat([sd[f'{p}.att.to_q.weight'], sd[f'{p}.att.to_kv.weight']], dim=0),
        w_out=sd[f'{p}.att.to_out.0.weight'], b_out=sd[f'{p}.att.to_out.0.bias'],
        w_pw1=sd[f'{p}.conv.pointwise_conv1.weight'][:, :, 0], b_pw1=sd[f'{p}.conv.pointwise_conv1.bias'],
        w_dw=(d('conv.depthwise_conv.weight')[:, 0, :] * scale[:, None]).t(),
        b_dw=(d('conv.depthwise_conv.bias') - d('conv.norm.running_mean')) * scale + d('conv.norm.bias'),
        w_pw2=sd[f'{p}.conv.pointwise_conv2.weight'][:, :, 0], b_pw2=sd[f'{p}.conv.pointwise_conv2.bias'])


class BlockWeights:
    """Device tensors of one conform_blocke (Gconform.py:37-63)."""

    def __init__(self, sd, p: str, device, reg: 'RoundingRegistry'):
        f32 = lambda t: t.to(device=device, dtype=torch.float32).contiguous()
        bf = reg.round
        c = checkpoint_block(sd, p)
        self.ln_g, self.ln_b = [f32(t) for t in c.ln_g], [f32(t) for t in c.ln_b]
        self.ffn = []
        for f in c.ffn:
            b1, b2 = f32(f['b1']), f32(f['b2'])
            self.ffn.append(dict(w1=bf(f['w1'], b1), b1=b1, w2=bf(f['w2'], b2), b2=b2))
        self.w_qkv = bf(c.w_qkv)                        # no bias to correct
        self.b_out = f32(c.b_out)
        self.w_out = bf(c.w_out, self.b_out)
        self.b_pw1 = f32(glu_pack_rows(c.b_pw1))
        self.w_pw1 = bf(glu_pack_rows(c.w_pw1), self.b_pw1)
        self.w_dw, self.b_dw = f32(c.w_dw), f32(c.b_dw)
        self.b_pw2 = f32(c.b_pw2)
        self.w_pw2 = bf(c.w_pw2, self.b_pw2)

        # ---- LayerNorm-folded consumers: (norm index, weight [N, 512], bias or None) -> (W' bf16, s f32, b' f32)
        def fold(i, w, b, pack=lambda t: t):
            g64, b64 = sd[f'{p}.norm{i}.weight'].double(), sd[f'{p}.norm{i}.bias'].double()
            w64 = w.double()
            bias = f32(pack((w64 @ b64 + (b.double() if b is not None else 0.0)).float()))
            wf = bf(pack((w64 * g64[None, :]).float()), bias)
            s_col = wf.double().sum(dim=1)                           # sums of the ROUNDED operand the tensor core sees
            return wf, f32(s_col), bias

        self.ffn_fold = [fold(i, f['w1'], f['b1']) for i, f in zip((1, 4), c.ffn)]
        self.qkv_fold = fold(2, c.w_qkv, None)
        self.pw1_fold = fold(3, c.w_pw1, c.b_pw1, pack=glu_pack_rows)


class ModelWeights:
    """All device tensors of Gmidi_conform (Gconform.py:92-140); index 0 = midi stream (att1), 1 = bound (att2)."""

    def __init__(self, sd, config: dict, device):
        c = checkpoint_model(sd, config)
        self.lay, self.outdim = c.lay, c.outdim
        self.rounding = reg = RoundingRegistry(device)      # dropped by Engine.calibrate()
        bf = reg.round
        f32 = lambda t: t.to(device=device, dtype=torch.float32).contiguous()
        self.b_in = [f32(t) for t in c.b_in]
        self.w_in = [bf(t, b) for t, b in zip(c.w_in, self.b_in)]
        self.blocks: List[List[BlockWeights]] = [[BlockWeights(sd, p, device, reg) for p in ps] for ps in c.prefixes]
        # [lay][2]: index 0 = glu1 (fed by midi), 1 = glu2 (fed by bound)
        self.glu_b = [[f32(glu_pack_rows(t)) for t in pair] for pair in c.glu_b]
        self.glu_w = [[bf(glu_pack_rows(t), b) for t, b in zip(ws, bs)] for ws, bs in zip(c.glu_w, self.glu_b)]
        self.b_head = f32(_pad32(c.b_head))
        self.w_head = bf(c.w_head, self.b_head)                          # [outdim, 512]
        self.w_cut, self.b_cut = f32(c.w_cut), c.b_cut                   # [512], a float
        assert self.w_in[0].shape == (DIM, config['units_dim'])


# --------------------------------------------------------------------------- the packed model's tensors
BF16, F32 = np.dtype('<u2'), np.dtype('<f4')       # as the model file stores them: bf16 as its raw bits
# The model file's tensors of a block, keys under 'blk{j}.': (some_block_weights field, count, dtype, shape).  BlockWeights
# holds ffn_w1 .. ffn_b2 as ffn[k]['w1'] .., every other field under its own name.
BLOCK_TENSORS = [
    ('ln_g', 5, F32, (DIM,)), ('ln_b', 5, F32, (DIM,)),
    ('ffn_w1', 2, BF16, (FFN_DIM, DIM)), ('ffn_b1', 2, F32, (FFN_DIM,)),
    ('ffn_w2', 2, BF16, (DIM, FFN_DIM)), ('ffn_b2', 2, F32, (DIM,)),
    ('w_qkv', 1, BF16, (3 * DIM, DIM)), ('w_out', 1, BF16, (DIM, DIM)), ('b_out', 1, F32, (DIM,)),
    ('w_pw1', 1, BF16, (2 * DIM, DIM)), ('b_pw1', 1, F32, (2 * DIM,)),
    ('w_dw', 1, F32, (_lib.CONV_K, DIM)), ('b_dw', 1, F32, (DIM,)),
    ('w_pw2', 1, BF16, (DIM, DIM)), ('b_pw2', 1, F32, (DIM,))]
# The LayerNorm-folded consumers (some_model.ln_fold), packed at load time, never written to a model file: the BlockWeights
# triples (W', s, b'), their count and their some_block_weights fields.
FOLDED_TENSORS = [('ffn_fold', 2, ('ffn_w1f', 'ffn_s1', 'ffn_b1f')), ('qkv_fold', 1, ('w_qkvf', 's_qkv', 'b_qkvf')),
                  ('pw1_fold', 1, ('w_pw1f', 's_pw1', 'b_pw1f'))]
# The model-level tensors before and after the blocks; 'outdim' / 'outdim32': the head width, and it padded to 32 lanes.
INPUT_TENSORS = [('w_in', 2, BF16, (DIM, _lib.N_MELS)), ('b_in', 2, F32, (DIM,))]
HEAD_TENSORS = [('w_head', 1, BF16, ('outdim', DIM)), ('b_head', 1, F32, ('outdim32',)), ('w_cut', 1, F32, (DIM,)),
                ('b_cut', 1, F32, (1,))]
# Tensor: key None for the folded ones, block None for the model level; index: into an array field.
Tensor = namedtuple('Tensor', 'key block field index dtype shape')


def model_tensors(lay: int, folded: bool = False) -> List[Tensor]:
    """Every tensor of a packed model with `lay` conformer layers in the model file's order, then the folded ones if
    `folded`.  An array field's tensors go index-major with the rows of its count (ln_g.0, ln_b.0, ln_g.1, ...).  Block i of
    stream s is entry j = 2 i + s of some_model.blocks; GLU mix j = 2 i + 0 is glu1 (fed by midi), 2 i + 1 glu2."""
    def rows(table, prefix='', block=None):
        for count, group in itertools.groupby(table, key=lambda r: r[1]):
            group = list(group)
            yield from (Tensor(prefix + (f'{f}.{k}' if count > 1 else f), block, f, k if count > 1 else None, dt, shape)
                        for k in range(count) for f, _, dt, shape in group)

    out = [*rows(INPUT_TENSORS), *(t for j in range(2 * (lay + 1)) for t in rows(BLOCK_TENSORS, f'blk{j}.', j))]
    out += [Tensor(f'glu{j}.{x}', None, f'glu_{x}', j, dt, shape) for j in range(2 * lay)
            for x, dt, shape in (('w', BF16, (2 * DIM, DIM)), ('b', F32, (2 * DIM,)))]
    out += rows(HEAD_TENSORS)
    return out + [Tensor(None, j, f, k if count > 1 else None, None, None) for j in range(2 * (lay + 1)) if folded
                  for _, count, fields in FOLDED_TENSORS for k in range(count) for f in fields]


def packed_tensor(w, t: Tensor):
    """Tensor t in w: a ModelWeights, or the checkpoint_model it was packed from (b_cut: a float)."""
    obj = w if t.block is None else w.blocks[t.block // 2][t.block % 2]
    if t.field.startswith('glu_'):
        return getattr(obj, t.field)[t.index // 2][t.index % 2]
    name, pos = next(((n, fs.index(t.field)) for n, _, fs in FOLDED_TENSORS if t.field in fs),
                     ('ffn', t.field[4:]) if t.field.startswith('ffn_') else (t.field, None))
    v = getattr(obj, name) if t.index is None else getattr(obj, name)[t.index]
    return v if pos is None else v[pos]


def _c_model(model_t, block_t, w, folded: bool, upload=lambda t: t):
    """A model_t (ModelC / ModelF32C) pointing to the tensors of w (ModelWeights or checkpoint_model), each passed through
    upload.  Returns (struct, keepalive): the struct only holds raw pointers, `keepalive` owns the arrays."""
    import ctypes as C
    blocks = (block_t * (2 * (w.lay + 1)))()
    glu_w, glu_b = (C.c_void_p * max(2 * w.lay, 1))(), (C.c_void_p * max(2 * w.lay, 1))()
    m = model_t(lay=w.lay, outdim=w.outdim, blocks=C.cast(blocks, C.POINTER(block_t)),
                glu_w=C.cast(glu_w, C.POINTER(C.c_void_p)), glu_b=C.cast(glu_b, C.POINTER(C.c_void_p)))
    for t in model_tensors(w.lay, folded):
        s, v = m if t.block is None else blocks[t.block], packed_tensor(w, t)
        if not hasattr(type(s), t.field):
            raise AttributeError(f'{type(s).__name__} has no field {t.field!r}')
        v = v if isinstance(v, float) else upload(v).data_ptr()
        if t.index is None:
            setattr(s, t.field, v)
        else:
            getattr(s, t.field)[t.index] = v
    return m, (blocks, glu_w, glu_b)


def build_c_model(w: ModelWeights, ln_fold: bool = True):
    """ctypes mirror (include/some_b200.h: some_model) of the packed weights for the native launch sequencer
    some_forward.  Returns (ModelC, keepalive): the struct only holds raw pointers, `keepalive` owns the arrays."""
    m, keep = _c_model(_lib.ModelC, _lib.BlockWeightsC, w, folded=True)
    m.ln_fold = int(bool(ln_fold))
    return m, keep


def checkpoint_model(sd, config: dict) -> SimpleNamespace:
    """The model-level checkpoint tensors under ModelWeights' names, unpacked like checkpoint_block, and the checkpoint
    prefixes of the blocks ([lay + 1][2], as ModelWeights.blocks)."""
    lay = config['midi_extractor_args']['lay']
    glu = lambda kind: [[sd[f'model.cf_lay.{i}.glu{s}.0.{kind}'] for s in (1, 2)] for i in range(lay)]
    return SimpleNamespace(
        lay=lay, outdim=config['midi_num_bins'], w_in=[sd['model.inln.weight'], sd['model.inln1.weight']],
        b_in=[sd['model.inln.bias'], sd['model.inln1.bias']], glu_w=glu('weight'), glu_b=glu('bias'),
        prefixes=[[f'model.cf_lay.{i}.att1', f'model.cf_lay.{i}.att2'] for i in range(lay)] + [['model.att1', 'model.att2']],
        w_head=sd['model.outln.weight'], b_head=sd['model.outln.bias'], w_cut=sd['model.cutheard.weight'][0],
        b_cut=float(sd['model.cutheard.bias'][0]))


def checkpoint_f32(sd, config: dict) -> SimpleNamespace:
    """checkpoint_model with its blocks: the fp32 model's tensors, readable by packed_tensor under model_tensors_f32."""
    ck = checkpoint_model(sd, config)
    ck.blocks = [[checkpoint_block(sd, p) for p in ps] for ps in ck.prefixes]
    return ck


def model_tensors_f32(lay: int) -> List[Tensor]:
    """The tensors of the fp32 model (some_model_f32; an fp32 model file, some_b200/export.py): model_tensors' names, order
    and fields, every one f32 (the checkpoint's own values, nothing rounded or packed), b_head unpadded.  The C mirror is
    kBlockRowsF32 / expected_tensors in csrc/session.cu."""
    return [t._replace(dtype=F32, shape=('outdim',) if t.field == 'b_head' else t.shape) for t in model_tensors(lay)]


def build_f32_model(sd, config: dict, device):
    """fp32 weights of some_forward_f32 / some_forward_f32_tiled (csrc/accurate.cu): checkpoint_model and checkpoint_block,
    nothing rounded or packed.  Returns (ModelF32C, keepalive)."""
    keep = []

    def upload(t):
        keep.append(t.to(device=device, dtype=torch.float32).contiguous())
        return keep[-1]

    m, arrays = _c_model(_lib.ModelF32C, _lib.BlockWeightsF32C, checkpoint_f32(sd, config), False, upload)
    return m, (keep, *arrays)

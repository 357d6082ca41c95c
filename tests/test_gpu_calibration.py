"""The load-time bias correction (Engine.calibrate): every bf16-rounded weight W of the packed model moves its layer's bias by
(W_master - bf16(W)) . E[a], with E[a] the column means of the GEMM operand that the native sequencer records on a 4 s
calibration clip (some_forward with a some_calibration, csrc/forward.cu; some_col_means, csrc/rowwise.cu).

* bookkeeping of the rounding registry against the checkpoint (CPU);
* the sequencer's records: one per GEMM, in launch order, with the right weights and K;
* the recorded operand means against a float64 restatement of the trunk that rounds to bf16 where the kernels store bf16;
* the corrected biases, bit for bit, and every other tensor of the model untouched;
* some_col_means at the sequencer's shapes and slot counts against float64, within a bound derived from its summation order;
* the drift of the boundary probabilities it removes, against the fp32 validation path on eight 30 s clips.

Every GPU test prints what it measured (run with -s to see the report)."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from some_b200 import _lib, synth
from some_b200.weights import ModelWeights, RoundingRegistry, build_c_model, glu_pack_rows

gpu = pytest.mark.gpu
KINDS = ('two_head', 'quant_two_head', 'midi_conformer')
SEED = 1234
CAL_SEED, CAL_SECONDS = 20240917, 4.0          # the clip Engine.calibrate() runs
U = 2.0 ** -24                                 # fp32 unit roundoff


def bf(t):
    """bf16 rounding of a float64 tensor, back in float64 (a kernel's bf16 store)."""
    return t.to(torch.bfloat16).double()


# ------------------------------------------------------------------------------------------------ packed model <-> checkpoint
def rounded_layers(sd, w: ModelWeights):
    """Every bf16 weight of the packed model: (field, bf16 weight, its bias tensor or None, the fp32 master it must be the
    rounding of, the fp32 bias the checkpoint gives it), restated from the checkpoint names."""
    d = lambda n: sd[n].double()
    glu = glu_pack_rows
    out = [(f'w_in[{s}]', w.w_in[s], w.b_in[s], sd[f'model.{n}.weight'], sd[f'model.{n}.bias'])
           for s, n in enumerate(('inln', 'inln1'))]
    prefixes = [[f'model.cf_lay.{i}.att{s + 1}' for s in range(2)] for i in range(w.lay)] + [['model.att1', 'model.att2']]
    for i, pair in enumerate(w.blocks):
        for s, bw in enumerate(pair):
            p, f = prefixes[i][s], f'blocks[{i}][{s}]'

            def folded(norm, wt, b, pack=lambda t: t):
                g, beta = d(f'{p}.norm{norm}.weight'), d(f'{p}.norm{norm}.bias')
                return pack((wt.double() * g[None, :]).float()), pack((wt.double() @ beta + (b.double() if b is not None else 0.0)).float())

            for k, name in enumerate(('ffn1', 'ffn2')):
                out.append((f'{f}.ffn[{k}].w1', bw.ffn[k]['w1'], bw.ffn[k]['b1'], sd[f'{p}.{name}.ln1.weight'], sd[f'{p}.{name}.ln1.bias']))
                out.append((f'{f}.ffn[{k}].w2', bw.ffn[k]['w2'], bw.ffn[k]['b2'], sd[f'{p}.{name}.ln2.weight'], sd[f'{p}.{name}.ln2.bias']))
                out.append((f'{f}.ffn_fold[{k}]', bw.ffn_fold[k][0], bw.ffn_fold[k][2],
                            *folded(1 + 3 * k, sd[f'{p}.{name}.ln1.weight'], sd[f'{p}.{name}.ln1.bias'])))
            qkv = torch.cat([sd[f'{p}.att.to_q.weight'], sd[f'{p}.att.to_kv.weight']], dim=0)
            out.append((f'{f}.w_qkv', bw.w_qkv, None, qkv, None))
            out.append((f'{f}.qkv_fold', bw.qkv_fold[0], bw.qkv_fold[2], *folded(2, qkv, None)))
            out.append((f'{f}.w_out', bw.w_out, bw.b_out, sd[f'{p}.att.to_out.0.weight'], sd[f'{p}.att.to_out.0.bias']))
            pw1, pw1_b = sd[f'{p}.conv.pointwise_conv1.weight'][:, :, 0], sd[f'{p}.conv.pointwise_conv1.bias']
            out.append((f'{f}.w_pw1', bw.w_pw1, bw.b_pw1, glu(pw1), glu(pw1_b)))
            out.append((f'{f}.pw1_fold', bw.pw1_fold[0], bw.pw1_fold[2], *folded(3, pw1, pw1_b, glu)))
            out.append((f'{f}.w_pw2', bw.w_pw2, bw.b_pw2, sd[f'{p}.conv.pointwise_conv2.weight'][:, :, 0],
                        sd[f'{p}.conv.pointwise_conv2.bias']))
    for i in range(w.lay):
        for s in range(2):
            n = f'model.cf_lay.{i}.glu{s + 1}.0'
            out.append((f'glu_w[{i}][{s}]', w.glu_w[i][s], w.glu_b[i][s], glu(sd[n + '.weight']), glu(sd[n + '.bias'])))
    out.append(('w_head', w.w_head, w.b_head, sd['model.outln.weight'], sd['model.outln.bias']))
    return out


def named_tensors(obj, name='w'):
    """(name, tensor) of every tensor a ModelWeights holds (the rounding registry aside)."""
    if isinstance(obj, torch.Tensor):
        yield name, obj
    elif isinstance(obj, (list, tuple)):
        for i, v in enumerate(obj):
            yield from named_tensors(v, f'{name}[{i}]')
    elif isinstance(obj, dict):
        for k, v in obj.items():
            yield from named_tensors(v, f'{name}[{k!r}]')
    elif hasattr(obj, '__dict__') and not isinstance(obj, RoundingRegistry):
        for k, v in vars(obj).items():
            yield from named_tensors(v, f'{name}.{k}')


@pytest.mark.parametrize('kind', KINDS)
def test_registry_pairs_every_rounded_weight_with_its_own_bias(kind):
    """CPU: the registry holds exactly the model's bf16 weights, each with the fp32 master it was rounded from (same packing)
    and the bias tensor of its own layer; no bias serves two weights; only to_q|to_kv (no bias in the model) has none.  The
    pointers the sequencer receives (build_c_model) pair every weight with that same bias."""
    config = synth.named_config(kind)
    sd = synth.fabricate_state_dict(config, seed=SEED)
    w = ModelWeights(sd, config, 'cpu')
    reg = w.rounding
    layers = rounded_layers(sd, w)
    assert len(layers) == 2 + 2 * 12 * (w.lay + 1) + 2 * w.lay + 1
    assert sorted(reg.entries) == sorted(t.data_ptr() for _, t, *_ in layers), 'registry and packed weights differ'
    seen_bias = {}
    for field, wt, bias, master_want, bias_want in layers:
        master, rounded, reg_bias = reg.entries[wt.data_ptr()]
        assert rounded is wt, field
        assert master.dtype == torch.float32 and master.shape == wt.shape, field
        assert torch.equal(master, master_want.float()), f'{field}: master is not the packed checkpoint tensor'
        assert torch.equal(master.to(torch.bfloat16), rounded), f'{field}: bf16(master) != rounded weight'
        if bias is None:
            assert reg_bias is None and field.endswith('.w_qkv'), field
            continue
        assert reg_bias is bias, f'{field}: registry bias is not the layer bias'
        n = bias_want.shape[0]
        assert bias.shape[0] == (n + 31) // 32 * 32 if field == 'w_head' else bias.shape[0] == n, field
        assert torch.equal(bias[:n], bias_want.float()), f'{field}: bias is not the checkpoint bias of this layer'
        assert not bias[n:].any(), f'{field}: padding lanes are not zero'
        assert bias.data_ptr() not in seen_bias, f'{field} and {seen_bias.get(bias.data_ptr())} share a bias tensor'
        seen_bias[bias.data_ptr()] = field
    assert sum(e[2] is None for e in reg.entries.values()) == 2 * (w.lay + 1)

    # the C mirror hands the sequencer each weight together with that bias
    by_ptr = {wt.data_ptr(): (bias.data_ptr() if bias is not None else None) for _, wt, bias, *_ in layers}
    for fold in (False, True):
        m, _keep = build_c_model(w, fold)
        pairs = [(m.w_in[s], m.b_in[s]) for s in range(2)] + [(m.glu_w[i], m.glu_b[i]) for i in range(2 * w.lay)]
        pairs.append((m.w_head, m.b_head))
        for j in range(2 * (w.lay + 1)):
            b = m.blocks[j]
            pairs += [(b.ffn_w1[k], b.ffn_b1[k]) for k in range(2)] + [(b.ffn_w2[k], b.ffn_b2[k]) for k in range(2)]
            pairs += [(b.ffn_w1f[k], b.ffn_b1f[k]) for k in range(2)]
            pairs += [(b.w_out, b.b_out), (b.w_pw1, b.b_pw1), (b.w_pw2, b.b_pw2), (b.w_qkvf, b.b_qkvf), (b.w_pw1f, b.b_pw1f)]
            assert by_ptr[b.w_qkv] is None
        assert len(pairs) == len(layers) - 2 * (w.lay + 1)
        for wp, bp in pairs:
            assert by_ptr[wp] == bp, 'the sequencer receives a weight with another layer\'s bias'


# ------------------------------------------------------------------------------------------------ launch order and float64 operands
def launch_order(w: ModelWeights, fold: bool):
    """(name, K, (stream-0 weight, stream-1 weight)) of every GEMM some_forward launches, in order (csrc/forward.cu)."""
    order = [('inln|inln1', 80, (w.w_in[0], w.w_in[1]))]

    def block(pair, tag):
        two = lambda f: (f(pair[0]), f(pair[1]))
        return [(f'{tag}.ffn1.ln1', 512, two(lambda b: b.ffn_fold[0][0] if fold else b.ffn[0]['w1'])),
                (f'{tag}.ffn1.ln2', 2048, two(lambda b: b.ffn[0]['w2'])),
                (f'{tag}.to_q|to_kv', 512, two(lambda b: b.qkv_fold[0] if fold else b.w_qkv)),
                (f'{tag}.to_out', 512, two(lambda b: b.w_out)),
                (f'{tag}.pointwise_conv1', 512, two(lambda b: b.pw1_fold[0] if fold else b.w_pw1)),
                (f'{tag}.pointwise_conv2', 512, two(lambda b: b.w_pw2)),
                (f'{tag}.ffn2.ln1', 512, two(lambda b: b.ffn_fold[1][0] if fold else b.ffn[1]['w1'])),
                (f'{tag}.ffn2.ln2', 2048, two(lambda b: b.ffn[1]['w2']))]

    for i in range(w.lay):
        order += block(w.blocks[i], f'cf_lay.{i}')
        order.append((f'cf_lay.{i}.glu2|glu1', 512, (w.glu_w[i][1], w.glu_w[i][0])))      # midi += GLU(glu2(bound)), ...
    order += block(w.blocks[w.lay], 'att')
    order.append(('outln', 512, (w.w_head, w.w_head)))                                      # one group
    return order


def glu(y):
    """GLU of a GEMM output with row-interleaved weights (weights.glu_pack_rows): 16 out columns then their 16 gates."""
    m, n = y.shape
    y = y.reshape(m, n // 32, 2, 16)
    return y[:, :, 0].reshape(m, n // 2) * torch.sigmoid(y[:, :, 1].reshape(m, n // 2))


def layer_norm(x, g, b):
    mu = x.mean(1, keepdim=True)
    var = ((x - mu) ** 2).mean(1, keepdim=True)
    return (x - mu) / torch.sqrt(var + 1e-5) * g.double() + b.double()


def normalised(x):
    """Operand of a LayerNorm-folded consumer: bf16(x) (the producer's bf16 copy) normalised with the statistics of the
    unrounded row."""
    mu = x.mean(1, keepdim=True)
    var = ((x - mu) ** 2).mean(1, keepdim=True)
    return (bf(x) - mu) / torch.sqrt(var + 1e-5)


def lin(a, wt, b=None):
    y = a @ wt.double().t()
    return y + b.double()[:y.shape[1]] if b is not None else y


def attention(qkv):
    m = qkv.shape[0]
    q, k, v = (qkv[:, j * 512:(j + 1) * 512].reshape(m, 8, 64).transpose(0, 1) for j in range(3))
    p = torch.softmax(q @ k.transpose(1, 2) / 8.0, dim=-1)
    return (p @ v).transpose(0, 1).reshape(m, 512)


def dwconv_bn_silu(g, bw):
    taps = bw.w_dw.double().t().unsqueeze(1)                                  # [C, 1, 31] BN-folded
    y = F.conv1d(g.t().unsqueeze(0), taps, bw.b_dw.double(), padding=taps.shape[-1] // 2, groups=g.shape[1])
    return F.silu(y[0].t())


def block_operands(bw, x, fold, last):
    """One conform_blocke on one stream in float64: (the operands of its 8 GEMMs in launch order, x after norm5)."""
    ops = []
    for f in range(2):
        if f == 1:
            if fold:
                a = normalised(x)
                qkv = bf(lin(a, bw.qkv_fold[0], bw.qkv_fold[2]))
            else:
                a = bf(layer_norm(x, bw.ln_g[1], bw.ln_b[1]))
                qkv = bf(lin(a, bw.w_qkv))
            ops.append(a)
            att = bf(attention(qkv))
            ops.append(att)
            x = x + lin(att, bw.w_out, bw.b_out)
            if fold:
                a = normalised(x)
                g = bf(glu(lin(a, bw.pw1_fold[0], bw.pw1_fold[2])))
            else:
                a = bf(layer_norm(x, bw.ln_g[2], bw.ln_b[2]))
                g = bf(glu(lin(a, bw.w_pw1, bw.b_pw1)))
            ops.append(a)
            d = bf(dwconv_bn_silu(g, bw))
            ops.append(d)
            x = x + lin(d, bw.w_pw2, bw.b_pw2)
        if fold:
            a = normalised(x)
            w1, b1 = bw.ffn_fold[f][0], bw.ffn_fold[f][2]
        else:
            a = bf(layer_norm(x, bw.ln_g[3 * f], bw.ln_b[3 * f]))
            w1, b1 = bw.ffn[f]['w1'], bw.ffn[f]['b1']
        ops.append(a)
        h = bf(F.silu(lin(a, w1, b1)))
        ops.append(h)
        x = x + 0.5 * lin(h, bw.ffn[f]['w2'], bw.ffn[f]['b2'])
    return ops, layer_norm(x, bw.ln_g[4], bw.ln_b[4])


def reference_operands(w: ModelWeights, units: torch.Tensor, fold: bool):
    """float64 operands (stream 0, stream 1 or None) of every GEMM of one trunk pass, in launch order, from the GPU's bf16
    units, the packed bf16 weights and the current fp32 biases."""
    u = units.double()
    ops = [(u, u)]
    x = [lin(u, w.w_in[s], w.b_in[s]) for s in range(2)]
    for i in range(w.lay + 1):
        res = [block_operands(w.blocks[i][s], x[s], fold, i == w.lay) for s in range(2)]
        ops += list(zip(res[0][0], res[1][0]))
        y = [r[1] for r in res]
        if i < w.lay:
            a5 = [bf(t) for t in y]
            ops.append((a5[1], a5[0]))
            x = [y[0] + glu(lin(a5[1], w.glu_w[i][1], w.glu_b[i][1])), y[1] + glu(lin(a5[0], w.glu_w[i][0], w.glu_b[i][0]))]
    ops.append((bf(y[0]), None))                                   # norm5 of the midi stream -> outln
    return ops


# ------------------------------------------------------------------------------------------------ calibration state
def record_pass(eng, ws, m, cu_d, fold):
    """One some_forward with a some_calibration: ([(K, (w0, w1))] in record order, means [count, 2, CALIB_K])."""
    means = torch.zeros((_lib.CALIB_MAX, 2, _lib.CALIB_K), dtype=torch.float32, device=eng.device)
    cal = _lib.CalibrationC()
    cal.means = means.data_ptr()
    cmodel, _keep = build_c_model(eng.w, fold)
    _lib.check(eng.lib.some_forward(C.byref(cmodel), C.byref(ws.c), m, 1, cu_d.data_ptr(), m, _lib.EPI_BIAS_F32, None,
                                    C.byref(cal), eng._stream), 'some_forward(calibration)')
    torch.cuda.synchronize(eng.device)
    recs = [(cal.k[i], (cal.w[i][0] or 0, cal.w[i][1] or 0)) for i in range(cal.count)]
    return recs, means[:cal.count].clone()


def apply_corrections(reg, recs, means, done):
    """bias += fp32((master - rounded) . mean) for every registered weight of this pass not corrected before; returns the
    bias pointers it moved."""
    moved = []
    for i, (k, ptrs) in enumerate(recs):
        for s in range(2):
            ent = reg.entries.get(ptrs[s])
            if ent is None or ptrs[s] in done:
                continue
            done.add(ptrs[s])
            master, rounded, bias = ent
            if bias is not None:
                delta = (master.double() - rounded.double()) @ means[i, s, :k].double()
                bias[:delta.numel()] += delta.float()
                moved.append(bias.data_ptr())
    return moved


@pytest.fixture(scope='module', params=[(k, f) for k in KINDS for f in (False, True)], ids=lambda p: f'{p[0]}-fold{int(p[1])}')
def calib(request):
    """An engine built without the correction, the two calibration passes replayed by hand (the engine's mode first, then the
    other one on top of the first one's corrections), the float64 operands of both, and the engine's own calibrate()."""
    kind, fold = request.param
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    from some_b200.engine import Engine
    config = synth.named_config(kind)
    sd = synth.fabricate_state_dict(config, seed=SEED)
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv('SOME_B200_BIAS_CORRECTION', '0')
        eng = Engine(config, sd, 'cuda')
    eng.set_ln_fold(fold)
    reg, w, dev = eng.w.rounding, eng.w, eng.device
    assert reg is not None and not eng._corrected
    wave = synth.synth_waveform(CAL_SEED, seconds=CAL_SECONDS, sr=config['audio_sample_rate'])
    host, tables, cu = eng.pack([wave])
    m = int(cu[-1])
    ws = eng.workspace(m)
    wave_d, tab_d, cu_d = host.to(dev), tables.to(dev), torch.from_numpy(cu).to(dev)
    eng.run_mel(wave_d, tab_d[:1], tab_d[1:], cu_d, 1, m, None, ws.units)
    units = ws.units[:m].clone()
    before = {n: t.clone() for n, t in named_tensors(w)}
    b_cut = w.b_cut
    passes, done = [], set()
    for mode in (fold, not fold):
        recs, means = record_pass(eng, ws, m, cu_d, mode)
        with torch.no_grad():
            ref = reference_operands(w, units, mode)
        moved = apply_corrections(reg, recs, means, done)
        passes.append(dict(fold=mode, recs=recs, means=means, ref=ref, moved=moved))
    expected = {n: t.clone() for n, t in named_tensors(w)}
    for n, t in named_tensors(w):
        t.copy_(before[n])                                          # back to the uncorrected model
    registry = {p: e for p, e in reg.entries.items()}
    eng.calibrate()
    torch.cuda.synchronize(dev)
    yield dict(kind=kind, fold=fold, eng=eng, w=w, m=m, passes=passes, before=before, expected=expected, b_cut=b_cut,
               registry=registry)


@gpu
def test_sequencer_records_every_gemm_in_launch_order(calib):
    w = calib['w']
    for p in calib['passes']:
        recs, want = p['recs'], launch_order(w, p['fold'])
        assert len(recs) == 8 * (w.lay + 1) + w.lay + 2 == len(want), (p['fold'], len(recs))
        for i, ((k, ptrs), (name, k_want, wts)) in enumerate(zip(recs, want)):
            assert k == k_want, (i, name, k)
            assert ptrs == tuple(t.data_ptr() for t in wts), f'record {i} ({name}) names other weights'
        assert {p for _, ptrs in recs for p in ptrs} == {t.data_ptr() for _, _, wts in want for t in wts}


# Largest |mean_gpu - mean_f64| over the columns of a GEMM operand, 4 s calibration clip (345 frames), measured on an H100
# (sm_90a) over the three models and both launch sequences:
#   input GEMM (the GPU's own units, only the fp32 summation of some_col_means differs)  4.2e-7
#   attention output (to_out; the kernel's bf16 operands inside are not restated)    2.6e-3
#   every other operand (bf16 stores of LayerNorm, SiLU, GLU, dwconv, norm5, folded rows)  1.2e-3
MEAN_TOL_UNITS = 2e-6
MEAN_TOL_ATTENTION = 5e-3
MEAN_TOL = 2.5e-3


def mean_tol(name):
    return MEAN_TOL_UNITS if name.startswith('inln') else MEAN_TOL_ATTENTION if name.endswith('to_out') else MEAN_TOL


@gpu
def test_operand_means_match_float64(calib):
    """Every recorded mean against the float64 operand of the same GEMM, and the right layer is the nearest of all the
    operands of that pass with the same K (so a record paired with a neighbouring layer fails even within the tolerance)."""
    w, bad = calib['w'], []
    for p in calib['passes']:
        names = [n for n, *_ in launch_order(w, p['fold'])]
        refs = [[o.mean(0) if o is not None else None for o in pair] for pair in p['ref']]
        worst = {}
        for i, (k, _) in enumerate(p['recs']):
            for s in range(2):
                if refs[i][s] is None:
                    continue
                got = p['means'][i, s, :k].double()
                err = float((got - refs[i][s]).abs().max())
                group = names[i].split('.', 2 if names[i].startswith('cf_lay') else 1)[-1]
                worst[group] = max(worst.get(group, 0.0), err)
                if err >= mean_tol(names[i]):
                    bad.append(f'fold={p["fold"]} {names[i]} stream {s}: max|mean err| {err:.3e}')
                dist = {(j, t): float((got - refs[j][t]).abs().max()) for j in range(len(refs)) for t in range(2)
                        if refs[j][t] is not None and refs[j][t].numel() == k and not torch.equal(refs[j][t], refs[i][s])}
                near = min(dist, key=dist.get) if dist else None
                if near is not None and dist[near] <= err:
                    bad.append(f'fold={p["fold"]} {names[i]} stream {s}: nearer to {names[near[0]]} stream {near[1]} '
                               f'({dist[near]:.3e}) than to its own operand ({err:.3e})')
        print(f'\n{calib["kind"]} fold={int(p["fold"])}: max|mean_gpu - mean_f64| ' +
              ' '.join(f'{k}={v:.2e}' for k, v in worst.items()), end='')
    assert not bad, f'{calib["kind"]}: ' + '; '.join(bad[:8])


@gpu
def test_calibrate_moves_exactly_the_registered_biases(calib):
    """After calibrate(): every registered weight is marked corrected; each bias equals the hand-replayed fp32
    bias + fp32((master - rounded) . mean) bit for bit (the second pass replayed on top of the first one's corrections);
    every other tensor of the model is unchanged bit for bit; and each correction agrees with the one the float64 operand
    means give, within |dW| . |mean_gpu - mean_f64| (a sign flip, a doubled or a missing correction fail here
    without relying on the replay)."""
    eng, w = calib['eng'], calib['w']
    assert eng.w.rounding is None
    assert eng._corrected == set(calib['registry'])
    assert float(w.b_cut) == float(calib['b_cut'])
    moved = {ptr for p in calib['passes'] for ptr in p['moved']}
    bias_ptrs = {e[2].data_ptr() for e in calib['registry'].values() if e[2] is not None}
    assert moved == bias_ptrs, 'a registered bias was not corrected by either pass, or one was corrected twice'
    assert len(calib['passes'][0]['moved']) + len(calib['passes'][1]['moved']) == len(bias_ptrs)
    changed = 0
    for n, t in named_tensors(w):
        want = calib['expected'][n] if t.data_ptr() in bias_ptrs else calib['before'][n]
        assert torch.equal(t, want), f'{n} differs from its expected value'
        changed += not torch.equal(t, calib['before'][n])
    assert changed == len(bias_ptrs), 'a corrected bias did not move'
    pad = w.b_head[w.outdim:]
    assert not pad.any(), 'padding lanes of b_head moved'

    by_ptr = {e[2].data_ptr(): e for e in calib['registry'].values() if e[2] is not None}
    before = {t.data_ptr(): calib['before'][n] for n, t in named_tensors(w)}
    worst = 0.0
    for p in calib['passes']:
        seen = set()
        for i, (k, ptrs) in enumerate(p['recs']):
            for s in range(2):
                ent = calib['registry'].get(ptrs[s])
                if ent is None or ent[2] is None or ent[2].data_ptr() not in p['moved'] or ent[2].data_ptr() in seen:
                    continue
                seen.add(ent[2].data_ptr())
                master, rounded, bias = by_ptr[ent[2].data_ptr()]
                dw = master.double() - rounded.double()
                n = dw.shape[0]
                delta = bias[:n].double() - before[bias.data_ptr()][:n].double()
                mean_ref = p['ref'][i][s].mean(0)
                ref = dw @ mean_ref
                # |dW . mean_gpu - dW . mean_ref| <= |dW| . |mean_gpu - mean_ref|, plus the fp32 rounding of the delta and
                # of the bias update
                err = (p['means'][i, s, :k].double() - mean_ref).abs()
                bound = dw.abs() @ err + 2 * U * (bias[:n].double().abs() + 2 * delta.abs()) + 1e-30
                excess = float(((delta - ref).abs() / bound).max())
                worst = max(worst, excess)
                assert excess <= 1.0, f'{calib["kind"]} fold={p["fold"]} record {i} stream {s}: correction off by {excess:.2f}x its bound'
    print(f'\n{calib["kind"]} fold={int(calib["fold"])}: corrections vs float64 means: worst {worst:.3f} of the bound')


# ------------------------------------------------------------------------------------------------ some_col_means
def gamma(n):
    return n * U / (1 - n * U)


def producer_rows(lib, m, parts, seed):
    """bf16 rows and their ln_stats slots as the sequencer's producers write them: some_row_stats (1 slot), the residual
    GEMM epilogue SOME_EPI_RESID_F32_LN (4 slots) or the GLU-mix epilogue SOME_EPI_GLU_RESID_F32_LN (8 slots)."""
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(m, 512, device=dev, generator=g) * 1.7 + 0.4
    xb = torch.full((m, 512), float('nan'), device=dev, dtype=torch.bfloat16)
    st = torch.full((m, _lib.LN_SLOTS, 2), float('nan'), device=dev)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if parts == 1:
        a = _lib.RowStatsArgs()
        a.x, a.out_bf16, a.ln_stats, a.groups, a.M = _lib.pair(x, x), _lib.pair(xb, xb), _lib.pair(st, st), 1, m
        _lib.check(lib.some_row_stats(C.byref(a), stream), 'some_row_stats')
    else:
        n = 512 if parts == 4 else 1024
        a_op = (torch.randn(m, 512, device=dev, generator=g) + 0.3).to(torch.bfloat16)
        wt = (torch.randn(n, 512, device=dev, generator=g) / 512 ** 0.5).to(torch.bfloat16)
        b = torch.randn(n, device=dev, generator=g) * 0.3
        ga = _lib.GemmArgs()
        ga.A, ga.W, ga.bias, ga.out, ga.resid = (_lib.pair(t, t) for t in (a_op, wt, b, x, x))
        ga.out_bf16, ga.ln_stats = _lib.pair(xb, xb), _lib.pair(st, st)
        ga.groups, ga.M, ga.N, ga.K, ga.lda, ga.ld_out, ga.alpha = 1, m, n, 512, 512, 512, 1.0
        ga.epilogue = _lib.EPI_RESID_F32_LN if parts == 4 else _lib.EPI_GLU_RESID_F32_LN
        _lib.check(lib.some_gemm(C.byref(ga), stream), 'some_gemm')
    torch.cuda.synchronize()
    assert not torch.isnan(st[:, :parts]).any() and not torch.isnan(xb.float()).any()
    return xb, st


def col_means_reference(a, st, parts):
    """float64 column means of the operand and the bound on the kernel's error, derived from its arithmetic: per row (when
    normalised) fp32 sums of `parts` slots, s / K, max(q / K - mean^2, 0), rsqrtf (2 ulp), (v - mean) * r; per column 8
    strided fp32 chains over the rows (warp w takes rows w, w + 8, ...), their 8 partials added, then x fp32(1 / M)."""
    m, k = a.shape
    v = a.double()
    e = torch.zeros_like(v)
    if st is not None:
        sl = st[:, :parts].double()
        s, q = sl[:, :, 0].sum(1, keepdim=True), sl[:, :, 1].sum(1, keepdim=True)
        es = gamma(parts - 1) * sl[:, :, 0].abs().sum(1, keepdim=True)
        eq = gamma(parts - 1) * q
        mu, var = s / k, q / k - (s / k) ** 2
        e_mu = es / k + U * (mu.abs() + es / k)
        e_var = ((eq / k) * (1 + U) + U * (q / k) + e_mu * (2 * mu.abs() + e_mu) + U * (mu.abs() + e_mu) ** 2
                 + U * (var.abs() + e_mu * (2 * mu.abs() + e_mu) + eq / k))
        t = var + 1e-5
        e_t = e_var + U * t + abs(float(np.float32(1e-5)) - 1e-5)
        r = 1.0 / torch.sqrt(t)
        e_r = r * (0.5 * e_t / (t - e_t) * 1.01 + 4 * U)           # rsqrtf: 2 ulp = 4 u relative
        d = v - mu
        v = d * r
        e = (e_mu + U * (d.abs() + e_mu)) * (r + e_r) + d.abs() * e_r + U * (v.abs() + e_r * d.abs())
    n_chain = (m + 7) // 8
    acc = gamma(n_chain - 1 + 7) * (v.abs() + e).sum(0)
    mean = v.mean(0)
    bound = (e.sum(0) + acc) / m * (1 + 3 * U) + 3 * U * mean.abs()
    return mean, bound


@gpu
@pytest.mark.parametrize('m', [1, 7, 8, 9, 345, 3001])
@pytest.mark.parametrize('k,parts', [(80, 0), (512, 0), (2048, 0), (512, 1), (512, 4), (512, 8)])
def test_col_means_at_the_sequencer_shapes(m, k, parts):
    """some_col_means with lda > K at the sequencer's K (80 is not a multiple of the kernel's 32-column blocks) and slot
    counts (1: some_row_stats in front of block 0, 4: residual GEMMs, 8: the GLU mix), on the statistics the producers
    write, against float64 within the bound derived from the kernel's order of operations."""
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    lib = _lib.load()
    lda = k + 24
    buf = torch.full((m, lda), float('nan'), device='cuda', dtype=torch.bfloat16)
    if parts:
        xb, st = producer_rows(lib, m, parts, seed=100 * parts + m)
        buf[:, :k] = xb
    else:
        g = torch.Generator(device='cuda').manual_seed(m + k)
        buf[:, :k] = (F.silu(torch.randn(m, k, device='cuda', generator=g) * 2) + 0.05).to(torch.bfloat16)
        st = None
    out = torch.full((k + 32,), float('nan'), device='cuda')
    _lib.check(lib.some_col_means(buf.data_ptr(), m, k, lda, st.data_ptr() if st is not None else None, max(parts, 1),
                                  out.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)), 'some_col_means')
    torch.cuda.synchronize()
    assert torch.isnan(out[k:]).all(), 'some_col_means wrote past column K'
    mean, bound = col_means_reference(buf[:, :k], st, parts)
    err = (out[:k].double() - mean).abs()
    worst = float((err / bound).max())
    print(f'\ncol_means M={m} K={k} parts={parts}: max err {float(err.max()):.2e}, worst {worst:.3f} of the bound')
    assert worst <= 1.0, (float(err.max()), float(bound.min()))


# ------------------------------------------------------------------------------------------------ the drift it removes
# Mean error of the boundary probabilities (bf16 path - fp32 validation path) per 30 s clip, measured on an H100 (sm_90a) over
# bench.py's eight clips; mean |.| over the clips without -> with the correction:
#   two_head        unfolded 3.35e-4 -> 3.4e-5   folded 3.24e-4 -> 8.6e-5
#   quant_two_head  unfolded 3.07e-4 -> 1.35e-4  folded 4.3e-5  -> 3.7e-5
#   midi_conformer  unfolded 2.93e-4 -> 8.0e-5   folded 2.12e-4 -> 6.9e-5
# Largest per-clip |mean| with the correction: 2.1e-4 (midi_conformer, folded); over both modes the correction divides the
# mean |.| by 5.5 (two_head), 2.0 (quant_two_head) and 3.4 (midi_conformer).  The run is deterministic; the margins leave
# room for changes of the kernels' rounding.
BOUNDS_MEAN_TOL = 3e-4
DRIFT_FACTOR = 1.5


@pytest.fixture(scope='module')
def drift_clips():
    return [synth.synth_waveform(1000 + j, seconds=30.0) for j in range(8)]      # bench.py's clip pool


@gpu
@pytest.mark.parametrize('kind', KINDS)
def test_correction_removes_the_bounds_drift(kind, drift_clips):
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    from some_b200.engine import Engine
    config = synth.named_config(kind)
    sd = synth.fabricate_state_dict(config, seed=SEED)
    quant = kind.startswith('quant')
    engines = {}
    for on in (False, True):
        with pytest.MonkeyPatch.context() as mp:
            mp.setenv('SOME_B200_BIAS_CORRECTION', '1' if on else '0')
            engines[on] = Engine(config, sd, 'cuda')
        assert bool(engines[on]._corrected) == on
    ref = engines[False].infer_accurate(drift_clips, quantized=quant)          # fp32 trunk: no rounded weights
    ref_probs = np.concatenate([r['probs'] for r in ref]).astype(np.float64)
    agg = {}
    for fold in (False, True):
        for on in (False, True):
            eng = engines[on]
            eng.set_ln_fold(fold)
            got = eng.infer(drift_clips, quantized=quant, return_intermediates=True)
            db = np.array([float((g['bounds'].astype(np.float64) - r['bounds']).mean()) for g, r in zip(got, ref)])
            dp = np.abs((np.concatenate([g['probs'] for g in got]) - ref_probs).mean(0)).max()
            agg[fold, on] = (db, float(np.abs(db).mean()), float(dp))
            print(f'\n{kind} fold={int(fold)} correction={"on " if on else "off"}: mean(bounds err) per clip '
                  + ' '.join(f'{v:+.1e}' for v in db)
                  + f' | mean |.| {agg[fold, on][1]:.2e} | max per-channel mean(probs err) {dp:.2e}', end='')
    for fold in (False, True):
        assert np.abs(agg[fold, True][0]).max() < BOUNDS_MEAN_TOL, (kind, fold, agg[fold, True][0])
    on, off = (sum(agg[fold, c][1] for fold in (False, True)) for c in (True, False))
    assert on * DRIFT_FACTOR < off, (kind, on, off)

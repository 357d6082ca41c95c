"""CPU-only tests of the host logic: the C-ABI library loads and exports every symbol the header declares,
config flattening / strict checkpoint schema, weight packing (GLU interleave, BN folding, mel tables),
clip sharding + the gloo all-gather of note records (world_size 2), and the drop-in package alias."""
import json
import os
import pathlib
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import yaml

from some_b200 import config as sconfig
from some_b200 import dist as sdist
from some_b200 import synth, weights

REPO = pathlib.Path(__file__).resolve().parent.parent


# --------------------------------------------------------------------------- C ABI
def test_library_exports_every_declared_symbol():
    from some_b200 import _lib
    lib = _lib.load()                        # raises if libsome_b200.so has not been built
    header = (REPO / 'include' / 'some_b200.h').read_text()
    header = re.sub(r'/\*.*?\*/', '', header, flags=re.S)
    declared = set(re.findall(r'\b(some_[a-z0-9_]+)\s*\(', header))
    assert declared == set(_lib.EXPORTS), (declared ^ set(_lib.EXPORTS))
    for name in declared:
        assert hasattr(lib, name), f'{name} declared in include/some_b200.h but not exported'
    assert lib.some_version() == 202
    assert lib.some_last_error() is not None


def test_abi_struct_sizes_match_header_layout():
    """ctypes mirrors of the header structs: pointer arrays first, then ints (catches field drift)."""
    from some_b200 import _lib
    import ctypes as C
    assert C.sizeof(_lib.GemmArgs) == 10 * 8 + 7 * 4 + 4 + 4 * 8 + 4 + 4 + 2 * 8   # + ln_s, ln_stats, ln_parts (+pad), out_bf16
    assert C.sizeof(_lib.LnArgs) == 10 * 8 + 2 * 4
    assert C.sizeof(_lib.AttnArgs) == 4 * 8 + 3 * 4 + 4 + 8 + 4 + 4  # incl. alignment / tail padding
    assert C.sizeof(_lib.DwconvArgs) == 8 * 8 + 2 * 4 + 8 + 4 + 4
    assert C.sizeof(_lib.DecodeArgs) == 3 * 8 + 4 * 4 + 4 * 4 + 8 * 8


def test_abi_struct_layouts_match_the_c_compiler(tmp_path):
    """sizeof / offsetof from gcc on include/some_b200.h vs the ctypes mirrors (the header is plain C)."""
    import ctypes as C
    import shutil
    from some_b200 import _lib
    if shutil.which('gcc') is None:
        pytest.skip('gcc not available')
    pairs = [('some_gemm_args', _lib.GemmArgs, 'out_bf16'), ('some_ln_args', _lib.LnArgs, 'M'),
             ('some_rowstats_args', _lib.RowStatsArgs, 'M'), ('some_profile_record', _lib.ProfileRecord, 'work'),
             ('some_attn_args', _lib.AttnArgs, 'max_frames'), ('some_dwconv_args', _lib.DwconvArgs, 'max_frames'),
             ('some_decode_args', _lib.DecodeArgs, 'scratch'), ('some_block_weights', _lib.BlockWeightsC, 'b_pw1f'),
             ('some_model', _lib.ModelC, 'ln_fold'), ('some_workspace', _lib.WorkspaceC, 'ln_stats'),
             ('some_block_weights_f32', _lib.BlockWeightsF32C, 'b_pw2'), ('some_model_f32', _lib.ModelF32C, 'b_cut'),
             ('some_workspace_f32', _lib.WorkspaceF32C, 'bounds'), ('some_calibration', _lib.CalibrationC, 'k')]
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "some_b200.h"\nint main(void){\n'
    for name, _, last in pairs:
        src += f'  printf("%zu %zu\\n", sizeof({name}), offsetof({name}, {last}));\n'
    src += '  return 0;\n}\n'
    (tmp_path / 't.c').write_text(src)
    subprocess.check_call(['gcc', '-I', os.path.join(REPO, 'include'), str(tmp_path / 't.c'), '-o', str(tmp_path / 't')])
    out = subprocess.check_output([str(tmp_path / 't')], text=True).split()
    for i, (name, cls, last) in enumerate(pairs):
        assert (int(out[2 * i]), int(out[2 * i + 1])) == (C.sizeof(cls), getattr(cls, last).offset), name


def test_workspace_sizing_and_carving():
    """some_workspace_bytes / some_workspace_carve: host-only arithmetic (no GPU needed): sizes add up, buffers are aligned and
    disjoint, ln_fold adds exactly its two buffers per stream."""
    import ctypes as C
    from some_b200 import _lib
    lib = _lib.load()
    m, outdim = 1000, 129
    n0, n1 = lib.some_workspace_bytes(m, outdim, 0), lib.some_workspace_bytes(m, outdim, 1)
    al = lambda b: (b + 255) & ~255
    want = 2 * al(m * 512 * 4) + 2 * al(m * 512 * 2) + 2 * al(m * 2048 * 2) + 2 * al(m * 1536 * 2) + 2 * al(m * 512 * 2) \
        + al(m * 80 * 2) + al(m * outdim * 4) + al(m * 4)
    assert n0 == want and n1 == want + 2 * al(m * 512 * 2) + 2 * al(m * 8 * 2 * 4)
    ws = _lib.WorkspaceC()
    base = 0x7f0000000000
    assert lib.some_workspace_carve(C.c_void_p(base), n1, m, outdim, 1, C.byref(ws)) == 0
    ptrs = sorted([ws.x[0], ws.x[1], ws.a[0], ws.a[1], ws.h[0], ws.h[1], ws.qkv[0], ws.qkv[1], ws.g[0], ws.g[1], ws.units, ws.probs,
                   ws.bounds, ws.xb[0], ws.xb[1], ws.ln_stats[0], ws.ln_stats[1]])
    assert ptrs[0] == base and all(p % 256 == 0 for p in ptrs) and len(set(ptrs)) == 17 and ptrs[-1] < base + n1
    assert lib.some_workspace_carve(C.c_void_p(base), n1 - 1, m, outdim, 1, C.byref(ws)) != 0
    assert b'too small' in lib.some_last_error()


def test_engine_refuses_cpu():
    from some_b200 import _lib, plugin
    cfg = synth.named_config('two_head')
    with pytest.raises(_lib.SomeB200Error):
        plugin.MIDIExtractionInference(config=cfg, model_path=pathlib.Path('/nonexistent.ckpt'), device='cpu')


# --------------------------------------------------------------------------- config / checkpoint schema
def test_flatten_config_chain(tmp_path):
    (tmp_path / 'configs').mkdir()
    (tmp_path / 'configs' / 'base.yaml').write_text(yaml.safe_dump({'a': 1, 'd': {'x': 1, 'y': 2}, 'keep': 7}))
    (tmp_path / 'configs' / 'mid.yaml').write_text(yaml.safe_dump({'base_config': 'configs/base.yaml', 'a': 2, 'd': {'y': 3}}))
    (tmp_path / 'configs' / 'top.yaml').write_text(yaml.safe_dump({'base_config': ['configs/mid.yaml'], 'd': {'z': 4}}))
    flat = sconfig.flatten_config(tmp_path / 'configs' / 'top.yaml', root=tmp_path)
    assert flat == {'a': 2, 'd': {'x': 1, 'y': 3, 'z': 4}, 'keep': 7}


@pytest.mark.parametrize('name,key', [('two_head_model', 'two_head'), ('midi_conformer', 'midi_conformer'),
                                      ('quant_two_head_model', 'quant_two_head')])
def test_named_configs_match_reference_yaml(name, key):
    # the reference's configs/<name>.yaml flattened through its base_config chain (tests/golden/make_golden_reference_meta.py)
    flat = json.loads((REPO / 'tests' / 'golden' / 'reference_configs.json').read_text())[name]
    mine = synth.named_config(key)
    for k, v in mine.items():
        if k in ('midi_prob_deviation', 'rest_threshold') and key == 'quant_two_head':
            assert k not in flat          # the stock chain lacks them (SURVEY.md discrepancy 6); injected by the harness
            continue
        assert flat[k] == v, (k, flat[k], v)


def test_state_dict_schema_and_strict_loading(tmp_path):
    cfg = synth.named_config('two_head', lay=1)
    ckpt = synth.write_checkpoint(tmp_path, cfg, seed=3)
    sd = sconfig.load_state_dict_strict(ckpt, cfg)
    assert list(sd) == list(sconfig.model_param_shapes(cfg))
    n_params = sum(int(np.prod(v.shape)) for k, v in sd.items() if 'num_batches' not in k and 'running' not in k)
    assert n_params == 4 * 6059008 + 2 * (1024 * 512 + 1024) + 2 * (512 * 80 + 512) + 128 * 512 + 128 + 512 + 1
    raw = torch.load(ckpt, weights_only=False)
    raw['state_dict'].pop('model.model.inln.bias')
    raw['state_dict']['model.model.bogus'] = torch.zeros(1)
    torch.save(raw, tmp_path / 'bad.ckpt')
    with pytest.raises(RuntimeError, match='Missing key.*inln.bias'):
        sconfig.load_state_dict_strict(tmp_path / 'bad.ckpt', cfg)
    with pytest.raises(NotImplementedError):
        sconfig.check_supported(dict(cfg, units_dim=768))


def test_check_supported_head_widths():
    """Widths the decode and scoring kernels refuse are refused when the model is loaded, naming the value: fewer than
    2 bins (the reference divides by N - 1 = 0), more than 256, and a quantized task with N != 129."""
    cont, quant = synth.named_config('two_head'), synth.named_config('quant_two_head')
    for n in (2, 64, 128, 129, 200, 256):
        sconfig.check_supported(dict(cont, midi_num_bins=n, midi_max=cont['midi_min'] + n - 1))
    sconfig.check_supported(quant)
    for n in (1, 0, -3, 257):
        with pytest.raises(NotImplementedError, match=rf'midi_num_bins={n} \(the decode takes 2 to 256 bins\)'):
            sconfig.check_supported(dict(cont, midi_num_bins=n))
        with pytest.raises(NotImplementedError, match=rf'midi_num_bins={n} '):
            sconfig.check_supported(dict(quant, midi_num_bins=n))
    for n in (2, 128, 130, 256):
        with pytest.raises(NotImplementedError, match=rf'midi_num_bins={n} for training.QuantizedMIDIExtractionTask'):
            sconfig.check_supported(dict(quant, midi_num_bins=n))


def test_schema_matches_reference_module():
    # parameter names / shapes of the reference's midi_conforms (tests/golden/make_golden_reference_meta.py)
    ref = json.loads((REPO / 'tests' / 'golden' / 'reference_state_dict_shapes.json').read_text())
    cfg = synth.named_config('two_head')
    mine = sconfig.model_param_shapes(cfg)
    assert set(ref) == set(mine)
    for k, v in ref.items():
        assert tuple(v) == tuple(mine[k]), k
    fab = synth.fabricate_state_dict(cfg)            # and the fabricated weights have exactly that schema
    assert set(fab) == set(ref)
    for k, v in fab.items():
        assert tuple(v.shape) == tuple(ref[k]), k


# --------------------------------------------------------------------------- weight packing
def test_glu_pack_rows_roundtrip():
    w = torch.arange(1024 * 3, dtype=torch.float32).reshape(1024, 3)
    p = weights.glu_pack_rows(w)
    for j in (0, 5, 31):
        assert torch.equal(p[32 * j:32 * j + 16], w[16 * j:16 * j + 16])
        assert torch.equal(p[32 * j + 16:32 * j + 32], w[512 + 16 * j:512 + 16 * j + 16])


def test_bn_folding_and_packing_match_torch():
    cfg = synth.named_config('two_head', lay=1)
    sd = synth.fabricate_state_dict(cfg, seed=11)
    p = 'model.att1'
    bw = weights.BlockWeights(sd, p, 'cpu', weights.RoundingRegistry('cpu'))
    x = torch.randn(1, 512, 50)
    ref = torch.nn.functional.batch_norm(
        torch.nn.functional.conv1d(x, sd[p + '.conv.depthwise_conv.weight'], sd[p + '.conv.depthwise_conv.bias'],
                                   padding=15, groups=512),
        sd[p + '.conv.norm.running_mean'], sd[p + '.conv.norm.running_var'], sd[p + '.conv.norm.weight'],
        sd[p + '.conv.norm.bias'], False, 0.1, 1e-5)
    got = torch.nn.functional.conv1d(x, bw.w_dw.t().unsqueeze(1), bw.b_dw, padding=15, groups=512)
    torch.testing.assert_close(got, ref, atol=1e-5, rtol=1e-5)
    assert bw.w_qkv.shape == (1536, 512) and bw.w_qkv.dtype == torch.bfloat16
    assert torch.equal(bw.w_qkv[:512].float(), sd[p + '.att.to_q.weight'].bfloat16().float())
    assert torch.equal(bw.w_qkv[512:].float(), sd[p + '.att.to_kv.weight'].bfloat16().float())


def test_mel_tables_match_golden_basis(golden_dir):
    cfg = synth.named_config('two_head')
    t = weights.mel_tables(cfg, 'cpu')
    ref = np.load(golden_dir / 'mel.npz')['mel_basis']          # buffer of the reference's MelSpectrogram
    assert np.array_equal(t['bank'], ref)
    dense = np.zeros_like(ref)
    for m in range(80):
        s, c = int(t['mel_start'][m]), int(t['mel_count'][m])
        dense[m, s:s + c] = t['mel_weights'][m, :c].numpy()
    assert np.array_equal(dense, ref)
    assert torch.equal(t['window'], torch.hann_window(2048))
    tw = t['twiddle'].double()
    assert tw.shape == (1396, 2)
    assert abs(float(tw[16 * 32 + 16, 0])) < 1e-7 and abs(float(tw[16 * 32 + 16, 1]) + 1.0) < 1e-7   # W_1024^(16 * 16) = -i
    assert abs(float(tw[3 * 32 + 5, 0]) - np.cos(-2 * np.pi * 15 / 1024)) < 1e-7       # [k1 = 3][n2 = 5]
    assert abs(float(tw[1024 + 256, 0]) - np.cos(-2 * np.pi * 256 / 2048)) < 1e-7      # unpack table W_2048^k


# --------------------------------------------------------------------------- sharding + gather
def test_shard_clips_balanced_and_complete():
    rng = np.random.default_rng(0)
    lengths = [int(x) for x in rng.integers(44100 * 5, 44100 * 15, size=37)] + [44100 * 300]
    for world in (1, 2, 4, 8):
        shards = sdist.shard_clips(lengths, world)
        assert sorted(i for s in shards for i in s) == list(range(len(lengths)))
        loads = [sum(sdist.clip_cost(lengths[i]) for i in s) for s in shards]
        biggest = max(sdist.clip_cost(n) for n in lengths)
        assert max(loads) - min(loads) <= biggest + 1e-6        # LPT bound


def _fake_notes(n_samples):
    t = 1 + n_samples // 512
    rng = np.random.default_rng(n_samples)
    n = int(rng.integers(1, t + 1))
    dur = rng.multinomial(t, np.ones(n) / n).astype(np.int64)
    return {'note_midi': rng.uniform(30, 90, n).astype(np.float32), 'note_dur': dur * (512 / 44100),
            'note_rest': rng.random(n) < 0.2}


def test_pack_unpack_roundtrip():
    lengths = [5000, 300, 44100, 0]
    res = [_fake_notes(n) for n in lengths]
    frames = [1 + n // 512 for n in lengths]
    slab = sdist.pack_results(res, frames, sdist.slab_bytes(lengths, [list(range(4))]), 512 / 44100)
    back = sdist.unpack_results(slab, frames, 512 / 44100)
    for a, b in zip(res, back):
        for k in a:
            np.testing.assert_array_equal(a[k], b[k])


def _gloo_worker(rank, world, port, lengths, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)

    class FakePlugin:
        timestep = 512 / 44100

        def infer(self, waves):
            return [_fake_notes(len(w)) for w in waves]

    waves = [np.zeros(n, dtype=np.float32) for n in lengths]
    merged = sdist.infer_sharded(FakePlugin(), waves)
    ok = all(np.array_equal(m[k], _fake_notes(n)[k]) for m, n in zip(merged, lengths) for k in m)

    # C5 across ranks: one recording, the cuts come from the slicer (here: fixed ranges), the chunks are sharded
    class FakeSlicer:
        sr = 44100

        def ranges(self, w):
            cuts = np.cumsum([0] + lengths)
            return [(int(a), int(b)) for a, b in zip(cuts[:-1], cuts[1:]) if b > a]

    rec = np.zeros(int(sum(lengths)), dtype=np.float32)
    offsets, notes = sdist.infer_sliced_sharded(FakePlugin(), rec, FakeSlicer())
    kept = [n for n in lengths if n > 0]
    ok = ok and len(offsets) == len(notes) == len(kept) and offsets[0] == 0.0
    ok = ok and all(np.array_equal(m[k], _fake_notes(n)[k]) for m, n in zip(notes, kept) for k in m)
    q.put((rank, ok, len(merged)))
    dist.destroy_process_group()


def test_infer_sharded_gloo_world2():
    import torch.multiprocessing as mp
    lengths = [44100, 512 * 7 + 3, 90000, 1000, 250000, 0, 333]
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + os.getpid() % 1000
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, lengths, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(r[0] for r in results) == [0, 1]
    assert all(ok and n == len(lengths) for _, ok, n in results)


# --------------------------------------------------------------------------- drop-in alias
def test_inference_package_is_the_drop_in():
    code = ("import inference, some_b200.plugin as p; "
            "assert inference.MIDIExtractionInference is p.MIDIExtractionInference; "
            "assert issubclass(inference.QuantizedMIDIExtractionInference, inference.BaseInference); "
            "assert inference.task_inference_mapping['training.MIDIExtractionTask'] == 'inference.MIDIExtractionInference'; "
            "print('ok')")
    env = dict(os.environ, PYTHONPATH=str(REPO))
    out = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, env=env, cwd='/tmp')
    assert out.returncode == 0 and 'ok' in out.stdout, out.stderr


# --------------------------------------------------------------------------- engine host helpers (no GPU: pure numpy)
def _bare_engine():
    from some_b200.engine import Engine
    eng = Engine.__new__(Engine)           # host helpers only: no library, no device
    eng.timestep = 512 / 44100
    return eng


def test_engine_tables_and_chunk_layout():
    eng = _bare_engine()
    rng = np.random.default_rng(3)
    lens = rng.integers(0, 400000, size=37)
    lens[5] = 0
    starts, lens64, cu, total = eng.tables(lens)
    assert np.all(starts % 4 == 0) and total % 4 == 0                         # 16-byte aligned clip starts (float4 loads)
    assert np.all(np.diff(starts) >= lens64[:-1]) and total >= starts[-1] + lens64[-1]
    np.testing.assert_array_equal(np.diff(cu), 1 + lens64 // 512)            # T = 1 + L // hop (spec.py:48-60)
    chunks = eng._chunks(cu)
    assert chunks[0][0] == 0 and chunks[-1][1] == len(lens) and len(chunks) <= 3
    assert all(a[1] == b[0] for a, b in zip(chunks[:-1], chunks[1:])) and all(c1 > c0 for c0, c1 in chunks)
    frames = [int(cu[c1] - cu[c0]) for c0, c1 in chunks]
    assert frames[0] == min(frames)                                            # small first chunk gets the GPU going
    assert eng._chunks(np.asarray([0, 100, 250], dtype=np.int32)) == [(0, 2)]  # small batches are not split
    cu2, layout, nbytes = eng.slab_layout(lens)
    np.testing.assert_array_equal(cu2, cu)
    off = 0
    for (c0, c1, o, bc, mc), (d0, d1) in zip(layout, chunks):
        assert (c0, c1, o, bc, mc) == (d0, d1, off, d1 - d0, int(cu[d1] - cu[d0])) and o % 16 == 0
        off += (4 * bc + 9 * mc + 15) & ~15
    assert nbytes == off


def test_engine_unpack_slab_reads_the_decode_slab_format():
    """unpack_slab must read exactly the [counts | dur | midi | rest] slab that decode.cu writes and dist.pack_results mirrors."""
    eng = _bare_engine()
    lens = [70000, 0, 512 * 40 + 7, 90000, 300]
    cu, layout, nbytes = eng.slab_layout(lens)
    notes = [_fake_notes(n) for n in lens]
    host = np.zeros(nbytes, dtype=np.uint8)
    for c0, c1, off, bc, mc in layout:
        frames = [int(cu[i + 1] - cu[i]) for i in range(c0, c1)]
        slab = sdist.pack_results(notes[c0:c1], frames, 4 * bc + 9 * mc, 512 / 44100)
        host[off:off + slab.size] = slab
    back = eng.unpack_slab(host, cu, layout)
    assert len(back) == len(lens)
    for a, b in zip(notes, back):
        assert b['note_midi'].dtype == np.float32 and b['note_dur'].dtype == np.float64 and b['note_rest'].dtype == bool
        for k in a:
            np.testing.assert_array_equal(a[k], b[k])
    # the results own their data (the pinned landing buffer the slab lives in is reused by the next call)
    snapshot = [{k: v.copy() for k, v in r.items()} for r in back]
    host[:] = 0xFF
    for a, b in zip(snapshot, back):
        for k in a:
            np.testing.assert_array_equal(a[k], b[k])
    assert eng.slab_layout_cached(lens) is eng.slab_layout_cached(list(lens))           # memoised on the lengths
    cu3, layout3, nbytes3 = eng.slab_layout_cached(lens)
    np.testing.assert_array_equal(cu3, cu)
    assert layout3 == layout and nbytes3 == nbytes


def test_sharded_results_are_lazy_per_rank_and_survive_buffer_reuse():
    """dist.ShardedResults (what infer_sharded returns on the NCCL path): a rank's slab is unpacked when one of ITS clips is first
    touched; the slabs live in a landing buffer the next call overwrites, so infer_sharded materialises whatever is still lazy
    before it reuses the buffer (here: emulated with the same calls)."""
    eng = _bare_engine()
    lens = [[70000, 512 * 40 + 7], [90000, 300, 0]]                 # two ranks' shards
    shards = [[0, 3], [1, 2, 4]]                                     # global clip index of each shard entry
    layouts = [eng.slab_layout_cached(l) for l in lens]
    nbytes = max(l[2] for l in layouts)
    landing = np.zeros(2 * nbytes, dtype=np.uint8)
    notes = {}
    for r, (cu, layout, _) in enumerate(layouts):
        fake = [_fake_notes(n + 17 * r) for n in lens[r]]
        for i, f in zip(shards[r], fake):
            notes[i] = f
        for c0, c1, off, bc, mc in layout:
            frames = [int(cu[i + 1] - cu[i]) for i in range(c0, c1)]
            slab = sdist.pack_results(fake[c0:c1], frames, 4 * bc + 9 * mc, 512 / 44100)
            landing[r * nbytes + off:r * nbytes + off + slab.size] = slab
    calls = []

    def unpacker(r):
        cu_r, layout_r, _ = layouts[r]

        def run():
            calls.append(r)
            return list(zip(shards[r], eng.unpack_slab(landing[r * nbytes:(r + 1) * nbytes], cu_r, layout_r)))
        return run

    owner = [0, 1, 1, 0, 1]
    res = sdist.ShardedResults(5, owner, [unpacker(0), unpacker(1)])
    res._materialise_rank(0)                                         # a rank's own shard is unpacked eagerly
    assert calls == [0] and len(res) == 5
    np.testing.assert_array_equal(res[3]['note_midi'], notes[3]['note_midi'])
    assert calls == [0]                                              # touching an own clip unpacks nothing new
    res.materialise()                                                # what infer_sharded does before reusing the buffer
    assert calls == [0, 1]
    landing[:] = 0xFF                                                # the next call's gather lands
    for i in range(5):
        for k in ('note_midi', 'note_dur', 'note_rest'):
            np.testing.assert_array_equal(res[i][k], notes[i][k])
    assert calls == [0, 1] and [r['note_midi'].shape for r in res[1:3]] == [notes[1]['note_midi'].shape, notes[2]['note_midi'].shape]


# ----------------------------------------------------------------------------- csrc/pack.cu: the C restatement of weights.py
def _p(a):
    import ctypes as C
    return a.ctypes.data_as(C.c_void_p)


def test_c_pack_functions_match_the_python_packing():
    """Host-only C packing entry points (for non-Python hosts) against what some_b200/weights.py does with torch."""
    from some_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(5)
    # bf16 rounding: RNE, ties, denormals, infinities, NaN
    x = np.concatenate([rng.standard_normal(4096).astype(np.float32) * 3,
                        np.array([0.0, -0.0, 1.0, 1.00390625, 1.01171875, 3.3895314e38, np.inf, -np.inf, 1e-40, np.nan], np.float32)])
    out = np.zeros(x.size, np.uint16)
    assert lib.some_pack_bf16(_p(x), x.size, _p(out)) == 0
    ref = torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    ok = ~np.isnan(x)
    np.testing.assert_array_equal(out[ok], ref[ok])
    assert np.isnan(torch.from_numpy(out[~ok].view(np.int16)).view(torch.bfloat16).float().numpy()).all()
    # GLU row interleave, fp32 weights and bf16-sized elements
    w = rng.standard_normal((1024, 24)).astype(np.float32)
    got = np.zeros_like(w)
    assert lib.some_pack_glu_rows(_p(w), 4, 1024, 24, _p(got)) == 0
    np.testing.assert_array_equal(got, weights.glu_pack_rows(torch.from_numpy(w)).numpy())
    b16 = rng.integers(0, 65535, size=(64, 1), dtype=np.uint16)
    got16 = np.zeros_like(b16)
    assert lib.some_pack_glu_rows(_p(b16), 2, 64, 1, _p(got16)) == 0
    np.testing.assert_array_equal(got16, weights.glu_pack_rows(torch.from_numpy(b16.astype(np.int32))).numpy().astype(np.uint16))
    assert lib.some_pack_glu_rows(_p(w), 4, 1000, 24, _p(got)) != 0 and b'multiple of 32' in lib.some_last_error()
    # depthwise conv + BatchNorm(eval) folding (BlockWeights: float64 inside, taps transposed to [K][C])
    c, k = 512, 31
    dw, db = rng.standard_normal((c, k)).astype(np.float32), rng.standard_normal(c).astype(np.float32)
    g, be = rng.standard_normal(c).astype(np.float32), rng.standard_normal(c).astype(np.float32)
    mu, var = rng.standard_normal(c).astype(np.float32), (rng.random(c).astype(np.float32) + 0.1)
    taps, bias = np.zeros((k, c), np.float32), np.zeros(c, np.float32)
    assert lib.some_pack_dwconv_bn(_p(dw), _p(db), _p(g), _p(be), _p(mu), _p(var), c, k, _p(taps), _p(bias)) == 0
    t = lambda a: torch.from_numpy(a)
    scale = t(g).double() / torch.sqrt(t(var).double() + weights.BN_EPS)
    np.testing.assert_array_equal(taps, (t(dw).double() * scale[:, None]).t().float().numpy())
    np.testing.assert_array_equal(bias, ((t(db).double() - t(mu).double()) * scale + t(be).double()).float().numpy())
    # LayerNorm folding (BlockWeights.fold): rounded weights identical, column sums of the ROUNDED weights, bias = W beta + b
    n, kk = 1024, 512
    W, b = (rng.standard_normal((n, kk)) / 22).astype(np.float32), rng.standard_normal(n).astype(np.float32)
    gam, bet = (1 + 0.1 * rng.standard_normal(kk)).astype(np.float32), (0.1 * rng.standard_normal(kk)).astype(np.float32)
    for glu in (0, 1):
        pack = weights.glu_pack_rows if glu else (lambda z: z)
        w_out, s_out, b_out = np.zeros((n, kk), np.uint16), np.zeros(n, np.float32), np.zeros(n, np.float32)
        assert lib.some_pack_ln_fold(_p(W), _p(b), _p(gam), _p(bet), n, kk, glu, _p(w_out), _p(s_out), _p(b_out)) == 0
        w64 = t(W).double()
        wf = pack((w64 * t(gam).double()[None, :]).float()).to(torch.bfloat16)
        np.testing.assert_array_equal(w_out, wf.view(torch.int16).numpy().view(np.uint16))
        np.testing.assert_array_equal(s_out, wf.double().sum(dim=1).float().numpy())
        np.testing.assert_allclose(b_out, pack((w64 @ t(bet).double() + t(b).double()).float()).numpy(), rtol=0, atol=1e-6)


def test_c_mel_tables_match_the_python_tables():
    """some_mel_tables (librosa.filters.mel restated in C, float64) against weights.mel_tables (numpy / torch restatement that is
    itself pinned to the reference's basis by tests/golden): identical sparsity, values to the last float32 ulp or two."""
    from some_b200 import _lib
    lib = _lib.load()
    cfg = synth.named_config('two_head')
    ref = weights.mel_tables(cfg, 'cpu')
    start, count = np.zeros(80, np.int32), np.zeros(80, np.int32)
    w = np.full((80, _lib.MEL_MAXW), np.nan, np.float32)
    tw, win = np.zeros((_lib.MEL_TW, 2), np.float32), np.zeros(2048, np.float32)
    rc = lib.some_mel_tables(cfg['audio_sample_rate'], cfg['win_size'], cfg['units_dim'], float(cfg['fmin']), float(cfg['fmax']),
                             _p(start), _p(count), _p(w), _p(tw), _p(win))
    assert rc == 0, lib.some_last_error()
    np.testing.assert_array_equal(start, ref['mel_start'].numpy())
    np.testing.assert_array_equal(count, ref['mel_count'].numpy())
    np.testing.assert_allclose(w, ref['mel_weights'].numpy(), rtol=3e-7, atol=1e-12)
    np.testing.assert_allclose(tw, ref['twiddle'].numpy(), rtol=0, atol=6e-8)
    np.testing.assert_allclose(win, ref['window'].numpy(), rtol=0, atol=2e-7)
    assert lib.some_mel_tables(44100, 1024, 80, 40.0, 8000.0, _p(start), _p(count), _p(w), _p(tw), _p(win)) != 0
    assert lib.some_mel_tables(44100, 2048, 80, 40.0, 20000.0, _p(start), _p(count), _p(w), _p(tw), _p(win)) != 0   # filters beyond bin 371

"""Batched SOME inference engine: packs clips var-len, launches the sm_90a kernels of
libsome_b200.so in order on the current CUDA stream and unpacks the decoded notes.

Equivalent to running the reference's batch-1 loop (inference/base_infer.py:46-53) once per clip:
clips never interact (per-clip attention, per-clip zero-padded depthwise conv, per-clip decode).
The trunk is sequenced natively (csrc/forward.cu: some_forward); per conform_blocke (Gconform.py:56-63), both streams
(midi / bound) in every launch:
    LN1 -> GEMM(ffn1.ln1)+SiLU -> GEMM(ffn1.ln2)*0.5+x -> LN2 -> GEMM(to_q|to_kv) -> attention ->
    GEMM(to_out)+x -> LN3 -> GEMM(pointwise_conv1)+GLU -> dwconv+BN+SiLU -> GEMM(pointwise_conv2)+x ->
    LN4 -> GEMM(ffn2.ln1)+SiLU -> GEMM(ffn2.ln2)*0.5+x -> LN5
SOME_B200_LN_FOLD=1 selects the variant with norm1..norm4 folded into the GEMMs around them (11 instead of 15 launches per
block), kept as a validated option; stand-alone LayerNorm launches are the default.
The residual stream x is fp32 [M, 512]; GEMM operands are bf16; accumulation is fp32.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .config import DIM, FFN_DIM, check_supported
from .weights import ModelWeights, build_c_model, mel_tables

HOP = 512


def frames_of(num_samples: int) -> int:
    return 1 + num_samples // HOP


def pinned_array(num_samples: int) -> np.ndarray:
    """float32 numpy array in page-locked host memory.  A loader that decodes audio into such buffers lets Engine.infer
    copy host -> device straight from them (no staging memcpy); ordinary numpy arrays work too, through a staging copy."""
    return torch.empty(int(num_samples), dtype=torch.float32).pin_memory().numpy()


class _Workspace:
    _count = 0

    def __init__(self, m: int, outdim: int, device):
        bf, f32 = torch.bfloat16, torch.float32
        _Workspace._count += 1
        self.serial = _Workspace._count       # never reused (CUDA-graph cache keys)
        self.m = m
        self.x = torch.empty((2, m, DIM), dtype=f32, device=device)          # residual streams
        self.a = torch.empty((2, m, DIM), dtype=bf, device=device)           # LN out / attention out / dwconv out
        self.h = torch.empty((2, m, FFN_DIM), dtype=bf, device=device)       # FFN hidden
        self.qkv = torch.empty((2, m, 3 * DIM), dtype=bf, device=device)
        self.g = torch.empty((2, m, DIM), dtype=bf, device=device)           # GLU out (dwconv in)
        self.xb = torch.empty((2, m, DIM), dtype=bf, device=device)          # bf16 copy of x (LayerNorm-folded consumers)
        self.ln_stats = torch.empty((2, m, _lib.LN_SLOTS, 2), dtype=f32, device=device)   # per-row partial (sum, sum sq)
        self.units = torch.empty((m, 80), dtype=bf, device=device)
        self.probs = torch.empty((m, outdim), dtype=f32, device=device)
        self.bounds = torch.empty((m,), dtype=f32, device=device)
        self.note_midi = torch.empty((m,), dtype=f32, device=device)
        self.note_dur = torch.empty((m,), dtype=torch.int32, device=device)
        self.note_rest = torch.empty((m,), dtype=torch.uint8, device=device)
        self.scratch = torch.empty((int(_lib.load().some_decode_scratch_bytes(m)),), dtype=torch.uint8, device=device)
        c = self.c = _lib.WorkspaceC()                    # some_workspace for the native sequencer
        for s in range(2):
            c.x[s], c.a[s], c.h[s] = self.x[s].data_ptr(), self.a[s].data_ptr(), self.h[s].data_ptr()
            c.qkv[s], c.g[s] = self.qkv[s].data_ptr(), self.g[s].data_ptr()
            c.xb[s], c.ln_stats[s] = self.xb[s].data_ptr(), self.ln_stats[s].data_ptr()
        c.units, c.probs, c.bounds = self.units.data_ptr(), self.probs.data_ptr(), self.bounds.data_ptr()


class Engine:
    def __init__(self, config: dict, state_dict, device='cuda'):
        self.lib = _lib.load()
        check_supported(config)
        self.config = config
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise _lib.SomeB200Error('some_b200 runs on CUDA devices only (sm_90a); there is no CPU path')
        self.quantized = False
        self._state_dict = state_dict        # fp32 masters for the validation path (infer_accurate), built lazily
        self._f32 = None
        self.w = ModelWeights(state_dict, config, self.device)
        self.ln_fold = os.environ.get('SOME_B200_LN_FOLD', '0') != '0'
        self._cmodel, self._cmodel_keep = build_c_model(self.w, self.ln_fold)
        self.mel = mel_tables(config, self.device)
        self.outdim = config['midi_num_bins']
        self.timestep = config['hop_size'] / config['audio_sample_rate']
        self._ws: Optional[_Workspace] = None
        self.launches = 0
        self._sum_t2 = 0.0
        # launches of one trunk pass: inln (+ row_stats) + (lay + 1) blocks x 11 (15 unfolded) + lay GLU mixes
        # + (final LN + bound head instead of LN5) + head
        self._count_trunk_launches()
        # optional per-kernel timing (bench.py): CUDA events around every launch — the native sequencer records its own
        # (some_profiler), the kernels launched from here (mel, decode) are bracketed by _mark()
        self.prof: Optional[dict] = None
        self._cprof = None
        self._graphs: dict = {}
        self._graph_seen: dict = {}
        self.use_graphs = os.environ.get('SOME_B200_GRAPHS', '1') != '0'
        # programmatic dependent launch of the trunk kernels: 'small' = chunks that also replay as a CUDA graph, 'all', 'off'
        self.pdl = {'0': 'off', 'off': 'off', '1': 'all', 'all': 'all'}.get(os.environ.get('SOME_B200_PDL', 'small'), 'small')
        self._corrected: set = set()
        self.bias_correction = os.environ.get('SOME_B200_BIAS_CORRECTION', '1') != '0'
        if self.bias_correction:
            self.calibrate()

    def _count_trunk_launches(self):
        per_block = 11 if self.ln_fold else 15
        self.trunk_launches = 1 + int(self.ln_fold) + per_block * (self.w.lay + 1) + self.w.lay + 1 + 1

    def set_ln_fold(self, flag: bool):
        """Switches between the LayerNorm-folded launch sequence and the stand-alone LayerNorm launches (tests, A/B)."""
        self.ln_fold = bool(flag)
        self._cmodel, self._cmodel_keep = build_c_model(self.w, self.ln_fold)
        self._count_trunk_launches()

    def calibrate(self, seconds: float = 4.0):
        """Load-time bias correction for the bf16 rounding of the weights.  Rounding W to bf16 is a FIXED perturbation of the
        model: its mean effect on a layer's output, (W - bf16(W)) . E[a], is a constant per output channel that survives to
        the boundary probabilities as a systematic offset (measured +3.5e-4 on `bounds` with the seeded weights) and is then
        integrated by the decoder's cumsum (utils/infer_utils.py:28) into a drift of about one note per 30 s clip.  The
        standard post-training-quantisation remedy is applied here: one short calibration clip (a seeded synthetic sung-note
        signal; with stand-alone LayerNorms the operand means are dominated by the LayerNorm biases and the positive mean of
        SiLU outputs, i.e. by the weights, and white noise calibrates equally well; with folded LayerNorms the operand is the
        normalised row itself and a voice-like signal matters: residual -7e-5 vs -1.5e-4) runs through the sequencer, which
        records the column means of every GEMM's effective operand (some_forward, `calib`), and each layer's bias absorbs
        (W_master - bf16(W)) . mean.  After it the mean error of `bounds` is within +-1e-4 (clip dependent, +-3e-5 on most
        clips) and zero-mean rounding noise remains.  (A second, head-level calibration against the library's own fp32 path
        was tried and removed: what is left after this step depends on the input, not on the weights.)"""
        reg = getattr(self.w, 'rounding', None)
        if reg is None:
            return
        dev = self.device
        with torch.cuda.device(dev):
            from .synth import synth_waveform
            wave = synth_waveform(20240917, seconds=seconds, sr=self.config['audio_sample_rate'])
            host, tables, cu = self.pack([wave])
            m = int(cu[-1])
            ws = self.workspace(m)
            wave_d, tab_d, cu_d = host.to(dev), tables.to(dev), torch.from_numpy(cu).to(dev)
            self.run_mel(wave_d, tab_d[:1], tab_d[1:], cu_d, 1, m, None, ws.units)
            means = torch.zeros((_lib.CALIB_MAX, 2, _lib.CALIB_K), dtype=torch.float32, device=dev)
            cal = _lib.CalibrationC()
            cal.means = means.data_ptr()
            # both launch sequences (LayerNorm-folded and not) so that every layer's bias is corrected exactly once,
            # whichever mode is selected later (set_ln_fold)
            for fold in (self.ln_fold, not self.ln_fold):
                cmodel, keep = build_c_model(self.w, fold)
                _lib.check(self.lib.some_forward(C.byref(cmodel), C.byref(ws.c), m, 1, cu_d.data_ptr(), m, _lib.EPI_BIAS_F32,
                                                 None, C.byref(cal), self._stream), 'some_forward(calibration)')
                torch.cuda.synchronize(dev)
                for i in range(cal.count):
                    k = cal.k[i]
                    for s in range(2):
                        ptr = cal.w[i][s]
                        ent = reg.entries.get(ptr)
                        if ent is None or ptr in self._corrected:
                            continue
                        self._corrected.add(ptr)
                        master, rounded, bias = ent
                        if bias is None:
                            continue
                        delta = (master.double() - rounded.double()) @ means[i, s, :k].double()
                        bias[:delta.numel()] += delta.float()
                del cmodel, keep
        self.w.rounding = None                 # drop the fp32 masters

    def start_profile(self, cu_frames_host=None):
        self.prof = {}
        if cu_frames_host is not None:
            t = np.diff(np.asarray(cu_frames_host)).astype(np.float64)
            self._sum_t2 = float((t * t).sum())
        if self._cprof is None:
            h = C.c_void_p()
            _lib.check(self.lib.some_profiler_create(1 << 14, C.byref(h)), 'some_profiler_create')
            self._cprof = h
        _lib.check(self.lib.some_profiler_reset(self._cprof), 'some_profiler_reset')

    def stop_profile(self) -> Dict[str, dict]:
        """Returns {kernel: {launches, ms, work, shapes}} from the CUDA events recorded since start_profile(): the native
        sequencer's records (some_profiler_read) plus the launches bracketed from Python (mel, decode)."""
        torch.cuda.synchronize(self.device)
        out = {}
        for name, recs in (self.prof or {}).items():
            out[name] = {'launches': len(recs), 'ms': float(sum(a.elapsed_time(b) for a, b, _ in recs)),
                         'work': float(sum(w for _, _, w in recs))}
        self.prof = None
        cap = 1 << 14
        recs = (_lib.ProfileRecord * cap)()
        n = self.lib.some_profiler_read(self._cprof, cap, recs)
        if n < 0:
            _lib.check(n, 'some_profiler_read')
        att_flops = float(2 * 2 * 2 * 512 * self._sum_t2)      # QK^T + PV, 8 heads x 64, both streams, 2 FLOP / MAC
        for r in recs[:min(n, cap)]:
            name = _lib.KERNEL_NAMES.get(r.kernel, f'kernel{r.kernel}')
            d = out.setdefault(name, {'launches': 0, 'ms': 0.0, 'work': 0.0})
            d['launches'] += 1
            d['ms'] += float(r.ms)
            d['work'] += att_flops if r.kernel == _lib.K_ATTENTION else float(r.work)
            if r.kernel == _lib.K_GEMM:
                sh = d.setdefault('shapes', {}).setdefault(f'epi{r.epilogue}_N{r.n}_K{r.k}', {'launches': 0, 'ms': 0.0, 'work': 0.0})
                sh['launches'] += 1
                sh['ms'] += float(r.ms)
                sh['work'] += float(r.work)
        return out

    def _mark(self, name: str, work: float):
        """Context manager: CUDA events on the launching stream around one kernel launch."""
        eng = self

        class _M:
            def __enter__(self_m):
                if eng.prof is not None:
                    self_m.a = torch.cuda.Event(enable_timing=True)
                    self_m.b = torch.cuda.Event(enable_timing=True)
                    self_m.a.record(torch.cuda.current_stream(eng.device))
                return self_m

            def __exit__(self_m, *exc):
                if eng.prof is not None:
                    self_m.b.record(torch.cuda.current_stream(eng.device))
                    eng.prof.setdefault(name, []).append((self_m.a, self_m.b, work))
                eng.launches += 1
                return False

        return _M()

    # ------------------------------------------------------------------ helpers
    @property
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def workspace(self, m: int) -> _Workspace:
        if self._ws is None or self._ws.m < m:
            self._ws = None
            self._ws = _Workspace(max(m, 1), self.outdim, self.device)
        return self._ws

    # ------------------------------------------------------------------ stages
    def run_mel(self, wave: torch.Tensor, clip_start: torch.Tensor, clip_len: torch.Tensor, cu_frames: torch.Tensor,
                b: int, max_frames: int, out_f32: Optional[torch.Tensor], out_bf16: Optional[torch.Tensor]):
        """K-mel (spec.py:38-72).  wave f32; clip i = wave[start_i : start_i + len_i]; outputs [M, 80]."""
        t = self.mel
        m = (out_f32 if out_f32 is not None else out_bf16).shape[0]
        with self._mark('some_mel_logmel', m * (512 * 4 + 80 * 4.0)):        # 2368 B / frame (SURVEY.md §8d)
            _lib.check(self.lib.some_mel_logmel(
                wave.data_ptr(), clip_start.data_ptr(), clip_len.data_ptr(), cu_frames.data_ptr(), b, max_frames,
                t['mel_start'].data_ptr(), t['mel_count'].data_ptr(), t['mel_weights'].data_ptr(),
                t['twiddle'].data_ptr(), t['window'].data_ptr(), _lib.ptr(out_f32), _lib.ptr(out_bf16),
                1e-5, self._stream), 'some_mel_logmel')

    def run_trunk(self, ws: _Workspace, m: int, b: int, cu_frames: torch.Tensor, max_frames: int,
                  head: str = 'sigmoid'):
        """Gmidi_conform.forward (Gconform.py:119-140) + the head activation of midi_conforms.forward
        (Gmidi_conform.py:30-40): ONE native call enqueues the whole launch sequence (csrc/forward.cu).
        Reads ws.units; writes ws.probs [m, outdim] and ws.bounds [m].  head: 'sigmoid' | 'softmax' | 'logits'."""
        epi = {'sigmoid': _lib.EPI_SIGMOID_F32, 'softmax': _lib.EPI_SOFTMAX_F32, 'logits': _lib.EPI_BIAS_F32}[head]
        prof = self._cprof if self.prof is not None else None
        _lib.check(self.lib.some_forward(C.byref(self._cmodel), C.byref(ws.c), m, b, cu_frames.data_ptr(), max_frames,
                                         epi, prof, None, self._stream), 'some_forward')
        self.launches += self.trunk_launches

    def run_decode(self, ws: _Workspace, m: int, b: int, cu_frames: torch.Tensor, note_count: torch.Tensor,
                   quantized: bool, dbg: Optional[dict] = None, probs=None, bounds=None, out=None):
        cfg = self.config
        d = _lib.DecodeArgs()
        d.probs = (probs if probs is not None else ws.probs).data_ptr()
        d.bounds = (bounds if bounds is not None else ws.bounds).data_ptr()
        d.cu_frames = cu_frames.data_ptr()
        d.B, d.M, d.N, d.quantized = b, m, self.outdim, int(quantized)
        d.vmin, d.vmax = float(cfg['midi_min']), float(cfg['midi_max'])
        d.deviation = float(cfg.get('midi_prob_deviation', 1.0))
        d.threshold = float(cfg.get('rest_threshold', 0.1))
        nm_t, nd_t, nr_t = out if out is not None else (ws.note_midi, ws.note_dur, ws.note_rest)
        d.note_midi, d.note_dur, d.note_rest = nm_t.data_ptr(), nd_t.data_ptr(), nr_t.data_ptr()
        d.note_count = note_count.data_ptr()
        if dbg is not None:
            dbg['frame2item'] = torch.zeros(m, dtype=torch.int32, device=self.device)
            dbg['values'] = torch.zeros(m, dtype=torch.float32, device=self.device)
            dbg['rest'] = torch.zeros(m, dtype=torch.uint8, device=self.device)
            d.dbg_frame2item, d.dbg_values, d.dbg_rest = (dbg[k].data_ptr() for k in ('frame2item', 'values', 'rest'))
        d.scratch = ws.scratch.data_ptr()
        with self._mark('some_decode_notes', m * (self.outdim * 4.0 + 4.0)):
            _lib.check(self.lib.some_decode_notes(C.byref(d), self._stream), 'some_decode_notes')
        self.launches += 2                     # frames + align + notes kernels behind the one call

    # ------------------------------------------------------------------ public batched entry point
    def tables(self, lens: np.ndarray):
        """Var-len tables for clips of ``lens`` samples: 16-byte aligned starts, cu_frames (T = 1 + L // hop,
        spec.py:48-60).  Host only."""
        lens = np.asarray(lens, dtype=np.int64)
        padded = (lens + 3) & ~3
        starts = np.zeros(len(lens), dtype=np.int64)
        np.cumsum(padded[:-1], out=starts[1:])
        cu = np.zeros(len(lens) + 1, dtype=np.int32)
        np.cumsum(1 + lens // HOP, out=cu[1:])
        return starts, lens, cu, int(padded.sum())

    def pack(self, waveforms: Sequence[np.ndarray]):
        """Concatenates clips into one pinned host buffer (test / bench helper).  Returns
        (pinned wave f32, pinned [starts | lens] int64, cu_frames int32 numpy)."""
        starts, lens, cu, total = self.tables([int(w.shape[0]) for w in waveforms])
        host = torch.empty(max(total, 4), dtype=torch.float32).pin_memory()
        for s, w, n in zip(starts, waveforms, lens):
            host[s:s + n].copy_(torch.from_numpy(np.ascontiguousarray(w, dtype=np.float32)))
        tables = torch.from_numpy(np.concatenate([starts, lens])).pin_memory()
        return host, tables, cu

    def _staging(self, total: int, b: int, m: int):
        """Grow-only pinned staging + device input buffers (cudaHostAlloc per call would dominate the step)."""
        st = getattr(self, '_stage', None)
        if st is None or st['wave_h'].numel() < total or st['tab_h'].numel() < 4 * b + 8 or st['out_h'].numel() < 9 * m + 4 * b + 64:
            cap_w = max(total, 4, int(1.25 * st['wave_h'].numel()) if st else 0)
            cap_b = max(4 * b + 8, st['tab_h'].numel() if st else 0)
            cap_o = max(9 * m + 4 * b + 64, int(1.25 * st['out_h'].numel()) if st else 0)
            st = {
                'wave_h': torch.empty(cap_w, dtype=torch.float32).pin_memory(),
                'wave_d': torch.empty(cap_w, dtype=torch.float32, device=self.device),
                'tab_h': torch.empty(cap_b, dtype=torch.int64).pin_memory(),
                'tab_d': torch.empty(cap_b, dtype=torch.int64, device=self.device),
                'cu_h': torch.empty(cap_b, dtype=torch.int32).pin_memory(),       # per-chunk cu_frames, staged as int32
                'cu_d': torch.empty(cap_b, dtype=torch.int32, device=self.device),
                'out_h': torch.empty(cap_o, dtype=torch.uint8).pin_memory(),
                'out_d': torch.empty(cap_o, dtype=torch.uint8, device=self.device),
            }
            self._stage = st
        return st

    # Pipeline chunks of a large batch: staging + H2D of chunk c+1 overlap the kernels of chunk c.  Small chunks cost
    # kernel efficiency (measured on 64 x 30 s: 1 / 2 / 4 / 8 equal chunks -> 38.0 / 38.9 / 40.7 / 44.9 ms of kernels), so
    # the split is geometric: a small first chunk gets the GPU going, the later ones stay big.
    CHUNK_FRACTIONS = (0.125, 0.375, 0.5)
    MIN_CHUNK_FRAMES = 16384
    GRAPH_MAX_FRAMES = 1024       # chunks up to this many frames (one ~10 s clip) go through CUDA-graph replay: -17 % device
                                  # time at 862 frames, no gain beyond ~2000 (measured); SOME_B200_GRAPHS=0 disables

    def _graphed(self, key, fn):
        """Runs ``fn`` (kernel launches on the current stream, no allocation, no sync) through a cached CUDA graph: eager the
        first time a key is seen (function attributes / tensor maps get set up, one-off shapes are never captured), captured
        on the second, replayed from then on.  At most 32 graphs are kept."""
        seen = self._graph_seen.get(key, 0)
        self._graph_seen[key] = seen + 1
        g = self._graphs.get(key)
        if g is None:
            if seen == 0 or len(self._graphs) >= 32:
                if len(self._graph_seen) > 4096:
                    self._graph_seen.clear()
                fn()
                return
            launches0 = self.launches
            stream = torch.cuda.current_stream(self.device)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=self._graph_stream(stream)):
                fn()
            self._graphs[key] = (g, self.launches - launches0)
            self.launches = launches0
            g = self._graphs[key]
        g[0].replay()
        self.launches += g[1]

    def _graph_stream(self, stream):
        if getattr(self, '_gstream', None) is None:
            self._gstream = torch.cuda.Stream(self.device)
        return self._gstream

    def _chunks(self, cu: np.ndarray) -> List[tuple]:
        b, m = len(cu) - 1, int(cu[-1])
        if b < 2 or m < 2 * self.MIN_CHUNK_FRAMES:
            return [(0, b)]
        bounds, acc = [0], 0.0
        for f in self.CHUNK_FRACTIONS[:-1]:
            acc += f
            i = int(np.searchsorted(cu, acc * m, side='left'))
            i = min(max(i, bounds[-1] + 1), b - 1)
            if cu[i] - cu[bounds[-1]] >= self.MIN_CHUNK_FRAMES // 2 and i > bounds[-1]:
                bounds.append(i)
        bounds.append(b)
        return [(bounds[i], bounds[i + 1]) for i in range(len(bounds) - 1) if bounds[i + 1] > bounds[i]]

    def _pool(self):
        if getattr(self, '_tp', None) is None:
            import concurrent.futures
            import os
            # staging threads: memcpy-bound; leave cores to the other ranks of a one-process-per-GPU job
            local_world = int(os.environ.get('LOCAL_WORLD_SIZE', '1') or 1)
            cores = len(os.sched_getaffinity(0)) if hasattr(os, 'sched_getaffinity') else (os.cpu_count() or 4)
            self._tp = concurrent.futures.ThreadPoolExecutor(max_workers=min(8, max(2, cores // (2 * local_world))))
        return self._tp

    def slab_layout_cached(self, lens: Sequence[int]):
        """slab_layout memoised on the clip lengths (a data-parallel step derives every rank's layout on every rank)."""
        key = tuple(int(x) for x in lens)
        cache = self.__dict__.setdefault('_layout_cache', {})
        hit = cache.get(key)
        if hit is None:
            if len(cache) >= 256:
                cache.clear()
            hit = cache[key] = self.slab_layout(key)
        return hit

    def slab_layout(self, lens: Sequence[int]):
        """Deterministic layout of the packed note slab of a batch with these clip lengths: per pipeline chunk
        (c0, c1, byte offset, clips, frames) and the total size.  Chunk slab = [counts i32 [bc] | dur i32 [mc] | midi f32 [mc]
        | rest u8 [mc]].  Every rank of a data-parallel job can compute every other rank's layout from the lengths alone."""
        _, _, cu, _ = self.tables(lens)
        layout, off = [], 0
        for c0, c1 in self._chunks(cu):
            bc, mc = c1 - c0, int(cu[c1] - cu[c0])
            layout.append((c0, c1, off, bc, mc))
            off += (4 * bc + 9 * mc + 15) & ~15
        return cu, layout, off

    def enqueue(self, waveforms: Sequence[np.ndarray], quantized: bool = False, return_intermediates: bool = False,
                resident=None, out: Optional[torch.Tensor] = None):
        """Stages, copies and enqueues the whole batch WITHOUT synchronising.  Returns (device slab uint8 [nbytes], cu, layout,
        extra): the decoded notes land in the device slab (see slab_layout); the caller copies it to the host (infer) or
        hands it to the all-gather (dist.infer_sharded).

        ``out``: optional device uint8 buffer (16-byte aligned, >= the slab size) the decode kernel writes the slab into instead
        of the engine's own — dist.infer_sharded passes this rank's slot of the all-gather buffer, so the notes go from the
        decode kernel to the collective without a staging copy.

        Contract: the engine owns ONE set of staging / slab buffers.  A second enqueue() may only be issued after the consumer
        of the previous one has synchronised (or waited on the stream): infer(), infer_sliced(), dist.infer_sharded() and the
        dataset driver all do.  The call itself first makes the copy stream wait for everything enqueued so far.

        ``resident = (wave_d, ranges)``: the audio is already on the device (f32 tensor) and the clips are the sample ranges
        ``[(begin, end), ...]`` inside it (``waveforms`` is ignored): no staging, no audio H2D — the slicer path
        (infer_sliced) cuts the recording where it lies."""
        dev = self.device
        if resident is not None:
            wave_res, ranges = resident
            b = len(ranges)
            starts = np.asarray([r[0] for r in ranges], dtype=np.int64)
            lens = np.asarray([r[1] - r[0] for r in ranges], dtype=np.int64)
            cu = np.zeros(b + 1, dtype=np.int32)
            np.cumsum(1 + lens // HOP, out=cu[1:])
            total = 0
        else:
            b = len(waveforms)
            starts, lens, cu, total = self.tables([int(w.shape[0]) for w in waveforms])
        m = int(cu[-1])
        if return_intermediates:
            layout, nbytes_total = [(0, b, 0, b, m)], (4 * b + 9 * m + 15) & ~15
        else:
            _, layout, nbytes_total = self.slab_layout(lens)
        st = self._staging(total, b, m)
        stream = torch.cuda.current_stream(dev)
        if getattr(self, '_copy_stream', None) is None:
            self._copy_stream = torch.cuda.Stream(dev)
        copy_stream = self._copy_stream
        if getattr(self, '_h2d_done', None) is not None:
            self._h2d_done.synchronize()      # the previous call's H2D copies have finished READING the pinned staging buffers
        copy_stream.wait_stream(stream)       # previous users of the staging / device buffers are done
        wave_h, wave_d, tab_h, tab_d, out_d = (st[k] for k in ('wave_h', 'wave_d', 'tab_h', 'tab_d', 'out_d'))
        if out is not None:
            assert out.dtype == torch.uint8 and out.is_cuda and out.numel() >= nbytes_total and out.data_ptr() % 16 == 0
            out_d = out
        if resident is not None:
            wave_d = wave_res
            direct = []
        else:
            hv = wave_h.numpy()
            pool = self._pool()

            def stage(i):
                n = int(lens[i])
                if n:
                    hv[starts[i]:starts[i] + n] = waveforms[i]          # dtype cast (if any) + memcpy, GIL released

            # Clips that already live in page-locked memory (pinned_array(), or any float32 view of a pinned torch tensor)
            # are copied H2D straight from the caller's buffer: no staging memcpy at all.  Everything else goes through the
            # pinned staging buffer.
            direct = [bool(lens[i]) and w.dtype == np.float32 and w.flags.c_contiguous and torch.from_numpy(w).is_pinned()
                      for i, w in enumerate(waveforms)]

        ws = self.workspace(max(mc for *_, mc in layout))
        extra = None
        cu_h, cu_dev = st['cu_h'], st['cu_d']
        for ci, (c0, c1, out_off, bc, mc) in enumerate(layout):
            lo = int(starts[c0])
            todo = []
            if resident is None:
                todo = [i for i in range(c0, c1) if not direct[i]]
                if todo:
                    list(pool.map(stage, todo))
                hi = int(starts[c1 - 1] + ((lens[c1 - 1] + 3) & ~3))
            # var-len tables of this chunk, relative to its own first sample / first frame
            tab = tab_h[2 * c0:2 * c0 + 2 * bc]
            tab[:bc] = torch.from_numpy(starts[c0:c1] - lo)
            tab[bc:2 * bc] = torch.from_numpy(lens[c0:c1])
            tab_dev = tab_d[2 * c0:2 * c0 + 2 * bc]
            cu_c = cu_h[c0 + ci:c1 + ci + 1]                 # chunk ci owns entries [c0 + ci, c1 + ci]: no overlap
            cu_c.copy_(torch.from_numpy(cu[c0:c1 + 1] - cu[c0]))
            cu_d = cu_dev[c0 + ci:c1 + ci + 1]
            with torch.cuda.stream(copy_stream):
                if resident is not None:
                    pass
                elif len(todo) == c1 - c0:
                    if hi > lo:
                        wave_d[lo:hi].copy_(wave_h[lo:hi], non_blocking=True)
                else:
                    for i in range(c0, c1):
                        n = int(lens[i])
                        if n:
                            src = torch.from_numpy(waveforms[i]) if direct[i] else wave_h[starts[i]:starts[i] + n]
                            wave_d[starts[i]:starts[i] + n].copy_(src, non_blocking=True)
                tab_dev.copy_(tab, non_blocking=True)
                cu_d.copy_(cu_c, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(copy_stream)
            stream.wait_event(ev)
            max_frames = int(np.diff(cu[c0:c1 + 1]).max())
            # decode writes straight into this chunk's slab
            o = out_d[out_off:out_off + 4 * bc + 9 * mc]
            note_count = o[:4 * bc].view(torch.int32)
            note_dur = o[4 * bc:4 * bc + 4 * mc].view(torch.int32)
            note_midi = o[4 * bc + 4 * mc:4 * bc + 8 * mc].view(torch.float32)
            note_rest = o[4 * bc + 8 * mc:]
            mel_f32 = torch.empty((mc, 80), dtype=torch.float32, device=dev) if return_intermediates else None
            pdl = self.pdl == 'all' or (self.pdl == 'small' and mc <= self.GRAPH_MAX_FRAMES)

            def launch_chunk():
                self.run_mel(wave_d[lo:], tab_dev[:bc], tab_dev[bc:2 * bc], cu_d, bc, max_frames, mel_f32, ws.units)
                was = self.lib.some_set_pdl(1) if pdl else 0    # programmatic dependent launch of the trunk kernels
                try:
                    self.run_trunk(ws, mc, bc, cu_d, max_frames, 'softmax' if quantized else 'sigmoid')
                finally:
                    if pdl:
                        self.lib.some_set_pdl(was)
                self.run_decode(ws, mc, bc, cu_d, note_count, quantized, out=(note_midi, note_dur, note_rest))

            if mc <= self.GRAPH_MAX_FRAMES and self.use_graphs and self.prof is None and not return_intermediates:
                # small batches are launch-bound (~56 launches of a few microseconds each): replay them as ONE CUDA graph,
                # keyed by everything the captured kernel arguments depend on
                self._graphed((wave_d.data_ptr() + 4 * lo, tab_dev.data_ptr(), cu_d.data_ptr(), o.data_ptr(), ws.serial, bc, mc,
                               max_frames, bool(quantized), self.ln_fold, pdl), launch_chunk)
            else:
                launch_chunk()
            if return_intermediates:
                extra = (mel_f32, ws.probs[:mc], ws.bounds[:mc])
        self._h2d_done = ev if layout else None
        return out_d[:nbytes_total], cu, layout, extra

    def rms_frames(self, wave_d: torch.Tensor, frame_length: int, hop: int) -> np.ndarray:
        """Short-time RMS of a device-resident f32 waveform (some_slicer_rms), bit-identical to the reference's get_rms
        (utils/slicer2.py:5-38).  Returns the host copy (one small D2H + sync): the slicer's state machine runs on the host."""
        n = int(wave_d.numel())
        n_frames = 1 + (n + 2 * (frame_length // 2) - frame_length) // hop
        rms_d = torch.empty(n_frames, dtype=torch.float32, device=self.device)
        _lib.check(self.lib.some_slicer_rms(wave_d.data_ptr(), n, frame_length, hop, rms_d.data_ptr(), n_frames, self._stream),
                   'some_slicer_rms')
        self.launches += 1
        return rms_d.cpu().numpy()

    def rms_frames_many(self, waves_d: Sequence[torch.Tensor], frame_length: int, hop: int) -> List[np.ndarray]:
        """RMS lists of several device-resident recordings: one launch each into ONE buffer, one D2H copy and sync for all
        (the dataset driver, some_b200/batch.py)."""
        counts = [1 + (int(w.numel()) + 2 * (frame_length // 2) - frame_length) // hop for w in waves_d]
        if not counts:
            return []
        cuts = np.zeros(len(counts) + 1, dtype=np.int64)
        np.cumsum(counts, out=cuts[1:])
        rms_d = torch.empty(int(cuts[-1]), dtype=torch.float32, device=self.device)
        for w, a, n in zip(waves_d, cuts, counts):
            _lib.check(self.lib.some_slicer_rms(w.data_ptr(), int(w.numel()), frame_length, hop, rms_d[a:].data_ptr(), n,
                                                self._stream), 'some_slicer_rms')
            self.launches += 1
        host = rms_d.cpu().numpy()
        return [host[a:b] for a, b in zip(cuts[:-1], cuts[1:])]

    def infer_sliced(self, waveform: np.ndarray, slicer, quantized: bool = False):
        """One long mono recording -> (chunk offsets in seconds, per-chunk notes): the flow of infer.py:38-41 /
        batch_infer.py:50-54 (Slicer.slice, then infer on the chunks) with the recording uploaded ONCE.  The RMS frames are
        computed on the device, the slicer's decisions are taken on the host from the copied RMS list (15 k floats for 5 min),
        and the chunks are then processed where they lie in device memory as one var-len batch."""
        from .slicer import chunk_ranges, silence_tags
        samples = np.ascontiguousarray(waveform, dtype=np.float32)
        assert samples.ndim == 1, 'infer_sliced expects a mono waveform (infer.py loads with mono=True)'
        n = int(samples.shape[0])
        dev = self.device
        with torch.cuda.device(dev):
            if (n + slicer.hop_size - 1) // slicer.hop_size <= slicer.min_length:   # slicer2.py:79-80
                return [0], self.infer([samples], quantized)
            src = torch.from_numpy(samples)
            if not src.is_pinned():
                st = self._staging(n, 1, 1 + n // HOP)
                st['wave_h'][:n].copy_(src)
                src = st['wave_h'][:n]
            wave_d = torch.empty(n, dtype=torch.float32, device=dev)
            wave_d.copy_(src, non_blocking=True)
            rms = self.rms_frames(wave_d, slicer.win_size, slicer.hop_size)
            ranges = chunk_ranges(silence_tags(rms, slicer), rms.shape[0], slicer.hop_size, n)
            if not ranges:
                return [], []
            slab, cu, layout, _ = self.enqueue(None, quantized, resident=(wave_d, ranges))
            self._staging(0, len(ranges), int(cu[-1]))
            out_h = self._stage['out_h']
            out_h[:slab.numel()].copy_(slab, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
            results = self.unpack_slab(out_h[:slab.numel()].numpy(), cu, layout)
        offsets = [begin / slicer.sr for begin, _ in ranges]
        return offsets, results

    def unpack_slab(self, host: np.ndarray, cu: np.ndarray, layout, extra=None) -> List[Dict[str, np.ndarray]]:
        """Host copy of a packed note slab -> one dict per clip (input order).  Conversions are done once per chunk on the
        whole arrays; the per-clip entries are slices."""
        results: List[Dict[str, np.ndarray]] = []
        for c0, c1, off, bc, mc in layout:
            h = host[off:off + 4 * bc + 9 * mc]
            results.extend(self.unpack(cu[c0:c1 + 1] - cu[c0], h[:4 * bc].view(np.int32),
                                       h[4 * bc + 4 * mc:4 * bc + 8 * mc].view(np.float32),
                                       h[4 * bc:4 * bc + 4 * mc].view(np.int32), h[4 * bc + 8 * mc:4 * bc + 9 * mc], extra))
        return results

    def infer(self, waveforms: Sequence[np.ndarray], quantized: bool = False,
              return_intermediates: bool = False) -> List[Dict[str, np.ndarray]]:
        """waveform-in -> notes-out for a list of clips: the batched equivalent of BaseInference.infer
        (base_infer.py:46-53).  Host buffers in, host buffers out.  The batch is cut into up to 3 chunks of whole clips
        (small first chunk); for each chunk the clips are staged into pinned memory by a small thread pool (memcpy releases
        the GIL), copied H2D on a copy stream, and the kernels of the chunk are enqueued behind an event — so staging and
        H2D of chunk c+1 overlap the kernels of chunk c.  The notes come back in ONE packed D2H copy
        [counts | dur | midi | rest] per chunk slab; there is a single host synchronisation at the end."""
        if len(waveforms) == 0:
            return []
        dev = self.device
        with torch.cuda.device(dev):
            slab, cu, layout, extra = self.enqueue(waveforms, quantized, return_intermediates)
            out_h = self._stage['out_h']
            out_h[:slab.numel()].copy_(slab, non_blocking=True)
            if extra is not None:
                extra = tuple(t.cpu() for t in extra)
            torch.cuda.current_stream(dev).synchronize()
            return self.unpack_slab(out_h[:slab.numel()].numpy(), cu, layout, extra)

    def infer_accurate(self, waveforms: Sequence[np.ndarray], quantized: bool = False) -> List[Dict[str, np.ndarray]]:
        """VALIDATION mode: the same waveform -> notes path with the trunk in fp32 on the CUDA cores (some_forward_f32,
        csrc/accurate.cu) — no bf16, no tensor cores, exact activations.  Asserts the "within 1e-3 fp32" line of the contract
        (tests/test_gpu_accurate.py) and shows that operand rounding is the only source of note differences in the product
        path.  ~100x slower than infer(); one clip at a time; returns mel / probs / bounds with the notes."""
        from .weights import build_f32_model
        dev = self.device
        out = []
        with torch.cuda.device(dev):
            if self._f32 is None:
                self._f32 = build_f32_model(self._state_dict, self.config, dev)
            cmodel = self._f32[0]
            head = _lib.EPI_SOFTMAX_F32 if quantized else _lib.EPI_SIGMOID_F32
            for w in waveforms:
                host, tables, cu = self.pack([w])
                m = int(cu[-1])
                wave_d, tab_d, cu_d = host.to(dev), tables.to(dev), torch.from_numpy(cu).to(dev)
                f = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)
                t = {'x': f(2, m, DIM), 'a': f(2, m, DIM), 'h': f(2, m, FFN_DIM), 'qkv': f(2, m, 3 * DIM), 'g': f(2, m, DIM),
                     'y': f(2, m, 2 * DIM), 'units': f(m, 80), 'probs': f(m, self.outdim), 'bounds': f(m)}
                c = _lib.WorkspaceF32C()
                for s in range(2):
                    for k in ('x', 'a', 'h', 'qkv', 'g', 'y'):
                        getattr(c, k)[s] = t[k][s].data_ptr()
                c.units, c.probs, c.bounds = t['units'].data_ptr(), t['probs'].data_ptr(), t['bounds'].data_ptr()
                self.run_mel(wave_d, tab_d[:1], tab_d[1:], cu_d, 1, m, t['units'], None)
                _lib.check(self.lib.some_forward_f32(C.byref(cmodel), C.byref(c), m, 1, cu_d.data_ptr(), m, head, self._stream),
                           'some_forward_f32')
                ws = self.workspace(m)
                nc = torch.empty(1, dtype=torch.int32, device=dev)
                self.run_decode(ws, m, 1, cu_d, nc, quantized, probs=t['probs'], bounds=t['bounds'])
                n = int(nc.item())
                out.append({'note_midi': ws.note_midi[:n].cpu().numpy(),
                            'note_dur': ws.note_dur[:n].cpu().numpy().astype(np.int64) * self.timestep,
                            'note_rest': ws.note_rest[:n].cpu().numpy().astype(bool),
                            'mel': t['units'].cpu().numpy(), 'probs': t['probs'].cpu().numpy(), 'bounds': t['bounds'].cpu().numpy()})
        return out

    def unpack(self, cu, nc, nm, nd, nr, extra=None) -> List[Dict[str, np.ndarray]]:
        # The slab has room for one note per FRAME (notes of clip j start at row cu[j]); only ~1 row in 5 is used.  Gather the
        # used rows first (three fancy-index copies of `total` elements: they also detach the result from the pinned landing
        # buffer, which the next call reuses) and convert only those.
        count = np.asarray(nc, dtype=np.int64)
        ends = np.cumsum(count)
        total = int(ends[-1]) if len(ends) else 0
        starts = ends - count
        rows = np.repeat(np.asarray(cu[:-1], dtype=np.int64) - starts, count) + np.arange(total, dtype=np.int64)
        dur_s = nd[rows] * self.timestep   # me_infer.py:95: int64 * python float -> float64; int32 * float gives the same float64s
        rest_b = nr[rows].astype(bool)
        midi = nm[rows]
        lo, hi = starts.tolist(), ends.tolist()
        if extra is None:
            return [{'note_midi': midi[a:b], 'note_dur': dur_s[a:b], 'note_rest': rest_b[a:b]} for a, b in zip(lo, hi)]
        out = []
        for i, (a, b) in enumerate(zip(lo, hi)):
            r0, e1 = int(cu[i]), int(cu[i + 1])
            out.append({'note_midi': midi[a:b], 'note_dur': dur_s[a:b], 'note_rest': rest_b[a:b],
                        'mel': extra[0][r0:e1].numpy(), 'probs': extra[1][r0:e1].numpy(), 'bounds': extra[2][r0:e1].numpy()})
        return out

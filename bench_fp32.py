"""Measures the fp32 trunk: what Engine.infer(precision='fp32') (some_forward_f32_tiled) costs next to the bf16 product
path and the fp32 checker it is bit-identical to (some_forward_f32, one clip at a time as Engine.infer_accurate runs it).

Workloads, in one process, on seeded synthetic weights and audio:
- C2: two_head, 64 clips of 30 s;
- C4: midi_conformer, 32 clips of 10 s.

Per workload:
- audio-s/s of waveform -> notes for bf16 (Engine.infer), the fp32 checker (Engine.infer_accurate, one run) and the tiled
  fp32 path (Engine.infer(precision='fp32')); wall time around calls that end in a synchronise, median of --rounds;
- per-kernel device time of the three tiled kernels over one tiled trunk pass (torch.profiler), with their FLOP counted
  from the shapes and the rate against the 67 TFLOP/s FP32 data-sheet figure of the H100 SXM;
- the card's name and power limit, and the median SM clock sampled while the tiled path runs;
- torch.equal of every workspace buffer of the tiled trunk against the checker's trunk on the same timed batch, and of
  the tiled path's notes against the checker's.

    python bench_fp32.py [--rounds 3] [--workloads C2,C4]

Prints one JSON line per workload."""
import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

FP32_PEAK_TFLOPS = 67.0                    # H100 SXM data sheet, dense FP32
WORKLOADS = {'C2': ('two_head', 64, 30.0), 'C4': ('midi_conformer', 32, 10.0)}
TILED = {'gemm': 'sgemm_tiled_kernel', 'attention': 'attention_f32_tiled_kernel', 'dwconv': 'dwconv_f32_tiled_kernel'}


def card_static():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(',')]
        return {'gpu': name, 'power_limit_w': float(power)}
    except Exception as e:                 # noqa: BLE001
        return {'gpu': f'unknown ({e})', 'power_limit_w': None}


class ClockSampler:
    """Samples the SM clock with nvidia-smi while the block runs; median on exit."""

    def __enter__(self):
        self.samples, self.stop = [], threading.Event()

        def run():
            while not self.stop.is_set():
                try:
                    out = subprocess.run(['nvidia-smi', '--query-gpu=clocks.sm', '--format=csv,noheader,nounits', '-i', '0'],
                                         capture_output=True, text=True, timeout=10).stdout.strip()
                    self.samples.append(float(out.splitlines()[0]))
                except Exception:          # noqa: BLE001
                    pass
                self.stop.wait(0.2)
        self.thread = threading.Thread(target=run, daemon=True)
        self.thread.start()
        return self

    def __exit__(self, *exc):
        self.stop.set()
        self.thread.join()
        self.median = statistics.median(self.samples) if self.samples else None
        return False


def flops(lay, outdim, m, sum_t2, d=512):
    """Algorithmic FLOP of one trunk pass (both streams), by kernel."""
    blocks = 2 * (lay + 1)
    gemm = blocks * 46 * m * d * d + lay * 8 * m * d * d + 2 * 2 * m * 80 * d + 2 * m * d * outdim
    attention = blocks * 4 * d * sum_t2          # QK^T and P.V, 8 heads x 64 channels, 2 FLOP per multiply-add
    dwconv = blocks * 2 * 31 * m * d
    return {'gemm': gemm, 'attention': attention, 'dwconv': dwconv}


def timed(fn, rounds):
    import torch
    times = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return statistics.median(times), out


def trunk_pass(eng, fn, units, cu, ws_cls):
    """One trunk pass of `fn` (some_forward_f32 or _tiled) over the batch's mel; returns the workspace tensors."""
    import torch
    from some_b200 import _lib
    m, b = int(cu[-1]), len(cu) - 1
    ws = ws_cls(m, eng.outdim, eng.device)
    ws.block.zero_()                                               # the gaps between the buffers too: blocks compare whole
    ws.units[:m].copy_(units)
    cu_d = torch.from_numpy(cu.astype(np.int32)).to(eng.device)
    _lib.check(fn(C.byref(eng.model_f32()), C.byref(ws.c), m, b, cu_d.data_ptr(), int(np.diff(cu).max()),
                  _lib.EPI_SIGMOID_F32, eng._stream), 'trunk')
    torch.cuda.synchronize()
    return ws


def kernel_times(eng, units, cu, ws_cls):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ws = trunk_pass(eng, eng.lib.some_forward_f32_tiled, units, cu, ws_cls)
    del ws
    ms = {k: 0.0 for k in TILED}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            for k, name in TILED.items():
                if name in e.name:
                    ms[k] += e.time_range.elapsed_us() / 1000.0
    return ms


def run(name, rounds):
    import torch
    from some_b200 import engine, plugin, synth
    cfg, n, seconds = WORKLOADS[name]
    config = synth.named_config(cfg)
    with tempfile.TemporaryDirectory() as d:
        ckpt = synth.write_checkpoint(d, config, seed=1234)
        ins = plugin.MIDIExtractionInference(config=config, model_path=ckpt, device='cuda:0')
    eng = ins.model
    waves = [synth.synth_waveform(5000 + i, seconds=seconds) for i in range(n)]
    audio_s = n * seconds
    res = {'workload': name, 'config': cfg, 'clips': n, 'seconds': seconds}

    eng.infer(waves)                                             # warm-up: module load, staging buffers
    t_bf16, _ = timed(lambda: eng.infer(waves), rounds)
    eng.infer(waves, precision='fp32')
    with ClockSampler() as clk:
        t_f32, got = timed(lambda: eng.infer(waves, precision='fp32'), rounds)
    eng.infer_accurate(waves[:1])
    t_chk, want = timed(lambda: eng.infer_accurate(waves), 1)
    res['audio_s_per_s'] = {'bf16': audio_s / t_bf16, 'fp32_checker': audio_s / t_chk, 'fp32_tiled': audio_s / t_f32}
    res['call_s'] = {'bf16': t_bf16, 'fp32_checker': t_chk, 'fp32_tiled': t_f32}
    res['notes_equal_checker'] = all(np.array_equal(g[k], w[k]) for g, w in zip(got, want)
                                     for k in ('note_midi', 'note_dur', 'note_rest'))
    del got, want

    # trunk alone on the timed batch: per-kernel times, and tiled == checker on every output
    host, tables, cu = eng.pack(waves)
    m = int(cu[-1])
    units = torch.empty((m, 80), dtype=torch.float32, device=eng.device)
    tab = tables.to(eng.device)
    eng.run_mel(host.to(eng.device), tab[:n], tab[n:], torch.from_numpy(cu).to(eng.device), n, int(np.diff(cu).max()),
                units, None)
    ms = kernel_times(eng, units, cu, engine._WorkspaceF32)
    t = np.diff(cu).astype(np.float64)
    fl = flops(eng.w.lay, eng.outdim, m, float((t * t).sum()))
    res['kernels'] = {k: {'ms': ms[k], 'tflop': fl[k] / 1e12, 'tflops': fl[k] / (ms[k] * 1e9) if ms[k] else None,
                          'of_fp32_peak': fl[k] / (ms[k] * 1e9) / FP32_PEAK_TFLOPS if ms[k] else None} for k in TILED}
    eng._ws32 = None
    torch.cuda.empty_cache()
    tiled = trunk_pass(eng, eng.lib.some_forward_f32_tiled, units, cu, engine._WorkspaceF32)
    chk = trunk_pass(eng, eng.lib.some_forward_f32, units, cu, engine._WorkspaceF32)
    # same carve of two zeroed blocks: equal blocks = every buffer (x a h qkv g y units probs bounds) equal
    res['tiled_equals_checker'] = bool(torch.equal(tiled.block, chk.block))
    del tiled, chk
    torch.cuda.empty_cache()
    res.update(card_static())
    res['sm_clock_median_mhz'] = clk.median
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--workloads', default='C2,C4')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_fp32.py needs a CUDA device')
    torch.cuda.set_device(0)
    ok = True
    for name in args.workloads.split(','):
        res = run(name, args.rounds)
        ok &= res['tiled_equals_checker'] and res['notes_equal_checker']
        print(json.dumps(res), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == '__main__':
    main()

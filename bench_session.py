"""Times the native session (csrc/session.cu) against the Python plugin in one process, runs alternated:

* C2: a batch of 64 x 30 s clips through some_session_transcribe vs plugin.infer();
* C5: one 5-minute recording with silences through some_session_transcribe_sliced vs Engine.infer_sliced.

Both sides get the same numpy float32 inputs in ordinary (pageable) host memory and return notes on the host; the outputs are
compared bit for bit.  Prints the card's name and power limit with the numbers, then one JSON line.

    python bench_session.py [--steps 10] [--config two_head] [--profile DIR]

``--profile DIR`` then traces three C5 calls of each side with torch.profiler (CUDA activities: the session's copies and
kernels are recorded too, being in the same process), writes the chrome traces under DIR and prints, per call, where the wall
clock went: device time of the kernels, host-to-device and device-to-host copies, and the time the GPU was idle inside the call.
Tracing slows the host, so these splits are taken in a run of their own, after the timed runs.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REPO)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:              # noqa: BLE001
        q = f'nvidia-smi unavailable ({e!r})'
    return q


def same(a, b):
    return len(a) == len(b) and all(np.array_equal(x['note_midi'].view(np.uint32), y['note_midi'].view(np.uint32))
                                    and np.array_equal(x['note_dur'], y['note_dur']) and np.array_equal(x['note_rest'], y['note_rest'])
                                    for x, y in zip(a, b))


def split_trace(path, label):
    """Per traced call ``label`` (a record_function range): wall ms, kernel ms, H2D ms, D2H ms, GPU idle ms."""
    with open(path) as f:
        ev = [e for e in json.load(f)['traceEvents'] if e.get('ph') == 'X']
    calls = sorted((e['ts'], e['ts'] + e['dur']) for e in ev if e.get('name') == label and e.get('cat') == 'user_annotation')
    gpu = [e for e in ev if e.get('cat') in ('kernel', 'gpu_memcpy', 'gpu_memset')]
    out = []
    for t0, t1 in calls:
        inside = sorted((e['ts'], e['ts'] + e['dur'], e) for e in gpu if t0 <= e['ts'] < t1)
        busy, end = 0.0, t0
        for a, b, _ in inside:                  # union of the device intervals
            a = max(a, end)
            if b > a:
                busy += b - a
                end = b
        k = sum(e['dur'] for _, _, e in inside if e['cat'] == 'kernel')
        h2d = sum(e['dur'] for _, _, e in inside if e['cat'] == 'gpu_memcpy' and 'HtoD' in e['name'])
        d2h = sum(e['dur'] for _, _, e in inside if e['cat'] == 'gpu_memcpy' and 'DtoH' in e['name'])
        first = inside[0][0] - t0 if inside else 0.0
        out.append({'wall_ms': (t1 - t0) / 1e3, 'kernels_ms': k / 1e3, 'h2d_ms': h2d / 1e3, 'd2h_ms': d2h / 1e3,
                    'gpu_idle_ms': (t1 - t0 - busy) / 1e3, 'before_first_gpu_op_ms': first / 1e3})
    return out


def profile_c5(runs, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile, record_function
    os.makedirs(out_dir, exist_ok=True)
    res = {}
    for name in ('c5_engine', 'c5_session'):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                torch.cuda.synchronize()
                with record_function(name):
                    runs[name]()
                    torch.cuda.synchronize()
        path = os.path.join(out_dir, f'{name}.trace.json')
        prof.export_chrome_trace(path)
        res[name] = split_trace(path, name)
    return res


def timed(fn, steps):
    import torch
    out, ts = None, []
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return out, ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--config', default='two_head', choices=['two_head', 'quant_two_head'])
    ap.add_argument('--profile', metavar='DIR', help='also trace C5 calls of both sides and split their time (see above)')
    args = ap.parse_args()
    import torch

    from some_b200 import export, plugin, synth
    from some_b200 import session as nsess
    from some_b200.slicer import Slicer
    if not torch.cuda.is_available():
        raise SystemExit('bench_session.py needs a CUDA device')
    torch.cuda.set_device(0)
    cls = plugin.QuantizedMIDIExtractionInference if args.config == 'quant_two_head' else plugin.MIDIExtractionInference
    with tempfile.TemporaryDirectory() as d:
        config = synth.named_config(args.config)
        ckpt = synth.write_checkpoint(d, config, seed=1234)
        path = export.export(ckpt)
        ins = cls(config=config, model_path=ckpt, device='cuda:0')
        sess = nsess.Session(path, 0)
    n = int(30.0 * synth.SR)
    pool = [synth.synth_waveform(1000 + j, num_samples=n) for j in range(8)]       # bench.py's C2 clips
    clips = [np.ascontiguousarray(np.roll(pool[i % 8], 4099 * (i // 8)) * np.float32(1.0 - 0.01 * (i % 7))) for i in range(64)]
    rec = synth.synth_waveform(9002, seconds=300.0, silence_gaps=True)               # bench.py's C5 recording
    slicer = Slicer(synth.SR, max_sil_kept=1000)

    runs = {
        'c2_plugin': lambda: ins.infer(clips),
        'c2_session': lambda: sess.transcribe(clips),
        'c5_engine': lambda: ins.model.infer_sliced(rec, slicer, quantized=ins.quantized)[1],
        'c5_session': lambda: sess.transcribe_sliced(rec)[2],
    }
    outs = {k: fn() for k, fn in runs.items()}                   # warm-up: every shape once
    outs = {k: fn() for k, fn in runs.items()}
    times = {k: [] for k in runs}
    for _ in range(args.steps):                                  # alternated
        for k, fn in runs.items():
            _, ts = timed(fn, 1)
            times[k] += ts
    med = {k: float(np.median(v)) for k, v in times.items()}
    spread = {k: [float(min(v)), float(max(v))] for k, v in times.items()}
    res = {
        'card': card(),
        'config': args.config,
        'steps': args.steps,
        'C2_64x30s': {'plugin_ms': med['c2_plugin'], 'session_ms': med['c2_session'],
                      'plugin_audio_s_per_s': 64 * 30.0 / (med['c2_plugin'] / 1e3),
                      'session_audio_s_per_s': 64 * 30.0 / (med['c2_session'] / 1e3),
                      'session_over_plugin': med['c2_session'] / med['c2_plugin'],
                      'identical_notes': same(outs['c2_session'], outs['c2_plugin'])},
        'C5_5min_sliced': {'engine_ms': med['c5_engine'], 'session_ms': med['c5_session'],
                           'session_over_engine': med['c5_session'] / med['c5_engine'],
                           'chunks': len(outs['c5_session']),
                           'identical_notes': same(outs['c5_session'], outs['c5_engine'])},
        'min_max_ms': spread,
    }
    print(f'card: {res["card"]}')
    print(f'C2 64 x 30 s: plugin.infer {med["c2_plugin"]:.1f} ms, session {med["c2_session"]:.1f} ms '
          f'(x{res["C2_64x30s"]["session_over_plugin"]:.3f}), identical notes: {res["C2_64x30s"]["identical_notes"]}')
    print(f'C5 5 min sliced: Engine.infer_sliced {med["c5_engine"]:.1f} ms, session {med["c5_session"]:.1f} ms '
          f'(x{res["C5_5min_sliced"]["session_over_engine"]:.3f}), identical notes: {res["C5_5min_sliced"]["identical_notes"]}')
    if args.profile:
        res['C5_profile'] = profile_c5(runs, args.profile)
        for name, calls in res['C5_profile'].items():
            for c in calls:
                print(f'{name}: ' + ', '.join(f'{k} {v:.2f}' for k, v in c.items()))
    print(json.dumps(res))
    sess.close()


if __name__ == '__main__':
    main()

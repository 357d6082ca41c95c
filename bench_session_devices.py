"""Times one native session opened on several devices (some_session_open_devices) against the same session on one device:

* (a) 64 recordings of 30 s, WAV and FLAC mixed, through some_session_transcribe_encoded;
* (b) one 20-minute recording with silences (the web UI's upper limit) through some_session_transcribe_sliced;
* (c) 256 streams pushing 20 ms ticks through some_stream_push_many: p50 and p99 tick latency.

Configurations: [0], [0, 0] (two replicas on one GPU), and [0 .. k-1] for every k from 2 to the number of visible GPUs.  For
each it prints the median time of (a) and (b), the speed-up over [0], each replica's chunks and frames in the last call
(some_session_get_load), the tick latencies of (c), and whether every timed call's notes equal those of [0].  Every card's name
and power limit are read in the same run.  With one GPU visible, k >= 2 is reported as not measured.  The last line is JSON.

    python bench_session_devices.py [--steps 5] [--config two_head] [--stream-seconds 20]
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REPO)


def cards():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=index,name,power.limit', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    except Exception as e:              # noqa: BLE001
        return [f'nvidia-smi unavailable ({e!r})']


def pcm16(x):
    return np.clip(np.round(x * 32768), -32768, 32767)


def wav16(x, rate):
    raw = pcm16(x).astype('<i2').tobytes()
    fmt = struct.pack('<HHIIHH', 1, 1, rate, rate * 2, 2, 16)
    body = b'WAVE' + b'fmt ' + struct.pack('<I', 16) + fmt + b'data' + struct.pack('<I', len(raw)) + raw
    return b'RIFF' + struct.pack('<I', len(body)) + body


def key(res):
    """A result's ranges and the bits of its notes, for comparing calls."""
    if isinstance(res, tuple):
        return (res[1], [key(r) for r in res[2]])
    if isinstance(res, list):
        return [key(r) for r in res]
    return (res['note_midi'].view(np.uint32).tobytes(), res['note_frames'].tobytes(), res['note_rest'].tobytes())


def median_ms(fn, steps):
    out, ts = None, []
    for _ in range(steps):
        t = time.perf_counter()
        out = fn()
        ts.append(1e3 * (time.perf_counter() - t))
    return float(np.median(ts)), [float(min(ts)), float(max(ts))], out


def ticks(sess, waves, block):
    """256 streams, one push_many per 20 ms tick until every stream has finished: (tick latencies in ms, notes)."""
    streams = [sess.stream(44100) for _ in waves]
    got, lat = [[] for _ in waves], []
    try:
        n = max(len(w) for w in waves)
        for a in range(0, n + block, block):
            items = [(st, w[a:a + block]) for st, w in zip(streams, waves)]
            fin = [a + block >= n] * len(waves)
            t = time.perf_counter()
            res = sess.push_many(items, fin)
            lat.append(1e3 * (time.perf_counter() - t))
            for g, r in zip(got, res):
                g.append(key(r))
            if fin[0]:
                break
    finally:
        for st in streams:
            st.close()
    return np.array(lat), got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--config', default='two_head', choices=['two_head', 'quant_two_head', 'midi_conformer'])
    ap.add_argument('--stream-seconds', type=float, default=20.0)
    args = ap.parse_args()
    import torch

    from oracle import flac as of
    from some_b200 import export, synth
    from some_b200 import session as nsess
    if not torch.cuda.is_available():
        raise SystemExit('bench_session_devices.py needs a CUDA device')
    gpus = torch.cuda.device_count()
    print('cards:', *cards(), sep='\n  ', flush=True)

    n30 = int(30.0 * synth.SR)
    base = [synth.synth_waveform(1000 + j, num_samples=n30, silence_gaps=True) * np.float32(0.8) for j in range(8)]
    flacs = [of.encode(pcm16(x).astype(np.int64), rate=synth.SR, bps=16, subframe={'type': 'fixed', 'order': 2})
             for x in base[:4]]
    items = [flacs[i // 2 % 4] if i % 2 else wav16(np.roll(base[i % 8], 4099 * i), synth.SR) for i in range(64)]
    rec = synth.synth_waveform(9002, seconds=1200.0, silence_gaps=True)
    waves = [np.roll(base[i % 8], 977 * i)[:int(args.stream_seconds * synth.SR)] for i in range(256)]
    block = synth.SR * 20 // 1000

    configs = [[0], [0, 0]] + [list(range(k)) for k in range(2, gpus + 1)]
    report = {'cards': cards(), 'config': args.config, 'steps': args.steps, 'gpus_visible': gpus, 'runs': []}
    with tempfile.TemporaryDirectory() as d:
        path = export.export(synth.write_checkpoint(d, synth.named_config(args.config), seed=1234))
        want, base_ms = None, None
        for devices in configs:
            sess = nsess.Session(path, devices)
            calls = {'encoded_64x30s': lambda: sess.transcribe_encoded(items),
                     'sliced_20min': lambda: sess.transcribe_sliced(rec)}
            row = {'devices': devices}
            keys = {}
            for name, fn in calls.items():
                first = key(fn())                                       # warm-up: every buffer grown once
                ms, spread, out = median_ms(fn, args.steps)
                keys[name] = [first, key(out)]
                row[name] = {'ms': round(ms, 2), 'min_max_ms': [round(v, 2) for v in spread], 'load': sess.load()}
            lat, got = ticks(sess, waves, block)
            keys['streams_256x20ms'] = [got]
            row['streams_256x20ms'] = {'ticks': len(lat), 'p50_ms': round(float(np.percentile(lat, 50)), 3),
                                       'p99_ms': round(float(np.percentile(lat, 99)), 3), 'load_last_tick': sess.load()}
            sess.close()
            if want is None:
                want, base_ms = {k: v[0] for k, v in keys.items()}, {k: row[k].get('ms') for k in calls}
            row['notes_equal_to_[0]'] = all(all(v == want[k] for v in vs) for k, vs in keys.items())
            for k in calls:
                row[k]['speedup_over_[0]'] = round(base_ms[k] / row[k]['ms'], 3)
            report['runs'].append(row)
            print(f'{devices}: encoded {row["encoded_64x30s"]["ms"]:.1f} ms (x{row["encoded_64x30s"]["speedup_over_[0]"]:.2f}, '
                  f'load {row["encoded_64x30s"]["load"]}), sliced 20 min {row["sliced_20min"]["ms"]:.1f} ms '
                  f'(x{row["sliced_20min"]["speedup_over_[0]"]:.2f}, load {row["sliced_20min"]["load"]}), 256 streams: tick p50 '
                  f'{row["streams_256x20ms"]["p50_ms"]:.2f} ms p99 {row["streams_256x20ms"]["p99_ms"]:.2f} ms; notes equal to [0]: '
                  f'{row["notes_equal_to_[0]"]}', flush=True)
    if gpus < 2:
        report['k>=2'] = f'not measured: {gpus} GPU visible'
        print(report['k>=2'])
    print(json.dumps(report))


if __name__ == '__main__':
    main()

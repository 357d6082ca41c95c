"""Measures calls from many threads on one native session, whose queued calls run together as one GPU step, against the
same threads taking turns.  Two arms per configuration, alternated in one process:

- locked: every thread holds one Python lock around each session call, so every call runs as a step of its own (the
  schedule of a session that runs one call per step);
- free: the same threads without the lock; calls that queue behind a running step share the next one.

Configurations:

- encoded: T threads (1, 4, 16, 64) share 64 calls, each one 3-minute 16-bit WAV file (Session.transcribe_encoded);
- stream: T threads (1, 16, 128), each pushing one PCM stream in fixed blocks (20 ms and 100 ms) and finishing it, on the
  recordings bench_stream.py uses (synth_waveform(7000 + i, silence_gaps=True), 44.1 kHz).

Reports the aggregate audio-seconds per second, the wall time of a call (median and p99), the steps and the calls per step
(some_session_get_stats), and whether every result equals the single call's result (the same ranges and note bits).  Prints
the card's name and power limit beside the numbers, and one JSON line per configuration, arm and round.

    python bench_session_threads.py [--encoded-threads 1,4,16,64] [--stream-threads 1,16,128] [--blocks-ms 20,100]
                                    [--stream-seconds 30] [--rounds 2]"""
import argparse
import contextlib
import json
import struct
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                 # noqa: BLE001
        return f'unknown ({e})'


def wav16(x, rate):
    raw = np.clip(np.round(x * 32768), -32768, 32767).astype('<i2').tobytes()
    fmt = struct.pack('<HHIIHH', 1, 1, rate, rate * 2, 2, 16)
    body = b'WAVE' + b'fmt ' + struct.pack('<I', 16) + fmt + b'data' + struct.pack('<I', len(raw)) + raw
    return b'RIFF' + struct.pack('<I', len(body)) + body


def key(res):
    """One call's result as comparable values: ranges and the bits of every note."""
    offsets, ranges, notes = res
    return ranges, [(n['note_midi'].view(np.uint32).tobytes(), n['note_frames'].tobytes(), n['note_rest'].tobytes())
                    for n in notes]


def run_arm(sess, n_threads, work, locked):
    """work(t, call) runs thread t's calls, each through call(fn) -> fn(); returns (wall, per-call seconds, stats delta,
    errors)."""
    lock = threading.Lock() if locked else None
    times, errors = [[] for _ in range(n_threads)], []

    def call(t, fn):
        t0 = time.perf_counter()
        with (lock if lock else contextlib.nullcontext()):
            r = fn()
        times[t].append(time.perf_counter() - t0)
        return r

    def body(t):
        try:
            work(t, lambda fn: call(t, fn))
        except Exception as e:         # noqa: BLE001
            errors.append(repr(e))
    before = sess.stats()
    threads = [threading.Thread(target=body, args=(t,)) for t in range(n_threads)]
    t = time.perf_counter()
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    wall = time.perf_counter() - t
    after = sess.stats()
    return wall, [x for ts in times for x in ts], {k: after[k] - before[k] for k in ('calls', 'steps')}, errors


def report(config, arm, rnd, audio_s, wall, lat, st, identical, errors, name):
    lat = np.array(lat) * 1e3
    res = {'config': config, 'arm': arm, 'round': rnd, 'audio_s_per_s': round(audio_s / wall, 1),
           'call_ms_p50': round(float(np.median(lat)), 3), 'call_ms_p99': round(float(np.percentile(lat, 99)), 3),
           'calls': st['calls'], 'steps': st['steps'], 'calls_per_step': round(st['calls'] / max(st['steps'], 1), 2),
           'identical': identical and not errors, 'card': name}
    if errors:
        res['errors'] = errors[:3]
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--encoded-threads', default='1,4,16,64')
    ap.add_argument('--encoded-calls', type=int, default=64)
    ap.add_argument('--stream-threads', default='1,16,128')
    ap.add_argument('--blocks-ms', default='20,100')
    ap.add_argument('--stream-seconds', type=float, default=30.0)
    ap.add_argument('--rounds', type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_session_threads.py needs a CUDA device')
    from some_b200 import export, synth, session as nsess
    name = card()
    print(f'# card: {name}', flush=True)
    rate = 44100
    with tempfile.TemporaryDirectory() as d:
        sess = nsess.Session(export.export(synth.write_checkpoint(d, synth.named_config('two_head'), seed=1234)), 0)
        # ---- encoded files: one 3-minute file per call
        files = [wav16(synth.synth_waveform(9100 + i, seconds=180.0, sr=rate, silence_gaps=True) * np.float32(0.8), rate)
                 for i in range(8)]
        want = [key(sess.transcribe_encoded([f])[0]) for f in files]
        k = args.encoded_calls
        for n in [int(v) for v in args.encoded_threads.split(',')]:
            for rnd in range(args.rounds):
                for arm in ('locked', 'free'):
                    ok = [True]

                    def work(t, call):
                        for c in range(t, k, n):
                            if key(call(lambda c=c: sess.transcribe_encoded([files[c % len(files)]]))[0]) != want[c % len(files)]:
                                ok[0] = False
                    wall, lat, st, errors = run_arm(sess, n, work, arm == 'locked')
                    report(f'encoded 3 min x{k} calls, {n} threads', arm, rnd, 180.0 * k, wall, lat, st, ok[0], errors, name)
        # ---- PCM streams: one per thread, fixed blocks
        pool = [synth.synth_waveform(7000 + i, seconds=args.stream_seconds, sr=rate, silence_gaps=True) for i in range(8)]
        want_s = [key(sess.transcribe_sliced(w, rate)) for w in pool]
        for block_ms in [int(v) for v in args.blocks_ms.split(',')]:
            block = rate * block_ms // 1000
            for n in [int(v) for v in args.stream_threads.split(',')]:
                for rnd in range(args.rounds):
                    for arm in ('locked', 'free'):
                        ok = [True]

                        def work(t, call):
                            w = pool[t % len(pool)]
                            ranges, notes = [], []
                            with sess.stream(rate) as st:
                                for a in range(0, w.shape[0], block):
                                    r = call(lambda a=a: st.push(w[a:a + block]))
                                    ranges += r[1]
                                    notes += key(r)[1]
                                r = call(st.finish)
                                ranges += r[1]
                                notes += key(r)[1]
                            if (ranges, notes) != want_s[t % len(pool)]:
                                ok[0] = False
                        wall, lat, st, errors = run_arm(sess, n, work, arm == 'locked')
                        report(f'stream {block_ms} ms, {n} threads', arm, rnd, args.stream_seconds * n, wall, lat, st, ok[0],
                               errors, name)
        sess.close()


if __name__ == '__main__':
    main()

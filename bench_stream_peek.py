"""Measures provisional notes on live streams (some_stream_peek_many): S PCM streams of synthetic singing at 44.1 kHz push 20 ms
blocks through Session.push_many, and every P ms of audio one Session.peek_many call transcribes the open region of every
stream.  Two arms per (S, P), run alternately in one process:

- plain: the push_many ticks alone.
- peek: the same ticks with a peek_many call on all streams after every P ms of audio.

Reports, per arm, the push_many tick's wall time (median and p99); for the peek arm also the peek_many call's wall time
(median and p99; the call ends in a synchronise), the mean open-region length in seconds over every stream peeked, and the
audio-seconds peeked per wall-second spent in peek_many.  Both arms check that every stream's chunks equal
some_session_transcribe_sliced on its recording.

    python bench_stream_peek.py [--streams 16,128] [--peek-ms 100,250,500] [--seconds 30] [--block-ms 20] [--rounds 1]

Prints the card's name and power limit, then one JSON line per (S, P, arm, round)."""
import argparse
import json
import subprocess
import sys
import tempfile
import time

import numpy as np

SR = 44100


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                 # noqa: BLE001
        return f'unknown ({e})'


def ms_stats(xs):
    a = np.array(xs) * 1e3
    return (round(float(np.median(a)), 3), round(float(np.percentile(a, 99)), 3)) if a.size else (None, None)


def run_arm(sess, pool, want, n, block, peek_every, args):
    """One pass of n streams over their recordings; peek_every: blocks between peek_many calls (0: none)."""
    waves = [pool[i % len(pool)] for i in range(n)]
    streams = [sess.stream(SR) for _ in range(n)]
    got = [[] for _ in range(n)]
    pos, live = [0] * n, list(range(n))
    ticks, peeks, region_s = [], [], []
    k = 0
    t = time.perf_counter()
    try:
        while live:
            items, fin = [], []
            for i in live:
                part = waves[i][pos[i]:pos[i] + block]
                pos[i] += part.shape[0]
                items.append((streams[i], part))
                fin.append(pos[i] >= waves[i].shape[0])
            t0 = time.perf_counter()
            res = sess.push_many(items, fin)
            ticks.append(time.perf_counter() - t0)
            for i, r in zip(live, res):
                got[i] += r[1]
            live = [i for i, f in zip(live, fin) if not f]
            k += 1
            if peek_every and live and k % peek_every == 0:
                t0 = time.perf_counter()
                res = sess.peek_many([streams[i] for i in live])
                peeks.append(time.perf_counter() - t0)
                region_s += [(b - a) / SR for r in res for a, b in r[1]]
    finally:
        wall = time.perf_counter() - t
        for st in streams:
            st.close()
    tick = ms_stats(ticks)
    out = {'streams': n, 'peek_ms': peek_every * args.block_ms if peek_every else None,
           'arm': 'peek' if peek_every else 'plain', 'seconds': args.seconds, 'block_ms': args.block_ms,
           'wall_s': round(wall, 3), 'ticks': len(ticks), 'tick_ms_median': tick[0], 'tick_ms_p99': tick[1],
           'identical': all(got[i] == want[i % len(pool)][1] for i in range(n))}
    if peek_every:
        pk = ms_stats(peeks)
        out.update(peeks=len(peeks), peek_ms_median=pk[0], peek_ms_p99=pk[1],
                   region_s_mean=round(float(np.mean(region_s)), 3) if region_s else None,
                   peeked_audio_s_per_s=round(sum(region_s) / sum(peeks), 1) if peeks else None)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', default='16,128')
    ap.add_argument('--peek-ms', default='100,250,500')
    ap.add_argument('--seconds', type=float, default=30.0)
    ap.add_argument('--block-ms', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_stream_peek.py needs a CUDA device')
    from some_b200 import export, synth, session as nsess
    print(f'# card: {card()}', flush=True)
    block = SR * args.block_ms // 1000
    with tempfile.TemporaryDirectory() as d:
        sess = nsess.Session(export.export(synth.write_checkpoint(d, synth.named_config('two_head'), seed=1234)), 0)
        pool = [synth.synth_waveform(7000 + i, seconds=args.seconds, sr=SR, silence_gaps=True) for i in range(8)]
        want = [sess.transcribe_sliced(w, SR) for w in pool]
        run_arm(sess, pool, want, 4, block, 5, args)                        # warm-up: pushes and peeks
        for n in [int(v) for v in args.streams.split(',')]:
            for p in [int(v) for v in args.peek_ms.split(',')]:
                every = max(1, p // args.block_ms)
                for r in range(args.rounds):
                    for arm_every in (0, every):                            # the arms alternate
                        res = run_arm(sess, pool, want, n, block, arm_every, args)
                        res.update(round=r, peek_ms=p)
                        print(json.dumps(res), flush=True)
        sess.close()


if __name__ == '__main__':
    main()

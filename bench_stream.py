"""Measures streaming transcription (some_stream_*) of N streams on one session, every stream pushing a synthetic recording
with silence gaps in fixed-size blocks as fast as it can, in two arms run alternately in one process:

- threaded: one thread per stream, each calling Stream.push.  Reports the aggregate audio-seconds per second, the wall time
  of a push (median and p99, split into pushes that delivered a chunk and pushes that did not), and the CUDA-event time of the
  windowed front-end kernels for a push of one block (the launches such a push makes, replayed on their own outside the
  streams at a fixed position 1 s into the recording, 200 times back to back: not timed inside the pushes).
- push_many: one thread; per tick one Session.push_many call with one block for every stream that still has samples, and
  finish at each stream's end.  Reports the aggregate audio-seconds per second, the tick wall time (median and p99) and the
  chunks per forward batch (ticks that delivered chunks).

Both arms check that every stream's chunks equal some_session_transcribe_sliced on the same recording, which is also timed
as the one-shot reference.

    python bench_stream.py [--streams 1,16,128,1024] [--blocks-ms 20,100] [--seconds 300] [--rate 44100]
                           [--arms threaded,push_many] [--threaded-max 128]

The threaded arm is skipped above --threaded-max streams: its pushes serialise on the session, so 1024 threads take about
eight times as long as 128 for the same total rate.  Prints the card's name and power limit beside the numbers, and one JSON
line per configuration and arm."""
import argparse
import ctypes as C
import json
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


def kernel_times(rate, block, sr=44100, reps=200):
    """CUDA-event time of the windowed launches a push of `block` samples makes (resampling when rate != sr, then the RMS
    frames those samples complete), replayed on their own at a fixed position: a stand-in, not a time taken inside a push."""
    import torch
    from some_b200 import _lib, audio, slicer
    lib = _lib.load()
    f = slicer.slicer_frames(sr)
    x = torch.randn(rate * 4, device='cuda') * 0.1
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = torch.empty(sr * 4, device='cuda')
    rms = torch.empty(4096, device='cuda')
    table = audio._device_table(rate, sr, 'cuda') if rate != sr else None
    t_end, x_first = C.c_longlong(), C.c_longlong()
    received = rate * 2
    t0 = sr * 1                                            # outputs fixed so far
    if table is not None:
        _lib.check(lib.some_resample_window_plan(received, 0, t0, rate, sr, int(table.numel()), C.byref(t_end), C.byref(x_first)))
    n_out = (t_end.value - t0) if table is not None else block
    f0 = (t0 - f.win_size) // f.hop_size
    nf = max(1, n_out // f.hop_size)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def launch():
        if table is not None:
            _lib.check(lib.some_resample_kaiser_window(x.data_ptr(), 0, received, 0, out.data_ptr(), 0, t0, t_end.value, rate,
                                                       sr, table.data_ptr(), int(table.numel()), stream))
        _lib.check(lib.some_slicer_rms_window(out.data_ptr(), 0, sr * 4, -1, f.win_size, f.hop_size, rms.data_ptr(), f0,
                                              f0 + nf, stream))
    for _ in range(10):
        launch()
    ev[0].record()
    for _ in range(reps):
        launch()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def threaded_arm(sess, pool, want, n, block, block_ms, args, kern):
    times = [[] for _ in range(n)]
    errors, mismatches = [], []

    def work(i):
        w = pool[i % len(pool)]
        got = []
        try:
            with sess.stream(args.rate) as st:
                for a in range(0, w.shape[0], block):
                    t0 = time.perf_counter()
                    o, r, nt = st.push(w[a:a + block])
                    times[i].append((time.perf_counter() - t0, bool(r)))
                    got += r
                got += st.finish()[1]
            if got != want[i % len(pool)][1]:
                mismatches.append(i)
        except Exception as e:         # noqa: BLE001
            errors.append(repr(e))

    threads = [threading.Thread(target=work, args=(i,)) for i in range(n)]
    t = time.perf_counter()
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    wall = time.perf_counter() - t
    flat = [x for ts in times for x in ts]
    dl = np.array([x for x, d in flat if d]) * 1e3
    nd = np.array([x for x, d in flat if not d]) * 1e3
    res = {'config': f'stream x{n}', 'arm': 'threaded', 'block_ms': block_ms, 'seconds': args.seconds,
           'audio_s_per_s': round(n * args.seconds / wall, 1), 'pushes': len(flat),
           'push_ms_no_chunk_median': round(float(np.median(nd)), 3) if nd.size else None,
           'push_ms_no_chunk_p99': round(float(np.percentile(nd, 99)), 3) if nd.size else None,
           'push_ms_chunk_median': round(float(np.median(dl)), 3) if dl.size else None,
           'push_ms_chunk_p99': round(float(np.percentile(dl, 99)), 3) if dl.size else None,
           'window_kernels_ms_replayed_push': round(kern, 4), 'identical': not mismatches and not errors}
    if errors:
        res['errors'] = errors[:3]
    return res


def push_many_arm(sess, pool, want, n, block, block_ms, args):
    waves = [pool[i % len(pool)] for i in range(n)]
    streams = [sess.stream(args.rate) for _ in range(n)]
    got = [[] for _ in range(n)]
    pos, live = [0] * n, list(range(n))
    ticks, batches, errors = [], [], []
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
            chunks = sum(len(r[1]) for r in res)
            if chunks:
                batches.append(chunks)
            for i, r in zip(live, res):
                got[i] += r[1]
            live = [i for i, f in zip(live, fin) if not f]
    except Exception as e:             # noqa: BLE001
        errors.append(repr(e))
    wall = time.perf_counter() - t
    for st in streams:
        st.close()
    tk = np.array(ticks) * 1e3
    res = {'config': f'stream x{n}', 'arm': 'push_many', 'block_ms': block_ms, 'seconds': args.seconds,
           'audio_s_per_s': round(n * args.seconds / wall, 1), 'ticks': len(ticks),
           'tick_ms_median': round(float(np.median(tk)), 3) if tk.size else None,
           'tick_ms_p99': round(float(np.percentile(tk, 99)), 3) if tk.size else None,
           'chunks_per_batch_mean': round(float(np.mean(batches)), 2) if batches else None,
           'chunks_per_batch_max': int(max(batches)) if batches else None,
           'identical': not errors and all(got[i] == want[i % len(pool)][1] for i in range(n))}
    if errors:
        res['errors'] = errors[:3]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', default='1,16,128,1024')
    ap.add_argument('--blocks-ms', default='20,100')
    ap.add_argument('--seconds', type=float, default=300.0)
    ap.add_argument('--rate', type=int, default=44100)
    ap.add_argument('--arms', default='threaded,push_many')
    ap.add_argument('--threaded-max', type=int, default=128)
    args = ap.parse_args()
    arms = args.arms.split(',')
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_stream.py needs a CUDA device')
    from some_b200 import export, synth, session as nsess
    print(f'# card: {card()}', flush=True)
    counts = [int(v) for v in args.streams.split(',')]
    with tempfile.TemporaryDirectory() as d:
        sess = nsess.Session(export.export(synth.write_checkpoint(d, synth.named_config('two_head'), seed=1234)), 0)
        pool = [synth.synth_waveform(7000 + i, seconds=args.seconds, sr=args.rate, silence_gaps=True) for i in range(8)]
        sess.transcribe_sliced(pool[0], args.rate)                         # warm-up
        t = time.perf_counter()
        want = [sess.transcribe_sliced(w, args.rate) for w in pool]
        one_shot = time.perf_counter() - t
        print(json.dumps({'config': 'transcribe_sliced', 'recordings': len(pool), 'seconds': args.seconds,
                          'audio_s_per_s': round(len(pool) * args.seconds / one_shot, 1),
                          'ms_per_recording': round(1e3 * one_shot / len(pool), 2)}), flush=True)
        for block_ms in [int(v) for v in args.blocks_ms.split(',')]:
            block = args.rate * block_ms // 1000
            kern = kernel_times(args.rate, block)
            for n in counts:
                if 'threaded' in arms and n <= args.threaded_max:
                    print(json.dumps(threaded_arm(sess, pool, want, n, block, block_ms, args, kern)), flush=True)
                if 'push_many' in arms:
                    print(json.dumps(push_many_arm(sess, pool, want, n, block, block_ms, args)), flush=True)
        sess.close()


if __name__ == '__main__':
    main()

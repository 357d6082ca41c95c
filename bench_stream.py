"""Measures streaming transcription (some_stream_*): N concurrent streams on one session, one thread each, every stream
pushing a synthetic recording with silence gaps in fixed-size blocks as fast as it can.  Reports the aggregate audio-seconds
per second, the wall time of a push (median and p99, split into pushes that delivered a chunk and pushes that did not), the
CUDA-event time of the windowed front-end kernels for a push of one block (the launches such a push makes, replayed on their
own outside the streams at a fixed position 1 s into the recording, 200 times back to back: not timed inside the pushes), and
some_session_transcribe_sliced on the same recordings as the one-shot reference.  Checks that every stream's chunks equal the one-shot result.

    python bench_stream.py [--streams 1,16,128] [--blocks-ms 20,100] [--seconds 300] [--rate 44100]

Prints the card's name and power limit beside the numbers, and one JSON line per configuration."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', default='1,16,128')
    ap.add_argument('--blocks-ms', default='20,100')
    ap.add_argument('--seconds', type=float, default=300.0)
    ap.add_argument('--rate', type=int, default=44100)
    args = ap.parse_args()
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
                res = {'config': f'stream x{n}', 'block_ms': block_ms, 'seconds': args.seconds,
                       'audio_s_per_s': round(n * args.seconds / wall, 1), 'pushes': len(flat),
                       'push_ms_no_chunk_median': round(float(np.median(nd)), 3) if nd.size else None,
                       'push_ms_no_chunk_p99': round(float(np.percentile(nd, 99)), 3) if nd.size else None,
                       'push_ms_chunk_median': round(float(np.median(dl)), 3) if dl.size else None,
                       'push_ms_chunk_p99': round(float(np.percentile(dl, 99)), 3) if dl.size else None,
                       'window_kernels_ms_replayed_push': round(kern, 4), 'identical': not mismatches and not errors}
                if errors:
                    res['errors'] = errors[:3]
                print(json.dumps(res), flush=True)
        sess.close()


if __name__ == '__main__':
    main()

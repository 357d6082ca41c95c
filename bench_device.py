"""Measures transcribing audio that is already on the GPU: 64 stereo planar 30 s stems (float32 CUDA tensors [2, n], the
shape a vocal-separation model leaves; half at 44.1 kHz, half at 48 kHz), two arms alternated over several rounds in one
process:

- host: what a caller had to do before Session.transcribe_device: each stem's ``.cpu()``, ``np.mean(axis=0)`` (librosa.to_mono)
  and Session.transcribe_sliced, one call per stem from T threads, so that queued calls share session steps;
- device: one Session.transcribe_device call with the 64 tensors.

Reports the wall time of the 64 stems per arm and round (the stems are written and synchronised before the clock starts),
the host-to-device and device-to-host bytes of one round of each arm from a torch.profiler trace, and the time of one
some_downmix launch over the 64 stems (CUDA events around repeated launches) with its rate in GB/s and its share of the
H100 SXM's 3.35 TB/s: it reads every channel once and writes the mono samples once.  Asserts that both arms give
bit-identical notes.  Prints the card's name and power limit beside the numbers, one JSON line per arm and round, and a
summary line.

    python bench_device.py [--stems 64] [--seconds 30] [--rounds 3] [--threads 16] [--trace-dir DIR]"""
import argparse
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


def key(res):
    """One recording's result as comparable values: ranges and the bits of every note."""
    _, ranges, notes = res
    return ranges, [(n['note_midi'].view(np.uint32).tobytes(), n['note_frames'].tobytes(), n['note_rest'].tobytes())
                    for n in notes]


def host_arm(sess, stems, rates, n_threads):
    """Every stem down-mixed on the host and transcribed by transcribe_sliced, from n_threads threads."""
    out, errors = [None] * len(stems), []

    def body(t):
        try:
            for i in range(t, len(stems), n_threads):
                m = np.mean(stems[i].cpu().numpy(), axis=0)
                out[i] = sess.transcribe_sliced(m, rates[i])
        except Exception as e:             # noqa: BLE001
            errors.append(repr(e))
    threads = [threading.Thread(target=body, args=(t,)) for t in range(n_threads)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    return out


def device_arm(sess, stems, rates):
    return sess.transcribe_device(stems, rates)


def traced_bytes(fn, trace_path):
    """Runs fn under torch.profiler with CUDA activities; returns the host-to-device and device-to-host bytes of the trace
    and its some_downmix kernel time in ms."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace_path)
    with open(trace_path) as f:
        events = json.load(f)['traceEvents']
    h2d = d2h = 0
    dm_us = 0.0
    for e in events:
        name, args = e.get('name', ''), e.get('args', {}) or {}
        if e.get('cat') in ('gpu_memcpy', 'Memcpy') or name.startswith('Memcpy'):
            b = int(args.get('bytes', 0))
            if 'HtoD' in name:
                h2d += b
            elif 'DtoH' in name:
                d2h += b
        if e.get('cat') == 'kernel' and 'downmix_kernel' in name:
            dm_us += float(e.get('dur', 0.0))
    return h2d, d2h, dm_us / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--stems', type=int, default=64)
    ap.add_argument('--seconds', type=float, default=30.0)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--threads', type=int, default=16)
    ap.add_argument('--trace-dir', default=None, help='where the profiler traces go (default: a temporary directory)')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_device.py needs a CUDA device')
    from some_b200 import audio, export, synth, session as nsess
    name = card()
    print(f'# card: {name}', flush=True)
    dev = torch.device('cuda:0')
    rates = [(44100, 48000)[i % 2] for i in range(args.stems)]
    rng = np.random.default_rng(0)
    base = {r: [synth.synth_waveform(8000 + 10 * k + r % 7, seconds=args.seconds, sr=r, silence_gaps=True) for k in range(4)]
            for r in (44100, 48000)}
    stems = []
    for i, r in enumerate(rates):
        x = np.roll(base[r][(i // 2) % 4], 4099 * (i // 8))
        g = rng.uniform(0.4, 1.1, (2, 1)).astype(np.float32)
        stems.append(torch.from_numpy((g * x[None]).astype(np.float32)).to(dev))      # planar [2, n]
    torch.cuda.synchronize()
    audio_s = sum(s.shape[1] / r for s, r in zip(stems, rates))
    with tempfile.TemporaryDirectory() as d:
        sess = nsess.Session(export.export(synth.write_checkpoint(d, synth.named_config('two_head'), seed=1234)), 0)
        try:
            want = [key(r) for r in host_arm(sess, stems, rates, args.threads)]             # warm-up of both arms
            assert [key(r) for r in device_arm(sess, stems, rates)] == want, 'the arms disagree'
            walls = {'host': [], 'device': []}
            for rnd in range(args.rounds):
                for arm in ('host', 'device'):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    res = host_arm(sess, stems, rates, args.threads) if arm == 'host' else device_arm(sess, stems, rates)
                    wall = time.perf_counter() - t0
                    identical = [key(r) for r in res] == want
                    assert identical, f'{arm} round {rnd}: notes differ'
                    walls[arm].append(wall)
                    print(json.dumps({'arm': arm, 'round': rnd, 'stems': args.stems, 'wall_s': round(wall, 4),
                                      'audio_s_per_s': round(audio_s / wall, 1), 'identical': identical, 'card': name}),
                          flush=True)
            # bytes over the bus, from one traced round of each arm
            tdir = args.trace_dir or d
            h_h2d, h_d2h, _ = traced_bytes(lambda: host_arm(sess, stems, rates, args.threads), f'{tdir}/host_trace.json')
            d_h2d, d_d2h, dm_trace_ms = traced_bytes(lambda: device_arm(sess, stems, rates), f'{tdir}/device_trace.json')
            # the down-mix alone: one launch over every stem, repeated between CUDA events
            total = sum(s.shape[1] for s in stems)
            out = torch.empty(total, device=dev)
            starts = np.concatenate([[0], np.cumsum([s.shape[1] for s in stems])])
            items = [(s, out, int(a)) for s, a in zip(stems, starts)]
            for _ in range(3):
                audio.downmix_into(items)
            reps = 50
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                audio.downmix_into(items)
            e1.record()
            torch.cuda.synchronize()
            launch_ms = e0.elapsed_time(e1) / reps            # includes the descriptors' upload of each call
            moved = sum(4 * (s.shape[0] + 1) * s.shape[1] for s in stems)
            kernel_ms = dm_trace_ms if dm_trace_ms > 0 else launch_ms
            print(json.dumps({
                'summary': True, 'stems': args.stems, 'seconds': args.seconds, 'threads': args.threads, 'rounds': args.rounds,
                'host_wall_s_median': round(float(np.median(walls['host'])), 4),
                'device_wall_s_median': round(float(np.median(walls['device'])), 4),
                'host_h2d_bytes': h_h2d, 'host_d2h_bytes': h_d2h, 'device_h2d_bytes': d_h2d, 'device_d2h_bytes': d_d2h,
                'downmix_bytes': moved, 'downmix_kernel_ms_trace': round(dm_trace_ms, 4),
                'downmix_call_ms_events': round(launch_ms, 4),
                'downmix_GBps': round(moved / kernel_ms / 1e6, 1), 'downmix_share_of_3_35_TBps': round(moved / kernel_ms / 1e6 / 3350, 3),
                'identical': True, 'card': name}), flush=True)
        finally:
            sess.close()


if __name__ == '__main__':
    main()

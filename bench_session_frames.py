"""Measures what the frame curves (some_notes_set_frames) cost the native session.  Three arms, run alternately in one process:

- off: the calls as they were, frames=False;
- on:  the same calls with frames=True (the curves of every clip / chunk come down with the notes);
- native: frames on in the native result, but the wrapper does not copy the curves out into numpy (Notes.curves skipped):
  the native cost alone, without the Python copy-out.

Workloads (a two_head model exported from a synth checkpoint):
- batch:   64 clips of 30 s through Session.transcribe (some_session_transcribe);
- sliced:  one 5-minute recording through Session.transcribe_sliced;
- streams: S PCM streams at 44.1 kHz with 10 s pushed; one tick = push_many of 20 ms to every stream, then peek_many of all
           of them (S = 16 and 128).

Per workload and arm: the wall time per call (median and spread over the rounds; each call ends in a synchronise), the bytes
the call copies device-to-host (from a torch.profiler trace of one call, taken outside the timed rounds) and the frames the
call transcribes.  The arms check that their notes are bit-identical.

    python bench_session_frames.py [--rounds 5] [--arms off,on,native] [--streams 16,128]

`--arms off` runs only the frames-off arm, which a tree without frame curves can also run, to compare two builds.  Prints
the card's name, power limit and SM clock, then one JSON line per (workload, arm)."""
import argparse
import json
import pathlib
import subprocess
import sys
import tempfile
import time

import numpy as np

SR, HOP = 44100, 512


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                 # noqa: BLE001
        return f'unknown ({e})'


def download_bytes(fn):
    """(bytes, copies) device-to-host in fn(), from a torch.profiler trace."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = pathlib.Path(d) / 'trace.json'
        prof.export_chrome_trace(str(path))
        events = json.loads(path.read_text())['traceEvents']
    copies = [e for e in events if e.get('cat') == 'gpu_memcpy' and 'DtoH' in e.get('name', '')]
    return sum(int(e['args'].get('bytes', 0)) for e in copies), len(copies)


def notes_key(res):
    """The notes of a result, as bytes, to compare the arms."""
    out = []
    for n in res:
        out += [n['note_midi'].tobytes(), n['note_frames'].tobytes(), n['note_rest'].tobytes()]
    return b''.join(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--arms', default='off,on,native')
    ap.add_argument('--streams', default='16,128')
    args = ap.parse_args()
    sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent))
    from some_b200 import export, synth
    from some_b200 import session as nsess
    arms = args.arms.split(',')
    print(json.dumps({'card': card(), 'tree': str(pathlib.Path(__file__).resolve().parent)}), flush=True)
    with tempfile.TemporaryDirectory() as d:
        sess = nsess.Session(export.export(synth.write_checkpoint(d, synth.named_config('two_head'), seed=1234)), 0)
        pool = [synth.synth_waveform(1000 + j, seconds=30.0) for j in range(4)]
        clips = [np.ascontiguousarray(np.roll(pool[i % 4], 4099 * (i // 4))) for i in range(64)]
        rec = synth.synth_waveform(9002, seconds=300.0, silence_gaps=True)
        kw = lambda arm: {} if arm == 'off' else {'frames': True}
        copy_out = getattr(nsess.Notes, 'curves', None)     # None in a tree without frame curves (--arms off)

        def batch(arm):
            r = sess.transcribe(clips, **kw(arm))
            return r if arm == 'off' else r[0]

        def sliced(arm):
            return sess.transcribe_sliced(rec, **kw(arm))[2]

        workloads = [('batch_64x30s', batch, sum(1 + c.shape[0] // HOP for c in clips)),
                     ('sliced_300s', sliced, None)]
        for n in [int(v) for v in args.streams.split(',') if v]:
            streams = [sess.stream(SR) for _ in range(n)]
            waves = [synth.synth_waveform(5000 + i, seconds=60.0, silence_gaps=True) for i in range(n)]
            sess.push_many([(st, w[:10 * SR]) for st, w in zip(streams, waves)])
            state = {'pos': 10 * SR}

            def tick(arm, streams=streams, waves=waves, state=state):
                a = state['pos']
                state['pos'] = a + SR // 50 if a + SR // 50 < 55 * SR else 10 * SR + SR // 50
                sess.push_many([(st, w[a:a + SR // 50]) for st, w in zip(streams, waves)], **kw(arm))
                return [x for r in sess.peek_many(streams, **kw(arm)) for x in r[2]]
            workloads.append((f'streams_{n}_tick', tick, None))

        for name, fn, frames in workloads:
            for arm in arms:                                 # warm-up: every shape and buffer of every arm
                fn(arm)
            times = {arm: [] for arm in arms}
            keys = {}
            for _ in range(args.rounds):
                for arm in arms:
                    if arm == 'native':
                        nsess.Notes.curves = lambda self: []
                    t0 = time.perf_counter()
                    res = fn(arm)
                    times[arm].append(time.perf_counter() - t0)
                    if arm == 'native':
                        nsess.Notes.curves = copy_out
                    if not name.startswith('streams'):
                        keys.setdefault(arm, notes_key(res))
            copied = {arm: download_bytes(lambda: fn(arm)) for arm in arms}
            for arm in arms:
                t = np.array(times[arm]) * 1e3
                line = {'workload': name, 'arm': arm, 'rounds': args.rounds, 'ms_median': round(float(np.median(t)), 3),
                        'ms_min': round(float(t.min()), 3), 'ms_max': round(float(t.max()), 3),
                        'dtoh_bytes': copied[arm][0], 'dtoh_copies': copied[arm][1]}
                if frames:
                    line['frames'] = frames
                if 'off' in keys and len(keys) > 1:
                    line['notes_identical'] = keys[arm] == keys['off']
                print(json.dumps(line), flush=True)
        sess.close()


if __name__ == '__main__':
    main()

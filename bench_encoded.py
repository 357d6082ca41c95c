"""Times WAV and FLAC files through the native session (some_session_transcribe_encoded) against the per-file and Python paths.

Input: N seeded recordings of S seconds held in memory (default 64 x 180 s). Half are FLAC, stereo 48 kHz 24-bit; the other
half are WAV, s16 stereo 44.1 kHz. The model is seeded and random (two_head); its rate is 44.1 kHz, so every FLAC file is
resampled.

Arms, alternated over --rounds rounds:
  encoded_k       some_session_transcribe_encoded over all files, k items per call (k = 1, 16, 64): file bytes in, notes out
  sliced_per_file some_session_transcribe_sliced once per file, on samples decoded on the host beforehand (audio.load(sr=None),
                  not timed: this arm is charged for the upload, resampling, slicer and model only)
  python          batch.transcribe_recordings(plugin, ...) in batches of --py-batch files, with FLAC read by audio.read_encoded
                  and WAV by audio.load_native (timed, from files in a temporary directory)
Every arm's chunk offsets and notes are compared with the sliced_per_file arm's, bit for bit.

A separate run traces one call of --profile-k items with torch.profiler (CUDA activities). It splits the device time into
upload (host-to-device copies), FLAC scan, decode (the FLAC decode and emit kernels, some_pcm_decode), resample + RMS, and
forward (mel, trunk, decode of notes). Tracing slows the host, so these numbers are not used for the rates.

    python bench_encoded.py [--files 64] [--seconds 180] [--rounds 2] [--py-batch 16] [--profile-k 16]

Prints the card's name and power limit with the numbers, then one JSON line. Nothing is written to the repository: the files
and the model go to a temporary directory.
"""
import argparse
import ctypes as C
import json
import multiprocessing as mp
import os
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REPO)


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:              # noqa: BLE001
        return f'nvidia-smi unavailable ({e!r})'


def wav_s16(x: np.ndarray, rate: int) -> bytes:
    v = np.clip(np.round(x * 32768), -32768, 32767).astype('<i2')
    n, ch = v.shape
    raw = v.tobytes()
    fmt = struct.pack('<HHIIHH', 1, ch, rate, rate * ch * 2, ch * 2, 16)
    body = b'WAVE' + b'fmt ' + struct.pack('<I', 16) + fmt + b'data' + struct.pack('<I', len(raw)) + raw
    return b'RIFF' + struct.pack('<I', len(body)) + body


def make_file(args):
    """File i: FLAC for even i, WAV for odd i; two seeded synthetic voices as the channels, with silences."""
    i, seconds = args
    from oracle import flac as of
    from some_b200 import synth
    rate = 48000 if i % 2 == 0 else 44100
    x = np.stack([synth.synth_waveform(7000 + 2 * i + c, seconds=seconds, sr=rate, silence_gaps=True) for c in range(2)], 1)
    x = x * np.float32(0.9)
    if i % 2 == 0:
        v = np.clip(np.round(x * 2 ** 23), -2 ** 23, 2 ** 23 - 1).astype(np.int64)
        return 'flac', of.encode(v, rate=rate, bps=24, subframe={'type': 'fixed', 'order': 2, 'porder': 4, 'method': 1})
    return 'wav', wav_s16(x, rate)


def same(a, b):
    """(offsets, notes) pairs equal bit for bit."""
    (oa, na), (ob, nb) = a, b
    return list(oa) == list(ob) and len(na) == len(nb) and all(
        np.array_equal(np.asarray(x['note_midi'], np.float32).view(np.uint32), np.asarray(y['note_midi'], np.float32).view(np.uint32))
        and np.array_equal(np.asarray(x['note_dur'], np.float64).view(np.uint64), np.asarray(y['note_dur'], np.float64).view(np.uint64))
        and np.array_equal(np.asarray(x['note_rest'], bool), np.asarray(y['note_rest'], bool)) for x, y in zip(na, nb))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--files', type=int, default=64)
    ap.add_argument('--seconds', type=float, default=180.0)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--ks', default='1,16,64')
    ap.add_argument('--py-batch', type=int, default=16)
    ap.add_argument('--profile-k', type=int, default=16)
    ap.add_argument('--config', default='two_head')
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_encoded.py measures on a CUDA device; none is available')
    from some_b200 import _lib, audio, batch, export, plugin, synth
    from some_b200 import session as nsess

    t0 = time.perf_counter()
    with mp.Pool(min(len(os.sched_getaffinity(0)), 32)) as pool:
        files = pool.map(make_file, [(i, a.seconds) for i in range(a.files)])
    gen_s = time.perf_counter() - t0
    audio_s = a.files * a.seconds
    ks = [k for k in (int(x) for x in a.ks.split(',')) if k <= a.files]
    print(f'card: {card()}', flush=True)
    print(f'{a.files} files ({sum(len(d) for _, d in files) / 1e6:.0f} MB, {audio_s:.0f} audio-s) made in {gen_s:.1f} s',
          flush=True)

    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for i, (kind, data) in enumerate(files):
            p = os.path.join(tmp, f'f{i:03d}.{kind}')
            with open(p, 'wb') as f:
                f.write(data)
            paths.append(p)
        config = synth.named_config(a.config)
        ckpt = synth.write_checkpoint(tmp, config, seed=1234)
        model_path = export.export(ckpt)
        sess = nsess.Session(model_path, 0)
        ins = plugin.MIDIExtractionInference(config=config, model_path=ckpt, device='cuda:0')
        lib = sess.lib

        # encoded: the items' bytes and result objects made once, outside the timed window
        bufs = [C.create_string_buffer(d, len(d)) for _, d in files]
        enc = (_lib.Encoded * a.files)(*[_lib.Encoded(C.cast(b, C.c_void_p), len(d)) for b, (_, d) in zip(bufs, files)])
        notes = [nsess.Notes() for _ in range(a.files)]
        handles = (C.c_void_p * a.files)(*[n.handle for n in notes])
        size = C.sizeof(_lib.Encoded)

        def run_encoded(k, lo=0, hi=None):
            hi = a.files if hi is None else hi
            for s in range(lo, hi, k):
                m = min(k, hi - s)
                e = C.cast(C.addressof(enc) + s * size, C.POINTER(_lib.Encoded))
                o = C.cast(C.addressof(handles) + s * C.sizeof(C.c_void_p), C.c_void_p)
                _lib.check(lib.some_session_transcribe_encoded(sess.handle, e, m, None, o), 'some_session_transcribe_encoded')

        def encoded_results():
            out = []
            for n in notes:
                ranges, res = n.results(sess.timestep)
                out.append(([b / sess.sample_rate for b, _ in ranges], res))
            return out

        decoded = [audio.load(p, sr=None) for p in paths]          # the per-file arm's host decoding, not timed

        def run_sliced():
            return [tuple(sess.transcribe_sliced(y, rate)[i] for i in (0, 2)) for y, rate in decoded]

        def run_python():
            out = []
            for s in range(0, a.files, a.py_batch):
                group = paths[s:s + a.py_batch]
                waves, rates = [], []
                for p in group:
                    if p.endswith('.flac'):
                        waves.append(audio.read_encoded(p))
                        rates.append(None)
                    else:
                        y, rate = audio.load_native(p)
                        waves.append(y)
                        rates.append(rate)
                out += batch.transcribe_recordings(ins, waves, rates=rates)
            return out

        # warm-up: every arm and shape once
        for k in ks:
            run_encoded(k, 0, min(k, a.files))
        sess.transcribe_sliced(*decoded[0])
        sess.transcribe_sliced(*decoded[1])
        batch.transcribe_recordings(ins, [audio.read_encoded(paths[0])], rates=[None])
        torch.cuda.synchronize()

        times = {'sliced_per_file': [], **{f'encoded_{k}': [] for k in ks}, 'python': []}
        equal = {name: True for name in times}
        want = None
        for r in range(a.rounds):
            t = time.perf_counter()
            sl = run_sliced()
            times['sliced_per_file'].append(time.perf_counter() - t)
            want = sl if want is None else want
            equal['sliced_per_file'] &= all(map(same, sl, want))
            for k in ks:
                t = time.perf_counter()
                run_encoded(k)
                times[f'encoded_{k}'].append(time.perf_counter() - t)
                equal[f'encoded_{k}'] &= all(map(same, encoded_results(), want))
            t = time.perf_counter()
            py = run_python()
            torch.cuda.synchronize()
            times['python'].append(time.perf_counter() - t)
            equal['python'] &= all(map(same, py, want))

        arms = {}
        for name, ts in times.items():
            best = min(ts)
            arms[name] = {'audio_s_per_s': round(audio_s / best, 1), 'best_s': round(best, 3),
                          'runs_s': [round(x, 3) for x in ts], 'outputs_equal_sliced_per_file': bool(equal[name])}
            print(f'{name:16s} {audio_s / best:9.1f} audio-s/s   best {best:7.3f} s   runs {[round(x, 3) for x in ts]}   '
                  f'equal {equal[name]}', flush=True)

        # the split of one encoded call's device time, in a traced run of its own
        k = min(a.profile_k, a.files)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            t = time.perf_counter()
            run_encoded(k, 0, k)
            wall = time.perf_counter() - t
        split = {'upload': 0.0, 'flac_scan': 0.0, 'decode': 0.0, 'resample_rms': 0.0, 'forward': 0.0, 'download': 0.0, 'other_copy': 0.0}
        for ev in prof.key_averages():
            us = getattr(ev, 'self_device_time_total', None)
            if us is None:
                us = getattr(ev, 'self_cuda_time_total', 0)
            if not us:
                continue
            n = ev.key
            if 'Memcpy HtoD' in n:
                split['upload'] += us
            elif 'Memcpy DtoH' in n:
                split['download'] += us
            elif 'Memcpy' in n or 'Memset' in n:
                split['other_copy'] += us
            elif any(s in n for s in ('flac_count', 'flac_offsets', 'flac_write', 'flac_parse')):
                split['flac_scan'] += us
            elif 'flac_decode' in n or 'flac_emit' in n or 'pcm_decode' in n:
                split['decode'] += us
            elif 'resample' in n or 'slicer_rms' in n:
                split['resample_rms'] += us
            else:                                             # mel, trunk and note decoding
                split['forward'] += us
        split_ms = {kk: round(v / 1000.0, 2) for kk, v in split.items()}
        print(f'one traced call of {k} items ({k * a.seconds:.0f} audio-s): wall {wall * 1000:.1f} ms, device ms {split_ms}',
              flush=True)
        for n in notes:
            n.close()
        sess.close()

    print(json.dumps({'metric': 'encoded files through the native session', 'unit': 'audio-s/s', 'card': card(),
                      'files': a.files, 'seconds_per_file': a.seconds, 'mix': 'half FLAC stereo 48 kHz 24-bit, half WAV s16 '
                      'stereo 44.1 kHz', 'arms': arms, 'profile': {'items': k, 'wall_ms': round(wall * 1000, 1),
                                                                     'device_ms': split_ms}}))


if __name__ == '__main__':
    main()

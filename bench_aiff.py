"""Times AIFF files through the native session against the same recordings as WAV, and the PCM kernel on each sample layout.

Input: N seeded stereo recordings of S seconds at 44.1 kHz (default 32 x 120 s), each held in memory three ways: 16-bit WAV
(little-endian), 16-bit AIFF (big-endian, SOME_PCM_S16BE) and 24-bit AIFF (SOME_PCM_S24BE).  The WAV and 16-bit AIFF files
hold the same samples; the 24-bit files the same voices at 24 bits.  The model is seeded and random (two_head).

Arms:
  session_<fmt>  some_session_transcribe_encoded over all files of one format, --k items per call, host clock around the
                 calls (each ends in a synchronise); the three formats alternate over --rounds rounds, and the notes of the
                 16-bit WAV and AIFF files are compared bit for bit.
  pcm_<fmt>      some_pcm_decode alone: one launch over every recording's sample bytes, already on the device, to mono
                 float32; CUDA events over --launches launches after a warm-up.  Rate = (bytes read + bytes written) / time,
                 and that rate over the H100 SXM's 3.35 TB/s of HBM3 (the data sheet's figure; the card's own power limit is
                 printed with the numbers).

    python bench_aiff.py [--files 32] [--seconds 120] [--rounds 3] [--k 16] [--launches 50]

Prints the card's name and power limit with the numbers, then one JSON line.  Nothing is written to the repository: the
model goes to a temporary directory.
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
HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:              # noqa: BLE001
        return f'nvidia-smi unavailable ({e!r})'


def make_files(args, rate=44100):
    """Recording i as (16-bit WAV, 16-bit AIFF, 24-bit AIFF) bytes."""
    i, seconds = args
    from oracle import aiff as oa
    from some_b200 import synth
    x = np.stack([synth.synth_waveform(9000 + 2 * i + c, seconds=seconds, sr=rate, silence_gaps=True) for c in range(2)], 1)
    x = x * np.float32(0.9)
    v16 = np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)
    v24 = np.clip(np.round(x * 2 ** 23), -2 ** 23, 2 ** 23 - 1).astype('>i4')
    raw = v16.astype('<i2').tobytes()
    fmt = struct.pack('<HHIIHH', 1, 2, rate, rate * 4, 4, 16)
    body = b'WAVE' + b'fmt ' + struct.pack('<I', 16) + fmt + b'data' + struct.pack('<I', len(raw)) + raw
    wav = b'RIFF' + struct.pack('<I', len(body)) + body
    aiff16 = oa.aiff_bytes(v16.astype('>i2').tobytes(), 2, 16, float(rate))
    aiff24 = oa.aiff_bytes(v24.view(np.uint8).reshape(-1, 4)[:, 1:].tobytes(), 2, 24, float(rate))
    return wav, aiff16, aiff24


def same(a, b):
    """(ranges, notes) equal bit for bit."""
    (ra, na), (rb, nb) = a, b
    return ra == rb and len(na) == len(nb) and all(
        np.array_equal(np.asarray(x['note_midi'], np.float32).view(np.uint32), np.asarray(y['note_midi'], np.float32).view(np.uint32))
        and np.array_equal(np.asarray(x['note_dur'], np.float64).view(np.uint64), np.asarray(y['note_dur'], np.float64).view(np.uint64))
        and np.array_equal(np.asarray(x['note_rest'], bool), np.asarray(y['note_rest'], bool)) for x, y in zip(na, nb))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--files', type=int, default=32)
    ap.add_argument('--seconds', type=float, default=120.0)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--k', type=int, default=16)
    ap.add_argument('--launches', type=int, default=50)
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_aiff.py measures on a CUDA device; none is available')
    from some_b200 import _lib, audio, export, synth
    from some_b200 import session as nsess

    fmts = ('wav16', 'aiff16', 'aiff24')
    with mp.Pool(min(len(os.sched_getaffinity(0)), 32)) as pool:     # the synthesis is slow and not what is measured
        made = pool.map(make_files, [(i, a.seconds) for i in range(a.files)])
    files = {f: [m[j] for m in made] for j, f in enumerate(fmts)}
    audio_s = a.files * a.seconds
    print(f'card: {card()}', flush=True)
    print(f'{a.files} recordings x {a.seconds:.0f} s, stereo 44.1 kHz: ' +
          ', '.join(f'{f} {sum(map(len, files[f])) / 1e6:.0f} MB' for f in fmts), flush=True)

    with tempfile.TemporaryDirectory() as tmp:
        config = synth.named_config('two_head')
        sess = nsess.Session(export.export(synth.write_checkpoint(tmp, config, seed=1234)), 0)
        lib = sess.lib

        def run_session(f):
            out = []
            for s in range(0, a.files, a.k):
                out += [r[1:] for r in sess.transcribe_encoded(files[f][s:s + a.k])]
            return out

        for f in fmts:                                    # warm-up
            sess.transcribe_encoded(files[f][:min(a.k, a.files)])
        times = {f: [] for f in fmts}
        results = {}
        for _ in range(a.rounds):
            for f in fmts:
                t = time.perf_counter()
                results[f] = run_session(f)
                times[f].append(time.perf_counter() - t)
        aiff_equals_wav = all(map(same, results['aiff16'], results['wav16']))

        # the kernel alone, over device-resident bytes
        stream = torch.cuda.current_stream()
        kernel = {}
        for f in fmts:
            metas = [audio.audio_info(d) for d in files[f]]
            offs = np.concatenate([[0], np.cumsum([-(-m.data_bytes // 16) * 16 for m in metas])]).astype(np.int64)
            host = np.zeros(int(offs[-1]) + 16, np.uint8)
            for d, m, o in zip(files[f], metas, offs):
                host[o:o + m.data_bytes] = np.frombuffer(d, np.uint8, count=m.data_bytes, offset=m.data_offset)
            src = torch.from_numpy(host).cuda()
            starts = np.concatenate([[0], np.cumsum([m.frames for m in metas])]).astype(np.int64)
            out = torch.empty(int(starts[-1]), dtype=torch.float32, device='cuda')
            items = (_lib.PcmItem * a.files)(*[_lib.PcmItem(src.data_ptr() + int(o), m.frames, m.channels, m.kind, 1, 0,
                                                            out.data_ptr() + 4 * int(s)) for m, o, s in zip(metas, offs, starts)])
            desc = np.zeros(lib.some_pcm_decode_bytes(a.files), np.uint8)
            _lib.check(lib.some_pcm_decode_pack(items, a.files, desc.ctypes.data), 'some_pcm_decode_pack')
            desc_d = torch.from_numpy(desc).cuda()
            launch = lambda: _lib.check(lib.some_pcm_decode(desc.ctypes.data, desc_d.data_ptr(),            # noqa: E731
                                                            C.c_void_p(stream.cuda_stream)), 'some_pcm_decode')
            for _ in range(5):
                launch()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(a.launches):
                launch()
            e1.record(stream)
            e1.synchronize()
            us = e0.elapsed_time(e1) * 1000.0 / a.launches
            moved = sum(m.data_bytes for m in metas) + 4 * int(starts[-1])
            kernel[f] = {'us': round(us, 1), 'bytes': moved, 'GB_per_s': round(moved / us / 1e3, 1),
                         'of_3_35_TB_per_s': round(moved / (us * 1e-6) / HBM_BYTES_PER_S, 3), 'kind': metas[0].kind}
        sess.close()

    arms = {}
    for f in fmts:
        best = min(times[f])
        arms[f'session_{f}'] = {'audio_s_per_s': round(audio_s / best, 1), 'best_s': round(best, 3),
                                'runs_s': [round(x, 3) for x in times[f]]}
        print(f'session_{f:7s} {audio_s / best:9.1f} audio-s/s   best {best:7.3f} s   runs {[round(x, 3) for x in times[f]]}',
              flush=True)
    for f in fmts:
        k = kernel[f]
        print(f'pcm_{f:7s} {k["us"]:9.1f} us per launch   {k["GB_per_s"]:8.1f} GB/s read + written   '
              f'{100 * k["of_3_35_TB_per_s"]:5.1f}% of 3.35 TB/s', flush=True)
    print(f'16-bit AIFF notes equal 16-bit WAV notes: {aiff_equals_wav}', flush=True)
    print(json.dumps({'metric': 'AIFF against WAV through the native session', 'unit': 'audio-s/s', 'card': card(),
                      'files': a.files, 'seconds_per_file': a.seconds, 'k': a.k, 'arms': arms,
                      'pcm_decode': kernel, 'aiff16_equals_wav16': aiff_equals_wav}))


if __name__ == '__main__':
    main()

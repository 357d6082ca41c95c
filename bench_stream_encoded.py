"""Measures encoded streams (some_stream_push_bytes_many): N streams of one session, each pushing a synthetic file's bytes in
fixed-size blocks as fast as it can, against the same audio pushed as samples and against the one-shot call.  Three arms,
alternated in one process for each input kind, block size and stream count:

- push_bytes_many: one Session.push_bytes_many call per tick with one byte block for every stream that still has bytes, and
  finish at each stream's end (blocks worth --blocks-ms of audio at the file's average bytes per second).
- push_many: the same audio decoded on the host beforehand (audio.load(sr=None), not timed), one Session.push_many call per
  tick with blocks of the same duration.
- transcribe_encoded: the same files, 16 per one-shot call.

Inputs: 60 s FLAC (48 kHz stereo 24-bit) and WAV (s16 stereo 44.1 kHz) files with silence gaps, measured separately, so
that the WAV and FLAC tick times show what the extra synchronise of a FLAC step (scan, candidate download, host chain) costs.
Every arm checks that each stream's chunks equal transcribe_encoded's, notes compared as raw bits.  Reports audio-seconds
per second and the tick wall time (median and p99), one JSON line per arm, with the card's name and power limit.

    python bench_stream_encoded.py [--kinds flac,wav] [--streams 1,16,128] [--blocks-ms 20,100] [--seconds 60] [--rounds 1]
"""
import argparse
import json
import os
import struct
import sys
import tempfile
import time

import numpy as np

from bench_stream import card


def wav_s16(x: np.ndarray, rate: int) -> bytes:
    raw = np.clip(np.round(x * 32768), -32768, 32767).astype('<i2').tobytes()
    ch = x.shape[1]
    fmt = struct.pack('<HHIIHH', 1, ch, rate, rate * ch * 2, ch * 2, 16)
    body = b'WAVE' + b'fmt ' + struct.pack('<I', 16) + fmt + b'data' + struct.pack('<I', len(raw)) + raw
    return b'RIFF' + struct.pack('<I', len(body)) + body


def flac24(x: np.ndarray, rate: int) -> bytes:
    from oracle import flac as of
    v = np.clip(np.round(x * 2 ** 23), -2 ** 23, 2 ** 23 - 1).astype(np.int64)
    return of.encode(v, rate=rate, bps=24, subframe={'type': 'fixed', 'order': 2}, channel_mode='mid_side')


def same(got, want) -> bool:
    """Chunk ranges equal and notes bit-identical."""
    if got[0] != want[0] or len(got[1]) != len(want[1]):
        return False
    for g, w in zip(got[1], want[1]):
        for k, view in (('note_midi', np.uint32), ('note_dur', np.uint64), ('note_rest', np.uint8)):
            a, b = np.asarray(g[k]), np.asarray(w[k])
            if a.shape != b.shape or not np.array_equal(a.view(view) if k != 'note_rest' else a, b.view(view) if k != 'note_rest' else b):
                return False
    return True


def ticks_arm(push, streams, blocks, want, n, seconds):
    """One call per tick over the streams that still have data; finish at each stream's end."""
    got = [([], []) for _ in range(n)]
    pos, live, ticks = [0] * n, list(range(n)), []
    t = time.perf_counter()
    while live:
        items, fin = [], []
        for i in live:
            data, size = blocks[i]
            part = data[pos[i]:pos[i] + size]
            pos[i] += size
            items.append((streams[i], part))
            fin.append(pos[i] >= len(data))
        t0 = time.perf_counter()
        res = push(items, fin)
        ticks.append(time.perf_counter() - t0)
        for i, r in zip(live, res):
            got[i][0].extend(r[1])
            got[i][1].extend(r[2])
        live = [i for i, f in zip(live, fin) if not f]
    wall = time.perf_counter() - t
    tk = np.array(ticks) * 1e3
    return {'audio_s_per_s': round(n * seconds / wall, 1), 'ticks': len(ticks),
            'tick_ms_median': round(float(np.median(tk)), 3), 'tick_ms_p99': round(float(np.percentile(tk, 99)), 3),
            'identical': all(same(got[i], want[i]) for i in range(n))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--kinds', default='flac,wav')
    ap.add_argument('--streams', default='1,16,128')
    ap.add_argument('--blocks-ms', default='20,100')
    ap.add_argument('--seconds', type=float, default=60.0)
    ap.add_argument('--pool', type=int, default=4, help='distinct files per kind (streams cycle through them)')
    ap.add_argument('--rounds', type=int, default=1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_stream_encoded.py needs a CUDA device')
    from some_b200 import audio, export, synth, session as nsess
    print(f'# card: {card()}', flush=True)
    counts = [int(v) for v in args.streams.split(',')]
    with tempfile.TemporaryDirectory() as d:
        sess = nsess.Session(export.export(synth.write_checkpoint(d, synth.named_config('two_head'), seed=1234)), 0)
        for kind in args.kinds.split(','):
            rate = 48000 if kind == 'flac' else 44100
            files, samples = [], []
            for k in range(args.pool):
                x = np.stack([synth.synth_waveform(9000 + 2 * k + c, seconds=args.seconds, sr=rate, silence_gaps=True)
                              for c in range(2)], axis=1) * np.float32(0.9)
                data = flac24(x, rate) if kind == 'flac' else wav_s16(x, rate)
                path = os.path.join(d, f'{kind}{k}.{kind}')
                with open(path, 'wb') as f:
                    f.write(data)
                files.append(data)
                samples.append(audio.load(path, sr=None)[0])          # the host decode of the push_many arm (not timed)
            want_pool = [r[1:] for r in sess.transcribe_encoded(files)]
            for block_ms in [int(v) for v in args.blocks_ms.split(',')]:
                for n in counts:
                    idx = [i % args.pool for i in range(n)]
                    want = [want_pool[i] for i in idx]
                    for rnd in range(args.rounds):
                        base = {'kind': kind, 'streams': n, 'block_ms': block_ms, 'seconds': args.seconds, 'round': rnd}
                        # push_bytes_many
                        streams = [sess.stream_encoded() for _ in range(n)]
                        blocks = [(files[i], max(1, int(len(files[i]) * block_ms / (1000 * args.seconds)))) for i in idx]
                        r = ticks_arm(sess.push_bytes_many, streams, blocks, want, n, args.seconds)
                        for st in streams:
                            st.close()
                        print(json.dumps({**base, 'arm': 'push_bytes_many', **r}), flush=True)
                        # push_many of the host-decoded samples
                        streams = [sess.stream(rate) for _ in range(n)]
                        blocks = [(samples[i], rate * block_ms // 1000) for i in idx]
                        r = ticks_arm(sess.push_many, streams, blocks, want, n, args.seconds)
                        for st in streams:
                            st.close()
                        print(json.dumps({**base, 'arm': 'push_many_host_decoded', **r}), flush=True)
                        # one-shot, 16 files per call
                        t = time.perf_counter()
                        got = []
                        for a in range(0, n, 16):
                            got += [g[1:] for g in sess.transcribe_encoded([files[i] for i in idx[a:a + 16]])]
                        wall = time.perf_counter() - t
                        print(json.dumps({**base, 'arm': 'transcribe_encoded', 'audio_s_per_s': round(n * args.seconds / wall, 1),
                                          'identical': all(same(g, w) for g, w in zip(got, want))}), flush=True)
        sess.close()


if __name__ == '__main__':
    main()

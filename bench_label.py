"""Times labelling a DiffSinger dataset: the native command (some_session_label_dataset through Session.label_dataset)
against the Python driver (batch.batch_infer_dataset with load_audio=audio.load_native), on the same checkpoint.

Input: N seeded synthetic items (default 1000) of 5-15 s in a temporary dataset directory (transcriptions.csv and wavs/),
16-bit WAV at mixed rates (44.1, 48 and 22.05 kHz; two of every three items are resampled on the device), two_head model with
seeded random weights. Each arm labels the whole dataset --rounds times, the arms alternating; the best round counts. The
two outputs are compared byte for byte.

Reported per arm: items/s and audio-s/s (seconds of audio labelled per wall second). For the native command also the host
share: the part of its wall time spent outside some_session_transcribe_encoded (reading and checking the table, waiting for
the file reader, labelling, writing), as some_label_report gives it.

    python bench_label.py [--items 1000] [--rounds 2]

Prints the card's name and power limit with the numbers, then one JSON line. Nothing is written to the repository.
"""
import argparse
import csv
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REPO)


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def make_dataset(d, n_items, seed=9):
    from some_b200 import synth
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(d, 'wavs'), exist_ok=True)
    rates = (44100, 48000, 22050)
    total = 0.0
    rows = []
    for i in range(n_items):
        secs = float(rng.uniform(5, 15))
        rate = rates[i % 3]
        x = synth.synth_waveform(10_000 + i, seconds=secs, sr=rate, silence_gaps=True)
        synth.write_wav16(os.path.join(d, 'wavs', f'item{i:05d}.wav'), x, rate)
        n_ph = int(rng.integers(6, 30))
        cuts = np.sort(rng.uniform(0, secs, size=n_ph - 1))
        durs = np.diff(np.concatenate([[0.0], cuts, [secs]]))
        nums, left = [], n_ph
        while left:
            k = int(min(left, rng.integers(1, 4)))
            nums.append(k)
            left -= k
        rows.append({'name': f'item{i:05d}', 'ph_seq': ' '.join(['a'] * n_ph), 'ph_dur': ' '.join(f'{v:.6f}' for v in durs),
                     'ph_num': ' '.join(map(str, nums))})
        total += secs
    with open(os.path.join(d, 'transcriptions.csv'), 'w', encoding='utf8', newline='') as f:
        w = csv.DictWriter(f, fieldnames=['name', 'ph_seq', 'ph_dur', 'ph_num'])
        w.writeheader()
        w.writerows(rows)
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--items', type=int, default=1000)
    ap.add_argument('--rounds', type=int, default=2)
    args = ap.parse_args()

    import torch
    from some_b200 import audio, batch, export, plugin, synth
    from some_b200 import session as nsess

    with tempfile.TemporaryDirectory() as tmp:
        ds = os.path.join(tmp, 'ds')
        t0 = time.perf_counter()
        seconds = make_dataset(ds, args.items)
        print(f'dataset: {args.items} items, {seconds:.0f} s of audio, made in {time.perf_counter() - t0:.0f} s', flush=True)
        config = synth.named_config('two_head')
        ckpt = synth.write_checkpoint(tmp, config, seed=1234)
        path = export.export(ckpt)
        ins = plugin.MIDIExtractionInference(config=config, model_path=ckpt, device='cuda:0')
        sess = nsess.Session(path, 0)
        best = {'native': None, 'python': None}
        host_share = None
        out_n, out_p = os.path.join(tmp, 'native.csv'), os.path.join(tmp, 'python.csv')
        for r in range(args.rounds):
            rep = {}
            t = time.perf_counter()
            sess.label_dataset(ds, out_n, overwrite=True, report=rep)
            dt = time.perf_counter() - t
            if best['native'] is None or dt < best['native']:
                best['native'], host_share = dt, 1.0 - rep['gpu_seconds'] / rep['seconds']
            torch.cuda.synchronize()
            t = time.perf_counter()
            batch.batch_infer_dataset(ds, ins, config, csv=out_p, overwrite=True, load_audio=audio.load_native)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t
            best['python'] = dt if best['python'] is None else min(best['python'], dt)
            print(f'round {r}: native {best["native"]:.2f} s, python {best["python"]:.2f} s (best so far)', flush=True)
        with open(out_n, 'rb') as f, open(out_p, 'rb') as g:
            same = f.read() == g.read()
        sess.close()
    res = {'bench': 'label_dataset', 'card': card(), 'items': args.items, 'audio_seconds': round(seconds, 1), 'same_bytes': same}
    for arm, dt in best.items():
        res[f'{arm}_items_per_s'] = round(args.items / dt, 2)
        res[f'{arm}_audio_s_per_s'] = round(seconds / dt, 1)
    res['native_host_share'] = round(host_share, 3)
    res['speedup'] = round(best['python'] / best['native'], 2)
    print(f'card: {res["card"]}')
    print(json.dumps(res))


if __name__ == '__main__':
    main()

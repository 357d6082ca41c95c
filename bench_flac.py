"""Measures the GPU FLAC decoder (some_flac_scan + some_flac_decode, librosa.load's FLAC decode) on the audio of one C2
batch (64 recordings x 30 s of synthetic voice, stereo), encoded once by oracle/flac.py with settings like ``flac -5``
(4096-sample blocks, LPC order <= 8, partition order <= 5, mid/side; encoding is not timed), at 16-bit 48 kHz and at 24-bit
44.1 kHz, and prints one JSON line:

- device decode of the whole batch, median of --repeats after warm-up: ``scan_ms``, the scan kernels alone (CUDA events);
  ``chain_ms``, a host clock around ``audio.FlacBatch(...)``: the upload of the bytes, the scan, its one device-to-host
  copy and the chain on the host; ``decode_ms``, decode + emit to mono (CUDA events); ``total_ms``, both steps (host clock);
- the host baseline: the oracle's sequential decoder (numba, one core) on a subset, scaled to the batch.  It is a
  restatement written for tests, NOT libFLAC, which is not available here;
- batch.transcribe_recordings wall time with EncodedAudio inputs against the same call with the pre-decoded mono arrays
  and their rates, alternated, with the notes of both checked equal.

The card's name, power limit and max SM clock are read in the same run.  Nothing is written to the tree: --out DIR (optional)
receives a copy of the JSON line.

    python bench_flac.py [--recordings 64] [--seconds 30] [--repeats 20] [--cpu-recordings 2] [--out DIR]
"""
import argparse
import json
import os
import pathlib
import subprocess
import sys
import time

import numpy as np

REPO = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(REPO))


def gpu_info():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in out.split(',')]
    return {'gpu': name, 'power_limit': power, 'max_sm_clock': clock}


def encode_one(i, seconds, rate, bps):
    from oracle import flac as of
    from some_b200 import synth
    full = (1 << (bps - 1)) - 1
    gain = np.random.default_rng(i).uniform(0.3, 1.0)
    w = synth.synth_waveform(1000 + i, seconds=seconds, sr=rate, silence_gaps=bool(i % 2)) * gain
    x = np.round(np.stack([w, 0.8 * w + 0.05 * np.roll(w, 7)], 1).clip(-1, 1) * full).astype(np.int64)
    return of.encode(x, rate, bps, blocksize=4096, channel_mode='mid_side', max_lpc_order=8, max_porder=5), x


def encode_batch(n, seconds, rate, bps):
    """n recordings encoded by the oracle, one process per core (the encoder is slow and not what is measured)."""
    import concurrent.futures
    from some_b200 import audio
    with concurrent.futures.ProcessPoolExecutor(max_workers=min(n, os.cpu_count() or 1)) as pool:
        done = list(pool.map(encode_one, range(n), [seconds] * n, [rate] * n, [bps] * n))
    return [audio.parse_flac(data, f'rec{i}') for i, (data, _) in enumerate(done)], [x for _, x in done]


def device_decode(recs, repeats):
    """(median / min ms of scan, FlacBatch (upload + scan + chain), decode + emit and their total; the mono output; the
    FlacBatch)"""
    import torch
    from some_b200 import audio
    dev = torch.device('cuda', 0)
    times = {'scan_ms': [], 'chain_ms': [], 'decode_ms': [], 'total_ms': []}
    out = None
    for it in range(repeats + 3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fb = audio.FlacBatch(recs, dev)                     # upload + scan + one D2H + chain
        t1 = time.perf_counter()
        starts = np.concatenate([[0], np.cumsum(fb.lengths)])
        if out is None:
            out = torch.empty(int(starts[-1]), dtype=torch.float32, device=dev)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        status = fb.emit(out, {r: int(starts[r]) for r in range(len(recs))})
        b.record()
        b.synchronize()
        t2 = time.perf_counter()
        assert int(status.item()) == 0
        if it >= 3:
            times['chain_ms'].append((t1 - t0) * 1e3)
            times['decode_ms'].append(a.elapsed_time(b))
            times['total_ms'].append((t2 - t0) * 1e3)
    # the scan alone, on the device, with the upload done once
    import ctypes as C
    from some_b200 import _lib
    lib = _lib.load()
    ws = torch.empty(int(lib.some_flac_scan_workspace_bytes(fb.data.numel())), dtype=torch.uint8, device=dev)
    cap = fb.frames.numel() // 40
    count = torch.zeros(1, dtype=torch.int32, device=dev)
    for it in range(repeats + 3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        _lib.check(lib.some_flac_scan(fb.data.data_ptr(), fb.data.numel(), fb.streams.data_ptr(), len(recs),
                                      fb.frames.data_ptr(), cap, count.data_ptr(), ws.data_ptr(),
                                      C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), 'some_flac_scan')
        b.record()
        b.synchronize()
        if it >= 3:
            times['scan_ms'].append(a.elapsed_time(b))
    stats = {k: round(float(np.median(v)), 3) for k, v in times.items()}
    stats.update({k.replace('_ms', '_ms_min'): round(float(np.min(v)), 3) for k, v in times.items()})
    return stats, out.cpu().numpy(), fb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--recordings', type=int, default=64)
    ap.add_argument('--seconds', type=float, default=30.0)
    ap.add_argument('--repeats', type=int, default=20)
    ap.add_argument('--cpu-recordings', type=int, default=2, help='recordings the oracle decoder is timed on')
    ap.add_argument('--e2e-repeats', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()

    import torch
    from oracle import flac as of
    from some_b200 import audio, batch, plugin, synth
    assert torch.cuda.is_available(), 'bench_flac.py measures the GPU: no CUDA device found'
    res = dict(gpu_info())
    res.update(recordings=a.recordings, seconds=a.seconds, audio_seconds=a.recordings * a.seconds, channels=2)
    batches = {}
    for rate, bps in ((48000, 16), (44100, 24)):
        tag = f'{bps}bit_{rate}'
        t0 = time.perf_counter()
        recs, ints = batches[tag] = encode_batch(a.recordings, a.seconds, rate, bps)
        res[f'encode_s_{tag}'] = round(time.perf_counter() - t0, 1)
        nbytes = sum(len(r.data) for r in recs)
        stats, mono, fb = device_decode(recs, a.repeats)
        frames = sum(len(c) for c in fb.chains)
        first = ints[0].astype(np.float32) * np.float32(2.0 ** -(bps - 1))
        exact = bool(np.array_equal(mono[:len(first)], audio.to_mono(first.T)))
        res[tag] = dict(stats, flac_bytes=nbytes, frames=frames, candidates=fb.n_candidates,
                        compression=round(nbytes / sum(x.size * bps / 8 for x in ints), 3),
                        audio_s_per_s=round(a.recordings * a.seconds / (stats['total_ms'] / 1e3)),
                        first_recording_matches_input=exact)
        # host baseline: the oracle decoder (numba, one core), JIT compiled outside the timed region
        of.decode(recs[-1].data)
        t0 = time.perf_counter()
        for r in recs[:a.cpu_recordings]:
            of.decode(r.data)
        cpu_s = time.perf_counter() - t0
        res[tag].update(oracle_not_libflac_s_for_subset=round(cpu_s, 3), oracle_subset_recordings=a.cpu_recordings,
                        oracle_not_libflac_s_for_batch_scaled=round(cpu_s * a.recordings / a.cpu_recordings, 2))
    res['cpu_count'] = os.cpu_count()

    # transcribe_recordings: EncodedAudio (48 kHz, 16-bit) against the same audio pre-decoded to mono arrays + rates
    config = synth.named_config('two_head')
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        ckpt = synth.write_checkpoint(d, config, seed=1234)
        ins = plugin.MIDIExtractionInference(config=config, model_path=ckpt, device='cuda:0')
    recs, ints = batches['16bit_48000']
    pre = [audio.to_mono((x.astype(np.float32) * np.float32(2.0 ** -15)).T) for x in ints]
    rates = [48000] * len(pre)

    def run_encoded():
        return batch.transcribe_recordings(ins, recs)

    def run_pre():
        return batch.transcribe_recordings(ins, pre, rates=rates)

    r_enc, r_pre = run_encoded(), run_pre()
    same = all(o1 == o2 and all(np.array_equal(x[k], y[k]) for x, y in zip(n1, n2) for k in ('note_midi', 'note_dur', 'note_rest'))
               for (o1, n1), (o2, n2) in zip(r_enc, r_pre))
    t_enc, t_pre = [], []
    for _ in range(a.e2e_repeats):
        for fn, acc in ((run_encoded, t_enc), (run_pre, t_pre)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            acc.append(time.perf_counter() - t0)
    res.update(transcribe_ms_encoded_flac_48k=[round(t * 1e3, 1) for t in t_enc],
               transcribe_ms_predecoded_48k=[round(t * 1e3, 1) for t in t_pre],
               transcribe_notes_identical=bool(same))
    line = json.dumps(res)
    print(line)
    if a.out:
        pathlib.Path(a.out).mkdir(parents=True, exist_ok=True)
        (pathlib.Path(a.out) / 'bench_flac.json').write_text(line + '\n')


if __name__ == '__main__':
    main()

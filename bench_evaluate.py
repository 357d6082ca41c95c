"""Measures the evaluator (some_b200/evaluate.py): a synthetic labelled DiffSinger dataset (default 64 x 30 s, seeded
synth.synth_labelled, 16-bit WAV in a temporary directory) scored with the bf16 product trunk and the fp32 validation
trunk.  Prints one JSON line:

- items/s and audio-seconds/s of evaluate_dataset, bf16 (every item) and fp32 (``--fp32-items`` items), wall clock around
  calls that end in a device synchronise, best of ``--repeats`` after one warm-up;
- the split of one bf16 pass: host loading (labels + WAV decode, timed separately on the host), and the device time of the
  trunk kernels, of some_eval_clips and of the decode, from CUDA events (Engine.start_profile);
- the CPU oracle (oracle/decode.py forward + oracle/evaluate.py losses and accuracy) on ``--oracle-items`` items.

    python bench_evaluate.py [--items 64] [--seconds 30] [--repeats 3] [--fp32-items 8] [--oracle-items 1]
"""
import argparse
import json
import pathlib
import sys
import tempfile
import time

REPO = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(REPO))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--items', type=int, default=64)
    ap.add_argument('--seconds', type=float, default=30.0)
    ap.add_argument('--config', default='two_head')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--fp32-items', type=int, default=8)
    ap.add_argument('--oracle-items', type=int, default=1)
    args = ap.parse_args()

    import numpy as np
    import torch

    from oracle import decode as odecode
    from oracle import evaluate as oev
    from some_b200 import audio, evaluate, plugin, synth

    assert torch.cuda.is_available(), 'bench_evaluate.py measures on a CUDA device'
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    config = synth.named_config(args.config)
    quantized = args.config.startswith('quant')
    out = {'config': args.config, 'items': args.items, 'seconds_per_item': args.seconds,
           'gpu': torch.cuda.get_device_name(dev)}
    with tempfile.TemporaryDirectory() as d:
        d = pathlib.Path(d)
        ckpt = synth.write_checkpoint(d / 'ckpt', config, seed=1234)
        cls = plugin.QuantizedMIDIExtractionInference if quantized else plugin.MIDIExtractionInference
        ins = cls(config=config, model_path=ckpt, device='cuda:0')
        items = [(f'b{k:03d}',) + synth.synth_labelled(5000 + k, args.seconds) for k in range(args.items)]
        data = synth.write_labelled_dataset(d / 'data', items)
        sub = synth.write_labelled_dataset(d / 'sub', items[:args.fp32_items])
        audio_s = args.items * args.seconds

        def timed(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn()
            torch.cuda.synchronize()
            return time.perf_counter() - t0, r

        evaluate.evaluate_dataset(ins, data, config)                                    # warm-up
        bf = [timed(lambda: evaluate.evaluate_dataset(ins, data, config)) for _ in range(args.repeats)]
        t_bf = min(t for t, _ in bf)
        out['bf16'] = {'s': t_bf, 'all_s': [t for t, _ in bf], 'items_per_s': args.items / t_bf,
                       'audio_s_per_s': audio_s / t_bf, 'summary': bf[0][1].summary}

        # host loading alone: labels + WAV decode of every item, as the driver's loader threads do it
        t0 = time.perf_counter()
        labs = evaluate.load_labels(data, config, quantized)
        for it in labs:
            audio.load_native(it['wav_fn'])
        out['host_load_s'] = time.perf_counter() - t0

        # device split of one bf16 pass
        eng = ins.model
        eng.start_profile()
        evaluate.evaluate_dataset(ins, data, config)
        prof = eng.stop_profile()
        trunk = sum(v['ms'] for k, v in prof.items() if k not in ('some_eval_clips', 'some_decode_notes', 'some_mel_logmel'))
        out['device_ms'] = {'mel': prof.get('some_mel_logmel', {}).get('ms', 0.0), 'trunk': trunk,
                            'eval_clips': prof.get('some_eval_clips', {}).get('ms', 0.0),
                            'eval_clips_launches': prof.get('some_eval_clips', {}).get('launches', 0),
                            'decode': prof.get('some_decode_notes', {}).get('ms', 0.0)}

        evaluate.evaluate_dataset(ins, sub, config, precision='fp32')                  # warm-up (builds the fp32 model)
        t_f, rep_f = timed(lambda: evaluate.evaluate_dataset(ins, sub, config, precision='fp32'))
        n_f = len(rep_f.items)
        out['fp32'] = {'items': n_f, 's': t_f, 'items_per_s': n_f / t_f, 'audio_s_per_s': n_f * args.seconds / t_f,
                       'summary': rep_f.summary}

        # CPU oracle: fp32 forward on the CPU, then the restated losses and accuracy
        sd = synth.fabricate_state_dict(config, seed=1234)
        t0 = time.perf_counter()
        for it in labs[:args.oracle_items]:
            w, _ = audio.load_native(it['wav_fn'])
            r = odecode.infer_clip(sd, config, w, quantized=quantized, return_intermediates=True)
            arr = evaluate.item_labels(it, r['bounds'].shape[0], config['hop_size'] / config['audio_sample_rate'], quantized)
            p = np.clip(r['probs'].astype(np.float64), 1e-7, 1 - 1e-7)
            logits = np.log(p) if quantized else np.log(p / (1 - p))
            oev.losses(logits.astype(np.float32), r['bounds'], arr, config, quantized)
            oev.accuracy_counts(logits.astype(np.float32), arr, config, quantized)
        t_o = time.perf_counter() - t0
        out['oracle_cpu'] = {'items': args.oracle_items, 's': t_o,
                             'audio_s_per_s': args.oracle_items * args.seconds / t_o, 'threads': torch.get_num_threads()}
    print(json.dumps(out))


if __name__ == '__main__':
    main()

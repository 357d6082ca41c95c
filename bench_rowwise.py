"""Per-kernel timing of the HBM-bound kernels of one step at the benchmark shape (64 clips x 30 s, both streams):
log-mel, LayerNorm (bf16 out, bf16 + f32 out), the bound head and the depthwise conv.

    python bench_rowwise.py [--iters 50] [--warmup 5] [--dump DIR] [--lib PATH]

Each kernel is timed alone with CUDA events over --iters back-to-back launches after a warm-up.  Its algorithmic bytes (and
for dwconv its FMAs) come from the shapes; the rate is printed against two ceilings measured or quoted in the same run: a
device-to-device cudaMemcpyAsync of 1 GB (read + write counted) and the 3.35 TB/s of the H100 SXM data sheet.  The occupancy
is the occupancy calculator's CTAs per SM for the kernel as the library launches it.  --dump DIR writes every kernel's output
on seeded inputs as .npy, so that two builds (--lib) can be compared bit for bit.  Prints one JSON line."""
import argparse
import ctypes as C
import json
import os
import pathlib
import subprocess
import sys

import numpy as np
import torch

REPO = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(REPO))

from some_b200 import _lib  # noqa: E402
from some_b200 import synth  # noqa: E402
from some_b200.weights import mel_tables  # noqa: E402

CLIPS, SECONDS, SR = 64, 30.0, 44100
DATASHEET_BPS = 3.35e12
# entry symbols of the kernels (their host stubs are exported by libsome_b200.so)
KERNEL_SYMBOLS = {
    'mel': '_ZN4some10mel_kernelEPKfPKlS3_PKiiS5_S5_S1_S1_S1_PfP13__nv_bfloat16f',
    'layernorm': '_ZN4some16layernorm_kernelENS_8LnParamsE',
    'bound_head': '_ZN4some17bound_head_kernelEPKfS1_S1_S1_fiPf',
    'dwconv': '_ZN4some13dwconv_kernelENS_8DwParamsE',
}


class FuncAttributes(C.Structure):   # cudaFuncAttributes (CUDA 12), with room to spare at the end
    _fields_ = [('sharedSizeBytes', C.c_size_t), ('constSizeBytes', C.c_size_t), ('localSizeBytes', C.c_size_t),
                ('maxThreadsPerBlock', C.c_int), ('numRegs', C.c_int), ('ptxVersion', C.c_int),
                ('binaryVersion', C.c_int), ('cacheModeCA', C.c_int), ('maxDynamicSharedSizeBytes', C.c_int),
                ('preferredShmemCarveout', C.c_int), ('rest', C.c_int * 32)]


def occupancy(lib, name):
    """CTAs per SM for the kernel's launch-bounds block size and the dynamic shared memory the library set on it."""
    rt = C.CDLL('libcudart.so.12')
    fn = C.cast(getattr(lib, KERNEL_SYMBOLS[name]), C.c_void_p)
    attr = FuncAttributes()
    rc = rt.cudaFuncGetAttributes(C.byref(attr), fn)
    if rc != 0:
        return {'error': f'cudaFuncGetAttributes = {rc}'}
    ctas = C.c_int(0)
    block = attr.maxThreadsPerBlock
    rc = rt.cudaOccupancyMaxActiveBlocksPerMultiprocessor(C.byref(ctas), fn, block,
                                                          C.c_size_t(attr.maxDynamicSharedSizeBytes))
    if rc != 0:
        return {'error': f'cudaOccupancyMaxActiveBlocksPerMultiprocessor = {rc}'}
    return {'ctas_per_sm': ctas.value, 'warps_per_sm': ctas.value * block // 32, 'threads_per_cta': block,
            'registers': attr.numRegs, 'local_bytes': int(attr.localSizeBytes),
            'dynamic_smem': attr.maxDynamicSharedSizeBytes, 'static_smem': int(attr.sharedSizeBytes)}


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader,nounits', '-i',
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, power, sm, sm_max = [s.strip() for s in out.strip().split(',')]
        return {'gpu': name, 'power_limit_w': float(power), 'sm_clock_mhz': float(sm), 'sm_clock_max_mhz': float(sm_max)}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {'gpu': torch.cuda.get_device_name(), 'power_limit_w': None, 'sm_clock_mhz': None, 'sm_clock_max_mhz': None}


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--dump', metavar='DIR', default=None, help='write every kernel output as DIR/<kernel>.npy')
    ap.add_argument('--lib', default=None, help='libsome_b200.so to load (default: the one in this tree)')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_rowwise.py measures on a CUDA device'
    if args.lib is not None:
        _lib.LIB_PATH = pathlib.Path(args.lib).resolve()
    lib = _lib.load()
    dev = torch.device('cuda')
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    gen = torch.Generator(device=dev)
    gen.manual_seed(20261017)

    # ---- shapes: 64 clips of 30 s, T = 1 + samples // 512 frames each; both streams (groups = 2) for the trunk kernels
    n = int(SECONDS * SR)
    t_clip = 1 + n // _lib.HOP
    m = CLIPS * t_clip
    cu = torch.arange(0, CLIPS + 1, dtype=torch.int32, device=dev) * t_clip
    wave = torch.randn(CLIPS * n, device=dev, generator=gen) * 0.1
    starts = torch.arange(CLIPS, dtype=torch.int64, device=dev) * n
    lens = torch.full((CLIPS,), n, dtype=torch.int64, device=dev)
    tab = mel_tables(synth.named_config('two_head'), dev)
    mel_out = torch.empty(m, _lib.N_MELS, device=dev, dtype=torch.bfloat16)

    x = [torch.randn(m, _lib.DIM, device=dev, generator=gen) * 3 + 1.5 for _ in range(2)]
    gamma = [torch.rand(_lib.DIM, device=dev, generator=gen) + 0.5 for _ in range(2)]
    beta = [torch.randn(_lib.DIM, device=dev, generator=gen) * 0.1 for _ in range(2)]
    ln_bf16 = [torch.empty(m, _lib.DIM, device=dev, dtype=torch.bfloat16) for _ in range(2)]
    ln_f32 = [torch.empty(m, _lib.DIM, device=dev) for _ in range(2)]
    head_w = torch.randn(_lib.DIM, device=dev, generator=gen) / _lib.DIM ** 0.5
    bounds = torch.empty(m, device=dev)
    dw_x = [(torch.randn(m, _lib.DIM, device=dev, generator=gen)).to(torch.bfloat16) for _ in range(2)]
    dw_w = [torch.randn(_lib.CONV_K, _lib.DIM, device=dev, generator=gen) * 0.2 for _ in range(2)]
    dw_b = [torch.randn(_lib.DIM, device=dev, generator=gen) * 0.1 for _ in range(2)]
    dw_out = [torch.empty(m, _lib.DIM, device=dev, dtype=torch.bfloat16) for _ in range(2)]

    def mel():
        _lib.check(lib.some_mel_logmel(wave.data_ptr(), starts.data_ptr(), lens.data_ptr(), cu.data_ptr(), CLIPS, t_clip,
                                       tab['mel_start'].data_ptr(), tab['mel_count'].data_ptr(),
                                       tab['mel_weights'].data_ptr(), tab['twiddle'].data_ptr(), tab['window'].data_ptr(),
                                       None, mel_out.data_ptr(), 1e-5, stream), 'some_mel_logmel')

    def layernorm(with_f32):
        a = _lib.LnArgs()
        a.x, a.gamma, a.beta = _lib.pair(*x), _lib.pair(*gamma), _lib.pair(*beta)
        a.out_bf16 = _lib.pair(*ln_bf16)
        a.out_f32 = _lib.pair(*ln_f32) if with_f32 else (C.c_void_p * 2)()
        a.groups, a.M = 2, m
        return lambda: _lib.check(lib.some_layernorm(C.byref(a), stream), 'some_layernorm')

    def bound_head():
        _lib.check(lib.some_bound_head(x[0].data_ptr(), gamma[0].data_ptr(), beta[0].data_ptr(), head_w.data_ptr(), 0.3, m,
                                       bounds.data_ptr(), stream), 'some_bound_head')

    dwa = _lib.DwconvArgs()
    dwa.x, dwa.w, dwa.b, dwa.out = _lib.pair(*dw_x), _lib.pair(*dw_w), _lib.pair(*dw_b), _lib.pair(*dw_out)
    dwa.groups, dwa.B, dwa.cu_frames, dwa.max_frames = 2, CLIPS, cu.data_ptr(), t_clip

    def dwconv():
        _lib.check(lib.some_dwconv_bn_silu(C.byref(dwa), stream), 'some_dwconv_bn_silu')

    d = _lib.DIM
    kernels = {   # name: (launch, algorithmic bytes, fp32 FMAs, kernel symbol)
        'mel': (mel, m * (_lib.N_FFT // 4 * 4 + _lib.N_MELS * 2), 0, 'mel'),   # hop of new samples in, bf16 mel out
        'layernorm_bf16': (layernorm(False), 2 * m * (d * 4 + d * 2), 0, 'layernorm'),
        'layernorm_bf16_f32': (layernorm(True), 2 * m * (d * 4 + d * 2 + d * 4), 0, 'layernorm'),
        'bound_head': (bound_head, m * (d * 4 + 4), 0, 'bound_head'),
        'dwconv': (dwconv, 2 * m * (d * 2 + d * 2), 2 * m * d * _lib.CONV_K, 'dwconv'),
    }

    # ---- ceilings: 1 GB device-to-device copy (cudaMemcpyAsync), read + write
    src = torch.empty(1 << 30, dtype=torch.uint8, device=dev)
    dst = torch.empty_like(src)
    copy_ms = time_ms(lambda: dst.copy_(src), max(args.iters, 20), args.warmup)
    copy_bps = 2 * src.numel() / (copy_ms * 1e-3)
    del src, dst

    results = {}
    for name, (fn, nbytes, fmas, sym) in kernels.items():
        ms = time_ms(fn, args.iters, args.warmup)
        bps = nbytes / (ms * 1e-3)
        r = {'ms': round(ms, 4), 'gb': round(nbytes / 1e9, 4), 'gb_per_s': round(bps / 1e9, 1),
             'of_copy_rate': round(bps / copy_bps, 3), 'of_datasheet': round(bps / DATASHEET_BPS, 3)}
        if fmas:
            r['gfma_per_s'] = round(fmas / (ms * 1e-3) / 1e9, 1)
        r['occupancy'] = occupancy(lib, sym)
        results[name] = r
    clocks = card()

    if args.dump is not None:
        os.makedirs(args.dump, exist_ok=True)
        outs = {}
        mel()
        outs['mel_bf16'] = mel_out
        layernorm(True)()
        outs['ln_bf16_g0'], outs['ln_bf16_g1'], outs['ln_f32_g0'], outs['ln_f32_g1'] = ln_bf16 + ln_f32
        ln_bf16b = [t.clone() for t in ln_bf16]
        layernorm(False)()
        outs['ln_bf16only_g0'], outs['ln_bf16only_g1'] = ln_bf16
        bound_head()
        outs['bounds'] = bounds
        dwconv()
        outs['dwconv_g0'], outs['dwconv_g1'] = dw_out
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(ln_bf16b, ln_bf16)), 'LayerNorm bf16 output depends on the f32 output'
        for k, t in outs.items():
            a = t.view(torch.int16) if t.dtype == torch.bfloat16 else t
            np.save(os.path.join(args.dump, f'{k}.npy'), a.cpu().numpy())

    line = {'bench': 'rowwise', 'shape': {'clips': CLIPS, 'seconds': SECONDS, 'M': m, 'groups': 2},
            'library': str(_lib.LIB_PATH), **clocks, 'copy_1gb_ms': round(copy_ms, 4),
            'copy_gb_per_s': round(copy_bps / 1e9, 1), 'datasheet_gb_per_s': DATASHEET_BPS / 1e9, 'kernels': results}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()

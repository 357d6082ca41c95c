"""ctypes binding of libsome_b200.so (include/some_b200.h).  There is no fallback: if the CUDA
library is missing or a call fails, this module raises."""
from __future__ import annotations

import ctypes as C
import os
import pathlib

_HERE = pathlib.Path(__file__).resolve().parent
LIB_PATH = _HERE / 'libsome_b200.so'

EPI_STORE_BF16, EPI_SILU_BF16, EPI_GLU_BF16, EPI_RESID_F32, EPI_GLU_RESID_F32, EPI_BIAS_F32, \
    EPI_SIGMOID_F32, EPI_SOFTMAX_F32, EPI_LN_STORE_BF16, EPI_LN_SILU_BF16, EPI_LN_GLU_BF16, EPI_RESID_F32_LN, \
    EPI_GLU_RESID_F32_LN = range(13)
LN_SLOTS = 8
ABI_VERSION = 202
K_GEMM, K_ATTENTION, K_LAYERNORM, K_DWCONV, K_BOUND_HEAD, K_ROW_STATS = range(6)
KERNEL_NAMES = {K_GEMM: 'some_gemm', K_ATTENTION: 'some_attention_varlen', K_LAYERNORM: 'some_layernorm',
                K_DWCONV: 'some_dwconv_bn_silu', K_BOUND_HEAD: 'some_bound_head', K_ROW_STATS: 'some_row_stats'}

DIM, HEADS, HEAD_DIM, CONV_K, N_MELS, N_FFT, HOP, MEL_BINS, MEL_MAXW = 512, 8, 64, 31, 80, 2048, 512, 372, 24
MEL_TW = 1396

_vp = C.c_void_p


class LnArgs(C.Structure):
    _fields_ = [('x', _vp * 2), ('gamma', _vp * 2), ('beta', _vp * 2), ('out_bf16', _vp * 2),
                ('out_f32', _vp * 2), ('groups', C.c_int), ('M', C.c_int)]


class GemmArgs(C.Structure):
    _fields_ = [('A', _vp * 2), ('W', _vp * 2), ('bias', _vp * 2), ('out', _vp * 2), ('resid', _vp * 2),
                ('groups', C.c_int), ('M', C.c_int), ('N', C.c_int), ('K', C.c_int), ('lda', C.c_int),
                ('ld_out', C.c_int), ('epilogue', C.c_int), ('alpha', C.c_float),
                ('ln_s', _vp * 2), ('ln_stats', _vp * 2), ('ln_parts', C.c_int), ('out_bf16', _vp * 2)]


class RowStatsArgs(C.Structure):
    _fields_ = [('x', _vp * 2), ('out_bf16', _vp * 2), ('ln_stats', _vp * 2), ('groups', C.c_int), ('M', C.c_int)]


CALIB_MAX, CALIB_K = 512, 2048


class CalibrationC(C.Structure):
    _fields_ = [('means', _vp), ('count', C.c_int), ('w', (_vp * 2) * CALIB_MAX), ('k', C.c_int * CALIB_MAX)]


class ProfileRecord(C.Structure):
    _fields_ = [('kernel', C.c_int), ('epilogue', C.c_int), ('n', C.c_int), ('k', C.c_int), ('ms', C.c_float),
                ('work', C.c_double)]


class AttnArgs(C.Structure):
    _fields_ = [('qkv', _vp * 2), ('out', _vp * 2), ('groups', C.c_int), ('B', C.c_int), ('M', C.c_int),
                ('cu_frames', _vp), ('max_frames', C.c_int)]


class DwconvArgs(C.Structure):
    _fields_ = [('x', _vp * 2), ('w', _vp * 2), ('b', _vp * 2), ('out', _vp * 2), ('groups', C.c_int),
                ('B', C.c_int), ('cu_frames', _vp), ('max_frames', C.c_int)]


class DecodeArgs(C.Structure):
    _fields_ = [('probs', _vp), ('bounds', _vp), ('cu_frames', _vp), ('B', C.c_int), ('M', C.c_int),
                ('N', C.c_int), ('quantized', C.c_int), ('vmin', C.c_float), ('vmax', C.c_float),
                ('deviation', C.c_float), ('threshold', C.c_float), ('note_midi', _vp), ('note_dur', _vp),
                ('note_rest', _vp), ('note_count', _vp), ('dbg_frame2item', _vp), ('dbg_values', _vp),
                ('dbg_rest', _vp), ('scratch', _vp)]


class BlockWeightsC(C.Structure):
    _fields_ = [('ln_g', _vp * 5), ('ln_b', _vp * 5), ('ffn_w1', _vp * 2), ('ffn_b1', _vp * 2), ('ffn_w2', _vp * 2),
                ('ffn_b2', _vp * 2), ('w_qkv', _vp), ('w_out', _vp), ('b_out', _vp), ('w_pw1', _vp), ('b_pw1', _vp),
                ('w_dw', _vp), ('b_dw', _vp), ('w_pw2', _vp), ('b_pw2', _vp),
                ('ffn_w1f', _vp * 2), ('ffn_s1', _vp * 2), ('ffn_b1f', _vp * 2), ('w_qkvf', _vp), ('s_qkv', _vp),
                ('b_qkvf', _vp), ('w_pw1f', _vp), ('s_pw1', _vp), ('b_pw1f', _vp)]


class ModelC(C.Structure):
    _fields_ = [('lay', C.c_int), ('outdim', C.c_int), ('w_in', _vp * 2), ('b_in', _vp * 2),
                ('blocks', C.POINTER(BlockWeightsC)), ('glu_w', C.POINTER(_vp)), ('glu_b', C.POINTER(_vp)),
                ('w_head', _vp), ('b_head', _vp), ('w_cut', _vp), ('b_cut', C.c_float), ('ln_fold', C.c_int)]


class WorkspaceC(C.Structure):
    _fields_ = [('x', _vp * 2), ('a', _vp * 2), ('h', _vp * 2), ('qkv', _vp * 2), ('g', _vp * 2), ('units', _vp),
                ('probs', _vp), ('bounds', _vp), ('xb', _vp * 2), ('ln_stats', _vp * 2)]


class BlockWeightsF32C(C.Structure):
    _fields_ = [('ln_g', _vp * 5), ('ln_b', _vp * 5), ('ffn_w1', _vp * 2), ('ffn_b1', _vp * 2), ('ffn_w2', _vp * 2),
                ('ffn_b2', _vp * 2), ('w_qkv', _vp), ('w_out', _vp), ('b_out', _vp), ('w_pw1', _vp), ('b_pw1', _vp),
                ('w_dw', _vp), ('b_dw', _vp), ('w_pw2', _vp), ('b_pw2', _vp)]


class ModelF32C(C.Structure):
    _fields_ = [('lay', C.c_int), ('outdim', C.c_int), ('w_in', _vp * 2), ('b_in', _vp * 2),
                ('blocks', C.POINTER(BlockWeightsF32C)), ('glu_w', C.POINTER(_vp)), ('glu_b', C.POINTER(_vp)),
                ('w_head', _vp), ('b_head', _vp), ('w_cut', _vp), ('b_cut', C.c_float)]


class WorkspaceF32C(C.Structure):
    _fields_ = [('x', _vp * 2), ('a', _vp * 2), ('h', _vp * 2), ('qkv', _vp * 2), ('g', _vp * 2), ('y', _vp * 2),
                ('units', _vp), ('probs', _vp), ('bounds', _vp)]


EXPORTS = {
    # name: (restype, argtypes)
    'some_version': (C.c_int, []),
    'some_last_error': (C.c_char_p, []),
    'some_set_pdl': (C.c_int, [C.c_int]),
    'some_pack_bf16': (C.c_int, [_vp, C.c_longlong, _vp]),
    'some_pack_glu_rows': (C.c_int, [_vp, C.c_int, C.c_int, C.c_longlong, _vp]),
    'some_pack_dwconv_bn': (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, C.c_int, C.c_int, _vp, _vp]),
    'some_pack_ln_fold': (C.c_int, [_vp, _vp, _vp, _vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp]),
    'some_mel_tables': (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, _vp, _vp, _vp, _vp, _vp]),
    'some_mel_logmel': (C.c_int, [_vp, _vp, _vp, _vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                  C.c_float, _vp]),
    'some_mel_logmel_keyshift': (C.c_int, [_vp, _vp, _vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, _vp, _vp,
                                           _vp, _vp, _vp, _vp, _vp, C.c_float, _vp]),
    'some_layernorm': (C.c_int, [C.POINTER(LnArgs), _vp]),
    'some_gemm': (C.c_int, [C.POINTER(GemmArgs), _vp]),
    'some_attention_varlen': (C.c_int, [C.POINTER(AttnArgs), _vp]),
    'some_dwconv_bn_silu': (C.c_int, [C.POINTER(DwconvArgs), _vp]),
    'some_bound_head': (C.c_int, [_vp, _vp, _vp, _vp, C.c_float, C.c_int, _vp, _vp]),
    'some_decode_scratch_bytes': (C.c_uint64, [C.c_int]),
    'some_decode_notes': (C.c_int, [C.POINTER(DecodeArgs), _vp]),
    'some_slicer_rms': (C.c_int, [_vp, C.c_longlong, C.c_int, C.c_int, _vp, C.c_int, _vp]),
    'some_row_stats': (C.c_int, [C.POINTER(RowStatsArgs), _vp]),
    'some_col_means': (C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, _vp]),
    'some_forward': (C.c_int, [C.POINTER(ModelC), C.POINTER(WorkspaceC), C.c_int, C.c_int, _vp, C.c_int, C.c_int, _vp,
                               C.POINTER(CalibrationC), _vp]),
    'some_forward_f32': (C.c_int, [C.POINTER(ModelF32C), C.POINTER(WorkspaceF32C), C.c_int, C.c_int, _vp, C.c_int, C.c_int,
                                   _vp]),
    'some_workspace_bytes': (C.c_uint64, [C.c_int, C.c_int, C.c_int]),
    'some_workspace_carve': (C.c_int, [_vp, C.c_uint64, C.c_int, C.c_int, C.c_int, C.POINTER(WorkspaceC)]),
    'some_profiler_create': (C.c_int, [C.c_int, C.POINTER(_vp)]),
    'some_profiler_destroy': (C.c_int, [_vp]),
    'some_profiler_reset': (C.c_int, [_vp]),
    'some_profiler_read': (C.c_int, [_vp, C.c_int, C.POINTER(ProfileRecord)]),
}

_lib = None


class SomeB200Error(RuntimeError):
    pass


def load():
    """Loads the shared library (once).  Raises if it has not been built: there is no CPU path."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.is_file():
        raise SomeB200Error(
            f'{LIB_PATH} not found: build it with `python -c "import __graft_entry__ as g; g.build()"` '
            f'or `make -C {_HERE / "csrc"}` (nvcc, sm_90a). some_b200 has no CPU fallback.')
    lib = C.CDLL(os.fspath(LIB_PATH))
    for name, (restype, argtypes) in EXPORTS.items():
        fn = getattr(lib, name)  # AttributeError if the header and the library disagree
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.some_version() != ABI_VERSION:
        raise SomeB200Error(f'{LIB_PATH} is ABI version {lib.some_version()}, this package expects {ABI_VERSION}: rebuild it '
                            f'(make -C {_HERE / "csrc"})')
    _lib = lib
    return lib


def check(rc: int, what: str = ''):
    if rc != 0:
        msg = load().some_last_error().decode('utf8', 'replace')
        raise SomeB200Error(f'{what or "libsome_b200"} failed ({rc}): {msg}')


def ptr(t):
    """Device (or host) address of a torch tensor, or None."""
    return None if t is None else t.data_ptr()


def pair(a, b=None):
    arr = (_vp * 2)()
    arr[0] = ptr(a)
    arr[1] = ptr(b if b is not None else a)
    return arr

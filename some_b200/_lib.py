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


EVAL_HEAD_TC, EVAL_HEAD_F32 = 0, 1


class EvalArgs(C.Structure):
    _fields_ = [('logits', _vp), ('bounds', _vp), ('cu_frames', _vp), ('unit2note', _vp), ('cu_notes', _vp),
                ('note_midi', _vp), ('note_rest', _vp), ('B', C.c_int), ('M', C.c_int), ('N', C.c_int),
                ('quantized', C.c_int), ('head', C.c_int), ('vmin', C.c_float), ('vmax', C.c_float),
                ('deviation', C.c_float), ('threshold', C.c_float), ('midi_loss', _vp), ('bound_loss', _vp),
                ('correct', _vp), ('probs', _vp)]


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


class SessionInfo(C.Structure):
    _fields_ = [('sample_rate', C.c_int), ('hop', C.c_int), ('outdim', C.c_int), ('quantized', C.c_int),
                ('bias_corrected', C.c_int), ('timestep', C.c_double)]


class SessionStats(C.Structure):
    _fields_ = [('calls', C.c_int64), ('steps', C.c_int64), ('max_calls', C.c_int64), ('queued', C.c_int64)]


class SlicerParams(C.Structure):
    _fields_ = [('threshold_db', C.c_double), ('min_length_ms', C.c_double), ('min_interval_ms', C.c_double),
                ('hop_size_ms', C.c_double), ('max_sil_kept_ms', C.c_double)]


class SlicerFrames(C.Structure):
    _fields_ = [('threshold', C.c_float), ('hop_size', C.c_int), ('win_size', C.c_int), ('min_length', C.c_int),
                ('min_interval', C.c_int), ('max_sil_kept', C.c_int)]


class StreamInfo(C.Structure):
    _fields_ = [('received', C.c_int64), ('fixed', C.c_int64), ('held', C.c_int64)]


class ResampleWindow(C.Structure):
    _fields_ = [('x', _vp), ('x_first', C.c_longlong), ('received', C.c_longlong), ('final', C.c_int), ('y', _vp),
                ('y_first', C.c_longlong), ('t_begin', C.c_longlong), ('t_end', C.c_longlong), ('sr_orig', C.c_int),
                ('sr_new', C.c_int), ('win', _vp), ('nwin', C.c_int)]


class RmsWindow(C.Structure):
    _fields_ = [('wave', _vp), ('base', C.c_longlong), ('held', C.c_longlong), ('n_samples', C.c_longlong),
                ('frame_length', C.c_int), ('hop', C.c_int), ('rms', _vp), ('f_begin', C.c_longlong),
                ('f_end', C.c_longlong)]


class FlacRange(C.Structure):
    _fields_ = [('base', C.c_int64), ('audio_start', C.c_int64), ('end', C.c_int64), ('length', C.c_int64)]


class FlacWalk(C.Structure):
    _fields_ = [('pos', C.c_int64), ('got', C.c_int64), ('count', C.c_int64), ('strategy', C.c_int32), ('done', C.c_int32)]


class AudioMeta(C.Structure):
    _fields_ = [('container', C.c_int), ('rate', C.c_int), ('channels', C.c_int), ('bits', C.c_int), ('kind', C.c_int),
                ('min_blocksize', C.c_int), ('max_blocksize', C.c_int), ('reserved', C.c_int), ('frames', C.c_longlong),
                ('data_offset', C.c_longlong), ('data_bytes', C.c_longlong)]


class PcmItem(C.Structure):
    _fields_ = [('data', _vp), ('frames', C.c_longlong), ('channels', C.c_int), ('kind', C.c_int), ('mono', C.c_int),
                ('reserved', C.c_int), ('out', _vp)]


DOWNMIX_MONO, DOWNMIX_PLANAR, DOWNMIX_INTERLEAVED = range(3)      # SOME_DOWNMIX_*


class DownmixItem(C.Structure):
    _fields_ = [('data', _vp), ('frames', C.c_longlong), ('channels', C.c_int), ('layout', C.c_int),
                ('channel_stride', C.c_longlong), ('out', _vp)]


class DeviceAudio(C.Structure):
    _fields_ = [('data', _vp), ('device', C.c_int), ('frames', C.c_longlong), ('channels', C.c_int),
                ('channel_stride', C.c_longlong), ('frame_stride', C.c_longlong), ('sample_rate', C.c_int), ('stream', _vp)]


class Encoded(C.Structure):
    _fields_ = [('data', _vp), ('n_bytes', C.c_longlong)]


class LabelParams(C.Structure):
    _fields_ = [('slicer', C.POINTER(SlicerParams)), ('max_frames', C.c_longlong)]


class LabelReport(C.Structure):
    _fields_ = [('rows', C.c_int64), ('labelled', C.c_int64), ('missing', C.c_int64), ('groups', C.c_int64),
                ('chunks', C.c_int64), ('audio_seconds', C.c_double), ('seconds', C.c_double), ('gpu_seconds', C.c_double)]


LABEL_MISSING_FN = C.CFUNCTYPE(None, C.c_char_p, _vp)     # some_label_missing_fn


AUDIO_WAV, AUDIO_FLAC, AUDIO_AIFF = 1, 2, 3
PCM_U8, PCM_S16, PCM_S24, PCM_S32, PCM_F32, PCM_F64 = range(1, 7)
PCM_S8, PCM_S16BE, PCM_S24BE, PCM_S32BE, PCM_F32BE, PCM_F64BE, PCM_ULAW, PCM_ALAW = range(7, 15)
PCM_BYTES = {PCM_U8: 1, PCM_S16: 2, PCM_S24: 3, PCM_S32: 4, PCM_F32: 4, PCM_F64: 8, PCM_S8: 1, PCM_S16BE: 2, PCM_S24BE: 3,
             PCM_S32BE: 4, PCM_F32BE: 4, PCM_F64BE: 8, PCM_ULAW: 1, PCM_ALAW: 1}     # the bytes of one sample

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
    'some_eval_clips': (C.c_int, [C.POINTER(EvalArgs), _vp]),
    'some_slicer_rms': (C.c_int, [_vp, C.c_longlong, C.c_int, C.c_int, _vp, C.c_int, _vp]),
    'some_resample_kaiser': (C.c_int, [_vp, _vp, _vp, _vp, _vp, C.c_int, C.c_longlong, C.c_int, C.c_int, _vp, C.c_int, _vp]),
    'some_slicer_rms_window': (C.c_int, [_vp, C.c_longlong, C.c_longlong, C.c_longlong, C.c_int, C.c_int, _vp, C.c_longlong,
                                         C.c_longlong, _vp]),
    'some_resample_kaiser_window': (C.c_int, [_vp, C.c_longlong, C.c_longlong, C.c_int, _vp, C.c_longlong, C.c_longlong,
                                              C.c_longlong, C.c_int, C.c_int, _vp, C.c_int, _vp]),
    'some_resample_window_plan': (C.c_int, [C.c_longlong, C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_int,
                                            C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]),
    'some_resample_windows_bytes': (C.c_longlong, [C.c_int]),
    'some_resample_windows_pack': (C.c_int, [C.POINTER(ResampleWindow), C.c_int, _vp]),
    'some_resample_kaiser_windows': (C.c_int, [_vp, _vp, _vp]),
    'some_slicer_rms_windows_bytes': (C.c_longlong, [C.c_int]),
    'some_slicer_rms_windows_pack': (C.c_int, [C.POINTER(RmsWindow), C.c_int, _vp]),
    'some_slicer_rms_windows': (C.c_int, [_vp, _vp, _vp]),
    'some_flac_scan_workspace_bytes': (C.c_uint64, [C.c_longlong]),
    'some_flac_scan': (C.c_int, [_vp, C.c_longlong, _vp, C.c_int, _vp, C.c_int, _vp, _vp, _vp]),
    'some_flac_decode': (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, C.c_int, _vp, _vp, C.c_int, _vp, _vp]),
    'some_flac_chain': (C.c_int, [_vp, C.c_int, C.POINTER(FlacRange), C.c_int, _vp, C.c_int, _vp, _vp, C.POINTER(C.c_int)]),
    'some_flac_chain_resume': (C.c_int, [_vp, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.POINTER(FlacWalk), _vp, C.c_int,
                                         C.POINTER(C.c_int)]),
    'some_audio_info': (C.c_int, [_vp, C.c_longlong, C.POINTER(AudioMeta)]),
    'some_audio_walk_create': (C.c_int, [C.c_int, C.POINTER(_vp)]),
    'some_audio_walk_feed': (C.c_int, [_vp, _vp, C.c_longlong, C.c_int, C.POINTER(C.c_int), C.POINTER(AudioMeta),
                                       C.POINTER(C.c_longlong), C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]),
    'some_audio_walk_destroy': (C.c_int, [_vp]),
    'some_pcm_decode_bytes': (C.c_longlong, [C.c_int]),
    'some_pcm_decode_pack': (C.c_int, [C.POINTER(PcmItem), C.c_int, _vp]),
    'some_pcm_decode': (C.c_int, [_vp, _vp, _vp]),
    'some_downmix_layout': (C.c_int, [C.c_int, C.c_longlong, C.c_longlong, C.c_longlong, C.POINTER(C.c_int)]),
    'some_downmix_bytes': (C.c_longlong, [C.c_int]),
    'some_downmix_pack': (C.c_int, [C.POINTER(DownmixItem), C.c_int, _vp]),
    'some_downmix': (C.c_int, [_vp, _vp, _vp]),
    'some_midi_write': (C.c_int, [C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_double, C.c_double, _vp, C.c_size_t,
                                  C.POINTER(C.c_size_t)]),
    'some_notes_midi': (C.c_int, [_vp, C.c_int, C.c_double, C.c_double, _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    'some_session_transcribe_encoded': (C.c_int, [_vp, C.POINTER(Encoded), C.c_int, C.POINTER(SlicerParams), _vp]),
    'some_label_write': (C.c_int, [C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_double, C.c_char_p, C.c_char_p, C.c_int, _vp, C.c_size_t,
                                   C.POINTER(C.c_size_t), _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    'some_notes_label': (C.c_int, [_vp, C.c_int, C.c_double, C.c_char_p, C.c_char_p, C.c_int, _vp, C.c_size_t,
                                   C.POINTER(C.c_size_t), _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    'some_session_label_dataset': (C.c_int, [_vp, C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.POINTER(LabelParams),
                                             LABEL_MISSING_FN, _vp, C.POINTER(LabelReport)]),
    'some_row_stats': (C.c_int, [C.POINTER(RowStatsArgs), _vp]),
    'some_col_means': (C.c_int, [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, _vp]),
    'some_forward': (C.c_int, [C.POINTER(ModelC), C.POINTER(WorkspaceC), C.c_int, C.c_int, _vp, C.c_int, C.c_int, _vp,
                               C.POINTER(CalibrationC), _vp]),
    'some_forward_f32': (C.c_int, [C.POINTER(ModelF32C), C.POINTER(WorkspaceF32C), C.c_int, C.c_int, _vp, C.c_int, C.c_int,
                                   _vp]),
    'some_forward_f32_tiled': (C.c_int, [C.POINTER(ModelF32C), C.POINTER(WorkspaceF32C), C.c_int, C.c_int, _vp, C.c_int,
                                         C.c_int, _vp]),
    'some_workspace_f32_bytes': (C.c_uint64, [C.c_int, C.c_int]),
    'some_workspace_f32_carve': (C.c_int, [_vp, C.c_uint64, C.c_int, C.c_int, C.POINTER(WorkspaceF32C)]),
    'some_workspace_bytes': (C.c_uint64, [C.c_int, C.c_int, C.c_int]),
    'some_workspace_carve': (C.c_int, [_vp, C.c_uint64, C.c_int, C.c_int, C.c_int, C.POINTER(WorkspaceC)]),
    'some_profiler_create': (C.c_int, [C.c_int, C.POINTER(_vp)]),
    'some_profiler_destroy': (C.c_int, [_vp]),
    'some_profiler_reset': (C.c_int, [_vp]),
    'some_profiler_read': (C.c_int, [_vp, C.c_int, C.POINTER(ProfileRecord)]),
    'some_session_open': (C.c_int, [C.c_char_p, C.c_int, C.POINTER(_vp)]),
    'some_session_close': (C.c_int, [_vp]),
    'some_session_open_devices': (C.c_int, [C.c_char_p, C.POINTER(C.c_int), C.c_int, C.POINTER(_vp)]),
    'some_session_get_devices': (C.c_int, [_vp, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int)]),
    'some_session_get_load': (C.c_int, [_vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int, C.POINTER(C.c_int)]),
    'some_session_get_stats': (C.c_int, [_vp, C.POINTER(SessionStats)]),
    'some_shard_clips': (C.c_int, [_vp, C.c_int, C.c_int, _vp]),
    'some_session_get_info': (C.c_int, [_vp, C.POINTER(SessionInfo)]),
    'some_session_get_precision': (C.c_int, [_vp, C.POINTER(C.c_int)]),
    'some_session_transcribe': (C.c_int, [_vp, _vp, _vp, C.c_int, _vp]),
    'some_session_transcribe_sliced': (C.c_int, [_vp, _vp, C.c_longlong, C.c_int, C.POINTER(SlicerParams), _vp]),
    'some_notes_create': (C.c_int, [C.POINTER(_vp)]),
    'some_notes_destroy': (C.c_int, [_vp]),
    'some_notes_clips': (C.c_int, [_vp]),
    'some_notes_get': (C.c_int, [_vp, C.c_int, C.POINTER(C.c_int), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp),
                                 C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    'some_notes_set_frames': (C.c_int, [_vp, C.c_int]),
    'some_notes_get_frames': (C.c_int, [_vp, C.c_int, C.POINTER(C.c_int), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp),
                                        C.POINTER(_vp)]),
    'some_slicer_derive': (C.c_int, [C.c_int, C.POINTER(SlicerParams), C.POINTER(SlicerFrames)]),
    'some_slicer_ranges': (C.c_int, [_vp, C.c_int, C.c_longlong, C.POINTER(SlicerFrames), _vp, C.c_int,
                                     C.POINTER(C.c_int)]),
    'some_slicer_stream_create': (C.c_int, [C.POINTER(SlicerFrames), C.POINTER(_vp)]),
    'some_slicer_stream_feed': (C.c_int, [_vp, _vp, C.c_int, C.c_longlong, C.POINTER(_vp), C.POINTER(C.c_int)]),
    'some_slicer_stream_finish': (C.c_int, [_vp, _vp, C.c_int, C.c_longlong, C.POINTER(_vp), C.POINTER(C.c_int)]),
    'some_slicer_stream_keep_from': (C.c_int, [_vp, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong),
                                               C.POINTER(C.c_longlong)]),
    'some_slicer_stream_destroy': (C.c_int, [_vp]),
    'some_stream_open': (C.c_int, [_vp, C.c_int, C.POINTER(SlicerParams), C.POINTER(_vp)]),
    'some_stream_push': (C.c_int, [_vp, _vp, C.c_longlong, _vp]),
    'some_stream_finish': (C.c_int, [_vp, _vp]),
    'some_stream_get_info': (C.c_int, [_vp, C.POINTER(StreamInfo)]),
    'some_stream_close': (C.c_int, [_vp]),
    'some_stream_push_many': (C.c_int, [_vp, _vp, _vp, _vp, C.c_int, _vp]),
    'some_stream_open_encoded': (C.c_int, [_vp, C.POINTER(SlicerParams), C.POINTER(_vp)]),
    'some_stream_push_bytes': (C.c_int, [_vp, _vp, C.c_longlong, _vp]),
    'some_stream_push_bytes_many': (C.c_int, [_vp, _vp, _vp, _vp, C.c_int, _vp]),
    'some_stream_get_meta': (C.c_int, [_vp, C.POINTER(AudioMeta), C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]),
    'some_stream_peek': (C.c_int, [_vp, _vp]),
    'some_stream_peek_many': (C.c_int, [_vp, C.c_int, _vp]),
    'some_session_transcribe_device': (C.c_int, [_vp, C.POINTER(DeviceAudio), C.c_int, C.POINTER(SlicerParams), _vp]),
    'some_stream_push_device': (C.c_int, [_vp, C.POINTER(DeviceAudio), _vp]),
    'some_stream_push_device_many': (C.c_int, [_vp, C.POINTER(DeviceAudio), _vp, C.c_int, _vp]),
}

_lib = None


class SomeB200Error(RuntimeError):
    pass


STREAM_REFUSED = -3       # SOME_STREAM_REFUSED: a stream was refused on its content; the call's other streams completed


class StreamRefused(SomeB200Error):
    """An encoded stream was refused on its content.  `results` holds what every item of the call returned (the refused
    stream's entry holds no chunks): the other streams completed their step, and their chunks are there."""

    def __init__(self, message: str, results):
        super().__init__(message)
        self.results = results


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

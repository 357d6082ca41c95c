"""Drop-in for the reference's ``modules.rmvpe.spec.MelSpectrogram`` (modules/rmvpe/spec.py:7-72) on the sm_90a mel kernels:
same constructor, same ``forward(audio, keyshift=0, speed=1, center=True)`` contract (float32 ``[B, n_mels, T]``), including
the key-shift / speed path the binarizer uses for pitch augmentation (preprocessing/me_binarizer.py:235-247; SURVEY.md §8f-4).

keyshift = 0, speed = 1, center = True runs the fused register-FFT kernel (some_mel_logmel); everything else runs the direct-DFT
kernel (some_mel_logmel_keyshift): n_fft' = round(n_fft * 2^(keyshift / 12)) is an arbitrary integer and only bins 0..371 of
it reach the filterbank.  CUDA only — there is no CPU path."""
from __future__ import annotations

import ctypes as C
from typing import Dict

import numpy as np
import torch

from . import _lib
from .weights import mel_tables


class MelSpectrogram(torch.nn.Module):
    def __init__(self, n_mel_channels, sampling_rate, win_length, hop_length, n_fft=None, mel_fmin=0, mel_fmax=None,
                 clamp=1e-5):
        super().__init__()
        n_fft = win_length if n_fft is None else n_fft                       # spec.py:20
        if (n_mel_channels, n_fft, win_length) != (_lib.N_MELS, _lib.N_FFT, _lib.N_FFT):
            raise NotImplementedError('the mel kernels are specialised for 80 mel bands over a 2048-point STFT (all shipped configs)')
        self.n_fft, self.win_length, self.hop_length = n_fft, win_length, hop_length
        self.sampling_rate, self.n_mel_channels, self.clamp = sampling_rate, n_mel_channels, clamp
        self._cfg = {'audio_sample_rate': sampling_rate, 'win_size': n_fft, 'units_dim': n_mel_channels, 'fmin': mel_fmin,
                     'fmax': mel_fmax}
        self._tables: Dict[str, dict] = {}
        self._shift: Dict[tuple, tuple] = {}
        self.register_buffer('mel_basis', torch.from_numpy(mel_tables(self._cfg, 'cpu')['bank']))   # spec.py:29-30

    def _dev_tables(self, device):
        key = str(device)
        if key not in self._tables:
            self._tables[key] = mel_tables(self._cfg, device)
        return self._tables[key]

    def _shift_tables(self, n_fft_new: int, device):
        key = (n_fft_new, str(device))
        if key not in self._shift:
            ang = -2.0 * np.pi * np.arange(n_fft_new, dtype=np.float64) / n_fft_new
            tw = torch.from_numpy(np.stack([np.cos(ang), np.sin(ang)], axis=1).astype(np.float32)).to(device)
            win = torch.hann_window(n_fft_new, dtype=torch.float32).to(device)      # spec.py:45 (periodic)
            self._shift[key] = (tw, win)
        return self._shift[key]

    @torch.no_grad()
    def forward(self, audio: torch.Tensor, keyshift=0, speed=1, center=True) -> torch.Tensor:
        if not audio.is_cuda:
            raise _lib.SomeB200Error('some_b200.spec.MelSpectrogram runs on CUDA tensors only (sm_90a kernels, no CPU path)')
        lib = _lib.load()
        squeeze = audio.dim() == 1
        x = (audio.unsqueeze(0) if squeeze else audio).to(torch.float32).contiguous()
        b, n = x.shape
        dev = x.device
        factor = 2 ** (keyshift / 12)                                        # spec.py:39-42
        n_fft_new = int(np.round(self.n_fft * factor))
        win_new = int(np.round(self.win_length * factor))
        hop_new = int(np.round(self.hop_length * speed))
        pad_left = win_new // 2 if center else 0                             # spec.py:46-50
        pad_total = (win_new // 2 + (win_new + 1) // 2) if center else 0
        if n + pad_total < n_fft_new:
            raise RuntimeError(f'audio of {n} samples is shorter than one STFT window of {n_fft_new}')   # torch.stft would raise
        t = 1 + (n + pad_total - n_fft_new) // hop_new
        tab = self._dev_tables(dev)
        start = (torch.arange(b, dtype=torch.int64, device=dev) * n).contiguous()
        length = torch.full((b,), n, dtype=torch.int64, device=dev)
        cu = (torch.arange(b + 1, dtype=torch.int32, device=dev) * t).contiguous()
        out = torch.empty((b * t, self.n_mel_channels), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            if keyshift == 0 and hop_new == self.hop_length and center and n_fft_new == self.n_fft:
                _lib.check(lib.some_mel_logmel(x.data_ptr(), start.data_ptr(), length.data_ptr(), cu.data_ptr(), b, t,
                                               tab['mel_start'].data_ptr(), tab['mel_count'].data_ptr(),
                                               tab['mel_weights'].data_ptr(), tab['twiddle'].data_ptr(), tab['window'].data_ptr(),
                                               out.data_ptr(), None, float(self.clamp), stream), 'some_mel_logmel')
            else:
                tw, win = self._shift_tables(n_fft_new, dev)
                scale = float(self.win_length) / float(win_new) if keyshift != 0 else 1.0   # spec.py:63-68
                _lib.check(lib.some_mel_logmel_keyshift(x.data_ptr(), start.data_ptr(), length.data_ptr(), cu.data_ptr(), b, t,
                                                        n_fft_new, hop_new, pad_left, scale, tab['mel_start'].data_ptr(),
                                                        tab['mel_count'].data_ptr(), tab['mel_weights'].data_ptr(),
                                                        tw.data_ptr(), win.data_ptr(), out.data_ptr(), None, float(self.clamp),
                                                        stream), 'some_mel_logmel_keyshift')
        mel = out.view(b, t, self.n_mel_channels).transpose(1, 2)             # [B, n_mels, T] like spec.py:70-72
        return mel[0] if squeeze else mel

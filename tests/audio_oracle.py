"""CPU oracle of the audio front-end -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A torch-CPU restatement of ``np.log1p(librosa.feature.melspectrogram(y, sr=22050, n_mels=128, hop_length=128,
n_fft=512)).astype(np.float16)`` (mug/util.py:138-143) with librosa >= 0.10 defaults, in librosa's precisions:

    torch.stft in float64 (periodic Hann, center=True, pad_mode="constant") -> complex64 -> |X| in float32, squared in float32
    -> float64 dot with the Slaney filterbank -> float32 -> log1p -> float16

It needs neither librosa nor torchaudio.  librosa is not available where this project is tested, so there is no reference
golden: the filterbank and window are pinned to independent implementations (torchaudio, scipy, and a per-element restatement
in tests/test_audio.py) and the STFT is torch's own.
"""
from __future__ import annotations

import numpy as np
import torch

from mug_diffusion_b200 import audio


def log_mel(y: np.ndarray, cfg: audio.MelConfig = audio.MelConfig()) -> torch.Tensor:
    """y [n] or [B, n] float32 -> [B, n_mels, 1 + n // hop] float32 holding fp16 values"""
    y = torch.from_numpy(np.atleast_2d(np.asarray(y, dtype=np.float32))).double()
    win = torch.from_numpy(audio.hann_window(cfg.n_fft))
    spec = torch.stft(y, n_fft=cfg.n_fft, hop_length=cfg.hop_length, window=win, center=True, pad_mode="constant",
                      return_complex=True)                                     # [B, 257, T] complex128
    power = spec.to(torch.complex64).abs() ** 2                                # float32
    basis = torch.from_numpy(audio.mel_basis(cfg)).double()
    mel = torch.matmul(basis, power.double()).float()
    return torch.log1p(mel).half().float()

"""Audio front-end on the GPU: decoded samples -> the log-mel spectrogram the audio encoder reads (SURVEY §8f row N6).

Reference: ``load_audio_without_cache`` (mug/util.py:133-144) with the shipped ``common_params`` (mug_diffusion.yaml:101-105)

    np.log1p(librosa.feature.melspectrogram(y=y, sr=22050, n_mels=128, hop_length=128, n_fft=512)).astype(np.float16)

followed by webui's choice of z_length and its zero pad to 64 * z_length frames (webui.py:349-377).  librosa >= 0.10's defaults
are the contract (DESIGN §2): ``center=True`` with constant (zero) padding, a periodic Hann window, power 2, and the Slaney
filterbank (fmin 0, fmax sr/2, ``norm='slaney'``, float32 weights).  Decoding and resampling (``librosa.load``) stay with the
caller: the input is the float32 mono waveform at ``sr``.

The whole numeric pass is one kernel (csrc/melspec.cu, ``mugd_melspec``); this file builds its tables on the host -- the
fp64 window and FFT twiddles and the filterbank as CSR -- uploads them once per engine, and calls it.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import lib as L_
from .engine import View


@dataclass(frozen=True)
class MelConfig:
    """``common_params`` of configs/mug/mug_diffusion.yaml:101-105 (hop = n_fft // 4, webui.py:341).  They are dataset settings,
    not weights, so they cannot be read off a state_dict."""
    sr: int = 22050
    n_fft: int = 512
    hop_length: int = 128
    n_mels: int = 128


# ---- librosa's definitions, restated in numpy with librosa's dtypes ------------------------------------------------------
_F_SP = 200.0 / 3                 # Slaney mel scale: linear below 1 kHz, logarithmic above
_MIN_LOG_HZ = 1000.0
_MIN_LOG_MEL = _MIN_LOG_HZ / _F_SP
_LOGSTEP = np.log(6.4) / 27.0


def hz_to_mel(f) -> np.ndarray:
    """librosa.hz_to_mel(f, htk=False)"""
    f = np.asarray(f, dtype=np.float64)
    mels = f / _F_SP
    log_t = f >= _MIN_LOG_HZ
    return np.where(log_t, _MIN_LOG_MEL + np.log(np.where(log_t, f, _MIN_LOG_HZ) / _MIN_LOG_HZ) / _LOGSTEP, mels)


def mel_to_hz(m) -> np.ndarray:
    """librosa.mel_to_hz(m, htk=False)"""
    m = np.asarray(m, dtype=np.float64)
    freqs = _F_SP * m
    log_t = m >= _MIN_LOG_MEL
    return np.where(log_t, _MIN_LOG_HZ * np.exp(_LOGSTEP * (np.where(log_t, m, _MIN_LOG_MEL) - _MIN_LOG_MEL)), freqs)


def mel_basis(cfg: MelConfig = MelConfig()) -> np.ndarray:
    """librosa.filters.mel(sr, n_fft, n_mels, fmin=0, fmax=sr/2, htk=False, norm='slaney', dtype=float32): [n_mels, 1 + n_fft/2].
    The triangular ramps are float64 and stored into the float32 matrix, which is then scaled in place by the float64 Slaney
    norm 2 / (f[i+2] - f[i]) (numpy computes that product in float64 and rounds it to float32)."""
    fftfreqs = np.fft.rfftfreq(n=cfg.n_fft, d=1.0 / cfg.sr)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(0.0), hz_to_mel(cfg.sr / 2.0), cfg.n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    weights = np.zeros((cfg.n_mels, 1 + cfg.n_fft // 2), dtype=np.float32)
    for i in range(cfg.n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:cfg.n_mels + 2] - mel_f[:cfg.n_mels])
    weights *= enorm[:, np.newaxis]
    return weights


def hann_window(n_fft: int) -> np.ndarray:
    """scipy.signal.get_window('hann', n_fft, fftbins=True) (what librosa's STFT uses), float64: the symmetric window of
    n_fft + 1 points, 0.5 + 0.5 cos(x) on linspace(-pi, pi), without its last point."""
    fac = np.linspace(-np.pi, np.pi, n_fft + 1)
    w = np.zeros(n_fft + 1)
    w += 0.5 * np.cos(0 * fac)
    w += 0.5 * np.cos(1 * fac)
    return w[:-1]


def fft_twiddles(n_fft: int) -> np.ndarray:
    """[n_fft/2, 2] float64: exp(-2 pi i k / n_fft) for k < n_fft/2, (re, im) pairs."""
    ang = 2.0 * np.pi * np.arange(n_fft // 2) / n_fft
    return np.stack([np.cos(ang), -np.sin(ang)], axis=1)


def filter_csr(basis: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(band_start, band_len, weights): band m covers the contiguous bins from its first to its last non-zero weight; the weights of
    all bands are concatenated in band order."""
    starts, lens, ws = [], [], []
    for row in basis:
        nz = np.flatnonzero(row)
        s, e = (int(nz[0]), int(nz[-1]) + 1) if len(nz) else (0, 0)
        starts.append(s)
        lens.append(e - s)
        ws.append(row[s:e])
    return (np.asarray(starts, dtype=np.int32), np.asarray(lens, dtype=np.int32),
            np.concatenate(ws).astype(np.float32) if ws else np.zeros(0, np.float32))


def n_frames(n: int, hop: int) -> int:
    """STFT frames of n samples with center=True: 1 + n // hop."""
    return 1 + n // hop


def frames_per_latent(wave_levels: int, unet_levels: int) -> int:
    """mel frames per latent frame: the U-Net's first level reads the wave encoder's output at level wave_levels - unet_levels
    (unet.py:527-543), 2^(10 - 4) = 64 for the shipped model -- webui's max_audio_frame // z_length (webui.py:351)."""
    return 1 << (wave_levels - unet_levels)


def z_length_for(frames: int, per_latent: int = 64) -> int:
    """webui.py:351-353: (int(t / 64 / 32) + 1) * 32 -- a multiple of 32 that always exceeds t / 64, so a length that is already
    an exact multiple still gains 32 latent frames."""
    return (int(frames / per_latent / 32) + 1) * 32


# The longest latent a request may have.  The U-Net's S4 layers generate their convolution kernels with a one-shot DFT of length
# L_internal, which a trained checkpoint's L buffers (512 / 256 / 128 / 64) reach by doubling: at z_length 8192 every layer runs at
# L_internal 8192, the next doubling would need 16384, past what that DFT holds in shared memory.
MAX_Z_LENGTH = 8192


def max_samples(per_latent: int = 64, hop_length: int = MelConfig.hop_length) -> int:
    """the most samples an audio may have so that ``z_length_for`` stays within MAX_Z_LENGTH: 67,108,735 for the shipped model"""
    return (MAX_Z_LENGTH * per_latent - 1) * hop_length - 1


def check_z_length(z_length: int, per_latent: int = 64, cfg: MelConfig = MelConfig()) -> None:
    """Refuses a latent longer than MAX_Z_LENGTH with the audio length it corresponds to.  Host only: runs before any GPU work."""
    if int(z_length) > MAX_Z_LENGTH:
        n = max_samples(per_latent, cfg.hop_length)
        secs = (n + 1) / cfg.sr
        raise L_.MugdError(
            f"z_length {int(z_length)} is longer than the supported maximum {MAX_Z_LENGTH}: audio of at most {n:,} samples at "
            f"{cfg.sr:,} Hz ({secs:.1f} s, {int(secs) // 60} min {secs % 60:.0f} s) can be charted")


# ---- device -------------------------------------------------------------------------------------------------------------
class MelFrontEnd:
    """The kernel's tables on one engine's device, and the calls that run it."""

    def __init__(self, engine, cfg: MelConfig = MelConfig()):
        self.engine, self.cfg = engine, cfg
        dev = engine.device
        start, length, w = filter_csr(mel_basis(cfg))
        self.window = torch.from_numpy(hann_window(cfg.n_fft)).to(dev)
        self.twiddle = torch.from_numpy(fft_twiddles(cfg.n_fft)).to(dev)
        self.weights = torch.from_numpy(w).to(dev)
        self.band_start = (C.c_int32 * cfg.n_mels)(*start.tolist())
        self.band_len = (C.c_int32 * cfg.n_mels)(*length.tolist())

    def samples(self, y: Union[np.ndarray, torch.Tensor]) -> torch.Tensor:
        """[n] or [B, n] float32 samples (numpy, or torch on any device) -> contiguous [B, n] on the engine's device"""
        t = torch.from_numpy(np.ascontiguousarray(y)) if isinstance(y, np.ndarray) else y
        if t.dtype != torch.float32:
            raise TypeError(f"audio samples must be float32 (what librosa.load returns), got {t.dtype}")
        if t.dim() == 1:
            t = t[None]
        if t.dim() != 2 or t.shape[0] < 1 or t.shape[1] < 1:
            raise ValueError(f"audio samples must be [n] or [B, n] with n >= 1, got {tuple(t.shape)}")
        return t.to(self.engine.device).contiguous()

    def write_rows(self, y: torch.Tensor, rows: View, T_out: int):
        """log-mel of the [B, n] device samples y into channels-last rows [B * T_out, n_mels] at ``rows``; frames past
        1 + n // hop are zeros"""
        cfg, eng = self.cfg, self.engine
        B, n = y.shape
        assert rows.cols >= cfg.n_mels and rows.rows == B * T_out, (rows, B, T_out)
        L_.check(eng.lib.mugd_melspec(eng.handle, y.data_ptr(), n, n, B, self.window.data_ptr(), self.twiddle.data_ptr(), cfg.n_fft,
                                      self.band_start, self.band_len, self.weights.data_ptr(), cfg.n_mels, cfg.hop_length,
                                      rows.ptr, rows.ld, T_out, torch.cuda.current_stream().cuda_stream), "mugd_melspec")

    def melspectrogram(self, y) -> torch.Tensor:
        """[B, n_mels, 1 + n // hop] on the device, values representable in fp16"""
        y = self.samples(y)
        B, n = y.shape
        T, M = n_frames(n, self.cfg.hop_length), self.cfg.n_mels
        scratch = torch.empty(B * T, M, device=self.engine.device)
        rows = View(scratch.data_ptr(), M, B * T, M)
        self.write_rows(y, rows, T)
        return self.engine.rows_to_ncl(rows, B, M, T)

    def audio_features(self, y, count: int, unet_levels: int) -> Tuple[List[Optional[torch.Tensor]], int]:
        """webui.py:349-377 for one waveform: z_length, the padded mel written straight into the audio encoder's input rows, one
        encoder pass, and the level outputs expanded to ``count`` identical samples"""
        y = self.samples(y)
        if y.shape[0] != 1:
            raise ValueError(f"audio_features takes one waveform, got {y.shape[0]}")
        if count < 1:
            raise ValueError(f"count must be >= 1, got {count}")
        wcfg = self.engine.blob.meta.get("wave_cfg")
        if wcfg is None:
            raise L_.MugdError("this engine was packed without model.wave_model.* weights")
        if wcfg.n_freq != self.cfg.n_mels:
            raise L_.MugdError(f"the audio encoder reads {wcfg.n_freq} mel bands, the front-end makes {self.cfg.n_mels}")
        per = frames_per_latent(len(wcfg.channel_mult), unet_levels)
        zl = z_length_for(n_frames(y.shape[1], self.cfg.hop_length), per)
        check_z_length(zl, per, self.cfg)
        sess = self.engine.wave_session(1, per * zl)
        self.write_rows(y, sess.mel, per * zl)
        hs = sess.run()
        return [None if h is None else h.expand(count, -1, -1) for h in hs], zl


def pad_features(per_song_features: Sequence[Sequence[Optional[torch.Tensor]]]) -> Tuple[List[Optional[torch.Tensor]], List[int]]:
    """One ragged batch from several songs: ``per_song_features[k]`` is the audio-encoder list of song k (``audio_features``'s first
    result, or the wave encoder's 10-entry list), whose level-l maps are [b_k, C_l, L_k >> l] at the song's own z_length L_k.
    Returns (w, z_lengths): w holds, per entry, the songs' maps concatenated along the batch and zero-padded to Lmax >> l
    (Lmax = max L_k; entries that are None for every song stay None), and z_lengths one L_k per chart (b_k charts of song k), for
    ``sample(..., shape=(C, Lmax), z_lengths=z_lengths)``.  ValueError for songs whose lists do not line up."""
    songs = [list(f) for f in per_song_features]
    if not songs:
        raise ValueError("pad_features needs at least one song")
    n = len(songs[0])
    if any(len(f) != n for f in songs):
        raise ValueError("every song's feature list must have the same number of entries")
    used = [i for i in range(n) if any(f[i] is not None for f in songs)]
    if not used or any(f[i] is None for f in songs for i in used):
        raise ValueError("every song must carry the same feature entries")
    top = max(used, key=lambda i: songs[0][i].shape[-1])      # the full-resolution entry: its length is the song's z_length
    lens, counts = [], []
    for f in songs:
        b, Lk = int(f[top].shape[0]), int(f[top].shape[-1])
        for i in used:
            if f[i].dim() != 3 or f[i].shape[0] != b or Lk % f[i].shape[-1] or f[i].shape[1] != songs[0][i].shape[1]:
                raise ValueError(f"entry {i}: shape {tuple(f[i].shape)} does not line up with the song's {tuple(f[top].shape)}")
        lens.append(Lk)
        counts.append(b)
    Lmax = max(lens)
    w: List[Optional[torch.Tensor]] = [None] * n
    for i in used:
        ds = lens[0] // int(songs[0][i].shape[-1])
        ref = songs[0][i]
        out = torch.zeros(sum(counts), int(ref.shape[1]), Lmax // ds, dtype=ref.dtype, device=ref.device)
        row = 0
        for f, b in zip(songs, counts):
            out[row:row + b, :, :f[i].shape[-1]] = f[i]
            row += b
        w[i] = out
    return w, [Lk for Lk, b in zip(lens, counts) for _ in range(b)]

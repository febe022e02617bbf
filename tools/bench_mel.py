"""Time the audio front-end (mugd_melspec and model.model.audio_features) on the GPU.

    python tools/bench_mel.py [--iters 200] [--warmup 20] [--calls 20]

For 3- and 6-minute waveforms at B = 1 and B = 4 the mel kernel writes the padded rows audio_features uses (T_out = 64 * z_length
frames) and is timed between two CUDA events over ``--iters`` launches after ``--warmup``.  Achieved bandwidth counts the bytes
the kernel must move: the float32 samples read once and the [B * T_out, 128] float32 rows written, against the H100 SXM data
sheet's 3.35 TB/s.  Then the whole ``audio_features`` call (mel kernel + audio encoder plan + output transposes) for a 3-minute
song, and, for scale, a torch-CPU stand-in of the host mel (float32 torch.stft + mel matmul + log1p + fp16; it is NOT librosa).
Prints one JSON line per measurement with the card's name, power limit and max SM clock read in the same run.  Needs a CUDA
device: there is no CPU measurement of the kernel.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mug_diffusion_b200 import audio, synth, wave  # noqa: E402
from mug_diffusion_b200.engine import View  # noqa: E402
from mug_diffusion_b200.sampler import MugDiffusionB200  # noqa: E402

HBM_TBS = 3.35


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().split(", ") + [None] * 3)[:3] if q.returncode == 0 else (torch.cuda.get_device_name(), None, None)
    return dict(gpu=name, power_limit_w=float(power) if power else None, sm_max_mhz=int(clock) if clock else None)


def samples(B: int, n: int) -> np.ndarray:
    return (synth._rng(9, "bench_mel").random(size=(B, n), dtype=np.float32) * 1.8 - 0.9)


def events_ms(fn, iters: int) -> float:
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / iters


def cpu_standin_s(y: np.ndarray, cfg: audio.MelConfig, reps: int = 3) -> float:
    yt = torch.from_numpy(y)
    win = torch.hann_window(cfg.n_fft, periodic=True)
    basis = torch.from_numpy(audio.mel_basis(cfg))
    best = float("inf")
    for _ in range(reps):
        t = time.perf_counter()
        s = torch.stft(yt, cfg.n_fft, cfg.hop_length, window=win, center=True, pad_mode="constant", return_complex=True)
        torch.log1p(basis @ (s.abs() ** 2)).half()
        best = min(best, time.perf_counter() - t)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mel needs a CUDA device")
    info = card()
    sd = {**synth.synthetic_state_dict(512), **wave.synthetic_wave_state_dict()}
    model = MugDiffusionB200.from_state_dict(sd, z_length=512)
    fe = model.mel_frontend
    cfg = fe.cfg
    per = audio.frames_per_latent(len(wave.WaveConfig().channel_mult), model.cfg.unet.levels)
    for minutes in (3, 6):
        for B in (1, 4):
            n = minutes * 60 * cfg.sr
            T = audio.n_frames(n, cfg.hop_length)
            T_out = per * audio.z_length_for(T, per)
            y = torch.from_numpy(samples(B, n)).cuda()
            rows_t = torch.empty(B * T_out, cfg.n_mels, device="cuda")
            rows = View(rows_t.data_ptr(), cfg.n_mels, B * T_out, cfg.n_mels)
            for _ in range(a.warmup):
                fe.write_rows(y, rows, T_out)
            ms = events_ms(lambda: fe.write_rows(y, rows, T_out), a.iters)
            nbytes = 4 * B * n + 4 * B * T_out * cfg.n_mels
            print(json.dumps(dict(what="mugd_melspec", minutes=minutes, B=B, samples=n, frames=T, T_out=T_out, us=round(ms * 1e3, 2),
                                  mbytes=round(nbytes / 1e6, 2), gbs=round(nbytes / ms / 1e6, 1),
                                  share_of_hbm=round(nbytes / ms / 1e9 / HBM_TBS, 3), **info)), flush=True)
            del y, rows_t
    n = 3 * 60 * cfg.sr
    y = samples(1, n)[0]
    yd = torch.from_numpy(y).cuda()
    for what, fn in (("melspectrogram", lambda: model.model.melspectrogram(yd)),
                     ("audio_features", lambda: model.model.audio_features(yd, 1))):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in range(a.calls):
            fn()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t) / a.calls * 1e3
        print(json.dumps(dict(what=what, minutes=3, B=1, ms_per_call=round(ms, 3), **info)), flush=True)
    print(json.dumps(dict(what="cpu_standin_not_librosa", minutes=3, threads=torch.get_num_threads(),
                          s=round(cpu_standin_s(y, cfg), 3))), flush=True)


if __name__ == "__main__":
    main()

"""Per-chart seeds: which random number of a seeded request feeds what.

Every random number of a seeded request comes from libmugd's counter-based generator (``mugd_randn``, csrc/randn.cu): element e of
chart b for a (purpose, draw) pair is a fixed function of (seed_b, purpose, draw, e).  It never depends on the batch, on the chart's
place in it or on what was drawn before, so chart b of a request can be regenerated alone with seed_b, re-run with another sampler or
step count, or inpainted and remixed with its own noise.

Purposes:
    X_T     the start latent x_T (draw 0)
    STEP    a step's noise: DDIM at eta > 0, DDPM
    Q       the inpainting blend's noise (q_sample's randn_like(x0))
    ENCODE  stochastic_encode's noise (draw 0)
The draw of a step is its row in the sampler's schedule, not the loop iteration: the DDIM / DPM-Solver++ / UniPC coefficient row,
and t for DDPM.  So a chart gets the same noise alone, in any batch, with any per-chart start, under any ``timesteps=`` truncation,
with any split of the loop into calls, and in the per-step loop.  DDIM and DDPM walk their rows downwards, so their tables are
filled with draw_stride = -1.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np
import torch

from . import lib as L_

X_T, STEP, Q, ENCODE = 0, 1, 2, 3

_U64 = 1 << 64


def chart_seeds(seeds, B: int) -> list:
    """One 64-bit seed per chart: an int s gives s + b mod 2^64 for chart b (the batch convention of image UIs), a sequence must hold
    exactly B integers in [0, 2^64).  ValueError for anything else: bools, negative numbers, floats, a wrong length."""
    if isinstance(seeds, (int, np.integer)) and not isinstance(seeds, (bool, np.bool_)):
        s = int(seeds)
        if not 0 <= s < _U64:
            raise ValueError(f"seeds={s}: a seed is an integer in [0, 2^64)")
        return [(s + b) % _U64 for b in range(B)]
    if isinstance(seeds, (np.ndarray, torch.Tensor)):
        seeds = seeds.tolist()
    if not isinstance(seeds, (list, tuple)):
        raise ValueError(f"seeds={seeds!r} must be an integer or one integer per chart")
    if len(seeds) != B:
        raise ValueError(f"seeds has {len(seeds)} entries for {B} charts")
    out = []
    for s in seeds:
        if isinstance(s, (bool, np.bool_)) or not isinstance(s, (int, np.integer)) or not 0 <= int(s) < _U64:
            raise ValueError(f"seeds={list(seeds)!r}: every seed must be an integer in [0, 2^64)")
        out.append(int(s))
    return out


def seed_array(seeds: Sequence[int]) -> np.ndarray:
    """the seeds as the uint64 array mugd_randn reads"""
    return np.asarray(seeds, dtype=np.uint64)


def randn(out: torch.Tensor, seeds_dev: torch.Tensor, purpose: int, first_draw: int, n_draws: int, draw_stride: int = 1):
    """One mugd_randn launch on the current stream: out [n_draws, B, ...] (contiguous float32 on the device), row k = the normals of
    draw first_draw + draw_stride * k for the B charts of ``seeds_dev`` (a device int64 tensor holding the uint64 seeds)."""
    B = int(seeds_dev.numel())
    d = L_.Normal()
    d.out, d.seeds = out.data_ptr(), seeds_dev.data_ptr()
    d.n = out.numel() // max(1, n_draws * B)
    d.B, d.purpose, d.first_draw, d.n_draws, d.draw_stride = B, purpose, first_draw, n_draws, draw_stride
    if not out.is_contiguous() or out.dtype != torch.float32 or out.numel() != n_draws * B * d.n:
        raise ValueError(f"out must be a contiguous float32 tensor of {n_draws} x {B} rows")
    L_.check(L_.load().mugd_randn(C.byref(d), torch.cuda.current_stream().cuda_stream), "mugd_randn")


class ChartNoise:
    """The random numbers of one seeded request of ``shape`` = (B, C, L): its seeds on the device and the two ways to draw.
    ``lens`` (a ragged request: chart b valid for its first lens[b] of the L positions): chart b is drawn at its own length, as a
    [C, lens[b]] chart requested alone, and placed into the padded [C, L] slot with zeros behind it.  An element's counter is
    c * L + l, so one launch over the padded table would give a shorter chart other values."""

    def __init__(self, seeds: Sequence[int], shape, device, lens: Optional[Sequence[int]] = None):
        self.shape = tuple(int(v) for v in shape)
        if len(seeds) != self.shape[0]:
            raise ValueError(f"{len(seeds)} seeds for {self.shape[0]} charts")
        self.seeds_dev = torch.from_numpy(seed_array(seeds).view(np.int64)).to(device)
        self.device = device
        self.lens = None if lens is None else [int(v) for v in lens]

    def fill(self, table: torch.Tensor, purpose: int, first_draw: int, n_draws: int, draw_stride: int = 1):
        """rows 0 .. n_draws - 1 of a [>= n_draws, B, C, L] table: draws first_draw + draw_stride * k, one launch (one per chart when
        ragged)"""
        if self.lens is None:
            randn(table[:n_draws], self.seeds_dev, purpose, first_draw, n_draws, draw_stride)
            return
        _, C_, L = self.shape
        for b, Lb in enumerate(self.lens):
            part = torch.empty(n_draws, 1, C_, Lb, device=self.device)
            randn(part, self.seeds_dev[b:b + 1], purpose, first_draw, n_draws, draw_stride)
            table[:n_draws, b, :, :Lb].copy_(part[:, 0])
            table[:n_draws, b, :, Lb:].zero_()

    def draw(self, purpose: int, draw: int) -> torch.Tensor:
        """a fresh [B, C, L] tensor of one draw"""
        out = torch.empty(self.shape, device=self.device)
        if self.lens is None:
            randn(out, self.seeds_dev, purpose, draw, 1)
        else:
            self.fill(out[None], purpose, draw, 1)
        return out

"""CPU oracle of the chart-encoder path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Functional torch-fp32 restatements in the style of oracle/mug_oracle.py (whose leaf ops they reuse) of

    OsuManiaConvertor.objects_to_array   mug/data/convertor.py:125-129, 266-320
    Encoder.forward                      mug/firststage/autoencoder.py:244-265
    DiagonalGaussianDistribution         mug/firststage/autoencoder.py:356-387

pinned to the unmodified reference by tests/golden/encoder_L96_B2.npz and tests/golden/objects_to_array.json.gz
(tools/make_goldens.py --only encoder / objects).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from oracle import mug_oracle as orc

ENCODER_PREFIX = "model.first_stage_model.encoder."


def encoder_forward(p: orc.Params, x: torch.Tensor, cfg: dict = orc.DEFAULT_DECODER, prefix: str = ENCODER_PREFIX) -> torch.Tensor:
    """Encoder.forward  -- autoencoder.py:244-265 (built by :185-242).  x [B, x_channels, T] -> moments [B, 2 z_channels, T / 2^(levels-1)]."""
    g = cfg["num_groups"]
    nres = len(cfg["channel_mult"])
    h = orc.conv1d(p, prefix + "conv_in.", x, padding=1)
    for lvl in range(nres):
        for b in range(cfg["num_res_blocks"]):
            h = orc.resnet_block(p, f"{prefix}down.{lvl}.block.{b}.", h, g)
        if lvl != nres - 1:
            h = orc.downsample(p, f"{prefix}down.{lvl}.downsample.", h)          # models.py:84-91
    h = orc.resnet_block(p, prefix + "mid.block_1.", h, g)
    h = orc.resnet_block(p, prefix + "mid.block_2.", h, g)
    h = F.silu(orc.group_norm(p, prefix + "norm_out.", h, g))
    return orc.conv1d(p, prefix + "conv_out.", h, padding=1)


def posterior(parameters: torch.Tensor, scale: float = 1.0, noise: Optional[torch.Tensor] = None) -> dict:
    """DiagonalGaussianDistribution(parameters, scale=scale)  -- autoencoder.py:356-372, 386-387.  ``noise`` stands for the
    torch.randn(mean.shape) of sample(); without it only mode() is formed."""
    mean, logvar = torch.chunk(parameters, 2, dim=1)
    logvar = torch.clamp(logvar, -10.0, 20.0)
    std = torch.exp(0.5 * logvar)
    out = dict(mean=mean, logvar=logvar, std=std, var=torch.exp(logvar), mode=mean * scale)
    if noise is not None:
        out["sample"] = (mean + std * noise) * scale
    return out


def objects_to_array(hit_objects: Sequence[str], key_count: int, frame_ms: float, max_frame: int, rate: float = 1.0,
                     offset_ms: float = 0.0):
    """OsuManiaConvertor.objects_to_array without mirror / random column maps  -- convertor.py:266-320 with read_time :125-129.
    Returns (array [4K, max_frame] float32, valid_flag [max_frame] float64)."""

    def read_time(text):
        t = int(float(text)) / rate + offset_ms
        index = int(t / frame_ms)
        offset = (t - index * frame_ms) / frame_ms
        return int(round(t)), index, offset

    column_width = int(512 / key_count)
    array_length = min(max_frame, int(max_frame / rate))
    array = np.zeros((array_length, key_count * 4), dtype=np.float32)
    max_index = 0
    for line in hit_objects:
        params = line.split(",")
        _, start_index, start_offset = read_time(params[2])
        if start_index >= len(array):
            continue
        column = int(int(float(params[0])) / column_width)
        if column >= key_count or column < 0:
            continue
        array[start_index, column] = 1
        array[start_index, column + key_count] = start_offset
        max_index = max(start_index, max_index)
        if int(params[3]) == 128:
            _, end_index, end_offset = read_time(params[5].split(":")[0])
            if end_index >= len(array):
                end_index = len(array) - 1
                end_offset = 1
            for i in range(start_index + 1, end_index + 1):
                array[i, column + key_count * 2] = 1
            array[end_index, column + key_count * 3] = end_offset
            max_index = max(end_index, max_index)
    if len(array) < max_frame:
        array = np.concatenate([array, np.zeros((max_frame - len(array), array.shape[1]), dtype=np.float32)], axis=0)
    valid_flag = np.zeros((len(array),))
    valid_flag[:max_index] = 1
    return np.transpose(array), valid_flag


def chart_arrays(charts: List[Sequence[str]], frame_ms: float, frames: int, key_count: int = 4) -> torch.Tensor:
    """[B, 4K, frames] note arrays of a batch of charts"""
    return torch.from_numpy(np.stack([objects_to_array(c, key_count, frame_ms, frames)[0] for c in charts]))

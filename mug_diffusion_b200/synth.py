"""Seeded synthetic weights and inputs.

The shipped checkpoint is not in the reference repo (README.md:82), so every parity and benchmark run
uses random-init weights of the shipped architecture.  Values are drawn with numpy's PCG64 *uniform*
stream (exactly reproducible on any host, no transcendental in the generator) and scaled so the network
stays O(1) end to end.  Zero-initialised reference modules (zero_module, relative_position_embedding) get
non-zero values -- an all-zero residual branch would make every parity check trivially pass (SURVEY H6).

The S4 state (``C`` and the internal-length buffer ``L``) is generated in its *post-_setup_C* form, i.e.
like a checkpoint saved after the model has run once at ``z_length`` (s4.py:557-584): ``L`` holds the
per-level sequence length and ``C`` is taken as the already transformed C~.
"""
from __future__ import annotations

import math
import zlib
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from .config import DecoderConfig, EncoderConfig, ModelConfig, UNetConfig
from .netspec import decoder_param_specs, encoder_param_specs, unet_layout, unet_param_specs


def _rng(seed: int, name: str) -> np.random.Generator:
    return np.random.Generator(np.random.PCG64([seed, zlib.crc32(name.encode())]))


def _uniform(rng: np.random.Generator, shape, std: float) -> np.ndarray:
    a = math.sqrt(3.0) * std
    u = rng.random(size=shape, dtype=np.float32) if len(shape) else rng.random(dtype=np.float32)
    return ((u * 2.0 - 1.0) * a).astype(np.float32)


def _init(name: str, shape, role: str, seed: int) -> torch.Tensor:
    rng = _rng(seed, name)
    if role == "w":
        fan_in = int(np.prod(shape[1:]))
        t = _uniform(rng, shape, 1.0 / math.sqrt(fan_in))
    elif role == "b":
        t = _uniform(rng, shape, 0.05)
    elif role == "gamma":
        t = 1.0 + _uniform(rng, shape, 0.1)
    elif role == "beta":
        t = _uniform(rng, shape, 0.1)
    elif role == "relpos":
        t = _uniform(rng, shape, 0.5)
    elif role == "cemb":
        t = 1.0 + _uniform(rng, shape, 0.1)
    elif role == "s4_D":
        t = _uniform(rng, shape, 1.0)
    elif role in ("s4_C", "s4_B"):
        t = _uniform(rng, shape, 0.7)
    elif role == "s4_P":
        t = _uniform(rng, shape, 0.4)
    elif role == "s4_log_dt":
        lo, hi = math.log(0.001), math.log(0.1)
        t = (rng.random(size=shape, dtype=np.float32) * (hi - lo) + lo).astype(np.float32)
    elif role == "s4_inv_w_real":
        t = (math.log(0.5) + _uniform(rng, shape, 0.2)).astype(np.float32)
    elif role == "s4_w_imag":
        n = shape[-1]
        base = (math.pi * np.arange(n, dtype=np.float32))[None, :]
        t = (base * (1.0 + _uniform(rng, shape, 0.05)) + _uniform(rng, shape, 0.3)).astype(np.float32)
    elif role == "s4_L":
        return torch.tensor(0, dtype=torch.int64)
    else:
        raise ValueError(role)
    return torch.from_numpy(np.ascontiguousarray(t))


def synthetic_state_dict(z_length: int, cfg: Optional[ModelConfig] = None, seed: int = 0,
                         unet: bool = True, decoder: bool = True) -> Dict[str, torch.Tensor]:
    """Flat ``{reference state_dict key: tensor}`` for the U-Net and the first-stage decoder."""
    cfg = cfg or ModelConfig()
    sd: Dict[str, torch.Tensor] = {}
    if unet:
        for name, (shape, role) in unet_param_specs(cfg.unet).items():
            sd[name] = _init(name, shape, role, seed)
        for b in unet_layout(cfg.unet).blocks():
            if b.kind == "s4":
                assert z_length % b.ds == 0
                sd[b.prefix + "s4_model.kernel.kernel.L"] = torch.tensor(z_length // b.ds, dtype=torch.int64)
    if decoder:
        for name, (shape, role) in decoder_param_specs(cfg.decoder).items():
            sd[name] = _init(name, shape, role, seed)
    return sd


def synthetic_encoder_state_dict(cfg: Optional[EncoderConfig] = None, seed: int = 0) -> Dict[str, torch.Tensor]:
    """``model.first_stage_model.encoder.*`` tensors of the chart encoder, same per-name seeded initialiser as the rest."""
    return {name: _init(name, shape, role, seed) for name, (shape, role) in encoder_param_specs(cfg or EncoderConfig()).items()}


def _gauss(rng: np.random.Generator, shape) -> torch.Tensor:
    """Approximately N(0,1): Irwin-Hall sum of 12 uniforms, exact in float64 -> identical on every host."""
    acc = np.zeros(shape, dtype=np.float64)
    for _ in range(12):
        acc += rng.random(size=shape, dtype=np.float32)
    return torch.from_numpy((acc - 6.0).astype(np.float32))


def synthetic_inputs(B: int, z_length: int, cfg: Optional[ModelConfig] = None, seed: int = 1234,
                     with_uncond: bool = True) -> dict:
    """x_T ``[B,16,L]``, prompt tokens c / uc ``[B,128,21]`` and the four consumed audio feature maps
    ``[B,256,L],[B,512,L/2],[B,512,L/4],[B,512,L/8]`` (unet.py:527-543), all from seeded host streams so
    the reference, the oracle and the CUDA path share bit-identical inputs (SURVEY §8d)."""
    cfg = cfg or ModelConfig()
    u = cfg.unet
    x_T = _gauss(_rng(seed, "x_T"), (B, cfg.z_channels, z_length))
    c = _gauss(_rng(seed, "c"), (B, u.context_dim, 21))
    uc = _gauss(_rng(seed, "uc"), (1, u.context_dim, 21)).expand(B, -1, -1).contiguous()
    w: List[torch.Tensor] = []
    for lvl in range(u.levels):
        w.append(_gauss(_rng(seed, f"w{lvl}"), (B, u.audio_channels[lvl], z_length >> lvl)))
    out = dict(x_T=x_T, c=c, w=w)
    if with_uncond:
        out["uc"] = uc
    return out


def synthetic_inpainting(B: int, z_length: int, z_channels: int = 16, seed: int = 31):
    """(x0 ``[B,16,L]``, mask ``[B,1,L]``) of an inpainting request: keep the first half of every latent chart, with a soft edge
    (0.5) over the next eighth, and regenerate the rest."""
    x0 = _gauss(_rng(seed, "x0"), (B, z_channels, z_length))
    mask = torch.zeros(B, 1, z_length)
    mask[:, :, :z_length // 2] = 1.0
    mask[:, :, z_length // 2:z_length // 2 + z_length // 8] = 0.5
    return x0, mask


def wave_list(w4: Sequence[torch.Tensor]) -> List[torch.Tensor]:
    """The reference passes the 10-entry wave-encoder output list; only the last 4 are read
    (unet.py:527-543).  Pad the front with empty placeholders."""
    return [torch.empty(0)] * 6 + list(w4)

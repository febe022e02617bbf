"""Architecture description of the shipped model (configs/mug/mug_diffusion.yaml:28-58 in the reference).

Plain dataclasses; ``UNetConfig.from_module`` / ``DecoderConfig.from_module`` read the same numbers off a
live reference ``UNetModel`` / ``Decoder`` so the sampler can be built from the caller's ``model`` object.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Optional, Tuple


@dataclass(frozen=True)
class UNetConfig:
    in_channels: int = 16
    model_channels: int = 128
    out_channels: int = 16
    num_res_blocks: int = 2
    attention_resolutions: Tuple[int, ...] = (8, 4, 2)
    channel_mult: Tuple[int, ...] = (1, 2, 3, 4)
    num_heads: int = 8
    context_dim: int = 128
    audio_channels: Tuple[int, ...] = (256, 512, 512, 512)
    s4_layer: bool = True
    s4_state: int = 64          # S4 d_state; 32 conjugate-half poles are stored (s4.py:1361)
    pos_max: int = 64           # CrossAttention.position_max_embedding (attention.py:68)
    gn_groups: int = 32

    @property
    def time_embed_dim(self) -> int:
        return 4 * self.model_channels

    @property
    def levels(self) -> int:
        return len(self.channel_mult)

    def as_dict(self) -> dict:
        return dict(in_channels=self.in_channels, model_channels=self.model_channels,
                    out_channels=self.out_channels, num_res_blocks=self.num_res_blocks,
                    attention_resolutions=tuple(self.attention_resolutions),
                    channel_mult=tuple(self.channel_mult), num_heads=self.num_heads,
                    context_dim=self.context_dim, audio_channels=tuple(self.audio_channels),
                    s4_layer=self.s4_layer, s4_state=self.s4_state, pos_max=self.pos_max)

    @staticmethod
    def from_module(unet) -> "UNetConfig":
        """Read the architecture off a reference ``UNetModel`` instance (mug/diffusion/unet.py:262-333)."""
        sd = unet.state_dict()
        nlev = len(unet.channel_mult)
        audio = []
        ch = unet.model_channels
        # the first ResBlock of every down level sees ch + audio_channels[level] input channels
        idx = 1
        for level, mult in enumerate(unet.channel_mult):
            w = sd[f"input_blocks.{idx + 1}.0.in_layers.2.weight"]
            audio.append(int(w.shape[1]) - ch)
            ch = mult * unet.model_channels
            idx += 1 + unet.num_res_blocks + (1 if level != nlev - 1 else 0)
        has_s4 = any(".s4_model." in k for k in sd)
        ctx = None
        for k, v in sd.items():
            if k.endswith("attn2.to_k.weight"):
                ctx = int(v.shape[1])
                break
        return UNetConfig(in_channels=unet.in_channels, model_channels=unet.model_channels,
                          out_channels=unet.out_channels, num_res_blocks=unet.num_res_blocks,
                          attention_resolutions=tuple(int(a) for a in unet.attention_resolutions),
                          channel_mult=tuple(int(m) for m in unet.channel_mult),
                          num_heads=int(unet.num_heads), context_dim=ctx or 128,
                          audio_channels=tuple(audio), s4_layer=has_s4)


@dataclass(frozen=True)
class DecoderConfig:
    x_channels: int = 16
    middle_channels: int = 64
    z_channels: int = 16
    num_groups: int = 8
    channel_mult: Tuple[int, ...] = (1, 2, 4, 4)
    num_res_blocks: int = 1
    scale: float = 1.0          # AutoencoderKL.scale (autoencoder.py:23,76)

    def as_dict(self) -> dict:
        return dict(x_channels=self.x_channels, middle_channels=self.middle_channels,
                    z_channels=self.z_channels, num_groups=self.num_groups,
                    channel_mult=tuple(self.channel_mult), num_res_blocks=self.num_res_blocks,
                    scale=self.scale)


@dataclass(frozen=True)
class EncoderConfig(DecoderConfig):
    """The first-stage encoder (autoencoder.py:185-242).  It is built from the same ``ddconfig`` as the decoder, so it has the same
    fields: it reads [B, x_channels, 2^(levels-1) L] note arrays and writes 2 * z_channels moment channels at L."""


@dataclass(frozen=True)
class ModelConfig:
    unet: UNetConfig = field(default_factory=UNetConfig)
    decoder: DecoderConfig = field(default_factory=DecoderConfig)
    z_channels: int = 16
    timesteps: int = 1000
    linear_start: float = 1e-4
    linear_end: float = 2e-2
    encoder: Optional[EncoderConfig] = None      # None: no chart encoder (a blob with encoder weights then uses EncoderConfig())
    # the DDPM sampler's settings (diffusion.py:75-85): x_recon clamped to [-10, 10], the posterior variance's share of beta, and what
    # the U-Net predicts (only "eps" is supported)
    clip_denoised: bool = True
    v_posterior: float = 0.0
    parameterization: str = "eps"

"""The drop-in constructor reads the architecture off a live reference DDPM.  The reference's module attributes and state_dict
shapes are stored in tests/golden/ddpm_surface.json.gz (tools/make_ddpm_surface_golden.py, run against the unmodified reference);
the test rebuilds a stand-in DDPM with exactly that surface, so it runs without the reference tree."""
import gzip
import json
import os
from types import SimpleNamespace

import torch


def _standin_ddpm(surface):
    shapes = surface["state_dict"]
    zero = torch.zeros(())

    def state_dict_of(prefix):
        return lambda: {k[len(prefix):]: zero.expand(torch.Size(s)) for k, s in shapes.items() if k.startswith(prefix)}

    u = surface["unet"]
    unet = SimpleNamespace(**u, state_dict=state_dict_of("model.unet_model."))
    d = surface["decoder"]
    decoder = SimpleNamespace(num_resolutions=d["num_resolutions"], num_res_blocks=d["num_res_blocks"],
                              norm_out=SimpleNamespace(num_groups=d["norm_out_num_groups"]))
    first_stage = SimpleNamespace(decoder=decoder, scale=surface["first_stage"]["scale"])
    return SimpleNamespace(**surface["ddpm"], model=SimpleNamespace(unet_model=unet, first_stage_model=first_stage),
                           state_dict=state_dict_of(""))


def test_config_from_reference_matches_shipped_yaml(golden_dir):
    from mug_diffusion_b200 import netspec
    from mug_diffusion_b200.config import ModelConfig
    from mug_diffusion_b200.sampler import MugDiffusionB200

    with gzip.open(os.path.join(golden_dir, "ddpm_surface.json.gz"), "rt") as f:
        model = _standin_ddpm(json.load(f))
    sd, cfg = MugDiffusionB200.config_from_reference(model)
    want = ModelConfig()
    assert cfg.unet == want.unet
    assert cfg.decoder == want.decoder
    assert (cfg.z_channels, cfg.timesteps, cfg.linear_start, cfg.linear_end) == (16, 1000, 1e-4, 2e-2)
    # every tensor the packer needs is present in the reference state_dict under the names netspec generates
    need = {**netspec.unet_param_specs(cfg.unet), **netspec.decoder_param_specs(cfg.decoder)}
    assert all(k in sd and tuple(sd[k].shape) == tuple(shape) for k, (shape, _) in need.items())

"""Record what MugDiffusionB200.config_from_reference reads off a live reference DDPM into tests/golden/ddpm_surface.json.gz:
the module attributes it consults and the name / shape of every U-Net and first-stage state_dict tensor.  Runs where the reference tree exists;
tests/test_from_reference.py rebuilds a stand-in DDPM from the file, so the test itself needs no reference tree.

    MUG_REFERENCE_ROOT=<reference checkout> python tools/make_ddpm_surface_golden.py
"""
import gzip
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    import ref_shim

    model, _ = ref_shim.load_reference_model()
    unet = model.model.unet_model
    fs = model.model.first_stage_model
    dd = fs.decoder
    surface = dict(
        ddpm=dict(z_channels=int(model.z_channels), num_timesteps=int(model.num_timesteps), linear_start=float(model.linear_start),
                  linear_end=float(model.linear_end), z_length=int(model.z_length)),
        unet=dict(in_channels=int(unet.in_channels), model_channels=int(unet.model_channels), out_channels=int(unet.out_channels),
                  num_res_blocks=int(unet.num_res_blocks), attention_resolutions=[int(a) for a in unet.attention_resolutions],
                  channel_mult=[int(m) for m in unet.channel_mult], num_heads=int(unet.num_heads)),
        first_stage=dict(scale=float(fs.scale)),
        decoder=dict(num_resolutions=int(dd.num_resolutions), num_res_blocks=int(dd.num_res_blocks), norm_out_num_groups=int(dd.norm_out.num_groups)),
        # the U-Net and the first stage: the parts config_from_reference and the packer read (the audio / prompt encoders are
        # checked by their own goldens)
        state_dict={k: list(v.shape) for k, v in model.state_dict().items()
                    if k.startswith(("model.unet_model.", "model.first_stage_model."))},
    )
    out = os.path.join(ROOT, "tests", "golden", "ddpm_surface.json.gz")
    with gzip.open(out, "wt") as f:
        json.dump(surface, f, sort_keys=True, separators=(",", ":"))
    print(out, len(surface["state_dict"]), "tensors")


if __name__ == "__main__":
    main()

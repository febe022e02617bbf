"""The PLMS golden cases shared by tools/make_plms_goldens.py (which runs the UNMODIFIED reference plms.py and writes
tests/golden/plms_*.npz) and the tests that replay them.  Inputs come from the seeds of mug_diffusion_b200.synth, as for the DDIM
goldens; only reference outputs are stored."""
import numpy as np

# PLMS trajectories: (z_length, batch, S, cfg scale); intermediates recorded every LOG_EVERY_T steps
PLMS_CASES = {
    "plms_L96_B2_S10_cfg5":  dict(L=96, B=2, S=10, scale=5.0),
    "plms_L96_B1_S10_nocfg": dict(L=96, B=1, S=10, scale=1.0),
}
LOG_EVERY_T = 4


def intermediates(g: dict, key: str) -> list:
    """the golden's x_inter / pred_x0 list, in order"""
    n = sum(1 for k in g if k.startswith(key + "_"))
    return [g[f"{key}_{k}"] for k in range(n)]


def n_logged(S: int, log_every_t: int) -> int:
    """entries plms.py:134,166-168 records for an S-step request: x_T, then every step with index % log_every_t == 0 or the first"""
    total = len(range(0, 1000, 1000 // S))
    return 1 + sum(1 for i in range(total) if (total - i - 1) % log_every_t == 0 or i == 0)

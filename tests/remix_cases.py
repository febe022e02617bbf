"""The truncated-schedule golden cases shared by tools/make_remix_goldens.py (which runs the UNMODIFIED reference ddim.py / plms.py with
``timesteps=k`` and writes tests/golden/remix_*.npz) and the tests that replay them.  Inputs come from the seeds of
mug_diffusion_b200.synth, as for the full-schedule goldens; only reference outputs are stored."""
import numpy as np

# (sampler, z_length, batch, S, cfg scale, timesteps=k); intermediates recorded every LOG_EVERY_T steps
REMIX_CASES = {
    "remix_ddim_L96_B2_S10_k1":  dict(sampler="ddim", L=96, B=2, S=10, scale=5.0, k=1),     # 0 steps: x_T comes back
    "remix_ddim_L96_B2_S10_k4":  dict(sampler="ddim", L=96, B=2, S=10, scale=5.0, k=4),     # 3 steps
    "remix_ddim_L96_B2_S10_k10": dict(sampler="ddim", L=96, B=2, S=10, scale=5.0, k=10),    # 9 of the 10 steps
    "remix_ddim_L96_B2_S10_k11": dict(sampler="ddim", L=96, B=2, S=10, scale=5.0, k=11),    # k > n: n - 1 steps as well
    "remix_ddim_L96_B2_S30_k10": dict(sampler="ddim", L=96, B=2, S=30, scale=5.0, k=10),    # S = 30 has 31 timesteps
    "remix_ddim_L96_B2_S50_k29": dict(sampler="ddim", L=96, B=2, S=50, scale=5.0, k=29),    # 29 / 50 * 50 < 29: 27 steps
    "remix_plms_L96_B2_S10_k2":  dict(sampler="plms", L=96, B=2, S=10, scale=5.0, k=2),     # 1 step: the Heun step alone
    "remix_plms_L96_B2_S10_k4":  dict(sampler="plms", L=96, B=2, S=10, scale=5.0, k=4),
    "remix_plms_L96_B2_S10_k11": dict(sampler="plms", L=96, B=2, S=10, scale=5.0, k=11),
}
LOG_EVERY_T = 3


def subset_end(k, n: int) -> int:
    """the reference's slice end of ddim_timesteps for timesteps=k (ddim.py:126, plms.py:131), float expression and all"""
    return int(min(k / n, 1) * n) - 1


def ddim_timesteps(S: int, T: int = 1000) -> np.ndarray:
    """make_ddim_timesteps(uniform) (mug/diffusion/utils.py:52-63)"""
    return np.asarray(list(range(0, T, T // S))) + 1


def intermediates(g: dict, key: str) -> list:
    """the golden's x_inter / pred_x0 list, in order"""
    n = sum(1 for k in g if k.startswith(key + "_"))
    return [g[f"{key}_{k}"] for k in range(n)]

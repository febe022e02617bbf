"""Per-chart seeds without a device: the numpy oracle of mugd_randn against Random123's known answers and the normal distribution,
seeding.chart_seeds, the C descriptor checks, the header's layout, and the samplers' refusals before any GPU work."""
import ctypes as C
import os
import re
import subprocess
import types

import numpy as np
import pytest
import torch
from scipy import stats

from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import seeding, synth
from mug_diffusion_b200.config import ModelConfig
from mug_diffusion_b200.sampler import (DDIMSampler, DDPMSampler, DPMSolverSampler, PLMSSampler, UniPCSampler,
                                        register_schedule)

from seed_oracle import normals, philox4x32_10

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the oracle ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_oracle_philox_reproduces_the_random123_known_answers(ctr, key, want):
    assert tuple(int(v) for v in philox4x32_10(ctr, key)) == want


def test_oracle_normals_are_standard_normal():
    z = normals([12345], 1 << 18, seeding.STEP, 7, 1)[0, 0]
    assert abs(z.mean()) < 5 / np.sqrt(z.size)                  # 5 sigma
    assert abs(z.var() - 1) < 5 * np.sqrt(2 / z.size)
    assert stats.kstest(z, "norm").pvalue > 1e-3
    assert np.isfinite(z).all() and np.abs(z).max() < 6.0       # |z| <= sqrt(-2 ln 2^-24) = 5.77


def test_oracle_neighbouring_seeds_purposes_and_draws_are_uncorrelated():
    n = 1 << 16
    a = normals([41, 42], n, seeding.X_T, 0, 2)
    b = normals([41], n, seeding.Q, 0, 1)
    pairs = [(a[0, 0], a[0, 1]), (a[0, 0], a[1, 0]), (a[0, 0], b[0, 0])]
    for x, y in pairs:
        assert abs(np.corrcoef(x, y)[0, 1]) < 5 / np.sqrt(n)
    # the even/odd halves of one Box-Muller pair are independent too
    assert abs(np.corrcoef(a[0, 0, 0::2], a[0, 0, 1::2])[0, 1]) < 5 / np.sqrt(n / 2)


def test_oracle_layout_and_draw_stride():
    up = normals([3, 9], 10, seeding.STEP, 4, 3)
    down = normals([3, 9], 10, seeding.STEP, 6, 3, -1)
    assert up.shape == (3, 2, 10)
    np.testing.assert_array_equal(up[::-1], down)
    np.testing.assert_array_equal(normals([9], 10, seeding.STEP, 5, 1)[0, 0], up[1, 1])


# ---- chart_seeds -----------------------------------------------------------------------------------------------------------------
def test_chart_seeds_normalises():
    assert seeding.chart_seeds(7, 3) == [7, 8, 9]
    assert seeding.chart_seeds(2 ** 64 - 1, 2) == [2 ** 64 - 1, 0]
    assert seeding.chart_seeds(np.int64(5), 1) == [5]
    assert seeding.chart_seeds([4, 2 ** 64 - 1], 2) == [4, 2 ** 64 - 1]
    assert seeding.chart_seeds((1, 1), 2) == [1, 1]
    assert seeding.chart_seeds(np.array([3, 4]), 2) == [3, 4]
    assert seeding.chart_seeds(torch.tensor([5]), 1) == [5]


@pytest.mark.parametrize("seeds,B,msg", [(True, 1, "integer or one integer per chart"), (-1, 1, r"\[0, 2\^64\)"),
                                         (2 ** 64, 1, r"\[0, 2\^64\)"), (1.0, 1, "integer or one integer per chart"),
                                         ("7", 1, "integer or one integer per chart"), ([1, 2], 3, "2 entries for 3 charts"),
                                         ([1, -2], 2, "every seed"), ([1, 2.0], 2, "every seed"), ([True, 1], 2, "every seed"),
                                         ([1, 2 ** 64], 2, "every seed"), (None, 1, "integer or one integer per chart")])
def test_chart_seeds_refuses(seeds, B, msg):
    with pytest.raises(ValueError, match=msg):
        seeding.chart_seeds(seeds, B)


# ---- the C ABI -------------------------------------------------------------------------------------------------------------------
def _normal(**kw):
    d = L_.Normal()
    d.out, d.seeds, d.n, d.B, d.purpose, d.first_draw, d.n_draws, d.draw_stride = 256, 512, 1536, 2, 1, 0, 3, 1
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("kw,msg", [
    (dict(out=None), "out and seeds must be given"), (dict(seeds=None), "out and seeds must be given"),
    (dict(B=0), "must be at least 1"), (dict(n=0), "must be at least 1"), (dict(n_draws=0), "must be at least 1"),
    (dict(first_draw=-1), "must not be negative"), (dict(purpose=-1), "must not be negative"),
    (dict(draw_stride=0), "draw_stride=0"), (dict(draw_stride=2), "draw_stride=2"),
    (dict(first_draw=2 ** 31 - 2, n_draws=3), r"leave \[0, 2\^31\)"), (dict(first_draw=1, n_draws=3, draw_stride=-1), r"leave \[0, 2\^31\)"),
    (dict(n=(1 << 34) + 1), "past 2\\^32"),
])
def test_randn_refuses_bad_descriptors_without_a_device(kw, msg):
    lib = L_.load()
    assert lib.mugd_randn(C.byref(_normal(**kw)), None) == 1
    assert re.search(msg, lib.mugd_last_error().decode())
    assert lib.mugd_randn(None, None) == 1 and "null descriptor" in lib.mugd_last_error().decode()


def test_header_declares_mugd_randn_outside_the_op_union():
    hdr = open(os.path.join(ROOT, "include", "mugd.h")).read()
    assert "int  mugd_randn(const mugd_normal* d, void* stream);" in hdr
    assert "mugd_randn" in L_.EXPORTED_SYMBOLS and L_.ABI_VERSION == 13
    lib = L_.load()
    assert lib.mugd_abi_version() == 13
    sizes = (C.c_int32 * 13)()
    assert lib.mugd_abi_sizes(sizes, 13) == 0 and sizes[0] == C.sizeof(L_.Op) == 256


def test_ctypes_normal_matches_the_c_layout(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "mugd.h"\nint main(void) {\n'
                   '  printf("%zu", sizeof(mugd_normal));\n'
                   + "".join(f'  printf(" %zu", offsetof(mugd_normal, {f}));\n' for f, _ in L_.Normal._fields_)
                   + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-o", str(exe), str(src), "-I" + os.path.join(ROOT, "include")], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(L_.Normal)] + [getattr(L_.Normal, f).offset for f, _ in L_.Normal._fields_]


def test_c_host_compiles_against_the_header(tmp_path):
    from mug_diffusion_b200 import build
    build.build()
    host = os.path.join(ROOT, "examples", "host_c")
    r = subprocess.run(["gcc", "-O2", "-Wall", "-Werror", "-fsyntax-only", os.path.join(host, "sample_host.c"), "-I/usr/local/cuda/include"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


# ---- the samplers refuse before any GPU work -------------------------------------------------------------------------------------
class _NoGpu:
    def __getattr__(self, name):
        raise AssertionError(f"engine.{name} used before the refusal")


def _cpu(cls):
    s = object.__new__(cls)
    sch = register_schedule()
    s.model = types.SimpleNamespace(engine=_NoGpu(), z_channels=16, z_length=96, num_timesteps=1000, cfg=ModelConfig(),
                                    clip_denoised=True, **sch)
    s.ddpm_num_timesteps, s.device, s.last_launches_per_step = 1000, torch.device("cpu"), 0
    return s


def _req(**kw):
    inp = synth.synthetic_inputs(2, 96)
    out = dict(c=inp["c"], w=inp["w"], batch_size=2, shape=(16, 96), verbose=False, unconditional_guidance_scale=5.0,
               unconditional_conditioning=inp["uc"])
    out.update(kw)
    return out


X0 = torch.zeros(2, 16, 96)
MASK = torch.ones(2, 1, 96)
BAD_SEEDS = [([1], "1 entries for 2 charts"), (-1, r"\[0, 2\^64\)"), (1.5, "integer or one integer"), (True, "integer or one integer"),
             ([1, 2 ** 64], "every seed")]
CALLS = {
    "ddim": lambda s, **kw: _cpu(DDIMSampler).sample(S=10, **_req(**kw)),
    "ddim_eta": lambda s, **kw: _cpu(DDIMSampler).sample(S=10, eta=1.0, mask=MASK, x0=X0, **_req(**kw)),
    "plms": lambda s, **kw: _cpu(PLMSSampler).sample(S=10, **_req(**kw)),
    "ddpm": lambda s, **kw: _cpu(DDPMSampler).sample(**_req(**kw)),
    "dpm": lambda s, **kw: _cpu(DPMSolverSampler).sample(S=10, **_req(**kw)),
    "dpm_inpaint": lambda s, **kw: _cpu(DPMSolverSampler).inpaint(S=10, mask=MASK, x0=X0, **_req(**kw)),
    "unipc": lambda s, **kw: _cpu(UniPCSampler).sample(S=10, **_req(**kw)),
    "unipc_inpaint": lambda s, **kw: _cpu(UniPCSampler).inpaint(S=10, mask=MASK, x0=X0, **_req(**kw)),
}


@pytest.mark.parametrize("which", sorted(CALLS))
@pytest.mark.parametrize("seeds,msg", BAD_SEEDS, ids=[f"bad{i}" for i in range(len(BAD_SEEDS))])
def test_samplers_refuse_bad_seeds_before_any_gpu_work(which, seeds, msg):
    with pytest.raises(ValueError, match=msg):
        CALLS[which](None, seeds=seeds)


@pytest.mark.parametrize("which", ["ddim", "ddim_eta", "plms"])
@pytest.mark.parametrize("kw,msg", [(dict(noise_dropout=0.1), "noise_dropout=0.1"), (dict(match_reference_rng=True), "match_reference_rng")])
def test_seeds_refuse_noise_dropout_and_match_reference_rng(which, kw, msg):
    with pytest.raises(ValueError, match=msg):
        CALLS[which](None, seeds=7, **kw)


def test_stochastic_encode_refuses_noise_with_seeds_and_bad_seeds():
    from mug_diffusion_b200 import dpm_solver, unipc
    from mug_diffusion_b200.sampler import alphas_cumprod_f64
    acp = alphas_cumprod_f64(ModelConfig())
    ddim = _cpu(DDIMSampler)
    ddim.make_schedule(10, verbose=False)
    encs = [lambda **kw: ddim.stochastic_encode(X0, torch.tensor([1, 2]), **kw),
            lambda **kw: _cpu(DPMSolverSampler).stochastic_encode(X0, 3, dpm_solver.multistep_schedule(acp, 10, 2), **kw),
            lambda **kw: _cpu(UniPCSampler).stochastic_encode(X0, 3, unipc.multistep_schedule(acp, 10, 2), **kw)]
    for enc in encs:
        with pytest.raises(ValueError, match="not both"):
            enc(noise=torch.zeros_like(X0), seeds=1)
        with pytest.raises(ValueError, match="3 entries for 2 charts"):
            enc(seeds=[1, 2, 3])


def test_seeded_requests_reach_the_engine():
    """valid seeds pass every check: the request then needs the engine (here: the stand-in raises)"""
    for which in ("ddim", "ddim_eta", "ddpm", "dpm", "unipc_inpaint"):
        with pytest.raises(AssertionError, match="engine"):
            CALLS[which](None, seeds=[3, 2 ** 64 - 1])

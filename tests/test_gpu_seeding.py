"""Per-chart seeds on the GPU: mugd_randn against the float64 oracle and bit-invariant under batch, draw range, table size and
alignment; seeded deterministic requests equal the same request from x_T = chart_noise(seeds); every stochastic flow's device loop
equals its per-step loop bit for bit, repeats itself and leaves torch's generator alone; chart b of a seeded batch is the B = 1
request with seed s_b; a seeded bundle run by the C host reproduces the Python run."""
import os
import subprocess

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from gpu_util import rel_err  # noqa: E402
from seed_oracle import normals  # noqa: E402
from mug_diffusion_b200 import sampler as sampler_mod  # noqa: E402
from mug_diffusion_b200 import seeding, synth  # noqa: E402
from mug_diffusion_b200.sampler import (DDIMSampler, DDPMSampler, DPMSolverSampler, MugDiffusionB200, PLMSSampler,  # noqa: E402
                                        UniPCSampler)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_DIR = os.path.join(ROOT, "examples", "host_c")
_models = {}


def model_for(L):
    if L not in _models:
        _models.clear()
        _models[L] = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L)
    return _models[L]


def table(seeds, n, purpose, first_draw, n_draws, draw_stride=1, offset=0):
    """mugd_randn into a fresh buffer (starting ``offset`` floats in, to leave the 16-byte store path)"""
    sd = torch.from_numpy(seeding.seed_array(seeds).view(np.int64)).cuda()
    buf = torch.full((offset + n_draws * len(seeds) * n,), float("nan"), device="cuda")
    out = buf[offset:]
    seeding.randn(out, sd, purpose, first_draw, n_draws, draw_stride)
    return out.view(n_draws, len(seeds), n)


def request(B, L, seed=1234, cfg=True):
    inp = synth.synthetic_inputs(B, L, seed=seed)
    kw = dict(c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, shape=(16, L), verbose=False)
    if cfg:
        kw.update(unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    return kw


def one_chart(kw, b):
    """the B = 1 request of chart b of ``kw``"""
    out = dict(kw, c=kw["c"][b:b + 1], w=[w[b:b + 1] for w in kw["w"]], batch_size=1)
    if "unconditional_conditioning" in kw:
        out["unconditional_conditioning"] = kw["unconditional_conditioning"][b:b + 1]
    for k in ("mask", "x0"):
        if k in kw:
            out[k] = kw[k][b:b + 1] if kw[k].shape[0] > 1 else kw[k]
    return out


# ---- the generator -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seeds,n,purpose,first,count,stride", [
    ([0], 1536, seeding.X_T, 0, 1, 1), ([7, 8, 2 ** 64 - 1], 1531, seeding.STEP, 3, 5, 1), ([12345], 7, seeding.Q, 999, 4, -1),
    ([1, 2], 1, seeding.ENCODE, 0, 3, 1), ([2 ** 40 + 5] * 2, 16 * 512, seeding.STEP, 2 ** 31 - 1, 2, -1), ([3], 4097, 9, 1000, 1, 1)])
def test_randn_matches_the_float64_oracle(seeds, n, purpose, first, count, stride):
    got = table(seeds, n, purpose, first, count, stride).cpu().double().numpy()
    want = normals(seeds, n, purpose, first, count, stride)
    err = np.abs(got - want) / (1 + np.abs(want))
    print(f"max |z - z64| / (1 + |z|) = {err.max():.3e} over {got.size} values")
    assert np.isfinite(got).all() and err.max() <= 2e-6


def test_randn_bits_do_not_depend_on_batch_draw_range_table_size_or_alignment():
    seeds, n = [11, 12, 13, 14], 16 * 96
    full = table(seeds, n, seeding.STEP, 0, 10)
    for b, s in enumerate(seeds):                                            # a B = 4 table is four B = 1 tables
        assert torch.equal(full[:, b], table([s], n, seeding.STEP, 0, 10)[:, 0])
    assert torch.equal(table(seeds, n, seeding.STEP, 3, 2), full[3:5])       # draws [3, 5) are rows 3-4 of [0, 10)
    assert torch.equal(table(seeds, n, seeding.STEP, 9, 10, -1), full.flip(0))
    assert torch.equal(table(seeds, n, seeding.STEP, 0, 10, offset=1), full)  # scalar stores
    assert torch.equal(table(seeds[1:3], n - 3, seeding.STEP, 0, 10), full[:, 1:3, :n - 3])
    # every table size the samplers use: one step, a stretch, a STAGE_TABLE_BYTES table of B = 4 at L = 512
    per_call = sampler_mod.STAGE_TABLE_BYTES // (4 * 4 * 16 * 512)
    big = table(seeds, 16 * 512, seeding.Q, 0, per_call)
    for first, count in ((0, 1), (per_call - 1, 1), (17, 50)):
        assert torch.equal(table(seeds, 16 * 512, seeding.Q, first, count), big[first:first + count])


def test_randn_touches_no_torch_generator_state():
    before = torch.cuda.get_rng_state()
    table([5], 100, seeding.X_T, 0, 1)
    assert torch.equal(torch.cuda.get_rng_state(), before)


# ---- deterministic samplers: a seed is just an x_T -----------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["ddim", "plms", "dpm", "unipc"])
def test_seeded_deterministic_request_is_the_request_from_chart_noise(kind):
    L, B = 96, 2
    m = model_for(L)
    seeds = [5, 2 ** 63 + 7]
    run = {"ddim": lambda **kw: DDIMSampler(m).sample(S=10, eta=0.0, **kw),
           "plms": lambda **kw: PLMSSampler(m).sample(S=10, **kw),
           "dpm": lambda **kw: DPMSolverSampler(m).sample(S=10, **kw),
           "unipc": lambda **kw: UniPCSampler(m).sample(S=6, **kw)}[kind]
    kw = request(B, L)
    state = torch.cuda.get_rng_state()
    z, inter = run(seeds=seeds, **kw)
    assert torch.equal(torch.cuda.get_rng_state(), state)
    x_T = m.chart_noise(seeds, (B, 16, L))
    assert torch.equal(inter["x_inter"][0], x_T)
    assert torch.equal(m.chart_noise(seeds, (16, L)), x_T) and torch.equal(m.chart_noise(5, (16, L)), x_T[:1])
    z2, _ = run(x_T=x_T, **kw)
    assert torch.equal(z, z2)
    z3, _ = run(x_T=x_T, seeds=[1, 2], **kw)                                # x_T wins; the seeds drive nothing else here
    assert torch.equal(z, z3)


# ---- stochastic flows: device loop == per-step loop, repeatable, generator untouched -------------------------------------------
def _flows(m, L, B):
    x0, mask = synth.synthetic_inpainting(B, L)
    x0, mask = x0.cuda(), mask.cuda()
    dpm, uni = DPMSolverSampler(m), UniPCSampler(m)
    return {
        "ddim_eta1": lambda cb, **kw: DDIMSampler(m).sample(S=10, eta=1.0, callback=cb, **kw),
        "ddim_inpaint": lambda cb, **kw: DDIMSampler(m).sample(S=10, eta=0.0, mask=mask, x0=x0, callback=cb, **kw),
        "ddim_inpaint_eta1": lambda cb, **kw: DDIMSampler(m).sample(S=10, eta=1.0, mask=mask, x0=x0, callback=cb, log_every_t=3, **kw),
        "dpm_inpaint": lambda cb, **kw: dpm.inpaint(S=10, mask=mask, x0=x0, callback=cb, **kw),
        "unipc_inpaint": lambda cb, **kw: uni.inpaint(S=6, mask=mask, x0=x0, callback=cb, **kw),
        "plms_inpaint": lambda cb, **kw: PLMSSampler(m).sample(S=10, mask=mask, x0=x0, callback=cb, **kw),
    }


@pytest.mark.parametrize("flow", ["ddim_eta1", "ddim_inpaint", "ddim_inpaint_eta1", "dpm_inpaint", "unipc_inpaint", "plms_inpaint"])
def test_seeded_stochastic_flow_device_loop_equals_per_step_loop(flow, monkeypatch):
    L, B = 96, 2
    m = model_for(L)
    run = _flows(m, L, B)[flow]
    kw = request(B, L)
    state = torch.cuda.get_rng_state()
    z_dev, inter = run(None, seeds=[21, 22], **kw)
    z_again, _ = run(None, seeds=[21, 22], **kw)
    z_step, inter_step = run(lambda i: None, seeds=[21, 22], **kw)
    monkeypatch.setattr(sampler_mod, "STAGE_TABLE_BYTES", 3 * 4 * B * 16 * L)     # split the stretches into 3-step tables
    z_split, _ = run(None, seeds=[21, 22], **kw)
    assert torch.equal(torch.cuda.get_rng_state(), state)
    assert torch.equal(z_dev, z_again) and torch.equal(z_dev, z_step) and torch.equal(z_dev, z_split)
    for a, b in zip(inter["x_inter"], inter_step["x_inter"]):
        assert torch.equal(a, b)
    z_other, _ = run(None, seeds=[21, 23], **kw)                              # another seed, another chart
    assert not torch.equal(z_other[1], z_dev[1])


def test_seeded_ddpm_device_loop_equals_per_step_loop(monkeypatch):
    L, B = 96, 2
    m = model_for(L)
    kw = request(B, L)
    state = torch.cuda.get_rng_state()
    s = DDPMSampler(m)
    z_dev, _ = s.sample(seeds=9, log_every_t=250, **kw)
    z_step, _ = s.sample(seeds=9, log_every_t=250, callback=lambda i: None, **kw)
    monkeypatch.setattr(sampler_mod, "STAGE_TABLE_BYTES", 37 * 4 * B * 16 * L)
    z_split, _ = s.sample(seeds=[9, 10], log_every_t=250, **kw)
    assert torch.equal(torch.cuda.get_rng_state(), state)
    assert torch.equal(z_dev, z_step) and torch.equal(z_dev, z_split)
    assert torch.isfinite(z_dev).all()


@pytest.mark.parametrize("kind", ["ddim", "dpm", "unipc"])
def test_seeded_stochastic_encode_and_decode(kind):
    L, B = 96, 2
    m = model_for(L)
    x0, _ = synth.synthetic_inpainting(B, L)
    x0 = x0.cuda()
    kw = request(B, L)
    del kw["batch_size"], kw["shape"], kw["verbose"]
    if kind == "ddim":
        s = DDIMSampler(m)
        s.make_schedule(10, verbose=False)
        t = torch.tensor([3, 7])
        enc = lambda **a: s.stochastic_encode(x0, t, **a)
        dec = lambda z: s.decode(z, t_start=[4, 8], **kw)
    else:
        s = DPMSolverSampler(m) if kind == "dpm" else UniPCSampler(m)
        sched = s.make_dpm_schedule(10) if kind == "dpm" else s.make_unipc_schedule(6)
        enc = lambda **a: s.stochastic_encode(x0, [3, 5], sched, **a)
        dec = lambda z: s.decode(z, t_start=[3, 5], sched=sched, **kw)
    state = torch.cuda.get_rng_state()
    z = enc(seeds=[4, 5])
    assert torch.equal(z, enc(seeds=4))
    assert torch.equal(z, enc(noise=seeding.ChartNoise([4, 5], x0.shape, "cuda").draw(seeding.ENCODE, 0)))
    assert torch.equal(z[1:], enc(seeds=[6, 5])[1:]) and not torch.equal(z[0], enc(seeds=[6, 5])[0])
    out = dec(z)
    assert torch.equal(out, dec(enc(seeds=[4, 5])))
    assert torch.equal(torch.cuda.get_rng_state(), state)


# ---- one chart of a batch, regenerated alone -----------------------------------------------------------------------------------
def test_chart_of_a_seeded_batch_is_the_single_chart_request():
    L, B = 96, 4
    m = model_for(L)
    kw = request(B, L)
    x0, mask = synth.synthetic_inpainting(B, L)
    x0, mask = x0.cuda(), mask.cuda()
    seed = 1000
    worst = {}
    runs = {
        "ddim_eta1": lambda **a: DDIMSampler(m).sample(S=10, eta=1.0, **a)[0],
        "unipc": lambda **a: UniPCSampler(m).sample(S=6, **a)[0],
        "ddim_inpaint_eta1": lambda **a: DDIMSampler(m).sample(S=10, eta=1.0, **a)[0],
    }
    for name, run in runs.items():
        extra = dict(mask=mask, x0=x0) if "inpaint" in name else {}
        z = run(seeds=seed, **kw, **extra)
        for b in range(B):
            one = one_chart(dict(kw, **extra), b)
            zb = run(seeds=[seed + b], **one)
            worst[name] = max(worst.get(name, 0.0), rel_err(zb[0], z[b]))
    # remix with per-chart strengths: DPM-Solver++ encode + decode
    dpm = DPMSolverSampler(m)
    sched = dpm.make_dpm_schedule(10)
    strengths = [2, 4, 7, 10]
    dkw = {k: v for k, v in kw.items() if k not in ("batch_size", "shape", "verbose")}
    z = dpm.decode(dpm.stochastic_encode(x0, strengths, sched, seeds=seed), t_start=strengths, sched=sched, **dkw)
    for b in range(B):
        one = {k: v for k, v in one_chart(kw, b).items() if k not in ("batch_size", "shape", "verbose")}
        zb = dpm.decode(dpm.stochastic_encode(x0[b:b + 1], [strengths[b]], sched, seeds=seed + b), t_start=[strengths[b]], sched=sched,
                        **one)
        worst["dpm_remix"] = max(worst.get("dpm_remix", 0.0), rel_err(zb[0], z[b]))
    print("chart b of B = 4 vs the B = 1 request, max rel_err:", worst)
    assert all(v < 1e-4 for v in worst.values()), worst


# ---- the C host ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("eta,inpaint", [(0.0, False), (1.0, True)])
def test_c_host_runs_a_seeded_bundle(tmp_path, eta, inpaint):
    from mug_diffusion_b200.bundle import export_bundle
    L, B, S = 96, 2, 10
    m = model_for(L)
    inp = synth.synthetic_inputs(B, L)
    x0, mask = synth.synthetic_inpainting(B, L)
    out = str(tmp_path / "bundle")
    state = torch.cuda.get_rng_state()
    res = export_bundle(m, inp, S, 5.0, out, eta=eta, inpaint=(x0, mask) if inpaint else None, seeds=[7, 8])
    assert torch.equal(torch.cuda.get_rng_state(), state)
    extra = dict(mask=mask.cuda(), x0=x0.cuda()) if inpaint else {}
    z, _ = DDIMSampler(m).sample(S=S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, eta=eta,
                                 shape=(16, L), unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda(),
                                 seeds=[7, 8], **extra)
    assert rel_err(res["z"], z) < 1e-5
    manifest = open(os.path.join(out, "manifest.txt")).read()
    assert "seeds seeds.bin 2" in manifest and "randn in_x 0 0 1 1 2 1536" in manifest
    assert not os.path.exists(os.path.join(out, "in_x.bin")) and not os.path.exists(os.path.join(out, "in_noise.bin"))
    if inpaint:
        assert "randn in_qnoise 2 9 10 -1 2 1536" in manifest and "randn in_noise 1 9 10 -1 2 1536" in manifest
    _models.clear()
    del m
    torch.cuda.empty_cache()
    subprocess.run(["make", "-C", HOST_DIR], check=True, capture_output=True)
    r = subprocess.run([os.path.join(HOST_DIR, "sample_host"), out], capture_output=True, text=True, timeout=600)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count(" OK") == 2 and "drew in_x" in r.stdout
    r = subprocess.run([os.path.join(HOST_DIR, "sample_host"), out, "--seed", "100"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert " OK" not in r.stdout and "not compared: charts drawn from --seed 100" in r.stdout

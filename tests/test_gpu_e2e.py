"""End-to-end parity on the GPU through the reference-shaped surface (DDIMSampler.sample,
model.model.forward, model.model.decode), against (a) the committed outputs of the UNMODIFIED reference
(tests/golden/, made by tools/make_goldens.py) and (b) the CPU oracle on the same seeded inputs.

Stated fp32 tolerances (max-abs error relative to the tensor's max magnitude):
  one U-Net eval                      <= 1e-4
  10-step DDIM latent / decoder logits<= 1e-3
  50-step CFG-5 trajectory (L=512)    <= 5e-3   (random-weight CFG trajectory amplifies rounding noise)
  note on/off masks: identical except where the REFERENCE logit magnitude is below the logit tolerance.
The U-Net goldens, the small and ragged lengths and the two L=96 DDIM trajectories also run on a `simt` engine (every GEMM on the
exact-fp32 FFMA kernel) at the same tolerances.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

import golden_cases as gc  # noqa: E402
from gpu_util import rel_err  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.sampler import DDIMSampler, MugDiffusionB200  # noqa: E402
from oracle import mug_oracle as orc  # noqa: E402

_models = {}


def model_for(L, impl="auto"):
    if (L, impl) not in _models:
        _models.clear()                      # one resident model at a time
        _models[L, impl] = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L, gemm_impl=impl)
    return _models[L, impl]


def with_simt(cases, ids):
    """each case on the default engine (its id unchanged) and on a `simt` engine (id + "-simt"); cases: tuples of arguments"""
    return [pytest.param(*c, "auto", id=i) for c, i in zip(cases, ids)] + [pytest.param(*c, "simt", id=f"{i}-simt")
                                                                           for c, i in zip(cases, ids)]


@pytest.mark.parametrize("name,impl", with_simt([(n,) for n in gc.UNET_CASES], list(gc.UNET_CASES)))
def test_unet_forward_vs_reference_golden(name, impl, golden_dir):
    case = gc.UNET_CASES[name]
    m = model_for(case["L"], impl)
    inp = synth.synthetic_inputs(case["B"], case["L"])
    eps = m.model.forward(inp["x_T"].cuda(), torch.tensor(case["t"]).cuda(), inp["c"].cuda(), synth.wave_list([w.cuda() for w in inp["w"]]))
    gold = gc.load_golden(os.path.join(golden_dir, name + ".npz"))["eps"]
    assert eps.shape == gold.shape
    assert rel_err(eps, gold) < 1e-4


def test_unet_forward_lengthens_s4_state_like_reference(golden_dir):
    """weights persisted at z_length 48, request at 96: every S4 layer must double its C~ (s4.py:557-584)"""
    _models.clear()
    m = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(48), z_length=96)
    inp = synth.synthetic_inputs(2, 96)
    eps = m.model.forward(inp["x_T"].cuda(), torch.tensor([981, 1]).cuda(), inp["c"].cuda(), [w.cuda() for w in inp["w"]])
    gold = gc.load_golden(os.path.join(golden_dir, "unet_L96_from48.npz"))["eps"]
    assert rel_err(eps, gold) < 1e-4
    key = "model.unet_model.input_blocks.2.1.s4_model.kernel.kernel.L"
    assert m.engine.s4_L[key] == 96
    # the lengthened C~ lives in THIS engine's device weights; the shared host blob (and its length record) is untouched, so a second
    # engine built from the same blob lengthens again and reproduces the result instead of pairing the short C~ with the long L
    assert m.engine.blob.meta[key] == 48
    m2 = MugDiffusionB200(None, m.cfg, z_length=96, blob=m.engine.blob)
    eps2 = m2.model.forward(inp["x_T"].cuda(), torch.tensor([981, 1]).cuda(), inp["c"].cuda(), [w.cuda() for w in inp["w"]])
    assert rel_err(eps2, gold) < 1e-4 and m2.engine.s4_L[key] == 96


def test_unet_forward_vs_oracle_other_batch():
    """a shape with no golden: B=3, L=160, distinct timesteps -> live oracle"""
    L, B = 160, 3
    sd = synth.synthetic_state_dict(L)
    m = model_for(L)
    inp = synth.synthetic_inputs(B, L, seed=99)
    t = torch.tensor([7, 480, 999])
    with torch.no_grad():
        ref = orc.unet_forward(sd, inp["x_T"], t, inp["c"], inp["w"])
    eps = m.model.forward(inp["x_T"].cuda(), t.cuda(), inp["c"].cuda(), [w.cuda() for w in inp["w"]])
    assert rel_err(eps, ref) < 1e-4


@pytest.mark.parametrize("L,B,impl", with_simt([(32, 3), (224, 2), (64, 5)], ["32-3", "224-2", "64-5"]))
def test_unet_forward_small_and_ragged_lengths(L, B, impl):
    """shortest legal chart (L=32 -> level lengths 32/16/8/4), lengths that are not multiples of the 128-row GEMM tile
    (224 -> 224/112/56/28: partial tiles and several samples per tile), odd batch: live oracle"""
    sd = synth.synthetic_state_dict(L)
    m = model_for(L, impl)
    inp = synth.synthetic_inputs(B, L, seed=7 + L)
    t = torch.arange(B) * 211 + 3
    with torch.no_grad():
        ref = orc.unet_forward(sd, inp["x_T"], t, inp["c"], inp["w"])
        zref = orc.decoder_forward(sd, inp["x_T"])
    eps = m.model.forward(inp["x_T"].cuda(), t.cuda(), inp["c"].cuda(), [w.cuda() for w in inp["w"]])
    assert rel_err(eps, ref) < 1e-4
    assert rel_err(m.model.decode(inp["x_T"].cuda()), zref) < 1e-4


def _notes_match(logits, ref_logits, tol_abs):
    mine, ref = orc.notes_from_logits(logits.cpu()), orc.notes_from_logits(ref_logits)
    flips = mine != ref
    ref8 = torch.cat([ref_logits[:, 0:4], ref_logits[:, 8:12]], dim=1)
    return int(flips.sum()), bool((ref8[flips].abs() <= tol_abs).all())


_DDIM = [("ddim_L96_B1_S10_nocfg", 1e-3), ("ddim_L96_B2_S10_cfg5", 1e-3), ("ddim_L512_B1_S50_cfg5", 5e-3)]


# the 50-step L=512 trajectory on the default engine only
@pytest.mark.parametrize("name,tol,impl", with_simt(_DDIM, [f"{n}-{t}" for n, t in _DDIM])[:-1])
def test_ddim_sample_and_decode_vs_reference_golden(name, tol, impl, golden_dir):
    case = gc.DDIM_CASES[name]
    m = model_for(case["L"], impl)
    m.z_length = case["L"]
    inp = synth.synthetic_inputs(case["B"], case["L"])
    sampler = DDIMSampler(m)
    preds = []
    z, inter = sampler.sample(S=case["S"], c=inp["c"].cuda(), w=synth.wave_list([w.cuda() for w in inp["w"]]), batch_size=case["B"],
                              shape=None, verbose=False, x_T=inp["x_T"].cuda(), eta=0.0,
                              unconditional_guidance_scale=case["scale"], unconditional_conditioning=inp["uc"].cuda(),
                              img_callback=lambda p, i: preds.append(p.clone()))
    logits = m.model.decode(z)
    gold = gc.load_golden(os.path.join(golden_dir, name + ".npz"))
    assert len(preds) == case["S"] and len(inter["x_inter"]) == 3
    assert rel_err(preds[0], gold["pred_x0_first"]) < 1e-4
    assert rel_err(z, gold["z"]) < tol
    assert rel_err(logits, gold["logits"]) < tol
    nflips, ok = _notes_match(logits, gold["logits"], tol * float(gold["logits"].abs().max()))
    assert ok, f"{nflips} note decisions differ where the reference logit is not within tolerance of 0"
    assert sampler.last_launches_per_step > 100


def test_graph_replay_matches_eager():
    """CUDA-graph replay and eager launches of the same plan give bit-identical eps"""
    L, B = 96, 2
    m = model_for(L)
    inp = synth.synthetic_inputs(B, L)
    s = m.engine.session(B, L, per_sample_t=True)
    s.set_timestep_table([500, 20])
    s.set_context(inp["c"].cuda())
    s.set_audio([w.cuda() for w in inp["w"]])
    s.load_x(inp["x_T"].cuda(), dup=False)
    s.eval(graph=False)
    a = s.read_rows(s.eps, B, 16, L).clone()
    s.eval(graph=True)
    s.eval(graph=True)
    b = s.read_rows(s.eps, B, 16, L)
    assert torch.equal(a, b)


def test_decode_vs_oracle_batch():
    L, B = 96, 3
    sd = synth.synthetic_state_dict(L)
    m = model_for(L)
    z = synth._gauss(synth._rng(5, "z"), (B, 16, L)) * 3
    with torch.no_grad():
        ref = orc.decoder_forward(sd, z)
    out = m.model.decode(z.cuda())
    assert out.shape == (B, 16, 8 * L)
    assert rel_err(out, ref) < 1e-4


def test_eta_noise_path_runs_and_is_seeded():
    L, B = 96, 1
    m = model_for(L)
    inp = synth.synthetic_inputs(B, L)
    sampler = DDIMSampler(m)
    outs = []
    for _ in range(2):
        torch.manual_seed(11)
        torch.cuda.manual_seed(11)
        z, _ = sampler.sample(S=5, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False,
                              x_T=inp["x_T"].cuda(), eta=1.0, shape=(16, L))
        outs.append(z)
    assert torch.isfinite(outs[0]).all() and torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("dropout", [0.0, 0.25])
def test_eta_noise_and_noise_dropout_match_oracle(dropout):
    """eta = 1 (sigma > 0), temperature != 1 and noise_dropout (ddim.py:192-194) against the CPU oracle fed with the very noise
    the GPU run draws: the sampler's only RNG calls are randn(shape) [+ dropout] per step on the CUDA generator, so re-seeding
    and repeating them here reproduces the sequence"""
    L, B, S = 96, 2, 5
    m = model_for(L)
    inp = synth.synthetic_inputs(B, L)
    sampler = DDIMSampler(m)
    torch.cuda.manual_seed(123)
    z, _ = sampler.sample(S=S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(),
                          eta=1.0, shape=(16, L), temperature=0.8, noise_dropout=dropout, unconditional_guidance_scale=3.0,
                          unconditional_conditioning=inp["uc"].cuda())
    torch.cuda.manual_seed(123)
    seq = []
    for _ in range(S):
        nz = torch.randn((B, 16, L), device="cuda")
        if dropout > 0:
            nz = torch.nn.functional.dropout(nz, p=dropout)
        seq.append(nz.cpu())
    with torch.no_grad():
        ref = orc.ddim_sample(synth.synthetic_state_dict(L), S, inp["c"], inp["w"], inp["x_T"], scale=3.0, uc=inp["uc"], eta=1.0,
                              noise_seq=seq, temperature=0.8)
    assert rel_err(z, ref) < 2e-4
    if dropout > 0:
        assert any((t == 0).any() for t in seq)


def test_match_reference_rng_consumes_the_generator_like_the_reference():
    """at eta = 0 the reference still draws randn(shape) every step (ddim.py:192); with match_reference_rng the CUDA generator
    ends where S draws leave it, without it the generator is untouched -- and the samples are identical either way"""
    L, B, S = 96, 1, 4
    m = model_for(L)
    inp = synth.synthetic_inputs(B, L)
    sampler = DDIMSampler(m)
    kw = dict(S=S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(), shape=(16, L))
    torch.cuda.manual_seed(5)
    z0, _ = sampler.sample(**kw)
    after_plain = torch.randn(4, device="cuda")
    torch.cuda.manual_seed(5)
    z1, _ = sampler.sample(match_reference_rng=True, **kw)
    after_match = torch.randn(4, device="cuda")
    torch.cuda.manual_seed(5)
    for _ in range(S):
        torch.randn((B, 16, L), device="cuda")
    want = torch.randn(4, device="cuda")
    torch.cuda.manual_seed(5)
    untouched = torch.randn(4, device="cuda")
    assert torch.equal(z0, z1)
    assert torch.equal(after_match, want) and torch.equal(after_plain, untouched)


def test_full_size_batch32_is_consistent_with_batch4_chunks():
    """BASELINE configs[2] size (L=512, 32 charts, CFG -> 64 U-Net rows per step): samples are independent (no cross-sample op),
    so a batch-32 run must agree with the same charts sampled 4 at a time.  Tile packing and K splits differ between the two
    plans, so this is a tolerance (accumulation order; measured 2.2e-5 after 5 guided steps), not a bit test."""
    L, B, S = 512, 32, 5
    m = model_for(L)
    m.z_length = L
    inp = synth.synthetic_inputs(B, L, seed=77)
    sampler = DDIMSampler(m)

    def run(sl):
        z, _ = sampler.sample(S=S, c=inp["c"][sl].cuda(), w=[w[sl].cuda() for w in inp["w"]], batch_size=sl.stop - sl.start, verbose=False,
                              x_T=inp["x_T"][sl].cuda(), eta=0.0, shape=(16, L), unconditional_guidance_scale=5.0,
                              unconditional_conditioning=inp["uc"][sl].cuda())
        return z

    big = run(slice(0, B))
    assert torch.isfinite(big).all()
    for b0 in (0, 12, 28):
        small = run(slice(b0, b0 + 4))
        assert rel_err(big[b0:b0 + 4], small) < 1e-4
    # guidance scale 1 takes the Beff = B path (ddim.py:170-171): identical to passing no unconditional prompt at all
    kw = dict(S=4, c=inp["c"][:4].cuda(), w=[w[:4].cuda() for w in inp["w"]], batch_size=4, verbose=False, x_T=inp["x_T"][:4].cuda(),
              eta=0.0, shape=(16, L))
    z_a, _ = sampler.sample(unconditional_guidance_scale=1.0, unconditional_conditioning=inp["uc"][:4].cuda(), **kw)
    z_b, _ = sampler.sample(**kw)
    assert torch.equal(z_a, z_b)


def test_mask_branch_with_zero_mask_is_identity():
    """ddim.py:141-144 inpainting blend x = q_sample(x0,t)*mask + (1-mask)*x : with mask == 0 the trajectory must equal
    the unmasked one bit for bit (the noisy x0 is multiplied by zero), which exercises the per-step host round trip"""
    L, B = 96, 1
    m = model_for(L)
    inp = synth.synthetic_inputs(B, L)
    sampler = DDIMSampler(m)
    kw = dict(S=4, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(), shape=(16, L))
    z0, _ = sampler.sample(**kw)
    z1, _ = sampler.sample(mask=torch.zeros(B, 16, L).cuda(), x0=torch.ones(B, 16, L).cuda(), **kw)
    assert torch.equal(z0, z1)


def test_mask_branch_matches_oracle_with_shared_noise():
    """non-trivial inpainting mask (ddim.py:140-143): the first half of the chart is pinned to q_sample(x0, t) every step.  The
    sampler's only RNG call per step at eta = 0 is q_sample's randn_like(x0) on the CUDA generator, so re-seeding and repeating
    the draws hands the oracle the very same noise."""
    L, B, S = 96, 2, 6
    m = model_for(L)
    inp = synth.synthetic_inputs(B, L)
    sampler = DDIMSampler(m)
    x0 = synth._gauss(synth._rng(31, "x0"), (B, 16, L))
    mask = torch.zeros(B, 16, L)
    mask[:, :, :L // 2] = 1.0
    mask[1, 4:, L // 4:L // 2] = 0.5                                   # soft edge on one sample
    torch.cuda.manual_seed(77)
    z, _ = sampler.sample(S=S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(),
                          eta=0.0, shape=(16, L), mask=mask.cuda(), x0=x0.cuda(), unconditional_guidance_scale=3.0,
                          unconditional_conditioning=inp["uc"].cuda())
    torch.cuda.manual_seed(77)
    n_steps = len(range(0, 1000, 1000 // S))                           # S = 6 gives 7 DDIM steps (utils.py:52-63)
    qseq = [torch.randn((B, 16, L), device="cuda").cpu() for _ in range(n_steps)]
    with torch.no_grad():
        ref = orc.ddim_sample(synth.synthetic_state_dict(L), S, inp["c"], inp["w"], inp["x_T"], scale=3.0, uc=inp["uc"], mask=mask, x0=x0,
                              q_noise_seq=qseq)
        plain = orc.ddim_sample(synth.synthetic_state_dict(L), S, inp["c"], inp["w"], inp["x_T"], scale=3.0, uc=inp["uc"])
    assert rel_err(z, ref) < 2e-4
    assert rel_err(plain, ref) > 1e-2                                  # the mask really changed the trajectory


def test_config2_shape_ten_guided_steps_vs_live_oracle():
    """BASELINE config 2's own shape -- 4 charts, z_length 512, CFG 5 -- for 10 DDIM steps against the LIVE CPU oracle (not another
    GPU run), then decode and compare logits and note decisions"""
    L, B, S = 512, 4, 10
    sd = synth.synthetic_state_dict(L)
    m = model_for(L)
    m.z_length = L
    inp = synth.synthetic_inputs(B, L, seed=404)
    sampler = DDIMSampler(m)
    z, _ = sampler.sample(S=S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(),
                          eta=0.0, shape=(16, L), unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    logits = m.model.decode(z)
    with torch.no_grad():
        z_ref = orc.ddim_sample(sd, S, inp["c"], inp["w"], inp["x_T"], scale=5.0, uc=inp["uc"])
        l_ref = orc.decoder_forward(sd, z_ref)
    ez, el = rel_err(z, z_ref), rel_err(logits, l_ref)
    print(f"config2 shape: z {ez:.2e} logits {el:.2e}")
    assert ez < 1e-3 and el < 1e-3
    rows = [0, 1, 2, 3, 8, 9, 10, 11]                                  # note-on / hold channels (convertor.py:211-264)
    flips = ((logits.cpu()[:, rows] > 0) != (l_ref[:, rows] > 0))
    assert (l_ref[:, rows][flips].abs() <= 1e-3 * l_ref.abs().max()).all(), "a note decision flipped away from logit ~ 0"


def test_long_chart_guided_trajectory_and_decode_vs_live_oracle():
    """BASELINE config 5's length (6-min audio, z_length 992 -> levels 992/496/248/124): 5 guided steps of 2 charts + decode against the
    live CPU oracle"""
    L, B, S = 992, 2, 5
    sd = synth.synthetic_state_dict(L)
    m = model_for(L)
    m.z_length = L
    inp = synth.synthetic_inputs(B, L, seed=992)
    sampler = DDIMSampler(m)
    z, _ = sampler.sample(S=S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(),
                          eta=0.0, shape=(16, L), unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    logits = m.model.decode(z)
    with torch.no_grad():
        z_ref = orc.ddim_sample(sd, S, inp["c"], inp["w"], inp["x_T"], scale=5.0, uc=inp["uc"])
        l_ref = orc.decoder_forward(sd, z_ref)
    ez, el = rel_err(z, z_ref), rel_err(logits, l_ref)
    print(f"L=992: z {ez:.2e} logits {el:.2e}")
    assert ez < 1e-3 and el < 1e-3

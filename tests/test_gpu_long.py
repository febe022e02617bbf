"""Long songs on the GPU: z_length past 1568, where the level-0 S4 layers no longer fit the resident convolution kernel and run the
streamed one (csrc/s4.cu), up to the supported maximum 8192.

* the streamed s4conv against a float64 FFT convolution (2e-5, the s4conv bound of test_gpu_ops), and bit for bit against the
  resident kernel at every length the resident kernel takes (mugd_set_s4conv_impl forces either);
* S4 kernel generation at L_internal 2048 / 4096 / 8192 against the oracle (1e-5), the tensor-core attention at the self-attention
  shapes of z_length 4096 and 8192 against float64;
* U-Net evaluations against the reference's outputs (tests/golden/, tools/make_long_goldens.py) and at z_length 8192 against the
  live oracle (1e-4); a 4-step guided DDIM trajectory against the reference (1e-3);
* a 10-minute song through the public API: audio_features (z_length 1632), DDIM, decode, hit objects, post-processing;
* one guided step and decode at the ceiling, z_length 8192.
"""
import os
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import attention_cases as ac  # noqa: E402
import golden_cases as gc  # noqa: E402
import long_cases as lc  # noqa: E402
from gpu_util import OpRunner, ncl, nlc, ptr, rel_err, view  # noqa: E402
from mug_diffusion_b200 import audio, synth  # noqa: E402
from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200.engine import OpList  # noqa: E402
from oracle import mug_oracle as orc  # noqa: E402

AUTO, RESIDENT, STREAMED = 0, 1, 2


@pytest.fixture(scope="module")
def R():
    return OpRunner()


class s4conv_impl:
    """mugd_set_s4conv_impl for a block (per handle: always back to automatic)"""

    def __init__(self, R, impl):
        self.R, self.impl = R, impl

    def __enter__(self):
        L_.check(self.R.lib.mugd_set_s4conv_impl(self.R.handle, self.impl), "s4conv_impl")

    def __exit__(self, *exc):
        L_.check(self.R.lib.mugd_set_s4conv_impl(self.R.handle, AUTO), "s4conv_impl")


def g(name, shape, seed=5):
    return synth._gauss(synth._rng(seed, name), shape)


def s4_operands(B, L, H):
    """u [B,H,L], taps K [H,L] that decay over about a thousand steps (so the far taps matter), D [H]"""
    u = g(f"lu{B}.{L}.{H}", (B, H, L))
    K = g(f"lk{L}.{H}", (H, L)) * torch.exp(-torch.arange(L) / 1000.0)[None]
    return u, K, g(f"ld{H}", (H,))


def run_s4conv(R, u, K, D, impl=AUTO):
    B, H, L = u.shape
    uc, kt, dc = nlc(u).cuda(), K.t().contiguous().cuda(), D.cuda()
    out = torch.zeros(B * L, H).cuda()
    ops = OpList()
    ops.s4conv(view(uc), ptr(kt), ptr(dc), view(out), B, L)
    with s4conv_impl(R, impl):
        R.run(ops)
    return out


@pytest.mark.parametrize("B,L,H", [(1, 1600, 128), (2, 1999, 256), (1, 2048, 512), (3, 2048, 128), (1, 4096, 256), (2, 4096, 128),
                                   (1, 8192, 128), (1, 8192, 512)])
def test_streamed_s4conv_vs_fp64(R, B, L, H):
    u, K, D = s4_operands(B, L, H)
    u64, K64 = u.double(), K.double()
    y = torch.fft.irfft(torch.fft.rfft(u64, n=2 * L) * torch.fft.rfft(K64, n=2 * L)[None], n=2 * L)[..., :L]
    ref = F.gelu(y + u64 * D.double()[None, :, None])
    out = run_s4conv(R, u, K, D)                                   # automatic: the streamed kernel past L = 1584
    err = rel_err(ncl(out.cpu(), B).double(), ref)
    print(f"s4conv streamed B={B} L={L} H={H}: rel_err {err:.2e}")
    assert err < 2e-5
    assert torch.equal(out, run_s4conv(R, u, K, D, STREAMED))


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("H", [64, 128, 512])
@pytest.mark.parametrize("L", [96, 250, 512, 992, 1568, 1584])
def test_streamed_equals_resident_bit_for_bit(R, B, L, H):
    u, K, D = s4_operands(B, L, H)
    resident = run_s4conv(R, u, K, D, RESIDENT)
    assert torch.equal(resident, run_s4conv(R, u, K, D, AUTO))      # automatic keeps the resident kernel wherever it fits
    streamed = run_s4conv(R, u, K, D, STREAMED)
    assert torch.equal(resident.view(torch.int32), streamed.view(torch.int32))


def test_s4conv_impl_switch(R):
    u, K, D = s4_operands(1, 1600, 64)
    with pytest.raises(L_.MugdError, match="L=1600 needs 234432 B of shared memory"):
        run_s4conv(R, u, K, D, RESIDENT)
    assert R.lib.mugd_set_s4conv_impl(R.handle, 3) != 0
    assert R.lib.mugd_set_s4conv_impl(R.handle, -1) != 0
    # y on top of u is refused: later windows still read rows an in-place write would have replaced
    uc, kt, dc = nlc(u).cuda(), K.t().contiguous().cuda(), D.cuda()
    ops = OpList()
    ops.s4conv(view(uc), ptr(kt), ptr(dc), view(uc), 1, 1600)
    with pytest.raises(L_.MugdError, match="overlaps"):
        R.run(ops)


@pytest.mark.parametrize("L_int", [2048, 4096, 8192])
def test_s4_kernel_gen_long_vs_oracle(R, L_int):
    from mug_diffusion_b200.runtime import s4_fft_nodes
    H, N, pre = 128, 32, "k."
    sd = {pre + n: synth._init("t." + n, shp, role, 3) for n, shp, role in [
        ("C", (1, H, N, 2), "s4_C"), ("log_dt", (H,), "s4_log_dt"), ("B", (1, H, N, 2), "s4_B"), ("P", (1, H, N, 2), "s4_P"),
        ("inv_w_real", (H, N), "s4_inv_w_real"), ("w_imag", (H, N), "s4_w_imag")]}
    sd[pre + "L"] = torch.tensor(L_int)
    ref = orc.s4_nplr_kernel(sd, pre, L_int)
    dev = {k: v.cuda() for k, v in sd.items() if k != pre + "L"}
    kt = torch.zeros(L_int, H).cuda()
    ws = torch.zeros(2 * H * (L_int // 2 + 1) + 8, dtype=torch.float64).cuda()
    args = [ptr(dev[pre + n]) for n in ("log_dt", "B", "C", "P", "inv_w_real", "w_imag")]
    om = s4_fft_nodes(L_int).cuda()
    L_.check(R.lib.mugd_s4_kernel_gen(R.handle, *args, ptr(om), H, N, L_int, L_int, ptr(kt), ptr(ws), ws.numel() * 8,
                                      torch.cuda.current_stream().cuda_stream), "s4_kernel_gen")
    torch.cuda.synchronize()
    assert rel_err(kt.t(), ref) < 1e-5


# the self-attention of U-Net levels 1-3 (head dims 32 / 48 / 64) at z_length 8192 and at one shorter length each
@pytest.mark.parametrize("D,L", [(32, 4096), (32, 2048), (48, 2048), (48, 1024), (64, 1024), (64, 512)])
def test_attention_long_vs_fp64(R, D, L):
    c = ac.layout(1, 8, D, L, L)
    q, k, v, rel, cg = ac.make_inputs(c)
    buf = torch.cat([q, k, v], dim=-1).reshape(L, 3 * c.C).contiguous().cuda()
    out = torch.zeros(L, c.C).cuda()
    rel_d, cg_d = rel.cuda(), cg.cuda()
    ops = OpList()
    ops.attention(view(buf, 0, c.C), view(buf, c.C, 2 * c.C), view(buf, 2 * c.C, 3 * c.C), view(out), ptr(rel_d), ptr(cg_d),
                  1, c.H, L, L, c.pos_max)
    R.run(ops)
    o = out.cpu().reshape(1, L, c.C)
    err = 0.0
    for h in range(c.H):                                           # one head at a time: the float64 logits of all heads would be 8 GB
        s = slice(h * D, (h + 1) * D)
        ref, mag = ac.ref_attention(q[..., s], k[..., s], v[..., s], rel[:, h:h + 1], cg[:, h:h + 1], 1, c.pos_max, c.scale)
        err = max(err, ac.row_error(o[..., s], ref, mag, 1))
    print(f"attention tc D={D} L={L}: row_err {err:.2e}")
    assert err < 1.4e-5                                            # test_gpu_attention's bound for the wgmma kernel on randn data


_models = {}


def model_for(L, persisted=None, wave=False):
    key = (L, persisted, wave)
    if key not in _models:
        from mug_diffusion_b200 import wave as wave_mod
        from mug_diffusion_b200.sampler import MugDiffusionB200
        _models.clear()                                            # one resident model at a time
        sd = dict(synth.synthetic_state_dict(persisted or L))
        if wave:
            sd.update(wave_mod.synthetic_wave_state_dict())
        _models[key] = (sd, MugDiffusionB200.from_state_dict(sd, z_length=L))
    return _models[key]


@pytest.mark.parametrize("name", list(lc.LONG_UNET_CASES))
def test_unet_eval_vs_reference_golden(name, golden_dir):
    case = lc.LONG_UNET_CASES[name]
    _, m = model_for(case["L"], case["persisted"])
    inp = synth.synthetic_inputs(case["B"], case["L"])
    eps = m.model.forward(inp["x_T"].cuda(), torch.tensor(case["t"]).cuda(), inp["c"].cuda(), synth.wave_list([w.cuda() for w in inp["w"]]))
    gold = gc.load_golden(os.path.join(golden_dir, name + ".npz"))["eps"]
    assert eps.shape == gold.shape
    err = rel_err(eps, gold)
    print(f"{name}: rel_err {err:.2e}")
    assert err < 1e-4
    if case["persisted"]:
        assert m.engine.s4_L["model.unet_model.input_blocks.2.1.s4_model.kernel.kernel.L"] == case["L"]


def test_unet_eval_at_the_ceiling_vs_oracle():
    L = audio.MAX_Z_LENGTH
    sd, m = model_for(L)
    inp = synth.synthetic_inputs(1, L, seed=8192)
    t = torch.tensor([517])
    eps = m.model.forward(inp["x_T"].cuda(), t.cuda(), inp["c"].cuda(), [w.cuda() for w in inp["w"]])
    t0 = time.time()
    with torch.no_grad():
        ref = orc.unet_forward(sd, inp["x_T"], t, inp["c"], inp["w"])
    err = rel_err(eps, ref)
    print(f"unet L={L} B=1: rel_err {err:.2e}; oracle host time {time.time() - t0:.1f} s")
    assert err < 1e-4


def test_ddim_trajectory_vs_reference_golden(golden_dir):
    from mug_diffusion_b200.sampler import DDIMSampler
    name = "ddim_L1600_B1_S4_cfg5"
    case = lc.LONG_DDIM_CASES[name]
    _, m = model_for(case["L"])
    m.z_length = case["L"]
    inp = synth.synthetic_inputs(case["B"], case["L"])
    preds = []
    z, _ = DDIMSampler(m).sample(S=case["S"], c=inp["c"].cuda(), w=synth.wave_list([w.cuda() for w in inp["w"]]), batch_size=case["B"],
                                 shape=None, verbose=False, x_T=inp["x_T"].cuda(), eta=0.0, unconditional_guidance_scale=case["scale"],
                                 unconditional_conditioning=inp["uc"].cuda(), img_callback=lambda p, i: preds.append(p.clone()))
    logits = m.model.decode(z)
    gold = gc.load_golden(os.path.join(golden_dir, name + ".npz"))
    assert rel_err(preds[0], gold["pred_x0_first"]) < 1e-4
    ez, el = rel_err(z, gold["z"]), rel_err(logits, gold["logits"])
    print(f"{name}: z {ez:.2e} logits {el:.2e}")
    assert ez < 1e-3 and el < 1e-3


def song(seconds: float, sr: int = 22050, seed: int = 10) -> np.ndarray:
    """a seeded stand-in for music: a chord whose notes change every half second under a beat-rate envelope, plus noise"""
    rng = np.random.default_rng(seed)
    n = int(seconds * sr)
    t = np.arange(n, dtype=np.float64) / sr
    beat = np.floor(t * 2).astype(np.int64)
    y = 1e-3 * rng.standard_normal(n)
    for k in range(3):
        f = 110.0 * 2 ** (rng.integers(0, 36, beat[-1] + 1) / 12)
        y += np.sin(2 * np.pi * np.cumsum(f[beat]) / sr) * np.exp(-4 * (t * 2 - beat)) * 0.3
    return (0.9 * y / np.abs(y).max()).astype(np.float32)


def test_ten_minute_song_end_to_end():
    """webui's request for a 10-minute song (z_length 1632): audio_features, 5 guided DDIM steps for 2 charts, decode, hit objects
    and post-processing, each stage against its host statement"""
    import audio_oracle
    from mug_diffusion_b200 import postprocess as pp
    from mug_diffusion_b200.sampler import DDIMSampler
    from oracle import wave_oracle as worc
    B, S = 2, 5
    y = song(600.0)
    sd, m = model_for(1632, wave=True)
    w, zl = m.model.audio_features(y, B)
    assert zl == 1632 and len(w) == 10
    with torch.no_grad():
        mel = audio_oracle.log_mel(y)
        w_ref = worc.wave_forward(sd, F.pad(mel, (0, 64 * zl - mel.shape[-1])))
    for i in range(6, 10):
        assert rel_err(w[i][:1], w_ref[i]) < 1e-4, i
    m.z_length = zl
    inp = synth.synthetic_inputs(B, zl, seed=1632)
    z, _ = DDIMSampler(m).sample(S=S, c=inp["c"].cuda(), w=w, batch_size=B, verbose=False, x_T=inp["x_T"].cuda(), eta=0.0,
                                 unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    logits = m.model.decode(z)
    w4 = [h.cpu().contiguous() for h in w[6:]]
    with torch.no_grad():
        z_ref = orc.ddim_sample(sd, S, inp["c"], w4, inp["x_T"], scale=5.0, uc=inp["uc"])
        l_ref = orc.decoder_forward(sd, z_ref)
    ez, el = rel_err(z, z_ref), rel_err(logits, l_ref)
    print(f"10-minute song (z_length {zl}): z {ez:.2e} logits {el:.2e}")
    assert ez < 1e-3 and el < 1e-3
    rows = [0, 1, 2, 3, 8, 9, 10, 11]                              # note-on / hold channels
    flips = (logits.cpu()[:, rows] > 0) != (l_ref[:, rows] > 0)
    assert (l_ref[:, rows][flips].abs() <= 1e-3 * l_ref.abs().max()).all(), "a note decision flipped away from logit ~ 0"

    frame_ms = 1000.0 * 1024 / 22050                               # a latent frame is 64 mel frames of hop 128, and 8 note frames
    charts = m.model.decode_to_hit_objects(z, frame_ms)
    assert len(charts) == B and all(len(c) > 0 for c in charts)
    got = m.model.postprocess_charts(charts)
    for c, (bpm, off, lines) in zip(charts, got):
        new, hbpm, hoff = pp.gridify(c, verbose=False)               # webui.py:401-407
        assert type(bpm) is type(hbpm) and bpm == hbpm and type(off) is type(hoff) and off == hoff
        assert lines == pp.remove_intractable_mania_mini_jacks(new, verbose=False, jack_interval=90)


def test_one_guided_step_at_the_ceiling():
    from mug_diffusion_b200.sampler import DDIMSampler
    L = audio.MAX_Z_LENGTH
    _, m = model_for(L)
    m.z_length = L
    inp = synth.synthetic_inputs(1, L, seed=7)
    z, _ = DDIMSampler(m).sample(S=1, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=1, verbose=False,
                                 x_T=inp["x_T"].cuda(), eta=0.0, unconditional_guidance_scale=5.0,
                                 unconditional_conditioning=inp["uc"].cuda())
    logits = m.model.decode(z)
    assert z.shape == (1, 16, L) and logits.shape[-1] == 8 * L
    assert bool(torch.isfinite(z).all()) and bool(torch.isfinite(logits).all())
    arena = {k: s.arena_t.numel() * 4 for k, s in m.engine.sessions.items()}
    print(f"z_length {L}: U-Net session arenas {arena} bytes, peak device memory {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


def test_over_the_ceiling_is_refused_before_gpu_work():
    _, m = model_for(96)
    L = audio.MAX_Z_LENGTH + 32
    before = dict(m.engine.sessions)
    with pytest.raises(L_.MugdError, match="maximum 8192"):
        m.engine.session(2, L)
    with pytest.raises(L_.MugdError, match="maximum 8192"):
        m.engine.decoder_session(1, L)
    assert dict(m.engine.sessions) == before

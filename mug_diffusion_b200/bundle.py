"""Export one compiled sampling request as a bundle a host WITHOUT Python can run (examples/host_c/sample_host.c):

    python -m mug_diffusion_b200.bundle --out /tmp/bundle --L 96 --B 1 --S 10 --scale 5
    python -m mug_diffusion_b200.bundle --out /tmp/bundle --L 96 --B 2 --S 10 --scale 5 --eta 1 --inpaint     (regenerate half a chart)

The network -> launch-plan compiler is Python (engine.py); what it produces is plain data: arrays of mugd_op whose pointers fall
into a handful of device allocations.  The bundle holds
    manifest.txt        region table (name, bytes, initial contents), the plans in execution order, test inputs, expected outputs
    *.plan              mugd_plan_save files (pointers stored as region + offset)
    *.bin               region contents: the packed weight blob as it is resident (hi in place) + its lo buffer, the S4 convolution kernels, the per-request tables (timestep
                        sinusoids and DDIM coefficients for the chosen S -- host float math, kept out of the C demo), test vectors
Request flow = DDIMSampler.sample + model.decode (ddim.py:56-196, diffusion.py:49-50):
    emb (time-embedding table) -> ctx (cross-attention K|V) -> audio (concat slots) -> loadx -> S x {eval graph ; update ; advance}
    -> readz -> decode -> readlogits
An inpainting or eta > 0 request stages x0, the mask and the random numbers of every step (drawn up front from torch's CUDA generator in
the sampler's order) as input regions, with the q_sample coefficients in stage_coef.bin, and runs its loop as one mugd_sample_staged
call: `stage <field> <region> <offset>` lines describe the mugd_stage, `staged eval.plan tail.plan <steps> <coef file> <B> <C> <L>` runs it.
A seeded bundle (--seeds 7,8) carries no random numbers: `seeds <file> <B>` gives the charts' 64-bit seeds and each
`randn <region> <purpose> <first_draw> <n_draws> <draw_stride> <B> <n>` line fills x_T or a noise table with one mugd_randn call
(seeding.py's convention), so the host can also draw new charts from seeds of its own.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import lib as L_
from . import seeding
from .engine import OpList
from .runtime import Plan, _ptr
from .sampler import draw_step_noise, q_coef_table


def _save_plan(eng, ops: OpList, regions: List[L_.Region], path: str) -> Plan:
    pl = Plan(eng, ops)
    arr = (L_.Region * len(regions))(*regions)
    L_.check(eng.lib.mugd_plan_save(pl.handle, arr, len(regions), path.encode()), f"plan_save {path}")
    return pl


def export_bundle(model, inp: Dict[str, torch.Tensor], S: int, scale: float, out_dir: str, eta: float = 0.0, temperature: float = 1.0,
                  noise_dropout: float = 0.0, inpaint: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                  seeds=None) -> Dict[str, torch.Tensor]:
    """Compile the request (inp: x_T, c, uc, w[4] on the host; inpaint: (x0, mask) of DDIMSampler.sample), write the bundle, run it
    once through the very same plans and return the results (z, logits) that the C host must reproduce.  The random numbers of an
    eta > 0 or inpainting request are drawn here from the CUDA generator as DDIMSampler.sample draws them.  With ``seeds``
    (seeding.chart_seeds) x_T and every noise table are the charts' seeded draws, DDIMSampler.sample(seeds=...)'s, and the bundle
    holds the seeds and `randn` lines instead of their contents; inp's x_T is not used."""
    from .sampler import DDIMSampler

    os.makedirs(out_dir, exist_ok=True)
    eng = model.engine
    dev = eng.device
    cfg = eng.cfg
    B, Cz, Lz = inp["x_T"].shape
    if seeds is not None:
        if noise_dropout > 0.:
            raise ValueError("a seeded bundle draws no dropout mask")
        seeds = seeding.chart_seeds(seeds, B)
    cfg_on = scale != 1.0
    Beff = 2 * B if cfg_on else B
    sampler = DDIMSampler(model)
    sampler.make_schedule(S, ddim_eta=eta, verbose=False)
    ts = np.flip(sampler.ddim_timesteps)
    total = len(ts)

    with eng.lock:
        sess = eng.session(Beff, Lz, per_sample_t=False)
        dec = eng.decoder_session(B, Lz)
        T = inp["c"].shape[2]
        sess.set_ctx_tokens(T)
        # ---- staging buffers of the caller (inputs / outputs in the reference's NCL layout) ----
        seeded = None if seeds is None else seeding.ChartNoise(seeds, (B, Cz, Lz), dev)
        x_T = inp["x_T"] if seeded is None else seeded.draw(seeding.X_T, 0)
        st = dict(in_x=x_T.to(dev).contiguous(), in_c=inp["c"].to(dev).contiguous(), in_uc=inp["uc"].to(dev).contiguous(),
                  pred=torch.zeros(B * Lz * Cz, device=dev), out_z=torch.zeros(B, Cz, Lz, device=dev),
                  out_logits=torch.zeros(B, cfg.decoder.x_channels, dec.Lout, device=dev))
        w4 = [w.to(dev).contiguous() for w in list(inp["w"])[-cfg.unet.levels:]]
        for i, w in enumerate(w4):
            st[f"in_w{i}"] = w
        # the staged loop's operands: x0, the expanded mask and one [B, C, L] row per step of each noise table
        has_noise = bool(np.any(np.asarray(sampler.ddim_sigmas) != 0))
        staged = has_noise or inpaint is not None
        shape = (B, Cz, Lz)
        if has_noise:
            st["noise_rows"] = torch.zeros(B * Lz * Cz, device=dev)
            st["in_noise"] = torch.empty((total,) + shape, device=dev)
        if inpaint is not None:
            st["in_x0"] = inpaint[0].to(dev, torch.float32).contiguous()
            st["in_mask"] = inpaint[1].to(dev, torch.float32).expand(shape).contiguous()
            st["in_qnoise"] = torch.empty((total,) + shape, device=dev)
            qcoef = q_coef_table(model, ts)
            qcoef.tofile(os.path.join(out_dir, "stage_coef.bin"))
        # step i reads the DDIM coefficient row total - 1 - i, so a seeded table walks the draws downwards from total - 1
        randn_rows = {} if seeded is None else dict(seeded=seeded, first_draw=total - 1, draw_stride=-1)
        draw_step_noise(total, shape, st.get("in_x0"), st.get("in_qnoise"), has_noise, st.get("in_noise"), noise_dropout, dev,
                        **randn_rows)
        # what a seeded bundle draws on the host instead of loading: region -> (purpose, first_draw, n_draws, draw_stride)
        drawn = {} if seeded is None else {"in_x": (seeding.X_T, 0, 1, 1)}
        if seeded is not None:
            drawn.update({k: (p, total - 1, total, -1) for k, p in (("in_noise", seeding.STEP), ("in_qnoise", seeding.Q)) if k in st})
        # per-request host tables for this S
        sess.set_timestep_table(ts.copy())
        sess.set_ddim_schedule(sampler.ddim_alphas, sampler.ddim_alphas_prev, sampler.ddim_sigmas, sampler.ddim_sqrt_one_minus_alphas)

        # ---- regions: every device allocation a plan may point into ----
        tensors: Dict[str, torch.Tensor] = dict(weights=eng.weights, weights_lo=eng.weights_lo, arena=sess.arena_t, emb_table=sess.emb_table, temb=sess.temb,
                                                emb_h1=sess.emb_h1, emb_h2=sess.emb_h2, step=sess.step, coef=sess.coef, ctx=sess.ctx,
                                                tc_ws=eng.tc_ws, tc_counters=eng.tc_counters, dec_arena=dec.arena_t)
        for i, t in enumerate(sess.ctx_kv):
            tensors[f"ctx_kv{i}"] = t
        for i, (_, t) in enumerate(sorted(sess.s4_kt.items())):
            tensors[f"s4_kt{i}"] = t
        tensors.update(st)
        contents = {"weights", "weights_lo", "temb", "coef"} | {k for k in tensors if k.startswith("s4_kt")}       # saved; everything else starts zeroed
        inputs = {k for k in st if k.startswith("in_")}
        names = list(tensors)
        keep = [n.encode() for n in names]
        regions = [L_.Region(keep[i], _ptr(tensors[n]), tensors[n].numel() * tensors[n].element_size()) for i, n in enumerate(names)]

        # ---- the plans ----
        tail = sess.ddim_tail(B, total, cfg_on, scale, temperature, _ptr(st["pred"]), _ptr(st["noise_rows"]) if has_noise else 0)
        stage = None
        if staged:
            stage = sess.ddim_stage(B, cfg_on, _ptr(st["noise_rows"]) if has_noise else 0)
            if has_noise:
                stage.noise = _ptr(st["in_noise"])
            if inpaint is not None:
                stage.x0, stage.mask, stage.q_noise = _ptr(st["in_x0"]), _ptr(st["in_mask"]), _ptr(st["in_qnoise"])
                stage.q_coef = qcoef.ctypes.data
        readz = OpList()
        readz.transpose(sess.xin.ptr, _ptr(st["out_z"]), sess.xin.ld, 0, B, Cz, Lz, False)
        dec_in = OpList()
        assert cfg.decoder.scale == 1.0, "bundle export assumes first-stage scale 1 (the shipped config)"
        dec_in.transpose(_ptr(st["out_z"]), dec.zin.ptr, 0, dec.zin.ld, B, cfg.decoder.z_channels, Lz, True)
        dec_out = OpList()
        dec_out.transpose(dec.logits.ptr, _ptr(st["out_logits"]), dec.logits.ld, 0, B, cfg.decoder.x_channels, dec.Lout, False)
        ctx_parts = [(_ptr(st["in_uc"]), B), (_ptr(st["in_c"]), B)] if cfg_on else [(_ptr(st["in_c"]), B)]
        seq = [("emb", sess.timestep_ops(total), "run"), ("ctx", sess.context_ops(ctx_parts, T), "run"),
               ("audio", sess.audio_ops([_ptr(w) for w in w4], cfg_on), "run"), ("loadx", sess.loadx_ops(_ptr(st["in_x"]), B, cfg_on), "run"),
               ("eval", None, "graph"), ("tail", tail, "tail"), ("readz", readz, "run"), ("dec_in", dec_in, "run"), ("dec", None, "graph"),
               ("dec_out", dec_out, "run")]
        plans = {}
        lines = ["mugd_bundle 1", f"# z_length {Lz} batch {B} guidance {scale} steps {total} (S={S})"]
        for n in names:
            t = tensors[n]
            nbytes = t.numel() * t.element_size()
            if (n in contents or n in inputs) and n not in drawn:
                t.detach().cpu().contiguous().numpy().tofile(os.path.join(out_dir, n + ".bin"))
                lines.append(f"region {n} {nbytes} file {n}.bin")
            else:
                lines.append(f"region {n} {nbytes} zero -")
        if seeded is not None:
            seeding.seed_array(seeds).tofile(os.path.join(out_dir, "seeds.bin"))
            lines.append(f"seeds seeds.bin {B}")
            for n, (purpose, first, count, stride) in drawn.items():
                lines.append(f"randn {n} {purpose} {first} {count} {stride} {B} {Cz * Lz}")
        for name, ops, mode in seq:
            path = os.path.join(out_dir, name + ".plan")
            if ops is None:
                pl = sess.plan if name == "eval" else dec.plan
                arr = (L_.Region * len(regions))(*regions)
                L_.check(eng.lib.mugd_plan_save(pl.handle, arr, len(regions), path.encode()), f"plan_save {name}")
            else:
                pl = _save_plan(eng, ops, regions, path)
            plans[name] = pl
            if mode == "tail":
                continue
            if name == "eval" and staged:
                for field in ("x", "x_dup", "x0", "mask", "q_noise", "noise", "noise_rows"):
                    ptr = getattr(stage, field)
                    if ptr:
                        region = next(n for n in names if 0 <= ptr - _ptr(tensors[n]) < tensors[n].numel() * tensors[n].element_size())
                        lines.append(f"stage {field} {region} {ptr - _ptr(tensors[region])}")
                lines.append(f"staged eval.plan tail.plan {total} {'stage_coef.bin' if inpaint is not None else '-'} {B} {Cz} {Lz}")
            elif name == "eval":
                lines.append(f"sample eval.plan tail.plan {total}")
            else:
                lines.append(f"plan {name}.plan {mode}")

        # ---- run the request once through these very plans: the expected outputs ----
        sess.set_step(0)
        for name in ("emb", "ctx", "audio", "loadx"):
            plans[name].run()
        sess.plan.launch(total, tail, stage)
        for name in ("readz", "dec_in"):
            plans[name].run()
        dec.plan.launch()
        plans["dec_out"].run()
        torch.cuda.synchronize()
        for n in ("out_z", "out_logits"):
            st[n].cpu().numpy().tofile(os.path.join(out_dir, n + ".expected.bin"))
            lines.append(f"expect {n} {st[n].numel() * 4} {n}.expected.bin")
        open(os.path.join(out_dir, "manifest.txt"), "w").write("\n".join(lines) + "\n")
        return dict(z=st["out_z"].clone(), logits=st["out_logits"].clone())


def main():
    from . import synth
    from .sampler import MugDiffusionB200

    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--L", type=int, default=96)
    ap.add_argument("--B", type=int, default=1)
    ap.add_argument("--S", type=int, default=10)
    ap.add_argument("--scale", type=float, default=5.0)
    ap.add_argument("--eta", type=float, default=0.0)
    ap.add_argument("--temperature", type=float, default=1.0)
    ap.add_argument("--noise-dropout", type=float, default=0.0)
    ap.add_argument("--inpaint", action="store_true", help="keep the first half of a synthetic chart latent, regenerate the rest")
    ap.add_argument("--seed", type=int, default=0, help="torch CUDA generator seed of the staged random numbers")
    ap.add_argument("--seeds", default=None, help="per-chart seeds, e.g. 7,8 (or one int s for charts s, s + 1, ...): the bundle "
                                                  "draws x_T and its noise tables with mugd_randn instead of carrying them")
    a = ap.parse_args()
    seeds = None if a.seeds is None else [int(v) for v in a.seeds.split(",")]
    if seeds is not None and len(seeds) == 1:
        seeds = seeds[0]
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(a.L), z_length=a.L)
    inp = synth.synthetic_inputs(a.B, a.L)
    torch.cuda.manual_seed(a.seed)
    res = export_bundle(model, inp, a.S, a.scale, a.out, eta=a.eta, temperature=a.temperature, noise_dropout=a.noise_dropout,
                        inpaint=synth.synthetic_inpainting(a.B, a.L) if a.inpaint else None, seeds=seeds)
    print("bundle written to", a.out, "| z", tuple(res["z"].shape), "logits", tuple(res["logits"].shape))


if __name__ == "__main__":
    main()

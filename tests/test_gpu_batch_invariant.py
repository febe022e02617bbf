"""Batch-invariant plans on the GPU (torch.equal throughout): the serial-split GEMM equals split kernel + reduce at every op the
invariant plans launch it for; every chart of a seeded batch equals the chart requested alone, for the samplers, inpainting, remix,
inversion, the encoder and the decoder; at one chart the invariant engine is today's engine.  A `simt` engine keeps its plans (no serial
split, no TF32 operand) and is batch-invariant through the FFMA kernel alone, also where a batch moves its GEMMs to 128 x 128 tiles."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200 import packer, synth  # noqa: E402
from mug_diffusion_b200.config import ModelConfig  # noqa: E402
from mug_diffusion_b200.engine import OpList, View, unit_batch_splits  # noqa: E402
from mug_diffusion_b200.sampler import (DDIMSampler, DDPMSampler, DPMSolverSampler, MugDiffusionB200, PLMSSampler,  # noqa: E402
                                        UniPCSampler)

_models = {}


def model_for(L, invariant=True, T=1000, impl="auto"):
    key = (L, invariant, T, impl)
    if key not in _models:
        if len(_models) > 1:
            _models.clear()
        cfg = ModelConfig(timesteps=T)
        sd = {**synth.synthetic_state_dict(L), **synth.synthetic_encoder_state_dict()}
        blob = packer.pack_model(sd, cfg.unet, cfg.decoder, encoder_cfg=cfg.encoder)
        _models[key] = MugDiffusionB200(sd, cfg, z_length=L, blob=blob, batch_invariant=invariant, gemm_impl=impl)
    return _models[key]


def request(B, L, seed=1234, cfg=True):
    inp = synth.synthetic_inputs(B, L, seed=seed)
    kw = dict(c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, shape=(16, L), verbose=False)
    if cfg:
        kw.update(unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    return kw


def one_chart(kw, b):
    out = dict(kw, c=kw["c"][b:b + 1], w=[w[b:b + 1] for w in kw["w"]], batch_size=1)
    if "unconditional_conditioning" in kw:
        out["unconditional_conditioning"] = kw["unconditional_conditioning"][b:b + 1]
    for k in ("mask", "x0"):
        if k in kw:
            out[k] = kw[k][b:b + 1] if kw[k].shape[0] > 1 else kw[k]
    return out


def _cond(kw):
    return {k: v for k, v in kw.items() if k not in ("batch_size", "shape", "verbose")}


# ---- 1. the serial variant is split kernel + reduce, bit for bit ------------------------------------------------------------------
@pytest.mark.parametrize("L", [512, 992])
def test_serial_split_equals_split_kernel_and_reduce(L):
    m = model_for(L)
    eng = m.engine
    B = 32
    kw = request(B, L)
    s = eng.session(2 * B, L, unit=2)
    s.set_timestep_table(list(range(999, 0, -20)))
    s.set_context([kw["unconditional_conditioning"], kw["c"]])
    s.set_audio(list(kw["w"])[-m.cfg.unet.levels:], dup=True)
    s.load_x(torch.randn(B, 16, L, device="cuda"), dup=True)
    s.set_step(3)
    s.eval(graph=False)                                  # the arena holds this evaluation's activations
    torch.cuda.synchronize()
    ops = [op for op in s.plan._arr if op.kind == L_.OP_GEMM_SERIAL]
    assert ops, "the B = 32 plan launches the serial variant"
    seen = set()
    for op in ops:
        g = op.u.gemm
        rows = g.M
        ncols = g.N // 2 if g.gate else g.N
        outs = {}
        for kind in (L_.OP_GEMM_SERIAL, L_.OP_GEMM):
            d = L_.Gemm.from_buffer_copy(g)
            out = torch.full((rows, d.ldc), float("nan"), device="cuda")
            d.C = out.data_ptr()
            mom = None
            if d.row_moments:
                mom = torch.zeros(rows, 2, dtype=torch.float64, device="cuda")
                d.row_moments = mom.data_ptr()
            # the split kernel's partial tiles of a forced one-chart split at B = 32: more than the engine's workspace holds
            sup, sp, ws, tiles = C.c_int32(), C.c_int32(), C.c_int64(), C.c_int32()
            L_.check(eng.lib.mugd_gemm_tc_query(None, C.byref(d), eng.sm_count, C.byref(sup), C.byref(sp), C.byref(ws), C.byref(tiles)), "query")
            assert sup.value and sp.value == g.split_k
            wsp = torch.empty(max(ws.value // 4, 4), device="cuda")
            d.workspace, d.workspace_bytes = wsp.data_ptr(), wsp.numel() * 4
            one = L_.make_op(kind, d)
            L_.check(eng.lib.mugd_op_run(eng.handle, C.byref(one), torch.cuda.current_stream().cuda_stream), f"kind {kind}")
            torch.cuda.synchronize()
            outs[kind] = (out[:, :ncols].clone(), mom)
        a, b = outs[L_.OP_GEMM_SERIAL], outs[L_.OP_GEMM]
        key = (g.M, g.N, g.K, g.taps, g.K2, g.split_k, bool(g.bias), bool(g.residual), bool(g.rowvec), g.act, g.gate,
               bool(g.row_moments), bool(g.ln_stats))
        assert torch.equal(a[0], b[0]), key
        assert not torch.isnan(a[0]).any(), key
        if a[1] is not None:
            assert torch.equal(a[1], b[1]), key
        seen.add(key)
    assert len(seen) >= 3


# one op in isolation: the policy picks kind and split for B charts of L rows; each chart's rows equal the one-chart op's.  L = 48:
# several samples share a 128-row tile and the last tile is part-filled; L = 200: a sample spans two tiles.
ONE_OP_EPIS = {
    "none_rowvec_res": dict(taps=3, mode=L_.CONV_SAME, rowvec=True, residual=True),
    "sink": dict(sink=True),
    "ln": dict(ln=True),
    "glu": dict(gate=L_.GATE_GLU),
}


def _one_op(eng, epi, Beff, L, x, keep):
    """the GEMM of ``epi`` over Beff samples of L rows whose operands are the one-chart operands ``x`` repeated; returns (op, out,
    row moments or None)"""
    e = ONE_OP_EPIS[epi]
    reps = Beff // x["unit"]
    K, N = x["A"].shape[1], x["W"].shape[0]
    a = x["A"].repeat(reps, 1).cuda()
    nout = N // 2 if e.get("gate") else N
    out = torch.full((Beff * L, nout), float("nan"), device="cuda")
    keep += [a, out]
    kw = dict(bias=x["bias"].data_ptr(), W_hi=x["hi"].data_ptr(), W_lo=x["lo"].data_ptr(), impl=L_.GEMM_TC, gate=e.get("gate", 0),
              taps=e.get("taps", 1), mode=e.get("mode", L_.CONV_NONE), Lin=L, Lout=L)
    if e.get("rowvec"):
        t = x["table"].repeat(reps, 1).cuda()
        kw.update(rowvec=t.data_ptr(), rowvec_b_stride=N)
        keep.append(t)
    if e.get("residual"):
        r = x["res"].repeat(reps, 1).cuda()
        kw["residual"] = View(r.data_ptr(), N, Beff * L, N)
        keep.append(r)
    if e.get("ln"):
        st = x["stats"].repeat(reps, 1).cuda()
        kw["ln"] = (st.data_ptr(), x["colsum"].data_ptr(), 1e-5)
        keep.append(st)
    ops = OpList()
    ops.gemm(View(a.data_ptr(), K, Beff * L, K), x["W"].data_ptr(), N, K, View(out.data_ptr(), nout, Beff * L, nout), **kw)
    mom = None
    if e.get("sink"):
        mom = torch.zeros(Beff * L, 2, dtype=torch.float64, device="cuda")
        ops.ops[0].u.gemm.row_moments = mom.data_ptr()
        keep.append(mom)
    ops = unit_batch_splits(ops, Beff, x["unit"], eng.sm_count)
    op = ops.ops[0]
    d = op.u.gemm
    ws = C.c_int64()
    L_.check(eng.lib.mugd_gemm_tc_query(None, C.byref(d), eng.sm_count, None, None, C.byref(ws), None), "query")
    wsp = torch.empty(max(ws.value // 4, 4), device="cuda")
    keep.append(wsp)
    d.workspace, d.workspace_bytes = wsp.data_ptr(), wsp.numel() * 4
    L_.check(eng.lib.mugd_op_run(eng.handle, C.byref(op), torch.cuda.current_stream().cuda_stream), f"{epi} Beff={Beff} L={L}")
    return op, out, mom


@pytest.mark.parametrize("epi", list(ONE_OP_EPIS))
def test_one_op_every_chart_equals_the_chart_alone(epi):
    """for L in {48, 200, 512}, B in {3, 8, 32} charts and a one-chart unit of 1 and 2 samples: each sample's rows (and row moments)
    of the B-chart op, kind and split chosen by engine.unit_batch_splits, equal the one-chart op's; the serial kind is taken at least
    once"""
    eng = model_for(96).engine
    e = ONE_OP_EPIS[epi]
    K, N = 256, 192
    kinds = set()
    for L in (48, 200, 512):
        for unit in (1, 2):
            name = f"{epi}.{L}.{unit}"
            kt = e.get("taps", 1) * K
            W = synth._gauss(synth._rng(5, name + ".W"), (N, kt)) / kt ** 0.5
            hi, lo = packer.tf32_split(W)
            A = synth._gauss(synth._rng(5, name + ".A"), (unit * L, K))
            a64 = A.double()
            x = dict(unit=unit, A=A, W=W.cuda(), hi=hi.cuda(), lo=lo.cuda(), bias=(0.1 * synth._gauss(synth._rng(5, name + ".b"), (N,))).cuda(),
                     table=synth._gauss(synth._rng(5, name + ".t"), (unit, N)), res=synth._gauss(synth._rng(5, name + ".r"), (unit * L, N)),
                     stats=torch.stack([a64.sum(1), (a64 * a64).sum(1)], dim=1), colsum=W.double().sum(1).float().cuda())
            keep = []
            _, one, mom1 = _one_op(eng, epi, unit, L, x, keep)
            for B in (3, 8, 32):
                op, many, mom = _one_op(eng, epi, B * unit, L, x, keep)
                kinds.add(op.kind)
                torch.cuda.synchronize()
                what = (epi, L, unit, B, op.kind, op.u.gemm.split_k)
                assert not torch.isnan(many).any(), what
                assert torch.equal(many.view(B, unit * L, -1), one.view(1, unit * L, -1).expand(B, -1, -1)), what
                if mom is not None:
                    assert torch.equal(mom.view(B, unit * L, 2), mom1.view(1, unit * L, 2).expand(B, -1, -1)), what
    assert L_.OP_GEMM_SERIAL in kinds, epi


# ---- 2. op by op: every output row of a plan for B charts is the one-chart plan's --------------------------------------------------
def _region(op):
    """(address, leading dimension, rows, columns) of the rows ``op`` writes, or None for an op that writes no activation rows"""
    k, u = op.kind, op.u
    if k in (L_.OP_GEMM, L_.OP_GEMM_SERIAL):
        return u.gemm.C, u.gemm.ldc, u.gemm.M, u.gemm.N // 2 if u.gemm.gate else u.gemm.N
    if k == L_.OP_GROUPNORM:
        return u.gn.y, u.gn.ldy, u.gn.B * u.gn.L, u.gn.C
    if k == L_.OP_LAYERNORM:
        return u.ln.y, u.ln.ldy, u.ln.rows, u.ln.C
    if k == L_.OP_ATTENTION:
        return u.attn.o, u.attn.ldo, u.attn.B * u.attn.Lq, u.attn.H * u.attn.D
    if k == L_.OP_S4CONV:
        return u.s4.y, u.s4.ldy, u.s4.B * u.s4.L, u.s4.H
    if k == L_.OP_COPY2D:
        return u.cp.dst, u.cp.ldd, u.cp.rows, u.cp.cols
    if k == L_.OP_TRANSPOSE and u.tr.to_nlc:
        return u.tr.out, u.tr.ldo, u.tr.B * u.tr.L, u.tr.C
    return None


def _run_op_by_op(eng, ops):
    """run ``ops`` one at a time; after each, a copy of the rows it wrote ([rows, cols]), or None"""
    st = torch.cuda.current_stream().cuda_stream
    outs = []
    for i, op in enumerate(ops):
        L_.check(eng.lib.mugd_op_run(eng.handle, C.byref(op), st), f"op {i} kind {op.kind}")
        r = _region(op)
        if r is None or not r[0] or r[3] % 4 or r[1] % 4 or r[0] % 16:
            outs.append(None)
            continue
        ptr, ld, rows, cols = r
        t = torch.empty(rows, cols, device="cuda")
        cp = L_.Copy2D()
        cp.src, cp.lds, cp.dst, cp.ldd, cp.rows, cp.cols = ptr, ld, t.data_ptr(), cols, rows, cols
        one = L_.make_op(L_.OP_COPY2D, cp)
        L_.check(eng.lib.mugd_op_run(eng.handle, C.byref(one), st), "copy2d")
        outs.append(t)
    torch.cuda.synchronize()
    return outs


def _same_rows_as_one_chart(ops, outs, ops1, outs1, Beff, unit, what):
    """sample j of the Beff-sample plan against sample j // (Beff / unit) of the unit plan, op by op; returns the ops compared"""
    assert len(ops) == len(ops1), what
    per = Beff // unit
    n = 0
    for i, (op, t, op1, t1) in enumerate(zip(ops, outs, ops1, outs1)):
        gemm = (L_.OP_GEMM, L_.OP_GEMM_SERIAL)
        assert op.kind == op1.kind or (op.kind in gemm and op1.kind in gemm), (what, i)
        if t is None or t1 is None or t.shape[0] % Beff:
            continue
        rps = t.shape[0] // Beff
        assert t1.shape == (rps * unit, t.shape[1]), (what, i)
        got = t.view(Beff, rps, -1)
        want = t1.view(unit, rps, -1).repeat_interleave(per, dim=0)
        assert torch.equal(got, want), (what, i, op.kind, [j for j in range(Beff) if not torch.equal(got[j], want[j])][:8])
        n += 1
    return n


BATCHES = [1, 2, 3, 8, 32]


def test_unet_op_by_op_every_batch_equals_one_chart():
    """every sample of the U-Net plan for B charts (CFG: Beff = 2B) fed B copies of one chart equals the one-chart plan, op by op"""
    L = 512
    m = model_for(L)
    eng = m.engine
    kw = request(1, L)
    x = torch.randn(1, 16, L, device="cuda", generator=torch.Generator("cuda").manual_seed(5))

    def run(B):
        s = eng.session(2 * B, L, unit=2)
        s.set_timestep_table(list(range(999, 0, -20)))
        s.set_context([kw["unconditional_conditioning"].repeat(B, 1, 1), kw["c"].repeat(B, 1, 1)])
        s.set_audio([w.repeat(B, 1, 1) for w in list(kw["w"])[-m.cfg.unet.levels:]], dup=True)
        s.load_x(x.repeat(B, 1, 1), dup=True)
        s.set_step(7)
        torch.cuda.synchronize()
        ops = list(s.plan._arr)
        return ops, _run_op_by_op(eng, ops)

    ops1, outs1 = run(1)
    for B in BATCHES:
        ops, outs = run(B)
        assert _same_rows_as_one_chart(ops, outs, ops1, outs1, 2 * B, 2, f"unet B={B}") > 250
        del ops, outs


def test_decoder_and_encoder_op_by_op_every_batch_equals_one_chart():
    L = 512
    m = model_for(L)
    eng = m.engine
    z = torch.randn(1, 16, L, device="cuda", generator=torch.Generator("cuda").manual_seed(6))
    notes = (torch.rand(1, eng.encoder_cfg.x_channels, 8 * L, device="cuda", generator=torch.Generator("cuda").manual_seed(7)) > 0.9)

    def dec(B):
        ds = eng.decoder_session(B, L)
        eng.ncl_to_rows(z.repeat(B, 1, 1).contiguous(), ds.zin)
        ops = list(ds.plan._arr)
        return ops, _run_op_by_op(eng, ops)

    def enc(B):
        es = eng.encoder_session(B, L)
        eng.ncl_to_rows(notes.float().repeat(B, 1, 1).contiguous(), es.notes_rows)
        ops = list(es.plan._arr)
        return ops, _run_op_by_op(eng, ops)

    for name, make in (("decoder", dec), ("encoder", enc)):
        ops1, outs1 = make(1)
        for B in BATCHES:
            ops, outs = make(B)
            assert _same_rows_as_one_chart(ops, outs, ops1, outs1, B, 1, f"{name} B={B}") > 10
            del ops, outs


@pytest.mark.parametrize("B,name", [(8, "unipc_bh2"), (32, "ddim_eta1")])
def test_every_chart_of_a_large_batch_is_the_chart_alone(B, name):
    """whole requests at the batches where most split GEMMs take the serial kernel and the LayerNorm fold is set by one chart"""
    L = 512
    m = model_for(L)
    kw = request(B, L, seed=99)
    run = RUNS[name]
    z = run(m, seeds=900, **kw)
    for b in range(B):
        assert torch.equal(run(m, seeds=[900 + b], **one_chart(kw, b))[0], z[b]), (name, b)


# ---- 3. every chart of a seeded batch is the chart requested alone -------------------------------------------------------------
RUNS = {
    "ddim_eta0": lambda m, **a: DDIMSampler(m).sample(S=10, eta=0.0, **a)[0],
    "ddim_eta1": lambda m, **a: DDIMSampler(m).sample(S=10, eta=1.0, **a)[0],
    "plms": lambda m, **a: PLMSSampler(m).sample(S=10, **a)[0],
    "dpm2m": lambda m, **a: DPMSolverSampler(m).sample(S=10, **a)[0],
    "unipc_bh2": lambda m, **a: UniPCSampler(m).sample(S=6, **a)[0],
}


def _notes(m, z):
    return m.model.decode_to_hit_objects(z, frame_ms=1000.0 / 60.0)


@pytest.mark.parametrize("L,B", [(96, 4), (512, 4)])
def test_every_chart_of_a_batch_is_the_chart_alone(L, B):
    m = model_for(L)
    kw = request(B, L)
    seed = 500
    for name, run in RUNS.items():
        z = run(m, seeds=seed, **kw)
        logits = m.model.decode(z)
        notes = _notes(m, z)
        for b in range(B):
            zb = run(m, seeds=[seed + b], **one_chart(kw, b))
            assert torch.equal(zb[0], z[b]), (name, b)
            assert torch.equal(m.model.decode(zb)[0], logits[b]), (name, b)
            assert _notes(m, zb)[0] == notes[b], (name, b)


def _simt_plans_are_plain(eng):
    """every op of the `simt` engine's plans: no serial split, no K split, no TF32 hi / lo operand"""
    plans = [s.plan._arr for s in list(eng.sessions.values()) + list(eng.dec_sessions.values())]
    assert plans
    for arr in plans:
        for o in arr:
            assert o.kind != L_.OP_GEMM_SERIAL
            if o.kind == L_.OP_GEMM:
                assert not o.u.gemm.W_hi and not o.u.gemm.W_lo and not o.u.gemm.split_k


def test_simt_engine_every_chart_of_a_batch_is_the_chart_alone():
    """gemm_impl="simt" with batch_invariant: batch_ops leaves the plans alone, and a seeded chart's z, logits and notes are still
    the chart requested alone"""
    L, B = 96, 4
    m = model_for(L, impl="simt")
    kw = request(B, L)
    run = RUNS["ddim_eta0"]
    z = run(m, seeds=500, **kw)
    logits = m.model.decode(z)
    notes = _notes(m, z)
    for b in range(B):
        zb = run(m, seeds=[500 + b], **one_chart(kw, b))
        assert torch.equal(zb[0], z[b]), b
        assert torch.equal(m.model.decode(zb)[0], logits[b]), b
        assert _notes(m, zb)[0] == notes[b], b
    _simt_plans_are_plain(m.engine)


def test_simt_engine_decode_where_the_ffma_tile_flips():
    """32 charts at L = 512: the decoder's plan puts GEMMs on the FFMA kernel's 128 x 128 tiles that one chart runs on 64 x 64
    tiles; every chart's logits are its own decode's, bit for bit"""
    from gemm_cases import ffma_tile
    L, B = 512, 32
    m = model_for(L, impl="simt")
    eng = m.engine
    tiles = lambda n: [ffma_tile(o.u.gemm.M, o.u.gemm.N, eng.sm_count) for o in eng.decoder_session(n, L).plan._arr  # noqa: E731
                       if o.kind == L_.OP_GEMM]
    assert 128 in tiles(B) and 128 not in tiles(1)
    z = torch.randn(B, 16, L, device="cuda", generator=torch.Generator("cuda").manual_seed(11))
    logits = m.model.decode(z)
    for b in range(B):
        assert torch.equal(m.model.decode(z[b:b + 1])[0], logits[b]), b
    _simt_plans_are_plain(eng)


def test_every_chart_of_a_long_batch_is_the_chart_alone():
    L, B = 2048, 2
    m = model_for(L)
    kw = request(B, L)
    z = RUNS["ddim_eta1"](m, seeds=77, **kw)
    for b in range(B):
        zb = RUNS["ddim_eta1"](m, seeds=[77 + b], **one_chart(kw, b))
        assert torch.equal(zb[0], z[b]), b


@pytest.mark.parametrize("L", [96, 512])
def test_ddpm_every_chart_of_a_batch_is_the_chart_alone_and_todays_at_one_chart(L):
    """DDPM with T = 50: chart b of a seeded B = 4 request is the chart alone; the one-chart request is the default engine's"""
    B, T = 4, 50
    m = model_for(L, True, T)
    kw = request(B, L)
    run = lambda mm, **a: DDPMSampler(mm).sample(**a)[0]      # noqa: E731
    z = run(m, seeds=300, **kw)
    for b in range(B):
        assert torch.equal(run(m, seeds=[300 + b], **one_chart(kw, b))[0], z[b]), b
    one = one_chart(kw, 1)
    z_inv = run(m, seeds=301, **one)
    assert torch.equal(run(model_for(L, False, T), seeds=301, **one), z_inv)


# ---- 4. flows from an existing chart -------------------------------------------------------------------------------------------
def test_inpainting_remix_invert_and_encode_are_batch_invariant():
    L, B = 96, 4
    m = model_for(L)
    kw = request(B, L)
    x0, mask = synth.synthetic_inpainting(B, L)
    x0, mask = x0.cuda(), mask.cuda()
    inpaint = {
        "ddim": lambda **a: DDIMSampler(m).sample(S=10, eta=1.0, **a)[0],
        "dpm": lambda **a: DPMSolverSampler(m).inpaint(S=10, **a)[0],
        "unipc": lambda **a: UniPCSampler(m).inpaint(S=6, **a)[0],
    }
    for name, run in inpaint.items():
        ikw = dict(kw, mask=mask, x0=x0)
        z = run(seeds=40, **ikw)
        for b in range(B):
            assert torch.equal(run(seeds=[40 + b], **one_chart(ikw, b))[0], z[b]), (name, b)
    # remix with per-chart strengths (DPM-Solver++ stochastic_encode / decode)
    dpm = DPMSolverSampler(m)
    sched = dpm.make_dpm_schedule(10)
    strengths = [2, 4, 7, 10]
    z = dpm.decode(dpm.stochastic_encode(x0, strengths, sched, seeds=60), t_start=strengths, sched=sched, **_cond(kw))
    for b in range(B):
        one = _cond(one_chart(kw, b))
        zb = dpm.decode(dpm.stochastic_encode(x0[b:b + 1], [strengths[b]], sched, seeds=[60 + b]), t_start=[strengths[b]], sched=sched, **one)
        assert torch.equal(zb[0], z[b]), b
    # DDIM inversion with per-chart t_enc
    ddim = DDIMSampler(m)
    ddim.make_schedule(10, verbose=False)
    t_enc = [3, 5, 7, 10]
    zi = ddim.invert(x0, t_enc=t_enc, **_cond(kw))
    for b in range(B):
        one = _cond(one_chart(kw, b))
        assert torch.equal(ddim.invert(x0[b:b + 1], t_enc=[t_enc[b]], **one)[0], zi[b]), b
    # the chart encoder
    charts = _notes(m, x0)
    mo = m.model.encode_hit_objects(charts, frame_ms=1000.0 / 60.0).mode()
    for b in range(B):
        assert torch.equal(m.model.encode_hit_objects(charts[b:b + 1], frame_ms=1000.0 / 60.0).mode()[0], mo[b]), b


# ---- 5. one chart: the invariant engine is today's engine ---------------------------------------------------------------------
def test_one_chart_is_todays_chart():
    L = 96
    kw = request(1, L)
    for name, run in RUNS.items():
        z_inv = run(model_for(L, True), seeds=9, **kw)
        z_def = run(model_for(L, False), seeds=9, **kw)
        assert torch.equal(z_inv, z_def), name


# ---- 6. the device loop still equals the per-step loop ------------------------------------------------------------------------
def test_device_loop_equals_per_step_loop():
    L, B = 96, 4
    m = model_for(L)
    kw = request(B, L)
    s = DDIMSampler(m)
    z_dev = s.sample(S=10, eta=1.0, seeds=3, **kw)[0]
    z_step = s.sample(S=10, eta=1.0, seeds=3, callback=lambda i: None, **kw)[0]
    assert torch.equal(z_dev, z_step)


# ---- 7. sharded vs one GPU ----------------------------------------------------------------------------------------------------
def _free_port():
    import socket
    sk = socket.socket()
    sk.bind(("127.0.0.1", 0))
    port = sk.getsockname()[1]
    sk.close()
    return port


def _shard_worker(rank, world, port, L, B, out_path):
    import os

    import torch.distributed as dist
    from mug_diffusion_b200.dist import broadcast_blob, sample_sharded

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device(f"cuda:{rank}")
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    cfg = ModelConfig()
    blob = broadcast_blob(synth.synthetic_state_dict(L) if rank == 0 else None, cfg, dev)
    m = MugDiffusionB200(None, cfg, z_length=L, device=dev, blob=blob, batch_invariant=True)
    shapes = dict(x_T=(B, 16, L), c=(B, 128, 21), uc=(B, 128, 21), w0=(B, 256, L), w1=(B, 512, L // 2), w2=(B, 512, L // 4),
                  w3=(B, 512, L // 8))
    req = None
    if rank == 0:
        inp = synth.synthetic_inputs(B, L, seed=3)
        req = dict(x_T=inp["x_T"], c=inp["c"], uc=inp["uc"], w=list(inp["w"])[-4:])

    def run(xT, c, uc, w):
        z, _ = DDIMSampler(m).sample(S=6, c=c, w=w, batch_size=c.shape[0], verbose=False, x_T=xT, eta=0.0, shape=(16, L),
                                     unconditional_guidance_scale=5.0, unconditional_conditioning=uc)
        return m.model.decode(z)

    full = sample_sharded(run, req, shapes, dev)
    if rank == 0:
        torch.save(full.cpu(), out_path)
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_sharded_equals_one_gpu(tmp_path):
    """dist.sample_sharded over two GPUs (two charts per GPU) against the whole batch of four on one GPU, both batch-invariant"""
    import torch.multiprocessing as mp
    L, B = 96, 4
    out_path = str(tmp_path / "gathered.pt")
    mp.spawn(_shard_worker, args=(2, _free_port(), L, B, out_path), nprocs=2, join=True)
    gathered = torch.load(out_path)
    m = MugDiffusionB200(synth.synthetic_state_dict(L), ModelConfig(), z_length=L, batch_invariant=True)
    inp = synth.synthetic_inputs(B, L, seed=3)
    z, _ = DDIMSampler(m).sample(S=6, c=inp["c"].cuda(), w=[t.cuda() for t in inp["w"]], batch_size=B, verbose=False,
                                 x_T=inp["x_T"].cuda(), eta=0.0, shape=(16, L), unconditional_guidance_scale=5.0,
                                 unconditional_conditioning=inp["uc"].cuda())
    assert torch.equal(gathered, m.model.decode(z).cpu())

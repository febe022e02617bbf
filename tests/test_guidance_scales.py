"""Per-chart guidance scales on the CPU: every sampler entry point refuses malformed scales before any device call, a list of equal
scales (or all 1) takes exactly today's call, a mix takes the guided-scales session, whose plan is a copy op + today's U-Net op list +
one MUGD_OP_CFG_SCALES, and the new op kind is laid out and checked as the C header says."""
import ctypes as C
import hashlib
import os
import subprocess
import threading
import types

import numpy as np
import pytest
import torch

from mug_diffusion_b200 import dpm_solver, packer, synth, unipc
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200.config import ModelConfig
from mug_diffusion_b200.engine import Arena, UNetCompiler, View, guided_scales_ops, tc_weight_map
from mug_diffusion_b200.runtime import MugEngine, Session
from mug_diffusion_b200.sampler import (DDIMSampler, DDPMSampler, DPMSolverSampler, PLMSSampler, UniPCSampler, alphas_cumprod_f64,
                                        guidance_scales, register_schedule)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WBASE = 1 << 45                                   # fake weight address, far from any host allocation
VALID = 1 << 43                                   # fake device address of the valid-length arrays
OUT, SCALES = 1 << 44, (1 << 44) + (1 << 30)      # fake device addresses of the guided rows and the scales


# ---- refusals before any device call ----------------------------------------------------------------------------------------------
class _NoGpu:
    def __getattr__(self, name):
        raise AssertionError(f"engine.{name} used before the refusal")


def _cpu(cls, engine=None):
    s = object.__new__(cls)
    s.model = types.SimpleNamespace(engine=engine or _NoGpu(), z_channels=16, z_length=96, num_timesteps=1000, cfg=ModelConfig(),
                                    clip_denoised=True, **register_schedule())
    s.ddpm_num_timesteps, s.device, s.last_launches_per_step = 1000, torch.device("cpu"), 0
    return s


INP = synth.synthetic_inputs(2, 96)
X0 = torch.zeros(2, 16, 96)
MASK = torch.ones(2, 1, 96)
ACP = alphas_cumprod_f64(ModelConfig())
DSCH, USCH = dpm_solver.multistep_schedule(ACP, 10, 2), unipc.multistep_schedule(ACP, 10, 2)


def _req(scale, **kw):
    out = dict(c=INP["c"], w=INP["w"], batch_size=2, shape=(16, 96), verbose=False, unconditional_guidance_scale=scale,
               unconditional_conditioning=INP["uc"], x_T=INP["x_T"].expand(2, 16, 96).contiguous())
    out.update(kw)
    return out


def _ddim(engine=None):
    s = _cpu(DDIMSampler, engine)
    s.make_schedule(10, verbose=False)
    return s


def _plms(engine=None):
    s = _cpu(PLMSSampler, engine)
    s.make_schedule(10, verbose=False)
    return s


FLOWS = {
    "ddim.sample": lambda s, e: _cpu(DDIMSampler, e).sample(S=10, **_req(s)),
    "ddim.ddim_sampling": lambda s, e: _ddim(e).ddim_sampling(INP["w"], INP["c"], (2, 16, 96), x_T=X0, unconditional_guidance_scale=s,
                                                              unconditional_conditioning=INP["uc"]),
    "ddim.inpaint": lambda s, e: _cpu(DDIMSampler, e).sample(S=10, mask=MASK, x0=X0, **_req(s)),
    "ddim.decode": lambda s, e: _ddim(e).decode(X0, INP["c"], INP["w"], 3, unconditional_guidance_scale=s,
                                                unconditional_conditioning=INP["uc"]),
    "ddim.invert": lambda s, e: _ddim(e).invert(X0, INP["c"], INP["w"], 3, unconditional_guidance_scale=s,
                                                unconditional_conditioning=INP["uc"], verbose=False),
    "plms.sample": lambda s, e: _cpu(PLMSSampler, e).sample(S=10, **_req(s)),
    "plms.plms_sampling": lambda s, e: _plms(e).plms_sampling(INP["w"], INP["c"], (2, 16, 96), x_T=X0, unconditional_guidance_scale=s,
                                                              unconditional_conditioning=INP["uc"]),
    "ddpm.sample": lambda s, e: _cpu(DDPMSampler, e).sample(**_req(s)),
    "dpm.sample": lambda s, e: _cpu(DPMSolverSampler, e).sample(S=10, **_req(s)),
    "dpm.inpaint": lambda s, e: _cpu(DPMSolverSampler, e).inpaint(S=10, mask=MASK, x0=X0, **_req(s)),
    "dpm.decode": lambda s, e: _cpu(DPMSolverSampler, e).decode(X0, INP["c"], INP["w"], 3, DSCH, unconditional_guidance_scale=s,
                                                                unconditional_conditioning=INP["uc"]),
    "dpm.invert": lambda s, e: _cpu(DPMSolverSampler, e).invert(X0, INP["c"], INP["w"], 3, DSCH, unconditional_guidance_scale=s,
                                                                unconditional_conditioning=INP["uc"], verbose=False),
    "unipc.sample": lambda s, e: _cpu(UniPCSampler, e).sample(S=10, **_req(s)),
    "unipc.inpaint": lambda s, e: _cpu(UniPCSampler, e).inpaint(S=10, mask=MASK, x0=X0, **_req(s)),
    "unipc.decode": lambda s, e: _cpu(UniPCSampler, e).decode(X0, INP["c"], INP["w"], 3, USCH, unconditional_guidance_scale=s,
                                                              unconditional_conditioning=INP["uc"]),
    "unipc.invert": lambda s, e: _cpu(UniPCSampler, e).invert(X0, INP["c"], INP["w"], 3, USCH, unconditional_guidance_scale=s,
                                                              unconditional_conditioning=INP["uc"], verbose=False),
}


BAD = [([5.0], "1 entries for 2 charts"), ([5.0, 5.0, 5.0], "3 entries for 2 charts"), (np.array([5.0]), "1 entries"),
       ([5.0, float("nan")], "finite number"), ([float("inf"), 5.0], "finite number"), (torch.tensor([5.0, float("-inf")]), "finite"),
       ([True, 5.0], "finite number"), ([5.0, "7"], "finite number"), ((5.0, None), "finite number"),
       (torch.tensor([True, False]), "finite number"), ([[5.0], [5.0]], "finite number")]


@pytest.mark.parametrize("flow", sorted(FLOWS))
@pytest.mark.parametrize("scale,msg", BAD, ids=[f"bad{i}" for i in range(len(BAD))])
def test_every_flow_refuses_malformed_scales_before_any_gpu_work(flow, scale, msg):
    with pytest.raises(ValueError, match=msg):
        FLOWS[flow](scale, None)


def test_guidance_scales_normalises():
    assert guidance_scales(5.0, 2) == 5.0 and guidance_scales(7, 3) == 7
    assert guidance_scales([3, 3], 2) == 3.0 and isinstance(guidance_scales([3, 3], 2), float)
    assert guidance_scales(np.array([1.0, 1.0], np.float32), 2) == 1.0
    assert guidance_scales(torch.tensor([1.0, 3.0, 5.0, 7.5]), 4) == [1.0, 3.0, 5.0, 7.5]
    assert guidance_scales((np.float32(2.5), np.int64(4)), 2) == [2.5, 4.0]
    t = torch.tensor(5.0)                                        # a 0-d tensor is one number, passed on as today
    assert guidance_scales(t, 2) is t


# ---- which path a request takes ---------------------------------------------------------------------------------------------------
class _Reached(Exception):
    pass


class _Stop:
    """stands in for the engine up to its first session: records how the session was asked for, then stops the request"""

    def __init__(self):
        self.lock = threading.RLock()
        self.calls = []

    def session(self, *a, **kw):
        self.calls.append((a, kw))
        raise _Reached


SAMPLE_FLOWS = ["ddim.sample", "plms.sample", "ddpm.sample", "dpm.sample", "unipc.sample", "dpm.inpaint", "unipc.inpaint",
                "ddim.decode", "dpm.decode", "unipc.decode", "ddim.invert", "dpm.invert", "unipc.invert"]


def _session_call(flow, scale):
    e = _Stop()
    with pytest.raises(_Reached):
        FLOWS[flow](scale, e)
    assert len(e.calls) == 1
    return e.calls[0]


@pytest.mark.parametrize("flow", SAMPLE_FLOWS)
def test_equal_scales_take_todays_call_and_a_mix_the_guided_session(flow):
    today = _session_call(flow, 5.0)
    assert today == ((4, 96), dict(per_sample_t=False, ragged=False, unit=2))
    for same in ([5.0, 5.0], (5, 5), np.array([5.0, 5.0]), torch.tensor([5.0, 5.0])):
        assert _session_call(flow, same) == today
    unguided = _session_call(flow, 1.0)
    assert unguided == ((2, 96), dict(per_sample_t=False, ragged=False, unit=1))
    assert _session_call(flow, [1.0, 1.0]) == unguided
    assert _session_call(flow, [1.0, 5.0]) == ((4, 96), dict(per_sample_t=False, ragged=False, unit=2, guided=True))
    assert _session_call(flow, torch.tensor([3.0, 7.5])) == ((4, 96), dict(per_sample_t=False, ragged=False, unit=2, guided=True))


def test_scales_without_unconditional_conditioning_are_unguided():
    e = _Stop()
    with pytest.raises(_Reached):
        _cpu(DDIMSampler, e).sample(S=10, **_req([1.0, 5.0], unconditional_conditioning=None))
    assert e.calls == [((2, 96), dict(per_sample_t=False, ragged=False, unit=1))]


def test_forced_path_and_ragged_requests_take_the_guided_session(monkeypatch):
    e = _Stop()
    s = _cpu(DDIMSampler, e)
    monkeypatch.setattr(s, "force_per_chart_scales", True)
    with pytest.raises(_Reached):
        s.sample(S=10, **_req(5.0))
    with pytest.raises(_Reached):
        _cpu(DDIMSampler, e).sample(S=10, **_req([2.0, 5.0], z_lengths=[64, 96]))
    assert e.calls == [((4, 96), dict(per_sample_t=False, ragged=False, unit=2, guided=True)),
                       ((4, 96), dict(per_sample_t=False, ragged=True, unit=2, guided=True))]


# ---- the guided-scales plan --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def blob():
    cfg = ModelConfig()
    b = packer.pack_model(synth.synthetic_state_dict(96), cfg.unet, cfg.decoder)
    return cfg, b, tc_weight_map(b, WBASE)


def _ext(comp, Beff, Lz):
    blocks = list(comp.lay.blocks())
    ctx_kv = [View((1 << 41) + i * (1 << 24), 2 * b.cin, Beff * 21, 2 * b.cin) for i, b in enumerate(x for x in blocks if x.kind == "attn")]
    s4 = {b.prefix: View((1 << 42) + i * (1 << 24), b.cin, Lz // b.ds, b.cin) for i, b in enumerate(x for x in blocks if x.kind == "s4")}
    return dict(emb_table=1 << 40, step=(1 << 40) + 4096, ctx_tokens=21, ctx_kv=ctx_kv, s4_kt=s4)


def _compile(blob, Beff, Lz, ragged):
    cfg, b, tc = blob
    comp = UNetCompiler(cfg.unet, b, WBASE, tc)
    valid = [VALID + 256 * l for l in range(cfg.unet.levels)] if ragged else None
    return comp.compile(Arena(1 << 32), Beff, Lz, _ext(comp, Beff, Lz), False, None, valid)


def _check_guided(ops, plain, xin, eps, B, Lz, out, scales):
    """ops = the copy of x into the second half + ``plain`` field for field + one MUGD_OP_CFG_SCALES"""
    assert len(ops) == len(plain) + 2
    cp = ops[0]
    assert cp.kind == L_.OP_COPY2D
    assert (cp.u.cp.src, cp.u.cp.lds, cp.u.cp.dst, cp.u.cp.ldd) == (xin.ptr, xin.ld, xin.ptr + 4 * B * Lz * xin.ld, xin.ld)
    assert (cp.u.cp.rows, cp.u.cp.cols) == (B * Lz, 16)
    assert all(bytes(a) == bytes(b) for a, b in zip(ops[1:-1], plain))
    g = ops[-1]
    assert g.kind == L_.OP_CFG_SCALES
    d = g.u.cfgs
    assert (d.eps, d.ld, d.out, d.scales, d.B, d.L, d.C) == (eps.ptr, eps.ld, out, scales, B, Lz, 16)


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("B", [1, 2, 4])
def test_guided_plan_is_copy_plus_todays_unet_plus_cfg_scales(blob, B, ragged):
    Lz = 96
    res = _compile(blob, 2 * B, Lz, ragged)
    before = hashlib.sha256(bytes(res["ops"].array())).hexdigest()
    plain = [L_.Op.from_buffer_copy(o) for o in res["ops"].ops]
    g = guided_scales_ops(res["ops"], res["xin"], res["eps"], B, Lz, OUT, SCALES)
    _check_guided(g.ops, plain, res["xin"], res["eps"], B, Lz, OUT, SCALES)
    assert hashlib.sha256(bytes(res["ops"].array())).hexdigest() == before          # today's list is left as it was


def test_plain_plans_keep_their_hashes(blob):
    """the hashes pinned for today's plans (tests/test_ragged.py) are those of the op lists compiled here"""
    cfg = ModelConfig()
    b = blob[1]
    comp = UNetCompiler(cfg.unet, b, 1 << 30)
    want = {(8, 512): "7ca81e628501890132bbf980e5645f86545e4c3eeb48aae468995a5eea4816cd",
            (2, 96): "ec77cfd9f7afb8773494f2c4ec05d6ac29ad014b3e95f5c39e72c6380890c619"}
    for (Beff, Lz), h in want.items():
        res = comp.compile(Arena(1 << 32), Beff, Lz, _ext(comp, Beff, Lz), False, None, None)
        assert hashlib.sha256(bytes(res["ops"].array())).hexdigest() == h


class _HostEngine(MugEngine):
    def __del__(self):                                          # its handle is a zeroed host buffer, not one mugd_create made
        pass


def _cpu_engine(blob, on: bool):
    """a MugEngine whose plans are compiled and created but never run (mugd_plan_create only stores the ops)"""
    cfg, b, tc = blob
    e = object.__new__(_HostEngine)
    e.batch_invariant, e.gemm_impl, e.sm_count = on, "auto", 132
    e._handle_buf = (C.c_char * 4096)()
    e.cfg, e.blob, e.device, e.lib, e.handle = cfg, b, torch.device("cpu"), L_.load(), C.c_void_p(C.addressof(e._handle_buf))
    e.wbase, e.tc_map, e.fold_ln = WBASE, tc, None
    e.tc_ws, e.tc_counters = torch.zeros(64), torch.zeros(64, dtype=torch.int32)
    e.sessions, e.dec_sessions, e.max_sessions = {}, {}, 4
    return e


def _cpu_session(eng, Beff, Lz, unit, guided, like=None):
    """runtime.Session._build on the host: the side buffers __init__ makes (those of ``like`` when given), without its S4 kernel
    generation on the device"""
    s = object.__new__(Session)
    cfg = eng.cfg.unet
    s.engine, s.Beff, s.Lz, s.per_sample_t, s.unit, s.valid, s.lens = eng, Beff, Lz, False, unit, None, None
    if guided:
        s.scales, s.e_guided = torch.ones(Beff // 2), torch.zeros(Beff // 2 * Lz, cfg.out_channels)
    s.comp = UNetCompiler(cfg, eng.blob, eng.wbase, eng.tc_map)
    if like is not None:
        for k in ("emb_table", "temb", "emb_h1", "emb_h2", "step", "coef", "ctx", "ctx_kv", "ctx_tokens", "s4_kt"):
            setattr(s, k, getattr(like, k))
    else:
        s.emb_table = torch.zeros(1000, eng.blob.meta["emb_total"])
        s.temb, s.emb_h1, s.emb_h2 = (torch.zeros(1000, c) for c in (cfg.model_channels, cfg.time_embed_dim, cfg.time_embed_dim))
        s.step, s.coef = torch.zeros(1, dtype=torch.int32), torch.zeros(1000, 4)
        s.ctx = torch.zeros(Beff * 64, cfg.context_dim)
        s.ctx_kv = [torch.zeros(Beff * 64, 2 * b.cin) for b in s.comp.lay.blocks() if b.kind == "attn"]
        s.ctx_tokens = 21
        s.s4_kt = {b.prefix: torch.zeros(Lz // b.ds, b.cin) for b in s.comp.lay.blocks() if b.kind == "s4"}
    s._build()
    return s


def _arena(s):
    return (s.arena_t.data_ptr() + 255) // 256 * 256, s.arena_t.numel() * 4


def _pointer_offsets(t, base=0):
    """byte offsets of the pointer fields of the ctypes structure ``t`` (nested structures included)"""
    out = []
    for name, ft in t._fields_:
        off = base + getattr(t, name).offset
        if ft is C.c_void_p:
            out.append(off)
        elif isinstance(ft, type) and issubclass(ft, C.Structure):
            out += _pointer_offsets(ft, off)
    return out


def _rebased(ops, old, new: int):
    """the raw bytes of ``ops`` with every pointer field inside the arena ``old`` = (base, bytes) moved to the same offset from
    ``new`` (two sessions' arenas)"""
    out = []
    for o in ops:
        raw = bytearray(bytes(o))
        member = L_._KIND_FIELD[o.kind]
        for off in _pointer_offsets(type(getattr(o.u, member)), L_.Op.u.offset + getattr(L_._OpU, member).offset):
            v = int.from_bytes(raw[off:off + 8], "little")
            if old[0] <= v < old[0] + old[1]:
                raw[off:off + 8] = (v - old[0] + new).to_bytes(8, "little")
        out.append(bytes(raw))
    return out


@pytest.mark.parametrize("invariant", [False, True])
def test_guided_session_plan_and_descriptors(blob, invariant):
    """through runtime.Session: the guided plan is the copy + the plain session's U-Net op list (batch policy included) + CFG_SCALES;
    every update descriptor reads the guided rows unguided and writes the first half of x only"""
    eng = _cpu_engine(blob, invariant)
    B, Lz = 4, 96
    plain = _cpu_session(eng, 2 * B, Lz, 2, False)
    guided = _cpu_session(eng, 2 * B, Lz, 2, True, like=plain)
    g_ops, p_ops = list(guided.plan._arr), list(plain.plan._arr)
    assert guided.plan.n_ops == plain.plan.n_ops + 2
    # the sessions share their side buffers; their arenas differ, so the guided ops are compared with their arena moved onto the plain one
    assert _rebased(g_ops[1:-1], _arena(guided), _arena(plain)[0]) == [bytes(o) for o in p_ops]
    assert invariant == any(o.kind == L_.OP_GEMM_SERIAL or o.kind == L_.OP_GEMM and o.u.gemm.split_k for o in p_ops)
    _check_guided(g_ops, g_ops[1:-1], guided.xin, guided.eps, B, Lz, guided.e_guided.data_ptr(), guided.scales.data_ptr())
    # descriptors: eps = the guided rows, cfg = 0, x_dup = NULL
    ring, coef = torch.zeros(3, B * Lz * 16), torch.zeros(10, 8)
    for d in (guided.ddim_update(B, 10, True, 5.0, 1.0, 0), guided.dpm(B, 10, True, 5.0, 0, ring, coef),
              guided.ddpm(B, 10, True, 5.0, True, 0, 0, torch.zeros(10, 5))):
        assert (d.eps, d.cfg, d.x_dup, d.x) == (guided.e_guided.data_ptr(), 0, None, guided.xin.ptr)
    p = guided.plms(B, 10, True, 5.0, 0, torch.zeros(5, B * Lz * 16))
    assert (p.eps, p.cfg, p.update.x_dup) == (guided.e_guided.data_ptr(), 0, None)
    assert (guided.ddim_stage(B, True).x_dup, guided.join(B, True, 0, 0).x_dup) == (None, None)
    # today's session keeps its descriptors
    d = plain.ddim_update(B, 10, True, 5.0, 1.0, 0)
    assert (d.eps, d.cfg, d.scale, d.x_dup) == (plain.eps.ptr, 1, 5.0, plain.xin.r(B * Lz, 2 * B * Lz).ptr)


# ---- C ABI ---------------------------------------------------------------------------------------------------------------------
def test_abi_cfg_scales_layout(tmp_path):
    assert L_.ABI_VERSION == 13 and C.sizeof(L_.Op) == 256 and L_.OP_CFG_SCALES == 18
    t = L_.CfgScales
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mugd.h"\nint main(void) {\n'
                   '  printf("%zu %d %zu", sizeof(mugd_op), MUGD_OP_CFG_SCALES, sizeof(mugd_cfg_scales));\n'
                   + "".join(f'  printf(" %zu", offsetof(mugd_cfg_scales, {f}));\n' for f, _ in t._fields_)
                   + '  printf(" %zu\\n", offsetof(mugd_op, u.cfgs));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-o", str(exe), str(src), "-I" + os.path.join(ROOT, "include")], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [256, 18, C.sizeof(t)] + [getattr(t, f).offset for f, _ in t._fields_] + [L_.Op.u.offset]
    assert C.sizeof(t) == 48


def test_abi_sizes_fills_entry_16_only_at_17():
    lib = L_.load()
    sizes = (C.c_int32 * 17)(*([-1] * 17))
    assert lib.mugd_abi_sizes(sizes, 16) == 0 and sizes[15] == C.sizeof(L_.RowMask) and sizes[16] == -1
    assert lib.mugd_abi_sizes(sizes, 17) == 0 and sizes[16] == C.sizeof(L_.CfgScales)
    assert lib.mugd_abi_version() == 13


def _desc(**kw):
    d = L_.CfgScales()
    d.eps, d.ld, d.out, d.scales, d.B, d.L, d.C = 1 << 32, 16, (1 << 32) + (1 << 24), 1 << 33, 2, 96, 16
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("kw,msg", [
    (dict(eps=None), "must be given"), (dict(out=None), "must be given"), (dict(scales=None), "must be given"),
    (dict(B=0), "bad shape"), (dict(L=0), "bad shape"), (dict(C=0), "bad shape"), (dict(ld=15), "bad shape"),
    (dict(out=(1 << 32) + 4 * (4 * 96 - 1) * 16), "overlaps"), (dict(out=(1 << 32) - 4 * 2 * 96 * 16 + 4), "overlaps"),
    (dict(B=1 << 16, L=1 << 12), "bad shape")])
def test_cfg_scales_refusals_before_any_device_call(kw, msg):
    """mugd_op_run on a zeroed handle (no device behind it): every refusal comes from the host checks"""
    lib = L_.load()
    handle = (C.c_char * 4096)()
    op = L_.make_op(L_.OP_CFG_SCALES, _desc(**kw))
    assert lib.mugd_op_run(C.cast(handle, C.c_void_p), C.byref(op), None) == 1
    assert msg in lib.mugd_last_error().decode()

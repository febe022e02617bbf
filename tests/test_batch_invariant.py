"""Batch-invariant plans on the CPU: with the policy off every plan is today's, field for field; with it on every tensor-core GEMM of a
plan for B charts takes the tile width, K split and K-range bounds of the one-chart plan, and the serial-split op kind is checked
before any device call and laid out as the C header says."""
import ctypes as C
import os
import subprocess
import types

import pytest
import torch

from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import packer, synth
from mug_diffusion_b200.config import EncoderConfig, ModelConfig
from mug_diffusion_b200.engine import (Arena, DecoderCompiler, EncoderCompiler, UNetCompiler, View, gemm_runs_tc, tc_plan_of,
                                       tc_weight_map, unit_batch_splits)
from mug_diffusion_b200.runtime import DecoderSession, EncoderSession, MugEngine, Session

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMS = 132
WBASE = 1 << 30
GEMMS = (L_.OP_GEMM, L_.OP_GEMM_SERIAL)


@pytest.fixture(scope="module")
def blob():
    cfg = ModelConfig()
    sd = {**synth.synthetic_state_dict(96), **synth.synthetic_encoder_state_dict()}
    b = packer.pack_model(sd, cfg.unet, cfg.decoder, encoder_cfg=cfg.encoder)
    return cfg, b, tc_weight_map(b, WBASE)


def _ext(comp, Beff, Lz):
    blocks = list(comp.lay.blocks())
    ctx_kv = [View((1 << 41) + i * (1 << 24), 2 * b.cin, Beff * 21, 2 * b.cin) for i, b in enumerate(x for x in blocks if x.kind == "attn")]
    s4 = {b.prefix: View((1 << 42) + i * (1 << 24), b.cin, Lz // b.ds, b.cin) for i, b in enumerate(x for x in blocks if x.kind == "s4")}
    return dict(emb_table=1 << 40, step=(1 << 40) + 4096, ctx_tokens=21, ctx_kv=ctx_kv, s4_kt=s4)


def _unet(blob, Beff, Lz, per_sample_t=False, fold=None):
    cfg, b, tc = blob
    comp = UNetCompiler(cfg.unet, b, WBASE, tc)
    return comp.compile(Arena(1 << 32), Beff, Lz, _ext(comp, Beff, Lz), per_sample_t, fold, None)["ops"]


def _engine(on: bool, impl: str = "auto"):
    """a MugEngine without a device: only the batch policy (batch_ops) is used"""
    e = object.__new__(MugEngine)
    e.batch_invariant, e.gemm_impl, e.sm_count = on, impl, SMS
    return e


def _geometry(g) -> tuple:
    """(tile width, K splits, K-range bounds in k-steps) the tensor-core planner runs ``g`` with at 132 SMs"""
    tile_n, per_sm, ctas = C.c_int32(), C.c_int32(), C.c_int32()
    assert L_.load().mugd_gemm_tc_variant(C.byref(g), SMS, C.byref(tile_n), C.byref(per_sm), C.byref(ctas)) == 0
    sup, sp, _ = tc_plan_of(g, SMS)
    assert sup
    total = (g.taps * g.K + g.K2) // 32
    base, rem = divmod(total, sp)
    bounds = [z * base + min(z, rem) for z in range(sp + 1)]
    return tile_n.value, sp, tuple(bounds)


# ---- policy off: today's plans -----------------------------------------------------------------------------------------------
def test_policy_off_leaves_every_plan_as_it_is(blob):
    cfg, b, tc = blob
    off = _engine(False)
    for per_sample_t in (False, True):
        ops = _unet(blob, 8, 512, per_sample_t)
        want = bytes(ops.array())
        assert bytes(off.batch_ops(ops, 8, 2).array()) == want
    dec = DecoderCompiler(cfg.decoder, b, WBASE, tc).compile(Arena(1 << 32), 4, 512)["ops"]
    want = bytes(dec.array())
    assert bytes(off.batch_ops(dec, 4, 1).array()) == want
    enc = EncoderCompiler(EncoderConfig(), b, WBASE, tc).compile(Arena(1 << 32), 4, 96)["ops"]
    want = bytes(enc.array())
    assert bytes(off.batch_ops(enc, 4, 1).array()) == want
    # the exact-fp32 FFMA path keeps its plans under the policy too
    ops = _unet(blob, 8, 96)
    want = bytes(ops.array())
    assert bytes(_engine(True, "simt").batch_ops(ops, 8, 1).array()) == want


# ---- policy on: every GEMM takes the one-chart geometry ------------------------------------------------------------------------
@pytest.mark.parametrize("Lz", [96, 512, 2048])
@pytest.mark.parametrize("cfg_on", [True, False])
def test_unet_gemms_take_the_one_chart_geometry(blob, Lz, cfg_on):
    unit = 2 if cfg_on else 1
    fold = unit * Lz < 8192                                     # Session._build's rule under the policy
    one = _unet(blob, unit, Lz, fold=fold)
    one_bytes = bytes(one.array())
    geo1 = [_geometry(o.u.gemm) if o.kind == L_.OP_GEMM and tc_plan_of(o.u.gemm, SMS)[0] else None for o in one.ops]
    # at one chart the invariant plan is today's plan
    assert bytes(unit_batch_splits(one, unit, unit, SMS).array()) == one_bytes
    n_serial = {}
    for B in (2, 3, 4, 8, 32):
        ops = unit_batch_splits(_unet(blob, B * unit, Lz, fold=fold), B * unit, unit, SMS)
        assert len(ops.ops) == len(one.ops)
        checked = 0
        for o, o1, g1 in zip(ops.ops, one.ops, geo1):
            if o1.kind != L_.OP_GEMM:
                assert o.kind == o1.kind
                continue
            assert o.kind in GEMMS
            if g1 is None:                                      # FFMA-path shape: no K split to pin
                assert o.kind == L_.OP_GEMM and o.u.gemm.split_k == 0
                continue
            g = o.u.gemm
            assert _geometry(g) == g1, (B, g.M, g.N, g.K)
            _, _, tiles = tc_plan_of(g, SMS)
            # the serial kind exactly where the forced split would exceed the split-K kernel's partial-tile bound
            assert (o.kind == L_.OP_GEMM_SERIAL) == (g1[1] > 1 and tiles * g1[1] > 2 * SMS and g.split_k > 0)
            checked += 1
        assert checked > 100
        n_serial[B] = sum(o.kind == L_.OP_GEMM_SERIAL for o in ops.ops)
    if Lz == 512:
        assert n_serial[32] > 0                                 # the large batches do take the serial variant


def test_per_sample_t_decoder_and_encoder_take_the_one_chart_geometry(blob):
    cfg, b, tc = blob

    def check(make, unit):
        one = make(unit).ops
        for B in (2, 3, 8, 32):
            ops = unit_batch_splits(make(B * unit), B * unit, unit, SMS).ops
            n = 0
            for o, o1 in zip(ops, one):
                if o1.kind == L_.OP_GEMM and tc_plan_of(o1.u.gemm, SMS)[0]:
                    assert _geometry(o.u.gemm) == _geometry(o1.u.gemm)
                    n += 1
            assert n > 5

    check(lambda Beff: _unet(blob, Beff, 96, per_sample_t=True, fold=True), 1)
    check(lambda B: DecoderCompiler(cfg.decoder, b, WBASE, tc).compile(Arena(1 << 32), B, 96)["ops"], 1)
    check(lambda B: EncoderCompiler(EncoderConfig(), b, WBASE, tc).compile(Arena(1 << 32), B, 96)["ops"], 1)


def test_policy_refuses_a_batch_that_is_not_whole_charts(blob):
    ops = _unet(blob, 3, 96)
    with pytest.raises(ValueError):
        unit_batch_splits(ops, 3, 2, SMS)


def test_session_keys_are_todays_with_the_policy_off():
    made = []
    for on in (False, True):
        e = _engine(on)
        e.sessions, e.max_sessions = {}, 4
        e._lru_get = lambda cache, key, make: made.append(key)
        e.session(4, 96, unit=2)
    assert made[0] == (4, 96, False) and made[1] == (4, 96, False, ("unit", 2))


# ---- the serial-split op kind --------------------------------------------------------------------------------------------------
def test_serial_op_layout_matches_the_header(tmp_path):
    assert L_.OP_GEMM_SERIAL == 17 and L_.ABI_VERSION == 13 and C.sizeof(L_.Op) == 256
    op = L_.make_op(L_.OP_GEMM_SERIAL, L_.Gemm())
    assert C.addressof(op.u.gemm) == C.addressof(op.u)
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mugd.h"\nint main(void) {\n'
                   '  printf("%d %d %zu %zu %zu\\n", MUGD_ABI_VERSION, MUGD_OP_GEMM_SERIAL, sizeof(mugd_op), sizeof(mugd_gemm), '
                   'offsetof(mugd_op, u.gemm));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-o", str(exe), str(src), "-I" + os.path.join(ROOT, "include")], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert out == ["13", "17", "256", str(C.sizeof(L_.Gemm)), str(L_.Op.u.offset)]
    lib = L_.load()
    sizes = (C.c_int32 * 16)()
    assert lib.mugd_abi_sizes(sizes, 13) == 0 and lib.mugd_abi_sizes(sizes, 16) == 0 and sizes[1] == C.sizeof(L_.Gemm)


def _serial_gemm(**kw):
    """a valid serial-split descriptor at fake, aligned device addresses"""
    g = L_.Gemm()
    g.A, g.lda, g.W, g.W_hi, g.W_lo = 1 << 40, 512, 1 << 41, 1 << 41, 1 << 42
    g.C, g.ldc = 1 << 43, 512
    g.M, g.N, g.K, g.taps, g.conv_mode, g.Lin, g.Lout = 2048, 512, 512, 1, L_.CONV_NONE, 64, 64
    g.impl, g.split_k = L_.GEMM_TC, 4
    for k, v in kw.items():
        setattr(g, k, v)
    return g


@pytest.mark.parametrize("kw,msg", [
    (dict(impl=L_.GEMM_SIMT), "tensor-core path only"),
    (dict(split_k=0), "forced K split"),
    (dict(split_k=17), "more splits than k-steps"),
    (dict(K=48), "does not take"),
    (dict(W_lo=0), "hi / lo"),
    (dict(ldc=3), "C alignment"),
])
def test_serial_op_refuses_bad_descriptors_before_any_device_call(kw, msg):
    """mugd_op_run on a zeroed handle (no device behind it): every refusal comes from the host checks"""
    lib = L_.load()
    handle = (C.c_char * 4096)()
    op = L_.make_op(L_.OP_GEMM_SERIAL, _serial_gemm(**kw))
    assert lib.mugd_op_run(C.cast(handle, C.c_void_p), C.byref(op), None) == 1
    assert msg in lib.mugd_last_error().decode()


# ---- through the sessions: the plans, fold rule and per-request ops the engine builds -----------------------------------------
class _HostEngine(MugEngine):
    def __del__(self):                                          # its handle is a zeroed host buffer, not one mugd_create made
        pass


def _cpu_engine(blob, on: bool):
    """a MugEngine whose plans are compiled and created but never run: arenas on the host, a zeroed handle (mugd_plan_create only
    stores the ops)"""
    cfg, b, tc = blob
    e = object.__new__(_HostEngine)
    e.batch_invariant, e.gemm_impl, e.sm_count = on, "auto", SMS
    e._handle_buf = (C.c_char * 4096)()
    e.cfg, e.blob, e.device, e.lib, e.handle = cfg, b, torch.device("cpu"), L_.load(), C.c_void_p(C.addressof(e._handle_buf))
    e.wbase, e.tc_map, e.fold_ln = WBASE, tc, None
    e.tc_ws, e.tc_counters = torch.zeros(64), torch.zeros(64, dtype=torch.int32)
    e.sessions, e.dec_sessions, e.max_sessions = {}, {}, 4
    return e


def _cpu_session(eng, Beff, Lz, unit, per_sample_t=False):
    """runtime.Session._build on the host: the side buffers __init__ makes, without its S4 kernel generation on the device"""
    s = object.__new__(Session)
    cfg = eng.cfg.unet
    s.engine, s.Beff, s.Lz, s.per_sample_t, s.unit, s.valid, s.lens = eng, Beff, Lz, per_sample_t, unit, None, None
    s.comp = UNetCompiler(cfg, eng.blob, eng.wbase, eng.tc_map)
    rows = Beff if per_sample_t else 1000
    s.emb_table = torch.zeros(rows, eng.blob.meta["emb_total"])
    s.temb, s.emb_h1, s.emb_h2 = (torch.zeros(rows, c) for c in (cfg.model_channels, cfg.time_embed_dim, cfg.time_embed_dim))
    s.step = torch.zeros(1, dtype=torch.int32)
    s.ctx = torch.zeros(Beff * 64, cfg.context_dim)
    s.ctx_kv = [torch.zeros(Beff * 64, 2 * b.cin) for b in s.comp.lay.blocks() if b.kind == "attn"]
    s.ctx_tokens = 21
    s.s4_kt = {b.prefix: torch.zeros(Lz // b.ds, b.cin) for b in s.comp.lay.blocks() if b.kind == "s4"}
    s._build()
    return s


def _geometries(ops):
    return [_geometry(o.u.gemm) if o.kind in GEMMS and gemm_runs_tc(o.u.gemm, SMS) else (o.kind,) for o in ops]


def test_sessions_take_the_one_chart_plan_and_fold_rule(blob):
    cfg, b, tc = blob
    L = 1024                                                    # 8 charts' rows cross the LayerNorm fold's 8192-row rule
    on, off = _cpu_engine(blob, True), _cpu_engine(blob, False)
    one = _cpu_session(on, 2, L, 2)
    many = _cpu_session(on, 8, L, 2)
    today = _cpu_session(off, 8, L, 1)
    assert one.ln_folded and many.ln_folded and not today.ln_folded
    assert _geometries(many.plan._arr) == _geometries(one.plan._arr)
    assert any(o.kind == L_.OP_GEMM_SERIAL or o.u.gemm.split_k for o in many.plan._arr if o.kind in GEMMS)
    assert all(o.kind != L_.OP_GEMM_SERIAL and not (o.kind == L_.OP_GEMM and o.u.gemm.split_k) for o in today.plan._arr)
    # per-request ops: cross-attention K|V projections of the whole batch, per-sample timestep rows
    ctx = lambda s: s.context_ops([(1 << 44, s.Beff)], 21).ops          # noqa: E731
    assert _geometries(ctx(many)) == _geometries(ctx(one))
    assert not any(o.kind == L_.OP_GEMM and o.u.gemm.split_k for o in ctx(today))
    t1, t8 = _cpu_session(on, 1, 96, 1, per_sample_t=True), _cpu_session(on, 32, 96, 1, per_sample_t=True)
    assert _geometries(t8.timestep_ops(32).ops) == _geometries(t1.timestep_ops(1).ops)
    assert _geometries(t8.plan._arr) == _geometries(t1.plan._arr)


def test_decoder_and_encoder_sessions_take_the_one_chart_plan(blob):
    on, off = _cpu_engine(blob, True), _cpu_engine(blob, False)
    for make in (DecoderSession, EncoderSession):
        g1 = _geometries(make(on, 1, 96).plan._arr)
        for B in (3, 32):
            assert _geometries(make(on, B, 96).plan._arr) == g1
        ops = make(off, 32, 96).plan._arr
        assert all(o.kind != L_.OP_GEMM_SERIAL and not (o.kind == L_.OP_GEMM and o.u.gemm.split_k) for o in ops)


def test_policy_leaves_ops_off_the_tensor_cores_alone(blob):
    """an op the runtime would run on the FFMA kernel (here: an A operand off its 16-byte alignment) keeps its kind and split"""
    ops = _unet(blob, 64, 512)
    i = next(k for k, o in enumerate(ops.ops) if o.kind == L_.OP_GEMM and o.u.gemm.K % 32 == 0 and gemm_runs_tc(o.u.gemm, SMS))
    ops.ops[i].u.gemm.A += 4
    assert not gemm_runs_tc(ops.ops[i].u.gemm, SMS)
    out = unit_batch_splits(ops, 64, 2, SMS)
    assert out.ops[i].kind == L_.OP_GEMM and out.ops[i].u.gemm.split_k == 0
    assert sum(o.kind == L_.OP_GEMM_SERIAL for o in out.ops) > 0

"""The GEMM tests' fp64 statement and cases, without a GPU: ref_gemm (gemm_cases.py) against independent float64 torch statements of
every addressing mode and epilogue operand -- were it wrong in the same way as a kernel, the GPU tests would pass both -- and the
serial-split cases against the planner and the batch-invariant plans: every class of serial op the plans contain has a GPU case,
every case runs the K split and K-range remainder it claims, and the GPU cases launch all 16 serial instantiations.  For the FFMA
kernel: the bound admits a float32 computation of every case and rejects wrong kernels on each case's own operands, every class of
FFMA op in the plans has a GPU case, every case takes the tile it claims at 132 and 114 SMs, and bad descriptors are refused."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import packer, synth
from mug_diffusion_b200.config import ModelConfig
from mug_diffusion_b200.engine import OpList
from mug_diffusion_b200.packer import tf32_split

from gemm_cases import (EPIS, EXTRA, FFMA_C, FFMA_SMS, LAYOUT_BASES, LAYOUTS, LN_EPS, MATRIX, SERIAL, SPLIT, STEP, Case, Operands,
                        case_gemm, epilogue_of, ffma_bound, ffma_class, ffma_gpu_cases, ffma_tile, layout_split, matrix_case,
                        plan_ffma_classes, plan_serial_classes, ref_finish, ref_gemm, rowvec_rows, serial_class, src_rows)

SMS = 132


def rnd(name, *shape):
    return synth._gauss(synth._rng(11, name), shape).double()


def close(a, b, tol=1e-12):
    assert a.shape == b.shape, (a.shape, b.shape)
    assert float((a - b).abs().max()) <= tol * float(b.abs().max()), float((a - b).abs().max())


def rows(x):
    """[B, C, L] -> [B*L, C]"""
    return x.permute(0, 2, 1).reshape(-1, x.shape[1])


# ---- ref_gemm against torch float64 --------------------------------------------------------------------------------------------
def test_linear():
    x, w, b, r = rnd("x", 37, 64), rnd("w", 48, 64), rnd("b", 48), rnd("r", 37, 48)
    close(ref_gemm(x, w, B=1, Lin=37, Lout=37, K=64, bias=b, residual=r), F.linear(x, w, b) + r)
    for act, f in ((L_.ACT_SILU, F.silu), (L_.ACT_GELU, F.gelu)):
        close(ref_gemm(x, w, B=1, Lin=37, Lout=37, K=64, bias=b, act=act, residual=r), f(F.linear(x, w, b)) + r)


def test_conv3_same():
    B, K, N, L = 3, 24, 40, 19
    x, w, b = rnd("x", B, K, L), rnd("w", N, K, 3), rnd("b", N)
    got = ref_gemm(rows(x), packer._conv3(w), B=B, Lin=L, Lout=L, K=K, taps=3, mode=L_.CONV_SAME, bias=b)
    close(got, rows(F.conv1d(x, w, b, padding=1)))


@pytest.mark.parametrize("L", [20, 21])
def test_downsample_stride2_right_pad(L):
    """the Downsample's conv: stride 2, one zero row on the right only"""
    B, K, N = 2, 16, 24
    x, w, b = rnd("x", B, K, L), rnd("w", N, K, 3), rnd("b", N)
    want = F.conv1d(F.pad(x, (0, 1)), w, b, stride=2)
    got = ref_gemm(rows(x), packer._conv3(w), B=B, Lin=L, Lout=want.shape[2], K=K, taps=3, mode=L_.CONV_DOWN, bias=b)
    close(got, rows(want))


def test_upsample_as_two_parity_gemms():
    """nearest x2 + conv3 == the even rows of a 2-tap GEMM (shift -1) on up_even + the odd rows of one (shift 0) on up_odd, with the
    packer's weights of an Upsample block of the U-Net"""
    cfg = ModelConfig()
    sd = synth.synthetic_state_dict(96)
    blob = packer.pack_model(sd, cfg.unet, cfg.decoder)
    name = next(n for n in blob.entries if n.endswith("conv.up_even.weight"))
    p = name[:-len("conv.up_even.weight")]
    w, b = sd[p + "conv.weight"].double(), sd[p + "conv.bias"].double()
    N, K, _ = w.shape
    B, L = 2, 9
    x = rnd("x", B, K, L)
    want = rows(F.conv1d(F.interpolate(x, scale_factor=2, mode="nearest"), w, b, padding=1)).reshape(B, L, 2, N)
    for parity, entry, shift in ((0, "conv.up_even.weight", -1), (1, "conv.up_odd.weight", 0)):
        wp = blob.view(p + entry).double()
        got = ref_gemm(rows(x), wp, B=B, Lin=L, Lout=L, K=K, taps=2, mode=L_.CONV_TAPS, tap_shift=shift, bias=b)
        close(got, want[:, :, parity].reshape(B * L, N), tol=1e-6)     # the composed taps are packed in fp32


@pytest.mark.parametrize("d", [1, 2, 4, 8])
def test_dilated_taps(d):
    """wave.py's dilated convs: conv1d(dilation=d, padding=d) as 3 taps at rows l + (t-1)*d"""
    B, K, N, L = 2, 16, 24, 29
    x, w, b = rnd("x", B, K, L), rnd("w", N, K, 3), rnd("b", N)
    got = ref_gemm(rows(x), packer._conv3(w), B=B, Lin=L, Lout=L, K=K, taps=3, mode=L_.CONV_TAPS, tap_shift=-1, dilation=d, bias=b)
    close(got, rows(F.conv1d(x, w, b, dilation=d, padding=d)))


def test_second_source():
    """conv3 on A plus a 1x1 term on A2: W = [conv3 taps | K2 columns]"""
    B, K, K2, N, L = 2, 16, 8, 24, 13
    x, x2, w, w2 = rnd("x", B, K, L), rnd("x2", B, K2, L), rnd("w", N, K, 3), rnd("w2", N, K2)
    W = torch.cat([packer._conv3(w), w2], dim=1)
    got = ref_gemm(rows(x), W, B=B, Lin=L, Lout=L, K=K, taps=3, mode=L_.CONV_SAME, A2=rows(x2))
    close(got, rows(F.conv1d(x, w, padding=1)) + rows(x2) @ w2.T)
    a, a2, wl = rnd("a", 30, K), rnd("a2", 30, K2), rnd("wl", N, K + K2)
    close(ref_gemm(a, wl, B=1, Lin=30, Lout=30, K=K, A2=a2), F.linear(torch.cat([a, a2], dim=1), wl))


@pytest.mark.parametrize("gate", [L_.GATE_GEGLU, L_.GATE_GLU])
def test_gates_on_interleaved_weights(gate):
    """GEGLU / GLU (proj -> chunk(2) -> value * gelu / sigmoid(gate)) on the packer's interleaved weight and bias rows"""
    x, w, b, r = rnd("x", 21, 32), rnd("w", 48, 32), rnd("b", 48), rnd("r", 21, 24)
    v, gt = F.linear(x, w, b).chunk(2, dim=-1)
    want = v * (F.gelu(gt) if gate == L_.GATE_GEGLU else torch.sigmoid(gt)) + r
    got = ref_gemm(x, packer._interleave_halves(w), B=1, Lin=21, Lout=21, K=32, bias=packer._interleave_halves(b), gate=gate,
                   residual=r)
    close(got, want)


@pytest.mark.parametrize("gate", [L_.GATE_NONE, L_.GATE_GEGLU])
def test_folded_layernorm(gate):
    """Linear(LayerNorm(x)) as the packer folds it: W' = W diag(gamma), colsum = W' 1, b' = W beta + b, the row moments of x; rows
    with |mean| of a few sigma included"""
    K, N = 64, 48
    x = rnd("x", 33, K) + 3.0 * rnd("m", 33, 1)
    gamma, beta, w, b = 1 + 0.1 * rnd("g", K), 0.1 * rnd("be", K), rnd("w", N, K), rnd("b", N)
    y = F.linear(F.layer_norm(x, (K,), gamma, beta, LN_EPS), w, b)
    if gate:
        v, gt = y.chunk(2, dim=-1)
        y = v * F.gelu(gt)
        perm = packer._interleave_halves
    else:
        perm = lambda t: t                                   # noqa: E731
    wg = w * gamma[None]
    stats = torch.stack([x.sum(1), (x * x).sum(1)], dim=1)
    got = ref_gemm(x, perm(wg), B=1, Lin=33, Lout=33, K=K, bias=perm(w @ beta + b), gate=gate, ln=(stats, perm(wg).sum(1), LN_EPS))
    assert float((got - y).abs().max()) <= 1e-10 * float(y.abs().max())


@pytest.mark.parametrize("kind", ["sample", "step", "both"])
def test_rowvec_strides(kind):
    """the time-embedding row: per sample (b_stride N), by step (step_stride N), or both ([STEPS, B, N], step_stride B*N)"""
    B, L, K, N, S, step = 3, 5, 16, 24, 4, 2
    x, w = rnd("x", B * L, K), rnd("w", N, K)
    y = F.linear(x, w).reshape(B, L, N)
    if kind == "sample":
        t, bs, ss, want = rnd("t", B, N), N, 0, y + rnd("t", B, N)[:, None]
    elif kind == "step":
        t, bs, ss, want = rnd("t", S, N), 0, N, y + rnd("t", S, N)[step][None, None]
    else:
        t, bs, ss, want = rnd("t", S, B, N), N, B * N, y + rnd("t", S, B, N)[step][:, None]
    got = ref_gemm(x, w, B=B, Lin=L, Lout=L, K=K, rowvec=t, rowvec_b_stride=bs, rowvec_step_stride=ss, step=step)
    close(got, want.reshape(B * L, N))


# ---- the serial-split cases against the planner and the plans --------------------------------------------------------------------
def _gemm(c: Case, split: int):
    """the descriptor test_gpu_gemm_epilogue.Device builds for ``c``, at fake 256-byte aligned addresses"""
    names = ("a", "w", "w_hi", "w_lo", "out", "a2", "res", "bias", "table", "step", "stats", "colsum", "moments")
    ops = OpList()
    i = case_gemm(ops, c, split, **{n: (1 << 40) + (k << 32) for k, n in enumerate(names)})
    return ops.ops[i].u.gemm


class _tile:
    def __init__(self, c: Case, bn: int):
        self.bn = bn if (bn == 64 and c.N >= 128) else 0       # test_gpu_gemm_epilogue.check_case's forcing

    def __enter__(self):
        L_.check(L_.load().mugd_debug_set_tc_tile_n(self.bn), "tile_n")

    def __exit__(self, *exc):
        L_.check(L_.load().mugd_debug_set_tc_tile_n(0), "tile_n")


def serial_gpu_cases():
    """every serial-split GPU case of test_gpu_gemm_epilogue.py: name -> (case, split, tile width, claimed short last K-range)"""
    out = {}
    for e, cv, s in MATRIX:
        for bn in (128, 64):
            out[f"test_epilogue_matrix[{e}-{cv}-{s}-serial-{bn}]"] = (matrix_case(e, cv, s), SPLIT, bn, True)
    for name, (c, split, bn) in EXTRA.items():
        out[f"test_addressing_modes[{name}-serial]"] = (c, split, bn, True)
    for name, (c, split, bn, uneven) in SERIAL.items():
        out[f"test_serial_plan_classes[{name}]"] = (c, split, bn, uneven)
    for base, c in LAYOUT_BASES.items():
        for bn in (128, 64):
            for lay, (_, uneven) in LAYOUTS.items():
                out[f"test_serial_k_range_layouts[{base}-{bn}-{lay}]"] = (c, layout_split(base, lay), bn, uneven)
    return out


def _planned(c, split, bn):
    """(split, tile width, short last K-range) the planner gives the case's descriptor, and its serial class"""
    gm = _gemm(c, split)
    with _tile(c, bn):
        sp, b = C.c_int32(), C.c_int32()
        L_.check(L_.load().mugd_gemm_tc_query(None, C.byref(gm), SMS, None, C.byref(sp), None, None), "tc_query")
        L_.check(L_.load().mugd_gemm_tc_variant(C.byref(gm), SMS, C.byref(b), None, None), "tc_variant")
        cls = serial_class(gm, SMS)
    return (sp.value, b.value, c.ksteps % sp.value != 0), cls


def test_every_case_runs_the_k_range_layout_it_claims():
    for name, (c, split, bn, uneven) in serial_gpu_cases().items():
        got, _ = _planned(c, split, bn)
        assert got == (split, bn, uneven), name


def test_every_serial_instantiation_is_launched():
    """8 epilogues x BN in {64, 128}: all 16 serial kernels"""
    seen = {(cls[0], cls[1]) for c, split, bn, _ in serial_gpu_cases().values() for cls in [_planned(c, split, bn)[1]]}
    assert seen == {(e, bn) for e in EPIS for bn in (64, 128)}, sorted(seen)


def test_every_plan_serial_class_has_a_gpu_case():
    """every class of serial op in the batch-invariant plans at 132 SMs (U-Net plain / per-sample-t, decoder, encoder; L in
    {96, 512, 992, 2048}, B in {2, 3, 4, 8, 32}, CFG on / off) is the class of a serial GPU case: a plan change that makes a new
    class fails here"""
    covered = {}
    for name, (c, split, bn, _) in serial_gpu_cases().items():
        covered.setdefault(_planned(c, split, bn)[1], name)
    plans = plan_serial_classes()
    print(f"{len(plans)} classes of serial op in the plans (epilogue, BN, conv mode, K2, rowvec, residual, Lrows < 128, short last range):")
    for cls, where in sorted(plans.items(), key=str):
        print(f"  {cls}  first in {where}  <- {covered.get(cls, 'NOT COVERED')}")
    missing = [cls for cls in plans if cls not in covered]
    assert not missing, missing
    assert len(plans) >= 27


def test_epilogue_of_matches_the_op_fields():
    for e, kw in EPIS.items():
        c = Case(2, 100, 100, 128, 192, rowvec="", residual=False, **kw)
        assert epilogue_of(_gemm(c, 2)) == e


# ---- the FFMA kernel: the generic Upsample, the error bound, the plan classes and the host refusals ---------------------------
def test_generic_upsample_conv_up():
    """CONV_UP: nearest x2 then conv3, output row l tap t reads source (l+t-1) >> 1 where 0 <= l+t-1 < Lout"""
    for L in (1, 2, 9):
        B, K, N = 2, 16, 24
        x, w, b = rnd("x", B, K, L), rnd("w", N, K, 3), rnd("b", N)
        want = F.conv1d(x.repeat_interleave(2, dim=-1), w, b, padding=1)
        got = ref_gemm(rows(x), packer._conv3(w), B=B, Lin=L, Lout=2 * L, K=K, taps=3, mode=L_.CONV_UP, bias=b)
        close(got, rows(want))


def ffma32(o: Operands):
    """the case in float32 on the CPU, one rounding per tap sum, bias, time-embedding row and epilogue step"""
    c = o.c
    kw = o.kwargs()
    a = o.A.float().reshape(c.B, c.Lin, c.K)
    lo = torch.arange(c.Lout)
    y = torch.zeros(c.B, c.Lout, c.N)
    for t in range(c.taps):
        src = src_rows(c.mode, t, lo, c.Lin, c.Lout, c.shift, c.dilation)
        xs = torch.zeros(c.B, c.Lout, c.K)
        xs[:, src >= 0] = a[:, src[src >= 0]]
        y += xs @ o.W[:, t * c.K:(t + 1) * c.K].T
    if c.K2:
        y += o.A2.reshape(c.B, c.Lout, -1) @ o.W[:, c.taps * c.K:].T
    y = y.reshape(c.M, c.N)
    if o.bias is not None:
        y = y + o.bias
    if o.table is not None:
        y = y + rowvec_rows(o.table, c.B, c.Lout, c.N, *c.rowvec_strides, STEP).float()
    y = {L_.ACT_SILU: F.silu, L_.ACT_GELU: F.gelu}.get(c.act, lambda v: v)(y)
    if c.gate:
        y = y[:, 0::2] * (F.gelu(y[:, 1::2]) if c.gate == L_.GATE_GEGLU else torch.sigmoid(y[:, 1::2]))
    if kw["residual"] is not None:
        y = y + kw["residual"]
    return y


@pytest.fixture(scope="module")
def ffma_operands():
    return {name: (c, Operands(c, name)) for name, (c, _) in ffma_gpu_cases().items()}


@pytest.fixture(scope="module")
def ffma_refs(ffma_operands):
    return {name: (o.ref(), ffma_bound(o)) for name, (c, o) in ffma_operands.items()}


def test_ffma_bound_passes_a_float32_computation_of_every_case(ffma_operands, ffma_refs):
    worst = 0.0
    for name, (c, o) in ffma_operands.items():
        ref, E = ffma_refs[name]
        r = float(((ffma32(o).double() - ref).abs() / E).max())
        worst = max(worst, r)
        assert r <= FFMA_C, (name, r)
        if r == worst:
            at = name
    print(f"at {at}: worst |y32 - y64| / E over {len(ffma_operands)} cases: {worst:.3f} (c = {FFMA_C})")


def _clamped(mode, t, lo, Lin, Lout, *_):                       # the SAME halo clamped to the sample's edge rows
    return (lo + t - 1).clamp(0, Lin - 1)


def _left_padded(mode, t, lo, Lin, Lout, *_):                   # DOWN padded on the left instead of the right
    src = 2 * lo + t - 1
    return torch.where((src >= 0) & (src < Lin), src, torch.full_like(src, -1))


def mutations(o: Operands) -> dict:
    """fp64 results of wrong kernels on the case's own operands: name -> output"""
    c, out = o.c, {}
    for t in range(c.taps):                                     # the last k-step of a tap, and of the second source, dropped
        W = o.W.clone()
        W[:, (t + 1) * c.K - 16:(t + 1) * c.K] = 0
        out[f"drop_last_kstep_of_tap{t}"] = o.ref(W=W)
    if c.K2:
        W = o.W.clone()
        W[:, -16:] = 0
        out["drop_last_k2_kstep"] = o.ref(W=W)
    if c.mode == L_.CONV_SAME:
        out["same_halo_clamped"] = o.ref(rows=_clamped)
    if c.mode == L_.CONV_DOWN:
        out["down_left_padded"] = o.ref(rows=_left_padded)
    if c.mode == L_.CONV_TAPS:
        out["tap_shift_off_by_one"] = o.ref(tap_shift=c.shift + 1)
    if c.dilation > 1:
        out["dilation_1"] = o.ref(dilation=1)
    if c.rowvec in ("both", "batch") and c.B > 1:
        out["rowvec_of_sample_0"] = o.ref(rowvec_b_stride=0)
    if c.gate:
        z = o.ref(pre=True)
        z = torch.stack([z[:, 1::2], z[:, 0::2]], dim=2).reshape(z.shape)
        out["gate_halves_swapped"] = ref_finish(z, c.act, c.gate, o.residual)
    if c.residual:
        out["residual_one_column_off"] = o.ref(residual=o.res[:, 17:17 + c.nout])
    out["a_rounded_to_tf32"] = o.ref(A=tf32_split(o.A)[0])
    return out


def test_ffma_bound_rejects_wrong_kernels(ffma_operands, ffma_refs):
    """every mutation that changes a case's fp64 result at all (a dropped k-step of a tap that only reads the zero padding, as at
    L = 1, does not) exceeds the bound somewhere"""
    kinds = set()
    for name, (c, o) in ffma_operands.items():
        ref, E = ffma_refs[name]
        for what, y in mutations(o).items():
            if torch.equal(y, ref):
                continue
            kinds.add(what.split("_of_tap")[0])
            assert bool(((y - ref).abs() > FFMA_C * E).any()), (name, what)
    assert {"drop_last_kstep", "drop_last_k2_kstep", "same_halo_clamped", "down_left_padded", "tap_shift_off_by_one",
            "dilation_1", "rowvec_of_sample_0", "gate_halves_swapped", "residual_one_column_off", "a_rounded_to_tf32"} <= kinds


def _ffma_gemm(c: Case):
    """the FFMA descriptor test_gpu_gemm_epilogue.Device builds for ``c``, at fake 256-byte aligned addresses"""
    names = ("a", "w", "out", "a2", "res", "bias", "table", "step")
    ops = OpList()
    i = case_gemm(ops, c, 0, w_hi=0, w_lo=0, impl=L_.GEMM_SIMT, **{n: (1 << 40) + (k << 32) for k, n in enumerate(names)})
    return ops.ops[i].u.gemm


@pytest.mark.parametrize("sms", FFMA_SMS)
def test_every_ffma_case_takes_the_tile_it_claims(sms):
    for name, (c, tile) in ffma_gpu_cases().items():
        assert ffma_tile(c.M, c.N, sms) == tile, name
        assert ffma_class(_ffma_gemm(c), sms)[-1] == tile, name
    tiles = {t for _, t in ffma_gpu_cases().values()}
    assert tiles == {64, 128}


def test_every_plan_ffma_class_has_a_gpu_case():
    """every class of GEMM the plans run on the FFMA kernel (plan_ffma_classes: default and empty TF32 map) is the class of an FFMA
    GPU case: a plan change that makes a new class fails here, naming it"""
    covered = {}
    for name, (c, _) in ffma_gpu_cases().items():
        covered.setdefault(ffma_class(_ffma_gemm(c), SMS), name)
    plans = plan_ffma_classes()
    print(f"{len(plans)} classes of FFMA op in the plans (mode, taps, dilated, shift, K2, act, gate, bias, rowvec, residual, strided, "
          "K % 32, N < 64, tile):")
    for cls, where in sorted(plans.items(), key=str):
        print(f"  {cls}  first in {where}  <- {covered.get(cls, 'NOT COVERED')}")
    missing = [(cls, where) for cls, where in plans.items() if cls not in covered]
    assert not missing, missing
    assert len(plans) >= 45
    # the default engine's own FFMA GEMMs: the K = 16 convs (U-Net input conv into its concat window, decoder and encoder inputs)
    assert {cls[11] for cls, where in plans.items() if where.startswith("auto")} == {True}


def _simt_gemm(**kw):
    """a valid FFMA descriptor at fake, aligned device addresses"""
    g = L_.Gemm()
    g.A, g.lda, g.W = 1 << 40, 64, 1 << 41
    g.C, g.ldc = 1 << 43, 64
    g.M, g.N, g.K, g.taps, g.conv_mode, g.Lin, g.Lout = 128, 64, 48, 3, L_.CONV_SAME, 64, 64
    g.impl = L_.GEMM_SIMT
    for k, v in kw.items():
        setattr(g, k, v)
    return g


@pytest.mark.parametrize("kw,msg", [
    (dict(W_hi=1 << 41), "split into TF32 hi/lo in place"),
    (dict(row_moments=1 << 44), "tensor-core path only"),
    (dict(ln_stats=1 << 44, ln_colsum=1 << 45), "tensor-core path only"),
    (dict(K=24, lda=24), "multiple of 16"),
    (dict(N=66), "multiple of 4"),
    (dict(conv_mode=L_.CONV_DOWN, Lin=64, Lout=32, M=64, A2=1 << 44, lda2=16, K2=16), "second source"),
    (dict(conv_mode=L_.CONV_UP, Lin=32, Lout=64, A2=1 << 44, lda2=16, K2=16), "second source"),
    (dict(A=(1 << 40) + 4), "A/W alignment"),
    (dict(C=(1 << 43) + 4), "C alignment"),
    (dict(residual=(1 << 44) + 4, ldr=64), "residual alignment"),
    (dict(residual=(1 << 44) + 4, ldr=64, gate=L_.GATE_GLU, ldc=32), "residual alignment"),
], ids=["w_split_in_place", "row_moments", "folded_ln", "k24", "n66", "k2_down", "k2_up", "a_misaligned", "c_misaligned",
        "residual_misaligned", "gated_residual_misaligned"])
def test_ffma_refuses_bad_descriptors_before_any_device_call(kw, msg):
    """mugd_op_run on a zeroed handle (no device behind it): every refusal comes from the host checks"""
    lib = L_.load()
    handle = (C.c_char * 4096)()
    op = L_.make_op(L_.OP_GEMM, _simt_gemm(**kw))
    assert lib.mugd_op_run(C.cast(handle, C.c_void_p), C.byref(op), None) == 1
    assert msg in lib.mugd_last_error().decode()

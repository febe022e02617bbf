"""Fused epilogues of the wgmma GEMM (gemm_tc.cuh) on its three ways to finish an output tile -- the direct tile store
(tc_store_tile, split_k = 1), the split-K second pass (tc_reduce), which finishes most output tiles of a small-batch U-Net
evaluation, and the serial split (gemm_tc_serial_kernel, MUGD_OP_GEMM_SERIAL: one CTA runs every K-range of its tile and stores it
through tc_store_tile), which the batch-invariant plans take for large batches -- against ONE fp64 statement of mugd_gemm
(gemm_cases.ref_gemm), with every operand each epilogue takes: bias, the time-embedding row (per sample and chosen by the device
step counter), A / residual / output column windows, the second source, the row-moment sink and the folded LayerNorm.  The serial
split is also bit-equal to split kernel + reduce at the same split (the batch-invariance guarantee rests on it) at every epilogue,
tile width, addressing mode, class of serial op the invariant plans contain and K-range layout.  Also the step counter under
CUDA-graph replay and the opt-in single-pass TF32 mode.

The exact-fp32 FFMA kernel (gemm_simt.cu) is one more path of the same matrix, addressing modes and graph replay, held element by
element to the bound gemm_cases.ffma_bound (|y - y64| <= FFMA_C E) at its factor cases and one case of every class of FFMA op the
plans contain; the row-moment sink and the folded LayerNorm are refused on it.  A sample's rows from a launch on 128 x 128 tiles
are bit-equal to the same sample launched alone on 64 x 64 tiles: what lets a `simt` engine keep its plans under batch_invariant.

Tolerances of the tensor-core paths are those of test_gpu_gemm_tc.py / test_gpu_fusion.py: 1e-5 of max |ref| (2e-5 with the folded
LayerNorm)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200.engine import OpList  # noqa: E402
from mug_diffusion_b200.packer import tf32_split  # noqa: E402

from gemm_cases import (EXTRA, FFMA, FFMA_C, LAYOUT_BASES, LAYOUTS, MATRIX, SENT, SERIAL, SPLIT, STEP, STEPS, TOL,  # noqa: E402
                        TOL_LN, Case, Operands, case_gemm, ffma_bound, ffma_gpu_cases, ffma_tile, layout_split, matrix_case,
                        ref_gemm)
from gpu_util import OpRunner, ptr, rel_err  # noqa: E402


class Device:
    """the operands of a case on the GPU, an output buffer pre-filled with SENT and the op list of the GEMM (serial: the
    MUGD_OP_GEMM_SERIAL op at the same forced split; ffma: forced to the FFMA kernel, plain fp32 weight only)"""

    def __init__(self, o: Operands, split: int, serial: bool = False, ffma: bool = False, a_off: int = 32):
        c = o.c
        self.c = c
        a = torch.zeros(c.B * c.Lin, c.K + 64)                       # A is columns a_off .. a_off+K of a wider buffer
        a[:, a_off:a_off + c.K] = o.A
        self.a = a.cuda()
        kw = {}
        if c.K2:
            a2 = torch.zeros(c.M, c.K2 + 64)
            a2[:, 32:32 + c.K2] = o.A2
            self.a2 = a2.cuda()
            kw["a2"] = ptr(self.a2)
        self.w = o.W.cuda()
        if not ffma:
            hi, lo = tf32_split(o.W)
            self.w_hi, self.w_lo = hi.cuda(), lo.cuda()
        self.step = torch.tensor([STEP], dtype=torch.int32).cuda()
        if c.bias:
            self.bias = o.bias.cuda()
            kw["bias"] = ptr(self.bias)
        if c.rowvec:
            self.table = o.table.cuda()
            kw.update(table=ptr(self.table), step=ptr(self.step))
        if c.residual:
            self.res = o.res.cuda()
            kw["res"] = ptr(self.res)
        if c.parity >= 0:
            self.out = torch.full((2 * c.M, c.nout), SENT).cuda()
        elif c.dense:
            self.out = torch.full((c.M + 2, c.nout), SENT).cuda()     # the output is rows 1 .. M+1
        else:
            self.out = torch.full((c.M, c.nout + 64), SENT).cuda()   # the output is columns 32 .. 32+nout
        if c.ln:
            self.stats, self.colsum = o.ln[0].cuda(), o.ln[1].cuda()
            kw.update(stats=self.stats.data_ptr(), colsum=ptr(self.colsum))
        self.moments = None
        if c.sink:
            self.moments = torch.zeros(c.M, 2, dtype=torch.float64).cuda()
            kw["moments"] = self.moments.data_ptr()
        self.ops = OpList()
        out = ptr(self.out) + (4 * c.nout if c.dense else 0)
        if ffma:
            kw.update(w_hi=0, w_lo=0, impl=L_.GEMM_SIMT)
        else:
            kw.update(w_hi=ptr(self.w_hi), w_lo=ptr(self.w_lo))
        self.i = case_gemm(self.ops, c, split, a=ptr(self.a), w=ptr(self.w), out=out, a_off=a_off, **kw)
        if serial:
            self.ops.ops[self.i].kind = L_.OP_GEMM_SERIAL

    @property
    def gemm(self):
        return self.ops.ops[self.i].u.gemm

    def output(self):
        """the output window (host), and whether every element outside it still holds SENT"""
        c, o = self.c, self.out.cpu()
        if c.parity >= 0:
            win, rest = o[c.parity::2], o[1 - c.parity::2]
        elif c.dense:
            win, rest = o[1:-1], torch.cat([o[:1], o[-1:]])
        else:
            win, rest = o[:, 32:32 + c.nout], torch.cat([o[:, :32], o[:, 32 + c.nout:]], dim=1)
        return win.clone(), bool((rest == SENT).all())


def sm_count(R):
    n = C.c_int32()
    L_.check(R.lib.mugd_device_info(R.handle, C.byref(n), None, None), "device_info")
    return n.value


def planned(R, gm):
    """(K splits, tile width) the planner picks for this GEMM on this device"""
    sp, bn = C.c_int32(), C.c_int32()
    L_.check(R.lib.mugd_gemm_tc_query(None, C.byref(gm), sm_count(R), None, C.byref(sp), None, None), "tc_query")
    L_.check(R.lib.mugd_gemm_tc_variant(C.byref(gm), sm_count(R), C.byref(bn), None, None), "tc_variant")
    return sp.value, bn.value


class tile_width:
    """mugd_debug_set_tc_tile_n for a block (process-wide: always reset to the cost model)"""

    def __init__(self, R, bn):
        self.R, self.bn = R, bn

    def __enter__(self):
        L_.check(self.R.lib.mugd_debug_set_tc_tile_n(self.bn), "tile_n")

    def __exit__(self, *exc):
        L_.check(self.R.lib.mugd_debug_set_tc_tile_n(0), "tile_n")


@pytest.fixture(scope="module")
def R():
    return OpRunner()


def check_case(R, c: Case, name: str, split: int, bn: int, tol: float, serial: bool = False):
    """the GEMM of ``c`` at ``split`` (serial: the serial-split op) against fp64, the output window's surroundings untouched, two
    runs equal; the reduce path within ``tol`` of the direct path, the serial split bit-equal to split kernel + reduce at ``split``
    (split 1: the direct path), row moments included"""
    o = Operands(c, name)
    ref = o.ref()
    force = bn if (bn == 64 and c.N >= 128) else 0
    with tile_width(R, force):
        d = Device(o, split, serial)
        assert planned(R, d.gemm) == (split, bn)                   # the path under test is the one that runs
        R.run(d.ops)
        out, kept = d.output()
        d2 = Device(o, split, serial)
        R.run(d2.ops)
        out2, _ = d2.output()
        if serial:
            dr = Device(o, split)
            R.run(dr.ops)
            twin, _ = dr.output()
        elif split > 1:
            dd = Device(o, 1)
            assert planned(R, dd.gemm) == (1, bn)
            R.run(dd.ops)
            direct, _ = dd.output()
    e = rel_err(out, ref)
    print(f"{name} split={split} bn={bn} serial={serial} rel_err={e:.2e}")
    assert e < tol
    assert kept, "a store left the output window"
    assert torch.equal(out, out2), "two runs differ"
    if serial:
        assert torch.equal(out, twin), "the serial split differs from split kernel + reduce"
        if c.sink:
            assert torch.equal(d.moments, dr.moments), "row moments of the serial split differ from the reduce's"
            assert torch.equal(d.moments, d2.moments)
    elif split > 1:
        assert float((out - direct).abs().max()) < tol * float(ref.abs().max())
    if c.sink:
        s = out.double()
        exp = torch.stack([s.sum(1), (s * s).sum(1)], dim=1)
        assert float((d.moments.cpu() - exp).abs().max() / exp.abs().max()) < 1e-6


def check_ffma(R, c: Case, name: str, tile: int, o: Operands = None):
    """the GEMM of ``c`` forced to the FFMA kernel on ``tile`` x ``tile`` tiles against fp64, element by element within FFMA_C times
    ffma_bound; the output window's surroundings untouched, two runs equal.  The row-moment sink and the folded LayerNorm are
    refused.  Returns |y - y64| / E at its worst and the output."""
    o = o or Operands(c, name)
    if c.sink or c.ln:
        with pytest.raises(L_.MugdError, match="tensor-core path only"):
            R.run(Device(o, 0, ffma=True).ops)
        return 0.0, None
    assert ffma_tile(c.M, c.N, sm_count(R)) == tile                 # the variant under test is the one that runs
    d = Device(o, 0, ffma=True)
    R.run(d.ops)
    out, kept = d.output()
    d2 = Device(o, 0, ffma=True)
    R.run(d2.ops)
    ratio = float(((out.double() - o.ref()).abs() / ffma_bound(o)).max())
    print(f"{name} ffma tile={tile} |y - y64| / E = {ratio:.3f}")
    assert ratio <= FFMA_C, ratio
    assert kept, "a store left the output window"
    assert torch.equal(out, d2.output()[0]), "two runs differ"
    return ratio, out


PATHS = ["direct", "reduce", "serial"]
MATRIX_PATHS = [(p, bn) for p in PATHS for bn in (128, 64)] + [("ffma", 64)]      # FFMA: these shapes take its 64-tile variant


@pytest.mark.parametrize("path,bn", MATRIX_PATHS, ids=[f"{p}-{bn}" for p, bn in MATRIX_PATHS])
@pytest.mark.parametrize("epi,conv,shape", MATRIX, ids=["-".join(m) for m in MATRIX])
def test_epilogue_matrix(R, epi, conv, shape, path, bn):
    """every epilogue at both tile widths on every path: with the serial path, all 16 serial instantiations (8 epilogues x BN); on
    the FFMA kernel the sink and the folded LayerNorm are refused"""
    c = matrix_case(epi, conv, shape)
    assert c.ksteps % SPLIT != 0                                   # the last split owns fewer k-steps (it_rem != 0)
    if path == "ffma":
        check_ffma(R, c, f"{epi}-{conv}-{shape}", bn)
        return
    check_case(R, c, f"{epi}-{conv}-{shape}", 1 if path == "direct" else SPLIT, bn, TOL_LN if c.ln else TOL, serial=path == "serial")


@pytest.mark.parametrize("path", PATHS + ["ffma"])
@pytest.mark.parametrize("name", list(EXTRA))
def test_addressing_modes(R, name, path):
    c, split, bn = EXTRA[name]
    assert c.ksteps % split != 0
    if path == "ffma":
        check_ffma(R, c, name, ffma_tile(c.M, c.N, sm_count(R)))
        return
    check_case(R, c, name, 1 if path == "direct" else split, bn, TOL, serial=path == "serial")


# ---- the FFMA kernel ------------------------------------------------------------------------------------------------------------
def test_ffma_cases_within_the_bound(R):
    """the FFMA factor cases and one case of every class of FFMA op the plans contain (test_gemm_cases.py checks both lists):
    within the bound, sentinels intact, two runs bit-equal; the worst ratio per tile variant is what DESIGN §2 records"""
    worst = {}
    for name, (c, tile) in ffma_gpu_cases().items():
        r, _ = check_ffma(R, c, name, tile)
        worst[tile] = max(worst.get(tile, (0.0, "")), (r, name))
    print("worst |y - y64| / E per tile variant:", worst)
    assert set(worst) == {64, 128}


ROW_INVARIANCE = ["big_none", "big_same", "big_down", "big_up", "big_taps_d2", "big_k2", "big_glu", "big_l1"]


@pytest.mark.parametrize("name", ROW_INVARIANCE)
def test_ffma_rows_do_not_depend_on_the_batch(R, name):
    """each sample's rows of a B-sample launch on 128 x 128 tiles are bit-equal to the same sample launched alone on 64 x 64 tiles
    with A at another column offset: the FFMA kernel sums every element in the same order whatever its tile and batch, the claim
    MugEngine.batch_ops relies on when it leaves a `simt` engine's plans alone under batch_invariant"""
    c, tile = FFMA[name]
    assert tile == 128
    o = Operands(c, name)
    _, out = check_ffma(R, c, name, tile, o)
    for b in sorted({0, 1, c.B // 2, c.B - 1}):
        one = o.sample(b)
        assert ffma_tile(one.c.M, one.c.N, sm_count(R)) == 64
        d = Device(one, 0, ffma=True, a_off=4)
        R.run(d.ops)
        alone, kept = d.output()
        assert kept
        assert torch.equal(alone, out[b * c.Lout:(b + 1) * c.Lout]), (name, b)


@pytest.mark.parametrize("name", list(SERIAL))
def test_serial_plan_classes(R, name):
    """one serial op of every class the batch-invariant plans contain (test_gemm_cases.py checks that every class of the plans is
    here), at its even or uneven K-range layout"""
    c, split, bn, uneven = SERIAL[name]
    assert (c.ksteps % split != 0) == uneven
    check_case(R, c, name, split, bn, TOL_LN if c.ln else TOL, serial=True)


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("bn", [128, 64])
@pytest.mark.parametrize("base", list(LAYOUT_BASES))
def test_serial_k_range_layouts(R, base, bn, layout):
    """one K-range (= the direct path), an even split, a short last range, k-steps - 1 ranges and one k-step per range: each bit-equal
    to split kernel + reduce at the same split and within the fp64 tolerance"""
    c = LAYOUT_BASES[base]
    split = layout_split(base, layout)
    assert (c.ksteps % split != 0) == LAYOUTS[layout][1]
    check_case(R, c, f"{base}-{layout}", split, bn, TOL, serial=True)


# ---- one captured graph serves every DDIM step --------------------------------------------------------------------------------
def make_plan(R, ops: OpList):
    for op in ops.ops:
        if op.kind == L_.OP_GEMM:
            gm = op.u.gemm
            gm.workspace, gm.workspace_bytes = R.ws.data_ptr(), R.ws.numel() * 4
            gm.counters, gm.n_counters = R.counters.data_ptr(), R.counters.numel()
    arr = ops.array()
    plan = C.c_void_p()
    L_.check(R.lib.mugd_plan_create(R.handle, arr, len(ops.ops), C.byref(plan)), "plan_create")
    return plan


@pytest.mark.parametrize("path", PATHS + ["ffma"])
def test_step_counter_under_graph_replay(R, path):
    """[ResBlock conv3 + time-embedding row of the current step ; STEP_ADVANCE] captured once, replayed once per step: replay i
    adds table row i (mugd.h: step-dependent rows are selected on the device, so one graph serves all steps).  The reduce reads the
    counter in its second pass, the direct path and the serial split in the tile's epilogue-operand preload, the FFMA kernel in its
    epilogue."""
    split = 1 if path == "direct" else 4
    c = Case(2, 200, 200, 64, 192, taps=3, mode=L_.CONV_SAME, rowvec="step", residual=False)
    assert c.ksteps % 4 != 0
    o = Operands(c, "graph")
    ffma = path == "ffma"
    d = Device(o, 0 if ffma else split, serial=path == "serial", ffma=ffma)
    d.step.zero_()
    if not ffma:
        assert planned(R, d.gemm)[0] == split
    adv = L_.StepAdvance()
    adv.step = ptr(d.step)
    d.ops.add(L_.OP_STEP_ADVANCE, adv)
    plan = make_plan(R, d.ops)
    st = torch.cuda.Stream()
    try:
        torch.cuda.synchronize()
        L_.check(R.lib.mugd_plan_capture(plan, C.c_void_p(st.cuda_stream)), "capture")
        assert int(d.step.item()) == 0                             # capturing runs nothing
        for i in range(STEPS):
            d.out.fill_(SENT)
            torch.cuda.synchronize()
            L_.check(R.lib.mugd_plan_replay(plan, 1, C.c_void_p(st.cuda_stream)), "replay")
            st.synchronize()
            out, kept = d.output()
            if ffma:
                assert bool(((out.double() - o.ref(step=i)).abs() <= FFMA_C * ffma_bound(o, step=i)).all()), i
            else:
                assert rel_err(out, o.ref(step=i)) < TOL, i
            assert kept
        assert int(d.step.item()) == STEPS
    finally:
        R.lib.mugd_plan_destroy(plan)


# ---- opt-in single-pass TF32 ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def R1():
    """a second handle: the single-pass switch is per handle"""
    r = OpRunner()
    yield r
    r.lib.mugd_set_tc_single_pass_tf32(r.handle, 0)
    r.lib.mugd_destroy(r.handle)


@pytest.mark.parametrize("path", PATHS)
def test_single_pass_tf32(R, R1, path):
    """plain TF32 products: each element within 2^-9 (|A| |W|^T) of fp64 (two round-to-nearest TF32 operands: <= 2^-10 per product,
    the rest is headroom for fp32 accumulation) and clearly worse than 3xTF32, so the mode is in effect.  The mode is read at every
    launch: a graph captured with it keeps it, eager runs take the current one.  The serial split in single-pass mode is bit-equal to
    split kernel + reduce in single-pass mode."""
    split, serial = (1 if path == "direct" else SPLIT), path == "serial"
    c = Case(2, 200, 200, 64, 192, taps=3, mode=L_.CONV_SAME, K2=32, bias=False, rowvec="", residual=False)
    o = Operands(c, "tf32")
    ref = o.ref()
    bound = 2.0 ** -9 * ref_gemm(o.A.abs(), o.W.abs(), B=c.B, Lin=c.Lin, Lout=c.Lout, K=c.K, taps=3, mode=L_.CONV_SAME, A2=o.A2.abs())
    d0 = Device(o, split, serial)                                  # on a handle that never switched
    assert planned(R, d0.gemm)[0] == split
    R.run(d0.ops)
    exact, _ = d0.output()
    lib, h = R1.lib, R1.handle
    plan = None
    try:
        L_.check(lib.mugd_set_tc_single_pass_tf32(h, 1), "single_pass")
        d = Device(o, split, serial)
        R1.run(d.ops)
        sp, kept = d.output()
        assert kept
        err = (sp.double() - ref).abs()
        assert bool((err <= bound).all()), float((err / bound).max())
        e = rel_err(sp, ref)
        print(f"single-pass TF32 {path} rel_err={e:.2e} (3xTF32: {rel_err(exact, ref):.2e})")
        assert e > TOL
        if serial:
            dr = Device(o, split)
            R1.run(dr.ops)
            assert torch.equal(dr.output()[0], sp), "single-pass serial split differs from split kernel + reduce"
        # a graph captured in single-pass mode keeps it after the switch goes off
        dg = Device(o, split, serial)
        plan = make_plan(R1, dg.ops)
        st = torch.cuda.Stream()
        torch.cuda.synchronize()
        L_.check(lib.mugd_plan_capture(plan, C.c_void_p(st.cuda_stream)), "capture")
        L_.check(lib.mugd_set_tc_single_pass_tf32(h, 0), "single_pass")
        L_.check(lib.mugd_plan_replay(plan, 1, C.c_void_p(st.cuda_stream)), "replay")
        st.synchronize()
        assert torch.equal(dg.output()[0], sp)
        # eager runs take the mode current at run time: the same plan run eagerly, and a single op, are 3xTF32 again
        dg.out.fill_(SENT)
        torch.cuda.synchronize()
        L_.check(lib.mugd_plan_run(plan, C.c_void_p(st.cuda_stream)), "plan_run")
        st.synchronize()
        assert torch.equal(dg.output()[0], exact)
        d1 = Device(o, split, serial)
        R1.run(d1.ops)
        assert torch.equal(d1.output()[0], exact)
    finally:
        lib.mugd_set_tc_single_pass_tf32(h, 0)
        if plan is not None:
            lib.mugd_plan_destroy(plan)

"""The S4 layer's kernels (csrc/s4.cu) against float64 on the GPU; the references, bounds and case lists are in s4_cases.py.

* ``mugd_s4_kernel_gen`` tap by tap against ``kgen64`` with both node paths (the reference's table and exact nodes), at every
  (H, L_internal, L_out) the runtime generates for the plans' z_lengths, at odd L_internal and up to 8192: per tap
  |Kt - K64| <= c (2^-24 |K64| + eps64 max|K64|); taps past L_out are not written.
* s4conv against a float64 FFT convolution with a bound per output, at every (Beff, L, H) the U-Net plans launch and at the edges,
  through the automatic dispatch and, wherever the resident kernel fits, both forced kernels; the edges on column windows of wider
  buffers whose other rows and columns must stay untouched.  Each case prints its branch of the launch rule for this device.
* Causality: NaN / +-1e30 at and past a cut change no bit of the outputs before it.  One S4 block as a ragged plan emits it
  (ragged GroupNorm -> s4conv -> GLU GEMM -> row mask -> k = 3 conv) against the block run alone at each valid length.
* The same block captured with programmatic launch edges and replayed over NaN-filled intermediates: the bits of the eager run.
* y overlapping u is refused by both kernels.
"""
import ctypes as C
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

import s4_cases as sc  # noqa: E402
from gpu_util import OpRunner, ptr, rel_err  # noqa: E402
from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200.engine import OpList, View  # noqa: E402
from mug_diffusion_b200.packer import tf32_split  # noqa: E402
from mug_diffusion_b200.runtime import s4_fft_nodes  # noqa: E402

NAN = float("nan")
SENT = -7777.0
# kernel generation's bound constant c: 4x the worst ratio measured on an H100 80GB HBM3 (700 W), 0.999 (DESIGN §2)
KGEN_BOUND = 4.0
IMPL_NAME = {sc.AUTO: "auto", sc.RESIDENT: "resident", sc.STREAMED: "streamed"}


@pytest.fixture(scope="module")
def R():
    return OpRunner()


@pytest.fixture(scope="module")
def dev(R):
    """(sm_count, max opt-in shared memory per block) of this device: the inputs of the launch rule"""
    sm = C.c_int32()
    L_.check(R.lib.mugd_device_info(R.handle, C.byref(sm), None, None), "device_info")
    return sm.value, torch.cuda.get_device_properties(0).shared_memory_per_block_optin


class s4conv_impl:
    def __init__(self, R, impl):
        self.R, self.impl = R, impl

    def __enter__(self):
        L_.check(self.R.lib.mugd_set_s4conv_impl(self.R.handle, self.impl), "s4conv_impl")

    def __exit__(self, *exc):
        L_.check(self.R.lib.mugd_set_s4conv_impl(self.R.handle, sc.AUTO), "s4conv_impl")


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.detach().contiguous().view(torch.int32)


# ---- kernel generation --------------------------------------------------------------------------------------------------------
# the plans' shapes, then: odd lengths (no Nyquist bin), L_out < L_int on odd lengths, the shortest lengths, and the longest the
# one-shot DFT takes (shared memory 16 (L/2 + 1 + L) B close to its 200 KB limit)
KGEN_CASES = sc.kgen_plan_shapes() + [(64, 63, 63), (48, 255, 200), (32, 1023, 1023), (16, 2, 2), (16, 3, 1), (16, 8191, 8191),
                                      (64, 8192, 5000), (32, 4096, 4096)]


def kernel_gen(R, dp, om, H, L_int, L_out):
    """mugd_s4_kernel_gen into Kt rows [0, L_out) of a buffer with 32 more rows of sentinel"""
    kt = torch.full((L_out + 32, H), SENT, device="cuda")
    ws = torch.zeros(2 * H * (L_int // 2 + 1) + 8, dtype=torch.float64, device="cuda")
    args = [ptr(dp[n]) for n in ("log_dt", "B", "C", "P", "inv_w_real", "w_imag")]
    L_.check(R.lib.mugd_s4_kernel_gen(R.handle, *args, ptr(om) if om is not None else None, H, 32, L_int, L_out, ptr(kt),
                                      ptr(ws), ws.numel() * 8, torch.cuda.current_stream().cuda_stream), "s4_kernel_gen")
    torch.cuda.synchronize()
    assert bool((kt[L_out:] == SENT).all()), "taps past L_out written"
    return kt[:L_out]


@pytest.mark.parametrize("H,L_int,L_out", KGEN_CASES, ids=lambda v: str(v))
def test_kernel_gen_tap_by_tap(R, H, L_int, L_out):
    p = sc.s4_params(H, seed=H + L_int)
    dp = {k: v.cuda() for k, v in p.items()}
    table = s4_fft_nodes(L_int)
    worst = {}
    for name, om, nodes in (("table", table.cuda(), sc.nodes64(L_int, table)), ("exact", None, sc.nodes64(L_int))):
        kt = kernel_gen(R, dp, om, H, L_int, L_out)
        k64 = sc.kgen64(p, L_int, L_out, nodes)
        worst[name] = float(sc.kgen_ratio(kt, k64).max())
    print(f"s4_kernel_gen H={H} L_int={L_int} L_out={L_out}: worst |Kt - K64| / (2^-24 |K64| + {sc.KGEN_EPS64:g} max|K64|) "
          f"table nodes {worst['table']:.3f}, exact nodes {worst['exact']:.3f}")
    assert max(worst.values()) <= KGEN_BOUND, worst


# ---- the convolution --------------------------------------------------------------------------------------------------------------
def run_conv(R, u, K, D, impl=sc.AUTO, strided=False):
    """s4conv of u [B, L, H] with taps K [L, H]; strided: u and y are column windows (8 columns in, 24 more after) of wider buffers,
    one row below their first row; u's other rows and columns hold NaN, y's a sentinel that must stay put.  Returns y [B, L, H]."""
    B, L, H = u.shape
    if strided:
        ld, c0 = H + 32, 8
        ub = torch.full((B * L + 2, ld), NAN, device="cuda")
        ub[1:-1, c0:c0 + H] = u.reshape(B * L, H)
        yb = torch.full((B * L + 2, ld), SENT, device="cuda")
        uv, yv = View(ptr(ub) + 4 * (ld + c0), ld, B * L, H), View(ptr(yb) + 4 * (ld + c0), ld, B * L, H)
    else:
        ub, yb = u.reshape(B * L, H).contiguous(), torch.full((B * L, H), SENT, device="cuda")
        uv, yv = View(ptr(ub), H, B * L, H), View(ptr(yb), H, B * L, H)
    Kc, Dc = K.contiguous(), D.contiguous()
    ops = OpList()
    ops.s4conv(uv, ptr(Kc), ptr(Dc), yv, B, L)
    with s4conv_impl(R, impl):
        R.run(ops)
    if not strided:
        return yb.view(B, L, H)
    outside = torch.ones_like(yb, dtype=torch.bool)
    outside[1:-1, c0:c0 + H] = False
    assert bool((yb[outside] == SENT).all()), "s4conv wrote outside its window"
    return yb[1:-1, c0:c0 + H].reshape(B, L, H)


def _case_id(c):
    B, L, H, strided = c
    return f"B{B}-L{L}-H{H}" + ("-strided" if strided else "")


@pytest.mark.parametrize("case", sc.conv_cases(), ids=_case_id)
def test_s4conv_against_fp64(R, dev, case):
    B, L, H, strided = case
    sm, smem = dev
    gen = torch.Generator(device="cuda").manual_seed(B * 100003 + L * 131 + H)
    u = torch.randn(B, L, H, generator=gen, device="cuda")
    D = torch.randn(H, generator=gen, device="cuda")
    worst = 0.0
    for kind in ("slow", "tail"):
        K = sc.taps(kind, L, H, gen, "cuda")
        y64, S = sc.conv64(u, K, D)
        for impl in sc.case_impls(B, L, H, smem):
            y = run_conv(R, u, K, D, impl, strided)
            r = float(sc.conv_ratio(y, y64, S).max())
            br = sc.s4conv_branch(B, L, H, sm, smem, impl)
            print(f"s4conv {_case_id(case):24s} taps={kind:4s} impl={IMPL_NAME[impl]:8s} {br.kernel:20s} nsplit={br.nsplit:<2d} "
                  f"{'odd ' if br.odd else 'even'}  worst ratio {r:.3f}")
            worst = max(worst, r)
        del y64, S
    assert worst <= sc.CONV_BOUND, worst


# ---- causality --------------------------------------------------------------------------------------------------------------------
# (impl, B, L, H, cuts): super-block edges (multiples of 16) and cuts inside one, the streamed kernel's window edges, and 1
CAUSAL = [(sc.RESIDENT, 2, 1584, 64, (512, 504, 500, 1)), (sc.RESIDENT, 3, 512, 128, (256, 17, 1)),
          (sc.STREAMED, 2, 2048, 64, (256, 768, 1000, 1)), (sc.STREAMED, 1, 1024, 32, (512, 255, 1)),
          (sc.AUTO, 2, 2048, 128, (1584, 1585, 512, 1))]


@pytest.mark.parametrize("impl,B,L,H,cuts", CAUSAL, ids=lambda v: str(v))
def test_s4conv_is_causal_bit_for_bit(R, dev, impl, B, L, H, cuts):
    """rows at and past a cut Lv hold NaN, +1e30 and -1e30: the outputs before Lv are the bits of the same call on u[:, :Lv]"""
    sm, smem = dev
    gen = torch.Generator(device="cuda").manual_seed(L + H)
    u = torch.randn(B, L, H, generator=gen, device="cuda")
    K, D = sc.taps("slow", L, H, gen, "cuda"), torch.randn(H, generator=gen, device="cuda")
    junk = torch.tensor([NAN, 1e30, -1e30], device="cuda").repeat((L * H + 2) // 3 + 1)[:L * H].view(L, H)
    for Lv in cuts:
        bad = u.clone()
        bad[:, Lv:] = junk[Lv:]
        full = run_conv(R, bad, K, D, impl)
        alone = run_conv(R, u[:, :Lv].contiguous(), K[:Lv], D, impl)
        print(f"causal {IMPL_NAME[impl]} B={B} L={L} H={H} cut {Lv}: {sc.s4conv_branch(B, L, H, sm, smem, impl)} / "
              f"{sc.s4conv_branch(B, Lv, H, sm, smem, impl)}")
        assert torch.equal(_bits(full[:, :Lv]), _bits(alone)), Lv


# ---- one S4 block, ragged, and captured -------------------------------------------------------------------------------------------
class Block:
    """an S4 block as UNetCompiler.emit_s4 emits it: GroupNorm(32) x -> g; s4conv g -> y; GLU GEMM y -> z (= g); [row mask z];
    k = 3 conv z -> out with residual x; tensor-core GEMMs over TF32-split weights"""

    def __init__(self, H, L, seed=0):
        gen = torch.Generator().manual_seed(seed)
        self.H = H
        self.gamma, self.beta = 1 + 0.1 * torch.randn(H, generator=gen), 0.1 * torch.randn(H, generator=gen)
        self.K = sc.taps("slow", L, H, gen) * 0.1
        self.D = torch.randn(H, generator=gen)
        self.Wg, self.bg = torch.randn(2 * H, H, generator=gen) / H ** 0.5, 0.1 * torch.randn(2 * H, generator=gen)
        self.Wo, self.bo = torch.randn(H, 3 * H, generator=gen) / (3 * H) ** 0.5, 0.1 * torch.randn(H, generator=gen)
        self.d = {k: v.cuda().contiguous() for k, v in vars(self).items() if isinstance(v, torch.Tensor)}
        for w in ("Wg", "Wo"):
            self.d[w + "_hi"], self.d[w + "_lo"] = (t.contiguous() for t in tf32_split(self.d[w]))

    def ops(self, x, g, y, out, B, L, valid=None):
        d, H = self.d, self.H
        v = lambda t: View(ptr(t), H, B * L, H)  # noqa: E731
        ops = OpList(valid=None if valid is None else {L: ptr(valid)})
        ops.groupnorm(v(x), v(g), ptr(d["gamma"]), ptr(d["beta"]), B, L, 32, False)
        ops.s4conv(v(g), ptr(d["K"]), ptr(d["D"]), v(y), B, L)
        ops.gemm(v(y), ptr(d["Wg"]), 2 * H, H, v(g), bias=ptr(d["bg"]), gate=L_.GATE_GLU, Lout=L, W_hi=ptr(d["Wg_hi"]),
                 W_lo=ptr(d["Wg_lo"]), impl=L_.GEMM_TC)
        if valid is not None:
            ops.row_mask(v(g), B, L)
        ops.gemm(v(g), ptr(d["Wo"]), H, H, v(out), bias=ptr(d["bo"]), taps=3, mode=L_.CONV_SAME, Lin=L, Lout=L, residual=v(x),
                 W_hi=ptr(d["Wo_hi"]), W_lo=ptr(d["Wo_lo"]), impl=L_.GEMM_TC)
        return ops


def _block_inputs(B, L, H, lens, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, L, H, generator=gen, device="cuda") * 2 + 0.3
    for b, Lv in enumerate(lens):
        x[b, Lv:] = NAN                                            # padding: never read into a valid row
    return x


BLOCKS = [(4, 512, 128, [512, 300, 1, 511]), (2, 2048, 128, [2048, 1500])]


@pytest.mark.parametrize("B,L,H,lens", BLOCKS, ids=lambda v: str(v))
def test_ragged_s4_block_equals_the_block_alone(R, dev, B, L, H, lens):
    sm, smem = dev
    blk = Block(H, L, seed=L)
    x = _block_inputs(B, L, H, lens, L)
    g, y, out = (torch.full((B, L, H), NAN, device="cuda") for _ in range(3))
    valid = torch.tensor(lens, dtype=torch.int32, device="cuda")
    R.run(blk.ops(x, g, y, out, B, L, valid))
    worst = 0.0
    for b, Lv in enumerate(lens):
        assert bool((g[b, Lv:] == 0).all()), b                     # the k = 3 conv reads zeros past the valid rows
        xa = x[b:b + 1, :Lv].contiguous()
        ga, ya, oa = (torch.full((1, Lv, H), NAN, device="cuda") for _ in range(3))
        R.run(blk.ops(xa, ga, ya, oa, 1, Lv))
        assert bool(torch.isfinite(out[b, :Lv]).all())
        worst = max(worst, rel_err(out[b, :Lv], oa[0]))
    print(f"ragged S4 block B={B} L={L} H={H} lengths {lens} ({sc.s4conv_branch(B, L, H, sm, smem)}): "
          f"valid rows vs the block alone, max rel err {worst:.2e}")
    assert worst <= 1e-5, worst


def make_plan(R, ops: OpList):
    for op in ops.ops:
        if op.kind == L_.OP_GEMM:
            gm = op.u.gemm
            gm.workspace, gm.workspace_bytes = R.ws.data_ptr(), R.ws.numel() * 4
            gm.counters, gm.n_counters = R.counters.data_ptr(), R.counters.numel()
    plan = C.c_void_p()
    L_.check(R.lib.mugd_plan_create(R.handle, ops.array(), len(ops.ops), C.byref(plan)), "plan_create")
    return plan


@pytest.mark.parametrize("B,L,H,lens", BLOCKS, ids=lambda v: str(v))
def test_captured_plan_orders_the_s4_block(R, dev, B, L, H, lens):
    """the ragged S4 block captured on a side stream with programmatic launch edges (PDL) and replayed once over g / y / out filled
    with NaN: the bits of the ops run one by one.  An s4conv that read g before the GroupNorm finished, a GEMM that read y early or
    a conv that read z before the row mask would leave NaN or other bits."""
    sm, smem = dev
    blk = Block(H, L, seed=L + 1)
    x = _block_inputs(B, L, H, lens, L + 1)
    g, y, out = (torch.full((B, L, H), NAN, device="cuda") for _ in range(3))
    valid = torch.tensor(lens, dtype=torch.int32, device="cuda")
    ops = blk.ops(x, g, y, out, B, L, valid)
    plan = make_plan(R, ops)
    st = torch.cuda.Stream()
    try:
        L_.check(R.lib.mugd_set_pdl(1), "pdl")
        R.run(ops)
        eager = [t.clone() for t in (g, y, out)]
        for t in (g, y, out):
            t.fill_(NAN)
        torch.cuda.synchronize()
        L_.check(R.lib.mugd_plan_capture(plan, C.c_void_p(st.cuda_stream)), "capture")
        assert bool(torch.isnan(out).all())                        # capturing runs nothing
        L_.check(R.lib.mugd_plan_replay(plan, 1, C.c_void_p(st.cuda_stream)), "replay")
        st.synchronize()
        for name, e, t in zip(("z", "y", "out"), eager, (g, y, out)):
            assert torch.equal(_bits(e), _bits(t)), name
        print(f"captured S4 block B={B} L={L} H={H}: s4conv {sc.s4conv_branch(B, L, H, sm, smem)}, replay bit-identical")
    finally:
        R.lib.mugd_set_pdl(int(os.environ.get("MUGD_PDL", "1") != "0"))
        R.lib.mugd_plan_destroy(plan)


# ---- y overlapping u ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", [sc.RESIDENT, sc.STREAMED], ids=["resident", "streamed"])
@pytest.mark.parametrize("B,L,H", [(2, 512, 128), (1, 96, 128)])
def test_s4conv_refuses_y_overlapping_u(R, dev, impl, B, L, H):
    """in place, or y one row into u, is refused by both kernels -- on the resident kernel both where this device splits a sample's
    outputs over CTAs (nsplit > 1 on an H100 for the first shape) and where it does not; y just past u runs"""
    sm, smem = dev
    br = sc.s4conv_branch(B, L, H, sm, smem, impl)
    print(f"overlap refusal {IMPL_NAME[impl]} B={B} L={L} H={H}: {br}")
    if impl == sc.RESIDENT and sm == sc.H100_SMS:
        assert (br.nsplit > 1) == (L == 512)
    buf = torch.randn(2 * B * L + 1, H, device="cuda")
    K, D = torch.randn(L, H, device="cuda"), torch.randn(H, device="cuda")
    u = View(ptr(buf), H, B * L, H)
    for y_row, refused in ((0, True), (1, True), (B * L - 1, True), (B * L, False)):
        ops = OpList()
        ops.s4conv(u, ptr(K), ptr(D), View(ptr(buf) + 4 * H * y_row, H, B * L, H), B, L)
        with s4conv_impl(R, impl):
            if refused:
                with pytest.raises(L_.MugdError, match="overlaps"):
                    R.run(ops)
            else:
                R.run(ops)

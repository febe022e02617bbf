"""CPU checks of the S4 references and case lists in s4_cases.py: the float64 kernel generator against its Nyquist limit, the
reference's complex64 oracle and its node drift; the per-output convolution bound against small mistakes it must catch; the
launch-rule restatement and the branch coverage of the GPU cases at the H100 SXM's 132 SMs."""
import pytest
import torch

import s4_cases as sc
from mug_diffusion_b200.runtime import s4_fft_nodes
from oracle import mug_oracle as orc


# ---- kernel generation ------------------------------------------------------------------------------------------------------------
def test_nyquist_limit_is_the_limit_of_the_woodbury_form():
    """k(-exp(i eps)) in the reference's Woodbury form tends to the closed form (dt/2) sum B C linearly in eps"""
    p = sc.s4_params(64)
    lim = sc.nyquist_limit(p)
    prev = None
    for e in (1e-2, 1e-3, 1e-4, 1e-5, 1e-6):
        k = sc.woodbury(p, -torch.exp(torch.tensor([1j * e], dtype=torch.complex128)))[:, 0]
        d = float(((k - lim).abs() / lim.abs()).max())
        assert d <= 10 * e, (e, d)
        if prev is not None:
            assert 8 <= prev / d <= 12, (e, prev, d)                   # first order in eps: a decade per decade
        prev = d


def test_kgen64_handles_the_nyquist_bin_only_for_exact_nodes():
    L = 96
    assert bool((sc.nodes64(L) == -1).any()) and not bool((sc.nodes64(L, s4_fft_nodes(L)) == -1).any())
    assert not bool((sc.nodes64(63) == -1).any())                        # odd length: no Nyquist bin
    k = sc.kgen64(sc.s4_params(32), L, L, sc.nodes64(L))
    assert bool(torch.isfinite(k).all())


def _oracle(p, L_int, L_out):
    sd = {"k." + n: v for n, v in p.items()}
    sd["k.L"] = torch.tensor(L_int)
    return orc.s4_nplr_kernel(sd, "k.", L_out).double()


@pytest.mark.parametrize("L_int,L_out", [(96, 96), (63, 63), (124, 124), (128, 100), (512, 512), (992, 992)])
def test_kgen64_at_the_table_nodes_matches_the_oracle(L_int, L_out):
    """the oracle is complex64 (mug_oracle.py:175-193): within its own rounding of 1e-5 of max|K| (measured <= 3.3e-6)"""
    p = sc.s4_params(64)
    k64 = sc.kgen64(p, L_int, L_out, sc.nodes64(L_int, s4_fft_nodes(L_int)))
    ref = _oracle(p, L_int, L_out)
    assert float((k64 - ref).abs().max() / ref.abs().max()) < 1e-5


def test_table_nodes_drift_from_exact_nodes_as_design_reports():
    """DESIGN §2: the reference's complex64 powers omega**f move K by 4e-5 (L = 96) ... 4e-4 (L = 992) of max|K|, growing with L"""
    p = sc.s4_params(64)
    drift = {}
    for L in (96, 512, 992):
        kt = sc.kgen64(p, L, L, sc.nodes64(L, s4_fft_nodes(L)))
        ke = sc.kgen64(p, L, L, sc.nodes64(L))
        drift[L] = float((kt - ke).abs().max() / kt.abs().max())
    assert 2e-5 <= drift[96] <= 8e-5 and 2e-4 <= drift[992] <= 8e-4, drift
    assert drift[96] < drift[512] < drift[992], drift


def test_kgen_ratio_rejects_a_wrong_tail_tap():
    """an error confined to the far taps, far below 1e-5 of max|K|, is still many fp32 roundings of those taps"""
    p = sc.s4_params(16)
    k64 = sc.kgen64(p, 512, 512, sc.nodes64(512))
    kt = k64.float().t().contiguous()
    assert float(sc.kgen_ratio(kt, k64).max()) <= 1.0 + 1e-6
    bad = kt.clone()
    bad[500] *= 1 + 2e-6                                                 # |K[500]| << max|K|: invisible to a max-relative bound
    assert float((bad.double().t() - k64).abs().max() / k64.abs().max()) < 1e-6
    assert float(sc.kgen_ratio(bad, k64).max()) > 4


def test_kgen_plan_shapes_follow_the_lengthen_rule():
    shapes = sc.kgen_plan_shapes()
    assert (128, 8192, 8192) in shapes and (128, 512, 96) in shapes and (512, 12, 12) in shapes
    assert any(L_out < L_int for _, L_int, L_out in shapes)
    ds = {128: 1, 256: 2, 384: 4, 512: 8}
    for H, L_int, L_out in shapes:
        assert L_out <= L_int
        # persisted at the request, or at 512 and doubled until it covers the request (s4_setup.lengthen)
        assert L_int in (L_out, sc.lengthened(512 // ds[H], L_out)), (H, L_int, L_out)
        assert 16 * (L_int // 2 + 1 + L_int) <= 200 * 1024           # within the one-shot DFT's shared memory (s4.cu)
    assert sc.lengthened(12, 1024) == 1536 and sc.lengthened(512, 96) == 512 and sc.lengthened(0, 100) == 100


# ---- the convolution bound --------------------------------------------------------------------------------------------------------
def _conv_case(L=1024, H=16, B=1, seed=0):
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(B, L, H, generator=g)
    K = sc.taps("slow", L, H, g)
    D = torch.randn(H, generator=g)
    return u, K, D


def _y(u, K, D):
    """gelu(conv(u, K) + D u) in float64, rounded to float32 like a kernel output"""
    return sc.conv64(u, K, D)[0].float()


def test_conv64_matches_a_direct_sum():
    u, K, D = _conv_case(L=200, H=4, B=2)
    y64, S = sc.conv64(u, K, D)
    ud, Kd, Dd = u.double(), K.double(), D.double()
    x = torch.stack([(Kd[:l + 1].flip(0)[None] * ud[:, :l + 1]).sum(1) for l in range(200)], dim=1) + ud * Dd
    s = torch.stack([(Kd[:l + 1].flip(0).abs()[None] * ud[:, :l + 1].abs()).sum(1) for l in range(200)], dim=1) + (ud * Dd).abs()
    assert float((y64 - sc.gelu64(x)).abs().max()) < 1e-12 and float((S - s).abs().max()) < 1e-11


def test_conv_bound_accepts_float32_sums():
    """a float32 causal sum in plain order (a Toeplitz matmul) and the float64 result rounded to float32 pass the bound"""
    u, K, D = _conv_case()
    y64, S = sc.conv64(u, K, D)
    L = u.shape[1]
    idx = torch.arange(L)[:, None] - torch.arange(L)[None, :]
    x32 = torch.einsum("lmh,bmh->blh", torch.where((idx >= 0)[..., None], K[idx.clamp(min=0)], 0.0), u) + u * D
    y32 = torch.nn.functional.gelu(x32)
    for y in (y64.float(), y32):
        assert float(sc.conv_ratio(y, y64, S).max()) <= sc.CONV_BOUND


def _shift_u(u):
    v = torch.zeros_like(u)
    v[:, 1:] = u[:, :-1]
    return v


def _drop_diag(u, K, D):
    """tap j = l dropped from every output l (it multiplies u[0])"""
    L = u.shape[1]
    x = sc._causal(u.double(), K.double(), L) + u.double() * D.double() - K.double()[None] * u.double()[:, :1]
    return sc.gelu64(x).float()


def _k_shifted(u, K, D):
    K2 = K.clone()
    K2[256:-1] = K[257:]
    K2[-1] = 0
    return _y(u, K2, D)


def _bf16_tile(u, K, D):
    u2 = u.clone()
    u2[:, 256:512] = u2[:, 256:512].bfloat16().float()
    return _y(u2, K, D)


MISTAKES = {
    "drop tap j = l": _drop_diag,
    "u shifted by one row": lambda u, K, D: _y(_shift_u(u), K, D),
    "K[j + 1] for j >= 256": _k_shifted,
    "u rounded to bf16 in one tile": _bf16_tile,
}


@pytest.mark.parametrize("name", list(MISTAKES))
def test_conv_bound_rejects_small_mistakes(name):
    u, K, D = _conv_case()
    y64, S = sc.conv64(u, K, D)
    bad = MISTAKES[name](u, K, D)
    r = float(sc.conv_ratio(bad, y64, S).max())
    print(f"{name}: worst ratio {r:.3g} (bound {sc.CONV_BOUND})")
    assert r > sc.CONV_BOUND, name


def test_taps_carry_weight_in_every_tile():
    g = torch.Generator().manual_seed(1)
    K = sc.taps("slow", 8192, 16, g)
    assert float(K[-256:].abs().max()) > 0.2 * float(K[:256].abs().max())
    T = sc.taps("tail", 1000, 16, g)
    assert bool((T[:744] == 0).all()) and bool((T[744:] != 0).all())


# ---- the launch rule and coverage -------------------------------------------------------------------------------------------------
def test_launch_rule_matches_the_sources_limits():
    """s4.cu: the resident kernel takes L <= 1584 on an H100 (L = 1600 needs 234,432 B, the refusal test_gpu_long checks); the
    streamed stage is 112,896 B"""
    assert sc.resident_smem(1584) <= sc.H100_SMEM_OPTIN < sc.resident_smem(1585) == sc.resident_smem(1600) == 234432
    assert sc.s4conv_branch(1, 1600, 64, impl=sc.RESIDENT) is None
    assert sc.s4conv_branch(1, 1584, 64).kernel.startswith("resident") and sc.s4conv_branch(1, 1585, 64).kernel == "streamed"
    assert sc.s4conv_branch(2, 512, 128) == sc.Branch("resident-interleaved", 2, False)
    assert sc.s4conv_branch(2, 1568, 128) == sc.Branch("resident-blocked", 4, False)
    assert sc.s4conv_branch(3, 1000, 48) == sc.Branch("resident-interleaved", 4, True)
    assert sc.s4conv_branch(32, 2048, 256) == sc.Branch("streamed", 1, False)
    assert sc.s4conv_branch(2, 1600, 128) == sc.Branch("streamed", 4, True)


def test_resident_nsplit_stops_at_4_on_an_h100():
    """the resident kernel holds at most 99 super blocks (50 pairs), and a split past 4 needs 64 pairs: nsplit >= 8 is not reachable
    at 132 SMs (it is on a device with more shared memory)"""
    classes = sc.reachable_classes()
    assert not any(c[1] == "nsplit>=8" for c in classes)
    assert ("resident-blocked", "nsplit>=8", "even") in sc.reachable_classes(132, 2 * sc.H100_SMEM_OPTIN, 64)


def test_gpu_cases_reach_every_branch_at_132_sms():
    reach = sc.reachable_classes()
    got = sc.case_branches(sc.conv_cases())
    assert reach - got == set(), sorted(reach - got)
    # the ones named in the S4 test plan
    assert ("resident-interleaved", "nsplit=2", "even") in got or ("resident-interleaved", "nsplit=2", "odd") in got
    for ns in (1, 2, 4):
        assert any(c[0].startswith("resident") and c[1] == f"nsplit={ns}" for c in got), ns
    assert {("streamed", "nsplit=1"), ("streamed", "nsplit>1")} <= {c[:2] for c in got}
    assert any(c[0] == "streamed" and c[2] == "odd" for c in got)


def test_plan_walk_finds_every_s4_layer():
    shapes = sc.plan_s4conv_shapes()
    assert len(shapes) == len(sc.PLAN_Z) * len(sc.PLAN_BEFF) * 4
    for Beff in sc.PLAN_BEFF:
        for Lz in sc.PLAN_Z:
            for H, ds in ((128, 1), (256, 2), (384, 4), (512, 8)):
                assert (Beff, Lz // ds, H) in shapes
    assert {h for h, _ in sc.s4_blocks()} == {128, 256, 384, 512} and len(sc.s4_blocks()) == 16

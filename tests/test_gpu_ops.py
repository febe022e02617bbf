"""Per-kernel parity: every libmugd op, called through the C ABI (mugd_op_run), against the CPU oracle /
a plain torch fp32 statement of the same op on the same seeded inputs.  Run on the GPU: pytest -m gpu.

Tolerances (fp32 path): 2e-5 relative to the output's max magnitude for contractions (different
summation order only), bit-exact for the DDIM update and the copies.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.engine import OpList  # noqa: E402

import golden_cases as gc  # noqa: E402
from gpu_util import OpRunner, ncl, nlc, ptr, rel_err, view  # noqa: E402
from oracle import mug_oracle as orc  # noqa: E402


@pytest.fixture(scope="module")
def R():
    return OpRunner()


def g(name, shape, seed=5):
    return synth._gauss(synth._rng(seed, name), shape)


# ---------------------------------------------------------------------------------------------------
# the GroupNorm / LayerNorm kernels on their own: test_gpu_norm.py


# ---------------------------------------------------------------------------------------------------
def run_gemm(R, A, Wp, N, K, M, ncols_out, **kw):
    out = torch.zeros(M, ncols_out).cuda()
    ops = OpList()
    ops.gemm(view(A), ptr(Wp), N, K, view(out), **kw)
    R.run(ops)
    return out


@pytest.mark.parametrize("M,K,N,act", [(100, 128, 512, L_.ACT_SILU), (50, 512, 7424, L_.ACT_NONE), (777, 256, 16, L_.ACT_GELU),
                                       (8192, 64, 1024, L_.ACT_NONE)])
def test_gemm_linear(R, M, K, N, act):
    x, w, b = g("lx", (M, K)), g("lw", (N, K)) / math.sqrt(K), 0.1 * g("lb", (N,))
    ref = F.linear(x, w, b)
    ref = F.silu(ref) if act == L_.ACT_SILU else F.gelu(ref) if act == L_.ACT_GELU else ref
    wc, bc = w.cuda(), b.cuda()
    out = run_gemm(R, x.cuda(), wc, N, K, M, N, bias=ptr(bc), act=act)
    assert rel_err(out, ref) < 2e-5


@pytest.mark.parametrize("B,L,Cin,Cout", [(2, 48, 384, 128), (3, 12, 1536, 512), (1, 100, 16, 128), (2, 96, 128, 16)])
def test_gemm_conv3_same_rowvec_residual(R, B, L, Cin, Cout):
    x, w, b = g("cx", (B, Cin, L)), g("cw", (Cout, Cin, 3)) / math.sqrt(3 * Cin), 0.1 * g("cb", (Cout,))
    emb, res = g("ce", (B, Cout)), g("cr", (B, Cout, L))
    ref = F.conv1d(x, w, b, padding=1) + emb[:, :, None] + res
    wp = w.permute(0, 2, 1).contiguous().reshape(Cout, 3 * Cin).cuda()
    bc, ec, rc = b.cuda(), emb.cuda(), nlc(res).cuda()
    out = run_gemm(R, nlc(x).cuda(), wp, Cout, Cin, B * L, Cout, bias=ptr(bc), taps=3, mode=L_.CONV_SAME, Lin=L, Lout=L,
                   rowvec=ptr(ec), rowvec_b_stride=Cout, residual=view(rc))
    assert rel_err(ncl(out.cpu(), B), ref) < 2e-5


def test_gemm_rowvec_step_indexing(R):
    """time-embedding row selected on the device: rowvec[step*stride + n], shared by all samples"""
    B, L, Cin, Cout, S = 2, 16, 64, 128, 5
    x, w = g("sx", (B, Cin, L)), g("sw", (Cout, Cin, 3)) / math.sqrt(3 * Cin)
    table = g("st", (S, Cout))
    wp = w.permute(0, 2, 1).contiguous().reshape(Cout, 3 * Cin).cuda()
    tc = table.cuda()
    step = torch.tensor([3], dtype=torch.int32).cuda()
    out = run_gemm(R, nlc(x).cuda(), wp, Cout, Cin, B * L, Cout, taps=3, mode=L_.CONV_SAME, Lin=L, Lout=L, rowvec=ptr(tc),
                   rowvec_b_stride=0, rowvec_step_stride=Cout, step=ptr(step))
    ref = F.conv1d(x, w, None, padding=1) + table[3][None, :, None]
    assert rel_err(ncl(out.cpu(), B), ref) < 2e-5


# the FFMA GEMM's addressing modes, gates, column windows and refusals: test_gpu_gemm_epilogue.py (ffma path) and test_gemm_cases.py


# ---------------------------------------------------------------------------------------------------
# the attention kernels on their own: test_gpu_attention.py
@pytest.mark.parametrize("name", list(gc.ATTN_CORE_CASES))
def test_attention_vs_reference_golden(R, name, golden_dir):
    """whole CrossAttention module (to_q/k/v GEMMs + attention + to_out) against the reference's output"""
    import os
    case = gc.ATTN_CORE_CASES[name]
    sd = synth.synthetic_state_dict(gc.BLOCK_L, decoder=False)
    x, ctx = gc.attn_core_inputs(name, case)
    p = case["prefix"]
    B, Lq, C = x.shape
    src = x if ctx is None else ctx
    Lk = src.shape[1]
    xc, sc = x.reshape(B * Lq, C).cuda(), src.reshape(B * Lk, -1).contiguous().cuda()
    wq, wk, wv = sd[p + "to_q.weight"].cuda(), sd[p + "to_k.weight"].cuda(), sd[p + "to_v.weight"].cuda()
    wo, bo = sd[p + "to_out.0.weight"].cuda(), sd[p + "to_out.0.bias"].cuda()
    rel, cg = sd[p + "relative_position_embedding"].cuda(), sd[p + "C_embedding"].cuda()
    q, k, v = torch.zeros(B * Lq, C).cuda(), torch.zeros(B * Lk, C).cuda(), torch.zeros(B * Lk, C).cuda()
    ao, out = torch.zeros(B * Lq, C).cuda(), torch.zeros(B * Lq, C).cuda()
    ops = OpList()
    ops.gemm(view(xc), ptr(wq), C, C, view(q))
    ops.gemm(view(sc), ptr(wk), C, sc.shape[1], view(k))
    ops.gemm(view(sc), ptr(wv), C, sc.shape[1], view(v))
    ops.attention(view(q), view(k), view(v), view(ao), ptr(rel), ptr(cg), B, 8, Lq, Lk, 64)
    ops.gemm(view(ao), ptr(wo), C, C, view(out), bias=ptr(bo))
    R.run(ops)
    gold = gc.load_golden(os.path.join(golden_dir, "blocks_L96.npz"))["core." + name]
    assert rel_err(out.view(B, Lq, C), gold) < 3e-5


# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,L,H", [(2, 96, 128), (1, 512, 128), (3, 124, 512), (2, 250, 64), (1, 992, 128)])
def test_s4conv(R, B, L, H):
    u, K, D = g("su", (B, H, L)), g("sk", (H, L)) * torch.exp(-torch.arange(L) / 40.0)[None], g("sd", (H,))
    y = torch.fft.irfft(torch.fft.rfft(u, n=2 * L) * torch.fft.rfft(K, n=2 * L)[None], n=2 * L)[..., :L]
    ref = F.gelu(y + u * D[None, :, None])
    uc, kt, dc = nlc(u).cuda(), K.t().contiguous().cuda(), D.cuda()
    out = torch.zeros(B * L, H).cuda()
    ops = OpList()
    ops.s4conv(view(uc), ptr(kt), ptr(dc), view(out), B, L)
    R.run(ops)
    assert rel_err(ncl(out.cpu(), B), ref) < 2e-5


@pytest.mark.parametrize("L_int,L_out,H", [(96, 96, 128), (24, 24, 384), (512, 512, 128), (124, 124, 512), (128, 100, 64), (63, 63, 32),
                                           (992, 992, 128)])
def test_s4_kernel_gen_vs_oracle(R, L_int, L_out, H):
    import ctypes as C
    N = 32
    pre = "k."
    sd = {pre + n: synth._init("t." + n, shp, role, 3) for n, shp, role in [
        ("C", (1, H, N, 2), "s4_C"), ("log_dt", (H,), "s4_log_dt"), ("B", (1, H, N, 2), "s4_B"), ("P", (1, H, N, 2), "s4_P"),
        ("inv_w_real", (H, N), "s4_inv_w_real"), ("w_imag", (H, N), "s4_w_imag")]}
    sd[pre + "L"] = torch.tensor(L_int)
    ref = orc.s4_nplr_kernel(sd, pre, L_out)                     # [H, L_out]
    dev = {k: v.cuda() for k, v in sd.items() if k != pre + "L"}
    kt = torch.zeros(L_out, H).cuda()
    ws = torch.zeros(2 * H * (L_int // 2 + 1) + 8, dtype=torch.float64).cuda()
    from mug_diffusion_b200.runtime import s4_fft_nodes
    st = torch.cuda.current_stream().cuda_stream
    args = [ptr(dev[pre + n]) for n in ("log_dt", "B", "C", "P", "inv_w_real", "w_imag")]
    om = s4_fft_nodes(L_int).cuda()
    L_.check(R.lib.mugd_s4_kernel_gen(R.handle, *args, ptr(om), H, N, L_int, L_out, ptr(kt), ptr(ws), ws.numel() * 8, st), "s4_kernel_gen")
    torch.cuda.synchronize()
    # with the reference's own FFT nodes the fp64 generator reproduces the reference's fp32 kernel to its rounding noise
    assert rel_err(kt.t(), ref) < 1e-5
    # with exact nodes (omega = NULL) it differs by the drift of the reference's complex64 omega**f: ~4e-5 @96 .. 4e-4 @992
    L_.check(R.lib.mugd_s4_kernel_gen(R.handle, *args, None, H, N, L_int, L_out, ptr(kt), ptr(ws), ws.numel() * 8, st), "s4_kernel_gen")
    torch.cuda.synchronize()
    assert rel_err(kt.t(), ref) < 1e-3


def test_s4_kernel_gen_vs_reference_golden(R, golden_dir):
    import os
    gold = gc.load_golden(os.path.join(golden_dir, "blocks_L96.npz"))
    sd = synth.synthetic_state_dict(gc.BLOCK_L, decoder=False)
    for name in ("s4_l0", "s4_l2"):
        case = gc.BLOCK_CASES[name]
        k = case["prefix"] + "s4_model.kernel.kernel."
        H, Lr = case["cin"], gc.BLOCK_L // case["ds"]
        dev = {n: sd[k + n].cuda() for n in ("log_dt", "B", "C", "P", "inv_w_real", "w_imag")}
        kt = torch.zeros(Lr, H).cuda()
        ws = torch.zeros(2 * H * (Lr // 2 + 1) + 8, dtype=torch.float64).cuda()
        from mug_diffusion_b200.runtime import s4_fft_nodes
        om = s4_fft_nodes(Lr).cuda()
        L_.check(R.lib.mugd_s4_kernel_gen(R.handle, ptr(dev["log_dt"]), ptr(dev["B"]), ptr(dev["C"]), ptr(dev["P"]), ptr(dev["inv_w_real"]),
                                          ptr(dev["w_imag"]), ptr(om), H, 32, Lr, Lr, ptr(kt), ptr(ws), ws.numel() * 8,
                                          torch.cuda.current_stream().cuda_stream), "s4_kernel_gen")
        torch.cuda.synchronize()
        assert rel_err(kt.t(), gold[name + ".K"]) < 1e-5


# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg,sigma", [(False, 0.0), (True, 0.0), (True, 0.37)])
def test_ddim_update_bit_exact(R, cfg, sigma):
    B, L, Cc, S = 2, 40, 16, 7
    n = B * L * Cc
    x, eu, ec, nz = g("dx", (n,)), g("du", (n,)), g("dc", (n,)), g("dn", (n,))
    coef = torch.rand(S, 4, generator=torch.Generator().manual_seed(1)) * 0.5 + 0.2
    coef[:, 2] = sigma
    step, scale, temp = 2, 5.0, 0.9
    idx = S - 1 - step
    a_t, a_prev, sg, s1m = (coef[idx, j] for j in range(4))
    e = eu + scale * (ec - eu) if cfg else ec
    pred = (x - s1m * e) / a_t.sqrt()
    xp = a_prev.sqrt() * pred + (1.0 - a_prev - sg ** 2).sqrt() * e + sg * nz * temp
    xc, epsc, nzc, cc = x.cuda(), (torch.cat([eu, ec]) if cfg else ec).cuda(), nz.cuda(), coef.cuda()
    predc, dup, stp = torch.zeros(n).cuda(), torch.zeros(n).cuda(), torch.tensor([step], dtype=torch.int32).cuda()
    d = L_.DdimUpdate()
    d.x, d.x_dup, d.eps, d.noise, d.pred_x0, d.coef, d.step = ptr(xc), ptr(dup), ptr(epsc), ptr(nzc) if sigma else None, ptr(predc), ptr(cc), ptr(stp)
    d.S, d.n, d.cfg, d.scale, d.temperature = S, n, int(cfg), scale, temp
    adv = L_.StepAdvance()
    adv.step = ptr(stp)
    ops = OpList()
    ops.add(L_.OP_DDIM_UPDATE, d)
    ops.add(L_.OP_STEP_ADVANCE, adv)
    R.run(ops)
    assert torch.equal(xc.cpu(), xp) and torch.equal(dup.cpu(), xp) and torch.equal(predc.cpu(), pred)
    assert int(stp.item()) == step + 1


def test_transpose_and_copy(R):
    B, Cc, L = 3, 100, 77
    x = g("tx", (B, Cc, L)).cuda()
    wide = torch.zeros(B * L, Cc + 28).cuda()
    ops = OpList()
    ops.transpose(ptr(x), wide.data_ptr() + 4 * 12, 0, Cc + 28, B, Cc, L, True)
    R.run(ops)
    assert torch.equal(wide[:, 12:12 + Cc].reshape(B, L, Cc).permute(0, 2, 1), x)
    back = torch.zeros(B, Cc, L).cuda()
    ops = OpList()
    ops.transpose(wide.data_ptr() + 4 * 12, ptr(back), Cc + 28, 0, B, Cc, L, False)
    R.run(ops)
    assert torch.equal(back, x)
    dst = torch.zeros(B * L, 128).cuda()
    ops = OpList()
    ops.copy2d(view(wide, 12, 112), view(dst, 8, 108))
    R.run(ops)
    assert torch.equal(dst[:, 8:108], wide[:, 12:112])

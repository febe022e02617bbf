"""LayerNorm fold of the U-Net plan (round 2): the producer of a LayerNorm's input accumulates the row moments in its epilogue /
split-K reduce, the Linear behind the LayerNorm runs on the raw rows and corrects in its epilogue -- against a plain torch fp64
statement of the reference ops (attention.py:136-151 LayerNorm eps 1e-5 + Linear), through the C ABI."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.engine import OpList  # noqa: E402
from mug_diffusion_b200.packer import _interleave_halves, tf32_split  # noqa: E402

from gpu_util import OpRunner, ncl, nlc, ptr, rel_err, view  # noqa: E402


@pytest.fixture(scope="module")
def R():
    return OpRunner()


def g(name, shape, seed=21):
    return synth._gauss(synth._rng(seed, name), shape)


def _tc_weights(w2d):
    hi, lo = tf32_split(w2d)
    return w2d.cuda(), hi.cuda(), lo.cuda()


@pytest.mark.parametrize("M,K,N,split", [(1024, 256, 256, 0), (512, 512, 512, 4), (300, 384, 384, 0), (2048, 128, 64, 0), (640, 256, 512, 2)])
def test_row_moment_sinks(R, M, K, N, split):
    """Linear whose output rows a LayerNorm will normalise: every column tile adds its share of the row's moments"""
    x, w, b = g("rx", (M, K)), g("rw", (N, K)) / math.sqrt(K), 0.1 * g("rb", (N,))
    wc, hc, lc = _tc_weights(w)
    xc, bc = x.cuda(), b.cuda()
    out = torch.zeros(M, N).cuda()
    stats = torch.zeros(M, 2, dtype=torch.float64).cuda()
    ops = OpList()
    i = ops.gemm(view(xc), ptr(wc), N, K, view(out), W_hi=ptr(hc), W_lo=ptr(lc), bias=ptr(bc), impl=L_.GEMM_TC, split_k=split)
    assert ops.can_deliver_row_moments(i)
    ops.ops[i].u.gemm.row_moments = stats.data_ptr()
    R.run(ops)
    o = out.cpu().double()
    exp = torch.stack([o.sum(-1), (o ** 2).sum(-1)], dim=1)
    assert float((stats.cpu() - exp).abs().max() / exp.abs().max()) < 1e-6        # row sums reduce in fp32 inside a tile


@pytest.mark.parametrize("gate", [L_.GATE_NONE, L_.GATE_GEGLU], ids=["linear", "geglu"])
@pytest.mark.parametrize("M,C,N,split", [(1024, 256, 768, 0), (512, 512, 512, 4), (200, 384, 384, 0), (512, 512, 1024, 0)])
def test_layernorm_folded_into_linear(R, M, C, N, split, gate):
    """Linear(LayerNorm(h)) (attention.py:147-151) as one GEMM on the raw rows: W' = W diag(gamma), epilogue rstd*(acc - mean*colsum) + b',
    with the row moments delivered by the producer of h (here: a first GEMM with row_moments set).  Rows with a large mean included."""
    if gate == L_.GATE_GEGLU and N % 2:
        pytest.skip("gated N must be even")
    a, w0 = g("la", (M, C)), g("lw0", (C, C)) / math.sqrt(C)
    b0 = 3.0 * g("lb0", (C,))                                     # pushes |mean| of h above its spread: the cancellation case
    gam, bet = 1 + 0.2 * g("lg", (C,)), 0.1 * g("lbt", (C,))
    w1, b1 = g("lw1", (N, C)) / math.sqrt(C), 0.1 * g("lb1", (N,))
    h = F.linear(a.double(), w0.double(), b0.double())
    y = F.linear(F.layer_norm(h, (C,), gam.double(), bet.double(), 1e-5), w1.double(), b1.double())
    if gate == L_.GATE_GEGLU:
        v, gt = y.chunk(2, dim=-1)
        y = v * F.gelu(gt)
        w1p, b1p = _interleave_halves(w1), _interleave_halves(b1)
    else:
        w1p, b1p = w1, b1
    wg = (w1p.double() * gam.double()[None]).float()
    colsum = wg.double().sum(1).float()
    bias = (w1p.double() @ bet.double() + b1p.double()).float()
    w0c, h0c, l0c = _tc_weights(w0)
    wgc, hgc, lgc = _tc_weights(wg)
    ac, b0c, csc, bc = a.cuda(), b0.cuda(), colsum.cuda(), bias.cuda()
    hbuf = torch.zeros(M, C).cuda()
    out = torch.zeros(M, N // 2 if gate else N).cuda()
    stats = torch.zeros(M, 2, dtype=torch.float64).cuda()
    ops = OpList()
    i = ops.gemm(view(ac), ptr(w0c), C, C, view(hbuf), W_hi=ptr(h0c), W_lo=ptr(l0c), bias=ptr(b0c), impl=L_.GEMM_TC)
    ops.ops[i].u.gemm.row_moments = stats.data_ptr()
    ops.gemm(view(hbuf), ptr(wgc), N, C, view(out), W_hi=ptr(hgc), W_lo=ptr(lgc), bias=ptr(bc), gate=gate, impl=L_.GEMM_TC, split_k=split,
             ln=(stats.data_ptr(), ptr(csc), 1e-5))
    R.run(ops)
    e = rel_err(out, y)
    print(f"ln-fold M={M} C={C} N={N} split={split} gate={gate} rel_err={e:.2e}")
    assert e < 2e-5


def test_folded_plan_equals_plain_plan():
    """one U-Net evaluation with every LayerNorm folded against the same engine compiled with stand-alone LayerNorm kernels:
    same network, different launch plan"""
    from mug_diffusion_b200.sampler import MugDiffusionB200
    L, B = 160, 3
    sd = synth.synthetic_state_dict(L)
    inp = synth.synthetic_inputs(B, L, seed=5)
    t = torch.tensor([3, 500, 999]).cuda()
    outs = []
    for fuse in (True, False):
        m = MugDiffusionB200(sd, z_length=L, fold_ln=fuse)
        outs.append(m.model.forward(inp["x_T"].cuda(), t, inp["c"].cuda(), [w.cuda() for w in inp["w"]]).cpu())
        sess = next(iter(m.engine.sessions.values()))
        kinds = [sess.plan._arr[i].kind for i in range(sess.plan.n_ops)]
        assert (kinds.count(L_.OP_LAYERNORM) == 0) == fuse
        del m
    assert rel_err(outs[0], outs[1]) < 2e-5


def test_device_side_tf32_split_is_bit_identical_to_the_host_statement(R):
    """MUGD_OP_TF32_SPLIT: hi over the plain weight, lo beside it -- the same two roundings as packer.tf32_split, bit for bit"""
    w = g("split_w", (384, 1152), seed=5) * torch.logspace(-6, 3, 1152)[None, :]     # a wide range of exponents
    hi, lo = tf32_split(w)
    wc, lc = w.cuda(), torch.full_like(w, 7.0).cuda()
    ops = OpList()
    d = L_.Tf32Split()
    d.w_hi, d.lo, d.n = ptr(wc), ptr(lc), w.numel()
    ops.add(L_.OP_TF32_SPLIT, d)
    R.run(ops)
    assert torch.equal(wc.cpu().view(torch.int32), hi.view(torch.int32))
    assert torch.equal(lc.cpu().view(torch.int32), lo.view(torch.int32))
    assert int((wc.view(torch.int32) & 0x1FFF).abs().max()) == 0          # TF32 operands: 13 low mantissa bits clear


def test_engine_keeps_every_weight_once_plus_the_lo_halves():
    """resident weights = the packed fp32 blob (tensor-core weights overwritten by their hi halves) + one lo buffer; the host blob
    stays plain fp32 and an engine switched to the exact-fp32 FFMA path gets the plain weights back"""
    from mug_diffusion_b200.config import ModelConfig
    from mug_diffusion_b200.runtime import MugEngine
    cfg = ModelConfig()
    sd = synth.synthetic_state_dict(96)
    eng = MugEngine(sd, cfg, torch.device("cuda:0"))
    blob = eng.blob
    assert eng.weights.numel() == blob.numel and eng.weights_lo.numel() == blob.tc_lo_numel
    assert blob.tc_lo_numel < blob.numel                                   # lo exists for the tensor-core weights only
    assert blob.data.device.type == "cpu"
    name, off, n, lo = blob.tc[len(blob.tc) // 2]
    hi_ref, lo_ref = tf32_split(blob.data[off:off + n])
    assert torch.equal(eng.weights[off:off + n].cpu(), hi_ref) and torch.equal(eng.weights_lo[lo:lo + n].cpu(), lo_ref)
    in_tc = torch.zeros(blob.numel, dtype=torch.bool)
    for _, o, m, _ in blob.tc:
        in_tc[o:o + m] = True
    assert torch.equal(eng.weights.cpu()[~in_tc], blob.data[~in_tc])       # everything else is untouched
    eng.set_gemm_impl("simt")
    assert torch.equal(eng.weights.cpu(), blob.data)
    eng.set_gemm_impl("auto")
    assert torch.equal(eng.weights[off:off + n].cpu(), hi_ref)


def test_engines_over_one_device_resident_blob_share_its_split():
    """a second engine over the same device-resident blob tensor (what dist.broadcast_blob hands every rank) takes the first engine's
    lo buffer instead of splitting the tensor again, which would leave a zero lo; with no host copy the FFMA path is refused"""
    from mug_diffusion_b200.config import ModelConfig
    from mug_diffusion_b200.packer import pack_model
    from mug_diffusion_b200.runtime import MugEngine
    cfg = ModelConfig()
    blob = pack_model(synth.synthetic_state_dict(96), cfg.unet, cfg.decoder)
    host = blob.data
    blob.data = host.cuda()
    e1 = MugEngine(None, cfg, torch.device("cuda:0"), blob=blob)
    e2 = MugEngine(None, cfg, torch.device("cuda:0"), blob=blob)
    assert e1.weights is blob.data and e2.weights is blob.data and e2.weights_lo is e1.weights_lo and e2.tc_map == e1.tc_map
    name, off, n, lo = blob.tc[len(blob.tc) // 2]
    hi_ref, lo_ref = tf32_split(host[off:off + n])
    assert torch.equal(blob.data[off:off + n].cpu(), hi_ref) and torch.equal(e2.weights_lo[lo:lo + n].cpu(), lo_ref)
    with pytest.raises(L_.MugdError):
        e2.set_gemm_impl("simt")

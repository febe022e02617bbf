"""Multi-GPU path on real devices (needs >= 2 GPUs; skipped otherwise): rank 0 packs, one NCCL broadcast of the blob, every rank
samples its contiguous shard of the batch, logits are gathered on rank 0 -- and must equal the single-GPU run of the whole batch
bit for bit (samples are independent; the per-rank plans have the same per-GPU batch as the chunks of the single-GPU reference)."""
import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, L, B, S, out_path):
    import torch.distributed as dist
    from mug_diffusion_b200 import synth
    from mug_diffusion_b200.config import ModelConfig
    from mug_diffusion_b200.dist import broadcast_blob, sample_sharded
    from mug_diffusion_b200.sampler import DDIMSampler, MugDiffusionB200

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device(f"cuda:{rank}")
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    cfg = ModelConfig()
    sd = synth.synthetic_state_dict(L) if rank == 0 else None
    blob = broadcast_blob(sd, cfg, dev)
    m = MugDiffusionB200(None, cfg, z_length=L, device=dev, blob=blob)
    # the request lives on rank 0 only; the other ranks know its shapes
    shapes = dict(x_T=(B, 16, L), c=(B, 128, 21), uc=(B, 128, 21), w0=(B, 256, L), w1=(B, 512, L // 2), w2=(B, 512, L // 4), w3=(B, 512, L // 8))
    req = None
    if rank == 0:
        inp = synth.synthetic_inputs(B, L, seed=3)
        req = dict(x_T=inp["x_T"], c=inp["c"], uc=inp["uc"], w=list(inp["w"])[-4:])
    sampler = DDIMSampler(m)

    def run(xT, c, uc, w):
        z, _ = sampler.sample(S=S, c=c, w=w, batch_size=c.shape[0], verbose=False, x_T=xT, eta=0.0, shape=(16, L),
                              unconditional_guidance_scale=5.0, unconditional_conditioning=uc)
        return m.model.decode(z)

    full = sample_sharded(run, req, shapes, dev)
    if rank == 0:
        torch.save(full.cpu(), out_path)
    dist.destroy_process_group()


def test_two_rank_sharded_sampling_equals_single_gpu(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from mug_diffusion_b200 import synth
    from mug_diffusion_b200.sampler import DDIMSampler, MugDiffusionB200

    L, B, S, world = 96, 4, 4, 2
    out_path = str(tmp_path / "gathered.pt")
    mp.spawn(_worker, args=(world, _free_port(), L, B, S, out_path), nprocs=world, join=True)
    gathered = torch.load(out_path)
    # single-GPU reference: the same charts, sampled in the same per-GPU chunks (identical plans -> bit-identical results)
    m = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L)
    inp = synth.synthetic_inputs(B, L, seed=3)
    sampler = DDIMSampler(m)
    chunks = []
    for lo in range(0, B, B // world):
        sl = slice(lo, lo + B // world)
        z, _ = sampler.sample(S=S, c=inp["c"][sl].cuda(), w=[t[sl].cuda() for t in inp["w"]], batch_size=B // world, verbose=False,
                              x_T=inp["x_T"][sl].cuda(), eta=0.0, shape=(16, L), unconditional_guidance_scale=5.0,
                              unconditional_conditioning=inp["uc"][sl].cuda())
        chunks.append(m.model.decode(z).cpu())
    single = torch.cat(chunks)
    assert gathered.shape == single.shape == (B, 16, 8 * L)
    assert torch.equal(gathered, single)


def test_ops_bit_identical_on_two_devices_of_one_process():
    """One process, one handle per device: the tensor-core GEMM, the tensor-core attention and the S4 convolution (each needs more than
    48 KB of shared memory, an attribute of the device's context) run on cuda:0 and cuda:1 and agree bit for bit."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import ctypes as C
    import math

    import torch.nn.functional as F
    from gpu_util import ptr, rel_err, view
    from mug_diffusion_b200 import lib as L_
    from mug_diffusion_b200 import synth
    from mug_diffusion_b200.engine import OpList
    from mug_diffusion_b200.packer import tf32_split

    def g(name, shape):
        return synth._gauss(synth._rng(13, name), shape)

    M, K, N = 1024, 256, 384                              # GEMM
    B, H, D, L = 2, 8, 64, 256                            # attention: 256 keys -> tensor-core kernel
    Bs, Ls, Hs = 2, 512, 128                              # S4 convolution
    x, w = g("x", (M, K)), g("w", (N, K)) / math.sqrt(K)
    w_hi, w_lo = tf32_split(w)
    q, k, v = g("q", (B * L, H * D)), g("k", (B * L, H * D)), g("v", (B * L, H * D))
    rel, cg = 0.5 * g("rel", (129, H)), 1 + 0.1 * g("cg", (129, H))
    u, kt, dsk = g("u", (Bs * Ls, Hs)), g("kt", (Ls, Hs)) * 0.05, g("d", (Hs,))
    lib = L_.load()
    results = []
    for dev in (0, 1):
        with torch.cuda.device(dev):
            handle = C.c_void_p()
            L_.check(lib.mugd_create(dev, C.byref(handle)), f"mugd_create({dev})")
            try:
                xc, wc, hc, lc = (t.to(f"cuda:{dev}") for t in (x, w, w_hi, w_lo))
                qc, kc, vc, relc, cgc = (t.to(f"cuda:{dev}") for t in (q, k, v, rel, cg))
                uc, ktc, dc = (t.to(f"cuda:{dev}") for t in (u, kt, dsk))
                ws = torch.zeros(16 * 1024 * 1024, device=f"cuda:{dev}")
                out_g = torch.zeros(M, N, device=f"cuda:{dev}")
                out_a = torch.zeros(B * L, H * D, device=f"cuda:{dev}")
                out_s = torch.zeros(Bs * Ls, Hs, device=f"cuda:{dev}")
                ops = OpList()
                ops.gemm(view(xc), ptr(wc), N, K, view(out_g), W_hi=ptr(hc), W_lo=ptr(lc), impl=L_.GEMM_TC)
                ops.ops[0].u.gemm.workspace, ops.ops[0].u.gemm.workspace_bytes = ws.data_ptr(), ws.numel() * 4
                ops.attention(view(qc), view(kc), view(vc), view(out_a), ptr(relc), ptr(cgc), B, H, L, L, 64)
                ops.s4conv(view(uc), ptr(ktc), ptr(dc), view(out_s), Bs, Ls)
                st = torch.cuda.current_stream().cuda_stream
                for op in ops.ops:
                    L_.check(lib.mugd_op_run(handle, C.byref(op), st), f"op {op.kind} on cuda:{dev}")
                torch.cuda.synchronize()
                results.append([t.cpu() for t in (out_g, out_a, out_s)])
            finally:
                lib.mugd_destroy(handle)
    assert rel_err(results[0][0], F.linear(x.double(), w.double())) < 1e-5
    for a, b in zip(*results):
        assert torch.equal(a, b)

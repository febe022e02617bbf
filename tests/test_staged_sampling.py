"""The host side of the device loop for inpainting and eta > 0 requests, without a GPU: the up-front draw of a stretch's random numbers
reproduces the per-step loop's sequence and leaves the generator where that loop leaves it, and the routing keeps the requests on which
the per-step ops would promote or raise on the per-step loop."""
import pytest
import torch

from mug_diffusion_b200.sampler import draw_step_noise, takes_device_loop

SHAPE = (2, 16, 24)
STEPS = 7


def per_step_sequence(mask: bool, draw: bool, dropout: float, x0):
    """the draws of ddim_sampling's per-step branch, step by step: q_sample's randn_like(x0), then randn(shape) [+ dropout]"""
    qs, ns = [], []
    for _ in range(STEPS):
        if mask:
            qs.append(torch.randn_like(x0))
        if draw:
            nz = torch.randn(SHAPE)
            if dropout > 0:
                nz = torch.nn.functional.dropout(nz, p=dropout)
            ns.append(nz)
    return qs, ns


@pytest.mark.parametrize("cap", [1, 3, STEPS])
@pytest.mark.parametrize("mask,eta,dropout", [(True, False, 0.0), (False, True, 0.0), (True, True, 0.0), (True, True, 0.25),
                                              (False, True, 0.25)])
def test_predraw_reproduces_the_per_step_sequence(mask, eta, dropout, cap):
    x0 = torch.randn(SHAPE[0], SHAPE[2], SHAPE[1], generator=torch.Generator().manual_seed(2)).transpose(1, 2)   # not contiguous
    torch.manual_seed(9)
    qs, ns = per_step_sequence(mask, eta, dropout, x0)
    after_ref = torch.randn(4)
    torch.manual_seed(9)
    q_tab = torch.full((cap,) + SHAPE, float("nan")) if mask else None
    n_tab = torch.full((cap,) + SHAPE, float("nan")) if eta else None
    got_q, got_n = [], []
    k = 0
    while k < STEPS:                                   # one table fill per mugd_sample_staged call
        n = min(cap, STEPS - k)
        draw_step_noise(n, SHAPE, x0, q_tab, eta, n_tab, dropout, "cpu")
        got_q += [q_tab[i].clone() for i in range(n)] if mask else []
        got_n += [n_tab[i].clone() for i in range(n)] if eta else []
        k += n
    assert torch.equal(torch.randn(4), after_ref)
    assert len(got_q) == len(qs) and all(torch.equal(a, b) for a, b in zip(got_q, qs))
    assert len(got_n) == len(ns) and all(torch.equal(a, b) for a, b in zip(got_n, ns))
    if dropout > 0:
        assert any((t == 0).any() for t in got_n)


@pytest.mark.parametrize("dropout", [0.0, 0.25])
def test_predraw_that_discards_consumes_the_generator_like_the_per_step_loop(dropout):
    """match_reference_rng at eta = 0: the draws happen, nothing is kept"""
    torch.manual_seed(4)
    per_step_sequence(False, True, dropout, None)
    want = torch.randn(4)
    torch.manual_seed(4)
    draw_step_noise(STEPS, SHAPE, None, None, True, None, dropout, "cpu")
    assert torch.equal(torch.randn(4), want)


CPU = torch.device("cpu")
CUDA = torch.device("cuda:0")
B, Cz, L = SHAPE


@pytest.mark.parametrize("case,kw,dev,want", [
    ("no mask", dict(), CPU, True),
    ("no mask, x0 ignored", dict(x0=torch.zeros(3)), CPU, True),
    ("full mask", dict(mask=torch.ones(B, Cz, L), x0=torch.zeros(B, Cz, L)), CPU, True),
    ("[1,1,L] mask", dict(mask=torch.ones(1, 1, L), x0=torch.zeros(B, Cz, L)), CPU, True),
    ("[B,1,L] mask", dict(mask=torch.ones(B, 1, L), x0=torch.zeros(B, Cz, L)), CPU, True),
    ("[L] mask", dict(mask=torch.ones(L), x0=torch.zeros(B, Cz, L)), CPU, True),
    ("callback", dict(callback=lambda i: None), CPU, False),
    ("img_callback", dict(img_callback=lambda x, i: None), CPU, False),
    ("callback with mask", dict(callback=lambda i: None, mask=torch.ones(B, Cz, L), x0=torch.zeros(B, Cz, L)), CPU, False),
    ("float64 mask", dict(mask=torch.ones(B, Cz, L, dtype=torch.float64), x0=torch.zeros(B, Cz, L)), CPU, False),
    ("bool mask", dict(mask=torch.ones(B, Cz, L, dtype=torch.bool), x0=torch.zeros(B, Cz, L)), CPU, False),
    ("float16 x0", dict(mask=torch.ones(B, Cz, L), x0=torch.zeros(B, Cz, L, dtype=torch.float16)), CPU, False),
    ("CPU mask", dict(mask=torch.ones(B, Cz, L), x0=torch.zeros(B, Cz, L)), CUDA, False),
    ("mask without x0", dict(mask=torch.ones(B, Cz, L)), CPU, False),
    ("mask as a list", dict(mask=[1.0], x0=torch.zeros(B, Cz, L)), CPU, False),
    ("x0 of the wrong shape", dict(mask=torch.ones(B, Cz, L), x0=torch.zeros(1, Cz, L)), CPU, False),
    ("x0 [B,1,L]", dict(mask=torch.ones(B, Cz, L), x0=torch.zeros(B, 1, L)), CPU, False),
    ("mask broadcasting wider", dict(mask=torch.ones(3, B, Cz, L), x0=torch.zeros(B, Cz, L)), CPU, False),
    ("mask that does not broadcast", dict(mask=torch.ones(B, Cz, L + 1), x0=torch.zeros(B, Cz, L)), CPU, False),
])
def test_routing(case, kw, dev, want):
    assert takes_device_loop(SHAPE, dev, **kw) is want, case

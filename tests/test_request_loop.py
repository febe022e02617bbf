"""The samplers' host request loop without a GPU: every ``*_sampling`` method runs against a recording stand-in for the engine, the
session and its plan, and must issue exactly the C calls and step-noise draws of a plain restatement of the loop's rules.  Device
loop: the request is cut into stretches that end at each logged step (``(total - i - 1) % log_every_t == 0`` or i = 0), a stretch
into calls of at most ``per_call`` steps where the sampler stages tables; one intermediate is recorded after each stretch.  Per-step
loop (with a callback): one ``Session.eval`` per step (two at PLMS step 0), the sampler's update, the callbacks, and an intermediate
at every logged step."""
import threading
import types

import numpy as np
import pytest
import torch

from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import sampler as sampler_mod
from mug_diffusion_b200.engine import OpList
from mug_diffusion_b200.sampler import DDIMSampler, DDPMSampler, DPMSolverSampler, PLMSSampler, register_schedule

B, CZ, LZ = 2, 16, 8
SHAPE = (B, CZ, LZ)
STEP_BYTES = 4 * B * CZ * LZ
PLAN_LAUNCHES = 100
SMALL_CAP = 3                                                                   # steps per call under the small STAGE_TABLE_BYTES


class _Recorder:
    """stands in for the engine, the session and its plan of one request: keeps the step counter the calls advance and records
    every call in ``trace``"""
    launches = PLAN_LAUNCHES

    def __init__(self):
        self.at, self.trace, self.q_rows = 0, [], []
        self.lock = threading.RLock()
        self.plan = self
        self.step = torch.zeros(1, dtype=torch.int32)
        self.xin = types.SimpleNamespace(ptr=0, r=lambda a, b: None)
        self.lib = types.SimpleNamespace(mugd_plms_combine=lambda d, i, heun, st: self._c("plms_combine", i, heun),
                                         mugd_ddpm_update=lambda d, st: self._c("ddpm_update"),
                                         mugd_dpm_update=lambda d, st: self._c("dpm_update"))

    def _c(self, *what):
        self.trace.append(what)
        return 0

    # ---- the plan's C entry points
    def _device(self, entry, first, n):
        assert first == self.at and n >= 1
        self.trace.append((entry, first, n))
        self.at += n

    def launch(self, steps=1, tail=None, stage=None):
        assert tail is not None
        if stage is not None and stage.q_coef:
            self.q_rows.append(stage.q_coef)
        self._device("sample" if stage is None else "staged", self.at, steps)

    def launch_plms(self, p, first, n):
        self._device("plms", first, n)

    def launch_ddpm(self, d, first, n):
        self._device("ddpm", first, n)

    def launch_dpm(self, d, first, n):
        self._device("dpm", first, n)

    # ---- the session
    def read_rows(self, view, b, c, l):
        return torch.full((b, c, l), float(self.at))

    def rows_to_ncl(self, view, b, c, l):
        return torch.full((b, c, l), self.at + 0.5)

    def ncl_to_rows(self, t, view):
        self.trace.append(("noise_rows",))

    def eval(self, graph=True):
        self.trace.append(("eval", self.at))

    def run_ops(self, ops):
        kinds = tuple(op.kind for op in ops.ops)
        self.trace.append(("ops",) + kinds)
        self.at += kinds.count(L_.OP_STEP_ADVANCE)

    def load_x(self, x, dup):
        self.trace.append(("load_x",))

    def set_step(self, v):
        self.trace.append(("set_step", v))
        self.at = v

    def ddim_tail(self, *a):
        tail = OpList()
        tail.add(L_.OP_DDIM_UPDATE, L_.DdimUpdate())
        tail.add(L_.OP_STEP_ADVANCE, L_.StepAdvance())
        return tail

    def ddim_stage(self, *a):
        return L_.Stage()

    def plms(self, *a):
        return L_.Plms()

    def ddpm(self, *a):
        return L_.Ddpm()

    def dpm(self, *a):
        return L_.Dpm()


class _Bar:
    """a tqdm_class that records the step counter at every advance"""

    def __init__(self, it, desc, total, ticks, rec):
        self.it, self.ticks, self.rec = it, ticks, rec
        assert total == len(it)

    def __iter__(self):
        for v in self.it:
            self.ticks.append(self.rec.at)
            yield v


def _ddim_s(total):
    """the make_schedule S of a ``total``-step request (S = 30 would give 31 steps)"""
    return {1: 1, 2: 2, 10: 10, 25: 25}[total]


def _run(monkeypatch, kind, total, log_every_t, cap=None, mask=False, eta=0.0, match=False, callback=False):
    """one request of ``kind`` through its *_sampling method on a recorder; returns (recorder, z, intermediates, ticks, sampler)"""
    rec = _Recorder()
    if cap is not None:
        monkeypatch.setattr(sampler_mod, "STAGE_TABLE_BYTES", cap * STEP_BYTES + 5)

    def draw(steps, shape, x0, q_table, draw_noise, noise_table, noise_dropout, device):
        assert tuple(shape) == SHAPE and steps >= 1
        for t in (q_table, noise_table):
            assert t is None or t.shape[0] >= steps
        rec.trace.append(("draw", steps, q_table is not None, bool(draw_noise), noise_table is not None))

    monkeypatch.setattr(sampler_mod, "draw_step_noise", draw)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: types.SimpleNamespace(cuda_stream=0))
    sch = register_schedule()
    T = total if kind == "ddpm" else 1000
    model = types.SimpleNamespace(engine=rec, z_channels=CZ, z_length=LZ, num_timesteps=T, clip_denoised=True,
                                  ddpm_coef_table=lambda: torch.zeros(T, 5), q_sample=lambda x0, t: x0, **sch)
    cls = dict(ddim=DDIMSampler, plms=PLMSSampler, ddpm=DDPMSampler, dpm=DPMSolverSampler)[kind]
    s = object.__new__(cls)
    s.model, s.ddpm_num_timesteps, s.device, s.last_launches_per_step = model, T, "cpu", 0
    x = torch.zeros(SHAPE)

    def load_request(w, c, shape, x_T, scale, uc, ts=None):
        return x, False, rec, np.flip(ts)

    def load_session(w, c, shape, x_T, scale, uc, time_range):
        return x, False, rec, time_range

    if kind in ("ddim", "plms"):
        monkeypatch.setattr(s, "_load_request", load_request)
    else:
        monkeypatch.setattr(s, "_load_session", load_session)
    ticks = []
    kw = dict(tqdm_class=lambda it, desc, total: _Bar(it, desc, total, ticks, rec), log_every_t=log_every_t)
    if callback:
        kw["callback"] = lambda i: rec.trace.append(("callback", i))
        kw["img_callback"] = lambda pred, i: rec.trace.append(("img", i, float(pred.flatten()[0])))
    if kind in ("ddim", "plms"):
        s.make_schedule(_ddim_s(total), ddim_eta=eta, verbose=False)
        assert s.ddim_timesteps.shape[0] == total
        if mask:
            kw.update(mask=torch.ones(1, 1, LZ), x0=torch.zeros(SHAPE))
        run = s.ddim_sampling if kind == "ddim" else s.plms_sampling
        z, inter = run([], None, SHAPE, match_reference_rng=match, **kw)
    elif kind == "ddpm":
        z, inter = s.ddpm_sampling([], None, SHAPE, **kw)
    else:
        sched = types.SimpleNamespace(S=total, model_times=np.linspace(1.0, 0.001, total),
                                      rows_f32=lambda: np.zeros((total, 8), np.float32))
        z, inter = s.dpm_sampling([], None, SHAPE, sched, **kw)
    return rec, z, inter, ticks, s


# ---- the restatement ------------------------------------------------------------------------------------------------------------
def _logged(i, total, log_every_t):
    return (total - i - 1) % log_every_t == 0 or i == 0


def _stretches(total, log_every_t):
    """(first, n) of every stretch: each ends at a logged step"""
    out, first = [], 0
    for j in range(total):
        if _logged(j, total, log_every_t):
            out.append((first, j - first + 1))
            first = j + 1
    return out


def _calls(first, n, per_call):
    return [(k, min(per_call, first + n - k)) for k in range(first, first + n, per_call)]


def _per_call(cap):
    return 1 << 40 if cap is None else cap


def _check_intermediates(inter, z, ends):
    """x_T first, then x / pred read at each step counter in ``ends``; the result is x at the end"""
    assert [float(t.flatten()[0]) for t in inter["x_inter"]] == [0.0] + [float(e) for e in ends]
    assert [float(t.flatten()[0]) for t in inter["pred_x0"]] == [0.0] + [e + 0.5 for e in ends]
    assert float(z.flatten()[0]) == float(ends[-1]) and len(inter["x_inter"]) == len(inter["pred_x0"])


TOTALS = [1, 2, 10, 25]
LOGS = [1, 7, 100]
CAPS = [None, SMALL_CAP]


# ---- the device loop ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mask,eta,match", [(False, 0.0, False), (True, 0.0, False), (False, 1.0, False), (False, 0.0, True),
                                            (True, 1.0, True)])
@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("log_every_t", LOGS)
@pytest.mark.parametrize("total", TOTALS)
def test_ddim_device_loop(monkeypatch, total, log_every_t, cap, mask, eta, match):
    rec, z, inter, ticks, s = _run(monkeypatch, "ddim", total, log_every_t, cap, mask=mask, eta=eta, match=match)
    staged, draws = mask or eta > 0, mask or eta > 0 or match
    want = []
    for first, n in _stretches(total, log_every_t):
        for k, m in _calls(first, n, _per_call(cap)):                  # DDIM splits its calls even when nothing is staged
            if draws:
                want.append(("draw", m, mask, eta > 0 or match, eta > 0))
            want.append(("staged" if staged else "sample", k, m))
    assert rec.trace == want
    firsts = [c[1] for c in want if c[0] == "staged"]
    assert [q - rec.q_rows[0] for q in rec.q_rows] == ([8 * k for k in firsts] if mask else [])     # q_coef row k of call k
    ends = [f + n for f, n in _stretches(total, log_every_t)]
    _check_intermediates(inter, z, ends)
    assert ticks == [e for f, n in _stretches(total, log_every_t) for e in [f + n] * n]
    assert s.last_launches_per_step == PLAN_LAUNCHES + (3 if staged else 2)


@pytest.mark.parametrize("match", [False, True])
@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("log_every_t", LOGS)
@pytest.mark.parametrize("total", TOTALS)
def test_plms_device_loop(monkeypatch, total, log_every_t, cap, match):
    rec, z, inter, ticks, s = _run(monkeypatch, "plms", total, log_every_t, cap, match=match)
    want = []
    for first, n in _stretches(total, log_every_t):                        # no split: PLMS stages no tables
        if match:
            want.append(("draw", n + (first == 0), False, True, False))    # step 0 draws twice
        want.append(("plms", first, n))
    assert rec.trace == want
    _check_intermediates(inter, z, [f + n for f, n in _stretches(total, log_every_t)])
    assert len(ticks) == total
    assert s.last_launches_per_step == PLAN_LAUNCHES + 3


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("log_every_t", LOGS)
@pytest.mark.parametrize("total", TOTALS)
def test_ddpm_device_loop(monkeypatch, total, log_every_t, cap):
    rec, z, inter, ticks, s = _run(monkeypatch, "ddpm", total, log_every_t, cap)
    want = []
    for first, n in _stretches(total, log_every_t):
        for k, m in _calls(first, n, _per_call(cap)):
            want += [("draw", m, False, True, True), ("ddpm", k, m)]
    assert rec.trace == want
    _check_intermediates(inter, z, [f + n for f, n in _stretches(total, log_every_t)])
    assert len(ticks) == total
    assert s.last_launches_per_step == PLAN_LAUNCHES + 2


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("log_every_t", LOGS)
@pytest.mark.parametrize("total", TOTALS)
def test_dpm_device_loop(monkeypatch, total, log_every_t, cap):
    rec, z, inter, ticks, s = _run(monkeypatch, "dpm", total, log_every_t, cap)
    assert rec.trace == [("dpm", first, n) for first, n in _stretches(total, log_every_t)]    # no split: no tables staged
    _check_intermediates(inter, z, [f + n for f, n in _stretches(total, log_every_t)])
    assert len(ticks) == total
    assert s.last_launches_per_step == PLAN_LAUNCHES + 2


# ---- the per-step loop ----------------------------------------------------------------------------------------------------------
def _step_trace(kind, i, total, mask, eta, match):
    """the calls of step i of the per-step loop, before its callbacks"""
    upd, adv = L_.OP_DDIM_UPDATE, L_.OP_STEP_ADVANCE
    pre = [("load_x",)] if mask else []
    if kind == "ddim":
        return pre + ([("noise_rows",)] if eta > 0 else []) + [("eval", i), ("ops", upd, adv)]
    if kind == "plms":
        draw = [("draw", 1, False, True, False)] if match else []
        out = pre + [("eval", i), ("plms_combine", i, 0)]
        if i == 0:                                                              # improved Euler: a second evaluation at t_next
            out += draw + [("ops", upd), ("set_step", 1 if total > 1 else 0), ("eval", 1 if total > 1 else 0), ("load_x",),
                           ("plms_combine", 0, 1), ("set_step", 0)]
        return out + draw + [("ops", upd, adv)]
    if kind == "ddpm":
        return [("eval", i), ("draw", 1, False, True, True), ("ddpm_update",), ("ops", adv)]
    return [("eval", i), ("dpm_update",), ("ops", adv)]


@pytest.mark.parametrize("kind,mask,eta,match", [("ddim", False, 0.0, False), ("ddim", True, 1.0, True), ("plms", False, 0.0, False),
                                                 ("plms", True, 0.0, True), ("ddpm", False, 0.0, False), ("dpm", False, 0.0, False)])
@pytest.mark.parametrize("log_every_t", [1, 7])
@pytest.mark.parametrize("total", [1, 2, 10])
def test_per_step_loop(monkeypatch, kind, total, log_every_t, mask, eta, match):
    rec, z, inter, ticks, s = _run(monkeypatch, kind, total, log_every_t, SMALL_CAP, mask=mask, eta=eta, match=match, callback=True)
    want = []
    for i in range(total):
        want += _step_trace(kind, i, total, mask, eta, match) + [("callback", i), ("img", i, i + 1.5)]
    assert rec.trace == want
    _check_intermediates(inter, z, [i + 1 for i in range(total) if _logged(i, total, log_every_t)])
    assert ticks == list(range(total))
    assert s.last_launches_per_step == PLAN_LAUNCHES + (3 if kind == "plms" else 2)

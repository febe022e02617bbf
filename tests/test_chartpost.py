"""Chart clean-up on the GPU (DESIGN §6b N4): the snap and mini-jack kernels, ``model.model.remove_mini_jacks`` and
``model.model.postprocess_charts``, against the host functions of postprocess.py.

CPU: the numpy snap oracle and the array-form mini-jack oracle of tests/chartpost_oracle.py equal snap_lines and
remove_intractable_mania_mini_jacks on the golden, sweep and edge charts, on random (t, bpm, offset) triples and on random charts;
chartpost.Lines re-emits untouched lines as given and rebuilds the host functions' lines; argument validation of both entry points.
GPU: the kernels against the oracles bit for bit, and the public calls against the host functions.
"""
import ctypes as C
import gzip
import json
import os
import sys

import numpy as np
import pytest

import chartpost_oracle as orc
import grid_oracle
from mug_diffusion_b200 import chartpost as cp
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import postprocess as pp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from make_postprocess_goldens import chart  # noqa: E402
from test_gridify import CHARTS  # noqa: E402  (golden, sweep and edge charts, as gridify sees them)

GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "postprocess.json")))
with gzip.open(os.path.join(ROOT, "tests", "golden", "postprocess_random.json.gz"), "rt") as _f:
    GOLD_RANDOM = json.load(_f)
INTERVALS = (0, 60, 90, 120.5, 200)


def _line(x, t, end=None):
    return f"{x},192,{t},128,0,{end}:0:0:0:0:" if end is not None else f"{x},192,{t},1,0,0:0:0:0:"


# ---- inputs ----------------------------------------------------------------------------------------------------------------
def snap_triples(seed=5, n_charts=2200, per_chart=50):
    """[(times, bpm, offset)]: 110,000 triples in charts of 50 times sharing (bpm, offset); half with np.float32 offsets.  Random
    grids with bpm 30 .. 1,000 and negative t - offset, plus dyadic bpm (power-of-two steps) with times at exact half ties of pos
    and at |pos - k| exactly 10 / step"""
    rng = np.random.default_rng(seed)
    out = []
    for c in range(n_charts):
        f32 = c % 2 == 1
        kind = c % 5
        if kind < 3:
            bpm = np.float64(rng.uniform(150, 300) if kind == 0 else rng.uniform(30, 1000))
            off = rng.uniform(-5000, 5000)
            step = 60000 / bpm / rng.choice([1, 2, 4, 3, 6, 8, 16, 32])
            k = rng.integers(-200, 4000, per_chart)
            t = np.round(off + k * step + rng.normal(0, rng.uniform(0, 12), per_chart)).astype(np.int64)
            t[:5] = rng.integers(-2_000_000, 2_000_000, 5)
        else:
            bpm = np.float64(rng.choice([117.1875, 234.375, 468.75, 937.5, 150.0, 300.0, 75.0]))
            off = float(rng.integers(-4000, 4000)) + rng.choice([0.0, 0.125, 0.5, 0.75, 0.03125])
            div = rng.choice(orc.DIVS)
            step = 60000 / (bpm * div)
            k = rng.integers(-100, 3000, per_chart)
            frac = 0.5 if kind == 3 else 10 / step
            sign = rng.choice([-1.0, 1.0], per_chart)
            t = np.round(off + (k + sign * frac) * step).astype(np.int64)
        out.append((t, bpm, np.float32(off) if f32 else np.float64(off)))
    return out


def _host_snap(times, bpm, off):
    return np.array([int(l.split(",")[2]) for l in pp.snap_lines([_line(64, v) for v in times], bpm, off)], np.int64)


def random_jack_chart(rng, n=None):
    """hit objects with mini-jacks: rice or long-note mixes, jack_ratio 0 .. 0.5, chords, duplicate times, float times, x values
    outside [0, 512) (negative columns and columns past 3), and a list that is not always sorted by time"""
    n = int(rng.integers(0, 260)) if n is None else n
    bpm = rng.uniform(120, 320)
    step = 60000 / bpm / rng.choice([2, 4, 8])
    ln_ratio = 0.0 if rng.random() < 0.4 else rng.uniform(0.05, 0.5)
    jack_ratio = rng.uniform(0, 0.5)
    wide = rng.random() < 0.3
    t = int(rng.integers(-500, 3000))
    rows = []
    while len(rows) < n:
        t += int(step * rng.integers(1, 4))
        cols = rng.choice(4, rng.choice([1, 1, 1, 2, 3]), replace=False)
        for c in cols:
            x = int((c + 0.5) * 128) if not wide or rng.random() < 0.6 else int(rng.integers(-700, 1200))
            xs = str(x) if rng.random() < 0.9 else f"{x}.0"
            ts = str(t) if rng.random() < 0.95 else f"{t}.5"
            if rng.random() < ln_ratio:
                rows.append(f"{xs},192,{ts},128,0,{t + int(step * rng.integers(1, 9))}:0:0:0:0:")
            else:
                rows.append(f"{xs},192,{ts},1,0,0:0:0:0:")
        if rng.random() < jack_ratio:
            c = int(rng.choice(cols))
            tj = t + int(rng.integers(0, 95))
            rows.append(_line(int((c + 0.5) * 128), tj))
    rows = rows[:n]
    if rng.random() < 0.3 and n > 2:                                  # not sorted by time
        for _ in range(max(1, n // 20)):
            a = int(rng.integers(0, n - 1))
            rows[a], rows[a + 1] = rows[a + 1], rows[a]
    return rows


def jack_cases():
    """(name, lines, jack_interval): the golden passes and 320 random charts"""
    cases = []
    for g in GOLD:
        cases.append((f"gold{g['case']['seed']}", chart(**g["case"]), 90))
        cases.append((f"gold{g['case']['seed']}_after_grid", g["grid"], 60))
    for r in GOLD_RANDOM:
        s = r["seed"]
        cases.append((f"random{s}", chart(seed=s, bpm=150 + 13.7 * s % 140, offset=300 + s, n=150, div=4 if s % 2 else 8,
                                         jack_ratio=0.15), 90))
    # the earlier note of a column-6 jack moves to dst = 5 - 6 = -1, which near() reads as "any column" and which writes x = -64
    # (column 0); its walk forward stops at the note listed after it but timed outside the radius
    cases.append(("dst_minus_1", [_line(832, 1000), _line(64, 1150), _line(832, 1090), _line(192, 1100)], 90))
    rng = np.random.default_rng(31)
    for i in range(320):
        cases.append((f"rand{i}", random_jack_chart(rng), INTERVALS[i % len(INTERVALS)]))
    return cases


JACK_CASES = jack_cases()


def _oracle_lines(lines, jack_interval, stats=None):
    L = cp.Lines([lines])
    state, x = orc.mini_jacks(L.start_ms(), L.end_ms(), L.is_long, L.x(), jack_interval, stats)
    return L.format(state=state, x=x)[0]


# ---- CPU -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def timing():
    """gridify's (bpm, offset) of every chart of tests/test_gridify.py"""
    return {name: pp.gridify(lines, verbose=False)[1:] for name, lines in CHARTS.items()}


def _other_type(off):
    return np.float64(off) if isinstance(off, np.float32) else np.float32(off)


def test_snap_oracle_equals_snap_lines_on_charts(timing):
    for name, lines in CHARTS.items():
        bpm, off = timing[name]
        L = cp.Lines([lines])
        times, _, pos = L.snap_times()
        for o in (off, _other_type(off)):
            got = L.format(snapped=orc.snap(times, bpm, o), pos=pos)[0]
            assert got == pp.snap_lines(lines, bpm, o), (name, type(o))


def test_snap_oracle_equals_snap_lines_on_random_triples():
    triples = snap_triples()
    assert sum(len(t) for t, _, _ in triples) >= 100_000
    ties = edges = f32_matters = negative = 0
    for t, bpm, off in triples:
        ref = _host_snap(t, bpm, off)
        got = orc.snap(t, bpm, off)
        assert np.array_equal(got, ref), (bpm, off, t[got != ref], got[got != ref], ref[got != ref])
        if isinstance(off, np.float32):
            f32_matters += int(np.sum(orc.snap(t, bpm, np.float64(off)) != ref))
        negative += int(np.sum(t < off))
        for div in orc.DIVS:
            step = 60000 / (bpm * div)
            pos = (t.astype(np.float64) - np.float64(off)) / step
            ties += int(np.sum(np.abs(pos - np.floor(pos)) == 0.5))
            edges += int(np.sum(np.abs(pos - np.rint(pos)) == 10 / step))
    assert ties > 1000 and edges > 1000 and f32_matters > 0 and negative > 1000, (ties, edges, f32_matters, negative)


def test_mini_jack_oracle_equals_host():
    stats = {}
    for name, lines, jack in JACK_CASES:
        ref = pp.remove_intractable_mania_mini_jacks(lines, verbose=False, jack_interval=jack)
        assert _oracle_lines(lines, jack, stats) == ref, name
    for g in GOLD:                                                     # and the reference's own outputs
        assert _oracle_lines(chart(**g["case"]), 90) == g["dejack"]
        assert _oracle_lines(g["grid"], 60) == g["dejack_after_grid"]
    # every branch of the loop is taken, moves to a negative column (dst = -1) included
    for key in ("ignored", "moved", "moved_earlier", "dropped", "dropped_earlier", "dst-1"):
        assert stats.get(key, 0) > 0, (key, stats)


def test_lines_round_trip():
    for name, lines, _ in JACK_CASES[:40]:
        L = cp.Lines([lines, [], lines[:3]])
        assert L.format() == [list(lines), [], list(lines[:3])], name
        assert L.format(state=np.ones(len(L.lines), np.uint8), x=L.x()) == [list(lines), [], list(lines[:3])], name


def test_lines_parse_like_the_host():
    lines = ["64.5,192,1000.5,1,0,0:0:0:0:", "-200,192,1200,128,0,1500:0:0:0:0:", "700,192,900,1,0,0:0:0:0:"]
    L = cp.Lines([lines])
    assert list(L.start_ms()) == [1000.5, 1200.0, 900.0] and list(L.end_ms()) == [0.0, 1500.0, 0.0]
    assert list(L.x()) == [64, -200, 700] and list(L.is_long) == [0, 1, 0]
    assert [orc.column(v) for v in L.x()] == [0, -1, 5] == [int(int(float(l.split(",")[0])) / 128) for l in lines]


def test_snap_times_must_fit_int32():
    with pytest.raises(ValueError, match="int32"):
        cp.Lines([[_line(64, 1 << 31)]]).snap_times()
    with pytest.raises(ValueError, match="int32"):
        cp.Lines([[_line(64, 0, -(1 << 31) - 1)]]).snap_times()
    times, start, pos = cp.Lines([[_line(64, (1 << 31) - 1)], [_line(64, 5, 9), _line(64, -(1 << 31))]]).snap_times()
    assert list(times) == [(1 << 31) - 1, 5, 9, -(1 << 31)] and list(start) == [0, 1, 4] and list(pos) == [0, 1, 3]


def test_host_checks_before_any_device_work():
    post = cp.ChartPost(engine=None)                                   # no device is touched before these checks
    with pytest.raises(ValueError, match="x="):
        post.mini_jacks(np.array([0, 1]), np.zeros(1), np.zeros(1), np.zeros(1, np.uint8), np.array([1 << 30]), 90)
    with pytest.raises(ValueError, match="jack_interval"):
        post.mini_jacks(np.array([0, 1]), np.zeros(1), np.zeros(1), np.zeros(1, np.uint8), np.array([64]), float("nan"))
    with pytest.raises(TypeError, match="offset"):
        post.snap(np.array([1], np.int32), np.array([0, 1]), [np.float64(200)], [np.float16(3)])
    with pytest.raises(TypeError, match="bpm"):
        post.snap(np.array([1], np.int32), np.array([0, 1]), [np.float32(200)], [np.float64(3)])


class _OraclePost:
    """ChartPost with the oracles in place of the kernels"""

    def snap(self, times, chart_start, bpm, offset):
        return np.concatenate([np.zeros(0, np.int64)] + [orc.snap(times[chart_start[c]:chart_start[c + 1]], bpm[c], offset[c])
                                                         for c in range(len(chart_start) - 1)])

    def mini_jacks(self, chart_start, start, end, is_long, x, jack_interval):
        out = [orc.mini_jacks(*(a[chart_start[c]:chart_start[c + 1]] for a in (start, end, is_long, x)), jack_interval)
               for c in range(len(chart_start) - 1)]
        return np.concatenate([s for s, _ in out]), np.concatenate([v for _, v in out])


class _OracleScanner:
    def search(self, times_list):
        return pp.search_timing(times_list, grid_oracle.scan_states(times_list, pp.CANDIDATES))


def _custom_gridify(lines, auto_snap, jack):
    """webui.py:401-407"""
    new, bpm, off = pp.gridify(lines, verbose=False)
    if auto_snap:
        lines = new
    return bpm, off, pp.remove_intractable_mania_mini_jacks(lines, verbose=False, jack_interval=jack)


def _same(got, ref):
    return (got[2] == ref[2] and type(got[0]) is type(ref[0]) and got[0] == ref[0] and type(got[1]) is type(ref[1])
            and got[1] == ref[1])


def test_postprocess_composition_with_oracle_kernels():
    """chartpost.postprocess_charts and chartpost.gridify driven by the oracles equal the host composition"""
    dst_minus_1 = next(lines for name, lines, _ in JACK_CASES if name == "dst_minus_1")
    charts = [CHARTS[n] for n in ("golden4", "random12", "one_note", "chord", "two_notes")] + [chart(**GOLD[0]["case"]), dst_minus_1]
    for auto_snap in (True, False):
        for jack in (60, 90):
            got = cp.postprocess_charts(_OracleScanner(), _OraclePost(), charts, auto_snap, jack)
            for i, c in enumerate(charts):
                assert _same(got[i], _custom_gridify(c, auto_snap, jack)), (i, auto_snap, jack)
    for c, (lines, bpm, off) in zip(charts, cp.gridify(_OracleScanner(), _OraclePost(), charts)):
        ref = pp.gridify(c, verbose=False)
        assert lines == ref[0] and _same((bpm, off, lines), (ref[1], ref[2], ref[0]))
    assert cp.remove_mini_jacks(_OraclePost(), charts + [[]], 90) == [
        pp.remove_intractable_mania_mini_jacks(c, verbose=False) for c in charts] + [[]]


# ---- argument validation of the entry points (host side, no device needed) -----------------------------------------------
def _arr(ct, v, size):
    if v is None:
        return None
    return (ct * size)(*(list(v) + [0] * size)[:size])


def _snap_call(lib, **kw):
    a = dict(h=None, times=1 << 20, chart_start=[0, 3, 7], n_charts=2, bpm=[200.0, 187.3], offset=[10.0, 0.5], f32=[0, 1],
             out=1 << 24)
    a.update(kw)
    m = max(a["n_charts"], 1)
    return lib.mugd_chart_snap(a["h"], a["times"], _arr(C.c_int32, a["chart_start"], m + 1), a["n_charts"],
                               _arr(C.c_double, a["bpm"], m), _arr(C.c_double, a["offset"], m), _arr(C.c_int32, a["f32"], m),
                               a["out"], None)


def _jack_call(lib, **kw):
    a = dict(h=None, chart_start=[0, 3, 7], n_charts=2, jack=90.0, start=1 << 20, end=1 << 21, is_long=1 << 22, x=1 << 23,
             state=1 << 24, workspace=1 << 25)
    a.update(kw)
    m = max(a["n_charts"], 1)
    return lib.mugd_remove_mini_jacks(a["h"], _arr(C.c_int32, a["chart_start"], m + 1), a["n_charts"], a["jack"], a["start"],
                                      a["end"], a["is_long"], a["x"], a["state"], a["workspace"], None)


def _expect_invalid(lib, rc, msg, what):
    assert rc == 1, rc                                                # MUGD_ERR_INVALID
    assert msg in lib.mugd_last_error().decode(), lib.mugd_last_error().decode()
    with pytest.raises(L_.MugdError):
        L_.check(rc, what)


@pytest.mark.parametrize("bad,msg", [
    (dict(times=None), "NULL"), (dict(chart_start=None), "NULL"), (dict(bpm=None), "NULL"), (dict(offset=None), "NULL"),
    (dict(f32=None), "NULL"), (dict(out=None), "NULL"), (dict(n_charts=0), "n_charts"), (dict(n_charts=-3), "n_charts"),
    (dict(chart_start=[1, 3, 7]), "chart_start[0]"), (dict(chart_start=[0, 5, 4]), "decreases at chart 1"),
    (dict(chart_start=[0, -1, 4]), "decreases at chart 0"), (dict(bpm=[0.0, 200.0]), "bpm"), (dict(bpm=[200.0, -1.0]), "bpm"),
    (dict(bpm=[float("nan"), 1.0]), "bpm"), (dict(bpm=[2e9, 1.0]), "bpm"), (dict(offset=[float("inf"), 0.5]), "offset"),
    (dict(offset=[2.0 ** 53, 0.5]), "offset"), (dict(offset=[10.0, 0.1]), "not a float32 value"), (dict(f32=[2, 1]), "offset_is_f32"),
    (dict(times=(1 << 20) + 2), "alignment"), (dict(out=(1 << 24) + 4), "alignment"), (dict(), "null handle"),
], ids=lambda v: None if isinstance(v, dict) else v.replace(" ", "_"))
def test_chart_snap_argument_validation(bad, msg):
    lib = L_.load()
    _expect_invalid(lib, _snap_call(lib, **bad), msg, "mugd_chart_snap")


@pytest.mark.parametrize("bad,msg", [
    (dict(start=None), "NULL"), (dict(end=None), "NULL"), (dict(is_long=None), "NULL"), (dict(x=None), "NULL"),
    (dict(state=None), "NULL"), (dict(workspace=None), "NULL"), (dict(chart_start=None), "NULL"), (dict(n_charts=0), "n_charts"),
    (dict(n_charts=-1), "n_charts"), (dict(chart_start=[2, 3, 7]), "chart_start[0]"), (dict(chart_start=[0, 3, 1]), "decreases at chart 1"),
    (dict(chart_start=[0, -2, 1]), "decreases at chart 0"), (dict(jack=float("nan")), "NaN"), (dict(start=(1 << 20) + 4), "alignment"),
    (dict(x=(1 << 23) + 2), "alignment"), (dict(), "null handle"),
], ids=lambda v: None if isinstance(v, dict) else v.replace(" ", "_"))
def test_remove_mini_jacks_argument_validation(bad, msg):
    lib = L_.load()
    _expect_invalid(lib, _jack_call(lib, **bad), msg, "mugd_remove_mini_jacks")


# ---- GPU -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model():
    from mug_diffusion_b200 import synth
    from mug_diffusion_b200.sampler import MugDiffusionB200
    return MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(96), z_length=96)


@pytest.mark.gpu
def test_gpu_snap_kernel_vs_oracle(model, timing):
    post = model.chart_post
    triples = snap_triples()
    for name, lines in CHARTS.items():
        bpm, off = timing[name]
        times, _, _ = cp.Lines([lines]).snap_times()
        triples += [(times, bpm, off), (times, bpm, _other_type(off))]
    for b in range(0, len(triples), 700):                              # several launches of 128 charts per call
        batch = triples[b:b + 700]
        start = np.zeros(len(batch) + 1, np.int32)
        start[1:] = np.cumsum([len(t) for t, _, _ in batch])
        got = post.snap(np.concatenate([t for t, _, _ in batch]).astype(np.int32), start, [p[1] for p in batch],
                        [p[2] for p in batch])
        assert got.dtype == np.int64
        for c, (t, bpm, off) in enumerate(batch):
            ref = orc.snap(t, bpm, off)
            assert np.array_equal(got[start[c]:start[c + 1]], ref), (b + c, bpm, off)


def _rice_chart(seed, n):
    """a rice chart (no long notes) with jack_ratio 0.3"""
    return chart(seed=seed, bpm=200.0, offset=300, n=n, div=4, jitter=2.0, ln_ratio=0.0, jack_ratio=0.3)


def _big_chart():
    """31,744 notes (4 x 8 x 992, the most decode_to_hit_objects can produce), long notes and jacks"""
    lines = chart(seed=8, bpm=240.0, offset=500, n=22000, div=8, jitter=2.0, ln_ratio=0.15, jack_ratio=0.3)
    assert len(lines) >= 31744
    return lines[:31744]


@pytest.mark.gpu
def test_gpu_remove_mini_jacks_equals_host(model):
    rice = _rice_chart(41, 5050)
    assert 9000 < len(rice) < 10500, len(rice)
    big = _big_chart()
    for jack in INTERVALS:
        cases = [lines for _, lines, j in JACK_CASES if j == jack]
        if jack == 90:
            cases += [rice, big]
        ref = [pp.remove_intractable_mania_mini_jacks(c, verbose=False, jack_interval=jack) for c in cases]
        got = model.model.remove_mini_jacks(cases, jack_interval=jack)
        assert got == ref, jack
        assert model.model.remove_mini_jacks(cases, jack_interval=jack) == got, jack
        if jack in (60, 90):
            for c, r in zip(cases[:60], ref):
                assert model.model.remove_mini_jacks([c], jack_interval=jack) == [r]
    for g in GOLD:
        assert model.model.remove_mini_jacks([chart(**g["case"]), g["grid"]], jack_interval=90)[0] == g["dejack"]
        assert model.model.remove_mini_jacks([g["grid"]], jack_interval=60) == [g["dejack_after_grid"]]
    assert model.model.remove_mini_jacks([[], []]) == [[], []] and model.model.remove_mini_jacks([]) == []
    assert model.model.remove_mini_jacks([[], CHARTS["golden1"], []]) == [[], pp.remove_intractable_mania_mini_jacks(
        CHARTS["golden1"], verbose=False), []]


def _decoded_chart(model):
    import torch
    torch.manual_seed(3)
    z = torch.randn(2, 16, 96, device=model.device) * 2.0
    charts = [c for c in model.model.decode_to_hit_objects(z, 23.219954648526077) if c]
    assert charts, "the synthetic latent decoded to no notes"
    return charts[0]


@pytest.mark.gpu
def test_gpu_postprocess_charts_equals_custom_gridify(model):
    names = ["golden1", "golden3", "golden4", "random11", "one_note", "chord", "two_notes", "bpm150_n60_div4_j3.0",
             "bpm450_n900_div4_j6.0"]
    dst_minus_1 = next(lines for name, lines, _ in JACK_CASES if name == "dst_minus_1")
    charts = [CHARTS[n] for n in names] + [chart(**GOLD[3]["case"]), _rice_chart(42, 600), dst_minus_1, _decoded_chart(model)]
    for auto_snap in (True, False):
        for jack in (60, 90):
            got = model.model.postprocess_charts(charts, auto_snap=auto_snap, jack_interval=jack)
            assert len(got) == len(charts)
            for i, (c, g) in enumerate(zip(charts, got)):
                assert _same(g, _custom_gridify(c, auto_snap, jack)), (i, auto_snap, jack)
            assert {type(g[1]) for g in got} == {np.float32, np.float64}
    single, = model.model.postprocess_charts([charts[0]])
    assert _same(single, model.model.postprocess_charts(charts)[0])
    with pytest.raises(ValueError, match="chart 1 is empty"):
        model.model.postprocess_charts([charts[0], []])
    assert model.model.postprocess_charts([]) == []

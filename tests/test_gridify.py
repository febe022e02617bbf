"""Chart timing as scans (SURVEY §8f N4, DESIGN §6b N4): postprocess.search_timing and the grid-scan kernel.

CPU: search_timing driven by the numpy scan of tests/grid_oracle.py equals estimate_timing exactly (value and numpy type) on the
golden charts and a generated sweep; the oracle's phase fill equals np.arange; snap_lines + search_timing reproduce gridify; and
argument validation of mugd_grid_scan.  GPU: mugd_grid_scan against the oracle scan on random states, bit for bit, and
``model.model.gridify`` against ``postprocess.gridify``.
"""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

import grid_oracle
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import postprocess as pp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from make_postprocess_goldens import CASES, chart  # noqa: E402

GOLD_RANDOM_SEEDS = [11, 12, 13]                # tests/test_postprocess.py's live-reference cases


def _random_case(seed):
    return dict(seed=seed, bpm=150 + 13.7 * seed % 140, offset=300 + seed, n=150, div=4 if seed % 2 else 8, jack_ratio=0.15)


def golden_charts():
    """the golden cases after dejack, as gridify sees them"""
    out = {}
    for c in CASES:
        out[f"golden{c['seed']}"] = pp.remove_intractable_mania_mini_jacks(chart(**c), verbose=False)
    for s in GOLD_RANDOM_SEEDS:
        out[f"random{s}"] = pp.remove_intractable_mania_mini_jacks(chart(**_random_case(s)), verbose=False)
    return out


SWEEP_BPMS = [95, 131, 150, 187.3, 240, 299, 310, 450]
SWEEP_DIVS = [1, 3, 4, 6, 8]


def sweep_charts(sizes=(1, 7, 60, 400, 1200, 2500, 2600, 900)):
    """one chart per bpm: note counts 1 .. 4,000, divisions 1/3/4/6/8, jitter 0 .. 6 ms, long notes"""
    out = {}
    for i, (bpm, n) in enumerate(zip(SWEEP_BPMS, sizes)):
        div = SWEEP_DIVS[i % len(SWEEP_DIVS)]
        jitter = [0.0, 1.5, 3.0, 6.0][i % 4]
        out[f"bpm{bpm}_n{n}_div{div}_j{jitter}"] = chart(seed=100 + i, bpm=bpm, offset=137 + 211 * i, n=n, div=div, jitter=jitter,
                                                          ln_ratio=0.2, jack_ratio=0.0)
    return out


def edge_charts():
    """a 1-note chart and a chord-only chart (no refit succeeds: offset stays float32) and a 2-note chart"""
    return {"one_note": ["64,192,1234,1,0,0:0:0:0:"],
            "chord": [f"{x},192,5000,1,0,0:0:0:0:" for x in (64, 192, 320, 448)],
            "two_notes": ["64,192,1000,1,0,0:0:0:0:", "192,192,1321,128,0,1500:0:0:0:0:"]}


CHARTS = {**golden_charts(), **sweep_charts(), **edge_charts()}


@pytest.fixture(scope="module")
def cpu_results():
    """postprocess.gridify(verbose=False) of every chart (the referee), computed once"""
    return {name: pp.gridify(lines, verbose=False) for name, lines in CHARTS.items()}


def _same_scalar(a, b):
    return type(a) is type(b) and (a == b or (np.isnan(a) and np.isnan(b)))


# ---- CPU -----------------------------------------------------------------------------------------------------------------
def test_search_timing_with_oracle_scan_equals_estimate_timing(cpu_results):
    names = list(CHARTS)
    times = [pp.note_times(CHARTS[n]) for n in names]
    got = pp.search_timing(times, grid_oracle.scan_states(times, pp.CANDIDATES))
    for name, (bpm, off) in zip(names, got):
        _, bpm_ref, off_ref = cpu_results[name]
        assert _same_scalar(bpm, bpm_ref), (name, bpm, bpm_ref)
        assert _same_scalar(off, off_ref), (name, off, off_ref)


def test_offset_stays_float32_without_a_refit(cpu_results):
    for name in ("one_note", "chord"):
        _, bpm, off = cpu_results[name]
        assert type(off) is np.float32 and type(bpm) is np.float64, (name, type(bpm), type(off))
    assert type(cpu_results["two_notes"][2]) is np.float64


def test_golden_timing_matches_reference_values():
    gold = {g["case"]["seed"]: g for g in json.load(open(os.path.join(ROOT, "tests", "golden", "postprocess.json")))}
    for c in CASES:
        times = pp.note_times(gold[c["seed"]]["dejack"])
        (bpm, off), = pp.search_timing([times], grid_oracle.scan_states([times], pp.CANDIDATES))
        assert float(bpm) == gold[c["seed"]]["bpm"] and float(off) == gold[c["seed"]]["offset"]


def test_snap_lines_and_search_timing_reproduce_gridify(cpu_results):
    names = list(CHARTS)
    times = [pp.note_times(CHARTS[n]) for n in names]
    got = pp.search_timing(times, grid_oracle.scan_states(times, pp.CANDIDATES))
    for name, (bpm, off) in zip(names, got):
        assert pp.snap_lines(CHARTS[name], bpm, off) == cpu_results[name][0], name


def test_phase_fill_equals_np_arange():
    rng = np.random.default_rng(7)
    offsets = [np.float32(0.0), np.float32(412.0), np.float32(-37.25), np.float32(123456.78)]
    offsets += [np.float32(v) for v in rng.uniform(-2000, 400000, 6)]
    offsets += [np.float64(v) for v in rng.uniform(-2000, 400000, 8)] + [np.float64(1033.3333333333333), np.float64(-0.1)]
    lengths = set()
    for off in offsets:
        for c in pp.CANDIDATES:
            ref = pp.phase_list(off, c)
            got = grid_oracle.phase_fill(off, c)
            assert ref.dtype == np.float64 and np.array_equal(ref.view(np.int64), got.view(np.int64)), (off, c)
            lengths.add(len(ref))
    assert lengths == {4, 5}


def test_candidate_table():
    assert len(pp.CANDIDATES) == 1500 and pp.CANDIDATES.dtype == np.float64
    assert np.array_equal(pp.CANDIDATES, np.arange(150, 300, 0.1))


# ---- argument validation of mugd_grid_scan (host side, no device needed) -------------------------------------------------
def _call(lib, **kw):
    n = kw.get("n_charts", 2)
    a = dict(h=None, times=1 << 20, chart_start=[0, 3, 7], n_charts=2, cands=1 << 21, n_cands=1500, k0=[0, 10], head_len=[0, 5],
             best_off=[0.0, 100.0], best_score=[-1.0, 0.5], first=[0.0, 1.0], head_bpm=[0.0, 200.0], head_off=[0.0] * 10,
             workspace=1 << 22, out_i=1 << 23, out_d=1 << 24)
    a.update(kw)
    m = max(n, 1)

    def arr(ct, v, size):
        if v is None:
            return None
        return (ct * size)(*(list(v) + [0] * size)[:size])

    return lib.mugd_grid_scan(a["h"], a["times"], arr(C.c_int32, a["chart_start"], m + 1), a["n_charts"], a["cands"], a["n_cands"],
                              arr(C.c_int32, a["k0"], m), arr(C.c_int32, a["head_len"], m), arr(C.c_double, a["best_off"], m),
                              arr(C.c_double, a["best_score"], m), arr(C.c_float, a["first"], m), arr(C.c_double, a["head_bpm"], m),
                              arr(C.c_double, a["head_off"], 5 * m), a["workspace"], a["out_i"], a["out_d"], None)


@pytest.mark.parametrize("bad,msg", [
    (dict(times=None), "NULL"), (dict(cands=None), "NULL"), (dict(chart_start=None), "NULL"), (dict(k0=None), "NULL"),
    (dict(head_off=None), "NULL"), (dict(workspace=None), "NULL"), (dict(out_i=None), "NULL"), (dict(out_d=None), "NULL"),
    (dict(n_charts=0), "n_charts"), (dict(n_cands=0), "n_cands"), (dict(chart_start=[0, 3, 3]), "chart 1 is empty"),
    (dict(chart_start=[0, 0, 7]), "chart 0 is empty"), (dict(chart_start=[0, 5, 4]), "chart 1 is empty"),
    (dict(chart_start=[2, 3, 7]), "chart_start[0]"), (dict(head_len=[0, 6]), "head_len"), (dict(head_len=[-1, 0]), "head_len"),
    (dict(k0=[0, 1501]), "k0"), (dict(k0=[-1, 0]), "k0"), (dict(best_off=[float("nan"), 0.0]), "best_off"),
    (dict(head_bpm=[0.0, 0.0]), "head_bpm"), (dict(cands=(1 << 21) + 4), "alignment"), (dict(out_d=(1 << 24) + 4), "alignment"),
    (dict(workspace=(1 << 22) + 4), "alignment"), (dict(), "null handle"),
], ids=lambda v: None if isinstance(v, dict) else v.replace(" ", "_"))
def test_grid_scan_argument_validation(bad, msg):
    """every check runs on the host before the launch: no device is needed to see them fail"""
    lib = L_.load()
    rc = _call(lib, **bad)
    assert rc == 1, rc                                            # MUGD_ERR_INVALID
    assert msg in lib.mugd_last_error().decode(), lib.mugd_last_error().decode()
    with pytest.raises(L_.MugdError):
        L_.check(rc, "mugd_grid_scan")


# ---- GPU -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model():
    from mug_diffusion_b200 import synth
    from mug_diffusion_b200.sampler import MugDiffusionB200
    return MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(96), z_length=96)


def _random_times(rng, n):
    """n note times: a jittered grid of a random bpm and division with chords, float32, sorted"""
    bpm = rng.uniform(90, 460)
    step = 60000 / bpm / rng.choice([1, 2, 3, 4, 6, 8])
    slots = np.sort(rng.integers(0, 3 * n + 1, n))
    t = rng.uniform(-50, 3000) + slots * step + rng.normal(0, rng.uniform(0, 6), n)
    return np.round(t).astype(np.float32) if rng.random() < 0.7 else t.astype(np.float32)


def _random_state(rng, times, cands):
    first = times[0]
    k0 = int(rng.integers(0, len(cands) + 1)) if rng.random() < 0.8 else int(rng.integers(len(cands) - 20, len(cands) + 1))
    best_off = first if rng.random() < 0.3 else np.float64(first + rng.uniform(-400, 400))
    n_head = int(rng.integers(0, pp.MAX_PHASES + 1))
    head_bpm = np.float64(rng.uniform(150, 300))
    base = pp.phase_list(np.float64(first + rng.uniform(-300, 300)), head_bpm)
    head_off = np.concatenate([base, base[-1:] - 60000 / head_bpm / 4])[-n_head:] if n_head else np.zeros(0)
    u = rng.random()
    best_score = np.float64(-1.0) if u < 0.15 else np.float64(rng.uniform(0, 1.1) * len(times) / 150)
    state = pp.ScanState(first, k0, best_off, best_score, head_bpm, head_off)
    if u > 0.8:                                     # exactly the score of the first improving trial: the comparison is strict
        hit = grid_oracle.scan(times, cands, first, k0, best_off, best_score, head_bpm, head_off)
        if hit is not None:
            state.best_score = hit.score
    return state


def _bits(x):
    return np.float64(x).view(np.int64)


@pytest.mark.gpu
def test_gpu_grid_scan_vs_oracle(model):
    from mug_diffusion_b200.gridscan import GridScanner
    rng = np.random.default_rng(2026)
    cands = pp.CANDIDATES
    scanner = GridScanner(model.engine)
    n_checked, n_hits, kinds = 0, 0, set()
    for batch in range(8):
        sizes = [int(np.exp(rng.uniform(0, np.log(8000)))) for _ in range(32)]
        sizes[0], sizes[1] = 1, 8000
        times = [_random_times(rng, n) for n in sizes]
        scanner.load(times)
        for rep in range(2):
            states = [_random_state(rng, t, cands) for t in times]
            got = scanner.scan(states)
            for t, s, g in zip(times, states, got):
                ref = grid_oracle.scan(t, cands, s.first, s.k0, s.best_off, s.best_score, s.head_bpm, s.head_off)
                n_checked += 1
                if ref is None:
                    assert g is None, (len(t), s, g)
                    continue
                n_hits += 1
                kinds.add(ref.kind)
                assert g is not None, (len(t), s, ref)
                assert (g.pos, g.kind, g.n_on) == (ref.pos, ref.kind, ref.n_on), (len(t), s, g, ref)
                assert _bits(g.bpm) == _bits(ref.bpm) and _bits(g.offset) == _bits(ref.offset) and _bits(g.score) == _bits(ref.score)
    assert n_checked == 512 and n_hits > 100 and kinds == {pp.HEAD, pp.CANDIDATE, pp.PHASE}, (n_hits, kinds)


def _long_chart():
    """5.3 minutes at 187.3 bpm on a 1/16 grid: about 8,500 notes"""
    return chart(seed=77, bpm=187.3, offset=523, n=5300, div=16, jitter=2.0, ln_ratio=0.15, jack_ratio=0.0)


@pytest.mark.gpu
def test_gpu_gridify_equals_cpu(model, cpu_results):
    long_lines = _long_chart()
    assert 7000 < len(long_lines) < 9000 and int(long_lines[-1].split(",")[2]) > 5 * 60 * 1000
    refs = dict(cpu_results)
    refs["long"] = pp.gridify(long_lines, verbose=False)
    charts = {**CHARTS, "long": long_lines}
    names = list(charts)
    batch = model.model.gridify([charts[n] for n in names])
    assert len(batch) == len(names)
    for name, got in zip(names, batch):
        lines, bpm, off = got
        ref_lines, ref_bpm, ref_off = refs[name]
        assert lines == ref_lines, name
        assert _same_scalar(bpm, ref_bpm) and _same_scalar(off, ref_off), (name, bpm, ref_bpm, off, ref_off)
        single, = model.model.gridify([charts[name]])
        assert single[0] == lines and _same_scalar(single[1], bpm) and _same_scalar(single[2], off), name


@pytest.mark.gpu
def test_gpu_gridify_empty_chart(model):
    with pytest.raises(ValueError, match="chart 1 is empty"):
        model.model.gridify([CHARTS["golden1"], [], CHARTS["golden2"]])
    assert model.model.gridify([]) == []

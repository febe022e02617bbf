"""mug_diffusion_b200/postprocess.py (SURVEY §8f N4: gridify + mini-jack removal) against golden vectors produced by the UNMODIFIED
reference (tools/make_postprocess_goldens.py -> tests/golden/postprocess.json, tools/make_live_goldens.py ->
tests/golden/postprocess_random.json.gz).
String / integer results: the bar is equality."""
import gzip
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from make_postprocess_goldens import chart  # noqa: E402
from mug_diffusion_b200 import postprocess as pp  # noqa: E402

GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "postprocess.json")))


@pytest.mark.parametrize("g", GOLD, ids=[f"seed{g['case']['seed']}" for g in GOLD])
def test_dejack_gridify_dejack_equal_reference_golden(g):
    lines = chart(**g["case"])
    assert len(lines) == g["n_in"]
    dejack = pp.remove_intractable_mania_mini_jacks(lines, verbose=False)
    assert dejack == g["dejack"]
    grid, bpm, off = pp.gridify(dejack, verbose=False)
    assert grid == g["grid"]
    assert float(bpm) == g["bpm"] and float(off) == g["offset"]
    assert pp.remove_intractable_mania_mini_jacks(grid, verbose=False, jack_interval=60) == g["dejack_after_grid"]


def test_long_notes_are_never_moved_and_snapped_at_both_ends():
    lines = ["64,192,1000,128,0,1480:0:0:0:0:", "64,192,1060,1,0,0:0:0:0:", "192,192,1120,1,0,0:0:0:0:", "320,192,1240,1,0,0:0:0:0:"]
    out = pp.remove_intractable_mania_mini_jacks(lines, verbose=False)
    assert out[0] == lines[0] and len(out) == 4 and out[1].split(",")[0] != "64"      # the short note left the held column
    grid, bpm, off = pp.gridify(lines, verbose=False)
    assert len(grid) == 4 and all(l.split(",")[3] == o.split(",")[3] for l, o in zip(grid, lines))


RANDOM_SEEDS = [11, 12, 13]


def random_chart_case(seed):
    return dict(seed=seed, bpm=150 + 13.7 * seed % 140, offset=300 + seed, n=150, div=4 if seed % 2 else 8, jack_ratio=0.15)


@pytest.mark.parametrize("seed", RANDOM_SEEDS)
def test_live_reference(seed):
    with gzip.open(os.path.join(ROOT, "tests", "golden", "postprocess_random.json.gz"), "rt") as f:
        ref = {c["seed"]: c for c in json.load(f)}[seed]
    lines = chart(**random_chart_case(seed))
    b = pp.remove_intractable_mania_mini_jacks(lines, verbose=False)
    assert b == ref["dejack"]
    gb, bpm_b, off_b = pp.gridify(b, verbose=False)
    assert gb == ref["grid"] and float(bpm_b) == ref["bpm"] and float(off_b) == ref["offset"]

"""Inputs of the chart-encoder goldens (tests/golden/encoder_L96_B2.npz, tests/golden/objects_to_array.json.gz).  Only the reference's
outputs are stored; the inputs are listed here or regenerated from seeds, so tools/make_goldens.py and the tests share them."""
import json
import os

import numpy as np

from mug_diffusion_b200 import synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

ENCODER_L, ENCODER_B = 96, 2
ENCODER_SEED = 0                 # synth.synthetic_encoder_state_dict
SAMPLE_SEED = 4321               # torch.manual_seed before DiagonalGaussianDistribution.sample()


def golden_charts() -> dict:
    """tests/golden/hit_objects.json: the reference's .osu lines of the golden decoder outputs, and their frame_ms"""
    return json.load(open(os.path.join(GOLD, "hit_objects.json")))


def dense_notes(frames: int, seed: int = 5) -> np.ndarray:
    """a dense uniform [16, frames] note array in [0, 1): every channel of every frame non-zero"""
    return synth._rng(seed, "dense_notes").random(size=(16, frames), dtype=np.float32)


def encoder_chart_lines() -> list:
    """the real chart of the encoder golden: the first ddim_L96_B2_S10_cfg5 chart"""
    return golden_charts()["ddim_L96_B2_S10_cfg5"][0]


# objects_to_array cases: (name, lines, key_count, frame_ms, max_frame, rate, offset_ms).  The golden charts are added by
# objects_cases(); these hand cases hit the corners of convertor.py:266-320.
FRAME_MS = 512 / 4 / 22050 * 8 * 1000           # webui.py:341-342
_HAND = [
    ("start_past_array", ["64,192,100,1,0,0:0:0:0:", "192,192,35000,1,0,0:0:0:0:", "320,192,35700,1,0,0:0:0:0:",
                          "448,192,34000,128,0,90000:0:0:0:0:"], 4, FRAME_MS, 768, 1.0, 0.0),
    ("ln_end_past_array", ["64,192,1000,128,0,99999:0:0:0:0:", "192,192,35600,128,0,35700:0:0:0:0:"], 4, FRAME_MS, 768, 1.0, 0.0),
    ("x_out_of_range", ["512,192,100,1,0,0:0:0:0:", "-10,192,200,1,0,0:0:0:0:", "-200,192,300,1,0,0:0:0:0:",
                        "511,192,400,1,0,0:0:0:0:", "600,192,500,128,0,900:0:0:0:0:"], 4, FRAME_MS, 768, 1.0, 0.0),
    ("rate_1_5", ["64,192,100,1,0,0:0:0:0:", "192,192,5000,128,0,9000:0:0:0:0:", "320,192,20000,1,0,0:0:0:0:",
                  "448,192,30000,128,0,34000:0:0:0:0:"], 4, FRAME_MS, 768, 1.5, 0.0),
    ("offset_ms", ["64,192,0,1,0,0:0:0:0:", "192,192,1000,128,0,2000:0:0:0:0:", "448,192,35650,1,0,0:0:0:0:"], 4, FRAME_MS, 768, 1.0, 37.5),
    ("negative_offset_ms", ["64,192,10,1,0,0:0:0:0:", "192,192,500,128,0,800:0:0:0:0:"], 4, FRAME_MS, 768, 1.0, -30.0),
    ("fractional_times", ["64,192,1234.7,1,0,0:0:0:0:", "192,192,99.99,128,0,1500.9:0:0:0:0:", "320,192,46.44,1,0,0:0:0:0:"],
     4, FRAME_MS, 768, 1.0, 0.0),
    ("ln_overlapped_by_later_start", ["64,192,100,128,0,1000:0:0:0:0:", "64,192,500,1,0,0:0:0:0:", "64,192,700,128,0,1200:0:0:0:0:"],
     4, FRAME_MS, 768, 1.0, 0.0),
    ("seven_keys", ["36,192,100,1,0,0:0:0:0:", "475,192,200,128,0,800:0:0:0:0:", "256,192,300,1,0,0:0:0:0:"], 7, 40.0, 256, 1.0, 0.0),
]


def objects_cases() -> list:
    """every objects_to_array case as dicts (name, lines, key_count, frame_ms, max_frame, rate, offset_ms)"""
    keys = ("name", "lines", "key_count", "frame_ms", "max_frame", "rate", "offset_ms")
    g = golden_charts()
    cases = []
    for src, max_frame in (("ddim_L512_B1_S50_cfg5", 4096), ("ddim_L96_B2_S10_cfg5", 768), ("synthetic", 768)):
        for i, lines in enumerate(g[src]):
            cases.append(dict(zip(keys, (f"{src}.{i}", lines, 4, g["frame_ms"], max_frame, 1.0, 0.0))))
    cases += [dict(zip(keys, c)) for c in _HAND]
    return cases

"""Store what the unmodified reference returns for the randomised cases of tests/test_prompt.py and tests/test_postprocess.py
(tests/golden/prompt_random.json.gz, tests/golden/postprocess_random.json.gz), so those comparisons run without the reference tree.

    MUG_REFERENCE_ROOT=<reference checkout> python tools/make_live_goldens.py
"""
import gzip
import importlib.util
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import ref_shim
    from make_postprocess_goldens import chart
    from test_postprocess import RANDOM_SEEDS, random_chart_case
    from test_prompt import SPEC_COUNT, random_dicts

    gold_dir = os.path.join(ROOT, "tests", "golden")
    ref_shim.install_shims()
    sys.path.insert(0, ref_shim.REF_ROOT)
    from mug.util import count_beatmap_features, feature_dict_to_embedding_ids

    spec0 = json.load(open(os.path.join(gold_dir, "prompt.json")))["spec"]
    out = []
    for spec in (spec0, SPEC_COUNT):
        out.append(dict(count=count_beatmap_features(spec), ids=[feature_dict_to_embedding_ids(d, spec) for d in random_dicts(spec)]))
    with gzip.open(os.path.join(gold_dir, "prompt_random.json.gz"), "wt") as f:
        json.dump(out, f, separators=(",", ":"))

    spec = importlib.util.spec_from_file_location("ref_utils", os.path.join(ref_shim.REF_ROOT, "mug", "data", "utils.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    cases = []
    for seed in RANDOM_SEEDS:
        lines = chart(**random_chart_case(seed))
        a = ref.remove_intractable_mania_mini_jacks(lines, verbose=False)
        ga, bpm, off = ref.gridify(a, verbose=False)
        cases.append(dict(seed=seed, dejack=a, grid=ga, bpm=float(bpm), offset=float(off)))
    with gzip.open(os.path.join(gold_dir, "postprocess_random.json.gz"), "wt") as f:
        json.dump(cases, f, separators=(",", ":"))


if __name__ == "__main__":
    main()

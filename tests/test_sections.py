"""Section prompts without a GPU (DESIGN §6b N20): the request checks, the sectioned plan against today's, and the C layout of
mugd_attention_sec."""
import ctypes as C
import hashlib
import os
import subprocess

import pytest
import torch

from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import packer, synth
from mug_diffusion_b200.config import ModelConfig
from mug_diffusion_b200.engine import Arena, UNetCompiler, View
from mug_diffusion_b200.sampler import section_prompts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STARTS = 1 << 38                     # fake device address of a [levels, Beff, 8] start table


# ---- the request checks ------------------------------------------------------------------------------------------------------------
def _c(B=2, T=21):
    return torch.randn(B, 128, T)


def test_no_sections_or_all_empty_is_todays_request():
    c = _c()
    assert section_prompts(None, c, 2, 96) is None
    assert section_prompts([[], ()], c, 2, 96) is None
    got = section_prompts([[(8, c[1]), (64, c[0])], []], c, 2, 96)
    assert [[s for s, _ in ch] for ch in got] == [[8, 64], []]


@pytest.mark.parametrize("sections,msg", [
    ([[]], "2 charts, got 1"),
    ("x", "one list"),
    ([[(8, None)], []], r"sections\[0\]: the context at 8"),
    ([[], [(12, "c")]], r"sections\[1\]: start 12 must be a multiple of 8"),
    ([[], [(True, "c")]], r"sections\[1\]: start True"),
    ([[], [(0, "c")]], r"sections\[1\]: start 0 must lie in \(0, 96\)"),
    ([[], [(96, "c")]], r"sections\[1\]: start 96 must lie"),
    ([[(16, "c"), (8, "c")], []], r"sections\[0\]: starts must be strictly increasing"),
    ([[(16, "c"), (16, "c")], []], r"sections\[0\]: starts must be strictly increasing"),
    ([[(8 * i, "c") for i in range(1, 9)], []], r"sections\[0\]: 8 changes; a chart has at most 7"),
    ([[(8, "short")], []], r"sections\[0\]: the context at 8 must be a \[128, 21\] tensor"),
    ([[(8, "nan")], []], r"sections\[0\]: the context at 8 holds a non-finite value"),
    ([[], (8, "c")], r"sections\[1\]: every entry must be a \(start, context\) pair"),
])
def test_malformed_sections_are_refused(sections, msg):
    c = _c()
    fill = {"c": c[0], "short": torch.zeros(128, 20), "nan": torch.full((128, 21), float("nan"))}

    def sub(v):
        if isinstance(v, (list, tuple)) and len(v) == 2 and isinstance(v[1], str):
            return (v[0], fill[v[1]])
        return [sub(x) for x in v] if isinstance(v, list) else v

    with pytest.raises(ValueError, match=msg):
        section_prompts(sub(sections), c, 2, 96)


def test_a_ragged_request_bounds_starts_by_each_charts_length():
    c = _c()
    assert section_prompts([[(24, c[0])], [(88, c[1])]], c, 2, 96, lens=[32, 96]) is not None
    with pytest.raises(ValueError, match=r"sections\[0\]: start 32 must lie in \(0, 32\)"):
        section_prompts([[(32, c[0])], []], c, 2, 96, lens=[32, 96])


class _NoDevice:
    """a stand-in engine: any session request means GPU work began"""

    def __getattr__(self, name):
        raise AssertionError(f"engine.{name} used before the request was checked")


def test_forward_refuses_before_any_gpu_work():
    from mug_diffusion_b200 import sampler as S
    m = object.__new__(S.MugDiffusionB200)
    m.engine = _NoDevice()
    c = _c()
    w = [torch.zeros(2, 4, 96 >> l) for l in range(4)]
    with pytest.raises(ValueError, match="multiple of 8"):
        S._Wrapper(m).forward(torch.zeros(2, 16, 96), torch.zeros(2), c, w, sections=[[(12, c[0])], []])


# ---- the plan --------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def comp():
    cfg = ModelConfig()
    b = packer.pack_model(synth.synthetic_state_dict(96), cfg.unet, cfg.decoder)
    return cfg, UNetCompiler(cfg.unet, b, 1 << 30)


def _ext(comp, Beff, Lz, n_sec):
    blocks = list(comp.lay.blocks())
    ctx_kv = [View((1 << 41) + i * (1 << 26), 2 * b.cin, Beff * n_sec * 21, 2 * b.cin)
              for i, b in enumerate(x for x in blocks if x.kind == "attn")]
    s4 = {b.prefix: View((1 << 42) + i * (1 << 24), b.cin, Lz // b.ds, b.cin) for i, b in enumerate(x for x in blocks if x.kind == "s4")}
    return dict(emb_table=1 << 40, step=(1 << 40) + 4096, ctx_tokens=21, ctx_kv=ctx_kv, s4_kt=s4)


@pytest.mark.parametrize("Beff,Lz", [(1, 96), (4, 96), (2, 512), (8, 512), (2, 2048)])
def test_sectioned_plan_changes_only_the_cross_attentions(comp, Beff, Lz):
    cfg, cp = comp
    plain = cp.compile(Arena(1 << 32), Beff, Lz, _ext(cp, Beff, Lz, 1), False)["ops"].ops
    sec = cp.compile(Arena(1 << 32), Beff, Lz, _ext(cp, Beff, Lz, L_.SECTIONS), False, sections=STARTS)["ops"].ops
    assert len(plain) == len(sec)
    n_sec = n_self = 0
    for a, b in zip(plain, sec):
        if b.kind == L_.OP_ATTENTION_SEC:
            assert a.kind == L_.OP_ATTENTION and a.u.attn.Lk == 21
            d = b.u.attns
            x = a.u.attn
            assert bytes(d.attn) == bytes(x)                                     # same q / k / v / o / tables / shape
            lvl = {Lz >> l: l for l in range(cfg.unet.levels)}[x.Lq]
            assert d.starts == STARTS + 4 * lvl * Beff * L_.SECTIONS and d.sec_stride == 21
            n_sec += 1
        else:
            assert bytes(a) == bytes(b)
            n_self += a.kind == L_.OP_ATTENTION
    assert n_sec == 16 and n_self == 16


def test_sections_none_is_todays_op_list(comp):
    """sections=None compiles today's op list byte for byte (whose hashes tests/test_ragged.py pins)"""
    cfg, cp = comp
    for Beff, Lz in ((2, 96), (8, 512)):
        ext = _ext(cp, Beff, Lz, 1)
        a = cp.compile(Arena(1 << 32), Beff, Lz, ext, False)["ops"].array()
        b = cp.compile(Arena(1 << 32), Beff, Lz, ext, False, None, None, sections=None)["ops"].array()
        assert hashlib.sha256(bytes(a)).hexdigest() == hashlib.sha256(bytes(b)).hexdigest()


# ---- C ABI -------------------------------------------------------------------------------------------------------------------------
def test_abi_attention_sec_layout(tmp_path):
    assert L_.ABI_VERSION == 13 and C.sizeof(L_.Op) == 256 and L_.OP_ATTENTION_SEC == 19
    t = L_.AttentionSec
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mugd.h"\nint main(void) {\n'
                   '  printf("%zu %d %d %zu", sizeof(mugd_op), MUGD_OP_ATTENTION_SEC, MUGD_SECTIONS, sizeof(mugd_attention_sec));\n'
                   + "".join(f'  printf(" %zu", offsetof(mugd_attention_sec, {f}));\n' for f, _ in t._fields_)
                   + '  printf(" %zu\\n", offsetof(mugd_op, u.attns));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-o", str(exe), str(src), "-I" + os.path.join(ROOT, "include")], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [256, 19, L_.SECTIONS, C.sizeof(t)] + [getattr(t, f).offset for f, _ in t._fields_] + [L_.Op.u.offset]


@pytest.mark.parametrize("n", [17, 18, 19, 20])
def test_abi_sizes_fills_entry_17_only_from_18(n):
    lib = L_.load()
    sizes = (C.c_int32 * 20)(*([-1] * 20))
    assert lib.mugd_abi_sizes(sizes, n) == 0
    assert sizes[16] == C.sizeof(L_.CfgScales)
    assert sizes[17] == (C.sizeof(L_.AttentionSec) if n >= 18 else -1)
    assert list(sizes[18:]) == [-1, -1]


# ---- the oracle's section rule and the reference goldens ---------------------------------------------------------------------------
def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _oracle_case():
    import section_cases as sc
    inp = synth.synthetic_inputs(sc.B, sc.L)
    sd = synth.synthetic_state_dict(sc.L)
    return sc, inp, sd


def _cfg_eval(orc, sd, sc, inp):
    return orc.unet_forward(sd, torch.cat([inp["x_T"]] * 2), torch.tensor(sc.T_EVAL * 2), torch.cat([inp["uc"], inp["c"]]),
                            [torch.cat([w, w]) for w in inp["w"]])


def test_oracle_rule_with_every_section_at_c_is_the_plain_oracle():
    from oracle import mug_oracle as orc
    from section_oracle import oracle_sections
    sc, inp, sd = _oracle_case()
    with torch.no_grad():
        plain = _cfg_eval(orc, sd, sc, inp)
        same = [[(32, inp["c"][0]), (64, inp["c"][0])], [(8, inp["c"][1])]]
        with oracle_sections({2 * sc.B: [[]] * sc.B + same}, sc.L):
            got = _cfg_eval(orc, sd, sc, inp)
    assert torch.equal(got, plain)


def test_oracle_rule_equals_the_reference_goldens(golden_dir):
    import golden_cases as gc
    from oracle import mug_oracle as orc
    from section_oracle import oracle_sections
    sc, inp, sd = _oracle_case()
    lay = sc.layouts()
    ge = gc.load_golden(os.path.join(golden_dir, sc.EVAL_NAME + ".npz"))["eps"]
    gd = gc.load_golden(os.path.join(golden_dir, sc.DDIM_NAME + ".npz"))
    with torch.no_grad():
        plain = _cfg_eval(orc, sd, sc, inp)
        with oracle_sections({2 * sc.B: [[]] * sc.B + lay}, sc.L):
            eps = _cfg_eval(orc, sd, sc, inp)
            z = orc.ddim_sample(sd, sc.S, inp["c"], inp["w"], inp["x_T"], scale=sc.SCALE, uc=inp["uc"])
        logits = orc.decoder_forward(sd, z)
    assert _rel(eps, ge) < 1e-4
    assert _rel(z, gd["z"]) < 1e-3 and _rel(logits, gd["logits"]) < 1e-3
    # the sections reach the chart: the cond half moved, the uncond half (uc on every row) did not
    assert torch.equal(eps[:sc.B], plain[:sc.B]) and _rel(eps[sc.B:], plain[sc.B:]) > 1e-3


@pytest.mark.skipif(not os.path.isdir(os.environ.get("MUG_REFERENCE_ROOT", "/root/reference")),
                    reason="the reference is not installed here")
def test_section_goldens_regenerate_bit_for_bit(tmp_path, golden_dir):
    import golden_cases as gc
    import section_cases as sc
    subprocess.run([os.sys.executable, os.path.join(ROOT, "tools", "make_section_goldens.py"), str(tmp_path)], check=True,
                   capture_output=True)
    for name in (sc.EVAL_NAME, sc.DDIM_NAME):
        a, b = (gc.load_golden(os.path.join(d, name + ".npz")) for d in (golden_dir, str(tmp_path)))
        assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


def test_prompts_of_more_than_32_tokens_are_refused():
    c = _c(T=33)
    with pytest.raises(L_.MugdError, match="33 tokens; section prompts take at most 32"):
        section_prompts([[(8, c[0])], []], c, 2, 96)
    assert section_prompts([[], []], _c(T=64), 2, 96) is None            # no sections: any prompt length, today's path

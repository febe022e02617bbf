"""The section-prompt rule (DESIGN §6b N20) over oracle/mug_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A cross-attention is pointwise in its query rows: row i's output depends on its own query, on the prompt tokens' K / V and on
clamp(j - i, +-pos_max).  So a prompt per section is CrossAttention.forward (mug/model/attention.py:91-126) run once per section
slot with that slot's context over all rows, keeping the rows of the slot: exact in the reference's arithmetic.  Query row r of a
level with Lq = Lz >> l rows belongs to the section holding latent frame r << l."""
import contextlib
from typing import Dict, List, Sequence, Tuple

import torch

from oracle import mug_oracle as orc

SLOTS = 8


def section_rule(attend, x: torch.Tensor, context: torch.Tensor, layouts: Sequence[Sequence[Tuple[int, torch.Tensor]]], Lz: int):
    """``attend(x, ctx)``: one cross-attention over x [B, Lq, C] with context ctx [B, T, Cc] (tokens first, as the transformer block
    passes it); ``layouts[b]``: sample b's (start in latent frames, context [Cc, T]) pairs after its opening prompt ``context[b]``.
    Returns the output whose rows come from the pass of their own section slot."""
    out = attend(x, context)
    Bx, Lq = x.shape[0], x.shape[1]
    shift = (Lz // Lq).bit_length() - 1
    for s in range(1, SLOTS):
        users = [b for b in range(Bx) if len(layouts[b]) >= s]
        if not users:
            break
        ctx = context.clone()
        for b in users:
            ctx[b] = layouts[b][s - 1][1].t()
        o = attend(x, ctx)
        out = out.clone()
        for b in users:
            lo = layouts[b][s - 1][0] >> shift
            hi = layouts[b][s][0] >> shift if len(layouts[b]) > s else Lq
            out[b, lo:hi] = o[b, lo:hi]
    return out


@contextlib.contextmanager
def oracle_sections(by_batch: Dict[int, List], Lz: int):
    """While active, every cross-attention of oracle/mug_oracle.py over a batch of n samples with ``by_batch[n]`` present takes
    section_rule with those layouts (e.g. {2B: [[]] * B + charts} for a CFG evaluation, whose uncond half keeps uc on every row)."""
    orig = orc.cross_attention

    def patched(p, pre, x, context, heads, pos_max=64):
        lay = by_batch.get(x.shape[0]) if context is not None else None
        if not lay or all(not e for e in lay):
            return orig(p, pre, x, context, heads, pos_max)
        return section_rule(lambda xx, cc: orig(p, pre, xx, cc, heads, pos_max), x, context, lay, Lz)

    orc.cross_attention = patched
    try:
        yield
    finally:
        orc.cross_attention = orig

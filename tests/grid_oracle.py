"""One scan of the chart-timing search (postprocess.search_timing, DESIGN §6b N4) restated in numpy with every cast written out:
the referee of the grid-scan kernel and the scan that drives search_timing in the CPU tests.

A trial (bpm, off) over the float32 note times t:  step = 60000 / bpm;  d = t - off, a float32 subtraction for a candidate trial
(off = first, np.float32) and an fp64 subtraction for a phase (off is np.float64);  pos = d / step;
on = |pos - rint(pos)| < 10 / step;  score = n_on / bpm.  Phases follow numpy's arange fill (phase_fill)."""
import numpy as np

from mug_diffusion_b200.postprocess import CANDIDATE, HEAD, MAX_PHASES, PHASE, SCAN_SLOTS, ScanHit

BLOCK = 64                                      # candidates evaluated per numpy pass


def phase_fill(start, bpm) -> np.ndarray:
    """np.arange(start, start - beat, -beat / 4), beat = 60000 / bpm, by numpy's rule: length ceil((stop - start) / step),
    p0 = start, p1 = start + step, p_j = start + j * (p1 - start) for j >= 2 (not start + j * step)"""
    start, bpm = np.float64(start), np.float64(bpm)
    beat = np.float64(60000.0) / bpm
    step = -beat / np.float64(4.0)
    n = int(np.ceil(((start - beat) - start) / step))
    p1 = start + step
    delta = p1 - start
    return np.array([start, p1] + [start + np.float64(j) * delta for j in range(2, n)], np.float64)[:n]


def _n_on(d: np.ndarray, bpm: np.ndarray) -> np.ndarray:
    """d [..., N] float64 distances to the grid origin, bpm [...] -> notes on the grid per trial"""
    step = np.float64(60000.0) / bpm
    pos = d / step[..., None]
    return (np.abs(pos - np.rint(pos)) < (np.float64(10.0) / step)[..., None]).sum(-1)


def scan(times: np.ndarray, cands: np.ndarray, first, k0: int, best_off, best_score, head_bpm=0.0, head_off=()):
    """the first trial, in estimate_timing's loop order, whose score beats best_score, as a ScanHit, or None"""
    times = np.asarray(times, np.float32)
    t64 = times.astype(np.float64)
    best_score = np.float64(best_score)
    head_off = np.asarray(head_off, np.float64)
    assert len(head_off) <= MAX_PHASES
    if len(head_off):
        bpm = np.full(len(head_off), np.float64(head_bpm))
        n_on = _n_on(t64[None, :] - head_off[:, None], bpm)
        score = n_on / bpm
        hit = np.flatnonzero(score > best_score)
        if len(hit):
            j = int(hit[0])
            return ScanHit(1 + j, HEAD, bpm[j], head_off[j], int(n_on[j]), score[j])
    d_cand = (times - np.float32(first)).astype(np.float64)             # float32 subtraction, then widened
    for b0 in range(k0, len(cands), BLOCK):
        ks = np.arange(b0, min(b0 + BLOCK, len(cands)))
        bpm = cands[ks].astype(np.float64)
        phases = [phase_fill(best_off, c) for c in bpm]
        off = np.zeros((len(ks), MAX_PHASES))
        valid = np.zeros((len(ks), SCAN_SLOTS), bool)
        valid[:, 0] = True
        for i, p in enumerate(phases):
            off[i, :len(p)] = p
            valid[i, 1:1 + len(p)] = True
        n_on = np.zeros((len(ks), SCAN_SLOTS), np.int64)
        n_on[:, 0] = _n_on(np.broadcast_to(d_cand, (len(ks), len(times))), bpm)
        n_on[:, 1:] = _n_on(t64[None, None, :] - off[:, :, None], np.repeat(bpm[:, None], MAX_PHASES, 1))
        score = n_on / bpm[:, None]
        hit = np.flatnonzero((valid & (score > best_score)).ravel())
        if len(hit):
            i, slot = divmod(int(hit[0]), SCAN_SLOTS)
            pos = (ks[i] - k0 + 1) * SCAN_SLOTS + slot
            offset = np.float64(np.float32(first)) if slot == 0 else off[i, slot - 1]
            return ScanHit(int(pos), CANDIDATE if slot == 0 else PHASE, bpm[i], offset, int(n_on[i, slot]), score[i, slot])
    return None


def scan_states(times_list, cands):
    """a scan function for postprocess.search_timing over these charts"""
    def run(states):
        return [scan(t, cands, s.first, s.k0, s.best_off, s.best_score, s.head_bpm, s.head_off) for t, s in zip(times_list, states)]
    return run

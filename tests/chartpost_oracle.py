"""The chart clean-up kernels (csrc/chartpost.cu, DESIGN §6b N4) restated on the host: the referee of the kernels, itself checked
against postprocess.snap_lines and postprocess.remove_intractable_mania_mini_jacks.

snap: numpy over int times with every cast written out.  t - offset is a float32 subtraction of t rounded to float32 when the
offset is an np.float32 (NumPy 2 evaluates int - np.float32 in float32), else fp64; step = 60000 / (bpm * div), pos = d / step,
k = rint(pos); the first div with |pos - k| < 10 / step gives trunc(k * step + offset) in fp64.

mini_jacks: the kernel's algorithm over per-note arrays (start, end, is_long, x -> state, x), the notes in list order.  Columns are
x / 128 truncated toward zero; near() walks away from a note and stops at the first live note outside the radius; held_at() walks
the chart's list of long notes backwards from the note's rank in it."""
import numpy as np

DIVS = (1, 2, 4, 3, 6, 8, 16, 32)


def snap(times, bpm, offset) -> np.ndarray:
    t = np.asarray(times, np.int64)
    bpm = np.float64(bpm)
    if isinstance(offset, np.float32):
        d = (t.astype(np.float32) - offset).astype(np.float64)
    else:
        d = t.astype(np.float64) - np.float64(offset)
    off = np.float64(offset)
    out = t.copy()
    done = np.zeros(len(t), bool)
    for div in DIVS:
        step = np.float64(60000.0) / (bpm * np.float64(div))
        pos = d / step
        k = np.rint(pos)
        hit = ~done & (np.abs(pos - k) < np.float64(10.0) / step)
        out[hit] = (k[hit] * step + off).astype(np.int64)          # astype truncates toward zero, as int()
        done |= hit
    return out


def column(x: int) -> int:
    return int(x / 128)                                            # exact for |x| < 2^53, truncation toward zero


def mini_jacks(start, end, is_long, x, jack_interval, stats=None):
    """one chart: returns (state, x) with state 0 dropped / 1 kept / 2 kept and moved.  ``stats`` (a dict) counts the outcomes."""
    n = len(start)
    start = [float(v) for v in start]
    end = [float(v) for v in end]
    is_long = [bool(v) for v in is_long]
    x = [int(v) for v in x]
    state = [1] * n
    ln_idx = [k for k in range(n) if is_long[k]]
    ln_rank, r = [], 0
    for k in range(n):
        ln_rank.append(r)
        r += is_long[k]
    J = float(jack_interval)
    J2 = J * 2.0

    def count(key):
        if stats is not None:
            stats[key] = stats.get(key, 0) + 1

    def near(i, t, radius, col, back, forth, tol=False):
        found = []
        for go, rng in ((back, range(i - 1, -1, -1)), (forth, range(i + 1, n))):
            if not go:
                continue
            for k in rng:
                if state[k] == 0:
                    continue
                dt = abs(start[k] - t)
                if dt > radius:
                    break
                if (col < 0 or column(x[k]) == col) and (not tol or dt >= 10.0):
                    found.append(k)
        return found

    def held_at(before, col, t):
        for j in range(ln_rank[before] - 1, -1, -1):
            m = ln_idx[j]
            if state[m] != 0 and column(x[m]) == col and start[m] <= t:
                return end[m] >= t - 50.0
        return False

    for i in range(n):
        t, col = start[i], column(x[i])
        earlier = near(i, t, J, col, True, False)
        if not earlier:
            continue
        if not near(i, t, J2, -1, False, True, tol=True):
            count("ignored")
            continue
        e = earlier[0]
        moved = False
        for idx, when, src in ((i, t, col), (e, start[e], column(x[e]))):
            if idx == i and is_long[i]:
                continue
            targets = (1 - src, 2, 3) if src in (0, 1) else (5 - src, 1, 0)
            for dst in targets:
                if held_at(idx, dst, when):
                    continue
                if not near(idx, when, J, dst, True, True):
                    x[idx] = dst * 128 + 64
                    state[idx] = 2
                    moved = True
                    count("moved" if idx == i else "moved_earlier")
                    count(f"dst{dst}")
                    break
            if moved:
                break
        if moved:
            continue
        chord_here = len(near(i, t, 10.0, -1, True, True)) + 1
        chord_prev = len(near(e, start[e], 10.0, -1, True, True)) + 1
        if chord_here > 1 and chord_here >= chord_prev and not is_long[i]:
            victim = i
        elif chord_prev > 1 and chord_prev >= chord_here:
            victim = e
        elif is_long[i]:
            victim = e
        else:
            victim = i
        state[victim] = 0
        count("dropped_earlier" if victim == e else "dropped")
    return np.array(state, np.uint8), np.array(x, np.int64)

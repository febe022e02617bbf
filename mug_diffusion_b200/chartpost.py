"""Chart clean-up on the GPU: gridify's snapping and the mini-jack removal (SURVEY §8f N4, DESIGN §6b N4), equal to the host
functions of postprocess.py (snap_lines, remove_intractable_mania_mini_jacks), which stay the specification.

``Lines`` splits a batch of charts' hit-object lines into fields once and writes the changed fields back: field 2 and the first
sub-field of field 5 when a note is snapped, field 0 when it is moved; untouched lines are returned as given.  ``ChartPost`` runs
the two kernels (csrc/chartpost.cu): ``mugd_chart_snap``, one thread per note time, and ``mugd_remove_mini_jacks``, one warp per
chart.  ``gridify``, ``remove_mini_jacks`` and ``postprocess_charts`` compose them with the timing search of gridscan.GridScanner.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch

from . import lib as L_

X_LIMIT = 1 << 30            # |int(float(x))| below this keeps every moved x in int32 (mugd_remove_mini_jacks)
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1


class Lines:
    """the hit-object lines of a batch of charts, split once: chart c is lines chart_start[c] .. chart_start[c+1] - 1"""

    def __init__(self, charts: Sequence[Sequence[str]]):
        self.lines: List[str] = [l for lines in charts for l in lines]
        self.fields = [l.split(",") for l in self.lines]
        self.chart_start = np.zeros(len(charts) + 1, np.int32)
        self.chart_start[1:] = np.cumsum([len(lines) for lines in charts])
        self.tails: List[Optional[List[str]]] = [f[5].split(":") if int(f[3]) == 128 else None for f in self.fields]
        self.is_long = np.array([t is not None for t in self.tails], np.uint8)

    @property
    def n_charts(self) -> int:
        return len(self.chart_start) - 1

    def chart(self, a: np.ndarray, c: int) -> np.ndarray:
        return a[self.chart_start[c]:self.chart_start[c + 1]]

    def start_ms(self) -> np.ndarray:
        """float(f[2]) of every line"""
        return np.array([float(f[2]) for f in self.fields], np.float64)

    def end_ms(self) -> np.ndarray:
        """float(f[5].split(":")[0]) of every long note, 0 for the others"""
        return np.array([float(t[0]) if t is not None else 0.0 for t in self.tails], np.float64)

    def x(self) -> np.ndarray:
        """int(float(f[0])) of every line"""
        return np.array([int(float(f[0])) for f in self.fields], np.int64)

    def snap_times(self):
        """the times snap_lines snaps, int(f[2]) of every line followed by int(end) of a long note, as int32, with the chart
        boundaries of that list and each line's position in it"""
        t = []
        for f, tail in zip(self.fields, self.tails):
            t.append(int(f[2]))
            if tail is not None:
                t.append(int(tail[0]))
        times = np.array(t, np.int64)
        bad = np.flatnonzero((times < INT32_MIN) | (times > INT32_MAX))
        if len(bad):
            raise ValueError(f"note time {times[bad[0]]} does not fit in int32")
        count = 1 + self.is_long.astype(np.int64)
        pos = np.zeros(len(count) + 1, np.int64)
        pos[1:] = np.cumsum(count)
        return times.astype(np.int32), pos[self.chart_start].astype(np.int32), pos[:-1]

    def format(self, state: Optional[np.ndarray] = None, x: Optional[np.ndarray] = None, snapped: Optional[np.ndarray] = None,
               pos: Optional[np.ndarray] = None) -> List[List[str]]:
        """the lines of every chart after the clean-up: state 0 drops a line, 2 writes x into field 0; ``snapped`` (indexed by
        ``pos``, as snap_times lays it out) rewrites the times"""
        state = [1] * len(self.lines) if state is None else state.tolist()
        x = None if x is None else x.tolist()
        snapped = None if snapped is None else snapped.tolist()
        pos = None if pos is None else pos.tolist()
        bounds = self.chart_start.tolist()
        out = []
        for c in range(self.n_charts):
            rows = []
            for j in range(bounds[c], bounds[c + 1]):
                s = state[j]
                if s == 0:
                    continue
                if snapped is None and s == 1:
                    rows.append(self.lines[j])
                    continue
                f = list(self.fields[j])
                if s == 2:
                    f[0] = str(x[j])
                if snapped is not None:
                    p = pos[j]
                    f[2] = str(snapped[p])
                    tail = self.tails[j]
                    if tail is not None:
                        f[5] = ":".join([str(snapped[p + 1])] + tail[1:])
                rows.append(",".join(f))
            out.append(rows)
        return out


def _offset_is_f32(offset) -> int:
    """1 for an np.float32 offset (gridify's when no refit succeeds), 0 for an fp64 one"""
    if isinstance(offset, np.float32):
        return 1
    if isinstance(offset, (float, np.float64)):
        return 0
    raise TypeError(f"offset of type {type(offset).__name__}: gridify returns np.float32 or np.float64")


class ChartPost:
    """the clean-up kernels on one engine's device"""

    def __init__(self, engine):
        self.engine = engine
        self.kernel_ms: Optional[List[float]] = None       # set to [] to record the CUDA-event time of every launch

    def _launch(self, call, what: str):
        stream = torch.cuda.current_stream()
        if self.kernel_ms is not None:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record(stream)
        L_.check(call(stream.cuda_stream), what)
        if self.kernel_ms is not None:
            ev[1].record(stream)
            ev[1].synchronize()
            self.kernel_ms.append(ev[0].elapsed_time(ev[1]))

    def snap(self, times: np.ndarray, chart_start: np.ndarray, bpm: Sequence, offset: Sequence) -> np.ndarray:
        """snap_lines' snap(t) of every int32 time (chart c's at chart_start[c] ..) for that chart's (bpm, offset) as gridify
        returns them; int64"""
        n = len(times)
        if n == 0:
            return np.zeros(0, np.int64)
        for b in bpm:
            if not isinstance(b, (float, np.float64)):
                raise TypeError(f"bpm of type {type(b).__name__}: gridify returns np.float64")
        f32 = np.array([_offset_is_f32(o) for o in offset], np.int32)
        off = np.array(offset, np.float64)
        bpm_h = np.array(bpm, np.float64)
        chart_start = np.ascontiguousarray(chart_start, np.int32)
        dev = self.engine.device
        t = torch.from_numpy(np.ascontiguousarray(times, np.int32)).to(dev)
        out = torch.empty(n, dtype=torch.int64, device=dev)
        lib, h = self.engine.lib, self.engine.handle
        self._launch(lambda s: lib.mugd_chart_snap(h, t.data_ptr(), chart_start.ctypes.data, len(chart_start) - 1, bpm_h.ctypes.data,
                                                   off.ctypes.data, f32.ctypes.data, out.data_ptr(), s), "mugd_chart_snap")
        return out.cpu().numpy()

    def mini_jacks(self, chart_start: np.ndarray, start: np.ndarray, end: np.ndarray, is_long: np.ndarray, x: np.ndarray,
                   jack_interval) -> tuple:
        """remove_intractable_mania_mini_jacks over per-note arrays: returns (state, x), state 0 dropped / 1 kept / 2 moved"""
        n = len(start)
        if n == 0:
            return np.zeros(0, np.uint8), np.zeros(0, np.int32)
        radius = float(jack_interval)
        if radius != jack_interval or np.isnan(radius):
            raise ValueError(f"jack_interval={jack_interval!r} is not a number exactly representable as a float")
        x = np.asarray(x)
        bad = np.flatnonzero(np.abs(x.astype(np.int64)) >= X_LIMIT)
        if len(bad):
            raise ValueError(f"note {bad[0]}: x={x[bad[0]]} outside (-2^30, 2^30)")
        chart_start = np.ascontiguousarray(chart_start, np.int32)
        dev = self.engine.device
        st = torch.from_numpy(np.ascontiguousarray(start, np.float64)).to(dev)
        en = torch.from_numpy(np.ascontiguousarray(end, np.float64)).to(dev)
        ln = torch.from_numpy(np.ascontiguousarray(is_long, np.uint8)).to(dev)
        xd = torch.from_numpy(np.ascontiguousarray(x, np.int32)).to(dev)
        state = torch.empty(n, dtype=torch.uint8, device=dev)
        ws = torch.empty(2 * n, dtype=torch.int32, device=dev)
        lib, h = self.engine.lib, self.engine.handle
        self._launch(lambda s: lib.mugd_remove_mini_jacks(h, chart_start.ctypes.data, len(chart_start) - 1, radius, st.data_ptr(),
                                                          en.data_ptr(), ln.data_ptr(), xd.data_ptr(), state.data_ptr(),
                                                          ws.data_ptr(), s), "mugd_remove_mini_jacks")
        return state.cpu().numpy(), xd.cpu().numpy()


def _check_not_empty(charts):
    for i, lines in enumerate(charts):
        if len(lines) == 0:
            raise ValueError(f"chart {i} is empty: gridify needs at least one hit object")


def _timing(scanner, lines: Lines):
    start32 = lines.start_ms().astype(np.float32)                   # postprocess.note_times
    return scanner.search([lines.chart(start32, c) for c in range(lines.n_charts)])


def gridify(scanner, post: ChartPost, charts: Sequence[Sequence[str]]):
    """[postprocess.gridify(lines, verbose=False) for lines in charts]: the timing search batched over the charts, the snapping on
    the device"""
    _check_not_empty(charts)
    if not charts:
        return []
    lines = Lines(charts)
    timing = _timing(scanner, lines)
    return [(rows, bpm, off) for rows, (bpm, off) in zip(snap_charts(post, lines, timing), timing)]


def snap_charts(post: ChartPost, lines: Lines, timing) -> List[List[str]]:
    """[postprocess.snap_lines(chart, bpm, offset) ...] for every chart of ``lines`` and its (bpm, offset) in ``timing``"""
    times, t_start, pos = lines.snap_times()
    snapped = post.snap(times, t_start, [b for b, _ in timing], [o for _, o in timing])
    return lines.format(snapped=snapped, pos=pos)


def remove_mini_jacks(post: ChartPost, charts: Sequence[Sequence[str]], jack_interval=90):
    """[postprocess.remove_intractable_mania_mini_jacks(c, verbose=False, jack_interval=jack_interval) for c in charts]"""
    if not charts:
        return []
    lines = Lines(charts)
    state, x = post.mini_jacks(lines.chart_start, lines.start_ms(), lines.end_ms(), lines.is_long, lines.x(), jack_interval)
    return lines.format(state=state, x=x)


def postprocess_charts(scanner, post: ChartPost, charts: Sequence[Sequence[str]], auto_snap: bool = True, jack_interval=90):
    """webui's custom_gridify (webui.py:401-407) for every chart: [(bpm, offset, lines)], where lines are gridify's snapped lines
    if ``auto_snap`` else the input, after remove_intractable_mania_mini_jacks(..., verbose=False, jack_interval)"""
    _check_not_empty(charts)
    if not charts:
        return []
    lines = Lines(charts)
    timing = _timing(scanner, lines)
    times, t_start, pos = lines.snap_times()                        # parsed whether or not they are used, as gridify does
    x = lines.x()
    snapped = None
    if auto_snap:
        snapped = post.snap(times, t_start, [b for b, _ in timing], [o for _, o in timing])
        start = snapped[pos].astype(np.float64)                     # float() of the snapped lines' fields
        end = np.where(lines.is_long != 0, snapped[np.minimum(pos + 1, len(snapped) - 1)], 0).astype(np.float64)
    else:
        start, end = lines.start_ms(), lines.end_ms()
    state, x = post.mini_jacks(lines.chart_start, start, end, lines.is_long, x, jack_interval)
    rows = lines.format(state=state, x=x, snapped=snapped, pos=pos)
    return [(bpm, off, r) for r, (bpm, off) in zip(rows, timing)]

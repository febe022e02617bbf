"""Chart timing on the GPU: gridify's BPM / offset search (SURVEY §8f N4, DESIGN §6b N4) with its scans on the device.

``postprocess.search_timing`` runs estimate_timing as a sequence of scans, each the first improving trial of every chart still
searching, and refits that trial on the host.  ``GridScanner.scan`` is one such scan for a batch of charts: one ``mugd_grid_scan``
call (csrc/gridscan.cu) and one small device-to-host copy.  The candidate table is uploaded once per engine, the charts' note times
once per batch.
"""
from __future__ import annotations

import time
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import lib as L_
from . import postprocess as pp


class GridScanner:
    """the scan kernel's tables and buffers on one engine's device"""

    def __init__(self, engine, cands: np.ndarray = pp.CANDIDATES):
        self.engine = engine
        self.cands_host = np.ascontiguousarray(cands, dtype=np.float64)
        self.cands = torch.from_numpy(self.cands_host).to(engine.device)
        self.n_charts = 0
        self.kernel_ms: Optional[List[float]] = None       # set to [] to record the CUDA-event time of every scan
        self.scan_s = 0.0                                  # wall time spent in scan() calls, synchronisation included

    def load(self, times_list: Sequence[np.ndarray]):
        """pack the charts' float32 note times (each non-empty) on the device"""
        n = len(times_list)
        sizes = [len(t) for t in times_list]
        self.chart_start = np.zeros(n + 1, np.int32)
        self.chart_start[1:] = np.cumsum(sizes)
        packed = np.concatenate([np.asarray(t, np.float32) for t in times_list])
        dev = self.engine.device
        self.times = torch.from_numpy(packed).to(dev)
        self.n_charts = n
        self.k0 = np.zeros(n, np.int32)
        self.head_len = np.zeros(n, np.int32)
        self.best_off = np.zeros(n, np.float64)
        self.best_score = np.zeros(n, np.float64)
        self.first = np.zeros(n, np.float32)
        self.head_bpm = np.zeros(n, np.float64)
        self.head_off = np.zeros((n, pp.MAX_PHASES), np.float64)
        # one device buffer: workspace [n] u64 | out_d [n][3] fp64 | out_i [n][3] int32
        self.buf = torch.empty(n * (8 + 24 + 12), dtype=torch.uint8, device=dev)
        self.out_host = torch.empty(n * (24 + 12), dtype=torch.uint8).pin_memory()

    def scan(self, states: Sequence[pp.ScanState]) -> List[Optional[pp.ScanHit]]:
        """one scan of every loaded chart from its state"""
        t0 = time.perf_counter()
        n = self.n_charts
        assert len(states) == n
        for c, s in enumerate(states):
            self.k0[c] = s.k0
            self.head_len[c] = len(s.head_off)
            self.best_off[c] = s.best_off
            self.best_score[c] = s.best_score
            self.first[c] = s.first
            self.head_bpm[c] = s.head_bpm
            self.head_off[c, :len(s.head_off)] = s.head_off
        eng = self.engine
        stream = torch.cuda.current_stream()
        base = self.buf.data_ptr()
        timed = self.kernel_ms is not None
        if timed:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record(stream)
        L_.check(eng.lib.mugd_grid_scan(eng.handle, self.times.data_ptr(), self.chart_start.ctypes.data, n, self.cands.data_ptr(),
                                        len(self.cands_host), self.k0.ctypes.data, self.head_len.ctypes.data, self.best_off.ctypes.data,
                                        self.best_score.ctypes.data, self.first.ctypes.data, self.head_bpm.ctypes.data,
                                        self.head_off.ctypes.data, base, base + n * 32, base + n * 8, stream.cuda_stream),
                 "mugd_grid_scan")
        if timed:
            ev[1].record(stream)
        self.out_host.copy_(self.buf[n * 8:], non_blocking=True)
        stream.synchronize()
        if timed:
            self.kernel_ms.append(ev[0].elapsed_time(ev[1]))
        raw = self.out_host.numpy()
        out_d = raw[:n * 24].view(np.float64).reshape(n, 3)
        out_i = raw[n * 24:].view(np.int32).reshape(n, 3)
        hits = [None if out_i[c, 0] < 0 else
                pp.ScanHit(int(out_i[c, 0]), int(out_i[c, 1]), out_d[c, 0], out_d[c, 1], int(out_i[c, 2]), out_d[c, 2])
                for c in range(n)]
        self.scan_s += time.perf_counter() - t0
        return hits

    def search(self, times_list: Sequence[np.ndarray]):
        """postprocess.search_timing over these charts with the scans on the device: [(bpm, offset)]"""
        self.load(times_list)
        return pp.search_timing(times_list, self.scan, self.cands_host)

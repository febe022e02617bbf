// One scan of the chart-timing search: the first trial, in the loop order of estimate_timing (mug/data/utils.py:46-101), whose
// score beats the incumbent's.
//
// postprocess.search_timing runs the search as a sequence of scans (DESIGN §6b N4): between two improvements every trial is fixed
// in advance, so one scan evaluates them all at once; the host refits the first improving one and starts the next scan.  A scan of
// chart c is a list of rows of GS_SLOTS trials:
//     row 0      the head: (head_bpm, head_off[j]) in slot 1 + j, j < head_len;
//     row r >= 1 candidate k = k0 + r - 1: slot 0 is (cands[k], first), slot 1 + j is (cands[k], phase j of best_off),
// and a trial's position is row * GS_SLOTS + slot.  A trial (bpm, off) is the reference's fit_grid without refit, operand for
// operand in IEEE arithmetic (no contraction, no reciprocal): step = 60000 / bpm; d = t - off, a float32 subtraction for the
// candidate trial (off = first is np.float32) and an fp64 one for a phase; pos = d / step; on = |pos - rint(pos)| < 10 / step;
// score = n_on / bpm.  The phases are np.arange(best_off, best_off - beat, -beat / 4), beat = 60000 / bpm, filled as numpy fills
// it: p0 = start, p1 = start + step, p_j = start + j * (p1 - start).  n_on is an integer, so the result does not depend on the
// order of the reduction.
//
// One CTA per (chart, tile of GS_ROWS rows), one warp per row: the CTA stages the chart's note times through shared memory in
// chunks, each lane counts the notes on the grid of its row's trials, and after the last chunk lane 0 of a warp offers the row's
// first improving trial to the chart's slot with a 64-bit atomicMin of (position << 32 | n_on).  A CTA whose first position is
// already beaten stops at the next chunk.  A second kernel turns each chart's slot into the outputs.
#include "common.cuh"

#include <math.h>

#include <algorithm>

namespace mugd {

constexpr int GS_MAX_HEAD = 5;                // np.arange of four quarter-beat steps has 4 or 5 entries
constexpr int GS_SLOTS = 1 + GS_MAX_HEAD;     // trials per row
constexpr int GS_ROWS = 8;                    // rows (warps) per CTA
constexpr int GS_CHUNK = 2048;                // note times staged per pass
constexpr int GS_GROUP = 32;                  // charts per launch: their state travels as one kernel parameter
constexpr int GS_MAX_CANDS = 65536;
constexpr unsigned long long GS_NONE = ~0ull;

struct GridChart {
    double best_off, best_score, head_bpm;
    double head_off[GS_MAX_HEAD];
    int32_t start, n, k0, head_len;
    float first;
    int32_t reserved_;
};

struct GridGroup {
    GridChart c[GS_GROUP];
};

struct RowTrials {
    double bpm;
    double off[GS_MAX_HEAD];
    int n_phase;
    bool cand;
};

__device__ __forceinline__ void row_trials(const GridChart& s, const double* __restrict__ cands, int row, RowTrials& t) {
    if (row == 0) {
        t.bpm = s.head_bpm;
        t.cand = false;
        t.n_phase = s.head_len;
#pragma unroll
        for (int j = 0; j < GS_MAX_HEAD; ++j) t.off[j] = s.head_off[j];
        return;
    }
    t.bpm = cands[s.k0 + row - 1];
    t.cand = true;
    const double start = s.best_off;
    const double beat = __ddiv_rn(60000.0, t.bpm);
    const double step = __ddiv_rn(-beat, 4.0);
    const double stop = __dsub_rn(start, beat);
    t.n_phase = min((int)ceil(__ddiv_rn(__dsub_rn(stop, start), step)), GS_MAX_HEAD);
    const double p1 = __dadd_rn(start, step);
    const double delta = __dsub_rn(p1, start);
    t.off[0] = start;
    t.off[1] = p1;
#pragma unroll
    for (int j = 2; j < GS_MAX_HEAD; ++j) t.off[j] = __dadd_rn(start, __dmul_rn((double)j, delta));
}

__device__ __forceinline__ int on_grid(double d, double step, double tol) {
    const double pos = __ddiv_rn(d, step);
    return fabs(__dsub_rn(pos, rint(pos))) < tol ? 1 : 0;
}

__global__ void __launch_bounds__(32 * GS_ROWS)
grid_scan_kernel(const float* __restrict__ times, const double* __restrict__ cands, int n_cands, const __grid_constant__ GridGroup g,
                 unsigned long long* __restrict__ slot_min) {
    __shared__ float s_t[GS_CHUNK];
    __shared__ int s_beaten;
    const GridChart& s = g.c[blockIdx.x];
    const int n_rows = 1 + n_cands - s.k0;
    const int row0 = blockIdx.y * GS_ROWS;
    if (row0 >= n_rows) return;
    const int lane = threadIdx.x & 31, row = row0 + (threadIdx.x >> 5);
    const bool active = row < n_rows;
    unsigned long long* mine = slot_min + blockIdx.x;
    RowTrials t;
    t.bpm = 1.0;
    t.cand = false;
    t.n_phase = 0;
    if (active) row_trials(s, cands, row, t);
    const double step = __ddiv_rn(60000.0, t.bpm);
    const double tol = __ddiv_rn(10.0, step);
    int cnt[GS_SLOTS] = {0, 0, 0, 0, 0, 0};
    for (int base = 0; base < s.n; base += GS_CHUNK) {
        if (threadIdx.x == 0) s_beaten = (*(volatile unsigned long long*)mine >> 32) < (unsigned long long)row0 * GS_SLOTS;
        const int m = min(GS_CHUNK, s.n - base);
        for (int i = threadIdx.x; i < m; i += blockDim.x) s_t[i] = times[s.start + base + i];
        __syncthreads();
        if (s_beaten) return;                                   // uniform: an earlier trial of this chart already improves
        if (active) {
            for (int i = lane; i < m; i += 32) {
                const float x = s_t[i];
                if (t.cand) cnt[0] += on_grid((double)__fsub_rn(x, s.first), step, tol);
#pragma unroll
                for (int j = 0; j < GS_MAX_HEAD; ++j)
                    if (j < t.n_phase) cnt[1 + j] += on_grid(__dsub_rn((double)x, t.off[j]), step, tol);
            }
        }
        __syncthreads();
    }
    if (!active) return;
#pragma unroll
    for (int k = 0; k < GS_SLOTS; ++k) {
        const int n_on = warp_sum(cnt[k]);
        const bool valid = k == 0 ? t.cand : k - 1 < t.n_phase;
        if (valid && __ddiv_rn((double)n_on, t.bpm) > s.best_score) {
            if (lane == 0) atomicMin(mine, ((unsigned long long)(row * GS_SLOTS + k) << 32) | (unsigned)n_on);
            break;
        }
    }
}

// per chart: position, kind (0 head, 1 candidate, 2 phase; -1 none), n_on | bpm, offset, score of the winning trial
__global__ void grid_finish_kernel(const double* __restrict__ cands, const __grid_constant__ GridGroup g, int n,
                                   const unsigned long long* __restrict__ slot_min, int32_t* __restrict__ out_i, double* __restrict__ out_d) {
    const int c = threadIdx.x;
    if (c >= n) return;
    const unsigned long long v = slot_min[c];
    int32_t* oi = out_i + 3 * c;
    double* od = out_d + 3 * c;
    if (v == GS_NONE) {
        oi[0] = -1; oi[1] = -1; oi[2] = 0;
        od[0] = 0.0; od[1] = 0.0; od[2] = 0.0;
        return;
    }
    const int pos = (int)(v >> 32), n_on = (int)(unsigned)v;
    const int row = pos / GS_SLOTS, k = pos - row * GS_SLOTS;
    RowTrials t;
    row_trials(g.c[c], cands, row, t);
    oi[0] = pos;
    oi[1] = row == 0 ? 0 : (k == 0 ? 1 : 2);
    oi[2] = n_on;
    double off = (double)g.c[c].first;
#pragma unroll
    for (int j = 0; j < GS_MAX_HEAD; ++j)
        if (k == 1 + j) off = t.off[j];
    od[0] = t.bpm;
    od[1] = off;
    od[2] = __ddiv_rn((double)n_on, t.bpm);
}

}  // namespace mugd

extern "C" int mugd_grid_scan(mugd_handle* h, const float* times, const int32_t* chart_start, int32_t n_charts,
                              const double* cands, int32_t n_cands, const int32_t* k0, const int32_t* head_len,
                              const double* best_off, const double* best_score, const float* first, const double* head_bpm,
                              const double* head_off, void* workspace, int32_t* out_i, double* out_d, void* stream) {
    using namespace mugd;
    MUGD_REQUIRE(times && chart_start && cands && k0 && head_len && best_off && best_score && first && head_bpm && head_off &&
                 workspace && out_i && out_d, "grid_scan: NULL pointer argument");
    MUGD_REQUIRE(n_charts >= 1, "grid_scan: n_charts=%d < 1", n_charts);
    MUGD_REQUIRE(n_cands >= 1 && n_cands <= GS_MAX_CANDS, "grid_scan: n_cands=%d outside [1, %d]", n_cands, GS_MAX_CANDS);
    MUGD_REQUIRE(((uintptr_t)cands & 7u) == 0 && ((uintptr_t)out_d & 7u) == 0 && ((uintptr_t)workspace & 7u) == 0 &&
                 ((uintptr_t)out_i & 3u) == 0, "grid_scan: cands / out_d / workspace alignment (8 bytes)");
    MUGD_REQUIRE(chart_start[0] == 0, "grid_scan: chart_start[0]=%d, must be 0", chart_start[0]);
    for (int c = 0; c < n_charts; ++c) {
        MUGD_REQUIRE(chart_start[c + 1] > chart_start[c], "grid_scan: chart %d is empty or chart_start decreases (%d -> %d)", c,
                     chart_start[c], chart_start[c + 1]);
        MUGD_REQUIRE(head_len[c] >= 0 && head_len[c] <= GS_MAX_HEAD, "grid_scan: chart %d head_len=%d outside [0, %d]", c, head_len[c],
                     GS_MAX_HEAD);
        MUGD_REQUIRE(k0[c] >= 0 && k0[c] <= n_cands, "grid_scan: chart %d k0=%d outside [0, %d]", c, k0[c], n_cands);
        // |best_off| < 2^53 keeps its phase list at 4 or 5 entries (the rounding of (best_off - beat) - best_off stays far below beat / 4)
        MUGD_REQUIRE(isfinite(best_off[c]) && fabs(best_off[c]) < 0x1p53, "grid_scan: chart %d best_off=%g is not finite or too large",
                     c, best_off[c]);
        MUGD_REQUIRE(head_len[c] == 0 || (isfinite(head_bpm[c]) && head_bpm[c] > 0.0), "grid_scan: chart %d head_bpm=%g must be > 0",
                     c, head_bpm[c]);
    }
    int32_t sm_count = 0;
    MUGD_REQUIRE(h && mugd_device_info(h, &sm_count, nullptr, nullptr) == MUGD_OK, "grid_scan: null handle");
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long* slot_min = (unsigned long long*)workspace;
    MUGD_CHECK_CUDA(cudaMemsetAsync(slot_min, 0xff, sizeof(unsigned long long) * n_charts, st));
    for (int c0 = 0; c0 < n_charts; c0 += GS_GROUP) {
        const int n = std::min(GS_GROUP, n_charts - c0);
        GridGroup g;
        memset(&g, 0, sizeof(g));
        int max_rows = 0;
        for (int i = 0; i < n; ++i) {
            const int c = c0 + i;
            GridChart& s = g.c[i];
            s.start = chart_start[c];
            s.n = chart_start[c + 1] - chart_start[c];
            s.k0 = k0[c];
            s.head_len = head_len[c];
            s.first = first[c];
            s.best_off = best_off[c];
            s.best_score = best_score[c];
            s.head_bpm = head_len[c] ? head_bpm[c] : 1.0;
            for (int j = 0; j < head_len[c]; ++j) s.head_off[j] = head_off[c * GS_MAX_HEAD + j];
            max_rows = std::max(max_rows, 1 + n_cands - k0[c]);
        }
        const dim3 grid((unsigned)n, (unsigned)((max_rows + GS_ROWS - 1) / GS_ROWS));
        grid_scan_kernel<<<grid, 32 * GS_ROWS, 0, st>>>(times, cands, n_cands, g, slot_min + c0);
        MUGD_CHECK_CUDA(cudaGetLastError());
        grid_finish_kernel<<<1, GS_GROUP, 0, st>>>(cands, g, n, slot_min + c0, out_i + 3 * c0, out_d + 3 * c0);
        MUGD_CHECK_CUDA(cudaGetLastError());
    }
    return MUGD_OK;
}

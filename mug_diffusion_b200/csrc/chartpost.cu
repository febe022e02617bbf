// Chart clean-up after the timing search: gridify's snapping and remove_intractable_mania_mini_jacks (mug/data/utils.py:110-268,
// postprocess.snap_lines / postprocess.remove_intractable_mania_mini_jacks), equal to the host functions.
//
// Snapping (chart_snap_kernel): one thread per note time t (an int32), restating snap_lines' snap(t) operand for operand in IEEE
// round-to-nearest with no contraction: for div in (1, 2, 4, 3, 6, 8, 16, 32): step = 60000 / (bpm * div); pos = (t - offset) /
// step; k = rint(pos) (Python's round is half to even); snap on the first div where |pos - k| < 10 / step, to
// (int64)(k * step + offset), truncated toward zero like int(); else keep t.  When gridify's offset is an np.float32 (no refit
// succeeded), NumPy 2 evaluates t - offset in float32: t is rounded to float32 and the subtraction is a float32 one; the division
// and k * step + offset are fp64 (the offset widens exactly).
//
// Mini-jack removal (mini_jack_kernel): one warp per chart runs the host loop over the notes in list order.  Every neighbour query
// of _Chart (near, held_at) walks away from a note and stops at the first live note outside the radius; the warp looks at 32
// candidates per step and finds the stop and the matches with a ballot.  held_at only ever looks at long notes, so it walks the
// chart's list of long notes (built by the warp before the loop) rather than every note.  The mutable state, each note's x and
// alive flag, lives in global memory (L1-resident for the notes a query touches); __syncwarp orders a write by lane 0 before the
// next query's reads.
#include "common.cuh"

#include <math.h>
#include <string.h>

#include <algorithm>

namespace mugd {

constexpr int CS_GROUP = 128;                 // charts per snap launch: their bpm / offset travel as one kernel parameter
constexpr int CS_THREADS = 256;
constexpr int MJ_GROUP = 512;                 // charts per mini-jack launch: their boundaries travel as one kernel parameter
constexpr int MJ_COLUMN_WIDTH = 128;          // 512 / 4 keys
constexpr double CS_MAX_BPM = 1e9;            // keeps pos = (t - offset) / step finite

struct SnapGroup {
    double bpm[CS_GROUP], offset[CS_GROUP];
    int32_t start[CS_GROUP + 1];
    int32_t offset_f32[CS_GROUP];
};

struct JackGroup {
    int32_t start[MJ_GROUP + 1];
};

__global__ void __launch_bounds__(CS_THREADS)
chart_snap_kernel(const int32_t* __restrict__ times, const __grid_constant__ SnapGroup g, int64_t* __restrict__ out) {
    const int c = blockIdx.y;
    const int i = g.start[c] + blockIdx.x * CS_THREADS + threadIdx.x;
    if (i >= g.start[c + 1]) return;
    const int32_t t = times[i];
    const double bpm = g.bpm[c], off = g.offset[c];
    const bool f32 = g.offset_f32[c] != 0;
    const double d = f32 ? (double)__fsub_rn(__int2float_rn(t), (float)off) : __dsub_rn((double)t, off);
    int64_t r = t;
    const int divs[8] = {1, 2, 4, 3, 6, 8, 16, 32};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const double step = __ddiv_rn(60000.0, __dmul_rn(bpm, (double)divs[j]));
        const double pos = __ddiv_rn(d, step);
        const double k = rint(pos);
        if (fabs(__dsub_rn(pos, k)) < __ddiv_rn(10.0, step)) {
            r = (int64_t)__dadd_rn(__dmul_rn(k, step), off);
            break;
        }
    }
    out[i] = r;
}

// mini-jack removal: one chart's arrays (chart-local indices)
struct JackChart {
    const double* start;      // float(f[2])
    const double* end;        // float(f[5].split(":")[0]) of a long note
    const uint8_t* is_long;
    int32_t* x;               // int(float(f[0])); a move rewrites it
    uint8_t* state;           // 0 dropped, 1 kept, 2 kept and moved
    int32_t* ln_rank;         // long notes before note i
    int32_t* ln_idx;          // the long notes, in list order
    int n;
    double radius;            // jack_interval
};

__device__ __forceinline__ int column_of(int32_t x) { return x / MJ_COLUMN_WIDTH; }   // int(x / 128): truncation toward zero

struct Near {
    int count;                // live notes found
    int first;                // the first of them in walk order (backwards first), -1 if none
};

// _Chart.near(i, t, radius, column, back, forth): live notes within radius of t, walking away from i in each direction until the
// first live note outside the radius; column < 0 matches any column.  With `tol`, only notes at least 10 ms from t count (the
// followers filter).  With `any`, the walk ends at the first match (only emptiness is asked).
__device__ Near near(const JackChart& ch, int i, double t, double radius, int column, bool back, bool forth, bool tol, bool any) {
    const int lane = threadIdx.x & 31;
    Near r{0, -1};
    for (int dir = 0; dir < 2; ++dir) {
        if (dir == 0 ? !back : !forth) continue;
        const int step = dir == 0 ? -1 : 1;
        for (int base = 1;; base += 32) {
            const int k = i + step * (base + lane);
            const bool in = k >= 0 && k < ch.n;
            bool live = false, out = false, match = false;
            if (in && ch.state[k] != 0) {
                live = true;
                const double dt = fabs(__dsub_rn(ch.start[k], t));
                out = dt > radius;
                match = !out && (column < 0 || column_of(ch.x[k]) == column) && (!tol || dt >= 10.0);
            }
            const unsigned stop = __ballot_sync(0xffffffffu, !in || (live && out));
            const unsigned valid = stop ? (1u << (__ffs(stop) - 1)) - 1u : 0xffffffffu;
            const unsigned hits = __ballot_sync(0xffffffffu, match) & valid;
            if (hits && r.first < 0) r.first = i + step * (base + __ffs(hits) - 1);
            r.count += __popc(hits);
            if (stop || (any && r.count)) break;
        }
        if (any && r.count) break;
    }
    return r;
}

// _Chart.held_at(before, column, t): the nearest earlier live long note of `column` that started by t decides whether it still
// holds at t (end >= t - 50).
__device__ bool held_at(const JackChart& ch, int before, int column, double t) {
    const int lane = threadIdx.x & 31;
    for (int j0 = ch.ln_rank[before] - 1; j0 >= 0; j0 -= 32) {
        const int j = j0 - lane;
        int k = -1;
        if (j >= 0) {
            const int m = ch.ln_idx[j];
            if (ch.state[m] != 0 && column_of(ch.x[m]) == column && ch.start[m] <= t) k = m;
        }
        const unsigned hits = __ballot_sync(0xffffffffu, k >= 0);
        if (hits) {
            const int m = __shfl_sync(0xffffffffu, k, __ffs(hits) - 1);
            return ch.end[m] >= __dsub_rn(t, 50.0);
        }
    }
    return false;
}

__global__ void __launch_bounds__(32)
mini_jack_kernel(const double* __restrict__ start, const double* __restrict__ end, const uint8_t* __restrict__ is_long,
                 int32_t* x, uint8_t* state, int32_t* workspace, int32_t n_total, double jack_interval,
                 const __grid_constant__ JackGroup g) {
    const int lane = threadIdx.x;
    const int c0 = g.start[blockIdx.x];
    JackChart ch;
    ch.start = start + c0;
    ch.end = end + c0;
    ch.is_long = is_long + c0;
    ch.x = x + c0;
    ch.state = state + c0;
    ch.ln_rank = workspace + c0;
    ch.ln_idx = workspace + n_total + c0;
    ch.n = g.start[blockIdx.x + 1] - c0;
    ch.radius = jack_interval;
    // every note alive; the list of long notes and each note's rank in it
    int n_ln = 0;
    for (int b = 0; b < ch.n; b += 32) {
        const int k = b + lane;
        const bool ln = k < ch.n && ch.is_long[k] != 0;
        const unsigned m = __ballot_sync(0xffffffffu, ln);
        if (k < ch.n) {
            const int rank = n_ln + __popc(m & ((1u << lane) - 1u));
            ch.state[k] = 1;
            ch.ln_rank[k] = rank;
            if (ln) ch.ln_idx[rank] = k;
        }
        n_ln += __popc(m);
    }
    __syncwarp();
    const double J = jack_interval, J2 = __dmul_rn(jack_interval, 2.0);
    for (int i = 0; i < ch.n; ++i) {
        // note i is alive: a drop only ever hits i or an earlier note
        const double t = ch.start[i];
        const int column = column_of(ch.x[i]);
        const Near earlier = near(ch, i, t, J, column, true, false, false, true);
        if (earlier.count == 0) continue;
        if (near(ch, i, t, J2, -1, false, true, true, true).count == 0) continue;        // end of a stream
        const int e = earlier.first;
        const double t_e = ch.start[e];
        bool moved = false;
        for (int pass = 0; pass < 2 && !moved; ++pass) {
            if (pass == 0 && ch.is_long[i]) continue;                                     // a long note is never moved
            const int idx = pass == 0 ? i : e;
            const double when = pass == 0 ? t : t_e;
            const int src = pass == 0 ? column : column_of(ch.x[e]);
            const int targets[3] = {src == 0 || src == 1 ? 1 - src : 5 - src, src == 0 || src == 1 ? 2 : 1,
                                    src == 0 || src == 1 ? 3 : 0};
            for (int q = 0; q < 3; ++q) {
                const int dst = targets[q];
                if (held_at(ch, idx, dst, when)) continue;
                if (near(ch, idx, when, J, dst, true, true, false, true).count == 0) {
                    if (lane == 0) {
                        ch.x[idx] = dst * MJ_COLUMN_WIDTH + MJ_COLUMN_WIDTH / 2;       // int(round((dst + 0.5) * 128))
                        ch.state[idx] = 2;
                    }
                    moved = true;
                    break;
                }
            }
        }
        if (!moved) {
            const int chord_here = near(ch, i, t, 10.0, -1, true, true, false, false).count + 1;
            const int chord_prev = near(ch, e, t_e, 10.0, -1, true, true, false, false).count + 1;
            int victim;
            if (chord_here > 1 && chord_here >= chord_prev && !ch.is_long[i]) victim = i;
            else if (chord_prev > 1 && chord_prev >= chord_here) victim = e;
            else if (ch.is_long[i]) victim = e;
            else victim = i;
            if (lane == 0) ch.state[victim] = 0;
        }
        __syncwarp();
    }
}

}  // namespace mugd

extern "C" int mugd_chart_snap(mugd_handle* h, const int32_t* times, const int32_t* chart_start, int32_t n_charts,
                               const double* bpm, const double* offset, const int32_t* offset_is_f32, int64_t* out, void* stream) {
    using namespace mugd;
    MUGD_REQUIRE(times && chart_start && bpm && offset && offset_is_f32 && out, "chart_snap: NULL pointer argument");
    MUGD_REQUIRE(n_charts >= 1, "chart_snap: n_charts=%d < 1", n_charts);
    MUGD_REQUIRE(((uintptr_t)times & 3u) == 0 && ((uintptr_t)out & 7u) == 0, "chart_snap: times / out alignment (4 / 8 bytes)");
    MUGD_REQUIRE(chart_start[0] == 0, "chart_snap: chart_start[0]=%d, must be 0", chart_start[0]);
    for (int c = 0; c < n_charts; ++c) {
        MUGD_REQUIRE(chart_start[c + 1] >= chart_start[c], "chart_snap: chart_start decreases at chart %d (%d -> %d)", c,
                     chart_start[c], chart_start[c + 1]);
        MUGD_REQUIRE(isfinite(bpm[c]) && bpm[c] > 0.0 && bpm[c] <= CS_MAX_BPM, "chart_snap: chart %d bpm=%g outside (0, %g]", c,
                     bpm[c], CS_MAX_BPM);
        MUGD_REQUIRE(isfinite(offset[c]) && fabs(offset[c]) < 0x1p52, "chart_snap: chart %d offset=%g is not finite or too large", c,
                     offset[c]);
        MUGD_REQUIRE(offset_is_f32[c] == 0 || offset_is_f32[c] == 1, "chart_snap: chart %d offset_is_f32=%d, must be 0 or 1", c,
                     offset_is_f32[c]);
        MUGD_REQUIRE(!offset_is_f32[c] || (double)(float)offset[c] == offset[c],
                     "chart_snap: chart %d offset=%.17g is flagged float32 but is not a float32 value", c, offset[c]);
    }
    int32_t sm_count = 0;
    MUGD_REQUIRE(h && mugd_device_info(h, &sm_count, nullptr, nullptr) == MUGD_OK, "chart_snap: null handle");
    cudaStream_t st = (cudaStream_t)stream;
    for (int c0 = 0; c0 < n_charts; c0 += CS_GROUP) {
        const int n = std::min(CS_GROUP, n_charts - c0);
        SnapGroup g;
        memset(&g, 0, sizeof(g));
        int longest = 0;
        for (int i = 0; i < n; ++i) {
            g.bpm[i] = bpm[c0 + i];
            g.offset[i] = offset[c0 + i];
            g.offset_f32[i] = offset_is_f32[c0 + i];
            g.start[i] = chart_start[c0 + i];
            longest = std::max(longest, chart_start[c0 + i + 1] - chart_start[c0 + i]);
        }
        g.start[n] = chart_start[c0 + n];
        if (longest == 0) continue;
        const dim3 grid((unsigned)((longest + CS_THREADS - 1) / CS_THREADS), (unsigned)n);
        chart_snap_kernel<<<grid, CS_THREADS, 0, st>>>(times, g, out);
        MUGD_CHECK_CUDA(cudaGetLastError());
    }
    return MUGD_OK;
}

extern "C" int mugd_remove_mini_jacks(mugd_handle* h, const int32_t* chart_start, int32_t n_charts, double jack_interval,
                                      const double* start, const double* end, const uint8_t* is_long, int32_t* x, uint8_t* state,
                                      void* workspace, void* stream) {
    using namespace mugd;
    MUGD_REQUIRE(chart_start && start && end && is_long && x && state && workspace, "remove_mini_jacks: NULL pointer argument");
    MUGD_REQUIRE(n_charts >= 1, "remove_mini_jacks: n_charts=%d < 1", n_charts);
    MUGD_REQUIRE(((uintptr_t)start & 7u) == 0 && ((uintptr_t)end & 7u) == 0 && ((uintptr_t)x & 3u) == 0 &&
                 ((uintptr_t)workspace & 3u) == 0, "remove_mini_jacks: start / end / x / workspace alignment (8 / 8 / 4 / 4 bytes)");
    MUGD_REQUIRE(!isnan(jack_interval), "remove_mini_jacks: jack_interval is NaN");
    MUGD_REQUIRE(chart_start[0] == 0, "remove_mini_jacks: chart_start[0]=%d, must be 0", chart_start[0]);
    for (int c = 0; c < n_charts; ++c)
        MUGD_REQUIRE(chart_start[c + 1] >= chart_start[c], "remove_mini_jacks: chart_start decreases at chart %d (%d -> %d)", c,
                     chart_start[c], chart_start[c + 1]);
    MUGD_REQUIRE(chart_start[n_charts] <= (1 << 30), "remove_mini_jacks: %d notes, at most 2^30", chart_start[n_charts]);
    int32_t sm_count = 0;
    MUGD_REQUIRE(h && mugd_device_info(h, &sm_count, nullptr, nullptr) == MUGD_OK, "remove_mini_jacks: null handle");
    cudaStream_t st = (cudaStream_t)stream;
    const int32_t n_total = chart_start[n_charts];
    for (int c0 = 0; c0 < n_charts; c0 += MJ_GROUP) {
        const int n = std::min(MJ_GROUP, n_charts - c0);
        JackGroup g;
        for (int i = 0; i <= n; ++i) g.start[i] = chart_start[c0 + i];
        mini_jack_kernel<<<n, 32, 0, st>>>(start, end, is_long, x, state, (int32_t*)workspace, n_total, jack_interval, g);
        MUGD_CHECK_CUDA(cudaGetLastError());
    }
    return MUGD_OK;
}

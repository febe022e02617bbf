// Device side of the wgmma (Hopper warpgroup MMA) implicit GEMM of gemm_tc.cu.  fp32 in / fp32 out with the 3xTF32 split so results
// stay at fp32 accuracy (DESIGN.md §4 "Precision"):
//
//     a = a_hi + a_lo (both exactly representable in TF32, round-to-nearest),   w = w_hi + w_lo
//     acc += a_lo*w_hi + a_hi*w_lo + a_hi*w_hi          (fp32 accumulation in registers, dropped term ~2^-22)
//
// One call of gemm_tc_tile<BN>() computes one 128 x BN output tile (or its split-K partial) with the two warpgroups of a CTA:
//   TMA          : one elected lane of warp 0 keeps a STAGES-deep ring of (raw A tile, W_hi tile, W_lo tile) in flight; per k-step
//                  (32 fp32 = one 128-byte swizzle row) the raw A tile comes through a 3-D tensor map (k, l, b) -- the conv k=3 halo
//                  is the TMA out-of-bounds zero fill on the l axis, so no im2col / padding copy exists -- plus the pre-split
//                  W_hi / W_lo tiles; completion on an mbarrier, release of a stage by one arrival per warp.
//   warpgroups   : warpgroup w owns tile rows 64w..64w+63.  Each thread reads its A fragment out of the swizzled raw tile, splits
//                  it into a_hi / a_lo (to_tf32) in registers and issues 12 wgmma.m64nBNk8.tf32 per k-step (A from
//                  registers, B = weight tile through a shared-memory descriptor); the next stage is split while they run, and one
//                  k-step of MMAs stays in flight across the k-step boundary.
//   prefetch     : the producer lane also pulls its CTA's slice of the NEXT tensor-core GEMM's weights into L2.
//   epilogue 1   : accumulator registers -> shared memory (row pitch BN+4), over the then idle pipeline buffers
//   epilogue 2   : all warps: bias / time-embedding row / SiLU / GELU / GEGLU / GLU / residual, row-contiguous coalesced stores;
//                  with split-K the partial tile goes to an L2-resident workspace and tc_reduce() sums the splits in fixed
//                  order (deterministic) and runs the same fused epilogue.
#pragma once
#include <cuda.h>
#include <stddef.h>

#include <type_traits>

#include "common.cuh"
#include "wgmma.cuh"

namespace mugd {

constexpr int TC_BM = 128;
constexpr int TC_BK = 32;                 // fp32 elements per k-step = 128 bytes = one swizzle row
constexpr int TC_THREADS = 256;
constexpr uint32_t TC_A_BYTES = TC_BM * TC_BK * 4;   // 16 KB

struct TcParams {
    // What the tile prologue and the TMA producer read before the first load leaves, packed into the first 64 bytes: kernel
    // parameters live in constant memory, a fresh launch misses on every line it touches, and those misses are serial on the
    // producer's critical path.  Filled by tc_geometry() (single_pass: by tc_plan()).
    struct Hot {
        int32_t Lrows, Bs;        // row structure of the A tensor map (Lrows = rows per sample, Bs samples)
        int32_t box_l, box_b;     // TMA box: box_l rows of box_b consecutive samples (box_l*box_b <= 128)
        int32_t tiles_per_sample; // when Lrows >= 128
        int32_t it_base, it_rem;  // split z owns k-steps [z*it_base + min(z, it_rem), +it_base + (z < it_rem)): no division on the device
        int32_t it_main;          // taps * K / 32: k-steps >= it_main read the second source (A2, 1x1 term)
        int32_t kblocks;          // K / 32
        int32_t total_it;         // (taps * K + K2) / 32
        int32_t splits;
        int32_t single_pass;      // 1: plain TF32 (a_hi*w_hi only, ~2^-11 relative) -- opt-in speed mode, NOT used for parity/bench
        int32_t conv_mode, tap_shift, tap_dilation;
        int32_t gx;               // column tiles (grid: gx x gy x splits)
    } hot;
    mugd_gemm g;
    float* ws;                    // split-K partial tiles [tile][split][128][BN]
    int32_t gy;                   // row tiles
    double ln_invK;               // 1 / K (folded LayerNorm: moments -> mean / variance)
    // W_hi / W_lo of the next tensor-core GEMM of the plan (pf_lo NULL in single-pass mode, pf_bytes 0 = none), prefetched into L2
    // while this GEMM runs: the next launch then reads its first stages from L2 instead of HBM.  Weights are written once, when the
    // engine is built, so the prefetch cannot race with a producer.
    const float* pf_hi;
    const float* pf_lo;
    int64_t pf_bytes;
#ifdef MUGD_TC_TIMELINE
    long long* dbg;               // CTA (0,0,0) writes globaltimer stamps (TC_STAMP, tools/bench_gemm.py)
#endif
};
static_assert(sizeof(TcParams::Hot) == 64 && offsetof(TcParams, hot) == 0, "the hot fields are the first 64 bytes of the parameters");

#ifdef __CUDACC__
__device__ __forceinline__ long long gtimer() {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t) :: "memory");
    return t;
}
// Phase stamps of CTA (0,0,0), thread 0 (MUGD_TC_TIMELINE builds): [0] entry, [1] barriers armed, [2] main loop done, [3] tile staged
// in shared memory, [4] tile stored.  tools/bench_gemm.py prints the differences as setup / main / stage / epi.
#ifdef MUGD_TC_TIMELINE
#define TC_STAMP(p, k, cta0) do { if ((p).dbg && (cta0) && threadIdx.x == 0) (p).dbg[k] = gtimer(); } while (0)
#else
#define TC_STAMP(p, k, cta0) do { } while (0)
#endif
// Pipeline of one CTA: STAGES x (raw A tile + W_hi tile + W_lo tile), filled by TMA, consumed by both warpgroups.
template <int BN>
struct TcSmem {
    static_assert(BN == 64 || BN == 128, "tile widths of the wgmma kernel");
    static constexpr uint32_t B_BYTES = BN * TC_BK * 4;
    static constexpr uint32_t STAGE_BYTES = TC_A_BYTES + 2 * B_BYTES;     // raw A tile + W_hi + W_lo (a_hi / a_lo are made in registers)
    static constexpr int STAGES = BN == 128 ? 4 : 6;                      // 192 KB either way
    static constexpr uint32_t TILE_BYTES = STAGES * STAGE_BYTES;
    static constexpr uint32_t BAR_BYTES = 256;
    static constexpr uint32_t TOTAL = TILE_BYTES + 1024 /*align slack*/ + BAR_BYTES;
    static_assert(TOTAL <= 227u * 1024u, "shared memory budget");
    static_assert(128u * (BN + 4) * 4u + 1024u <= TILE_BYTES, "the staged accumulator tile + row statistics must fit the pipeline buffers");
};

// ---- row moments of the OUTPUT for the LayerNorm that follows, accumulated while the tile is written (mugd_gemm.row_moments) ----
// The SEG lanes that hold one output row of this tile reduce with shuffles (fp32: at
// most 128 values), the segment leader adds the tile's share of the row to the row's two doubles -- one address per row, so no
// contention.  Every lane of the warp must call it (inactive: v = 0, m < 0).
template <int SEG>
__device__ __forceinline__ void tc_row_sink(double* buf, int m, float4 v) {
    float s = (v.x + v.y) + (v.z + v.w);
    float ss = (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
#pragma unroll
    for (int o = SEG / 2; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        ss += __shfl_xor_sync(0xffffffffu, ss, o);
    }
    if ((threadIdx.x & (SEG - 1)) == 0 && m >= 0) {
        atomicAdd(buf + (int64_t)m * 2, (double)s);
        atomicAdd(buf + (int64_t)m * 2 + 1, (double)ss);
    }
}
// mean / rstd of a row from its two moments (LayerNorm folded into the GEMM, mugd_gemm.ln_stats).  The variance is formed in fp64
// (E[x^2] - mean^2 cancels), the reciprocal square root in fp32 with one Newton step (~1 ulp): a handful of instructions instead of the
// ~100-deep fp64 divide / sqrt chains, which sat on the critical path between the main loop and the epilogue.
__device__ __forceinline__ float2 tc_ln_from_moments(double s, double ss, double invK, float eps) {
    const double mean = s * invK;
    double var = ss * invK - mean * mean;
    const float v = fmaxf((float)var, 0.f) + eps;
    float r = rsqrtf(v);
    r = r * (1.5f - 0.5f * v * r * r);
    return make_float2((float)mean, r);
}

// epilogue modes of a tile / reduce pass
constexpr int TC_EPI_PLAIN = 0, TC_EPI_SINK = 1 /* act == gate == NONE + row moments of the output */, TC_EPI_LN = 2 /* LayerNorm folded in */;

// Fused epilogue math on 4 consecutive accumulator columns.  ACT / GATE are compile-time so that the compiler
// cannot if-convert the branches into "compute SiLU, GELU and both gates for every element, then select"
// (which it did); callers dispatch once per tile on the (uniform) act/gate values.
// LNF: acc is A W'^T of the un-normalised rows; (acc - mean*colsum)*rstd is the product with the LayerNorm'd rows.
// Returns the stored float4 (GATE_NONE) for the row-moment sink.
template <int ACT, int GATE, bool LNF>
__device__ __forceinline__ float4 tc_finish4(const mugd_gemm& g, float* dst, float4 acc, float4 bia, float4 rvv, float4 res, float4 cs, float2 ln,
                                             int m, int no) {
    // dst = &C[m][no]  (no = output column: the accumulator column, or half of it for gated epilogues)
    float x[4];
    if constexpr (LNF) {
        x[0] = (acc.x - ln.x * cs.x) * ln.y + bia.x + rvv.x; x[1] = (acc.y - ln.x * cs.y) * ln.y + bia.y + rvv.y;
        x[2] = (acc.z - ln.x * cs.z) * ln.y + bia.z + rvv.z; x[3] = (acc.w - ln.x * cs.w) * ln.y + bia.w + rvv.w;
    } else {
        x[0] = acc.x + bia.x + rvv.x; x[1] = acc.y + bia.y + rvv.y; x[2] = acc.z + bia.z + rvv.z; x[3] = acc.w + bia.w + rvv.w;
    }
    if constexpr (ACT == MUGD_ACT_SILU) {
#pragma unroll
        for (int j = 0; j < 4; ++j) x[j] = silu_f(x[j]);
    } else if constexpr (ACT == MUGD_ACT_GELU) {
#pragma unroll
        for (int j = 0; j < 4; ++j) x[j] = gelu_f(x[j]);
    }
    if constexpr (GATE == MUGD_GATE_NONE) {
        const float4 o = make_float4(x[0] + res.x, x[1] + res.y, x[2] + res.z, x[3] + res.w);
        st_f4(dst, o);
        return o;
    } else {
        float o0, o1;
        if constexpr (GATE == MUGD_GATE_GEGLU) { o0 = x[0] * gelu_f(x[1]); o1 = x[2] * gelu_f(x[3]); }
        else { o0 = x[0] * sigmoid_f(x[1]); o1 = x[2] * sigmoid_f(x[3]); }
        if (g.residual) {
            const float2 rr = *reinterpret_cast<const float2*>(g.residual + (int64_t)m * g.ldr + no);
            o0 += rr.x; o1 += rr.y;
        }
        *reinterpret_cast<float2*>(dst) = make_float2(o0, o1);
        return make_float4(o0, o1, 0.f, 0.f);
    }
}

// phase 2 of the epilogue for one CTA: read the staged accumulator tile from shared memory (row pitch BN+4) and
// finish it with coalesced global traffic; U float4 per thread in flight, every global load issued before any use.
// MODE = TC_EPI_LN reads the (mean, rstd) of tile row r from shared memory at rowstat + 8*r (written in phase 1).
template <int BN, int ACT, int GATE, int MODE>
__device__ __forceinline__ void tc_store_tile(const mugd_gemm& g, uint32_t stage, int m_base, int n0, int rows_valid, const float* rowvec,
                                              uint32_t rowstat, float4 bia, float4 cs) {
    constexpr int SP = BN + 4;
    constexpr int C4 = BN / 4;
    constexpr int NU = TC_BM * C4 / TC_THREADS;          // float4 per thread: 8 / 16 / 32 for BN = 64 / 128 / 256
    constexpr int U = NU < 16 ? NU : 16;                 // in flight together
    constexpr int SEG = C4 < 32 ? C4 : 32;
    static_assert(TC_THREADS % C4 == 0, "a thread keeps its column quad for the whole tile");
    // this thread's column quad is the same for every row it visits: bias / column sums (bia, cs) were loaded once, before the main loop
    const int c4 = (int)threadIdx.x % C4;
    const int nn = n0 + c4 * 4;
    const bool col_ok = nn < g.N;
    const bool has_res = GATE == MUGD_GATE_NONE && g.residual != nullptr;
    // Row bookkeeping is incremental (the SASS of the first version spent ~75 instructions per float4 on it: 64-bit address products,
    // an integer division per row for the time-embedding row): a thread's rows are row0, row0 + RPP, ... ; pointers advance by
    // RPP rows; the sample of a row (for the per-sample row vector) is found by ONE division and then by comparison.
    constexpr int RPP = TC_THREADS / C4;                 // rows between two float4s of a thread
    const int row0 = (int)threadIdx.x / C4;
    const int n_rows = min(rows_valid, g.M - m_base);    // rows of this tile that exist
    const int no = (GATE == MUGD_GATE_NONE) ? nn : (nn >> 1);
    float* cp = g.C + (int64_t)(m_base + row0) * g.ldc + no;
    const float* rp = has_res ? g.residual + (int64_t)(m_base + row0) * g.ldr + nn : nullptr;
    const int64_t c_step = (int64_t)RPP * g.ldc, r_step = (int64_t)RPP * g.ldr;
    int smp = 0, smp_end = 0;                            // sample of the current row, first row (tile-relative... absolute m) of the next sample
    if (rowvec) { smp = (m_base + row0) / g.Lout; smp_end = (smp + 1) * g.Lout; }
    // A tile that lies fully inside the matrix (the common case) runs the loop without any per-element predicate, so that the
    // compiler can put all shared-memory reads of a pass in flight; edge tiles take the predicated copy.
    auto pass = [&](auto full_tag) {
        constexpr bool FULL = decltype(full_tag)::value;
#pragma unroll 1
        for (int i0 = 0; i0 < NU; i0 += U) {
            // every global load of this pass is issued before anything is consumed: ONE memory round trip per 16 rows
            float4 res[U], rvv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int row = row0 + (i0 + u) * RPP;
                res[u] = rvv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (FULL || (row < n_rows && col_ok)) {
                    if (has_res) res[u] = ld_f4(rp + (int64_t)(i0 + u) * r_step);
                    if (rowvec) {
                        const int m = m_base + row;
                        while (m >= smp_end) { ++smp; smp_end += g.Lout; }
                        rvv[u] = ld_f4(rowvec + (int64_t)smp * g.rowvec_b_stride + nn);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int row = row0 + (i0 + u) * RPP;
                const int m = m_base + row;
                const bool ok = FULL || (row < n_rows && col_ok);
                const float4 acc = lds_f4(stage + (uint32_t)(row * SP + c4 * 4) * 4u);
                float2 ln = make_float2(0.f, 1.f);
                if constexpr (MODE == TC_EPI_LN) ln = lds_f2(rowstat + (uint32_t)row * 8u);
                float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
                if (ok) o = tc_finish4<ACT, GATE, MODE == TC_EPI_LN>(g, cp + (int64_t)(i0 + u) * c_step, acc, bia, rvv[u], res[u], cs, ln, m, no);
                if constexpr (MODE == TC_EPI_SINK) tc_row_sink<SEG>(g.row_moments, ok ? m : -1, o);
            }
        }
    };
    if (n_rows >= TC_BM && n0 + BN <= g.N) pass(std::true_type{});
    else pass(std::false_type{});
}

// Epilogue variant of a kernel instantiation.  Every variant is its own kernel (template parameter), so a launch only carries the
// store loop it executes: with all eight variants inlined in one kernel the hot kernel grew by 60 % and every GEMM of the step
// got slower (instruction fetch), fused or not.
enum TcEpi { TC_E_NONE = 0, TC_E_GEGLU, TC_E_GLU, TC_E_SILU, TC_E_GELU, TC_E_SINK, TC_E_LN, TC_E_LN_GEGLU, TC_E_COUNT };
template <int EPI> struct TcEpiTraits;
template <> struct TcEpiTraits<TC_E_NONE>     { static constexpr int ACT = MUGD_ACT_NONE, GATE = MUGD_GATE_NONE,  MODE = TC_EPI_PLAIN; };
template <> struct TcEpiTraits<TC_E_GEGLU>    { static constexpr int ACT = MUGD_ACT_NONE, GATE = MUGD_GATE_GEGLU, MODE = TC_EPI_PLAIN; };
template <> struct TcEpiTraits<TC_E_GLU>      { static constexpr int ACT = MUGD_ACT_NONE, GATE = MUGD_GATE_GLU,   MODE = TC_EPI_PLAIN; };
template <> struct TcEpiTraits<TC_E_SILU>     { static constexpr int ACT = MUGD_ACT_SILU, GATE = MUGD_GATE_NONE,  MODE = TC_EPI_PLAIN; };
template <> struct TcEpiTraits<TC_E_GELU>     { static constexpr int ACT = MUGD_ACT_GELU, GATE = MUGD_GATE_NONE,  MODE = TC_EPI_PLAIN; };
template <> struct TcEpiTraits<TC_E_SINK>     { static constexpr int ACT = MUGD_ACT_NONE, GATE = MUGD_GATE_NONE,  MODE = TC_EPI_SINK; };
template <> struct TcEpiTraits<TC_E_LN>       { static constexpr int ACT = MUGD_ACT_NONE, GATE = MUGD_GATE_NONE,  MODE = TC_EPI_LN; };
template <> struct TcEpiTraits<TC_E_LN_GEGLU> { static constexpr int ACT = MUGD_ACT_NONE, GATE = MUGD_GATE_GEGLU, MODE = TC_EPI_LN; };

inline int tc_epi_of(const mugd_gemm& g) {
    if (g.ln_stats) return g.gate == MUGD_GATE_GEGLU ? TC_E_LN_GEGLU : TC_E_LN;
    if (g.row_moments) return TC_E_SINK;
    if (g.gate == MUGD_GATE_GEGLU) return TC_E_GEGLU;
    if (g.gate == MUGD_GATE_GLU) return TC_E_GLU;
    if (g.act == MUGD_ACT_SILU) return TC_E_SILU;
    if (g.act == MUGD_ACT_GELU) return TC_E_GELU;
    return TC_E_NONE;
}

// rows of output tile `by`
__device__ __forceinline__ void tc_tile_rows(const TcParams& p, int by, int& b_base, int& l_base, int& rows_valid) {
    const TcParams::Hot& h = p.hot;
    if (h.Lrows >= TC_BM) {
        b_base = by / h.tiles_per_sample;
        l_base = (by % h.tiles_per_sample) * TC_BM;
        rows_valid = min(TC_BM, h.Lrows - l_base);
    } else {
        b_base = by * h.box_b;
        l_base = 0;
        rows_valid = min(h.box_b, h.Bs - b_base) * h.Lrows;
    }
}

// Barrier block of one CTA (at base + TILE_BYTES): full[STAGES] (TMA landed) empty[STAGES] (both warpgroups done with the stage).
template <int BN>
struct TcBars {
    using S = TcSmem<BN>;
    static constexpr int COUNT = 2 * S::STAGES;
    static_assert(8 * COUNT <= (int)S::BAR_BYTES, "barrier block");
    uint32_t bars;
    __device__ __forceinline__ explicit TcBars(uint32_t base) : bars(base + S::TILE_BYTES) {}
    __device__ __forceinline__ uint32_t full(int s) const { return bars + 8u * s; }
    __device__ __forceinline__ uint32_t empty(int s) const { return bars + 8u * (S::STAGES + s); }
    // arm every barrier: thread t (t < COUNT) arms barrier t; call from the first warp, then sync the CTA
    __device__ __forceinline__ void init_parallel(int t) const {
        if (t >= COUNT) return;
        mbar_init(bars + 8u * t, t < S::STAGES ? 1u : (uint32_t)(TC_THREADS / 32));    // empty: one arrival per warp
        mbar_init_fence();
    }
};

// this thread's A fragments of one k-step (32 columns = 4 x k8), split into TF32 hi / lo.  Row r of the 128B-swizzled raw tile keeps
// its 16-byte chunk c at chunk c ^ (r & 7): the 32 lanes of a load hit 32 distinct banks.
struct TcAFrag {
    uint32_t hi[4][4], lo[4][4];
};
__device__ __forceinline__ void tc_load_split(uint32_t a_tile, int r0, int t, TcAFrag& f) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int r = r0 + (e & 1) * 8;                  // a[0] / a[2]: row g, a[1] / a[3]: row g + 8
            const int chunk = 2 * kk + (e >> 1);             // a[2] / a[3]: column t + 4
            const float x = lds_f1(a_tile + (uint32_t)r * 128u + (uint32_t)((chunk ^ (r & 7)) << 4) + (uint32_t)t * 4u);
            const float h = to_tf32(x);
            f.hi[kk][e] = __float_as_uint(h);
            f.lo[kk][e] = __float_as_uint(to_tf32(x - h));
        }
    }
}

// One 128 x BN output tile (bx, by) of split bz.  `base` = 1024-byte aligned shared-memory address of the CTA's tile pool
// (TcSmem<BN>::TILE_BYTES + barrier block), barriers armed by the caller (TcBars::init_parallel) and visible to all threads.  All 256
// threads call it: warpgroup w computes rows 64w..64w+63 with wgmma (A = the split activation rows from registers, B = the weight
// tiles from shared memory); one elected lane of warp 0 also drives the TMA ring.  On return every TMA has landed, every MMA has
// retired, and the tile (or its split-K partial) is on its way to global memory.
// SERIAL (gemm_tc_serial_kernel): the CTA runs all h.splits K-ranges of its tile one after another (bz = 0) and keeps a running fp32
// sum: after each range the accumulator is added to it and restarted from zero, the same adds in the same order as tc_reduce's sum
// of the partial tiles, and the sum goes through the tile epilogue.  The result equals split kernel + reduce bit for bit, without
// the workspace round trip and the second launch.
template <int BN, int EPI, bool SERIAL = false>
__device__ __forceinline__ void gemm_tc_tile(const CUtensorMap* tmA, const CUtensorMap* tmA1, const CUtensorMap* tmA2, const CUtensorMap* tmB,
                                             const CUtensorMap* tmWhi, const CUtensorMap* tmWlo, const TcParams& p, int bx, int by, int bz,
                                             uint32_t base) {
    using S = TcSmem<BN>;
    constexpr int STAGES = S::STAGES;
    constexpr int NACC = BN / 2;
    const TcBars<BN> B(base);
    auto a_raw = [&](int s) { return base + s * S::STAGE_BYTES; };
    auto b_hi = [&](int s) { return base + s * S::STAGE_BYTES + TC_A_BYTES; };
    auto b_lo = [&](int s) { return b_hi(s) + S::B_BYTES; };

    const mugd_gemm& g = p.g;
    const TcParams::Hot& h = p.hot;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n0 = bx * BN;
    int b_base, l_base, rows_valid;
    tc_tile_rows(p, by, b_base, l_base, rows_valid);
    const int m_base = b_base * h.Lrows + l_base;
    const int it_begin = SERIAL ? 0 : bz * h.it_base + min(bz, h.it_rem);
    const int nit = SERIAL ? h.total_it : h.it_base + (bz < h.it_rem ? 1 : 0);
    const uint32_t a_tx = (uint32_t)(h.box_l * h.box_b) * TC_BK * 4;
    const uint32_t w_tx = (h.single_pass ? 1u : 2u) * S::B_BYTES;

    // k-step i of this split -> stage i % STAGES.  Weights first: they do not depend on the previous kernel.
    auto issue_w = [&](int i) {
        const int s = i % STAGES, it = it_begin + i;
        mbar_expect_tx(B.full(s), a_tx + w_tx);
        tma_load_2d(b_hi(s), tmWhi, B.full(s), it * TC_BK, n0);
        if (!h.single_pass) tma_load_2d(b_lo(s), tmWlo, B.full(s), it * TC_BK, n0);
    };
    auto issue_a = [&](int i) {
        const int s = i % STAGES, it = it_begin + i;
        if (it < h.it_main) {
            const int t = it / h.kblocks;
            const int kb = it - t * h.kblocks;
            // row addressing per tap: SAME = l+t-1, TAPS = l+(t+shift)*dilation (zero fill outside the sample by TMA
            // bounds); DOWN (stride 2, right pad) uses one strided tensor map per tap (row l of map t = source row 2l+t)
            const CUtensorMap* ma = tmA;
            int lshift = 0;
            if (h.conv_mode == MUGD_CONV_SAME) lshift = t - 1;
            else if (h.conv_mode == MUGD_CONV_TAPS) lshift = (t + h.tap_shift) * (h.tap_dilation > 1 ? h.tap_dilation : 1);
            else if (h.conv_mode == MUGD_CONV_DOWN) ma = (t == 0) ? tmA : (t == 1 ? tmA1 : tmA2);
            tma_load_3d(a_raw(s), ma, B.full(s), kb * TC_BK, l_base + lshift, b_base);
        } else {
            tma_load_3d(a_raw(s), tmB, B.full(s), (it - h.it_main) * TC_BK, l_base, b_base);   // second source: 1x1 term
        }
    };
    if (warp == 0) {
        if (elect_one()) {
            const int pro = nit < STAGES ? nit : STAGES;
            for (int i = 0; i < pro; ++i) issue_w(i);
            pdl_wait();                          // activations written by the previous kernel are touched from here on
            for (int i = 0; i < pro; ++i) issue_a(i);
            if (p.pf_bytes > 0) {                // after this CTA's own loads: CTA c prefetches slice c of the next GEMM's weights
                const int64_t ncta = (int64_t)h.gx * p.gy * (SERIAL ? 1 : h.splits);
                const int64_t per = (p.pf_bytes / ncta + 15) & ~(int64_t)15;
                const int64_t off = (((int64_t)bz * p.gy + by) * h.gx + bx) * per;
                const int64_t n = min(per, p.pf_bytes - off);
                if (n > 0) {
                    prefetch_l2(reinterpret_cast<const char*>(p.pf_hi) + off, (uint32_t)n);
                    if (p.pf_lo) prefetch_l2(reinterpret_cast<const char*>(p.pf_lo) + off, (uint32_t)n);
                }
            }
        }
        __syncwarp();
    }

    // Epilogue operands that do not depend on the accumulator are requested now, so that their memory latency hides behind the main
    // loop: the device step counter (selects the time-embedding row), this thread's bias / column-sum quad (its column quad is the
    // same for every row of the tile) and, with a folded LayerNorm, the moments of tile row threadIdx.x.
    int epi_step = 0;
    float4 epi_bias = make_float4(0.f, 0.f, 0.f, 0.f), epi_cs = epi_bias;
    double ln_s = 0.0, ln_ss = 0.0;
    {
        pdl_wait();                                          // the step counter / LayerNorm moments are written by the previous kernels
        if (SERIAL || h.splits == 1) {
            const int nn = n0 + ((int)threadIdx.x % (BN / 4)) * 4;
            if (g.step) epi_step = *g.step;
            if (g.bias && nn < g.N) epi_bias = ld_f4(g.bias + nn);
            if constexpr (TcEpiTraits<EPI>::MODE == TC_EPI_LN) {
                if (nn < g.N) epi_cs = ld_f4(g.ln_colsum + nn);
            }
        }
        if constexpr (TcEpiTraits<EPI>::MODE == TC_EPI_LN) {
            const int rr = (int)threadIdx.x;
            if (rr < TC_BM && rr < rows_valid && m_base + rr < g.M) {
                const double2 mo = *reinterpret_cast<const double2*>(g.ln_stats + (int64_t)m_base * 2 + rr * 2);
                ln_s = mo.x; ln_ss = mo.y;
            }
        }
    }

    // ===================================== main loop (both warpgroups) =====================================
    // One k-step of MMAs stays in flight.  Step i reads one of two A-fragment register sets; once it is issued, step i-1 is retired
    // (wgmma_wait<1>), which frees the other set for step i+1's split and lets this warp release step i-1's stage.  Warp 0 refills
    // that stage when both warpgroups have released it: at that point its own warpgroup still has step i queued on the tensor cores,
    // so neither warpgroup drains its MMAs to wait for the other.
    const int wg = warp >> 2, g8 = lane >> 2, t4 = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + g8;                 // this thread's first fragment row (the second is r0 + 8)
    float acc[NACC];
#pragma unroll
    for (int j = 0; j < NACC; ++j) acc[j] = 0.f;
    float run[SERIAL ? NACC : 1];                                  // SERIAL: sum of the finished K-ranges
    int seg = 0, seg_end = 0;                                      // SERIAL: current K-range and its end (k-steps)
    if constexpr (SERIAL) {
#pragma unroll
        for (int j = 0; j < NACC; ++j) run[j] = 0.f;
        seg_end = h.it_base + (0 < h.it_rem ? 1 : 0);
    }
    TcAFrag f0, f1;
    if (nit > 0) {
        mbar_wait(B.full(0), 0u);
        tc_load_split(a_raw(0), r0, t4, f0);
    }
    auto main_loop = [&](auto single_tag) {
        constexpr bool SINGLE = decltype(single_tag)::value;
        auto kstep = [&](int i, const TcAFrag& cur, TcAFrag& nxt) {
            const int s = i % STAGES;
            const uint64_t dbh = wgmma_desc(b_hi(s)), dbl = wgmma_desc(b_lo(s));
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < TC_BK / 8; ++kk) {
                const uint64_t ko = (uint64_t)(kk * 2);      // 8 fp32 = 32 bytes = 2 x 16-byte units
                if constexpr (SINGLE) {
                    Wgmma<BN>::mma(acc, cur.hi[kk], dbh + ko);
                } else {
                    Wgmma<BN>::mma(acc, cur.lo[kk], dbh + ko);
                    Wgmma<BN>::mma(acc, cur.hi[kk], dbl + ko);
                    Wgmma<BN>::mma(acc, cur.hi[kk], dbh + ko);
                }
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (i > 0) {
                const int j = i - 1, sj = j % STAGES;
                __syncwarp();
                if (lane == 0) mbar_arrive(B.empty(sj));
                if (warp == 0 && j + STAGES < nit) {
                    mbar_wait(B.empty(sj), (uint32_t)(j / STAGES) & 1u);    // both warpgroups are done with stage sj: refill it
                    if (elect_one()) { issue_w(j + STAGES); issue_a(j + STAGES); }
                    __syncwarp();
                }
            }
            // the next stage's activations are split while the tensor cores work on this one
            if (i + 1 < nit) {
                mbar_wait(B.full((i + 1) % STAGES), (uint32_t)((i + 1) / STAGES) & 1u);
                tc_load_split(a_raw((i + 1) % STAGES), r0, t4, nxt);
            }
            if constexpr (SERIAL) {
                if (i + 1 == seg_end) {                           // last k-step of a K-range: run += its accumulator, restart it
                    wgmma_wait<0>();
#pragma unroll
                    for (int j = 0; j < NACC; ++j) { run[j] = __fadd_rn(run[j], acc[j]); acc[j] = 0.f; }
                    ++seg;
                    seg_end += h.it_base + (seg < h.it_rem ? 1 : 0);
                }
            }
        };
        for (int i = 0; i < nit; i += 2) {
            kstep(i, f0, f1);
            if (i + 1 < nit) kstep(i + 1, f1, f0);
        }
    };
    if (h.single_pass) main_loop(std::true_type{});
    else main_loop(std::false_type{});
    wgmma_wait<0>();
    TC_STAMP(p, 2, bx == 0 && by == 0 && bz == 0);
    // LayerNorm folded into this GEMM: the moments of tile row threadIdx.x -> mean / rstd
    float2 lnrow = make_float2(0.f, 1.f);
    if constexpr (TcEpiTraits<EPI>::MODE == TC_EPI_LN) lnrow = tc_ln_from_moments(ln_s, ln_ss, p.ln_invK, g.ln_eps);
    // ===================================== epilogue, phase 1 ================================
    // every warpgroup has retired its MMAs: the pipeline buffers are free for the staged tile (row pitch BN+4 floats)
    __syncthreads();
    constexpr int SP = BN + 4;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int c = j * 8 + 2 * t4;
        const float* fin = SERIAL ? run : acc;
        sts_f2(base + (uint32_t)(r0 * SP + c) * 4u, fin[4 * j], fin[4 * j + 1]);
        sts_f2(base + (uint32_t)((r0 + 8) * SP + c) * 4u, fin[4 * j + 2], fin[4 * j + 3]);
    }
    if constexpr (TcEpiTraits<EPI>::MODE == TC_EPI_LN) {     // (mean, rstd) of tile row r for phase 2, in the last KB of the pipeline buffers
        if (threadIdx.x < TC_BM) sts_f2(base + S::TILE_BYTES - 1024u + (uint32_t)threadIdx.x * 8u, lnrow.x, lnrow.y);
    }
    // ---- phase 2 (all 8 warps): consecutive threads take consecutive float4 of a row -> coalesced global traffic.
    __syncthreads();
    TC_STAMP(p, 3, bx == 0 && by == 0 && bz == 0);
    {
        const float* rowvec = g.rowvec ? g.rowvec + (int64_t)epi_step * g.rowvec_step_stride : nullptr;
        if (!SERIAL && h.splits > 1) {
            const int tile_lin = by * h.gx + bx;
            float* wsp = p.ws + ((int64_t)tile_lin * h.splits + bz) * (TC_BM * BN);
            constexpr int C4 = BN / 4;
            constexpr int U = 8;
#pragma unroll 1
            for (int i0 = 0; i0 < TC_BM * C4; i0 += TC_THREADS * U) {
                float4 a4[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int idx = i0 + u * TC_THREADS + (int)threadIdx.x;
                    const int row = idx / C4, c4 = idx - row * C4;
                    a4[u] = lds_f4(base + (uint32_t)(row * SP + c4 * 4) * 4u);
                }
#pragma unroll
                for (int u = 0; u < U; ++u) st_f4(wsp + (i0 + u * TC_THREADS + (int)threadIdx.x) * 4, a4[u]);   // [row][BN] dense
            }
        } else {
            using E = TcEpiTraits<EPI>;
            tc_store_tile<BN, E::ACT, E::GATE, E::MODE>(g, base, m_base, n0, rows_valid, rowvec, base + S::TILE_BYTES - 1024u, epi_bias, epi_cs);
        }
    }
    TC_STAMP(p, 4, bx == 0 && by == 0 && bz == 0);
}

// split-K second pass, one output row x one 4-column group per thread: a block of TC_THREADS covers TC_RED_ROWS<BN> rows of one tile
// (the reduce of a small GEMM is latency-bound, more and smaller blocks finish sooner).  The partial tiles are summed in fixed split
// order (deterministic), then the fused epilogue (+ row-moment sink / folded LayerNorm) runs.
template <int BN> constexpr int TC_RED_ROWS = TC_THREADS / (BN / 4);

template <int BN, int EPI>
__device__ __forceinline__ void tc_reduce(const TcParams& p, int blk) {
    constexpr int ACT = TcEpiTraits<EPI>::ACT, GATE = TcEpiTraits<EPI>::GATE, MODE = TcEpiTraits<EPI>::MODE;
    constexpr int C4 = BN / 4;
    constexpr int BPT = TC_BM / TC_RED_ROWS<BN>;       // blocks per tile
    constexpr int SEG = C4 < 32 ? C4 : 32;
    constexpr int ZU = 8;                              // partial tiles in flight per thread
    const mugd_gemm& g = p.g;
    const TcParams::Hot& h = p.hot;
    const int tile_lin = blk / BPT;
    const int bx = tile_lin % h.gx, by = tile_lin / h.gx;
    int b_base, l_base, rows_valid;
    tc_tile_rows(p, by, b_base, l_base, rows_valid);
    const int m_base = b_base * h.Lrows + l_base;
    const int c4 = (int)threadIdx.x % C4;
    const int r = (blk % BPT) * TC_RED_ROWS<BN> + (int)threadIdx.x / C4;
    const int n = bx * BN + c4 * 4;
    const int m = m_base + r;
    const bool ok = r < rows_valid && m < g.M && n < g.N;
    // The kernel is one dependent chain of memory round trips; everything that can be asked for early is: bias / column sums are
    // weights (requested before the wait for the GEMM), then -- behind the wait -- the step counter, the residual quad and the row's
    // LayerNorm moments go out BEFORE the partial tiles, and up to 8 partial tiles are in flight together.
    float4 bia = make_float4(0.f, 0.f, 0.f, 0.f), rvv = bia, res = bia, cs = bia;
    if (ok && g.bias) bia = ld_f4(g.bias + n);
    if constexpr (MODE == TC_EPI_LN) {
        if (ok) cs = ld_f4(g.ln_colsum + n);
    }
    pdl_wait();
    int step = 0;
    if (g.step) step = *g.step;
    if (GATE == MUGD_GATE_NONE && g.residual && ok) res = ld_f4(g.residual + (int64_t)m * g.ldr + n);
    double2 mo = make_double2(0.0, 1.0);
    if constexpr (MODE == TC_EPI_LN) {
        if (ok) mo = *reinterpret_cast<const double2*>(g.ln_stats + (int64_t)m * 2);
    }
    const float* src = p.ws + ((long long)tile_lin * h.splits) * (TC_BM * BN) + (long long)r * BN + c4 * 4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int z0 = 0; z0 < h.splits; z0 += ZU) {                            // fixed order -> deterministic
        float4 t4[ZU];
#pragma unroll
        for (int u = 0; u < ZU; ++u) {
            t4[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ok && z0 + u < h.splits) t4[u] = __ldcg(reinterpret_cast<const float4*>(src + (long long)(z0 + u) * (TC_BM * BN)));
        }
        if (z0 == 0 && g.rowvec && ok)                                      // needs the step counter: by now it has arrived
            rvv = ld_f4(g.rowvec + (int64_t)step * g.rowvec_step_stride + (int64_t)(m / g.Lout) * g.rowvec_b_stride + n);
#pragma unroll
        for (int u = 0; u < ZU; ++u) { acc.x += t4[u].x; acc.y += t4[u].y; acc.z += t4[u].z; acc.w += t4[u].w; }
    }
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ok) {
        float2 ln = make_float2(0.f, 1.f);
        if constexpr (MODE == TC_EPI_LN) ln = tc_ln_from_moments(mo.x, mo.y, p.ln_invK, g.ln_eps);
        const int no = (GATE == MUGD_GATE_NONE) ? n : (n >> 1);
        o = tc_finish4<ACT, GATE, MODE == TC_EPI_LN>(g, g.C + (int64_t)m * g.ldc + no, acc, bia, rvv, res, cs, ln, m, no);
    }
    if constexpr (MODE == TC_EPI_SINK) tc_row_sink<SEG>(g.row_moments, ok ? m : -1, o);
}

#endif  // __CUDACC__

// ---- host side (gemm_tc.cu) -------------------------------------------------------------------------
struct TcGeometry {
    TcParams::Hot hot;        // every field but single_pass (a per-handle switch)
    int BN, gy;
    int64_t ws_floats;
};
// one planned tensor-core GEMM: kernel parameters + its six tensor maps (A taps 0..2, second source, W_hi, W_lo) + the tile width
struct alignas(64) TcPlanned {
    CUtensorMap maps[6];
    TcParams p;
    int BN;
};
TcGeometry tc_geometry(const mugd_gemm& g, int sm_count, int forced_split);
// validates, picks the geometry, encodes the maps; `next` (or NULL): the tensor-core GEMM whose weights this one prefetches into L2;
// `serial`: the K splits run inside one CTA (gemm_tc_serial_kernel), no workspace
int tc_plan(const DeviceInfo& dev, const mugd_gemm& g, const mugd_gemm* next, TcPlanned* out, bool serial = false);

}  // namespace mugd

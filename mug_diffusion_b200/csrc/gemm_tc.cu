// wgmma implicit GEMM: kernels + host side (geometry planner, tensor-map encoding, launch).  The device code lives in gemm_tc.cuh.
//
// Reference call sites are the same as gemm_simt.cu (which remains the exact-fp32 referee and the fallback for
// shapes this kernel does not take: K % 32 != 0, N < 16, generic upsampling addressing).
#include "gemm_tc.cuh"

namespace mugd {

// one-time CTA setup of the wgmma kernels: arm the barriers and warm the TMA descriptor cache; nothing here touches memory written by
// the previous kernel.  Returns the 1024-byte aligned shared-memory base of the tile pool.
template <int BN>
__device__ __forceinline__ uint32_t tc_cta_setup(uint8_t* smem_raw, const CUtensorMap* tmA, const CUtensorMap* tmA1, const CUtensorMap* tmA2,
                                                 const CUtensorMap* tmB, const CUtensorMap* tmWhi, const CUtensorMap* tmWlo, const TcParams& p) {
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;       // SWIZZLE_128B needs 1024-B alignment
    const TcBars<BN> B(base);
    TC_STAMP(p, 0, blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0);
    if (threadIdx.x < 32) {
        B.init_parallel((int)threadIdx.x);
    } else if (threadIdx.x < 38) {
        // warm the TMA descriptor cache while the barriers are set up
        const CUtensorMap* m = threadIdx.x == 32 ? tmA : threadIdx.x == 33 ? tmA1 : threadIdx.x == 34 ? tmA2
                             : threadIdx.x == 35 ? tmB : threadIdx.x == 36 ? tmWhi : tmWlo;
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
    }
    __syncthreads();
    TC_STAMP(p, 1, blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0);
    return base;
}

template <int BN, int EPI>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA1,
               const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmWhi,
               const __grid_constant__ CUtensorMap tmWlo, const __grid_constant__ TcParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = tc_cta_setup<BN>(smem_raw, &tmA, &tmA1, &tmA2, &tmB, &tmWhi, &tmWlo, p);
    gemm_tc_tile<BN, EPI>(&tmA, &tmA1, &tmA2, &tmB, &tmWhi, &tmWlo, p, blockIdx.x, blockIdx.y, blockIdx.z, base);
}

// split-K finished inside the CTA (MUGD_OP_GEMM_SERIAL): grid gx x gy, each CTA runs the h.splits K-ranges of its tile in turn and
// sums them in the reduce kernel's order before the fused epilogue (gemm_tc_tile, SERIAL).
template <int BN, int EPI>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_serial_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA1,
                      const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB,
                      const __grid_constant__ CUtensorMap tmWhi, const __grid_constant__ CUtensorMap tmWlo, const __grid_constant__ TcParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = tc_cta_setup<BN>(smem_raw, &tmA, &tmA1, &tmA2, &tmB, &tmWhi, &tmWlo, p);
    gemm_tc_tile<BN, EPI, true>(&tmA, &tmA1, &tmA2, &tmB, &tmWhi, &tmWlo, p, blockIdx.x, blockIdx.y, 0, base);
}

// split-K second pass: fully parallel over the GPU and L2-resident (see tc_reduce).
template <int BN, int EPI>
__global__ void __launch_bounds__(TC_THREADS)
gemm_tc_reduce_kernel(const __grid_constant__ TcParams p) {
    tc_reduce<BN, EPI>(p, blockIdx.x);                 // waits for the GEMM (griddepcontrol.wait) after requesting its weight-side operands
}

#ifdef MUGD_TC_TIMELINE
static long long* g_tc_dbg = nullptr;
#endif
// planner constants: relative weights of the tile-width / K-split decision (mugd_debug_set_tc_cost for sweeps)
static float g_tc_kstep128 = 0.55f;  // per k-step of a 128-wide tile
static float g_tc_split = 3.0f;      // per split-K round trip (workspace + reduce launch)
static int g_tc_force_bn = 0;        // experiments: 0 = cost model, 64 / 128 = force the tile width where legal

// =====================================================================================================
// host side
// =====================================================================================================
static bool tc_shape_ok(const mugd_gemm& g) {
    if (!(g.conv_mode == MUGD_CONV_NONE || g.conv_mode == MUGD_CONV_SAME || g.conv_mode == MUGD_CONV_DOWN ||
          g.conv_mode == MUGD_CONV_TAPS)) return false;
    if (g.conv_mode == MUGD_CONV_DOWN && g.Lout < 2) return false;
    if (g.K2 % TC_BK != 0 || (g.K2 > 0 && g.conv_mode == MUGD_CONV_DOWN)) return false;
    return g.K % TC_BK == 0 && g.N >= 16 && g.N % 4 == 0;      // narrow outputs (the 16-channel output convs) take a 64-wide tile: the TMA zero-fills the missing weight rows
}

bool gemm_tc_supported(const mugd_gemm& g) {
    if (!tc_shape_ok(g)) return false;
    if (!g.W_hi || !g.W_lo) return false;
    if (g.lda % 4 != 0 || !aligned16(g.A) || !aligned16(g.W_hi) || !aligned16(g.W_lo)) return false;
    if (g.K2 > 0 && (!g.A2 || g.lda2 % 4 != 0 || !aligned16(g.A2))) return false;
    return true;
}

// the row-moment sink and the folded LayerNorm exist on the tensor-core path only
static int tc_validate_fusions(const mugd_gemm& g) {
    if (g.row_moments)
        MUGD_REQUIRE(g.act == MUGD_ACT_NONE && g.gate == MUGD_GATE_NONE && !g.ln_stats && (reinterpret_cast<uintptr_t>(g.row_moments) & 15u) == 0,
                     "gemm: row_moments needs act == gate == NONE, no folded LayerNorm and a 16-byte aligned buffer");
    if (g.ln_stats) {
        MUGD_REQUIRE(g.ln_colsum && aligned16(g.ln_colsum) && (reinterpret_cast<uintptr_t>(g.ln_stats) & 15u) == 0 && g.taps == 1 && g.K2 == 0 &&
                         g.act == MUGD_ACT_NONE && (g.gate == MUGD_GATE_NONE || g.gate == MUGD_GATE_GEGLU) && !g.rowvec,
                     "gemm: folded LayerNorm needs a single-source Linear with act NONE and gate NONE/GEGLU");
    }
    return MUGD_OK;
}

TcGeometry tc_geometry(const mugd_gemm& g, int sm_count, int forced_split) {
    TcGeometry t = {};
    TcParams::Hot& h = t.hot;
    t.BN = (g.N >= 128) ? 128 : 64;
    if (g.conv_mode == MUGD_CONV_NONE) { h.Lrows = g.M; h.Bs = 1; }
    else { h.Lrows = g.Lout; h.Bs = g.M / g.Lout; }
    if (h.Lrows >= TC_BM) {
        h.box_l = TC_BM; h.box_b = 1;
        h.tiles_per_sample = (h.Lrows + TC_BM - 1) / TC_BM;
        t.gy = h.tiles_per_sample * h.Bs;
    } else {
        h.box_l = h.Lrows;
        h.box_b = TC_BM / h.Lrows;
        if (h.box_b > h.Bs) h.box_b = h.Bs;
        h.tiles_per_sample = 1;
        t.gy = (h.Bs + h.box_b - 1) / h.box_b;
    }
    h.kblocks = g.K / TC_BK;
    h.it_main = g.taps * h.kblocks;
    h.total_it = h.it_main + g.K2 / TC_BK;
    // Cost model: a CTA needs ~1 unit to fill its pipeline and g_tc_kstep128 per k-step of a 128-wide tile (0.4 with 64-wide tiles);
    // splitting K adds the workspace round trip and a second (reduce) launch, g_tc_split.
    // Candidates: tile width 64 (narrow N, or forced), 128 when N allows it, each with its best K split.
    int splits = 1;
    float best = 1e30f;
    static const int cands[2] = {64, 128};
    for (int cand = 0; cand < 2; ++cand) {
        const int bn = cands[cand];
        if (bn > 64 && g.N < bn) continue;
        if (bn == 64 && g.N >= 128 && g_tc_force_bn != 64) continue;
        if (g_tc_force_bn && bn != g_tc_force_bn && !(g_tc_force_bn > g.N && bn == 64)) continue;
        const int gx = (g.N + bn - 1) / bn;
        const int tiles = gx * t.gy;
        const float kstep = bn == 128 ? g_tc_kstep128 : 0.4f;
        const int sp_max = forced_split > 0 ? forced_split : (tiles < sm_count ? 16 : 1);
        for (int sp = forced_split > 0 ? forced_split : 1; sp <= sp_max && sp <= h.total_it; ++sp) {
            const int per = (h.total_it + sp - 1) / sp;
            if (forced_split <= 0 && sp > 1 && per < 2) break;
            if (forced_split <= 0 && sp > 1 && tiles * sp > 2 * sm_count) break;   // bounds the workspace: < 2*SMs partial tiles
            const int waves = (tiles * sp + sm_count - 1) / sm_count;
            const float est = waves * (1.0f + kstep * per) + (sp > 1 ? g_tc_split : 0.0f);
            if (est < best - 0.25f) { best = est; splits = sp; t.BN = bn; }
        }
    }
    h.gx = (g.N + t.BN - 1) / t.BN;
    if (splits > h.total_it) splits = h.total_it;
    if (splits < 1) splits = 1;
    h.splits = splits;
    h.it_base = h.total_it / splits;
    h.it_rem = h.total_it % splits;
    h.conv_mode = g.conv_mode;
    h.tap_shift = g.tap_shift;
    h.tap_dilation = g.tap_dilation;
    t.ws_floats = splits > 1 ? (int64_t)h.gx * t.gy * splits * TC_BM * t.BN : 0;
    return t;
}

int tc_plan(const DeviceInfo& dev, const mugd_gemm& g, const mugd_gemm* next, TcPlanned* out, bool serial) {
    MUGD_REQUIRE(gemm_tc_supported(g), "gemm_tc: unsupported shape/operands");
    int rc = tc_validate_fusions(g);
    if (rc != MUGD_OK) return rc;
    const TcGeometry t = tc_geometry(g, dev.sm_count, g.split_k);
    const TcParams::Hot& h = t.hot;
    if (h.splits > 1 && !serial) {
        MUGD_REQUIRE(g.workspace, "gemm_tc: split-K needs a workspace");
        MUGD_REQUIRE(g.workspace_bytes >= t.ws_floats * 4, "gemm_tc: workspace too small (%lld < %lld)", (long long)g.workspace_bytes,
                     (long long)t.ws_floats * 4);
    }
    const cuuint32_t a_box[3] = {(cuuint32_t)TC_BK, (cuuint32_t)h.box_l, (cuuint32_t)h.box_b};
    for (int tap = 0; tap < 3; ++tap) {
        if (tap > 0 && g.conv_mode != MUGD_CONV_DOWN) { out->maps[tap] = out->maps[0]; continue; }
        const bool down = g.conv_mode == MUGD_CONV_DOWN;
        // DOWN: row l of the map of tap t is source row 2l+t; the last row of tap 2 is the right padding -> out of bounds
        const cuuint64_t rows = down ? (cuuint64_t)(h.Lrows - (tap == 2 ? 1 : 0)) : (cuuint64_t)h.Lrows;
        const cuuint64_t sample_rows = down ? (cuuint64_t)g.Lin : (cuuint64_t)h.Lrows;
        const cuuint64_t dims[3] = {(cuuint64_t)g.K, rows, (cuuint64_t)h.Bs};
        const cuuint64_t strides[2] = {(cuuint64_t)g.lda * 4 * (down ? 2 : 1), sample_rows * (cuuint64_t)g.lda * 4};
        rc = encode_f32_tma(&out->maps[tap], g.A + (down ? (int64_t)tap * g.lda : 0), 3, dims, strides, a_box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                            "gemm_tc A");
        if (rc != MUGD_OK) return rc;
    }
    if (g.K2 > 0) {
        // second source: same row structure as the output (Lrows rows per sample), no tap shift
        const cuuint64_t dims[3] = {(cuuint64_t)g.K2, (cuuint64_t)h.Lrows, (cuuint64_t)h.Bs};
        const cuuint64_t strides[2] = {(cuuint64_t)g.lda2 * 4, (cuuint64_t)h.Lrows * (cuuint64_t)g.lda2 * 4};
        rc = encode_f32_tma(&out->maps[3], g.A2, 3, dims, strides, a_box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "gemm_tc A2");
        if (rc != MUGD_OK) return rc;
    } else {
        out->maps[3] = out->maps[0];
    }
    const cuuint64_t ktot = (cuuint64_t)g.taps * g.K + g.K2;
    const cuuint64_t w_dims[2] = {ktot, (cuuint64_t)g.N};
    const cuuint64_t w_strides[1] = {ktot * 4};
    const cuuint32_t w_box[2] = {(cuuint32_t)TC_BK, (cuuint32_t)t.BN};
    for (int w = 0; w < 2; ++w) {
        rc = encode_f32_tma(&out->maps[4 + w], w == 0 ? g.W_hi : g.W_lo, 2, w_dims, w_strides, w_box, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            "gemm_tc W");
        if (rc != MUGD_OK) return rc;
    }
    TcParams& p = out->p;
    memset(&p, 0, sizeof(p));
    p.hot = h;
    p.hot.single_pass = dev.tc_single_pass ? 1 : 0;
    p.g = g;
    p.ws = (float*)g.workspace;
    p.gy = t.gy;
    p.ln_invK = 1.0 / (double)g.K;
    if (next) {
        p.pf_hi = next->W_hi;
        p.pf_lo = p.hot.single_pass ? nullptr : next->W_lo;
        p.pf_bytes = (int64_t)next->N * ((int64_t)next->taps * next->K + next->K2) * 4;
    }
#ifdef MUGD_TC_TIMELINE
    p.dbg = g_tc_dbg;
#endif
    out->BN = t.BN;
    return MUGD_OK;
}

template <int BN, int EPI>
static int tc_launch(const TcPlanned& pl, cudaStream_t st) {
    const TcParams& p = pl.p;
    const TcParams::Hot& h = p.hot;
    if (h.splits > 1) {
        // the main kernel only writes partial tiles: it runs the smallest instantiation, the epilogue variant lives in the reduce
        MUGD_CHECK_CUDA(launch_k(gemm_tc_kernel<BN, TC_E_NONE>, dim3(h.gx, p.gy, h.splits), dim3(TC_THREADS), TcSmem<BN>::TOTAL, st, pl.maps[0],
                                 pl.maps[1], pl.maps[2], pl.maps[3], pl.maps[4], pl.maps[5], p));
        MUGD_CHECK_CUDA(launch_k(gemm_tc_reduce_kernel<BN, EPI>, dim3((unsigned)(h.gx * p.gy * (TC_BM / TC_RED_ROWS<BN>))), dim3(TC_THREADS), 0,
                                 st, p));
        return MUGD_OK;
    }
    MUGD_CHECK_CUDA(launch_k(gemm_tc_kernel<BN, EPI>, dim3(h.gx, p.gy, 1), dim3(TC_THREADS), TcSmem<BN>::TOTAL, st, pl.maps[0], pl.maps[1],
                             pl.maps[2], pl.maps[3], pl.maps[4], pl.maps[5], p));
    return MUGD_OK;
}

template <int BN, int EPI>
static int tc_launch_serial(const TcPlanned& pl, cudaStream_t st) {
    const TcParams& p = pl.p;
    MUGD_CHECK_CUDA(launch_k(gemm_tc_serial_kernel<BN, EPI>, dim3(p.hot.gx, p.gy, 1), dim3(TC_THREADS), TcSmem<BN>::TOTAL, st, pl.maps[0],
                             pl.maps[1], pl.maps[2], pl.maps[3], pl.maps[4], pl.maps[5], p));
    return MUGD_OK;
}

template <int BN, int... EPI>
static cudaError_t allow_smem_bn(int bytes, std::integer_sequence<int, EPI...>) {
    const cudaError_t e = allow_dynamic_smem(bytes, gemm_tc_kernel<BN, EPI>...);
    return e != cudaSuccess ? e : allow_dynamic_smem(bytes, gemm_tc_serial_kernel<BN, EPI>...);
}
cudaError_t gemm_tc_allow_smem(int bytes) {
    const cudaError_t e = allow_smem_bn<64>(bytes, std::make_integer_sequence<int, TC_E_COUNT>{});
    return e != cudaSuccess ? e : allow_smem_bn<128>(bytes, std::make_integer_sequence<int, TC_E_COUNT>{});
}

template <int BN, template <int, int> class Launch>
static int tc_launch_bn(const TcPlanned& pl, cudaStream_t st) {
    switch (tc_epi_of(pl.p.g)) {
        case TC_E_GEGLU: return Launch<BN, TC_E_GEGLU>::run(pl, st);
        case TC_E_GLU: return Launch<BN, TC_E_GLU>::run(pl, st);
        case TC_E_SILU: return Launch<BN, TC_E_SILU>::run(pl, st);
        case TC_E_GELU: return Launch<BN, TC_E_GELU>::run(pl, st);
        case TC_E_SINK: return Launch<BN, TC_E_SINK>::run(pl, st);
        case TC_E_LN: return Launch<BN, TC_E_LN>::run(pl, st);
        case TC_E_LN_GEGLU: return Launch<BN, TC_E_LN_GEGLU>::run(pl, st);
        default: return Launch<BN, TC_E_NONE>::run(pl, st);
    }
}
template <int BN, int EPI> struct TcSplitLaunch { static int run(const TcPlanned& pl, cudaStream_t st) { return tc_launch<BN, EPI>(pl, st); } };
template <int BN, int EPI> struct TcSerialLaunch { static int run(const TcPlanned& pl, cudaStream_t st) { return tc_launch_serial<BN, EPI>(pl, st); } };

int launch_gemm_tc(const DeviceInfo& dev, const mugd_gemm& g, const mugd_gemm* next, cudaStream_t st, int* launches) {
    TcPlanned pl;
    int rc = tc_plan(dev, g, next, &pl);
    if (rc != MUGD_OK) return rc;
    if (pl.BN == 128) rc = tc_launch_bn<128, TcSplitLaunch>(pl, st);
    else rc = tc_launch_bn<64, TcSplitLaunch>(pl, st);
    if (rc != MUGD_OK) return rc;
    if (launches) *launches += pl.p.hot.splits > 1 ? 2 : 1;
    return MUGD_OK;
}

int validate_gemm_serial(const mugd_gemm& g, int default_impl) {
    const int impl = g.impl == MUGD_GEMM_AUTO ? default_impl : g.impl;
    MUGD_REQUIRE(impl == MUGD_GEMM_TC, "gemm_serial: runs on the tensor-core path only (impl %d)", impl);
    MUGD_REQUIRE(g.split_k >= 1, "gemm_serial: needs a forced K split (split_k = %d)", g.split_k);
    MUGD_REQUIRE(tc_shape_ok(g) && g.split_k <= (g.taps * g.K + g.K2) / TC_BK,
                 "gemm_serial: shape the tensor-core kernel does not take, or more splits than k-steps (M=%d N=%d K=%d taps=%d K2=%d split_k=%d)",
                 g.M, g.N, g.K, g.taps, g.K2, g.split_k);
    MUGD_REQUIRE(gemm_tc_supported(g), "gemm_serial: needs TF32 hi / lo weights and 16-byte aligned operands (M=%d N=%d K=%d)", g.M, g.N, g.K);
    return MUGD_OK;
}

int launch_gemm_serial(const DeviceInfo& dev, const mugd_gemm& g, int default_impl, const mugd_gemm* next, cudaStream_t st, int* launches) {
    int rc = validate_gemm(g);
    if (rc != MUGD_OK) return rc;
    if ((rc = validate_gemm_serial(g, default_impl)) != MUGD_OK) return rc;
    TcPlanned pl;
    if ((rc = tc_plan(dev, g, next, &pl, true)) != MUGD_OK) return rc;
    if (pl.BN == 128) rc = tc_launch_bn<128, TcSerialLaunch>(pl, st);
    else rc = tc_launch_bn<64, TcSerialLaunch>(pl, st);
    if (rc != MUGD_OK) return rc;
    if (launches) *launches += 1;
    return MUGD_OK;
}

}  // namespace mugd

// kstep256_us and two_cta_fixed_us are accepted for ABI compatibility and ignored: no such kernel variant exists
extern "C" int mugd_debug_set_tc_cost(float kstep128_us, float kstep256_us, float split_us, float two_cta_fixed_us) {
    (void)kstep256_us;
    (void)two_cta_fixed_us;
    if (kstep128_us > 0.f) mugd::g_tc_kstep128 = kstep128_us;
    if (split_us > 0.f) mugd::g_tc_split = split_us;
    return MUGD_OK;
}

extern "C" int mugd_debug_set_tc_tile_n(int bn) {
    mugd::g_tc_force_bn = (bn == 64 || bn == 128) ? bn : 0;
    return MUGD_OK;
}

extern "C" int mugd_debug_set_tc_timing(long long* device_buf) {
#ifdef MUGD_TC_TIMELINE
    mugd::g_tc_dbg = device_buf;
    return MUGD_OK;
#else
    (void)device_buf;
    mugd::set_error("mugd_debug_set_tc_timing: this build has no timeline hooks (rebuild with -DMUGD_TC_TIMELINE, tools/build_variant.py)");
    return MUGD_ERR_INVALID;
#endif
}

extern "C" int mugd_gemm_tc_variant(const mugd_gemm* g, int32_t sm_count, int32_t* tile_n, int32_t* ctas_per_sm, int32_t* grid_ctas) {
    using namespace mugd;
    MUGD_REQUIRE(g, "gemm_tc_variant: null");
    if (!tc_shape_ok(*g)) {
        if (tile_n) *tile_n = 0;
        if (ctas_per_sm) *ctas_per_sm = 0;
        if (grid_ctas) *grid_ctas = 0;
        return MUGD_OK;
    }
    const int sms = sm_count > 0 ? sm_count : 132;
    const TcGeometry t = tc_geometry(*g, sms, g->split_k);
    if (tile_n) *tile_n = t.BN;
    if (ctas_per_sm) *ctas_per_sm = 1;
    if (grid_ctas) *grid_ctas = t.hot.gx * t.gy * t.hot.splits;
    return MUGD_OK;
}

extern "C" int mugd_gemm_tc_query(mugd_handle*, const mugd_gemm* g, int32_t sm_count, int32_t* supported, int32_t* splits,
                                  int64_t* workspace_bytes, int32_t* n_tiles) {
    using namespace mugd;
    MUGD_REQUIRE(g, "gemm_tc_query: null");
    const bool ok = tc_shape_ok(*g);
    if (supported) *supported = ok ? 1 : 0;
    if (!ok) {
        if (splits) *splits = 0;
        if (workspace_bytes) *workspace_bytes = 0;
        if (n_tiles) *n_tiles = 0;
        return MUGD_OK;
    }
    const TcGeometry t = tc_geometry(*g, sm_count > 0 ? sm_count : 132, g->split_k);
    if (splits) *splits = t.hot.splits;
    if (workspace_bytes) *workspace_bytes = t.ws_floats * 4;
    if (n_tiles) *n_tiles = t.hot.gx * t.gy;
    return MUGD_OK;
}

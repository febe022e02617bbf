// Attention of mug/model/attention.py:91-126 (CrossAttention.forward) with both contractions on the Hopper warpgroup tensor
// cores (wgmma), fp32 in / fp32 out through the same 3xTF32 split as gemm_tc.cu:
//
//     idx_ij = clamp(j - i, -P, P) + P
//     s_ij   = (q_i . k_j + relpos[idx_ij, h]) * scale                 S = Q K^T   : wgmma, A = Q from registers
//     o_i    = sum_j softmax_j(s_i)_j * cgain[idx_ij, h] * v_j         O = P V     : wgmma, A = P from registers
//
// One CTA owns 128 queries of one (sample, head) and streams 128-key tiles (flash style: no [Lq, Lk] matrix in memory, running
// max / sum per query row).  Warpgroup w owns query rows 64w..64w+63; a thread holds two rows (g, g+8 of its warp's 16):
//   * Q is split into q_hi / q_lo once and stays in registers for the whole CTA, in the wgmma A-fragment layout;
//   * the raw K and V head slices of a key tile arrive by TMA (3-D tensor maps (channel, key, sample), 128B swizzle, keys past Lk
//     zero-filled by the TMA bounds check), one tile ahead of the math when two stages fit (head dim 32 / 48);
//     the key tile is split in place into k_hi / k_lo (row = key, 128 bytes of channels: the K-major B operand of S = Q K^T);
//     the value tile is split and transposed shared -> shared into V^T hi / lo (row = channel, keys contiguous: the K-major B
//     operand of O = P V) while the tensor cores compute S, one conflict-free 32-key x 4-channel block per warp step;
//   * S lands in registers; bias, scale, key mask and the online softmax run there (a row is spread over the 4 threads of a
//     quad: two shuffles for its max, its sum is kept per thread and reduced once at the end);
//   * P * gain is split into hi / lo and fed straight back as the A fragments of P V.  The accumulator holds keys 2t, 2t+1 of
//     each 8-key group where the A fragment expects keys t, t+4, so V^T stores the keys of every 8-group in the order
//     0 2 4 6 1 3 5 7: the contraction runs over the same pairs and P never leaves the registers;
//   * O accumulates in registers, rescaled by exp(m_old - m_new) before each tile's P V.
// The FFMA kernel in attention.cu stays as the exact-fp32 referee (mugd_set_attention_impl(0)).
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

#include <math.h>

namespace mugd {
namespace atc {

constexpr int THREADS = 256;
constexpr int BQ = 128;
constexpr int BKV = 128;
constexpr uint32_t SLAB = BKV * 128;          // 128 keys x (32 fp32 channels = 128 B): one swizzle-atom column of a tile

template <int D>
struct Smem {
    static constexpr int KSLABS = (D + 31) / 32;           // 32-channel slabs per head slice (head dim 48: 1.5 used)
    static constexpr int STAGES = (D == 64) ? 1 : 2;       // two key tiles in flight do not fit for head dim 64
    static constexpr uint32_t OPER = KSLABS * SLAB;        // one [128 keys x head slice] tile
    static constexpr uint32_t STAGE_BYTES = 2 * OPER;      // k raw -> k_hi in place | v raw
    static constexpr uint32_t VT_SLAB = D * 128;           // V^T: D channel rows x (32 keys = 128 B)
    static constexpr uint32_t VT_BYTES = (BKV / 32) * VT_SLAB;
    static constexpr uint32_t TILE_BYTES = STAGES * STAGE_BYTES + OPER + 2 * VT_BYTES;   // + k_lo + V^T hi + V^T lo
    static constexpr uint32_t AUX_BYTES = 64;              // mbarriers
    static size_t total(int pos_max) { return TILE_BYTES + AUX_BYTES + 2 * (2 * pos_max + 1) * 4 + 1024; }
};

// Ragged batches (Desc = mugd_attention_var): only the lk valid keys of the sample are scored.  Key tiles fully past lk are never
// loaded; in the last one the rows past lk (which the TMA box still brings in, NaN or not) are replaced by zeros before any MMA,
// exactly as the plain kernel zeroes keys past Lk.  Query rows past lq are written as zeros; a CTA of padded rows only writes its zeros.
template <int D, typename Desc = mugd_attention>
__global__ void __launch_bounds__(THREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV, const Desc d, float* dbg) {
    const mugd_attention& a = attn_desc(d);
    using S = Smem<D>;
    constexpr int STAGES = S::STAGES;
    constexpr int KD = D / 8;                               // k8 steps of S = Q K^T
    constexpr int NO = D / 2;                               // O accumulator registers per thread
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;           // SWIZZLE_128B operands need 1024-byte alignment
    auto k_hi = [&](int s) { return base + (uint32_t)s * S::STAGE_BYTES; };
    auto v_raw = [&](int s) { return base + (uint32_t)s * S::STAGE_BYTES + S::OPER; };
    const uint32_t k_lo = base + STAGES * S::STAGE_BYTES, vt_hi = k_lo + S::OPER, vt_lo = vt_hi + S::VT_BYTES;
    const uint32_t aux = base + S::TILE_BYTES;
    auto bar_full = [&](int s) { return aux + 8u * s; };
    float* rel = reinterpret_cast<float*>(smem_raw + (aux - raw) + 64);
    const int P = a.pos_max, NT = 2 * P + 1;
    float* cg = rel + NT;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g8 = lane >> 2, t4 = lane & 3;
    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * BQ;
    const int rq = (warp >> 2) * 64 + (warp & 3) * 16 + g8;  // this thread's query rows: rq, rq + 8 (tile-relative)
    const int qa = q0 + rq, qb = qa + 8;
    const int ntiles_all = (a.Lk + BKV - 1) / BKV;

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) mbar_init(bar_full(s), 1);
        mbar_init_fence();
    }
    __syncthreads();
    pdl_wait();
    const int lq = attn_rows(d, b, a.Lq), lk = attn_rows(d, b, a.Lk);
    const int ntiles = attn_is_var<Desc> ? (lk + BKV - 1) / BKV : ntiles_all;
    if constexpr (attn_is_var<Desc>) {
        if (q0 >= lq) {                                     // uniform over the CTA; no copy has been issued yet
            for (int t = tid; t < BQ * D; t += THREADS) {
                const int r = t / D, c = t - r * D;
                if (q0 + r < a.Lq) a.o[((int64_t)b * a.Lq + q0 + r) * a.ldo + h * D + c] = 0.f;
            }
            return;
        }
    }

    // raw K / V head slices of key tile t -> stage t % STAGES (keys >= Lk and channels >= H*D arrive as zeros)
    auto issue_tile = [&](int t) {
        const int s = t % STAGES;
        mbar_expect_tx(bar_full(s), 2u * S::OPER);
#pragma unroll
        for (int sl = 0; sl < S::KSLABS; ++sl) {
            tma_load_3d(k_hi(s) + sl * SLAB, &tmK, bar_full(s), h * D + sl * 32, t * BKV, b);
            tma_load_3d(v_raw(s) + sl * SLAB, &tmV, bar_full(s), h * D + sl * 32, t * BKV, b);
        }
    };
    if (warp == 0) {
        if (elect_one()) {
            issue_tile(0);
            if (STAGES > 1 && ntiles > 1) issue_tile(1);
        }
        __syncwarp();
    }
    for (int t = tid; t < NT; t += THREADS) {
        rel[t] = a.relpos[t * a.H + h] * a.scale;      // (s + rel) * scale == fma(s, scale, rel * scale) up to one rounding
        cg[t] = a.cgain[t * a.H + h];
    }
    // ---- Q rows -> q_hi / q_lo A fragments (a[0] row g col t, a[1] row g+8 col t, a[2] row g col t+4, a[3] row g+8 col t+4) ----
    uint32_t qhi[KD][4], qlo[KD][4];
    {
        const float* qpa = a.q + ((int64_t)b * a.Lq + qa) * a.ldq + h * D;
        const float* qpb = a.q + ((int64_t)b * a.Lq + qb) * a.ldq + h * D;
#pragma unroll
        for (int kk = 0; kk < KD; ++kk) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int c = kk * 8 + t4 + (e >> 1) * 4;
                const bool rb = e & 1;
                float x = 0.f;
                if ((rb ? qb : qa) < lq) x = (rb ? qpb : qpa)[c];
                const float hi = to_tf32(x);
                qhi[kk][e] = __float_as_uint(hi);
                qlo[kk][e] = __float_as_uint(to_tf32(x - hi));
            }
        }
    }
    float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f, o[NO];
#pragma unroll
    for (int c = 0; c < NO; ++c) o[c] = 0.f;

    for (int t = 0; t < ntiles; ++t) {
        const int s = t % STAGES;
        const int j0 = t * BKV;
        const int nk = min(BKV, lk - j0);
        mbar_wait(bar_full(s), (uint32_t)(t / STAGES) & 1u);
        // ---- key tile: raw -> k_hi in place, k_lo beside it (elementwise, so swizzle-agnostic); keys past Lk -> 0 -------------
        for (int f = tid; f < S::KSLABS * 1024; f += THREADS) {
            const int row = (f & 1023) >> 3;                // key within the tile
            float4 x = lds_f4(k_hi(s) + (uint32_t)f * 16u);
            if (row >= nk) x = make_float4(0.f, 0.f, 0.f, 0.f);
            float4 hi, lo;
            hi.x = to_tf32(x.x); hi.y = to_tf32(x.y); hi.z = to_tf32(x.z); hi.w = to_tf32(x.w);
            lo.x = to_tf32(x.x - hi.x); lo.y = to_tf32(x.y - hi.y); lo.z = to_tf32(x.z - hi.z); lo.w = to_tf32(x.w - hi.w);
            sts_f4(k_hi(s) + (uint32_t)f * 16u, hi);
            sts_f4(k_lo + (uint32_t)f * 16u, lo);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy smem writes -> visible to the tensor cores
        __syncthreads();
        // ---- S = Q K^T (asynchronous: the value tile is prepared meanwhile) ---------------------------------------------------
        float sacc[BKV / 2];
#pragma unroll
        for (int j = 0; j < BKV / 2; ++j) sacc[j] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < KD; ++kk) {
            const uint32_t so = (uint32_t)(kk >> 2) * SLAB;
            const uint64_t ko = (uint64_t)((kk & 3) * 2);          // 8 channels = 32 bytes = 2 x 16-byte units
            const uint64_t dh = wgmma_desc(k_hi(s) + so) + ko, dl = wgmma_desc(k_lo + so) + ko;
            Wgmma<BKV>::mma(sacc, qlo[kk], dh);
            Wgmma<BKV>::mma(sacc, qhi[kk], dl);
            Wgmma<BKV>::mma(sacc, qhi[kk], dh);
        }
        wgmma_commit();
        // ---- value tile: split + transpose into V^T (row = channel, 32-key slabs; keys of each 8-group stored 0 2 4 6 1 3 5 7).
        // One warp step = 32 keys x one 16-byte channel chunk: the reads hit 8 distinct swizzled chunks per quarter warp and the
        // 32 lanes of each scalar store fill one 128-byte row, so both sides are bank-conflict free.
        for (int it = warp; it < (BKV / 32) * (D / 4); it += THREADS / 32) {
            const int kg = it / (D / 4), c = it - kg * (D / 4);
            const int key = kg * 32 + lane;
            float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
            if (key < nk) x = lds_f4(v_raw(s) + (uint32_t)(c >> 3) * SLAB + (uint32_t)key * 128u + (uint32_t)(((c & 7) ^ (key & 7)) << 4));
            const float xs[4] = {x.x, x.y, x.z, x.w};
            const int kp = (lane & 24) | ((lane & 1) << 2) | ((lane & 7) >> 1);   // position of the key inside its 32-key slab row
            const uint32_t col = (uint32_t)kg * S::VT_SLAB + (uint32_t)((kp & 3) << 2);
            const int kc = kp >> 2;                         // 16-byte chunk of this key inside its 32-key slab row
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int d = c * 4 + j;
                const float hi = to_tf32(xs[j]), lo = to_tf32(xs[j] - hi);
                const uint32_t off = col + (uint32_t)d * 128u + (uint32_t)((kc ^ (d & 7)) << 4);
                sts_f1(vt_hi + off, hi);
                sts_f1(vt_lo + off, lo);
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // V^T writes -> visible to the P V MMAs (behind the barrier below)
        wgmma_wait<0>();
        if (dbg && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && t == 0) {       // logits 0..15 of row rq
            for (int j = 0; j < 4; ++j) dbg[rq * 40 + (j >> 1) * 8 + 2 * t4 + (j & 1)] = sacc[(j >> 1) * 4 + (j & 1)];
        }
        // ---- bias, scale, mask, online softmax (row rq: even/odd sacc of each quad, row rq + 8: the other two) ----------------
        float mxa = -INFINITY, mxb = -INFINITY;
#pragma unroll
        for (int j = 0; j < BKV / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int kj = j0 + j * 8 + 2 * t4 + (e & 1);
                const int qi = (e & 2) ? qb : qa;
                const int idx = max(-P, min(P, kj - qi)) + P;
                const float sc = (kj < lk) ? fmaf(sacc[4 * j + e], a.scale, rel[idx]) : -INFINITY;
                sacc[4 * j + e] = sc;
                if (e & 2) mxb = fmaxf(mxb, sc); else mxa = fmaxf(mxa, sc);
            }
        }
        mxa = fmaxf(mxa, __shfl_xor_sync(0xffffffffu, mxa, 1)); mxa = fmaxf(mxa, __shfl_xor_sync(0xffffffffu, mxa, 2));
        mxb = fmaxf(mxb, __shfl_xor_sync(0xffffffffu, mxb, 1)); mxb = fmaxf(mxb, __shfl_xor_sync(0xffffffffu, mxb, 2));
        const float mna = fmaxf(m_a, mxa), mnb = fmaxf(m_b, mxb);      // finite: key j0 is always valid
        const float ca = expf(m_a - mna), cb = expf(m_b - mnb);
        m_a = mna; m_b = mnb;
        l_a *= ca; l_b *= cb;
#pragma unroll
        for (int j = 0; j < NO / 4; ++j) { o[4 * j] *= ca; o[4 * j + 1] *= ca; o[4 * j + 2] *= cb; o[4 * j + 3] *= cb; }
        __syncthreads();                                    // V^T of this tile complete
        // ---- O += P V, in two halves of the key tile (half the P fragments live at a time) ---------------------------------------
        // P * gain as hi / lo A fragments of k8 chunk j: a[0] = (row g, key 2t) = sacc[4j], a[1] = (g+8, 2t) = sacc[4j+2],
        // a[2] = (g, 2t+1) = sacc[4j+1], a[3] = (g+8, 2t+1) = sacc[4j+3] -- V^T holds its keys in the matching order
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            if (half * (BKV / 2) >= nk) break;              // uniform: keys past the last one contribute zeros
            uint32_t phi[BKV / 16][4], plo[BKV / 16][4];
#pragma unroll
            for (int jj = 0; jj < BKV / 16; ++jj) {
                const int j = half * (BKV / 16) + jj;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int src = 4 * j + ((e & 1) << 1) + (e >> 1);
                    const bool rb = e & 1;
                    const int kj = j0 + j * 8 + 2 * t4 + (e >> 1);
                    const int qi = rb ? qb : qa;
                    const int idx = max(-P, min(P, kj - qi)) + P;
                    const float pe = expf(sacc[src] - (rb ? mnb : mna));       // 0 for masked keys
                    if (rb) l_b += pe; else l_a += pe;
                    const float pg = pe * cg[idx];
                    const float hi = to_tf32(pg);
                    phi[jj][e] = __float_as_uint(hi);
                    plo[jj][e] = __float_as_uint(to_tf32(pg - hi));
                }
            }
            wgmma_fence();
#pragma unroll
            for (int jj = 0; jj < BKV / 16; ++jj) {
                const int j = half * (BKV / 16) + jj;
                const uint32_t so = (uint32_t)(j >> 2) * S::VT_SLAB;
                const uint64_t ko = (uint64_t)((j & 3) * 2);       // 8 keys = 32 bytes = 2 x 16-byte units
                const uint64_t dh = wgmma_desc(vt_hi + so) + ko, dl = wgmma_desc(vt_lo + so) + ko;
                Wgmma<D>::mma(o, plo[jj], dh);
                Wgmma<D>::mma(o, phi[jj], dl);
                Wgmma<D>::mma(o, phi[jj], dh);
            }
            wgmma_commit();
            wgmma_wait<0>();
        }
        __syncthreads();                                    // every MMA that read stage s, k_lo and V^T has retired
        if (warp == 0 && t + STAGES < ntiles) {
            if (elect_one()) issue_tile(t + STAGES);
            __syncwarp();
        }
    }
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 1); l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 1); l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
    const float ia = 1.0f / l_a, ib = 1.0f / l_b;
    float* opa = a.o + ((int64_t)b * a.Lq + qa) * a.ldo + h * D;
    float* opb = a.o + ((int64_t)b * a.Lq + qb) * a.ldo + h * D;
#pragma unroll
    for (int j = 0; j < NO / 4; ++j) {
        const int c = j * 8 + 2 * t4;
        if (qa < a.Lq) *reinterpret_cast<float2*>(opa + c) = qa < lq ? make_float2(o[4 * j] * ia, o[4 * j + 1] * ia) : make_float2(0.f, 0.f);
        if (qb < a.Lq) *reinterpret_cast<float2*>(opb + c) = qb < lq ? make_float2(o[4 * j + 2] * ib, o[4 * j + 3] * ib) : make_float2(0.f, 0.f);
    }
}

// (channel, key, sample) view of a [B*Lk, ld] row-major buffer whose first H*D columns are the head slices
static int encode_kv(CUtensorMap* tm, const float* p, int64_t ld, int cols, int Lk, int B) {
    const cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)Lk, (cuuint64_t)B};
    const cuuint64_t strides[2] = {(cuuint64_t)ld * 4, (cuuint64_t)Lk * (cuuint64_t)ld * 4};
    const cuuint32_t box[3] = {32, (cuuint32_t)BKV, 1};
    return encode_f32_tma(tm, p, 3, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "attention_tc");
}

static float* g_dbg = nullptr;      // debugging aid: CTA (0,0,0) dumps the raw logits of its first key tile (16 of each row's 40 floats)

template <int D, typename Desc>
static int launch(const Desc& d, cudaStream_t st) {
    const mugd_attention& a = attn_desc(d);
    CUtensorMap tmK, tmV;
    int rc = encode_kv(&tmK, a.k, a.ldk, a.H * D, a.Lk, a.B);
    if (rc != MUGD_OK) return rc;
    rc = encode_kv(&tmV, a.v, a.ldv, a.H * D, a.Lk, a.B);
    if (rc != MUGD_OK) return rc;
    const size_t bytes = Smem<D>::total(a.pos_max);
    dim3 grid((a.Lq + BQ - 1) / BQ, a.H, a.B);
    MUGD_CHECK_CUDA(launch_k(attention_tc_kernel<D, Desc>, grid, dim3(THREADS), bytes, st, tmK, tmV, d, g_dbg));
    return MUGD_OK;
}

}  // namespace atc

cudaError_t attention_tc_allow_smem(int bytes) {
    return allow_dynamic_smem(bytes, atc::attention_tc_kernel<32>, atc::attention_tc_kernel<48>, atc::attention_tc_kernel<64>,
                              atc::attention_tc_kernel<32, mugd_attention_var>, atc::attention_tc_kernel<48, mugd_attention_var>,
                              atc::attention_tc_kernel<64, mugd_attention_var>);
}

int launch_attention_tc(const DeviceInfo&, const mugd_attention& a, cudaStream_t st) {
    return (a.D == 32) ? atc::launch<32>(a, st) : (a.D == 48) ? atc::launch<48>(a, st) : atc::launch<64>(a, st);
}

int launch_attention_tc(const DeviceInfo&, const mugd_attention_var& v, cudaStream_t st) {
    const int D = v.attn.D;
    return (D == 32) ? atc::launch<32>(v, st) : (D == 48) ? atc::launch<48>(v, st) : atc::launch<64>(v, st);
}

}  // namespace mugd

extern "C" int mugd_debug_set_attention_dump(float* buf) {
    mugd::atc::g_dbg = buf;
    return MUGD_OK;
}

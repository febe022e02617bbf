// Attention of mug/model/attention.py:91-126 (CrossAttention.forward), fp32, flash-style (no [Lq,Lk]
// matrix in memory):
//     idx_ij = clamp(j - i, -P, P) + P
//     s_ij   = (q_i . k_j + relpos[idx_ij, h]) * scale
//     o_i    = sum_j softmax_j(s_i)_j * cgain[idx_ij, h] * v_j
// The post-softmax gain multiplies the numerator only; the softmax denominator accumulates plain p.
// Self attention (Lk = Lq) and cross attention to the 21 prompt tokens (Lk = 21) share the kernel.
//
// Register-tiled FFMA formulation: a CTA of 256 threads (16 x 16) owns 64 queries of one (sample, head) and
// streams 64-key tiles.  S = Q K^T is a 64x64xD smem-tiled product with 4x4 micro-tiles (operands stored
// k-major so both are read as conflict-free float4), the online softmax runs on the micro-tile with
// 16-lane shuffle reductions, P*gain goes back to shared memory transposed, and O += P V is a second
// 64 x D x 64 product.  Exact fp32 (expf, IEEE division): this is 2.6 % of the FLOPs, the parity-critical
// part (non-standard bias + gain) rather than the fast part of the network.
#include "common.cuh"

#include <math.h>

namespace mugd {

constexpr int AT_BQ = 64;
constexpr int AT_BK = 64;
constexpr int AT_PAD = 4;
constexpr int AT_THREADS = 256;

template <int D>
struct AttSmem {
    static constexpr int QT = D * (AT_BQ + AT_PAD);
    static constexpr int KT = D * (AT_BK + AT_PAD);
    static constexpr int VS = AT_BK * D;
    static constexpr int PT = AT_BK * (AT_BQ + AT_PAD);
    static constexpr int FLOATS = QT + KT + VS + PT;
};

// the section slot of query row i of sample b: the number of slots 1 .. 7 whose start is at or before i (unused slots hold Lq)
__device__ __forceinline__ int attn_section(const mugd_attention_sec& d, int b, int i) {
    const int32_t* st = d.starts + MUGD_SECTIONS * b;
    int s = 0;
#pragma unroll
    for (int t = 1; t < MUGD_SECTIONS; ++t) s += st[t] <= i;
    return s;
}

// The key-tile loop and the store of attention_kernel, for the section kernel (attention_kernel keeps its own copy, so the plain and
// ragged instances compile to the code they had before sections existed): rows q0 .. q0 + AT_BQ - 1 of (b, h) against keys kb / vb (lk of them) with Qt,
// rel and cg staged; rows for which store_ok(row) is false are computed and not stored.
template <int D, typename StoreOk>
__device__ __forceinline__ void attention_tiles(const mugd_attention& a, float* Qt, float* Kt, float* Vs, float* Pt, const float* rel,
                                                const float* cg, const float* kb, const float* vb, int b, int h, int q0, int lq, int lk,
                                                int tid, int tx, int ty, StoreOk store_ok) {
    constexpr int DC = D / 16;
    constexpr int SQ = AT_BQ + AT_PAD, SK = AT_BK + AT_PAD;
    constexpr int QD = D / 4;
    const int P = a.pos_max;
    float m_i[4], l_i[4], o[4][DC];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        m_i[i] = -INFINITY; l_i[i] = 0.f;
#pragma unroll
        for (int c = 0; c < DC; ++c) o[i][c] = 0.f;
    }

    for (int j0 = 0; j0 < lk; j0 += AT_BK) {
        __syncthreads();                       // previous tile consumed (first pass: Qt / tables written)
        for (int t = tid; t < AT_BK * QD; t += AT_THREADS) {
            const int r = t / QD, c = (t - r * QD) * 4;
            float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
            if (j0 + r < lk) {
                kv = ld_f4(kb + (int64_t)(j0 + r) * a.ldk + c);
                vv = ld_f4(vb + (int64_t)(j0 + r) * a.ldv + c);
            }
            Kt[(c + 0) * SK + r] = kv.x; Kt[(c + 1) * SK + r] = kv.y; Kt[(c + 2) * SK + r] = kv.z; Kt[(c + 3) * SK + r] = kv.w;
            *reinterpret_cast<float4*>(&Vs[r * D + c]) = vv;
        }
        __syncthreads();
        // ---- S = Q K^T on a 4x4 micro-tile ---------------------------------------------------------------
        float s[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 8
        for (int kk = 0; kk < D; ++kk) {
            const float4 qa = *reinterpret_cast<const float4*>(&Qt[kk * SQ + ty * 4]);
            const float4 kv = *reinterpret_cast<const float4*>(&Kt[kk * SK + tx * 4]);
            const float qf[4] = {qa.x, qa.y, qa.z, qa.w}, kf[4] = {kv.x, kv.y, kv.z, kv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) s[i][j] = fmaf(qf[i], kf[j], s[i][j]);
        }
        // ---- bias, scale, mask, online softmax ------------------------------------------------------------
        float pc[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int qi = q0 + ty * 4 + i;
            float mx = -INFINITY;
            int idx[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int kj = j0 + tx * 4 + j;
                idx[j] = max(-P, min(P, kj - qi)) + P;
                s[i][j] = (kj < lk) ? (s[i][j] + rel[idx[j]]) * a.scale : -INFINITY;
                mx = fmaxf(mx, s[i][j]);
            }
#pragma unroll
            for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
            const float mnew = fmaxf(m_i[i], mx);          // finite: column j0 of every tile is a valid key
            const float corr = expf(m_i[i] - mnew);
            float rs = 0.f;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float pe = expf(s[i][j] - mnew);      // 0 for masked keys
                rs += pe;
                pc[i][j] = pe * cg[idx[j]];
            }
#pragma unroll
            for (int off = 8; off > 0; off >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, off);
            l_i[i] = l_i[i] * corr + rs;
            m_i[i] = mnew;
#pragma unroll
            for (int c = 0; c < DC; ++c) o[i][c] *= corr;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j)
            *reinterpret_cast<float4*>(&Pt[(tx * 4 + j) * SQ + ty * 4]) = make_float4(pc[0][j], pc[1][j], pc[2][j], pc[3][j]);
        __syncthreads();
        // ---- O += P V ----------------------------------------------------------------------------------------
        const int nk = min(AT_BK, lk - j0);
#pragma unroll 4
        for (int kk = 0; kk < nk; ++kk) {
            const float4 pa = *reinterpret_cast<const float4*>(&Pt[kk * SQ + ty * 4]);
            const float pf[4] = {pa.x, pa.y, pa.z, pa.w};
            float vf[DC];
#pragma unroll
            for (int c = 0; c < DC; ++c) vf[c] = Vs[kk * D + tx * DC + c];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int c = 0; c < DC; ++c) o[i][c] = fmaf(pf[i], vf[c], o[i][c]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int qi = q0 + ty * 4 + i;
        if (qi < a.Lq && store_ok(qi)) {
            const float inv = 1.0f / l_i[i];
            float* op = a.o + ((int64_t)b * a.Lq + qi) * a.ldo + h * D + tx * DC;
#pragma unroll
            for (int c = 0; c < DC; ++c) op[c] = qi < lq ? o[i][c] * inv : 0.f;
        }
    }
}

// Padded rows of a ragged batch (Desc = mugd_attention_var): keys j >= lk are neither read nor scored, query rows i >= lq are
// written as zeros, and a CTA whose rows are all padding only writes its zeros.
template <int D, typename Desc = mugd_attention>
__global__ void __launch_bounds__(AT_THREADS)
attention_kernel(const Desc d) {
    const mugd_attention& a = attn_desc(d);
    constexpr int DC = D / 16;                 // output columns per thread
    constexpr int SQ = AT_BQ + AT_PAD, SK = AT_BK + AT_PAD;
    extern __shared__ __align__(16) float sm[];
    float* Qt = sm;                            // [D][SQ]   Qt[k][row]
    float* Kt = Qt + AttSmem<D>::QT;           // [D][SK]   Kt[k][col]
    float* Vs = Kt + AttSmem<D>::KT;           // [BK][D]
    float* Pt = Vs + AttSmem<D>::VS;           // [BK][SQ]  Pt[key][row] = p * gain
    float* rel = Pt + AttSmem<D>::PT;          // [2P+1]
    const int P = a.pos_max, NT = 2 * P + 1;
    float* cg = rel + NT;

    pdl_wait();
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int b = blockIdx.z, h = blockIdx.y;
    const int q0 = blockIdx.x * AT_BQ;
    const int lq = attn_rows(d, b, a.Lq), lk = attn_rows(d, b, a.Lk);
    if constexpr (attn_is_var<Desc>) {
        if (q0 >= lq) {
            for (int t = tid; t < AT_BQ * D; t += AT_THREADS) {
                const int r = t / D, c = t - r * D;
                if (q0 + r < a.Lq) a.o[((int64_t)b * a.Lq + q0 + r) * a.ldo + h * D + c] = 0.f;
            }
            return;
        }
    }
    for (int t = tid; t < NT; t += AT_THREADS) {
        rel[t] = a.relpos[t * a.H + h];
        cg[t] = a.cgain[t * a.H + h];
    }
    constexpr int QD = D / 4;
    {
        const float* qb = a.q + (int64_t)b * a.Lq * a.ldq + h * D;
        for (int t = tid; t < AT_BQ * QD; t += AT_THREADS) {
            const int r = t / QD, c = (t - r * QD) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (q0 + r < lq) v = ld_f4(qb + (int64_t)(q0 + r) * a.ldq + c);
            Qt[(c + 0) * SQ + r] = v.x; Qt[(c + 1) * SQ + r] = v.y; Qt[(c + 2) * SQ + r] = v.z; Qt[(c + 3) * SQ + r] = v.w;
        }
    }
    float m_i[4], l_i[4], o[4][DC];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        m_i[i] = -INFINITY; l_i[i] = 0.f;
#pragma unroll
        for (int c = 0; c < DC; ++c) o[i][c] = 0.f;
    }
    const float* kb = a.k + (int64_t)b * a.Lk * a.ldk + h * D;
    const float* vb = a.v + (int64_t)b * a.Lk * a.ldv + h * D;

    for (int j0 = 0; j0 < lk; j0 += AT_BK) {
        __syncthreads();                       // previous tile consumed (first pass: Qt / tables written)
        for (int t = tid; t < AT_BK * QD; t += AT_THREADS) {
            const int r = t / QD, c = (t - r * QD) * 4;
            float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
            if (j0 + r < lk) {
                kv = ld_f4(kb + (int64_t)(j0 + r) * a.ldk + c);
                vv = ld_f4(vb + (int64_t)(j0 + r) * a.ldv + c);
            }
            Kt[(c + 0) * SK + r] = kv.x; Kt[(c + 1) * SK + r] = kv.y; Kt[(c + 2) * SK + r] = kv.z; Kt[(c + 3) * SK + r] = kv.w;
            *reinterpret_cast<float4*>(&Vs[r * D + c]) = vv;
        }
        __syncthreads();
        // ---- S = Q K^T on a 4x4 micro-tile ---------------------------------------------------------------
        float s[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 8
        for (int kk = 0; kk < D; ++kk) {
            const float4 qa = *reinterpret_cast<const float4*>(&Qt[kk * SQ + ty * 4]);
            const float4 kv = *reinterpret_cast<const float4*>(&Kt[kk * SK + tx * 4]);
            const float qf[4] = {qa.x, qa.y, qa.z, qa.w}, kf[4] = {kv.x, kv.y, kv.z, kv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) s[i][j] = fmaf(qf[i], kf[j], s[i][j]);
        }
        // ---- bias, scale, mask, online softmax ------------------------------------------------------------
        float pc[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int qi = q0 + ty * 4 + i;
            float mx = -INFINITY;
            int idx[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int kj = j0 + tx * 4 + j;
                idx[j] = max(-P, min(P, kj - qi)) + P;
                s[i][j] = (kj < lk) ? (s[i][j] + rel[idx[j]]) * a.scale : -INFINITY;
                mx = fmaxf(mx, s[i][j]);
            }
#pragma unroll
            for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
            const float mnew = fmaxf(m_i[i], mx);          // finite: column j0 of every tile is a valid key
            const float corr = expf(m_i[i] - mnew);
            float rs = 0.f;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float pe = expf(s[i][j] - mnew);      // 0 for masked keys
                rs += pe;
                pc[i][j] = pe * cg[idx[j]];
            }
#pragma unroll
            for (int off = 8; off > 0; off >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, off);
            l_i[i] = l_i[i] * corr + rs;
            m_i[i] = mnew;
#pragma unroll
            for (int c = 0; c < DC; ++c) o[i][c] *= corr;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j)
            *reinterpret_cast<float4*>(&Pt[(tx * 4 + j) * SQ + ty * 4]) = make_float4(pc[0][j], pc[1][j], pc[2][j], pc[3][j]);
        __syncthreads();
        // ---- O += P V ----------------------------------------------------------------------------------------
        const int nk = min(AT_BK, lk - j0);
#pragma unroll 4
        for (int kk = 0; kk < nk; ++kk) {
            const float4 pa = *reinterpret_cast<const float4*>(&Pt[kk * SQ + ty * 4]);
            const float pf[4] = {pa.x, pa.y, pa.z, pa.w};
            float vf[DC];
#pragma unroll
            for (int c = 0; c < DC; ++c) vf[c] = Vs[kk * D + tx * DC + c];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int c = 0; c < DC; ++c) o[i][c] = fmaf(pf[i], vf[c], o[i][c]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int qi = q0 + ty * 4 + i;
        if (qi < a.Lq) {
            const float inv = 1.0f / l_i[i];
            float* op = a.o + ((int64_t)b * a.Lq + qi) * a.ldo + h * D + tx * DC;
#pragma unroll
            for (int c = 0; c < DC; ++c) op[c] = qi < lq ? o[i][c] * inv : 0.f;
        }
    }
}

// Section prompts (mugd_attention_sec): the CTA's rows run once per section slot they fall in, against that slot's keys, and each
// row is stored from the pass of its own slot.  A CTA inside one section makes one pass, as attention_kernel does.
template <int D>
__global__ void __launch_bounds__(AT_THREADS, 1)
attention_sec_kernel(const mugd_attention_sec d) {
    const mugd_attention& a = d.attn;
    constexpr int SQ = AT_BQ + AT_PAD;
    extern __shared__ __align__(16) float sm[];
    float* Qt = sm;
    float* Kt = Qt + AttSmem<D>::QT;
    float* Vs = Kt + AttSmem<D>::KT;
    float* Pt = Vs + AttSmem<D>::VS;
    float* rel = Pt + AttSmem<D>::PT;
    const int P = a.pos_max, NT = 2 * P + 1;
    float* cg = rel + NT;

    pdl_wait();
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int b = blockIdx.z, h = blockIdx.y;
    const int q0 = blockIdx.x * AT_BQ;
    for (int t = tid; t < NT; t += AT_THREADS) {
        rel[t] = a.relpos[t * a.H + h];
        cg[t] = a.cgain[t * a.H + h];
    }
    constexpr int QD = D / 4;
    {
        const float* qb = a.q + (int64_t)b * a.Lq * a.ldq + h * D;
        for (int t = tid; t < AT_BQ * QD; t += AT_THREADS) {
            const int r = t / QD, c = (t - r * QD) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (q0 + r < a.Lq) v = ld_f4(qb + (int64_t)(q0 + r) * a.ldq + c);
            Qt[(c + 0) * SQ + r] = v.x; Qt[(c + 1) * SQ + r] = v.y; Qt[(c + 2) * SQ + r] = v.z; Qt[(c + 3) * SQ + r] = v.w;
        }
    }
    const int last = attn_section(d, b, min(q0 + AT_BQ, a.Lq) - 1);
#pragma unroll 1
    for (int sec = attn_section(d, b, q0); sec <= last; ++sec) {
        const int64_t row0 = (int64_t)(MUGD_SECTIONS * b + sec) * d.sec_stride;
        // attention_tiles opens every key tile with a barrier, so the previous pass is consumed before this one stages keys
        attention_tiles<D>(a, Qt, Kt, Vs, Pt, rel, cg, a.k + row0 * a.ldk + h * D, a.v + row0 * a.ldv + h * D, b, h, q0, a.Lq, a.Lk,
                           tid, tx, ty, [&](int qi) { return attn_section(d, b, qi) == sec; });
    }
}

template <int D, typename Desc>
static int attention_launch(const Desc& d, cudaStream_t st) {
    const mugd_attention& a = attn_desc(d);
    const size_t bytes = sizeof(float) * (AttSmem<D>::FLOATS + 2 * (2 * a.pos_max + 1));
    dim3 grid((a.Lq + AT_BQ - 1) / AT_BQ, a.H, a.B);
    MUGD_CHECK_CUDA(launch_k(attention_kernel<D, Desc>, grid, dim3(AT_THREADS), bytes, st, d));
    return MUGD_OK;
}

// =====================================================================================================
// Few keys (Lk <= 32): the cross attention to the 21 prompt tokens, 16 of the 32 attention launches of an evaluation.
// A 128-key tensor-core tile would be 5/6 zero fill behind a fixed cost (barriers, TMA, operand splits);
// here ONE LANE OWNS ONE KEY: lane j keeps k_j in registers, a warp takes four query rows at a time (four independent dependency
// chains) -- the rows are read back from shared memory as broadcast float4s for the D-long dot products, max / sum are warp shuffles, and for O = (P*gain) V lane d owns output
// channels d, d+32 and receives p_j from lane j by shuffle.  Exact fp32, same formula order as the FFMA referee above.
// =====================================================================================================
constexpr int ASK_WARPS = 8;
constexpr int ASK_RW = 4;         // query rows a warp carries together
constexpr int ASK_ROWS = ASK_WARPS * ASK_RW;      // query rows per CTA

// The K / V fill of attention_smallk_kernel, for the section kernel (attention_smallk_kernel keeps its own copy, as above): the (at most 32) keys at kb / vb into Ks [32][D + 1] and Vs [32][D], zeros past lk.
template <int D>
__device__ __forceinline__ void smallk_stage_kv(const mugd_attention& a, const float* kb, const float* vb, int lk, float* Ks, float* Vs,
                                                int tid) {
    constexpr int KP = D + 1;
    constexpr int QD = D / 4;
    for (int t = tid; t < 32 * QD; t += ASK_WARPS * 32) {
        const int r = t / QD, c = (t - r * QD) * 4;
        float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
        if (r < lk) {
            kv = ld_f4(kb + (int64_t)r * a.ldk + c);
            vv = ld_f4(vb + (int64_t)r * a.ldv + c);
        }
        Ks[r * KP + c] = kv.x; Ks[r * KP + c + 1] = kv.y; Ks[r * KP + c + 2] = kv.z; Ks[r * KP + c + 3] = kv.w;
        *reinterpret_cast<float4*>(&Vs[r * D + c]) = vv;
    }
}

// The rows of attention_smallk_kernel, for the section kernel: the warp's ASK_RW query rows from qbase (staged in qrows) against the staged keys; rows for which
// store_ok(row) is false are computed and not stored.  Uniform over the warp (shuffles over all 32 lanes).
template <int D, typename StoreOk>
__device__ __forceinline__ void smallk_rows(const mugd_attention& a, const float* Ks, const float* Vs, const float* qrows, int lane, int b,
                                            int h, int qbase, int lq, int lk, bool key_ok, const float* relv, const float* cgv,
                                            StoreOk store_ok) {
    constexpr int DV = (D + 31) / 32;
    constexpr int KP = D + 1;
    constexpr int QD = D / 4;
    float kreg[D];
#pragma unroll
    for (int d = 0; d < D; ++d) kreg[d] = Ks[lane * KP + d];
    float s[ASK_RW];
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i) s[i] = 0.f;
#pragma unroll
    for (int c = 0; c < QD; ++c) {
#pragma unroll
        for (int i = 0; i < ASK_RW; ++i) {
            const float4 qv = *reinterpret_cast<const float4*>(&qrows[i * D + c * 4]);       // broadcast
            s[i] = fmaf(qv.x, kreg[c * 4], s[i]); s[i] = fmaf(qv.y, kreg[c * 4 + 1], s[i]);
            s[i] = fmaf(qv.z, kreg[c * 4 + 2], s[i]); s[i] = fmaf(qv.w, kreg[c * 4 + 3], s[i]);
        }
    }
    float mx[ASK_RW], pe[ASK_RW], sum[ASK_RW], pg[ASK_RW];
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i) {
        s[i] = key_ok ? (s[i] + relv[i]) * a.scale : -INFINITY;
        mx[i] = s[i];
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
#pragma unroll
        for (int i = 0; i < ASK_RW; ++i) mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], off));
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i) { pe[i] = expf(s[i] - mx[i]); sum[i] = pe[i]; pg[i] = pe[i] * cgv[i]; }   // pe = 0 for lanes without a key
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
#pragma unroll
        for (int i = 0; i < ASK_RW; ++i) sum[i] += __shfl_xor_sync(0xffffffffu, sum[i], off);
    float o[ASK_RW][DV];
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i)
#pragma unroll
        for (int c = 0; c < DV; ++c) o[i][c] = 0.f;
    for (int j = 0; j < lk; ++j) {
        float vj[DV];
#pragma unroll
        for (int c = 0; c < DV; ++c) vj[c] = (lane + c * 32 < D) ? Vs[j * D + lane + c * 32] : 0.f;
#pragma unroll
        for (int i = 0; i < ASK_RW; ++i) {
            const float pj = __shfl_sync(0xffffffffu, pg[i], j);
#pragma unroll
            for (int c = 0; c < DV; ++c) o[i][c] = fmaf(pj, vj[c], o[i][c]);
        }
    }
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i) {
        const int qi = qbase + i;
        if (qi < a.Lq && store_ok(qi)) {
            const float inv = 1.0f / sum[i];
            float* op = a.o + ((int64_t)b * a.Lq + qi) * a.ldo + h * D;
#pragma unroll
            for (int c = 0; c < DV; ++c)
                if (lane + c * 32 < D) op[lane + c * 32] = qi < lq ? o[i][c] * inv : 0.f;
        }
    }
}

template <int D, typename Desc = mugd_attention>
__global__ void __launch_bounds__(ASK_WARPS * 32)
attention_smallk_kernel(const Desc d) {
    const mugd_attention& a = attn_desc(d);
    constexpr int DV = (D + 31) / 32;                 // output channels per lane
    constexpr int KP = D + 1;                         // K row pitch: lane j reads row j, the odd pitch keeps the lanes on distinct banks
    constexpr int QD = D / 4;
    extern __shared__ __align__(16) float sm[];
    float* Ks = sm;                                   // [32][KP]
    float* Vs = Ks + 32 * KP;                         // [32][D]
    float* Qs = Vs + 32 * D;                          // [ASK_ROWS][D]
    pdl_wait();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * ASK_ROWS;
    const int P = a.pos_max;
    const int qbase = q0 + warp * ASK_RW;             // the warp's ASK_RW query rows go through the kernel together
    const int lq = attn_rows(d, b, a.Lq), lk = attn_rows(d, b, a.Lk);
    if constexpr (attn_is_var<Desc>) {              // a CTA of padded rows only: zeros (uniform over the CTA, before any barrier)
        if (q0 >= lq) {
            for (int t = tid; t < ASK_ROWS * D; t += ASK_WARPS * 32) {
                const int r = t / D, c = t - r * D;
                if (q0 + r < a.Lq) a.o[((int64_t)b * a.Lq + q0 + r) * a.ldo + h * D + c] = 0.f;
            }
            return;
        }
    }
    const bool key_ok = lane < lk;
    // everything this thread needs from global memory is requested up front, in one round trip with the K / V fill: its slice of
    // the warp's query rows and the bias / gain of (its key, each row) -- 2 x ASK_RW table entries, not the whole 2P+1 table
    float qpre[ASK_RW][DV], relv[ASK_RW], cgv[ASK_RW];
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i) {
        const int qi = min(qbase + i, a.Lq - 1);      // rows past the end recompute the last row (never stored)
        const float* qp = a.q + ((int64_t)b * a.Lq + qi) * a.ldq + h * D;
#pragma unroll
        for (int c = 0; c < DV; ++c) qpre[i][c] = (lane + c * 32 < D) ? qp[lane + c * 32] : 0.f;
        const int idx = max(-P, min(P, lane - (qbase + i))) + P;
        relv[i] = a.relpos[idx * a.H + h];
        cgv[i] = a.cgain[idx * a.H + h];
    }
    const float* kb = a.k + (int64_t)b * a.Lk * a.ldk + h * D;
    const float* vb = a.v + (int64_t)b * a.Lk * a.ldv + h * D;
    for (int t = tid; t < 32 * QD; t += ASK_WARPS * 32) {
        const int r = t / QD, c = (t - r * QD) * 4;
        float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
        if (r < lk) {
            kv = ld_f4(kb + (int64_t)r * a.ldk + c);
            vv = ld_f4(vb + (int64_t)r * a.ldv + c);
        }
        Ks[r * KP + c] = kv.x; Ks[r * KP + c + 1] = kv.y; Ks[r * KP + c + 2] = kv.z; Ks[r * KP + c + 3] = kv.w;
        *reinterpret_cast<float4*>(&Vs[r * D + c]) = vv;
    }
    float* qrows = Qs + warp * ASK_RW * D;
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i)
#pragma unroll
        for (int c = 0; c < DV; ++c)
            if (lane + c * 32 < D) qrows[i * D + lane + c * 32] = qpre[i][c];
    __syncthreads();
    if (qbase >= a.Lq) return;                        // uniform over the warp; no barrier follows
    float kreg[D];
#pragma unroll
    for (int d = 0; d < D; ++d) kreg[d] = Ks[lane * KP + d];
    float s[ASK_RW];
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i) s[i] = 0.f;
#pragma unroll
    for (int c = 0; c < QD; ++c) {
#pragma unroll
        for (int i = 0; i < ASK_RW; ++i) {
            const float4 qv = *reinterpret_cast<const float4*>(&qrows[i * D + c * 4]);       // broadcast
            s[i] = fmaf(qv.x, kreg[c * 4], s[i]); s[i] = fmaf(qv.y, kreg[c * 4 + 1], s[i]);
            s[i] = fmaf(qv.z, kreg[c * 4 + 2], s[i]); s[i] = fmaf(qv.w, kreg[c * 4 + 3], s[i]);
        }
    }
    float mx[ASK_RW], pe[ASK_RW], sum[ASK_RW], pg[ASK_RW];
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i) {
        s[i] = key_ok ? (s[i] + relv[i]) * a.scale : -INFINITY;
        mx[i] = s[i];
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
#pragma unroll
        for (int i = 0; i < ASK_RW; ++i) mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], off));
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i) { pe[i] = expf(s[i] - mx[i]); sum[i] = pe[i]; pg[i] = pe[i] * cgv[i]; }   // pe = 0 for lanes without a key
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
#pragma unroll
        for (int i = 0; i < ASK_RW; ++i) sum[i] += __shfl_xor_sync(0xffffffffu, sum[i], off);
    float o[ASK_RW][DV];
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i)
#pragma unroll
        for (int c = 0; c < DV; ++c) o[i][c] = 0.f;
    for (int j = 0; j < lk; ++j) {
        float vj[DV];
#pragma unroll
        for (int c = 0; c < DV; ++c) vj[c] = (lane + c * 32 < D) ? Vs[j * D + lane + c * 32] : 0.f;
#pragma unroll
        for (int i = 0; i < ASK_RW; ++i) {
            const float pj = __shfl_sync(0xffffffffu, pg[i], j);
#pragma unroll
            for (int c = 0; c < DV; ++c) o[i][c] = fmaf(pj, vj[c], o[i][c]);
        }
    }
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i) {
        const int qi = qbase + i;
        if (qi < a.Lq) {
            const float inv = 1.0f / sum[i];
            float* op = a.o + ((int64_t)b * a.Lq + qi) * a.ldo + h * D;
#pragma unroll
            for (int c = 0; c < DV; ++c)
                if (lane + c * 32 < D) op[lane + c * 32] = qi < lq ? o[i][c] * inv : 0.f;
        }
    }
}

// Section prompts (mugd_attention_sec): one pass per section slot the CTA's rows fall in, each staging that slot's keys; a warp takes
// part in the passes of its rows' slots and stores each row from the pass of its own slot.  A CTA inside one section makes one pass,
// as attention_smallk_kernel does.
template <int D>
__global__ void __launch_bounds__(ASK_WARPS * 32)
attention_smallk_sec_kernel(const mugd_attention_sec d) {
    const mugd_attention& a = d.attn;
    constexpr int DV = (D + 31) / 32;
    constexpr int KP = D + 1;
    extern __shared__ __align__(16) float sm[];
    float* Ks = sm;
    float* Vs = Ks + 32 * KP;
    float* Qs = Vs + 32 * D;
    pdl_wait();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * ASK_ROWS;
    const int P = a.pos_max;
    const int qbase = q0 + warp * ASK_RW;
    const bool key_ok = lane < a.Lk;
    float qpre[ASK_RW][DV], relv[ASK_RW], cgv[ASK_RW];
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i) {
        const int qi = min(qbase + i, a.Lq - 1);
        const float* qp = a.q + ((int64_t)b * a.Lq + qi) * a.ldq + h * D;
#pragma unroll
        for (int c = 0; c < DV; ++c) qpre[i][c] = (lane + c * 32 < D) ? qp[lane + c * 32] : 0.f;
        const int idx = max(-P, min(P, lane - (qbase + i))) + P;
        relv[i] = a.relpos[idx * a.H + h];
        cgv[i] = a.cgain[idx * a.H + h];
    }
    float* qrows = Qs + warp * ASK_RW * D;
#pragma unroll
    for (int i = 0; i < ASK_RW; ++i)
#pragma unroll
        for (int c = 0; c < DV; ++c)
            if (lane + c * 32 < D) qrows[i * D + lane + c * 32] = qpre[i][c];
    const int first = attn_section(d, b, q0), last = attn_section(d, b, min(q0 + ASK_ROWS, a.Lq) - 1);
    // the warp's rows span slots w_first .. w_last (uniform over the warp)
    const int w_first = qbase < a.Lq ? attn_section(d, b, qbase) : MUGD_SECTIONS;
    const int w_last = qbase < a.Lq ? attn_section(d, b, min(qbase + ASK_RW, a.Lq) - 1) : -1;
    for (int sec = first; sec <= last; ++sec) {
        if (sec > first) __syncthreads();             // the previous slot's keys consumed
        const int64_t row0 = (int64_t)(MUGD_SECTIONS * b + sec) * d.sec_stride;
        smallk_stage_kv<D>(a, a.k + row0 * a.ldk + h * D, a.v + row0 * a.ldv + h * D, a.Lk, Ks, Vs, tid);
        __syncthreads();
        if (w_first <= sec && sec <= w_last)
            smallk_rows<D>(a, Ks, Vs, qrows, lane, b, h, qbase, a.Lq, a.Lk, key_ok, relv, cgv,
                           [&](int qi) { return attn_section(d, b, qi) == sec; });
    }
}

template <int D, typename Desc>
static int attention_smallk_launch(const Desc& d, cudaStream_t st) {
    const mugd_attention& a = attn_desc(d);
    const size_t bytes = sizeof(float) * (32 * (D + 1) + 32 * D + ASK_ROWS * D + 4);
    dim3 grid((a.Lq + ASK_ROWS - 1) / ASK_ROWS, a.H, a.B);      // (more rows per CTA -- fewer re-reads of K / V -- measured slower)
    MUGD_CHECK_CUDA(launch_k(attention_smallk_kernel<D, Desc>, grid, dim3(ASK_WARPS * 32), bytes, st, d));
    return MUGD_OK;
}

cudaError_t attention_allow_smem(int bytes) {
    return allow_dynamic_smem(bytes, attention_kernel<32>, attention_kernel<48>, attention_kernel<64>,
                              attention_kernel<32, mugd_attention_var>, attention_kernel<48, mugd_attention_var>,
                              attention_kernel<64, mugd_attention_var>, attention_sec_kernel<32>, attention_sec_kernel<48>,
                              attention_sec_kernel<64>);
}

int launch_attention_tc(const DeviceInfo& dev, const mugd_attention& a, cudaStream_t st);       // attention_tc.cu
int launch_attention_tc(const DeviceInfo& dev, const mugd_attention_var& a, cudaStream_t st);

static int check_attention(const mugd_attention& a) {
    MUGD_REQUIRE(a.B > 0 && a.H > 0 && a.Lq > 0 && a.Lk > 0, "attention: empty shape");
    MUGD_REQUIRE(a.D == 32 || a.D == 48 || a.D == 64, "attention: head dim %d not in {32,48,64}", a.D);
    MUGD_REQUIRE(a.pos_max >= 0 && a.pos_max <= 1024, "attention: pos_max %d", a.pos_max);
    MUGD_REQUIRE(aligned16(a.q) && aligned16(a.k) && aligned16(a.v) && aligned16(a.o) && a.ldq % 4 == 0 && a.ldk % 4 == 0 &&
                     a.ldv % 4 == 0 && a.ldo % 4 == 0, "attention: alignment");
    MUGD_REQUIRE(a.ldq >= a.H * a.D && a.ldk >= a.H * a.D && a.ldv >= a.H * a.D && a.ldo >= a.H * a.D, "attention: ld < H*D");
    MUGD_REQUIRE(a.relpos && a.cgain, "attention: tables missing");
    return MUGD_OK;
}

// 1 (default): both contractions on the wgmma tensor cores (attention_tc.cu), a lane-per-key kernel when there are at most 32 keys;
// 0: the tiled FFMA kernel above for everything (referee).  A ragged op takes the same kernel as the plain op of its shape.
template <typename Desc>
static int dispatch_attention(const DeviceInfo& dev, const Desc& d, cudaStream_t st, int* launches) {
    const mugd_attention& a = attn_desc(d);
    int rc = check_attention(a);
    if (rc != MUGD_OK) return rc;
    // per shape (tools/profile_ops.py --only attention): with head dim 32 (Lq = 256 at the default length) the rows are many
    // and short and the FFMA lanes saturate; with head dim 48 / 64 the lane-per-key kernel wins
    if (dev.attention_impl == 1 && a.Lk <= 32 && a.D >= 48)
        rc = (a.D == 48) ? attention_smallk_launch<48>(d, st) : attention_smallk_launch<64>(d, st);
    else if (dev.attention_impl == 1) rc = launch_attention_tc(dev, d, st);
    else rc = (a.D == 32) ? attention_launch<32>(d, st) : (a.D == 48) ? attention_launch<48>(d, st) : attention_launch<64>(d, st);
    if (rc != MUGD_OK) return rc;
    if (launches) *launches += 1;
    return MUGD_OK;
}

int launch_attention(const DeviceInfo& dev, const mugd_attention& a, cudaStream_t st, int* launches) {
    return dispatch_attention(dev, a, st, launches);
}

int launch_attention_var(const DeviceInfo& dev, const mugd_attention_var& a, cudaStream_t st, int* launches) {
    MUGD_REQUIRE(a.valid, "attention_var: valid lengths missing");
    MUGD_REQUIRE(a.attn.Lq == a.attn.Lk, "attention_var: self-attention only (Lq=%d, Lk=%d)", a.attn.Lq, a.attn.Lk);
    return dispatch_attention(dev, a, st, launches);
}

// Section prompts: the lane-per-key kernel at every head dim under attention_impl 1 (so at most 32 keys per section), the FFMA referee
// under 0.  The sections' rows differ from the plain op's only in which keys they read, so a sample with one section computes what
// the plain op's kernel of the same family computes.
template <int D>
static int attention_sec_launch(const DeviceInfo& dev, const mugd_attention_sec& d, cudaStream_t st) {
    const mugd_attention& a = d.attn;
    if (dev.attention_impl == 1) {
        const size_t bytes = sizeof(float) * (32 * (D + 1) + 32 * D + ASK_ROWS * D + 4);
        dim3 grid((a.Lq + ASK_ROWS - 1) / ASK_ROWS, a.H, a.B);
        MUGD_CHECK_CUDA(launch_k(attention_smallk_sec_kernel<D>, grid, dim3(ASK_WARPS * 32), bytes, st, d));
    } else {
        const size_t bytes = sizeof(float) * (AttSmem<D>::FLOATS + 2 * (2 * a.pos_max + 1));
        dim3 grid((a.Lq + AT_BQ - 1) / AT_BQ, a.H, a.B);
        MUGD_CHECK_CUDA(launch_k(attention_sec_kernel<D>, grid, dim3(AT_THREADS), bytes, st, d));
    }
    return MUGD_OK;
}

int launch_attention_sec(const DeviceInfo& dev, const mugd_attention_sec& d, cudaStream_t st, int* launches) {
    const mugd_attention& a = d.attn;
    int rc = check_attention(a);
    if (rc != MUGD_OK) return rc;
    MUGD_REQUIRE(d.starts, "attention_sec: section starts missing");
    MUGD_REQUIRE(d.sec_stride >= a.Lk, "attention_sec: section stride %d < Lk %d", d.sec_stride, a.Lk);
    MUGD_REQUIRE(dev.attention_impl != 1 || a.Lk <= 32, "attention_sec: %d keys per section; the lane-per-key kernel takes at most 32",
                 a.Lk);
    rc = (a.D == 32) ? attention_sec_launch<32>(dev, d, st) : (a.D == 48) ? attention_sec_launch<48>(dev, d, st)
                                                                           : attention_sec_launch<64>(dev, d, st);
    if (rc != MUGD_OK) return rc;
    if (launches) *launches += 1;
    return MUGD_OK;
}

}  // namespace mugd

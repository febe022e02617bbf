// Small fused elementwise kernels of the sampler loop:
//   ddim_update : classifier-free-guidance combine + DDIM x_{t-1} update   mug/diffusion/ddim.py:170-195
//   stage       : inpainting blend + step noise in front of a step of mugd_sample_staged   ddim.py:141-144,192-194
//   transpose   : [B,C,L] <-> channels-last [B*L, ld] at the Python boundary (reference tensors are NCL)
//   copy2d      : strided row copy (the 4 per-level tensors that live in two concat buffers)
//   step_advance: device-side step counter so one CUDA graph serves every DDIM step
//   cfg_scales  : classifier-free guidance at one scale per chart, in front of an unguided update
//   posterior   : first-stage encoder moments -> mean / logvar / std / z   mug/firststage/autoencoder.py:356-387
#include "common.cuh"
#include "wgmma.cuh"

namespace mugd {

// x_prev = sqrt(a_prev) * (x - sqrt(1-a_t) e)/sqrt(a_t) + sqrt(1 - a_prev - sigma^2) e + sigma*noise*T
// written with explicit _rn intrinsics: same operation order and roundings as the reference's separate
// ATen ops (no FMA contraction), so given identical eps the update is bit-identical.
__global__ void __launch_bounds__(256)
ddim_update_kernel(const mugd_ddim_update d) {
    pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d.n) return;
    const int step = d.step ? *d.step : 0;
    const int index = d.S - 1 - step;                     // ddim.py:138
    const float* cf = d.coef + 4 * index;
    const float a_t = cf[0], a_prev = cf[1], sigma = cf[2], s1m = cf[3];
    const float e = cfg_eps(d.eps, i, d.n, d.cfg, d.scale);   // ddim.py:175
    const float x = d.x[i];
    const float pred = __fdiv_rn(__fsub_rn(x, __fmul_rn(s1m, e)), __fsqrt_rn(a_t));            // :189
    const float dir = __fmul_rn(__fsqrt_rn(__fsub_rn(__fsub_rn(1.0f, a_prev), __fmul_rn(sigma, sigma))), e);  // :191
    float xp = __fadd_rn(__fmul_rn(__fsqrt_rn(a_prev), pred), dir);
    const float nz = d.noise ? __fmul_rn(__fmul_rn(sigma, d.noise[i]), d.temperature) : 0.0f;  // :192
    xp = __fadd_rn(xp, nz);                                                                     // :195
    d.x[i] = xp;
    if (d.x_dup) d.x_dup[i] = xp;
    if (d.pred_x0) d.pred_x0[i] = pred;
}

int launch_ddim_update(const DeviceInfo&, const mugd_ddim_update& d, cudaStream_t st, int* launches) {
    MUGD_REQUIRE(d.n > 0 && d.S > 0 && d.x && d.eps && d.coef, "ddim_update: bad arguments");
    MUGD_CHECK_CUDA(launch_k(ddim_update_kernel, dim3((d.n + 255) / 256), dim3(256), 0, st, d));
    if (launches) *launches += 1;
    return MUGD_OK;
}

// Stage of one step of mugd_sample_staged: the inpainting blend on the x rows and the step noise into the DDIM op's noise rows.
// 32x32 tiles as in transpose_kernel: the NCL operands are read coalesced along L, the rows written along C.  The blend restates
// `a * x0 + b * noise` (q_sample) and `x_orig * mask + (1. - mask) * x` (ddim.py:141-144) op for op with _rn intrinsics.
__global__ void __launch_bounds__(256)
stage_kernel(const mugd_stage s, const float* __restrict__ qn, const float* __restrict__ nz, float a, float b) {
    __shared__ float t_x0[32][33], t_m[32][33], t_q[32][33], t_n[32][33];
    pdl_wait();
    const int bb = blockIdx.z;
    const int c0 = blockIdx.y * 32, l0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
    const int C = s.C, L = s.L;
    const int64_t base = (int64_t)bb * C * L;
    // load_ncl_tile's loop, once for all four tiles: four calls would load the tiles one after another instead of interleaved
#pragma unroll
    for (int r = ty; r < 32; r += 8) {
        const int c = c0 + r, l = l0 + tx;
        if (c < C && l < L) {
            const int64_t j = base + (int64_t)c * L + l;
            if (s.x0) {
                t_x0[r][tx] = s.x0[j];
                t_m[r][tx] = s.mask[j];
                t_q[r][tx] = qn[j];
            }
            if (nz) t_n[r][tx] = nz[j];
        }
    }
    __syncthreads();
#pragma unroll
    for (int r = ty; r < 32; r += 8) {
        const int l = l0 + r, c = c0 + tx;
        if (c >= C || l >= L) continue;
        const int64_t row = ((int64_t)bb * L + l) * C + c;
        if (s.x0) {
            const float m = t_m[tx][r];
            const float xo = __fadd_rn(__fmul_rn(a, t_x0[tx][r]), __fmul_rn(b, t_q[tx][r]));
            const float v = __fadd_rn(__fmul_rn(xo, m), __fmul_rn(__fsub_rn(1.0f, m), s.x[row]));
            s.x[row] = v;
            if (s.x_dup) s.x_dup[row] = v;
        }
        if (nz) s.noise_rows[row] = t_n[tx][r];
    }
}

int check_stage(const mugd_stage& s, int32_t n_steps) {
    MUGD_REQUIRE(s.x, "sample_staged: stage.x is NULL");
    int rc = check_tile_grid("sample_staged", s.B, s.C, s.L);
    if (rc != MUGD_OK) return rc;
    MUGD_REQUIRE(!s.q_coef || s.q_noise, "sample_staged: q_coef given without a q-noise table");
    MUGD_REQUIRE(!s.q_noise || s.x0, "sample_staged: q-noise table given without x0");
    MUGD_REQUIRE(!s.mask || s.x0, "sample_staged: mask given without x0");
    MUGD_REQUIRE(!s.x0 || (s.mask && s.q_noise && s.q_coef), "sample_staged: x0 needs mask, q_noise and q_coef");
    MUGD_REQUIRE(!s.noise == !s.noise_rows, "sample_staged: noise and noise_rows go together");
    if (s.q_coef)
        for (int32_t i = 0; i < 2 * n_steps; ++i)
            MUGD_REQUIRE(isfinite(s.q_coef[i]), "sample_staged: q_coef[%d][%d] = %g is not finite", i / 2, i % 2, s.q_coef[i]);
    return MUGD_OK;
}

int launch_stage(const mugd_stage& s, int32_t i, cudaStream_t st) {
    const int64_t n = (int64_t)s.B * s.C * s.L;
    const float* qn = s.q_noise ? s.q_noise + i * n : nullptr;
    const float* nz = s.noise ? s.noise + i * n : nullptr;
    const float a = s.q_coef ? s.q_coef[2 * i] : 0.0f, b = s.q_coef ? s.q_coef[2 * i + 1] : 0.0f;
    const dim3 grid((s.L + 31) / 32, (s.C + 31) / 32, s.B);
    MUGD_CHECK_CUDA(launch_k(stage_kernel, grid, dim3(256), 0, st, s, qn, nz, a, b));
    return MUGD_OK;
}

// 32x32 smem-tiled transpose, coalesced on both sides.
__global__ void __launch_bounds__(256)
transpose_kernel(const mugd_transpose t) {
    __shared__ float tile[32][33];
    pdl_wait();
    const int b = blockIdx.z;
    const int c0 = blockIdx.y * 32, l0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
    if (t.to_nlc) {
        const float* in = t.in + (int64_t)b * t.C * t.L;
#pragma unroll
        for (int r = ty; r < 32; r += 8) {
            const int c = c0 + r, l = l0 + tx;
            tile[r][tx] = (c < t.C && l < t.L) ? in[(int64_t)c * t.L + l] : 0.f;
        }
        __syncthreads();
        float* out = t.out + (int64_t)b * t.L * t.ldo;
#pragma unroll
        for (int r = ty; r < 32; r += 8) {
            const int l = l0 + r, c = c0 + tx;
            if (c < t.C && l < t.L) out[(int64_t)l * t.ldo + c] = tile[tx][r];
        }
    } else {
        const float* in = t.in + (int64_t)b * t.L * t.ldi;
#pragma unroll
        for (int r = ty; r < 32; r += 8) {
            const int l = l0 + r, c = c0 + tx;
            tile[r][tx] = (c < t.C && l < t.L) ? in[(int64_t)l * t.ldi + c] : 0.f;
        }
        __syncthreads();
        float* out = t.out + (int64_t)b * t.C * t.L;
#pragma unroll
        for (int r = ty; r < 32; r += 8) {
            const int c = c0 + r, l = l0 + tx;
            if (c < t.C && l < t.L) out[(int64_t)c * t.L + l] = tile[tx][r];
        }
    }
}

int launch_transpose(const DeviceInfo&, const mugd_transpose& t, cudaStream_t st, int* launches) {
    MUGD_REQUIRE(t.B > 0 && t.C > 0 && t.L > 0 && t.in && t.out, "transpose: bad arguments");
    MUGD_REQUIRE(t.B <= 65535 && (t.C + 31) / 32 <= 65535, "transpose: grid too large");
    if (t.to_nlc) MUGD_REQUIRE(t.ldo >= t.C, "transpose: ldo < C");
    else MUGD_REQUIRE(t.ldi >= t.C, "transpose: ldi < C");
    dim3 grid((t.L + 31) / 32, (t.C + 31) / 32, t.B);
    MUGD_CHECK_CUDA(launch_k(transpose_kernel, grid, dim3(256), 0, st, t));
    if (launches) *launches += 1;
    return MUGD_OK;
}

__global__ void __launch_bounds__(256)
copy2d_kernel(const mugd_copy2d c) {
    pdl_wait();
    const int q = c.cols >> 2;
    const int64_t total = (int64_t)c.rows * q;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / q;
        const int cc = (int)(i - r * q) * 4;
        st_f4(c.dst + r * c.ldd + cc, ld_f4(c.src + r * c.lds + cc));
    }
}

int launch_copy2d(const DeviceInfo& dev, const mugd_copy2d& c, cudaStream_t st, int* launches) {
    MUGD_REQUIRE(c.rows > 0 && c.cols > 0 && c.cols % 4 == 0 && c.lds % 4 == 0 && c.ldd % 4 == 0 && aligned16(c.src) && aligned16(c.dst),
                 "copy2d: shape/alignment");
    const int64_t total = (int64_t)c.rows * (c.cols / 4);
    int blocks = (int)((total + 255) / 256);
    if (blocks > dev.sm_count * 8) blocks = dev.sm_count * 8;
    MUGD_CHECK_CUDA(launch_k(copy2d_kernel, dim3(blocks), dim3(256), 0, st, c));
    if (launches) *launches += 1;
    return MUGD_OK;
}

// ragged batches: rows l >= clamp(valid[b], 0, L) of sample b, columns 0 .. cols - 1, set to 0 by a store (padded rows may hold NaN,
// which a multiply by 0 would keep).  Grid (x, B): the CTAs of one sample stride over its padded elements only.
__global__ void __launch_bounds__(256)
row_mask_kernel(const mugd_row_mask m) {
    pdl_wait();
    const int b = blockIdx.y;
    const int Lv = min(max(m.valid[b], 0), m.L);
    const int64_t total = (int64_t)(m.L - Lv) * m.cols;
    float* xb = m.x + ((int64_t)b * m.L + Lv) * m.ld;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / m.cols;
        xb[r * m.ld + (i - r * m.cols)] = 0.f;
    }
}

int launch_row_mask(const DeviceInfo& dev, const mugd_row_mask& m, cudaStream_t st, int* launches) {
    MUGD_REQUIRE(m.x && m.valid && m.B > 0 && m.B <= 65535 && m.L > 0 && m.cols > 0 && m.ld >= m.cols,
                 "row_mask: bad descriptor B=%d L=%d cols=%d ld=%lld", m.B, m.L, m.cols, (long long)m.ld);
    const int64_t per_sample = (int64_t)m.L * m.cols;
    int blocks = (int)((per_sample + 255) / 256);
    if (blocks > 64) blocks = 64;
    MUGD_CHECK_CUDA(launch_k(row_mask_kernel, dim3(blocks, m.B), dim3(256), 0, st, m));
    if (launches) *launches += 1;
    return MUGD_OK;
}

// Per-chart guidance scales (MUGD_OP_CFG_SCALES): output row r belongs to chart r / L and gets cfg_guide(e_u, e_c, s_b), or e_c itself
// where s_b == 1 (the uncond row is then not read).  VEC: four columns per thread through 16-byte loads and stores (C and ld multiples
// of 4, eps and out 16-byte aligned); otherwise one element per thread.
template <bool VEC>
__global__ void __launch_bounds__(256)
cfg_scales_kernel(const mugd_cfg_scales g) {
    pdl_wait();
    constexpr int W = VEC ? 4 : 1;
    const int cw = g.C / W;
    const int rows = g.B * g.L;                           // the launcher keeps B * L * C within int32
    const int total = rows * cw;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int r = i / cw;
        const int c = (i - r * cw) * W;
        const float s = g.scales[r / g.L];
        const float* pu = g.eps + (int64_t)r * g.ld + c;
        const float* pc = pu + (int64_t)rows * g.ld;
        float* po = g.out + (int64_t)r * g.C + c;
        if constexpr (VEC) {
            const float4 ec = ld_f4(pc);
            if (s == 1.0f) {
                st_f4(po, ec);
            } else {
                const float4 eu = ld_f4(pu);
                st_f4(po, make_float4(cfg_guide(eu.x, ec.x, s), cfg_guide(eu.y, ec.y, s), cfg_guide(eu.z, ec.z, s),
                                      cfg_guide(eu.w, ec.w, s)));
            }
        } else {
            *po = s == 1.0f ? *pc : cfg_guide(*pu, *pc, s);
        }
    }
}

int launch_cfg_scales(const DeviceInfo& dev, const mugd_cfg_scales& g, cudaStream_t st, int* launches) {
    MUGD_REQUIRE(g.eps && g.out && g.scales, "cfg_scales: eps, out and scales must be given");
    MUGD_REQUIRE(g.B > 0 && g.L > 0 && g.C > 0 && g.ld >= g.C && (int64_t)g.B * g.L * g.C <= INT32_MAX,
                 "cfg_scales: bad shape B=%d L=%d C=%d ld=%lld", g.B, g.L, g.C, (long long)g.ld);
    const int64_t rows = (int64_t)g.B * g.L;
    const uintptr_t e0 = reinterpret_cast<uintptr_t>(g.eps), e1 = e0 + 4 * ((2 * rows - 1) * g.ld + g.C);
    const uintptr_t o0 = reinterpret_cast<uintptr_t>(g.out), o1 = o0 + 4 * rows * g.C;
    MUGD_REQUIRE(o1 <= e0 || e1 <= o0, "cfg_scales: out overlaps the eps rows");
    const bool vec = g.C % 4 == 0 && g.ld % 4 == 0 && aligned16(g.eps) && aligned16(g.out);
    const int64_t total = rows * (vec ? g.C / 4 : g.C);
    int blocks = (int)((total + 255) / 256 < (int64_t)dev.sm_count * 8 ? (total + 255) / 256 : (int64_t)dev.sm_count * 8);
    if (vec) MUGD_CHECK_CUDA(launch_k(cfg_scales_kernel<true>, dim3(blocks), dim3(256), 0, st, g));
    else MUGD_CHECK_CUDA(launch_k(cfg_scales_kernel<false>, dim3(blocks), dim3(256), 0, st, g));
    if (launches) *launches += 1;
    return MUGD_OK;
}

// weight preprocessing for the 3xTF32 GEMM: hi over w, lo beside it (same roundings as the converter warps apply to activations)
__global__ void __launch_bounds__(256)
tf32_split_kernel(float* __restrict__ w_hi, float* __restrict__ lo, int64_t n4) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 w = ld_f4(w_hi + i * 4);
        const float4 h = make_float4(to_tf32(w.x), to_tf32(w.y), to_tf32(w.z), to_tf32(w.w));
        const float4 l = make_float4(to_tf32(w.x - h.x), to_tf32(w.y - h.y), to_tf32(w.z - h.z), to_tf32(w.w - h.w));
        st_f4(w_hi + i * 4, h);
        st_f4(lo + i * 4, l);
    }
}

int launch_tf32_split(const DeviceInfo& dev, const mugd_tf32_split& s, cudaStream_t st, int* launches) {
    MUGD_REQUIRE(s.w_hi && s.lo && s.n > 0 && s.n % 4 == 0 && aligned16(s.w_hi) && aligned16(s.lo), "tf32_split: needs 16-byte aligned buffers and n %% 4 == 0");
    const int64_t n4 = s.n / 4;
    int blocks = (int)((n4 + 255) / 256);
    if (blocks > dev.sm_count * 16) blocks = dev.sm_count * 16;
    MUGD_CHECK_CUDA(launch_k(tf32_split_kernel, dim3(blocks), dim3(256), 0, st, s.w_hi, s.lo, n4));
    if (launches) *launches += 1;
    return MUGD_OK;
}

__global__ void step_advance_kernel(int32_t* step) {
    pdl_wait();
    *step += 1;
}
__global__ void fill_i32_kernel(int32_t* p, int32_t v) { *p = v; }

int launch_step_advance(const DeviceInfo&, const mugd_step_advance& a, cudaStream_t st, int* launches) {
    MUGD_REQUIRE(a.step, "step_advance: null counter");
    MUGD_CHECK_CUDA(launch_k(step_advance_kernel, dim3(1), dim3(1), 0, st, a.step));
    if (launches) *launches += 1;
    return MUGD_OK;
}

// ---- note extraction (SURVEY §8f N2): OsuManiaConvertor.array_to_objects, mug/data/convertor.py:232-264 -------------
// One CTA per (key column, chart).  Frames are visited in order in chunks of 256; the notes found in a chunk are
// compacted with a ballot/prefix scan so the output is ordered by frame like the reference's np.where loop.
__global__ void __launch_bounds__(256)
notes_kernel(const mugd_notes n) {
    pdl_wait();
    const int c = blockIdx.x, b = blockIdx.y;
    const int K = n.K, T = n.T;
    const float* Lg = n.logits + (int64_t)b * T * n.ld;
    int32_t* st_out = n.start_ms + ((int64_t)b * K + c) * T;
    int32_t* en_out = n.end_ms + ((int64_t)b * K + c) * T;
    __shared__ int warp_cnt[8];
    __shared__ int base_s;
    if (threadIdx.x == 0) base_s = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int t0 = 0; t0 < T; t0 += 256) {
        const int t = t0 + threadIdx.x;
        bool is = false;
        int start = 0, end = -1;
        if (t < T && Lg[(int64_t)t * n.ld + c] > 0.f) {
            is = true;
            const float so = fminf(fmaxf(Lg[(int64_t)t * n.ld + K + c], 0.f), 1.f);
            start = (int)rint(((double)t + (double)so) * n.frame_ms);           // python round(): half to even
            if (t != T - 1) {
                int i = t + 1;
                while (i < T && Lg[(int64_t)i * n.ld + 2 * K + c] > 0.f && !(Lg[(int64_t)i * n.ld + c] > 0.f)) ++i;
                const int ei = i - 1;
                if (ei != t) {
                    const float eo = fminf(fmaxf(Lg[(int64_t)ei * n.ld + 3 * K + c], 0.f), 1.f);
                    end = (int)rint(((double)ei + (double)eo) * n.frame_ms);
                }
            }
        }
        const unsigned m = __ballot_sync(0xffffffffu, is);
        if (lane == 0) warp_cnt[warp] = __popc(m);
        __syncthreads();
        int off = base_s;
        for (int w = 0; w < warp; ++w) off += warp_cnt[w];
        if (is) {
            const int pos = off + __popc(m & ((1u << lane) - 1u));
            st_out[pos] = start;
            en_out[pos] = end;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int tot = 0;
            for (int w = 0; w < 8; ++w) tot += warp_cnt[w];
            base_s += tot;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) n.count[b * K + c] = base_s;
}

int launch_notes(const DeviceInfo&, const mugd_notes& n, cudaStream_t st, int* launches) {
    MUGD_REQUIRE(n.B > 0 && n.T > 0 && n.K > 0 && n.K <= 16 && n.ld >= 4 * n.K, "notes: bad shape B=%d T=%d K=%d", n.B, n.T, n.K);
    MUGD_REQUIRE(n.logits && n.count && n.start_ms && n.end_ms && n.frame_ms > 0, "notes: null argument");
    MUGD_CHECK_CUDA(launch_k(notes_kernel, dim3(n.K, n.B), dim3(256), 0, st, n));
    if (launches) *launches += 1;
    return MUGD_OK;
}

// ---- prompt embedding (mug/cond/feature.py:15-21): gather + "b f h -> b h f" ------------------------------------------
// One CTA per (sample, feature slot): the table row is read coalesced, the store is strided by F (21 slots x 128 channels per
// sample: 10 KB per request, latency only).
__global__ void __launch_bounds__(128)
embed_kernel(const mugd_embed e) {
    pdl_wait();
    const int f = blockIdx.x, b = blockIdx.y;
    const int id = e.ids[b * e.F + f];
    const float* row = e.table + (int64_t)id * e.H;
    float* out = e.out + (int64_t)b * e.H * e.F + f;
    for (int h = threadIdx.x; h < e.H; h += blockDim.x) out[(int64_t)h * e.F] = row[h];
}

int launch_embed(const DeviceInfo&, const mugd_embed& e, cudaStream_t st, int* launches) {
    MUGD_REQUIRE(e.B > 0 && e.F > 0 && e.H > 0 && e.n_embed > 0, "embed: bad shape B=%d F=%d H=%d n=%d", e.B, e.F, e.H, e.n_embed);
    MUGD_REQUIRE(e.table && e.ids && e.out, "embed: null argument");
    MUGD_REQUIRE(e.B <= 65535, "embed: B=%d too large for one launch", e.B);
    MUGD_CHECK_CUDA(launch_k(embed_kernel, dim3(e.F, e.B), dim3(128), 0, st, e));
    if (launches) *launches += 1;
    return MUGD_OK;
}

// ---- posterior of the first-stage encoder (DiagonalGaussianDistribution, mug/firststage/autoencoder.py:356-387) -----------
// One thread per latent element.  clamp -> 0.5*logvar -> expf in that order (autoencoder.py:362-364), full-precision expf; the
// sample is mean + std*noise, then * scale (:371-372) with _rn intrinsics so no FMA contraction changes the rounding.
__global__ void __launch_bounds__(256)
posterior_kernel(const mugd_posterior p) {
    pdl_wait();
    const int64_t zl = (int64_t)p.Z * p.L;
    const int64_t n = (int64_t)p.B * zl;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = i / zl;
        const float* src = p.params + b * zl + i;             // sample b starts at 2*b*zl: mean rows, then logvar rows
        const float mean = src[0];
        const float raw = src[zl];
        const float lv = raw != raw ? raw : fminf(fmaxf(raw, -10.0f), 20.0f);       // torch.clamp propagates NaN
        const float sd = expf(__fmul_rn(0.5f, lv));
        if (p.mean) p.mean[i] = mean;
        if (p.logvar) p.logvar[i] = lv;
        if (p.std) p.std[i] = sd;
        if (p.z) p.z[i] = __fmul_rn(p.noise ? __fadd_rn(mean, __fmul_rn(sd, p.noise[i])) : mean, p.scale);
    }
}

int launch_posterior(const DeviceInfo& dev, const mugd_posterior& p, cudaStream_t st, int* launches) {
    MUGD_REQUIRE(p.B > 0 && p.Z > 0 && p.L > 0 && p.params, "posterior: bad arguments B=%d Z=%d L=%d", p.B, p.Z, p.L);
    const int64_t n = (int64_t)p.B * p.Z * p.L;
    int blocks = (int)((n + 255) / 256);
    if (blocks > dev.sm_count * 16) blocks = dev.sm_count * 16;
    MUGD_CHECK_CUDA(launch_k(posterior_kernel, dim3(blocks), dim3(256), 0, st, p));
    if (launches) *launches += 1;
    return MUGD_OK;
}

}  // namespace mugd

extern "C" int mugd_fill_i32(int32_t* dst, int32_t value, void* stream) {
    using namespace mugd;
    MUGD_REQUIRE(dst, "fill_i32: null");
    fill_i32_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(dst, value);
    MUGD_CHECK_CUDA(cudaGetLastError());
    return MUGD_OK;
}

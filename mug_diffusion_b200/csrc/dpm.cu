// DPM-Solver++ multistep sampler (data prediction, Lu et al. 2022; Stable Diffusion 2's DPM_Solver(predict_x0=True) "multistep"):
// the update of one step.  The host (mug_diffusion_b200/dpm_solver.py) expands each step into one coefficient row; the loops
// mugd_sample_dpm / mugd_sample_dpm_ex / mugd_sample_dpm_stop live in api.cu beside mugd_sample; mugd_dpm_update /
// mugd_dpm_ex_update / mugd_dpm_stop_update run the update alone.  The UniPC predictor-corrector update (mugd_sample_unipc /
// mugd_unipc_update; rows from mug_diffusion_b200/unipc.py) shares the DPM-Solver++ arithmetic, and so do its inpainting / remix
// (mugd_sample_unipc_ex / mugd_unipc_ex_update) and inversion (mugd_sample_unipc_stop / mugd_unipc_stop_update) updates.
#include "common.cuh"

namespace mugd {

// The update of element i at step `step` with coefficient row `row` of order `order` (1..3):
//   e  = eps rows (CFG: e_u + scale * (e_c - e_u), uncond half first, as the DDIM update)
//   m0 = (x - sigma * e) / alpha                                    the data prediction at t_i
//   x  = ((A * x + c0 * m0) + c1 * m1) + c2 * m2                      m1 / m2: the predictions of steps i-1 / i-2 (ring slots)
// in this order, every product, sum and the quotient one IEEE round-to-nearest, no contraction.  Terms past the order are not
// formed: their ring slots may not have been written yet (and 0 * NaN is NaN).  x goes to x and x_dup, m0 to pred_x0 and to ring
// slot step mod 3.  Every DPM-Solver++ update kernel and the UniPC update run these functions, so a chart computes the same bits in
// each.
__device__ __forceinline__ float dpm_data_prediction(const mugd_dpm& d, float alpha, float sigma, int i, float x) {
    const float e = cfg_eps(d.eps, i, d.n, d.cfg, d.scale);
    return __fdiv_rn(__fsub_rn(x, __fmul_rn(sigma, e)), alpha);
}

// the multistep update ((A * x + c0 * m0) + c1 * m1) + c2 * m2 of row `row` (A = row[2], c0 = row[3]), terms up to `order`
__device__ __forceinline__ float dpm_predict(const mugd_dpm& d, const float* row, float A, float c0, int order, int step, int i, float x,
                                             float m0) {
    const int64_t N = d.n;
    float xn = __fadd_rn(__fmul_rn(A, x), __fmul_rn(c0, m0));
    if (order >= 2) xn = __fadd_rn(xn, __fmul_rn(row[4], d.ring[((step + 2) % 3) * N + i]));
    if (order >= 3) xn = __fadd_rn(xn, __fmul_rn(row[5], d.ring[((step + 1) % 3) * N + i]));
    return xn;
}

__device__ __forceinline__ void dpm_element(const mugd_dpm& d, const float* row, int order, int step, int i) {
    const float alpha = row[0], sigma = row[1], A = row[2], c0 = row[3];
    const int64_t N = d.n;
    const float x = d.x[i];
    const float m0 = dpm_data_prediction(d, alpha, sigma, i, x);
    const float xn = dpm_predict(d, row, A, c0, order, step, i, x, m0);
    d.ring[(step % 3) * N + i] = m0;
    d.x[i] = xn;
    if (d.x_dup) d.x_dup[i] = xn;
    if (d.pred_x0) d.pred_x0[i] = m0;
}

// One thread per element of the dense [B*L, C] rows.  Step i = *step applies coefficient row i = (alpha, sigma, A, c0, c1, c2,
// order) with its own order.  A counter outside [0, S) leaves everything unchanged.
__global__ void __launch_bounds__(256)
dpm_update_kernel(const mugd_dpm d) {
    pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int step = *d.step;
    if (i >= d.n || (unsigned)step >= (unsigned)d.S) return;
    const float* row = d.coef + 8 * (int64_t)step;
    dpm_element(d, row, (int)row[6], step, i);
}

// The same update with one start per chart (the B charts own consecutive blocks of n / B elements): chart b runs from step start[b]
// on.  Before that it is left untouched (x, x_dup, its ring slots and pred_x0 are neither read nor written), so its rows keep the
// latent they were loaded with.  From its start on it takes the order min(order of row i, i - start[b] + 1), warming up like a fresh
// request, and applies row (i, order - 1) of the per-order table [S][3][8]; it reads only the ring slots of its own steps.
__global__ void __launch_bounds__(256)
dpm_update_starts_kernel(const mugd_dpm d, const int32_t* __restrict__ start, const float* __restrict__ order_coef, int per_chart) {
    pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int step = *d.step;
    if (i >= d.n || (unsigned)step >= (unsigned)d.S) return;
    const int first = start[i / per_chart];
    if (step < first) return;
    const int order = max(1, min(min((int)d.coef[8 * (int64_t)step + 6], step - first + 1), 3));
    dpm_element(d, order_coef + 8 * (3 * (int64_t)step + order - 1), order, step, i);
}

// An inversion row in DDIM's form (ROW_FORM = 1, order 1): m0 as above, then x = alpha_next * m0 + sigma_next * e with
// (alpha_next, sigma_next) = (row[4], row[5]), each product and the sum one IEEE round-to-nearest.  Same outputs as dpm_element.
__device__ __forceinline__ void dpm_eps_form_element(const mugd_dpm& d, const float* row, int step, int i) {
    const int64_t N = d.n;
    const float e = cfg_eps(d.eps, i, N, d.cfg, d.scale);
    const float m0 = __fdiv_rn(__fsub_rn(d.x[i], __fmul_rn(row[1], e)), row[0]);
    const float xn = __fadd_rn(__fmul_rn(row[4], m0), __fmul_rn(row[5], e));
    d.ring[(step % 3) * N + i] = m0;
    d.x[i] = xn;
    if (d.x_dup) d.x_dup[i] = xn;
    if (d.pred_x0) d.pred_x0[i] = m0;
}

// Inversion with one stop per chart (the mirror of dpm_update_starts_kernel): chart b runs steps 0 .. stop[b] - 1.  From its stop on
// it is left untouched (x, x_dup, its ring slots and pred_x0 are neither read nor written).  A running chart applies coefficient row
// i: through dpm_element, as dpm_update_kernel does, or, for a row with ROW_FORM = 1, in DDIM's form.
__global__ void __launch_bounds__(256)
dpm_update_stops_kernel(const mugd_dpm d, const int32_t* __restrict__ stop, int per_chart) {
    pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int step = *d.step;
    if (i >= d.n || (unsigned)step >= (unsigned)d.S) return;
    if (step >= stop[i / per_chart]) return;
    const float* row = d.coef + 8 * (int64_t)step;
    if (row[7] != 0.f) dpm_eps_form_element(d, row, step, i);
    else dpm_element(d, row, (int)row[6], step, i);
}

// UniPC (mug_diffusion_b200/unipc.py): iteration i evaluated the U-Net at the predicted x~_i (x, x_dup).  With m_i its data prediction as in
// dpm_element, corrector row i = (A', dn, d0, d1, d2, k, on) gives the corrected latent of step i from xc = x_i-1:
//   x_i = (((A' * xc + dn * m_i) + d0 * m_i-1) + d1 * m_i-2) + d2 * m_i-3     (the d1 term for k >= 2, d2 for k = 3)
// or x_i = x~_i when the row is off.  Then the predictor row i (dpm_predict on x_i and m_i) gives x~_i+1.  xc <- x_i, x and x_dup <-
// x~_i+1, pred_x0 <- m_i, and ring slot i mod 3 <- m_i after its m_i-3 has been read.  Each product and sum one IEEE round-to-nearest,
// no contraction.
__device__ __forceinline__ float unipc_correct(const mugd_unipc& u, const float* corr, int k, int step, int i, float m0) {
    const mugd_dpm& d = u.dpm;
    const int64_t N = d.n;
    float x = __fadd_rn(__fmul_rn(corr[0], u.xc[i]), __fmul_rn(corr[1], m0));
    x = __fadd_rn(x, __fmul_rn(corr[2], d.ring[((step + 2) % 3) * N + i]));
    if (k >= 2) x = __fadd_rn(x, __fmul_rn(corr[3], d.ring[((step + 1) % 3) * N + i]));
    if (k >= 3) x = __fadd_rn(x, __fmul_rn(corr[4], d.ring[(step % 3) * N + i]));
    return x;
}

__device__ __forceinline__ void unipc_store(const mugd_unipc& u, int step, int i, float x, float m0, float xn) {
    const mugd_dpm& d = u.dpm;
    u.xc[i] = x;
    d.ring[(step % 3) * (int64_t)d.n + i] = m0;
    d.x[i] = xn;
    if (d.x_dup) d.x_dup[i] = xn;
    if (d.pred_x0) d.pred_x0[i] = m0;
}

// The UniPC update of element i with predictor row `row` of order kp: m_i, then x_i = correct(x~_i, m_i) (unipc_correct, or x~_i where
// the corrector does not run), then x~_i+1.  Every UniPC update kernel runs it for expanded-form rows, so a chart computes the same
// bits in each.
template <typename Correct>
__device__ __forceinline__ void unipc_element(const mugd_unipc& u, const float* row, int kp, int step, int i, Correct correct) {
    const mugd_dpm& d = u.dpm;
    const float alpha = row[0], sigma = row[1], A = row[2], c0 = row[3];
    const float xt = d.x[i];
    const float m0 = dpm_data_prediction(d, alpha, sigma, i, xt);
    const float x = correct(xt, m0);
    const float xn = dpm_predict(d, row, A, c0, kp, step, i, x, m0);
    unipc_store(u, step, i, x, m0, xn);
}

// One thread per element of the dense [B*L, C] rows.  A counter outside [0, S) leaves everything unchanged.
__global__ void __launch_bounds__(256)
unipc_update_kernel(const mugd_unipc u) {
    pdl_wait();
    const mugd_dpm& d = u.dpm;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int step = *d.step;
    if (i >= d.n || (unsigned)step >= (unsigned)d.S) return;
    const float* row = d.coef + 8 * (int64_t)step;
    const float* corr = u.corr + 8 * (int64_t)step;
    unipc_element(u, row, (int)row[6], step, i,
                  [&](float xt, float m0) { return corr[6] != 0.f ? unipc_correct(u, corr, (int)corr[5], step, i, m0) : xt; });
}

// The same update with one start per chart (the B charts own consecutive blocks of n / B elements): chart b runs from step start[b]
// on and is left untouched before it (x, x_dup, xc, its ring slots and pred_x0 neither read nor written).  From its start f on it
// warms up like a fresh request: predictor order min(order of row i, i - f + 1) from row (i, order - 1) of order_coef [S][3][8]; the
// corrector only where corrector row i is on and i > f (a chart's first iteration has no previous evaluation), at order
// min(order of corrector row i, i - f) from row (i, order - 1) of order_corr [S][3][8].  It reads only the ring slots of its own steps.
__global__ void __launch_bounds__(256)
unipc_update_starts_kernel(const mugd_unipc u, const int32_t* __restrict__ start, const float* __restrict__ order_coef,
                           const float* __restrict__ order_corr, int per_chart) {
    pdl_wait();
    const mugd_dpm& d = u.dpm;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int step = *d.step;
    if (i >= d.n || (unsigned)step >= (unsigned)d.S) return;
    const int first = start[i / per_chart];
    if (step < first) return;
    const int kp = max(1, min(min((int)d.coef[8 * (int64_t)step + 6], step - first + 1), 3));
    const float* corr = u.corr + 8 * (int64_t)step;
    const int kc = max(1, min(min((int)corr[5], step - first), 3));
    const bool on = corr[6] != 0.f && step > first;
    const float* oc = order_corr + 8 * (3 * (int64_t)step + kc - 1);
    unipc_element(u, order_coef + 8 * (3 * (int64_t)step + kp - 1), kp, step, i,
                  [&](float xt, float m0) { return on ? unipc_correct(u, oc, kc, step, i, m0) : xt; });
}

// Inversion with one stop per chart (the mirror of unipc_update_starts_kernel): chart b runs iterations 0 .. stop[b] - 1 and is left
// untouched from its stop on (x, x_dup, xc, its ring slots and pred_x0 neither read nor written).  A running chart applies corrector row i
// and predictor row i as unipc_update_kernel does, except in the inversion's row forms:
//   a corrector row with column 7 nonzero (the correction form): c = ((dn * (m_i - m_i-1) + d1 * (m_i-2 - m_i-1)) + d2 * (m_i-3 - m_i-1))
//     (the d1 term for k >= 2, d2 for k = 3), x_i = x~_i + c;
//   a predictor row with column 7 nonzero (order 1 in DDIM's form): x~_i+1 = alpha_next * m_i + sigma_next * e with (alpha_next,
//     sigma_next) = (row[4], row[5]), then + A * c when a correction-form corrector ran.
// Each difference, product and sum one IEEE round-to-nearest.
__global__ void __launch_bounds__(256)
unipc_update_stops_kernel(const mugd_unipc u, const int32_t* __restrict__ stop, int per_chart) {
    pdl_wait();
    const mugd_dpm& d = u.dpm;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int step = *d.step;
    if (i >= d.n || (unsigned)step >= (unsigned)d.S) return;
    if (step >= stop[i / per_chart]) return;
    const int64_t N = d.n;
    const float* row = d.coef + 8 * (int64_t)step;
    const float* corr = u.corr + 8 * (int64_t)step;
    const int kc = (int)corr[5];
    const bool on = corr[6] != 0.f, diff = on && corr[7] != 0.f;
    if (row[7] == 0.f && !diff) {
        unipc_element(u, row, (int)row[6], step, i,
                      [&](float xt, float m0) { return on ? unipc_correct(u, corr, kc, step, i, m0) : xt; });
        return;
    }
    const float xt = d.x[i];
    const float e = cfg_eps(d.eps, i, N, d.cfg, d.scale);
    const float m0 = __fdiv_rn(__fsub_rn(xt, __fmul_rn(row[1], e)), row[0]);
    float x = xt, c = 0.f;
    if (diff) {
        const float m1 = d.ring[((step + 2) % 3) * N + i];
        c = __fmul_rn(corr[1], __fsub_rn(m0, m1));
        if (kc >= 2) c = __fadd_rn(c, __fmul_rn(corr[3], __fsub_rn(d.ring[((step + 1) % 3) * N + i], m1)));
        if (kc >= 3) c = __fadd_rn(c, __fmul_rn(corr[4], __fsub_rn(d.ring[(step % 3) * N + i], m1)));
        x = __fadd_rn(xt, c);
    } else if (on) {
        x = unipc_correct(u, corr, kc, step, i, m0);
    }
    float xn;
    if (row[7] != 0.f) {
        xn = __fadd_rn(__fmul_rn(row[4], m0), __fmul_rn(row[5], e));
        if (diff) xn = __fadd_rn(xn, __fmul_rn(row[2], c));
    } else {
        xn = dpm_predict(d, row, row[2], row[3], (int)row[6], step, i, x, m0);
    }
    unipc_store(u, step, i, x, m0, xn);
}

int check_dpm(const mugd_dpm& d) {
    MUGD_REQUIRE(d.x && d.eps && d.ring && d.coef && d.step, "dpm: x, eps, ring, coef and step must be given");
    MUGD_REQUIRE(d.n > 0, "dpm: n=%d", d.n);
    MUGD_REQUIRE(d.S > 0 && d.S <= MUGD_MAX_STEPS, "dpm: S=%d outside [1, %d]", d.S, MUGD_MAX_STEPS);
    int rc = check_cfg("dpm", d.cfg);
    if (rc != MUGD_OK) return rc;
    if ((rc = check_scale("dpm", d.scale)) != MUGD_OK) return rc;
    return check_x_dup("dpm", d.x_dup, d.cfg);
}

int launch_dpm_update(const mugd_dpm& d, cudaStream_t st) {
    MUGD_CHECK_CUDA(launch_k(dpm_update_kernel, dim3((d.n + 255) / 256), dim3(256), 0, st, d));
    return MUGD_OK;
}

// The inpainting stage of a multistep solver (`who`: the message prefix, `solver`: its name): the blend of the update's own x / x_dup
// over its n elements, and no step noise.
static int check_blend_stage(const char* who, const char* solver, const mugd_stage& s, int32_t n_steps, const mugd_dpm& d) {
    int rc = check_stage(s, n_steps);
    if (rc != MUGD_OK) return rc;
    MUGD_REQUIRE(s.x0, "%s: the stage has no x0 (a %s stage is the inpainting blend)", who, solver);
    MUGD_REQUIRE(!s.noise, "%s: the stage stages step noise; %s draws none", who, solver);
    MUGD_REQUIRE(s.x == d.x && s.x_dup == d.x_dup, "%s: the stage blends other rows than the update's x / x_dup", who);
    MUGD_REQUIRE((int64_t)s.B * s.C * s.L == d.n, "%s: the stage's B*C*L=%lld, the update's n=%d", who, (long long)s.B * s.C * s.L, d.n);
    return MUGD_OK;
}

int check_dpm_ex(const mugd_dpm_ex& e, int32_t n_steps) {
    int rc = check_dpm(e.dpm);
    if (rc != MUGD_OK) return rc;
    MUGD_REQUIRE(!e.stage || !e.start, "dpm_ex: a stage (inpainting) and per-chart starts cannot be combined");
    MUGD_REQUIRE(!e.start == !e.order_coef, "dpm_ex: start and order_coef go together");
    if (e.start) {
        MUGD_REQUIRE(e.B > 0 && e.dpm.n % e.B == 0, "dpm_ex: B=%d does not divide n=%d", e.B, e.dpm.n);
    }
    return e.stage ? check_blend_stage("dpm_ex", "DPM-Solver++", *e.stage, n_steps, e.dpm) : MUGD_OK;
}

int launch_dpm_ex_update(const mugd_dpm_ex& e, cudaStream_t st) {
    if (!e.start) return launch_dpm_update(e.dpm, st);
    MUGD_CHECK_CUDA(launch_k(dpm_update_starts_kernel, dim3((e.dpm.n + 255) / 256), dim3(256), 0, st, e.dpm, e.start, e.order_coef,
                             e.dpm.n / e.B));
    return MUGD_OK;
}

int check_dpm_stop(const mugd_dpm_stop& e) {
    int rc = check_dpm(e.dpm);
    if (rc != MUGD_OK) return rc;
    MUGD_REQUIRE(e.stop, "dpm_stop: stop must be given");
    MUGD_REQUIRE(e.B > 0 && e.dpm.n % e.B == 0, "dpm_stop: B=%d does not divide n=%d", e.B, e.dpm.n);
    MUGD_REQUIRE(e.reserved_ == 0, "dpm_stop: reserved_=%d must be 0", e.reserved_);
    return MUGD_OK;
}

int launch_dpm_stop_update(const mugd_dpm_stop& e, cudaStream_t st) {
    MUGD_CHECK_CUDA(launch_k(dpm_update_stops_kernel, dim3((e.dpm.n + 255) / 256), dim3(256), 0, st, e.dpm, e.stop, e.dpm.n / e.B));
    return MUGD_OK;
}

static bool overlaps(const float* a, int64_t na, const float* b, int64_t nb) {
    return a && b && a < b + nb && b < a + na;
}

int check_unipc(const mugd_unipc& u) {
    int rc = check_dpm(u.dpm);
    if (rc != MUGD_OK) return rc;
    const mugd_dpm& d = u.dpm;
    MUGD_REQUIRE(u.xc && u.corr, "unipc: xc and corr must be given");
    MUGD_REQUIRE(!overlaps(u.xc, d.n, d.x, d.n) && !overlaps(u.xc, d.n, d.x_dup, d.n) && !overlaps(u.xc, d.n, d.ring, 3 * (int64_t)d.n),
                 "unipc: xc overlaps x, x_dup or the ring");
    return MUGD_OK;
}

int launch_unipc_update(const mugd_unipc& u, cudaStream_t st) {
    MUGD_CHECK_CUDA(launch_k(unipc_update_kernel, dim3((u.dpm.n + 255) / 256), dim3(256), 0, st, u));
    return MUGD_OK;
}

int check_unipc_ex(const mugd_unipc_ex& e, int32_t n_steps) {
    int rc = check_unipc(e.unipc);
    if (rc != MUGD_OK) return rc;
    MUGD_REQUIRE(!e.stage || !e.start, "unipc_ex: a stage (inpainting) and per-chart starts cannot be combined");
    MUGD_REQUIRE(!e.start == !e.order_coef && !e.start == !e.order_corr, "unipc_ex: start, order_coef and order_corr go together");
    if (e.start) {
        MUGD_REQUIRE(e.B > 0 && e.unipc.dpm.n % e.B == 0, "unipc_ex: B=%d does not divide n=%d", e.B, e.unipc.dpm.n);
    }
    MUGD_REQUIRE(e.reserved_ == 0, "unipc_ex: reserved_=%d must be 0", e.reserved_);
    return e.stage ? check_blend_stage("unipc_ex", "UniPC", *e.stage, n_steps, e.unipc.dpm) : MUGD_OK;
}

int launch_unipc_ex_update(const mugd_unipc_ex& e, cudaStream_t st) {
    if (!e.start) return launch_unipc_update(e.unipc, st);
    MUGD_CHECK_CUDA(launch_k(unipc_update_starts_kernel, dim3((e.unipc.dpm.n + 255) / 256), dim3(256), 0, st, e.unipc, e.start,
                             e.order_coef, e.order_corr, e.unipc.dpm.n / e.B));
    return MUGD_OK;
}

int check_unipc_stop(const mugd_unipc_stop& e) {
    int rc = check_unipc(e.unipc);
    if (rc != MUGD_OK) return rc;
    MUGD_REQUIRE(e.stop, "unipc_stop: stop must be given");
    MUGD_REQUIRE(e.B > 0 && e.unipc.dpm.n % e.B == 0, "unipc_stop: B=%d does not divide n=%d", e.B, e.unipc.dpm.n);
    MUGD_REQUIRE(e.reserved_ == 0, "unipc_stop: reserved_=%d must be 0", e.reserved_);
    return MUGD_OK;
}

int launch_unipc_stop_update(const mugd_unipc_stop& e, cudaStream_t st) {
    MUGD_CHECK_CUDA(launch_k(unipc_update_stops_kernel, dim3((e.unipc.dpm.n + 255) / 256), dim3(256), 0, st, e.unipc, e.stop,
                             e.unipc.dpm.n / e.B));
    return MUGD_OK;
}

}  // namespace mugd

using namespace mugd;

extern "C" int mugd_dpm_update(const mugd_dpm* d, void* stream) {
    MUGD_REQUIRE(d, "mugd_dpm_update: null argument");
    int rc = check_dpm(*d);
    if (rc != MUGD_OK) return rc;
    return launch_dpm_update(*d, (cudaStream_t)stream);
}

extern "C" int mugd_dpm_ex_update(const mugd_dpm_ex* e, void* stream) {
    MUGD_REQUIRE(e, "mugd_dpm_ex_update: null argument");
    int rc = check_dpm_ex(*e, 0);
    if (rc != MUGD_OK) return rc;
    return launch_dpm_ex_update(*e, (cudaStream_t)stream);
}

extern "C" int mugd_dpm_stop_update(const mugd_dpm_stop* e, void* stream) {
    MUGD_REQUIRE(e, "mugd_dpm_stop_update: null argument");
    int rc = check_dpm_stop(*e);
    if (rc != MUGD_OK) return rc;
    return launch_dpm_stop_update(*e, (cudaStream_t)stream);
}

extern "C" int mugd_unipc_update(const mugd_unipc* u, void* stream) {
    MUGD_REQUIRE(u, "mugd_unipc_update: null argument");
    int rc = check_unipc(*u);
    if (rc != MUGD_OK) return rc;
    return launch_unipc_update(*u, (cudaStream_t)stream);
}

extern "C" int mugd_unipc_ex_update(const mugd_unipc_ex* e, void* stream) {
    MUGD_REQUIRE(e, "mugd_unipc_ex_update: null argument");
    int rc = check_unipc_ex(*e, 0);
    if (rc != MUGD_OK) return rc;
    return launch_unipc_ex_update(*e, (cudaStream_t)stream);
}

extern "C" int mugd_unipc_stop_update(const mugd_unipc_stop* e, void* stream) {
    MUGD_REQUIRE(e, "mugd_unipc_stop_update: null argument");
    int rc = check_unipc_stop(*e);
    if (rc != MUGD_OK) return rc;
    return launch_unipc_stop_update(*e, (cudaStream_t)stream);
}

// DPM-Solver++ multistep sampler (data prediction, Lu et al. 2022; Stable Diffusion 2's DPM_Solver(predict_x0=True) "multistep"):
// the update of one step.  The host (mug_diffusion_b200/dpm_solver.py) expands each step into one coefficient row; the loop
// mugd_sample_dpm lives in api.cu beside mugd_sample; mugd_dpm_update runs the update alone.
#include "common.cuh"

namespace mugd {

// One thread per element of the dense [B*L, C] rows.  Step i = *step reads coefficient row i = (alpha, sigma, A, c0, c1, c2, order):
//   e  = eps rows (CFG: e_u + scale * (e_c - e_u), uncond half first, as the DDIM update)
//   m0 = (x - sigma * e) / alpha                                    the data prediction at t_i
//   x  = ((A * x + c0 * m0) + c1 * m1) + c2 * m2                      m1 / m2: the predictions of steps i-1 / i-2 (ring slots)
// in this order, every product, sum and the quotient one IEEE round-to-nearest, no contraction.  Terms past the row's order are not
// formed: their ring slots may not have been written yet (and 0 * NaN is NaN).  x goes to x and x_dup, m0 to pred_x0 and to ring
// slot i mod 3.  A counter outside [0, S) leaves everything unchanged.
__global__ void __launch_bounds__(256)
dpm_update_kernel(const mugd_dpm d) {
    pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int step = *d.step;
    if (i >= d.n || (unsigned)step >= (unsigned)d.S) return;
    const float* row = d.coef + 8 * (int64_t)step;
    const float alpha = row[0], sigma = row[1], A = row[2], c0 = row[3];
    const int order = (int)row[6];
    const int64_t N = d.n;
    float e;
    if (d.cfg) {
        const float eu = d.eps[i], ec = d.eps[N + i];
        e = __fadd_rn(eu, __fmul_rn(d.scale, __fsub_rn(ec, eu)));
    } else {
        e = d.eps[i];
    }
    const float x = d.x[i];
    const float m0 = __fdiv_rn(__fsub_rn(x, __fmul_rn(sigma, e)), alpha);
    float xn = __fadd_rn(__fmul_rn(A, x), __fmul_rn(c0, m0));
    if (order >= 2) xn = __fadd_rn(xn, __fmul_rn(row[4], d.ring[((step + 2) % 3) * N + i]));
    if (order >= 3) xn = __fadd_rn(xn, __fmul_rn(row[5], d.ring[((step + 1) % 3) * N + i]));
    d.ring[(step % 3) * N + i] = m0;
    d.x[i] = xn;
    if (d.x_dup) d.x_dup[i] = xn;
    if (d.pred_x0) d.pred_x0[i] = m0;
}

int check_dpm(const mugd_dpm& d) {
    MUGD_REQUIRE(d.x && d.eps && d.ring && d.coef && d.step, "dpm: x, eps, ring, coef and step must be given");
    MUGD_REQUIRE(d.n > 0, "dpm: n=%d", d.n);
    MUGD_REQUIRE(d.S > 0 && d.S <= MUGD_MAX_STEPS, "dpm: S=%d outside [1, %d]", d.S, MUGD_MAX_STEPS);
    MUGD_REQUIRE(d.cfg == 0 || d.cfg == 1, "dpm: cfg=%d", d.cfg);
    MUGD_REQUIRE(isfinite(d.scale), "dpm: scale is not finite");
    MUGD_REQUIRE(!d.x_dup == !d.cfg, "dpm: x_dup must be given exactly when cfg = 1 (the evaluation reads x in both halves)");
    return MUGD_OK;
}

int launch_dpm_update(const mugd_dpm& d, cudaStream_t st) {
    MUGD_CHECK_CUDA(launch_k(dpm_update_kernel, dim3((d.n + 255) / 256), dim3(256), 0, st, d));
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

// DDPM ancestral sampler (DDPM.log_beatmap, mug/diffusion/diffusion.py:255-282): the posterior update of one step.  The loop
// mugd_sample_ddpm lives in api.cu beside mugd_sample; mugd_ddpm_update runs the update alone.
#include "common.cuh"

namespace mugd {

// One CTA per 32x32 (channel, position) tile of one sample, as stage_kernel: the step's noise is read from the NCL table coalesced
// along L, the [B*L, C] rows (eps, x, x_dup, pred_x0) coalesced along C.  Restates diffusion.py:259-277 op for op, one IEEE
// round-to-nearest per torch eager op and no contraction, so with equal eps and noise the result is bit-identical to torch:
//   e       = eps rows (CFG: e_u + scale * (e_c - e_u), uncond half first, as ddim.py:175)
//   x_recon = sqrt_recip[t] * x - sqrt_recipm1[t] * e                                  predict_start_from_noise, :211-215
//   x_recon = clamp(x_recon, -10, 10) when clip, NaN kept (torch's clamp)              :266-267
//   mean    = coef1[t] * x_recon + coef2[t] * x                                         :268-271
//   x       = mean + sigma[t] * noise,  sigma[t] = (1 - (t == 0)) * exp(0.5 * logvar[t]) :272-277 (the table's column 4)
// with t = T - 1 - *step.  A counter outside [0, T) leaves everything unchanged.
__global__ void __launch_bounds__(256)
ddpm_update_kernel(const mugd_ddpm d, const float* __restrict__ nz) {
    __shared__ float t_n[32][33];
    pdl_wait();
    const int bb = blockIdx.z;
    const int c0 = blockIdx.y * 32, l0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
    const int C = d.C, L = d.L;
    load_ncl_tile(t_n, nz + (int64_t)bb * C * L, c0, l0, C, L);
    __syncthreads();
    const int t = d.T - 1 - *d.step;
    if ((unsigned)t >= (unsigned)d.T) return;
    const float* cf = d.coef + 5 * t;
    const float sra = cf[0], srm1 = cf[1], c1 = cf[2], c2 = cf[3], sigma = cf[4];
    const int64_t n = (int64_t)d.B * C * L;
#pragma unroll
    for (int r = ty; r < 32; r += 8) {
        const int l = l0 + r, c = c0 + tx;
        if (c >= C || l >= L) continue;
        const int64_t row = ((int64_t)bb * L + l) * C + c;
        const float e = cfg_eps(d.eps, row, n, d.cfg, d.scale);
        const float x = d.x[row];
        float xr = __fsub_rn(__fmul_rn(sra, x), __fmul_rn(srm1, e));
        if (d.clip && !isnan(xr)) xr = fminf(fmaxf(xr, -10.0f), 10.0f);
        const float mean = __fadd_rn(__fmul_rn(c1, xr), __fmul_rn(c2, x));
        const float xn = __fadd_rn(mean, __fmul_rn(sigma, t_n[tx][r]));
        d.x[row] = xn;
        if (d.x_dup) d.x_dup[row] = xn;
        if (d.pred_x0) d.pred_x0[row] = xr;
    }
}

int check_ddpm(const mugd_ddpm& d) {
    MUGD_REQUIRE(d.x && d.eps && d.noise && d.coef && d.step, "ddpm: x, eps, noise, coef and step must be given");
    int rc = check_tile_grid("ddpm", d.B, d.C, d.L);
    if (rc != MUGD_OK) return rc;
    MUGD_REQUIRE(d.T > 0 && d.T <= MUGD_MAX_STEPS, "ddpm: T=%d outside [1, %d]", d.T, MUGD_MAX_STEPS);
    if ((rc = check_cfg("ddpm", d.cfg)) != MUGD_OK) return rc;
    MUGD_REQUIRE(d.clip == 0 || d.clip == 1, "ddpm: clip=%d", d.clip);
    if ((rc = check_scale("ddpm", d.scale)) != MUGD_OK) return rc;
    return check_x_dup("ddpm", d.x_dup, d.cfg);
}

int launch_ddpm_update(const mugd_ddpm& d, int32_t k, cudaStream_t st) {
    const float* nz = d.noise + (int64_t)k * d.B * d.C * d.L;
    const dim3 grid((d.L + 31) / 32, (d.C + 31) / 32, d.B);
    MUGD_CHECK_CUDA(launch_k(ddpm_update_kernel, grid, dim3(256), 0, st, d, nz));
    return MUGD_OK;
}

}  // namespace mugd

using namespace mugd;

extern "C" int mugd_ddpm_update(const mugd_ddpm* d, void* stream) {
    MUGD_REQUIRE(d, "mugd_ddpm_update: null argument");
    int rc = check_ddpm(*d);
    if (rc != MUGD_OK) return rc;
    return launch_ddpm_update(*d, 0, (cudaStream_t)stream);
}

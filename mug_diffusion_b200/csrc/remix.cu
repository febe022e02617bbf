// Remixing an existing chart (SDEdit / img2img): the forward noising of DDIMSampler.stochastic_encode and the join kernel of the
// per-chart-strength decode loop.  The loop mugd_sample_join lives in api.cu beside mugd_sample; mugd_stochastic_encode runs the
// noising alone.
#include "common.cuh"

namespace mugd {

// out = a[t[b]] * x0 + s[t[b]] * noise per sample b, NCL in and out: extract_into_tensor(a, t, shape) * x0 +
// extract_into_tensor(s, t, shape) * noise, each product and the sum one IEEE round-to-nearest (no contraction), so with the same
// tables and noise the result is bit-identical to torch's.  An index outside [0, n) writes NaN instead of reading past the tables.
__global__ void __launch_bounds__(256)
q_encode_kernel(const mugd_q_encode d) {
    pdl_wait();
    const int64_t per = (int64_t)d.C * d.L;
    const int64_t total = per * d.B;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = d.t[i / per];
        float v = __int_as_float(0x7fc00000);
        if (t >= 0 && t < d.n) v = __fadd_rn(__fmul_rn(d.sqrt_a[t], d.x0[i]), __fmul_rn(d.sqrt_1ma[t], d.noise[i]));
        d.out[i] = v;
    }
}

int check_q_encode(const mugd_q_encode& d) {
    MUGD_REQUIRE(d.x0 && d.noise && d.t && d.sqrt_a && d.sqrt_1ma && d.out, "stochastic_encode: x0, noise, t, sqrt_a, sqrt_1ma and out "
                 "must be given");
    MUGD_REQUIRE(d.B > 0 && d.C > 0 && d.L > 0, "stochastic_encode: bad shape B=%d C=%d L=%d", d.B, d.C, d.L);
    MUGD_REQUIRE(d.n > 0, "stochastic_encode: the coefficient tables have n=%d rows", d.n);
    return MUGD_OK;
}

// Join kernel of mugd_sample_join: while the step counter has not passed chart b's join iteration (step <= join[b]), chart b's dense
// x rows (and their CFG copy) are set to x_latent[b], so the chart enters the loop at iteration join[b] from its own latent.  32x32
// tiles as stage_kernel: x_latent is read coalesced along L, the rows written along C.  A CTA of a chart that has joined returns
// before it reads anything.
__global__ void __launch_bounds__(256)
join_kernel(const mugd_join j, const int32_t* __restrict__ step) {
    __shared__ float tile[32][33];
    pdl_wait();
    const int bb = blockIdx.z;
    if (*step > j.join[bb]) return;
    const int c0 = blockIdx.y * 32, l0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
    const int C = j.C, L = j.L;
    load_ncl_tile(tile, j.x_latent + (int64_t)bb * C * L, c0, l0, C, L);
    __syncthreads();
#pragma unroll
    for (int r = ty; r < 32; r += 8) {
        const int l = l0 + r, c = c0 + tx;
        if (c >= C || l >= L) continue;
        const int64_t row = ((int64_t)bb * L + l) * C + c;
        j.x[row] = tile[tx][r];
        if (j.x_dup) j.x_dup[row] = tile[tx][r];
    }
}

int check_join(const mugd_join& j) {
    MUGD_REQUIRE(j.x && j.x_latent && j.join, "sample_join: x, x_latent and join must be given");
    return check_tile_grid("sample_join", j.B, j.C, j.L);
}

int launch_join(const mugd_join& j, const int32_t* step, cudaStream_t st) {
    const dim3 grid((j.L + 31) / 32, (j.C + 31) / 32, j.B);
    MUGD_CHECK_CUDA(launch_k(join_kernel, grid, dim3(256), 0, st, j, step));
    return MUGD_OK;
}

}  // namespace mugd

using namespace mugd;

extern "C" int mugd_stochastic_encode(const mugd_q_encode* d, void* stream) {
    MUGD_REQUIRE(d, "mugd_stochastic_encode: null argument");
    int rc = check_q_encode(*d);
    if (rc != MUGD_OK) return rc;
    const int64_t total = (int64_t)d->B * d->C * d->L;
    const int64_t blocks = (total + 255) / 256;
    MUGD_CHECK_CUDA(launch_k(q_encode_kernel, dim3((unsigned)(blocks < 4096 ? blocks : 4096)), dim3(256), 0, (cudaStream_t)stream, *d));
    return MUGD_OK;
}

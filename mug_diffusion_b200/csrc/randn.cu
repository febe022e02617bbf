// Per-chart standard normals (mugd_randn): a counter-based generator whose values depend only on (seed, purpose, draw, element),
// never on the batch, the launch configuration or the device, so any chart of a request can be regenerated alone.
//   q = e >> 2 for element e = c * L + l of a chart of n elements;
//   (x0, x1, x2, x3) = Philox4x32-10(counter = (q, draw, purpose, 0), key = (lo32(seed), hi32(seed)));
//   Box-Muller on (x0, x1) gives elements 4q, 4q + 1 and on (x2, x3) elements 4q + 2, 4q + 3:
//     u1 = ((xa >> 8) + 1) * 2^-24 in (0, 1],  u2 = (xb >> 8) * 2^-24,  r = sqrtf(-2 logf(u1)),
//     z_even = r * cospi(2 u2),  z_odd = r * sinpi(2 u2)   (one sincospif).
// Each element is one fixed expression of correctly rounded or library-accurate float operations (no fast math), so every launch
// shape gives the same bits.
#include "common.cuh"

namespace mugd {

__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
}

// Philox4x32 with 10 rounds (Salmon et al., 2011; Random123's philox4x32_10)
__device__ __forceinline__ void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        philox_round(c, k0, k1);
    }
}

__device__ __forceinline__ float2 box_muller(uint32_t xa, uint32_t xb) {
    const float u1 = __uint2float_rn((xa >> 8) + 1u) * 0x1p-24f;
    const float u2 = __uint2float_rn(xb >> 8) * 0x1p-24f;
    const float r = __fsqrt_rn(__fmul_rn(-2.0f, logf(u1)));
    float s, c;
    sincospif(__fmul_rn(2.0f, u2), &s, &c);
    return make_float2(__fmul_rn(r, c), __fmul_rn(r, s));
}

// One thread per quad (k, b, q): the four normals of elements 4q .. 4q + 3 of chart b's row for draw first_draw + draw_stride * k,
// one 16-byte store when the row allows it.  Grid-stride over the n_draws * B * ceil(n / 4) quads.
__global__ void __launch_bounds__(256)
randn_kernel(const mugd_normal d, int64_t quads_per_row, bool vec) {
    pdl_wait();                                                         // out may still be read by the previous kernel
    const int64_t total = quads_per_row * d.B * d.n_draws;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / quads_per_row;                          // k * B + b
        const int64_t q = i - row * quads_per_row;
        const int32_t k = (int32_t)(row / d.B), b = (int32_t)(row - (int64_t)k * d.B);
        const uint64_t seed = d.seeds[b];
        uint32_t c[4] = {(uint32_t)q, (uint32_t)(d.first_draw + d.draw_stride * k), (uint32_t)d.purpose, 0u};
        philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
        const float2 z01 = box_muller(c[0], c[1]), z23 = box_muller(c[2], c[3]);
        float* out = d.out + row * d.n + 4 * q;
        if (vec) {
            st_f4(out, make_float4(z01.x, z01.y, z23.x, z23.y));
        } else {
            const int64_t left = d.n - 4 * q;
            out[0] = z01.x;
            if (left > 1) out[1] = z01.y;
            if (left > 2) out[2] = z23.x;
            if (left > 3) out[3] = z23.y;
        }
    }
}

int check_normal(const mugd_normal& d) {
    MUGD_REQUIRE(d.out && d.seeds, "randn: out and seeds must be given");
    MUGD_REQUIRE(d.B >= 1 && d.n >= 1 && d.n_draws >= 1, "randn: B=%d, n=%lld and n_draws=%d must be at least 1", d.B,
                 (long long)d.n, d.n_draws);
    MUGD_REQUIRE(d.first_draw >= 0 && d.purpose >= 0, "randn: first_draw=%d and purpose=%d must not be negative", d.first_draw,
                 d.purpose);
    MUGD_REQUIRE(d.draw_stride == 1 || d.draw_stride == -1, "randn: draw_stride=%d must be 1 or -1", d.draw_stride);
    const int64_t last = (int64_t)d.first_draw + (int64_t)d.draw_stride * (d.n_draws - 1);
    MUGD_REQUIRE(last >= 0 && last < ((int64_t)1 << 31), "randn: draws %d .. %lld leave [0, 2^31)", d.first_draw, (long long)last);
    MUGD_REQUIRE((d.n - 1) >> 2 < ((int64_t)1 << 32), "randn: n=%lld puts the quad counter n/4 past 2^32", (long long)d.n);
    MUGD_REQUIRE(d.n <= INT64_MAX / 4 / d.B / d.n_draws, "randn: n_draws * B * n = %d * %d * %lld elements overflow", d.n_draws, d.B,
                 (long long)d.n);
    return MUGD_OK;
}

}  // namespace mugd

using namespace mugd;

extern "C" int mugd_randn(const mugd_normal* d, void* stream) {
    // the descriptor is checked before any device call, so a host can test its arguments without a device
    MUGD_REQUIRE(d, "mugd_randn: null descriptor");
    int rc = check_normal(*d);
    if (rc != MUGD_OK) return rc;
    const int64_t quads = (d->n + 3) / 4;
    const int64_t total = quads * d->B * d->n_draws;
    const int64_t blocks = (total + 255) / 256;
    const bool vec = d->n % 4 == 0 && aligned16(d->out);
    MUGD_CHECK_CUDA(launch_k(randn_kernel, dim3((unsigned)(blocks < 8192 ? blocks : 8192)), dim3(256), 0, (cudaStream_t)stream, *d,
                             quads, vec));
    return MUGD_OK;
}

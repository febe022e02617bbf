// Log-mel spectrogram of decoded audio: the audio front-end of webui's request path.
//
// Reference: load_audio_without_cache (mug/util.py:138-143) with the shipped common_params (mug_diffusion.yaml:101-105):
//     np.log1p(librosa.feature.melspectrogram(y=y, sr=22050, n_mels=128, hop_length=128, n_fft=512)).astype(np.float16)
// under librosa >= 0.10 defaults: center=True with zero padding (n_fft/2 on each side, T = 1 + n // hop frames), periodic Hann
// window, power 2, Slaney filterbank.  librosa's STFT multiplies the float64 window by the float32 frame, runs numpy's float64
// rfft and rounds the result into a complex64 matrix; |X| is float32 (hypotf) and squared in float32.  The kernel does the same:
// window and FFT in fp64, spectrum rounded to fp32, |X|^2 in fp32, then the sparse mel dot accumulated in fp64 and rounded to
// fp32, log1p, and the fp16 rounding of .astype(np.float16), stored back as fp32.
//
// One warp per frame, four frames per CTA in flight, grid-stride over the B * T_out output rows: the frame is read straight
// from the waveform (samples outside [0, n) are the zero padding), a 512-point real FFT is a 256-point complex FFT of
// (x[2j], x[2j+1]) in shared memory plus the split step, and each lane finishes every 32nd mel band.  Rows t >= T of each
// sample are webui's zero pad to 64 * z_length frames (webui.py:360-365) and are written as zeros.
#include "common.cuh"

#include <cuda_fp16.h>
#include <math.h>

#include <algorithm>

namespace mugd {

constexpr int MEL_NFFT = 512;                 // the shipped config's n_fft, the only one supported
constexpr int MEL_NC = MEL_NFFT / 2;          // length of the complex FFT
constexpr int MEL_NBINS = MEL_NFFT / 2 + 1;   // rfft bins
constexpr int MEL_WARPS = 4;                  // frames per CTA
constexpr int MEL_MAX_MELS = 256;

// The filterbank's bands as kernel parameters: band m is weights[off[m] .. off[m] + len[m]) over bins start[m] .. start[m] + len[m].
// The host copies them here from its own arrays, so their ranges are checked before the launch.
struct MelBands {
    int32_t off[MEL_MAX_MELS];
    int16_t start[MEL_MAX_MELS];
    int16_t len[MEL_MAX_MELS];
};

__global__ void __launch_bounds__(32 * MEL_WARPS)
melspec_kernel(const float* __restrict__ y, int64_t n, int64_t ldy, const double* __restrict__ window,
               const double2* __restrict__ twiddle, const float* __restrict__ weights, const __grid_constant__ MelBands bands,
               int n_mels, int hop, int T, int T_out, int64_t n_rows, float* __restrict__ out, int64_t ldo) {
    __shared__ double s_win[MEL_NFFT];
    __shared__ double2 s_tw[MEL_NC];                     // exp(-2 pi i k / 512), k < 256
    __shared__ double2 s_z[MEL_WARPS][MEL_NC];
    __shared__ float s_p[MEL_WARPS][MEL_NBINS + 3];
    for (int i = threadIdx.x; i < MEL_NFFT; i += blockDim.x) s_win[i] = window[i];
    for (int i = threadIdx.x; i < MEL_NC; i += blockDim.x) s_tw[i] = twiddle[i];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double2* z = s_z[warp];
    float* p = s_p[warp];
    for (int64_t f = (int64_t)blockIdx.x * MEL_WARPS + warp; f < n_rows; f += (int64_t)gridDim.x * MEL_WARPS) {
        const int b = (int)(f / T_out);
        const int t = (int)(f - (int64_t)b * T_out);
        float* o = out + f * ldo;
        if (t >= T) {
            for (int m = lane; m < n_mels; m += 32) o[m] = 0.f;
            continue;
        }
        // windowed frame as 256 complex samples z[j] = x[2j] + i x[2j+1], stored in bit-reversed order for the in-place DIT FFT
        const float* yb = y + (int64_t)b * ldy;
        const int64_t s0 = (int64_t)t * hop - MEL_NFFT / 2;
        for (int j = lane; j < MEL_NC; j += 32) {
            const int64_t s = s0 + 2 * j;
            const double x0 = (s >= 0 && s < n) ? (double)yb[s] : 0.0;
            const double x1 = (s + 1 >= 0 && s + 1 < n) ? (double)yb[s + 1] : 0.0;
            z[__brev(j) >> 24] = make_double2(x0 * s_win[2 * j], x1 * s_win[2 * j + 1]);
        }
        __syncwarp();
        // radix-2 stages: butterflies of span 2*half use W_span^pos = W_512^(pos * 256 / half)
        for (int half = 1; half < MEL_NC; half <<= 1) {
            const int tstride = MEL_NC / half;
            for (int bf = lane; bf < MEL_NC / 2; bf += 32) {
                const int pos = bf & (half - 1);
                const int i0 = ((bf - pos) << 1) + pos, i1 = i0 + half;
                const double2 w = s_tw[pos * tstride];
                const double2 a = z[i0], c = z[i1];
                const double cr = c.x * w.x - c.y * w.y, ci = c.x * w.y + c.y * w.x;
                z[i0] = make_double2(a.x + cr, a.y + ci);
                z[i1] = make_double2(a.x - cr, a.y - ci);
            }
            __syncwarp();
        }
        // split step: X[k] = E[k] + W_512^k O[k] with E = (Z[k] + conj(Z[256-k])) / 2, O = (Z[k] - conj(Z[256-k])) / 2i, k = 0..256;
        // the spectrum is rounded to complex64 and |X| taken like hypotf (fp64 sum of the exact squares, one rounding to fp32)
        for (int k = lane; k < MEL_NBINS; k += 32) {
            const double2 zk = z[k & (MEL_NC - 1)], zr = z[(MEL_NC - k) & (MEL_NC - 1)];
            const double er = 0.5 * (zk.x + zr.x), ei = 0.5 * (zk.y - zr.y);
            const double orr = 0.5 * (zk.y + zr.y), oi = -0.5 * (zk.x - zr.x);
            const double2 w = k < MEL_NC ? s_tw[k] : make_double2(-1.0, 0.0);
            const float xr = (float)(er + (orr * w.x - oi * w.y));
            const float xi = (float)(ei + (orr * w.y + oi * w.x));
            const float mag = (float)sqrt((double)xr * xr + (double)xi * xi);
            p[k] = mag * mag;
        }
        __syncwarp();
        for (int m = lane; m < n_mels; m += 32) {
            const float* wm = weights + bands.off[m];
            const float* pm = p + bands.start[m];
            const int len = bands.len[m];
            double acc = 0.0;
            for (int j = 0; j < len; ++j) acc += (double)__ldg(wm + j) * (double)pm[j];
            const float mel = (float)acc;
            const float v = (float)log1p((double)mel);      // the correctly rounded float32 log1p
            o[m] = __half2float(__float2half_rn(v));
        }
        __syncwarp();                                       // z and p are rewritten by this warp's next frame
    }
}

}  // namespace mugd

extern "C" int mugd_melspec(mugd_handle* h, const float* y, int64_t n, int64_t ldy, int32_t B,
                            const double* window, const double* twiddle, int32_t n_fft,
                            const int32_t* band_start, const int32_t* band_len, const float* weights, int32_t n_mels,
                            int32_t hop, float* out, int64_t ldo, int32_t T_out, void* stream) {
    using namespace mugd;
    MUGD_REQUIRE(y && window && twiddle && band_start && band_len && weights && out, "melspec: NULL pointer argument");
    MUGD_REQUIRE(n_fft == MEL_NFFT, "melspec: n_fft=%d is not supported (only %d)", n_fft, MEL_NFFT);
    MUGD_REQUIRE(n >= 1 && B >= 1 && hop >= 1, "melspec: need n >= 1, B >= 1, hop >= 1 (n=%lld B=%d hop=%d)", (long long)n, B, hop);
    MUGD_REQUIRE(ldy >= n, "melspec: ldy=%lld < n=%lld", (long long)ldy, (long long)n);
    const int64_t T = 1 + n / hop;
    MUGD_REQUIRE(T_out >= T, "melspec: T_out=%d < 1 + n/hop = %lld frames (truncation is not supported)", T_out, (long long)T);
    MUGD_REQUIRE(n_mels >= 1 && n_mels <= MEL_MAX_MELS, "melspec: n_mels=%d outside [1, %d]", n_mels, MEL_MAX_MELS);
    MUGD_REQUIRE(ldo >= n_mels, "melspec: ldo=%lld < n_mels=%d", (long long)ldo, n_mels);
    MUGD_REQUIRE(aligned16(twiddle) && ((uintptr_t)window & 7u) == 0, "melspec: window / twiddle table alignment");
    MelBands bands;
    int32_t off = 0;
    for (int m = 0; m < n_mels; ++m) {
        MUGD_REQUIRE(band_start[m] >= 0 && band_len[m] >= 0 && band_start[m] + band_len[m] <= MEL_NBINS,
                     "melspec: band %d covers bins [%d, %d + %d), outside [0, %d)", m, band_start[m], band_start[m], band_len[m], MEL_NBINS);
        bands.off[m] = off;
        bands.start[m] = (int16_t)band_start[m];
        bands.len[m] = (int16_t)band_len[m];
        off += band_len[m];
    }
    int32_t sm_count = 0;
    MUGD_REQUIRE(h && mugd_device_info(h, &sm_count, nullptr, nullptr) == MUGD_OK, "melspec: null handle");
    const int64_t n_rows = (int64_t)B * T_out;
    const int64_t blocks = std::min<int64_t>((n_rows + MEL_WARPS - 1) / MEL_WARPS, (int64_t)sm_count * 8);
    melspec_kernel<<<(unsigned)blocks, 32 * MEL_WARPS, 0, (cudaStream_t)stream>>>(
        y, n, ldy, window, reinterpret_cast<const double2*>(twiddle), weights, bands, n_mels, hop, (int)T, T_out, n_rows, out, ldo);
    MUGD_CHECK_CUDA(cudaGetLastError());
    return MUGD_OK;
}

// Shared host/device helpers of libmugd (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <type_traits>
#include <utility>

#include "../../include/mugd.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libmugd is written for sm_90a (H100) only"
#endif

namespace mugd {

void set_error(const char* fmt, ...);

#define MUGD_CHECK_CUDA(expr)                                                             \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            ::mugd::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr,                \
                              cudaGetErrorString(_e));                                    \
            return MUGD_ERR_CUDA;                                                         \
        }                                                                                 \
    } while (0)

#define MUGD_REQUIRE(cond, ...)                                                           \
    do {                                                                                  \
        if (!(cond)) {                                                                    \
            ::mugd::set_error(__VA_ARGS__);                                               \
            return MUGD_ERR_INVALID;                                                      \
        }                                                                                 \
    } while (0)

struct DeviceInfo {
    int device = 0;
    int sm_count = 132;
    int cc_major = 0, cc_minor = 0;
    int max_smem_optin = 0;
    // per-handle switches
    int tc_single_pass = 0;     // opt-in plain-TF32 tensor-core products (NOT fp32-accurate; never used by parity tests / bench)
    int attention_impl = 1;     // 1 = wgmma attention, 0 = exact-fp32 FFMA referee
    int s4conv_impl = 0;        // 0 = automatic, 1 = resident kernel, 2 = streamed kernel (mugd_set_s4conv_impl)
};

// per-family launchers (each validates its descriptor and enqueues kernels on `st`);
// they return the number of kernels launched through *launches (may be null)
// next: the plan's next GEMM that runs on the tensor cores (or NULL); a tensor-core GEMM prefetches its weights into L2
int launch_gemm(const DeviceInfo& dev, const mugd_gemm& g, int default_impl, const mugd_gemm* next, cudaStream_t st, int* launches);
bool gemm_runs_tc(const mugd_gemm& g, int default_impl);
int launch_groupnorm(const DeviceInfo& dev, const mugd_groupnorm& g, cudaStream_t st, int* launches);
int launch_layernorm(const DeviceInfo& dev, const mugd_layernorm& g, cudaStream_t st, int* launches);
int launch_attention(const DeviceInfo& dev, const mugd_attention& a, cudaStream_t st, int* launches);
int launch_s4conv(const DeviceInfo& dev, const mugd_s4conv& s, cudaStream_t st, int* launches);
int launch_ddim_update(const DeviceInfo& dev, const mugd_ddim_update& d, cudaStream_t st, int* launches);
int launch_transpose(const DeviceInfo& dev, const mugd_transpose& t, cudaStream_t st, int* launches);
int launch_copy2d(const DeviceInfo& dev, const mugd_copy2d& c, cudaStream_t st, int* launches);
int launch_step_advance(const DeviceInfo& dev, const mugd_step_advance& a, cudaStream_t st, int* launches);
int launch_notes(const DeviceInfo& dev, const mugd_notes& n, cudaStream_t st, int* launches);
int launch_embed(const DeviceInfo& dev, const mugd_embed& e, cudaStream_t st, int* launches);
int launch_tf32_split(const DeviceInfo& dev, const mugd_tf32_split& s, cudaStream_t st, int* launches);
int launch_posterior(const DeviceInfo& dev, const mugd_posterior& p, cudaStream_t st, int* launches);
// ragged batches: valid[b] rows per sample (norm.cu, attention.cu, elementwise.cu)
int launch_groupnorm_var(const DeviceInfo& dev, const mugd_groupnorm_var& g, cudaStream_t st, int* launches);
int launch_attention_var(const DeviceInfo& dev, const mugd_attention_var& a, cudaStream_t st, int* launches);
int launch_row_mask(const DeviceInfo& dev, const mugd_row_mask& m, cudaStream_t st, int* launches);
// section prompts: a cross-attention whose keys / values change along the rows (attention.cu)
int launch_attention_sec(const DeviceInfo& dev, const mugd_attention_sec& a, cudaStream_t st, int* launches);
// per-chart guidance scales (elementwise.cu)
int launch_cfg_scales(const DeviceInfo& dev, const mugd_cfg_scales& g, cudaStream_t st, int* launches);
// mugd_sample_staged: check_stage validates a stage for n_steps (host arrays included); launch_stage runs step i of it
int check_stage(const mugd_stage& s, int32_t n_steps);
int launch_stage(const mugd_stage& s, int32_t i, cudaStream_t st);
// mugd_sample_plms / mugd_plms_combine: check_plms validates the descriptor; launch_plms_combine runs the combine of step `step`
// (heun = 1: the second half of step 0)
int check_plms(const mugd_plms& p);
int launch_plms_combine(const mugd_plms& p, int32_t step, int heun, cudaStream_t st);
// mugd_sample_ddpm / mugd_ddpm_update: check_ddpm validates the descriptor; launch_ddpm_update runs the update on noise row k
int check_ddpm(const mugd_ddpm& d);
int launch_ddpm_update(const mugd_ddpm& d, int32_t k, cudaStream_t st);
// mugd_sample_dpm / mugd_dpm_update: check_dpm validates the descriptor; launch_dpm_update runs the update of the counter's step
int check_dpm(const mugd_dpm& d);
int launch_dpm_update(const mugd_dpm& d, cudaStream_t st);
// mugd_sample_dpm_ex / mugd_dpm_ex_update: check_dpm_ex validates the descriptor for a call of n_steps (the stage's host table
// included); launch_dpm_ex_update runs the update of the counter's step, per-chart when starts are given
int check_dpm_ex(const mugd_dpm_ex& e, int32_t n_steps);
int launch_dpm_ex_update(const mugd_dpm_ex& e, cudaStream_t st);
// mugd_sample_dpm_stop / mugd_dpm_stop_update: check_dpm_stop validates the descriptor; launch_dpm_stop_update runs the inversion
// update of the counter's step for the charts that have not reached their stop
int check_dpm_stop(const mugd_dpm_stop& e);
int launch_dpm_stop_update(const mugd_dpm_stop& e, cudaStream_t st);
// mugd_sample_unipc / mugd_unipc_update: check_unipc validates the descriptor; launch_unipc_update runs the UniPC update of the
// counter's step
int check_unipc(const mugd_unipc& u);
int launch_unipc_update(const mugd_unipc& u, cudaStream_t st);
// mugd_sample_unipc_ex / mugd_unipc_ex_update and mugd_sample_unipc_stop / mugd_unipc_stop_update: the UniPC counterparts of the
// DPM-Solver++ ex and stop pairs above
int check_unipc_ex(const mugd_unipc_ex& e, int32_t n_steps);
int launch_unipc_ex_update(const mugd_unipc_ex& e, cudaStream_t st);
int check_unipc_stop(const mugd_unipc_stop& e);
int launch_unipc_stop_update(const mugd_unipc_stop& e, cudaStream_t st);
// mugd_sample_join: check_join validates the descriptor; launch_join runs the join kernel against the device step counter
int check_join(const mugd_join& j);
int launch_join(const mugd_join& j, const int32_t* step, cudaStream_t st);
int launch_gemm_tc(const DeviceInfo& dev, const mugd_gemm& g, const mugd_gemm* next, cudaStream_t st, int* launches);
// MUGD_OP_GEMM_SERIAL: the forced K split (g.split_k) of a tensor-core GEMM finished inside each CTA.  validate_gemm_serial runs every
// check of the op on the host; launch_gemm_serial runs them before its launch.
int validate_gemm(const mugd_gemm& g);
int validate_gemm_serial(const mugd_gemm& g, int default_impl);
int launch_gemm_serial(const DeviceInfo& dev, const mugd_gemm& g, int default_impl, const mugd_gemm* next, cudaStream_t st, int* launches);
bool gemm_tc_supported(const mugd_gemm& g);

// Descriptor checks shared by the sampler kernels; `who` prefixes the message ("ddpm", "dpm", ...).
// cfg selects classifier-free guidance: 0 or 1.
inline int check_cfg(const char* who, int cfg) {
    MUGD_REQUIRE(cfg == 0 || cfg == 1, "%s: cfg=%d", who, cfg);
    return MUGD_OK;
}
inline int check_scale(const char* who, float scale) {
    MUGD_REQUIRE(isfinite(scale), "%s: scale is not finite", who);
    return MUGD_OK;
}
// The evaluation reads x in both CFG halves, so an update that writes x writes its CFG copy exactly when cfg = 1.
inline int check_x_dup(const char* who, const float* x_dup, int cfg) {
    MUGD_REQUIRE(!x_dup == !cfg, "%s: x_dup must be given exactly when cfg = 1 (the evaluation reads x in both halves)", who);
    return MUGD_OK;
}
// A kernel over 32x32 (channel, position) tiles of B samples [C, L]: int32 element indices, grid (L/32, C/32, B).
inline int check_tile_grid(const char* who, int32_t B, int32_t C, int32_t L) {
    MUGD_REQUIRE(B > 0 && C > 0 && L > 0 && (int64_t)B * C * L <= INT32_MAX, "%s: bad shape B=%d C=%d L=%d", who, B, C, L);
    MUGD_REQUIRE(B <= 65535 && (C + 31) / 32 <= 65535, "%s: B=%d / C=%d too large for one launch", who, B, C);
    return MUGD_OK;
}

// Kernels that need more than 48 KB of dynamic shared memory are allowed the device's opt-in maximum (`bytes`) by mugd_create, after
// its cudaSetDevice: the attribute belongs to the current device's context, so it is set once for every device a handle is created
// on.  A launch still asks for only its own byte count, so occupancy and the shared-memory carve-out do not change.  Each kernel
// file lists its own instantiations.
cudaError_t gemm_tc_allow_smem(int bytes);
cudaError_t attention_tc_allow_smem(int bytes);
cudaError_t attention_allow_smem(int bytes);
cudaError_t s4_allow_smem(int bytes);

// Programmatic dependent launch (PDL): every hot-path kernel is launched with the programmatic-stream-serialization
// attribute and executes `griddepcontrol.wait` (pdl_wait) before its first access to memory the previous kernel wrote.  The next
// kernel's launch latency and prologue (block scheduling, barrier init, tensor-map fetch) then overlap the tail of the current one;
// data hazards are unchanged because the wait only returns when the prerequisite grid has completed and flushed.
extern bool g_use_pdl;

#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = g_use_pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
// Lets each kernel launch with up to `bytes` of dynamic shared memory on the current device.
template <typename... Kernels>
inline cudaError_t allow_dynamic_smem(int bytes, Kernels... kernels) {
    cudaError_t e = cudaSuccess;
    ((e = (e == cudaSuccess) ? cudaFuncSetAttribute(kernels, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) : e), ...);
    return e;
}
// No kernel signals launch_dependents explicitly: the trigger is implicit at grid completion, so PDL only overlaps the dependent's
// launch with this grid's memory flush.  Explicit triggers
// (at entry, in the short kernels only, after the GEMM main loop) were tried and not kept.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// The guidance combine e_u + scale * (e_c - e_u) (ddim.py:175), each operation one IEEE round-to-nearest in torch's eager order, no
// contraction.  cfg_eps and the per-chart-scale kernel (MUGD_OP_CFG_SCALES) both form it here, so they agree bit for bit.
__device__ __forceinline__ float cfg_guide(float eu, float ec, float scale) {
    return __fadd_rn(eu, __fmul_rn(scale, __fsub_rn(ec, eu)));
}

// The noise prediction of element i of the sampler's eps rows: with cfg, cfg_guide of the uncond half [0, n) and the cond half
// [n, 2n).  Every update kernel forms e here, so all of them match torch bit for bit.
__device__ __forceinline__ float cfg_eps(const float* eps, int64_t i, int64_t n, int cfg, float scale) {
    if (!cfg) return eps[i];
    return cfg_guide(eps[i], eps[n + i], scale);
}

// Loads the 32x32 tile at (c0, l0) of one sample's NCL rows `in` [C, L] into tile[c - c0][l - l0], coalesced along L by a CTA of
// 32 x 8 threads; entries past C or L are left unwritten.  The [32][33] padding keeps the transposed reads tile[tx][r] free of bank
// conflicts.
__device__ __forceinline__ void load_ncl_tile(float (&tile)[32][33], const float* in, int c0, int l0, int C, int L) {
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
    for (int r = ty; r < 32; r += 8) {
        const int c = c0 + r, l = l0 + tx;
        if (c < C && l < L) tile[r][tx] = in[(int64_t)c * L + l];
    }
}

// ---- device helpers ---------------------------------------------------------------------------
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }
// exact-erf GELU (nn.GELU() default; attention.py:45, s4.py:187-188)
__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// Attention kernels are instantiated for the descriptors: mugd_attention (every row valid), mugd_attention_var (ragged batches,
// sample b's first clamp(valid[b], 0, n) rows valid) and, in attention.cu, mugd_attention_sec (section prompts, every row valid).
// With the plain descriptor attn_rows() is n, so those instances compile to the code they had before ragged batches existed.
__host__ __device__ __forceinline__ const mugd_attention& attn_desc(const mugd_attention& a) { return a; }
__host__ __device__ __forceinline__ const mugd_attention& attn_desc(const mugd_attention_var& a) { return a.attn; }
__host__ __device__ __forceinline__ const mugd_attention& attn_desc(const mugd_attention_sec& a) { return a.attn; }
__device__ __forceinline__ int attn_rows(const mugd_attention&, int, int n) { return n; }
__device__ __forceinline__ int attn_rows(const mugd_attention_var& a, int b, int n) { return min(max(a.valid[b], 0), n); }
__device__ __forceinline__ int attn_rows(const mugd_attention_sec&, int, int n) { return n; }
template <typename Desc> constexpr bool attn_is_var = std::is_same<Desc, mugd_attention_var>::value;
template <typename Desc> constexpr bool attn_is_sec = std::is_same<Desc, mugd_attention_sec>::value;

__device__ __forceinline__ float4 ld_f4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st_f4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
#endif

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace mugd

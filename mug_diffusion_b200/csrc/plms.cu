// PLMS sampler (pseudo linear multistep, mug/diffusion/plms.py:115-236): the noise-prediction combine of one step.  The x update
// that follows it is MUGD_OP_DDIM_UPDATE with cfg = 0 on e' (get_x_prev_and_pred_x0, plms.py:199-216, is p_sample_ddim's update);
// the loop mugd_sample_plms lives in api.cu beside mugd_sample.
#include "common.cuh"

namespace mugd {

// One thread per element of the [B*L, C] rows.  e_t is the CFG combine of plms.py:182-186 (uncond half first); e' follows
// plms.py:219-232.  Every operation is one IEEE round-to-nearest in torch's eager order, no contraction.  torch's CUDA eager ops
// divide by a Python scalar as a multiply by its float reciprocal (div_true with a CPU scalar), so `/ 2`, `/ 12` and `/ 24` are
// multiplies by 0.5f, 1.0f/12 and 1.0f/24 rounded to float.
//   heun = 0: order k = min(step, 3) previous e_t in the ring (slot of step j = j mod 3); e_t goes to slot `slot`
//   heun = 1: e' = (e_t + e_t_next) / 2 with e_t in slot 0 and this evaluation giving e_t_next; the ring is not written
__global__ void __launch_bounds__(256)
plms_combine_kernel(const float* __restrict__ eps, float* __restrict__ hist, float* __restrict__ e_prime, int n, int cfg, float scale,
                    int order, int slot, int heun) {
    pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float e = cfg_eps(eps, i, n, cfg, scale);                                                // plms.py:186
    const int64_t N = n;
    float ep;
    if (heun) {
        ep = __fmul_rn(__fadd_rn(hist[i], e), 0.5f);                                               // :223
    } else {
        const float o1 = order >= 1 ? hist[((slot + 2) % 3) * N + i] : 0.0f;                      // old_eps[-1]: step - 1
        const float o2 = order >= 2 ? hist[((slot + 1) % 3) * N + i] : 0.0f;                      // old_eps[-2]: step - 2
        const float o3 = order >= 3 ? hist[slot * N + i] : 0.0f;                                  // old_eps[-3]: step - 3, read first
        if (order == 0) {
            ep = e;                                                                                // the Euler half of step 0
        } else if (order == 1) {
            ep = __fmul_rn(__fsub_rn(__fmul_rn(3.0f, e), o1), 0.5f);                              // :226
        } else if (order == 2) {
            ep = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(23.0f, e), __fmul_rn(16.0f, o1)), __fmul_rn(5.0f, o2)), 1.0f / 12.0f);  // :229
        } else {
            ep = __fmul_rn(__fsub_rn(__fadd_rn(__fsub_rn(__fmul_rn(55.0f, e), __fmul_rn(59.0f, o1)), __fmul_rn(37.0f, o2)),
                                     __fmul_rn(9.0f, o3)),
                           1.0f / 24.0f);                                                          // :232
        }
        hist[slot * N + i] = e;                                                                    // old_eps.append(e_t), :160-162
    }
    e_prime[i] = ep;
}

int check_plms(const mugd_plms& p) {
    const mugd_ddim_update& u = p.update;
    MUGD_REQUIRE(p.eps && p.e_prime && p.hist && p.x_stash, "plms: eps, e_prime, hist and x_stash must be given");
    MUGD_REQUIRE(u.x && u.coef && u.step, "plms: update.x, update.coef and update.step must be given");
    MUGD_REQUIRE(u.n > 0 && u.S > 0, "plms: bad update (n=%d, S=%d)", u.n, u.S);
    MUGD_REQUIRE(u.eps == p.e_prime, "plms: update.eps must be e_prime (the update runs on e')");
    MUGD_REQUIRE(u.cfg == 0, "plms: update.cfg must be 0 (the combine kernel applies the guidance)");
    MUGD_REQUIRE(u.noise == nullptr, "plms: update.noise must be NULL (PLMS runs at eta = 0)");
    int rc = check_cfg("plms", p.cfg);
    if (rc != MUGD_OK) return rc;
    return check_scale("plms", p.scale);
}

int launch_plms_combine(const mugd_plms& p, int32_t step, int heun, cudaStream_t st) {
    const int n = p.update.n;
    const int order = heun ? 0 : (step < 3 ? step : 3);
    MUGD_CHECK_CUDA(launch_k(plms_combine_kernel, dim3((n + 255) / 256), dim3(256), 0, st, p.eps, p.hist, p.e_prime, n, p.cfg, p.scale,
                             order, (int)(step % 3), heun));
    return MUGD_OK;
}

}  // namespace mugd

using namespace mugd;

extern "C" int mugd_plms_combine(const mugd_plms* p, int32_t step, int32_t heun, void* stream) {
    MUGD_REQUIRE(p, "mugd_plms_combine: null argument");
    int rc = check_plms(*p);
    if (rc != MUGD_OK) return rc;
    MUGD_REQUIRE(step >= 0 && step < p->update.S, "mugd_plms_combine: step=%d outside [0, S=%d)", step, p->update.S);
    MUGD_REQUIRE(heun == 0 || (heun == 1 && step == 0), "mugd_plms_combine: heun=%d at step %d (Heun mode is step 0's)", heun, step);
    return launch_plms_combine(*p, step, heun, (cudaStream_t)stream);
}

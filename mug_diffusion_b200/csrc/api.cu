// C ABI glue of libmugd: handle, op dispatch, launch plans and CUDA-graph capture/replay.
#include <stdarg.h>
#include <string.h>

#include <vector>

#include "common.cuh"

namespace mugd {

static thread_local char g_err[1024] = "";
// Programmatic launch edges with the implicit (grid-completion) trigger: a shorter edge between dependent kernels.  This is a
// launch attribute without numerical effect; it is process-wide because launch_k() has no handle (mugd_set_pdl is an A/B switch).
bool g_use_pdl = true;

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

}  // namespace mugd

struct mugd_handle {
    mugd::DeviceInfo dev;
    int default_gemm_impl = MUGD_GEMM_SIMT;
};

struct mugd_plan {
    mugd_handle* h = nullptr;
    std::vector<mugd_op> ops;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    int launches = 0;
};

namespace mugd {

const std::vector<mugd_op>& plan_ops(const mugd_plan* p) { return p->ops; }
int plan_from_ops(mugd_handle* h, const mugd_op* ops, int32_t n, mugd_plan** out) { return mugd_plan_create(h, ops, n, out); }

// next_tc: the next tensor-core GEMM after `op` in its plan (NULL outside a plan): a GEMM op prefetches its weights
static int dispatch(mugd_handle* h, const mugd_op& op, cudaStream_t st, int* launches, const mugd_gemm* next_tc = nullptr) {
    switch (op.kind) {
        case MUGD_OP_GEMM: return launch_gemm(h->dev, op.u.gemm, h->default_gemm_impl, next_tc, st, launches);
        case MUGD_OP_GROUPNORM: return launch_groupnorm(h->dev, op.u.gn, st, launches);
        case MUGD_OP_LAYERNORM: return launch_layernorm(h->dev, op.u.ln, st, launches);
        case MUGD_OP_ATTENTION: return launch_attention(h->dev, op.u.attn, st, launches);
        case MUGD_OP_S4CONV: return launch_s4conv(h->dev, op.u.s4, st, launches);
        case MUGD_OP_DDIM_UPDATE: return launch_ddim_update(h->dev, op.u.ddim, st, launches);
        case MUGD_OP_TRANSPOSE: return launch_transpose(h->dev, op.u.tr, st, launches);
        case MUGD_OP_COPY2D: return launch_copy2d(h->dev, op.u.cp, st, launches);
        case MUGD_OP_STEP_ADVANCE: return launch_step_advance(h->dev, op.u.adv, st, launches);
        case MUGD_OP_NOTES: return launch_notes(h->dev, op.u.notes, st, launches);
        case MUGD_OP_EMBED: return launch_embed(h->dev, op.u.embed, st, launches);
        case MUGD_OP_TF32_SPLIT: return launch_tf32_split(h->dev, op.u.split, st, launches);
        case MUGD_OP_POSTERIOR: return launch_posterior(h->dev, op.u.post, st, launches);
        default:
            set_error("unknown op kind %d", op.kind);
            return MUGD_ERR_INVALID;
    }
}

}  // namespace mugd

using namespace mugd;

extern "C" {

int mugd_abi_version(void) { return MUGD_ABI_VERSION; }

const char* mugd_last_error(void) { return g_err; }

int mugd_create(int device, mugd_handle** out) {
    MUGD_REQUIRE(out, "mugd_create: null out");
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0 || device < 0 || device >= n) {
        set_error("mugd_create: no CUDA device %d (count=%d, %s). libmugd has no CPU fallback.", device, n,
                  e == cudaSuccess ? "ok" : cudaGetErrorString(e));
        return MUGD_ERR_NO_DEVICE;
    }
    cudaDeviceProp prop;
    MUGD_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_error("mugd_create: device %d is sm_%d%d; libmugd is built for sm_90a (H100) only", device, prop.major, prop.minor);
        return MUGD_ERR_NO_DEVICE;
    }
    MUGD_CHECK_CUDA(cudaSetDevice(device));
    const int smem_optin = (int)prop.sharedMemPerBlockOptin;
    MUGD_CHECK_CUDA(gemm_tc_allow_smem(smem_optin));
    MUGD_CHECK_CUDA(attention_tc_allow_smem(smem_optin));
    MUGD_CHECK_CUDA(attention_allow_smem(smem_optin));
    MUGD_CHECK_CUDA(s4_allow_smem(smem_optin));
    mugd_handle* h = new mugd_handle();
    h->dev.device = device;
    h->dev.sm_count = prop.multiProcessorCount;
    h->dev.cc_major = prop.major;
    h->dev.cc_minor = prop.minor;
    h->dev.max_smem_optin = smem_optin;
    *out = h;
    return MUGD_OK;
}

void mugd_destroy(mugd_handle* h) { delete h; }

int mugd_device_info(mugd_handle* h, int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor) {
    MUGD_REQUIRE(h, "null handle");
    if (sm_count) *sm_count = h->dev.sm_count;
    if (cc_major) *cc_major = h->dev.cc_major;
    if (cc_minor) *cc_minor = h->dev.cc_minor;
    return MUGD_OK;
}

int mugd_set_gemm_impl(mugd_handle* h, int impl) {
    MUGD_REQUIRE(h, "null handle");
    MUGD_REQUIRE(impl == MUGD_GEMM_SIMT || impl == MUGD_GEMM_TC, "set_gemm_impl: %d", impl);
    h->default_gemm_impl = impl;
    return MUGD_OK;
}

int mugd_set_tc_single_pass_tf32(mugd_handle* h, int enabled) {
    MUGD_REQUIRE(h, "null handle");
    h->dev.tc_single_pass = enabled ? 1 : 0;
    return MUGD_OK;
}

int mugd_set_attention_impl(mugd_handle* h, int impl) {
    MUGD_REQUIRE(h, "null handle");
    h->dev.attention_impl = impl ? 1 : 0;
    return MUGD_OK;
}

int mugd_set_s4conv_impl(mugd_handle* h, int impl) {
    MUGD_REQUIRE(h, "null handle");
    MUGD_REQUIRE(impl >= 0 && impl <= 2, "set_s4conv_impl: %d (0 = automatic, 1 = resident, 2 = streamed)", impl);
    h->dev.s4conv_impl = impl;
    return MUGD_OK;
}

int mugd_set_pdl(int enabled) {
    g_use_pdl = enabled != 0;
    return MUGD_OK;
}

int mugd_op_run(mugd_handle* h, const mugd_op* op, void* stream) {
    MUGD_REQUIRE(h && op, "mugd_op_run: null argument");
    return dispatch(h, *op, (cudaStream_t)stream, nullptr);
}

int mugd_plan_create(mugd_handle* h, const mugd_op* ops, int32_t n_ops, mugd_plan** out) {
    MUGD_REQUIRE(h && ops && out && n_ops > 0, "mugd_plan_create: bad arguments");
    mugd_plan* p = new mugd_plan();
    p->h = h;
    p->ops.assign(ops, ops + n_ops);
    *out = p;
    return MUGD_OK;
}

int mugd_plan_run(mugd_plan* p, void* stream) {
    MUGD_REQUIRE(p, "null plan");
    int launches = 0;
    const size_t n = p->ops.size();
    std::vector<const mugd_gemm*> next_tc(n, nullptr);
    for (size_t i = n; i-- > 1;) {
        const mugd_op& o = p->ops[i];
        next_tc[i - 1] = o.kind == MUGD_OP_GEMM && gemm_runs_tc(o.u.gemm, p->h->default_gemm_impl) ? &o.u.gemm : next_tc[i];
    }
    for (size_t i = 0; i < n; ++i) {
        int rc = dispatch(p->h, p->ops[i], (cudaStream_t)stream, &launches, next_tc[i]);
        if (rc != MUGD_OK) {
            char prev[900];
            strncpy(prev, g_err, sizeof(prev) - 1);
            prev[sizeof(prev) - 1] = 0;
            set_error("plan op %zu (kind %d, tag %d): %s", i, p->ops[i].kind, p->ops[i].tag, prev);
            return rc;
        }
    }
    p->launches = launches;
    return MUGD_OK;
}

int mugd_plan_capture(mugd_plan* p, void* stream) {
    MUGD_REQUIRE(p, "null plan");
    cudaStream_t st = (cudaStream_t)stream;
    MUGD_REQUIRE(st != nullptr, "plan_capture: needs a non-default stream");
    if (p->exec) { cudaGraphExecDestroy(p->exec); p->exec = nullptr; }
    if (p->graph) { cudaGraphDestroy(p->graph); p->graph = nullptr; }
    MUGD_CHECK_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    int rc = mugd_plan_run(p, stream);
    cudaGraph_t g = nullptr;
    cudaError_t e = cudaStreamEndCapture(st, &g);
    if (rc != MUGD_OK) {
        if (g) cudaGraphDestroy(g);
        return rc;
    }
    if (e != cudaSuccess) {
        set_error("cudaStreamEndCapture: %s", cudaGetErrorString(e));
        return MUGD_ERR_CUDA;
    }
    p->graph = g;
    MUGD_CHECK_CUDA(cudaGraphInstantiate(&p->exec, p->graph, 0));
    return MUGD_OK;
}

int mugd_plan_replay(mugd_plan* p, int32_t times, void* stream) {
    MUGD_REQUIRE(p && p->exec, "plan_replay: plan not captured");
    for (int i = 0; i < times; ++i) MUGD_CHECK_CUDA(cudaGraphLaunch(p->exec, (cudaStream_t)stream));
    return MUGD_OK;
}

int mugd_sample(mugd_plan* eval_plan, const mugd_op* tail, int32_t n_tail, int32_t n_steps, void* stream) {
    MUGD_REQUIRE(eval_plan && eval_plan->exec, "mugd_sample: the evaluation plan must be captured (mugd_plan_capture)");
    MUGD_REQUIRE(n_steps >= 0 && n_tail >= 0 && (n_tail == 0 || tail), "mugd_sample: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    for (int i = 0; i < n_steps; ++i) {
        MUGD_CHECK_CUDA(cudaGraphLaunch(eval_plan->exec, st));
        for (int k = 0; k < n_tail; ++k) {
            int rc = dispatch(eval_plan->h, tail[k], st, nullptr);
            if (rc != MUGD_OK) return rc;
        }
    }
    return MUGD_OK;
}

int mugd_sample_staged(mugd_plan* eval_plan, const mugd_stage* stage, const mugd_op* tail, int32_t n_tail, int32_t n_steps,
                       void* stream) {
    MUGD_REQUIRE(eval_plan && eval_plan->exec, "mugd_sample_staged: the evaluation plan must be captured (mugd_plan_capture)");
    MUGD_REQUIRE(stage, "mugd_sample_staged: null stage");
    MUGD_REQUIRE(n_steps >= 0, "mugd_sample_staged: n_steps=%d < 0", n_steps);
    MUGD_REQUIRE(n_tail >= 0 && (n_tail == 0 || tail), "mugd_sample_staged: bad tail (n_tail=%d)", n_tail);
    const mugd_stage& s = *stage;
    int rc = check_stage(s, n_steps);
    if (rc != MUGD_OK) return rc;
    const int64_t n = (int64_t)s.B * s.C * s.L;
    for (int k = 0; k < n_tail; ++k) {
        if (tail[k].kind != MUGD_OP_DDIM_UPDATE) continue;
        const mugd_ddim_update& d = tail[k].u.ddim;
        MUGD_REQUIRE(d.x == s.x && d.x_dup == s.x_dup, "mugd_sample_staged: tail op %d updates other rows than the stage's x / x_dup", k);
        MUGD_REQUIRE(d.n == n, "mugd_sample_staged: tail op %d updates n=%d elements, the stage B*C*L=%lld", k, d.n, (long long)n);
        MUGD_REQUIRE(!s.noise || d.noise == s.noise_rows, "mugd_sample_staged: tail op %d reads its noise from other rows than noise_rows",
                     k);
    }
    const bool staged = s.x0 || s.noise;
    cudaStream_t st = (cudaStream_t)stream;
    for (int i = 0; i < n_steps; ++i) {
        if (staged) {
            rc = launch_stage(s, i, st);
            if (rc != MUGD_OK) return rc;
        }
        MUGD_CHECK_CUDA(cudaGraphLaunch(eval_plan->exec, st));
        for (int k = 0; k < n_tail; ++k) {
            rc = dispatch(eval_plan->h, tail[k], st, nullptr);
            if (rc != MUGD_OK) return rc;
        }
    }
    return MUGD_OK;
}

int mugd_sample_plms(mugd_plan* eval_plan, const mugd_plms* p, int32_t first_step, int32_t n_steps, void* stream) {
    MUGD_REQUIRE(eval_plan && eval_plan->exec, "mugd_sample_plms: the evaluation plan must be captured (mugd_plan_capture)");
    MUGD_REQUIRE(p, "mugd_sample_plms: null plms");
    int rc = check_plms(*p);
    if (rc != MUGD_OK) return rc;
    const mugd_ddim_update& u = p->update;
    MUGD_REQUIRE(first_step >= 0 && n_steps >= 0 && (int64_t)first_step + n_steps <= u.S,
                 "mugd_sample_plms: first_step=%d, n_steps=%d outside the S=%d steps of the request", first_step, n_steps, u.S);
    const DeviceInfo& dev = eval_plan->h->dev;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t xbytes = sizeof(float) * (size_t)u.n;
    int32_t* const step = const_cast<int32_t*>(u.step);      // the update reads the counter this loop sets and advances
    mugd_step_advance adv;
    adv.step = step;
    for (int32_t i = first_step; i < first_step + n_steps; ++i) {
        MUGD_CHECK_CUDA(cudaGraphLaunch(eval_plan->exec, st));
        if ((rc = launch_plms_combine(*p, i, 0, st)) != MUGD_OK) return rc;
        if (i == 0) {
            // pseudo improved Euler (plms.py:219-223): the Euler x_prev of e_t goes into both CFG halves of the input rows, the plan
            // evaluates it at t_next = time_range[min(1, S - 1)] (:145), then x is restored and e' = (e_t + e_t_next) / 2
            MUGD_CHECK_CUDA(cudaMemcpyAsync(p->x_stash, u.x, xbytes, cudaMemcpyDeviceToDevice, st));
            if ((rc = launch_ddim_update(dev, u, st, nullptr)) != MUGD_OK) return rc;
            if ((rc = mugd_fill_i32(step, u.S > 1 ? 1 : 0, stream)) != MUGD_OK) return rc;
            MUGD_CHECK_CUDA(cudaGraphLaunch(eval_plan->exec, st));
            MUGD_CHECK_CUDA(cudaMemcpyAsync(u.x, p->x_stash, xbytes, cudaMemcpyDeviceToDevice, st));
            if ((rc = launch_plms_combine(*p, 0, 1, st)) != MUGD_OK) return rc;
            if ((rc = mugd_fill_i32(step, 0, stream)) != MUGD_OK) return rc;
        }
        if ((rc = launch_ddim_update(dev, u, st, nullptr)) != MUGD_OK) return rc;
        if ((rc = launch_step_advance(dev, adv, st, nullptr)) != MUGD_OK) return rc;
    }
    return MUGD_OK;
}

int mugd_sample_ddpm(mugd_plan* eval_plan, const mugd_ddpm* d, int32_t first_step, int32_t n_steps, void* stream) {
    MUGD_REQUIRE(eval_plan && eval_plan->exec, "mugd_sample_ddpm: the evaluation plan must be captured (mugd_plan_capture)");
    MUGD_REQUIRE(d, "mugd_sample_ddpm: null ddpm");
    int rc = check_ddpm(*d);
    if (rc != MUGD_OK) return rc;
    MUGD_REQUIRE(first_step >= 0 && n_steps >= 0 && (int64_t)first_step + n_steps <= d->T,
                 "mugd_sample_ddpm: first_step=%d, n_steps=%d outside the T=%d steps of the request", first_step, n_steps, d->T);
    const DeviceInfo& dev = eval_plan->h->dev;
    cudaStream_t st = (cudaStream_t)stream;
    mugd_step_advance adv;
    adv.step = d->step;
    for (int32_t k = 0; k < n_steps; ++k) {
        MUGD_CHECK_CUDA(cudaGraphLaunch(eval_plan->exec, st));
        if ((rc = launch_ddpm_update(*d, k, st)) != MUGD_OK) return rc;
        if ((rc = launch_step_advance(dev, adv, st, nullptr)) != MUGD_OK) return rc;
    }
    return MUGD_OK;
}

int mugd_sample_dpm(mugd_plan* eval_plan, const mugd_dpm* d, int32_t first_step, int32_t n_steps, void* stream) {
    MUGD_REQUIRE(eval_plan && eval_plan->exec, "mugd_sample_dpm: the evaluation plan must be captured (mugd_plan_capture)");
    MUGD_REQUIRE(d, "mugd_sample_dpm: null dpm");
    int rc = check_dpm(*d);
    if (rc != MUGD_OK) return rc;
    MUGD_REQUIRE(first_step >= 0 && n_steps >= 0 && (int64_t)first_step + n_steps <= d->S,
                 "mugd_sample_dpm: first_step=%d, n_steps=%d outside the S=%d steps of the request", first_step, n_steps, d->S);
    const DeviceInfo& dev = eval_plan->h->dev;
    cudaStream_t st = (cudaStream_t)stream;
    mugd_step_advance adv;
    adv.step = d->step;
    for (int32_t k = 0; k < n_steps; ++k) {
        MUGD_CHECK_CUDA(cudaGraphLaunch(eval_plan->exec, st));
        if ((rc = launch_dpm_update(*d, st)) != MUGD_OK) return rc;
        if ((rc = launch_step_advance(dev, adv, st, nullptr)) != MUGD_OK) return rc;
    }
    return MUGD_OK;
}

int mugd_sample_dpm_ex(mugd_plan* eval_plan, const mugd_dpm_ex* e, int32_t first_step, int32_t n_steps, void* stream) {
    // the descriptor is checked before the plan, so a host can test its arguments without a device
    MUGD_REQUIRE(e, "mugd_sample_dpm_ex: null descriptor");
    int rc = check_dpm_ex(*e, n_steps);
    if (rc != MUGD_OK) return rc;
    MUGD_REQUIRE(first_step >= 0 && n_steps >= 0 && (int64_t)first_step + n_steps <= e->dpm.S,
                 "mugd_sample_dpm_ex: first_step=%d, n_steps=%d outside the S=%d steps of the request", first_step, n_steps, e->dpm.S);
    MUGD_REQUIRE(eval_plan && eval_plan->exec, "mugd_sample_dpm_ex: the evaluation plan must be captured (mugd_plan_capture)");
    const DeviceInfo& dev = eval_plan->h->dev;
    cudaStream_t st = (cudaStream_t)stream;
    mugd_step_advance adv;
    adv.step = e->dpm.step;
    for (int32_t k = 0; k < n_steps; ++k) {
        if (e->stage && (rc = launch_stage(*e->stage, k, st)) != MUGD_OK) return rc;
        MUGD_CHECK_CUDA(cudaGraphLaunch(eval_plan->exec, st));
        if ((rc = launch_dpm_ex_update(*e, st)) != MUGD_OK) return rc;
        if ((rc = launch_step_advance(dev, adv, st, nullptr)) != MUGD_OK) return rc;
    }
    return MUGD_OK;
}

int mugd_sample_join(mugd_plan* eval_plan, const mugd_join* join, const mugd_op* tail, int32_t n_tail, int32_t first_step,
                     int32_t n_steps, void* stream) {
    MUGD_REQUIRE(eval_plan && eval_plan->exec, "mugd_sample_join: the evaluation plan must be captured (mugd_plan_capture)");
    MUGD_REQUIRE(join, "mugd_sample_join: null join");
    MUGD_REQUIRE(n_tail >= 0 && (n_tail == 0 || tail), "mugd_sample_join: bad tail (n_tail=%d)", n_tail);
    const mugd_join& j = *join;
    int rc = check_join(j);
    if (rc != MUGD_OK) return rc;
    const int64_t n = (int64_t)j.B * j.C * j.L;
    const mugd_ddim_update* upd = nullptr;
    for (int k = 0; k < n_tail; ++k) {
        if (tail[k].kind != MUGD_OP_DDIM_UPDATE) continue;
        MUGD_REQUIRE(!upd, "mugd_sample_join: the tail holds more than one DDIM update (op %d)", k);
        upd = &tail[k].u.ddim;
        MUGD_REQUIRE(upd->x == j.x && upd->x_dup == j.x_dup, "mugd_sample_join: tail op %d updates other rows than the join's x / x_dup", k);
        MUGD_REQUIRE(upd->n == n, "mugd_sample_join: tail op %d updates n=%d elements, the join B*C*L=%lld", k, upd->n, (long long)n);
        MUGD_REQUIRE(upd->step, "mugd_sample_join: tail op %d has no device step counter", k);
    }
    MUGD_REQUIRE(upd, "mugd_sample_join: the tail holds no DDIM update");
    MUGD_REQUIRE(first_step >= 0 && n_steps >= 0 && (int64_t)first_step + n_steps <= upd->S,
                 "mugd_sample_join: first_step=%d, n_steps=%d outside the S=%d steps of the request", first_step, n_steps, upd->S);
    cudaStream_t st = (cudaStream_t)stream;
    for (int i = 0; i < n_steps; ++i) {
        if ((rc = launch_join(j, upd->step, st)) != MUGD_OK) return rc;
        MUGD_CHECK_CUDA(cudaGraphLaunch(eval_plan->exec, st));
        for (int k = 0; k < n_tail; ++k) {
            rc = dispatch(eval_plan->h, tail[k], st, nullptr);
            if (rc != MUGD_OK) return rc;
        }
    }
    return MUGD_OK;
}

int mugd_abi_sizes(int32_t* out, int32_t n) {
    MUGD_REQUIRE(out && n >= 13, "abi_sizes: need room for 13 entries");
    out[0] = sizeof(mugd_op); out[1] = sizeof(mugd_gemm); out[2] = sizeof(mugd_groupnorm);
    out[3] = sizeof(mugd_layernorm); out[4] = sizeof(mugd_attention); out[5] = sizeof(mugd_s4conv);
    out[6] = sizeof(mugd_ddim_update); out[7] = sizeof(mugd_transpose); out[8] = sizeof(mugd_copy2d);
    out[9] = sizeof(mugd_notes); out[10] = sizeof(mugd_embed); out[11] = sizeof(mugd_tf32_split);
    out[12] = sizeof(mugd_posterior);
    return MUGD_OK;
}

int mugd_plan_ops(mugd_plan* p, const mugd_op** ops, int32_t* n_ops) {
    MUGD_REQUIRE(p && ops && n_ops, "plan_ops: bad arguments");
    *ops = p->ops.data();
    *n_ops = (int32_t)p->ops.size();
    return MUGD_OK;
}

int mugd_plan_launch_count(mugd_plan* p) { return p ? p->launches : 0; }

void mugd_plan_destroy(mugd_plan* p) {
    if (!p) return;
    if (p->exec) cudaGraphExecDestroy(p->exec);
    if (p->graph) cudaGraphDestroy(p->graph);
    delete p;
}

}  // extern "C"

/*
 * mugd.h -- C ABI of libmugd.so, the sm_90a (H100) denoising engine for Mug-Diffusion.
 *
 * The reference (Keytoyze/Mug-Diffusion) has no FFI: its hot path is Python calling ATen.  The boundary
 * this library replaces is therefore the set of Python call sites
 *     DDIMSampler.sample / ddim_sampling / p_sample_ddim   mug/diffusion/ddim.py:56-196
 *     MugDiffusionWrapper.forward -> UNetModel.forward       mug/diffusion/diffusion.py:52-54, unet.py:511-550
 *     MugDiffusionWrapper.decode  -> Decoder.forward         mug/diffusion/diffusion.py:49-50, autoencoder.py:329-354
 * and the entry points below are what a ctypes binding on the reference side would call
 * (INTEGRATION.md shows that binding).  Plain pointers and sizes only: every pointer is a DEVICE pointer
 * into memory the caller owns (torch allocations in the Python host), `stream` is a cudaStream_t passed
 * as void*.  No CPU fallback exists: mugd_create fails on anything that is not compute capability 9.0.
 *
 * Execution model: the host "compiles" a network evaluation into a flat launch plan (array of mugd_op,
 * pointers fully resolved), the library validates it, optionally captures it into a CUDA graph, and
 * replays it once per DDIM step with zero host synchronisation.  Step-dependent data (time-embedding
 * rows, DDIM coefficients) is indexed on the device through a step counter, so one graph serves all steps.
 *
 * Activation layout: channels-last  [B * L, C]  fp32 row-major with explicit leading dimension, so a
 * channel concat is a column range of a wider buffer (unet.py:114-118,545 torch.cat -> zero copies).
 */
#ifndef MUGD_H
#define MUGD_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MUGD_ABI_VERSION 13

typedef struct mugd_handle mugd_handle;   /* one device + scratch state            */
typedef struct mugd_plan mugd_plan;       /* validated launch plan (+ CUDA graph)  */

enum mugd_status {
    MUGD_OK = 0,
    MUGD_ERR_INVALID = 1,      /* bad argument / unsupported shape            */
    MUGD_ERR_CUDA = 2,         /* CUDA runtime error (see mugd_last_error)    */
    MUGD_ERR_NO_DEVICE = 3,    /* not an sm_90 device; there is no fallback   */
    MUGD_ERR_OOM = 4
};

enum mugd_op_kind {
    MUGD_OP_GEMM = 1,          /* Linear / 1x1 conv / conv3 / strided conv / upsample+conv, fused epilogue */
    MUGD_OP_GROUPNORM = 2,     /* GroupNorm(eps) [+ SiLU]                                                    */
    MUGD_OP_LAYERNORM = 3,
    MUGD_OP_ATTENTION = 4,     /* rel-pos-biased softmax attention with post-softmax gain                   */
    MUGD_OP_S4CONV = 5,        /* causal long convolution + D*u + GELU                                       */
    MUGD_OP_DDIM_UPDATE = 6,   /* CFG combine + x_{t-1} update                                              */
    MUGD_OP_TRANSPOSE = 7,     /* [B,C,L] <-> [B,L,C] with leading dimensions                                */
    MUGD_OP_COPY2D = 8,        /* strided row copy                                                           */
    MUGD_OP_STEP_ADVANCE = 9,  /* *step += 1                                                                 */
    MUGD_OP_NOTES = 10,        /* decoder logits -> ordered note list (OsuManiaConvertor.array_to_objects)   */
    MUGD_OP_EMBED = 11,        /* prompt ids -> [B, H, F] embedding (BeatmapFeatureEmbedder.forward)         */
    MUGD_OP_TF32_SPLIT = 12,   /* weight preprocessing: w -> (hi in place, lo) for the 3xTF32 tensor-core GEMM */
    MUGD_OP_POSTERIOR = 13     /* first-stage encoder moments -> mean / logvar / std / z (DiagonalGaussianDistribution)  */
};

/* A-operand row addressing of MUGD_OP_GEMM (rows are tokens of B samples, Lout output rows each) */
enum mugd_conv_mode {
    MUGD_CONV_NONE = 0,        /* taps=1: Linear / 1x1 conv (unet.py skip_connection, attention.py proj_in)  */
    MUGD_CONV_SAME = 1,        /* taps=3, pad 1: nn.Conv1d(k=3,padding=1)                                    */
    MUGD_CONV_DOWN = 2,        /* taps=3, right-pad 1, stride 2: models.py:84-91 Downsample                  */
    MUGD_CONV_UP = 3,          /* nearest x2 then taps=3 pad 1: models.py:66-70 Upsample                     */
    MUGD_CONV_TAPS = 4         /* `taps` consecutive rows l+tap_shift .. (zero outside the sample), Lin == Lout: the
                                  two parity halves of Upsample (y[2j] = W0 x[j-1] + (W1+W2) x[j],
                                  y[2j+1] = (W0+W1) x[j] + W2 x[j+1]) run as 2-tap GEMMs on half the rows         */
};
enum mugd_act { MUGD_ACT_NONE = 0, MUGD_ACT_SILU = 1, MUGD_ACT_GELU = 2 };
/* gated epilogues: weight rows are interleaved (value_j, gate_j) by the packer; output has N/2 columns */
enum mugd_gate { MUGD_GATE_NONE = 0, MUGD_GATE_GEGLU = 1 /* a*gelu(g), attention.py:38-45 */,
                 MUGD_GATE_GLU = 2 /* a*sigmoid(g), s4.py:191-192,1536 */ };
enum mugd_gemm_impl { MUGD_GEMM_AUTO = 0, MUGD_GEMM_SIMT = 1 /* exact fp32 FMA */,
                      MUGD_GEMM_TC = 2 /* wgmma 3xTF32 split, fp32 accumulate in registers */ };

typedef struct mugd_gemm {
    const float* A;  int64_t lda;          /* [B*Lin, K] activations                                       */
    const float* W;                        /* [N][taps*K], K-major per tap (conv weight [Cout][k][Cin])    */
    const float* W_hi;                     /* optional: W rounded to TF32 (rna)            } tensor-core path, */
    const float* W_lo;                     /* optional: rna_tf32(W - W_hi)                 } same layout as W  */
    const float* bias;                     /* [N] or NULL                                                  */
    const float* rowvec;                   /* per-sample row vector added before act: time embedding       */
    int64_t rowvec_b_stride;               /*   rowvec[step*step_stride + b*b_stride + n]                  */
    int64_t rowvec_step_stride;
    const int32_t* step;                   /* device step counter or NULL (=0)                             */
    const float* residual; int64_t ldr;    /* added after act/gate, or NULL                                */
    float* C;        int64_t ldc;          /* [B*Lout, N] (N/2 when gated)                                 */
    int32_t M, N, K;                       /* M = B*Lout rows, N weight rows, K channels per tap           */
    int32_t taps, conv_mode, Lin, Lout;
    int32_t act, gate, impl;
    int32_t split_k;                       /* tensor-core path: 0 = auto, >0 forces the K split            */
    int32_t n_counters;                    /* entries available in `counters`                              */
    int32_t tap_shift;                     /* MUGD_CONV_TAPS: source row of tap t is l + (t + tap_shift) * dilation */
    int32_t tap_dilation;                  /* MUGD_CONV_TAPS: 0/1 = dense taps; d = dilated conv (wave.py:425-433)  */
    void* workspace; int64_t workspace_bytes; /* split-K partial tiles (see mugd_gemm_tc_query)            */
    int32_t* counters;                     /* unused since ABI 8 (kept for layout stability)               */
    /* optional SECOND activation source: K2 more channels read at the output row itself (a 1x1 term), weights in columns
     * taps*K .. taps*K+K2 of every W row.  One GEMM then computes  conv3(A) + conv1(A2):  out_layers conv + skip_connection
     * of a TimestepResBlock (unet.py:187-193,237-239), and  proj_out(ff.net.2(ff) + h) = (Wp Wf) ff + Wp h  of the transformer
     * block (attention.py:57-65,194-199) with the packer-composed weight.  NULL / 0 = single source. */
    const float* A2; int64_t lda2;         /* [B*Lout, K2]                                                 */
    int32_t K2; int32_t reserved_;
    /* Row moments of the OUTPUT for a LayerNorm that follows (tensor-core path, act == gate == NONE only): while the tile is stored,
     * row_moments[m*2 + {0,1}] += {sum, sum of squares} of the columns of output row m (fp64 atomics; the plan zeroes the buffer at
     * the start of every evaluation).  GroupNorm-moment sinks + a single-pass apply kernel were also built;
     * they lost at every batch size and were removed. */
    double* row_moments;
    /* LayerNorm folded into this GEMM (attention.py:147-151: norm_i followed by a Linear): with W' = W diag(gamma) packed as the
     * weight, colsum[n] = sum_k W'[n][k] and bias' = W beta + b,   C = rstd_m * (A W'^T - mean_m * colsum) + bias'   where mean_m,
     * rstd_m come from the row moments ln_stats[m*2 + {0,1}] = {sum, sum of squares} over the K channels of A's row m (the row_moments
     * of A's producer).  The normalised tensor is never materialised.  NULL = plain GEMM. */
    const double* ln_stats; const float* ln_colsum; float ln_eps; int32_t reserved2_;
} mugd_gemm;

typedef struct mugd_groupnorm {
    const float* x; int64_t ldx; float* y; int64_t ldy;
    const float* gamma; const float* beta;
    int32_t B, L, C, G; float eps; int32_t silu;
} mugd_groupnorm;

typedef struct mugd_layernorm {
    const float* x; int64_t ldx; float* y; int64_t ldy;
    const float* gamma; const float* beta;
    int32_t rows, C; float eps;
} mugd_layernorm;

typedef struct mugd_attention {
    const float* q; int64_t ldq;           /* [B*Lq, H*D] head h at columns h*D..                          */
    const float* k; int64_t ldk;           /* [B*Lk, H*D]                                                  */
    const float* v; int64_t ldv;
    float* o; int64_t ldo;
    const float* relpos;                   /* [2*pos_max+1][H] additive, inside the scale (attention.py:113) */
    const float* cgain;                    /* [2*pos_max+1][H] post-softmax multiplier (attention.py:122)   */
    int32_t B, H, D, Lq, Lk, pos_max; float scale;
} mugd_attention;

typedef struct mugd_s4conv {
    const float* u; int64_t ldu;           /* [B*L, H]                                                     */
    const float* Kt;                       /* [L][H] kernel taps, tap-major (from mugd_s4_kernel_gen)      */
    const float* D;                        /* [H]                                                          */
    float* y; int64_t ldy;                 /* gelu(conv + D*u); must not overlap u                         */
    int32_t B, L, H;
} mugd_s4conv;

typedef struct mugd_ddim_update {
    float* x;                              /* [B*L, C] in place -> x_{t-1}                                  */
    float* x_dup;                          /* optional second copy of x_{t-1} (the cfg half of the 2B batch) */
    const float* eps;                      /* [Beff*L, C]; Beff = 2B when cfg (uncond first, ddim.py:173)   */
    const float* noise;                    /* [B*L, C] or NULL (sigma = 0)                                  */
    float* pred_x0;                        /* [B*L, C] or NULL                                              */
    const float* coef;                     /* [S][4] = a_t, a_prev, sigma_t, sqrt(1-a_t) per DDIM index     */
    const int32_t* step;                   /* device step counter i; row used = S-1-i (ddim.py:138)         */
    int32_t S; int32_t n;                  /* n = B*L*C elements                                            */
    int32_t cfg; float scale; float temperature;
} mugd_ddim_update;

typedef struct mugd_transpose {            /* to_nlc=1: in [B,C,L] (contiguous) -> out [B*L, ldo] cols 0..C  */
    const float* in; float* out;           /* to_nlc=0: in [B*L, ldi] -> out [B,C,L]                          */
    int64_t ldi, ldo; int32_t B, C, L, to_nlc;
} mugd_transpose;

typedef struct mugd_copy2d {
    const float* src; int64_t lds; float* dst; int64_t ldd; int32_t rows, cols;
} mugd_copy2d;

typedef struct mugd_step_advance { int32_t* step; } mugd_step_advance;

/* Note extraction, mug/data/convertor.py:232-264 (from_logits): for key column c of chart b a note starts at every frame
 * t with logit[t][c] > 0; start = round((t + clip(logit[t][K+c],0,1)) * frame_ms); it is a long note when the following
 * frames have logit[.][2K+c] > 0 and no new start, end = round((t_end + clip(logit[t_end][3K+c],0,1)) * frame_ms), else -1.
 * Output is compact and ordered by frame per (chart, column): count[b*K+c], start_ms/end_ms[(b*K+c)*T + i]. */
typedef struct mugd_notes {
    const float* logits; int64_t ld;       /* [B*T, 4K] channels-last decoder output                        */
    int32_t* count; int32_t* start_ms; int32_t* end_ms;
    double frame_ms;
    int32_t B, T, K;
} mugd_notes;

/* Prompt embedding, mug/cond/feature.py:15-21 (BeatmapFeatureEmbedder.forward): out[b][h][f] = table[ids[b][f]][h], the
 * nn.Embedding lookup followed by rearrange "b f h -> b h f".  ids must lie in [0, n_embed) (the host checks, like torch). */
typedef struct mugd_embed {
    const float* table;                    /* [n_embed, H] row-major                                         */
    const int32_t* ids;                    /* [B, F]                                                         */
    float* out;                            /* [B, H, F]                                                      */
    int32_t B, F, H, n_embed;
} mugd_embed;

/* hi = rna_tf32(w) written over w, lo = rna_tf32(w - hi): the two TF32 operands whose products reconstruct an fp32 weight.
 * Run once per engine after the (plain fp32) weight blob has reached the device -- the blob that is packed, stored and broadcast holds
 * every weight once; the resident copy holds hi + lo of the tensor-core weights and no plain duplicate. */
typedef struct mugd_tf32_split { float* w_hi; float* lo; int64_t n; } mugd_tf32_split;

/* Posterior of the first-stage encoder, mug/firststage/autoencoder.py:356-387 (DiagonalGaussianDistribution): mean, logvar =
 * chunk(params, 2, dim=1); logvar = clamp(logvar, -10, 20); std = exp(0.5 * logvar); z = mean * scale (mode()) or, with noise,
 * (mean + std * noise) * scale (sample()).  Same operation order as the reference's separate ATen ops, no FMA contraction: mean,
 * logvar and mode() are bit-identical to torch; std and z differ from it by the ulp difference of two exp implementations.
 * All tensors are NCL; every output may be NULL. */
typedef struct mugd_posterior {
    const float* params;                   /* [B, 2Z, L] encoder output (moments)                            */
    const float* noise;                    /* [B, Z, L] standard normal draw, or NULL = mode()                */
    float *mean, *logvar, *std, *z;        /* [B, Z, L] each                                                  */
    float scale;                           /* AutoencoderKL.scale                                             */
    int32_t B, Z, L;
} mugd_posterior;

typedef struct mugd_op {
    int32_t kind;
    int32_t tag;                           /* free for the host (profiling labels)                          */
    union {
        mugd_gemm gemm; mugd_groupnorm gn; mugd_layernorm ln; mugd_attention attn; mugd_s4conv s4;
        mugd_ddim_update ddim; mugd_transpose tr; mugd_copy2d cp; mugd_step_advance adv; mugd_notes notes;
        mugd_embed embed; mugd_tf32_split split; mugd_posterior post;
    } u;
} mugd_op;

/* ---- lifecycle -------------------------------------------------------------------------------- */
int  mugd_abi_version(void);
const char* mugd_last_error(void);                         /* thread-local message of the last failure */
int  mugd_create(int device, mugd_handle** out);           /* MUGD_ERR_NO_DEVICE unless sm_90           */
void mugd_destroy(mugd_handle* h);
int  mugd_device_info(mugd_handle* h, int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor);
int  mugd_set_gemm_impl(mugd_handle* h, int impl);         /* default for ops with impl == AUTO         */
int  mugd_set_pdl(int enabled);                            /* programmatic launch edges (default on; process-wide A/B switch) */

/* ---- single op (parity tests call every kernel through this) ---------------------------------- */
int  mugd_op_run(mugd_handle* h, const mugd_op* op, void* stream);

/* ---- plans ------------------------------------------------------------------------------------ */
int  mugd_plan_create(mugd_handle* h, const mugd_op* ops, int32_t n_ops, mugd_plan** out);
int  mugd_plan_run(mugd_plan* p, void* stream);            /* eager launches                            */
int  mugd_plan_capture(mugd_plan* p, void* stream);        /* build + instantiate a CUDA graph          */
int  mugd_plan_replay(mugd_plan* p, int32_t times, void* stream); /* launch the graph `times` times     */
int  mugd_plan_launch_count(mugd_plan* p);                 /* kernels launched by one run of the plan   */
void mugd_plan_destroy(mugd_plan* p);

/* ---- the sampler loop from ONE call: DDIMSampler.ddim_sampling's for-loop (ddim.py:136-157) -------------------------------
 * n_steps x { replay the captured evaluation plan (one CUDA graph = Beff U-Net evaluations) ; run the `tail` ops eagerly on the same
 * stream: MUGD_OP_DDIM_UPDATE (CFG combine + x_{t-1}) and MUGD_OP_STEP_ADVANCE (device step counter) }.  Nothing synchronises; the
 * step-dependent rows (time embedding, DDIM coefficients) are selected on the device by the counter.  `eval_plan` must be captured. */
int  mugd_sample(mugd_plan* eval_plan, const mugd_op* tail, int32_t n_tail, int32_t n_steps, void* stream);

/* ---- the same loop for inpainting and eta > 0 requests: what the host stages in front of each step ---------------------------
 * Step i of a mugd_sample_staged call first runs one stage kernel over the dense x rows [B*L, C] that MUGD_OP_DDIM_UPDATE updates:
 *   inpainting blend (ddim.py:141-144, diffusion.py:327-333), when x0 is given:
 *       xo = a_i * x0 + b_i * q_noise[i];   x <- xo * mask + (1 - mask) * x   (written to x and, if given, x_dup)
 *     in torch's eager operation order with IEEE round-to-nearest and no contraction, so the result is bit-identical to those ops;
 *   step noise, when noise is given: noise_rows <- noise[i] transposed to rows (the DDIM op's `noise`).
 * x0, mask, q_noise and noise are device NCL tensors as torch holds them ([B, C, L]; the tables [n_steps][B, C, L], row i for step i of
 * this call); the mask is expanded to [B, C, L].  q_coef is a HOST array [n_steps][2] = (sqrt_alphas_cumprod[t_i],
 * sqrt_one_minus_alphas_cumprod[t_i]) read by the call.  Either part may be absent (NULL); x0, mask, q_noise and q_coef go together,
 * as do noise and noise_rows. */
typedef struct mugd_stage {
    float* x; float* x_dup;                /* [B*L, C] dense rows; x_dup = the CFG copy or NULL                  */
    const float* x0;                       /* [B, C, L] or NULL (no blend)                                     */
    const float* mask;                     /* [B, C, L]                                                        */
    const float* q_noise;                  /* [n_steps][B, C, L] q_sample's randn_like(x0) per step            */
    const float* q_coef;                   /* HOST [n_steps][2]                                                */
    const float* noise;                    /* [n_steps][B, C, L] randn(shape) [+ dropout] per step, or NULL    */
    float* noise_rows;                     /* [B*L, C] the DDIM op's noise rows                                */
    int32_t B, C, L, reserved_;
} mugd_stage;
/* n_steps x { stage kernel for step i ; replay of the captured evaluation plan ; the tail ops }.  Every argument is checked before the
 * first launch: each MUGD_OP_DDIM_UPDATE of the tail must update the same rows (x, x_dup, n = B*C*L) and, with noise, read noise_rows.
 * A standalone entry point: the ABI version is unchanged. */
int  mugd_sample_staged(mugd_plan* eval_plan, const mugd_stage* stage, const mugd_op* tail, int32_t n_tail, int32_t n_steps,
                        void* stream);

/* ---- the PLMS sampler loop: PLMSSampler.plms_sampling / p_sample_plms, mug/diffusion/plms.py:115-236 (eta = 0 only) -----------
 * n = B*L*C elements of the dense x rows.  Step i of an S-step request:
 *   replay the evaluation plan; combine: e_t = eps rows (CFG: e_u + scale * (e_c - e_u), uncond half first, :182-186), written to
 *   slot i mod 3 of `hist` (old_eps keeps the last 3, :160-162), and e' into e_prime by the Adams-Bashforth order min(i, 3):
 *   (3 e_t - o1) / 2, (23 e_t - 16 o1 + 5 o2) / 12, (55 e_t - 59 o1 + 37 o2 - 9 o3) / 24 (:224-232, o_k = e_t of step i - k);
 *   then `update` (x_{t-1} from e', :199-216) and *update.step += 1.
 * Step 0 (pseudo improved Euler, :219-223) evaluates twice:
 *   1. replay at t (timestep row 0); combine with e' = e_t; 2. x_stash <- x; 3. `update` (coefficient row 0) writes the Euler x_prev into
 *   x and x_dup; 4. *step <- 1 (0 when S = 1: t_next = time_range[min(1, S - 1)], :145) and replay, so the time-embedding rows follow;
 *   5. x <- x_stash; 6. Heun combine: e' = (e_t + e_t_next) / 2, e_t read from slot 0; 7. *step <- 0, `update`, *step += 1.
 * Every intermediate is one IEEE round-to-nearest in torch's CUDA eager order (a division by a Python scalar is torch's multiply by
 * the float reciprocal), no contraction: bit-identical to the torch expressions.
 * The ring and the step counter live on the device, so a request can run as several calls (first_step = steps already run, the
 * counter holding first_step) with intermediates recorded between them. */
typedef struct mugd_plms {
    mugd_ddim_update update;               /* the x update on e': cfg = 0, eps = e_prime, noise = NULL; x, x_dup, pred_x0, coef, step
                                              and S as for mugd_sample (coef rows at eta = 0)                                    */
    const float* eps;                      /* [Beff*L, C] the evaluation plan's output rows; Beff = 2B when cfg                   */
    float* e_prime;                        /* [n] e' of the current step                                                         */
    float* hist;                           /* [3][n] e_t of the last three steps (slot j mod 3 for step j)                      */
    float* x_stash;                        /* [n] x across step 0's second evaluation                                           */
    int32_t cfg; float scale;              /* classifier-free guidance: cfg = 1 and its scale                                  */
} mugd_plms;
/* steps first_step .. first_step + n_steps - 1 of the update's S-step request, no host synchronisation.  Every argument is checked before
 * the first launch.  Launches per step: the plan's graph, the combine kernel, the update and the advance (step 0: one more graph replay,
 * combine and update, two counter fills and two copies).  A standalone entry point: the ABI version is unchanged. */
int  mugd_sample_plms(mugd_plan* eval_plan, const mugd_plms* p, int32_t first_step, int32_t n_steps, void* stream);
/* the combine kernel alone for step `step` (heun = 1: step 0's second combine), for a host that runs the PLMS steps one by one */
int  mugd_plms_combine(const mugd_plms* p, int32_t step, int32_t heun, void* stream);

/* ---- the DDPM ancestral sampler loop: DDPM.log_beatmap, mug/diffusion/diffusion.py:255-282 (parameterization "eps") ------------
 * Step i of a T-step request (timestep t = T - 1 - i, the device counter holding i): replay the evaluation plan, then one update kernel
 *   e       = eps rows; with cfg: e_u + scale * (e_c - e_u), uncond half first (an extension: the reference loop has no guidance;
 *             the combine is ddim.py:175's)
 *   x_recon = coef[t][0] * x - coef[t][1] * e;  with clip: x_recon = clamp(x_recon, -10, 10), NaN kept        (:260-267, :211-215)
 *   x       = coef[t][2] * x_recon + coef[t][3] * x + coef[t][4] * noise                                        (:268-277)
 * written to x (and x_dup), x_recon to pred_x0 (if given); then *step += 1.  Every intermediate is one IEEE round-to-nearest in
 * torch's eager order, no contraction: with equal eps and noise the result is bit-identical to the reference's torch expressions.
 * coef is a device table [T][5] = (sqrt_recip_alphas_cumprod, sqrt_recipm1_alphas_cumprod, posterior_mean_coef1,
 * posterior_mean_coef2, sigma) of the model's float32 schedule buffers, where sigma[t] = (1 - (t == 0)) * exp(0.5 *
 * posterior_log_variance_clipped[t]) evaluated in float32 by torch's CUDA ops (the Python host builds the column with them, so exp is
 * torch's; another host must reproduce torch's CUDA expf to stay bit-identical).  noise is a device table [n_steps][B, C, L] (NCL, as
 * torch draws it): row k is the noise of step first_step + k of a mugd_sample_ddpm call; mugd_ddpm_update reads row 0.  The step
 * counter lives on the device, so a request can run as several calls with intermediates recorded between them. */
#define MUGD_MAX_STEPS 1000                /* rows of the time-embedding table a sampling session holds: T <= MUGD_MAX_STEPS  */
typedef struct mugd_ddpm {
    float* x; float* x_dup;                /* [B*L, C] dense rows in place; x_dup = the CFG copy (given exactly when cfg = 1)     */
    const float* eps;                      /* [Beff*L, C] the evaluation plan's output rows; Beff = 2B when cfg                  */
    float* pred_x0;                        /* [B*L, C] x_recon of the step, or NULL                                             */
    const float* noise;                    /* [n_steps][B, C, L]                                                                */
    const float* coef;                     /* [T][5]                                                                            */
    int32_t* step;                         /* device step counter i                                                             */
    int32_t T, B, C, L;
    int32_t cfg; float scale;              /* classifier-free guidance: cfg = 1 and its scale                                  */
    int32_t clip;                          /* 1 = clip_denoised                                                                 */
    int32_t reserved_;
} mugd_ddpm;
/* steps first_step .. first_step + n_steps - 1 of the T-step request, no host synchronisation: n_steps x { graph replay, update with
 * noise row k, *step += 1 }, the same launches per step as mugd_sample.  Every argument is checked before the first launch
 * (first_step + n_steps <= T <= MUGD_MAX_STEPS).  A standalone entry point: the ABI version is unchanged. */
int  mugd_sample_ddpm(mugd_plan* eval_plan, const mugd_ddpm* d, int32_t first_step, int32_t n_steps, void* stream);
/* the update kernel alone (noise row 0, the counter not advanced), for a host that runs the DDPM steps one by one */
int  mugd_ddpm_update(const mugd_ddpm* d, void* stream);

/* ---- the DPM-Solver++ multistep sampler loop (data prediction; Stable Diffusion 2's DPM_Solver(predict_x0=True), "multistep") ----
 * n = B*L*C elements of the dense x rows.  Step i of an S-step request (the device counter holding i): replay the evaluation plan
 * (timestep row i = the model time of t_i), then one update kernel with coefficient row i = coef[8i .. 8i+7] = (alpha_i, sigma_i,
 * A, c0, c1, c2, order, unused):
 *   e  = eps rows; with cfg: e_u + scale * (e_c - e_u), uncond half first (the DDIM combine)
 *   m0 = (x - sigma_i * e) / alpha_i                                                    the data prediction at t_i
 *   x  = ((A * x + c0 * m0) + c1 * m1) + c2 * m2   (the c1 term only for order >= 2, c2 only for order 3)
 * where m1 / m2 are the predictions of steps i-1 / i-2, read from ring slots (i-1) mod 3 / (i-2) mod 3; m0 goes to slot i mod 3 and
 * to pred_x0 (if given), x to x and x_dup; then *step += 1.  Every intermediate is one IEEE round-to-nearest in this order, no
 * contraction.  The rows come from the host (mug_diffusion_b200/dpm_solver.py), which expands the solver's D-form updates in float64.
 * The ring and the counter live on the device, so a request can run as several calls (first_step = steps already run, the counter
 * holding first_step), including a split inside the warm-up. */
typedef struct mugd_dpm {
    float* x; float* x_dup;                /* [B*L, C] dense rows in place; x_dup = the CFG copy (given exactly when cfg = 1)     */
    const float* eps;                      /* [Beff*L, C] the evaluation plan's output rows; Beff = 2B when cfg                  */
    float* pred_x0;                        /* [n] the data prediction m0 of the step, or NULL                                  */
    float* ring;                           /* [3][n] m0 of the last three steps (slot j mod 3 for step j)                      */
    const float* coef;                     /* [S][8] coefficient rows                                                           */
    int32_t* step;                         /* device step counter i                                                             */
    int32_t n, S;                          /* elements of x; steps of the request (S <= MUGD_MAX_STEPS)                         */
    int32_t cfg; float scale;              /* classifier-free guidance: cfg = 1 and its scale                                  */
} mugd_dpm;
/* steps first_step .. first_step + n_steps - 1 of the S-step request, no host synchronisation: n_steps x { graph replay, update,
 * *step += 1 }, the same launches per step as mugd_sample.  Every argument is checked before the first launch
 * (first_step + n_steps <= S <= MUGD_MAX_STEPS).  A standalone entry point: the ABI version is unchanged. */
int  mugd_sample_dpm(mugd_plan* eval_plan, const mugd_dpm* d, int32_t first_step, int32_t n_steps, void* stream);
/* the update kernel alone (the counter not advanced), for a host that runs the DPM-Solver++ steps one by one */
int  mugd_dpm_update(const mugd_dpm* d, void* stream);

/* ---- DPM-Solver++ from an existing chart: inpainting and per-chart-strength remix ---------------------------------------------
 * mugd_dpm_ex extends a mugd_dpm request by one of:
 *   stage  inpainting: step k of a mugd_sample_dpm_ex call first runs the mugd_sample_staged stage kernel for row k of the stage's
 *          tables (x <- (alpha_i * x0 + sigma_i * q_noise[k]) * mask + (1 - mask) * x with q_coef[k] = (alpha_i, sigma_i) of the step);
 *          the stage must blend the update's x / x_dup over n = B*C*L elements and stage no step noise.
 *   start  remix: chart b (elements b * n/B .. (b+1) * n/B - 1 of the dense rows) runs from step start[b] on; before that it is left
 *          untouched (x, x_dup, ring and pred_x0), so its rows keep the latent they were loaded with.  From step start[b] on chart b
 *          takes order k = min(coef row i's order, i - start[b] + 1) and applies row (i, k - 1) = order_coef[8 (3i + k - 1) ..] of the
 *          per-order table [S][3][8] (same layout as coef; row (i, order_i - 1) equals coef row i), reading only the ring slots of its
 *          own steps.  Everything else is the mugd_dpm update, bit for bit.
 * Neither (both NULL) is mugd_sample_dpm.  stage and start are exclusive; start and order_coef go together. */
typedef struct mugd_dpm_ex {
    mugd_dpm dpm;                          /* the update (coef [S][8], ring, step counter, ...)                                 */
    const mugd_stage* stage;               /* inpainting blend in front of each step, or NULL                                  */
    const int32_t* start;                  /* [B] device: the first step of each chart, or NULL                                */
    const float* order_coef;               /* [S][3][8] device per-order rows, given exactly with start                         */
    int32_t B, reserved_;                  /* charts (with start)                                                              */
} mugd_dpm_ex;
/* steps first_step .. first_step + n_steps - 1 of the S-step request (the counter holding first_step), no host synchronisation:
 * n_steps x { stage kernel (with stage) ; graph replay ; update ; *step += 1 }: with a stage the launches per step of
 * mugd_sample_staged, otherwise those of mugd_sample_dpm.  Every argument is checked before the first launch (first_step + n_steps <=
 * S, the stage's q_coef rows finite).  A standalone entry point: the ABI version is unchanged. */
int  mugd_sample_dpm_ex(mugd_plan* eval_plan, const mugd_dpm_ex* e, int32_t first_step, int32_t n_steps, void* stream);
/* the update alone for the counter's step (per chart with start; the stage is not run), for a host that runs the steps one by one */
int  mugd_dpm_ex_update(const mugd_dpm_ex* e, void* stream);

/* ---- remixing an existing chart (SDEdit / img2img): DDIMSampler.stochastic_encode and decode with a per-chart start ---------------
 * mugd_stochastic_encode: out[b] = sqrt_a[t[b]] * x0[b] + sqrt_1ma[t[b]] * noise[b], each product and the sum one IEEE
 * round-to-nearest (no contraction), bit-identical to torch's extract_into_tensor expressions.  x0, noise and out are device NCL
 * [B, C, L]; t is a device [B] int64 array of table rows; sqrt_a / sqrt_1ma are device tables of n rows (sqrt(ddim_alphas) and
 * ddim_sqrt_one_minus_alphas, or the model's sqrt_alphas_cumprod / sqrt_one_minus_alphas_cumprod).  The host checks the indices
 * before the call; an index outside [0, n) writes NaN for that sample and never reads past the tables.  One launch. */
typedef struct mugd_q_encode {
    const float* x0; const float* noise;   /* [B, C, L]                                                        */
    const int64_t* t;                      /* [B] table rows                                                   */
    const float* sqrt_a; const float* sqrt_1ma;  /* [n]                                                        */
    float* out;                            /* [B, C, L]                                                        */
    int32_t B, C, L, n;
} mugd_q_encode;
int  mugd_stochastic_encode(const mugd_q_encode* d, void* stream);

/* mugd_sample_join: the mugd_sample loop with one join kernel in front of each step, for charts that enter the loop at different
 * iterations.  Chart b joins at iteration join[b]: while the device step counter (the tail's MUGD_OP_DDIM_UPDATE `step`) is <= join[b],
 * the join kernel sets chart b's dense x rows [L, C] (and its CFG copy in x_dup) to x_latent[b] (NCL).  From its join on, chart b
 * follows the coefficient rows of a run that started from x_latent[b] with S - join[b] steps.  A chart with join[b] >= S never runs;
 * its rows hold whatever the last update wrote, and the host returns x_latent[b] for it. */
typedef struct mugd_join {
    float* x; float* x_dup;                /* [B*L, C] dense rows; x_dup = the CFG copy or NULL                  */
    const float* x_latent;                 /* [B, C, L]                                                        */
    const int32_t* join;                   /* [B] device: the iteration at which chart b joins                 */
    int32_t B, C, L, reserved_;
} mugd_join;
/* steps first_step .. first_step + n_steps - 1 (the counter holding first_step): n_steps x { join kernel ; replay of the captured
 * evaluation plan ; the tail ops }, no host synchronisation: one launch per step more than mugd_sample.  Every argument is checked
 * before the first launch: the tail holds exactly one MUGD_OP_DDIM_UPDATE, on the join's x / x_dup with n = B*C*L, and
 * first_step + n_steps <= its S.  A standalone entry point: the ABI version is unchanged. */
int  mugd_sample_join(mugd_plan* eval_plan, const mugd_join* join, const mugd_op* tail, int32_t n_tail, int32_t first_step,
                      int32_t n_steps, void* stream);

/* ---- plans on disk: a host without Python (examples/host_c) loads what the Python plan compiler produced ---------------------
 * Every pointer of a plan lies in one of a few device allocations ("regions": weight blob, activation arena, side tables, the
 * caller's staging buffers).  mugd_plan_save stores each pointer as (region, offset); mugd_plan_load resolves them against the
 * loader's allocations, matched by name (each at least as large as recorded).  Region contents are the caller's business. */
typedef struct mugd_region { const char* name; void* base; int64_t bytes; } mugd_region;
int  mugd_plan_save(mugd_plan* p, const mugd_region* regions, int32_t n_regions, const char* path);
int  mugd_plan_load(mugd_handle* h, const char* path, const mugd_region* regions, int32_t n_regions, mugd_plan** out);
/* the (relocated) ops of a plan, e.g. to hand a loaded update/advance plan to mugd_sample as its tail; owned by the plan */
int  mugd_plan_ops(mugd_plan* p, const mugd_op** ops, int32_t* n_ops);
/* names and sizes of the regions a plan file refers to (names[i] receives the text, out[i].name points at it); n_regions always set */
int  mugd_plan_regions(const char* path, mugd_region* out, char (*names)[48], int32_t max_regions, int32_t* n_regions);

/* ---- S4 kernel generation: SSKernelNPLR.forward, s4.py:706-832 (once per model and length) ----- */
int  mugd_s4_kernel_gen(mugd_handle* h,
                        const float* log_dt,      /* [H]        */
                        const float* Bri,         /* [H][N][2]  */
                        const float* Cri,         /* [H][N][2]  */
                        const float* Pri,         /* [H][N][2]  */
                        const float* inv_w_real,  /* [H][N]     */
                        const float* w_imag,      /* [H][N]     */
                        const float* omega_ri,    /* [L_internal/2+1][2] FFT nodes as the reference computes them
                                                     (complex64 omega**arange, s4.py:595-598) or NULL = exact */
                        int32_t H, int32_t N, int32_t L_internal, int32_t L_out,
                        float* Kt,                /* [L_out][H] */
                        void* workspace, int64_t workspace_bytes, /* >= 16*H*(L_internal/2+1) bytes */
                        void* stream);

/* ---- log-mel spectrogram of decoded audio: load_audio_without_cache, mug/util.py:138-143 (once per request) ----------------
 * out[b*T_out + t][m] = fp16-rounded log1p(sum_k mel[m][k] |STFT(y_b)[k][t]|^2) for t < T = 1 + n/hop, 0 for T <= t < T_out (webui's
 * pad to 64 * z_length frames, webui.py:360-365), with librosa >= 0.10's STFT: center=True, zero padding, n_fft = 512 only.
 * window [n_fft] and twiddle [n_fft/2][2] = exp(-2 pi i k / n_fft) are fp64 device tables; band m of the filterbank is
 * weights[sum of band_len[<m]] .. over rfft bins band_start[m] .. band_start[m] + band_len[m] - 1.  band_start and band_len are
 * HOST arrays of n_mels entries (read by the call and checked before the launch); y, weights and out are device memory. */
int  mugd_melspec(mugd_handle* h,
                  const float* y, int64_t n, int64_t ldy, int32_t B,  /* [B][ldy] mono samples at the model's rate    */
                  const double* window, const double* twiddle, int32_t n_fft,
                  const int32_t* band_start, const int32_t* band_len, const float* weights, int32_t n_mels,
                  int32_t hop,
                  float* out, int64_t ldo, int32_t T_out,              /* [B*T_out][ldo] channels-last, T_out >= 1+n/hop */
                  void* stream);

/* ---- chart timing: one scan of the BPM / offset search of gridify, mug/data/utils.py:46-101 (postprocess.search_timing) ---------
 * For each chart c, the first trial in the reference loop's order whose score n_on / bpm beats best_score[c].  The trials are rows
 * of 6: row 0 holds head_len[c] <= 5 phases (head_bpm[c], head_off[c*5 + j]) in slots 1 + j; row r >= 1 is candidate
 * k = k0[c] + r - 1, slot 0 = (cands[k], first[c]) and slot 1 + j = (cands[k], np.arange(best_off, best_off - beat, -beat/4)[j]),
 * beat = 60000 / cands[k].  A trial counts the notes t with |pos - rint(pos)| < 10 / step, step = 60000 / bpm, pos = (t - off) / step
 * (t - off in float32 for slot 0, in fp64 otherwise), all IEEE round-to-nearest, so results are bit-equal to the numpy loop.
 * times: device float32 note times of all charts, chart c at chart_start[c] .. chart_start[c+1] - 1; cands: device fp64 candidate
 * table [n_cands].  chart_start [n_charts + 1], k0, head_len, best_off, best_score, first, head_bpm [n_charts] and head_off
 * [n_charts * 5] are HOST arrays (read by the call and checked before the launch; every chart needs >= 1 note, 0 <= k0 <= n_cands).
 * workspace: device scratch of 8 * n_charts bytes.  Outputs (device): out_i[c*3 + {0,1,2}] = position row * 6 + slot (-1: no trial
 * improves), kind (0 head, 1 candidate, 2 phase; -1), n_on; out_d[c*3 + {0,1,2}] = bpm, offset, score of that trial. */
int  mugd_grid_scan(mugd_handle* h, const float* times, const int32_t* chart_start, int32_t n_charts,
                    const double* cands, int32_t n_cands,
                    const int32_t* k0, const int32_t* head_len, const double* best_off, const double* best_score,
                    const float* first, const double* head_bpm, const double* head_off,
                    void* workspace, int32_t* out_i, double* out_d, void* stream);

/* ---- chart clean-up: gridify's snapping, mug/data/utils.py:120-139 (postprocess.snap_lines) ------------------------------------
 * out[i] = the snapped time of note time times[i] of chart c (chart_start[c] <= i < chart_start[c+1]): for div in
 * (1, 2, 4, 3, 6, 8, 16, 32), step = 60000 / (bpm[c] * div), pos = (t - offset[c]) / step, k = rint(pos); the first div with
 * |pos - k| < 10 / step gives (int64)(k * step + offset[c]) (truncated toward zero); no div keeps t.  All IEEE round-to-nearest
 * with no contraction, so results equal the numpy-scalar loop.  offset_is_f32[c] = 1 when gridify's offset is an np.float32: then
 * t - offset is a float32 subtraction of t rounded to float32, as NumPy 2 evaluates int - np.float32.  times (int32) and out
 * (int64) are device memory; chart_start [n_charts + 1], bpm, offset and offset_is_f32 [n_charts] are HOST arrays (read by the
 * call and checked before the launch: chart_start[0] = 0 and non-decreasing, 0 < bpm <= 1e9, |offset| < 2^52, a float32-flagged
 * offset is a float32 value).  Empty charts are allowed. */
int  mugd_chart_snap(mugd_handle* h, const int32_t* times, const int32_t* chart_start, int32_t n_charts,
                     const double* bpm, const double* offset, const int32_t* offset_is_f32, int64_t* out, void* stream);

/* ---- chart clean-up: remove_intractable_mania_mini_jacks(lines, verbose=False, jack_interval), mug/data/utils.py:142-268 ------
 * Runs the reference's greedy loop over every chart's notes in list order (one warp per chart).  Per note i (device memory):
 * start[i] = float(f[2]); end[i] = float(f[5].split(":")[0]) when is_long[i] (int(f[3]) == 128; end is not read otherwise);
 * x[i] = int(float(f[0])), with |x| < 2^30 (columns are x / 128 truncated toward zero, so negative and out-of-range columns
 * behave as in the reference).  On return x[i] is the note's final x and state[i] is 0 (dropped), 1 (kept) or 2 (kept and moved:
 * f[0] becomes str(x[i])).  workspace: device scratch of 8 * chart_start[n_charts] bytes.  chart_start [n_charts + 1] is a HOST
 * array (chart_start[0] = 0, non-decreasing; empty charts are allowed); jack_interval must not be NaN. */
int  mugd_remove_mini_jacks(mugd_handle* h, const int32_t* chart_start, int32_t n_charts, double jack_interval,
                            const double* start, const double* end, const uint8_t* is_long, int32_t* x, uint8_t* state,
                            void* workspace, void* stream);

/* ---- tensor-core GEMM planning: is this GEMM taken by the wgmma kernel, with which K split, and how much
 * split-K workspace / how many tile counters does it need (the host allocates them once per plan) ------ */
int  mugd_gemm_tc_query(mugd_handle* h, const mugd_gemm* g, int32_t sm_count, int32_t* supported, int32_t* splits,
                        int64_t* workspace_bytes, int32_t* n_tiles);
/* which kernel variant the planner picks for this GEMM on a machine with sm_count SMs: tile width (64 / 128; 0 = not taken by the
 * tensor-core kernel), CTAs per SM it is built for (always 1), CTAs launched */
int  mugd_gemm_tc_variant(const mugd_gemm* g, int32_t sm_count, int32_t* tile_n, int32_t* ctas_per_sm, int32_t* grid_ctas);

/* ---- per-handle switches -------------------------------------------------------------------------
 * OPT-IN speed mode of the tensor-core GEMM: 1 = plain TF32 products (a_hi*w_hi only, ~2^-11 relative error per product, like
 * cuDNN's allow_tf32 that the reference's own GPU path uses for convs); 0 (default) = 3xTF32, fp32-accurate.  Parity tests and
 * bench.py use 0.  The mode is read when a GEMM is launched: mugd_op_run and mugd_plan_run use the mode current at the call, whenever
 * the plan was created; a captured graph keeps the mode that was current at mugd_plan_capture. */
int  mugd_set_tc_single_pass_tf32(mugd_handle* h, int enabled);

/* attention kernel: 1 (default) = QK^T and PV on the wgmma tensor cores (3xTF32, fp32 accuracy); 0 = exact-fp32 FFMA kernel
 * (the referee of the parity tests).  Replaces the einsum/softmax body of CrossAttention.forward, attention.py:99-121 */
int  mugd_set_attention_impl(mugd_handle* h, int impl);

/* causal S4 convolution kernel: 0 (default) = automatic: the resident kernel, which holds all of u and K of its 16 channels in
 * shared memory, wherever that fits (L <= 1584 on an H100), the streamed kernel beyond; 1 = resident (refuses a longer L);
 * 2 = streamed at any length.  The two agree bit for bit; the switch lets tests and benchmarks run both at one length.  Read when
 * the op is launched, like the attention switch. */
int  mugd_set_s4conv_impl(mugd_handle* h, int impl);

/* ---- measurement aids (process-wide, not needed in production) -------------------------------------
 * planner cost constants of the tensor-core GEMM (relative cost of a 32-deep k-step of a 128-column tile, unused, of a
 * split-K round trip, unused); values <= 0 keep the current one.  For tuning sweeps (tools/). */
int  mugd_debug_set_tc_cost(float kstep128_us, float kstep256_us, float split_us, float two_cta_fixed_us);

/* force the tensor-core tile width (64 or 128 columns) where legal; 0 = cost model */
int  mugd_debug_set_tc_tile_n(int bn);

/* CTA (0,0,0) of the tensor-core attention kernel dumps the first 16 raw logits of every query row of its
 * first key tile into buf[128*40] (floats 0..15 of each 40-float row); NULL switches it off */
int  mugd_debug_set_attention_dump(float* buf);

/* builds with -DMUGD_TC_TIMELINE only (tools/build_variant.py): CTA (0,0,0) of every tensor-core GEMM launch writes
 * %globaltimer stamps into the device buffer (tools/gemm_timeline.py); otherwise returns MUGD_ERR_INVALID */
int  mugd_debug_set_tc_timing(long long* device_buf);

/* ---- utility ---------------------------------------------------------------------------------- */
int  mugd_fill_i32(int32_t* dst, int32_t value, void* stream);
/* sizeof() of {mugd_op, mugd_gemm, mugd_groupnorm, mugd_layernorm, mugd_attention, mugd_s4conv, mugd_ddim_update, mugd_transpose,
 * mugd_copy2d, mugd_notes, mugd_embed, mugd_tf32_split, mugd_posterior} so a foreign-language mirror can verify its layout */
int  mugd_abi_sizes(int32_t* out, int32_t n);

#ifdef __cplusplus
}
#endif
#endif /* MUGD_H */

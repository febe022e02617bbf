/* A host without Python: run one Mug-Diffusion sampling request (S DDIM steps with classifier-free guidance + first-stage decode)
 * from a bundle written by `python -m mug_diffusion_b200.bundle`, through the C ABI of libmugd.so only.
 *
 *   make -C examples/host_c            (gcc + the CUDA runtime; no torch, no Python)
 *   examples/host_c/sample_host <bundle dir>             (reproduce the bundle's request, compare with its expected outputs)
 *   examples/host_c/sample_host <bundle dir> --seed N    (a seeded bundle: draw charts N, N + 1, ... instead; no comparison)
 *
 * manifest.txt lines:  region <name> <bytes> zero|file <file>   |  plan <file> run|graph  |  sample <eval> <tail> <steps>
 *                      stage <field> <region> <offset>          (one pointer of the mugd_stage of the next `staged` line)
 *                      staged <eval> <tail> <steps> <q_coef file>|- <B> <C> <L>   (inpainting / eta > 0: mugd_sample_staged)
 *                      seeds <file> <B>                         (a seeded bundle: the charts' uint64 seeds, uploaded once)
 *                      randn <region> <purpose> <first_draw> <n_draws> <draw_stride> <B> <n>   (fill a region with mugd_randn)
 *                      expect <region> <bytes> <file>           (outputs to compare; exit status 1 on mismatch)
 * This mirrors what DDIMSampler.sample + model.decode do in the reference (mug/diffusion/ddim.py:56-196, diffusion.py:49-50). */
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/mugd.h"

#define MAXR 128
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); exit(2); } } while (0)
#define MK(x) do { int r_ = (x); if (r_ != MUGD_OK) { fprintf(stderr, "%s:%d libmugd status %d: %s\n", __FILE__, __LINE__, r_, mugd_last_error()); exit(2); } } while (0)

static mugd_region regions[MAXR];
static char names[MAXR][48];
static int n_regions = 0;

static void* read_file(const char* dir, const char* name, long long expect_bytes) {
    char path[1024];
    snprintf(path, sizeof(path), "%s/%s", dir, name);
    FILE* f = fopen(path, "rb");
    if (!f) { fprintf(stderr, "cannot open %s\n", path); exit(2); }
    void* buf = malloc((size_t)expect_bytes);
    if (fread(buf, 1, (size_t)expect_bytes, f) != (size_t)expect_bytes) { fprintf(stderr, "%s is shorter than %lld bytes\n", path, expect_bytes); exit(2); }
    fclose(f);
    return buf;
}

static mugd_region* find_region(const char* name) {
    for (int i = 0; i < n_regions; ++i)
        if (strcmp(names[i], name) == 0) return &regions[i];
    fprintf(stderr, "unknown region %s\n", name);
    exit(2);
}

int main(int argc, char** argv) {
    if (argc != 2 && !(argc == 4 && strcmp(argv[2], "--seed") == 0)) { fprintf(stderr, "usage: %s <bundle dir> [--seed N]\n", argv[0]); return 2; }
    const char* dir = argv[1];
    const int own_seed = argc == 4;
    const unsigned long long seed0 = own_seed ? strtoull(argv[3], NULL, 10) : 0;
    char path[1024], line[2048];
    snprintf(path, sizeof(path), "%s/manifest.txt", dir);
    FILE* mf = fopen(path, "r");
    if (!mf) { fprintf(stderr, "cannot open %s\n", path); return 2; }

    mugd_handle* h = NULL;
    MK(mugd_create(0, &h));
    MK(mugd_set_gemm_impl(h, MUGD_GEMM_TC));
    cudaStream_t st;
    CK(cudaStreamCreate(&st));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    int bad = 0;
    float sample_ms = 0.f;
    mugd_stage stage;
    memset(&stage, 0, sizeof(stage));
    uint64_t* seeds = NULL;                /* device [B]: the charts' seeds of a seeded bundle */
    int n_seeds = 0;

    while (fgets(line, sizeof(line), mf)) {
        char a[64], b[256], c[256], d[256];
        long long nbytes;
        if (line[0] == '#' || sscanf(line, "%63s", a) != 1) continue;
        if (strcmp(a, "region") == 0) {
            if (sscanf(line, "%*s %47s %lld %255s %255s", names[n_regions], &nbytes, b, c) != 4 || n_regions >= MAXR) { fprintf(stderr, "bad line: %s", line); return 2; }
            mugd_region* r = &regions[n_regions];
            r->name = names[n_regions];
            r->bytes = nbytes;
            CK(cudaMalloc(&r->base, (size_t)nbytes));
            CK(cudaMemset(r->base, 0, (size_t)nbytes));
            if (strcmp(b, "file") == 0) {
                void* buf = read_file(dir, c, nbytes);
                CK(cudaMemcpy(r->base, buf, (size_t)nbytes, cudaMemcpyHostToDevice));
                free(buf);
            }
            ++n_regions;
        } else if (strcmp(a, "plan") == 0) {
            if (sscanf(line, "%*s %255s %255s", b, c) != 2) { fprintf(stderr, "bad line: %s", line); return 2; }
            snprintf(path, sizeof(path), "%s/%s", dir, b);
            mugd_plan* p = NULL;
            MK(mugd_plan_load(h, path, regions, n_regions, &p));
            if (strcmp(c, "graph") == 0) {
                MK(mugd_plan_run(p, st));                  /* warm-up outside capture (lazy module load) */
                MK(mugd_plan_capture(p, st));
                MK(mugd_plan_replay(p, 1, st));
            } else {
                MK(mugd_plan_run(p, st));
            }
            CK(cudaStreamSynchronize(st));
            printf("ran %-12s (%s, %d launches)\n", b, c, mugd_plan_launch_count(p));
            mugd_plan_destroy(p);
        } else if (strcmp(a, "stage") == 0) {
            long long off = 0;
            if (sscanf(line, "%*s %63s %255s %lld", d, b, &off) != 3) { fprintf(stderr, "bad line: %s", line); return 2; }
            mugd_region* r = find_region(b);
            if (off < 0 || off >= r->bytes) { fprintf(stderr, "offset outside region %s: %s", b, line); return 2; }
            void* p = (char*)r->base + off;
            if (strcmp(d, "x") == 0) stage.x = (float*)p;
            else if (strcmp(d, "x_dup") == 0) stage.x_dup = (float*)p;
            else if (strcmp(d, "x0") == 0) stage.x0 = (const float*)p;
            else if (strcmp(d, "mask") == 0) stage.mask = (const float*)p;
            else if (strcmp(d, "q_noise") == 0) stage.q_noise = (const float*)p;
            else if (strcmp(d, "noise") == 0) stage.noise = (const float*)p;
            else if (strcmp(d, "noise_rows") == 0) stage.noise_rows = (float*)p;
            else { fprintf(stderr, "unknown stage field: %s", line); return 2; }
        } else if (strcmp(a, "sample") == 0 || strcmp(a, "staged") == 0) {
            const int staged = strcmp(a, "staged") == 0;
            int steps = 0;
            float* q_coef = NULL;
            if (staged) {
                if (sscanf(line, "%*s %255s %255s %d %255s %d %d %d", b, c, &steps, d, &stage.B, &stage.C, &stage.L) != 7 || steps < 0) {
                    fprintf(stderr, "bad line: %s", line);
                    return 2;
                }
                if (strcmp(d, "-") != 0) q_coef = (float*)read_file(dir, d, 8LL * steps);   /* host array [steps][2] */
                stage.q_coef = q_coef;
            } else if (sscanf(line, "%*s %255s %255s %d", b, c, &steps) != 3) { fprintf(stderr, "bad line: %s", line); return 2; }
            mugd_plan *pe = NULL, *pt = NULL;
            snprintf(path, sizeof(path), "%s/%s", dir, b);
            MK(mugd_plan_load(h, path, regions, n_regions, &pe));
            snprintf(path, sizeof(path), "%s/%s", dir, c);
            MK(mugd_plan_load(h, path, regions, n_regions, &pt));
            const mugd_op* tail = NULL;
            int32_t n_tail = 0;
            MK(mugd_plan_ops(pt, &tail, &n_tail));
            /* capture needs one eager pass first; that pass must not disturb the request, so save / restore the latent and counters:
             * here simply: run the eager warm-up BEFORE loadx would be wrong, so warm up on a copy of the state */
            mugd_region* arena = find_region("arena");
            void* snap = NULL;
            CK(cudaMalloc(&snap, (size_t)arena->bytes));
            CK(cudaMemcpy(snap, arena->base, (size_t)arena->bytes, cudaMemcpyDeviceToDevice));
            MK(mugd_plan_run(pe, st));
            MK(mugd_plan_capture(pe, st));
            CK(cudaStreamSynchronize(st));
            CK(cudaMemcpy(arena->base, snap, (size_t)arena->bytes, cudaMemcpyDeviceToDevice));
            CK(cudaFree(snap));
            CK(cudaEventRecord(e0, st));
            /* the whole DDIM loop: one call, no synchronisation inside */
            if (staged) MK(mugd_sample_staged(pe, &stage, tail, n_tail, steps, st));
            else MK(mugd_sample(pe, tail, n_tail, steps, st));
            CK(cudaEventRecord(e1, st));
            CK(cudaStreamSynchronize(st));
            CK(cudaEventElapsedTime(&sample_ms, e0, e1));
            printf("sampled %d DDIM steps in %.3f ms (%.1f steps/s, %d launches per evaluation)%s\n", steps, sample_ms, 1000.0 * steps / sample_ms,
                   mugd_plan_launch_count(pe), staged ? (q_coef ? ", staged: inpainting" : ", staged: step noise") : "");
            free(q_coef);
            mugd_plan_destroy(pe);
            mugd_plan_destroy(pt);
        } else if (strcmp(a, "seeds") == 0) {
            if (sscanf(line, "%*s %255s %d", b, &n_seeds) != 2 || n_seeds < 1 || seeds) { fprintf(stderr, "bad line: %s", line); return 2; }
            uint64_t* host = (uint64_t*)read_file(dir, b, 8LL * n_seeds);
            for (int i = 0; own_seed && i < n_seeds; ++i) host[i] = seed0 + (unsigned long long)i;   /* chart i = seed + i (mod 2^64) */
            CK(cudaMalloc((void**)&seeds, 8 * (size_t)n_seeds));
            CK(cudaMemcpy(seeds, host, 8 * (size_t)n_seeds, cudaMemcpyHostToDevice));
            free(host);
        } else if (strcmp(a, "randn") == 0) {
            mugd_normal nd;
            memset(&nd, 0, sizeof(nd));
            long long n = 0;
            if (sscanf(line, "%*s %63s %d %d %d %d %d %lld", d, &nd.purpose, &nd.first_draw, &nd.n_draws, &nd.draw_stride, &nd.B, &n) != 7 ||
                !seeds || nd.B != n_seeds) {
                fprintf(stderr, "bad line (or no seeds line before it): %s", line);
                return 2;
            }
            mugd_region* r = find_region(d);
            if (4LL * n * nd.B * nd.n_draws > r->bytes) { fprintf(stderr, "randn table larger than region %s: %s", d, line); return 2; }
            nd.out = (float*)r->base;
            nd.seeds = seeds;
            nd.n = n;
            MK(mugd_randn(&nd, st));
            CK(cudaStreamSynchronize(st));
            printf("drew %-12s purpose %d, draws %d x %d from %d, %d charts\n", d, nd.purpose, nd.n_draws, nd.draw_stride, nd.first_draw, nd.B);
        } else if (strcmp(a, "expect") == 0) {
            if (own_seed) {
                if (sscanf(line, "%*s %63s", d) == 1) printf("%-12s not compared: charts drawn from --seed %llu\n", d, seed0);
                continue;
            }
            if (sscanf(line, "%*s %63s %lld %255s", d, &nbytes, b) != 3) { fprintf(stderr, "bad line: %s", line); return 2; }
            mugd_region* r = find_region(d);
            float* got = (float*)malloc((size_t)nbytes);
            float* want = (float*)read_file(dir, b, nbytes);
            CK(cudaMemcpy(got, r->base, (size_t)nbytes, cudaMemcpyDeviceToHost));
            double maxabs = 0.0, maxerr = 0.0;
            long long n = nbytes / 4, nonfinite = 0;
            for (long long i = 0; i < n; ++i) {
                if (!isfinite(got[i])) ++nonfinite;
                if (fabs(want[i]) > maxabs) maxabs = fabs(want[i]);
                if (fabs((double)got[i] - want[i]) > maxerr) maxerr = fabs((double)got[i] - want[i]);
            }
            const double rel = maxerr / (maxabs > 0 ? maxabs : 1.0);
            /* same kernels, same plans, same data: equal up to the summation order of the fp64 row-moment atomics */
            const int ok = nonfinite == 0 && rel < 1e-5;
            printf("%-12s %lld values, max |x| %.4f, max abs diff to the Python run %.3e (rel %.2e)  %s\n", d, n, maxabs, maxerr, rel, ok ? "OK" : "MISMATCH");
            if (!ok) bad = 1;
            free(got);
            free(want);
        }
    }
    fclose(mf);
    if (own_seed && !seeds) { fprintf(stderr, "--seed needs a seeded bundle (python -m mug_diffusion_b200.bundle ... --seeds ...)\n"); return 2; }
    if (seeds) CK(cudaFree(seeds));
    mugd_destroy(h);
    return bad;
}

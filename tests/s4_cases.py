"""The S4 layer's kernels (csrc/s4.cu) against float64: the references, the per-output bound, the launch rule and the case lists
shared by tests/test_s4_cases.py (CPU) and tests/test_gpu_s4.py (GPU).

* ``kgen64`` restates SSKernelNPLR.forward (mug/model/s4.py:771-792, oracle.s4_nplr_kernel) in complex128, in the reference's own
  Woodbury / Cauchy form -- not the (1+omega)-scaled form the kernel evaluates -- with the closed-form limit at the exact Nyquist node.
* ``conv64`` is the causal convolution y = gelu(conv(u, K) + D u) in float64 by FFT, with the condition sum of every output, and
  ``conv_ratio`` the per-output error bound every s4conv result is held to.
* ``s4conv_branch`` restates the branch rule of ``launch_s4conv`` (s4.cu:278-304): which kernel, how many CTAs share a sample's
  outputs (nsplit), and whether the middle super block / window pairs with itself.
* ``plan_s4conv_shapes`` walks the compiled U-Net plans for the (Beff, L, H) of every s4conv they launch; ``kgen_plan_shapes`` gives
  the (H, L_internal, L_out) the runtime generates for them (runtime.Session._gen_s4_kernels with the s4_setup.lengthen rule).
"""
import math
from collections import namedtuple
from functools import lru_cache

import torch

from mug_diffusion_b200 import synth

U32 = 2.0 ** -24                      # unit roundoff of float32

# ---- kernel generation --------------------------------------------------------------------------------------------------------
S4_PARAMS = (("C", "s4_C", True), ("log_dt", "s4_log_dt", False), ("B", "s4_B", True), ("P", "s4_P", True),
             ("inv_w_real", "s4_inv_w_real", False), ("w_imag", "s4_w_imag", False))


def s4_params(H: int, N: int = 32, seed: int = 3) -> dict:
    """one S4 layer's kernel parameters as the synthetic model draws them (float32, CPU): B, C, P [1,H,N,2], log_dt [H],
    inv_w_real, w_imag [H,N]"""
    return {n: synth._init("t." + n, (1, H, N, 2) if cplx else ((H,) if n == "log_dt" else (H, N)), role, seed)
            for n, role, cplx in S4_PARAMS}


def _poles(p: dict):
    dt = torch.exp(p["log_dt"].double())                                            # (H)
    cx = {n: torch.view_as_complex(p[n].double().contiguous())[0] for n in ("B", "C", "P")}   # (H,N)
    w = (-torch.exp(p["inv_w_real"].double()) + 1j * p["w_imag"].double()) * dt[:, None]      # w' = w dt (H,N)
    return dt, cx["B"], cx["C"], cx["P"], w


def woodbury(p: dict, om: torch.Tensor) -> torch.Tensor:
    """k(omega) of the reference at the nodes ``om`` (complex128 [F], none equal to -1):
    z = 2(1-omega)/(1+omega),  r_xy = dt sum_n v_xy[n] / (z - w'_n),  k = (r00 - r01 r10 / (1 + r11)) 2/(1+omega)
    with v00 = B C, v01 = B conj(P), v10 = P C, v11 = P conj(P).  Returns [H, F] complex128."""
    dt, Bc, Cc, Pc, w = _poles(p)
    Qc = Pc.conj()
    z = 2 * (1 - om) / (1 + om)                                                     # (F)
    r = [torch.zeros(w.shape[0], om.numel(), dtype=torch.complex128) for _ in range(4)]
    for n in range(w.shape[1]):                                                     # Cauchy sums, one pole at a time
        inv = 1.0 / (z[None, :] - w[:, n:n + 1])                                    # (H,F)
        for i, v in enumerate((Bc[:, n] * Cc[:, n], Bc[:, n] * Qc[:, n], Pc[:, n] * Cc[:, n], Pc[:, n] * Qc[:, n])):
            r[i] += v[:, None] * inv
    r00, r01, r10, r11 = (x * dt[:, None] for x in r)
    return (r00 - r01 * r10 / (1 + r11)) * 2 / (1 + om)[None, :]


def nyquist_limit(p: dict) -> torch.Tensor:
    """lim k(omega) as omega -> -1: z ~ 4/(1+omega) grows without bound, so r_xy ~ dt (1+omega)/4 sum_n v_xy[n]; then
    2/(1+omega) r00 -> (dt/2) sum_n B_n C_n, while the Woodbury correction is O((1+omega)^2) / (1+omega) -> 0.  [H] complex128"""
    dt, Bc, Cc, _, _ = _poles(p)
    return dt / 2 * (Bc * Cc).sum(-1)


def nodes64(L_int: int, table=None) -> torch.Tensor:
    """omega_f, f = 0..L_int/2, complex128: the reference's complex64 table (runtime.s4_fft_nodes, [nf, 2] float32) upcast, or
    the exact nodes exp(-2 pi i f / L_int), with the Nyquist node exactly -1"""
    nf = L_int // 2 + 1
    if table is not None:
        t = table.double()
        return torch.complex(t[:, 0], t[:, 1])
    f = torch.arange(nf, dtype=torch.float64)
    om = torch.exp(-2j * math.pi * f / L_int)
    if L_int % 2 == 0:
        om[-1] = -1.0
    return om


def kgen64(p: dict, L_int: int, L_out: int, nodes: torch.Tensor) -> torch.Tensor:
    """SSKernelNPLR's K in float64: irfft(k(omega_f), L_int)[:L_out] (C2R: the imaginary parts of the DC and Nyquist bins are
    ignored).  ``nodes`` from nodes64; a node equal to -1 takes the closed-form limit.  Returns [H, L_out] float64 (CPU)."""
    nyq = nodes == -1
    kf = torch.empty(p["log_dt"].numel(), nodes.numel(), dtype=torch.complex128)
    kf[:, ~nyq] = woodbury(p, nodes[~nyq])
    if bool(nyq.any()):
        kf[:, nyq] = nyquist_limit(p)[:, None]
    return torch.fft.irfft(kf, n=L_int)[:, :L_out]


KGEN_EPS64 = 1e-12                    # the fp64 DFT and Cauchy sums, relative to max|K| (calibrated: DESIGN §2)


def kgen_ratio(kt: torch.Tensor, k64: torch.Tensor) -> torch.Tensor:
    """|Kt - K64| / (2^-24 |K64| + eps64 max|K64|) per tap: one float32 rounding of each output plus the fp64 work. kt [L, H]"""
    e = (kt.double().cpu().t() - k64).abs()
    return e / (U32 * k64.abs() + KGEN_EPS64 * k64.abs().max())


# ---- the convolution ----------------------------------------------------------------------------------------------------------
GELU_D_MAX = 1.1289                   # max |gelu'(x)| (at x = sqrt(2), 1.12886...)


def gelu64(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2.0)))


def _causal(a, b, L):
    """sum_{j <= l} b[j] a[l - j] along dim 1 of a [B, L, H] (b [L, H]) by a float64 FFT of length 2L"""
    fa = torch.fft.rfft(a, n=2 * L, dim=1)
    fb = torch.fft.rfft(b, n=2 * L, dim=0)
    return torch.fft.irfft(fa * fb[None], n=2 * L, dim=1)[:, :L]


def conv64(u: torch.Tensor, K: torch.Tensor, D: torch.Tensor):
    """u [B, L, H], K [L, H] (tap j of channel h at K[j, h]), D [H], on any device.  Returns (y64, S): y64 = gelu(conv + D u) in
    float64 and the condition sum S[l] = sum_j |K[j]| |u[l-j]| + |D u[l]| of every pre-activation output."""
    L = u.shape[1]
    u, K, D = u.double(), K.double(), D.double()
    du = u * D
    x = _causal(u, K, L) + du
    S = (_causal(u.abs(), K.abs(), L) + du.abs()).clamp_min(0)
    return gelu64(x), S


# the per-output bound constant c1 = c2: 4x the worst ratio measured on an H100 80GB HBM3 (700 W), 1.51 (DESIGN §2)
CONV_BOUND = 6.0
# the float64 FFT reference's own error, relative to max S: it is absolute, not per output, and shows where the exact output is 0
# (taps that are all zero up to l, and u[l] == 0: the kernel returns 0, the FFT about 1e-16)
CONV_EPS64 = 1e-13


def conv_ratio(y: torch.Tensor, y64: torch.Tensor, S: torch.Tensor) -> torch.Tensor:
    """|y - y64| / (2^-24 (|y64| + sqrt(l+1) S[l] max|gelu'|) + eps64 max S) per output; y, y64, S [B, L, H].  A float32 sum of
    l+1 products in any order stays within a few of sqrt(l+1) u S[l] (random-walk rounding); gelu adds a few ulp of |y| and passes
    the pre-activation error on with a factor |gelu'| <= 1.129.  The check is ratio <= CONV_BOUND for every element."""
    L = y.shape[1]
    sq = torch.sqrt(torch.arange(1, L + 1, dtype=torch.float64, device=y64.device))[None, :, None]
    return (y.double() - y64).abs() / (U32 * (y64.abs() + sq * S * GELU_D_MAX) + CONV_EPS64 * S.max())


def taps(kind: str, L: int, H: int, gen: torch.Generator, device="cpu") -> torch.Tensor:
    """[L, H] float32 taps that carry weight in every tap tile: 'slow' = randn * exp(-j / L) (decays by e over the whole length),
    'tail' = only the last min(L, 256) taps nonzero"""
    K = torch.randn(L, H, generator=gen, device=device)
    if kind == "slow":
        return K * torch.exp(-torch.arange(L, device=device, dtype=torch.float32) / L)[:, None]
    assert kind == "tail"
    K[:max(0, L - 256)] = 0
    return K


# ---- the launch rule (s4.cu:278-304) ------------------------------------------------------------------------------------------
H100_SMS = 132                        # H100 SXM
H100_SMEM_OPTIN = 232448              # cudaDevAttrMaxSharedMemoryPerBlockOptin on sm_90
AUTO, RESIDENT, STREAMED = 0, 1, 2    # mugd_set_s4conv_impl
S4_WARPS, S4_R, S4_CH, S4_PITCH, S4_PAD = 16, 8, 16, 18, 32
S4S_W, S4S_SMEM = 256, 112896

Branch = namedtuple("Branch", "kernel nsplit odd")
Branch.__doc__ = """kernel: 'resident-blocked' / 'resident-interleaved' / 'streamed'; nsplit: CTAs per (16 channels, sample); odd: an odd
number of super blocks (resident) or windows (streamed), so the middle one is paired with itself"""


def resident_smem(L: int) -> int:
    Lpad = (L + 2 * S4_R - 1) // (2 * S4_R) * (2 * S4_R)
    return ((S4_PAD + Lpad) + (Lpad + 3 * S4_R)) * S4_PITCH * 4


def s4conv_branch(B: int, L: int, H: int, sm_count: int = H100_SMS, smem_optin: int = H100_SMEM_OPTIN, impl: int = AUTO):
    """the kernel launch_s4conv picks for (B, L, H) on a device with ``sm_count`` SMs, or None where it refuses (forced resident
    kernel beyond its shared memory)"""
    base = (H // S4_CH) * B
    if impl == STREAMED or (impl == AUTO and resident_smem(L) > smem_optin):
        if S4S_SMEM > smem_optin:
            return None
        nwin = (L + S4S_W - 1) // S4S_W
        npairs = (nwin + 1) // 2
        nsplit = 1
        while nsplit < npairs and base * nsplit < 2 * sm_count:
            nsplit += 1
        return Branch("streamed", nsplit, nwin % 2 == 1)
    if resident_smem(L) > smem_optin:
        return None
    Lpad = (L + 2 * S4_R - 1) // (2 * S4_R) * (2 * S4_R)
    nsb = Lpad // (2 * S4_R)
    npairs = (nsb + 1) // 2
    nsplit = 1
    while nsplit < 16 and ((base * nsplit < 2 * sm_count and nsplit * 2 * S4_WARPS <= npairs) or
                           (base * nsplit < sm_count and nsplit * S4_WARPS <= npairs)):
        nsplit *= 2
    kernel = "resident-interleaved" if 2 * npairs <= nsplit * S4_WARPS else "resident-blocked"
    return Branch(kernel, nsplit, nsb % 2 == 1)


def case_impls(B: int, L: int, H: int, smem_optin: int = H100_SMEM_OPTIN):
    """the impls a convolution case runs: the automatic dispatch, and both forced kernels wherever the resident one fits"""
    return (AUTO, RESIDENT, STREAMED) if resident_smem(L) <= smem_optin else (AUTO,)


def branch_class(br: Branch) -> tuple:
    """the coverage classes of a branch (the nsplit values that change what a CTA does: 1, 2, 4, >= 8; for the streamed kernel 1 or
    more)"""
    if br.kernel == "streamed":
        return (br.kernel, "nsplit=1" if br.nsplit == 1 else "nsplit>1", "odd" if br.odd else "even")
    ns = "nsplit>=8" if br.nsplit >= 8 else f"nsplit={br.nsplit}"
    return (br.kernel, ns, "odd" if br.odd else "even")


def reachable_classes(sm_count: int = H100_SMS, smem_optin: int = H100_SMEM_OPTIN, max_base: int = 1024) -> set:
    """every branch class the rule can produce on this device: nsplit depends on (B, H) only through base = B H / 16, and on L only
    through the super-block or window count"""
    out = set()
    for base in range(1, max_base + 1):
        L = 16
        while resident_smem(L) <= smem_optin:                      # one L per super-block count
            out.add(branch_class(s4conv_branch(base, L, S4_CH, sm_count, smem_optin, RESIDENT)))
            L += 16
        for nwin in range(1, 8192 // S4S_W + 1):                    # one L per window count, up to z_length 8192
            out.add(branch_class(s4conv_branch(base, nwin * S4S_W, S4_CH, sm_count, smem_optin, STREAMED)))
    return out


# ---- the plans ------------------------------------------------------------------------------------------------------------------
PLAN_Z = (96, 512, 992, 1568, 1600, 2048, 4096, 8192)
PLAN_BEFF = (2, 8, 32)                # the effective batch (CFG doubles the charts): 1, 4 and 16 guided charts


@lru_cache(maxsize=None)
def _compiler():
    from mug_diffusion_b200 import packer
    from mug_diffusion_b200.config import ModelConfig
    from mug_diffusion_b200.engine import UNetCompiler
    cfg = ModelConfig()
    blob = packer.pack_model(synth.synthetic_state_dict(96), cfg.unet, cfg.decoder)
    return UNetCompiler(cfg.unet, blob, 1 << 30)


def s4_blocks():
    """(H, ds) of every S4 layer of the U-Net, in plan order"""
    return [(b.cin, b.ds) for b in _compiler().lay.blocks() if b.kind == "s4"]


@lru_cache(maxsize=None)
def plan_s4conv_shapes(zs=PLAN_Z, beffs=PLAN_BEFF) -> tuple:
    """(Beff, L, H) of every s4conv op in the compiled U-Net plans (plain and ragged) for these z_lengths and effective batches"""
    from mug_diffusion_b200 import lib as L_
    from mug_diffusion_b200.engine import Arena, View
    comp = _compiler()
    blocks = list(comp.lay.blocks())
    shapes = {}
    for Beff in beffs:
        for Lz in zs:
            ext = dict(emb_table=1 << 40, step=(1 << 40) + 4096, ctx_tokens=21,
                       ctx_kv=[View((1 << 41) + i * (1 << 24), 2 * b.cin, Beff * 21, 2 * b.cin)
                               for i, b in enumerate(x for x in blocks if x.kind == "attn")],
                       s4_kt={b.prefix: View((1 << 42) + i * (1 << 26), b.cin, Lz // b.ds, b.cin)
                              for i, b in enumerate(x for x in blocks if x.kind == "s4")})
            for valid in (None, [1 << 43] * comp.cfg.levels):
                for o in comp.compile(Arena(1 << 44), Beff, Lz, ext, False, None, valid)["ops"].ops:
                    if o.kind == L_.OP_S4CONV:
                        s = o.u.s4
                        assert s.ldu == s.H and s.ldy == s.H, "the plans run s4conv on whole buffers"
                        shapes.setdefault((s.B, s.L, s.H), None)
    return tuple(shapes)


def lengthened(L_persisted: int, L_req: int) -> int:
    """the internal length s4_setup.lengthen leaves for a request of L_req on a layer persisted at L_persisted"""
    L = L_persisted
    if L == 0:
        return L_req
    while L < L_req:
        L *= 2
    return L


# a fresh model (its kernel length set by the first request) and a trained checkpoint, whose S4 lengths were persisted at z_length
# 512 (DESIGN §6b, long songs): it is lengthened by doubling, or is longer than a short request
KGEN_PERSISTED = (None, 512)


def kgen_plan_shapes(zs=PLAN_Z) -> list:
    """(H, L_internal, L_out) the runtime generates for every S4 layer at these z_lengths, for each model of KGEN_PERSISTED"""
    out = {}
    for Lz in zs:
        for H, ds in s4_blocks():
            for zp in KGEN_PERSISTED:
                out.setdefault((H, lengthened((zp or Lz) // ds, Lz // ds), Lz // ds), None)
    return sorted(out, key=lambda s: (s[1], s[2], s[0]))


# ---- the convolution case list --------------------------------------------------------------------------------------------------
EDGE_L = (1, 7, 15, 16, 17, 257, 511, 513, 1000, 1583, 1584, 1585)


def conv_cases() -> list:
    """(B, L, H, strided) of every convolution case: the plan shapes (whole buffers, as the plans run them), and the edges --
    lengths around a super block (16), a streamed window (256) and the resident kernel's limit (1584) -- at H = 16, B = 1, and at
    (B, H) = (3, 48); the edges with u and y as column windows of wider buffers"""
    cases = [(B, L, H, False) for B, L, H in plan_s4conv_shapes()]
    cases += [(1, L, 16, True) for L in EDGE_L] + [(3, L, 48, True) for L in EDGE_L]
    return cases


def case_branches(cases, sm_count: int = H100_SMS, smem_optin: int = H100_SMEM_OPTIN) -> set:
    """the branch classes the convolution cases reach: every case under each impl it runs"""
    out = set()
    for B, L, H, _ in cases:
        for impl in case_impls(B, L, H, smem_optin):
            out.add(branch_class(s4conv_branch(B, L, H, sm_count, smem_optin, impl)))
    return out

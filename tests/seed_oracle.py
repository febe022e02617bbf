"""numpy oracle of mugd_randn (csrc/randn.cu): Philox4x32-10 in exact integer arithmetic and Box-Muller in float64."""
import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """Random123's philox4x32_10 on uint64 arrays holding 32-bit words: ctr = (c0, c1, c2, c3), key = (k0, k1), broadcast"""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & MASK for c in ctr)
    k0, k1 = (np.asarray(k, dtype=np.uint64) & MASK for k in key)
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
        p0, p1 = np.uint64(M0) * c0, np.uint64(M1) * c2            # < 2^64: exact
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & MASK, (p0 >> 32) ^ c3 ^ k1, p0 & MASK
    return c0, c1, c2, c3


def box_muller64(xa, xb):
    """(z_even, z_odd) in float64 from the same 24-bit uniforms the kernel forms"""
    u1 = ((np.asarray(xa, np.uint64) >> 8) + 1).astype(np.float64) * 2.0 ** -24
    u2 = (np.asarray(xb, np.uint64) >> 8).astype(np.float64) * 2.0 ** -24
    r = np.sqrt(-2.0 * np.log(u1))
    return r * np.cos(2 * np.pi * u2), r * np.sin(2 * np.pi * u2)


def normals(seeds, n, purpose, first_draw, n_draws, draw_stride=1):
    """the float64 table out[k][b][e] mugd_randn fills: draw first_draw + draw_stride * k of chart b (seed seeds[b]), n elements"""
    seeds = np.asarray([int(s) for s in seeds], dtype=np.uint64)
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    out = np.empty((n_draws, len(seeds), 4 * q.size))
    for k in range(n_draws):
        draw = first_draw + draw_stride * k
        for b, s in enumerate(seeds):
            x = philox4x32_10((q, draw, purpose, 0), (s & MASK, s >> np.uint64(32)))
            z0, z1 = box_muller64(x[0], x[1])
            z2, z3 = box_muller64(x[2], x[3])
            out[k, b] = np.stack([z0, z1, z2, z3], 1).reshape(-1)
    return out[:, :, :n]

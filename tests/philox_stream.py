"""Python port of philox4x32 (csrc/rp_philox.cuh, Philox4x32-10) and of the scalable cross-entropy head's normal draw
(sce_draw_kernel in csrc/rp_sce_head.cu): uint32 arithmetic on uint64 numpy arrays.

Pair p of a draw keyed by seed_eff = seed + *rng_counter is r = philox4x32(seed_eff, SCE_SITE + p) and
  u1 = (float(r.x) + 1) * 2^-32   in (0, 1]      (fp32 steps, as the kernel)
  u2 = float(r.y) * 2^-32         in [0, 1)
  draw[2p] = sqrt(-2 log u1) cos(2 pi u2),  draw[2p + 1] = sqrt(-2 log u1) sin(2 pi u2)   (when 2p + 1 < n)
The port evaluates log / sqrt / cos / sin in float64 from the fp32 u1, u2: the kernel's fast-math logf is accurate in
absolute terms only, so a comparison needs an absolute slack (tests/test_gpu_sce_head.py).  test_sce_reference_cpu.py
pins the constants and the lines restated here against the sources."""
import numpy as np

_M32 = np.uint64(0xFFFFFFFF)
_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
SCE_SITE = 0x5CE << 40           # kSceSite: Philox counter offset of the SCE bucket draw
_TWO_M32 = np.float32(2.3283064365386963e-10)


def philox4x32(seed, ctr):
    """(x, y, z, w) uint64 arrays holding the four uint32 words of philox4x32(seed, ctr) for every counter in ``ctr``."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    ctr = np.asarray(ctr, dtype=np.uint64)
    c0, c1 = ctr & _M32, ctr >> np.uint64(32)
    c2 = np.zeros_like(c0)
    c3 = np.zeros_like(c0)
    k0, k1 = seed & 0xFFFFFFFF, seed >> 32
    for _ in range(10):
        p0 = np.uint64(_M0) * c0                      # < 2^64: exact in uint64
        p1 = np.uint64(_M1) * c2
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & _M32, p1 >> np.uint64(32), p1 & _M32
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return c0, c1, c2, c3


def sce_uniforms(seed_eff, n_pairs):
    """fp32 (u1, u2) of pairs 0 .. n_pairs - 1, exactly as the kernel forms them."""
    r = philox4x32(seed_eff, np.uint64(SCE_SITE) + np.arange(n_pairs, dtype=np.uint64))
    u1 = (r[0].astype(np.float64).astype(np.float32) + np.float32(1.0)) * _TWO_M32
    u2 = r[1].astype(np.float64).astype(np.float32) * _TWO_M32
    return u1, u2


def sce_normals(seed, counter, n):
    """float64 [n]: the SCE head's standard normals for seed + counter (uint64 wrap-around)."""
    u1, u2 = sce_uniforms((int(seed) + int(counter)) & 0xFFFFFFFFFFFFFFFF, (n + 1) // 2)
    rad = np.sqrt(-2.0 * np.log(u1.astype(np.float64)))
    ang = np.pi * (np.float32(2.0) * u2).astype(np.float64)
    out = np.empty(2 * len(u1))
    out[0::2] = rad * np.cos(ang)
    out[1::2] = rad * np.sin(ang)
    return out[:n]

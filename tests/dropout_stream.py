"""Python port of the dropout stream of csrc/rp_philox.cuh (drop_row_key / drop_col_key / drop_mix): uint32 arithmetic
on uint64 numpy arrays.  Element (row r, column j) of a dropout site with offset ``off`` is kept iff
drop_mix(drop_row_key(seed + *seed_ptr, off, r), drop_col_key(j)) >= (uint32)(p * 2^32).  Shared by the kernel-level
test files; test_gpu_attention.py pins it bit for bit against rp_dropout_bwd."""
import numpy as np
import torch

_M32 = 0xFFFFFFFF


def _u64(x):
    return np.asarray(x, dtype=np.uint64)


def _fmix32(h):
    h = _u64(h)
    h = h ^ (h >> np.uint64(16))
    h = (h * np.uint64(0x85EBCA6B)) & np.uint64(_M32)
    h = h ^ (h >> np.uint64(13))
    h = (h * np.uint64(0xC2B2AE35)) & np.uint64(_M32)
    return h ^ (h >> np.uint64(16))


def drop_row_key(seed, off, row):
    seed, off = int(seed) & 0xFFFFFFFFFFFFFFFF, int(off)
    s = int(_fmix32((seed & _M32) ^ (((seed >> 32) * 0x85EBCA77) & _M32) ^ ((((off >> 32) & _M32) * 0xC2B2AE3D) & _M32)
                    ^ (((off & _M32) * 0x27D4EB2F) & _M32)))
    row = _u64(row)
    lo = (row & np.uint64(_M32)) * np.uint64(0x9E3779B1) & np.uint64(_M32)
    hi = (row >> np.uint64(32)) * np.uint64(0x165667B1) & np.uint64(_M32)
    return _fmix32((np.uint64(s) + lo + hi) & np.uint64(_M32))


def drop_col_key(j):
    return _fmix32((_u64(j) * np.uint64(0x9E3779B1) + np.uint64(0x27D4EB2F)) & np.uint64(_M32))


def drop_mix(row_key, col_key):
    x = ((_u64(row_key) ^ _u64(col_key)) * np.uint64(0x9E3779B1)) & np.uint64(_M32)
    x = x ^ (x >> np.uint64(15))
    return (x * np.uint64(0x85EBCA77)) & np.uint64(_M32)


def _threshold(p):
    return int(float(np.float32(p)) * 4294967296.0)   # (uint32_t)(drop_p * 4294967296.0), drop_p a float


def keep_draws(seed_eff, off, p, rows, n_cols):
    """bool [len(rows), n_cols]: element (row r, column j) of the site is kept."""
    rk = drop_row_key(seed_eff, off, rows)
    ck = drop_col_key(np.arange(n_cols))
    return torch.from_numpy(drop_mix(rk[:, None], ck[None, :]) >= np.uint64(_threshold(p)))


def drop_keep(seed_eff, off, p, B, H, L, row_pitch):
    """float64 [B, H, L, L]: 0 or 1/(1-p) for (query i, key j) of head bz = b*H + h, row key at bz*row_pitch + i."""
    rows = (np.arange(B * H)[:, None] * row_pitch + np.arange(L)[None, :]).reshape(-1)
    keep = keep_draws(seed_eff, off, p, rows, L).view(B, H, L, L)
    return keep.double() / (1.0 - float(np.float32(p)))

"""Golden files of BERT4Rec at padded shapes (tests/golden/bert4rec_d*.npz, written by tools/gen_bert_shapes_golden.py from
the real reference).  Their weights are not stored: a hidden size of 512 has 3 M weights per block.  The generator draws them
with ``golden_weights`` from a seed that the file records, loads them into the reference model and runs it there.  The
tests draw the same weights again.

Every gradient of the model is stored, but a matrix with more than ROWS rows keeps ROWS of them (``rows::``): the half with
the largest norms (the items of the batch, the busiest units) and an evenly spaced half, each row with all its columns, so
every feature slot and the whole FFN inner axis are covered.  Values are float16 scaled by the largest stored magnitude
(``gscale::``): a relative precision of 2^-11, far inside the tolerances that read them."""
import numpy as np
import torch

# (hidden, heads, tied, n_items, blocks, batch, L, seed): the reference tutorial's 300 / 4 at a small catalog and L, a tied
# 96 / 2, head_dim 16, and an unpadded 512 / 8 whose biased head runs the d = 512 materialised-G backward
SHAPES = {"d300h4": (300, 4, False, 500, 1, 4, 20, 41), "d96h2_tied": (96, 2, True, 400, 2, 5, 16, 42),
          "d64h4": (64, 4, False, 300, 2, 5, 16, 43), "d512h8": (512, 8, False, 600, 1, 3, 16, 44)}


def golden_weights(names, shapes, seed):
    """Reference state_dict (key -> fp32 tensor) drawn on the CPU in key order: xavier-normal matrices, LayerNorm weights
    1 + N(0, 0.05), other vectors N(0, 0.05), the head bias N(0, 0.5) so that it moves the softmax / sigmoid visibly."""
    g = torch.Generator().manual_seed(int(seed))
    out = {}
    for k, shp in zip(names, shapes):
        shp = tuple(int(s) for s in shp)
        if len(shp) == 2:
            v = torch.randn(shp, generator=g) * (2.0 / (shp[0] + shp[1])) ** 0.5
        elif k.endswith(("norm.weight",)):
            v = 1.0 + 0.05 * torch.randn(shp, generator=g)
        elif k in ("_head.linear.bias", "_head.out_bias"):
            v = 0.5 * torch.randn(shp, generator=g)
        else:
            v = 0.05 * torch.randn(shp, generator=g)
        out[k] = v
    return out


ROWS = 64


def grad_rows(v: np.ndarray):
    """indices of the stored rows of gradient ``v``, or None when all of it is stored"""
    if v.ndim != 2 or v.shape[0] <= ROWS:
        return None
    top = np.argsort(-np.linalg.norm(v.astype(np.float64), axis=1), kind="stable")[: ROWS // 2]
    even = np.linspace(0, v.shape[0] - 1, ROWS // 2).round().astype(np.int64)
    return np.unique(np.concatenate([top, even]))


def pack_grads(grads: dict) -> dict:
    out = {}
    for k, v in grads.items():
        v = np.asarray(v, dtype=np.float32)
        rows = grad_rows(v)
        if rows is not None:
            out["rows::" + k] = rows
            v = v[rows]
        s = float(np.abs(v).max()) or 1.0
        out["grad16::" + k] = (v / s).astype(np.float16)
        out["gscale::" + k] = np.float32(s)
    return out


def unpack_grads(z) -> dict:
    """reference key -> (stored row indices (LongTensor) or None, fp32 gradient of those rows)"""
    out = {}
    for f in z.files:
        if f.startswith("grad16::"):
            k = f[8:]
            rows = torch.from_numpy(z["rows::" + k]).long() if "rows::" + k in z.files else None
            out[k] = (rows, torch.from_numpy(z[f].astype(np.float32) * z["gscale::" + k]))
    return out


def load(path):
    """(z, state_dict, grads): the npz, the reference weights and the reference gradients (unpack_grads)"""
    z = np.load(path)
    names = [str(n) for n in z["param_names"]]
    shapes = [tuple(s[s > 0]) for s in z["param_shapes"]]
    sd = golden_weights(names, shapes, int(z["init_seed"]))
    return z, sd, unpack_grads(z)

"""Error measures, LayerNorm references and the worst-error report shared by the fp64 body tests
(test_gpu_bert_body.py, test_gpu_sasrec_body.py).

- ``ulp_err``: element-wise, in units of half a bf16 ulp of the float64 reference plus an absolute slack, for outputs that
  are one rounding away from the exact value;
- ``block_err`` / ``seq_block_err``: the largest norm-relative error over 64-row blocks, for reductions, gradients and
  whole training steps, so that one wrong block cannot hide in a global norm.
"""
import os

import torch
import torch.nn.functional as F

BLOCK_FLOOR = 0.05       # a block whose reference norm is below this fraction of the typical block is measured against it


# ----------------------------------------------------------------------------------------------------------------------
# error measures
# ----------------------------------------------------------------------------------------------------------------------
def ulp_err(got, ref, atol):
    """max |got - ref| / (half a bf16 ulp of ref + atol), element-wise.  ``ref`` float64, ``atol`` >= 0 (tensor or scalar)."""
    r = ref.abs()
    half_ulp = torch.exp2(torch.floor(torch.log2(r.clamp_min(1e-300))) - 8)
    return float(((got.double() - ref).abs() / (half_ulp + atol)).max())


def block_err(got, ref, blk=64):
    """Largest norm-relative error over blocks of ``blk`` leading-axis entries of [R, ...] arrays.  A block whose reference
    norm is below BLOCK_FLOOR x the RMS block norm is measured against that floor."""
    got, ref = got.double().reshape(ref.shape[0], -1), ref.double().reshape(ref.shape[0], -1)
    R = ref.shape[0]
    nb = -(-R // blk)
    pad = (0, 0, 0, nb * blk - R)
    diff = F.pad(got - ref, pad).reshape(nb, -1).norm(dim=-1)
    den = F.pad(ref, pad).reshape(nb, -1).norm(dim=-1)
    floor = BLOCK_FLOOR * float(den.square().mean().sqrt()) + 1e-300
    return float((diff / den.clamp_min(floor)).max())


def seq_block_err(got, ref, real):
    """[B, L, d] hidden states: largest norm-relative error over (sequence, 64-row block)s of the real rows."""
    m = real[..., None].to(ref.dtype)
    return max(block_err(got[b] * m[b], ref[b] * m[b]) for b in range(ref.shape[0]))


# ----------------------------------------------------------------------------------------------------------------------
# float64 LayerNorm over the real features of a padded layout
# ----------------------------------------------------------------------------------------------------------------------
def feat_mask(d, hd_valid):
    """bool [d]: the real features of a padded layout (hd_valid 0 = all real)."""
    if hd_valid == 0:
        return torch.ones(d, dtype=torch.bool)
    slot = 64 if hd_valid <= 64 else 128
    return (torch.arange(d) % slot) < hd_valid


def ln_ref(x, w, b, eps, valid):
    """LayerNorm over the real features only -> (y, mean, rstd); padded outputs 0 (their w, b are 0)."""
    v = valid.to(x.device, x.dtype)
    n = float(v.sum())
    mean = (x * v).sum(-1, keepdim=True) / n
    var = (((x - mean) * v) ** 2).sum(-1, keepdim=True) / n
    rstd = 1.0 / torch.sqrt(var + eps)
    return ((x - mean) * rstd * w + b) * v, mean[..., 0], rstd[..., 0]


def ln_bwd_ref(dy, x, w, mean, rstd, valid):
    """dx (padded inputs get 0), sum_r dy * xhat, sum_r dy for one LayerNorm over the real features."""
    v = valid.to(x.device, x.dtype)
    n = float(v.sum())
    xh = (x - mean[:, None]) * rstd[:, None] * v
    g = dy * w * v
    dx = rstd[:, None] * (g - g.sum(-1, keepdim=True) / n - xh * (g * xh).sum(-1, keepdim=True) / n) * v
    return dx, (dy * xh).sum(0), dy.sum(0)


# ----------------------------------------------------------------------------------------------------------------------
# worst error of each family, printed at the end of a module (run pytest with -s to see it)
# ----------------------------------------------------------------------------------------------------------------------
class WorstErrors:
    def __init__(self):
        self.worst = {}

    def note(self, family, value):
        """Record the worst error of a family (and the case it came from); returns ``value`` as a float."""
        value = float(value)
        if value >= self.worst.get(family, (0.0, ""))[0]:
            self.worst[family] = (value, os.environ.get("PYTEST_CURRENT_TEST", "").split("::")[-1].split(" ")[0])
        return value

    def report(self):
        if self.worst:
            print("\nworst observed error per family:")
            for k, (v, case) in sorted(self.worst.items()):
                print(f"  {k:28s} {v:.3g}  {case}")

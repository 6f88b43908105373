"""The full-catalog BCE as this project states it (the float64 bodies of oracle/ and the BCE of tests/bce_reference.py) against
the REAL reference classes: replay.nn.loss.BCE through the new-path SasRec and the legacy Bert4Rec._compute_loss_bce, untied
and tied (tests/golden/full_bce_losses.npz, written by tools/gen_bce_golden.py).  This pins the rows the loss is taken over
(target_padding_mask; BERT4Rec's real and masked positions), the tied head's out_bias, and the gradients."""
import os

import numpy as np
import torch

from bce_reference import reference


def _leaf(P):
    return {k: ([{kk: vv.double().requires_grad_() for kk, vv in b.items()} for b in v] if k == "blocks"
                else v.double().requires_grad_()) for k, v in P.items()}


def _bce(h, W, b, y):
    x = h @ W.T + (0 if b is None else b)
    return (torch.nn.functional.softplus(x).sum() - x.gather(1, y[:, None]).sum()) / h.shape[0]


def _close(a, b, rtol=1e-4):
    a, b = torch.as_tensor(a).double(), torch.from_numpy(np.asarray(b)).double()
    assert a.shape == b.shape, (a.shape, b.shape)
    assert float((a - b).abs().max()) <= rtol * float(b.abs().max()) + 1e-9


def test_new_path_bce_matches_reference(golden_dir):
    from oracle import sasrec as osr

    z = np.load(os.path.join(golden_dir, "sasrec_new_tiny.npz"))
    zb = np.load(os.path.join(golden_dir, "full_bce_losses.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    P = _leaf(osr.params_from_new_state_dict(sd))
    n_items = int(z["n_items"])
    ids, pm = torch.from_numpy(z["ids"]), torch.from_numpy(z["pad_mask"])
    lab, tm = torch.from_numpy(z["labels"]), torch.from_numpy(z["target_mask"])
    hidden = osr.sasrec_body(P, ids, pm, int(z["H"]), variant="new")
    loss = _bce(hidden[tm], P["item_emb"][:n_items], None, lab[tm])
    loss.backward()
    _close(loss.detach(), zb["new_loss"], 1e-6)
    # row n_items is the padding embedding (padding_idx in the reference: no gradient; the float64 body does not mask it)
    assert not zb["new_gE"][n_items].any()
    _close(P["item_emb"].grad[:n_items], zb["new_gE"][:n_items])
    _close(P["blocks"][0]["in_w"].grad, zb["new_gW"])
    # the head restatement the GPU tests use gives the same loss and head gradient on these rows
    r = reference(hidden[tm].detach(), P["item_emb"][:n_items].detach(), None, lab[tm].int(), int(tm.sum()))
    _close(r["loss"], zb["new_loss"], 1e-6)


def _bert_case(golden_dir, tag, name):
    from oracle import bert4rec as ob

    z = np.load(os.path.join(golden_dir, f"bert4rec_{tag}.npz"))
    zb = np.load(os.path.join(golden_dir, "full_bce_losses.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    P = _leaf(ob.params_from_state_dict(sd))
    ids, pm, tok = (torch.from_numpy(z[k]) for k in ("ids", "pad_mask", "token_mask"))
    lab = torch.from_numpy(z["labels"])
    h = ob.bert4rec_body(P, ids, pm, tok, int(z["H"]))
    W, b = ob.head_weights(P)
    sel = pm & ~tok   # real and masked positions: ~((~pad_mask) + token_mask) of bert4rec/lightning.py:283-284
    loss = _bce(h[sel], W, b, lab[sel])
    loss.backward()
    _close(loss.detach(), zb[f"bert_{name}_loss"], 1e-6)
    _close(P["item_emb"].grad, zb[f"bert_{name}_gE"])
    _close(P["blocks"][0]["in_w"].grad, zb[f"bert_{name}_gW"])
    _close(P["head_b"].grad, zb[f"bert_{name}_gBias"])
    if "head_w" in P:
        _close(P["head_w"].grad, zb[f"bert_{name}_gHead"])


def test_bert4rec_bce_untied_matches_reference(golden_dir):
    _bert_case(golden_dir, "tiny", "untied")


def test_bert4rec_bce_tied_matches_reference(golden_dir):
    _bert_case(golden_dir, "tiny_tied", "tied")

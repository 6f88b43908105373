"""The GPU tests of the CE head (test_gpu_ce_pipeline.py, test_gpu_ce_head_fp64.py) choose their shapes from a restatement
of the kernel's tile table and split heuristic (tests/ce_reference.py); this checks that restatement against rp_ce_head.cu
without a GPU."""
import os
import re

import ce_reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "replay_b200", "csrc", "rp_ce_head.cu")


def test_tile_table_matches_dispatch():
    src = open(SRC).read()
    body = src[src.index("static int dispatch_ce_bwd("):]
    body = body[:body.index("default:")]
    table = {int(d): (int(tn), int(ns)) for d, _kch, ns, tn in
             re.findall(r"case (\d+):\s*return launch_ce_bwd<(\d+), (\d+), (\d+), MODE>", body)}
    assert table == ce_reference.TILE


def test_split_grid_and_heuristic_match_source():
    src = open(SRC).read()
    assert int(re.search(r"static constexpr int kTN = (\d+);", src).group(1)) == ce_reference.GRID
    ps = src[src.index("static int pick_splits("):]
    ps = ps[:ps.index("\n}\n")]
    assert "int max_splits = 8" in ps and "eff > best_eff + 0.02" in ps and "p <= n_col_tiles" in ps
    # the fused pass asks for splits over 128-item tiles of the catalog, with the row-tile hint
    assert "pick_splits(hint_tiles, n_item_tiles)" in src and "n_item_tiles = (n_items + kT - 1) / kT" in src

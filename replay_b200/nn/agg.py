"""Mirror of ``replay.nn.agg`` (config only: the fused embedding kernel sums the item embedding and the positions)."""
from __future__ import annotations


class SumAggregator:
    """replay/nn/agg.py: sums the embeddings of the sequence's features (here: the item id only)."""

    def __init__(self, embedding_dim: int) -> None:
        self.embedding_dim = embedding_dim

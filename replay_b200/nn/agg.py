"""Mirror of ``replay.nn.agg`` (config only: the fused embedding kernels sum or concatenate the feature embeddings)."""
from __future__ import annotations


class SumAggregator:
    """replay/nn/agg.py: sums the embeddings of the sequence's features (here: the item id only)."""

    def __init__(self, embedding_dim: int) -> None:
        self.embedding_dim = embedding_dim


class ConcatAggregator:
    """replay/nn/agg.py:56-109: concatenates the feature embeddings in ascending order of feature name and, with more than
    one input, projects them with ``feat_projection = Linear(sum(input_embedding_dims), output_embedding_dim)``.  A single
    input must already be ``output_embedding_dim`` wide."""

    def __init__(self, input_embedding_dims: list[int], output_embedding_dim: int) -> None:
        self.input_embedding_dims = list(input_embedding_dims)
        self._embedding_dim = output_embedding_dim
        concat_size = sum(self.input_embedding_dims)
        self.has_projection = len(self.input_embedding_dims) > 1
        if not self.has_projection and concat_size != output_embedding_dim:
            raise ValueError(f"Input embedding dim is not equal to embedding_dim ({concat_size} != {output_embedding_dim})")

    @property
    def embedding_dim(self) -> int:
        return self._embedding_dim

"""Mirror of ``replay.nn.ffn`` (config only): the item encoder of the TwoTower model runs as CUDA kernels
(replay_b200/engine_twotower.py)."""
from __future__ import annotations


class SwiGLUEncoder:
    """replay/nn/ffn.py:102-135: ``x = norm1(sw1(x) + x); x = norm2(sw2(x) + x)`` with SwiGLU feed-forward layers of width
    ``hidden_dim`` and torch.nn.RMSNorm(embedding_dim).  The CUDA path supports ``hidden_dim == 2 * embedding_dim``, the
    width TwoTower.from_params uses."""

    def __init__(self, embedding_dim: int, hidden_dim: int) -> None:
        self.embedding_dim, self.hidden_dim = embedding_dim, hidden_dim

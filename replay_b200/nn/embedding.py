"""Mirror of ``replay.nn.embedding`` (config only: the item table lives in the engine's flat parameter buffer)."""
from __future__ import annotations


class SequenceEmbedding:
    """replay/nn/embedding.py: one embedding per schema feature.  The CUDA path embeds the item id feature only; any other
    feature that is not excluded is rejected when the model is built."""

    def __init__(self, schema, excluded_features=None, categorical_list_feature_aggregation_method: str = "sum"):
        self.schema = schema
        self.excluded_features = list(excluded_features or [])
        self.categorical_list_feature_aggregation_method = categorical_list_feature_aggregation_method

"""Mirror of ``replay.nn.embedding`` (config only: the item table lives in the engine's flat parameter buffer)."""
from __future__ import annotations


class SequenceEmbedding:
    """replay/nn/embedding.py: one embedding per schema feature that is not in ``excluded_features``.  The CUDA path
    (csrc/rp_features.cu) embeds categorical features, categorical lists ("sum" / "mean") and numerical features next to
    the item id: at the model's width under SumAggregator, at their own widths under ConcatAggregator; the new-path SASRec
    body with SasRecTransformerLayer takes them."""

    def __init__(self, schema, excluded_features=None, categorical_list_feature_aggregation_method: str = "sum"):
        self.schema = schema
        self.excluded_features = list(excluded_features or [])
        self.categorical_list_feature_aggregation_method = categorical_list_feature_aggregation_method

from .sasrec import DiffTransformerLayer, PositionAwareAggregator, SasRec, SasRecBody, SasRecTransformerLayer  # noqa: F401

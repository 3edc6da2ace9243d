"""`de.keras.layers` (python/keras/layers/__init__.py:17-24)"""
from ..layers import AllToAllEmbedding, BasicEmbedding, Embedding, FieldWiseEmbedding, SparseEmbedding, SquashedEmbedding

HvdAllToAllEmbedding = AllToAllEmbedding  # python/keras/layers/embedding.py:545-595

__all__ = ["Embedding", "BasicEmbedding", "FieldWiseEmbedding", "SquashedEmbedding", "HvdAllToAllEmbedding",
           "AllToAllEmbedding", "SparseEmbedding"]

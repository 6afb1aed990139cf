"""Feature multiplexing (layers/feature_multiplexing/__init__.py): Unified Embedding."""
from . import unified_embedding
from .unified_embedding import UnifiedEmbedding, UnifiedEmbeddingConfig

__all__ = ["unified_embedding", "UnifiedEmbedding", "UnifiedEmbeddingConfig"]

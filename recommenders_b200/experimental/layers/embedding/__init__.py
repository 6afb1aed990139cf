"""Experimental embedding layers (tensorflow_recommenders/experimental/layers/embedding/__init__.py)."""
from .partial_tpu_embedding import PartialTPUEmbedding

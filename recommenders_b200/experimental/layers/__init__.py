"""Experimental layers (tensorflow_recommenders/experimental/layers/__init__.py)."""
from . import embedding

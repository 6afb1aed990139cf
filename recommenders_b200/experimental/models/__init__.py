"""Experimental models namespace (tensorflow_recommenders/experimental/models/__init__.py)."""
from .ranking import Ranking

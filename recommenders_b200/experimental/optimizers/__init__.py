"""Experimental optimizers (tensorflow_recommenders/experimental/optimizers/__init__.py)."""
from .clippy_adagrad import ClippyAdagrad, shrink_by_references
from .composite_optimizer import CompositeOptimizer

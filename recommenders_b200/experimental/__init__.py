"""Experimental namespace (tensorflow_recommenders/experimental/__init__.py): layers, the ranking model and the
optimizers."""
from . import layers
from . import models
from . import optimizers

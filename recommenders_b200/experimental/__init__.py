"""Experimental namespace (tensorflow_recommenders/experimental/__init__.py): the ranking model and the optimizers."""
from . import models
from . import optimizers

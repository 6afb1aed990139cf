"""Experimental namespace (tensorflow_recommenders/experimental/__init__.py): the ranking model."""
from . import models

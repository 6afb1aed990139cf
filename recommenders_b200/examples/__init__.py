"""Helpers of the reference's tutorials: mirror of tensorflow_recommenders/examples."""
from . import movielens

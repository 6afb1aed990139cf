"""recommenders_b200 -- an H100-native (sm_90a) implementation of the TensorFlow Recommenders retrieval /
ranking hot path behind the reference's own API surface:

    import recommenders_b200 as tfrs
    tfrs.Model, tfrs.tasks.Retrieval, tfrs.metrics.FactorizedTopK,
    tfrs.layers.factorized_top_k.{BruteForce, Streaming}, tfrs.layers.dcn.Cross,
    tfrs.layers.blocks.MLP, tfrs.tasks.Ranking, tfrs.experimental.models.Ranking, tfrs.losses,
    tfrs.examples.movielens.sample_listwise

(namespace per tensorflow_recommenders/__init__.py:51-61 and layers/__init__.py:18-23).  Tensors are CUDA
torch tensors; all arithmetic on the path runs in libtfrs_b200.so (include/tfrs_b200.h).  No CPU fallback.
"""
from . import backend
from . import data
from . import examples
from . import layers
from . import losses
from . import metrics
from . import models
from . import optimizers
from . import tasks
from . import experimental
from .models import Model

__version__ = "0.1.0"

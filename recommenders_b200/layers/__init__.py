"""Layers namespace, shaped like tensorflow_recommenders/layers/__init__.py:18-23."""
from . import attention
from . import blocks
from . import convolution
from . import embedding
from . import factorized_top_k
from . import feature_interaction
from . import loss
from . import normalization
from . import pooling
from . import preprocessing
from . import recurrent
from . import regularization
from .attention import AdditiveAttention, Attention, MultiHeadAttention
from .convolution import Conv1D
from .feature_interaction import dcn
from .normalization import BatchNormalization, LayerNormalization
from .pooling import GlobalAveragePooling1D
from .preprocessing import Discretization, Hashing, IntegerLookup, Normalization, StringLookup, TextVectorization
from .recurrent import GRU, LSTM
from .regularization import Dropout, SpatialDropout1D

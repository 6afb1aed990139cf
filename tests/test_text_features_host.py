"""Host-side tests of layers.TextVectorization, Discretization, Normalization, GlobalAveragePooling1D and Embedding's
mask_zero: argument errors, the index layout, config and extra-state round trips, the oracle (tests/text_oracle.py)
against every tf-keras docstring known answer, and the byte sets compiled into csrc/text.cu.  No GPU needed."""
import string

import numpy as np
import pytest
import torch

import recommenders_b200 as tfrs
import text_oracle as to
from recommenders_b200.layers.pooling import GlobalAveragePooling1D
from recommenders_b200.layers.preprocessing import Discretization, Normalization, StringLookup, TextVectorization


def test_exports():
  assert tfrs.layers.TextVectorization is TextVectorization and tfrs.layers.Discretization is Discretization
  assert tfrs.layers.Normalization is Normalization and tfrs.layers.GlobalAveragePooling1D is GlobalAveragePooling1D


def test_kernel_byte_sets_are_punctuation_and_ascii_whitespace():
  sets = to.kernel_byte_sets()
  assert sets["TX_PUNCT"] == string.punctuation.encode() and len(sets["TX_PUNCT"]) == 32
  assert sorted(sets["TX_SPACE"]) == sorted(b" \t\n\v\f\r")
  assert to.PUNCTUATION == sets["TX_PUNCT"] and sorted(to.WHITESPACE) == sorted(sets["TX_SPACE"])


def test_text_vectorization_errors():
  with pytest.raises(NotImplementedError):
    TextVectorization(standardize=lambda x: x)
  with pytest.raises(ValueError):
    TextVectorization(standardize="upper")
  for split in ("character", None, lambda x: x):
    with pytest.raises(NotImplementedError):
      TextVectorization(split=split)
  with pytest.raises(ValueError):
    TextVectorization(split="comma")
  with pytest.raises(NotImplementedError):
    TextVectorization(ngrams=2)
  for mode in ("multi_hot", "count", "tf_idf"):
    with pytest.raises(NotImplementedError):
      TextVectorization(output_mode=mode)
  with pytest.raises(ValueError):
    TextVectorization(output_mode="one_hot_ish")
  for osl in (0, -1, 2.5, True):
    with pytest.raises(ValueError):
      TextVectorization(output_sequence_length=osl)
  with pytest.raises(NotImplementedError):
    TextVectorization(ragged=True)
  with pytest.raises(NotImplementedError):
    TextVectorization(sparse=True)
  with pytest.raises(NotImplementedError):
    TextVectorization(pad_to_max_tokens=True)
  with pytest.raises(NotImplementedError):
    TextVectorization(idf_weights=[1.0])
  with pytest.raises(NotImplementedError):
    TextVectorization(encoding="latin-1")
  with pytest.raises(NotImplementedError):
    TextVectorization(vocabulary="vocab.txt")
  with pytest.raises(ValueError):
    TextVectorization(max_tokens=0)
  with pytest.raises(ValueError):
    TextVectorization(max_tokens=4, vocabulary=["a", "b", "c"])          # 2 + 3 indices
  with pytest.raises(NotImplementedError):
    TextVectorization()((np.array(["a"]), np.array([0, 1])))
  with pytest.raises(TypeError):
    TextVectorization()(torch.zeros(2))
  with pytest.raises(ValueError):
    TextVectorization()(np.array([["a", "b"]]))


def test_text_vectorization_index_layout_and_config():
  tv = TextVectorization(max_tokens=10, vocabulary=["earth", "wind"])
  assert tv.get_vocabulary() == ["", "[UNK]", "earth", "wind"]
  assert tv.get_vocabulary(include_special_tokens=False) == ["earth", "wind"]
  assert tv.vocabulary_size() == 4
  cfg = tv.get_config()
  assert cfg["vocabulary"] == ["earth", "wind"] and cfg["max_tokens"] == 10 and cfg["output_mode"] == "int"
  tv2 = TextVectorization.from_config(cfg)
  assert tv2.get_config() == cfg and tv2.get_vocabulary() == tv.get_vocabulary()
  # the inner lookup is K15's StringLookup with Keras's text settings, and its extra state travels in the state_dict
  lk = tv._lookup_layer
  assert isinstance(lk, StringLookup) and lk.mask_token == "" and lk.oov_token == "[UNK]" and lk.num_oov_indices == 1
  sd = tv.state_dict()
  assert sd["_lookup_layer._extra_state"]["vocabulary"] == ["earth", "wind"]
  tv3 = TextVectorization()
  tv3.load_state_dict(sd)
  assert tv3.get_vocabulary() == tv.get_vocabulary()


def test_oracle_known_answers():
  k = to.KNOWN_ADAPT
  vocab = to.adapt_vocabulary(k["adapt"], k["max_tokens"])
  assert vocab == [b"foo", b"baz", b"bar"]
  assert to.vectorize([s[0] for s in k["inputs"]], vocab, k["output_sequence_length"]).tolist() == k["expected"]
  k = to.KNOWN_VOCAB
  assert to.vectorize([s[0] for s in k["inputs"]], k["vocabulary"]).tolist() == k["expected"]
  k = to.KNOWN_NORMALIZATION
  mean, var = to.adapt_moments(to.array_batches(np.array(k["adapt"], np.float32)), 1)
  assert mean.tolist() == [k["mean"]] and var.tolist() == [k["variance"]]
  assert to.normalize(np.array(k["inputs"]), mean[0], var[0]).tolist() == np.float32(k["expected"]).tolist()
  assert to.normalize(np.array(k["inputs"]), k["mean"], k["variance"]).tolist() == np.float32(k["expected"]).tolist()


def test_oracle_rules():
  assert to.tokens("Don't") == [b"dont"] and to.tokens("a.b") == [b"ab"] and to.tokens("a - b") == [b"a", b"b"]
  # ASCII-only lowercase; look-alike separators do not split
  assert to.tokens("ÉCOLE CafÉ") == ["École".encode(), "cafÉ".encode()]
  for sep in ("\x1c", "\x1d", "\x1e", "\x1f", " ", "　", "\u0085"):
    assert to.tokens(f"a{sep}b") == [f"a{sep}b".encode()]
  for sep in " \t\n\v\f\r":
    assert to.tokens(f"a{sep}{sep}b{sep}") == [b"a", b"b"]
  assert to.tokens("!!! ... ???") == [] and to.tokens("") == []
  assert to.tokens("A.B", lower=False) == [b"AB"] and to.tokens("A.B", strip=False) == [b"a.b"]
  # vocabulary entries are not standardized: an upper-case entry never matches
  assert to.vectorize(["Earth earth"], ["Earth", "earth"]).tolist() == [[3, 3]]
  # adapt: count descending, ties by token descending
  assert to.adapt_vocabulary(["b a c a", "c"]) == [b"c", b"a", b"b"]
  assert to.adapt_vocabulary(["b a c a", "c"], max_tokens=3) == [b"c"]
  # Discretization: the float32 rounding of int64 timestamps is visible
  b = [978300760.0 + 64.0 * 0.5]                    # rounds to a float32 with a 64-second ulp
  b32 = float(np.float32(b[0]))
  x = np.array([int(b32) - 1, int(b32), int(b32) + 31, int(b32) + 32, int(b32) + 33], np.int64)
  assert to.bucketize(x, b).tolist() == [int(np.float32(v) >= np.float32(b32)) for v in x]
  assert to.bucketize(np.array([np.nan, -np.inf, np.inf]), [0.0, 1.0]).tolist() == [2, 0, 2]
  assert to.bucketize(np.array([1.0, 2.0]), [1.0, 1.0, 2.0]).tolist() == [2, 3]
  assert to.bucketize(np.array([5], np.int64), []).tolist() == [0]
  # pooling: all-masked rows are 0/0, Inf at a masked position propagates through x * 0
  x = np.ones((2, 3, 2), np.float32)
  x[1, 2] = np.inf
  got = to.pool(x, np.array([[0, 0, 0], [1, 1, 0]]))
  assert np.isnan(got[0]).all() and np.isnan(got[1]).all()
  assert to.pool(x[:1], np.array([[1, 0, 1]])).tolist() == [[1.0, 1.0]]
  assert to.pool_grad(np.array([[3.0, 6.0]]), np.array([[1, 0, 1]]), 3).tolist() == [[[1.5, 3.0], [0, 0], [1.5, 3.0]]]


def test_discretization_errors_and_config():
  with pytest.raises(NotImplementedError):
    Discretization(num_bins=4)
  with pytest.raises(ValueError):
    Discretization(bin_boundaries=[0.0], num_bins=4)
  with pytest.raises(NotImplementedError):
    Discretization(bin_boundaries=[0.0], epsilon=0.1)
  with pytest.raises(NotImplementedError):
    Discretization()
  with pytest.raises(NotImplementedError):
    Discretization(bin_boundaries=[0.0]).adapt(np.zeros(3))
  for mode in ("one_hot", "multi_hot", "count"):
    with pytest.raises(NotImplementedError):
      Discretization(bin_boundaries=[0.0], output_mode=mode)
  with pytest.raises(ValueError):
    Discretization(bin_boundaries=[0.0], output_mode="bogus")
  with pytest.raises(NotImplementedError):
    Discretization(bin_boundaries=[0.0], sparse=True)
  with pytest.raises(ValueError):
    Discretization(bin_boundaries=[1.0, 0.0])
  with pytest.raises(ValueError):
    Discretization(bin_boundaries=[0.0, float("nan")])
  # the order is checked after rounding to float32: these two are equal there
  assert Discretization(bin_boundaries=[1.0 + 2 ** -30, 1.0])._b32.tolist() == [1.0, 1.0]
  d = Discretization(bin_boundaries=[0.5, 1.5], name="d")
  assert Discretization.from_config(d.get_config()).get_config() == d.get_config()
  with pytest.raises(TypeError):
    d(np.array(["a"]))


def test_normalization_errors_and_config():
  for axis in (0, 1, (0, 1), -2):
    with pytest.raises(NotImplementedError):
      Normalization(axis=axis)
  Normalization(axis=[-1])
  with pytest.raises(ValueError):
    Normalization(mean=1.0)
  with pytest.raises(ValueError):
    Normalization(variance=1.0)
  with pytest.raises(ValueError):
    Normalization(axis=None, mean=[1.0, 2.0], variance=[1.0, 1.0])
  with pytest.raises(ValueError):
    Normalization(mean=1.0, variance=2.0).adapt(np.zeros(3))
  n = Normalization(axis=None, mean=3.0, variance=2.0, invert=True, name="n")
  assert Normalization.from_config(n.get_config()).get_config() == n.get_config()
  with pytest.raises(NotImplementedError):
    n(torch.zeros(3, requires_grad=True))
  with pytest.raises(NotImplementedError):
    Normalization(axis=-1).adapt(np.zeros(5))               # axis=-1 needs rank >= 2
  assert Normalization().get_extra_state() == {}


def test_pooling_and_embedding_mask_errors():
  with pytest.raises(NotImplementedError):
    GlobalAveragePooling1D(data_format="channels_first")
  with pytest.raises(ValueError):
    GlobalAveragePooling1D(data_format="nhwc")
  p = GlobalAveragePooling1D(keepdims=True)
  assert GlobalAveragePooling1D.from_config(p.get_config()).keepdims
  from recommenders_b200 import ops
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.mean_pool(torch.zeros(2, 3, 4))
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.bucketize(torch.zeros(3), torch.zeros(2))
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.normalize(torch.zeros(3), torch.zeros(1), torch.ones(1))
  t = torch.zeros(2, 3, 4)
  assert ops.attached_mask(t) is None

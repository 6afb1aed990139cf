"""CPU tests of tf-keras `Hashing` (K18): the oracle against the published examples, constructor errors, the config round
trip and the export.  Nothing here needs a GPU."""
import numpy as np
import pytest

import hashing_oracle as ho

ABCDE = ["A", "B", "C", "D", "E"]


def test_doc_examples_on_the_oracle():
  # tf.keras.layers.Hashing and tf.strings.to_hash_bucket_fast API documentation
  assert ho.hashing(ABCDE, 3).tolist() == [1, 0, 1, 1, 2]
  assert ho.hashing(["A", "B", "", "C", "D"], 3, mask="").tolist() == [1, 1, 0, 2, 2]
  assert ho.hashing(["Hello", "TensorFlow", "2.x"], 3).tolist() == [0, 2, 2]
  assert ho.hashing(ABCDE, 3, salt=133).tolist() == [0, 0, 2, 1, 0]
  assert ho.hashing(ABCDE, 3, salt=[133, 137]).tolist() == [1, 2, 1, 0, 2]


def test_fingerprint64_known_answers():
  assert ho.fingerprint64(b"") == 0x9ae16a3b2f90404f          # the empty-input branch returns k2
  # TensorFlow's fingerprint_test.cc (Fingerprint64 "IsForeverFrozen")
  assert ho.fingerprint64(b"Hello") == 15404698994557526151
  assert ho.fingerprint64(b"World") == 18308117990299812472


def test_oracle_integers_hash_as_their_text():
  v = np.array([0, -1, 7, 10**18, -2**63, 2**63 - 1], np.int64)
  for salt in (None, 5):
    assert ho.hashing(v, 1000, salt).tolist() == ho.hashing([str(x) for x in v.tolist()], 1000, salt).tolist()
  # num_bins == 1 reserves nothing, even with a mask
  assert ho.hashing(v, 1, mask=0).tolist() == [0] * 6
  assert ho.hashing(v, 2, mask=-1).tolist()[1] == 0 and set(ho.hashing(v, 2, mask=-1).tolist()) <= {0, 1}


def _layer_cls():
  from recommenders_b200.layers.preprocessing import Hashing
  return Hashing


def test_export():
  import recommenders_b200 as tfrs
  from recommenders_b200.layers import preprocessing
  assert tfrs.layers.Hashing is preprocessing.Hashing


@pytest.mark.parametrize("kw,err", [
    (dict(num_bins=None), ValueError),
    (dict(num_bins=0), ValueError),
    (dict(num_bins=-3), ValueError),
    (dict(num_bins=2.5), ValueError),
    (dict(num_bins=2**63), ValueError),
    (dict(num_bins=3, salt=[1, 2, 3]), ValueError),
    (dict(num_bins=3, salt="x"), ValueError),
    (dict(num_bins=3, salt=1.5), ValueError),
    (dict(num_bins=3, salt=[1, "a"]), ValueError),
    (dict(num_bins=3, salt=[2**64, 0]), ValueError),
    (dict(num_bins=3, mask_value=1.5), ValueError),
    (dict(num_bins=3, output_mode="one_hot"), NotImplementedError),
    (dict(num_bins=3, output_mode="multi_hot"), NotImplementedError),
    (dict(num_bins=3, output_mode="count"), NotImplementedError),
    (dict(num_bins=3, output_mode="bogus"), ValueError),
    (dict(num_bins=3, sparse=True), NotImplementedError),
])
def test_constructor_errors(kw, err):
  with pytest.raises(err):
    _layer_cls()(**kw)


def test_cpu_and_float_inputs_raise_type_error():
  import torch
  layer = _layer_cls()(num_bins=3)
  with pytest.raises(TypeError):
    layer(torch.arange(4))                         # a CPU tensor: there is no CPU path
  with pytest.raises(TypeError):
    layer(np.array([0.5, 1.5]))
  with pytest.raises(NotImplementedError):
    layer((np.array([1, 2]), np.array([0, 2])))    # ragged


@pytest.mark.parametrize("kw", [
    dict(num_bins=3),
    dict(num_bins=200_000, salt=133),
    dict(num_bins=7, salt=(133, 137), mask_value="", name="h"),
    dict(num_bins=2**63 - 1, mask_value=-1),
    dict(num_bins=1, mask_value=b"x"),
])
def test_config_round_trip(kw):
  H = _layer_cls()
  layer = H(**kw)
  cfg = layer.get_config()
  assert cfg["num_bins"] == kw["num_bins"] and cfg["output_mode"] == "int" and cfg["sparse"] is False
  salt = kw.get("salt")
  assert cfg["salt"] == (None if salt is None else ([salt, salt] if isinstance(salt, int) else list(salt)))
  again = H.from_config(cfg)
  assert again.get_config() == cfg

"""CPU tests of TPUEmbedding: the oracle against the hand-computed answers of the reference's fixture
(layers/embedding/tpu_embedding_layer_test.py:51-111), and the config plumbing of TPUEmbedding, PartialTPUEmbedding and
SGD (tables built on the CPU; nothing here launches a kernel)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import embedding_bag_oracle as ebo  # noqa: E402

from recommenders_b200 import optimizers  # noqa: E402
from recommenders_b200.experimental.layers.embedding import PartialTPUEmbedding  # noqa: E402
from recommenders_b200.layers.embedding import Embedding, FeatureConfig, TableConfig, TPUEmbedding  # noqa: E402

CPU = torch.device("cpu")
VIDEO = np.arange(8, dtype=np.float32).reshape(2, 4)     # 0 1 2 3 / 4 5 6 7
USER = np.arange(8, dtype=np.float32).reshape(4, 2)      # 0 1 / 2 3 / 4 5 / 6 7
WATCHED = (np.array([0, 0, 1, 0, 1, 1]), np.array([0, 1, 3, 5, 6]))
FAVORITED = (np.array([0, 1, 1, 0, 0, 1]), np.array([0, 2, 3, 4, 6]))
FRIENDS = (np.array([3, 0, 1, 2, 3, 0, 1, 2]), np.array([0, 1, 4, 5, 8]))


def test_oracle_reference_fixture():
  w, _ = ebo.lookup(VIDEO, *WATCHED, combiner="sum")
  np.testing.assert_array_equal(w, [[0, 1, 2, 3], [4, 6, 8, 10], [4, 6, 8, 10], [4, 5, 6, 7]])
  f, _ = ebo.lookup(VIDEO, *FAVORITED, combiner="sum")
  np.testing.assert_array_equal(f, [[4, 6, 8, 10], [4, 5, 6, 7], [0, 1, 2, 3], [4, 6, 8, 10]])
  fr, den = ebo.lookup(USER, *FRIENDS, combiner="mean")
  np.testing.assert_array_equal(fr, [[6, 7], [2, 3], [6, 7], [2, 3]])
  np.testing.assert_array_equal(den, [1, 3, 1, 3])


def test_oracle_combiners_weights_and_dropped_ids():
  table = np.arange(12, dtype=np.float32).reshape(3, 4)
  vals, sp = np.array([0, 2, 7, -1, 1]), np.array([0, 3, 3, 5])
  w = np.array([2, 0.5, 9, 9, 3], np.float32)
  s, _ = ebo.lookup(table, vals, sp, w, "sum")
  np.testing.assert_array_equal(s, [2 * table[0] + 0.5 * table[2], np.zeros(4), 3 * table[1]])
  m, den = ebo.lookup(table, vals, sp, w, "mean")
  np.testing.assert_array_equal(den[[0, 2]], [2.5, 3])
  np.testing.assert_array_equal(m[0], (2 * table[0] + 0.5 * table[2]) / np.float32(2.5))
  np.testing.assert_array_equal(m[1], np.zeros(4))
  q, den = ebo.lookup(table, vals, sp, w, "sqrtn")
  np.testing.assert_array_equal(den[0], np.sqrt(np.float32(4.25)))
  g = np.arange(12, dtype=np.float32).reshape(3, 4)
  r = ebo.lookup_bwd(table.shape, vals, g, sp, w, "mean")
  np.testing.assert_array_equal(r[0], g[0] * np.float32(2) / np.float32(2.5))
  np.testing.assert_array_equal(r[2:4], np.zeros((2, 4)))   # dropped ids
  np.testing.assert_array_equal(r[4], g[2] * np.float32(3) / np.float32(3))


def test_oracle_sequence_and_dense():
  table = np.arange(8, dtype=np.float32).reshape(4, 2)
  vals, sp = np.array([1, 2, 3, 0, 9]), np.array([0, 3, 3, 5])
  out, _ = ebo.lookup(table, vals, sp, None, "mean", max_sequence_length=2)
  np.testing.assert_array_equal(out, [[table[1], table[2]], [[0, 0], [0, 0]], [table[0], [0, 0]]])
  g = np.arange(12, dtype=np.float32).reshape(3, 2, 2)
  r = ebo.lookup_bwd(table.shape, vals, g, sp, None, "mean", max_sequence_length=2)
  np.testing.assert_array_equal(r, [g[0, 0], g[0, 1], [0, 0], g[2, 0], [0, 0]])
  d, _ = ebo.lookup(table, np.array([[1, 5], [3, 0]]))
  np.testing.assert_array_equal(d, [[table[1], [0, 0]], [table[3], table[0]]])


def test_oracle_sgd():
  t = np.ones((3, 2), np.float32)
  out = ebo.sgd_sparse(t, [2, 0, 2, 7], np.array([[1, 2], [3, 4], [5, 6], [7, 8]], np.float32), 0.5)
  np.testing.assert_array_equal(out, [[-0.5, -1], [1, 1], [1 - 0.5 - 2.5, 1 - 1 - 3]])


def _config():
  video = TableConfig(2, 4, initializer="zeros", combiner="sum", name="video")
  user = TableConfig(4, 2, initializer="zeros", name="user")
  return video, user, {"watched": FeatureConfig(video, name="watched"), "favorited": FeatureConfig(video),
                       "friends": FeatureConfig(user)}


def test_shared_tables_by_identity_and_nesting():
  video, user, fc = _config()
  layer = TPUEmbedding(fc, optimizer=None, device=CPU)
  assert len(layer._tables) == 2 and set(layer.embedding_tables) == {video, user}
  assert all(isinstance(t, Embedding) for t in layer.embedding_tables.values())
  assert len(optimizers.embedding_tables(layer)) == 2
  # an equal but distinct TableConfig is a table of its own
  other = TableConfig(2, 4, initializer="zeros", combiner="sum")
  layer2 = TPUEmbedding([FeatureConfig(video), (FeatureConfig(other), {"a": FeatureConfig(video)})], device=CPU)
  assert len(layer2._tables) == 2 and layer2._table_of == [0, 1, 0]


def test_default_initializer_is_truncated_normal():
  t = TPUEmbedding({"a": FeatureConfig(TableConfig(1000, 16))}, device=CPU)._tables[0].weight
  assert float(t.abs().max()) <= 2.0 / 4.0 and abs(float(t.std()) - 0.25) < 0.05


def test_config_errors():
  with pytest.raises(NotImplementedError):
    FeatureConfig(TableConfig(2, 4), output_shape=[3])
  with pytest.raises(NotImplementedError):
    TableConfig(2, 4, quantization_config=object())
  with pytest.raises(ValueError):
    TableConfig(2, 4, combiner="max")
  with pytest.raises(ValueError):
    TPUEmbedding({"a": TableConfig(2, 4)}, device=CPU)
  with pytest.raises(NotImplementedError):
    TPUEmbedding({"a": FeatureConfig(TableConfig(2, 4))}, device=CPU).serving_config
  with pytest.raises(NotImplementedError):
    optimizers.SGD(0.1, momentum=0.9)
  with pytest.raises(NotImplementedError):
    optimizers.SGD(0.1, nesterov=True)
  assert optimizers.SGD.from_config(optimizers.SGD(0.25).get_config()).learning_rate == 0.25


def test_dense_weights_raise():
  layer = TPUEmbedding({"a": FeatureConfig(TableConfig(2, 4))}, device=CPU)
  with pytest.raises(ValueError, match="weights"):
    layer({"a": torch.zeros(3, dtype=torch.int64)}, weights={"a": torch.ones(3)})


@pytest.mark.parametrize("threshold, keras, tpu", [(None, {"small", "large"}, set()), (0, set(), {"small", "large"}),
                                                   (-1, set(), {"small", "large"}), (20, {"small"}, {"large"})])
def test_partial_routing(threshold, keras, tpu):
  small, large = TableConfig(10, 4), TableConfig(100, 4)
  fc = {"small": FeatureConfig(small), "small2": FeatureConfig(small), "large": FeatureConfig(large)}
  layer = PartialTPUEmbedding(fc, None, size_threshold=threshold, device=CPU)
  k = set(layer.keras_embedding_layers)
  if "small" in keras:
    keras = keras | {"small2"}
  else:
    tpu = tpu | {"small2"}
  assert k == keras
  if tpu:
    assert set(layer.tpu_embedding._feature_config) == tpu
  else:
    assert layer.tpu_embedding is None
  if "small" in keras:
    assert layer.keras_embedding_layers["small"] is layer.keras_embedding_layers["small2"]
  assert len(optimizers.embedding_tables(layer)) == len({id(f.table) for f in fc.values()})


def test_partial_keras_tables_take_dense_inputs_only():
  layer = PartialTPUEmbedding({"a": FeatureConfig(TableConfig(10, 4))}, None, size_threshold=None, device=CPU)
  with pytest.raises(ValueError, match="Only dense"):
    layer({"a": (torch.zeros(2, dtype=torch.int64), np.array([0, 1, 2]))})

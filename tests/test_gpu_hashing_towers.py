"""End to end on the H100: the uet tutorial's HashEmbeddingModel (`Sequential([Hashing(num_bins=buckets),
Embedding(buckets, d)])` per feature, Concatenate, MLP, `tasks.Ranking`) trained with Adam on seeded synthetic string
features, against the same model fed ids hashed on the host by the C oracle; and the featurization tutorial's title
cell, `Hashing(num_bins=200_000)` -> `Embedding`."""
import numpy as np
import pytest
import torch

import hashing_oracle as ho
import recommenders_b200 as tfrs
from recommenders_b200.layers.embedding import Embedding

pytestmark = pytest.mark.gpu

# the bucket dict the uet tutorial evaluates HashEmbeddingModel with
BUCKETS = {"movie_id": 600, "user_id": 400, "user_gender": 20, "user_zip_code": 400, "user_occupation_text": 20}
DIM = 16


class _OracleHashing(torch.nn.Module):
  """What the model computes without a device Hashing layer: the oracle's bins on the host, then one upload."""

  def __init__(self, num_bins):
    super().__init__()
    self.num_bins = num_bins

  def forward(self, x):
    return torch.from_numpy(ho.hashing(x, self.num_bins)).cuda()


class _HashEmbeddingModel(tfrs.models.Model):
  def __init__(self, hashing):
    super().__init__()
    self.towers = torch.nn.ModuleDict({f: torch.nn.Sequential(hashing(b), Embedding(b, DIM)) for f, b in BUCKETS.items()})
    self.network = tfrs.layers.blocks.MLP([64, 32, 1], final_activation="sigmoid")
    self.task = tfrs.tasks.Ranking(metrics=[tfrs.metrics.AUC(name="AUC")])

  def compute_loss(self, inputs, training=False):
    feats, labels = inputs
    x = torch.cat([self.towers[f](feats[f]) for f in BUCKETS], -1)
    return self.task(labels, self.network(x))


def _data(steps=8, batch=512):
  rng = np.random.default_rng(11)
  occupations = np.array(["doctor", "artist", "student", "other", "lawyer", "K-12 student", "retired"])
  out = []
  for _ in range(steps):
    uid, mid = rng.integers(0, 943, size=batch), rng.integers(0, 1682, size=batch)
    feats = {"movie_id": np.char.mod("%d", mid), "user_id": np.char.mod("%d", uid),
             "user_gender": np.where(uid % 2 == 0, "True", "False"),
             "user_zip_code": np.char.mod("%05d", uid * 37 % 100000),
             "user_occupation_text": occupations[uid % len(occupations)]}
    labels = torch.from_numpy(((uid * 7 + mid) % 3 == 0).astype(np.float32)).cuda().reshape(-1, 1)
    out.append((feats, labels))
  return out


def _bits(t):
  return t.detach().cpu().numpy().view(np.uint32)


def test_hash_embedding_model_matches_host_hashed_ids():
  data = _data()
  torch.manual_seed(0)
  dev_model = _HashEmbeddingModel(lambda b: tfrs.layers.Hashing(num_bins=b))
  host_model = _HashEmbeddingModel(_OracleHashing)
  with torch.no_grad():                          # builds the MLP's weights, then one set of weights for both
    dev_model.compute_loss(data[0]); host_model.compute_loss(data[0])
  host_model.load_state_dict(dev_model.state_dict())
  for f, b in BUCKETS.items():                   # the device bins are the oracle's
    got = dev_model.towers[f][0](data[0][0][f]).cpu().numpy()
    np.testing.assert_array_equal(got, ho.hashing(data[0][0][f], b))
  w0 = dev_model.towers["movie_id"][1].weight.detach().clone()
  dev_model.compile(optimizer=tfrs.optimizers.Adam(0.01))
  host_model.compile(optimizer=tfrs.optimizers.Adam(0.01))
  la = [float(dev_model.train_step(b)["loss"]) for b in data]
  lb = [float(host_model.train_step(b)["loss"]) for b in data]
  assert la == lb and np.isfinite(la).all()
  sa, sb = dev_model.state_dict(), host_model.state_dict()
  assert sa.keys() == sb.keys() and any(k.endswith("weight") for k in sa)
  for k in sa:
    if sa[k].dtype == torch.float32:
      np.testing.assert_array_equal(_bits(sa[k]), _bits(sb[k]), err_msg=k)
    else:
      assert torch.equal(sa[k], sb[k]), k
  assert not torch.equal(dev_model.towers["movie_id"][1].weight, w0)          # the tables trained


def test_featurization_title_cell():
  rng = np.random.default_rng(3)
  titles = np.array([f"Movie {i}: {'The ' if i % 3 else ''}Story of {'x' * (i % 60)} ({1950 + i % 70})"
                     for i in rng.integers(0, 100_000, size=2048)])
  torch.manual_seed(1)
  hashing = tfrs.layers.Hashing(num_bins=200_000)
  emb = Embedding(200_000, 32)
  with torch.no_grad():
    got = emb(hashing(titles))
  bins = ho.hashing(titles, 200_000)
  assert got.shape == (2048, 32)
  np.testing.assert_array_equal(_bits(got), _bits(emb.weight[torch.from_numpy(bins).cuda()]))

"""End to end on the H100: the quickstart tutorial's towers, `Sequential(StringLookup, Embedding)`, on a seeded synthetic
dataset of string user and movie ids.  Training runs, and retrieval and evaluation give what the same towers give when
the ids are mapped on the host with a dict."""
import numpy as np
import pytest
import torch

import recommenders_b200 as tfrs
from recommenders_b200.data import Dataset
from recommenders_b200.examples import movielens
from recommenders_b200.layers.embedding import Embedding

pytestmark = pytest.mark.gpu


def _data(seed=0, users=300, movies=500, rows=6000):
  rng = np.random.RandomState(seed)
  user_ids = np.array([f"{i}" for i in rng.permutation(users)])
  titles = np.array([f"Movie {i} ({1950 + i % 70})" for i in range(movies)])
  u = user_ids[rng.randint(0, users, size=rows)]
  m = titles[(rng.zipf(1.3, size=rows) - 1) % movies]
  return user_ids, titles, u, m


class _HostMapped(torch.nn.Module):
  """What a user writes without a lookup layer: a dict from id to index (0 for an unknown id), then the upload."""

  def __init__(self, vocab, emb):
    super().__init__()
    self.map = {v: i + 1 for i, v in enumerate(vocab.tolist())}
    self.emb = emb

  def forward(self, x):
    ids = np.array([self.map.get(v, 0) for v in np.asarray(x).reshape(-1).tolist()], np.int64)
    return self.emb(torch.from_numpy(ids).cuda()).reshape(*np.shape(x), -1)


class _Model(tfrs.Model):
  def __init__(self, user_model, movie_model):
    super().__init__()
    self.user_model, self.movie_model = user_model, movie_model
    self.task = tfrs.tasks.Retrieval()

  def compute_loss(self, features, training=False):
    return self.task(self.user_model(features["user_id"]), self.movie_model(features["movie_title"]),
                     compute_metrics=False)


def _towers(user_ids, titles, dim=32):
  torch.manual_seed(0)
  user_model = torch.nn.Sequential(tfrs.layers.StringLookup(vocabulary=user_ids, mask_token=None),
                                   Embedding(len(user_ids) + 1, dim))
  movie_model = torch.nn.Sequential(tfrs.layers.StringLookup(vocabulary=titles, mask_token=None),
                                    Embedding(len(titles) + 1, dim))
  return user_model, movie_model


def test_fit_retrieve_and_evaluate_match_host_mapped_towers():
  user_ids, titles, u, m = _data()
  user_model, movie_model = _towers(user_ids, titles)
  model = _Model(user_model, movie_model)
  model.compile(optimizer=tfrs.optimizers.Adagrad(0.5))
  before = movie_model[1].weight.clone()
  ratings = Dataset.from_tensor_slices({"user_id": u, "movie_title": m}).batch(512)
  hist = model.fit(ratings, epochs=1)
  assert np.isfinite(float(hist[-1]["loss"])) and not torch.equal(before, movie_model[1].weight)

  host_user = _HostMapped(user_ids, user_model[1])
  host_movie = _HostMapped(titles, movie_model[1])
  movies = Dataset.from_tensor_slices(titles)
  queries = np.concatenate([user_ids[:50], ["nobody", "0x"]])    # two unknown users go to the OOV row
  with torch.no_grad():
    a = tfrs.layers.factorized_top_k.BruteForce(user_model)
    a.index_from_dataset(movies.batch(100).map(lambda t: (t, movie_model(t))))
    sa, ta = a(queries)
    b = tfrs.layers.factorized_top_k.BruteForce(host_user)
    b.index_from_dataset(movies.batch(100).map(lambda t: (t, host_movie(t))))
    sb, tb = b(queries)
  assert isinstance(ta, np.ndarray) and ta.shape == (len(queries), 10)
  assert np.array_equal(ta, tb) and torch.equal(sa, sb)

  # examples.movielens.evaluate with the lookup towers and with the host-mapped ones
  rng = np.random.RandomState(1)
  split = rng.rand(len(u)) < 0.8
  train = Dataset.from_tensor_slices({"user_id": u[split], "movie_id": m[split]}).batch(1000)
  test = Dataset.from_tensor_slices({"user_id": u[~split], "movie_id": m[~split]}).batch(1000)
  mv = Dataset.from_tensor_slices({"movie_id": titles}).batch(128)
  got = movielens.evaluate(lambda f: user_model(f["user_id"]), lambda f: movie_model(f["movie_id"]), test, mv, train,
                           k=10)
  exp = movielens.evaluate(lambda f: host_user(f["user_id"]), lambda f: host_movie(f["movie_id"]), test, mv, train,
                           k=10)
  assert got == exp and got["recall_at_k"] > 0

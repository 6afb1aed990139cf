"""End to end on the H100: the deep_recommenders / context_features towers -- user id, bucketized and normalized
timestamps, movie title id and title text -- on a seeded synthetic ratings set, trained for one epoch with Adagrad.
Towers fed by the device preprocessing layers and identical towers fed by the host oracle (tests/text_oracle.py) give
the same per-step losses, final tables, BruteForce results and examples.movielens.evaluate results."""
import copy

import numpy as np
import pytest
import torch

import recommenders_b200 as tfrs
import text_oracle as to
from recommenders_b200.data import Dataset
from recommenders_b200.examples import movielens
from recommenders_b200.layers.blocks import Dense
from recommenders_b200.layers.embedding import Embedding
from recommenders_b200.layers.pooling import GlobalAveragePooling1D

pytestmark = pytest.mark.gpu

WORDS = ["the", "Love", "war", "Night", "of", "Story", "man", "city", "Dark", "dream", "II", "a", "l'amour", "re-run"]


def _data(seed=0, users=200, movies=400, rows=5000):
  rng = np.random.RandomState(seed)
  user_ids = np.array([f"{i}" for i in rng.permutation(users)])
  titles = np.array([" ".join(rng.choice(WORDS, rng.randint(1, 5))).title() + f": Part {i} ({1950 + i % 70})"
                     for i in range(movies)])
  u = user_ids[rng.randint(0, users, size=rows)]
  m = titles[(rng.zipf(1.3, size=rows) - 1) % movies]
  ts = np.sort(rng.randint(874724710, 893286638, size=rows)).astype(np.int64)
  return user_ids, titles, u, m, ts


class _Learned(torch.nn.Module):
  """The trained parts, shared in structure by both models."""

  def __init__(self, n_users, n_buckets, n_titles, dim=32):
    super().__init__()
    self.user = Embedding(n_users + 1, dim)
    self.ts = Embedding(n_buckets + 1, dim)
    self.title = Embedding(n_titles + 1, dim)
    self.text = Embedding(10_000, dim, mask_zero=True)
    self.pool = GlobalAveragePooling1D()
    self.q = Dense(32)
    self.c = Dense(32)

  def query(self, user_ids, buckets, normalized):
    return self.q(torch.cat([self.user(user_ids), self.ts(buckets), normalized.reshape(-1, 1)], dim=1))

  def candidate(self, title_ids, tokens, mask=None):
    return self.c(torch.cat([self.title(title_ids), self.pool(self.text(tokens), mask=mask)], dim=1))


class _Device(torch.nn.Module):
  """The tutorial's preprocessing layers, on the device."""

  def __init__(self, user_ids, titles, buckets, ts):
    super().__init__()
    L = tfrs.layers
    self.user_lookup = L.StringLookup(vocabulary=user_ids, mask_token=None)
    self.discretize = L.Discretization(buckets.tolist())
    self.normalize = L.Normalization(axis=None)
    self.normalize.adapt(ts)
    self.title_lookup = L.StringLookup(vocabulary=titles, mask_token=None)
    self.vectorize = L.TextVectorization(max_tokens=10_000)
    self.vectorize.adapt(Dataset.from_tensor_slices(titles))

  def query(self, learned, u, t):
    return learned.query(self.user_lookup(u), self.discretize(t), self.normalize(t))

  def candidate(self, learned, m):
    return learned.candidate(self.title_lookup(m), self.vectorize(m))      # the mask rides on the embedding output


class _Host:
  """The same preprocessing restated on the host by the oracle, uploaded as ids and floats."""

  def __init__(self, user_ids, titles, buckets, ts):
    self.users = {v: i + 1 for i, v in enumerate(user_ids.tolist())}
    self.titles = {v: i + 1 for i, v in enumerate(titles.tolist())}
    self.buckets = buckets
    self.mean, self.var = to.adapt_moments(to.array_batches(ts, 32), 1)
    self.vocab = to.adapt_vocabulary(titles.tolist(), 10_000)

  @staticmethod
  def _up(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()

  def query(self, learned, u, t):
    ids = np.array([self.users.get(v, 0) for v in np.asarray(u).tolist()], np.int64)
    t = np.asarray(t)
    return learned.query(self._up(ids), self._up(to.bucketize(t, self.buckets)),
                         self._up(to.normalize(t, self.mean[0], self.var[0])))

  def candidate(self, learned, m):
    ids = np.array([self.titles.get(v, 0) for v in np.asarray(m).tolist()], np.int64)
    tokens = self._up(to.vectorize(np.asarray(m).tolist(), self.vocab))
    return learned.candidate(self._up(ids), tokens, mask=tokens)


class _Model(tfrs.Model):

  def __init__(self, prep, learned):
    super().__init__()
    self.prep, self.learned = prep, learned
    self.task = tfrs.tasks.Retrieval()

  def compute_loss(self, features, training=False):
    q = self.prep.query(self.learned, features["user_id"], features["timestamp"])
    return self.task(q, self.prep.candidate(self.learned, features["movie_title"]), compute_metrics=False)


def test_deep_recommenders_towers_match_host_preprocessed_towers():
  user_ids, titles, u, m, ts = _data()
  buckets = np.linspace(ts.min(), ts.max(), num=1000)
  dev = _Device(user_ids, titles, buckets, ts)
  host = _Host(user_ids, titles, buckets, ts)
  assert dev.vectorize.get_vocabulary(include_special_tokens=False) == [t.decode() for t in host.vocab]

  torch.manual_seed(0)
  learned_a = _Learned(len(user_ids), len(buckets), len(titles))
  with torch.no_grad():                                   # builds the Dense kernels before the copy
    dev.query(learned_a, u[:2], ts[:2])
    dev.candidate(learned_a, m[:2])
  learned_b = copy.deepcopy(learned_a)
  model_a, model_b = _Model(dev, learned_a), _Model(host, learned_b)
  model_a.compile(optimizer=tfrs.optimizers.Adagrad(0.5))
  model_b.compile(optimizer=tfrs.optimizers.Adagrad(0.5))

  text0 = learned_a.text.weight.clone()
  ratings = Dataset.from_tensor_slices({"user_id": u, "timestamp": ts, "movie_title": m}).batch(512)
  losses_a = [float(model_a.train_step(b)["loss"]) for b in ratings]
  losses_b = [float(model_b.train_step(b)["loss"]) for b in ratings]
  assert len(losses_a) == 10 and losses_a == losses_b and np.isfinite(losses_a).all()
  for (na, pa), (nb, pb) in zip(learned_a.state_dict().items(), learned_b.state_dict().items()):
    assert na == nb and torch.equal(pa, pb), na
  assert not torch.equal(text0, learned_a.text.weight)

  t_mid = int(np.median(ts))
  queries = np.concatenate([user_ids[:40], ["nobody"]])
  qt = np.full(len(queries), t_mid, np.int64)
  results = []
  with torch.no_grad():
    for prep, learned in ((dev, learned_a), (host, learned_b)):
      index = tfrs.layers.factorized_top_k.BruteForce()
      index.index_from_dataset(Dataset.from_tensor_slices(titles).batch(100).map(
          lambda t: (t, prep.candidate(learned, t))))
      results.append(index(prep.query(learned, queries, qt)))
  (sa, ta), (sb, tb) = results
  assert ta.shape == (len(queries), 10) and np.array_equal(ta, tb) and torch.equal(sa, sb)

  rng = np.random.RandomState(1)
  split = rng.rand(len(u)) < 0.8
  train = Dataset.from_tensor_slices({"user_id": u[split], "movie_id": m[split]}).batch(1000)
  test = Dataset.from_tensor_slices({"user_id": u[~split], "movie_id": m[~split]}).batch(1000)
  mv = Dataset.from_tensor_slices({"movie_id": titles}).batch(128)
  got = []
  for prep, learned in ((dev, learned_a), (host, learned_b)):
    got.append(movielens.evaluate(
        lambda f: prep.query(learned, f["user_id"], np.full(len(f["user_id"]), t_mid, np.int64)),
        lambda f: prep.candidate(learned, f["movie_id"]), test, mv, train, k=10))
  assert got[0] == got[1] and got[0]["recall_at_k"] > 0

"""CPU checks of `examples.movielens.sample_listwise` and of dict elements in `data.Dataset`."""
import numpy as np
import pytest
import torch

from recommenders_b200 import data
from recommenders_b200.examples import movielens


def _ratings():
  # users b"a" (5 ratings), b"b" (2: too few for lists of 3), b"c" (4), interleaved
  users = [b"a", b"b", b"c", b"a", b"a", b"c", b"b", b"a", b"c", b"a", b"c"]
  titles = [f"m{i}".encode() for i in range(len(users))]
  ratings = np.float32([1, 2, 3, 4, 5, 1, 2, 3, 4, 5, 1])
  return users, titles, ratings


def _expected(users, titles, ratings, n_lists, m, seed):
  rs = np.random.RandomState(seed)
  order = list(dict.fromkeys(users))
  out = []
  for u in order:
    rows = [i for i, x in enumerate(users) if x == u]
    for _ in range(n_lists):
      if len(rows) < m:
        continue
      pick = rs.choice(range(len(rows)), size=m, replace=False)
      out.append((u, [titles[rows[k]] for k in pick], [ratings[rows[k]] for k in pick]))
  return out


@pytest.mark.parametrize("batched", [False, True])
def test_sample_listwise_reproduces_the_reference_draws(batched):
  users, titles, ratings = _ratings()
  ds = data.Dataset.from_tensor_slices({"user_id": np.array(users), "movie_title": np.array(titles), "user_rating": ratings})
  if batched:
    ds = ds.batch(4)
  got = movielens.sample_listwise(ds, num_list_per_user=3, num_examples_per_list=3, seed=42)
  (el,) = list(got)
  want = _expected(users, titles, ratings, 3, 3, 42)
  assert len(el["user_id"]) == len(want) == 6                 # "b" is skipped
  for k, (u, t, r) in enumerate(want):
    assert el["user_id"][k] == u
    assert list(el["movie_title"][k]) == t
    np.testing.assert_array_equal(el["user_rating"][k], np.float32(r))


def test_sample_listwise_skips_short_users_without_drawing():
  users, titles, ratings = _ratings()
  ds = {"user_id": np.array(users), "movie_title": np.array(titles), "user_rating": ratings}
  # with m = 5 only "a" qualifies; its draws must be the first draws of the generator
  (el,) = list(movielens.sample_listwise(data.Dataset.from_tensor_slices(ds), 2, 5, seed=7))
  rs = np.random.RandomState(7)
  rows = [i for i, x in enumerate(users) if x == b"a"]
  for k in range(2):
    pick = rs.choice(range(5), size=5, replace=False)
    assert list(el["movie_title"][k]) == [titles[rows[j]] for j in pick]
  assert list(el["user_id"]) == [b"a", b"a"]


def test_sample_listwise_shapes_and_dtypes():
  n = 40
  ids = torch.arange(n) % 4
  movies = torch.arange(n) + 100
  rating = (torch.arange(n) % 5 + 1).to(torch.float64)
  ds = data.Dataset.from_tensor_slices({"user_id": ids, "movie_title": movies, "user_rating": rating})
  (el,) = list(movielens.sample_listwise(ds, num_list_per_user=5, num_examples_per_list=4, seed=1))
  assert tuple(el["user_id"].shape) == (20,) and tuple(el["movie_title"].shape) == (20, 4)
  assert el["user_rating"].dtype == torch.float32 and tuple(el["user_rating"].shape) == (20, 4)
  assert isinstance(el["movie_title"], torch.Tensor) and el["movie_title"].dtype == torch.int64
  strs = {"user_id": np.array(["u1"] * 6), "movie_title": np.array([f"t{i}" for i in range(6)]), "user_rating": np.ones(6)}
  (el,) = list(movielens.sample_listwise(data.Dataset.from_tensor_slices(strs), 2, 3, seed=0))
  assert isinstance(el["movie_title"], np.ndarray) and el["movie_title"].shape == (2, 3) and el["user_id"].shape == (2,)
  assert el["user_rating"].dtype == np.float32


def test_dataset_dict_batching():
  d = {"a": np.arange(10), "b": torch.arange(20).reshape(10, 2), "c": ["x"] * 10}
  ds = data.Dataset.from_tensor_slices(d)
  assert not ds.is_tuple
  batches = list(ds.batch(4))
  assert [len(b["a"]) for b in batches] == [4, 4, 2]
  assert torch.equal(batches[1]["b"], torch.arange(8, 16).reshape(4, 2))
  assert list(batches[2]["c"]) == ["x", "x"]
  assert [len(b["a"]) for b in ds.batch(4, drop_remainder=True)] == [4, 4]
  (whole,) = list(ds)
  assert set(whole) == {"a", "b", "c"}
  assert [int(x["a"].sum()) for x in ds.batch(5).map(lambda el: {"a": el["a"] * 2})] == [20, 70]
  with pytest.raises(ValueError):
    data.Dataset.from_tensor_slices({"a": np.arange(3), "b": np.arange(4)})

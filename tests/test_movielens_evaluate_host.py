"""CPU checks of `examples.movielens.evaluate`: its NumPy oracle against a transcription of the reference's loop, and the
host side (vocabulary, user order, per-user CSR lists, unknown ids, string and int ids) that runs before the GPU."""
import numpy as np
import pytest
import torch

import movielens_eval_oracle as meo
from recommenders_b200 import data, ops
from recommenders_b200.examples import movielens


def _tie_free(rng, n_movies, n_users, n_test, n_train, k, dup_movies=0):
  """Integer scores that are exact in fp32 and distinct per user: movie j = (p_j, 1), user = (a_u, b_u), a_u != 0.
  Every user keeps at least k untrained movies or has N <= k, so the reference's unpinned tie order among the -1e6 rows
  cannot change which rows reach the top k."""
  movie_ids = rng.permutation(1000)[:n_movies] + 5000
  if dup_movies:
    movie_ids[-dup_movies:] = movie_ids[:dup_movies]          # duplicate ids: the later row wins the vocabulary
  emb = np.stack([rng.permutation(n_movies).astype(np.float32) - n_movies // 2, np.ones(n_movies, np.float32)], 1)
  users = rng.permutation(100)[:n_users] + 10
  ue = {int(u): np.float32([rng.choice([-3, -1, 1, 2]), rng.randint(-5, 5)]) for u in users}
  vocab = np.unique(movie_ids)
  test = (rng.choice(users, n_test), rng.choice(vocab, n_test))
  limit = len(vocab) if n_movies <= k else max(0, len(vocab) - k)   # N <= k: the top k are all N rows in any order
  tr_u, tr_m = [], []
  for u in users:
    m = rng.choice(vocab, min(limit, rng.randint(0, n_train + 1)), replace=False) if limit else []
    tr_u += [u] * len(m); tr_m += list(m)
  tr_u += [999] * 3; tr_m += list(vocab[:3])                   # a user who is not in test: ignored
  train = (np.array(tr_u), np.array(tr_m))
  return movie_ids, emb, (lambda u: ue[int(u)]), test, train


@pytest.mark.parametrize("k,n_movies,dup", [(1, 40, 0), (5, 40, 3), (10, 60, 5), (10, 8, 0), (30, 25, 2)])
def test_oracle_matches_the_reference_loop_on_tie_free_data(k, n_movies, dup):
  rng = np.random.RandomState(k * 100 + n_movies)
  movie_ids, emb, ue, test, train = _tie_free(rng, n_movies, 12, 80, 15, k, dup)
  for tr in (None, train):
    want = meo.reference_loop(ue, emb, movie_ids, test, tr, k)
    got = meo.evaluate(ue, emb, movie_ids, test, tr, k)
    assert got == want and type(got["precision_at_k"]) is type(want["precision_at_k"]), (got, want)


def test_oracle_tie_rule_and_override():
  # every score ties: the top k are the lowest rows; listed rows sit at -1e6, after every unlisted row
  q = np.zeros((2, 3), np.float32); c = np.ones((6, 3), np.float32)
  s, i = meo.topk_overriding(q, c, 4, [0, 2, 6], np.array([0, 3, 0, 1, 2, 4]))
  assert i.tolist() == [[1, 2, 4, 5], [3, 5, 0, 1]]
  assert s.tolist() == [[0, 0, 0, 0], [0, 0, -1e6, -1e6]]
  # a row scoring below -1e6 ranks after the listed rows; N < k returns N rows
  c2 = np.float32([[1], [-3e6], [2]]); q2 = np.float32([[1]])
  s, i = meo.topk_overriding(q2, c2, 5, [0, 1], np.array([2]))
  assert i.tolist() == [[0, 2, 1]] and s.tolist() == [[1, -1e6, -3e6]]
  assert meo.count_listed(np.array([[0, 2, 1]]), [0, 4], np.array([2, 2, 7, 0])).tolist() == [3]


def _columns(users, movies, kind):
  if kind == "torch":
    return {"user_id": torch.as_tensor(users), "movie_id": torch.as_tensor(movies)}
  if kind == "bytes":
    return {"user_id": np.array([b"u%d" % u for u in users]), "movie_id": np.array([b"m%d" % m for m in movies])}
  return {"user_id": np.array(["u%d" % u for u in users]), "movie_id": np.array(["m%d" % m for m in movies])}


@pytest.mark.parametrize("kind", ["int", "torch", "bytes", "str"])
def test_evaluation_lists_match_the_reference_dicts(kind):
  rng = np.random.RandomState(3)
  movie_ids = np.concatenate([np.arange(30), [4, 9, 4]])       # rows 30..32 repeat ids 4, 9, 4: the last row wins
  test_u, test_m = rng.randint(0, 9, 70), rng.choice(30, 70)
  train_u, train_m = rng.randint(0, 12, 90), rng.choice(30, 90)   # users 9..11 are not in test
  conv = lambda cols: {k: (v.numpy() if isinstance(v, torch.Tensor) else v) for k, v in cols.items()}
  test, train = conv(_columns(test_u, test_m, kind)), conv(_columns(train_u, train_m, kind))
  mids = conv(_columns(np.zeros_like(movie_ids), movie_ids, kind))["movie_id"]
  users, (toff, trows), (roff, rrows) = movielens.evaluation_lists(mids, test, train)
  vocab, test_lists, train_lists = meo._lists(mids, (test["user_id"], test["movie_id"]), (train["user_id"], train["movie_id"]))
  assert vocab[mids[4].item()] == 32 and vocab[mids[9].item()] == 31
  assert users.tolist() == list(test_lists)                    # order of first appearance in test
  for u, uid in enumerate(users.tolist()):
    assert trows[toff[u]:toff[u + 1]].tolist() == list(test_lists[uid])
    assert rrows[roff[u]:roff[u + 1]].tolist() == sorted(set(train_lists[uid]))
  assert len(users) == 9 and toff[-1] == 70


def test_evaluation_lists_without_train_and_empty_test():
  users, (toff, trows), (roff, rrows) = movielens.evaluation_lists(
      np.arange(5), {"user_id": np.array([7, 3, 7]), "movie_id": np.array([4, 4, 0])}, None)
  assert users.tolist() == [7, 3] and toff.tolist() == [0, 2, 3] and trows.tolist() == [4, 0, 4]
  assert roff.tolist() == [0, 0, 0] and rrows.size == 0
  users, (toff, _), _ = movielens.evaluation_lists(np.arange(5), {"user_id": np.zeros(0, int), "movie_id": np.zeros(0, int)}, None)
  assert len(users) == 0 and toff.tolist() == [0]


def _never(_):
  raise AssertionError("no model call before the ids are checked")


@pytest.mark.parametrize("where", ["test", "train", "train_other_user", "type"])
def test_unknown_movie_raises_key_error(where):
  movies = data.Dataset.from_tensor_slices({"movie_id": np.arange(10)})
  test = {"user_id": np.array([1, 2]), "movie_id": np.array([3, 4])}
  train = {"user_id": np.array([1, 2]), "movie_id": np.array([5, 6])}
  if where == "test":
    test["movie_id"] = np.array([3, 42])
  elif where == "train":
    train["movie_id"] = np.array([5, 42])
  elif where == "train_other_user":
    train = {"user_id": np.array([1, 77]), "movie_id": np.array([5, 42])}
  else:
    test["movie_id"] = np.array(["3", "4"])
  with pytest.raises(KeyError) as e:
    movielens.evaluate(_never, _never, data.Dataset.from_tensor_slices(test), movies,
                       data.Dataset.from_tensor_slices(train).batch(1), k=3)
  assert e.value.args[0] in (42, "3")


def test_override_width_classes():
  e = np.array([0, 1, 5, 6, 100, 118, 246, 247, 5000])
  for N in (3, 100, 300, 70000):
    for k in (1, 10, 100, 256):
      w = ops.override_width(k, e[e <= N], N)
      need = np.minimum(N, k + e[e <= N])
      scan = need <= ops.TC_MAX_K
      assert (w[~scan] == 0).all()
      assert (w[scan] >= need[scan]).all() and (w[scan] >= min(k, N)).all() and (w[scan] <= min(N, ops.TC_MAX_K)).all()
      assert len(np.unique(w)) <= 10

"""CPU restatement of `examples.movielens.evaluate` (examples/movielens.py:26-93) and of the K14 ops behind it.

`topk_overriding` / `count_listed` / `evaluate` use the canonical fmaf-chain scores (`oracle.scores`) and the pinned tie
rule (score descending, ties to the lower row; `oracle.top_k_rows`).  `reference_loop` is a literal transcription of the
reference's loop (BLAS matmul, `np.argsort(-scores)[:k]`), used to check `evaluate` on data without ties."""
import array
import collections

import numpy as np

from oracle import oracle as orc

OVERRIDE = np.float32(-1e6)


def topk_overriding(q, c, k, offsets, rows):
  """([Q, min(k, N)] scores, rows): canonical scores, the listed rows of each query set to -1e6, top k by the tie rule."""
  s = orc.scores(q, c)
  off = np.asarray(offsets, np.int64)
  owner = np.repeat(np.arange(s.shape[0]), np.diff(off))
  s[owner, np.asarray(rows, np.int64)] = OVERRIDE
  return orc.top_k_rows(s, min(k, s.shape[1]))


def count_listed(top_rows, offsets, rows):
  off = np.asarray(offsets, np.int64)
  return np.array([sum(int(x in set(top_rows[u].tolist())) for x in rows[off[u]:off[u + 1]]) for u in range(len(off) - 1)],
                  np.int32)


def _lists(movie_ids, test, train):
  """The reference's vocabulary and per-user lists (movielens.py:47-64), as plain dicts: (vocabulary, test lists, train
  lists), users in order of first appearance in `test`."""
  vocabulary = dict(zip(movie_ids.tolist(), range(len(movie_ids))))
  train_lists = collections.defaultdict(lambda: array.array("i"))
  test_lists = collections.defaultdict(lambda: array.array("i"))
  if train is not None:
    for user_id, movie_id in zip(*train):
      train_lists[user_id].append(vocabulary[movie_id])
  for user_id, movie_id in zip(*test):
    test_lists[user_id].append(vocabulary[movie_id])
  return vocabulary, test_lists, train_lists


def evaluate(user_embedding, movie_embeddings, movie_ids, test, train=None, k=10):
  """The reference's metrics with canonical scores and the pinned tie rule.  `test` / `train` are (user ids, movie ids)
  column pairs, `user_embedding(user_id)` returns the user's [d] embedding, `movie_embeddings` is [N, d]."""
  _, test_lists, train_lists = _lists(np.asarray(movie_ids), test, train)
  users = list(test_lists)
  q = np.stack([np.asarray(user_embedding(u), np.float32) for u in users]) if users else np.zeros((0, 1), np.float32)
  lists = [np.sort(np.unique(np.frombuffer(train_lists[u], np.int32))) if train is not None else np.zeros(0, np.int64)
           for u in users]
  offsets = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
  rows = np.concatenate(lists).astype(np.int64) if lists else np.zeros(0, np.int64)
  precision_values, recall_values = [], []
  if users:
    _, top = topk_overriding(q, movie_embeddings, k, offsets, rows)
    for u, user_id in enumerate(users):
      test_movies = np.frombuffer(test_lists[user_id], dtype=np.int32)
      hits = sum(x in top[u] for x in test_movies)
      precision_values.append(hits / k)
      recall_values.append(hits / len(test_movies))
  return {"precision_at_k": np.mean(precision_values), "recall_at_k": np.mean(recall_values)}


def reference_loop(user_embedding, movie_embeddings, movie_ids, test, train=None, k=10):
  """examples/movielens.py:71-93 transcribed line by line (NumPy matmul and argsort)."""
  _, test_user_to_movies, train_user_to_movies = _lists(np.asarray(movie_ids), test, train)
  movie_embeddings = np.asarray(movie_embeddings, np.float32)
  precision_values = []
  recall_values = []
  for user_id, test_movies in test_user_to_movies.items():
    user_embedding_ = np.asarray(user_embedding(user_id), np.float32)[None, :]
    scores = (user_embedding_ @ movie_embeddings.T).flatten()
    test_movies = np.frombuffer(test_movies, dtype=np.int32)
    if train is not None:
      train_movies = np.frombuffer(train_user_to_movies[user_id], dtype=np.int32)
      scores[train_movies] = -1e6
    top_movies = np.argsort(-scores)[:k]
    num_test_movies_in_k = sum(x in top_movies for x in test_movies)
    precision_values.append(num_test_movies_in_k / k)
    recall_values.append(num_test_movies_in_k / len(test_movies))
  return {"precision_at_k": np.mean(precision_values), "recall_at_k": np.mean(recall_values)}

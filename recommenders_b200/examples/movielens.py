"""MovieLens helpers: mirror of tensorflow_recommenders/examples/movielens.py (`evaluate`, `sample_listwise`)."""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

from .. import ops
from ..data import Dataset

MOVIE_BATCH = 4096   # movies per movie_model call, as the reference batches them
USER_BATCH = 4096    # users per user_model call


def _rows(rating_dataset, names=("user_id", "movie_title", "user_rating")):
  """The `names` columns of a dataset of dict elements (batched or not) or of a dict of columns, and the first value of
  each column (its container)."""
  parts = {name: [] for name in names}
  batches = [rating_dataset] if isinstance(rating_dataset, dict) else rating_dataset
  kind = {}
  for batch in batches:
    for name in parts:
      v = batch[name]
      kind.setdefault(name, v)
      parts[name].append(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v))
  return {k: (np.concatenate(v) if v else np.zeros((0,))) for k, v in parts.items()}, kind


def _is_text(a: np.ndarray) -> bool:
  return a.dtype.kind in "USO"


def _positions(keys: np.ndarray, values: np.ndarray):
  """For each value, the LAST position of an equal key (what dict(zip(keys, range(n))) maps it to), or -1."""
  if not len(values):
    return np.zeros((0,), np.int64)
  if not len(keys) or _is_text(keys) != _is_text(values) or (_is_text(keys) and keys.dtype.kind != values.dtype.kind):
    return np.full(len(values), -1, np.int64)   # keys of another type never compare equal
  order = np.argsort(keys, kind="stable")
  sk = keys[order]
  pos = np.searchsorted(sk, values, side="right") - 1
  hit = pos >= 0
  hit[hit] = sk[pos[hit]] == values[hit]
  return np.where(hit, order[np.maximum(pos, 0)], -1)


def _vocabulary_rows(movie_ids: np.ndarray, ids: np.ndarray) -> np.ndarray:
  rows = _positions(movie_ids, ids)
  if (rows < 0).any():
    raise KeyError(ids[np.argmax(rows < 0)].item())   # the first unknown id, as the reference's dict lookup raises
  return rows


def _lists(owner: np.ndarray, rows: np.ndarray, n: int, unique: bool):
  """CSR of `rows` grouped by `owner` in 0..n-1: offsets [n+1] and the rows, in order of appearance, or sorted and
  deduplicated when `unique`."""
  order = np.lexsort((rows, owner)) if unique else np.argsort(owner, kind="stable")
  o, r = owner[order], rows[order]
  if unique and len(r):
    keep = np.ones(len(r), bool)
    keep[1:] = (o[1:] != o[:-1]) | (r[1:] != r[:-1])
    o, r = o[keep], r[keep]
  offsets = np.zeros(n + 1, np.int64)
  np.cumsum(np.bincount(o, minlength=n), out=offsets[1:])
  return offsets, r.astype(np.int64)


def evaluation_lists(movie_ids: np.ndarray, test: dict, train: Optional[dict]):
  """`evaluate`'s host side (examples/movielens.py:47-64) on "user_id" / "movie_id" NumPy columns: the test users in
  order of first appearance, then per user the CSR (offsets, vocabulary rows) of its test movies in order of appearance
  and of its train movies sorted and deduplicated.  Train rows of other users are ignored, but every train movie is
  looked up.  An unknown movie raises KeyError."""
  test_rows = _vocabulary_rows(movie_ids, test["movie_id"])
  if train is not None:
    train_rows = _vocabulary_rows(movie_ids, train["movie_id"])
  uniq, first, inverse = np.unique(test["user_id"], return_index=True, return_inverse=True)
  by_appearance = np.argsort(first, kind="stable")
  user_pos = np.empty(len(uniq), np.int64)
  user_pos[by_appearance] = np.arange(len(uniq))
  U = len(uniq)
  test_csr = _lists(user_pos[inverse.reshape(-1)], test_rows, U, unique=False)
  if train is None:
    return uniq[by_appearance], test_csr, (np.zeros(U + 1, np.int64), np.zeros((0,), np.int64))
  owner = _positions(uniq, train["user_id"])   # uniq holds each test user once
  known = owner >= 0
  return uniq[by_appearance], test_csr, _lists(user_pos[owner[known]], train_rows[known], U, unique=True)


def _embed(model, name: str, ids: np.ndarray, template, batch: int) -> torch.Tensor:
  out = []
  with torch.no_grad():
    for lo in range(0, len(ids), batch):
      e = model({name: _like(ids[lo:lo + batch], template)})
      out.append(e if isinstance(e, torch.Tensor) else torch.as_tensor(np.asarray(e)))
  e = torch.cat(out)
  return (e if e.is_cuda else e.to(torch.cuda.current_device())).to(torch.float32).contiguous()


def evaluate(user_model, movie_model, test, movies, train=None, k: int = 10) -> Dict[str, float]:
  """Precision and recall at k of retrieving each test user's test movies (examples/movielens.py:26-93).

  `test`, `train` and `movies` are datasets of dict elements (batched or not) with "user_id" / "movie_id" columns
  (torch tensors or NumPy arrays, string ids included).  Same rules as the reference: the vocabulary is
  dict(zip(movie ids, rows)) (the last row of a duplicate id wins; every row keeps its embedding), an unknown test or
  train movie raises KeyError, users come in order of first appearance in `test`, and each user's train movies score
  -1e6 (they are not removed).  Ranking is by score descending, ties to the lower row.  Hits count the test entries
  with multiplicity; precision = hits / k, recall = hits / #test entries, and the means are NumPy's over the users.

  The movies are embedded in calls of 4096, as in the reference.  Unlike the reference, `user_model` is called on
  batches of up to 4096 users instead of one user per call: results are identical for towers that treat rows
  independently, but a Dense layer picks its kernel by batch shape, so an MLP tower may differ in the last bits.
  The top k of every user is one `ops.topk_overriding` call; only the [U] hit counts come back to the host."""
  (mcols, mkind) = _rows(movies, ("movie_id",))
  movie_ids = mcols["movie_id"]
  tcols, tkind = _rows(test, ("user_id", "movie_id"))
  rcols = None if train is None else _rows(train, ("user_id", "movie_id"))[0]
  users, (test_off, test_lists), (train_off, train_lists) = evaluation_lists(movie_ids, tcols, rcols)

  hits, n_test = [], np.diff(test_off).tolist()
  if len(users):
    movie_emb = _embed(movie_model, "movie_id", movie_ids, mkind.get("movie_id"), MOVIE_BATCH)
    user_emb = _embed(user_model, "user_id", users, tkind.get("user_id"), USER_BATCH)
    _, top_rows = ops.topk_overriding(user_emb, movie_emb, k, train_off, train_lists, image="movielens_eval")
    hits = ops.count_listed(top_rows, test_off, test_lists).cpu().numpy().tolist()
  precision_values = [h / k for h in hits]
  recall_values = [h / n for h, n in zip(hits, n_test)]
  return {
      "precision_at_k": np.mean(precision_values),
      "recall_at_k": np.mean(recall_values),
  }


def _like(values: np.ndarray, template, dtype=None):
  """`values` in the container of the input column: a torch tensor on its device, or a NumPy array (e.g. strings)."""
  if dtype is not None:
    values = values.astype(dtype)
  if isinstance(template, torch.Tensor) and values.dtype.kind in "biuf":
    return torch.from_numpy(np.ascontiguousarray(values)).to(template.device)
  return values


def sample_listwise(rating_dataset, num_list_per_user: int = 10, num_examples_per_list: int = 10,
                    seed: Optional[int] = None) -> Dataset:
  """Turns ratings into lists of `num_examples_per_list` movies per user (movielens.py:129-192).

  Makes the reference's draws: one `np.random.RandomState(seed)`, users in the order they first appear, and for each of a
  user's `num_list_per_user` lists one `choice(range(n), size=num_examples_per_list, replace=False)` over the user's n
  ratings in their order of appearance.  A user with fewer ratings than `num_examples_per_list` is skipped and consumes no
  draw.  Returns `Dataset.from_tensor_slices` of {"user_id": [N], "movie_title": [N, m], "user_rating": [N, m] float32}; every
  column keeps the container of the input column (NumPy for strings, a torch tensor on its device for torch inputs)."""
  random_state = np.random.RandomState(seed)
  cols, kind = _rows(rating_dataset)
  by_user = {}
  for row, user in enumerate(cols["user_id"].tolist()):
    by_user.setdefault(user, []).append(row)

  users, titles, ratings = [], [], []
  for user, rows in by_user.items():
    for _ in range(num_list_per_user):
      if len(rows) < num_examples_per_list:   # drop the user if they don't have enough ratings
        continue
      sampled = random_state.choice(range(len(rows)), size=num_examples_per_list, replace=False)
      picked = np.asarray(rows)[sampled]
      users.append(user)
      titles.append(cols["movie_title"][picked])
      ratings.append(cols["user_rating"][picked])

  m = num_examples_per_list
  uid = np.asarray(users, dtype=cols["user_id"].dtype) if users else np.zeros((0,), dtype=cols["user_id"].dtype)
  title = np.stack(titles) if titles else np.zeros((0, m), dtype=cols["movie_title"].dtype)
  rating = np.stack(ratings) if ratings else np.zeros((0, m), dtype=np.float32)
  return Dataset.from_tensor_slices({
      "user_id": _like(uid, kind.get("user_id")),
      "movie_title": _like(title, kind.get("movie_title")),
      "user_rating": _like(rating, kind.get("user_rating"), np.float32),
  })

"""MovieLens helpers: mirror of tensorflow_recommenders/examples/movielens.py (`sample_listwise`)."""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from ..data import Dataset


def _rows(rating_dataset):
  """(user_id, movie_title, user_rating) columns of a dataset of dict elements (batched or not) or of a dict of columns."""
  parts = {"user_id": [], "movie_title": [], "user_rating": []}
  batches = [rating_dataset] if isinstance(rating_dataset, dict) else rating_dataset
  kind = {}
  for batch in batches:
    for name in parts:
      v = batch[name]
      kind.setdefault(name, v)
      parts[name].append(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v))
  return {k: (np.concatenate(v) if v else np.zeros((0,))) for k, v in parts.items()}, kind


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

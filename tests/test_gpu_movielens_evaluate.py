"""K14 on the GPU: `ops.topk_overriding` (scan and dense routes), `ops.count_listed` and `examples.movielens.evaluate`,
byte for byte against tests/movielens_eval_oracle.py."""
import numpy as np
import pytest
import torch

import movielens_eval_oracle as meo
from recommenders_b200 import _ffi, data, ops
from recommenders_b200.examples import movielens

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _csr(rng, N, lengths):
  lists = [np.sort(rng.choice(N, e, replace=False)) for e in lengths]
  off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
  return off, (np.concatenate(lists) if lists else np.zeros(0)).astype(np.int64)


def _check(q, c, k, off, rows, image=None, max_chunk_bytes=None):
  """Both entry points equal the oracle bit for bit; returns the mixed-route result."""
  ws, wi = meo.topk_overriding(q, c, k, off, rows)
  qd, cd = torch.from_numpy(q).to(DEV), torch.from_numpy(c).to(DEV)
  if image == "build":
    image = ops.index_build(cd)
  got = ops.topk_overriding(qd, cd, k, off, rows, image=image)
  dense = ops.topk_overriding_dense(qd, cd, k, off, rows, max_chunk_bytes=max_chunk_bytes)
  for name, (s, i) in (("mixed", got), ("dense", dense)):
    assert s.shape == ws.shape and i.shape == wi.shape, name
    assert np.array_equal(i.cpu().numpy(), wi), name
    assert s.cpu().numpy().tobytes() == ws.tobytes(), name
  return got


def _data(rng, Q, N, d):
  return rng.normal(size=(Q, d)).astype(np.float32), rng.normal(size=(N, d)).astype(np.float32)


# list lengths on every route edge at k = 10: k + e = 255, 256 (scan) and 257 (dense), e = 0, e >= N - k, all rows
def _edge_lengths(N, k=10):
  return [0, 1, 7, 245, 246, 247, 600, N - k, N - k + 3, N, 0, 3]


@pytest.mark.parametrize("N", [ops.TC_MIN_N - 1, ops.TC_MIN_N, 70000])
def test_topk_overriding_on_both_sides_of_the_tensor_core_range(N):
  rng = np.random.RandomState(N % 1000)
  lengths = _edge_lengths(N)
  q, c = _data(rng, len(lengths), N, 64)
  off, rows = _csr(rng, N, lengths)
  widths = set(ops.override_width(10, np.array(lengths), N).tolist())
  assert 0 in widths and 256 in widths
  if N >= ops.TC_MIN_N:
    assert any(ops.uses_tc_scan(len(lengths), N, 64, w) for w in widths if w)
  _check(q, c, 10, off, rows, image="build")


@pytest.mark.parametrize("d", [1, 64, 128, 129])
def test_topk_overriding_widths(d):
  rng = np.random.RandomState(d)
  N = 20000 if d == 128 else 3000
  lengths = [0, 5, 60, 155, 156, 157, 2000, N - 100, N]
  q, c = _data(rng, len(lengths), N, d)
  off, rows = _csr(rng, N, lengths)
  _check(q, c, 100, off, rows, image="build" if d <= 128 and N >= ops.TC_MIN_N else None)
  _check(q, c, 256, off, rows)
  _check(q, c, 1, off, rows)


def test_topk_overriding_fewer_rows_than_k():
  rng = np.random.RandomState(1)
  q, c = _data(rng, 4, 6, 8)
  off, rows = _csr(rng, 6, [0, 2, 6, 5])
  s, i = _check(q, c, 10, off, rows)
  assert s.shape == (4, 6)


def test_topk_overriding_ties_and_scores_at_or_below_the_override():
  rng = np.random.RandomState(2)
  N, d = 400, 4
  c = rng.normal(size=(N, d)).astype(np.float32)
  c[10:20] = c[5]                                  # exact ties with row 5
  c[30:40] = np.float32([-1e6, 0, 0, 0])           # exactly -1e6 for the queries below
  c[40:45] = np.float32([-3e6, 0, 0, 0])           # below -1e6
  q = np.zeros((6, d), np.float32); q[:, 0] = 1
  q[3:] = rng.normal(size=(3, d)).astype(np.float32)
  q[5] = 0                                         # every score ties (+0)
  lengths = [0, 395, 398, 390, 100, 200]
  off, rows = _csr(rng, N, lengths)
  for k in (1, 10, 64):
    _check(q, c, k, off, rows)
  # listed rows among the -1e6 rows: rows 31 and 35 are listed, so every -1e6 row ties and ranks by row
  off2, rows2 = np.array([0, 2, 2]), np.array([31, 35])
  c2 = c.copy(); c2[100:] = np.float32([-2e6, 0, 0, 0])
  _check(q[:2], c2, 120, off2, rows2)


def test_dense_route_chunk_boundaries_and_route_agreement():
  rng = np.random.RandomState(3)
  N, d, k = 5000, 32, 20
  lengths = [0, 10, 236, 237, 300, 4980, 5000]
  q, c = _data(rng, len(lengths), N, d)
  off, rows = _csr(rng, N, lengths)
  for chunk in (1, 2, 3):
    _check(q, c, k, off, rows, max_chunk_bytes=_ffi.lib().tfrs_topk_overriding_dense_workspace_bytes(chunk, N, d, k))
  # the scan route's users through the dense route give the same bits
  qd, cd = torch.from_numpy(q).to(DEV), torch.from_numpy(c).to(DEV)
  a = ops.topk_overriding(qd, cd, k, off, rows)
  b = ops.topk_overriding_dense(qd, cd, k, off, rows)
  assert torch.equal(a[1], b[1]) and a[0].cpu().numpy().tobytes() == b[0].cpu().numpy().tobytes()


def test_workspace_garbage_changes_nothing():
  rng = np.random.RandomState(4)
  N, d, k = 20000, 64, 10
  lengths = [0, 3, 246, 247, 1000]
  q, c = _data(rng, len(lengths), N, d)
  off, rows = _csr(rng, N, lengths)
  for slot in ("override", "scan", "tc"):
    _ffi.workspace(64 << 20, DEV, slot).random_(0, 256)
  _check(q, c, k, off, rows, image="build")


def test_count_listed_matches_the_oracle():
  rng = np.random.RandomState(5)
  Q, kk = 37, 50
  top = np.stack([rng.choice(1000, kk, replace=False) for _ in range(Q)]).astype(np.int64)
  lengths = rng.randint(0, 120, Q); lengths[3] = 0
  off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
  rows = rng.randint(0, 1000, off[-1]).astype(np.int64)
  rows[:20] = top[0, :1].repeat(20)                # duplicates count each time
  got = ops.count_listed(torch.from_numpy(top).to(DEV), off, rows).cpu().numpy()
  assert np.array_equal(got, meo.count_listed(top, off, rows))
  assert np.array_equal(ops.count_listed(torch.zeros((3, 0), dtype=torch.int64, device=DEV), [0, 1, 1, 2], [4, 5]).cpu().numpy(),
                        [0, 0, 0])


def _movielens(rng, n_users, n_movies, d, n_test, text):
  movie_ids = np.arange(n_movies) * 3 + 1
  movie_ids[-4:] = movie_ids[:4]                   # duplicate ids: the later rows win the vocabulary
  users = np.arange(n_users) * 7 + 2
  U_tab = rng.normal(size=(n_users, d)).astype(np.float32)
  M_tab = rng.normal(size=(n_movies, d)).astype(np.float32)
  vocab = np.unique(movie_ids)
  hist = np.minimum((rng.pareto(1.2, n_users) * 20).astype(int), len(vocab) - 1)
  hist[:3] = [0, len(vocab) - 1, 300]              # no history, every movie, the dense route
  tr_u = np.repeat(users, hist)
  tr_m = np.concatenate([rng.choice(vocab, h, replace=False) for h in hist])
  te_u = rng.choice(users, n_test); te_m = rng.choice(vocab, n_test)
  urow = {int(u): r for r, u in enumerate(users)}
  if text:
    fmt = lambda a, p: np.array(["%s%d" % (p, x) for x in a])
    movie_ids, tr_u, tr_m, te_u, te_m = fmt(movie_ids, "m"), fmt(tr_u, "u"), fmt(tr_m, "m"), fmt(te_u, "u"), fmt(te_m, "m")
    urow = {"u%d" % u: r for u, r in urow.items()}
  return movie_ids, (te_u, te_m), (tr_u, tr_m), U_tab, M_tab, urow


@pytest.mark.parametrize("kind", ["torch", "numpy_text"])
def test_evaluate_returns_the_oracle_dict(kind):
  rng = np.random.RandomState(6)
  text = kind == "numpy_text"
  movie_ids, test, train, U_tab, M_tab, urow = _movielens(rng, 700, 5000, 32, 5000, text)
  Ud, Md = torch.from_numpy(U_tab).to(DEV), torch.from_numpy(M_tab).to(DEV)
  calls = {"movie": [], "user": []}

  def movie_model(f):                              # the movie ids arrive in row order, 4096 at a time
    ids = f["movie_id"]
    calls["movie"].append(len(ids))
    lo = sum(calls["movie"][:-1])
    return Md[lo:lo + len(ids)]

  def user_model(f):
    ids = f["user_id"]
    calls["user"].append(len(ids))
    keys = ids.cpu().tolist() if isinstance(ids, torch.Tensor) else ids.tolist()
    return Ud[torch.tensor([urow[x] for x in keys], device=DEV)]

  def col(a):
    return torch.from_numpy(a).to(DEV) if kind == "torch" else a

  mk = lambda cols: data.Dataset.from_tensor_slices({kk: col(v) for kk, v in cols.items()})
  ds_movies = mk({"movie_id": movie_ids})
  ds_test = mk({"user_id": test[0], "movie_id": test[1]}).batch(999)
  ds_train = mk({"user_id": train[0], "movie_id": train[1]}).batch(1234)
  for k in (10, 100):
    for tr in (None, ds_train):
      calls["movie"].clear(); calls["user"].clear()
      got = movielens.evaluate(user_model, movie_model, ds_test, ds_movies, tr, k=k)
      want = meo.evaluate(lambda u: U_tab[urow[u]], M_tab, movie_ids, test, None if tr is None else train, k)
      assert got == want, (got, want)
      assert all(n == 4096 for n in calls["movie"][:-1]) and sum(calls["movie"]) == len(movie_ids)
      assert len(calls["user"]) == 1 and calls["user"][0] == len(set(test[0].tolist()))

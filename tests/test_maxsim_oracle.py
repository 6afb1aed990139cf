"""CPU tests of multi-interest (maxsim) retrieval: the NumPy oracle against the reference's multipoint known answer, the
exactness argument of K26 (per-head top-k, then the head merge) replayed in NumPy against the full maxsim order on data
with planted ties, the C ABI's argument errors (checked before any device work) and the ABI declarations."""
import ctypes
import os
import re

import numpy as np
import pytest

import maxsim_oracle as mo
from oracle import oracle as orc
from recommenders_b200 import _ffi, ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _bits(a):
  return np.asarray(a, F32).view(np.uint32)


def test_multipoint_known_answer():
  """retrieval_test.py:255-298 (RetrievalTestWithMultipointQueries): two heads per query, three candidates."""
  q = np.array([[[3, 2, 1], [1, 2, 3]], [[2, 3, 4], [4, 3, 2]]], F32)
  c = np.array([[0, 1, 0], [0, 1, 1], [1, 1, 0]], F32)
  for s, i in (mo.topk_maxsim(q, c, 3), mo.per_head_then_merge(q, c, 3)):
    np.testing.assert_array_equal(s, np.array([[5, 5, 2], [7, 7, 3]], F32))
    np.testing.assert_array_equal(i, np.array([[1, 2, 0], [1, 2, 0]]))


def test_head_max_keeps_the_lowest_head_among_ties():
  z = np.array([[[0.0, -0.0, 1.0]], [[-0.0, 0.0, 1.0]]], F32).transpose(1, 0, 2)   # [1, H=2, 3]
  got = mo.head_max(z)
  np.testing.assert_array_equal(_bits(got), _bits(np.array([[0.0, -0.0, 1.0]], F32)))


@pytest.mark.parametrize("Q,H,N,d,k", [
    (5, 1, 40, 3, 7), (6, 2, 50, 2, 10), (4, 3, 30, 1, 30), (6, 4, 64, 3, 1), (6, 4, 64, 3, 20), (5, 5, 29, 2, 40),
    (4, 8, 120, 4, 33), (3, 16, 70, 1, 64)])
def test_per_head_topk_then_merge_is_the_maxsim_topk(Q, H, N, d, k):
  """The exactness argument, replayed: every head row's own top-min(k, N), merged by K26's rule, equals the top of the
  full maxsim order -- ids and score bits -- with duplicate rows, duplicate / zero / tiny heads and +-0 planted."""
  q, c = mo.planted_case(Q, H, N, d, seed=Q * 1000 + H * 10 + d)
  es, ei = mo.topk_maxsim(q, c, k)
  gs, gi = mo.per_head_then_merge(q, c, k)
  np.testing.assert_array_equal(gi, ei)
  np.testing.assert_array_equal(_bits(gs), _bits(es))
  if H >= 4:   # the planted signed zeros took part: some retrieved score is -0 somewhere, some +0 elsewhere
    m = mo.maxsim_scores(q, c)
    assert (_bits(m) == 0x80000000).any() and (_bits(m) == 0).any()


@pytest.mark.parametrize("H", [1, 3])
def test_single_and_repeated_heads_equal_the_2d_scan(H):
  q, c = mo.planted_case(7, 1, 90, 3, seed=11)
  q3 = np.repeat(q, H, axis=1)
  s2, i2 = orc.topk_scan(q[:, 0], c, 25)
  for s, i in (mo.topk_maxsim(q3, c, 25), mo.per_head_then_merge(q3, c, 25)):
    np.testing.assert_array_equal(i, i2)
    np.testing.assert_array_equal(_bits(s), _bits(s2))


def test_rowwise_maxsim_oracle():
  q, c = mo.planted_case(9, 4, 9, 3, seed=5)
  per = np.stack([[orc.scores(q[r:r + 1, h], c[r:r + 1])[0, 0] for h in range(4)] for r in range(9)])
  want = np.array([row[np.argmax(row == row.max())] for row in per], F32)   # first head reaching the maximum
  np.testing.assert_array_equal(_bits(mo.rowwise_maxsim(q, c)), _bits(want))


# ------------------------------------------------------------------------------------------------
# the C ABI rejects bad arguments before any device work
# ------------------------------------------------------------------------------------------------
def _err():
  return _ffi.last_error()


@pytest.mark.parametrize("H,w,k_out,rc", [
    (0, 4, 1, -1), (2, 0, 1, -1), (2, 4, 0, -1), (2, 4, 5, -1), (8193, 1, 1, -2), (33, 256, 1, -2), (2, 4097, 1, -2),
    (8192, 1, 1, 0), (32, 256, 256, 0)])
def test_merge_abi_shape_checks(H, w, k_out, rc):
  got = _ffi.lib().tfrs_topk_maxsim_merge_f32(None, None, 0, H, w, k_out, None, None, None)
  assert got == rc, _err()
  if rc == -2:
    assert f"H={H}" in _err()


def test_merge_abi_null_pointers_and_negative_q():
  l = _ffi.lib()
  assert l.tfrs_topk_maxsim_merge_f32(None, None, 1, 2, 4, 4, None, None, None) == -1
  assert "NULL" in _err()
  assert l.tfrs_topk_maxsim_merge_f32(None, None, -1, 2, 4, 4, None, None, None) == -1


def test_rowwise_maxsim_abi_checks():
  l = _ffi.lib()
  assert l.tfrs_rowwise_maxsim_f32(None, None, 0, 2, 3, None, None) == 0
  for rows, H, d in ((1, 2, 3), (-1, 2, 3), (1, 0, 3), (1, 2, 0)):
    assert l.tfrs_rowwise_maxsim_f32(None, None, rows, H, d, None, None) == -1


def test_python_limit_names_h():
  ops._maxsim_limit(32, 256)
  ops._maxsim_limit(8192, 1)
  with pytest.raises(NotImplementedError, match="H=33"):
    ops._maxsim_limit(33, 256)


def test_abi_declarations():
  src = open(os.path.join(ROOT, "include", "tfrs_b200.h")).read()
  assert int(re.search(r"#define TFRS_MAXSIM_MAX_ENTRIES (\d+)", src).group(1)) == ops.MAXSIM_MAX_ENTRIES == \
      ops.TC_MAX_K * 32
  for name in ("tfrs_topk_maxsim_merge_f32", "tfrs_rowwise_maxsim_f32"):
    assert re.search(name + r"\s*\(", src), name
    assert name in _ffi.EXPORTS
    assert hasattr(ctypes.CDLL(_ffi.LIB_PATH), name)

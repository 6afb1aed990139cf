"""Which C entry points the top-K host code calls, shape by shape, with the kernels replaced by a recorder (CPU only).

`ops.lib` becomes a recorder that runs the pure planning functions (workspace and index sizes, which decide the
tensor-core range) in the real library and records the name of every other entry point; scratch requests are recorded
as "ws:<slot>".  Tensors stay on the CPU.  The tables pin the routes of BruteForce, Streaming, FactorizedTopK and the
hard-negative loss at every edge of the tensor-core range: the TC_MIN_N corpus floor, d = 128, k = 256, k + E = 256,
the width of Streaming's carried state, the query model, the identifier type and query chunking by TC_MAX_Q_PER_CALL."""
import warnings

import numpy as np
import pytest
import torch

from recommenders_b200 import _ffi, metrics, ops
from recommenders_b200.layers import factorized_top_k as ftk

N0 = ops.TC_MIN_N
N4 = 4 * ops.TC_MIN_N                  # large enough for k = 256 on the tensor cores
Q2 = ops.TC_MAX_Q_PER_CALL + 1         # two query chunks
PLANNING = ("tfrs_topk_tc_workspace_bytes", "tfrs_topk_scan_workspace_bytes", "tfrs_index_bytes")

BUILD = ["tfrs_index_build"]
TC = ["ws:tc", "tfrs_topk_tc_f32"]
SCAN = ["ws:scan", "tfrs_topk_scan_f32"]
EXCL = ["ws:tc", "tfrs_topk_tc_exclude_f32"]
COUNT = ["ws:tc", "tfrs_topk_tc_count_f32"]
MERGE = ["tfrs_topk_merge_strided"]           # _exclude's host path: rank the adjusted scores
MERGE_SORTED = ["tfrs_topk_merge_sorted_strided"]
STREAM_TC = ["ws:stream_index"] + BUILD + TC
HARDNEG_TC = ["ws:hardneg_index"] + BUILD + TC


class _Recorder:

  def __init__(self, real, calls):
    self._real, self._calls = real, calls

  def __getattr__(self, name):
    if name in PLANNING:
      return getattr(self._real, name)

    def launch(*args):
      self._calls.append(name)
      return 0
    return launch


class _Stager:
  """Streaming's host staging without pinned buffers or side streams: the batches are used where they are."""

  def __init__(self, device, rows, d):
    self.device, self.rows, self.d = device, rows, d

  def stage(self, pieces):
    return torch.cat(pieces, 0)

  def release(self):
    pass


@pytest.fixture
def calls(monkeypatch):
  calls = []
  rec = _Recorder(_ffi.lib(), calls)
  monkeypatch.setattr(ops, "lib", lambda: rec)
  monkeypatch.setattr(ops, "f32c", lambda t, name: t.to(torch.float32).contiguous())
  monkeypatch.setattr(ops, "require_cuda", lambda t, name: t)
  monkeypatch.setattr(ops, "workspace",
                      lambda nbytes, device, slot="default": (calls.append("ws:" + slot), torch.empty(0, dtype=torch.uint8))[1])
  monkeypatch.setattr(ops, "stream", lambda: None)
  monkeypatch.setattr(torch, "empty", torch.zeros)      # the recorder writes nothing: outputs hold valid indices
  monkeypatch.setattr(ftk, "_HostStager", _Stager)
  monkeypatch.setattr(ftk.BruteForce, "_warned_slow_path", False)
  return calls


def _run(fn):
  """-> whether fn warned (RuntimeWarning)."""
  with warnings.catch_warnings(record=True) as w:
    warnings.simplefilter("always")
    fn()
  return any(issubclass(x.category, RuntimeWarning) for x in w)


def _ids(kind, n):
  return {None: None, "int": torch.arange(n), "numpy": np.arange(n).astype(str)}[kind]


def _brute(N, d, ids=None, query_model=None, use_tensor_cores=True):
  layer = ftk.BruteForce(query_model=query_model, k=10)
  layer.use_tensor_cores = use_tensor_cores
  return layer.index(torch.zeros(N, d), _ids(ids, N))


# (N, d, Q, k, ids, query model, use_tensor_cores) -> index-time calls, call-time calls, warned
BRUTE_FORCE_CALL = [
    ((N0 - 1, 64, 8, 10, None, False, True), [], SCAN, False),
    ((N0, 64, 8, 10, None, False, True), BUILD, TC, False),
    ((N0, 128, 8, 10, "int", False, True), BUILD, TC, False),
    ((N0, 129, 8, 10, None, False, True), [], SCAN, True),
    ((N0, 64, 8, 65, None, False, True), BUILD, SCAN, True),                  # k above the range of a TC_MIN_N corpus
    ((N4, 64, 8, 256, "numpy", False, True), BUILD, TC, False),
    ((N4, 64, 8, 257, None, False, True), BUILD, SCAN, True),
    ((N0, 64, Q2, 10, None, False, True), BUILD, TC + TC, False),
    ((N0, 64, 8, 10, None, True, True), BUILD, TC, False),
    ((N0, 64, 8, 10, None, False, False), [], SCAN, False),
]


@pytest.mark.parametrize("shape,at_index,at_call,warned", BRUTE_FORCE_CALL)
def test_brute_force_call_routes(calls, shape, at_index, at_call, warned):
  N, d, Q, k, ids, qm, use_tc = shape
  layer = _brute(N, d, ids, torch.nn.Identity() if qm else None, use_tc)
  assert calls == at_index
  calls.clear()
  assert _run(lambda: layer(torch.zeros(Q, d), k=k)) == warned
  assert calls == at_call


# (N, Q, k, E, ids) -> call-time calls
BRUTE_FORCE_EXCLUSIONS = [
    ((N4, 8, 200, 56, None), EXCL),
    ((N4, 8, 200, 57, None), SCAN + MERGE),                                    # k + E = 257: over-fetch, then _exclude
    ((N4, 8, 200, 56, "int"), EXCL),
    ((N4, 8, 200, 56, "numpy"), TC + MERGE),
    ((N0, Q2, 10, 5, None), EXCL + EXCL),
    ((N0, 8, 10, 0, None), TC + MERGE),
    ((N0 - 1, 8, 10, 5, None), SCAN + MERGE),
]


@pytest.mark.parametrize("shape,at_call", BRUTE_FORCE_EXCLUSIONS)
def test_brute_force_exclusion_routes(calls, shape, at_call):
  N, Q, k, E, ids = shape
  layer = _brute(N, 64, ids)
  calls.clear()
  _run(lambda: layer.query_with_exclusions(torch.zeros(Q, 64), torch.zeros(Q, E, dtype=torch.int64), k=k))
  assert calls == at_call


def _streaming(batches, d, ids=None, use_tensor_cores=True):
  layer = ftk.Streaming(k=10)
  layer.use_tensor_cores = use_tensor_cores
  layer._coalesce_rows = 1           # every batch is a chunk of its own
  embs = [torch.zeros(n, d) for n in batches]
  if ids is None:
    return layer.index_from_dataset(embs)
  return layer.index_from_dataset([(_ids(ids, n), e) for n, e in zip(batches, embs)])


# (batch rows, d, Q, k, use_tensor_cores) -> calls
STREAMING_CALL = [
    (([N0 - 1], 64, 8, 10, True), SCAN),
    (([N0], 64, 8, 10, True), STREAM_TC),
    (([N0], 128, 8, 10, True), STREAM_TC),
    (([N0], 129, 8, 10, True), SCAN),
    (([N4], 64, 8, 256, True), STREAM_TC),
    (([N4], 64, 8, 257, True), SCAN),
    (([N0, N0], 64, 8, 10, True), STREAM_TC + STREAM_TC + MERGE_SORTED),      # carried state of width k
    (([N0 - 1, N0], 64, 8, 64, True), SCAN + STREAM_TC + MERGE_SORTED),
    (([50, N0], 64, 8, 64, True), SCAN + SCAN),                                # carried state of width 50: not k
    (([N0], 64, Q2, 10, True), STREAM_TC + TC),
    (([N0], 64, 8, 10, False), SCAN),
]


@pytest.mark.parametrize("shape,at_call", STREAMING_CALL)
def test_streaming_call_routes(calls, shape, at_call):
  batches, d, Q, k, use_tc = shape
  layer = _streaming(batches, d, use_tensor_cores=use_tc)
  assert not _run(lambda: layer(torch.zeros(Q, d), k=k))
  assert calls == at_call


# (batch rows, k, E, ids) -> calls
STREAMING_EXCLUSIONS = [
    (([N0], 10, 5, None), STREAM_TC + ["tfrs_topk_exclude_rerank_f32"]),
    (([N0], 10, 5, "int"), STREAM_TC + MERGE),
    (([N0], 10, 5, "numpy"), STREAM_TC + MERGE),
    (([N0, N0], 50, 5, None), STREAM_TC + STREAM_TC + MERGE_SORTED + ["tfrs_topk_exclude_rerank_f32"]),
    (([N0], 60, 5, None), SCAN + ["tfrs_topk_exclude_rerank_f32"]),           # k + E = 65: above this corpus's range
]


@pytest.mark.parametrize("shape,at_call", STREAMING_EXCLUSIONS)
def test_streaming_exclusion_routes(calls, shape, at_call):
  batches, k, E, ids = shape
  layer = _streaming(batches, 64, ids)
  layer.query_with_exclusions(torch.zeros(8, 64), torch.zeros(8, E, dtype=torch.int64), k=k)
  assert calls == at_call


ROWWISE, HITS, COUNT_ABOVE = ["tfrs_rowwise_dot_f32"], ["tfrs_topk_hits_accumulate"], ["tfrs_count_above_f32"]
# (layer, N, d, Q, max(ks), query model) -> update_state calls
FACTORIZED_TOP_K = [
    (("brute", N0, 64, 8, 10, False), ROWWISE + COUNT + HITS),
    (("brute", N0, 128, 8, 10, False), ROWWISE + COUNT + HITS),
    (("brute", N0, 64, 8, 10, True), ROWWISE + TC + COUNT_ABOVE + HITS),     # the query model must run: no fused count
    (("brute", N0 - 1, 64, 8, 10, False), ROWWISE + SCAN + COUNT_ABOVE + HITS),
    (("brute", N0, 129, 8, 10, False), ROWWISE + SCAN + COUNT_ABOVE + HITS),
    (("brute", N4, 64, 8, 256, False), ROWWISE + COUNT + HITS),
    (("brute", N4, 64, 8, 257, False), ROWWISE + SCAN + COUNT_ABOVE + HITS),
    (("brute", N0, 64, Q2, 10, False), ROWWISE + COUNT + COUNT + HITS),
    (("streaming", N0, 64, 8, 10, False), ROWWISE + STREAM_TC + COUNT_ABOVE + HITS),
]


@pytest.mark.parametrize("shape,at_update", FACTORIZED_TOP_K)
def test_factorized_top_k_update_routes(calls, shape, at_update):
  kind, N, d, Q, kmax, qm = shape
  layer = _brute(N, d, query_model=torch.nn.Identity() if qm else None) if kind == "brute" else _streaming([N], d)
  metric = metrics.FactorizedTopK(layer, ks=(1, kmax))
  calls.clear()
  _run(lambda: metric.update_state(torch.zeros(Q, d), torch.zeros(Q, d)))
  assert calls == at_update


# (C, d, B, num_hard_negatives) -> forward calls
HARD_NEGATIVES = [
    ((N0 - 1, 64, 8, 9), SCAN),
    ((N0, 64, 8, 9), HARDNEG_TC),
    ((N0, 128, 8, 9), HARDNEG_TC),
    ((N0, 129, 8, 9), SCAN),
    ((N4, 64, 8, 255), HARDNEG_TC),
    ((N4, 64, 8, 256), SCAN),
    ((N0, 64, Q2, 9), HARDNEG_TC + TC),
]


@pytest.mark.parametrize("shape,at_forward", HARD_NEGATIVES)
def test_hard_negative_forward_routes(calls, shape, at_forward):
  C, d, B, n = shape
  assert not _run(lambda: ops.hard_negative_softmax_loss(torch.zeros(B, d), torch.zeros(C, d), n))
  assert calls == at_forward + ["tfrs_rowwise_dot_f32", "tfrs_hardneg_loss_fwd"]

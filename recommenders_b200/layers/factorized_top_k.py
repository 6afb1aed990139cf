"""Top-K retrieval layers: the H100 mirror of tensorflow_recommenders/layers/factorized_top_k.py.

Same classes, constructor arguments, method names and error behaviour as the reference
(`TopK` :140-333, `Streaming` :336-512, `BruteForce` :515-610, `ScaNN` stub :613-796), plus `TreeAH`, ScaNN's
algorithm under its own name; tensors are CUDA `torch.Tensor`s and the arithmetic runs in libtfrs_b200.so (exact fp32
scan or wgmma screening + exact rescoring; tree-AH scoring for `TreeAH`).  Results follow tf.math.top_k's contract:
scores descending, ties -> lower index.
"""
from __future__ import annotations

import abc
import os
from typing import Dict, Optional, Text, Tuple, Union

import numpy as np
import torch

from .. import ops
from ..data import Dataset, as_dataset

Tensor = torch.Tensor
Identifiers = Union[torch.Tensor, np.ndarray]


def _wrap_batch_too_small_error(k: int) -> ValueError:
  """factorized_top_k.py:34-54 -- the helpful message for chunks smaller than k."""
  return ValueError(
      "Tried to retrieve k={k} top items, but the candidate "
      "dataset batch size is too small. This may be because "
      "your candidate batch size is too small or the last "
      "batch of your dataset is too small. "
      "To resolve this, increase your batch size, set the "
      "drop_remainder argument to True when batching your "
      "candidates, or set the handle_incomplete_batches "
      "argument to True in the constructor. ".format(k=k))


def _take_along_axis(arr, indices: Tensor):
  """factorized_top_k.py:57-80 -- arr[i, indices[i, j]] for torch tensors or NumPy arrays."""
  if isinstance(arr, np.ndarray):
    return np.take_along_axis(arr, indices.cpu().numpy(), 1)
  return torch.gather(arr, 1, indices)


def _gather_identifiers(identifiers: Identifiers, idx: Tensor):
  """tf.gather(identifiers, indices) (:607, :438): torch ids stay on device, others go through NumPy."""
  if isinstance(identifiers, torch.Tensor):
    return identifiers[idx]
  return np.asarray(identifiers)[idx.cpu().numpy()]


def _exclude(scores: Tensor, identifiers, exclude, k: int):
  """Removes a subset of candidates from top K candidates (factorized_top_k.py:83-115).

  Scores of excluded identifiers are lowered by 1e5, the top min(k, cols) of the adjusted scores are
  taken, and the ORIGINAL scores / identifiers at those positions are returned.  Integer tensor identifiers run
  in one kernel (`tfrs_topk_exclude_rerank_f32`); other identifier types (e.g. NumPy strings) are matched on the
  host and ranked by the merge kernel."""
  if isinstance(identifiers, torch.Tensor) and not identifiers.dtype.is_floating_point and identifiers.is_cuda:
    out_s, out_i = ops.exclude_rerank(scores, identifiers, exclude, k)  # the identifier matrix is its own "index"
    return out_s, out_i.to(identifiers.dtype)
  if isinstance(identifiers, torch.Tensor):
    exclude_t = exclude if isinstance(exclude, torch.Tensor) else torch.as_tensor(np.asarray(exclude))
    isin = (identifiers.unsqueeze(-1) == exclude_t.to(identifiers.device).unsqueeze(1)).any(-1)
  else:
    ex = exclude.cpu().numpy() if isinstance(exclude, torch.Tensor) else np.asarray(exclude)
    isin = torch.from_numpy((np.asarray(identifiers)[:, :, None] == ex[:, None, :]).any(-1)).to(scores.device)
  adjusted = scores - isin.to(torch.float32) * 1.0e5
  k = min(k, scores.shape[1])
  pos = torch.arange(scores.shape[1], device=scores.device, dtype=torch.int64).expand_as(scores)
  _, indices = ops.topk_merge(adjusted.unsqueeze(0), pos.unsqueeze(0), k)  # top_k(adjusted): ties -> lower index
  return _take_along_axis(scores, indices), _take_along_axis(identifiers, indices)


def _check_candidates_with_identifiers(element) -> None:
  """factorized_top_k.py:118-137 -- dataset elements are embeddings or (identifiers, embeddings)."""
  if isinstance(element, tuple):
    if len(element) != 2:
      raise ValueError("The dataset must yield candidate embeddings or "
                       "tuples of (candidate identifiers, candidate embeddings). "
                       f"Got a tuple of length {len(element)} instead.")
    ids, emb = element
    if emb.shape[0] != ids.shape[0]:
      raise ValueError("Candidates and identifiers have to have the same batch dimension. "
                       f"Got {emb.shape[0]} and {ids.shape[0]}.")


def _concat_ids(chunks):
  if isinstance(chunks[0], torch.Tensor):
    return torch.cat(chunks, 0)
  return np.concatenate([np.asarray(c) for c in chunks], 0)


def shard_bounds(num_rows: int, rank: int, world: int) -> Tuple[int, int]:
  """Contiguous row block [lo, hi) of shard `rank`: global index order == (shard, local index) order, so
  the lowest-index tie rule survives the merge."""
  per = (num_rows + world - 1) // world
  lo = min(rank * per, num_rows)
  return lo, min(lo + per, num_rows)


class ShardComm:
  """The C-ABI communicator of the sharded scan (`tfrs_comm_*`, include/tfrs_b200.h).  torch.distributed (any backend)
  is used ONCE, as the control plane that hands rank 0's 128-byte NCCL id to the other ranks; every collective on the
  data path is issued by libtfrs_b200.so itself."""

  def __init__(self, group=None):
    import ctypes
    import torch.distributed as dist
    from .. import _ffi
    self.rank = dist.get_rank(group)
    self.world = dist.get_world_size(group)
    uid = (ctypes.c_char * 128)()
    if self.rank == 0:
      _ffi.check(_ffi.lib().tfrs_comm_unique_id(uid), "comm_unique_id")
    box = [bytes(uid)]
    dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    self._handle = ctypes.c_void_p()
    raw = (ctypes.c_char * 128).from_buffer_copy(box[0])
    _ffi.check(_ffi.lib().tfrs_comm_create(ctypes.byref(self._handle), self.rank, self.world, raw), "comm_create")
    # peer-memory exchange (NVLink stores + epoch flags) instead of the NCCL all-gather; TFRS_SHARD_EXCHANGE=nccl keeps NCCL
    self.p2p = self.world > 1 and os.environ.get("TFRS_SHARD_EXCHANGE", "p2p").lower() != "nccl"
    if os.environ.get("TFRS_SHARD_THRESHOLD_EXCHANGE", "1") == "0":   # A/B switch; must be the same on every rank
      _ffi.check(_ffi.lib().tfrs_comm_set_option(self._handle, 0, 0), "comm_set_option")

  def ensure_p2p(self, Q: int, k: int) -> bool:
    """Maps the exchange buffers for (Q, k) calls if they are not big enough yet (collective: all ranks see the same
    Q, k and therefore take the same decision).  False -> the NCCL all-gather path is used."""
    from .. import _ffi
    if not self.p2p:
      return False
    if _ffi.lib().tfrs_comm_p2p_capacity(self._handle, Q, k):
      return True
    rc = _ffi.lib().tfrs_comm_enable_p2p(self._handle, max(Q, 1024), max(k, 16))
    if rc == -2:          # some peer cannot be mapped: every rank got the same answer
      self.p2p = False
      return False
    _ffi.check(rc, "comm_enable_p2p")
    return True

  @property
  def handle(self):
    return self._handle

  def close(self):
    from .. import _ffi
    if self._handle:
      _ffi.lib().tfrs_comm_destroy(self._handle)
      self._handle = None


class TopK(torch.nn.Module, abc.ABC):
  """Interface for top K layers (factorized_top_k.py:140-333)."""

  def __init__(self, k: int, **kwargs) -> None:
    name = kwargs.pop("name", None)
    super().__init__()
    self._k = k
    self.name = name

  @abc.abstractmethod
  def index(self, candidates: Tensor, identifiers: Optional[Identifiers] = None) -> "TopK":
    raise NotImplementedError()

  def index_from_dataset(self, candidates) -> "TopK":
    """Builds the retrieval index from a dataset of embeddings or (identifier, embedding) batches (:179-215)."""
    ds = as_dataset(candidates)
    elements = list(ds)
    for el in elements:
      _check_candidates_with_identifiers(el)
    if elements and isinstance(elements[0], tuple):
      cands = torch.cat([emb for _, emb in elements], 0)
      identifiers = _concat_ids([ids for ids, _ in elements])
    else:
      cands = torch.cat(elements, 0)
      identifiers = None
    return self.index(cands, identifiers)

  @abc.abstractmethod
  def call(self, queries: Union[Tensor, Dict[Text, Tensor]], k: Optional[int] = None) -> Tuple[Tensor, Tensor]:
    raise NotImplementedError()

  def forward(self, queries, k: Optional[int] = None):
    return self.call(queries, k=k)

  def query_with_exclusions(self, queries, exclusions, k: Optional[int] = None):
    """Query the index, excluding per-query identifiers (:242-288): over-fetch k+E, then `_exclude`."""
    k = k if k is not None else self._k
    adjusted_k = k + exclusions.shape[1]
    x, y = self(queries=queries, k=adjusted_k)
    return _exclude(x, y, exclude=exclusions, k=k)

  def in_top_k_count(self, queries: Tensor, positive_scores: Tensor, k: int) -> Optional[Tensor]:
    """min(k, #{candidates scoring strictly above positive_scores[q]}) per query (int32 [Q]) when the layer can count
    without retrieving a top-k list; None when it cannot, and the caller counts on `self(queries, k=k)` instead."""
    return None

  @abc.abstractmethod
  def is_exact(self) -> bool:
    raise NotImplementedError()

  def _reset_tf_function_cache(self):
    """No tf.function cache exists here (:303-318); kept so subclasses written for the reference still run."""

  def _compute_score(self, queries: Tensor, candidates: Tensor) -> Tensor:
    """The standard dot product score matmul(q, c^T) (:320-333) -- exact fp32."""
    return ops.scores(queries, candidates)


class _HostStager:
  """Pinned, double-buffered host->device staging for corpora that do not live in HBM (SURVEY 8f-1): chunk i+1 is copied
  (cudaMemcpyAsync from pinned memory on a side stream) while chunk i is being scanned."""

  def __init__(self, device: torch.device, rows: int, d: int):
    self.device, self.rows, self.d = device, rows, d
    self.pinned = [torch.empty((rows, d), dtype=torch.float32).pin_memory() for _ in range(2)]
    self.dev = [torch.empty((rows, d), dtype=torch.float32, device=device) for _ in range(2)]
    self.copy_stream = torch.cuda.Stream(device=device)
    self.h2d_done = [torch.cuda.Event(), torch.cuda.Event()]     # the pinned buffer may be refilled after this
    self.scan_done = [torch.cuda.Event(), torch.cuda.Event()]    # the device buffer may be overwritten after this
    self.used = [False, False]
    self.slot = 0
    self.h2d_bytes = 0

  def stage(self, pieces) -> Tensor:
    """pieces: host/device [r_i, d] tensors of one chunk -> one device tensor [sum r_i, d] (valid on the CURRENT stream)."""
    s = self.slot
    self.slot ^= 1
    n = sum(int(p.shape[0]) for p in pieces)
    if self.used[s]:
      self.h2d_done[s].synchronize()            # host: the previous copy out of pinned[s] has finished
      self.copy_stream.wait_event(self.scan_done[s])   # device: the scan that read dev[s] has finished
    # pageable host pieces are packed into the pinned staging buffer (contiguous runs -> one H2D each); pieces that are
    # ALREADY pinned (a corpus kept in page-locked memory) are copied straight from where they are: no host memcpy
    at = 0
    for p in pieces:
      r = int(p.shape[0])
      if not p.is_cuda and not p.is_pinned():
        self.pinned[s][at:at + r].copy_(p)
      at += r
    with torch.cuda.stream(self.copy_stream):
      at = 0
      run0 = None
      for p in pieces + [None]:
        staged_host = p is not None and not p.is_cuda and not p.is_pinned()
        if staged_host and run0 is None:
          run0 = at
        if (not staged_host) and run0 is not None:       # flush the contiguous staged run [run0, at)
          self.dev[s][run0:at].copy_(self.pinned[s][run0:at], non_blocking=True)
          self.h2d_bytes += (at - run0) * self.d * 4
          run0 = None
        if p is not None:
          r = int(p.shape[0])
          if p.is_cuda or p.is_pinned():
            self.dev[s][at:at + r].copy_(p, non_blocking=True)
            if not p.is_cuda:
              self.h2d_bytes += r * self.d * 4
          at += r
      self.h2d_done[s].record(self.copy_stream)
    torch.cuda.current_stream().wait_event(self.h2d_done[s])
    self.used[s] = True
    self._last = s
    return self.dev[s][:n]

  def release(self) -> None:
    """Call after enqueuing the scan of the chunk returned by the last stage()."""
    self.scan_done[self._last].record(torch.cuda.current_stream())


class Streaming(TopK):
  """Retrieves K highest scoring items and their ids from a large dataset (factorized_top_k.py:336-512).

  Dataset batches (the README uses 128 rows) are coalesced into chunks of `_coalesce_rows`; every chunk is scanned by
  the wgmma screening kernel (its fp16 image is built on the fly) with the running row counter as index offset and
  merged into the carried [Q,k] state -- ties resolve to the lower running index, i.e. state first (:462-463), so the
  result equals BruteForce's.  Batches that live in host memory are staged through pinned double buffers so the copy of
  chunk i+1 overlaps the scan of chunk i (corpora larger than HBM).  Small chunks use the exact CUDA-core scan, which
  takes the carried state directly."""

  def __init__(self, query_model: Optional[torch.nn.Module] = None, k: int = 10,
               handle_incomplete_batches: bool = True, num_parallel_calls: Optional[int] = None,
               sorted_order: bool = True) -> None:
    super().__init__(k=k)
    self.query_model = query_model
    self._candidates = None
    self._handle_incomplete_batches = handle_incomplete_batches
    self._num_parallel_calls = num_parallel_calls
    self._sorted = sorted_order
    self._coalesce_rows = 262144
    self.use_tensor_cores = True
    self._stager = None
    self.register_buffer("_counter", torch.zeros((), dtype=torch.int32), persistent=False)

  def index_from_dataset(self, candidates) -> "TopK":
    ds = as_dataset(candidates)
    self._candidates = ds
    return self

  def index(self, candidates, identifiers=None) -> "Streaming":
    """Not implemented. Please call `index_from_dataset` instead (:392-402)."""
    raise NotImplementedError("The streaming top k class only accepts datasets. "
                              "Please call `index_from_dataset` instead.")

  def _run(self, queries, k: int):
    """-> (scores [Q,k'], running row indices [Q,k'] i64, identifier chunks or None)."""
    if self._candidates is None:
      raise ValueError("The `index` method must be called first to create the retrieval index.")
    if self.query_model is not None:
      queries = self.query_model(queries)
    queries = ops.f32c(queries, "queries")
    Q = queries.shape[0]
    state = (torch.zeros((Q, 0), dtype=torch.float32, device=queries.device),
             torch.zeros((Q, 0), dtype=torch.int64, device=queries.device))
    counter = 0
    id_chunks = []
    pending, pending_rows = [], 0

    def flush():
      nonlocal state, counter, pending, pending_rows
      if not pending:
        return
      staged = any(not p.is_cuda for p in pending)
      if staged:   # host-resident corpus: pinned double-buffered H2D, one chunk ahead of the scan
        d = int(pending[0].shape[1])
        st = self._stager
        if st is None or st.d != d or st.device != queries.device or st.rows < pending_rows:
          st = self._stager = _HostStager(queries.device, max(self._coalesce_rows + 65536, pending_rows), d)
        emb = st.stage([p if p.is_cuda else p.to(torch.float32) for p in pending])
      else:
        emb = pending[0] if len(pending) == 1 else torch.cat(pending, 0)
      # state + top-k of the chunk, its rows numbered with the running counter (enumerate_rows, :474-485); the chunk's
      # tensor-core image is built in a per-stream scratch slot
      state = ops.topk(queries, ops.f32c(emb, "candidates"), k, image="stream_index" if self.use_tensor_cores else None,
                       index_offset=counter, state=state)
      if staged:
        self._stager.release()
      counter += int(emb.shape[0])
      pending, pending_rows = [], 0

    for el in self._candidates:
      _check_candidates_with_identifiers(el)
      if isinstance(el, tuple):
        ids, emb = el
        id_chunks.append(ids)
      else:
        emb = el
      if not self._handle_incomplete_batches and emb.shape[0] < k:
        raise _wrap_batch_too_small_error(k)
      # Dataset batches are tiny (README uses 128): coalesce them.  The result is the same as merging per
      # batch -- indices are the running row numbers either way.
      pending.append(emb); pending_rows += int(emb.shape[0])
      if pending_rows >= self._coalesce_rows:
        flush()
    flush()
    self._counter.fill_(counter)
    return state[0], state[1], (id_chunks if id_chunks else None)

  def call(self, queries, k: Optional[int] = None):
    k = k if k is not None else self._k
    scores, idx, id_chunks = self._run(queries, k)
    if id_chunks is not None:
      return scores, _gather_identifiers(_concat_ids(id_chunks), idx)
    return scores, idx.to(torch.int32)

  def query_with_exclusions(self, queries, exclusions, k: Optional[int] = None):
    """:242-288 -- scan for k + E with the carried state, then `_exclude` in one kernel (integer identifiers)."""
    k = k if k is not None else self._k
    scores, idx, id_chunks = self._run(queries, k + exclusions.shape[1])
    if id_chunks is None:
      s, i = ops.exclude_rerank(scores, idx, exclusions, k)
      return s, i.to(torch.int32)
    ids = _concat_ids(id_chunks)
    if isinstance(ids, torch.Tensor) and not ids.dtype.is_floating_point and ids.is_cuda:
      s, i = ops.exclude_rerank(scores, idx, exclusions, k, identifiers=ids)
      return s, ids[i]
    return _exclude(scores, _gather_identifiers(ids, idx), exclude=exclusions, k=k)

  def is_exact(self) -> bool:
    return True


class BruteForce(TopK):
  """Brute force retrieval (factorized_top_k.py:515-610).

  `index` keeps the fp32 corpus and, for large corpora, builds the fp16 tensor-core screening image;
  `call` returns exactly the top-k of the fp32 scores either way.  `index_shard` adds the row-sharded
  multi-GPU mode: every rank scans its contiguous shard, ONE all-gather of the per-shard (score, index)
  lists (issued by libtfrs_b200.so through its own NCCL communicator) is merged on every rank."""

  def __init__(self, query_model: Optional[torch.nn.Module] = None, k: int = 10, name: Optional[Text] = None):
    super().__init__(k=k, name=name)
    self.query_model = query_model
    self._candidates = None
    self._identifiers = None
    self._tc_index = None
    self._shard = None  # (global_offset, ShardComm)
    self.use_tensor_cores = True

  _warned_slow_path = False

  def index(self, candidates: Tensor, identifiers: Optional[Identifiers] = None) -> "BruteForce":
    if identifiers is None:
      identifiers_ = None
      n_ids = candidates.shape[0]
    else:
      identifiers_ = identifiers
      n_ids = identifiers.shape[0]
    if candidates.dim() != 2:
      raise ValueError(f"The candidates tensor must be 2D (got {tuple(candidates.shape)}).")
    if candidates.shape[0] != n_ids:
      raise ValueError("The candidates and identifiers tensors must have the same number of"
                       f" rows (got {candidates.shape[0]} candidates rows and"
                       f" {n_ids} identifier rows). ")
    self._set_index(ops.f32c(candidates, "candidates").detach(), identifiers_)
    self._shard = None
    self._reset_tf_function_cache()
    return self

  def index_shard(self, local_candidates: Tensor, global_offset: int, identifiers: Optional[Identifiers] = None,
                  group=None, comm: Optional[ShardComm] = None, copy: bool = True) -> "BruteForce":
    """Row-sharded index: this rank owns corpus rows [global_offset, global_offset + len(local_candidates)).
    `identifiers`, when given, covers the WHOLE corpus (it is only used to map the merged indices).  Collective:
    every rank of `group` must call it (the C-ABI communicator is created here unless `comm` is passed)."""
    if local_candidates.dim() != 2:
      raise ValueError(f"The candidates tensor must be 2D (got {tuple(local_candidates.shape)}).")
    self._set_index(ops.f32c(local_candidates, "candidates").detach(), identifiers, copy=copy)
    self._shard = (int(global_offset), comm if comm is not None else ShardComm(group))
    return self

  def _set_index(self, cands: Tensor, identifiers, copy: bool = True) -> None:
    # the index OWNS its corpus (the reference copies with .assign(), :571-580): later in-place updates of the
    # caller's tensor (e.g. an Embedding.weight that keeps training) must not desynchronise the fp32 rows from
    # the fp16 screening image built from them
    if copy:
      cands = cands.clone()
    self._candidates = cands
    self._identifiers = identifiers
    self._tc_index = None
    if self.use_tensor_cores and cands.shape[0] >= ops.TC_MIN_N and cands.shape[1] <= 128:
      self._tc_index = ops.index_build(cands)

  def _tc_ok(self, Q: int, k: int) -> bool:
    return self._tc_index is not None and ops.uses_tc_scan(Q, self._candidates.shape[0], self._candidates.shape[1], k)

  def _local_topk(self, queries: Tensor, k: int, offset: int, out=None):
    n, d = self._candidates.shape
    if (self.use_tensor_cores and n >= ops.TC_MIN_N and not BruteForce._warned_slow_path and
        not self._tc_ok(queries.shape[0], k)):
      # same results, ~20x slower: say so once instead of silently leaving the tensor-core path
      BruteForce._warned_slow_path = True
      import warnings
      warnings.warn(f"BruteForce: a {n} x {d} corpus with k={k} is outside the tensor-core scan's range (d <= 128, k <= "
                    f"{ops.TC_MAX_K}, corpus >= ~256*k rows); running the exact CUDA-core scan instead (same results, "
                    "roughly 20x slower).", RuntimeWarning, stacklevel=3)
    return ops.topk(queries, self._candidates, k, image=self._tc_index, index_offset=offset, out=out)

  def in_top_k_count(self, queries: Tensor, positive_scores: Tensor, k: int) -> Optional[Tensor]:
    """Counted inside the tensor-core scan (`tfrs_topk_tc_count_f32`) when the index is unsharded and has no query
    model, so `queries` are already the embeddings the corpus is scored against."""
    if self._candidates is None or self._shard is not None or self.query_model is not None:
      return None
    k = min(k, self._candidates.shape[0])
    if not self._tc_ok(queries.shape[0], k):
      return None
    return ops.topk_tc_count(queries, self._candidates, self._tc_index, k, positive_scores)

  def call(self, queries, k: Optional[int] = None):
    k = k if k is not None else self._k
    if self._candidates is None:
      raise ValueError("The `index` method must be called first to create the retrieval index.")
    if self.query_model is not None:
      queries = self.query_model(queries)
    if self._shard is None:
      n_total = self._candidates.shape[0]
      if k > n_total:
        raise ValueError(f"input must have at least k columns. Had {n_total}, needed {k}")
      values, indices = self._local_topk(queries, k, 0)
    else:
      values, indices = self._sharded_topk(queries, k)
    if self._identifiers is None:
      return values, indices.to(torch.int32)  # default identifiers = range(N) int32 (:544-545)
    return values, _gather_identifiers(self._identifiers, indices)

  def query_with_exclusions(self, queries, exclusions, k: Optional[int] = None):
    """:242-288.  On the tensor-core path the exclusion test runs inside the scan's finalize step
    (`tfrs_topk_tc_exclude_f32`): no [Q, k+E] list round trip, no eager ops."""
    k = k if k is not None else self._k
    E = int(exclusions.shape[1])
    ids = self._identifiers
    int_ids = ids is None or (isinstance(ids, torch.Tensor) and not ids.dtype.is_floating_point)
    if (self._candidates is not None and self._shard is None and int_ids and E > 0 and
        k + E <= self._candidates.shape[0]):
      q = self.query_model(queries) if self.query_model is not None else queries
      if self._tc_ok(q.shape[0], k + E):
        s, i = ops.topk_tc_exclude(q, self._candidates, self._tc_index, k, exclusions, identifiers=ids)
        if ids is None:
          return s, i.to(torch.int32)
        return s, _gather_identifiers(ids, i)
    return super().query_with_exclusions(queries, exclusions, k)

  def _sharded_topk(self, queries: Tensor, k: int):
    """The whole sharded call is ONE C-ABI entry point (`tfrs_topk_sharded_f32`): local scan written straight into the
    send block -> one NCCL all-gather -> sorted-list merge reading the receive buffer in place."""
    offset, comm = self._shard
    return ops.topk_sharded(comm, queries, self._candidates, self._tc_index, k, offset)

  def is_exact(self) -> bool:
    return True

  # -- checkpointing: the index is model state (reference keeps it as non-trainable weights, :562-580)
  def get_extra_state(self):
    ids = self._identifiers
    return {"candidates": None if self._candidates is None else self._candidates.cpu(),
            "identifiers": ids.cpu() if isinstance(ids, torch.Tensor) else ids}

  def set_extra_state(self, state):
    if state and state.get("candidates") is not None:
      dev = torch.device("cuda", torch.cuda.current_device())
      ids = state.get("identifiers")
      if isinstance(ids, torch.Tensor):
        ids = ids.to(dev)
      self.index(state["candidates"].to(dev), ids)


class ScaNN(TopK):
  """ScaNN approximate retrieval lives in the un-vendored `scann` pip package (factorized_top_k.py:25-31);
  as in the reference without that package, constructing it raises ImportError (:675-679)."""

  def __init__(self, *args, **kwargs):
    raise ImportError("The scann library is not present. Please install it using `pip install scann` to use "
                      "the ScaNN layer.")

  def index(self, candidates, identifiers=None):  # pragma: no cover
    raise NotImplementedError()

  def call(self, queries, k=None):  # pragma: no cover
    raise NotImplementedError()

  def is_exact(self) -> bool:  # pragma: no cover
    return False


class TreeAH(TopK):
  """Tree-AH approximate retrieval: the algorithm of the reference's ScaNN layer (factorized_top_k.py:613-796) on K9.

  Takes ScaNN's constructor arguments and defaults, so `ScaNN(` -> `TreeAH(` moves code over.  `index` trains a k-means
  tree of `num_leaves` leaves and 4-bit codebooks of the residuals (`dimensions_per_block` dims per code); `call` scores
  the rows of the best `num_leaves_to_search` leaves with int8 lookup tables and, when `num_reordering_candidates` is
  set, rescores that many survivors with the exact fp32 dot.  Every rule is pinned in DESIGN.md §2; parity with the
  scann package itself is not.  `parallelize_batch_searches` is accepted and has no effect: batches always run as one
  call on the GPU."""

  def __init__(self, query_model: Optional[torch.nn.Module] = None, k: int = 10, distance_measure: Text = "dot_product",
               num_leaves: int = 100, num_leaves_to_search: int = 10, training_iterations: int = 12,
               dimensions_per_block: int = 2, num_reordering_candidates: Optional[int] = None,
               parallelize_batch_searches: bool = True, name: Optional[Text] = None):
    super().__init__(k=k, name=name)
    if distance_measure == "squared_l2":
      raise NotImplementedError("TreeAH supports distance_measure='dot_product' only.")
    if distance_measure != "dot_product":
      raise ValueError(f"Unknown distance_measure {distance_measure!r}; expected 'dot_product'.")
    for arg, v in (("k", k), ("num_leaves", num_leaves), ("num_leaves_to_search", num_leaves_to_search),
                   ("num_reordering_candidates", num_reordering_candidates)):
      if v is not None and v <= 0:
        raise ValueError(f"{arg} must be positive, got {v}.")
    if training_iterations < 0:
      raise ValueError(f"training_iterations must be non-negative, got {training_iterations}.")
    if not 1 <= dimensions_per_block <= 8:
      raise ValueError(f"dimensions_per_block must be in 1..8, got {dimensions_per_block}.")
    for arg, v in (("k", k), ("num_leaves_to_search", num_leaves_to_search),
                   ("num_reordering_candidates", num_reordering_candidates)):
      if v is not None and v > ops.TREE_AH_MAX_K:
        raise ValueError(f"{arg} must be at most {ops.TREE_AH_MAX_K}, got {v}.")
    self.query_model = query_model
    self._num_leaves = num_leaves
    self._num_leaves_to_search = num_leaves_to_search
    self._training_iterations = training_iterations
    self._dpb = dimensions_per_block
    self._num_reordering_candidates = num_reordering_candidates
    self._parallelize_batch_searches = parallelize_batch_searches
    self._index = None       # ops.tree_ah_build's tensors
    self._rows = None        # fp32 rows, kept only for reordering
    self._identifiers = None

  def index(self, candidates: Tensor, identifiers: Optional[Identifiers] = None) -> "TreeAH":
    if candidates.dim() != 2:
      raise ValueError(f"The candidates tensor must be 2D (got {tuple(candidates.shape)}).")
    if identifiers is not None and candidates.shape[0] != identifiers.shape[0]:
      raise ValueError("The candidates and identifiers tensors must have the same number of"
                       f" rows (got {candidates.shape[0]} candidates rows and"
                       f" {identifiers.shape[0]} identifier rows). ")
    n, d = candidates.shape
    if not 1 <= d <= 256:
      raise ValueError(f"TreeAH needs 1 <= d <= 256, got d={d}.")
    if not 1 <= n < ops.TREE_AH_MAX_ROWS:
      raise ValueError(f"TreeAH needs 1 <= N < 2^24 candidates, got {n}.")
    cands = ops.f32c(candidates, "candidates").detach()
    self._index = ops.tree_ah_build(cands, self._num_leaves, self._training_iterations, self._dpb)
    self._rows = cands.clone() if self._num_reordering_candidates is not None else None
    self._identifiers = identifiers
    self._reset_tf_function_cache()
    return self

  def call(self, queries, k: Optional[int] = None):
    k = k if k is not None else self._k
    if self._index is None:
      raise ValueError("The `index` method must be called first to create the retrieval index.")
    if self.query_model is not None:
      queries = self.query_model(queries)
    if not isinstance(queries, torch.Tensor):
      raise ValueError(f"Queries must be a tensor, got {type(queries)}.")
    if queries.dim() not in (1, 2):
      raise ValueError(f"Queries must be of rank 2 or 1, got {queries.dim()}.")
    if not 1 <= k <= ops.TREE_AH_MAX_K:
      raise ValueError(f"k must be in 1..{ops.TREE_AH_MAX_K}, got {k}.")
    q = queries.unsqueeze(0) if queries.dim() == 1 else queries
    k_pre = max(self._num_reordering_candidates or k, k)
    # every size (d, dimensions per block, L, N) is taken from the index tensors, which ops checks against the queries
    scores, idx = ops.tree_ah_search(q, self._index, self._rows, self._num_leaves_to_search, k, k_pre)
    if queries.dim() == 1:
      scores, idx = scores[0], idx[0]
    if self._identifiers is None:
      return scores, idx.to(torch.int32)
    return scores, _gather_identifiers(self._identifiers, idx)

  def is_exact(self) -> bool:
    return False

  # -- checkpointing: the trained index is model state (the reference serializes its searcher into the module, :728-730)
  def get_extra_state(self):
    ids = self._identifiers
    return {"index": None if self._index is None else {n: t.cpu() for n, t in self._index.items()},
            "rows": None if self._rows is None else self._rows.cpu(),
            "identifiers": ids.cpu() if isinstance(ids, torch.Tensor) else ids}

  def set_extra_state(self, state):
    if state and state.get("index") is not None:
      if (state.get("rows") is not None) != (self._num_reordering_candidates is not None):
        raise ValueError("The saved TreeAH index was built " + ("with" if state.get("rows") is not None else "without") +
                         " reordering rows; construct the layer with the same num_reordering_candidates setting "
                         "(None or not None) to restore it.")
      dev = torch.device("cuda", torch.cuda.current_device())
      self._index = {n: t.to(dev) for n, t in state["index"].items()}
      self._rows = None if state.get("rows") is None else state["rows"].to(dev)
      ids = state.get("identifiers")
      self._identifiers = ids.to(dev) if isinstance(ids, torch.Tensor) else ids

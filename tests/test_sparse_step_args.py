"""The argument checks of the sparse and dense optimizer steps.

The library: every tfrs_sparse_*_f32 entry point runs ag_check_args (csrc/adagrad.cu) before its first CUDA call, so a
bad argument is refused without a device, with TFRS_ERR_INVALID_ARG and a message that starts with the entry point's
name.  The four optimizers that sum runs also refuse d > 1024 before any launch; SGD has no such limit.

The Python wrappers (ops._sparse_step_args, ops._dense_step_args): a refused call raises ValueError before any launch and
leaves every state tensor as it was.  Their device rules are host-side, so the CPU cases reach them with CPU and meta
tensors (the CUDA-only rule and the library lifted); the GPU cases cover the shape and length rules on real tensors.
"""
import ctypes

import pytest
import torch

gpu = pytest.mark.gpu

SPARSE = ("sparse_sgd", "sparse_adagrad", "sparse_clippy_adagrad", "sparse_adam", "sparse_ftrl")
INVALID_ARG = -1


# ------------------------------------------------------------------------------------------------
# The library's checks, without a device
# ------------------------------------------------------------------------------------------------
def _call(name, ws, table, slot, rows, d, ids, ids_dtype, n, grad):
  """One call of the entry point `name`; `slot` stands for every slot of the optimizer.  The workspace is large enough
  and the scalars are valid, so only the arguments given here can be refused."""
  from recommenders_b200 import _ffi
  l = _ffi.lib()
  common = (rows, d, ids, ids_dtype, n, grad)
  ws = (ws, 1 << 40, None)
  if name == "sparse_sgd":
    return l.tfrs_sparse_sgd_f32(table, *common, 0.1, *ws)
  if name == "sparse_adagrad":
    return l.tfrs_sparse_adagrad_f32(table, slot, *common, 0.1, 1e-7, 1, *ws)
  if name == "sparse_clippy_adagrad":
    return l.tfrs_sparse_clippy_adagrad_f32(table, slot, *common, 0.1, 1e-7, 0.1, 0.0, 1e-7, 0, None, *ws)
  if name == "sparse_adam":
    return l.tfrs_sparse_adam_f32(table, slot, slot, *common, 1e-3, 0.9, 0.999, 1e-7, 0, *ws)
  return l.tfrs_sparse_ftrl_f32(table, slot, slot, *common, 0.1, -0.5, 0.0, 0.0, 0.0, *ws)


def _bad_arguments(name):
  """(what, overrides, text in the message) of every single-argument refusal the entry point makes."""
  cases = [("NULL table", dict(table=None), "bad table"),
           ("rows 0", dict(rows=0), "bad table"),
           ("d 0", dict(d=0), "bad table"),
           ("ids_dtype", dict(ids_dtype=2), "ids_dtype must be I32 or I64"),
           ("n 2^24", dict(n=1 << 24), "n=16777216 must be < 2^24"),
           ("n < 0", dict(n=-1), "must be < 2^24"),
           ("rows 2^40", dict(rows=1 << 40), "rows must be < 2^40"),
           ("NULL ids", dict(ids=None), "NULL ids/grad"),
           ("NULL grad", dict(grad=None), "NULL ids/grad")]
  if name != "sparse_sgd":
    cases += [("NULL slot", dict(slot=None), "bad table"), ("d 1025", dict(d=1025), "d=1025 > 1024")]
  return cases


@pytest.mark.parametrize("name", SPARSE)
def test_sparse_entry_points_refuse_each_bad_argument(name):
  from recommenders_b200 import _ffi
  buf = ctypes.create_string_buffer(256)   # stands for every pointer: a refused call reads no memory
  ptr = ctypes.addressof(buf)
  good = dict(ws=ptr, table=ptr, slot=ptr, rows=100, d=64, ids=ptr, ids_dtype=_ffi.I32, n=8, grad=ptr)
  for what, over, text in _bad_arguments(name):
    rc = _call(name, **dict(good, **over))
    msg = _ffi.last_error()
    assert rc == INVALID_ARG, (name, what, rc, msg)
    assert msg.startswith(name + ": ") and text in msg, (name, what, msg)


# ------------------------------------------------------------------------------------------------
# The wrappers' device rules, on the host
# ------------------------------------------------------------------------------------------------
@pytest.fixture
def host_ops(monkeypatch):
  """ops with the CUDA-only rule lifted and the library replaced by a stub that fails the test when it is reached."""
  from recommenders_b200 import _ffi, ops

  def no_library():
    raise AssertionError("the call reached the library")

  monkeypatch.setattr(_ffi, "require_cuda", lambda t, name: t)
  monkeypatch.setattr(ops, "require_cuda", lambda t, name: t)
  monkeypatch.setattr(ops, "lib", no_library)
  return ops


def _sparse_calls(ops, table, slots, ids, g):
  """name -> a call of the sparse wrapper with these tensors (`slots` as many as it takes)."""
  rule_c = dict(lr=0.1, eps=1e-7, variable_relative_threshold=0.1, accumulator_relative_threshold=0.0,
                absolute_threshold=1e-7)
  return {
      "sparse_sgd_": lambda: ops.sparse_sgd_(table, ids, g, 0.1),
      "sparse_adagrad_": lambda: ops.sparse_adagrad_(table, slots[0], ids, g, 0.1),
      "sparse_clippy_adagrad_": lambda: ops.sparse_clippy_adagrad_(table, slots[0], ids, g, **rule_c),
      "sparse_adam_": lambda: ops.sparse_adam_(table, slots[0], slots[1], ids, g, 1e-3, 0.9, 0.999, 1e-7),
      "sparse_ftrl_": lambda: ops.sparse_ftrl_(table, slots[0], slots[1], ids, g, 0.1, -0.5, 0.0, 0.0, 0.0),
  }


@pytest.mark.parametrize("wrapper", ["sparse_sgd_", "sparse_adagrad_", "sparse_clippy_adagrad_", "sparse_adam_",
                                     "sparse_ftrl_"])
def test_sparse_wrappers_refuse_tensors_on_another_device(host_ops, wrapper):
  table = torch.zeros((10, 4))
  slots = [torch.full((10, 4), 0.1), torch.zeros((10, 4))]
  ids, g = torch.zeros(3, dtype=torch.int64), torch.ones((3, 4))
  other = torch.device("meta")
  cases = [("ids and grad_rows", (slots, ids.to(other), g)),   # (message, wrapper arguments)
           ("ids and grad_rows", (slots, ids, g.to(other)))]
  if wrapper != "sparse_sgd_":
    cases.append((r"must be \(10, 4\) on cpu, got \(10, 4\) on meta", ([s.to(other) for s in slots], ids, g)))
  for text, (ss, i, gg) in cases:
    with pytest.raises(ValueError, match=text):
      _sparse_calls(host_ops, table, ss, i, gg)[wrapper]()
  assert torch.count_nonzero(table) == 0 and bool((slots[0] == 0.1).all()) and torch.count_nonzero(slots[1]) == 0


def test_sgd_dense_refuses_tensors_on_another_device(host_ops):
  p, q = torch.zeros(5), torch.zeros((2, 3))
  with pytest.raises(ValueError, match="one device"):
    host_ops.sgd_dense_([p, q], [torch.ones(5), torch.ones((2, 3), device="meta")], 0.1)
  with pytest.raises(ValueError, match="one device"):
    host_ops.sgd_dense_([p, q.to("meta")], [torch.ones(5), torch.ones((2, 3), device="meta")], 0.1)
  assert torch.count_nonzero(p) == 0 and torch.count_nonzero(q) == 0


# ------------------------------------------------------------------------------------------------
# The wrappers' shape and length rules, on the device
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


def _unchanged(before, after):
  torch.cuda.synchronize()
  return all(torch.equal(a, b) for a, b in zip(before, after))


@gpu
def test_sparse_adagrad_refuses_an_accumulator_of_another_shape(ops):
  table = torch.rand((10, 4), device="cuda")
  ids = torch.tensor([0, 9, 9], device="cuda")
  g = torch.ones((3, 4), device="cuda")
  for accum in (torch.full((5, 4), 0.1, device="cuda"), torch.full((10, 5), 0.1, device="cuda"),
                torch.full((40,), 0.1, device="cuda")):
    state = [table, accum]
    before = [t.clone() for t in state]
    with pytest.raises(ValueError, match="accum must be"):
      ops.sparse_adagrad_(table, accum, ids, g, 0.1)
    assert _unchanged(before, state)


@gpu
def test_sparse_sgd_takes_grad_rows_of_exactly_n_by_d(ops):
  table = torch.rand((10, 4), device="cuda")
  ids = torch.tensor([0, 9, 9, 3], device="cuda")
  before = table.clone()
  for g in (torch.ones(16, device="cuda"), torch.ones((4, 2, 2), device="cuda"), torch.ones((2, 8), device="cuda"),
            torch.ones((8, 2), device="cuda")):
    with pytest.raises(ValueError, match="grad_rows must be"):
      ops.sparse_sgd_(table, ids, g, 0.1)
    assert _unchanged([before], [table])


@gpu
def test_sgd_dense_refuses_lists_of_different_lengths(ops):
  ps = [torch.rand(5, device="cuda"), torch.rand((2, 3), device="cuda")]
  before = [p.clone() for p in ps]
  with pytest.raises(ValueError, match="same length"):
    ops.sgd_dense_(ps, [torch.ones(5, device="cuda")], 0.1)
  with pytest.raises(ValueError, match="same length"):
    ops.sgd_dense_(ps[:1], [torch.ones(5, device="cuda"), torch.ones((2, 3), device="cuda")], 0.1)
  assert _unchanged(before, ps)

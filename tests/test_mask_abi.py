"""The C ABI refuses a Keras mask of an unknown kind (TFRS_CHECK_MASK, csrc/common.cuh).

Every masked entry point checks its masks before it returns early for an empty batch, so these calls (B = 0, a dummy
mask pointer that is never read) need no device: with the check missing, the bad kind would return TFRS_OK like the
good one does.  tfrs_batch_norm_* is left out: it refuses N = 0 before the mask, so a missing check would reach a launch.
"""
import ctypes

import pytest

from recommenders_b200 import _ffi, ops

INVALID_ARG = -1
BAD_KIND = 99
MASK = ctypes.c_void_p(0x1000)


def _masks(struct, which, kind):
  """byref(struct) with the mask `which` set to the dummy pointer and `kind`."""
  s = struct()
  setattr(s, which, MASK)
  setattr(s, which + "_kind", kind)
  return ctypes.byref(s)


# name -> call(lib, kind) with B = 0 and the smallest valid other sizes
CALLS = {
    "mean_pool_fwd": lambda l, k: l.tfrs_mean_pool_fwd(None, 0, 1, 1, 1, 1, 1, MASK, k, None, None),
    "mean_pool_bwd": lambda l, k: l.tfrs_mean_pool_bwd(None, 0, 1, 1, MASK, k, None, None),
    "gru_fwd": lambda l, k: l.tfrs_gru_fwd_f32(None, None, None, None, MASK, k, 0, 1, 1, None, None, None, None, None),
    "gru_bwd": lambda l, k: l.tfrs_gru_bwd_f32(None, None, None, MASK, k, None, None, 0, 1, 1, None, None, None, None,
                                               None, 0, None),
    "lstm_fwd": lambda l, k: l.tfrs_lstm_fwd_f32(None, None, None, None, MASK, k, 0, 1, 1, None, None, None, None, None,
                                                 None, None),
    "lstm_bwd": lambda l, k: l.tfrs_lstm_bwd_f32(None, None, None, None, None, MASK, k, None, None, None, 0, 1, 1, None,
                                                 None, None, None, None, 0, None),
}
for _w in ("query", "value", "key", "attention"):
  CALLS[f"mha_fwd-{_w}"] = lambda l, k, w=_w: l.tfrs_mha_fwd_f32(
      None, None, None, _masks(ops._MhaMasks, w, k), 0, 1, 1, 1, 1, 1, None, None, None, None)
  CALLS[f"mha_bwd-{_w}"] = lambda l, k, w=_w: l.tfrs_mha_bwd_f32(
      None, None, None, _masks(ops._MhaMasks, w, k), None, None, None, 0, 1, 1, 1, 1, 1, None, None, None, None,
      0, None)
for _w in ("query_mask", "value_mask"):
  CALLS[f"dense_attention_fwd-{_w}"] = lambda l, k, w=_w: l.tfrs_dense_attention_fwd_f32(
      None, None, None, _masks(ops._DenseAttentionDesc, w, k), 0, 1, 1, 1, 1, None, None, None, None)
  CALLS[f"dense_attention_bwd-{_w}"] = lambda l, k, w=_w: l.tfrs_dense_attention_bwd_f32(
      None, None, None, _masks(ops._DenseAttentionDesc, w, k), None, None, None, 0, 1, 1, 1, 1, None, None, None, None,
      None, None, 0, None)


@pytest.mark.parametrize("name", sorted(CALLS))
def test_an_unknown_mask_kind_is_refused_before_the_empty_batch_return(name):
  l = _ffi.lib()
  assert CALLS[name](l, _ffi.BOOL) == 0, _ffi.last_error()
  assert CALLS[name](l, BAD_KIND) == INVALID_ARG
  assert "I32, I64 or BOOL" in _ffi.last_error()

"""layers.StringLookup / IntegerLookup on the H100 (K15, csrc/lookup.cu): every output equal to the dict oracle
(tests/lookup_oracle.py) bit for bit.  The crafted vocabularies of lookup_oracle.int_case / string_case give probe chains
of >= 3 slots and chains that wrap past the last slot (tests/test_lookup_host.py checks that rule)."""
import io

import numpy as np
import pytest
import torch

import lookup_oracle as lo
from recommenders_b200 import ops
from recommenders_b200.layers.embedding import Embedding
from recommenders_b200.layers.preprocessing import IntegerLookup, StringLookup

pytestmark = pytest.mark.gpu
INT64_MIN, INT64_MAX = lo.INT64_MIN, lo.INT64_MAX
I32_MIN, I32_MAX = -2**31, 2**31 - 1
EDGES = [0, -1, INT64_MIN, INT64_MAX]


def _dev():
  return torch.device("cuda", torch.cuda.current_device())


def _cuda(a, dtype=torch.int64):
  return torch.from_numpy(np.ascontiguousarray(a)).to(_dev()).to(dtype)


def _lookup_np(values, vocab, mask=None, oov=1):
  """The dict oracle's rule, vectorised for large vocabularies (sorted keys + searchsorted)."""
  v = np.asarray(vocab, np.int64)
  x = np.asarray(values, np.int64)
  m = 0 if mask is None else 1
  order = np.argsort(v, kind="stable")
  sv = v[order]
  p = np.minimum(np.searchsorted(sv, x), max(len(sv) - 1, 0))
  hit = (sv[p] == x) if len(sv) else np.zeros(x.shape, bool)
  out = np.where(hit, m + oov + order[p], m)
  if mask is not None:
    out[x == mask] = 0
  return out


def _shapes(x: np.ndarray):
  n = x.size
  yield x[:0]
  yield x
  if n % 4 == 0:
    yield x.reshape(n // 4, 4)
    yield x.reshape(2, n // 8, 4) if n % 8 == 0 else x.reshape(1, n // 4, 4)


# ---- integers ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [1, 2, 31, 32, 33, 1000])
def test_integer_cases_match_the_oracle(V):
  vocab, oov = lo.int_case(V)
  oov_token = -5 if -5 not in vocab else 5
  layer = IntegerLookup(vocabulary=vocab, oov_token=oov_token)
  x = np.concatenate([vocab, oov, EDGES, vocab[::-1]]).astype(np.int64)
  x = np.concatenate([x, x[: (-len(x)) % 8]])
  for s in _shapes(x):
    got = layer(_cuda(s))
    assert got.dtype == torch.int64 and tuple(got.shape) == s.shape
    assert np.array_equal(got.cpu().numpy(), lo.lookup(s, vocab.tolist(), None, 1)), (V, s.shape)
  # NumPy input, uploaded once, gives the same
  assert np.array_equal(layer(x).cpu().numpy(), lo.lookup(x, vocab.tolist()))


def test_integer_mask_zero_and_oov_minus_one():
  vocab, oov = lo.int_case(1000, seed=3)
  vocab = vocab[~np.isin(vocab, [0, -1])]
  layer = IntegerLookup(vocabulary=vocab, mask_token=0, oov_token=-1)
  x = np.concatenate([vocab, oov, EDGES, [0, 0, -1]]).astype(np.int64)
  got = layer(_cuda(x)).cpu().numpy()
  assert np.array_equal(got, lo.lookup(x, vocab.tolist(), 0, 1))
  assert got[-3] == 0 and got[-1] == 1 and layer.vocabulary_size() == len(vocab) + 2


def test_int32_inputs():
  rng = np.random.RandomState(1)
  vocab = np.unique(rng.randint(I32_MIN, I32_MAX, size=5000).astype(np.int64))[:4000]
  vocab = rng.permutation(np.concatenate([vocab[~np.isin(vocab, [0, -1, I32_MIN, I32_MAX])], [I32_MIN, I32_MAX, 0]]))
  layer = IntegerLookup(vocabulary=vocab)
  x = np.concatenate([vocab, rng.randint(I32_MIN, I32_MAX, size=3000), [0, -1, I32_MIN, I32_MAX]]).astype(np.int32)
  for s in _shapes(x[: len(x) // 8 * 8]):
    got = layer(_cuda(s, torch.int32))
    assert np.array_equal(got.cpu().numpy(), lo.lookup(s, vocab.tolist()))


@pytest.mark.parametrize("V", [1 << 20, 10 * (1 << 20)])
def test_large_integer_vocabularies_uniform_and_zipf(V):
  rng = np.random.RandomState(V % 997)
  keys = np.unique(rng.randint(INT64_MIN, INT64_MAX, size=V + V // 8, dtype=np.int64))
  vocab = rng.permutation(keys)[:V]
  layer = IntegerLookup(vocabulary=_cuda(vocab))              # a CUDA vocabulary
  B = 65536
  uniform = np.where(rng.rand(B) < 0.9, vocab[rng.randint(0, V, size=B)], rng.randint(INT64_MIN, INT64_MAX, size=B,
                                                                                       dtype=np.int64))
  zipf = vocab[(rng.zipf(1.2, size=B) - 1) % V]
  for x in (uniform, zipf):
    assert np.array_equal(layer(_cuda(x)).cpu().numpy(), _lookup_np(x, vocab))


# ---- strings ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [1, 2, 16, 33, 1000])
@pytest.mark.parametrize("mask", [None, "MASK"])
def test_string_cases_match_the_oracle(V, mask):
  vocab, oov = lo.string_case(V)
  layer = StringLookup(vocabulary=vocab, mask_token=mask)
  words = vocab + oov + ([mask] if mask else []) + vocab[::-1]
  words += words[: (-len(words)) % 8]
  x = np.array(words, dtype=object)
  for s in _shapes(x):
    exp = lo.lookup(s, vocab, mask, 1, strings=True)
    got = layer(s)
    assert got.dtype == torch.int64 and tuple(got.shape) == s.shape
    assert np.array_equal(got.cpu().numpy(), exp), (V, s.shape)
    # str against bytes inputs: the same values
    enc = np.array([w.encode() for w in s.reshape(-1)], dtype=object).reshape(s.shape)
    assert np.array_equal(layer(enc).cpu().numpy(), exp)
  assert np.array_equal(layer(list(words)).cpu().numpy(), lo.lookup(words, vocab, mask, 1, True))


def test_string_empty_mask_and_bytes_vocabulary():
  vocab, oov = lo.string_case(1000, seed=2)
  vocab = [v for v in vocab if v != ""]
  bvocab = [v.encode() for v in vocab]
  layer = StringLookup(vocabulary=np.array(bvocab, dtype=object), mask_token="")
  words = vocab + oov + ["", ""]
  got = layer(np.array(words)).cpu().numpy()
  assert np.array_equal(got, lo.lookup(words, vocab, "", 1, True))
  assert got[-1] == 0


def test_large_string_vocabulary():
  rng = np.random.RandomState(5)
  V, B = 1 << 20, 65536
  lens = rng.randint(8, 65, size=V)
  vocab = [f"{i:07d}:" + "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789 éü"[: n - 8] for i, n in
           enumerate(lens)]
  layer = StringLookup(vocabulary=np.array(vocab))
  pos = rng.randint(0, V, size=B)
  x = np.array([vocab[p] if p % 10 else vocab[p][:-1] + "#" for p in pos])   # 10 % OOV, same length
  assert np.array_equal(layer(x).cpu().numpy(), lo.lookup(x, vocab, None, 1, True))


# ---- invert, o = 0, duplicates, determinism, checkpoints, launches ---------------------------------------------------
def test_invert_round_trips():
  vocab, oov = lo.int_case(1000, seed=4)
  vocab = vocab[~np.isin(vocab, [0, -1])]
  fwd = IntegerLookup(vocabulary=vocab, mask_token=0)
  inv = IntegerLookup(vocabulary=vocab, mask_token=0, invert=True)
  x = np.concatenate([vocab, oov, [0]]).astype(np.int64)
  idx = fwd(_cuda(x))
  back = inv(idx)
  assert back.dtype == torch.int64 and back.is_cuda
  assert back.cpu().numpy().tolist() == lo.invert(idx.cpu().numpy(), vocab.tolist(), 0, -1)
  odd = np.array([-5, 0, 1, 2, len(vocab) + 1, len(vocab) + 2, INT64_MAX, INT64_MIN], np.int64)
  assert inv(_cuda(odd)).cpu().numpy().tolist() == lo.invert(odd, vocab.tolist(), 0, -1)
  assert inv(_cuda(np.clip(odd, I32_MIN, I32_MAX), torch.int32)).cpu().numpy().tolist() == \
      lo.invert(np.clip(odd, I32_MIN, I32_MAX), vocab.tolist(), 0, -1)

  svocab, soov = lo.string_case(1000, seed=4)
  for kind_vocab in (svocab, [v.encode() for v in svocab]):
    sinv = StringLookup(vocabulary=np.array(kind_vocab, dtype=object), mask_token="MASK", invert=True)
    sfwd = StringLookup(vocabulary=np.array(kind_vocab, dtype=object), mask_token="MASK")
    words = svocab + soov + ["MASK"]
    idx = sfwd(np.array(words))
    out = sinv(idx)
    kind = "S" if isinstance(kind_vocab[0], bytes) else "U"
    tok = (lambda t: t.encode()) if kind == "S" else (lambda t: t)
    assert isinstance(out, np.ndarray) and out.dtype.kind == kind
    assert out.tolist() == lo.invert(idx.cpu().numpy(), kind_vocab, tok("MASK"), tok("[UNK]"))
    assert sinv(odd).tolist() == lo.invert(odd, kind_vocab, tok("MASK"), tok("[UNK]"))


def test_no_oov_index_raises_on_oov_only():
  vocab, oov = lo.int_case(33)
  layer = IntegerLookup(vocabulary=vocab, num_oov_indices=0, oov_token=7 if 7 not in vocab else 8)
  assert np.array_equal(layer(_cuda(vocab)).cpu().numpy(), np.arange(len(vocab)))
  with pytest.raises(ValueError):
    layer(_cuda(np.concatenate([vocab, oov[:1]])))
  svocab, soov = lo.string_case(33)
  s = StringLookup(vocabulary=svocab, num_oov_indices=0, mask_token="MASK")
  assert np.array_equal(s(np.array(svocab + ["MASK"])).cpu().numpy(), np.r_[np.arange(1, 34), 0])
  with pytest.raises(ValueError):
    s(np.array(svocab[:3] + soov[-1:]))


def test_duplicate_vocabularies_raise():
  with pytest.raises(ValueError):
    IntegerLookup(vocabulary=[3, INT64_MIN, 3])
  with pytest.raises(ValueError):
    IntegerLookup(vocabulary=_cuda(np.array([5, 6, 7, 5])))
  with pytest.raises(ValueError):
    StringLookup(vocabulary=["a", "z" * 1024, "b", "z" * 1024])
  with pytest.raises(ValueError):
    StringLookup(vocabulary=np.array(["é", "x", "é"]))
  # equal prefixes and lengths are not duplicates
  StringLookup(vocabulary=["ab" * 12 + "c", "ab" * 12 + "d", "z" * 1023 + "a", "z" * 1023 + "b"])


def test_repeated_calls_and_rebuilt_tables_are_byte_identical():
  vocab, oov = lo.string_case(1000, seed=6)
  words = np.array(vocab + oov)
  layer = StringLookup(vocabulary=vocab)
  a = layer(words).cpu().numpy()
  assert np.array_equal(a, layer(words).cpu().numpy())
  layer.set_vocabulary(vocab)
  assert np.array_equal(a, layer(words).cpu().numpy())
  assert np.array_equal(a, StringLookup(vocabulary=vocab)(words).cpu().numpy())
  ivocab, ioov = lo.int_case(1000, seed=6)
  x = _cuda(np.concatenate([ivocab, ioov]))
  first = IntegerLookup(vocabulary=ivocab, oov_token=-7)(x).cpu().numpy()
  for _ in range(3):
    assert np.array_equal(first, IntegerLookup(vocabulary=ivocab, oov_token=-7)(x).cpu().numpy())


def test_state_dict_restore():
  vocab, oov = lo.string_case(1000, seed=7)
  tower = torch.nn.Sequential(StringLookup(vocabulary=vocab, mask_token=None), Embedding(len(vocab) + 1, 8))
  buf = io.BytesIO()
  torch.save(tower.state_dict(), buf)
  buf.seek(0)
  fresh = torch.nn.Sequential(StringLookup(mask_token=None), Embedding(len(vocab) + 1, 8))
  fresh.load_state_dict(torch.load(buf, weights_only=True))
  words = np.array(vocab + oov)
  with torch.no_grad():
    assert torch.equal(tower(words), fresh(words))
  ivocab, _ = lo.int_case(1000, seed=7)
  il = IntegerLookup(vocabulary=ivocab, oov_token=-7)
  buf = io.BytesIO()
  torch.save(il.state_dict(), buf)
  buf.seek(0)
  again = IntegerLookup(oov_token=-7)
  again.load_state_dict(torch.load(buf, weights_only=True))
  x = _cuda(np.concatenate([ivocab, [1, 2, 3]]))
  assert torch.equal(il(x), again(x)) and again.get_vocabulary() == il.get_vocabulary()


def test_one_launch_per_call_and_empty_inputs():
  vocab, oov = lo.int_case(1000)
  layer = IntegerLookup(vocabulary=vocab, oov_token=-7)
  x = _cuda(np.concatenate([vocab, oov]))
  layer(x)
  for inp in (x, x.to(torch.int32)):
    c0 = ops.launch_count()
    layer(inp)
    assert ops.launch_count() - c0 == 1
  zero = IntegerLookup(vocabulary=vocab, num_oov_indices=0, oov_token=-7)
  c0 = ops.launch_count()
  zero(_cuda(vocab))
  assert ops.launch_count() - c0 == 1
  svocab, soov = lo.string_case(1000)
  s = StringLookup(vocabulary=svocab)
  s(np.array(svocab))
  c0 = ops.launch_count()
  s(np.array(svocab + soov))
  assert ops.launch_count() - c0 == 1
  assert tuple(layer(_cuda(np.zeros((0, 3), np.int64))).shape) == (0, 3)
  assert tuple(s(np.zeros((0,), "U1")).shape) == (0,) and tuple(s([]).shape) == (0,)

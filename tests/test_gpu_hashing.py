"""tf-keras `Hashing` on the GPU (K18): `ops.hashing` and `layers.Hashing` byte-equal to the C oracle
(tests/hashing_oracle.c) for every FarmHash branch and tail length at every start alignment, both hashes, masks, every
decimal-length boundary of int32 / int64 values, shapes, and one launch per call."""
import numpy as np
import pytest
import torch

import hashing_oracle as ho
import unified_oracle as uo

pytestmark = pytest.mark.gpu

INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
NUM_BINS = [1, 2, 3, 200_000, 2**31 + 11, 2**63 - 1]
ABCDE = ["A", "B", "C", "D", "E"]


@pytest.fixture(scope="module")
def tfrs():
  import recommenders_b200 as t
  return t


def _strings(seed=0):
  """Random bytes of every length 0..300 (0x00, 0xFF and everything between), plus multi-byte UTF-8."""
  rng = np.random.default_rng(seed)
  strs = [rng.integers(0, 256, size=k, dtype=np.uint8).tobytes() for k in range(301)]
  strs += [b"\x00" * 17, b"\xff" * 65, b"\x00\xff" * 40, "日本語 héllo wörld ✓".encode(), ("é" * 50).encode()]
  return strs


def _device_pair(strs, shift=0):
  """The packed strings as CUDA (bytes, offsets), every string moved `shift` bytes into the byte buffer."""
  data, off = uo.pack(strs)
  junk = np.full(shift, 0xA5, np.uint8)
  buf = np.concatenate([junk, data[:int(off[-1])]]) if off[-1] or shift else np.zeros(1, np.uint8)
  return torch.from_numpy(buf).cuda(), torch.from_numpy(off + shift).cuda()


@pytest.mark.parametrize("shift", range(16))
def test_every_length_at_every_alignment(tfrs, shift):
  strs = _strings(shift)
  pair = _device_pair(strs, shift)
  for num_bins in (2**63 - 1, 200_000):
    got = tfrs.ops.hashing(pair, num_bins).cpu().numpy()
    np.testing.assert_array_equal(got, ho.hashing(strs, num_bins))
  salt = [shift, 2**64 - 1 - shift]
  got = tfrs.ops.hashing(pair, 2**63 - 1, salt=salt).cpu().numpy()
  np.testing.assert_array_equal(got, ho.hashing(strs, 2**63 - 1, salt=salt))


@pytest.mark.parametrize("num_bins", NUM_BINS)
def test_strings_every_num_bins(tfrs, num_bins):
  strs = _strings(100)
  pair = _device_pair(strs, 3)
  np.testing.assert_array_equal(tfrs.ops.hashing(pair, num_bins).cpu().numpy(), ho.hashing(strs, num_bins))
  for salt in (133, [133, 137]):
    got = tfrs.ops.hashing(pair, num_bins, salt=salt).cpu().numpy()
    np.testing.assert_array_equal(got, ho.hashing(strs, num_bins, salt=salt))
    # the salted route is tfrs_hash_bins's
    np.testing.assert_array_equal(got, tfrs.ops.hash_bins(pair, num_bins, salt).cpu().numpy())


def _int_edges():
  e = [0, -1, 1, INT64_MIN, INT64_MAX, INT64_MIN + 1, INT32_MIN, INT32_MAX]
  for k in range(19):
    p = 10**k
    e += [p, p - 1, -p, -(p - 1), p + 1, -(p + 1)]
  e += [10**18 * 9, -10**18 * 9]
  return np.array(sorted(set(v for v in e if INT64_MIN <= v <= INT64_MAX)), np.int64)


@pytest.mark.parametrize("num_bins", NUM_BINS)
def test_integers_every_decimal_length(tfrs, num_bins):
  rng = np.random.default_rng(num_bins % 1000)
  v64 = np.concatenate([_int_edges(), rng.integers(INT64_MIN, INT64_MAX, size=50_000, dtype=np.int64)])
  v32 = v64[(v64 >= INT32_MIN) & (v64 <= INT32_MAX)].astype(np.int32)
  for v in (v64, v32):
    x = torch.from_numpy(v).cuda()
    for salt in (None, [7, 2**64 - 1]):
      got = tfrs.ops.hashing(x, num_bins, salt=salt).cpu().numpy()
      np.testing.assert_array_equal(got, ho.hashing(v.astype(np.int64), num_bins, salt=salt))
    # the layer: a CUDA tensor, NumPy ints and a list of Python ints
    layer = tfrs.layers.Hashing(num_bins)
    exp = ho.hashing(v.astype(np.int64), num_bins)
    np.testing.assert_array_equal(layer(x).cpu().numpy(), exp)
    np.testing.assert_array_equal(layer(v).cpu().numpy(), exp)
  np.testing.assert_array_equal(tfrs.layers.Hashing(num_bins)(v64[:40].tolist()).cpu().numpy(),
                                ho.hashing(v64[:40], num_bins))


@pytest.mark.parametrize("num_bins", [1, 2, 3, 200_000, 2**63 - 1])
def test_masks(tfrs, num_bins):
  v = _int_edges()
  for mask in (0, -1, INT64_MIN, INT64_MAX, 12345):
    exp = ho.hashing(v, num_bins, mask=mask)
    if num_bins > 1 and mask in v:
      assert (exp[v == mask] == 0).all() and (exp[v != mask] >= 1).all()
    for salt in (None, 9):
      got = tfrs.ops.hashing(torch.from_numpy(v).cuda(), num_bins, salt=salt, mask=mask).cpu().numpy()
      np.testing.assert_array_equal(got, ho.hashing(v, num_bins, salt=salt, mask=mask))
    np.testing.assert_array_equal(tfrs.layers.Hashing(num_bins, mask_value=mask)(torch.from_numpy(v).cuda()).cpu().numpy(), exp)
    v32 = v[(v >= INT32_MIN) & (v <= INT32_MAX)]
    got = tfrs.layers.Hashing(num_bins, mask_value=mask)(torch.from_numpy(v32.astype(np.int32)).cuda()).cpu().numpy()
    np.testing.assert_array_equal(got, ho.hashing(v32, num_bins, mask=mask))
  strs = ["", "A", "B", "", "[UNK]", "A\x00b", "日本", "x" * 70] + [f"w{k}" for k in range(50)]
  for mask in ("", "A", "[UNK]", "A\x00b", "日本", "x" * 70, "absent", b"B"):
    for salt in (None, [1, 2]):
      exp = ho.hashing(strs, num_bins, salt=salt, mask=mask)
      got = tfrs.layers.Hashing(num_bins, mask_value=mask, salt=salt)(strs).cpu().numpy()
      np.testing.assert_array_equal(got, exp)
      m = np.frombuffer(ho._as_bytes(mask), np.uint8).copy()
      got = tfrs.ops.hashing(_device_pair(strs, 5), num_bins, salt=salt, mask=torch.from_numpy(m).cuda()).cpu().numpy()
      np.testing.assert_array_equal(got, exp)
  if num_bins == 1:
    assert not tfrs.layers.Hashing(1, mask_value="")(strs).any()


def test_doc_examples_on_the_device(tfrs):
  H = tfrs.layers.Hashing
  assert H(num_bins=3)(ABCDE).tolist() == [1, 0, 1, 1, 2]
  assert H(num_bins=3, mask_value="")(["A", "B", "", "C", "D"]).tolist() == [1, 1, 0, 2, 2]
  assert H(num_bins=3)(np.array(["Hello", "TensorFlow", "2.x"])).tolist() == [0, 2, 2]
  assert H(num_bins=3, salt=133)(np.array(ABCDE)).tolist() == [0, 0, 2, 1, 0]
  assert H(num_bins=3, salt=[133, 137])([[s] for s in ABCDE]).tolist() == [[1], [2], [1], [0], [2]]
  # str and bytes are the same value
  assert H(num_bins=3)([s.encode() for s in ABCDE]).tolist() == [1, 0, 1, 1, 2]


def test_layer_on_strings_of_every_length(tfrs):
  rng = np.random.default_rng(9)
  # no trailing NUL: NumPy's fixed-width bytes drop it, as for StringLookup
  strs = [bytes(rng.integers(1, 256, size=k, dtype=np.uint8)) for k in range(301)]
  for salt in (None, 77):
    got = tfrs.layers.Hashing(2**63 - 1, salt=salt)(strs).cpu().numpy()
    np.testing.assert_array_equal(got, ho.hashing(strs, 2**63 - 1, salt=salt))
  words = ["zürich", "日本語", "✓✓✓", "Ωmega" * 20]
  np.testing.assert_array_equal(tfrs.layers.Hashing(1000)(words).cpu().numpy(), ho.hashing(words, 1000))


def test_shapes(tfrs):
  layer = tfrs.layers.Hashing(1000, mask_value=3)
  rng = np.random.default_rng(4)
  for shape in [(7,), (7, 1), (5, 6), (2, 3, 4)]:
    v = rng.integers(0, 10, size=shape)
    out = layer(torch.from_numpy(v).cuda())
    assert out.dtype == torch.int64 and out.is_cuda and tuple(out.shape) == shape
    np.testing.assert_array_equal(out.cpu().numpy(), ho.hashing(v, 1000, mask=3))
    s = np.char.mod("s%d", v)
    out = tfrs.layers.Hashing(1000, mask_value="s3")(s)
    assert tuple(out.shape) == shape
    np.testing.assert_array_equal(out.cpu().numpy(), ho.hashing(s, 1000, mask="s3"))
  for empty in (torch.zeros((0,), dtype=torch.int64, device="cuda"), torch.zeros((3, 0), dtype=torch.int32, device="cuda"),
                np.zeros((0,), "U1"), np.zeros((0, 2), "S1"), []):
    out = layer(empty) if not (isinstance(empty, np.ndarray) and empty.dtype.kind in "US") else \
        tfrs.layers.Hashing(5)(empty)
    assert out.numel() == 0 and tuple(out.shape) == tuple(np.shape(empty)) and out.dtype == torch.int64
  # a non-contiguous CUDA tensor
  v = torch.from_numpy(rng.integers(-10**9, 10**9, size=(64, 8))).cuda()
  np.testing.assert_array_equal(layer(v.t()).cpu().numpy(), ho.hashing(v.t().cpu().numpy(), 1000, mask=3))


def test_one_launch_per_call(tfrs):
  x = torch.arange(4096, device="cuda")
  for layer in (tfrs.layers.Hashing(600), tfrs.layers.Hashing(600, salt=5, mask_value=7)):
    layer(x)
    torch.cuda.synchronize()
    c0 = tfrs.ops.launch_count()
    layer(x)
    assert tfrs.ops.launch_count() == c0 + 1
  c0 = tfrs.ops.launch_count()
  tfrs.layers.Hashing(600, mask_value="")(["a", "", "b"])
  assert tfrs.ops.launch_count() == c0 + 1


def test_input_errors(tfrs):
  layer = tfrs.layers.Hashing(10)
  with pytest.raises(TypeError):
    layer(torch.rand(4, device="cuda"))
  with pytest.raises(TypeError):
    layer(torch.arange(4))
  with pytest.raises(TypeError):
    tfrs.layers.Hashing(10, mask_value="a")(torch.arange(4, device="cuda"))
  with pytest.raises(TypeError):
    tfrs.layers.Hashing(10, mask_value=1)(["a"])
  with pytest.raises(ValueError):
    tfrs.ops.hashing(torch.arange(4, device="cuda"), 0)

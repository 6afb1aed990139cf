"""layers.TextVectorization (K16, csrc/text.cu), Discretization, Normalization and GlobalAveragePooling1D (K17,
csrc/features.cu) on the H100: every output equal to the oracle (tests/text_oracle.py) bit for bit."""
import io

import numpy as np
import pytest
import torch

import text_oracle as to
from recommenders_b200 import ops
from recommenders_b200.data import Dataset
from recommenders_b200.layers.embedding import Embedding
from recommenders_b200.layers.pooling import GlobalAveragePooling1D
from recommenders_b200.layers.preprocessing import Discretization, Normalization, TextVectorization

pytestmark = pytest.mark.gpu


def _vec(tv, strings, osl=None, flags=(True, True)):
  got = tv(strings).cpu().numpy()
  flat = np.asarray(strings, dtype=object).reshape(-1).tolist()
  exp = to.vectorize(flat, tv.get_vocabulary(include_special_tokens=False), osl, *flags)
  assert got.dtype == np.int64 and got.shape == exp.shape, (got.shape, exp.shape)
  assert np.array_equal(got, exp)
  return got


def _same_bits(a, b):
  """Bit-equal float32 arrays; two NaNs count as equal whatever their payloads (0/0 gives different ones on the GPU and
  on the host)."""
  a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
  assert a.shape == b.shape
  nan = np.isnan(a)
  assert np.array_equal(nan, np.isnan(b)), np.argwhere(nan != np.isnan(b))[:5]
  ai, bi = a.view(np.int32)[~nan], b.view(np.int32)[~nan]
  assert np.array_equal(ai, bi), (a[~nan][ai != bi][:5], b[~nan][ai != bi][:5])


# ---- TextVectorization -----------------------------------------------------------------------------------------------
def test_known_answers():
  k = to.KNOWN_ADAPT
  tv = TextVectorization(max_tokens=k["max_tokens"], output_sequence_length=k["output_sequence_length"])
  tv.adapt(k["adapt"])
  assert tv.get_vocabulary() == ["", "[UNK]", "foo", "baz", "bar"]
  assert tv(np.array(k["inputs"])).cpu().tolist() == k["expected"]
  k = to.KNOWN_VOCAB
  tv = TextVectorization(vocabulary=k["vocabulary"])
  assert tv(np.array(k["inputs"])).cpu().tolist() == k["expected"]


@pytest.mark.parametrize("standardize", [None, "lower", "strip_punctuation", "lower_and_strip_punctuation"])
def test_every_ascii_byte_and_look_alikes(standardize):
  flags = (standardize in ("lower", "lower_and_strip_punctuation"), standardize in ("strip_punctuation",
                                                                                    "lower_and_strip_punctuation"))
  strings = [bytes([c]) + b"x" + bytes([c]) + b"Y" for c in range(1, 128)]          # every ASCII byte inside a token
  strings += [b"a" + bytes([c]) + b"b" for c in range(128, 256)]
  strings += ["a\x1cb\x1dc\x1ed\x1fe", "a b", "a　b", "a\u0085b", "ÉCOLE CafÉ Ωmega", "!!! ... ???", "",
              "Don't stop", "a.b a - b", " \t\n\v\f\r ", "x\t\ty\r\nz"]
  strings = [to.as_bytes(s) for s in strings]
  vocab = sorted({t for s in strings for t in to.tokens(s, *flags)})[::2]
  tv = TextVectorization(standardize=standardize, vocabulary=np.array(vocab, dtype=object))
  _vec(tv, np.array(strings, dtype=object), flags=flags)
  tv3 = TextVectorization(standardize=standardize, vocabulary=np.array(vocab, dtype=object), output_sequence_length=3)
  _vec(tv3, np.array(strings, dtype=object), osl=3, flags=flags)


def test_empty_strings_and_empty_batches():
  tv = TextVectorization(vocabulary=["a"])
  assert tuple(tv(np.array(["", " ", "..."])).shape) == (3, 0)                     # every string empty: T = 0
  assert tv(np.array(["", "a"])).cpu().tolist() == [[0], [2]]
  assert tuple(tv(np.array([], dtype="U1")).shape) == (0, 0)
  assert tuple(TextVectorization(output_sequence_length=5, vocabulary=["a"])(np.array([], dtype="U1")).shape) == (0, 5)
  assert TextVectorization(output_sequence_length=2, vocabulary=["a"])(["", "..."]).cpu().tolist() == [[0, 0], [0, 0]]


def test_register_edge_lengths():
  """Standardized tokens of 22, 23 and 24 bytes (SipHash's register / memory edge) from longer raw strings."""
  rng = np.random.RandomState(0)
  strings, vocab = [], []
  for n in (21, 22, 23, 24, 25):
    for _ in range(4):
      tok = "".join(rng.choice(list("abcdefghij"), n))
      raw = "".join(c.upper() + ("." if rng.rand() < 0.5 else "") for c in tok)         # raw length > n
      strings.append(f"{raw} {tok[:-1]}! {tok}X")
      vocab.append(tok)
  tv = TextVectorization(vocabulary=vocab[::2] + [v + "x" for v in vocab[1::2]])
  _vec(tv, np.array(strings))


def test_megabyte_string_and_sequence_lengths():
  rng = np.random.RandomState(1)
  words = [f"w{i}" for i in range(500)]
  big = " ".join(rng.choice(words, 250_000))[:1 << 20]
  tv = TextVectorization(vocabulary=words[:300])
  for osl in (None, 1, 7, 300_000):
    tvo = TextVectorization(vocabulary=words[:300], output_sequence_length=osl)
    _vec(tvo, np.array([big, "w1 w2", ""]), osl)
  # [B] and [B, 1], str and bytes give the same result
  a = np.array(["w1 W2. w999", "w3"])
  r = _vec(tv, a)
  assert np.array_equal(tv(a.reshape(-1, 1)).cpu().numpy(), r)
  assert np.array_equal(tv(np.char.encode(a, "utf-8")).cpu().numpy(), r)
  assert np.array_equal(tv(a.tolist()).cpu().numpy(), r)


@pytest.mark.parametrize("V", [1, 10, 10_000, 1_000_000])
def test_vocabulary_sizes_with_oov(V):
  rng = np.random.RandomState(V)
  vocab = np.array([f"t{i:x}" for i in rng.permutation(2 * V)[:V]])
  strings = [" ".join(f"t{j:x}" for j in rng.randint(0, 2 * V, size=rng.randint(0, 12))) for _ in range(2048)]
  tv = TextVectorization(vocabulary=vocab)
  _vec(tv, np.array(strings))
  _vec(TextVectorization(vocabulary=vocab, output_sequence_length=5), np.array(strings), 5)


def test_adapt_from_arrays_and_datasets():
  rng = np.random.RandomState(2)
  words = ["Alpha", "beta", "GAMMA.", "delta!", "eps", "zeta", "Ωmega", "a-b", "x_y"]
  titles = np.array([" ".join(rng.choice(words, rng.randint(1, 6))) + f" ({1950 + i % 40})" for i in range(3000)])
  exp = [t.decode() for t in to.adapt_vocabulary(titles.tolist(), 30)]
  tvs = []
  for data in (titles, titles.tolist(), Dataset.from_tensor_slices(titles), Dataset.from_tensor_slices(titles).batch(128),
               Dataset.from_tensor_slices(titles.reshape(-1, 1)).batch(100)):
    tv = TextVectorization(max_tokens=30)
    tv.adapt(data)
    assert tv.get_vocabulary(include_special_tokens=False) == exp
    tvs.append(tv)
  _vec(tvs[0], titles[:500])
  one = TextVectorization()
  one.adapt(Dataset.from_batches([np.array(t) for t in titles[:50]]))       # a Dataset of scalars
  assert one.get_vocabulary(include_special_tokens=False) == [t.decode() for t in to.adapt_vocabulary(titles[:50].tolist())]


def test_state_dict_restore_and_launch_counts():
  tv = TextVectorization(max_tokens=100, output_sequence_length=6)
  tv.adapt(["the cat sat", "the dog ran", "a cat ran"])
  buf = io.BytesIO()
  torch.save(tv.state_dict(), buf)
  buf.seek(0)
  tv2 = TextVectorization(max_tokens=100, output_sequence_length=6)
  tv2.load_state_dict(torch.load(buf, weights_only=True))
  x = np.array(["The cat ran.", "a dog?", "unknown words here"])
  assert torch.equal(tv(x), tv2(x))
  torch.cuda.synchronize()
  n0 = ops.launch_count()
  tv(x)
  assert ops.launch_count() - n0 == 2
  n0 = ops.launch_count()
  TextVectorization(vocabulary=["a"])(x)
  assert ops.launch_count() - n0 == 2 + 2          # the table build (fingerprints + inserts), then the call


# ---- Discretization --------------------------------------------------------------------------------------------------
def test_discretization_timestamps_near_float32_boundaries():
  lo, hi = 874724710, 893286638                      # MovieLens 100K's timestamp range
  bounds = np.linspace(lo, hi, num=1000)
  d = Discretization(bounds.tolist())
  b32 = bounds.astype(np.float32).astype(np.int64)
  x = (b32[:, None] + np.arange(-64, 65)[None, :]).reshape(-1)
  assert np.array_equal(d(torch.from_numpy(x).cuda()).cpu().numpy(), to.bucketize(x, bounds))
  assert np.array_equal(d(x.reshape(1000, 129)).cpu().numpy(), to.bucketize(x, bounds).reshape(1000, 129))
  # the float32 rule differs from an exact comparison for some of these
  assert (to.bucketize(x, bounds) != np.searchsorted(bounds, x, side="right")).any()
  xi = np.random.RandomState(0).randint(-2 ** 31, 2 ** 31 - 1, size=10000).astype(np.int32)
  d2 = Discretization(np.linspace(-2e9, 2e9, 101).tolist())
  assert np.array_equal(d2(torch.from_numpy(xi).cuda()).cpu().numpy(), to.bucketize(xi, np.linspace(-2e9, 2e9, 101)))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_discretization_floats_inf_nan_equal_and_empty(dtype):
  rng = np.random.RandomState(3)
  bounds = [-1.0, 0.0, 0.0, 0.1, 1e-30, 1.0 + 2 ** -30, 2.0, 2.0, 1e30]
  bounds = sorted(bounds, key=np.float32)
  x = np.concatenate([rng.randn(5000) * 3, np.float64(bounds), np.nextafter(np.float64(bounds), np.inf),
                      [np.inf, -np.inf, np.nan, -0.0, 0.0, 2 ** -30]]).astype(dtype)
  for b in (bounds, [], [0.5], np.linspace(-5, 5, 20000).tolist()):        # 20000 > the shared-memory stage
    d = Discretization(b)
    got = d(torch.from_numpy(x).cuda())
    assert got.dtype == torch.int64 and np.array_equal(got.cpu().numpy(), to.bucketize(x, b))


# ---- Normalization ---------------------------------------------------------------------------------------------------
def test_normalization_known_answer_and_given_statistics():
  k = to.KNOWN_NORMALIZATION
  n = Normalization(axis=None)
  n.adapt(np.array(k["adapt"]))
  assert n(np.array(k["inputs"])).cpu().tolist() == np.float32(k["expected"]).tolist()
  n2 = Normalization(axis=None, mean=k["mean"], variance=k["variance"])
  assert n2(np.array(k["inputs"])).cpu().tolist() == np.float32(k["expected"]).tolist()
  inv = Normalization(axis=None, mean=k["mean"], variance=k["variance"], invert=True)
  _same_bits(inv(n2(np.array(k["inputs"]))).cpu(), to.normalize(to.normalize(np.array(k["inputs"]), 3.0, 2.0), 3.0, 2.0,
                                                                 True))


def test_normalization_adapt_array_and_dataset():
  rng = np.random.RandomState(4)
  ts = rng.randint(874724710, 893286638, size=10_000).astype(np.int64)
  n = Normalization(axis=None)
  n.adapt(ts)                                            # batches of 32
  m, v = to.adapt_moments(to.array_batches(ts, 32), 1)
  _same_bits(n.mean.cpu(), m)
  _same_bits(n.variance.cpu(), v)
  _same_bits(n(ts).cpu(), to.normalize(ts, m[0], v[0]))
  n128 = Normalization(axis=None)
  n128.adapt(Dataset.from_tensor_slices(ts).batch(128))  # one batch per element
  m2, v2 = to.adapt_moments(to.array_batches(ts, 128), 1)
  _same_bits(n128.mean.cpu(), m2)
  _same_bits(n128.variance.cpu(), v2)
  nt = Normalization(axis=None)
  nt.adapt(torch.from_numpy(ts).cuda(), batch_size=1000)
  m3, v3 = to.adapt_moments(to.array_batches(ts, 1000), 1)
  _same_bits(nt.mean.cpu(), m3)
  torch.cuda.synchronize()
  c0 = ops.launch_count()
  Normalization(axis=None).adapt(ts)
  assert ops.launch_count() - c0 == 2


def test_normalization_zero_variance_last_axis_and_invert():
  x = np.full((100,), 7.0, np.float32)
  n = Normalization(axis=None)
  n.adapt(x, batch_size=128)                               # one batch: the variance is exactly 0
  assert n.variance.item() == 0.0
  _same_bits(n(np.array([7.0, 8.0], np.float32)).cpu(), to.normalize(np.array([7.0, 8.0]), 7.0, 0.0))   # / 1e-7
  rng = np.random.RandomState(5)
  x = (rng.randn(333, 4, 5) * [1, 10, 100, 1e-3, 0]).astype(np.float64)
  n = Normalization(axis=-1)
  n.adapt(x)
  m, v = to.adapt_moments(to.array_batches(x, 32), 5)
  _same_bits(n.mean.cpu(), m)
  _same_bits(n.variance.cpu(), v)
  y = n(x).cpu().numpy()
  _same_bits(y, to.normalize(x, m, v))
  inv = Normalization(axis=-1, mean=m, variance=v, invert=True)
  _same_bits(inv(torch.from_numpy(y).cuda()).cpu(), to.normalize(y, m, v, True))
  for dt in (np.int32, np.int64, np.float32):
    xi = (rng.randn(64, 3) * 1000).astype(dt)
    nn = Normalization(axis=-1)
    nn.adapt(xi)
    mi, vi = to.adapt_moments(to.array_batches(xi, 32), 3)
    _same_bits(nn.mean.cpu(), mi)
    _same_bits(nn(xi).cpu(), to.normalize(xi, mi, vi))
  buf = io.BytesIO()
  torch.save(n.state_dict(), buf)
  buf.seek(0)
  n2 = Normalization(axis=-1)
  n2.load_state_dict(torch.load(buf, weights_only=True))
  assert torch.equal(n2(x), n(x))


# ---- GlobalAveragePooling1D ------------------------------------------------------------------------------------------
def _pool_case(B, T, d, seed):
  rng = np.random.RandomState(seed)
  x = rng.randn(B, T, d).astype(np.float32)
  ids = rng.randint(0, 4, size=(B, T)) * rng.randint(0, 2, size=(B, T))
  ids[0] = 0                                              # an all-masked row
  return x, ids


@pytest.mark.parametrize("mask_kind", ["ids64", "ids32", "bool", "none"])
@pytest.mark.parametrize("B,T,d", [(7, 5, 3), (64, 13, 32), (3, 1, 1), (5, 0, 4)])
def test_pooling_forward_backward(mask_kind, B, T, d):
  x, ids = _pool_case(B, T, d, B * T + d)
  mask = {"ids64": torch.from_numpy(ids).cuda(), "ids32": torch.from_numpy(ids.astype(np.int32)).cuda(),
          "bool": torch.from_numpy(ids != 0).cuda(), "none": None}[mask_kind]
  m = None if mask is None else ids
  xt = torch.from_numpy(x).cuda().requires_grad_(True)
  for keepdims in (False, True):
    out = GlobalAveragePooling1D(keepdims=keepdims)(xt, mask=mask)
    assert tuple(out.shape) == ((B, 1, d) if keepdims else (B, d))
    _same_bits(out.detach().cpu().reshape(B, d), to.pool(x, m))
  g = np.random.RandomState(9).randn(B, d).astype(np.float32)
  out = GlobalAveragePooling1D()(xt, mask=mask)
  (dx,) = torch.autograd.grad(out, xt, torch.from_numpy(g).cuda())
  _same_bits(dx.cpu(), to.pool_grad(g, m, T))


def test_pooling_inf_at_masked_positions_and_noncontiguous_input():
  x, ids = _pool_case(6, 9, 5, 11)
  x[ids == 0] = np.inf
  x[1, 0, 0] = -np.inf
  ids[1, 0] = 0
  out = GlobalAveragePooling1D()(torch.from_numpy(x).cuda(), mask=torch.from_numpy(ids).cuda())
  _same_bits(out.cpu(), to.pool(x, ids))
  assert np.isnan(out.cpu().numpy()).all()
  base = np.random.RandomState(12).randn(9, 8, 6).astype(np.float32)
  xt = torch.from_numpy(base).cuda().permute(1, 0, 2)[:, ::2, 1:]     # [8, 5, 5], strided
  assert not xt.is_contiguous()
  mk = np.random.RandomState(13).randint(0, 2, size=(8, 5))
  _same_bits(GlobalAveragePooling1D()(xt, mask=mk.astype(bool)).cpu(), to.pool(xt.cpu().numpy(), mk))
  _same_bits(GlobalAveragePooling1D()(xt).cpu(), to.pool(xt.cpu().numpy()))


def test_embedding_mask_zero_carries_its_mask_into_the_pooling():
  torch.manual_seed(0)
  emb = Embedding(10, 6, mask_zero=True)
  ids = torch.tensor([[1, 2, 0, 0], [0, 0, 0, 0], [3, 3, 3, 9]], device="cuda")
  assert torch.equal(emb.compute_mask(ids), ids != 0) and Embedding(10, 6).compute_mask(ids) is None
  e = emb(ids)
  assert ops.attached_mask(e) is ids
  out = GlobalAveragePooling1D()(e)
  w = emb.weight.cpu().numpy()
  _same_bits(out.detach().cpu(), to.pool(w[ids.cpu().numpy()], ids.cpu().numpy()))
  (out[2].sum() + out[0].sum()).backward()
  (rid, rows), = emb.pop_sparse_grads()
  assert torch.equal(rid, ids.reshape(-1))                      # every position keeps its row
  g = np.zeros((3, 6), np.float32)
  g[[0, 2]] = 1
  _same_bits(rows.cpu().reshape(3, 4, 6), to.pool_grad(g, ids.cpu().numpy(), 4))
  # a modified output no longer carries the mask; mask_zero=False leaves the output as it was
  e2 = emb(ids)
  e2.mul_(1.0)
  assert ops.attached_mask(e2) is None
  plain = Embedding(10, 6)
  plain.weight.copy_(emb.weight)
  assert torch.equal(plain(ids), emb(ids)) and not hasattr(plain(ids), "_tfrs_mask")

"""Host-side tests of layers.StringLookup / IntegerLookup: argument errors, the index layout for every (mask, OOV) pair,
adapt's order and cut on the oracle, the config round trip, and the coverage of the GPU cases' probe chains.  No GPU
needed (with a GPU present, set_vocabulary also builds the table)."""
import numpy as np
import pytest

import lookup_oracle as lo
import recommenders_b200 as tfrs
from recommenders_b200.layers.preprocessing import IntegerLookup, StringLookup

GPU_INT_SIZES = (31, 32, 33, 1000)        # the crafted integer vocabularies of tests/test_gpu_lookup.py
GPU_STRING_SIZES = (16, 33, 1000)         # and the crafted string ones


def test_exports():
  assert tfrs.layers.StringLookup is StringLookup and tfrs.layers.IntegerLookup is IntegerLookup


@pytest.mark.parametrize("cls", [StringLookup, IntegerLookup])
def test_constructor_errors(cls):
  with pytest.raises(NotImplementedError):
    cls(output_mode="one_hot")
  with pytest.raises(ValueError):
    cls(output_mode="bogus")
  with pytest.raises(NotImplementedError):
    cls(sparse=True)
  with pytest.raises(NotImplementedError):
    cls(pad_to_max_tokens=True)
  with pytest.raises(NotImplementedError):
    cls(idf_weights=[1.0])
  with pytest.raises(NotImplementedError):
    cls(num_oov_indices=2)
  with pytest.raises(ValueError):
    cls(num_oov_indices=-1)
  with pytest.raises(ValueError):
    cls(max_tokens=1)
  with pytest.raises(NotImplementedError):
    cls().set_vocabulary("vocab.txt")
  with pytest.raises(NotImplementedError):
    cls()((np.array([1]), np.array([0, 1])))


def test_string_and_integer_specific_errors():
  with pytest.raises(NotImplementedError):
    StringLookup(encoding="latin-1")
  with pytest.raises(NotImplementedError):
    IntegerLookup(vocabulary_dtype="int32")
  with pytest.raises(ValueError):
    IntegerLookup(mask_token="x")
  with pytest.raises(ValueError):
    StringLookup(vocabulary=["a", "[UNK]"])                  # the OOV token inside the vocabulary
  with pytest.raises(ValueError):
    StringLookup(vocabulary=[b"", b"a"], mask_token="")      # the mask token, compared as bytes
  with pytest.raises(ValueError):
    IntegerLookup(vocabulary=[3, -1])
  with pytest.raises(ValueError):
    IntegerLookup(vocabulary=[0, 3], mask_token=0)
  with pytest.raises(ValueError):
    IntegerLookup(vocabulary=[1, 2, 3], max_tokens=3)        # 1 + 3 indices
  IntegerLookup(vocabulary=[1, 2, 3], max_tokens=4)
  with pytest.raises(TypeError):
    IntegerLookup(vocabulary=[1.5, 2.0])
  with pytest.raises(TypeError):
    StringLookup(vocabulary=[["a", "b"]])
  with pytest.raises(TypeError):
    StringLookup(vocabulary=["a", 3])


@pytest.mark.parametrize("mask", [None, "MASK"])
@pytest.mark.parametrize("oov", [0, 1])
def test_vocabulary_layout_string(mask, oov):
  vocab = ["b", "a", "日本"]
  layer = StringLookup(vocabulary=vocab, mask_token=mask, num_oov_indices=oov)
  assert layer.get_vocabulary() == lo.vocabulary_list(vocab, mask, "[UNK]", oov)
  assert layer.get_vocabulary(include_special_tokens=False) == vocab
  assert layer.vocabulary_size() == (mask is not None) + oov + 3
  b = StringLookup(vocabulary=[v.encode() for v in vocab], mask_token=mask, num_oov_indices=oov)
  assert b.get_vocabulary() == lo.vocabulary_list([v.encode() for v in vocab], mask and mask.encode(), b"[UNK]", oov)


@pytest.mark.parametrize("mask", [None, 0])
@pytest.mark.parametrize("oov", [0, 1])
def test_vocabulary_layout_integer(mask, oov):
  vocab = [7, -3, 2**63 - 1]
  layer = IntegerLookup(vocabulary=np.array(vocab), mask_token=mask, num_oov_indices=oov, oov_token=-9)
  assert layer.get_vocabulary() == lo.vocabulary_list(vocab, mask, -9, oov)
  assert layer.vocabulary_size() == (mask is not None) + oov + 3
  assert IntegerLookup().vocabulary_size() == 1 and IntegerLookup().get_vocabulary() == [-1]


def test_adapt_order_and_cut():
  rng = np.random.RandomState(0)
  ints = rng.zipf(1.3, size=5000) % 200 - 100
  for max_tokens, mask in ((None, None), (20, None), (20, 0), (5, 3)):
    layer = IntegerLookup(max_tokens=max_tokens, mask_token=mask)
    layer.adapt(ints)
    exp = lo.adapt(ints, mask, -1, max_tokens, 1)
    assert layer.get_vocabulary(include_special_tokens=False) == exp, (max_tokens, mask)
  words = np.array(["b", "a", "c", "a", "b", "é", "é", "", "[UNK]", "[UNK]", "[UNK]", "ab", "ab"])
  for max_tokens, mask in ((None, None), (4, None), (6, "")):
    layer = StringLookup(max_tokens=max_tokens, mask_token=mask)
    layer.adapt(words)
    assert layer.get_vocabulary(include_special_tokens=False) == lo.adapt(words, mask, "[UNK]", max_tokens, 1, True)
  # ties are bytewise for strings ("a" < "ab" < "b" < "é"), and a Dataset of batches counts like the whole array
  ds = tfrs.data.Dataset.from_tensor_slices(words).batch(4)
  layer = StringLookup()
  layer.adapt(ds)
  assert layer.get_vocabulary(include_special_tokens=False) == ["a", "ab", "b", "é", "", "c"]
  b = StringLookup()
  b.adapt(np.char.encode(words, "utf-8"))
  assert b.get_vocabulary(include_special_tokens=False) == [w.encode() for w in ["a", "ab", "b", "é", "", "c"]]


def test_config_round_trip():
  for layer in (StringLookup(vocabulary=["x", "y"], mask_token="", num_oov_indices=0, name="s", max_tokens=10),
                IntegerLookup(vocabulary=[4, 5], mask_token=0, oov_token=-7, invert=True, name="i")):
    cfg = layer.get_config()
    again = type(layer).from_config(cfg)
    assert again.get_config() == cfg
    assert again.get_vocabulary() == layer.get_vocabulary()
    state = layer.get_extra_state()
    fresh = type(layer).from_config({**cfg, "vocabulary": None})
    fresh.set_extra_state(state)
    assert fresh.get_vocabulary() == layer.get_vocabulary()
  with pytest.raises(ValueError):
    StringLookup(mask_token="m").set_extra_state(StringLookup(vocabulary=["a"]).get_extra_state())


def test_slot_hash_matches_known_answers():
  # splitmix64's output function of 0 (the first output of a generator seeded with 0) and the SipHash-2-4 paper vector
  assert int(lo.mix64(np.array([0]))[0]) == 0xE220A8397B1DCDAF
  c = lo.source_constants()
  assert (c["k0"], c["k1"]) == (0x0706050403020100, 0x0F0E0D0C0B0A0908)
  assert int(lo.home_bytes([bytes(range(15))], 1 << 40)[0]) == 0xA129CA6149BE45E5 & ((1 << 40) - 1)
  assert [lo.slots(v) for v in (0, 1, 32, 33, 1000)] == [64, 64, 64, 128, 2048]


def test_gpu_cases_cover_long_and_wrapping_probe_chains():
  """Every crafted GPU case, whatever order the build's atomics insert its keys in, has a hit probe of >= 3 slots, a hit
  probe that wraps past the last slot, and the same for OOV queries.  The slot count and hash constants come from
  csrc/lookup.cu, so a changed constant re-derives the cases and this check runs on the new ones."""
  for V in GPU_INT_SIZES:
    vocab, oov = lo.int_case(V)
    cap = lo.slots(V)
    assert len(np.unique(vocab)) == V and not np.isin(oov, vocab).any()
    cov = lo.coverage(lo.home_int(vocab, cap), lo.home_int(oov, cap), cap)
    assert all(cov.values()), (V, cov)
  for V in GPU_STRING_SIZES:
    vocab, oov = lo.string_case(V)
    cap = lo.slots(V)
    assert len(set(vocab)) == V and not set(oov) & set(vocab)
    cov = lo.coverage(lo.home_bytes(vocab, cap), lo.home_bytes(oov, cap), cap)
    assert all(cov.values()), (V, cov)

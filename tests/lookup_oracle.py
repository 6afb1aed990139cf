"""Dict oracle of layers.StringLookup / IntegerLookup (DESIGN.md §2, A20), and a restatement of K15's slot hash
(csrc/lookup.cu) for the coverage rule of the GPU cases.  Test infrastructure: the product never imports it.

Index layout: m = 1 with a mask token, o = num_oov_indices; mask -> 0, an OOV value -> m, vocabulary[i] -> m + o + i.
Strings are compared as bytes (str is UTF-8).  The slot constants are read back from the CUDA source, so the case sets
below are derived from the code they exercise."""
from __future__ import annotations

import collections
import os
import re
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

import unified_oracle as uo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
M64 = 2**64 - 1


def _b(x) -> bytes:
  return x.encode("utf-8") if isinstance(x, str) else bytes(x)


def _key(x, strings: bool):
  return _b(x) if strings else int(x)


# ---- the layer's rules --------------------------------------------------------------------------------------------
def lookup(values, vocabulary: Sequence, mask_token=None, num_oov_indices: int = 1, strings: bool = False) -> np.ndarray:
  """int64 indices of `values` (any shape).  With num_oov_indices = 0 an OOV value raises KeyError."""
  m = 0 if mask_token is None else 1
  table: Dict = {}
  for i, v in enumerate(vocabulary):
    table[_key(v, strings)] = m + num_oov_indices + i
  mask = None if mask_token is None else _key(mask_token, strings)
  a = np.asarray(values, dtype=object)
  out = np.empty(a.shape, np.int64)
  for pos, v in np.ndenumerate(a):
    k = _key(v, strings)
    if mask is not None and k == mask:
      out[pos] = 0
    elif k in table:
      out[pos] = table[k]
    elif num_oov_indices:
      out[pos] = m
    else:
      raise KeyError(v)
  return out


def invert(indices, vocabulary: Sequence, mask_token, oov_token, num_oov_indices: int = 1) -> List:
  """Tokens of `indices` (flattened): the mask token for 0 with a mask, vocabulary[i - m - o] inside the vocabulary range,
  the OOV token for anything else."""
  m = 0 if mask_token is None else 1
  base = m + num_oov_indices
  out = []
  for x in np.asarray(indices).reshape(-1).tolist():
    if base <= x < base + len(vocabulary):
      out.append(vocabulary[x - base])
    elif m and x == 0:
      out.append(mask_token)
    else:
      out.append(oov_token)
  return out


def vocabulary_list(vocabulary: Sequence, mask_token, oov_token, num_oov_indices: int) -> List:
  return ([mask_token] if mask_token is not None else []) + [oov_token] * num_oov_indices + list(vocabulary)


def adapt(values, mask_token=None, oov_token=None, max_tokens: Optional[int] = None, num_oov_indices: int = 1,
          strings: bool = False) -> List:
  """Distinct values without the special tokens, by count descending, ties ascending (bytewise for strings)."""
  special = {_key(t, strings) for t in (mask_token, oov_token) if t is not None}
  first = {}
  counts = collections.Counter()
  for v in np.asarray(values, dtype=object).reshape(-1).tolist():
    k = _key(v, strings)
    if k in special:
      continue
    counts[k] += 1
    first.setdefault(k, v)
  order = sorted(counts, key=lambda k: (-counts[k], k))
  if max_tokens is not None:
    order = order[:max(max_tokens - (mask_token is not None) - num_oov_indices, 0)]
  return [first[k] for k in order]


# ---- K15's slot hash, restated ------------------------------------------------------------------------------------
def source_constants() -> Dict[str, int]:
  src = open(os.path.join(ROOT, "recommenders_b200", "csrc", "lookup.cu")).read()
  c = {"min_slots": int(re.search(r"LK_MIN_SLOTS\s*=\s*(\d+)", src).group(1))}
  k = re.search(r"LK_K0\s*=\s*(0x[0-9a-fA-F]+)ull,\s*LK_K1\s*=\s*(0x[0-9a-fA-F]+)ull", src)
  c["k0"], c["k1"] = int(k.group(1), 16), int(k.group(2), 16)
  body = re.search(r"lk_mix64\(uint64_t z\) \{(.*?)\n\}", src, re.S).group(1)
  c["mix"] = [int(x, 16) for x in re.findall(r"0x[0-9a-fA-F]+", body)]
  c["shifts"] = [int(x) for x in re.findall(r">> (\d+)", body)]
  return c


_C = None


def _consts():
  global _C
  if _C is None:
    _C = source_constants()
  return _C


def slots(V: int) -> int:
  cap = _consts()["min_slots"]
  while cap < 2 * V:
    cap *= 2
  return cap


def mix64(x: np.ndarray) -> np.ndarray:
  c = _consts()
  add, m1, m2 = c["mix"]
  s1, s2, s3 = c["shifts"]
  with np.errstate(over="ignore"):
    z = np.asarray(x, np.int64).view(np.uint64) + np.uint64(add)
    z = (z ^ (z >> np.uint64(s1))) * np.uint64(m1)
    z = (z ^ (z >> np.uint64(s2))) * np.uint64(m2)
    return z ^ (z >> np.uint64(s3))


def home_int(keys, cap: int) -> np.ndarray:
  return (mix64(np.asarray(keys, np.int64)) & np.uint64(cap - 1)).astype(np.int64)


def home_bytes(strings, cap: int) -> np.ndarray:
  c = _consts()
  if len(strings) == 0:
    return np.zeros(0, np.int64)
  return uo.hash_bins(list(strings), cap, (c["k0"], c["k1"])).reshape(-1)


def occupied(homes: np.ndarray, cap: int) -> np.ndarray:
  """Occupied slots after inserting keys with these home slots by linear probing (the same set in any insertion order)."""
  occ = np.zeros(cap, bool)
  for h in homes.tolist():
    while occ[h]:
      h = (h + 1) % cap
    occ[h] = True
  return occ


def coverage(homes: np.ndarray, miss_homes: np.ndarray, cap: int) -> Dict[str, bool]:
  """What every insertion order guarantees about the probes of a case:
  hit_chain3   some key reads >= 3 slots (3 keys share a home slot, so one sits 2 slots past it);
  hit_wrap     some key's probe wraps past slot cap - 1 (more keys have homes in [s, cap) than the cap - s slots there);
  miss_chain3  some OOV value reads >= 3 slots (its home and the next slot are occupied);
  miss_wrap    some OOV value's probe wraps (every slot from its home to cap - 1 is occupied)."""
  cnt = np.bincount(homes, minlength=cap)
  suffix = np.cumsum(cnt[::-1])[::-1]
  occ = occupied(homes, cap)
  run = np.zeros(cap + 1, np.int64)            # run[s] = occupied slots from s up to cap - 1 without a gap
  for s in range(cap - 1, -1, -1):
    run[s] = run[s + 1] + 1 if occ[s] else 0
  mh = np.asarray(miss_homes, np.int64)
  return {"hit_chain3": bool((cnt >= 3).any()),
          "hit_wrap": bool((suffix > cap - np.arange(cap)).any()),
          "miss_chain3": bool(len(mh) and (occ[mh] & occ[(mh + 1) % cap]).any()),
          "miss_wrap": bool(len(mh) and (run[mh] == cap - mh).any())}


# ---- the GPU test's case sets -------------------------------------------------------------------------------------
def _pick(homes: np.ndarray, want, n: int, taken: set) -> List[int]:
  out = []
  for i in np.nonzero(np.isin(homes, want))[0].tolist():
    if i not in taken:
      out.append(i); taken.add(i)
      if len(out) == n:
        break
  return out


def int_case(V: int, seed: int = 0) -> Tuple[np.ndarray, np.ndarray]:
  """(vocabulary int64 [V], OOV queries): the int64 edges and, from V = 8 up, three keys sharing a home slot, two keys
  homed at cap - 1 and one at cap - 2 (so a probe wraps), and OOV queries homed on those clusters."""
  cap = slots(V)
  rng = np.random.RandomState(seed)
  edges = [0, -1, INT64_MIN, INT64_MAX]
  vocab: List[int] = edges[:V]
  if V >= 8:
    cand = rng.randint(-2**62, 2**62, size=200000, dtype=np.int64)
    cand = cand[~np.isin(cand, edges)]
    h = home_int(cand, cap)
    taken: set = set()
    target = int(h[0])
    vocab += [int(cand[i]) for i in _pick(h, [target], 3, taken)]
    vocab += [int(cand[i]) for i in _pick(h, [cap - 1], 2, taken)]
    vocab += [int(cand[i]) for i in _pick(h, [cap - 2], 1, taken)]
    oov = [int(cand[i]) for i in _pick(h, [target, cap - 1, cap - 2], 6, taken)]
  else:
    oov = []
  rest = V - len(vocab)
  if rest > 0:
    fill = np.unique(rng.randint(-2**40, 2**40, size=rest * 2 + 16, dtype=np.int64))
    fill = fill[~np.isin(fill, vocab + oov)]
    vocab += rng.permutation(fill)[:rest].tolist()
  vocab = np.asarray(vocab[:V], np.int64)
  more = rng.randint(-2**40, 2**40, size=64, dtype=np.int64)
  oov = np.asarray(oov + [int(x) for x in more if x not in set(vocab.tolist())], np.int64)
  return vocab, oov


def string_case(V: int, seed: int = 0) -> Tuple[List[str], List[str]]:
  """(vocabulary, OOV queries) of distinct strings: the same crafted collisions as int_case from V = 8 up, lengths
  around K8's register / memory boundary (23 / 24 bytes) and multi-byte UTF-8."""
  cap = slots(V)
  rng = np.random.RandomState(seed)
  base = ["", "a", "é", "日本語", "x" * 23, "y" * 24, "z" * 1024, "ab" * 11 + "c", "ab" * 11 + "d", "ab" * 12 + "c",
          "ab" * 12 + "d"]
  vocab: List[str] = base[:V]
  oov: List[str] = []
  if V >= 16:
    cand = [f"c{seed}-{i}" for i in range(50000)]
    h = home_bytes(cand, cap)
    taken: set = set()
    target = int(h[0])
    vocab += [cand[i] for i in _pick(h, [target], 3, taken)]
    vocab += [cand[i] for i in _pick(h, [cap - 1], 2, taken)]
    vocab += [cand[i] for i in _pick(h, [cap - 2], 1, taken)]
    oov = [cand[i] for i in _pick(h, [target, cap - 1, cap - 2], 6, taken)]
  i = 0
  while len(vocab) < V:
    n = int(rng.randint(1, 64))
    vocab.append(f"w{i}-" + "q" * n)
    i += 1
  oov += ["b", "x" * 22, "y" * 25, "z" * 1023 + "y", "ab" * 11 + "e", "日本", "[UNK]x"]
  return vocab[:V], oov

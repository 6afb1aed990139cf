"""Host-side tests of UnifiedEmbedding: the hashing oracle against published known answers, the config bookkeeping of
the reference, string packing, and the register budget of the K8 kernels.  No GPU needed."""
import os
import re
import subprocess

import numpy as np
import pytest

import unified_oracle as uo
from recommenders_b200.layers.feature_multiplexing import unified_embedding as ue

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1


def test_siphash_paper_vectors():
  # SipHash paper, appendix A: key 00..0f, message 00..0e; and the empty message with the same key
  k0, k1 = 0x0706050403020100, 0x0F0E0D0C0B0A0908
  assert uo.siphash(k0, k1, bytes(range(15))) == 0xA129CA6149BE45E5
  assert uo.siphash(k0, k1, b"") == 0x726FDB47DD0E0E31


def test_hash_bucket_strong_and_hashing_known_answers():
  # tf.strings.to_hash_bucket_strong and tf.keras.layers.Hashing API documentation examples
  assert uo.hash_bins(["Hello", "TF"], 3, [1, 2]).tolist() == [2, 0]
  assert uo.hash_bins(np.array(["A", "B", "C", "D", "E"]), 3, 133).tolist() == [0, 0, 2, 1, 0]


def test_as_string():
  assert [uo.as_string(x) for x in (0, -1, INT64_MIN, INT64_MAX, 1950)] == \
      [b"0", b"-1", b"-9223372036854775808", b"9223372036854775807", b"1950"]
  # an integer hashes as its decimal text
  ints = np.array([0, -1, INT64_MIN, INT64_MAX, 7], np.int64)
  assert uo.hash_bins(ints, 1000, [3, 4]).tolist() == uo.hash_bins([str(v) for v in ints], 1000, [3, 4]).tolist()


def _config(name, num_tables, features, **kw):
  c = ue.UnifiedEmbeddingConfig(buckets_per_table=10, dim_per_table=8, num_tables=num_tables, name=name, **kw)
  for f, n in features:
    c.add_feature(f, n)
  return c


def test_config_matches_reference_bookkeeping():
  # test_save_model's config: tables round-robin with a cursor carried across features, salt [feature index, chunk]
  c = _config("ue_table", 4, [("year", 1), ("city", 3), ("genre", 2)])
  assert c.hashing_config == {
      "year": {"ue_table_year_lookup_0": {"num_bins": 10, "salt": [0, 0]}},
      "city": {"ue_table_city_lookup_0": {"num_bins": 10, "salt": [1, 0]},
               "ue_table_city_lookup_1": {"num_bins": 10, "salt": [1, 1]},
               "ue_table_city_lookup_2": {"num_bins": 10, "salt": [1, 2]}},
      "genre": {"ue_table_genre_lookup_0": {"num_bins": 10, "salt": [2, 0]},
                "ue_table_genre_lookup_1": {"num_bins": 10, "salt": [2, 1]}},
  }
  tables = {f: [fc.table for fc in chunks.values()] for f, chunks in c.embedding_config.items()}
  assert tables == {"year": ["ue_table_0"], "city": ["ue_table_1", "ue_table_2", "ue_table_3"],
                    "genre": ["ue_table_0", "ue_table_1"]}
  assert [fc.name for fc in c.embedding_config["city"].values()] == [f"ue_table_city_lookup_{i}" for i in range(3)]
  # test_multiple_features / test_feature_output_order
  c = _config("multiple_ue_table", 3, [("genre", 1), ("year", 2), ("city", 3)])
  assert [[h["salt"] for h in c.hashing_config[f].values()] for f in ("genre", "year", "city")] == \
      [[[0, 0]], [[1, 0], [1, 1]], [[2, 0], [2, 1], [2, 2]]]
  assert [fc.table for f in ("genre", "year", "city") for fc in c.embedding_config[f].values()] == \
      ["multiple_ue_table_" + s for s in "012012"]
  # the oracle's independent restatement gives the same tables
  assert [(f, [t for _, t, _, _ in ch]) for f, ch in uo.plan([("genre", 1), ("year", 2), ("city", 3)], 3, "x")] == \
      [("genre", [0]), ("year", [1, 2]), ("city", [0, 1, 2])]


def _layer_plan(config):
  """The (feature, [(table, key, column slot)]) plan the layer runs, in the oracle's (chunk, table, salt, slot) form."""
  return [(f, [(c, t, key, pos) for c, (t, key, pos) in enumerate(ch)]) for f, ch in config._lookup_plan()]


@pytest.mark.parametrize("name,num_tables,spec", [
    ("ue_table", 4, [("year", 1), ("city", 3), ("genre", 2)]),
    ("multiple_ue_table", 3, [("genre", 1), ("year", 2), ("city", 3)]),
    ("many", 5, [("a", 12), ("b", 1), ("c", 11)]),
])
def test_layer_plan_matches_oracle(name, num_tables, spec):
  """Tables, SipHash keys and sorted()-name column slots of the layer's lookups, against the oracle's restatement."""
  assert _layer_plan(_config(name, num_tables, spec)) == uo.plan(spec, num_tables, name)


def test_sorted_chunk_name_order():
  # 12 chunks: the reference concatenates in sorted() order of the names, so chunk 10 comes before chunk 2
  for plan in (uo.plan([("f", 12)], 5, "n"), _layer_plan(_config("n", 5, [("f", 12)]))):
    cols = {c: pos for c, _, _, pos in plan[0][1]}
    assert [c for c, _ in sorted(cols.items(), key=lambda kv: kv[1])] == [0, 1, 10, 11, 2, 3, 4, 5, 6, 7, 8, 9]


def test_unsupported_arguments():
  with pytest.raises(TypeError, match="vocabulary_size"):
    ue.UnifiedEmbeddingConfig(10, 8, 1, "t", vocabulary_size=3)
  with pytest.raises(ValueError, match="combiner"):
    ue.UnifiedEmbeddingConfig(10, 8, 1, "t", combiner="max")
  c = ue.UnifiedEmbeddingConfig(10, 8, 1, "t", combiner="sqrtn", initializer="zeros")
  with pytest.raises(TypeError, match="max_sequence_length"):
    c.add_feature("a", 1, max_sequence_length=4)


def test_empty_list_is_not_strings():
  assert not ue._is_strings([])


@pytest.mark.parametrize("values", [
    np.array(["", "a", "héllo", "日本語テキスト", "x" * 40]),
    np.array([b"", b"a", b"\xff\x00z", b"y" * 33]),
    np.array(["", "ü", "abc"], dtype=object),
    np.array([b"", b"ab"], dtype=object),
    ["romance", "", "drama"],
    np.array([["a", "bb"], ["", "ccc"]]),
    np.array([], dtype="U1"),
    np.array(["", ""]),
])
def test_string_packing(values):
  data, offsets, shape = ue._pack_strings(values)
  ref_data, ref_off = uo.pack(values)
  assert shape == np.shape(values)
  assert offsets.dtype == np.int64 and offsets.tolist() == ref_off.tolist()
  assert data.dtype == np.uint8 and data.tobytes() == ref_data.tobytes()[:int(ref_off[-1])]


def test_k8_kernels_do_not_spill():
  """ptxas: no spill stores or loads and a 0-byte stack in every K8 kernel."""
  nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else "nvcc"
  src = os.path.join(ROOT, "recommenders_b200", "csrc", "unified_embedding.cu")
  r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                      "--expt-relaxed-constexpr", "-DTFRS_BUILD", "-c", src, "-o", os.devnull],
                     capture_output=True, text=True)
  assert r.returncode == 0, r.stderr
  props = re.findall(r"Function properties for (\w+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                     r"(\d+) bytes spill loads", r.stderr)
  kernels = {name: rest for name, *rest in props if "ue_" in name}
  assert len(kernels) == 3, r.stderr
  assert all(v == ["0", "0", "0"] for v in kernels.values()), kernels

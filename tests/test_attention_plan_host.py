"""CPU checks of tests/test_gpu_attention_edges.py's shapes (tests/attention_edge_cases.py): the plan's constants are
read back from csrc/attention.cuh, and the generated cases must reach every kernel instance E, the 1- and 2-row tiles
of dk = dv = 128, a CTA holding 32 sequences with dead teams, a dense dropout case whose dK / dV walk draws keep bytes
at t0 > 0 from the middle of a Philox group, and dense causal cases with Tq < Tv and Tq > Tv.  A changed constant
then fails here instead of silently dropping coverage."""
import os
import re

import numpy as np

import attention_edge_cases as cases
import attention_oracle as ao
import dense_attention_oracle as dao

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _const(name):
  with open(os.path.join(ROOT, "recommenders_b200", "csrc", "attention.cuh")) as f:
    m = re.search(rf"constexpr int {name} = ([^;]+);", f.read())
  assert m, name
  return m.group(1).strip()


def test_the_plan_mirrors_the_kernel_constants():
  assert int(_const("MHA_THREADS")) // int(_const("MHA_LANES")) == cases.TEAMS
  assert int(_const("MHA_LANES")) == cases.LANES
  assert int(_const("MHA_MAX_TILE")) == cases.MAX_TILE
  assert _const("MHA_SMEM_BUDGET") == "64 * 1024" and cases.BUDGET == 65536
  assert cases.plan(1, 56) == (32, 9) and cases.plan(10, 32) == (5, 64) and cases.plan(33, 32) == (2, 64)


def test_the_widths_reach_every_instance_and_mix_them():
  pairs = cases.width_pairs()
  assert {cases.elems(dk, dv) for dk, dv in pairs} == {1, 2, 4, 8, 16}
  assert {d for p in pairs for d in p} == set(cases.HEAD_DIMS)
  mixed = [(a, b) for a, b in pairs if cases.elems(a, 1) != cases.elems(b, 1)]
  assert mixed and all((b, a) in pairs for a, b in mixed)


def test_the_core_cases_walk_every_tile_edge_at_128():
  c = set(cases.core_tile_cases())
  assert cases.plan(1, 256)[1] == 2 and cases.plan(1, 259)[1] == 1
  assert {(1, 3, 128, 128), (3, 1, 128, 128), (5, 1, 128, 128)} <= c
  for dk, dv in cases.width_pairs():
    for own in (1, 33):
      tile = cases.plan(own, dk + dv)[1]
      assert {(own, s, dk, dv) for s in (tile, tile + 1, 2 * tile + 1, 3 * tile)} <= c
      tile = cases.plan(own, dk + dv + 3)[1]
      assert {(t, own, dk, dv) for t in (tile, tile + 1, 2 * tile + 1, 3 * tile)} <= c


def test_the_packed_cases_fill_a_cta_with_32_sequences_and_dead_teams():
  packed = cases.packing_cases()
  rows = [B * H * T for B, H, T in packed]
  assert {r % 32 for r in rows} == {0, 1, 31}
  assert {T for _, _, T in packed} == {1, 2, 3, 5, 31, 33} and max(H for _, H, _ in packed) == 16
  assert any(cases.cta_sequences(B * H * T, T, 0) == 32 for B, H, T in packed)
  assert any((B * H * T) % 32 and cases.cta_sequences(B * H * T, T, (B * H * T) // 32) < 32 for B, H, T in packed)


def test_the_dense_dropout_cases_draw_key_row_keep_bytes_past_the_first_tile():
  c = cases.dense_dropout_cases()
  assert (5, 17, 1, 32, 24) in c and {7, 8, 9} <= {tq for _, tq, tv, d, e in c if (tv, d, e) == (1, 32, 24)}
  later = [x for x in c if len(cases.dense_kv_starts(*x)) > 1]
  assert later
  # a key-row CTA of a later tile starts in the middle of a Philox group and spans sequences
  def mid_group_ctas(B, Tq, Tv, dim, dv):
    for t0 in cases.dense_kv_starts(B, Tq, Tv, dim, dv)[1:]:
      for cta in range((B * Tv + 31) // 32):
        b, s = divmod(cta * 32, Tv)
        if ((b * Tq + t0) * Tv + s) & 3 and cases.cta_sequences(B * Tv, Tv, cta) > 1:
          yield t0, cta
  assert any(Tv % 4 and any(mid_group_ctas(*x)) for x in later for Tv in [x[2]])
  tiles = {cases.plan(tv, d + v + 3)[1] for _, _, tv, d, v in c} | {cases.plan(tq, d + v)[1] for _, tq, _, d, v in c}
  assert {1, 2} <= tiles


def test_the_dense_causal_cases_run_both_directions():
  c = cases.dense_causal_cases()
  assert any(tq < tv for _, tq, tv, _, _ in c) and any(tq > tv for _, tq, tv, _, _ in c)
  assert all(tq != tv for _, tq, tv, _, _ in c)


def test_the_core_bounds_cover_a_float32_evaluation():
  """The per-element bounds hold for a float32 NumPy evaluation of the same core (another summation order, errors of
  the same size), and are far below the oracle's values: loose enough for any fp32 order, tight enough to matter."""
  rng = np.random.RandomState(0)
  B, T, S, H, dk, dv = 2, 5, 9, 2, 33, 17
  Q, K, V, dO = (rng.normal(size=s).astype(np.float32) for s in ((B, T, H, dk), (B, S, H, dk), (B, S, H, dv),
                                                                 (B, T, H, dv)))
  K[..., 0] *= 40                                  # scores of tens
  q, k, v, g = (a.astype(np.float64) for a in (Q, K, V, dO))
  eO, eP, Qs = ao.core_forward(q, k, v, None)
  bd = ao.core_error_bounds(q, k, v, eP, Qs, g)
  s = np.einsum("bthd,bshd->bhts", Q * np.float32(ao.scale_of(dk)), K).astype(np.float32)
  e = np.exp(s - s.max(-1, keepdims=True)).astype(np.float32)
  P = (e / e.sum(-1, keepdims=True, dtype=np.float32)).astype(np.float32)
  O = np.einsum("bhts,bshd->bthd", P, V).astype(np.float32)
  for name, got, ex in (("P", P, eP), ("O", O, eO)):
    bar = 2 * 2.0 ** -24 * bd[name].max(-1, keepdims=True)
    assert np.all(np.abs(got - ex) <= bar), name
    assert np.all(bar <= 1e-3 * np.abs(ex).max(-1, keepdims=True)), name


def test_the_dense_bounds_cover_a_float32_evaluation():
  rng = np.random.RandomState(1)
  for mode in dao.MODES:
    q, k = (rng.normal(size=(2, n, 12)).astype(np.float32) * 0.5 for n in (4, 7))
    v = rng.normal(size=(2, 7, 5)).astype(np.float32)
    scale = rng.uniform(-0.5, 0.5, 12).astype(np.float32) if mode == "additive" else np.float32(0.8)
    cw = np.float32(1.3) if mode == "concat" else None
    eo, ew, cache = dao.forward(q, k, v, mode, scale, cw)
    bd = dao.error_bounds(cache, rng.normal(size=(2, 4, 5)))
    w32 = ew.astype(np.float32)
    o32 = np.einsum("bts,bsd->btd", w32, v).astype(np.float32)
    bar = 2 * 2.0 ** -24 * bd["out"].max(-1, keepdims=True)
    assert np.all(np.abs(o32 - eo) <= bar) and np.all(bar <= 1e-4 * np.abs(eo).max(-1, keepdims=True)), mode

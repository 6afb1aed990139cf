"""The shapes tests/test_gpu_attention_edges.py runs, generated from K21 / K25's staged-tile plan (csrc/attention.cuh
mha_plan, mha_elems) rather than a Cartesian product.  Plain Python: tests/test_attention_plan_host.py checks on the
CPU that the lists reach every kernel instance, tile, packing and dropout edge they are meant to.

The three kernels and what they walk:
  forward, dQ    one team per query row (b, h, t); rows of one CTA span sequences planned from T, width dk + dv; the
                 team walks the S key rows in tiles.
  dK / dV        one team per key row (b, h, s); planned from S, width dk + dv + 3; the team walks the T query rows.
"""
TEAMS = 32               # MHA_TEAMS: rows per CTA
MAX_TILE = 64            # MHA_MAX_TILE
BUDGET = 64 * 1024       # MHA_SMEM_BUDGET, bytes
LANES = 8                # MHA_LANES

HEAD_DIMS = [1, 7, 8, 9, 16, 17, 32, 33, 64, 65, 127, 128]


def plan(L, width):
  """(nseq, tile): sequences a CTA of 32 rows of length L can touch, and rows staged per sequence at `width` floats."""
  nseq = min((TEAMS - 1 + L - 1) // L + 1, TEAMS)
  return nseq, max(1, min(MAX_TILE, BUDGET // (nseq * width * 4)))


def elems(dk, dv):
  """Head elements per lane: the kernel instance E (1, 2, 4, 8 or 16)."""
  e = 1
  while e * LANES < max(dk, dv):
    e *= 2
  return e


def walked(tile):
  """Walked lengths at a tile's edges: one short, exact, one over, two tiles and one row, three tiles, three and two
  rows (5 at tile 1)."""
  return sorted({n for n in (tile - 1, tile, tile + 1, 2 * tile + 1, 3 * tile, 3 * tile + 2) if n >= 1})


def width_pairs():
  """(dk, dv): every head dim with itself, and with a dim of another instance, in both orders."""
  d = HEAD_DIMS
  pairs = {(x, x) for x in d} | {(d[i], d[(i + 5) % len(d)]) for i in range(len(d))}
  return sorted(pairs | {(b, a) for a, b in pairs})


def core_tile_cases():
  """(T, S, dk, dv) of the MHA core: at each width the forward / dQ walk over S at the edges of the tile planned from
  T, and the dK / dV walk over T at the edges of the tile planned from S, for an owning length of 1 (32 sequences per
  CTA) and 33 (two)."""
  cases = set()
  for dk, dv in width_pairs():
    for own in (1, 33):
      cases |= {(own, s, dk, dv) for s in walked(plan(own, dk + dv)[1])}
      cases |= {(t, own, dk, dv) for t in walked(plan(own, dk + dv + 3)[1])}
  return sorted(cases)


def packing_cases():
  """(B, H, T) with B * H * T at 32k - 1, 32k and 32k + 1 rows (the least k that T divides, none when no k <= T
  does), H <= 16 the largest that divides: CTAs that hold up to 32 sequences and end in dead teams."""
  out = []
  for T in (1, 2, 3, 5, 31, 33):
    for off in (-1, 0, 1):
      n = next((TEAMS * k + off for k in range(1, T + 1) if (TEAMS * k + off) % T == 0), None)
      if n is None:
        continue
      H = next(h for h in range(16, 0, -1) if (n // T) % h == 0)
      out.append((n // (T * H), H, T))
  return out


def cta_sequences(rows, L, cta):
  """The (b, h) sequences CTA `cta` of 32 rows over rows of length L holds (MhaRow's n0 .. last)."""
  r0 = cta * TEAMS
  last = min(r0 + TEAMS, rows) - 1
  return last // L - r0 // L + 1


# ---- the dense modes (H = 1) ----------------------------------------------------------------------------------------
DENSE_WIDTHS = [(32, 24), (7, 9), (128, 128)]


def dense_dropout_cases():
  """(B, Tq, Tv, dim, dv) with dropout: the dK / dV walk over Tq at the edges of the tile planned from Tv (Tq above
  one tile, so the key-row keep bytes are drawn at t0 > 0), and the forward / dQ walk over Tv at the edges of the tile
  planned from Tq.  Tv not a multiple of 4 and B * Tv > 32 put key-row CTAs in the middle of a Philox group and across
  sequences."""
  cases = set()
  for dim, dv in DENSE_WIDTHS:
    for Tv in (1, 3, 6, 13):
      cases |= {(5, tq, Tv, dim, dv) for tq in walked(plan(Tv, dim + dv + 3)[1])}
    for Tq in (1, 5):
      cases |= {(5, Tq, tv, dim, dv) for tv in walked(plan(Tq, dim + dv)[1])}
  return sorted(cases)


def dense_kv_starts(B, Tq, Tv, dim, dv):
  """The query-row offsets t0 at which the dK / dV kernel stages a tile (and draws keep bytes) in this case."""
  tile = plan(Tv, dim + dv + 3)[1]
  return list(range(0, Tq, tile))


def dense_causal_cases():
  """(B, Tq, Tv, dim, dv): causal masks with Tq != Tv in both directions, across tile edges."""
  out = []
  for dim, dv in ((32, 24), (128, 128)):
    for L in (1, 33):
      for n in walked(plan(L, dim + dv)[1])[:3]:
        if n != L:
          out += [(3, L, n, dim, dv), (3, n, L, dim, dv)]
  return sorted(set(out))

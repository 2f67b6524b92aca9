"""The 2-opt kernels (`k_twoopt_eval` / `k_twoopt_apply`, SURVEY 8f row f3) where they can go wrong: exact ties between
moves (first occurrence must win through the thread, warp, block, tile and batch reductions), tile edges, batches
wider than the apply block, the size limits and the stopping rule's corner cases.  Every comparison is exact: tours
and iteration counts against the reference's answers in tests/golden/two_opt_ties.npz or against `oracle.two_opt`,
the reference's expression in float64 numpy."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))

from difusco_b200.utils import tsp_utils as tu
from oracle import tsp_decode_oracle as orc
from conftest import golden as _load_golden

CAPS = (1, 7, 10**9)
TIE_NAMES = sorted(orc.tie_instances())


def gpu_two_opt(pts, tours, cap):
  return tu.batched_two_opt_torch(np.asarray(pts, np.float64), tours, max_iterations=cap, device="cuda")


def check_against_oracle(pts, tours, caps=CAPS):
  for cap in caps:
    want, ns_want = orc.two_opt(pts, tours, cap)
    got, ns = gpu_two_opt(pts, tours, cap)
    assert ns == ns_want, (cap, ns, ns_want)
    assert np.array_equal(got, want), cap


def best_changes(pts, tours):
  """Each tour's smallest change of the reference's masked matrix (the value its arg-min applies)."""
  head, nxt = pts[tours[:, :-1]], pts[tours[:, 1:]]
  d = lambda u, v: np.sqrt(np.sum((u - v) ** 2, axis=-1))
  change = (d(head[:, :, None], head[:, None, :]) + d(nxt[:, :, None], nxt[:, None, :])
            - d(head, nxt)[:, :, None] - d(head, nxt)[:, None, :])
  return np.triu(change, k=2).reshape(len(tours), -1).min(axis=1)


def circle(n, phase=0.0):
  a = 2.0 * np.pi * np.arange(n) / n + phase
  return np.stack([np.cos(a), np.sin(a)], -1)


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 4, 5, 63, 64, 65, 127, 128, 129, 191, 192, 193])
def test_two_opt_tile_edges(n):
  """Tours whose last position sits on, or one either side of, a 64-wide tile edge."""
  pts = np.random.default_rng(1000 + n).random((n, 2))
  check_against_oracle(pts, orc.random_tours(n, 3, seed=n))


@pytest.mark.gpu
@pytest.mark.parametrize("name", TIE_NAMES)
@pytest.mark.parametrize("b", [1, 3])
def test_two_opt_ties_match_reference(name, b):
  """Grids, a regular polygon, collinear and repeated points: many moves tie exactly, and the three tours of a batch
  meet their ties on different iterations."""
  g = _load_golden("two_opt_ties")
  pts, tours = g[f"{name}/points"], g[f"{name}/tours"][:b]
  for cap in (1, 7, 1000):
    got, ns = gpu_two_opt(pts, tours, cap)
    assert ns == int(g[f"{name}/b{b}_cap{cap}_iters"]), cap
    assert np.array_equal(got, g[f"{name}/b{b}_cap{cap}"]), cap


@pytest.mark.gpu
def test_two_opt_ties_across_tile_candidate_warps():
  """520 equally spaced collinear points make 45 tiles per tour, more than one warp of `k_twoopt_apply` holds.  Two
  identical defects (adjacent nodes swapped at positions 10 and 500) tie exactly at -2, in tiles 0 and 42: the first
  one must be undone first."""
  n = 520
  pts = np.stack([np.arange(n), np.zeros(n)], -1).astype(np.float64)
  tour = np.concatenate([np.arange(n), [0]]).astype(np.int64)
  for p in (10, 500):
    tour[[p, p + 1]] = tour[[p + 1, p]]
  check_against_oracle(pts, tour[None], caps=(1, 2, 10**9))


@pytest.mark.gpu
def test_two_opt_batch_wider_than_apply_block():
  """1 025 tours: more than the 1 024 threads of the apply block."""
  pts = np.random.default_rng(7).random((20, 2))
  check_against_oracle(pts, orc.random_tours(20, 1025, seed=8))


@pytest.mark.gpu
def test_two_opt_largest_batch():
  """B = 65 535 (the grid's y limit) at N = 12, cap 3.  Every chunk of 4 096 random tours keeps a move below -1e-6 for
  all 3 iterations, so the batch-wide stopping rule never binds and the oracle may run chunk by chunk."""
  n, b, cap = 12, 65535, 3
  pts = np.random.default_rng(9).random((n, 2))
  tours = orc.random_tours(n, b, seed=10)
  want = []
  for s in range(0, b, 4096):
    w, ns = orc.two_opt(pts, tours[s:s + 4096], cap)
    assert ns == cap
    want.append(w)
  got, ns = gpu_two_opt(pts, tours, cap)
  assert ns == cap and np.array_equal(got, np.concatenate(want))


@pytest.mark.gpu
def test_two_opt_batch_mixing_optimal_and_random_tours():
  n = 60
  pts = np.random.default_rng(11).random((n, 2))
  rand = orc.random_tours(n, 2, seed=12)
  solved, _ = orc.two_opt(pts, orc.random_tours(n, 2, seed=13), 10**9)
  assert (best_changes(pts, solved) >= -1e-6).all()
  check_against_oracle(pts, np.stack([solved[0], rand[0], solved[1], rand[1]]))


@pytest.mark.gpu
def test_two_opt_applies_tiny_moves_while_the_batch_improves():
  """Tour 0's own best move improves by less than 1e-6, tour 1's by more: while tour 1 keeps the batch going, the
  reference applies tour 0's tiny move as well."""
  n = 16
  pts = circle(n)
  pts = np.concatenate([pts, [[np.cos(2 * np.pi * 3 / n + 3e-7), np.sin(2 * np.pi * 3 / n + 3e-7)]]])   # node 16 just past node 3
  tiny = np.array([0, 1, 2, 16, 3] + list(range(4, n)) + [0])        # visits 16 before 3: a detour of ~1e-7
  big = np.array([0, 1, 2, 3, 16] + list(range(10, 3, -1)) + list(range(11, n)) + [0])
  tours = np.stack([tiny, big]).astype(np.int64)
  bc = best_changes(pts, tours)
  assert -1e-6 < bc[0] < 0 and bc[1] < -1e-6
  once, ns = orc.two_opt(pts, tours, 1)
  assert ns == 1 and not np.array_equal(once[0], tiny)
  check_against_oracle(pts, tours)


@pytest.mark.gpu
def test_two_opt_tour_not_starting_at_node_zero():
  n = 50
  pts = np.random.default_rng(14).random((n, 2))
  rng = np.random.default_rng(15)
  tours = []
  for start in (7, 49):
    perm = np.concatenate([[start], rng.permutation(np.delete(np.arange(n), start))])
    tours.append(np.concatenate([perm, [start]]))
  check_against_oracle(pts, np.stack(tours).astype(np.int64))


def _oracle_first_move_chunked(pts, tour, rows=256):
  """oracle.two_opt's first iteration for one tour, evaluated in row chunks (the full matrix has N^2 fp64 entries):
  (min change, first flat index attaining it)."""
  head, nxt = pts[tour[:-1]], pts[tour[1:]]
  n = len(head)
  edge = np.sqrt(np.sum((head - nxt) ** 2, axis=-1))
  best, best_idx = 0.0, 0
  j = np.arange(n)

  def dist(u, r0, r1):            # np.sqrt(np.sum((u_i - u_j) ** 2, axis=-1)) without the (rows, n, 2) temporary
    dx = u[r0:r1, 0, None] - u[None, :, 0]
    dy = u[r0:r1, 1, None] - u[None, :, 1]
    dx *= dx
    dy *= dy
    dx += dy
    return np.sqrt(dx, out=dx)

  for r0 in range(0, n, rows):
    r1 = min(n, r0 + rows)
    a = dist(head, r0, r1)
    a += dist(nxt, r0, r1)
    a -= edge[r0:r1, None]
    a -= edge[None]
    a[j[None] < np.arange(r0, r1)[:, None] + 2] = 0.0              # np.triu(change, k=2)
    k = int(a.argmin())
    if a.flat[k] < best:
      best, best_idx = float(a.flat[k]), r0 * n + k
  return best, best_idx


@pytest.mark.gpu
def test_two_opt_largest_instance_flat_index():
  """N = 46 340, where the flattened move index i*N + j comes within 0.05 % of 2^31: points in convex position in tour
  order, with one reversed segment planted at the end of the index range."""
  n = 46340
  pts = circle(n)
  tour = np.concatenate([np.arange(n), [0]]).astype(np.int64)
  tour[n - 20:n] = tour[n - 20:n][::-1].copy()
  best, idx = _oracle_first_move_chunked(pts, tour)
  assert best < -1e-6 and idx > (n - 25) * n
  want = tour.copy()
  i, j = idx // n, idx % n
  want[i + 1:j + 1] = want[i + 1:j + 1][::-1].copy()
  got, ns = gpu_two_opt(pts, tour[None], 1)
  assert ns == 1 and np.array_equal(got[0], want)


@pytest.mark.gpu
def test_two_opt_size_limits():
  with pytest.raises(ValueError):
    gpu_two_opt(circle(46341), np.concatenate([np.arange(46341), [0]])[None], 1)
  with pytest.raises(ValueError):
    gpu_two_opt(circle(3), np.tile(np.array([0, 1, 2, 0]), (65536, 1)), 1)


@pytest.mark.gpu
@pytest.mark.parametrize("cap", [0, -3])
def test_two_opt_non_positive_cap(cap):
  """The reference tests its cap only after a move: a cap <= 0 still makes one move (and reports 1), none at N = 3."""
  pts = np.random.default_rng(16).random((30, 2))
  tours = orc.random_tours(30, 2, seed=17)
  want, ns_want = orc.two_opt(pts, tours, cap)
  assert ns_want == 1
  got, ns = gpu_two_opt(pts, tours, cap)
  assert ns == 1 and np.array_equal(got, want)
  tri = np.array([[0, 2, 1, 0]], dtype=np.int64)
  got, ns = gpu_two_opt(np.random.default_rng(18).random((3, 2)), tri, cap)
  assert ns == 0 and np.array_equal(got, tri)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 4, 9, 60])
@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_two_opt_non_finite_point_returns_input(n, bad):
  """torch.min propagates the NaN such a point puts in the change matrix: the reference stops before its first move."""
  pts = np.random.default_rng(19 + n).random((n, 2))
  pts[n // 2, 1] = bad
  tours = orc.random_tours(n, 2, seed=n)
  want, ns_want = orc.two_opt(pts, tours, 1000)
  assert ns_want == 0 and np.array_equal(want, tours)
  got, ns = gpu_two_opt(pts, tours, 1000)
  assert ns == 0 and np.array_equal(got, tours)

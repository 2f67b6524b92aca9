"""CPU oracle of the TSP decode rows (SURVEY 8f f2/f3).  TEST INFRASTRUCTURE ONLY: imported by tests/ (and nothing
in difusco_b200/).  numpy restatement of

  greedy_merge       utils/tsp_utils.py:89-145 + utils/cython_merge/cython_merge.pyx:19-120
  two_opt            utils/tsp_utils.py:12-49
  tour_length        utils/tsp_utils.py:148-156

and of the k-NN graph's order rule (co_datasets/tsp_graph_dataset.py:56-57 queries sklearn's KDTree):

  knn_bruteforce     float64 squared distances, ascending, exact ties to the smaller index

Pinned: tests/test_tsp_decode.py checks every function against tests/golden/tsp_decode.npz, which
tests/golden/make_golden.py produced by running the reference's own functions (Cython merge compiled from the
reference's .pyx, batched_two_opt_torch on the CPU device); two_opt also against tests/golden/two_opt_ties.npz (the
reference's 2-opt on the exact-tie instances of `tie_instances`).  tests/test_dataset_knn.py pins knn_bruteforce on
KDTree for inputs without ties.
"""
import numpy as np
import scipy.sparse


def symmetric_heat(n, heat, edge_index=None):
  """tsp_utils.py:99-110: float32 matrix A + A^T (dense heat) or coo(h,(r,c)) + coo(h,(c,r)) (sparse)."""
  if edge_index is None:
    return heat + heat.T
  r, c = edge_index
  return (scipy.sparse.coo_matrix((heat, (r, c)), shape=(n, n)).toarray() +
          scipy.sparse.coo_matrix((heat, (c, r)), shape=(n, n)).toarray())


def greedy_merge(points, sym):
  """cython_merge.pyx:19-104 -> (tour of n+1 nodes per tsp_utils.py:133-141, merge_iterations)."""
  n = points.shape[0]
  p = points.astype("double")
  with np.errstate(divide="ignore", invalid="ignore"):
    order = np.argsort((-sym.astype("double") / np.linalg.norm(p[:, None] - p, axis=-1)).flatten())
  frag = list(range(n))          # fragment id of each node
  nbrs = [[] for _ in range(n)]
  members = {i: [i] for i in range(n)}
  merged = iterations = 0
  for flat in order:
    iterations += 1
    i, j = int(flat) // n, int(flat) % n
    if frag[i] == frag[j] or len(nbrs[i]) == 2 or len(nbrs[j]) == 2:
      continue
    nbrs[i].append(j)
    nbrs[j].append(i)
    fi, fj = frag[i], frag[j]
    for v in members[fi]:
      frag[v] = fj
    members[fj] += members.pop(fi)
    merged += 1
    if merged == n - 1:
      break
  a, b = [v for v in range(n) if len(nbrs[v]) < 2]
  nbrs[a].append(b)
  nbrs[b].append(a)
  tour = [0]
  while len(tour) < n + 1:
    cand = [v for v in nbrs[tour[-1]] if len(tour) == 1 or v != tour[-2]]
    tour.append(max(cand))
  return tour, iterations


def two_opt(points, tours, max_iterations):
  """tsp_utils.py:12-49 in float64 numpy: every tour applies its own best move while the batch-wide best move
  improves by more than 1e-6."""
  pts = np.asarray(points, dtype=np.float64)
  tours = np.array(tours, dtype=np.int64)
  n = pts.shape[0]
  iterations = 0
  while True:
    head, nxt = pts[tours[:, :-1]], pts[tours[:, 1:]]                     # (B, n, 2)
    d = lambda u, v: np.sqrt(np.sum((u - v) ** 2, axis=-1))
    change = (d(head[:, :, None], head[:, None, :]) + d(nxt[:, :, None], nxt[:, None, :])
              - d(head, nxt)[:, :, None] - d(head, nxt)[:, None, :])
    change = np.triu(change, k=2)
    flat = change.reshape(len(tours), -1)
    pick = flat.argmin(axis=1)
    if not flat.min() < -1e-6:
      break
    for b, idx in enumerate(pick):
      i, j = idx // n, idx % n
      tours[b, i + 1:j + 1] = tours[b, i + 1:j + 1][::-1].copy()
    iterations += 1
    if iterations >= max_iterations:
      break
  return tours, iterations


def knn_bruteforce(queries, k, points=None):
  """k nearest of `points` (default: the queries themselves) for each query -> (Q, k) int64 indices: float64
  dx*dx + dy*dy (numpy never contracts to an FMA), each row ordered by (d2, j), so exact ties go to the smaller index
  and NaN comes after every number."""
  q = np.asarray(queries, dtype=np.float64)
  p = q if points is None else np.asarray(points, dtype=np.float64)
  j = np.arange(p.shape[0])
  out = np.empty((q.shape[0], k), dtype=np.int64)
  with np.errstate(over="ignore", invalid="ignore"):
    for r in range(q.shape[0]):
      dx, dy = p[:, 0] - q[r, 0], p[:, 1] - q[r, 1]
      out[r] = np.lexsort((j, dx * dx + dy * dy))[:k]
  return out


def tie_instances():
  """Deterministic instances whose pairwise distances tie exactly in float64: name -> (N, 2) float64 points."""
  rng = np.random.default_rng(20261015)
  grid = lambda a, b: np.stack(np.meshgrid(np.arange(a), np.arange(b), indexing="ij"), -1).reshape(-1, 2).astype(np.float64)
  out = {"grid12": grid(12, 12),                                     # integer grid, row-major labels
         "grid7x19": grid(7, 19)[rng.permutation(133)],              # non-square, shuffled labels
         "grid12s": grid(12, 12) / 11.0}                             # scaled to [0, 1]: rounding keeps many ties
  a = 2.0 * np.pi * np.arange(97) / 97.0
  out["polygon97"] = np.stack([np.cos(a), np.sin(a)], -1)[rng.permutation(97)]
  out["collinear64"] = np.stack([np.arange(64) / 64.0, np.full(64, 0.25)], -1)[rng.permutation(64)]
  base = rng.random((50, 2))
  out["repeat3"] = np.repeat(base, 3, axis=0)[rng.permutation(150)]
  base = rng.random((40, 2))
  out["repeat23"] = np.repeat(base, rng.integers(2, 4, 40), axis=0)
  out["repeat23"] = out["repeat23"][rng.permutation(len(out["repeat23"]))]
  mixed = np.concatenate([grid(10, 10), 9.0 * rng.random((20, 2))])
  out["gridmix"] = mixed[rng.permutation(120)]
  return out


def random_tours(n, b, seed):
  """b random tours over n nodes that start and end at node 0: (b, n + 1) int64."""
  rng = np.random.default_rng(seed)
  return np.stack([np.concatenate([[0], 1 + rng.permutation(n - 1), [0]]) for _ in range(b)]).astype(np.int64)


def tour_length(points, route):
  import warnings
  import scipy.spatial
  with warnings.catch_warnings():
    warnings.simplefilter("ignore", DeprecationWarning)
    dm = scipy.spatial.distance_matrix(points, points)
  total = 0
  for a, b in zip(route[:-1], route[1:]):
    total += dm[a, b]
  return total

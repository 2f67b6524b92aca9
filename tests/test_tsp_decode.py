"""SURVEY 8f rows f2 / f3: tour merge (host C++), 2-opt (CUDA) and the evaluator against the reference's outputs
(tests/golden/tsp_decode.npz, produced by the reference's own merge_tours / batched_two_opt_torch / TSPEvaluator)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))

from difusco_b200 import _cabi
from difusco_b200.utils import tsp_utils as tu
from oracle import tsp_decode_oracle as orc
from conftest import golden as _load_golden

# name, K (0 = dense input), parallel_sampling
CASES = [("s50", 8, 1), ("s200", 10, 2), ("s120r", 5, 1), ("s300g", 12, 1), ("s30full", 30, 2), ("s40fullg", 40, 1),
         ("d20", 0, 2), ("d45", 0, 1)]


def load(name, k):
  g = _load_golden("tsp_decode")
  return g, g[f"{name}/points"], g[f"{name}/heat"], (g[f"{name}/edge_index"] if k else None)


def is_tour(t, n):
  return len(t) == n + 1 and t[0] == t[-1] == 0 and sorted(t[:-1]) == list(range(n))


@pytest.mark.parametrize("name,k,par", CASES)
def test_merge_tours_matches_reference(name, k, par):
  g, pts, heat, ei = load(name, k)
  tours, it = tu.merge_tours(heat, pts, ei, sparse_graph=bool(k), parallel_sampling=par)
  want, want_it = g[f"{name}/tours"], float(g[f"{name}/merge_iterations"])
  closes_inside_graph = name in ("s30full", "s40fullg", "d20", "d45")
  if not closes_inside_graph:
    # These tours need entries outside the sparse graph, which all tie at key 0: their order is whatever numpy's
    # unstable argsort leaves, and that depends on the CPU's SIMD sort kernels.  If this machine's argsort differs
    # from the one that produced the fixture, the reference itself would not reproduce it here: pin on the oracle
    # (the reference's expression evaluated on this machine) instead.
    orc_res = [orc.greedy_merge(pts, orc.symmetric_heat(len(pts), part, ei)) for part in np.split(heat, par, axis=0)]
    if not np.array_equal(np.array([t for t, _ in orc_res]), want):
      want, want_it = np.array([t for t, _ in orc_res]), float(np.mean([i for _, i in orc_res]))
  assert np.array_equal(np.array(tours), want)
  assert it == want_it


@pytest.mark.parametrize("name,k,par", [c for c in CASES if c[0] in ("s50", "s30full", "s40fullg", "d20")])
def test_merge_oracle_matches_reference(name, k, par):
  g, pts, heat, ei = load(name, k)
  for p, part in enumerate(np.split(heat, par, axis=0)):
    sym = orc.symmetric_heat(len(pts), part if k else part[0], ei)
    tour, it = orc.greedy_merge(pts, sym)
    if name == "s50" and not np.array_equal(tour, g[f"{name}/tours"][p]):
      pytest.skip("this CPU's numpy argsort orders the exact ties at key 0 differently from the fixture's machine")
    assert np.array_equal(tour, g[f"{name}/tours"][p])
  # merge_iterations is the mean over the parallel samples; check it on the single-sample cases
  if par == 1:
    assert it == float(g[f"{name}/merge_iterations"])


def test_merge_fast_path_needs_no_dense_order():
  """Tours that close inside the non-zero entries come from the sparse scan alone (status 0), counter included."""
  g, pts, heat, ei = load("s30full", 30)
  for p, part in enumerate(np.split(heat, 2)):
    status, tour, it = _cabi.tsp_merge_sparse(pts, part, ei, mode=0)
    assert status == _cabi.MERGE_COMPLETE
    assert np.array_equal(tour, g["s30full/tours"][p])
  g, pts, heat, ei = load("s50", 8)
  assert _cabi.tsp_merge_sparse(pts, heat, ei, mode=0)[0] == _cabi.MERGE_INCOMPLETE


@pytest.mark.parametrize("name,k,par", CASES)
def test_merge_distance_completion_gives_valid_tours(name, k, par):
  g, pts, heat, ei = load(name, k)
  tours, _ = tu.merge_tours(heat, pts, ei, sparse_graph=bool(k), parallel_sampling=par, exact=False)
  ev = tu.TSPEvaluator(pts)
  for p, t in enumerate(tours):
    assert is_tour(t, len(pts))
    if not k or name.endswith("full") or name.endswith("fullg"):     # closes inside the candidates: same as exact
      assert np.array_equal(t, g[f"{name}/tours"][p])
    else:                                                             # nearest-end completion beats arbitrary ties
      assert ev.evaluate(t) <= g[f"{name}/cost_merged"][p] + 1e-9


def test_merge_exact_key_tie_falls_back_to_reference_order():
  """Two different pairs with bit-identical keys: the scan reports it and merge_tours resolves it like the reference
  (through the argsort); the oracle does the same argsort, so both agree."""
  pts = np.array([[0, 0], [1, 0], [1, 1], [0, 1], [0.5, 2.0]], dtype=np.float32)
  ei = np.array([[0, 1, 2, 3, 0, 1, 2], [1, 2, 3, 0, 4, 4, 4]], dtype=np.int64)
  heat = np.array([0.5, 0.5, 0.5, 0.5, 0.1, 0.2, 0.3], dtype=np.float32)
  assert _cabi.tsp_merge_sparse(pts, heat, ei, mode=0)[0] == _cabi.MERGE_AMBIGUOUS
  tours, it = tu.merge_tours(heat, pts, ei, sparse_graph=True)
  tour, it_o = orc.greedy_merge(pts, orc.symmetric_heat(5, heat, ei))
  assert tours[0] == list(tour) and it == it_o


def test_merge_argument_errors():
  pts = np.zeros((4, 2))
  with pytest.raises(ValueError):
    _cabi.tsp_merge_sparse(pts, np.ones(2, np.float32), np.array([[0, 9], [1, 2]]))       # node index out of range
  with pytest.raises(ValueError):
    _cabi.tsp_merge_sparse(pts[:2], np.ones(1, np.float32), np.array([[0], [1]]))          # n < 3
  with pytest.raises(ValueError):
    _cabi.tsp_merge_sparse(pts, np.ones(3, np.float32), np.array([[0, 1], [1, 2]]))        # heat / edge mismatch
  with pytest.raises(ValueError):
    _cabi.tsp_merge_order(4, np.array([1]))                                                # order cannot finish a tour


@pytest.mark.parametrize("name,k,par", CASES)
def test_evaluator_matches_reference(name, k, par):
  g, pts, _, _ = load(name, k)
  ev = tu.TSPEvaluator(pts)
  for p in range(par):
    assert ev.evaluate(g[f"{name}/tours"][p]) == g[f"{name}/cost_merged"][p]
    assert ev.evaluate(g[f"{name}/two_opt_1000"][p]) == g[f"{name}/cost_solved"][p]
    assert orc.tour_length(pts, g[f"{name}/tours"][p]) == g[f"{name}/cost_merged"][p]


@pytest.mark.parametrize("name,k,par", [c for c in CASES if c[0] in ("s50", "s200", "d20")])
def test_two_opt_oracle_matches_reference(name, k, par):
  g, pts, _, _ = load(name, k)
  for cap in (3, 1000):
    solved, ns = orc.two_opt(pts, g[f"{name}/tours"], cap)
    assert np.array_equal(solved, g[f"{name}/two_opt_{cap}"]) and ns == int(g[f"{name}/two_opt_{cap}_iters"])


@pytest.mark.parametrize("name", sorted(orc.tie_instances()))
def test_two_opt_oracle_matches_reference_on_ties(name):
  """tests/golden/two_opt_ties.npz: the reference's 2-opt on instances whose moves tie exactly (first occurrence wins),
  as one batch of three tours and as the first tour alone.  The fixture's points are the generator's."""
  g = _load_golden("two_opt_ties")
  pts = g[f"{name}/points"]
  assert np.array_equal(pts, orc.tie_instances()[name])
  for b in (1, 3):
    for cap in (1, 7, 1000):
      solved, ns = orc.two_opt(pts, g[f"{name}/tours"][:b], cap)
      assert ns == int(g[f"{name}/b{b}_cap{cap}_iters"]) and np.array_equal(solved, g[f"{name}/b{b}_cap{cap}"])


def test_two_opt_requires_cuda_device():
  with pytest.raises(RuntimeError):
    tu.batched_two_opt_torch(np.zeros((4, 2)), np.array([[0, 1, 2, 3, 0]]), device="cpu")


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,k,par", CASES)
def test_two_opt_matches_reference(name, k, par):
  g, pts, _, _ = load(name, k)
  for cap in (3, 1000):
    solved, ns = tu.batched_two_opt_torch(pts.astype("float64"), g[f"{name}/tours"], max_iterations=cap, device="cuda")
    assert ns == int(g[f"{name}/two_opt_{cap}_iters"])
    assert np.array_equal(solved, g[f"{name}/two_opt_{cap}"])


@pytest.mark.gpu
def test_two_opt_matches_oracle_on_random_tours():
  """Random permutations (many improving moves, several tiles per row, batch-wide stopping rule with B = 3)."""
  rng = np.random.default_rng(5)
  n = 150
  pts = rng.random((n, 2)).astype(np.float32)
  tours = np.stack([np.concatenate([[0], 1 + rng.permutation(n - 1), [0]]) for _ in range(3)]).astype(np.int64)
  for cap in (1, 40, 5000):
    want, ns_want = orc.two_opt(pts, tours, cap)
    got, ns = tu.batched_two_opt_torch(pts.astype("float64"), tours, max_iterations=cap, device="cuda")
    assert ns == ns_want and np.array_equal(got, want)


@pytest.mark.gpu
def test_two_opt_large_instance_properties():
  """TSP-2000 (beyond what the oracle finishes quickly): result is a permutation, never longer than the input,
  locally optimal when it stops by itself, and the iteration cap is honoured."""
  rng = np.random.default_rng(6)
  n = 2000
  pts = rng.random((n, 2))
  order = np.argsort(pts[:, 0] + 0.05 * rng.random(n))              # a crude but not random start
  order = np.concatenate([[0], order[order != 0], [0]])
  tours = np.stack([order, order]).astype(np.int64)
  ev = tu.TSPEvaluator(pts)
  capped, ns = tu.batched_two_opt_torch(pts, tours, max_iterations=25, device="cuda")
  assert ns == 25 and is_tour(list(capped[0]), n) and ev.evaluate(capped[0]) < ev.evaluate(tours[0])
  assert np.array_equal(capped[0], capped[1])
  solved, ns = tu.batched_two_opt_torch(pts, tours, max_iterations=100000, device="cuda")
  assert is_tour(list(solved[0]), n) and ev.evaluate(solved[0]) < ev.evaluate(capped[0])
  again, ns2 = tu.batched_two_opt_torch(pts, solved, max_iterations=100000, device="cuda")
  assert ns2 == 0 and np.array_equal(again, solved)


@pytest.mark.gpu
def test_two_opt_argument_errors():
  with pytest.raises(ValueError):
    tu.batched_two_opt_torch(np.zeros((4, 2)), np.array([[0, 1, 2, 7, 0]]), device="cuda")
  with pytest.raises(ValueError):
    tu.batched_two_opt_torch(np.zeros((4, 2)), np.array([[0, 1, 2, 0]]), device="cuda")


def _dataset_file(tmp, n, count, seed):
  rng = np.random.default_rng(seed)
  f = os.path.join(tmp, "tsp.txt")
  with open(f, "w") as fh:
    for _ in range(count):
      p = rng.random((n, 2))
      t = np.r_[0, 1 + rng.permutation(n - 1), 0]
      fh.write(" ".join(f"{float(x)!r} {float(y)!r}" for x, y in p) + " output " + " ".join(str(i + 1) for i in t) + "\n")
  return f


@pytest.mark.gpu
@pytest.mark.parametrize("sparse_factor,par,dtype", [(10, 2, "categorical"), (12, 1, "gaussian"), (-1, 2, "categorical")])
def test_tsp_test_step_end_to_end(sparse_factor, par, dtype, tmp_path):
  """TSPModel.test_step on a batch built like the reference's DataLoader builds it: dataset mirror (GPU kNN) ->
  fused denoise loop -> merge -> 2-opt -> evaluator.  Metrics keys are the reference's; every number is re-derived
  from the artefacts through the oracle."""
  import torch
  from types import SimpleNamespace as NS
  import gpu_util as G
  from difusco_b200 import synthetic as syn
  from difusco_b200.co_datasets.tsp_graph_dataset import TSPGraphDataset
  n = 60
  ds = TSPGraphDataset(_dataset_file(str(tmp_path), n, 2, 3), sparse_factor=sparse_factor)
  oc = 1 if dtype == "gaussian" else 2
  m = G.tsp_model(syn.make_encoder_weights(seed=oc, out_channels=oc), "tc", sparse_factor=sparse_factor,
                  parallel_sampling=par, diffusion_type=dtype, inference_diffusion_steps=4, two_opt_iterations=50,
                  save_numpy_heatmap=(par == 1), storage_path=str(tmp_path))
  item = ds[1]
  if sparse_factor > 0:
    idx, graph, pi, ei_ind, tour = item
    graph = NS(x=graph.x.cuda(), edge_index=graph.edge_index.cuda(), edge_attr=graph.edge_attr.cuda())
    batch = (idx.reshape(1, 1), graph, pi.reshape(1, 1).cuda(), ei_ind.reshape(1, 1).cuda(), tour.reshape(1, -1).cuda())
    pts, ei = graph.x.cpu().numpy(), graph.edge_index.cpu().numpy()
  else:
    idx, p, adj, tour = item
    batch = (idx.reshape(1, 1), p[None].cuda(), adj[None].cuda(), tour.reshape(1, -1).cuda())
    pts, ei = p.numpy(), None
  torch.manual_seed(1)
  metrics = m.test_step(batch, 0)
  assert set(metrics) == {"test/gt_cost", "test/2opt_iterations", "test/merge_iterations"}
  assert metrics["test/gt_cost"] == orc.tour_length(pts, tour.numpy().reshape(-1))
  heat = m.last_heatmap
  want_tours, its = [], []
  for part in np.split(heat, par, axis=0):
    t, it = orc.greedy_merge(pts, orc.symmetric_heat(n, part if ei is not None else part[0], ei))
    want_tours.append(t)
    its.append(it)
  assert metrics["test/merge_iterations"] == np.mean(its)
  solved, ns = orc.two_opt(pts, np.array(want_tours), 50)
  assert metrics["test/2opt_iterations"] == ns and np.array_equal(solved, m.last_solved_tours)
  assert m.last_solved_cost == min(orc.tour_length(pts, t) for t in solved)
  if par == 1:
    saved = np.load(os.path.join(str(tmp_path), "numpy_heatmap", "test-heatmap-1.npy"))
    assert np.array_equal(saved, heat)
    assert np.array_equal(np.load(os.path.join(str(tmp_path), "numpy_heatmap", "test-points-1.npy")), pts)


def test_dense_order_equals_the_reference_expression():
  """merge_tours' exact fallback argsorts keys that are built faster than the reference builds them; the visiting
  order must equal the reference expression's (cython_merge.pyx:21,38 on tsp_utils.py:104-110) on the same machine -
  duplicates, self loops, negative and zero heat included."""
  import scipy.sparse
  rng = np.random.default_rng(3)
  for n, e in ((40, 300), (333, 9000)):
    pts = rng.random((n, 2)).astype(np.float32)
    ei = rng.integers(0, n, (2, e))
    heat = rng.standard_normal(e).astype(np.float32)
    heat[::7] = 0.0
    sym = (scipy.sparse.coo_matrix((heat, (ei[0], ei[1])), shape=(n, n)).toarray() +
           scipy.sparse.coo_matrix((heat, (ei[1], ei[0])), shape=(n, n)).toarray())
    p = pts.astype("double")
    with np.errstate(divide="ignore", invalid="ignore"):
      want = np.argsort((-sym.astype("double") / np.linalg.norm(p[:, None] - p, axis=-1)).flatten())
    assert np.array_equal(tu._dense_order(pts, heat, ei), want)


def test_merge_tours_equals_oracle_on_random_graphs():
  """60 random instances (sparse with duplicate / self edges, negative and zero heat, coincident points; dense with
  parallel sampling): the C++ merge with its exact fallback and the numpy oracle (the reference's expression on this
  machine) give the same tours and the same merge_iterations."""
  rng = np.random.default_rng(11)
  for case in range(60):
    n = int(rng.integers(3, 60))
    pts = rng.random((n, 2)).astype(np.float32)
    if case % 7 == 0 and n > 4:
      pts[1] = pts[0]                                   # coincident points: +-inf keys
    if case % 3 == 0:                                   # dense input, two samples
      heat = rng.random((2, n, n)).astype(np.float32)
      tours, it = tu.merge_tours(heat, pts, None, sparse_graph=False, parallel_sampling=2)
      want = [orc.greedy_merge(pts, orc.symmetric_heat(n, h)) for h in heat]
    else:
      e = int(rng.integers(n, 6 * n))
      ei = rng.integers(0, n, (2, e))
      heat = rng.standard_normal(e).astype(np.float32) if case % 2 else rng.random(e).astype(np.float32)
      heat[:: int(rng.integers(2, 9))] = 0.0
      tours, it = tu.merge_tours(heat, pts, ei, sparse_graph=True)
      want = [orc.greedy_merge(pts, orc.symmetric_heat(n, heat, ei))]
    assert [list(map(int, w[0])) for w in want] == tours, case
    assert it == np.mean([w[1] for w in want]), case
    assert all(is_tour(t, n) for t in tours)
    fast, _ = (tu.merge_tours(heat, pts, None, sparse_graph=False, parallel_sampling=2, exact=False) if case % 3 == 0
               else tu.merge_tours(heat, pts, ei, sparse_graph=True, exact=False))
    assert all(is_tour(t, n) for t in fast), case      # the nearest-end completion always yields a Hamiltonian cycle


def test_merge_parallel_sampling_thread_pool_equals_sequential():
  """tsp_utils.py:121-126: more than 1000 nodes and parallel_sampling > 1 -> the samples are merged concurrently (thread
  pool around the GIL-free C++ merge); the tours must be the ones the sequential path gives, in the same order."""
  from sklearn.neighbors import KDTree
  rng = np.random.default_rng(7)
  n, k, P = 1200, 8, 3
  pts = rng.random((n, 2))
  _, idx = KDTree(pts).query(pts, k=k)
  ei = np.stack([np.repeat(np.arange(n), k), idx.reshape(-1)]).astype(np.int64)
  heat = rng.random((P, n * k)).astype(np.float32)
  par_tours, par_it = tu.merge_tours(heat, pts, ei, sparse_graph=True, parallel_sampling=P, exact=False)
  seq = [tu.merge_tours(heat[p:p + 1], pts, ei, sparse_graph=True, parallel_sampling=1, exact=False) for p in range(P)]
  assert par_tours == [s[0][0] for s in seq]
  assert np.isclose(par_it, np.mean([s[1] for s in seq]))
  for t in par_tours:
    assert len(t) == n + 1 and t[0] == t[-1] and sorted(t[:-1]) == list(range(n))

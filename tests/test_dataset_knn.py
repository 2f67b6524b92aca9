"""SURVEY 8(f) row f1: TSP line parsing + k-NN graph construction.  The oracle for the graph is the reference's own
algorithm, sklearn's KDTree(leaf_size=30, euclidean).query on float64 points (co_datasets/tsp_graph_dataset.py:56-57),
evaluated by the KDTree installed where the test runs.  The kernel alone is checked against `oracle.knn_bruteforce`
(exact ties to the smaller index), which is pinned on KDTree for inputs without ties."""
import os
import tempfile

import numpy as np
import pytest
import torch

from difusco_b200 import _cabi
from difusco_b200.co_datasets.tsp_graph_dataset import TSPGraphDataset, knn_edge_index_gpu
from oracle import tsp_decode_oracle as orc

TIES = orc.tie_instances()


def _points(kind, n, k):
  if kind == "random":
    return np.random.default_rng(n + k).random((n, 2))
  if kind == "grid160":
    return np.stack(np.meshgrid(np.arange(160), np.arange(160), indexing="ij"), -1).reshape(-1, 2).astype(np.float64)
  return TIES[kind]


def _kernel_rows(pts, k):
  """dfb_knn_graph alone (no tie resolution): (N, k) neighbour indices."""
  n = len(pts)
  d = torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float64)).cuda()
  out = torch.empty((2, n * k), dtype=torch.int64, device="cuda")
  _cabi.device_context(torch.cuda.current_device()).knn_graph(d.data_ptr(), n, k, 0, out.data_ptr(),
                                                            torch.cuda.current_stream().cuda_stream)
  return out[1].cpu().numpy().reshape(n, k)


# (kind, N, K); the ids of the first five are those the test has always had
KNN_CASES = ([pytest.param("random", n, k, id=f"{n}-{k}") for n, k in [(50, 5), (500, 50), (1000, 100), (2000, 50),
                                                                       (10000, 50)]]
             + [pytest.param(name, len(p), k, id=f"{name}-{k}") for name, p in sorted(TIES.items()) for k in (1, 5, 50)]
             + [pytest.param("random", n, k, id=f"random{n}-{k}")
                for n, ks in [(1, (1,)), (2, (1, 2)), (255, (1, 255)), (256, (1, 256)), (257, (1, 257)),
                              (513, (1, 300, 513))] for k in ks]
             + [pytest.param("random", 25600, 50, id="random25600-50"), pytest.param("grid160", 25600, 50, id="grid160-50")])


def test_knn_oracle_matches_kdtree_without_ties():
  from sklearn.neighbors import KDTree
  for n, k in [(1, 1), (7, 7), (300, 5), (1000, 50)]:
    pts = np.random.default_rng(n).random((n, 2))
    _, ref = KDTree(pts, leaf_size=30, metric="euclidean").query(pts, k=k, return_distance=True)
    assert np.array_equal(orc.knn_bruteforce(pts, k), ref)
  pts = TIES["grid12"]                       # ties: the oracle keeps the smaller index, KDTree need not
  d2 = np.sum((pts[orc.knn_bruteforce(pts, 6)] - pts[:, None]) ** 2, axis=-1)
  assert (np.diff(d2, axis=1) >= 0).all() and (orc.knn_bruteforce(pts, 6)[:, 0] == np.arange(len(pts))).all()


def _write(tmp, pts, tours):
  f = os.path.join(tmp, "tsp.txt")
  with open(f, "w") as fh:
    for p, t in zip(pts, tours):
      fh.write(" ".join(f"{float(x)!r} {float(y)!r}" for x, y in p) + " output " + " ".join(str(i + 1) for i in t) + "\n")
  return f


def test_line_parser_and_dense_item_cpu():
  rng = np.random.default_rng(0)
  pts = [rng.random((7, 2)) for _ in range(3)]
  tours = [np.r_[rng.permutation(7), 0] for _ in range(3)]
  for t in tours:
    t[-1] = t[0]
  with tempfile.TemporaryDirectory() as tmp:
    ds = TSPGraphDataset(_write(tmp, pts, tours), sparse_factor=-1)
    assert len(ds) == 3
    for i in range(3):
      p, t = ds.get_example(i)
      assert np.array_equal(p, pts[i]) and np.array_equal(t, tours[i])     # repr() round-trips float64 exactly
      idx, pt, adj, tour = ds[i]
      assert idx.tolist() == [i] and pt.dtype == torch.float32 and adj.shape == (7, 7)
      assert adj.sum() == 7 and all(adj[tours[i][j], tours[i][j + 1]] == 1 for j in range(7))


@pytest.mark.gpu
@pytest.mark.parametrize("kind,n,k", KNN_CASES)
def test_knn_graph_matches_kdtree(kind, n, k):
  """Random points; grids, a polygon, collinear and repeated points whose distances tie exactly; N on and either side
  of the 256-thread block stride; K = 1, K = N and K > 256; N = 25 600, the shared-memory limit."""
  from sklearn.neighbors import KDTree
  pts = _points(kind, n, k)
  assert pts.shape == (n, 2)
  _, ref = KDTree(pts, leaf_size=30, metric="euclidean").query(pts, k=k, return_distance=True)
  ei = knn_edge_index_gpu(pts, k).cpu().numpy()
  assert ei.shape == (2, n * k)
  assert np.array_equal(ei[0], np.repeat(np.arange(n), k))
  assert np.array_equal(ei[1].reshape(n, k), ref), "neighbour indices differ from the reference's KDTree query"
  on_device = knn_edge_index_gpu(torch.from_numpy(pts).cuda(), k).cpu().numpy()
  assert np.array_equal(on_device, ei)
  off = knn_edge_index_gpu(pts, k, node_offset=7 * n).cpu().numpy()
  assert np.array_equal(off, ei + 7 * n)
  # the kernel's own order: exact ties to the smaller index (every row when N is small, a stride of rows otherwise)
  rows = slice(None) if n <= 2000 else slice(None, None, 97)
  assert np.array_equal(_kernel_rows(pts, k)[rows], orc.knn_bruteforce(pts[rows], k, pts))


@pytest.mark.gpu
def test_knn_node_offset_beyond_32_bits():
  pts = TIES["grid12"]
  base = knn_edge_index_gpu(pts, 5).cpu().numpy()
  off = knn_edge_index_gpu(pts, 5, node_offset=3 * 2**31).cpu().numpy()
  assert np.array_equal(off, base + 3 * 2**31)


@pytest.mark.gpu
def test_knn_size_limit():
  pts = np.random.default_rng(1).random((25601, 2))
  with pytest.raises(NotImplementedError):
    knn_edge_index_gpu(pts, 5)


@pytest.mark.gpu
@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_knn_rejects_non_finite_points(bad):
  """KDTree raises ValueError on NaN and inf; so do the wrapper (host and device input) and, for host points, the
  C-ABI itself, before anything reaches the kernel."""
  import ctypes
  pts = np.random.default_rng(2).random((40, 2))
  pts[17, 0] = bad
  with pytest.raises(ValueError):
    knn_edge_index_gpu(pts, 5)
  with pytest.raises(ValueError):
    knn_edge_index_gpu(torch.from_numpy(pts).cuda(), 5)
  eng = _cabi.device_context(torch.cuda.current_device())
  out = torch.full((2, 40 * 5), -1, dtype=torch.int64, device="cuda")
  host = np.ascontiguousarray(pts)
  rc = _cabi.lib().dfb_knn_graph(eng._h, host.ctypes.data_as(ctypes.c_void_p), 40, 5, 0, out.data_ptr(), None)
  assert rc == _cabi.DFB_E_INVALID
  torch.cuda.synchronize()
  assert (out == -1).all()


@pytest.mark.gpu
def test_knn_overflowing_distances():
  """Finite coordinates near 1e200: far pairs' squared distances overflow to +inf and tie there.  Every row still
  lists K distinct indices in [0, N), in the fp64 oracle's order (the +inf ties by index, as no KDTree order exists)."""
  rng = np.random.default_rng(4)
  n, k = 300, 50
  pts = np.concatenate([rng.uniform(-1e153, 1e153, (150, 2)), rng.uniform(-1e200, 1e200, (150, 2))])[rng.permutation(n)]
  with np.errstate(over="ignore"):
    want = orc.knn_bruteforce(pts, k)
  got = knn_edge_index_gpu(pts, k).cpu().numpy()[1].reshape(n, k)
  assert all(len(set(r)) == k for r in got.tolist()) and got.min() >= 0 and got.max() < n
  assert np.array_equal(got, want)


def _check_sparse_item(pts, tour, k):
  from sklearn.neighbors import KDTree
  n = len(pts)
  with tempfile.TemporaryDirectory() as tmp:
    ds = TSPGraphDataset(_write(tmp, [pts], [tour]), sparse_factor=k)
    idx, graph, pind, eind, tour_t = ds[0]
  assert pind.tolist() == [n] and eind.tolist() == [n * k] and graph.x.dtype == torch.float32
  assert graph.edge_index.device.type == "cpu" and graph.edge_attr.device.type == "cpu" and graph.x.device.type == "cpu"
  _, ref = KDTree(pts, leaf_size=30, metric="euclidean").query(pts, k=k, return_distance=True)
  assert np.array_equal(graph.edge_index[0].numpy(), np.repeat(np.arange(n), k))
  assert np.array_equal(graph.edge_index[1].numpy().reshape(n, k), ref)
  succ = np.zeros(n, dtype=np.int64)
  succ[tour[:-1]] = tour[1:]
  assert np.array_equal(graph.edge_attr.numpy(), (ref == succ[:, None]).reshape(-1, 1))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["grid12", "repeat3"])
def test_sparse_item_on_tied_points_matches_reference_semantics(name):
  pts = TIES[name]
  tour = np.r_[np.random.default_rng(5).permutation(len(pts)), 0]
  tour[-1] = tour[0]
  _check_sparse_item(pts, tour, 8)


@pytest.mark.gpu
def test_sparse_item_layout_matches_reference_semantics():
  from sklearn.neighbors import KDTree
  rng = np.random.default_rng(3)
  n, k = 40, 6
  pts = [rng.random((n, 2))]
  tours = [np.r_[rng.permutation(n), 0]]
  tours[0][-1] = tours[0][0]
  with tempfile.TemporaryDirectory() as tmp:
    ds = TSPGraphDataset(_write(tmp, pts, tours), sparse_factor=k)
    idx, graph, pind, eind, tour = ds[0]
  assert pind.tolist() == [n] and eind.tolist() == [n * k] and graph.x.dtype == torch.float32
  # the item is made of CPU tensors like the reference's (DataLoader pin_memory / the model's own .to(device) work)
  assert graph.edge_index.device.type == "cpu" and graph.edge_attr.device.type == "cpu" and graph.x.device.type == "cpu"
  _, ref = KDTree(pts[0], leaf_size=30, metric="euclidean").query(pts[0], k=k, return_distance=True)
  assert np.array_equal(graph.edge_index[1].cpu().numpy().reshape(n, k), ref)
  succ = np.zeros(n, dtype=np.int64)
  succ[tours[0][:-1]] = tours[0][1:]
  want = (ref == succ[:, None]).reshape(-1, 1)
  assert np.array_equal(graph.edge_attr.cpu().numpy(), want)

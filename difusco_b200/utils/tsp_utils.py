"""Drop-in for the reference's difusco/utils/tsp_utils.py (SURVEY 8f rows f2 / f3): the decode that follows the
denoise path in TSPModel.test_step (pl_tsp_model.py:227-247).

  merge_tours(adj_mat, np_points, edge_index_np, sparse_graph=False, parallel_sampling=1)   tsp_utils.py:89-145
  batched_two_opt_torch(points, tour, max_iterations=1000, device="cpu")                    tsp_utils.py:12-49
  batched_two_opt_instances(points_list, tours_list, max_iterations=1000, device="cuda")   batched_two_opt_torch per
                                                                                           instance, in one call
  TSPEvaluator(points).evaluate(route)                                                      tsp_utils.py:148-156

merge_tours is host C++ in libdifusco_b200.so (csrc/tsp_decode.cuh): only the non-zero heat entries are sorted.  The
reference sorts all N*N entries of -A/dist; the entries outside the sparse graph all tie at key 0 and the order
numpy's (unstable) argsort leaves them in decides the last few insertions whenever the tour does not close inside
the graph's own edges.  `exact=True` (default) reproduces that bit for bit by running the same argsort for exactly
those cases; `exact=False` joins the leftover fragment ends by increasing distance instead and never builds an N*N
array (the only choice that scales to N = 10 k; documented divergence, DESIGN.md 9).

batched_two_opt_torch runs on the GPU only (two kernels per iteration, no (B, N, N) temporaries); `device` must be a
CUDA device.  There is no CPU fallback.
"""
import numpy as np
import scipy.sparse

from .. import _cabi

def _engine(device):
  import torch
  dev = torch.device(device)
  if dev.type != "cuda":
    raise RuntimeError("difusco_b200.batched_two_opt_torch runs on a CUDA device only (no CPU fallback)")
  idx = dev.index if dev.index is not None else torch.cuda.current_device()
  return _cabi.device_context(idx)   # shared with the model and the k-NN builder: one dfb_ctx per GPU


def batched_two_opt_torch(points, tour, max_iterations=1000, device="cuda"):
  """points (N, 2) float64 numpy, tour (B, N+1) int64 numpy -> (tour, iterations), both as the reference returns."""
  tours, iterations = _engine(device).two_opt(np.asarray(points, dtype=np.float64), tour, max_iterations)
  return tours, iterations


def batched_two_opt_instances(points_list, tours_list, max_iterations=1000, device="cuda"):
  """batched_two_opt_torch on many instances in one call: points_list[i] (n_i, 2), tours_list[i] (B_i, n_i + 1) of
  local node ids -> (tours_list, iterations_list), each instance exactly as batched_two_opt_torch on it alone (its own
  stopping rule and iteration cap).  Runs on torch's current stream of the device, so that under
  `torch.cuda.stream(s)` it runs beside the work of other streams."""
  import torch
  _cabi.two_opt_instances_arrays(points_list, tours_list)   # argument checks before any device work
  ctx = _engine(device)
  return ctx.two_opt_instances(points_list, tours_list, max_iterations,
                               torch.cuda.current_stream(ctx.device).cuda_stream)


def _dense_order(points, heat, edge_index):
  """The reference's visiting order (cython_merge.pyx:21, :35-38 on the matrix of tsp_utils.py:104-110): needed only
  to resolve its ties, so the SAME float64 keys go through the same np.argsort.  The keys are bit-identical to the
  reference's but cost a fraction: coo(h,(c,r)).toarray() is the transpose of coo(h,(r,c)).toarray(), and
  np.linalg.norm(p[:, None] - p, axis=-1) is sqrt(dx*dx + dy*dy) evaluated through a 3-D temporary
  (tests/test_tsp_decode.py checks both identities bit for bit)."""
  n = points.shape[0]
  half = scipy.sparse.coo_matrix((heat, (edge_index[0], edge_index[1])), shape=(n, n)).toarray()
  keys = (half + half.T).astype("double")
  pts = points.astype("double")
  dist = pts[:, 0][:, None] - pts[:, 0][None, :]
  np.multiply(dist, dist, out=dist)
  dy = pts[:, 1][:, None] - pts[:, 1][None, :]
  np.multiply(dy, dy, out=dy)
  np.add(dist, dy, out=dist)
  del dy
  np.sqrt(dist, out=dist)
  with np.errstate(divide="ignore", invalid="ignore"):
    np.negative(keys, out=keys)
    np.divide(keys, dist, out=keys)
  del dist
  return np.argsort(keys.reshape(-1))


def _complete_graph(n):
  idx = np.arange(n, dtype=np.int64)
  return np.stack([np.repeat(idx, n), np.tile(idx, n)])


def merge_tours(adj_mat, np_points, edge_index_np, sparse_graph=False, parallel_sampling=1, exact=True):
  """Returns (tours: list of parallel_sampling lists of N+1 ints, mean merge_iterations)."""
  points = np.asarray(np_points)
  n = points.shape[0]
  pts64 = points.astype("double")
  def one(part):
    if sparse_graph:
      edge_index, heat = np.asarray(edge_index_np), part.reshape(-1)
    else:                         # adj_mat[0] + adj_mat[0].T  ==  both orientations of the complete graph
      edge_index, heat = _complete_graph(n), part[0].reshape(-1)
    if heat.dtype != np.float32 and exact:
      # the reference builds its keys in the caller's dtype; a float64 heat map can order edges differently from its
      # float32 rounding, so it takes the reference's own dense formulation instead of the float32 sparse path
      status = _cabi.MERGE_INCOMPLETE
    else:
      status, tour, it = _cabi.tsp_merge_sparse(pts64, heat, edge_index, mode=0 if exact else 1)
    if status != _cabi.MERGE_COMPLETE:
      tour, it = _cabi.tsp_merge_order(n, _dense_order(points, heat, edge_index))
    return [int(v) for v in tour], it

  parts = np.split(np.asarray(adj_mat), parallel_sampling, axis=0)
  if n > 1000 and parallel_sampling > 1:
    # tsp_utils.py:121-126 runs the samples in a multiprocessing.Pool(parallel_sampling); the C++ merge releases the GIL
    # (ctypes), so a thread pool gives the same parallelism without pickling the heat maps
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=parallel_sampling) as pool:
      results = list(pool.map(one, parts))
  else:
    results = [one(part) for part in parts]
  tours = [r[0] for r in results]
  iterations = [r[1] for r in results]
  return tours, np.mean(iterations)


class TSPEvaluator(object):
  """Tour length under the reference's float64 distance matrix (scipy.spatial.distance_matrix ==
  sum(|x - y| ** 2) ** 0.5), evaluated only for the consecutive pairs of the route."""

  def __init__(self, points):
    self.points = np.asarray(points)
    self._p64 = self.points.astype(np.promote_types(self.points.dtype, "float64"))

  def evaluate(self, route):
    route = np.asarray(route).reshape(-1)
    a, b = self._p64[route[:-1]], self._p64[route[1:]]
    legs = np.sum(np.abs(b - a) ** 2, axis=-1) ** (1.0 / 2)
    total_cost = 0
    for leg in legs:
      total_cost += leg
    return total_cost

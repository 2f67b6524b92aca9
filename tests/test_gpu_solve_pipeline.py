"""Solving a stream of batches (TSPModel / MISModel.solve_batches) and the library calls it rests on: graph and point
preparation from host inputs that does not wait for the loops already enqueued, and the multi-instance 2-opt on a
stream of its own beside a running loop.  Run with -m gpu on an H100.

solve_batches must give exactly what solve_batch gives on each batch alone, on a fresh model: tours, costs, metrics and
the logged epoch means, bitwise."""
import numpy as np
import pytest
import torch

from difusco_b200 import synthetic as syn
import gpu_util as G

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
STEPS = 5


class _Graph(object):
  def __init__(self, **kw):
    self.__dict__.update(kw)


def _sparse_tsp_batch(sizes, seed):
  """A PyG-like collated batch of sparse TSP instances of (n, k) each; points and edges on the host."""
  parts = [(syn.tsp_points(n, seed, i), k) for i, (n, k) in enumerate(sizes)]
  parts = [(p, syn.knn_edge_index(p, k)) for p, k in parts]
  ptr = syn.node_ptr([p.shape[0] for p, _ in parts])
  x = torch.from_numpy(np.concatenate([p for p, _ in parts])).float()
  ei = torch.from_numpy(np.concatenate([e + ptr[i] for i, (_, e) in enumerate(parts)], 1))
  gt = torch.from_numpy(np.concatenate([np.concatenate([np.arange(p.shape[0]), [0]]) for p, _ in parts]))
  return (torch.arange(len(parts)), _Graph(x=x, edge_index=ei, edge_attr=torch.zeros((ei.shape[1], 1), dtype=torch.bool)),
          torch.tensor([p.shape[0] for p, _ in parts]), torch.tensor([e.shape[1] for _, e in parts]), gt)


def _dense_tsp_batch(b, seed):
  pts = np.stack([syn.tsp_points(64, seed, i) for i in range(b)]).astype(np.float32)
  gt = np.tile(np.concatenate([np.arange(64), [0]]), (b, 1))
  return torch.arange(b), torch.from_numpy(pts), torch.zeros(b, 64, 64), torch.from_numpy(gt)


def _mis_batch(sizes, seed):
  graphs = [syn.er_graph_edge_index(n, 0.1, seed, i) for i, n in enumerate(sizes)]
  ptr = syn.node_ptr(sizes)
  ei = np.concatenate([g + ptr[i] for i, g in enumerate(graphs)], 1)
  x = torch.from_numpy((syn.initial_noise(int(ptr[-1]), seed) > 0).astype(np.float32))
  return torch.arange(len(sizes)), _Graph(x=x, edge_index=torch.from_numpy(ei)), torch.tensor(sizes)


# A sequence that alternates between two shapes, has a one-instance batch, and ends with a batch larger than every
# earlier one (the context's arena grows mid-stream).
_SPARSE = [[(64, 16), (100, 32)], [(50, 8)], [(64, 16), (100, 32)], [(50, 8)], [(300, 20), (200, 20), (64, 16)]]
_CASES = {
    "tsp_p1": dict(kw=dict(sparse_factor=16)),
    "tsp_p4": dict(kw=dict(sparse_factor=16, parallel_sampling=4)),
    "tsp_s2": dict(kw=dict(sparse_factor=16, sequential_sampling=2)),
    "tsp_gauss": dict(kw=dict(sparse_factor=16, diffusion_type="gaussian"), w=1),
    "tsp_dense": dict(kw=dict(sparse_factor=-1, parallel_sampling=2), dense=[2, 1, 2, 1, 4]),
    "mis": dict(kw=dict(parallel_sampling=2), mis=[[40, 78, 130], [25], [40, 78, 130], [25], [300, 200, 130, 90]]),
}


def _model(case, w):
  c = _CASES[case]
  kw = dict(c["kw"], inference_diffusion_steps=STEPS)
  return G.mis_model(w, **kw) if "mis" in c else G.tsp_model(w, **kw)


def _batches(case):
  c = _CASES[case]
  if "mis" in c:
    return [_mis_batch(s, 600 + k) for k, s in enumerate(c["mis"])]
  if "dense" in c:
    return [_dense_tsp_batch(b, 500 + k) for k, b in enumerate(c["dense"])]
  return [_sparse_tsp_batch(s, 400 + k) for k, s in enumerate(_SPARSE)]


def _seeds(batch, k):
  n = batch[1].shape[0] if isinstance(batch[1], torch.Tensor) else len(batch[2])
  return [1000 * k + i for i in range(n)]


def _artefacts(m):
  return ([t.copy() for t in m.last_solved_tours] if hasattr(m, "last_solved_tours") else None,
          list(m.last_solved_costs))


def _same_results(a, b):
  assert len(a) == len(b)
  for x, y in zip(a, b):
    assert x.keys() == y.keys()
    for k in x:
      assert np.array_equal(np.asarray(x[k]), np.asarray(y[k])), k


def _same_artefacts(a, b):
  if a[0] is not None:
    assert len(a[0]) == len(b[0]) and all(np.array_equal(x, y) for x, y in zip(a[0], b[0]))
  assert np.array_equal(np.asarray(a[1]), np.asarray(b[1]))


@pytest.mark.parametrize("case", list(_CASES))
def test_solve_batches_is_solve_batch_on_each_batch(weights1, weights2, case):
  w = weights1 if _CASES[case].get("w") == 1 else weights2
  batches = _batches(case)
  seeds = [_seeds(b, k) for k, b in enumerate(batches)]
  m = _model(case, w)
  serial = _model(case, w)        # the same batches one solve_batch after another: the logged epoch means
  for k, got in enumerate(m.solve_batches(iter(batches), seeds)):
    fresh = _model(case, w)
    _same_results(got, fresh.solve_batch(batches[k], seeds[k]))
    _same_artefacts(_artefacts(m), _artefacts(fresh))
    serial.solve_batch(batches[k], seeds[k])
  assert k == len(batches) - 1
  assert m.logged_metrics() == serial.logged_metrics()


def test_a_loader_that_refills_its_tensors_in_place(weights2):
  """Batch k is decoded after batch k + 1 was drawn: it must not read batch k + 1's points, edges or tours."""
  batches = [_sparse_tsp_batch(s, 400 + k) for k, s in enumerate(_SPARSE[:1] * 3)]   # same shapes, new points
  seeds = [_seeds(b, k) for k, b in enumerate(batches)]
  buf = _sparse_tsp_batch(_SPARSE[0], 0)

  def refilled():
    for b in batches:
      buf[1].x.copy_(b[1].x)
      buf[1].edge_index.copy_(b[1].edge_index)
      buf[4].copy_(b[4])
      yield buf

  m = _model("tsp_p1", weights2)
  for k, got in enumerate(m.solve_batches(refilled(), seeds)):
    fresh = _model("tsp_p1", weights2)
    _same_results(got, fresh.solve_batch(batches[k], seeds[k]))
    _same_artefacts(_artefacts(m), _artefacts(fresh))


def test_an_error_surfaces_at_its_batch_and_the_model_stays_usable(weights2):
  batches = _batches("tsp_p1")[:3]
  seeds = [_seeds(b, k) for k, b in enumerate(batches)]
  for bad_seeds, bad_batch in ((seeds[1][:-1] + [0.5], batches[1]),
                               (seeds[1], batches[1][:2] + (torch.tensor([3]),) + batches[1][3:])):
    m = _model("tsp_p1", weights2)
    gen = m.solve_batches(batches[:1] + [bad_batch] + batches[2:], [seeds[0], bad_seeds, seeds[2]])
    first = next(gen)
    _same_results(first, _model("tsp_p1", weights2).solve_batch(batches[0], seeds[0]))
    with pytest.raises(ValueError):
      next(gen)
    with pytest.raises(StopIteration):
      next(gen)
    fresh = _model("tsp_p1", weights2)
    _same_results(m.solve_batch(batches[2], seeds[2]), fresh.solve_batch(batches[2], seeds[2]))
    _same_artefacts(_artefacts(m), _artefacts(fresh))


# ------------------------------------------------------------------------------------------------
# the library calls: host-input preparation does not wait for the stream; 2-opt beside a loop
# ------------------------------------------------------------------------------------------------
def _c2_graph():
  """16 x TSP-500 k=50 in one block-diagonal graph (host arrays)."""
  parts = [syn.tsp_points(500, 77, i) for i in range(16)]
  ptr = syn.node_ptr([500] * 16)
  ei = np.concatenate([syn.knn_edge_index(p, 50) + ptr[i] for i, p in enumerate(parts)], 1)
  return np.concatenate(parts).astype(np.float32), np.ascontiguousarray(ei, np.int64)


def _long_loop(m, pts, ei, steps):
  """Prepare (host inputs), enqueue a `steps`-step loop and record an event after it -> (device xt, event)."""
  m.model.set_graph(torch.from_numpy(ei), pts.shape[0])
  m.model.set_points(torch.from_numpy(pts))
  x = torch.from_numpy((syn.initial_noise(ei.shape[1], 9) > 0).astype(np.float32)).cuda()
  torch.cuda.synchronize()
  m._fused_loop(x, steps, seed=123)
  ev = torch.cuda.Event()
  ev.record()
  return x, ev


def _small_graph(seed):
  p = syn.tsp_points(100, seed, 0).astype(np.float32)
  return p, np.ascontiguousarray(syn.knn_edge_index(p, 16), np.int64)


def test_host_input_preparation_does_not_wait_for_the_stream(weights2):
  pts, ei = _c2_graph()
  m = G.tsp_model(weights2, sparse_factor=50)
  x_long, ev = _long_loop(m, pts, ei, 200)
  ctx = m.model.engine()
  p2, e2 = _small_graph(5)
  h_ei = e2.copy()                                      # pageable edges
  h_pts = torch.from_numpy(p2.copy()).pin_memory()      # pinned points: consumed before the call returns as well
  ctx.prepare_graph(h_ei.ctypes.data, p2.shape[0], e2.shape[1], 1, torch.cuda.current_stream().cuda_stream)
  ctx.set_points(h_pts.data_ptr(), torch.cuda.current_stream().cuda_stream)
  assert not ev.query(), "host-input preparation waited for the loop already enqueued"
  h_ei[...] = -7                                        # the caller's buffers are free as soon as the calls return
  h_pts.fill_(float("nan"))
  x2 = torch.from_numpy((syn.initial_noise(e2.shape[1], 3) > 0).astype(np.float32)).cuda()
  m._fused_loop(x2, STEPS, seed=44)
  torch.cuda.synchronize()
  ref = G.tsp_model(weights2, sparse_factor=50)
  x_ref, _ = _long_loop(ref, pts, ei, 200)
  torch.cuda.synchronize()
  assert torch.equal(x_long, x_ref)
  fresh = G.tsp_model(weights2, sparse_factor=50)
  want = fresh.denoise_heatmap(torch.from_numpy(p2), torch.from_numpy(e2),
                               torch.from_numpy((syn.initial_noise(e2.shape[1], 3) > 0).astype(np.float32)),
                               steps=STEPS, seed=44)
  assert torch.equal(x2, want)


def test_invalid_host_graphs_fail_and_leave_the_graph_in_use(weights2):
  m = G.tsp_model(weights2, sparse_factor=16)
  p, e = _small_graph(6)
  x0 = torch.from_numpy((syn.initial_noise(e.shape[1], 2) > 0).astype(np.float32))
  before = m.denoise_heatmap(torch.from_numpy(p), torch.from_numpy(e), x0, steps=STEPS, seed=8).clone()
  ctx = m.model.engine()
  two = np.concatenate([e, e + 100], 1)
  joined = two.copy()
  joined[1, 0] = 150
  bad = [(np.where(e == 3, 100, e), 100, None),   # an index out of range
         (joined, 200, [0, 100, 200]),           # an edge joining two instances
         (two, 200, [0, 100, 199]),              # node_ptr not ending at num_nodes
         (two, 200, [0, 120, 100, 200]),         # node_ptr not increasing
         (two, 200, [1, 100, 200])]              # node_ptr not starting at 0
  for ei, V, ptr in bad:
    ei = np.ascontiguousarray(ei, np.int64)
    with pytest.raises(ValueError):
      if ptr is None:
        ctx.prepare_graph(ei.ctypes.data, V, ei.shape[1], 1)
      else:
        ctx.prepare_graph_instances(ei.ctypes.data, V, ei.shape[1], np.asarray(ptr, np.int64))
  x = x0.cuda()
  m._fused_loop(x, STEPS, seed=8)
  assert torch.equal(x, before)


def _merged_tours(n_inst, seed):
  rng = np.random.default_rng(seed)
  pts = [syn.tsp_points(200 + 50 * i, seed, i).astype(np.float64) for i in range(n_inst)]
  tours = [np.stack([np.concatenate([rng.permutation(p.shape[0]), [0]]) for _ in range(2)]) for p in pts]
  for t in tours:
    t[:, -1] = t[:, 0]
  return pts, tours


def test_two_opt_beside_a_loop_is_the_serial_run(weights2):
  pts, ei = _c2_graph()
  p2o, t2o = _merged_tours(6, 31)
  m = G.tsp_model(weights2, sparse_factor=50)
  ctx = m.model.engine()                                # the loop's own context
  want_tours, want_its = ctx.two_opt_instances(p2o, t2o, 200)
  x_long, ev = _long_loop(m, pts, ei, 100)
  side = torch.cuda.Stream(priority=-1)
  got_tours, got_its = ctx.two_opt_instances(p2o, t2o, 200, side.cuda_stream)
  torch.cuda.synchronize()
  assert got_its == want_its
  assert all(np.array_equal(a, b) for a, b in zip(got_tours, want_tours))
  ref = G.tsp_model(weights2, sparse_factor=50)
  x_ref, _ = _long_loop(ref, pts, ei, 100)
  torch.cuda.synchronize()
  assert torch.equal(x_long, x_ref)


def test_two_opt_growth_does_not_recapture_the_loop(weights2):
  m = G.tsp_model(weights2, sparse_factor=16)
  p, e = _small_graph(7)
  x0 = torch.from_numpy((syn.initial_noise(e.shape[1], 2) > 0).astype(np.float32))
  first = m.denoise_heatmap(torch.from_numpy(p), torch.from_numpy(e), x0, steps=STEPS, seed=1).clone()
  captures = m.model.engine().loop_captures()
  pts, tours = _merged_tours(8, 32)                     # the first 2-opt on this context: its buffers grow
  m.model.engine().two_opt_instances(pts, tours, 5)
  again = m.denoise_heatmap(torch.from_numpy(p), torch.from_numpy(e), x0, steps=STEPS, seed=1)
  assert m.model.engine().loop_captures() == captures
  assert torch.equal(first, again)

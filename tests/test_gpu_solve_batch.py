"""Batches of TSP / MIS instances solved in one call: sampling keyed per instance (dfb_denoise_instances; the
instance_seeds argument of TSPModel.denoise_heatmap / MISModel.denoise_labels), the multi-instance 2-opt
(dfb_two_opt_instances, batched_two_opt_instances) and TSPModel / MISModel.solve_batch.  Run with -m gpu on an H100.

An instance's result must not depend on what else is in its batch.  Where every instance's edge count is a multiple of
32, the edge kernel's 32-edge message groups and the head GroupNorm blocks start at each instance, and a batched loop is
bitwise the instance's own loop with its seed."""
import numpy as np
import pytest
import torch

from conftest import rel_linf
from difusco_b200 import _cabi, synthetic as syn
from difusco_b200.utils import tsp_utils as tu
from oracle import difusco_oracle as dorc
from oracle import philox
from oracle import tsp_decode_oracle as orc
import gpu_util as G

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = torch.device("cuda")


def _local_ranks(owner, n_inst):
  """Rank of each element among its instance's elements, in the given (caller) order."""
  seen = np.zeros(n_inst, np.int64)
  out = np.empty(owner.size, np.int64)
  for k, s in enumerate(owner):
    out[k] = seen[s]
    seen[s] += 1
  return out


def _tsp_batch(sizes, seed, shuffle=False):
  """Ragged sparse TSP batch: (points, edge_index, node_ptr, owner instance of each edge, per-instance (pts, ei))."""
  parts = [(syn.tsp_points(n, seed, i), k) for i, (n, k) in enumerate(sizes)]
  parts = [(p, syn.knn_edge_index(p, k)) for p, k in parts]
  ptr = syn.node_ptr([p.shape[0] for p, _ in parts])
  ei = np.concatenate([e + ptr[i] for i, (_, e) in enumerate(parts)], 1)
  owner = np.concatenate([np.full(e.shape[1], i) for i, (_, e) in enumerate(parts)])
  if shuffle:
    perm = np.random.default_rng(seed).permutation(ei.shape[1])
    ei, owner = ei[:, perm], owner[perm]
  return np.concatenate([p for p, _ in parts]), np.ascontiguousarray(ei), ptr, owner, parts


def _mis_graphs(sizes, seed, multiple=1):
  """ER graphs (with self loops) of the given sizes; with multiple > 1 each one's edge count is a multiple of it."""
  out = []
  for i, n in enumerate(sizes):
    for tag in range(1000):
      e = syn.er_graph_edge_index(n, 0.1, seed + tag, i)
      if e.shape[1] % multiple == 0:
        out.append(e)
        break
    else:
      raise AssertionError("no graph with an aligned edge count")
  return out


def _draw_check(m, x0, rec, owner, seeds, categorical):
  """Every recorded sample (and Gaussian DDPM update) uses Philox at (seeds[instance], step, local rank)."""
  local = _local_ranks(owner, len(seeds))
  sd = np.asarray(seeds, np.uint64)[owner]
  steps = rec["xt"].shape[0]
  for s in range(steps - 1 if categorical else steps):
    if categorical:
      u = np.array([philox.uniform(int(a), s, np.array([int(b)]))[0] for a, b in zip(sd, local)], np.float32)
      assert np.array_equal(rec["xt"][s], (u < np.clip(rec["p"][s], 0, 1)).astype(np.float32)), s
    else:
      c, _ = m.posterior_consts(*_sched(m, steps)[s])
      if c[3] == 0:
        continue
      xin = x0 if s == 0 else rec["xt"][s - 1]
      l0 = rec["out"][s][:, 0]
      y = np.float32(c[0]) * (xin - np.float32(c[1]) * l0) + np.float32(c[2]) * l0
      z = np.array([philox.normal(int(a), s, np.array([int(b)]))[0] for a, b in zip(sd, local)])
      assert np.allclose(rec["xt"][s], y + np.float32(c[3]) * z, rtol=1e-5, atol=1e-5), s


def _sched(m, steps):
  return list(dorc.inference_schedule(m.args.inference_schedule, 1000, steps))


# ------------------------------------------------------------------------------------------------
# (a) the draws of dfb_denoise_instances are Philox at (seed_s, step, local)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["tsp", "mis", "gauss_ddpm"])
def test_draws_are_keyed_per_instance(weights2, weights1, case):
  steps = 6
  seeds = [11, 2 ** 63 + 5, 7, 123456789, 42]
  if case == "mis":
    graphs = _mis_graphs([20, 57, 131, 300, 203], 93)
    ptr = syn.node_ptr([20, 57, 131, 300, 203])
    ei = np.concatenate([g + ptr[i] for i, g in enumerate(graphs)], 1)
    ei = ei[:, np.random.default_rng(3).permutation(ei.shape[1])]
    owner = np.searchsorted(ptr, np.arange(ptr[-1]), side="right") - 1
    x0 = (syn.initial_noise(int(ptr[-1]), 4) > 0).astype(np.float32)
    m = G.mis_model(weights2, inference_diffusion_steps=steps)
    _, tr = m.denoise_labels(G.cu(ei), G.cu(x0), record_steps="all", node_ptr=ptr, instance_seeds=seeds)
  else:
    gauss = case == "gauss_ddpm"
    pts, ei, ptr, owner, _ = _tsp_batch([(1, 1), (7, 7), (50, 20), (200, 20), (500, 50)], 91, shuffle=True)
    z = syn.initial_noise(ei.shape[1], 5)
    x0 = z if gauss else (z > 0).astype(np.float32)
    m = G.tsp_model(weights1 if gauss else weights2, sparse_factor=20, inference_diffusion_steps=steps,
                    **(dict(diffusion_type="gaussian", inference_trick=None) if gauss else {}))
    _, tr = m.denoise_heatmap(G.cu(pts), G.cu(ei), G.cu(x0), record_steps="all", node_ptr=ptr, instance_seeds=seeds)
  tr = {k: v.cpu().numpy() for k, v in tr.items()}
  _draw_check(m, x0, tr, owner, seeds, case != "gauss_ddpm")


# ------------------------------------------------------------------------------------------------
# (b) independence from the batch, bitwise, when every instance is aligned to 32 edges
# ------------------------------------------------------------------------------------------------
def _alone_and_batched_tsp(m, parts, seeds, order, steps):
  """final heat map of each instance alone (seed) and of the batch in `order` (instance_seeds) -> (alone, batched)."""
  alone = []
  for (p, e), s in zip(parts, seeds):
    x0 = (syn.initial_noise(e.shape[1], 1000 + p.shape[0]) > 0).astype(np.float32)
    alone.append(m.denoise_heatmap(G.cu(p), G.cu(e), G.cu(x0), steps=steps, seed=s).cpu().numpy())
  sel = [parts[i] for i in order]
  ptr = syn.node_ptr([p.shape[0] for p, _ in sel])
  ei = np.concatenate([e + ptr[j] for j, (_, e) in enumerate(sel)], 1)
  x0 = np.concatenate([(syn.initial_noise(e.shape[1], 1000 + p.shape[0]) > 0).astype(np.float32) for p, e in sel])
  out = m.denoise_heatmap(G.cu(np.concatenate([p for p, _ in sel])), G.cu(ei), G.cu(x0), steps=steps,
                          node_ptr=ptr, instance_seeds=[seeds[i] for i in order]).cpu().numpy()
  lens = [e.shape[1] for _, e in sel]
  return alone, np.split(out, np.cumsum(lens)[:-1])


@pytest.mark.parametrize("order", [[0, 1, 2], [2, 0, 1], [1], list(range(3)) * 5 + [0, 2]])
def test_aligned_tsp_batch_is_bitwise_each_instance_alone(weights2, order):
  steps = 8
  parts = [(syn.tsp_points(n, 71, i), None) for i, n in enumerate([64, 100, 64])]
  parts = [(p, syn.knn_edge_index(p, k)) for (p, _), k in zip(parts, [16, 32, 16])]
  assert all(e.shape[1] % 32 == 0 for _, e in parts)
  seeds = [5, 6, 7]
  m = G.tsp_model(weights2, sparse_factor=16, inference_diffusion_steps=steps)
  alone, got = _alone_and_batched_tsp(m, parts, seeds, order, steps)
  for j, i in enumerate(order):
    assert np.array_equal(got[j], alone[i]), (order, j)


def test_aligned_dense_batch_is_bitwise_each_sample_alone(weights2):
  steps, V = 6, 64
  m = G.tsp_model(weights2, sparse_factor=-1, inference_diffusion_steps=steps)
  pts = [syn.tsp_points(V, 72, i) for i in range(3)]
  x0 = [(syn.initial_noise(V * V, 73 + i) > 0).astype(np.float32).reshape(1, V, V) for i in range(3)]
  seeds = [9, 10, 11]
  alone = [m.denoise_heatmap(G.cu(p[None]), None, G.cu(x), seed=s).cpu().numpy() for p, x, s in zip(pts, x0, seeds)]
  for order in ([0, 1, 2], [2, 1, 0]):
    got = m.denoise_heatmap(G.cu(np.stack([pts[i] for i in order])), None, G.cu(np.concatenate([x0[i] for i in order])),
                            instance_seeds=[seeds[i] for i in order]).cpu().numpy()
    for j, i in enumerate(order):
      assert np.array_equal(got[j:j + 1], alone[i]), (order, j)


def test_aligned_mis_batch_is_bitwise_each_graph_alone(weights2):
  steps = 8
  sizes = [40, 78, 130]   # even: 2m + n edges (both directions, self loops)
  graphs = _mis_graphs(sizes, 300, multiple=32)
  seeds = [3, 1 << 40, 99]
  m = G.mis_model(weights2, inference_diffusion_steps=steps)
  x0 = [(syn.initial_noise(n, 400 + n) > 0).astype(np.float32) for n in sizes]
  alone = [m.denoise_labels(G.cu(g), G.cu(x), seed=s).cpu().numpy() for g, x, s in zip(graphs, x0, seeds)]
  for order in ([0, 1, 2], [2, 0, 1], [1], [0, 1, 2] * 5 + [2, 1]):
    ptr = syn.node_ptr([sizes[i] for i in order])
    ei = np.concatenate([graphs[i] + ptr[j] for j, i in enumerate(order)], 1)
    got = m.denoise_labels(G.cu(ei), G.cu(np.concatenate([x0[i] for i in order])), node_ptr=ptr,
                           instance_seeds=[seeds[i] for i in order]).cpu().numpy()
    for j, i in enumerate(order):
      assert np.array_equal(got[ptr[j]:ptr[j + 1]], alone[i]), (order, j)


# ------------------------------------------------------------------------------------------------
# (c) arbitrary ragged sizes: the 32-edge message groups straddle instances, so the logits differ from each instance
# alone in the last bits.  Each instance's trajectory equals its alone run until a sample differs, and a sample may
# differ only where its draw lies within 1e-4 of p; every recorded step meets the value-range rule against the fp64
# oracle on the instance alone, evaluated on the recorded input state.
# ------------------------------------------------------------------------------------------------
TOL = 1e-4
P_BIG = 1e-3


def _p_errors(p, ref):
  big = ref >= P_BIG
  return float(np.abs(p - ref).max()), float(np.abs(p[big] / ref[big] - 1).max()) if big.any() else 0.0


def _ragged_case(task, w, steps, seeds):
  """Batched record + per instance (oracle fn, x0, element mask, alone run)."""
  if task == "tsp":
    pts, ei, ptr, owner, _ = _tsp_batch([(1, 1), (7, 7), (50, 20), (200, 20), (500, 50)], 95, shuffle=True)
    x0 = (syn.initial_noise(ei.shape[1], 96) > 0).astype(np.float32)
    m = G.tsp_model(w, sparse_factor=20, inference_diffusion_steps=steps)
    final, tr = m.denoise_heatmap(G.cu(pts), G.cu(ei), G.cu(x0), record_steps="all", node_ptr=ptr,
                                  instance_seeds=seeds)
    inst = []
    for i in range(len(seeds)):
      sel = owner == i
      p, e = pts[ptr[i]:ptr[i + 1]], np.ascontiguousarray(ei[:, sel] - ptr[i])   # its edges in the batch's order
      inst.append((sel, x0[sel], lambda x, t, dt, p=p, e=e: dorc.encoder_forward_sparse_tsp(
          dorc.Weights(w, dt), p, x, np.array([t]), e).numpy(),
          lambda s, p=p, e=e, x=x0[sel]: m.denoise_heatmap(G.cu(p), G.cu(e), G.cu(x), seed=s, record_steps="all")))
  else:
    sizes = [20, 57, 131, 300, 203]
    ptr = syn.node_ptr(sizes)
    ei = np.concatenate([g + ptr[i] for i, g in enumerate(_mis_graphs(sizes, 97))], 1)
    ei = np.ascontiguousarray(ei[:, np.random.default_rng(98).permutation(ei.shape[1])])
    edge_owner = np.searchsorted(ptr, ei[0], side="right") - 1
    owner = np.searchsorted(ptr, np.arange(ptr[-1]), side="right") - 1
    x0 = (syn.initial_noise(int(ptr[-1]), 99) > 0).astype(np.float32)
    m = G.mis_model(w, inference_diffusion_steps=steps)
    final, tr = m.denoise_labels(G.cu(ei), G.cu(x0), record_steps="all", node_ptr=ptr, instance_seeds=seeds)
    inst = []
    for i in range(len(seeds)):
      sel = owner == i
      e = np.ascontiguousarray(ei[:, edge_owner == i] - ptr[i])
      inst.append((sel, x0[sel], lambda x, t, dt, e=e: dorc.encoder_forward_mis(
          dorc.Weights(w, dt), x, np.array([t]), e).numpy(),
          lambda s, e=e, x=x0[sel]: m.denoise_labels(G.cu(e), G.cu(x), seed=s, record_steps="all")))
  return final.cpu().numpy(), {k: v.cpu().numpy() for k, v in tr.items()}, inst


@pytest.mark.parametrize("task", ["tsp", "mis"])
def test_ragged_batch_matches_each_instance_alone(weights2, task):
  steps = 4
  seeds = [3, 1 << 50, 17, 2 ** 64 - 1, 8]
  torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
  final, tr, inst = _ragged_case(task, weights2, steps, seeds)
  sched = dorc.inference_schedule("cosine", 1000, steps)
  _, Q_bar = dorc.categorical_tables(1000, "linear")
  to_end = 0
  for i, (sel, x0, fwd, alone) in enumerate(inst):
    fa, ta = alone(seeds[i])
    ta = {k: v.cpu().numpy() for k, v in ta.items()}
    tb = {k: tr[k][:, sel] for k in ("xt", "p", "out")}
    same = True        # the batched trajectory still equals the alone one
    for s, (t1, t2) in enumerate(sched):
      xin = x0 if s == 0 else tb["xt"][s - 1]
      r64, r32 = fwd(xin, t1, torch.float64), fwd(xin, t1, torch.float32)
      got, yard = rel_linf(tb["out"][s], r64), rel_linf(r32, r64)
      assert got <= max(G.TOL["tc"], 4 * yard), (task, i, s, got, yard)
      x = torch.as_tensor(xin)
      p64 = dorc.categorical_posterior(Q_bar, t1, t2, torch.as_tensor(r64).softmax(-1), x.double())[0].numpy()
      p32 = dorc.categorical_posterior(Q_bar, t1, t2, torch.as_tensor(r32).softmax(-1), x.float())[0].numpy()
      e_abs, e_rel = _p_errors(tb["p"][s].astype(np.float64), p64)
      y_abs, y_rel = _p_errors(p32.astype(np.float64), p64)
      assert e_abs <= max(TOL, 4 * y_abs) and e_rel <= max(TOL, 4 * y_rel), (task, i, s, e_abs, e_rel, y_abs, y_rel)
      if not same:
        continue
      if s < steps - 1:
        u = philox.uniform(seeds[i], s, np.arange(x0.size))
        near = (np.abs(u - ta["p"][s]) < TOL) | (np.abs(u - tb["p"][s]) < TOL)
        diff = ta["xt"][s] != tb["xt"][s]
        assert not (diff & ~near).any(), (task, i, s, int((diff & ~near).sum()))
        same = not diff.any()
      else:
        assert np.abs(fa.cpu().numpy() - final[sel]).max() <= TOL, (task, i)
        to_end += 1
  assert to_end >= len(inst) - 1, to_end   # a flip needs |u - p| within p's last-bit difference: expect none, allow one


# ------------------------------------------------------------------------------------------------
# (d) captured and plain launches agree; one captured graph serves every seed set; dfb_denoise is unchanged
# ------------------------------------------------------------------------------------------------
def test_capture_seed_sets_and_the_plain_loop(weights2):
  steps = 6
  pts, ei, ptr, _, _ = _tsp_batch([(7, 7), (50, 20), (120, 20)], 81, shuffle=True)
  d_pts, d_ei, d_x0 = G.cu(pts), G.cu(ei), G.cu((syn.initial_noise(ei.shape[1], 82) > 0).astype(np.float32))
  m = G.tsp_model(weights2, sparse_factor=20, inference_diffusion_steps=steps)
  run = lambda **kw: m.denoise_heatmap(d_pts, d_ei, d_x0, node_ptr=ptr, **kw).cpu().numpy()
  plain_old = run(seed=5)
  ctx = m.model.engine()
  captures = ctx.loop_captures()
  assert captures >= 1
  a, b = run(instance_seeds=[1, 2, 3]), run(instance_seeds=[4, 5, 6])
  assert np.array_equal(run(instance_seeds=[1, 2, 3]), a)
  assert np.array_equal(run(seed=5), plain_old)
  assert not np.array_equal(a, b)
  assert ctx.loop_captures() == captures        # both seed sets and the call seed replayed the one captured graph
  ctx.set_graph_capture(False)
  try:
    assert np.array_equal(run(instance_seeds=[1, 2, 3]), a) and np.array_equal(run(instance_seeds=[4, 5, 6]), b)
    assert np.array_equal(run(seed=5), plain_old)
  finally:
    ctx.set_graph_capture(True)


def test_denoise_instances_rejects_bad_arguments(weights2):
  steps = 4
  pts, ei, ptr, _, _ = _tsp_batch([(7, 7), (50, 20)], 83)
  m = G.tsp_model(weights2, sparse_factor=20, inference_diffusion_steps=steps)
  x = G.cu((syn.initial_noise(ei.shape[1], 84) > 0).astype(np.float32))
  m.denoise_heatmap(G.cu(pts), G.cu(ei), x, node_ptr=ptr, instance_seeds=[1, 2])
  ctx = m.model.engine()
  t1 = (C_int := _cabi.C.c_int32 * steps)(*[900, 600, 300, 100])
  cs = (_cabi.C.c_float * (4 * steps))(*([0.5] * 4 * steps))
  ls = C_int(0, 0, 0, 1)
  rec = C_int(0)
  d3 = torch.tensor([1, 2, 3], dtype=torch.int64, device=DEV)
  h2 = np.array([1, 2], np.uint64)
  before = x.clone()
  st = torch.cuda.current_stream().cuda_stream
  for seeds, n in ((None, 2), (d3.data_ptr(), 3), (d3.data_ptr(), 1), (h2.ctypes.data, 2)):
    rc = _cabi.lib().dfb_denoise_instances(ctx._h, 0, x.data_ptr(), steps, t1, cs, ls, seeds, n, 0, rec, None, None,
                                           None, st)
    assert rc == _cabi.DFB_E_INVALID, (seeds, n)
  assert torch.equal(x, before)
  with pytest.raises(ValueError):
    m.denoise_heatmap(G.cu(pts), G.cu(ei), x, node_ptr=ptr, instance_seeds=[1, 2, 3])
  with pytest.raises(ValueError):
    m.denoise_heatmap(G.cu(pts), G.cu(ei), x, node_ptr=ptr, instance_seeds=[1, 2], seed=4)


# ------------------------------------------------------------------------------------------------
# multi-instance 2-opt: each instance exactly dfb_two_opt on it alone
# ------------------------------------------------------------------------------------------------
def _per_instance(points_list, tours_list, cap):
  eng = _cabi.device_context(torch.cuda.current_device())
  return [eng.two_opt(p, t, cap) for p, t in zip(points_list, tours_list)]


def _check_two_opt(points_list, tours_list, cap, oracle=True):
  got, its = tu.batched_two_opt_instances(points_list, tours_list, cap)
  for i, (want, n) in enumerate(_per_instance(points_list, tours_list, cap)):
    assert its[i] == n and np.array_equal(got[i], want), i
    if oracle:
      o, on = orc.two_opt(points_list[i], tours_list[i], cap)
      assert on == n and np.array_equal(o, want), i
  return its


def test_two_opt_instances_on_the_tie_fixture():
  g = np.load("tests/golden/two_opt_ties.npz")
  names = sorted({k.split("/")[0] for k in g.files})
  for cap in (1, 7, 1000):
    got, its = tu.batched_two_opt_instances([g[f"{n}/points"] for n in names], [g[f"{n}/tours"] for n in names], cap)
    for i, n in enumerate(names):
      assert np.array_equal(got[i], g[f"{n}/b3_cap{cap}"]) and its[i] == int(g[f"{n}/b3_cap{cap}_iters"]), (n, cap)


def test_two_opt_instances_random_optimal_capped_and_nan():
  rng = np.random.default_rng(61)
  sizes = [3, 4, 30, 65, 129, 200, 50]
  pts = [rng.random((n, 2)) for n in sizes]
  tours = [orc.random_tours(n, b, 62 + n) for n, b in zip(sizes, [1, 2, 3, 2, 4, 1, 2])]
  solved, _ = orc.two_opt(pts[2], tours[2], 10 ** 6)
  tours[2] = solved                                     # already optimal: stops at 0 iterations
  nan_pts = pts[5].copy()
  nan_pts[7, 1] = np.nan
  pts[5] = nan_pts
  its = _check_two_opt(pts, tours, 25)
  assert its[2] == 0 and its[5] == 0 and 25 in its and len(set(its)) > 2
  _check_two_opt(pts, tours, 1000)


def test_two_opt_instances_mixed_sizes_and_many_tours():
  rng = np.random.default_rng(63)
  pts = [rng.random((3, 2)), rng.random((10000, 2)), rng.random((50, 2))]
  tours = [orc.random_tours(3, 2, 1), orc.random_tours(10000, 2, 2), orc.random_tours(50, 3, 3)]
  _check_two_opt(pts, tours, 5, oracle=False)
  n_inst = 4096
  sizes = rng.integers(3, 40, n_inst)
  counts = np.full(n_inst, 17)
  counts[:70000 - 17 * n_inst] += 1          # 70 000 tours in all: more than dfb_two_opt's 65 535 per call
  pts = [rng.random((int(n), 2)) for n in sizes]
  tours = [orc.random_tours(int(n), int(b), 1000 + i) for i, (n, b) in enumerate(zip(sizes, counts))]
  got, its = tu.batched_two_opt_instances(pts, tours, 1000)
  for i in (0, 1, 77, 2048, 4095):
    want, n = _per_instance([pts[i]], [tours[i]], 1000)[0]
    assert its[i] == n and np.array_equal(got[i], want), i


def test_two_opt_instances_rejects_bad_arguments():
  rng = np.random.default_rng(64)
  pts = [rng.random((10, 2)), rng.random((12, 2))]
  tours = [orc.random_tours(10, 2, 1), orc.random_tours(12, 1, 2)]
  P, nptr, tptr, T = _cabi.two_opt_instances_arrays(pts, tours)
  eng = _cabi.device_context(torch.cuda.current_device())
  its = np.zeros(2, np.int64)
  bad_t = T.copy()
  bad_t[3] = 10
  cases = [(P, nptr, 2, tptr, T), (P, np.array([0, 2, 22]), 2, tptr, T), (P, nptr, 2, np.array([0, 0, 3]), T),
           (P, nptr, 2, np.array([1, 2, 3]), T), (P, nptr, 0, tptr, T), (P, nptr, 2, tptr, bad_t)]
  for k, (p, n, ni, t, tr) in enumerate(cases[1:]):
    tr = tr.copy()
    before = tr.copy()
    n, t = np.ascontiguousarray(n, np.int64), np.ascontiguousarray(t, np.int64)
    rc = _cabi.lib().dfb_two_opt_instances(eng._h, p.ctypes.data, n.ctypes.data, ni, t.ctypes.data, tr.ctypes.data,
                                           100, its.ctypes.data, 0)
    assert rc == _cabi.DFB_E_INVALID and np.array_equal(tr, before), k
  rc = _cabi.lib().dfb_two_opt_instances(eng._h, P.ctypes.data, nptr.ctypes.data, 2, tptr.ctypes.data, None, 100,
                                         its.ctypes.data, 0)
  assert rc == _cabi.DFB_E_INVALID


# ------------------------------------------------------------------------------------------------
# solve_batch end to end: a batch equals each instance alone; the decode is test_step's
# ------------------------------------------------------------------------------------------------
class _Graph(object):
  def __init__(self, **kw):
    self.__dict__.update(kw)


def _sparse_tsp_batch(parts):
  """A PyG-like collated batch of sparse TSP instances (points, edge_index local, tour)."""
  ptr = syn.node_ptr([p.shape[0] for p, _, _ in parts])
  x = torch.from_numpy(np.concatenate([p for p, _, _ in parts])).float()
  ei = torch.from_numpy(np.concatenate([e + ptr[i] for i, (_, e, _) in enumerate(parts)], 1))
  lab = torch.zeros((ei.shape[1], 1), dtype=torch.bool)
  gt = torch.from_numpy(np.concatenate([t for _, _, t in parts]))
  return (torch.arange(len(parts)), _Graph(x=x, edge_index=ei, edge_attr=lab),
          torch.tensor([p.shape[0] for p, _, _ in parts]), torch.tensor([e.shape[1] for _, e, _ in parts]), gt.cuda())


def _tsp_parts(sizes, seed):
  out = []
  for i, (n, k) in enumerate(sizes):
    p = syn.tsp_points(n, seed, i)
    out.append((p, syn.knn_edge_index(p, k), np.concatenate([np.arange(n), [0]]).astype(np.int64)))
  return out


def _same(a, b):
  assert a.keys() == b.keys()
  for k in a:
    assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


@pytest.mark.parametrize("copies", [1, 4])
def test_sparse_tsp_solve_batch_equals_each_instance_alone(weights2, copies):
  m = G.tsp_model(weights2, sparse_factor=16, inference_diffusion_steps=5, parallel_sampling=copies,
                  sequential_sampling=2)
  parts = _tsp_parts([(64, 16), (100, 32), (64, 16)], 51)
  seeds = [17, 18, 19]
  got = m.solve_batch(_sparse_tsp_batch(parts), seeds)
  tours = m.last_solved_tours
  for i in range(3):
    alone = m.solve_batch(_sparse_tsp_batch([parts[i]]), [seeds[i]])
    _same(got[i], alone[0])
    assert np.array_equal(tours[i], m.last_solved_tours[0])


def test_dense_tsp_solve_batch_equals_each_instance_alone(weights2):
  m = G.tsp_model(weights2, sparse_factor=-1, inference_diffusion_steps=5, parallel_sampling=2)
  pts = np.stack([syn.tsp_points(64, 52, i) for i in range(3)])
  gt = np.tile(np.concatenate([np.arange(64), [0]]), (3, 1))
  batch = lambda idx: (torch.tensor(idx), torch.from_numpy(pts[idx]), torch.zeros(len(idx), 64, 64),
                       torch.from_numpy(gt[idx]).cuda())
  got = m.solve_batch(batch([0, 1, 2]), [1, 2, 3])
  for i in range(3):
    _same(got[i], m.solve_batch(batch([i]), [i + 1])[0])


def test_mis_solve_batch_equals_each_graph_alone(weights2):
  m = G.mis_model(weights2, inference_diffusion_steps=5, parallel_sampling=2, sequential_sampling=2)
  sizes = [40, 78, 130]   # even: 2m + n edges (both directions, self loops)
  graphs = _mis_graphs(sizes, 300, multiple=32)
  labels = [torch.from_numpy((syn.initial_noise(n, n) > 0).astype(np.float32)) for n in sizes]

  def batch(idx):
    ptr = syn.node_ptr([sizes[i] for i in idx])
    ei = np.concatenate([graphs[i] + ptr[j] for j, i in enumerate(idx)], 1)
    return (torch.tensor(idx), _Graph(x=torch.cat([labels[i] for i in idx]), edge_index=torch.from_numpy(ei)),
            torch.tensor([sizes[i] for i in idx]).cuda())

  got = m.solve_batch(batch([0, 1, 2]), [7, 8, 9])
  costs = m.last_solved_costs
  for i in range(3):
    _same(got[i], m.solve_batch(batch([i]), [7 + i])[0])
    assert m.last_solved_costs[0] == costs[i]


def test_solve_batch_decode_and_logs_are_test_steps(weights2):
  """On fixed heat maps (denoise_heatmap replaced) solve_batch decodes exactly as test_step, and the logged epoch
  means of one solve_batch equal those of n test_step calls."""
  parts = _tsp_parts([(50, 16), (80, 16), (30, 16)], 53)
  heats = [np.random.default_rng(i).random(p[1].shape[1]).astype(np.float32) for i, p in enumerate(parts)]
  m = G.tsp_model(weights2, sparse_factor=16, inference_diffusion_steps=3)
  m.denoise_heatmap = lambda pts, ei, xt, **kw: torch.from_numpy(
      np.concatenate([heats[i] for i in m._fixed])).cuda()
  want, tours = [], []
  for i in range(3):
    m._fixed = [i]
    want.append(m.test_step(_sparse_tsp_batch([parts[i]]), i))
    tours.append(m.last_solved_tours)
  ref_logs = m.logged_metrics(reset=True)
  m._fixed = [0, 1, 2]
  sizes, log = [], m.log
  m.log = lambda *a, **kw: (sizes.append(kw.get("batch_size")), log(*a, **kw))[1]
  got = m.solve_batch(_sparse_tsp_batch(parts), [1, 2, 3])
  assert len(sizes) == 12 and set(sizes) == {1}    # every value is one instance's, as Lightning must weight it
  for i in range(3):
    _same(got[i], want[i])
    assert np.array_equal(m.last_solved_tours[i], tours[i])
  logs = m.logged_metrics(reset=True)
  assert logs.keys() == ref_logs.keys()
  for k in logs:
    assert logs[k] == pytest.approx(ref_logs[k], rel=1e-12, abs=0), k

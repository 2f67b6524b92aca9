"""Ragged batches of independent instances in one block-diagonal call, each with its own head GroupNorm
(dfb_prepare_graph_instances; the node_ptr argument of GNNEncoder.forward, TSPModel.denoise_heatmap and
MISModel.denoise_labels).  Run with -m gpu on an H100.

The reference evaluates one instance per forward, so the fp64 oracle here always runs on each instance ALONE, and each
instance of the batched call must meet the metric rule of test_gpu_value_ranges.py against it: logits rel-Linf,
max |p - p64| <= 1e-4 and max |p / p64 - 1| where p64 >= 1e-3, each bounded by max(base, 4 x the fp32 oracle's own
error).  Instances have edge counts that are not multiples of 32 or 128, and xt = 0, xt = 1 or random, so their
GroupNorm statistics differ; the same batch with one coupled GroupNorm misses the bound by far (test 3)."""
import numpy as np
import pytest
import torch

from conftest import rel_linf
from difusco_b200 import _cabi, synthetic as syn
from oracle import difusco_oracle as orc
import gpu_util as G

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = torch.device("cuda")
TOL = 1e-4
P_BIG = 1e-3
T = 500.0
IMPLS = ["tc", "tc1", "fp32"]
AGGS = ["sum", "mean", "max"]

# (N, K) per TSP instance: 1, 49, 1 000, 4 000 and 25 000 edges
TSP_SIZES = [(1, 1), (7, 7), (50, 20), (200, 20), (500, 50)]
MIS_SIZES = [20, 57, 131, 300, 203]
XT_KINDS = ["one", "random", "zero", "one", "random"]


# ------------------------------------------------------------------------------------------------
# batches: the block-diagonal arrays, node_ptr and each instance alone (local node numbering)
# ------------------------------------------------------------------------------------------------
def _xt(kind, n, gauss, seed):
  if kind == "zero":
    return np.zeros(n, np.float32)
  if kind == "one":
    return np.ones(n, np.float32)
  z = syn.initial_noise(n, seed)
  return z if gauss else (z > 0).astype(np.float32)


def _concat(parts, sizes, pts=None):
  """parts: per instance (edge_index local, xt) -> (edge_index, xt, node_ptr, row offsets of each instance's elements)."""
  ptr = syn.node_ptr(sizes)
  ei = np.concatenate([p[0] + ptr[i] for i, p in enumerate(parts)], 1)
  xt = np.concatenate([p[1] for p in parts])
  off = np.concatenate([[0], np.cumsum([p[1].size for p in parts])])
  return ei, xt, ptr, off


def tsp_batch(sizes=TSP_SIZES, kinds=XT_KINDS, gauss=False, seed=91):
  inst = []
  for i, ((n, k), kind) in enumerate(zip(sizes, kinds)):
    p = syn.tsp_points(n, seed, i)
    ei = syn.knn_edge_index(p, k)
    inst.append((p, ei, _xt(kind, ei.shape[1], gauss, seed + 1 + i)))
  ei, xt, ptr, off = _concat([(e, x) for _, e, x in inst], [p.shape[0] for p, _, _ in inst])
  return dict(pts=np.concatenate([p for p, _, _ in inst]), ei=ei, xt=xt, ptr=ptr, off=off, inst=inst)


def mis_batch(sizes=MIS_SIZES, kinds=XT_KINDS, gauss=False, seed=93):
  inst = []
  for i, (n, kind) in enumerate(zip(sizes, kinds)):
    inst.append((None, syn.er_graph_edge_index(n, 0.1, seed, i), _xt(kind, n, gauss, seed + 1 + i)))
  ei, xt, ptr, off = _concat([(e, x) for _, e, x in inst], sizes)
  return dict(pts=None, ei=ei, xt=xt, ptr=ptr, off=off, inst=inst)


def shuffled(b, seed=5):
  """The batch with its edges in a random global order (instances interleaved); 'perm' maps new -> old position.
  The TSP state moves with the edges; the MIS state stays on the nodes."""
  perm = np.random.default_rng(seed).permutation(b["ei"].shape[1])
  out = dict(b, ei=b["ei"][:, perm], perm=perm)
  if b["pts"] is not None:    # TSP: the state lives on the edges
    out["xt"] = b["xt"][perm]
  return out


# ------------------------------------------------------------------------------------------------
# oracle on each instance alone, and the metric rule
# ------------------------------------------------------------------------------------------------
_oracles = {}


def _oracle(w, tag, task, inst, i, agg, t=T, xt=None):
  """(fp64 logits, fp32 logits) of instance i alone; cached under (tag, ...) unless xt is given."""
  pts, ei, x = inst[i]
  key = (tag, task, i, agg, t)
  if xt is None and key in _oracles:
    return _oracles[key]
  x = x if xt is None else xt
  res = []
  for dt in (torch.float64, torch.float32):
    W = orc.Weights(w, dt)
    if task == "tsp":
      res.append(orc.encoder_forward_sparse_tsp(W, pts, x, np.array([t]), ei, aggregation=agg).numpy())
    else:
      res.append(orc.encoder_forward_mis(W, x, np.array([t]), ei, aggregation=agg).numpy())
  if xt is None:
    _oracles[key] = tuple(res)
  return tuple(res)


def _softmax(x):
  return torch.softmax(torch.as_tensor(np.asarray(x, np.float64)), -1).numpy()


def _errors(out, ref):
  e = {"logits": rel_linf(out, ref)}
  if ref.shape[-1] == 2:
    p, pr = _softmax(out), _softmax(ref)
    e["p_abs"] = float(np.abs(p - pr).max())
    big = pr >= P_BIG
    e["p_rel"] = float(np.abs(p[big] / pr[big] - 1).max()) if big.any() else 0.0
  return e


def _bounds(yard, impl):
  base = {"logits": G.TOL[impl], "p_abs": TOL, "p_rel": TOL}
  return {k: max(base[k], 4 * v) for k, v in yard.items()}


def _check(out, ref64, ref32, impl, what=""):
  assert out.shape == ref64.shape and np.isfinite(out).all(), what
  got, yard = _errors(out, ref64), _errors(ref32, ref64)
  bound = _bounds(yard, impl)
  bad = [k for k in got if not got[k] <= bound[k]]
  assert not bad, f"{what} failing {bad}: kernel {got} | fp32 oracle {yard} | bounds {bound}"


def _split(b, out):
  """Per-instance slices of an output in the batch's element order (TSP: possibly shuffled edges)."""
  if "perm" in b and b["pts"] is not None:
    o = np.empty_like(out)
    o[b["perm"]] = out
    out = o
  return [out[b["off"][i]:b["off"][i + 1]] for i in range(len(b["inst"]))]


def _forward(enc, task, b, node_ptr, t=T):
  if task == "tsp":
    out = enc(G.cu(b["pts"]), torch.tensor([t]), G.cu(b["xt"]), G.cu(b["ei"]), node_ptr=node_ptr)
  else:
    out = enc(G.cu(b["xt"]), torch.tensor([t]), edge_index=G.cu(b["ei"]), node_ptr=node_ptr)
  return out.cpu().numpy()


def _encoder(w, task, impl="tc", agg="sum"):
  return G.encoder(w, w["out.2.bias"].shape[0], node_only=task == "mis", impl=impl, aggregation=agg)


# ------------------------------------------------------------------------------------------------
# 1 / 2. ragged TSP and MIS batches: every instance against the oracle on it alone
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("diffusion", ["categorical", "gaussian"])
@pytest.mark.parametrize("order", ["sorted", "shuffled"])
def test_ragged_tsp_batch_per_instance_vs_oracle(weights2, weights1, order, diffusion, agg, impl):
  gauss = diffusion == "gaussian"
  w, wkey = (weights1, "w1") if gauss else (weights2, "w2")
  b = tsp_batch(gauss=gauss)
  if order == "shuffled":
    b = shuffled(b)
  out = _forward(_encoder(w, "tsp", impl, agg), "tsp", b, b["ptr"])
  for i, o in enumerate(_split(b, out)):
    r64, r32 = _oracle(w, wkey + ("g" if gauss else ""), "tsp", b["inst"], i, agg)
    _check(o, r64, r32, impl, f"tsp instance {i} (E={o.shape[0]}) {order} {diffusion} {agg} {impl}")


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("agg", AGGS)
def test_ragged_mis_batch_per_instance_vs_oracle(weights2, agg, impl):
  b = shuffled(mis_batch())
  out = _forward(_encoder(weights2, "mis", impl, agg), "mis", b, b["ptr"])
  for i in range(len(b["inst"])):
    r64, r32 = _oracle(weights2, "w2", "mis", b["inst"], i, agg)
    _check(out[b["off"][i]:b["off"][i + 1]], r64, r32, impl, f"mis instance {i} {agg} {impl}")


# ------------------------------------------------------------------------------------------------
# 3. the per-instance oracle tells the two semantics apart
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task", ["tsp", "mis"])
def test_coupled_call_misses_the_per_instance_oracle(weights2, task):
  b = tsp_batch() if task == "tsp" else mis_batch()
  out = _forward(_encoder(weights2, task), task, b, None)
  worst = 0.0
  for i in range(len(b["inst"])):
    r64, r32 = _oracle(weights2, "w2", task, b["inst"], i, "sum")
    o = out[b["off"][i]:b["off"][i + 1]]
    got, bound = _errors(o, r64), _bounds(_errors(r32, r64), "tc")
    worst = max(worst, max(got[k] / bound[k] for k in got))
  assert worst > 10, worst


# ------------------------------------------------------------------------------------------------
# 4. bitwise: one instance is the plain call, equal node blocks of the dense graph are gn_segments = B
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task", ["tsp", "mis"])
def test_single_instance_is_bitwise_the_plain_call(weights2, task):
  b = shuffled(tsp_batch() if task == "tsp" else mis_batch())
  enc = _encoder(weights2, task)
  plain = _forward(enc, task, b, None)
  one = _forward(enc, task, b, torch.tensor([0, int(b["ptr"][-1])]))
  assert np.array_equal(plain, one)
  assert np.array_equal(plain, _forward(enc, task, b, None))


def test_dense_node_blocks_are_bitwise_gn_segments(weights2):
  V, B = 30, 3
  pts = np.concatenate([syn.tsp_points(V, 95, b) for b in range(B)]).astype(np.float32)
  ei = np.concatenate([syn.complete_edge_index(V) + b * V for b in range(B)], 1)
  xt = np.concatenate([np.zeros(V * V), np.ones(V * V), syn.initial_noise(V * V, 96) > 0]).astype(np.float32)
  enc = _encoder(weights2, "tsp")
  ctx = enc.engine()
  st = torch.cuda.current_stream().cuda_stream
  d_ei, d_pts, d_xt = G.cu(ei), G.cu(pts), G.cu(xt)
  outs = []
  for seg in ("gn_segments", "node_ptr"):
    if seg == "gn_segments":
      ctx.prepare_graph(d_ei.data_ptr(), B * V, ei.shape[1], B, st)
    else:
      ctx.prepare_graph_instances(d_ei.data_ptr(), B * V, ei.shape[1], syn.node_ptr([V] * B), st)
    ctx.set_points(d_pts.data_ptr(), st)
    out = torch.empty((ei.shape[1], 2), device=DEV)
    ctx.encoder_forward(d_xt.data_ptr(), T, out.data_ptr(), st)
    outs.append(out.cpu().numpy())
  assert np.array_equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------------
# 5. the denoise loop on ragged batches: every recorded step per instance against the oracle on its input state
# ------------------------------------------------------------------------------------------------
def _loop_case(task, w, steps):
  if task == "tsp":
    b = shuffled(tsp_batch(sizes=[(1, 1), (7, 7), (50, 20), (120, 20)], kinds=["one", "random", "zero", "random"]))
    m = G.tsp_model(w, sparse_factor=20, inference_diffusion_steps=steps)
    run = lambda: m.denoise_heatmap(G.cu(b["pts"]), G.cu(b["ei"]), G.cu(b["xt"]), seed=11, record_steps="all",
                                    node_ptr=b["ptr"])
  else:
    b = shuffled(mis_batch(sizes=[20, 57, 131, 300], kinds=["one", "random", "zero", "random"]))
    m = G.mis_model(w, inference_diffusion_steps=steps)
    run = lambda: m.denoise_labels(G.cu(b["ei"]), G.cu(b["xt"]), seed=11, record_steps="all", node_ptr=b["ptr"])
  return b, m, run


@pytest.mark.parametrize("task", ["tsp", "mis"])
def test_ragged_denoise_loop_every_step_vs_oracle(weights2, task):
  steps = 20
  torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
  b, m, run = _loop_case(task, weights2, steps)
  final, tr = run()
  tr = {k: v.cpu().numpy() for k, v in tr.items()}
  final = final.cpu().numpy()
  m.model.engine().set_graph_capture(False)
  try:
    final_plain, tr_plain = run()
  finally:
    m.model.engine().set_graph_capture(True)
  assert np.array_equal(final, final_plain.cpu().numpy())
  for k in ("xt", "p", "out"):
    assert np.array_equal(tr[k], tr_plain[k].cpu().numpy()), k
  _, Q_bar = orc.categorical_tables(1000, "linear")
  sched = orc.inference_schedule("cosine", 1000, steps)
  for s, (t1, t2) in enumerate(sched):
    xin = b["xt"] if s == 0 else tr["xt"][s - 1]
    outs, ps, xins = _split(b, tr["out"][s]), _split(b, tr["p"][s]), _split(b, xin)
    for i in range(len(b["inst"])):
      r64, r32 = _oracle(weights2, "w2", task, b["inst"], i, "sum", float(t1), xt=xins[i])
      _check(outs[i], r64, r32, "tc", f"{task} step {s} instance {i}")
      x = torch.as_tensor(xins[i])
      p64 = orc.categorical_posterior(Q_bar, t1, t2, torch.as_tensor(r64).softmax(-1), x.double())[0].numpy()
      p32 = orc.categorical_posterior(Q_bar, t1, t2, torch.as_tensor(r32).softmax(-1), x.float())[0].numpy()
      e_abs, y_abs = float(np.abs(ps[i] - p64).max()), float(np.abs(p32 - p64).max())
      big = p64 >= P_BIG
      e_rel = float(np.abs(ps[i][big] / p64[big] - 1).max()) if big.any() else 0.0
      y_rel = float(np.abs(p32[big] / p64[big] - 1).max()) if big.any() else 0.0
      assert e_abs <= max(TOL, 4 * y_abs) and e_rel <= max(TOL, 4 * y_rel), (task, s, i, e_abs, e_rel, y_abs, y_rel)


# ------------------------------------------------------------------------------------------------
# 6. re-segmenting one context: each result bitwise a fresh context's
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task", ["tsp", "mis"])
def test_resegmentation_matches_a_fresh_context(weights2, task):
  steps = 5
  b = shuffled(tsp_batch() if task == "tsp" else mis_batch())
  ptr_a = b["ptr"]
  ptr_b = ptr_a[[0, 2, 3, 5]]     # instances 0-1, 2 and 3-4 merged: still closed under the edges
  model = G.tsp_model if task == "tsp" else G.mis_model
  kw = dict(sparse_factor=20) if task == "tsp" else {}

  def run(m, ptr):
    if task == "tsp":
      fwd = _forward(m.model, task, b, ptr)
      x = m.denoise_heatmap(G.cu(b["pts"]), G.cu(b["ei"]), G.cu(b["xt"]), steps=steps, seed=3, node_ptr=ptr)
    else:
      fwd = _forward(m.model, task, b, ptr)
      x = m.denoise_labels(G.cu(b["ei"]), G.cu(b["xt"]), steps=steps, seed=3, node_ptr=ptr)
    return fwd, x.cpu().numpy()

  shared = model(weights2, **kw)
  got = [run(shared, ptr_a), run(shared, ptr_b), run(shared, ptr_a)]
  fresh_a, fresh_b = run(model(weights2, **kw), ptr_a), run(model(weights2, **kw), ptr_b)
  for g, f in zip(got, (fresh_a, fresh_b, fresh_a)):
    assert np.array_equal(g[0], f[0]) and np.array_equal(g[1], f[1])
  assert not np.array_equal(fresh_a[0], fresh_b[0])


# ------------------------------------------------------------------------------------------------
# 7. size limits
# ------------------------------------------------------------------------------------------------
def test_4096_instances_in_one_call(weights2):
  n_inst = 4096
  sizes = [int(s) for s in np.random.default_rng(97).integers(3, 13, n_inst)]
  kinds = [("zero", "one", "random")[i % 3] for i in range(n_inst)]
  b = mis_batch(sizes=sizes, kinds=kinds, seed=98)
  out = _forward(_encoder(weights2, "mis"), "mis", b, torch.from_numpy(b["ptr"]))
  assert np.isfinite(out).all()
  for i in (0, 1, 2, 1000, 2047, 3001, 4094, 4095):
    r64, r32 = _oracle(weights2, "w2_4096", "mis", b["inst"], i, "sum")
    _check(out[b["off"][i]:b["off"][i + 1]], r64, r32, "tc", f"instance {i}")


def test_single_row_instance_next_to_one_over_65536_rows(weights2):
  b = tsp_batch(sizes=[(1, 1), (1400, 50)], kinds=["one", "random"], seed=99)
  assert b["off"][2] - b["off"][1] > 65536
  out = _forward(_encoder(weights2, "tsp"), "tsp", b, b["ptr"])
  for i, o in enumerate(_split(b, out)):
    r64, r32 = _oracle(weights2, "w2_big", "tsp", b["inst"], i, "sum")
    _check(o, r64, r32, "tc", f"instance {i} (E={o.shape[0]})")


# ------------------------------------------------------------------------------------------------
# 8. invalid arguments: DFB_E_INVALID, and the previously prepared graph still gives its result bitwise
# ------------------------------------------------------------------------------------------------
def test_invalid_arguments_keep_the_prepared_graph(weights2):
  b = tsp_batch()
  enc = _encoder(weights2, "tsp")
  ref = _forward(enc, "tsp", b, b["ptr"])
  ctx = enc.engine()
  st = torch.cuda.current_stream().cuda_stream
  V, E = int(b["ptr"][-1]), b["ei"].shape[1]
  ptr = b["ptr"]
  # instance 2 without its edges: its nodes have none
  keep = np.ones(E, bool)
  keep[b["off"][2]:b["off"][3]] = False
  no_edges = np.ascontiguousarray(b["ei"][:, keep])
  split = np.sort(np.concatenate([ptr, [ptr[2] + 3]]))    # cuts instance 2 in two: its k-NN edges cross the cut
  d_ei, d_no = G.cu(b["ei"]), G.cu(no_edges)
  cases = [("no instances", d_ei, E, ptr[:1]), ("first offset not 0", d_ei, E, ptr + 1),
           ("last offset not num_nodes", d_ei, E, np.concatenate([ptr[:-1], [V - 1]])),
           ("not strictly increasing", d_ei, E, np.concatenate([ptr[:2], ptr[1:]])),
           ("decreasing", d_ei, E, ptr[[0, 2, 1, 3, 4, 5]]),
           ("edge across instances", d_ei, E, split), ("instance without edges", d_no, no_edges.shape[1], ptr)]
  for what, ei, e, p in cases:
    p = np.ascontiguousarray(p, np.int64)
    rc = _cabi.lib().dfb_prepare_graph_instances(ctx._h, ei.data_ptr(), V, e, p.size - 1,
                                                 p.ctypes.data_as(_cabi.C.POINTER(_cabi.C.c_int64)), st)
    assert rc == _cabi.DFB_E_INVALID, (what, rc)
    out = torch.empty((E, 2), device=DEV)
    ctx.encoder_forward(G.cu(b["xt"]).data_ptr(), T, out.data_ptr(), st)
    assert np.array_equal(out.cpu().numpy(), ref), what
  with pytest.raises(ValueError):
    ctx.prepare_graph_instances(d_ei.data_ptr(), V, E, split, st)

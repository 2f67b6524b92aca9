"""A timestep per element on the H100: dfb_encoder_forward_timesteps and GNNEncoder.forward with the reference's
training-step timesteps (one t per graph, per node or per dense sample, or any t per edge).

  1. Golden parity: every case of tests/golden/fwd_tsteps.npz (the reference's own training steps) within G.TOL[impl],
     and the CE / MSE loss of our output against the loss the reference returned.
  2. The per-row variant is the product path: t_index all zeros is bitwise dfb_encoder_forward at t_values[0].
  3. Per instance: with node_ptr, each instance at its own t matches its own single-t forward alone.
  4. At size against the fp64 oracle: TSP-200 k = 20 x 4 graphs, MIS ER-200 x 3.
  5. Dense in one call, argument errors, and an out-of-range index."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import golden, rel_linf
from difusco_b200 import _cabi, synthetic as syn
from oracle import difusco_oracle as orc
import gpu_util as G

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = torch.device("cuda")
IMPLS = ["fp32", "tc", "tc1"]
P_BIG = 1e-3


def _stream():
  return torch.cuda.current_stream().cuda_stream


def _enc(w, task, impl, ckpt=False):
  enc = G.encoder(w, w["out.2.bias"].shape[0], node_only=task == "mis", sparse=task != "dense", impl=impl)
  enc.use_activation_checkpoint = ckpt
  return enc


def _loss(name, out, g):
  out = torch.as_tensor(np.asarray(out, np.float32))
  if name in ("tsp_cat", "tsp_ckpt", "mis_cat"):
    return float(F.cross_entropy(out, torch.from_numpy(g[f"{name}/labels"])))
  return float(F.mse_loss(out.squeeze(1), torch.from_numpy(g[f"{name}/eps"])))


def _golden_forward(name, g, impl, weights1, weights2):
  w = weights1 if "gauss" in name else weights2
  a = lambda k: G.cu(g[f"{name}/{k}"])
  if name.startswith("tsp"):
    enc = _enc(w, "tsp", impl, ckpt=name == "tsp_ckpt")
    return enc(a("points"), a("t"), a("xt"), a("edge_index")).cpu().numpy()   # edge_index float, as in training
  if name == "dense_gauss":
    return _enc(w, "dense", impl)(a("points"), a("t"), a("xt")).cpu().numpy()
  return _enc(w, "mis", impl)(a("xt"), a("t"), edge_index=a("edge_index")).cpu().numpy()


# ------------------------------------------------------------------------------------------------
# 1. golden parity
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("name", ["tsp_cat", "tsp_ckpt", "dense_gauss", "mis_cat", "mis_gauss", "tsp_edge_t"])
def test_golden_training_step_forwards(name, impl, weights1, weights2):
  g = golden("fwd_tsteps")
  out = _golden_forward(name, g, impl, weights1, weights2)
  ref = g[f"{name}/out"]
  assert out.shape == ref.shape and np.isfinite(out).all()
  err = rel_linf(out, ref)
  assert err < G.TOL[impl], f"{name} {impl}: rel L-inf {err:.3g}"
  if f"{name}/loss" in g.files:
    rel = abs(_loss(name, out, g) / float(g[f"{name}/loss"]) - 1)
    assert rel < 1e-5, f"{name} {impl}: loss off by {rel:.3g} relative"


# ------------------------------------------------------------------------------------------------
# 2. the per-row variant against the product path, bitwise
# ------------------------------------------------------------------------------------------------
def _prepared(enc, task, seed=3):
  """A TSP (3 graphs of 50 nodes, k = 20, unsorted edges) or MIS (ER-150) graph prepared on enc's context ->
  (ctx, device xt, N)."""
  rng = np.random.default_rng(seed)
  if task == "tsp":
    pts, ei = syn.tsp_sparse_batch(50, 20, 3, seed=seed)
    ei = ei[:, rng.permutation(ei.shape[1])]
    enc.set_graph(G.cu(ei), pts.shape[0])
    enc.set_points(G.cu(pts))
    n = ei.shape[1]
  else:
    ei = syn.er_graph_edge_index(150, 0.05, seed=seed)
    enc.set_graph(G.cu(ei), 150)
    n = 150
  return enc.engine(), G.cu(syn.initial_noise(n, seed)), n


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("task", ["tsp", "mis"])
def test_zero_index_is_bitwise_the_product_call(weights2, task, impl):
  enc = _enc(weights2, task, impl)
  ctx, xt, n = _prepared(enc, task)
  st = _stream()
  ref = torch.empty((n, 2), device=DEV)
  ctx.encoder_forward(xt.data_ptr(), 412.0, ref.data_ptr(), st)
  zeros = torch.zeros(n, dtype=torch.int32, device=DEV)
  for values in ([412.0], [412.0, 7.0, 999.0]):
    out = torch.full((n, 2), float("nan"), device=DEV)
    ctx.encoder_forward_timesteps(xt.data_ptr(), values, zeros.data_ptr(), out.data_ptr(), st)
    assert torch.equal(out, ref), (values, impl)
  out = torch.empty((n, 2), device=DEV)
  ctx.encoder_forward_timesteps(xt.data_ptr(), [412.0], None, out.data_ptr(), st)
  assert torch.equal(out, ref)


@pytest.mark.parametrize("task", ["tsp", "mis", "dense"])
def test_equal_per_element_t_is_bitwise_the_scalar_call(weights2, task):
  enc = _enc(weights2, task, "tc")
  if task == "tsp":
    pts, ei = syn.tsp_sparse_batch(50, 20, 2, seed=4)
    args = lambda t: (G.cu(pts), t, G.cu(syn.initial_noise(ei.shape[1], 4)), G.cu(ei))
    n = ei.shape[1]
  elif task == "mis":
    ei = syn.er_graph_edge_index(150, 0.05, seed=4)
    args = lambda t: (G.cu(syn.initial_noise(150, 4)), t, None, G.cu(ei))
    n = 150
  else:
    pts = np.stack([syn.tsp_points(20, 4, b) for b in range(3)])
    args = lambda t: (G.cu(pts), t, G.cu((syn.initial_noise(3 * 400, 4) > 0).astype(np.float32).reshape(3, 20, 20)))
    n = 3
  scalar = enc(*args(torch.tensor([300.0], device=DEV))).cpu()
  assert torch.equal(enc(*args(torch.full((n,), 300.0, device=DEV))).cpu(), scalar)


# ------------------------------------------------------------------------------------------------
# 3. per-instance timesteps against each instance alone
# ------------------------------------------------------------------------------------------------
def _tsp_instances(sizes, seed):
  parts = [(syn.tsp_points(n, seed, i), syn.knn_edge_index(syn.tsp_points(n, seed, i), k)) for i, (n, k) in enumerate(sizes)]
  pts = np.concatenate([p for p, _ in parts]).astype(np.float32)
  off = syn.node_ptr([n for n, _ in sizes])
  ei = np.concatenate([e + off[i] for i, (_, e) in enumerate(parts)], 1)
  return parts, pts, ei, off


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("aligned", [True, False])
def test_tsp_instances_at_their_own_t_match_each_alone(weights2, impl, aligned):
  # aligned: every instance's edge count is a multiple of 32, so no 32-edge message group straddles two instances
  sizes = [(40, 8), (64, 10), (16, 6)] if aligned else [(37, 7), (61, 9), (13, 5)]
  ts = [1.0, 1000.0, 431.0]
  parts, pts, ei, off = _tsp_instances(sizes, 71)
  E = [n * k for n, k in sizes]
  xt = syn.initial_noise(sum(E), 72)
  enc = _enc(weights2, "tsp", impl)
  t_edge = torch.from_numpy(np.repeat(ts, E).astype(np.float32)).to(DEV)
  out = enc(G.cu(pts), t_edge, G.cu(xt), G.cu(ei), node_ptr=torch.from_numpy(off)).cpu().numpy()
  e0 = 0
  for i, ((p, e), t) in enumerate(zip(parts, ts)):
    alone = enc(G.cu(p), torch.tensor([t]), G.cu(xt[e0:e0 + E[i]]), G.cu(e)).cpu().numpy()
    got = out[e0:e0 + E[i]]
    if aligned:
      assert np.array_equal(got, alone), f"instance {i}: {rel_linf(got, alone):.3g}"
    else:
      assert rel_linf(got, alone) < G.TOL[impl], f"instance {i}: {rel_linf(got, alone):.3g}"
    e0 += E[i]


@pytest.mark.parametrize("impl", IMPLS)
def test_mis_instances_at_their_own_t_match_each_alone(weights2, impl):
  sizes, ts = [60, 45, 90], [5.0, 640.0, 1000.0]
  eis = [syn.er_graph_edge_index(n, 0.1, seed=80, instance=i) for i, n in enumerate(sizes)]
  off = syn.node_ptr(sizes)
  ei = np.concatenate([e + off[i] for i, e in enumerate(eis)], 1)
  xt = syn.initial_noise(int(off[-1]), 81)
  enc = _enc(weights2, "mis", impl)
  t_node = G.cu(np.repeat(ts, sizes).astype(np.float32))
  out = enc(G.cu(xt), t_node, edge_index=G.cu(ei), node_ptr=torch.from_numpy(off)).cpu().numpy()
  for i, t in enumerate(ts):
    alone = enc(G.cu(xt[off[i]:off[i + 1]]), torch.tensor([t]), edge_index=G.cu(eis[i])).cpu().numpy()
    assert rel_linf(out[off[i]:off[i + 1]], alone) < G.TOL[impl]


# ------------------------------------------------------------------------------------------------
# 4. at size against the fp64 oracle (metrics of test_gpu_instance_batch.py: logits, and probabilities of
#    categorical heads; bound max(base, 4 x the fp32 oracle's error))
# ------------------------------------------------------------------------------------------------
def _errors(out, ref):
  e = {"logits": rel_linf(out, ref)}
  p = torch.softmax(torch.as_tensor(np.asarray(out, np.float64)), -1).numpy()
  pr = torch.softmax(torch.as_tensor(np.asarray(ref, np.float64)), -1).numpy()
  e["p_abs"] = float(np.abs(p - pr).max())
  big = pr >= P_BIG
  e["p_rel"] = float(np.abs(p[big] / pr[big] - 1).max())
  return e


_oracle_cache = {}


def _check_vs_oracle(out, key, fwd, impl):
  if key not in _oracle_cache:
    _oracle_cache[key] = fwd(torch.float64).numpy(), fwd(torch.float32).numpy()
  ref64, ref32 = _oracle_cache[key]
  assert out.shape == ref64.shape and np.isfinite(out).all()
  got, yard = _errors(out, ref64), _errors(ref32, ref64)
  bound = {k: max(G.TOL[impl] if k == "logits" else 1e-4, 4 * v) for k, v in yard.items()}
  bad = [k for k in got if not got[k] <= bound[k]]
  assert not bad, f"failing {bad}: kernel {got} | fp32 oracle {yard} | bounds {bound}"


@pytest.mark.parametrize("impl", IMPLS)
def test_tsp200_per_graph_t_vs_fp64_oracle(weights2, impl):
  pts, ei = syn.tsp_sparse_batch(200, 20, 4, seed=90)
  t = np.repeat([1.0, 250.0, 777.0, 1000.0], 200 * 20).astype(np.float32)
  xt = syn.initial_noise(ei.shape[1], 91) * np.float32(1.02)
  out = _enc(weights2, "tsp", impl)(G.cu(pts), G.cu(t), G.cu(xt), G.cu(ei)).cpu().numpy()
  _check_vs_oracle(out, "tsp200", lambda dt: orc.encoder_forward_sparse_tsp(orc.Weights(weights2, dt), pts, xt, t, ei), impl)


@pytest.mark.parametrize("impl", IMPLS)
def test_mis_er200_per_node_t_vs_fp64_oracle(weights2, impl):
  ei, sizes = syn.mis_batch(200, 200, 0.05, 3, seed=92)
  t = np.random.default_rng(93).integers(1, 1001, sum(sizes)).astype(np.float32)   # any t per node
  xt = syn.initial_noise(sum(sizes), 94)
  out = _enc(weights2, "mis", impl)(G.cu(xt), G.cu(t), edge_index=G.cu(ei)).cpu().numpy()
  _check_vs_oracle(out, "mis200", lambda dt: orc.encoder_forward_mis(orc.Weights(weights2, dt), xt, t, ei), impl)


# ------------------------------------------------------------------------------------------------
# 5. dense in one call, argument errors, out-of-range index
# ------------------------------------------------------------------------------------------------
def test_dense_per_sample_t_is_one_call(weights2):
  enc = _enc(weights2, "dense", "tc")
  B, V = 8, 20
  pts = G.cu(np.stack([syn.tsp_points(V, 5, b) for b in range(B)]))
  xt = G.cu((syn.initial_noise(B * V * V, 5) > 0).astype(np.float32).reshape(B, V, V))
  enc(pts, torch.tensor([10.0]), xt)   # prepares the graph and points
  ctx = enc.engine()
  deltas = []
  for t in (torch.tensor([500.0]), torch.arange(1, B + 1, dtype=torch.float32) * 100):
    n0 = ctx.launch_count()
    enc(pts, t, xt)
    deltas.append(ctx.launch_count() - n0)
  assert deltas[0] == deltas[1], deltas


@pytest.mark.parametrize("impl", IMPLS)
def test_dense_fixture_with_two_timesteps(weights2, impl):
  g = golden("fwd_dense_cat")
  out = _enc(weights2, "dense", impl)(G.cu(g["points"]), G.cu(g["t"]), G.cu(g["xt"])).cpu().numpy()
  assert rel_linf(out, g["out"]) < G.TOL[impl]


def test_argument_errors_before_device_work(weights2):
  enc = _enc(weights2, "tsp", "tc")
  ctx, xt, n = _prepared(enc, "tsp")
  L = _cabi.lib()
  out = torch.full((n, 2), 7.0, device=DEV)
  idx = torch.zeros(n, dtype=torch.int32, device=DEV)
  host_idx = np.zeros(n, np.int32)
  vals = np.array([5.0], np.float32)
  fp = vals.ctypes.data_as(_cabi.C.POINTER(_cabi.C.c_float))
  big = np.ones(4097, np.float32)
  torch.cuda.synchronize()
  n0 = ctx.launch_count()
  cases = [(1, None, idx.data_ptr(), _cabi.DFB_E_INVALID), (0, fp, idx.data_ptr(), _cabi.DFB_E_INVALID),
           (-3, fp, idx.data_ptr(), _cabi.DFB_E_INVALID), (1, fp, host_idx.ctypes.data, _cabi.DFB_E_INVALID),
           (4097, big.ctypes.data_as(_cabi.C.POINTER(_cabi.C.c_float)), idx.data_ptr(), _cabi.DFB_E_UNSUPPORTED)]
  for n_t, tv, ti, code in cases:
    assert L.dfb_encoder_forward_timesteps(ctx._h, xt.data_ptr(), n_t, tv, ti, out.data_ptr(), _stream()) == code
  assert ctx.launch_count() == n0
  torch.cuda.synchronize()
  assert bool((out == 7.0).all())
  with pytest.raises(NotImplementedError):
    ctx.encoder_forward_timesteps(xt.data_ptr(), big, idx.data_ptr(), out.data_ptr(), _stream())
  # wrong lengths through the module
  pts, ei = syn.tsp_sparse_batch(20, 5, 1, seed=1)
  with pytest.raises(ValueError, match="timesteps"):
    enc(G.cu(pts), torch.ones(7, device=DEV), G.cu(np.zeros(100, np.float32)), G.cu(ei))


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("task", ["tsp", "mis"])
def test_out_of_range_index_gives_nan_and_the_context_stays_usable(weights2, task, impl):
  # the NaN time row makes the head GroupNorm statistics NaN; the head's ReLU (fmaxf) maps NaN to 0, so every output
  # row of the call becomes the 1x1 conv's bias
  enc = _enc(weights2, task, impl)
  ctx, xt, n = _prepared(enc, task)
  st = _stream()
  ref = torch.empty((n, 2), device=DEV)
  ctx.encoder_forward(xt.data_ptr(), 50.0, ref.data_ptr(), st)
  for bad in (2, -1):
    idx = torch.zeros(n, dtype=torch.int32, device=DEV)
    idx[n // 2] = bad
    out = torch.empty((n, 2), device=DEV)
    ctx.encoder_forward_timesteps(xt.data_ptr(), [50.0, 60.0], idx.data_ptr(), out.data_ptr(), st)
    torch.cuda.synchronize()   # raises if the call faulted
    bias = torch.from_numpy(weights2["out.2.bias"]).to(DEV).expand(n, 2)
    assert torch.equal(out, bias) and not torch.equal(ref, bias), bad
  out = torch.empty((n, 2), device=DEV)
  ctx.encoder_forward_timesteps(xt.data_ptr(), [50.0, 60.0], torch.zeros(n, dtype=torch.int32, device=DEV).data_ptr(),
                                out.data_ptr(), st)
  assert torch.equal(out, ref)



@pytest.mark.parametrize("task", ["tsp", "mis"])
def test_host_per_element_timesteps_raise_and_device_ones_run(weights2, task):
  """The sparse forwards read different per-element timesteps on the model's device, as the training steps pass them;
  a host tensor of them keeps raising NotImplementedError, and one host value or n equal host values keep working."""
  enc = _enc(weights2, task, "tc")
  if task == "tsp":
    pts, ei = syn.tsp_sparse_batch(20, 5, 2, seed=6)
    n = ei.shape[1]
    run = lambda t: enc(G.cu(pts), t, G.cu(syn.initial_noise(n, 6)), G.cu(ei))
  else:
    ei = syn.er_graph_edge_index(40, 0.1, seed=6)
    n = 40
    run = lambda t: enc(G.cu(syn.initial_noise(n, 6)), t, edge_index=G.cu(ei))
  t = torch.arange(1, n + 1, dtype=torch.float32)
  with pytest.raises(NotImplementedError, match="device"):
    run(t)
  out = run(t.to(DEV))
  assert out.shape == (n, 2) and bool(torch.isfinite(out).all())
  assert torch.equal(run(torch.full((n,), 300.0)), run(torch.tensor([300.0])))

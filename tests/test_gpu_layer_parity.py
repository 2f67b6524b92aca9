"""Each GNN layer in isolation against the fp64 oracle, and encoders of 1 to 64 layers.

Everything else in the suite compares the encoder after its head (GroupNorm over all rows, ReLU, a 256 -> 2
projection) at 12 layers, so a fault in one layer's epilogue has to survive up to eleven more layers and the head
before a test sees it.  Here dfb_debug_gnn_layer runs one layer of the product code (run_layer: node linears, fused
edge layer, node update) on a state the test sets, and oracle.layer_step runs the same layer in fp64.

  a. Teacher-forced layers: the fp64 oracle's state entering each of the 12 layers, rounded to fp32, through the hook
     on sparse TSP (sorted and shuffled), an unsorted MIS ER graph, the complete graph of dense TSP-50, the irregular
     graphs of gpu_util (hub, isolated nodes, segment ends at tile boundaries, 1 to 129 edges, duplicates) and
     V = 1, 127, 128, 129 node-linear row tiles; tc, tc1, fp32 and sum / mean / max.
  b. One layer at value edges: offset e rows, near-constant e_hat rows (variance around LN_EPS), saturated sigmoids,
     all-negative messages under max, mean over degree-1 nodes, nodes without edges.
  c. Depth: the public forward at L = 1, 2, 5, 64; the captured loop against plain launches and dfb_denoise_step at
     L = 1, 2; one context reloaded across depths; n_layers outside [1, 64] rejected.

Metric of a and b, for each of h_out and e_out: the largest per-row relative L-inf error, max_r |d_r|_inf / |ref_r|_inf,
so one wrong row cannot hide under the global maximum.  Bound: max(BASE[impl], 4 x the fp32 oracle's error on the same
fp32 input), the rule of test_gpu_value_ranges.py.  DESIGN section 2 records the measured margins."""
import numpy as np
import pytest
import torch

from conftest import rel_linf
from difusco_b200 import _cabi, synthetic as syn
from difusco_b200.models.gnn_encoder import GNNEncoder, reference_frequency_tables
from oracle import difusco_oracle as orc
import gpu_util as G

torch.set_grad_enabled(False)

IMPLS = ["tc", "tc1", "fp32"]
AGGS = ["sum", "mean", "max"]
BASE = {"tc": 1.8e-5, "tc1": 1.8e-5, "fp32": 1.8e-6}   # <= 2 x the largest error measured on an H100 (DESIGN section 2)
T_LAYER = 700.0
N_LAYERS = 12


def _stream():
  return torch.cuda.current_stream().cuda_stream


def row_rel(out, ref):
  """max over rows r of |out_r - ref_r|_inf / |ref_r|_inf."""
  out, ref = np.asarray(out, np.float64), np.asarray(ref, np.float64)
  return float((np.abs(out - ref).max(1) / np.maximum(np.abs(ref).max(1), 1e-30)).max())


def _assert_within(got, yard, impl, what):
  bound = {k: max(BASE[impl], 4 * v) for k, v in yard.items()}
  bad = [k for k in got if not got[k] <= bound[k]]
  assert not bad, f"{what} failing {bad}: kernel {got} | fp32 oracle {yard} | bounds {bound}"


# ------------------------------------------------------------------------------------------------
# cases: name -> (task, V, edge_index, points (V,2), edge xt (E,), node xt (V,)); edge_index in the caller's order
# ------------------------------------------------------------------------------------------------
def _small_v(V):
  rng = np.random.default_rng(900 + V)
  return G.graph_from_degrees(rng.integers(1, 5, V), rng)


_GRAPHS = {
    "tsp": lambda: syn.tsp_sparse_batch(50, 20, 2, seed=61)[1],
    "mis": lambda: syn.er_graph_edge_index(150, 0.05, seed=62),
    "dense50": lambda: syn.complete_edge_index(50),
    "hub": lambda: G.hub_graph()[1],
    "isolated": lambda: G.isolated_graph()[1],
    "degseq": lambda: G.degseq_graph()[1],
    "dup": lambda: G.dup_graph()[1],
    "deg1": lambda: np.stack([np.arange(300), np.random.default_rng(63).integers(0, 300, 300)]).astype(np.int64),
}
_GRAPHS.update({f"tiny{E}": (lambda E=E: G.tiny_graph(E)[1]) for E in G.TINY})
_GRAPHS.update({f"V{V}": (lambda V=V: _small_v(V)[1]) for V in (1, 127, 128, 129)})
_NODES = {"tsp": 100, "mis": 150, "dense50": 50, "hub": 1201, "isolated": 240, "degseq": len(G.DEGREES), "dup": 150,
          "deg1": 300, **{f"tiny{E}": V for E, V in G.TINY.items()}, **{f"V{V}": V for V in (1, 127, 128, 129)}}

_case_cache = {}


def _case(name):
  """name = graph[_shuf]: the graph's edges, in a seeded random order with _shuf; points and binary xt."""
  if name not in _case_cache:
    shuf = name.endswith("_shuf")
    graph = name[:-5] if shuf else name
    ei = _GRAPHS[graph]()
    V = _NODES[graph]
    assert ei.max() < V
    seed = sum(map(ord, name))
    if shuf:
      ei = ei[:, np.random.default_rng(seed).permutation(ei.shape[1])]
    rng = np.random.default_rng(seed + 1)
    pts = rng.random((V, 2), dtype=np.float32)
    xe = (rng.random(ei.shape[1]) < 0.3).astype(np.float32)
    xv = (rng.random(V) < 0.5).astype(np.float32)
    _case_cache[name] = (V, np.ascontiguousarray(ei), pts, xe, xv)
  return _case_cache[name]


def _initial_state(W, task, case):
  """(h0, e0) entering layer 0 (gnn_encoder.py:394-395 for TSP, :405-407 for MIS) and the time embedding."""
  V, ei, pts, xe, xv = _case(case)
  if task == "tsp":
    h = W.lin("node_embed", orc.pos_embed_2d(torch.as_tensor(pts).to(W.dtype), W.hidden))
    e = W.lin("edge_embed", orc.scalar_embed(torch.as_tensor(xe).to(W.dtype), W.hidden))
  else:
    h = W.lin("node_embed", orc.scalar_embed(torch.as_tensor(xv).to(W.dtype), W.hidden))
    e = torch.zeros((ei.shape[1], W.hidden), dtype=W.dtype)
  return h, e, orc._time_emb(W, torch.tensor([T_LAYER], dtype=torch.float32))


# ------------------------------------------------------------------------------------------------
# the hook
# ------------------------------------------------------------------------------------------------
_engines = {}


def _engine(weights, task, n_layers=N_LAYERS):
  """One context per (weights, task, depth), loaded through GNNEncoder's own weight path."""
  key = (id(weights), task, n_layers)
  if key not in _engines:
    enc = G.load(GNNEncoder(n_layers, 256, weights["out.2.bias"].shape[0], sparse=True,
                            node_feature_only=task == "mis"), weights)
    _engines[key] = (enc, weights)
  return _engines[key][0].engine()


def _run_layer(ctx, ei, V, layer, h, e, impl, agg, t=T_LAYER, t_index=None):
  """dfb_debug_gnn_layer on fp32 h (V,256) and e (E,256) in the caller's edge order -> (h_out, e_out), same order.
  With t_index (int32, one per edge for TSP or per node for MIS, caller's order), dfb_debug_gnn_layer_timesteps with
  t the sequence of distinct timesteps."""
  ctx.set_edge_impl(G.IMPLS[impl])
  ctx.set_aggregation(agg)
  eid = G.cu(ei)
  ctx.prepare_graph(eid.data_ptr(), V, ei.shape[1], 1, _stream())
  perm = np.argsort(ei[0], kind="stable")
  hd, ed = G.cu(np.asarray(h, np.float32)), G.cu(np.asarray(e, np.float32)[perm])
  if t_index is None:
    ctx.debug_gnn_layer(layer, t, hd.data_ptr(), ed.data_ptr(), _stream())
  else:
    idx = G.cu(np.asarray(t_index, np.int32))
    ctx.debug_gnn_layer_timesteps(layer, t, idx.data_ptr(), hd.data_ptr(), ed.data_ptr(), _stream())
  torch.cuda.synchronize()
  e_out = np.empty_like(ed.cpu().numpy())
  e_out[perm] = ed.cpu().numpy()
  return hd.cpu().numpy(), e_out


def _check_layer(got_h, got_e, h_in, e_in, r64, r32, task, layer, n_layers, impl, what):
  """h and e against the fp64 layer within the bound; the output the product does not compute stays bitwise unchanged:
  h after the last TSP layer, e after the last MIS layer."""
  last = layer == n_layers - 1
  assert np.isfinite(got_h).all() and np.isfinite(got_e).all(), what
  got, yard = {}, {}
  if task == "tsp" and last:
    assert np.array_equal(got_h, h_in), f"{what}: h changed after the last TSP layer"
  else:
    got["h"], yard["h"] = row_rel(got_h, r64[0]), row_rel(r32[0], r64[0])
  if task == "mis" and last:
    assert np.array_equal(got_e, e_in), f"{what}: e changed after the last MIS layer"
  else:
    got["e"], yard["e"] = row_rel(got_e, r64[1]), row_rel(r32[1], r64[1])
  _assert_within(got, yard, impl, what)


def _refs(weights, task, case, layer, h, e, agg, t=(T_LAYER,)):
  """(fp64, fp32) oracle layer `layer` on the fp32 state (h, e), caller's edge order, as numpy; t one timestep, or
  one per edge (TSP) or node (MIS) in the caller's order."""
  V, ei, *_ = _case(case)
  row, col = torch.as_tensor(ei[0]), torch.as_tensor(ei[1])
  out = []
  for dt in (torch.float64, torch.float32):
    W = _weights(weights, dt)
    temb = orc._time_emb(W, torch.as_tensor(np.asarray(t, np.float32)))
    hh, ee = orc.layer_step(W, layer, torch.as_tensor(h).to(dt), torch.as_tensor(e).to(dt), row, col, temb,
                            task == "tsp", agg)
    out.append((hh.numpy(), ee.numpy()))
  return out


_wcache = {}


def _weights(weights, dtype):
  """orc.Weights of a state dict, cached; the entry holds the dict, so its id is not reused while cached."""
  key = (id(weights), dtype)
  if key not in _wcache:
    _wcache[key] = (weights, orc.Weights(weights, dtype=dtype))
  return _wcache[key][1]


# ------------------------------------------------------------------------------------------------
# a. teacher-forced layers
# ------------------------------------------------------------------------------------------------
IRREGULAR = ["hub", "isolated", "degseq", "dup"] + [f"tiny{E}" for E in G.TINY]
TF_CASES = ([("tsp", "tsp"), ("tsp_shuf", "tsp"), ("mis", "mis"), ("dense50", "tsp")] +
            [(c, t) for c in IRREGULAR for t in ("tsp", "mis")] + [(f"V{V}", "mis") for V in (1, 127, 128, 129)])

_tf_cache = {}


def _teacher_forced(weights, case, task, agg, t=(T_LAYER,), t_key=None):
  """Per layer l: the fp64 forward's state entering l rounded to fp32, and the fp64 / fp32 oracle layer l on it; t as
  _refs, t_key names it.  Only the latest (case, task, agg, t_key) is kept: the parameters run in that order."""
  key = (case, task, agg, t_key)
  if key not in _tf_cache:
    _tf_cache.clear()
    V, ei, *_ = _case(case)
    W = _weights(weights, torch.float64)
    h, e, _ = _initial_state(W, task, case)
    temb = orc._time_emb(W, torch.as_tensor(np.asarray(t, np.float32)))
    taps = []
    orc._sparse_encoding(W, h, e, torch.as_tensor(ei[0]), torch.as_tensor(ei[1]), temb, task == "tsp", agg, taps)
    states = [(h, e)] + taps[:-1]
    layers = []
    for l, (hs, es) in enumerate(states):
      h32, e32 = hs.numpy().astype(np.float32), es.numpy().astype(np.float32)
      layers.append((h32, e32) + tuple(_refs(weights, task, case, l, h32, e32, agg, t)))
    _tf_cache[key] = layers
  return _tf_cache[key]


@pytest.mark.gpu
@pytest.mark.parametrize("case,task,agg,impl", [(c, t, a, i) for c, t in TF_CASES for a in AGGS for i in IMPLS])
def test_teacher_forced_layer_vs_fp64_oracle(weights2, case, task, agg, impl):
  V, ei, *_ = _case(case)
  ctx = _engine(weights2, task)
  for l, (h32, e32, r64, r32) in enumerate(_teacher_forced(weights2, case, task, agg)):
    got_h, got_e = _run_layer(ctx, ei, V, l, h32, e32, impl, agg)
    _check_layer(got_h, got_e, h32, e32, r64, r32, task, l, N_LAYERS, impl, f"{case} {task} {agg} {impl} layer {l}")


@pytest.mark.gpu
def test_hook_rejects_bad_layer_and_host_pointers(weights2):
  V, ei, *_ = _case("tiny33")
  ctx = _engine(weights2, "tsp")
  eid = G.cu(ei)
  ctx.prepare_graph(eid.data_ptr(), V, ei.shape[1], 1, _stream())
  h, e = torch.zeros((V, 256), device="cuda"), torch.zeros((ei.shape[1], 256), device="cuda")
  for layer in (-1, N_LAYERS):
    with pytest.raises(ValueError):
      ctx.debug_gnn_layer(layer, T_LAYER, h.data_ptr(), e.data_ptr(), _stream())
  hh = np.zeros((V, 256), np.float32)
  with pytest.raises(ValueError):
    ctx.debug_gnn_layer(0, T_LAYER, hh.ctypes.data, e.data_ptr(), _stream())


# ------------------------------------------------------------------------------------------------
# b. one layer at value edges, set by the test
# ------------------------------------------------------------------------------------------------
MID = 5


def _edge_case(name):
  """-> (weights, task, case, agg, h (V,256), e (E,256)) for edge case `name`."""
  w = {k: v.copy() for k, v in syn.make_encoder_weights(5, out_channels=2).items()}
  rng = np.random.default_rng(sum(map(ord, name)))
  p = f"layers.{MID}."
  task, case, agg = "tsp", "tsp", "sum"
  if name.startswith("flat"):                    # e_hat rows nearly constant: per-row variance ~ var around mean 3
    var = {"flat1e-4": 1e-4, "flat1e-5": 1e-5, "flat1e-6": 1e-6}[name]
    for n in "ABC":
      w[p + n + ".weight"] *= np.float32(1e-4)
      w[p + n + ".bias"][:] = 0
    w[p + "A.bias"][:] = (3.0 + np.sqrt(var) * rng.standard_normal(256)).astype(np.float32)
  elif name == "saturated":                      # e_hat at +-20 ... +-90: sigmoid saturates
    w[p + "A.bias"][:] = (rng.choice([-1, 1], 256) * rng.uniform(20, 90, 256)).astype(np.float32)
  elif name == "max_negative":                   # every message negative: V h = b_V < 0
    w[p + "V.weight"][:] = 0
    w[p + "V.bias"][:] = -rng.uniform(0.5, 2.0, 256).astype(np.float32)
    agg = "max"
  elif name == "mean_deg1":
    case, agg = "deg1", "mean"
  elif name == "isolated_max":                   # nodes without edges: the oracle's max turns -inf into 0
    task, case, agg = "mis", "isolated", "max"
  V, ei, *_ = _case(case)
  h = rng.standard_normal((V, 256)).astype(np.float32)
  e = rng.standard_normal((ei.shape[1], 256)).astype(np.float32)
  if name == "offset_e":                         # |mean| / std = 1e3 per row
    e = (e + 1e3 * rng.choice([-1, 1], (ei.shape[1], 1))).astype(np.float32)
  return w, task, case, agg, h, e


EDGE_CASES = ["offset_e", "flat1e-4", "flat1e-5", "flat1e-6", "saturated", "max_negative", "mean_deg1", "isolated_max"]
_edge_cache = {}


# measured on an H100 (DESIGN section 2); strict, so the test reports when the loss goes away
_OFFSET_BF16X3 = pytest.mark.xfail(strict=True, reason=(
    "offset e rows, bf16x3 GEMM1: C e at |mean| / std = 1e3 carries ~8x the fp32 error into e_hat, and the gates pass "
    "it to h: h rel 2.1e-4 against a bound of 1.05e-4 (4 x the fp32 oracle's 2.6e-5); e rel 6.8e-8"))


@pytest.mark.gpu
@pytest.mark.parametrize("name,impl", [pytest.param(n, i, marks=[_OFFSET_BF16X3] if (n, i) in (("offset_e", "tc"),
                                                                                             ("offset_e", "tc1")) else [])
                                       for n in EDGE_CASES for i in IMPLS])
def test_one_layer_value_edges_vs_fp64_oracle(name, impl):
  if name not in _edge_cache:
    _edge_cache.clear()
    w, task, case, agg, h, e = _edge_case(name)
    _edge_cache[name] = (w, task, case, agg, h, e, _refs(w, task, case, MID, h, e, agg))
  w, task, case, agg, h, e, (r64, r32) = _edge_cache[name]
  V, ei, *_ = _case(case)
  got_h, got_e = _run_layer(_engine(w, task), ei, V, MID, h, e, impl, agg)
  _check_layer(got_h, got_e, h, e, r64, r32, task, MID, N_LAYERS, impl, f"{name} {impl}")


def test_value_edges_reach_their_targets():
  """The edge cases put the layer where they claim (fp64 oracle pieces, CPU)."""
  for name in EDGE_CASES:
    w, task, case, agg, h, e = _edge_case(name)
    V, ei, *_ = _case(case)
    W = orc.Weights(w, torch.float64)
    p = f"layers.{MID}."
    hd, ed = torch.as_tensor(h, dtype=torch.float64), torch.as_tensor(e, dtype=torch.float64)
    row, col = torch.as_tensor(ei[0]), torch.as_tensor(ei[1])
    e_hat = W.lin(p + "A", hd)[col] + W.lin(p + "B", hd)[row] + W.lin(p + "C", ed)
    if name == "offset_e":
      r = ed.mean(1).abs() / ed.std(1)
      assert (r > 500).all() and (r < 2000).all()
    elif name.startswith("flat"):
      var = float(name[4:])
      v = e_hat.var(1, unbiased=False).numpy()
      assert (v > var / 3).all() and (v < 3 * var).all(), (name, v.min(), v.max())
      assert (e_hat.mean(1) - 3).abs().max() < 0.01
    elif name == "saturated":
      assert (e_hat.abs() > 15).float().mean() > 0.95
    elif name == "max_negative":
      assert (torch.sigmoid(e_hat) * W.lin(p + "V", hd)[col] < 0).all()
    elif name == "mean_deg1":
      assert (np.bincount(ei[0], minlength=V) == 1).all()
    elif name == "isolated_max":
      assert set(np.flatnonzero(np.bincount(ei[0], minlength=V) == 0)) == set(G.ISOLATED)


# ------------------------------------------------------------------------------------------------
# c. depth: L = 1, 2, 5, 64 through the public API
# ------------------------------------------------------------------------------------------------
DEPTHS = [1, 2, 5, 64]
TOL = 1e-4
P_BIG = 1e-3
T_FWD = 500.0
_depth_weights = {}


def _dweights(L, out_channels):
  key = (L, out_channels)
  if key not in _depth_weights:
    _depth_weights[key] = syn.make_encoder_weights(10 + L, n_layers=L, out_channels=out_channels)
  return _depth_weights[key]


_depth_inputs = {}


def _depth_case(case):
  if case not in _depth_inputs:
    if case in ("tsp", "tsp_gauss"):
      pts, ei = syn.tsp_sparse_batch(50, 20, 2, seed=64)
      xt = syn.initial_noise(ei.shape[1], 65)
      _depth_inputs[case] = (pts, ei, xt if case == "tsp_gauss" else (xt > 0).astype(np.float32))
    elif case == "mis":
      _depth_inputs[case] = (syn.er_graph_edge_index(150, 0.05, seed=66), (syn.initial_noise(150, 67) > 0).astype(np.float32))
    else:   # dense TSP-20, B = 2
      pts = np.stack([syn.tsp_points(20, 68, b) for b in range(2)]).astype(np.float32)
      _depth_inputs[case] = (pts, (syn.initial_noise(800, 69) > 0).astype(np.float32).reshape(2, 20, 20))
  return _depth_inputs[case]


def _depth_oracle(L, case, dtype):
  w = _dweights(L, 1 if case == "tsp_gauss" else 2)
  W = orc.Weights(w, dtype=dtype)
  tt = np.array([T_FWD])
  if case in ("tsp", "tsp_gauss"):
    pts, ei, xt = _depth_case(case)
    return orc.encoder_forward_sparse_tsp(W, pts, xt, tt, ei).numpy()
  if case == "mis":
    ei, xt = _depth_case(case)
    return orc.encoder_forward_mis(W, xt, tt, ei).numpy()
  pts, xt = _depth_case(case)
  outs = [orc.encoder_forward_dense(W, pts[b:b + 1], xt[b:b + 1], tt.astype(np.float32)) for b in range(2)]
  return np.stack([o[0].permute(1, 2, 0).reshape(-1, o.shape[1]).numpy() for o in outs])


def _errors(out, ref):
  e = {"logits": rel_linf(out, ref)}
  if ref.shape[-1] == 2:
    p = torch.softmax(torch.as_tensor(np.asarray(out, np.float64)), -1).numpy()
    pr = torch.softmax(torch.as_tensor(np.asarray(ref, np.float64)), -1).numpy()
    e["p_abs"] = float(np.abs(p - pr).max())
    big = pr >= P_BIG
    e["p_rel"] = float(np.abs(p[big] / pr[big] - 1).max())
  return e


@pytest.mark.gpu
@pytest.mark.parametrize("L,case,impl", [(L, c, i) for L in DEPTHS for c in ("tsp", "tsp_gauss", "mis", "dense20")
                                         for i in IMPLS])
def test_encoder_depth_vs_fp64_oracle(L, case, impl):
  """logits rel-L-inf within G.TOL[impl], softmax p within 1e-4 (absolute, and relative where p >= 1e-3); each bound
  max(that, 4 x the fp32 oracle's error)."""
  oc = 1 if case == "tsp_gauss" else 2
  w = _dweights(L, oc)
  if case == "mis":
    ei, xt = _depth_case(case)
    enc = G.load(GNNEncoder(L, 256, oc, sparse=True, node_feature_only=True), w)
    enc.engine().set_edge_impl(G.IMPLS[impl])
    out = enc(G.cu(xt), torch.tensor([T_FWD]), edge_index=G.cu(ei)).cpu().numpy()
  elif case == "dense20":
    pts, xt = _depth_case(case)
    enc = G.load(GNNEncoder(L, 256, oc, sparse=False), w)
    enc.engine().set_edge_impl(G.IMPLS[impl])
    out = enc(G.cu(pts), torch.tensor([T_FWD]), G.cu(xt)).cpu().numpy().transpose(0, 2, 3, 1).reshape(2, 400, oc)
  elif case == "tsp_gauss":
    pts, ei, xt = _depth_case(case)
    enc = G.load(GNNEncoder(L, 256, oc, sparse=True), w)
    enc.engine().set_edge_impl(G.IMPLS[impl])
    out = enc(G.cu(pts), torch.tensor([T_FWD]), G.cu(xt), G.cu(ei)).cpu().numpy()
  else:   # categorical TSP: dfb_denoise_step's network output, whose layer 0 reads the 2-row LUT
    pts, ei, xt = _depth_case(case)
    enc = G.load(GNNEncoder(L, 256, oc, sparse=True), w)
    ctx = enc.set_graph(G.cu(ei), pts.shape[0], 1)
    enc.set_points(G.cu(pts))
    ctx.set_edge_impl(G.IMPLS[impl])
    _, Q_bar = orc.categorical_tables(1000, "linear")
    n = ei.shape[1]
    x, xo, net = G.cu(xt), torch.empty(n, device="cuda"), torch.empty((n, 2), device="cuda")
    ctx.denoise_step(_cabi.CATEGORICAL, x.data_ptr(), T_FWD, orc.categorical_posterior_consts(Q_bar, 500, 480).reshape(-1),
                     0, G.cu(syn.uniforms(n, 71)).data_ptr(), 0, 0, xo.data_ptr(), None, net.data_ptr(), _stream())
    torch.cuda.synchronize()
    out = net.cpu().numpy()
  r64, r32 = _depth_oracle(L, case, torch.float64), _depth_oracle(L, case, torch.float32)
  assert out.shape == r64.shape and np.isfinite(out).all()
  for b in range(r64.shape[0]) if case == "dense20" else [None]:
    o, a, c = (out, r64, r32) if b is None else (out[b], r64[b], r32[b])
    got, yard = _errors(o, a), _errors(c, a)
    base = {"logits": G.TOL[impl], "p_abs": TOL, "p_rel": TOL}
    bound = {k: max(base[k], 4 * v) for k, v in yard.items()}
    assert all(got[k] <= bound[k] for k in got), f"L={L} {case} {impl} sample {b}: {got} | fp32 {yard} | {bound}"


STEPS = 5


def _loop_model(L, task):
  w = _dweights(L, 2)
  kw = dict(n_layers=L, inference_diffusion_steps=STEPS)
  return G.tsp_model(w, "tc", sparse_factor=20, **kw) if task == "tsp" else G.mis_model(w, "tc", **kw), w


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 2])
@pytest.mark.parametrize("task", ["tsp", "mis"])
def test_shallow_denoise_loop_captured_plain_stepwise_and_oracle(L, task):
  """dfb_denoise captured == plain launches == a loop of dfb_denoise_step, bitwise, with injected uniforms; against
  orc.denoise the heat map is within 1e-4 unless the oracle's trajectory has a tie |p - u| < 1e-4 (as in
  test_gpu_parity_full.py)."""
  m, w = _loop_model(L, task)
  if task == "tsp":
    pts, ei, xt = _depth_case("tsp")
    m._prepare(G.cu(pts), G.cu(ei), torch.device("cuda"))
    n = ei.shape[1]
  else:
    ei, xt = _depth_case("mis")
    n = xt.size
    m.model.set_graph(G.cu(ei), n, 1)
  ctx = m.model.engine()
  st = _stream()
  sched = orc.inference_schedule("cosine", 1000, STEPS)
  t1s, cs, ls = [], [], []
  for t1, t2 in sched:
    c, last = m.posterior_consts(t1, t2)
    t1s.append(int(t1)); cs.append(c); ls.append(last)
  us = [syn.uniforms(n, 70 + L, i) for i in range(STEPS)]
  ud = G.cu(np.stack(us))
  runs = []
  for capture in (True, False):
    ctx.set_graph_capture(capture)
    x = G.cu(xt)
    ctx.denoise(_cabi.CATEGORICAL, x.data_ptr(), t1s, cs, ls, ud.data_ptr(), 0, st)
    torch.cuda.synchronize()
    runs.append(x.cpu().numpy())
  ctx.set_graph_capture(True)
  y = G.cu(xt)
  for i in range(STEPS):
    yo = torch.empty_like(y)
    ctx.denoise_step(_cabi.CATEGORICAL, y.data_ptr(), float(t1s[i]), cs[i], ls[i], G.cu(us[i]).data_ptr(), 0, i,
                     yo.data_ptr(), None, None, st)
    y = yo
  torch.cuda.synchronize()
  assert np.array_equal(runs[0], runs[1]) and np.array_equal(runs[0], y.cpu().numpy())
  rec = []
  orc.denoise(orc.Weights(w, torch.float64), task, "categorical", ei, xt, points=pts if task == "tsp" else None,
              steps=STEPS, uniforms=us, record=rec)
  ref = rec[-1]["xt_out"].numpy()
  got = runs[0]
  big = ref > P_BIG
  ok = np.abs(got - ref).max() < TOL * max(ref.max(), 1e-3) and np.abs(got[big] / ref[big] - 1).max() < TOL
  if not ok:
    near = [np.abs(r["p"].numpy() - us[i]) < TOL for i, r in enumerate(rec[:-1])]
    if any(nm.any() for nm in near):
      pytest.skip("oracle trajectory has a tie |p - u| < 1e-4 and the loop took the other branch")
  assert ok


def _raw_context(w, L):
  ctx = _cabi.Context(torch.cuda.current_device())
  ctx.load_weights(w, L, 256, 2, 0, consts=reference_frequency_tables(256))
  return ctx


def _raw_run(ctx, L):
  """Forward logits and a captured 3-step loop's heat map on the TSP depth case."""
  pts, ei, xt = _depth_case("tsp")
  E = ei.shape[1]
  eid, pd = G.cu(ei), G.cu(pts)
  st = _stream()
  ctx.prepare_graph(eid.data_ptr(), pts.shape[0], E, 1, st)
  ctx.set_points(pd.data_ptr(), st)
  x, out = G.cu(xt), torch.empty((E, 2), device="cuda")
  ctx.encoder_forward(x.data_ptr(), T_FWD, out.data_ptr(), st)
  sched = orc.inference_schedule("cosine", 1000, 3)
  _, Q_bar = orc.categorical_tables(1000, "linear")
  cs = [orc.categorical_posterior_consts(Q_bar, t1, t2).reshape(-1) for t1, t2 in sched]
  ls = [int(t2 == 0) for _, t2 in sched]
  u = G.cu(np.stack([syn.uniforms(E, 80, i) for i in range(3)]))
  y = G.cu(xt)
  ctx.denoise(_cabi.CATEGORICAL, y.data_ptr(), [t1 for t1, _ in sched], cs, ls, u.data_ptr(), 0, st)
  torch.cuda.synchronize()
  return out.cpu().numpy(), y.cpu().numpy()


@pytest.mark.gpu
def test_one_context_reloaded_across_depths_matches_fresh_contexts():
  """12 -> 1 -> 64 -> 12 layers on one context: the bf16 arena and its tensor map are rebound, tvec grows, the captured
  loop is re-captured; forward and loop must equal a fresh context's bitwise."""
  shared = None
  for L in (12, 1, 64, 12):
    w = _dweights(L, 2)
    if shared is None:
      shared = _raw_context(w, L)
    else:
      shared.load_weights(w, L, 256, 2, 0, consts=reference_frequency_tables(256))
    fwd, loop = _raw_run(shared, L)
    fresh = _raw_context(w, L)
    fwd0, loop0 = _raw_run(fresh, L)
    fresh.close()
    assert np.array_equal(fwd, fwd0) and np.array_equal(loop, loop0), L
  shared.close()


@pytest.mark.gpu
@pytest.mark.parametrize("L", [0, 65])
def test_n_layers_out_of_range_raises(L):
  ctx = _cabi.Context(torch.cuda.current_device())
  with pytest.raises(ValueError):
    ctx.load_weights(_dweights(1, 2), L, 256, 2, 0)
  ctx.close()


# ------------------------------------------------------------------------------------------------
# d. the oracle's layer_step is the encoder loop's layer (CPU)
# ------------------------------------------------------------------------------------------------
def test_layer_step_chain_reproduces_forward_taps_bitwise(weights2):
  V, ei, pts, xe, xv = _case("tsp_shuf")
  W = orc.Weights(weights2)
  taps = []
  orc.encoder_forward_sparse_tsp(W, pts, xe, np.array([T_LAYER]), ei, taps=taps)
  h, e, temb = _initial_state(W, "tsp", "tsp_shuf")
  row, col = torch.as_tensor(ei[0]), torch.as_tensor(ei[1])
  assert len(taps) == N_LAYERS
  for l in range(N_LAYERS):
    h, e = orc.layer_step(W, l, h, e, row, col, temb, True)
    assert torch.equal(h, taps[l][0]) and torch.equal(e, taps[l][1]), l

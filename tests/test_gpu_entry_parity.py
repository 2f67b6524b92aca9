"""The first stage of the forward alone against the fp64 oracle, through dfb_debug_entry, and denoise loops of 1000 and
4096 steps.

dfb_debug_gnn_layer runs a layer on a state the test sets, so it never reads what only a forward's layer 0 reads: the
categorical edge-embedding LUT, the MIS e0 = 0 and the layer-0 node linears cached by dfb_set_points.  dfb_debug_entry
runs run_entry (node / edge embeddings through k_pos_features, k_scalar_features, the embedding linears and k_lut_expand)
and layer 0 as run_forward runs it, after the staged time MLP (k_time_vectors).

  a. h0 and e0: points at 0, at 1 and at coordinates in the 10^3 range; Gaussian xt at +-0, +-1e-3, +-5 on shuffled
     edges; the LUT rows categorical TSP selects; V and E at 65535, 65536, 65537 (the 65536-row chunk loops).
  b. The time vectors of all 12 layers at t = 1, 2, 500, 999, 1000.
  c. Layer 0 as the forward runs it against oracle.layer_step on the fp64 embeddings: categorical TSP (LUT) sorted and
     shuffled, Gaussian TSP, MIS with e0 = 0; tc, tc1, fp32; sum, mean, max.
  d. Loops on TSP-20 (K = 5): 1000 steps categorical, Gaussian DDIM and DDPM; 4096 steps at L = 1; logits and p of
     recorded steps against the oracle on the recorded input state; captured == plain launches bitwise; 4097 steps
     rejected; test_step at 1000 steps returns valid tours.

Metric of a-c: the largest per-row relative L-inf (row_rel of test_gpu_layer_parity.py) with its bound
max(BASE[impl], 4 x the fp32 oracle's error); the embeddings and time MLP are fp32 kernels under every impl except the
tensor-core embedding linears.
"""
import numpy as np
import pytest
import torch

from conftest import rel_linf
from difusco_b200 import _cabi, synthetic as syn
from difusco_b200.models.gnn_encoder import reference_frequency_tables
from oracle import difusco_oracle as orc
import gpu_util as G
from test_gpu_layer_parity import BASE, row_rel

torch.set_grad_enabled(False)

IMPLS = ["tc", "tc1", "fp32"]
AGGS = ["sum", "mean", "max"]
T = 700.0


def _stream():
  return torch.cuda.current_stream().cuda_stream


_ctx = {}
_w = {}


def _weights(oc, L=12):
  if (oc, L) not in _w:
    _w[(oc, L)] = syn.make_encoder_weights(40 + oc + L, n_layers=L, out_channels=oc)
  return _w[(oc, L)]


def _context(oc, node_only, L=12):
  key = (oc, node_only, L)
  if key not in _ctx:
    ctx = _cabi.Context(torch.cuda.current_device())
    ctx.load_weights(_weights(oc, L), L, 256, oc, int(node_only), consts=reference_frequency_tables(256))
    _ctx[key] = ctx
  return _ctx[key]


def _within(got, yard, base, what):
  bound = {k: max(base, 4 * v) for k, v in yard.items()}
  print(f"\n{what}: {got} | fp32 oracle {yard}")
  bad = [k for k in got if not got[k] <= bound[k]]
  assert not bad, f"{what} failing {bad}: kernel {got} | fp32 oracle {yard} | bounds {bound}"


# ------------------------------------------------------------------------------------------------
# cases: name -> (task, diffusion, V, edge_index caller order, points, xt)
# ------------------------------------------------------------------------------------------------
def _case(name):
  rng = np.random.default_rng(sum(map(ord, name)))
  if name.startswith("chunk"):   # V = E = n: a ring with a self loop on node 0 instead of the edge 0 -> 1
    n = int(name[5:].split("_")[0])
    ei = np.stack([np.arange(n), (np.arange(n) + 1) % n]).astype(np.int64)
    ei[1, 0] = 0
    task = "mis" if name.endswith("mis") else "tsp"
    pts = rng.random((n, 2)).astype(np.float32)
    xt = rng.standard_normal(n).astype(np.float32) if task == "tsp" else (rng.random(n) < 0.5).astype(np.float32)
    return task, "gaussian" if task == "tsp" else "categorical", n, ei, pts, xt
  if name == "mis":
    V = 150
    return "mis", "categorical", V, syn.er_graph_edge_index(V, 0.05, seed=62), None, (rng.random(V) < 0.5).astype(np.float32)
  V = 60
  pts = rng.random((V, 2)).astype(np.float32)
  if name.startswith("pts_edges"):   # points at exactly 0 and 1, and TSPLIB-like coordinates in the 10^3 range
    pts[:10] = 0.0
    pts[10:20] = 1.0
    pts[20:30, 0] = 0.0
    pts[30:40, 1] = 1.0
    pts[40:] = (rng.random((20, 2)) * 4000.0).round(1).astype(np.float32)
  ei = syn.knn_edge_index(pts.astype(np.float64), 8)
  if name.endswith("_shuf"):
    ei = ei[:, rng.permutation(ei.shape[1])]
  E = ei.shape[1]
  if "gauss" in name:   # +-0, +-1e-3, +-5 and ordinary values
    xt = rng.choice(np.array([0.0, -0.0, 1e-3, -1e-3, 5.0, -5.0, 0.3, -1.7], np.float32), E)
    return "tsp", "gaussian", V, ei, pts, xt
  return "tsp", "categorical", V, ei, pts, (rng.random(E) < 0.3).astype(np.float32)


def _oc(diffusion):
  return 2 if diffusion == "categorical" else 1


def _run_entry(name, impl="tc", agg="sum", t=T, outputs=("h0", "e0", "tvec", "h", "e")):
  task, diff, V, ei, pts, xt = _case(name)
  ctx = _context(_oc(diff), task == "mis")
  ctx.set_edge_impl(G.IMPLS[impl])
  ctx.set_aggregation(agg)
  E = ei.shape[1]
  eid = G.cu(ei)
  ctx.prepare_graph(eid.data_ptr(), V, E, 1, _stream())
  if task == "tsp":
    pd = G.cu(pts)
    ctx.set_points(pd.data_ptr(), _stream())
  shapes = {"h0": (V, 256), "e0": (E, 256), "tvec": (12, 256), "h": (V, 256), "e": (E, 256)}
  bufs = {k: torch.full(shapes[k], float("nan"), device="cuda") for k in outputs}
  ptr = lambda k: bufs[k].data_ptr() if k in bufs else None
  x = G.cu(xt)
  ctx.debug_entry(_cabi.CATEGORICAL if diff == "categorical" else _cabi.GAUSSIAN, x.data_ptr(), t, ptr("h0"), ptr("e0"),
                  ptr("tvec"), ptr("h"), ptr("e"), _stream())
  torch.cuda.synchronize()
  out = {k: v.cpu().numpy() for k, v in bufs.items()}
  perm = np.argsort(ei[0], kind="stable")
  for k in ("e0", "e"):   # row-sorted -> caller order
    if k in out:
      o = np.empty_like(out[k])
      o[perm] = out[k]
      out[k] = o
  return out


def _embeddings(name, dtype):
  task, diff, V, ei, pts, xt = _case(name)
  W = orc.Weights(_weights(_oc(diff)), dtype)
  if task == "tsp":
    h = W.lin("node_embed", orc.pos_embed_2d(torch.as_tensor(pts).to(dtype), 256))
    e = W.lin("edge_embed", orc.scalar_embed(torch.as_tensor(xt).to(dtype), 256))
  else:
    h = W.lin("node_embed", orc.scalar_embed(torch.as_tensor(xt).to(dtype), 256))
    e = torch.zeros((ei.shape[1], 256), dtype=dtype)
  return W, h, e


# ------------------------------------------------------------------------------------------------
# a. h0 and e0
# ------------------------------------------------------------------------------------------------
EMBED_CASES = ["pts_edges", "pts_edges_gauss_shuf", "tsp_shuf", "mis"] + \
              [f"chunk{n}{s}" for n in (65535, 65536, 65537) for s in ("", "_mis")]


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("name", EMBED_CASES)
def test_embeddings_vs_fp64_oracle(name, impl):
  task, diff, *_ = _case(name)
  out = _run_entry(name, impl, outputs=("h0", "e0"))
  _, h64, e64 = _embeddings(name, torch.float64)
  _, h32, e32 = _embeddings(name, torch.float32)
  got, yard = {"h0": row_rel(out["h0"], h64)}, {"h0": row_rel(h32, h64)}
  if task == "tsp":
    got["e0"], yard["e0"] = row_rel(out["e0"], e64), row_rel(e32, e64)
  else:
    assert np.isnan(out["e0"]).all(), "MIS has no e0 to write"
  _within(got, yard, BASE[impl], f"{name} {impl}")


@pytest.mark.gpu
def test_lut_rows_equal_fp64_edge_embedding_of_0_and_1():
  out = _run_entry("tsp_shuf", "tc", outputs=("e0",))
  _, _, _, ei, _, xt = _case("tsp_shuf")
  W64, W32 = orc.Weights(_weights(2), torch.float64), orc.Weights(_weights(2), torch.float32)
  r64 = W64.lin("edge_embed", orc.scalar_embed(torch.tensor([0.0, 1.0], dtype=torch.float64), 256)).numpy()
  r32 = W32.lin("edge_embed", orc.scalar_embed(torch.tensor([0.0, 1.0]), 256)).numpy()
  sel = xt.astype(np.int64)
  assert 0 < sel.mean() < 1
  for v in (0, 1):   # every edge with xt = v holds the same row, bit for bit
    rows = out["e0"][sel == v]
    assert (rows == rows[0]).all()
  _within({"lut": row_rel(out["e0"], r64[sel])}, {"lut": row_rel(r32, r64)}, BASE["fp32"], "LUT rows")


# ------------------------------------------------------------------------------------------------
# b. time vectors
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("t", [1.0, 2.0, 500.0, 999.0, 1000.0])
def test_time_vectors_vs_fp64_oracle(t):
  out = _run_entry("tsp_shuf", "fp32", t=t, outputs=("tvec",))["tvec"]
  ref = {}
  for dt in (torch.float64, torch.float32):
    W = orc.Weights(_weights(2), dt)
    temb = orc._time_emb(W, torch.tensor([t]))
    ref[dt] = np.concatenate([W.lin(f"time_embed_layers.{l}.1", torch.relu(temb)).numpy() for l in range(12)])
  _within({"tvec": row_rel(out, ref[torch.float64])}, {"tvec": row_rel(ref[torch.float32], ref[torch.float64])},
          BASE["fp32"], f"t={t}")


# ------------------------------------------------------------------------------------------------
# c. layer 0 as the forward runs it
# ------------------------------------------------------------------------------------------------
LAYER0_CASES = ["tsp", "tsp_shuf", "tsp_gauss_shuf", "mis"]


@pytest.mark.gpu
@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("name", LAYER0_CASES)
def test_layer0_as_forward_runs_it_vs_fp64_oracle(name, impl, agg):
  task, diff, V, ei, pts, xt = _case(name)
  out = _run_entry(name, impl, agg, outputs=("h", "e"))
  row, col = torch.as_tensor(ei[0]), torch.as_tensor(ei[1])
  ref = {}
  for dt in (torch.float64, torch.float32):
    W, h, e = _embeddings(name, dt)
    temb = orc._time_emb(W, torch.tensor([T]))
    hh, ee = orc.layer_step(W, 0, h, e, row, col, temb, task == "tsp", agg)
    ref[dt] = (hh.numpy(), ee.numpy())
  got = {"h": row_rel(out["h"], ref[torch.float64][0]), "e": row_rel(out["e"], ref[torch.float64][1])}
  yard = {"h": row_rel(ref[torch.float32][0], ref[torch.float64][0]),
          "e": row_rel(ref[torch.float32][1], ref[torch.float64][1])}
  _within(got, yard, BASE[impl], f"{name} {impl} {agg}")


@pytest.mark.gpu
def test_entry_hook_rejects_bad_arguments():
  ctx = _context(2, False)
  _, _, V, ei, pts, xt = _case("tsp")
  eid = G.cu(ei)
  ctx.prepare_graph(eid.data_ptr(), V, ei.shape[1], 1, _stream())
  x = G.cu(xt)
  with pytest.raises(ValueError):   # TSP before dfb_set_points
    ctx.debug_entry(_cabi.CATEGORICAL, x.data_ptr(), T, stream=_stream())
  ctx.set_points(G.cu(pts).data_ptr(), _stream())
  with pytest.raises(ValueError):   # a 2-channel head is not Gaussian
    ctx.debug_entry(_cabi.GAUSSIAN, x.data_ptr(), T, stream=_stream())
  with pytest.raises(ValueError):
    ctx.debug_entry(_cabi.CATEGORICAL, xt.ctypes.data, T, stream=_stream())


# ------------------------------------------------------------------------------------------------
# d. long loops
# ------------------------------------------------------------------------------------------------
N_LOOP, K_LOOP = 20, 5
LOOP_MODES = ["categorical", "ddim", "ddpm"]


def _loop_model(mode, L, steps):
  oc = 2 if mode == "categorical" else 1
  kw = dict(n_layers=L, inference_diffusion_steps=steps, sparse_factor=K_LOOP,
            diffusion_type="categorical" if mode == "categorical" else "gaussian",
            inference_trick=None if mode == "ddpm" else "ddim")
  return G.tsp_model(_weights(oc, L), "tc", **kw)


def _loop(mode, L, steps, record):
  """-> (points, edge_index, per recorded step (t1, t2, xt_in, net_out, p or None, xt_out), loop handles)."""
  m = _loop_model(mode, L, steps)
  pts = syn.tsp_points(N_LOOP, 91)
  ei = syn.knn_edge_index(pts, K_LOOP)
  E = ei.shape[1]
  m._prepare(G.cu(pts.astype(np.float32)), G.cu(ei), torch.device("cuda"))
  ctx = m.model.engine()
  sched = orc.inference_schedule("cosine", 1000, steps)
  t1s, cs, ls = [], [], []
  for t1, t2 in sched:
    c, last = m.posterior_consts(t1, t2)
    t1s.append(int(t1)); cs.append(c); ls.append(last)
  t2s = [int(t2) for _, t2 in sched]
  noise = syn.initial_noise(E, 92)
  xt0 = (noise > 0).astype(np.float32) if mode == "categorical" else noise.astype(np.float32)
  # every recorded step and the step before it, whose output is the recorded step's input
  rs = sorted(set(record) | {s - 1 for s in record if s > 0})
  oc = 2 if mode == "categorical" else 1
  runs = []
  for capture in (True, False):
    ctx.set_graph_capture(capture)
    x = G.cu(xt0)
    rx, ro = torch.full((len(rs), E), np.nan, device="cuda"), torch.full((len(rs), E, oc), np.nan, device="cuda")
    rp = torch.full((len(rs), E), np.nan, device="cuda") if mode == "categorical" else None
    ctx.denoise_record(_cabi.CATEGORICAL if mode == "categorical" else _cabi.GAUSSIAN, x.data_ptr(), t1s, cs, ls, rs,
                       rx.data_ptr(), None if rp is None else rp.data_ptr(), ro.data_ptr(), None, 5, _stream())
    torch.cuda.synchronize()
    runs.append((x.cpu().numpy(), rx.cpu().numpy(), ro.cpu().numpy(), None if rp is None else rp.cpu().numpy()))
  ctx.set_graph_capture(True)
  for a, b in zip(runs[0], runs[1]):
    assert (a is None and b is None) or np.array_equal(a, b, equal_nan=True), "captured loop != plain launches"
  x, rx, ro, rp = runs[0]
  steps_out = []
  for s in record:
    j = rs.index(s)
    xin = xt0 if s == 0 else rx[rs.index(s - 1)]
    steps_out.append((t1s[s], t2s[s], xin, ro[j], None if rp is None else rp[j], rx[j]))
  return pts, ei, steps_out, (m, ctx, t1s, cs, ls, xt0)


def _check_steps(mode, L, pts, ei, steps_out):
  for t1, t2, xin, net, p, _ in steps_out:
    assert np.isfinite(net).all()
    ref = {dt: orc.encoder_forward_sparse_tsp(orc.Weights(_weights(net.shape[1], L), dt), pts, xin, np.array([t1]),
                                              ei).numpy() for dt in (torch.float64, torch.float32)}
    got, yard = {"logits": rel_linf(net, ref[torch.float64])}, {"logits": rel_linf(ref[torch.float32], ref[torch.float64])}
    base = {"logits": G.TOL["tc"]}
    if p is not None:
      _, Q_bar = orc.categorical_tables(1000, "linear")
      pr = {}
      for dt, r in ref.items():
        pr[dt] = orc.categorical_posterior(Q_bar, t1, t2, torch.softmax(torch.as_tensor(r), -1),
                                           torch.as_tensor(xin).to(dt), np.zeros(len(xin), np.float32))[0].numpy()
      got["p_abs"], yard["p_abs"] = float(np.abs(p - pr[torch.float64]).max()), float(np.abs(pr[torch.float32] -
                                                                                             pr[torch.float64]).max())
      base["p_abs"] = 1e-4
    bound = {k: max(base[k], 4 * v) for k, v in yard.items()}
    print(f"\n{mode} L={L} t1={t1}: {got} | fp32 {yard}")
    assert all(got[k] <= bound[k] for k in got), (mode, L, t1, got, yard, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", LOOP_MODES)
def test_1000_step_loop_recorded_steps_vs_fp64_oracle(mode):
  pts, ei, steps_out, _ = _loop(mode, 12, 1000, [0, 1, 499, 998, 999])
  _check_steps(mode, 12, pts, ei, steps_out)


@pytest.mark.gpu
def test_4096_step_loop_at_one_layer_and_4097_rejected():
  pts, ei, steps_out, (m, ctx, t1s, cs, ls, xt0) = _loop("categorical", 1, 4096, [0, 2047, 4095])
  _check_steps("categorical", 1, pts, ei, steps_out)
  E = ei.shape[1]
  x = G.cu(xt0)
  rx = torch.full((1, E), 7.0, device="cuda")
  with pytest.raises(ValueError):
    ctx.denoise_record(_cabi.CATEGORICAL, x.data_ptr(), t1s + [1], cs + [cs[-1]], ls + [1], [0], rx.data_ptr(),
                       None, None, None, 5, _stream())
  torch.cuda.synchronize()
  assert np.array_equal(x.cpu().numpy(), xt0) and (rx.cpu().numpy() == 7.0).all()


@pytest.mark.gpu
def test_test_step_with_1000_inference_steps_returns_valid_tours():
  from test_gpu_solve_batch import _sparse_tsp_batch, _tsp_parts
  m = _loop_model("categorical", 12, 1000)
  parts = _tsp_parts([(N_LOOP, K_LOOP)], 93)
  torch.manual_seed(0)
  m.test_step(_sparse_tsp_batch(parts), 0)
  tour = np.asarray(m.last_solved_tours).reshape(-1, N_LOOP + 1)
  for t in tour:
    assert t[0] == t[-1] and sorted(t[:-1]) == list(range(N_LOOP))
  assert np.isfinite(m.last_solved_cost) and m.last_solved_cost > 0

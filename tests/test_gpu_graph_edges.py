"""The fused encoder on irregular graphs, at tile / chunk boundaries, and the in-kernel Philox sampler.

Every other parity test builds a regular graph (k-NN rows of exactly K edges, ER graphs with self loops, the
complete graph).  The index arithmetic of the deterministic message reduction (per-(32-edge group, node) partials
written by the edge kernel, combined by k_node_update), the persistent tile loop, the host-side 65 536-row chunk
loops and the caller-order keying of the sampler only go wrong on graphs that are not, so the generators here
build: a hub spanning many tiles with degree-1 leaves, nodes without edges, degree sequences whose segment ends
land on and next to the 32 / 64 / 128-row boundaries, graphs smaller than one tile, duplicate edges without self
loops, and each of them again in a random edge order.  All generators are deterministic from integer seeds.

The sampler is checked element for element against oracle/philox.py, the host restatement of common.cuh."""
import numpy as np
import pytest
import torch

from conftest import rel_linf
from difusco_b200 import _cabi, synthetic as syn
from oracle import difusco_oracle as orc
from oracle import philox
import gpu_util as G

pytestmark = pytest.mark.gpu
TOL = 1e-4
T_FWD = 700.0


FAMILIES = {"hub": G.hub_graph, "isolated": G.isolated_graph, "degseq": G.degseq_graph, "dup": G.dup_graph}
FAMILIES.update({f"tiny{E}": (lambda E=E: G.tiny_graph(E)) for E in G.TINY})
CASES = [f + s for f in FAMILIES for s in ("", "_shuf")]

_case_cache = {}


def _case(name):
  """-> V, edge_index, points (V,2), binary edge xt (E,), binary node xt (V,)."""
  if name not in _case_cache:
    shuf = name.endswith("_shuf")
    V, ei = FAMILIES[name[:-5] if shuf else name]()
    seed = sum(map(ord, name))
    if shuf:
      ei = ei[:, np.random.default_rng(seed).permutation(ei.shape[1])]
    rng = np.random.default_rng(seed + 1)
    pts = rng.random((V, 2), dtype=np.float32)
    xe = (rng.random(ei.shape[1]) < 0.3).astype(np.float32)
    xv = (rng.random(V) < 0.5).astype(np.float32)
    _case_cache[name] = (V, np.ascontiguousarray(ei), pts, xe, xv)
  return _case_cache[name]


def _forward(enc, task, case, t=T_FWD):
  V, ei, pts, xe, xv = _case(case)
  if task == "tsp":
    out = enc(G.cu(pts), torch.tensor([t]), G.cu(xe), G.cu(ei))
  else:
    out = enc(G.cu(xv), torch.tensor([t]), edge_index=G.cu(ei))
  return out.cpu().numpy()


@pytest.fixture(scope="module")
def encoders(weights2):
  made = {}

  def get(task, impl, agg):
    key = (task, impl, agg)
    if key not in made:
      made[key] = G.encoder(weights2, 2, node_only=task == "mis", impl=impl, aggregation=agg)
    return made[key]
  yield get
  made.clear()


_ref_cache = {}


def _ref64(weights2, case, task, agg):
  key = (case, task, agg)
  if key not in _ref_cache:
    V, ei, pts, xe, xv = _case(case)
    w = orc.Weights(weights2, dtype=torch.float64)
    if task == "tsp":
      r = orc.encoder_forward_sparse_tsp(w, pts, xe, np.array([T_FWD]), ei, aggregation=agg)
    else:
      r = orc.encoder_forward_mis(w, xv, np.array([T_FWD]), ei, aggregation=agg)
    _ref_cache[key] = r.numpy()
  return _ref_cache[key]


def test_generators_reach_the_boundaries_they_are_meant_to():
  ends = np.cumsum(G.DEGREES)
  for b in (32, 64, 128):
    assert {-1, 0, 1} <= {int(x) for x in ((ends + 1) % b) - 1}, b
  V, ei = G.hub_graph()
  deg = np.bincount(ei[0], minlength=V)
  assert deg.max() == 3000 and (deg.max() + 127) // 128 > 20 and (np.sort(deg)[:-1] == 1).all()
  V, ei = G.isolated_graph()
  deg = np.bincount(ei[0], minlength=V)
  assert set(np.flatnonzero(deg == 0)) == set(G.ISOLATED)
  V, ei = G.dup_graph()
  assert (ei[0] != ei[1]).all() and len({(a, b) for a, b in ei.T}) < ei.shape[1]
  for E, V in G.TINY.items():
    v, ei = G.tiny_graph(E)
    assert ei.shape == (2, E) and v == V and ei.max() < V
  for c in CASES:
    ei = _case(c)[1]
    if not c.endswith("_shuf"):
      assert (np.diff(ei[0]) >= 0).all(), c
    elif ei.shape[1] > 2:
      assert not (np.diff(ei[0]) >= 0).all(), c


# ------------------------------------------------------------------------------------------------
# a. irregular topologies, every implementation and aggregation, against the fp64 oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", ["tc", "tc1", "fp32"])
@pytest.mark.parametrize("agg", ["sum", "mean", "max"])
@pytest.mark.parametrize("task", ["tsp", "mis"])
@pytest.mark.parametrize("case", CASES)
def test_irregular_graph_vs_fp64_oracle(weights2, encoders, case, task, agg, impl):
  """TSP: edge outputs in the caller's edge order (the shuffled cases compare against the oracle run on the same
  shuffled list).  MIS: node outputs, including nodes without edges."""
  ref = _ref64(weights2, case, task, agg)
  out = _forward(encoders(task, impl, agg), task, case)
  assert out.shape == ref.shape and np.isfinite(out).all()
  err, perr = rel_linf(out, ref), G.prob_rel(out, ref)
  assert err < G.TOL[impl] and perr < TOL, (err, perr)


# ------------------------------------------------------------------------------------------------
# b. tile counts around the SM count of the device (the persistent grid is min(n_tiles, num_sms))
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", ["tc", "tc1"])
@pytest.mark.parametrize("which", ["sms-1", "sms", "sms+1", "2sms+1"])
def test_tile_counts_around_sm_count_vs_oracle(weights2, impl, which):
  sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
  n_tiles = {"sms-1": sms - 1, "sms": sms, "sms+1": sms + 1, "2sms+1": 2 * sms + 1}[which]
  tile = 128 if impl == "tc" else 64
  E = n_tiles * tile - 37                     # the last tile is partial
  rng = np.random.default_rng(n_tiles * 10 + tile)
  V = E // 6
  ei = np.stack([np.sort(rng.integers(0, V, E)), rng.integers(0, V, E)]).astype(np.int64)
  pts = rng.random((V, 2), dtype=np.float32)
  xt = (rng.random(E) < 0.3).astype(np.float32)
  assert (E + tile - 1) // tile == n_tiles
  torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
  ref = orc.encoder_forward_sparse_tsp(orc.Weights(weights2), pts, xt, np.array([T_FWD]), ei,
                                       gather_then_gemm=False).numpy()
  enc = G.encoder(weights2, 2, impl=impl)
  a = enc(G.cu(pts), torch.tensor([T_FWD]), G.cu(xt), G.cu(ei)).cpu().numpy()
  b = enc(G.cu(pts), torch.tensor([T_FWD]), G.cu(xt), G.cu(ei)).cpu().numpy()
  assert np.array_equal(a, b), "two runs on the same graph must be bitwise equal"
  assert rel_linf(a, ref) < TOL and G.prob_rel(a, ref) < TOL, (rel_linf(a, ref), G.prob_rel(a, ref))


# ------------------------------------------------------------------------------------------------
# c. the host-side 65 536-row chunk loops (feature rows are built 65 536 at a time), against the fp32 oracle
# ------------------------------------------------------------------------------------------------
CH = 65536


def _ring(V, offsets):
  i = np.arange(V, dtype=np.int64)
  return np.stack([np.repeat(i, len(offsets)), ((i[:, None] + np.array(offsets)) % V).reshape(-1)])


def test_chunked_tsp_points_vs_oracle(weights2):
  """dfb_set_points with V > 65 536: node embeddings of the second chunk."""
  V = CH + 300
  ei = _ring(V, [0, 1])
  rng = np.random.default_rng(31)
  pts = rng.random((V, 2), dtype=np.float32)
  xt = (rng.random(ei.shape[1]) < 0.5).astype(np.float32)
  torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
  ref = orc.encoder_forward_sparse_tsp(orc.Weights(weights2), pts, xt, np.array([T_FWD]), ei,
                                       gather_then_gemm=False).numpy()
  out = G.encoder(weights2, 2, impl="tc")(G.cu(pts), torch.tensor([T_FWD]), G.cu(xt), G.cu(ei)).cpu().numpy()
  assert rel_linf(out, ref) < TOL and G.prob_rel(out, ref) < TOL, (rel_linf(out, ref), G.prob_rel(out, ref))


def test_chunked_gaussian_edge_embedding_unsorted_vs_oracle(weights1):
  """Continuous xt with an unsorted edge list and E > 65 536: the edge embedding gathers xt through the sorting
  permutation chunk by chunk."""
  V = 17501
  ei = _ring(V, [0, 1, 2, 3])
  E = ei.shape[1]
  assert E > CH and (E - CH) % 128
  rng = np.random.default_rng(32)
  ei = np.ascontiguousarray(ei[:, rng.permutation(E)])
  pts = rng.random((V, 2), dtype=np.float32)
  xt = syn.initial_noise(E, 33)
  torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
  ref = orc.encoder_forward_sparse_tsp(orc.Weights(weights1), pts, xt, np.array([T_FWD]), ei,
                                       gather_then_gemm=False).numpy()
  out = G.encoder(weights1, 1, impl="tc")(G.cu(pts), torch.tensor([T_FWD]), G.cu(xt), G.cu(ei)).cpu().numpy()
  assert rel_linf(out, ref) < TOL, rel_linf(out, ref)


def test_chunked_mis_node_embedding_vs_oracle(weights2):
  """MIS with V > 65 536 on a ring with self loops: node embeddings of the second chunk."""
  V = CH + 300
  ei = _ring(V, [0, 1])
  xt = (np.random.default_rng(34).random(V) < 0.5).astype(np.float32)
  torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
  ref = orc.encoder_forward_mis(orc.Weights(weights2), xt, np.array([T_FWD]), ei, gather_then_gemm=False).numpy()
  out = G.encoder(weights2, 2, node_only=True, impl="tc")(G.cu(xt), torch.tensor([T_FWD]),
                                                         edge_index=G.cu(ei)).cpu().numpy()
  assert rel_linf(out, ref) < TOL and G.prob_rel(out, ref) < TOL, (rel_linf(out, ref), G.prob_rel(out, ref))


# ------------------------------------------------------------------------------------------------
# d. one context across many graphs == a fresh context per graph (arena, permutation, partials, captured loop)
# ------------------------------------------------------------------------------------------------
SEQUENCE = ["hub", "tiny1", "isolated_shuf", "degseq", "tiny129_shuf", "hub_shuf", "dup", "tiny33", "degseq_shuf",
            "isolated"]


@pytest.mark.parametrize("task", ["tsp", "mis"])
def test_one_context_across_graphs_matches_fresh_context(weights2, task):
  def model():
    if task == "tsp":
      return G.tsp_model(weights2, "tc", sparse_factor=8, inference_diffusion_steps=3)
    return G.mis_model(weights2, "tc", inference_diffusion_steps=3)

  def run(m, case):
    V, ei, pts, xe, xv = _case(case)
    fwd = _forward(m.model, task, case)
    if task == "tsp":
      loop = m.denoise_heatmap(G.cu(pts), G.cu(ei), G.cu(xe), seed=2 ** 40 + 7)
    else:
      loop = m.denoise_labels(G.cu(ei), G.cu(xv), seed=2 ** 40 + 7)
    return fwd, loop.cpu().numpy()

  shared = model()
  for case in SEQUENCE:
    fwd, loop = run(shared, case)
    fwd0, loop0 = run(model(), case)
    assert np.array_equal(fwd, fwd0), case
    assert np.array_equal(loop, loop0), case


# ------------------------------------------------------------------------------------------------
# e. the in-kernel sampler against oracle/philox.py
# ------------------------------------------------------------------------------------------------
SEED = (0xA5A5F00D << 32) | 0x1234567   # both 32-bit halves of the key non-zero
STEP = 7


def _tsp_setup(weights, n_nodes, offsets, shuffle_seed, **kw):
  m = G.tsp_model(weights, "tc", **kw)
  ei = _ring(n_nodes, offsets)
  rng = np.random.default_rng(shuffle_seed)
  ei = np.ascontiguousarray(ei[:, rng.permutation(ei.shape[1])])
  pts = rng.random((n_nodes, 2), dtype=np.float32)
  m._prepare(G.cu(pts), G.cu(ei), torch.device("cuda"))
  return m, ei


def _categorical_step(m, xt, seed, step, t1=500, t2=480):
  consts, last = m.posterior_consts(t1, t2)
  assert not last
  n = xt.numel()
  xo, p = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
  m.model.engine().denoise_step(_cabi.CATEGORICAL, xt.data_ptr(), float(t1), consts, last, None, seed, step,
                                xo.data_ptr(), p.data_ptr(), None, torch.cuda.current_stream().cuda_stream)
  return xo.cpu().numpy(), p.cpu().numpy()


@pytest.mark.parametrize("task", ["tsp", "mis"])
def test_categorical_sample_is_philox_uniform_of_caller_element(weights2, task):
  """xt_out == (u < clip(p, 0, 1)) exactly, u = philox.uniform(seed, step, caller element index).  The TSP edge
  list is unsorted, so a draw keyed by the sorted position would fail."""
  if task == "tsp":
    m, ei = _tsp_setup(weights2, 1500, [0, 3, 7, 11], 41)
    n = ei.shape[1]
  else:
    ei = syn.er_graph_edge_index(900, 0.02, seed=42)
    n = 900
    m = G.mis_model(weights2, "tc")
    m.model.set_graph(G.cu(ei), n, 1)
  xt = G.cu((syn.initial_noise(n, 43) > 0).astype(np.float32))
  xo, p = _categorical_step(m, xt, SEED, STEP)
  u = philox.uniform(SEED, STEP, np.arange(n, dtype=np.uint64))
  want = (u < np.clip(p, 0.0, 1.0)).astype(np.float32)
  assert 0.05 < want.mean() < 0.95
  bad = np.flatnonzero(xo != want)
  assert bad.size == 0, (bad.size, bad[:8])


def test_fused_loop_step_counter_is_loop_index(weights2):
  """dfb_denoise with Philox == dfb_denoise_step with step_index 0, 1, ... (same seed), bitwise."""
  m, ei = _tsp_setup(weights2, 700, [0, 2, 5], 44, inference_diffusion_steps=50)
  n = ei.shape[1]
  sched = orc.inference_schedule("cosine", 1000, 50)[:2]
  t1s, cs, ls = [], [], []
  for t1, t2 in sched:
    c, last = m.posterior_consts(t1, t2)
    assert not last
    t1s.append(int(t1)); cs.append(c); ls.append(last)
  x0 = G.cu((syn.initial_noise(n, 45) > 0).astype(np.float32))
  ctx = m.model.engine()
  st = torch.cuda.current_stream().cuda_stream
  x = x0.clone()
  ctx.denoise(_cabi.CATEGORICAL, x.data_ptr(), t1s, cs, ls, None, SEED, st)
  y = x0.clone()
  for i in range(2):
    yo = torch.empty_like(y)
    ctx.denoise_step(_cabi.CATEGORICAL, y.data_ptr(), float(t1s[i]), cs[i], ls[i], None, SEED, i, yo.data_ptr(),
                     None, None, st)
    y = yo
  torch.cuda.synchronize()
  assert np.array_equal(x.cpu().numpy(), y.cpu().numpy())
  assert not np.array_equal(x.cpu().numpy(), x0.cpu().numpy())


def test_gaussian_ddpm_noise_is_philox_normal(weights1):
  """DDPM (inference_trick=None) at t > 1: xt_out = a (x - b1 l0) + noise z with z = philox.normal(seed, step,
  caller element).  The kernel rounds a (x - b1 l0) exactly as numpy float32 does; what remains is one fma and the
  device's logf / sqrtf / cospif (a few ulps of z), so the bound is 4 float32 ulps of the output scale.  The z
  recovered from the output must also pass a KS test against N(0,1) over 120 000 elements."""
  from scipy import stats
  m, ei = _tsp_setup(weights1, 20000, [0, 1, 2, 3, 4, 5], 46, diffusion_type="gaussian", inference_trick=None)
  n = ei.shape[1]
  consts, last = m.posterior_consts(500, 480)
  a, b1, b2, c3 = [np.float32(c) for c in consts]
  assert not last and b2 == 0 and c3 > 0.01
  x = G.cu(syn.initial_noise(n, 47))
  xo, net = torch.empty(n, device="cuda"), torch.empty((n, 1), device="cuda")
  m.model.engine().denoise_step(_cabi.GAUSSIAN, x.data_ptr(), 500.0, consts, last, None, SEED, STEP, xo.data_ptr(),
                                None, net.data_ptr(), torch.cuda.current_stream().cuda_stream)
  xo, l0, xv = xo.cpu().numpy(), net.cpu().numpy()[:, 0], x.cpu().numpy()
  det = a * (xv - b1 * l0) + b2 * l0                    # float32, the kernel's operation order
  z = philox.normal(SEED, STEP, np.arange(n, dtype=np.uint64))
  want = det.astype(np.float64) + float(c3) * z
  scale = np.abs(xo).max()
  err = np.abs(xo - want).max()
  assert err <= 4 * np.spacing(np.float32(scale)), (err, scale)
  zr = (xo.astype(np.float64) - det) / float(c3)
  assert stats.kstest(zr, "norm").pvalue > 1e-3

"""A timestep per element at the places where the per-row time vector can go wrong: edges in the caller's order (the
`perm` branch of the lookup), row runs that change at the warpgroup and tile boundaries, more tiles than CTAs,
irregular graphs, mean / max aggregation, ragged instances, the 4096-entry table and the state it shares with the
captured loop.

test_gpu_timesteps.py checks dfb_encoder_forward_timesteps after 12 layers and the head, mostly on row-sorted edges.
Here dfb_debug_gnn_layer_timesteps runs one layer of the product code (run_layer, as the forward runs it) with a time
vector per row, so a wrong tau row meets the comparison in the layer that reads it.

  a. Teacher-forced layers: the fp64 forward with per-row time embeddings, the state entering each of the 12 layers
     rounded to fp32, through the hook (metric and bound of test_gpu_layer_parity.py: per-row relative L-inf within
     max(BASE[impl], 4 x the fp32 oracle's error)).  Shuffled TSP graphs with an independent t per edge, or t constant
     over runs of 64 sorted rows (changing at sorted rows 63/64 and 127/128); unsorted MIS with a t per node.
  b. Bitwise, through the hook: an all-zero index is dfb_debug_gnn_layer at values[0]; an out-of-range index makes
     exactly its own row NaN (e for TSP, h for MIS) and leaves every other value as the run with index 0 there.
  c. The public forward against the fp64 oracle (_check_vs_oracle of test_gpu_timesteps.py): shuffled TSP-50 batches,
     at least 3 tiles per CTA, irregular graphs, mean / max, dense per-sample t, a ragged node_ptr batch.
  d. 4096 distinct timesteps, the NaN row that grows the table, and the loop captured before and after on one
     context."""
import numpy as np
import pytest
import torch

from difusco_b200 import _cabi, synthetic as syn
from oracle import difusco_oracle as orc
import gpu_util as G
import test_gpu_layer_parity as LP
from test_gpu_timesteps import _check_vs_oracle

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = torch.device("cuda")
IMPLS = ["tc", "tc1", "fp32"]
N_LAYERS = 12
MID = 5
INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1
MAX_T = 4096


def _stream():
  return torch.cuda.current_stream().cuda_stream


def _sorted_perm(ei):
  """perm[s] = the caller's edge at row-sorted position s (dfb_prepare_graph's stable sort of edge_index[0])."""
  return np.argsort(ei[0], kind="stable")


# ------------------------------------------------------------------------------------------------
# timestep patterns: t per element in the caller's order -> (values, index)
# ------------------------------------------------------------------------------------------------
BLOCK = 64                                                   # one consumer warpgroup's rows; 2 blocks = one tile
BLOCK_T = np.array([3.0, 997.0, 120.0, 610.0, 45.0, 830.0], np.float32)   # consecutive entries differ


def t_pattern(case, task, pattern):
  """t (N,) fp32 in the caller's order: "edge" an independent integer t per caller edge, "block" t constant over runs
  of BLOCK row-sorted edges, "node" an integer t per node (MIS)."""
  V, ei, *_ = LP._case(case)
  rng = np.random.default_rng(sum(map(ord, case + pattern)))
  if pattern == "node":
    return rng.integers(1, 1001, V).astype(np.float32)
  E = ei.shape[1]
  if pattern == "edge":
    return rng.integers(1, 1001, E).astype(np.float32)
  t = np.empty(E, np.float32)
  t[_sorted_perm(ei)] = BLOCK_T[(np.arange(E) // BLOCK) % BLOCK_T.size]
  return t


def values_index(t):
  values, index = np.unique(np.asarray(t, np.float32), return_inverse=True)
  return values, index.astype(np.int32)


def max_t_values():
  """MAX_T distinct, non-integer timesteps in (1, 1000), distinct in fp32."""
  return (1.0 + 998.0 * (np.arange(MAX_T) + 0.5) / MAX_T).astype(np.float32)


# ------------------------------------------------------------------------------------------------
# a. teacher-forced layers with per-row tau
# ------------------------------------------------------------------------------------------------
SHUF_TSP = ["tsp_shuf", "hub_shuf", "degseq_shuf", "isolated_shuf", "dup_shuf"] + \
           [f"tiny{E}_shuf" for E in G.TINY]
TF_CASES = [(c, "tsp", p) for c in SHUF_TSP for p in ("edge", "block")] + [("mis", "mis", "node")]
AGG_CASES = {"tsp_shuf", "hub_shuf", "mis"}
TF_PARAMS = [(c, t, p, a, i) for c, t, p in TF_CASES for a in LP.AGGS if a == "sum" or c in AGG_CASES
             for i in IMPLS]


@pytest.mark.parametrize("case,task,pattern,agg,impl", TF_PARAMS)
def test_teacher_forced_layer_per_row_t_vs_fp64_oracle(weights2, case, task, pattern, agg, impl):
  V, ei, *_ = LP._case(case)
  t = t_pattern(case, task, pattern)
  values, index = values_index(t)
  ctx = LP._engine(weights2, task)
  layers = LP._teacher_forced(weights2, case, task, agg, t, t_key=pattern)
  for l, (h32, e32, r64, r32) in enumerate(layers):
    got_h, got_e = LP._run_layer(ctx, ei, V, l, h32, e32, impl, agg, values, index)
    LP._check_layer(got_h, got_e, h32, e32, r64, r32, task, l, N_LAYERS, impl,
                    f"{case} {pattern} {agg} {impl} layer {l}")


# ------------------------------------------------------------------------------------------------
# b. bitwise identities through the hook
# ------------------------------------------------------------------------------------------------
BIT_CASES = [(c, "tsp") for c in SHUF_TSP] + [("mis", "mis")]
BAD = [MAX_T, -1, INT32_MIN, INT32_MAX]   # MAX_T stands for n_t: replaced by the call's n_t


def _state(case, task):
  """A seeded fp32 state (h, e) entering a layer, caller's edge order."""
  V, ei, *_ = LP._case(case)
  rng = np.random.default_rng(sum(map(ord, case)) + 7)
  return rng.standard_normal((V, 256)).astype(np.float32), rng.standard_normal((ei.shape[1], 256)).astype(np.float32)


def nan_rows(case, task):
  """The elements given an out-of-range index: the first row, sorted rows 63, 64, 127, 128 and the last row (TSP:
  through the permutation to caller edges; MIS: those nodes)."""
  V, ei, *_ = LP._case(case)
  n = V if task == "mis" else ei.shape[1]
  pos = sorted({s for s in (0, 63, 64, 127, 128, n - 1) if s < n})
  return np.array(pos if task == "mis" else _sorted_perm(ei)[pos], np.int64)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("case,task", BIT_CASES)
def test_zero_index_is_bitwise_the_one_timestep_hook(weights2, case, task, impl):
  V, ei, *_ = LP._case(case)
  ctx = LP._engine(weights2, task)
  h, e = _state(case, task)
  zeros = np.zeros(V if task == "mis" else ei.shape[1], np.int32)
  for layer in (0, MID, N_LAYERS - 1):
    ref = LP._run_layer(ctx, ei, V, layer, h, e, impl, "sum", 412.0)
    got = LP._run_layer(ctx, ei, V, layer, h, e, impl, "sum", [412.0, 7.0, 999.0], zeros)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1]), (case, layer)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("case,task", BIT_CASES)
def test_out_of_range_index_is_nan_in_its_own_row_only(weights2, case, task, impl):
  """tau reaches, within one layer, only its own row: TSP e after the messages, MIS h of the node."""
  V, ei, *_ = LP._case(case)
  ctx = LP._engine(weights2, task)
  h, e = _state(case, task)
  t = t_pattern(case, task, "node" if task == "mis" else "edge")
  values, index = values_index(t)
  rows = nan_rows(case, task)
  base = index.copy()
  base[rows] = 0
  bad = base.copy()
  bad[rows] = [values.size if b == MAX_T else b for b in np.resize(BAD, rows.size)]
  for layer in (0, MID):
    ref_h, ref_e = LP._run_layer(ctx, ei, V, layer, h, e, impl, "sum", values, base)
    got_h, got_e = LP._run_layer(ctx, ei, V, layer, h, e, impl, "sum", values, bad)
    got, ref, other = (got_h, ref_h, (got_e, ref_e)) if task == "mis" else (got_e, ref_e, (got_h, ref_h))
    hit = np.zeros(got.shape[0], bool)
    hit[rows] = True
    what = f"{case} {impl} layer {layer}"
    assert np.isnan(got[hit]).all(), f"{what}: rows {rows} not NaN in every column"
    assert np.isfinite(ref).all() and np.array_equal(got[~hit], ref[~hit]), f"{what}: the NaN left its row"
    assert np.array_equal(other[0], other[1]), f"{what}: the NaN reached {'e' if task == 'mis' else 'h'}"


@pytest.mark.parametrize("impl", IMPLS)
def test_index_of_4096_grows_the_table_by_its_nan_row(weights2, impl):
  """On a fresh context, the first call with n_t = 4096 and an index is the one that grows tvec to 4097 rows."""
  case = "tsp_shuf"
  V, ei, *_ = LP._case(case)
  w = {k: v.copy() for k, v in weights2.items()}   # a new key: its own fresh context
  ctx = LP._engine(w, "tsp")
  h, e = _state(case, "tsp")
  values = max_t_values()
  index = (np.arange(ei.shape[1]) % MAX_T).astype(np.int32)
  rows = nan_rows(case, "tsp")
  bad = index.copy()
  bad[rows] = MAX_T
  got_h, got_e = LP._run_layer(ctx, ei, V, MID, h, e, impl, "sum", values, bad)
  index[rows] = 0
  ref_h, ref_e = LP._run_layer(ctx, ei, V, MID, h, e, impl, "sum", values, index)
  hit = np.zeros(ei.shape[1], bool)
  hit[rows] = True
  assert np.isnan(got_e[hit]).all() and np.array_equal(got_e[~hit], ref_e[~hit]) and np.array_equal(got_h, ref_h)
  LP._engines.pop((id(w), "tsp", N_LAYERS))


def test_hook_rejects_what_the_forward_rejects(weights2):
  V, ei, *_ = LP._case("tiny33_shuf")
  ctx = LP._engine(weights2, "tsp")
  eid = G.cu(ei)
  st = _stream()
  ctx.prepare_graph(eid.data_ptr(), V, ei.shape[1], 1, st)
  h0, e0 = _state("tiny33_shuf", "tsp")
  h, e = G.cu(h0), G.cu(e0)
  idx = torch.zeros(ei.shape[1], dtype=torch.int32, device=DEV)
  host_idx = np.zeros(ei.shape[1], np.int32)
  host_h = np.zeros((V, 256), np.float32)
  L = _cabi.lib()
  fp = lambda a: np.ascontiguousarray(a, np.float32).ctypes.data_as(_cabi.C.POINTER(_cabi.C.c_float))
  one, big = np.array([5.0], np.float32), np.ones(MAX_T + 1, np.float32)
  cases = [(MID, 1, None, idx.data_ptr(), h.data_ptr(), e.data_ptr(), _cabi.DFB_E_INVALID),
           (MID, 0, one, idx.data_ptr(), h.data_ptr(), e.data_ptr(), _cabi.DFB_E_INVALID),
           (MID, -1, one, idx.data_ptr(), h.data_ptr(), e.data_ptr(), _cabi.DFB_E_INVALID),
           (MID, MAX_T + 1, big, idx.data_ptr(), h.data_ptr(), e.data_ptr(), _cabi.DFB_E_UNSUPPORTED),
           (MID, 1, one, host_idx.ctypes.data, h.data_ptr(), e.data_ptr(), _cabi.DFB_E_INVALID),
           (-1, 1, one, idx.data_ptr(), h.data_ptr(), e.data_ptr(), _cabi.DFB_E_INVALID),
           (N_LAYERS, 1, one, idx.data_ptr(), h.data_ptr(), e.data_ptr(), _cabi.DFB_E_INVALID),
           (MID, 1, one, idx.data_ptr(), host_h.ctypes.data, e.data_ptr(), _cabi.DFB_E_INVALID),
           (MID, 1, one, idx.data_ptr(), h.data_ptr(), host_h.ctypes.data, _cabi.DFB_E_INVALID)]
  torch.cuda.synchronize()
  n0 = ctx.launch_count()
  for layer, n_t, tv, ti, hp, ep, code in cases:
    rc = L.dfb_debug_gnn_layer_timesteps(ctx._h, layer, n_t, None if tv is None else fp(tv), ti, hp, ep, st)
    assert rc == code, (layer, n_t, rc)
  assert ctx.launch_count() == n0
  torch.cuda.synchronize()
  assert np.array_equal(h.cpu().numpy(), h0) and np.array_equal(e.cpu().numpy(), e0)
  with pytest.raises(ValueError):
    ctx.debug_gnn_layer_timesteps(N_LAYERS, [5.0], idx.data_ptr(), h.data_ptr(), e.data_ptr(), st)


# ------------------------------------------------------------------------------------------------
# c. the public forward against the fp64 oracle
# ------------------------------------------------------------------------------------------------
def _shuffle(ei, seed):
  """-> (shuffled edge_index, q): caller edge j of the shuffled graph is edge q[j] of ei."""
  q = np.random.default_rng(seed).permutation(ei.shape[1])
  return np.ascontiguousarray(ei[:, q]), q


def _unshuffle(out, q):
  r = np.empty_like(out)
  r[q] = out
  return r


def _tsp_forward(w, impl, pts, t, xt, ei, agg="sum", node_ptr=None):
  enc = G.encoder(w, w["out.2.bias"].shape[0], impl=impl, aggregation=agg)
  kw = {} if node_ptr is None else {"node_ptr": torch.from_numpy(node_ptr)}
  return enc(G.cu(pts), G.cu(t), G.cu(xt), G.cu(ei), **kw).cpu().numpy()


def _tsp_oracle(w, pts, xt, t, ei, agg="sum"):
  return lambda dt: orc.encoder_forward_sparse_tsp(orc.Weights(w, dt), pts, xt, t, ei, agg)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("diffusion", ["categorical", "gaussian"])
def test_tsp50_batch_shuffled_per_graph_t_vs_fp64_oracle(weights1, weights2, diffusion, impl):
  w = weights2 if diffusion == "categorical" else weights1
  pts, ei = syn.tsp_sparse_batch(50, 20, 8, seed=110)
  xt = syn.initial_noise(ei.shape[1], 111)
  if diffusion == "categorical":
    xt = (xt > 0).astype(np.float32)
  t = np.repeat([1.0, 999.0, 250.0, 500.0, 17.0, 760.0, 1000.0, 333.0], 50 * 20).astype(np.float32)
  eis, q = _shuffle(ei, 112)
  out = _unshuffle(_tsp_forward(w, impl, pts, t[q], xt[q], eis), q)
  _check_vs_oracle(out, f"edges/tsp50x8/{diffusion}", _tsp_oracle(w, pts, xt, t, ei), impl)


def _multi_tile_case():
  """TSP-200 k = 20 with enough graphs for 3 tiles of 128 rows per CTA of the persistent grid."""
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  B = -(-3 * 128 * sms // (200 * 20)) + 1
  pts, ei = syn.tsp_sparse_batch(200, 20, B, seed=120)
  assert ei.shape[1] >= 3 * 128 * sms
  return B, pts, ei, syn.initial_noise(ei.shape[1], 121) * np.float32(1.02)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("order", ["sorted", "shuffled"])
@pytest.mark.parametrize("tk", ["graph", "edge"])
def test_multi_tile_per_cta_vs_fp64_oracle(weights2, tk, order, impl):
  B, pts, ei, xt = _multi_tile_case()
  rng = np.random.default_rng(122)
  t = (np.repeat(rng.integers(1, 1001, B), 200 * 20) if tk == "graph" else rng.integers(1, 1001, ei.shape[1]))
  t = t.astype(np.float32)
  if order == "sorted":
    out = _tsp_forward(weights2, impl, pts, t, xt, ei)
  else:   # the oracle is invariant to edge order (test_timesteps_cpu.py): one oracle run serves both
    eis, q = _shuffle(ei, 123)
    out = _unshuffle(_tsp_forward(weights2, impl, pts, t[q], xt[q], eis), q)
  _check_vs_oracle(out, f"edges/multitile/{tk}", _tsp_oracle(weights2, pts, xt, t, ei), impl)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("graph", ["hub", "isolated", "degseq"])
def test_irregular_shuffled_per_edge_t_vs_fp64_oracle(weights2, graph, impl):
  case = graph + "_shuf"
  V, ei, pts, xe, _ = LP._case(case)
  t = t_pattern(case, "tsp", "edge")
  out = _tsp_forward(weights2, impl, pts, t, xe, ei)
  _check_vs_oracle(out, f"edges/{case}", _tsp_oracle(weights2, pts, xe, t, ei), impl)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("agg", ["mean", "max"])
@pytest.mark.parametrize("task", ["tsp", "mis"])
def test_mean_max_per_graph_t_vs_fp64_oracle(weights2, task, agg, impl):
  if task == "tsp":
    pts, ei = syn.tsp_sparse_batch(50, 20, 4, seed=130)
    xt = (syn.initial_noise(ei.shape[1], 131) > 0).astype(np.float32)
    t = np.repeat([5.0, 400.0, 1000.0, 77.0], 50 * 20).astype(np.float32)
    eis, q = _shuffle(ei, 132)
    out = _unshuffle(_tsp_forward(weights2, impl, pts, t[q], xt[q], eis, agg), q)
    fwd = _tsp_oracle(weights2, pts, xt, t, ei, agg)
  else:
    ei, sizes = syn.mis_batch(100, 150, 0.05, 3, seed=133)
    xt = (syn.initial_noise(sum(sizes), 134) > 0).astype(np.float32)
    t = np.repeat([900.0, 12.0, 455.0], sizes).astype(np.float32)
    enc = G.encoder(weights2, 2, node_only=True, impl=impl, aggregation=agg)
    out = enc(G.cu(xt), G.cu(t), edge_index=G.cu(ei)).cpu().numpy()
    fwd = lambda dt: orc.encoder_forward_mis(orc.Weights(weights2, dt), xt, t, ei, agg)
  _check_vs_oracle(out, f"edges/{task}/{agg}", fwd, impl)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("diffusion", ["categorical", "gaussian"])
def test_dense_per_sample_t_b16_vs_fp64_oracle(weights1, weights2, diffusion, impl):
  w = weights2 if diffusion == "categorical" else weights1
  B, V = 16, 50
  pts = np.stack([syn.tsp_points(V, 140, b) for b in range(B)]).astype(np.float32)
  xt = syn.initial_noise(B * V * V, 141).reshape(B, V, V)
  if diffusion == "categorical":
    xt = (xt > 0).astype(np.float32)
  t = np.random.default_rng(142).integers(1, 1001, B).astype(np.float32)
  enc = G.encoder(w, w["out.2.bias"].shape[0], sparse=False, impl=impl)
  out = enc(G.cu(pts), torch.from_numpy(t), G.cu(xt)).cpu().numpy()
  _check_vs_oracle(out, f"edges/dense16/{diffusion}",
                   lambda dt: orc.encoder_forward_dense(orc.Weights(w, dt), pts, xt, t), impl)


RAGGED = [(1, 1), (7, 7), (50, 20), (200, 20)]   # (nodes, k) per instance


@pytest.mark.parametrize("impl", IMPLS)
def test_ragged_instances_shuffled_per_graph_t_vs_fp64_oracle_alone(weights2, impl):
  parts = [(syn.tsp_points(n, 150, i), None) for i, (n, _) in enumerate(RAGGED)]
  parts = [(p, syn.knn_edge_index(p, k)) for (p, _), (_, k) in zip(parts, RAGGED)]
  off = syn.node_ptr([n for n, _ in RAGGED])
  pts = np.concatenate([p for p, _ in parts]).astype(np.float32)
  ei = np.concatenate([e + off[i] for i, (_, e) in enumerate(parts)], 1)
  E = [n * k for n, k in RAGGED]
  ts = [640.0, 3.0, 1000.0, 271.0]
  t = np.repeat(ts, E).astype(np.float32)
  xt = (syn.initial_noise(ei.shape[1], 151) > 0).astype(np.float32)
  eis, q = _shuffle(ei, 152)
  out = _unshuffle(_tsp_forward(weights2, impl, pts, t[q], xt[q], eis, node_ptr=off), q)
  e0 = 0
  for i, ((p, e), ti) in enumerate(zip(parts, ts)):
    x = xt[e0:e0 + E[i]]
    _check_vs_oracle(out[e0:e0 + E[i]], f"edges/ragged/{i}", _tsp_oracle(weights2, p, x, np.array([ti]), e), impl)
    e0 += E[i]


# ------------------------------------------------------------------------------------------------
# d. the 4096-entry table and the state it shares with the loop
# ------------------------------------------------------------------------------------------------
def _max_t_case():
  """A shuffled TSP-50 k = 20 x 5 graph (5000 edges) on which each of the 4096 timesteps is used."""
  pts, ei = syn.tsp_sparse_batch(50, 20, 5, seed=160)
  eis, q = _shuffle(ei, 161)
  index = (np.random.default_rng(162).permutation(eis.shape[1]) % MAX_T).astype(np.int32)
  xt = (syn.initial_noise(eis.shape[1], 163) > 0).astype(np.float32)
  return pts, eis, xt, index


@pytest.mark.parametrize("impl", IMPLS)
def test_4096_distinct_timesteps_vs_fp64_oracle(weights2, impl):
  pts, ei, xt, index = _max_t_case()
  values = max_t_values()
  t = values[index]
  enc = G.encoder(weights2, 2, impl=impl)
  ctx = enc.set_graph(G.cu(ei), pts.shape[0])
  enc.set_points(G.cu(pts))
  xd, idx, out = G.cu(xt), G.cu(index), torch.empty((ei.shape[1], 2), device=DEV)
  ctx.encoder_forward_timesteps(xd.data_ptr(), values, idx.data_ptr(), out.data_ptr(), _stream())
  _check_vs_oracle(out.cpu().numpy(), "edges/t4096", _tsp_oracle(weights2, pts, xt, t, ei), impl)


LOOP_STEPS = 50


class _Loop(object):
  """A captured categorical dfb_denoise and per-element forwards on one context (TSP, shuffled edges)."""

  def __init__(self, w):
    self.pts, self.ei, self.xt, self.index = _max_t_case()
    self.E = self.ei.shape[1]
    self.ctx = LP._raw_context(w, N_LAYERS)
    st = _stream()
    self.eid, self.pd = G.cu(self.ei), G.cu(self.pts)
    self.ctx.prepare_graph(self.eid.data_ptr(), self.pts.shape[0], self.E, 1, st)
    self.ctx.set_points(self.pd.data_ptr(), st)
    sched = orc.inference_schedule("cosine", 1000, LOOP_STEPS)
    _, Q_bar = orc.categorical_tables(1000, "linear")
    self.t1 = [t1 for t1, _ in sched]
    self.cs = [orc.categorical_posterior_consts(Q_bar, t1, t2).reshape(-1) for t1, t2 in sched]
    self.ls = [int(t2 == 0) for _, t2 in sched]
    self.u = G.cu(np.stack([syn.uniforms(self.E, 170, i) for i in range(LOOP_STEPS)]))   # one pointer: the loop key
    self.xd = G.cu(self.xt)

  def loop(self):
    y = G.cu(self.xt)
    self.ctx.denoise(_cabi.CATEGORICAL, y.data_ptr(), self.t1, self.cs, self.ls, self.u.data_ptr(), 0, _stream())
    torch.cuda.synchronize()
    return y.cpu().numpy()

  def forward(self, values):
    """dfb_encoder_forward_timesteps with edge j at values[index[j] % len(values)]."""
    idx = G.cu(self.index % np.int32(len(values)))
    out = torch.empty((self.E, 2), device=DEV)
    self.ctx.encoder_forward_timesteps(self.xd.data_ptr(), values, idx.data_ptr(), out.data_ptr(), _stream())
    torch.cuda.synchronize()
    return out.cpu().numpy()

  def step(self):
    yo = torch.empty(self.E, device=DEV)
    self.ctx.denoise_step(_cabi.CATEGORICAL, self.xd.data_ptr(), float(self.t1[0]), self.cs[0], self.ls[0],
                          self.u.data_ptr(), 0, 0, yo.data_ptr(), None, None, _stream())
    torch.cuda.synchronize()


def test_4096_table_and_the_captured_loop_share_one_context():
  """tvec grows under a captured loop: the loop re-captures once, computes the same state, and is not re-captured by
  a forward that fits the grown table."""
  run = _Loop(syn.make_encoder_weights(171, out_channels=2))
  values = max_t_values()
  first = run.loop()
  c0 = run.ctx.loop_captures()
  assert c0 >= 1
  f1 = run.forward(values)
  assert np.isfinite(f1).all()
  assert np.array_equal(run.loop(), first)
  assert run.ctx.loop_captures() == c0 + 1, "tvec grew: the loop must be re-captured exactly once"
  f2 = run.forward(values)
  assert np.array_equal(f2, f1)
  assert np.array_equal(run.loop(), first)
  assert run.ctx.loop_captures() == c0 + 1, "a forward that fits the table must not force a re-capture"
  run.ctx.close()


def test_per_element_forward_unchanged_by_a_loop_and_a_step():
  run = _Loop(syn.make_encoder_weights(172, out_channels=2))
  values = np.random.default_rng(173).integers(1, 1001, MAX_T).astype(np.float32)
  before = [run.forward(values[:n]) for n in (MAX_T, 7)]
  run.loop()
  run.step()
  after = [run.forward(values[:n]) for n in (MAX_T, 7)]
  assert all(np.array_equal(a, b) for a, b in zip(before, after))
  run.ctx.close()

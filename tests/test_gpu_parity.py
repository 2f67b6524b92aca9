"""Parity of the CUDA path (through the C-ABI) against the committed reference outputs
(tests/golden) and against the CPU oracle on fresh seeded inputs.  Run with -m gpu on an H100."""
import numpy as np
import pytest
import torch

from conftest import golden, rel_linf
from difusco_b200 import _cabi, synthetic as syn
from oracle import difusco_oracle as orc
import gpu_util as G

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------
# building block: split-bf16 GEMM on wgmma (descriptors, TMA, mbarrier plumbing)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", ["tc", "tc1"])
@pytest.mark.parametrize("E", [128, 1000, 128 * 150 + 17, 128 * 301])
def test_tc_gemm_matches_fp64_matmul(weights2, E, impl):
  enc = G.encoder(weights2, 2, impl=impl)
  V = 64
  rng = np.random.default_rng(E)
  ei = np.stack([np.sort(rng.integers(0, V, E)), rng.integers(0, V, E)]).astype(np.int64)
  ctx = enc.set_graph(G.cu(ei), V, 1)
  x = (rng.standard_normal((E, 256)) * 3).astype(np.float32)
  xin = G.cu(x)
  acc = torch.full((E, 256), float("nan"), device="cuda")
  for layer in (0, 7):
    ctx.debug_edge_gemm(layer, xin.data_ptr(), acc.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ref = x.astype(np.float64) @ weights2[f"layers.{layer}.C.weight"].astype(np.float64).T
    got = acc.cpu().numpy()
    assert np.isfinite(got).all()
    # error model: 2 * 2^-17 relative per product, sqrt(K) accumulation
    assert rel_linf(got, ref) < 2e-5, (layer, rel_linf(got, ref))


# ------------------------------------------------------------------------------------------------
# forward parity against outputs of the reference itself (golden fixtures)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", ["fp32", "tc"])
def test_forward_tsp_categorical_golden(weights2, impl):
  g = golden("fwd_tsp_cat")
  enc = G.encoder(weights2, 2, impl=impl)
  out = enc(G.cu(g["points"]), G.cu(g["t"]), G.cu(g["xt"]), G.cu(g["edge_index"]))
  assert out.shape == g["logits"].shape
  assert rel_linf(out.cpu().numpy(), g["logits"]) < G.TOL[impl]
  # softmax probabilities (what the posterior consumes): relative 1e-4 contract
  p = torch.softmax(out, -1).cpu().numpy()
  pr = torch.softmax(torch.from_numpy(g["logits"]), -1).numpy()
  assert np.abs(p / pr - 1).max() < G.TOL[impl]


@pytest.mark.parametrize("impl", ["fp32", "tc"])
def test_forward_tsp_gaussian_golden(weights1, impl):
  g = golden("fwd_tsp_gauss")
  enc = G.encoder(weights1, 1, impl=impl)
  out = enc(G.cu(g["points"]), G.cu(g["t"]), G.cu(g["xt"]), G.cu(g["edge_index"]))
  assert rel_linf(out.cpu().numpy(), g["pred"]) < G.TOL[impl]


@pytest.mark.parametrize("impl", ["fp32", "tc"])
@pytest.mark.parametrize("agg", ["sum", "mean", "max"])
def test_forward_mis_golden(weights2, impl, agg):
  g = golden("fwd_mis_cat")
  ref = g["logits"] if agg == "sum" else golden(f"fwd_mis_cat_{agg}")["logits"]
  enc = G.encoder(weights2, 2, node_only=True, impl=impl, aggregation=agg)
  out = enc(G.cu(g["xt"]), G.cu(g["t"]), edge_index=G.cu(g["edge_index"]))   # unsorted edge list
  assert rel_linf(out.cpu().numpy(), ref) < G.TOL[impl]


@pytest.mark.parametrize("impl", ["fp32", "tc"])
def test_forward_dense_golden(weights2, impl):
  g = golden("fwd_dense_cat")    # B=2 with a different timestep per sample
  enc = G.encoder(weights2, 2, sparse=False, impl=impl)
  out = enc(G.cu(g["points"]), G.cu(g["t"]), G.cu(g["xt"]), None)
  assert out.shape == g["out"].shape
  assert rel_linf(out.cpu().numpy(), g["out"]) < G.TOL[impl]
  # same timestep for both samples exercises the batched (gn_segments = B) path
  w = orc.Weights(weights2)
  t_same = np.array([444.0, 444.0], np.float32)
  ref = orc.encoder_forward_dense(w, g["points"], g["xt"], t_same).numpy()
  out = enc(G.cu(g["points"]), G.cu(t_same), G.cu(g["xt"]), None)
  assert rel_linf(out.cpu().numpy(), ref) < G.TOL[impl]


def test_dense_node_only_raises(weights2):
  enc = G.encoder(weights2, 2, node_only=True, sparse=False)
  with pytest.raises(NotImplementedError):
    enc(torch.zeros(4, device="cuda"), torch.tensor([1.0]), edge_index=None)


# ------------------------------------------------------------------------------------------------
# teacher-forced trajectories (SURVEY section 7 H2): every step gets the reference's own xt_in; compare the
# network output, the pre-sampling probability p and the final heatmap; sampled states may only
# differ where |p - u| is inside fp32 noise.
# ------------------------------------------------------------------------------------------------
def _traj(model, task, g, useed, impl, diffusion):
  V, K, P, steps = [int(x) for x in g["meta"]]
  dev = torch.device("cuda")
  ei = G.cu(g["edge_index"]) if "edge_index" in g.files else None
  sched = orc.inference_schedule(model.args.inference_schedule, 1000, steps)
  tol = G.TOL[impl]
  xt_in = g["xt0"].astype(np.float32).reshape(-1)
  n = xt_in.size
  if task == "tsp":
    pts = G.cu(np.tile(g["points"], (P, 1)))
    model._prepare(pts, ei, dev)
  else:
    model.model.set_graph(ei, n, 1)
  ctx = model.model.engine()
  mode = _cabi.CATEGORICAL if diffusion == "categorical" else _cabi.GAUSSIAN
  out_ch = 2 if diffusion == "categorical" else 1
  for i, (t1, t2) in enumerate(sched):
    consts, last = model.posterior_consts(t1, t2)
    x = G.cu(xt_in)
    u = G.cu(syn.uniforms(n, useed, i))
    xo = torch.empty(n, device=dev)
    p = torch.empty(n, device=dev)
    net = torch.empty((n, out_ch), device=dev)
    ctx.denoise_step(mode, x.data_ptr(), float(t1), consts, last, u.data_ptr(), 0, i, xo.data_ptr(),
                     p.data_ptr(), net.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ref_net = g["net_out"][i].reshape(n, out_ch)
    assert rel_linf(net.cpu().numpy(), ref_net) < tol, (i, rel_linf(net.cpu().numpy(), ref_net))
    ref_next = g["xt_out"][i].reshape(-1)
    if diffusion == "categorical":
      if i < steps - 1:
        pc = p.cpu().numpy().clip(0, 1)
        assert np.abs(pc - g["p"][i]).max() < tol
        flips = xo.cpu().numpy() != ref_next
        near = np.abs(g["p"][i] - syn.uniforms(n, useed, i)) < 10 * tol
        assert not np.any(flips & ~near)
      else:
        hm, ref = xo.cpu().numpy(), ref_next
        assert np.abs(hm - ref).max() < tol * max(ref.max(), 1e-3)
        big = ref > 1e-3
        assert np.abs(hm[big] / ref[big] - 1).max() < 10 * tol
    else:
      assert rel_linf(xo.cpu().numpy(), ref_next) < tol
    xt_in = ref_next.astype(np.float32)


@pytest.mark.parametrize("impl", ["fp32", "tc"])
def test_traj_tsp_categorical_golden(weights2, impl):
  g = golden("traj_tsp_cat")
  m = G.tsp_model(weights2, impl, sparse_factor=6, parallel_sampling=2, inference_diffusion_steps=10)
  _traj(m, "tsp", g, 100, impl, "categorical")


@pytest.mark.parametrize("impl", ["fp32", "tc"])
def test_traj_tsp_gaussian_golden(weights1, impl):
  g = golden("traj_tsp_gauss")
  m = G.tsp_model(weights1, impl, diffusion_type="gaussian", sparse_factor=8, inference_diffusion_steps=6)
  _traj(m, "tsp", g, 101, impl, "gaussian")


@pytest.mark.parametrize("impl", ["fp32", "tc"])
def test_traj_mis_categorical_golden(weights2, impl):
  g = golden("traj_mis_cat")
  m = G.mis_model(weights2, impl, parallel_sampling=2, inference_diffusion_steps=8)
  _traj(m, "mis", g, 102, impl, "categorical")


@pytest.mark.parametrize("impl", ["fp32", "tc"])
def test_traj_mis_gaussian_golden(weights1, impl):
  g = golden("traj_mis_gauss")
  m = G.mis_model(weights1, impl, diffusion_type="gaussian", inference_diffusion_steps=5,
                  inference_schedule="linear")
  _traj(m, "mis", g, 103, impl, "gaussian")


@pytest.mark.parametrize("impl", ["fp32", "tc"])
def test_traj_dense_categorical_golden(weights2, impl):
  """Reference dense trajectory (config C1 family) through TSPModel.categorical_denoise_step."""
  g = golden("traj_dense_cat")
  V, _, _, steps = [int(x) for x in g["meta"]]
  m = G.tsp_model(weights2, impl, sparse_factor=-1, inference_diffusion_steps=steps)
  dev = torch.device("cuda")
  pts = G.cu(g["points"])[None]
  sched = orc.inference_schedule("cosine", 1000, steps)
  xt = G.cu(g["xt0"].astype(np.float32))
  t1, t2 = sched[-1]
  # last step is deterministic given xt_in: feed the reference's xt_in of the last step
  xt_in = G.cu(g["xt_out"][steps - 2].astype(np.float32))
  out = m.categorical_denoise_step(pts, xt_in, np.array([t1]), dev, None, target_t=np.array([t2]))
  assert out.shape == (1, V, V)
  ref = g["xt_out"][-1]
  assert np.abs(out.cpu().numpy() - ref).max() < G.TOL[impl] * max(ref.max(), 1e-3)
  # an intermediate step returns a {0,1} sample of the right shape
  t1, t2 = sched[0]
  o0 = m.categorical_denoise_step(pts, xt, np.array([t1]), dev, None, target_t=np.array([t2]))
  assert o0.shape == (1, V, V) and set(np.unique(o0.cpu().numpy())) <= {0.0, 1.0}


# ------------------------------------------------------------------------------------------------
# fresh seeded inputs against the oracle, at sizes the oracle finishes in seconds
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", ["fp32", "tc"])
@pytest.mark.parametrize("N,K,B", [(100, 20, 3), (37, 5, 1), (200, 50, 2)])
def test_forward_tsp_vs_oracle(weights2, impl, N, K, B):
  pts, ei = syn.tsp_sparse_batch(N, K, B, seed=N)
  xt = (syn.initial_noise(ei.shape[1], N) > 0).astype(np.float32)
  ref = orc.encoder_forward_sparse_tsp(orc.Weights(weights2), pts, xt, np.array([873.0]), ei).numpy()
  enc = G.encoder(weights2, 2, impl=impl)
  out = enc(G.cu(pts), torch.tensor([873.0]), G.cu(xt), G.cu(ei))
  assert rel_linf(out.cpu().numpy(), ref) < G.TOL[impl]


def test_forward_tsp500_full_size_vs_oracle(weights2):
  """BASELINE config 2 shape (TSP-500, k=50), 4 instances in one call, full forward vs the CPU oracle."""
  pts, ei = syn.tsp_sparse_batch(500, 50, 4, seed=1234)
  xt = (syn.initial_noise(ei.shape[1], 0) > 0).astype(np.float32)
  ref = orc.encoder_forward_sparse_tsp(orc.Weights(weights2), pts, xt, np.array([1000.0]), ei,
                                       gather_then_gemm=False).numpy()
  enc = G.encoder(weights2, 2, impl="tc")
  out = enc(G.cu(pts), torch.tensor([1000.0]), G.cu(xt), G.cu(ei))
  err = rel_linf(out.cpu().numpy(), ref)
  p = torch.softmax(out, -1).cpu().numpy()
  pr = torch.softmax(torch.from_numpy(ref), -1).numpy()
  assert err < 1e-4 and np.abs(p / pr - 1).max() < 1e-4, (err, np.abs(p / pr - 1).max())


@pytest.mark.parametrize("impl", ["fp32", "tc"])
def test_forward_mis_vs_oracle(weights2, impl):
  ei, sizes = syn.mis_batch(90, 120, 0.15, 3, seed=11)
  V = sum(sizes)
  xt = (syn.initial_noise(V, 4) > 0).astype(np.float32)
  ref = orc.encoder_forward_mis(orc.Weights(weights2), xt, np.array([640.0]), ei).numpy()
  enc = G.encoder(weights2, 2, node_only=True, impl=impl)
  out = enc(G.cu(xt), torch.tensor([640.0]), edge_index=G.cu(ei))
  assert rel_linf(out.cpu().numpy(), ref) < G.TOL[impl]
  # edge order must not matter: a random permutation of the edge list gives the same node outputs
  perm = np.random.default_rng(0).permutation(ei.shape[1])
  out2 = enc(G.cu(xt), torch.tensor([640.0]), edge_index=G.cu(ei[:, perm]))
  assert rel_linf(out2.cpu().numpy(), ref) < G.TOL[impl]


def test_tsp_unsorted_edge_list_keeps_caller_order(weights2):
  """Edge-valued I/O stays in the caller's edge order even when the list is not row sorted."""
  pts, ei = syn.tsp_sparse_batch(40, 8, 1, seed=3)
  xt = (syn.initial_noise(ei.shape[1], 5) > 0).astype(np.float32)
  enc = G.encoder(weights2, 2, impl="tc")
  base = enc(G.cu(pts), torch.tensor([300.0]), G.cu(xt), G.cu(ei)).cpu().numpy()
  perm = np.random.default_rng(1).permutation(ei.shape[1])
  out = enc(G.cu(pts), torch.tensor([300.0]), G.cu(xt[perm]), G.cu(ei[:, perm])).cpu().numpy()
  assert rel_linf(out, base[perm]) < 1e-5


# ------------------------------------------------------------------------------------------------
# the fused loop: determinism, seeding, host-buffer entry point
# ------------------------------------------------------------------------------------------------
def test_fused_loop_deterministic_and_seeded(weights2):
  m = G.tsp_model(weights2, "tc", sparse_factor=10, inference_diffusion_steps=12)
  pts, ei = syn.tsp_sparse_batch(60, 10, 2, seed=9)
  xt0 = (syn.initial_noise(ei.shape[1], 2) > 0).astype(np.float32)
  a = m.denoise_heatmap(G.cu(pts), G.cu(ei), G.cu(xt0), seed=77).cpu().numpy()
  b = m.denoise_heatmap(G.cu(pts), G.cu(ei), G.cu(xt0), seed=77).cpu().numpy()
  c = m.denoise_heatmap(G.cu(pts), G.cu(ei), G.cu(xt0), seed=78).cpu().numpy()
  assert np.array_equal(a, b), "same seed must be bitwise reproducible (no atomics on the path)"
  assert not np.array_equal(a, c)
  assert a.min() >= 0.0 and a.max() <= 1.0 + 1e-5 and np.isfinite(a).all()
  # the free-running heatmap is a valid probability field close to the oracle's in distribution:
  # run the oracle free with its own draws and compare the mean edge probability
  w = orc.Weights(weights2)
  ref = orc.denoise(w, "tsp", "categorical", ei, xt0, points=pts, steps=12).numpy()
  assert abs(a.mean() - ref.mean()) < 0.05


def test_denoise_host_entry_matches_device_entry(weights2):
  m = G.tsp_model(weights2, "tc", sparse_factor=10, inference_diffusion_steps=6)
  pts, ei = syn.tsp_sparse_batch(50, 10, 2, seed=21)
  xt0 = (syn.initial_noise(ei.shape[1], 8) > 0).astype(np.float32)
  dev = m.denoise_heatmap(G.cu(pts), G.cu(ei), G.cu(xt0), seed=5).cpu().numpy()
  sched = orc.inference_schedule("cosine", 1000, 6)
  t1s, cs, ls = [], [], []
  for t1, t2 in sched:
    c, last = m.posterior_consts(t1, t2)
    t1s.append(t1); cs.append(c); ls.append(last)
  ctx = m.model.engine()
  hm = np.empty(ei.shape[1], np.float32)
  pts_c, ei_c = np.ascontiguousarray(pts), np.ascontiguousarray(ei)
  ctx.denoise_host(_cabi.CATEGORICAL, pts_c.ctypes.data, ei_c.ctypes.data, pts.shape[0], ei.shape[1], 1,
                   xt0.ctypes.data, t1s, cs, ls, 5, hm.ctypes.data, 0)
  assert np.array_equal(hm, dev)


def test_error_paths(weights2):
  enc = G.encoder(weights2, 2)
  ctx = enc.engine()
  bad = torch.tensor([[0, 1, 99], [1, 0, 2]], dtype=torch.long, device="cuda")
  with pytest.raises(ValueError, match="out of range"):
    ctx.prepare_graph(bad.data_ptr(), 3, 3, 1, 0)
  with pytest.raises(ValueError):
    ctx.set_aggregation("median")
  with pytest.raises(NotImplementedError):
    enc(torch.zeros(4, 2, device="cuda"), torch.tensor([1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0]),
        torch.zeros(8, device="cuda"), torch.zeros(2, 8, dtype=torch.long, device="cuda"))


# ------------------------------------------------------------------------------------------------
# BASELINE.json configs at (or near) full size, one instance each, against the oracle
# ------------------------------------------------------------------------------------------------
def test_config3_tsp1000_k100_gaussian_vs_oracle(weights1):
  """configs[2]: TSP-1000 sparse k=100, Gaussian diffusion (continuous xt -> general edge embedding)."""
  pts, ei = syn.tsp_sparse_batch(1000, 100, 1, seed=31)
  xt = syn.initial_noise(ei.shape[1], 6)
  w = orc.Weights(weights1)
  ref = orc.encoder_forward_sparse_tsp(w, pts, xt, np.array([777.0]), ei, gather_then_gemm=False).numpy()
  m = G.tsp_model(weights1, "tc", diffusion_type="gaussian", sparse_factor=100, inference_diffusion_steps=50)
  out = m.model(G.cu(pts), torch.tensor([777.0]), G.cu(xt), G.cu(ei))
  assert rel_linf(out.cpu().numpy(), ref) < 1e-4
  # one fused DDIM step through the reference-signature method
  nxt = m.gaussian_denoise_step(G.cu(pts), G.cu(xt), np.array([777]), torch.device("cuda"), G.cu(ei),
                                target_t=np.array([740]))
  beta, alpha, ab = orc.gaussian_tables(1000, "linear")
  ref_next = orc.gaussian_posterior(beta, alpha, ab, 777, 740, torch.from_numpy(ref).squeeze(1), torch.from_numpy(xt))
  assert rel_linf(nxt.cpu().numpy(), ref_next.numpy()) < 1e-4


def test_config4_mis_er750_vs_oracle(weights2):
  """configs[3]: MIS on an ER-[700,800] p=0.15 graph (unsorted edge list, ~85k directed+self edges)."""
  ei, sizes = syn.mis_batch(700, 800, 0.15, 1, seed=41)
  V = sum(sizes)
  xt = (syn.initial_noise(V, 7) > 0).astype(np.float32)
  ref = orc.encoder_forward_mis(orc.Weights(weights2), xt, np.array([905.0]), ei, gather_then_gemm=False).numpy()
  enc = G.encoder(weights2, 2, node_only=True, impl="tc")
  out = enc(G.cu(xt), torch.tensor([905.0]), edge_index=G.cu(ei))
  assert rel_linf(out.cpu().numpy(), ref) < 1e-4
  # batch of 4 graphs: runs, finite, and graph 0's outputs differ from the single-graph call only through the
  # shared head GroupNorm (SURVEY D4) - i.e. they are NOT bitwise equal but stay close
  ei4, sizes4 = syn.mis_batch(700, 800, 0.15, 4, seed=41)
  V4 = sum(sizes4)
  xt4 = np.concatenate([xt, (syn.initial_noise(V4 - V, 8) > 0).astype(np.float32)])
  out4 = enc(G.cu(xt4), torch.tensor([905.0]), edge_index=G.cu(ei4)).cpu().numpy()
  assert np.isfinite(out4).all() and out4.shape == (V4, 2)


def test_config5_tsp2000_parallel_sampling_vs_oracle(weights2):
  """configs[4] family (TSP-10000 k=50, 4x parallel sampling) at a size the oracle finishes in seconds:
  TSP-2000 k=50 with parallel_sampling = 2 through duplicate_edge_index."""
  m = G.tsp_model(weights2, "tc", sparse_factor=50, parallel_sampling=2, inference_diffusion_steps=50)
  pts = syn.tsp_points(2000, 55, 0)
  ei1 = torch.from_numpy(syn.knn_edge_index(pts, 50))
  ei = m.duplicate_edge_index(ei1, 2000, torch.device("cpu")).numpy()
  pts2 = np.tile(pts, (2, 1))
  xt = (syn.initial_noise(ei.shape[1], 9) > 0).astype(np.float32)
  ref = orc.encoder_forward_sparse_tsp(orc.Weights(weights2), pts2, xt, np.array([31.0]), ei,
                                       gather_then_gemm=False).numpy()
  out = m.model(G.cu(pts2), torch.tensor([31.0]), G.cu(xt), G.cu(ei))
  assert rel_linf(out.cpu().numpy(), ref) < 1e-4


def test_config5_tsp10000_full_size_properties(weights2):
  """configs[4] at full size (TSP-10000, k=50, P=4: V=40000, E=2M): too big for the CPU oracle, so check
  size-independent properties: finite probabilities in [0,1], bitwise determinism, and replica symmetry
  (all P replicas get identical xt -> identical heatmaps, since replicas only couple through shared statistics)."""
  m = G.tsp_model(weights2, "tc", sparse_factor=50, parallel_sampling=4, inference_diffusion_steps=3)
  pts = syn.tsp_points(10000, 77, 0)
  ei1 = torch.from_numpy(syn.knn_edge_index(pts, 50))
  ei = m.duplicate_edge_index(ei1, 10000, torch.device("cpu"))
  pts4 = torch.from_numpy(np.tile(pts, (4, 1)))
  x1 = (syn.initial_noise(ei1.shape[1], 10) > 0).astype(np.float32)
  xt = torch.from_numpy(np.tile(x1, 4))
  # last-step (deterministic) heatmap from identical replicas
  c, last = m.posterior_consts(31, 0)
  dev = torch.device("cuda")
  a = m.categorical_denoise_step(pts4.cuda(), xt.cuda(), np.array([31]), dev, ei.cuda(), target_t=np.array([0]))
  b = m.categorical_denoise_step(pts4.cuda(), xt.cuda(), np.array([31]), dev, ei.cuda(), target_t=np.array([0]))
  a, b = a.cpu().numpy(), b.cpu().numpy()
  assert np.array_equal(a, b)
  assert np.isfinite(a).all() and a.min() >= 0 and a.max() <= 1 + 1e-5
  reps = a.reshape(4, -1)
  for p in range(1, 4):
    assert np.abs(reps[p] - reps[0]).max() < 1e-5


def test_repeated_runs_bitwise_identical(weights2):
  """Race detector: the path has no atomics and a fixed summation structure, so repeated forwards over multi-tile
  graphs (persistent CTAs looping over tiles, MIS last layer without GEMM2, TSP with the TMA store path) must be
  bitwise identical.  A synchronisation bug between the tile phases shows up here as run-to-run noise."""
  ei, sizes = syn.mis_batch(700, 800, 0.15, 2, seed=43)
  V = sum(sizes)
  xt = (syn.initial_noise(V, 12) > 0).astype(np.float32)
  enc = G.encoder(weights2, 2, node_only=True, impl="tc")
  first = enc(G.cu(xt), torch.tensor([100.0]), edge_index=G.cu(ei)).cpu().numpy()
  for _ in range(6):
    again = enc(G.cu(xt), torch.tensor([100.0]), edge_index=G.cu(ei)).cpu().numpy()
    assert np.array_equal(first, again)
  pts, eit = syn.tsp_sparse_batch(500, 50, 8, seed=77)
  xte = (syn.initial_noise(eit.shape[1], 13) > 0).astype(np.float32)
  enc2 = G.encoder(weights2, 2, impl="tc")
  a = enc2(G.cu(pts), torch.tensor([640.0]), G.cu(xte), G.cu(eit)).cpu().numpy()
  for _ in range(6):
    b = enc2(G.cu(pts), torch.tensor([640.0]), G.cu(xte), G.cu(eit)).cpu().numpy()
    assert np.array_equal(a, b)


def test_mis_test_step_end_to_end(weights2):
  """MISModel.test_step with the reference's batch tuple: denoise loop on the GPU + greedy decode; returns the
  reference's metrics dict and yields a valid independent set for every parallel sample."""
  from types import SimpleNamespace as NS
  from difusco_b200.utils.mis_utils import mis_decode_np
  import scipy.sparse
  m = G.mis_model(weights2, "tc", parallel_sampling=2, inference_diffusion_steps=5)
  ei = syn.er_graph_edge_index(120, 0.1, seed=8, instance=0)
  labels = torch.zeros(120, dtype=torch.long, device="cuda")
  graph = NS(x=labels, edge_index=torch.from_numpy(ei).cuda())
  batch = (torch.tensor([0]), graph, torch.tensor([120], device="cuda"))
  torch.manual_seed(0)
  metrics = m.test_step(batch, 0)
  assert set(metrics) == {"test/gt_cost"} and metrics["test/gt_cost"] == 0
  pl = m.last_predict_labels
  assert pl.shape == (240,) and np.isfinite(pl).all()
  adj = scipy.sparse.coo_matrix((np.ones_like(ei[0]), (ei[0], ei[1]))).tocsr()
  best = 0
  for part in np.split(pl, 2):
    sol = mis_decode_np(part, adj)
    sel = np.flatnonzero(sol)
    for i in sel:
      nb = adj.indices[adj.indptr[i]:adj.indptr[i + 1]]
      assert not np.any(sol[nb[nb != i]])
    best = max(best, int(sol.sum()))
  assert best == m.last_solved_cost and best > 0

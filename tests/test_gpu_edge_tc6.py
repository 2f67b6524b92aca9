"""DFB_EDGE_IMPL_TC6 (GNNEncoder(edge_precision="bf16x6")): the tensor-core edge layer with three bf16 parts per
operand, held to the full 1e-4 heat-map contract where bf16x3 (`tc`, `tc1`) is xfail: confident heads (R1, R6), the R6
teacher-forced run, dense R1 and offset e rows.  The cases, oracles and bounds are those of test_gpu_value_ranges.py and
test_gpu_layer_parity.py, imported from there; only the implementation differs.  The few cases TC6 still misses are
strict xfails with their measured numbers (_TC6_MISSES and the marks below).  Then the other entry points under TC6:
the golden fixtures, a timestep per element, the captured loop against its steps and a batch against its instances
alone."""
import numpy as np
import pytest
import torch

from conftest import golden, rel_linf
from difusco_b200 import _cabi, synthetic as syn
from difusco_b200.models.gnn_encoder import GNNEncoder
from difusco_b200.pl_tsp_model import TSPModel
from oracle import difusco_oracle as orc
import gpu_util as G
import test_gpu_layer_parity as LP
import test_gpu_parity as GP
import test_gpu_solve_batch as SB
import test_gpu_value_ranges as VR

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

TOL_TC6 = 1e-4   # logits rel-L-inf, as for tc (the bounds below take max(this, 4 x the fp32 oracle's error))


def encoder(weights, out_channels, node_only=False, sparse=True, aggregation="sum"):
  enc = G.encoder(weights, out_channels, node_only=node_only, sparse=sparse, aggregation=aggregation)
  enc.engine().set_edge_impl(_cabi.EDGE_IMPL_TC6)
  return enc


def tsp_model(weights, **kw):
  m = G.tsp_model(weights, "tc", **kw)
  m.model.engine().set_edge_impl(_cabi.EDGE_IMPL_TC6)
  return m


def mis_model(weights, **kw):
  m = G.mis_model(weights, "tc", **kw)
  m.model.engine().set_edge_impl(_cabi.EDGE_IMPL_TC6)
  return m


def _tsp_model_with(weights, **kw):
  """A TSPModel whose args carry kw (edge_precision reaches GNNEncoder through COMetaModel)."""
  m = TSPModel(G.args(sparse_factor=20, **kw))
  G.load(m.model, weights)
  return m.cuda()


def _check(out, ref64, ref32, what=""):
  """test_gpu_value_ranges._check with the TC6 logits tolerance."""
  assert out.shape == ref64.shape and np.isfinite(out).all(), what
  got, yard = VR._errors(out, ref64), VR._errors(ref32, ref64)
  base = {"logits": TOL_TC6, "p_abs": VR.TOL, "p_rel": VR.TOL}
  bound = {k: max(base[k], 4 * v) for k, v in yard.items()}
  bad = [k for k in got if not got[k] <= bound[k]]
  assert not bad, f"{what} failing {bad}: kernel {got} | fp32 oracle {yard} | bounds {bound}"


def _stream():
  return torch.cuda.current_stream().cuda_stream


# Cases TC6 still misses, measured on an H100 80GB HBM3 at 700 W (DESIGN section 5).  Its logits' relative error is
# 1.0-1.1e-5 in R1 and R6, against 2-5e-5 for bf16x3 and 3-4e-6 for the fp32 oracle; the CPU emulation of its operand
# rounding predicts the oracle's.  Strict, so the test reports when the loss goes away.
def _xfail_tc6(reason):
  return pytest.mark.xfail(strict=True, reason="TC6: " + reason)


_TC6_MISSES = {
    ("R1", "mis", 500.0): "R1 ER-200 t=500: max |p - p64| 1.047e-4 against 1e-4 (logits 1.06e-5, fp32 oracle 4.1e-6)",
}


# ------------------------------------------------------------------------------------------------
# a. the public option selects TC6; the default stays bf16x3
# ------------------------------------------------------------------------------------------------
def test_edge_precision_option_selects_tc6(weights2):
  pts, ei, xt = VR._case_inputs("tsp")
  args = (G.cu(pts), torch.tensor([500.0]), G.cu(xt), G.cu(ei))
  outs = {}
  for prec in ("bf16x3", "bf16x6"):
    outs[prec] = G.load(GNNEncoder(12, 256, 2, sparse=True, edge_precision=prec), weights2)(*args).cpu().numpy()
  outs["tc"] = G.encoder(weights2, 2)(*args).cpu().numpy()
  outs["tc6"] = encoder(weights2, 2)(*args).cpu().numpy()
  m = _tsp_model_with(weights2, edge_precision="bf16x6")
  outs["model"] = m.model(*args).cpu().numpy()
  assert np.array_equal(outs["bf16x3"], outs["tc"])
  assert np.array_equal(outs["bf16x6"], outs["tc6"]) and np.array_equal(outs["model"], outs["tc6"])


# ------------------------------------------------------------------------------------------------
# b. the value-range matrix of test_gpu_value_ranges.py, every case passing
# ------------------------------------------------------------------------------------------------
def _gpu_forward(w, case, t):
  if case == "mis":
    ei, xt = VR._case_inputs(case)
    enc = encoder(w, 2, node_only=True)
    return enc(G.cu(xt), torch.tensor([t]), edge_index=G.cu(ei)).cpu().numpy()
  pts, ei, xt = VR._case_inputs(case)
  enc = encoder(w, w["out.2.bias"].shape[0])
  return enc(G.cu(pts), torch.tensor([t]), G.cu(xt), G.cu(ei)).cpu().numpy()


@pytest.mark.parametrize("regime,case,t", [
    pytest.param(r, c, t, marks=[_xfail_tc6(_TC6_MISSES[r, c, t])] if (r, c, t) in _TC6_MISSES else [])
    for r in G.REGIMES for c in ("tsp", "mis") for t in VR.TS])
def test_categorical_forward_in_regime_vs_fp64_oracle(regime, case, t):
  r64, r32, _ = VR._oracle(regime, case, t)
  _check(_gpu_forward(VR._regime(regime, case), case, t), r64, r32, f"{regime} {case} t={t} tc6")


@pytest.mark.parametrize("regime,t", [(r, t) for r in VR.GAUSS_REGIMES for t in VR.TS])
def test_gaussian_forward_in_regime_vs_fp64_oracle(regime, t):
  r64, r32, _ = VR._oracle(regime, "tsp_gauss", t)
  _check(_gpu_forward(VR._regime(regime, "tsp_gauss"), "tsp_gauss", t), r64, r32, f"{regime} tsp_gauss t={t} tc6")


@pytest.mark.parametrize("regime", ["R0", pytest.param("R1", marks=_xfail_tc6(
    "R1 dense: heat map of sample 0, max rel 1.9e-4 (dense50) / 2.0e-4 (dense100) against 1e-4; logits and max "
    "|p - p64| (4.8e-5 / 4.0e-5) pass"))])
@pytest.mark.parametrize("case", list(VR.DENSE))
def test_dense_multi_segment_vs_oracle_per_sample(regime, case):
  """test_gpu_value_ranges' dense case under TC6: forward logits per sample, then the heat map of one
  categorical_denoise_step (t = 500 -> 0) per sample against the fp64 oracle's."""
  V, B = VR.DENSE[case]
  pts, xt = VR._case_inputs(case)
  w = VR._regime(regime, case)
  r64, r32, _ = VR._oracle(regime, case, VR.T_CAL)
  m = tsp_model(w, sparse_factor=-1)
  out = m.model(G.cu(pts), torch.tensor([VR.T_CAL]), G.cu(xt), None).cpu().numpy()
  assert out.shape == (B, 2, V, V)
  out = out.transpose(0, 2, 3, 1).reshape(B, V * V, 2)
  for b in range(B):
    _check(out[b], r64[b], r32[b], f"{regime} {case} sample {b}")
  hm = m.categorical_denoise_step(G.cu(pts), G.cu(xt), np.array([int(VR.T_CAL)]), torch.device("cuda"), None,
                                  target_t=np.array([0])).cpu().numpy().reshape(B, -1)
  _, Q_bar = orc.categorical_tables(1000, "linear")
  for b in range(B):
    xb = torch.as_tensor(xt[b].reshape(-1))
    bound, e32 = VR._posterior_bound(r32[b], r64[b], xb, Q_bar, int(VR.T_CAL), 0)
    _, ref = orc.categorical_posterior(Q_bar, int(VR.T_CAL), 0, torch.as_tensor(VR._softmax(r64[b])), xb)
    ref = ref.numpy()
    big = ref > VR.P_BIG
    err, rel = float(np.abs(hm[b] - ref).max()), float(np.abs(hm[b][big] / ref[big] - 1).max())
    assert err <= bound and rel <= bound, (b, err, rel, e32, bound)


_tf = {}


def _r6_teacher_forced():
  """test_gpu_value_ranges._r6_teacher_forced under TC6."""
  if "tc6" not in _tf:
    rec = VR._r6_oracle_trajectory()
    pts, ei, _ = VR._case_inputs("tsp")
    n = ei.shape[1]
    m = tsp_model(VR._regime("R6", "tsp"), sparse_factor=20, inference_diffusion_steps=VR.STEPS_TF)
    dev = torch.device("cuda")
    m._prepare(G.cu(pts), G.cu(ei), dev)
    ctx = m.model.engine()
    out = []
    for i, r in enumerate(rec):
      consts, last = m.posterior_consts(r["t1"], r["t2"])
      x, u = G.cu(r["xt_in"].numpy().astype(np.float32)), G.cu(r["u"])
      xo, p, net = torch.empty(n, device=dev), torch.empty(n, device=dev), torch.empty((n, 2), device=dev)
      ctx.denoise_step(_cabi.CATEGORICAL, x.data_ptr(), float(r["t1"]), consts, last, u.data_ptr(), 0, i,
                       xo.data_ptr(), p.data_ptr(), net.data_ptr(), _stream())
      torch.cuda.synchronize()
      out.append(dict(net=net.cpu().numpy(), p=p.cpu().numpy().astype(np.float64), xo=xo.cpu().numpy(), last=last))
    _tf["tc6"] = out
  return _tf["tc6"]


@_xfail_tc6("R6 teacher-forced: network output of step 23, max rel p 2.63e-4 against 2.62e-4 (4 x the fp32 oracle's "
            "6.5e-5); logits 1.05e-5")
def test_r6_teacher_forced_50_steps_precision_vs_fp64_oracle():
  """Network output and p of every step within the bounds; the final heat map within the p bound, absolute and
  relative where it is >= 1e-3 (test_gpu_value_ranges, where tc is xfail)."""
  for i, (s, r) in enumerate(zip(_r6_teacher_forced(), VR._r6_oracle_trajectory())):
    _check(s["net"], r["net_out"].numpy(), r["r32"], f"step {i}")
    pk, pr = s["p"], r["p"].numpy()
    if not s["last"]:
      err = float(np.abs(pk.clip(0, 1) - pr.clip(0, 1)).max())
      assert err <= r["bound"], (i, err, r["e32"], r["bound"])
    else:
      hm, ref = s["xo"], r["xt_out"].numpy()
      big = ref > VR.P_BIG
      err, rel = float(np.abs(hm - ref).max()), float(np.abs(hm[big] / ref[big] - 1).max())
      assert err <= r["bound"] and rel <= r["bound"], (err, rel, r["e32"], r["bound"])


def test_r6_teacher_forced_samples_differ_only_near_ties():
  flips_total = 0
  for i, (s, r) in enumerate(zip(_r6_teacher_forced()[:-1], VR._r6_oracle_trajectory()[:-1])):
    pk, pr = s["p"].clip(0, 1), r["p"].numpy().clip(0, 1)
    flips = s["xo"] != r["xt_out"].numpy()
    allowed = (np.abs(pr - r["u"]) <= np.abs(pk - pr)) & (np.abs(pr - r["u"]) < VR.FLIP_BAND)
    assert not np.any(flips & ~allowed), (i, int(flips.sum()), int((flips & ~allowed).sum()))
    flips_total += int(flips.sum())
  assert flips_total <= 50, flips_total


# ------------------------------------------------------------------------------------------------
# c. one layer at a time (test_gpu_layer_parity.py), held to the tensor-core bound BASE["tc"]
# ------------------------------------------------------------------------------------------------
def _run_layer(ctx, ei, V, layer, h, e, agg):
  """test_gpu_layer_parity._run_layer under TC6."""
  ctx.set_edge_impl(_cabi.EDGE_IMPL_TC6)
  ctx.set_aggregation(agg)
  eid = G.cu(ei)
  ctx.prepare_graph(eid.data_ptr(), V, ei.shape[1], 1, _stream())
  perm = np.argsort(ei[0], kind="stable")
  hd, ed = G.cu(np.asarray(h, np.float32)), G.cu(np.asarray(e, np.float32)[perm])
  ctx.debug_gnn_layer(layer, LP.T_LAYER, hd.data_ptr(), ed.data_ptr(), _stream())
  torch.cuda.synchronize()
  e_out = np.empty_like(ed.cpu().numpy())
  e_out[perm] = ed.cpu().numpy()
  return hd.cpu().numpy(), e_out


@pytest.mark.parametrize("name", LP.EDGE_CASES)
def test_one_layer_value_edges_vs_fp64_oracle(name):
  """offset_e is xfail for tc and tc1 (h rel 2.1e-4 against 1.05e-4); TC6 must pass it with the rest."""
  w, task, case, agg, h, e = LP._edge_case(name)
  r64, r32 = LP._refs(w, task, case, LP.MID, h, e, agg)
  V, ei, *_ = LP._case(case)
  got_h, got_e = _run_layer(LP._engine(w, task), ei, V, LP.MID, h, e, agg)
  LP._check_layer(got_h, got_e, h, e, r64, r32, task, LP.MID, LP.N_LAYERS, "tc", f"{name} tc6")


@pytest.mark.parametrize("case,task", [("tsp_shuf", "tsp"), ("mis", "mis"), ("degseq", "tsp"), ("hub", "mis"),
                                       ("tiny33", "tsp"), ("V129", "mis")])
def test_teacher_forced_layer_vs_fp64_oracle(weights2, case, task):
  V, ei, *_ = LP._case(case)
  ctx = LP._engine(weights2, task)
  for l, (h32, e32, r64, r32) in enumerate(LP._teacher_forced(weights2, case, task, "sum")):
    got_h, got_e = _run_layer(ctx, ei, V, l, h32, e32, "sum")
    LP._check_layer(got_h, got_e, h32, e32, r64, r32, task, l, LP.N_LAYERS, "tc", f"{case} {task} tc6 layer {l}")


@pytest.mark.parametrize("E", [64, 1000, 64 * 301 + 17])
def test_gemm_hook_matches_fp64_matmul(weights2, E):
  """dfb_debug_edge_gemm under TC6 (64-row tiles): both operands are exact in three bf16 parts, so only the dropped
  third-order products (~2^-24) and fp32 accumulation remain."""
  enc = encoder(weights2, 2)
  V = 64
  rng = np.random.default_rng(E)
  ei = np.stack([np.sort(rng.integers(0, V, E)), rng.integers(0, V, E)]).astype(np.int64)
  ctx = enc.set_graph(G.cu(ei), V, 1)
  x = (rng.standard_normal((E, 256)) * 3).astype(np.float32)
  xin = G.cu(x)
  acc = torch.full((E, 256), float("nan"), device="cuda")
  for layer in (0, 7):
    ctx.debug_edge_gemm(layer, xin.data_ptr(), acc.data_ptr(), _stream())
    torch.cuda.synchronize()
    ref = x.astype(np.float64) @ weights2[f"layers.{layer}.C.weight"].astype(np.float64).T
    got = acc.cpu().numpy()
    assert np.isfinite(got).all()
    assert rel_linf(got, ref) < 4e-6, (layer, rel_linf(got, ref))


# ------------------------------------------------------------------------------------------------
# d. golden fixtures (outputs of the reference itself)
# ------------------------------------------------------------------------------------------------
def test_forward_tsp_categorical_golden(weights2):
  g = golden("fwd_tsp_cat")
  out = encoder(weights2, 2)(G.cu(g["points"]), G.cu(g["t"]), G.cu(g["xt"]), G.cu(g["edge_index"]))
  assert rel_linf(out.cpu().numpy(), g["logits"]) < TOL_TC6
  p = torch.softmax(out, -1).cpu().numpy()
  pr = torch.softmax(torch.from_numpy(g["logits"]), -1).numpy()
  assert np.abs(p / pr - 1).max() < TOL_TC6


def test_forward_tsp_gaussian_golden(weights1):
  g = golden("fwd_tsp_gauss")
  out = encoder(weights1, 1)(G.cu(g["points"]), G.cu(g["t"]), G.cu(g["xt"]), G.cu(g["edge_index"]))
  assert rel_linf(out.cpu().numpy(), g["pred"]) < TOL_TC6


@pytest.mark.parametrize("agg", ["sum", "mean", "max"])
def test_forward_mis_golden(weights2, agg):
  g = golden("fwd_mis_cat")
  ref = g["logits"] if agg == "sum" else golden(f"fwd_mis_cat_{agg}")["logits"]
  enc = encoder(weights2, 2, node_only=True, aggregation=agg)
  out = enc(G.cu(g["xt"]), G.cu(g["t"]), edge_index=G.cu(g["edge_index"]))
  assert rel_linf(out.cpu().numpy(), ref) < TOL_TC6


def test_forward_dense_golden(weights2):
  g = golden("fwd_dense_cat")
  out = encoder(weights2, 2, sparse=False)(G.cu(g["points"]), G.cu(g["t"]), G.cu(g["xt"]), None)
  assert out.shape == g["out"].shape
  assert rel_linf(out.cpu().numpy(), g["out"]) < TOL_TC6


@pytest.mark.parametrize("name", ["tsp_cat", "mis_cat", "tsp_gauss", "mis_gauss", "dense_cat"])
def test_traj_golden(weights1, weights2, name):
  """test_gpu_parity's teacher-forced golden trajectories (dense: its last step) under TC6."""
  g = golden(f"traj_{name}")
  w = weights1 if "gauss" in name else weights2
  gauss = dict(diffusion_type="gaussian")
  if name == "tsp_cat":
    m = tsp_model(w, sparse_factor=6, parallel_sampling=2, inference_diffusion_steps=10)
  elif name == "tsp_gauss":
    m = tsp_model(w, sparse_factor=8, inference_diffusion_steps=6, **gauss)
  elif name == "mis_cat":
    m = mis_model(w, parallel_sampling=2, inference_diffusion_steps=8)
  elif name == "mis_gauss":
    m = mis_model(w, inference_diffusion_steps=5, inference_schedule="linear", **gauss)
  else:
    V, _, _, steps = [int(x) for x in g["meta"]]
    m = tsp_model(w, sparse_factor=-1, inference_diffusion_steps=steps)
    t1, t2 = orc.inference_schedule("cosine", 1000, steps)[-1]
    xt_in = G.cu(g["xt_out"][steps - 2].astype(np.float32))
    out = m.categorical_denoise_step(G.cu(g["points"])[None], xt_in, np.array([t1]), torch.device("cuda"), None,
                                     target_t=np.array([t2])).cpu().numpy()
    ref = g["xt_out"][-1]
    assert out.shape == (1, V, V) and np.abs(out - ref).max() < TOL_TC6 * max(ref.max(), 1e-3)
    return
  # _traj reads its tolerance from G.TOL[impl]; "tc" is TC6's (TOL_TC6)
  GP._traj(m, name[:3], g, {"tsp_cat": 100, "tsp_gauss": 101, "mis_cat": 102, "mis_gauss": 103}[name], "tc",
           "gaussian" if "gauss" in name else "categorical")


# ------------------------------------------------------------------------------------------------
# e. the other entry points under TC6
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tsp_edge_t", "mis_cat", "dense_gauss"])
def test_timestep_per_element_golden(weights1, weights2, name):
  """dfb_encoder_forward_timesteps (per-edge t: k_edge_layer_tc6_trows) against the reference's training-step
  forwards."""
  g = golden("fwd_tsteps")
  a = lambda k: G.cu(g[f"{name}/{k}"])
  w = weights1 if "gauss" in name else weights2
  oc = w["out.2.bias"].shape[0]
  if name.startswith("tsp"):
    out = encoder(w, oc)(a("points"), a("t"), a("xt"), a("edge_index"))
  elif name == "dense_gauss":
    out = encoder(w, oc, sparse=False)(a("points"), a("t"), a("xt"))
  else:
    out = encoder(w, oc, node_only=True)(a("xt"), a("t"), edge_index=a("edge_index"))
  out, ref = out.cpu().numpy(), g[f"{name}/out"]
  assert out.shape == ref.shape and np.isfinite(out).all()
  assert rel_linf(out, ref) < TOL_TC6, rel_linf(out, ref)


@pytest.mark.parametrize("task", ["tsp", "mis"])
def test_denoise_loop_is_bitwise_its_steps(weights2, task):
  """dfb_denoise, captured after a captured bf16x3 loop on the same context (the switch re-captures) and with plain
  launches, equals a loop of dfb_denoise_step under TC6, bitwise, with injected uniforms."""
  steps = 6
  if task == "tsp":
    pts, ei = syn.tsp_sparse_batch(100, 20, 2, seed=91)
    m = G.tsp_model(weights2, "tc", sparse_factor=20, inference_diffusion_steps=steps)
    m._prepare(G.cu(pts), G.cu(ei), torch.device("cuda"))
    n = ei.shape[1]
  else:
    ei = syn.er_graph_edge_index(300, 0.05, seed=92)
    n = 300
    m = G.mis_model(weights2, "tc", inference_diffusion_steps=steps)
    m.model.set_graph(G.cu(ei), n, 1)
  xt = (syn.initial_noise(n, 93) > 0).astype(np.float32)
  ctx = m.model.engine()
  sched = orc.inference_schedule("cosine", 1000, steps)
  t1s, cs, ls = [], [], []
  for t1, t2 in sched:
    c, last = m.posterior_consts(t1, t2)
    t1s.append(int(t1)); cs.append(c); ls.append(last)
  us = [syn.uniforms(n, 94, i) for i in range(steps)]
  ud = G.cu(np.stack(us))

  def loop():
    x = G.cu(xt)
    ctx.denoise(_cabi.CATEGORICAL, x.data_ptr(), t1s, cs, ls, ud.data_ptr(), 0, _stream())
    torch.cuda.synchronize()
    return x.cpu().numpy()

  loop()   # bf16x3, captured
  captures = ctx.loop_captures()
  ctx.set_edge_impl(_cabi.EDGE_IMPL_TC6)
  captured = loop()
  assert ctx.loop_captures() == captures + 1
  ctx.set_graph_capture(False)
  plain = loop()
  ctx.set_graph_capture(True)
  y = G.cu(xt)
  for i in range(steps):
    yo = torch.empty_like(y)
    ctx.denoise_step(_cabi.CATEGORICAL, y.data_ptr(), float(t1s[i]), cs[i], ls[i], G.cu(us[i]).data_ptr(), 0, i,
                     yo.data_ptr(), None, None, _stream())
    y = yo
  torch.cuda.synchronize()
  assert np.array_equal(captured, plain) and np.array_equal(captured, y.cpu().numpy())


def test_aligned_tsp_batch_is_bitwise_each_instance_alone(weights2):
  """test_gpu_solve_batch's aligned batch under TC6: each instance of a dfb_denoise_instances batch equals its run
  alone, bitwise."""
  steps = 8
  parts = [(syn.tsp_points(n, 71, i), None) for i, n in enumerate([64, 100, 64])]
  parts = [(p, syn.knn_edge_index(p, k)) for (p, _), k in zip(parts, [16, 32, 16])]
  assert all(e.shape[1] % 32 == 0 for _, e in parts)
  m = tsp_model(weights2, sparse_factor=16, inference_diffusion_steps=steps)
  order = [2, 0, 1, 0]
  alone, got = SB._alone_and_batched_tsp(m, parts, [5, 6, 7], order, steps)
  for j, i in enumerate(order):
    assert np.array_equal(got[j], alone[i]), (order, j)

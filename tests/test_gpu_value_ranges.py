"""The encoder and the denoise step at the value ranges of a trained model, against the fp64 oracle.

Every other parity test runs the synthetic weights, whose logits stay below 1 in magnitude, so every softmax
probability lies in about [0.2, 0.8].  A trained DIFUSCO checkpoint is confident (p near 0 or 1), its head GroupNorm
input need not be centred, and the reference's own init zeroes the per-layer output linears.  The regimes of
gpu_util.regime put the kernels there, each calibrated on the fp64 oracle at t = 500 on the graph it runs on:

  R0 control; R1 confident head (max |l1 - l0| = 24, >= 30 % of rows with min(p0, p1) < 1e-3); R1x logits of ~100;
  R2 per_layer_out.*.2 = 0; R3 U, V, A, B, C and per_layer_out.*.2 weights x 3; R4_r head input with per-group
  |mean| / std = r for r = 10, 100, 1000; R5 norm gains log-uniform in [0.05, 5] (some at 1e-3), biases N(0, 1);
  R6 = R3 + R4_10 + R1.  The Gaussian (one-channel) encoder runs R0, R1 (max |x0| = 24) and R4.

Metrics, each against the fp64 oracle:
  * logits: rel-Linf < G.TOL[impl] (1e-4 for the wgmma kernels, 2e-5 for the fp32 validation kernel);
  * softmax probabilities: max |p - p64| <= 1e-4 (the heat-map contract: p lies in [0, 1]), and max |p / p64 - 1|
    <= 1e-4 where p64 >= 1e-3;
  * yardstick: each bound is max(the bound above, 4 x the fp32 oracle's own error on that metric).  The kernels are
    held to the reference's fp32 path, not to fp64: fp32 arithmetic in another order may lose what the fp32 oracle
    loses, a few times over, and no more.
Every assertion message prints the kernel's errors and the fp32 oracle's errors."""
import numpy as np
import pytest
import torch

from conftest import rel_linf
from difusco_b200 import _cabi, synthetic as syn
from oracle import difusco_oracle as orc
import gpu_util as G

TOL = 1e-4
P_BIG = 1e-3
T_CAL = 500.0
TS = [1.0, 500.0, 999.0]
IMPLS = ["tc", "tc1", "fp32"]
GAUSS_REGIMES = ["R0", "R1", "R4_10", "R4_100", "R4_1000"]
DENSE = {"dense50": (50, 4), "dense100": (100, 3)}      # V, B: 2 500 and 10 000 rows per GroupNorm segment
torch.set_grad_enabled(False)


# ------------------------------------------------------------------------------------------------
# cases: graphs and inputs, deterministic from fixed seeds
# ------------------------------------------------------------------------------------------------
_inputs = {}


def _case_inputs(case):
  """tsp / tsp_gauss: (pts, edge_index, xt) TSP-200, K = 20, B = 2.  mis: (edge_index, xt) ER-200.
  dense*: (pts (B,V,2), xt (B,V,V)) with sample 0 all zeros, sample 1 all ones and the rest random."""
  if case not in _inputs:
    if case in ("tsp", "tsp_gauss"):
      pts, ei = syn.tsp_sparse_batch(200, 20, 2, seed=71)
      xt = syn.initial_noise(ei.shape[1], 72)
      _inputs[case] = (pts, ei, xt if case == "tsp_gauss" else (xt > 0).astype(np.float32))
    elif case == "mis":
      _inputs[case] = (syn.er_graph_edge_index(200, 0.05, seed=73), (syn.initial_noise(200, 74) > 0).astype(np.float32))
    else:
      V, B = DENSE[case]
      pts = np.stack([syn.tsp_points(V, 75, b) for b in range(B)]).astype(np.float32)
      xt = np.zeros((B, V, V), np.float32)
      xt[1] = 1
      for b in range(2, B):
        xt[b] = (syn.initial_noise(V * V, 76 + b) > 0).reshape(V, V)
      _inputs[case] = (pts, xt)
  return _inputs[case]


def _base(case):
  return syn.make_encoder_weights(1, out_channels=1) if case == "tsp_gauss" else syn.make_encoder_weights(0, out_channels=2)


def _oracle_forward(w, case, t, dtype=torch.float64):
  """-> (logits, head input): sparse cases (rows, out) in the caller's order; dense cases (B, V*V, out), no head
  input.  Dense samples run one at a time: the reference's GroupNorm is per sample."""
  W = orc.Weights(w, dtype=dtype)
  tt = np.array([t])
  if case in ("tsp", "tsp_gauss"):
    pts, ei, xt = _case_inputs(case)
    taps = []
    out = orc.encoder_forward_sparse_tsp(W, pts, xt, tt, ei, taps=taps)
    return out.numpy(), taps[-1][1].numpy()
  if case == "mis":
    ei, xt = _case_inputs(case)
    taps = []
    out = orc.encoder_forward_mis(W, xt, tt, ei, taps=taps)
    return out.numpy(), taps[-1][0].numpy()
  pts, xt = _case_inputs(case)
  outs = [orc.encoder_forward_dense(W, pts[b:b + 1], xt[b:b + 1], tt.astype(np.float32)) for b in range(len(pts))]
  return np.stack([o[0].permute(1, 2, 0).reshape(-1, o.shape[1]).numpy() for o in outs]), None


_regimes = {}


def _regime(name, case):
  key = (name, case)
  if key not in _regimes:
    _regimes[key] = G.regime(name, _base(case), lambda w: _oracle_forward(w, case, T_CAL), node_head=case == "mis")
  return _regimes[key]


_oracles = {}


def _oracle(name, case, t):
  """(fp64 logits, fp32 logits, fp64 head input) of regime `name`, cached."""
  key = (name, case, t)
  if key not in _oracles:
    w = _regime(name, case)
    r64, z = _oracle_forward(w, case, t)
    r32, _ = _oracle_forward(w, case, t, torch.float32)
    _oracles[key] = (r64, r32, z)
  return _oracles[key]


def _softmax(x):
  return torch.softmax(torch.as_tensor(np.asarray(x, np.float64)), -1).numpy()


def _errors(out, ref):
  """logits rel-Linf; for two channels also max |p - p_ref| and max |p / p_ref - 1| where p_ref >= 1e-3."""
  e = {"logits": rel_linf(out, ref)}
  if ref.shape[-1] == 2:
    p, pr = _softmax(out), _softmax(ref)
    e["p_abs"] = float(np.abs(p - pr).max())
    big = pr >= P_BIG
    e["p_rel"] = float(np.abs(p[big] / pr[big] - 1).max())
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


# ------------------------------------------------------------------------------------------------
# a. every regime reaches the range it is meant to (CPU, fp64 oracle, the graphs the GPU tests run)
# ------------------------------------------------------------------------------------------------
def _confident(out):
  p = _softmax(out)
  d = out[:, 1] - out[:, 0]
  return float(np.abs(d).max()), float((p.min(-1) < 1e-3).mean())


@pytest.mark.parametrize("case", ["tsp", "mis"])
def test_regimes_reach_their_targets(case):
  base = _base(case)
  r0 = _oracle("R0", case, T_CAL)[0]
  assert np.abs(r0).max() < 1.0
  for name in ("R1", "R6"):
    dmax, frac = _confident(_oracle(name, case, T_CAL)[0])
    assert 10 <= dmax <= 25 and frac >= 0.3, (name, dmax, frac)
  r1x = _oracle("R1x", case, T_CAL)[0]
  assert 90 <= np.abs(r1x).max() <= 110 and np.abs(r1x).max() > np.log(np.finfo(np.float32).max), np.abs(r1x).max()
  w = _regime("R2", case)
  assert all(not w[f"per_layer_out.{l}.2.{s}"].any() for l in range(12) for s in ("weight", "bias"))
  w = _regime("R3", case)
  assert np.array_equal(w["layers.11.C.weight"], base["layers.11.C.weight"] * 3)
  assert np.array_equal(w["per_layer_out.0.2.weight"], base["per_layer_out.0.2.weight"] * 3)
  for name, ratio in (("R4_10", 10), ("R4_100", 100), ("R4_1000", 1000), ("R6", 10)):
    m, s = G.head_group_stats(_oracle(name, case, T_CAL)[2])
    assert np.allclose(np.abs(m) / s, ratio, rtol=1e-3), (name, np.abs(m) / s)
    for t in (1.0, 999.0):     # the offset is calibrated at t = 500; the other timesteps stay in the same range
      m, s = G.head_group_stats(_oracle(name, case, t)[2])
      assert (ratio / 2 < np.abs(m) / s).all() and (np.abs(m) / s < 2 * ratio).all(), (name, t)
  w = _regime("R5", case)
  for p in G.NORM_PREFIXES:
    g = w[p + "weight"]
    assert (g == np.float32(1e-3)).sum() == 4 and g.max() <= 5 and np.sort(g)[4] >= 0.05, p
  gains = np.concatenate([w[p + "weight"] for p in G.NORM_PREFIXES])
  assert (gains < 0.1).mean() > 0.05 and (gains > 2.5).mean() > 0.05
  assert 0.8 < np.concatenate([w[p + "bias"] for p in G.NORM_PREFIXES]).std() < 1.2


def test_gaussian_and_dense_regimes_reach_their_targets():
  assert np.isclose(np.abs(_oracle("R1", "tsp_gauss", T_CAL)[0]).max(), 24, rtol=1e-4)
  for name, ratio in (("R4_10", 10), ("R4_100", 100), ("R4_1000", 1000)):
    m, s = G.head_group_stats(_oracle(name, "tsp_gauss", T_CAL)[2])
    assert np.allclose(np.abs(m) / s, ratio, rtol=1e-3), name
  for case in DENSE:
    r1 = _oracle("R1", case, T_CAL)[0]
    dmax, frac = _confident(r1.reshape(-1, 2))
    assert 10 <= dmax <= 25 and frac >= 0.3, (case, dmax, frac)
    per_sample_max = np.abs(r1[:, :, 1] - r1[:, :, 0]).max(1)
    assert len(set(np.round(per_sample_max, 3))) == len(per_sample_max), "samples should differ"


# ------------------------------------------------------------------------------------------------
# b. forwards, every regime x implementation x timestep, against the fp64 oracle
# ------------------------------------------------------------------------------------------------
def _gpu_forward(w, case, t, impl):
  if case == "mis":
    ei, xt = _case_inputs(case)
    enc = G.encoder(w, 2, node_only=True, impl=impl)
    return enc(G.cu(xt), torch.tensor([t]), edge_index=G.cu(ei)).cpu().numpy()
  pts, ei, xt = _case_inputs(case)
  enc = G.encoder(w, w["out.2.bias"].shape[0], impl=impl)
  return enc(G.cu(pts), torch.tensor([t]), G.cu(xt), G.cu(ei)).cpu().numpy()


# (regime, case, t, impl) -> reason, measured on an H100 (DESIGN.md section 5)
_BF16X3 = {
    "R1": "R1, bf16x3 edge GEMMs: logits rel 2-5e-5 become max |p - p64| 1.0-2.0e-4, max rel 5-15e-4",
    "R6": "R6, bf16x3 edge GEMMs: max |p - p64| 1.8-2.6e-4, max rel 6-11e-4",
}
XFAIL = {(r, c, t, i): _BF16X3[r] for r in ("R1", "R6") for c in ("tsp", "mis") for t in TS for i in ("tc", "tc1")}


def _params(regimes, cases, impls):
  out = []
  for r in regimes:
    for c in cases:
      for t in TS:
        for i in impls:
          reason = XFAIL.get((r, c, t, i))
          out.append(pytest.param(r, c, t, i, marks=[pytest.mark.xfail(strict=True, reason=reason)] if reason else []))
  return out


@pytest.mark.gpu
@pytest.mark.parametrize("regime,case,t,impl", _params(G.REGIMES, ["tsp", "mis"], IMPLS))
def test_categorical_forward_in_regime_vs_fp64_oracle(regime, case, t, impl):
  r64, r32, _ = _oracle(regime, case, t)
  _check(_gpu_forward(_regime(regime, case), case, t, impl), r64, r32, impl, f"{regime} {case} t={t} {impl}")


@pytest.mark.gpu
@pytest.mark.parametrize("regime,case,t,impl", _params(GAUSS_REGIMES, ["tsp_gauss"], IMPLS))
def test_gaussian_forward_in_regime_vs_fp64_oracle(regime, case, t, impl):
  r64, r32, _ = _oracle(regime, case, t)
  _check(_gpu_forward(_regime(regime, case), case, t, impl), r64, r32, impl, f"{regime} {case} t={t} {impl}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["tsp", "mis"])
def test_r1x_denoise_step_softmax_vs_fp64_oracle(case):
  """The forward returns logits; dfb_denoise_step also runs the head's own softmax and posterior.  At logits of ~100
  exp() overflows fp32 unless the maximum is subtracted first: p must be finite and within 1e-4 of the oracle's."""
  w = _regime("R1x", case)
  t1, t2 = 500, 480
  if case == "tsp":
    pts, ei, xt = _case_inputs(case)
    m = G.tsp_model(w, "tc", sparse_factor=20)
    m._prepare(G.cu(pts), G.cu(ei), torch.device("cuda"))
    ref = orc.encoder_forward_sparse_tsp(orc.Weights(w, torch.float64), pts, xt, np.array([float(t1)]), ei)
  else:
    ei, xt = _case_inputs(case)
    m = G.mis_model(w, "tc")
    m.model.set_graph(G.cu(ei), xt.size, 1)
    ref = orc.encoder_forward_mis(orc.Weights(w, torch.float64), xt, np.array([float(t1)]), ei)
  n = xt.size
  consts, last = m.posterior_consts(t1, t2)
  x, u = G.cu(xt), G.cu(syn.uniforms(n, 85, 0))
  xo, p = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
  m.model.engine().denoise_step(_cabi.CATEGORICAL, x.data_ptr(), float(t1), consts, last, u.data_ptr(), 0, 0,
                                xo.data_ptr(), p.data_ptr(), None, torch.cuda.current_stream().cuda_stream)
  _, Q_bar = orc.categorical_tables(1000, "linear")
  pr, _ = orc.categorical_posterior(Q_bar, t1, t2, ref.softmax(-1), torch.as_tensor(xt))
  p = p.cpu().numpy()
  assert np.isfinite(p).all()
  assert np.abs(p - pr.numpy()).max() <= TOL, np.abs(p - pr.numpy()).max()


# ------------------------------------------------------------------------------------------------
# c. R6 through dfb_denoise_step (teacher-forced, 50 steps) and through the fused dfb_denoise loop
# ------------------------------------------------------------------------------------------------
def _posterior_bound(r32_out, r64_out, xt, Q_bar, t1, t2):
  """max(1e-4, 4 x the fp32 oracle's max |p - p64|) for the posterior p of one step."""
  p32, _ = orc.categorical_posterior(Q_bar, t1, t2, torch.as_tensor(_softmax(r32_out)), torch.as_tensor(xt))
  p64, _ = orc.categorical_posterior(Q_bar, t1, t2, torch.as_tensor(_softmax(r64_out)), torch.as_tensor(xt))
  e = float((p32.clamp(0, 1) - p64.clamp(0, 1)).abs().max())
  return max(TOL, 4 * e), e


_traj = {}
STEPS_TF = 50
FLIP_BAND = 10 * TOL      # a flip needs |p64 - u| inside this band, as in the TSP-500 teacher-forced test


def _r6_oracle_trajectory():
  """The fp64 oracle's 50-step categorical trajectory on the TSP case in R6 with injected uniforms, and per step the
  fp32 oracle's logits on the same xt_in and the p bound."""
  if "oracle" not in _traj:
    pts, ei, _ = _case_inputs("tsp")
    n = ei.shape[1]
    w = _regime("R6", "tsp")
    xt0 = (syn.initial_noise(n, 81) > 0).astype(np.float32)
    us = [syn.uniforms(n, 82, i) for i in range(STEPS_TF)]
    rec = []
    orc.denoise(orc.Weights(w, torch.float64), "tsp", "categorical", ei, xt0, points=pts, steps=STEPS_TF,
                uniforms=us, record=rec)
    _, Q_bar = orc.categorical_tables(1000, "linear")
    W32 = orc.Weights(w)
    for i, r in enumerate(rec):
      xin = r["xt_in"].numpy().astype(np.float32)
      r["u"] = us[i]
      r["r32"] = orc.encoder_forward_sparse_tsp(W32, pts, xin, torch.tensor([float(r["t1"])]), ei).numpy()
      r["bound"], r["e32"] = _posterior_bound(r["r32"], r["net_out"].numpy(), xin, Q_bar, r["t1"], r["t2"])
    _traj["oracle"] = rec
  return _traj["oracle"]


def _r6_teacher_forced(impl):
  """dfb_denoise_step fed the oracle's xt_in at every step: per step the kernel's net / p / xt_out."""
  if impl not in _traj:
    rec = _r6_oracle_trajectory()
    pts, ei, _ = _case_inputs("tsp")
    n = ei.shape[1]
    m = G.tsp_model(_regime("R6", "tsp"), impl, sparse_factor=20, inference_diffusion_steps=STEPS_TF)
    dev = torch.device("cuda")
    m._prepare(G.cu(pts), G.cu(ei), dev)
    ctx = m.model.engine()
    st = torch.cuda.current_stream().cuda_stream
    out = []
    for i, r in enumerate(rec):
      consts, last = m.posterior_consts(r["t1"], r["t2"])
      x, u = G.cu(r["xt_in"].numpy().astype(np.float32)), G.cu(r["u"])
      xo, p, net = torch.empty(n, device=dev), torch.empty(n, device=dev), torch.empty((n, 2), device=dev)
      ctx.denoise_step(_cabi.CATEGORICAL, x.data_ptr(), float(r["t1"]), consts, last, u.data_ptr(), 0, i,
                       xo.data_ptr(), p.data_ptr(), net.data_ptr(), st)
      torch.cuda.synchronize()
      out.append(dict(net=net.cpu().numpy(), p=p.cpu().numpy().astype(np.float64), xo=xo.cpu().numpy(), last=last))
    _traj[impl] = out
  return _traj[impl]


def _xfail_bf16x3(reason):
  return pytest.mark.xfail(strict=True, reason=reason)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["tc", "fp32"])
def test_r6_teacher_forced_samples_differ_only_near_ties(impl):
  """A sampled state may differ from the oracle's only where u lies between the kernel's p and the oracle's (the
  only place two Bernoulli draws 1 iff u < clamp(p, 0, 1) with the same u can disagree) and within 1e-3 of the
  oracle's p."""
  flips_total = 0
  for i, (s, r) in enumerate(zip(_r6_teacher_forced(impl)[:-1], _r6_oracle_trajectory()[:-1])):
    pk, pr = s["p"].clip(0, 1), r["p"].numpy().clip(0, 1)
    flips = s["xo"] != r["xt_out"].numpy()
    allowed = (np.abs(pr - r["u"]) <= np.abs(pk - pr)) & (np.abs(pr - r["u"]) < FLIP_BAND)
    assert not np.any(flips & ~allowed), (i, int(flips.sum()), int((flips & ~allowed).sum()))
    flips_total += int(flips.sum())
  assert flips_total <= 50, flips_total


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [pytest.param("tc", marks=_xfail_bf16x3(
    "R6, bf16x3 edge GEMMs: softmax p from the first step on, max |p - p64| 1.8e-4, max rel 9.1e-4")), "fp32"])
def test_r6_teacher_forced_50_steps_precision_vs_fp64_oracle(impl):
  """Network output and p of every step as in (b); the final heat map (clamp(p, min=0)) within the p bound, absolute
  and relative where it is >= 1e-3."""
  for i, (s, r) in enumerate(zip(_r6_teacher_forced(impl), _r6_oracle_trajectory())):
    _check(s["net"], r["net_out"].numpy(), r["r32"], impl, f"step {i}")
    pk, pr = s["p"], r["p"].numpy()
    if not s["last"]:
      err = float(np.abs(pk.clip(0, 1) - pr.clip(0, 1)).max())
      assert err <= r["bound"], (i, err, r["e32"], r["bound"])
    else:
      hm, ref = s["xo"], r["xt_out"].numpy()
      big = ref > P_BIG
      err, rel = float(np.abs(hm - ref).max()), float(np.abs(hm[big] / ref[big] - 1).max())
      assert err <= r["bound"] and rel <= r["bound"], (err, rel, r["e32"], r["bound"])


NUDGE = 1e-3


@pytest.mark.gpu
def test_r6_fused_loop_free_running_follows_oracle_trajectory():
  """Free-running 10-step dfb_denoise with injected uniforms.  The oracle runs the same loop, moving each uniform
  that falls within 1e-3 of its p to 1e-3 above p (1e-3 below where p > 1 - 1e-3), so its trajectory has no tie the kernel's
  p error could break.  The fused loop must then take the oracle's every sample: its heat map is bitwise the one
  dfb_denoise_step gives when fed the oracle's states."""
  steps = 10
  pts, ei, _ = _case_inputs("tsp")
  n = ei.shape[1]
  w = _regime("R6", "tsp")
  Wd = orc.Weights(w, torch.float64)
  _, Q_bar = orc.categorical_tables(1000, "linear")
  sched = orc.inference_schedule("cosine", 1000, steps)
  x = torch.as_tensor((syn.initial_noise(n, 83) > 0).astype(np.float64))
  states, us = [], []
  for i, (t1, t2) in enumerate(sched):
    states.append(x.numpy().astype(np.float32))
    out = orc.encoder_forward_sparse_tsp(Wd, pts, x, torch.tensor([float(t1)]), ei)
    p, _ = orc.categorical_posterior(Q_bar, t1, t2, out.softmax(-1), x)
    pc = p.clamp(0, 1).numpy()
    u = syn.uniforms(n, 84, i).astype(np.float64)
    near = np.abs(u - pc) < NUDGE
    u = np.where(near, np.where((u >= pc) & (pc + NUDGE < 1) | (pc < NUDGE), pc + NUDGE, pc - NUDGE), u)
    u = u.astype(np.float32)
    assert (np.abs(u - pc) >= NUDGE * 0.99).all() and (u >= 0).all() and (u < 1).all()
    us.append(u)
    _, x = orc.categorical_posterior(Q_bar, t1, t2, out.softmax(-1), x, u)
  m = G.tsp_model(w, "tc", sparse_factor=20, inference_diffusion_steps=steps)
  m._prepare(G.cu(pts), G.cu(ei), torch.device("cuda"))
  ctx = m.model.engine()
  st = torch.cuda.current_stream().cuda_stream
  t1s, cs, ls = [], [], []
  for t1, t2 in sched:
    c, last = m.posterior_consts(t1, t2)
    t1s.append(int(t1)); cs.append(c); ls.append(last)
  xf = G.cu(states[0])
  ctx.denoise(_cabi.CATEGORICAL, xf.data_ptr(), t1s, cs, ls, G.cu(np.stack(us)).data_ptr(), 0, st)
  xs, xo = G.cu(states[-1]), torch.empty(n, device="cuda")
  ctx.denoise_step(_cabi.CATEGORICAL, xs.data_ptr(), float(t1s[-1]), cs[-1], ls[-1], G.cu(us[-1]).data_ptr(), 0,
                   steps - 1, xo.data_ptr(), None, None, st)
  torch.cuda.synchronize()
  hm, hm_forced = xf.cpu().numpy(), xo.cpu().numpy()
  assert np.array_equal(hm, hm_forced), float(np.abs(hm - hm_forced).max())


# ------------------------------------------------------------------------------------------------
# d. dense TSP with several GroupNorm segments (one per sample), samples with different statistics
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["R0", pytest.param("R1", marks=_xfail_bf16x3(
    "R1, bf16x3 edge GEMMs: softmax p of sample 0, max |p - p64| 2.3e-4, max rel 1.2e-3"))])
@pytest.mark.parametrize("case", list(DENSE))
def test_dense_multi_segment_vs_oracle_per_sample(regime, case):
  """B samples in one call, GroupNorm per sample over V*V rows: several 256-row statistics blocks per segment and
  k_head warps that straddle two segments (2 500 mod 32 = 4).  Sample 0 has xt = 0, sample 1 xt = 1, the rest are
  random.  Forward logits per sample, then the heat map of categorical_denoise_step (t = 500 -> 0)."""
  V, B = DENSE[case]
  pts, xt = _case_inputs(case)
  w = _regime(regime, case)
  r64, r32, _ = _oracle(regime, case, T_CAL)
  m = G.tsp_model(w, "tc", sparse_factor=-1)
  out = m.model(G.cu(pts), torch.tensor([T_CAL]), G.cu(xt), None).cpu().numpy()        # (B, 2, V, V)
  assert out.shape == (B, 2, V, V)
  out = out.transpose(0, 2, 3, 1).reshape(B, V * V, 2)
  for b in range(B):
    _check(out[b], r64[b], r32[b], "tc", f"{regime} {case} sample {b}")
  dev = torch.device("cuda")
  hm = m.categorical_denoise_step(G.cu(pts), G.cu(xt), np.array([int(T_CAL)]), dev, None,
                                  target_t=np.array([0])).cpu().numpy().reshape(B, -1)
  _, Q_bar = orc.categorical_tables(1000, "linear")
  for b in range(B):
    xb = torch.as_tensor(xt[b].reshape(-1))
    bound, e32 = _posterior_bound(r32[b], r64[b], xb, Q_bar, int(T_CAL), 0)
    _, ref = orc.categorical_posterior(Q_bar, int(T_CAL), 0, torch.as_tensor(_softmax(r64[b])), xb)
    ref = ref.numpy()
    err = float(np.abs(hm[b] - ref).max())
    big = ref > P_BIG
    rel = float(np.abs(hm[b][big] / ref[big] - 1).max())
    assert err <= bound and rel <= bound, (b, err, rel, e32, bound)

"""Trajectory recording of the fused denoise loop (dfb_denoise_record; TSPModel.denoise_heatmap / MISModel.denoise_labels
with record_steps).  Run with -m gpu on an H100.

Recording must not change the loop: the final xt is bitwise dfb_denoise's, captured or not.  What it records must be
the loop's own steps: each row is internally consistent (sample vs p and the Philox draw, p vs the logits), equals what
dfb_denoise_step gives on the recorded input state, and meets the 1e-4 contract against the fp64 oracle at every step
of the free-running product loop, with no near-tie skips: the oracle is evaluated on the GPU's own trajectory."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_linf
from difusco_b200 import _cabi, synthetic as syn
from oracle import difusco_oracle as orc
from oracle import philox
import gpu_util as G

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = torch.device("cuda")
SEED = 0x5EED1234
SENT = -7.25     # sentinel: no kernel output of these loops has this value
TOL = 1e-4
P_BIG = 1e-3


# ------------------------------------------------------------------------------------------------
# cases and raw C-ABI loops
# ------------------------------------------------------------------------------------------------
def _case(name, w2, w1, steps):
  """(model with its graph prepared, xt0 flat float32, categorical?) for one small input."""
  if name == "tsp":
    m = G.tsp_model(w2, sparse_factor=10, inference_diffusion_steps=steps)
    pts, ei = syn.tsp_sparse_batch(80, 10, 2, seed=31)
    m._prepare(G.cu(pts), G.cu(ei), DEV)
    x0 = syn.initial_noise(ei.shape[1], 32) > 0
  elif name == "dense":
    m = G.tsp_model(w2, sparse_factor=-1, inference_diffusion_steps=steps)
    pts = np.stack([syn.tsp_points(20, 33, b) for b in range(2)]).astype(np.float32)
    m._prepare(G.cu(pts), None, DEV)
    x0 = syn.initial_noise(2 * 20 * 20, 34) > 0
  elif name == "mis":
    m = G.mis_model(w2, inference_diffusion_steps=steps)
    m.model.set_graph(G.cu(syn.er_graph_edge_index(200, 0.05, seed=35)), 200, 1)
    x0 = syn.initial_noise(200, 36) > 0
  elif name in ("gauss_ddim", "gauss_ddpm"):
    m = G.tsp_model(w1, diffusion_type="gaussian", sparse_factor=10, inference_diffusion_steps=steps,
                    inference_trick="ddim" if name == "gauss_ddim" else None)
    pts, ei = syn.tsp_sparse_batch(80, 10, 2, seed=37)
    m._prepare(G.cu(pts), G.cu(ei), DEV)
    x0 = syn.initial_noise(ei.shape[1], 38)
  else:
    raise ValueError(name)
  return m, np.asarray(x0, np.float32).reshape(-1), m.diffusion_type == "categorical"


def _sched(m, steps):
  t1s, cs, ls = [], [], []
  for t1, t2 in orc.inference_schedule(m.args.inference_schedule, 1000, steps):
    c, last = m.posterior_consts(t1, t2)
    t1s.append(int(t1)); cs.append(c); ls.append(last)
  return t1s, cs, ls


def _mode(m):
  return _cabi.CATEGORICAL if m.diffusion_type == "categorical" else _cabi.GAUSSIAN


def _buffers(m, n, rows, what=("xt", "p", "out")):
  oc = 2 if m.diffusion_type == "categorical" else 1
  shapes = {"xt": (rows, n), "p": (rows, n), "out": (rows, n, oc)}
  return {k: torch.full(shapes[k], SENT, device=DEV) for k in what}


def _ptr(bufs, k):
  return bufs[k].data_ptr() if k in bufs else None


def _loop(m, x0, steps, rec=None, uniforms=None, seed=SEED, bufs=None):
  """dfb_denoise (rec None) or dfb_denoise_record -> (final xt, record buffers as numpy)."""
  ctx = m.model.engine()
  t1s, cs, ls = _sched(m, steps)
  x = G.cu(x0)
  u = G.cu(np.stack(uniforms)) if uniforms is not None else None
  up = u.data_ptr() if u is not None else None
  st = torch.cuda.current_stream().cuda_stream
  if rec is None:
    ctx.denoise(_mode(m), x.data_ptr(), t1s, cs, ls, up, seed, st)
    bufs = {}
  else:
    if bufs is None:
      bufs = _buffers(m, x0.size, max(len(rec), 1), ("xt", "p", "out") if _mode(m) == _cabi.CATEGORICAL
                      else ("xt", "out"))
    ctx.denoise_record(_mode(m), x.data_ptr(), t1s, cs, ls, rec, _ptr(bufs, "xt"), _ptr(bufs, "p"),
                       _ptr(bufs, "out"), up, seed, st)
  torch.cuda.synchronize()
  return x.cpu().numpy(), {k: v.cpu().numpy() for k, v in bufs.items()}


# ------------------------------------------------------------------------------------------------
# 1. recording changes nothing: final xt bitwise dfb_denoise's, captured and plain, for any record set
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("capture", [True, False])
@pytest.mark.parametrize("case", ["tsp", "dense", "mis", "gauss_ddim", "gauss_ddpm"])
def test_recording_leaves_final_xt_bitwise_unchanged(weights2, weights1, case, capture):
  steps = 15
  m, x0, _ = _case(case, weights2, weights1, steps)
  m.model.engine().set_graph_capture(capture)
  try:
    ref, _ = _loop(m, x0, steps)
    assert np.isfinite(ref).all()
    full = None
    for rec in ([], list(range(steps)), [0, steps - 1], list(range(0, steps, 7))):
      got, bufs = _loop(m, x0, steps, rec)
      assert np.array_equal(got, ref), (case, capture, rec)
      if rec == list(range(steps)):
        full = bufs
        assert np.array_equal(bufs["xt"][-1], ref)
      elif rec:
        for k in bufs:   # a subset records exactly the rows the full record has at those steps
          assert np.array_equal(bufs[k][:len(rec)], full[k][rec]), (case, k, rec)
      else:
        assert all((v == SENT).all() for v in bufs.values())
  finally:
    m.model.engine().set_graph_capture(True)


# ------------------------------------------------------------------------------------------------
# 2. record buffers and steps are not baked into the captured graph
# ------------------------------------------------------------------------------------------------
def test_record_buffers_are_not_baked_into_the_graph(weights2, weights1):
  steps = 12
  m, x0, _ = _case("tsp", weights2, weights1, steps)
  ctx = m.model.engine()
  ctx.set_graph_capture(False)
  _, full = _loop(m, x0, steps, list(range(steps)))
  ctx.set_graph_capture(True)
  n = x0.size
  rec_a, rec_b = [1, 4, 11], [0, 2, 3, 9]
  a = _buffers(m, n, steps)
  _loop(m, x0, steps, rec_a, bufs=a)            # captures
  a_after = {k: v.cpu().numpy() for k, v in a.items()}
  b = _buffers(m, n, steps)
  _loop(m, x0, steps, rec_b, bufs=b)            # replays with other buffers and steps
  for bufs, rec, snap in ((a, rec_a, a_after), (b, rec_b, None)):
    for k, v in bufs.items():
      v = v.cpu().numpy()
      assert np.array_equal(v[:len(rec)], full[k][rec]), (k, rec)
      assert (v[len(rec):] == SENT).all(), (k, rec)
      if snap is not None:
        assert np.array_equal(v, snap[k]), k   # the second call wrote nothing into the first call's buffers


# ------------------------------------------------------------------------------------------------
# 3. internal consistency of a categorical record, bitwise
# ------------------------------------------------------------------------------------------------
def _p_from_logits(out, xin, c):
  """The kernel's posterior p in fp32, in its operation order (expf may differ from numpy's by a few ulp)."""
  l0, l1 = out[:, 0].astype(np.float32), out[:, 1].astype(np.float32)
  m = np.maximum(l0, l1)
  e0, e1 = np.exp(l0 - m), np.exp(l1 - m)
  inv = np.float32(1) / (e0 + e1)
  p0, p1 = e0 * inv, e1 * inv
  x = (xin != 0).astype(np.int64)
  c = np.asarray(c, np.float32)
  a, b = c[2 * x], c[2 * x + 1]
  return a * p0 + b * p1, np.abs(a) * p0 + np.abs(b) * p1


@pytest.mark.parametrize("case", ["tsp", "mis"])
@pytest.mark.parametrize("draws", ["injected", "philox"])
def test_categorical_record_is_internally_consistent(weights2, weights1, case, draws):
  steps = 10
  m, x0, _ = _case(case, weights2, weights1, steps)
  n = x0.size
  us = [syn.uniforms(n, 41, i) for i in range(steps)] if draws == "injected" else None
  final, r = _loop(m, x0, steps, list(range(steps)), uniforms=us)
  _, cs, ls = _sched(m, steps)
  for i in range(steps):
    xin = x0 if i == 0 else r["xt"][i - 1]
    p = r["p"][i]
    if i < steps - 1:
      u = us[i] if us is not None else philox.uniform(SEED, i, np.arange(n))
      assert np.array_equal(r["xt"][i], (u < np.clip(p, 0, 1)).astype(np.float32)), i
    else:
      assert ls[i] == 1
      assert np.array_equal(r["xt"][i], np.maximum(p, 0)) and np.array_equal(r["xt"][i], final)
    p_np, scale = _p_from_logits(r["out"][i], xin, cs[i])
    assert (np.abs(p - p_np) <= 8 * np.finfo(np.float32).eps * scale).all(), (i, float(np.abs(p - p_np).max()))


# ------------------------------------------------------------------------------------------------
# 4. every recorded step equals dfb_denoise_step on the recorded input state, bitwise
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["tsp200", "mis200"])
def test_record_matches_step_api(weights2, case):
  steps = 10
  if case == "tsp200":
    m = G.tsp_model(weights2, sparse_factor=20, inference_diffusion_steps=steps)
    pts, ei = syn.tsp_sparse_batch(200, 20, 1, seed=51)
    m._prepare(G.cu(pts), G.cu(ei), DEV)
    x0 = (syn.initial_noise(ei.shape[1], 52) > 0).astype(np.float32)
  else:
    m = G.mis_model(weights2, inference_diffusion_steps=steps)
    m.model.set_graph(G.cu(syn.er_graph_edge_index(200, 0.05, seed=53)), 200, 1)
    x0 = (syn.initial_noise(200, 54) > 0).astype(np.float32)
  n = x0.size
  _, r = _loop(m, x0, steps, list(range(steps)))
  ctx = m.model.engine()
  st = torch.cuda.current_stream().cuda_stream
  t1s, cs, ls = _sched(m, steps)
  for i in range(steps):
    xin = G.cu(x0 if i == 0 else r["xt"][i - 1])
    xo, p, net = torch.empty(n, device=DEV), torch.empty(n, device=DEV), torch.empty((n, 2), device=DEV)
    ctx.denoise_step(_cabi.CATEGORICAL, xin.data_ptr(), float(t1s[i]), cs[i], ls[i], None, SEED, i, xo.data_ptr(),
                     p.data_ptr(), net.data_ptr(), st)
    torch.cuda.synchronize()
    assert np.array_equal(net.cpu().numpy(), r["out"][i]), i
    assert np.array_equal(p.cpu().numpy(), r["p"][i]), i
    assert np.array_equal(xo.cpu().numpy(), r["xt"][i]), i


def test_gaussian_step_leaves_p_out_untouched(weights2, weights1):
  """A gaussian step has no p: dfb_denoise_step accepts a p_out and writes nothing into it."""
  steps = 4
  m, x0, _ = _case("gauss_ddpm", weights2, weights1, steps)
  n = x0.size
  _, r = _loop(m, x0, steps, [0])
  t1s, cs, ls = _sched(m, steps)
  xin = G.cu(x0)
  xo, p, net = torch.empty(n, device=DEV), torch.full((n,), SENT, device=DEV), torch.empty((n, 1), device=DEV)
  m.model.engine().denoise_step(_cabi.GAUSSIAN, xin.data_ptr(), float(t1s[0]), cs[0], ls[0], None, SEED, 0,
                                xo.data_ptr(), p.data_ptr(), net.data_ptr(), torch.cuda.current_stream().cuda_stream)
  torch.cuda.synchronize()
  assert (p.cpu().numpy() == SENT).all()
  assert np.array_equal(net.cpu().numpy(), r["out"][0]) and np.array_equal(xo.cpu().numpy(), r["xt"][0])


# ------------------------------------------------------------------------------------------------
# 5. every recorded step of the free-running product loop (Philox) against the fp64 oracle, no skips
# ------------------------------------------------------------------------------------------------
def _oracle_fn(kind, data):
  """(xin, t, dtype) -> logits (N, out) in the caller's element order."""
  _w = {}

  def f(xin, t, dtype):
    if dtype not in _w:
      _w[dtype] = orc.Weights(data["w"], dtype)
    W, tt = _w[dtype], np.array([float(t)])
    if kind == "tsp":
      return orc.encoder_forward_sparse_tsp(W, data["pts"], xin, tt, data["ei"]).numpy()
    if kind == "mis":
      return orc.encoder_forward_mis(W, xin, tt, data["ei"]).numpy()
    pts, B, V = data["pts"], data["pts"].shape[0], data["pts"].shape[1]
    x = xin.reshape(B, V, V)
    outs = [orc.encoder_forward_dense(W, pts[b:b + 1], x[b:b + 1], tt.astype(np.float32)) for b in range(B)]
    return np.concatenate([o[0].permute(1, 2, 0).reshape(V * V, -1).numpy() for o in outs])
  return f


def _p_errors(p, ref):
  big = ref >= P_BIG
  return float(np.abs(p - ref).max()), float(np.abs(p[big] / ref[big] - 1).max()) if big.any() else 0.0


@pytest.mark.parametrize("case", ["tsp500", "mis200", "tsp200_gauss", "dense50"])
def test_every_step_of_the_product_loop_vs_fp64_oracle(weights2, weights1, case):
  steps = 50
  torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
  if case == "tsp500":
    m = G.tsp_model(weights2, sparse_factor=50, inference_diffusion_steps=steps)
    pts, ei = syn.tsp_sparse_batch(500, 50, 1, seed=61)
    data, kind = dict(w=weights2, pts=pts, ei=ei), "tsp"
    m._prepare(G.cu(pts), G.cu(ei), DEV)
    x0 = syn.initial_noise(ei.shape[1], 62) > 0
    check = list(range(0, steps, 5))                       # every 5th step, and the step before it for its input
  elif case == "mis200":
    m = G.mis_model(weights2, inference_diffusion_steps=steps)
    ei = syn.er_graph_edge_index(200, 0.05, seed=63)
    data, kind = dict(w=weights2, ei=ei), "mis"
    m.model.set_graph(G.cu(ei), 200, 1)
    x0 = syn.initial_noise(200, 64) > 0
    check = list(range(steps))
  elif case == "tsp200_gauss":
    m = G.tsp_model(weights1, diffusion_type="gaussian", sparse_factor=20, inference_diffusion_steps=steps)
    pts, ei = syn.tsp_sparse_batch(200, 20, 1, seed=65)
    data, kind = dict(w=weights1, pts=pts, ei=ei), "tsp"
    m._prepare(G.cu(pts), G.cu(ei), DEV)
    x0 = syn.initial_noise(ei.shape[1], 66)
    check = list(range(steps))
  else:
    m = G.tsp_model(weights2, sparse_factor=-1, inference_diffusion_steps=steps)
    pts = np.stack([syn.tsp_points(50, 67, b) for b in range(2)]).astype(np.float32)
    data, kind = dict(w=weights2, pts=pts), "dense"
    m._prepare(G.cu(pts), None, DEV)
    x0 = syn.initial_noise(2 * 50 * 50, 68) > 0
    check = list(range(0, steps, 5)) + [steps - 1]
  x0 = np.asarray(x0, np.float32).reshape(-1)
  rec = sorted(set(check) | {i - 1 for i in check if i > 0})
  row = {s: j for j, s in enumerate(rec)}
  _, r = _loop(m, x0, steps, rec)
  fwd = _oracle_fn(kind, data)
  sched = orc.inference_schedule("cosine", 1000, steps)
  cat = m.diffusion_type == "categorical"
  if cat:
    _, Q_bar = orc.categorical_tables(1000, "linear")
  for i in check:
    t1, t2 = sched[i]
    xin = x0 if i == 0 else r["xt"][row[i - 1]]
    r64, r32 = fwd(xin, t1, torch.float64), fwd(xin, t1, torch.float32)
    out = r["out"][row[i]]
    got, yard = rel_linf(out, r64), rel_linf(r32, r64)
    assert got <= max(G.TOL["tc"], 4 * yard), (case, i, got, yard)
    if cat:
      x = torch.as_tensor(xin)
      p64 = orc.categorical_posterior(Q_bar, t1, t2, torch.as_tensor(r64).softmax(-1), x.double())[0].numpy()
      p32 = orc.categorical_posterior(Q_bar, t1, t2, torch.as_tensor(r32).softmax(-1), x.float())[0].numpy()
      e_abs, e_rel = _p_errors(r["p"][row[i]].astype(np.float64), p64)
      y_abs, y_rel = _p_errors(p32.astype(np.float64), p64)
      assert e_abs <= max(TOL, 4 * y_abs) and e_rel <= max(TOL, 4 * y_rel), (case, i, e_abs, e_rel, y_abs, y_rel)


# ------------------------------------------------------------------------------------------------
# 6. the Python surface
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["tsp", "dense", "mis", "tsp_gauss", "mis_gauss"])
def test_python_trace_surface(weights2, weights1, case):
  steps = 6
  gauss = case.endswith("gauss")
  w = weights1 if gauss else weights2
  kw = dict(inference_diffusion_steps=steps, diffusion_type="gaussian" if gauss else "categorical")
  if case.startswith("mis"):
    m = G.mis_model(w, **kw)
    ei = G.cu(syn.er_graph_edge_index(120, 0.05, seed=71))
    x0 = syn.initial_noise(120, 72)
    shape = (120,)
    run = lambda rs: m.denoise_labels(ei, G.cu((x0 if gauss else x0 > 0).astype(np.float32)), seed=7, record_steps=rs)
  elif case == "dense":
    m = G.tsp_model(w, sparse_factor=-1, **kw)
    pts = G.cu(np.stack([syn.tsp_points(20, 73, b) for b in range(2)]).astype(np.float32))
    x0 = syn.initial_noise(2 * 20 * 20, 74).reshape(2, 20, 20)
    shape = (2, 20, 20)
    run = lambda rs: m.denoise_heatmap(pts, None, G.cu((x0 > 0).astype(np.float32)), seed=7, record_steps=rs)
  else:
    m = G.tsp_model(w, sparse_factor=10, **kw)
    pts, ei = syn.tsp_sparse_batch(60, 10, 2, seed=75)
    pts, ei = G.cu(pts), G.cu(ei)
    x0 = syn.initial_noise(ei.shape[1], 76)
    shape = (ei.shape[1],)
    run = lambda rs: m.denoise_heatmap(pts, ei, G.cu((x0 if gauss else x0 > 0).astype(np.float32)), seed=7,
                                       record_steps=rs)
  plain = run(None)
  assert isinstance(plain, torch.Tensor) and tuple(plain.shape) == shape
  res, tr = run("all")
  assert torch.equal(res, plain)
  keys = {"steps", "t", "xt", "out"} | (set() if gauss else {"p"})
  assert set(tr) == keys
  oc = 1 if gauss else 2
  assert tuple(tr["xt"].shape) == (steps,) + shape and tuple(tr["out"].shape) == (steps,) + shape + (oc,)
  if not gauss:
    assert tuple(tr["p"].shape) == (steps,) + shape
  assert all(v.is_cuda for v in tr.values())
  assert tr["steps"].tolist() == list(range(steps))
  assert tr["t"].tolist() == [t1 for t1, _ in orc.inference_schedule("cosine", 1000, steps)]
  assert torch.equal(tr["xt"][-1], res)
  res2, tr2 = run(list(range(steps)))
  assert torch.equal(res2, res) and all(torch.equal(tr[k], tr2[k]) for k in keys)
  res3, tr3 = run([1, steps - 1])
  assert torch.equal(res3, res) and all(torch.equal(tr3[k], tr[k][[1, steps - 1]]) for k in keys)


# ------------------------------------------------------------------------------------------------
# 7. rejected arguments: DFB_E_INVALID before any device work, nothing written
# ------------------------------------------------------------------------------------------------
def _raw_record(m, x, steps, n_record, rec, bufs):
  t1s, cs, ls = _sched(m, steps)
  t1a = (C.c_int32 * steps)(*t1s)
  ca = (C.c_float * (4 * steps))(*[float(v) for c in cs for v in c])
  la = (C.c_int32 * steps)(*ls)
  ra = (C.c_int32 * max(len(rec), 1))(*rec)
  return _cabi.lib().dfb_denoise_record(m.model.engine()._h, _mode(m), x.data_ptr(), steps, t1a, ca, la, None,
                                        SEED, n_record, ra, _ptr(bufs, "xt"), _ptr(bufs, "p"), _ptr(bufs, "out"),
                                        torch.cuda.current_stream().cuda_stream)


def test_rejected_arguments_write_nothing(weights2, weights1):
  steps = 6
  for case in ("tsp", "gauss_ddim"):
    m, x0, cat = _case(case, weights2, weights1, steps)
    bad = [("unsorted", [3, 1], ("xt",)), ("duplicate", [2, 2], ("xt",)), ("too large", [0, steps], ("xt",)),
           ("negative", [-1, 2], ("xt",)), ("no buffer", [0, 1], ()), ("negative count", [], ("xt",))]
    if not cat:
      bad.append(("p with gaussian", [0, 1], ("p",)))
    for what, rec, kinds in bad:
      bufs = _buffers(m, x0.size, 2, ("xt", "p", "out"))
      passed = {k: bufs[k] for k in kinds}
      x = G.cu(x0)
      rc = _raw_record(m, x, steps, -1 if what == "negative count" else len(rec), rec, passed)
      torch.cuda.synchronize()
      assert rc == _cabi.DFB_E_INVALID, (case, what, rc)
      assert all((v == SENT).all() for v in bufs.values()), (case, what)
      assert np.array_equal(x.cpu().numpy(), x0), (case, what)
    # the context is still usable and the model-level check agrees
    got, _ = _loop(m, x0, steps, [0, steps - 1])
    assert np.array_equal(got, _loop(m, x0, steps)[0])
    with pytest.raises(ValueError):
      m._fused_loop(G.cu(x0), steps, SEED, [2, 1])

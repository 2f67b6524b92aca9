"""The phase timers of the edge kernel (dfb_set_phase_timing / dfb_debug_phase_cycles): the timed copy of the product
kernel gives bitwise the product kernel's outputs, its counters are filled and consistent, and with timing off they
stay zero.  Run with -m gpu on an H100."""
import numpy as np
import pytest
import torch

from difusco_b200 import synthetic as syn
import gpu_util as G

pytestmark = pytest.mark.gpu

N_PHASES = 9   # slots 2..10: convert, gemm1 wait, gemm1 mma, e1, reduce, layernorms, gemm2 wait, gemm2 mma, e4


def _forward(enc, pts, xt, ei, t=500.0):
  with torch.no_grad():
    out = enc(G.cu(pts), torch.tensor([t]), G.cu(xt), G.cu(ei))
  torch.cuda.synchronize()
  return out.cpu().numpy()


def _timed_vs_plain(enc, pts, xt, ei):
  ctx = enc.engine()
  plain = _forward(enc, pts, xt, ei)
  ctx.debug_phase_cycles()   # reset
  ctx.set_phase_timing(True)
  try:
    timed = _forward(enc, pts, xt, ei)
    c = ctx.debug_phase_cycles()
  finally:
    ctx.set_phase_timing(False)
  return plain, timed, c


def _check_counters(c, E, layers=12):
  tiles, total, phases = c[0], c[1], c[2:2 + N_PHASES]
  # every layer's launch covers ceil(E / 128) tiles of two warpgroups each
  assert tiles == layers * 2 * ((E + 127) // 128), c[:12]
  assert total > 0 and all(p > 0 for p in phases), c[:12]
  assert sum(phases) <= total, (sum(phases), total)
  assert not any(c[2 + N_PHASES:]), c


def test_timed_kernel_bitwise_equal_c2_forward(weights2):
  pts, ei = syn.tsp_sparse_batch(500, 50, 16, seed=1234)
  xt = (syn.initial_noise(ei.shape[1], 0) > 0).astype(np.float32)
  enc = G.encoder(weights2, 2, impl="tc")
  plain, timed, c = _timed_vs_plain(enc, pts, xt, ei)
  assert np.array_equal(plain, timed)
  _check_counters(c, ei.shape[1])


def test_timed_kernel_bitwise_equal_irregular_graph(weights2):
  """A hub of degree 3000 among degree-1 leaves and nodes without edges, in a shuffled edge order."""
  rng = np.random.default_rng(5)
  V, hub = 1300, 500
  deg = np.ones(V, np.int64)
  deg[hub] = 3000
  deg[[0, 1, 700, 1299]] = 0
  rows = np.repeat(np.arange(V), deg)
  cols = np.where(rows == hub, rng.integers(0, V, rows.size), hub)
  ei = np.stack([rows, cols]).astype(np.int64)[:, rng.permutation(rows.size)]
  pts = rng.random((V, 2)).astype(np.float32)
  xt = (rng.random(ei.shape[1]) > 0.5).astype(np.float32)
  enc = G.encoder(weights2, 2, impl="tc")
  plain, timed, c = _timed_vs_plain(enc, pts, xt, ei)
  assert np.array_equal(plain, timed)
  _check_counters(c, ei.shape[1])


def test_timing_switch_recaptures_the_denoise_graph(weights2):
  """dfb_denoise replays a captured graph: switching the timers on or off must re-capture it, so the counters follow
  the switch and the heat map stays bitwise the same."""
  m = G.tsp_model(weights2, "tc", sparse_factor=10, inference_diffusion_steps=4)
  pts, ei = syn.tsp_sparse_batch(80, 10, 2, seed=12)
  xt0 = (syn.initial_noise(ei.shape[1], 4) > 0).astype(np.float32)
  ctx = m.model.engine()
  ctx.set_graph_capture(True)
  d_pts, d_ei = G.cu(pts), G.cu(ei)   # the same tensors every call: the prepared graph alone never forces a re-capture

  def run():
    hm = m.denoise_heatmap(d_pts, d_ei, G.cu(xt0), seed=5).cpu().numpy()
    return hm, ctx.debug_phase_cycles()

  plain, c0 = run()   # captures without timers
  ctx.set_phase_timing(True)
  try:
    timed, c1 = run()
  finally:
    ctx.set_phase_timing(False)
  again, c2 = run()
  assert c0 == [0] * 32 and c2 == [0] * 32
  assert c1[0] == 4 * 12 * 2 * ((ei.shape[1] + 127) // 128) and c1[1] > 0, c1[:12]
  assert np.array_equal(plain, timed) and np.array_equal(plain, again)


def test_counters_zero_when_timing_off(weights2):
  pts, ei = syn.tsp_sparse_batch(100, 20, 2, seed=9)
  xt = (syn.initial_noise(ei.shape[1], 1) > 0).astype(np.float32)
  enc = G.encoder(weights2, 2, impl="tc")
  ctx = enc.engine()
  ctx.set_phase_timing(True)
  _forward(enc, pts, xt, ei)
  ctx.set_phase_timing(False)
  ctx.debug_phase_cycles()   # read and reset what the timed forward recorded
  _forward(enc, pts, xt, ei)
  assert ctx.debug_phase_cycles() == [0] * 32

"""The GroupNorm head alone against an fp64 head, through dfb_debug_head (run_head: k_gn_partial, k_gn_final, k_head).

Everywhere else the head is seen only after 12 layers, whose own error already uses a good part of the 1e-4 budget.
Here the test sets the head input z itself.

  a. GroupNorm statistics read back through stats_out, against a two-pass fp64 GroupNorm of the same fp32 z: one value
     per segment and group displaced 10 to 1e4 sigma in the segment's first row (for sparse TSP that row is always a
     self-loop edge), groups offset to |mean| / sigma = 1e4, channel means spread over 1e3 sigma, constant groups;
     segments of 1 to 2 M rows, 4096 segments, 32 one-row segments in one warp, a segment boundary at every lane.
     rstd relative error and mean error (sigma units, beyond the fp32 rounding of the mean) <= 1e-5 each.
  b. Logits against the fp64 head per segment: out_channels 1 and 2, an unsorted TSP edge list, MIS, dense samples,
     ragged instance batches, and the a-shapes.  Metric: the largest per-segment relative L-inf; bound
     max(BASE, 4 x the fp32 head's error).
  c. The posterior on the kernel's own logits, bitwise where the operation is exact: u < clamp(p, 0, 1) including
     u == p and u == 0, the `last` clamp, Gaussian DDIM / DDPM, and the Philox draws under call and per-instance keying.
"""
import numpy as np
import pytest
import torch

from difusco_b200 import _cabi, synthetic as syn
from difusco_b200.models.gnn_encoder import reference_frequency_tables
from oracle import difusco_oracle as orc
from oracle import philox
import gpu_util as G

torch.set_grad_enabled(False)

STATS_TOL = 1e-5
BASE = 1e-6   # <= 2 x the largest logit error measured on an H100 (DESIGN section 2)
EPS = 1e-5


def _stream():
  return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------
# contexts and graphs
# ------------------------------------------------------------------------------------------------
_ctx = {}


def _weights(out_channels, seed=0):
  return syn.make_encoder_weights(30 + seed, n_layers=1, out_channels=out_channels)


def _context(out_channels, node_only=False):
  key = (out_channels, node_only)
  if key not in _ctx:
    ctx = _cabi.Context(torch.cuda.current_device())
    ctx.load_weights(_weights(out_channels), 1, 256, out_channels, int(node_only), consts=reference_frequency_tables(256))
    _ctx[key] = ctx
  return _ctx[key]


def _seg_graph(lengths):
  """One node per segment, with lengths[i] self-loop edges: a TSP head of one GroupNorm segment per node."""
  lengths = np.asarray(lengths, np.int64)
  rows = np.repeat(np.arange(lengths.size, dtype=np.int64), lengths)
  return lengths.size, np.stack([rows, rows]), np.arange(lengths.size + 1, dtype=np.int64)


class Prepared(object):
  """A prepared graph: the head rows' segment of each sorted row and the sort (sorted position -> caller index)."""

  def __init__(self, ctx, V, ei, node_ptr=None, gn_segments=1, node_only=False):
    eid = G.cu(ei)
    if node_ptr is not None:
      ctx.prepare_graph_instances(eid.data_ptr(), V, ei.shape[1], node_ptr, _stream())
    else:
      ctx.prepare_graph(eid.data_ptr(), V, ei.shape[1], gn_segments, _stream())
    torch.cuda.synchronize()
    self.ctx = ctx
    if node_only:
      self.R = V
      self.perm = np.arange(V)
      starts = node_ptr if node_ptr is not None else np.arange(gn_segments + 1) * (V // gn_segments)
    else:
      self.R = ei.shape[1]
      self.perm = np.argsort(ei[0], kind="stable")
      if node_ptr is not None:
        rowptr = np.concatenate([[0], np.cumsum(np.bincount(ei[0], minlength=V))])
        starts = rowptr[node_ptr]
      else:
        starts = np.arange(gn_segments + 1) * (self.R // gn_segments)
    self.starts = np.asarray(starts, np.int64)
    self.S = self.starts.size - 1
    self.seg_sorted = np.repeat(np.arange(self.S), np.diff(self.starts))
    self.seg = np.empty(self.R, np.int64)     # segment of each caller element
    self.seg[self.perm] = self.seg_sorted
    self.local = np.empty(self.R, np.int64)   # rank of each caller element among its segment's, in caller order
    counts = np.zeros(self.S, np.int64)
    for s in range(self.R):
      self.local[s] = counts[self.seg[s]]
      counts[self.seg[s]] += 1


# ------------------------------------------------------------------------------------------------
# fp64 / fp32 references
# ------------------------------------------------------------------------------------------------
def ref_stats(z, starts):
  """Two-pass GroupNorm32 statistics of each segment of z (R,256) (torch, any device) in fp64 -> (mean, var) (S,32)."""
  lengths = torch.as_tensor(np.diff(starts), device=z.device)
  S, R = lengths.numel(), z.shape[0]
  seg = torch.repeat_interleave(torch.arange(S, device=z.device), lengths)
  zd = z.double().view(R, 32, 8)
  n = (lengths * 8).double()[:, None]
  mean = torch.zeros((S, 32), dtype=torch.float64, device=z.device).index_add_(0, seg, zd.sum(2)) / n
  dev = zd - mean[seg][:, :, None]
  var = torch.zeros((S, 32), dtype=torch.float64, device=z.device).index_add_(0, seg, (dev * dev).sum(2)) / n
  return mean, var


def ref_head(W, z, seg, S):
  """oracle._head (GroupNorm32 over each segment's rows, ReLU, 1x1 conv) in W's dtype; z (R,256) in any row order,
  seg (R,) its segments.  Rows of a segment are normalised together, as _head does over one call."""
  z = z.to(W.dtype)
  out = torch.empty((z.shape[0], W.out_channels), dtype=W.dtype, device=z.device)
  for s in range(S):
    rows = torch.nonzero(seg == s).flatten()
    out[rows] = orc._head(W, z[rows])
  return out


def seg_rel(got, ref, seg, S):
  """The largest per-segment relative L-inf error: max over segments of |d|_inf / |ref|_inf over the segment's rows."""
  got, ref = np.asarray(got, np.float64).reshape(len(seg), -1), np.asarray(ref, np.float64).reshape(len(seg), -1)
  d = np.abs(got - ref).max(1)
  a = np.abs(ref).max(1)
  num = np.zeros(S)
  den = np.zeros(S)
  np.maximum.at(num, seg, d)
  np.maximum.at(den, seg, a)
  return float((num / np.maximum(den, 1e-30)).max())


def _cuda_weights(out_channels, dtype):
  W = orc.Weights(_weights(out_channels), dtype)
  W.t = {k: v.cuda() for k, v in W.t.items()}
  return W


def test_ref_head_matches_oracle_head_per_segment():
  """ref_head on CPU is oracle._head applied to each segment alone (CPU)."""
  W = orc.Weights(_weights(2), torch.float64)
  rng = np.random.default_rng(1)
  z = torch.as_tensor(rng.standard_normal((70, 256)))
  seg = torch.as_tensor(rng.integers(0, 3, 70))
  out = ref_head(W, z, seg, 3)
  for s in range(3):
    assert torch.equal(out[seg == s], orc._head(W, z[seg == s]))
  mean, var = ref_stats(z[:40], np.array([0, 15, 40]))
  g = z[15:40].view(25, 32, 8)
  assert torch.allclose(mean[1], g.mean((0, 2)), rtol=0, atol=1e-14)
  assert torch.allclose(var[1], g.var((0, 2), unbiased=False), rtol=1e-12, atol=0)


# ------------------------------------------------------------------------------------------------
# a. statistics
# ------------------------------------------------------------------------------------------------
SHAPES = {
    "R1": [1],
    "len31": [31], "len32": [32], "len33": [33], "len255": [255], "len256": [256], "len257": [257],
    "len256k": [256 * 7 - 1, 256 * 7 + 1, 256 * 40 - 1, 256 * 40 + 1],
    "len2M": [2 * 1024 * 1024],
    "segs4096": "segs4096",
    "onerow_warp": [5] + [1] * 32 + [27],
    "every_lane": [33] * 32 + [7],
    "ragged": [1000, 3, 77],
}
DATA = ["pivot10", "pivot100", "pivot1000", "pivot1e4", "offset1e4", "spread1e3", "const"]


def _lengths(shape):
  if SHAPES[shape] == "segs4096":
    return list(np.random.default_rng(5).integers(1, 600, 4096))
  return SHAPES[shape]


def _make_z(data, starts, seed):
  """z (R,256) fp32 on the GPU: per group a mean and sigma; `data` displaces or reshapes it (see the module doc)."""
  R = int(starts[-1])
  g = torch.Generator(device="cuda").manual_seed(seed)
  rng = np.random.default_rng(seed)
  mu = rng.uniform(-3, 3, 32)
  sd = np.exp(rng.uniform(np.log(0.1), np.log(10.0), 32))
  if data == "offset1e4":
    mu = rng.choice([-1, 1], 32) * 1e4 * sd
  chan_mu = np.repeat(mu, 8)
  if data == "spread1e3":
    chan_mu = chan_mu + np.repeat(sd, 8) * 1e3 * (np.tile(np.arange(8), 32) / 7 - 0.5)
  if data == "const":
    return torch.as_tensor(np.repeat(mu, 8), dtype=torch.float32, device="cuda")[None].expand(R, 256).contiguous()
  z = torch.randn((R, 256), generator=g, device="cuda", dtype=torch.float32)
  z = z.mul_(torch.as_tensor(np.repeat(sd, 8), dtype=torch.float32, device="cuda"))
  z = z.add_(torch.as_tensor(chan_mu, dtype=torch.float32, device="cuda"))
  if data.startswith("pivot"):   # channel 0 of every group in each segment's first row
    k = float(data[5:])
    first = torch.as_tensor(starts[:-1], device="cuda")
    z[first[:, None], torch.arange(0, 256, 8, device="cuda")[None]] = torch.as_tensor(
        mu + k * sd, dtype=torch.float32, device="cuda")
  return z


def _stats_errors(stats, mean, var):
  """(rstd relative error, mean error in sigma units beyond the fp32 rounding of the mean; absolute where var = 0)."""
  m_k, r_k = stats[..., 0].double(), stats[..., 1].double()
  r_ref = 1.0 / torch.sqrt(var + EPS)
  rstd_err = float(((r_k - r_ref).abs() / r_ref).max())
  ulp = torch.as_tensor(np.spacing(mean.float().abs().cpu().numpy()), dtype=torch.float64, device=mean.device)
  d = ((m_k - mean).abs() - 0.5 * ulp).clamp(min=0)
  sd = torch.sqrt(var)
  mean_err = float(torch.where(sd > 0, d / sd.clamp(min=1e-300), d).max())
  return rstd_err, mean_err


def _run_stats(shape, data):
  lengths = _lengths(shape)
  V, ei, node_ptr = _seg_graph(lengths)
  ctx = _context(2)
  p = Prepared(ctx, V, ei, node_ptr)
  z = _make_z(data, p.starts, seed=sum(map(ord, shape + data)))
  stats = torch.empty((p.S, 32, 2), device="cuda")
  net = torch.empty((p.R, 2), device="cuda")
  ctx.debug_head(_cabi.HEAD_FORWARD, z.data_ptr(), net_out_ptr=net.data_ptr(), stats_out_ptr=stats.data_ptr(),
                 stream=_stream())
  torch.cuda.synchronize()
  return p, z, stats, net


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("data", DATA)
def test_groupnorm_stats_vs_fp64(shape, data):
  p, z, stats, net = _run_stats(shape, data)
  mean, var = ref_stats(z, p.starts)
  if data == "const":
    assert float(var.max()) == 0.0
  rstd_err, mean_err = _stats_errors(stats, mean, var)
  print(f"\nSTATS {shape} {data}: rstd {rstd_err:.3e} mean {mean_err:.3e}")
  assert rstd_err <= STATS_TOL and mean_err <= STATS_TOL, (shape, data, rstd_err, mean_err)
  if p.R <= 300_000:   # the logits of the same call (the largest shapes are covered by their statistics)
    seg = torch.as_tensor(p.seg_sorted, device="cuda")
    r64 = ref_head(_cuda_weights(2, torch.float64), z, seg, p.S).cpu().numpy()
    r32 = ref_head(_cuda_weights(2, torch.float32), z, seg, p.S).cpu().numpy()
    got, yard = seg_rel(net.cpu().numpy(), r64, p.seg_sorted, p.S), seg_rel(r32, r64, p.seg_sorted, p.S)
    print(f"LOGITS {shape} {data}: {got:.3e} fp32 head {yard:.3e}")
    if data != "const":   # a constant group normalises to 0: every logit is the bias, and the fp32 head matches it
      assert got <= max(BASE, 4 * yard), (shape, data, got, yard)


# ------------------------------------------------------------------------------------------------
# b. logits on the product's graph layouts
# ------------------------------------------------------------------------------------------------
def _layout(name):
  """-> (out_channels, node_only, V, edge_index (caller order), node_ptr or None, gn_segments)."""
  if name.startswith("tsp_shuf"):
    pts, ei = syn.tsp_sparse_batch(60, 10, 1, seed=3)
    ei = ei[:, np.random.default_rng(4).permutation(ei.shape[1])]
    return (1 if name.endswith("oc1") else 2), False, 60, ei, None, 1
  if name == "mis":
    return 2, True, 300, syn.er_graph_edge_index(300, 0.02, seed=5), None, 1
  if name == "dense":
    n, B = 20, 3
    ei = np.concatenate([syn.complete_edge_index(n) + b * n for b in range(B)], 1)
    return 2, False, n * B, ei, None, B
  if name == "ragged_tsp_shuf":
    sizes = [7, 30, 1, 12]
    nptr = syn.node_ptr(sizes)
    parts = [syn.complete_edge_index(s) + o for s, o in zip(sizes, nptr[:-1]) if s > 1] + [np.array([[37], [37]])]
    ei = np.concatenate(parts, 1)
    ei = ei[:, np.random.default_rng(6).permutation(ei.shape[1])]
    return 2, False, sum(sizes), ei, nptr, 1
  if name == "ragged_mis":
    sizes = [5, 90, 33, 1, 64]
    nptr = syn.node_ptr(sizes)
    ei = np.concatenate([syn.er_graph_edge_index(s, 0.2, seed=7 + i) + o
                         for i, (s, o) in enumerate(zip(sizes, nptr[:-1])) if s > 1], 1)
    return 1, True, sum(sizes), ei, nptr, 1
  raise ValueError(name)


LAYOUTS = ["tsp_shuf_oc1", "tsp_shuf_oc2", "mis", "dense", "ragged_tsp_shuf", "ragged_mis"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", LAYOUTS)
def test_head_logits_vs_fp64(name):
  oc, node_only, V, ei, nptr, gs = _layout(name)
  ctx = _context(oc, node_only)
  p = Prepared(ctx, V, ei, nptr, gs, node_only)
  rng = np.random.default_rng(sum(map(ord, name)))
  z_caller = (rng.standard_normal((p.R, 256)) * rng.uniform(0.2, 3, 256) + rng.uniform(-2, 2, 256)).astype(np.float32)
  zs = G.cu(z_caller[p.perm])
  net = torch.empty((p.R, oc), device="cuda")
  ctx.debug_head(_cabi.HEAD_FORWARD, zs.data_ptr(), net_out_ptr=net.data_ptr(), stream=_stream())
  torch.cuda.synchronize()
  zc, seg = torch.as_tensor(z_caller), torch.as_tensor(p.seg)
  r64 = ref_head(orc.Weights(_weights(oc), torch.float64), zc, seg, p.S).numpy()
  r32 = ref_head(orc.Weights(_weights(oc), torch.float32), zc, seg, p.S).numpy()
  got, yard = seg_rel(net.cpu().numpy(), r64, p.seg, p.S), seg_rel(r32, r64, p.seg, p.S)
  print(f"\nLOGITS {name}: {got:.3e} fp32 head {yard:.3e}")
  assert got <= max(BASE, 4 * yard), (name, got, yard)


@pytest.mark.gpu
def test_head_hook_rejects_bad_arguments():
  ctx = _context(2)
  V, ei, nptr = _seg_graph([40])
  Prepared(ctx, V, ei, nptr)
  z = torch.zeros((40, 256), device="cuda")
  x = torch.zeros(40, device="cuda")
  for mode in (-1, 3, _cabi.HEAD_GAUSSIAN):   # unknown, and Gaussian on a 2-channel head
    with pytest.raises(ValueError):
      ctx.debug_head(mode, z.data_ptr(), xt_in_ptr=x.data_ptr(), xt_out_ptr=x.data_ptr(), stream=_stream())
  with pytest.raises(ValueError):   # a posterior needs its state
    ctx.debug_head(_cabi.HEAD_CATEGORICAL, z.data_ptr(), stream=_stream())
  zh = np.zeros((40, 256), np.float32)
  with pytest.raises(ValueError):
    ctx.debug_head(_cabi.HEAD_FORWARD, zh.ctypes.data, stream=_stream())


# ------------------------------------------------------------------------------------------------
# c. the posterior on the kernel's own logits
# ------------------------------------------------------------------------------------------------
def _post_setup(oc, name="ragged_tsp_shuf"):
  _, node_only, V, ei, nptr, gs = _layout(name)
  ctx = _context(oc, node_only)
  p = Prepared(ctx, V, ei, nptr, gs, node_only)
  rng = np.random.default_rng(11)
  zs = G.cu(rng.standard_normal((p.R, 256)).astype(np.float32) * 2)
  xt = G.cu((rng.random(p.R) < 0.4).astype(np.float32))
  return ctx, p, zs, xt


def _cat(ctx, zs, xt, consts, last, u=None, seed=0, step=0, iseeds=None):
  R = xt.numel()
  xo, pp, net = torch.empty(R, device="cuda"), torch.empty(R, device="cuda"), torch.empty((R, 2), device="cuda")
  ctx.debug_head(_cabi.HEAD_CATEGORICAL, zs.data_ptr(), consts, last, None if u is None else u.data_ptr(), seed, step,
                 None if iseeds is None else iseeds.data_ptr(), xt.data_ptr(), xo.data_ptr(), pp.data_ptr(),
                 net.data_ptr(), stream=_stream())
  torch.cuda.synchronize()
  return xo.cpu().numpy(), pp.cpu().numpy(), net.cpu().numpy()


def _consts():
  _, Q_bar = orc.categorical_tables(1000, "linear")
  return orc.categorical_posterior_consts(Q_bar, 500, 480).reshape(-1)


@pytest.mark.gpu
def test_categorical_sample_on_known_p_is_exact():
  ctx, p, zs, xt = _post_setup(2)
  c = _consts()
  _, pr, net = _cat(ctx, zs, xt, c, 0, u=G.cu(np.zeros(p.R, np.float32)))
  # p from the logits in fp64: a few fp32 roundings away
  l = net.astype(np.float64)
  p0 = np.exp(l - l.max(1, keepdims=True))
  p0 /= p0.sum(1, keepdims=True)
  x = xt.cpu().numpy().astype(int)
  cc = c.reshape(2, 2).astype(np.float64)
  assert np.abs(pr - (cc[x, 0] * p0[:, 0] + cc[x, 1] * p0[:, 1])).max() < 1e-6
  rng = np.random.default_rng(12)
  pc = np.clip(pr, 0, 1).astype(np.float32)
  u = rng.random(p.R).astype(np.float32)
  kind = rng.integers(0, 5, p.R)
  u = np.where(kind == 0, pc, u)                                   # u == p: 0
  u = np.where(kind == 1, 0, u)                                    # u == 0: 1 iff p > 0
  u = np.where(kind == 2, np.nextafter(pc, np.float32(0)), u)      # one ulp below p: 1
  u = np.where(kind == 3, np.nextafter(pc, np.float32(1)), u)      # one ulp above p: 0
  u = u.astype(np.float32)
  xo, pr2, _ = _cat(ctx, zs, xt, c, 0, u=G.cu(u))
  assert np.array_equal(pr2, pr)
  assert np.array_equal(xo, (u < pc).astype(np.float32))
  assert (kind == 0).any() and not xo[kind == 0].any()


@pytest.mark.gpu
@pytest.mark.parametrize("side", ["above1", "below0"])
def test_last_clamp_and_sample_clamp_a_few_ulp_outside(side):
  """consts that put p a few ulp above 1 or below 0: `last` returns clamp(p, min=0) (p above 1 kept), a sample
  compares u with clamp(p, 0, 1)."""
  ctx, p, zs, xt = _post_setup(2)
  c = np.full(4, 1 + 2.0 ** -21, np.float32) if side == "above1" else np.full(4, -2.0 ** -23, np.float32)
  xo, pr, _ = _cat(ctx, zs, xt, c, 1)
  assert (pr > 1).any() if side == "above1" else (pr < 0).all()
  assert np.array_equal(xo, np.maximum(pr, np.float32(0)))
  u = np.full(p.R, 1 - 2.0 ** -24, np.float32)   # the largest uniform: 1 iff p was clamped to 1
  xo, pr, _ = _cat(ctx, zs, xt, c, 0, u=G.cu(u))
  assert np.array_equal(xo, (u < np.clip(pr, 0, 1)).astype(np.float32))
  assert xo.any() if side == "above1" else not xo.any()


def _gauss(ctx, zs, x, consts, u=None, seed=0, step=0, iseeds=None):
  R = x.numel()
  xo, net = torch.empty(R, device="cuda"), torch.empty((R, 1), device="cuda")
  ctx.debug_head(_cabi.HEAD_GAUSSIAN, zs.data_ptr(), consts, 0, None if u is None else u.data_ptr(), seed, step,
                 None if iseeds is None else iseeds.data_ptr(), x.data_ptr(), xo.data_ptr(), None, net.data_ptr(),
                 stream=_stream())
  torch.cuda.synchronize()
  return xo.cpu().numpy(), net.cpu().numpy()[:, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("trick", ["ddim", None])
def test_gaussian_posterior_on_known_logits_is_exact(trick):
  ctx, p, zs, _ = _post_setup(1, "ragged_mis")
  beta, alpha, alphabar = orc.gaussian_tables(1000, "linear")
  kind, a, b1, c = orc.gaussian_posterior_consts(beta, alpha, alphabar, 500, 480, trick)
  consts = np.array([a, b1, 0.0, c] if kind == "ddpm" else [a, b1, c, 0.0], np.float32)
  rng = np.random.default_rng(14)
  x = rng.standard_normal(p.R).astype(np.float32)
  zn = rng.standard_normal(p.R).astype(np.float32)
  xo, l0 = _gauss(ctx, zs, G.cu(x), consts, u=G.cu(zn))
  f = np.float32
  y = (consts[0] * (x - (consts[1] * l0).astype(f)).astype(f)).astype(f)
  y = (y + (consts[2] * l0).astype(f)).astype(f)
  if consts[3] != 0:
    y = (consts[3].astype(np.float64) * zn + y).astype(f)   # fmaf: the fp64 product is exact
  assert np.array_equal(xo, y)
  # against the oracle's posterior in fp64 on the same logits
  ref = orc.gaussian_posterior(beta, alpha, alphabar, 500, 480, torch.as_tensor(l0, dtype=torch.float64),
                               torch.as_tensor(x, dtype=torch.float64), trick, z=torch.as_tensor(zn, dtype=torch.float64))
  assert np.abs(xo - ref.numpy()).max() <= 1e-5 * max(1.0, np.abs(ref.numpy()).max())


@pytest.mark.gpu
@pytest.mark.parametrize("keying", ["call", "instance"])
@pytest.mark.parametrize("name", ["ragged_tsp_shuf", "ragged_mis"])
def test_philox_draws_match_oracle(keying, name):
  """Uniforms through the categorical sample (bitwise: xt == u < clamp(p, 0, 1)) and normals through a Gaussian step
  whose consts leave xt_out = z; call keying by caller index, per-instance keying by instance seed and the element's
  rank within its instance in caller order (the `local` table of an unsorted batch)."""
  oc = 2 if name == "ragged_tsp_shuf" else 1
  ctx, p, zs, xt = _post_setup(oc, name)
  seed, step = 0x1234_5678_9ABC_DEF0, 7
  iseeds = np.arange(p.S, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(3)
  if keying == "instance":
    key_seed, elem = iseeds[p.seg], p.local
    dev_seeds = G.cu(iseeds.view(np.int64))
  else:
    key_seed, elem = np.full(p.R, seed, np.uint64), np.arange(p.R)
    dev_seeds = None
  if oc == 2:
    u = np.array([philox.uniform(int(s), step, int(e)) for s, e in zip(key_seed, elem)], np.float32)
    xo, pr, _ = _cat(ctx, zs, xt, _consts(), 0, seed=seed, step=step, iseeds=dev_seeds)
    assert np.array_equal(xo, (u < np.clip(pr, 0, 1)).astype(np.float32))
    assert 0 < xo.mean() < 1
  else:
    zn = np.array([philox.normal(int(s), step, int(e)) for s, e in zip(key_seed, elem)])
    xo, _ = _gauss(ctx, zs, torch.zeros(p.R, device="cuda"), np.array([0, 0, 0, 1], np.float32), seed=seed,
                   step=step, iseeds=dev_seeds)
    assert np.abs(xo - zn).max() < 1e-5 * max(1.0, np.abs(zn).max())

"""Helpers for the -m gpu parity tests (run on an H100; they read nothing outside the repository)."""
from types import SimpleNamespace as NS

import numpy as np
import torch

from difusco_b200 import _cabi, synthetic as syn
from difusco_b200.models.gnn_encoder import GNNEncoder
from difusco_b200.pl_mis_model import MISModel
from difusco_b200.pl_tsp_model import TSPModel

IMPLS = {"tc": _cabi.EDGE_IMPL_TC, "fp32": _cabi.EDGE_IMPL_FP32, "tc1": _cabi.EDGE_IMPL_TC1}
# fp32 validation kernel: fp32 reassociation only.  wgmma kernels: 3-term bf16 split (~2^-17 per product).
TOL = {"fp32": 2e-5, "tc": 1e-4, "tc1": 1e-4}


def args(**kw):
  a = dict(diffusion_type="categorical", diffusion_schedule="linear", diffusion_steps=1000, sparse_factor=50,
           n_layers=12, hidden_dim=256, aggregation="sum", parallel_sampling=1, sequential_sampling=1,
           inference_schedule="cosine", inference_diffusion_steps=50, inference_trick="ddim")
  a.update(kw)
  return NS(**a)


def load(module, weights):
  module.load_state_dict({k: torch.from_numpy(v) for k, v in weights.items()}, strict=True)
  return module.cuda().eval()


def encoder(weights, out_channels, node_only=False, sparse=True, impl="tc", aggregation="sum"):
  enc = load(GNNEncoder(12, 256, out_channels, aggregation=aggregation, sparse=sparse,
                        node_feature_only=node_only), weights)
  enc.engine().set_edge_impl(IMPLS[impl])
  return enc


def tsp_model(weights, impl="tc", **kw):
  m = TSPModel(args(**kw))
  load(m.model, weights)
  m.cuda()
  m.model.engine().set_edge_impl(IMPLS[impl])
  return m


def mis_model(weights, impl="tc", **kw):
  kw.setdefault("sparse_factor", -1)
  m = MISModel(args(**kw))
  load(m.model, weights)
  m.cuda()
  m.model.engine().set_edge_impl(IMPLS[impl])
  return m


def prob_rel(out, ref):
  """Largest relative error of the softmax probabilities of `out` against those of `ref` (last axis)."""
  p = torch.softmax(torch.as_tensor(out), -1).numpy()
  pr = torch.softmax(torch.as_tensor(ref), -1).numpy()
  return float(np.abs(p / pr - 1).max())


def cu(a, dtype=None):
  t = torch.from_numpy(np.ascontiguousarray(a))
  if dtype is not None:
    t = t.to(dtype)
  return t.cuda()


# ------------------------------------------------------------------------------------------------
# Weight regimes: the synthetic weights moved into value ranges a trained checkpoint reaches (confident heads, large
# linears, an offset head GroupNorm input, extreme norm gains, the reference's zero-initialised output layers).
# `fwd(w)` -> (logits (R, out), head input (R, 256)) is the fp64 oracle on the graph the regime is calibrated on;
# `node_head` says the head reads h (MIS) rather than e.
# ------------------------------------------------------------------------------------------------
REGIMES = ["R0", "R1", "R1x", "R2", "R3", "R4_10", "R4_100", "R4_1000", "R5", "R6"]
N_LAYERS = 12
NORM_PREFIXES = ["out.0."] + [f"layers.{l}.norm_{s}." for l in range(N_LAYERS) for s in "he"] + \
                [f"per_layer_out.{l}.0." for l in range(N_LAYERS)]


def head_group_stats(z):
  """Per-group mean and (biased) std of the head GroupNorm32 input z (R, 256), over all rows."""
  g = np.asarray(z, np.float64).reshape(z.shape[0], 32, -1)
  return g.mean((0, 2)), g.std((0, 2))


def _scale_linears(w, f):
  for l in range(N_LAYERS):
    for n in "UVABC":
      w[f"layers.{l}.{n}.weight"] *= f
    w[f"per_layer_out.{l}.2.weight"] *= f


def _offset_head_input(w, fwd, node_head, ratio):
  """Shift each head group by a constant so that its |mean| / std is `ratio` on the calibration graph."""
  m, s = head_group_stats(fwd(w)[1])
  key = f"time_embed_layers.{N_LAYERS - 1}.1.bias" if node_head else f"per_layer_out.{N_LAYERS - 1}.2.bias"
  w[key] += np.repeat(ratio * s - m, 8).astype(np.float32)


def _confident_head(w, fwd, target):
  """Scale out.2 so that the largest |l1 - l0| (|x0| for one channel) is `target`; two channels: also move the
  decision point to the 90th percentile of l1 - l0, so most rows are confidently class 0, as in a trained TSP head
  (2 of the K = 20 edges of a node are tour edges)."""
  out = fwd(w)[0]
  out = out.reshape(-1, out.shape[-1])
  if out.shape[1] == 1:
    a = target / np.abs(out).max()
    q = 0.0
  else:
    d = out[:, 1] - out[:, 0]
    q = float(np.quantile(d, 0.9))
    a = target / np.abs(d - q).max()
  w["out.2.weight"] *= np.float32(a)
  w["out.2.bias"] *= np.float32(a)
  if out.shape[1] == 2:
    w["out.2.bias"][1] -= np.float32(a * q)


def regime(name, weights, fwd, node_head, seed=0):
  """A new state dict: `name` in REGIMES applied to `weights` (not modified)."""
  w = {k: v.copy() for k, v in weights.items()}
  if name == "R0":                       # control
    pass
  elif name == "R1":                     # confident head: max |l1 - l0| = 24
    _confident_head(w, fwd, 24.0)
  elif name == "R1x":                    # logits of ~100: exp() without max-subtraction overflows in fp32
    a = np.float32(100.0 / np.abs(fwd(w)[0]).max())
    w["out.2.weight"] *= a
    w["out.2.bias"] *= a
  elif name == "R2":                     # the reference's own init (gnn_encoder.py:343-345)
    for l in range(N_LAYERS):
      w[f"per_layer_out.{l}.2.weight"][:] = 0
      w[f"per_layer_out.{l}.2.bias"][:] = 0
  elif name == "R3":                     # U, V, A, B, C and per_layer_out.*.2 weights x 3
    _scale_linears(w, 3.0)
  elif name.startswith("R4_"):           # head GroupNorm input with |mean| / std = ratio
    _offset_head_input(w, fwd, node_head, float(name[3:]))
  elif name == "R5":                     # norm affines: gains log-uniform [0.05, 5] (4 channels at 1e-3), biases N(0,1)
    rng = np.random.default_rng(seed)
    for p in NORM_PREFIXES:
      g = np.exp(rng.uniform(np.log(0.05), np.log(5.0), 256))
      g[rng.choice(256, 4, replace=False)] = 1e-3
      w[p + "weight"] = g.astype(np.float32)
      w[p + "bias"] = rng.standard_normal(256).astype(np.float32)
  elif name == "R6":                     # R3, then R4 at 10, then R1
    _scale_linears(w, 3.0)
    _offset_head_input(w, fwd, node_head, 10.0)
    _confident_head(w, fwd, 24.0)
  else:
    raise ValueError(name)
  return w


# ------------------------------------------------------------------------------------------------
# Irregular graphs: (V, edge_index (2,E) int64), rows sorted; deterministic from fixed seeds
# ------------------------------------------------------------------------------------------------
def graph_from_degrees(deg, rng, cols=None):
  deg = np.asarray(deg, np.int64)
  V = deg.size
  rows = np.repeat(np.arange(V, dtype=np.int64), deg)
  if cols is None:
    cols = rng.integers(0, V, rows.size)
  return V, np.stack([rows, np.asarray(cols, np.int64)])


def hub_graph():
  """Node 500 has degree 3000 (edges 500..3499: 24 tiles of 128 rows, 94 groups); the other 1200 nodes are
  degree-1 leaves pointing at the hub, so each of the groups before and after it holds 32 distinct nodes."""
  rng = np.random.default_rng(11)
  V, hub = 1201, 500
  deg = np.ones(V, np.int64)
  deg[hub] = 3000
  rows = np.repeat(np.arange(V), deg)
  cols = np.where(rows == hub, rng.integers(0, V, rows.size), hub)
  return graph_from_degrees(deg, rng, cols)


ISOLATED = [0, 1, 2, 60, 61, 62, 63, 64, 130, 132, 134, 234, 235, 236, 237, 238, 239]


def isolated_graph():
  """Nodes without edges at the start, as a run and singly between nodes that share a 32-edge group, and at the
  end of the index range (the caller passes points / xt for them too)."""
  rng = np.random.default_rng(12)
  deg = rng.integers(1, 5, 240)
  deg[ISOLATED] = 0
  return graph_from_degrees(deg, rng)


# cumulative ends land on, one before and one after multiples of 32, 64 and 128 (test_gpu_graph_edges.py checks it)
DEGREES = [31, 1, 32, 33, 31, 1, 63, 65, 127, 1, 128, 129, 127, 64, 64, 1, 31, 33, 2, 62, 65, 63, 129, 128, 124, 1,
           63, 1, 127, 129]


def degseq_graph():
  return graph_from_degrees(DEGREES, np.random.default_rng(13))


def dup_graph():
  """A ring without self loops in which every edge appears one to three times."""
  rng = np.random.default_rng(14)
  V = 150
  r, c = [], []
  for i in range(V):
    for j in ((i + 1) % V, (i - 1) % V):
      k = int(rng.integers(1, 4))
      r += [i] * k
      c += [j] * k
  return V, np.array([r, c], np.int64)


TINY = {1: 1, 2: 2, 31: 3, 33: 4, 63: 9, 65: 5, 127: 7, 129: 9}   # E -> V


def tiny_graph(E):
  """E < 129 edges on at most 9 nodes: one partial tile, the second warpgroup idle for E < 64, duplicates."""
  rng = np.random.default_rng(100 + E)
  V = TINY[E]
  rows = np.sort(rng.integers(0, V, E))
  return V, np.stack([rows, rng.integers(0, V, E)]).astype(np.int64)

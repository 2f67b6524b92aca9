"""Synthetic workloads for the denoise path: instances, graphs and weights.

Everything here is deterministic from integer seeds (numpy PCG64, which is stable across
platforms and numpy versions) and independent of the reference tree, so the SAME tensors can be
rebuilt in this container (golden generation, CPU tests) and on the GPU box (parity tests, bench).

Input distributions follow the reference's own generators (no datasets are available offline):
  * TSP points ~ U[0,1)^2                      data/generate_tsp_data.py:44
  * sparse kNN graph: KDTree(leaf_size=30, euclidean).query(points, k=K); self is neighbour 0,
    ascending distance; edge_index = [arange(N).repeat_interleave(K); knn.flatten()]
                                                difusco/co_datasets/tsp_graph_dataset.py:56-62
  * MIS: Erdos-Renyi G(n, p), edges -> [edges; reversed; self loops], NOT row-sorted
                                                difusco/co_datasets/mis_dataset.py:43-48
  * weights: torch-default-like init scale; `per_layer_out.*.2` is re-randomised because the
    reference zero-initialises it (gnn_encoder.py:343-345) which would hide half of every layer.
"""
import zlib

import numpy as np


def _rng(seed, tag):
  return np.random.Generator(np.random.PCG64([int(seed), zlib.crc32(tag.encode())]))


# --------------------------------------------------------------------------------------------
# weights
# --------------------------------------------------------------------------------------------
def encoder_param_shapes(n_layers=12, hidden_dim=256, out_channels=2):
  """state_dict key -> shape, in the reference's registration order
  (gnn_encoder.py:294-348; key list confirmed against the reference module in make_golden.py)."""
  H, T = hidden_dim, hidden_dim // 2
  shapes = {
      "node_embed.weight": (H, H), "node_embed.bias": (H,),
      "edge_embed.weight": (H, H), "edge_embed.bias": (H,),
      "time_embed.0.weight": (T, H), "time_embed.0.bias": (T,),
      "time_embed.2.weight": (T, T), "time_embed.2.bias": (T,),
      "out.0.weight": (H,), "out.0.bias": (H,),
      "out.2.weight": (out_channels, H, 1, 1), "out.2.bias": (out_channels,),
  }
  for l in range(n_layers):
    for name in "UVABC":
      shapes[f"layers.{l}.{name}.weight"] = (H, H)
      shapes[f"layers.{l}.{name}.bias"] = (H,)
    for name in ("norm_h", "norm_e"):
      shapes[f"layers.{l}.{name}.weight"] = (H,)
      shapes[f"layers.{l}.{name}.bias"] = (H,)
  for l in range(n_layers):
    shapes[f"time_embed_layers.{l}.1.weight"] = (H, T)
    shapes[f"time_embed_layers.{l}.1.bias"] = (H,)
  for l in range(n_layers):
    shapes[f"per_layer_out.{l}.0.weight"] = (H,)
    shapes[f"per_layer_out.{l}.0.bias"] = (H,)
    shapes[f"per_layer_out.{l}.2.weight"] = (H, H)
    shapes[f"per_layer_out.{l}.2.bias"] = (H,)
  return shapes


def make_encoder_weights(seed=0, n_layers=12, hidden_dim=256, out_channels=2):
  """Deterministic fp32 weights keyed like GNNEncoder.state_dict().

  Linear / conv: U(-1/sqrt(fan_in), 1/sqrt(fan_in)) (torch's default scale), biases likewise.
  Norm affine: weight = 1 + 0.1 N(0,1), bias = 0.1 N(0,1) (non-trivial so a dropped affine
  term is caught).  per_layer_out.*.2: U(-1/16, 1/16) for H=256 (BASELINE.md section 3)."""
  out = {}
  for key, shape in encoder_param_shapes(n_layers, hidden_dim, out_channels).items():
    g = _rng(seed, key)
    parts = key.split(".")
    is_norm = (".norm_" in key) or key.startswith("out.0.") or (
        parts[0] == "per_layer_out" and parts[2] == "0")
    if is_norm:
      if key.endswith("weight"):
        w = 1.0 + 0.1 * g.standard_normal(shape)
      else:
        w = 0.1 * g.standard_normal(shape)
    else:
      if key.endswith("weight"):
        fan_in = int(np.prod(shape[1:]))
      else:
        wshape = encoder_param_shapes(n_layers, hidden_dim, out_channels)[key[:-4] + "weight"]
        fan_in = int(np.prod(wshape[1:]))
      bound = 1.0 / np.sqrt(fan_in)
      w = g.uniform(-bound, bound, size=shape)
    out[key] = np.ascontiguousarray(w, dtype=np.float32)
  return out


# --------------------------------------------------------------------------------------------
# TSP instances
# --------------------------------------------------------------------------------------------
def tsp_points(num_nodes, seed=1234, instance=0):
  return _rng(seed, f"tsp{instance}").random((num_nodes, 2)).astype(np.float32)


def knn_edge_index(points, k):
  """(2, N*k) int64, row-major K per node, self first (tsp_graph_dataset.py:56-62)."""
  from sklearn.neighbors import KDTree
  n = points.shape[0]
  tree = KDTree(points, leaf_size=30, metric="euclidean")
  _, idx = tree.query(points, k=k)
  row = np.repeat(np.arange(n, dtype=np.int64), k)
  return np.stack([row, idx.reshape(-1).astype(np.int64)], axis=0)


def complete_edge_index(n):
  """Row-major complete graph INCLUDING self pairs: the sparse image of the dense path
  (gnn_encoder.py:365 sets graph = ones; the masking at :166 is commented out)."""
  row = np.repeat(np.arange(n, dtype=np.int64), n)
  col = np.tile(np.arange(n, dtype=np.int64), n)
  return np.stack([row, col], axis=0)


def tsp_sparse_batch(num_nodes, k, batch, seed=1234):
  """`batch` independent instances concatenated block-diagonally with node offsets, exactly the
  shape a PyG batch / duplicate_edge_index call gives (pl_meta_model.py:177-184).
  Returns points (B*N, 2) fp32, edge_index (2, B*N*k) int64."""
  pts, eis = [], []
  for b in range(batch):
    p = tsp_points(num_nodes, seed, b)
    ei = knn_edge_index(p, k) + b * num_nodes
    pts.append(p)
    eis.append(ei)
  return np.concatenate(pts, 0), np.concatenate(eis, 1)


# --------------------------------------------------------------------------------------------
# MIS instances
# --------------------------------------------------------------------------------------------
def er_graph_edge_index(n, p, seed=0, instance=0):
  """Erdos-Renyi G(n,p) -> directed edge list [edges; reversed; self loops] (mis_dataset.py:43-48).
  Edge order is NOT row sorted, as in the reference."""
  g = _rng(seed, f"er{instance}")
  iu = np.triu_indices(n, k=1)
  keep = g.random(iu[0].shape[0]) < p
  a, b = iu[0][keep].astype(np.int64), iu[1][keep].astype(np.int64)
  self_loop = np.arange(n, dtype=np.int64)
  row = np.concatenate([a, b, self_loop])
  col = np.concatenate([b, a, self_loop])
  return np.stack([row, col], axis=0)


def mis_batch(n_lo, n_hi, p, batch, seed=0):
  """`batch` ER graphs with n ~ U{n_lo..n_hi}, concatenated block-diagonally.
  Returns edge_index (2, E) int64, sizes list."""
  g = _rng(seed, "mis_sizes")
  sizes = [int(g.integers(n_lo, n_hi + 1)) for _ in range(batch)]
  eis, off = [], 0
  for b, n in enumerate(sizes):
    eis.append(er_graph_edge_index(n, p, seed, b) + off)
    off += n
  return np.concatenate(eis, 1), sizes


def node_ptr(sizes):
  """Node offsets (PyG's Batch.ptr) of graphs with `sizes` nodes concatenated block-diagonally: (len(sizes) + 1,)
  int64, node_ptr[i] the first node of graph i."""
  return np.concatenate([[0], np.cumsum(np.asarray(sizes, np.int64))]).astype(np.int64)


# --------------------------------------------------------------------------------------------
# noise
# --------------------------------------------------------------------------------------------
def initial_noise(n, seed=0, tag="xt0"):
  """Standard normal initial noise; categorical uses (z > 0) (pl_tsp_model.py:186-197)."""
  return _rng(seed, tag).standard_normal(n).astype(np.float32)


def uniforms(n, seed=0, step=0):
  """Injected U[0,1) draws for the Bernoulli posterior sample (teacher-forced parity)."""
  return _rng(seed, f"u{step}").random(n, dtype=np.float32)

"""GNNEncoder: drop-in for the reference's `models.gnn_encoder.GNNEncoder` at inference.

Same constructor signature, same parameter tree (so `state_dict()` keys and shapes are identical
and Lightning checkpoints load with `load_state_dict`), same `forward(x, timesteps, graph,
edge_index)` contract (difusco/models/gnn_encoder.py:290-462) - but `forward` does no PyTorch
math: it hands raw device pointers to the sm_100a CUDA library through the C-ABI
(include/difusco_b200.h).  There is no eager fallback: without the library or without an H100
the call raises.

Interface notes (reference behaviour kept):
  * sparse TSP  : forward(x (V,2), t (1,) or (E,), graph=xt (E,), edge_index (2,E)) -> (E, out)    :383-402
  * MIS         : forward(xt (V,), t (1,) or (V,), edge_index=(2,E))               -> (V, out)      :404-414
  * dense TSP   : forward(x (B,V,2), t (1,) or (B,), graph=xt (B,V,V))             -> (B,out,V,V)   :350-381
    evaluated as the row-major complete graph incl. self pairs (gnn_encoder.py:365 makes the
    graph all-ones), GroupNorm per sample, in one call whatever the timesteps.
  * a timestep per element (the reference's training steps, pl_tsp_model.py:66-67, pl_mis_model.py:54) runs in the
    same single call (dfb_encoder_forward_timesteps); with use_activation_checkpoint=True the sparse forwards run
    every element at t[0], as the reference's checkpointed branch does (gnn_encoder.py:429).  The sparse forwards read
    different per-element timesteps on the model's device, where the training steps put them; a host tensor of them
    raises NotImplementedError.
  * dense + node_feature_only raises NotImplementedError (:457), as in the reference.
  * sparse TSP and MIS take a keyword-only node_ptr (PyG's Batch.ptr: instance i owns nodes
    [node_ptr[i], node_ptr[i+1])): one block-diagonal call over a ragged batch whose head GroupNorm
    runs per instance, so every instance gets the result it would get alone (the reference's test
    loader runs batch size 1).  Without it the GroupNorm statistics span every row of the call.
  * edge_precision (keyword only, not in the reference) picks the tensor-core edge GEMMs' split: "bf16x3" (default,
    three bf16 products) keeps the heat map within 1e-4 of the reference for logits of synthetic range; "bf16x6" (six
    products of three-part operands, several times slower) keeps it there at any confidence, as a trained
    checkpoint's heads need (include/difusco_b200.h, DFB_EDGE_IMPL_TC6).
Only the forward is in scope: autograd is not supported - outputs carry no grad_fn, and a call with grad mode enabled
on parameters that require grad warns once.  A training-step loss is evaluated under torch.no_grad().
"""
import math

import numpy as np
import torch
from torch import nn

from .. import _cabi


def reference_frequency_tables(hidden_dim):
  """The three tiny frequency tables, evaluated with the reference's own torch expressions so
  the device uses bit-identical values (nn.py:113-116; gnn_encoder.py:216-217, :243-244)."""
  half = hidden_dim // 2
  freqs = torch.exp(-math.log(10000) * torch.arange(start=0, end=half, dtype=torch.float32) / half)
  i = torch.arange(half, dtype=torch.float32)
  dimt_pos = 10000 ** (2.0 * (torch.div(i, 2, rounding_mode="trunc")) / half)
  i = torch.arange(hidden_dim, dtype=torch.float32)
  dimt_scalar = 10000 ** (2 * torch.div(i, 2, rounding_mode="trunc") / hidden_dim)
  return {"__const.time_freqs": freqs.numpy(), "__const.dimt_pos": dimt_pos.numpy(),
          "__const.dimt_scalar": dimt_scalar.numpy()}


# GNNEncoder(edge_precision=...) -> the edge implementation it selects
EDGE_PRECISION = {"bf16x3": _cabi.EDGE_IMPL_TC, "bf16x6": _cabi.EDGE_IMPL_TC6}

MAX_TIMESTEPS = 4096   # distinct timesteps of one call (the device step table of dfb_encoder_forward_timesteps)


def timestep_args(timesteps, n, first_only=False, device=None):
  """The timesteps of a forward over n elements (edges, nodes or dense samples) -> a float, the one timestep of the
  call, or (values, index): the distinct timesteps as a host float32 array and, on the device of `timesteps`, each
  element's position among them as int32 (n,).  One value, or n equal values, give the float.  first_only (the
  reference's checkpointed sparse layers, gnn_encoder.py:429) gives t[0] for any length.  With `device` (the sparse
  forwards), different timesteps must lie on it, where the reference's training steps put them
  (pl_tsp_model.py:76-81, pl_mis_model.py:65-69): a host tensor of them raises NotImplementedError, as every
  per-element call of the sparse forwards did before they were supported."""
  t = timesteps.reshape(-1).float()
  if t.numel() == 0 or (t.numel() not in (1, n) and not first_only):
    raise ValueError(f"timesteps must hold 1 or {n} values (one per element), got {t.numel()}")
  if t.numel() == 1:
    return float(t[0])
  if device is not None and t.device != torch.device(device) and not bool((t == t[0]).all()):
    raise NotImplementedError(f"different timesteps per element are read on the model's device ({device}), where "
                              f"the reference's training steps put them; got a {t.device} tensor")
  if first_only:
    return float(t[0])
  values, index = torch.unique(t, return_inverse=True)
  if values.numel() == 1:
    return float(values[0])
  if values.numel() > MAX_TIMESTEPS:
    raise NotImplementedError(f"{values.numel()} distinct timesteps in one forward; at most {MAX_TIMESTEPS} are "
                              "supported (integer timesteps in [1, T] never exceed it)")
  return values.cpu().numpy(), index.to(torch.int32)


def node_ptr_array(node_ptr):
  """node_ptr, a 1-D integer tensor or sequence of n_instances + 1 node offsets (PyG's Batch.ptr) -> host int64
  numpy array.  Checks its shape and dtype; dfb_prepare_graph_instances checks the offsets against the graph."""
  if isinstance(node_ptr, torch.Tensor):
    if node_ptr.dtype not in (torch.int8, torch.int16, torch.int32, torch.int64, torch.uint8):
      raise ValueError(f"node_ptr must hold integers, got {node_ptr.dtype}")
    a = node_ptr.detach().cpu().numpy()
  else:
    a = np.asarray(node_ptr)
    if a.dtype.kind not in "iu":
      raise ValueError(f"node_ptr must hold integers, got {a.dtype}")
  if a.ndim != 1 or a.shape[0] < 2:
    raise ValueError(f"node_ptr must be 1-D with n_instances + 1 >= 2 entries, got shape {tuple(a.shape)}")
  return np.ascontiguousarray(a, dtype=np.int64)


class GNNLayer(nn.Module):
  """Parameter holder of one gated-GCN layer (gnn_encoder.py:20-65).  Compute is fused in CUDA."""

  def __init__(self, hidden_dim, aggregation="sum", norm="layer", learn_norm=True, track_norm=False,
               gated=True):
    super().__init__()
    if not gated:
      raise AssertionError("Use gating with GCN, pass the `--gated` flag")   # gnn_encoder.py:49
    if norm != "layer" or not learn_norm:
      raise NotImplementedError("difusco_b200 implements the reference default norm='layer' with affine")
    self.hidden_dim, self.aggregation = hidden_dim, aggregation
    for name in "UVABC":
      setattr(self, name, nn.Linear(hidden_dim, hidden_dim, bias=True))
    self.norm_h = nn.LayerNorm(hidden_dim, elementwise_affine=True)
    self.norm_e = nn.LayerNorm(hidden_dim, elementwise_affine=True)

  def forward(self, *a, **k):
    raise NotImplementedError("GNNLayer is fused into the edge-layer CUDA kernel; call GNNEncoder.forward")


class GNNEncoder(nn.Module):
  _warned_no_grad = False

  def __init__(self, n_layers, hidden_dim, out_channels=1, aggregation="sum", norm="layer",
               learn_norm=True, track_norm=False, gated=True,
               sparse=False, use_activation_checkpoint=False, node_feature_only=False,
               *args, edge_precision="bf16x3", **kwargs):
    super().__init__()
    if edge_precision not in EDGE_PRECISION:
      raise ValueError(f"edge_precision must be one of {sorted(EDGE_PRECISION)}, got {edge_precision!r}")
    self.edge_precision = edge_precision
    self.sparse = sparse
    self.node_feature_only = node_feature_only
    self.hidden_dim = hidden_dim
    self.n_layers = n_layers
    self.out_channels = out_channels
    self.aggregation = aggregation
    # a training memory knob; the reference's checkpointed sparse layers run every element at t[0] (gnn_encoder.py:429),
    # which the sparse forwards reproduce.  The dense forward ignores it (the reference raises there, :370-371).
    self.use_activation_checkpoint = use_activation_checkpoint
    ted = hidden_dim // 2
    self.node_embed = nn.Linear(hidden_dim, hidden_dim)
    self.edge_embed = nn.Linear(hidden_dim, hidden_dim)
    self.time_embed = nn.Sequential(nn.Linear(hidden_dim, ted), nn.ReLU(), nn.Linear(ted, ted))
    self.out = nn.Sequential(nn.GroupNorm(32, hidden_dim), nn.ReLU(),
                             nn.Conv2d(hidden_dim, out_channels, kernel_size=1, bias=True))
    self.layers = nn.ModuleList([GNNLayer(hidden_dim, aggregation, norm, learn_norm, track_norm, gated)
                                 for _ in range(n_layers)])
    self.time_embed_layers = nn.ModuleList([nn.Sequential(nn.ReLU(), nn.Linear(ted, hidden_dim))
                                            for _ in range(n_layers)])
    self.per_layer_out = nn.ModuleList([
        nn.Sequential(nn.LayerNorm(hidden_dim, elementwise_affine=learn_norm), nn.SiLU(),
                      nn.Linear(hidden_dim, hidden_dim)) for _ in range(n_layers)])
    for seq in self.per_layer_out:            # zero_module (gnn_encoder.py:343-345, nn.py:68-74)
      for p in seq[2].parameters():
        p.detach().zero_()
    self._ctx = None
    self._weights_key = None
    self._graph_key = None
    self._points_key = None
    self._n_segments = 0      # GroupNorm segments of the prepared graph: instances, dense samples or 1
    self._complete_cache = {}

  # ------------------------------------------------------------------------------------------
  # engine plumbing
  # ------------------------------------------------------------------------------------------
  def _device(self):
    dev = self.node_embed.weight.device
    if dev.type != "cuda":
      raise RuntimeError("difusco_b200.GNNEncoder runs on a CUDA device only (no CPU fallback); "
                         "move the module with .cuda() first")
    return dev

  def engine(self):
    dev = self._device()
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    if self._ctx is None or self._ctx.device != idx:
      self._ctx = _cabi.Context(idx)
      _cabi.device_context(idx, prefer=self._ctx)   # k-NN / 2-opt helpers share the first model's context
      self._ctx.set_aggregation(self.aggregation)
      self._ctx.set_edge_impl(EDGE_PRECISION[self.edge_precision])
      self._weights_key = self._graph_key = self._points_key = None
    self._sync_weights()
    return self._ctx

  def _sync_weights(self):
    key = tuple((p.data_ptr(), p._version) for p in self.parameters())
    if key == self._weights_key:
      return
    sd = {k: v.detach().float().cpu().numpy() for k, v in self.state_dict().items()}
    self._ctx.load_weights(sd, self.n_layers, self.hidden_dim, self.out_channels, self.node_feature_only,
                           consts=reference_frequency_tables(self.hidden_dim))
    self._weights_key = key
    self._graph_key = self._points_key = None

  @staticmethod
  def _stream():
    return torch.cuda.current_stream().cuda_stream

  def set_graph(self, edge_index, num_nodes, gn_segments=1, node_ptr=None):
    """Prepare (and cache) the graph of subsequent calls.  edge_index (2,E) int64, any device.  The head GroupNorm
    runs over gn_segments equal row blocks, or, with node_ptr (n_instances + 1 node offsets), once per instance."""
    ptr = None if node_ptr is None else node_ptr_array(node_ptr)
    if ptr is not None and int(gn_segments) != 1:
      raise ValueError("give node_ptr or gn_segments, not both")
    ctx = self.engine()
    ei = edge_index.long().contiguous()
    key = (ei.data_ptr(), tuple(ei.shape), ei._version, int(num_nodes), int(gn_segments), str(ei.device),
           None if ptr is None else ptr.tobytes())
    if key != self._graph_key:
      if ei.dim() != 2 or ei.shape[0] != 2:
        raise ValueError("edge_index must have shape (2, E)")
      if ptr is None:
        ctx.prepare_graph(ei.data_ptr(), int(num_nodes), int(ei.shape[1]), int(gn_segments), self._stream())
      else:
        ctx.prepare_graph_instances(ei.data_ptr(), int(num_nodes), int(ei.shape[1]), ptr, self._stream())
      self._graph_key = key
      self._n_segments = int(gn_segments) if ptr is None else ptr.size - 1
      self._graph_hold = ei
      self._points_key = None
    return ctx

  def set_points(self, points):
    ctx = self.engine()
    p = points.float().contiguous()
    key = (p.data_ptr(), tuple(p.shape), p._version, self._graph_key)
    if key != self._points_key:
      ctx.set_points(p.data_ptr(), self._stream())
      self._points_key = key
      self._points_hold = p
    return ctx

  def _complete_graph(self, B, V, device):
    key = (B, V, str(device))
    if key not in self._complete_cache:
      r = torch.arange(V, device=device).repeat_interleave(V)
      c = torch.arange(V, device=device).repeat(V)
      off = (torch.arange(B, device=device) * V).repeat_interleave(V * V)
      self._complete_cache[key] = torch.stack([r.repeat(B) + off, c.repeat(B) + off]).long().contiguous()
    return self._complete_cache[key]

  def _run(self, ctx, xt, t, out):
    """One forward at t: a float (dfb_encoder_forward) or timestep_args' (values, index)."""
    if isinstance(t, float):
      ctx.encoder_forward(xt.data_ptr(), t, out.data_ptr(), self._stream())
      return
    values, index = t
    index = index.to(self._device()).contiguous()
    ctx.encoder_forward_timesteps(xt.data_ptr(), values, index.data_ptr(), out.data_ptr(), self._stream())

  # ------------------------------------------------------------------------------------------
  # forward variants (gnn_encoder.py:350-462)
  # ------------------------------------------------------------------------------------------
  def sparse_forward(self, x, graph, timesteps, edge_index, node_ptr=None):
    V, E = x.shape[0], edge_index.shape[1]
    t = timestep_args(timesteps, E, self.use_activation_checkpoint, self.node_embed.weight.device)
    ctx = self.set_graph(edge_index, V, 1, node_ptr)
    self.set_points(x.to(self._device()))
    xt = graph.reshape(-1).float().contiguous().to(self._device())
    out = torch.empty((E, self.out_channels), device=self._device(), dtype=torch.float32)
    self._run(ctx, xt, t, out)
    return out

  def sparse_forward_node_feature_only(self, x, timesteps, edge_index, node_ptr=None):
    V = x.shape[0]
    t = timestep_args(timesteps, V, self.use_activation_checkpoint, self.node_embed.weight.device)
    ctx = self.set_graph(edge_index, V, 1, node_ptr)
    xt = x.reshape(-1).float().contiguous().to(self._device())
    out = torch.empty((V, self.out_channels), device=self._device(), dtype=torch.float32)
    self._run(ctx, xt, t, out)
    return out

  def dense_forward(self, x, graph, timesteps, edge_index=None):
    """One block-diagonal call over the B complete graphs, GroupNorm per sample (gn_segments = B); a timestep per
    sample (:364, :375) indexes each sample's V * V edges."""
    del edge_index
    B, V, _ = x.shape
    t = timestep_args(timesteps, B)
    if not isinstance(t, float):
      t = (t[0], t[1].repeat_interleave(V * V))
    dev = self._device()
    out = torch.empty((B, self.out_channels, V, V), device=dev, dtype=torch.float32)
    ctx = self.set_graph(self._complete_graph(B, V, dev), B * V, B)
    self.set_points(x.reshape(B * V, 2).to(dev))
    xt = graph.reshape(-1).float().contiguous().to(dev)
    flat = torch.empty((B * V * V, self.out_channels), device=dev, dtype=torch.float32)
    self._run(ctx, xt, t, flat)
    out.copy_(flat.reshape(B, V, V, self.out_channels).permute(0, 3, 1, 2))
    return out

  def forward(self, x, timesteps, graph=None, edge_index=None, *, node_ptr=None):
    """node_ptr (sparse TSP and MIS only): node offsets of the instances of a block-diagonal batch, each of which
    then gets its own head GroupNorm.  The dense forward already normalises each sample on its own."""
    if node_ptr is not None and not self.sparse:
      raise ValueError("node_ptr is for sparse graphs: the dense forward already normalises each sample on its own")
    if torch.is_grad_enabled() and not GNNEncoder._warned_no_grad and any(p.requires_grad for p in self.parameters()):
      # inference engine: never builds an autograd graph; make misuse visible (once)
      import warnings
      warnings.warn("difusco_b200.GNNEncoder is an inference engine: outputs carry no grad_fn "
                    "(call it under torch.no_grad(); training is outside this package's scope)")
      GNNEncoder._warned_no_grad = True
    if self.node_feature_only:
      if self.sparse:
        return self.sparse_forward_node_feature_only(x, timesteps, edge_index, node_ptr)
      raise NotImplementedError
    if self.sparse:
      return self.sparse_forward(x, graph, timesteps, edge_index, node_ptr)
    return self.dense_forward(x, graph, timesteps, edge_index)

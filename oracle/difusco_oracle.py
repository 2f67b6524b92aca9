"""CPU oracle for DIFUSCO's denoising-inference hot path.  TEST INFRASTRUCTURE, NOT PRODUCT.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this file.  The product path (difusco_b200/) never does; it fails loudly without its
CUDA library.

What it is: a restatement, in plain PyTorch CPU tensor ops (fp32 by default, fp64 on request as
the "who is closer" arbiter), of the reference's algorithm for
    GNNEncoder.forward (sparse TSP / node-only MIS / dense TSP)  difusco/models/gnn_encoder.py
    timestep / sinusoidal embeddings                             difusco/models/nn.py
    Categorical/GaussianDiffusion tables, InferenceSchedule      difusco/utils/diffusion_schedulers.py
    categorical_posterior / gaussian_posterior                   difusco/pl_meta_model.py
    the test_step denoise loop                                   difusco/pl_tsp_model.py, pl_mis_model.py
Each function cites the reference file:line it follows.  The reference is a floating-point
PyTorch program, so the restatement is torch (not numpy/C): same library kernels, same dtype.

Pinning: the reference ships no tests or golden vectors (SURVEY.md section 4), so the oracle is
pinned against outputs of the reference ITSELF, imported unmodified in the build container by
tests/golden/make_golden.py (via tests/golden/ref_shims.py) and committed as tests/golden/*.npz;
tests/test_oracle_golden.py checks every fixture.  One boundary stays unpinned by upstream:
torch-sparse==0.6.15 / torch-scatter==2.0.9 (environment.yml:131,133) are absent from
/root/reference and from this image; their `sum(SparseTensor, dim=1)` is restated as an exact
row-wise segmented sum (index_add_), which is its documented semantics.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


# ============================================================================================
# diffusion schedules (host side, float64)           difusco/utils/diffusion_schedulers.py
# ============================================================================================
def _betas(T, schedule):
  """:15-23 / :52-60.  linear: linspace(1e-4, 2e-2, T); cosine: Nichol-Dhariwal with offset .008."""
  if schedule == "linear":
    return np.linspace(1e-4, 2e-2, T)
  if schedule == "cosine":
    def cosn(t):
      return np.cos(math.pi * 0.5 * (t / T + 0.008) / (1 + 0.008)) ** 2
    ab = cosn(np.arange(0, T + 1, 1)) / cosn(0)
    return np.clip(1 - (ab[1:] / ab[:-1]), None, 0.999)
  raise ValueError(schedule)


def categorical_tables(T, schedule="linear"):
  """Qs (T,2,2) and cumulative Q_bar (T+1,2,2), Q_bar[0] = I.   :62-72"""
  beta = _betas(T, schedule).reshape(-1, 1, 1)
  Qs = (1 - beta) * np.eye(2)[None] + (beta / 2) * np.ones((1, 2, 2))
  qb = [np.eye(2)]
  for q in Qs:
    qb.append(qb[-1] @ q)
  return Qs, np.stack(qb, 0)


def gaussian_tables(T, schedule="linear"):
  """beta (T), alpha (T+1, alpha[0]=1), alphabar = cumprod(alpha) (T+1).   :25-28"""
  beta = _betas(T, schedule)
  alpha = np.concatenate((np.array([1.0]), 1 - beta))
  return beta, alpha, np.cumprod(alpha)


def inference_schedule(kind, T, steps):
  """[(t1, t2)] for i in range(steps).   :91-109"""
  out = []
  for i in range(steps):
    if kind == "linear":
      a = T - int((float(i) / steps) * T)
      b = T - int((float(i + 1) / steps) * T)
    elif kind == "cosine":
      a = T - int(np.sin((float(i) / steps) * np.pi / 2) * T)
      b = T - int(np.sin((float(i + 1) / steps) * np.pi / 2) * T)
    else:
      raise ValueError("Unknown inference schedule: {}".format(kind))
    out.append((int(np.clip(a, 1, T)), int(np.clip(b, 0, T - 1))))
  return out


# ============================================================================================
# embeddings
# ============================================================================================
def _sincos_interleave(arg):
  """arg (..., F) with arg[..., 2m] == arg[..., 2m+1]: out[2m] = sin, out[2m+1] = cos."""
  out = torch.empty_like(arg)
  out[..., 0::2] = arg[..., 0::2].sin()
  out[..., 1::2] = arg[..., 1::2].cos()
  return out


def _dim_t(nfeat, dtype):
  """temperature ** (2*(i//2)/nfeat), computed in fp32 like the reference (gnn_encoder.py:216-217,
  :243-244) and only then widened, so an fp64 oracle run sees the same frequencies."""
  i = torch.arange(nfeat, dtype=torch.float32)
  ex = 2.0 * torch.div(i, 2, rounding_mode="trunc") / nfeat
  return torch.pow(torch.tensor(10000.0), ex).to(dtype)


def pos_embed_2d(x, hidden):
  """PositionEmbeddingSine(hidden//2, normalize=True): x (V,2) -> (V,hidden).
  gnn_encoder.py:211-227.  First half from x[:,0] ("y_embed"), second half from x[:,1]; scale 2*pi."""
  d = _dim_t(hidden // 2, x.dtype)
  y = (x[:, 0] * (2 * math.pi))[:, None] / d
  xx = (x[:, 1] * (2 * math.pi))[:, None] / d
  return torch.cat([_sincos_interleave(y), _sincos_interleave(xx)], dim=1)


def scalar_embed(s, hidden):
  """ScalarEmbeddingSine / ScalarEmbeddingSine1D(hidden, normalize=False): (...,) -> (..., hidden).
  gnn_encoder.py:242-249, :264-271 (no 2*pi)."""
  return _sincos_interleave(s[..., None] / _dim_t(hidden, s.dtype))


def timestep_embedding(t, dim, dtype):
  """nn.py:103-121: [cos(t f) | sin(t f)], f_m = exp(-ln(1e4) m / half) in fp32."""
  half = dim // 2
  f = torch.exp(-math.log(10000) * torch.arange(0, half, dtype=torch.float32) / half)
  args = t[:, None].float().to(dtype) * f[None].to(dtype)
  return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


# ============================================================================================
# encoder
# ============================================================================================
class Weights(object):
  """state_dict (numpy or torch) -> torch CPU tensors of one dtype; accepts a `model.` prefix."""

  def __init__(self, sd, dtype=torch.float32):
    self.dtype = dtype
    self.t = {}
    for k, v in sd.items():
      if k.startswith("model."):
        k = k[len("model."):]
      self.t[k] = torch.as_tensor(np.asarray(v)).to(dtype)
    self.n_layers = 1 + max(int(k.split(".")[1]) for k in self.t if k.startswith("layers."))
    self.hidden = self.t["node_embed.weight"].shape[0]
    self.out_channels = self.t["out.2.weight"].shape[0]

  def lin(self, name, x):
    return F.linear(x, self.t[name + ".weight"], self.t[name + ".bias"])


def _time_emb(w, timesteps):
  """time_embed = Linear -> ReLU -> Linear on timestep_embedding(t, H).   gnn_encoder.py:311-315,:396"""
  te = timestep_embedding(timesteps, w.hidden, w.dtype)
  return w.lin("time_embed.2", F.relu(w.lin("time_embed.0", te)))


def _layer_sparse(w, l, h, e, row, col, V, aggregation="sum", gather_then_gemm=True):
  """One GNNLayer.forward(mode="direct", sparse=True).   gnn_encoder.py:67-142, aggregate :144-191
  row = edge_index[0] (owner i), col = edge_index[1] (neighbour j)."""
  p = f"layers.{l}."
  Uh = w.lin(p + "U", h)
  if gather_then_gemm:
    Vh = w.lin(p + "V", h[col])            # :99 the reference runs V on E gathered rows
  else:
    Vh = w.lin(p + "V", h)[col]
  Ah, Bh, Ce = w.lin(p + "A", h), w.lin(p + "B", h), w.lin(p + "C", e)
  e_hat = Ah[col] + Bh[row] + Ce           # :110
  msg = torch.sigmoid(e_hat) * Vh          # :112, :163
  agg = torch.zeros((V, h.shape[1]), dtype=h.dtype).index_add_(0, row, msg)   # :177-191 sum
  if aggregation == "mean":
    cnt = torch.zeros(V, dtype=h.dtype).index_add_(0, row, torch.ones_like(row, dtype=h.dtype))
    agg = agg / cnt.clamp(min=1)[:, None]
  elif aggregation == "max":
    agg = torch.full_like(agg, float("-inf")).scatter_reduce(
        0, row[:, None].expand_as(msg), msg, reduce="amax", include_self=True)
    agg = torch.where(torch.isinf(agg), torch.zeros_like(agg), agg)
  elif aggregation != "sum":
    raise ValueError(aggregation)
  H = h.shape[1]
  h_new = F.relu(F.layer_norm(Uh + agg, (H,), w.t[p + "norm_h.weight"], w.t[p + "norm_h.bias"]))
  e_new = F.relu(F.layer_norm(e_hat, (H,), w.t[p + "norm_e.weight"], w.t[p + "norm_e.bias"]))
  return h_new, e_new                      # mode == "direct": no inner residual (:138)


def layer_step(w, l, h, e, row, col, temb, time_on_edge, aggregation="sum", gather_then_gemm=True):
  """Layer l of the encoder loop, gnn_encoder.py:442-449: the GNN layer, its time vector (on e for TSP, on h for
  MIS), the residual on h and per_layer_out on e.  h (V,H), e (E,H) in the caller's edge order -> (h, e)."""
  V, H = h.shape
  h_in, e_in = h, e
  h, e = _layer_sparse(w, l, h_in, e_in, row, col, V, aggregation, gather_then_gemm)
  tv = w.lin(f"time_embed_layers.{l}.1", F.relu(temb))              # :329-337
  if time_on_edge:
    e = e + tv                                                       # :445
  else:
    h = h + tv                                                       # :447
  h = h_in + h                                                       # :448
  o = f"per_layer_out.{l}."
  s = F.silu(F.layer_norm(e, (H,), w.t[o + "0.weight"], w.t[o + "0.bias"]))
  e = e_in + w.lin(o + "2", s)                                       # :449
  return h, e


def _sparse_encoding(w, h, e, row, col, temb, time_on_edge, aggregation="sum", taps=None,
                     gather_then_gemm=True):
  """gnn_encoder.py:416-450 (non-checkpointed branch :442-449)."""
  for l in range(w.n_layers):
    h, e = layer_step(w, l, h, e, row, col, temb, time_on_edge, aggregation, gather_then_gemm)
    if taps is not None:
      taps.append((h, e))
  return h, e


def _head(w, z):
  """GroupNorm32(32, H) with batch dim 1 over ALL rows of z (rows = every edge / node in the call),
  ReLU, 1x1 conv.   gnn_encoder.py:316-322, :400-401, :412-413; nn.py:17-19.   z (R,H) -> (R,out)"""
  H = z.shape[1]
  g = F.group_norm(z.t().reshape(1, H, -1), 32, w.t["out.0.weight"], w.t["out.0.bias"], eps=1e-5)
  g = F.relu(g).reshape(H, -1).t()
  return F.linear(g, w.t["out.2.weight"].reshape(w.out_channels, H), w.t["out.2.bias"])


def encoder_forward_sparse_tsp(w, points, xt, t, edge_index, aggregation="sum", taps=None,
                               gather_then_gemm=True):
  """GNNEncoder.sparse_forward.   gnn_encoder.py:383-402
  points (V,2), xt (E,) float, t (1,) float, edge_index (2,E) int64 -> (E, out)."""
  dt = w.dtype
  points, xt = torch.as_tensor(points).to(dt), torch.as_tensor(xt).to(dt)
  ei = torch.as_tensor(edge_index).long()
  t = torch.as_tensor(t).reshape(-1).to(torch.float32)
  h = w.lin("node_embed", pos_embed_2d(points, w.hidden))           # :394
  e = w.lin("edge_embed", scalar_embed(xt, w.hidden))               # :395
  temb = _time_emb(w, t)                                            # :396
  h, e = _sparse_encoding(w, h, e, ei[0], ei[1], temb, True, aggregation, taps, gather_then_gemm)
  return _head(w, e)                                                # :400-401


def encoder_forward_mis(w, xt, t, edge_index, aggregation="sum", taps=None, gather_then_gemm=True):
  """GNNEncoder.sparse_forward_node_feature_only.   gnn_encoder.py:404-414
  xt (V,) float, t (1,), edge_index (2,E) -> (V, out).  e0 = 0, time vector added on nodes."""
  dt = w.dtype
  xt = torch.as_tensor(xt).to(dt)
  ei = torch.as_tensor(edge_index).long()
  t = torch.as_tensor(t).reshape(-1).to(torch.float32)
  h = w.lin("node_embed", scalar_embed(xt, w.hidden))               # :405
  e = torch.zeros((ei.shape[1], w.hidden), dtype=dt)                # :407
  temb = _time_emb(w, t)
  h, e = _sparse_encoding(w, h, e, ei[0], ei[1], temb, False, aggregation, taps, gather_then_gemm)
  return _head(w, h)                                                # :412-413


def encoder_forward_dense(w, points, graph, t, aggregation="sum"):
  """GNNEncoder.dense_forward.   gnn_encoder.py:350-381
  points (B,V,2), graph = xt (B,V,V) float, t (B,) -> (B, out, V, V).  Written directly on
  (B,V,V,H) tensors (NOT via the sparse path) so that it independently checks the
  complete-graph mapping the CUDA path uses for config C1."""
  dt = w.dtype
  points, graph = torch.as_tensor(points).to(dt), torch.as_tensor(graph).to(dt)
  t = torch.as_tensor(t).reshape(-1).to(torch.float32)
  B, V, _ = points.shape
  H = w.hidden
  h = w.lin("node_embed", torch.stack([pos_embed_2d(points[b], H) for b in range(B)]))
  e = w.lin("edge_embed", scalar_embed(graph, H))                   # (B,V,V,H)
  temb = _time_emb(w, t)                                            # (B,128)
  for l in range(w.n_layers):
    p = f"layers.{l}."
    h_in, e_in = h, e
    Uh, Vh, Ah, Bh = (w.lin(p + n, h) for n in "UVAB")
    e_hat = Ah[:, None, :, :] + Bh[:, :, None, :] + w.lin(p + "C", e)      # :108
    msg = torch.sigmoid(e_hat) * Vh[:, None, :, :]
    if aggregation == "sum":
      agg = msg.sum(dim=2)
    elif aggregation == "mean":
      agg = msg.sum(dim=2) / float(V)       # graph = ones (:365)
    elif aggregation == "max":
      agg = msg.max(dim=2)[0]
    else:
      raise ValueError(aggregation)
    h = F.relu(F.layer_norm(Uh + agg, (H,), w.t[p + "norm_h.weight"], w.t[p + "norm_h.bias"]))
    e = F.relu(F.layer_norm(e_hat, (H,), w.t[p + "norm_e.weight"], w.t[p + "norm_e.bias"]))
    e = e + w.lin(f"time_embed_layers.{l}.1", F.relu(temb))[:, None, None, :]   # :375
    h = h_in + h
    o = f"per_layer_out.{l}."
    e = e_in + w.lin(o + "2", F.silu(F.layer_norm(e, (H,), w.t[o + "0.weight"], w.t[o + "0.bias"])))
  z = e.permute(0, 3, 1, 2)                                         # (B,H,V,V): GN per sample
  g = F.relu(F.group_norm(z, 32, w.t["out.0.weight"], w.t["out.0.bias"], eps=1e-5))
  return F.conv2d(g, w.t["out.2.weight"], w.t["out.2.bias"])        # :380


# ============================================================================================
# posteriors                                             difusco/pl_meta_model.py:102-175
# ============================================================================================
def categorical_posterior_consts(Q_bar, t, target_t):
  """The four fp32 numbers the per-element update needs, from float64 host tables.
  p = c[xt][0] * p0[...,0] + c[xt][1] * p0[...,1]   with, for x = xt in {0,1}:
     c[x][k] = Q[1,x] * Qbar_target[k,1] / Qbar_source[k,x],  Q = inv(Qbar_target) @ Qbar_source
  which is what :113-137 evaluates through one-hot matmuls (each factor cast to fp32 first,
  :115-120, then multiplied and divided in fp32 - reproduced in that order)."""
  Q = (np.linalg.inv(Q_bar[target_t]) @ Q_bar[t]).astype(np.float32)
  qs, qt = Q_bar[t].astype(np.float32), Q_bar[target_t].astype(np.float32)
  c = np.zeros((2, 2), dtype=np.float32)
  for x in (0, 1):
    for k in (0, 1):
      c[x, k] = np.float32(Q[1, x] * qt[k, 1]) / qs[k, x]
  return c


def categorical_posterior(Q_bar, t, target_t, p0, xt, u=None):
  """p0 (...,2) softmax probs, xt (...) in {0,1}.  Returns (p, xt_next).
  t2 > 0: xt_next = (u < clamp(p,0,1)) [torch.bernoulli semantic: 1 iff u < p]; t2 == 0:
  xt_next = clamp(p, min=0) - the heatmap (:139-142).  `u` None -> torch.bernoulli."""
  c = torch.as_tensor(categorical_posterior_consts(Q_bar, t, target_t))
  xi = xt.long()
  p = c[xi, 0].to(p0.dtype) * p0[..., 0] + c[xi, 1].to(p0.dtype) * p0[..., 1]
  if target_t > 0:
    pc = p.clamp(0, 1)
    nxt = torch.bernoulli(pc) if u is None else (torch.as_tensor(u).to(pc.dtype) < pc).to(pc.dtype)
  else:
    nxt = p.clamp(min=0)
  return p, nxt


def gaussian_posterior_consts(beta, alpha, alphabar, t, target_t, inference_trick="ddim"):
  """xt_next = a * xt + b * pred (+ c * z).   :160-174
  ddim (t > 1):  a = sqrt(ab_g/ab_s), b = sqrt(1-ab_g) - a*sqrt(1-ab_s), c = 0
  ddpm (trick None or t <= 1): a = 1/sqrt(alpha_t), b = -a*(1-alpha_t)/sqrt(1-ab_t),
                               c = sqrt(beta[t-1]*(1-ab[t-1])/(1-ab[t]))  (= 0 at t = 1)."""
  if inference_trick is None or t <= 1:
    at = alpha[t]
    a = float(1 / np.sqrt(at))
    b1 = float((1 - at) / np.sqrt(1 - alphabar[t]))
    c = float(np.sqrt(beta[t - 1] * (1 - alphabar[t - 1]) / (1 - alphabar[t])))
    return ("ddpm", a, b1, c)
  if inference_trick == "ddim":
    a = float(np.sqrt(alphabar[target_t] / alphabar[t]))
    b1 = float(np.sqrt(1 - alphabar[t]))
    b2 = float(np.sqrt(1 - alphabar[target_t]))
    return ("ddim", a, b1, b2)
  raise ValueError("Unknown inference trick {}".format(inference_trick))


def gaussian_posterior(beta, alpha, alphabar, t, target_t, pred, xt, inference_trick="ddim", z=None):
  kind, a, b1, c = gaussian_posterior_consts(beta, alpha, alphabar, t, target_t, inference_trick)
  if kind == "ddpm":
    z = torch.randn_like(xt) if z is None else torch.as_tensor(z).to(xt.dtype)
    return a * (xt - b1 * pred) + c * z                          # :166-169
  return a * (xt - b1 * pred) + c * pred                         # :171-172  (c = sqrt(1-ab_g))


# ============================================================================================
# the denoise loop                    pl_tsp_model.py:185-222, pl_mis_model.py:156-192
# ============================================================================================
def denoise(w, task, diffusion_type, edge_index, xt0, points=None, T=1000, schedule="linear",
            inference_schedule_kind="cosine", steps=50, inference_trick="ddim", uniforms=None,
            forced_xt=None, record=None, gather_then_gemm=True):
  """Runs the test_step loop up to the heatmap (the device->host boundary at pl_tsp_model.py:219-222).
  task "tsp" (sparse) or "mis".  xt0: categorical {0,1} or gaussian float.
  uniforms: list (per step) of U[0,1) arrays injected instead of torch.bernoulli.
  forced_xt: list of per-step xt inputs (teacher forcing, SURVEY.md section 7 H2).
  record: list receiving dict(xt_in, net_out, p, xt_out) per step.
  Returns the raw final xt (categorical: clamp(p,min=0); gaussian: xt) - the caller applies the
  +1e-6 / *0.5+0.5 host-side post-map (pl_tsp_model.py:219-222)."""
  sched = inference_schedule(inference_schedule_kind, T, steps)
  if diffusion_type == "categorical":
    _, Q_bar = categorical_tables(T, schedule)
  else:
    beta, alpha, alphabar = gaussian_tables(T, schedule)
  xt = torch.as_tensor(xt0).to(w.dtype)
  ei = torch.as_tensor(edge_index).long()
  for i, (t1, t2) in enumerate(sched):
    if forced_xt is not None:
      xt = torch.as_tensor(forced_xt[i]).to(w.dtype)
    tt = torch.tensor([float(t1)])
    if task == "tsp":
      out = encoder_forward_sparse_tsp(w, points, xt, tt, ei, gather_then_gemm=gather_then_gemm)
    else:
      out = encoder_forward_mis(w, xt, tt, ei, gather_then_gemm=gather_then_gemm)
    rec = {"xt_in": xt, "net_out": out, "t1": t1, "t2": t2}
    if diffusion_type == "categorical":
      p0 = out.softmax(dim=-1)                                    # pl_tsp_model.py:135
      u = None if uniforms is None else uniforms[i]
      p, xt = categorical_posterior(Q_bar, t1, t2, p0, xt, u)
      rec["p"] = p
    else:
      xt = gaussian_posterior(beta, alpha, alphabar, t1, t2, out.squeeze(1), xt, inference_trick,
                              z=torch.zeros_like(xt))             # ddpm noise coefficient is 0 at t=1
    rec["xt_out"] = xt
    if record is not None:
      record.append(rec)
  return xt

"""Generate tests/golden/fwd_tsteps.npz: the encoder forward with a timestep per element, as the UNMODIFIED
reference's training steps (/root/reference/difusco) run it.

Run in the build container only, like make_golden.py, whose reference import and helpers it reuses:
    python tests/golden/make_golden_timesteps.py
The reference's own categorical_training_step / gaussian_training_step run on seeded inputs; a forward hook takes the
encoder's arguments and output, and the returned loss is recorded.
"""
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden import (make_mis_model, make_tsp_model, ref_encoder, save, sd_torch,  # noqa: E402
                         syn)


class Batch(object):
  """Stand-in for the torch_geometric Batch the reference's sparse training steps read (graph_data.x, .edge_index,
  .edge_attr): the block-diagonal tensors as attributes."""

  def __init__(self, **kw):
    self.__dict__.update(kw)


class FixedT(object):
  """np.random.randint of the reference's training steps (the timestep draw, pl_tsp_model.py:45,47,
  pl_mis_model.py:45,76) returns the given timesteps, so that a case can pin chosen values such as t = 1 and 1000.
  Every other draw (the diffusion sample, the xt jitter) stays the seeded torch generator's."""

  def __init__(self, t):
    self.t = np.asarray(t, dtype=int)

  def __enter__(self):
    self.orig = np.random.randint

    def fake(lo, hi, size, *a, **k):
      assert size == self.t.size and lo <= self.t.min() and self.t.max() < hi, (lo, hi, size, self.t)
      return self.t.copy()
    np.random.randint = fake
    return self

  def __exit__(self, *a):
    np.random.randint = self.orig


def training_step_io(model, batch, t):
  """The reference's own training step on `batch` with timesteps t, torch seeded with 0: (encoder positional
  arguments, keyword arguments, output, loss), taken with a forward hook exactly as the step passes them."""
  seen = {}

  def hook(mod, args, kwargs, out):
    seen["args"] = [a.clone() if torch.is_tensor(a) else a for a in args]
    seen["kwargs"] = {k: v.clone() for k, v in kwargs.items() if torch.is_tensor(v)}
    seen["out"] = out.clone()
  h = model.model.register_forward_hook(hook, with_kwargs=True)
  torch.manual_seed(0)
  with FixedT(t):
    loss = model.training_step(batch, 0)
  h.remove()
  return seen["args"], seen["kwargs"], seen["out"].numpy(), float(loss)


def gen_timesteps():
  """A timestep per element, as the reference's training steps run the encoder (pl_tsp_model.py:41-115,
  pl_mis_model.py:41-104), the checkpointed sparse forward (gnn_encoder.py:429) and one graph with an independent
  timestep per edge.  Weights: synthetic seed 0 (out_channels 2) for categorical, seed 1 (out_channels 1) for
  Gaussian."""
  tmp = tempfile.mkdtemp()
  out = {}
  w2 = syn.make_encoder_weights(seed=0, out_channels=2)
  w1 = syn.make_encoder_weights(seed=1, out_channels=1)
  # 1 and 4. sparse TSP, categorical, 3 graphs of 40 nodes, K = 8: one t per graph repeated over its edges, jittered
  # xt, edge_index handed over as float (pl_tsp_model.py:71); once more with use_activation_checkpoint=True
  N, K, B = 40, 8, 3
  pts, ei = syn.tsp_sparse_batch(N, K, B, seed=2024)
  labels = (np.random.default_rng(7).random(ei.shape[1]) < 2.0 / K).astype(np.int64)
  batch = (None, Batch(x=torch.from_numpy(pts), edge_index=torch.from_numpy(ei),
                                 edge_attr=torch.from_numpy(labels)),
           torch.full((B, 1), N), torch.full((B, 1), N * K), None)
  for name, ckpt in (("tsp_cat", False), ("tsp_ckpt", True)):
    model = make_tsp_model(tmp, diffusion_type="categorical", sparse_factor=K, use_activation_checkpoint=ckpt)
    model.model.load_state_dict(sd_torch(w2), strict=True)
    args, _, o, loss = training_step_io(model, batch, [1, 1000, 517])
    assert args[3].dtype == torch.float32   # the float edge_index of the training step
    out.update({f"{name}/points": args[0].numpy(), f"{name}/t": args[1].numpy(), f"{name}/xt": args[2].numpy(),
                f"{name}/edge_index": args[3].numpy(), f"{name}/labels": labels, f"{name}/out": o,
                f"{name}/loss": np.float64(loss)})
  # 2. dense TSP, Gaussian, B = 3 samples of 12 nodes, one t per sample
  B, V = 3, 12
  tb = np.array([3, 990, 250])
  ptsd = np.stack([syn.tsp_points(V, 4322, b) for b in range(B)])
  adj = (np.random.default_rng(8).random((B, V, V)) < 0.15).astype(np.float32)
  model = make_tsp_model(tmp, diffusion_type="gaussian", sparse_factor=-1)
  model.model.load_state_dict(sd_torch(w1), strict=True)
  args, _, o, loss = training_step_io(model, (None, torch.from_numpy(ptsd), torch.from_numpy(adj), None), tb)
  # the step's MSE target, epsilon of diffusion.sample, drawn again from the same seed and checked against xt
  torch.manual_seed(0)
  x0 = torch.from_numpy(adj) * 2 - 1
  x0 = x0 * (1.0 + 0.05 * torch.rand_like(x0))
  ab = torch.from_numpy(model.diffusion.alphabar[tb]).view(B, 1, 1)
  eps = torch.randn_like(x0)
  assert torch.equal((torch.sqrt(ab) * x0 + torch.sqrt(1.0 - ab) * eps).float(), args[2])
  out.update({"dense_gauss/points": args[0].numpy(), "dense_gauss/t": args[1].numpy(), "dense_gauss/xt": args[2].numpy(),
              "dense_gauss/out": o, "dense_gauss/eps": eps.float().numpy(), "dense_gauss/loss": np.float64(loss)})
  # 3. MIS, categorical and Gaussian, 2 ER graphs: one t per graph repeated over its nodes (repeat_interleave)
  ei, sizes = syn.mis_batch(30, 45, 0.15, 2, seed=6)
  V = sum(sizes)
  tb = np.array([77, 904])
  nl = (np.random.default_rng(9).random(V) < 0.3).astype(np.int64)
  batch = (None, Batch(x=torch.from_numpy(nl), edge_index=torch.from_numpy(ei)), torch.tensor(sizes))
  for name, dt, w in (("mis_cat", "categorical", w2), ("mis_gauss", "gaussian", w1)):
    model = make_mis_model(tmp, diffusion_type=dt)
    model.model.load_state_dict(sd_torch(w), strict=True)
    args, kw, o, loss = training_step_io(model, batch, tb)
    out.update({f"{name}/xt": args[0].numpy(), f"{name}/t": args[1].numpy(), f"{name}/edge_index": kw["edge_index"].numpy(),
                f"{name}/labels": nl, f"{name}/sizes": np.array(sizes), f"{name}/out": o, f"{name}/loss": np.float64(loss)})
    if dt == "gaussian":   # the MSE target, recovered as for the dense case
      torch.manual_seed(0)
      x0 = torch.from_numpy(nl).float() * 2 - 1
      x0 = (x0 * (1.0 + 0.05 * torch.rand_like(x0))).reshape(V, 1, 1)
      ab = torch.from_numpy(model.diffusion.alphabar[np.repeat(tb, sizes)]).view(V, 1, 1)
      eps = torch.randn_like(x0)
      assert torch.equal((torch.sqrt(ab) * x0 + torch.sqrt(1.0 - ab) * eps).reshape(-1).float(), args[0])
      out[f"{name}/eps"] = eps.reshape(-1).float().numpy()
  # 5. one sparse TSP graph, an independent integer t per edge (hundreds of distinct values; E = 873 is not a
  #    multiple of 32, 64 or 128)
  N, K = 97, 9
  pts = syn.tsp_points(N, 555, 0)
  ei = syn.knn_edge_index(pts, K)
  E = ei.shape[1]
  te = np.random.default_rng(10).integers(1, 1001, E).astype(np.float32)
  xt = (syn.initial_noise(E, 12) > 0).astype(np.float32)
  o = ref_encoder(w2, 2, False)(torch.from_numpy(pts), torch.from_numpy(te), torch.from_numpy(xt),
                                torch.from_numpy(ei)).numpy()
  out.update({"tsp_edge_t/points": pts, "tsp_edge_t/edge_index": ei, "tsp_edge_t/t": te, "tsp_edge_t/xt": xt,
              "tsp_edge_t/out": o})
  save("fwd_tsteps", **out)


if __name__ == "__main__":
  gen_timesteps()

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

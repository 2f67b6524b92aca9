"""MISModel: inference-side drop-in for the reference's difusco/pl_mis_model.py (node-only GNN).

  forward(x, t, edge_index)                                               :40-41
  categorical_denoise_step(xt, t, device, edge_index=None, target_t=None) :118-128
  gaussian_denoise_step(xt, t, device, edge_index=None, target_t=None)    :130-140
  test_step(batch, batch_idx, draw=False, split='test')                   :142-209
Greedy MIS decoding (mis_decode_np, :194-196; SURVEY 8f row f4) is `difusco_b200.utils.mis_utils.mis_decode_np`,
applied by test_step exactly as the reference does (best of all samples -> `{split}/solved_cost`).
"""
import numpy as np
import torch

from .pl_meta_model import COMetaModel
from .utils.mis_utils import mis_decode_np


class MISModel(COMetaModel):
  def __init__(self, param_args=None):
    super().__init__(param_args=param_args, node_feature_only=True)

  def forward(self, x, t, edge_index):
    return self.model(x, t, edge_index=edge_index)

  def _denoise_step(self, xt, t, device, edge_index, target_t):
    with torch.no_grad():
      self.model.set_graph(edge_index.long().to(device), xt.shape[0], 1)
      return self._fused_step(xt.float().to(device), t, target_t).reshape(-1)

  def categorical_denoise_step(self, xt, t, device, edge_index=None, target_t=None):
    return self._denoise_step(xt, t, device, edge_index, target_t)

  def gaussian_denoise_step(self, xt, t, device, edge_index=None, target_t=None):
    return self._denoise_step(xt, t, device, edge_index, target_t)

  def denoise_labels(self, edge_index, xt, steps=None, seed=None, record_steps=None, node_ptr=None):
    """xt0 (V,) -> raw final node labels on device, the whole loop fused.  record_steps (step indices or "all"):
    returns (labels, trace) instead, trace as COMetaModel._fused_loop: "xt" / "p" (n_rec, V), "out" (n_rec, V, out).
    node_ptr: node offsets of the graphs of a block-diagonal batch (PyG's Batch.ptr); each graph then gets its own
    head GroupNorm, as if it were denoised alone."""
    steps = steps or self.args.inference_diffusion_steps
    with torch.no_grad():
      dev = self.model._device()
      self.model.set_graph(edge_index.long().to(dev), xt.shape[0], 1, node_ptr)
      x = xt.reshape(-1).float().contiguous().to(dev).clone()
      return self._fused_loop(x, steps, seed, record_steps)

  def test_step(self, batch, batch_idx, draw=False, split="test"):
    device = batch[-1].device
    real_batch_idx, graph_data, point_indicator = batch
    node_labels = graph_data.x
    edge_index = graph_data.edge_index.to(node_labels.device).reshape(2, -1)
    base_edge_index = edge_index
    P = self.args.parallel_sampling
    if P > 1:   # the reference re-duplicates inside the sequential loop (:168-169, a bug for S>1); done once here
      edge_index = self.duplicate_edge_index(edge_index, node_labels.shape[0], device)
    stacked = []
    for _ in range(self.args.sequential_sampling):
      xt = torch.randn_like(node_labels.float())
      if P > 1:
        xt = xt.repeat(P, 1, 1)
        xt = torch.randn_like(xt)
      if self.diffusion_type != "gaussian":
        xt = (xt > 0).long()
      xt = self.denoise_labels(edge_index, xt.reshape(-1).float())
      if self.diffusion_type == "gaussian":
        stacked.append(xt.float().cpu().detach().numpy() * 0.5 + 0.5)
      else:
        stacked.append(xt.float().cpu().detach().numpy() + 1e-6)
    predict_labels = np.concatenate(stacked, axis=0)
    # decode every sample greedily and keep the largest independent set (pl_mis_model.py:194-209)
    import scipy.sparse
    ei_np = base_edge_index.cpu().numpy()
    adj_mat = scipy.sparse.coo_matrix((np.ones_like(ei_np[0]), (ei_np[0], ei_np[1])))
    all_sampling = self.args.sequential_sampling * P
    solved = [mis_decode_np(pl, adj_mat) for pl in np.split(predict_labels, all_sampling)]
    best_solved_cost = np.max([sol.sum() for sol in solved])
    gt_cost = node_labels.cpu().numpy().sum()
    metrics = {f"{split}/gt_cost": gt_cost}
    for k, v in metrics.items():
      self.log(k, v, on_epoch=True, sync_dist=True)
    self.log(f"{split}/solved_cost", best_solved_cost, prog_bar=True, on_epoch=True, sync_dist=True)
    self.last_predict_labels = predict_labels          # raw heatmaps of the last call (not part of the reference API)
    self.last_solved_cost = best_solved_cost
    return metrics

  def validation_step(self, batch, batch_idx):
    return self.test_step(batch, batch_idx, split="val")

"""MISModel: inference-side drop-in for the reference's difusco/pl_mis_model.py (node-only GNN).

  forward(x, t, edge_index)                                               :40-41
  categorical_denoise_step(xt, t, device, edge_index=None, target_t=None) :118-128
  gaussian_denoise_step(xt, t, device, edge_index=None, target_t=None)    :130-140
  test_step(batch, batch_idx, draw=False, split='test')                   :142-209
Greedy MIS decoding (mis_decode_np, :194-196; SURVEY 8f row f4) is `difusco_b200.utils.mis_utils.mis_decode_np`,
applied by test_step exactly as the reference does (best of all samples -> `{split}/solved_cost`).
solve_batch(batch, seeds, split='test') runs test_step for every graph of a collated batch at once, each graph's result
independent of the rest of the batch; solve_batches(batches, seeds, split='test') runs it over a stream of batches with
each batch's decode hidden behind the next batch's loops (COMetaModel.solve_batches).
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

  def denoise_labels(self, edge_index, xt, steps=None, seed=None, record_steps=None, node_ptr=None,
                     instance_seeds=None):
    """xt0 (V,) -> raw final node labels on device, the whole loop fused.  record_steps (step indices or "all"):
    returns (labels, trace) instead, trace as COMetaModel._fused_loop: "xt" / "p" (n_rec, V), "out" (n_rec, V, out).
    node_ptr: node offsets of the graphs of a block-diagonal batch (PyG's Batch.ptr); each graph then gets its own
    head GroupNorm, as if it were denoised alone.  instance_seeds (one int per graph of node_ptr, or one for the call):
    sampling keyed per graph, so that each graph's labels are those it gets alone with that seed."""
    steps = steps or self.args.inference_diffusion_steps
    with torch.no_grad():
      dev = self.model._device()
      self.model.set_graph(edge_index.long(), xt.shape[0], 1, node_ptr)   # host edges: staged without a wait
      x = xt.reshape(-1).float().contiguous().to(dev).clone()
      return self._fused_loop(x, steps, seed, record_steps, instance_seeds)

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

  def _solve_enqueue(self, batch, seeds):
    """solve_batch's device half for a collated batch (index, graph, point_indicator): graph.x / graph.edge_index
    concatenated in graph order with node offsets, point_indicator the node counts.  Each graph's parallel_sampling
    replicas share one GroupNorm as in test_step; all graphs run in one fused loop per sequential round, enqueued with
    its labels copied to pinned host memory.  Checks the batch and the seeds before any device work, and waits for no
    earlier loop.  -> the job _solve_finish decodes."""
    _, graph_data, point_indicator = batch
    labels = graph_data.x.reshape(-1)
    edge_index = graph_data.edge_index.reshape(2, -1)
    sizes = [int(c) for c in point_indicator.reshape(-1)]
    if sum(sizes) != labels.shape[0] or min(sizes, default=0) < 1:
      raise ValueError(f"point_indicator {sizes} does not match {labels.shape[0]} nodes")
    gens = self._solve_seeds(seeds, len(sizes))
    node0 = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    ei = edge_index.cpu().numpy()
    owner = np.searchsorted(node0, ei[0], side="right") - 1
    if ei.size and (owner != np.searchsorted(node0, ei[1], side="right") - 1).any():
      raise ValueError("an edge joins two graphs of the batch")
    P, rounds = self.args.parallel_sampling, self.args.sequential_sampling
    dev = self.model._device()
    local = [np.ascontiguousarray(ei[:, owner == i] - node0[i]) for i in range(len(sizes))]
    ptr = np.concatenate([[0], np.cumsum([P * n for n in sizes])]).astype(np.int64)
    edges = torch.cat([self.duplicate_edge_index(torch.from_numpy(e), n, "cpu") + int(ptr[i])
                       for i, (e, n) in enumerate(zip(local, sizes))], 1)
    outs = []
    for _ in range(rounds):
      round_seeds, noise = [], []
      for g, n in zip(gens, sizes):
        round_seeds.append(self._round_seed(g))
        z = torch.randn(P * n, generator=g)
        noise.append((z > 0).float() if self.diffusion_type != "gaussian" else z)
      xt = self._pinned_to_device(torch.cat(noise), dev)
      outs.append(self._to_host_async(self.denoise_labels(edges, xt, node_ptr=ptr, instance_seeds=round_seeds)))
    return dict(sizes=sizes, local=local, ptr=ptr, outs=outs,
                gt=[labels[node0[i]:node0[i + 1]].cpu().numpy().sum() for i in range(len(sizes))])

  def _solve_finish(self, job, split):
    """solve_batch's host half: mis_decode_np per graph and sample, the metrics and the logs."""
    import scipy.sparse
    P, rounds = self.args.parallel_sampling, self.args.sequential_sampling
    sizes, local = job["sizes"], job["local"]
    samples = [[] for _ in sizes]
    for host, ev in job["outs"]:
      ev.synchronize()
      xt = host.float().numpy()
      xt = xt * 0.5 + 0.5 if self.diffusion_type == "gaussian" else xt + 1e-6
      for i, part in enumerate(np.split(xt, job["ptr"][1:-1])):
        samples[i].append(part)
    out, costs = [], []
    for i, n in enumerate(sizes):
      adj_mat = scipy.sparse.coo_matrix((np.ones_like(local[i][0]), (local[i][0], local[i][1])))
      predict_labels = np.concatenate(samples[i], axis=0)
      solved = [mis_decode_np(pl, adj_mat) for pl in np.split(predict_labels, rounds * P)]
      best = np.max([sol.sum() for sol in solved])
      metrics = {f"{split}/gt_cost": job["gt"][i]}
      # batch_size=1: each value is one graph's, as test_step logs it; Lightning would otherwise weight it by the size
      # it infers from the collated batch
      for k, v in metrics.items():
        self.log(k, v, on_epoch=True, sync_dist=True, batch_size=1)
      self.log(f"{split}/solved_cost", best, prog_bar=True, on_epoch=True, sync_dist=True, batch_size=1)
      out.append(metrics)
      costs.append(best)
    self.last_solved_costs = costs      # per-graph artefact of the last call (not part of the metrics)
    return out

  def validation_step(self, batch, batch_idx):
    return self.test_step(batch, batch_idx, split="val")

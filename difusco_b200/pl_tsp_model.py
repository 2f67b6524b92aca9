"""TSPModel: inference-side drop-in for the reference's difusco/pl_tsp_model.py.

Same method names and signatures on the denoise path:
  forward(x, adj, t, edge_index)                                              :38-39
  categorical_denoise_step(points, xt, t, device, edge_index=None, target_t=None)   :122-138
  gaussian_denoise_step(points, xt, t, device, edge_index=None, target_t=None)      :140-151
  test_step(batch, batch_idx, split='test')                                   :153-256
plus solve_batch(batch, seeds, split='test'): test_step for the n instances of a collated batch in one fused loop per
sequential round and one multi-instance 2-opt, each instance's result independent of the rest of the batch, and
solve_batches(batches, seeds, split='test'): solve_batch over a stream of batches, with each batch's decode hidden behind
the next batch's loops (COMetaModel.solve_batches).
test_step runs the reference's loop (:185-222) as ONE fused device loop, then the reference's decode
(:227-256; SURVEY 8f rows f2/f3): merge_tours (host C++), batched 2-opt (CUDA), TSPEvaluator - and returns the
reference's metrics dict.  `--save_numpy_heatmap` (:224-225, :258-267) is honoured.
"""
import os

import numpy as np
import torch

from .pl_meta_model import COMetaModel
from .utils.tsp_utils import TSPEvaluator, batched_two_opt_instances, batched_two_opt_torch, merge_tours


def _shape_trace(trace, shape):
  """The (n_rec, N[, out_channels]) record tensors reshaped to (n_rec, *shape[, out_channels])."""
  out = dict(trace)
  for k in ("xt", "p"):
    if k in out:
      out[k] = out[k].reshape((-1,) + tuple(shape))
  out["out"] = out["out"].reshape((-1,) + tuple(shape) + (out["out"].shape[-1],))
  return out


class TSPModel(COMetaModel):
  def __init__(self, param_args=None):
    super().__init__(param_args=param_args, node_feature_only=False)

  def forward(self, x, adj, t, edge_index):
    return self.model(x, t, adj, edge_index)

  # ------------------------------------------------------------------------------------
  def _prepare(self, points, edge_index, device, node_ptr=None):
    """Make self.model's engine hold this call's graph + coordinates; returns dense batch B or 0.  Host tensors go to
    the engine as they are: it stages them through pinned memory without waiting for the loops already enqueued."""
    if self.sparse:
      V = points.shape[0]
      self.model.set_graph(edge_index.long(), V, 1, node_ptr)
      self.model.set_points(points.float())
      return 0
    if node_ptr is not None:
      raise ValueError("node_ptr is for sparse graphs: the dense path already normalises each sample on its own")
    B, V, _ = points.shape
    self.model.set_graph(self.model._complete_graph(B, V, torch.device("cpu")), B * V, B)
    self.model.set_points(points.reshape(B * V, 2).float())
    return B

  def _denoise_step(self, points, xt, t, device, edge_index, target_t):
    with torch.no_grad():
      self._prepare(points, edge_index, device)
      shape = xt.shape
      out = self._fused_step(xt.float().to(device), t, target_t)
      return out.reshape(-1) if self.sparse else out.reshape(shape)

  def categorical_denoise_step(self, points, xt, t, device, edge_index=None, target_t=None):
    return self._denoise_step(points, xt, t, device, edge_index, target_t)

  def gaussian_denoise_step(self, points, xt, t, device, edge_index=None, target_t=None):
    return self._denoise_step(points, xt, t, device, edge_index, target_t)

  # ------------------------------------------------------------------------------------
  def denoise_heatmap(self, points, edge_index, xt, steps=None, seed=None, record_steps=None, node_ptr=None,
                      instance_seeds=None):
    """xt0 -> raw final xt on device, the whole loop fused (no host sync inside).

    node_ptr (sparse only): node offsets of the instances of a block-diagonal batch (PyG's Batch.ptr); each instance
    then gets its own head GroupNorm, as if it were denoised alone.

    instance_seeds (one int per instance of node_ptr, or per sample of a dense batch): sampling keyed per instance, so
    that each instance's heat map is the one it gets alone with seed=instance_seeds[i], whatever else is in the call.
    Without it the draws are keyed by an element's position in the call.

    record_steps (step indices or "all"): returns (heatmap, trace) instead, trace as COMetaModel._fused_loop with
    each tensor shaped like xt after its leading step dimension: (n_rec, E) sparse, (n_rec, B, V, V) dense; "out"
    has a trailing out_channels dimension."""
    steps = steps or self.args.inference_diffusion_steps
    with torch.no_grad():
      dev = self.model._device()
      self._prepare(points, edge_index, dev, node_ptr)
      x = xt.reshape(-1).float().contiguous().to(dev).clone()
      if record_steps is None:
        self._fused_loop(x, steps, seed, instance_seeds=instance_seeds)
        return x.reshape(xt.shape)
      _, trace = self._fused_loop(x, steps, seed, record_steps, instance_seeds)
      return x.reshape(xt.shape), _shape_trace(trace, xt.shape)

  # ------------------------------------------------------------------------------------
  # test_step = unpack -> (sample, fused denoise loop, decode) x sequential_sampling -> metrics
  # ------------------------------------------------------------------------------------
  def _unpack(self, batch):
    """The two batch layouts of the reference's datasets (pl_tsp_model.py:158-171)."""
    if self.sparse:
      index, graph, node_counts, _, gt_tour = batch
      coords = graph.x.reshape((-1, 2))
      edges = graph.edge_index.reshape((2, -1))
      n_graphs = node_counts.shape[0]
      labels = graph.edge_attr.reshape((n_graphs, edges.shape[1] // n_graphs))
      return index, coords, edges, labels, gt_tour, coords.cpu().numpy(), edges.cpu().numpy()
    index, coords, labels, gt_tour = batch
    return index, coords, None, labels, gt_tour, coords.cpu().numpy()[0], None

  def _initial_noise(self, like, copies):
    """pl_tsp_model.py:186-199: the noise tensor is drawn twice when parallel sampling is on (only the second
    draw is used); kept so torch's generator advances exactly as in the reference."""
    noise = torch.randn_like(like.float())
    if copies > 1:
      noise = noise.repeat(copies, 1) if self.sparse else noise.repeat(copies, 1, 1)
      noise = torch.randn_like(noise)
    if self.diffusion_type != "gaussian":
      noise = (noise > 0).long()
    return (noise.reshape(-1) if self.sparse else noise).float()

  def _heatmap_to_numpy(self, xt):
    if self.diffusion_type == "gaussian":
      return xt.cpu().detach().numpy() * 0.5 + 0.5          # :219-220
    return xt.float().cpu().detach().numpy() + 1e-6         # :221-222

  def test_step(self, batch, batch_idx, split="test"):
    device = batch[-1].device
    index, coords, edges, labels, gt_tour, np_points, np_edge_index = self._unpack(batch)
    copies, rounds = self.args.parallel_sampling, self.args.sequential_sampling
    if copies > 1:
      coords = coords.repeat(copies, 1) if self.sparse else coords.repeat(copies, 1, 1)
      if self.sparse:
        edges = self.duplicate_edge_index(edges, np_points.shape[0], device)
    two_opt_cap = getattr(self.args, "two_opt_iterations", 1000)
    ns, merge_iterations = 0, 0
    heatmaps, refined = [], []
    for _ in range(rounds):
      heat = self._heatmap_to_numpy(self.denoise_heatmap(coords, edges, self._initial_noise(labels, copies)))
      heatmaps.append(heat)
      if getattr(self.args, "save_numpy_heatmap", False):
        self.run_save_numpy_heatmap(heat, np_points, index, split)
      tours, merge_iterations = merge_tours(heat, np_points, np_edge_index, sparse_graph=self.sparse,
                                            parallel_sampling=copies, exact=getattr(self.args, "exact_merge", True))
      better, ns = batched_two_opt_torch(np_points.astype("float64"), np.array(tours).astype("int64"),
                                         max_iterations=two_opt_cap, device=device)
      refined.append(better)
    refined = np.concatenate(refined, axis=0)
    scorer = TSPEvaluator(np_points)
    best = np.min([scorer.evaluate(refined[i]) for i in range(copies * rounds)])
    metrics = {f"{split}/gt_cost": scorer.evaluate(gt_tour.cpu().numpy().reshape(-1)),
               f"{split}/2opt_iterations": ns, f"{split}/merge_iterations": merge_iterations}
    for name, value in metrics.items():
      self.log(name, value, on_epoch=True, sync_dist=True)
    self.log(f"{split}/solved_cost", best, prog_bar=True, on_epoch=True, sync_dist=True)
    # not part of the reference's return value: artefacts of the last call for callers that want them
    self.last_heatmap = heatmaps[0] if rounds == 1 else np.stack(heatmaps)
    self.last_solved_tours, self.last_solved_cost = refined, best
    return metrics

  # ------------------------------------------------------------------------------------
  # solve_batch: test_step for every instance of a collated batch at once
  # ------------------------------------------------------------------------------------
  def _instances(self, batch):
    """n instances collated together -> per instance (points (n_i, 2) tensor, local edge_index (2, E_i) tensor or None,
    ground-truth tour (n_i + 1,) numpy).  Sparse: TSPGraphDataset items collated by PyG (graph.x / graph.edge_index
    concatenated in instance order with node offsets, point_indicator / edge_indicator the per-instance node and edge
    counts, tours stacked (n, n_i + 1) or concatenated).  Dense: (index, points (B, N, 2), adj, tours (B, N + 1))."""
    if not self.sparse:
      _, coords, _, gt = batch
      if coords.dim() != 3 or coords.shape[-1] != 2:
        raise ValueError(f"dense points must be (B, N, 2), got {tuple(coords.shape)}")
      gt = gt.reshape(coords.shape[0], -1).cpu().numpy()
      return [(coords[i], None, gt[i]) for i in range(coords.shape[0])]
    _, graph, point_indicator, edge_indicator, gt = batch
    coords = graph.x.reshape((-1, 2))
    edges = graph.edge_index.reshape((2, -1))
    nodes = [int(c) for c in point_indicator.reshape(-1)]
    counts = [int(c) for c in edge_indicator.reshape(-1)]
    if len(nodes) != len(counts) or sum(nodes) != coords.shape[0] or sum(counts) != edges.shape[1]:
      raise ValueError(f"point_indicator {nodes} / edge_indicator {counts} do not match {coords.shape[0]} nodes and "
                       f"{edges.shape[1]} edges")
    gt = gt.reshape(-1).cpu().numpy()
    if gt.size != sum(nodes) + len(nodes):
      raise ValueError(f"{gt.size} tour entries for instances of {nodes} nodes")
    out, v0, e0 = [], 0, 0
    for n, e in zip(nodes, counts):
      ei = edges[:, e0:e0 + e] - v0
      if e and (int(ei.min()) < 0 or int(ei.max()) >= n):
        raise ValueError("each instance's edges must follow the previous instance's, inside its own nodes")
      out.append((coords[v0:v0 + n], ei, gt[v0 + len(out):v0 + len(out) + n + 1]))
      v0, e0 = v0 + n, e0 + e
    return out

  def _solve_enqueue(self, batch, seeds):
    """solve_batch's device half: each instance's parallel_sampling replicas in one fused denoise loop per sequential
    round (the replicas of a sparse instance share one GroupNorm, as in test_step; a dense replica is a sample of its
    own), every round enqueued with its heat map copied to pinned host memory.  Checks the batch and the seeds before
    any device work, and waits for no earlier loop.  -> the job _solve_finish decodes."""
    if getattr(self.args, "save_numpy_heatmap", False):
      raise NotImplementedError("solve_batch does not save heat maps: use test_step for --save_numpy_heatmap")
    inst = self._instances(batch)
    gens = self._solve_seeds(seeds, len(inst))
    copies, rounds = self.args.parallel_sampling, self.args.sequential_sampling
    dev = self.model._device()
    # copies: _solve_finish runs after the next batch was drawn, and a loader may refill its tensors in place
    np_points = [p.cpu().numpy().copy() for p, _, _ in inst]
    np_edges = [None if e is None else e.cpu().numpy().copy() for _, e, _ in inst]
    if self.sparse:
      sizes = [p.shape[0] for p in np_points]
      ptr = np.concatenate([[0], np.cumsum([copies * n for n in sizes])]).astype(np.int64)
      coords = torch.cat([p.cpu().repeat(copies, 1) for p, _, _ in inst])
      edges = torch.cat([self.duplicate_edge_index(torch.from_numpy(e), n, "cpu") + int(ptr[i])
                         for i, (e, n) in enumerate(zip(np_edges, sizes))], 1)
      lens = [copies * e.shape[1] for e in np_edges]
    else:
      ptr = None
      coords = torch.stack([p.cpu() for p, _, _ in inst]).repeat_interleave(copies, 0)
      edges = None
      lens = [copies] * len(inst)
    heats = []
    for _ in range(rounds):
      round_seeds, noise = [], []
      for g, n_el in zip(gens, lens):
        round_seeds += [self._round_seed(g) for _ in range(1 if self.sparse else copies)]
        shape = (n_el,) if self.sparse else (copies,) + tuple(inst[0][0].shape[:1]) * 2
        z = torch.randn(shape, generator=g)
        noise.append((z > 0).float() if self.diffusion_type != "gaussian" else z)
      xt = self._pinned_to_device(torch.cat(noise), dev)
      heats.append(self._to_host_async(self.denoise_heatmap(coords, edges, xt, node_ptr=ptr,
                                                            instance_seeds=round_seeds)))
    return dict(dev=dev, gt=[t.copy() for _, _, t in inst], np_points=np_points, np_edges=np_edges, lens=lens, heats=heats)

  def _solve_finish(self, job, split):
    """solve_batch's host half: merge_tours per instance and round on a thread pool, one batched_two_opt_instances,
    the metrics and the logs."""
    copies, rounds = self.args.parallel_sampling, self.args.sequential_sampling
    np_points, np_edges = job["np_points"], job["np_edges"]
    heats = []
    for host, ev in job["heats"]:
      ev.synchronize()
      heats.append(np.split(self._heatmap_to_numpy(host), np.cumsum(job["lens"])[:-1]))
    exact = getattr(self.args, "exact_merge", True)
    jobs = [(i, r) for i in range(len(np_points)) for r in range(rounds)]

    def merge(job):
      i, r = job
      return merge_tours(heats[r][i], np_points[i], np_edges[i], sparse_graph=self.sparse, parallel_sampling=copies,
                         exact=exact)

    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 1)) as pool:
      merged = list(pool.map(merge, jobs))
    dev = job["dev"]
    with torch.cuda.stream(self._two_opt_stream(dev)):
      refined, iterations = batched_two_opt_instances(
          [np_points[i].astype("float64") for i, _ in jobs], [np.array(t).astype("int64") for t, _ in merged],
          max_iterations=getattr(self.args, "two_opt_iterations", 1000), device=dev)
    out, tours_out, costs = [], [], []
    for i in range(len(np_points)):
      k = [jobs.index((i, r)) for r in range(rounds)]
      solved = np.concatenate([refined[j] for j in k], axis=0)
      scorer = TSPEvaluator(np_points[i])
      best = np.min([scorer.evaluate(solved[s]) for s in range(copies * rounds)])
      metrics = {f"{split}/gt_cost": scorer.evaluate(job["gt"][i]),
                 f"{split}/2opt_iterations": iterations[k[-1]], f"{split}/merge_iterations": merged[k[-1]][1]}
      # batch_size=1: each value is one instance's, as test_step logs it; Lightning would otherwise weight it by the
      # size it infers from the collated batch
      for name, value in metrics.items():
        self.log(name, value, on_epoch=True, sync_dist=True, batch_size=1)
      self.log(f"{split}/solved_cost", best, prog_bar=True, on_epoch=True, sync_dist=True, batch_size=1)
      out.append(metrics)
      tours_out.append(solved)
      costs.append(best)
    # not part of the metrics: per-instance artefacts of the last call
    self.last_solved_tours, self.last_solved_costs = tours_out, costs
    return out

  def run_save_numpy_heatmap(self, adj_mat, np_points, real_batch_idx, split):
    """--save_numpy_heatmap (pl_tsp_model.py:258-267): <save_dir>/<name>/<version>/numpy_heatmap/{split}-heatmap-<idx>.npy
    and {split}-points-<idx>.npy, the input format of tsp_mcts/convert_numpy_to_txt.py."""
    if self.args.parallel_sampling > 1 or self.args.sequential_sampling > 1:
      raise NotImplementedError("Save numpy heatmap only support single sampling")
    logger = getattr(self, "logger", None)
    root = (os.path.join(logger.save_dir, logger.name, logger.version) if logger is not None
            else getattr(self.args, "storage_path", "."))
    target = os.path.join(root, "numpy_heatmap")
    os.makedirs(target, exist_ok=True)
    tag = real_batch_idx.cpu().numpy().reshape(-1)[0]
    np.save(os.path.join(target, f"{split}-heatmap-{tag}.npy"), adj_mat)
    np.save(os.path.join(target, f"{split}-points-{tag}.npy"), np_points)

  def validation_step(self, batch, batch_idx):
    return self.test_step(batch, batch_idx, split="val")

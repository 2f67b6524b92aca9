"""Solving a test set in batches: n x test_step against solve_batch and solve_batches, and the multi-instance 2-opt.

    python scripts/bench_solve.py [--rounds 3] [--steps 50]

Workloads, timed end to end (denoise loops, merge, 2-opt, metrics) with synthetic weights and a synchronise at the end:
  64 x TSP-500 k=50 (sparse) with parallel_sampling 1 and 4, 256 x TSP-50 (dense) and 32 x MIS ER-[700, 800] p=0.15,
  each solved as
    single        one test_step per instance (TSP-500 P=1 and TSP-50 only)
    batchB        solve_batch over batches of B instances, one batch after another
    pipelinedB    solve_batches over the same batches: each batch's decode hidden behind the next batch's loops
    loop_onlyB    the same batches' inputs and denoise loops alone, no decode: the ceiling of pipelinedB
  with B = 16 and 64 (16 and 32 for MIS).  For TSP-500 P=4 also
    pipelinedB_between  pipelinedB with each batch's 2-opt on the loops' stream, after the next batch's loops that are
                        already enqueued there, instead of beside them
  and the decode alone, on the tours merge_tours gives for the TSP-500 instances' heat maps:
    two_opt_each       one dfb_two_opt call per instance
    two_opt_instances  one dfb_two_opt_instances call for all of them
Batches are built as CPU tensors, as a DataLoader yields them: a device tensor in a batch would make building it, and
reading it back, wait for the loops already enqueued.  --select REGEX times only the "workload: way" pairs it matches.
The ways are alternated within each round (the order rotates from round to round), so clock and load drift hit them
alike.  Every way is run once before timing (graphs prepared, loops captured).  Prints one JSON line per workload:
instances/s per way (median over the rounds, and every round), the card's name and power limit, and the median SM
clock sampled during the timed runs."""
import argparse
import json
import re
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench import ClockSampler  # noqa: E402
from bench_instances import card  # noqa: E402
from difusco_b200 import synthetic as syn  # noqa: E402
from difusco_b200.utils import tsp_utils as tu  # noqa: E402
import gpu_util as G  # noqa: E402


class _Graph(object):
  def __init__(self, **kw):
    self.__dict__.update(kw)


def sparse_batch(parts):
  ptr = syn.node_ptr([p.shape[0] for p, _ in parts])
  x = torch.from_numpy(np.concatenate([p for p, _ in parts])).float()
  ei = torch.from_numpy(np.concatenate([e + ptr[i] for i, (_, e) in enumerate(parts)], 1))
  gt = torch.from_numpy(np.concatenate([np.concatenate([np.arange(p.shape[0]), [0]]) for p, _ in parts]))
  return (torch.arange(len(parts)), _Graph(x=x, edge_index=ei, edge_attr=torch.zeros((ei.shape[1], 1), dtype=torch.bool)),
          torch.tensor([p.shape[0] for p, _ in parts]), torch.tensor([e.shape[1] for _, e in parts]), gt)


def dense_batch(pts):
  n = pts.shape[1]
  gt = np.tile(np.concatenate([np.arange(n), [0]]), (pts.shape[0], 1))
  return torch.arange(pts.shape[0]), torch.from_numpy(pts), torch.zeros(pts.shape[0], n, n), torch.from_numpy(gt)


def mis_batch(graphs, labels):
  ptr = syn.node_ptr([l.shape[0] for l in labels])
  ei = torch.from_numpy(np.concatenate([g + ptr[i] for i, g in enumerate(graphs)], 1))
  return (torch.arange(len(graphs)), _Graph(x=torch.from_numpy(np.concatenate(labels)), edge_index=ei),
          torch.tensor([l.shape[0] for l in labels]))


def solve_ways(model, batches_of, n, sizes=(16, 64), single=True, between=False):
  """way -> callable solving all n instances."""
  def split(b):
    return [list(range(s, min(n, s + b))) for s in range(0, n, b)]

  def one_by_one():   # test_step runs its 2-opt on the device of the batch's last tensor, as the reference does
    for i in range(n):
      b = batches_of([i])
      model.test_step(b[:-1] + (b[-1].cuda(),), i)

  def batched(b):
    return lambda: [model.solve_batch(batches_of(idx), idx) for idx in split(b)]

  def pipelined(b, beside=True):
    def run():
      model._two_opt_beside_loop = beside
      try:
        return list(model.solve_batches((batches_of(idx) for idx in split(b)), split(b)))
      finally:
        model._two_opt_beside_loop = True
    return run

  def loop_only(b):
    def run():
      for idx in split(b):
        model._solve_enqueue(batches_of(idx), idx)
    return run

  ways = {"single": one_by_one} if single else {}
  for b in sizes:
    ways.update({f"batch{b}": batched(b), f"pipelined{b}": pipelined(b), f"loop_only{b}": loop_only(b)})
    if between:
      ways[f"pipelined{b}_between"] = pipelined(b, beside=False)
  return ways


def timed_rounds(ways, rounds):
  names = list(ways)
  for f in ways.values():        # warm-up: graphs prepared, loops captured
    f()
  torch.cuda.synchronize()
  sampler = ClockSampler(torch.cuda.current_device())
  sampler.start()
  per = {k: [] for k in names}
  for r in range(rounds):
    for k in names[r % len(names):] + names[:r % len(names)]:
      t0 = time.perf_counter()
      ways[k]()
      torch.cuda.synchronize()
      per[k].append(time.perf_counter() - t0)
  return per, sampler.stop()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--steps", type=int, default=50)
  ap.add_argument("--select", default="", help='regex over "workload: way"; default: every way')
  a = ap.parse_args()
  torch.set_grad_enabled(False)
  info = card()
  w = syn.make_encoder_weights(0, out_channels=2)

  # 64 x TSP-500 k=50, sparse
  n = 64
  parts = [(syn.tsp_points(500, 1234, i), None) for i in range(n)]
  parts = [(p, syn.knn_edge_index(p, 50)) for p, _ in parts]
  m = G.tsp_model(w, sparse_factor=50, inference_diffusion_steps=a.steps)
  workloads = [("64 x TSP-500 k=50", n, solve_ways(m, lambda idx: sparse_batch([parts[i] for i in idx]), n))]
  m4 = G.tsp_model(w, sparse_factor=50, inference_diffusion_steps=a.steps, parallel_sampling=4)
  workloads.append(("64 x TSP-500 k=50 P=4", n, solve_ways(m4, lambda idx: sparse_batch([parts[i] for i in idx]), n,
                                                          single=False, between=True)))
  # 256 x TSP-50, dense
  nd = 256
  pts = np.stack([syn.tsp_points(50, 4321, i) for i in range(nd)]).astype(np.float32)
  md = G.tsp_model(w, sparse_factor=-1, inference_diffusion_steps=a.steps)
  workloads.append(("256 x TSP-50 dense", nd, solve_ways(md, lambda idx: dense_batch(pts[idx]), nd)))
  # 32 x MIS ER-[700, 800] p=0.15
  nm = 32
  msizes = np.random.default_rng(7).integers(700, 801, nm)
  graphs = [syn.er_graph_edge_index(int(s), 0.15, 77, i) for i, s in enumerate(msizes)]
  labels = [(syn.initial_noise(int(s), i) > 0).astype(np.float32) for i, s in enumerate(msizes)]
  mm = G.mis_model(w, inference_diffusion_steps=a.steps)
  workloads.append(("32 x MIS ER-[700, 800] p=0.15", nm,
                    solve_ways(mm, lambda idx: mis_batch([graphs[i] for i in idx], [labels[i] for i in idx]), nm,
                               sizes=(16, 32), single=False)))

  # the decode alone: merged tours of the TSP-500 heat maps
  tours = []
  for i, (p, e) in enumerate(parts):
    x0 = (syn.initial_noise(e.shape[1], i) > 0).astype(np.float32)
    heat = m.denoise_heatmap(G.cu(p), G.cu(e), G.cu(x0), seed=i).cpu().numpy() + 1e-6
    t, _ = tu.merge_tours(heat, p, e, sparse_graph=True)
    tours.append(np.array(t, np.int64))
  p64 = [p.astype(np.float64) for p, _ in parts]
  workloads.append(("2-opt of 64 x TSP-500 merged tours", n, {
      "two_opt_each": lambda: [tu.batched_two_opt_torch(p, t, 1000, "cuda") for p, t in zip(p64, tours)],
      "two_opt_instances": lambda: tu.batched_two_opt_instances(p64, tours, 1000, "cuda")}))

  for label, count, ways in workloads:
    ways = {k: f for k, f in ways.items() if re.search(a.select, f"{label}: {k}")}
    if not ways:
      continue
    per, clocks = timed_rounds(ways, a.rounds)
    print(json.dumps({"workload": label, "steps": a.steps,
                      "instances_per_s_median": {k: count / float(np.median(v)) for k, v in per.items()},
                      "seconds_per_round": per, "gpu": info["name"], "power_limit": info["power_limit"],
                      "sm_clock_mhz_median": clocks.get("sm_mhz"), "clock_event_reasons": clocks.get("reasons")}),
          flush=True)


if __name__ == "__main__":
  main()

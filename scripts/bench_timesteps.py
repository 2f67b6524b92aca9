"""What a timestep per element costs: the encoder forward of the reference's training steps, timed on the GPU.

    python scripts/bench_timesteps.py [--rounds 5] [--reps 10]

Workloads (synthetic weights and graphs; each forward under no_grad, as a loss evaluation runs it):
  dense    TSP-50 dense, B = 64 samples, one t per sample.  `loop`: B single-sample forwards, the way the dense forward
           handled per-sample timesteps before it ran them as one call; `one_call`: GNNEncoder.forward with t (B,).
  tsp      TSP-500 k = 50 x 8 graphs, one t per graph repeated over its edges, against one t for the whole call.
  mis      MIS ER-750 p = 0.15 x 8 graphs, one t per graph repeated over its nodes, against one t for the call.
The two ways of a workload alternate within each round (the order flips from round to round), so that clock and load
drift hits them alike; each way's time is the median over the rounds of reps forwards between CUDA events.  For tsp and
mis a separate pass reads the edge-layer kernel time of one forward of each way from dfb_profile_begin / _end: the per-row
time-vector reads are the only difference between the two edge kernels.  Prints one JSON line per workload with the
card's name and power limit, read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench_instances import card  # noqa: E402
from difusco_b200 import synthetic as syn  # noqa: E402
import gpu_util as G  # noqa: E402


def timed(fn, reps):
  ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  ev0.record()
  for _ in range(reps):
    fn()
  ev1.record()
  torch.cuda.synchronize()
  return ev0.elapsed_time(ev1) / reps


def dense_case(w):
  B, V = 64, 50
  enc = G.encoder(w, 2, sparse=False)
  pts = G.cu(np.stack([syn.tsp_points(V, 31, b) for b in range(B)]))
  xt = G.cu(syn.initial_noise(B * V * V, 32).reshape(B, V, V)) * 0.5
  t = G.cu(np.random.default_rng(33).integers(1, 1001, B).astype(np.float32))
  # the single-sample forwards share one context, so each re-prepares its graph as the removed loop did
  return enc, {"loop": lambda: [enc(pts[b:b + 1], t[b:b + 1], xt[b:b + 1]) for b in range(B)],
               "one_call": lambda: enc(pts, t, xt)}


def tsp_case(w):
  N, K, B = 500, 50, 8
  pts, ei = syn.tsp_sparse_batch(N, K, B, seed=41)
  enc = G.encoder(w, 2)
  d_pts, d_ei, xt = G.cu(pts), G.cu(ei), G.cu(syn.initial_noise(ei.shape[1], 42))
  t_graph = G.cu(np.repeat(np.random.default_rng(43).integers(1, 1001, B), N * K).astype(np.float32))
  t_one = torch.tensor([500.0], device="cuda")
  return enc, {"per_graph_t": lambda: enc(d_pts, t_graph, xt, d_ei), "uniform_t": lambda: enc(d_pts, t_one, xt, d_ei)}


def mis_case(w):
  B = 8
  ei, sizes = syn.mis_batch(750, 750, 0.15, B, seed=51)
  enc = G.encoder(w, 2, node_only=True)
  d_ei, xt = G.cu(ei), G.cu(syn.initial_noise(sum(sizes), 52))
  t_graph = G.cu(np.repeat(np.random.default_rng(53).integers(1, 1001, B), sizes).astype(np.float32))
  t_one = torch.tensor([500.0], device="cuda")
  return enc, {"per_graph_t": lambda: enc(xt, t_graph, edge_index=d_ei),
               "uniform_t": lambda: enc(xt, t_one, edge_index=d_ei)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--reps", type=int, default=10)
  ap.add_argument("--only", default="", help="dense, tsp or mis")
  a = ap.parse_args()
  torch.set_grad_enabled(False)
  info = card()
  w = syn.make_encoder_weights(seed=0, out_channels=2)
  for name, make in (("dense", dense_case), ("tsp", tsp_case), ("mis", mis_case)):
    if a.only and a.only != name:
      continue
    enc, ways = make(w)
    keys = list(ways)
    for k in keys:   # warm up every shape and way
      ways[k]()
    torch.cuda.synchronize()
    rounds = {k: [] for k in keys}
    for r in range(a.rounds):
      for k in (keys if r % 2 == 0 else keys[::-1]):
        rounds[k].append(timed(ways[k], a.reps))
    line = {"workload": name, "gpu": info["name"], "power_limit": info["power_limit"],
            "ms_per_forward_median": {k: float(np.median(v)) for k, v in rounds.items()},
            "ms_per_forward_rounds": rounds}
    if name != "dense":
      ctx = enc.engine()
      kern = {}
      for k in keys:
        ctx.profile_begin()
        ways[k]()
        ms, n = ctx.profile_end()
        kern[k] = {"edge_kernel_ms": ms, "edge_kernel_launches": n}
      line["edge_kernel_one_forward"] = kern
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
  main()

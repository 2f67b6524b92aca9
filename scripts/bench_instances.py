"""Ragged batches three ways: per-instance GroupNorm in one call, the coupled call, and one call per instance.

    python scripts/bench_instances.py [--rounds 3] [--reps 2] [--profile]

Workloads: 16 TSP-500 k=50 instances (bench.py's C2 shape) and 32 MIS ER-[700,800] p=0.15 graphs (C4), each denoised
by the 50-step categorical loop with in-kernel Philox draws, three ways:
  instances  one block-diagonal call, head GroupNorm per instance (node_ptr): each instance's reference answer
  coupled    one block-diagonal call, one GroupNorm over every row of the call (what bench.py times as C2 / C4)
  single     one call per instance, one after another, each on its own context
Every way has its graphs prepared and its loop captured before timing, so the timed region is the denoise loops alone.
The ways are alternated within each round (the order rotates from round to round) so that clock and load drift hits
them alike.  Prints one JSON line per workload: graphs/s per way (median over the rounds, and every round), the card's
name and power limit, and the median SM clock sampled during the timed runs.  --profile also runs one loop of
`instances` and `coupled` under torch.profiler and reports the mean time of the head kernels (k_gn_partial,
k_gn_final, k_head) in each, in a separate pass after the timed rounds."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench import ClockSampler  # noqa: E402
from difusco_b200 import synthetic as syn  # noqa: E402
import gpu_util as G  # noqa: E402

STEPS = 50
WAYS = ["instances", "coupled", "single"]


def card():
  idx = torch.cuda.current_device()
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(idx)],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, power = [x.strip() for x in out.split(",")]
  except Exception:
    name, power = torch.cuda.get_device_name(idx), "unknown"
  return {"name": name, "power_limit": power}


def tsp_workload():
  pts, ei = syn.tsp_sparse_batch(500, 50, 16, seed=1234)
  sizes = [500] * 16
  xt = (syn.initial_noise(ei.shape[1], 0) > 0).astype(np.float32)
  return dict(task="tsp", label="16 x TSP-500 k=50", pts=pts, ei=ei, xt=xt, sizes=sizes, per_node_state=False)


def mis_workload():
  ei, sizes = syn.mis_batch(700, 800, 0.15, 32, seed=1234)
  xt = (syn.initial_noise(int(sum(sizes)), 0) > 0).astype(np.float32)
  return dict(task="mis", label="32 x MIS ER-[700,800] p=0.15", pts=None, ei=ei, xt=xt, sizes=sizes,
              per_node_state=True)


def _model(task, w):
  if task == "tsp":
    return G.tsp_model(w, sparse_factor=50, inference_diffusion_steps=STEPS)
  return G.mis_model(w, inference_diffusion_steps=STEPS)


def _runner(wl, w, node_ptr, pts, ei, xt):
  """A prepared model and a closure that runs one 50-step loop on device copies of its inputs."""
  m = _model(wl["task"], w)
  d_ei, d_xt = G.cu(ei), G.cu(xt)
  d_pts = G.cu(pts) if pts is not None else None
  x = torch.empty_like(d_xt)

  def run():
    x.copy_(d_xt)
    if wl["task"] == "tsp":
      m.denoise_heatmap(d_pts, d_ei, x, seed=7, node_ptr=node_ptr)
    else:
      m.denoise_labels(d_ei, x, seed=7, node_ptr=node_ptr)
  run.ctx = m.model.engine()
  return run


def build_ways(wl, w):
  ptr = syn.node_ptr(wl["sizes"])
  ways = {"instances": [_runner(wl, w, ptr, wl["pts"], wl["ei"], wl["xt"])],
          "coupled": [_runner(wl, w, None, wl["pts"], wl["ei"], wl["xt"])], "single": []}
  # instance i alone: its nodes renumbered from 0; its edges are the batch's edges whose row lies in its node range
  row = wl["ei"][0]
  for i in range(len(wl["sizes"])):
    a, b = int(ptr[i]), int(ptr[i + 1])
    sel = (row >= a) & (row < b)
    ei = wl["ei"][:, sel] - a
    xt = wl["xt"][a:b] if wl["per_node_state"] else wl["xt"][sel]
    pts = wl["pts"][a:b] if wl["pts"] is not None else None
    ways["single"].append(_runner(wl, w, None, pts, ei, xt))
  return ways


def time_way(runs, reps):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  e0.record()
  for _ in range(reps):
    for r in runs:
      r()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / 1e3


def head_kernel_ms(runs):
  from torch.profiler import ProfilerActivity, profile
  for r in runs:   # plain launches: every kernel is its own profiler event
    r.ctx.set_graph_capture(False)
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for r in runs:
      r()
    torch.cuda.synchronize()
  for r in runs:
    r.ctx.set_graph_capture(True)
  out = {}
  for ev in prof.key_averages():
    for k in ("k_gn_partial", "k_gn_final", "k_head"):
      if k in ev.key:
        out[k] = ev.device_time_total / max(ev.count, 1) / 1e3
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--reps", type=int, default=2, help="loops of every instance per way and round")
  ap.add_argument("--profile", action="store_true")
  a = ap.parse_args()
  torch.set_grad_enabled(False)
  assert torch.cuda.is_available(), "bench_instances.py measures on the GPU only"
  info = card()
  w = syn.make_encoder_weights(0, out_channels=2)
  for wl in (tsp_workload(), mis_workload()):
    ways = build_ways(wl, w)
    for runs in ways.values():   # prepare, capture, warm up
      time_way(runs, 1)
    n = len(wl["sizes"])
    rates = {k: [] for k in WAYS}
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    for rnd in range(a.rounds):
      order = WAYS[rnd % 3:] + WAYS[:rnd % 3]
      for k in order:
        rates[k].append(n * a.reps / time_way(ways[k], a.reps))
    clocks = sampler.stop()
    line = {"workload": wl["label"] + ", 50-step categorical denoise, in-kernel Philox",
            "graphs_per_s": {k: float(np.median(v)) for k, v in rates.items()},
            "graphs_per_s_rounds": rates, "rounds": a.rounds, "reps": a.reps,
            "instances_vs_coupled": float(np.median(rates["instances"]) / np.median(rates["coupled"])),
            "instances_vs_single": float(np.median(rates["instances"]) / np.median(rates["single"])),
            "gpu": info["name"], "power_limit": info["power_limit"], "sm_clock_mhz_median": clocks.get("sm_mhz"),
            "clock_event_reasons": clocks.get("reasons")}
    if a.profile:
      line["head_kernel_ms"] = {k: head_kernel_ms(ways[k]) for k in ("instances", "coupled")}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
  main()

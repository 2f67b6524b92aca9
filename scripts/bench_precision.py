"""What the edge-layer precision costs: the fused 50-step denoise loop under bf16x3 (tc), bf16x6 (tc6) and the fp32
validation kernels (fp32), timed on the GPU.

    python scripts/bench_precision.py [--rounds 3] [--reps 2] [--configs C2,C4]

Workloads: bench.py's C2 (16 x TSP-500 k = 50, categorical) and C4 (32 x MIS ER-[700, 800] p = 0.15, categorical), built
by bench.py's own build_workload, synthetic weights.  Each loop is one dfb_denoise call (the captured loop) with seeded
in-kernel sampling.  Per round the three implementations run in turn on one context (the order rotates from round to
round, so that clock and load drift hits them alike); each one's time is reps loops between CUDA events after a
warm-up loop that re-captures it, and the result is the median over the rounds.  Prints one JSON line per workload with
graphs/s per implementation, the ratios to tc and the card's name and power limit, read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench  # noqa: E402
from bench_instances import card  # noqa: E402
from difusco_b200 import _cabi, synthetic as syn  # noqa: E402
from difusco_b200.pl_mis_model import MISModel  # noqa: E402
from difusco_b200.pl_tsp_model import TSPModel  # noqa: E402
from difusco_b200.utils.diffusion_schedulers import InferenceSchedule  # noqa: E402

IMPLS = {"tc": _cabi.EDGE_IMPL_TC, "tc6": _cabi.EDGE_IMPL_TC6, "fp32": _cabi.EDGE_IMPL_FP32}


def workload(name):
  """-> (run(seed) running one 50-step loop, graphs per loop, the context)."""
  wl = bench.build_workload(bench.CONFIGS[name], 0)
  model = (MISModel if wl["node_only"] else TSPModel)(wl["args"])
  model.model.load_state_dict({k: torch.from_numpy(v) for k, v in syn.make_encoder_weights(0, out_channels=2).items()})
  model.cuda().eval()
  ctx = model.model.engine()
  sched = InferenceSchedule("cosine", bench.T, bench.DENOISE_STEPS)
  t1s, cs, ls = [], [], []
  for i in range(bench.DENOISE_STEPS):
    t1, t2 = sched(i)
    c, last = model.posterior_consts(int(t1), int(t2))
    t1s.append(int(t1)); cs.append(c); ls.append(last)
  model.model.set_graph(torch.from_numpy(wl["edge_index"]).cuda(), wl["V"], wl["gn_segments"])
  if wl["points"] is not None:
    model.model.set_points(torch.from_numpy(wl["points"]).cuda())
  x0 = torch.from_numpy(wl["xt0"]).cuda()
  x = torch.empty_like(x0)
  stream = torch.cuda.current_stream().cuda_stream

  def run(seed):
    x.copy_(x0)
    ctx.denoise(_cabi.CATEGORICAL, x.data_ptr(), t1s, cs, ls, None, seed, stream)

  return run, wl["graphs"], ctx, wl


def measure(name, rounds, reps):
  run, graphs, ctx, wl = workload(name)
  order = list(IMPLS)
  ms = {k: [] for k in IMPLS}
  for r in range(rounds):
    for impl in order[r % len(order):] + order[:r % len(order)]:
      ctx.set_edge_impl(IMPLS[impl])
      run(0)   # re-captures the loop for this implementation
      torch.cuda.synchronize()
      ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      ev0.record()
      for i in range(reps):
        run(1 + i)
      ev1.record()
      torch.cuda.synchronize()
      ms[impl].append(ev0.elapsed_time(ev1) / reps)
  med = {k: float(np.median(v)) for k, v in ms.items()}
  gps = {k: graphs / (v / 1e3) for k, v in med.items()}
  return {"workload": name, "label": bench.CONFIGS[name]["label"] or bench.METRIC, "E": int(wl["E"]),
          "graphs_per_loop": graphs, "steps": bench.DENOISE_STEPS, "rounds": rounds, "reps": reps,
          "ms_per_loop": {k: round(v, 2) for k, v in med.items()},
          "ms_per_loop_rounds": {k: [round(x, 2) for x in v] for k, v in ms.items()},
          "graphs_per_s": {k: round(v, 3) for k, v in gps.items()},
          "time_vs_tc": {k: round(med[k] / med["tc"], 2) for k in IMPLS}, "card": card()}


def main():
  ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--reps", type=int, default=2)
  ap.add_argument("--configs", default="C2,C4")
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_precision.py times the GPU kernels: no CUDA device")
  for name in a.configs.split(","):
    print(json.dumps(measure(name, a.rounds, a.reps)), flush=True)


if __name__ == "__main__":
  main()

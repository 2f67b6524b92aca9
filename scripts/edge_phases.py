"""Where the time goes inside the fused edge layer: one encoder forward of a bench.py workload (default C2: TSP-500,
k = 50, 16 instances, E = 400 000) with the phase timers of k_edge_layer_wg2_timed, printed as one JSON line.

    python scripts/edge_phases.py [--config C2] [--forwards 1]

Cycles are SM clock cycles read by thread 0 of each consumer warpgroup and summed over every warpgroup and layer;
per_tile divides by the tiles each warpgroup processed, so it is the time one warpgroup spends on one tile.  The timed
kernel is a copy of the product kernel with clock reads added; its outputs are identical, its speed a little lower.
The phases partition the tile loop except for the waits of a warpgroup for its turn on the tensor cores (the other
warpgroup's GEMM), which no phase slot holds: turn_wait is the rest of the loop's cycles.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ["convert", "gemm1_wait", "gemm1_mma", "e1_gather_gate", "reduce", "layernorms", "gemm2_wait", "gemm2_mma",
          "e4_residual"]


def gpu_info():
  q = "name,power.limit,clocks.sm,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
  except Exception as ex:   # the counters are still meaningful without the card's description
    return {"error": str(ex)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--config", default="C2")
  ap.add_argument("--forwards", type=int, default=1)
  args = ap.parse_args()

  import torch
  import bench
  from difusco_b200 import synthetic as syn
  from difusco_b200.pl_tsp_model import TSPModel

  cfg = bench.CONFIGS[args.config]
  if cfg["task"] != "tsp" or cfg["knn"] <= 0:
    raise SystemExit("edge_phases.py times the sparse TSP workloads (C2, C3, C5, B1)")
  wl = bench.build_workload(cfg, 0)
  torch.cuda.set_device(0)
  model = TSPModel(wl["args"])
  w = syn.make_encoder_weights(0, out_channels=2 if cfg["diffusion"] == "categorical" else 1)
  model.model.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
  model.cuda().eval()
  enc = model.model
  ctx = enc.engine()
  pts = torch.from_numpy(wl["points"]).cuda()
  ei = torch.from_numpy(wl["edge_index"]).cuda()
  xt = torch.from_numpy(wl["xt0"]).cuda()
  t = torch.tensor([500.0])

  with torch.no_grad():
    enc(pts, t, xt, ei)   # warm-up: graph preparation, module load
    torch.cuda.synchronize()
    ctx.debug_phase_cycles()   # reset
    ctx.set_phase_timing(True)
    for _ in range(args.forwards):
      enc(pts, t, xt, ei)
    torch.cuda.synchronize()
    c = ctx.debug_phase_cycles()
    ctx.set_phase_timing(False)

  tiles, total = c[0], c[1]
  phases = dict(zip(PHASES, c[2:2 + len(PHASES)]))
  if tiles == 0 or total == 0:
    raise SystemExit(f"phase counters are empty: {c[:12]}")
  line = {"config": args.config, "E": int(wl["E"]), "forwards": args.forwards, "warpgroup_tiles": tiles,
          "cycles_per_tile": total / tiles,
          "per_tile": {k: v / tiles for k, v in phases.items()},
          "share": {k: v / total for k, v in phases.items()},
          "turn_wait_per_tile": (total - sum(phases.values())) / tiles,
          "turn_wait_share": 1.0 - sum(phases.values()) / total,
          "gpu": gpu_info()}
  print(json.dumps(line))


if __name__ == "__main__":
  main()

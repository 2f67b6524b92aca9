"""Cost of recording the denoise trajectory: dfb_denoise against dfb_denoise_record with the state, p and network
output recorded at every step, on bench.py's headline workload (C2: TSP-500 k = 50, batch 16, 50 categorical steps).

    python scripts/record_cost.py [--reps 10] [--config C2]

The two calls alternate on one context, timed with CUDA events around each whole loop (both replay the same captured
graph).  Prints one JSON line: median ms per loop of each, their difference and the bytes recorded.  Writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=10)
  ap.add_argument("--config", default="C2")
  a = ap.parse_args()
  import torch
  import bench
  from difusco_b200 import _cabi, synthetic as syn
  from difusco_b200.pl_tsp_model import TSPModel
  from oracle import difusco_oracle as orc

  cfg = bench.CONFIGS[a.config]
  wl = bench.build_workload(cfg, 0)
  if wl["node_only"]:
    raise SystemExit("TSP configs only")
  args = wl["args"]
  m = TSPModel(args)
  w = syn.make_encoder_weights(0, out_channels=2 if args.diffusion_type == "categorical" else 1)
  m.model.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
  m.cuda().eval()
  dev = torch.device("cuda")
  if wl["gn_segments"] > 1:
    m.model.set_graph(torch.from_numpy(wl["edge_index"]).to(dev), wl["V"], wl["gn_segments"])
    m.model.set_points(torch.from_numpy(wl["points"]).to(dev))
  else:
    m._prepare(torch.from_numpy(wl["points"]).to(dev), torch.from_numpy(wl["edge_index"]).to(dev), dev)
  ctx = m.model.engine()
  steps = args.inference_diffusion_steps
  t1s, cs, ls = [], [], []
  for t1, t2 in orc.inference_schedule(args.inference_schedule, 1000, steps):
    c, last = m.posterior_consts(t1, t2)
    t1s.append(int(t1)); cs.append(c); ls.append(last)
  cat = args.diffusion_type == "categorical"
  mode = _cabi.CATEGORICAL if cat else _cabi.GAUSSIAN
  n = wl["n_state"]
  oc = 2 if cat else 1
  rec_xt = torch.empty((steps, n), device=dev)
  rec_p = torch.empty((steps, n), device=dev) if cat else None
  rec_out = torch.empty((steps, n, oc), device=dev)
  x0 = torch.from_numpy(wl["xt0"]).to(dev)
  x = torch.empty_like(x0)
  st = torch.cuda.current_stream()

  def once(record):
    x.copy_(x0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    if record:
      ctx.denoise_record(mode, x.data_ptr(), t1s, cs, ls, list(range(steps)), rec_xt.data_ptr(),
                         rec_p.data_ptr() if rec_p is not None else None, rec_out.data_ptr(), None, 7, st.cuda_stream)
    else:
      ctx.denoise(mode, x.data_ptr(), t1s, cs, ls, None, 7, st.cuda_stream)
    e1.record(st)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)

  for _ in range(2):   # capture, warm-up
    once(False)
    once(True)
  plain, rec = [], []
  for _ in range(a.reps):
    plain.append(once(False))
    rec.append(once(True))
  mp, mr = float(np.median(plain)), float(np.median(rec))
  props = torch.cuda.get_device_properties(0)
  print(json.dumps({"config": a.config, "device": props.name, "steps": steps, "elements": n,
                    "record_bytes": int(steps * n * (4 * oc + (8 if cat else 4))),
                    "ms_plain": mp, "ms_record_all": mr, "ms_delta": mr - mp, "rel_delta": mr / mp - 1,
                    "ms_plain_minmax": [min(plain), max(plain)], "ms_record_minmax": [min(rec), max(rec)]}))


if __name__ == "__main__":
  main()

"""Rows f2/f3 timing on the GPU box: tour merge (host C++) and batched 2-opt (CUDA) against the formulation the
reference uses (dense N*N argsort merge on the CPU; torch (B,N,N)-temporaries 2-opt on the same GPU).

    python tests/tools/bench_decode.py [--sizes 500,1000,2000] [--out decode_bench.jsonl]
Lives under tests/ because the comparison arms come from oracle/tsp_decode_oracle.py (test infrastructure; only tests/,
smoke() and bench.py's CPU baseline may touch oracle/); the 2-opt arm is the same formulation with torch on the GPU.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
from difusco_b200 import synthetic as syn            # noqa: E402
from difusco_b200.utils import tsp_utils as tu       # noqa: E402
from oracle import tsp_decode_oracle as orc          # noqa: E402


def torch_two_opt(points, tours, max_iterations, device):
  """oracle.two_opt with torch tensors on `device` (how the reference spends its 2-opt time on a GPU)."""
  pts = torch.from_numpy(points).to(device)
  tr = torch.from_numpy(tours.copy()).to(device)
  n, it = pts.shape[0], 0
  d = lambda u, v: torch.sqrt(torch.sum((u - v) ** 2, dim=-1))
  while True:
    head, nxt = pts[tr[:, :-1]], pts[tr[:, 1:]]
    step = d(head, nxt)
    change = d(head[:, :, None], head[:, None, :]) + d(nxt[:, :, None], nxt[:, None, :]) - step[:, :, None] - step[:, None, :]
    flat = torch.triu(change, diagonal=2).reshape(len(tr), -1)
    pick = flat.argmin(dim=1)
    if not float(flat.min()) < -1e-6:
      break
    for b in range(len(tr)):
      i, j = int(pick[b]) // n, int(pick[b]) % n
      tr[b, i + 1:j + 1] = torch.flip(tr[b, i + 1:j + 1], dims=(0,))
    it += 1
    if it >= max_iterations:
      break
  return tr.cpu().numpy(), it


def timed(fn, reps=1):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(reps):
    out = fn()
  torch.cuda.synchronize()
  return out, (time.perf_counter() - t0) / reps * 1e3


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--sizes", default="500,1000,2000")
  ap.add_argument("--k", type=int, default=50)
  ap.add_argument("--par", type=int, default=1)
  ap.add_argument("--two_opt_iterations", type=int, default=1000)
  ap.add_argument("--out", default="decode_bench.jsonl")
  a = ap.parse_args()
  os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
  tu.batched_two_opt_torch(np.random.rand(8, 2), np.array([[0, 1, 2, 3, 4, 5, 6, 7, 0]]), device="cuda")   # context + warm-up
  with open(a.out, "a") as fh:
    for n in [int(s) for s in a.sizes.split(",")]:
      pts = syn.tsp_points(n, seed=11, instance=0).astype(np.float32)
      ei = syn.knn_edge_index(pts, a.k)
      rng = np.random.default_rng(n)
      dist = np.linalg.norm(pts[ei[0]] - pts[ei[1]], axis=-1)
      heat = np.tile((np.exp(-4.0 * dist * np.sqrt(n)) * (0.5 + 0.5 * rng.random(dist.shape)) + 1e-6), a.par).astype(np.float32)
      rec = {"n": n, "k": a.k, "parallel_sampling": a.par, "two_opt_cap": a.two_opt_iterations}
      (tours, it), rec["merge_exact_ms"] = timed(lambda: tu.merge_tours(heat, pts, ei, True, a.par))
      (tours_f, _), rec["merge_nearest_end_ms"] = timed(lambda: tu.merge_tours(heat, pts, ei, True, a.par, exact=False))
      if n <= 2000:
        def dense():
          return [orc.greedy_merge(pts, orc.symmetric_heat(n, h, ei)) for h in np.split(heat, a.par)]
        res, rec["merge_reference_formulation_ms"] = timed(dense)
        rec["merge_identical"] = bool(all(list(r[0]) == t for r, t in zip(res, tours)))
      tours = np.array(tours).astype(np.int64)
      p64 = pts.astype("float64")
      (solved, ns), rec["two_opt_ms"] = timed(lambda: tu.batched_two_opt_torch(p64, tours, a.two_opt_iterations, "cuda"))
      rec["two_opt_iterations"] = int(ns)
      torch_two_opt(p64, tours, 2, "cuda")
      (solved_t, ns_t), rec["two_opt_torch_formulation_ms"] = timed(lambda: torch_two_opt(p64, tours, a.two_opt_iterations, "cuda"))
      rec["two_opt_identical_to_torch_gpu"] = bool(ns_t == ns and np.array_equal(solved_t, solved))
      ev = tu.TSPEvaluator(pts)
      rec["cost_merged"], rec["cost_two_opt"] = float(ev.evaluate(tours[0])), float(ev.evaluate(solved[0]))
      rec["cost_merged_nearest_end"] = float(ev.evaluate(tours_f[0]))
      print(json.dumps(rec), flush=True)
      fh.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
  main()

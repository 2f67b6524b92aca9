"""Row f1 timing: GPU brute-force k-NN graph vs the reference's sklearn KDTree on the host (same points).  gpu_ms is
the whole knn_edge_index_gpu call: the kernel, and the host's check of the extra rank for exact ties."""
import os, sys, time, json
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sklearn.neighbors import KDTree
from difusco_b200.co_datasets.tsp_graph_dataset import knn_edge_index_gpu
print(json.dumps({"device": torch.cuda.get_device_name()}), flush=True)
for n, k in [(500, 50), (1000, 100), (10000, 50), (10000, 100), (25600, 50)]:
  pts = np.random.default_rng(1).random((n, 2))
  t0 = time.perf_counter(); _, ref = KDTree(pts, leaf_size=30, metric="euclidean").query(pts, k=k); cpu_ms = (time.perf_counter() - t0) * 1e3
  d = torch.from_numpy(pts).cuda()
  knn_edge_index_gpu(d, k); torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(5): ei = knn_edge_index_gpu(d, k)
  e1.record(); torch.cuda.synchronize()
  ok = bool(np.array_equal(ei[1].cpu().numpy().reshape(n, k), ref))
  print(json.dumps({"N": n, "K": k, "gpu_ms": e0.elapsed_time(e1) / 5, "kdtree_cpu_ms": cpu_ms, "identical": ok}), flush=True)

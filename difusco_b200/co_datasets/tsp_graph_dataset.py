"""TSPGraphDataset: drop-in for the reference's co_datasets/tsp_graph_dataset.py (SURVEY 8f row f1 - the step
immediately BEFORE the denoise path).

Same constructor, `get_example`, `__len__` and `__getitem__` item layout:
  dense  (sparse_factor <= 0): (idx[1], points (N,2) f32, adj (N,N) f32, tour (N+1,) i64)              :39-51
  sparse (sparse_factor  > 0): (idx[1], GraphData(x (N,2) f32, edge_index (2,N*K) i64, edge_attr (N*K,1) bool),
                                point_indicator[1], edge_indicator[1], tour)                           :52-81
The k-NN graph (KDTree(leaf_size=30, euclidean).query in float64, :56-57) is built by the CUDA kernel behind
`dfb_knn_graph` (brute force in fp64, neighbours ascending with self first, exact ties to the smaller index).  Where
no two of a row's first K + 1 neighbours tie exactly, that order is the only one and KDTree returns it too.  KDTree
breaks exact ties (integer or rounded coordinates: grids, repeated points) in the order its tree traversal meets
them, and a tie across rank K changes which neighbours are in the row.  So the kernel ranks K + 1 neighbours, the
host recomputes their squared distances with the same expression, and only the rows with an exact tie are queried
again with the reference's own KDTree (its queries are independent per point).  Without a GPU the dataset raises:
the kernel builds every row, the KDTree query only resolves ties.
"""
import numpy as np
import torch

from .. import _cabi

try:
  from torch_geometric.data import Data as GraphData
except Exception:   # torch_geometric is not in this image: minimal attribute container with the same field names
  class GraphData(object):
    def __init__(self, **kw):
      self.__dict__.update(kw)


def _engine(device_index):
  return _cabi.device_context(device_index)   # shared with the model and 2-opt: one dfb_ctx per GPU


def knn_edge_index_gpu(points64, k, device=None, node_offset=0):
  """points64 (N,2) float64 numpy / tensor -> edge_index (2, N*k) int64 CUDA tensor (tsp_graph_dataset.py:56-62)."""
  if not torch.cuda.is_available():
    raise RuntimeError("difusco_b200 k-NN graph construction needs a CUDA device (no CPU fallback)")
  dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
  if isinstance(points64, torch.Tensor):
    pts = points64.to(device=dev, dtype=torch.float64).contiguous()
    host = pts.cpu().numpy()
  else:
    host = np.ascontiguousarray(points64, dtype=np.float64)
    pts = None
  if host.ndim != 2 or host.shape[1] != 2:
    raise ValueError(f"points must be (N, 2), got {tuple(host.shape)}")
  if not np.isfinite(host).all():
    raise ValueError("k-NN graph: points must be finite (the reference's KDTree rejects NaN and inf)")
  if pts is None:
    pts = torch.from_numpy(host).to(dev)
  n = host.shape[0]
  kq = min(k + 1, n) if 0 < k <= n else k          # one rank beyond k shows a tie across the row's last place
  ranked = torch.empty((2, n * kq), dtype=torch.int64, device=dev)
  _engine(dev.index if dev.index is not None else torch.cuda.current_device()).knn_graph(
      pts.data_ptr(), n, kq, node_offset, ranked.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
  cols = ranked[1].view(n, kq)
  nbr = cols.cpu().numpy() - node_offset
  x, y = np.ascontiguousarray(host[:, 0]), np.ascontiguousarray(host[:, 1])
  with np.errstate(over="ignore"):                 # the kernel's expression: float64 (x_j - x_q)^2 + (y_j - y_q)^2
    d2 = np.take(x, nbr)
    d2 -= x[:, None]
    d2 *= d2
    dy = np.take(y, nbr)
    dy -= y[:, None]
    dy *= dy
    d2 += dy
  # distances that overflow to +inf are no order KDTree can reproduce either: those rows keep the kernel's
  tied = np.flatnonzero(((d2[:, 1:] == d2[:, :-1]) & (d2[:, 1:] < np.inf)).any(axis=1))
  out = torch.empty((2, n * k), dtype=torch.int64, device=dev)
  out[0] = ranked[0].view(n, kq)[:, :k].reshape(-1)
  out[1] = cols[:, :k].reshape(-1)
  if len(tied):
    from sklearn.neighbors import KDTree
    _, idx = KDTree(host, leaf_size=30, metric="euclidean").query(host[tied], k=k, return_distance=True)
    out[1].view(n, k)[torch.from_numpy(tied).to(dev)] = torch.from_numpy(idx.astype(np.int64) + node_offset).to(dev)
  return out


class TSPGraphDataset(torch.utils.data.Dataset):
  def __init__(self, data_file, sparse_factor=-1, device=None):
    self.data_file = data_file
    self.sparse_factor = sparse_factor
    self.device = device
    self.file_lines = open(data_file).read().splitlines()
    print(f'Loaded "{data_file}" with {len(self.file_lines)} lines')

  def __len__(self):
    return len(self.file_lines)

  def get_example(self, idx):
    """'x0 y0 x1 y1 ... output t0 t1 ... t0' -> (points (N,2) float64, tour (N+1,) int64, 0-based)   :20-36"""
    head, tail = self.file_lines[idx].strip().split(" output ")
    coords = np.array(head.split(" "), dtype=np.float64)
    points = coords.reshape(-1, 2)
    tour = np.array(tail.split(" "), dtype=np.int64) - 1
    return points, tour

  def __getitem__(self, idx):
    points, tour = self.get_example(idx)
    n = points.shape[0]
    index = torch.LongTensor(np.array([idx], dtype=np.int64))
    if self.sparse_factor <= 0:
      adj = np.zeros((n, n))
      adj[tour[:-1], tour[1:]] = 1
      return index, torch.from_numpy(points).float(), torch.from_numpy(adj).float(), torch.from_numpy(tour).long()
    k = self.sparse_factor
    if torch.utils.data.get_worker_info() is not None:
      raise RuntimeError("difusco_b200.TSPGraphDataset builds the k-NN graph on the GPU: use num_workers=0 "
                         "(CUDA cannot be initialised in forked DataLoader workers)")
    # the GPU k-NN is an internal accelerator: the item is made of CPU tensors like the reference's (pin_memory and the
    # model's own .to(device) work unchanged)
    edge_index = knn_edge_index_gpu(points, k, self.device).cpu()
    succ = np.zeros(n, dtype=np.int64)          # tour successor of every node (:65-66)
    succ[tour[:-1]] = tour[1:]
    succ = torch.from_numpy(succ)
    tour_edges = torch.eq(edge_index[1], succ.repeat_interleave(k)).reshape(-1, 1)
    graph = GraphData(x=torch.from_numpy(points).float(), edge_index=edge_index, edge_attr=tour_edges)
    return (index, graph, torch.from_numpy(np.array([n], dtype=np.int64)).long(),
            torch.from_numpy(np.array([edge_index.shape[1]], dtype=np.int64)).long(), torch.from_numpy(tour).long())

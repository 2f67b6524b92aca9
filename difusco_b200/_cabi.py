"""ctypes binding of include/difusco_b200.h.  The ONLY compute backend: if the shared library is
missing or no H100 is present every call fails loudly - there is no eager/CPU fallback."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libdifusco_b200.so")

DFB_OK, DFB_E_INVALID, DFB_E_CUDA, DFB_E_UNSUPPORTED, DFB_E_NOMEM = 0, -1, -2, -3, -4
CATEGORICAL, GAUSSIAN = 0, 1
EDGE_IMPL_TC, EDGE_IMPL_FP32, EDGE_IMPL_TC1, EDGE_IMPL_TC6 = 0, 1, 2, 3
AGGREGATION = {"sum": 0, "mean": 1, "max": 2}
HEAD_FORWARD, HEAD_CATEGORICAL, HEAD_GAUSSIAN = 0, 1, 2

# every symbol include/difusco_b200.h declares (tests check the library exports all of them)
SYMBOLS = [
    "dfb_abi_version", "dfb_create", "dfb_destroy", "dfb_last_error", "dfb_set_aggregation",
    "dfb_set_edge_impl", "dfb_load_weights", "dfb_prepare_graph", "dfb_prepare_graph_instances", "dfb_set_points",
    "dfb_encoder_forward", "dfb_encoder_forward_timesteps", "dfb_denoise_step", "dfb_denoise", "dfb_denoise_record", "dfb_denoise_instances",
    "dfb_denoise_host",
    "dfb_launch_count", "dfb_profile_begin", "dfb_profile_end", "dfb_debug_edge_gemm", "dfb_debug_gnn_layer",
    "dfb_debug_gnn_layer_timesteps", "dfb_debug_head", "dfb_debug_entry", "dfb_debug_loop_captures",
    "dfb_debug_phase_cycles", "dfb_debug_watchdog", "dfb_knn_graph", "dfb_set_graph_capture",
    "dfb_set_phase_timing", "dfb_tsp_merge_sparse", "dfb_tsp_merge_order", "dfb_two_opt", "dfb_two_opt_instances",
    "dfb_write_heatmap_txt",
]

_lib = None


def lib():
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise RuntimeError(
        f"{LIB_PATH} not found: build it with `python -m difusco_b200.build` "
        "(difusco_b200 has no fallback path; the CUDA library is the product)")
  L = C.CDLL(LIB_PATH)
  vp, i32, i64, u64, f32 = C.c_void_p, C.c_int, C.c_int64, C.c_uint64, C.c_float
  L.dfb_abi_version.restype = i32
  L.dfb_create.argtypes = [C.POINTER(vp), i32]
  L.dfb_destroy.argtypes = [vp]
  L.dfb_last_error.argtypes = [vp]
  L.dfb_last_error.restype = C.c_char_p
  L.dfb_set_aggregation.argtypes = [vp, i32]
  L.dfb_set_edge_impl.argtypes = [vp, i32]
  L.dfb_load_weights.argtypes = [vp, i32, i32, i32, i32, i32, C.POINTER(C.c_char_p), C.POINTER(vp),
                                 C.POINTER(i64)]
  L.dfb_prepare_graph.argtypes = [vp, vp, i64, i64, i32, vp]
  L.dfb_prepare_graph_instances.argtypes = [vp, vp, i64, i64, i32, C.POINTER(i64), vp]
  L.dfb_set_points.argtypes = [vp, vp, vp]
  L.dfb_encoder_forward.argtypes = [vp, vp, f32, vp, vp]
  L.dfb_encoder_forward_timesteps.argtypes = [vp, vp, i32, C.POINTER(f32), vp, vp, vp]
  L.dfb_denoise_step.argtypes = [vp, i32, vp, f32, C.POINTER(f32), i32, vp, u64, i32, vp, vp, vp, vp]
  L.dfb_denoise.argtypes = [vp, i32, vp, i32, C.POINTER(C.c_int32), C.POINTER(f32),
                            C.POINTER(C.c_int32), vp, u64, vp]
  L.dfb_denoise_record.argtypes = [vp, i32, vp, i32, C.POINTER(C.c_int32), C.POINTER(f32), C.POINTER(C.c_int32), vp,
                                   u64, i32, C.POINTER(C.c_int32), vp, vp, vp, vp]
  L.dfb_denoise_instances.argtypes = [vp, i32, vp, i32, C.POINTER(C.c_int32), C.POINTER(f32), C.POINTER(C.c_int32),
                                      vp, i32, i32, C.POINTER(C.c_int32), vp, vp, vp, vp]
  L.dfb_denoise_host.argtypes = [vp, i32, vp, vp, i64, i64, i32, vp, i32, C.POINTER(C.c_int32),
                                 C.POINTER(f32), C.POINTER(C.c_int32), u64, vp, vp]
  L.dfb_launch_count.argtypes = [vp]
  L.dfb_launch_count.restype = i64
  L.dfb_debug_loop_captures.argtypes = [vp]
  L.dfb_debug_loop_captures.restype = i64
  L.dfb_profile_begin.argtypes = [vp]
  L.dfb_profile_end.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(i64)]
  L.dfb_debug_edge_gemm.argtypes = [vp, i32, vp, vp, vp]
  L.dfb_debug_gnn_layer.argtypes = [vp, i32, f32, vp, vp, vp]
  L.dfb_debug_gnn_layer_timesteps.argtypes = [vp, i32, i32, C.POINTER(f32), vp, vp, vp, vp]
  L.dfb_debug_head.argtypes = [vp, i32, vp, C.POINTER(f32), i32, vp, u64, i32, vp, vp, vp, vp, vp, vp, vp]
  L.dfb_debug_entry.argtypes = [vp, i32, vp, f32, vp, vp, vp, vp, vp, vp]
  L.dfb_debug_phase_cycles.argtypes = [vp, C.POINTER(C.c_uint64)]
  L.dfb_debug_watchdog.argtypes = [vp, C.POINTER(C.c_int)]
  L.dfb_set_graph_capture.argtypes = [vp, i32]
  L.dfb_set_phase_timing.argtypes = [vp, i32]
  L.dfb_knn_graph.argtypes = [vp, vp, i64, i32, i64, vp, vp]
  L.dfb_tsp_merge_sparse.argtypes = [vp, i64, vp, vp, i64, i32, vp, C.POINTER(i64)]
  L.dfb_tsp_merge_order.argtypes = [i64, vp, i64, vp, C.POINTER(i64)]
  L.dfb_two_opt.argtypes = [vp, vp, i64, vp, i64, i64, C.POINTER(i64), vp]
  L.dfb_two_opt_instances.argtypes = [vp, vp, vp, i64, vp, vp, i64, vp, vp]
  L.dfb_write_heatmap_txt.argtypes = [C.c_char_p, i64, vp]
  for name in SYMBOLS:
    fn = getattr(L, name)
    if fn.restype is C.c_int and name not in ("dfb_abi_version",):
      fn.restype = i32
  _lib = L
  return L


class DfbError(RuntimeError):
  pass


def _raise(code, msg):
  msg = msg.decode() if isinstance(msg, bytes) else msg
  if code == DFB_E_INVALID:
    raise ValueError(msg)
  if code == DFB_E_UNSUPPORTED:
    raise NotImplementedError(msg)
  if code == DFB_E_NOMEM:
    raise MemoryError(msg)
  raise DfbError(msg)


MERGE_COMPLETE, MERGE_INCOMPLETE, MERGE_AMBIGUOUS = 0, 1, 2


def instance_seeds_array(seeds, n_segments):
  """instance_seeds (a sequence of Python / numpy integers in [0, 2**64), one per GroupNorm segment of the prepared
  graph) -> uint64 numpy array.  Raises ValueError on anything else, before any device work."""
  if isinstance(seeds, (str, bytes)) or not hasattr(seeds, "__len__"):
    raise ValueError(f"instance_seeds must be a sequence of integers, got {type(seeds).__name__}")
  out = []
  for s in seeds:
    if isinstance(s, (bool, np.bool_)) or not isinstance(s, (int, np.integer)):
      raise ValueError(f"instance_seeds must hold integers, got {type(s).__name__}")
    if not 0 <= int(s) < 2 ** 64:
      raise ValueError(f"instance seed {int(s)} outside [0, 2**64)")
    out.append(int(s))
  if len(out) != int(n_segments):
    raise ValueError(f"{len(out)} instance seeds for a prepared graph of {int(n_segments)} instances / samples")
  return np.array(out, dtype=np.uint64)


def two_opt_instances_arrays(points_list, tours_list):
  """Per-instance points (n_i, 2) and tours (B_i, n_i + 1) -> the concatenated host arrays of dfb_two_opt_instances
  (points (V, 2) float64, node_ptr, tour_ptr, tours int64).  Checks shapes, dtypes and sizes."""
  if len(points_list) != len(tours_list):
    raise ValueError(f"{len(points_list)} point sets for {len(tours_list)} tour sets")
  if len(points_list) < 1:
    raise ValueError("at least one instance is required")
  pts, trs, node_ptr, tour_ptr = [], [], [0], [0]
  for i, (p, t) in enumerate(zip(points_list, tours_list)):
    p = np.asarray(p)
    t = np.asarray(t)
    if p.dtype.kind != "f" or p.ndim != 2 or p.shape[1] != 2:
      raise ValueError(f"instance {i}: points must be a float (n, 2) array, got {p.dtype} {tuple(p.shape)}")
    if not 3 <= p.shape[0] <= 46340:
      raise ValueError(f"instance {i}: {p.shape[0]} nodes (must be in [3, 46340])")
    if t.dtype.kind not in "iu" or t.ndim != 2 or t.shape[1] != p.shape[0] + 1 or t.shape[0] < 1:
      raise ValueError(f"instance {i}: tours must be an integer (B >= 1, n + 1 = {p.shape[0] + 1}) array, got "
                       f"{t.dtype} {tuple(t.shape)}")
    if t.min() < 0 or t.max() >= p.shape[0]:
      raise ValueError(f"instance {i}: tour entries must be local node ids in [0, {p.shape[0]})")
    pts.append(np.asarray(p, np.float64))
    trs.append(np.asarray(t, np.int64).reshape(-1))
    node_ptr.append(node_ptr[-1] + p.shape[0])
    tour_ptr.append(tour_ptr[-1] + t.shape[0])
  return (np.ascontiguousarray(np.concatenate(pts)), np.array(node_ptr, np.int64), np.array(tour_ptr, np.int64),
          np.ascontiguousarray(np.concatenate(trs)))


def tsp_merge_sparse(points, heat, edge_index, mode=0):
  """dfb_tsp_merge_sparse on host arrays -> (status, tour (n+1,) int64, merge_iterations)."""
  points = np.ascontiguousarray(points, dtype=np.float64)
  heat = np.ascontiguousarray(heat, dtype=np.float32).reshape(-1)
  edge_index = np.ascontiguousarray(edge_index, dtype=np.int64)
  n = points.shape[0]
  if edge_index.ndim != 2 or edge_index.shape[0] != 2 or edge_index.shape[1] != heat.shape[0]:
    raise ValueError("edge_index must be (2, E) with one heat value per edge")
  tour = np.empty(n + 1, dtype=np.int64)
  it = C.c_int64(0)
  rc = lib().dfb_tsp_merge_sparse(points.ctypes.data, n, heat.ctypes.data, edge_index.ctypes.data, heat.shape[0],
                                  int(mode), tour.ctypes.data, C.byref(it))
  if rc < 0:
    _raise(rc, "dfb_tsp_merge_sparse: invalid argument (n >= 3, indices inside [0, n), mode 0/1)")
  return rc, tour, it.value


def tsp_merge_order(n, order):
  """dfb_tsp_merge_order: the reference loop over an explicit order of flattened (i*n + j) entries."""
  order = np.ascontiguousarray(order, dtype=np.int64).reshape(-1)
  tour = np.empty(n + 1, dtype=np.int64)
  it = C.c_int64(0)
  rc = lib().dfb_tsp_merge_order(int(n), order.ctypes.data, order.shape[0], tour.ctypes.data, C.byref(it))
  if rc < 0:
    _raise(rc, "dfb_tsp_merge_order: invalid argument or the order does not complete a tour")
  return tour, it.value


def write_heatmap_txt(path, matrix):
  """dfb_write_heatmap_txt: (n, n) matrix -> the tsp_mcts text format.  float32 input is widened exactly."""
  m = np.ascontiguousarray(matrix, dtype=np.float64)
  if m.ndim != 2 or m.shape[0] != m.shape[1]:
    raise ValueError("matrix must be square")
  rc = lib().dfb_write_heatmap_txt(os.fsencode(path), m.shape[0], m.ctypes.data)
  if rc != DFB_OK:
    _raise(rc, f"dfb_write_heatmap_txt: cannot write {path}")


_DEVICE_CTX = {}


def device_context(device_index, prefer=None):
  """The ONE dfb_ctx per device that the helpers around the path (k-NN graph, 2-opt) run on.  A model registers its
  own context with `prefer=` when it is created first, so model + k-NN + 2-opt share one context (and one set of
  kernel attributes / scratch buffers) per GPU; without a model a plain context is created on first use."""
  ctx = _DEVICE_CTX.get(device_index)
  if ctx is None or getattr(ctx, "_h", None) is None:
    ctx = prefer if prefer is not None else Context(device_index)
    _DEVICE_CTX[device_index] = ctx
  return ctx


class Context(object):
  """One dfb_ctx: one GPU, one model, one prepared graph at a time."""

  def __init__(self, device=0):
    L = lib()
    h = C.c_void_p()
    rc = L.dfb_create(C.byref(h), int(device))
    if rc != DFB_OK:
      _raise(rc, L.dfb_last_error(None))
    self._h = h
    self.device = int(device)
    self._keep = []

  def close(self):
    if getattr(self, "_h", None):
      lib().dfb_destroy(self._h)
      self._h = None

  def __del__(self):
    try:
      self.close()
    except Exception:
      pass

  def _ck(self, rc):
    if rc != DFB_OK:
      _raise(rc, lib().dfb_last_error(self._h))

  # ---- model ----
  def load_weights(self, state_dict, n_layers, hidden_dim, out_channels, node_feature_only, consts=None):
    """state_dict: name -> numpy fp32 array (GNNEncoder.state_dict() keys, optional 'model.' prefix)."""
    items = [(k, np.ascontiguousarray(v, dtype=np.float32)) for k, v in state_dict.items()]
    for k, v in (consts or {}).items():
      items.append((k, np.ascontiguousarray(v, dtype=np.float32)))
    n = len(items)
    names = (C.c_char_p * n)(*[k.encode() for k, _ in items])
    ptrs = (C.c_void_p * n)(*[v.ctypes.data for _, v in items])
    numels = (C.c_int64 * n)(*[v.size for _, v in items])
    self._ck(lib().dfb_load_weights(self._h, n_layers, hidden_dim, out_channels, int(bool(node_feature_only)),
                                    n, names, ptrs, numels))

  def set_aggregation(self, name):
    if name not in AGGREGATION:
      raise ValueError(f"unknown aggregation {name}")
    self._ck(lib().dfb_set_aggregation(self._h, AGGREGATION[name]))

  def set_edge_impl(self, impl):
    self._ck(lib().dfb_set_edge_impl(self._h, impl))

  # ---- graph ----
  def prepare_graph(self, edge_index_ptr, num_nodes, num_edges, gn_segments=1, stream=0):
    self._ck(lib().dfb_prepare_graph(self._h, edge_index_ptr, num_nodes, num_edges, gn_segments, stream))

  def prepare_graph_instances(self, edge_index_ptr, num_nodes, num_edges, node_ptr, stream=0):
    """One GroupNorm segment per instance; node_ptr: host int64 array of n_instances + 1 node offsets."""
    node_ptr = np.ascontiguousarray(node_ptr, dtype=np.int64)
    self._ck(lib().dfb_prepare_graph_instances(self._h, edge_index_ptr, num_nodes, num_edges, node_ptr.size - 1,
                                               node_ptr.ctypes.data_as(C.POINTER(C.c_int64)), stream))

  def set_points(self, points_ptr, stream=0):
    self._ck(lib().dfb_set_points(self._h, points_ptr, stream))

  # ---- compute ----
  def encoder_forward(self, xt_ptr, t, out_ptr, stream=0):
    self._ck(lib().dfb_encoder_forward(self._h, xt_ptr, float(t), out_ptr, stream))

  def encoder_forward_timesteps(self, xt_ptr, t_values, t_index_ptr, out_ptr, stream=0):
    """encoder_forward with a timestep per element: t_values the distinct timesteps (host sequence), t_index_ptr a
    device int32 (N,) array of positions in t_values, or None for every element at t_values[0]."""
    v = np.ascontiguousarray(t_values, dtype=np.float32).reshape(-1)
    self._ck(lib().dfb_encoder_forward_timesteps(self._h, xt_ptr, v.size, v.ctypes.data_as(C.POINTER(C.c_float)),
                                                 t_index_ptr, out_ptr, stream))

  def denoise_step(self, diffusion, xt_in_ptr, t, consts, last, uniforms_ptr, seed, step_index, xt_out_ptr,
                   p_out_ptr=None, net_out_ptr=None, stream=0):
    c = (C.c_float * 4)(*[float(x) for x in consts])
    self._ck(lib().dfb_denoise_step(self._h, diffusion, xt_in_ptr, float(t), c, int(last), uniforms_ptr,
                                    int(seed) & 0xFFFFFFFFFFFFFFFF, int(step_index), xt_out_ptr, p_out_ptr,
                                    net_out_ptr, stream))

  @staticmethod
  def _sched_arrays(t1, consts, last):
    steps = len(t1)
    t1a = (C.c_int32 * steps)(*[int(x) for x in t1])
    ca = (C.c_float * (4 * steps))(*[float(x) for row in consts for x in row])
    la = (C.c_int32 * steps)(*[int(x) for x in last])
    return steps, t1a, ca, la

  def denoise(self, diffusion, xt_ptr, t1, consts, last, uniforms_ptr=None, seed=0, stream=0):
    steps, t1a, ca, la = self._sched_arrays(t1, consts, last)
    self._ck(lib().dfb_denoise(self._h, diffusion, xt_ptr, steps, t1a, ca, la, uniforms_ptr,
                               int(seed) & 0xFFFFFFFFFFFFFFFF, stream))

  def denoise_record(self, diffusion, xt_ptr, t1, consts, last, record_steps, rec_xt_ptr=None, rec_p_ptr=None,
                     rec_out_ptr=None, uniforms_ptr=None, seed=0, stream=0):
    """denoise that also writes, at each step record_steps[j], row j of the device buffers rec_xt (n_rec, N),
    rec_p (n_rec, N) and rec_out (n_rec, N, out_channels); any of them may be None."""
    steps, t1a, ca, la = self._sched_arrays(t1, consts, last)
    n_rec = len(record_steps)
    ra = (C.c_int32 * max(n_rec, 1))(*[int(x) for x in record_steps])
    self._ck(lib().dfb_denoise_record(self._h, diffusion, xt_ptr, steps, t1a, ca, la, uniforms_ptr,
                                      int(seed) & 0xFFFFFFFFFFFFFFFF, n_rec, ra, rec_xt_ptr, rec_p_ptr, rec_out_ptr,
                                      stream))

  def denoise_instances(self, diffusion, xt_ptr, t1, consts, last, instance_seeds_ptr, n_instances, record_steps=(),
                        rec_xt_ptr=None, rec_p_ptr=None, rec_out_ptr=None, stream=0):
    """denoise_record with Philox draws keyed per instance: instance_seeds_ptr is a device uint64 (n_instances,)
    array, one seed per GroupNorm segment of the prepared graph."""
    steps, t1a, ca, la = self._sched_arrays(t1, consts, last)
    n_rec = len(record_steps)
    ra = (C.c_int32 * max(n_rec, 1))(*[int(x) for x in record_steps])
    self._ck(lib().dfb_denoise_instances(self._h, diffusion, xt_ptr, steps, t1a, ca, la, instance_seeds_ptr,
                                         int(n_instances), n_rec, ra, rec_xt_ptr, rec_p_ptr, rec_out_ptr, stream))

  def denoise_host(self, diffusion, points_ptr, edge_index_ptr, num_nodes, num_edges, gn_segments, xt0_ptr,
                   t1, consts, last, seed, heatmap_ptr, stream=0):
    steps, t1a, ca, la = self._sched_arrays(t1, consts, last)
    self._ck(lib().dfb_denoise_host(self._h, diffusion, points_ptr, edge_index_ptr, num_nodes, num_edges,
                                    gn_segments, xt0_ptr, steps, t1a, ca, la,
                                    int(seed) & 0xFFFFFFFFFFFFFFFF, heatmap_ptr, stream))

  # ---- the step before the path (SURVEY 8f row f1) ----
  def two_opt(self, points, tours, max_iterations, stream=0):
    """dfb_two_opt on host arrays: returns (tours (B, n+1) int64 copy, iterations)."""
    points = np.ascontiguousarray(points, dtype=np.float64)
    tours = np.array(tours, dtype=np.int64, order="C", copy=True)
    if tours.ndim != 2 or tours.shape[1] != points.shape[0] + 1:
      raise ValueError("tours must be (batch, n + 1)")
    it = C.c_int64(0)
    self._ck(lib().dfb_two_opt(self._h, points.ctypes.data, points.shape[0], tours.ctypes.data, tours.shape[0],
                               int(max_iterations), C.byref(it), stream))
    return tours, it.value

  def two_opt_instances(self, points_list, tours_list, max_iterations, stream=0):
    """dfb_two_opt_instances: per-instance points (n_i, 2) and tours (B_i, n_i + 1) -> (list of refined tour arrays,
    list of iteration counts); each instance as two_opt on it alone."""
    points, node_ptr, tour_ptr, tours = two_opt_instances_arrays(points_list, tours_list)
    its = np.zeros(len(points_list), np.int64)
    self._ck(lib().dfb_two_opt_instances(self._h, points.ctypes.data, node_ptr.ctypes.data, len(points_list),
                                         tour_ptr.ctypes.data, tours.ctypes.data, int(max_iterations),
                                         its.ctypes.data, stream))
    out, e = [], 0
    for p, t in zip(points_list, tours_list):
      b, n1 = np.shape(t)
      out.append(tours[e:e + b * n1].reshape(b, n1))
      e += b * n1
    return out, [int(x) for x in its]

  def knn_graph(self, points_ptr, num_nodes, k, node_offset, edge_index_ptr, stream=0):
    self._ck(lib().dfb_knn_graph(self._h, points_ptr, int(num_nodes), int(k), int(node_offset), edge_index_ptr, stream))

  # ---- accounting ----
  def launch_count(self):
    return int(lib().dfb_launch_count(self._h))

  def loop_captures(self):
    """How many times the denoise loop has been captured into a CUDA graph on this context."""
    return int(lib().dfb_debug_loop_captures(self._h))

  def profile_begin(self):
    self._ck(lib().dfb_profile_begin(self._h))

  def profile_end(self):
    ms, n = C.c_double(0), C.c_int64(0)
    self._ck(lib().dfb_profile_end(self._h, C.byref(ms), C.byref(n)))
    return ms.value, n.value

  def set_graph_capture(self, enabled):
    self._ck(lib().dfb_set_graph_capture(self._h, int(bool(enabled))))

  def debug_watchdog(self):
    out = (C.c_int * 4)()
    lib().dfb_debug_watchdog(self._h, out)
    return [int(x) for x in out]

  def set_phase_timing(self, enabled):
    """Route the product edge-layer launches to the kernel with phase timers (read them with debug_phase_cycles)."""
    self._ck(lib().dfb_set_phase_timing(self._h, int(bool(enabled))))

  def debug_phase_cycles(self):
    """Read and reset the 32 phase counters: [tiles, total, convert, gemm1 wait, gemm1 mma, e1, reduce, ln, gemm2 wait,
    gemm2 mma, e4, 0...] (cycles summed over consumer warpgroups; see include/difusco_b200.h)."""
    out = (C.c_uint64 * 32)()
    self._ck(lib().dfb_debug_phase_cycles(self._h, out))
    return [int(x) for x in out]

  def debug_edge_gemm(self, layer, e_in_ptr, acc_out_ptr, stream=0):
    self._ck(lib().dfb_debug_edge_gemm(self._h, layer, e_in_ptr, acc_out_ptr, stream))

  def debug_gnn_layer(self, layer, t, h_ptr, e_ptr, stream=0):
    """Run GNN layer `layer` alone at timestep t, in place on device h (V,256) and e (E,256); e rows in the prepared
    graph's stable row-sorted order."""
    self._ck(lib().dfb_debug_gnn_layer(self._h, int(layer), float(t), h_ptr, e_ptr, stream))

  def debug_gnn_layer_timesteps(self, layer, t_values, t_index_ptr, h_ptr, e_ptr, stream=0):
    """debug_gnn_layer with a timestep per element, as encoder_forward_timesteps runs each layer: t_values the distinct
    timesteps (host sequence), t_index_ptr a device int32 (N,) array in the caller's element order, or None."""
    v = np.ascontiguousarray(t_values, dtype=np.float32).reshape(-1)
    self._ck(lib().dfb_debug_gnn_layer_timesteps(self._h, int(layer), v.size, v.ctypes.data_as(C.POINTER(C.c_float)),
                                                 t_index_ptr, h_ptr, e_ptr, stream))

  def debug_head(self, mode, z_ptr, consts=(0, 0, 0, 0), last=0, uniforms_ptr=None, seed=0, step_index=0,
                 instance_seeds_ptr=None, xt_in_ptr=None, xt_out_ptr=None, p_out_ptr=None, net_out_ptr=None,
                 stats_out_ptr=None, stream=0):
    """Run the head of a forward (mode HEAD_*) on device z (R,256): E row-sorted edges (TSP) or V nodes (MIS).  All
    buffers are device pointers in the caller's order; stats_out (segments, 32, 2) gets the GroupNorm mean and rstd."""
    c = (C.c_float * 4)(*[float(x) for x in consts])
    self._ck(lib().dfb_debug_head(self._h, int(mode), z_ptr, c, int(last), uniforms_ptr,
                                  int(seed) & 0xFFFFFFFFFFFFFFFF, int(step_index), instance_seeds_ptr, xt_in_ptr,
                                  xt_out_ptr, p_out_ptr, net_out_ptr, stats_out_ptr, stream))

  def debug_entry(self, diffusion, xt_ptr, t, h0_out_ptr=None, e0_out_ptr=None, tvec_out_ptr=None, h_out_ptr=None,
                  e_out_ptr=None, stream=0):
    """Run the forward up to and including layer 0 at timestep t on device xt; outputs as dfb_debug_entry documents."""
    self._ck(lib().dfb_debug_entry(self._h, int(diffusion), xt_ptr, float(t), h0_out_ptr, e0_out_ptr, tvec_out_ptr,
                                   h_out_ptr, e_out_ptr, stream))

"""Segment ends of the tensor-core edge kernel's message reduction.

The kernel marks, per 32-edge group, the rows that end a (group, node) segment with a warp ballot over the row
table, and walks the group's rows without rereading the table, storing the running sum at each marked row.  These
graphs put the marks where that bookkeeping could slip: every row its own segment, and a last valid row inside a
group (E not a multiple of 32), with a segment that crosses a group boundary before it ends there.  The 128-row (tc)
and 64-row (tc1) tilings see the same 32-edge groups and reduce them in the same order, so their outputs are bitwise
equal.  Both run the same kernel body, so that equality checks the tiling, not the mask; the independent check of the
segment ends is the comparison with the fp64 oracle.  The degree-sequence check needs no GPU."""
import numpy as np
import pytest
import torch

from conftest import rel_linf
from oracle import difusco_oracle as orc
import gpu_util as G

TOL = 1e-4
T_FWD = 700.0


def _from_degrees(deg, seed):
  deg = np.asarray(deg, np.int64)
  V = deg.size
  rows = np.repeat(np.arange(V, dtype=np.int64), deg)
  cols = np.random.default_rng(seed).integers(0, V, rows.size)
  return V, np.stack([rows, cols])


# name -> degree sequence (rows sorted by node)
GRAPHS = {
    # 200 edges: every row ends a segment, the last group holds 8 valid rows
    "singletons": [1] * 200,
    # segment lengths 1, 2, 3 in turn, E = 305 = 9 * 32 + 17: ends on both parities, tail inside group 9
    "short_runs": ([1, 2, 3] * 51)[:152] + [2],
    # singletons, a 2-row node, then a node of degree 45 on rows 276 .. 320: it starts in group 8, fills group 9
    # and ends as the only valid row of group 10
    "tail_span": [1] * 274 + [2, 45],
}


def _case(name):
  V, ei = _from_degrees(GRAPHS[name], seed=sum(map(ord, name)))
  rng = np.random.default_rng(len(name))
  pts = rng.random((V, 2), dtype=np.float32)
  xe = (rng.random(ei.shape[1]) < 0.3).astype(np.float32)
  xv = (rng.random(V) < 0.5).astype(np.float32)
  return V, np.ascontiguousarray(ei), pts, xe, xv


def test_graphs_put_segment_ends_where_intended():
  E = {n: int(np.sum(d)) for n, d in GRAPHS.items()}
  assert E == {"singletons": 200, "short_runs": 305, "tail_span": 321}
  for n in ("singletons", "short_runs", "tail_span"):
    assert E[n] % 32 != 0, n
  ends = np.cumsum(GRAPHS["tail_span"])
  assert ends[-2] == 276 and ends[-1] - 45 < 288 and (ends[-1] - 1) // 32 == 10


def _forward(weights, task, impl, agg, case):
  V, ei, pts, xe, xv = case
  enc = G.encoder(weights, 2, node_only=task == "mis", impl=impl, aggregation=agg)
  if task == "tsp":
    out = enc(G.cu(pts), torch.tensor([T_FWD]), G.cu(xe), G.cu(ei))
  else:
    out = enc(G.cu(xv), torch.tensor([T_FWD]), edge_index=G.cu(ei))
  return out.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("agg", ["sum", "mean", "max"])
@pytest.mark.parametrize("task", ["tsp", "mis"])
@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_segment_ends_tc_equals_tc1_and_oracle(weights2, name, task, agg):
  case = _case(name)
  V, ei, pts, xe, xv = case
  w = orc.Weights(weights2, dtype=torch.float64)
  if task == "tsp":
    ref = orc.encoder_forward_sparse_tsp(w, pts, xe, np.array([T_FWD]), ei, aggregation=agg).numpy()
  else:
    ref = orc.encoder_forward_mis(w, xv, np.array([T_FWD]), ei, aggregation=agg).numpy()
  tc = _forward(weights2, task, "tc", agg, case)
  tc1 = _forward(weights2, task, "tc1", agg, case)
  assert np.array_equal(tc, tc1)
  assert tc.shape == ref.shape and np.isfinite(tc).all()
  err, perr = rel_linf(tc, ref), G.prob_rel(tc, ref)
  assert err < G.TOL["tc"] and perr < TOL, (err, perr)

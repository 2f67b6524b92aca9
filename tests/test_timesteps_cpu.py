"""A timestep per element (the reference's training-step forwards), without a GPU: the fp32 oracle against the
reference's outputs and losses in tests/golden/fwd_tsteps.npz, the Python timestep classification, the code
footprint of the edge kernel that reads a time vector per row, and the inputs of test_gpu_timesteps_edges.py."""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import golden, rel_linf
from oracle import difusco_oracle as orc
from difusco_b200.models.gnn_encoder import MAX_TIMESTEPS, GNNEncoder, timestep_args
import test_gpu_layer_parity as LP
import test_gpu_timesteps_edges as TE
import test_kernel_footprint as fp

TOL = 1e-5   # fp32 restatement vs fp32 reference, as tests/test_oracle_golden.py


def tsteps():
  return golden("fwd_tsteps")


def loss_of(name, out, g):
  """The training step's loss from an encoder output: CE on the labels (categorical) or MSE on epsilon."""
  out = torch.as_tensor(np.asarray(out, np.float32))
  if name in ("tsp_cat", "tsp_ckpt", "mis_cat"):
    return float(F.cross_entropy(out, torch.from_numpy(g[f"{name}/labels"])))
  return float(F.mse_loss(out.squeeze(1), torch.from_numpy(g[f"{name}/eps"])))


def oracle_forward(name, w, g):
  """The oracle's forward of fixture case `name` with oracle weights w."""
  if name in ("tsp_cat", "tsp_ckpt", "tsp_edge_t"):
    t = g[f"{name}/t"][:1] if name == "tsp_ckpt" else g[f"{name}/t"]   # the checkpointed layers run at t[0]
    return orc.encoder_forward_sparse_tsp(w, g[f"{name}/points"], g[f"{name}/xt"], t, g[f"{name}/edge_index"])
  if name == "dense_gauss":
    return orc.encoder_forward_dense(w, g[f"{name}/points"], g[f"{name}/xt"], g[f"{name}/t"])
  return orc.encoder_forward_mis(w, g[f"{name}/xt"], g[f"{name}/t"], g[f"{name}/edge_index"])


CASES = ["tsp_cat", "tsp_ckpt", "dense_gauss", "mis_cat", "mis_gauss", "tsp_edge_t"]


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_per_element_t(name, weights1, weights2):
  g = tsteps()
  w = orc.Weights(weights1 if "gauss" in name else weights2)
  out = oracle_forward(name, w, g).numpy()
  assert out.shape == g[f"{name}/out"].shape
  assert rel_linf(out, g[f"{name}/out"]) < TOL
  if f"{name}/loss" in g.files:
    assert abs(loss_of(name, out, g) / float(g[f"{name}/loss"]) - 1) < 1e-5
    assert abs(loss_of(name, g[f"{name}/out"], g) / float(g[f"{name}/loss"]) - 1) < 1e-6


def test_fixture_pins_what_it_claims():
  g = tsteps()
  for name in ("tsp_cat", "tsp_ckpt"):
    assert g[f"{name}/edge_index"].dtype == np.float32       # the training step's float edge_index
    t = g[f"{name}/t"].reshape(3, -1)
    assert (t == t[:, :1]).all() and t[:, 0].tolist() == [1.0, 1000.0, 517.0]
    xt = np.abs(g[f"{name}/xt"])
    assert xt.min() >= 1.0 and xt.max() <= 1.05 and len(np.unique(xt)) > 100   # jittered +-1
  assert not np.array_equal(g["tsp_cat/out"], g["tsp_ckpt/out"])
  assert len(np.unique(g["tsp_edge_t/t"])) > 300 and g["tsp_edge_t/t"].size % 32
  for name in ("mis_cat", "mis_gauss"):
    assert g[f"{name}/t"].tolist() == np.repeat([77.0, 904.0], g[f"{name}/sizes"]).tolist()


def test_oracle_fp64_per_element_t(weights2):
  g = tsteps()
  out = oracle_forward("tsp_edge_t", orc.Weights(weights2, torch.float64), g)
  assert out.dtype == torch.float64
  assert rel_linf(out.numpy(), g["tsp_edge_t/out"]) < 2e-5


# ---- timestep classification (models/gnn_encoder.py:timestep_args) ----
@pytest.mark.parametrize("t", [torch.tensor([37.0]), torch.full((6,), 37.0), torch.tensor(37.0),
                               torch.full((6,), 37, dtype=torch.int64)])
def test_one_timestep_is_the_scalar_call(t):
  r = timestep_args(t, 6)
  assert isinstance(r, float) and r == 37.0


def test_per_element_timesteps_give_values_and_index():
  t = torch.tensor([5.0, 900.0, 5.0, 1.0, 900.0])
  values, index = timestep_args(t, 5)
  assert values.dtype == np.float32 and values.tolist() == [1.0, 5.0, 900.0]
  assert index.dtype == torch.int32 and index.tolist() == [1, 2, 1, 0, 2]
  assert np.array_equal(values[index.numpy()], t.numpy())


def test_checkpoint_quirk_runs_every_element_at_the_first_t():
  assert timestep_args(torch.tensor([3.0, 900.0, 1.0]), 3, first_only=True) == 3.0
  assert timestep_args(torch.tensor([3.0, 900.0]), 7, first_only=True) == 3.0   # any length, as the reference


def test_host_per_element_timesteps_for_a_device_model_raise_not_implemented():
  t = torch.tensor([3.0, 900.0, 1.0])
  for first_only in (False, True):
    with pytest.raises(NotImplementedError, match="device"):
      timestep_args(t, 3, first_only, device=torch.device("cuda", 0))
  assert timestep_args(torch.full((3,), 7.0), 3, device=torch.device("cuda", 0)) == 7.0
  assert timestep_args(torch.tensor([7.0]), 3, device=torch.device("cuda", 0)) == 7.0
  assert isinstance(timestep_args(t, 3, device=torch.device("cpu")), tuple)


@pytest.mark.parametrize("n_t", [0, 2, 5])
def test_wrong_timestep_length_raises_value_error(n_t):
  with pytest.raises(ValueError, match="timesteps"):
    timestep_args(torch.arange(n_t, dtype=torch.float32), 4)


def test_too_many_distinct_timesteps_raise_not_implemented():
  n = MAX_TIMESTEPS + 1
  assert isinstance(timestep_args(torch.arange(1, MAX_TIMESTEPS + 1).float(), MAX_TIMESTEPS), tuple)
  with pytest.raises(NotImplementedError, match="distinct timesteps"):
    timestep_args(torch.arange(n).float(), n)


@pytest.mark.parametrize("kind", ["tsp", "mis", "dense"])
def test_forward_rejects_wrong_timestep_length_before_device_work(kind):
  enc = GNNEncoder(2, 256, 2, sparse=kind != "dense", node_feature_only=kind == "mis")
  t = torch.tensor([1.0, 2.0, 3.0])
  ei = torch.tensor([[0, 0, 1, 1], [0, 1, 0, 1]])
  with pytest.raises(ValueError, match="timesteps"):
    if kind == "tsp":
      enc(torch.rand(2, 2), t, torch.zeros(4), ei)
    elif kind == "mis":
      enc(torch.zeros(2), t, edge_index=ei)
    else:
      enc(torch.rand(2, 5, 2), t, torch.zeros(2, 5, 5))


# ---- code footprint of the per-row time-vector edge kernel ----
KERNEL_TROWS = "_ZN3dfb22k_edge_layer_wg2_trowsE14CUtensorMap_stNS_8TcParamsE"


def test_trows_edge_kernel_text_within_budget():
  sizes = [int(m.group(1), 16) for m in re.finditer(
      r"^\s*\w+\s+\w+\s+(\w+)\s.*PROGBITS.*\s\.text\." + KERNEL_TROWS + r"\s*$", fp._dump("-elf"), re.M)]
  assert sizes, "no .text section for k_edge_layer_wg2_trows in the library"
  assert max(sizes) <= fp.TEXT_BUDGET, f"k_edge_layer_wg2_trows .text is {max(sizes):#x}, budget {fp.TEXT_BUDGET:#x}"


def test_trows_edge_kernel_registers_and_spills():
  m = re.search(r"Function " + KERNEL_TROWS + r":\s*\n\s*REG:(\d+) STACK:(\d+)", fp._dump("-res-usage"))
  assert m, "no resource usage for k_edge_layer_wg2_trows in the library"
  assert int(m.group(1)) == fp.REGS
  assert int(m.group(2)) <= fp.STACK_LIMIT, f"k_edge_layer_wg2_trows spill frame is {m.group(2)} bytes"


# ---- the inputs of test_gpu_timesteps_edges.py are what they claim to be ----

@pytest.mark.parametrize("case", TE.SHUF_TSP)
def test_shuffled_graphs_are_unsorted(case):
  """Every shuffled graph with two or more distinct rows reaches the kernels in an order the row sort changes, so
  the lookup's perm branch runs (tiny1 and tiny2 have fewer edges than that can show)."""
  V, ei, *_ = LP._case(case)
  if len(np.unique(ei[0])) < 2:
    pytest.skip(f"{case}: one distinct row")
  assert (np.diff(ei[0]) < 0).any(), case
  assert not np.array_equal(TE._sorted_perm(ei), np.arange(ei.shape[1]))


@pytest.mark.parametrize("case", ["tsp_shuf", "hub_shuf", "degseq_shuf", "isolated_shuf", "dup_shuf", "tiny129_shuf"])
def test_block_pattern_changes_exactly_at_warpgroup_and_tile_boundaries(case):
  V, ei, *_ = LP._case(case)
  t = TE.t_pattern(case, "tsp", "block")[TE._sorted_perm(ei)]   # sorted order
  change = np.flatnonzero(np.diff(t) != 0) + 1                   # first sorted row of each new run
  assert {64, 128} <= set(change.tolist()), case
  assert (change % 64 == 0).all(), case
  assert len(np.unique(t[:128])) == 2 and len(np.unique(t[:192])) == 3
  values, index = TE.values_index(TE.t_pattern(case, "tsp", "block"))
  assert np.array_equal(values[index], TE.t_pattern(case, "tsp", "block"))


def test_nan_rows_are_the_boundary_rows_through_the_permutation():
  V, ei, *_ = LP._case("hub_shuf")
  rows = TE.nan_rows("hub_shuf", "tsp")
  pos = np.argsort(TE._sorted_perm(ei))[rows]                    # sorted position of each chosen caller edge
  assert sorted(pos.tolist()) == [0, 63, 64, 127, 128, ei.shape[1] - 1]
  assert TE.nan_rows("mis", "mis").tolist() == [0, 63, 64, 127, 128, 149]


def test_4096_timesteps_are_distinct_non_integers_in_fp32():
  v = TE.max_t_values()
  assert v.dtype == np.float32 and v.size == TE.MAX_T == MAX_TIMESTEPS
  assert len(np.unique(v)) == v.size and (v != np.round(v)).all() and v.min() > 1 and v.max() < 1000
  pts, ei, xt, index = TE._max_t_case()
  assert ei.shape[1] >= TE.MAX_T and set(index.tolist()) == set(range(TE.MAX_T))
  assert (np.diff(ei[0]) < 0).any()


def test_oracle_per_row_layer_step_at_one_t_is_the_single_t_call(weights2):
  V, ei, *_ = LP._case("tsp_shuf")
  W = orc.Weights(weights2, torch.float64)
  h, e, temb = LP._initial_state(W, "tsp", "tsp_shuf")
  row, col = torch.as_tensor(ei[0]), torch.as_tensor(ei[1])
  temb_rows = orc._time_emb(W, torch.full((ei.shape[1],), LP.T_LAYER, dtype=torch.float32))
  for time_on_edge, rows in ((True, temb_rows), (False, temb_rows[:V])):
    a = orc.layer_step(W, 3, h, e, row, col, temb, time_on_edge)
    b = orc.layer_step(W, 3, h, e, row, col, rows, time_on_edge)
    for x, y in zip(a, b):   # not bitwise: the time MLP runs as a GEMM on E rows and as a GEMV on one
      assert float((x - y).abs().max() / y.abs().max()) < 1e-14


def test_oracle_per_element_forward_is_invariant_to_edge_order(weights2):
  """So one oracle run on the sorted graph serves the shuffled one (test_gpu_timesteps_edges.py)."""
  pts, ei = TE.syn.tsp_sparse_batch(50, 20, 2, seed=5)
  rng = np.random.default_rng(6)
  t = rng.integers(1, 1001, ei.shape[1]).astype(np.float32)
  xt = (rng.random(ei.shape[1]) < 0.3).astype(np.float32)
  W = orc.Weights(weights2, torch.float64)
  ref = orc.encoder_forward_sparse_tsp(W, pts, xt, t, ei).numpy()
  eis, q = TE._shuffle(ei, 7)
  got = TE._unshuffle(orc.encoder_forward_sparse_tsp(W, pts, xt[q], t[q], eis).numpy(), q)
  assert rel_linf(got, ref) < 1e-12
  V = 150
  eim = TE.syn.er_graph_edge_index(V, 0.05, seed=8)
  tv = rng.integers(1, 1001, V).astype(np.float32)
  xv = (rng.random(V) < 0.5).astype(np.float32)
  refm = orc.encoder_forward_mis(W, xv, tv, eim).numpy()
  eims, _ = TE._shuffle(eim, 9)
  assert rel_linf(orc.encoder_forward_mis(W, xv, tv, eims).numpy(), refm) < 1e-12

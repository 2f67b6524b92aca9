"""Argument checks of the batched solve path that run before any device work: instance_seeds, the multi-instance 2-opt
arrays and solve_batch's seeds and batch layout.  No GPU needed."""
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from difusco_b200 import _cabi
from difusco_b200.pl_meta_model import COMetaModel
from difusco_b200.pl_tsp_model import TSPModel
from difusco_b200.utils import tsp_utils as tu


def test_instance_seeds_array():
  assert _cabi.instance_seeds_array([1, 2 ** 64 - 1, np.int64(3)], 3).dtype == np.uint64
  assert list(_cabi.instance_seeds_array((5,), 1)) == [5]
  for bad, n in (([1, 2], 3), ([1, 2, 3], 2), ([1.5], 1), ([True], 1), ([-1], 1), ([2 ** 64], 1), (7, 1),
                 ("12", 2), ([], 1)):
    with pytest.raises(ValueError):
      _cabi.instance_seeds_array(bad, n)


def test_two_opt_instances_arrays():
  rng = np.random.default_rng(0)
  pts = [rng.random((4, 2)), rng.random((3, 2))]
  tours = [np.array([[0, 1, 2, 3, 0], [0, 2, 1, 3, 0]]), np.array([[0, 1, 2, 0]])]
  P, nptr, tptr, T = _cabi.two_opt_instances_arrays(pts, tours)
  assert P.shape == (7, 2) and P.dtype == np.float64
  assert list(nptr) == [0, 4, 7] and list(tptr) == [0, 2, 3] and T.tolist() == [0, 1, 2, 3, 0, 0, 2, 1, 3, 0, 0, 1, 2, 0]
  bad = [
      ([pts[0]], tours),                                   # count mismatch
      ([], []),                                            # no instance
      ([rng.random((2, 2))], [np.array([[0, 1, 0]])]),     # n < 3
      ([rng.random((4, 3))], [tours[0]]),                  # points not (n, 2)
      ([pts[0].astype(np.int64)], [tours[0]]),             # integer points
      ([pts[0]], [tours[0][:, :-1]]),                      # rows of n entries
      ([pts[0]], [tours[0].astype(np.float64)]),           # float tours
      ([pts[0]], [np.zeros((0, 5), np.int64)]),            # no tour
      ([pts[0]], [tours[0] + 1]),                          # id n
      ([pts[0]], [tours[0] - 1]),                          # negative id
  ]
  for p, t in bad:
    with pytest.raises(ValueError):
      _cabi.two_opt_instances_arrays(p, t)
    with pytest.raises(ValueError):
      tu.batched_two_opt_instances(p, t)                 # checked before a device is looked for


def test_batched_two_opt_instances_needs_cuda():
  with pytest.raises(RuntimeError):
    tu.batched_two_opt_instances([np.random.default_rng(1).random((4, 2))], [np.array([[0, 1, 2, 3, 0]])],
                                 device="cpu")


def test_solve_seeds():
  gens = COMetaModel._solve_seeds([3, np.int64(4)], 2)
  a = COMetaModel._round_seed(gens[0])
  assert a == COMetaModel._round_seed(torch.Generator().manual_seed(3))
  for bad, n in (([1], 2), ([1.0], 1), ([False], 1), ([-2], 1), ([2 ** 63], 1), (5, 1)):
    with pytest.raises(ValueError):
      COMetaModel._solve_seeds(bad, n)


def _args(**kw):
  a = dict(diffusion_type="categorical", diffusion_schedule="linear", diffusion_steps=1000, sparse_factor=4,
           n_layers=2, hidden_dim=256, aggregation="sum", parallel_sampling=1, sequential_sampling=1,
           inference_schedule="cosine", inference_diffusion_steps=2, inference_trick="ddim")
  a.update(kw)
  return NS(**a)


def test_sparse_batch_layout_checks():
  m = TSPModel(_args())
  g = NS(x=torch.rand(7, 2), edge_index=torch.tensor([[0, 1, 2, 3, 4, 5, 6], [1, 2, 0, 4, 5, 6, 3]]))
  good = (torch.arange(2), g, torch.tensor([3, 4]), torch.tensor([3, 4]), torch.arange(9))
  inst = m._instances(good)
  assert [p.shape[0] for p, _, _ in inst] == [3, 4]
  assert inst[1][1].tolist() == [[0, 1, 2, 3], [1, 2, 3, 0]] and inst[1][2].tolist() == [4, 5, 6, 7, 8]
  for bad in ((torch.arange(2), g, torch.tensor([3, 3]), torch.tensor([3, 4]), torch.arange(9)),
              (torch.arange(2), g, torch.tensor([3, 4]), torch.tensor([4, 3]), torch.arange(9)),
              (torch.arange(2), g, torch.tensor([3, 4]), torch.tensor([3, 4]), torch.arange(8))):
    with pytest.raises(ValueError):
      m._instances(bad)


def test_solve_batch_rejects_bad_seeds_before_device_work():
  m = TSPModel(_args())
  g = NS(x=torch.rand(3, 2), edge_index=torch.tensor([[0, 1, 2], [1, 2, 0]]))
  batch = (torch.arange(1), g, torch.tensor([3]), torch.tensor([3]), torch.arange(4))
  for seeds in ([], [1, 2], [0.5]):
    with pytest.raises(ValueError):
      m.solve_batch(batch, seeds)
  m = TSPModel(_args(save_numpy_heatmap=True))
  with pytest.raises(NotImplementedError):
    m.solve_batch(batch, [1])

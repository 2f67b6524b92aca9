"""solve_batches' argument checks, which run before any device work, and its laziness.  No GPU needed."""
from types import SimpleNamespace as NS

import pytest
import torch

from difusco_b200.pl_mis_model import MISModel
from difusco_b200.pl_tsp_model import TSPModel


def _args(**kw):
  a = dict(diffusion_type="categorical", diffusion_schedule="linear", diffusion_steps=1000, sparse_factor=4,
           n_layers=2, hidden_dim=256, aggregation="sum", parallel_sampling=1, sequential_sampling=1,
           inference_schedule="cosine", inference_diffusion_steps=2, inference_trick="ddim")
  a.update(kw)
  return NS(**a)


def _tsp_batch():
  g = NS(x=torch.rand(3, 2), edge_index=torch.tensor([[0, 1, 2], [1, 2, 0]]))
  return (torch.arange(1), g, torch.tensor([3]), torch.tensor([3]), torch.arange(4))


def _mis_batch():
  g = NS(x=torch.ones(3), edge_index=torch.tensor([[0, 1, 2], [1, 2, 0]]))
  return (torch.arange(1), g, torch.tensor([3]))


def test_empty_stream_yields_nothing():
  assert list(TSPModel(_args()).solve_batches([], [])) == []
  assert list(MISModel(_args()).solve_batches(iter([]), iter([]))) == []


@pytest.mark.parametrize("model,batch", [(TSPModel, _tsp_batch), (MISModel, _mis_batch)])
def test_seed_lists_are_checked_before_device_work(model, batch):
  m = model(_args())
  for batches, seeds in (([batch()], []),             # fewer seed lists than batches
                         ([], [[1]]),                 # more seed lists than batches
                         ([batch()], [[1, 2]]),       # two seeds for one instance
                         ([batch()], [[]]),
                         ([batch()], [[0.5]]),
                         ([batch()], [7])):
    with pytest.raises(ValueError):
      next(m.solve_batches(batches, seeds))


def test_malformed_batch_and_saved_heat_maps_are_rejected():
  bad = _tsp_batch()[:2] + (torch.tensor([4]),) + _tsp_batch()[3:]
  with pytest.raises(ValueError):
    next(TSPModel(_args()).solve_batches([bad], [[1]]))
  with pytest.raises(NotImplementedError):
    next(TSPModel(_args(save_numpy_heatmap=True)).solve_batches([_tsp_batch()], [[1]]))


def test_the_generator_is_lazy():
  taken = []

  def batches():
    taken.append(1)
    yield _tsp_batch()

  gen = TSPModel(_args()).solve_batches(batches(), [[1]])
  assert taken == []                                  # nothing is read before the first result is asked for
  with pytest.raises(RuntimeError):                   # then the first batch is enqueued, which needs a CUDA device
    next(gen)
  assert taken == [1]

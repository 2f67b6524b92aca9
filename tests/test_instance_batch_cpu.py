"""node_ptr on the Python surface (per-instance GroupNorm of a block-diagonal batch): the argument checks that run
before any device work, so they hold without a GPU."""
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from difusco_b200 import synthetic as syn
from difusco_b200.models.gnn_encoder import GNNEncoder, node_ptr_array
from difusco_b200.pl_tsp_model import TSPModel


def test_synthetic_node_ptr():
  p = syn.node_ptr([3, 1, 5])
  assert p.dtype == np.int64 and p.tolist() == [0, 3, 4, 9]
  assert syn.node_ptr([7]).tolist() == [0, 7]


@pytest.mark.parametrize("ptr", [[0, 3, 9], (0, 3, 9), np.array([0, 3, 9], np.int32), np.array([0, 3, 9], np.uint16),
                                 torch.tensor([0, 3, 9]), torch.tensor([0, 3, 9], dtype=torch.int32)])
def test_node_ptr_accepts_integer_sequences_and_tensors(ptr):
  a = node_ptr_array(ptr)
  assert a.dtype == np.int64 and a.tolist() == [0, 3, 9]


@pytest.mark.parametrize("ptr", [[], [0], [[0, 3], [3, 9]], [0.0, 3.0], np.array([0, 3], np.float32),
                                 [True, False], torch.tensor([0.0, 3.0]), torch.tensor([True, True]),
                                 torch.tensor([[0, 3]]), torch.tensor(3)])
def test_node_ptr_rejects_wrong_shape_or_dtype(ptr):
  with pytest.raises(ValueError):
    node_ptr_array(ptr)


def test_dense_forward_rejects_node_ptr():
  enc = GNNEncoder(2, 256, 2, sparse=False)
  with pytest.raises(ValueError, match="node_ptr"):
    enc(torch.zeros(1, 5, 2), torch.tensor([1.0]), torch.zeros(1, 5, 5), node_ptr=[0, 5])


def test_set_graph_checks_node_ptr_before_device_work():
  enc = GNNEncoder(2, 256, 2, sparse=True)
  ei = torch.tensor([[0, 1], [1, 0]])
  with pytest.raises(ValueError):
    enc.set_graph(ei, 2, node_ptr=[0.0, 2.0])
  with pytest.raises(ValueError):
    enc.set_graph(ei, 2, node_ptr=torch.tensor([[0, 2]]))
  with pytest.raises(ValueError, match="not both"):
    enc.set_graph(ei, 2, gn_segments=2, node_ptr=[0, 1, 2])


def test_dense_tsp_model_rejects_node_ptr():
  args = NS(diffusion_type="categorical", diffusion_schedule="linear", diffusion_steps=1000, sparse_factor=-1,
            n_layers=2, hidden_dim=256, aggregation="sum", parallel_sampling=1, sequential_sampling=1,
            inference_schedule="cosine", inference_diffusion_steps=5, inference_trick="ddim")
  m = TSPModel(args)
  with pytest.raises(ValueError, match="node_ptr"):
    m._prepare(torch.zeros(2, 5, 2), None, torch.device("cpu"), node_ptr=[0, 5, 10])

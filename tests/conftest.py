import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
  config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def golden(name):
  return np.load(os.path.join(GOLDEN, name + ".npz"))


def rel_linf(a, b):
  """L-inf error relative to the L-inf scale of the reference tensor b."""
  a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
  return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.fixture(scope="session")
def weights2():
  from difusco_b200 import synthetic as syn
  return syn.make_encoder_weights(seed=0, out_channels=2)


@pytest.fixture(scope="session")
def weights1():
  from difusco_b200 import synthetic as syn
  return syn.make_encoder_weights(seed=1, out_channels=1)

"""oracle/_ref (the UNMODIFIED reference files that `bench.py --impl reference` runs, copied by oracle/make_ref.py when
build() finds the reference tree): every file matches the sha256 recorded from the reference in
tests/golden/ref_copy.npz, the copy's manifest is consistent, and the copy's own GNNEncoder forward reproduces the
reference's output stored there (run in a subprocess: the dependency shims install stand-in modules that must not leak
into the other tests).  The stored output is also pinned against the oracle port, so that check runs everywhere."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import make_ref  # noqa: E402


def _sha(path):
  return hashlib.sha256(open(path, "rb").read()).hexdigest()


def _have_copy():
  if os.path.isdir(make_ref.SRC):
    return make_ref.make(verbose=False) is not None
  return make_ref.available()


def test_ref_copy_is_byte_identical_and_manifest_matches():
  g = golden("ref_copy")
  recorded = dict(zip(g["files"].tolist(), g["sha256"].tolist()))
  assert sorted(recorded) == sorted(make_ref.FILES)
  # no reference source may enter the history: the directory is git-ignored
  assert "oracle/_ref/" in open(os.path.join(ROOT, ".gitignore")).read()
  if not _have_copy():
    pytest.skip("oracle/_ref not built (build() copies it where the reference tree is present)")
  manifest = {}
  for line in open(os.path.join(make_ref.DST, "MANIFEST.sha256")):
    h, rel = line.split()
    manifest[rel] = h
  assert sorted(manifest) == sorted(make_ref.FILES)
  for rel in make_ref.FILES:
    assert _sha(os.path.join(make_ref.DST, rel)) == manifest[rel] == recorded[rel], rel   # unmodified


def test_recorded_reference_forward_matches_oracle_port():
  from difusco_b200 import synthetic as syn
  from oracle import difusco_oracle as orc
  w = syn.make_encoder_weights(0, out_channels=2)
  pts, ei = syn.tsp_sparse_batch(30, 7, 2, seed=5)
  xt = (syn.initial_noise(ei.shape[1], 3) > 0).astype(np.float32)
  out = orc.encoder_forward_sparse_tsp(orc.Weights(w), pts, xt, np.array([321.0], np.float32), ei).numpy()
  ref = golden("ref_copy")["out"]
  assert np.abs(ref - out).max() / np.abs(ref).max() < 1e-5


_CHILD = r"""
import os, sys
import numpy as np, torch
ROOT = sys.argv[1]
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "oracle")); sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import ref_shims
ref_shims.install(os.path.join(ROOT, "oracle", "_ref", "difusco"))
from models.gnn_encoder import GNNEncoder as RefEncoder          # the reference's own class from the copy
from difusco_b200 import synthetic as syn
torch.manual_seed(0)
w = syn.make_encoder_weights(0, out_channels=2)
enc = RefEncoder(12, 256, 2, aggregation="sum", sparse=True, use_activation_checkpoint=False, node_feature_only=False)
enc.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
enc.eval()
pts, ei = syn.tsp_sparse_batch(30, 7, 2, seed=5)
xt = (syn.initial_noise(ei.shape[1], 3) > 0).astype(np.float32)
with torch.no_grad():
  out = enc(torch.from_numpy(pts), torch.tensor([321.0]), torch.from_numpy(xt), torch.from_numpy(ei)).numpy()
ref = np.load(os.path.join(ROOT, "tests", "golden", "ref_copy.npz"))["out"]
err = float(np.abs(ref - out).max() / np.abs(ref).max())
print("REL_ERR", err)
assert err < 1e-5, err
"""


def test_ref_copy_forward_matches_recorded_reference():
  if not _have_copy():
    pytest.skip("oracle/_ref not built (build() copies it where the reference tree is present)")
  r = subprocess.run([sys.executable, "-c", _CHILD, ROOT], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
  assert r.returncode == 0 and "REL_ERR" in r.stdout, r.stdout[-2000:]

"""oracle/philox.py, the host restatement of the in-kernel sampler, against the Random123 known-answer vectors
(Philox4x32-10).  The GPU tests compare the kernel's samples with this module element for element."""
import numpy as np
import pytest

from oracle import philox

KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox4x32_10_known_answers(ctr, key, want):
  got = philox.philox4x32_10(ctr, key)
  assert [int(x) for x in got] == list(want)


def test_philox_vectorised_matches_scalar_calls():
  ctr = [np.array([0, 0xFFFFFFFF, 0x243F6A88], np.uint64), np.array([0, 0xFFFFFFFF, 0x85A308D3], np.uint64),
         np.array([0, 0xFFFFFFFF, 0x13198A2E], np.uint64), np.array([0, 0xFFFFFFFF, 0x03707344], np.uint64)]
  got = philox.philox4x32_10(ctr, (0, 0))
  for i in range(3):
    one = philox.philox4x32_10([c[i] for c in ctr], (0, 0))
    assert [int(w[i]) for w in got] == [int(x) for x in one]


def test_uniform_and_normal_use_the_documented_counter_layout():
  seed, step = (0x1234ABCD << 32) | 0x9E3779B9, 7
  elem = np.array([0, 1, 5, (3 << 32) | 11], np.uint64)
  r0 = philox.philox4x32_10((elem & 0xFFFFFFFF, elem >> 32, step, 0), (seed & 0xFFFFFFFF, seed >> 32))
  u = philox.uniform(seed, step, elem)
  assert u.dtype == np.float32
  assert np.array_equal(u, (r0[0] >> 8).astype(np.float32) * np.float32(2.0 ** -24))
  r1 = philox.philox4x32_10((elem & 0xFFFFFFFF, elem >> 32, step, 1), (seed & 0xFFFFFFFF, seed >> 32))
  u1 = ((r1[0] >> 8).astype(np.float32) + np.float32(0.5)).astype(np.float64) * 2.0 ** -24
  u2 = (r1[1] >> 8) * 2.0 ** -24
  assert np.array_equal(philox.normal(seed, step, elem), np.sqrt(-2 * np.log(u1)) * np.cos(2 * np.pi * u2))
  # every word of the counter and key changes the draw: the seed's high word and the element's high word included
  assert not np.array_equal(u, philox.uniform(seed & 0xFFFFFFFF, step, elem))
  assert philox.uniform(seed, step, elem[3]) != philox.uniform(seed, step, elem[3] & 0xFFFFFFFF)
  assert not np.array_equal(u, philox.uniform(seed, step + 1, elem))


def test_uniform_and_normal_distributions():
  from scipy import stats
  n = 200_000
  u = philox.uniform(2 ** 40 + 3, 1, np.arange(n, dtype=np.uint64))
  assert u.min() >= 0.0 and u.max() < 1.0
  assert stats.kstest(u, "uniform").pvalue > 1e-3
  z = philox.normal(2 ** 40 + 3, 1, np.arange(n, dtype=np.uint64))
  assert np.isfinite(z).all()
  assert stats.kstest(z, "norm").pvalue > 1e-3

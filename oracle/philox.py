"""Host restatement of the in-kernel sampler (difusco_b200/csrc/common.cuh).  TEST INFRASTRUCTURE, NOT PRODUCT.

Philox4x32-10 (Salmon, Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC 2011) in plain
numpy, vectorised over elements.  The device keys every draw by the caller's element index:
    counter = (elem_lo, elem_hi, step, w3),  key = (seed_lo, seed_hi)
with w3 = 0 for the Bernoulli uniform and w3 = 1 for the Gaussian normal, so a test can recompute the exact
draw the kernel used for any element and compare the sampled state against it.
"""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def philox4x32_10(ctr, key):
  """ctr: 4 arrays (or ints) of uint32 words, key: 2 words.  Returns the 4 output words as uint32 arrays."""
  c = [np.asarray(x, dtype=np.uint64) & _MASK for x in ctr]
  c = np.broadcast_arrays(*c)
  c = [x.copy() for x in c]
  k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
  for _ in range(10):
    p0 = M0 * c[0]          # < 2^64: no wrap in uint64
    p1 = M1 * c[2]
    c = [((p1 >> _S32) ^ c[1] ^ np.uint64(k0)) & _MASK, p1 & _MASK,
         ((p0 >> _S32) ^ c[3] ^ np.uint64(k1)) & _MASK, p0 & _MASK]
    k0 = (k0 + W0) & 0xFFFFFFFF
    k1 = (k1 + W1) & 0xFFFFFFFF
  return [x.astype(np.uint32) for x in c]


def _words(seed, step, elem, w3):
  elem = np.asarray(elem, dtype=np.uint64)
  seed = int(seed) & 0xFFFFFFFFFFFFFFFF
  return philox4x32_10((elem & _MASK, elem >> _S32, np.uint64(int(step) & 0xFFFFFFFF), np.uint64(w3)),
                       (seed & 0xFFFFFFFF, seed >> 32))


def uniform(seed, step, elem):
  """U[0,1) with 24 random bits, bit for bit the device's philox_uniform: (r.x >> 8) * 2^-24 (float32)."""
  r = _words(seed, step, elem, 0)
  return ((r[0] >> np.uint32(8)).astype(np.float64) * 2.0 ** -24).astype(np.float32)


def normal(seed, step, elem):
  """N(0,1) from the device's philox_normal words (counter word 3 = 1), Box-Muller evaluated in float64 on the
  device's float32 inputs: u1 = fl32(fl32(r.x >> 8) + 0.5) 2^-24 in (0,1] (the float32 sum rounds to even once
  r.x >> 8 >= 2^23, exactly as on the device), u2 = (r.y >> 8) 2^-24, z = sqrt(-2 ln u1) cos(2 pi u2)."""
  r = _words(seed, step, elem, 1)
  u1 = ((r[0] >> np.uint32(8)).astype(np.float32) + np.float32(0.5)).astype(np.float64) * 2.0 ** -24
  u2 = (r[1] >> np.uint32(8)).astype(np.float64) * 2.0 ** -24
  return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)

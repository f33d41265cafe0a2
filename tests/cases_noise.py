"""The seeded noise streams of the kernels (include/idiff_b200.h, "Seeded noise") restated in numpy: Philox4x32-10 in
integers, then Box-Muller in float64.  Every mirror of a kernel's noise draws through `normals`.

* `philox4x32(ctr, key)`: Philox4x32-10 on arrays.
* `DDIM_ETA`, `START`, `POSTERIOR`, `INPAINT`: counter word 3 of each stream (csrc/common.cuh NoiseStream); `STREAMS`
  names them.
* `normals(seed, stream, word2, n)`: z_0 .. z_{n-1} of a stream: Philox4x32-10 with key (seed lo, seed hi) and counter
  (c lo, c hi, word2, stream) for c = i // 4, then Box-Muller on the word pairs (v0, v1) and (v2, v3).
"""
from __future__ import annotations

import numpy as np

# ------------------------------------------------------------------------------------------------
# Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11)
# ------------------------------------------------------------------------------------------------
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)


def philox4x32(ctr, key):
    """Philox4x32-10 on arrays: ctr (4, n) and key (2, n) of uint32 (or broadcastable) -> (4, n) uint32."""
    c = [np.asarray(v, dtype=np.uint32).astype(np.uint64) for v in ctr]
    k0, k1 = (np.asarray(v, dtype=np.uint32) for v in key)
    with np.errstate(over="ignore"):
        for r in range(10):
            p0, p1 = _M0 * c[0], _M1 * c[2]
            c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0.astype(np.uint64), p1 & _LO,
                 (p0 >> np.uint64(32)) ^ c[3] ^ k1.astype(np.uint64), p0 & _LO]
            k0, k1 = k0 + _W0, k1 + _W1
    return np.stack([np.broadcast_to(v, np.broadcast(*c).shape) for v in c]).astype(np.uint32)


# word 2 of each stream: DDIM_ETA the step index, START 0, POSTERIOR the image's index in its request, INPAINT t
DDIM_ETA, START, POSTERIOR, INPAINT = 0, 1, 2, 3
STREAMS = {"ddim_eta": DDIM_ETA, "start": START, "posterior": POSTERIOR, "inpaint": INPAINT}


def normals(seed: int, stream: int, word2: int, n: int) -> np.ndarray:
    """The standard normals z_0 .. z_{n-1} of `stream` at (seed, word2), float64."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    c = np.arange((n + 3) // 4, dtype=np.uint64)
    v = philox4x32([c & _LO, c >> np.uint64(32), np.full(c.shape, word2, np.uint32), np.full(c.shape, stream, np.uint32)],
                   [np.uint32(seed & 0xFFFFFFFF), np.uint32(seed >> 32)]).astype(np.float64)
    u = (v + 0.5) * 2.0 ** -32
    z = np.empty((c.shape[0], 4))
    for a, b in ((0, 1), (2, 3)):
        r = np.sqrt(-2.0 * np.log(u[a]))
        z[:, a], z[:, b] = r * np.cos(2 * np.pi * u[b]), r * np.sin(2 * np.pi * u[b])
    return z.reshape(-1)[:n]

"""NumPy restatement of the device random streams of the MultiVAE / MultiDAE kernels.  TEST INFRASTRUCTURE ONLY.

`philox4x32` is eb::Philox::gen (elliot_b200/csrc/common.cuh): Philox4x32-10 (Salmon et al. 2011) with key = seed and
counter words (ctr lo, ctr hi, attempt, 0x454c4c49), vectorised over counters.  On top of it:
  - `keep`: the dropout rule of eb_vae_embed_fwd / _bwd (vae.cu): draw (seed, batch row b, position p in the user's CSR
    row), the item is dropped when (r[0] >> 8) / 2^24 < drop;
  - `reparam_eps`: the N(0, 1) noise of eb_vae_reparam_fwd / _bwd: draw (seed, step, element e = b L + l), Box-Muller on
    r[0], r[1] in fp64 (the device evaluates it with __logf / __cosf, so it agrees to ~1e-6, not bit for bit).
"""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
TAG = 0x454C4C49
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 of the counter words c0..c3 (arrays, broadcast together) under the key (k0, k1): four uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & MASK32 for x in np.broadcast_arrays(c0, c1, c2, c3)]
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]                         # 32 x 32 -> 64-bit products, exact in uint64
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & MASK32,
             (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1), p0 & MASK32]
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return [x.astype(np.uint32) for x in c]


def gen(seed, ctr, attempt):
    """eb::Philox::gen(seed, ctr, attempt) over arrays of 64-bit counters and 32-bit attempts."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    ctr = np.asarray(ctr, dtype=np.uint64)
    return philox4x32(ctr & MASK32, ctr >> np.uint64(32), np.asarray(attempt, dtype=np.uint64), TAG, seed, seed >> 32)


def keep(seed, b, p, drop):
    """Dropout keep bits of (batch row b, position p within the user's CSR row) at rate `drop` (drop == 0: all kept)."""
    b, p = np.broadcast_arrays(np.asarray(b, dtype=np.uint64), np.asarray(p, dtype=np.uint64))
    if drop <= 0:
        return np.ones(b.shape, dtype=bool)
    r0 = gen(seed, b, p)[0]
    # the device compares in fp32: (float)(r >> 8) * 2^-24 is exact (24-bit integer times a power of two), drop rounds to fp32
    return (r0 >> np.uint32(8)).astype(np.float64) * 2.0 ** -24 >= np.float64(np.float32(drop))


def reparam_eps(seed, step, n):
    """The noise of elements e = 0 .. n-1 (e = b L + l) at `step`, in fp64."""
    e = np.arange(n, dtype=np.uint64)
    r = gen(seed, np.full(n, step, dtype=np.uint64), e)
    u1 = ((r[0] >> np.uint32(8)).astype(np.float64) + 0.5) * 2.0 ** -24
    u2 = (r[1] >> np.uint32(8)).astype(np.float64) * 2.0 ** -24
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def csr_keep_mask(seed, indptr, indices, rows, n_items, drop):
    """Dense [B][n_items] fp64 keep mask of the batch rows `rows` (user ids) for the train CSR (indptr, indices): 1 where
    the user's item is kept, 0 where it is dropped or absent."""
    K = np.zeros((len(rows), n_items))
    for b, u in enumerate(rows):
        beg, end = int(indptr[u]), int(indptr[u + 1])
        K[b, indices[beg:end]] = keep(seed, b, np.arange(end - beg), drop)
    return K

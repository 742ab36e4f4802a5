"""NumPy restatement of the on-device sampler (bagel_sample_rows_bf16), independent of the product: Philox4x32-10
(Salmon et al., SC'11) and the Gumbel-max scores in fp64."""
import numpy as np

_MASK = np.uint64(0xFFFFFFFF)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)


def philox4x32_10(ctr, key):
    """ctr uint32 [..., 4], key uint32 [..., 2] (broadcast) -> uint32 [..., 4]."""
    ctr = np.asarray(ctr, dtype=np.uint64)
    key = np.asarray(key, dtype=np.uint64)
    c0, c1, c2, c3 = (ctr[..., i] for i in range(4))
    k0, k1 = key[..., 0], key[..., 1]
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
        p0, p1 = _M0 * c0, _M1 * c2          # < 2^64: exact in uint64
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _MASK
    return np.stack(np.broadcast_arrays(c0, c1, c2, c3), axis=-1).astype(np.uint32)


def uniforms(key64: int, step: int, V: int) -> np.ndarray:
    """u_j, j < V, of one row: counter (step, j // 4, 0, 0), word j % 4, key (low, high 32 bits of key64)."""
    j = np.arange(V, dtype=np.uint64)
    ctr = np.stack([np.full(V, step, np.uint64), j >> np.uint64(2), np.zeros(V, np.uint64), np.zeros(V, np.uint64)], -1)
    key = np.array([key64 & 0xFFFFFFFF, (key64 >> 32) & 0xFFFFFFFF], dtype=np.uint64)
    words = philox4x32_10(ctr, key)[np.arange(V), (j & np.uint64(3)).astype(np.int64)]
    return ((words >> np.uint32(9)).astype(np.float64) + 0.5) * 2.0 ** -23


def gumbel_scores(logits_row, temperature: float, key64: int, step: int) -> np.ndarray:
    """fp64 l_j / T - log(-log u_j) of one row of (exactly representable) logits."""
    logits_row = np.asarray(logits_row, dtype=np.float64)
    u = uniforms(key64, step, logits_row.shape[0])
    return logits_row / temperature - np.log(-np.log(u))

"""Host restatement of generate()'s per-sequence sampling controls (include/mistral_b200.h: mb200_select_tokens), in numpy.

  philox4x32_10  Philox4x32-10 (Salmon et al., SC'11) with the Random123 constants, on uint32 arrays
  uniforms       a seeded sequence's uniform at step t: (x0 >> 8) * 2^-24 of Philox at key (seed mod 2^32, seed >> 32), counter (t, 0, 0, 0)
  penalised      l'[v] = fp32(l[v] - pen[v]), pen[v] = fp32(fp32(c[v]) * frequency), then + presence (one fp32 add) where c[v] > 0
"""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: 4 uint32 arrays (broadcastable), key: 2 uint32 arrays -> the 4 output words as uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint32) for x in ctr]
    k0, k1 = (np.asarray(x, dtype=np.uint32) for x in key)
    with np.errstate(over="ignore"):
        for r in range(10):
            if r:
                k0 = (k0 + W0).astype(np.uint32)
                k1 = (k1 + W1).astype(np.uint32)
            p0 = M0 * c[0].astype(np.uint64)
            p1 = M1 * c[2].astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & _LO).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & _LO).astype(np.uint32)
            c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return c


def uniforms(seed: int, steps) -> np.ndarray:
    """float32 uniforms of the sequence with this uint64 seed at the given steps."""
    steps = np.asarray(steps, dtype=np.uint32)
    z = np.zeros_like(steps)
    x0 = philox4x32_10((steps, z, z, z), (np.uint32(seed & 0xFFFFFFFF), np.uint32(seed >> 32)))[0]
    return ((x0 >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)).astype(np.float32)


def sequence_seeds(random_seed, B: int):
    """generate()'s per-sequence seeds: an int s gives (s + b) mod 2^64, a list is taken as it is."""
    if isinstance(random_seed, (list, tuple)):
        return [int(s) for s in random_seed]
    return [(int(random_seed) + b) % (1 << 64) for b in range(B)]


def penalised(logits: np.ndarray, counts: np.ndarray, presence, frequency) -> np.ndarray:
    """float32 l' of rows [B, V] (or one row [V]) with counts of the same shape and per-row penalties (scalars or [B])."""
    l = np.asarray(logits, dtype=np.float32)
    c = np.asarray(counts)
    f = np.asarray(frequency, dtype=np.float32)
    p = np.asarray(presence, dtype=np.float32)
    if l.ndim == 2:
        f, p = np.broadcast_to(f, l.shape[:1])[:, None], np.broadcast_to(p, l.shape[:1])[:, None]
    pen = (c.astype(np.float32) * f).astype(np.float32)
    pen = np.where(c > 0, (pen + p).astype(np.float32), pen)
    out = (l - pen).astype(np.float32)
    # a row with both penalties 0 reads its logits unchanged (NaN payloads and -0.0 included)
    off = (f == 0) & (p == 0)
    return np.where(np.broadcast_to(off, l.shape), l, out)

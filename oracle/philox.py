"""CPU restatement of the per-sequence counter-based random numbers of csrc/sq_rng.cu (stream layout in
include/sequoia_b200.h, "per-sequence counter-based random numbers"), in vectorised numpy integer arithmetic.

Random123 philox4x32-10: key (seed & 0xffffffff, seed >> 32); element e of stream (seed, purpose, step) is word e % 4 of
the block for counter (i & 0xffffffff, i >> 32, purpose, step), i = e // 4.  Purposes: 0 = r, 1 = rand, 2 = bonus noise.
"""
import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF
R, RAND, NOISE = 0, 1, 2


def philox4x32_10(ctr, key):
    """ctr: 4 uint32 arrays (or ints) of one shape, key: 2 ints -> 4 uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & MASK for x in ctr]
    k0, k1 = int(key[0]) & MASK, int(key[1]) & MASK
    for _ in range(10):
        p0 = c[0] * np.uint64(M0)
        p1 = c[2] * np.uint64(M1)
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & np.uint64(MASK),
             (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1), p0 & np.uint64(MASK)]
        k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return [x.astype(np.uint32) for x in c]


def words(seed: int, purpose: int, step: int, n: int) -> np.ndarray:
    """The first n uint32 words of stream (seed, purpose, step)."""
    i = np.arange((n + 3) // 4, dtype=np.uint64)
    shape = i.shape
    out = philox4x32_10((i & np.uint64(MASK), i >> np.uint64(32), np.full(shape, purpose, np.uint64),
                         np.full(shape, step & MASK, np.uint64)), (seed & MASK, seed >> 32))
    return np.stack(out, axis=1).reshape(-1)[:n]


def uniform_from_words(w: np.ndarray) -> np.ndarray:
    """u = fp16((w >> 21) * 2^-11): the 2048 values k / 2048"""
    return ((w >> 21).astype(np.float32) * np.float32(2.0 ** -11)).astype(np.float16)


def uniforms(seed: int, purpose: int, n: int) -> np.ndarray:
    """r (purpose 0, n = M) or rand (purpose 1, n = S * V, node-major) of one sequence, fp16"""
    return uniform_from_words(words(seed, purpose, 0, n))


def noise_u(w: np.ndarray) -> np.ndarray:
    """u = fp32((w >> 8) + 0.5) * 2^-24 with one round-to-nearest-even, as float64"""
    return (((w >> 8).astype(np.float64) + 0.5) * 2.0 ** -24).astype(np.float32).astype(np.float64)


def noise(seed: int, step: int, V: int):
    """Bonus noise of one sequence at `step`: (fp16(max(-log(u), 2^-24)) with the log in float64, the float64 value
    before the fp16 rounding)."""
    x = np.maximum(-np.log(noise_u(words(seed, NOISE, step, V))), 2.0 ** -24)
    return x.astype(np.float16), x

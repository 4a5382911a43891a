"""Float64 restatement of the learner's target-noise generator (include/r2d2_b200.h r2d2_target_smoothing), in numpy
uint32 arithmetic: key = (seed, rank), counter = (e >> 2, iter_lo, iter_hi, 0); words (x0, x1) serve e % 4 in {0, 1},
(x2, x3) serve {2, 3}; u = (2 (x >> 9) + 1) 2^-24; z = sqrt(-2 ln u_a) {cos, sin}(2 pi u_b);
a' = clip(mu + clip(sigma z, -c, c), -1, 1).

TEST INFRASTRUCTURE, like the rest of oracle/: the product path never imports it."""
import numpy as np

_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: four uint32 arrays (or scalars), key: two.  Returns the four output words as uint32 arrays."""
    c = [np.asarray(x, np.uint64) & _MASK for x in ctr]
    k0, k1 = (np.asarray(x, np.uint64) & _MASK for x in key)
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(_W0)) & _MASK, (k1 + np.uint64(_W1)) & _MASK
        p0 = np.uint64(_M0) * c[0]
        p1 = np.uint64(_M1) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & _MASK
        hi1, lo1 = p1 >> np.uint64(32), p1 & _MASK
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return [x.astype(np.uint32) for x in c]


def unit_open(x):
    return (2.0 * (np.asarray(x, np.uint32) >> np.uint32(9)).astype(np.float64) + 1.0) * 2.0 ** -24


def normal(n, seed, rank, it):
    """z_e for e < n."""
    e = np.arange(n, dtype=np.uint64)
    g = e >> np.uint64(2)
    z = np.zeros_like(g)
    x = philox4x32_10((g, z + np.uint64(it & 0xFFFFFFFF), z + np.uint64(it >> 32), z), (z + np.uint64(seed), z + np.uint64(rank)))
    pair = ((e & np.uint64(3)) >> np.uint64(1)).astype(bool)
    ua = unit_open(np.where(pair, x[2], x[0]))
    ub = unit_open(np.where(pair, x[3], x[1]))
    rad = np.sqrt(-2.0 * np.log(ua))
    odd = (e & np.uint64(1)).astype(bool)
    return rad * np.where(odd, np.sin(2.0 * np.pi * ub), np.cos(2.0 * np.pi * ub))


def smooth(mu, sigma, clip, seed, rank, it):
    mu = np.asarray(mu, np.float64)
    noise = np.clip(sigma * normal(mu.size, seed, rank, it).reshape(mu.shape), -clip, clip)
    return np.clip(mu + noise, -1.0, 1.0)

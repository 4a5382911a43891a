"""Host restatement of observation normalisation (r2d2_b200.obs_norm, include/r2d2_b200.h): float64 moments of a set of
rows, Chan's merge with the library's operation order, the fp32 pair, and the numpy float32 transform."""
import numpy as np


def moments(x):
    """[1 + 2 O] float64 block (count, mean, M2) of the rows of x [n, O], in two passes."""
    x = np.asarray(x, np.float64)
    O = x.shape[1]
    if x.shape[0] == 0:
        return np.zeros(1 + 2 * O)
    m = x.mean(axis=0)
    return np.concatenate([[float(x.shape[0])], m, ((x - m) ** 2).sum(axis=0)])


def merge(a, b):
    """Chan's parallel formula, the library's order of operations; an empty side takes the other's values."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    O = (a.size - 1) // 2
    na, nb = a[0], b[0]
    if nb == 0:
        return a.copy()
    if na == 0:
        out = b.copy()
        out[0] = na + nb
        return out
    n = na + nb
    ma, mb, m2a, m2b = a[1:1 + O], b[1:1 + O], a[1 + O:], b[1 + O:]
    d = mb - ma
    return np.concatenate([[n], ma + (d * nb) / n, (m2a + m2b) + (((d * d) * na) * nb) / n])


def pair(block):
    """(mean_f, inv_std_f) float32 from a block; (0, 1) when it holds no row."""
    block = np.asarray(block, np.float64)
    O = (block.size - 1) // 2
    n = block[0]
    if n == 0:
        return np.zeros(O, np.float32), np.ones(O, np.float32)
    return block[1:1 + O].astype(np.float32), (1.0 / np.sqrt(block[1 + O:] / n + 1e-8)).astype(np.float32)


def normalize(x, mean_f, inv_std_f, clip):
    """x_hat = clamp(fl(fl(x - mean_f) * inv_std_f), -c, c) in float32, NaN passing through."""
    x = np.asarray(x, np.float32)
    c = np.float32(clip)
    with np.errstate(invalid="ignore", over="ignore"):
        v = (x - np.asarray(mean_f, np.float32)) * np.asarray(inv_std_f, np.float32)
        return np.where(v < -c, -c, np.where(v > c, c, v)).astype(np.float32)


def episode_rows(episodes, n_step):
    """The rows the moments cover: every episode's obs without its last n_step (pad) rows, rows with a NaN / inf out."""
    rows = np.concatenate([np.asarray(e[0], np.float32)[:len(e[0]) - n_step] for e in episodes])
    return rows[np.isfinite(rows).all(axis=1)]

"""Float64 oracle of observation normalization (obs_norm): the valid-row sums of a batch in the order
impala_obs_normalize adds them, Chan's merge, the float32 statistics the kernels normalize with, the normalized
rows, and the fold / unfold of a first layer into raw-observation coordinates."""
import numpy as np

TILE_LANES, MAX_CHUNKS = 8, 1024  # impala_obs_normalize: row lanes per CTA, at most 1024 row chunks


def dense_rows(obs, T: int, frames: int = 1) -> np.ndarray:
    """(T+1, B, O) float64 observation rows of a slab's obs: dense (T+1, B, O), or frames (T+k, B, F) stacked
    oldest first."""
    obs = np.asarray(obs)
    if frames == 1:
        return obs.astype(np.float64)
    return np.concatenate([obs[j:j + T + 1] for j in range(frames)], axis=-1).astype(np.float64)


def valid_rows(lens, T: int) -> np.ndarray:
    """(T+1, B) bool: the rows that count, t < lens[b] (the bootstrap row and padding do not)."""
    t = np.arange(T + 1)[:, None]
    return (t < np.minimum(np.asarray(lens)[None, :], T))


def _seq(x, axis: int) -> np.ndarray:
    """Sum along `axis` strictly left to right (numpy's own sum is pairwise)."""
    x = np.moveaxis(x, axis, 0)
    acc = x[0].copy()
    for i in range(1, x.shape[0]):
        acc = acc + x[i]
    return acc


def batch_sums(x, lens, T: int):
    """(sum x (O), sum x^2 (O), rows) over the valid rows of dense rows x (T+1, B, O), added in the kernel's order:
    chunks of a size fixed by the row count, eight row lanes per chunk (lane l: rows l, l + 8, ..), the lanes in
    order, then lane g of the final pass over chunks g, g + 8, .. and those lanes in order."""
    x = np.asarray(x, np.float64)
    R, O = x.shape[0] * x.shape[1], x.shape[2]
    flat = np.where(valid_rows(lens, T).reshape(R, 1), x.reshape(R, O), 0.0)
    n = min(MAX_CHUNKS, max(1, (R + 63) // 64))
    per = -(-(-(-R // n)) // TILE_LANES) * TILE_LANES  # ceil(R / n), rounded up to a multiple of the lanes
    n = -(-R // per)
    out = []
    for v in (flat, flat * flat):
        v = np.concatenate([v, np.zeros((n * per - R, O))]).reshape(n, per // TILE_LANES, TILE_LANES, O)
        part = _seq(_seq(v, 1), 1)                                        # (n, O): lanes, then lanes in order
        part = np.concatenate([part, np.zeros((-(-n // TILE_LANES) * TILE_LANES - n, O))])
        out.append(_seq(_seq(part.reshape(-1, TILE_LANES, O), 0), 0))    # lane g: chunks g, g + 8, ..
    return out[0], out[1], float(valid_rows(lens, T).sum())


def merge(count, mean, var, s1, s2, n_b):
    """Chan's parallel merge of a batch's sums into (count, mean, var), in the kernel's operation order."""
    if not n_b > 0:
        return count, np.array(mean, np.float64), np.array(var, np.float64)
    mean, var = np.asarray(mean, np.float64), np.asarray(var, np.float64)
    n = count + n_b
    mean_b = s1 / n_b
    m2_b = np.maximum(s2 - s1 * mean_b, 0.0)
    d = mean_b - mean
    new_mean = mean + d * (n_b / n)
    m2 = (var * count + m2_b) + (d * d) * ((count * n_b) / n)
    return n, new_mean, m2 / n


def stats_of(x):
    """Population mean and variance of rows x (N, O), the reference the merge must reproduce."""
    x = np.asarray(x, np.float64)
    return float(x.shape[0]), x.mean(0), x.var(0)


def norm_f32(mean, var, eps: float):
    """(mu_f, r_f): float32 mean and 1 / sqrt(var + eps)."""
    return (np.asarray(mean, np.float64).astype(np.float32),
            (1.0 / np.sqrt(np.asarray(var, np.float64) + eps)).astype(np.float32))


def normalize(x, mu_f, r_f) -> np.ndarray:
    """x_n = (x - mu_f) * r_f in float32."""
    return (np.asarray(x, np.float32) - mu_f) * r_f


def fold(W1, b1, mu_f, r_f):
    """First layer in raw-observation coordinates: W1' = W1 diag(r_f), b1' = b1 - W1' mu_f (float64)."""
    W = np.asarray(W1, np.float64) * np.asarray(r_f, np.float64)[None, :]
    return W, np.asarray(b1, np.float64) - W @ np.asarray(mu_f, np.float64)


def unfold(W1f, b1f, mu_f, r_f):
    """The inverse of `fold`: W1 = W1' / r_f, b1 = b1' + W1' mu_f."""
    W = np.asarray(W1f, np.float64)
    return W / np.asarray(r_f, np.float64)[None, :], np.asarray(b1f, np.float64) + W @ np.asarray(mu_f, np.float64)


class Running:
    """The engine's statistics over successive batches (fresh: count 0, mean 0, var 1)."""

    def __init__(self, O: int, eps: float = 1e-8):
        self.count, self.mean, self.var, self.eps = 0.0, np.zeros(O), np.ones(O), eps

    def f32(self):
        return norm_f32(self.mean, self.var, self.eps)

    def update(self, x, lens, T: int):
        s1, s2, n = batch_sums(x, lens, T)
        self.count, self.mean, self.var = merge(self.count, self.mean, self.var, s1, s2, n)


def scaled_obs(seed: int, T: int, B: int, O: int, lens) -> np.ndarray:
    """(T+1, B, O) float32 observations whose features have means up to about 100 and spreads from 1e-2 to 1e2,
    feature 0 constant; rows past the bootstrap row are zero, as in a slab.  The features' means and spreads are the
    same for every seed (the seed draws the values), so successive batches come from one distribution."""
    feat = np.random.default_rng(2718 + O)
    means = feat.uniform(-100.0, 100.0, O)
    spreads = 10.0 ** feat.uniform(-2.0, 2.0, O)
    spreads[0] = 0.0
    x = (means + spreads * np.random.default_rng(seed).standard_normal((T + 1, B, O))).astype(np.float32)
    x[np.arange(T + 1)[:, None] > np.asarray(lens)[None, :]] = 0
    return x

"""numpy restatement of d2b_sample_labels (include/d2b200.h): SplitMix64 keys, the reference's counts (sampling.py:41-47)
and the k smallest-key positives / negatives in ascending key order.  The GPU tests compare the kernel with it bit for bit;
the host tests check its keys against known SplitMix64 outputs and its law against uniformity."""
import numpy as np

STREAM_GAMMA = 0xD1B54A32D192ED03  # image n's stream: mix(seed + (n + 1) * STREAM_GAMMA)
KEY_GAMMA = 0x9E3779B97F4A7C15     # key i: mix(s_n + (i + 1) * KEY_GAMMA), output i + 1 of SplitMix64 seeded with s_n


def mix(z):
    """SplitMix64 finaliser on uint64 arrays (arithmetic mod 2^64)."""
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = z ^ (z >> np.uint64(30))
        z = z * np.uint64(0xBF58476D1CE4E5B9)
        z = z ^ (z >> np.uint64(27))
        z = z * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return z


def image_stream(seed, n):
    """s_n for seed (uint64 array or int) and image n."""
    with np.errstate(over="ignore"):
        return mix(np.asarray(seed, dtype=np.uint64) + np.uint64((n + 1) * STREAM_GAMMA % (1 << 64)))


def keys(s, count: int):
    """[..., count] keys of candidates 0..count-1 for streams s [...]."""
    i = np.arange(1, count + 1, dtype=np.uint64)
    with np.errstate(over="ignore"):
        return mix(np.asarray(s, dtype=np.uint64)[..., None] + i * np.uint64(KEY_GAMMA))


def seed_bits(seed: int) -> int:
    """The uint64 a [1] int64 seed tensor holding `seed` carries."""
    return seed % (1 << 64)


def subsample(labels: np.ndarray, num_samples: int, max_pos: int, bg_label: int, seed: int):
    """labels [N, P] -> (sampled [N, num_samples] int64 with -1 padding, num_pos [N], num_neg [N], rpn_labels [N, P] int8)."""
    labels = np.asarray(labels).astype(np.int64)
    n_img, p = labels.shape
    sampled = np.full((n_img, num_samples), -1, dtype=np.int64)
    rpn = np.full((n_img, p), -1, dtype=np.int8)
    num_pos = np.zeros(n_img, dtype=np.int64)
    num_neg = np.zeros(n_img, dtype=np.int64)
    for n in range(n_img):
        k = keys(image_stream(seed_bits(seed), n), p)
        pos = np.nonzero((labels[n] != -1) & (labels[n] != bg_label))[0]
        neg = np.nonzero(labels[n] == bg_label)[0]
        k_pos = min(len(pos), max_pos)
        k_neg = min(len(neg), num_samples - k_pos)
        fg = pos[np.argsort(k[pos], kind="stable")[:k_pos]]
        bg = neg[np.argsort(k[neg], kind="stable")[:k_neg]]
        sampled[n, :k_pos] = fg
        sampled[n, k_pos:k_pos + k_neg] = bg
        rpn[n, fg] = 1
        rpn[n, bg] = 0
        num_pos[n], num_neg[n] = k_pos, k_neg
    return sampled, num_pos, num_neg, rpn

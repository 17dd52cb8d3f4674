"""CPU checks of the label sampler: the numpy restatement (tests/sampling_ref.py) against known SplitMix64 outputs, the
reference's count rules and a chi-square test of its law (next to the reference's own subsample_labels on the same case),
and the argument checks of d2b_sample_labels, which run before any CUDA call."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch
from scipy import stats

import sampling_ref as sr


def test_keys_match_known_splitmix64_outputs():
    assert [int(k) for k in sr.keys(0, 3)] == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]
    assert [int(k) for k in sr.keys(1234567, 3)] == [6457827717110365317, 3203168211198807973, 9817491932198370423]


def _splitmix64_python(seed: int, count: int):
    out, state = [], seed
    for _ in range(count):
        state = (state + sr.KEY_GAMMA) % (1 << 64)
        z = state
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) % (1 << 64)
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) % (1 << 64)
        out.append(z ^ (z >> 31))
    return out


def test_image_streams_are_plain_splitmix64():
    for seed in (0, 1, 2**63 - 1, 2**64 - 1, 0x123456789ABCDEF):
        for n in (0, 1, 7):
            s = int(sr.image_stream(seed, n))
            z =(seed + (n + 1) * sr.STREAM_GAMMA) % (1 << 64)
            z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) % (1 << 64)
            z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) % (1 << 64)
            assert s == z ^ (z >> 31)
            assert [int(k) for k in sr.keys(s, 5)] == _splitmix64_python(s, 5)


def test_counts_follow_the_reference():
    from detectron2_b200.sampling import max_positive

    assert max_positive(100, 0.29) == int(100 * 0.29) == 28
    assert max_positive(256, 0.5) == 128 and max_positive(512, 0.25) == 128
    rng = np.random.default_rng(0)

    def case(npos, nneg, nign, bg=0, num_samples=100, frac=0.29):
        lab = np.concatenate([np.full(npos, 1 if bg != 1 else 2), np.full(nneg, bg), np.full(nign, -1)])
        lab = rng.permutation(lab)[None]
        sampled, num_pos, num_neg, rpn = sr.subsample(lab, num_samples, max_positive(num_samples, frac), bg, 11)
        k_pos = min(npos, max_positive(num_samples, frac))
        k_neg = min(nneg, num_samples - k_pos)
        assert (int(num_pos[0]), int(num_neg[0])) == (k_pos, k_neg)
        fg, bgs = sampled[0, :k_pos], sampled[0, k_pos:k_pos + k_neg]
        assert (lab[0, fg] != bg).all() and (lab[0, fg] != -1).all() and (lab[0, bgs] == bg).all()
        assert len(set(fg.tolist()) | set(bgs.tolist())) == k_pos + k_neg
        assert (sampled[0, k_pos + k_neg:] == -1).all()
        assert (rpn[0, fg] == 1).all() and (rpn[0, bgs] == 0).all() and int((rpn[0] >= 0).sum()) == k_pos + k_neg
        return k_pos, k_neg

    assert case(50, 200, 30) == (28, 72)  # int(100 * 0.29) == 28 positives
    assert case(0, 300, 5) == (0, 100)    # no positives: all negatives
    assert case(40, 0, 5) == (28, 0)      # no negatives
    assert case(0, 0, 50) == (0, 0)       # all ignored
    assert case(10, 20, 3) == (10, 20)    # fewer candidates than num_samples: -1 padding
    assert case(10, 20, 3, bg=7) == (10, 20)  # bg_label != 0
    assert case(3, 9, 0, num_samples=0) == (0, 0)


def _chi2_pvalue(pairs, n):
    outcomes = list(itertools.permutations(range(n), 2))
    counts = np.array([sum(1 for p in pairs if p == o) for o in outcomes], dtype=np.float64)
    return stats.chisquare(counts).pvalue


SEEDS = 20000


def test_restatement_draws_uniform_ordered_pairs():
    """2 of 5 positives over 20 000 fixed seeds: every ordered pair equally likely (chi-square, p > 1e-4)."""
    seeds = np.arange(SEEDS, dtype=np.uint64)
    k = sr.keys(sr.image_stream(seeds, 0), 5)  # [SEEDS, 5]
    order = np.argsort(k, axis=1, kind="stable")[:, :2]
    pairs = [tuple(int(x) for x in row) for row in order]
    assert _chi2_pvalue(pairs, 5) > 1e-4
    # the same draw through the per-image restatement, for a few seeds
    lab = np.array([[3, 3, 3, 3, 3]])
    for s in range(5):
        sampled = sr.subsample(lab, 2, 2, 0, s)[0]
        assert tuple(sampled[0].tolist()) == pairs[s]


def test_reference_subsample_labels_draws_uniform_ordered_pairs():
    """matching.subsample_labels (the reference's code) on the same case passes the same test."""
    from detectron2_b200.matching import subsample_labels

    labels = torch.full((5,), 3, dtype=torch.int64)
    pairs = []
    for s in range(SEEDS):
        torch.manual_seed(s)
        pos, neg = subsample_labels(labels, 2, 1.0, 0)
        assert neg.numel() == 0
        pairs.append(tuple(pos.tolist()))
    assert _chi2_pvalue(pairs, 5) > 1e-4


def test_sample_labels_rejects_bad_arguments():
    """Every argument is checked before the first CUDA call: these return D2B_EINVAL without a GPU."""
    from detectron2_b200 import _C

    lib = _C.lib()
    EINVAL = -1
    p, q = C.c_void_p(16), C.c_void_p(4096)  # never dereferenced: the checks fail first
    names = ["labels", "kind", "N", "P", "bg", "num_samples", "max_pos", "seed", "out_labels", "sampled", "num_pos",
             "num_neg", "ws", "ws_bytes", "stream"]
    ws = int(lib.d2b_sample_labels_workspace_bytes(2, 1000, 256))
    assert 0 < ws < int(lib.d2b_sample_labels_workspace_bytes(2, 1000, 512))
    assert lib.d2b_sample_labels_workspace_bytes(0, 1000, 256) == 0
    good = [p, _C.LABELS_I8, 2, 1000, 0, 256, 128, p, q, q, q, q, q, ws, None]

    def call(**over):
        a = list(good)
        for k, v in over.items():
            a[names.index(k)] = v
        return lib.d2b_sample_labels(*a)

    bad = [dict(kind=2), dict(kind=-1), dict(N=-1), dict(P=-1), dict(num_samples=-1), dict(max_pos=-1),
           dict(max_pos=257), dict(num_samples=100, max_pos=101), dict(out_labels=None, sampled=None), dict(out_labels=p),
           dict(ws_bytes=ws - 1), dict(ws=None), dict(seed=None), dict(num_pos=None), dict(num_neg=None),
           dict(labels=None), dict(N=65536), dict(num_samples=_C.SAMPLE_MAX_SAMPLES + 1, max_pos=0),
           dict(kind=_C.LABELS_I64, out_labels=p)]
    for over in bad:
        assert call(**over) == EINVAL, over
    assert call(N=0) == 0  # nothing to do: no launch


def test_sample_labels_op_is_cuda_only():
    from detectron2_b200 import sampling

    with pytest.raises(NotImplementedError):
        sampling.subsample_labels_fixed(torch.zeros((2, 10), dtype=torch.int64), 4, 0.5, 0,
                                        seed=torch.zeros((1,), dtype=torch.int64))

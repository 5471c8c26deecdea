"""CPU: the N-best list Viterbi oracle (tests/_nbest_oracle.py) against enumeration of every path, and its rank 0 against
the Viterbi oracle."""
import numpy as np
import pytest

from oracle import crf

import _nbest_oracle as nb


def _case(seed, K, L, integer):
    rng = np.random.default_rng(seed)
    if integer:         # integer-valued inputs: many paths share a score
        x = rng.integers(-2, 3, (1, L, K)).astype(np.float32)
        tr = rng.integers(-2, 3, (K, K)).astype(np.float32)
    else:
        x = rng.standard_normal((1, L, K)).astype(np.float32)
        tr = rng.standard_normal((K, K)).astype(np.float32)
    return x, tr


@pytest.mark.parametrize("K", [1, 2, 3, 5])
@pytest.mark.parametrize("N", [1, 2, 3, 8, 16])
@pytest.mark.parametrize("integer", [False, True])
def test_oracle_against_enumeration(K, N, integer):
    for n in range(1, 7 if K <= 3 else 6):
        for seed in range(3):
            x, tr = _case(1000 * n + seed, K, n, integer)
            tags, scores, counts = nb.nbest(x, tr, [n], N)
            paths, pscores = nb.all_paths(x[0], tr, n)
            c = min(N, K ** n)
            assert counts[0] == c
            assert np.all(scores[0, c:] == -np.inf) and not tags[0, c:].any()
            got = [tuple(p) for p in tags[0, :c, :n]]
            assert len(set(got)) == c                                           # pairwise distinct
            for p, s in zip(tags[0, :c, :n], scores[0, :c]):
                assert nb.path_score(x[0], tr, p) == s                          # bit for bit
            assert sorted(scores[0, :c].tolist()) == sorted(pscores[:c].tolist())
            if not integer:                                                      # no ties: the ordered list itself
                assert got == [tuple(p) for p in paths[:c]]


@pytest.mark.parametrize("K", [1, 2, 3, 5, 10])
def test_rank0_is_viterbi(K):
    rng = np.random.default_rng(K)
    B, L = 12, 9
    x = rng.integers(-2, 3, (B, L, K)).astype(np.float32)
    tr = rng.integers(-2, 3, (K, K)).astype(np.float32)
    lens = rng.integers(1, L + 1, B)
    tags, scores, counts = nb.nbest(x, tr, lens, 4)
    vt, vs = crf.crf_decode(x, tr, lens, dtype=np.float32)
    assert np.array_equal(tags[:, 0], vt)
    assert np.array_equal(scores[:, 0], vs.astype(np.float32))
    assert np.array_equal(counts, np.minimum(4, K ** np.minimum(lens, 6)))


def test_counts_saturate_and_lengths_clamp():
    rng = np.random.default_rng(7)
    x = rng.standard_normal((5, 40, 3)).astype(np.float32)
    tr = rng.standard_normal((3, 3)).astype(np.float32)
    lens = np.array([-3, 0, 1, 2, 40])
    tags, scores, counts = nb.nbest(x, tr, lens, 16)
    assert counts.tolist() == [3, 3, 3, 9, 16]                   # seq_len <= 0 decodes like length 1
    for b, n in enumerate(np.clip(lens, 1, 40)):
        assert not tags[b, :, n:].any()

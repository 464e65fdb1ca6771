"""The fp64 forced-alignment reference (tests/align_reference.py) against path enumeration, its own rescoring, the
uniform-logit closed forms and the loss references.  CPU only."""
import numpy as np
import pytest

import align_reference as ar
import modified_reference as mr
import pruned_reference as pr

TOPOLOGIES = [False, True]


def _factors(rng, T, U, V=6, blank=0, scale=1.0):
    logits = rng.standard_normal((T, U, V)) * scale
    labels = rng.integers(1, V, max(U - 1, 0))
    lpb, lpy = ar.utterance_factors(logits, labels, np.zeros(T, np.int64), T, U, blank)
    return logits, labels, lpb, lpy


@pytest.mark.parametrize("modified", TOPOLOGIES)
@pytest.mark.parametrize("T,U", [(1, 1), (1, 2), (3, 1), (3, 3), (4, 3), (5, 4), (2, 4), (6, 2)])
def test_against_brute_force(modified, T, U):
    rng = np.random.default_rng(T * 10 + U + 100 * modified)
    for _ in range(3):
        _, _, lpb, lpy = _factors(rng, T, U, scale=2.0)
        best, frames = ar.align_factors(lpb, lpy, modified)
        bf, bf_frames, _, _ = ar.brute_force(lpb, lpy, modified)
        if bf_frames is None:
            assert best == -np.inf and (frames == -1).all()
            continue
        assert best == pytest.approx(bf, rel=1e-12, abs=1e-12)
        np.testing.assert_array_equal(frames, bf_frames)   # continuous inputs: the argmax is unique
        assert ar.valid_alignment(frames, T, U, modified)


@pytest.mark.parametrize("modified", TOPOLOGIES)
def test_rescore_of_alignment_is_best(modified):
    rng = np.random.default_rng(7 + modified)
    N, T, U, V = 4, 9, 5, 7
    logits = rng.standard_normal((N, T, U, V))
    labels = rng.integers(1, V, (N, U - 1))
    tl = np.array([9, 7, 5, 9])
    ul = np.array([4, 2, 4, 0])
    scores, frames = ar.align(logits, labels, tl, ul, modified=modified)
    np.testing.assert_allclose(ar.rescore(frames, logits, labels, tl, ul, modified=modified), scores, rtol=1e-13)
    for b in range(N):
        assert ar.valid_alignment(frames[b], tl[b], ul[b] + 1, modified)
        assert (frames[b, ul[b]:] == -1).all()


@pytest.mark.parametrize("modified", TOPOLOGIES)
@pytest.mark.parametrize("T,U,V", [(1, 1, 3), (4, 4, 5), (7, 3, 4), (12, 6, 9)])
def test_uniform_closed_form(modified, T, U, V):
    logits = np.zeros((1, T, U, V))
    labels = np.arange(1, U)[None] % (V - 1) + 1
    scores, frames = ar.align(logits, labels, [T], [U - 1], modified=modified)
    if modified and U - 1 > T:
        assert scores[0] == -np.inf and (frames == -1).all()
        return
    n_factors = T if modified else T + U - 1
    assert scores[0] == pytest.approx(-n_factors * np.log(V), rel=1e-14)
    expect = np.arange(U - 1) if modified else np.zeros(U - 1)
    np.testing.assert_array_equal(frames[0], expect)


@pytest.mark.parametrize("modified", TOPOLOGIES)
def test_best_bounds_the_loss(modified):
    """best <= log P(all paths) = -loss <= best + log(#paths), with the loss references."""
    rng = np.random.default_rng(11 + modified)
    N, T, U, V = 3, 6, 4, 5
    logits = rng.standard_normal((N, T, U, V)) * 1.5
    labels = rng.integers(1, V, (N, U - 1))
    tl = np.array([6, 5, 4])
    ul = np.array([3, 1, 3])
    scores, _ = ar.align(logits, labels, tl, ul, modified=modified)
    if modified:
        costs = mr.dense_loss(logits, labels, tl, ul)[0]
    else:
        costs = pr.pruned_loss(logits, labels, tl, ul, np.zeros((N, T), np.int64))[0]
    for b in range(N):
        n_paths = len(ar.all_alignments(int(tl[b]), int(ul[b]) + 1, modified))
        assert scores[b] <= -costs[b] + 1e-12
        assert -costs[b] <= scores[b] + np.log(n_paths) + 1e-12


def test_pruned_windows_restrict_the_path():
    """The pruned alignment of logits with R = maxU and ranges 0 is the dense one; narrower windows keep the path
    inside them."""
    rng = np.random.default_rng(3)
    N, T, U, V, R = 3, 8, 6, 5, 3
    logits = rng.standard_normal((N, T, U, V))
    labels = rng.integers(1, V, (N, U - 1))
    tl, ul = np.array([8, 6, 8]), np.array([5, 4, 2])
    for modified in TOPOLOGIES:
        dense = ar.align(logits, labels, tl, ul, modified=modified)
        full = ar.align(logits, labels, tl, ul, np.zeros((N, T), np.int64), modified=modified)
        np.testing.assert_array_equal(dense[1], full[1])
        np.testing.assert_array_equal(dense[0], full[0])
    ranges = pr.random_monotone_ranges(rng, tl, ul, T, R)
    pl = np.stack([logits[b][np.arange(T)[:, None], np.clip(ranges[b][:, None] + np.arange(R), 0, U - 1)]
                   for b in range(N)])
    scores, frames = ar.align(pl, labels, tl, ul, ranges)
    for b in range(N):
        T_b, U_b = tl[b], ul[b] + 1
        assert ar.valid_alignment(frames[b], T_b, U_b)
        assert scores[b] <= ar.align(logits[b:b + 1], labels[b:b + 1], tl[b:b + 1], ul[b:b + 1])[0][0] + 1e-12
        # every cell the path visits lies in its frame's window
        f = frames[b, :U_b - 1]
        for t in range(T_b):
            lo, hi = np.searchsorted(f, t, 'left'), np.searchsorted(f, t, 'right')   # cells (t, lo..hi)
            assert ranges[b, t] <= lo and hi <= ranges[b, t] + R - 1


def test_no_path_and_nan():
    rng = np.random.default_rng(5)
    _, _, lpb, lpy = _factors(rng, 3, 5)
    s, f = ar.align_factors(lpb, lpy, modified=True)   # 4 labels, 3 frames
    assert s == -np.inf and (f == -1).all()
    lpb2 = lpb.copy()
    lpb2[2, 0] = np.nan
    for modified in TOPOLOGIES:
        s, f = ar.align_factors(lpb2, lpy, modified)
        assert np.isnan(s) and (f == -1).all()


@pytest.mark.parametrize("modified", TOPOLOGIES)
def test_planted_path_is_the_best(modified):
    rng = np.random.default_rng(21 + modified)
    T, U, V = 10, 5, 8
    for _ in range(4):
        logits = rng.standard_normal((1, T, U, V))
        labels = rng.integers(1, V, (1, U - 1))
        want = ar.random_alignment(rng, T, U, modified)
        ar.plant(rng, logits[0], labels[0], want, T, U, modified=modified)
        _, frames = ar.align(logits, labels, [T], [U - 1], modified=modified)
        np.testing.assert_array_equal(frames[0], want)

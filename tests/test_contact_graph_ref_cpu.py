"""CPU: the vectorised contact-graph rule (tests.parity_helpers.ContactRule), which tests/test_contact_graph_ref_gpu.py
holds contact_kernel to at up to 3000 points, against the loop-and-sort oracle (oracle.inputs.contact_graph) edge for edge,
and its knn-only mode against float64 geometry.  Grid: sizes on both sides of torch.cdist's direct / matrix-product switch
(25 / 26 points), cut-offs giving no, few and all hits (one equal to a distance that occurs, so strict ``<`` is exercised),
K below, at and above the per-centre hit counts, and point sets with exact duplicates (of the centre too) and exact
distance ties (small integer coordinates: both distance forms are exact there)."""
import numpy as np
import pytest

from tests.parity_helpers import ContactRule, contact_paths


def _point_sets(n, seed):
    rng = np.random.default_rng(seed)
    rand = (rng.normal(size=(n, 3)) * 6.0 + 30.0).astype(np.float32)
    dup = rand.copy()
    if n > 2:
        src = rng.choice(n, size=max(1, n // 8), replace=False)
        dst = rng.choice(n, size=len(src), replace=False)
        dup[dst] = rand[src]                    # copies on both sides of their source's index (and some no-ops)
    lattice = rng.integers(0, 4, size=(n, 3)).astype(np.float32)     # exact distances, many ties and duplicates
    return {'random': rand, 'duplicates': dup, 'lattice': lattice}


@pytest.mark.parametrize('n', [1, 2, 25, 26, 300])
def test_rule_matches_oracle(n):
    from oracle.inputs import cdist_f32, contact_graph
    reached, relations = set(), set()
    for kind, pts in _point_sets(n, seed=n).items():
        rule = ContactRule(pts)
        d = cdist_f32(pts)
        off = d[~np.eye(n, dtype=bool)]
        cutoffs = [0.0, float(np.max(d)) + 1.0]
        if off.size:
            cutoffs.append(float(np.sort(off)[off.size // 20]))            # a distance that occurs: strict < decides
        for cutoff in cutoffs:
            _, hits = rule.graph(cutoff, n + 7)
            ks = {1, 2, int(hits.min()), int(np.median(hits)), int(hits.max()), int(hits.max()) + 1, None}
            for k in sorted(ks - {0}, key=lambda v: (v is None, v)):
                ei, hits = rule.graph(cutoff, k)
                want = contact_graph(pts, cutoff, k)
                assert np.array_equal(ei, want), (kind, cutoff, k)
                kk = k or 1000
                reached |= set(contact_paths(hits, k).tolist())
                relations |= {('none' if h == 0 else 'below' if h < kk else 'at' if h == kk else 'above') for h in hits}
    if n >= 25:
        assert relations == {'none', 'below', 'at', 'above'}
        assert {'nearest', 'list_index', 'list_select'} <= reached


def test_rule_breaks_ties_by_index_and_keeps_duplicates_of_the_centre():
    """Hand-checked: centre 0 has two exact copies (indices 3 and 5, d = 0) and two points at distance exactly 2 (1 and 4)."""
    pts = np.array([[0, 0, 0], [2, 0, 0], [9, 9, 9], [0, 0, 0], [0, 2, 0], [0, 0, 0]], np.float32)
    rule = ContactRule(pts)
    ei, hits = rule.graph(2.5, 3)
    assert hits[0] == 4
    assert ei[0][ei[1] == 0].tolist() == [3, 5, 1]               # (d, j) order: the copies, then the lower index of the tie
    assert ei[0][ei[1] == 2].tolist() == [1]                     # no hit: nearest other, |(7, 9, 9)| < |(9, 7, 9)|
    ei, _ = rule.graph(2.5, 4)
    assert ei[0][ei[1] == 0].tolist() == [1, 3, 4, 5]            # hits <= K: index order
    ei, _ = rule.graph(0.0, 4, knn_only=True)
    assert ei[0][ei[1] == 3].tolist() == [0, 5, 1, 4]


@pytest.mark.parametrize('n', [25, 26, 300])
@pytest.mark.parametrize('k', [1, 7, 24])
def test_knn_rule_is_the_exact_k_nearest(n, k):
    """knn_only: the K nearest others by float64 geometry, as a set, on points whose K-th and (K+1)-th nearest float64
    distances are more than 1e-4 apart for every centre - ten times the fp32 rounding of
    these distances, so the set is not decided by a tie."""
    rng = np.random.default_rng(1 if n == 300 else 0)           # seeds checked by the margin assertion below
    pts = (rng.normal(size=(n, 3)) * 8.0).astype(np.float32)
    d64 = np.sqrt(((pts[:, None, :].astype(np.float64) - pts[None, :, :]) ** 2).sum(-1))
    np.fill_diagonal(d64, np.inf)
    srt = np.sort(d64, axis=1)
    assert np.all(srt[:, k] - srt[:, k - 1] > 1e-4), 'near-tie at rank K: pick another seed'
    ei, hits = ContactRule(pts).graph(0.0, k, knn_only=True)
    assert np.all(hits == n - 1) and np.array_equal(ei[1], np.repeat(np.arange(n), k))
    got = np.sort(ei[0].reshape(n, k), axis=1)
    want = np.sort(np.argsort(d64, axis=1)[:, :k], axis=1)
    assert np.array_equal(got, want)
    assert np.all(np.diff(np.take_along_axis(d64, ei[0].reshape(n, k), 1), axis=1) >= 0)      # listed nearest first

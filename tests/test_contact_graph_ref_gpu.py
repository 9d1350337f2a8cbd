"""GPU: contact_kernel (csrc/inputs.cu, behind ddb200_contact_count / _fill and diffdock_b200.inputs.contact_graph) past
its shared-memory hit list, edge for edge and in order against the vectorised rule tests.parity_helpers.ContactRule
(itself checked against oracle.inputs.contact_graph in tests/test_contact_graph_ref_cpu.py).

The kernel keeps at most CAP = 1024 hits per centre in shared memory; beyond that it rescans global memory, on separate
code paths for index-order output, K-nearest selection and knn-only selection.  Each case asserts, from the rule's own hit
counts, that it reaches the path it is about (tests.parity_helpers.contact_paths names them), so a change of inputs cannot
quietly stop covering one.  Cases: a centre with exactly 1023 / 1024 / 1025 hits crossed with K = m - 1, m, m + 1, 1000;
index-order rescans at scale; receptors at C-alpha density with 2999 and 3000 residues (the size limit) through
new_extract_receptor_structure / build_complex at the radius and knn-only settings of the reference's models; knn-only graphs
of 1025 - 1027 and 3000 points; exact fp32 distance ties at rank K and at the nearest-other pick, on the list and rescan
paths; and points one ulp either side of the cut-off at 25 and 26 points, where torch.cdist changes its distance formula.

Every case also checks ddb200_contact_count against the rows the fill writes (the exclusive scan of the counts places the
rows) and that the fill writes nothing past the last row."""
import functools

import numpy as np
import pytest
import torch

from tests.parity_helpers import CONTACT_CAP, ContactRule, contact_paths

pytestmark = pytest.mark.gpu
CA_DENSITY = 0.0085           # C-alpha atoms per cubic angstrom in a folded protein
SENTINEL = -7


def _ball(n, seed, density=CA_DENSITY):
    """n points uniform in a ball of the given density, fp32."""
    rng = np.random.default_rng(seed)
    R = (3.0 * n / (4.0 * np.pi * density)) ** (1.0 / 3.0)
    v = rng.normal(size=(n, 3))
    r = R * rng.uniform(size=(n, 1)) ** (1.0 / 3.0)
    return (v / np.linalg.norm(v, axis=1, keepdims=True) * r + np.array([12.5, -3.0, 40.0])).astype(np.float32)


@functools.lru_cache(maxsize=None)
def _receptor(n):
    pos = _ball(n, seed=n)
    return pos, ContactRule(pos)


def _device(pos, cutoff, k, knn_only=False):
    """(edge_index of inputs.contact_graph, counts of ddb200_contact_count) after checking that a fill into a buffer with
    spare room writes the same rows and nothing past them."""
    from diffdock_b200 import _lib
    from diffdock_b200.inputs import contact_graph
    from diffdock_b200.ops import _ptr, _stream
    p = torch.from_numpy(pos).cuda()
    n, kk = p.shape[0], (k if k else 1000)
    lib = _lib.lib()
    count = torch.empty(n, dtype=torch.int32, device='cuda')
    _lib.check(lib.ddb200_contact_count(_ptr(p), n, float(cutoff), kk, int(knn_only), _ptr(count), _stream()), 'count')
    incl = torch.cumsum(count, 0, dtype=torch.int32)
    E = int(incl[-1])
    nbr = torch.full((E + 64,), SENTINEL, dtype=torch.int32, device='cuda')
    ctr = torch.full((E + 64,), SENTINEL, dtype=torch.int32, device='cuda')
    _lib.check(lib.ddb200_contact_fill(_ptr(p), n, float(cutoff), kk, int(knn_only), _ptr((incl - count).contiguous()),
                                       _ptr(nbr), _ptr(ctr), _stream()), 'fill')
    ei = contact_graph(p, cutoff, k, knn_only=knn_only)
    assert torch.equal(ei, torch.stack([nbr[:E], ctr[:E]]).long()), 'contact_graph and the raw fill disagree'
    assert bool((nbr[E:] == SENTINEL).all()) and bool((ctr[E:] == SENTINEL).all()), 'fill wrote past the last row'
    return ei.cpu().numpy(), count.cpu().numpy()


def _check(got, count, want):
    n = count.shape[0]
    assert np.array_equal(count, np.bincount(want[1], minlength=n)), 'ddb200_contact_count vs the rule'
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = np.flatnonzero((got != want).any(0))
    assert bad.size == 0, f'{bad.size} edges differ, first at {bad[0]}: centre {want[1, bad[0]]}'


def _compare(pos, rule, cutoff, k, knn_only=False):
    """Runs the kernel, checks it against the rule, returns the rule's (hits, per-centre path)."""
    want, hits = rule.graph(cutoff, k, knn_only)
    got, count = _device(pos, cutoff, k, knn_only)
    _check(got, count, want)
    return hits, contact_paths(hits, k, knn_only)


def _rank_k_tie(rule, i, n_out):
    """Whether centre i's n_out-th and (n_out + 1)-th candidates by (distance, index) are at the same fp32 distance, so that
    the index alone decides which one is kept."""
    o = rule.order[i]
    return n_out < o.shape[0] and rule.d[i, o[n_out - 1]] == rule.d[i, o[n_out]]


# ------------------------------------------------------------------------------------------------ the list's capacity
@functools.lru_cache(maxsize=None)
def _designated(m, cutoff=12.0):
    """Centre c with exactly m hits: m points within 0.95 x cut-off of it, 300 more beyond 1.05 x cut-off, in shuffled
    index order."""
    rng = np.random.default_rng(m)
    centre = np.array([[20.25, -7.5, 33.0]])

    def shell(k, r0, r1):
        v = rng.normal(size=(k, 3))
        r = (r0 ** 3 + (r1 ** 3 - r0 ** 3) * rng.uniform(size=(k, 1))) ** (1.0 / 3.0)
        return v / np.linalg.norm(v, axis=1, keepdims=True) * r + centre

    pts = np.concatenate([centre, shell(m, 0.0, 0.95 * cutoff), shell(300, 1.05 * cutoff, 1.6 * cutoff)])
    perm = rng.permutation(len(pts))
    pos = pts[perm].astype(np.float32)
    return pos, ContactRule(pos), int(np.flatnonzero(perm == 0)[0])


@pytest.mark.parametrize('m', [1023, 1024, 1025])
@pytest.mark.parametrize('dk', ['m-1', 'm', 'm+1', 1000])
def test_cap_boundary(built_lib, m, dk):
    pos, rule, c = _designated(m)
    k = {'m-1': m - 1, 'm': m, 'm+1': m + 1}.get(dk, dk)
    hits, paths = _compare(pos, rule, 12.0, k)
    assert hits[c] == m
    want = ('list' if m <= CONTACT_CAP else 'rescan') + ('_index' if m <= k else '_select')
    assert paths[c] == want, (paths[c], want)


def test_index_order_rescan_at_scale(built_lib):
    """K = n and a cut-off covering most of a 1500-point receptor: most centres list more than 1024 hits in index order."""
    pos = _ball(1500, seed=15)
    _, paths = _compare(pos, ContactRule(pos), 50.0, 1500)
    assert np.sum(paths == 'rescan_index') > 750 and np.sum(paths == 'list_index') > 0


# --------------------------------------------------------------------------------------------------- realistic receptors
RECEPTOR_CASES = {
    # name: (receptor graph settings, K the settings imply, paths that must be reached)
    'radius30_defaults': (dict(), 1000, {'list_index'}),                  # build_complex's defaults: 30 A, K = 1000
    'radius34': (dict(receptor_radius=34.0), 1000, {'list_index', 'rescan_select'}),
    'radius15_k24': (dict(receptor_radius=15.0, c_alpha_max_neighbors=24), 24, {'list_select'}),
    'knn24': (dict(knn_only_graph=True, c_alpha_max_neighbors=24), 24, {'knn_rescan'}),
    'knn_default': (dict(knn_only_graph=True), 32, {'knn_rescan'}),        # knn-only default K = 32
}


@pytest.mark.parametrize('case', list(RECEPTOR_CASES))
@pytest.mark.parametrize('n', [3000, 2999])
def test_receptor_graph(built_lib, n, case):
    """C-alpha-density receptors at the size limit (2999: not a multiple of the 4 centres per CTA) through build_complex,
    whose graph settings reach new_extract_receptor_structure and contact_graph."""
    from diffdock_b200.inputs import build_complex
    settings, k, reach = RECEPTOR_CASES[case]
    pos, rule = _receptor(n)
    all_coords = np.stack([pos - 1.0, pos, pos + 1.0], 1)
    g = build_complex('rec', 'A' * n, all_coords, torch.zeros(3, 4), [0, 1], [1, 2], [0, 0],
                      np.array([[0, 0, 0], [1.5, 0, 0], [3, 0, 0]], np.float32), device='cuda:0', **settings)
    knn = settings.get('knn_only_graph', False)
    cutoff = settings.get('receptor_radius', 30.0)
    want, hits = rule.graph(cutoff, k, knn)
    got, count = _device(pos, cutoff, k, knn)
    _check(got, count, want)
    assert np.array_equal(g['receptor', 'receptor'].edge_index.cpu().numpy(), want)
    paths = contact_paths(hits, k, knn)
    assert reach <= set(paths.tolist()), np.unique(paths, return_counts=True)
    if case == 'radius34':
        assert np.sum(paths == 'rescan_select') > 300


@pytest.mark.parametrize('n', [1025, 1026, 1027, 3000])
@pytest.mark.parametrize('dk', [1, 24, 'n-1', 'n+5'])
def test_knn_only_around_cap(built_lib, n, dk):
    """n - 1 = 1024 other points still fit the list; from 1026 points on every selection rescans."""
    pos, rule = _receptor(n)
    k = {'n-1': n - 1, 'n+5': n + 5}.get(dk, dk)
    _, paths = _compare(pos, rule, 0.0, k, knn_only=True)
    assert set(paths.tolist()) == {'knn_list' if n <= CONTACT_CAP + 1 else 'knn_rescan'}


# ------------------------------------------------------------------------------------------------------------ exact ties
@functools.lru_cache(maxsize=None)
def _lattice(L):
    """Integer lattice {0..L-1}^3 (every distance exact in fp32 by either formula, whole shells at equal distance) in
    shuffled order, plus, spread over the index range in shuffled order: 5 copies of q = c + (1, 2, 2), 2 copies of the
    centre c itself, and a far trio a, a + (0, 0, 10), a - (0, 0, 10) whose a has no hit and two nearest others at exactly
    10.  Returns pos, rule, c, the indices of q and its copies, of the copies of c, and of a."""
    rng = np.random.default_rng(L)
    g = rng.permutation(np.stack(np.meshgrid(*[np.arange(L)] * 3, indexing='ij'), -1).reshape(-1, 3))
    mid = L // 2
    c, q, a = np.array([mid] * 3), np.array([mid + 1, mid + 2, mid + 2]), np.array([100, 100, 100])
    extra = np.array([q] * 5 + [c] * 2 + [a, a + [0, 0, 10], a - [0, 0, 10]])[rng.permutation(10)]
    slots = np.linspace(0, len(g), len(extra) + 2)[1:-1].astype(int)
    pos = np.insert(g, slots, extra, axis=0).astype(np.float32)
    rows = lambda p: np.flatnonzero((pos == p).all(1))
    ci = rows(c)
    return pos, ContactRule(pos), int(ci[0]), rows(q), ci[1:], int(rows(a)[0])


@pytest.mark.parametrize('L', [10, 14])
@pytest.mark.parametrize('mode', ['radius', 'knn'])
@pytest.mark.parametrize('at', ['q_copies', 'centre_copies'])
def test_exact_ties(built_lib, L, mode, at):
    """Exact fp32 ties at rank K: K ends inside the group q and its copies (indices on both sides of other points), or inside
    the centre's own copies (d = 0 with j != i).  Such input would trip the reference's ``argsort(...)[1:]`` (its
    ``assert i not in dst``); the kernel's documented rule - ties by index, the centre excluded by index - is what is pinned.
    L = 10 (1010 points) stays on the shared-memory list, L = 14 (2754 points) rescans: the radius graph's centre has more
    than 1024 hits at 6.5, and knn-only selection rescans for more than 1025 points.  The far trio's centre, with no hit,
    takes its nearest other point from a tie at distance 10."""
    pos, rule, c, qi, cdup, a = _lattice(L)
    group = qi if at == 'q_copies' else cdup
    assert np.ptp(group) >= len(group) and np.all(rule.d[c, cdup] == 0)     # other points' indices lie between the copies
    knn = mode == 'knn'
    ranks = np.sort(np.flatnonzero(np.isin(rule.order[c], group)))
    k = int(ranks[len(group) // 2 - 1]) + 1             # keeps the first half of the group by index, drops the rest
    hits, paths = _compare(pos, rule, 6.5, k, knn_only=knn)
    kept = np.isin(group, rule.order[c, :k])
    assert _rank_k_tie(rule, c, k) and kept.any() and not kept.all()
    want = ('knn_' if knn else '') + ('list' if (pos.shape[0] - 1 if knn else hits[c]) <= CONTACT_CAP else 'rescan')
    assert paths[c] == want + ('' if knn else '_select'), (paths[c], want)
    assert want.endswith('list' if L == 10 else 'rescan')
    if not knn:
        assert paths[a] == 'nearest' and _rank_k_tie(rule, a, 1)


# ------------------------------------------------------------------------------------------- distance formula switch
def _pair_d(a, b, mm):
    """fp32 torch.cdist distance of a to each row of b, by the matrix-product (mm) or the direct formula."""
    from oracle.inputs import cdist_f32
    if mm:
        return cdist_f32(np.vstack([a[None], b, np.zeros((max(0, 25 - len(b)), 3), np.float32)]))[0, 1:1 + len(b)]
    return np.array([cdist_f32(np.stack([a, p]))[0, 1] for p in b], np.float32)


def _form_boundary(n, cutoff=np.float32(15.0)):
    """n points: centre 0, the points whose distance to it under torch.cdist's formula for n points is one ulp below, equal
    to and one ulp above the cut-off, one more that the two formulas place on opposite sides of the cut-off, and random
    fill.  Returns pos and the index of that last point."""
    f = np.float32
    mm = n > 25
    c = np.array([0.3, -0.7, 1.1], f)          # near the origin: the matrix form resolves single ulps of d there
    rng = np.random.default_rng(n)
    cand = []
    for ry, rz in (c[1:] + rng.uniform(-4.0, 4.0, size=(64, 2))).astype(f):
        dy, dz = float(c[1]) - float(ry), float(c[2]) - float(rz)
        x = f(c[0] + f(np.sqrt(float(cutoff) ** 2 - dy * dy - dz * dz)))
        for _ in range(24):
            x = np.nextafter(x, f(-np.inf))
        for _ in range(48):
            cand.append([x, ry, rz])
            x = np.nextafter(x, f(np.inf))
    cand = np.asarray(cand, f)
    d_own, d_other = _pair_d(c, cand, mm), _pair_d(c, cand, not mm)
    chosen = []
    for target in (np.nextafter(cutoff, f(0)), cutoff, np.nextafter(cutoff, f(np.inf))):
        hit = np.flatnonzero(d_own == target)
        assert hit.size, f'no point at distance {target!r}'
        chosen.append(cand[hit[0]])
    split = np.flatnonzero((d_own < cutoff) != (d_other < cutoff))
    assert split.size, 'no point on which the two formulas disagree'
    chosen.append(cand[split[0]])
    fill = (c + rng.normal(size=(n - 5, 3)) * 9.0).astype(f)
    pos = np.concatenate([c[None], np.asarray(chosen, f), fill]).astype(f)
    return pos, 4


@pytest.mark.parametrize('n', [25, 26])
def test_distance_formula_switch(built_lib, n):
    """Centre 0 has points one ulp inside, on and one ulp outside the 15 A cut-off under torch.cdist's formula for n points
    (direct up to 25, matrix product from 26), and one point the other formula would place on the other side - so a kernel
    switching formulas at another n lists a different graph."""
    pos, s = _form_boundary(n)
    rule = ContactRule(pos)
    cut = np.float32(15.0)
    assert np.array_equal(rule.d[0, 1:4], [np.nextafter(cut, np.float32(0)), cut, np.nextafter(cut, np.float32(np.inf))])
    _, paths = _compare(pos, rule, 15.0, None)
    assert (rule.d[0, s] < 15.0) != (_pair_d(pos[0], pos[s:s + 1], n <= 25)[0] < 15.0)
    assert paths[0] == 'list_index'

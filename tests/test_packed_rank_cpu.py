"""CPU: the host side of ranking packed complexes - which route ``sample_packed`` ranks by, the ranking pack plan (its own
costs, receptor atoms counted for an all-atom ranker), ``_rank_packed``'s positions, pack order and per-complex split with a
stand-in confidence model, and ``AAOldModel``'s per-batch index maps on packed and shared-receptor all-atom batches (every
sorted edge reads its distinct receptor's attributes; messages summed over the distinct receptors and gathered through the
node maps equal the batch's sums)."""
from argparse import Namespace

import pytest
import torch


def _complexes(all_atoms=True, n_poses=(3, 2, 2, 4), sizes=((20, 12), (24, 20), (20, 9), (16, 7))):
    """Pose lists; complex 2 uses complex 0's receptor (after a different one: interleaved)."""
    from diffdock_b200.synthetic import make_pose_list
    out = [make_pose_list(n, n_res=r, n_atoms=a, seed=3 + k, tr_sigma_max=5.0, lm_dim=0, all_atoms=all_atoms)
           for k, ((r, a), n) in enumerate(zip(sizes, n_poses))]
    for d in out[2]:
        for nt in [k for k in d._nodes if k != 'ligand']:
            d._nodes[nt] = out[0][0]._nodes[nt]
        for et in [k for k in d._edges if 'ligand' not in k]:
            d._edges[et] = out[0][0]._edges[et]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# route and pack plan
def test_rank_route():
    from diffdock_b200.sampling import _rank_route
    cx = _complexes()
    m = object()
    args = Namespace(all_atoms=True, crop_beyond=None)
    assert _rank_route(None, args, cx) is None
    assert _rank_route(m, args, None) == 'score'
    assert _rank_route(m, args, cx) == 'packed'
    assert _rank_route(m, Namespace(all_atoms=True, crop_beyond=20.0), cx) == 'complex'
    assert _rank_route(m, args, [[Namespace()]] + cx[1:]) == 'complex'       # not a HeteroGraph


def test_ranking_pack_cost_counts_receptor_atoms_for_all_atom_rankers():
    from diffdock_b200.sampling import pack_cost, pack_plan
    cx = _complexes()
    for p in cx:
        n_res, n_atom, n_lig = p[0]['receptor'].num_nodes, p[0]['atom'].num_nodes, p[0]['ligand'].num_nodes
        assert pack_cost(p) == len(p) * n_lig * n_res
        assert pack_cost(p, all_atoms=True) == len(p) * n_lig * (n_res + n_atom)
    cg, aa = [pack_cost(p) for p in cx], [pack_cost(p, True) for p in cx]
    budget = sum(cg)
    assert pack_plan(cg, budget) == [[0, 1, 2, 3]]
    plan = pack_plan(aa, budget)
    assert len(plan) > 1 and [k for p in plan for k in p] == [0, 1, 2, 3]     # in order, every complex once
    assert pack_plan([5, 50, 5], 10) == [[0], [1], [2]]                      # larger than the budget: a pack of its own


class _Ranker:
    """Stands in for a confidence model: per graph, the mean ligand x coordinate plus 1000 x its receptor's first residue
    x coordinate (which receptor it was collated with), NaN for graphs whose ligand mean is exactly 12345."""

    def __init__(self, as_tuple=False):
        self.calls, self.as_tuple = [], as_tuple

    def __call__(self, g):
        self.calls.append(g.num_graphs)
        assert g._uniform_t and float(g.complex_t['tr'].abs().max()) == 0.0
        lig, rec = g['ligand'], g['receptor']
        B = g.num_graphs
        s = torch.zeros(B).index_add_(0, lig.batch, lig.pos[:, 0].float())
        n = torch.zeros(B).index_add_(0, lig.batch, torch.ones(lig.batch.shape[0]))
        first = rec.pos[rec.ptr[:-1].long(), 0].float()
        out = s / n + 1000 * first
        out = torch.where(s / n == 12345.0, torch.nan, out)
        return (out, None) if self.as_tuple else out


@pytest.mark.parametrize('as_tuple', [False, True])
def test_rank_packed_copies_positions_and_splits_in_input_order(as_tuple):
    from diffdock_b200.sampling import _rank_packed, pack_cost, pack_plan
    cx = _complexes()
    finals = [torch.cat([d['ligand'].pos + 0.25 * (k + 1) for d in p]).float() for k, p in enumerate(cx)]
    finals[1][:cx[1][0]['ligand'].num_nodes] = 0.0
    finals[1][:cx[1][0]['ligand'].num_nodes, 0] = 12345.0                   # complex 1, pose 0: NaN -> -1000
    args = Namespace(all_atoms=True, crop_beyond=None)
    budget = pack_cost(cx[0], True) + pack_cost(cx[1], True)
    plan = pack_plan([pack_cost(p, True) for p in cx], budget)
    assert len(plan) >= 2
    r = _Ranker(as_tuple)
    before = [[d['ligand'].pos.clone() for d in p] for p in cx]
    out = _rank_packed(r, args, cx, finals, budget, 'cpu')
    assert r.calls == [sum(len(cx[k]) for k in p) for p in plan]            # one forward per ranking pack
    for k, p in enumerate(cx):
        n = p[0]['ligand'].num_nodes
        want = torch.stack([finals[k][i * n:(i + 1) * n, 0].mean() + 1000 * p[0]['receptor'].pos[0, 0] for i in range(len(p))])
        if k == 1:
            want[0] = -1000.0
        assert out[k].shape == (len(p),) and torch.allclose(out[k], want, rtol=1e-5, atol=1e-3), (k, out[k], want)
        for d, b in zip(p, before[k]):                                       # the confidence graphs are not written to
            assert torch.equal(d['ligand'].pos, b)


def test_rank_packed_refuses_ligands_of_another_size():
    from diffdock_b200.sampling import _rank_packed
    cx = _complexes()
    finals = [torch.cat([d['ligand'].pos for d in p]).float() for p in cx]
    finals[2] = finals[2][1:]
    with pytest.raises(ValueError, match='complex 2'):
        _rank_packed(_Ranker(), Namespace(all_atoms=True, crop_beyond=None), cx, finals, 10 ** 9, 'cpu')


def test_sample_packed_no_longer_refuses_missing_confidence_graphs():
    from diffdock_b200.sampling import sample_packed
    from tests.test_packed_aa_cpu import _aa_model
    m, a = _aa_model()
    cx = _complexes()
    with pytest.raises(RuntimeError, match='CUDA device only'):     # past the argument checks
        sample_packed(cx, m, 2, [1.0, 0.5], [1.0, 0.5], [1.0, 0.5], 'cpu', None, a, seed=0, confidence_model=m)
    with pytest.raises(ValueError, match='one list of confidence graphs per complex'):
        sample_packed(cx, m, 2, [1.0, 0.5], [1.0, 0.5], [1.0, 0.5], 'cpu', None, a, seed=0, confidence_model=m,
                      confidence_data=cx[:2])


# ---------------------------------------------------------------------------------------------------------------------
# AAOldModel's index maps
def _cpu_sort(t32, n_rows, want_row_ptr=False):
    t, order = torch.sort(t32.long(), stable=True)
    return t.to(torch.int32), order, None


def _aaold():
    from diffdock_b200.diffusion_utils import get_timestep_embedding
    from diffdock_b200.old_aa_model import AAOldModel
    torch.manual_seed(0)
    return AAOldModel(None, 'cpu', get_timestep_embedding('sinusoidal', 16, 1000), ns=16, nv=4, num_conv_layers=3,
                      sigma_embed_dim=16, distance_embed_dim=16, cross_distance_embed_dim=16, confidence_mode=True,
                      use_old_atom_encoder=True).eval()


def _static(g, monkeypatch):
    from diffdock_b200 import ops
    monkeypatch.setattr(ops, 'csr_sort_by_target', _cpu_sort)
    with torch.no_grad():
        return _aaold()._static(g)


def _batches():
    from diffdock_b200.hetero import collate, collate_packed, collate_shared_receptor
    cx = _complexes()
    return {'packed': collate_packed(cx, 'cpu'), 'shared': collate_shared_receptor(cx[3], 'cpu'),
            'plain': collate([d for p in cx for d in p])}


@pytest.mark.parametrize('kind', ['packed', 'shared', 'plain'])
def test_aaold_static_maps_every_edge_onto_its_distinct_receptor(kind, monkeypatch):
    g = _batches()[kind]
    c = _static(g, monkeypatch)
    if kind == 'plain':                    # no layout: per-edge attributes only, nothing shared
        assert 'perm_u' not in c['ra'] and 'shared' not in c
        return
    for k in ('rr', 'aa', 'ar'):
        d = c[k]
        assert torch.equal(d['vec_u'][d['perm'].long()], d['vec'])
        assert (d['ew_u'] is None) == (d['ew'] is None)      # a weight per edge only with smooth_edges
        if d['ew'] is not None:
            assert torch.equal(d['ew_u'][d['perm'].long()], d['ew'])
    assert torch.equal(c['ra']['perm_u'], c['ar']['perm'][c['ra']['perm'].long()])
    assert 'shared' in c
    # the base embeddings of every copy are its distinct receptor's
    rows_r, rows_a, map_r, map_a, _ = c['shared']
    assert torch.equal(c['rec_base'], c['rec_base'][rows_r][map_r])
    assert torch.equal(c['atom_base'], c['atom_base'][rows_a][map_a])


def _sums(x, tgt, src, vec, perm, n_out):
    """A stand-in convolution: sum over each target's edges of x[src] * |vec| (vec read through perm)."""
    w = vec[perm.long()].norm(dim=-1, keepdim=True)
    return torch.zeros((n_out, x.shape[1])).index_add_(0, tgt.long(), x[src.long()] * w)


@pytest.mark.parametrize('kind', ['packed', 'shared'])
@pytest.mark.parametrize('mutate', [None, 'node_map'])
def test_distinct_receptor_sums_gathered_equal_the_batch_sums(kind, mutate, monkeypatch):
    """What ``_shared_static_messages`` relies on: for the four layer-0 groups, sums over the distinct receptors' edges
    (local numbering [distinct residues | distinct atoms]) gathered through the node maps equal the batch's sums, for
    node features that are the same in every copy.  A wrong node map breaks it."""
    g = _batches()[kind]
    c = _static(g, monkeypatch)
    rows_r, rows_a, map_r, map_a, local = c['shared']
    if mutate == 'node_map':
        map_r = map_r.roll(1)
    nr_u, na_u = rows_r.shape[0], rows_a.shape[0]
    n_lig, n_rec = g['ligand'].num_nodes, g['receptor'].num_nodes
    o_r, o_a, N = n_lig, n_lig + n_rec, n_lig + n_rec + g['atom'].num_nodes
    gen = torch.Generator().manual_seed(0)
    xr_u, xa_u = torch.randn(nr_u, 5, generator=gen), torch.randn(na_u, 5, generator=gen)
    x = torch.cat([torch.randn(n_lig, 5, generator=gen), xr_u[c['shared'][2]], xa_u[c['shared'][3]]])
    x0 = torch.cat([xr_u, xa_u])
    ok = []
    for key, att, lo, hi, part, m in (('rr', 'rr', o_r, o_a, slice(0, nr_u), map_r), ('ra', 'ar', o_r, o_a, slice(0, nr_u), map_r),
                                      ('aa', 'aa', o_a, N, slice(nr_u, None), map_a), ('ar', 'ar', o_a, N, slice(nr_u, None), map_a)):
        d = c[key]
        vec_u = c[att]['vec_u']
        batch = _sums(x, d['tgt'], d['src'], vec_u, d['perm_u'] if key == 'ra' else d['perm'], N)
        t, s, perm = local[key]
        dist = _sums(x0, t, s, vec_u, perm, nr_u + na_u)
        ok.append(torch.allclose(dist[part][m], batch[lo:hi], atol=1e-5))
    assert all(ok) == (mutate is None), ok

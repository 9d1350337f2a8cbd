"""CPU: the v1.0 confidence models at fused-kernel widths - the oracle against the unmodified reference
(tests/golden/ref_confidence_v10_fused.pt), the all-atom shared-receptor collate against the general collate, and the
predicates that choose the sync-free forward."""
import copy

import pytest
import torch

from tests.confidence_v10_fused_helpers import batch_of, build, fixture


@pytest.mark.parametrize('i', range(4))
def test_oracle_matches_reference_fixture(i):
    case = fixture()['cases'][i]
    m, poses = build(case, 'oracle')
    with torch.no_grad():
        conf = m(batch_of(poses, case['times'], 'cpu', all_atoms=case['all_atoms']))
    ref = case['confidence']
    assert conf.shape == ref.shape
    assert float((conf - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max())), (conf, ref)


def test_fixture_covers_the_requested_flags():
    cases = fixture()['cases']
    kw = [c['kw'] for c in cases]
    assert all(k['ns'] == 16 and k['nv'] == 4 for k in kw)
    cg = [c for c in cases if c['cls'] == 'CGOldModel']
    aa = [c for c in cases if c['cls'] == 'AAOldModel']
    for group in (cg, aa):
        assert {c['kw']['num_conv_layers'] for c in group} & {2} and {c['kw']['num_conv_layers'] for c in group} & {3, 4}
        assert {bool(c['lm_dim']) for c in group} == {True, False}
        assert any(c['kw']['dynamic_max_cross'] for c in group) and any(c['kw']['affinity_prediction'] for c in group)
    assert any(c['kw']['smooth_edges'] for c in cg)
    assert fixture()['sampling']['confidence'].shape == (3,)


# ---------------------------------------------------------------------------------------------- shared-receptor collate
def _poses(n=3, seed=4, **kw):
    from diffdock_b200.synthetic import make_pose_list
    return make_pose_list(n, n_res=30, n_atoms=8, seed=seed, tr_sigma_max=2.0, lm_dim=0, all_atoms=True, **kw)


def _public(st):
    return {k: v for k, v in st.__dict__.items() if not k.startswith('_')}


def _assert_same(a, b):
    """Every public attribute of every store and every global, tensor for tensor (values, dtype, shape)."""
    assert sorted(a._nodes) == sorted(b._nodes) and sorted(a._edges) == sorted(b._edges)
    for sa, sb in [(a._nodes[k], b._nodes[k]) for k in a._nodes] + [(a._edges[k], b._edges[k]) for k in a._edges]:
        pa, pb = _public(sa), _public(sb)
        assert sorted(pa) == sorted(pb)
        for k in pa:
            va, vb = pa[k], pb[k]
            if torch.is_tensor(va):
                assert va.dtype == vb.dtype and va.shape == vb.shape and torch.equal(va, vb), k
            elif isinstance(va, list):          # per-graph Python objects (names, torsion masks)
                assert isinstance(vb, list) and len(va) == len(vb), k
            else:
                assert va == vb, k
    assert sorted(a._globals) == sorted(b._globals)


@pytest.mark.parametrize('share', [False, True])
def test_all_atom_shared_collate_equals_general_collate(share):
    """Deep copies (inference.py's N copies of one complex) and poses sharing the receptor storage."""
    from diffdock_b200.hetero import collate, collate_shared_receptor
    poses = _poses(share_receptor=share)
    got = collate_shared_receptor(poses, 'cpu')
    ref = collate(copy.deepcopy(poses))
    _assert_same(got, ref)
    n_res, n_atom = poses[0]['receptor'].num_nodes, poses[0]['atom'].num_nodes
    assert got['receptor']._unique == (n_res, poses[0]['receptor', 'receptor'].num_edges, 3)
    assert got['atom']._unique == (n_atom, poses[0]['atom', 'atom'].num_edges, 3)
    # per-copy offsets of the atom and residue indices
    ar, ar1 = got['atom', 'receptor'].edge_index, poses[0]['atom', 'receptor'].edge_index
    e1 = ar1.shape[1]
    for b in range(3):
        assert torch.equal(ar[:, b * e1:(b + 1) * e1], ar1 + torch.tensor([[b * n_atom], [b * n_res]]))


def test_shared_collate_falls_back_when_receptors_differ():
    from diffdock_b200.hetero import collate, collate_shared_receptor
    poses = _poses()
    poses[2]['atom'].pos = poses[2]['atom'].pos + 0.5               # one complex's atoms differ: a different receptor
    got = collate_shared_receptor(poses, 'cpu')
    _assert_same(got, collate(copy.deepcopy(poses)))
    assert not hasattr(got['receptor'], '_unique') and not hasattr(got['atom'], '_unique')
    other = _poses(seed=5)                                          # a different complex altogether
    got = collate_shared_receptor(poses[:1] + other[:1], 'cpu')
    assert not hasattr(got['atom'], '_unique')


def test_shared_collate_leaves_the_items_untouched():
    from diffdock_b200.hetero import collate_shared_receptor
    poses = _poses()
    before = copy.deepcopy(poses)
    ids = [{k: id(s) for k, s in list(p._nodes.items()) + list(p._edges.items())} for p in poses]
    b = collate_shared_receptor(poses, 'cpu')
    b['receptor'].x.add_(1.0)
    b['atom'].pos.add_(1.0)
    b['ligand'].pos.add_(1.0)
    for p, q, i in zip(poses, before, ids):
        _assert_same(p, q)
        assert i == {k: id(s) for k, s in list(p._nodes.items()) + list(p._edges.items())}


# ---------------------------------------------------------------------------------------------- path predicates
@pytest.mark.parametrize('i', range(4))
def test_fixture_widths_take_the_sync_free_path(i):
    m, _ = build(fixture()['cases'][i], 'product-cpu')
    assert m.sync_free_capable()


def test_narrow_or_disabled_models_keep_the_host_sized_path(monkeypatch):
    from tests.parity_helpers import load_golden
    case = load_golden('ref_confidence_aa.pt')[0]                   # ns=6, nv=3: outside the fused kernel
    from diffdock_b200.old_aa_model import AAOldModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding
    kw = dict(case['kw'], lm_embedding_dim=case['lm_dim']) if case['lm_dim'] else dict(case['kw'])
    assert not AAOldModel(None, 'cpu', get_timestep_embedding('sinusoidal', 8, 1000), **kw).eval().sync_free_capable()
    monkeypatch.setenv('DDB200_SYNC_FREE', '0')
    for i in (0, 2):
        m, _ = build(fixture()['cases'][i], 'product-cpu')
        assert not m.sync_free_capable()


def test_copies_predicate():
    """``_unique`` counts only when it describes this batch: B copies of the nodes and of the edges."""
    from diffdock_b200.hetero import Store
    from diffdock_b200.old_aa_model import _uniq
    st = Store(pos=torch.zeros(12, 3), _unique=(4, 5, 3))
    assert _uniq(st, 3, 15)
    assert not _uniq(st, 2, 15) and not _uniq(st, 3, 14) and not _uniq(Store(pos=torch.zeros(12, 3)), 3, 15)

"""GPU: the v1.0 confidence models (``CGOldModel`` / ``AAOldModel`` in confidence mode, inference.py's default rankers) on
the sync-free forward: the product against the unmodified reference (tests/golden/ref_confidence_v10_fused.pt) on that
path, sync-free against host-sized against the oracle at ns=48 / nv=10, a full-size all-atom pose, no host read after the
per-batch constants, shared layer-0 messages, the sampler's ranking from the shared-receptor batch, zero-edge groups, and
three mutations the comparisons must catch."""
import copy
from argparse import Namespace
from functools import partial

import numpy as np
import pytest
import torch

from tests.confidence_v10_fused_helpers import batch_of, build, fixture, pair
from tests.parity_helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def _close(got, ref, tol=1e-4):
    return got.shape == ref.shape and float((got - ref).abs().max()) <= tol * max(1.0, float(ref.abs().max()))


def _spy(monkeypatch, cls, name):
    """Counts the calls of ``cls.name``."""
    calls = []
    real = getattr(cls, name)

    def wrapped(self, *a, **kw):
        calls.append(1)
        return real(self, *a, **kw)
    monkeypatch.setattr(cls, name, wrapped)
    return calls


def _conf(m, batch):
    with torch.no_grad():
        return m(batch).float().cpu()


def _run_case(m, case, shared=False):
    return _conf(m, batch_of(_poses_of(case), case['times'], DEV, all_atoms=case['all_atoms'], shared=shared))


def _poses_of(case):
    from diffdock_b200.hetero import graph_from_dict
    return [graph_from_dict(d) for d in case['poses']]


def _cls(case):
    from diffdock_b200.old_aa_model import AAOldModel
    from diffdock_b200.old_cg_model import CGOldModel
    return AAOldModel if case['cls'] == 'AAOldModel' else CGOldModel


@pytest.mark.parametrize('i', range(4))
def test_product_matches_reference_fixture_on_the_sync_free_path(built_lib, monkeypatch, i):
    case = fixture()['cases'][i]
    m, _ = build(case, 'product')
    assert m.sync_free_capable()
    calls = _spy(monkeypatch, _cls(case), '_forward_sync_free')
    host = _spy(monkeypatch, _cls(case), '_forward_host_sized')
    conf = _run_case(m, case)
    assert calls and not host
    assert _close(conf, case['confidence']), (conf, case['confidence'])


def _mixed(all_atoms, lm_dim=0):
    from diffdock_b200.synthetic import make_pose_list
    kw = dict(tr_sigma_max=2.0, lm_dim=lm_dim, all_atoms=all_atoms)
    return make_pose_list(2, n_res=60, n_atoms=14, seed=5, **kw) + make_pose_list(2, n_res=45, n_atoms=11, seed=6, **kw)


@pytest.mark.parametrize('cls_name,flags', [('AAOldModel', dict()), ('AAOldModel', dict(smooth_edges=True, num_conv_layers=4)),
                                            ('CGOldModel', dict(affinity_prediction=True))])
def test_sync_free_vs_host_sized_vs_oracle_at_full_widths(built_lib, cls_name, flags):
    """ns=48, nv=10, two complexes of different sizes and one time per pose: no ``_unique``, no shared messages."""
    aa = cls_name == 'AAOldModel'
    o, p = pair(cls_name, 11, lm_embedding_type='esm', lm_embedding_dim=32, **flags)
    poses = _mixed(aa, lm_dim=32)
    times = [0.0, 0.35, 0.8, 0.1]
    ref = _conf(o, batch_of(poses, times, 'cpu', all_atoms=aa))
    assert p.sync_free_capable()
    sf = _conf(p, batch_of(poses, times, DEV, all_atoms=aa))
    p._sync_free = False
    hs = _conf(p, batch_of(poses, times, DEV, all_atoms=aa))
    for got in (sf, hs):
        assert _close(got, ref), (got, ref)
    assert _close(sf, hs, 1e-5)


def test_full_size_all_atom_pose_matches_oracle(built_lib, monkeypatch):
    from diffdock_b200.old_aa_model import AAOldModel
    from diffdock_b200.synthetic import make_pose_list
    o, p = pair('AAOldModel', 21, ns=16, nv=4, num_conv_layers=2, dynamic_max_cross=False, cross_max_distance=80.0,
                lm_embedding_type='esm', lm_embedding_dim=1280)
    poses = make_pose_list(1, n_res=1500, n_atoms=40, seed=9, tr_sigma_max=2.0, all_atoms=True)
    ref = _conf(o, batch_of(poses, [0.0], 'cpu', all_atoms=True))
    calls = _spy(monkeypatch, AAOldModel, '_forward_sync_free')
    got = _conf(p, batch_of(poses, [0.0], DEV, all_atoms=True))
    assert calls and _close(got, ref), (got, ref)


@pytest.mark.parametrize('i,shared', [(1, False), (3, False), (2, True)])
def test_no_host_read_after_the_per_batch_constants(built_lib, i, shared):
    case = fixture()['cases'][i]
    m, poses = build(case, 'product')
    times = [0.0] * len(poses) if shared else case['times']
    b = batch_of(poses, times, DEV, all_atoms=case['all_atoms'], shared=shared)
    with torch.no_grad():
        first = m(b).clone()               # builds the per-batch constants (host reads of the node counts)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            again = m(b)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.equal(first, again)


# ---------------------------------------------------------------------------------------------- shared layer-0 messages
def _one_receptor(n=5, n_res=80, seed=31, lm_dim=32):
    from diffdock_b200.synthetic import make_pose_list
    return make_pose_list(n, n_res=n_res, n_atoms=12, seed=seed, tr_sigma_max=2.0, lm_dim=lm_dim, all_atoms=True)


@pytest.mark.parametrize('cls_name', ['AAOldModel', 'CGOldModel'])
def test_shared_messages_equal_unshared_ones(built_lib, monkeypatch, cls_name):
    from diffdock_b200.old_aa_model import AAOldModel
    o, p = pair(cls_name, 41, lm_embedding_type='esm', lm_embedding_dim=32)
    poses = _one_receptor()
    t = [0.0] * len(poses)
    calls = _spy(monkeypatch, AAOldModel, '_shared_static_messages')
    shared_batch = batch_of(poses, t, DEV, all_atoms=True, shared=True)
    assert shared_batch._uniform_t and shared_batch['atom']._unique[2] == len(poses)
    sh = _conf(p, shared_batch)
    assert bool(calls) == (cls_name == 'AAOldModel')
    plain = _conf(p, batch_of(poses, t, DEV, all_atoms=True))
    ref = _conf(o, batch_of(poses, t, 'cpu', all_atoms=True))
    assert _close(sh, plain, 1e-5) and _close(sh, ref), (sh, plain, ref)


def test_mutation_shared_messages_across_different_times_is_caught(built_lib):
    """Marking a batch of different times ``_uniform_t`` reuses copy 0's layer-0 messages for every pose: the comparison
    against the unshared forward of the shared-messages test fails."""
    o, p = pair('AAOldModel', 41, lm_embedding_type='esm', lm_embedding_dim=32)
    poses = _one_receptor()
    t = [0.0, 0.3, 0.6, 0.9, 0.45]
    wrong = batch_of(poses, t, DEV, all_atoms=True, shared=True)
    wrong._uniform_t = True
    plain = _conf(p, batch_of(poses, t, DEV, all_atoms=True))
    assert not _close(_conf(p, wrong), plain, 1e-5)


# ---------------------------------------------------------------------------------------------- mutations vs the fixture
def _caught(monkeypatch, i, mutate):
    case = fixture()['cases'][i]
    m, _ = build(case, 'product')
    mutate(monkeypatch, m)
    return not _close(_run_case(m, case), case['confidence'])


def test_mutation_negated_vector_on_a_reversed_group_is_caught(built_lib, monkeypatch):
    """atom <- ligand and residue <- ligand with Y(-v), as the coarse-grained score model evaluates its reversed group."""
    from diffdock_b200.old_aa_model import AAOldModel

    def mutate(mp, m):
        real = AAOldModel._cross_graph_sync_free
        mp.setattr(AAOldModel, '_cross_graph_sync_free', lambda self, *a, **kw: real(self, *a, **dict(kw, vec_sign=-1.0)))
    assert _caught(monkeypatch, 2, mutate)


def test_mutation_sigma_left_out_of_the_folded_embedding_is_caught(built_lib, monkeypatch):
    import diffdock_b200.old_aa_model as oa

    def mutate(mp, m):
        real = oa.sigma_map
        mp.setattr(oa, 'sigma_map', lambda enc, S, cols: torch.zeros_like(real(enc, S, cols)))
    assert _caught(monkeypatch, 3, mutate)


# ---------------------------------------------------------------------------------------------- zero-edge groups
def _three_paths(o, p, poses, times):
    ref = _conf(o, batch_of(poses, times, 'cpu', all_atoms=True))
    sf = _conf(p, batch_of(poses, times, DEV, all_atoms=True))
    p._sync_free = False
    hs = _conf(p, batch_of(poses, times, DEV, all_atoms=True))
    p._sync_free = True
    return sf, hs, ref


def test_empty_ligand_atom_group_matches_the_host_sized_path(built_lib):
    """One complex whose ligand is farther than 5 A from every receptor atom: its ligand <- atom and atom <- ligand groups
    are empty, and the convolution contributes zeros before the epilogue (DESIGN section 2), as on the host-sized path."""
    o, p = pair('AAOldModel', 51, ns=16, nv=4, num_conv_layers=3, dynamic_max_cross=False, cross_max_distance=200.0)
    poses = _mixed(True)
    far = poses[1]['ligand']
    far.pos = far.pos + (poses[1]['atom'].pos.max(0).values - far.pos.min(0).values + 8.0)
    d = torch.cdist(far.pos, poses[1]['atom'].pos)
    assert float(d.min()) > 5.0
    sf, hs, ref = _three_paths(o, p, poses, [0.0, 0.2, 0.4, 0.6])
    assert _close(sf, hs, 1e-5) and _close(sf, ref) and torch.isfinite(sf).all()


def test_receptor_without_contact_edges(built_lib):
    o, p = pair('AAOldModel', 52, ns=16, nv=4, num_conv_layers=3)
    poses = _mixed(True)
    for q in poses:
        q['receptor', 'receptor'].edge_index = q['receptor', 'receptor'].edge_index[:, :0]
    sf, hs, _ = _three_paths(o, p, poses, [0.0, 0.2, 0.4, 0.6])
    assert _close(sf, hs, 1e-5) and torch.isfinite(sf).all()


# ---------------------------------------------------------------------------------------------- sampler
def test_sampling_ranks_from_the_shared_batch(built_lib, monkeypatch):
    """sampling() ranks with AAOldModel from the shared-receptor batch: the reference's confidences (fixture), the old
    route's (deep copy, general collate, upload, host-sized forward) within atomics tolerance, the same ranking, and the
    caller's confidence_data_list unchanged (values and store identity)."""
    from diffdock_b200.diffusion_utils import set_time, t_to_sigma
    from diffdock_b200.hetero import collate, graph_from_dict
    from diffdock_b200.old_aa_model import AAOldModel
    from diffdock_b200.sampling import rank_poses, sampling
    from tests.test_confidence_v10_fused_cpu import _assert_same
    from tests.test_confidence_v11_cpu import _score_model
    f = fixture()
    s = f['sampling']
    score, a = _score_model(s['score'], 'product')
    conf_model, _ = build(f['cases'][s['confidence_case']], 'product')
    poses = [graph_from_dict(d) for d in s['poses']]
    conf_poses = [graph_from_dict(d) for d in s['conf_poses']]
    before = copy.deepcopy(conf_poses)
    ids = [{k: id(st) for k, st in list(p._nodes.items()) + list(p._edges.items())} for p in conf_poses]
    calls = _spy(monkeypatch, AAOldModel, '_shared_static_messages')
    torch.manual_seed(s['seed'])
    noise = lambda kind, shape: torch.normal(mean=0, std=1, size=shape)           # the reference's CPU draws
    out, conf = sampling(copy.deepcopy(poses), score, s['steps'], s['schedule'], s['schedule'], s['schedule'], 'cuda:0',
                         partial(t_to_sigma, args=a), a, batch_size=3, no_final_step_noise=True, confidence_model=conf_model,
                         confidence_data_list=conf_poses, confidence_model_args=Namespace(all_atoms=True, crop_beyond=None),
                         noise_fn=noise)
    assert calls                                                   # the shared layer-0 messages ran
    for d, ref in zip(out, s['final_pos']):
        assert rel_err(d['ligand'].pos.cpu(), ref) < 1e-4
    assert _close(conf.cpu(), s['confidence'])
    for p, q, i in zip(conf_poses, before, ids):
        _assert_same(p, q)
        assert i == {k: id(st) for k, st in list(p._nodes.items()) + list(p._edges.items())}
    # the old route on the same final poses
    old = collate(copy.deepcopy(conf_poses))
    old['ligand'].pos = torch.cat([d['ligand'].pos for d in out]).cpu()
    old = old.to(DEV)
    set_time(old, 0, 0, 0, 0, len(out), True, DEV)
    conf_model._sync_free = False
    ref = _conf(conf_model, old)
    assert _close(conf.cpu(), ref, 1e-5), (conf, ref)
    _, ranked, order = rank_poses(out, conf, torch.zeros(3))
    assert list(order) == list(np.argsort(ref.numpy())[::-1]) and (ranked[:-1] >= ranked[1:]).all()

"""GPU: several complexes in one batch - the packed pose-update kernel (ddb200_pose_update_packed) against per-ligand
ddb200_pose_update_dev calls, the score models' forward on a packed batch against each complex's own batch, and
sample_packed against one sampling() call per complex."""
import copy
from functools import partial
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests.parity_helpers import make_model_pair, rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _args(**over):
    from diffdock_b200.synthetic import default_model_args
    kw = dict(ns=16, nv=4, sh_lmax=2, num_conv_layers=3, distance_embed_dim=16, cross_distance_embed_dim=16, sigma_embed_dim=16)
    kw.update(over)
    return default_model_args(**kw)


def _rigid(poses):
    """The ligand of every pose without rotatable bonds."""
    for d in poses:
        lig = d['ligand']
        lig.edge_mask = torch.zeros_like(lig.edge_mask)
        lig.mask_rotate = [np.zeros((0, lig.num_nodes), dtype=bool)]
    return poses


def _complexes(shared=True, n_poses=(3, 2, 4), sizes=((60, 12), (70, 20), (60, 9)), seed=5, rigid=()):
    """Pose lists of len(sizes) complexes; with ``shared`` the first and the last use the same receptor."""
    from diffdock_b200.synthetic import make_pose_list
    out = []
    for k, ((n_res, n_atoms), n) in enumerate(zip(sizes, n_poses)):
        poses = make_pose_list(n, n_res=n_res, n_atoms=n_atoms, seed=seed + k, tr_sigma_max=5.0)
        out.append(_rigid(poses) if k in rigid else poses)
    if shared:
        rec, rr = out[0][0]._nodes['receptor'], out[0][0]._edges[('receptor', 'receptor')]
        for d in out[-1]:
            d._nodes['receptor'], d._edges[('receptor', 'receptor')] = rec, rr
    return out


# ---------------------------------------------------------------------------------------------------------------------
# kernel
def _dev_call(pos, n_poses, bu, bv, mask, tr, rot, tor, table, step, keys, tr_z, rot_z, tor_z):
    from diffdock_b200 import ops
    return ops.pose_update_dev(pos.clone(), n_poses, bu, bv, mask, tr, rot, tor, table, step_dev=step, tr_z=tr_z, rot_z=rot_z,
                               tor_z=tor_z, seed=7, pose_key=keys, use_torsion=tor is not None)


@pytest.mark.parametrize("philox", [True, False])
@pytest.mark.parametrize("step", [0, 3, 5])
def test_packed_kernel_is_bit_identical_to_per_ligand_calls(built_lib, philox, step):
    from diffdock_b200 import ops
    from diffdock_b200.hetero import pose_layout
    cx = _complexes(shared=False, sizes=((40, 14), (40, 31), (40, 9)), rigid=(2,))
    layout, bu, bv, mask, max_atoms = pose_layout(cx)
    assert max_atoms == 31 and layout[-1, 3] == 0                      # the third ligand has no rotatable bond
    gen = torch.Generator().manual_seed(step)
    pos = torch.cat([d['ligand'].pos for p in cx for d in p]).to(DEV)
    B, n_tor = layout.shape[0], int(layout[-1, 4] + layout[-1, 3])
    r = lambda *s: torch.randn(*s, generator=gen).to(DEV)
    tr, rot, tor = r(B, 3), r(B, 3), r(n_tor)
    tr_z, rot_z, tor_z = (r(B, 3), r(B, 3), r(n_tor)) if not philox else (None, None, None)
    table = torch.rand(6, 6, generator=gen).to(DEV)
    step_dev = torch.tensor([step], dtype=torch.int32, device=DEV)
    keys = torch.cat([(k << 32) + torch.arange(len(p)) for k, p in enumerate(cx)]).to(DEV) if philox else None
    err = torch.zeros(1, dtype=torch.int32, device=DEV)
    L = [t.to(DEV) for t in (layout, bu, bv, mask)]
    got = ops.pose_update_packed(pos.clone(), L[0], max_atoms, L[1], L[2], L[3], tr, rot, tor, table, err, step_dev=step_dev,
                                 tr_z=tr_z, rot_z=rot_z, tor_z=tor_z, seed=7, pose_key=keys)
    p0 = 0
    for k, poses in enumerate(cx):
        n_p, lo = len(poses), layout[p0]
        a0, n, b0, nb, t0, m0 = [int(v) for v in lo]
        sl = slice(a0, a0 + n_p * n)
        ps = slice(p0, p0 + n_p)
        ts = slice(t0, t0 + n_p * nb)
        want = _dev_call(pos[sl], n_p, L[1][b0:b0 + nb], L[2][b0:b0 + nb], L[3][m0:m0 + nb * n], tr[ps], rot[ps],
                         tor[ts] if nb else None, table, step_dev, keys[ps] if philox else None,
                         tr_z[ps] if tr_z is not None else None, rot_z[ps] if rot_z is not None else None,
                         tor_z[ts] if tor_z is not None and nb else None)
        assert torch.equal(got[sl], want), k
        p0 += n_p
    assert int(err.item()) == 0


def test_packed_kernel_refuses_a_pose_larger_than_declared(built_lib):
    from diffdock_b200 import ops
    from diffdock_b200.hetero import pose_layout
    cx = _complexes(shared=False, sizes=((40, 14), (40, 31), (40, 9)))
    layout, bu, bv, mask, _ = pose_layout(cx)
    pos = torch.cat([d['ligand'].pos for p in cx for d in p]).to(DEV)
    B, n_tor = layout.shape[0], int(layout[-1, 4] + layout[-1, 3])
    tr, rot, tor = torch.ones(B, 3, device=DEV), torch.ones(B, 3, device=DEV), torch.ones(n_tor, device=DEV)
    table = torch.full((1, 6), 0.1, device=DEV)
    err = torch.zeros(1, dtype=torch.int32, device=DEV)
    out = pos.clone()
    ops.pose_update_packed(out, layout.to(DEV), 20, bu.to(DEV), bv.to(DEV), mask.to(DEV), tr, rot, tor, table, err, out=out)
    big = slice(int(layout[3, 0]), int(layout[5, 0]))                  # the two poses of the 31-atom ligand
    assert int(err.item()) == 1
    assert torch.equal(out[big], pos[big])
    assert not torch.equal(out[:big.start], pos[:big.start]) and not torch.equal(out[big.stop:], pos[big.stop:])
    with pytest.raises(RuntimeError, match='DDB200_EINVAL'):           # no error word
        from diffdock_b200 import _lib
        import ctypes as C
        rc = _lib.lib().ddb200_pose_update_packed(C.c_void_p(out.data_ptr()), B, C.c_void_p(layout.to(DEV).data_ptr()), 20,
                                                  None, None, None, C.c_void_p(tr.data_ptr()), C.c_void_p(rot.data_ptr()),
                                                  None, None, None, None, C.c_void_p(table.data_ptr()), None, 0, None, 0,
                                                  None, C.c_void_p(out.data_ptr()), None)
        _lib.check(rc, 'ddb200_pose_update_packed')


# ---------------------------------------------------------------------------------------------------------------------
# forward
def _old_model(fixed_center_conv):
    from tests.old_score_helpers import model_pair
    _, p, a = model_pair(seed=3, ns=16, nv=4, num_conv_layers=3, sigma_embed_dim=16, distance_embed_dim=16,
                         fixed_center_conv=fixed_center_conv)
    return p, a


def _cg_model(fixed_center_conv, full=False):
    args = _args(fixed_center_conv=fixed_center_conv) if not full else _args(
        ns=48, nv=10, num_conv_layers=4, distance_embed_dim=64, cross_distance_embed_dim=64, sigma_embed_dim=64,
        fixed_center_conv=fixed_center_conv)
    _, p = make_model_pair(args, seed=3)
    return p, args


def _scores(model, g):
    out = model(g)
    torch.cuda.synchronize()
    return [t.clone() for t in out[:3]]


def _packed_vs_alone(model, cx, t=0.4, drop_centre=False):
    from diffdock_b200.diffusion_utils import set_time
    from diffdock_b200.hetero import collate_packed, collate_shared_receptor
    g = collate_packed([[d.clone() for d in p] for p in cx], DEV)
    set_time(g, None, t, t, t, g.num_graphs, False, DEV)
    g._uniform_t = True
    if drop_centre:
        del g._globals['_center_node']
    got = _scores(model, g)
    want = [[], [], []]
    for p in cx:
        gs = collate_shared_receptor([d.clone() for d in p], DEV)
        set_time(gs, None, t, t, t, gs.num_graphs, False, DEV)
        gs._uniform_t = True
        for i, s in enumerate(_scores(model, gs)):
            want[i].append(s)
    return max(rel_err(a, torch.cat(b)) for a, b in zip(got, want))


@pytest.mark.parametrize("which", ['cg16', 'cgL2', 'old'])
@pytest.mark.parametrize("fixed", [False, True])
def test_packed_forward_matches_each_complex_alone(built_lib, which, fixed):
    model = _old_model(fixed)[0] if which == 'old' else _cg_model(fixed, full=which == 'cgL2')[0]
    assert model.sync_free_capable()
    assert _packed_vs_alone(model, _complexes()) < 1e-4


@pytest.mark.parametrize("which", ['cg16', 'old'])
def test_dropping_the_centre_nodes_breaks_the_default_centre_convolution(built_lib, which):
    model = _old_model(False)[0] if which == 'old' else _cg_model(False)[0]
    assert _packed_vs_alone(model, _complexes(), drop_centre=True) > 1e-3


@pytest.mark.parametrize("which", ['cg16', 'old'])
def test_receptor_embedded_once_per_distinct_receptor_and_shared_messages(built_lib, which):
    from diffdock_b200.diffusion_utils import set_time
    from diffdock_b200.hetero import collate_packed
    model = _old_model(False)[0] if which == 'old' else _cg_model(False)[0]
    cx = _complexes()                                  # receptors: A (complexes 0 and 2) and B (complex 1)
    g = collate_packed(cx, DEV)
    assert [b[2:] for b in g['receptor']._blocks] == [(3, 0), (2, 1), (4, 0)]
    rows = []
    orig = model.rec_node_embedding.forward
    model.rec_node_embedding.forward = lambda x: (rows.append(x.shape[0]), orig(x))[1]
    try:
        set_time(g, None, 0.5, 0.5, 0.5, g.num_graphs, False, DEV)
        shared = _scores(model, (setattr(g, '_uniform_t', True), g)[1])
    finally:
        del model.rec_node_embedding.forward
    assert rows == [60 + 70]                           # one embedding call over the two distinct receptors
    g2 = collate_packed(cx, DEV)
    set_time(g2, None, 0.5, 0.5, 0.5, g2.num_graphs, False, DEV)   # no uniform-time promise: every copy computed
    unshared = _scores(model, g2)
    for a, b in zip(shared, unshared):
        assert rel_err(a, b) < 1e-5


# ---------------------------------------------------------------------------------------------------------------------
# sampler
def _run_both(model, args, cx, steps=6, **kw):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sample_packed, sampling
    sched = get_t_schedule('expbeta', steps)
    t2s = partial(t_to_sigma, args=args)
    conf_kw = kw.pop('confidence', {})
    max_pairs = kw.pop('max_pairs', None)
    packed = sample_packed([[d.clone() for d in p] for p in cx], model, steps, sched, sched, sched, DEV, t2s, args, seed=11,
                           complex_ids=[5, 9, 2][:len(cx)], no_final_step_noise=True, max_pairs=max_pairs, **conf_kw, **kw)
    alone = []
    for k, (cid, p) in enumerate(zip([5, 9, 2], cx)):
        ck = {}
        if conf_kw:
            ck = dict(confidence_model=conf_kw['confidence_model'], confidence_data_list=conf_kw['confidence_data'][k],
                      confidence_model_args=conf_kw['confidence_model_args'])
        alone.append(sampling([d.clone() for d in p], model, steps, sched, sched, sched, DEV, t2s, args, batch_size=len(p),
                              no_final_step_noise=True, rng='philox', seed=11,
                              pose_keys=(cid << 32) + torch.arange(len(p)), **ck, **kw))
    torch.cuda.synchronize()
    d = 0.0
    for (pl, pc), (al, ac) in zip(packed, alone):
        a = torch.stack([x['ligand'].pos for x in pl]).cpu()
        b = torch.stack([x['ligand'].pos for x in al]).cpu()
        assert torch.isfinite(a).all()
        d = max(d, float((a - b).abs().max()))
        if ac is not None:
            assert rel_err(pc, ac) < 1e-4
    return d


@pytest.mark.parametrize("cuda_graph", [True, False])
def test_sample_packed_matches_sampling_per_complex(built_lib, cuda_graph):
    model, args = _cg_model(False)
    assert _run_both(model, args, _complexes(shared=False, rigid=(1,)), cuda_graph=cuda_graph) < 2e-3


def test_sample_packed_shared_receptor_and_crop(built_lib):
    model, args = _cg_model(False)
    args.crop_beyond = 20.0
    assert model.sync_free_crop_capable()
    assert _run_both(model, args, _complexes(shared=True), cuda_graph=True) < 2e-3


def test_sample_packed_old_score_model_and_packing_budget(built_lib):
    model, a = _old_model(False)
    cx = _complexes(shared=True)
    # a budget below the second complex: three packs of one complex each
    assert _run_both(model, a, cx, max_pairs=2 * 70 * 20 - 1) < 2e-3


def test_sample_packed_ranks_with_a_v10_confidence_model(built_lib):
    from diffdock_b200.diffusion_utils import get_timestep_embedding
    from diffdock_b200.old_cg_model import CGOldModel
    model, args = _cg_model(False)
    torch.manual_seed(4)
    conf = CGOldModel(None, torch.device(DEV), get_timestep_embedding('sinusoidal', 16, args.embedding_scale), ns=16, nv=4,
                      num_conv_layers=2, sigma_embed_dim=16, distance_embed_dim=16, cross_distance_embed_dim=16,
                      confidence_mode=True, use_old_atom_encoder=True, lm_embedding_type='esm', lm_embedding_dim=1280,
                      dynamic_max_cross=True, cross_max_distance=80.0).eval().to(DEV)
    cx = _complexes(shared=True)
    kw = dict(confidence_model=conf, confidence_data=[[d.clone() for d in p] for p in cx],
              confidence_model_args=SimpleNamespace(crop_beyond=None, all_atoms=False))
    assert _run_both(model, args, cx, confidence=kw) < 2e-3


def test_sample_packed_refusals(built_lib):
    from diffdock_b200.sampling import sample_packed
    model, args = _cg_model(False)
    for bad in (dict(noise_fn=lambda k, s: torch.zeros(s)), dict(visualization_list=[]), dict(t_schedule=[0.5])):
        with pytest.raises(NotImplementedError):
            sample_packed(_complexes(), model, 2, [1.0, 0.5], [1.0, 0.5], [1.0, 0.5], DEV, None, args, seed=0, **bad)
    aa = copy.copy(args)
    aa.all_atoms = True
    with pytest.raises(NotImplementedError):
        sample_packed(_complexes(), model, 2, [1.0, 0.5], [1.0, 0.5], [1.0, 0.5], DEV, None, aa, seed=0)


def test_packed_graphed_step_is_sync_free(built_lib):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.hetero import collate_packed
    from diffdock_b200.sampling import GraphedSteps, _step_tables
    model, args = _cg_model(False)
    cx = _complexes()
    g = collate_packed(cx, DEV)
    g._pose_err = torch.zeros(1, dtype=torch.int32, device=DEV)
    sched = get_t_schedule('expbeta', 6)
    coef, t_rows = _step_tables(6, sched, sched, sched, partial(t_to_sigma, args=args), args, False, False, True, 1.0, 0.0,
                                0.5)
    keys = torch.arange(g.num_graphs, device=DEV)
    steps = GraphedSteps(model, g, g.num_graphs, coef, t_rows, None, None, None, True, DEV, draw_noise=True,
                         philox=(3, keys), packed=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        steps.run(6)
        done = steps.step.clone()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert int(done.item()) == 6 and torch.isfinite(steps.pos).all() and int(g._pose_err.item()) == 0

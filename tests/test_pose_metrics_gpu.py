"""GPU: ddb200_pose_metrics (csrc/metrics.cu through diffdock_b200.evaluation) against the float64 oracle (oracle/metrics.py)
and against tests/golden/ref_pose_metrics.pt (spyrmsd's symmrmsd and evaluate.py's expressions): every fixture molecule, the
packed launch against per-complex launches bit for bit, repeat calls bit for bit, edge cases, the absence of host
synchronisation, and the final poses of a real ``sample_packed`` call."""
from functools import partial

import numpy as np
import pytest
import torch

from oracle.metrics import pose_metrics as oracle_metrics
from tests.test_pose_metrics_cpu import CASES

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TOL = 1e-9           # Angstrom; the sums are float64, the oracle's order differs
KEYS = ('rmsd', 'rmsd_min', 'centroid_distance', 'min_self_distance')


def _inputs(name):
    c = CASES[name]
    return (c['poses'].to(torch.float32).to(DEV), c['refs'].to(DEV), c['automorphisms'].to(torch.int32).to(DEV))


def _host(m):
    return {k: getattr(m, k).cpu().numpy() for k in KEYS + ('best_automorphism',)}


def _check(got, poses, refs, aut, want=None):
    """got (host dict) against the oracle on the same float32 poses; best_automorphism attains rmsd_min."""
    ref = oracle_metrics(poses, refs, aut)
    for k in KEYS:
        fin = np.isfinite(ref[k])
        assert np.array_equal(fin, np.isfinite(got[k])), k
        assert np.abs(got[k][fin] - ref[k][fin]).max(initial=0) <= TOL, (k, np.abs(got[k][fin] - ref[k][fin]).max())
        if want is not None:
            assert np.abs(got[k][fin] - want[k][fin]).max(initial=0) <= TOL, k
    n = poses.shape[1]
    for p, a in enumerate(got['best_automorphism']):
        assert 0 <= a < aut.shape[0]
        s = min(np.sum((refs[g] - poses[p][aut[a]]) ** 2) for g in range(refs.shape[0]))
        assert abs(np.sqrt(s / n) - ref['rmsd_min'][p]) <= TOL


@pytest.mark.parametrize('name', sorted(CASES))
def test_kernel_matches_oracle_and_fixture(built_lib, name):
    from diffdock_b200.evaluation import pose_metrics
    c = CASES[name]
    got = _host(pose_metrics(*_inputs(name)))
    assert got['rmsd'].shape == tuple(c['rmsd'].shape)
    want = {k: c[k].numpy() for k in KEYS}
    _check(got, c['poses'].numpy(), c['refs'].numpy(), c['automorphisms'].numpy().astype(np.int64), want)


def test_packed_launch_equals_per_complex_launches_and_repeats(built_lib):
    from diffdock_b200.evaluation import pose_metrics, pose_metrics_packed
    names = sorted(CASES)
    ins = [_inputs(k) for k in names]
    packed = pose_metrics_packed([i[0] for i in ins], [i[1] for i in ins], [i[2] for i in ins])
    again = pose_metrics_packed([i[0] for i in ins], [i[1] for i in ins], [i[2] for i in ins])
    for k, i, a, b in zip(names, ins, packed, again):
        alone = pose_metrics(*i)
        for f in alone._fields:
            assert torch.equal(getattr(a, f), getattr(alone, f)), (k, f)
            assert torch.equal(getattr(a, f), getattr(b, f)), (k, f)


def test_edge_cases(built_lib):
    from diffdock_b200.evaluation import ligand_automorphisms, pose_metrics
    # one heavy atom, one pose, one crystal pose, M = 1
    one = pose_metrics(*_inputs('single_atom'))
    assert one.rmsd.shape == (1, 1) and torch.isinf(one.min_self_distance).all() and one.best_automorphism.tolist() == [0]
    # M = 1 on a chain with a single pose: the plain RMSD
    c = CASES['chain']
    poses, refs = c['poses'][:1], c['refs']
    table, corrected = ligand_automorphisms(c['atomic_nums'], c['bonds'])
    assert corrected and table.shape[0] == 1
    m = pose_metrics(poses.float().to(DEV), refs.to(DEV), table.to(DEV))
    plain = np.sqrt(((poses.numpy() - refs.numpy()[0]) ** 2).sum(-1).mean(-1))
    assert abs(m.rmsd_min.item() - plain[0]) <= TOL
    # a capped table (identity only) on a symmetric molecule gives evaluate.py's uncorrected RMSD
    c = CASES['benzene']
    capped, corrected = ligand_automorphisms(c['atomic_nums'], c['bonds'], max_count=2)
    assert not corrected
    m = pose_metrics(c['poses'].float().to(DEV), c['refs'].to(DEV), capped)            # host table: uploaded
    plain = np.sqrt(((c['poses'].numpy() - c['refs'].numpy()[0]) ** 2).sum(-1).mean(-1))
    assert np.abs(m.rmsd_min.cpu().numpy() - plain).max() <= TOL
    # float32 crystal poses are widened; a NaN pose scores +inf RMSD (spyrmsd's loop keeps +inf) and NaN distances
    poses = c['poses'].float().clone()
    poses[1, 2, 0] = float('nan')
    m = pose_metrics(poses.to(DEV), c['refs'].float().to(DEV), c['automorphisms'].int().to(DEV))
    assert torch.isinf(m.rmsd_min[1]) and m.best_automorphism[1].item() == -1
    assert torch.isnan(m.centroid_distance[1]) and torch.isnan(m.min_self_distance[1])
    assert torch.isfinite(m.rmsd_min[[0, 2, 3, 4]]).all()


def test_no_host_synchronisation_after_the_table_upload(built_lib):
    from diffdock_b200.evaluation import pose_metrics, pose_metrics_packed
    names = sorted(CASES)
    ins = [_inputs(k) for k in names]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        one = pose_metrics(*ins[0])
        packed = pose_metrics_packed([i[0] for i in ins], [i[1] for i in ins], [i[2] for i in ins])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.equal(one.rmsd, packed[0].rmsd)


def test_scores_sample_packed_output(built_lib):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.evaluation import heavy_poses, ligand_automorphisms, ligand_inputs, pose_metrics_packed
    from diffdock_b200.sampling import sample_packed
    from tests.test_packed_gpu import _cg_model, _complexes
    model, args = _cg_model(False)
    cx = _complexes(shared=False)
    inputs, refs, tables = [], [], []
    for poses in cx:
        heavy, z, bonds = ligand_inputs(poses[0])
        assert heavy.numel() >= 1
        inputs.append(heavy)
        refs.append(torch.stack([d['ligand'].pos[heavy] for d in poses[:2]]).double())    # two "crystal" poses
        tables.append(ligand_automorphisms(z, bonds)[0])
    steps = 4
    sched = get_t_schedule('expbeta', steps)
    out = sample_packed(cx, model, steps, sched, sched, sched, DEV, partial(t_to_sigma, args=args), args, seed=3,
                        no_final_step_noise=True)
    poses = [heavy_poses(dl, h) for (dl, _), h in zip(out, inputs)]
    got = pose_metrics_packed(poses, refs, tables)
    for m, p, r, t in zip(got, poses, refs, tables):
        _check(_host(m), p.cpu().numpy(), r.numpy(), t.numpy().astype(np.int64))

"""GPU: the v1.0 score model (diffdock_b200.old_cg_model.CGOldModel, confidence_mode=False) against the unmodified reference
(tests/golden/ref_old_score_model.pt, ref_sampling_old_score.pt) and the CPU oracle, its sync-free forward, the captured
sampler step, and checks that the comparisons catch the three wiring traps of the v1.0 architecture."""
import copy
from functools import partial

import pytest
import torch

from tests.old_score_helpers import fixture_case, fixture_model, fixture_state, model_pair, score, set_times
from tests.parity_helpers import load_golden, golden_confidence_model, rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def _errs(got, ref):
    return [rel_err(a, b) for a, b in zip(got, ref) if b.numel()]


def _fixture_err(i):
    case = fixture_case(i)
    m, poses = fixture_model(case, 'product')
    got = score(m, poses, case['times'], DEV)
    assert [g.shape for g in got] == [case[k].shape for k in ('tr', 'rot', 'tor')]
    return max(_errs(got, (case['tr'], case['rot'], case['tor']))), m


@pytest.mark.parametrize('i', range(5))
def test_product_matches_reference_fixture(built_lib, i):
    err, m = _fixture_err(i)
    assert err < 1e-4, err
    # case 4 has fused-kernel widths: it runs the sync-free forward, the others the host-sized one
    assert m.sync_free_capable() == (i == 4)


def test_reference_keyed_state_dict_loads_strictly(built_lib):
    case = fixture_case(4)
    state = fixture_state(case)
    assert any(k.startswith('final_tp_tor.') for k in state) and any('.tp.' in k for k in state)
    m, _ = fixture_model(case, 'product')          # load_state_dict(strict=True) inside
    assert isinstance(m.load_state_dict(state, strict=True), tuple)


def _mid_poses(seed=77, n=4, n_res=120, n_atoms=24):
    from diffdock_b200.synthetic import make_pose_list
    return make_pose_list(n, n_res=n_res, n_atoms=n_atoms, seed=seed, tr_sigma_max=2.0)


@pytest.fixture(scope='module')
def cfg_l2_pair(built_lib):
    return model_pair(seed=3)


def test_cfg_l2_widths_match_oracle(cfg_l2_pair):
    o, p, _ = cfg_l2_pair
    assert p.sync_free_capable()
    poses = _mid_poses()
    ref = score(o, poses, [0.6] * 4, 'cpu')
    assert max(_errs(score(p, poses, [0.6] * 4, DEV, shared=True), ref)) < 1e-4
    assert max(_errs(score(p, poses, [0.6] * 4, DEV), ref)) < 1e-4


@pytest.mark.parametrize('kind', ['per_graph_times', 'different_complexes'])
def test_sync_free_and_host_sized_match_oracle(cfg_l2_pair, monkeypatch, kind):
    """No shared-receptor shortcut applies: different times per graph (sigma enters the receptor embeddings per complex),
    or a batch of different complexes."""
    o, p, _ = cfg_l2_pair
    if kind == 'per_graph_times':
        poses, times = _mid_poses(seed=78), [0.15, 0.5, 0.8, 0.95]
    else:
        poses = _mid_poses(seed=79, n=1) + _mid_poses(seed=80, n=1, n_res=90, n_atoms=17) + _mid_poses(seed=81, n=1, n_res=140)
        times = [0.4, 0.4, 0.4]
    ref = score(o, poses, times, 'cpu')
    shared = kind == 'per_graph_times'        # the sampler's collate; _uniform_t must not be trusted with mixed times
    sync_free = score(p, poses, times, DEV, shared=False)
    monkeypatch.setattr(p, '_sync_free', False)
    host = score(p, poses, times, DEV)
    assert max(_errs(sync_free, ref)) < 1e-4 and max(_errs(host, ref)) < 1e-4
    if shared:
        from diffdock_b200.hetero import collate_shared_receptor
        b = collate_shared_receptor(copy.deepcopy(poses), DEV)
        set_times(b, times, DEV)           # no _uniform_t: per-graph times
        monkeypatch.setattr(p, '_sync_free', True)
        with torch.no_grad():
            got = [t.cpu() for t in p(b)]
        assert max(_errs(got, ref)) < 1e-4


def test_one_full_size_pose_matches_oracle(cfg_l2_pair):
    """The benchmarked size: one pose of the 1500-residue / 40-atom complex, full 1280-wide LM embedding."""
    from diffdock_b200.synthetic import make_pose_list
    o, p, _ = cfg_l2_pair
    poses = make_pose_list(1, n_res=1500, n_atoms=40, seed=100, tr_sigma_max=19.0)
    got = score(p, poses, [0.5], DEV)
    torch.set_num_threads(min(torch.get_num_threads(), 32))
    ref = score(o, poses, [0.5], 'cpu')
    assert max(_errs(got, ref)) < 1e-4, _errs(got, ref)


def test_equivariance(cfg_l2_pair):
    """Rotating and translating the whole complex rotates tr and rot and leaves tor unchanged."""
    from scipy.spatial.transform import Rotation
    _, p, _ = cfg_l2_pair
    poses = _mid_poses(seed=82, n=2)
    R = torch.tensor(Rotation.random(random_state=5).as_matrix(), dtype=torch.float32)
    moved = copy.deepcopy(poses)
    for g in moved:
        for nt in ('ligand', 'receptor'):
            g[nt].pos = g[nt].pos @ R.T + torch.tensor([3.0, -1.0, 2.0])
    a = score(p, poses, [0.5, 0.7], DEV)
    b = score(p, moved, [0.5, 0.7], DEV)
    assert rel_err(b[0], a[0] @ R.T) < 1e-4 and rel_err(b[1], a[1] @ R.T) < 1e-4 and rel_err(b[2], a[2]) < 1e-4


def test_sync_free_forward_has_no_host_sync(cfg_l2_pair):
    from diffdock_b200.hetero import collate_shared_receptor
    _, p, _ = cfg_l2_pair
    b = collate_shared_receptor(_mid_poses(seed=83), DEV)
    set_times(b, [0.5] * 4, DEV)
    b._uniform_t = True
    with torch.no_grad():
        p(b)                                   # per-batch constants (one host read) and lazy plans
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = p(b)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert all(torch.isfinite(t).all() for t in out)


def test_sampling_matches_reference_fixture(built_lib):
    """sampling() with the v1.0 score model and the v1.0 confidence model vs utils/sampling.py run unmodified, replaying
    the reference's CPU noise draws."""
    from argparse import Namespace
    from diffdock_b200.diffusion_utils import t_to_sigma
    from diffdock_b200.sampling import sampling
    s = load_golden('ref_sampling_old_score.pt')
    case = fixture_case(s['score_case'])
    score_m, poses = fixture_model(case, 'product')
    a = Namespace(**case['args'])
    conf_m, _ = golden_confidence_model(load_golden('ref_confidence.pt')[s['confidence_case']], 'product')
    torch.manual_seed(s['seed'])
    noise = lambda kind, shape: torch.normal(mean=0, std=1, size=shape)
    sched = s['schedule']
    out, conf = sampling(copy.deepcopy(poses), score_m, len(sched), sched, sched, sched, 'cuda:0', partial(t_to_sigma, args=a),
                         a, batch_size=3, no_final_step_noise=True, confidence_model=conf_m,
                         confidence_data_list=copy.deepcopy(poses),
                         confidence_model_args=Namespace(all_atoms=False, crop_beyond=None), noise_fn=noise)
    for d, ref in zip(out, s['final_pos']):
        assert rel_err(d['ligand'].pos, ref) < 1e-4
    assert (conf.cpu() - s['confidence']).abs().max() < 1e-4, (conf, s['confidence'])


def test_graphed_sampler_matches_eager(cfg_l2_pair):
    """sampling() captures the v1.0 step by default; with counter-based noise the captured and the op-by-op runs draw the
    same numbers, so their final poses agree.  The v1.0 confidence model ranks them."""
    from argparse import Namespace
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import _use_cuda_graph, sampling
    _, p, a = cfg_l2_pair
    conf_m, _ = golden_confidence_model(load_golden('ref_confidence.pt')[2], 'product')     # no LM embedding
    assert _use_cuda_graph(p, a, None, None, 4, 4, None)
    poses = _mid_poses(seed=84)
    for g in poses:
        g['receptor'].x = g['receptor'].x[:, :1]        # the ranking model reads residue types only
    poses_lm = _mid_poses(seed=84)
    sched = get_t_schedule('expbeta', 5)
    runs = {}
    for graphed in (True, False):
        out, conf = sampling(copy.deepcopy(poses_lm), p, 5, sched, sched, sched, 'cuda:0', partial(t_to_sigma, args=a), a,
                             batch_size=4, no_final_step_noise=True, rng='philox', seed=11, cuda_graph=graphed,
                             confidence_model=conf_m, confidence_data_list=copy.deepcopy(poses),
                             confidence_model_args=Namespace(all_atoms=False, crop_beyond=None))
        runs[graphed] = (torch.stack([d['ligand'].pos.cpu() for d in out]), conf.cpu())
    assert rel_err(runs[True][0], runs[False][0]) < 1e-4
    assert torch.isfinite(runs[True][1]).all() and (runs[True][1] - runs[False][1]).abs().max() < 1e-3


def test_crop_beyond_runs_eager(cfg_l2_pair):
    from argparse import Namespace
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import _use_cuda_graph, sampling
    _, p, a = cfg_l2_pair
    args = Namespace(**dict(vars(a), crop_beyond=60.0))       # keeps residues around the drifting ligand of random weights
    assert not p.sync_free_crop_capable() and not _use_cuda_graph(p, args, None, None, 2, 2, None)
    sched = get_t_schedule('expbeta', 2)
    out, _ = sampling(_mid_poses(seed=85, n=2), p, 2, sched, sched, sched, 'cuda:0', partial(t_to_sigma, args=args), args,
                      batch_size=2)
    assert all(torch.isfinite(d['ligand'].pos).all() for d in out)


# ------------------------------------------------------------------------------------------------------ mutation checks
def test_fixture_comparison_catches_an_unswapped_rec_lig_w1(built_lib, monkeypatch):
    from diffdock_b200.tensor_layers import TensorProductConvLayer
    orig = TensorProductConvLayer._fused_plan
    monkeypatch.setattr(TensorProductConvLayer, '_fused_plan', lambda self, fc, table, k_in, swap_ns=0:
                        orig(self, fc, table, k_in, 0))
    assert _fixture_err(4)[0] > 1e-3


def test_fixture_comparison_catches_negated_rec_lig_harmonics(built_lib, monkeypatch):
    from diffdock_b200.old_cg_model import CGOldModel
    orig = CGOldModel._cross_graph_sync_free
    monkeypatch.setattr(CGOldModel, '_cross_graph_sync_free', lambda self, *args, vec_sign: orig(self, *args, vec_sign=-1.0))
    assert _fixture_err(4)[0] > 1e-3


def test_fixture_comparison_catches_sigma_per_batch(built_lib, monkeypatch):
    """Case 4 has one time per complex: receptor node and contact-edge embeddings that take the first complex's sigma for
    the whole batch must fail the comparison."""
    from diffdock_b200.old_cg_model import CGOldModel
    orig = CGOldModel._static

    def first_complex_sigma(self, data):
        c = orig(self, data)
        return dict(c, rr_gid32=torch.zeros_like(c['rr_gid32']), rec_gid=torch.zeros_like(c['rec_gid']))

    monkeypatch.setattr(CGOldModel, '_static', first_complex_sigma)
    assert _fixture_err(4)[0] > 1e-3


def test_sample_complexes_sharded_takes_the_v10_model(cfg_l2_pair):
    """distributed.sample_complexes_sharded with one process: each complex is sampled as one batch of its poses by the
    v1.0 model; the gathered coordinates are those of the per-complex runs."""
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.distributed import sample_complexes_sharded
    from diffdock_b200.sampling import sampling
    _, p, a = cfg_l2_pair
    sched = get_t_schedule('expbeta', 3)
    complexes = [_mid_poses(seed=86, n=3, n_res=80, n_atoms=14), _mid_poses(seed=87, n=2, n_res=100, n_atoms=19)]

    def sample_one(i):
        out, _ = sampling(copy.deepcopy(complexes[i]), p, 3, sched, sched, sched, 'cuda:0', partial(t_to_sigma, args=a), a,
                          batch_size=len(complexes[i]), no_final_step_noise=True, rng='philox', seed=5,
                          pose_keys=[(i << 32) | j for j in range(len(complexes[i]))])
        return torch.stack([d['ligand'].pos.float() for d in out]).to('cuda:0')

    shapes = [(len(c), c[0]['ligand'].pos.shape[0], 3) for c in complexes]
    got = sample_complexes_sharded(2, [3.0, 2.0], shapes, sample_one, device=DEV)
    for i in range(2):
        assert got[i].shape == shapes[i] and rel_err(got[i], sample_one(i)) < 1e-4


def test_receptor_without_contact_edges(cfg_l2_pair, monkeypatch):
    """A receptor cropped down to residues without contact edges between them: the sync-free forward embeds no contact
    edge and agrees with the host-sized one."""
    _, p, _ = cfg_l2_pair
    poses = _mid_poses(seed=88, n=2)
    for g in poses:
        g['receptor', 'receptor'].edge_index = g['receptor', 'receptor'].edge_index[:, :0]
    sync_free = score(p, poses, [0.5, 0.5], DEV, shared=True)
    monkeypatch.setattr(p, '_sync_free', False)
    host = score(p, poses, [0.5, 0.5], DEV)
    assert all(torch.isfinite(t).all() for t in sync_free) and max(_errs(sync_free, host)) < 1e-4

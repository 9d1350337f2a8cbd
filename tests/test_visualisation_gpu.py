"""GPU: the reverse-diffusion frames ``sampling(..., visualization_list=...)`` records in a device buffer, on the eager loop
and on the captured step, against the unmodified reference (tests/golden/ref_sampling_visualisation.pt) and against each
other under Philox noise."""
import copy
from functools import partial
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests.parity_helpers import golden_model, load_golden, make_model_pair
from tests.visualisation_helpers import BATCH_SIZE, max_rel_diff, fused_case_model, prepopulated

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TEMPS = dict(temp_sampling=[1.170050527854316, 2.06391612594481, 7.044261621607846],
             temp_psi=[0.727287304570729, 0.9022615585677628, 0.5946212391366862],
             temp_sigma_data=[0.9299802531572672, 0.7464326999906034, 0.6943254174849822])


def _fixture():
    from diffdock_b200.hetero import graph_from_dict
    fx = load_golden('ref_sampling_visualisation.pt')
    return fx, [graph_from_dict(d) for d in fx['poses']]


def _recording_graphed_steps(monkeypatch):
    from diffdock_b200 import sampling as smod
    made = []

    class Recorder(smod.GraphedSteps):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)

    monkeypatch.setattr(smod, 'GraphedSteps', Recorder)
    return made


def _check_against_fixture(run, vis, out, fx):
    for i, (v, ref) in enumerate(zip(vis, run['content'])):
        got = v.content()
        assert max_rel_diff(got, ref) < 1e-4, i
        assert torch.equal(got[1][2], out[i]['ligand'].pos.cpu() + fx['original_center'][i])


def test_eager_frames_match_reference_run_a(built_lib):
    """Injected CPU noise (the reference's draws, same seed and call order) forces the eager loop; two batches of 2."""
    from diffdock_b200.diffusion_utils import t_to_sigma
    from diffdock_b200.sampling import sampling
    fx, poses = _fixture()
    run = fx['runs']['a']
    m, _, a = golden_model(load_golden('ref_cg_model.pt')[run['model_case']], 'product')
    vis = prepopulated(poses, fx['crystal'])
    torch.manual_seed(run['seed'])
    noise = lambda kind, shape: torch.normal(mean=0, std=1, size=shape)
    sched = fx['schedule']
    out, _ = sampling(copy.deepcopy(poses), m, fx['steps'], sched, sched, sched, DEV, partial(t_to_sigma, args=a), a,
                      batch_size=fx['batch_size'], no_final_step_noise=True, noise_fn=noise, visualization_list=vis,
                      **TEMPS)
    _check_against_fixture(run, vis, out, fx)


def test_graphed_frames_match_reference_run_b(built_lib, monkeypatch):
    from diffdock_b200.diffusion_utils import t_to_sigma
    from diffdock_b200.sampling import sampling
    fx, poses = _fixture()
    run = fx['runs']['b']
    m, a = fused_case_model(fx['fused_case'])
    made = _recording_graphed_steps(monkeypatch)
    vis = prepopulated(poses, fx['crystal'])
    sched = fx['schedule']
    out, _ = sampling(copy.deepcopy(poses), m, fx['steps'], sched, sched, sched, DEV, partial(t_to_sigma, args=a), a,
                      batch_size=fx['batch_size'], no_final_step_noise=True, no_random=True, cuda_graph=True,
                      visualization_list=vis, **TEMPS)
    assert len(made) == 2 and all(s.frames is not None for s in made)       # both batches captured, frames in the graph
    _check_against_fixture(run, vis, out, fx)


def _args(**over):
    from diffdock_b200.synthetic import default_model_args
    kw = dict(ns=16, nv=4, sh_lmax=2, num_conv_layers=3, distance_embed_dim=16, cross_distance_embed_dim=16, sigma_embed_dim=16)
    kw.update(over)
    return default_model_args(**kw)


def _poses(n=3, seed=41):
    from diffdock_b200.synthetic import make_pose_list
    poses = make_pose_list(n, n_res=120, n_atoms=12, seed=seed, tr_sigma_max=19.0)
    for i, p in enumerate(poses):
        p.original_center = torch.tensor([[4.0 * i - 20.0, 11.5, -3.25 * i]])
    return poses


def _sample(model, args, poses, steps=6, vis=True, **kw):
    """(recorders or None, final positions [N, n_atoms, 3], confidence); 3 poses in batches of 2 make a partial last batch."""
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sampling
    sched = get_t_schedule('expbeta', steps)
    rec = prepopulated(poses, poses[0]['ligand'].pos) if vis else None
    out, conf = sampling(copy.deepcopy(poses), model, steps, sched, sched, sched, DEV, partial(t_to_sigma, args=args), args,
                         batch_size=BATCH_SIZE, no_final_step_noise=True, rng='philox', seed=123, visualization_list=rec,
                         **TEMPS, **kw)
    return rec, torch.stack([d['ligand'].pos for d in out]).cpu(), conf


def _frame_diff(ra, rb):
    d = 0.0
    for x, y in zip(ra, rb):
        cx, cy = x.content(), y.content()
        assert cx.keys() == cy.keys() and all(cx[p].keys() == cy[p].keys() for p in cx)
        for p in cx:
            for o, v in cx[p].items():
                if torch.is_tensor(v):
                    d = max(d, float((v - cy[p][o]).abs().max()))
    return d


def test_graphed_frames_match_eager_under_philox(built_lib, monkeypatch):
    args = _args()
    _, p = make_model_pair(args, seed=9)
    poses = _poses()
    made = _recording_graphed_steps(monkeypatch)
    rg, pg, _ = _sample(p, args, poses, cuda_graph=True)
    assert len(made) == 2 and all(s.frames is not None for s in made)
    re, pe, _ = _sample(p, args, poses, cuda_graph=False)
    assert torch.isfinite(pg).all()
    assert float((pg - pe).abs().max()) < 2e-3          # 6 chained steps; scatter-atomic order differs run to run
    assert _frame_diff(rg, re) < 2e-3
    for r in rg:                                        # part 1: the prior sample, then orders 2 .. steps + 1
        assert sorted(r.parts[1]) == list(range(1, 8))


def test_graphed_step_with_frames_is_sync_free(built_lib):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.hetero import collate_shared_receptor
    from diffdock_b200.sampling import GraphedSteps, _step_tables
    args = _args()
    _, model = make_model_pair(args, seed=9)
    poses = _poses(4)
    g = collate_shared_receptor(poses, DEV)
    b, n = g.num_graphs, poses[0]['ligand'].num_nodes
    lig0 = poses[0]['ligand']
    mask_u8 = torch.from_numpy(np.asarray(lig0.mask_rotate[0]).astype(np.uint8)).to(DEV)
    rb = poses[0]['ligand', 'ligand'].edge_index.T[lig0.edge_mask]
    bu, bv = rb[:, 0].int().contiguous().to(DEV), rb[:, 1].int().contiguous().to(DEV)
    sched = get_t_schedule('expbeta', 6)
    coef, t_rows = _step_tables(6, sched, sched, sched, partial(t_to_sigma, args=args), args, False, False, True, 1.0, 0.0,
                                0.5)
    frames = torch.full((6, b * n, 3), float('nan'), device=DEV)
    steps = GraphedSteps(model, g, b, coef, t_rows, bu, bv, mask_u8, True, DEV, draw_noise=True,
                         philox=(3, torch.arange(b, device=DEV)), frames=frames)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        steps.run(6)
        done = steps.step.clone()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert int(done.item()) == 6 and torch.isfinite(frames).all()
    assert torch.equal(frames[-1], steps.pos)
    assert all(float((frames[t + 1] - frames[t]).abs().max()) > 0 for t in range(5))


@pytest.mark.parametrize("crop_beyond", [None, 20.0])
def test_frames_change_nothing_else(built_lib, monkeypatch, crop_beyond):
    """Graphed, Philox noise, ranked, with and without the per-step crop: the same final poses and confidences with and
    without frames (up to the scatter-atomic order of two runs), and the last frame is the final pose exactly."""
    from diffdock_b200.diffusion_utils import get_timestep_embedding
    from diffdock_b200.old_cg_model import CGOldModel
    args = _args(crop_beyond=crop_beyond)
    _, p = make_model_pair(args, seed=9)
    assert p.sync_free_crop_capable()
    made = _recording_graphed_steps(monkeypatch)
    torch.manual_seed(4)
    conf = CGOldModel(None, torch.device(DEV), get_timestep_embedding('sinusoidal', 16, args.embedding_scale), ns=16, nv=4,
                      num_conv_layers=2, sigma_embed_dim=16, distance_embed_dim=16, cross_distance_embed_dim=16,
                      confidence_mode=True, use_old_atom_encoder=True, lm_embedding_type='esm', lm_embedding_dim=1280,
                      dynamic_max_cross=True, cross_max_distance=80.0).eval().to(DEV)
    poses = _poses()
    kw = dict(confidence_model=conf, confidence_data_list=[d.clone() for d in poses],
              confidence_model_args=SimpleNamespace(crop_beyond=None, all_atoms=False), cuda_graph=True)
    rec, pos, c1 = _sample(p, args, poses, **kw)
    _, pos0, c0 = _sample(p, args, poses, vis=False, **kw)
    assert [s.frames is not None for s in made] == [True, True, False, False]
    assert all((s.crop is not None) == (crop_beyond is not None) for s in made)
    assert float((pos - pos0).abs().max()) < 2e-3
    assert float((c1 - c0).abs().max()) < 2e-3
    for i, r in enumerate(rec):
        final = pos[i] + poses[i].original_center
        assert torch.equal(r.parts[1][2], final) and torch.equal(r.parts[1][7], final)

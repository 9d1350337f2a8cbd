"""GPU parity of the all-atom score model (SURVEY.md section 8, row f3): diffdock_b200.aa_model.AAModel vs the reference
fixture (models/aa_model.py run unmodified, tests/golden/make_golden_aa_model.py), vs the CPU oracle at DiffDock-L widths, and
inside the sampler."""
import copy
from functools import partial

import pytest
import torch

from diffdock_b200.hetero import collate
from tests.parity_helpers import golden_model, load_golden, rand_bn_, rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("idx", [0, 1, 2])
def test_all_atom_score_model_matches_reference_fixture(built_lib, idx):
    from diffdock_b200.diffusion_utils import set_time
    case = load_golden('ref_aa_model.pt')[idx]
    m, poses, a = golden_model(case, 'product', all_atoms=True)
    b = collate(copy.deepcopy(poses)).to('cuda:0')
    t = case['t']
    set_time(b, None, t, t, t, len(poses), True, 'cuda:0')
    tr, rot, tor, _ = m(b)
    torch.cuda.synchronize()
    for got, key in ((tr, 'tr'), (rot, 'rot'), (tor, 'tor')):
        assert got.shape == case[key].shape and rel_err(got, case[key]) < 1e-4, key
    # the caches the reference leaves on the batch (models/aa_model.py:319-333)
    assert hasattr(b['receptor'], 'rec_node_attr') and hasattr(b['atom'], 'atom_node_attr')
    again = m(b)                                              # second call takes the cached receptor / atom part
    assert rel_err(again[0], tr) < 1e-5


def test_all_atom_score_model_full_width_matches_oracle(built_lib):
    """ns=48, nv=10: all nine groups on the fully fused wgmma kernel."""
    from oracle.aa_model import AAModel as OModel
    from oracle.diffusion import set_time as o_set_time, t_to_sigma as o_t2s
    from oracle.layers import get_timestep_embedding as o_temb
    from diffdock_b200.aa_model import AAModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, set_time, t_to_sigma
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    a = default_model_args(num_conv_layers=3, distance_embed_dim=16, cross_distance_embed_dim=16, sigma_embed_dim=16)
    kw = dict(sigma_embed_dim=16, sh_lmax=2, ns=48, nv=10, num_conv_layers=3, lig_max_radius=a.max_radius,
              rec_max_radius=a.rec_max_radius, cross_max_distance=a.cross_max_distance, center_max_distance=a.center_max_distance,
              distance_embed_dim=16, cross_distance_embed_dim=16, dynamic_max_cross=True, lm_embedding_type=None,
              embed_also_ligand=True)
    torch.manual_seed(21)
    mo = OModel(partial(o_t2s, args=a), 'cpu', o_temb('sinusoidal', 16, a.embedding_scale), **kw).eval()
    g = torch.Generator().manual_seed(22)
    for mod in mo.modules():
        if mod.__class__.__name__ == 'BatchNorm':
            rand_bn_(mod, g)
    mp = AAModel(partial(t_to_sigma, args=a), torch.device('cuda:0'), get_timestep_embedding('sinusoidal', 16, a.embedding_scale),
                 **kw).eval()
    mp.load_state_dict(mo.state_dict(), strict=True)
    mp = mp.to('cuda:0')
    assert all(layer.fused_capable(48, 48) for layer in mp.conv_layers)
    poses = make_pose_list(2, n_res=40, n_atoms=12, seed=91, tr_sigma_max=a.tr_sigma_max * 0.3, lm_dim=0, all_atoms=True)
    t = 0.3
    b = collate(copy.deepcopy(poses))
    o_set_time(b, t, t, t, 2, 'cpu', all_atoms=True)
    with torch.no_grad():
        ref = mo(b)
    bg = collate(copy.deepcopy(poses)).to('cuda:0')
    set_time(bg, None, t, t, t, 2, True, 'cuda:0')
    assert mp.sync_free_capable()                 # the forward below has no device->host read (capacity buffers)
    got = mp(bg)
    for x, y in zip(got[:3], ref[:3]):
        assert rel_err(x, y) < 1e-4
    # the host-sized forward (exact neighbour-list sizes read back) gives the same scores
    mp._sync_free = False
    bh = collate(copy.deepcopy(poses)).to('cuda:0')
    set_time(bh, None, t, t, t, 2, True, 'cuda:0')
    host = mp(bh)
    for x, y in zip(got[:3], host[:3]):
        assert rel_err(x, y) < 2e-5


def test_all_atom_step_in_a_cuda_graph_matches_the_eager_loop(built_lib):
    """Full-width all-atom model: sampling() captures the nine-group step in a CUDA graph; same poses as the eager loop."""
    from argparse import Namespace
    from diffdock_b200.aa_model import AAModel
    from diffdock_b200.diffusion_utils import get_t_schedule, get_timestep_embedding, t_to_sigma
    from diffdock_b200.sampling import sampling
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    a = default_model_args(num_conv_layers=2, distance_embed_dim=16, cross_distance_embed_dim=16, sigma_embed_dim=16, all_atoms=True)
    kw = dict(sigma_embed_dim=16, sh_lmax=2, ns=48, nv=10, num_conv_layers=2, lig_max_radius=a.max_radius,
              rec_max_radius=a.rec_max_radius, cross_max_distance=a.cross_max_distance, center_max_distance=a.center_max_distance,
              distance_embed_dim=16, cross_distance_embed_dim=16, dynamic_max_cross=True, lm_embedding_type=None,
              embed_also_ligand=True)
    torch.manual_seed(5)
    m = AAModel(partial(t_to_sigma, args=a), torch.device('cuda:0'), get_timestep_embedding('sinusoidal', 16, a.embedding_scale),
                **kw).eval().to('cuda:0')
    assert m.sync_free_capable()
    poses = make_pose_list(3, n_res=40, n_atoms=12, seed=17, tr_sigma_max=a.tr_sigma_max * 0.5, lm_dim=0, all_atoms=True)
    sched = get_t_schedule('expbeta', 4)
    run = lambda graph: torch.stack([d['ligand'].pos for d in sampling(
        copy.deepcopy(poses), m, 4, sched, sched, sched, 'cuda:0', partial(t_to_sigma, args=a), a, batch_size=3, no_random=True,
        cuda_graph=graph)[0]]).cpu()
    eager, graphed = run(False), run(True)
    assert torch.isfinite(graphed).all() and float((eager - graphed).abs().max()) < 2e-3


def test_sampler_runs_the_all_atom_score_model(built_lib):
    """sampling() with model_args.all_atoms=True: set_time covers the atom nodes, the eager step loop is used."""
    from argparse import Namespace
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sampling
    case = load_golden('ref_aa_model.pt')[0]
    m, poses, a = golden_model(case, 'product', all_atoms=True)
    margs = Namespace(**{**case['args'], 'all_atoms': True})
    sched = get_t_schedule('expbeta', 3)
    torch.manual_seed(0)
    out, _ = sampling(copy.deepcopy(poses), m, 3, sched, sched, sched, 'cuda:0', partial(t_to_sigma, args=a), margs,
                      batch_size=3, no_final_step_noise=True)
    pos = torch.stack([d['ligand'].pos for d in out])
    assert torch.isfinite(pos).all() and pos.shape == (3, 9, 3)

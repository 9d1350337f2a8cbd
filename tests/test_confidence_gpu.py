"""GPU parity of the confidence model (SURVEY.md section 8, row f2): diffdock_b200.old_cg_model.CGOldModel vs the reference
fixture (models/old_cg_model.py run unmodified, tests/golden/make_golden_confidence.py) and vs the CPU oracle."""
import copy
from functools import partial

import pytest
import torch

from diffdock_b200.hetero import collate
from tests.parity_helpers import golden_confidence_model, golden_model, load_golden

pytestmark = pytest.mark.gpu


def _confidence(m, poses, dev):
    from diffdock_b200.diffusion_utils import set_time
    b = collate(copy.deepcopy(poses)).to(dev)
    set_time(b, 0, 0, 0, 0, len(poses), False, dev)
    return m(b).float().cpu()


@pytest.mark.parametrize("idx", [0, 1, 2])
def test_confidence_matches_reference_fixture(built_lib, idx):
    case = load_golden('ref_confidence.pt')[idx]
    m, poses = golden_confidence_model(case, 'product')
    conf = _confidence(m, poses, torch.device('cuda:0'))
    ref = case['confidence']
    assert conf.shape == ref.shape
    assert (conf - ref).abs().max() < 1e-4 * max(1.0, float(ref.abs().max())), (conf, ref)     # tolerance: 1e-4 relative


def test_confidence_full_width_matches_oracle(built_lib):
    """DiffDock-L-sized widths (ns=48, nv=10: the fully fused wgmma path) on a 60-residue complex, against the oracle."""
    from oracle.diffusion import set_time as o_set_time, t_to_sigma as o_t2s
    from oracle.layers import get_timestep_embedding as o_temb
    from oracle.old_cg_model import CGOldModel as OModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    from diffdock_b200.old_cg_model import CGOldModel
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    from tests.parity_helpers import rand_bn_
    a = default_model_args()
    kw = dict(sigma_embed_dim=16, sh_lmax=2, ns=48, nv=10, num_conv_layers=4, cross_max_distance=30.0,
              distance_embed_dim=16, cross_distance_embed_dim=16, lm_embedding_type='esm', lm_embedding_dim=32,
              confidence_mode=True, use_old_atom_encoder=True)
    torch.manual_seed(5)
    mo = OModel(partial(o_t2s, args=a), 'cpu', o_temb('sinusoidal', 16, a.embedding_scale), **kw).eval()
    g = torch.Generator().manual_seed(6)
    for mod in mo.modules():
        if mod.__class__.__name__ in ('BatchNorm', 'BatchNorm1d'):
            rand_bn_(mod, g)
    mp = CGOldModel(partial(t_to_sigma, args=a), torch.device('cuda:0'),
                    get_timestep_embedding('sinusoidal', 16, a.embedding_scale), **kw).eval()
    mp.load_state_dict(mo.state_dict(), strict=True)
    mp = mp.to('cuda:0')
    poses = make_pose_list(4, n_res=60, n_atoms=14, seed=77, tr_sigma_max=1.0, lm_dim=32)
    b = collate(copy.deepcopy(poses))
    o_set_time(b, 0, 0, 0, len(poses), 'cpu')
    with torch.no_grad():
        ref = mo(b)
    conf = _confidence(mp, poses, torch.device('cuda:0'))
    assert (conf - ref).abs().max() < 1e-4 * max(1.0, float(ref.abs().max())), (conf, ref)


def test_sampling_returns_confidence(built_lib):
    """sampling(confidence_model=...) ranks the final poses like utils/sampling.py:208-227: the confidences it returns
    equal the confidence model applied to the returned poses."""
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sampling
    case = load_golden('ref_cg_model.pt')[0]
    score, poses, a = golden_model(case, 'product')
    ccase = load_golden('ref_confidence.pt')[0]
    conf_model, _ = golden_confidence_model(ccase, 'product')
    sched = get_t_schedule('expbeta', 3)
    torch.manual_seed(0)
    out, conf = sampling(copy.deepcopy(poses), score, 3, sched, sched, sched, 'cuda:0', partial(t_to_sigma, args=a), a,
                         batch_size=3, no_final_step_noise=True, confidence_model=conf_model,
                         confidence_data_list=copy.deepcopy(poses), confidence_model_args=a)
    assert conf.shape == (3,) and torch.isfinite(conf).all()
    again = _confidence(conf_model, [d.to('cpu') if hasattr(d, 'to') else d for d in out], torch.device('cuda:0'))
    assert (conf.cpu() - again).abs().max() < 1e-5


@pytest.mark.parametrize("run", [0, 1])
def test_sampling_with_confidence_matches_reference_fixture(built_lib, run):
    """Product sampling() + confidence model vs the reference's utils/sampling.py run (fixture): final poses and ranking
    scores, without and with confidence_model_args.crop_beyond (device-side crop_receptor instead of the reference's
    to_data_list / crop / re-collate)."""
    from argparse import Namespace
    from diffdock_b200.diffusion_utils import t_to_sigma
    from diffdock_b200.sampling import sampling
    s = load_golden('ref_sampling_confidence.pt')
    r = s['runs'][run]
    score, poses, a = golden_model(load_golden('ref_cg_model.pt')[s['score_case']], 'product')
    conf_model, _ = golden_confidence_model(load_golden('ref_confidence.pt')[s['confidence_case']], 'product')
    torch.manual_seed(s['seed'])
    noise = lambda kind, shape: torch.normal(mean=0, std=1, size=shape)           # the reference's CPU draws
    out, conf = sampling(copy.deepcopy(poses), score, len(s['schedule']), s['schedule'], s['schedule'], s['schedule'],
                         'cuda:0', partial(t_to_sigma, args=a), a, batch_size=3, no_final_step_noise=True,
                         confidence_model=conf_model, confidence_data_list=copy.deepcopy(poses),
                         confidence_model_args=Namespace(all_atoms=False, crop_beyond=r['crop_beyond']), noise_fn=noise)
    for d, ref in zip(out, r['final_pos']):
        err = float((d['ligand'].pos.cpu() - ref).abs().max() / ref.abs().max())
        assert err < 1e-4, err
    assert (conf.cpu() - r['confidence']).abs().max() < 1e-4, (conf, r['confidence'])


# ---------------------------------------------------------------------------------------------- all-atom confidence model
def _confidence_aa(m, poses, dev):
    from diffdock_b200.diffusion_utils import set_time
    b = collate(copy.deepcopy(poses)).to(dev)
    set_time(b, 0, 0, 0, 0, len(poses), True, dev)
    return m(b).float().cpu()


@pytest.mark.parametrize("idx", [0, 1, 2])
def test_all_atom_confidence_matches_reference_fixture(built_lib, idx):
    """diffdock_b200.old_aa_model.AAOldModel vs models/old_aa_model.py run unmodified (ref_confidence_aa.pt)."""
    case = load_golden('ref_confidence_aa.pt')[idx]
    m, poses = golden_confidence_model(case, 'product', all_atoms=True)
    conf = _confidence_aa(m, poses, torch.device('cuda:0'))
    ref = case['confidence']
    assert conf.shape == ref.shape
    assert (conf - ref).abs().max() < 1e-4 * max(1.0, float(ref.abs().max())), (conf, ref)


def test_all_atom_confidence_full_width_matches_oracle(built_lib):
    """DiffDock-L-sized widths (ns=48, nv=10: the fully fused wgmma path for all nine convolutions) vs the oracle."""
    from oracle.diffusion import set_time as o_set_time, t_to_sigma as o_t2s
    from oracle.layers import get_timestep_embedding as o_temb
    from oracle.old_aa_model import AAOldModel as OModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    from diffdock_b200.old_aa_model import AAOldModel
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    from tests.parity_helpers import rand_bn_
    a = default_model_args()
    kw = dict(sigma_embed_dim=16, sh_lmax=2, ns=48, nv=10, num_conv_layers=3, cross_max_distance=30.0,
              distance_embed_dim=16, cross_distance_embed_dim=16, lm_embedding_type='esm', lm_embedding_dim=32,
              confidence_mode=True, use_old_atom_encoder=True)
    torch.manual_seed(15)
    mo = OModel(partial(o_t2s, args=a), 'cpu', o_temb('sinusoidal', 16, a.embedding_scale), **kw).eval()
    g = torch.Generator().manual_seed(16)
    for mod in mo.modules():
        if mod.__class__.__name__ in ('BatchNorm', 'BatchNorm1d'):
            rand_bn_(mod, g)
    mp = AAOldModel(partial(t_to_sigma, args=a), torch.device('cuda:0'),
                    get_timestep_embedding('sinusoidal', 16, a.embedding_scale), **kw).eval()
    mp.load_state_dict(mo.state_dict(), strict=True)
    mp = mp.to('cuda:0')
    poses = make_pose_list(3, n_res=40, n_atoms=12, seed=87, tr_sigma_max=1.0, lm_dim=32, all_atoms=True)
    b = collate(copy.deepcopy(poses))
    o_set_time(b, 0, 0, 0, len(poses), 'cpu', all_atoms=True)
    with torch.no_grad():
        ref = mo(b)
    conf = _confidence_aa(mp, poses, torch.device('cuda:0'))
    assert (conf - ref).abs().max() < 1e-4 * max(1.0, float(ref.abs().max())), (conf, ref)


def test_sampling_ranks_with_all_atom_confidence_model(built_lib):
    """sampling(confidence_model=AAOldModel, confidence_model_args.all_atoms=True): the coarse-grained score model moves the
    poses, the all-atom model ranks them on its own (all-atom) copies of the complexes, utils/sampling.py:208-227."""
    from argparse import Namespace
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.hetero import graph_from_dict
    from diffdock_b200.sampling import sampling
    case = load_golden('ref_cg_model.pt')[0]
    score, poses, a = golden_model(case, 'product')
    ccase = load_golden('ref_confidence_aa.pt')[0]
    conf_model, aa_poses = golden_confidence_model(ccase, 'product', all_atoms=True)
    # the ranking model sees its own featurisation of the same complex: give the all-atom graphs the score model's ligand
    lig_keys = ('x', 'pos', 'edge_mask', 'mask_rotate')
    conf_list = []
    for p, q in zip(poses, aa_poses):
        c = copy.deepcopy(q)
        for k in lig_keys:
            setattr(c['ligand'], k, copy.deepcopy(getattr(p['ligand'], k)))
        c['ligand', 'ligand'].edge_index = p['ligand', 'ligand'].edge_index.clone()
        c['ligand', 'ligand'].edge_attr = p['ligand', 'ligand'].edge_attr.clone()
        conf_list.append(c)
    sched = get_t_schedule('expbeta', 3)
    torch.manual_seed(0)
    out, conf = sampling(copy.deepcopy(poses), score, 3, sched, sched, sched, 'cuda:0', partial(t_to_sigma, args=a), a,
                         batch_size=3, no_final_step_noise=True, confidence_model=conf_model,
                         confidence_data_list=conf_list, confidence_model_args=Namespace(all_atoms=True, crop_beyond=None))
    assert conf.shape == (3,) and torch.isfinite(conf).all()
    again = []
    for d, c in zip(out, conf_list):
        c2 = copy.deepcopy(c)
        c2['ligand'].pos = d['ligand'].pos.cpu()
        again.append(c2)
    ref = _confidence_aa(conf_model, again, torch.device('cuda:0'))
    assert (conf.cpu() - ref).abs().max() < 1e-5

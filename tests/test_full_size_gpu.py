"""Full-size (BASELINE config 2: 1500 residues / 40 ligand atoms / 32 poses, CFG-L2 widths) checks through size-independent
properties - the CPU oracle cannot run this size in seconds:
  * SE(3) equivariance: rotating + translating every complex rotates the translation / rotation scores and leaves the torsion
    scores unchanged;
  * pose permutation: reversing the order of the poses in the batch reverses the scores (run with fixed_center_conv=True - with
    the default False the reference itself makes tr/rot depend on the batch composition)."""
import copy
import math
from functools import partial

import pytest
import torch

pytestmark = pytest.mark.gpu


def _rotation(seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(4, generator=g, dtype=torch.float64)
    r, i, j, k = (q / q.norm()).tolist()
    return torch.tensor([[1 - 2 * (j * j + k * k), 2 * (i * j - k * r), 2 * (i * k + j * r)],
                         [2 * (i * j + k * r), 1 - 2 * (i * i + k * k), 2 * (j * k - i * r)],
                         [2 * (i * k - j * r), 2 * (j * k + i * r), 1 - 2 * (i * i + j * j)]], dtype=torch.float64)


def test_full_size_equivariance_and_pose_permutation(built_lib):
    from bench import model_kwargs, randomise_bn
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, set_time, t_to_sigma
    from diffdock_b200.hetero import collate
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    dev = torch.device('cuda:0')
    a = default_model_args()
    torch.manual_seed(0)
    model = CGModel(partial(t_to_sigma, args=a), dev, get_timestep_embedding('sinusoidal', a.sigma_embed_dim, a.embedding_scale),
                    fixed_center_conv=True, **model_kwargs(a)).eval()
    randomise_bn(model, 1)
    model = model.to(dev)
    n_poses, t = 32, 0.3
    poses = make_pose_list(n_poses, n_res=1500, n_atoms=40, seed=100, tr_sigma_max=a.tr_sigma_max * t)

    def scores(plist):
        g = collate(plist).to(dev)
        set_time(g, None, t, t, t, len(plist), False, dev)
        tr, rot, tor = model(g)[:3]
        torch.cuda.synchronize()
        return tr.double().cpu(), rot.double().cpu(), tor.double().cpu()

    tr, rot, tor = scores(copy.deepcopy(poses))
    assert tr.shape == (n_poses, 3) and rot.shape == (n_poses, 3) and tor.numel() > 0
    assert torch.isfinite(tr).all() and torch.isfinite(rot).all() and torch.isfinite(tor).all()
    rel = lambda x, y: float((x - y).abs().max() / y.abs().max())

    # --- rigid motion of every complex ---
    R, shift = _rotation(7), torch.tensor([3.0, -4.0, 2.5], dtype=torch.float64)
    moved = copy.deepcopy(poses)
    for p in moved:
        for nt in ('ligand', 'receptor'):
            p[nt].pos = (p[nt].pos.double() @ R.T + shift).float()
    tr2, rot2, tor2 = scores(moved)
    e = (rel(tr2, tr @ R.T), rel(rot2, rot @ R.T), rel(tor2, tor))
    assert max(e) < 5e-4, e            # fp32 positions after the motion + split-bf16 radial MLP; scores themselves hold 1e-4

    # --- order of the poses in the batch ---
    tr3, rot3, tor3 = scores(copy.deepcopy(poses)[::-1])
    nb = tor.numel() // n_poses
    e = (rel(tr3.flip(0), tr), rel(rot3.flip(0), rot), rel(tor3.reshape(n_poses, nb).flip(0).reshape(-1), tor))
    assert max(e) < 1e-4, e

"""GPU: the sync-free ligand graph where radius_graph's cap of 32 neighbours binds.

radius_graph caps the neighbours of each CENTRE atom, and its edges point from the centre to the neighbour, which is the
convolution's target (models/cg_model.py:478-483).  A 40-atom ligand folded by its torsions has atoms with more than 32
others within 5 A, so the graph is not symmetric there.  The sync-free forward used to search per target instead, which
gives the transposed lists wherever the cap binds.  A lone pose of the test complex stayed below the cap, so full-size
single poses agreed with the oracle; batches of several poses were off by up to 1.5e-2 for the default model.  The
comparisons here are against the host-sized forward, whose ligand graph is the reference's (tests/test_full_size_parity_gpu.py
pins it to the oracle)."""
import copy

import pytest
import torch

from tests.parity_helpers import make_model_pair, rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _batch(poses, t, shared):
    from diffdock_b200.diffusion_utils import set_time
    from diffdock_b200.hetero import collate, collate_shared_receptor
    g = collate_shared_receptor([q.clone() for q in poses], DEV) if shared else collate(copy.deepcopy(poses)).to(DEV)
    set_time(g, None, t, t, t, len(poses), False, DEV)
    g._uniform_t = shared            # the sampler's promise: one diffusion time for the whole batch
    return g


def test_sync_free_ligand_graph_is_the_references_where_the_cap_binds(built_lib):
    from diffdock_b200 import ops
    from diffdock_b200.layers import ligand_graph
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    args = default_model_args(ns=16, nv=4, num_conv_layers=3, distance_embed_dim=16, cross_distance_embed_dim=16,
                              sigma_embed_dim=16)
    _, p = make_model_pair(args, seed=1)
    poses = make_pose_list(4, n_res=60, n_atoms=40, seed=100, tr_sigma_max=args.tr_sigma_max * 0.5)
    g = _batch(poses, 0.5, shared=False)
    c = p._static(g)
    pos = g['ligand'].pos.float()
    _, _, n_within = ops.radius(pos, pos, c['lig_ptr'], g['ligand'].batch, r=p.lig_max_radius, max_num_neighbors=1 << 30,
                                exclude_self=True)
    assert int(n_within.max()) > 32, 'the cap must bind for this test to mean anything'
    tgt_h, src_h, _, vec_h, _, _ = ligand_graph(p, g, c['lig_ptr'])
    n_bonds = g['ligand', 'ligand'].edge_index.shape[1]
    # where the cap binds the radius edges are not symmetric: some (neighbour, centre) pair has no (centre, neighbour)
    key = tgt_h[n_bonds:] * pos.shape[0] + src_h[n_bonds:]
    key_t = src_h[n_bonds:] * pos.shape[0] + tgt_h[n_bonds:]
    assert not torch.equal(torch.sort(key).values, torch.sort(key_t).values)
    tgt_h, order = torch.sort(tgt_h, stable=True)
    src_h, vec_h = src_h[order], vec_h[order]
    tgt, src, _, vec, _, extra = p._ligand_edges_sync_free(g, c)
    n = int(extra['n_edges_dev'].item())
    assert n == tgt_h.shape[0] and n <= tgt.shape[0]
    assert torch.equal(tgt[:n].long(), tgt_h) and torch.equal(src[:n].long(), src_h)
    assert torch.equal(vec[:n], vec_h)


@pytest.mark.parametrize('shared', [False, True])
def test_several_full_size_poses_match_host_sized(built_lib, shared):
    """Three 1500-residue / 40-atom poses of config 3's complex in one batch, default model (ns=48, nv=10, 6 layers); with
    ``shared`` through the sampler's collate and the shared layer-0 receptor messages."""
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    args = default_model_args()
    _, p = make_model_pair(args, seed=0)
    assert p.sync_free_capable()
    host = copy.deepcopy(p)
    host._sync_free = False
    for t in (1.0, 0.5):
        poses = make_pose_list(3, n_res=1500, n_atoms=40, seed=100, tr_sigma_max=args.tr_sigma_max * t)
        got, ref = p(_batch(poses, t, shared)), host(_batch(poses, t, shared))
        torch.cuda.synchronize()
        for a, b in zip(got[:3], ref[:3]):
            assert rel_err(a, b) < 1e-4, (t, rel_err(a, b))

"""CPU: the host side of packing all-atom complexes - the pack cost with receptor atoms, the index maps between a packed or
shared-receptor all-atom batch and its distinct receptors (residues, receptor atoms, atom-atom and atom-residue edges), and
``sample_packed``'s refusals for the all-atom score model."""
from functools import partial

import numpy as np
import pytest
import torch


def _complexes(shared=True, n_poses=(3, 2, 4), sizes=((20, 12), (24, 20), (20, 9)), seed=5, rigid=()):
    """Pose lists of all-atom complexes; with ``shared`` the first and the last use the same receptor (residues, atoms and
    their edges)."""
    from diffdock_b200.synthetic import make_pose_list
    out = []
    for k, ((n_res, n_atoms), n) in enumerate(zip(sizes, n_poses)):
        poses = make_pose_list(n, n_res=n_res, n_atoms=n_atoms, seed=seed + k, tr_sigma_max=5.0, lm_dim=8, all_atoms=True)
        if k in rigid:
            for d in poses:
                d['ligand'].edge_mask = torch.zeros_like(d['ligand'].edge_mask)
                d['ligand'].mask_rotate = [np.zeros((0, d['ligand'].num_nodes), dtype=bool)]
        out.append(poses)
    if shared:
        src = out[0][0]
        for d in out[-1]:
            for nt in ('receptor', 'atom'):
                d._nodes[nt] = src._nodes[nt]
            for et in (('receptor', 'receptor'), ('atom', 'atom'), ('atom', 'receptor')):
                d._edges[et] = src._edges[et]
    return out


def _tiles(g):
    from diffdock_b200.aa_model import AAModel
    ei = lambda et: g[et].edge_index.long()
    return AAModel._receptor_tiles(g, g.num_graphs, ei(('receptor', 'receptor')), ei(('atom', 'atom')),
                                   ei(('atom', 'receptor')))


def _check_maps(g, t):
    """Every batch row and edge is its distinct copy's: features, positions and (in the distinct numbering) edge ends."""
    rt, at, lt = t['rec'], t['atom'], t['ar']
    for st, tt in ((g['receptor'], rt), (g['atom'], at)):
        for k in ('x', 'pos'):
            v = getattr(st, k)
            assert torch.equal(v[tt['nodes']][tt['node_map']], v)
    for et, tt, m0, m1 in ((('receptor', 'receptor'), rt, rt, rt), (('atom', 'atom'), at, at, at),
                           (('atom', 'receptor'), lt, at, rt)):
        ei = g[et].edge_index.long()
        ends = torch.stack([m0['node_map'][ei[0]], m1['node_map'][ei[1]]])
        assert torch.equal(tt['edge_index'][:, tt['edge_map']], ends), et
        assert torch.equal(tt['edge_index'], ends[:, tt['edges']]), et


def test_packed_all_atom_batch_maps_onto_its_distinct_receptors():
    from diffdock_b200.hetero import collate_packed
    cx = _complexes()
    g = collate_packed(cx, 'cpu')
    t = _tiles(g)
    assert t is not None
    n_res = [cx[k][0]['receptor'].num_nodes for k in (0, 1)]
    n_atom = [cx[k][0]['atom'].num_nodes for k in (0, 1)]
    n_ar = [cx[k][0]['atom', 'receptor'].num_edges for k in (0, 1)]
    assert t['rec']['nodes'].shape[0] == sum(n_res) and t['atom']['nodes'].shape[0] == sum(n_atom)
    assert t['ar']['edges'].shape[0] == sum(n_ar) and t['ar']['edge_map'].shape[0] == 7 * n_ar[0] + 2 * n_ar[1]
    _check_maps(g, t)


def test_shared_receptor_all_atom_batch_maps_onto_one_copy():
    from diffdock_b200.hetero import collate_shared_receptor
    poses = _complexes(shared=False)[1]
    g = collate_shared_receptor(poses, 'cpu')
    assert g['atom']._unique[2] == len(poses)
    t = _tiles(g)
    assert t['atom']['nodes'].tolist() == list(range(poses[0]['atom'].num_nodes))
    assert t['ar']['edges'].tolist() == list(range(poses[0]['atom', 'receptor'].num_edges))
    _check_maps(g, t)


def test_no_maps_without_a_layout_or_when_the_edges_break_it():
    from diffdock_b200.hetero import collate, collate_packed
    cx = _complexes()
    assert _tiles(collate([d for p in cx for d in p])) is None
    g = collate_packed(cx, 'cpu')
    ar = g['atom', 'receptor']
    ar.edge_index = ar.edge_index.clone()
    ar.edge_index[1, 0] = (ar.edge_index[1, 0] + 1) % cx[0][0]['receptor'].num_nodes
    assert _tiles(g) is None                     # copy 0 joins an atom to another residue than the other copies do
    g = collate_packed(cx, 'cpu')
    ar = g['atom', 'receptor']
    ar.edge_index = ar.edge_index[:, 1:]         # one copy short of an edge
    assert _tiles(g) is None


def test_pack_cost_counts_receptor_atoms_for_all_atom_models():
    from diffdock_b200.sampling import PACK_MAX_PAIRS, pack_cost, pack_plan
    cx = _complexes(shared=False)
    for p in cx:
        n_res, n_atom, n_lig = p[0]['receptor'].num_nodes, p[0]['atom'].num_nodes, p[0]['ligand'].num_nodes
        assert n_atom > 2 * n_res
        assert pack_cost(p) == len(p) * n_lig * n_res
        assert pack_cost(p, all_atoms=True) == len(p) * n_lig * (n_res + n_atom)
    cg, aa = [pack_cost(p) for p in cx], [pack_cost(p, True) for p in cx]
    budget = sum(cg)                              # holds every complex when residues are counted alone
    assert pack_plan(cg, budget) == [[0, 1, 2]] and len(pack_plan(aa, budget)) == 3
    assert PACK_MAX_PAIRS == 40 * 40 * 1500


def _aa_model():
    from diffdock_b200.aa_model import AAModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    from diffdock_b200.synthetic import default_model_args
    a = default_model_args(ns=16, nv=4, num_conv_layers=2, distance_embed_dim=16, cross_distance_embed_dim=16,
                           sigma_embed_dim=16, all_atoms=True)
    m = AAModel(partial(t_to_sigma, args=a), torch.device('cpu'), get_timestep_embedding('sinusoidal', 16, a.embedding_scale),
                ns=16, nv=4, num_conv_layers=2, sigma_embed_dim=16, distance_embed_dim=16, cross_distance_embed_dim=16,
                dynamic_max_cross=True, lm_embedding_type=None, embed_also_ligand=True).eval()
    return m, a


def test_sample_packed_refuses_per_step_cropping_of_all_atom_receptors():
    from diffdock_b200.sampling import sample_packed
    m, a = _aa_model()
    a.crop_beyond = 20.0
    with pytest.raises(NotImplementedError, match='crop_beyond'):
        sample_packed(_complexes(), m, 2, [1.0, 0.5], [1.0, 0.5], [1.0, 0.5], 'cpu', None, a, seed=0)
    a.crop_beyond = None
    with pytest.raises(RuntimeError, match='CUDA device only'):      # past the refusals: the all-atom model is accepted
        sample_packed(_complexes(), m, 2, [1.0, 0.5], [1.0, 0.5], [1.0, 0.5], 'cpu', None, a, seed=0)

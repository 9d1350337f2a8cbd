"""GPU: the all-atom score model (``AAModel``) on packed batches of several complexes - its forward on ``collate_packed``
against each complex's own batch, the receptor part computed once per distinct receptor, and ``sample_packed`` against one
``sampling()`` call per complex, captured and eager."""
import copy
from functools import partial

import numpy as np
import pytest
import torch

from tests.parity_helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _complexes(shared=True, n_poses=(3, 2, 4), sizes=((40, 12), (48, 20), (40, 9)), seed=5, rigid=(1,)):
    """Pose lists of all-atom complexes with different ligand sizes; with ``shared`` the first and the last use the same
    receptor (residues, receptor atoms and their edges); the ligands of ``rigid`` have no rotatable bond."""
    from diffdock_b200.synthetic import make_pose_list
    out = []
    for k, ((n_res, n_atoms), n) in enumerate(zip(sizes, n_poses)):
        poses = make_pose_list(n, n_res=n_res, n_atoms=n_atoms, seed=seed + k, tr_sigma_max=5.0, lm_dim=0, all_atoms=True)
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


def _aa_model(fixed_center_conv=False, full=False, seed=3):
    """A randomly initialised AAModel (BatchNorm statistics randomised) and its arguments: ns=16 / nv=4, or with ``full``
    ns=48 / nv=10 and one protein embedding layer."""
    from diffdock_b200.aa_model import AAModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    from diffdock_b200.synthetic import default_model_args
    a = default_model_args(ns=48 if full else 16, nv=10 if full else 4, num_conv_layers=3, distance_embed_dim=16,
                           cross_distance_embed_dim=16, sigma_embed_dim=16, num_prot_emb_layers=1 if full else 0,
                           all_atoms=True, fixed_center_conv=fixed_center_conv)
    kw = dict(sigma_embed_dim=a.sigma_embed_dim, sh_lmax=a.sh_lmax, ns=a.ns, nv=a.nv, num_conv_layers=a.num_conv_layers,
              lig_max_radius=a.max_radius, rec_max_radius=a.rec_max_radius, cross_max_distance=a.cross_max_distance,
              center_max_distance=a.center_max_distance, distance_embed_dim=a.distance_embed_dim,
              cross_distance_embed_dim=a.cross_distance_embed_dim, dynamic_max_cross=a.dynamic_max_cross,
              lm_embedding_type=None, embed_also_ligand=True, num_prot_emb_layers=a.num_prot_emb_layers,
              fixed_center_conv=fixed_center_conv)
    torch.manual_seed(seed)
    m = AAModel(partial(t_to_sigma, args=a), torch.device(DEV),
                get_timestep_embedding('sinusoidal', a.sigma_embed_dim, a.embedding_scale), **kw).eval()
    gen = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for mod in m.modules():
            if hasattr(mod, 'running_var') and hasattr(mod, 'running_mean'):
                mod.running_mean.copy_(0.1 * torch.randn(mod.running_mean.shape, generator=gen))
                mod.running_var.copy_(0.5 + torch.rand(mod.running_var.shape, generator=gen))
    return m.to(DEV), a


def _scores(model, g):
    out = model(g)
    torch.cuda.synchronize()
    return [t.clone() for t in out[:3]]


def _timed(g, t, uniform=True):
    from diffdock_b200.diffusion_utils import set_time
    set_time(g, None, t, t, t, g.num_graphs, True, DEV)
    if uniform:
        g._uniform_t = True
    return g


def _packed_vs_alone(model, cx, t=0.4, drop_centre=False):
    """Largest relative error of the packed forward against each complex's own shared-receptor batch; also checks it
    against the plain collate of all poses with the same centre nodes (no receptor layout: every copy computed)."""
    from diffdock_b200.hetero import collate, collate_packed, collate_shared_receptor
    g = _timed(collate_packed([[d.clone() for d in p] for p in cx], DEV), t)
    if drop_centre:
        del g._globals['_center_node']
    got = _scores(model, g)
    want = [[], [], []]
    for p in cx:
        for i, s in enumerate(_scores(model, _timed(collate_shared_receptor([d.clone() for d in p], DEV), t))):
            want[i].append(s)
    alone = max(rel_err(a, torch.cat(b)) for a, b in zip(got, want))
    if drop_centre:
        return alone
    plain = _timed(collate([d.clone() for p in cx for d in p]).to(DEV), t, uniform=False)
    plain._center_node = g._center_node
    for a, b in zip(got, _scores(model, plain)):
        assert rel_err(a, b) < 1e-4
    return alone


# ---------------------------------------------------------------------------------------------------------------------
# forward
@pytest.mark.parametrize("full", [False, True])
@pytest.mark.parametrize("fixed", [False, True])
def test_packed_forward_matches_each_complex_alone(built_lib, full, fixed):
    model, _ = _aa_model(fixed, full=full)
    assert model.sync_free_capable()
    assert _packed_vs_alone(model, _complexes()) < 1e-4


def test_dropping_the_centre_nodes_breaks_the_default_centre_convolution(built_lib):
    model, _ = _aa_model(False)
    assert _packed_vs_alone(model, _complexes(), drop_centre=True) > 1e-3


def test_receptor_embedded_once_per_distinct_receptor_and_shared_messages(built_lib):
    from diffdock_b200.hetero import collate_packed
    model, _ = _aa_model(False)
    cx = _complexes()                                  # receptors: A (complexes 0 and 2) and B (complex 1)
    n_res = [cx[k][0]['receptor'].num_nodes for k in (0, 1)]
    n_atom = [cx[k][0]['atom'].num_nodes for k in (0, 1)]
    g = collate_packed(cx, DEV)
    assert [b[2:] for b in g['atom']._blocks] == [(3, 0), (2, 1), (4, 0)]
    rows = {'rec': [], 'atom': [], 'shared': 0}
    enc = {'rec': model.rec_node_embedding, 'atom': model.atom_node_embedding}
    for k, m in enc.items():
        m.forward = (lambda k, f: lambda x: (rows[k].append(x.shape[0]), f(x))[1])(k, m.forward)
    acc = model.conv_layers[0].accumulate_group

    def count(*a, **kw):
        rows['shared'] += 1
        return acc(*a, **kw)
    model.conv_layers[0].accumulate_group = count
    try:
        shared = _scores(model, _timed(g, 0.5))
    finally:
        for m in enc.values():
            del m.forward
        del model.conv_layers[0].accumulate_group
    assert rows['rec'] == [sum(n_res)] and rows['atom'] == [sum(n_atom)]    # one call over the two distinct receptors
    assert rows['shared'] == 4                         # the four static groups of layer 0, once for both receptors
    unshared = _scores(model, _timed(collate_packed(cx, DEV), 0.5, uniform=False))   # no uniform-time promise
    for a, b in zip(shared, unshared):
        assert rel_err(a, b) < 1e-5


# ---------------------------------------------------------------------------------------------------------------------
# sampler
def _run_both(model, args, cx, steps=6, max_pairs=None, **kw):
    """Largest |difference| of the final coordinates: sample_packed against one sampling() call per complex."""
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sample_packed, sampling
    sched = get_t_schedule('expbeta', steps)
    t2s = partial(t_to_sigma, args=args)
    ids = [5, 9, 2]
    packed = sample_packed([[d.clone() for d in p] for p in cx], model, steps, sched, sched, sched, DEV, t2s, args, seed=11,
                           complex_ids=ids[:len(cx)], no_final_step_noise=True, max_pairs=max_pairs, **kw)
    alone = [sampling([d.clone() for d in p], model, steps, sched, sched, sched, DEV, t2s, args, batch_size=len(p),
                      no_final_step_noise=True, rng='philox', seed=11, pose_keys=(cid << 32) + torch.arange(len(p)), **kw)
             for cid, p in zip(ids, cx)]
    torch.cuda.synchronize()
    d = 0.0
    for (pl, _), (al, _) in zip(packed, alone):
        a = torch.stack([x['ligand'].pos for x in pl]).cpu()
        b = torch.stack([x['ligand'].pos for x in al]).cpu()
        assert torch.isfinite(a).all()
        d = max(d, float((a - b).abs().max()))
    return d


@pytest.mark.parametrize("cuda_graph", [True, False])
def test_sample_packed_matches_sampling_per_complex(built_lib, cuda_graph):
    model, args = _aa_model(False)
    assert _run_both(model, args, _complexes(), cuda_graph=cuda_graph) < 2e-3


def test_sample_packed_budget_counts_receptor_atoms(built_lib, monkeypatch):
    from diffdock_b200 import sampling as smod
    model, args = _aa_model(False)
    cx = _complexes()
    residues_only = [smod.pack_cost(p) for p in cx]
    assert smod.pack_plan(residues_only, sum(residues_only)) == [[0, 1, 2]]
    packs = []
    orig = smod.collate_packed
    monkeypatch.setattr(smod, 'collate_packed', lambda c, *a, **k: (packs.append(len(c)), orig(c, *a, **k))[1])
    # the residue-only cost of all three complexes: with their receptor atoms each one needs a pack of its own
    assert _run_both(model, args, cx, max_pairs=sum(residues_only)) < 2e-3
    assert packs == [1, 1, 1]


def test_packed_graphed_all_atom_step_is_sync_free(built_lib):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.hetero import collate_packed
    from diffdock_b200.sampling import GraphedSteps, _step_tables
    model, args = _aa_model(False)
    g = collate_packed(_complexes(), DEV)
    g._pose_err = torch.zeros(1, dtype=torch.int32, device=DEV)
    sched = get_t_schedule('expbeta', 6)
    coef, t_rows = _step_tables(6, sched, sched, sched, partial(t_to_sigma, args=args), args, False, False, True, 1.0, 0.0,
                                0.5)
    keys = torch.arange(g.num_graphs, device=DEV)
    steps = GraphedSteps(model, g, g.num_graphs, coef, t_rows, None, None, None, True, DEV, draw_noise=True,
                         philox=(3, keys), packed=True)
    assert 'shared_static' in g['receptor', 'receptor']._b200aa      # the step shares layer-0 receptor messages
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        steps.run(6)
        done = steps.step.clone()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert int(done.item()) == 6 and torch.isfinite(steps.pos).all() and int(g._pose_err.item()) == 0


def test_sample_packed_refuses_cropping_all_atom_receptors(built_lib):
    from diffdock_b200.sampling import sample_packed
    model, args = _aa_model(False)
    args = copy.copy(args)
    args.crop_beyond = 20.0
    with pytest.raises(NotImplementedError):
        sample_packed(_complexes(), model, 2, [1.0, 0.5], [1.0, 0.5], [1.0, 0.5], DEV, None, args, seed=0)

"""GPU: score models built with ``reduce_pseudoscalars`` (the DiffDock-L flag set) on the fused convolution kernel and the
captured sampler step.  The kernel's two consumer kinds for the ``nv x0o`` block - (10, 1) and (4, 1) - against the float64
reference of tests/parity_helpers.py:fused_conv_reference per output irrep block (3e-5, as in test_fused_conv_fp64_gpu.py),
with two mutations that the comparison must catch; the product against the unmodified reference
(tests/golden/ref_cg_model_l.pt) and the CPU oracle; the captured sampler, with and without per-step cropping, against the
eager one; and the all-atom model with the same flag."""
import copy
from functools import partial

import pytest
import torch

from tests.parity_helpers import block_errors, rand_bn_, rel_err
from tests.test_fused_conv_cta128_gpu import _runs, _sms
from tests.test_fused_conv_fp64_gpu import TOL, Case, _check
from tests.test_reduce_pseudoscalars_cpu import _layer_tables, fixture, l_model

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
# the DiffDock-L flag set (tests/golden/make_golden_get_model.py, "DiffDock-L score yml")
L_FLAGS = dict(sh_lmax=1, num_prot_emb_layers=3, reduce_pseudoscalars=True, embed_also_ligand=True, smooth_edges=True,
               odd_parity=True)


def l_pair(args, seed=0, lm=True):
    """(oracle CGModel on CPU, product CGModel on cuda:0) sharing one random state_dict, BatchNorm statistics randomised;
    unlike tests/parity_helpers.py:make_model_pair it passes ``odd_parity``."""
    from oracle.cg_model import CGModel as OModel
    from oracle.diffusion import t_to_sigma as o_t2s
    from oracle.layers import get_timestep_embedding as o_emb
    from diffdock_b200.cg_model import CGModel as PModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding as p_emb, t_to_sigma as p_t2s
    kw = dict(sigma_embed_dim=args.sigma_embed_dim, sh_lmax=args.sh_lmax, ns=args.ns, nv=args.nv,
              num_conv_layers=args.num_conv_layers, lig_max_radius=args.max_radius, rec_max_radius=args.rec_max_radius,
              cross_max_distance=args.cross_max_distance, center_max_distance=args.center_max_distance,
              distance_embed_dim=args.distance_embed_dim, cross_distance_embed_dim=args.cross_distance_embed_dim,
              dynamic_max_cross=args.dynamic_max_cross, lm_embedding_type='precomputed' if lm else None,
              embed_also_ligand=args.embed_also_ligand, num_prot_emb_layers=args.num_prot_emb_layers,
              no_torsion=args.no_torsion, smooth_edges=args.smooth_edges, odd_parity=args.odd_parity,
              reduce_pseudoscalars=args.reduce_pseudoscalars, differentiate_convolutions=args.differentiate_convolutions)
    torch.manual_seed(seed)
    o = OModel(partial(o_t2s, args=args), 'cpu', o_emb('sinusoidal', args.sigma_embed_dim, args.embedding_scale), **kw).eval()
    gen = torch.Generator().manual_seed(seed + 1)
    for m in o.modules():
        if m.__class__.__name__ == 'BatchNorm':
            rand_bn_(m, gen)
    p = PModel(partial(p_t2s, args=args), torch.device(DEV), p_emb('sinusoidal', args.sigma_embed_dim, args.embedding_scale),
               **kw).eval()
    p.load_state_dict(o.state_dict(), strict=True)
    return o, p.to(DEV)


def l_args(**over):
    from diffdock_b200.synthetic import default_model_args
    kw = dict(L_FLAGS, ns=48, nv=10, num_conv_layers=4, distance_embed_dim=32, cross_distance_embed_dim=32,
              sigma_embed_dim=32)
    kw.update(over)
    return default_model_args(**kw)


def _oracle_scores(o, poses, t):
    from diffdock_b200.hetero import collate
    from oracle.diffusion import set_time
    g = collate(copy.deepcopy(poses))
    set_time(g, t, t, t, len(poses), 'cpu')
    with torch.no_grad():
        return o(g)


def _product_scores(p, poses, t):
    from diffdock_b200.diffusion_utils import set_time
    from diffdock_b200.hetero import collate
    g = collate(copy.deepcopy(poses)).to(DEV)
    set_time(g, None, t, t, t, len(poses), False, DEV)
    out = p(g)
    torch.cuda.synchronize()
    return out


def _assert_close(got, ref, tol):
    for a, b in zip(got[:3], ref[:3]):
        assert a.shape == b.shape
        if b.numel():
            assert rel_err(a, b) < tol, rel_err(a, b)


# ------------------------------------------------------------------------------------------------------------ kernel
EDGES = {'127': lambda s: 127, '128': lambda s: 128, '129': lambda s: 129, 'sms*128-1': lambda s: s * 128 - 1,
         'sms*128+1': lambda s: s * 128 + 1, 'sms*128+64': lambda s: s * 128 + 64,
         '2*sms*128+57': lambda s: 2 * s * 128 + 57}


@pytest.mark.parametrize('edges', list(EDGES))
@pytest.mark.parametrize('stage', [2, 3])
@pytest.mark.parametrize('lmax', [1, 2])
@pytest.mark.parametrize('ns,nv', [(48, 10), (16, 4)])
def test_kernel_nv_0o_layers_match_fp64(built_lib, ns, nv, lmax, stage, edges):
    table = _layer_tables(ns, nv, lmax)[stage - 2]
    c = Case(table, ns, ns, 3 * ns, EDGES[edges](_sms()), seed=700 + 10 * stage + lmax + ns, n_nodes=400)
    assert any(t[0] == {10: 4, 4: 5}[nv] for t in c.plan.tiles.tolist())
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f'nv x0o ns={ns} lmax={lmax} stage={stage} E={c.E}')


@pytest.mark.parametrize('lmax', [1, 2])
@pytest.mark.parametrize('ns,nv', [(48, 10), (16, 4)])
def test_kernel_nv_0o_csr_runs_across_tiles(built_lib, ns, nv, lmax):
    E = 3 * _sms() * 128 + 17
    tgt, n_out = _runs(E, torch.Generator().manual_seed(lmax + ns))
    c = Case(_layer_tables(ns, nv, lmax)[1], ns, ns, 3 * ns, E, seed=800 + lmax + ns, n_nodes=max(500, n_out),
             n_out=n_out)
    c.tgt = tgt.cuda()
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f'nv x0o runs ns={ns} lmax={lmax}')


def _mutated_errors(mutate):
    """Block errors of the (10, 1) layer (ns=48, nv=10, lmax 1, stage 3) run with a plan changed by ``mutate(case)``."""
    from diffdock_b200 import fused
    table = _layer_tables(48, 10, 1)[1]
    c = Case(table, 48, 48, 144, 2 * _sms() * 128 + 57, seed=901, n_nodes=400)
    ref, _ = c.reference()
    got, _ = c.run()
    assert max(block_errors(got, ref, table.out_irreps).values()) < TOL
    plan = mutate(c, fused)
    got, _ = c.run(plan=plan)
    return block_errors(got, ref, table.out_irreps)


def _odd_paths(table):
    paths = sorted(table.paths, key=lambda p: (p.i_out, p.w_ref_off))
    return paths, [i for i, p in enumerate(paths) if (p.mul_out, 2 * p.l_out + 1) == (10, 1)]


def test_comparison_catches_a_wrong_channel_map_in_the_10x1_flush(built_lib):
    """The (10, 1) tiles' output channels rotated by one (as a flush writing channel w to w + 1 would): built by rotating
    the channels of the weight rows of every path into 10x0o."""
    def rotate(c, fused):
        w1, b1, w2, b2 = c.w
        rows = torch.arange(w2.shape[0], device=w2.device)
        paths, odd = _odd_paths(c.table)
        for i in odd:
            p = paths[i]
            blk = rows[p.w_ref_off:p.w_ref_off + p.mul_in * 10].view(p.mul_in, 10)
            rows[p.w_ref_off:p.w_ref_off + p.mul_in * 10] = blk.roll(1, dims=1).reshape(-1)
        return fused.FusedPlan(c.table, w1, b1, w2[rows], b2[rows])
    errs = _mutated_errors(rotate)
    odd = [k for k in errs if k.startswith('10x0o')]
    assert odd and all(errs[k] > 100 * TOL for k in odd), errs
    assert all(v < TOL for k, v in errs.items() if k not in odd), errs


def test_comparison_catches_a_wrong_cg_row_for_a_path_into_0o(built_lib):
    """The dense Clebsch-Gordan table of the 1e x 1o -> 0o path with two input rows swapped."""
    def swap_rows(c, fused):
        plan = fused.FusedPlan(c.table, *c.w)
        paths, odd = _odd_paths(c.table)
        i = next(i for i in odd if paths[i].l_in == 1)
        m = plan.mtab[i, :45].view(3, 3, 5)
        m[[0, 1]] = m[[1, 0]].clone()
        return plan
    errs = _mutated_errors(swap_rows)
    odd = [k for k in errs if k.startswith('10x0o')]
    assert odd and all(errs[k] > 100 * TOL for k in odd), errs


# ------------------------------------------------------------------------------------------------------------ model
@pytest.mark.parametrize('i', range(3))
def test_product_matches_reference_fixture(built_lib, i):
    case = fixture()['cases'][i]
    m, poses, _ = l_model(case, 'product')
    assert m.sync_free_capable() and m.sync_free_crop_capable()
    got = _product_scores(m, poses, case['t'])
    _assert_close(got, (case['tr'], case['rot'], case['tor']), 1e-4)


@pytest.fixture(scope='module')
def l_model_pair(built_lib):
    args = l_args()
    o, p = l_pair(args, seed=5)
    assert p.sync_free_capable() and p.sync_free_crop_capable()
    return o, p, args


@pytest.mark.parametrize('t', [0.3, 0.8])
def test_sync_free_matches_host_sized_and_oracle(l_model_pair, t):
    from diffdock_b200.synthetic import make_pose_list
    o, p, args = l_model_pair
    poses = make_pose_list(2, n_res=90, n_atoms=15, seed=21, tr_sigma_max=args.tr_sigma_max * t)
    got = _product_scores(p, poses, t)
    host = copy.deepcopy(p)
    host._sync_free = False                           # the exactly-sized path with host-side counts
    _assert_close(got, _product_scores(host, poses, t), 1e-4)
    _assert_close(got, _oracle_scores(o, poses, t), 1e-4)


def test_several_full_size_poses_through_the_samplers_collate(l_model_pair):
    """Three 1500-residue / 40-atom poses of one complex in one batch, collated as sampling() collates them (one receptor
    copy, shared layer-0 receptor messages): the sync-free forward against the host-sized one, and the general collate
    against the CPU oracle.  The ligand folds past radius_graph's cap of 32 neighbours (tests/test_ligand_graph_cap_gpu.py)."""
    from diffdock_b200.diffusion_utils import set_time
    from diffdock_b200.hetero import collate_shared_receptor
    from diffdock_b200.synthetic import make_pose_list
    o, p, args = l_model_pair
    host = copy.deepcopy(p)
    host._sync_free = False
    t = 0.5
    poses = make_pose_list(3, n_res=1500, n_atoms=40, seed=100, tr_sigma_max=args.tr_sigma_max * t)
    outs = []
    for m in (p, host):
        g = collate_shared_receptor([q.clone() for q in poses], DEV)
        set_time(g, None, t, t, t, 3, False, DEV)
        g._uniform_t = True
        outs.append(m(g))
    torch.cuda.synchronize()
    _assert_close(outs[0], outs[1], 1e-4)
    torch.set_num_threads(min(torch.get_num_threads(), 32))
    _assert_close(_product_scores(p, poses, t), _oracle_scores(o, poses, t), 1e-4)


def test_one_full_size_pose_matches_oracle(built_lib):
    """The 1500-residue / 40-atom complex of config 3 with the DiffDock-L flag set at ns=48, nv=10, six layers."""
    from diffdock_b200.synthetic import make_pose_list
    args = l_args(num_conv_layers=6, distance_embed_dim=64, cross_distance_embed_dim=64, sigma_embed_dim=64)
    o, p = l_pair(args, seed=0)
    assert p.sync_free_capable()
    t = 0.5
    poses = make_pose_list(1, n_res=1500, n_atoms=40, seed=100, tr_sigma_max=args.tr_sigma_max * t)
    torch.set_num_threads(min(torch.get_num_threads(), 32))
    _assert_close(_product_scores(p, poses, t), _oracle_scores(o, poses, t), 1e-4)


def _sample(p, args, poses, crop_beyond=None, steps=6, **kw):
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sampling
    a = copy.copy(args)
    a.crop_beyond = crop_beyond
    sched = get_t_schedule('expbeta', steps)
    out, _ = sampling([q.clone() for q in poses], p, steps, sched, sched, sched, DEV, partial(t_to_sigma, args=a), a,
                      batch_size=len(poses), no_final_step_noise=True, **kw)
    torch.cuda.synchronize()
    return torch.stack([d['ligand'].pos for d in out]).cpu()


@pytest.mark.parametrize('crop_beyond', [None, 20.0])
def test_captured_sampler_matches_eager(l_model_pair, monkeypatch, crop_beyond):
    from diffdock_b200 import sampling as smod
    from diffdock_b200.synthetic import make_pose_list
    _, p, args = l_model_pair
    args = copy.copy(args)
    args.tr_sigma_max = 5.0        # every ligand stays within reach of some residue: the eager crop needs one
    poses = make_pose_list(4, n_res=120, n_atoms=12, seed=41, tr_sigma_max=args.tr_sigma_max)
    made = []

    class Recorder(smod.GraphedSteps):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)

    monkeypatch.setattr(smod, 'GraphedSteps', Recorder)
    graphed = _sample(p, args, poses, crop_beyond, rng='philox', seed=123, cuda_graph=True)
    assert len(made) == 1 and (made[0].crop is not None) == (crop_beyond is not None)
    eager = _sample(p, args, poses, crop_beyond, rng='philox', seed=123, cuda_graph=False)
    assert len(made) == 1
    assert torch.isfinite(graphed).all()
    assert float((eager - graphed).abs().max()) < 2e-3      # 6 chained steps; scatter order differs run to run


def test_cropped_sampling_reproduces_reference_fixture(built_lib):
    from diffdock_b200.diffusion_utils import t_to_sigma
    from diffdock_b200.sampling import sampling
    f = fixture()
    s = f['sampling']
    m, poses, a = l_model(f['cases'][s['model_case']], 'product')
    a.crop_beyond = s['crop_beyond']
    torch.manual_seed(s['seed'])
    noise = lambda kind, shape: torch.normal(mean=0, std=1, size=shape)
    out, _ = sampling(copy.deepcopy(poses), m, s['steps'], s['schedule'], s['schedule'], s['schedule'], DEV,
                      partial(t_to_sigma, args=a), a, batch_size=3, no_final_step_noise=True,
                      temp_sampling=s['temp_sampling'], temp_psi=s['temp_psi'], temp_sigma_data=s['temp_sigma_data'],
                      noise_fn=noise)
    for d, ref in zip(out, s['final_pos']):
        assert rel_err(d['ligand'].pos, ref) < 1e-4


def test_graphed_cropped_step_is_sync_free(l_model_pair):
    import numpy as np
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.hetero import collate_shared_receptor
    from diffdock_b200.sampling import GraphedSteps, crop_cutoff2, step_coefficients
    from diffdock_b200.synthetic import make_pose_list
    _, p, args = l_model_pair
    n = 4
    poses = make_pose_list(n, n_res=120, n_atoms=12, seed=71, tr_sigma_max=args.tr_sigma_max)
    g = collate_shared_receptor(poses, DEV)
    sched = get_t_schedule('expbeta', 6)
    t2s = partial(t_to_sigma, args=args)
    coef = [step_coefficients(i, 6, sched, sched, sched, t2s, args, False, 1.0, 0.0, 0.5) for i in range(6)]
    lig0 = poses[0]['ligand']
    rb = poses[0]['ligand', 'ligand'].edge_index.T[lig0.edge_mask]
    bu, bv = rb[:, 0].int().contiguous().to(DEV), rb[:, 1].int().contiguous().to(DEV)
    mask = torch.from_numpy(lig0.mask_rotate[0].astype(np.uint8)).to(DEV)
    steps = GraphedSteps(p, g, n, coef, [[float(t)] * 3 for t in sched], bu, bv, mask, True, DEV, draw_noise=True,
                         philox=(3, torch.arange(n, device=DEV)),
                         crop_rows=[crop_cutoff2(t2s, t, t, t, 20.0) for t in sched])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        steps.run(6)
        done = steps.step.clone()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert int(done.item()) == 6 and torch.isfinite(steps.pos).all()


def test_all_atom_model_with_reduce_pseudoscalars_matches_oracle(built_lib):
    from oracle.aa_model import AAModel as OModel
    from oracle.diffusion import set_time as o_set_time, t_to_sigma as o_t2s
    from oracle.layers import get_timestep_embedding as o_temb
    from diffdock_b200.aa_model import AAModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, set_time, t_to_sigma
    from diffdock_b200.hetero import collate
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    a = default_model_args(num_conv_layers=3, distance_embed_dim=16, cross_distance_embed_dim=16, sigma_embed_dim=16)
    kw = dict(sigma_embed_dim=16, sh_lmax=2, ns=48, nv=10, num_conv_layers=3, lig_max_radius=a.max_radius,
              rec_max_radius=a.rec_max_radius, cross_max_distance=a.cross_max_distance, center_max_distance=a.center_max_distance,
              distance_embed_dim=16, cross_distance_embed_dim=16, dynamic_max_cross=True, lm_embedding_type=None,
              embed_also_ligand=True, reduce_pseudoscalars=True, odd_parity=True)
    torch.manual_seed(23)
    mo = OModel(partial(o_t2s, args=a), 'cpu', o_temb('sinusoidal', 16, a.embedding_scale), **kw).eval()
    g = torch.Generator().manual_seed(24)
    for mod in mo.modules():
        if mod.__class__.__name__ == 'BatchNorm':
            rand_bn_(mod, g)
    mp = AAModel(partial(t_to_sigma, args=a), torch.device(DEV), get_timestep_embedding('sinusoidal', 16, a.embedding_scale),
                 **kw).eval()
    mp.load_state_dict(mo.state_dict(), strict=True)
    mp = mp.to(DEV)
    assert mp.sync_free_capable()
    poses = make_pose_list(2, n_res=40, n_atoms=12, seed=93, tr_sigma_max=a.tr_sigma_max * 0.3, lm_dim=0, all_atoms=True)
    t = 0.3
    b = collate(copy.deepcopy(poses))
    o_set_time(b, t, t, t, 2, 'cpu', all_atoms=True)
    with torch.no_grad():
        ref = mo(b)
    bg = collate(copy.deepcopy(poses)).to(DEV)
    set_time(bg, None, t, t, t, 2, True, DEV)
    _assert_close(mp(bg), ref, 1e-4)

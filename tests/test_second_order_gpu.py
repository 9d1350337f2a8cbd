"""GPU: score models built with ``use_second_order_repr`` on the fused convolution kernel's second-order instantiation and
the captured sampler step.  Every second-order layer against the float64 reference of
tests/parity_helpers.py:fused_conv_reference per output irrep block (3e-5, as in test_fused_conv_fp64_gpu.py), with the
indirections the models use and two mutations that the comparison must catch; the product against the CPU oracle (and the
unmodified reference, tests/golden/ref_cg_model_so.pt); the captured sampler, with and without per-step cropping, against
the eager one; and the all-atom model with the same flag."""
import copy
from functools import partial

import pytest
import torch

from tests.parity_helpers import block_errors, rand_bn_, rel_err
from tests.test_fused_conv_cta128_gpu import _runs, _sms
from tests.test_fused_conv_fp64_gpu import TOL, Case, _check
from tests.test_reduce_pseudoscalars_gpu import _assert_close, _oracle_scores, _product_scores, _sample
from tests.test_reduce_pseudoscalars_cpu import l_model
from tests.test_second_order_cpu import WIDTHS, fixture, so_tables

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def so_pair(args, seed=0, model='cg'):
    """(oracle model on CPU, product model on cuda:0) with ``use_second_order_repr`` sharing one random state_dict,
    BatchNorm statistics randomised."""
    from diffdock_b200.diffusion_utils import get_timestep_embedding as p_emb, t_to_sigma as p_t2s
    from oracle.diffusion import t_to_sigma as o_t2s
    from oracle.layers import get_timestep_embedding as o_emb
    if model == 'cg':
        from diffdock_b200.cg_model import CGModel as PModel
        from oracle.cg_model import CGModel as OModel
    else:
        from diffdock_b200.aa_model import AAModel as PModel
        from oracle.aa_model import AAModel as OModel
    kw = dict(sigma_embed_dim=args.sigma_embed_dim, sh_lmax=args.sh_lmax, ns=args.ns, nv=args.nv,
              num_conv_layers=args.num_conv_layers, lig_max_radius=args.max_radius, rec_max_radius=args.rec_max_radius,
              cross_max_distance=args.cross_max_distance, center_max_distance=args.center_max_distance,
              distance_embed_dim=args.distance_embed_dim, cross_distance_embed_dim=args.cross_distance_embed_dim,
              dynamic_max_cross=args.dynamic_max_cross, lm_embedding_type=None, embed_also_ligand=args.embed_also_ligand,
              num_prot_emb_layers=args.num_prot_emb_layers, no_torsion=args.no_torsion, use_second_order_repr=True)
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


def so_args(**over):
    from diffdock_b200.synthetic import default_model_args
    kw = dict(ns=48, nv=10, sh_lmax=2, num_conv_layers=4, distance_embed_dim=32, cross_distance_embed_dim=32,
              sigma_embed_dim=32, use_second_order_repr=True, embed_also_ligand=True)
    kw.update(over)
    return default_model_args(**kw)


# ------------------------------------------------------------------------------------------------------------ kernel
EDGES = {'127': lambda s: 127, '129': lambda s: 129, 'sms*128-1': lambda s: s * 128 - 1,
         'sms*128+64': lambda s: s * 128 + 64, '2*sms*128+57': lambda s: 2 * s * 128 + 57}


@pytest.mark.parametrize('edges', list(EDGES))
@pytest.mark.parametrize('stage', range(4))
@pytest.mark.parametrize('lmax', [1, 2])
@pytest.mark.parametrize('ns,nv', WIDTHS)
def test_kernel_second_order_layers_match_fp64(built_lib, ns, nv, lmax, stage, edges):
    table = so_tables(ns, nv, lmax)[stage]
    c = Case(table, ns, ns, 3 * ns, EDGES[edges](_sms()), seed=1700 + 10 * stage + lmax + ns, n_nodes=400)
    assert c.plan.second_order == (stage > 0 or lmax == 2)
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f'second order ns={ns} lmax={lmax} stage={stage} E={c.E}')


@pytest.mark.parametrize('lmax', [1, 2])
@pytest.mark.parametrize('ns,nv', WIDTHS)
def test_kernel_second_order_csr_runs_across_tiles(built_lib, ns, nv, lmax):
    E = 3 * _sms() * 128 + 17
    tgt, n_out = _runs(E, torch.Generator().manual_seed(lmax + ns))
    c = Case(so_tables(ns, nv, lmax)[3], ns, ns, 3 * ns, E, seed=1800 + lmax + ns, n_nodes=max(500, n_out), n_out=n_out)
    c.tgt = tgt.cuda()
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f'second order runs ns={ns} lmax={lmax}')


@pytest.mark.parametrize('ns,nv', WIDTHS)
def test_kernel_second_order_indirections(built_lib, ns, nv):
    """edge_perm into a larger store, vec_sign = -1, ea_add, edge_weight and a device-side live count together."""
    table = so_tables(ns, nv, 2)[3]
    E = 2 * _sms() * 128 + 57
    rows = 2 * E
    c = Case(table, ns, ns, 3 * ns, E, seed=1900 + ns, rows=rows, n_nodes=400)
    g = c.gen
    n_live = E - 2 * 64 - 5
    c.tgt[n_live:] = 0
    c.kw = dict(edge_perm=torch.randperm(rows, generator=g)[:E].int().cuda(), vec_sign=-1.0,
                ea_add=torch.randn(7, ns, generator=g).cuda(), ea_add_idx=torch.randint(0, 7, (E,), generator=g).int().cuda(),
                edge_weight=torch.rand(rows, generator=g).cuda(),
                n_edges_dev=torch.tensor([n_live], dtype=torch.int32, device='cuda'))
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(n_live), f'second order indirections ns={ns}')


def _mutated_errors(mutate):
    """Block errors of the last second-order layer (ns=48, nv=10, lmax 2) run with a plan changed by ``mutate(case)``."""
    from diffdock_b200 import fused
    table = so_tables(48, 10, 2)[3]
    c = Case(table, 48, 48, 144, 2 * _sms() * 128 + 57, seed=1901, n_nodes=400)
    ref, _ = c.reference()
    got, _ = c.run()
    assert max(block_errors(got, ref, table.out_irreps).values()) < TOL
    plan = mutate(c, fused)
    got, _ = c.run(plan=plan)
    return block_errors(got, ref, table.out_irreps)


def _paths(table):
    return sorted(table.paths, key=lambda p: (p.i_out, p.w_ref_off))


def test_comparison_catches_a_wrong_channel_map_in_the_10x5_flush(built_lib):
    """The (10, 5) tiles' output channels rotated by one (as a flush writing channel w to w + 1 would): built by rotating
    the channels of the weight rows of every path into an l = 2 block."""
    def rotate(c, fused):
        w1, b1, w2, b2 = c.w
        rows = torch.arange(w2.shape[0], device=w2.device)
        for p in _paths(c.table):
            if p.l_out == 2:
                blk = rows[p.w_ref_off:p.w_ref_off + p.mul_in * 10].view(p.mul_in, 10)
                rows[p.w_ref_off:p.w_ref_off + p.mul_in * 10] = blk.roll(1, dims=1).reshape(-1)
        return fused.FusedPlan(c.table, w1, b1, w2[rows], b2[rows])
    errs = _mutated_errors(rotate)
    l2 = [k for k in errs if k.startswith('10x2')]
    assert len(l2) == 2 and all(errs[k] > 100 * TOL for k in l2), errs
    assert all(v < TOL for k, v in errs.items() if k not in l2), errs


def test_comparison_catches_a_wrong_cg_row_for_a_2x2_path(built_lib):
    """The dense Clebsch-Gordan table of the 2e x 2e -> 2e path with two input rows swapped."""
    def swap_rows(c, fused):
        plan = fused.FusedPlan(c.table, *c.w)
        paths = _paths(c.table)
        i = next(i for i, p in enumerate(paths) if p.l_in == 2 and p.l_sh == 2 and p.l_out == 2)
        m = plan.mtab[i, :125].view(5, 5, 5)
        m[[0, 3]] = m[[3, 0]].clone()
        return plan
    errs = _mutated_errors(swap_rows)
    assert max(errs.values()) > 100 * TOL, errs


# ------------------------------------------------------------------------------------------------------------ model
@pytest.mark.parametrize('i', range(3))
def test_product_matches_reference_fixture(built_lib, i):
    case = fixture()['cases'][i]
    m, poses, _ = l_model(case, 'product')
    assert m.sync_free_capable() and m.sync_free_crop_capable()
    got = _product_scores(m, poses, case['t'])
    _assert_close(got, (case['tr'], case['rot'], case['tor']), 1e-4)


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


@pytest.fixture(scope='module')
def so_model_pair(built_lib):
    args = so_args()
    o, p = so_pair(args, seed=5)
    assert p.sync_free_capable() and p.sync_free_crop_capable()
    return o, p, args


@pytest.mark.parametrize('t', [0.3, 0.8])
def test_sync_free_matches_host_sized_and_oracle(so_model_pair, t):
    from diffdock_b200.synthetic import make_pose_list
    o, p, args = so_model_pair
    poses = make_pose_list(2, n_res=90, n_atoms=15, seed=21, tr_sigma_max=args.tr_sigma_max * t, lm_dim=0)
    got = _product_scores(p, poses, t)
    host = copy.deepcopy(p)
    host._sync_free = False                           # the exactly-sized path with host-side counts
    _assert_close(got, _product_scores(host, poses, t), 1e-4)
    _assert_close(got, _oracle_scores(o, poses, t), 1e-4)


def test_small_widths_match_oracle(built_lib):
    """ns=16, nv=4 at sh_lmax 1 and 2: the (4, 5) kind through the whole model."""
    from diffdock_b200.synthetic import make_pose_list
    for lmax in (1, 2):
        args = so_args(ns=16, nv=4, sh_lmax=lmax, distance_embed_dim=16, cross_distance_embed_dim=16, sigma_embed_dim=16)
        o, p = so_pair(args, seed=7 + lmax)
        assert p.sync_free_capable()
        poses = make_pose_list(2, n_res=90, n_atoms=15, seed=22, tr_sigma_max=args.tr_sigma_max * 0.4, lm_dim=0)
        _assert_close(_product_scores(p, poses, 0.4), _oracle_scores(o, poses, 0.4), 1e-4)


def test_one_full_size_pose_matches_oracle(built_lib):
    """The 1500-residue / 40-atom complex of config 3, second order at ns=48, nv=10, six layers."""
    from diffdock_b200.synthetic import make_pose_list
    args = so_args(num_conv_layers=6, distance_embed_dim=64, cross_distance_embed_dim=64, sigma_embed_dim=64)
    o, p = so_pair(args, seed=0)
    assert p.sync_free_capable()
    t = 0.5
    poses = make_pose_list(1, n_res=1500, n_atoms=40, seed=100, tr_sigma_max=args.tr_sigma_max * t, lm_dim=0)
    torch.set_num_threads(min(torch.get_num_threads(), 32))
    _assert_close(_product_scores(p, poses, t), _oracle_scores(o, poses, t), 1e-4)


@pytest.mark.parametrize('crop_beyond', [None, 20.0])
def test_captured_sampler_matches_eager(so_model_pair, monkeypatch, crop_beyond):
    from diffdock_b200 import sampling as smod
    from diffdock_b200.synthetic import make_pose_list
    _, p, args = so_model_pair
    args = copy.copy(args)
    args.tr_sigma_max = 5.0        # every ligand stays within reach of some residue: the eager crop needs one
    poses = make_pose_list(4, n_res=120, n_atoms=12, seed=41, tr_sigma_max=args.tr_sigma_max, lm_dim=0)
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


def test_graphed_cropped_step_is_sync_free(so_model_pair):
    import numpy as np
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.hetero import collate_shared_receptor
    from diffdock_b200.sampling import GraphedSteps, crop_cutoff2, step_coefficients
    from diffdock_b200.synthetic import make_pose_list
    _, p, args = so_model_pair
    n = 4
    poses = make_pose_list(n, n_res=120, n_atoms=12, seed=71, tr_sigma_max=args.tr_sigma_max, lm_dim=0)
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


def test_all_atom_model_with_second_order_repr_matches_oracle(built_lib):
    from diffdock_b200.diffusion_utils import set_time
    from diffdock_b200.hetero import collate
    from diffdock_b200.synthetic import make_pose_list
    from oracle.diffusion import set_time as o_set_time
    a = so_args(num_conv_layers=3, distance_embed_dim=16, cross_distance_embed_dim=16, sigma_embed_dim=16)
    mo, mp = so_pair(a, seed=23, model='aa')
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

"""GPU: score models built with ``tp_weights_layers`` > 2 on the fused convolution kernel and the captured sampler step.
The kernel with the extra H x H hidden layers against the float64 reference of tests/test_tp_weights_layers_cpu.py per
output irrep block (3e-5, as in test_fused_conv_fp64_gpu.py), with the indirections the models use and two mutations that
the comparison must catch; the product against the unmodified reference (tests/golden/ref_cg_model_tw.pt) and the CPU
oracle; the captured sampler, with and without per-step cropping, against the eager one; and the all-atom model."""
import copy
from functools import partial

import pytest
import torch

from tests.parity_helpers import block_errors, fused_table, rand_bn_, rel_err
from tests.test_fused_conv_cta128_gpu import _runs, _sms
from tests.test_fused_conv_fp64_gpu import TOL, Case, _check
from tests.test_reduce_pseudoscalars_gpu import _assert_close, _oracle_scores, _product_scores, _sample
from tests.test_second_order_cpu import so_tables
from tests.test_tp_weights_layers_cpu import WIDTHS, fixture, fused_conv_reference_deep, hidden_weights, tw_model

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


class DeepCase(Case):
    """A fused-convolution launch whose FCBlock has ``layers`` - 2 extra H x H hidden layers."""

    def __init__(self, table, ne, ns, H, E, seed, layers, **kw):
        from diffdock_b200 import fused
        super().__init__(table, ne, ns, H, E, seed, **kw)
        self.hidden = [(w.cuda(), b.cuda()) for w, b in hidden_weights(H, layers - 2, self.gen)]
        self.plan = fused.FusedPlan(table, *self.w, hidden=self.hidden)

    def reference(self, n_live=None, hidden=None):
        n = self.E if n_live is None else n_live
        kw = {k: v for k, v in self.kw.items() if k not in ('n_edges_dev', 'edge_weight')}
        for k in ('edge_perm', 'ea_add_idx'):
            if k in kw:
                kw[k] = kw[k][:n]
        w1, b1, w2, b2 = self.w
        return fused_conv_reference_deep(self.table, w1, b1, self.hidden if hidden is None else hidden, w2, b2, self.ea,
                                         self.node, self.ns, self.tgt[:n], self.src[:n], self.x, self.vec, self.n_out,
                                         ew=self.kw.get('edge_weight'), **kw)


# ------------------------------------------------------------------------------------------------------------ kernel
EDGES = {'127': lambda s: 127, 'sms*128-1': lambda s: s * 128 - 1, 'sms*128+64': lambda s: s * 128 + 64,
         '2*sms*128+57': lambda s: 2 * s * 128 + 57}


@pytest.mark.parametrize('edges', list(EDGES))
@pytest.mark.parametrize('lmax', [1, 2])
@pytest.mark.parametrize('ns,nv', WIDTHS)
@pytest.mark.parametrize('layers', [3, 4])
def test_kernel_deep_mlp_matches_fp64(built_lib, layers, ns, nv, lmax, edges):
    """The last conv stage (every first-order consumer kind of the width) at the production (ne, ns, H)."""
    table = fused_table(ns, nv, 3, lmax, False)
    c = DeepCase(table, ns, ns, 3 * ns, EDGES[edges](_sms()), seed=2100 + 10 * layers + lmax + ns, layers=layers,
                 n_nodes=400)
    assert c.plan.n_hidden == layers - 2 and not c.plan.second_order
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f'tp_weights_layers={layers} ns={ns} lmax={lmax} E={c.E}')


@pytest.mark.parametrize('stage', [1, 2])
@pytest.mark.parametrize('ns,nv', WIDTHS)
@pytest.mark.parametrize('layers', [3, 4])
def test_kernel_deep_mlp_second_order_matches_fp64(built_lib, layers, ns, nv, stage):
    """The second-order instantiation (use_second_order_repr) with the hidden stack."""
    table = so_tables(ns, nv, 2)[stage]
    c = DeepCase(table, ns, ns, 3 * ns, 2 * _sms() * 128 + 57, seed=2200 + 10 * layers + stage + ns, layers=layers,
                 n_nodes=400)
    assert c.plan.second_order and c.plan.n_hidden == layers - 2
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f'second order tp_weights_layers={layers} ns={ns} stage={stage}')


@pytest.mark.parametrize('ne,ns,H', [(48, 0, 48), (20, 5, 100), (16, 16, 144), (48, 48, 40)])
def test_kernel_deep_mlp_radial_shapes(built_lib, ne, ns, H):
    """K1 != H, H not a multiple of 16, H < 64 and the element-wise A0 path: the Wh' products use the W2' geometry."""
    table = fused_table(48, 10, 3, 2, False)
    c = DeepCase(table, ne, ns, H, 3 * _sms() * 128 + 17, seed=2300 + H + ne, layers=4, n_nodes=400,
                 node_width=max(ns, 1) + 3)
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f'deep shape ne={ne} ns={ns} H={H}')


@pytest.mark.parametrize('layers', [3, 4])
def test_kernel_deep_mlp_csr_runs_across_tiles(built_lib, layers):
    E = 3 * _sms() * 128 + 17
    tgt, n_out = _runs(E, torch.Generator().manual_seed(layers))
    c = DeepCase(fused_table(48, 10, 3, 2, False), 48, 48, 144, E, seed=2400 + layers, layers=layers,
                 n_nodes=max(500, n_out), n_out=n_out)
    c.tgt = tgt.cuda()
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f'deep runs tp_weights_layers={layers}')


@pytest.mark.parametrize('second_order', [False, True])
@pytest.mark.parametrize('ns,nv', WIDTHS)
def test_kernel_deep_mlp_indirections(built_lib, ns, nv, second_order):
    """edge_perm into a larger store, vec_sign = -1, ea_add, edge_weight and a device-side live count together."""
    table = so_tables(ns, nv, 2)[3] if second_order else fused_table(ns, nv, 3, 2, False)
    E = 2 * _sms() * 128 + 57
    rows = 2 * E
    c = DeepCase(table, ns, ns, 3 * ns, E, seed=2500 + ns + second_order, layers=3, rows=rows, n_nodes=400)
    g = c.gen
    n_live = E - 2 * 64 - 5
    c.tgt[n_live:] = 0
    c.kw = dict(edge_perm=torch.randperm(rows, generator=g)[:E].int().cuda(), vec_sign=-1.0,
                ea_add=torch.randn(7, ns, generator=g).cuda(), ea_add_idx=torch.randint(0, 7, (E,), generator=g).int().cuda(),
                edge_weight=torch.rand(rows, generator=g).cuda(),
                n_edges_dev=torch.tensor([n_live], dtype=torch.int32, device='cuda'))
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(n_live), f'deep indirections ns={ns} second_order={second_order}')


def _mutated_errors(mutate):
    """Block errors of a tp_weights_layers=4 launch (ns=48, last stage) run with the hidden layers changed by
    ``mutate(hidden)``; the unmutated launch passes."""
    from diffdock_b200 import fused
    table = fused_table(48, 10, 3, 2, False)
    c = DeepCase(table, 48, 48, 144, 2 * _sms() * 128 + 57, seed=2601, layers=4, n_nodes=400)
    ref, _ = c.reference()
    got, _ = c.run()
    assert max(block_errors(got, ref, table.out_irreps).values()) < TOL
    got, _ = c.run(plan=fused.FusedPlan(table, *c.w, hidden=mutate(c.hidden)))
    return block_errors(got, ref, table.out_irreps)


def test_comparison_catches_swapped_hidden_layers(built_lib):
    errs = _mutated_errors(lambda h: [h[1], h[0]])
    assert max(errs.values()) > 100 * TOL, errs


def test_comparison_catches_a_dropped_hidden_bias(built_lib):
    errs = _mutated_errors(lambda h: [h[0], (h[1][0], torch.zeros_like(h[1][1]))])
    assert max(errs.values()) > TOL, errs


def test_launcher_rejects_invalid_hidden_stacks(built_lib):
    """n_hidden < 0, and n_hidden > 0 without images: DDB200_EINVAL before any launch."""
    from diffdock_b200 import fused
    c = DeepCase(fused_table(16, 4, 3, 2, False), 16, 16, 48, 300, seed=2700, layers=3)
    for n_hidden, images in ((-1, None), (1, None), (-1, c.plan.wh_images)):
        bad = copy.copy(c.plan)
        bad.n_hidden, bad.wh_images = n_hidden, images
        with pytest.raises(RuntimeError, match='DDB200_EINVAL'):
            c.run(plan=bad)
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), 'after the rejected launches')


# ------------------------------------------------------------------------------------------------------------ model
def _fixture_scores(m, poses, case):
    from diffdock_b200.diffusion_utils import set_time
    from diffdock_b200.hetero import collate
    t, aa = case['t'], case['model'] == 'aa'
    g = collate(copy.deepcopy(poses)).to(DEV)
    set_time(g, None, t, t, t, len(poses), aa, DEV)
    out = m(g)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('i', range(4))
def test_product_matches_reference_fixture(built_lib, i):
    case = fixture()['cases'][i]
    m, poses, _ = tw_model(case, 'product')
    assert m.sync_free_capable() and m.sync_free_crop_capable() == (case['model'] == 'cg')
    _assert_close(_fixture_scores(m, poses, case), (case['tr'], case['rot'], case['tor']), 1e-4)


def test_cropped_sampling_reproduces_reference_fixture(built_lib):
    from diffdock_b200.diffusion_utils import t_to_sigma
    from diffdock_b200.sampling import sampling
    f = fixture()
    s = f['sampling']
    m, poses, a = tw_model(f['cases'][s['model_case']], 'product')
    a.crop_beyond = s['crop_beyond']
    torch.manual_seed(s['seed'])
    noise = lambda kind, shape: torch.normal(mean=0, std=1, size=shape)
    out, _ = sampling(copy.deepcopy(poses), m, s['steps'], s['schedule'], s['schedule'], s['schedule'], DEV,
                      partial(t_to_sigma, args=a), a, batch_size=3, no_final_step_noise=True,
                      temp_sampling=s['temp_sampling'], temp_psi=s['temp_psi'], temp_sigma_data=s['temp_sigma_data'],
                      noise_fn=noise)
    for d, ref in zip(out, s['final_pos']):
        assert rel_err(d['ligand'].pos, ref) < 1e-4


def tw_args(**over):
    from diffdock_b200.synthetic import default_model_args
    kw = dict(ns=48, nv=10, sh_lmax=2, num_conv_layers=4, distance_embed_dim=32, cross_distance_embed_dim=32,
              sigma_embed_dim=32, embed_also_ligand=True, num_prot_emb_layers=1, tp_weights_layers=3)
    kw.update(over)
    return default_model_args(**kw)


def tw_pair(args, seed=0, model='cg'):
    """(oracle model on CPU, product model on cuda:0) with ``args.tp_weights_layers`` sharing one random state_dict,
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
              num_prot_emb_layers=args.num_prot_emb_layers, no_torsion=args.no_torsion,
              tp_weights_layers=args.tp_weights_layers)
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


@pytest.fixture(scope='module')
def tw_model_pair(built_lib):
    args = tw_args()
    o, p = tw_pair(args, seed=5)
    assert p.sync_free_capable() and p.sync_free_crop_capable()
    return o, p, args


@pytest.mark.parametrize('t', [0.3, 0.8])
def test_sync_free_matches_host_sized_and_oracle(tw_model_pair, t):
    from diffdock_b200.synthetic import make_pose_list
    o, p, args = tw_model_pair
    poses = make_pose_list(2, n_res=90, n_atoms=15, seed=21, tr_sigma_max=args.tr_sigma_max * t, lm_dim=0)
    got = _product_scores(p, poses, t)
    host = copy.deepcopy(p)
    host._sync_free = False                           # the exactly-sized path with host-side counts
    _assert_close(got, _product_scores(host, poses, t), 1e-4)
    _assert_close(got, _oracle_scores(o, poses, t), 1e-4)


def test_one_full_size_pose_matches_oracle(built_lib):
    """The 1500-residue / 40-atom complex of config 3 at ns=48, nv=10, six layers, tp_weights_layers=3."""
    from diffdock_b200.synthetic import make_pose_list
    args = tw_args(num_conv_layers=6, distance_embed_dim=64, cross_distance_embed_dim=64, sigma_embed_dim=64,
                   num_prot_emb_layers=0)
    o, p = tw_pair(args, seed=0)
    assert p.sync_free_capable()
    t = 0.5
    poses = make_pose_list(1, n_res=1500, n_atoms=40, seed=100, tr_sigma_max=args.tr_sigma_max * t, lm_dim=0)
    torch.set_num_threads(min(torch.get_num_threads(), 32))
    _assert_close(_product_scores(p, poses, t), _oracle_scores(o, poses, t), 1e-4)


def _graphed_vs_eager(p, args, crop_beyond, monkeypatch, all_atoms=False):
    from diffdock_b200 import sampling as smod
    from diffdock_b200.synthetic import make_pose_list
    args = copy.copy(args)
    args.tr_sigma_max = 5.0        # every ligand stays within reach of some residue: the eager crop needs one
    args.all_atoms = all_atoms
    poses = make_pose_list(4, n_res=120 if not all_atoms else 40, n_atoms=12, seed=41, tr_sigma_max=args.tr_sigma_max,
                           lm_dim=0, all_atoms=all_atoms)
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


@pytest.mark.parametrize('crop_beyond', [None, 20.0])
def test_captured_sampler_matches_eager(tw_model_pair, monkeypatch, crop_beyond):
    _, p, args = tw_model_pair
    _graphed_vs_eager(p, args, crop_beyond, monkeypatch)


def test_graphed_cropped_step_is_sync_free(tw_model_pair):
    import numpy as np
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.hetero import collate_shared_receptor
    from diffdock_b200.sampling import GraphedSteps, crop_cutoff2, step_coefficients
    from diffdock_b200.synthetic import make_pose_list
    _, p, args = tw_model_pair
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


@pytest.fixture(scope='module')
def tw_aa_pair(built_lib):
    a = tw_args(num_conv_layers=3, distance_embed_dim=16, cross_distance_embed_dim=16, sigma_embed_dim=16)
    mo, mp = tw_pair(a, seed=23, model='aa')
    assert mp.sync_free_capable()        # (the all-atom model keeps the eager crop: AAModel.sync_free_crop_capable)
    return mo, mp, a


def test_all_atom_model_matches_oracle(tw_aa_pair):
    from diffdock_b200.diffusion_utils import set_time
    from diffdock_b200.hetero import collate
    from diffdock_b200.synthetic import make_pose_list
    from oracle.diffusion import set_time as o_set_time
    mo, mp, a = tw_aa_pair
    poses = make_pose_list(2, n_res=40, n_atoms=12, seed=93, tr_sigma_max=a.tr_sigma_max * 0.3, lm_dim=0, all_atoms=True)
    t = 0.3
    b = collate(copy.deepcopy(poses))
    o_set_time(b, t, t, t, 2, 'cpu', all_atoms=True)
    with torch.no_grad():
        ref = mo(b)
    bg = collate(copy.deepcopy(poses)).to(DEV)
    set_time(bg, None, t, t, t, 2, True, DEV)
    got = mp(bg)
    host = copy.deepcopy(mp)
    host._sync_free = False
    bh = collate(copy.deepcopy(poses)).to(DEV)
    set_time(bh, None, t, t, t, 2, True, DEV)
    _assert_close(got, host(bh), 1e-4)
    _assert_close(got, ref, 1e-4)


def test_all_atom_captured_sampler_matches_eager(tw_aa_pair, monkeypatch):
    _, p, args = tw_aa_pair
    _graphed_vs_eager(p, args, None, monkeypatch, all_atoms=True)

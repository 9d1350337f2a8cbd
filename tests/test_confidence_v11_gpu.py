"""GPU: confidence models built by the current training code (``CGModel`` / ``AAModel`` with ``confidence_mode=True``) on
the sync-free forward and the one-kernel confidence head (ddb200_confidence_head): the product against the unmodified
reference (tests/golden/ref_confidence_v11.pt), sync-free against host-sized against the oracle at DiffDock-L widths, a
full-size all-atom pose, no host read after the per-batch constants, the head kernel against float64, the ranked sampling
run, and two mutations the fixture must catch."""
import copy
from argparse import Namespace
from functools import partial
from types import SimpleNamespace

import pytest
import torch
from torch import nn

from tests.confidence_v11_helpers import batch_of, build, fixture, head_f64
from tests.parity_helpers import rand_bn_, rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def _run(m, poses, times, all_atoms):
    with torch.no_grad():
        conf, atom = m(batch_of(poses, times, DEV, all_atoms=all_atoms))
    return conf.float().cpu(), atom.float().cpu()


def _close(got, ref, tol=1e-4):
    return got.shape == ref.shape and float((got - ref).abs().max()) <= tol * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize('i', range(5))
def test_product_matches_reference_fixture_on_the_sync_free_path(built_lib, i):
    case = fixture()['cases'][i]
    m, poses = build(case, 'product')
    assert m.sync_free_capable()
    conf, atom = _run(m, poses, case['times'], case['all_atoms'])
    assert _close(conf, case['confidence']), (conf, case['confidence'])
    assert _close(atom, case['atom_confidence']), (atom, case['atom_confidence'])


def _caught(monkeypatch, i, mutate):
    """The fixture check the product passes (``_close`` at 1e-4 on both outputs) fails for the mutated model."""
    case = fixture()['cases'][i]
    m, poses = build(case, 'product')
    mutate(monkeypatch, m, case)
    conf, atom = _run(m, poses, case['times'], case['all_atoms'])
    return not (_close(conf, case['confidence']) and _close(atom, case['atom_confidence']))


def test_mutation_wrong_pseudoscalar_block_is_caught(built_lib, monkeypatch):
    """The head reads the block before the last ``tail`` columns instead of the last block (case 3: the ns x0o block)."""
    import diffdock_b200.cg_model as cg

    def mutate(mp, m, case):
        tail, real = m._conf_tail, cg.confidence_head
        mp.setattr(cg, 'confidence_head', lambda model, x, ptr: real(model, torch.cat([x[:, :-tail], x[:, -2 * tail:-tail]], 1),
                                                                     ptr))
    assert _caught(monkeypatch, 3, mutate)


def test_mutation_t_to_sigma_on_the_confidence_times_is_caught(built_lib, monkeypatch):
    """Case 1 (dynamic_max_cross, smooth_edges): sigma sets the cross cut-off and so every cross edge weight."""
    from diffdock_b200.diffusion_utils import t_to_sigma

    def mutate(mp, m, case):
        a = Namespace(**case['args'])
        mp.setattr(m, '_sigmas', lambda data: t_to_sigma(*[data.complex_t[k] for k in ('tr', 'rot', 'tor')], args=a))
    assert _caught(monkeypatch, 1, mutate)


def _pair(cls_name, seed, **kw):
    """(oracle on CPU, product on cuda:0) confidence models with identical seeded weights and random BatchNorm statistics."""
    from diffdock_b200.diffusion_utils import get_timestep_embedding
    from oracle.layers import get_timestep_embedding as o_temb
    from tests.confidence_v11_oracle import AAConfidenceModel, CGConfidenceModel
    if cls_name == 'CGModel':
        from diffdock_b200.cg_model import CGModel as P
        O = CGConfidenceModel
    else:
        from diffdock_b200.aa_model import AAModel as P
        O = AAConfidenceModel
    base = dict(sigma_embed_dim=16, sh_lmax=2, ns=48, nv=10, num_conv_layers=3, distance_embed_dim=16,
                cross_distance_embed_dim=16, cross_max_distance=30.0, dynamic_max_cross=True, embed_also_ligand=True,
                confidence_mode=True, atom_confidence=True, num_confidence_outputs=3)
    base.update(kw)
    torch.manual_seed(seed)
    o = O(None, 'cpu', o_temb('sinusoidal', 16, 1000), **base).eval()
    g = torch.Generator().manual_seed(seed + 1)
    for mod in o.modules():
        if mod.__class__.__name__ in ('BatchNorm', 'BatchNorm1d'):
            rand_bn_(mod, g)
    p = P(None, DEV, get_timestep_embedding('sinusoidal', 16, 1000), **base).eval()
    p.load_state_dict(o.state_dict(), strict=True)
    return o, p.to(DEV)


@pytest.mark.parametrize('flags', [dict(), dict(reduce_pseudoscalars=True, num_prot_emb_layers=1, sh_lmax=1,
                                                  differentiate_convolutions=False, smooth_edges=True)])
def test_sync_free_vs_host_sized_vs_oracle_at_diffdock_l_widths(built_lib, flags):
    """ns=48, nv=10, two complexes of different sizes in one batch, one time per pose."""
    from diffdock_b200.synthetic import make_pose_list
    o, p = _pair('CGModel', 11, **flags)
    poses = make_pose_list(2, n_res=60, n_atoms=14, seed=5, tr_sigma_max=2.0, lm_dim=0) + \
        make_pose_list(2, n_res=45, n_atoms=11, seed=6, tr_sigma_max=2.0, lm_dim=0)
    times = [0.0, 0.35, 0.8, 0.1]
    with torch.no_grad():
        ref = o(batch_of(poses, times, 'cpu'))
    assert p.sync_free_capable()
    sf = _run(p, poses, times, False)
    p._sync_free = False
    hs = _run(p, poses, times, False)
    for got in (sf, hs):
        assert _close(got[0], ref[0]) and _close(got[1], ref[1]), (got[0], ref[0])
    assert _close(sf[0], hs[0], 1e-5)


def test_full_size_all_atom_pose_matches_oracle(built_lib):
    from diffdock_b200.synthetic import make_pose_list
    o, p = _pair('AAModel', 21, ns=16, nv=4, num_conv_layers=2, num_confidence_outputs=1)
    poses = make_pose_list(1, n_res=1500, n_atoms=40, seed=9, tr_sigma_max=2.0, lm_dim=0, all_atoms=True)
    with torch.no_grad():
        ref = o(batch_of(poses, [0.0], 'cpu', all_atoms=True))
    assert p.sync_free_capable()
    got = _run(p, poses, [0.0], True)
    assert _close(got[0], ref[0]) and _close(got[1], ref[1]), (got[0], ref[0])


@pytest.mark.parametrize('i', [1, 3])
def test_no_host_read_after_the_per_batch_constants(built_lib, i):
    case = fixture()['cases'][i]
    m, poses = build(case, 'product')
    b = batch_of(poses, case['times'], DEV, all_atoms=case['all_atoms'])
    with torch.no_grad():
        first = m(b)[0].clone()               # builds the per-batch constants (one host read)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            again = m(b)[0]
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.equal(first, again)


# ---------------------------------------------------------------------------------------------- head kernel vs float64
def _seq(n_in, ns, n_out, g, bn=True):
    s = nn.Sequential(nn.Linear(n_in, ns), nn.BatchNorm1d(ns) if bn else nn.Identity(), nn.ReLU(), nn.Dropout(0.0),
                      nn.Linear(ns, ns), nn.BatchNorm1d(ns) if bn else nn.Identity(), nn.ReLU(), nn.Dropout(0.0),
                      nn.Linear(ns, n_out)).eval()
    with torch.no_grad():
        for mod in s.modules():
            if isinstance(mod, nn.Linear):
                mod.weight.copy_((2 * torch.rand(mod.weight.shape, generator=g) - 1) * mod.in_features ** -0.5)
                mod.bias.copy_(0.1 * torch.randn(mod.bias.shape, generator=g))
            elif isinstance(mod, nn.BatchNorm1d):
                rand_bn_(mod, g)
    return s


@pytest.mark.parametrize('ns,nv', [(16, 4), (48, 10)])
@pytest.mark.parametrize('tail', ['none', 'nv', 'ns'])
@pytest.mark.parametrize('atom', [False, True])
@pytest.mark.parametrize('k', [1, 4])
def test_head_kernel_matches_float64(built_lib, ns, nv, tail, atom, k):
    from diffdock_b200.layers import confidence_head
    g = torch.Generator().manual_seed(ns + 7 * k + (3 if atom else 0) + len(tail))
    n_tail = {'none': 0, 'nv': nv, 'ns': ns}[tail]
    D = ns + 3 * nv + 3 * nv + n_tail
    counts = [9, 1, 23, 0, 40, 17]                             # unequal poses, one of a single atom, one empty
    ptr = torch.tensor([0] + counts).cumsum(0).int()
    x = torch.randn(int(ptr[-1]), D, generator=g)
    n_in = ns + n_tail
    model = SimpleNamespace(ns=ns, _conf_tail=n_tail, atom_confidence=atom, atom_num_confidence_outputs=2 if atom else 1)
    if atom:
        model.atom_confidence_predictor = _seq(n_in, ns, 2 + ns, g)
        n_in = ns
    model.confidence_predictor = _seq(n_in, ns, k, g, bn=(k == 1))
    ref, ref_atom = head_f64(x, ptr, ns, n_tail, model.confidence_predictor,
                             model.atom_confidence_predictor if atom else None, 2)
    for name in ('confidence_predictor', 'atom_confidence_predictor'):
        if hasattr(model, name):
            getattr(model, name).to(DEV)
    xd, pd = x.to(DEV), ptr.to(DEV)
    conf, atom_conf = confidence_head(model, xd, pd)
    conf2, atom_conf2 = confidence_head(model, xd, pd)
    assert torch.equal(conf, conf2) and torch.equal(atom_conf, atom_conf2)              # fixed order, no atomics
    assert conf.shape == ((len(counts),) if k == 1 else (len(counts), k))
    assert (conf.cpu().double() - ref.squeeze(-1)).abs().max() < 2e-5 * max(1.0, float(ref.abs().max()))
    if atom:
        assert atom_conf.shape == (x.shape[0], 2)
        assert (atom_conf.cpu().double() - ref_atom).abs().max() < 2e-5 * max(1.0, float(ref_atom.abs().max()))
    else:
        assert atom_conf.shape == (x.shape[0],) and not atom_conf.any()


def test_head_kernel_rejects_bad_arguments(built_lib):
    from diffdock_b200 import ops
    x = torch.zeros((4, 16), device=DEV)
    ptr = torch.tensor([0, 4], dtype=torch.int32, device=DEV)
    mlp = torch.zeros(4096, device=DEV)
    with pytest.raises(RuntimeError, match='DDB200_EINVAL'):
        ops.confidence_head(x, ptr, 16, 0, mlp, (20, 16, 1))                  # selection width != MLP input width
    with pytest.raises(RuntimeError, match='DDB200_EINVAL'):
        ops.confidence_head(x, ptr, 8, 8, mlp, (16, ops.CONF_MAX_HIDDEN + 1, 1))


# ---------------------------------------------------------------------------------------------- sampling and ranking
def test_sampling_confidence_matches_fixture_and_ranks(built_lib):
    from diffdock_b200.diffusion_utils import t_to_sigma
    from diffdock_b200.hetero import graph_from_dict
    from diffdock_b200.sampling import rank_poses, sampling
    from tests.test_confidence_v11_cpu import _score_model
    f = fixture()
    s = f['sampling']
    score, a = _score_model(s['score'], 'product')
    a.crop_beyond = s['crop_beyond']
    conf_model, _ = build(f['cases'][s['confidence_case']], 'product')
    poses = [graph_from_dict(d) for d in s['poses']]
    conf_poses = [graph_from_dict(d) for d in s['conf_poses']]
    torch.manual_seed(s['seed'])
    noise = lambda kind, shape: torch.normal(mean=0, std=1, size=shape)           # the reference's CPU draws
    out, conf = sampling(copy.deepcopy(poses), score, s['steps'], s['schedule'], s['schedule'], s['schedule'], 'cuda:0',
                         partial(t_to_sigma, args=a), a, batch_size=3, no_final_step_noise=True, confidence_model=conf_model,
                         confidence_data_list=conf_poses, confidence_model_args=Namespace(all_atoms=True, crop_beyond=None),
                         noise_fn=noise)
    for d, ref in zip(out, s['final_pos']):
        assert rel_err(d['ligand'].pos.cpu(), ref) < 1e-4
    assert _close(conf.cpu(), s['confidence'])
    _, ranked, order = rank_poses(out, conf, torch.zeros(3))
    c = conf.cpu().numpy()
    assert (ranked == c[order]).all() and (ranked[:-1] >= ranked[1:]).all()

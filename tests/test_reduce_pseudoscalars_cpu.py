"""CPU: score models built with ``reduce_pseudoscalars`` (the DiffDock-L flag set: the last irrep of layers 2 and up is
``nv x0o``).  The oracle against the unmodified reference (tests/golden/ref_cg_model_l.pt, make_golden_diffdock_l.py), the
product's parameter names, and the fused plan of the two consumer kinds these layers need: ``(nv, 1)`` = (10, 1) and
(4, 1), 16 rows per tile.  The plan emulation of tests/test_fused_plan_cpu.py reads only what the kernel reads."""
import copy
from argparse import Namespace
from functools import partial

import pytest
import torch

import tests.test_fused_plan_cpu as plan_cpu
from diffdock_b200 import fused
from diffdock_b200.tensor_layers import get_irrep_seq
from diffdock_b200.tp_table import build_table
from tests.old_score_helpers import fixture_state
from tests.parity_helpers import block_errors, fused_conv_reference, fused_weights, load_golden, rel_err

NEW_KINDS = {4: (10, 1, 16), 5: (4, 1, 16)}      # kind -> (mul_out, 2l_out+1, rows per tile)
SH = {1: '1x0e + 1x1o', 2: '1x0e + 1x1o + 1x2e'}


def fixture():
    return load_golden('ref_cg_model_l.pt')


def l_model(case, which):
    """('oracle' on CPU | 'product' on cuda:0) CGModel with a ref_cg_model_l.pt case's weights, and its pose list."""
    from diffdock_b200.hetero import graph_from_dict
    a = Namespace(**case['args'])
    if which == 'oracle':
        from oracle.cg_model import CGModel
        from oracle.diffusion import t_to_sigma
        from oracle.layers import get_timestep_embedding
        dev = 'cpu'
    else:
        from diffdock_b200.cg_model import CGModel
        from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
        dev = torch.device('cuda:0')
    m = CGModel(partial(t_to_sigma, args=a), dev, get_timestep_embedding('sinusoidal', 8, a.embedding_scale),
                **case['kw']).eval()
    ns = case['kw']['ns']
    if case['lm_dim']:   # the fixture shrinks the 1280-wide LM embedding to 16 columns
        m.rec_node_embedding.additional_features_dim = case['lm_dim']
        m.rec_node_embedding.additional_features_embedder = torch.nn.Linear(case['lm_dim'] + ns, ns)
    m.load_state_dict(fixture_state(case), strict=True)
    return m.to(dev), [graph_from_dict(d) for d in case['poses']], a


def test_fixture_covers_the_flag_set():
    f = fixture()
    kws = [c['kw'] for c in f['cases']]
    assert all(k['reduce_pseudoscalars'] and (k['ns'], k['nv']) == (16, 4) for k in kws)
    a = kws[0]
    assert (a['sh_lmax'], a['num_prot_emb_layers'], a['embed_also_ligand'], a['smooth_edges'], a['odd_parity']) == \
        (1, 2, True, True, True) and f['cases'][0]['lm_dim'] == 16
    assert (kws[1]['sh_lmax'], kws[1]['odd_parity']) == (2, False)
    assert kws[2]['odd_parity'] and kws[2]['no_torsion'] and f['cases'][2]['tor'].numel() == 0
    s = f['sampling']
    assert s['crop_beyond'] is not None and 0 < min(s['kept']) and max(s['kept']) < 24     # the crop keeps part of it


@pytest.mark.parametrize('i', range(3))
def test_oracle_matches_reference_fixture(i):
    from diffdock_b200.hetero import collate
    from oracle.diffusion import set_time
    case = fixture()['cases'][i]
    m, poses, _ = l_model(case, 'oracle')
    b = collate(copy.deepcopy(poses))
    set_time(b, case['t'], case['t'], case['t'], len(poses), 'cpu')
    with torch.no_grad():
        tr, rot, tor = m(b)[:3]
    assert rel_err(tr, case['tr']) < 1e-5 and rel_err(rot, case['rot']) < 1e-5
    assert tor.shape == case['tor'].shape and (tor.numel() == 0 or rel_err(tor, case['tor']) < 1e-5)


def test_oracle_reproduces_the_cropped_sampling_run():
    from oracle.diffusion import t_to_sigma
    from oracle.sampling import sampling
    f = fixture()
    s = f['sampling']
    m, poses, a = l_model(f['cases'][s['model_case']], 'oracle')
    a.crop_beyond = s['crop_beyond']
    torch.manual_seed(s['seed'])
    out, _ = sampling(copy.deepcopy(poses), m, s['steps'], s['schedule'], s['schedule'], s['schedule'], 'cpu',
                      partial(t_to_sigma, args=a), a, batch_size=3, no_final_step_noise=True,
                      temp_sampling=s['temp_sampling'], temp_psi=s['temp_psi'], temp_sigma_data=s['temp_sigma_data'])
    for d, ref in zip(out, s['final_pos']):
        assert rel_err(d['ligand'].pos, ref) < 1e-5


def _product(kw, lm_dim=0):
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    from diffdock_b200.synthetic import default_model_args
    a = default_model_args()
    m = CGModel(partial(t_to_sigma, args=a), torch.device('cpu'), get_timestep_embedding('sinusoidal', 8, 1000), **kw)
    if lm_dim:
        m.rec_node_embedding.additional_features_dim = lm_dim
        m.rec_node_embedding.additional_features_embedder = torch.nn.Linear(lm_dim + kw['ns'], kw['ns'])
    return m


@pytest.mark.parametrize('i', range(3))
def test_state_dict_keys_equal_the_reference_module(i):
    """Same parameter and buffer names as the reference module; its extra entries are e3nn's tensor-product buffers
    (``*.tp.*``, ``final_tp_tor.*``), which the product's load_state_dict accepts and drops."""
    case = fixture()['cases'][i]
    ref = {k for k in fixture_state(case) if '.tp.' not in k and not k.startswith('final_tp_tor.')}
    m = _product(case['kw'], case['lm_dim'])
    assert set(m.state_dict()) == ref
    m.load_state_dict(fixture_state(case), strict=True)


def test_diffdock_l_flag_set_takes_the_sync_free_path():
    """The DiffDock-L flag set at ns=48, nv=10 (sh_lmax=1, three receptor embedding layers): every convolution is on the
    fused kernel, so the step runs without host synchronisation and crops inside the captured step."""
    kw = dict(sigma_embed_dim=64, sh_lmax=1, ns=48, nv=10, num_conv_layers=6, distance_embed_dim=64,
              cross_distance_embed_dim=64, dynamic_max_cross=True, lm_embedding_type=None, embed_also_ligand=True,
              num_prot_emb_layers=3, reduce_pseudoscalars=True, smooth_edges=True, odd_parity=True)
    m = _product(kw)
    assert m.sync_free_capable() and m.sync_free_crop_capable()
    # widths outside the fused kernel still take the host-sized path: ns=6, nv=3 ends layers in 3x0o
    m6 = _product(dict(kw, ns=6, nv=3, sigma_embed_dim=8, distance_embed_dim=8, cross_distance_embed_dim=8))
    assert not m6.sync_free_capable()


def _layer_tables(ns, nv, lmax):
    """fctp tables of the conv stages whose output ends in ``nv x0o`` (stages 2 -> 3 and 3 -> 3)."""
    seq = get_irrep_seq(ns, nv, False, True)
    assert seq[3].endswith(f'{nv}x0o') and '0o' not in seq[2]
    return [build_table(seq[s], SH[lmax], seq[3], 'fctp') for s in (2, 3)]


@pytest.mark.parametrize('ns,nv', [(48, 10), (16, 4)])
@pytest.mark.parametrize('lmax', [1, 2])
def test_plan_tiles_of_the_pseudoscalar_block(ns, nv, lmax):
    """Tiles into the nv x0o block: kind 4 / 5 with 16 rows of nv columns, widths rounded to 32-column chunks, the
    first / last / new-path flags, 8-byte node gathers, and each tile's weight rows taken from the reference rows of its
    path (decoded from the split-bf16 image: hi + lo of a small integer is exact)."""
    kind = {10: 4, 4: 5}[nv]
    for table in _layer_tables(ns, nv, lmax):
        H = 3 * ns
        assert fused.supported(table, H, H)
        n_w = table.weight_numel
        w2 = torch.zeros(n_w, H)
        w2[:, 0] = torch.arange(n_w, dtype=torch.float32)                  # column 0 of weight row i holds i
        plan = fused.FusedPlan(table, torch.zeros(H, H), torch.zeros(H), w2, torch.zeros(n_w))
        img = plan_cpu._deswizzle(plan.w2_images)                         # [T, 256, K']
        Kp = (H + 15) // 16 * 16
        row_ref = img[:, :, 0] + img[:, :, Kp]                            # hi + lo of column 0
        tiles = plan.tiles.tolist()
        paths = sorted(table.paths, key=lambda p: (p.i_out, p.w_ref_off))
        odd = [p for p in paths if (p.mul_out, 2 * p.l_out + 1) == (nv, 1)]
        assert odd, 'no path into the nv x0o block'
        x_pairs = all(t[2] % 2 == 0 and (t[3] * t[4]) % 2 == 0 for t in tiles)
        assert plan.x_pairs_ok == int(x_pairs)
        seen = []
        for t, (k, n_mma, x_off, nrow, d_in, out_off, flags, pi) in enumerate(tiles):
            p = paths[pi]
            if (p.mul_out, 2 * p.l_out + 1) != (nv, 1):
                assert k not in NEW_KINDS
                continue
            assert k == kind and NEW_KINDS[k][:2] == (nv, 1)
            assert out_off == p.out_off and out_off + nv <= table.d_out and d_in == 2 * p.l_in + 1
            u0 = (x_off - p.in_off) // d_in
            assert (x_off - p.in_off) % d_in == 0 and u0 % 16 == 0 and nrow == min(16, p.mul_in - u0)
            assert n_mma == min(16 * nv, (nrow * nv + 31) // 32 * 32)
            assert bool(flags & 4) == (t == 0 or tiles[t - 1][7] != pi)
            assert bool(flags & 1) == (t == 0 or tiles[t - 1][5] != out_off)
            assert bool(flags & 2) == (t == len(tiles) - 1 or tiles[t + 1][5] != out_off)
            assert (flags >> 8) == p.sh_off
            want = p.w_ref_off + u0 * nv + torch.arange(nrow * nv, dtype=torch.float64)
            assert torch.equal(row_ref[t, :nrow * nv], want)
            assert not row_ref[t, nrow * nv:].any()                      # padding rows are zero
            seen.append(pi)
        assert sorted(set(seen)) == sorted(paths.index(p) for p in odd)


@pytest.mark.parametrize('ns,nv', [(48, 10), (16, 4)])
@pytest.mark.parametrize('lmax', [1, 2])
@pytest.mark.parametrize('stage', [2, 3])
def test_emulation_of_the_new_kinds_matches_the_reference(monkeypatch, ns, nv, lmax, stage):
    """The plan emulation (the kernel's MMA schedule and tile bookkeeping) against the float64 reference, per output
    block, for layers whose last block is nv x0o."""
    for k, v in NEW_KINDS.items():
        monkeypatch.setitem(plan_cpu.KINDS, k, v)
    table = _layer_tables(ns, nv, lmax)[stage - 2]
    H, K1 = 3 * ns, 3 * ns
    g = torch.Generator().manual_seed(300 + 10 * stage + lmax + ns)
    w = fused_weights(table, H, K1, g)
    plan = fused.FusedPlan(table, *w)
    assert any(t[0] in NEW_KINDS for t in plan.tiles.tolist())
    n_nodes, E = 11, 150
    x = torch.randn(n_nodes, table.d_in, generator=g)
    tgt = torch.randint(0, n_nodes, (E,), generator=g)
    src = torch.randint(0, n_nodes, (E,), generator=g)
    ea, vec, ew = torch.randn(E, ns, generator=g), torch.randn(E, 3, generator=g), torch.rand(E, generator=g)
    got = plan_cpu.emulate(plan, ea, x, ns, tgt, src, x, vec, n_nodes, ew)
    ref, _ = fused_conv_reference(table, *w, ea, x, ns, tgt, src, x, vec, n_nodes, ew=ew)
    errs = block_errors(got, ref, table.out_irreps)
    assert max(errs.values()) < 3e-5, errs


@pytest.mark.parametrize('lmax', [1, 2])
def test_emulation_matches_the_oracle_layer(monkeypatch, lmax):
    """Stage 3 -> 3 of the reduced irreps ladder at ns=48, nv=10 through the oracle TensorProductConvLayer."""
    from oracle import e3nn_lite as o3
    from oracle.tensor_layers import TensorProductConvLayer as OLayer
    from oracle.tensor_layers import get_irrep_seq as o_seq
    for k, v in NEW_KINDS.items():
        monkeypatch.setitem(plan_cpu.KINDS, k, v)
    ns, nv = 48, 10
    seq = o_seq(ns, nv, False, True)
    assert seq[3].endswith(f'{nv}x0o')
    torch.manual_seed(lmax)
    layer = OLayer(seq[3], SH[lmax], seq[3], 3 * ns, residual=False, batch_norm=False, hidden_features=3 * ns).eval()
    table = build_table(seq[3], SH[lmax], seq[3], 'fctp')
    plan = fused.FusedPlan(table, layer.fc[0].weight, layer.fc[0].bias, layer.fc[-1].weight, layer.fc[-1].bias)
    g = torch.Generator().manual_seed(500 + lmax)
    n_nodes, E = 11, 150
    x = torch.randn(n_nodes, table.d_in, generator=g)
    tgt = torch.sort(torch.randint(0, n_nodes, (E,), generator=g)).values
    src = torch.randint(0, n_nodes, (E,), generator=g)
    vec, ea, ew = torch.randn(E, 3, generator=g), torch.randn(E, ns, generator=g), torch.rand(E, 1, generator=g)
    sh = o3.spherical_harmonics(o3.Irreps(SH[lmax]), vec, normalize=True, normalization='component')
    with torch.no_grad():
        ref = layer(x, torch.stack([tgt, src]), torch.cat([ea, x[tgt, :ns], x[src, :ns]], 1), sh, reduce='sum',
                    edge_weight=ew)
    got = plan_cpu.emulate(plan, ea, x, ns, tgt, src, x, vec, n_nodes, ew)
    errs = block_errors(got, ref.double(), table.out_irreps)
    assert max(errs.values()) < 3e-5, errs

"""CPU: score models built with ``use_second_order_repr`` (node irreps with ``nv x2e`` / ``nv x2o`` blocks) on the fused
convolution kernel's second-order instantiation.  The plan of the two consumer kinds these layers add - (10, 5) and
(4, 5), 16 rows per tile - with its [5][5][5] Clebsch-Gordan tables, an emulation of the plan that reads only what the
kernel reads (including the two-slice scatter of the (10, 5) tiles), the models' sync-free capability, and the oracle
against the unmodified reference (tests/golden/ref_cg_model_so.pt, make_golden_second_order.py)."""
import copy
from functools import partial

import pytest
import torch

import tests.test_fused_plan_cpu as plan_cpu
from diffdock_b200 import fused
from diffdock_b200.tensor_layers import get_irrep_seq
from diffdock_b200.tp_table import build_table
from tests.old_score_helpers import fixture_state
from tests.parity_helpers import block_errors, fused_conv_reference, fused_weights, load_golden, rel_err
from tests.test_reduce_pseudoscalars_cpu import l_model

KINDS = {**plan_cpu.KINDS, 4: (10, 1, 16), 5: (4, 1, 16), 6: (10, 5, 16), 7: (4, 5, 16)}
NEW_KINDS = {6: (10, 5, 16), 7: (4, 5, 16)}
SH = {1: '1x0e + 1x1o', 2: '1x0e + 1x1o + 1x2e'}
WIDTHS = [(48, 10), (16, 4)]


def so_tables(ns, nv, lmax):
    """fctp tables of the four conv stages of the second-order irreps ladder (0 -> 1, 1 -> 2, 2 -> 3, 3 -> 3)."""
    seq = get_irrep_seq(ns, nv, True, False)
    return [build_table(seq[s], SH[lmax], seq[min(s + 1, 3)], 'fctp') for s in range(4)]


def emulate(plan, ea, node, ns, tgt, src, x, vec, n_out, ew=None):
    """The kernel's arithmetic on the plan: the MMA schedule of tests/test_fused_plan_cpu.py, M = C . Y from the dense
    [D][D][5] tables (D = 5 for second-order plans), z from the tile's rows and the scatter at the end of an output irrep -
    or, for kind 6, at the end of each tile in two slices (components 0-2, then 3-4)."""
    E = ea.shape[0]
    a0 = torch.cat([ea, node[tgt, :ns], node[src, :ns]], 1) if ns else ea
    w1 = plan_cpu._deswizzle(plan.w1_images)[0]
    H = plan.hidden
    hid = torch.relu(plan_cpu._mma(plan_cpu._split_operand(a0), w1[:H], a0.shape[1])).float()
    A = plan_cpu._split_operand(hid)
    w2 = plan_cpu._deswizzle(plan.w2_images)
    Y = plan_cpu._sh(vec)
    D = 5 if plan.second_order else 3
    mtab = plan.mtab.double()[:, :D * D * 5].reshape(-1, D, D, 5)
    out = torch.zeros(n_out, plan.table.d_out, dtype=torch.float64)
    acc = None

    def scatter(vals, out_off, mul_out, dout, k0=0, dfull=None):
        dfull = dfull or dout
        full = torch.zeros(E, plan.table.d_out, dtype=torch.float64)
        blk = full[:, out_off:out_off + mul_out * dfull].view(E, mul_out, dfull)
        blk[:, :, k0:k0 + dout] = vals
        out.index_add_(0, tgt, full)

    for t, (kind, n_mma, x_off, nrow, d_in, out_off, flags, path) in enumerate(plan.tiles.tolist()):
        mul_out, dout, rows = KINDS[kind]
        assert n_mma % 32 == 0 and nrow * mul_out <= n_mma <= mul_out * rows <= 192 and d_in <= D and dout <= D
        Wt = torch.zeros(E, mul_out * rows, dtype=torch.float64)
        Wt[:, :n_mma] = plan_cpu._mma(A, w2[t, :n_mma], H)
        sh_off = (flags >> 8) & 0xff
        yb = torch.stack([Y[:, min(sh_off + j, 8)] for j in range(5)], 1)
        M = torch.einsum('ikj,ej->eik', mtab[path], yb)
        if ew is not None:
            M = M * ew.double().reshape(-1, 1, 1)
        xs = torch.zeros(E, rows, d_in, dtype=torch.float64)
        xs[:, :nrow] = x[src][:, x_off:x_off + nrow * d_in].double().reshape(E, nrow, d_in)
        z = torch.einsum('eri,eik->erk', xs, M[:, :d_in, :dout])
        z[:, (n_mma // mul_out) + (1 if n_mma % mul_out else 0):] = 0
        part = torch.einsum('erw,erk->ewk', Wt.reshape(E, rows, mul_out), z)
        if kind == 6:
            scatter(part[:, :, :3], out_off, mul_out, 3, 0, 5)
            scatter(part[:, :, 3:], out_off, mul_out, 2, 3, 5)
            continue
        if flags & 1:
            acc = torch.zeros(E, mul_out, dout, dtype=torch.float64)
        acc = acc + part
        if flags & 2:
            scatter(acc, out_off, mul_out, dout)
    return out


@pytest.mark.parametrize('ns,nv', WIDTHS)
@pytest.mark.parametrize('lmax', [1, 2])
def test_every_second_order_layer_is_supported(ns, nv, lmax):
    """Every conv stage of the ladder is accepted, on the second-order instantiation, within its path and tile limits;
    the first-order ladder keeps the first-order instantiation.  Stage 0 at sh_lmax = 1 has no path into its l = 2 output
    block (0e x 1o reaches 1o only): it stays on the first-order instantiation."""
    for s, table in enumerate(so_tables(ns, nv, lmax)):
        assert fused.supported(table, 3 * ns, 3 * ns), s
        assert fused.second_order(table) == (s > 0 or lmax == 2) and len(table.paths) <= fused.MAX_PATHS_SO
    seq = get_irrep_seq(ns, nv, False, False)
    assert not any(fused.second_order(build_table(seq[s], SH[lmax], seq[min(s + 1, 3)], 'fctp')) for s in range(4))


@pytest.mark.parametrize('ns,nv', WIDTHS)
@pytest.mark.parametrize('lmax', [1, 2])
def test_plan_tiles_of_the_l2_blocks(ns, nv, lmax):
    """Tiles into the nv x2e / nv x2o blocks: kind 6 / 7 with 16 rows of nv columns, widths rounded to 32-column chunks,
    the flags, inputs of 1, 3 or 5 components, each tile's weight rows taken from the reference rows of its path, and the
    [5][5][5] table of every path equal to coef * C."""
    from diffdock_b200.irreps import real_cg
    kind = {10: 6, 4: 7}[nv]
    for table in so_tables(ns, nv, lmax)[0 if lmax == 2 else 1:]:
        H = 3 * ns
        n_w = table.weight_numel
        w2 = torch.zeros(n_w, H)
        w2[:, 0] = torch.arange(n_w, dtype=torch.float32)
        plan = fused.FusedPlan(table, torch.zeros(H, H), torch.zeros(H), w2, torch.zeros(n_w))
        assert plan.second_order and plan.mtab.shape == (len(table.paths), fused.MTAB_SO)
        img = plan_cpu._deswizzle(plan.w2_images)
        Kp = (H + 15) // 16 * 16
        row_ref = img[:, :, 0] + img[:, :, Kp]
        tiles = plan.tiles.tolist()
        assert len(tiles) <= fused.MAX_TILES
        paths = sorted(table.paths, key=lambda p: (p.i_out, p.w_ref_off))
        for pi, p in enumerate(paths):
            C = torch.as_tensor(real_cg(p.l_in, p.l_sh, p.l_out))
            m = plan.mtab[pi, :125].double().view(5, 5, 5)
            want = torch.zeros(5, 5, 5, dtype=torch.float64)
            want[:C.shape[0], :C.shape[2], :C.shape[1]] = p.coef * C.permute(0, 2, 1)
            assert torch.allclose(m, want, atol=1e-7) and not plan.mtab[pi, 125:].any()
        l2 = [p for p in paths if p.l_out == 2]
        assert l2
        seen = []
        for t, (k, n_mma, x_off, nrow, d_in, out_off, flags, pi) in enumerate(tiles):
            p = paths[pi]
            assert d_in == 2 * p.l_in + 1 and d_in in (1, 3, 5)
            if p.l_out != 2:
                assert k not in NEW_KINDS
                continue
            assert k == kind and NEW_KINDS[k][:2] == (nv, 5)
            assert out_off == p.out_off and out_off + 5 * nv <= table.d_out
            u0 = (x_off - p.in_off) // d_in
            assert (x_off - p.in_off) % d_in == 0 and u0 % 16 == 0 and nrow == min(16, p.mul_in - u0)
            assert n_mma == min(16 * nv, (nrow * nv + 31) // 32 * 32)
            assert bool(flags & 4) == (t == 0 or tiles[t - 1][7] != pi)
            assert bool(flags & 1) == (t == 0 or tiles[t - 1][5] != out_off)
            assert bool(flags & 2) == (t == len(tiles) - 1 or tiles[t + 1][5] != out_off)
            assert (flags >> 8) == p.sh_off
            want = p.w_ref_off + u0 * nv + torch.arange(nrow * nv, dtype=torch.float64)
            assert torch.equal(row_ref[t, :nrow * nv], want)
            assert not row_ref[t, nrow * nv:].any()
            seen.append(pi)
        assert sorted(set(seen)) == sorted(paths.index(p) for p in l2)
        assert sum(t[3] * KINDS[t[0]][0] for t in tiles) == table.weight_numel
        assert plan.x_pairs_ok == int(all(t[2] % 2 == 0 and (t[3] * t[4]) % 2 == 0 for t in tiles))


@pytest.mark.parametrize('ns,nv', WIDTHS)
@pytest.mark.parametrize('lmax', [1, 2])
@pytest.mark.parametrize('stage', range(4))
def test_emulation_matches_the_fp64_reference(ns, nv, lmax, stage):
    """The plan emulation against the float64 reference, per output block, for every layer of both widths."""
    table = so_tables(ns, nv, lmax)[stage]
    H, K1 = 3 * ns, 3 * ns
    g = torch.Generator().manual_seed(1000 + 10 * stage + lmax + ns)
    w = fused_weights(table, H, K1, g)
    plan = fused.FusedPlan(table, *w)
    n_nodes, E = 11, 150
    x = torch.randn(n_nodes, table.d_in, generator=g)
    tgt = torch.randint(0, n_nodes, (E,), generator=g)
    src = torch.randint(0, n_nodes, (E,), generator=g)
    ea, vec, ew = torch.randn(E, ns, generator=g), torch.randn(E, 3, generator=g), torch.rand(E, generator=g)
    got = emulate(plan, ea, x, ns, tgt, src, x, vec, n_nodes, ew)
    ref, _ = fused_conv_reference(table, *w, ea, x, ns, tgt, src, x, vec, n_nodes, ew=ew)
    errs = block_errors(got, ref, table.out_irreps)
    assert max(errs.values()) < 3e-5, errs


@pytest.mark.parametrize('ns,nv', WIDTHS)
@pytest.mark.parametrize('lmax', [1, 2])
@pytest.mark.parametrize('stage', range(4))
def test_emulation_matches_the_oracle_layer(ns, nv, lmax, stage):
    """Every stage of the second-order ladder through the oracle TensorProductConvLayer."""
    from oracle import e3nn_lite as o3
    from oracle.tensor_layers import TensorProductConvLayer as OLayer
    from oracle.tensor_layers import get_irrep_seq as o_seq
    seq = o_seq(ns, nv, True, False)
    ins, outs = seq[stage], seq[min(stage + 1, 3)]
    torch.manual_seed(lmax + 10 * stage + ns)
    layer = OLayer(ins, SH[lmax], outs, 3 * ns, residual=False, batch_norm=False, hidden_features=3 * ns).eval()
    table = build_table(ins, SH[lmax], outs, 'fctp')
    plan = fused.FusedPlan(table, layer.fc[0].weight, layer.fc[0].bias, layer.fc[-1].weight, layer.fc[-1].bias)
    g = torch.Generator().manual_seed(1500 + lmax + 10 * stage + ns)
    n_nodes, E = 11, 150
    x = torch.randn(n_nodes, table.d_in, generator=g)
    tgt = torch.sort(torch.randint(0, n_nodes, (E,), generator=g)).values
    src = torch.randint(0, n_nodes, (E,), generator=g)
    vec, ea, ew = torch.randn(E, 3, generator=g), torch.randn(E, ns, generator=g), torch.rand(E, 1, generator=g)
    sh = o3.spherical_harmonics(o3.Irreps(SH[lmax]), vec, normalize=True, normalization='component')
    with torch.no_grad():
        ref = layer(x, torch.stack([tgt, src]), torch.cat([ea, x[tgt, :ns], x[src, :ns]], 1), sh, reduce='sum',
                    edge_weight=ew)
    got = emulate(plan, ea, x, ns, tgt, src, x, vec, n_nodes, ew)
    errs = block_errors(got, ref.double(), table.out_irreps)
    assert max(errs.values()) < 3e-5, errs


def so_model_kw(ns=48, nv=10, **over):
    kw = dict(sigma_embed_dim=32, sh_lmax=2, ns=ns, nv=nv, num_conv_layers=4, distance_embed_dim=32,
              cross_distance_embed_dim=32, dynamic_max_cross=True, lm_embedding_type=None, embed_also_ligand=True,
              use_second_order_repr=True)
    kw.update(over)
    return kw


def _product(kw):
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    from diffdock_b200.synthetic import default_model_args
    a = default_model_args()
    return CGModel(partial(t_to_sigma, args=a), torch.device('cpu'), get_timestep_embedding('sinusoidal', 8, 1000), **kw)


@pytest.mark.parametrize('ns,nv', WIDTHS)
@pytest.mark.parametrize('lmax', [1, 2])
def test_second_order_model_takes_the_sync_free_path(ns, nv, lmax):
    """Every convolution of a second-order CGModel is on the fused kernel, so the step runs without host synchronisation
    and crops inside the captured step."""
    m = _product(so_model_kw(ns, nv, sh_lmax=lmax))
    assert all(layer.fused_capable(ns, ns) for layer in m.conv_layers)
    assert m.sync_free_capable() and m.sync_free_crop_capable()


def test_second_order_kernel_issues_each_k_block_as_one_chain(built_lib):
    """The one-chain-per-k-block check of tests/test_fused_chain_sass_cpu.py applied to the second-order instantiation by
    name: one register fence in front of each staged k-block's MMAs, the group's scoreboard on the last one only, eight
    MMAs in the longest chain."""
    import os
    import shutil
    import sys
    from tests.test_fused_chain_sass_cpu import ROOT, _chains, _is_mma
    if shutil.which('cuobjdump') is None:
        pytest.skip('cuobjdump not on PATH')
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import sass_histogram as sh
    body = sh.kernels(os.path.join(ROOT, 'diffdock_b200', 'libdiffdock_b200.so'), operands=True)
    names = [k for k in body if 'fused_conv_kernel' in k]
    so = [k for k in names if 'fused_conv_kernel_so' in k]
    assert len(names) == 2 and len(so) == 1, names
    runs = _chains(body[so[0]])
    assert runs
    for r in runs:
        b = r['body']
        b = b[:max(k for k, i in enumerate(b) if _is_mma(i)) + 1]
        mmas = [i for i in b if _is_mma(i)]
        assert sum(i.startswith('WARPGROUP.ARRIVE') for i in r['lead']) == 1, r
        assert not any(i.startswith('WARPGROUP') for i in b), b
        assert all('gsb0' not in i for i in mmas[:-1]) and 'gsb0' in mmas[-1], mmas
    assert max(sum(_is_mma(i) for i in r['body']) for r in runs) == 8


def fixture():
    return load_golden('ref_cg_model_so.pt')


def test_fixture_covers_the_flag():
    f = fixture()
    kws = [c['kw'] for c in f['cases']]
    assert all(k['use_second_order_repr'] and (k['ns'], k['nv']) == (16, 4) for k in kws)
    assert (kws[0]['sh_lmax'], kws[0]['num_conv_layers']) == (2, 4) and f['cases'][0]['lm_dim'] == 16
    assert (kws[1]['sh_lmax'], kws[1]['reduce_pseudoscalars'], kws[1]['num_prot_emb_layers']) == (1, True, 1)
    assert kws[2]['no_torsion'] and f['cases'][2]['tor'].numel() == 0
    s = f['sampling']
    assert s['crop_beyond'] is not None and 0 < min(s['kept']) < 24


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


@pytest.mark.parametrize('i', range(3))
def test_state_dict_keys_equal_the_reference_module(i):
    """Same parameter and buffer names as the reference module, except e3nn's tensor-product buffers (``*.tp.*``,
    ``final_tp_tor.*``), which the product's load_state_dict accepts and drops."""
    case = fixture()['cases'][i]
    ref = {k for k in fixture_state(case) if '.tp.' not in k and not k.startswith('final_tp_tor.')}
    m = _product(case['kw'])
    if case['lm_dim']:
        ns = case['kw']['ns']
        m.rec_node_embedding.additional_features_dim = case['lm_dim']
        m.rec_node_embedding.additional_features_embedder = torch.nn.Linear(case['lm_dim'] + ns, ns)
    assert set(m.state_dict()) == ref
    m.load_state_dict(fixture_state(case), strict=True)

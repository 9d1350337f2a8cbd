"""CPU: score models built with ``tp_weights_layers`` > 2 (DiffDock-L's ``--tp_weights_layers``: the radial MLP of every
embedding and interaction convolution has ``tp_weights_layers - 2`` extra H x H hidden layers) on the fused convolution
kernel.  The predicate that admits such an FCBlock to the fused kernel, the extra layers' operand images, a two-layer plan
unchanged by the new ``hidden`` argument, the float64 reference the GPU tests compare against, the models' sync-free
capability, and the oracle against the unmodified reference (tests/golden/ref_cg_model_tw.pt,
make_golden_tp_weights.py)."""
import copy
from argparse import Namespace
from functools import partial

import pytest
import torch
from torch import nn

import tests.test_fused_plan_cpu as plan_cpu
from diffdock_b200 import fused
from diffdock_b200.tensor_layers import FCBlock, TensorProductConvLayer
from tests.old_score_helpers import fixture_state
from tests.parity_helpers import (_reference_tp, block_errors, fused_table, fused_weights, load_golden, rel_err,
                                  tp_scatter_reference)

WIDTHS = [(48, 10), (16, 4)]
SH = {1: '1x0e + 1x1o', 2: '1x0e + 1x1o + 1x2e'}


def hidden_weights(H, n_hidden, gen):
    """``n_hidden`` extra H x H hidden layers ``[(W, b)]`` at a trained model's scale."""
    return [(torch.randn(H, H, generator=gen) / H ** 0.5, 0.1 * torch.randn(H, generator=gen)) for _ in range(n_hidden)]


def fused_conv_reference_deep(table, w1, b1, hidden, w2, b2, ea, node, ns, tgt, src, x, vec, n_out, ew=None,
                              edge_perm=None, vec_sign=1.0, ea_add=None, ea_add_idx=None, device=None, chunk=2048):
    """tests/parity_helpers.py:fused_conv_reference with the radial MLP of an FCBlock built with ``tp_weights_layers`` =
    2 + len(hidden):
        h = relu(a W1^T + b1),  h = relu(h Wh^T + bh) for (Wh, bh) in hidden,  w = h W2^T + b2
    in float64, chunk by chunk over the edges.  Returns (sum [n_out, d_out], cnt [n_out]) on ``device`` (default: ea's)."""
    dev = torch.device(device) if device is not None else ea.device
    tp = _reference_tp(table, dev)
    assert w2.shape[0] == table.weight_numel
    d = lambda t: t.to(dev, torch.float64)
    w1, b1, w2, b2, x = d(w1), d(b1), d(w2), d(b2), d(x)
    hidden = [(d(w), d(b)) for w, b in hidden]
    ne = w1.shape[1] - 2 * ns
    tgt, src = tgt.to(dev).long(), src.to(dev).long()
    ea, vec = d(ea[:, :ne]), d(vec)
    node = d(node[:, :ns]) if ns else None
    ew = d(ew.reshape(-1)) if ew is not None else None
    ea_add = d(ea_add) if ea_add is not None else None
    out = torch.zeros(n_out, table.d_out, dtype=torch.float64, device=dev)
    for c0 in range(0, tgt.shape[0], chunk):
        c1 = min(tgt.shape[0], c0 + chunk)
        r = edge_perm[c0:c1].to(dev).long() if edge_perm is not None else torch.arange(c0, c1, device=dev)
        t, s = tgt[c0:c1], src[c0:c1]
        a = ea[r]
        if ea_add is not None:
            a = a + ea_add[ea_add_idx[c0:c1].to(dev).long()]
        if ns:
            a = torch.cat([a, node[t], node[s]], 1)
        h = torch.relu(a @ w1.T + b1)
        for wh, bh in hidden:
            h = torch.relu(h @ wh.T + bh)
        tp_scatter_reference(table, x, s, t, vec_sign * vec[r], h @ w2.T + b2, n_out,
                             ew=ew[r] if ew is not None else None, device=dev, chunk=c1 - c0, tp=tp, out=out)
    return out, torch.bincount(tgt, minlength=n_out).double()


# ------------------------------------------------------------------------------------------------------------ predicate
@pytest.mark.parametrize('layers', [2, 3, 4])
def test_predicate_accepts_relu_fcblocks(layers):
    fc = FCBlock(144, 144, 500, layers, 0.0)
    assert TensorProductConvLayer._fused_mlp(fc, 144)
    assert TensorProductConvLayer._fused_mlp(FCBlock(48, 48, 100, layers, 0.1), 48)


def test_predicate_rejects_other_mlps():
    ok = TensorProductConvLayer._fused_mlp
    assert not ok(FCBlock(48, 48, 100, 3, 0.0, activation='silu'), 48)
    assert not ok(FCBlock(48, 48, 100, 2, 0.0, activation='silu'), 48)
    rect = nn.Sequential(nn.Linear(48, 48), nn.ReLU(), nn.Dropout(0.0), nn.Linear(48, 32), nn.ReLU(), nn.Dropout(0.0),
                         nn.Linear(32, 100))
    assert not ok(rect, 48)                                       # a hidden layer that is not square
    assert not ok(FCBlock(160, 160, 100, 3, 0.0), 160)            # H > 144
    assert not ok(FCBlock(48, 48, 100, 3, 0.0)[:-1], 48)         # no output Linear
    no_drop = nn.Sequential(nn.Linear(48, 48), nn.ReLU(), nn.Linear(48, 48), nn.ReLU(), nn.Linear(48, 100))
    assert not ok(no_drop, 48)


def test_radial_mlp_gate_stays_two_layer():
    """The host-sized path's one-kernel radial MLP (ddb200_radial_mlp) takes two-layer FCBlocks only; deeper ones run
    there as torch Linears + radial_gemm, as before."""
    assert TensorProductConvLayer._fusable(FCBlock(48, 48, 100, 2, 0.0), 48)
    assert not TensorProductConvLayer._fusable(FCBlock(48, 48, 100, 3, 0.0), 48)
    assert not TensorProductConvLayer._fusable(FCBlock(48, 48, 100, 4, 0.0), 48)


@pytest.mark.parametrize('layers', [3, 4])
def test_layer_plan_carries_every_hidden_layer_and_follows_parameter_updates(layers):
    """The layer's cached plan holds the extra layers in order and is rebuilt when any Linear changes, not just the
    first and the last."""
    seq = ['48x0e', '48x0e + 10x1o']
    layer = TensorProductConvLayer(seq[0], SH[2], seq[1], 144, hidden_features=144, tp_weights_layers=layers).eval()
    assert layer.fused_capable(48, 48)
    table = layer.tp.table_vec
    plan = layer._fused_plan(layer.fc, table, 144)
    assert plan is not None and plan.n_hidden == layers - 2
    assert layer._fused_plan(layer.fc, table, 144) is plan
    lin = layer.fc[3]
    with torch.no_grad():
        lin.bias.add_(1.0)
    plan2 = layer._fused_plan(layer.fc, table, 144)
    assert plan2 is not plan
    dec = _decode(plan2.wh_images)[0]
    Kp = 144
    assert torch.allclose(dec[:144, 2 * Kp] + dec[:144, 2 * Kp + 1], lin.bias.double(), atol=1e-5)


# ------------------------------------------------------------------------------------------------------------ plan
def _decode(img):
    return plan_cpu._deswizzle(img)


@pytest.mark.parametrize('H', [144, 48, 40])
@pytest.mark.parametrize('n_hidden', [1, 2])
def test_hidden_images_decode_to_the_layers(H, n_hidden):
    """Each extra layer is one N tile in the W2' layout: hi + lo of its columns is W within the split-bf16 error, the
    folded bias columns give b, every padding row and column is zero."""
    table = fused_table(48, 10, 3, 2, False)
    g = torch.Generator().manual_seed(H + n_hidden)
    w = fused_weights(table, H, 144, g)
    hidden = hidden_weights(H, n_hidden, g)
    plan = fused.FusedPlan(table, *w, hidden=hidden)
    Kp = (H + 15) // 16 * 16
    n_kb = (2 * Kp + 16 + 63) // 64
    assert plan.n_hidden == n_hidden and tuple(plan.wh_images.shape) == (n_hidden, n_kb, 256, 8, 8)
    assert plan.wh_images.dtype == torch.bfloat16 and plan.wh_images.is_contiguous()
    dec = _decode(plan.wh_images)
    for l, (W, b) in enumerate(hidden):
        got = dec[l, :H, :H] + dec[l, :H, Kp:Kp + H]
        assert (got - W.double()).abs().max() <= 2 ** -16 * W.abs().max() + 1e-12
        gb = dec[l, :H, 2 * Kp] + dec[l, :H, 2 * Kp + 1]
        assert (gb - b.double()).abs().max() <= 2 ** -16 * b.abs().max() + 1e-12
        assert not dec[l, H:].any() and not dec[l, :, H:Kp].any() and not dec[l, :, Kp + H:2 * Kp].any()
        assert not dec[l, :, 2 * Kp + 2:].any()


@pytest.mark.parametrize('ns,nv', WIDTHS)
@pytest.mark.parametrize('stage', range(4))
def test_two_layer_plan_is_unchanged(ns, nv, stage):
    """A plan built with ``hidden=()`` is byte for byte the plan of the positional four-argument call: images, tiles,
    tables and FLOP counts; it streams no extra layer."""
    table = fused_table(ns, nv, stage, 2, False)
    w = fused_weights(table, 3 * ns, 3 * ns, torch.Generator().manual_seed(stage + ns))
    old, new = fused.FusedPlan(table, *w), fused.FusedPlan(table, *w, hidden=())
    for k in ('w1_images', 'w2_images', 'tiles', 'mtab'):
        assert torch.equal(getattr(old, k), getattr(new, k)), k
    for k in ('mma_flops_per_tile', 'alg_flops_per_edge', 'n_tiles', 'n_paths', 'x_pairs_ok', 'hidden', 'k1'):
        assert getattr(old, k) == getattr(new, k), k
    assert new.n_hidden == 0 and new.wh_images is None


def test_flop_counts_include_the_hidden_products():
    table = fused_table(48, 10, 3, 2, False)
    g = torch.Generator().manual_seed(3)
    w = fused_weights(table, 144, 144, g)
    two = fused.FusedPlan(table, *w)
    deep = fused.FusedPlan(table, *w, hidden=hidden_weights(144, 2, g))
    s2 = 3 * (144 // 16) + 1
    assert deep.mma_flops_per_tile - two.mma_flops_per_tile == 2 * 2 * 64 * 16 * 192 * s2
    assert deep.alg_flops_per_edge - two.alg_flops_per_edge == 2 * 2 * 144 * 144


@pytest.mark.parametrize('layers', [3, 4])
@pytest.mark.parametrize('lmax', [1, 2])
def test_deep_reference_matches_the_oracle_layer(layers, lmax):
    """The float64 reference of the GPU tests against the oracle TensorProductConvLayer with ``tp_weights_layers``."""
    from oracle import e3nn_lite as o3
    from oracle.tensor_layers import TensorProductConvLayer as OLayer
    ns, nv = 16, 4
    seq = ['16x0e', '16x0e + 4x1o']
    torch.manual_seed(layers + 10 * lmax)
    layer = OLayer(seq[0], SH[lmax], seq[1], 3 * ns, residual=False, batch_norm=False, hidden_features=3 * ns,
                   tp_weights_layers=layers).eval()
    lins = [m for m in layer.fc if isinstance(m, nn.Linear)]
    assert len(lins) == layers
    table = fused_table(ns, nv, 0, lmax, False)
    g = torch.Generator().manual_seed(2000 + layers + lmax)
    n_nodes, E = 11, 150
    x = torch.randn(n_nodes, table.d_in, generator=g)
    tgt = torch.randint(0, n_nodes, (E,), generator=g)
    src = torch.randint(0, n_nodes, (E,), generator=g)
    vec, ea, ew = torch.randn(E, 3, generator=g), torch.randn(E, ns, generator=g), torch.rand(E, 1, generator=g)
    sh = o3.spherical_harmonics(o3.Irreps(SH[lmax]), vec, normalize=True, normalization='component')
    with torch.no_grad():
        ref = layer(x, torch.stack([tgt, src]), torch.cat([ea, x[tgt, :ns], x[src, :ns]], 1), sh, reduce='sum',
                    edge_weight=ew)
        got, _ = fused_conv_reference_deep(table, lins[0].weight, lins[0].bias,
                                           [(m.weight, m.bias) for m in lins[1:-1]], lins[-1].weight, lins[-1].bias,
                                           ea, x, ns, tgt, src, x, vec, n_nodes, ew=ew)
    errs = block_errors(got, ref.double(), table.out_irreps)
    assert max(errs.values()) < 1e-5, errs


# ------------------------------------------------------------------------------------------------------------ models
def _product(kw, model='cg'):
    from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    from diffdock_b200.synthetic import default_model_args
    if model == 'aa':
        from diffdock_b200.aa_model import AAModel as Model
    else:
        from diffdock_b200.cg_model import CGModel as Model
    a = default_model_args()
    return Model(partial(t_to_sigma, args=a), torch.device('cpu'), get_timestep_embedding('sinusoidal', 8, 1000), **kw)


def tw_model_kw(ns=48, nv=10, layers=3, **over):
    kw = dict(sigma_embed_dim=32, sh_lmax=2, ns=ns, nv=nv, num_conv_layers=4, distance_embed_dim=32,
              cross_distance_embed_dim=32, dynamic_max_cross=True, lm_embedding_type=None, embed_also_ligand=True,
              num_prot_emb_layers=1, tp_weights_layers=layers)
    kw.update(over)
    return kw


@pytest.mark.parametrize('model', ['cg', 'aa'])
@pytest.mark.parametrize('layers', [3, 4])
@pytest.mark.parametrize('ns,nv', WIDTHS)
def test_deep_mlp_models_take_the_sync_free_path(ns, nv, layers, model):
    """Every convolution of the model (embedding and interaction layers) is on the fused kernel, so the step runs
    without host synchronisation and (score model; the all-atom model keeps the eager crop) crops inside the captured
    step."""
    m = _product(tw_model_kw(ns, nv, layers), model)
    convs = list(m.conv_layers) + list(getattr(m, 'lig_emb_layers', [])) + list(m.rec_emb_layers)
    assert len(convs) > len(m.conv_layers)
    assert all(len([x for x in layer.fc.modules() if isinstance(x, nn.Linear)]) >= layers for layer in convs)
    assert all(layer.fused_capable(ns, ns) for layer in convs)
    assert m.sync_free_capable() and m.sync_free_crop_capable() == (model == 'cg')


def test_silu_mlp_models_stay_on_the_host_sized_path():
    import diffdock_b200.tensor_layers as tl
    m = _product(tw_model_kw(48, 10, 3))
    with torch.no_grad():
        for layer in m.conv_layers:
            fcs = layer.fc if isinstance(layer.fc, nn.ModuleList) else [layer.fc]
            for fc in fcs:
                fc[1] = tl.ACTIVATIONS['silu']()
    m._sync_free = None
    assert not m.sync_free_capable()


# ------------------------------------------------------------------------------------------------------------ fixture
def fixture():
    return load_golden('ref_cg_model_tw.pt')


def tw_model(case, which):
    """('oracle' on CPU | 'product' on cuda:0) CGModel or AAModel with a ref_cg_model_tw.pt case's weights, and its pose
    list and arguments."""
    from diffdock_b200.hetero import graph_from_dict
    a = Namespace(**case['args'])
    aa = case['model'] == 'aa'
    if which == 'oracle':
        from oracle.aa_model import AAModel
        from oracle.cg_model import CGModel
        from oracle.diffusion import t_to_sigma
        from oracle.layers import get_timestep_embedding
        dev = 'cpu'
    else:
        from diffdock_b200.aa_model import AAModel
        from diffdock_b200.cg_model import CGModel
        from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
        dev = torch.device('cuda:0')
    cls = AAModel if aa else CGModel
    m = cls(partial(t_to_sigma, args=a), dev, get_timestep_embedding('sinusoidal', 8, a.embedding_scale),
            **case['kw']).eval()
    ns = case['kw']['ns']
    if case['lm_dim']:   # the fixture shrinks the 1280-wide LM embedding to 16 columns
        m.rec_node_embedding.additional_features_dim = case['lm_dim']
        m.rec_node_embedding.additional_features_embedder = torch.nn.Linear(case['lm_dim'] + ns, ns)
    m.load_state_dict(fixture_state(case), strict=True)
    return m.to(dev), [graph_from_dict(d) for d in case['poses']], a


def test_fixture_covers_the_flag():
    f = fixture()
    cs = f['cases']
    assert all((c['kw']['ns'], c['kw']['nv']) == (16, 4) for c in cs)
    assert [(c['model'], c['kw']['tp_weights_layers'], c['kw']['sh_lmax']) for c in cs] == \
        [('cg', 3, 2), ('cg', 4, 1), ('cg', 3, 2), ('aa', 3, 2)]
    assert cs[1]['kw']['reduce_pseudoscalars'] and cs[1]['kw']['num_prot_emb_layers'] == 1
    assert cs[2]['kw']['use_second_order_repr']
    s = f['sampling']
    assert s['crop_beyond'] is not None and 0 < min(s['kept']) < 24


@pytest.mark.parametrize('i', range(4))
def test_oracle_matches_reference_fixture(i):
    from diffdock_b200.hetero import collate
    from oracle.diffusion import set_time
    case = fixture()['cases'][i]
    m, poses, _ = tw_model(case, 'oracle')
    b = collate(copy.deepcopy(poses))
    set_time(b, case['t'], case['t'], case['t'], len(poses), 'cpu', all_atoms=case['model'] == 'aa')
    with torch.no_grad():
        tr, rot, tor = m(b)[:3]
    assert rel_err(tr, case['tr']) < 1e-5 and rel_err(rot, case['rot']) < 1e-5
    assert tor.shape == case['tor'].shape and (tor.numel() == 0 or rel_err(tor, case['tor']) < 1e-5)


def test_oracle_reproduces_the_cropped_sampling_run():
    from oracle.diffusion import t_to_sigma
    from oracle.sampling import sampling
    f = fixture()
    s = f['sampling']
    m, poses, a = tw_model(f['cases'][s['model_case']], 'oracle')
    a.crop_beyond = s['crop_beyond']
    torch.manual_seed(s['seed'])
    out, _ = sampling(copy.deepcopy(poses), m, s['steps'], s['schedule'], s['schedule'], s['schedule'], 'cpu',
                      partial(t_to_sigma, args=a), a, batch_size=3, no_final_step_noise=True,
                      temp_sampling=s['temp_sampling'], temp_psi=s['temp_psi'], temp_sigma_data=s['temp_sigma_data'])
    for d, ref in zip(out, s['final_pos']):
        assert rel_err(d['ligand'].pos, ref) < 1e-5


@pytest.mark.parametrize('i', range(4))
def test_state_dict_keys_equal_the_reference_module(i):
    """Same parameter and buffer names as the reference module (the extra hidden Linears at fc.3, fc.6, ...), except
    e3nn's tensor-product buffers, which the product's load_state_dict accepts and drops."""
    case = fixture()['cases'][i]
    ref = {k for k in fixture_state(case) if '.tp.' not in k and not k.startswith('final_tp_tor.')}
    m = _product(case['kw'], case['model'])
    if case['lm_dim']:
        ns = case['kw']['ns']
        m.rec_node_embedding.additional_features_dim = case['lm_dim']
        m.rec_node_embedding.additional_features_embedder = torch.nn.Linear(case['lm_dim'] + ns, ns)
    assert set(m.state_dict()) == ref
    m.load_state_dict(fixture_state(case), strict=True)

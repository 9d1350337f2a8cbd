"""CPU: confidence models built by the current training code (``CGModel`` / ``AAModel`` with ``confidence_mode=True``).
The oracle (tests/confidence_v11_oracle.py) against the unmodified reference (tests/golden/ref_confidence_v11.pt), the
get_model keywords, the product's parameter names and modules, what keeps raising, and the confidence kernel's build."""
import copy
import os
import re
import subprocess
import tempfile
from argparse import Namespace

import pytest
import torch

from tests.confidence_v11_helpers import batch_of, build, fixture
from tests.old_score_helpers import fixture_state
from tests.parity_helpers import rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCORE_HEADS = ('center_distance_expansion', 'center_edge_embedding', 'final_conv', 'tr_final_layer', 'rot_final_layer',
               'final_edge_embedding', 'tor_bond_conv', 'tor_final_layer', '_so3_table', '_torus_table')


def test_fixture_covers_the_cases():
    cases = fixture()['cases']
    kws = [c['kw'] for c in cases]
    assert all(k['confidence_mode'] and (k['ns'], k['nv']) == (16, 4) for k in kws)
    assert [c['cls'] for c in cases] == ['CGModel', 'CGModel', 'CGModel', 'AAModel', 'CGModel']
    assert kws[0]['num_conv_layers'] == 3 and kws[0]['sh_lmax'] == 2
    k = kws[1]
    assert (k['reduce_pseudoscalars'], k['smooth_edges'], k['sh_lmax'], k['num_prot_emb_layers'], k['dynamic_max_cross']) == \
        (True, True, 1, 1, True)
    assert cases[1]['confidence'].shape == (3, 5) and k['affinity_prediction']
    assert kws[2]['num_conv_layers'] == 2 and kws[2]['atom_confidence'] and cases[2]['atom_confidence'].shape[1] == 2
    assert kws[3]['num_conv_layers'] == 3 and kws[3]['atom_confidence']
    assert kws[4]['tp_weights_layers'] == 3
    assert len({tuple(c['times'].tolist()) for c in cases}) > 2                 # per-graph times, not all zero


@pytest.mark.parametrize('i', range(5))
def test_oracle_matches_reference_fixture(i):
    case = fixture()['cases'][i]
    m, poses = build(case, 'oracle')
    b = batch_of(poses, case['times'], 'cpu', all_atoms=case['all_atoms'])
    with torch.no_grad():
        conf, atom = m(b)
    assert conf.shape == case['confidence'].shape and rel_err(conf, case['confidence']) < 1e-5
    assert atom.shape == case['atom_confidence'].shape
    if case['kw'].get('atom_confidence'):
        assert rel_err(atom, case['atom_confidence']) < 1e-5


def _score_model(s, which):
    from functools import partial
    a = Namespace(**s['args'])
    if which == 'oracle':
        from oracle.cg_model import CGModel
        from oracle.diffusion import t_to_sigma
        from oracle.layers import get_timestep_embedding
        dev = 'cpu'
    else:
        from diffdock_b200.cg_model import CGModel
        from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
        dev = torch.device('cuda:0')
    m = CGModel(partial(t_to_sigma, args=a), dev, get_timestep_embedding('sinusoidal', 8, a.embedding_scale), **s['kw']).eval()
    m.load_state_dict(fixture_state(s), strict=True)
    return m.to(dev), a


def test_oracle_reproduces_the_ranked_sampling_run():
    from functools import partial
    from diffdock_b200.hetero import graph_from_dict
    from oracle.diffusion import t_to_sigma
    from oracle.sampling import sampling
    f = fixture()
    s = f['sampling']
    score, a = _score_model(s['score'], 'oracle')
    a.crop_beyond = s['crop_beyond']
    conf_model, _ = build(f['cases'][s['confidence_case']], 'oracle')
    poses = [graph_from_dict(d) for d in s['poses']]
    conf_poses = [graph_from_dict(d) for d in s['conf_poses']]
    torch.manual_seed(s['seed'])
    out, conf = sampling(copy.deepcopy(poses), score, s['steps'], s['schedule'], s['schedule'], s['schedule'], 'cpu',
                         partial(t_to_sigma, args=a), a, batch_size=3, no_final_step_noise=True, confidence_model=conf_model,
                         confidence_data_list=conf_poses, confidence_model_args=Namespace(all_atoms=True, crop_beyond=None))
    for d, ref in zip(out, s['final_pos']):
        assert rel_err(d['ligand'].pos, ref) < 1e-5
    assert rel_err(conf, s['confidence']) < 1e-5


@pytest.mark.parametrize('i', range(2))
def test_get_model_keywords_match_the_reference(i):
    from diffdock_b200.utils import model_kwargs
    g = fixture()['get_model'][i]
    name, kw = model_kwargs(Namespace(**g['args']), confidence_mode=True, old=False)
    assert name == g['cls'] == ('AAModel' if g['args']['all_atoms'] else 'CGModel')
    assert kw == g['kwargs']


def test_get_model_builds_the_confidence_classes():
    from diffdock_b200.aa_model import AAModel
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.utils import get_model
    for g, cls in zip(fixture()['get_model'], (AAModel, CGModel)):
        m = get_model(Namespace(**g['args']), 'cpu', None, no_parallel=True, confidence_mode=True)
        assert type(m) is cls and m.confidence_mode and hasattr(m, 'confidence_predictor')


@pytest.mark.parametrize('i', range(5))
def test_fixture_state_dict_loads_strict_and_has_no_score_heads(i):
    case = fixture()['cases'][i]
    m, _ = build(case, 'product-cpu')
    ref = {k for k in fixture_state(case) if '.tp.' not in k}
    assert set(m.state_dict()) == ref
    names = {n.split('.')[0] for n, _ in m.named_modules()} | {n for n, _ in m.named_buffers()}
    assert not names & set(SCORE_HEADS)
    assert hasattr(m, 'atom_confidence_predictor') == bool(case['kw'].get('atom_confidence'))


def _kw(**over):
    kw = dict(sigma_embed_dim=8, ns=16, nv=4, num_conv_layers=2, distance_embed_dim=8, cross_distance_embed_dim=8,
              embed_also_ligand=True, confidence_mode=True)
    kw.update(over)
    return kw


def _make(cls_name='CGModel', **over):
    from diffdock_b200.diffusion_utils import get_timestep_embedding
    if cls_name == 'CGModel':
        from diffdock_b200.cg_model import CGModel as cls
    else:
        from diffdock_b200.aa_model import AAModel as cls
    return cls(None, 'cpu', get_timestep_embedding('sinusoidal', 8, 1000), **_kw(**over))


@pytest.mark.parametrize('over,width', [(dict(), 16), (dict(num_conv_layers=3), 32), (dict(num_conv_layers=2, num_prot_emb_layers=1), 32),
                                        (dict(num_conv_layers=3, reduce_pseudoscalars=True), 20),
                                        (dict(num_conv_layers=3, atom_confidence=True), 16)])
def test_input_width_counts_embedding_and_interaction_layers(over, width):
    """input_size = ns + (nv | ns) when num_conv_layers + num_prot_emb_layers >= 3, else ns; ns after the atom head."""
    m = _make(**over)
    assert m.confidence_predictor[0].in_features == width
    if over.get('atom_confidence'):
        assert m.atom_confidence_predictor[0].in_features == 32 and m.atom_confidence_predictor[-1].out_features == 17


@pytest.mark.parametrize('cls_name', ['CGModel', 'AAModel'])
def test_what_keeps_raising(cls_name):
    with pytest.raises(NotImplementedError):
        _make(cls_name, sidechain_pred=True)
    with pytest.raises((AssertionError, NotImplementedError)):
        _make(cls_name, parallel=2)
    with pytest.raises(NotImplementedError):
        _make(cls_name, include_miscellaneous_atoms=True)
    with pytest.raises(NotImplementedError):
        _make(cls_name, separate_noise_schedule=True)
    if cls_name == 'AAModel':
        with pytest.raises(NotImplementedError):
            _make(cls_name, crop_beyond=20.0)


def test_heads_wider_than_the_kernel_are_rejected_at_construction():
    from diffdock_b200 import ops
    with pytest.raises(NotImplementedError):
        _make(ns=ops.CONF_MAX_HIDDEN + 16, nv=4)
    with pytest.raises(NotImplementedError):
        _make(num_confidence_outputs=ops.CONF_MAX_OUT + 1)
    with pytest.raises(NotImplementedError):
        _make(atom_confidence=True, atom_num_confidence_outputs=ops.CONF_MAX_OUT + 1)


def test_kernel_limits_match_the_header():
    from diffdock_b200 import ops
    h = open(os.path.join(ROOT, 'include', 'diffdock_b200.h')).read()
    got = {k: int(v) for k, v in re.findall(r'#define DDB200_CONF_MAX_(\w+) (\d+)', h)}
    assert got == {'IN': ops.CONF_MAX_IN, 'HIDDEN': ops.CONF_MAX_HIDDEN, 'OUT': ops.CONF_MAX_OUT}


def test_library_exports_the_confidence_head(built_lib):
    assert hasattr(built_lib, 'ddb200_confidence_head')


def test_confidence_kernel_has_no_spills():
    import __graft_entry__ as g
    src = os.path.join(ROOT, 'diffdock_b200', 'csrc', 'confidence.cu')
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([g._nvcc()] + g.NVCC_FLAGS + ['-Xptxas', '-v', '-c', src, '-o', os.path.join(d, 'c.o')],
                           capture_output=True, text=True, check=True)
    lines = r.stderr.splitlines()
    i = next(k for k, line in enumerate(lines) if 'confidence_head_kernel' in line and 'Function properties' in line)
    assert re.search(r'0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads', lines[i + 1]), lines[i:i + 3]

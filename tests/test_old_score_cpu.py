"""CPU: the v1.0 score model (models/old_cg_model.py:CGOldModel with confidence_mode=False) - oracle vs the unmodified
reference (tests/golden/ref_old_score_model.pt, tests/golden/make_golden_old_score.py), the factory route
``get_model(..., old=True)`` and the product's parameter layout."""
from argparse import Namespace
from functools import partial

import pytest
import torch

from tests.old_score_helpers import fixture_case, fixture_model, fixture_state, score
from tests.parity_helpers import load_golden, rel_err


@pytest.mark.parametrize('i', range(5))
def test_oracle_matches_reference_fixture(i):
    case = fixture_case(i)
    m, poses = fixture_model(case, 'oracle')
    tr, rot, tor = score(m, poses, case['times'], 'cpu')
    assert tr.shape == case['tr'].shape and rot.shape == case['rot'].shape and tor.shape == case['tor'].shape
    for got, ref in ((tr, case['tr']), (rot, case['rot']), (tor, case['tor'])):
        if ref.numel():
            assert rel_err(got, ref) < 1e-5, rel_err(got, ref)


def test_fixture_covers_the_v10_options():
    cases = [fixture_case(i) for i in range(5)]
    kws = [c['kw'] for c in cases]
    assert {k['num_conv_layers'] for k in kws} >= {2, 3, 4}
    assert any(k['dynamic_max_cross'] for k in kws) and any(not k['dynamic_max_cross'] for k in kws)
    assert any(k['lm_embedding_type'] for k in kws) and any(not k['lm_embedding_type'] for k in kws)
    assert any(k['smooth_edges'] for k in kws) and any(k['fixed_center_conv'] for k in kws)
    assert any(k['no_torsion'] for k in kws)
    assert any(c['tor'].numel() == 0 and not c['kw']['no_torsion'] for c in cases)          # no rotatable bond
    assert any(len(set(c['times'])) > 1 for c in cases)                                   # per-complex times


def test_get_model_old_builds_the_score_model_with_the_reference_keywords(monkeypatch):
    """utils/utils.py:179-218 passes ``confidence_mode`` through unchanged, so the keywords of the v1.0 score model are those
    the reference produced for the v1.0 confidence model (ref_get_model.pt) with confidence_mode=False."""
    from diffdock_b200 import utils as U
    c = next(c for c in load_golden('ref_get_model.pt') if c['class'] == 'CGOldModel')
    made = {}

    class Recorder:
        def __init__(self, **kw):
            made.update(kw)

        def to(self, device):
            return self

    monkeypatch.setattr(U, '_model_class', lambda name: made.setdefault('_class', name) and Recorder)
    U.get_model(Namespace(**c['args']), 'cpu', t_to_sigma='T2S', no_parallel=True, old=True)
    assert made.pop('_class') == 'CGOldModel'
    for k in ('t_to_sigma', 'device', 'timestep_emb_func'):
        made.pop(k)
    assert made == dict(c['kwargs'], confidence_mode=False)


def _product(**kw):
    from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    from diffdock_b200.old_cg_model import CGOldModel
    from diffdock_b200.synthetic import default_model_args
    a = default_model_args()
    return CGOldModel(partial(t_to_sigma, args=a), torch.device('cpu'), get_timestep_embedding('sinusoidal', 8, 1000), **kw)


@pytest.mark.parametrize('i', range(5))
def test_state_dict_keys_equal_the_reference_module(i):
    """Same parameter and buffer names as the reference class; the reference's extra entries are e3nn's tensor-product
    buffers (``*.tp.*``, ``final_tp_tor.*``), which load_state_dict drops."""
    case = fixture_case(i)
    kw = dict(case['kw'])
    if case['lm_dim']:
        kw['lm_embedding_dim'] = case['lm_dim']
    ref = {k for k in fixture_state(case) if '.tp.' not in k and not k.startswith('final_tp_tor.')}
    assert set(_product(**kw).state_dict()) == ref


@pytest.mark.parametrize('bad', [dict(include_miscellaneous_atoms=True), dict(separate_noise_schedule=True),
                                 dict(asyncronous_noise_schedule=True), dict(use_second_order_repr=True),
                                 dict(use_old_atom_encoder=False)])
def test_score_mode_still_refuses_what_is_out_of_scope(bad):
    kw = dict(ns=16, nv=4, sigma_embed_dim=8, distance_embed_dim=8, cross_distance_embed_dim=8, use_old_atom_encoder=True)
    kw.update(bad)
    with pytest.raises(NotImplementedError):
        _product(**kw)


def test_all_atom_v10_model_refuses_score_mode():
    from diffdock_b200.old_aa_model import AAOldModel
    with pytest.raises(NotImplementedError):
        AAOldModel(None, torch.device('cpu'), None, ns=16, nv=4, use_old_atom_encoder=True, confidence_mode=False)

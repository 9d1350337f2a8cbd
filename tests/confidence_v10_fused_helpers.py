"""Helpers of the v1.0 confidence-model tests at fused-kernel widths: models and poses rebuilt from
tests/golden/ref_confidence_v10_fused.pt (make_golden_confidence_v10_fused.py), and seeded oracle / product pairs."""
import copy
from functools import partial

import torch

from tests.old_score_helpers import fixture_state, set_times
from tests.parity_helpers import load_golden, rand_bn_


def fixture():
    return load_golden('ref_confidence_v10_fused.pt')


def _classes(which):
    if which == 'oracle':
        from oracle.old_aa_model import AAOldModel
        from oracle.old_cg_model import CGOldModel
        from oracle.layers import get_timestep_embedding
        from oracle.diffusion import t_to_sigma
    else:
        from diffdock_b200.old_aa_model import AAOldModel
        from diffdock_b200.old_cg_model import CGOldModel
        from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    return AAOldModel, CGOldModel, get_timestep_embedding, t_to_sigma


def build(case, which):
    """('oracle' on CPU | 'product' on cuda:0 | 'product-cpu' unmoved) v1.0 confidence model of a fixture case with its
    weights, and its pose list."""
    from diffdock_b200.hetero import graph_from_dict
    from diffdock_b200.synthetic import default_model_args
    AA, CG, temb, t2s = _classes(which)
    dev = 'cpu' if which in ('oracle', 'product-cpu') else torch.device('cuda:0')
    kw = dict(case['kw'])
    if case['lm_dim']:
        kw['lm_embedding_dim'] = case['lm_dim']     # the fixture shrinks the 1280-wide LM embedding to 16 columns
    a = default_model_args()
    cls = AA if case['cls'] == 'AAOldModel' else CG
    m = cls(partial(t2s, args=a), dev, temb('sinusoidal', 8, a.embedding_scale), **kw).eval()
    m.load_state_dict(fixture_state(case), strict=True)
    return m.to(dev), [graph_from_dict(d) for d in case['poses']]


def batch_of(poses, times, device, all_atoms=False, shared=False):
    """The poses collated at per-complex ``times``; ``shared``: the sampler's collate (one receptor copy uploaded), and
    ``_uniform_t`` set when every time is the same."""
    from diffdock_b200.hetero import collate, collate_shared_receptor
    b = collate_shared_receptor(poses, device) if shared else collate(copy.deepcopy(poses)).to(device)
    set_times(b, times, device)
    t = torch.as_tensor(times, dtype=torch.float32, device=device)
    if all_atoms:
        b['atom'].node_t = {k: t[b['atom'].batch] for k in ('tr', 'rot', 'tor')}
    if shared and bool((t == t[0]).all()):
        b._uniform_t = True
    return b


def pair(cls_name, seed, **kw):
    """(oracle on CPU, product on cuda:0) v1.0 confidence models with identical seeded weights and random BatchNorm
    statistics."""
    AA_o, CG_o, temb_o, t2s_o = _classes('oracle')
    AA_p, CG_p, temb_p, t2s_p = _classes('product')
    from diffdock_b200.synthetic import default_model_args
    a = default_model_args()
    base = dict(sigma_embed_dim=16, sh_lmax=2, ns=48, nv=10, num_conv_layers=3, cross_max_distance=30.0,
                distance_embed_dim=16, cross_distance_embed_dim=16, dynamic_max_cross=True, confidence_mode=True,
                use_old_atom_encoder=True)
    base.update(kw)
    O, P = (AA_o, AA_p) if cls_name == 'AAOldModel' else (CG_o, CG_p)
    torch.manual_seed(seed)
    o = O(partial(t2s_o, args=a), 'cpu', temb_o('sinusoidal', base['sigma_embed_dim'], 1000), **base).eval()
    g = torch.Generator().manual_seed(seed + 1)
    for mod in o.modules():
        if mod.__class__.__name__ in ('BatchNorm', 'BatchNorm1d'):
            rand_bn_(mod, g)
    p = P(partial(t2s_p, args=a), torch.device('cuda:0'), temb_p('sinusoidal', base['sigma_embed_dim'], 1000), **base).eval()
    p.load_state_dict(o.state_dict(), strict=True)
    return o, p.to('cuda:0')

"""Helpers of the v1.0 score-model tests (CGOldModel with confidence_mode=False): models rebuilt from the
ref_old_score_model.pt fixture or made as seeded oracle / product pairs, and per-complex diffusion times."""
import copy
from functools import partial

import torch

from tests.parity_helpers import load_golden, rand_bn_


def generated(key):
    """Entries of the reference state_dict the fixture draws from a seed instead of storing: the parameters and the
    BatchNorm statistics; the RBF offsets and e3nn's tensor-product buffers are stored as they are."""
    return not ('.tp.' in key or key.startswith('final_tp_tor.') or key.endswith('offset')
                or key.endswith('num_batches_tracked'))


def seeded_values(shapes, seed):
    """``{key: tensor}`` for ``shapes`` = ``{key: shape}``, drawn in sorted key order from one seeded generator: Linear and
    embedding weights uniform in +-1/sqrt(fan_in), biases in +-0.1, non-trivial eval-mode BatchNorm statistics."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k in sorted(shapes):
        shape = tuple(shapes[k])
        if k.endswith('running_mean'):
            v = 0.1 * torch.randn(shape, generator=g)
        elif k.endswith('running_var'):
            v = 0.5 + torch.rand(shape, generator=g)
        elif 'batch_norm.' in k and k.endswith('weight'):
            v = 1.0 + 0.2 * torch.randn(shape, generator=g)
        else:
            bound = shape[1] ** -0.5 if len(shape) == 2 else 0.1
            v = (2 * torch.rand(shape, generator=g) - 1) * bound
        out[k] = v
    return out


def fixture_state(case):
    """The reference-keyed state_dict of a ref_old_score_model.pt case: stored buffers + seeded parameters."""
    return dict(case['fixed'], **seeded_values(case['shapes'], case['seed']))


def set_times(batch, t, device='cpu'):
    """One diffusion time per complex (``t`` [B]) on every node and graph: utils/diffusion_utils.py:146-168 with per-graph
    instead of per-batch times, as tests/golden/make_golden_old_score.py sets them."""
    t = torch.as_tensor(t, dtype=torch.float32, device=device)
    for nt in ('ligand', 'receptor'):
        batch[nt].node_t = {k: t[batch[nt].batch] for k in ('tr', 'rot', 'tor')}
    batch.complex_t = {k: t.clone() for k in ('tr', 'rot', 'tor')}


def fixture_model(case, which):
    """('oracle' on CPU | 'product' on cuda:0) v1.0 score model with the fixture's weights, and its pose list."""
    from diffdock_b200.hetero import graph_from_dict
    from diffdock_b200.synthetic import default_model_args
    if which == 'oracle':
        from tests.old_score_oracle import CGOldScoreModel as CGOldModel
        from oracle.layers import get_timestep_embedding
        from oracle.diffusion import t_to_sigma
        dev = 'cpu'
    else:
        from diffdock_b200.old_cg_model import CGOldModel
        from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
        dev = torch.device('cuda:0')
    a = default_model_args()
    kw = dict(case['kw'])
    if case['lm_dim']:
        kw['lm_embedding_dim'] = case['lm_dim']     # the fixture shrinks the 1280-wide LM embedding to 16 columns
    m = CGOldModel(partial(t_to_sigma, args=a), dev, get_timestep_embedding('sinusoidal', 8, a.embedding_scale), **kw).eval()
    m.load_state_dict(fixture_state(case), strict=True)
    return m.to(dev), [graph_from_dict(d) for d in case['poses']]


def fixture_case(i):
    return load_golden('ref_old_score_model.pt')[i]


def score(model, poses, times, device, shared=False):
    """(tr, rot, tor) on the CPU for ``poses`` at per-complex ``times``.  ``shared``: the sampler's collate of N poses of one
    complex at one time (receptor stored once, ``_uniform_t`` set)."""
    from diffdock_b200.hetero import collate, collate_shared_receptor
    if shared:
        b = collate_shared_receptor(copy.deepcopy(poses), device)
        b._uniform_t = True
    else:
        b = collate(copy.deepcopy(poses)).to(device)
    set_times(b, times, device)
    with torch.no_grad():
        out = model(b)
    return tuple(o.float().cpu() for o in out)


def model_pair(seed=0, ns=48, nv=10, num_conv_layers=6, sigma_embed_dim=64, distance_embed_dim=64, lm_dim=1280, **extra):
    """(oracle on CPU, product on cuda:0) v1.0 score models with identical seeded weights and non-trivial BatchNorm
    statistics; default widths are the v1.0 training flags (CFG-L2, SURVEY.md section 8)."""
    from oracle.diffusion import t_to_sigma as o_t2s
    from oracle.layers import get_timestep_embedding as o_temb
    from tests.old_score_oracle import CGOldScoreModel as OModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    from diffdock_b200.old_cg_model import CGOldModel
    from diffdock_b200.synthetic import default_model_args
    a = default_model_args()
    kw = dict(sigma_embed_dim=sigma_embed_dim, sh_lmax=2, ns=ns, nv=nv, num_conv_layers=num_conv_layers,
              lig_max_radius=5.0, rec_max_radius=30.0, cross_max_distance=80.0, distance_embed_dim=distance_embed_dim,
              cross_distance_embed_dim=distance_embed_dim, dynamic_max_cross=True, confidence_mode=False,
              use_old_atom_encoder=True, lm_embedding_type='esm' if lm_dim else None)
    if lm_dim:
        kw['lm_embedding_dim'] = lm_dim
    kw.update(extra)
    torch.manual_seed(seed)
    o = OModel(partial(o_t2s, args=a), 'cpu', o_temb('sinusoidal', sigma_embed_dim, a.embedding_scale), **kw).eval()
    g = torch.Generator().manual_seed(seed + 1)
    for mod in o.modules():
        if mod.__class__.__name__ in ('BatchNorm', 'BatchNorm1d'):
            rand_bn_(mod, g)
    p = CGOldModel(partial(t_to_sigma, args=a), torch.device('cuda:0'),
                   get_timestep_embedding('sinusoidal', sigma_embed_dim, a.embedding_scale), **kw).eval()
    p.load_state_dict(o.state_dict(), strict=True)
    return o, p.to('cuda:0'), a

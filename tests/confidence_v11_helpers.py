"""Helpers of the v1.1 confidence-model tests: models and poses rebuilt from tests/golden/ref_confidence_v11.pt
(make_golden_confidence_v11.py), and a float64 restatement of the confidence head."""
import copy

import torch

from tests.old_score_helpers import fixture_state, set_times
from tests.parity_helpers import load_golden


def fixture():
    return load_golden('ref_confidence_v11.pt')


def build(case, which, t_to_sigma=None):
    """('oracle' on CPU | 'product' on cuda:0 | 'product-cpu' unmoved) confidence model of a fixture case with its weights,
    and its pose list.  The confidence trainer passes ``t_to_sigma=None``."""
    from diffdock_b200.hetero import graph_from_dict
    if which == 'oracle':
        from tests.confidence_v11_oracle import AAConfidenceModel as AA, CGConfidenceModel as CG
        from oracle.layers import get_timestep_embedding
        dev = 'cpu'
    else:
        from diffdock_b200.aa_model import AAModel as AA
        from diffdock_b200.cg_model import CGModel as CG
        from diffdock_b200.diffusion_utils import get_timestep_embedding
        dev = torch.device('cuda:0') if which == 'product' else 'cpu'
    cls = AA if case['cls'] == 'AAModel' else CG
    m = cls(t_to_sigma, dev, get_timestep_embedding('sinusoidal', 8, case['args']['embedding_scale']), **case['kw']).eval()
    m.load_state_dict(fixture_state(case), strict=True)
    return m.to(dev), [graph_from_dict(d) for d in case['poses']]


def batch_of(poses, times, device, all_atoms=False):
    from diffdock_b200.hetero import collate
    b = collate(copy.deepcopy(poses)).to(device)
    set_times(b, times, device)
    if all_atoms:
        t = torch.as_tensor(times, dtype=torch.float32, device=device)
        b['atom'].node_t = {k: t[b['atom'].batch] for k in ('tr', 'rot', 'tor')}
    return b


def head_f64(lig_node, lig_ptr, n_head, n_tail, head, atom_head=None, n_atom_out=0):
    """The confidence head in float64 from the nn.Sequential modules: ``(confidence [B, k], atom_confidence | None)``."""
    with torch.no_grad():
        return _head_f64(lig_node, lig_ptr, n_head, n_tail, head, atom_head, n_atom_out)


def _head_f64(lig_node, lig_ptr, n_head, n_tail, head, atom_head, n_atom_out):
    x = lig_node.double().cpu()
    s = torch.cat([x[:, :n_head], x[:, x.shape[1] - n_tail:]], 1) if n_tail else x[:, :n_head]
    atom = None
    if atom_head is not None:
        s = copy.deepcopy(atom_head).double().cpu()(s)
        atom, s = s[:, :n_atom_out], s[:, n_atom_out:]
    ptr = lig_ptr.long().cpu().tolist()
    pooled = torch.stack([s[a:b].sum(0) / max(b - a, 1) for a, b in zip(ptr[:-1], ptr[1:])])
    return copy.deepcopy(head).double().cpu()(pooled), atom

"""Shared pieces of the visualisation-frame tests and their fixture generator: a recording stand-in for the caller's
``utils/visualise.py:PDBFile``, pre-populated as inference.py does, and the fixture's models."""
from collections import defaultdict
from functools import partial

import torch

# 4 poses in 2 batches: the reference cannot sample a partial last batch with a stochastic or a no_random step (it draws
# min(batch_size, N) rows of tr / rot noise, which meet a smaller batch in a bmm, utils/diffusion_utils.py:69)
N_POSES, BATCH_SIZE = 4, 2


class RecordingPDB:
    """``PDBFile.add(coords, order, part=0, repeat=1)`` without RDKit: ``parts[part][order]`` keeps what the last ``add``
    for that slot was given, as ``PDBFile.parts`` keeps the PDB block made from it."""

    def __init__(self):
        self.parts = defaultdict(dict)

    def add(self, coords, order, part=0, repeat=1):
        self.parts[part][order] = coords.clone() if torch.is_tensor(coords) else coords

    def content(self):
        return {p: dict(o) for p, o in self.parts.items()}


def prepopulated(poses, crystal):
    """One recorder per pose with what inference.py:248-255 adds before ``sampling``: the molecule (a placeholder here),
    the input ligand and the pose's prior sample, each + ``original_center``.  ``crystal`` [n_atoms, 3]: the input ligand."""
    out = []
    for g in poses:
        center = g.original_center.detach().cpu()
        r = RecordingPDB()
        r.add('molecule', 0, 0)
        r.add(crystal + center, 1, 0)
        r.add((g['ligand'].pos + g.original_center).detach().cpu(), part=1, order=1)
        out.append(r)
    return out


def original_centers(n):
    """The ``original_center`` [1, 3] of each fixture pose: distinct per pose, so a frame added with another pose's centre
    shows."""
    return [torch.tensor([[12.5 + 3.0 * i, -33.25 + i, 7.75 - 2.0 * i]]) for i in range(n)]


def max_rel_diff(got, ref):
    """Largest |got - ref| / max |ref| over the coordinate entries of two ``content()`` dicts (inf when the part / order
    slots differ); non-tensor entries must be equal."""
    worst = 0.0
    if got.keys() != ref.keys():
        return float('inf')
    for p in ref:
        if got[p].keys() != ref[p].keys():
            return float('inf')
        for o, r in ref[p].items():
            g = got[p][o]
            if not torch.is_tensor(r):
                if g != r:
                    return float('inf')
                continue
            if not torch.is_tensor(g) or g.shape != r.shape:
                return float('inf')
            worst = max(worst, float((g.double() - r.double()).abs().max() / r.double().abs().max().clamp_min(1e-30)))
    return worst


def fused_case_model(case, device='cuda:0'):
    """The product CGModel of the fixture's ns=16 / nv=4 case (parameters drawn from the stored seed,
    tests/old_score_helpers.py:fixture_state), with its 16-wide LM embedding layer."""
    from argparse import Namespace
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    from tests.old_score_helpers import fixture_state
    a = Namespace(**case['args'])
    m = CGModel(partial(t_to_sigma, args=a), torch.device(device),
                get_timestep_embedding('sinusoidal', case['kw']['sigma_embed_dim'], a.embedding_scale), **case['kw']).eval()
    ns = case['kw']['ns']
    m.rec_node_embedding.additional_features_dim = case['lm_dim']
    m.rec_node_embedding.additional_features_embedder = torch.nn.Linear(case['lm_dim'] + ns, ns)
    m.load_state_dict(fixture_state(case), strict=True)
    return m.to(device), a

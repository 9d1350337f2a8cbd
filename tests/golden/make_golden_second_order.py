"""Golden vectors for score models built with ``use_second_order_repr`` (node irreps with ``nv x2e`` / ``nv x2o`` blocks):
runs the UNMODIFIED reference models/cg_model.py and utils/sampling.py from a checkout of the reference DiffDock code base,
with the third-party packages supplied by oracle/ref_shims.py.  The so3/torus tables take about 1.5 minutes at import; run
it from a scratch working directory (utils/so3.py writes its .npy caches there):

    cd <scratch dir> && DIFFDOCK_REFERENCE=<reference checkout> python <this repository>/tests/golden/make_golden_second_order.py

The model parameters and BatchNorm statistics are drawn from a seed (tests/old_score_helpers.py:seeded_values) and only
the seed, the shapes and the remaining buffers are stored, which keeps the fixture small.  All cases have fused-kernel
widths (ns=16, nv=4), so the l = 2 blocks are ``4x2e`` / ``4x2o``.

Fixture ref_cg_model_so.pt, a dict:
  cases     CGModel.forward in score mode, all with use_second_order_repr and embed_also_ligand:
              (a) sh_lmax=2, four conv layers, a 16-wide LM embedding
              (b) sh_lmax=1, reduce_pseudoscalars, num_prot_emb_layers=1, three conv layers
              (c) sh_lmax=2, no_torsion, three conv layers
  sampling  utils/sampling.py: 4 reverse-diffusion steps of case (a) with crop_beyond=12 on a late schedule (the cut-off
            3 sigma_tr + 12 A keeps part of the receptor for two of the three poses); seeded CPU noise
            (torch.manual_seed(seed) then torch.normal in the reference's order), which the GPU test replays through
            ``noise_fn``
"""
import copy
import os
import sys
from argparse import Namespace
from functools import partial

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402

ref_shims.install()
sys.path.insert(0, os.environ['DIFFDOCK_REFERENCE'])
import models.cg_model as r_cg              # noqa: E402
import utils.diffusion_utils as r_du        # noqa: E402
import utils.sampling as r_sampling         # noqa: E402
import utils.utils as r_utils               # noqa: E402
from utils import torus as r_torus          # noqa: E402

from diffdock_b200.hetero import collate, graph_to_dict   # noqa: E402
from diffdock_b200.synthetic import default_model_args, make_pose_list   # noqa: E402
from tests.old_score_helpers import generated, seeded_values    # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
torch.set_num_threads(4)
# the stored Monte-Carlo torus table instance, shared with the product and the oracle (the import above re-drew it)
r_torus.score_norm_ = np.load(os.path.join(ROOT, 'diffdock_b200', 'tables', 'score_norm_tables.npz'))['torus_score_norm']
NS, NV, LM = 16, 4, 16


def compact(d):
    """A pose dict whose tensors own exactly their data (torch.save writes a view's whole storage)."""
    if isinstance(d, dict):
        return {k: compact(v) for k, v in d.items()}
    return d.clone() if torch.is_tensor(d) else d


def build(c):
    """The reference CGModel of a case dict (``kw``, ``args``, ``lm_dim``) with the fixture's 16-wide LM layer."""
    a = Namespace(**c['args'])
    model = r_cg.CGModel(partial(r_du.t_to_sigma, args=a), torch.device('cpu'),
                         r_du.get_timestep_embedding('sinusoidal', 8, a.embedding_scale), **c['kw']).eval()
    if c['lm_dim']:   # shrink the LM embedding (1280 -> 16) to keep the fixture small: patch the encoder's input Linear
        model.rec_node_embedding.additional_features_dim = c['lm_dim']
        model.rec_node_embedding.additional_features_embedder = torch.nn.Linear(c['lm_dim'] + NS, NS)
    return model


def case(seed, t, sh_lmax, lm=True, num_prot_emb_layers=0, layers=3, **flags):
    a = default_model_args(ns=NS, nv=NV, sh_lmax=sh_lmax, num_conv_layers=layers, use_second_order_repr=True,
                           distance_embed_dim=8, cross_distance_embed_dim=8, sigma_embed_dim=8,
                           num_prot_emb_layers=num_prot_emb_layers, **flags)
    kw = dict(sigma_embed_dim=8, sh_lmax=sh_lmax, ns=NS, nv=NV, num_conv_layers=layers, lig_max_radius=a.max_radius,
              rec_max_radius=a.rec_max_radius, cross_max_distance=a.cross_max_distance,
              center_max_distance=a.center_max_distance, distance_embed_dim=8, cross_distance_embed_dim=8,
              dynamic_max_cross=True, lm_embedding_type='precomputed' if lm else None, embed_also_ligand=True,
              num_prot_emb_layers=num_prot_emb_layers, differentiate_convolutions=a.differentiate_convolutions,
              reduce_pseudoscalars=a.reduce_pseudoscalars, odd_parity=a.odd_parity, smooth_edges=a.smooth_edges,
              no_torsion=a.no_torsion, use_second_order_repr=True)
    c = dict(args=vars(a), kw=kw, lm_dim=LM if lm else 0, t=t)
    torch.manual_seed(seed)
    model = build(c)
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items() if generated(k)}
    missing, unexpected = model.load_state_dict(seeded_values(shapes, seed + 1), strict=False)
    assert not unexpected and all(not generated(k) for k in missing)
    fixed = {k: v.clone() for k, v in model.state_dict().items() if not generated(k)}
    poses = make_pose_list(3, n_res=24, n_atoms=9, seed=seed + 2, tr_sigma_max=a.tr_sigma_max * t, lm_dim=LM if lm else 0)
    batch = collate(copy.deepcopy(poses))
    r_du.set_time(batch, t, t, t, t, len(poses), False, 'cpu')
    with torch.no_grad():
        tr, rot, tor, _ = model(batch)
    print('case', seed, 'tr', tr[0].tolist(), 'tor', tuple(tor.shape))
    c.update(fixed=fixed, shapes=shapes, seed=seed + 1, poses=[compact(graph_to_dict(p)) for p in poses], tr=tr, rot=rot, tor=tor)
    return c, model, poses


ca, ma, pa = case(70, 0.45, 2, layers=4)
cb, _, _ = case(71, 0.7, 1, lm=False, num_prot_emb_layers=1, reduce_pseudoscalars=True)
cc, _, _ = case(72, 0.3, 2, lm=False, no_torsion=True)

# ------------------------------------------------------------------------------------------------ cropped sampling
kept = []
_orig_crop = r_utils.crop_beyond


def _spy(graph, cutoff, all_atoms):
    _orig_crop(graph, cutoff, all_atoms)
    kept.append(int(graph['receptor'].pos.shape[0]))


r_sampling.crop_beyond = _spy
margs = Namespace(**ca['args'])
steps, seed, CROP = 4, 551, 12.0
margs.crop_beyond = CROP
sched = np.array([0.30, 0.22, 0.15, 0.08])     # late, small-sigma steps: the cut-off 3*sigma_tr + 7 A crops partially
torch.manual_seed(seed)
out_list, _ = r_sampling.sampling(data_list=copy.deepcopy(pa), model=ma, inference_steps=steps, tr_schedule=sched,
                                  rot_schedule=sched, tor_schedule=sched, device=torch.device('cpu'),
                                  t_to_sigma=partial(r_du.t_to_sigma, args=Namespace(**ca['args'])), model_args=margs,
                                  batch_size=3, no_final_step_noise=True, temp_sampling=[1.17, 2.06, 7.04],
                                  temp_psi=[0.73, 0.90, 0.59], temp_sigma_data=[0.93, 0.75, 0.69])
print('residues kept per (step, pose):', kept)
assert 0 < min(kept) < 24     # no pose loses its whole receptor, some lose part of it
sampling = dict(model_case=0, steps=steps, seed=seed, schedule=sched, crop_beyond=CROP, kept=kept,
                temp_sampling=[1.17, 2.06, 7.04], temp_psi=[0.73, 0.90, 0.59], temp_sigma_data=[0.93, 0.75, 0.69],
                final_pos=[d['ligand'].pos.clone() for d in out_list])
torch.save(dict(cases=[ca, cb, cc], sampling=sampling), os.path.join(OUT, 'ref_cg_model_so.pt'))
print('ref_cg_model_so.pt', os.path.getsize(os.path.join(OUT, 'ref_cg_model_so.pt')) // 1024, 'KiB')

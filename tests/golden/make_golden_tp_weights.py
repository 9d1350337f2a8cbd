"""Golden vectors for score models built with ``tp_weights_layers`` > 2 (DiffDock-L's ``--tp_weights_layers``: every
receptor-embedding, ligand-embedding and interaction convolution builds its radial MLP with that many Linear layers, the
extra ones H x H): runs the UNMODIFIED reference models/cg_model.py, models/aa_model.py and utils/sampling.py from a
checkout of the reference DiffDock code base, with the third-party packages supplied by oracle/ref_shims.py.  The
so3/torus tables take about 1.5 minutes at import; run it from a scratch working directory (utils/so3.py writes its .npy
caches there):

    cd <scratch dir> && DIFFDOCK_REFERENCE=<reference checkout> python <this repository>/tests/golden/make_golden_tp_weights.py

The model parameters and BatchNorm statistics are drawn from a seed (tests/old_score_helpers.py:seeded_values) and only
the seed, the shapes and the remaining buffers are stored, which keeps the fixture small.  All cases have fused-kernel
widths (ns=16, nv=4).

Fixture ref_cg_model_tw.pt, a dict:
  cases     forward in score mode, ``model`` = 'cg' (CGModel) or 'aa' (AAModel), all with embed_also_ligand:
              (a) cg, tp_weights_layers=3, sh_lmax=2, three conv layers, a 16-wide LM embedding
              (b) cg, tp_weights_layers=4, sh_lmax=1, reduce_pseudoscalars, num_prot_emb_layers=1, one edge group per
                  convolution (the reference runs sh_lmax=1 on FasterTensorProduct, which its multi-group scatter cannot
                  take)
              (c) cg, tp_weights_layers=3, use_second_order_repr, sh_lmax=2
              (d) aa, tp_weights_layers=3, sh_lmax=2, num_prot_emb_layers=1
  sampling  utils/sampling.py: 4 reverse-diffusion steps of case (a) with crop_beyond=12 on a late schedule (the cut-off
            keeps part of the receptor for some poses); seeded CPU noise (torch.manual_seed(seed) then torch.normal in the
            reference's order), which the GPU test replays through ``noise_fn``
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
import models.aa_model as r_aa              # noqa: E402
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
    """The reference model of a case dict (``model``, ``kw``, ``args``, ``lm_dim``) with the fixture's 16-wide LM layer."""
    a = Namespace(**c['args'])
    cls = r_aa.AAModel if c['model'] == 'aa' else r_cg.CGModel
    model = cls(partial(r_du.t_to_sigma, args=a), torch.device('cpu'),
                r_du.get_timestep_embedding('sinusoidal', 8, a.embedding_scale), **c['kw']).eval()
    if c['lm_dim']:   # shrink the LM embedding (1280 -> 16) to keep the fixture small: patch the encoder's input Linear
        model.rec_node_embedding.additional_features_dim = c['lm_dim']
        model.rec_node_embedding.additional_features_embedder = torch.nn.Linear(c['lm_dim'] + NS, NS)
    return model


def case(seed, t, sh_lmax, tp_weights_layers, model='cg', lm=True, num_prot_emb_layers=0, layers=3, **flags):
    a = default_model_args(ns=NS, nv=NV, sh_lmax=sh_lmax, num_conv_layers=layers, distance_embed_dim=8,
                           cross_distance_embed_dim=8, sigma_embed_dim=8, num_prot_emb_layers=num_prot_emb_layers,
                           tp_weights_layers=tp_weights_layers, **flags)
    kw = dict(sigma_embed_dim=8, sh_lmax=sh_lmax, ns=NS, nv=NV, num_conv_layers=layers, lig_max_radius=a.max_radius,
              rec_max_radius=a.rec_max_radius, cross_max_distance=a.cross_max_distance,
              center_max_distance=a.center_max_distance, distance_embed_dim=8, cross_distance_embed_dim=8,
              dynamic_max_cross=True, lm_embedding_type='precomputed' if lm else None, embed_also_ligand=True,
              num_prot_emb_layers=num_prot_emb_layers, differentiate_convolutions=a.differentiate_convolutions,
              tp_weights_layers=tp_weights_layers)
    if model == 'cg':
        kw.update(reduce_pseudoscalars=a.reduce_pseudoscalars, odd_parity=a.odd_parity, smooth_edges=a.smooth_edges,
                  no_torsion=a.no_torsion, use_second_order_repr=a.use_second_order_repr)
    c = dict(model=model, args=vars(a), kw=kw, lm_dim=LM if lm else 0, t=t)
    torch.manual_seed(seed)
    m = build(c)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items() if generated(k)}
    missing, unexpected = m.load_state_dict(seeded_values(shapes, seed + 1), strict=False)
    assert not unexpected and all(not generated(k) for k in missing)
    # the extra hidden layers exist: fc.{0, 3, ..., 3 (L - 1)} are Linear layers of every convolution's radial MLP
    assert any(k.endswith(f'fc.{3 * (tp_weights_layers - 1)}.weight') or f'fc.0.{3 * (tp_weights_layers - 1)}.weight' in k
               for k in shapes)
    fixed = {k: v.clone() for k, v in m.state_dict().items() if not generated(k)}
    all_atoms = model == 'aa'
    poses = make_pose_list(3, n_res=24, n_atoms=9, seed=seed + 2, tr_sigma_max=a.tr_sigma_max * t, lm_dim=LM if lm else 0,
                           all_atoms=all_atoms)
    batch = collate(copy.deepcopy(poses))
    r_du.set_time(batch, t, t, t, t, len(poses), all_atoms, 'cpu')
    with torch.no_grad():
        tr, rot, tor, _ = m(batch)
    print('case', seed, model, 'tr', tr[0].tolist(), 'tor', tuple(tor.shape))
    c.update(fixed=fixed, shapes=shapes, seed=seed + 1, poses=[compact(graph_to_dict(p)) for p in poses], tr=tr, rot=rot, tor=tor)
    return c, m, poses


ca, ma, pa = case(80, 0.45, 2, 3)
cb, _, _ = case(81, 0.7, 1, 4, lm=False, num_prot_emb_layers=1, reduce_pseudoscalars=True,
                differentiate_convolutions=False)
cc, _, _ = case(82, 0.3, 2, 3, lm=False, use_second_order_repr=True)
cd, _, _ = case(83, 0.4, 2, 3, model='aa', lm=False, num_prot_emb_layers=1)

# ------------------------------------------------------------------------------------------------ cropped sampling
kept = []
_orig_crop = r_utils.crop_beyond


def _spy(graph, cutoff, all_atoms):
    _orig_crop(graph, cutoff, all_atoms)
    kept.append(int(graph['receptor'].pos.shape[0]))


r_sampling.crop_beyond = _spy
margs = Namespace(**ca['args'])
steps, seed, CROP = 4, 561, 12.0
margs.crop_beyond = CROP
sched = np.array([0.30, 0.22, 0.15, 0.08])     # late, small-sigma steps: the cut-off 3 sigma_tr + 12 A crops partially
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
torch.save(dict(cases=[ca, cb, cc, cd], sampling=sampling), os.path.join(OUT, 'ref_cg_model_tw.pt'))
print('ref_cg_model_tw.pt', os.path.getsize(os.path.join(OUT, 'ref_cg_model_tw.pt')) // 1024, 'KiB')

"""Golden vectors for the v1.0 confidence models at fused-kernel widths (ns=16, nv=4): ``CGOldModel`` and ``AAOldModel`` in
confidence mode, the ranking models ``inference.py`` builds by default (``--old_confidence_model``).  Runs the UNMODIFIED
reference models/old_cg_model.py, models/old_aa_model.py and utils/sampling.py from a checkout of the reference DiffDock
code base, with the third-party packages supplied by oracle/ref_shims.py.  The so3/torus tables take about 1.5 minutes at
import; run it from a scratch working directory (utils/so3.py writes its .npy caches there):

    cd <scratch dir> && DIFFDOCK_REFERENCE=<reference checkout> python <this repository>/tests/golden/make_golden_confidence_v10_fused.py

Parameters are drawn from a seed (tests/old_score_helpers.py:seeded_values); the BatchNorm1d layers of the confidence head
get rand_bn_ statistics and are stored with the other fixed entries.  A case with an LM embedding shrinks it from 1280 to
16 columns (``lm_dim``), as the other v1.0 fixtures do.

Fixture ref_confidence_v10_fused.pt, a dict:
  cases     forward in confidence mode at per-complex times t (the times are the sigmas), ``confidence``:
              (0) CGOldModel, 2 layers, LM embedding
              (1) CGOldModel, 3 layers, dynamic_max_cross, smooth_edges, affinity_prediction
              (2) AAOldModel, 2 layers, LM embedding
              (3) AAOldModel, 4 layers, dynamic_max_cross, affinity_prediction
  sampling  utils/sampling.py: 3 reverse-diffusion steps of a CGModel score model, ranked by case (2)'s AAOldModel on an
            all-atom confidence_data_list; seeded CPU noise (torch.manual_seed(seed), the reference's order)
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
sys.path.insert(0, os.environ.get('DIFFDOCK_REFERENCE', '/root/reference'))
import models.cg_model as r_cg              # noqa: E402
import models.old_aa_model as r_old_aa      # noqa: E402
import models.old_cg_model as r_old_cg      # noqa: E402
import utils.diffusion_utils as r_du        # noqa: E402
import utils.sampling as r_sampling         # noqa: E402
from utils import torus as r_torus          # noqa: E402

from diffdock_b200.hetero import collate, graph_to_dict   # noqa: E402
from diffdock_b200.synthetic import default_model_args, make_pose_list   # noqa: E402
from tests.old_score_helpers import generated, seeded_values, set_times    # noqa: E402
from tests.parity_helpers import rand_bn_    # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
torch.set_num_threads(4)
r_torus.score_norm_ = np.load(os.path.join(ROOT, 'diffdock_b200', 'tables', 'score_norm_tables.npz'))['torus_score_norm']
NS, NV, LM = 16, 4, 16


def compact(d):
    if isinstance(d, dict):
        return {k: compact(v) for k, v in d.items()}
    return d.clone() if torch.is_tensor(d) else d


def seeded(model, seed):
    """Seeded parameters, rand_bn_ on the BatchNorm1d layers of the head: ``(fixed, shapes)``."""
    bn1d = {n for n, m in model.named_modules() if isinstance(m, torch.nn.BatchNorm1d)}
    is_bn1d = lambda k: k.rsplit('.', 1)[0] in bn1d
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items() if generated(k) and not is_bn1d(k)}
    _, unexpected = model.load_state_dict(seeded_values(shapes, seed), strict=False)
    assert not unexpected
    g = torch.Generator().manual_seed(seed + 7)
    for n in sorted(bn1d):
        rand_bn_(model.get_submodule(n), g)
    fixed = {k: v.clone() for k, v in model.state_dict().items() if not (generated(k) and not is_bn1d(k))}
    return fixed, shapes


def case(seed, cls, times, num_conv_layers, lm=False, dynamic=False, smooth=False, affinity=False):
    a = default_model_args()
    all_atoms = cls is r_old_aa.AAOldModel
    kw = dict(sigma_embed_dim=8, sh_lmax=2, ns=NS, nv=NV, num_conv_layers=num_conv_layers, lig_max_radius=5.0,
              rec_max_radius=30.0, cross_max_distance=25.0, distance_embed_dim=8, cross_distance_embed_dim=8,
              dynamic_max_cross=dynamic, smooth_edges=smooth, lm_embedding_type='esm' if lm else None,
              confidence_mode=True, use_old_atom_encoder=True, affinity_prediction=affinity)
    torch.manual_seed(seed)
    model = cls(partial(r_du.t_to_sigma, args=a), torch.device('cpu'),
                r_du.get_timestep_embedding('sinusoidal', 8, a.embedding_scale), **kw).eval()
    if lm:       # shrink the LM embedding (1280 -> 16) to keep the fixture small
        model.rec_node_embedding.lm_embedding_dim = LM
        model.rec_node_embedding.lm_embedding_layer = torch.nn.Linear(LM + NS, NS)
    fixed, shapes = seeded(model, seed + 1)
    poses = make_pose_list(len(times), n_res=20, n_atoms=9, seed=seed + 2, tr_sigma_max=1.5, lm_dim=LM if lm else 0,
                           all_atoms=all_atoms)
    batch = collate(copy.deepcopy(poses))
    set_times(batch, times)
    if all_atoms:
        batch['atom'].node_t = {k: torch.as_tensor(times, dtype=torch.float32)[batch['atom'].batch]
                                for k in ('tr', 'rot', 'tor')}
    with torch.no_grad():
        conf = model(batch)
    print('case', seed, cls.__name__, 'confidence', conf.tolist())
    c = dict(cls=cls.__name__, args=vars(a), kw=kw, lm_dim=LM if lm else 0, times=torch.as_tensor(times, dtype=torch.float32),
             fixed=fixed, shapes=shapes, seed=seed + 1, all_atoms=all_atoms,
             poses=[compact(graph_to_dict(p)) for p in poses], confidence=conf)
    return c, model, poses


c0, _, _ = case(90, r_old_cg.CGOldModel, [0.0, 0.3, 0.7], 2, lm=True)
c1, _, _ = case(91, r_old_cg.CGOldModel, [0.1, 0.0, 0.9], 3, dynamic=True, smooth=True, affinity=True)
c2, m2, p2 = case(92, r_old_aa.AAOldModel, [0.0, 0.45, 0.2], 2, lm=True)
c3, _, _ = case(93, r_old_aa.AAOldModel, [0.6, 0.0, 0.15], 4, dynamic=True, affinity=True)
cases = [c0, c1, c2, c3]
assert c1['confidence'].shape == (3, 2) and c3['confidence'].shape == (3, 2) and c2['confidence'].shape == (3,)

# ---------------------------------------------------------------------------------------- sampling ranked by AAOldModel
sa = default_model_args(ns=NS, nv=NV, num_conv_layers=2, sh_lmax=2)
skw = dict(sigma_embed_dim=8, sh_lmax=2, ns=NS, nv=NV, num_conv_layers=2, lig_max_radius=sa.max_radius,
           rec_max_radius=sa.rec_max_radius, cross_max_distance=sa.cross_max_distance,
           center_max_distance=sa.center_max_distance, distance_embed_dim=8, cross_distance_embed_dim=8,
           dynamic_max_cross=sa.dynamic_max_cross, lm_embedding_type=None, embed_also_ligand=True,
           num_prot_emb_layers=sa.num_prot_emb_layers, reduce_pseudoscalars=sa.reduce_pseudoscalars,
           smooth_edges=sa.smooth_edges, tp_weights_layers=sa.tp_weights_layers)
torch.manual_seed(95)
score = r_cg.CGModel(partial(r_du.t_to_sigma, args=sa), torch.device('cpu'),
                     r_du.get_timestep_embedding('sinusoidal', 8, sa.embedding_scale), **skw).eval()
s_fixed, s_shapes = seeded(score, 96)
poses = make_pose_list(3, n_res=20, n_atoms=9, seed=97, tr_sigma_max=sa.tr_sigma_max * 0.3, lm_dim=0)
conf_list = []                      # the ranking model's all-atom graphs of case (2)'s complex, with the score model's ligand
for p, q in zip(poses, p2):
    c = copy.deepcopy(q)
    for k in ('x', 'pos', 'edge_mask', 'mask_rotate'):
        setattr(c['ligand'], k, copy.deepcopy(getattr(p['ligand'], k)))
    c['ligand', 'ligand'].edge_index = p['ligand', 'ligand'].edge_index.clone()
    c['ligand', 'ligand'].edge_attr = p['ligand', 'ligand'].edge_attr.clone()
    conf_list.append(c)
steps, seed = 3, 463
sched = np.array([0.30, 0.18, 0.08])
torch.manual_seed(seed)
out_list, confidence = r_sampling.sampling(
    data_list=copy.deepcopy(poses), model=score, inference_steps=steps, tr_schedule=sched, rot_schedule=sched,
    tor_schedule=sched, device=torch.device('cpu'), t_to_sigma=partial(r_du.t_to_sigma, args=sa), model_args=Namespace(**vars(sa)),
    batch_size=3, no_final_step_noise=True, confidence_model=m2, confidence_data_list=copy.deepcopy(conf_list),
    confidence_model_args=Namespace(all_atoms=True, crop_beyond=None))
print('sampling confidence', confidence)
sampling = dict(score=dict(args=vars(sa), kw=skw, fixed=s_fixed, shapes=s_shapes, seed=96), confidence_case=2,
                poses=[compact(graph_to_dict(p)) for p in poses], conf_poses=[compact(graph_to_dict(p)) for p in conf_list],
                steps=steps, seed=seed, schedule=sched, confidence=confidence,
                final_pos=[d['ligand'].pos.clone() for d in out_list])

torch.save(dict(cases=cases, sampling=sampling), os.path.join(OUT, 'ref_confidence_v10_fused.pt'))
print('ref_confidence_v10_fused.pt', os.path.getsize(os.path.join(OUT, 'ref_confidence_v10_fused.pt')) // 1024, 'KiB')

"""Golden vectors for the v1.0 score model: runs the UNMODIFIED reference models/old_cg_model.py (CGOldModel with
confidence_mode=False, the model ``inference.py --old_score_model`` builds) from a checkout of the reference DiffDock
code base, with the third-party packages supplied by oracle/ref_shims.py.  The so3/torus tables take about 1.5 minutes at
import; run it from a scratch working directory (utils/so3.py writes its .npy caches there):

    cd <scratch dir> && DIFFDOCK_REFERENCE=<reference checkout> python <this repository>/tests/golden/make_golden_old_score.py

The model parameters and BatchNorm statistics are drawn from a seed (tests/old_score_helpers.py:seeded_values) and only
the seed, the shapes and the remaining buffers are stored, which keeps the fixture small.

Fixtures:
  ref_old_score_model.pt     CGOldModel.forward in score mode over five configurations (LM on/off, dynamic_max_cross,
                             smooth_edges, 2-4 layers, fixed_center_conv, no_torsion, a ligand without rotatable bonds,
                             per-complex diffusion times); the last one has fused-kernel widths (ns=16, nv=4)
  ref_sampling_old_score.pt  utils/sampling.py: 3 reverse-diffusion steps of case 4 with the v1.0 confidence model of
                             ref_confidence.pt[0]; seeded CPU noise (torch.manual_seed(seed) then torch.normal in the
                             reference's order), which the GPU test replays through ``noise_fn``
"""
import copy
import os
import sys
from functools import partial

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402

ref_shims.install()
sys.path.insert(0, os.environ['DIFFDOCK_REFERENCE'])
import models.old_cg_model as r_old          # noqa: E402
import utils.diffusion_utils as r_du        # noqa: E402
import utils.sampling as r_sampling         # noqa: E402
from utils import torus as r_torus          # noqa: E402

from diffdock_b200.hetero import collate, graph_to_dict   # noqa: E402
from diffdock_b200.synthetic import default_model_args, make_pose_list   # noqa: E402
from tests.old_score_helpers import fixture_state, generated, seeded_values    # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
torch.set_num_threads(4)
# the stored Monte-Carlo torus table instance, shared with the product and the oracle (the import above re-drew it)
r_torus.score_norm_ = np.load(os.path.join(ROOT, 'diffdock_b200', 'tables', 'score_norm_tables.npz'))['torus_score_norm']


def set_times(batch, t):
    """Per-complex diffusion times ``t`` [B] on every node and graph (utils/diffusion_utils.py:146-168 with one time per
    complex instead of one per batch)."""
    t = torch.as_tensor(t, dtype=torch.float32)
    for nt in ('ligand', 'receptor'):
        batch[nt].node_t = {k: t[batch[nt].batch] for k in ('tr', 'rot', 'tor')}
    batch.complex_t = {k: t.clone() for k in ('tr', 'rot', 'tor')}


def compact(d):
    """A pose dict whose tensors own exactly their data (torch.save writes a view's whole storage)."""
    if isinstance(d, dict):
        return {k: compact(v) for k, v in d.items()}
    return d.clone() if torch.is_tensor(d) else d


def case(seed, num_conv_layers, times, lm=True, dynamic=False, smooth=False, fixed_center=False, no_torsion=False,
         rigid=False, ns=6, nv=3, n_poses=3):
    a = default_model_args()
    kw = dict(sigma_embed_dim=8, sh_lmax=2, ns=ns, nv=nv, num_conv_layers=num_conv_layers, lig_max_radius=5.0,
              rec_max_radius=30.0, cross_max_distance=25.0, distance_embed_dim=8, cross_distance_embed_dim=8,
              dynamic_max_cross=dynamic, smooth_edges=smooth, fixed_center_conv=fixed_center, no_torsion=no_torsion,
              lm_embedding_type='esm' if lm else None, confidence_mode=False, use_old_atom_encoder=True)
    torch.manual_seed(seed)
    model = r_old.CGOldModel(partial(r_du.t_to_sigma, args=a), torch.device('cpu'),
                             r_du.get_timestep_embedding('sinusoidal', 8, a.embedding_scale), **kw).eval()
    poses = make_pose_list(n_poses, n_res=24, n_atoms=9, seed=seed + 2, tr_sigma_max=1.5, lm_dim=16 if lm else 0)
    if rigid:    # no rotatable bond: the torsion head returns an empty tensor (models/old_cg_model.py:331)
        for p in poses:
            p['ligand'].edge_mask = torch.zeros_like(p['ligand'].edge_mask)
    if lm:       # shrink the LM embedding (1280 -> 16) to keep the fixture small
        model.rec_node_embedding.lm_embedding_dim = 16
        model.rec_node_embedding.lm_embedding_layer = torch.nn.Linear(16 + ns, ns)
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items() if generated(k)}
    missing, unexpected = model.load_state_dict(seeded_values(shapes, seed + 1), strict=False)
    assert not unexpected and all(not generated(k) for k in missing)
    fixed = {k: v.clone() for k, v in model.state_dict().items() if not generated(k)}
    batch = collate(copy.deepcopy(poses))
    set_times(batch, times)
    with torch.no_grad():
        tr, rot, tor = model(batch)
    print('case', seed, 'tr', tr[0].tolist(), 'tor', tuple(tor.shape))
    return dict(kw=kw, args=vars(a), lm_dim=16 if lm else 0, times=list(times), fixed=fixed, shapes=shapes, seed=seed + 1,
                poses=[compact(graph_to_dict(p)) for p in poses], tr=tr, rot=rot, tor=tor)


cases = [case(40, 3, [0.5, 0.5, 0.5]),
         case(41, 4, [0.2, 0.55, 0.9], lm=False, dynamic=True, fixed_center=True),
         case(42, 2, [0.35, 0.35, 0.35], smooth=True, no_torsion=True),
         case(43, 3, [0.7, 0.7, 0.7], lm=False, rigid=True),
         case(44, 2, [0.3, 0.6, 0.45], ns=16, nv=4)]
torch.save(cases, os.path.join(OUT, 'ref_old_score_model.pt'))
print('ref_old_score_model.pt', os.path.getsize(os.path.join(OUT, 'ref_old_score_model.pt')) // 1024, 'KiB')

# ------------------------------------------------------------------------------------------------ sampling + confidence
from argparse import Namespace              # noqa: E402
from diffdock_b200.hetero import graph_from_dict   # noqa: E402

sc = cases[4]
sa = Namespace(**sc['args'])
score = r_old.CGOldModel(partial(r_du.t_to_sigma, args=sa), torch.device('cpu'),
                         r_du.get_timestep_embedding('sinusoidal', 8, sa.embedding_scale), **sc['kw']).eval()
score.rec_node_embedding.lm_embedding_dim = 16
score.rec_node_embedding.lm_embedding_layer = torch.nn.Linear(16 + 16, 16)
score.load_state_dict(fixture_state(sc), strict=True)
poses = [graph_from_dict(d) for d in sc['poses']]

ccase = torch.load(os.path.join(OUT, 'ref_confidence.pt'), weights_only=False)[0]
ca = default_model_args()
conf = r_old.CGOldModel(partial(r_du.t_to_sigma, args=ca), torch.device('cpu'),
                        r_du.get_timestep_embedding('sinusoidal', 8, ca.embedding_scale), **ccase['kw']).eval()
conf.rec_node_embedding.lm_embedding_dim = 16
conf.rec_node_embedding.lm_embedding_layer = torch.nn.Linear(16 + 6, 6)
conf.load_state_dict(ccase['state'], strict=True)

sched = np.array([0.45, 0.25, 0.08])
seed = 91
torch.manual_seed(seed)
out_list, c = r_sampling.sampling(data_list=copy.deepcopy(poses), model=score, inference_steps=3, tr_schedule=sched,
                                  rot_schedule=sched, tor_schedule=sched, device=torch.device('cpu'),
                                  t_to_sigma=partial(r_du.t_to_sigma, args=sa), model_args=copy.deepcopy(sa),
                                  batch_size=3, no_final_step_noise=True, confidence_model=conf,
                                  confidence_data_list=copy.deepcopy(poses),
                                  confidence_model_args=Namespace(all_atoms=False, crop_beyond=None))
print('sampling confidence', c)
torch.save(dict(score_case=4, confidence_case=0, seed=seed, schedule=sched, confidence=c,
                final_pos=[d['ligand'].pos.clone() for d in out_list]),
           os.path.join(OUT, 'ref_sampling_old_score.pt'))
print('ref_sampling_old_score.pt written')

"""Golden vectors for confidence models built by the current training code: ``CGModel`` / ``AAModel`` with
``confidence_mode=True`` (confidence/confidence_train.py:284 calls ``get_model(..., confidence_mode=True)`` with old=False).
Runs the UNMODIFIED reference models/cg_model.py, models/aa_model.py, utils/sampling.py and utils/utils.py:get_model from a
checkout of the reference DiffDock code base, with the third-party packages supplied by oracle/ref_shims.py.  The so3/torus
tables take about 1.5 minutes at import; run it from a scratch working directory (utils/so3.py writes its .npy caches there):

    cd <scratch dir> && DIFFDOCK_REFERENCE=<reference checkout> python <this repository>/tests/golden/make_golden_confidence_v11.py

Parameters are drawn from a seed (tests/old_score_helpers.py:seeded_values); the BatchNorm1d layers of the confidence heads
get rand_bn_ statistics and are stored with the other fixed entries.  All cases have fused-kernel widths (ns=16, nv=4).

Fixture ref_confidence_v11.pt, a dict:
  cases     forward in confidence mode at per-complex times t (the times are the sigmas), ``confidence`` / ``atom_confidence``:
              (0) CGModel, 3 interaction layers, sh_lmax=2
              (1) CGModel, DiffDock-L flags (reduce_pseudoscalars, smooth_edges, sh_lmax=1, num_prot_emb_layers=1,
                  dynamic_max_cross; one edge group per convolution, as in make_golden_diffdock_l.py), three
                  rmsd_classification_cutoff values (4 outputs) and affinity_prediction (+1)
              (2) CGModel, 2 layers, atom_confidence (the input_size = ns branch), two atom outputs
              (3) AAModel, 3 layers, atom_confidence
              (4) CGModel, 3 layers, tp_weights_layers=3
  sampling  utils/sampling.py: 3 reverse-diffusion steps of a CGModel score model with crop_beyond=7, ranked by case (3)'s
            AAModel on an all-atom confidence_data_list; seeded CPU noise (torch.manual_seed(seed), the reference's order)
  get_model the class and keywords utils/utils.py:get_model passes with confidence_mode=True, old=False, for the confidence
            trainer's defaults with all_atoms True and False
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
import models.aa_model as r_aa              # noqa: E402
import models.cg_model as r_cg              # noqa: E402
import utils.diffusion_utils as r_du        # noqa: E402
import utils.sampling as r_sampling         # noqa: E402
import utils.utils as r_utils               # noqa: E402
from utils import torus as r_torus          # noqa: E402

from diffdock_b200.hetero import collate, graph_to_dict   # noqa: E402
from diffdock_b200.synthetic import default_model_args, make_pose_list   # noqa: E402
from tests.old_score_helpers import generated, seeded_values, set_times    # noqa: E402
from tests.parity_helpers import rand_bn_    # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
torch.set_num_threads(4)
r_torus.score_norm_ = np.load(os.path.join(ROOT, 'diffdock_b200', 'tables', 'score_norm_tables.npz'))['torus_score_norm']
NS, NV = 16, 4


def compact(d):
    if isinstance(d, dict):
        return {k: compact(v) for k, v in d.items()}
    return d.clone() if torch.is_tensor(d) else d


def model_kw(a, **extra):
    kw = dict(sigma_embed_dim=8, sh_lmax=a.sh_lmax, ns=NS, nv=NV, num_conv_layers=a.num_conv_layers,
              lig_max_radius=a.max_radius, rec_max_radius=a.rec_max_radius, cross_max_distance=a.cross_max_distance,
              center_max_distance=a.center_max_distance, distance_embed_dim=8, cross_distance_embed_dim=8,
              dynamic_max_cross=a.dynamic_max_cross, lm_embedding_type=None, embed_also_ligand=True,
              num_prot_emb_layers=a.num_prot_emb_layers, reduce_pseudoscalars=a.reduce_pseudoscalars,
              smooth_edges=a.smooth_edges, tp_weights_layers=a.tp_weights_layers)
    kw.update(extra)
    return kw


def seeded(model, seed):
    """Seeded parameters (tests/old_score_helpers.py), rand_bn_ on the BatchNorm1d layers of the heads: ``(fixed, shapes)``."""
    bn1d = {n for n, m in model.named_modules() if isinstance(m, torch.nn.BatchNorm1d)}
    is_bn1d = lambda k: k.rsplit('.', 1)[0] in bn1d
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items() if generated(k) and not is_bn1d(k)}
    missing, unexpected = model.load_state_dict(seeded_values(shapes, seed), strict=False)
    assert not unexpected
    g = torch.Generator().manual_seed(seed + 7)
    for n in sorted(bn1d):
        rand_bn_(model.get_submodule(n), g)
    fixed = {k: v.clone() for k, v in model.state_dict().items() if not (generated(k) and not is_bn1d(k))}
    return fixed, shapes


def case(seed, cls, times, n_res=24, n_atoms=9, all_atoms=False, args=None, **kw):
    a = default_model_args(ns=NS, nv=NV, **(args or {}))
    kw = model_kw(a, confidence_mode=True, **kw)
    torch.manual_seed(seed)
    model = cls(None, torch.device('cpu'), r_du.get_timestep_embedding('sinusoidal', 8, a.embedding_scale), **kw).eval()
    fixed, shapes = seeded(model, seed + 1)
    poses = make_pose_list(len(times), n_res=n_res, n_atoms=n_atoms, seed=seed + 2, tr_sigma_max=2.0, all_atoms=all_atoms,
                           lm_dim=0)
    batch = collate(copy.deepcopy(poses))
    set_times(batch, times)
    if all_atoms:
        batch['atom'].node_t = {k: torch.as_tensor(times, dtype=torch.float32)[batch['atom'].batch]
                                for k in ('tr', 'rot', 'tor')}
    with torch.no_grad():
        conf, atom_conf = model(batch)
    print('case', seed, cls.__name__, 'confidence', tuple(conf.shape), conf.flatten()[:3].tolist(), 'atom', tuple(atom_conf.shape))
    c = dict(cls=cls.__name__, args=vars(a), kw=kw, times=torch.as_tensor(times, dtype=torch.float32), fixed=fixed,
             shapes=shapes, seed=seed + 1, all_atoms=all_atoms, poses=[compact(graph_to_dict(p)) for p in poses],
             confidence=conf, atom_confidence=atom_conf)
    return c, model, poses


L_FLAGS = dict(sh_lmax=1, num_prot_emb_layers=1, reduce_pseudoscalars=True, smooth_edges=True, dynamic_max_cross=True,
               num_conv_layers=3)
c0, _, _ = case(70, r_cg.CGModel, [0.0, 0.4, 1.0], args=dict(num_conv_layers=3, sh_lmax=2, dynamic_max_cross=False,
                                                                cross_max_distance=20.0))
# the reference runs sh_lmax=1 on FasterTensorProduct, which its multi-group scatter cannot take (make_golden_diffdock_l.py)
c1, _, _ = case(71, r_cg.CGModel, [0.2, 0.9, 0.05], args=L_FLAGS, num_confidence_outputs=4, affinity_prediction=True,
                differentiate_convolutions=False)
c2, _, _ = case(72, r_cg.CGModel, [0.0, 0.0, 0.0], args=dict(num_conv_layers=2, sh_lmax=2), atom_confidence=True,
                atom_num_confidence_outputs=2)
c3, m3, p3 = case(73, r_aa.AAModel, [0.0, 0.0, 0.0], n_res=20, all_atoms=True, args=dict(num_conv_layers=3, sh_lmax=2),
                  atom_confidence=True)
c4, _, _ = case(74, r_cg.CGModel, [0.3, 0.0, 0.8], args=dict(num_conv_layers=3, sh_lmax=2, tp_weights_layers=3))
cases = [c0, c1, c2, c3, c4]
assert c1['confidence'].shape == (3, 5) and c2['atom_confidence'].shape == (27, 2) and c0['atom_confidence'].shape == (27,)

# ------------------------------------------------------------------------------- cropped sampling ranked by AAModel
sa = default_model_args(ns=NS, nv=NV, num_conv_layers=2, sh_lmax=2)
skw = model_kw(sa)
torch.manual_seed(80)
score = r_cg.CGModel(partial(r_du.t_to_sigma, args=sa), torch.device('cpu'),
                     r_du.get_timestep_embedding('sinusoidal', 8, sa.embedding_scale), **skw).eval()
s_fixed, s_shapes = seeded(score, 81)
poses = make_pose_list(3, n_res=20, n_atoms=9, seed=82, tr_sigma_max=sa.tr_sigma_max * 0.3, lm_dim=0)
conf_list = []                      # the ranking model's all-atom graphs of the same complex, with the score model's ligand
for p, q in zip(poses, p3):
    c = copy.deepcopy(q)
    for k in ('x', 'pos', 'edge_mask', 'mask_rotate'):
        setattr(c['ligand'], k, copy.deepcopy(getattr(p['ligand'], k)))
    c['ligand', 'ligand'].edge_index = p['ligand', 'ligand'].edge_index.clone()
    c['ligand', 'ligand'].edge_attr = p['ligand', 'ligand'].edge_attr.clone()
    conf_list.append(c)
margs = Namespace(**vars(sa))
margs.crop_beyond = 7.0
steps, seed = 3, 461
sched = np.array([0.30, 0.18, 0.08])
torch.manual_seed(seed)
out_list, confidence = r_sampling.sampling(
    data_list=copy.deepcopy(poses), model=score, inference_steps=steps, tr_schedule=sched, rot_schedule=sched,
    tor_schedule=sched, device=torch.device('cpu'), t_to_sigma=partial(r_du.t_to_sigma, args=sa), model_args=margs,
    batch_size=3, no_final_step_noise=True, confidence_model=m3, confidence_data_list=copy.deepcopy(conf_list),
    confidence_model_args=Namespace(all_atoms=True, crop_beyond=None))
print('sampling confidence', confidence)
sampling = dict(score=dict(args=vars(sa), kw=skw, fixed=s_fixed, shapes=s_shapes, seed=81), confidence_case=3,
                poses=[compact(graph_to_dict(p)) for p in poses], conf_poses=[compact(graph_to_dict(p)) for p in conf_list],
                steps=steps, seed=seed, schedule=sched, crop_beyond=7.0, confidence=confidence,
                final_pos=[d['ligand'].pos.clone() for d in out_list])


# ------------------------------------------------------------------------------------------------ get_model keywords
def recorder(name):
    class R:
        def __init__(self, **kw):
            self.name, self.kw = name, kw

        def to(self, device):
            return self
    return R


TRAINER = dict(no_torsion=False, num_conv_layers=2, max_radius=5.0, scale_by_sigma=True, sigma_embed_dim=32, ns=16, nv=4,
               distance_embed_dim=32, cross_distance_embed_dim=32, no_batch_norm=False, dropout=0.0,
               use_second_order_repr=False, cross_max_distance=80, dynamic_max_cross=False, esm_embeddings_path=None,
               rmsd_classification_cutoff=2, embedding_type='sinusoidal', embedding_scale=1000)
r_utils.CGModel, r_utils.AAModel = recorder('CGModel'), recorder('AAModel')
get_model = []
for all_atoms in (True, False):
    a = dict(TRAINER, all_atoms=all_atoms)
    m = r_utils.get_model(Namespace(**a), torch.device('cpu'), t_to_sigma=None, no_parallel=True, confidence_mode=True)
    k = dict(m.kw)
    for key in ('t_to_sigma', 'device', 'timestep_emb_func'):
        k.pop(key)
    get_model.append(dict(args=a, cls=m.name, kwargs=k))
    print('get_model all_atoms', all_atoms, m.name, len(k))

torch.save(dict(cases=cases, sampling=sampling, get_model=get_model), os.path.join(OUT, 'ref_confidence_v11.pt'))
print('ref_confidence_v11.pt', os.path.getsize(os.path.join(OUT, 'ref_confidence_v11.pt')) // 1024, 'KiB')

"""Golden vectors for the reverse-diffusion frames that ``sampling(..., visualization_list=...)`` leaves in the caller's
visualisation objects: runs the UNMODIFIED reference utils/sampling.py (third-party packages supplied by
oracle/ref_shims.py), like make_golden.py.  The so3/torus tables take about 1.5 minutes at import; run it from a scratch
working directory (utils/so3.py writes its .npy caches there):

    cd <scratch dir> && python <this repository>/tests/golden/make_golden_visualisation.py

Poses: the 3 poses of ref_sampling.pt (model_case=0 of ref_cg_model.pt) and a 4th drawn by the same make_pose_list call,
each with its own ``original_center``; 4 steps of the same expbeta schedule; batch_size=2, so two batches.  The
reference cannot sample a partial last batch unless ``ode`` is set (tests/visualisation_helpers.py:N_POSES).  Every pose
gets a recorder with PDBFile.add's signature (tests/visualisation_helpers.py:RecordingPDB), pre-populated as
inference.py:248-255 does.

Fixture ref_sampling_visualisation.pt, a dict:
  poses, original_center, crystal   the 4 pose dicts, their centres [1, 3] and the pre-populated input ligand
  schedule, steps, batch_size
  runs['a']   model_case=0 of ref_cg_model.pt, seeded CPU noise (torch.manual_seed(seed), torch.normal in the reference's
              order, replayed by the GPU test through ``noise_fn``), inference.py's temperatures, no_final_step_noise
  runs['b']   no_random=True with the ns=16 / nv=4 model of ``fused_case`` (its parameters drawn from a stored seed,
              tests/old_score_helpers.py:seeded_values), whose convolutions all fit the fused kernel, so the product
              samples it on the captured step; inference.py's temperatures
  each run: ``content`` = every recorder's final {part: {order: coords}}, ``final_pos`` = the poses' final coordinates
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
OUT = os.path.join(ROOT, 'tests', 'golden')
torch.set_num_threads(4)

import models.cg_model as r_cg              # noqa: E402
import utils.diffusion_utils as r_du        # noqa: E402
import utils.sampling as r_sampling         # noqa: E402
from utils import torus as r_torus          # noqa: E402

from diffdock_b200.hetero import graph_from_dict, graph_to_dict   # noqa: E402
from diffdock_b200.synthetic import default_model_args, make_pose_list   # noqa: E402
from tests.old_score_helpers import generated, seeded_values    # noqa: E402
from tests.parity_helpers import load_golden    # noqa: E402
from tests.visualisation_helpers import BATCH_SIZE, N_POSES, original_centers, prepopulated   # noqa: E402

# the stored Monte-Carlo torus table instance, shared with the product and the oracle (the import above re-drew it)
r_torus.score_norm_ = np.load(os.path.join(ROOT, 'diffdock_b200', 'tables', 'score_norm_tables.npz'))['torus_score_norm']
TEMPS = dict(temp_sampling=[1.170050527854316, 2.06391612594481, 7.044261621607846],
             temp_psi=[0.727287304570729, 0.9022615585677628, 0.5946212391366862],
             temp_sigma_data=[0.9299802531572672, 0.7464326999906034, 0.6943254174849822])


def compact(d):
    """A pose dict whose tensors own exactly their data (torch.save writes a view's whole storage)."""
    if isinstance(d, dict):
        return {k: compact(v) for k, v in d.items()}
    return d.clone() if torch.is_tensor(d) else d


def build(c, ns):
    a = Namespace(**c['args'])
    model = r_cg.CGModel(partial(r_du.t_to_sigma, args=a), torch.device('cpu'),
                         r_du.get_timestep_embedding('sinusoidal', c['kw']['sigma_embed_dim'], a.embedding_scale),
                         **c['kw']).eval()
    model.rec_node_embedding.additional_features_dim = c['lm_dim']       # the 16-wide LM embedding of the poses
    model.rec_node_embedding.additional_features_embedder = torch.nn.Linear(c['lm_dim'] + ns, ns)
    return model, a


# ------------------------------------------------------------------------------------------------ models and poses
s = load_golden('ref_sampling.pt')
case0 = load_golden('ref_cg_model.pt')[s['model_case']]
m0, a0 = build(case0, case0['kw']['ns'])
m0.load_state_dict(case0['state'], strict=True)

# the 3 poses of case 0 came from make_pose_list(3, n_res=24, n_atoms=9, seed=12, ...): the same call with 4 draws them again
poses = make_pose_list(N_POSES, n_res=24, n_atoms=9, seed=12, tr_sigma_max=a0.tr_sigma_max * case0['t'], lm_dim=16)
for p, d in zip(poses, case0['poses']):
    ref = graph_from_dict(d)
    assert torch.equal(p['ligand'].pos, ref['ligand'].pos) and torch.equal(p['receptor'].pos, ref['receptor'].pos)
centers = original_centers(N_POSES)
for p, c in zip(poses, centers):
    p.original_center = c
crystal = poses[0]['ligand'].pos.clone()

a1 = default_model_args(ns=16, nv=4, sh_lmax=2, num_conv_layers=3, distance_embed_dim=8, cross_distance_embed_dim=8,
                        sigma_embed_dim=8)
kw1 = dict(case0['kw'], ns=16, nv=4)
fused_case = dict(args=vars(a1), kw=kw1, lm_dim=16)
torch.manual_seed(70)
m1, _ = build(fused_case, 16)
shapes = {k: tuple(v.shape) for k, v in m1.state_dict().items() if generated(k)}
missing, unexpected = m1.load_state_dict(seeded_values(shapes, 71), strict=False)
assert not unexpected and all(not generated(k) for k in missing)
fused_case.update(fixed={k: v.clone() for k, v in m1.state_dict().items() if not generated(k)}, shapes=shapes, seed=71)

steps, sched = s['steps'], s['schedule']


def run(model, a, **kw):
    data_list = copy.deepcopy(poses)
    vis = prepopulated(data_list, crystal)
    margs = Namespace(**vars(a))
    margs.crop_beyond = None
    out, _ = r_sampling.sampling(data_list=data_list, model=model, inference_steps=steps, tr_schedule=sched,
                                 rot_schedule=sched, tor_schedule=sched, device=torch.device('cpu'),
                                 t_to_sigma=partial(r_du.t_to_sigma, args=a), model_args=margs, visualization_list=vis,
                                 batch_size=BATCH_SIZE, no_final_step_noise=True, **TEMPS, **kw)
    content = [v.content() for v in vis]
    final = [d['ligand'].pos.clone() for d in out]
    for c, f, ctr in zip(content, final, centers):
        assert torch.equal(c[1][2], f + ctr) and sorted(c[1]) == list(range(1, steps + 2))
    return dict(content=content, final_pos=final)


seed_a = 123
torch.manual_seed(seed_a)
with torch.no_grad():
    run_a = run(m0, a0)
    run_b = run(m1, a1, no_random=True)
run_a.update(model_case=s['model_case'], seed=seed_a)
run_b.update(model='fused_case')
torch.save(dict(poses=[compact(graph_to_dict(p)) for p in poses], original_center=centers, crystal=crystal,
                schedule=sched, steps=steps, batch_size=BATCH_SIZE, fused_case=fused_case, runs={'a': run_a, 'b': run_b}),
           os.path.join(OUT, 'ref_sampling_visualisation.pt'))
print('ref_sampling_visualisation.pt', os.path.getsize(os.path.join(OUT, 'ref_sampling_visualisation.pt')) // 1024, 'KiB')

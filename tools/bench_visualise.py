#!/usr/bin/env python
"""tools/bench_visualise.py - ``sampling(..., visualization_list=...)`` on the captured step against the eager loop.

    python tools/bench_visualise.py [--repeats 7] [--workloads evaluate,inference]

Workloads, bench.py's CFG-L2 CGModel:
  evaluate    evaluate.py's defaults, where --save_visualisation cannot be switched off: 4 poses, 40 steps, batch_size=40,
              unit temperatures, final-step noise, one PDBBind-sized synthetic complex (400 residues, 30 ligand atoms)
  inference   inference.py --save_visualisation at its defaults on BASELINE config 3 (1500 residues, 40 ligand atoms):
              10 samples, 19 of 20 steps, batch_size=10, its temperatures, no_final_step_noise
Arms (torch.normal noise, as those scripts draw it):
  graphed_frames     the captured step, frames recorded in the graph
  eager_frames       cuda_graph=False: the route every visualising call took before frames were recorded on the device
  graphed_no_frames  the captured step without visualization_list: the cost of recording frames
The visualisation objects are recorders with ``PDBFile.add``'s signature that keep the tensor they are given, not RDKit
PDBFile objects: the host time of the caller's ``add`` (one MolToPDBBlock per call) is NOT part of these numbers.

Every arm runs once as warm-up (every shape, graph captures included), then the arms alternate ``--repeats`` times;
medians with min-max of a host clock that ends in a device synchronise.  ``frames_max_abs_A``: the largest difference of
any recorded frame between the graphed and the eager arm when both draw Philox noise (same draws; the rest is the
summation order of atomics).  The card's name and power limit come from the same run.  One JSON line per workload.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from collections import defaultdict
from functools import partial

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import TEMPS, model_kwargs, randomise_bn   # noqa: E402
from tools.bench_crop import card                   # noqa: E402
from tools.bench_pack import alternate, resetter    # noqa: E402
from tools.bench_rank import stats                  # noqa: E402

UNIT_TEMPS = dict(temp_sampling=1.0, temp_psi=0.0, temp_sigma_data=0.5)     # evaluate.py's argument defaults
WORKLOADS = {
    'evaluate': dict(n_res=400, n_atoms=30, poses=4, steps=40, sched_steps=40, batch_size=40, no_final_step_noise=False,
                     temps=UNIT_TEMPS),
    'inference': dict(n_res=1500, n_atoms=40, poses=10, steps=19, sched_steps=20, batch_size=10, no_final_step_noise=True,
                      temps=TEMPS),
}


class Recorder:
    """``PDBFile.add(coords, order, part=0, repeat=1)`` that keeps the coordinates instead of writing a PDB block."""

    def __init__(self):
        self.parts = defaultdict(dict)

    def add(self, coords, order, part=0, repeat=1):
        self.parts[part][order] = coords


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=7)
    ap.add_argument('--workloads', default='evaluate,inference')
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_visualise.py measures on a CUDA device; none found")
    import __graft_entry__ as ge
    ge.build()
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_t_schedule, get_timestep_embedding, t_to_sigma
    from diffdock_b200.sampling import sampling
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    dev = torch.device('cuda:0')
    info = card()
    args = default_model_args()
    t2s = partial(t_to_sigma, args=args)
    torch.manual_seed(0)
    model = CGModel(t2s, dev, get_timestep_embedding('sinusoidal', args.sigma_embed_dim, args.embedding_scale),
                    **model_kwargs(args)).eval()
    randomise_bn(model, 1)
    model = model.to(dev)

    for name in cli.workloads.split(','):
        w = WORKLOADS[name]
        poses = make_pose_list(w['poses'], n_res=w['n_res'], n_atoms=w['n_atoms'], seed=7, tr_sigma_max=args.tr_sigma_max,
                               share_receptor=True)     # one receptor upload per batch, as inputs.pose_copies gives
        for i, p in enumerate(poses):
            p.original_center = torch.tensor([[10.0 + i, -5.0, 2.5]])
        sched = get_t_schedule('expbeta', w['sched_steps'])

        def run(frames, graph, **kw):
            vis = [Recorder() for _ in poses] if frames else None
            out, _ = sampling(poses, model, w['steps'], sched, sched, sched, dev, t2s, args, batch_size=w['batch_size'],
                              no_final_step_noise=w['no_final_step_noise'], visualization_list=vis, cuda_graph=graph,
                              **w['temps'], **kw)
            return vis, torch.stack([d['ligand'].pos for d in out])

        arms = {'graphed_frames': lambda: run(True, True), 'eager_frames': lambda: run(True, False),
                'graphed_no_frames': lambda: run(False, True)}
        reset = resetter([poses])
        times, _ = alternate(arms, cli.repeats, reset)
        reset()
        vg, _ = run(True, True, rng='philox', seed=11)
        reset()
        ve, _ = run(True, False, rng='philox', seed=11)
        reset()
        diff = max(float((a.parts[1][o] - b.parts[1][o]).abs().max()) for a, b in zip(vg, ve) for o in range(2, w['steps'] + 2))
        med = {k: float(np.median(v)) for k, v in times.items()}
        print(json.dumps({'workload': name, 'receptor_residues': w['n_res'], 'ligand_atoms': w['n_atoms'],
                          'poses': w['poses'], 'steps': w['steps'], 'batch_size': w['batch_size'], 'repeats': cli.repeats,
                          'ms': {k: stats(v) for k, v in times.items()},
                          'ms_per_step': {k: round(v / w['steps'], 3) for k, v in med.items()},
                          'speedup_vs_eager_frames': round(med['eager_frames'] / med['graphed_frames'], 3),
                          'frames_cost_ms': round(med['graphed_frames'] - med['graphed_no_frames'], 3),
                          'frames_max_abs_A': diff, 'visualisation_objects': 'recording stub, PDBFile.add host time excluded',
                          'card': info}), flush=True)


if __name__ == '__main__':
    main()

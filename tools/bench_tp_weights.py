#!/usr/bin/env python
"""tools/bench_tp_weights.py - reverse diffusion with a score model built with ``tp_weights_layers=3`` (every radial MLP
of the embedding and interaction convolutions has one extra 3ns x 3ns hidden layer).

    python tools/bench_tp_weights.py [--repeats 5] [--poses 40] [--n-res 1500] [--n-atoms 40] [--layers 3]

Workload: BASELINE config 3 (1500 residues / 40 ligand atoms / 40 poses of one synthetic complex, 1280-wide LM embedding)
over the 20-step expbeta schedule at the CFG-L2 shape (ns=48, nv=10, sh_lmax=2, 6 layers, 64-dim embeddings) with
``tp_weights_layers=3``, seeded weights, default-yaml temperatures, counter-based (Philox) noise from one seed; without
and with ``crop_beyond=20``.  Arms, all through ``sampling()``:
  graphed      the sync-free forward with the step captured in a CUDA graph (with the crop inside the captured step)
  host_eager   a copy of the same model with ``_sync_free = False``: the host-sized forward launched op by op (its
               convolutions still on the fused kernel), and with ``crop_beyond`` the eager per-step crop
  unfused      host_eager with the fused kernel switched off (``fused.ENABLED = False`` around the call): the path these
               models took before the fused kernel ran the extra hidden layers (torch Linears, radial_gemm and the
               streaming kernel, per-edge weights through HBM)
Each arm runs once as warm-up, then the arms alternate ``--repeats`` times in this process; the times are CUDA events
around whole sampling() calls, the median is reported.  Final coordinates: the largest difference between the arms from
the same seed, and between two graphed runs from the same seed (the noise floor of the scatter atomics' order).
The card's name and power limit are printed with the numbers.  One JSON line per crop setting.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import sys
from functools import partial

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import N_SCHED, TEMPS, randomise_bn      # noqa: E402
from tools.bench_crop import card                   # noqa: E402


def tw_model(args, dev):
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding, t_to_sigma
    kw = dict(sigma_embed_dim=args.sigma_embed_dim, sh_lmax=args.sh_lmax, ns=args.ns, nv=args.nv,
              num_conv_layers=args.num_conv_layers, lig_max_radius=args.max_radius, rec_max_radius=args.rec_max_radius,
              cross_max_distance=args.cross_max_distance, center_max_distance=args.center_max_distance,
              distance_embed_dim=args.distance_embed_dim, cross_distance_embed_dim=args.cross_distance_embed_dim,
              dynamic_max_cross=args.dynamic_max_cross, lm_embedding_type='precomputed', embed_also_ligand=True,
              num_prot_emb_layers=args.num_prot_emb_layers, tp_weights_layers=args.tp_weights_layers)
    torch.manual_seed(0)
    m = CGModel(partial(t_to_sigma, args=args), dev, get_timestep_embedding('sinusoidal', args.sigma_embed_dim,
                                                                             args.embedding_scale), **kw).eval()
    randomise_bn(m, 1)
    return m.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--poses', type=int, default=40)
    ap.add_argument('--n-res', dest='n_res', type=int, default=1500)
    ap.add_argument('--n-atoms', dest='n_atoms', type=int, default=40)
    ap.add_argument('--layers', type=int, default=3, help='tp_weights_layers')
    ap.add_argument('--crop-beyond', dest='crop_beyond', type=float, nargs='*', default=[None, 20.0])
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tp_weights.py measures on a CUDA device; none found")
    import __graft_entry__ as ge
    ge.build()
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sampling
    from diffdock_b200.synthetic import default_model_args, make_pose_list

    dev = torch.device('cuda', 0)
    args = default_model_args(embed_also_ligand=True, tp_weights_layers=cli.layers)
    graphed_model = tw_model(args, dev)
    assert graphed_model.sync_free_capable() and graphed_model.sync_free_crop_capable()
    host_model = copy.deepcopy(graphed_model)
    host_model._sync_free = False           # host-sized forward; sampling() then runs the steps eagerly
    n = cli.poses
    poses = make_pose_list(n, n_res=cli.n_res, n_atoms=cli.n_atoms, seed=100, tr_sigma_max=args.tr_sigma_max)
    sched = get_t_schedule('expbeta', N_SCHED)
    info = card()

    for crop in cli.crop_beyond:
        a = copy.copy(args)
        a.crop_beyond = crop
        t2s = partial(t_to_sigma, args=a)

        def run(model, graphed):
            out, _ = sampling([q.clone() for q in poses], model, N_SCHED, sched, sched, sched, dev, t2s, a, batch_size=n,
                              no_final_step_noise=True, cuda_graph=graphed, rng='philox', seed=1234, **TEMPS)
            return torch.stack([d['ligand'].pos for d in out])

        def unfused():
            from diffdock_b200 import fused
            fused.ENABLED = False
            try:
                return run(host_model, False)
            finally:
                fused.ENABLED = True

        arms = {'graphed': lambda: run(graphed_model, True), 'host_eager': lambda: run(host_model, False),
                'unfused': unfused}
        final = {k: fn() for k, fn in arms.items()}          # warm-up: one whole run each
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for _ in range(cli.repeats):
            for k, fn in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1))
        ms = {k: float(np.median(v)) for k, v in times.items()}
        again = arms['graphed']()
        torch.cuda.synchronize()
        line = {'tool': 'bench_tp_weights', 'card': info, 'crop_beyond': crop,
                'workload': f'{cli.n_res} residues / {cli.n_atoms} ligand atoms / {n} poses, tp_weights_layers='
                            f'{cli.layers} at ns=48, nv=10, sh_lmax=2, 6 layers, {N_SCHED}-step expbeta schedule',
                'ms_per_run': ms, 'ms_per_step': {k: v / N_SCHED for k, v in ms.items()},
                'ms_per_run_all': times, 'poses_per_s': {k: n / (v / 1000.0) for k, v in ms.items()},
                'speedup_graphed_vs_host_eager': ms['host_eager'] / ms['graphed'],
                'speedup_graphed_vs_unfused': ms['unfused'] / ms['graphed'],
                'final_pos_max_abs_diff_A': {
                    'graphed_vs_host_eager': float((final['graphed'] - final['host_eager']).abs().max()),
                    'graphed_vs_unfused': float((final['graphed'] - final['unfused']).abs().max()),
                    'host_eager_vs_unfused': float((final['host_eager'] - final['unfused']).abs().max()),
                    'graphed_vs_graphed': float((final['graphed'] - again).abs().max())},
                'how': f'CUDA events around whole sampling() calls, median of {cli.repeats} alternated repeats after one '
                       f'warm-up run each'}
        print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()

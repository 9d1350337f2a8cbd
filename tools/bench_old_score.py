#!/usr/bin/env python
"""tools/bench_old_score.py - reverse-diffusion steps of the v1.0 score model (CGOldModel, confidence_mode=False).

    python tools/bench_old_score.py [--repeats 5] [--no-oracle]

Workload: BASELINE config 3 (1500 residues / 40 ligand atoms / 40 poses of one synthetic complex, 1280-wide LM embedding)
over the 20-step expbeta schedule, with the v1.0 model at CFG-L2 widths (ns=48, nv=10, 6 layers, 64-dim embeddings).
Arms, timed with CUDA events over whole 20-step runs after one warm-up run each, alternated ``--repeats`` times in this
process:
  graphed_v10    the captured step (sampling.GraphedSteps) of the v1.0 model
  eager_v10      the same step launched op by op
  graphed_v11    the captured step of the v1.1 model (CGModel) of bench.py on the same poses, for comparison
Also one pose of the same complex at t=0.5 against the CPU oracle, and the card's name and power limit.  One JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from functools import partial

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import N_SCHED, TEMPS, model_kwargs, randomise_bn      # noqa: E402
from tools.bench_crop import card                                 # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--poses', type=int, default=40)
    ap.add_argument('--n-res', dest='n_res', type=int, default=1500)
    ap.add_argument('--n-atoms', dest='n_atoms', type=int, default=40)
    ap.add_argument('--no-oracle', dest='no_oracle', action='store_true')
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_old_score.py measures on a CUDA device; none found")
    import __graft_entry__ as ge
    ge.build()
    from diffdock_b200 import ops
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_t_schedule, get_timestep_embedding, set_time, t_to_sigma
    from diffdock_b200.hetero import collate_shared_receptor
    from diffdock_b200.sampling import GraphedSteps, step_coefficients
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    from tests.old_score_helpers import model_pair, score

    dev = torch.device('cuda', 0)
    args = default_model_args()
    t2s = partial(t_to_sigma, args=args)
    oracle, v10, _ = model_pair(seed=0)            # oracle on the CPU, product with the same weights
    assert v10.sync_free_capable()
    torch.manual_seed(0)
    v11 = CGModel(t2s, dev, get_timestep_embedding('sinusoidal', args.sigma_embed_dim, args.embedding_scale),
                  **model_kwargs(args)).eval()
    randomise_bn(v11, 1)
    v11 = v11.to(dev)
    n = cli.poses
    poses = make_pose_list(n, n_res=cli.n_res, n_atoms=cli.n_atoms, seed=100, tr_sigma_max=args.tr_sigma_max)
    sched = get_t_schedule('expbeta', N_SCHED)
    coef = []
    for t_idx in range(N_SCHED):
        c = step_coefficients(t_idx, N_SCHED, sched, sched, sched, t2s, args, False, **TEMPS)
        if t_idx == N_SCHED - 1:
            c[1] = c[3] = c[5] = 0.0
        coef.append(c)
    t_rows = [[float(t)] * 3 for t in sched]
    lig0 = poses[0]['ligand']
    rb = poses[0]['ligand', 'ligand'].edge_index.T[lig0.edge_mask]
    bu, bv = rb[:, 0].int().contiguous().to(dev), rb[:, 1].int().contiguous().to(dev)
    mask = torch.from_numpy(lig0.mask_rotate[0].astype(np.uint8)).to(dev)
    keys = torch.arange(n, device=dev)

    def graphed(model):
        g = collate_shared_receptor(poses, dev)
        s = GraphedSteps(model, g, n, coef, t_rows, bu, bv, mask, True, dev, draw_noise=True, philox=(1234, keys))
        pos0 = s.pos.clone()

        def run():
            s.pos.copy_(pos0)
            s.step.zero_()
            for _ in range(N_SCHED):
                s.graph.replay()
        return s, run

    s_v10, run_v10 = graphed(v10)
    _, run_v11 = graphed(v11)
    g_eager = collate_shared_receptor(poses, dev)
    pos0 = g_eager['ligand'].pos.float().contiguous().clone()
    coef_dev = torch.tensor(coef, dtype=torch.float32, device=dev)

    def run_eager():
        g_eager['ligand'].pos = pos0.clone()
        for t_idx in range(N_SCHED):
            t = float(sched[t_idx])
            set_time(g_eager, None, t, t, t, n, False, dev)
            g_eager._uniform_t = True
            tr, rot, tor = v10(g_eager)
            g_eager['ligand'].pos = ops.pose_update_dev(
                g_eager['ligand'].pos.float().contiguous(), n, bu, bv, mask, tr, rot, tor, coef_dev,
                step_dev=torch.full((1,), t_idx, dtype=torch.int32, device=dev), seed=1234, pose_key=keys)
        return g_eager['ligand'].pos

    arms = {'graphed_v10': run_v10, 'eager_v10': run_eager, 'graphed_v11': run_v11}
    for fn in arms.values():        # warm-up: one whole run each
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(cli.repeats):
        for k, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / N_SCHED)
    ms = {k: float(np.median(v)) for k, v in times.items()}
    # the captured and the op-by-op runs draw the same counter-based noise: their final poses agree
    run_v10()
    eager_pos = run_eager()
    torch.cuda.synchronize()
    graphed_vs_eager = float((s_v10.pos - eager_pos).abs().max() / eager_pos.abs().max())

    parity = None
    if not cli.no_oracle:           # one pose at t = 0.5 against the oracle
        one = make_pose_list(1, n_res=cli.n_res, n_atoms=cli.n_atoms, seed=100, tr_sigma_max=args.tr_sigma_max * 0.5)
        got = score(v10, one, [0.5], dev)
        torch.set_num_threads(min(os.cpu_count() or 1, 32))
        ref = score(oracle, one, [0.5], 'cpu')
        rel = lambda a, b: float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))
        v10._sync_free = False          # the host-sized forward: receptor encoder evaluated whole every step
        host = score(v10, one, [0.5], dev)
        v10._sync_free = None
        parity = {'t': 0.5, 'tolerance': 1e-4}
        for name, out in (('sync_free', got), ('host_sized', host)):
            parity[name] = {'tr_rel_err': rel(out[0], ref[0]), 'rot_rel_err': rel(out[1], ref[1]),
                            'tor_rel_err': rel(out[2], ref[2]) if ref[2].numel() else None}

    line = {'tool': 'bench_old_score', 'card': card(),
            'workload': f'{cli.n_res} residues / {cli.n_atoms} ligand atoms / {n} poses, v1.0 score model at CFG-L2 widths, '
                        f'20-step expbeta schedule',
            'ms_per_step': ms, 'ms_per_step_runs': times,
            'poses_per_s': {k: n / (v * N_SCHED / 1000.0) for k, v in ms.items()},
            'graphed_vs_eager_final_pos_rel_err': graphed_vs_eager,
            'how': f'CUDA events around whole 20-step runs, median of {cli.repeats} alternated repeats after one warm-up run each',
            'parity': parity}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()

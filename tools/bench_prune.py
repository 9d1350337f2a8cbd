#!/usr/bin/env python
"""tools/bench_prune.py - the captured reverse-diffusion step with and without the receptor <- receptor pruning of the
sync-free forward (CGModel._pruned_contact_groups: a layer only computes contact messages into residues that can still pass
a message to a ligand atom).

    python tools/bench_prune.py [--repeats 5]

Workload: BASELINE config 3 (1500 residues / 40 ligand atoms / 40 poses of one synthetic complex, the CFG-L2 model of
bench.py) over the 20-step expbeta schedule, GraphedSteps with Philox noise from one seed.  Two arms of the same model,
``pruned`` (the default) and ``unpruned`` (``_prune_receptor = False``), timed with CUDA events around whole 20-step runs
after one warm-up run each, alternated ``--repeats`` times in this process.  After the timed region: the live contact-edge
count of every layer at every schedule point of one pruned run, the fused kernel's work of both arms weighted by each
layer's (weight tiles + 1) - its cost per edge - and the final coordinates of the two arms against each other and against a
second unpruned run.  The card's name and power limit are read in the same process.  One JSON line.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
from functools import partial

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import N_SCHED, TEMPS, model_kwargs, randomise_bn      # noqa: E402


def card():
    out = subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, power = [s.strip() for s in out.split(',')[:2]]
    return {'name': name, 'power_limit': power, 'torch_name': torch.cuda.get_device_name(0)}


def layer_tiles(layer):
    """Weight tiles of the fused kernel's plan for ``layer`` (diffdock_b200/fused.py:supported)."""
    from diffdock_b200 import fused
    return sum(-(-p.mul_in // fused.CONSUMER_KINDS[(p.mul_out, 2 * p.l_out + 1)][1]) for p in layer.tp.table_vec.paths)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--poses', type=int, default=40)
    ap.add_argument('--n-res', dest='n_res', type=int, default=1500)
    ap.add_argument('--n-atoms', dest='n_atoms', type=int, default=40)
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_prune.py measures on a CUDA device; none found")
    import __graft_entry__ as ge
    ge.build()
    from diffdock_b200 import ops
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_t_schedule, get_timestep_embedding, t_to_sigma
    from diffdock_b200.hetero import collate_shared_receptor
    from diffdock_b200.layers import cross_cutoff
    from diffdock_b200.sampling import GraphedSteps, step_coefficients
    from diffdock_b200.synthetic import default_model_args, make_pose_list

    dev = torch.device('cuda', 0)
    args = default_model_args()
    t2s = partial(t_to_sigma, args=args)
    torch.manual_seed(0)
    model = CGModel(t2s, dev, get_timestep_embedding('sinusoidal', args.sigma_embed_dim, args.embedding_scale),
                    **model_kwargs(args)).eval()
    randomise_bn(model, 1)
    model = model.to(dev)
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

    def graphed(prune):
        model._prune_receptor = prune
        g = collate_shared_receptor(copy.deepcopy(poses), dev)
        s = GraphedSteps(model, g, n, coef, t_rows, bu, bv, mask, True, dev, draw_noise=True, philox=(1234, keys))
        model._prune_receptor = True
        pos0 = s.pos.clone()

        def run():
            s.pos.copy_(pos0)
            s.step.zero_()
            for _ in range(N_SCHED):
                s.graph.replay()
        return s, g, pos0, run

    arms = {'pruned': graphed(True), 'unpruned': graphed(False)}
    for _, _, _, run in arms.values():          # warm-up: one whole run each
        run()
    torch.cuda.synchronize()
    times, final = {k: [] for k in arms}, {k: [] for k in arms}
    for _ in range(cli.repeats):
        for k, (s, _, _, run) in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / N_SCHED)
            final[k].append(s.pos.clone())
    ms = {k: {'median': float(np.median(v)), 'min': float(min(v)), 'max': float(max(v))} for k, v in times.items()}

    # -- untimed: live edge counts of every layer at every schedule point of one pruned run -----------------------------
    s, g, pos0, _ = arms['pruned']
    c = model._static(g)
    key = next(k for k in c if isinstance(k, tuple) and k[0] == 'prune')
    _, bufs = c[key]
    L = len(model.conv_layers)
    shared = c['tiles'] is not None
    levels = model._need_levels(L, shared)
    tiles = [layer_tiles(layer) for layer in model.conv_layers]
    n_rr = int(c['rr_tgt'].shape[0])
    n_rr0 = int(c['tiles']['edges'].shape[0]) if shared else n_rr          # layer 0's shared messages: one receptor copy
    rec, lig = g['receptor'], g['ligand']
    s.pos.copy_(pos0)
    s.step.zero_()
    per_step, work = [], {'pruned': 0.0, 'unpruned': 0.0}
    for t_idx in range(N_SCHED):
        t = float(sched[t_idx])
        r, rpg = cross_cutoff(model, t2s(torch.full((n,), t, device=dev), 0, 0)[0])
        n_x = int(ops.radius_count(rec.pos.float().contiguous(), s.pos, c['rec_ptr'], c['lig_batch32'], r=r, r_per_graph=rpg,
                                   max_num_neighbors=10000).sum())
        n_ll = int(ops.radius_count(s.pos, s.pos, c['lig_ptr'], c['lig_batch32'], r=model.lig_max_radius,
                                    max_num_neighbors=33, exclude_self=True).sum()) + int(c['pre_tgt'].shape[0])
        s.graph.replay()
        torch.cuda.synchronize()
        rr = []
        for l, k in enumerate(levels):
            if l == L - 1:
                rr.append(0)
            elif k is None:
                rr.append(n_rr0)
            else:
                rr.append(int(bufs[k - 1][5].item()))
        rr_full = [0 if l == L - 1 else (n_rr0 if (l == 0 and shared) else n_rr) for l in range(L)]
        for arm, counts in (('pruned', rr), ('unpruned', rr_full)):
            work[arm] += sum((tiles[l] + 1) * (n_ll + (n_x if l == L - 1 else 2 * n_x) + counts[l]) for l in range(L))
        per_step.append({'t': t, 'cross_edges': n_x, 'ligand_edges': n_ll, 'contact_edges_per_layer': rr,
                         'contact_edges_per_layer_unpruned': rr_full})

    ref_a, ref_b = final['unpruned'][0], final['unpruned'][1 if cli.repeats > 1 else 0]
    d = (final['pruned'][0] - ref_a).abs()
    spread = (ref_a - ref_b).abs()
    line = {'tool': 'bench_prune', 'card': card(),
            'workload': f'{cli.n_res} residues / {cli.n_atoms} ligand atoms / {n} poses, CFG-L2, 20-step expbeta schedule, '
                        f'GraphedSteps with Philox noise (seed 1234)',
            'ms_per_step': ms, 'ms_per_step_runs': times,
            'speedup_median': ms['unpruned']['median'] / ms['pruned']['median'],
            'how': f'CUDA events around whole 20-step runs, {cli.repeats} alternated repeats per arm after one warm-up run each',
            'layer_tiles': tiles, 'need_level_per_layer': levels, 'contact_edges_per_pose': n_rr // n,
            'per_step': per_step,
            'weighted_work_ratio': work['pruned'] / work['unpruned'],
            'weighted_work_def': 'sum over steps and layers of (tiles + 1) x live edges (ligand graph + cross edges, both '
                                 'directions except in the last layer, + contact edges); layer 0 runs one receptor copy',
            'final_pos_vs_unpruned_A': {'max': float(d.max()), 'median': float(d.median())},
            'unpruned_run_to_run_A': {'max': float(spread.max()), 'median': float(spread.median())}}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()

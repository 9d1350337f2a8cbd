#!/usr/bin/env python
"""tools/bench_crop.py - reverse-diffusion steps with per-step receptor cropping (crop_beyond, utils/sampling.py:104-109).

    python tools/bench_crop.py [--crop-beyond 20] [--repeats 5]

Workload: BASELINE config 3 (1500 residues / 40 ligand atoms / 40 poses of one synthetic complex, the CFG-L2 model of
bench.py) over the 20-step expbeta schedule.  Three arms, timed with CUDA events over whole 20-step runs after one warm-up
run each, alternated ``--repeats`` times in this process:
  graphed_crop     the captured step with the device-side crop (GraphedSteps(crop_rows=...))
  eager_crop       the op-by-op step through sampling.crop_receptor (what runs without the device-side crop)
  graphed_nocrop   the captured step with crop_beyond=None (bench.py's timed path)
Also: the live receptor-receptor and ligand-receptor edge counts of every step of the graphed crop run, one pose of the same
complex at t=0.5 against the CPU oracle on the reference's cropped batch, and the card's name and power limit.  One JSON line.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--crop-beyond', dest='crop_beyond', type=float, default=20.0)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--poses', type=int, default=40)
    ap.add_argument('--n-res', dest='n_res', type=int, default=1500)
    ap.add_argument('--n-atoms', dest='n_atoms', type=int, default=40)
    ap.add_argument('--no-oracle', dest='no_oracle', action='store_true')
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_crop.py measures on a CUDA device; none found")
    import __graft_entry__ as ge
    ge.build()
    from diffdock_b200 import ops
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_t_schedule, get_timestep_embedding, set_time, t_to_sigma
    from diffdock_b200.hetero import collate, collate_shared_receptor
    from diffdock_b200.layers import cross_cutoff
    from diffdock_b200.sampling import GraphedSteps, crop_cutoff2, crop_receptor, step_coefficients
    from diffdock_b200.synthetic import default_model_args, make_pose_list

    dev = torch.device('cuda', 0)
    args = default_model_args()
    t2s = partial(t_to_sigma, args=args)
    torch.manual_seed(0)
    model = CGModel(t2s, dev, get_timestep_embedding('sinusoidal', args.sigma_embed_dim, args.embedding_scale),
                    **model_kwargs(args)).eval()
    randomise_bn(model, 1)
    model = model.to(dev)
    assert model.sync_free_crop_capable()
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
    crop_rows = [crop_cutoff2(t2s, t, t, t, cli.crop_beyond) for t in sched]
    cutoffs = [float(t2s(t, t, t)[0]) * 3 + cli.crop_beyond for t in sched]
    lig0 = poses[0]['ligand']
    rb = poses[0]['ligand', 'ligand'].edge_index.T[lig0.edge_mask]
    bu, bv = rb[:, 0].int().contiguous().to(dev), rb[:, 1].int().contiguous().to(dev)
    mask = torch.from_numpy(lig0.mask_rotate[0].astype(np.uint8)).to(dev)
    keys = torch.arange(n, device=dev)

    def graphed(crop):
        g = collate_shared_receptor(poses, dev)
        s = GraphedSteps(model, g, n, coef, t_rows, bu, bv, mask, True, dev, draw_noise=True, philox=(1234, keys),
                         crop_rows=crop_rows if crop else None)
        pos0 = s.pos.clone()

        def run():
            s.pos.copy_(pos0)
            s.step.zero_()
            for _ in range(N_SCHED):
                s.graph.replay()
        return s, g, run

    s_crop, g_crop, run_crop = graphed(True)
    _, _, run_nocrop = graphed(False)
    g_eager = collate_shared_receptor(poses, dev)
    pos0 = g_eager['ligand'].pos.float().contiguous().clone()
    coef_dev = torch.tensor(coef, dtype=torch.float32, device=dev)

    def run_eager():
        g_eager['ligand'].pos = pos0.clone()
        for t_idx in range(N_SCHED):
            t = float(sched[t_idx])
            mod = crop_receptor(g_eager, cutoffs[t_idx])
            set_time(mod, None, t, t, t, n, False, dev)
            mod._uniform_t = True
            tr, rot, tor = model(mod)[:3]
            g_eager['ligand'].pos = ops.pose_update_dev(
                g_eager['ligand'].pos.float().contiguous(), n, bu, bv, mask, tr, rot, tor, coef_dev,
                step_dev=torch.full((1,), t_idx, dtype=torch.int32, device=dev), seed=1234, pose_key=keys)

    arms = {'graphed_crop': run_crop, 'eager_crop': run_eager, 'graphed_nocrop': run_nocrop}
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

    # live edge counts of every step of one graphed crop run (recomputed from the pose that enters the step, untimed)
    c = model._static(g_crop)
    rec, lig = g_crop['receptor'], g_crop['ligand']
    s_crop.pos.copy_(pos0)
    s_crop.step.zero_()
    rr32 = (c['rr_tgt'].int().contiguous(), c['rr_src'].int().contiguous())
    counts = []
    for t_idx in range(N_SCHED):
        keep, masked = ops.crop_flags(s_crop.pos, c['lig_ptr'], rec.pos.float().contiguous(), c['rec_batch32'], s_crop.crop,
                                      s_crop.step)
        n_rr = ops.crop_select_edges(*rr32, keep)[4]
        r, rpg = cross_cutoff(model, t2s(torch.full((n,), float(sched[t_idx]), device=dev), 0, 0)[0])
        n_x = ops.radius_count(masked, s_crop.pos, c['rec_ptr'], c['lig_batch32'], r=r, r_per_graph=rpg,
                               max_num_neighbors=10000).sum()
        n_x_full = ops.radius_count(rec.pos.float().contiguous(), s_crop.pos, c['rec_ptr'], c['lig_batch32'], r=r,
                                    r_per_graph=rpg, max_num_neighbors=10000).sum()
        counts.append({'t': float(sched[t_idx]), 'cutoff': cutoffs[t_idx], 'residues_kept': int(keep.sum()),
                       'rec_rec_edges': int(n_rr.item()), 'cross_edges': int(n_x), 'cross_edges_uncropped': int(n_x_full)})
        s_crop.graph.replay()
    torch.cuda.synchronize()

    parity = None
    if not cli.no_oracle:           # one pose at t = 0.5 against the oracle on the reference's cropped batch
        from oracle.diffusion import crop_beyond as o_crop, set_time as o_set_time, t_to_sigma as o_t2s
        from tests.parity_helpers import make_model_pair
        o, p = make_model_pair(args, seed=0)
        t = float(sched[10])
        one = make_pose_list(1, n_res=cli.n_res, n_atoms=cli.n_atoms, seed=100, tr_sigma_max=args.tr_sigma_max * t)
        g1 = collate(one).to(dev)
        set_time(g1, None, t, t, t, 1, False, dev)
        g1._crop = (torch.tensor([crop_cutoff2(t2s, t, t, t, cli.crop_beyond)], device=dev),
                    torch.zeros(1, dtype=torch.int32, device=dev))
        got = p(g1)
        cropped = [o_crop(q, o_t2s(t, t, t, args)[0] * 3 + cli.crop_beyond) for q in copy.deepcopy(one)]
        gc = collate(cropped)
        o_set_time(gc, t, t, t, 1, 'cpu')
        torch.set_num_threads(min(os.cpu_count() or 1, 32))
        with torch.no_grad():
            ref = o(gc)
        rel = lambda a, b: float((a.double().cpu() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))
        parity = {'t': t, 'residues_kept': int(cropped[0]['receptor'].pos.shape[0]), 'residues': cli.n_res,
                  'tr_rel_err': rel(got[0], ref[0]), 'rot_rel_err': rel(got[1], ref[1]),
                  'tor_rel_err': rel(got[2], ref[2]) if ref[2].numel() else None, 'tolerance': 1e-4}

    line = {'tool': 'bench_crop', 'crop_beyond': cli.crop_beyond, 'card': card(),
            'workload': f'{cli.n_res} residues / {cli.n_atoms} ligand atoms / {n} poses, CFG-L2, 20-step expbeta schedule',
            'ms_per_step': ms, 'ms_per_step_runs': times,
            'speedup_graphed_crop_vs_eager_crop': ms['eager_crop'] / ms['graphed_crop'],
            'how': f'CUDA events around whole 20-step runs, median of {cli.repeats} alternated repeats after one warm-up run each',
            'rec_rec_edges_uncropped': int(c['rr_tgt'].shape[0]), 'per_step': counts, 'parity': parity}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()

#!/usr/bin/env python
"""tools/bench_pack_sharded.py - BASELINE config 5 over the GPUs of a box: one ``sampling()`` call per complex against
packed sampling, both sharded by whole complexes.

    torchrun --nproc_per_node=<GPUs> tools/bench_pack_sharded.py [--repeats 3] [--complexes 64] [--poses 40] [--ranker aaold]
    python tools/bench_pack_sharded.py [...]          # one process, no process group

Workload: bench.py's config 5 - ``--complexes`` complexes of ``synthetic.config5_sizes(seed=0)`` (N_r ~ U(200, 600),
N_l ~ U(15, 50)) x ``--poses`` poses, 20 steps, bench.py's CFG-L2 ``CGModel``, inference.py's temperatures,
``no_final_step_noise``, Philox seed 2024 keyed (complex << 32) | pose; each rank builds only the complexes it owns.
Arms, alternated in one process after one untimed warm-up each:
  per_complex  ``distributed.sample_complexes_sharded`` with one ``sampling()`` per complex (``bench.py --workload config5``)
  packed       ``distributed.sample_packed_sharded``: one ``sample_packed`` per rank
``--ranker aaold`` ranks in both arms with an ``AAOldModel`` at the trainer defaults, seeded as in
tools/bench_rank_packed.py, on all-atom confidence graphs of the same complexes.

The timed region starts after a device synchronise and a barrier, includes the gather and ends in a device synchronise and
a barrier; the maximum over ranks is reported.  A rank's busy time is its own sampling: from the start of the region to
its first collective, after a device synchronise there.  Printed on rank 0: one JSON line with the median and min-max per
arm, every rank's busy time (median over repeats), complexes and packs per rank, the max and median |difference| of the
final coordinates (and confidences) between the arms, and the card's name and power limit from the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from argparse import Namespace
from functools import partial

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import TEMPS, model_kwargs, randomise_bn   # noqa: E402
from tools.bench_confidence import WIDTHS           # noqa: E402
from tools.bench_crop import card                   # noqa: E402
from tools.bench_pack import delta, resetter        # noqa: E402
from tools.bench_rank import ranker, stats          # noqa: E402

N_STEPS = 20


def confidence_graphs(poses, n_res, n_atoms, seed):
    """All-atom confidence graphs of ``poses``: each pose's ligand store and residues, plus the receptor atoms of the same
    synthetic complex (``make_complex`` with ``all_atoms`` draws its residues and ligand as without), shared by all poses."""
    from diffdock_b200.hetero import HeteroGraph
    from diffdock_b200.synthetic import make_complex
    base = make_complex(n_res, n_atoms, seed, all_atoms=True)
    out = []
    for d in poses:
        c = HeteroGraph()
        c._nodes['ligand'] = d._nodes['ligand']
        c._edges[('ligand', 'ligand')] = d._edges[('ligand', 'ligand')]
        c._globals.update(d._globals)
        c._nodes['receptor'] = poses[0]._nodes['receptor']
        c._edges[('receptor', 'receptor')] = poses[0]._edges[('receptor', 'receptor')]
        c._nodes['atom'] = base._nodes['atom']
        for et in (('atom', 'atom'), ('atom', 'receptor')):
            c._edges[et] = base._edges[et]
        out.append(c)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--complexes', type=int, default=64)
    ap.add_argument('--poses', type=int, default=40)
    ap.add_argument('--ranker', default='none', choices=['none', 'aaold'])
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pack_sharded.py measures on CUDA devices; none found")
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    import __graft_entry__ as ge
    if rank == 0:
        ge.build()
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
        dist.barrier()
        ge.build()                                       # rank 0 built it; the others only load it
    import diffdock_b200.distributed as D
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_t_schedule, get_timestep_embedding, t_to_sigma
    from diffdock_b200.sampling import PACK_MAX_PAIRS, pack_cost, pack_plan, sampling
    from diffdock_b200.synthetic import config5_sizes, default_model_args, make_pose_list
    info = card() if rank == 0 else None
    args = default_model_args()
    t2s = partial(t_to_sigma, args=args)
    torch.manual_seed(0)
    model = CGModel(t2s, dev, get_timestep_embedding('sinusoidal', args.sigma_embed_dim, args.embedding_scale),
                    **model_kwargs(args)).eval()
    randomise_bn(model, 1)
    model = model.to(dev)
    sched = get_t_schedule('expbeta', N_STEPS)
    rk = cargs = None
    n_cx, P = cli.complexes, cli.poses
    sizes = config5_sizes(n_cx, seed=0)
    costs = [r * a * P for r, a in sizes]
    shapes = [(P, a) for _, a in sizes]
    parts = D.assign_balanced(costs, world)
    mine = parts[rank]
    data = {i: make_pose_list(P, n_res=sizes[i][0], n_atoms=sizes[i][1], seed=1000 + i, tr_sigma_max=args.tr_sigma_max,
                              share_receptor=True) for i in mine}
    conf = {}
    C = 0
    if cli.ranker == 'aaold':
        rk, _ = ranker(WIDTHS['trainer_default'], dev)
        cargs = Namespace(all_atoms=True, crop_beyond=None)
        conf = {i: confidence_graphs(data[i], sizes[i][0], sizes[i][1], 1000 + i) for i in mine}
        C = rk.confidence_predictor[-1].out_features
    reset = resetter([data[i] for i in mine])
    rank_kw = dict(confidence_model=rk, confidence_model_args=cargs) if rk is not None else {}

    def sample_one(i):
        kw = dict(confidence_data_list=conf[i], **rank_kw) if rk is not None else {}
        out, cf = sampling(data[i], model, N_STEPS, sched, sched, sched, dev, t2s, args, batch_size=P,
                           no_final_step_noise=True, rng='philox', seed=2024, pose_keys=(i << 32) + torch.arange(P),
                           **kw, **TEMPS)
        pos = torch.stack([d['ligand'].pos for d in out]).reshape(P, -1)
        return torch.cat([pos, cf.reshape(P, -1)], 1) if rk is not None else pos

    def per_complex():
        flat = D.sample_complexes_sharded(n_cx, costs, [(p, 3 * a + C) for p, a in shapes], sample_one, device=dev)
        return [(f[:, :3 * a].reshape(p, a, 3), f[:, 3 * a:] if C else None) for f, (p, a) in zip(flat, shapes)]

    def packed():
        out = D.sample_packed_sharded(n_cx, costs, shapes, lambda i: (data[i], conf.get(i)), model, N_STEPS, sched,
                                      sched, sched, dev, t2s, args, seed=2024, gather_device=dev,
                                      no_final_step_noise=True, **rank_kw, **TEMPS)
        return [(p, c.reshape(p.shape[0], -1) if c is not None else None) for p, c in out]

    # a rank's busy time ends at its first collective: the gather of the per-complex arm, the status exchange of the
    # packed arm
    mark = {}

    def first_collective(f):
        def wrapped(*a, **kw):
            if 'busy' not in mark:
                torch.cuda.synchronize()
                mark['busy'] = time.perf_counter() - mark['t0']
            return f(*a, **kw)
        return wrapped
    D.gather_ragged = first_collective(D.gather_ragged)
    D.exchange_rows = first_collective(D.exchange_rows)

    def sync_all():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()

    def run(f):
        reset()
        sync_all()
        mark.clear()
        mark['t0'] = time.perf_counter()
        out = f()
        sync_all()
        return out, time.perf_counter() - mark['t0'], mark.get('busy', time.perf_counter() - mark['t0'])

    arms = {'per_complex': per_complex, 'packed': packed}
    times, busy, outs = {k: [] for k in arms}, {k: [] for k in arms}, {}
    for k, f in arms.items():
        _, w, _ = run(f)
        if rank == 0:
            print(f"# warm-up {k}: {w:.1f} s", file=sys.stderr, flush=True)
    for _ in range(cli.repeats):
        for k, f in arms.items():
            outs[k], w, b = run(f)
            t = torch.tensor([w], dtype=torch.float64, device=dev)
            if world > 1:
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
            times[k].append(float(t) * 1e3)
            busy[k].append(b * 1e3)
            if rank == 0:
                print(f"# {k}: {times[k][-1]:.0f} ms", file=sys.stderr, flush=True)
    mine_busy = {k: round(float(np.median(v)), 1) for k, v in busy.items()}
    packs = len(pack_plan([pack_cost(data[i]) for i in mine], PACK_MAX_PAIRS)) if mine else 0
    per_rank = [None] * world
    if world > 1:
        dist.all_gather_object(per_rank, {'busy_ms': mine_busy, 'complexes': len(mine), 'packs': packs})
    else:
        per_rank = [{'busy_ms': mine_busy, 'complexes': len(mine), 'packs': packs}]
    if rank == 0:
        a, b = outs['per_complex'], outs['packed']
        line = {'workload': 'config5', 'world': world, 'complexes': n_cx, 'poses': P, 'steps': N_STEPS,
                'ranker': 'AAOldModel trainer_default' if rk is not None else None, 'max_pairs': PACK_MAX_PAIRS,
                'repeats': cli.repeats, 'ms': {k: stats(v) for k, v in times.items()},
                'poses_per_s': {k: round(n_cx * P / (float(np.median(v)) / 1e3), 2) for k, v in times.items()},
                'busy_ms_per_rank': {k: [r['busy_ms'][k] for r in per_rank] for k in arms},
                'complexes_per_rank': [r['complexes'] for r in per_rank],
                'packs_per_rank': {'per_complex': [r['complexes'] for r in per_rank],
                                   'packed': [r['packs'] for r in per_rank]},
                'coords': delta([p.cpu() for p, _ in a], [p.cpu() for p, _ in b]), 'card': info}
        if rk is not None:
            d = delta([c.cpu() for _, c in a], [c.cpu() for _, c in b])
            line['confidence'] = {'max_abs': d['max_abs_A'], 'median_abs': d['median_abs_A']}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == '__main__':
    main()

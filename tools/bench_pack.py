#!/usr/bin/env python
"""tools/bench_pack.py - several complexes per reverse-diffusion step (``sample_packed``) against one ``sampling()`` call
per complex.

    python tools/bench_pack.py [--repeats 5] [--complexes 64] [--ligands 32] [--skip-config5] [--skip-screening]

Config 5 (BASELINE): ``--complexes`` complexes of ``synthetic.config5_sizes(seed=0)`` (N_r ~ U(200, 600), N_l ~ U(15, 50))
x 40 poses, 20 steps, bench.py's CFG-L2 CGModel, Philox noise keyed (complex << 32) | pose, inference.py's temperatures.
Arms: one ``sampling()`` call per complex (what ``bench.py --workload config5`` does on one GPU) and ``sample_packed``.

Screening: one 1500-residue receptor with ``--ligands`` different ligands of 15-50 atoms, 10 poses each, inference.py's
defaults (19 of 20 steps, its temperatures, no_final_step_noise).  Arms: per-ligand ``sampling()`` calls and
``sample_packed``, each without a ranker and with an AAOldModel ranker at the trainer defaults (all-atom receptor).

Every arm runs once as warm-up, then the arms alternate ``--repeats`` times; medians with min-max of a host clock that ends
in a device synchronise; the max and median |difference| of the final coordinates between the two arms; the card's name and
power limit from the same run.  One JSON line per measurement.
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import TEMPS, model_kwargs, randomise_bn   # noqa: E402
from tools.bench_confidence import WIDTHS           # noqa: E402
from tools.bench_crop import card                   # noqa: E402
from tools.bench_rank import ranker, stats          # noqa: E402


def alternate(arms, repeats, reset):
    """{arm: [ms]}, {arm: last output}: one warm-up run per arm, then the arms in turn; ``reset()`` restores the prior poses
    before every run."""
    times, outs = {k: [] for k in arms}, {}
    for k, f in arms.items():
        reset()
        t0 = time.perf_counter()
        f()
        print(f"# warm-up {k}: {time.perf_counter() - t0:.1f} s", file=sys.stderr, flush=True)
    for _ in range(repeats):
        for k, f in arms.items():
            reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            outs[k] = f()
            torch.cuda.synchronize()
            times[k].append(1e3 * (time.perf_counter() - t0))
            print(f"# {k}: {times[k][-1]:.0f} ms", file=sys.stderr, flush=True)
    return times, outs


def delta(a, b):
    d = torch.cat([(x - y).abs().reshape(-1) for x, y in zip(a, b)])
    return {'max_abs_A': float(d.max()), 'median_abs_A': float(d.median())}


def resetter(complexes):
    start = [[d['ligand'].pos.clone() for d in p] for p in complexes]

    def reset():
        for p, s in zip(complexes, start):
            for d, x in zip(p, s):
                d['ligand'].pos = x
    return reset


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--complexes', type=int, default=64)
    ap.add_argument('--poses', type=int, default=40)
    ap.add_argument('--ligands', type=int, default=32)
    ap.add_argument('--samples', type=int, default=10)
    ap.add_argument('--n-res', dest='n_res', type=int, default=1500)
    ap.add_argument('--skip-config5', dest='skip_config5', action='store_true')
    ap.add_argument('--skip-screening', dest='skip_screening', action='store_true')
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pack.py measures on a CUDA device; none found")
    import __graft_entry__ as ge
    ge.build()
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_t_schedule, get_timestep_embedding, t_to_sigma
    from diffdock_b200.hetero import HeteroGraph
    from diffdock_b200.sampling import pack_plan, PACK_MAX_PAIRS, sample_packed, sampling
    from diffdock_b200.synthetic import config5_sizes, default_model_args, make_complex, make_pose_list
    dev = torch.device('cuda:0')
    info = card()
    args = default_model_args()
    t2s = partial(t_to_sigma, args=args)
    torch.manual_seed(0)
    model = CGModel(t2s, dev, get_timestep_embedding('sinusoidal', args.sigma_embed_dim, args.embedding_scale),
                    **model_kwargs(args)).eval()
    randomise_bn(model, 1)
    model = model.to(dev)
    sched = get_t_schedule('expbeta', 20)

    if not cli.skip_config5:
        print("# building the config-5 complexes", file=sys.stderr, flush=True)
        sizes = config5_sizes(cli.complexes, seed=0)
        cx = [make_pose_list(cli.poses, n_res=r, n_atoms=a, seed=1000 + i, tr_sigma_max=args.tr_sigma_max,
                             share_receptor=True) for i, (r, a) in enumerate(sizes)]
        n_packs = len(pack_plan([cli.poses * r * a for r, a in sizes], PACK_MAX_PAIRS))

        def per_complex():
            return [torch.stack([d['ligand'].pos for d in sampling(
                p, model, 20, sched, sched, sched, dev, t2s, args, batch_size=cli.poses, no_final_step_noise=True,
                rng='philox', seed=2024, pose_keys=(i << 32) + torch.arange(cli.poses), **TEMPS)[0]])
                for i, p in enumerate(cx)]

        def packed():
            return [torch.stack([d['ligand'].pos for d in dl]) for dl, _ in sample_packed(
                cx, model, 20, sched, sched, sched, dev, t2s, args, seed=2024, no_final_step_noise=True, **TEMPS)]

        times, outs = alternate({'per_complex': per_complex, 'packed': packed}, cli.repeats, resetter(cx))
        n = cli.complexes * cli.poses
        print(json.dumps({'workload': 'config5', 'complexes': cli.complexes, 'poses': cli.poses, 'steps': 20,
                          'packs': n_packs, 'max_pairs': PACK_MAX_PAIRS,
                          'ms': {k: stats(v) for k, v in times.items()},
                          'poses_per_s': {k: round(n / (float(np.median(v)) / 1e3), 2) for k, v in times.items()},
                          'coords': delta(outs['per_complex'], outs['packed']), 'card': info}), flush=True)
        del cx, outs

    if not cli.skip_screening:
        base = make_complex(cli.n_res, 20, seed=0, all_atoms=True)
        rng = np.random.default_rng(1)
        atoms = [int(rng.integers(15, 51)) for _ in range(cli.ligands)]
        rec_nodes = {k: base._nodes[k] for k in ('receptor', 'atom')}
        rec_edges = {k: v for k, v in base._edges.items() if k[0] != 'ligand'}
        cx, conf = [], []
        for k, a in enumerate(atoms):
            poses = make_pose_list(cli.samples, n_res=40, n_atoms=a, seed=2000 + k, tr_sigma_max=args.tr_sigma_max)
            score_p, conf_p = [], []
            for d in poses:                        # the ligand of this pose against the one shared receptor
                s, c = HeteroGraph(), HeteroGraph()
                for h in (s, c):
                    h._nodes['ligand'] = d._nodes['ligand']
                    h._edges[('ligand', 'ligand')] = d._edges[('ligand', 'ligand')]
                    h._globals.update(d._globals)
                    h._nodes['receptor'] = rec_nodes['receptor']
                    h._edges[('receptor', 'receptor')] = rec_edges[('receptor', 'receptor')]
                c._nodes['atom'] = rec_nodes['atom']
                for et, st in rec_edges.items():
                    c._edges[et] = st
                score_p.append(s)
                conf_p.append(c)
            cx.append(score_p)
            conf.append(conf_p)
        rk, _ = ranker(WIDTHS['trainer_default'], dev)
        cargs = Namespace(all_atoms=True, crop_beyond=None)

        def per_ligand(rank):
            res = []
            for p, c in zip(cx, conf):
                kw = dict(confidence_model=rk, confidence_data_list=c, confidence_model_args=cargs) if rank else {}
                dl, cf = sampling(p, model, 19, sched, sched, sched, dev, t2s, args, batch_size=cli.samples,
                                  no_final_step_noise=True, rng='philox', seed=7,
                                  pose_keys=(len(res) << 32) + torch.arange(cli.samples), **kw, **TEMPS)
                res.append((torch.stack([d['ligand'].pos for d in dl]), cf))
            return res

        def packed(rank):
            kw = dict(confidence_model=rk, confidence_data=conf, confidence_model_args=cargs) if rank else {}
            out = sample_packed(cx, model, 19, sched, sched, sched, dev, t2s, args, seed=7, no_final_step_noise=True,
                                **kw, **TEMPS)
            return [(torch.stack([d['ligand'].pos for d in dl]), cf) for dl, cf in out]

        arms = {'per_ligand': lambda: per_ligand(False), 'packed': lambda: packed(False),
                'per_ligand_ranked': lambda: per_ligand(True), 'packed_ranked': lambda: packed(True)}
        times, outs = alternate(arms, cli.repeats, resetter(cx))
        conf_d = max(float((a[1] - b[1]).abs().max()) for a, b in zip(outs['per_ligand_ranked'], outs['packed_ranked']))
        print(json.dumps({'workload': 'screening', 'receptor_residues': cli.n_res, 'ligands': cli.ligands,
                          'ligand_atoms': [min(atoms), max(atoms)], 'samples': cli.samples, 'steps': 19,
                          'packs': len(pack_plan([cli.samples * a * cli.n_res for a in atoms], PACK_MAX_PAIRS)),
                          'ms': {k: stats(v) for k, v in times.items()},
                          'coords': delta([o[0] for o in outs['per_ligand']], [o[0] for o in outs['packed']]),
                          'coords_ranked': delta([o[0] for o in outs['per_ligand_ranked']],
                                                 [o[0] for o in outs['packed_ranked']]),
                          'confidence_max_abs': conf_d, 'card': info}), flush=True)


if __name__ == '__main__':
    main()

#!/usr/bin/env python
"""tools/bench_rank_packed.py - the ranking stage of ``sample_packed`` with the v1.0 all-atom ranker ``AAOldModel``
(inference.py's default): one confidence forward per ranking pack against one ``_rank_batch`` per complex.

    python tools/bench_rank_packed.py [--repeats 5] [--ligands 32] [--samples 10] [--n-res 1500] [--complexes 16]
                                      [--poses 40] [--budget-scales 1 8] [--skip-call]

Ranking stage alone (final ligand coordinates already on the device), both widths of tools/bench_confidence.py:
  screening  one ``--n-res``-residue all-atom receptor, ``--ligands`` ligands of 15-50 atoms, ``--samples`` poses each
             (the README's screening run)
  config5    ``--complexes`` config-5-sized complexes (``synthetic.config5_sizes(seed=0)``) with distinct all-atom
             receptors, ``--poses`` poses each
Arms: ``per_complex`` (what sample_packed did before: collate_shared_receptor + one forward per complex) and ``packed_xS``
(``_rank_packed`` with ``S x PACK_MAX_PAIRS`` as the ranking budget; S = 1 is sample_packed's default).  The all-atom pack
cost counts receptor atoms, so at S = 1 most of these complexes exceed the budget on their own and get a pack each.

Whole call (``--skip-call`` to leave out): the screening ``sample_packed`` call at inference.py's defaults (19 of 20 steps,
the default temperatures, bench.py's CGModel score model) with the AAOldModel ranker at the trainer defaults, ranking
complex by complex (the route before this change, forced through ``sampling._rank_route``) against ranking packs.

Every arm warms up twice, then the arms alternate ``--repeats`` times; medians with min-max of a host clock that ends in
a device synchronise; the largest |confidence difference| between the arms; the card's name and power limit from the same
run.  One JSON line per measurement.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from argparse import Namespace
from functools import partial

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import TEMPS, model_kwargs, randomise_bn   # noqa: E402
from tools.bench_confidence import WIDTHS           # noqa: E402
from tools.bench_crop import card                   # noqa: E402
from tools.bench_pack import resetter               # noqa: E402
from tools.bench_rank import alternate, ranker, stats   # noqa: E402


def screening_set(n_res, n_ligands, samples, tr_sigma_max):
    """(score pose lists on the residue graph, confidence pose lists on the all-atom graph) of ``n_ligands`` ligands
    against one receptor; both share each pose's ligand store."""
    from diffdock_b200.hetero import HeteroGraph
    from diffdock_b200.synthetic import make_complex, make_pose_list
    base = make_complex(n_res, 20, seed=0, all_atoms=True)
    rec_edges = {k: v for k, v in base._edges.items() if k[0] != 'ligand'}
    rng = np.random.default_rng(1)
    atoms = [int(rng.integers(15, 51)) for _ in range(n_ligands)]
    cx, conf = [], []
    for k, a in enumerate(atoms):
        score_p, conf_p = [], []
        for d in make_pose_list(samples, n_res=40, n_atoms=a, seed=2000 + k, tr_sigma_max=tr_sigma_max):
            s, c = HeteroGraph(), HeteroGraph()
            for h in (s, c):
                h._nodes['ligand'] = d._nodes['ligand']
                h._edges[('ligand', 'ligand')] = d._edges[('ligand', 'ligand')]
                h._globals.update(d._globals)
                h._nodes['receptor'] = base._nodes['receptor']
                h._edges[('receptor', 'receptor')] = rec_edges[('receptor', 'receptor')]
            c._nodes['atom'] = base._nodes['atom']
            for et, st in rec_edges.items():
                c._edges[et] = st
            score_p.append(s)
            conf_p.append(c)
        cx.append(score_p)
        conf.append(conf_p)
    return cx, conf, atoms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--ligands', type=int, default=32)
    ap.add_argument('--samples', type=int, default=10)
    ap.add_argument('--n-res', dest='n_res', type=int, default=1500)
    ap.add_argument('--complexes', type=int, default=16)
    ap.add_argument('--poses', type=int, default=40)
    ap.add_argument('--budget-scales', dest='scales', type=int, nargs='*', default=[1, 8])
    ap.add_argument('--widths', nargs='*', default=list(WIDTHS))
    ap.add_argument('--skip-call', dest='skip_call', action='store_true')
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rank_packed.py measures on a CUDA device; none found")
    import __graft_entry__ as ge
    ge.build()
    import diffdock_b200.sampling as S
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_t_schedule, get_timestep_embedding, t_to_sigma
    from diffdock_b200.synthetic import config5_sizes, default_model_args, make_pose_list
    dev = torch.device('cuda:0')
    info = card()
    args = default_model_args()
    cargs = Namespace(all_atoms=True, crop_beyond=None)

    # -- the ranking stage alone ----------------------------------------------------------------------------------------
    cx, conf, atoms = screening_set(cli.n_res, cli.ligands, cli.samples, args.tr_sigma_max)
    sizes = config5_sizes(cli.complexes, seed=0)
    c5 = [make_pose_list(cli.poses, n_res=r, n_atoms=a, seed=1000 + i, tr_sigma_max=2.0, all_atoms=True)
          for i, (r, a) in enumerate(sizes)]
    workloads = {'screening': conf, 'config5': c5}
    for name in cli.widths:
        rk, _ = ranker(WIDTHS[name], dev)
        for wl, data in workloads.items():
            finals = [torch.cat([d['ligand'].pos for d in p]).float().to(dev) for p in data]
            costs = [S.pack_cost(p, True) for p in data]
            arms = {'per_complex': lambda: [torch.nan_to_num(S._rank_batch(rk, cargs, p, None, f, len(p), dev), nan=-1000)
                                            for p, f in zip(data, finals)]}
            packs = {}
            for s in cli.scales:
                budget = s * S.PACK_MAX_PAIRS
                packs[f'packed_x{s}'] = len(S.pack_plan(costs, budget))
                arms[f'packed_x{s}'] = partial(S._rank_packed, rk, cargs, data, finals, budget, dev)
            times, outs = alternate(arms, cli.repeats)
            ref = torch.cat(outs['per_complex']).float()
            dconf = {k: float((torch.cat(v).float() - ref).abs().max()) for k, v in outs.items() if k != 'per_complex'}
            print(json.dumps({'measurement': 'ranking_stage', 'workload': wl, 'width': name, **WIDTHS[name],
                              'complexes': len(data), 'poses': sum(len(p) for p in data),
                              'receptor_atoms': [min(p[0]['atom'].num_nodes for p in data),
                                                 max(p[0]['atom'].num_nodes for p in data)],
                              'packs': packs, 'max_pairs': S.PACK_MAX_PAIRS, 'repeats': cli.repeats,
                              'ms': {k: stats(v) for k, v in times.items()}, 'max_abs_dconf': dconf, 'card': info}),
                  flush=True)
            del finals, outs
        del rk
        torch.cuda.empty_cache()
    del c5, workloads
    if cli.skip_call:
        return

    # -- the whole screening sample_packed call with the ranker -----------------------------------------------------------
    t2s = partial(t_to_sigma, args=args)
    torch.manual_seed(0)
    score = CGModel(t2s, dev, get_timestep_embedding('sinusoidal', args.sigma_embed_dim, args.embedding_scale),
                    **model_kwargs(args)).eval()
    randomise_bn(score, 1)
    score = score.to(dev)
    rk, _ = ranker(WIDTHS['trainer_default'], dev)
    sched = get_t_schedule('expbeta', 20)
    real_route = S._rank_route

    def call(per_complex):
        if per_complex:
            S._rank_route = lambda *a: 'complex' if real_route(*a) == 'packed' else real_route(*a)
        try:
            out = S.sample_packed(cx, score, 19, sched, sched, sched, dev, t2s, args, seed=7, no_final_step_noise=True,
                                  confidence_model=rk, confidence_data=conf, confidence_model_args=cargs, **TEMPS)
        finally:
            S._rank_route = real_route
        return torch.cat([c for _, c in out])

    reset = resetter(cx)

    def arm(per_complex):
        reset()
        return call(per_complex)

    times, outs = alternate({'rank_per_complex': lambda: arm(True), 'rank_packed': lambda: arm(False)}, cli.repeats)
    print(json.dumps({'measurement': 'sample_packed_call', 'workload': 'screening', 'receptor_residues': cli.n_res,
                      'ligands': cli.ligands, 'ligand_atoms': [min(atoms), max(atoms)], 'samples': cli.samples,
                      'steps': '19 of 20', 'score_model': 'CGModel (bench.py)', 'ranker': 'AAOldModel trainer_default',
                      'ranking_packs': len(S.pack_plan([S.pack_cost(p, True) for p in conf], S.PACK_MAX_PAIRS)),
                      'repeats': cli.repeats, 'ms': {k: stats(v) for k, v in times.items()},
                      'max_abs_dconf': float((outs['rank_per_complex'] - outs['rank_packed']).abs().max()),
                      'card': info}), flush=True)


if __name__ == '__main__':
    main()

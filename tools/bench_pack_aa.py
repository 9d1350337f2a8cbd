#!/usr/bin/env python
"""tools/bench_pack_aa.py - several complexes per reverse-diffusion step (``sample_packed``) against one ``sampling()`` call
per complex, with an all-atom score model (``AAModel``).

    python tools/bench_pack_aa.py [--repeats 3] [--complexes 16] [--poses 10] [--ligands 16] [--samples 10]
                                  [--n-res 500] [--skip-config5] [--skip-screening]

The score model is bench.py's CFG-L2 widths (ns=48, nv=10, six layers, precomputed language-model residue features) built
as an ``AAModel``, seeded, BatchNorm statistics randomised.  Philox noise keyed (complex << 32) | pose, inference.py's
temperatures, ``PACK_MAX_PAIRS`` as the budget, whose cost now counts residues + receptor atoms.

Config-5-like: ``--complexes`` all-atom complexes of ``synthetic.config5_sizes(seed=0)`` (N_r ~ U(200, 600), N_l ~
U(15, 50), 3-7 receptor atoms per residue) x ``--poses`` poses, 20 steps.  At config 5's 40 poses most of these complexes
exceed the budget on their own; the default 10 poses let packs hold several.

Screening: one ``--n-res``-residue all-atom receptor with ``--ligands`` ligands of 15-50 atoms, ``--samples`` poses each, 19
of 20 steps (inference.py's defaults).

Every arm runs once as warm-up, then the arms alternate ``--repeats`` times; medians with min-max of a host clock that ends
in a device synchronise; the number of packs; the max and median |difference| of the final coordinates between the arms;
the card's name and power limit from the same run.  One JSON line per workload.
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

from bench import TEMPS, model_kwargs, randomise_bn   # noqa: E402
from tools.bench_crop import card                   # noqa: E402
from tools.bench_pack import alternate, delta, resetter   # noqa: E402
from tools.bench_rank import stats                  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--complexes', type=int, default=16)
    ap.add_argument('--poses', type=int, default=10)
    ap.add_argument('--ligands', type=int, default=16)
    ap.add_argument('--samples', type=int, default=10)
    ap.add_argument('--n-res', dest='n_res', type=int, default=500)
    ap.add_argument('--skip-config5', dest='skip_config5', action='store_true')
    ap.add_argument('--skip-screening', dest='skip_screening', action='store_true')
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pack_aa.py measures on a CUDA device; none found")
    import __graft_entry__ as ge
    ge.build()
    from diffdock_b200.aa_model import AAModel
    from diffdock_b200.diffusion_utils import get_t_schedule, get_timestep_embedding, t_to_sigma
    from diffdock_b200.hetero import HeteroGraph
    from diffdock_b200.sampling import PACK_MAX_PAIRS, pack_cost, pack_plan, sample_packed, sampling
    from diffdock_b200.synthetic import config5_sizes, default_model_args, make_complex, make_pose_list
    dev = torch.device('cuda:0')
    info = card()
    args = default_model_args(all_atoms=True)
    t2s = partial(t_to_sigma, args=args)
    torch.manual_seed(0)
    model = AAModel(t2s, dev, get_timestep_embedding('sinusoidal', args.sigma_embed_dim, args.embedding_scale),
                    **model_kwargs(args)).eval()
    randomise_bn(model, 1)
    model = model.to(dev)
    assert model.sync_free_capable()
    sched = get_t_schedule('expbeta', 20)

    def run_pair(cx, steps, keyed):
        def per_complex():
            return [torch.stack([d['ligand'].pos for d in sampling(
                p, model, steps, sched, sched, sched, dev, t2s, args, batch_size=len(p), no_final_step_noise=True,
                rng='philox', seed=2024, pose_keys=(i << 32) + torch.arange(len(p)), **TEMPS)[0]])
                for i, p in enumerate(cx)]

        def packed():
            return [torch.stack([d['ligand'].pos for d in dl]) for dl, _ in sample_packed(
                cx, model, steps, sched, sched, sched, dev, t2s, args, seed=2024, no_final_step_noise=True, **TEMPS)]

        times, outs = alternate({keyed: per_complex, 'packed': packed}, cli.repeats, resetter(cx))
        return dict(packs=len(pack_plan([pack_cost(p, all_atoms=True) for p in cx], PACK_MAX_PAIRS)),
                    max_pairs=PACK_MAX_PAIRS, ms={k: stats(v) for k, v in times.items()},
                    coords=delta(outs[keyed], outs['packed']), card=info)

    if not cli.skip_config5:
        print("# building the config-5-like all-atom complexes", file=sys.stderr, flush=True)
        sizes = config5_sizes(cli.complexes, seed=0)
        cx = [make_pose_list(cli.poses, n_res=r, n_atoms=a, seed=1000 + i, tr_sigma_max=args.tr_sigma_max,
                             all_atoms=True) for i, (r, a) in enumerate(sizes)]
        res = run_pair(cx, 20, 'per_complex')
        n = cli.complexes * cli.poses
        print(json.dumps({'workload': 'config5_aa', 'complexes': cli.complexes, 'poses': cli.poses, 'steps': 20,
                          'receptor_atoms': [min(p[0]['atom'].num_nodes for p in cx), max(p[0]['atom'].num_nodes for p in cx)],
                          'poses_per_s': {k: round(n / (v['median'] / 1e3), 2) for k, v in res['ms'].items()}, **res}),
              flush=True)
        del cx

    if not cli.skip_screening:
        print("# building the screening set", file=sys.stderr, flush=True)
        base = make_complex(cli.n_res, 20, seed=0, all_atoms=True)
        rec_nodes = {k: base._nodes[k] for k in ('receptor', 'atom')}
        rec_edges = {k: v for k, v in base._edges.items() if k[0] != 'ligand'}
        rng = np.random.default_rng(1)
        atoms = [int(rng.integers(15, 51)) for _ in range(cli.ligands)]
        cx = []
        for k, a in enumerate(atoms):
            poses = make_pose_list(cli.samples, n_res=40, n_atoms=a, seed=2000 + k, tr_sigma_max=args.tr_sigma_max)
            score_p = []
            for d in poses:                        # the ligand of this pose against the one shared all-atom receptor
                s = HeteroGraph()
                s._nodes['ligand'] = d._nodes['ligand']
                s._edges[('ligand', 'ligand')] = d._edges[('ligand', 'ligand')]
                s._globals.update(d._globals)
                s._nodes.update(rec_nodes)
                s._edges.update(rec_edges)
                score_p.append(s)
            cx.append(score_p)
        res = run_pair(cx, 19, 'per_ligand')
        print(json.dumps({'workload': 'screening_aa', 'receptor_residues': cli.n_res,
                          'receptor_atoms': int(base['atom'].num_nodes), 'ligands': cli.ligands,
                          'ligand_atoms': [min(atoms), max(atoms)], 'samples': cli.samples, 'steps': 19, **res}), flush=True)


if __name__ == '__main__':
    main()

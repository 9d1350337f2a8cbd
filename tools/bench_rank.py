#!/usr/bin/env python
"""tools/bench_rank.py - the ranking stage of a docking run with the v1.0 all-atom confidence model ``AAOldModel``
(inference.py's default ranker, ``--old_confidence_model``), before and after the shared-receptor route.

    python tools/bench_rank.py [--repeats 7] [--poses 40] [--n-res 1500] [--n-atoms 40] [--samples 10]

Part 1, the ranking stage as ``sampling()`` performs it (utils/sampling.py:208-227): the BASELINE config-3 complex
(1500 residues / 40 ligand atoms, 1280-wide LM embedding) with its synthetic all-atom receptor, ``--poses`` deep copies
(inference.py's N copies of one complex) as the confidence_data_list, and the final ligand positions on the device.  Arms:
  old   deep copy of the list, general collate, final positions device -> host, upload, host-sized AAOldModel forward
  new   shared-receptor collate (one receptor copy uploaded, tiled on the device), positions device -> device,
        ``_uniform_t``, the sync-free AAOldModel forward with shared layer-0 messages
Host clock from the start of the stage to a device synchronise; both widths of tools/bench_confidence.py; the largest
|confidence difference| between the arms.

Part 2, a whole ``sampling()`` call at inference.py's defaults: ``--samples`` poses, 19 of 20 steps, the default
temperatures, no_final_step_noise, a CGModel score model (bench.py's) and an AAOldModel ranker at the trainer defaults.
Three calls alternate: without a ranker, with the ranker on the old route, with it on the new route; the ranking share is
(call with ranker - call without) / call with ranker.  The old route is forced by hiding the item type from
``sampling()``'s dispatch and disabling the sync-free forward, which is what the parent commit ran.

Each arm runs twice as warm-up, then the arms alternate ``--repeats`` times; medians with min-max; the card's name and
power limit from the same run.  One JSON line per measurement.
"""
from __future__ import annotations

import argparse
import copy
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


def ranker(w, dev):
    """(sync-free, host-sized) AAOldModel of width ``w`` with identical seeded weights."""
    from diffdock_b200.diffusion_utils import get_timestep_embedding
    from diffdock_b200.old_aa_model import AAOldModel
    E = w['emb']
    torch.manual_seed(0)
    m = AAOldModel(None, dev, get_timestep_embedding('sinusoidal', E, 1000), sigma_embed_dim=E, sh_lmax=2, ns=w['ns'],
                   nv=w['nv'], num_conv_layers=w['num_conv_layers'], lig_max_radius=5.0, rec_max_radius=30.0,
                   cross_max_distance=80.0, distance_embed_dim=E, cross_distance_embed_dim=E, dynamic_max_cross=False,
                   confidence_mode=True, lm_embedding_type='esm', use_old_atom_encoder=True).eval()
    randomise_bn(m, 1)
    host = copy.deepcopy(m)
    host._sync_free = False
    m, host = m.to(dev), host.to(dev)
    assert m.sync_free_capable()
    return m, host


def stats(v):
    return {'median': round(float(np.median(v)), 3), 'min': round(min(v), 3), 'max': round(max(v), 3)}


def alternate(arms, repeats):
    """{arm: [ms]} and {arm: last output}: two warm-up runs per arm, then the arms in turn ``repeats`` times."""
    for f in arms.values():
        f(), f()
    times, outs = {k: [] for k in arms}, {}
    for _ in range(repeats):
        for k, f in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            outs[k] = f()
            torch.cuda.synchronize()
            times[k].append(1e3 * (time.perf_counter() - t0))
    return times, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=7)
    ap.add_argument('--poses', type=int, default=40)
    ap.add_argument('--n-res', dest='n_res', type=int, default=1500)
    ap.add_argument('--n-atoms', dest='n_atoms', type=int, default=40)
    ap.add_argument('--samples', type=int, default=10)
    ap.add_argument('--widths', nargs='*', default=list(WIDTHS))
    ap.add_argument('--skip-sampling', dest='skip_sampling', action='store_true')
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rank.py measures on a CUDA device; none found")
    import __graft_entry__ as ge
    ge.build()
    import diffdock_b200.sampling as S
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_t_schedule, get_timestep_embedding, set_time, t_to_sigma
    from diffdock_b200.hetero import collate, collate_shared_receptor
    from diffdock_b200.synthetic import default_model_args, make_pose_list

    dev = torch.device('cuda', 0)
    info = card()
    conf_list = make_pose_list(cli.poses, n_res=cli.n_res, n_atoms=cli.n_atoms, seed=3, tr_sigma_max=2.0, all_atoms=True)
    final = torch.cat([p['ligand'].pos for p in conf_list]).float().to(dev)

    # -- part 1: the ranking stage ------------------------------------------------------------------------------------
    for name in cli.widths:
        new_m, old_m = ranker(WIDTHS[name], dev)
        b = len(conf_list)

        def old():                                        # the parent commit's sampling.py:474-481
            cg = collate(copy.deepcopy(conf_list))
            cg['ligand'].pos = final.cpu()
            cg = cg.to(dev)
            set_time(cg, 0, 0, 0, 0, b, True, dev)
            return old_m(cg)

        def new():                                        # this commit's route for HeteroGraph items
            cg = collate_shared_receptor(conf_list, dev)
            cg['ligand'].pos = final.clone()
            set_time(cg, 0, 0, 0, 0, b, True, dev)
            cg._uniform_t = True
            return new_m(cg)

        times, outs = alternate({'old': old, 'new': new}, cli.repeats)
        print(json.dumps({'measurement': 'ranking_stage', 'width': name, **WIDTHS[name], 'poses': cli.poses,
                          'n_res': cli.n_res, 'n_atoms': cli.n_atoms, 'repeats': cli.repeats,
                          'ms': {k: stats(v) for k, v in times.items()},
                          'max_abs_dconf': float((outs['old'].float() - outs['new'].float()).abs().max()),
                          'card': info}), flush=True)
        del new_m, old_m
        torch.cuda.empty_cache()
    if cli.skip_sampling:
        return

    # -- part 2: a whole sampling() call at inference.py's defaults ---------------------------------------------------
    args = default_model_args()
    t2s = partial(t_to_sigma, args=args)
    torch.manual_seed(0)
    score = CGModel(t2s, dev, get_timestep_embedding('sinusoidal', args.sigma_embed_dim, args.embedding_scale),
                    **model_kwargs(args)).eval()
    randomise_bn(score, 1)
    score = score.to(dev)
    new_m, old_m = ranker(WIDTHS['trainer_default'], dev)
    n = cli.samples
    poses = make_pose_list(n, n_res=cli.n_res, n_atoms=cli.n_atoms, seed=3, tr_sigma_max=args.tr_sigma_max)
    ranks = make_pose_list(n, n_res=cli.n_res, n_atoms=cli.n_atoms, seed=3, tr_sigma_max=args.tr_sigma_max, all_atoms=True)
    sched = get_t_schedule('expbeta', 20)
    conf_args = Namespace(all_atoms=True, crop_beyond=None)

    class Hidden:                                           # not a HeteroGraph to the dispatch: the old route
        pass

    def call(conf_model, old_route=False):
        kw = dict(confidence_model=conf_model, confidence_data_list=ranks, confidence_model_args=conf_args) \
            if conf_model is not None else {}
        real = S.HeteroGraph
        if old_route:
            S.HeteroGraph = Hidden
        try:
            _, conf = S.sampling(copy.deepcopy(poses), score, 19, sched, sched, sched, dev, t2s, args, batch_size=n,
                                 no_final_step_noise=True, **TEMPS, **kw)
        finally:
            S.HeteroGraph = real
        return conf

    torch.manual_seed(7)
    times, outs = alternate({'score_only': lambda: call(None), 'old_route': lambda: call(old_m, True),
                             'new_route': lambda: call(new_m)}, cli.repeats)
    med = {k: float(np.median(v)) for k, v in times.items()}
    share = {k: round((med[k] - med['score_only']) / med[k], 4) for k in ('old_route', 'new_route')}
    print(json.dumps({'measurement': 'sampling_call', 'samples': n, 'steps': '19 of 20', 'score_model': 'CGModel (bench.py)',
                      'ranker': 'AAOldModel trainer_default', 'repeats': cli.repeats,
                      'ms': {k: stats(v) for k, v in times.items()}, 'ranking_share': share, 'card': info}), flush=True)


if __name__ == '__main__':
    main()

#!/usr/bin/env python
"""tools/bench_confidence.py - one confidence pass (the ranking call after sampling, utils/sampling.py:208-227) of the
all-atom confidence model the current training code builds: ``AAModel(confidence_mode=True)``.

    python tools/bench_confidence.py [--repeats 7] [--poses 40] [--n-res 1500] [--n-atoms 40]

Workload: the BASELINE config-3 complex (1500 residues / 40 ligand atoms, 1280-wide LM embedding) with its synthetic
all-atom receptor, 40 poses collated into one batch at t = 0, seeded weights and BatchNorm statistics.  Two widths: the
confidence trainer's defaults (ns=16, nv=4, 2 layers, 32-dim embeddings, confidence/confidence_train.py) and the CFG-L2
widths (ns=48, nv=10, 3 layers, 64-dim embeddings).  Arms:
  sync_free    AAModel(confidence_mode=True): the sync-free forward and the one-kernel confidence head
  host_sized   a copy of the same model with ``_sync_free = False``: exactly-sized neighbour lists read back to the host
  v10          AAOldModel (the DiffDock v1.0 all-atom confidence class) of the same widths, for comparison
Every pass gets a fresh device copy of the batch (the per-batch constants are part of a confidence call).  Each arm runs
twice as warm-up, then the arms alternate ``--repeats`` times; CUDA events around the forward, median reported.  Also the
largest |confidence difference| between sync_free and host_sized, and the card's name and power limit.  One JSON line per
width.
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

from bench import randomise_bn                      # noqa: E402
from tools.bench_crop import card                   # noqa: E402

WIDTHS = {'trainer_default': dict(ns=16, nv=4, num_conv_layers=2, emb=32),
          'cfg_l2': dict(ns=48, nv=10, num_conv_layers=3, emb=64)}


def models(w, dev):
    from diffdock_b200.aa_model import AAModel
    from diffdock_b200.diffusion_utils import get_timestep_embedding
    from diffdock_b200.old_aa_model import AAOldModel
    E = w['emb']
    kw = dict(sigma_embed_dim=E, sh_lmax=2, ns=w['ns'], nv=w['nv'], num_conv_layers=w['num_conv_layers'],
              lig_max_radius=5.0, rec_max_radius=30.0, cross_max_distance=80.0, distance_embed_dim=E,
              cross_distance_embed_dim=E, dynamic_max_cross=False, confidence_mode=True)
    emb = get_timestep_embedding('sinusoidal', E, 1000)
    torch.manual_seed(0)
    new = AAModel(None, dev, emb, lm_embedding_type='precomputed', embed_also_ligand=True, **kw).eval()
    randomise_bn(new, 1)
    torch.manual_seed(0)
    old = AAOldModel(None, dev, emb, lm_embedding_type='esm', use_old_atom_encoder=True, **kw).eval()
    randomise_bn(old, 1)
    host = copy.deepcopy(new)
    host._sync_free = False
    return new.to(dev), host.to(dev), old.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=7)
    ap.add_argument('--poses', type=int, default=40)
    ap.add_argument('--n-res', dest='n_res', type=int, default=1500)
    ap.add_argument('--n-atoms', dest='n_atoms', type=int, default=40)
    ap.add_argument('--widths', nargs='*', default=list(WIDTHS))
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_confidence.py measures on a CUDA device; none found")
    import __graft_entry__ as ge
    ge.build()
    from diffdock_b200.diffusion_utils import set_time
    from diffdock_b200.hetero import collate
    from diffdock_b200.synthetic import make_pose_list

    dev = torch.device('cuda', 0)
    poses = make_pose_list(cli.poses, n_res=cli.n_res, n_atoms=cli.n_atoms, seed=3, tr_sigma_max=2.0, all_atoms=True,
                           share_receptor=True)
    pristine = collate(poses).to(dev)
    set_time(pristine, 0, 0, 0, 0, cli.poses, True, dev)
    info = card()
    for name in cli.widths:
        new, host, old = models(WIDTHS[name], dev)
        assert new.sync_free_capable()
        arms = {'sync_free': new, 'host_sized': host, 'v10': old}

        def one(m):
            b = copy.deepcopy(pristine)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.no_grad():
                e0.record()
                out = m(b)
                e1.record()
            torch.cuda.synchronize()
            conf = out[0] if isinstance(out, tuple) else out
            return e0.elapsed_time(e1), conf.float().cpu()

        for m in arms.values():
            one(m), one(m)
        times = {k: [] for k in arms}
        confs = {}
        for _ in range(cli.repeats):
            for k, m in arms.items():
                t, confs[k] = one(m)
                times[k].append(t)
        res = {'width': name, **{k: v for k, v in WIDTHS[name].items()}, 'poses': cli.poses, 'n_res': cli.n_res,
               'n_atoms': cli.n_atoms, 'repeats': cli.repeats,
               'ms_per_pass': {k: round(float(np.median(v)), 3) for k, v in times.items()},
               'ms_spread': {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
               'max_abs_dconf_sync_free_vs_host_sized': float((confs['sync_free'] - confs['host_sized']).abs().max()),
               'card': info}
        print(json.dumps(res), flush=True)
        del new, host, old, arms
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()

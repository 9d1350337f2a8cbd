#!/usr/bin/env python
"""tools/bench_pose_metrics.py - the pose metrics of evaluation (evaluate.py:474-505) per complex on the CPU against one
device launch for many complexes.

    python tools/bench_pose_metrics.py [--complexes 64] [--poses 40] [--repeats 5] [--skip-cpu]

Molecules: the heavy-atom graphs of tests/golden/ref_pose_metrics.pt (M = 1 to 5184 automorphisms), one crystal pose
each; a complex's poses are its crystal pose relabelled by random automorphisms plus 0.5 A of noise (seeded).
Arms, one JSON line each:
  cpu_reference     per complex (``--poses`` poses, one crystal pose), what evaluate.py does on the host: spyrmsd's
                    ``symmrmsd`` (its own enumeration included) if spyrmsd is importable, else oracle/metrics.py's
                    brute-force loop over the enumerated automorphisms plus the enumeration; then the centroid and
                    self-distance expressions.  Median over ``--repeats`` runs, per molecule.
  host_enumeration  ``evaluation.ligand_automorphisms`` per molecule (once per molecule in a run).
  device_launch     one ``pose_metrics_packed`` call over ``--complexes`` complexes (the molecules in turn) x ``--poses``
                    poses, tables and crystal poses already on the device; CUDA events around the call over
                    ``--repeats`` x 20 calls after a warm-up, median and min-max per call; the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'ref_pose_metrics.pt')


def molecules():
    cases = torch.load(GOLDEN, weights_only=False)['cases']
    return {k: (c['atomic_nums'].numpy(), c['bonds'].numpy(), c['refs'][0].numpy()) for k, c in cases.items()}


def make_poses(ref, table, n_poses, rng):
    """``n_poses`` copies of ``ref`` relabelled by random automorphisms, plus noise: float32 values in float64."""
    out = np.empty((n_poses,) + ref.shape)
    for p in range(n_poses):
        s = table[int(rng.integers(0, len(table)))]
        out[p, s] = ref + rng.normal(scale=0.5, size=ref.shape)
    return out.astype(np.float32).astype(np.float64)


def cpu_reference(z, bonds, ref, poses):
    """One complex's metrics the way evaluate.py computes them on the host; returns the formulation's name."""
    n = len(z)
    try:
        from spyrmsd import rmsd as srmsd
        am = np.zeros((n, n), dtype=int)
        for u, v in bonds:
            am[u, v] = am[v, u] = 1
        srmsd.symmrmsd(ref, [p for p in poses], z, z, am, am)
        name = 'spyrmsd'
    except ImportError:
        from diffdock_b200.evaluation import ligand_automorphisms
        from oracle.metrics import pose_metrics
        pose_metrics(poses, ref[None], ligand_automorphisms(z, bonds)[0].numpy())
        name = 'oracle'
    np.min(np.linalg.norm(poses.mean(axis=1)[None, :] - ref[None].mean(axis=1)[:, None], axis=2), axis=0)
    d = np.linalg.norm(poses[:, :, None, :] - poses[:, None, :, :], axis=-1)
    np.min(np.where(np.eye(n), np.inf, d), axis=(1, 2))
    return name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--complexes', type=int, default=64)
    ap.add_argument('--poses', type=int, default=40)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--skip-cpu', action='store_true')
    a = ap.parse_args()
    from diffdock_b200.evaluation import ligand_automorphisms, pose_metrics_packed
    rng = np.random.default_rng(0)
    mols = molecules()

    ligand_automorphisms([6, 6], [(0, 1)])          # first call imports networkx's matcher
    tables, enum_ms = {}, {}
    for k, (z, bonds, _) in mols.items():
        t0 = time.perf_counter()
        tables[k] = ligand_automorphisms(z, bonds)[0]
        enum_ms[k] = (time.perf_counter() - t0) * 1e3
    print(json.dumps({'arm': 'host_enumeration', 'ms_per_molecule': {k: round(v, 3) for k, v in enum_ms.items()},
                      'automorphisms': {k: int(t.shape[0]) for k, t in tables.items()}}))

    if not a.skip_cpu:
        per, name = {}, None
        for k, (z, bonds, ref) in mols.items():
            poses = make_poses(ref, tables[k].numpy(), a.poses, rng)
            ts = []
            for _ in range(a.repeats):
                t0 = time.perf_counter()
                name = cpu_reference(z, bonds, ref, poses)
                ts.append((time.perf_counter() - t0) * 1e3)
            per[k] = round(statistics.median(ts), 3)
        print(json.dumps({'arm': 'cpu_reference', 'formulation': name, 'poses': a.poses, 'crystal_poses': 1,
                          'median_ms_per_complex': per, 'mean_over_molecules_ms': round(float(np.mean(list(per.values()))), 3)}))

    if not torch.cuda.is_available():
        raise SystemExit("device_launch needs a CUDA device")
    from tools.bench_crop import card
    dev = 'cuda:0'
    names = list(mols)
    poses, refs, auts = [], [], []
    for c in range(a.complexes):
        k = names[c % len(names)]
        ref = mols[k][2]
        poses.append(torch.from_numpy(make_poses(ref, tables[k].numpy(), a.poses, rng)).float().to(dev))
        refs.append(torch.from_numpy(ref[None]).to(dev))
        auts.append(tables[k].to(dev))
    for _ in range(3):
        pose_metrics_packed(poses, refs, auts)
    torch.cuda.synchronize()
    ms = []
    for _ in range(a.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            pose_metrics_packed(poses, refs, auts)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / 20)
    print(json.dumps({'arm': 'device_launch', 'complexes': a.complexes, 'poses': a.poses, 'crystal_poses': 1,
                      'molecules': names, 'median_ms_per_call': round(statistics.median(ms), 4),
                      'min_ms': round(min(ms), 4), 'max_ms': round(max(ms), 4), 'card': card()}))


if __name__ == '__main__':
    main()

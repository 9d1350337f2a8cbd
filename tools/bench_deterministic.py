#!/usr/bin/env python
"""tools/bench_deterministic.py - the cost of ``torch.use_deterministic_algorithms(True)`` (fixed-point convolution
scatter, DESIGN section 6.7), flag off against flag on, in one process on one GPU.

    CUBLAS_WORKSPACE_CONFIG=:4096:8 python tools/bench_deterministic.py [--repeats 5] [--complexes 64] [--poses 40]

Arms, alternated after one untimed warm-up each, median and min-max over ``--repeats``:
  step_off / step_on / step_on_nofill   bench.py's config-3 workload (1500 residues, 40 atoms, 40 poses, CFG-L2 CGModel):
                                        one captured reverse-diffusion step replayed, ms per step (mean over 20 replays);
                                        ``_nofill`` with ``torch.utils.deterministic.fill_uninitialized_memory`` off
  packed_off / packed_on                one ``sample_packed`` call over bench.py's config 5 (``--complexes`` x ``--poses``,
                                        20 steps, Philox seed 2024)
Printed: one JSON line with the times, the largest |difference| of the final coordinates between the arms (config 3
after 20 steps; config 5), whether two flag-on runs were bit-equal, and the card's name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from functools import partial

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import TEMPS, model_kwargs, randomise_bn   # noqa: E402
from tools.bench_crop import card                   # noqa: E402
from tools.bench_pack import resetter               # noqa: E402
from tools.bench_rank import stats                  # noqa: E402

STEPS = 20


class _Flag:
    """The deterministic flag (and the uninitialised-memory fill) set for the body of a with-block."""

    def __init__(self, on, fill=True):
        self.on, self.fill = on, fill

    def __enter__(self):
        self.prev = (torch.are_deterministic_algorithms_enabled(), torch.utils.deterministic.fill_uninitialized_memory)
        torch.use_deterministic_algorithms(self.on)
        torch.utils.deterministic.fill_uninitialized_memory = self.fill

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(self.prev[0])
        torch.utils.deterministic.fill_uninitialized_memory = self.prev[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--complexes', type=int, default=64)
    ap.add_argument('--poses', type=int, default=40)
    ap.add_argument('--n-res', dest='n_res', type=int, default=1500)
    ap.add_argument('--n-atoms', dest='n_atoms', type=int, default=40)
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deterministic.py measures on a CUDA device; none found")
    os.environ.setdefault('CUBLAS_WORKSPACE_CONFIG', ':4096:8')
    import __graft_entry__ as ge
    ge.build()
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_t_schedule, get_timestep_embedding, t_to_sigma
    from diffdock_b200.hetero import collate_shared_receptor
    from diffdock_b200.sampling import GraphedSteps, sample_packed, step_coefficients
    from diffdock_b200.synthetic import config5_sizes, default_model_args, make_pose_list
    dev = torch.device('cuda:0')
    info = card()
    args = default_model_args()
    t2s = partial(t_to_sigma, args=args)
    torch.manual_seed(0)
    model = CGModel(t2s, dev, get_timestep_embedding('sinusoidal', args.sigma_embed_dim, args.embedding_scale),
                    **model_kwargs(args)).eval()
    randomise_bn(model, 1)
    model = model.to(dev)
    sched = get_t_schedule('expbeta', STEPS)

    # ---- config 3: the captured step
    poses = make_pose_list(cli.poses, n_res=cli.n_res, n_atoms=cli.n_atoms, seed=100, tr_sigma_max=args.tr_sigma_max)
    lig0 = poses[0]['ligand']
    mask = torch.from_numpy(lig0.mask_rotate[0].astype(np.uint8)).to(dev)
    rb = poses[0]['ligand', 'ligand'].edge_index.T[lig0.edge_mask]
    bu, bv = rb[:, 0].int().contiguous().to(dev), rb[:, 1].int().contiguous().to(dev)
    coef = []
    for i in range(STEPS):
        c = step_coefficients(i, STEPS, sched, sched, sched, t2s, args, False, **TEMPS)
        if i == STEPS - 1:
            c[1] = c[3] = c[5] = 0.0
        coef.append(c)
    t_rows = [[float(t)] * 3 for t in sched]

    def captured(on, fill=True):
        with _Flag(on, fill):
            g = collate_shared_receptor([d.clone() for d in poses], dev)
            return GraphedSteps(model, g, cli.poses, coef, t_rows, bu, bv, mask, True, dev, draw_noise=True,
                                philox=(1234, torch.arange(cli.poses, device=dev)))
    arms = {'step_off': (False, True), 'step_on': (True, True), 'step_on_nofill': (True, False)}
    times = {k: [] for k in arms}
    finals = {}

    def run(k):
        s = captured(*arms[k])        # one captured step per run and arm (outside the timed region), alive alone
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(STEPS):
            s.graph.replay()
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t0) / STEPS, s.pos.clone()
    for k in arms:                           # warm-up
        run(k)
    for r in range(cli.repeats):
        for k in arms:
            ms, pos = run(k)
            times[k].append(ms)
            finals.setdefault(k, []).append(pos)
            print(f"# {k}: {ms:.2f} ms/step", file=sys.stderr, flush=True)
    step_bits = all(torch.equal(p, finals['step_on'][0]) for p in finals['step_on'] + finals['step_on_nofill'])
    step_delta = float((finals['step_on'][0] - finals['step_off'][0]).abs().max())

    # ---- config 5: one sample_packed call
    sizes = config5_sizes(cli.complexes, seed=0)
    cx = [make_pose_list(cli.poses, n_res=r, n_atoms=a, seed=1000 + i, tr_sigma_max=args.tr_sigma_max, share_receptor=True)
          for i, (r, a) in enumerate(sizes)]
    reset = resetter(cx)

    def packed(on):
        with _Flag(on):
            out = sample_packed(cx, model, STEPS, sched, sched, sched, dev, t2s, args, seed=2024, no_final_step_noise=True,
                                **TEMPS)
        return [torch.stack([d['ligand'].pos for d in dl]) for dl, _ in out]
    ptimes, pouts = {'packed_off': [], 'packed_on': []}, {'packed_off': [], 'packed_on': []}
    for k in ptimes:
        reset()
        packed(k == 'packed_on')
    for _ in range(cli.repeats):
        for k in ptimes:
            reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = packed(k == 'packed_on')
            torch.cuda.synchronize()
            ptimes[k].append(1e3 * (time.perf_counter() - t0))
            pouts[k].append(out)
            print(f"# {k}: {ptimes[k][-1]:.0f} ms", file=sys.stderr, flush=True)
    packed_bits = all(torch.equal(a, b) for o in pouts['packed_on'] for a, b in zip(o, pouts['packed_on'][0]))
    packed_delta = max(float((a - b).abs().max()) for a, b in zip(pouts['packed_on'][0], pouts['packed_off'][0]))
    print(json.dumps({'workload': 'deterministic flag', 'repeats': cli.repeats,
                      'config3_step_ms': {k: stats(v) for k, v in times.items()},
                      'config3_max_abs_dpos_A_after_20_steps': step_delta, 'config3_flag_on_bit_equal': step_bits,
                      'config5_sample_packed_ms': {k: stats(v) for k, v in ptimes.items()},
                      'config5_max_abs_dpos_A': packed_delta, 'config5_flag_on_bit_equal': packed_bits,
                      'complexes': cli.complexes, 'poses': cli.poses, 'card': info}), flush=True)


if __name__ == '__main__':
    main()

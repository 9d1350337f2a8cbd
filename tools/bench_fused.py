#!/usr/bin/env python
"""Micro-benchmark of the fully fused convolution kernel alone (csrc/fused_conv.cu) on receptor-like edges of the full-width
156 -> 156 layer: bf16 wgmma TFLOP/s issued, and - with DDB200_FUSED_DEBUG=1 - the clocks per edge tile.
    python tools/bench_fused.py [--edges 400000] [--layer 3 | --layers]"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

def scan():
    """BASELINE config 4 for the kernel the model runs: receptor sizes 500-5000 x ligand sizes 20-80, 32 poses, full-width
    156->156 layer, receptor contact edges (24 per residue) + cross edges at the mid-schedule cut-off are emulated by E
    CSR-sorted edges over 32 (N_r + N_l) nodes.  Prints one JSON line per shape: ms, issued bf16 TFLOP/s, and the
    SURVEY 8(d) equivalent HBM rate (algorithmic bytes of the un-fused formulation / time) as a fraction of the measured peak."""
    from diffdock_b200 import fused
    from diffdock_b200.tensor_layers import get_irrep_seq
    from diffdock_b200.tp_table import build_table
    peak = 6566.7
    try:
        peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'MEASURED_PEAKS.json')))['hbm_gbs']
    except Exception:
        pass
    ns = 48
    seq = get_irrep_seq(ns, 10, False, False)
    t = build_table(seq[3], '1x0e+1x1o+1x2e', seq[3], 'fctp')
    g = torch.Generator(device='cuda').manual_seed(0)
    H = K1 = 3 * ns
    plan = fused.FusedPlan(t, torch.randn(H, K1, device='cuda', generator=g) / K1 ** 0.5, torch.randn(H, device='cuda', generator=g) * 0.1,
                           torch.randn(t.weight_numel, H, device='cuda', generator=g) / H ** 0.5,
                           torch.randn(t.weight_numel, device='cuda', generator=g) * 0.1)
    for n_r in (500, 1000, 2000, 3000, 5000):
        for n_l in (20, 40, 80):
            N = 32 * (n_r + n_l)
            E = 32 * 24 * n_r + 32 * n_l * min(n_r, 300)        # contacts + ~300 residues within the cut-off per atom
            x = torch.randn(N, t.d_in, device='cuda', generator=g)
            tgt = torch.sort(torch.randint(0, N, (E,), device='cuda', generator=g)).values.int()
            src = torch.randint(0, N, (E,), device='cuda', generator=g).int()
            vec = torch.randn(E, 3, device='cuda', generator=g)
            ea = torch.randn(E, ns, device='cuda', generator=g)
            out, cnt = torch.zeros(N, t.d_out, device='cuda'), torch.zeros(N, device='cuda')
            ts = []
            for i in range(5):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fused.fused_conv(plan, ea, x, ns, tgt, src, x, vec, out, cnt)
                e1.record()
                torch.cuda.synchronize()
                if i >= 2:
                    ts.append(e0.elapsed_time(e1))
            ms = sorted(ts)[len(ts) // 2]
            nbytes = E * (4 * t.weight_numel + 16) + 4 * (N + 1) + 4 * N * t.d_in + 4 * N * t.d_out
            print(json.dumps({'n_res': n_r, 'n_lig': n_l, 'nodes': N, 'E': E, 'ms': round(ms, 3),
                              'bf16_issued_TFLOPs': round(((E + 63) // 64) * plan.mma_flops_per_tile / ms / 1e9, 1),
                              'algorithmic_TFLOPs': round(E * plan.alg_flops_per_edge / ms / 1e9, 1),
                              'equivalent_GBps': round(nbytes / ms / 1e6, 1), 'frac_of_hbm_peak': round(nbytes / ms / 1e6 / peak, 3)}),
                  flush=True)
            del x, tgt, src, vec, ea, out, cnt


def layer(li, E, N, deg):
    """Time the fused kernel on layer li's table (E edges, N nodes, `deg` edges per target); with DDB200_FUSED_DEBUG=1 also
    the clocks per 64 edges against the tensor-pipe ideal, the rate at which the operand images stream from L2, and where
    a warpgroup's time goes: waiting for weight stages to land, and contracting + scattering."""
    from diffdock_b200 import _lib, fused
    from diffdock_b200.tensor_layers import get_irrep_seq
    from diffdock_b200.tp_table import build_table
    ns = 48
    seq = get_irrep_seq(ns, 10, False, False)
    t = build_table(seq[min(li, 3)], '1x0e+1x1o+1x2e', seq[min(li + 1, 3)], 'fctp')
    g = torch.Generator(device='cuda').manual_seed(0)
    H, K1 = 3 * ns, 3 * ns
    w1 = torch.randn(H, K1, device='cuda', generator=g) / K1 ** 0.5
    b1 = torch.randn(H, device='cuda', generator=g) * 0.1
    w2 = torch.randn(t.weight_numel, H, device='cuda', generator=g) / H ** 0.5
    b2 = torch.randn(t.weight_numel, device='cuda', generator=g) * 0.1
    plan = fused.FusedPlan(t, w1, b1, w2, b2)
    x = torch.randn(N, t.d_in, device='cuda', generator=g)
    tgt = (torch.arange(E, device='cuda') // deg).clamp_max(N - 1).int()
    src = torch.randint(0, N, (E,), device='cuda', generator=g).int()
    vec = torch.randn(E, 3, device='cuda', generator=g)
    ea = torch.randn(E, ns, device='cuda', generator=g)
    out = torch.zeros(N, t.d_out, device='cuda')
    cnt = torch.zeros(N, device='cuda')
    run = lambda: fused.fused_conv(plan, ea, x, ns, tgt, src, x, vec, out, cnt)
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    dbg = (C.c_uint64 * 32)()
    have_dbg = _lib.lib().ddb200_fused_debug_read(dbg) == 0
    ts = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = sorted(ts)[2]
    flops = ((E + 63) // 64) * plan.mma_flops_per_tile
    r = {'layer': li, 'E': E, 'tiles': plan.n_tiles, 'ms': round(ms, 3), 'bf16_issued_TFLOPs': round(flops / ms / 1e9, 1)}
    if have_dbg and _lib.lib().ddb200_fused_debug_read(dbg) == 0:
        units = max(int(dbg[12]), 1)                  # 64-edge units: two per 128-edge CTA tile, one per warpgroup
        clk = int(dbg[11]) / units                     # CTA clocks per 64 edges
        s = 3 * ((H + 15) // 16) + 1                  # MMA steps per product (hidden layer and weight tiles alike here)
        r['clk_per_edge_tile'] = int(clk)
        # 4096 bf16 FLOP / clk / SM (H100 data sheet): one 64x192x16 MMA = 96 clocks
        r['ideal_clk_per_edge_tile'] = 96 * s * (plan.n_tiles + 1)
        r['frac_of_ideal'] = round(r['ideal_clk_per_edge_tile'] / clk, 3)
        # operand-image bytes streamed per 128-edge tile (one stream per CTA, read by both warpgroups), as the kernel's TMA
        # ring fetches them: the rows a product reads (W1': the padded hidden width; W2': each tile's MMA width) x 128 B per
        # k-block
        hp, k1p = (H + 15) // 16 * 16, (K1 + 15) // 16 * 16
        n_kb, n_kb1 = (2 * hp + 16 + 63) // 64, (2 * k1p + 16 + 63) // 64
        img_bytes = 128 * (n_kb1 * hp + n_kb * int(plan.tiles[:, 1].sum()))
        r['image_B_per_clk_per_sm'] = round(img_bytes / (2 * clk), 1)
        # a warpgroup spends 2 clk on its 64 edges; the share of it spent waiting for a stage to land and contracting
        wg_clk = 2 * clk
        r['stage_wait_clk_per_64'] = int(dbg[13] / units)
        r['contract_clk_per_64'] = int(dbg[14] / units)
        r['stage_wait_frac'] = round(dbg[13] / units / wg_clk, 3)
        r['contract_frac'] = round(dbg[14] / units / wg_clk, 3)
        r['edge_units_64'] = units // 5
        r['sm_clock_ghz_in_kernel'] = round(dbg[25] / max(dbg[26], 1), 3)     # clock64 ticks per globaltimer ns, CTA 0
    del x, tgt, src, vec, ea, out, cnt
    return r


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--scan', action='store_true', help='BASELINE config 4 size scan of the fused kernel')
    ap.add_argument('--layers', action='store_true', help='sweep the four tables of the benchmarked model (layers 0-3)')
    ap.add_argument('--edges', type=int, default=400000)
    ap.add_argument('--nodes', type=int, default=48000)
    ap.add_argument('--deg', type=int, default=24)
    ap.add_argument('--layer', type=int, default=3)
    a = ap.parse_args()
    if a.scan:
        scan()
        sys.exit(0)
    for li in (range(4) if a.layers else [a.layer]):
        print(json.dumps(layer(li, a.edges, a.nodes, a.deg)), flush=True)

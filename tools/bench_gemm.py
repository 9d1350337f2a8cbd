#!/usr/bin/env python
"""Micro-benchmark of the wgmma split-bf16 radial GEMM alone: fp32-equivalent TFLOP/s (2*E*K*N), bf16 tensor TFLOP/s
actually issued (3x, K padded to 448) and output-write GB/s.   python tools/bench_gemm.py [--edges 200000]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--edges', type=int, default=200000)
    a = ap.parse_args()
    from diffdock_b200.radial import build_b_images, radial_gemm
    for K, N in ((144, 7128), (144, 2784), (96, 312)):
        E = a.edges
        g = torch.Generator(device='cuda').manual_seed(0)
        h = torch.relu(torch.randn(E, K, device='cuda', generator=g))
        W = torch.randn(N, K, device='cuda', generator=g) / K ** 0.5
        b = torch.randn(N, device='cuda', generator=g)
        img, bp, nt = build_b_images(W, b)
        out = torch.empty(E, nt * 256, device='cuda')
        for _ in range(2):
            radial_gemm(h, img, bp, nt, out)
        torch.cuda.synchronize()
        ts = []
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            radial_gemm(h, img, bp, nt, out)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ms = sorted(ts)[2]
        n_kb = (3 * K + 63) // 64
        print(json.dumps({'E': E, 'K': K, 'N': N, 'ms': round(ms, 3), 'fp32_equiv_TFLOPs': round(2 * E * K * N / ms / 1e9, 1),
                          'bf16_issued_TFLOPs': round(2 * E * n_kb * 64 * nt * 256 / ms / 1e9, 1),
                          'write_GBps': round(E * nt * 256 * 4 / ms / 1e6, 1)}), flush=True)
        t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
        t0.record(); ref = torch.nn.functional.linear(h, W, b); t1.record(); torch.cuda.synchronize()
        print('  cublas fp32 ms', round(t0.elapsed_time(t1), 3))

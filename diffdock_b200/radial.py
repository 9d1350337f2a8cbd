"""Host side of the tensor-core radial GEMM (csrc/radial_gemm.cu): operand preparation and the launch wrapper.

The last Linear of the radial MLP (models/layers.py:16; ``[E, 3ns] x [3ns, weight_numel]``, 2 MFLOP per edge) runs as a
split-bf16 wgmma GEMM.  The static operand W2 is split ``W2 = hi + lo`` (bf16 each), concatenated along K as
``[hi | lo | hi]`` to pair with the in-kernel ``[hi | hi | lo]`` split of the activations, zero-padded to 256-row N tiles
and 64-column k-blocks, and stored as the exact 128B-swizzled shared-memory images the MMA consumes, so the kernel
streams them with plain 1-D TMA bulk copies.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from .ops import PROFILE, _need_cuda, _ptr, _stream

import os

BN, BK = 256, 64
MAX_K = 149
USE_TENSOR_CORES = os.environ.get('DDB200_RADIAL_GEMM', 'tc') != 'cublas'


def build_b_images(weight: torch.Tensor, bias: torch.Tensor):
    """weight [N, K] fp32 (rows already in kernel weight-row order), bias [N] ->
    (images bf16 [n_tiles, n_kb, 256, 64] swizzled, bias_padded fp32 [n_tiles*256], n_tiles)."""
    N, K = weight.shape
    n_tiles = (N + BN - 1) // BN
    n_kb = (3 * K + BK - 1) // BK
    dev = weight.device
    w = torch.zeros((n_tiles * BN, K), dtype=torch.float32, device=dev)
    w[:N] = weight.detach().float()
    hi = w.to(torch.bfloat16)
    lo = (w - hi.float()).to(torch.bfloat16)
    bp = torch.zeros((n_tiles * BN, n_kb * BK), dtype=torch.bfloat16, device=dev)
    bp[:, :K], bp[:, K:2 * K], bp[:, 2 * K:3 * K] = hi, lo, hi
    # [tile, row, kb, chunk, 8] -> [tile, kb, row, chunk, 8], then XOR-swizzle the 16-byte chunk index with row % 8
    img = bp.reshape(n_tiles, BN, n_kb, 8, 8).permute(0, 2, 1, 3, 4).contiguous()
    rows = torch.arange(BN, device=dev) % 8
    src_chunk = torch.arange(8, device=dev)[None, :] ^ rows[:, None]          # physical chunk p holds logical chunk p ^ (r%8)
    img = torch.gather(img, 3, src_chunk[None, None, :, :, None].expand(n_tiles, n_kb, BN, 8, 8)).contiguous()
    b = torch.zeros(n_tiles * BN, dtype=torch.float32, device=dev)
    b[:N] = bias.detach().float()
    return img, b, n_tiles


def radial_gemm(h: torch.Tensor, images: torch.Tensor, bias: torch.Tensor, n_tiles: int, out: torch.Tensor = None):
    """out[e, :] = h[e, :] @ W2.T + b  (kernel weight-row layout, row stride n_tiles*256)."""
    _need_cuda(h, images, bias)
    assert h.dtype == torch.float32 and h.stride(1) == 1 and h.shape[1] <= MAX_K
    E, K = h.shape
    ldo = n_tiles * BN
    if out is None:
        out = torch.empty((E, ldo), dtype=torch.float32, device=h.device)
    assert out.shape[0] >= E and out.stride(0) >= ldo and out.stride(1) == 1
    rc = _lib.lib().ddb200_radial_gemm(_ptr(h), h.stride(0), E, K, _ptr(images), _ptr(bias), n_tiles, _ptr(out),
                                       out.stride(0), _stream())
    _lib.check(rc, 'ddb200_radial_gemm')
    PROFILE.all_launches += 1
    return out


def radial_mlp(edge_attr, node, ns, tgt32, src32, w1_images, b1, hidden, w2_images, b2, n_tiles, out=None):
    """Whole two-layer radial MLP in one kernel (ddb200_radial_mlp): gathers the end-point scalars ``node[:, :ns]`` itself
    (``ns == 0``: ``edge_attr`` already holds every input column)."""
    _need_cuda(edge_attr, w1_images, w2_images)
    E, ne = edge_attr.shape
    assert edge_attr.dtype == torch.float32 and edge_attr.stride(1) == 1
    if ns:
        assert node.dtype == torch.float32 and node.stride(1) == 1 and node.shape[1] >= ns
        assert tgt32.dtype == torch.int32 and src32.dtype == torch.int32 and tgt32.is_contiguous() and src32.is_contiguous()
    ldo = n_tiles * BN
    if out is None:
        out = torch.empty((E, ldo), dtype=torch.float32, device=edge_attr.device)
    rc = _lib.lib().ddb200_radial_mlp(_ptr(edge_attr), edge_attr.stride(0), ne, _ptr(node) if ns else C.c_void_p(0),
                                      node.stride(0) if ns else 0, ns, _ptr(tgt32) if ns else C.c_void_p(0),
                                      _ptr(src32) if ns else C.c_void_p(0), _ptr(w1_images), _ptr(b1), hidden,
                                      _ptr(w2_images), _ptr(b2), n_tiles, E, _ptr(out), out.stride(0), _stream())
    _lib.check(rc, 'ddb200_radial_mlp')
    PROFILE.all_launches += 1
    return out

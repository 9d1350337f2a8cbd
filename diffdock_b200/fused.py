"""Host side of the fully fused convolution kernel (csrc/fused_conv.cu): per (layer, edge group) plan.
Replaces, per edge group, the reference's edge_attr_ assembly (models/cg_model.py:342-349), the radial FCBlock
(models/layers.py:10-17 at models/tensor_layers.py:140,211) and the tensor product + scatter (models/tensor_layers.py:139-144,204-221).

The fused kernel computes, for a tile of 64 edges, the radial MLP on the Hopper tensor cores (wgmma) and contracts the resulting
per-edge tensor-product weights with the edge's irreps *straight out of an on-chip accumulator tile* - the ``[E, weight_numel]`` weight
tensor (11-28 KB per edge) never exists in HBM.  To make that possible the weight columns are cut into N tiles that hold
whole rows ``u`` of one path block ``[mul_in, mul_out]``:

    (mul_out, 2l_out+1) = (48, 1): 4 rows x 48 columns = 192        (10, 3): 16 rows x 10 columns = 160
    (16, 1): 8 x 16 = 128                                            (4, 3): 16 x 4 = 64
    (10, 1): 16 x 10 = 160                                           (4, 1): 16 x 4 = 64

    (10, 5): 16 x 10 = 160                                           (4, 5): 16 x 4 = 64

(the two ``(nv, 1)`` kinds are the ``nv x0o`` blocks that ``reduce_pseudoscalars`` gives layers 2 and up; the two
``(nv, 5)`` kinds are the ``nv x2e`` / ``nv x2o`` blocks of ``use_second_order_repr``)

A plan with a 5-component input or output block (``use_second_order_repr``) runs on the kernel's second-order
instantiation (``ddb200_fused_conv_so``): up to 32 paths, dense [5][5][5] tables, and each (10, 5) tile scattered at its
own end in two slices (components 0-2, 3-4), because 100 partial sums per thread would not fit beside the accumulators.

A radial MLP built with ``tp_weights_layers`` > 2 passes its extra H x H hidden layers as ``FusedPlan(..., hidden=...)``:
one operand image each, streamed between W1' and the W2' tiles and applied in place over the activation image.

so that a consumer thread (one edge = one accumulator row) knows at compile time which register of its accumulator every
accumulator column feeds.  This module builds, from a ``TpTable`` and the radial MLP's second Linear:
  * the tile table (int32 [T, 8]) and one dense Clebsch-Gordan table per path ([3][3][5] floats: coef * C[i, j, k];
    second order: [5][5][5]),
  * the pre-split, pre-swizzled bf16 operand images of W2 per tile (rows permuted into tile order, zero padded), with the
    bias folded in as two extra K columns (hi, lo) that multiply constant-one columns of the activation operand.
    Image columns are [hi | lo | bias] in 16-column-aligned sections; the kernel's activation image is [hi | lo | 1 1] and
    its MMA schedule forms hi.hi + hi.lo + lo.hi + bias from them (a staged hi block of W2 is used by two MMAs).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from .ops import PROFILE, _need_cuda, _ptr, _stream, fixed_error_word

from .irreps import real_cg
from .radial import BK, BN
from .tp_table import TpTable

# (mul_out, d_out) -> (consumer kind id, rows per tile)
CONSUMER_KINDS = {(48, 1): (0, 4), (10, 3): (1, 16), (16, 1): (2, 8), (4, 3): (3, 16), (10, 1): (4, 16), (4, 1): (5, 16),
                  (10, 5): (6, 16), (4, 5): (7, 16)}
MAX_K = 144          # widest radial-MLP input / hidden layer (16-column sections: 2 * 144 + 16 = 304 -> 5 k-blocks of 64)
MAX_TILES = 128      # tile table capacity of the kernel (csrc/fused_conv.cu)
MTAB = 48            # floats per path in the dense Clebsch-Gordan table: [3][3][5] padded
MAX_PATHS = 16
MTAB_SO = 128        # second-order instantiation: [5][5][5] padded
MAX_PATHS_SO = 32
ENABLED = os.environ.get('DDB200_FUSED_CONV', '1') != '0'


def _pad16(k: int) -> int:
    return (k + 15) // 16 * 16


def second_order(table: TpTable) -> bool:
    """True when the layer has a 5-component input or output block: it runs on the second-order instantiation."""
    return any(p.l_in == 2 or p.l_out == 2 for p in table.paths)


def supported(table: TpTable, hidden: int, k1: int) -> bool:
    if table.sh_lmax < 0 or table.sh_lmax > 2:
        return False
    if _pad16(hidden) > MAX_K or _pad16(k1) > MAX_K:
        return False
    if len(table.paths) > (MAX_PATHS_SO if second_order(table) else MAX_PATHS):
        return False
    for p in table.paths:
        if (p.mul_out, 2 * p.l_out + 1) not in CONSUMER_KINDS:
            return False
        if (2 * p.l_in + 1) not in (1, 3, 5) or p.l_sh > 2:
            return False
    n_tiles = sum(-(-p.mul_in // CONSUMER_KINDS[(p.mul_out, 2 * p.l_out + 1)][1]) for p in table.paths)
    return n_tiles <= MAX_TILES


def _split_images(w_rows: torch.Tensor, bias_rows: torch.Tensor, K: int):
    """w_rows [T, 256, K] fp32 (zero rows where padded), bias_rows [T, 256] -> bf16 images [T, n_kb, 256, 8, 8]:
    columns [hi | lo | bias_hi, bias_lo, 0...] with both sections padded to Kp = 16 * ceil(K / 16) columns (one MMA step =
    16 columns; the kernel multiplies a hi step with the hi and the lo columns of the activation image [hi | lo | 1 1 0...],
    a lo step with the hi columns, the bias step with the ones), 128B-swizzled."""
    T = w_rows.shape[0]
    Kp = _pad16(K)
    n_kb = (2 * Kp + 16 + BK - 1) // BK
    dev = w_rows.device
    hi = w_rows.to(torch.bfloat16)
    lo = (w_rows - hi.float()).to(torch.bfloat16)
    bhi = bias_rows.to(torch.bfloat16)
    blo = (bias_rows - bhi.float()).to(torch.bfloat16)
    bp = torch.zeros((T, BN, n_kb * BK), dtype=torch.bfloat16, device=dev)
    bp[:, :, :K], bp[:, :, Kp:Kp + K] = hi, lo
    bp[:, :, 2 * Kp], bp[:, :, 2 * Kp + 1] = bhi, blo          # x constant-one activation columns
    img = bp.reshape(T, BN, n_kb, 8, 8).permute(0, 2, 1, 3, 4).contiguous()
    rows = torch.arange(BN, device=dev) % 8
    src_chunk = torch.arange(8, device=dev)[None, :] ^ rows[:, None]
    return torch.gather(img, 3, src_chunk[None, None, :, :, None].expand(T, n_kb, BN, 8, 8)).contiguous()


class FusedPlan:
    """Device-resident plan of one (layer, edge group)."""

    def __init__(self, table: TpTable, w1: torch.Tensor, b1: torch.Tensor, w2_ref: torch.Tensor, b2_ref: torch.Tensor,
                 hidden=()):
        """w1 [H, K1], b1 [H]; w2_ref [weight_numel, H], b2_ref [weight_numel] in the REFERENCE weight-row order;
        ``hidden``: the FCBlock's extra hidden layers (``tp_weights_layers - 2`` of them) in order, each ``(W [H, H], b [H])``,
        applied as ReLU(h W^T + b) after the first layer."""
        dev = w2_ref.device
        H, K1 = w1.shape
        assert supported(table, H, K1)
        assert all(tuple(w.shape) == (H, H) and tuple(b.shape) == (H,) for w, b in hidden)
        self.table, self.hidden, self.k1 = table, H, K1
        self.n_hidden = len(hidden)
        self.second_order = second_order(table)
        paths = sorted(table.paths, key=lambda p: (p.i_out, p.w_ref_off))
        tiles, row_src = [], []
        # dense Clebsch-Gordan table per path: mtab[path][i][k][j] = coef * C[i, j, k]   (i, k < D, j < 5; zero padded),
        # D = 3 (first order) or 5 (second order)
        D = 5 if self.second_order else 3
        mtab = np.zeros((len(paths), MTAB_SO if self.second_order else MTAB), dtype=np.float32)
        for pi, p in enumerate(paths):
            C = real_cg(p.l_in, p.l_sh, p.l_out)
            d_in, d_sh, d_out = C.shape
            blk = np.zeros((D, D, 5))
            blk[:d_in, :d_out, :d_sh] = p.coef * np.transpose(C, (0, 2, 1))
            mtab[pi, :D * D * 5] = blk.reshape(-1)
        group_prev = None
        path_prev = None
        for pi, p in enumerate(paths):
            d_in, d_out = 2 * p.l_in + 1, 2 * p.l_out + 1
            kind, rows_per = CONSUMER_KINDS[(p.mul_out, d_out)]
            for u0 in range(0, p.mul_in, rows_per):
                nrow = min(rows_per, p.mul_in - u0)
                # tile width: the valid columns rounded up to whole 32-column chunks (columns beyond are never read)
                n_mma = min(rows_per * p.mul_out, (nrow * p.mul_out + 31) // 32 * 32)
                first = group_prev != p.i_out
                group_prev = p.i_out
                new_path = path_prev is not p        # flag 4: the consumer rebuilds its C.Y matrix
                path_prev = p
                flags = (1 if first else 0) | (4 if new_path else 0) | (p.sh_off << 8)
                tiles.append([kind, n_mma, p.in_off + u0 * d_in, nrow, d_in, p.out_off, flags, pi])
                src = np.full(BN, -1, dtype=np.int64)
                cols = p.w_ref_off + (u0 * p.mul_out) + np.arange(nrow * p.mul_out)
                src[:nrow * p.mul_out] = cols
                row_src.append(src)
        for i in range(len(tiles)):          # last tile of an accumulator run
            if i == len(tiles) - 1 or tiles[i + 1][6] & 1:
                tiles[i][6] |= 2
        self.n_tiles = len(tiles)
        self.n_paths = len(paths)
        src = torch.as_tensor(np.stack(row_src), device=dev)                      # [T, 256] -> reference weight row or -1
        ok = src >= 0
        w_rows = torch.zeros((self.n_tiles, BN, H), dtype=torch.float32, device=dev)
        b_rows = torch.zeros((self.n_tiles, BN), dtype=torch.float32, device=dev)
        w_rows[ok] = w2_ref.detach().float()[src[ok]]
        b_rows[ok] = b2_ref.detach().float()[src[ok]]
        self.w2_images = _split_images(w_rows, b_rows, H)
        w1p = torch.zeros((1, BN, K1), dtype=torch.float32, device=dev)
        b1p = torch.zeros((1, BN), dtype=torch.float32, device=dev)
        w1p[0, :H], b1p[0, :H] = w1.detach().float(), b1.detach().float()
        self.w1_images = _split_images(w1p, b1p, K1)
        # one N tile per extra hidden layer, streamed between W1' and the W2' tiles: [n_hidden, n_kb, 256, 8, 8]
        self.wh_images = None
        if hidden:
            whp = torch.zeros((self.n_hidden, BN, H), dtype=torch.float32, device=dev)
            bhp = torch.zeros((self.n_hidden, BN), dtype=torch.float32, device=dev)
            for l, (w, b) in enumerate(hidden):
                whp[l, :H], bhp[l, :H] = w.detach().float(), b.detach().float()
            self.wh_images = _split_images(whp, bhp, H)
        self.tiles = torch.as_tensor(np.asarray(tiles, dtype=np.int32), device=dev).contiguous()
        self.mtab = torch.as_tensor(mtab, device=dev).contiguous()
        # 8-byte gathers of the node values are possible when every tile's offset and value count is even
        self.x_pairs_ok = int(all(t[2] % 2 == 0 and (t[3] * t[4]) % 2 == 0 for t in tiles))
        # bf16 tensor-core FLOPs issued per 64-edge tile (split-bf16 x3 + bias step, 16-column steps; the kernel issues every
        # product 192 columns wide)
        s2, s1 = 3 * (_pad16(H) // 16) + 1, 3 * (_pad16(K1) // 16) + 1
        self.mma_flops_per_tile = 2 * 64 * 16 * 192 * (s1 + (self.n_hidden + len(tiles)) * s2)
        # algorithmic FLOPs per edge of the same work (fp32 radial MLP + tensor-product contraction, SURVEY 8(d))
        self.alg_flops_per_edge = 2 * K1 * H + self.n_hidden * 2 * H * H + 2 * H * table.weight_numel + sum(
            2 * p.mul_in * p.mul_out * (2 * p.l_out + 1) + 2 * p.mul_in * (2 * p.l_in + 1) * (2 * p.l_sh + 1) * (2 * p.l_out + 1)
            for p in table.paths)


class _Args(C.Structure):
    """Mirror of ``ddb200_fused_args`` (include/diffdock_b200.h)."""
    _fields_ = [('edge_attr', C.c_void_p), ('ld_ea', C.c_int64), ('ne', C.c_int32),
                ('node', C.c_void_p), ('ld_node', C.c_int64), ('ns', C.c_int32),
                ('tgt', C.c_void_p), ('src', C.c_void_p), ('edge_perm', C.c_void_p),
                ('ea_add', C.c_void_p), ('ea_add_idx', C.c_void_p), ('vec_sign', C.c_float),
                ('w1_images', C.c_void_p), ('hidden', C.c_int32), ('w2_images', C.c_void_p),
                ('tiles', C.c_void_p), ('n_tiles', C.c_int32), ('mtab', C.c_void_p), ('n_paths', C.c_int32),
                ('x', C.c_void_p), ('ld_x', C.c_int64), ('x_pairs_ok', C.c_int32),
                ('edge_vec', C.c_void_p), ('edge_weight', C.c_void_p), ('sh_lmax', C.c_int32),
                ('n_edges', C.c_int64), ('n_edges_dev', C.c_void_p),
                ('sum', C.c_void_p), ('d_out', C.c_int32), ('cnt', C.c_void_p),
                ('wh_images', C.c_void_p), ('n_hidden', C.c_int32)]


def _p(t):
    return t.data_ptr() if t is not None else None


def fused_conv(plan: FusedPlan, edge_attr, node, ns, tgt32, src32, x, edge_vec, sum_buf, cnt_buf, edge_weight=None,
               edge_perm=None, vec_sign=1.0, ea_add=None, ea_add_idx=None, n_edges_dev=None, n_edges=None):
    """sum_buf[tgt] += TP(x[src], Y(vec), radial_mlp(...)) for one CSR-sorted edge group, in ONE kernel.

    ``edge_perm`` [E] int32: row of ``edge_attr`` / ``edge_vec`` / ``edge_weight`` for edge e (default e);
    ``vec_sign``: the edge vector is multiplied by it; ``ea_add`` [G, ne] + ``ea_add_idx`` [E] int32: per-edge row added to
    the attribute row; ``n_edges_dev``: int32 device scalar holding the live edge count (``tgt32.shape[0]`` is the capacity)."""
    _need_cuda(edge_attr, x, edge_vec, sum_buf)
    ne = edge_attr.shape[1]
    E = int(tgt32.shape[0]) if n_edges is None else int(n_edges)
    if E == 0:
        return
    t = plan.table
    assert edge_attr.dtype == torch.float32 and edge_attr.stride(1) == 1 and x.stride(1) == 1 and edge_vec.is_contiguous()
    assert edge_vec.dtype == torch.float32 and x.dtype == torch.float32 and sum_buf.dtype in (torch.float32, torch.int64)
    assert tgt32.dtype == torch.int32 and src32.dtype == torch.int32 and tgt32.is_contiguous() and src32.is_contiguous()
    assert ne + 2 * ns == plan.k1 and x.shape[1] == t.d_in and sum_buf.shape[1] == t.d_out and sum_buf.is_contiguous()
    if edge_perm is None:
        assert edge_attr.shape[0] >= E and edge_vec.shape[0] >= E
    else:
        assert edge_perm.dtype == torch.int32 and edge_perm.is_contiguous() and edge_perm.shape[0] >= E
    if edge_weight is not None:
        edge_weight = edge_weight.reshape(-1)
        assert edge_weight.dtype == torch.float32 and edge_weight.is_contiguous()
    if ea_add is not None:
        assert ea_add.dtype == torch.float32 and ea_add.is_contiguous() and ea_add.shape[1] == ne
        assert ea_add_idx.dtype == torch.int32 and ea_add_idx.is_contiguous() and ea_add_idx.shape[0] >= E
    if n_edges_dev is not None:
        assert n_edges_dev.dtype == torch.int32 and n_edges_dev.is_cuda
    fixed = sum_buf.dtype == torch.int64     # fixed-point accumulators (ops.new_accumulators under the deterministic flag)
    a = _Args(_p(edge_attr), edge_attr.stride(0), ne, _p(node) if ns else None, node.stride(0) if ns else 0, ns,
              _p(tgt32), _p(src32), _p(edge_perm), _p(ea_add), _p(ea_add_idx) if ea_add is not None else None,
              float(vec_sign), _p(plan.w1_images), plan.hidden, _p(plan.w2_images), _p(plan.tiles), plan.n_tiles,
              _p(plan.mtab), plan.n_paths, _p(x), x.stride(0), plan.x_pairs_ok, _p(edge_vec), _p(edge_weight),
              t.sh_lmax, E, _p(n_edges_dev), None if fixed else _p(sum_buf), t.d_out, _p(cnt_buf), _p(plan.wh_images),
              plan.n_hidden)
    prof = PROFILE.enabled
    if prof:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    L = _lib.lib()
    if fixed:
        launch = L.ddb200_fused_conv_so_fixed if plan.second_order else L.ddb200_fused_conv_fixed
        rc = launch(C.byref(a), _p(sum_buf), _p(fixed_error_word(sum_buf.device)), _stream())
    else:
        launch = L.ddb200_fused_conv_so if plan.second_order else L.ddb200_fused_conv
        rc = launch(C.byref(a), _stream())
    if prof:
        e1.record()
        n_live = int(n_edges_dev.item()) if n_edges_dev is not None else E      # profiling replay only (host sync)
        PROFILE.fused_pairs.append((e0, e1))
        PROFILE.fused_bytes += n_live * (4 * t.weight_numel + 12 + 4) + 4 * (sum_buf.shape[0] + 1) + \
            4 * x.shape[0] * t.d_in + 4 * sum_buf.shape[0] * t.d_out
        PROFILE.fused_flops += ((n_live + 63) // 64) * plan.mma_flops_per_tile
        PROFILE.fused_alg_flops += n_live * plan.alg_flops_per_edge
    PROFILE.all_launches += 1
    _lib.check(rc, 'ddb200_fused_conv_fixed' if fixed else 'ddb200_fused_conv')

"""Instruction-table generator for the fused tensor-product convolution kernel (csrc/tpconv.cu).

From ``(in_irreps, sh_irreps, out_irreps, kind)`` it produces, once per layer:

* the path list in the weight order of the reference's tensor product -
  ``kind='fctp'``  : e3nn ``FullyConnectedTensorProduct`` (instructions lexicographic in (in1, sh, out), mode 'uvw',
                     one ``[mul_in, 1, mul_out]`` block each, ``coef = sqrt((2 l_out + 1) / fan_in(out slot))``;
                     reference: models/tensor_layers.py:299, models/cg_model.py:220-228,241-249),
  ``kind='faster'``: the reference's in-tree ``FasterTensorProduct`` weight layout - four ``[fan_in, mul_out]`` blocks
                     0e | 1o | 1e | 0o, fan-in rows in the append order of models/tensor_layers.py:77-90, scale
                     1/sqrt(fan_in) (:92-98); the arithmetic is the same Clebsch-Gordan contraction;
* the flat int32/float32 blobs the CUDA kernel consumes (layout documented in include/diffdock_b200.h), including the
  TMA chunking of one per-edge weight row and the lane mapping of every weight tile;
* ``evaluate()`` - a numpy interpreter of exactly those blobs, used by the CPU tests to validate the tables
  against the oracle without a GPU.

A "path" computes, for one edge:  out[w, k] += sum_u W[u, w] * z[u, k],   z[u, k] = sum_i x[u, i] * M[i, k],
M[i, k] = coef * edge_weight * sum_j C[i, j, k] * Y[j].
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass, field
from typing import List

import numpy as np

from .irreps import irreps_dim, irreps_offsets, parse_irreps, real_cg

MAGIC = 0x44423232  # 'DB22'
HDR_INTS = 32
WARP = 32


@dataclass
class Path:
    i_in: int
    i_sh: int
    i_out: int
    mul_in: int
    mul_out: int
    l_in: int
    l_sh: int
    l_out: int
    in_off: int
    sh_off: int
    out_off: int
    w_off: int          # offset of the [mul_in, mul_out] block inside one (padded) weight row, floats
    w_ref_off: int      # offset of the same block in the reference's own (unpadded) layout
    coef: float


@dataclass
class TpTable:
    in_irreps: list
    sh_irreps: list
    out_irreps: list
    kind: str
    paths: List[Path]
    weight_numel: int            # reference layout (what the radial MLP's last Linear outputs)
    weight_numel_padded: int     # kernel layout (every block 16-byte aligned); == weight_numel for the usual configs
    w_perm: np.ndarray           # [weight_numel_padded] -> index into the reference row, or -1 for padding
    sh_lmax: int                 # >= 0: SH evaluated in-kernel from the edge vector; -1: SH given per edge
    iblob: np.ndarray = field(default=None, repr=False)
    fblob: np.ndarray = field(default=None, repr=False)
    fblob64: np.ndarray = field(default=None, repr=False)   # the same terms in float64 (fblob is their float32 rounding)
    stage_floats: int = 0
    n_chunks: int = 0

    @property
    def d_in(self):
        return irreps_dim(self.in_irreps)

    @property
    def d_sh(self):
        return irreps_dim(self.sh_irreps)

    @property
    def d_out(self):
        return irreps_dim(self.out_irreps)

    @property
    def identity_layout(self):
        return self.weight_numel == self.weight_numel_padded and bool(
            np.all(self.w_perm == np.arange(self.weight_numel)))


def _align4(n):
    return (n + 3) // 4 * 4


def _fctp_paths(ins, shs, outs):
    in_off, sh_off, out_off = irreps_offsets(ins), irreps_offsets(shs), irreps_offsets(outs)
    trip = []
    for a, (m1, l1, p1) in enumerate(ins):
        for b, (m2, l2, p2) in enumerate(shs):
            assert m2 == 1, "edge spherical harmonics carry multiplicity 1"
            for c, (m3, l3, p3) in enumerate(outs):
                if p1 * p2 == p3 and abs(l1 - l2) <= l3 <= l1 + l2:
                    trip.append((a, b, c))
    fan = {}
    for a, b, c in trip:
        fan[c] = fan.get(c, 0) + ins[a][0] * shs[b][0]
    paths, off = [], 0
    for a, b, c in trip:
        (m1, l1, _), (_, l2, _), (m3, l3, _) = ins[a], shs[b], outs[c]
        paths.append(Path(a, b, c, m1, m3, l1, l2, l3, in_off[a], sh_off[b], out_off[c], -1, off,
                          math.sqrt((2 * l3 + 1) / fan[c])))
        off += m1 * m3
    return paths, off


def _faster_paths(ins, shs, outs):
    assert shs == [(1, 0, 1), (1, 1, -1)], "FasterTensorProduct needs sh = 1x0e+1x1o"
    name = {(0, 1): '0e', (1, -1): '1o', (1, 1): '1e', (0, -1): '0o'}
    for m, l, p in ins + outs:
        assert (l, p) in name, "FasterTensorProduct handles 0e/1o/1e/0o only"
    idx_in = {name[(l, p)]: i for i, (m, l, p) in enumerate(ins)}
    idx_out = {name[(l, p)]: i for i, (m, l, p) in enumerate(outs)}
    in_off, out_off = irreps_offsets(ins), irreps_offsets(outs)
    # (out key) -> ordered list of (in key, sh index) : models/tensor_layers.py:77-90
    rows = {'0e': [('0e', 0), ('1o', 1)],
            '1o': [('0e', 1), ('1o', 0), ('1e', 1)],
            '1e': [('1o', 1), ('1e', 0), ('0o', 1)],
            '0o': [('1e', 1), ('0o', 0)]}
    paths, off = [], 0
    for ok in ('0e', '1o', '1e', '0o'):      # block order of weight_shapes, :63-68
        fan = sum(ins[idx_in[ik]][0] for ik, _ in rows[ok] if ik in idx_in)
        mo = outs[idx_out[ok]][0] if ok in idx_out else 0
        if mo == 0 or fan == 0:
            off += fan * mo
            continue
        c = idx_out[ok]
        l3 = outs[c][1]
        u0 = 0
        for ik, b in rows[ok]:
            if ik not in idx_in:
                continue
            a = idx_in[ik]
            m1, l1, _ = ins[a]
            paths.append(Path(a, b, c, m1, mo, l1, b, l3, in_off[a], b if b == 0 else 1, out_off[c], -1,
                              off + u0 * mo, math.sqrt((2 * l3 + 1) / fan)))
            u0 += m1
        off += fan * mo
    return paths, off


def build_table(in_irreps, sh_irreps, out_irreps, kind='fctp', sh_from_vector=True, stage_floats=None) -> TpTable:
    if stage_floats is None:   # TMA chunk size: 3 KB (16 warps x 2 stages)
        stage_floats = int(os.environ.get('DDB200_TPCONV_STAGE_FLOATS', 768))
    ins, shs, outs = parse_irreps(in_irreps), parse_irreps(sh_irreps), parse_irreps(out_irreps)
    if kind == 'fctp':
        paths, numel = _fctp_paths(ins, shs, outs)
    elif kind == 'faster':
        paths, numel = _faster_paths(ins, shs, outs)
    else:
        raise ValueError(kind)
    # kernel layout: blocks grouped by OUTPUT irrep (consecutive tiles then share register accumulators), reference
    # order inside a group, each block start rounded up to 4 floats (16 B, TMA bulk-copy alignment)
    order = sorted(range(len(paths)), key=lambda i: (paths[i].i_out, paths[i].w_ref_off))
    off = 0
    for i in order:
        off = _align4(off)
        paths[i].w_off = off
        off += paths[i].mul_in * paths[i].mul_out
    padded = _align4(off)
    w_perm = np.full(padded, -1, dtype=np.int64)
    for p in paths:
        n = p.mul_in * p.mul_out
        w_perm[p.w_off:p.w_off + n] = np.arange(p.w_ref_off, p.w_ref_off + n)
    lmax = -1
    if sh_from_vector:
        assert shs == [(1, l, (-1) ** l) for l in range(len(shs))] and len(shs) <= 3, \
            "in-kernel spherical harmonics need sh = Irreps.spherical_harmonics(lmax<=2)"
        lmax = len(shs) - 1
    t = TpTable(ins, shs, outs, kind, paths, numel, padded, w_perm, lmax)
    _compile(t, stage_floats)
    return t


# tile kinds of the contraction loop (csrc/tpconv.cu): (vector width of the weight loads, 2 l_out + 1)
_TILE_KIND = {(4, 1): 1, (4, 3): 2, (2, 1): 3, (2, 3): 4}
# z kinds: (2 l_in + 1, 2 l_out + 1) with a specialised z[u,k] = sum_i x[u,i] M[i,k] loop
_Z_KIND = {(1, 1): 1, (1, 3): 2, (3, 1): 3, (3, 3): 4}


def _compile(t: TpTable, stage_floats: int):
    paths = t.paths
    order = sorted(range(len(paths)), key=lambda i: paths[i].w_off)      # kernel (= weight-row) order
    # z / M scratch: z rows are padded to 4 floats when d_out == 3 (one LDS.128 per row)
    z_off, m_off, z_str = {}, {}, {}
    zo = mo = 0
    for pi in order:
        p = paths[pi]
        d_out = 2 * p.l_out + 1
        z_str[pi] = 1 if d_out == 1 else (4 if d_out == 3 else d_out)
        z_off[pi], m_off[pi] = zo, mo
        zo = _align4(zo + p.mul_in * z_str[pi])
        mo += (2 * p.l_in + 1) * d_out
    # per output irrep: vector width, lanes per row, column tiles, accumulator rows
    out_cfg, n_acc, lpr_list = {}, 0, []
    for c, (m3, l3, _) in enumerate(t.out_irreps):
        d = 2 * l3 + 1
        vec = 4 if m3 % 4 == 0 else (2 if m3 % 2 == 0 else 1)
        if (vec, d) not in _TILE_KIND:
            vec = 1
        cols_per_tile = min(m3, WARP * vec)
        tiles_c = []
        for c0 in range(0, m3, cols_per_tile):
            ncol = min(cols_per_tile, m3 - c0)
            lpr = ncol // vec
            if lpr not in lpr_list:
                lpr_list.append(lpr)
            tiles_c.append((c0, ncol, lpr, n_acc))
            n_acc += vec * d
        out_cfg[c] = (vec, d, tiles_c)
    assert len(lpr_list) <= 4, "more than 4 distinct lane-per-row values"
    # M entries and their CG terms
    ment, terms_y, terms_v = [], [], []
    for pi in order:
        p = paths[pi]
        C = real_cg(p.l_in, p.l_sh, p.l_out)
        for i in range(2 * p.l_in + 1):
            for k in range(2 * p.l_out + 1):
                js = [j for j in range(2 * p.l_sh + 1) if C[i, j, k] != 0.0]
                if not js:
                    continue
                ment.append((m_off[pi] + i * (2 * p.l_out + 1) + k, len(terms_y), len(js)))
                for j in js:
                    terms_y.append(p.sh_off + j)
                    terms_v.append(p.coef * C[i, j, k])
    # weight tiles (row pieces of path blocks) grouped into TMA chunks of <= stage_floats contiguous floats
    stage_floats = max(_align4(stage_floats), _align4(2 * max((p.mul_out for p in paths), default=4)))
    tiles, chunks, groups = [], [], []
    cur = None   # [tile_begin, g_off, n_floats]
    for pi in order:
        p = paths[pi]
        vec, d_out, tiles_c = out_cfg[p.i_out]
        m = p.mul_out
        rows_per_piece = max(1, stage_floats // m)
        u = 0
        while u < p.mul_in:
            nrow = min(rows_per_piece, p.mul_in - u)
            if u + nrow < p.mul_in:           # interior cut: keep the next piece 16-byte aligned
                while nrow > 1 and (nrow * m) % 4:
                    nrow -= 1
                assert (nrow * m) % 4 == 0, "cannot split weight block on a 16-byte boundary"
            g0 = p.w_off + u * m
            end_aligned = _align4(g0 + nrow * m)
            if cur is None or cur[1] + cur[2] != g0 or (end_aligned - cur[1]) > stage_floats:
                if cur is not None:
                    chunks.append((cur[0], len(tiles), cur[1], cur[2]))
                cur = [len(tiles), g0, 0]
            wloc0 = g0 - cur[1]
            for (c0, ncol, lpr, acc_row) in tiles_c:
                kind = _TILE_KIND.get((vec, d_out), 0)
                R = WARP // lpr
                # record = 4 x int4: A (per-tile) | B, C (per accumulator run) | D
                tiles.append([wloc0 + c0, z_off[pi] + u * z_str[pi], (nrow // R) | ((nrow % R) << 16), 0,
                              m, d_out, vec, lpr_list.index(lpr),
                              R, acc_row * WARP, z_str[pi], kind,
                              nrow, 0, 0, 0])
                groups.append((p.i_out, c0) if len(tiles_c) == 1 else ('solo', len(tiles)))
            cur[2] = end_aligned - cur[1]
            u += nrow
    if cur is not None:
        chunks.append((cur[0], len(tiles), cur[1], cur[2]))
    chunk_first = {c[0] for c in chunks}
    chunk_last = {c[1] - 1 for c in chunks}
    for i, tl in enumerate(tiles):     # first / last tile of a run that accumulates into the same registers
        first = i == 0 or groups[i - 1] != groups[i]
        last = i == len(tiles) - 1 or groups[i + 1] != groups[i]
        tl[3] = (1 if first else 0) | (2 if last else 0) | (4 if i in chunk_first else 0) | (8 if i in chunk_last else 0)
    for (_, _, g, n) in chunks:
        assert g % 4 == 0 and n % 4 == 0 and n <= stage_floats and g + n <= t.weight_numel_padded
    # output map: out column -> (first accumulator slot, lane stride between row groups, #row groups)
    outmap = []
    for c, (m3, l3, _) in enumerate(t.out_irreps):
        vec, d, tiles_c = out_cfg[c]
        for w in range(m3):
            c0, ncol, lpr, acc_row = next(tc for tc in tiles_c if tc[0] <= w < tc[0] + tc[1])
            cl, v = divmod(w - c0, vec)
            for k in range(d):
                outmap.append(((acc_row + v * d + k) * WARP + cl, lpr, WARP // lpr))
    assert len(outmap) == t.d_out

    def sect(rows, ncol):
        a = np.asarray(rows, dtype=np.int32).reshape(-1, ncol) if len(rows) else np.zeros((0, ncol), np.int32)
        return a.reshape(-1)

    s_paths = sect([(paths[pi].in_off, paths[pi].mul_in, 2 * paths[pi].l_in + 1, 2 * paths[pi].l_out + 1, z_off[pi],
                     m_off[pi], z_str[pi], _Z_KIND.get((2 * paths[pi].l_in + 1, 2 * paths[pi].l_out + 1), 0))
                    for pi in order], 8)
    s_tiles, s_chunks, s_ment = sect(tiles, 16), sect(chunks, 4), sect(ment, 3)
    s_ty, s_out = np.asarray(terms_y, dtype=np.int32), sect(outmap, 3)
    hdr = np.zeros(HDR_INTS, dtype=np.int32)
    offs, o = [], HDR_INTS
    for s in (s_paths, s_tiles, s_chunks, s_ment, s_ty, s_out):
        offs.append(o)
        o += len(s)
    hdr[:15] = [MAGIC, len(paths), len(tiles), len(chunks), len(ment), len(terms_y), t.d_in, t.d_sh, t.d_out,
                t.sh_lmax, max(zo, 4), max(mo, 1), n_acc, t.weight_numel_padded, stage_floats]
    hdr[15:21] = offs
    hdr[21] = o
    hdr[22:22 + len(lpr_list)] = lpr_list
    t.iblob = np.concatenate([hdr, s_paths, s_tiles, s_chunks, s_ment, s_ty, s_out]).astype(np.int32)
    t.fblob64 = np.asarray(terms_v if terms_v else [0.0], dtype=np.float64)
    t.fblob = t.fblob64.astype(np.float32)
    t.stage_floats, t.n_chunks = stage_floats, len(chunks)


# ------------------------------------------------------------------------------------------------
def spherical_harmonics_np(vec, lmax):
    """Component-normalised real SH (l<=2) of the normalised vector - the formula the kernel evaluates."""
    vec = np.asarray(vec, dtype=np.float64)
    n = np.maximum(np.linalg.norm(vec, axis=-1, keepdims=True), 1e-12)
    x, y, z = (vec / n)[..., 0], (vec / n)[..., 1], (vec / n)[..., 2]
    out = [np.ones_like(x)]
    if lmax >= 1:
        s3 = math.sqrt(3.0)
        out += [s3 * x, s3 * y, s3 * z]
    if lmax >= 2:
        s5, s15 = math.sqrt(5.0), math.sqrt(15.0)
        out += [s15 * x * z, s15 * x * y, s5 * (y * y - 0.5 * (x * x + z * z)), s15 * y * z,
                0.5 * s15 * (z * z - x * x)]
    return np.stack(out, -1)


def evaluate(t: TpTable, x, sh_or_vec, w_padded, edge_weight=None):
    """Numpy interpreter of the compiled blobs, lane by lane like the kernel: per-edge tensor-product messages
    [E, D_out] (float64).  ``w_padded`` is in the kernel layout ([E, weight_numel_padded]).  The Clebsch-Gordan terms are
    read in float64 (``fblob64``), so the result is the table's arithmetic without the float32 rounding of the terms."""
    ib, fb = t.iblob, np.asarray(t.fblob64 if t.fblob64 is not None else t.fblob, dtype=np.float64)
    (_, n_paths, n_tiles, n_chunks, n_ment, n_terms, d_in, d_sh, d_out, lmax, z_tot, m_tot, n_acc, wpad,
     _cap) = ib[:15]
    o_paths, o_tiles, o_chunks, o_ment, o_ty, o_out = ib[15:21]
    lprs = ib[22:26]
    paths = ib[o_paths:o_paths + 8 * n_paths].reshape(-1, 8)
    tiles = ib[o_tiles:o_tiles + 16 * n_tiles].reshape(-1, 16)
    chunks = ib[o_chunks:o_chunks + 4 * n_chunks].reshape(-1, 4)
    ment = ib[o_ment:o_ment + 3 * n_ment].reshape(-1, 3)
    ty = ib[o_ty:o_ty + n_terms]
    outmap = ib[o_out:o_out + 3 * d_out].reshape(-1, 3)
    x = np.asarray(x, np.float64)
    w = np.asarray(w_padded, np.float64)
    E = x.shape[0]
    Y = spherical_harmonics_np(sh_or_vec, lmax) if lmax >= 0 else np.asarray(sh_or_vec, np.float64)
    ew = np.ones(E) if edge_weight is None else np.asarray(edge_weight, np.float64).reshape(E)
    out = np.zeros((E, d_out))
    for e in range(E):
        M = np.zeros(m_tot)
        for (mi, tb, tc) in ment:
            M[mi] = ew[e] * sum(fb[q] * Y[e, ty[q]] for q in range(tb, tb + tc))
        z = np.zeros(z_tot)
        for (in_off, mul_in, din, dout, zo, mo, zs, _zk) in paths:
            xb = x[e, in_off:in_off + mul_in * din].reshape(mul_in, din)
            zz = xb @ M[mo:mo + din * dout].reshape(din, dout)
            for u in range(mul_in):
                z[zo + u * zs:zo + u * zs + dout] = zz[u]
        racc = np.zeros(n_acc * WARP)
        acc = np.zeros((WARP, 12))
        for (tb, te, g_off, nfl) in chunks:
            stage = w[e, g_off:g_off + nfl]
            for (wloc, zb, _nf, flags, rs, dout, vec, lpi, R, ab, zs, _kind, nrows, _a, _b, _c) in tiles[tb:te]:
                lpr = lprs[lpi]
                assert (_nf & 0xffff) == nrows // R and (_nf >> 16) == nrows % R
                if flags & 1:
                    acc[:] = 0
                for lane in range(WARP):
                    r, c = divmod(lane, lpr)
                    if r >= R:
                        continue
                    for u in range(r, nrows, R):
                        for v in range(vec):
                            wv = stage[wloc + u * rs + c * vec + v]
                            for k in range(dout):
                                acc[lane, v * dout + k] += wv * z[zb + u * zs + k]
                if flags & 2:
                    for lane in range(WARP):
                        for q in range(vec * dout):
                            racc[ab + q * WARP + lane] += acc[lane, q]
        for o, (base, stride, R) in enumerate(outmap):
            out[e, o] = sum(racc[base + r * stride] for r in range(R))
    return out


# ------------------------------------------------------------------------------------------------
def full_tensor_product(irreps_1, irreps_2):
    """Dense form of e3nn's ``o3.FullTensorProduct(irreps_1, irreps_2)`` (models/cg_model.py:240): returns
    (T [D1, D2, D_out] float64, out_irreps) with  out[c] = sum_ab T[a,b,c] x1[a] x2[b].  One 'uvuv' instruction per
    allowed (i1, i2, l_out) with coefficient sqrt(2 l_out + 1); output irreps sorted by (l, parity) with odd first,
    stably, as e3nn's Irreps.sort does on (l, p) tuples."""
    a, b = parse_irreps(irreps_1), parse_irreps(irreps_2)
    offa, offb = irreps_offsets(a), irreps_offsets(b)
    items = []
    for i, (m1, l1, p1) in enumerate(a):
        for j, (m2, l2, p2) in enumerate(b):
            for l3 in range(abs(l1 - l2), l1 + l2 + 1):
                items.append((i, j, m1 * m2, l3, p1 * p2))
    order = sorted(range(len(items)), key=lambda q: (items[q][3], items[q][4], q))
    out_irreps = [(items[q][2], items[q][3], items[q][4]) for q in order]
    offo = irreps_offsets(out_irreps)
    T = np.zeros((irreps_dim(a), irreps_dim(b), irreps_dim(out_irreps)))
    for pos, q in enumerate(order):
        i, j, mul, l3, _ = items[q]
        (m1, l1, _), (m2, l2, _) = a[i], b[j]
        C = real_cg(l1, l2, l3) * math.sqrt(2 * l3 + 1)
        for u in range(m1):
            for v in range(m2):
                o0 = offo[pos] + (u * m2 + v) * (2 * l3 + 1)
                T[offa[i] + u * (2 * l1 + 1):offa[i] + (u + 1) * (2 * l1 + 1),
                  offb[j] + v * (2 * l2 + 1):offb[j] + (v + 1) * (2 * l2 + 1), o0:o0 + 2 * l3 + 1] += C
    return T, out_irreps

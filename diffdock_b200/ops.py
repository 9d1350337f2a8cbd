"""Tensor-level wrappers over the C ABI (device pointers + current CUDA stream).  CUDA tensors only.

What each wrapper stands in for in the reference (details per entry point in include/diffdock_b200.h):
  deterministic / new_accumulators /    the convolutions' fixed-point scatter under torch.use_deterministic_algorithms(True)
  check_fixed_error
  tpconv_accumulate / tpconv_finalize   gather + o3.spherical_harmonics + tensor product + torch_scatter.scatter + bincount and
                                        the mean / BatchNorm / residual epilogue, models/tensor_layers.py:139-144,204-229,327-332
  radius                                torch_cluster.radius / radius_graph, models/cg_model.py:477,543-548,630
  segment_ptr                           the CSR row pointer of a sorted ``batch`` vector (PyG ``Batch.ptr``)
  pose_update                           utils/sampling.py:133-191 + utils/diffusion_utils.py:60-78 (modify_conformer_batch) +
                                        utils/torsion.py:75-90 + utils/geometry.py:246-276 (Kabsch); pose_update_packed does
                                        the same for poses of different ligands in one launch"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .tp_table import TpTable


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("diffdock_b200 ops run on CUDA tensors only (no CPU fallback)")


class _Profile:
    """Optional live accounting used by bench.py: CUDA-event pairs around every tensor-product conv launch (on the
    launching stream) with that launch's ALGORITHMIC bytes (SURVEY.md section 8(d)), and a count of all kernels
    launched through this module."""

    def __init__(self):
        self.reset(False)

    def reset(self, enabled=False):
        self.enabled, self.pairs, self.bytes, self.all_launches = enabled, [], 0, 0
        self.fused_pairs, self.fused_bytes, self.fused_flops, self.fused_alg_flops = [], 0, 0, 0

    def summary(self):
        torch.cuda.synchronize()
        return {'launches': len(self.pairs), 'ms': sum(a.elapsed_time(b) for a, b in self.pairs), 'bytes': self.bytes,
                'all_launches': self.all_launches, 'fused_launches': len(self.fused_pairs),
                'fused_ms': sum(a.elapsed_time(b) for a, b in self.fused_pairs), 'fused_bytes': self.fused_bytes,
                'fused_flops': self.fused_flops, 'fused_alg_flops': self.fused_alg_flops}


PROFILE = _Profile()


# ---------------------------------------------------------------------------------------------------------------------
# Deterministic convolutions.  Under torch.use_deterministic_algorithms(True) the convolution accumulators are int64 sums
# of 64-bit fixed-point values (2^-32 units, include/diffdock_b200.h: ddb200_tpconv_accumulate_fixed): integer addition is
# associative, so a forward gives the same bits whatever order the scatter reductions land in.  The flag is read where the
# accumulators are allocated (``new_accumulators``); every launch that takes an accumulator follows its dtype.
FIXED_SCALE = 2.0 ** 32
FIXED_LIMIT = 2.0 ** 31          # |value| of one edge (and of a sum) the fixed-point accumulators hold


def deterministic():
    """True when the convolutions use the fixed-point scatter: ``torch.are_deterministic_algorithms_enabled()``."""
    return torch.are_deterministic_algorithms_enabled()


def new_accumulators(n_rows, d_out, device):
    """Zeroed convolution accumulators ``(sum [n_rows, d_out], cnt [n_rows] fp32)``; ``sum`` is int64 fixed point when
    ``deterministic()``, else fp32."""
    dt = torch.int64 if deterministic() else torch.float32
    return (torch.zeros((n_rows, d_out), dtype=dt, device=device), torch.zeros((n_rows,), dtype=torch.float32, device=device))


_FIXED_ERR = {}


def fixed_error_word(device):
    """The device's sticky int32 error word of the fixed-point scatter (set when a value leaves the range).  Created on
    first use, which must not be inside a CUDA-graph capture (``GraphedSteps`` creates it before capturing)."""
    dev = torch.device(device)
    key = dev.index if dev.index is not None else torch.cuda.current_device()
    w = _FIXED_ERR.get(key)
    if w is None:
        w = _FIXED_ERR[key] = torch.zeros(1, dtype=torch.int32, device=torch.device('cuda', key))
    return w


def check_fixed_error(device=None):
    """Raise RuntimeError if a fixed-point scatter on ``device`` (None: every device used) saturated since the last check,
    and clear the word.  One device-to-host read per device; nothing to read when no fixed-point launch ran."""
    keys = list(_FIXED_ERR) if device is None else [torch.device(device).index if torch.device(device).index is not None
                                                    else torch.cuda.current_device()]
    for k in keys:
        w = _FIXED_ERR.get(k)
        if w is not None and int(w.item()):
            w.zero_()
            raise RuntimeError(f"deterministic convolution on cuda:{k}: a message value or sum left the fixed-point range "
                               f"|x| < 2^31 (torch.use_deterministic_algorithms(True))")


class TpHandle:
    """Device-resident tensor-product table (ddb200_tp_table)."""

    def __init__(self, table: TpTable):
        if not torch.cuda.is_available():
            raise RuntimeError("CUDA device required")
        self.table = table
        h = C.c_void_p()
        ib = np.ascontiguousarray(table.iblob, dtype=np.int32)
        fb = np.ascontiguousarray(table.fblob, dtype=np.float32)
        rc = _lib.lib().ddb200_tp_table_create(ib.ctypes.data_as(C.c_void_p), len(ib), fb.ctypes.data_as(C.c_void_p),
                                               len(fb), C.byref(h))
        _lib.check(rc, 'ddb200_tp_table_create')
        self._h = h

    def __deepcopy__(self, memo):
        return TpHandle(self.table)

    def info(self, what):
        return _lib.lib().ddb200_tp_table_info(self._h, what)

    def __del__(self):
        try:
            if getattr(self, '_h', None):
                _lib.lib().ddb200_tp_table_destroy(self._h)
        except Exception:
            pass


def tpconv_accumulate(h: TpHandle, x, edge_src, edge_dst, geo, w, sum_buf, cnt_buf=None, edge_weight=None,
                      count_node_bytes=True):
    """sum_buf[edge_dst[e]] += TP(x[edge_src[e]], Y(geo[e]), w[e]) (* edge_weight[e]);  cnt_buf[edge_dst[e]] += 1."""
    _need_cuda(x, edge_src, edge_dst, geo, w, sum_buf)
    E = edge_src.shape[0]
    if E == 0:
        return
    t = h.table
    assert x.dtype == torch.float32 and w.dtype == torch.float32 and geo.dtype == torch.float32
    assert sum_buf.dtype in (torch.float32, torch.int64)
    assert edge_src.dtype == torch.int32 and edge_dst.dtype == torch.int32
    assert x.stride(1) == 1 and w.stride(1) == 1 and geo.is_contiguous() and sum_buf.is_contiguous()
    assert edge_src.is_contiguous() and edge_dst.is_contiguous()
    assert x.shape[1] == t.d_in and w.shape[1] >= t.weight_numel_padded and sum_buf.shape[1] == t.d_out
    assert geo.shape[0] == E and w.shape[0] == E and geo.shape[1] == (3 if t.sh_lmax >= 0 else t.d_sh)
    if edge_weight is not None:
        edge_weight = edge_weight.reshape(-1).contiguous().float()
        assert edge_weight.shape[0] == E
    prof = PROFILE.enabled
    if prof:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    if sum_buf.dtype == torch.int64:        # fixed-point accumulators (new_accumulators under the deterministic flag)
        rc = _lib.lib().ddb200_tpconv_accumulate_fixed(h._h, _ptr(x), x.stride(0), _ptr(edge_src), _ptr(edge_dst), _ptr(geo),
                                                       _ptr(edge_weight), _ptr(w), w.stride(0), E, _ptr(sum_buf),
                                                       _ptr(cnt_buf), _ptr(fixed_error_word(sum_buf.device)), _stream())
    else:
        rc = _lib.lib().ddb200_tpconv_accumulate(h._h, _ptr(x), x.stride(0), _ptr(edge_src), _ptr(edge_dst), _ptr(geo),
                                                 _ptr(edge_weight), _ptr(w), w.stride(0), E, _ptr(sum_buf), _ptr(cnt_buf),
                                                 _stream())
    if prof:
        e1.record()
        PROFILE.pairs.append((e0, e1))
        PROFILE.bytes += E * (4 * t.weight_numel + 12 + 4) + (4 * E if edge_weight is not None else 0)
        if count_node_bytes:   # node tensors are compulsory traffic once per (layer, edge set), not per edge block
            PROFILE.bytes += 4 * (sum_buf.shape[0] + 1) + 4 * x.shape[0] * t.d_in + 4 * sum_buf.shape[0] * t.d_out
    PROFILE.all_launches += 1
    _lib.check(rc, 'ddb200_tpconv_accumulate_fixed' if sum_buf.dtype == torch.int64 else 'ddb200_tpconv_accumulate')


def tpconv_finalize(sum_buf, cnt_buf, mean, bn_scale=None, bn_shift=None, residual=None, out=None):
    """The epilogue into fp32 ``out``; int64 (fixed-point) ``sum_buf`` takes ddb200_tpconv_finalize_fixed."""
    _need_cuda(sum_buf)
    n, d = sum_buf.shape
    fixed = sum_buf.dtype == torch.int64
    if out is None:
        out = torch.empty(sum_buf.shape, dtype=torch.float32, device=sum_buf.device)
    res_stride = residual.stride(0) if residual is not None else 0
    res_dim = residual.shape[1] if residual is not None else 0
    if residual is not None:
        assert residual.stride(1) == 1 and residual.shape[0] == n and res_dim <= d
    fin = _lib.lib().ddb200_tpconv_finalize_fixed if fixed else _lib.lib().ddb200_tpconv_finalize
    rc = fin(_ptr(sum_buf), _ptr(cnt_buf), n, d, 1 if mean else 0, _ptr(bn_scale), _ptr(bn_shift), _ptr(residual),
             res_stride, res_dim, _ptr(out), _stream())
    _lib.check(rc, 'ddb200_tpconv_finalize_fixed' if fixed else 'ddb200_tpconv_finalize')
    PROFILE.all_launches += 1
    return out


def segment_ptr(batch, num_graphs):
    """CSR offsets [B+1] (int32) of a sorted batch vector."""
    counts = torch.bincount(batch, minlength=num_graphs)
    ptr = torch.zeros(num_graphs + 1, dtype=torch.int32, device=batch.device)
    ptr[1:] = torch.cumsum(counts, 0)
    return ptr


def radius(x, y, x_ptr, y_batch, r=1.0, r_per_graph=None, max_num_neighbors=32, exclude_self=False):
    """Neighbour pairs (row = index into y, col = index into x), int32, sorted by (row, col).
    Semantics of torch_cluster.radius(x, y, r, batch_x, batch_y, max_num_neighbors)."""
    _need_cuda(x, y, x_ptr, y_batch)
    x, y = x.float().contiguous(), y.float().contiguous()
    yb = y_batch.to(torch.int32).contiguous()
    n_y = y.shape[0]
    if r_per_graph is not None:
        r_per_graph = r_per_graph.reshape(-1).float().contiguous()
    count = torch.empty(n_y, dtype=torch.int32, device=x.device)
    if x.shape[0] == 0:
        # nothing to search (a receptor that crop_beyond cropped to no residue): no pair, as torch_cluster.radius returns;
        # the entry points take no null x
        count.zero_()
        return count.new_empty(0), count.new_empty(0), count
    L = _lib.lib()
    rc = L.ddb200_radius_count(_ptr(x), _ptr(y), _ptr(x_ptr), _ptr(yb), _ptr(r_per_graph), float(r), n_y,
                               int(max_num_neighbors), int(exclude_self), _ptr(count), _stream())
    _lib.check(rc, 'ddb200_radius_count')
    incl = torch.cumsum(count, 0, dtype=torch.int32)
    row_start = (incl - count).contiguous()
    n_edges = int(incl[-1].item()) if n_y else 0      # host sync: the edge count sizes the output buffers
    row = torch.empty(n_edges, dtype=torch.int32, device=x.device)
    col = torch.empty(n_edges, dtype=torch.int32, device=x.device)
    if n_edges:
        rc = L.ddb200_radius_fill(_ptr(x), _ptr(y), _ptr(x_ptr), _ptr(yb), _ptr(r_per_graph), float(r), n_y,
                                  int(max_num_neighbors), int(exclude_self), _ptr(row_start), _ptr(row), _ptr(col),
                                  _stream())
        _lib.check(rc, 'ddb200_radius_fill')
    PROFILE.all_launches += 2
    return row, col, count


def pose_update(pos, n_poses, bond_u, bond_v, mask_rotate_u8, tr_score, rot_score, tor_score, coef, tr_z=None,
                rot_z=None, tor_z=None, use_torsion=True):
    """New ligand coordinates [n_poses * n_atoms, 3] after one reverse-diffusion step (ddb200_pose_update)."""
    _need_cuda(pos, tr_score, rot_score)
    pos = pos.float().contiguous()
    n_atoms = pos.shape[0] // n_poses
    n_bonds = int(bond_u.shape[0]) if bond_u is not None else 0
    f = lambda t: t.float().contiguous() if t is not None else None
    tr_score, rot_score, tor_score, tr_z, rot_z, tor_z = map(f, (tr_score, rot_score, tor_score, tr_z, rot_z, tor_z))
    out = torch.empty_like(pos)
    c = (C.c_float * 6)(*[float(v) for v in coef])
    rc = _lib.lib().ddb200_pose_update(_ptr(pos), n_poses, n_atoms, n_bonds, _ptr(bond_u), _ptr(bond_v),
                                       _ptr(mask_rotate_u8), _ptr(tr_score), _ptr(rot_score), _ptr(tor_score),
                                       _ptr(tr_z), _ptr(rot_z), _ptr(tor_z), C.cast(c, C.c_void_p),
                                       1 if use_torsion else 0, _ptr(out), _stream())
    _lib.check(rc, 'ddb200_pose_update')
    PROFILE.all_launches += 1
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Sync-free graph construction: upper-bound buffers + the live edge count in device memory (no .item())
def radius_count(x, y, x_ptr, y_batch32, r=1.0, r_per_graph=None, max_num_neighbors=32, exclude_self=False):
    """count[j] = neighbours of y_j among the x of its complex (ddb200_radius_count); int32, no host sync."""
    _need_cuda(x, y, x_ptr, y_batch32)
    assert x.dtype == torch.float32 and y.dtype == torch.float32 and x.is_contiguous() and y.is_contiguous()
    assert y_batch32.dtype == torch.int32 and x_ptr.dtype == torch.int32
    n_y = y.shape[0]
    count = torch.empty(n_y, dtype=torch.int32, device=x.device)
    rc = _lib.lib().ddb200_radius_count(_ptr(x), _ptr(y), _ptr(x_ptr), _ptr(y_batch32), _ptr(r_per_graph), float(r), n_y,
                                        int(max_num_neighbors), int(exclude_self), _ptr(count), _stream())
    _lib.check(rc, 'ddb200_radius_count')
    PROFILE.all_launches += 1
    return count


def graph_fill(x, y, x_ptr, y_batch32, row_start, capacity, r=1.0, r_per_graph=None, max_num_neighbors=32,
               exclude_self=False, pre_ptr=None, pre_col=None, want_vec=True, want_eid=False, slot_out=None, slot_in=None,
               y_ptr=None, slot_ld=0, want_perm=False, row_offset=0, col_offset=0, fill_row=None):
    """Fill pass into buffers of ``capacity`` edges (ddb200_graph_fill).  Returns (row, col, vec | None, eid | None,
    perm | None); entries beyond the live count keep their initial value: ``fill_row`` for row (None = uninitialised),
    0 for col / perm, (1, 0, 0) for vec, -1 for eid - valid operands for padded library ops."""
    dev = x.device
    n_y = y.shape[0]
    cap = max(int(capacity), 1)
    init = fill_row is not None
    row = torch.full((cap,), int(fill_row), dtype=torch.int32, device=dev) if init else torch.empty(cap, dtype=torch.int32, device=dev)
    col = torch.zeros(cap, dtype=torch.int32, device=dev) if init else torch.empty(cap, dtype=torch.int32, device=dev)
    vec = eid = perm = None
    if want_vec:
        vec = torch.empty((cap, 3), dtype=torch.float32, device=dev)
        if init:
            vec.zero_()
            vec[:, 0] = 1.0
    if want_eid:
        eid = torch.full((cap,), -1, dtype=torch.int32, device=dev)
    if want_perm:
        perm = torch.zeros(cap, dtype=torch.int32, device=dev) if init else torch.empty(cap, dtype=torch.int32, device=dev)
    rc = _lib.lib().ddb200_graph_fill(_ptr(x), _ptr(y), _ptr(x_ptr), _ptr(y_batch32), _ptr(r_per_graph), float(r), n_y,
                                      int(max_num_neighbors), int(exclude_self), _ptr(row_start), _ptr(pre_ptr),
                                      _ptr(pre_col), _ptr(row), _ptr(col), _ptr(vec), _ptr(eid), _ptr(slot_out),
                                      _ptr(slot_in), _ptr(y_ptr), int(slot_ld), _ptr(perm), int(row_offset),
                                      int(col_offset), _stream())
    _lib.check(rc, 'ddb200_graph_fill')
    PROFILE.all_launches += 1
    return row, col, vec, eid, perm


EDGE_EMBED_SHAPES = {(64, 48), (32, 48), (64, 32), (32, 32), (64, 24), (32, 24), (64, 16), (32, 16), (16, 16), (8, 16),
                     (16, 24), (8, 24)}


def edge_embed(edge_vec, edge_row, u, w1_rbf, w2, b2, rbf_offset, rbf_coeff, n_edges_dev, out=None):
    """out[e] = W2 relu(u[edge_row[e]] + W1_rbf rbf(|edge_vec[e]|)) + b2 for e < *n_edges_dev (ddb200_edge_embed)."""
    _need_cuda(edge_vec, edge_row, u, w1_rbf, w2, b2)
    cap, ns, D = edge_vec.shape[0], u.shape[1], w1_rbf.shape[1]
    assert (D, ns) in EDGE_EMBED_SHAPES
    for t in (edge_vec, u, w1_rbf, w2, b2, rbf_offset):
        assert t.dtype == torch.float32 and t.is_contiguous()
    assert edge_row.dtype == torch.int32 and w1_rbf.shape[0] == ns and tuple(w2.shape) == (ns, ns) and rbf_offset.shape[0] == D
    if out is None:
        out = torch.empty((cap, ns), dtype=torch.float32, device=edge_vec.device)
    rc = _lib.lib().ddb200_edge_embed(_ptr(edge_vec), _ptr(edge_row), _ptr(u), _ptr(w1_rbf), _ptr(w2), _ptr(b2), D, ns,
                                      _ptr(rbf_offset), float(rbf_coeff), cap, _ptr(n_edges_dev), _ptr(out), _stream())
    _lib.check(rc, 'ddb200_edge_embed')
    PROFILE.all_launches += 1
    return out


def pose_update_dev(pos, n_poses, bond_u, bond_v, mask_rotate_u8, tr_score, rot_score, tor_score, coef_table, step_dev=None,
                    tr_z=None, rot_z=None, tor_z=None, seed=0, pose_key=None, use_torsion=True, out=None):
    """ddb200_pose_update_dev: SDE coefficients from a device table row, optional in-kernel Philox noise; ``out`` may be
    ``pos`` itself (in place)."""
    _need_cuda(pos, tr_score, rot_score, coef_table)
    assert pos.dtype == torch.float32 and pos.is_contiguous() and coef_table.dtype == torch.float32 and coef_table.is_contiguous()
    n_atoms = pos.shape[0] // n_poses
    n_bonds = int(bond_u.shape[0]) if bond_u is not None else 0
    f = lambda t: t.float().contiguous() if t is not None else None
    tr_score, rot_score, tor_score, tr_z, rot_z, tor_z = map(f, (tr_score, rot_score, tor_score, tr_z, rot_z, tor_z))
    if out is None:
        out = torch.empty_like(pos)
    if pose_key is not None:
        assert pose_key.dtype == torch.int64 and pose_key.is_cuda and pose_key.shape[0] >= n_poses
    if step_dev is not None:
        assert step_dev.dtype == torch.int32 and step_dev.is_cuda
    rc = _lib.lib().ddb200_pose_update_dev(_ptr(pos), n_poses, n_atoms, n_bonds, _ptr(bond_u), _ptr(bond_v),
                                           _ptr(mask_rotate_u8), _ptr(tr_score), _ptr(rot_score), _ptr(tor_score),
                                           _ptr(tr_z), _ptr(rot_z), _ptr(tor_z), _ptr(coef_table), _ptr(step_dev),
                                           C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), _ptr(pose_key),
                                           1 if use_torsion else 0, _ptr(out), _stream())
    _lib.check(rc, 'ddb200_pose_update_dev')
    PROFILE.all_launches += 1
    return out


def pose_update_packed(pos, layout, max_atoms, bond_u, bond_v, mask_u8, tr_score, rot_score, tor_score, coef_table, err,
                       step_dev=None, tr_z=None, rot_z=None, tor_z=None, seed=0, pose_key=None, use_torsion=True, out=None):
    """ddb200_pose_update_packed: ``pose_update_dev`` over poses of different ligands.  ``layout`` [n_poses, 6] int32 on the
    device (atom_off, n_atoms, bond_off, n_bonds, tor_off, mask_off per pose; include/diffdock_b200.h), ``max_atoms`` >= every
    pose's n_atoms; ``err`` a device int32 the kernel sets to 1 when a pose is out of range (never reset here).  ``out`` may
    be ``pos`` itself (in place)."""
    _need_cuda(pos, layout, tr_score, rot_score, coef_table, err)
    assert pos.dtype == torch.float32 and pos.is_contiguous() and coef_table.dtype == torch.float32 and coef_table.is_contiguous()
    assert layout.dtype == torch.int32 and layout.is_contiguous() and layout.dim() == 2 and layout.shape[1] == 6
    assert err.dtype == torch.int32 and err.numel() >= 1
    n_poses = layout.shape[0]
    f = lambda t: t.float().contiguous() if t is not None else None
    tr_score, rot_score, tor_score, tr_z, rot_z, tor_z = map(f, (tr_score, rot_score, tor_score, tr_z, rot_z, tor_z))
    if out is None:
        out = torch.empty_like(pos)
    if pose_key is not None:
        assert pose_key.dtype == torch.int64 and pose_key.is_cuda and pose_key.shape[0] >= n_poses
    if step_dev is not None:
        assert step_dev.dtype == torch.int32 and step_dev.is_cuda
    rc = _lib.lib().ddb200_pose_update_packed(_ptr(pos), n_poses, _ptr(layout), int(max_atoms), _ptr(bond_u), _ptr(bond_v),
                                              _ptr(mask_u8), _ptr(tr_score), _ptr(rot_score), _ptr(tor_score), _ptr(tr_z),
                                              _ptr(rot_z), _ptr(tor_z), _ptr(coef_table), _ptr(step_dev),
                                              C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), _ptr(pose_key),
                                              1 if use_torsion else 0, _ptr(err), _ptr(out), _stream())
    _lib.check(rc, 'ddb200_pose_update_packed')
    PROFILE.all_launches += 1
    return out


def crop_flags(lig_pos, lig_ptr, rec_pos, rec_batch32, cutoff2_table, step_dev=None):
    """Residues within the cut-off of some ligand atom of their complex (ddb200_crop_flags): ``(keep bool [n_rec], receptor
    positions with +inf at dropped residues [n_rec, 3])``; the squared cut-off is row ``*step_dev`` of ``cutoff2_table``."""
    _need_cuda(lig_pos, lig_ptr, rec_pos, rec_batch32, cutoff2_table)
    for t in (lig_pos, rec_pos, cutoff2_table):
        assert t.dtype == torch.float32 and t.is_contiguous()
    assert lig_ptr.dtype == torch.int32 and rec_batch32.dtype == torch.int32
    if step_dev is not None:
        assert step_dev.dtype == torch.int32 and step_dev.is_cuda
    n_rec = rec_pos.shape[0]
    keep = torch.empty(n_rec, dtype=torch.bool, device=rec_pos.device)
    masked = torch.empty_like(rec_pos)
    rc = _lib.lib().ddb200_crop_flags(_ptr(lig_pos), _ptr(lig_ptr), _ptr(rec_pos), _ptr(rec_batch32), n_rec,
                                      _ptr(cutoff2_table), _ptr(step_dev), _ptr(keep), _ptr(masked), _stream())
    _lib.check(rc, 'ddb200_crop_flags')
    PROFILE.all_launches += 1
    return keep, masked


def crop_select_edges(tgt32, src32, keep, gid32=None, offset=0, need=None, out=None):
    """The edges of a static list whose two ends are kept and whose target is needed, original order
    (ddb200_crop_select_edges): ``(tgt + offset, src + offset, perm, gid | None, n_dev)`` in buffers as long as the input;
    only the first ``n_dev[0]`` rows are live.  ``keep`` / ``need`` (bool / uint8 [n_rec]): None drops that condition.
    ``out``: buffers of an earlier call with the same list to write into (``select_edges_buffers``), so that a captured
    step allocates nothing.  No host synchronisation."""
    _need_cuda(tgt32, src32, keep, need)
    assert tgt32.dtype == torch.int32 and src32.dtype == torch.int32 and tgt32.is_contiguous() and src32.is_contiguous()
    for f in (keep, need):
        if f is not None:
            assert f.dtype in (torch.bool, torch.uint8) and f.is_contiguous()
    if gid32 is not None:
        assert gid32.dtype == torch.int32 and gid32.is_contiguous()
    n = tgt32.shape[0]
    if out is None:
        out = select_edges_buffers(n, tgt32.device, gid32 is not None)
    ws, out_t, out_s, perm, out_g, n_dev = out
    assert out_t.shape[0] >= n and (out_g is not None or gid32 is None)
    have = C.c_size_t(ws.numel())
    _lib.check(_lib.lib().ddb200_crop_select_edges(_ptr(tgt32), _ptr(src32), _ptr(gid32), n, _ptr(keep), _ptr(need),
                                                   int(offset), _ptr(out_t), _ptr(out_s), _ptr(perm),
                                                   _ptr(out_g if gid32 is not None else None), _ptr(n_dev), _ptr(ws),
                                                   C.byref(have), _stream()), 'ddb200_crop_select_edges')
    PROFILE.all_launches += 4
    return out_t[:n], out_s[:n], perm[:n], out_g[:n] if gid32 is not None else None, n_dev


def select_edges_buffers(n, dev, with_gid=True):
    """Workspace and outputs of ``crop_select_edges`` over a list of ``n`` edges: ``(workspace, tgt, src, perm, gid | None,
    n_dev)``."""
    L = _lib.lib()
    size = C.c_size_t(0)
    _lib.check(L.ddb200_crop_select_edges(None, None, None, n, None, None, 0, None, None, None, None, None, None,
                                          C.byref(size), _stream()), 'ddb200_crop_select_edges(size)')
    ws = torch.empty(max(int(size.value), 1), dtype=torch.uint8, device=dev)
    out_t, out_s, perm = (torch.empty(max(n, 1), dtype=torch.int32, device=dev) for _ in range(3))
    out_g = torch.empty(max(n, 1), dtype=torch.int32, device=dev) if with_gid else None
    return ws, out_t, out_s, perm, out_g, torch.empty(1, dtype=torch.int32, device=dev)


def receptor_need(cross_tgt32, n_cross, offset, tgt32, src32, n_rec, n_levels, keep=None, out=None):
    """The residues that can still pass a message to a ligand atom (ddb200_receptor_need): uint8 [n_levels, n_rec], row k
    = R_{k+1}.  R_1: ``cross_tgt32[e] - offset`` for e < ``n_cross[0]`` (the receptor <- ligand edges in the joint
    numbering, a capacity buffer); each further row adds the sources of the contact edges ``tgt32`` / ``src32`` (receptor
    numbering) into the previous one, over edges whose two ends are kept (``keep`` None: all).  No host synchronisation."""
    _need_cuda(cross_tgt32, n_cross, tgt32, src32, keep)
    for t in (cross_tgt32, n_cross, tgt32, src32):
        assert t.dtype == torch.int32 and t.is_contiguous()
    if keep is not None:
        assert keep.dtype in (torch.bool, torch.uint8) and keep.is_contiguous() and keep.shape[0] == n_rec
    if out is None:
        out = torch.empty((n_levels, n_rec), dtype=torch.uint8, device=tgt32.device)
    assert out.dtype == torch.uint8 and out.is_contiguous() and out.shape == (n_levels, n_rec)
    rc = _lib.lib().ddb200_receptor_need(_ptr(cross_tgt32), _ptr(n_cross), cross_tgt32.shape[0], int(offset), _ptr(tgt32),
                                         _ptr(src32), tgt32.shape[0], _ptr(keep), int(n_rec), int(n_levels), _ptr(out),
                                         _stream())
    _lib.check(rc, 'ddb200_receptor_need')
    PROFILE.all_launches += max(n_levels, 0)
    return out


CONF_MAX_IN, CONF_MAX_HIDDEN, CONF_MAX_OUT = 256, 128, 16       # DDB200_CONF_MAX_* of include/diffdock_b200.h


def confidence_head(x, lig_ptr, n_head, n_tail, mlp, dims, atom_mlp=None, atom_dims=None):
    """ddb200_confidence_head: ``(confidence [B, n_out], atom_confidence [n_lig, n_atom_out] | None)`` from the ligand node
    features ``x`` [n_lig, D] and the pose pointer ``lig_ptr`` [B+1] (int32, device).  The selected columns are the first
    ``n_head`` and the last ``n_tail`` of ``x``; ``mlp`` / ``atom_mlp`` are packed MLPs (layout in the header) of
    ``dims`` = (in, hidden, out) and ``atom_dims`` = (hidden, n_atom_out).  No host synchronisation."""
    _need_cuda(x, lig_ptr, mlp, atom_mlp)
    assert x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    assert lig_ptr.dtype == torch.int32 and lig_ptr.is_contiguous()
    assert mlp.dtype == torch.float32 and mlp.is_contiguous()
    n_in, n_hidden, n_out = dims
    B, n_lig, D = lig_ptr.shape[0] - 1, x.shape[0], x.shape[1]
    conf = torch.empty((B, n_out), dtype=torch.float32, device=x.device)
    atom_conf, a_h, a_out = None, 0, 0
    if atom_mlp is not None:
        assert atom_mlp.dtype == torch.float32 and atom_mlp.is_contiguous()
        a_h, a_out = atom_dims
        atom_conf = torch.empty((n_lig, a_out), dtype=torch.float32, device=x.device)
    rc = _lib.lib().ddb200_confidence_head(_ptr(x), max(x.stride(0), D), D, _ptr(lig_ptr), B, int(n_head), D - int(n_tail),
                                           int(n_tail), _ptr(atom_mlp), a_h, a_out, _ptr(mlp), n_in, n_hidden, n_out,
                                           _ptr(conf), _ptr(atom_conf), _stream())
    _lib.check(rc, 'ddb200_confidence_head')
    PROFILE.all_launches += 1
    return conf, atom_conf


def csr_sort_by_target(tgt32, n_rows, want_row_ptr=False):
    """Stable device-side sort of an edge list by target: (tgt_sorted int32, perm int64, row_ptr int32 | None);
    ddb200_csr_sort_by_target with a torch-allocated workspace.  No host synchronisation."""
    _need_cuda(tgt32)
    assert tgt32.dtype == torch.int32 and tgt32.is_contiguous()
    n = tgt32.shape[0]
    dev = tgt32.device
    L = _lib.lib()
    need = C.c_size_t(0)
    _lib.check(L.ddb200_csr_sort_by_target(None, n, int(n_rows), None, None, None, None, C.byref(need), _stream()),
               'ddb200_csr_sort_by_target(size)')
    ws = torch.empty(max(int(need.value), 1), dtype=torch.uint8, device=dev)
    out_t = torch.empty_like(tgt32)
    perm = torch.empty_like(tgt32)
    rp = torch.empty(int(n_rows) + 1, dtype=torch.int32, device=dev) if want_row_ptr else None
    have = C.c_size_t(ws.numel())
    _lib.check(L.ddb200_csr_sort_by_target(_ptr(tgt32), n, int(n_rows), _ptr(out_t), _ptr(perm), _ptr(rp), _ptr(ws),
                                           C.byref(have), _stream()), 'ddb200_csr_sort_by_target')
    PROFILE.all_launches += 2 + (1 if want_row_ptr else 0)
    return out_t, perm.long(), rp

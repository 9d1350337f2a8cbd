"""GPU: every kernel launch of real model forwards and sampler steps, replayed one launch at a time against the float64 or
oracle reference of that kernel's own test file.

The kernel tests feed synthetic inputs (random targets, ``randn`` edge vectors, hand-placed indirections); the model tests
compare only the final scores or confidences, at 1e-4 of the global maximum, where an error in one layer's 1o block is
diluted.  Here a recorder wraps the module attributes the product calls through (``fused.fused_conv``, ``ops.*``,
``radial.*``) and keeps, per launch, clones of the inputs, of the buffers the launch adds to or writes, and of its outputs.
After the workload, each launch is recomputed from its recorded inputs:

  fused_conv          parity_helpers.fused_conv_reference (test_tp_weights_layers_cpu.fused_conv_reference_deep for deep
                      radial MLPs) from the nn.Linear weights of the layer (``TensorProductConvLayer._fused_plan`` is
                      wrapped to map each plan to its FCBlock), with edge_perm, ea_add / ea_add_idx, vec_sign and the
                      device live count applied; swapped launches (v1.0 models) are given ``[ea | node[src] | node[tgt]]``.
                      The accumulator delta (after - before) per output irrep block < 3e-5 (test_fused_conv_fp64_gpu),
                      the count delta = bincount of the live targets exactly.
  tpconv_accumulate   tp_scatter_reference with the per-edge weights mapped back to reference order, 6e-6 per block
                      (test_tpconv_fp64_gpu TOL: the weights are exact fp32 inputs).
  tpconv_finalize     the float64 epilogue, FIN_TOL 1.6e-7 per block.
  radial_mlp / gemm   float64 of the layer's FCBlock in the kernel's weight-row layout: 6e-5 / 3e-5 of the output max
                      (test_radial_gemm_gpu).
  edge_embed          _embed_ref, EMBED_TOL 1.5e-6; rows at and past the live count bit-identical to before the launch.
  confidence_head     confidence_v11_helpers.head_f64, relative error per output column < 5e-6 (HEAD_TOL).
  radius_count, graph_fill, radius
                      exact against oracle.graph_ops.radius (test_graph_kernels_ref_gpu._oracle), edge vectors bit for
                      bit, padding rows at their fill values, a reverse pass's permutation pointing at the same pair of the
                      forward list.
  crop_flags          bit-exact against the oracle's crop expression (oracle/diffusion.py:crop_beyond).
  crop_select_edges   exact against boolean-mask indexing;  receptor_need exact against a host BFS (_bfs).
  pose updates        test_pose_update_fp64_gpu.reference with Philox noise from ddb200_philox_probe, 2.6e-5 of each
                      pose's extent (TOL_SIZES: tree ligands of up to 150 atoms).

Every ``ddb200_*`` entry point of the loaded library is also wrapped with a call counter: a call made during a workload
outside any recorded wrapper fails the test unless the entry point is on ``EXEMPT`` (with its reason).
tests/test_launch_replay_cpu.py keeps ``WRAPPED`` + ``EXEMPT`` equal to the library's signature table.

Largest errors of the replay per launch kind over the unmutated workloads, measured in one run on an NVIDIA H100 80GB HBM3
(700 W power limit); 917 launches, the whole file in 29 s:
  fused_conv 1.49e-5 (306 launches), swapped 1.52e-5 (4), second order 1.03e-5 (28), deep MLP 6.32e-6 (28)
  radial_mlp 1.03e-5, tpconv_accumulate 8.21e-7, tpconv_finalize 9.78e-8, edge_embed 4.60e-7, confidence_head 1.00e-6,
  pose_update_dev 8.76e-6, pose_update_packed 6.94e-6; graph, crop and need kernels exact.
A Clebsch-Gordan table of one l_out = 1 path scaled by 1 + 3e-4 in one layer's plan gives 2.96e-4 on that launch, while the
scores move by 4.5e-6 of their maxima, which the model-level 1e-4 check misses.  Run with -s for the table of every
workload and launch kind."""
import copy
import inspect
import types
from collections import Counter, defaultdict
from functools import partial

import numpy as np
import pytest
import torch
from torch import nn

from tests.confidence_v11_helpers import head_f64
from tests.parity_helpers import block_errors, fused_conv_reference, rel_err, tp_scatter_reference
from tests.test_graph_kernels_ref_gpu import EMBED_TOL, _embed_ref, _oracle
from tests.test_pose_update_fp64_gpu import TOL_SIZES, _probe, pose_err, reference as pose_reference
from tests.test_receptor_prune_gpu import _bfs
from tests.test_tp_weights_layers_cpu import fused_conv_reference_deep
from tests.test_tpconv_fp64_gpu import FIN_TOL, TOL as TP_TOL

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
FUSED_TOL = 3e-5         # tests/test_fused_conv_fp64_gpu.py
GEMM_TOL, MLP_TOL = 3e-5, 6e-5      # tests/test_radial_gemm_gpu.py
# per output column, relative to the column's max: test_confidence_v11_gpu's 2e-5 is of max(1, |ref|), a floor the pooled
# confidences of a random model sit far below; the largest measured here is 1.0e-6, so 5e-6
HEAD_TOL = 5e-6

# ddb200 entry point -> the wrappers (module attribute paths) whose calls make it; the recorder patches every one of them
WRAPPED = {
    'ddb200_fused_conv': ['fused.fused_conv'],
    'ddb200_fused_conv_so': ['fused.fused_conv'],
    'ddb200_tpconv_accumulate': ['ops.tpconv_accumulate'],
    'ddb200_tpconv_finalize': ['ops.tpconv_finalize'],
    'ddb200_radial_gemm': ['radial.radial_gemm'],
    'ddb200_radial_mlp': ['radial.radial_mlp'],
    'ddb200_edge_embed': ['ops.edge_embed'],
    'ddb200_confidence_head': ['ops.confidence_head'],
    'ddb200_radius_count': ['ops.radius_count', 'ops.radius'],
    'ddb200_radius_fill': ['ops.radius'],
    'ddb200_graph_fill': ['ops.graph_fill'],
    'ddb200_crop_flags': ['ops.crop_flags'],
    'ddb200_crop_select_edges': ['ops.crop_select_edges'],
    'ddb200_receptor_need': ['ops.receptor_need'],
    'ddb200_pose_update': ['ops.pose_update'],
    'ddb200_pose_update_dev': ['ops.pose_update_dev'],
    'ddb200_pose_update_packed': ['ops.pose_update_packed'],
}
# entry points a workload may call outside a recorded wrapper, and why they need no replay here
EXEMPT = {
    'ddb200_version': "a version string; no device work",
    'ddb200_tp_table_create': "uploads the static tables of tp_table.build_table (checked by test_tp_table)",
    'ddb200_tp_table_destroy': "frees a table handle",
    'ddb200_tp_table_info': "reads a table handle's host-side sizes",
    'ddb200_csr_sort_by_target': "a stable sort permutation, tested exactly by its own tests",
    'ddb200_crop_select_edges:size': "the workspace-size query of select_edges_buffers (null data pointers, no launch)",
    'ddb200_fused_debug_read': "a debug hook of the fused kernel, not called by a forward",
    'ddb200_philox_probe': "a test hook; the replay itself calls it for the reference noise",
    'ddb200_contact_count': "the input-side contact graph, not called by a forward (test_contact_graph_ref_*)",
    'ddb200_contact_fill': "the input-side contact graph, not called by a forward (test_contact_graph_ref_*)",
}
SIZE_QUERIES = ('ddb200_crop_select_edges', 'ddb200_csr_sort_by_target')    # first argument NULL: a size query

# buffers a launch adds to or writes besides its return value
WRITES = {'fused.fused_conv': ('sum_buf', 'cnt_buf'), 'ops.tpconv_accumulate': ('sum_buf', 'cnt_buf'),
          'ops.graph_fill': ('slot_out',), 'ops.pose_update_packed': ('err',)}

SUM_PTR = ('fused.fused_conv', 'ops.tpconv_accumulate', 'ops.tpconv_finalize')   # accumulator base address kept

TABLE = defaultdict(lambda: [0.0, 0])          # (workload, kind) -> [largest error / tolerance-relative value, launches]


def _clone(v):
    if torch.is_tensor(v):
        return v.detach().clone()
    if isinstance(v, (tuple, list)):
        return type(v)(_clone(x) for x in v)
    return v


def _resolve(path):
    from diffdock_b200 import fused, ops, radial
    mod, name = path.split('.')
    return {'fused': fused, 'ops': ops, 'radial': radial}[mod], name


class Recorder:
    """Wraps the product's kernel entry points (module attributes and ctypes functions) for the life of ``mp``."""

    def __init__(self, mp, conf_model=None):
        from diffdock_b200 import _lib
        from diffdock_b200.tensor_layers import TensorProductConvLayer
        # records of eager launches, and of launches made while a CUDA graph was being captured: the clones of the latter
        # are part of the graph, so every replay refreshes them with that replay's values
        self.records, self.captured, self.plans, self.depth, self.active = [], [], {}, 0, False
        self.matched, self.escaped = Counter(), Counter()
        self.cap_matched, self.cap_escaped = Counter(), Counter()       # the same counts, of calls made during a capture
        self.radial_ctx, self.conf_model, self.call_mutation = None, conf_model, {}
        for path in sorted({p for ps in WRAPPED.values() for p in ps}):
            mod, name = _resolve(path)
            mp.setattr(mod, name, self._wrap(path, getattr(mod, name)))
        L = _lib.lib()
        for name in _lib.SIGNATURES:
            mp.setattr(L, name, self._count(name, getattr(L, name)))
        plan_fn = TensorProductConvLayer._fused_plan

        def fused_plan(layer, fc, table, k_in, swap_ns=0):
            plan = plan_fn(layer, fc, table, k_in, swap_ns)
            if plan is not None:
                self.plans[id(plan)] = (plan, fc, table, swap_ns)
            return plan
        mp.setattr(TensorProductConvLayer, '_fused_plan', fused_plan)
        for meth in ('_edge_weights', '_edge_weights_fused'):
            mp.setattr(TensorProductConvLayer, meth, self._radial_context(getattr(TensorProductConvLayer, meth)))

    def _radial_context(self, f):
        def g(layer, fc, table, *a, **kw):
            self.radial_ctx = (fc, table)
            try:
                return f(layer, fc, table, *a, **kw)
            finally:
                self.radial_ctx = None
        return g

    def _count(self, name, fn):
        def g(*a):
            key = name + ':size' if name in SIZE_QUERIES and a and a[0] is None else name
            if self.active:
                (self.matched if self.depth else self.escaped)[key] += 1
                if torch.cuda.is_current_stream_capturing():
                    (self.cap_matched if self.depth else self.cap_escaped)[key] += 1
            if name in self.call_mutation:
                a = self.call_mutation[name](a)
            return fn(*a)
        return g

    def _wrap(self, path, f):
        sig = inspect.signature(f)

        def g(*a, **kw):
            b = sig.bind(*a, **kw)
            b.apply_defaults()
            args = b.arguments
            if path == 'ops.edge_embed' and args['out'] is None:       # the buffer the wrapper would allocate
                args['out'] = torch.empty((args['edge_vec'].shape[0], args['u'].shape[1]), dtype=torch.float32,
                                          device=args['edge_vec'].device)
            pre = {k: _clone(v) for k, v in args.items()}
            self.depth += 1
            try:
                ret = f(*b.args, **b.kwargs)
            finally:
                self.depth -= 1
            if self.active:
                post = {k: _clone(args[k]) for k in WRITES.get(path, ()) if args.get(k) is not None}
                if path == 'ops.graph_fill':         # a reverse pass reads the slots of its forward pass
                    post['slot_ptr'] = args['slot_out'].data_ptr() if args['slot_out'] is not None else None
                    pre['slot_in_ptr'] = args['slot_in'].data_ptr() if args['slot_in'] is not None else None
                if path in SUM_PTR:
                    pre['sum_ptr'] = args['sum_buf'].data_ptr()
                entry = (path, pre, _clone(ret), post, self.radial_ctx)
                (self.captured if torch.cuda.is_current_stream_capturing() else self.records).append(entry)
            return ret
        return g

    def start(self):
        torch.cuda.synchronize()
        for c in (self.records, self.captured, self.matched, self.escaped, self.cap_matched, self.cap_escaped):
            c.clear()
        self.active = True

    def stop(self):
        torch.cuda.synchronize()
        self.active = False


# ---------------------------------------------------------------------------------------------------------------------
# per-launch references: each returns (error, tolerance, detail)
def _live(n_dev, default):
    return int(n_dev.reshape(-1)[0]) if n_dev is not None else default


def check_fused(rec, a, ret, post, ctx):
    plan = a['plan']
    _, fc, table, swap = rec.plans[id(plan)]
    lins = [m for m in fc if isinstance(m, nn.Linear)]
    l1, l2, hidden = lins[0], lins[-1], [(m.weight, m.bias) for m in lins[1:-1]]
    E = int(a['tgt32'].shape[0]) if a['n_edges'] is None else int(a['n_edges'])
    n = _live(a['n_edges_dev'], E)
    tgt, src, ns = a['tgt32'][:n], a['src32'][:n], a['ns']
    perm = a['edge_perm'][:n] if a['edge_perm'] is not None else None
    idx = a['ea_add_idx'][:n] if a['ea_add'] is not None else None
    ew = a['edge_weight'].reshape(-1) if a['edge_weight'] is not None else None
    n_out = a['sum_buf'].shape[0]
    if swap:        # the reference model's order: [ea | node[src] | node[tgt]] (models/old_cg_model.py:264-265)
        r = perm.long() if perm is not None else torch.arange(n, device=tgt.device)
        ea = a['edge_attr'].double()[r]
        if idx is not None:
            ea = ea + a['ea_add'].double()[idx.long()]
        node = a['node'].double()
        ea = torch.cat([ea, node[src.long(), :ns], node[tgt.long(), :ns]], 1)
        kw = dict(ea=ea, node=None, ns=0, vec=a['edge_vec'][r], ew=ew[r] if ew is not None else None)
    else:
        kw = dict(ea=a['edge_attr'], node=a['node'], ns=ns, vec=a['edge_vec'], ew=ew, edge_perm=perm,
                  ea_add=a['ea_add'], ea_add_idx=idx)
    common = dict(tgt=tgt, src=src, x=a['x'], n_out=n_out, vec_sign=a['vec_sign'], **kw)
    if hidden:
        ref, rcnt = fused_conv_reference_deep(table, l1.weight, l1.bias, hidden, l2.weight, l2.bias, **common)
    else:
        ref, rcnt = fused_conv_reference(table, l1.weight, l1.bias, l2.weight, l2.bias, **common)
    got = post['sum_buf'].double() - a['sum_buf'].double()
    cnt = post['cnt_buf'].double() - a['cnt_buf'].double()
    assert torch.equal(cnt, rcnt), "fused_conv: count delta differs from bincount of the live targets"
    rec.irreps[(a['sum_ptr'], n_out * table.d_out, table.d_out)] = table.out_irreps
    errs = block_errors(got, ref, table.out_irreps)
    worst = max(errs, key=errs.get)
    kind = 'fused_conv_so' if plan.second_order else 'fused_conv'
    if swap:
        kind += '_swap'
    if hidden:
        kind += '_deep'
    return kind, errs[worst], FUSED_TOL, f"{worst} E={n}/{E}"


def check_tpconv(rec, a, ret, post, ctx):
    t = a['h'].table
    E = a['edge_src'].shape[0]
    perm = np.asarray(t.w_perm)
    cols = np.nonzero(perm >= 0)[0]
    w = a['w']
    w_ref = torch.zeros((E, t.weight_numel), dtype=torch.float64, device=w.device)
    w_ref[:, torch.as_tensor(perm[cols], device=w.device)] = w[:, torch.as_tensor(cols, device=w.device)].double()
    n_out = a['sum_buf'].shape[0]
    ref, rcnt = tp_scatter_reference(t, a['x'], a['edge_src'], a['edge_dst'], a['geo'], w_ref, n_out,
                                     ew=a['edge_weight'])
    got = post['sum_buf'].double() - a['sum_buf'].double()
    if a['cnt_buf'] is not None:
        assert torch.equal(post['cnt_buf'].double() - a['cnt_buf'].double(), rcnt), "tpconv: count delta"
    errs = block_errors(got, ref, t.out_irreps)
    worst = max(errs, key=errs.get)
    rec.irreps[(a['sum_ptr'], n_out * t.d_out, t.d_out)] = t.out_irreps
    return 'tpconv_accumulate', errs[worst], TP_TOL, f"{worst} E={E}"


def check_finalize(rec, a, ret, post, ctx):
    s, cnt = a['sum_buf'].double(), a['cnt_buf']
    ref = s
    if a['mean']:
        ref = ref / cnt.double().clamp_min(float(torch.finfo(torch.float32).eps))[:, None]
    if a['bn_scale'] is not None:
        ref = ref * a['bn_scale'].double() + a['bn_shift'].double()
    if a['residual'] is not None:
        ref[:, :a['residual'].shape[1]] += a['residual'].double()
    n, d = s.shape
    # the irreps of the accumulator this epilogue reads (the latest launch that added into the same memory), else one block
    irreps = next((v for (p, m, dd), v in reversed(list(rec.irreps.items()))
                   if p <= a['sum_ptr'] < p + 4 * m and dd == d), [(d, 0, 1)])
    errs = block_errors(ret, ref, irreps)
    worst = max(errs, key=errs.get)
    return 'tpconv_finalize', errs[worst], FIN_TOL, worst


def _layout_ref(table, ref, ldo):
    """float64 [E, weight_numel] in reference row order -> the kernel's weight-row layout [E, ldo] (padding zero)."""
    perm = np.asarray(table.w_perm)
    cols = np.nonzero(perm >= 0)[0]
    out = torch.zeros((ref.shape[0], ldo), dtype=torch.float64, device=ref.device)
    out[:, torch.as_tensor(cols, device=ref.device)] = ref[:, torch.as_tensor(perm[cols], device=ref.device)]
    return out


def check_radial_mlp(rec, a, ret, post, ctx):
    fc, table = ctx
    ns = a['ns']
    ea = a['edge_attr'].double()
    if ns:
        node = a['node'].double()
        ea = torch.cat([ea, node[a['tgt32'].long(), :ns], node[a['src32'].long(), :ns]], 1)
    l1, l2 = fc[0], fc[-1]
    ref = torch.relu(ea @ l1.weight.double().T + l1.bias.double()) @ l2.weight.double().T + l2.bias.double()
    exp = _layout_ref(table, ref, ret.shape[1])
    return 'radial_mlp', float((ret.double() - exp).abs().max() / exp.abs().max()), MLP_TOL, f"E={ea.shape[0]}"


def check_radial_gemm(rec, a, ret, post, ctx):
    fc, table = ctx
    l2 = fc[-1]
    h = a['h'].double()
    ref = h @ l2.weight.double().T + l2.bias.double()
    exp = _layout_ref(table, ref, ret.shape[1])
    got = ret[:h.shape[0]].double()
    return 'radial_gemm', float((got - exp).abs().max() / exp.abs().max()), GEMM_TOL, f"E={h.shape[0]}"


def check_edge_embed(rec, a, ret, post, ctx):
    cap = a['edge_vec'].shape[0]
    n = min(max(_live(a['n_edges_dev'], cap), 0), cap)
    before, after = a['out'], ret
    assert torch.equal(before[n:].view(torch.int32), after[n:].view(torch.int32)), "edge_embed wrote past the live count"
    if n == 0:
        return 'edge_embed', 0.0, EMBED_TOL, "no live edge"
    ref = _embed_ref(a['edge_vec'][:n], a['edge_row'][:n], a['u'], a['w1_rbf'], a['w2'], a['b2'], a['rbf_offset'],
                     a['rbf_coeff'])
    err = float((after[:n].double() - ref).abs().max()) / float(ref.abs().max())
    return 'edge_embed', err, EMBED_TOL, f"E={n}/{cap}"


def _col_err(got, ref):
    got, ref = got.double().cpu().reshape(ref.shape[0], -1), ref.double().cpu().reshape(ref.shape[0], -1)
    return float(((got - ref).abs().amax(0) / ref.abs().amax(0).clamp_min(1e-30)).max())


def check_conf_head(rec, a, ret, post, ctx):
    m = rec.conf_model
    atom = a['atom_mlp'] is not None
    ref, ref_atom = head_f64(a['x'], a['lig_ptr'], a['n_head'], a['n_tail'], m.confidence_predictor,
                             m.atom_confidence_predictor if atom else None, a['atom_dims'][1] if atom else 0)
    err = _col_err(ret[0], ref)
    if atom:
        err = max(err, _col_err(ret[1], ref_atom))
    return 'confidence_head', err, HEAD_TOL, f"B={ref.shape[0]}"


def _batch_of_ptr(ptr):
    ptr = ptr.long().cpu()
    return torch.repeat_interleave(torch.arange(ptr.shape[0] - 1), ptr[1:] - ptr[:-1])


def _radius_ref(a):
    return _oracle(a['x'], a['y'], _batch_of_ptr(a['x_ptr']), a['y_batch32'].long().cpu(), a['r'], a['r_per_graph'],
                   a['max_num_neighbors'], a['exclude_self'])


def check_radius_count(rec, a, ret, post, ctx):
    ref_row, _ = _radius_ref(dict(a, y_batch32=a['y_batch32']))
    assert torch.equal(ret.cpu().long(), torch.bincount(ref_row, minlength=a['y'].shape[0])), "radius_count"
    return 'radius_count', 0.0, 0.0, f"E={ref_row.shape[0]}"


def check_radius(rec, a, ret, post, ctx):
    ref_row, ref_col = _radius_ref(dict(a, y_batch32=a['y_batch']))
    row, col, cnt = ret
    assert torch.equal(row.cpu().long(), ref_row) and torch.equal(col.cpu().long(), ref_col), "radius"
    assert torch.equal(cnt.cpu().long(), torch.bincount(ref_row, minlength=a['y'].shape[0])), "radius count"
    return 'radius', 0.0, 0.0, f"E={ref_row.shape[0]}"


def check_graph_fill(rec, a, ret, post, ctx):
    assert a['pre_ptr'] is None, "static edges: not replayed (no forward passes them)"
    ref_row, ref_col = _radius_ref(a)
    E = ref_row.shape[0]
    row, col, vec, eid, perm = ret
    assert torch.equal(row[:E].cpu().long() - a['row_offset'], ref_row), "graph_fill rows"
    assert torch.equal(col[:E].cpu().long() - a['col_offset'], ref_col), "graph_fill columns"
    if vec is not None:
        assert torch.equal(vec[:E].cpu(), a['x'].cpu()[ref_col] - a['y'].cpu()[ref_row]), "edge vectors"
    if a['fill_row'] is not None:
        assert bool((row[E:] == a['fill_row']).all()) and bool((col[E:] == 0).all()), "graph_fill padding rows"
        if vec is not None:
            assert torch.equal(vec[E:], torch.tensor([1.0, 0.0, 0.0], device=vec.device).expand(vec.shape[0] - E, 3))
        if perm is not None:
            assert bool((perm[E:] == 0).all())
    kind = 'graph_fill'
    if a['slot_in'] is not None:          # reverse pass: perm[k] is the forward position of the same pair
        fwd = [r for r in rec._replaying[:rec._cur] if r[0] == 'ops.graph_fill'
               and r[3]['slot_ptr'] == a['slot_in_ptr']]
        assert fwd, "reverse pass without its forward pass"
        fa, fret = fwd[-1][1], fwd[-1][2]
        p = perm[:E].long()
        assert torch.equal(fret[0][p].long() - fa['row_offset'], col[:E].long() - a['col_offset']), "reverse perm (ligand)"
        assert torch.equal(fret[1][p].long() - fa['col_offset'], row[:E].long() - a['row_offset']), "reverse perm (x end)"
        kind = 'graph_fill_reverse'
    return kind, 0.0, 0.0, f"E={E}/{row.shape[0]}"


def check_crop_flags(rec, a, ret, post, ctx):
    keep, masked = ret
    step = int(a['step_dev'].reshape(-1)[0]) if a['step_dev'] is not None else 0
    c2 = a['cutoff2_table'].cpu()[step]
    lig, rec_pos = a['lig_pos'].cpu(), a['rec_pos'].cpu()
    ptr, rb = a['lig_ptr'].long().cpu(), a['rec_batch32'].long().cpu()
    ref = torch.zeros(rec_pos.shape[0], dtype=torch.bool)
    for b in range(ptr.shape[0] - 1):
        rows = torch.nonzero(rb == b).reshape(-1)
        l = lig[ptr[b]:ptr[b + 1]]
        if rows.numel() and l.shape[0]:       # oracle/diffusion.py:crop_beyond with the table's float32 squared cut-off
            ref[rows] = torch.any(torch.sum((l.unsqueeze(0) - rec_pos[rows].unsqueeze(1)) ** 2, -1) < c2, dim=1)
    keep, masked = keep.cpu(), masked.cpu()
    assert torch.equal(keep, ref), "crop_flags"
    assert torch.equal(masked[keep], rec_pos[keep]) and bool(torch.isposinf(masked[~keep]).all()), "crop positions"
    return 'crop_flags', 0.0, 0.0, f"kept {int(keep.sum())}/{keep.shape[0]}"


def check_select(rec, a, ret, post, ctx):
    t, s, perm, g, n_dev = ret
    tgt, src = a['tgt32'].long().cpu(), a['src32'].long().cpu()
    sel = torch.ones(tgt.shape[0], dtype=torch.bool)
    if a['keep'] is not None:
        k = a['keep'].bool().cpu()
        sel &= k[tgt] & k[src]
    if a['need'] is not None:
        sel &= a['need'].bool().cpu()[tgt]
    idx = torch.nonzero(sel).reshape(-1)
    n = int(n_dev.reshape(-1)[0])
    assert n == idx.shape[0], "crop_select_edges: live count"
    assert torch.equal(perm[:n].cpu().long(), idx), "crop_select_edges: perm"
    assert torch.equal(t[:n].cpu().long(), tgt[idx] + a['offset']) and torch.equal(s[:n].cpu().long(), src[idx] + a['offset'])
    if a['gid32'] is not None:
        assert torch.equal(g[:n].cpu().long(), a['gid32'].long().cpu()[idx])
    return 'crop_select_edges', 0.0, 0.0, f"{n}/{tgt.shape[0]}"


def check_need(rec, a, ret, post, ctx):
    keep = a['keep'].bool().cpu().numpy() if a['keep'] is not None else None
    want = _bfs(a['cross_tgt32'].cpu().numpy(), int(a['n_cross'].reshape(-1)[0]), a['offset'], a['tgt32'].cpu().numpy(),
                a['src32'].cpu().numpy(), a['n_rec'], a['n_levels'], keep)
    assert np.array_equal(ret.cpu().numpy(), want), "receptor_need"
    return 'receptor_need', 0.0, 0.0, f"levels {a['n_levels']}"


def _noise(seed, key, step, nb):
    z, _ = _probe(int(seed) & 0xFFFFFFFFFFFFFFFF, int(key), step, 2 + (nb + 3) // 4)
    z = z.cpu()
    q = torch.stack([z[2 + r // 4, r % 4] for r in range(nb)]) if nb else torch.zeros(0)
    return z[0, :3], z[1, :3], q


def _pose_ref(pos, n, bu, bv, mask, tr, rot, tor, coef, use_torsion, keys, seed, step, n_poses, zs=None):
    nb = int(bu.shape[0]) if bu is not None else 0
    lig = types.SimpleNamespace(n=n, bonds=np.stack([bu.cpu().numpy(), bv.cpu().numpy()], 1) if nb else np.zeros((0, 2), int),
                                mask=mask.cpu().numpy().astype(bool).reshape(nb, n) if nb else np.zeros((0, n), bool))
    tz = rz = qz = None
    if keys is not None:
        z = [_noise(seed, k, step, nb) for k in keys]
        tz, rz = torch.stack([v[0] for v in z]), torch.stack([v[1] for v in z])
        qz = torch.stack([v[2] for v in z]) if nb else None
    elif zs is not None:
        tz, rz, qz = zs
    ut = use_torsion and nb > 0 and tor is not None
    tor = tor.reshape(n_poses, nb) if ut else None
    qz = qz.reshape(n_poses, nb) if (ut and qz is not None) else None
    return pose_reference(lig, pos, n_poses, tr, rot, tor, coef, tz, rz, qz, use_torsion=ut)


def check_pose_dev(rec, a, ret, post, ctx):
    n_poses = a['n_poses']
    n = a['pos'].shape[0] // n_poses
    step = int(a['step_dev'].reshape(-1)[0]) if a['step_dev'] is not None else 0
    keys = a['pose_key'].cpu().tolist()[:n_poses] if a['pose_key'] is not None else None
    zs = (a['tr_z'], a['rot_z'], a['tor_z']) if a['tr_z'] is not None else None
    ref = _pose_ref(a['pos'], n, a['bond_u'], a['bond_v'], a['mask_rotate_u8'], a['tr_score'], a['rot_score'],
                    a['tor_score'], a['coef_table'][step].tolist(), a['use_torsion'], keys, a['seed'], step, n_poses, zs)
    return 'pose_update_dev', pose_err(ret, ref), TOL_SIZES, f"poses {n_poses}"


def check_pose_host(rec, a, ret, post, ctx):
    n_poses = a['n_poses']
    n = a['pos'].shape[0] // n_poses
    zs = (a['tr_z'], a['rot_z'], a['tor_z']) if a['tr_z'] is not None else None
    ref = _pose_ref(a['pos'], n, a['bond_u'], a['bond_v'], a['mask_rotate_u8'], a['tr_score'], a['rot_score'],
                    a['tor_score'], list(a['coef']), a['use_torsion'], None, 0, 0, n_poses, zs)
    return 'pose_update', pose_err(ret, ref), TOL_SIZES, f"poses {n_poses}"


def check_pose_packed(rec, a, ret, post, ctx):
    assert int(post['err'].reshape(-1)[0]) == 0, "pose_update_packed flagged a pose"
    lay = a['layout'].cpu().tolist()
    step = int(a['step_dev'].reshape(-1)[0]) if a['step_dev'] is not None else 0
    coef = a['coef_table'][step].tolist()
    keys = a['pose_key'].cpu().tolist()
    worst = 0.0
    for b, (a0, n, b0, nb, t0, m0) in enumerate(lay):
        ut = a['use_torsion'] and nb > 0
        bu = a['bond_u'][b0:b0 + nb] if ut else None
        bv = a['bond_v'][b0:b0 + nb] if ut else None
        mask = a['mask_u8'][m0:m0 + nb * n] if ut else None
        tor = a['tor_score'][t0:t0 + nb] if ut else None
        ref = _pose_ref(a['pos'][a0:a0 + n], n, bu, bv, mask, a['tr_score'][b:b + 1], a['rot_score'][b:b + 1], tor, coef,
                        ut, [keys[b]], a['seed'], step, 1)
        worst = max(worst, pose_err(ret[a0:a0 + n], ref))
    return 'pose_update_packed', worst, TOL_SIZES, f"poses {len(lay)}"


CHECKS = {'fused.fused_conv': check_fused, 'ops.tpconv_accumulate': check_tpconv, 'ops.tpconv_finalize': check_finalize,
          'radial.radial_mlp': check_radial_mlp, 'radial.radial_gemm': check_radial_gemm, 'ops.edge_embed': check_edge_embed,
          'ops.confidence_head': check_conf_head, 'ops.radius_count': check_radius_count, 'ops.radius': check_radius,
          'ops.graph_fill': check_graph_fill, 'ops.crop_flags': check_crop_flags, 'ops.crop_select_edges': check_select,
          'ops.receptor_need': check_need, 'ops.pose_update_dev': check_pose_dev, 'ops.pose_update': check_pose_host,
          'ops.pose_update_packed': check_pose_packed}


def replay(rec, workload, records=None, clear=True, table=TABLE):
    """Checks every launch of ``records`` (default: the eager records); returns {kind: (largest error, tolerance, launches,
    failures)} and asserts that no ddb200 call escaped the recorder.  ``clear``: empty ``records`` afterwards (the captured
    records are kept: the next replay of their graph refreshes them).  ``table``: where the largest errors are kept."""
    records = rec.records if records is None else records
    escaped = {k: v for k, v in rec.escaped.items() if k not in EXEMPT and k.split(':')[0] not in EXEMPT}
    assert not escaped, f"{workload}: ddb200 calls outside any recorded wrapper: {escaped}"
    rec.irreps = {}
    out = {}
    rec._replaying = records
    for i, (path, a, ret, post, ctx) in enumerate(records):
        rec._cur = i
        kind, err, tol, detail = CHECKS[path](rec, a, ret, post, ctx)
        e, t, n, bad = out.get(kind, (0.0, tol, 0, []))
        ok = err < tol if tol > 0 else err == 0.0
        out[kind] = (max(e, err), tol, n + 1, bad + ([(i, err, detail)] if not ok else []))
    if clear:
        records.clear()
    for kind, (e, t, n, bad) in out.items():
        cell = table[(workload, kind)]
        cell[0], cell[1] = max(cell[0], e), cell[1] + n
    torch.cuda.empty_cache()
    return out


def assert_clean(out, workload):
    bad = {k: v[3][:5] for k, v in out.items() if v[3]}
    assert not bad, f"{workload}: launches past their kernel's tolerance: {bad}"


@pytest.fixture(scope='module', autouse=True)
def _print_table():
    yield
    if not TABLE:
        return
    print(f"\n[launch replay] {torch.cuda.get_device_name(0)}; largest error per launch kind "
          f"(relative per block / column / pose extent; 0 = exact comparison):")
    kinds = defaultdict(lambda: [0.0, 0])
    for (w, k), (e, n) in sorted(TABLE.items()):
        print(f"  {w:<28s} {k:<24s} {n:6d} launches  max {e:.3e}")
        if not w.startswith('mutation'):
            kinds[k][0], kinds[k][1] = max(kinds[k][0], e), kinds[k][1] + n
    print("[launch replay] over the unmutated workloads:")
    for k, (e, n) in sorted(kinds.items()):
        print(f"  {k:<24s} {n:6d} launches  max {e:.3e}")
    print(f"  total {sum(n for _, n in kinds.values())} launches checked")


# ---------------------------------------------------------------------------------------------------------------------
# workloads
def _count(out, kind):
    return out.get(kind, (0, 0, 0, []))[2]


def _shared_batch(poses, t, args=None, crop_beyond=None, all_atoms=False):
    from diffdock_b200.diffusion_utils import set_time, t_to_sigma
    from diffdock_b200.hetero import collate_shared_receptor
    from diffdock_b200.sampling import crop_cutoff2
    g = collate_shared_receptor([q.clone() for q in poses], DEV)
    set_time(g, None, t, t, t, len(poses), all_atoms, DEV)
    g._uniform_t = True
    if crop_beyond is not None:
        table = torch.tensor([crop_cutoff2(partial(t_to_sigma, args=args), t, t, t, crop_beyond)], device=DEV)
        g._crop = (table, torch.zeros(1, dtype=torch.int32, device=DEV))
    return g


def _run(rec, model, g):
    rec.start()
    with torch.no_grad():
        out = model(g)
    rec.stop()
    return out


@pytest.fixture(scope='module')
def cg_l(built_lib):
    """CGModel at DiffDock-L shape (ns 48, nv 10, sh_lmax 2, 6 layers) and 2 poses of a 1500-residue / 40-atom complex."""
    from diffdock_b200.synthetic import default_model_args, make_pose_list
    from tests.parity_helpers import make_model_pair
    args = default_model_args(ns=48, nv=10, sh_lmax=2, num_conv_layers=6)
    _, p = make_model_pair(args, seed=3)
    poses = make_pose_list(2, n_res=1500, n_atoms=40, seed=4, tr_sigma_max=5.0)
    assert p.sync_free_crop_capable()
    return p, args, poses


@pytest.mark.parametrize('t', [1.0, 0.5, 0.05])
@pytest.mark.parametrize('crop', [False, True], ids=['plain', 'cropped'])
def test_diffdock_l_forward(cg_l, monkeypatch, t, crop):
    """Receptor pruning on (the default) in both runs; the cropped run sets ``g._crop`` as the captured sampler step does,
    which is the only way the device crop kernels run (the eager sampler crops on the host)."""
    p, args, poses = cg_l
    assert p._prune_receptor
    rec = Recorder(monkeypatch)
    _run(rec, p, _shared_batch(poses, t, args, 20.0 if crop else None))
    name = f"cg_l t={t} {'cropped' if crop else 'plain'}"
    out = replay(rec, name)
    L = len(p.conv_layers)
    assert _count(out, 'fused_conv') >= L * 2, out.keys()       # at least the two ligand groups in every layer
    assert _count(out, 'radius_count') >= 3 and _count(out, 'graph_fill') >= 2 and _count(out, 'graph_fill_reverse') >= 1
    assert _count(out, 'edge_embed') >= 1 and _count(out, 'receptor_need') == 1 and _count(out, 'crop_select_edges') >= 1
    assert _count(out, 'tpconv_finalize') >= L
    if crop:
        assert _count(out, 'crop_flags') == 1
    assert_clean(out, name)


def _small_args(**over):
    from diffdock_b200.synthetic import default_model_args
    kw = dict(ns=16, nv=4, sh_lmax=2, num_conv_layers=4, distance_embed_dim=16, cross_distance_embed_dim=16,
              sigma_embed_dim=16)
    kw.update(over)
    return default_model_args(**kw)


def _small_model(flag):
    if flag == 'reduce_pseudoscalars':
        from tests.test_reduce_pseudoscalars_gpu import l_pair
        a = _small_args(reduce_pseudoscalars=True, sh_lmax=1, smooth_edges=True, odd_parity=True,
                        differentiate_convolutions=False, num_prot_emb_layers=2)
        return l_pair(a, seed=7, lm=False)[1], a
    if flag == 'second_order':
        from tests.parity_helpers import make_model_pair
        a = _small_args(use_second_order_repr=True)
        return make_model_pair(a, seed=8, lm=False)[1], a
    from tests.test_tp_weights_layers_gpu import tw_pair
    a = _small_args(tp_weights_layers=3, embed_also_ligand=True)
    return tw_pair(a, seed=9)[1], a


@pytest.mark.parametrize('flag', ['reduce_pseudoscalars', 'second_order', 'tp_weights_layers'])
def test_small_flag_models(built_lib, monkeypatch, flag):
    """ns 16 / nv 4 models: the (16, 1) (4, 3) (4, 1) (4, 5) tile kinds, the second-order instantiation and a radial MLP
    with an extra hidden layer; plain and cropped."""
    from diffdock_b200.synthetic import make_pose_list
    p, a = _small_model(flag)
    poses = make_pose_list(3, n_res=300, n_atoms=25, seed=12, tr_sigma_max=4.0, lm_dim=0)
    for crop in (None, 15.0):
        rec = Recorder(monkeypatch)
        _run(rec, p, _shared_batch(poses, 0.4, a, crop))
        name = f"{flag} {'cropped' if crop else 'plain'}"
        out = replay(rec, name)
        kind = {'reduce_pseudoscalars': 'fused_conv', 'second_order': 'fused_conv_so',
                'tp_weights_layers': 'fused_conv_deep'}[flag]
        assert _count(out, kind) >= 2 * len(p.conv_layers), sorted(out)
        assert_clean(out, name)
        monkeypatch.undo()


def test_v10_score_model_swapped_launches(built_lib, monkeypatch):
    """CGOldModel in score mode: the lig_to_rec groups read the gathered node's scalars first (swap_gathered)."""
    from diffdock_b200.synthetic import make_pose_list
    from tests.old_score_helpers import model_pair, set_times
    from diffdock_b200.hetero import collate_shared_receptor
    _, p, _ = model_pair(seed=5, ns=16, nv=4, num_conv_layers=3, sigma_embed_dim=16, distance_embed_dim=16, lm_dim=0)
    poses = make_pose_list(2, n_res=250, n_atoms=20, seed=13, tr_sigma_max=4.0, lm_dim=0)
    for shared in (False, True):
        rec = Recorder(monkeypatch)
        from diffdock_b200.hetero import collate
        g = collate_shared_receptor([q.clone() for q in poses], DEV) if shared else collate([q.clone() for q in poses]).to(DEV)
        set_times(g, [0.3, 0.3] if shared else [0.3, 0.7], DEV)
        g._uniform_t = shared
        _run(rec, p, g)
        out = replay(rec, f"v1.0 score shared={shared}")
        assert _count(out, 'fused_conv_swap') >= len(p.lig_to_rec_conv_layers) - 1, sorted(out)
        assert_clean(out, f"v1.0 score shared={shared}")
        monkeypatch.undo()


def test_all_atom_score_model(built_lib, monkeypatch):
    """AAModel: nine edge groups per interaction layer."""
    from diffdock_b200.synthetic import make_pose_list
    from tests.test_tp_weights_layers_gpu import tw_pair
    from diffdock_b200.diffusion_utils import set_time
    from diffdock_b200.hetero import collate
    a = _small_args(num_conv_layers=3, tp_weights_layers=2, embed_also_ligand=True)
    p = tw_pair(a, seed=10, model='aa')[1]
    assert p.sync_free_capable()
    poses = make_pose_list(2, n_res=120, n_atoms=18, seed=14, tr_sigma_max=3.0, lm_dim=0, all_atoms=True)
    g = collate([q.clone() for q in poses]).to(DEV)
    set_time(g, None, 0.3, 0.3, 0.3, 2, True, DEV)
    rec = Recorder(monkeypatch)
    _run(rec, p, g)
    out = replay(rec, "aa score")
    assert _count(out, 'fused_conv') >= 9, sorted(out)
    assert_clean(out, "aa score")


def test_confidence_models(built_lib, monkeypatch):
    """CGModel(confidence_mode=True) at ns 48 / nv 10 with the atom head, and AAOldModel (v1.0 all-atom ranker)."""
    from diffdock_b200.synthetic import make_pose_list
    from tests.confidence_v10_fused_helpers import batch_of as v10_batch, pair as v10_pair
    from tests.confidence_v11_helpers import batch_of
    from tests.test_confidence_v11_gpu import _pair
    _, m = _pair('CGModel', 11)
    poses = make_pose_list(2, n_res=200, n_atoms=14, seed=5, tr_sigma_max=2.0, lm_dim=0)
    rec = Recorder(monkeypatch, conf_model=m)
    _run(rec, m, batch_of(poses, [0.0, 0.4], DEV))
    out = replay(rec, "confidence v1.1 CG")
    assert _count(out, 'confidence_head') == 1 and _count(out, 'fused_conv') >= 2 * len(m.conv_layers)
    assert_clean(out, "confidence v1.1 CG")
    monkeypatch.undo()
    _, m = v10_pair('AAOldModel', 11, lm_embedding_type='esm', lm_embedding_dim=32)
    poses = make_pose_list(2, n_res=120, n_atoms=14, seed=6, tr_sigma_max=2.0, lm_dim=32, all_atoms=True)
    rec = Recorder(monkeypatch, conf_model=m)
    _run(rec, m, v10_batch(poses, [0.2, 0.2], DEV, all_atoms=True, shared=True))
    out = replay(rec, "confidence v1.0 AA")
    assert _count(out, 'confidence_head') == 1 and _count(out, 'fused_conv') >= 3, sorted(out)
    assert_clean(out, "confidence v1.0 AA")


def test_sampler_steps(built_lib, monkeypatch):
    """sampling(rng='philox', cuda_graph=False) for 3 steps, and sample_packed eagerly for 2 steps over three complexes:
    the pose-update launches with in-kernel Philox noise, and the forwards of every step."""
    from diffdock_b200.diffusion_utils import get_t_schedule, t_to_sigma
    from diffdock_b200.sampling import sample_packed, sampling
    from diffdock_b200.synthetic import make_pose_list
    from tests.parity_helpers import make_model_pair
    from tests.test_packed_gpu import _complexes
    a = _small_args(num_conv_layers=3)
    _, p = make_model_pair(a, seed=15)
    poses = make_pose_list(3, n_res=150, n_atoms=22, seed=16, tr_sigma_max=a.tr_sigma_max)
    t2s = partial(t_to_sigma, args=a)
    sched = get_t_schedule('expbeta', 3)
    rec = Recorder(monkeypatch)
    rec.start()
    sampling([q.clone() for q in poses], p, 3, sched, sched, sched, DEV, t2s, a, batch_size=3, no_final_step_noise=True,
             rng='philox', seed=21, cuda_graph=False)
    rec.stop()
    out = replay(rec, "sampling philox 3 steps")
    assert _count(out, 'pose_update_dev') == 3 and _count(out, 'fused_conv') >= 3 * 2 * len(p.conv_layers)
    assert_clean(out, "sampling philox 3 steps")
    rec.start()
    sample_packed(_complexes(), p, 2, sched[:2], sched[:2], sched[:2], DEV, t2s, a, seed=11, complex_ids=[5, 9, 2],
                  no_final_step_noise=True, cuda_graph=False)
    rec.stop()
    out = replay(rec, "sample_packed 2 steps")
    assert _count(out, 'pose_update_packed') == 2, sorted(out)
    assert_clean(out, "sample_packed 2 steps")


# ---------------------------------------------------------------------------------------------------------------------
# mutations the replay must catch
def _failed(out, prefix):
    return [b for k, v in out.items() if k.startswith(prefix) for b in v[3]]


def test_mutation_mtab_of_one_interaction_layer(built_lib, monkeypatch):
    """One interaction layer's plan with the Clebsch-Gordan table of its widest l_out = 1 path scaled by 1 + 3e-4: the
    replay flags that layer's launches; whether the model-level 1e-4 check against the oracle notices is printed."""
    from diffdock_b200.synthetic import make_pose_list
    from diffdock_b200.tensor_layers import TensorProductConvLayer
    from oracle.diffusion import set_time as o_set_time
    from diffdock_b200.hetero import collate
    from tests.parity_helpers import make_model_pair
    a = _small_args(num_conv_layers=3)
    o, p = make_model_pair(a, seed=17, lm=False)
    layer = p.conv_layers[1]
    target = layer.fc[0] if isinstance(layer.fc, nn.ModuleList) else layer.fc
    orig, made = TensorProductConvLayer._fused_plan, {}

    def mutated(self, fc, table, k_in, swap_ns=0):
        plan = orig(self, fc, table, k_in, swap_ns)
        if fc is not target or plan is None:
            return plan
        if id(plan) not in made:
            m = copy.copy(plan)
            paths = sorted(table.paths, key=lambda q: (q.i_out, q.w_ref_off))
            l1 = [i for i, q in enumerate(paths) if q.l_out == 1]
            pi = max(l1, key=lambda i: paths[i].mul_in)
            m.mtab = plan.mtab.clone()
            m.mtab[pi] *= 1 + 3e-4
            made[id(plan)] = m
        return made[id(plan)]
    monkeypatch.setattr(TensorProductConvLayer, '_fused_plan', mutated)
    poses = make_pose_list(2, n_res=150, n_atoms=20, seed=18, tr_sigma_max=3.0, lm_dim=0)
    rec = Recorder(monkeypatch)
    got = _run(rec, p, _shared_batch(poses, 0.5, a))
    out = replay(rec, "mutation mtab")
    assert _failed(out, 'fused_conv'), "the replay missed a Clebsch-Gordan table scaled by 1 + 3e-4"
    g = collate([q.clone() for q in poses])
    o_set_time(g, 0.5, 0.5, 0.5, 2, 'cpu')
    with torch.no_grad():
        ref = o(g)
    errs = [rel_err(x, y) for x, y in zip(got[:3], ref[:3]) if y.numel()]
    print(f"\n[launch replay] mtab x (1 + 3e-4): replay flags {len(_failed(out, 'fused_conv'))} launches; model-level "
          f"max rel err {max(errs):.2e} {'notices' if max(errs) >= 1e-4 else 'misses'} it at 1e-4")


def test_mutation_v10_plan_without_the_swap(built_lib, monkeypatch):
    """The v1.0 lig_to_rec plans built with swap_ns = 0: the node blocks of W1 are in the kernel's order, not the model's."""
    from diffdock_b200.synthetic import make_pose_list
    from diffdock_b200.tensor_layers import TensorProductConvLayer
    from diffdock_b200.hetero import collate
    from tests.old_score_helpers import model_pair, set_times
    _, p, _ = model_pair(seed=19, ns=16, nv=4, num_conv_layers=3, sigma_embed_dim=16, distance_embed_dim=16, lm_dim=0)
    orig = TensorProductConvLayer._fused_plan
    monkeypatch.setattr(TensorProductConvLayer, '_fused_plan',
                        lambda self, fc, table, k_in, swap_ns=0: orig(self, fc, table, k_in, 0))
    poses = make_pose_list(2, n_res=150, n_atoms=20, seed=20, tr_sigma_max=3.0, lm_dim=0)
    g = collate([q.clone() for q in poses]).to(DEV)
    set_times(g, [0.3, 0.6], DEV)
    rec = Recorder(monkeypatch)
    _run(rec, p, g)
    out = replay(rec, "mutation swap_ns=0")
    assert _failed(out, 'fused_conv_swap'), "the replay missed lig_to_rec plans built without the swap"
    assert not _failed(out, 'tpconv') and not [b for k, v in out.items() if 'swap' not in k for b in v[3]
                                               if k.startswith('fused')], "only the swapped launches are wrong"


def test_mutation_confidence_head_tail_one_column_early(built_lib, monkeypatch):
    """The confidence head launched with tail_off one column before the last n_tail columns (the ns x0o block).  The
    pseudoscalars of a random model are small (with three layers the shift moved the pooled confidences by 4.6e-6 of their
    column maxima, with five layers and the per-atom head by 1.7e-5), hence the per-column tolerance of 5e-6."""
    from diffdock_b200.synthetic import make_pose_list
    from tests.confidence_v11_helpers import batch_of
    from tests.test_confidence_v11_gpu import _pair
    _, m = _pair('CGModel', 23, num_conv_layers=5)
    assert m._conf_tail > 0
    poses = make_pose_list(2, n_res=100, n_atoms=12, seed=7, tr_sigma_max=2.0, lm_dim=0)
    rec = Recorder(monkeypatch, conf_model=m)
    _run(rec, m, batch_of(poses, [0.1, 0.5], DEV))
    assert_clean(replay(rec, "confidence 5 layers"), "confidence 5 layers")       # the unmutated launch passes
    rec.call_mutation['ddb200_confidence_head'] = lambda a: a[:6] + (a[6] - 1,) + a[7:]
    _run(rec, m, batch_of(poses, [0.1, 0.5], DEV))
    out = replay(rec, "mutation tail_off - 1")
    assert _failed(out, 'confidence_head'), "the replay missed the head reading its tail one column early"

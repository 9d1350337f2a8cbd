"""GPU: the fully fused convolution (csrc/fused_conv.cu through diffdock_b200.fused.fused_conv) against the float64 reference
of tests/parity_helpers.py:fused_conv_reference, with the error taken per output irrep block (block_errors): a wrong 1o / 1e
block cannot hide behind the larger 0e scalars.

Edge counts are derived from the SM count: the kernel is persistent (grid = min(edge tiles, SMs), 64 edges per tile), and
only past one tile per SM does a CTA run a second tile - the path where the B ring has already requested the next tile's
W1' blocks and the mbarrier phases carry over from the previous tile.

Tolerance: 3e-5 of each block's max.  Two chained split-bf16 GEMMs feed an fp32 contraction; the largest per-block error
measured over these cases was 1.04e-5 (NVIDIA H100 80GB HBM3, 132 SMs, 700 W power limit).  Every case prints its largest
per-block error (run with -s to see them)."""
import copy

import pytest
import torch

from tests.parity_helpers import (block_errors, fused_conv_reference, fused_table, fused_weights, rel_err,
                                  KIND_GRID, SHAPE_GRID)

pytestmark = pytest.mark.gpu
TOL = 3e-5
OLD_TOL = 1e-4        # the tolerance of the older whole-output comparisons (max error / global max vs the fp32 oracle)

# edge counts as functions of the SM count
EDGE_COUNTS = {
    '1': lambda s: 1, '63': lambda s: 63, '64': lambda s: 64, '65': lambda s: 65,
    'sms*64-1': lambda s: s * 64 - 1, 'sms*64': lambda s: s * 64, 'sms*64+1': lambda s: s * 64 + 1,
    '3*sms*64+17': lambda s: 3 * s * 64 + 17,
}
MULTI = '3*sms*64+17'      # several edge tiles per CTA


def _edges(label):
    return EDGE_COUNTS[label](torch.cuda.get_device_properties(0).multi_processor_count)


def _padded(t, width, col0):
    """t [R, C] placed at columns col0 .. col0 + C of a NaN-filled [R, width] buffer: a view with row stride `width` whose
    base is col0 floats into the buffer (any read outside the view turns the result into NaN)."""
    buf = torch.full((t.shape[0], width), float('nan'), device=t.device)
    buf[:, col0:col0 + t.shape[1]] = t
    return buf[:, col0:col0 + t.shape[1]]


def _offset_contiguous(t):
    """A contiguous copy of t whose base pointer is 4 bytes past a 16-byte boundary."""
    store = torch.full((t.numel() + 4,), float('nan'), device=t.device)
    out = store[1:1 + t.numel()].view(t.shape)
    out.copy_(t)
    return out


class Case:
    """Random plan + inputs of one fused-convolution launch (weights and data drawn on the CPU from `seed`)."""

    def __init__(self, table, ne, ns, H, E, seed, n_nodes=300, n_out=None, rows=None, node_width=None):
        from diffdock_b200 import fused
        g = torch.Generator().manual_seed(seed)
        self.table, self.ne, self.ns, self.E = table, ne, ns, E
        self.n_out = n_out or n_nodes
        K1 = ne + 2 * ns
        assert fused.supported(table, H, K1)
        self.w = [t.cuda() for t in fused_weights(table, H, K1, g)]
        self.plan = fused.FusedPlan(table, *self.w)
        rows = rows or E
        r = lambda *s: torch.randn(*s, generator=g).cuda()
        self.x = r(n_nodes, table.d_in)
        self.node = self.x if node_width is None else r(n_nodes, node_width)
        self.tgt = torch.randint(0, self.n_out, (E,), generator=g).int().cuda()
        self.src = torch.randint(0, n_nodes, (E,), generator=g).int().cuda()
        self.ea, self.vec = r(rows, ne), r(rows, 3)
        self.kw = {}
        self.gen = g

    def run(self, plan=None, **over):
        a = dict(ea=self.ea, node=self.node, x=self.x, vec=self.vec, tgt=self.tgt, src=self.src)
        a.update(over)
        out = torch.zeros(self.n_out, self.table.d_out, device='cuda')
        cnt = torch.zeros(self.n_out, device='cuda')
        from diffdock_b200 import fused
        fused.fused_conv(plan or self.plan, a['ea'], a['node'], self.ns, a['tgt'], a['src'], a['x'], a['vec'], out, cnt,
                         **self.kw)
        torch.cuda.synchronize()
        return out, cnt

    def reference(self, n_live=None):
        n = self.E if n_live is None else n_live
        kw = {k: v for k, v in self.kw.items() if k not in ('n_edges_dev', 'edge_weight')}
        for k in ('edge_perm', 'ea_add_idx'):
            if k in kw:
                kw[k] = kw[k][:n]
        return fused_conv_reference(self.table, *self.w, self.ea, self.node, self.ns, self.tgt[:n], self.src[:n], self.x,
                                    self.vec, self.n_out, ew=self.kw.get('edge_weight'), **kw)


def _check(case, got, cnt, ref, rcnt, what):
    assert torch.equal(cnt.double(), rcnt), "edge counts differ from bincount"
    errs = block_errors(got, ref, case.table.out_irreps)
    worst = max(errs, key=errs.get)
    print(f"\n[fused fp64] {what}: max block err {errs[worst]:.2e} ({worst}), global {rel_err(got, ref):.2e}")
    assert errs[worst] < TOL, errs


@pytest.mark.parametrize("ns_nv,stage,lmax,faster", KIND_GRID)
def test_consumer_kinds_multi_tile(built_lib, ns_nv, stage, lmax, faster):
    """Every consumer kind, stage and spherical-harmonics variant at the production (ne, ns, H), several tiles per CTA."""
    ns, nv = ns_nv
    table = fused_table(ns, nv, stage, lmax, faster)
    c = Case(table, ns, ns, 3 * ns, _edges(MULTI), seed=100 + 10 * stage + lmax + 5 * faster + ns)
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f"kinds ns={ns} stage={stage} lmax={lmax} faster={faster}")


@pytest.mark.parametrize("edges", ['65', MULTI])
@pytest.mark.parametrize("ne,ns,H", SHAPE_GRID)
def test_radial_shapes(built_lib, ne, ns, H, edges):
    """(ne, ns, H): production shapes, the scalar A0 path (20, 5, 100), K1 > H, K1 < H, H < 64; node scalars gathered
    from a separate node tensor (the [ea | node[tgt] | node[src]] assembly against the independent reference)."""
    table = fused_table(48, 10, 3, 2, False)
    c = Case(table, ne, ns, H, _edges(edges), seed=ne + 3 * ns + H, node_width=max(ns, 1) + 3)
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f"shape ne={ne} ns={ns} H={H} E={c.E}")


@pytest.mark.parametrize("edges", list(EDGE_COUNTS))
def test_edge_counts(built_lib, edges):
    table = fused_table(48, 10, 3, 2, False)
    c = Case(table, 48, 48, 144, _edges(edges), seed=7, n_nodes=500)
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f"E={c.E}")


LAYOUTS = ['slices_ld_mult4', 'slices_ld_odd', 'node_separate', 'x_odd_ld', 'x_offset4', 'ea_offset4', 'node_offset4',
           'ea_add_offset4']


@pytest.mark.parametrize("layout", LAYOUTS)
def test_layouts(built_lib, layout):
    """Column slices of wider buffers (vector A0 path when every row start is 16-byte aligned, element path otherwise),
    x with an odd row stride or a 4-byte offset (element-wise node prefetch), misaligned attribute / node / ea_add bases."""
    table = fused_table(48, 10, 3, 2, False)
    ne = ns = 48
    c = Case(table, ne, ns, 144, _edges(MULTI), seed=40 + LAYOUTS.index(layout), node_width=ns)
    d_in = table.d_in
    over = {}
    if layout == 'slices_ld_mult4':
        over = dict(ea=_padded(c.ea, 56, 0), node=_padded(c.node, 60, 4))
    elif layout == 'slices_ld_odd':
        over = dict(ea=_padded(c.ea, 51, 0), node=_padded(c.node, 53, 2))
    elif layout == 'node_separate':
        pass                                          # node is a contiguous tensor of its own, x another
    elif layout == 'x_odd_ld':
        assert (d_in + 1) % 2 == 1
        over = dict(x=_padded(c.x, d_in + 1, 0))
    elif layout == 'x_offset4':
        over = dict(x=_padded(c.x, d_in + 2, 1))
    elif layout == 'ea_offset4':
        over = dict(ea=_padded(c.ea, 56, 1))
    elif layout == 'node_offset4':
        over = dict(node=_padded(c.node, 52, 1))
    elif layout == 'ea_add_offset4':
        add = torch.randn(5, ne, generator=c.gen).cuda()
        idx = torch.randint(0, 5, (c.E,), generator=c.gen).int().cuda()
        c.kw = dict(ea_add=_offset_contiguous(add), ea_add_idx=idx)
    got, cnt = c.run(**over)
    _check(c, got, cnt, *c.reference(), f"layout {layout}")


@pytest.mark.parametrize("what", ['perm', 'sign', 'add', 'weight', 'all_live'])
def test_indirections(built_lib, what):
    """edge_perm into a larger store, vec_sign = -1, ea_add, edge_weight; all of them together with a device-side live
    count below the capacity (rows past it hold indices of a real node, whose sum must not change)."""
    table = fused_table(48, 10, 3, 2, False)
    E = _edges(MULTI)
    rows = 2 * E if what in ('perm', 'all_live') else E
    c = Case(table, 48, 48, 144, E, seed=11 + len(what), rows=rows)
    g = c.gen
    kw = {}
    if what in ('perm', 'all_live'):
        kw['edge_perm'] = torch.randperm(rows, generator=g)[:E].int().cuda()
    if what in ('sign', 'all_live'):
        kw['vec_sign'] = -1.0
    if what in ('add', 'all_live'):
        kw['ea_add'] = torch.randn(7, 48, generator=g).cuda()
        kw['ea_add_idx'] = torch.randint(0, 7, (E,), generator=g).int().cuda()
    if what in ('weight', 'all_live'):
        kw['edge_weight'] = torch.rand(rows, generator=g).cuda()
    n_live = None
    if what == 'all_live':
        n_live = E - 2 * 64 - 5
        c.tgt[n_live:] = 0
        kw['n_edges_dev'] = torch.tensor([n_live], dtype=torch.int32, device='cuda')
    c.kw = kw
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(n_live), f"indirection {what}")


@pytest.mark.parametrize("what", ['sorted', 'one_target', 'out_nodes', 'zero_vec'])
def test_graphs(built_lib, what):
    """CSR-sorted targets (long runs reduced in the scatter stage), every edge on one node (atomics from every CTA),
    fewer output rows than nodes, a zero-length edge vector (Y = [1, 0, ...] as the oracle's normalize gives)."""
    table = fused_table(48, 10, 2, 2, False)
    E = _edges(MULTI)
    c = Case(table, 48, 48, 144, E, seed=21 + len(what), n_out=17 if what == 'out_nodes' else None)
    if what == 'sorted':
        c.tgt = torch.sort(c.tgt).values.contiguous()
    elif what == 'one_target':
        c.tgt.fill_(5)
    elif what == 'zero_vec':
        c.vec[E // 2] = 0.0
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f"graph {what}")


def _image_cols(img):
    """Swizzled plan image [T, n_kb, 256, 8, 8] <-> row-major [T, 256, n_kb * 64] (the 128B swizzle is an involution)."""
    T, n_kb, R = img.shape[:3]
    xor = torch.arange(8, device=img.device)[None, :] ^ (torch.arange(R, device=img.device) % 8)[:, None]
    lin = torch.gather(img, 3, xor[None, None, :, :, None].expand(T, n_kb, R, 8, 8))
    return lin.permute(0, 2, 1, 3, 4).reshape(T, R, n_kb * 64)


def _to_image(lin, like):
    T, n_kb, R = like.shape[:3]
    img = lin.reshape(T, R, n_kb, 8, 8).permute(0, 2, 1, 3, 4).contiguous()
    xor = torch.arange(8, device=img.device)[None, :] ^ (torch.arange(R, device=img.device) % 8)[:, None]
    return torch.gather(img, 3, xor[None, None, :, :, None].expand(T, n_kb, R, 8, 8)).contiguous()


@pytest.mark.parametrize("mutation", ['w2_lo_half', 'mtab_l1_path', 'w1_hidden_bias'])
def test_mutations_are_caught(built_lib, mutation):
    """The comparison is sharp enough to see subtle plan errors.  Only numeric plan data is perturbed (never the tile table
    or an index), so the mutated launch computes a wrong answer and nothing else.  The per-block metric must fail; the
    global metric (max error / global max) is printed beside it, judged at the older 1e-4 tolerance."""
    table = fused_table(48, 10, 1, 2, False)
    c = Case(table, 48, 48, 144, _edges(MULTI), seed=31)
    ref, rcnt = c.reference()
    got, _ = c.run()
    assert max(block_errors(got, ref, table.out_irreps).values()) < TOL      # the unmutated plan passes
    plan = copy.copy(c.plan)
    paths = sorted(table.paths, key=lambda p: (p.i_out, p.w_ref_off))
    l1 = [i for i, p in enumerate(paths) if p.l_out == 1]
    tiles = c.plan.tiles.tolist()
    Hp = (c.plan.hidden + 15) // 16 * 16
    K1p = (c.plan.k1 + 15) // 16 * 16
    if mutation == 'w2_lo_half':          # lo part of one tile into an l_out = 1 block: W2 at bf16 precision there
        t = next(i for i, ti in enumerate(tiles) if ti[7] in l1)
        lin = _image_cols(c.plan.w2_images).clone()
        lin[t, :, Hp:2 * Hp] = 0
        plan.w2_images = _to_image(lin, c.plan.w2_images)
    elif mutation == 'mtab_l1_path':      # Clebsch-Gordan entries of the widest path into an l_out = 1 block * (1 + 3e-4)
        pi = max(l1, key=lambda i: paths[i].mul_in)
        plan.mtab = c.plan.mtab.clone()
        plan.mtab[pi] *= 1 + 3e-4
    else:                                 # one hidden unit's folded bias (hi part) moved by 5e-3
        lin = _image_cols(c.plan.w1_images).clone()
        h = int(torch.argmax(c.w[1]))
        lin[0, h, 2 * K1p] = (lin[0, h, 2 * K1p].float() + 5e-3).to(lin.dtype)
        plan.w1_images = _to_image(lin, c.plan.w1_images)
    got, cnt = c.run(plan=plan)
    assert torch.equal(cnt.double(), rcnt)
    errs = block_errors(got, ref, table.out_irreps)
    glob = rel_err(got, ref)
    worst = max(errs, key=errs.get)
    print(f"\n[fused fp64] mutation {mutation}: max block err {errs[worst]:.2e} ({worst}), global {glob:.2e} "
          f"(global metric at {OLD_TOL:g} {'misses' if glob < OLD_TOL else 'catches'} it)")
    assert errs[worst] >= TOL, errs

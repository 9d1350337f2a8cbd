"""GPU: the neighbour-search kernels (csrc/graph.cu: radius_kernel behind ddb200_radius_count / ddb200_radius_fill,
graph_fill_kernel behind ddb200_graph_fill) edge for edge against oracle.graph_ops.radius on the CPU, and the edge-embedding
kernel (edge_embed_kernel) against a float64 restatement of the MLP.

The oracle uses the kernels' arithmetic (float32, d^2 = (dx^2 + dy^2) + dz^2, strict <, a per-graph cut-off c applied as
x / c, y / c with r = 1), so every (row, col) list must match it exactly and every edge vector bit for bit.  Each kernel is
compared with the oracle on its own, not with another kernel of the same file.  Cases: empty segments and segment lengths on
both sides of the 32-candidate chunk, caps that bind inside a chunk, the ligand graph's cap 33 with the self hit inside and
outside the first 33 hits, pairs one ulp either side of the cut-off, static edges listed first, index offsets, the reverse
pass and its permutation, and the score model's cross graph when one ligand atom has more than 10,000 residues in range.

Edge embedding: every shape of ops.EDGE_EMBED_SHAPES over a capacity of 300,001 edges, past the grid's 8 CTAs x 128 threads
per SM, so the grid-stride loop runs; device live counts 0, 1, cap - 1, cap, above cap (clamped) and negative (none); rows
past the live count keep their NaN fill.  The error is max |out - ref| / max |ref| per shape (fp32 FMA chains over up to 64
Gaussians and 48 hidden units).  Largest measured on an NVIDIA H100 80GB HBM3 (400 W power limit): 5.17e-7 (D = 64,
ns = 24) -> EMBED_TOL 1.5e-6."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from diffdock_b200.ops import EDGE_EMBED_SHAPES

pytestmark = pytest.mark.gpu
EMBED_TOL = 1.5e-6
EINVAL = -1


def _seg(sizes, dev='cuda'):
    return torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes, dtype=torch.long)).to(dev)


def _oracle(x, y, bx, by, r, rpg, cap, exclude_self=False):
    """(row = y index, col = x index) of oracle.graph_ops.radius on the CPU, sorted by (row, col); self pairs dropped after
    the cap, as radius_graph does."""
    from oracle.graph_ops import radius
    x, y, bx, by = x.cpu(), y.cpu(), bx.cpu(), by.cpu()
    if rpg is not None:
        rpg = rpg.cpu()
        x, y, r = x / rpg[bx][:, None], y / rpg[by][:, None], 1.0
    row, col = radius(x, y, r, bx, by, max_num_neighbors=cap)
    if exclude_self:
        keep = row != col
        row, col = row[keep], col[keep]
    return row, col


def _kernels(x, y, bx, by, r, rpg, cap, exclude_self=False, **fill_kw):
    """The three kernels' lists: count, (row, col) of ops.radius (count + fill) and (row, col, vec) of graph_fill."""
    from diffdock_b200 import ops
    B = int(max(bx.max() if bx.numel() else 0, by.max() if by.numel() else 0)) + 1
    x_ptr, by32 = ops.segment_ptr(bx, B), by.int().contiguous()
    cnt = ops.radius_count(x, y, x_ptr, by32, r=r, r_per_graph=rpg, max_num_neighbors=cap, exclude_self=exclude_self)
    row, col, _ = ops.radius(x, y, x_ptr, by, r=r, r_per_graph=rpg, max_num_neighbors=cap, exclude_self=exclude_self)
    incl = torch.cumsum(cnt, 0, dtype=torch.int32)
    E = int(incl[-1]) if cnt.numel() else 0
    g = ops.graph_fill(x, y, x_ptr, by32, (incl - cnt).contiguous(), E + 7, r=r, r_per_graph=rpg, max_num_neighbors=cap,
                       exclude_self=exclude_self, fill_row=-5, **fill_kw)
    return cnt, row, col, g, E, x_ptr


def _check_all(x, y, bx, by, r, rpg, cap, exclude_self=False):
    ref_row, ref_col = _oracle(x, y, bx, by, r, rpg, cap, exclude_self)
    cnt, row, col, (frow, fcol, fvec, _, _), E, _ = _kernels(x, y, bx, by, r, rpg, cap, exclude_self)
    assert torch.equal(cnt.cpu().long(), torch.bincount(ref_row, minlength=y.shape[0])), "radius_count"
    assert torch.equal(row.cpu().long(), ref_row) and torch.equal(col.cpu().long(), ref_col), "radius_fill"
    assert E == ref_row.shape[0]
    assert torch.equal(frow[:E].cpu().long(), ref_row) and torch.equal(fcol[:E].cpu().long(), ref_col), "graph_fill"
    assert bool((frow[E:] == -5).all()), "graph_fill wrote past the live count"
    assert torch.equal(fvec[:E].cpu(), x.cpu()[ref_col] - y.cpu()[ref_row]), "edge vectors"
    return E


SEG_X = [0, 1, 31, 32, 33, 64, 65, 3001, 5, 40]
SEG_Y = [4, 0, 3, 31, 33, 32, 65, 64, 0, 1]


@pytest.mark.parametrize("per_graph", [False, True])
def test_radius_segments_match_oracle(built_lib, per_graph):
    g = torch.Generator().manual_seed(11)
    bx, by = _seg(SEG_X), _seg(SEG_Y)
    x = (torch.rand(sum(SEG_X), 3, generator=g) * 30).cuda()
    y = (torch.rand(sum(SEG_Y), 3, generator=g) * 30).cuda()
    rpg = torch.linspace(6.0, 13.0, len(SEG_X)).cuda() if per_graph else None
    E = _check_all(x, y, bx, by, 1.0 if per_graph else 9.5, rpg, 10000)
    assert E > 1000


@pytest.mark.parametrize("cap", [5, 33, 40])
def test_radius_cap_binds_inside_a_chunk(built_lib, cap):
    """Dense segments: every query has more hits than the cap, and the cap falls in the middle of a 32-candidate chunk."""
    g = torch.Generator().manual_seed(cap)
    sizes_x, sizes_y = [70, 0, 100], [9, 3, 12]
    x = (torch.rand(sum(sizes_x), 3, generator=g) * 4).cuda()
    y = (torch.rand(sum(sizes_y), 3, generator=g) * 4).cuda()
    bx, by = _seg(sizes_x), _seg(sizes_y)
    _check_all(x, y, bx, by, 5.0, None, cap)
    cnt = _kernels(x, y, bx, by, 5.0, None, cap)[0]
    assert int(cnt.max()) == cap


def test_ligand_graph_cap_33_with_self_inside_and_outside(built_lib):
    """radius_graph semantics (cap 33, self excluded after the cap): in a segment where every atom is in range of every
    other, atom q < 33 has itself among its first 33 hits (32 edges kept), atom q >= 33 does not (33 edges kept)."""
    sizes = [50, 3, 40]
    g = torch.Generator().manual_seed(5)
    x = (torch.rand(sum(sizes), 3, generator=g) * 2).cuda()
    b = _seg(sizes)
    _check_all(x, x, b, b, 5.0, None, 33, exclude_self=True)
    cnt = _kernels(x, x, b, b, 5.0, None, 33, exclude_self=True)[0].cpu()
    assert cnt[:33].eq(32).all() and cnt[33:50].eq(33).all() and cnt[50:53].eq(2).all()


def _boundary_points(q, c, r):
    """Points p whose squared distance to q, computed as the kernels compute it (float32, both scaled by the cut-off c),
    is one ulp below, equal to and one ulp above r^2: candidates walk one ulp at a time along +x of the scaled query, with a
    small y step, as tests/test_crop_gpu.py builds its boundary residues; each is mapped back by c and judged by what the
    kernels' division gives back."""
    f = np.float32
    c, r2 = f(c), f(f(r) * f(r))
    qs = [f(f(v) / c) for v in q]
    want = {np.nextafter(r2, f(0)): None, r2: None, np.nextafter(r2, f(np.inf)): None}
    for k in range(64):
        py = f(qs[1] + f(k) * f(2 ** -9))
        dy = float(f(py - qs[1]))
        px = f(qs[0] + f(np.sqrt(max(float(r2) - dy * dy, 0.0))))
        for _ in range(24):
            px = np.nextafter(px, f(-np.inf))
        for _ in range(49):
            p = [f(px * c), f(py * c), f(qs[2] * c)]
            d = [f(f(v / c) - w) for v, w in zip(p, qs)]
            d2 = f(f(f(d[0] * d[0]) + f(d[1] * d[1])) + f(d[2] * d[2]))
            if d2 in want and want[d2] is None:
                want[d2] = p
            px = np.nextafter(px, f(np.inf))
        if all(v is not None for v in want.values()):
            break
    assert all(v is not None for v in want.values()), "no float32 positions at the cut-off found"
    return [list(map(float, v)) for v in want.values()]


@pytest.mark.parametrize("per_graph", [False, True])
def test_radius_pairs_at_the_cutoff(built_lib, per_graph):
    """Pairs whose d^2 is one ulp below, equal to and one ulp above r^2: only the first is an edge.  With a per-graph
    cut-off c = 3 sigma + 20 the search runs on x / c, y / c with r = 1, so the points are built in that scaled frame and
    mapped back by c."""
    f = np.float32
    q = [1.25, -3.5, 2.0]
    cs = [f(3 * 1.7 + 20), f(3 * 0.4 + 20)] if per_graph else [f(1), f(1)]
    r = 1.0 if per_graph else float(f(7.3))
    xs = _boundary_points(q, cs[0], r) + _boundary_points(q, cs[1], r)
    x, y = torch.tensor(xs).cuda(), torch.tensor([q, q]).cuda()
    rpg = torch.tensor(cs).cuda() if per_graph else None
    bx, by = _seg([3, 3]), _seg([1, 1])
    _check_all(x, y, bx, by, float(r), rpg, 10000)
    _, row, col, _, E, _ = _kernels(x, y, bx, by, float(r), rpg, 10000)
    assert E == 2 and col.tolist() == [0, 3], (row.tolist(), col.tolist())


def test_graph_fill_static_edges_and_offsets(built_lib):
    """Static (bond) edges listed first for each query with out_eid, then the radius hits; row / col offsets added."""
    from diffdock_b200 import ops
    sizes = [45, 0, 70]
    g = torch.Generator().manual_seed(21)
    x = (torch.rand(sum(sizes), 3, generator=g) * 6).cuda()
    b = _seg(sizes)
    n = x.shape[0]
    pre_cnt = torch.randint(0, 5, (n,), generator=g)
    seg_of = b.cpu()
    lo = torch.tensor([0, 45, 45])[seg_of]
    hi = torch.tensor([45, 45, 115])[seg_of]
    pre_col = torch.cat([torch.randint(int(lo[i]), int(hi[i]), (int(pre_cnt[i]),), generator=g) for i in range(n)]).int()
    pre_ptr = torch.zeros(n + 1, dtype=torch.int32)
    pre_ptr[1:] = torch.cumsum(pre_cnt, 0)
    ref_row, ref_col = _oracle(x, x, b, b, 4.0, None, 33, exclude_self=True)
    s_row = torch.repeat_interleave(torch.arange(n), pre_cnt)
    rows = torch.cat([s_row, ref_row])
    cols = torch.cat([pre_col.long(), ref_col])
    eids = torch.cat([torch.arange(pre_col.shape[0]), torch.full((ref_row.shape[0],), -1)])
    order = torch.sort(rows, stable=True).indices
    x_ptr = ops.segment_ptr(b, len(sizes))
    cnt = ops.radius_count(x, x, x_ptr, b.int(), r=4.0, max_num_neighbors=33, exclude_self=True) + pre_cnt.int().cuda()
    incl = torch.cumsum(cnt, 0, dtype=torch.int32)
    E = int(incl[-1])
    assert E == rows.shape[0]
    row, col, vec, eid, _ = ops.graph_fill(x, x, x_ptr, b.int(), (incl - cnt).contiguous(), E + 3, r=4.0,
                                           max_num_neighbors=33, exclude_self=True, pre_ptr=pre_ptr.cuda(),
                                           pre_col=pre_col.cuda(), want_eid=True, row_offset=1000, col_offset=77,
                                           fill_row=-5)
    assert torch.equal(row[:E].cpu().long() - 1000, rows[order]) and torch.equal(col[:E].cpu().long() - 77, cols[order])
    assert torch.equal(eid[:E].cpu().long(), eids[order]) and bool((eid[E:] == -1).all())
    xc = x.cpu()
    assert torch.equal(vec[:E].cpu(), xc[cols[order]] - xc[rows[order]])


@pytest.mark.parametrize("per_graph", [False, True])
def test_reverse_pass_is_the_forward_list_flipped(built_lib, per_graph):
    """The reverse pass (queries and candidates swapped, no cap) with perm from the forward pass's slots: the rows are the
    oracle's forward pairs flipped and sorted by x, perm is the stable argsort of the forward column."""
    from diffdock_b200 import ops
    sizes_x, sizes_y = [0, 33, 300, 65], [5, 0, 40, 31]
    g = torch.Generator().manual_seed(31)
    x = (torch.rand(sum(sizes_x), 3, generator=g) * 25).cuda()
    y = (torch.rand(sum(sizes_y), 3, generator=g) * 25).cuda()
    bx, by = _seg(sizes_x), _seg(sizes_y)
    rpg = torch.tensor([5.0, 9.0, 11.0, 30.0]).cuda() if per_graph else None
    r = 1.0 if per_graph else 10.0
    ref_row, ref_col = _oracle(x, y, bx, by, r, rpg, 10000)
    slot = torch.full((y.shape[0], max(sizes_x)), -1, dtype=torch.int32, device='cuda')
    _, _, _, (frow, fcol, _, _, _), E, x_ptr = _kernels(x, y, bx, by, r, rpg, 10000, slot_out=slot, slot_ld=slot.shape[1])
    assert torch.equal(frow[:E].cpu().long(), ref_row) and torch.equal(fcol[:E].cpu().long(), ref_col)
    y_ptr = ops.segment_ptr(by, len(sizes_y))
    cr = ops.radius_count(y, x, y_ptr, bx.int(), r=r, r_per_graph=rpg, max_num_neighbors=1 << 30)
    incr = torch.cumsum(cr, 0, dtype=torch.int32)
    assert int(incr[-1]) == E
    rrow, rcol, _, _, perm = ops.graph_fill(y, x, y_ptr, bx.int(), (incr - cr).contiguous(), E + 4, r=r, r_per_graph=rpg,
                                            max_num_neighbors=1 << 30, want_vec=False, slot_in=slot, y_ptr=x_ptr,
                                            slot_ld=slot.shape[1], want_perm=True, row_offset=500, fill_row=-5)
    order = torch.sort(ref_col, stable=True).indices
    assert torch.equal(rrow[:E].cpu().long() - 500, ref_col[order]) and torch.equal(rcol[:E].cpu().long(), ref_row[order])
    assert torch.equal(perm[:E].cpu().long(), order)


def _stub_model():
    """What CGModel._cross_graph_sync_free reads from the model besides its arguments: no smooth edge weight, and an edge
    embedding this test does not need."""
    return types.SimpleNamespace(smooth_edges=False, _edge_embed_in_kernel=lambda mlp, gs: True,
                                 _cross_edge_embedding=lambda *a: None)


@pytest.mark.parametrize("n_res", [300, 10050])
def test_model_cross_graph_reverse_when_the_cap_binds(built_lib, n_res):
    """The score model's sync-free cross graph (CGModel._cross_graph_sync_free) against the oracle's forward pairs
    (radius with max_num_neighbors=10000, models/cg_model.py:546) and their flip.  With 10,050 residues inside the cut-off
    of ligand atom 0 the forward cap binds: the reverse list must still hold exactly the forward pairs."""
    from diffdock_b200 import ops
    from diffdock_b200.cg_model import CGModel
    g = torch.Generator().manual_seed(n_res)
    n_lig = [3, 4]
    lig = torch.cat([torch.zeros(1, 3), torch.rand(2, 3, generator=g) * 40 + 20, torch.rand(4, 3, generator=g) * 10])
    rec = torch.cat([torch.rand(n_res, 3, generator=g) * 8 - 4, torch.rand(200, 3, generator=g) * 20])
    n_rec = [n_res, 200]
    lig, rec = lig.cuda(), rec.cuda()
    lb, rb = _seg(n_lig), _seg(n_rec)
    rpg = torch.tensor([15.0, 12.0]).cuda()
    ref_row, ref_col = _oracle(rec, lig, rb, lb, 1.0, rpg, 10000)
    if n_res > 10000:
        assert int((ref_row == 0).sum()) == 10000 and bool((torch.cdist(lig[:1], rec[:n_res]) < 15.0).all())
    col_off = sum(n_lig)
    c = {'lig_batch32': lb.int(), 'lig_ptr': ops.segment_ptr(lb, 2)}
    data = {'ligand': types.SimpleNamespace(pos=lig, node_sigma_emb=None, batch=lb)}
    rec_ptr = ops.segment_ptr(rb, 2)
    cap = sum(a * b for a, b in zip(n_lig, n_rec))
    fwd, rev = CGModel._cross_graph_sync_free(_stub_model(), data, c, rec, rec_ptr, rb.int(), max(n_rec), cap, 1.0, rpg,
                                              col_off, None, None, -1.0)
    f_tgt, f_src, _, vec, _, fkw = fwd
    b_tgt, b_src, _, _, _, rkw = rev
    E = int(fkw['n_edges_dev'][0])
    assert E == ref_row.shape[0] and rkw['n_edges_dev'] is fkw['n_edges_dev']
    assert torch.equal(f_tgt[:E].cpu().long(), ref_row) and torch.equal(f_src[:E].cpu().long() - col_off, ref_col)
    assert torch.equal(vec[:E].cpu(), rec.cpu()[ref_col] - lig.cpu()[ref_row])
    order = torch.sort(ref_col, stable=True).indices
    assert torch.equal(b_tgt[:E].cpu().long() - col_off, ref_col[order]), "reverse targets"
    assert torch.equal(b_src[:E].cpu().long(), ref_row[order]), "reverse sources"
    assert torch.equal(rkw['edge_perm'][:E].cpu().long(), order), "reverse permutation"


# ---- edge embedding ------------------------------------------------------------------------------------------------------
EMBED_CAP = 300_001


def _embed_case(D, ns, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    n_nodes = 97
    mu = torch.linspace(0.0, 30.0, D, device='cuda')
    coeff = float(-0.5 / (mu[1] - mu[0]) ** 2)
    vec = torch.randn(EMBED_CAP, 3, device='cuda', generator=g) * 12
    vec[:4] = torch.tensor([[0.0, 0.0, 0.0], [30.0, 0.0, 0.0], [0.0, -30.000002, 0.0], [0.0, 0.0, 95.0]], device='cuda')
    row = torch.randint(0, n_nodes, (EMBED_CAP,), device='cuda', generator=g).int()
    u = torch.randn(n_nodes, ns, device='cuda', generator=g)
    w1 = torch.randn(ns, D, device='cuda', generator=g) / D ** 0.5
    w2 = torch.randn(ns, ns, device='cuda', generator=g) / ns ** 0.5
    b2 = torch.randn(ns, device='cuda', generator=g)
    return vec, row, u, w1, w2, b2, mu, coeff


def _embed_ref(vec, row, u, w1, w2, b2, mu, coeff):
    d = vec.double().norm(dim=-1, keepdim=True)
    rbf = torch.exp(coeff * (d - mu.double()[None]) ** 2)
    h = torch.relu(u.double()[row.long()] + rbf @ w1.double().t())
    return h @ w2.double().t() + b2.double()


@pytest.mark.parametrize("D,ns", sorted(EDGE_EMBED_SHAPES))
def test_edge_embed_matches_fp64_over_the_grid_stride_loop(built_lib, D, ns):
    from diffdock_b200 import ops
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert EMBED_CAP > sms * 8 * 128 and EMBED_CAP % 128
    vec, row, u, w1, w2, b2, mu, coeff = _embed_case(D, ns, 100 * D + ns)
    ref = _embed_ref(vec, row, u, w1, w2, b2, mu, coeff)
    scale = float(ref.abs().max())
    worst = 0.0
    for live in (0, 1, EMBED_CAP - 1, EMBED_CAP, EMBED_CAP + 77, -3):
        out = torch.full((EMBED_CAP, ns), float('nan'), device='cuda')
        ops.edge_embed(vec, row, u, w1, w2, b2, mu, coeff, torch.tensor([live], dtype=torch.int32, device='cuda'), out=out)
        n = min(max(live, 0), EMBED_CAP)
        if n:
            err = float((out[:n].double() - ref[:n]).abs().max()) / scale
            worst = max(worst, err)
            assert err < EMBED_TOL, (live, err)
        assert bool(torch.isnan(out[n:]).all()), f"live count {live}: rows past it were written"
    print(f"edge_embed D={D} ns={ns}: max err {worst:.3e} (relative to max |ref| {scale:.3g})")


def test_edge_embed_rejects_shapes_outside_the_table(built_lib):
    from diffdock_b200 import _lib
    vec, row, u, w1, w2, b2, mu, coeff = _embed_case(64, 48, 0)
    out = torch.full((EMBED_CAP, 48), float('nan'), device='cuda')
    p = lambda t: C.c_void_p(t.data_ptr())
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for D, ns in ((48, 16), (64, 40), (128, 48), (64, 8)):
        rc = _lib.lib().ddb200_edge_embed(p(vec), p(row), p(u), p(w1), p(w2), p(b2), D, ns, p(mu), coeff, EMBED_CAP,
                                          None, p(out), stream)
        assert rc == EINVAL, (D, ns, rc)
    torch.cuda.synchronize()
    assert bool(torch.isnan(out).all())

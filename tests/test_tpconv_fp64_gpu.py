"""GPU: the streaming tensor-product convolution (csrc/tpconv.cu: tpconv_accumulate_kernel, tpconv_finalize_kernel) against
the float64 reference of tests/parity_helpers.py:tp_scatter_reference, with the error taken per output irrep block
(block_errors), so a wrong 1o / 1e block cannot hide behind larger scalars.

The kernel is called directly (ops.TpHandle / ops.tpconv_accumulate) for every table of parity_helpers.tp_table_grid.
It is persistent: one warp owns a unit of 32 edges, the grid has at most one CTA per SM, and only past
SMs x warps x 32 edges does a warp move on to a second unit - with its TMA weight ring and mbarrier phases carried over.
The edge counts are therefore derived from the SM count and from the warps per CTA that the handle planned
(DDB200_TPCONV_WARPS / DDB200_TPCONV_STAGES override the plan when the handle is created).

Every weight row comes from kernel_weights with a NaN fill and a row stride past weight_numel_padded, and x is a column
view of a NaN-filled wider buffer: a read of anything but a weight or an input feature shows up as NaN.

The layer cases at the end run the score model's head convolutions and the fallbacks of TensorProductConvLayer that route
to this kernel, against the oracle layer in float64, and assert through ops.PROFILE that no fused launch took part.

Tolerances are about 3x the largest per-block errors measured over these cases on an NVIDIA H100 80GB HBM3 (132 SMs,
700 W power limit):
  direct kernel cases   1.96e-6 (final, planner's 16 warps, 202,769 edges onto 64 rows)      -> TOL 6e-6
  layer cases           9.51e-6 (final_conv, 300 edges, radial MLP on split-bf16 wgmma)       -> LAYER_TOL 3e-5
  finalize              5.48e-8 (mean, BatchNorm and residual over the grid-stride loop)      -> FIN_TOL 1.6e-7
Every case prints its largest per-block and its global error (run with -s to see them)."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from tests.parity_helpers import (block_errors, kernel_weights, make_layer_pair, rel_err, table_sections,
                                  tp_scatter_reference, tp_table_grid)

pytestmark = pytest.mark.gpu
TOL = 6e-6            # direct kernel cases: fp32 FMA over exact fp32 inputs, per block
LAYER_TOL = 3e-5      # layer cases: the radial MLP's split-bf16 GEMMs feed the contraction
FIN_TOL = 1.6e-7      # the epilogue: a division, one FMA and one add in fp32
OLD_TOL = 2e-5        # the older whole-output comparison (max error / global max)
CHUNK = 8192


def _table(name):
    return tp_table_grid()[name]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _handle(table, monkeypatch, cfg):
    """A TpHandle planned with (warps, stages) = cfg, or the planner's choice for cfg None."""
    from diffdock_b200 import ops
    if cfg is not None:
        monkeypatch.setenv('DDB200_TPCONV_WARPS', str(cfg[0]))
        monkeypatch.setenv('DDB200_TPCONV_STAGES', str(cfg[1]))
    else:
        monkeypatch.delenv('DDB200_TPCONV_WARPS', raising=False)
        monkeypatch.delenv('DDB200_TPCONV_STAGES', raising=False)
    h = ops.TpHandle(table)
    if cfg is not None:
        assert (h.info(6), h.info(7)) == cfg, "the (warps, stages) override did not take effect"
    return h


def _padded(t, width, col0):
    """t [R, C] at columns col0 .. col0 + C of a NaN-filled [R, width] buffer (a strided column view)."""
    buf = torch.full((t.shape[0], width), float('nan'), device=t.device)
    buf[:, col0:col0 + t.shape[1]] = t
    return buf[:, col0:col0 + t.shape[1]]


def _targets(pattern, E, n_out, g):
    """(tgt int32 [E], n_out) for a destination pattern."""
    if pattern in ('random', 'n_out_gt'):
        return torch.randint(0, n_out, (E,), device='cuda', generator=g).int(), n_out + (41 if pattern == 'n_out_gt' else 0)
    if pattern == 'csr':
        return torch.sort(torch.randint(0, n_out, (E,), device='cuda', generator=g)).values.int(), n_out
    if pattern == 'poses':      # final_conv: B poses, each 20-80 consecutive edges onto its own row
        lens = torch.randint(20, 81, (E // 20 + 1,), device='cuda', generator=g)
        B = int((torch.cumsum(lens, 0) < E).sum()) + 1
        tgt = torch.repeat_interleave(torch.arange(B, device='cuda'), lens[:B])[:E]
        return tgt.int().contiguous(), B
    if pattern == 'own_row':
        return torch.randperm(E, device='cuda', generator=g).int(), E
    if pattern == 'one_row':
        return torch.full((E,), 3, dtype=torch.int32, device='cuda'), max(n_out, 4)
    raise ValueError(pattern)


class Case:
    """Random inputs of one accumulate launch, drawn on the GPU from `seed`."""

    def __init__(self, table, E, seed, pattern='random', n_nodes=257, ew=True, short_vecs=False):
        g = torch.Generator(device='cuda').manual_seed(seed)
        r = lambda *s: torch.randn(*s, device='cuda', generator=g)
        self.table, self.E = table, E
        self.x = _padded(r(n_nodes, table.d_in), table.d_in + 5, 2)
        self.src = torch.randint(0, n_nodes, (E,), device='cuda', generator=g).int()
        self.tgt, self.n_out = _targets(pattern, E, 64, g)
        self.geo = r(E, 3) if table.sh_lmax >= 0 else r(E, table.d_sh)
        if short_vecs:              # F.normalize semantics: x / max(|x|, 1e-12)
            assert table.sh_lmax >= 0 and E >= 3
            self.geo[E // 3] = 0.0
            self.geo[E // 2] = 1e-13 * self.geo[E // 2] / self.geo[E // 2].norm()
        self.w_ref = r(E, table.weight_numel)
        self.w = kernel_weights(table, self.w_ref, stride=table.weight_numel_padded + 8)
        self.ew = None
        if ew:
            self.ew = 2 * torch.rand(E, device='cuda', generator=g) - 1
            self.ew[::7] = 0.0
            if short_vecs:
                self.ew[E // 3] = self.ew[E // 2] = 1.0

    def run(self, h, sum_buf=None, cnt_buf=None, with_cnt=True, w=None, edges=None):
        from diffdock_b200 import ops
        s = sum_buf if sum_buf is not None else torch.zeros(self.n_out, self.table.d_out, device='cuda')
        c = cnt_buf if cnt_buf is not None else (torch.zeros(self.n_out, device='cuda') if with_cnt else None)
        sl = edges or slice(0, self.E)
        ops.tpconv_accumulate(h, self.x, self.src[sl], self.tgt[sl], self.geo[sl], (self.w if w is None else w)[sl], s, c,
                              edge_weight=self.ew[sl] if self.ew is not None else None)
        torch.cuda.synchronize()
        return s, c

    def reference(self):
        return tp_scatter_reference(self.table, self.x, self.src, self.tgt, self.geo, self.w_ref, self.n_out, ew=self.ew,
                                    chunk=CHUNK)


def _check(table, got, cnt, ref, rcnt, what, tol=TOL):
    if cnt is not None:
        assert torch.equal(cnt.double(), rcnt), "edge counts differ from bincount"
    assert torch.isfinite(got).all(), "NaN / inf in the output: a padding column or a column outside a view was read"
    errs = block_errors(got, ref, table.out_irreps)
    worst = max(errs, key=errs.get)
    print(f"\n[tpconv fp64] {what}: max block err {errs[worst]:.2e} ({worst}), global {rel_err(got, ref):.2e}")
    assert errs[worst] < tol, errs
    return errs[worst]


# ------------------------------------------------------------------------------------------------ every table
@pytest.mark.parametrize("name", sorted(tp_table_grid()))
def test_grid_tables(built_lib, monkeypatch, name):
    """Every table of the grid: 3 units + 1 edge, unsorted destinations, edge weights with zeros and negative values."""
    t = _table(name)
    h = _handle(t, monkeypatch, None)
    c = Case(t, 97, seed=sorted(tp_table_grid()).index(name))
    _check(t, *c.run(h), *c.reference(), f"table {name} (warps, stages) = ({h.info(6)}, {h.info(7)})")


# ------------------------------------------------------------------------------------------------ pipeline shape
EDGE_COUNTS = {'1': lambda n: 1, '31': lambda n: 31, '32': lambda n: 32, '33': lambda n: 33,
               'n-1': lambda n: n - 1, 'n+1': lambda n: n + 1, '3n+17': lambda n: 3 * n + 17}   # n = SMs * warps * 32
PIPELINE = [(cfg, name) for cfg in ((1, 2), (2, 3)) for name in ('final', 'tor')] + [(None, 'final')]


@pytest.mark.parametrize("edges", list(EDGE_COUNTS))
@pytest.mark.parametrize("cfg,name", PIPELINE)
def test_pipeline_and_edge_counts(built_lib, monkeypatch, cfg, name, edges):
    """(warps, stages) overrides and the planner's default; edge counts around one unit per warp of the whole grid, and
    three units or more per warp (the multi-unit loop, the producer moving to its next unit, ring phases carried over)."""
    t = _table(name)
    h = _handle(t, monkeypatch, cfg)
    warps, stages = h.info(6), h.info(7)
    n = _sms() * warps * 32
    E = EDGE_COUNTS[edges](n)
    c = Case(t, E, seed=len(edges) + 10 * warps + stages, pattern='random', n_nodes=1000)
    _check(t, *c.run(h), *c.reference(), f"{name} (warps, stages) = ({warps}, {stages}) E={E} (SMs*warps*32 = {n})")


# ------------------------------------------------------------------------------------------------ destinations
@pytest.mark.parametrize("pattern", ['random', 'csr', 'poses', 'own_row', 'one_row', 'n_out_gt'])
def test_destinations(built_lib, monkeypatch, pattern):
    """Runs of equal destinations that cross unit and warp boundaries, every edge on its own row, all edges on one row,
    and rows past the largest destination (they must stay exactly 0 in sum and cnt)."""
    t = _table('final')
    h = _handle(t, monkeypatch, (2, 3))
    E = 3 * _sms() * 2 * 32 + 17
    c = Case(t, E, seed=50 + len(pattern), pattern=pattern)
    got, cnt = c.run(h)
    _check(t, got, cnt, *c.reference(), f"destinations {pattern} E={E} n_out={c.n_out}")
    if pattern == 'n_out_gt':
        top = int(c.tgt.max()) + 1
        assert top < c.n_out and not got[top:].any() and not cnt[top:].any()


# ------------------------------------------------------------------------------------------------ views and inputs
@pytest.mark.parametrize("what", ['edge_weight', 'no_edge_weight', 'no_cnt', 'short_vectors', 'given_sh_no_ew'])
def test_inputs(built_lib, monkeypatch, what):
    """edge_weight given (zeros, negative values) or absent, cnt = None, a zero-length edge vector and one of length 1e-13
    (below the 1e-12 floor of the normalisation); x is always a NaN-padded column view, w NaN-padded past its width."""
    t = _table('tor' if what == 'given_sh_no_ew' else 'ladder_48_10_s3_l2')
    h = _handle(t, monkeypatch, (2, 3))
    E = _sms() * 2 * 32 + 1
    c = Case(t, E, seed=60 + len(what), ew=what not in ('no_edge_weight', 'given_sh_no_ew'),
             short_vecs=what == 'short_vectors')
    assert c.x.stride(0) > t.d_in and c.w.stride(0) > t.weight_numel_padded
    got, cnt = c.run(h, with_cnt=what != 'no_cnt')
    ref, rcnt = c.reference()
    _check(t, got, cnt, ref, rcnt, f"inputs {what}")
    if what == 'short_vectors':     # the two short edges alone, so their messages are not lost among the others
        for e in (E // 3, E // 2):
            one = slice(e, e + 1)
            g1, _ = c.run(h, edges=one)
            r1, _ = tp_scatter_reference(t, c.x, c.src[one], c.tgt[one], c.geo[one], c.w_ref[one], c.n_out, ew=c.ew[one])
            _check(t, g1, None, r1, None, f"single edge of length {float(c.geo[e].norm()):.0e}")


# ------------------------------------------------------------------------------------------------ additivity
@pytest.mark.parametrize("how", ['prefilled', 'two_launches'])
def test_accumulation_is_additive(built_lib, monkeypatch, how):
    """The kernel adds to sum and cnt: TensorProductConvLayer's edge blocks, several edge groups and accumulate_group
    rely on it."""
    t = _table('ladder_16_4_s2_l2')
    h = _handle(t, monkeypatch, (1, 2))
    E = 3 * _sms() * 32 + 17
    c = Case(t, E, seed=70 + len(how), pattern='csr')
    ref, rcnt = c.reference()
    if how == 'prefilled':
        g = torch.Generator(device='cuda').manual_seed(71)
        s0 = torch.randn(c.n_out, t.d_out, device='cuda', generator=g)
        c0 = torch.randint(0, 50, (c.n_out,), device='cuda', generator=g).float()
        got, cnt = c.run(h, sum_buf=s0.clone(), cnt_buf=c0.clone())
        ref, rcnt = ref + s0.double(), rcnt + c0.double()
    else:
        got, cnt = c.run(h, edges=slice(0, E // 2 + 5))
        got, cnt = c.run(h, sum_buf=got, cnt_buf=cnt, edges=slice(E // 2 + 5, E))
    _check(t, got, cnt, ref, rcnt, f"additive {how}")


# ------------------------------------------------------------------------------------------------ finalize
@pytest.mark.parametrize("what", ['mean_empty_rows', 'bn', 'residual', 'sum_only', 'grid_stride'])
def test_finalize(built_lib, what):
    """ops.tpconv_finalize against float64: mean over rows with cnt = 0, BatchNorm scale / shift, a residual narrower
    than the output from a strided view, the sum alone, and enough values for the grid-stride loop."""
    from diffdock_b200 import ops
    t = _table('ladder_48_10_s3_l2')
    d = t.d_out
    n = 4000 if what == 'grid_stride' else 300
    assert what != 'grid_stride' or n * d > 132 * 16 * 256
    g = torch.Generator(device='cuda').manual_seed(80 + len(what))
    s = torch.randn(n, d, device='cuda', generator=g)
    cnt = torch.randint(0, 9, (n,), device='cuda', generator=g).float()
    cnt[:7] = 0
    s[:7] = 0                     # rows without edges have nothing to average
    mean = what in ('mean_empty_rows', 'bn', 'residual', 'grid_stride')
    scale = shift = res = None
    if what in ('bn', 'grid_stride'):
        scale, shift = 1 + 0.2 * torch.randn(d, device='cuda', generator=g), 0.1 * torch.randn(d, device='cuda', generator=g)
    if what in ('residual', 'grid_stride'):
        res = _padded(torch.randn(n, 48 + 30, device='cuda', generator=g), 100, 3)
        assert res.shape[1] < d and res.stride(0) > res.shape[1]
    got = ops.tpconv_finalize(s, cnt, mean, scale, shift, res)
    torch.cuda.synchronize()
    ref = s.double()
    if mean:
        ref = ref / cnt.double().clamp_min(float(torch.finfo(torch.float32).eps))[:, None]
    if scale is not None:
        ref = ref * scale.double() + shift.double()
    if res is not None:
        ref[:, :res.shape[1]] += res.double()
    errs = block_errors(got, ref, t.out_irreps)
    worst = max(errs, key=errs.get)
    print(f"\n[tpconv fp64] finalize {what}: max block err {errs[worst]:.2e} ({worst})")
    assert errs[worst] < FIN_TOL, errs


# ------------------------------------------------------------------------------------------------ host validation
def test_host_validation(built_lib):
    """Documented return codes of the raw entry points for bad arguments.  Every buffer is large enough for what the
    arguments describe, and every call must be refused before a launch: the sum canary stays unchanged."""
    from diffdock_b200 import _lib, ops
    L = _lib.lib()
    t = _table('final')
    h = ops.TpHandle(t)
    E, n_out = 64, 8
    P = lambda x: C.c_void_p(x.data_ptr()) if x is not None else C.c_void_p(0)
    x = torch.randn(16, 2 * t.d_in, device='cuda')
    src = torch.zeros(E, dtype=torch.int32, device='cuda')
    dst = torch.zeros(E, dtype=torch.int32, device='cuda')
    geo = torch.randn(E, 3, device='cuda')
    Wp = t.weight_numel_padded
    wbuf = torch.randn(E * (Wp + 8) + 8, device='cuda')
    sum_buf = torch.full((n_out, t.d_out), 7.0, device='cuda')
    cnt = torch.full((n_out,), 5.0, device='cuda')
    canary = sum_buf.clone(), cnt.clone()

    def acc(w_ptr, w_stride, x_stride, n_edges=E):
        return L.ddb200_tpconv_accumulate(h._h, P(x), x_stride, P(src), P(dst), P(geo), None, C.c_void_p(w_ptr), w_stride,
                                          n_edges, P(sum_buf), P(cnt), None)

    base = wbuf.data_ptr()
    assert base % 16 == 0
    assert acc(base + 4, Wp, t.d_in) == -1                 # w 4 bytes off a 16-byte boundary
    assert acc(base, Wp + 2, t.d_in) == -1                 # w_stride % 4 != 0
    assert acc(base, Wp - 4, t.d_in) == -1                 # w_stride < weight_numel_padded
    assert acc(base, Wp, t.d_in - 1) == -1                 # x_stride < D_in
    assert acc(base, Wp, t.d_in, n_edges=0) == 0           # nothing to do
    torch.cuda.synchronize()
    assert torch.equal(sum_buf, canary[0]) and torch.equal(cnt, canary[1])

    ib = np.ascontiguousarray(t.iblob, dtype=np.int32)
    fb = np.ascontiguousarray(t.fblob, dtype=np.float32)
    out = C.c_void_p()
    bad = ib.copy()
    bad[0] ^= 1
    assert L.ddb200_tp_table_create(bad.ctypes.data_as(C.c_void_p), len(bad), fb.ctypes.data_as(C.c_void_p), len(fb),
                                    C.byref(out)) == -2                                     # wrong magic
    longer = np.concatenate([ib, np.zeros(4, np.int32)])
    assert L.ddb200_tp_table_create(longer.ctypes.data_as(C.c_void_p), len(longer), fb.ctypes.data_as(C.c_void_p),
                                    len(fb), C.byref(out)) == -2                            # n_ints != the blob's own
    assert not out.value

    scale = torch.ones(t.d_out, device='cuda')
    o = torch.full_like(sum_buf, 3.0)
    for sc, sh in ((scale, None), (None, scale)):
        assert L.ddb200_tpconv_finalize(P(sum_buf), P(cnt), n_out, t.d_out, 1, P(sc), P(sh), None, 0, 0, P(o), None) == -1
    torch.cuda.synchronize()
    assert bool((o == 3.0).all())


# ------------------------------------------------------------------------------------------------ mutations
def _mutate_term(table, l_out):
    """A copy of `table` with the largest Clebsch-Gordan term of its widest l_out path scaled by 1 + 3e-4."""
    paths, _, _, ment = table_sections(table)
    d = 2 * l_out + 1
    pa = max((p for p in paths if p[3] == d), key=lambda p: p[1])
    mo, n_m = pa[5], pa[2] * pa[3]
    terms = [q for mi, tb, tc in ment if mo <= mi < mo + n_m for q in range(tb, tb + tc)]
    q = max(terms, key=lambda q: abs(table.fblob[q]))
    t2 = copy.copy(table)
    t2.fblob = table.fblob.copy()
    t2.fblob[q] *= np.float32(1 + 3e-4)
    assert t2.fblob[q] != table.fblob[q]
    return t2


def _remainder_row_cols(table):
    """Kernel-layout columns of one remainder row (u >= (nrow // R) * R of a split piece) of a weight tile."""
    _, tiles, chunks, _ = table_sections(table)
    lprs = table.iblob[22:26]
    i = next(i for i, tl in enumerate(tiles) if tl[2] >> 16 > 0 and tl[12] > tl[8])
    tl = tiles[i]
    g_off = next(ch[2] for ch in chunks if ch[0] <= i < ch[1])
    u = (tl[12] // tl[8]) * tl[8]
    start = g_off + tl[0] + u * tl[4]
    return start, start + lprs[tl[7]] * tl[6]


@pytest.mark.parametrize("mutation", ['final_l1_term', 'second_order_l2_term', 'remainder_row'])
def test_mutations_are_caught(built_lib, monkeypatch, mutation):
    """The per-block comparison sees subtle table errors.  Only numeric data changes (Clebsch-Gordan terms, weight values),
    never an index or an offset.  The unmutated launch passes, the mutated one must fail; the global metric is printed
    beside it, judged at the older 2e-5 tolerance."""
    from diffdock_b200 import ops
    name = {'final_l1_term': 'final', 'second_order_l2_term': 'second_48_10', 'remainder_row': 'small_stages'}[mutation]
    t = _table(name)
    h = _handle(t, monkeypatch, (2, 3))
    c = Case(t, _sms() * 2 * 32 + 33, seed=90 + len(mutation))
    ref, rcnt = c.reference()
    _check(t, *c.run(h), ref, rcnt, f"unmutated {name}")
    w = None
    if mutation == 'final_l1_term':
        h = ops.TpHandle(_mutate_term(t, 1))
    elif mutation == 'second_order_l2_term':
        h = ops.TpHandle(_mutate_term(t, 2))
    else:
        a, b = _remainder_row_cols(t)
        assert (t.w_perm[a:b] >= 0).all()
        w = c.w.clone()
        w[:, a:b] = 0.0
    got, cnt = c.run(h, w=w)
    assert torch.equal(cnt.double(), rcnt)
    errs = block_errors(got, ref, t.out_irreps)
    glob = rel_err(got, ref)
    worst = max(errs, key=errs.get)
    print(f"\n[tpconv fp64] mutation {mutation}: max block err {errs[worst]:.2e} ({worst}), global {glob:.2e} "
          f"(global metric at {OLD_TOL:g} {'misses' if glob < OLD_TOL else 'catches'} it)")
    assert errs[worst] >= TOL, errs


# ------------------------------------------------------------------------------------------------ layers
def _layer_case(ins, shs, outs, n_feat, E, n_x, n_out, seed, given_sh=False, ew=None, sorted_tgt=False, **kw):
    """(product output, float64 oracle output) of one TensorProductConvLayer forward, with ops.PROFILE asserting that
    every convolution launch was the streaming kernel.  Returns (got, ref, accumulate launches)."""
    from diffdock_b200 import ops
    from oracle import e3nn_lite as o3
    o, p = make_layer_pair(ins, shs, outs, n_feat, seed=seed, **kw)
    o = o.double()
    g = torch.Generator().manual_seed(seed + 2)
    x = torch.randn(n_x, o3.Irreps(ins).dim, generator=g, dtype=torch.float64)
    tgt = torch.randint(0, n_out, (E,), generator=g)
    if sorted_tgt:
        tgt = torch.sort(tgt).values
    ei = torch.stack([tgt, torch.randint(0, n_x, (E,), generator=g)])
    vec = torch.randn(E, 3, generator=g, dtype=torch.float64)
    ea = torch.randn(E, n_feat, generator=g, dtype=torch.float64)
    if given_sh:
        sh = torch.randn(E, o3.Irreps(shs).dim, generator=g, dtype=torch.float64)
    else:
        sh = o3.spherical_harmonics(o3.Irreps(shs), vec, normalize=True, normalization='component')
    ew_o = ew(E, g) if callable(ew) else (1.0 if ew is None else ew)
    with torch.no_grad():
        ref = o(x, ei, ea, sh, out_nodes=n_out, reduce='mean', edge_weight=ew_o)
    p = p.cuda()
    f = lambda t: t.float().cuda() if torch.is_tensor(t) else t
    ops.PROFILE.reset(enabled=True)
    try:
        got = p(f(x), ei.cuda(), f(ea), f(sh), out_nodes=n_out, edge_weight=f(ew_o),
                edge_vec=None if given_sh else f(vec), assume_sorted=sorted_tgt)
        torch.cuda.synchronize()
        launches = len(ops.PROFILE.pairs)
        assert launches > 0 and ops.PROFILE.fused_pairs == [], "the layer did not run on the streaming kernel alone"
    finally:
        ops.PROFILE.reset(False)
    return got, ref, launches


def _check_layer(got, ref, outs, what):
    from diffdock_b200.irreps import parse_irreps
    assert torch.isfinite(got).all()
    errs = block_errors(got, ref, parse_irreps(outs))
    worst = max(errs, key=errs.get)
    print(f"\n[tpconv fp64] layer {what}: max block err {errs[worst]:.2e} ({worst}), global {rel_err(got, ref):.2e}")
    assert errs[worst] < LAYER_TOL, errs


SEQ = '48x0e + 10x1o + 10x1e + 48x0o'
SH1, SH2 = '1x0e + 1x1o', '1x0e + 1x1o + 1x2e'


@pytest.mark.parametrize("E", [300, 40])
@pytest.mark.parametrize("odd", [False, True])
def test_layer_final_conv(built_lib, E, odd):
    """The score model's final_conv: no residual, one output row per pose, edges sorted by pose; >= 64 edges go through
    the radial GEMM (weight rows padded to its column tiles), fewer through F.linear."""
    outs, shs = ('1x1o + 1x1e', SH1) if odd else ('2x1o + 2x1e', SH2)
    got, ref, _ = _layer_case(SEQ, shs, outs, 96, E, n_x=150, n_out=5, seed=100 + E + odd, sorted_tgt=True,
                              residual=False)
    _check_layer(got, ref, outs, f"final_conv odd={odd} E={E}")


@pytest.mark.parametrize("odd", [False, True])
def test_layer_tor_bond_conv(built_lib, odd):
    """tor_bond_conv: given spherical harmonics (FullTensorProduct(sh, 2e)), a per-edge weight tensor, reduce mean."""
    from diffdock_b200.irreps import irreps_str
    from diffdock_b200.tp_table import full_tensor_product
    shs = irreps_str(full_tensor_product(SH1 if odd else SH2, '1x2e')[1])
    outs = '48x0o' if odd else '48x0o + 48x0e'
    got, ref, _ = _layer_case(SEQ, shs, outs, 144, 500, n_x=120, n_out=30, seed=110 + odd, given_sh=True,
                              ew=lambda E, g: torch.rand(E, 1, generator=g, dtype=torch.float64), residual=False)
    _check_layer(got, ref, outs, f"tor_bond_conv odd={odd}")


@pytest.mark.parametrize("what", ['40_edges', 'scalar_edge_weight', 'second_order'])
def test_layer_fallbacks(built_lib, what):
    """Groups under 64 edges of a fused-kernel shape, a scalar edge_weight != 1, second-order representations."""
    from oracle.tensor_layers import get_irrep_seq
    if what == '40_edges':
        s = get_irrep_seq(16, 4, False, False)
        ins, outs, E, ew = s[2], s[3], 40, None
    elif what == 'scalar_edge_weight':
        ins, outs, E, ew = SEQ, SEQ, 400, 0.5
    else:
        s = get_irrep_seq(16, 4, True, False)
        ins, outs, E, ew = s[2], s[3], 400, None
    ns = 16 if what != 'scalar_edge_weight' else 48
    got, ref, _ = _layer_case(ins, SH2, outs, 3 * ns, E, n_x=60, n_out=60, seed=120 + len(what), ew=ew,
                              hidden_features=3 * ns)
    _check_layer(got, ref, outs, what)


def test_layer_weight_blocks(built_lib, monkeypatch):
    """Per-edge weights materialised in edge blocks: several accumulate launches into one buffer."""
    from diffdock_b200 import tensor_layers
    monkeypatch.setattr(tensor_layers, 'WEIGHT_BLOCK_BYTES', 1)      # -> the 1024-edge minimum block
    got, ref, launches = _layer_case(SEQ, SH2, SEQ, 144, 2500, n_x=200, n_out=200, seed=130, given_sh=True,
                                     hidden_features=144)
    assert launches == 3
    _check_layer(got, ref, SEQ, "weight blocks of 1024 edges")

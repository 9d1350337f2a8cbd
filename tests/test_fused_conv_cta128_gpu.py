"""GPU: the fused convolution at the edges of its 128-edge CTA tile, against the float64 reference of
tests/parity_helpers.py:fused_conv_reference (per output irrep block, 3e-5 as in test_fused_conv_fp64_gpu.py).

Each CTA tile holds 128 CSR-sorted edges, 64 per warpgroup, and both warpgroups read one stream of weight stages.  The
cases cover edge counts around one tile and around one tile per SM, a last tile whose second half is empty (from the
host count and from a device-side count), runs of equal targets that cross the boundary between the two halves or
between two tiles or cover a whole tile, and every consumer kind over several tiles per CTA."""
import pytest
import torch

from tests.parity_helpers import KIND_GRID, fused_table
from tests.test_fused_conv_fp64_gpu import Case, _check

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


EDGE_COUNTS = {
    '127': lambda s: 127, '128': lambda s: 128, '129': lambda s: 129,
    'sms*128-1': lambda s: s * 128 - 1, 'sms*128+1': lambda s: s * 128 + 1,
    'sms*128+64': lambda s: s * 128 + 64,              # the last tile's second half is empty
    '2*sms*128+64': lambda s: 2 * s * 128 + 64,
}


@pytest.mark.parametrize("edges", list(EDGE_COUNTS))
def test_cta_tile_edge_counts(built_lib, edges):
    table = fused_table(48, 10, 3, 2, False)
    c = Case(table, 48, 48, 144, EDGE_COUNTS[edges](_sms()), seed=3, n_nodes=500)
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f"E={c.E}")


def _runs(E, g):
    """CSR targets: a run over rows 50..139 (across the halves of tile 0 and into tile 1), one over exactly tile 2,
    one over tiles 3..4 and rows of tile 5, then random runs of 1..200 edges"""
    lengths = [50, 90, 116, 128, 300]
    while sum(lengths) < E:
        lengths.append(int(torch.randint(1, 201, (1,), generator=g)))
    tgt = torch.cat([torch.full((n,), i, dtype=torch.int32) for i, n in enumerate(lengths)])[:E]
    return tgt, len(lengths)


@pytest.mark.parametrize("edges", ['sms*128+64', '3*sms*128+17'])
def test_cta_tile_runs(built_lib, edges):
    sms = _sms()
    E = sms * 128 + 64 if edges == 'sms*128+64' else 3 * sms * 128 + 17
    g = torch.Generator().manual_seed(5)
    tgt, n_out = _runs(E, g)
    table = fused_table(48, 10, 3, 2, False)
    c = Case(table, 48, 48, 144, E, seed=9, n_nodes=max(500, n_out), n_out=n_out)     # node[tgt] feeds the radial MLP
    c.tgt = tgt.cuda()
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f"runs E={E}")


@pytest.mark.parametrize("n_live", ['half', 'half+1', 'half-1'])
def test_cta_tile_device_count(built_lib, n_live):
    """a device-side live count that ends the last tile in its first half (or one edge into / short of the second half);
    the rows past it hold a real target, whose sum must not change"""
    E = 3 * _sms() * 128
    n = E - 64 + {'half': 0, 'half+1': 1, 'half-1': -1}[n_live]
    table = fused_table(48, 10, 3, 2, False)
    c = Case(table, 48, 48, 144, E, seed=13, n_nodes=400)
    c.tgt = torch.sort(c.tgt).values.contiguous()
    c.tgt[n:] = 0
    c.kw = {'n_edges_dev': torch.tensor([n], dtype=torch.int32, device='cuda')}
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(n), f"device count {n} of {E}")


@pytest.mark.parametrize("ns_nv,stage,lmax,faster", KIND_GRID)
def test_cta_tile_kinds(built_lib, ns_nv, stage, lmax, faster):
    """every consumer kind with several 128-edge tiles per CTA and a last tile with an empty second half"""
    ns, nv = ns_nv
    table = fused_table(ns, nv, stage, lmax, faster)
    c = Case(table, ns, ns, 3 * ns, 2 * _sms() * 128 + 57, seed=200 + 10 * stage + lmax + 5 * faster + ns)
    c.tgt = torch.sort(c.tgt).values.contiguous()
    got, cnt = c.run()
    _check(c, got, cnt, *c.reference(), f"kinds ns={ns} stage={stage} lmax={lmax} faster={faster}")

"""Host logic of the fully fused convolution (diffdock_b200/fused.py): a numpy/torch emulation that reads ONLY the plan the
kernel reads (swizzled bf16 operand images with folded biases, tile table, dense Clebsch-Gordan tables) and forms the
products step by step like the kernel's MMA loop (16-column steps of the static operand paired with the activation image
through the step map) must reproduce the oracle layer.  Pins the image layout, the split-bf16 scheme, the step map and the
tile/accumulator bookkeeping without a GPU."""
import math

import pytest
import torch

from diffdock_b200 import fused
from diffdock_b200.tensor_layers import get_irrep_seq
from diffdock_b200.tp_table import build_table
from tests.parity_helpers import (KIND_GRID, SHAPE_GRID, block_errors, fused_conv_reference, fused_table,
                                  fused_weights)

KINDS = {0: (48, 1, 4), 1: (10, 3, 16), 2: (16, 1, 8), 3: (4, 3, 16)}     # kind -> (mul_out, 2l_out+1, rows per tile)


def _deswizzle(img):
    """[T, n_kb, 256, 8, 8] 128B-swizzled -> [T, 256, n_kb*64] row-major (the swizzle is an involution)."""
    T, n_kb, R = img.shape[:3]
    rows = torch.arange(R) % 8
    src = torch.arange(8)[None, :] ^ rows[:, None]
    lin = torch.gather(img, 3, src[None, None, :, :, None].expand(T, n_kb, R, 8, 8))
    return lin.permute(0, 2, 1, 3, 4).reshape(T, R, n_kb * 64).double()


def _split_operand(a):
    """fp32 activations [E, K] -> the kernel's A image [hi | lo | 1 1 0...] (sections padded to Kp) as float64."""
    hi = a.to(torch.bfloat16)
    lo = (a - hi.float()).to(torch.bfloat16)
    E, K = a.shape
    Kp = (K + 15) // 16 * 16
    out = torch.zeros(E, 2 * Kp + 16, dtype=torch.float64)
    out[:, :K], out[:, Kp:Kp + K] = hi.double(), lo.double()
    out[:, 2 * Kp:2 * Kp + 2] = 1.0
    return out


def _schedule(S, n_kb):
    """csrc/fused_conv.cu:build_ops - (A column block, B column block) of every MMA, k-block by k-block."""
    ops = []
    for kb in range(n_kb):
        for j in range(4):
            c = 4 * kb + j
            if c < S:
                ops += [(c, c), (S + c, c)]          # B hi step x A hi, x A lo
            elif c < 2 * S:
                ops.append((c - S, c))               # B lo step x A hi
            elif c == 2 * S:
                ops.append((2 * S, c))               # bias step x ones
    return ops


def _mma(A, Bimg, K):
    """A [E, 2Kp+16] x B [N, 2Kp+16 (+pad)]^T the way the kernel issues it: one 16-column MMA step at a time."""
    S = (K + 15) // 16
    out = torch.zeros(A.shape[0], Bimg.shape[0], dtype=torch.float64)
    ops = _schedule(S, Bimg.shape[1] // 64)
    assert len(ops) == 3 * S + 1
    for a, b in ops:
        out += A[:, 16 * a:16 * a + 16] @ Bimg[:, 16 * b:16 * b + 16].T
    return out


def _sh(vec):
    v = torch.nn.functional.normalize(vec.double(), dim=-1)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    s3, s5, s15 = math.sqrt(3), math.sqrt(5), math.sqrt(15)
    return torch.stack([torch.ones_like(x), s3 * x, s3 * y, s3 * z, s15 * x * z, s15 * x * y,
                        s5 * (y * y - 0.5 * (x * x + z * z)), s15 * y * z, 0.5 * s15 * (z * z - x * x)], 1)


def emulate(plan, ea, node, ns, tgt, src, x, vec, n_out, ew=None):
    E = ea.shape[0]
    a0 = torch.cat([ea, node[tgt, :ns], node[src, :ns]], 1) if ns else ea
    w1 = _deswizzle(plan.w1_images)[0]                                   # [256, K1']
    H = plan.hidden
    hid = torch.relu(_mma(_split_operand(a0), w1[:H], a0.shape[1])).float()      # fp32 accumulator -> ReLU
    A = _split_operand(hid)
    w2 = _deswizzle(plan.w2_images)                                      # [T, 256, K']
    Y = _sh(vec)
    tiles = plan.tiles.tolist()
    mtab = plan.mtab.double()[:, :45].reshape(-1, 3, 3, 5)               # [path][i][k][j]
    out = torch.zeros(n_out, plan.table.d_out, dtype=torch.float64)
    acc = None
    for t, (kind, n_mma, x_off, nrow, d_in, out_off, flags, path) in enumerate(tiles):
        mul_out, dout, rows = KINDS[kind]
        assert n_mma % 32 == 0 and nrow * mul_out <= n_mma <= mul_out * rows <= 192
        Wt = torch.zeros(E, mul_out * rows, dtype=torch.float64)         # columns beyond n_mma are never produced
        Wt[:, :n_mma] = _mma(A, w2[t, :n_mma], H)                        # [E, N]: the accumulator tile
        sh_off = (flags >> 8) & 0xff
        yb = torch.zeros(E, 5, dtype=torch.float64)
        for j in range(5):
            yb[:, j] = Y[:, min(sh_off + j, 8)]
        M = torch.einsum('ikj,ej->eik', mtab[path], yb)
        if ew is not None:
            M = M * ew.double().reshape(-1, 1, 1)
        xs = torch.zeros(E, rows, d_in, dtype=torch.float64)
        xs[:, :nrow] = x[src][:, x_off:x_off + nrow * d_in].double().reshape(E, nrow, d_in)
        z = torch.einsum('eri,eik->erk', xs, M[:, :d_in, :dout])         # [E, rows, dout]
        z[:, (n_mma // mul_out) + (1 if n_mma % mul_out else 0):] = 0   # rows whose columns lie beyond the MMA width
        if flags & 1:
            acc = torch.zeros(E, mul_out, dout, dtype=torch.float64)
        acc = acc + torch.einsum('erw,erk->ewk', Wt.reshape(E, rows, mul_out), z)
        if flags & 2:
            full = torch.zeros(E, plan.table.d_out, dtype=torch.float64)
            full[:, out_off:out_off + mul_out * dout] = acc.reshape(E, -1)
            out.index_add_(0, tgt, full)
    return out


@pytest.mark.parametrize("li", [0, 1, 2, 3])
def test_fused_plan_emulation_matches_oracle_layer(li):
    from oracle.tensor_layers import TensorProductConvLayer as OLayer
    ns, nv = 48, 10
    seq = get_irrep_seq(ns, nv, False, False)
    ins, outs, shs = seq[min(li, 3)], seq[min(li + 1, 3)], '1x0e+1x1o+1x2e'
    torch.manual_seed(li)
    layer = OLayer(ins, shs, outs, 3 * ns, residual=False, batch_norm=False, hidden_features=3 * ns).eval()
    table = build_table(ins, shs, outs, 'fctp')
    assert fused.supported(table, 3 * ns, 3 * ns)
    plan = fused.FusedPlan(table, layer.fc[0].weight, layer.fc[0].bias, layer.fc[-1].weight, layer.fc[-1].bias)
    g = torch.Generator().manual_seed(100 + li)
    n_nodes, E = 11, 150
    x = torch.randn(n_nodes, table.d_in, generator=g)
    tgt = torch.sort(torch.randint(0, n_nodes, (E,), generator=g)).values
    src = torch.randint(0, n_nodes, (E,), generator=g)
    vec = torch.randn(E, 3, generator=g)
    ea = torch.randn(E, ns, generator=g)
    ew = torch.rand(E, 1, generator=g)
    from oracle import e3nn_lite as o3
    sh = o3.spherical_harmonics(o3.Irreps(shs), vec, normalize=True, normalization='component')
    ea_full = torch.cat([ea, x[tgt, :ns], x[src, :ns]], 1)
    with torch.no_grad():
        ref = layer(x, torch.stack([tgt, src]), ea_full, sh, reduce='sum', edge_weight=ew)
    got = emulate(plan, ea, x, ns, tgt, src, x, vec, n_nodes, ew)
    err = float((got - ref.double()).abs().max() / ref.abs().max())
    assert err < 3e-5, err          # split-bf16 x3: ~2^-16 relative per product, fp32-level after accumulation
    assert plan.n_tiles == len(plan.tiles) and plan.mma_flops_per_tile > 0


@pytest.mark.parametrize("ns_nv,stage,lmax,faster", KIND_GRID)
def test_emulation_consumer_kinds(ns_nv, stage, lmax, faster):
    """Every consumer kind / stage / harmonics variant at the production (ne, ns, H): the emulated plan against the float64
    reference, per output block."""
    ns, nv = ns_nv
    table = fused_table(ns, nv, stage, lmax, faster)
    _emulation_case(table, ns, ns, 3 * ns, seed=200 + 10 * stage + lmax + 5 * faster + ns)


@pytest.mark.parametrize("ne,ns,H", SHAPE_GRID)
def test_emulation_radial_shapes(ne, ns, H):
    _emulation_case(fused_table(48, 10, 3, 2, False), ne, ns, H, seed=ne + 3 * ns + H)


def _emulation_case(table, ne, ns, H, seed, n_nodes=11, E=150):
    assert fused.supported(table, H, ne + 2 * ns)
    g = torch.Generator().manual_seed(seed)
    w = fused_weights(table, H, ne + 2 * ns, g)
    plan = fused.FusedPlan(table, *w)
    x = torch.randn(n_nodes, table.d_in, generator=g)
    node = torch.randn(n_nodes, max(ns, 1) + 2, generator=g)
    tgt = torch.randint(0, n_nodes, (E,), generator=g)
    src = torch.randint(0, n_nodes, (E,), generator=g)
    ea, vec, ew = torch.randn(E, ne, generator=g), torch.randn(E, 3, generator=g), torch.rand(E, generator=g)
    got = emulate(plan, ea, node, ns, tgt, src, x, vec, n_nodes, ew)
    ref, _ = fused_conv_reference(table, *w, ea, node, ns, tgt, src, x, vec, n_nodes, ew=ew)
    errs = block_errors(got, ref, table.out_irreps)
    assert max(errs.values()) < 3e-5, errs         # the kernel's per-block tolerance; measured <= 1e-5


@pytest.mark.parametrize("faster,ns,extras", [(False, 48, True), (False, 0, False), (True, 16, True), (True, 0, True)])
def test_fp64_reference_matches_oracle_layer(faster, ns, extras):
    """tests/parity_helpers.py:fused_conv_reference, followed by the mean, BatchNorm and residual, is the oracle
    TensorProductConvLayer run in float64 (edge_perm / vec_sign / ea_add / edge_weight applied to the layer's inputs)."""
    from oracle import e3nn_lite as o3
    from oracle.tensor_layers import TensorProductConvLayer as OLayer
    from tests.parity_helpers import irreps_str, rand_bn_
    nv = 10 if ns != 16 else 4
    table = fused_table(ns or 48, nv, 2, 1 if faster else 2, faster)
    ins, shs, outs = irreps_str(table.in_irreps), irreps_str(table.sh_irreps), irreps_str(table.out_irreps)
    ne, n_nodes, E = 24, 13, 200
    n_out = n_nodes
    K1 = ne + 2 * ns
    torch.manual_seed(ns + faster)
    layer = OLayer(ins, shs, outs, K1, hidden_features=40, faster=faster).double().eval()
    g = torch.Generator().manual_seed(7 + ns)
    rand_bn_(layer.batch_norm, g)
    w = (layer.fc[0].weight, layer.fc[0].bias, layer.fc[-1].weight, layer.fc[-1].bias)
    x = torch.randn(n_nodes, table.d_in, generator=g, dtype=torch.float64)
    tgt = torch.randint(0, n_out - 4, (E,), generator=g)          # the last rows receive no edge: mean of nothing = 0
    src = torch.randint(0, n_nodes, (E,), generator=g)
    rows = 2 * E
    ea, vec = torch.randn(rows, ne, generator=g, dtype=torch.float64), torch.randn(rows, 3, generator=g, dtype=torch.float64)
    vec[3] = 0.0                                          # a zero-length edge vector
    ew = torch.rand(rows, generator=g, dtype=torch.float64)
    kw = {}
    perm = torch.randperm(rows, generator=g)[:E] if extras else torch.arange(E)
    if extras:
        add, add_idx = torch.randn(3, ne, generator=g, dtype=torch.float64), torch.randint(0, 3, (E,), generator=g)
        kw = dict(edge_perm=perm, vec_sign=-1.0, ea_add=add, ea_add_idx=add_idx)
    sign = kw.get('vec_sign', 1.0)
    a = ea[perm] + (add[add_idx] if extras else 0)
    if ns:
        a = torch.cat([a, x[tgt, :ns], x[src, :ns]], 1)
    sh = o3.spherical_harmonics(o3.Irreps(shs), sign * vec[perm], normalize=True, normalization='component')
    with torch.no_grad():
        s, cnt = fused_conv_reference(table, *w, ea, x, ns, tgt, src, x, vec, n_out, ew=ew, **kw)
        got = layer.batch_norm(s / cnt.clamp_min(torch.finfo(torch.float64).eps)[:, None])
        got = got + torch.nn.functional.pad(x, (0, got.shape[1] - x.shape[1]))
        ref = layer(x, torch.stack([tgt, src]), a, sh, out_nodes=n_out, edge_weight=ew[perm][:, None])
    assert torch.equal(cnt, torch.bincount(tgt, minlength=n_out).double())
    err = float((got - ref).abs().max() / ref.abs().max())
    assert err < 1e-12, err


def test_fused_plan_tile_flags_and_limits():
    """Tile table invariants the kernel relies on: N a multiple of 16 and <= 192 (the kernel's MMA width), flag 1 on
    the first / flag 2 on the last tile of every output irrep, flag 4 exactly where the path changes, tiles of one output
    irrep contiguous."""
    ns, nv = 48, 10
    seq = get_irrep_seq(ns, nv, False, False)
    table = build_table(seq[3], '1x0e+1x1o+1x2e', seq[3], 'fctp')
    g = torch.Generator().manual_seed(0)
    H = 3 * ns
    plan = fused.FusedPlan(table, torch.randn(H, H, generator=g), torch.randn(H, generator=g),
                           torch.randn(table.weight_numel, H, generator=g), torch.randn(table.weight_numel, generator=g))
    tiles = plan.tiles.tolist()
    assert len(tiles) == plan.n_tiles <= 160
    assert tiles[0][6] & 1 and tiles[0][6] & 4 and tiles[-1][6] & 2
    seen_out = []
    for i, (kind, n, x_off, nrow, d_in, out_off, flags, ment) in enumerate(tiles):
        mul_out, dout, rows = KINDS[kind]
        assert nrow * mul_out <= n <= mul_out * rows and n % 32 == 0 and 32 <= n <= 192 and (n // 2) % 8 == 0
        assert (flags >> 8) in (0, 1, 4)            # offset of the path's l_sh block in the spherical-harmonics vector
        assert 1 <= nrow <= rows and d_in in (1, 3) and 0 <= x_off and x_off + nrow * d_in <= table.d_in
        assert out_off + mul_out * dout <= table.d_out
        flags &= 0xff
        if flags & 1:
            assert out_off not in seen_out, "tiles of one output irrep must be contiguous"
            seen_out.append(out_off)
            assert i == 0 or tiles[i - 1][6] & 2
        else:
            assert out_off == tiles[i - 1][5] and not (tiles[i - 1][6] & 2)
        if i and (ment != tiles[i - 1][7] or flags & 1):
            assert flags & 4 or ment == tiles[i - 1][7]
        if flags & 4 and i:
            assert ment != tiles[i - 1][7] or x_off <= tiles[i - 1][2]
    # every reference weight column is placed exactly once: total valid columns = weight_numel
    assert sum(t[3] * KINDS[t[0]][0] for t in tiles) == table.weight_numel
    assert not fused.supported(build_table('16x0e', '1x0e+1x1o+1x2e', '16x0e + 4x1o', 'fctp'), 400, 48)   # hidden too wide

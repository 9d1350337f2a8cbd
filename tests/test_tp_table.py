"""CPU: the kernel's instruction tables, interpreted in numpy (tp_table.evaluate), against the oracle tensor products;
plus the C ABI's load/export check."""
import os
import re

import numpy as np
import pytest
import torch

from diffdock_b200.irreps import real_cg
from diffdock_b200.tp_table import build_table, evaluate, full_tensor_product
from oracle import e3nn_lite as o3
from oracle.tensor_layers import FasterTensorProduct, get_irrep_seq
from tests.parity_helpers import kernel_weights, table_sections, tp_scatter_reference, tp_table_grid


def _case(ins, shs, outs, kind, lmax, given=False):
    t = build_table(ins, shs, outs, kind, sh_from_vector=not given)
    g = torch.Generator().manual_seed(len(ins) + lmax)
    E = 3
    x = torch.randn(E, t.d_in, generator=g, dtype=torch.float64)
    v = torch.randn(E, 3, generator=g, dtype=torch.float64)
    w = torch.randn(E, t.weight_numel, generator=g, dtype=torch.float64)
    sh = o3.spherical_harmonics(o3.Irreps(shs), v) if not given else torch.randn(E, t.d_sh, generator=g, dtype=torch.float64)
    ref = (o3.FullyConnectedTensorProduct(ins, shs, outs) if kind == 'fctp' else FasterTensorProduct(ins, shs, outs))(x, sh, w)
    wp = np.zeros((E, t.weight_numel_padded))
    m = t.w_perm >= 0
    wp[:, m] = w.numpy()[:, t.w_perm[m]]
    got = evaluate(t, x.numpy(), sh.numpy() if given else v.numpy(), wp)
    return float(np.abs(got - ref.numpy()).max() / np.abs(ref.numpy()).max()), t


@pytest.mark.parametrize("i", [0, 1, 2, 3])
def test_tables_match_oracle_tensor_products(i):
    seq = get_irrep_seq(48, 10, False, False)
    a, b = seq[i], seq[min(i + 1, 3)]
    for kind, shs, lmax in (('fctp', '1x0e+1x1o+1x2e', 2), ('faster', '1x0e+1x1o', 1), ('fctp', '1x0e+1x1o', 1)):
        err, t = _case(a, shs, b, kind, lmax)
        assert err < 1e-6
        assert t.weight_numel_padded % 4 == 0 and sorted(t.w_perm[t.w_perm >= 0]) == list(range(t.weight_numel))


def test_weight_numel_table_of_survey_appendix_b():
    seq = get_irrep_seq(48, 10, False, False)
    sh2, sh1 = '1x0e+1x1o+1x2e', '1x0e+1x1o'
    exp2, exp1 = [2784, 3564, 4344, 7128], [2784, 3464, 4144, 6928]
    for i in range(4):
        assert build_table(seq[i], sh2, seq[min(i + 1, 3)], 'fctp').weight_numel == exp2[i]
        assert build_table(seq[i], sh1, seq[min(i + 1, 3)], 'faster').weight_numel == exp1[i]
    assert build_table(seq[3], sh2, '2x1o + 2x1e', 'fctp').weight_numel == 312
    T, tor_sh = full_tensor_product(sh2, '1x2e')
    assert T.shape == (9, 5, 45)
    from diffdock_b200.irreps import irreps_str
    assert build_table(seq[3], irreps_str(tor_sh), '48x0o + 48x0e', 'fctp', sh_from_vector=False).weight_numel == 6528


def test_heads_second_order_and_padding():
    seq = get_irrep_seq(48, 10, False, False)
    assert _case(seq[3], '1x0e+1x1o+1x2e', '2x1o + 2x1e', 'fctp', 2)[0] < 1e-6
    seq5 = get_irrep_seq(5, 3, True, True)                     # odd multiplicities -> padded weight rows
    err, t = _case(seq5[3], '1x0e+1x1o+1x2e', seq5[3], 'fctp', 2)
    assert err < 1e-6 and t.weight_numel_padded > t.weight_numel and t.weight_numel_padded % 4 == 0
    T, tor_sh = full_tensor_product('1x0e+1x1o+1x2e', '1x2e')
    from diffdock_b200.irreps import irreps_str
    assert _case(seq[3], irreps_str(tor_sh), '48x0o + 48x0e', 'fctp', 2, given=True)[0] < 1e-6
    f = o3.FullTensorProduct(o3.Irreps.spherical_harmonics(2), '2e')
    a, b = torch.randn(4, 9, dtype=torch.float64), torch.randn(4, 5, dtype=torch.float64)
    assert torch.allclose(f(a, b), torch.einsum('ea,eb,abc->ec', a, b, torch.from_numpy(T)), atol=1e-12)


GRID = sorted(tp_table_grid())


@pytest.mark.parametrize("name", GRID)
def test_grid_tables_match_scatter_reference(name):
    """The numpy interpreter of the compiled blobs, on kernel-layout rows from kernel_weights (zero fill), scattered onto
    targets with repeats, against the float64 reference of the whole accumulate step (tp_scatter_reference)."""
    t = tp_table_grid()[name]
    g = torch.Generator().manual_seed(GRID.index(name))
    E, n_out = 3, 3
    x = torch.randn(5, t.d_in, generator=g, dtype=torch.float64)
    src, tgt = torch.tensor([4, 0, 4]), torch.tensor([2, 0, 2])
    geo = torch.randn(E, 3 if t.sh_lmax >= 0 else t.d_sh, generator=g, dtype=torch.float64)
    w = torch.randn(E, t.weight_numel, generator=g, dtype=torch.float64)
    ew = torch.tensor([0.5, -1.25, 2.0], dtype=torch.float64)
    ref, cnt = tp_scatter_reference(t, x, src, tgt, geo, w, n_out, ew=ew)
    msg = evaluate(t, x[src].numpy(), geo.numpy(), kernel_weights(t, w, fill=0.0).numpy(), edge_weight=ew.numpy())
    got = np.zeros((n_out, t.d_out))
    np.add.at(got, tgt.numpy(), msg)
    assert cnt.tolist() == [1.0, 0.0, 2.0]
    assert np.abs(got - ref.numpy()).max() <= 1e-12 * np.abs(ref.numpy()).max()
    assert not ref[1].any()


def test_grid_reaches_every_table_feature():
    """The grid above exercises every table feature the kernel branches on; narrowing it fails here."""
    kinds, zkinds, col_tiles, rem_rows, max_chunks, padded, d_in = set(), set(), 1, False, 0, False, 0
    for t in tp_table_grid().values():
        paths, tiles, chunks, _ = table_sections(t)
        kinds |= set(tiles[:, 11].tolist())
        zkinds |= set(paths[:, 7].tolist())
        rem_rows |= bool(np.any(tiles[:, 2] >> 16 > 0))
        max_chunks = max(max_chunks, len(chunks))
        padded |= t.weight_numel_padded > t.weight_numel
        d_in = max(d_in, t.d_in)
        # every column tile of an output irrep has its own accumulator rows: more of them than outputs = a split output
        col_tiles = max(col_tiles, len(set(tiles[:, 9].tolist())) - len(t.out_irreps) + 1)
    assert kinds >= {0, 1, 2, 3, 4} and zkinds >= {0, 1, 2, 3, 4}
    assert col_tiles > 1 and rem_rows and max_chunks > 8 and padded and d_in > 256


def test_tma_chunks_are_aligned_and_cover_the_row():
    seq = get_irrep_seq(48, 10, False, False)
    t = build_table(seq[3], '1x0e+1x1o+1x2e', seq[3], 'fctp')
    ib = t.iblob
    chunks = ib[ib[17]:ib[17] + 4 * ib[3]].reshape(-1, 4)
    covered = np.zeros(t.weight_numel_padded, dtype=int)
    for tb, te, g, n in chunks:
        assert g % 4 == 0 and n % 4 == 0 and n <= ib[14] and te > tb      # 16-byte aligned TMA bulk copies
        covered[g:g + n] += 1
    assert np.all(covered == 1)
    tiles = ib[ib[16]:ib[16] + 16 * ib[2]].reshape(-1, 16)
    assert tiles[0][3] & 1 and tiles[-1][3] & 2                          # accumulator runs open and close


def test_product_cg_blocks_equal_oracle_blocks():
    for l1 in range(3):
        for l2 in range(3):
            for l3 in range(abs(l1 - l2), l1 + l2 + 1):
                assert np.allclose(real_cg(l1, l2, l3), o3.wigner_3j(l1, l2, l3).numpy(), atol=1e-13)


def test_c_abi_library_exports_every_declared_symbol(built_lib):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(root, 'include', 'diffdock_b200.h')).read()
    declared = sorted(set(re.findall(r'\b(ddb200_\w+)\s*\(', hdr)))
    assert len(declared) >= 8
    from diffdock_b200 import _lib
    assert sorted(_lib.SIGNATURES) == declared
    for name in declared:
        assert getattr(built_lib, name) is not None
    assert b'sm_90a' in built_lib.ddb200_version()


def test_product_refuses_cpu_tensors():
    from diffdock_b200.tensor_layers import TensorProductConvLayer
    layer = TensorProductConvLayer('4x0e', '1x0e+1x1o', '4x0e + 2x1o', 6).eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        layer(torch.randn(3, 4), torch.zeros(2, 2, dtype=torch.long), torch.randn(2, 6), torch.randn(2, 4))

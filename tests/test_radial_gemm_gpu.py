"""GPU: wgmma split-bf16 radial GEMM (csrc/radial_gemm.cu) vs a float64 reference of the same Linear.
Tolerance: the 3-term bf16 split keeps ~16 mantissa bits per operand -> 3e-5 of the output's max magnitude.

Edge counts given as strings are functions of the SM count: the kernel is persistent over 128-row edge tiles (grid =
min(tiles, SMs)), so 'sms*128+-1' give CTAs a second tile, and '2*sms*128+72' ends in a tile whose second warpgroup has
rows e_a < E <= e_b (the e_b row guard)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

EDGES = {'sms*128-1': lambda s: s * 128 - 1, 'sms*128+1': lambda s: s * 128 + 1, '2*sms*128+72': lambda s: 2 * s * 128 + 72}


def _edges(E):
    return EDGES[E](torch.cuda.get_device_properties(0).multi_processor_count) if isinstance(E, str) else E


def _nan_view(rows, cols, width, col0=0, device='cuda'):
    """[rows, cols] view at column col0 of a NaN-filled [rows + 8, width] buffer, and the buffer."""
    buf = torch.full((rows + 8, width), float('nan'), device=device)
    return buf[:rows, col0:col0 + cols], buf


def _untouched_outside(buf, rows, cols):
    """Nothing was stored outside out = buf[:rows, :cols]."""
    outside = torch.ones_like(buf, dtype=torch.bool)
    outside[:rows, :cols] = False
    return bool(torch.isnan(buf[outside]).all())


def _gemm_case(E, K, N, ldh_pad=0, ldo_pad=0, device='cuda'):
    """radial_gemm with h a view of row stride K + ldh_pad and out a view of row stride n_tiles 256 + ldo_pad, both inside
    NaN-filled buffers: (error relative to the output max, padded columns zero, nothing stored outside out)."""
    from diffdock_b200.radial import BN, build_b_images, radial_gemm
    g = torch.Generator().manual_seed(E + N)
    h, _ = _nan_view(E, K, K + ldh_pad, device=device)
    h.copy_(torch.relu(torch.randn(E, K, generator=g)))
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(device)
    b = torch.randn(N, generator=g).to(device)
    img, bp, nt = build_b_images(W, b)
    out, obuf = _nan_view(E, nt * BN, nt * BN + ldo_pad, device=device)
    radial_gemm(h, img, bp, nt, out=out)
    torch.cuda.synchronize(device)
    ref = torch.nn.functional.linear(h.double(), W.double(), b.double())
    err = float((out[:, :N].double() - ref).abs().max() / ref.abs().max())
    return err, bool(torch.all(out[:, N:] == 0)), _untouched_outside(obuf, E, nt * BN)


KS = (1, 21, 22, 149)          # one column; one k-block (3K = 63); two (66); seven, the widest


def _check_gemm(E, K, N, ldh_pad=0, ldo_pad=0):
    err, pad_zero, untouched = _gemm_case(_edges(E), K, N, ldh_pad, ldo_pad)
    assert err < 3e-5, err
    assert pad_zero, "padded columns: zero weights + zero bias"
    assert untouched, "store outside [E, n_tiles 256]"


@pytest.mark.parametrize("E,K,N", [(1000, 144, 7128), (128, 144, 312), (77, 96, 312), (4099, 144, 2784), (300, 48, 500)]
                         + [('sms*128+1', K, N) for K in KS for N in (1, 255, 257, 7128)])
def test_radial_gemm_matches_fp32_linear(built_lib, E, K, N):
    _check_gemm(E, K, N)


@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("E", list(EDGES))
def test_radial_gemm_multi_tile_strided(built_lib, E, K):
    """Second edge tile per CTA and the e_b row guard, with ldh > K and ldo > n_tiles 256."""
    _check_gemm(E, K, 257, ldh_pad=3, ldo_pad=68)


def test_radial_gemm_second_device(built_lib):
    """The > 48 KB shared-memory opt-in is a per-device attribute: a launch on a second GPU, after one on the first in the
    same process, must run (and be right)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    for dev in ('cuda:0', 'cuda:1'):
        with torch.cuda.device(dev):
            err, pad_zero, untouched = _gemm_case(300, 144, 500, device=dev)
        assert err < 3e-5 and pad_zero and untouched, (dev, err)


@pytest.mark.parametrize("E,ne,ns,H,N", [(3000, 48, 48, 144, 7128), (500, 96, 0, 96, 312), (129, 48, 48, 144, 2784),
                                        (70, 16, 16, 48, 320)]
                         + [(E, 48, 21, 149, 257) for E in EDGES])
def test_radial_mlp_one_kernel_matches_fp32(built_lib, E, ne, ns, H, N):
    """Gather + Linear + ReLU + Linear in one kernel vs the float64 op sequence (two chained split-bf16 GEMMs: 6e-5).
    The node scalars are the first ns of 60 columns (ld_node > ns); out is wider than n_tiles 256."""
    from diffdock_b200.radial import BN, build_b_images, radial_mlp
    E = _edges(E)
    g = torch.Generator().manual_seed(E + N)
    n_nodes = 200
    node = torch.randn(n_nodes, 60 if ns else 4, generator=g).cuda()
    ea = torch.randn(E, ne, generator=g).cuda()
    tgt = torch.randint(0, n_nodes, (E,), generator=g).int().cuda()
    src = torch.randint(0, n_nodes, (E,), generator=g).int().cuda()
    K1 = ne + 2 * ns
    W1 = (torch.randn(H, K1, generator=g) / K1 ** 0.5).cuda()
    b1 = torch.randn(H, generator=g).cuda()
    W2 = (torch.randn(N, H, generator=g) / H ** 0.5).cuda()
    b2 = torch.randn(N, generator=g).cuda()
    i1, b1p, _ = build_b_images(W1, b1)
    i2, b2p, nt = build_b_images(W2, b2)
    out, obuf = _nan_view(E, nt * BN, nt * BN + 4)
    radial_mlp(ea, node, ns, tgt, src, i1, b1p, H, i2, b2p, nt, out=out)
    torch.cuda.synchronize()
    a = torch.cat([ea, node[tgt.long(), :ns], node[src.long(), :ns]], 1).double() if ns else ea.double()
    ref = torch.relu(a @ W1.double().T + b1.double()) @ W2.double().T + b2.double()
    err = (out[:, :N].double() - ref).abs().max() / ref.abs().max()
    assert err < 6e-5, float(err)
    assert _untouched_outside(obuf, E, nt * BN)

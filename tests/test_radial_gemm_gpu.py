"""GPU: wgmma split-bf16 radial GEMM (csrc/radial_gemm.cu) vs an fp32 reference of the same Linear.
Tolerance: the 3-term bf16 split keeps ~16 mantissa bits per operand -> 3e-5 of the output's max magnitude."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("E,K,N", [(1000, 144, 7128), (128, 144, 312), (77, 96, 312), (4099, 144, 2784), (300, 48, 500)])
def test_radial_gemm_matches_fp32_linear(built_lib, E, K, N):
    from diffdock_b200.radial import build_b_images, radial_gemm
    g = torch.Generator().manual_seed(E + N)
    h = torch.relu(torch.randn(E, K, generator=g)).cuda()
    W = (torch.randn(N, K, generator=g) / K ** 0.5).cuda()
    b = torch.randn(N, generator=g).cuda()
    img, bp, nt = build_b_images(W, b)
    out = radial_gemm(h, img, bp, nt)
    torch.cuda.synchronize()
    ref = torch.nn.functional.linear(h.double(), W.double(), b.double())
    err = (out[:, :N].double() - ref).abs().max() / ref.abs().max()
    assert err < 3e-5, float(err)
    assert torch.all(out[:, N:] == 0) or out.shape[1] == N     # padded columns: zero weights + zero bias


@pytest.mark.parametrize("E,ne,ns,H,N", [(3000, 48, 48, 144, 7128), (500, 96, 0, 96, 312), (129, 48, 48, 144, 2784),
                                        (70, 16, 16, 48, 320)])
def test_radial_mlp_one_kernel_matches_fp32(built_lib, E, ne, ns, H, N):
    """Gather + Linear + ReLU + Linear in one kernel vs the fp32 op sequence (two chained split-bf16 GEMMs: 6e-5)."""
    from diffdock_b200.radial import build_b_images, radial_mlp
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
    out = radial_mlp(ea, node, ns, tgt, src, i1, b1p, H, i2, b2p, nt)
    torch.cuda.synchronize()
    a = torch.cat([ea, node[tgt.long(), :ns], node[src.long(), :ns]], 1).double() if ns else ea.double()
    ref = torch.relu(a @ W1.double().T + b1.double()) @ W2.double().T + b2.double()
    err = (out[:, :N].double() - ref).abs().max() / ref.abs().max()
    assert err < 6e-5, float(err)

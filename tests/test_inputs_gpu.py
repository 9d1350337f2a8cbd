"""GPU: input side (SURVEY.md section 8, row f4).  ``ddb200_contact_count/_fill`` through the C ABI against the edge lists
the UNMODIFIED reference produced (tests/golden/ref_inputs.pt, datasets/process_mols.py:161-202) - index work, compared bit
for bit - and the device-resident complex (build_complex / PackedComplex / pose_copies) driven through ``sampling()``
against the host-graph path."""
import copy

import numpy as np
import pytest
import torch

from tests.parity_helpers import canonical_contact_edges, load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def fx():
    return load_golden('ref_inputs.pt')


@pytest.mark.parametrize('i', range(5))
def test_contact_graph_matches_reference(built_lib, fx, i):
    from diffdock_b200.hetero import HeteroGraph
    from diffdock_b200.inputs import new_extract_receptor_structure
    c = fx['receptor'][i]
    g = HeteroGraph()
    new_extract_receptor_structure(c['seq'], c['all_coords'].numpy(), g, neighbor_cutoff=c['cutoff'],
                                   max_neighbors=c['max_neighbors'], lm_embeddings=[e.numpy() for e in c['lm']], device='cuda:0')
    ei = g['receptor', 'receptor'].edge_index
    assert ei.dtype == torch.int64 and ei.is_cuda
    want = canonical_contact_edges(c['edge_index'].numpy(), c['pos'].numpy())
    assert np.array_equal(ei.cpu().numpy(), want)
    assert torch.equal(g['receptor'].x.cpu(), c['x']) and torch.equal(g['receptor'].pos.cpu(), c['pos'])


@pytest.mark.parametrize('n,cutoff,k', [(2500, 15.0, 24), (700, 40.0, 1000), (1400, 60.0, 1500), (900, 3.0, 5), (1, 5.0, 3),
                                        (2, 0.5, 3)])
def test_contact_graph_matches_oracle(built_lib, n, cutoff, k):
    """Sizes and regimes the fixture does not hold: a large receptor, every hit kept in index order from the shared-memory
    list (700 points, cut-off 40 A, K = 1000: at most 699 hits, within the list's 1024), every hit kept in index order with
    more hits than the list holds (1400 points, 60 A, K = 1500: the kernel rescans), mostly isolated points (nearest-other
    rule), degenerate sizes.  tests/test_contact_graph_ref_gpu.py covers the rescan paths at the list's capacity."""
    from oracle.inputs import contact_graph as oracle_graph
    from diffdock_b200.inputs import contact_graph
    rng = np.random.default_rng(n)
    R = (3.0 * n / (4.0 * np.pi * 0.0075)) ** (1.0 / 3.0)
    v = rng.normal(size=(n, 3))
    pos = (v / np.linalg.norm(v, axis=1, keepdims=True) * (R * rng.uniform(size=(n, 1)) ** (1.0 / 3.0)) + 12.5).astype(np.float32)
    got = contact_graph(torch.from_numpy(pos).cuda(), cutoff, k).cpu().numpy()
    want = oracle_graph(pos, cutoff, k)
    assert got.shape == want.shape and np.array_equal(got, want)


def test_knn_only_graph(built_lib):
    """knn_only_graph (process_mols.py:171-172, torch_cluster.knn_graph): the k nearest other points of every centre."""
    from diffdock_b200.inputs import contact_graph
    g = torch.Generator().manual_seed(0)
    pos = (torch.randn(400, 3, generator=g) * 15).float()
    ei = contact_graph(pos.cuda(), 0.0, 7, knn_only=True).cpu()
    assert ei.shape == (2, 400 * 7) and torch.equal(ei[1], torch.arange(400).repeat_interleave(7))
    d = torch.cdist(pos.double(), pos.double())
    d.fill_diagonal_(float('inf'))
    want = torch.topk(d, 7, dim=1, largest=False).indices
    assert torch.equal(ei[0].reshape(400, 7).sort(1).values, want.sort(1).values)


def test_device_resident_complex_through_the_sampler(built_lib, tmp_path):
    """build_complex (receptor on the GPU) -> PackedComplex file -> one H2D copy -> pose_copies -> sampling() gives the poses
    the host-graph path (N deep copies, per-call upload) gives."""
    from functools import partial
    from diffdock_b200.cg_model import CGModel
    from diffdock_b200.diffusion_utils import get_t_schedule, get_timestep_embedding, t_to_sigma
    from diffdock_b200.inputs import PackedComplex, build_complex, pose_copies
    from diffdock_b200.sampling import sampling
    from diffdock_b200.synthetic import default_model_args
    fxl = load_golden('ref_inputs.pt')
    rc, lc = fxl['receptor'][0], fxl['ligand'][1]
    args = default_model_args(ns=16, nv=4, num_conv_layers=2, distance_embed_dim=16, cross_distance_embed_dim=16,
                              sigma_embed_dim=16)
    lm = [torch.cat([e, torch.zeros(e.shape[0], 1280 - e.shape[1])], 1).numpy() for e in rc['lm']]
    g = build_complex('c0', rc['seq'], rc['all_coords'].numpy(), lc['atom_feats'], lc['bond_begin'], lc['bond_end'],
                      lc['bond_type'], lc['pos_in'].numpy(), lm_embeddings=lm, receptor_radius=15.0, c_alpha_max_neighbors=24,
                      device='cuda:0')
    assert g['receptor'].x.is_cuda and not g['ligand'].pos.is_cuda and g['success']
    assert abs(float(g['receptor'].pos.mean())) < 1e-4 and abs(float(g['ligand'].pos.mean())) < 1e-5
    path = tmp_path / 'c0.ddpk'
    PackedComplex.pack(g).save(path)
    h = PackedComplex.load(path).to('cuda:0')
    assert h['receptor'].x.is_cuda and torch.equal(h['receptor'].x, g['receptor'].x)
    assert torch.equal(h['receptor', 'receptor'].edge_index, g['receptor', 'receptor'].edge_index)
    torch.manual_seed(0)
    model = CGModel(partial(t_to_sigma, args=args), torch.device('cuda:0'),
                    get_timestep_embedding('sinusoidal', args.sigma_embed_dim, args.embedding_scale),
                    sigma_embed_dim=16, sh_lmax=2, ns=16, nv=4, num_conv_layers=2, lig_max_radius=args.max_radius,
                    rec_max_radius=args.rec_max_radius, cross_max_distance=args.cross_max_distance,
                    center_max_distance=args.center_max_distance, distance_embed_dim=16, cross_distance_embed_dim=16,
                    dynamic_max_cross=args.dynamic_max_cross, lm_embedding_type='precomputed', embed_also_ligand=True,
                    differentiate_convolutions=True).eval().to('cuda:0')
    sched = get_t_schedule(inference_steps=4)
    n_poses = 5

    shifts = torch.randn(n_poses, 1, 3, generator=torch.Generator().manual_seed(5)) * 4.0

    def poses_from(graph, deep):
        items = [copy.deepcopy(graph) for _ in range(n_poses)] if deep else pose_copies(graph, n_poses)
        for i, it in enumerate(items):
            it['ligand'].pos = it['ligand'].pos + shifts[i]
        return items

    host = g.cpu()
    out_a, _ = sampling(poses_from(host, True), model, 4, sched, sched, sched, 'cuda:0', partial(t_to_sigma, args=args), args,
                        no_random=True, batch_size=n_poses)
    out_b, _ = sampling(poses_from(h, False), model, 4, sched, sched, sched, 'cuda:0', partial(t_to_sigma, args=args), args,
                        no_random=True, batch_size=n_poses)
    for a, b in zip(out_a, out_b):
        assert torch.allclose(a['ligand'].pos.cpu(), b['ligand'].pos.cpu(), atol=2e-3), \
            float((a['ligand'].pos.cpu() - b['ligand'].pos.cpu()).abs().max())

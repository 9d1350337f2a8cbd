"""CPU: the host side of packed sampling - the packing plan, the pose-update descriptor, ``collate_packed`` against the
general collate, the per-complex NaN guard, the centre-node indices - and the packed pose kernel's symbol and resources."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _complexes(shared=True, n_poses=(3, 2, 4), sizes=((30, 12), (35, 20), (30, 9)), seed=5, rigid=()):
    from diffdock_b200.synthetic import make_pose_list
    out = []
    for k, ((n_res, n_atoms), n) in enumerate(zip(sizes, n_poses)):
        poses = make_pose_list(n, n_res=n_res, n_atoms=n_atoms, seed=seed + k, tr_sigma_max=5.0, lm_dim=8)
        if k in rigid:
            for d in poses:
                d['ligand'].edge_mask = torch.zeros_like(d['ligand'].edge_mask)
                d['ligand'].mask_rotate = [np.zeros((0, d['ligand'].num_nodes), dtype=bool)]
        out.append(poses)
    if shared:
        rec, rr = out[0][0]._nodes['receptor'], out[0][0]._edges[('receptor', 'receptor')]
        for d in out[-1]:
            d._nodes['receptor'], d._edges[('receptor', 'receptor')] = rec, rr
    return out


# ---------------------------------------------------------------------------------------------------------------------
def test_pack_plan_keeps_order_and_budget():
    from diffdock_b200.sampling import pack_plan
    costs = [5, 3, 4, 20, 1, 1, 9, 2]
    packs = pack_plan(costs, 10)
    assert [i for p in packs for i in p] == list(range(len(costs)))     # every complex once, in order
    assert [3] in packs                                                 # larger than the budget: a batch of its own
    for p in packs:
        assert len(p) == 1 or sum(costs[i] for i in p) <= 10
    assert packs == [[0, 1], [2], [3], [4, 5], [6], [7]]
    assert pack_plan([], 10) == [] and pack_plan([11], 10) == [[0]] and pack_plan([2, 2, 2], 10) == [[0, 1, 2]]


def test_pose_layout_offsets_by_hand():
    from diffdock_b200.hetero import pose_layout
    cx = _complexes(shared=False, n_poses=(2, 1, 2), sizes=((20, 12), (20, 5), (20, 9)), rigid=(1,))
    nb = [int(cx[k][0]['ligand'].edge_mask.sum()) for k in range(3)]
    assert nb[0] > 1 and nb[1] == 0 and nb[2] >= 1
    layout, bu, bv, mask, max_atoms = pose_layout(cx)
    n0, n2 = nb[0], nb[2]
    want = [[0, 12, 0, n0, 0, 0],
            [12, 12, 0, n0, n0, 0],
            [24, 5, n0, 0, 2 * n0, 12 * n0],
            [29, 9, n0, n2, 2 * n0, 12 * n0],
            [38, 9, n0, n2, 2 * n0 + n2, 12 * n0]]
    assert layout.dtype == torch.int32 and layout.tolist() == want and max_atoms == 12
    assert bu.dtype == torch.int32 and bu.shape[0] == n0 + n2 and mask.shape[0] == 12 * n0 + 9 * n2
    lig0 = cx[0][0]
    rb = lig0['ligand', 'ligand'].edge_index.T[lig0['ligand'].edge_mask]
    assert bu[:n0].tolist() == rb[:, 0].tolist() and bv[:n0].tolist() == rb[:, 1].tolist()
    assert torch.equal(mask[:12 * n0], torch.from_numpy(lig0['ligand'].mask_rotate[0].astype(np.uint8).reshape(-1)))


def test_pose_layout_rejects_poses_that_differ():
    from diffdock_b200.hetero import pose_layout
    cx = _complexes(shared=False, n_poses=(2,), sizes=((20, 12),))
    cx[0][1]['ligand'].edge_mask = torch.zeros_like(cx[0][1]['ligand'].edge_mask)
    with pytest.raises(ValueError):
        pose_layout(cx)


def test_collate_packed_equals_general_collate():
    from diffdock_b200.hetero import collate, collate_packed
    cx = _complexes(shared=True, rigid=(1,))           # complexes 0 and 2 share a receptor, 1 has its own
    got = collate_packed(cx, 'cpu')
    ref = collate([d for p in cx for d in p])
    for key in ref.node_types:
        for k, v in ref[key].__dict__.items():
            if torch.is_tensor(v):
                assert torch.equal(getattr(got[key], k), v), (key, k)
    for et in ref.edge_types:
        for k, v in ref[et].__dict__.items():
            if torch.is_tensor(v):
                assert torch.equal(getattr(got[et], k), v), (et, k)
    assert got.num_graphs == ref.num_graphs == 9
    rr = [cx[k][0]['receptor', 'receptor'].num_edges for k in range(3)]
    assert got['receptor']._blocks == ((30, rr[0], 3, 0), (35, rr[1], 2, 1), (30, rr[0], 4, 0))
    assert got._complex_ptr.tolist() == [0, 3, 5, 9]
    nb = [int(cx[k][0]['ligand'].edge_mask.sum()) for k in range(3)]
    assert got._complex_bond_ptr.tolist() == [0, 3 * nb[0], 3 * nb[0], 3 * nb[0] + 4 * nb[2]]
    assert int(got._pose_layout[0][-1, 4] + got._pose_layout[0][-1, 3]) == int(ref['ligand'].edge_mask.sum())


def test_collate_shared_receptor_is_the_one_complex_case():
    from diffdock_b200.hetero import collate, collate_shared_receptor
    cx = _complexes(shared=False)
    got = collate_shared_receptor(cx[0], 'cpu')
    ref = collate(cx[0])
    assert got['receptor']._unique == (30, cx[0][0]['receptor', 'receptor'].num_edges, 3)
    assert not hasattr(got['receptor'], '_blocks') and '_center_node' not in got._globals
    for k, v in ref['receptor'].__dict__.items():
        if torch.is_tensor(v):
            assert torch.equal(getattr(got['receptor'], k), v), k


def test_centre_nodes_for_mixed_pose_counts():
    from diffdock_b200.hetero import collate_packed
    cx = _complexes(shared=False, n_poses=(3, 1, 2), sizes=((20, 12), (20, 7), (20, 9)))
    g = collate_packed(cx, 'cpu')
    # pose j of complex c reads node lig_ptr[first pose of c] + j
    assert g._center_node.tolist() == [0, 1, 2, 36, 43, 44]
    one = collate_packed(cx[:1], 'cpu')
    assert one._center_node.tolist() == [0, 1, 2]                       # one complex: the graph ids, as before


# ---------------------------------------------------------------------------------------------------------------------
def _scores(seed, n_pose, n_bond):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n_pose, 3, generator=g), torch.randn(n_pose, 3, generator=g), torch.randn(n_bond, generator=g)


@pytest.mark.parametrize("where", [[], [1], [0, 2], [0, 1, 2]])
def test_segmented_nan_guard_matches_per_complex_guard(where):
    from diffdock_b200.sampling import _nan_guard, _nan_guard_packed
    poses, bonds = [3, 2, 4], [6, 0, 8]
    parts = [list(_scores(10 + k, p, b)) for k, (p, b) in enumerate(zip(poses, bonds))]
    for k in where:
        tr, rot, tor = parts[k]
        tr[1, 0] = float('nan')
        rot[0, 2], rot[-1, 1] = float('inf'), float('nan')
        if tor.numel():
            tor[0], tor[2], tor[-1] = float('-inf'), float('nan'), float('inf')
    ptr = torch.tensor([0, 3, 5, 9])
    bptr = torch.tensor([0, 6, 6, 14])
    got = _nan_guard_packed(*[torch.cat([p[i] for p in parts]) for i in range(3)], ptr, bptr)
    for k in range(3):
        want = _nan_guard(*parts[k])
        sl = [slice(ptr[k], ptr[k + 1])] * 2 + [slice(bptr[k], bptr[k + 1])]
        for i in range(3):
            a, b = got[i][sl[i]], want[i]
            if k not in where:
                assert torch.equal(a, b)                             # untouched complexes: bit-identical
            else:
                assert torch.allclose(a, b, rtol=1e-6, atol=0, equal_nan=True), (k, i)


# ---------------------------------------------------------------------------------------------------------------------
def test_library_exports_the_packed_pose_update(built_lib):
    out = subprocess.run(['nm', '-D', '--defined-only', os.path.join(ROOT, 'diffdock_b200', 'libdiffdock_b200.so')],
                         capture_output=True, text=True, check=True).stdout
    assert re.search(r'\bT ddb200_pose_update_packed\b', out)
    from diffdock_b200 import _lib
    assert 'ddb200_pose_update_packed' in _lib.SIGNATURES


def test_pose_kernel_has_no_spill():
    """The pose kernel keeps its working set in registers: no spill, and no stack beyond the 28-32 bytes the CUDA math
    library's sinf / cosf reserve for the Payne-Hanek reduction of huge arguments (replacing them would change results
    that must stay bit-identical)."""
    import __graft_entry__ as ge
    src = os.path.join(ROOT, 'diffdock_b200', 'csrc', 'pose.cu')
    r = subprocess.run([ge._nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v',
                        '-c', src, '-o', os.devnull], capture_output=True, text=True, check=True, cwd=ROOT)
    text = r.stderr
    i = text.index('pose_update_kernel')
    props = text[i:i + 600]
    m = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', props)
    assert m, props
    stack, st, ld = map(int, m.groups())
    assert st == 0 and ld == 0 and stack <= 32, props

"""CPU: the pose metrics of evaluation (diffdock_b200/evaluation.py, oracle/metrics.py) against tests/golden/ref_pose_metrics.pt,
recorded from spyrmsd's symmrmsd (networkx backend) and evaluate.py's expressions: the host automorphism enumeration, the
float64 oracle, the enumeration cap, the heavy-atom inputs of a ligand graph, and the C ABI declaration and machine code of
ddb200_pose_metrics."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle.metrics import pose_metrics as oracle_metrics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'ref_pose_metrics.pt')
CASES = torch.load(GOLDEN, weights_only=False)['cases']


@pytest.mark.parametrize('name', sorted(CASES))
def test_automorphisms_equal_spyrmsd_enumeration(name):
    from diffdock_b200.evaluation import ligand_automorphisms
    c = CASES[name]
    table, corrected = ligand_automorphisms(c['atomic_nums'], c['bonds'])
    want = c['automorphisms'].long()
    assert corrected and table.dtype == torch.int32 and table.shape == want.shape
    assert {tuple(r) for r in table.tolist()} == {tuple(r) for r in want.tolist()}
    assert torch.equal(table.long(), want)           # and in spyrmsd's order, so a tie resolves to the same row


def test_fixture_covers_the_symmetries_it_is_for():
    m = {k: c['automorphisms'].shape[0] for k, c in CASES.items()}
    assert m['chain'] == 1 and m['benzene'] == 12 and m['biphenyl'] == 8 and m['adamantane'] == 24
    assert m['tetra_tert_butylbenzene'] == 5184 and m['single_atom'] == 1
    assert sum(c['refs'].shape[0] > 1 for c in CASES.values()) >= 2
    # the permuted poses are won by a non-identity automorphism
    benz = CASES['benzene']
    assert not torch.equal(benz['best_permutation'][0, 0], torch.arange(6))


@pytest.mark.parametrize('name', sorted(CASES))
def test_oracle_reproduces_fixture(name):
    c = CASES[name]
    got = oracle_metrics(c['poses'].numpy(), c['refs'].numpy(), c['automorphisms'].numpy())
    for k in ('rmsd', 'rmsd_min', 'centroid_distance', 'min_self_distance'):
        want = c[k].numpy()
        assert got[k].shape == want.shape, k
        fin = np.isfinite(want)
        assert np.array_equal(fin, np.isfinite(got[k])), k
        assert np.abs(got[k][fin] - want[fin]).max(initial=0) <= 1e-12, (k, np.abs(got[k][fin] - want[fin]).max())
    # the oracle's best row attains the minimum, and so does spyrmsd's permutation
    aut, poses, refs = c['automorphisms'].numpy().astype(np.int64), c['poses'].numpy(), c['refs'].numpy()
    n = poses.shape[1]
    for p in range(poses.shape[0]):
        a = got['best_automorphism'][p]
        s = min(np.sum((refs[g] - poses[p][aut[a]]) ** 2) for g in range(refs.shape[0]))
        assert abs(np.sqrt(s / n) - got['rmsd_min'][p]) <= 1e-12
        for g in range(refs.shape[0]):
            perm = c['best_permutation'][g, p].numpy()
            assert abs(np.sqrt(np.sum((refs[g] - poses[p][perm]) ** 2) / n) - c['rmsd'][g, p].item()) <= 1e-12


def test_cap_falls_back_to_the_identity_and_flags_the_complex():
    from diffdock_b200.evaluation import ligand_automorphisms
    c = CASES['benzoate']
    table, corrected = ligand_automorphisms(c['atomic_nums'], c['bonds'], max_count=3)
    assert not corrected and torch.equal(table, torch.arange(9, dtype=torch.int32)[None])
    full, corrected = ligand_automorphisms(c['atomic_nums'], c['bonds'], max_count=4)
    assert corrected and full.shape == (4, 9)
    # scored with the identity alone: evaluate.py:481's uncorrected RMSD
    poses, refs = c['poses'].numpy(), c['refs'].numpy()
    got = oracle_metrics(poses, refs, table.numpy())
    want = np.stack([np.sqrt(((poses - refs[i]) ** 2).sum(axis=2).mean(axis=1)) for i in range(len(refs))])
    assert np.abs(got['rmsd'] - want).max() <= 1e-12
    assert (got['rmsd_min'] >= c['rmsd_min'].numpy() - 1e-12).all()
    assert (got['rmsd_min'] > c['rmsd_min'].numpy() + 1e-3).any()       # the correction mattered here
    tbb = CASES['tetra_tert_butylbenzene']
    table, corrected = ligand_automorphisms(tbb['atomic_nums'], tbb['bonds'], max_count=1000)
    assert not corrected and table.shape == (1, 22)


def test_ligand_inputs_keep_heavy_atoms_and_their_bonds():
    from diffdock_b200.evaluation import ligand_automorphisms, ligand_inputs
    from diffdock_b200.hetero import HeteroGraph
    # methanol-like: C(0) O(1) with hydrogens 2-5 (feature index 0 = hydrogen), plus a 'misc' atom (index 118)
    x0 = torch.tensor([5, 7, 0, 0, 0, 0, 118])
    g = HeteroGraph()
    g['ligand'].x = torch.stack([x0, torch.zeros_like(x0)], 1)
    pairs = [(0, 1), (0, 2), (0, 3), (0, 4), (1, 5), (1, 6)]
    g['ligand', 'ligand'].edge_index = torch.tensor([[u for a, b in pairs for u in (a, b)],
                                                     [v for a, b in pairs for v in (b, a)]])
    heavy, z, bonds = ligand_inputs(g)
    assert heavy.tolist() == [0, 1, 6] and z.tolist() == [6, 8, 0]
    assert bonds.tolist() == [[0, 1], [1, 2]]
    table, corrected = ligand_automorphisms(z, bonds)
    assert corrected and table.tolist() == [[0, 1, 2]]


def test_header_declares_the_ctypes_table(built_lib):
    import ctypes as C
    from diffdock_b200 import _lib
    hdr = open(os.path.join(ROOT, 'include', 'diffdock_b200_metrics.h')).read()
    decls = {m.group(1): m.group(2) for m in re.finditer(r'\bint\s+(ddb200_\w+)\s*\(([^;]*)\)\s*;', hdr)}
    assert sorted(decls) == sorted(_lib.METRICS_SIGNATURES) == ['ddb200_pose_metrics']
    ctype = {'int64_t': C.c_int64, 'int': C.c_int, 'int32_t': C.c_int32}
    for name, params in decls.items():
        args = [a.strip() for a in params.replace('\n', ' ').split(',')]
        res, want = _lib.METRICS_SIGNATURES[name]
        assert res is C.c_int and len(args) == len(want), name
        for a, w in zip(args, want):
            t = ' '.join(a.split()[:-1])
            assert (w is C.c_void_p) if '*' in t else ctype[t.replace('const ', '')] is w, (name, a)
        assert getattr(built_lib, name) is not None
    main = open(os.path.join(ROOT, 'include', 'diffdock_b200.h')).read()
    assert not set(decls) & set(re.findall(r'\b(ddb200_\w+)\s*\(', main))
    assert not set(decls) & (set(_lib.SIGNATURES) | set(_lib.FIXED_SIGNATURES))
    from diffdock_b200.evaluation import MAX_ATOMS
    assert f'#define DDB200_METRICS_MAX_ATOMS {MAX_ATOMS}' in hdr


def test_kernel_sums_in_float64_without_a_stack(built_lib):
    if shutil.which('cuobjdump') is None:
        pytest.skip('cuobjdump not on PATH')
    lib = os.path.join(ROOT, 'diffdock_b200', 'libdiffdock_b200.so')
    out = subprocess.run(['cuobjdump', '-res-usage', lib], capture_output=True, text=True, check=True).stdout.splitlines()
    usage = [out[k + 1] for k, l in enumerate(out[:-1]) if 'pose_metrics_kernel' in l and l.lstrip().startswith('Function')]
    assert len(usage) == 1
    m = re.search(r'STACK:(\d+)', usage[0])
    assert m and int(m.group(1)) == 0, usage[0]
    import sys
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import sass_histogram as sh
    ins = next(v for k, v in sh.kernels(lib).items() if 'pose_metrics_kernel' in k)
    assert any(i.startswith(('DFMA', 'DADD', 'DMUL')) for i in ins)
    assert not any(i.startswith(('ATOM', 'RED')) for i in ins)          # no atomics: results do not depend on timing

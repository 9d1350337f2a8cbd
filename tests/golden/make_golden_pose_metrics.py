"""Golden vectors of the pose metrics of evaluation: runs the UNMODIFIED reference code
    spyrmsd/rmsd.py        symmrmsd (:209-304) with the networkx backend (spyrmsd/graphs/nx.py), called with the
                           arguments of utils/molecules_utils.py:get_symmetry_rmsd
    evaluate.py            the RMSD minimum over crystal poses (:483-484), the centroid distance (:486) and the minimum
                           self-distance (:503-505) expressions, restated verbatim below
on hand-built heavy-atom graphs and stores inputs + outputs in tests/golden/ref_pose_metrics.pt.

    python tests/golden/make_golden_pose_metrics.py

The molecules are given as atomic numbers and bonds (what ``Molecule.from_rdkit`` hands spyrmsd after RemoveAllHs);
RDKit is not needed.  Coordinates are float32 values held in float64: crystal poses from a seeded 3D layout of the graph,
sampled poses as copies of a crystal pose relabelled by a random automorphism (so a non-identity automorphism wins) plus
noise, and as rigidly moved copies.  ``ligand_pos`` is passed to the evaluate.py expressions as float64, so they are
evaluated without evaluate.py's float32 rounding of the sampled coordinates (diffdock_b200/evaluation.py).
"""
import os
import sys

import networkx as nx
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.ref_shims import REFERENCE_ROOT  # noqa: E402

sys.path.insert(0, REFERENCE_ROOT)
import spyrmsd.graph as sgraph  # noqa: E402
from spyrmsd import rmsd as srmsd  # noqa: E402

assert sgraph.match_graphs.__module__ == 'spyrmsd.graphs.nx', sgraph.match_graphs.__module__

OUT = os.path.join(ROOT, 'tests', 'golden', 'ref_pose_metrics.pt')


def ring(start, size):
    return [(start + i, start + (i + 1) % size) for i in range(size)]


def tert_butyl(anchor, start):
    """C(CH3)3 on ``anchor``: quaternary carbon ``start``, methyls start + 1 .. start + 3."""
    return [(anchor, start)] + [(start, start + k) for k in (1, 2, 3)]


def molecules():
    out = {}
    out['chain'] = ([6, 6, 7, 6, 8, 6, 16], [(i, i + 1) for i in range(6)])
    out['benzene'] = ([6] * 6, ring(0, 6))
    out['benzenesulfonate'] = ([6] * 6 + [16, 8, 8, 8], ring(0, 6) + [(0, 6), (6, 7), (6, 8), (6, 9)])
    out['benzoate'] = ([6] * 7 + [8, 8], ring(0, 6) + [(0, 6), (6, 7), (6, 8)])
    out['biphenyl'] = ([6] * 12, ring(0, 6) + ring(6, 6) + [(0, 6)])
    # adamantane: bridgeheads 0-3, one CH2 (4-9) between every pair of bridgeheads
    pairs = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]
    out['adamantane'] = ([6] * 10, [b for k, (u, v) in enumerate(pairs) for b in ((u, 4 + k), (4 + k, v))])
    # 1,2,4,5-tetra-tert-butylbenzene: 4 x 3! methyl permutations x 4 ring symmetries = 5184 automorphisms
    bonds = ring(0, 6)
    for k, anchor in enumerate((0, 1, 3, 4)):
        bonds += tert_butyl(anchor, 6 + 4 * k)
    out['tetra_tert_butylbenzene'] = ([6] * 22, bonds)
    out['single_atom'] = ([8], [])
    return out


# crystal poses and sampled poses per molecule
N_REFS = {'benzoate': 3, 'biphenyl': 2}
N_POSES = {'tetra_tert_butylbenzene': 4, 'single_atom': 1}


def f32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def random_rotation(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def main():
    rng = np.random.default_rng(20261018)
    cases = {}
    for name, (z, bonds) in molecules().items():
        n = len(z)
        z = np.asarray(z, dtype=np.int64)
        am = np.zeros((n, n), dtype=int)
        for u, v in bonds:
            am[u, v] = am[v, u] = 1
        g = nx.Graph()
        g.add_nodes_from(range(n))
        g.add_edges_from(bonds)
        lay = nx.spring_layout(g, dim=3, seed=int(rng.integers(1 << 30))) if n > 1 else {0: np.zeros(3)}
        base = np.stack([lay[i] for i in range(n)]) * 1.5 * max(1.0, n ** (1 / 3))
        refs = f32([base + (0 if k == 0 else rng.normal(scale=0.6, size=base.shape)) for k in range(N_REFS.get(name, 1))])

        # spyrmsd's own enumeration (what symmrmsd does with these arguments), as (idx1, idx2) pairs
        G1 = sgraph.graph_from_adjacency_matrix(am, z)
        isos = sgraph.match_graphs(G1, G1)
        perms = np.empty((len(isos), n), dtype=np.int64)
        for a, (i1, i2) in enumerate(isos):
            perms[a, np.asarray(i1)] = np.asarray(i2)

        P = N_POSES.get(name, 5)
        poses = []
        for p in range(P):
            ref = refs[p % len(refs)]
            if p % 3 == 2:            # rigidly moved copy of a crystal pose
                pose = (ref - ref.mean(0)) @ random_rotation(rng).T + ref.mean(0) + rng.normal(scale=1.0, size=3)
            else:                     # relabelled by a (non-identity where one exists) automorphism, perturbed
                s = perms[int(rng.integers(1, len(perms))) if len(perms) > 1 else 0]
                pose = np.empty_like(ref)
                pose[s] = ref + rng.normal(scale=0.05 if p % 3 == 0 else 0.3, size=ref.shape)
            poses.append(pose)
        ligand_pos = f32(poses)
        orig_ligand_pos = refs

        # evaluate.py:474-484, with get_symmetry_rmsd's call
        rmsds, best = [], []
        for i in range(len(orig_ligand_pos)):
            r, min_iso = srmsd.symmrmsd(orig_ligand_pos[i], [l for l in ligand_pos], z, z, am, am, return_permutation=True)
            rmsds.append(r)
            best.append([np.asarray(m[1])[np.argsort(m[0])] if m is not None else np.full(n, -1) for m in min_iso])
        rmsds = np.asarray(rmsds)
        rmsd = np.min(rmsds, axis=0)
        # evaluate.py:486
        centroid_distance = np.min(np.linalg.norm(ligand_pos.mean(axis=1)[None, :] - orig_ligand_pos.mean(axis=1)[:, None],
                                                  axis=2), axis=0)
        # evaluate.py:503-505
        self_distances = np.linalg.norm(ligand_pos[:, :, None, :] - ligand_pos[:, None, :, :], axis=-1)
        self_distances = np.where(np.eye(self_distances.shape[2]), np.inf, self_distances)
        min_self_distance = np.min(self_distances, axis=(1, 2))

        ident = np.all(perms == np.arange(n), axis=1)
        cases[name] = {
            'atomic_nums': torch.from_numpy(z), 'bonds': torch.tensor(bonds, dtype=torch.int64).reshape(-1, 2),
            'refs': torch.from_numpy(orig_ligand_pos), 'poses': torch.from_numpy(ligand_pos),
            'automorphisms': torch.from_numpy(perms.astype(np.int8)),
            'rmsd': torch.from_numpy(rmsds), 'rmsd_min': torch.from_numpy(rmsd),
            'centroid_distance': torch.from_numpy(centroid_distance),
            'min_self_distance': torch.from_numpy(min_self_distance),
            'best_permutation': torch.from_numpy(np.asarray(best, dtype=np.int64)),      # [G, P, n], spyrmsd's min_iso
        }
        wins = int(sum(not ident[np.flatnonzero((perms == b).all(1))[0]] for row in best for b in row if b[0] >= 0))
        print(f"{name:26s} n={n:3d} M={len(perms):5d} G={len(refs)} P={P}  non-identity minima: {wins}")
    torch.save({'cases': cases, 'source': 'spyrmsd symmrmsd (networkx backend) + evaluate.py:474-505 expressions'}, OUT)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()

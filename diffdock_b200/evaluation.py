"""Pose metrics of evaluation on the device: drop-in for the per-complex scoring of ``evaluate.py:414-431,474-486,503-505``
(symmetry-corrected RMSD against every crystal pose through spyrmsd, centroid distances, minimum intra-ligand distances).

* ``ligand_inputs`` turns a ligand graph into the heavy-atom inputs (``filterHs``, atomic numbers, heavy-atom bonds);
* ``ligand_automorphisms`` enumerates the molecule's automorphisms once, on the host, with networkx's ``GraphMatcher`` as
  spyrmsd's networkx backend does (``spyrmsd/graphs/nx.py:match_graphs``);
* ``pose_metrics`` / ``pose_metrics_packed`` score poses of one / many complexes in one launch of ddb200_pose_metrics
  (include/diffdock_b200_metrics.h): float64 sums, order-independent, no host synchronisation.

Semantics (spyrmsd ``symmrmsd(ref, poses, a, a, am, am, center=False, minimize=False, cache=True)`` per crystal pose,
then evaluate.py's minimum over crystal poses):
  rmsd[g, p]            = sqrt(min over automorphisms s of sum_i |ref_g[i] - pose_p[s[i]]|^2 / n)
  rmsd_min[p]           = min_g rmsd[g, p]
  centroid_distance[p]  = min_g |mean(pose_p) - mean(ref_g)|
  min_self_distance[p]  = min_{i != j} |pose_p[i] - pose_p[j]|        (+inf for one atom)
all evaluated in float64 from the float32 poses.  evaluate.py evaluates the last one and the pose centroids on its float32
``ligand_pos`` array in float32; the values here are those expressions without the float32 rounding.

One divergence, on purpose: the reference enumerates isomorphisms under a 10 s wall-clock alarm
(``utils/molecules_utils.py:get_symmetry_rmsd``) and, on timeout or any error, prints a message and scores the complex
with the uncorrected RMSD (``evaluate.py:479-481``).  Here the enumeration stops at a deterministic count
(``max_count``); past it the complex is scored with the identity mapping only, which is the uncorrected RMSD, and flagged
``corrected=False`` - the same outcome, reached the same way on every machine."""
from __future__ import annotations

from typing import List, NamedTuple

import networkx as nx
import numpy as np
import torch

from . import _lib
from .ops import _need_cuda, _ptr, _stream

MAX_ATOMS = 1024                    # DDB200_METRICS_MAX_ATOMS of include/diffdock_b200_metrics.h
MAX_AUTOMORPHISMS = 100_000         # default enumeration cap of ligand_automorphisms


class PoseMetrics(NamedTuple):
    """Metrics of the P sampled poses of one complex against its G crystal poses (device tensors, float64 / int32)."""
    rmsd: torch.Tensor                # [G, P] symmetry-corrected RMSD against each crystal pose
    rmsd_min: torch.Tensor            # [P] minimum over the crystal poses
    centroid_distance: torch.Tensor   # [P] minimum over the crystal poses
    min_self_distance: torch.Tensor   # [P]
    best_automorphism: torch.Tensor   # [P] row of the automorphism table that attains rmsd_min (-1: none below +inf)


def ligand_inputs(graph):
    """The heavy-atom inputs of one ligand graph (a ``HeteroGraph`` with ``['ligand'].x`` and the ``('ligand', 'ligand')``
    bond edges): ``(heavy [n] int64, atomic_nums [n] int64, bonds [B, 2] int64)``, on the host.  ``heavy`` is
    ``evaluate.py:414``'s ``filterHs = x[:, 0] != 0`` as indices, in atom order; the atomic number of feature index k is
    k + 1 (``datasets/process_mols.py:lig_atom_featurizer``, ``possible_atomic_num_list = 1 .. 118, 'misc'``), and the
    'misc' index, which the featurizer gives atomic numbers outside 1 .. 118, is read as 0; ``bonds`` are the bond edges
    between heavy atoms in heavy-atom numbering, each bond once with u < v."""
    x0 = graph['ligand'].x[:, 0].detach().cpu().long()
    keep = x0 != 0
    heavy = torch.nonzero(keep).flatten()
    z = x0[heavy] + 1
    z = torch.where(z > 118, torch.zeros_like(z), z)
    ei = graph['ligand', 'ligand'].edge_index.detach().cpu().long()
    local = torch.full((x0.shape[0],), -1, dtype=torch.long)
    local[heavy] = torch.arange(heavy.shape[0])
    u, v = local[ei[0]], local[ei[1]]
    ok = (u >= 0) & (v >= 0) & (u != v)
    pairs = torch.stack([torch.minimum(u[ok], v[ok]), torch.maximum(u[ok], v[ok])], 1)
    bonds = torch.unique(pairs, dim=0) if pairs.numel() else pairs.reshape(0, 2)
    return heavy, z, bonds


def ligand_automorphisms(atomic_nums, bonds, max_count=MAX_AUTOMORPHISMS):
    """Every automorphism of the molecular graph (nodes 0 .. n-1 labelled by atomic number, edges = bonds without bond
    order), in the order networkx's ``GraphMatcher(G, G, node_match=atomic numbers equal).isomorphisms_iter()`` yields
    them, as spyrmsd enumerates them.  Returns ``(table int32 [M, n], corrected)``: row a maps crystal atom i to pose atom
    ``table[a, i]`` (spyrmsd's ``(idx1, idx2)`` pair sorted by idx1).  Past ``max_count`` automorphisms the enumeration
    stops and the table is the identity alone with ``corrected=False``: the complex is then scored with the uncorrected
    RMSD, ``evaluate.py:479-481``'s fallback, at a count instead of a 10 s alarm."""
    z = [int(a) for a in np.asarray(atomic_nums).reshape(-1)]
    n = len(z)
    if n < 1:
        raise ValueError("a molecule needs at least one heavy atom")
    b = np.asarray(bonds, dtype=np.int64).reshape(-1, 2)
    if b.size and (b.min() < 0 or b.max() >= n):
        raise ValueError("bond outside the molecule")
    am = np.zeros((n, n), dtype=np.int64)
    am[b[:, 0], b[:, 1]] = am[b[:, 1], b[:, 0]] = 1
    # built from the adjacency matrix as spyrmsd builds it, so the matcher yields the same automorphisms in the same order
    g = nx.Graph(am)
    nx.set_node_attributes(g, dict(enumerate(z)), 'aprops')
    gm = nx.algorithms.isomorphism.GraphMatcher(g, g, node_match=lambda a, c: a['aprops'] == c['aprops'])
    rows = []
    for m in gm.isomorphisms_iter():
        if len(rows) == max_count:
            return torch.arange(n, dtype=torch.int32)[None], False
        rows.append([m[i] for i in range(n)])
    return torch.tensor(rows, dtype=torch.int32).reshape(-1, n), True


def heavy_poses(data_list, heavy):
    """The heavy atoms of each pose's ligand coordinates, stacked on the poses' device: [P, n, 3] float32 (a device gather,
    no host copy).  ``data_list``: the poses of one complex as ``sampling`` / ``sample_packed`` return them."""
    pos = torch.stack([d['ligand'].pos for d in data_list])
    return pos.index_select(1, heavy.to(pos.device))


def pose_metrics(poses, refs, automorphisms) -> PoseMetrics:
    """Metrics of one complex: ``poses`` [P, n, 3] float32 on the device, ``refs`` [G, n, 3] float64 (float32 is widened),
    ``automorphisms`` [M, n] int32 (``ligand_automorphisms``).  ``refs`` and ``automorphisms`` are uploaded with
    non-blocking copies if they are on the host (a host table is checked to hold permutations); one launch, nothing is
    read back.  On the device, an entry outside [0, n) gives NaN RMSDs for the poses that read it."""
    return pose_metrics_packed([poses], [refs], [automorphisms])[0]


def pose_metrics_packed(poses: List[torch.Tensor], refs: List[torch.Tensor], automorphisms: List[torch.Tensor]
                        ) -> List[PoseMetrics]:
    """``pose_metrics`` of K complexes in ONE launch: lists of per-complex ``poses`` [P_k, n_k, 3], ``refs`` [G_k, n_k, 3]
    and ``automorphisms`` [M_k, n_k].  The inputs are concatenated on the device; the per-pose descriptor (the layout of
    ddb200_pose_metrics) is built from the shapes on the host and uploaded without a synchronisation, so nothing is read
    back.  A complex's results are bit-identical to its own ``pose_metrics`` call.  Returns one ``PoseMetrics`` per complex
    (views of the launch's output buffers)."""
    K = len(poses)
    if len(refs) != K or len(automorphisms) != K:
        raise ValueError("one refs tensor and one automorphism table per complex")
    if K == 0:
        return []
    dev = poses[0].device
    _need_cuda(*poses)
    rows, pos_cat, ref_cat, aut_cat = [], [], [], []
    pos_off = ref_off = aut_off = rmsd_off = 0
    max_atoms = 0
    for p, r, a in zip(poses, refs, automorphisms):
        if p.dim() != 3 or p.shape[2] != 3 or r.dim() != 3 or r.shape[1:] != p.shape[1:] or a.dim() != 2:
            raise ValueError(f"poses [P, n, 3], refs [G, n, 3], automorphisms [M, n]: got {tuple(p.shape)}, "
                             f"{tuple(r.shape)}, {tuple(a.shape)}")
        P, n, G, M = p.shape[0], p.shape[1], r.shape[0], a.shape[0]
        if a.shape[1] != n or n < 1 or n > MAX_ATOMS or G < 1 or M < 1:
            raise ValueError(f"a complex with {n} heavy atoms (1 .. {MAX_ATOMS}), {G} crystal poses and an automorphism "
                             f"table of shape {tuple(a.shape)}")
        if not a.is_cuda and not torch.equal(a.sort(1).values.long(), torch.arange(n).expand(M, n)):
            raise ValueError("every automorphism table row must be a permutation of 0 .. n-1")
        for i in range(P):
            rows.append([pos_off + i * n, n, ref_off, G, aut_off, M, rmsd_off + i, P])
        pos_cat.append(p.to(device=dev, dtype=torch.float32).reshape(-1, 3))
        ref_cat.append(r.to(device=dev, dtype=torch.float64, non_blocking=True).reshape(-1, 3))
        aut_cat.append(a.to(device=dev, dtype=torch.int32, non_blocking=True).reshape(-1))
        pos_off, ref_off, aut_off, rmsd_off = pos_off + P * n, ref_off + G * n, aut_off + M * n, rmsd_off + G * P
        max_atoms = max(max_atoms, n)
    if max(pos_off, ref_off, aut_off, rmsd_off) >= 2 ** 31:
        raise ValueError("packed metrics input too large for int32 offsets")
    n_poses = len(rows)
    layout = torch.tensor(rows, dtype=torch.int32).reshape(-1, 8).to(dev, non_blocking=True)
    pos = torch.cat(pos_cat).contiguous()
    ref = torch.cat(ref_cat).contiguous()
    aut = torch.cat(aut_cat).contiguous()
    rmsd = torch.empty(rmsd_off, dtype=torch.float64, device=dev)
    per_pose = torch.empty((3, n_poses), dtype=torch.float64, device=dev)
    best = torch.empty(n_poses, dtype=torch.int32, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    rc = _lib.lib().ddb200_pose_metrics(_ptr(pos), _ptr(ref), _ptr(aut), _ptr(layout), n_poses, max_atoms, _ptr(rmsd),
                                        _ptr(per_pose[0]), _ptr(per_pose[1]), _ptr(per_pose[2]), _ptr(best), _ptr(err),
                                        _stream())
    _lib.check(rc, 'ddb200_pose_metrics')
    out, p0, r0 = [], 0, 0
    for p, r in zip(poses, refs):
        P, G = p.shape[0], r.shape[0]
        out.append(PoseMetrics(rmsd[r0:r0 + G * P].view(G, P), per_pose[0, p0:p0 + P], per_pose[1, p0:p0 + P],
                               per_pose[2, p0:p0 + P], best[p0:p0 + P]))
        p0, r0 = p0 + P, r0 + G * P
    return out

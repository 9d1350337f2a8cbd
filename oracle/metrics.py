"""float64 CPU restatement of the pose metrics of evaluation (diffdock_b200/evaluation.py, include/diffdock_b200_metrics.h):
spyrmsd's ``_rmsd_isomorphic_core`` loop over automorphisms (center=False, minimize=False) per pose and crystal pose, and
evaluate.py's centroid-distance and minimum self-distance expressions, brute force, one pose at a time."""
import numpy as np


def pose_metrics(poses, refs, automorphisms):
    """``poses`` [P, n, 3], ``refs`` [G, n, 3], ``automorphisms`` [M, n] (row a maps crystal atom i to pose atom
    ``automorphisms[a, i]``).  Returns a dict of numpy arrays: rmsd [G, P], rmsd_min [P], centroid_distance [P],
    min_self_distance [P], best_automorphism [P] (lowest crystal pose, then lowest row, among equal minima; -1 if none is
    below +inf)."""
    poses = np.asarray(poses, dtype=np.float64)
    refs = np.asarray(refs, dtype=np.float64)
    aut = np.asarray(automorphisms, dtype=np.int64)
    P, n = poses.shape[0], poses.shape[1]
    G = refs.shape[0]
    rmsd = np.empty((G, P))
    best_sq = np.full(P, np.inf)
    best_aut = np.full(P, -1, dtype=np.int64)
    for p in range(P):
        for g in range(G):
            m_best, a_best = np.inf, -1
            for a in range(aut.shape[0]):
                s = np.sum((refs[g] - poses[p][aut[a]]) ** 2)
                if s < m_best:
                    m_best, a_best = s, a
            rmsd[g, p] = np.sqrt(m_best / n)
            if m_best < best_sq[p]:
                best_sq[p], best_aut[p] = m_best, a_best
    centroid = np.min(np.linalg.norm(poses.mean(axis=1)[None, :] - refs.mean(axis=1)[:, None], axis=2), axis=0)
    d = np.linalg.norm(poses[:, :, None, :] - poses[:, None, :, :], axis=-1)
    d = np.where(np.eye(n, dtype=bool), np.inf, d)
    return {'rmsd': rmsd, 'rmsd_min': rmsd.min(axis=0), 'centroid_distance': centroid,
            'min_self_distance': d.min(axis=(1, 2)), 'best_automorphism': best_aut}

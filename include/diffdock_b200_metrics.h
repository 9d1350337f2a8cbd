/*
 * diffdock_b200 - C ABI of the pose metrics of evaluation (sm_90a).  Conventions as include/diffdock_b200.h (caller-owned
 * device pointers, the caller's stream, int status return, no implicit synchronisation).  Kept out of the main header,
 * whose ctypes table the launch-replay tests pin to the score and confidence paths.
 */
#ifndef DIFFDOCK_B200_METRICS_H
#define DIFFDOCK_B200_METRICS_H

#include <stdint.h>

#include "diffdock_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------------------------------
 * ddb200_pose_metrics: symmetry-corrected RMSD, centroid distance and minimum self-distance of sampled poses against
 * crystal poses, for poses of any number of complexes in one launch.  Row b of the DEVICE descriptor layout
 * [n_poses, 8] (int32) gives pose b's
 *   pos_off, n          its heavy atoms are rows pos_off .. pos_off + n - 1 of pos [*, 3] (float32);
 *   ref_off, n_refs     crystal pose g is rows ref_off + g n .. ref_off + g n + n - 1 of refs [*, 3] (float64);
 *   aut_off, n_aut      automorphism a is aut[aut_off + a n .. aut_off + a n + n - 1] (int32): crystal atom i is matched
 *                       with pose atom aut[aut_off + a n + i];
 *   rmsd_off, rmsd_ld   rmsd[rmsd_off + g rmsd_ld] receives the RMSD against crystal pose g.
 * In float64, with no centring and no superposition (spyrmsd's symmrmsd with center=False, minimize=False):
 *   s[g][a]              = sum_i |ref_g[i] - pose[aut_a[i]]|^2
 *   rmsd[g]              = sqrt(min_a s[g][a] / n)
 *   rmsd_min[b]          = min_g rmsd[g];  best_aut[b] = the a attaining it (lowest g, then lowest a, among equal values;
 *                          -1 when no s is below +inf, e.g. a NaN coordinate: the RMSD is then +inf, as spyrmsd gives)
 *   centroid_dist[b]     = min_g |mean(pose) - mean(ref_g)|
 *   min_self_dist[b]     = min_{i != j} |pose[i] - pose[j]|   (+inf for one atom)
 * Every sum has a fixed order and there are no atomics: two calls give bit-identical results, and a pose's results do not
 * depend on the other poses of the launch.  The host does not read the descriptor: max_atoms (>= every pose's n, at most
 * DDB200_METRICS_MAX_ATOMS) sizes the shared memory.  A pose with n outside [1, max_atoms], n_refs or n_aut below 1, or
 * an automorphism entry outside [0, n) gets NaN results and sets *err (device int32) to 1; the caller zeroes it.
 * Replaces: evaluate.py:474-486 and :503-505 (utils/molecules_utils.py:get_symmetry_rmsd per crystal pose, the
 * centroid distances and the minimum intra-ligand distances), given the automorphisms spyrmsd enumerates.
 * ------------------------------------------------------------------------------------------------------------- */
#define DDB200_METRICS_MAX_ATOMS 1024
int ddb200_pose_metrics(const float* pos, const double* refs, const int32_t* aut, const int32_t* layout, int64_t n_poses,
                        int32_t max_atoms, double* rmsd, double* rmsd_min, double* centroid_dist, double* min_self_dist,
                        int32_t* best_aut, int32_t* err, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DIFFDOCK_B200_METRICS_H */

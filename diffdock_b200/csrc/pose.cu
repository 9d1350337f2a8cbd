// Reverse-diffusion pose update, one CTA per pose (replaces utils/sampling.py:133-191 perturbation arithmetic,
// utils/diffusion_utils.py:60-78 modify_conformer_batch, utils/torsion.py:75-90 sequential bond rotations and
// utils/geometry.py:246-276 batched Kabsch - a Python loop over rotatable bonds with host-sync asserts and a cuSOLVER
// batched SVD in the reference).
//
// Per pose b (all poses of a batch are copies of one ligand, as in the reference's sampler, or - packed - each pose with its
// own ligand layout):
//   perturb = a * score + c * z                       (a, c: host scalars of the SDE step, one pair per dof type)
//   rigid   = R(rot) (pos - centroid) + tr + centroid (axis-angle -> quaternion -> matrix, pytorch3d formulas)
//   flex    = rigid, then for every rotatable bond r in order: atoms of mask[r] rotate about pos[u]-pos[v] through
//             pos[v] by tor[r] (later bonds see updated coordinates)
//   out     = Kabsch-align flex onto rigid (rotation from the two leading singular directions of the 3x3 covariance,
//             third ones by cross products => proper rotation, identical to the SVD + reflection-fix formula)
// The 3x3 covariance / eigen problem runs in fp64 (a few hundred flops per pose).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/diffdock_b200.h"

namespace {

__device__ __forceinline__ void axis_angle_to_matrix(float ax, float ay, float az, float* M) {
  // utils/geometry.py:36-86
  const float ang = sqrtf(ax * ax + ay * ay + az * az);
  const float half = 0.5f * ang;
  const float s = (fabsf(ang) < 1e-6f) ? (0.5f - ang * ang / 48.f) : (sinf(half) / ang);
  const float r = cosf(half), i = ax * s, j = ay * s, k = az * s;
  const float two_s = 2.0f / (r * r + i * i + j * j + k * k);
  M[0] = 1 - two_s * (j * j + k * k); M[1] = two_s * (i * j - k * r);     M[2] = two_s * (i * k + j * r);
  M[3] = two_s * (i * j + k * r);     M[4] = 1 - two_s * (i * i + k * k); M[5] = two_s * (j * k - i * r);
  M[6] = two_s * (i * k - j * r);     M[7] = two_s * (j * k + i * r);     M[8] = 1 - two_s * (i * i + j * j);
}

__device__ __forceinline__ void block_sum(double* vals, int n, double* red, int tid, int nthreads) {
  // vals: per-thread partials (n of them); result broadcast in red[0..n).  Inlined with a constant n, so that vals stays in
  // registers.
#pragma unroll
  for (int q = 0; q < n; ++q) {
    double v = vals[q];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((tid & 31) == 0) red[32 * q + (tid >> 5)] = v;
  }
  __syncthreads();
  if (tid < n) {
    double v = 0;
    for (int w = 0; w < (nthreads >> 5); ++w) v += red[32 * tid + w];
    red[32 * n + tid] = v;
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < n; ++q) vals[q] = red[32 * n + q];
  __syncthreads();
}

__device__ __forceinline__ void swap3(double a[3], double b[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) { const double t = a[c]; a[c] = b[c]; b[c] = t; }
}

// Jacobi eigen-decomposition of a symmetric 3x3 (fp64): A = V diag(w) V^T.  Every index is a compile-time constant after
// unrolling, so A and V stay in registers.
__device__ __forceinline__ void jacobi3(double A[3][3], double V[3][3], double w[3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) V[i][j] = (i == j);
  for (int sweep = 0; sweep < 30; ++sweep) {
    const double off = fabs(A[0][1]) + fabs(A[0][2]) + fabs(A[1][2]);
    if (off < 1e-300 || off < 1e-18 * (fabs(A[0][0]) + fabs(A[1][1]) + fabs(A[2][2]))) break;
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
      for (int q = p + 1; q < 3; ++q) {
        if (fabs(A[p][q]) < 1e-300) continue;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - s * akq;
          A[k][q] = s * akp + c * akq;
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - s * aqk;
          A[q][k] = s * apk + c * aqk;
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq;
          V[k][q] = s * vkp + c * vkq;
        }
      }
  }
  for (int i = 0; i < 3; ++i) w[i] = A[i][i];
}

// ---- counter-based noise (Philox4x32-10, Salmon et al. 2011): one stream per pose, keyed by (seed, complex id, pose id) and
// indexed by (step, degree of freedom), so a sampling run draws the same noise whatever the batch split or GPU count
// (SURVEY.md section 8(e)).  The reference draws torch.normal blocks per batch (utils/sampling.py:140-145).
__device__ __forceinline__ void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}
// four standard normals from one Philox block (Box-Muller on two pairs of 24-bit uniforms in (0, 1))
__device__ __forceinline__ void philox_normal4(uint64_t seed, long long pose_key, uint32_t step, uint32_t block, float z[4]) {
  uint32_t c[4] = {(uint32_t)pose_key, (uint32_t)((unsigned long long)pose_key >> 32), step, block};
  philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float u1 = (float)(c[2 * h] >> 8) * 5.9604644775390625e-8f + 2.98023223876953125e-8f;      // (k + 0.5) / 2^24
    const float u2 = (float)(c[2 * h + 1] >> 8) * 5.9604644775390625e-8f + 2.98023223876953125e-8f;
    const float rad = sqrtf(-2.0f * logf(u1));
    float sn, cs;
    sincosf(6.283185307179586f * u2, &sn, &cs);
    z[2 * h] = rad * cs; z[2 * h + 1] = rad * sn;
  }
}

struct PoseNoise {
  const float* coef_dev;        // optional device table [*, 6]; row *step_dev (or 0)
  const int* step_dev;          // optional device scalar
  unsigned long long seed;      // Philox key
  const long long* pose_key;    // optional [n_poses]: (complex id << 32) | pose id  -> in-kernel noise
  int philox;
};

// Where pose b lives.  Uniform batch (layout == NULL): every pose is a copy of one ligand of n_atoms atoms and n_bonds
// rotatable bonds, pose-major.  Packed batch: row b of layout [n_poses, 6] int32 = (atom_off, n_atoms, bond_off, n_bonds,
// tor_off, mask_off): rows of pos / out, rows of bond_u / bond_v (local atom numbering), first entry in tor_score / tor_z,
// first byte of the pose's [n_bonds, n_atoms] mask block.  A packed pose with n_atoms outside [1, max_atoms] (the size the
// shared memory was sized for) or a negative bond count is left untouched and sets *err = 1.
__global__ void pose_update_kernel(const float* pos, int n_atoms, int n_bonds, const int* __restrict__ layout, int max_atoms,
                                   int* err, const int* __restrict__ bond_u, const int* __restrict__ bond_v,
                                   const unsigned char* __restrict__ mask, const float* __restrict__ tr_score,
                                   const float* __restrict__ rot_score, const float* __restrict__ tor_score,
                                   const float* __restrict__ tr_z, const float* __restrict__ rot_z,
                                   const float* __restrict__ tor_z, float a_tr, float c_tr, float a_rot, float c_rot,
                                   float a_tor, float c_tor, int use_torsion, const PoseNoise nz, float* out) {
  extern __shared__ float sm[];
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  size_t atom_off = (size_t)b * n_atoms, tor_off = (size_t)b * n_bonds;
  if (layout) {
    const int* d = layout + 6 * (size_t)b;
    atom_off = (size_t)d[0]; n_atoms = d[1]; n_bonds = d[3]; tor_off = (size_t)d[4];
    if (n_atoms < 1 || n_atoms > max_atoms || n_bonds < 0) {     // uniform over the CTA: nothing below runs
      if (tid == 0) *err = 1;
      return;
    }
    bond_u += d[2]; bond_v += d[2]; mask += d[5];
  }
  const int step = nz.step_dev ? *nz.step_dev : 0;
  if (nz.coef_dev) {         // SDE coefficients of this step from a device table: the host never touches the step loop
    const float* cf = nz.coef_dev + 6 * (long long)step;
    a_tr = cf[0]; c_tr = cf[1]; a_rot = cf[2]; c_rot = cf[3]; a_tor = cf[4]; c_tor = cf[5];
  }
  float* rig = sm;                         // [n_atoms*3]
  float* flex = rig + 3 * n_atoms;         // [n_atoms*3]
  float* mat = flex + 3 * n_atoms;         // [16]
  double* red = reinterpret_cast<double*>(mat + 16);   // [32*9 + 16]
  const float* p = pos + atom_off * 3;

  // centroid
  double part[9];
  part[0] = part[1] = part[2] = 0;
  for (int i = tid; i < n_atoms; i += nt) { part[0] += p[3 * i]; part[1] += p[3 * i + 1]; part[2] += p[3 * i + 2]; }
  block_sum(part, 3, red, tid, nt);
  const float cx = (float)(part[0] / n_atoms), cy = (float)(part[1] / n_atoms), cz = (float)(part[2] / n_atoms);

  if (tid == 0) {
    float zr[4] = {0.f, 0.f, 0.f, 0.f}, zt[4] = {0.f, 0.f, 0.f, 0.f};
    if (nz.philox) {
      philox_normal4(nz.seed, nz.pose_key[b], (uint32_t)step, 0u, zt);
      philox_normal4(nz.seed, nz.pose_key[b], (uint32_t)step, 1u, zr);
    } else {
      if (rot_z) { zr[0] = rot_z[3 * b]; zr[1] = rot_z[3 * b + 1]; zr[2] = rot_z[3 * b + 2]; }
      if (tr_z) { zt[0] = tr_z[3 * b]; zt[1] = tr_z[3 * b + 1]; zt[2] = tr_z[3 * b + 2]; }
    }
    axis_angle_to_matrix(a_rot * rot_score[3 * b] + c_rot * zr[0], a_rot * rot_score[3 * b + 1] + c_rot * zr[1],
                         a_rot * rot_score[3 * b + 2] + c_rot * zr[2], mat);
    for (int d = 0; d < 3; ++d) mat[9 + d] = a_tr * tr_score[3 * b + d] + c_tr * zt[d];
  }
  __syncthreads();
  for (int i = tid; i < n_atoms; i += nt) {
    const float x = p[3 * i] - cx, y = p[3 * i + 1] - cy, z = p[3 * i + 2] - cz;
    const float nx = mat[0] * x + mat[1] * y + mat[2] * z + mat[9] + cx;
    const float ny = mat[3] * x + mat[4] * y + mat[5] * z + mat[10] + cy;
    const float nz = mat[6] * x + mat[7] * y + mat[8] * z + mat[11] + cz;
    rig[3 * i] = nx; rig[3 * i + 1] = ny; rig[3 * i + 2] = nz;
    flex[3 * i] = nx; flex[3 * i + 1] = ny; flex[3 * i + 2] = nz;
  }
  __syncthreads();
  float* o = out + atom_off * 3;
  if (!use_torsion || n_bonds == 0) {
    for (int i = tid; i < 3 * n_atoms; i += nt) o[i] = rig[i];
    return;
  }

  // sequential torsion updates
  for (int r = 0; r < n_bonds; ++r) {
    const int u = bond_u[r], v = bond_v[r];
    const float pvx = flex[3 * v], pvy = flex[3 * v + 1], pvz = flex[3 * v + 2];
    if (tid == 0) {
      float ax = flex[3 * u] - pvx, ay = flex[3 * u + 1] - pvy, az = flex[3 * u + 2] - pvz;
      const float nrm = sqrtf(ax * ax + ay * ay + az * az);
      float zq = tor_z ? tor_z[tor_off + r] : 0.f;
      if (nz.philox) {
        float z4[4];
        philox_normal4(nz.seed, nz.pose_key[b], (uint32_t)step, 2u + (uint32_t)(r >> 2), z4);
        const int j = r & 3;                 // selected by value: a run-time index would put z4 on the stack
        zq = j == 0 ? z4[0] : j == 1 ? z4[1] : j == 2 ? z4[2] : z4[3];
      }
      const float ang = a_tor * tor_score[tor_off + r] + c_tor * zq;
      ax = ax / nrm * ang; ay = ay / nrm * ang; az = az / nrm * ang;
      axis_angle_to_matrix(ax, ay, az, mat);
    }
    __syncthreads();
    const unsigned char* mr = mask + (size_t)r * n_atoms;
    for (int i = tid; i < n_atoms; i += nt) {
      if (mr[i]) {
        const float x = flex[3 * i] - pvx, y = flex[3 * i + 1] - pvy, z = flex[3 * i + 2] - pvz;
        flex[3 * i] = mat[0] * x + mat[1] * y + mat[2] * z + pvx;
        flex[3 * i + 1] = mat[3] * x + mat[4] * y + mat[5] * z + pvy;
        flex[3 * i + 2] = mat[6] * x + mat[7] * y + mat[8] * z + pvz;
      }
    }
    __syncthreads();
  }

  // Kabsch: align flex (A) onto rig (B)
  part[0] = part[1] = part[2] = part[3] = part[4] = part[5] = 0;
  for (int i = tid; i < n_atoms; i += nt) {
    part[0] += flex[3 * i]; part[1] += flex[3 * i + 1]; part[2] += flex[3 * i + 2];
    part[3] += rig[3 * i]; part[4] += rig[3 * i + 1]; part[5] += rig[3 * i + 2];
  }
  block_sum(part, 6, red, tid, nt);
  const double cA[3] = {part[0] / n_atoms, part[1] / n_atoms, part[2] / n_atoms};
  const double cB[3] = {part[3] / n_atoms, part[4] / n_atoms, part[5] / n_atoms};
  for (int q = 0; q < 9; ++q) part[q] = 0;
  for (int i = tid; i < n_atoms; i += nt) {
    const double a[3] = {flex[3 * i] - cA[0], flex[3 * i + 1] - cA[1], flex[3 * i + 2] - cA[2]};
    const double bb[3] = {rig[3 * i] - cB[0], rig[3 * i + 1] - cB[1], rig[3 * i + 2] - cB[2]};
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) part[3 * r + c] += a[r] * bb[c];     // H = Am Bm^T
  }
  block_sum(part, 9, red, tid, nt);
  if (tid == 0) {
    double H[3][3], K[3][3], V[3][3], w[3];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) H[r][c] = part[3 * r + c];
    // H = U S Vt ; R = V diag(1,1,d) U^T.  Eigenvectors of K = H H^T are the columns of U; v_i = H^T u_i / s_i.
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) K[r][c] = H[r][0] * H[c][0] + H[r][1] * H[c][1] + H[r][2] * H[c][2];
    jacobi3(K, V, w);
    // sort eigenvalues descending, moving the eigenvectors by value (no indexing by a run-time index: registers only)
    double u1[3] = {V[0][0], V[1][0], V[2][0]}, u2[3] = {V[0][1], V[1][1], V[2][1]}, u3s[3] = {V[0][2], V[1][2], V[2][2]};
    double w0 = w[0], w1 = w[1], w2 = w[2];
    if (w0 < w1) { const double t = w0; w0 = w1; w1 = t; swap3(u1, u2); }
    if (w0 < w2) { const double t = w0; w0 = w2; w2 = t; swap3(u1, u3s); }
    if (w1 < w2) { const double t = w1; w1 = w2; w2 = t; swap3(u2, u3s); }
    double v1[3], v2[3];
    for (int c = 0; c < 3; ++c) {
      v1[c] = H[0][c] * u1[0] + H[1][c] * u1[1] + H[2][c] * u1[2];
      v2[c] = H[0][c] * u2[0] + H[1][c] * u2[1] + H[2][c] * u2[2];
    }
    // H of rank < 2 (every atom on one line, e.g. a linear ligand whose torsions cannot move an atom off it): v2 is then
    // arbitrary in the plane orthogonal to v1, and any choice gives a rotation about that line, which moves no atom
    const double n1 = sqrt(v1[0] * v1[0] + v1[1] * v1[1] + v1[2] * v1[2]);
    for (int c = 0; c < 3; ++c) v1[c] = n1 > 0 ? v1[c] / n1 : u1[c];     // n1 = 0: H = 0, every atom at the centroid
    double d12 = v1[0] * v2[0] + v1[1] * v2[1] + v1[2] * v2[2];
    for (int c = 0; c < 3; ++c) v2[c] -= d12 * v1[c];
    double n2 = sqrt(v2[0] * v2[0] + v2[1] * v2[1] + v2[2] * v2[2]);
    if (!(n2 > 1e-10 * n1)) {        // complete the frame with the coordinate axis least aligned with v1
      int k = fabs(v1[0]) <= fabs(v1[1]) ? 0 : 1;
      double v1k = k == 0 ? v1[0] : v1[1];
      if (fabs(v1[2]) < fabs(v1k)) { k = 2; v1k = v1[2]; }
#pragma unroll
      for (int c = 0; c < 3; ++c) v2[c] = (c == k) - v1k * v1[c];
      n2 = sqrt(v2[0] * v2[0] + v2[1] * v2[1] + v2[2] * v2[2]);
    }
    for (int c = 0; c < 3; ++c) v2[c] /= n2;
    const double u3[3] = {u1[1] * u2[2] - u1[2] * u2[1], u1[2] * u2[0] - u1[0] * u2[2], u1[0] * u2[1] - u1[1] * u2[0]};
    const double v3[3] = {v1[1] * v2[2] - v1[2] * v2[1], v1[2] * v2[0] - v1[0] * v2[2], v1[0] * v2[1] - v1[1] * v2[0]};
    double Rm[3][3];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) Rm[r][c] = v1[r] * u1[c] + v2[r] * u2[c] + v3[r] * u3[c];
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) mat[3 * r + c] = (float)Rm[r][c];
      mat[9 + r] = (float)(-(Rm[r][0] * cA[0] + Rm[r][1] * cA[1] + Rm[r][2] * cA[2]) + cB[r]);
    }
  }
  __syncthreads();
  for (int i = tid; i < n_atoms; i += nt) {
    const float x = flex[3 * i], y = flex[3 * i + 1], z = flex[3 * i + 2];
    o[3 * i] = mat[0] * x + mat[1] * y + mat[2] * z + mat[9];
    o[3 * i + 1] = mat[3] * x + mat[4] * y + mat[5] * z + mat[10];
    o[3 * i + 2] = mat[6] * x + mat[7] * y + mat[8] * z + mat[11];
  }
}

// Shared-memory size for ligands of up to max_atoms atoms, the opt-in above 48 KB, the launch.
int launch_pose_update(const float* pos, int64_t n_poses, int n_atoms, int n_bonds, const int32_t* layout, int max_atoms,
                       int32_t* err, const int32_t* bond_u, const int32_t* bond_v, const uint8_t* mask_rotate,
                       const float* tr_score, const float* rot_score, const float* tor_score, const float* tr_z,
                       const float* rot_z, const float* tor_z, const float* coef6, int use_torsion, const PoseNoise& nz,
                       float* out_pos, void* stream) {
  if (n_poses == 0) return 0;
  const size_t smem = sizeof(float) * (6 * (size_t)max_atoms + 16) + sizeof(double) * (32 * 9 + 16) + 16;
  if (smem > 200 * 1024) return DDB200_ESMEM;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(pose_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
  }
  const float c0 = coef6 ? coef6[0] : 0.f, c1 = coef6 ? coef6[1] : 0.f, c2 = coef6 ? coef6[2] : 0.f;
  const float c3 = coef6 ? coef6[3] : 0.f, c4 = coef6 ? coef6[4] : 0.f, c5 = coef6 ? coef6[5] : 0.f;
  pose_update_kernel<<<(unsigned)n_poses, 128, smem, (cudaStream_t)stream>>>(
      pos, n_atoms, n_bonds, layout, max_atoms, err, bond_u, bond_v, mask_rotate, tr_score, rot_score, tor_score, tr_z,
      rot_z, tor_z, c0, c1, c2, c3, c4, c5, use_torsion, nz, out_pos);
  return (int)cudaGetLastError();
}

PoseNoise device_noise(const float* coef_table, const int32_t* step_dev, uint64_t seed, const int64_t* pose_key) {
  PoseNoise nz;
  nz.coef_dev = coef_table; nz.step_dev = step_dev; nz.seed = seed;
  nz.pose_key = reinterpret_cast<const long long*>(pose_key); nz.philox = pose_key != nullptr;
  return nz;
}

}  // namespace

extern "C" int ddb200_pose_update(const float* pos, int64_t n_poses, int n_atoms, int n_bonds, const int32_t* bond_u,
                                  const int32_t* bond_v, const uint8_t* mask_rotate, const float* tr_score,
                                  const float* rot_score, const float* tor_score, const float* tr_z,
                                  const float* rot_z, const float* tor_z, const float* coef6, int use_torsion,
                                  float* out_pos, void* stream) {
  if (!pos || !out_pos || !tr_score || !rot_score || !coef6 || n_poses < 0 || n_atoms <= 0 || n_bonds < 0)
    return DDB200_EINVAL;
  if (use_torsion && n_bonds > 0 && (!bond_u || !bond_v || !mask_rotate || !tor_score)) return DDB200_EINVAL;
  return launch_pose_update(pos, n_poses, n_atoms, n_bonds, nullptr, n_atoms, nullptr, bond_u, bond_v, mask_rotate,
                            tr_score, rot_score, tor_score, tr_z, rot_z, tor_z, coef6, use_torsion, PoseNoise{}, out_pos,
                            stream);
}

// Same update with the step's SDE coefficients read from DEVICE memory (row *step_dev of coef_table [n_steps, 6]; step_dev
// NULL = row 0) and, if pose_key != NULL, the noise drawn in-kernel from Philox4x32-10 keyed by (seed, pose_key[b]) at
// counter (step, dof) - no host value enters the launch, so the whole reverse-diffusion step can sit in a CUDA graph, and a
// pose's noise does not depend on how poses are batched or sharded.  out_pos may alias pos (each pose is read completely
// before it is written).
extern "C" int ddb200_pose_update_dev(const float* pos, int64_t n_poses, int n_atoms, int n_bonds, const int32_t* bond_u,
                                      const int32_t* bond_v, const uint8_t* mask_rotate, const float* tr_score,
                                      const float* rot_score, const float* tor_score, const float* tr_z,
                                      const float* rot_z, const float* tor_z, const float* coef_table,
                                      const int32_t* step_dev, uint64_t seed, const int64_t* pose_key, int use_torsion,
                                      float* out_pos, void* stream) {
  if (!pos || !out_pos || !tr_score || !rot_score || !coef_table || n_poses < 0 || n_atoms <= 0 || n_bonds < 0)
    return DDB200_EINVAL;
  if (use_torsion && n_bonds > 0 && (!bond_u || !bond_v || !mask_rotate || !tor_score)) return DDB200_EINVAL;
  return launch_pose_update(pos, n_poses, n_atoms, n_bonds, nullptr, n_atoms, nullptr, bond_u, bond_v, mask_rotate,
                            tr_score, rot_score, tor_score, tr_z, rot_z, tor_z, nullptr, use_torsion,
                            device_noise(coef_table, step_dev, seed, pose_key), out_pos, stream);
}

// ddb200_pose_update_dev over poses of different ligands: pose b reads its layout from row b of the device descriptor
// (see pose_update_kernel).  The host never reads the descriptor; max_atoms sizes the shared memory.
extern "C" int ddb200_pose_update_packed(const float* pos, int64_t n_poses, const int32_t* layout, int max_atoms,
                                         const int32_t* bond_u, const int32_t* bond_v, const uint8_t* mask_rotate,
                                         const float* tr_score, const float* rot_score, const float* tor_score,
                                         const float* tr_z, const float* rot_z, const float* tor_z,
                                         const float* coef_table, const int32_t* step_dev, uint64_t seed,
                                         const int64_t* pose_key, int use_torsion, int32_t* err, float* out_pos,
                                         void* stream) {
  if (!pos || !out_pos || !tr_score || !rot_score || !coef_table || !layout || !err || n_poses < 0 || max_atoms <= 0)
    return DDB200_EINVAL;
  if (use_torsion && (!bond_u || !bond_v || !mask_rotate || !tor_score)) return DDB200_EINVAL;
  return launch_pose_update(pos, n_poses, 0, 0, layout, max_atoms, err, bond_u, bond_v, mask_rotate, tr_score, rot_score,
                            tor_score, tr_z, rot_z, tor_z, nullptr, use_torsion,
                            device_noise(coef_table, step_dev, seed, pose_key), out_pos, stream);
}

// Diagnostics / tests: out[4 * i .. 4 * i + 3] = the four normals of Philox block (seed, pose_key, step, block0 + i).
namespace {
__global__ void philox_probe_kernel(unsigned long long seed, long long pose_key, uint32_t step, uint32_t block0, int n,
                                    float* out, uint32_t* raw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float z[4];
  philox_normal4(seed, pose_key, step, block0 + i, z);
  for (int j = 0; j < 4; ++j) out[4 * i + j] = z[j];
  if (raw) {
    uint32_t c[4] = {(uint32_t)pose_key, (uint32_t)((unsigned long long)pose_key >> 32), step, block0 + (uint32_t)i};
    philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
    for (int j = 0; j < 4; ++j) raw[4 * i + j] = c[j];
  }
}
}  // namespace
extern "C" int ddb200_philox_probe(uint64_t seed, int64_t pose_key, uint32_t step, uint32_t block0, int n_blocks,
                                   float* out_normals, uint32_t* out_raw, void* stream) {
  if (!out_normals || n_blocks < 0) return DDB200_EINVAL;
  if (n_blocks == 0) return 0;
  philox_probe_kernel<<<(n_blocks + 127) / 128, 128, 0, (cudaStream_t)stream>>>(seed, pose_key, step, block0, n_blocks,
                                                                                 out_normals, out_raw);
  return (int)cudaGetLastError();
}

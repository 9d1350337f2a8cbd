// The confidence head of every confidence model (models/cg_model.py:354-366, models/aa_model.py:434-455,
// models/old_cg_model.py:296-299, models/old_aa_model.py:283-286) as one kernel: column selection of the ligand node
// features, the optional per-atom ``atom_confidence_predictor``, the segment mean per pose and the three-layer
// ``confidence_predictor``.  One CTA per pose; the pose's atom range comes from the device segment pointer, so nothing is
// read back to the host.  Every sum has a fixed order (dot products over k ascending, the pooled sum over the pose's atoms
// in index order, each column owned by one thread), and there are no atomics: two calls give bit-identical results.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/diffdock_b200.h"

namespace {

constexpr int kThreads = 128;
constexpr int kTile = 8;                                   // atoms per pass through the per-atom MLP
constexpr int kMaxIn = DDB200_CONF_MAX_IN;
constexpr int kMaxHidden = DDB200_CONF_MAX_HIDDEN;
constexpr int kMaxAtomOut = DDB200_CONF_MAX_OUT + DDB200_CONF_MAX_IN;    // atom outputs + the pooled columns

// Offsets into a packed MLP (layout in include/diffdock_b200.h).
struct Mlp {
  const float* p;
  int n_in, n_h, n_out;
  __device__ const float* w(int l) const { return p + off(l); }
  __device__ int rows(int l) const { return l < 2 ? n_h : n_out; }
  __device__ int cols(int l) const { return l == 0 ? n_in : n_h; }
  __device__ int off(int l) const {
    int o = 0;
    for (int i = 0; i < l; ++i) o += rows(i) * cols(i) + 3 * rows(i);
    return o;
  }
};

// out[r][o] = act((sum_k W[o][k] in[r][k] + b[o]) * scale[o] + shift[o]) for r < rows, layer l of ``m``; layers 0 and 1
// carry the folded BatchNorm and a ReLU, layer 2 is a plain Linear.
__device__ void dense(const Mlp& m, int l, const float* in, int ld_in, float* out, int ld_out, int rows) {
  const int n_out = m.rows(l), n_in = m.cols(l);
  const float* W = m.w(l);
  const float* b = W + n_out * n_in;
  for (int i = threadIdx.x; i < rows * n_out; i += blockDim.x) {
    const int r = i / n_out, o = i - r * n_out;
    const float* w = W + o * n_in;
    const float* v = in + r * ld_in;
    float acc = 0.f;
    for (int k = 0; k < n_in; ++k) acc = fmaf(__ldg(w + k), v[k], acc);
    acc += __ldg(b + o);
    if (l < 2) {
      acc = fmaf(acc, __ldg(b + n_out + o), __ldg(b + 2 * n_out + o));
      acc = fmaxf(acc, 0.f);
    }
    out[r * ld_out + o] = acc;
  }
}

__global__ void __launch_bounds__(kThreads) confidence_head_kernel(
    const float* __restrict__ x, long long ld_x, const int* __restrict__ lig_ptr, int n_head, int tail_off, int n_tail,
    Mlp atom, int n_atom_out, Mlp head, float* __restrict__ confidence, float* __restrict__ atom_confidence) {
  __shared__ float xin[kTile][kMaxIn];
  __shared__ float h1[kTile][kMaxHidden];
  __shared__ float h2[kTile][kMaxHidden];
  __shared__ float ao[kTile][kMaxAtomOut];
  __shared__ float pool[kMaxIn];

  const int b = blockIdx.x;
  const int beg = lig_ptr[b], end = lig_ptr[b + 1];
  const int n_sel = n_head + n_tail;
  const int P = head.n_in;                                 // pooled width
  for (int c = threadIdx.x; c < P; c += blockDim.x) pool[c] = 0.f;

  for (int a0 = beg; a0 < end; a0 += kTile) {
    const int rows = min(kTile, end - a0);
    for (int i = threadIdx.x; i < rows * n_sel; i += blockDim.x) {
      const int r = i / n_sel, k = i - r * n_sel;
      const int col = k < n_head ? k : tail_off + (k - n_head);
      xin[r][k] = x[(long long)(a0 + r) * ld_x + col];
    }
    __syncthreads();
    const float* src = &xin[0][0];
    int ld_src = kMaxIn;
    if (atom.p) {
      dense(atom, 0, &xin[0][0], kMaxIn, &h1[0][0], kMaxHidden, rows);
      __syncthreads();
      dense(atom, 1, &h1[0][0], kMaxHidden, &h2[0][0], kMaxHidden, rows);
      __syncthreads();
      dense(atom, 2, &h2[0][0], kMaxHidden, &ao[0][0], kMaxAtomOut, rows);
      __syncthreads();
      for (int i = threadIdx.x; i < rows * n_atom_out; i += blockDim.x) {
        const int r = i / n_atom_out, o = i - r * n_atom_out;
        atom_confidence[(long long)(a0 + r) * n_atom_out + o] = ao[r][o];
      }
      src = &ao[0][n_atom_out];
      ld_src = kMaxAtomOut;
    }
    for (int c = threadIdx.x; c < P; c += blockDim.x) {
      float s = pool[c];
      for (int r = 0; r < rows; ++r) s += src[r * ld_src + c];
      pool[c] = s;
    }
    __syncthreads();
  }

  // scatter_mean: the sum over the pose's atoms divided by their count (an empty pose pools to zero)
  const float n = (float)max(end - beg, 1);
  for (int c = threadIdx.x; c < P; c += blockDim.x) pool[c] = pool[c] / n;
  __syncthreads();
  dense(head, 0, pool, kMaxIn, &h1[0][0], kMaxHidden, 1);
  __syncthreads();
  dense(head, 1, &h1[0][0], kMaxHidden, &h2[0][0], kMaxHidden, 1);
  __syncthreads();
  dense(head, 2, &h2[0][0], kMaxHidden, confidence + (long long)b * head.n_out, 0, 1);
}

}  // namespace

extern "C" int ddb200_confidence_head(const float* x, int64_t ld_x, int64_t n_cols, const int32_t* lig_ptr,
                                      int32_t n_poses, int32_t n_head, int32_t tail_off, int32_t n_tail,
                                      const float* atom_mlp, int32_t atom_hidden, int32_t n_atom_out, const float* mlp,
                                      int32_t n_in, int32_t n_hidden, int32_t n_out, float* confidence,
                                      float* atom_confidence, void* stream) {
  if (n_poses < 0 || !lig_ptr || !mlp || !confidence) return DDB200_EINVAL;
  if (n_head < 0 || n_tail < 0 || tail_off < 0 || (int64_t)tail_off + n_tail > n_cols || n_head > n_cols ||
      n_cols > ld_x || n_head + n_tail < 1)
    return DDB200_EINVAL;
  if (n_in < 1 || n_in > DDB200_CONF_MAX_IN || n_hidden < 1 || n_hidden > DDB200_CONF_MAX_HIDDEN || n_out < 1 ||
      n_out > DDB200_CONF_MAX_OUT)
    return DDB200_EINVAL;
  const int n_sel = n_head + n_tail;
  if (n_sel > DDB200_CONF_MAX_IN) return DDB200_EINVAL;
  if (atom_mlp) {
    if (!atom_confidence || atom_hidden < 1 || atom_hidden > DDB200_CONF_MAX_HIDDEN || n_atom_out < 1 ||
        n_atom_out > DDB200_CONF_MAX_OUT)
      return DDB200_EINVAL;
  } else if (n_sel != n_in) {
    return DDB200_EINVAL;
  }
  if (n_poses == 0) return 0;
  if (!x) return DDB200_EINVAL;
  const Mlp atom{atom_mlp, n_sel, atom_hidden, n_atom_out + n_in};
  const Mlp head{mlp, n_in, n_hidden, n_out};
  confidence_head_kernel<<<n_poses, kThreads, 0, (cudaStream_t)stream>>>(
      x, (long long)ld_x, lig_ptr, n_head, tail_off, n_tail, atom, atom_mlp ? n_atom_out : 0, head, confidence,
      atom_confidence);
  return (int)cudaGetLastError();
}

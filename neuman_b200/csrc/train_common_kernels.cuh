// Shared by human_train_kernels.cuh and smpl_train_kernels.cuh: the build macros of the restricted CUDA subset (see
// human_train_kernels.cuh) and the 4x4 inverse, which warp.cu and smpl.cu use as well.
#pragma once
#ifndef NM_EMU
#define NM_KERNEL static __global__
#define NM_DEV __device__ __forceinline__
#define NM_ATOMIC_ADD(p, v) atomicAdd((p), (v))
#endif

// General 4x4 inverse by cofactors in float64 (torch.inverse, utils/ray_utils.py:91; the blended transforms are
// well-conditioned near-rigid matrices, and the float64 evaluation keeps the result within a float32 ulp of exact).
NM_DEV bool wd_inv4(const double* m, double* o) {
  double s0 = m[0] * m[5] - m[4] * m[1], s1 = m[0] * m[6] - m[4] * m[2], s2 = m[0] * m[7] - m[4] * m[3];
  double s3 = m[1] * m[6] - m[5] * m[2], s4 = m[1] * m[7] - m[5] * m[3], s5 = m[2] * m[7] - m[6] * m[3];
  double c5 = m[10] * m[15] - m[14] * m[11], c4 = m[9] * m[15] - m[13] * m[11], c3 = m[9] * m[14] - m[13] * m[10];
  double c2 = m[8] * m[15] - m[12] * m[11], c1 = m[8] * m[14] - m[12] * m[10], c0 = m[8] * m[13] - m[12] * m[9];
  double det = s0 * c5 - s1 * c4 + s2 * c3 + s3 * c2 - s4 * c1 + s5 * c0;
  if (det == 0.0) return false;
  double id = 1.0 / det;
  o[0] = (m[5] * c5 - m[6] * c4 + m[7] * c3) * id;     o[1] = (-m[1] * c5 + m[2] * c4 - m[3] * c3) * id;
  o[2] = (m[13] * s5 - m[14] * s4 + m[15] * s3) * id;  o[3] = (-m[9] * s5 + m[10] * s4 - m[11] * s3) * id;
  o[4] = (-m[4] * c5 + m[6] * c2 - m[7] * c1) * id;    o[5] = (m[0] * c5 - m[2] * c2 + m[3] * c1) * id;
  o[6] = (-m[12] * s5 + m[14] * s2 - m[15] * s1) * id; o[7] = (m[8] * s5 - m[10] * s2 + m[11] * s1) * id;
  o[8] = (m[4] * c4 - m[5] * c2 + m[7] * c0) * id;     o[9] = (-m[0] * c4 + m[1] * c2 - m[3] * c0) * id;
  o[10] = (m[12] * s4 - m[13] * s2 + m[15] * s0) * id; o[11] = (-m[8] * s4 + m[9] * s2 - m[11] * s0) * id;
  o[12] = (-m[4] * c3 + m[5] * c1 - m[6] * c0) * id;   o[13] = (m[0] * c3 - m[1] * c1 + m[2] * c0) * id;
  o[14] = (-m[12] * s3 + m[13] * s1 - m[14] * s0) * id; o[15] = (m[8] * s3 - m[9] * s1 + m[10] * s0) * id;
  return true;
}


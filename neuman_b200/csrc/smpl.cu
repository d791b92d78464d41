// Per-frame SMPL linear blend skinning on the device: the 6890 (+24) per-vertex 4x4 transforms that
// the observation->canonical warp consumes, and the scene-space transforms / vertices built from them.
//
//   nm_smpl_vertex_transforms  <- SMPL.verts_transformations models/smpl.py:109-162, lbs :266-360,
//                                 batch_rodrigues :407-438, batch_rigid_transform :454-505,
//                                 blend_shapes :383, vertices2joints :363   (float32, like the reference)
//   nm_smpl_scene_transforms   <- data_io/neuman_helper.py:299-330 (read_smpls; float64 after the float32
//                                 LBS, like the reference's numpy code) == HumanNeRF.vertex_forward
//                                 models/human_nerf.py:92-122
//
// Pose blend shapes are computed by the reference but NOT applied (v_posed = v_shaped, models/smpl.py:334),
// so they are not evaluated here.
#include "nm_internal.cuh"
#include "smpl_train_kernels.cuh"

// v_shaped = v_template + shapedirs . beta     (blend_shapes, models/smpl.py:383)
__global__ void k_smpl_shape(const float* __restrict__ v_template, const float* __restrict__ shapedirs,
                             const float* __restrict__ betas, int nv, int nb, float* __restrict__ v_shaped) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;      // over nv*3
  if (i >= nv * 3) return;
  float acc = 0.f;
  for (int l = 0; l < nb; ++l) acc = fmaf(betas[l], shapedirs[(size_t)i * nb + l], acc);
  v_shaped[i] = v_template[i] + acc;
}

// J = J_regressor . v_shaped   (vertices2joints, models/smpl.py:363): one block per (joint, component)
__global__ void __launch_bounds__(256) k_smpl_joints(const float* __restrict__ Jreg, const float* __restrict__ v_shaped,
                                                      int nv, float* __restrict__ J) {
  __shared__ float red[256];
  const int j = blockIdx.x / 3, c = blockIdx.x % 3;
  float acc = 0.f;
  for (int v = threadIdx.x; v < nv; v += 256) acc = fmaf(Jreg[(size_t)j * nv + v], v_shaped[3 * v + c], acc);
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) J[3 * j + c] = red[0];
}

// Rodrigues + kinematic chain + relative transforms A_j (models/smpl.py:407-438, :454-505). One thread.
__global__ void k_smpl_chain(const float* __restrict__ pose, const float* __restrict__ J, SmpltParents par, int nj,
                             float* __restrict__ A) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float G[SMPLT_MAX_J][16];
  for (int j = 0; j < nj; ++j) {
    float L[16];
    SmpltRod rod;
    smplt_rodrigues(pose + 3 * j, rod, L);
    const int p = par.p[j];
    for (int a = 0; a < 3; ++a) L[4 * a + 3] = J[3 * j + a] - (j > 0 ? J[3 * p + a] : 0.f);   // rel_joints (:479-480)
    L[12] = L[13] = L[14] = 0.f; L[15] = 1.f;
    if (j == 0) for (int k = 0; k < 16; ++k) G[0][k] = L[k];
    else smplt_mm4(G[p], L, G[j]);                                                 // sequential chain (:487-493)
  }
  for (int j = 0; j < nj; ++j) {                                                   // A = G - [0 | G.[J;0]] (:500-503)
    for (int k = 0; k < 16; ++k) A[16 * j + k] = G[j][k];
    for (int a = 0; a < 4; ++a) {
      float corr = G[j][4 * a] * J[3 * j] + G[j][4 * a + 1] * J[3 * j + 1] + G[j][4 * a + 2] * J[3 * j + 2];
      A[16 * j + 4 * a + 3] = G[j][4 * a + 3] - corr;
    }
  }
}

// T_v = sum_j W[v,j] A_j (models/smpl.py:344-345); rows nv.. = A, J when concat_joints (:347-349)
__global__ void k_smpl_blend(const float* __restrict__ W, const float* __restrict__ A, const float* __restrict__ v_shaped,
                             const float* __restrict__ J, int nv, int nj, int concat, float* __restrict__ T,
                             float* __restrict__ verts) {
  __shared__ float sA[SMPLT_MAX_J * 16];
  for (int k = threadIdx.x; k < nj * 16; k += blockDim.x) sA[k] = A[k];
  __syncthreads();
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  int total = nv + (concat ? nj : 0);
  if (v >= total) return;
  if (v < nv) {
    float acc[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) acc[k] = 0.f;
    for (int j = 0; j < nj; ++j) {
      float w = W[(size_t)v * nj + j];
#pragma unroll
      for (int k = 0; k < 16; ++k) acc[k] = fmaf(w, sA[16 * j + k], acc[k]);
    }
#pragma unroll
    for (int k = 0; k < 16; ++k) T[(size_t)16 * v + k] = acc[k];
    if (verts) { verts[3 * v] = v_shaped[3 * v]; verts[3 * v + 1] = v_shaped[3 * v + 1]; verts[3 * v + 2] = v_shaped[3 * v + 2]; }
  } else {
    int j = v - nv;
    for (int k = 0; k < 16; ++k) T[(size_t)16 * v + k] = sA[16 * j + k];
    if (verts) { verts[3 * v] = J[3 * j]; verts[3 * v + 1] = J[3 * j + 1]; verts[3 * v + 2] = J[3 * j + 2]; }
  }
}

static int smpl_lbs(nm_ctx* ctx, const nm_smpl_model* m, const float* pose_dev, const float* betas_dev, int concat,
                    float* v_shaped, float* J, float* A, float* T, float* verts, cudaStream_t st) {
  const int nv = m->n_verts, nj = m->n_joints;
  k_smpl_shape<<<(nv * 3 + 255) / 256, 256, 0, st>>>(m->v_template, m->shapedirs, betas_dev, nv, m->n_betas, v_shaped);
  NM_CHECK_LAUNCH(ctx);
  k_smpl_joints<<<nj * 3, 256, 0, st>>>(m->J_regressor, v_shaped, nv, J);
  NM_CHECK_LAUNCH(ctx);
  SmpltParents par;
  for (int j = 0; j < nj; ++j) par.p[j] = m->parents[j];
  k_smpl_chain<<<1, 32, 0, st>>>(pose_dev, J, par, nj, A);
  NM_CHECK_LAUNCH(ctx);
  const int total = nv + (concat ? nj : 0);
  k_smpl_blend<<<(total + 127) / 128, 128, 0, st>>>(m->weights, A, v_shaped, J, nv, nj, concat, T, verts);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

static int check_model(nm_ctx* ctx, const nm_smpl_model* m) {
  if (!m || !m->v_template || !m->shapedirs || !m->J_regressor || !m->weights || !m->parents || m->n_verts <= 0 ||
      m->n_joints <= 0 || m->n_joints > SMPLT_MAX_J || m->n_betas <= 0)
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_smpl: bad model");
  return NM_OK;
}

extern "C" int nm_smpl_vertex_transforms(nm_ctx* ctx, const nm_smpl_model* m, const float* pose, const float* betas,
                                         int32_t concat_joints, float* T, float* verts, void* stream) {
  NM_ENTER(ctx);
  int rc = check_model(ctx, m);
  if (rc) return rc;
  if (!pose || !betas || !T) NM_FAIL(ctx, NM_ERR_INVALID, "nm_smpl_vertex_transforms: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int nv = m->n_verts, nj = m->n_joints;
  char* ws;
  size_t floats = (size_t)nv * 3 + nj * 3 + nj * 16 + 128;
  if ((rc = nm_impl_workspace(ctx, floats * sizeof(float) + 1024, &ws))) return rc;
  float* v_shaped = reinterpret_cast<float*>(ws);
  float* J = v_shaped + (((size_t)nv * 3 + 63) & ~size_t(63));
  float* A = J + ((nj * 3 + 63) & ~63);
  return smpl_lbs(ctx, m, pose, betas, concat_joints, v_shaped, J, A, T, verts, st);
}

// --------------------------------------------------------------------------------------------------
struct Mat4d { double v[16]; };

// T_da2scene = S . align^T . T_t2pose . inv(T_t2da); world = T_da2scene . [da_vert;1]   (neuman_helper.py:316-326)
__global__ void k_smpl_scene(const float* __restrict__ T_pose, const float* __restrict__ T_da,
                             const float* __restrict__ rest /* v_shaped | J rows */, Mat4d pre /* S . align^T */, int total,
                             double* __restrict__ T_out, float* __restrict__ world) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= total) return;
  double P[16], D[16], Di[16], M[16], R[16];
  for (int k = 0; k < 16; ++k) { P[k] = (double)T_pose[(size_t)16 * v + k]; D[k] = (double)T_da[(size_t)16 * v + k]; }
  wd_inv4(D, Di);
  for (int a = 0; a < 4; ++a)
    for (int b = 0; b < 4; ++b) {
      double acc = 0.0;
      for (int k = 0; k < 4; ++k) acc += P[4 * a + k] * Di[4 * k + b];
      M[4 * a + b] = acc;
    }
  for (int a = 0; a < 4; ++a)
    for (int b = 0; b < 4; ++b) {
      double acc = 0.0;
      for (int k = 0; k < 4; ++k) acc += pre.v[4 * a + k] * M[4 * k + b];
      R[4 * a + b] = acc;
    }
  for (int k = 0; k < 16; ++k) T_out[(size_t)16 * v + k] = R[k];
  if (world) {
    // da-pose vertex = T_da . [rest;1] in float32 (SMPL.forward, models/smpl.py:352-357), then float64 transform
    float r0 = rest[3 * v], r1 = rest[3 * v + 1], r2 = rest[3 * v + 2];
    double dv[3];
    for (int a = 0; a < 3; ++a) {
      const float* t = T_da + (size_t)16 * v + 4 * a;
      dv[a] = (double)(fmaf(t[2], r2, fmaf(t[1], r1, t[0] * r0)) + t[3]);
    }
    for (int a = 0; a < 3; ++a)
      world[3 * v + a] = (float)(R[4 * a] * dv[0] + R[4 * a + 1] * dv[1] + R[4 * a + 2] * dv[2] + R[4 * a + 3]);
  }
}

extern "C" int nm_smpl_scene_transforms(nm_ctx* ctx, const nm_smpl_model* m, const float* pose, const float* da_pose,
                                        const float* betas, const double* alignment, double scale, double* T_da2scene,
                                        float* world_verts, void* stream) {
  NM_ENTER(ctx);
  int rc = check_model(ctx, m);
  if (rc) return rc;
  if (!pose || !da_pose || !betas || !alignment || !T_da2scene)
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_smpl_scene_transforms: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int nv = m->n_verts, nj = m->n_joints, total = nv + nj;
  char* ws;
  // the same rounding as `take` below, buffer by buffer: v_shaped, J, A, T_pose, T_da, rest
  auto pad64 = [](size_t n) { return (n + 63) & ~size_t(63); };
  const size_t floats = pad64((size_t)nv * 3) + pad64((size_t)nj * 3) + pad64((size_t)nj * 16) +
                        2 * pad64((size_t)total * 16) + pad64((size_t)total * 3);
  if ((rc = nm_impl_workspace(ctx, floats * sizeof(float), &ws))) return rc;
  float* p = reinterpret_cast<float*>(ws);
  auto take = [&](size_t n) { float* r = p; p += pad64(n); return r; };
  float* v_shaped = take((size_t)nv * 3);
  float* J = take(nj * 3);
  float* A = take(nj * 16);
  float* T_pose = take((size_t)total * 16);
  float* T_da = take((size_t)total * 16);
  float* rest = take((size_t)total * 3);
  if ((size_t)(reinterpret_cast<char*>(p) - ws) > ctx->ws_bytes)
    NM_FAIL(ctx, NM_ERR_STATE, "nm_smpl_scene_transforms: workspace overflow (internal sizing bug)");
  if ((rc = smpl_lbs(ctx, m, pose, betas, 1, v_shaped, J, A, T_pose, nullptr, st))) return rc;
  if ((rc = smpl_lbs(ctx, m, da_pose, betas, 1, v_shaped, J, A, T_da, rest, st))) return rc;
  Mat4d pre;   // S . align^T  (s = eye; s[:3,:3] *= scale; T = s @ (alignment.T @ T_da2pose), :318-321)
  for (int a = 0; a < 4; ++a)
    for (int b = 0; b < 4; ++b) pre.v[4 * a + b] = alignment[4 * b + a] * (a < 3 ? scale : 1.0);
  k_smpl_scene<<<(total + 127) / 128, 128, 0, st>>>(T_pose, T_da, rest, pre, total, T_da2scene, world_verts);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

// --------------------------------------------------------------------------------------------------
// Training-time scene transforms and their adjoint (smpl_train_kernels.cuh): HumanNeRF.vertex_forward
// (models/human_nerf.py:92-122) in float32 with the alignment read from DEVICE memory (it is an nn.Parameter the
// trainer optimises: no host round trip per step), and what loss.backward() sends to poses / betas / alignments.
// --------------------------------------------------------------------------------------------------
struct SmplTrainWs {
  float *v_shaped, *J, *A, *T_pose, *T_da, *gP, *gD, *grest, *gA_pose, *gA_da, *gJ, *gpre;
};

static int smpl_train_workspace(nm_ctx* ctx, int nv, int nj, bool backward, SmplTrainWs& w) {
  auto pad64 = [](size_t n) { return (n + 63) & ~size_t(63); };
  size_t floats = pad64((size_t)nv * 3) + pad64((size_t)nj * 3) + pad64((size_t)nj * 16) + 2 * pad64((size_t)nv * 16);
  if (backward) floats += 2 * pad64((size_t)nv * 16) + pad64((size_t)nv * 3) + 2 * pad64((size_t)nj * 16) + pad64((size_t)nj * 3) + 64;
  char* ws;
  int rc;
  if ((rc = nm_impl_workspace(ctx, floats * sizeof(float), &ws))) return rc;
  float* p = reinterpret_cast<float*>(ws);
  auto take = [&](size_t n) { float* r = p; p += pad64(n); return r; };
  w.v_shaped = take((size_t)nv * 3); w.J = take((size_t)nj * 3); w.A = take((size_t)nj * 16);
  w.T_pose = take((size_t)nv * 16); w.T_da = take((size_t)nv * 16);
  if (backward) {
    w.gP = take((size_t)nv * 16); w.gD = take((size_t)nv * 16); w.grest = take((size_t)nv * 3);
    w.gA_pose = take((size_t)nj * 16); w.gA_da = take((size_t)nj * 16); w.gJ = take((size_t)nj * 3); w.gpre = take(64);
  }
  if ((size_t)(reinterpret_cast<char*>(p) - ws) > ctx->ws_bytes)
    NM_FAIL(ctx, NM_ERR_STATE, "nm_smpl_scene_*_train: workspace overflow (internal sizing bug)");
  return NM_OK;
}

extern "C" int nm_smpl_scene_forward_train(nm_ctx* ctx, const nm_smpl_model* m, const float* pose, const float* da_pose,
                                           const float* betas, const float* alignment, float scale, float* T_da2scene,
                                           float* world_verts, void* stream) {
  NM_ENTER(ctx);
  int rc = check_model(ctx, m);
  if (rc) return rc;
  if (!pose || !da_pose || !betas || !alignment || !T_da2scene)
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_smpl_scene_forward_train: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int nv = m->n_verts, nj = m->n_joints;
  SmplTrainWs w{};
  if ((rc = smpl_train_workspace(ctx, nv, nj, false, w))) return rc;
  if ((rc = smpl_lbs(ctx, m, pose, betas, 0, w.v_shaped, w.J, w.A, w.T_pose, nullptr, st))) return rc;
  if ((rc = smpl_lbs(ctx, m, da_pose, betas, 0, w.v_shaped, w.J, w.A, w.T_da, nullptr, st))) return rc;
  k_smplt_scene_forward<<<(nv + 127) / 128, 128, 0, st>>>(w.T_pose, w.T_da, w.v_shaped, alignment, scale, nv, T_da2scene,
                                                          world_verts);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

extern "C" int nm_smpl_scene_backward(nm_ctx* ctx, const nm_smpl_model* m, const float* pose, const float* da_pose,
                                      const float* betas, const float* alignment, float scale, const float* g_T,
                                      const float* g_world, float* g_pose, float* g_betas, float* g_alignment,
                                      void* stream) {
  NM_ENTER(ctx);
  int rc = check_model(ctx, m);
  if (rc) return rc;
  if (!pose || !da_pose || !betas || !alignment || (!g_T && !g_world) || !g_pose || !g_betas || !g_alignment)
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_smpl_scene_backward: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int nv = m->n_verts, nj = m->n_joints, nb = m->n_betas;
  SmplTrainWs w{};
  if ((rc = smpl_train_workspace(ctx, nv, nj, true, w))) return rc;
  // forward intermediates (the LBS of both poses is ~10 us; recomputing it beats keeping 2 x 441 KB alive per step)
  if ((rc = smpl_lbs(ctx, m, pose, betas, 0, w.v_shaped, w.J, w.A, w.T_pose, nullptr, st))) return rc;
  if ((rc = smpl_lbs(ctx, m, da_pose, betas, 0, w.v_shaped, w.J, w.A, w.T_da, nullptr, st))) return rc;
  NM_CHECK_CUDA(ctx, cudaMemsetAsync(w.gA_pose, 0, (size_t)(w.gpre + 64 - w.gA_pose) * sizeof(float), st));   // gA_pose, gA_da, gJ, gpre
  NM_CHECK_CUDA(ctx, cudaMemsetAsync(g_betas, 0, (size_t)nb * sizeof(float), st));
  const int chunks = (nv + SMPLT_VPT - 1) / SMPLT_VPT;
  k_smplt_scene_backward<<<(chunks + 63) / 64, 64, 0, st>>>(w.T_pose, w.T_da, w.v_shaped, alignment, scale, g_T, g_world, nv,
                                                            w.gP, w.gD, w.grest, w.gpre);
  NM_CHECK_LAUNCH(ctx);
  k_smplt_blend_backward<<<(nv + 127) / 128, 128, 0, st>>>(m->weights, w.gP, w.gD, nv, nj, w.gA_pose, w.gA_da);
  NM_CHECK_LAUNCH(ctx);
  SmpltParents par;
  for (int j = 0; j < nj; ++j) par.p[j] = m->parents[j];
  k_smplt_chain_backward<<<1, 32, 0, st>>>(pose, da_pose, w.J, par, nj, w.gA_pose, w.gA_da, w.gpre, scale, g_pose, w.gJ,
                                           g_alignment);
  NM_CHECK_LAUNCH(ctx);
  k_smplt_vshaped_backward<<<(nv + 127) / 128, 128, 0, st>>>(m->J_regressor, w.gJ, nv, nj, w.grest);
  NM_CHECK_LAUNCH(ctx);
  const int n3 = nv * 3;
  k_smplt_betas_backward<<<((n3 + 63) / 64 + 63) / 64, 64, 0, st>>>(m->shapedirs, w.grest, n3, nb, g_betas);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

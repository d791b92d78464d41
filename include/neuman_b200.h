/*
 * neuman_b200.h -- C ABI of the H100-native NeuMan ray-marching path.
 *
 * The reference (apple/ml-neuman) is one Python process with no plugin/FFI layer (SURVEY.md §8b);
 * the drop-in boundary is the set of Python functions listed below.  This header declares the
 * C entry points that a binding of each of those functions calls -- `extern "C"`, plain pointers
 * and sizes, no torch types.  Each entry cites the reference function it replaces (file:line in
 * apple/ml-neuman).  INTEGRATION.md shows the ctypes binding (what neuman_b200/_lib.py does).
 *
 * Conventions
 *   - return 0 on success, a negative nm_status otherwise; nm_last_error() gives the text.
 *     Nothing throws across the boundary.
 *   - all `const float*` / `float*` tensor arguments are DEVICE pointers to contiguous memory owned
 *     by the caller (a torch CUDA tensor's data_ptr()), except in the *_host entry points and the
 *     small camera / option structs, which are host memory.
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*; 0 = default stream)
 *     unless stated otherwise.  A ctx is bound to one device and is not thread-safe.
 *   - row-major everywhere; rays are [R,3], samples [R,S], raw network outputs [R,S,4]=(r,g,b,sigma).
 */
#ifndef NEUMAN_B200_H
#define NEUMAN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nm_ctx nm_ctx;

typedef enum {
  NM_OK = 0,
  NM_ERR_INVALID = -1,     /* bad argument                              */
  NM_ERR_CUDA = -2,        /* CUDA runtime error (see nm_last_error)    */
  NM_ERR_UNSUPPORTED = -3, /* shape / option outside what is built      */
  NM_ERR_STATE = -4,       /* slot not packed, mesh not set, ...        */
  NM_ERR_RANGE = -5        /* fp16 operand range exceeded (nm_range_status) */
} nm_status;

/* positional encoding kinds: models/vanilla.py:60-79 ('posenc'), :44-58 ('rotate') */
enum { NM_PE_POSENC = 0, NM_PE_ROTATE = 1 };
/* MLP arithmetic: tensor cores (fp16 operands, fp32 accumulate -- same 11-bit significand as TF32)
 * or CUDA-core fp32 FMA (strict mode, used as the on-device cross-check). */
enum { NM_MLP_TC_F16 = 0, NM_MLP_SIMT_F32 = 1 };

#define NM_MAX_NET_SLOTS 16
#define NM_MAX_ACTORS 8

/* ---- context ------------------------------------------------------------------------------ */
int nm_ctx_create(int device, nm_ctx** out);
int nm_ctx_destroy(nm_ctx* ctx);
const char* nm_last_error(const nm_ctx* ctx);
/* library build id + the SM architecture the kernels were compiled for ("sm_90a") */
const char* nm_version(void);
/* number of kernels this library launched on ctx since creation (bench.py's gpu_launches) */
int64_t nm_launch_count(const nm_ctx* ctx);

/* ---- networks: models/vanilla.py:95-166 (NeRF, Joiner), build_nerf :208 ------------------- */
typedef struct {
  /* fp32 DEVICE pointers, nn.Linear layout [out,in] row-major, exactly the reference state dict:
   * pts_linears.0 [256,63]; .1-.4,.6,.7 [256,256]; .5 [256,319] (input first, models/vanilla.py:131);
   * feature_linear [256,256]; alpha_linear [1,256]; views_linears.0 [128,283] (feature first, :137);
   * rgb_linear [3,128]. */
  const float* pts_w[8];
  const float* pts_b[8];
  const float* feature_w; const float* feature_b;
  const float* alpha_w;   const float* alpha_b;
  const float* views_w;   const float* views_b;
  const float* rgb_w;     const float* rgb_b;
  int32_t pos_pe_kind;    /* NM_PE_* for the position input */
  int32_t dir_pe_kind;    /* NM_PE_* for the view-direction input */
  float pos_min_freq, pos_max_freq; int32_t pos_n_freqs;   /* options/options.py:62-66 */
  float dir_min_freq, dir_max_freq; int32_t dir_n_freqs;   /* options/options.py:67-69 */
} nm_nerf_desc;

/* Re-pack the weights of one Joiner into the kernel layouts (fp16 wgmma slabs + fp32 transposed).
 * Replaces nothing in the reference; it is the cost of `net.cuda()` / checkpoint load. */
int nm_net_pack(nm_ctx* ctx, int slot, const nm_nerf_desc* desc, void* stream);

/* A view-independent NeRF (use_viewdirs=False: the background nets' --use_viewdirs False, the canonical human net's
 * --specular_can False; models/vanilla.py:117-118,145-146): the same 8x256 trunk with one output_linear [4,256] on
 * layer 7 and no view-direction input.  fp32 DEVICE pointers in the reference's nn.Linear layout. */
typedef struct {
  const float* pts_w[8];
  const float* pts_b[8];
  const float* output_w;  const float* output_b;    /* output_linear [4,256], [4] */
  int32_t pos_pe_kind;                              /* NM_PE_* for the position input */
  float pos_min_freq, pos_max_freq; int32_t pos_n_freqs;
} nm_nerf_noview_desc;

/* Packs a view-independent net into `slot` (a slot may hold either kind; packing changes its kind).  Every entry point
 * that takes a slot serves both kinds; for a view-independent slot:
 *   nm_mlp_forward / nm_mlp_forward_rays: `views` may be NULL and is ignored, raw = output_linear(h7) (r, g, b, sigma);
 *   nm_mlp_forward_train: stash_f and stash_v are NULL, stash_m has 8 planes [8][n][8] (pts_linears 0..7);
 *   nm_mlp_backward: g_f and g_v are NULL (and stash_v is not read); g_pre as for view-dependent nets;
 *   nm_dw_gemm: with NULL g_f, g_v and stash_f only out[0..6] (pts_linears 1..7) are computed, out[7..8] are zero;
 *   nm_encode_f16 / nm_pe_backward with which = 1 return NM_ERR_UNSUPPORTED (there is no direction encoding);
 *   the frame drivers accept any mix of kinds over their coarse, fine and human slots. */
int nm_net_pack_noview(nm_ctx* ctx, int slot, const nm_nerf_noview_desc* desc, void* stream);

/* Packs a NeRF-T net (the reference's --ablate_nerft background nets, train.py:254-256: the position input is
 * (x, y, z, t), models/vanilla.py:60-79 with input_dims = 4) into `slot`: an nm_nerf_desc whose pts_linears.0 is
 * [256,84] and .5 [256,340] (columns in the reference's order [x, y, z, t, sin(f_0 xyzt), cos(f_0 xyzt), ...]).  Only
 * the posenc position mapping is accepted (the reference's rotate mapping asserts a 3-D input, models/vanilla.py:84).
 * For a NeRF-T slot:
 *   nm_mlp_forward / nm_mlp_forward_train read pts as [n,4] = (x, y, z, t), exactly the reference's input_pts; the stash
 *   and nm_mlp_backward are those of a view-dependent net;
 *   nm_encode_f16 with which = 0 reads x as [n,4] and writes [n][96]: the 84 channels in the reference's column order,
 *   1.0 at channel 84, zeros to 95 (g^T @ plane = pts_linears.0's weight gradient, bias gradient in column 84);
 *   nm_render_vanilla_t renders a frame at one time;
 *   nm_mlp_forward_rays, nm_pe_backward with which = 0 (no input gradient) and the drivers without a time argument
 *   (nm_render_vanilla, nm_render_smpl_nerf, nm_render_hybrid) return NM_ERR_UNSUPPORTED. */
int nm_net_pack_nerft(nm_ctx* ctx, int slot, const nm_nerf_desc* desc, void* stream);

/* Joiner.forward(input_pts, input_views) (models/vanilla.py:162-166) = Embedder.forward (:82-92)
 * on both inputs + NeRF.forward (:120-152).  pts, views: [n,3]; raw: [n,4].
 * If views_per_ray != 0, `views` is [n/views_per_ray, 3] and row i serves samples
 * [i*views_per_ray, (i+1)*views_per_ray) (the renderers pass `dirs` stacked along samples). */
int nm_mlp_forward(nm_ctx* ctx, int slot, int mode, const float* pts, const float* views,
                   int64_t n, int32_t views_per_ray, float* raw, void* stream);

/* Training forward of the same network (train.py -> trainers/*: Joiner.forward under autograd): as
 * nm_mlp_forward in NM_MLP_TC_F16 mode, and additionally writes the fp16 activations the backward
 * pass needs.  stash_x: [8][n][256] post-ReLU outputs of pts_linears 0..7; stash_f: [n][256]
 * feature_linear output; stash_v: [n][128] views_linears.0 post-ReLU; stash_m: [9][n][8] uint32 ReLU sign
 * words (16 bits per 16 outputs: bit j = [output 2j > 0], bit 8+j = [output 2j+1 > 0]): planes 0..7 =
 * pts_linears 0..7, plane 8 = views_linears.0 (words 0..3). */
int nm_mlp_forward_train(nm_ctx* ctx, int slot, const float* pts, const float* views, int64_t n,
                         int32_t views_per_ray, float* raw, void* stash_x, void* stash_f, void* stash_v,
                         void* stash_m, void* stream);

/* Embedder.forward (models/vanilla.py:82-92) of net `slot` in the fp16 form the tensor-core kernels multiply with:
 * which = 0: out [n][64] fp16 position encoding, channel 63 = 1.0; which = 1: out [n][32] direction encoding,
 * channel 27 = 1.0, 28.. zero.  x: [n,3] (or [n/group,3] when group > 0).  The constant channel makes
 * g^T @ out deliver the bias gradient next to the weight gradient of the layers that read the encoding. */
int nm_encode_f16(nm_ctx* ctx, int slot, int32_t which, const float* x, int64_t group, int64_t n, void* out,
                  void* stream);

/* Adjoint of NeRF.forward (models/vanilla.py:120-152) with respect to the layer pre-activations
 * (what torch autograd computes inside loss.backward() for trainers/vanilla_nerf_trainer.py:222).
 * d_raw: [n,4] fp32 dL/d(raw); loss_scale: device pointer to one float S (a power of two; all outputs
 * are S * gradient in fp16); stash_m: the forward's [9][n][8] sign words (stash_v is accepted for symmetry and
 * not read).  Outputs: g_pre [8][n][256] = dL/d(pre-activation of pts_linears l),
 * g_f [n][256] = dL/d(feature), g_v [n][128] = dL/d(pre-activation of views_linears.0).  The weight
 * gradients are then dW_l = g_l^T @ input_l over the forward stash (GEMMs with K = n, left to the
 * caller's BLAS), the bias gradients the column sums of g_l. */
int nm_mlp_backward(nm_ctx* ctx, int slot, const float* d_raw, const float* loss_scale, int64_t n,
                    const void* stash_v, const void* stash_m, void* g_pre, void* g_f, void* g_v, void* stream);

/* Adjoint of Embedder.forward (models/vanilla.py:82-92) of net `slot`: which = 0 position encoding, 1 direction
 * encoding.  x: the encoder input [n,3] (or [n/group,3] when group > 0, as nm_mlp_forward's views_per_ray);
 * d_enc: [n][ld] fp32 dL/d(encoding), ld >= encoding width; inv_scale: optional device scalar multiplied into the
 * result; d_x: [n,3] out (per sample, also when the input is shared by a group: sum over the group is the caller's). */
int nm_pe_backward(nm_ctx* ctx, int slot, int32_t which, const float* x, int64_t group, const float* d_enc,
                   int32_t ld, const float* inv_scale, int64_t n, float* d_x, void* stream);

/* The nine 256-wide weight-gradient GEMMs of one backward pass, dW = G^T @ X with K = n (torch autograd's
 * grad_output.t() @ input of nn.Linear), reading every fp16 plane once:
 *   out[k], k = 0..6 : pts_linears.(k+1) w.r.t. its 256 hidden inputs = g_pre[k+1]^T @ stash_x[k]
 *   out[7]           : feature_linear                                 = g_f^T @ stash_x[7]
 *   out[8][:128]     : views_linears.0, feature columns               = g_v^T @ stash_f   (rows 128.. are zero)
 * out: [9][256][256] fp32, overwritten; bias_out: [9][256] fp32, overwritten with the column sums of the item's
 * g plane (= the bias gradients of pts_linears 1..7, feature_linear, views_linears.0[:128]); both carry the
 * loss scale of the g planes. */
int nm_dw_gemm(nm_ctx* ctx, const void* g_pre, const void* g_f, const void* g_v, const void* stash_x,
               const void* stash_f, int64_t n, float* out, float* bias_out, void* stream);

/* Same network, but the sample positions are generated in-kernel: pts[r,s] = o[r] + d[r]*z[r,s],
 * views = d[r] (utils/ray_utils.py:131-132).  o,d: [R,3]; z: [R,S]; raw: [R,S,4]. */
int nm_mlp_forward_rays(nm_ctx* ctx, int slot, int mode, const float* origins, const float* dirs,
                        const float* z, int64_t R, int32_t S, float* raw, void* stream);

/* ---- rays: utils/ray_utils.py:23-38 (shot_rays, shot_all_rays) ---------------------------- */
typedef struct {
  double K[9];      /* intrinsic 3x3, row-major (cap.intrinsic_matrix)          */
  double c2w[16];   /* camera_to_world 4x4 (cap.cam_pose.camera_to_world)        */
  int32_t H, W;
} nm_camera;

/* mode 0: shot_rays semantics (point cast to f32, subtract + normalise in f32; :23-29)
 * mode 1: shot_all_rays semantics (all f64, cast last; :32-38 + render_utils.py:114-115)
 * Pixels are the row-major range [pix0, pix0+n) of the HxW grid, or, if xy != NULL, the n integer
 * (x,y) pairs in xy (device int32 [n,2]). */
int nm_raygen(nm_ctx* ctx, const nm_camera* cam, int mode, int64_t pix0, int64_t n,
              const int32_t* xy, float* origins, float* dirs, void* stream);

/* geometry_guided_near_far (utils/ray_utils.py:197-233): near/far [R]; miss => near=+inf,far=-inf */
int nm_near_far(nm_ctx* ctx, const float* origins, const float* dirs, int64_t R,
                const float* verts, int32_t n_verts, float geo_threshold,
                float* near_out, float* far_out, void* stream);

/* The same near/far against the mesh of `actor` set by nm_mesh_set, as the frame drivers compute it: vertex groups of 32
 * with a bounding sphere each, culled conservatively per ray, so the result equals the exhaustive loop's. */
int nm_near_far_mesh(nm_ctx* ctx, int actor, const float* origins, const float* dirs, int64_t R, float geo_threshold,
                     float* near_out, float* far_out, void* stream);

/* ray_to_samples (utils/ray_utils.py:96-135). near/far: [R] or NULL with the scalar fallback;
 * t_rand: [R,S] uniforms for perturb>0 (clipped to [0.01,0.99] inside, :121-125) or NULL.
 * pts/dirs may be NULL when only z is wanted. */
int nm_ray_to_samples(nm_ctx* ctx, const float* origins, const float* dirs, const float* near_v,
                      const float* far_v, float near_s, float far_s, int64_t R, int32_t S,
                      int32_t lindisp, const float* t_rand, float* pts, float* dirs_out, float* z,
                      void* stream);

/* sample_pdf (utils/ray_utils.py:164-194): bins [R,B], weights [R,B-1], u: [R,N] or NULL (det=True
 * linspace).  out [R,N]. */
int nm_sample_pdf(nm_ctx* ctx, const float* bins, const float* weights, int64_t R, int32_t B,
                  int32_t N, const float* u, float* out, void* stream);

/* ray_to_importance_samples (utils/ray_utils.py:138-160), det=True: z [R,S], weights [R,S] ->
 * z_out [R, S+N] sorted (including_old) or [R,N]; pts/dirs_out optional. */
int nm_importance_samples(nm_ctx* ctx, const float* origins, const float* dirs, const float* z,
                          const float* weights, int64_t R, int32_t S, int32_t N,
                          int32_t including_old, float* pts, float* dirs_out, float* z_out,
                          void* stream);

/* raw2outputs (utils/render_utils.py:69-105).  noise: [R,S] added to sigma or NULL; sigma_scale
 * folds `out[..., -1] *= interval_comp` (:229).  Any output pointer may be NULL. */
int nm_raw2outputs(nm_ctx* ctx, const float* raw, const float* z, const float* rays_d, int64_t R,
                   int32_t S, const float* noise, float sigma_scale, int32_t white_bkg,
                   float* rgb, float* disp, float* acc, float* weights, float* depth, void* stream);

/* Backward of raw2outputs for training (trainers/vanilla_nerf_trainer.py:64,80; SURVEY.md §8f-1): gradients of
 * rgb_map [R,3], depth_map [R], acc_map [R], weights [R,S] (each may be NULL) -> grad_raw [R,S,4].
 * disp_map is not differentiated (no caller uses its gradient). */
int nm_raw2outputs_backward(nm_ctx* ctx, const float* raw, const float* z, const float* rays_d, int64_t R,
                            int32_t S, const float* noise, float sigma_scale, int32_t white_bkg,
                            const float* grad_rgb, const float* grad_depth, const float* grad_acc,
                            const float* grad_weights, float* grad_raw, void* stream);

/* z-sorted merge of several per-ray sample lists + gather of raw (utils/render_utils.py:330-337,
 * :441-448): lists k=0..n_lists-1 with z_k [R,S_k], raw_k [R,S_k,4] -> z_out [R,sum S_k],
 * raw_out [R,sum S_k,4].  Ties keep list order then sample order (stable). */
int nm_merge_samples(nm_ctx* ctx, int32_t n_lists, const float* const* z_lists,
                     const float* const* raw_lists, const int32_t* S_list, int64_t R,
                     float* z_out, float* raw_out, void* stream);

/* ---- observation -> canonical warp: utils/ray_utils.py:48-66 ------------------------------ */
/* Per-frame mesh of one actor: verts [V,3] f32, faces [F,3] int32, T [>=V,4,4] f64 (HOST or DEVICE
 * pointers, flag `on_device`).  Builds the closest-point BVH.  T may be NULL (n_T = 0) when only
 * nm_signed_distance will query the mesh. */
int nm_mesh_set(nm_ctx* ctx, int actor, const float* verts, int32_t n_verts, const int32_t* faces,
                int32_t n_faces, const double* T, int32_t n_T, int32_t on_device, void* stream);
/* pts [R,S,3] f32 -> can_pts, can_dirs [R,S,3] f32 (the reference's float64 results cast with
 * .float(), utils/render_utils.py:226-227); closest [R,S,3] f32 and face_id [R,S] optional. */
int nm_warp_to_canonical(nm_ctx* ctx, int actor, const float* pts, int64_t R, int32_t S,
                         float* can_pts, float* can_dirs, float* closest, int32_t* face_id,
                         void* stream);

/* igl.signed_distance(P, V, F) as the reference calls it (utils/ray_utils.py:70, trainers/human_nerf_trainer.py:310,
 * 326) on the mesh of `actor`: S [n] f64 signed distance (pseudo-normal sign: negative inside), I [n] int32 closest
 * face, C [n,3] f64 closest point; any of the three may be NULL.  pts: [n,3] f32. */
int nm_signed_distance(nm_ctx* ctx, int actor, const float* pts, int64_t n, double* S, int32_t* I, double* C,
                       void* stream);

/* ---- SMPL per-vertex transforms: models/smpl.py:109-162,266-505; data_io/neuman_helper.py:299-330 ---- */
typedef struct {
  const float* v_template;   /* [V,3]      DEVICE  (models/smpl.py:81-83)  */
  const float* shapedirs;    /* [V,3,NB]   DEVICE  (:86-88)                */
  const float* J_regressor;  /* [J,V]      DEVICE  (:90-91)                */
  const float* weights;      /* [V,J]      DEVICE  lbs_weights (:106-107)  */
  const int32_t* parents;    /* [J]        HOST    kintree_table[0], parents[0] = -1 (:101-104) */
  int32_t n_verts, n_joints, n_betas;
} nm_smpl_model;

/* SMPL.verts_transformations(poses, betas, concat_joints) (models/smpl.py:109-162), float32:
 * pose [3*J], betas [NB] DEVICE -> T [V(+J),4,4], verts [V(+J),3] (v_shaped (+ joints); may be NULL). */
int nm_smpl_vertex_transforms(nm_ctx* ctx, const nm_smpl_model* model, const float* pose, const float* betas,
                              int32_t concat_joints, float* T, float* verts, void* stream);

/* read_smpls / HumanNeRF.vertex_forward (data_io/neuman_helper.py:299-330, models/human_nerf.py:92-122):
 * T_da2scene = S . alignment^T . T_t2pose . inv(T_t2da) as float64 [V+J,4,4] (the `Ts` the warp consumes) and
 * world_verts = T_da2scene . da_pose_verts as float32 [V+J,3] (vertices then joints; may be NULL).
 * pose, da_pose, betas DEVICE; alignment (4x4 row-major) HOST. */
int nm_smpl_scene_transforms(nm_ctx* ctx, const nm_smpl_model* model, const float* pose, const float* da_pose,
                             const float* betas, const double* alignment, double scale, double* T_da2scene,
                             float* world_verts, void* stream);

/* ---- human trainer: differentiable observation -> canonical map (SURVEY.md 8f-1) ------------------------------- */
/* warp_samples_to_canonical_diff (utils/ray_utils.py:69-93) after its igl.signed_distance call (:70; here
 * nm_signed_distance): f_id [n] closest face and closest [n,3] f64 closest point of every sample (constants of the step,
 * as in the reference), verts [V,3] f32, faces [F,3] int32, T [V,4,4] f32 (HumanNeRF.vertex_forward's raw_Ts)
 * -> Tinv [n,4,4] f32 = inverse of the barycentric blend of the three vertex transforms (:72-91). */
int nm_warp_diff_forward(nm_ctx* ctx, const int32_t* f_id, const double* closest, const float* verts,
                         const int32_t* faces, const float* T, int64_t n, float* Tinv, void* stream);
/* What torch autograd computes for those lines in loss.backward() (trainers/human_nerf_trainer.py:205): g_Tinv [n,4,4]
 * -> g_T [n_verts,4,4] (through blend and inverse) and g_verts [n_verts,3] (through the barycentric coordinates).
 * Both outputs are overwritten (zeroed, then accumulated with atomics); either may be NULL. */
int nm_warp_diff_backward(nm_ctx* ctx, const int32_t* f_id, const double* closest, const float* verts,
                          const int32_t* faces, const float* T, int64_t n, const float* g_Tinv, int32_t n_verts,
                          float* g_T, float* g_verts, void* stream);
/* The same map fused with what the trainer does next (trainers/human_nerf_trainer.py:272-276): pts [R,S,3] ->
 * can_pts = (Tinv @ [pts;1])[:3] + offset (offset [R,S,3] or NULL) and can_dirs = unit differences of consecutive
 * canonical points along the ray, the last sample repeating the previous direction (may be NULL).  S >= 2. */
int nm_human_canonicalize(nm_ctx* ctx, const int32_t* f_id, const double* closest, const float* verts,
                          const int32_t* faces, const float* T, const float* pts, const float* offset, int64_t R,
                          int32_t S, float* can_pts, float* can_dirs, void* stream);
/* Its adjoint: g_can_pts / g_can_dirs [R,S,3] (either may be NULL), can_pts = the forward's output ->
 * g_offset [R,S,3] (required; it is the total dL/d can_pts, i.e. also dL/d offset), g_T [n_verts,4,4], g_verts [n_verts,3]
 * (overwritten; may be NULL). */
int nm_human_canonicalize_backward(nm_ctx* ctx, const int32_t* f_id, const double* closest, const float* verts,
                                   const int32_t* faces, const float* T, const float* pts, const float* can_pts,
                                   const float* g_can_pts, const float* g_can_dirs, int64_t R, int32_t S,
                                   int32_t n_verts, float* g_offset, float* g_T, float* g_verts, void* stream);
/* HumanNeRF.vertex_forward (models/human_nerf.py:92-122) for training: float32 like the reference's torch code, all
 * parameters on the DEVICE (pose [3J], da_pose [3J], betas [NB], alignment [4,4] row-major = self.alignments[idx]):
 * T_da2scene [V,4,4] = S . alignment^T . T_t2pose . inv(T_t2da), world_verts [V,3] (may be NULL) = T_da2scene . da-pose
 * vertices.  Vertices only (the trainer does not use the joint rows). */
int nm_smpl_scene_forward_train(nm_ctx* ctx, const nm_smpl_model* model, const float* pose, const float* da_pose,
                                const float* betas, const float* alignment, float scale, float* T_da2scene,
                                float* world_verts, void* stream);
/* Its adjoint (what loss.backward() sends to HumanNeRF.poses / betas / alignments, models/human_nerf.py:36-38):
 * g_T [V,4,4], g_world [V,3] (either may be NULL) -> g_pose [3J], g_betas [NB], g_alignment [4,4] (overwritten). */
int nm_smpl_scene_backward(nm_ctx* ctx, const nm_smpl_model* model, const float* pose, const float* da_pose,
                           const float* betas, const float* alignment, float scale, const float* g_T,
                           const float* g_world, float* g_pose, float* g_betas, float* g_alignment, void* stream);

/* ---- frame drivers: utils/render_utils.py:108-461 ----------------------------------------- */
typedef struct {
  int32_t samples_per_ray;              /* S */
  int32_t importance_samples_per_ray;   /* N (0 = no fine pass) */
  int32_t white_bkg;
  int32_t mlp_mode;                     /* NM_MLP_* */
  int32_t rays_per_batch;               /* device-side chunk; results do not depend on it */
  int32_t render_can;                   /* render_smpl_nerf: skip the warp (:214-216) */
  float near_bkg, far_bkg;              /* cap.near['bkg'], cap.far['bkg'] */
  float geo_threshold;
  float interval_comp;
} nm_render_opts;

/* All drivers render n pixels of the frame into caller buffers rgb [n,3], depth [n], acc [n] (acc may be NULL):
 * the row-major pixel range [pix0, pix0+n) when `pixels` is NULL, else the row-major pixel indices pixels[0..n)
 * (DEVICE int32; pix0 ignored) -- the ray shard of one GPU, e.g. its interleaved 16x16 tiles (SURVEY.md §8e).
 * `host_out` != 0: the output pointers are HOST memory and the call copies device->host and synchronises before
 * returning. */
int nm_render_vanilla(nm_ctx* ctx, int coarse_slot, int fine_slot /* -1 = none */,
                      const nm_camera* cam, const nm_render_opts* opt, int64_t pix0, int64_t n,
                      const int32_t* pixels, float* rgb, float* depth, int32_t host_out, void* stream);
/* render_vanilla(..., ablate_nerft=True) (utils/render_utils.py:134-148) of NeRF-T coarse (and fine) nets: every sample
 * carries the time `frame_time` (the reference's float32 frame_id / total_frames).  Arguments otherwise as
 * nm_render_vanilla, whose chunk loop it shares. */
int nm_render_vanilla_t(nm_ctx* ctx, int coarse_slot, int fine_slot /* -1 = none */,
                        const nm_camera* cam, const nm_render_opts* opt, float frame_time, int64_t pix0, int64_t n,
                        const int32_t* pixels, float* rgb, float* depth, int32_t host_out, void* stream);
int nm_render_smpl_nerf(nm_ctx* ctx, int human_slot, int actor, const nm_camera* cam,
                        const nm_render_opts* opt, int64_t pix0, int64_t n, const int32_t* pixels, float* rgb,
                        float* depth, float* acc, int32_t host_out, void* stream);
int nm_render_hybrid(nm_ctx* ctx, int coarse_slot, int fine_slot, int32_t n_actors,
                     const int32_t* human_slots, const int32_t* actors, int32_t multi_person,
                     const nm_camera* cam, const nm_render_opts* opt, int64_t pix0, int64_t n,
                     const int32_t* pixels, float* rgb, float* depth, float* acc, int32_t host_out, void* stream);

/* Reassembly of a frame from the ranks' shards after the one gather of SURVEY.md §8e (the reference concatenates its
 * batches and reshapes, utils/render_utils.py:157-161; here a shard is a pixel list).  `shards` is the gathered buffer
 * [world][planes * per] floats, each shard laid out as rgb [per,3] | depth [per] | acc [per] (planes = 5) or without acc
 * (planes = 4); pixels_all [world * per] DEVICE int32 holds the row-major pixel index of every shard entry, < 0 for the
 * padding of short shards.  Writes rgb [HW,3], depth [HW] and acc [HW] (acc may be NULL). */
int nm_assemble_frame(nm_ctx* ctx, const float* shards, int32_t world, int64_t per, int32_t planes,
                      const int32_t* pixels_all, float* rgb, float* depth, float* acc, void* stream);

/* Optional timing of the MLP kernel launches (the dominant kernel; bench.py's roofline): when enabled,
 * every MLP launch is bracketed by CUDA events on its own stream.  nm_profile_read synchronises on
 * them and returns the summed device time, the number of launches and of network evaluations. */
int nm_profile_enable(nm_ctx* ctx, int32_t on);
int nm_profile_read(nm_ctx* ctx, double* mlp_ms, int64_t* mlp_launches, int64_t* mlp_evals);

/* Range guard of the tensor-core MLP (NM_MLP_TC_F16).  Its operands are fp16: conversions saturate at +-65504
 * (cvt.satfinite) instead of producing inf, and every kernel ORs a sticky flag into device memory when an encoded input
 * or a hidden activation reached that limit.  The reference has no counterpart (its fp32 nets cannot overflow at such
 * magnitudes, models/vanilla.py:120-152); this is the check a trained checkpoint with large activations needs.
 * Synchronises on `stream`, returns NM_ERR_RANGE if the flag was set since the last clearing call, NM_OK otherwise. */
int nm_range_status(nm_ctx* ctx, int32_t clear, void* stream);

/* statistics of the last driver call on this ctx: number of MLP evaluations executed (for the
 * roofline: x 1,186,816 FLOP, SURVEY.md §8d) and number of hit rays. */
int nm_last_render_stats(const nm_ctx* ctx, int64_t* mlp_evals, int64_t* hit_rays);

#ifdef __cplusplus
}
#endif
#endif /* NEUMAN_B200_H */

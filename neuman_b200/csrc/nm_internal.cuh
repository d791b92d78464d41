// Internal declarations shared by the translation units of libneuman_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>

#include "neuman_b200.h"

#define NM_WIDTH 256          // nerf_width  (options/options.py:55)
#define NM_DEPTH 8            // nerf_depth  (options/options.py:54)
#define NM_POS_PE 63          // 3 + 3*2*10  (models/vanilla.py:60-79)
#define NM_POS_PE_T 84        // 4 + 4*2*10: position encoding of a NeRF-T net, (x, y, z, t) (train.py:254-256)
#define NM_DIR_PE 27          // 3 + 3*2*4
#define NM_VIEWS_HID 128      // width/2     (models/vanilla.py:112)
#define NM_RANGE_FLAG_WORD 32  // word of ctx->d_counter the tensor-core kernels OR their range flag into

// ---- packed network ------------------------------------------------------------------------
// Net kinds: NeRF with use_viewdirs=True (alpha / feature / views / rgb heads, nm_net_pack) or use_viewdirs=False
// (one output_linear [4,256] on layer 7, no direction input, nm_net_pack_noview; models/vanilla.py:117-118,145-146),
// or a view-dependent NeRF-T net whose position input carries the time as a fourth column (--ablate_nerft,
// nm_net_pack_nerft; rendered and trained, no input gradients).
enum { NM_NET_VIEW = 0, NM_NET_NOVIEW = 1, NM_NET_NERFT = 2 };

// fp32 transposed weights ([in_padded][out]) for the SIMT kernel live in one device allocation per slot; the
// tensor-core kernels read fp16 slabs in the 128B-swizzled wgmma layout from their own allocations.
struct NmNet {
  bool packed = false;
  int kind = NM_NET_VIEW;
  nm_nerf_desc desc{};              // view-independent nets: the trunk and position-encoding fields; head pointers null
  // SIMT fp32 layout: Wt[k][n] (k = input index, n = output index), biases as given
  float* f32 = nullptr;             // base allocation
  size_t f32_floats = 0;
  int f32_pos_k = 0;                // position-encoding width the f32 layout is sized for (NM_POS_PE or NM_POS_PE_T)
  // offsets (in floats) into f32
  size_t o_pts_w[8], o_pts_b[8], o_feat_w, o_feat_b, o_alpha_w, o_alpha_b, o_views_w, o_views_b,
      o_rgb_w, o_rgb_b, o_pos_bv, o_dir_bv, o_pos_cyc, o_dir_cyc,
      o_out_w, o_out_b;             // output_linear of a view-independent net: Wt [256][4], bias [4]
  // tensor-core layout (see mlp_tc.cu for the tile format)
  __half* f16 = nullptr;
  size_t f16_halfs = 0;
  float* tc_bias = nullptr;         // epilogue constants: alpha weights, output biases (mlp_tc.cu k_tc_consts)
  __half* f16_bwd = nullptr;        // transposed slabs for the backward chain (mlp_tc_bwd.cu), packed on first use
  float* bw_wrgb = nullptr;         // backward kernel's constant bank: rgb_linear.weight as [3][128] (view-independent
                                    // nets: output_linear.weight as [4][256])
  size_t bwd_bytes = 0, bw_wrgb_floats = 0;   // sizes of the two, which depend on the kind
  bool bwd_packed = false;
  nm_nerf_desc pe_desc{};           // description the uploaded encoding tables were built from
  bool pe_valid = false;
};

struct NmMesh {
  bool set = false;
  int32_t n_verts = 0, n_faces = 0, n_T = 0;
  float* verts = nullptr;      // [V,3] f32
  int32_t* faces = nullptr;    // [F,3]
  double* T = nullptr;         // [n_T,16] f64
  size_t cap_verts = 0, cap_faces = 0, cap_T = 0;
  // closest-face queries (warp.cu): one device block holds the LBVH and its build buffers (warp.cu: bvh_layout)
  char* bvh = nullptr;
  size_t cap_bvh = 0;             // bytes
  // near/far culling (rays.cu): vertices in Morton order, 32 per group, one bounding sphere per group
  float4* vsorted = nullptr;      // [n_vgroups * 32] (x, y, z, 0); the tail of the last group repeats its first vertex
  float4* vgroup = nullptr;       // [n_vgroups] centre + radius
  int32_t n_vgroups = 0;
  float4 vbound = {0, 0, 0, 0};   // bounding sphere of all vertices (whole-block early out)
  size_t cap_vsorted = 0, cap_vgroup = 0;
  // signed-distance support (warp.cu): angle-weighted vertex pseudo-normals, face across each edge; built on first use
  bool has_T = false, pn_valid = false;
  double* vnorm = nullptr;        // [V,3]
  int32_t* adj = nullptr;         // [F,3]: face sharing edge (v0v1, v1v2, v2v0), -1 on a boundary
  char* pn_tmp = nullptr;         // sort buffers of the adjacency build
  size_t cap_vnorm = 0, cap_adj = 0, cap_pn_tmp = 0;
};

struct nm_ctx {
  int device = 0;
  int sm_count = 132;
  std::string err;
  int64_t launches = 0;
  NmNet nets[NM_MAX_NET_SLOTS];
  NmMesh meshes[NM_MAX_ACTORS];
  // grow-only workspace arena for the frame drivers
  char* ws = nullptr;
  size_t ws_bytes = 0;
  int64_t last_mlp_evals = 0;
  int64_t last_hit_rays = 0;
  uint32_t range_seq = 0;         // launch counter of the tensor-core MLP (rotates the phase of its sampled range check)
  int32_t* d_counter = nullptr;   // small device scratch (compaction counters)
  int32_t* h_counter = nullptr;   // pinned host mirror
  cudaEvent_t ev_counts = nullptr;   // marks the hit counts' arrival on the host (render.cu)
  double* can64 = nullptr;        // float64 canonical points scratch (warp.cu)
  // optional per-launch timing of the MLP kernel (bench.py roofline): event pairs on the launch stream
  bool profile = false;
  std::vector<cudaEvent_t> prof_events;   // start0, stop0, start1, stop1, ...
  size_t prof_used = 0;
  int64_t prof_evals = 0;
  size_t can64_cap = 0;
  int32_t* face_tmp = nullptr;    // winning-face scratch of the warp stage (warp.cu)
  size_t face_cap = 0;
};

// Every C entry point runs on the ctx's device whatever device the calling thread has current (a process may hold
// one ctx per GPU); the previous device is restored on return.
struct NmDeviceGuard {
  int prev = -1;
  explicit NmDeviceGuard(const nm_ctx* ctx) {
    int cur = -1;
    if (ctx && cudaGetDevice(&cur) == cudaSuccess && cur != ctx->device) {
      prev = cur;
      cudaSetDevice(ctx->device);
    }
  }
  ~NmDeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};
#define NM_ENTER(ctx)                       \
  if (!(ctx)) return NM_ERR_INVALID;        \
  NmDeviceGuard _nm_guard(ctx)

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per device: remember which devices a kernel was prepared on
#define NM_SET_SMEM_ONCE(ctx, kernel, bytes)                                                                  \
  do {                                                                                                        \
    static unsigned long long _done = 0ull;                                                                   \
    const unsigned long long _bit = 1ull << ((ctx)->device & 63);                                             \
    if (!(_done & _bit)) {                                                                                    \
      NM_CHECK_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (bytes))); \
      _done |= _bit;                                                                                          \
    }                                                                                                         \
  } while (0)

#define NM_CHECK_CUDA(ctx, call)                                                         \
  do {                                                                                   \
    cudaError_t _e = (call);                                                             \
    if (_e != cudaSuccess) {                                                             \
      (ctx)->err = std::string(#call) + ": " + cudaGetErrorString(_e) + " (" + __FILE__ + \
                   ":" + std::to_string(__LINE__) + ")";                                 \
      return NM_ERR_CUDA;                                                                \
    }                                                                                    \
  } while (0)

#define NM_FAIL(ctx, code, msg)     \
  do {                              \
    (ctx)->err = (msg);             \
    return (code);                  \
  } while (0)

#define NM_LAUNCHED(ctx) ((ctx)->launches++)

#define NM_CHECK_LAUNCH(ctx)                 \
  do {                                       \
    NM_LAUNCHED(ctx);                        \
    NM_CHECK_CUDA(ctx, cudaGetLastError());  \
  } while (0)

// Grow-only device buffer: *p holds at least `need` elements of T afterwards (*cap = its capacity).  Growing
// synchronises the device before the free, since work already queued on any stream may still read the old buffer,
// and reserves 1/8 more than asked so that slowly growing sizes do not reallocate every call.
template <typename T>
static int ensure(nm_ctx* ctx, T** p, size_t* cap, size_t need) {
  if (need <= *cap && *p) return NM_OK;
  if (*p) { NM_CHECK_CUDA(ctx, cudaDeviceSynchronize()); NM_CHECK_CUDA(ctx, cudaFree(*p)); *p = nullptr; }
  const size_t want = need + (need >> 3) + 16;
  NM_CHECK_CUDA(ctx, cudaMalloc(p, want * sizeof(T)));
  *cap = want;
  return NM_OK;
}

// torch.linspace(0, 1, steps) element i in float32: ATen computes start + i*step for the first half
// and end - (steps-1-i)*step for the second half, step = (end-start)/(steps-1).
// Compile units that use this are built with -fmad=false so nothing is contracted.
__host__ __device__ __forceinline__ float nm_linspace01(int i, int steps) {
  if (steps <= 1) return 0.f;
  const float step = 1.0f / (float)(steps - 1);
  if (i < steps / 2) return (float)i * step;
  return 1.0f - (float)(steps - 1 - i) * step;
}

// ---- implemented in the individual .cu files ------------------------------------------------
int nm_impl_workspace(nm_ctx* ctx, size_t bytes, char** out);

// rays.cu: vertex groups of a mesh for the near/far cull (called by nm_mesh_set with the host copy of the vertices), and
// geometry_guided_near_far against a set mesh
int nm_impl_build_vgroups(nm_ctx* ctx, NmMesh& m, const float* host_verts, const float* lo, const float* hi, cudaStream_t st);
int nm_impl_near_far_mesh(nm_ctx* ctx, const NmMesh& m, const float* origins, const float* dirs, int64_t R, float geo_threshold,
                          float* near_out, float* far_out, cudaStream_t st);
// rays.cu: nm_raygen with an optional list of row-major pixel indices
int nm_impl_raygen(nm_ctx* ctx, const nm_camera* cam, int mode, int64_t pix0, int64_t n, const int32_t* xy,
                   const int32_t* pixels, float* origins, float* dirs, cudaStream_t stream);
// composite.cu: raw2outputs whose last sample is followed by zero-density samples starting at z_end
int nm_impl_raw2outputs_zend(nm_ctx* ctx, const float* raw, const float* z, const float* rays_d, int64_t R, int32_t S,
                             int32_t white_bkg, float z_end, float* rgb, float* depth, cudaStream_t st);
// api.cu: nm_mlp_forward_rays with the time of every sample (t, read by NeRF-T slots only)
int nm_impl_mlp_forward_rays(nm_ctx* ctx, int slot, int mode, const float* origins, const float* dirs, const float* z,
                             int64_t R, int32_t S, float t, float* raw, cudaStream_t st);
// mlp_simt.cu
int nm_simt_forward(nm_ctx* ctx, const NmNet& net, const float* pts, const float* views,
                    const float* origins, const float* dirs, const float* z, int64_t n,
                    int32_t group, float t, float* raw, cudaStream_t st);
// mlp_tc.cu
int nm_tc_pack(nm_ctx* ctx, NmNet& net, cudaStream_t st);
// fp16 activation stash written by the training forward and read by the backward chain (mlp_tc_bwd.cu)
struct NmTrainStash {
  __half* x;     // [8][n][256] post-ReLU outputs of pts_linears 0..7
  __half* f;     // [n][256]    feature_linear output (null for view-independent nets)
  __half* v;     // [n][128]    views layer post-ReLU (null for view-independent nets)
  uint32_t* m;   // [9][n][8]   ReLU sign words: planes 0..7 pts_linears, plane 8 views layer (16 bits per 16 columns, mlp_tc.cu fwd_epi);
                 //             view-independent nets: [8][n][8]
};
int nm_impl_pe_backward(nm_ctx* ctx, const NmNet& net, int which, const float* x, int64_t group, const float* d_enc, int ld,
                        const float* inv_scale, int64_t n, float* d_x, cudaStream_t st);
int nm_tc_encode(nm_ctx* ctx, const NmNet& net, int which, const float* x, int64_t group, int64_t n, __half* out, cudaStream_t st);
int nm_impl_dw_gemm(nm_ctx* ctx, const __half* g_pre, const __half* g_f, const __half* g_v, const __half* st_x,
                    const __half* st_f, int64_t n, float* out, float* bias_out, cudaStream_t st);
int nm_tc_backward(nm_ctx* ctx, NmNet& net, const float* d_raw, const float* scale, int64_t n, const __half* st_v,
                   const uint32_t* st_m, __half* g_pre, __half* g_f, __half* g_v, cudaStream_t st);
int nm_tc_forward(nm_ctx* ctx, NmNet& net, const float* pts, const float* views,
                  const float* origins, const float* dirs, const float* z, int64_t n,
                  int32_t group, float t, float* raw, cudaStream_t st, const NmTrainStash* stash = nullptr);

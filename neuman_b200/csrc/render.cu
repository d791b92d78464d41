// Frame drivers: the per-batch loop bodies of the reference renderers, run as chains of the stage
// kernels over large ray chunks that stay resident in HBM.
//
//   nm_render_vanilla    <- utils/render_utils.py:108-161 (render_vanilla)
//   nm_render_smpl_nerf  <- utils/render_utils.py:164-246 (render_smpl_nerf)
//   nm_render_hybrid     <- utils/render_utils.py:249-362 (render_hybrid_nerf) and
//                           :365-461 (render_hybrid_nerf_multi_persons)
//
// The reference's `rays_per_batch` only bounds its memory; results do not depend on it, so the
// drivers pick their own chunk (opt->rays_per_batch, default 32768 rays) sized for HBM.
#include "nm_internal.cuh"

namespace {

// general torch.linspace(start, end, steps)[i] in float32 (see nm_linspace01)
__device__ __forceinline__ float linspace_f(float start, float end, int i, int steps) {
  if (steps <= 1) return start;
  float step = (end - start) / (float)(steps - 1);
  if (i < steps / 2) return start + step * (float)i;
  return end - step * (float)(steps - 1 - i);
}

__global__ void k_fill_placeholder(float* __restrict__ z, float4* __restrict__ raw, long long R, int S, float start,
                                   float end) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= R * S) return;
  int s = (int)(idx % S);
  z[idx] = linspace_f(start, end, s, S);          // utils/render_utils.py:419
  raw[idx] = make_float4(0.f, 0.f, 0.f, 0.f);     // :418
}

// hit test near < far (utils/render_utils.py:206 / :313) + compaction of hit-ray indices
__global__ void k_compact_hits(const float* __restrict__ near_v, const float* __restrict__ far_v, long long R,
                               int32_t* __restrict__ hit_idx, int32_t* __restrict__ counter) {
  long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  bool hit = r < R && near_v[r] < far_v[r];
  unsigned m = __ballot_sync(0xffffffffu, hit);
  int lane = threadIdx.x & 31;
  int base = 0;
  if (lane == 0 && m) base = atomicAdd(counter, __popc(m));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (hit) hit_idx[base + __popc(m & ((1u << lane) - 1))] = (int32_t)r;
}

__global__ void k_gather_rays(const int32_t* __restrict__ idx, int n, const float* __restrict__ o,
                              const float* __restrict__ d, const float* __restrict__ near_v,
                              const float* __restrict__ far_v, float* __restrict__ oh, float* __restrict__ dh,
                              float* __restrict__ nh, float* __restrict__ fh) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int r = idx[i];
#pragma unroll
  for (int c = 0; c < 3; ++c) { oh[3 * i + c] = o[3 * (size_t)r + c]; dh[3 * i + c] = d[3 * (size_t)r + c]; }
  nh[i] = near_v[r]; fh[i] = far_v[r];
}

// rows of `width` floats: dst[i] = src[idx[i]] (gather) or dst[idx[i]] = src[i] (scatter)
__global__ void k_move_rows(const int32_t* __restrict__ idx, long long n, int width, const float* __restrict__ src,
                            float* __restrict__ dst, int scatter) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * width) return;
  long long i = t / width;
  int c = (int)(t - i * width);
  long long r = idx[i];
  if (scatter) dst[r * width + c] = src[t];
  else dst[t] = src[r * width + c];
}

// flag[r] = 1 for the rays of a near/far pair that hit (near < far)
__global__ void k_mark_hits(const float* __restrict__ near_v, const float* __restrict__ far_v, long long R,
                            float* __restrict__ flag) {
  long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < R && near_v[r] < far_v[r]) flag[r] = 1.f;
}

__global__ void k_fill(float* __restrict__ p, long long n, float v) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) p[t] = v;
}

#define LAUNCH1D(kernel, n, st, ...)                                              \
  do {                                                                            \
    long long _n = (n);                                                           \
    if (_n > 0) {                                                                 \
      kernel<<<(unsigned)((_n + 255) / 256), 256, 0, st>>>(__VA_ARGS__);          \
      NM_CHECK_LAUNCH(ctx);                                                       \
    }                                                                             \
  } while (0)

#define TRY(call)                \
  do {                           \
    int _rc = (call);            \
    if (_rc != NM_OK) return _rc; \
  } while (0)

// Bump allocator over the drivers' workspace; every buffer starts on a 256-byte boundary.  With a zero base it
// only measures: render_frame runs a driver's layout once that way to size the workspace.
struct Arena {
  uintptr_t base = 0;
  size_t off = 0;
  template <typename T>
  T* take(size_t n) {
    off = (off + 255) & ~size_t(255);
    T* p = reinterpret_cast<T*>(base + off);
    off += n * sizeof(T);
    return p;
  }
};

// Output planes of n rays: rgb [n,3], depth [n], acc [n].
struct Planes {
  float *rgb = nullptr, *depth = nullptr, *acc = nullptr;
};

int check_frame(nm_ctx* ctx, const nm_camera* cam, const nm_render_opts* opt, int64_t pix0, int64_t n,
                const int32_t* pixels, const float* rgb, const char* who) {
  if (!cam || !opt || n < 0 || (!pixels && (pix0 < 0 || pix0 + n > (int64_t)cam->H * cam->W)))
    NM_FAIL(ctx, NM_ERR_INVALID, std::string(who) + ": bad camera/options/pixel range");
  if (opt->samples_per_ray <= 0 || opt->importance_samples_per_ray < 0)
    NM_FAIL(ctx, NM_ERR_INVALID, std::string(who) + ": bad sample counts");
  if (!rgb) NM_FAIL(ctx, NM_ERR_INVALID, std::string(who) + ": null rgb");
  return NM_OK;
}

// `nerft`: the driver takes a frame time and needs NeRF-T nets (nm_render_vanilla_t); every other driver takes no time
// and refuses them (the reference's hybrid renderers have no NeRF-T path)
int check_slot(nm_ctx* ctx, int slot, const char* who, bool nerft = false) {
  if (slot < 0 || slot >= NM_MAX_NET_SLOTS || !ctx->nets[slot].packed)
    NM_FAIL(ctx, NM_ERR_STATE, std::string(who) + ": net slot not packed");
  if ((ctx->nets[slot].kind == NM_NET_NERFT) != nerft)
    NM_FAIL(ctx, NM_ERR_UNSUPPORTED, std::string(who) + (nerft ? ": needs NeRF-T nets" : ": NeRF-T nets need the frame time (nm_render_vanilla_t)"));
  return NM_OK;
}

int check_mesh(nm_ctx* ctx, int actor, const char* who) {
  if (actor < 0 || actor >= NM_MAX_ACTORS || !ctx->meshes[actor].set)
    NM_FAIL(ctx, NM_ERR_STATE, std::string(who) + ": mesh not set");
  return NM_OK;
}

// The frame loop of every driver, over chunks of at most C rays.  layout(A, C) takes the driver's own buffers for such
// a chunk; it runs once on a zero base to size the workspace and once on the workspace.  For each chunk the rays are
// generated into o/d (ray_mode as in nm_raygen) and body(c, o, d, dst) runs on its c rays.  dst holds the chunk's
// output planes: the caller's device buffers, or staging when the output goes to the host or the caller's plane is
// null.  With host output the staged planes are copied back and the stream synchronised before the next chunk.
template <typename Layout, typename Body>
int render_frame(nm_ctx* ctx, const nm_camera* cam, const nm_render_opts* opt, int ray_mode, int64_t pix0, int64_t n,
                 const int32_t* pixels, const Planes& out, int host_out, cudaStream_t st, Layout&& layout, Body&& body) {
  const int64_t C = std::min<int64_t>(opt->rays_per_batch > 0 ? opt->rays_per_batch : 32768, n > 0 ? n : 1);
  float *o, *d;
  Planes stage;
  auto take_all = [&](Arena& A) {
    o = A.take<float>(3 * C); d = A.take<float>(3 * C);
    stage.rgb = A.take<float>(3 * C); stage.depth = A.take<float>(C); stage.acc = A.take<float>(C);
    layout(A, C);
  };
  Arena A;
  take_all(A);
  char* ws = nullptr;
  TRY(nm_impl_workspace(ctx, A.off, &ws));
  A = Arena{reinterpret_cast<uintptr_t>(ws)};
  take_all(A);
  ctx->last_mlp_evals = 0; ctx->last_hit_rays = 0;
  for (int64_t i = 0; i < n; i += C) {
    const int64_t c = std::min<int64_t>(C, n - i);
    TRY(nm_impl_raygen(ctx, cam, ray_mode, pix0 + i, c, nullptr, pixels ? pixels + i : nullptr, o, d, st));
    auto dst = [&](float* p, float* s, int w) { return host_out || !p ? s : p + w * i; };
    TRY(body(c, o, d, Planes{dst(out.rgb, stage.rgb, 3), dst(out.depth, stage.depth, 1), dst(out.acc, stage.acc, 1)}));
    if (host_out) {
      auto back = [&](float* p, const float* s, int w) {
        return p ? cudaMemcpyAsync(p + w * i, s, w * c * sizeof(float), cudaMemcpyDeviceToHost, st) : cudaSuccess;
      };
      NM_CHECK_CUDA(ctx, back(out.rgb, stage.rgb, 3));
      NM_CHECK_CUDA(ctx, back(out.depth, stage.depth, 1));
      NM_CHECK_CUDA(ctx, back(out.acc, stage.acc, 1));
      NM_CHECK_CUDA(ctx, cudaStreamSynchronize(st));
    }
  }
  return NM_OK;
}

// background coarse (+fine) pass over C rays already in o/d: leaves raw/z of the last pass in
// (*raw_out, *z_out) with *S_out samples.  utils/render_utils.py:141-153 / :287-298 / :398-409.  t: the time of every
// sample, read by NeRF-T nets only (:134-137)
int bkg_pass(nm_ctx* ctx, int coarse, int fine, const nm_render_opts* opt, const float* o, const float* d, int64_t C,
             float* z_c, float* raw_c, float* w_c, float* z_f, float* raw_f, float** raw_out, float** z_out,
             int* S_out, cudaStream_t st, float t = 0.f) {
  const int S = opt->samples_per_ray, N = opt->importance_samples_per_ray;
  TRY(nm_ray_to_samples(ctx, o, d, nullptr, nullptr, opt->near_bkg, opt->far_bkg, C, S, 0, nullptr, nullptr, nullptr,
                        z_c, st));
  TRY(nm_impl_mlp_forward_rays(ctx, coarse, opt->mlp_mode, o, d, z_c, C, S, t, raw_c, st));
  ctx->last_mlp_evals += C * S;
  if (fine >= 0 && N > 0) {
    TRY(nm_raw2outputs(ctx, raw_c, z_c, d, C, S, nullptr, 1.f, opt->white_bkg, nullptr, nullptr, nullptr, w_c, nullptr, st));
    TRY(nm_importance_samples(ctx, o, d, z_c, w_c, C, S, N, 1, nullptr, nullptr, z_f, st));
    TRY(nm_impl_mlp_forward_rays(ctx, fine, opt->mlp_mode, o, d, z_f, C, S + N, t, raw_f, st));
    ctx->last_mlp_evals += C * (S + N);
    *raw_out = raw_f; *z_out = z_f; *S_out = S + N;
  } else {
    *raw_out = raw_c; *z_out = z_c; *S_out = S;
  }
  return NM_OK;
}

// The rays the actors hit in one chunk: per actor, near/far against its set mesh and the indices of the rays with
// near < far; with `uni` (multi-person) also the rays any actor hits.  Plus the human branch's scratch for them.
struct Hits {
  int n; bool uni; const int32_t* actors;   // actors, multi-person, their mesh slots
  float *nr[NM_MAX_ACTORS], *fr[NM_MAX_ACTORS];
  int32_t* idx[NM_MAX_ACTORS];
  int64_t count[NM_MAX_ACTORS + 1];   // hit rays per actor, then of the union
  int32_t* uidx = nullptr;
  float *flag = nullptr, *zeros = nullptr;
  float *oh, *dh, *nh, *fh, *pts, *cpts, *cdirs, *z, *raw;   // gathered rays, samples, canonical points, net output
  float *rgb, *depth, *acc;                                  // their composite
  void take(Arena& A, int64_t C, int S) {
    for (int a = 0; a < n; ++a) { nr[a] = A.take<float>(C); fr[a] = A.take<float>(C); idx[a] = A.take<int32_t>(C); }
    if (uni) { uidx = A.take<int32_t>(C); flag = A.take<float>(C); zeros = A.take<float>(C); }
    oh = A.take<float>(3 * C); dh = A.take<float>(3 * C); nh = A.take<float>(C); fh = A.take<float>(C);
    pts = A.take<float>(3 * C * S); cpts = A.take<float>(3 * C * S); cdirs = A.take<float>(3 * C * S);
    z = A.take<float>(C * S); raw = A.take<float>(4 * C * S);
    rgb = A.take<float>(3 * C); depth = A.take<float>(C); acc = A.take<float>(C);
  }
};

// Queues the hit lists of the c rays in o/d (utils/render_utils.py:198-206 / :299 / :415) and the read-back of their
// counts, whose arrival on the host ctx->ev_counts marks.  hit_counts() waits for them.
int hit_lists(nm_ctx* ctx, Hits& h, float geo_threshold, const float* o, const float* d, int64_t c, cudaStream_t st) {
  if (!ctx->ev_counts) NM_CHECK_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_counts, cudaEventDisableTiming));
  NM_CHECK_CUDA(ctx, cudaMemsetAsync(ctx->d_counter, 0, sizeof(int32_t) * (h.n + 1), st));
  if (h.uni) { LAUNCH1D(k_fill, c, st, h.flag, c, 0.f); LAUNCH1D(k_fill, c, st, h.zeros, c, 0.f); }
  for (int a = 0; a < h.n; ++a) {
    TRY(nm_impl_near_far_mesh(ctx, ctx->meshes[h.actors[a]], o, d, c, geo_threshold, h.nr[a], h.fr[a], st));
    LAUNCH1D(k_compact_hits, c, st, h.nr[a], h.fr[a], c, h.idx[a], ctx->d_counter + a);
    if (h.uni) LAUNCH1D(k_mark_hits, c, st, h.nr[a], h.fr[a], c, h.flag);
  }
  if (h.uni) LAUNCH1D(k_compact_hits, c, st, h.zeros, h.flag, c, h.uidx, ctx->d_counter + h.n);
  NM_CHECK_CUDA(ctx, cudaMemcpyAsync(ctx->h_counter, ctx->d_counter, sizeof(int32_t) * (h.n + 1), cudaMemcpyDeviceToHost, st));
  NM_CHECK_CUDA(ctx, cudaEventRecord(ctx->ev_counts, st));
  return NM_OK;
}

// Waits for the counts of hit_lists() and adds the actors' hit rays to the frame's statistics (nm_last_render_stats).
int hit_counts(nm_ctx* ctx, Hits& h) {
  NM_CHECK_CUDA(ctx, cudaEventSynchronize(ctx->ev_counts));
  for (int a = 0; a <= h.n; ++a) h.count[a] = ctx->h_counter[a];
  for (int a = 0; a < h.n; ++a) ctx->last_hit_rays += h.count[a];
  return NM_OK;
}

// human branch for the rays actor a hits in one chunk: gathers them from o/d into h.oh/dh/nh/fh, then samples, warp,
// net.  Leaves h.raw [Rh,S,4] and h.z [Rh,S].
int human_branch(nm_ctx* ctx, int slot, const nm_render_opts* opt, const float* o, const float* d, const Hits& h, int a,
                 bool render_can, cudaStream_t st) {
  const int S = opt->samples_per_ray;
  const int64_t Rh = h.count[a];
  LAUNCH1D(k_gather_rays, Rh, st, h.idx[a], (int)Rh, o, d, h.nr[a], h.fr[a], h.oh, h.dh, h.nh, h.fh);
  if (render_can) {                                                          // (:214-216)
    TRY(nm_ray_to_samples(ctx, h.oh, h.dh, h.nh, h.fh, 0, 0, Rh, S, 0, nullptr, nullptr, nullptr, h.z, st));
    TRY(nm_mlp_forward_rays(ctx, slot, opt->mlp_mode, h.oh, h.dh, h.z, Rh, S, h.raw, st));
  } else {
    TRY(nm_ray_to_samples(ctx, h.oh, h.dh, h.nh, h.fh, 0, 0, Rh, S, 0, nullptr, h.pts, nullptr, h.z, st));
    TRY(nm_warp_to_canonical(ctx, h.actors[a], h.pts, Rh, S, h.cpts, h.cdirs, nullptr, nullptr, st));   // (:218-225)
    TRY(nm_mlp_forward(ctx, slot, opt->mlp_mode, h.cpts, h.cdirs, Rh * S, 0, h.raw, st));
  }
  ctx->last_mlp_evals += Rh * S;
  return NM_OK;
}

// nm_render_vanilla and nm_render_vanilla_t (nerft: NeRF-T nets, every sample at time t)
int render_vanilla(nm_ctx* ctx, int coarse_slot, int fine_slot, const nm_camera* cam, const nm_render_opts* opt, bool nerft,
                   float t, int64_t pix0, int64_t n, const int32_t* pixels, float* rgb, float* depth, int32_t host_out,
                   cudaStream_t st, const char* who) {
  TRY(check_frame(ctx, cam, opt, pix0, n, pixels, rgb, who));
  TRY(check_slot(ctx, coarse_slot, who, nerft));
  if (fine_slot >= 0) TRY(check_slot(ctx, fine_slot, who, nerft));
  const int S = opt->samples_per_ray, N = fine_slot >= 0 ? opt->importance_samples_per_ray : 0;
  float *z_c, *raw_c, *w_c, *z_f, *raw_f;
  return render_frame(ctx, cam, opt, 1, pix0, n, pixels, Planes{rgb, depth, nullptr}, host_out, st,   // shot_all_rays (:122)
    [&](Arena& A, int64_t C) {
      z_c = A.take<float>(C * S); raw_c = A.take<float>(4 * C * S); w_c = A.take<float>(C * S);
      z_f = A.take<float>(C * (S + N)); raw_f = A.take<float>(4 * C * (S + N));
    },
    [&](int64_t c, const float* o, const float* d, const Planes& dst) -> int {
      float *raw, *z; int St;
      TRY(bkg_pass(ctx, coarse_slot, fine_slot, opt, o, d, c, z_c, raw_c, w_c, z_f, raw_f, &raw, &z, &St, st, t));
      return nm_raw2outputs(ctx, raw, z, d, c, St, nullptr, 1.f, opt->white_bkg, dst.rgb, nullptr, nullptr, nullptr, dst.depth, st);
    });
}

}  // namespace

// ---------------------------------------------------------------------------------------------
extern "C" int nm_render_vanilla(nm_ctx* ctx, int coarse_slot, int fine_slot, const nm_camera* cam,
                                 const nm_render_opts* opt, int64_t pix0, int64_t n, const int32_t* pixels, float* rgb,
                                 float* depth, int32_t host_out, void* stream) {
  NM_ENTER(ctx);
  return render_vanilla(ctx, coarse_slot, fine_slot, cam, opt, false, 0.f, pix0, n, pixels, rgb, depth, host_out,
                        (cudaStream_t)stream, __func__);
}

extern "C" int nm_render_vanilla_t(nm_ctx* ctx, int coarse_slot, int fine_slot, const nm_camera* cam,
                                   const nm_render_opts* opt, float frame_time, int64_t pix0, int64_t n,
                                   const int32_t* pixels, float* rgb, float* depth, int32_t host_out, void* stream) {
  NM_ENTER(ctx);
  return render_vanilla(ctx, coarse_slot, fine_slot, cam, opt, true, frame_time, pix0, n, pixels, rgb, depth, host_out,
                        (cudaStream_t)stream, __func__);
}

// ---------------------------------------------------------------------------------------------
extern "C" int nm_render_smpl_nerf(nm_ctx* ctx, int human_slot, int actor, const nm_camera* cam,
                                   const nm_render_opts* opt, int64_t pix0, int64_t n, const int32_t* pixels, float* rgb,
                                   float* depth, float* acc, int32_t host_out, void* stream) {
  NM_ENTER(ctx);
  TRY(check_frame(ctx, cam, opt, pix0, n, pixels, rgb, __func__));
  TRY(check_slot(ctx, human_slot, __func__));
  TRY(check_mesh(ctx, actor, __func__));
  cudaStream_t st = (cudaStream_t)stream;
  const int S = opt->samples_per_ray;
  Hits h{1, false, &actor};
  return render_frame(ctx, cam, opt, 0, pix0, n, pixels, Planes{rgb, depth, acc}, host_out, st,   // shot_rays (:186)
    [&](Arena& A, int64_t C) { h.take(A, C, S); },
    [&](int64_t c, const float* o, const float* d, const Planes& dst) -> int {
      TRY(hit_lists(ctx, h, opt->geo_threshold, o, d, c, st));
      TRY(hit_counts(ctx, h));
      const int64_t Rh = h.count[0];
      LAUNCH1D(k_fill, 3 * c, st, dst.rgb, 3 * c, opt->white_bkg ? 1.f : 0.f);             // miss rays (:199-205)
      LAUNCH1D(k_fill, c, st, dst.depth, c, 0.f);
      LAUNCH1D(k_fill, c, st, dst.acc, c, 0.f);
      if (Rh > 0) {
        TRY(human_branch(ctx, human_slot, opt, o, d, h, 0, opt->render_can != 0, st));
        TRY(nm_raw2outputs(ctx, h.raw, h.z, h.dh, Rh, S, nullptr, opt->interval_comp, opt->white_bkg, h.rgb, nullptr, h.acc,
                           nullptr, h.depth, st));                                          // (:229-230)
        LAUNCH1D(k_move_rows, Rh * 3, st, h.idx[0], Rh, 3, h.rgb, dst.rgb, 1);             // (:231-233)
        LAUNCH1D(k_move_rows, Rh, st, h.idx[0], Rh, 1, h.depth, dst.depth, 1);
        LAUNCH1D(k_move_rows, Rh, st, h.idx[0], Rh, 1, h.acc, dst.acc, 1);
      }
      return NM_OK;
    });
}

// ---------------------------------------------------------------------------------------------
extern "C" int nm_render_hybrid(nm_ctx* ctx, int coarse_slot, int fine_slot, int32_t n_actors,
                                const int32_t* human_slots, const int32_t* actors, int32_t multi_person,
                                const nm_camera* cam, const nm_render_opts* opt, int64_t pix0, int64_t n,
                                const int32_t* pixels, float* rgb, float* depth, float* acc, int32_t host_out, void* stream) {
  NM_ENTER(ctx);
  TRY(check_frame(ctx, cam, opt, pix0, n, pixels, rgb, __func__));
  TRY(check_slot(ctx, coarse_slot, __func__));
  if (fine_slot >= 0) TRY(check_slot(ctx, fine_slot, __func__));
  if (n_actors < 1 || n_actors > NM_MAX_ACTORS || !human_slots || !actors || (!multi_person && n_actors != 1))
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_render_hybrid: bad actor list");
  for (int a = 0; a < n_actors; ++a) {
    TRY(check_slot(ctx, human_slots[a], __func__));
    TRY(check_mesh(ctx, actors[a], __func__));
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int S = opt->samples_per_ray, N = fine_slot >= 0 ? opt->importance_samples_per_ray : 0;
  const int Sb = S + N, Sm = Sb + n_actors * S;      // samples of the background and of the full merge
  Hits h{n_actors, multi_person != 0, actors};
  float *z_c, *raw_c, *w_c, *z_f, *raw_f, *z_bh, *raw_bh, *z_m, *raw_m;
  float *z_a[NM_MAX_ACTORS], *raw_a[NM_MAX_ACTORS];
  float *zu_a[NM_MAX_ACTORS], *rawu_a[NM_MAX_ACTORS];      // the same rows, compacted to the rays any actor hits
  return render_frame(ctx, cam, opt, 0, pix0, n, pixels, Planes{rgb, depth, acc}, host_out, st,   // shot_rays (:271 / :386)
    [&](Arena& A, int64_t C) {
      h.take(A, C, S);
      z_c = A.take<float>(C * S); raw_c = A.take<float>(4 * C * S); w_c = A.take<float>(C * S);
      z_f = A.take<float>(C * Sb); raw_f = A.take<float>(4 * C * Sb);
      z_bh = A.take<float>(C * Sb); raw_bh = A.take<float>(4 * C * Sb);   // bkg rows of the hit rays
      z_m = A.take<float>(C * Sm); raw_m = A.take<float>(4 * C * Sm);
      for (int a = 0; multi_person && a < n_actors; ++a) {
        z_a[a] = A.take<float>(C * S); raw_a[a] = A.take<float>(4 * C * S);
        zu_a[a] = A.take<float>(C * S); rawu_a[a] = A.take<float>(4 * C * S);
      }
    },
    [&](int64_t c, const float* o, const float* d, const Planes& dst) -> int {
      // Hit lists FIRST: the counts travel to the host while the background networks run, so the host never waits
      // for them with the GPU idle.
      TRY(hit_lists(ctx, h, opt->geo_threshold, o, d, c, st));
      float *raw_b, *z_b; int St;
      TRY(bkg_pass(ctx, coarse_slot, fine_slot, opt, o, d, c, z_c, raw_c, w_c, z_f, raw_f, &raw_b, &z_b, &St, st));
      TRY(hit_counts(ctx, h));
      if (!multi_person) {
        // all rays first get the background-only composite (miss rays keep it, :301-311)
        TRY(nm_raw2outputs(ctx, raw_b, z_b, d, c, St, nullptr, 1.f, opt->white_bkg, dst.rgb, nullptr, nullptr, nullptr, dst.depth, st));
        LAUNCH1D(k_fill, c, st, dst.acc, c, 0.f);
        const int64_t Rh = h.count[0];
        const int32_t* hit = h.idx[0];
        if (Rh > 0) {
          TRY(human_branch(ctx, human_slots[0], opt, o, d, h, 0, false, st));
          LAUNCH1D(k_move_rows, Rh * St, st, hit, Rh, St, z_b, z_bh, 0);
          LAUNCH1D(k_move_rows, Rh * St * 4, st, hit, Rh, St * 4, raw_b, raw_bh, 0);
          const float* zl[2] = {z_bh, h.z};
          const float* rl[2] = {raw_bh, h.raw};
          const int32_t Sl[2] = {St, S};
          TRY(nm_merge_samples(ctx, 2, zl, rl, Sl, Rh, z_m, raw_m, st));                  // (:330-337)
          TRY(nm_raw2outputs(ctx, raw_m, z_m, h.dh, Rh, St + S, nullptr, 1.f, opt->white_bkg, h.rgb, nullptr, nullptr, nullptr,
                             h.depth, st));                                                // (:338-343)
          TRY(nm_raw2outputs(ctx, h.raw, h.z, h.dh, Rh, S, nullptr, 1.f, opt->white_bkg, nullptr, nullptr, h.acc, nullptr,
                             nullptr, st));                                              // (:345-350)
          LAUNCH1D(k_move_rows, Rh * 3, st, hit, Rh, 3, h.rgb, dst.rgb, 1);
          LAUNCH1D(k_move_rows, Rh, st, hit, Rh, 1, h.depth, dst.depth, 1);
          LAUNCH1D(k_move_rows, Rh, st, hit, Rh, 1, h.acc, dst.acc, 1);
        }
        return NM_OK;
      }
      // Rays no actor hits carry only zero-density placeholders behind the background samples (:418-419): their
      // composite is the background composite whose last interval ends at the first placeholder (z = 2 far), no
      // sort needed.  Rays at least one actor hits go through the full z-sorted merge (:441-448), compacted.
      TRY(nm_impl_raw2outputs_zend(ctx, raw_b, z_b, d, c, St, opt->white_bkg, opt->far_bkg * 2.f, dst.rgb, dst.depth, st));
      for (int a = 0; a < n_actors; ++a) {
        LAUNCH1D(k_fill_placeholder, c * S, st, z_a[a], (float4*)raw_a[a], c, S, opt->far_bkg * 2.f, opt->far_bkg * 3.f);
        const int64_t Rh = h.count[a];
        if (Rh > 0) {
          TRY(human_branch(ctx, human_slots[a], opt, o, d, h, a, false, st));
          LAUNCH1D(k_move_rows, Rh * S, st, h.idx[a], Rh, S, h.z, z_a[a], 1);              // (:438-439)
          LAUNCH1D(k_move_rows, Rh * S * 4, st, h.idx[a], Rh, S * 4, h.raw, raw_a[a], 1);
        }
      }
      const int64_t Ru = h.count[n_actors];
      if (Ru > 0) {
        const float* zl[1 + NM_MAX_ACTORS]; const float* rl[1 + NM_MAX_ACTORS]; int32_t Sl[1 + NM_MAX_ACTORS];
        LAUNCH1D(k_gather_rays, Ru, st, h.uidx, (int)Ru, o, d, h.zeros, h.flag, h.oh, h.dh, h.nh, h.fh);
        LAUNCH1D(k_move_rows, Ru * St, st, h.uidx, Ru, St, z_b, z_bh, 0);
        LAUNCH1D(k_move_rows, Ru * St * 4, st, h.uidx, Ru, St * 4, raw_b, raw_bh, 0);
        zl[0] = z_bh; rl[0] = raw_bh; Sl[0] = St;
        for (int a = 0; a < n_actors; ++a) {
          LAUNCH1D(k_move_rows, Ru * S, st, h.uidx, Ru, S, z_a[a], zu_a[a], 0);
          LAUNCH1D(k_move_rows, Ru * S * 4, st, h.uidx, Ru, S * 4, raw_a[a], rawu_a[a], 0);
          zl[1 + a] = zu_a[a]; rl[1 + a] = rawu_a[a]; Sl[1 + a] = S;
        }
        TRY(nm_merge_samples(ctx, 1 + n_actors, zl, rl, Sl, Ru, z_m, raw_m, st));         // (:441-448)
        TRY(nm_raw2outputs(ctx, raw_m, z_m, h.dh, Ru, Sm, nullptr, 1.f, opt->white_bkg, h.rgb, nullptr, nullptr, nullptr,
                           h.depth, st));                                                // (:449-454)
        LAUNCH1D(k_move_rows, Ru * 3, st, h.uidx, Ru, 3, h.rgb, dst.rgb, 1);
        LAUNCH1D(k_move_rows, Ru, st, h.uidx, Ru, 1, h.depth, dst.depth, 1);
      }
      LAUNCH1D(k_fill, c, st, dst.acc, c, 0.f);
      return NM_OK;
    });
}

// ---------------------------------------------------------------------------------------------
// frame reassembly after the gather of the ranks' pixel-list shards (SURVEY.md §8e)
__global__ void k_assemble_frame(const float* __restrict__ shards, long long per, int planes, long long total,
                                 const int32_t* __restrict__ pixels_all, float* __restrict__ rgb, float* __restrict__ depth,
                                 float* __restrict__ acc) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long pix = pixels_all[i];
  if (pix < 0) return;
  const long long r = i / per, j = i - r * per;
  const float* base = shards + r * planes * per;
  rgb[3 * pix + 0] = base[3 * j + 0];
  rgb[3 * pix + 1] = base[3 * j + 1];
  rgb[3 * pix + 2] = base[3 * j + 2];
  if (depth) depth[pix] = base[3 * per + j];
  if (acc && planes > 4) acc[pix] = base[4 * per + j];
}

extern "C" int nm_assemble_frame(nm_ctx* ctx, const float* shards, int32_t world, int64_t per, int32_t planes,
                                 const int32_t* pixels_all, float* rgb, float* depth, float* acc, void* stream) {
  NM_ENTER(ctx);
  if (!shards || !pixels_all || !rgb || world < 1 || per < 0 || (planes != 4 && planes != 5))
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_assemble_frame: bad argument");
  const long long total = (long long)world * per;
  cudaStream_t st = (cudaStream_t)stream;
  LAUNCH1D(k_assemble_frame, total, st, shards, (long long)per, (int)planes, total, pixels_all, rgb, depth, acc);
  return NM_OK;
}

// Context, workspace, network packing and the MLP entry points of the C ABI.
#include <math.h>
#include <string.h>

#include "nm_internal.cuh"

extern "C" const char* nm_version(void) { return "neuman_b200 0.1 (sm_90a)"; }

extern "C" int nm_ctx_create(int device, nm_ctx** out) {
  if (!out) return NM_ERR_INVALID;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return NM_ERR_CUDA;
  if (cudaSetDevice(device) != cudaSuccess) return NM_ERR_CUDA;
  nm_ctx* c = new nm_ctx();
  c->device = device;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->sm_count = prop.multiProcessorCount;
  if (cudaMalloc(&c->d_counter, 64 * sizeof(int32_t)) != cudaSuccess ||
      cudaMallocHost(&c->h_counter, 64 * sizeof(int32_t)) != cudaSuccess) {
    delete c;
    return NM_ERR_CUDA;
  }
  cudaMemset(c->d_counter, 0, 64 * sizeof(int32_t));
  *out = c;
  return NM_OK;
}

static void free_net(NmNet& n) {
  if (n.f32) cudaFree(n.f32);
  if (n.f16) cudaFree(n.f16);
  if (n.tc_bias) cudaFree(n.tc_bias);
  if (n.f16_bwd) cudaFree(n.f16_bwd);
  if (n.bw_wrgb) cudaFree(n.bw_wrgb);
  n = NmNet();
}

static void free_mesh(NmMesh& m) {
  if (m.verts) cudaFree(m.verts);
  if (m.faces) cudaFree(m.faces);
  if (m.T) cudaFree(m.T);
  if (m.bvh) cudaFree(m.bvh);
  if (m.vnorm) cudaFree(m.vnorm);
  if (m.adj) cudaFree(m.adj);
  if (m.pn_tmp) cudaFree(m.pn_tmp);
  if (m.vsorted) cudaFree(m.vsorted);
  if (m.vgroup) cudaFree(m.vgroup);
  m = NmMesh();
}

extern "C" int nm_ctx_destroy(nm_ctx* ctx) {
  NM_ENTER(ctx);
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  for (auto& n : ctx->nets) free_net(n);
  for (auto& m : ctx->meshes) free_mesh(m);
  if (ctx->ws) cudaFree(ctx->ws);
  if (ctx->can64) cudaFree(ctx->can64);
  if (ctx->face_tmp) cudaFree(ctx->face_tmp);
  for (auto e : ctx->prof_events) cudaEventDestroy(e);
  if (ctx->ev_counts) cudaEventDestroy(ctx->ev_counts);
  if (ctx->d_counter) cudaFree(ctx->d_counter);
  if (ctx->h_counter) cudaFreeHost(ctx->h_counter);
  delete ctx;
  return NM_OK;
}

extern "C" const char* nm_last_error(const nm_ctx* ctx) { return ctx ? ctx->err.c_str() : "null ctx"; }
extern "C" int64_t nm_launch_count(const nm_ctx* ctx) { return ctx ? ctx->launches : 0; }

extern "C" int nm_profile_enable(nm_ctx* ctx, int32_t on) {
  NM_ENTER(ctx);
  ctx->profile = on != 0;
  ctx->prof_used = 0;
  ctx->prof_evals = 0;
  return NM_OK;
}

extern "C" int nm_profile_read(nm_ctx* ctx, double* mlp_ms, int64_t* mlp_launches, int64_t* mlp_evals) {
  NM_ENTER(ctx);
  double total = 0.0;
  for (size_t i = 0; i + 1 < ctx->prof_used; i += 2) {
    NM_CHECK_CUDA(ctx, cudaEventSynchronize(ctx->prof_events[i + 1]));
    float ms = 0.f;
    NM_CHECK_CUDA(ctx, cudaEventElapsedTime(&ms, ctx->prof_events[i], ctx->prof_events[i + 1]));
    total += ms;
  }
  if (mlp_ms) *mlp_ms = total;
  if (mlp_launches) *mlp_launches = (int64_t)(ctx->prof_used / 2);
  if (mlp_evals) *mlp_evals = ctx->prof_evals;
  return NM_OK;
}

extern "C" int nm_range_status(nm_ctx* ctx, int32_t clear, void* stream) {
  NM_ENTER(ctx);
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* d = ctx->d_counter + NM_RANGE_FLAG_WORD;
  int32_t* h = ctx->h_counter + NM_RANGE_FLAG_WORD;
  NM_CHECK_CUDA(ctx, cudaMemcpyAsync(h, d, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (clear) NM_CHECK_CUDA(ctx, cudaMemsetAsync(d, 0, sizeof(int32_t), st));
  NM_CHECK_CUDA(ctx, cudaStreamSynchronize(st));
  if (*h != 0)
    NM_FAIL(ctx, NM_ERR_RANGE, "tensor-core MLP: an input or hidden activation reached the fp16 range limit (|x| >= 65504) and was "
                               "saturated; results of the affected samples are not reliable (use NM_MLP_SIMT_F32 for such networks)");
  return NM_OK;
}

extern "C" int nm_last_render_stats(const nm_ctx* ctx, int64_t* mlp_evals, int64_t* hit_rays) {
  NM_ENTER(ctx);
  if (mlp_evals) *mlp_evals = ctx->last_mlp_evals;
  if (hit_rays) *hit_rays = ctx->last_hit_rays;
  return NM_OK;
}

int nm_impl_workspace(nm_ctx* ctx, size_t bytes, char** out) {
  const int rc = ensure(ctx, &ctx->ws, &ctx->ws_bytes, bytes);
  *out = ctx->ws;
  return rc;
}

// ---------------------------------------------------------------------------------------------
// fp32 packing: every nn.Linear weight [out][in] is stored transposed [in][out].
__global__ void k_transpose(const float* __restrict__ src, float* __restrict__ dst, int n_out, int n_in) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_out * n_in) return;
  int k = idx / n_out, n = idx - k * n_out;      // dst index = k*n_out + n
  dst[idx] = src[(size_t)n * n_in + k];
}

static void pe_table(int kind, float fmin, float fmax, int nf, std::vector<float>& out) {
  // posenc: freq_bands = 2**linspace(min,max,N) (models/vanilla.py:66-67)
  // rotate: bvals = (eye(3) * f_k) @ Rz(45)^T @ Rx(45)^T, cast to float (models/vanilla.py:44-53)
  std::vector<double> f(nf);
  for (int k = 0; k < nf; ++k) {
    double e = nf > 1 ? (double)fmin + ((double)fmax - (double)fmin) * k / (double)(nf - 1) : (double)fmin;
    f[k] = pow(2.0, e);
  }
  if (kind == NM_PE_POSENC) {
    out.resize(nf);
    for (int k = 0; k < nf; ++k) out[k] = (float)f[k];
    return;
  }
  const double h = pow(2.0, 0.5) / 2.0;
  const double rz[3][3] = {{h, -h, 0}, {h, h, 0}, {0, 0, 1}};
  const double rx[3][3] = {{1, 0, 0}, {0, h, -h}, {0, h, h}};
  out.resize((size_t)nf * 9);
  for (int k = 0; k < nf; ++k)
    for (int i = 0; i < 3; ++i) {
      double b[3] = {0, 0, 0}, t[3], u[3];
      b[i] = f[k];
      for (int c = 0; c < 3; ++c) t[c] = b[0] * rz[c][0] + b[1] * rz[c][1] + b[2] * rz[c][2];   // b @ rz.T
      for (int c = 0; c < 3; ++c) u[c] = t[0] * rx[c][0] + t[1] * rx[c][1] + t[2] * rx[c][2];   // @ rx.T
      for (int c = 0; c < 3; ++c) out[((size_t)k * 3 + i) * 3 + c] = (float)u[c];
    }
}

// Tables for the tensor-core path's range reduction "in cycles": every frequency (posenc) / projection row
// (rotate) divided by 2*pi, split into a float hi + float lo pair (double precision source).
static void pe_cycles_table(int kind, float fmin, float fmax, int nf, std::vector<float>& out) {
  const double inv2pi = 0.15915494309189533576888;
  std::vector<float> base;
  pe_table(kind, fmin, fmax, nf, base);              // the float tables the reference semantics use
  if (kind == NM_PE_POSENC) {
    out.resize((size_t)nf * 2);
    for (int k = 0; k < nf; ++k) {
      double v = (double)base[k] * inv2pi;
      float hi = (float)v;
      out[2 * k] = hi;
      out[2 * k + 1] = (float)(v - (double)hi);
    }
    return;
  }
  out.resize((size_t)nf * 3 * 6);
  for (int q = 0; q < 3 * nf; ++q)
    for (int i = 0; i < 3; ++i) {
      double v = (double)base[(size_t)q * 3 + i] * inv2pi;
      float hi = (float)v;
      out[(size_t)q * 6 + i] = hi;
      out[(size_t)q * 6 + 3 + i] = (float)(v - (double)hi);
    }
}

// Packs a validated description of any kind into `slot`.  For a view-independent net (kind NM_NET_NOVIEW) `d` carries
// the trunk and the position encoding, its head pointers are null and its direction-encoding fields a fixed placeholder;
// out_w / out_b are output_linear's weight and bias.  A NeRF-T net (NM_NET_NERFT) has pts_linears.0 [256,84] and .5
// [256,340]; the fp32 layout is sized for them, so a slot that changes between NeRF-T and the other kinds is reallocated.
static int net_pack(nm_ctx* ctx, int slot, const nm_nerf_desc* d, int kind, const float* out_w, const float* out_b,
                    cudaStream_t st) {
  NmNet& n = ctx->nets[slot];
  const int KP = kind == NM_NET_NERFT ? NM_POS_PE_T : NM_POS_PE;
  if (n.f32 && n.f32_pos_k != KP) {
    NM_CHECK_CUDA(ctx, cudaDeviceSynchronize());      // work already queued may still read the old weights
    NM_CHECK_CUDA(ctx, cudaFree(n.f32));
    n.f32 = nullptr;
    n.packed = false;
    n.pe_valid = false;                               // the encoding tables live in the freed layout
  }
  if (!n.f32) {
    // layout (floats)
    size_t off = 0;
    auto take = [&](size_t cnt) { size_t o = off; off += (cnt + 63) & ~size_t(63); return o; };
    for (int l = 0; l < 8; ++l) {
      int K = (l == 0) ? KP : (l == 5 ? KP + NM_WIDTH : NM_WIDTH);
      n.o_pts_w[l] = take((size_t)K * NM_WIDTH);
      n.o_pts_b[l] = take(NM_WIDTH);
    }
    n.o_feat_w = take((size_t)NM_WIDTH * NM_WIDTH); n.o_feat_b = take(NM_WIDTH);
    n.o_alpha_w = take(NM_WIDTH); n.o_alpha_b = take(1);
    n.o_views_w = take((size_t)(NM_WIDTH + NM_DIR_PE) * NM_VIEWS_HID); n.o_views_b = take(NM_VIEWS_HID);
    n.o_rgb_w = take((size_t)NM_VIEWS_HID * 3); n.o_rgb_b = take(3);
    n.o_pos_bv = take(128); n.o_dir_bv = take(128);
    n.o_pos_cyc = take(192); n.o_dir_cyc = take(192);
    n.o_out_w = take((size_t)NM_WIDTH * 4); n.o_out_b = take(4);
    n.f32_floats = off;
    n.f32_pos_k = KP;
    NM_CHECK_CUDA(ctx, cudaMalloc(&n.f32, off * sizeof(float)));
  }
  n.desc = *d;
  n.kind = kind;
  n.bwd_packed = false;
  auto tr = [&](const float* src, size_t dst_off, int n_out, int n_in) {
    int total = n_out * n_in;
    k_transpose<<<(total + 255) / 256, 256, 0, st>>>(src, n.f32 + dst_off, n_out, n_in);
    NM_LAUNCHED(ctx);
  };
  auto cp = [&](const float* src, size_t dst_off, int cnt) {
    return cudaMemcpyAsync(n.f32 + dst_off, src, cnt * sizeof(float), cudaMemcpyDeviceToDevice, st);
  };
  for (int l = 0; l < 8; ++l) {
    int K = (l == 0) ? KP : (l == 5 ? KP + NM_WIDTH : NM_WIDTH);
    tr(d->pts_w[l], n.o_pts_w[l], NM_WIDTH, K);
    NM_CHECK_CUDA(ctx, cp(d->pts_b[l], n.o_pts_b[l], NM_WIDTH));
  }
  if (kind != NM_NET_NOVIEW) {
    tr(d->feature_w, n.o_feat_w, NM_WIDTH, NM_WIDTH);
    NM_CHECK_CUDA(ctx, cp(d->feature_b, n.o_feat_b, NM_WIDTH));
    tr(d->alpha_w, n.o_alpha_w, 1, NM_WIDTH);
    NM_CHECK_CUDA(ctx, cp(d->alpha_b, n.o_alpha_b, 1));
    tr(d->views_w, n.o_views_w, NM_VIEWS_HID, NM_WIDTH + NM_DIR_PE);
    NM_CHECK_CUDA(ctx, cp(d->views_b, n.o_views_b, NM_VIEWS_HID));
    tr(d->rgb_w, n.o_rgb_w, 3, NM_VIEWS_HID);
    NM_CHECK_CUDA(ctx, cp(d->rgb_b, n.o_rgb_b, 3));
  } else {
    tr(out_w, n.o_out_w, 4, NM_WIDTH);
    NM_CHECK_CUDA(ctx, cp(out_b, n.o_out_b, 4));
  }
  NM_CHECK_CUDA(ctx, cudaGetLastError());
  // encoding tables: host-built, uploaded (with a sync, `tab` is a temporary) only when the description changes,
  // so that re-packing updated weights every training step stays asynchronous
  const bool same_pe = n.pe_valid && n.pe_desc.pos_pe_kind == d->pos_pe_kind && n.pe_desc.dir_pe_kind == d->dir_pe_kind &&
                       n.pe_desc.pos_min_freq == d->pos_min_freq && n.pe_desc.pos_max_freq == d->pos_max_freq &&
                       n.pe_desc.dir_min_freq == d->dir_min_freq && n.pe_desc.dir_max_freq == d->dir_max_freq &&
                       n.pe_desc.pos_n_freqs == d->pos_n_freqs && n.pe_desc.dir_n_freqs == d->dir_n_freqs;
  if (!same_pe) {
    std::vector<float> tab;
    pe_table(d->pos_pe_kind, d->pos_min_freq, d->pos_max_freq, d->pos_n_freqs, tab);
    NM_CHECK_CUDA(ctx, cudaMemcpyAsync(n.f32 + n.o_pos_bv, tab.data(), tab.size() * sizeof(float),
                                       cudaMemcpyHostToDevice, st));
    NM_CHECK_CUDA(ctx, cudaStreamSynchronize(st));   // tab is a stack temporary
    pe_table(d->dir_pe_kind, d->dir_min_freq, d->dir_max_freq, d->dir_n_freqs, tab);
    NM_CHECK_CUDA(ctx, cudaMemcpyAsync(n.f32 + n.o_dir_bv, tab.data(), tab.size() * sizeof(float),
                                       cudaMemcpyHostToDevice, st));
    NM_CHECK_CUDA(ctx, cudaStreamSynchronize(st));
    pe_cycles_table(d->pos_pe_kind, d->pos_min_freq, d->pos_max_freq, d->pos_n_freqs, tab);
    NM_CHECK_CUDA(ctx, cudaMemcpyAsync(n.f32 + n.o_pos_cyc, tab.data(), tab.size() * sizeof(float),
                                       cudaMemcpyHostToDevice, st));
    NM_CHECK_CUDA(ctx, cudaStreamSynchronize(st));
    pe_cycles_table(d->dir_pe_kind, d->dir_min_freq, d->dir_max_freq, d->dir_n_freqs, tab);
    NM_CHECK_CUDA(ctx, cudaMemcpyAsync(n.f32 + n.o_dir_cyc, tab.data(), tab.size() * sizeof(float),
                                       cudaMemcpyHostToDevice, st));
    NM_CHECK_CUDA(ctx, cudaStreamSynchronize(st));
    n.pe_desc = *d;
    n.pe_valid = true;
  }
  int rc = nm_tc_pack(ctx, n, st);
  if (rc != NM_OK) return rc;
  n.packed = true;
  return NM_OK;
}

static int check_view_desc(nm_ctx* ctx, const nm_nerf_desc* d, const char* who) {
  for (int l = 0; l < 8; ++l)
    if (!d->pts_w[l] || !d->pts_b[l]) NM_FAIL(ctx, NM_ERR_INVALID, std::string(who) + ": null pts_linears");
  if (!d->feature_w || !d->feature_b || !d->alpha_w || !d->alpha_b || !d->views_w || !d->views_b || !d->rgb_w ||
      !d->rgb_b)
    NM_FAIL(ctx, NM_ERR_INVALID, std::string(who) + ": null head weights (use_viewdirs=True nets only)");
  return NM_OK;
}

extern "C" int nm_net_pack(nm_ctx* ctx, int slot, const nm_nerf_desc* d, void* stream) {
  NM_ENTER(ctx);
  if (slot < 0 || slot >= NM_MAX_NET_SLOTS || !d) NM_FAIL(ctx, NM_ERR_INVALID, "nm_net_pack: bad slot/desc");
  if (d->pos_n_freqs != 10 || d->dir_n_freqs != 4)
    NM_FAIL(ctx, NM_ERR_UNSUPPORTED, "nm_net_pack: only pos_N_freqs=10 / dir_N_freqs=4 (63/27-d encodings) is built");
  const int rc = check_view_desc(ctx, d, __func__);
  if (rc != NM_OK) return rc;
  return net_pack(ctx, slot, d, NM_NET_VIEW, nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" int nm_net_pack_nerft(nm_ctx* ctx, int slot, const nm_nerf_desc* d, void* stream) {
  NM_ENTER(ctx);
  if (slot < 0 || slot >= NM_MAX_NET_SLOTS || !d) NM_FAIL(ctx, NM_ERR_INVALID, "nm_net_pack_nerft: bad slot/desc");
  if (d->pos_n_freqs != 10 || d->dir_n_freqs != 4)
    NM_FAIL(ctx, NM_ERR_UNSUPPORTED, "nm_net_pack_nerft: only pos_N_freqs=10 / dir_N_freqs=4 (84/27-d encodings) is built");
  if (d->pos_pe_kind != NM_PE_POSENC)      // the reference's rotate mapping asserts a 3-D input (models/vanilla.py:84)
    NM_FAIL(ctx, NM_ERR_UNSUPPORTED, "nm_net_pack_nerft: the position encoding of a NeRF-T net must be posenc");
  const int rc = check_view_desc(ctx, d, __func__);
  if (rc != NM_OK) return rc;
  return net_pack(ctx, slot, d, NM_NET_NERFT, nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" int nm_net_pack_noview(nm_ctx* ctx, int slot, const nm_nerf_noview_desc* d, void* stream) {
  NM_ENTER(ctx);
  if (slot < 0 || slot >= NM_MAX_NET_SLOTS || !d) NM_FAIL(ctx, NM_ERR_INVALID, "nm_net_pack_noview: bad slot/desc");
  if (d->pos_n_freqs != 10)
    NM_FAIL(ctx, NM_ERR_UNSUPPORTED, "nm_net_pack_noview: only pos_N_freqs=10 (63-d encoding) is built");
  for (int l = 0; l < 8; ++l)
    if (!d->pts_w[l] || !d->pts_b[l]) NM_FAIL(ctx, NM_ERR_INVALID, "nm_net_pack_noview: null pts_linears");
  if (!d->output_w || !d->output_b) NM_FAIL(ctx, NM_ERR_INVALID, "nm_net_pack_noview: null output_linear");
  nm_nerf_desc full{};
  for (int l = 0; l < 8; ++l) { full.pts_w[l] = d->pts_w[l]; full.pts_b[l] = d->pts_b[l]; }
  full.pos_pe_kind = d->pos_pe_kind;
  full.pos_min_freq = d->pos_min_freq; full.pos_max_freq = d->pos_max_freq; full.pos_n_freqs = d->pos_n_freqs;
  // no direction input: the placeholder only keeps the (unused) direction tables of the slot well defined
  full.dir_pe_kind = NM_PE_POSENC; full.dir_min_freq = 0.f; full.dir_max_freq = 3.f; full.dir_n_freqs = 4;
  return net_pack(ctx, slot, &full, NM_NET_NOVIEW, d->output_w, d->output_b, (cudaStream_t)stream);
}

static int mlp_dispatch(nm_ctx* ctx, int slot, int mode, const float* pts, const float* views, const float* origins,
                        const float* dirs, const float* z, int64_t n, int32_t group, float t, float* raw, void* stream,
                        const NmTrainStash* stash = nullptr) {
  if (slot < 0 || slot >= NM_MAX_NET_SLOTS || !ctx->nets[slot].packed)
    NM_FAIL(ctx, NM_ERR_STATE, "nm_mlp_forward: net slot not packed");
  if (n < 0 || !raw) NM_FAIL(ctx, NM_ERR_INVALID, "nm_mlp_forward: bad argument");
  if (n == 0) return NM_OK;
  NmNet& net = ctx->nets[slot];
  if (mode != NM_MLP_SIMT_F32 && mode != NM_MLP_TC_F16) NM_FAIL(ctx, NM_ERR_INVALID, "nm_mlp_forward: unknown mode");
  cudaStream_t st = (cudaStream_t)stream;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (ctx->profile) {
    if (ctx->prof_used + 2 > ctx->prof_events.size()) {
      for (int k = 0; k < 2; ++k) {
        cudaEvent_t e;
        NM_CHECK_CUDA(ctx, cudaEventCreate(&e));
        ctx->prof_events.push_back(e);
      }
    }
    e0 = ctx->prof_events[ctx->prof_used];
    e1 = ctx->prof_events[ctx->prof_used + 1];
    NM_CHECK_CUDA(ctx, cudaEventRecord(e0, st));
  }
  int rc = mode == NM_MLP_SIMT_F32 ? nm_simt_forward(ctx, net, pts, views, origins, dirs, z, n, group, t, raw, st)
                                   : nm_tc_forward(ctx, net, pts, views, origins, dirs, z, n, group, t, raw, st, stash);
  if (ctx->profile && rc == NM_OK) {
    NM_CHECK_CUDA(ctx, cudaEventRecord(e1, st));
    ctx->prof_used += 2;
    ctx->prof_evals += n;
  }
  return rc;
}

// views of a view-independent slot are never read and may be NULL
static bool views_ok(const nm_ctx* ctx, int slot, const void* views) {
  return views || (slot >= 0 && slot < NM_MAX_NET_SLOTS && ctx->nets[slot].packed && ctx->nets[slot].kind == NM_NET_NOVIEW);
}
static bool is_noview(const nm_ctx* ctx, int slot) {
  return slot >= 0 && slot < NM_MAX_NET_SLOTS && ctx->nets[slot].kind == NM_NET_NOVIEW;
}
static bool is_nerft(const nm_ctx* ctx, int slot) {
  return slot >= 0 && slot < NM_MAX_NET_SLOTS && ctx->nets[slot].packed && ctx->nets[slot].kind == NM_NET_NERFT;
}

extern "C" int nm_mlp_forward(nm_ctx* ctx, int slot, int mode, const float* pts, const float* views, int64_t n,
                              int32_t views_per_ray, float* raw, void* stream) {
  NM_ENTER(ctx);
  if (!pts || !views_ok(ctx, slot, views) || views_per_ray < 0) NM_FAIL(ctx, NM_ERR_INVALID, "nm_mlp_forward: null pts/views");
  if (views_per_ray > 0 && n % views_per_ray != 0)
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_mlp_forward: n is not a multiple of views_per_ray");
  return mlp_dispatch(ctx, slot, mode, pts, views, nullptr, nullptr, nullptr, n, views_per_ray, 0.f, raw, stream);
}

extern "C" int nm_mlp_forward_train(nm_ctx* ctx, int slot, const float* pts, const float* views, int64_t n,
                                    int32_t views_per_ray, float* raw, void* stash_x, void* stash_f, void* stash_v,
                                    void* stash_m, void* stream) {
  NM_ENTER(ctx);
  if (!pts || !views_ok(ctx, slot, views) || views_per_ray < 0) NM_FAIL(ctx, NM_ERR_INVALID, "nm_mlp_forward_train: null pts/views");
  const bool noview = is_noview(ctx, slot);
  if (!stash_x || !stash_m || (!noview && (!stash_f || !stash_v)))
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_mlp_forward_train: null stash");
  if (noview) stash_f = stash_v = nullptr;
  if (views_per_ray > 0 && n % views_per_ray != 0)
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_mlp_forward_train: n is not a multiple of views_per_ray");
  NmTrainStash sh{(__half*)stash_x, (__half*)stash_f, (__half*)stash_v, (uint32_t*)stash_m};
  return mlp_dispatch(ctx, slot, NM_MLP_TC_F16, pts, views, nullptr, nullptr, nullptr, n, views_per_ray, 0.f, raw, stream, &sh);
}

extern "C" int nm_mlp_backward(nm_ctx* ctx, int slot, const float* d_raw, const float* loss_scale, int64_t n,
                               const void* stash_v, const void* stash_m, void* g_pre, void* g_f, void* g_v, void* stream) {
  NM_ENTER(ctx);
  if (slot < 0 || slot >= NM_MAX_NET_SLOTS || !ctx->nets[slot].packed)
    NM_FAIL(ctx, NM_ERR_STATE, "nm_mlp_backward: net slot not packed");
  if (n < 0) NM_FAIL(ctx, NM_ERR_INVALID, "nm_mlp_backward: bad argument");
  if (n == 0) return NM_OK;
  const bool noview = is_noview(ctx, slot);
  if (!d_raw || !loss_scale || !stash_m || !g_pre || (!noview && (!stash_v || !g_f || !g_v)))
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_mlp_backward: null argument");
  if (noview) stash_v = g_f = g_v = nullptr;
  return nm_tc_backward(ctx, ctx->nets[slot], d_raw, loss_scale, n, (const __half*)stash_v, (const uint32_t*)stash_m,
                        (__half*)g_pre, (__half*)g_f, (__half*)g_v, (cudaStream_t)stream);
}

extern "C" int nm_encode_f16(nm_ctx* ctx, int slot, int32_t which, const float* x, int64_t group, int64_t n, void* out,
                             void* stream) {
  NM_ENTER(ctx);
  if (slot < 0 || slot >= NM_MAX_NET_SLOTS || !ctx->nets[slot].packed)
    NM_FAIL(ctx, NM_ERR_STATE, "nm_encode_f16: net slot not packed");
  if ((which != 0 && which != 1) || n < 0 || group < 0) NM_FAIL(ctx, NM_ERR_INVALID, "nm_encode_f16: bad argument");
  if (which == 1 && is_noview(ctx, slot)) NM_FAIL(ctx, NM_ERR_UNSUPPORTED, "nm_encode_f16: view-independent net has no direction encoding");
  if (n == 0) return NM_OK;
  if (!x || !out) NM_FAIL(ctx, NM_ERR_INVALID, "nm_encode_f16: null argument");
  return nm_tc_encode(ctx, ctx->nets[slot], which, x, group, n, (__half*)out, (cudaStream_t)stream);
}

extern "C" int nm_pe_backward(nm_ctx* ctx, int slot, int32_t which, const float* x, int64_t group, const float* d_enc,
                              int32_t ld, const float* inv_scale, int64_t n, float* d_x, void* stream) {
  NM_ENTER(ctx);
  if (slot < 0 || slot >= NM_MAX_NET_SLOTS || !ctx->nets[slot].packed)
    NM_FAIL(ctx, NM_ERR_STATE, "nm_pe_backward: net slot not packed");
  if ((which != 0 && which != 1) || n < 0 || group < 0) NM_FAIL(ctx, NM_ERR_INVALID, "nm_pe_backward: bad argument");
  if (which == 1 && is_noview(ctx, slot)) NM_FAIL(ctx, NM_ERR_UNSUPPORTED, "nm_pe_backward: view-independent net has no direction encoding");
  if (which == 0 && is_nerft(ctx, slot))           // nothing in the reference differentiates through a NeRF-T net's input
    NM_FAIL(ctx, NM_ERR_UNSUPPORTED, "nm_pe_backward: no position-input gradient for NeRF-T nets");
  const NmNet& net = ctx->nets[slot];
  const int width = 3 + 6 * (which == 0 ? net.desc.pos_n_freqs : net.desc.dir_n_freqs);
  if (ld < width) NM_FAIL(ctx, NM_ERR_INVALID, "nm_pe_backward: ld smaller than the encoding width");
  if (n == 0) return NM_OK;
  if (!x || !d_enc || !d_x) NM_FAIL(ctx, NM_ERR_INVALID, "nm_pe_backward: null argument");
  return nm_impl_pe_backward(ctx, net, which, x, group, d_enc, ld, inv_scale, n, d_x, (cudaStream_t)stream);
}

extern "C" int nm_dw_gemm(nm_ctx* ctx, const void* g_pre, const void* g_f, const void* g_v, const void* stash_x,
                          const void* stash_f, int64_t n, float* out, float* bias_out, void* stream) {
  NM_ENTER(ctx);
  if (n < 0 || !out || !bias_out) NM_FAIL(ctx, NM_ERR_INVALID, "nm_dw_gemm: bad argument");
  if (n == 0) {
    NM_CHECK_CUDA(ctx, cudaMemsetAsync(out, 0, (size_t)9 * 256 * 256 * sizeof(float), (cudaStream_t)stream));
    NM_CHECK_CUDA(ctx, cudaMemsetAsync(bias_out, 0, (size_t)9 * 256 * sizeof(float), (cudaStream_t)stream));
    return NM_OK;
  }
  // g_f, g_v and stash_f all NULL: a view-independent net's backward (items 0..6 only)
  const bool trunk_only = !g_f && !g_v && !stash_f;
  if (!g_pre || !stash_x || (!trunk_only && (!g_f || !g_v || !stash_f))) NM_FAIL(ctx, NM_ERR_INVALID, "nm_dw_gemm: null argument");
  return nm_impl_dw_gemm(ctx, (const __half*)g_pre, (const __half*)g_f, (const __half*)g_v, (const __half*)stash_x,
                         (const __half*)stash_f, n, out, bias_out, (cudaStream_t)stream);
}

int nm_impl_mlp_forward_rays(nm_ctx* ctx, int slot, int mode, const float* origins, const float* dirs, const float* z,
                             int64_t R, int32_t S, float t, float* raw, cudaStream_t st) {
  if (!origins || !dirs || !z || S <= 0 || R < 0) NM_FAIL(ctx, NM_ERR_INVALID, "nm_mlp_forward_rays: bad argument");
  return mlp_dispatch(ctx, slot, mode, nullptr, nullptr, origins, dirs, z, R * (int64_t)S, S, t, raw, st);
}

extern "C" int nm_mlp_forward_rays(nm_ctx* ctx, int slot, int mode, const float* origins, const float* dirs,
                                   const float* z, int64_t R, int32_t S, float* raw, void* stream) {
  NM_ENTER(ctx);
  if (is_nerft(ctx, slot)) NM_FAIL(ctx, NM_ERR_UNSUPPORTED, "nm_mlp_forward_rays: a NeRF-T net needs the time (nm_render_vanilla_t)");
  return nm_impl_mlp_forward_rays(ctx, slot, mode, origins, dirs, z, R, S, 0.f, raw, (cudaStream_t)stream);
}

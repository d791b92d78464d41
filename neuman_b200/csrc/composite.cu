// The alpha-composited volume integral and the z-sorted merge of per-ray sample lists.
// Compiled with -fmad=false (mirrors separately-rounded torch elementwise ops).
//
//   nm_raw2outputs    <- utils/render_utils.py:69-105 (raw2outputs)
//   nm_merge_samples  <- utils/render_utils.py:330-337, :441-448 (sort(cat(z)) + gather of raw)
//
// One warp owns one ray: samples are strided across lanes (coalesced float4 loads of raw), the
// exclusive transmittance product is a warp-shuffle scan with a running carry between 32-sample
// chunks, and the weighted sums are butterfly reductions.
#include "nm_internal.cuh"

#define FULL 0xffffffffu

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}

__global__ void __launch_bounds__(256) k_raw2outputs(
    const float4* __restrict__ raw, const float* __restrict__ z, const float* __restrict__ rays_d, long long R,
    int S, const float* __restrict__ noise, float sigma_scale, int white_bkg, float z_end, float* __restrict__ rgb_out,
    float* __restrict__ disp_out, float* __restrict__ acc_out, float* __restrict__ w_out,
    float* __restrict__ depth_out) {
  const int lane = threadIdx.x & 31;
  long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= R) return;
  const float dx = rays_d[3 * r], dy = rays_d[3 * r + 1], dz = rays_d[3 * r + 2];
  const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);              // torch.norm(rays_d) (:88)
  const float* zr = z + r * S;
  const float4* rr = raw + r * S;
  float carry = 1.f;                     // running exclusive product of (1 - alpha + 1e-10)
  float s_r = 0, s_g = 0, s_b = 0, s_d = 0, s_a = 0;
  for (int base = 0; base < S; base += 32) {
    int s = base + lane;
    bool live = s < S;
    float alpha = 0.f, zc = 0.f;
    float4 v = make_float4(0, 0, 0, 0);
    if (live) {
      v = rr[s];
      zc = zr[s];
      // z_end > 0: zero-density samples follow at z_end (multi-person placeholders, render_utils.py:418-419)
      float dist = (s + 1 < S) ? (zr[s + 1] - zc) : (z_end > 0.f ? z_end - zc : 1e10f);   // (:85-86)
      dist = dist * dnorm;                                             // (:88)
      float sg = v.w * sigma_scale;
      if (noise) sg = sg + noise[r * S + s];                           // (:91-94)
      sg = fmaxf(sg, 0.f);
      alpha = 1.f - expf(-sg * dist);                                  // (:83)
    }
    float f = live ? (1.f - alpha + 1e-10f) : 1.f;
    // inclusive scan of f across lanes
    float inc = f;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      float t = __shfl_up_sync(FULL, inc, o);
      if (lane >= o) inc = inc * t;
    }
    float exc = __shfl_up_sync(FULL, inc, 1);
    if (lane == 0) exc = 1.f;
    float T = carry * exc;
    float w = alpha * T;                                               // (:95)
    carry = carry * __shfl_sync(FULL, inc, 31);
    if (live) {
      if (w_out) w_out[r * S + s] = w;
      float cr = 1.f / (1.f + expf(-v.x)), cg = 1.f / (1.f + expf(-v.y)), cb = 1.f / (1.f + expf(-v.z));
      s_r += w * cr; s_g += w * cg; s_b += w * cb;                      // (:96)
      s_d += w * zc;                                                   // (:98)
      s_a += w;                                                        // (:100)
    }
  }
  s_r = warp_sum(s_r); s_g = warp_sum(s_g); s_b = warp_sum(s_b);
  s_d = warp_sum(s_d); s_a = warp_sum(s_a);
  if (lane == 0) {
    if (white_bkg) { float bgw = 1.f - s_a; s_r += bgw; s_g += bgw; s_b += bgw; }   // (:102-103)
    if (rgb_out) { rgb_out[3 * r] = s_r; rgb_out[3 * r + 1] = s_g; rgb_out[3 * r + 2] = s_b; }
    if (depth_out) depth_out[r] = s_d;
    if (acc_out) acc_out[r] = s_a;
    if (disp_out) {                                                    // (:99) torch.max propagates NaN (0/0)
      float q = s_d / s_a;
      disp_out[r] = 1.f / ((q != q) ? q : fmaxf(1e-10f, q));
    }
  }
}

int nm_impl_raw2outputs_zend(nm_ctx* ctx, const float* raw, const float* z, const float* rays_d, int64_t R, int32_t S,
                             int32_t white_bkg, float z_end, float* rgb, float* depth, cudaStream_t st) {
  if (R == 0) return NM_OK;
  unsigned blocks = (unsigned)((R * 32 + 255) / 256);
  k_raw2outputs<<<blocks, 256, 0, st>>>((const float4*)raw, z, rays_d, R, S, nullptr, 1.f, white_bkg, z_end, rgb, nullptr,
                                        nullptr, nullptr, depth);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

extern "C" int nm_raw2outputs(nm_ctx* ctx, const float* raw, const float* z, const float* rays_d, int64_t R,
                              int32_t S, const float* noise, float sigma_scale, int32_t white_bkg, float* rgb,
                              float* disp, float* acc, float* weights, float* depth, void* stream) {
  NM_ENTER(ctx);
  if (R == 0) return NM_OK;
  if (!raw || !z || !rays_d || R < 0 || S <= 0) NM_FAIL(ctx, NM_ERR_INVALID, "nm_raw2outputs: bad argument");
  unsigned blocks = (unsigned)((R * 32 + 255) / 256);
  k_raw2outputs<<<blocks, 256, 0, (cudaStream_t)stream>>>((const float4*)raw, z, rays_d, R, S, noise, sigma_scale,
                                                            white_bkg, -1.f, rgb, disp, acc, weights, depth);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

// ---------------------------------------------------------------------------------------------
// Merge: one warp per ray sorts (z, source index) pairs with a bitonic network in shared memory.
// The source index (position in the concatenated list) is the secondary key, which makes the
// order total and stable -- no assumption that the input lists are already sorted.
struct MergeParams {
  const float* z[1 + NM_MAX_ACTORS];
  const float4* raw[1 + NM_MAX_ACTORS];
  int S[1 + NM_MAX_ACTORS];
  int n_lists;
  int total;
  int pow2;
};

#include "nm_sort.cuh"

#define MERGE_WARPS 4
__global__ void __launch_bounds__(32 * MERGE_WARPS) k_merge(MergeParams p, long long R, float* __restrict__ z_out,
                                                             float4* __restrict__ raw_out) {
  extern __shared__ unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float* keys = reinterpret_cast<float*>(smem_raw) + (size_t)wid * p.pow2;
  int* idx = reinterpret_cast<int*>(smem_raw + sizeof(float) * (size_t)MERGE_WARPS * p.pow2) + (size_t)wid * p.pow2;
  long long r = (long long)blockIdx.x * MERGE_WARPS + wid;
  if (r >= R) return;
  int off = 0;
  for (int k = 0; k < p.n_lists; ++k) {
    const float* zk = p.z[k] + r * p.S[k];
    for (int i = lane; i < p.S[k]; i += 32) { keys[off + i] = zk[i]; idx[off + i] = off + i; }
    off += p.S[k];
  }
  for (int i = p.total + lane; i < p.pow2; i += 32) { keys[i] = INFINITY; idx[i] = i; }
  __syncwarp();
  nm_warp_bitonic_sort(keys, idx, p.pow2, lane);
  for (int i = lane; i < p.total; i += 32) {
    z_out[r * p.total + i] = keys[i];
    if (raw_out) {
      int src = idx[i], k = 0;
      while (src >= p.S[k]) { src -= p.S[k]; ++k; }
      raw_out[r * p.total + i] = p.raw[k][r * p.S[k] + src];
    }
  }
}

extern "C" int nm_merge_samples(nm_ctx* ctx, int32_t n_lists, const float* const* z_lists,
                                const float* const* raw_lists, const int32_t* S_list, int64_t R, float* z_out,
                                float* raw_out, void* stream) {
  NM_ENTER(ctx);
  if (R == 0) return NM_OK;
  if (n_lists < 1 || n_lists > 1 + NM_MAX_ACTORS || !z_lists || !S_list || !z_out || R < 0)
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_merge_samples: bad argument");
  MergeParams p;
  p.n_lists = n_lists;
  p.total = 0;
  for (int k = 0; k < n_lists; ++k) {
    p.z[k] = z_lists[k];
    p.raw[k] = raw_lists ? (const float4*)raw_lists[k] : nullptr;
    p.S[k] = S_list[k];
    p.total += S_list[k];
    if (!p.z[k] || (raw_out && !p.raw[k]) || p.S[k] <= 0)
      NM_FAIL(ctx, NM_ERR_INVALID, "nm_merge_samples: null list");
  }
  p.pow2 = 32;
  while (p.pow2 < p.total) p.pow2 <<= 1;
  if (p.pow2 > 4096) NM_FAIL(ctx, NM_ERR_UNSUPPORTED, "nm_merge_samples: more than 4096 samples per ray");
  size_t smem = (size_t)MERGE_WARPS * p.pow2 * 8;
  if (smem > 48 * 1024)
    NM_CHECK_CUDA(ctx, cudaFuncSetAttribute(k_merge, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  unsigned blocks = (unsigned)((R + MERGE_WARPS - 1) / MERGE_WARPS);
  k_merge<<<blocks, 32 * MERGE_WARPS, smem, (cudaStream_t)stream>>>(p, R, z_out, raw_out ? (float4*)raw_out : nullptr);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

// ---------------------------------------------------------------------------------------------
// Backward of raw2outputs (utils/render_utils.py:69-105) for training (SURVEY.md §8f-1): given the
// gradients of rgb_map [R,3], depth_map [R], acc_map [R] and weights [R,S] (any may be NULL) returns
// d raw [R,S,4].  With w_s = alpha_s T_s, T_s = prod_{j<s} (1 - alpha_j + 1e-10):
//   G_s      = dL/dw_s = sum_c g_rgb_c (c_{s,c} - [white]) + g_depth z_s + g_acc + g_w_s
//   dL/dalpha_s = G_s T_s - (sum_{k>s} G_k w_k) / (1 - alpha_s + 1e-10)
//   dL/dsigma_s = dL/dalpha_s * delta_s * exp(-relu(sigma_s) delta_s) * [sigma_s > 0] * sigma_scale
//   dL/draw_rgb_{s,c} = g_rgb_c w_s c_{s,c} (1 - c_{s,c})
// (disp_map is not differentiated: the trainers never use its gradient.)  One warp per ray: a forward
// shuffle scan rebuilds T, a reverse shuffle scan the suffix sums.
__global__ void __launch_bounds__(256) k_raw2outputs_bwd(
    const float4* __restrict__ raw, const float* __restrict__ z, const float* __restrict__ rays_d, long long R, int S,
    const float* __restrict__ noise, float sigma_scale, int white_bkg, const float* __restrict__ g_rgb,
    const float* __restrict__ g_depth, const float* __restrict__ g_acc, const float* __restrict__ g_w,
    float4* __restrict__ d_raw, float* __restrict__ scratch /* [R,S] G*w */) {
  const int lane = threadIdx.x & 31;
  long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= R) return;
  const float dx = rays_d[3 * r], dy = rays_d[3 * r + 1], dz = rays_d[3 * r + 2];
  const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);
  const float* zr = z + r * S;
  const float4* rr = raw + r * S;
  const float gr = g_rgb ? g_rgb[3 * r] : 0.f, gg = g_rgb ? g_rgb[3 * r + 1] : 0.f, gb = g_rgb ? g_rgb[3 * r + 2] : 0.f;
  const float gd = g_depth ? g_depth[r] : 0.f, ga = g_acc ? g_acc[r] : 0.f;
  const float wsub = white_bkg ? (gr + gg + gb) : 0.f;
  // pass 1 (forward): T_s, w_s; store G_s*w_s in scratch, partial results in d_raw
  float carry = 1.f;
  for (int base = 0; base < S; base += 32) {
    int s = base + lane;
    bool live = s < S;
    float alpha = 0.f, zc = 0.f, dist = 0.f, sg = 0.f;
    float4 v = make_float4(0, 0, 0, 0);
    if (live) {
      v = rr[s];
      zc = zr[s];
      dist = ((s + 1 < S) ? (zr[s + 1] - zc) : 1e10f) * dnorm;
      sg = v.w * sigma_scale;
      if (noise) sg = sg + noise[r * S + s];
      alpha = 1.f - expf(-fmaxf(sg, 0.f) * dist);
    }
    float f = live ? (1.f - alpha + 1e-10f) : 1.f;
    float inc = f;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      float t = __shfl_up_sync(FULL, inc, o);
      if (lane >= o) inc = inc * t;
    }
    float exc = __shfl_up_sync(FULL, inc, 1);
    if (lane == 0) exc = 1.f;
    float T = carry * exc;
    float w = alpha * T;
    carry = carry * __shfl_sync(FULL, inc, 31);
    if (live) {
      float cr = 1.f / (1.f + expf(-v.x)), cg = 1.f / (1.f + expf(-v.y)), cb = 1.f / (1.f + expf(-v.z));
      float G = gr * cr + gg * cg + gb * cb - wsub + gd * zc + ga + (g_w ? g_w[r * S + s] : 0.f);
      scratch[r * S + s] = G * w;
      // x,y,z final; w holds G*T for now (completed in pass 2)
      d_raw[r * S + s] = make_float4(gr * w * cr * (1.f - cr), gg * w * cg * (1.f - cg), gb * w * cb * (1.f - cb), G * T);
    }
  }
  __syncwarp();
  // pass 2 (reverse): suffix sums Q_s = sum_{k>s} G_k w_k
  float tail = 0.f;
  for (int base = ((S - 1) / 32) * 32; base >= 0; base -= 32) {
    int s = base + lane;
    bool live = s < S;
    float gw = live ? scratch[r * S + s] : 0.f;
    float inc = gw;                                   // inclusive suffix scan within the chunk
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      float t = __shfl_down_sync(FULL, inc, o);
      if (lane + o < 32) inc += t;
    }
    // exclusive (elements after s) as the next lane's inclusive sum, never inc - gw: behind an opaque sample Q is tiny next
    // to its own G*w, and the subtraction would leave only the rounding error of inc
    float exc = __shfl_down_sync(FULL, inc, 1);
    if (lane == 31) exc = 0.f;
    float Q = tail + exc;
    tail += __shfl_sync(FULL, inc, 0);
    if (live) {
      float4 v = rr[s];
      float zc = zr[s];
      float dist = ((s + 1 < S) ? (zr[s + 1] - zc) : 1e10f) * dnorm;
      float sg = v.w * sigma_scale;
      if (noise) sg = sg + noise[r * S + s];
      float e = expf(-fmaxf(sg, 0.f) * dist);
      float alpha = 1.f - e;
      float4 o = d_raw[r * S + s];
      float dalpha = o.w - Q / (1.f - alpha + 1e-10f);
      o.w = (sg > 0.f) ? dalpha * dist * e * sigma_scale : 0.f;
      d_raw[r * S + s] = o;
    }
  }
}

extern "C" int nm_raw2outputs_backward(nm_ctx* ctx, const float* raw, const float* z, const float* rays_d, int64_t R,
                                       int32_t S, const float* noise, float sigma_scale, int32_t white_bkg,
                                       const float* grad_rgb, const float* grad_depth, const float* grad_acc,
                                       const float* grad_weights, float* grad_raw, void* stream) {
  NM_ENTER(ctx);
  if (R == 0) return NM_OK;
  if (!raw || !z || !rays_d || !grad_raw || R < 0 || S <= 0) NM_FAIL(ctx, NM_ERR_INVALID, "nm_raw2outputs_backward: bad argument");
  char* ws;
  int rc = nm_impl_workspace(ctx, (size_t)R * S * sizeof(float), &ws);
  if (rc) return rc;
  unsigned blocks = (unsigned)((R * 32 + 255) / 256);
  k_raw2outputs_bwd<<<blocks, 256, 0, (cudaStream_t)stream>>>((const float4*)raw, z, rays_d, R, S, noise, sigma_scale, white_bkg,
                                                                grad_rgb, grad_depth, grad_acc, grad_weights,
                                                                (float4*)grad_raw, reinterpret_cast<float*>(ws));
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

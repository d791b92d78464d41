// Ray generation, SMPL-guided near/far, and per-ray sample placement.
// Compiled with -fmad=false: these kernels mirror chains of separately-rounded torch/numpy
// elementwise ops, so nothing may be contracted into FMAs.
//
//   nm_raygen           <- utils/ray_utils.py:23-38 + geometry/pcd_projector.py:85-120
//   nm_near_far         <- utils/ray_utils.py:197-233
//   nm_ray_to_samples   <- utils/ray_utils.py:96-135
#include "nm_internal.cuh"

// ---------------------------------------------------------------------------------------------
struct RaygenParams {
  double Kinv[9];
  double c2w[16];
  int W;
  int mode;
  long long pix0, n;
};

__global__ void __launch_bounds__(256) k_raygen(RaygenParams p, const int32_t* __restrict__ xy, const int32_t* __restrict__ pixels,
                                                 float* __restrict__ origins, float* __restrict__ dirs) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n) return;
  double x, y;
  if (xy) {
    x = (double)xy[2 * i];
    y = (double)xy[2 * i + 1];
  } else {
    long long pix = pixels ? (long long)pixels[i] : p.pix0 + i;
    y = (double)(pix / p.W);      // row-major, y outer (render_utils.py:185)
    x = (double)(pix % p.W);
  }
  // camera-space point at depth 1: Kinv * [x, y, 1]
  double cx = p.Kinv[0] * x + p.Kinv[1] * y + p.Kinv[2];
  double cy = p.Kinv[3] * x + p.Kinv[4] * y + p.Kinv[5];
  double cz = p.Kinv[6] * x + p.Kinv[7] * y + p.Kinv[8];
  // world = c2w * [c;1], then / w
  double wx = p.c2w[0] * cx + p.c2w[1] * cy + p.c2w[2] * cz + p.c2w[3];
  double wy = p.c2w[4] * cx + p.c2w[5] * cy + p.c2w[6] * cz + p.c2w[7];
  double wz = p.c2w[8] * cx + p.c2w[9] * cy + p.c2w[10] * cz + p.c2w[11];
  double ww = p.c2w[12] * cx + p.c2w[13] * cy + p.c2w[14] * cz + p.c2w[15];
  wx /= ww; wy /= ww; wz /= ww;
  float ox = (float)p.c2w[3], oy = (float)p.c2w[7], oz = (float)p.c2w[11];
  float dx, dy, dz;
  if (p.mode == 0) {
    // shot_rays: point cast to f32, subtraction and normalisation in f32 (ray_utils.py:25-28)
    float fx = (float)wx - ox, fy = (float)wy - oy, fz = (float)wz - oz;
    float nrm = sqrtf(fx * fx + fy * fy + fz * fz);
    dx = fx / nrm; dy = fy / nrm; dz = fz / nrm;
  } else {
    // shot_all_rays: float64 throughout, cast last (ray_utils.py:34-37, render_utils.py:114-115)
    double ex = wx - (double)ox, ey = wy - (double)oy, ez = wz - (double)oz;
    double nrm = sqrt(ex * ex + ey * ey + ez * ez);
    dx = (float)(ex / nrm); dy = (float)(ey / nrm); dz = (float)(ez / nrm);
  }
  origins[3 * i + 0] = ox; origins[3 * i + 1] = oy; origins[3 * i + 2] = oz;
  dirs[3 * i + 0] = dx; dirs[3 * i + 1] = dy; dirs[3 * i + 2] = dz;
}

static void invert3x3(const double* m, double* o) {
  double a = m[0], b = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], h = m[7], i = m[8];
  double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
  double id = 1.0 / det;
  o[0] = (e * i - f * h) * id; o[1] = (c * h - b * i) * id; o[2] = (b * f - c * e) * id;
  o[3] = (f * g - d * i) * id; o[4] = (a * i - c * g) * id; o[5] = (c * d - a * f) * id;
  o[6] = (d * h - e * g) * id; o[7] = (b * g - a * h) * id; o[8] = (a * e - b * d) * id;
}

extern "C" int nm_raygen(nm_ctx* ctx, const nm_camera* cam, int mode, int64_t pix0, int64_t n,
                         const int32_t* xy, float* origins, float* dirs, void* stream) {
  NM_ENTER(ctx);
  return nm_impl_raygen(ctx, cam, mode, pix0, n, xy, nullptr, origins, dirs, (cudaStream_t)stream);
}

// pixels != NULL: the n rays are the row-major pixel indices pixels[0..n) (the frame drivers' pixel lists)
int nm_impl_raygen(nm_ctx* ctx, const nm_camera* cam, int mode, int64_t pix0, int64_t n, const int32_t* xy,
                   const int32_t* pixels, float* origins, float* dirs, cudaStream_t stream) {
  if (n == 0) return NM_OK;
  if (!cam || !origins || !dirs || n < 0 || (mode != 0 && mode != 1))
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_raygen: bad argument");
  RaygenParams p;
  invert3x3(cam->K, p.Kinv);
  for (int i = 0; i < 16; ++i) p.c2w[i] = cam->c2w[i];
  p.W = cam->W; p.mode = mode; p.pix0 = pix0; p.n = n;
  if (!xy && !pixels && (pix0 < 0 || pix0 + n > (int64_t)cam->H * cam->W))
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_raygen: pixel range outside the image");
  unsigned blocks = (unsigned)((n + 255) / 256);
  k_raygen<<<blocks, 256, 0, stream>>>(p, xy, pixels, origins, dirs);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

// ---------------------------------------------------------------------------------------------
// near/far: four lanes per ray (each takes every 4th vertex, then a 2-step shuffle min/max), the vertex
// list streamed through shared memory in tiles.  6890 vertices x 16 B = 110 KB: four tiles of 2048.
#define NF_TILE 2048
#define NF_LANES 4
// bounding sphere of the vertices (bbox centre, max distance): lets whole warps of rays that pass farther than
// radius + threshold from it skip the vertex loop -- such a ray cannot touch any vertex sphere, so the result
// (near=+inf, far=-inf) is exactly what the loop would produce.
__global__ void __launch_bounds__(256) k_vert_bounds(const float* __restrict__ verts, int nv, float4* __restrict__ out) {
  __shared__ float red[6][256];
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int v = threadIdx.x; v < nv; v += 256)
    for (int c = 0; c < 3; ++c) { lo[c] = fminf(lo[c], verts[3 * v + c]); hi[c] = fmaxf(hi[c], verts[3 * v + c]); }
  for (int c = 0; c < 3; ++c) { red[c][threadIdx.x] = lo[c]; red[3 + c][threadIdx.x] = hi[c]; }
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o)
      for (int c = 0; c < 3; ++c) {
        red[c][threadIdx.x] = fminf(red[c][threadIdx.x], red[c][threadIdx.x + o]);
        red[3 + c][threadIdx.x] = fmaxf(red[3 + c][threadIdx.x], red[3 + c][threadIdx.x + o]);
      }
    __syncthreads();
  }
  const float cx = 0.5f * (red[0][0] + red[3][0]), cy = 0.5f * (red[1][0] + red[4][0]), cz = 0.5f * (red[2][0] + red[5][0]);
  __syncthreads();
  float r2 = 0.f;
  for (int v = threadIdx.x; v < nv; v += 256) {
    float ax = verts[3 * v] - cx, ay = verts[3 * v + 1] - cy, az = verts[3 * v + 2] - cz;
    r2 = fmaxf(r2, ax * ax + ay * ay + az * az);
  }
  red[0][threadIdx.x] = r2;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[0][threadIdx.x] = fmaxf(red[0][threadIdx.x], red[0][threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = make_float4(cx, cy, cz, sqrtf(red[0][0]));
}

__global__ void __launch_bounds__(256) k_near_far(const float* __restrict__ origins,
                                                   const float* __restrict__ dirs, long long R,
                                                   const float* __restrict__ verts, int nv, float thr2, float thr,
                                                   const float4* __restrict__ bounds,
                                                   float* __restrict__ near_out, float* __restrict__ far_out) {
  __shared__ float4 sv[NF_TILE];
  const int sl = threadIdx.x & (NF_LANES - 1);
  long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / NF_LANES;
  bool live = r < R;
  float ox = 0, oy = 0, oz = 0, dx = 0, dy = 0, dz = 1;
  if (live) {
    ox = origins[3 * r]; oy = origins[3 * r + 1]; oz = origins[3 * r + 2];
    dx = dirs[3 * r]; dy = dirs[3 * r + 1]; dz = dirs[3 * r + 2];
  }
  float nr = INFINITY, fr = -INFINITY;
  // conservative cull (0.1 % + 1e-6 slack): distance from the ray's LINE to the bounding-sphere centre
  bool may_hit = false;
  if (live) {
    const float4 b = *bounds;
    const float cx = b.x - ox, cy = b.y - oy, cz = b.z - oz;
    const float dn2 = dx * dx + dy * dy + dz * dz;
    const float t = (cx * dx + cy * dy + cz * dz);
    const float perp2 = (cx * cx + cy * cy + cz * cz) - t * t / dn2;
    const float lim = (b.w + thr) * 1.001f + 1e-6f;
    // the reference's discriminant equals the geometric one only for unit directions: no cull otherwise
    may_hit = !(perp2 > lim * lim) || fabsf(dn2 - 1.f) > 1e-3f;
  }
  if (!__syncthreads_or(may_hit)) {                 // the whole block's rays pass clear of the body
    if (live && sl == 0) { near_out[r] = nr; far_out[r] = fr; }
    return;
  }
  for (int base = 0; base < nv; base += NF_TILE) {
    int cnt = min(NF_TILE, nv - base);
    __syncthreads();
    for (int j = threadIdx.x; j < cnt; j += blockDim.x) {
      const float* v = verts + 3 * (size_t)(base + j);
      sv[j] = make_float4(v[0], v[1], v[2], 0.f);
    }
    __syncthreads();
    if (may_hit)
#pragma unroll 4
    for (int j = sl; j < cnt; j += NF_LANES) {
      float4 v = sv[j];
      float ax = v.x - ox, ay = v.y - oy, az = v.z - oz;          // orig_v (ray_utils.py:211)
      float z0 = ax * dx + ay * dy + az * dz;                      // einsum (:212)
      float nrm = sqrtf(ax * ax + ay * ay + az * az);              // torch.norm (:213)
      float disc = thr2 - (nrm * nrm - z0 * z0);
      if (disc >= 0.f) {                                           // sqrt of a negative -> NaN -> skipped
        float dzv = sqrtf(disc);
        nr = fminf(nr, z0 - dzv);
        fr = fmaxf(fr, z0 + dzv);
      }
    }
  }
#pragma unroll
  for (int o = 1; o < NF_LANES; o <<= 1) {
    nr = fminf(nr, __shfl_xor_sync(0xffffffffu, nr, o));
    fr = fmaxf(fr, __shfl_xor_sync(0xffffffffu, fr, o));
  }
  if (live && sl == 0) { near_out[r] = nr; far_out[r] = fr; }
}

extern "C" int nm_near_far(nm_ctx* ctx, const float* origins, const float* dirs, int64_t R,
                           const float* verts, int32_t n_verts, float geo_threshold, float* near_out,
                           float* far_out, void* stream) {
  NM_ENTER(ctx);
  if (R == 0) return NM_OK;
  if (!origins || !dirs || !verts || !near_out || !far_out || R < 0 || n_verts < 0)
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_near_far: bad argument");
  // geo_threshold**2 is a python double that torch casts to f32 for the subtraction (:213)
  float thr2 = (float)((double)geo_threshold * (double)geo_threshold);
  unsigned blocks = (unsigned)((R * NF_LANES + 255) / 256);
  float4* bounds = reinterpret_cast<float4*>(ctx->d_counter + 16);       // 16-byte aligned scratch in the ctx
  k_vert_bounds<<<1, 256, 0, (cudaStream_t)stream>>>(verts, n_verts, bounds);
  NM_CHECK_LAUNCH(ctx);
  k_near_far<<<blocks, 256, 0, (cudaStream_t)stream>>>(origins, dirs, R, verts, n_verts, thr2, geo_threshold, bounds,
                                                         near_out, far_out);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

// ---------------------------------------------------------------------------------------------
// near/far against a SET mesh (the frame drivers): the vertices are kept in Morton order in groups of 32 with one bounding
// sphere per group; a ray tests the 32 vertex spheres of a group only when its line passes within radius + threshold of
// the group's centre (conservative by 1 %: a culled vertex cannot yield a real root, so the result is exactly the
// exhaustive loop's -- min / max do not depend on the order).  SMPL: 6890 vertices = 216 groups, of which a ray meets a
// handful, instead of 6890 sphere tests per ray.
#define VG_SIZE 32
#define VG_TILE 64                   // groups per shared-memory tile (2048 vertices, 32 KB)
#include <algorithm>
#include <vector>

static inline uint32_t expand10(uint32_t v) {
  v = (v * 0x00010001u) & 0xFF0000FFu;
  v = (v * 0x00000101u) & 0x0F00F00Fu;
  v = (v * 0x00000011u) & 0xC30C30C3u;
  v = (v * 0x00000005u) & 0x49249249u;
  return v;
}

int nm_impl_build_vgroups(nm_ctx* ctx, NmMesh& m, const float* hv, const float* lo, const float* hi, cudaStream_t st) {
  const int nv = m.n_verts;
  const int ng = (nv + VG_SIZE - 1) / VG_SIZE;
  std::vector<std::pair<uint32_t, int>> key(nv);
  float inv[3];
  for (int c = 0; c < 3; ++c) inv[c] = 1023.f / fmaxf(hi[c] - lo[c], 1e-20f);
  for (int v = 0; v < nv; ++v) {
    uint32_t q[3];
    for (int c = 0; c < 3; ++c) q[c] = (uint32_t)fminf(fmaxf((hv[3 * v + c] - lo[c]) * inv[c], 0.f), 1023.f);
    key[v] = {(expand10(q[0]) << 2) | (expand10(q[1]) << 1) | expand10(q[2]), v};
  }
  std::sort(key.begin(), key.end());
  std::vector<float4> sorted((size_t)ng * VG_SIZE), sph(ng);
  for (int g = 0; g < ng; ++g) {
    float blo[3] = {INFINITY, INFINITY, INFINITY}, bhi[3] = {-INFINITY, -INFINITY, -INFINITY};
    const int first = key[g * VG_SIZE].second;
    for (int k = 0; k < VG_SIZE; ++k) {
      const int i = g * VG_SIZE + k;
      const int v = i < nv ? key[i].second : first;          // padding repeats a vertex of the group: no new roots
      sorted[i] = make_float4(hv[3 * v], hv[3 * v + 1], hv[3 * v + 2], 0.f);
      for (int c = 0; c < 3; ++c) { blo[c] = fminf(blo[c], hv[3 * v + c]); bhi[c] = fmaxf(bhi[c], hv[3 * v + c]); }
    }
    const float cx = 0.5f * (blo[0] + bhi[0]), cy = 0.5f * (blo[1] + bhi[1]), cz = 0.5f * (blo[2] + bhi[2]);
    float r2 = 0.f;
    for (int k = 0; k < VG_SIZE; ++k) {
      const float4 p = sorted[g * VG_SIZE + k];
      r2 = fmaxf(r2, (p.x - cx) * (p.x - cx) + (p.y - cy) * (p.y - cy) + (p.z - cz) * (p.z - cz));
    }
    sph[g] = make_float4(cx, cy, cz, sqrtf(r2));
  }
  if (m.cap_vsorted < sorted.size()) {
    if (m.vsorted) { NM_CHECK_CUDA(ctx, cudaStreamSynchronize(st)); NM_CHECK_CUDA(ctx, cudaFree(m.vsorted)); m.vsorted = nullptr; }
    NM_CHECK_CUDA(ctx, cudaMalloc(&m.vsorted, sorted.size() * sizeof(float4)));
    m.cap_vsorted = sorted.size();
  }
  if (m.cap_vgroup < (size_t)ng) {
    if (m.vgroup) { NM_CHECK_CUDA(ctx, cudaStreamSynchronize(st)); NM_CHECK_CUDA(ctx, cudaFree(m.vgroup)); m.vgroup = nullptr; }
    NM_CHECK_CUDA(ctx, cudaMalloc(&m.vgroup, (size_t)ng * sizeof(float4)));
    m.cap_vgroup = ng;
  }
  // pageable sources: the copies are complete (staged) when the calls return, so the vectors may go out of scope
  NM_CHECK_CUDA(ctx, cudaMemcpyAsync(m.vsorted, sorted.data(), sorted.size() * sizeof(float4), cudaMemcpyHostToDevice, st));
  NM_CHECK_CUDA(ctx, cudaMemcpyAsync(m.vgroup, sph.data(), (size_t)ng * sizeof(float4), cudaMemcpyHostToDevice, st));
  m.n_vgroups = ng;
  {
    const float cx = 0.5f * (lo[0] + hi[0]), cy = 0.5f * (lo[1] + hi[1]), cz = 0.5f * (lo[2] + hi[2]);
    float r2 = 0.f;
    for (int v = 0; v < nv; ++v)
      r2 = fmaxf(r2, (hv[3 * v] - cx) * (hv[3 * v] - cx) + (hv[3 * v + 1] - cy) * (hv[3 * v + 1] - cy) + (hv[3 * v + 2] - cz) * (hv[3 * v + 2] - cz));
    m.vbound = make_float4(cx, cy, cz, sqrtf(r2));
  }
  return NM_OK;
}

__global__ void __launch_bounds__(256) k_near_far_groups(const float* __restrict__ origins, const float* __restrict__ dirs,
                                                          long long R, const float4* __restrict__ vsorted,
                                                          const float4* __restrict__ vgroup, int ng, float4 bound, float thr2,
                                                          float thr, float* __restrict__ near_out, float* __restrict__ far_out) {
  __shared__ float4 sv[VG_TILE * VG_SIZE];
  __shared__ float4 sg[VG_TILE];
  const int sl = threadIdx.x & (NF_LANES - 1);
  long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / NF_LANES;
  const bool live = r < R;
  float ox = 0, oy = 0, oz = 0, dx = 0, dy = 0, dz = 1;
  if (live) {
    ox = origins[3 * r]; oy = origins[3 * r + 1]; oz = origins[3 * r + 2];
    dx = dirs[3 * r]; dy = dirs[3 * r + 1]; dz = dirs[3 * r + 2];
  }
  const float dn2 = dx * dx + dy * dy + dz * dz;
  // the reference's discriminant equals the geometric one only for unit directions: no cull otherwise
  const bool unit = fabsf(dn2 - 1.f) <= 1e-3f;
  float nr = INFINITY, fr = -INFINITY;
  {
    // whole-body cull: a block whose rays all pass clear of the mesh's bounding sphere (+ threshold) is done
    const float cx = bound.x - ox, cy = bound.y - oy, cz = bound.z - oz;
    const float t = cx * dx + cy * dy + cz * dz;
    const float perp2 = (cx * cx + cy * cy + cz * cz) - t * t / dn2;
    const float lim = (bound.w + thr) * 1.01f + 1e-5f;
    const bool may_hit = live && (!unit || !(perp2 > lim * lim));
    if (!__syncthreads_or(may_hit)) {
      if (live && sl == 0) { near_out[r] = nr; far_out[r] = fr; }
      return;
    }
  }
  for (int g0 = 0; g0 < ng; g0 += VG_TILE) {
    const int cnt = min(VG_TILE, ng - g0);
    __syncthreads();
    for (int j = threadIdx.x; j < cnt * VG_SIZE; j += blockDim.x) sv[j] = vsorted[(size_t)g0 * VG_SIZE + j];
    if (threadIdx.x < cnt) sg[threadIdx.x] = vgroup[g0 + threadIdx.x];
    __syncthreads();
    if (live)
      for (int g = sl; g < cnt; g += NF_LANES) {
        const float4 b = sg[g];
        const float cx = b.x - ox, cy = b.y - oy, cz = b.z - oz;
        const float t = cx * dx + cy * dy + cz * dz;
        const float perp2 = (cx * cx + cy * cy + cz * cz) - t * t / dn2;
        const float lim = (b.w + thr) * 1.01f + 1e-5f;
        if (unit && perp2 > lim * lim) continue;
#pragma unroll 8
        for (int k = 0; k < VG_SIZE; ++k) {
          const float4 v = sv[g * VG_SIZE + k];
          float ax = v.x - ox, ay = v.y - oy, az = v.z - oz;          // orig_v (ray_utils.py:211)
          float z0 = ax * dx + ay * dy + az * dz;                      // einsum (:212)
          float nrm = sqrtf(ax * ax + ay * ay + az * az);              // torch.norm (:213)
          float disc = thr2 - (nrm * nrm - z0 * z0);
          if (disc >= 0.f) {                                           // sqrt of a negative -> NaN -> skipped
            float dzv = sqrtf(disc);
            nr = fminf(nr, z0 - dzv);
            fr = fmaxf(fr, z0 + dzv);
          }
        }
      }
  }
#pragma unroll
  for (int o = 1; o < NF_LANES; o <<= 1) {
    nr = fminf(nr, __shfl_xor_sync(0xffffffffu, nr, o));
    fr = fmaxf(fr, __shfl_xor_sync(0xffffffffu, fr, o));
  }
  if (live && sl == 0) { near_out[r] = nr; far_out[r] = fr; }
}

int nm_impl_near_far_mesh(nm_ctx* ctx, const NmMesh& m, const float* origins, const float* dirs, int64_t R, float geo_threshold,
                          float* near_out, float* far_out, cudaStream_t st) {
  if (R == 0) return NM_OK;
  if (!m.vsorted || m.n_vgroups <= 0) return nm_near_far(ctx, origins, dirs, R, m.verts, m.n_verts, geo_threshold, near_out, far_out, st);
  float thr2 = (float)((double)geo_threshold * (double)geo_threshold);
  unsigned blocks = (unsigned)((R * NF_LANES + 255) / 256);
  k_near_far_groups<<<blocks, 256, 0, st>>>(origins, dirs, R, m.vsorted, m.vgroup, m.n_vgroups, m.vbound, thr2, geo_threshold, near_out, far_out);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

extern "C" int nm_near_far_mesh(nm_ctx* ctx, int actor, const float* origins, const float* dirs, int64_t R,
                                float geo_threshold, float* near_out, float* far_out, void* stream) {
  NM_ENTER(ctx);
  if (R == 0) return NM_OK;
  if (!origins || !dirs || !near_out || !far_out || R < 0) NM_FAIL(ctx, NM_ERR_INVALID, "nm_near_far_mesh: bad argument");
  if (actor < 0 || actor >= NM_MAX_ACTORS || !ctx->meshes[actor].set) NM_FAIL(ctx, NM_ERR_STATE, "nm_near_far_mesh: mesh not set");
  return nm_impl_near_far_mesh(ctx, ctx->meshes[actor], origins, dirs, R, geo_threshold, near_out, far_out, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------
// ray_to_samples: thread per sample (coalesced along the sample index).
__global__ void __launch_bounds__(256) k_ray_to_samples(
    const float* __restrict__ origins, const float* __restrict__ dirs, const float* __restrict__ near_v,
    const float* __restrict__ far_v, float near_s, float far_s, long long R, int S, int lindisp,
    const float* __restrict__ t_rand, float* __restrict__ pts, float* __restrict__ dirs_out,
    float* __restrict__ z_out) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= R * (long long)S) return;
  long long r = idx / S;
  int s = (int)(idx - r * S);
  float nr = near_v ? near_v[r] : near_s;
  float fr = far_v ? far_v[r] : far_s;
  auto zval = [&](int i) -> float {
    float t = nm_linspace01(i, S);
    if (!lindisp) return nr * (1.f - t) + fr * t;                       // (:113)
    return 1.f / (1.f / nr * (1.f - t) + 1.f / fr * t);                 // (:115)
  };
  float z = zval(s);
  if (t_rand) {                                                          // stratified (:117-129)
    float zl = s > 0 ? zval(s - 1) : z;
    float zu = s < S - 1 ? zval(s + 1) : z;
    float lower = s > 0 ? 0.5f * (z + zl) : z;
    float upper = s < S - 1 ? 0.5f * (zu + z) : z;
    float u = fminf(fmaxf(t_rand[idx], 0.01f), 1.f - 0.01f);            // PERTURB_EPSILON
    z = lower + (upper - lower) * u;
  }
  if (z_out) z_out[idx] = z;
  if (pts || dirs_out) {
    float dx = dirs[3 * r], dy = dirs[3 * r + 1], dz = dirs[3 * r + 2];
    if (pts) {
      pts[3 * idx + 0] = origins[3 * r + 0] + dx * z;                   // (:131)
      pts[3 * idx + 1] = origins[3 * r + 1] + dy * z;
      pts[3 * idx + 2] = origins[3 * r + 2] + dz * z;
    }
    if (dirs_out) { dirs_out[3 * idx] = dx; dirs_out[3 * idx + 1] = dy; dirs_out[3 * idx + 2] = dz; }
  }
}

extern "C" int nm_ray_to_samples(nm_ctx* ctx, const float* origins, const float* dirs, const float* near_v,
                                 const float* far_v, float near_s, float far_s, int64_t R, int32_t S,
                                 int32_t lindisp, const float* t_rand, float* pts, float* dirs_out, float* z,
                                 void* stream) {
  NM_ENTER(ctx);
  if (R == 0) return NM_OK;
  if (R < 0 || S <= 0 || ((pts || dirs_out) && (!origins || !dirs)))
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_ray_to_samples: bad argument");
  long long total = (long long)R * S;
  unsigned blocks = (unsigned)((total + 255) / 256);
  k_ray_to_samples<<<blocks, 256, 0, (cudaStream_t)stream>>>(origins, dirs, near_v, far_v, near_s, far_s, R, S,
                                                               lindisp, t_rand, pts, dirs_out, z);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

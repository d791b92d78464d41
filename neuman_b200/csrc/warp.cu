// Observation -> canonical warp: closest point on the posed SMPL mesh, barycentric blend of the
// three per-vertex 4x4 transforms, inverse, apply; canonical view directions by finite differences.
//
//   nm_mesh_set            per-frame inputs of warp_samples_to_canonical (verts, faces, T) + LBVH build
//   nm_signed_distance     <- igl.signed_distance as called by utils/ray_utils.py:70 (warp_samples_to_canonical_diff)
//                             and trainers/human_nerf_trainer.py:310,326 (inside/outside of the SMPL surface)
//   nm_warp_to_canonical   <- utils/ray_utils.py:48-66 (igl.point_mesh_squared_distance :53,
//                             igl.barycentric_coordinates_tri :55, blend :56, inverse :57, apply :58,
//                             finite-difference directions :62-64)
//
// The reference does this stage on the CPU in float64 (libigl AABB tree) with a device->host->device
// round trip per batch (utils/render_utils.py:218-227).  Here a linear BVH (Morton-sorted triangles,
// Karras 2012 hierarchy, bottom-up AABB refit) is rebuilt per frame (13 776 triangles: microseconds)
// and every sample runs an exact nearest-triangle traversal (stack, nearer child first, prune by the
// best squared distance).  The arg-min runs in fp32 (exact ties -> lowest face index); the winning
// triangle is then re-evaluated in float64 (closest point, barycentrics, blend, inverse, apply),
// which is what the reference's float64 chain produces before `.float()` (utils/render_utils.py:226).
#include <cub/device/device_radix_sort.cuh>
#include <float.h>
#include <math.h>

#include "nm_internal.cuh"
#include "train_common_kernels.cuh"

// ---------------------------------------------------------------------------------------------
// LBVH build
// ---------------------------------------------------------------------------------------------
struct BvhView {
  int n;                         // triangles (leaves); node ids: internal [0, n-1), leaf k -> n-1+k
  const float4* lo;              // [2n-1] AABB min
  const float4* hi;              // [2n-1] AABB max
  const int2* children;          // [n-1]
  const int32_t* leaf_face;      // [n]
  const float* tri9;             // [F][9] packed triangle vertices
};

__device__ __forceinline__ uint32_t expand_bits10(uint32_t v) {
  v = (v * 0x00010001u) & 0xFF0000FFu;
  v = (v * 0x00000101u) & 0x0F00F00Fu;
  v = (v * 0x00000011u) & 0xC30C30C3u;
  v = (v * 0x00000005u) & 0x49249249u;
  return v;
}

// packed triangles + Morton keys of the centroids (key = morton30 << 32 | face: unique)
// order-preserving float <-> int (for atomicMin / atomicMax on coordinates)
__device__ __forceinline__ int f2ord(float f) { const int k = __float_as_int(f); return k >= 0 ? k : k ^ 0x7fffffff; }
__device__ __forceinline__ float ord2f(int k) { return __int_as_float(k >= 0 ? k : k ^ 0x7fffffff); }

// bounding box of the vertices on the device (box[0..2] = min, box[3..5] = max as ordered ints; the host presets them with
// byte patterns 0x7f / 0x80): used when the mesh comes from device memory for distance queries only, so that setting it
// needs no device->host copy and no stream synchronisation (once per training step)
__global__ void k_bbox(const float* __restrict__ verts, int nv, int* __restrict__ box) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  const int vv = v < nv ? v : nv - 1;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int k = f2ord(verts[3 * vv + c]);
    const int lo = __reduce_min_sync(0xffffffffu, k), hi = __reduce_max_sync(0xffffffffu, k);
    if ((threadIdx.x & 31) == 0) { atomicMin(box + c, lo); atomicMax(box + 3 + c, hi); }
  }
}

__global__ void k_bvh_keys(const float* __restrict__ verts, const int32_t* __restrict__ faces, int nf, float3 bmin,
                           float3 binv, const int* __restrict__ box, float* __restrict__ tri9,
                           unsigned long long* __restrict__ keys) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  if (box) {                                   // bounds from k_bbox instead of the host's
    bmin = make_float3(ord2f(box[0]), ord2f(box[1]), ord2f(box[2]));
    binv = make_float3(1.f / fmaxf(ord2f(box[3]) - bmin.x, 1e-20f), 1.f / fmaxf(ord2f(box[4]) - bmin.y, 1e-20f),
                       1.f / fmaxf(ord2f(box[5]) - bmin.z, 1e-20f));
  }
  float v[9];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    int vi = faces[3 * f + k];
    v[3 * k] = verts[3 * vi]; v[3 * k + 1] = verts[3 * vi + 1]; v[3 * k + 2] = verts[3 * vi + 2];
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) tri9[9 * f + k] = v[k];
  float cx = ((v[0] + v[3] + v[6]) * (1.f / 3.f) - bmin.x) * binv.x;
  float cy = ((v[1] + v[4] + v[7]) * (1.f / 3.f) - bmin.y) * binv.y;
  float cz = ((v[2] + v[5] + v[8]) * (1.f / 3.f) - bmin.z) * binv.z;
  uint32_t x = (uint32_t)fminf(fmaxf(cx * 1024.f, 0.f), 1023.f), y = (uint32_t)fminf(fmaxf(cy * 1024.f, 0.f), 1023.f),
           z = (uint32_t)fminf(fmaxf(cz * 1024.f, 0.f), 1023.f);
  uint32_t m = (expand_bits10(x) << 2) | (expand_bits10(y) << 1) | expand_bits10(z);
  keys[f] = ((unsigned long long)m << 32) | (unsigned long long)(uint32_t)f;
}

__device__ __forceinline__ int bvh_delta(const unsigned long long* __restrict__ k, int n, int i, int j) {
  if (j < 0 || j >= n) return -1;
  return __clzll(k[i] ^ k[j]);
}

// Karras 2012: one thread per internal node
__global__ void k_bvh_hierarchy(const unsigned long long* __restrict__ keys, int n, int2* __restrict__ children,
                                int32_t* __restrict__ parent, int32_t* __restrict__ leaf_face) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) leaf_face[i] = (int32_t)(keys[i] & 0xffffffffull);
  if (i >= n - 1) return;
  int d = (bvh_delta(keys, n, i, i + 1) - bvh_delta(keys, n, i, i - 1)) >= 0 ? 1 : -1;
  int dmin = bvh_delta(keys, n, i, i - d);
  int lmax = 2;
  while (bvh_delta(keys, n, i, i + lmax * d) > dmin) lmax <<= 1;
  int l = 0;
  for (int t = lmax >> 1; t >= 1; t >>= 1)
    if (bvh_delta(keys, n, i, i + (l + t) * d) > dmin) l += t;
  int j = i + l * d;
  int dnode = bvh_delta(keys, n, i, j);
  int s = 0, t = l;
  do {
    t = (t + 1) >> 1;
    if (bvh_delta(keys, n, i, i + (s + t) * d) > dnode) s += t;
  } while (t > 1);
  int gamma = i + s * d + min(d, 0);
  int left = (min(i, j) == gamma) ? (n - 1 + gamma) : gamma;
  int right = (max(i, j) == gamma + 1) ? (n - 1 + gamma + 1) : (gamma + 1);
  children[i] = make_int2(left, right);
  parent[left] = i;
  parent[right] = i;
  if (i == 0) parent[0] = -1;
}

// bottom-up AABB refit: the second thread to reach a node merges its children
__global__ void k_bvh_refit(const float* __restrict__ tri9, const int32_t* __restrict__ leaf_face, int n,
                            const int2* __restrict__ children, const int32_t* __restrict__ parent,
                            int32_t* __restrict__ visit, float4* lo, float4* hi) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const float* t = tri9 + 9 * (size_t)leaf_face[k];
  float4 bl = make_float4(fminf(t[0], fminf(t[3], t[6])), fminf(t[1], fminf(t[4], t[7])), fminf(t[2], fminf(t[5], t[8])), 0.f);
  float4 bh = make_float4(fmaxf(t[0], fmaxf(t[3], t[6])), fmaxf(t[1], fmaxf(t[4], t[7])), fmaxf(t[2], fmaxf(t[5], t[8])), 0.f);
  int node = n - 1 + k;
  lo[node] = bl; hi[node] = bh;
  __threadfence();
  int cur = (n > 1) ? parent[node] : -1;
  while (cur >= 0) {
    if (atomicAdd(&visit[cur], 1) == 0) return;       // first arrival: the sibling subtree is not done yet
    __threadfence();
    int2 ch = children[cur];
    float4 l0 = __ldcg(lo + ch.x), l1 = __ldcg(lo + ch.y), h0 = __ldcg(hi + ch.x), h1 = __ldcg(hi + ch.y);
    lo[cur] = make_float4(fminf(l0.x, l1.x), fminf(l0.y, l1.y), fminf(l0.z, l1.z), 0.f);
    hi[cur] = make_float4(fmaxf(h0.x, h1.x), fmaxf(h0.y, h1.y), fmaxf(h0.z, h1.z), 0.f);
    __threadfence();
    cur = parent[cur];
  }
}

// ---------------------------------------------------------------------------------------------
template <typename T>
struct V3 { T x, y, z; };
template <typename T> __device__ __forceinline__ V3<T> sub(V3<T> a, V3<T> b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <typename T> __device__ __forceinline__ T dot(V3<T> a, V3<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename T> __device__ __forceinline__ V3<T> madd(V3<T> a, V3<T> d, T t) { return {a.x + d.x * t, a.y + d.y * t, a.z + d.z * t}; }
template <typename T> __device__ __forceinline__ V3<T> cross(V3<T> a, V3<T> b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}

// Exact closest point on triangle (a,b,c) to p: vertex / edge / face Voronoi regions (Ericson 5.1.5)
template <typename T>
__device__ __forceinline__ V3<T> closest_on_tri(V3<T> p, V3<T> a, V3<T> b, V3<T> c) {
  V3<T> ab = sub(b, a), ac = sub(c, a), ap = sub(p, a);
  T d1 = dot(ab, ap), d2 = dot(ac, ap);
  if (d1 <= 0 && d2 <= 0) return a;
  V3<T> bp = sub(p, b);
  T d3 = dot(ab, bp), d4 = dot(ac, bp);
  if (d3 >= 0 && d4 <= d3) return b;
  T vc = d1 * d4 - d3 * d2;
  if (vc <= 0 && d1 >= 0 && d3 <= 0) return madd(a, ab, d1 / (d1 - d3));
  V3<T> cp = sub(p, c);
  T d5 = dot(ab, cp), d6 = dot(ac, cp);
  if (d6 >= 0 && d5 <= d6) return c;
  T vb = d5 * d2 - d1 * d6;
  if (vb <= 0 && d2 >= 0 && d6 <= 0) return madd(a, ac, d2 / (d2 - d6));
  T va = d3 * d6 - d5 * d4;
  if (va <= 0 && (d4 - d3) >= 0 && (d5 - d6) >= 0) return madd(b, sub(c, b), (d4 - d3) / ((d4 - d3) + (d5 - d6)));
  T den = T(1) / (va + vb + vc);
  return madd(madd(a, ab, vb * den), ac, vc * den);
}

__device__ __forceinline__ float box_d2(const BvhView& B, int node, V3<float> p) {
  const float4 l = __ldg(B.lo + node), h = __ldg(B.hi + node);
  float dx = fmaxf(fmaxf(l.x - p.x, p.x - h.x), 0.f), dy = fmaxf(fmaxf(l.y - p.y, p.y - h.y), 0.f),
        dz = fmaxf(fmaxf(l.z - p.z, p.z - h.z), 0.f);
  return dx * dx + dy * dy + dz * dz;
}

// Exact nearest-triangle search, one BVH traversal per WARP (packet traversal): the 32 lanes hold 32
// consecutive samples (neighbours along a ray), a node is visited when ANY lane still needs it (its box is
// not farther than that lane's best, 1e-5 slack keeps exact ties alive so the lowest face index wins them),
// the nearer child is chosen by majority vote.  Control flow is warp-uniform; only the distances are per lane.
// All 32 lanes must call it (dead lanes with a copy of a live point); `stack`: 64 ints of shared memory per warp.
__device__ __forceinline__ int bvh_nearest_face(const BvhView& B, V3<float> p, int* stack) {
  float best = FLT_MAX;
  int best_f = 0x7fffffff;
  int sp = 0;
  int node = (B.n > 1) ? 0 : B.n - 1;
  while (true) {
    if (node >= B.n - 1) {
      const int f = __ldg(B.leaf_face + (node - (B.n - 1)));
      const float* t = B.tri9 + 9 * (size_t)f;
      V3<float> a{__ldg(t), __ldg(t + 1), __ldg(t + 2)}, b{__ldg(t + 3), __ldg(t + 4), __ldg(t + 5)},
          c{__ldg(t + 6), __ldg(t + 7), __ldg(t + 8)};
      V3<float> e = sub(closest_on_tri<float>(p, a, b, c), p);
      const float d2 = dot(e, e);
      if (d2 < best || (d2 == best && f < best_f)) { best = d2; best_f = f; }
      node = -1;
    } else {
      const int2 ch = __ldg(B.children + node);
      const float dl = box_d2(B, ch.x, p), dr = box_d2(B, ch.y, p);
      const float lim = best * 1.00001f;
      const bool needL = __any_sync(0xffffffffu, dl <= lim), needR = __any_sync(0xffffffffu, dr <= lim);
      const bool left_first = __popc(__ballot_sync(0xffffffffu, dl <= dr)) >= 16;
      if (needL && needR) {
        if (sp < 64) { if ((threadIdx.x & 31) == 0) stack[sp] = left_first ? ch.y : ch.x; ++sp; }
        node = left_first ? ch.x : ch.y;
      } else {
        node = needL ? ch.x : (needR ? ch.y : -1);
      }
    }
    if (node < 0) {
      // pop until a node some lane still needs
      bool found = false;
      while (sp > 0) {
        --sp;
        __syncwarp();
        const int cand = stack[sp];
        if (__any_sync(0xffffffffu, box_d2(B, cand, p) <= best * 1.00001f)) { node = cand; found = true; break; }
      }
      if (!found) break;
    }
  }
  return best_f;
}

// The search and the float64 evaluation are two kernels: the traversal is a latency-bound pointer chase that wants many
// resident warps (fp32, ~40 registers), the evaluation needs ~80 registers of float64 state.
// Packet shape: the 32 lanes of a warp take (1 << lg_rays) neighbouring rays x (32 >> lg_rays) consecutive samples, so the
// packet is a compact bundle instead of a long stretch of one ray and the union of the nodes its lanes need is small.
// The result per point does not depend on the packet it travels in (every node a lane needs is visited, ties go to the
// lowest face index).  lg_rays = 0 is the plain linear order (any S).
__global__ void __launch_bounds__(128) k_warp_nearest(BvhView B, const float* __restrict__ pts, long long R, int S, int lg_rays,
                                                       int32_t* __restrict__ face_out) {
  const long long w = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  long long i;
  bool live;
  if (lg_rays == 0) {
    i = w * 32 + lane;
    live = i < R * S;
    if (!live) i = R * S - 1;
  } else {
    const int per = 32 >> lg_rays;                       // samples of one ray in the packet
    const int groups = S / per;                          // packets along a ray (S % per == 0, checked by the host)
    const long long rg = w / groups;
    const int sg = (int)(w - rg * groups);
    long long ray = (rg << lg_rays) + (lane / per);
    live = ray < R;
    if (!live) ray = R - 1;
    i = ray * S + sg * per + (lane % per);
  }
  V3<float> p{pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
  __shared__ int s_stack[4][64];
  const int best_f = bvh_nearest_face(B, p, s_stack[threadIdx.x >> 5]);
  if (live) face_out[i] = best_f;
}

__global__ void __launch_bounds__(128) k_warp_points(const float* __restrict__ verts, const int32_t* __restrict__ faces,
                                                      const double* __restrict__ T, const float* __restrict__ pts, long long n,
                                                      const int32_t* __restrict__ face_in, double* __restrict__ can64,
                                                      float* __restrict__ closest_out) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  V3<float> p{pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
  const int best_f = face_in[i];
  // ---- float64 re-evaluation on the winning triangle (utils/ray_utils.py:53-58) ----
  int i0 = faces[3 * best_f], i1 = faces[3 * best_f + 1], i2 = faces[3 * best_f + 2];
  V3<double> P{(double)p.x, (double)p.y, (double)p.z};
  V3<double> A{(double)verts[3 * i0], (double)verts[3 * i0 + 1], (double)verts[3 * i0 + 2]};
  V3<double> Bv{(double)verts[3 * i1], (double)verts[3 * i1 + 1], (double)verts[3 * i1 + 2]};
  V3<double> C{(double)verts[3 * i2], (double)verts[3 * i2 + 1], (double)verts[3 * i2 + 2]};
  V3<double> Q = closest_on_tri<double>(P, A, Bv, C);
  // barycentric coordinates of Q w.r.t. (A,B,C): signed sub-areas over the area
  V3<double> nrm = cross(sub(Bv, A), sub(C, A));
  double nn = dot(nrm, nrm);
  double la = dot(nrm, cross(sub(C, Bv), sub(Q, Bv))) / nn;
  double lb = dot(nrm, cross(sub(A, C), sub(Q, C))) / nn;
  double lc = 1.0 - la - lb;
  double M[16], Mi[16];
  const double* Ta = T + 16 * (size_t)i0;
  const double* Tb = T + 16 * (size_t)i1;
  const double* Tc = T + 16 * (size_t)i2;
#pragma unroll
  for (int k = 0; k < 16; ++k) M[k] = Ta[k] * la + Tb[k] * lb + Tc[k] * lc;          // (:56)
  wd_inv4(M, Mi);                                                                   // (:57)
  double cx = Mi[0] * P.x + Mi[1] * P.y + Mi[2] * P.z + Mi[3];                       // (:58)
  double cy = Mi[4] * P.x + Mi[5] * P.y + Mi[6] * P.z + Mi[7];
  double cz = Mi[8] * P.x + Mi[9] * P.y + Mi[10] * P.z + Mi[11];
  can64[3 * i] = cx; can64[3 * i + 1] = cy; can64[3 * i + 2] = cz;
  if (closest_out) { closest_out[3 * i] = (float)Q.x; closest_out[3 * i + 1] = (float)Q.y; closest_out[3 * i + 2] = (float)Q.z; }
}

// can_dirs: normalised forward difference along the ray, last one duplicated (:62-64), in float64
__global__ void __launch_bounds__(256) k_warp_dirs(const double* __restrict__ can64, long long R, int S,
                                                    float* __restrict__ can_pts, float* __restrict__ can_dirs) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * S) return;
  int s = (int)(i % S);
  double x = can64[3 * i], y = can64[3 * i + 1], z = can64[3 * i + 2];
  can_pts[3 * i] = (float)x; can_pts[3 * i + 1] = (float)y; can_pts[3 * i + 2] = (float)z;
  if (!can_dirs) return;
  long long a = (s < S - 1) ? i : i - 1;      // difference (a+1) - a
  if (S == 1) { can_dirs[3 * i] = can_dirs[3 * i + 1] = can_dirs[3 * i + 2] = NAN; return; }
  double dx = can64[3 * (a + 1)] - can64[3 * a], dy = can64[3 * (a + 1) + 1] - can64[3 * a + 1],
         dz = can64[3 * (a + 1) + 2] - can64[3 * a + 2];
  double nrm = sqrt(dx * dx + dy * dy + dz * dz);
  can_dirs[3 * i] = (float)(dx / nrm); can_dirs[3 * i + 1] = (float)(dy / nrm); can_dirs[3 * i + 2] = (float)(dz / nrm);
}

// ---------------------------------------------------------------------------------------------
// one device allocation per mesh holds the whole BVH (+ sort buffers): NmMesh::bvh
struct BvhLayout {
  size_t keys_in, keys_out, lo, hi, children, parent, visit, leaf_face, tri9, cub_tmp, box, total;
};
static BvhLayout bvh_layout(int n, size_t cub_bytes) {
  BvhLayout L;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~size_t(255); return o; };
  L.keys_in = take(sizeof(unsigned long long) * n);
  L.keys_out = take(sizeof(unsigned long long) * n);
  L.lo = take(sizeof(float4) * (2 * (size_t)n));
  L.hi = take(sizeof(float4) * (2 * (size_t)n));
  L.children = take(sizeof(int2) * (size_t)n);
  L.parent = take(sizeof(int32_t) * (2 * (size_t)n));
  L.visit = take(sizeof(int32_t) * (size_t)n);
  L.leaf_face = take(sizeof(int32_t) * (size_t)n);
  L.tri9 = take(sizeof(float) * 9 * (size_t)n);
  L.cub_tmp = take(cub_bytes);
  L.box = take(64);                            // device-side bounding box of the vertices (6 order-preserving ints)
  L.total = off;
  return L;
}

static BvhView bvh_view(const NmMesh& m) {
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, cub_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, m.n_faces);
  BvhLayout L = bvh_layout(m.n_faces, cub_bytes);
  const char* base = m.bvh;
  BvhView B;
  B.n = m.n_faces;
  B.lo = reinterpret_cast<const float4*>(base + L.lo);
  B.hi = reinterpret_cast<const float4*>(base + L.hi);
  B.children = reinterpret_cast<const int2*>(base + L.children);
  B.leaf_face = reinterpret_cast<const int32_t*>(base + L.leaf_face);
  B.tri9 = reinterpret_cast<const float*>(base + L.tri9);
  return B;
}

extern "C" int nm_mesh_set(nm_ctx* ctx, int actor, const float* verts, int32_t n_verts, const int32_t* faces,
                           int32_t n_faces, const double* T, int32_t n_T, int32_t on_device, void* stream) {
  NM_ENTER(ctx);
  if (actor < 0 || actor >= NM_MAX_ACTORS || !verts || !faces || n_verts <= 0 || n_faces <= 0 || (T && n_T < n_verts))
    NM_FAIL(ctx, NM_ERR_INVALID, "nm_mesh_set: bad argument (need n_T >= n_verts)");
  if (!T) n_T = 0;                                   // distance queries only (nm_signed_distance)
  cudaStream_t st = (cudaStream_t)stream;
  NmMesh& m = ctx->meshes[actor];
  int rc;
  if ((rc = ensure(ctx, &m.verts, &m.cap_verts, (size_t)n_verts * 3))) return rc;
  if (T && (rc = ensure(ctx, &m.T, &m.cap_T, (size_t)n_T * 16))) return rc;
  if ((rc = ensure(ctx, &m.faces, &m.cap_faces, (size_t)n_faces * 3))) return rc;
  cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  NM_CHECK_CUDA(ctx, cudaMemcpyAsync(m.verts, verts, (size_t)n_verts * 3 * sizeof(float), kind, st));
  NM_CHECK_CUDA(ctx, cudaMemcpyAsync(m.faces, faces, (size_t)n_faces * 3 * sizeof(int32_t), kind, st));
  if (T) NM_CHECK_CUDA(ctx, cudaMemcpyAsync(m.T, T, (size_t)n_T * 16 * sizeof(double), kind, st));
  m.n_verts = n_verts; m.n_faces = n_faces; m.n_T = n_T;
  m.has_T = T != nullptr;
  m.pn_valid = false;
  // Bounds of the vertices, only used to normalise the Morton codes.  Renderer meshes (with T): on the host (82 KB, once per
  // frame), together with the vertex groups of the near/far cull.  Distance-only meshes from device memory (the trainer's
  // per-step queries): on the device -- no copy back, no synchronisation, no cull structure (nm_impl_near_far_mesh falls
  // back to the exhaustive loop when n_vgroups == 0).
  const bool device_bounds = on_device && !T;
  float3 bmin = make_float3(0.f, 0.f, 0.f), binv = make_float3(1.f, 1.f, 1.f);
  if (device_bounds) {
    m.n_vgroups = 0;
  } else {
    std::vector<float> hv((size_t)n_verts * 3);
    if (on_device) {
      NM_CHECK_CUDA(ctx, cudaMemcpyAsync(hv.data(), verts, hv.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
      NM_CHECK_CUDA(ctx, cudaStreamSynchronize(st));
    } else {
      memcpy(hv.data(), verts, hv.size() * sizeof(float));
    }
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int v = 0; v < n_verts; ++v)
      for (int c = 0; c < 3; ++c) { lo[c] = fminf(lo[c], hv[3 * v + c]); hi[c] = fmaxf(hi[c], hv[3 * v + c]); }
    if ((rc = nm_impl_build_vgroups(ctx, m, hv.data(), lo, hi, st))) return rc;      // near/far cull structure (rays.cu)
    bmin = make_float3(lo[0], lo[1], lo[2]);
    binv = make_float3(1.f / fmaxf(hi[0] - lo[0], 1e-20f), 1.f / fmaxf(hi[1] - lo[1], 1e-20f), 1.f / fmaxf(hi[2] - lo[2], 1e-20f));
  }
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, cub_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, n_faces);
  BvhLayout L = bvh_layout(n_faces, cub_bytes);
  if ((rc = ensure(ctx, &m.bvh, &m.cap_bvh, L.total))) return rc;
  char* base = m.bvh;
  auto* keys_in = reinterpret_cast<unsigned long long*>(base + L.keys_in);
  auto* keys_out = reinterpret_cast<unsigned long long*>(base + L.keys_out);
  float* tri9 = reinterpret_cast<float*>(base + L.tri9);
  int* box = nullptr;
  if (device_bounds) {
    box = reinterpret_cast<int*>(base + L.box);
    NM_CHECK_CUDA(ctx, cudaMemsetAsync(box, 0x7f, 3 * sizeof(int), st));
    NM_CHECK_CUDA(ctx, cudaMemsetAsync(box + 3, 0x80, 3 * sizeof(int), st));
    k_bbox<<<(n_verts + 255) / 256, 256, 0, st>>>(m.verts, n_verts, box);
    NM_CHECK_LAUNCH(ctx);
  }
  k_bvh_keys<<<(n_faces + 127) / 128, 128, 0, st>>>(m.verts, m.faces, n_faces, bmin, binv, box, tri9, keys_in);
  NM_CHECK_LAUNCH(ctx);
  NM_CHECK_CUDA(ctx, cub::DeviceRadixSort::SortKeys(base + L.cub_tmp, cub_bytes, keys_in, keys_out, n_faces, 0, 64, st));
  NM_LAUNCHED(ctx);
  auto* children = reinterpret_cast<int2*>(base + L.children);
  auto* parent = reinterpret_cast<int32_t*>(base + L.parent);
  auto* visit = reinterpret_cast<int32_t*>(base + L.visit);
  auto* leaf_face = reinterpret_cast<int32_t*>(base + L.leaf_face);
  NM_CHECK_CUDA(ctx, cudaMemsetAsync(visit, 0, sizeof(int32_t) * (size_t)n_faces, st));
  k_bvh_hierarchy<<<(n_faces + 127) / 128, 128, 0, st>>>(keys_out, n_faces, children, parent, leaf_face);
  NM_CHECK_LAUNCH(ctx);
  k_bvh_refit<<<(n_faces + 127) / 128, 128, 0, st>>>(tri9, leaf_face, n_faces, children, parent, visit,
                                                      reinterpret_cast<float4*>(base + L.lo), reinterpret_cast<float4*>(base + L.hi));
  NM_CHECK_LAUNCH(ctx);
  m.set = true;
  return NM_OK;
}

extern "C" int nm_warp_to_canonical(nm_ctx* ctx, int actor, const float* pts, int64_t R, int32_t S, float* can_pts,
                                    float* can_dirs, float* closest, int32_t* face_id, void* stream) {
  NM_ENTER(ctx);
  if (R == 0) return NM_OK;
  if (actor < 0 || actor >= NM_MAX_ACTORS || !ctx->meshes[actor].set || !ctx->meshes[actor].has_T)
    NM_FAIL(ctx, NM_ERR_STATE, "nm_warp_to_canonical: mesh (with per-vertex transforms) not set");
  if (!pts || !can_pts || R < 0 || S <= 0) NM_FAIL(ctx, NM_ERR_INVALID, "nm_warp_to_canonical: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  NmMesh& m = ctx->meshes[actor];
  long long n = (long long)R * S;
  // float64 canonical points: private scratch sized on demand (the frame drivers own ctx->ws)
  int rc;
  if ((rc = ensure(ctx, &ctx->can64, &ctx->can64_cap, (size_t)n * 3))) return rc;
  double* can64 = ctx->can64;
  BvhView B = bvh_view(m);
  // winning faces: the caller's buffer, or a private scratch
  int32_t* fid = face_id;
  if (!fid) {
    if ((rc = ensure(ctx, &ctx->face_tmp, &ctx->face_cap, (size_t)n))) return rc;
    fid = ctx->face_tmp;
  }
  {
    int lg = 1;                                           // packets of 2 rays x 16 samples, narrower where S or R need it
    while (lg > 0 && (S % (32 >> lg) != 0 || R < (1 << lg))) --lg;
    long long warps = lg == 0 ? (n + 31) / 32 : ((R + (1 << lg) - 1) >> lg) * (long long)(S / (32 >> lg));
    k_warp_nearest<<<(unsigned)((warps + 3) / 4), 128, 0, st>>>(B, pts, (long long)R, (int)S, lg, fid);
    NM_CHECK_LAUNCH(ctx);
  }
  k_warp_points<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(m.verts, m.faces, m.T, pts, n, fid, can64, closest);
  NM_CHECK_LAUNCH(ctx);
  k_warp_dirs<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(can64, R, S, can_pts, can_dirs);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

// ---------------------------------------------------------------------------------------------
// Signed distance to the mesh (igl.signed_distance, pseudo-normal sign): closest point and face as above, sign of
// (p - closest) . N with N = the face normal, or the sum of the two unit face normals at an edge, or the
// angle-weighted vertex normal, according to which barycentric coordinates of the closest point vanish
// (Baerentzen & Aanaes 2005, what igl::pseudonormal_test evaluates).  float64 after the fp32 arg-min.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ V3<double> ld3d(const float* v, int i) { return {(double)v[3 * i], (double)v[3 * i + 1], (double)v[3 * i + 2]}; }
__device__ __forceinline__ V3<double> unit_normal(V3<double> a, V3<double> b, V3<double> c) {
  V3<double> n = cross(sub(b, a), sub(c, a));
  const double l = sqrt(dot(n, n));
  const double s = 1.0 / fmax(l, 1e-300);
  return {n.x * s, n.y * s, n.z * s};
}
__device__ __forceinline__ double corner_angle(V3<double> u, V3<double> v) {
  const double c = dot(u, v) / fmax(sqrt(dot(u, u)) * sqrt(dot(v, v)), 1e-300);
  return acos(fmin(1.0, fmax(-1.0, c)));
}

__global__ void k_vertex_normals(const float* __restrict__ verts, const int32_t* __restrict__ faces, int nf, double* __restrict__ vnorm) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  const int i0 = faces[3 * f], i1 = faces[3 * f + 1], i2 = faces[3 * f + 2];
  const V3<double> A = ld3d(verts, i0), B = ld3d(verts, i1), C = ld3d(verts, i2);
  const V3<double> n = unit_normal(A, B, C);
  const double w0 = corner_angle(sub(B, A), sub(C, A)), w1 = corner_angle(sub(C, B), sub(A, B)), w2 = corner_angle(sub(A, C), sub(B, C));
  atomicAdd(vnorm + 3 * i0, n.x * w0); atomicAdd(vnorm + 3 * i0 + 1, n.y * w0); atomicAdd(vnorm + 3 * i0 + 2, n.z * w0);
  atomicAdd(vnorm + 3 * i1, n.x * w1); atomicAdd(vnorm + 3 * i1 + 1, n.y * w1); atomicAdd(vnorm + 3 * i1 + 2, n.z * w1);
  atomicAdd(vnorm + 3 * i2, n.x * w2); atomicAdd(vnorm + 3 * i2 + 1, n.y * w2); atomicAdd(vnorm + 3 * i2 + 2, n.z * w2);
}

// edge e of face f joins vertices (e, e+1 mod 3); key = (min << 32) | max, value = 3f + e
__global__ void k_edge_keys(const int32_t* __restrict__ faces, int nf, unsigned long long* __restrict__ keys, int32_t* __restrict__ vals) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= 3 * nf) return;
  const int f = q / 3, e = q - 3 * f;
  const unsigned a = (unsigned)faces[3 * f + e], b = (unsigned)faces[3 * f + (e + 1) % 3];
  keys[q] = ((unsigned long long)min(a, b) << 32) | (unsigned long long)max(a, b);
  vals[q] = q;
}
__global__ void k_edge_adjacency(const unsigned long long* __restrict__ keys, const int32_t* __restrict__ vals, int ne, int32_t* __restrict__ adj) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= ne) return;
  int other = -1;
  if (q + 1 < ne && keys[q + 1] == keys[q]) other = vals[q + 1] / 3;
  else if (q > 0 && keys[q - 1] == keys[q]) other = vals[q - 1] / 3;
  adj[vals[q]] = other;
}

__global__ void __launch_bounds__(128) k_signed_distance(BvhView B, const float* __restrict__ verts, const int32_t* __restrict__ faces,
                                                          const double* __restrict__ vnorm, const int32_t* __restrict__ adj,
                                                          const float* __restrict__ pts, long long n,
                                                          const int32_t* __restrict__ face_in, double* __restrict__ S_out,
                                                          int32_t* __restrict__ I_out, double* __restrict__ C_out) {
  // face_in: the winners of k_warp_nearest (the traversal runs as its own 38-register kernel, like the warp stage; this
  // kernel is then the float64 evaluation only)
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  V3<float> p{pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
  const int f = face_in[i];
  const int iv[3] = {faces[3 * f], faces[3 * f + 1], faces[3 * f + 2]};
  const V3<double> P{(double)p.x, (double)p.y, (double)p.z};
  const V3<double> A = ld3d(verts, iv[0]), Bv = ld3d(verts, iv[1]), C = ld3d(verts, iv[2]);
  const V3<double> Q = closest_on_tri<double>(P, A, Bv, C);
  const V3<double> nrm = cross(sub(Bv, A), sub(C, A));
  const double nn = dot(nrm, nrm);
  double L[3];
  L[0] = dot(nrm, cross(sub(C, Bv), sub(Q, Bv))) / nn;
  L[1] = dot(nrm, cross(sub(A, C), sub(Q, C))) / nn;
  L[2] = 1.0 - L[0] - L[1];
  const double eps = 1e-9;
  const bool on[3] = {L[0] > eps, L[1] > eps, L[2] > eps};
  const int cnt = (int)on[0] + (int)on[1] + (int)on[2];
  V3<double> N = unit_normal(A, Bv, C);
  if (cnt == 1) {
    const int k = L[0] >= L[1] ? (L[0] >= L[2] ? 0 : 2) : (L[1] >= L[2] ? 1 : 2);
    N = {vnorm[3 * iv[k]], vnorm[3 * iv[k] + 1], vnorm[3 * iv[k] + 2]};
  } else if (cnt == 2) {
    const int e = !on[2] ? 0 : (!on[0] ? 1 : 2);          // edge (v0v1), (v1v2), (v2v0)
    const int g = adj[3 * f + e];
    if (g >= 0) {
      const V3<double> M = unit_normal(ld3d(verts, faces[3 * g]), ld3d(verts, faces[3 * g + 1]), ld3d(verts, faces[3 * g + 2]));
      N = {N.x + M.x, N.y + M.y, N.z + M.z};
    }
  }
  const V3<double> d = sub(P, Q);
  const double s = dot(d, N);
  const double dist = sqrt(dot(d, d));
  if (S_out) S_out[i] = s < 0.0 ? -dist : dist;
  if (I_out) I_out[i] = f;
  if (C_out) { C_out[3 * i] = Q.x; C_out[3 * i + 1] = Q.y; C_out[3 * i + 2] = Q.z; }
}

static int build_pseudonormals(nm_ctx* ctx, NmMesh& m, cudaStream_t st) {
  int rc;
  const int nf = m.n_faces, ne = 3 * nf;
  if ((rc = ensure(ctx, &m.vnorm, &m.cap_vnorm, (size_t)m.n_verts * 3))) return rc;
  if ((rc = ensure(ctx, &m.adj, &m.cap_adj, (size_t)ne))) return rc;
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const int32_t*)nullptr, (int32_t*)nullptr, ne);
  const size_t kb = ((size_t)ne * 8 + 255) & ~size_t(255), vb = ((size_t)ne * 4 + 255) & ~size_t(255);
  if ((rc = ensure(ctx, &m.pn_tmp, &m.cap_pn_tmp, 2 * kb + 2 * vb + cub_bytes + 256))) return rc;
  auto* k_in = reinterpret_cast<unsigned long long*>(m.pn_tmp);
  auto* k_out = reinterpret_cast<unsigned long long*>(m.pn_tmp + kb);
  auto* v_in = reinterpret_cast<int32_t*>(m.pn_tmp + 2 * kb);
  auto* v_out = reinterpret_cast<int32_t*>(m.pn_tmp + 2 * kb + vb);
  char* tmp = m.pn_tmp + 2 * kb + 2 * vb;
  NM_CHECK_CUDA(ctx, cudaMemsetAsync(m.vnorm, 0, (size_t)m.n_verts * 3 * sizeof(double), st));
  k_vertex_normals<<<(nf + 127) / 128, 128, 0, st>>>(m.verts, m.faces, nf, m.vnorm);
  NM_CHECK_LAUNCH(ctx);
  k_edge_keys<<<(ne + 127) / 128, 128, 0, st>>>(m.faces, nf, k_in, v_in);
  NM_CHECK_LAUNCH(ctx);
  NM_CHECK_CUDA(ctx, cub::DeviceRadixSort::SortPairs(tmp, cub_bytes, k_in, k_out, v_in, v_out, ne, 0, 64, st));
  NM_LAUNCHED(ctx);
  k_edge_adjacency<<<(ne + 127) / 128, 128, 0, st>>>(k_out, v_out, ne, m.adj);
  NM_CHECK_LAUNCH(ctx);
  m.pn_valid = true;
  return NM_OK;
}

extern "C" int nm_signed_distance(nm_ctx* ctx, int actor, const float* pts, int64_t n, double* S, int32_t* I, double* C, void* stream) {
  NM_ENTER(ctx);
  if (n == 0) return NM_OK;
  if (actor < 0 || actor >= NM_MAX_ACTORS || !ctx->meshes[actor].set) NM_FAIL(ctx, NM_ERR_STATE, "nm_signed_distance: mesh not set");
  if (!pts || n < 0) NM_FAIL(ctx, NM_ERR_INVALID, "nm_signed_distance: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  NmMesh& m = ctx->meshes[actor];
  if (!m.pn_valid) {
    int rc = build_pseudonormals(ctx, m, st);
    if (rc != NM_OK) return rc;
  }
  // winning faces: the caller's buffer, or a private scratch
  int32_t* fid = I;
  if (!fid) {
    int rc = ensure(ctx, &ctx->face_tmp, &ctx->face_cap, (size_t)n);
    if (rc != NM_OK) return rc;
    fid = ctx->face_tmp;
  }
  const long long warps = (n + 31) / 32;
  k_warp_nearest<<<(unsigned)((warps + 3) / 4), 128, 0, st>>>(bvh_view(m), pts, (long long)n, 1, 0, fid);
  NM_CHECK_LAUNCH(ctx);
  k_signed_distance<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(bvh_view(m), m.verts, m.faces, m.vnorm, m.adj, pts, n, fid, S, I, C);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

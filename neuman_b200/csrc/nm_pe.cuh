// Sample fetch + positional encoding shared by the two MLP kernels.
//   Embedder.forward   models/vanilla.py:82-92   ('posenc' :60-79, 'rotate' :44-58)
//   pts = o + d * z    utils/ray_utils.py:131    (separately rounded multiply and add)
#pragma once
#include "nm_internal.cuh"

struct NmMlpInput {
  const float* pts;      // [n,3] or null (rays mode); NeRF-T nets: [n,4] = (x, y, z, t)
  const float* views;    // [n,3] / [n/group,3] or null
  const float* origins;  // rays mode: [R,3]
  const float* dirs;     // rays mode: [R,3]
  const float* z;        // rays mode: [R*S]
  long long n;           // number of samples
  int group;             // samples per ray (views broadcast); 0 = per-sample views
  float t;               // NeRF-T nets in rays mode: the time of every sample (one frame)
};

struct NmPeSpec {
  int kind;            // NM_PE_*
  int n_freqs;
  const float* table;  // posenc: freqs[n_freqs]; rotate: bvals[3*n_freqs][3]
};

// time of sample i of a NeRF-T net: column 3 of pts, or the frame's time in rays mode
__device__ __forceinline__ float nm_fetch_time(const NmMlpInput& in, long long i) {
  return in.pts ? in.pts[4 * i + 3] : in.t;
}

// Sample i whose ray (rays mode) / view row (pts mode) is g: i / group, or i in pts mode when group <= 0.
// kPtsLd: floats per row of pts (4 for NeRF-T nets, whose rows carry the time after x, y, z).
template <int kPtsLd = 3>
__device__ __forceinline__ void nm_fetch_sample_at(const NmMlpInput& in, long long i, long long g, float p[3], float v[3]) {
  if (in.pts) {
    p[0] = in.pts[kPtsLd * i]; p[1] = in.pts[kPtsLd * i + 1]; p[2] = in.pts[kPtsLd * i + 2];
    if (in.views) { v[0] = in.views[3 * g]; v[1] = in.views[3 * g + 1]; v[2] = in.views[3 * g + 2]; }
    else { v[0] = v[1] = v[2] = 0.f; }
  } else {
    float zz = in.z[i];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float d = in.dirs[3 * g + c];
      v[c] = d;
      p[c] = __fadd_rn(in.origins[3 * g + c], __fmul_rn(d, zz));
    }
  }
}
template <int kPtsLd = 3>
__device__ __forceinline__ void nm_fetch_sample(const NmMlpInput& in, long long i, float p[3], float v[3]) {
  nm_fetch_sample_at<kPtsLd>(in, i, in.pts && in.group <= 0 ? i : i / in.group, p, v);
}

// Writes the 2 channels produced by the (q)-th sin/cos pair of the encoding of x; q in [0, 3*n_freqs).
// Returns the channel indices through c_sin / c_cos (channel 0..2 = the raw input).
__device__ __forceinline__ void nm_pe_pair(const NmPeSpec& pe, const float x[3], int q, float& s, float& c,
                                           int& c_sin, int& c_cos) {
  float arg;
  if (pe.kind == NM_PE_ROTATE) {
    const float* b = pe.table + 3 * q;
    arg = fmaf(x[2], b[2], fmaf(x[1], b[1], x[0] * b[0]));          // inputs @ bvals.T (K=3)
    c_sin = 3 + q;
    c_cos = 3 + 3 * pe.n_freqs + q;
  } else {
    int k = q / 3, d = q - 3 * k;
    arg = x[d] * pe.table[k];                                        // x * freq (exact for 2^k)
    c_sin = 3 + 6 * k + d;
    c_cos = 3 + 6 * k + 3 + d;
  }
  sincosf(arg, &s, &c);
}

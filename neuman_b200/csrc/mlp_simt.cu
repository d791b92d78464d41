// CUDA-core fp32 implementation of Joiner.forward = positional encoding + the 8x256 NeRF MLP
// (models/vanilla.py:82-92, :120-152, :162-166).  "Strict" arithmetic (fp32 FMA accumulation, the
// same operation the reference's sgemm performs); it is the on-device cross-check for the
// tensor-core kernel (mlp_tc.cu) and the NM_MLP_SIMT_F32 mode of the API.
//
// One CTA = 64 samples, 256 threads; activations ping-pong between two [64][256] shared-memory
// buffers; weights are read transposed ([in][out], coalesced across lanes, L1/L2 resident).
#include "nm_internal.cuh"
#include "nm_pe.cuh"

#define TM 64
#define NT 256

struct SimtParams {
  const float* w[8]; const float* b[8];
  const float* feat_w; const float* feat_b;
  const float* alpha_w; const float* alpha_b;
  const float* views_w; const float* views_b;
  const float* rgb_w; const float* rgb_b;
  const float* out_w; const float* out_b;     // output_linear of a view-independent net: Wt [256][4], bias [4]
  NmPeSpec pos_pe, dir_pe;
};

// acc[8][NJ] += in[rows ty*8.., k] * Wt[k][tx + 32 j]
template <int NJ>
__device__ __forceinline__ void gemm_acc(float (&acc)[8][NJ], const float* __restrict__ in, int ldin, int K,
                                         const float* __restrict__ Wt, int N, int tx, int ty) {
  const float* in0 = in + (size_t)(ty * 8) * ldin;
#pragma unroll 4
  for (int k = 0; k < K; ++k) {
    float a[8], b[NJ];
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = in0[i * ldin + k];
#pragma unroll
    for (int j = 0; j < NJ; ++j) b[j] = __ldg(Wt + (size_t)k * N + tx + 32 * j);
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < NJ; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
  }
}

template <int NJ>
__device__ __forceinline__ void store_out(const float (&acc)[8][NJ], const float* __restrict__ bias, bool relu,
                                          float* out, int ldout, int tx, int ty) {
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    float bj = __ldg(bias + tx + 32 * j);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float v = acc[i][j] + bj;
      if (relu) v = fmaxf(v, 0.f);
      out[(size_t)(ty * 8 + i) * ldout + tx + 32 * j] = v;
    }
  }
}

template <int NJ>
__device__ __forceinline__ void zero_acc(float (&acc)[8][NJ]) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[i][j] = 0.f;
}

// kView: use_viewdirs=True (alpha, feature, views and rgb heads); otherwise output_linear on layer 7 (:145-146) and no
// direction input.  kTime: a NeRF-T net (view-dependent, position input (x, y, z, t)): its 84-wide position encoding is
// built in the reference's column order, so pts_linears.0 / .5 are used as given.
template <bool kView, bool kTime = false>
__device__ __forceinline__ void mlp_simt_body(const SimtParams& P, const NmMlpInput& in, float* __restrict__ raw) {
  constexpr int PE_LD = kTime ? 96 : 64;
  extern __shared__ float sm[];
  float* hA = sm;                    // [64][256]
  float* hB = hA + TM * 256;         // [64][256]
  float* pe = hB + TM * 256;         // [64][PE_LD]  (63 / 84 used)
  float* vpe = pe + TM * PE_LD;      // [64][32]  (27 used)
  float* s_alpha = vpe + TM * 32;    // [64]
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  const long long base = (long long)blockIdx.x * TM;

  // ---- positional encodings ----
  const int npos = (kTime ? 4 : 3) * P.pos_pe.n_freqs, ndir = kView ? 3 * P.dir_pe.n_freqs : 0;
  for (int t = tid; t < TM * (npos + ndir + 2); t += NT) {
    int s = t / (npos + ndir + 2), q = t - s * (npos + ndir + 2);
    long long i = base + s;
    float p[3] = {0, 0, 0}, v[3] = {0, 0, 0}, tm = 0.f;
    if (i < in.n) {
      nm_fetch_sample<kTime ? 4 : 3>(in, i, p, v);
      if (kTime) tm = nm_fetch_time(in, i);
    }
    if (kTime && q < npos) {
      // Embedder.forward with input_dims = 4 (:69-75): sin(x f_k) at column 4 + 8k + d, cos at 8 + 8k + d (d = 3: time)
      const int k = q >> 2, d = q & 3;
      float sn, cs;
      sincosf((d < 3 ? p[d] : tm) * P.pos_pe.table[k], &sn, &cs);
      pe[s * PE_LD + 4 + 8 * k + d] = sn; pe[s * PE_LD + 8 + 8 * k + d] = cs;
    } else if (q < npos) {
      float sn, cs; int ci, cj;
      nm_pe_pair(P.pos_pe, p, q, sn, cs, ci, cj);
      pe[s * PE_LD + ci] = sn; pe[s * PE_LD + cj] = cs;
    } else if (q < npos + ndir) {
      float sn, cs; int ci, cj;
      nm_pe_pair(P.dir_pe, v, q - npos, sn, cs, ci, cj);
      vpe[s * 32 + ci] = sn; vpe[s * 32 + cj] = cs;
    } else if (q == npos + ndir) {
      pe[s * PE_LD + 0] = p[0]; pe[s * PE_LD + 1] = p[1]; pe[s * PE_LD + 2] = p[2];
      if (kTime) pe[s * PE_LD + 3] = tm;
      else pe[s * PE_LD + 63] = 0.f;
    } else if (kView) {
      vpe[s * 32 + 0] = v[0]; vpe[s * 32 + 1] = v[1]; vpe[s * 32 + 2] = v[2];
#pragma unroll
      for (int c = 27; c < 32; ++c) vpe[s * 32 + c] = 0.f;
    }
  }
  __syncthreads();

  const int KP = kTime ? NM_POS_PE_T : 3 + 2 * npos;   // 63 / 84
  const int KV = 3 + 2 * ndir;   // 27
  float acc[8][8];
  float* cur = hA;
  float* nxt = hB;
  // layer 0
  zero_acc(acc);
  gemm_acc<8>(acc, pe, PE_LD, KP, P.w[0], 256, tx, ty);
  store_out<8>(acc, P.b[0], true, cur, 256, tx, ty);
  __syncthreads();
  for (int l = 1; l < 8; ++l) {
    zero_acc(acc);
    const float* W = P.w[l];
    if (l == 5) {                                   // cat([input_pts, h]) (models/vanilla.py:131)
      gemm_acc<8>(acc, pe, PE_LD, KP, W, 256, tx, ty);
      W += (size_t)KP * 256;
    }
    gemm_acc<8>(acc, cur, 256, 256, W, 256, tx, ty);
    store_out<8>(acc, P.b[l], true, nxt, 256, tx, ty);
    __syncthreads();
    float* t = cur; cur = nxt; nxt = t;
  }
  if (!kView) {
    // raw = output_linear(h7) (:146), fp32 FMAs over k in order, then the bias
    const int s = tid >> 2, o = tid & 3;
    const long long i = base + s;
    const float* h = cur + (size_t)s * 256;
    float a = 0.f;
    for (int k = 0; k < 256; ++k) a = fmaf(h[k], __ldg(P.out_w + (size_t)k * 4 + o), a);
    if (i < in.n) raw[4 * i + o] = a + __ldg(P.out_b + o);
    return;
  }
  // alpha = alpha_linear(h7)   (:135)
  if (tid < TM) {
    const float* h = cur + (size_t)tid * 256;
    float a = 0.f;
    for (int k = 0; k < 256; ++k) a = fmaf(h[k], __ldg(P.alpha_w + k), a);
    s_alpha[tid] = a + __ldg(P.alpha_b);
  }
  // feature = feature_linear(h7), no activation (:136)
  zero_acc(acc);
  gemm_acc<8>(acc, cur, 256, 256, P.feat_w, 256, tx, ty);
  store_out<8>(acc, P.feat_b, false, nxt, 256, tx, ty);
  __syncthreads();
  { float* t = cur; cur = nxt; nxt = t; }
  // views layer: relu(cat([feature, views_pe]) W + b), 283 -> 128 (:137-141)
  {
    float acc4[8][4];
    zero_acc(acc4);
    gemm_acc<4>(acc4, cur, 256, 256, P.views_w, 128, tx, ty);
    gemm_acc<4>(acc4, vpe, 32, KV, P.views_w + (size_t)256 * 128, 128, tx, ty);
    store_out<4>(acc4, P.views_b, true, nxt, 256, tx, ty);
  }
  __syncthreads();
  // rgb = rgb_linear(h) (:143); output order [r,g,b,sigma] (:144)
  {
    int s = tid >> 2, o = tid & 3;
    long long i = base + s;
    float val;
    if (o < 3) {
      const float* h = nxt + (size_t)s * 256;
      float a = 0.f;
      for (int k = 0; k < 128; ++k) a = fmaf(h[k], __ldg(P.rgb_w + (size_t)k * 3 + o), a);
      val = a + __ldg(P.rgb_b + o);
    } else {
      val = s_alpha[s];
    }
    if (i < in.n) raw[4 * i + o] = val;
  }
}

__global__ void __launch_bounds__(NT, 1) k_mlp_simt(SimtParams P, NmMlpInput in, float* __restrict__ raw) {
  mlp_simt_body<true>(P, in, raw);
}
__global__ void __launch_bounds__(NT, 1) k_mlp_simt_noview(SimtParams P, NmMlpInput in, float* __restrict__ raw) {
  mlp_simt_body<false>(P, in, raw);
}
__global__ void __launch_bounds__(NT, 1) k_mlp_simt_nerft(SimtParams P, NmMlpInput in, float* __restrict__ raw) {
  mlp_simt_body<true, true>(P, in, raw);
}

int nm_simt_forward(nm_ctx* ctx, const NmNet& net, const float* pts, const float* views, const float* origins,
                    const float* dirs, const float* z, int64_t n, int32_t group, float t, float* raw, cudaStream_t st) {
  SimtParams P;
  for (int l = 0; l < 8; ++l) { P.w[l] = net.f32 + net.o_pts_w[l]; P.b[l] = net.f32 + net.o_pts_b[l]; }
  P.feat_w = net.f32 + net.o_feat_w; P.feat_b = net.f32 + net.o_feat_b;
  P.alpha_w = net.f32 + net.o_alpha_w; P.alpha_b = net.f32 + net.o_alpha_b;
  P.views_w = net.f32 + net.o_views_w; P.views_b = net.f32 + net.o_views_b;
  P.rgb_w = net.f32 + net.o_rgb_w; P.rgb_b = net.f32 + net.o_rgb_b;
  P.out_w = net.f32 + net.o_out_w; P.out_b = net.f32 + net.o_out_b;
  P.pos_pe = {net.desc.pos_pe_kind, net.desc.pos_n_freqs, net.f32 + net.o_pos_bv};
  P.dir_pe = {net.desc.dir_pe_kind, net.desc.dir_n_freqs, net.f32 + net.o_dir_bv};
  NmMlpInput in{pts, views, origins, dirs, z, (long long)n, group, t};
  size_t smem = (size_t)(2 * TM * 256 + TM * 64 + TM * 32 + TM) * sizeof(float);
  unsigned blocks = (unsigned)((n + TM - 1) / TM);
  if (net.kind == NM_NET_NERFT) {
    smem += (size_t)TM * (96 - 64) * sizeof(float);
    NM_SET_SMEM_ONCE(ctx, (k_mlp_simt_nerft), (int)smem);
    k_mlp_simt_nerft<<<blocks, NT, smem, st>>>(P, in, raw);
  } else if (net.kind == NM_NET_VIEW) {
    NM_SET_SMEM_ONCE(ctx, (k_mlp_simt), (int)smem);
    k_mlp_simt<<<blocks, NT, smem, st>>>(P, in, raw);
  } else {
    NM_SET_SMEM_ONCE(ctx, (k_mlp_simt_noview), (int)smem);
    k_mlp_simt_noview<<<blocks, NT, smem, st>>>(P, in, raw);
  }
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

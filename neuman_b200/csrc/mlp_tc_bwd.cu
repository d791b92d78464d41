// Backward (input-gradient) chain of NeRF.forward (models/vanilla.py:120-152) on the tensor cores:
// the adjoint of mlp_tc.cu's training forward, same machinery (wgmma, fp16 operands, fp32 register
// accumulators, bulk-TMA weight ring, persistent CTAs of two 64-row warpgroups, activations kept on chip).
//
// For every sample row, with g = dL/d raw (4 values) scaled by the loss scale S:
//   dVpre = (g_rgb @ Wrgb) * [V > 0]                         (K = 3, plain FFMAs; [V > 0] from sign words)
//   b0: dF   = dVpre @ Wviews[:, :256]                        (K = 128)
//   b1: dX8  = dF @ Wfeature + g_alpha * w_alpha ;  dpre7 = dX8 * [X8 > 0]
//   b2..b8 (l = 7..1): dX_{l-1} = dpre_l @ W_l[:, -256:] ;   dpre_{l-1} = dX_{l-1} * [X_{l-1} > 0]
// A view-independent net (use_viewdirs=False, raw = output_linear(X7), :146) has the head
//   dpre7 = (g @ Wout) * [X7 > 0]                            (K = 4, plain FFMAs; [X7 > 0] from sign words)
// in place of dVpre, b0 and b1, then the same steps b2..b8.
// Every dpre_l, dF and dVpre is written to HBM in fp16 by TMA stores from the A buffer (they are the left operands of the weight-gradient
// GEMMs dW_l = dpre_l^T @ X_{l-1}, done by the caller with the forward's activation stash), and stays in shared
// memory as the next step's A operand.  The ReLU masks come from the forward's 256-bit sign words.
// Gradients w.r.t. the sample positions are not produced (the trainers treat samples as constants).
#include "nm_internal.cuh"
#include "nm_pe.cuh"
#include "tc_common.cuh"
#include <string.h>

#define BW_STEPS 9
__host__ __device__ constexpr int bw_nkb(int b) { return b == 0 ? 2 : 4; }
#define BW_SLABS (2 + 8 * 4)
#define BW_SLABS_NOVIEW (7 * 4)                           // b2..b8 only
#define BW_FIRST(view) ((view) ? 0 : 2)
__host__ __device__ constexpr int bw_slabs(bool view) { return view ? BW_SLABS : BW_SLABS_NOVIEW; }
__host__ __device__ constexpr int bw_const_floats(bool view) { return view ? 256 + 384 : 4 * 256; }

template <bool kView>
struct BwCfg {
  static constexpr int THREADS = 256;                      // two consumer warpgroups
  static constexpr int NSLOT = 4;                           // depth of the weight ring
  static constexpr int WG_BYTES = 4 * TC_KB_BYTES;          // per warpgroup: act[4 k-blocks]
  static constexpr int OFF_RING = 2 * WG_BYTES;
  static constexpr int OFF_BAR = OFF_RING + NSLOT * TC_SLAB_BYTES;
  static constexpr int OFF_CONST = OFF_BAR + 16 * NSLOT;     // w_alpha[256] | w_rgb[3][128] (or w_out[4][256]), fp32
  static constexpr int SMEM_USED = OFF_CONST + 4 * bw_const_floats(kView);
  static constexpr int SMEM_BYTES = SMEM_USED + 1024;
};
static_assert(BwCfg<true>::SMEM_BYTES <= 232448 && BwCfg<false>::SMEM_BYTES <= 232448,
              "shared memory of the backward kernel exceeds 227 KB");

struct BwParams {
  const uint8_t* wimg;      // transposed weight slabs
  const float* d_raw;       // [n][4] fp32 dL/d(r,g,b,sigma)
  const float* scale;       // device scalar: loss scale S (a power of two)
  const float* w_alpha;     // [256] fp32 alpha_linear.weight
  const float* w_rgb;       // [3][128] fp32 rgb_linear.weight (view-independent nets: [4][256] output_linear.weight)
  const uint32_t* st_m;     // [9][n][8] forward stash: ReLU sign words of pts_linears 0..7 and (plane 8, 4 words) of the views layer
  long long n, n_tiles;
  CUtensorMap map_pre, map_f, map_v;   // TMA store maps of g_pre [8][n][256] / g_f [n][256] / g_v [n][128]
};

// mask bit of column c = 8j + 2q + e in word j / 4 of a row's sign words (mlp_tc.cu fwd_epi)
__device__ __forceinline__ bool sign_bit(const uint32_t (&w)[8], int j, int q, int e) {
  return (w[j >> 2] >> (16 * ((j >> 1) & 1) + 8 * e + 4 * (j & 1) + q)) & 1u;
}

// 256 accumulator columns of this thread's rows rA, rA + 8: (+ rank-1 alpha term), ReLU mask from sign bits, pack,
// swizzled store into the next A operand (from where a TMA store takes it to the HBM gradient plane)
template <bool ALPHA, bool MASK>
__device__ __forceinline__ void bw_epi(const float (&d)[128], uint8_t* act, int rA, int q, const float* s_walpha, float daA,
                                       float daB, const uint32_t (&mA)[8], const uint32_t (&mB)[8]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c = 8 * j + 2 * q;
    float x0 = d[4 * j], x1 = d[4 * j + 1], y0 = d[4 * j + 2], y1 = d[4 * j + 3];
    if (ALPHA) {
      const float2 w = *reinterpret_cast<const float2*>(s_walpha + c);
      x0 = fmaf(daA, w.x, x0); x1 = fmaf(daA, w.y, x1);
      y0 = fmaf(daB, w.x, y0); y1 = fmaf(daB, w.y, y1);
    }
    if (MASK) {
      if (!sign_bit(mA, j, q, 0)) x0 = 0.f;
      if (!sign_bit(mA, j, q, 1)) x1 = 0.f;
      if (!sign_bit(mB, j, q, 0)) y0 = 0.f;
      if (!sign_bit(mB, j, q, 1)) y1 = 0.f;
    }
    uint8_t* blk = act + (j >> 3) * TC_KB_BYTES;
    *reinterpret_cast<uint32_t*>(blk + swz_off(rA, c)) = pack_f16x2(x0, x1, false);
    *reinterpret_cast<uint32_t*>(blk + swz_off(rA + 8, c)) = pack_f16x2(y0, y1, false);
  }
}

__device__ __forceinline__ void load_signs(const uint32_t* m, long long i, long long n, uint32_t (&w)[8]) {
  uint4 a = make_uint4(0, 0, 0, 0), b = a;
  if (i < n) { a = __ldg(reinterpret_cast<const uint4*>(m + i * 8)); b = __ldg(reinterpret_cast<const uint4*>(m + i * 8) + 1); }
  w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
}

// Head of a view-independent net: dpre7 = (S g[0..3] @ Wout) masked by [X7 > 0], for this thread's accumulator-layout
// share (rows rA, rA + 8; columns 8j + 2q, +1), stored swizzled into the A buffer like bw_epi
__device__ __forceinline__ void bw_head_noview(uint8_t* act, int rA, int q, const float* s_wout, const float4 gA,
                                               const float4 gB, const uint32_t (&mA)[8], const uint32_t (&mB)[8]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c = 8 * j + 2 * q;
    const float2 w0 = *reinterpret_cast<const float2*>(s_wout + c), w1 = *reinterpret_cast<const float2*>(s_wout + 256 + c);
    const float2 w2 = *reinterpret_cast<const float2*>(s_wout + 512 + c), w3 = *reinterpret_cast<const float2*>(s_wout + 768 + c);
    float x0 = fmaf(gA.x, w0.x, fmaf(gA.y, w1.x, fmaf(gA.z, w2.x, gA.w * w3.x)));
    float x1 = fmaf(gA.x, w0.y, fmaf(gA.y, w1.y, fmaf(gA.z, w2.y, gA.w * w3.y)));
    float y0 = fmaf(gB.x, w0.x, fmaf(gB.y, w1.x, fmaf(gB.z, w2.x, gB.w * w3.x)));
    float y1 = fmaf(gB.x, w0.y, fmaf(gB.y, w1.y, fmaf(gB.z, w2.y, gB.w * w3.y)));
    if (!sign_bit(mA, j, q, 0)) x0 = 0.f;
    if (!sign_bit(mA, j, q, 1)) x1 = 0.f;
    if (!sign_bit(mB, j, q, 0)) y0 = 0.f;
    if (!sign_bit(mB, j, q, 1)) y1 = 0.f;
    uint8_t* blk = act + (j >> 3) * TC_KB_BYTES;
    *reinterpret_cast<uint32_t*>(blk + swz_off(rA, c)) = pack_f16x2(x0, x1, false);
    *reinterpret_cast<uint32_t*>(blk + swz_off(rA + 8, c)) = pack_f16x2(y0, y1, false);
  }
}

template <bool kView>
__device__ __forceinline__ void mlp_tc_bwd_body(const BwParams& P) {
  using C = BwCfg<kView>;
  constexpr int SLABS = bw_slabs(kView);
  extern __shared__ uint8_t smem_dyn[];
  const uint32_t pad = (1024 - (smem_u32(smem_dyn) & 1023)) & 1023;          // SWIZZLE_128B atoms: 1024-byte aligned base
  uint8_t* smem = smem_dyn + pad;
  const uint32_t sbase = smem_u32(smem);
  const int wg = threadIdx.x >> 7, wtid = threadIdx.x & 127;
  const int lane = threadIdx.x & 31, q = lane & 3;
  const int rA = 16 * (wtid >> 5) + (lane >> 2);
  uint8_t* act = smem + wg * C::WG_BYTES;
  const uint32_t abase = sbase + wg * C::WG_BYTES;
  float* s_walpha = reinterpret_cast<float*>(smem + C::OFF_CONST);
  float* s_wrgb = s_walpha + 256;
  const TcRing<C::NSLOT> R{sbase + C::OFF_RING, sbase + C::OFF_BAR};

  if (kView) {
    s_walpha[threadIdx.x] = __ldg(P.w_alpha + threadIdx.x);
    for (int i = threadIdx.x; i < 384; i += C::THREADS) s_wrgb[i] = __ldg(P.w_rgb + i);
  } else {
    for (int i = threadIdx.x; i < 1024; i += C::THREADS) s_walpha[i] = __ldg(P.w_rgb + i);   // w_out [4][256]
  }
  const long long my_tiles = blockIdx.x < P.n_tiles ? (P.n_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
  const uint32_t total = (uint32_t)(my_tiles * SLABS);
  auto fill = [&](uint32_t qq) {
    mbar_arrive_expect_tx(R.full(qq), TC_SLAB_BYTES);
    bulk_g2s(R.slot(qq), P.wimg + (size_t)(qq % SLABS) * TC_SLAB_BYTES, TC_SLAB_BYTES, R.full(qq));
  };
  if (threadIdx.x == 0) R.init(total, fill);
  __syncthreads();
  const float S = __ldg(P.scale);

  float d[128];
  uint32_t qbase = 0;
  for (long long it = 0; it < my_tiles; ++it) {
    const long long row0 = (blockIdx.x + it * gridDim.x) * 128 + wg * TC_WG_ROWS;
    const long long iA = row0 + rA, iB = iA + 8;
    if (wtid == 0) tma_store_wait_read();           // the last step's gradient stores read the A buffer
    wg_sync(wg);
    float daA = 0.f, daB = 0.f;
    if (!kView) {
      // ---- head of a view-independent net: dpre7 -> A buffer and g_pre plane 7 ----
      float4 gA = make_float4(0.f, 0.f, 0.f, 0.f), gB = gA;
      if (iA < P.n) gA = __ldg(reinterpret_cast<const float4*>(P.d_raw) + iA);
      if (iB < P.n) gB = __ldg(reinterpret_cast<const float4*>(P.d_raw) + iB);
      gA.x *= S; gA.y *= S; gA.z *= S; gA.w *= S;
      gB.x *= S; gB.y *= S; gB.z *= S; gB.w *= S;
      uint32_t mA[8], mB[8];
      const uint32_t* m = P.st_m + (size_t)7 * P.n * 8;
      load_signs(m, iA, P.n, mA);
      load_signs(m, iB, P.n, mB);
      bw_head_noview(act, rA, q, s_walpha, gA, gB, mA, mB);
      fence_async_smem();
      wg_sync(wg);
      if (wtid == 0) tma_store_rows(&P.map_pre, abase, 0, 4, row0, 7);
    } else {
      // ---- head: dVpre of row wtid / 2, channels 64 (wtid & 1) .. +63 = A k-block wtid & 1 ----
      {
        const int r = wtid >> 1, h = wtid & 1;
        const long long i = row0 + r;
        float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
        uint4 vm = make_uint4(0, 0, 0, 0);
        if (i < P.n) {
          g = __ldg(reinterpret_cast<const float4*>(P.d_raw) + i);
          vm = __ldg(reinterpret_cast<const uint4*>(P.st_m + ((size_t)8 * P.n + i) * 8));
        }
        const float gx = g.x * S, gy = g.y * S, gz = g.z * S;
        const uint32_t vw[4] = {vm.x, vm.y, vm.z, vm.w};
        uint32_t head[32];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = 8 * h + jj;                   // columns 8j .. 8j+7: word j/4, 16-bit half (j/2)%2
          const uint32_t bits16 = vw[j >> 2] >> (16 * ((j >> 1) & 1));
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int c = 8 * j + 2 * k, pr = 4 * (j & 1) + k;
            float x0 = fmaf(gx, s_wrgb[c], fmaf(gy, s_wrgb[128 + c], gz * s_wrgb[256 + c]));
            float x1 = fmaf(gx, s_wrgb[c + 1], fmaf(gy, s_wrgb[129 + c], gz * s_wrgb[257 + c]));
            if (!((bits16 >> pr) & 1u)) x0 = 0.f;
            if (!((bits16 >> (8 + pr)) & 1u)) x1 = 0.f;
            head[4 * jj + k] = pack_f16x2(x0, x1, false);
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<uint4*>(act + h * TC_KB_BYTES + r * 128 + ((j ^ (r & 7)) << 4)) =
              make_uint4(head[4 * j], head[4 * j + 1], head[4 * j + 2], head[4 * j + 3]);
      }
      fence_async_smem();
      wg_sync(wg);
      if (wtid == 0) tma_store_rows(&P.map_v, abase, 0, 2, row0, 0);   // dL/d(views pre-activation)
      daA = iA < P.n ? S * __ldg(P.d_raw + 4 * iA + 3) : 0.f;
      daB = iB < P.n ? S * __ldg(P.d_raw + 4 * iB + 3) : 0.f;
    }

    for (int b = BW_FIRST(kView); b < BW_STEPS; ++b) {
      const int nkb = bw_nkb(b);
      // masks of this step (plane 8 - b), fetched while the MMAs run
      uint32_t mA[8], mB[8];
      if (b >= 1) {
        const uint32_t* m = P.st_m + (size_t)(8 - b) * P.n * 8;
        load_signs(m, iA, P.n, mA);
        load_signs(m, iB, P.n, mB);
      }
      wgmma_fence();
      for (int kb = 0; kb < nkb; ++kb) {
        const uint32_t qq = qbase + kb;
        R.wait_full(qq);
        const uint64_t a_desc = gmma_desc_k(abase + kb * TC_KB_BYTES), b_desc = gmma_desc_k(R.slot(qq));
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_n256(d, a_desc + 2 * k, b_desc + 2 * k, (kb | k) != 0);
        wgmma_commit();
        if (kb > 0) { wgmma_wait<1>(); R.release(qq - 1, total, fill); }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(d);
      R.release(qbase + nkb - 1, total, fill);
      qbase += nkb;
      if (wtid == 0) tma_store_wait_read();
      wg_sync(wg);
      if (b == 0) bw_epi<false, false>(d, act, rA, q, s_walpha, 0.f, 0.f, mA, mB);
      else if (b == 1) bw_epi<true, true>(d, act, rA, q, s_walpha, daA, daB, mA, mB);
      else bw_epi<false, true>(d, act, rA, q, s_walpha, 0.f, 0.f, mA, mB);
      fence_async_smem();
      wg_sync(wg);
      if (wtid == 0) {
        if (b == 0) tma_store_rows(&P.map_f, abase, 0, 4, row0, 0);
        else tma_store_rows(&P.map_pre, abase, 0, 4, row0, 8 - b);
      }
    }
  }
  if (wtid == 0) tma_store_wait_all();
}

__global__ void __launch_bounds__(BwCfg<true>::THREADS, 1) k_mlp_tc_bwd(const __grid_constant__ BwParams P) {
  mlp_tc_bwd_body<true>(P);
}
// view-independent nets (use_viewdirs=False)
__global__ void __launch_bounds__(BwCfg<false>::THREADS, 1) k_mlp_tc_bwd_noview(const __grid_constant__ BwParams P) {
  mlp_tc_bwd_body<false>(P);
}

// ---------------------------------------------------------------------------------------------
// Packing: transposed weights -> fp16 slabs [N = input channel][K = output channel], 128B-swizzled
// ---------------------------------------------------------------------------------------------
// Sources are the context-owned fp32 copies of the weights in the "Wt[k = input][n = output]" layout (api.cu)
struct BwPackSrc {
  const float* wt[8]; const float* feat_t; const float* views_t;
  int pos_k;                // width of the position encoding that precedes layer 5's hidden input (63, NeRF-T nets 84)
};

// slab k of the image: (step b, k-block kb); element (n = input channel, kk = output channel inside the k-block)
__device__ __forceinline__ float bw_src_weight(const BwPackSrc& S, int b, int n, int kb, int kk) {
  const int out = kb * 64 + kk;
  if (b == 0) return S.views_t[(size_t)n * NM_VIEWS_HID + out];                 // views input = [feature(256), dir PE]
  if (b == 1) return S.feat_t[(size_t)n * 256 + out];
  const int l = 9 - b;                                                          // b = 2..8 -> layer 7..1
  return S.wt[l][(size_t)((l == 5 ? S.pos_k : 0) + n) * 256 + out];            // layer 5 input = [PE(63 / 84), hidden]
}

// view = false: the image of a view-independent net (b2..b8 only) and output_linear's [256][4] -> [4][256]
__global__ void k_bw_pack(BwPackSrc S, uint32_t image_bytes, bool view, __half* __restrict__ out, const float* __restrict__ rgb_t,
                          float* __restrict__ wrgb) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (view && e < 384) wrgb[e] = rgb_t[(e & 127) * 3 + (e >> 7)];      // [128][3] (api.cu layout) -> [3][128]
  if (!view && e < 1024) wrgb[e] = rgb_t[(e & 255) * 4 + (e >> 8)];    // [256][4] -> [4][256]
  if (e * 2 >= image_bytes) return;
  const uint32_t byte = (uint32_t)(e * 2);
  const int k = byte / TC_SLAB_BYTES + (view ? 0 : 2 + 4);   // slab index of the view-dependent image (b2 starts at 6)
  const int b = k < 2 ? 0 : 1 + (k - 2) / 4;
  const int kb = k < 2 ? k : (k - 2) % 4;
  const uint32_t in_slab = byte % TC_SLAB_BYTES;
  const int n = in_slab >> 7;
  const int chunk = ((in_slab & 127) >> 4) ^ (n & 7);
  const int kk = chunk * 8 + ((in_slab & 15) >> 1);
  out[e] = __float2half_rn(bw_src_weight(S, b, n, kb, kk));
}

// ---------------------------------------------------------------------------------------------
// Adjoint of Embedder.forward (models/vanilla.py:82-92): d_x = J^T d_enc with
//   posenc: enc = [x, sin(f_k x), cos(f_k x)]_k          rotate: enc = [x, sin(x B^T), cos(x B^T)]
// One thread per sample; sin/cos recomputed in fp32 exactly as the fp32 forward does (nm_pe_pair).
// d_enc rows are `ld` floats apart and carry a scale whose inverse is *inv_scale (device scalar, may be null).
// ---------------------------------------------------------------------------------------------
__global__ void k_pe_backward(NmPeSpec pe, const float* __restrict__ x, long long group, const float* __restrict__ d_enc,
                              int ld, const float* __restrict__ inv_scale, long long n, float* __restrict__ d_x) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long xi = group > 0 ? i / group : i;
  const float xv[3] = {x[3 * xi], x[3 * xi + 1], x[3 * xi + 2]};
  const float* g = d_enc + (size_t)i * ld;
  float dx[3] = {g[0], g[1], g[2]};
  const int nq = 3 * pe.n_freqs;
  for (int q = 0; q < nq; ++q) {
    float sn, cs;
    int c_sin, c_cos;
    nm_pe_pair(pe, xv, q, sn, cs, c_sin, c_cos);
    const float w = cs * g[c_sin] - sn * g[c_cos];
    if (pe.kind == NM_PE_ROTATE) {
      const float* b = pe.table + 3 * q;
      dx[0] = fmaf(w, b[0], dx[0]); dx[1] = fmaf(w, b[1], dx[1]); dx[2] = fmaf(w, b[2], dx[2]);
    } else {
      const int k = q / 3, d = q - 3 * k;
      dx[d] = fmaf(w, pe.table[k], dx[d]);
    }
  }
  const float sc = inv_scale ? *inv_scale : 1.f;
  d_x[3 * i] = dx[0] * sc; d_x[3 * i + 1] = dx[1] * sc; d_x[3 * i + 2] = dx[2] * sc;
}

int nm_impl_pe_backward(nm_ctx* ctx, const NmNet& net, int which, const float* x, int64_t group, const float* d_enc, int ld,
                        const float* inv_scale, int64_t n, float* d_x, cudaStream_t st) {
  NmPeSpec pe = which == 0 ? NmPeSpec{net.desc.pos_pe_kind, net.desc.pos_n_freqs, net.f32 + net.o_pos_bv}
                           : NmPeSpec{net.desc.dir_pe_kind, net.desc.dir_n_freqs, net.f32 + net.o_dir_bv};
  k_pe_backward<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(pe, x, group, d_enc, ld, inv_scale, n, d_x);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

int nm_tc_pack_bwd(nm_ctx* ctx, NmNet& net, cudaStream_t st) {
  // both buffers depend on the kind of the net: a slot that changed kind gets them at the new sizes
  const bool view = net.kind != NM_NET_NOVIEW;
  const uint32_t image_bytes = (uint32_t)bw_slabs(view) * TC_SLAB_BYTES;
  const size_t wfloats = view ? 384 : 1024;
  if (net.f16_bwd && net.bwd_bytes != image_bytes) {
    NM_CHECK_CUDA(ctx, cudaDeviceSynchronize());
    NM_CHECK_CUDA(ctx, cudaFree(net.f16_bwd));
    net.f16_bwd = nullptr;
  }
  if (net.bw_wrgb && net.bw_wrgb_floats != wfloats) {
    NM_CHECK_CUDA(ctx, cudaDeviceSynchronize());
    NM_CHECK_CUDA(ctx, cudaFree(net.bw_wrgb));
    net.bw_wrgb = nullptr;
  }
  if (!net.f16_bwd) { NM_CHECK_CUDA(ctx, cudaMalloc(&net.f16_bwd, image_bytes)); net.bwd_bytes = image_bytes; }
  if (!net.bw_wrgb) { NM_CHECK_CUDA(ctx, cudaMalloc(&net.bw_wrgb, wfloats * sizeof(float))); net.bw_wrgb_floats = wfloats; }
  BwPackSrc S;
  for (int l = 0; l < 8; ++l) S.wt[l] = net.f32 + net.o_pts_w[l];
  S.feat_t = net.f32 + net.o_feat_w; S.views_t = net.f32 + net.o_views_w;
  S.pos_k = net.f32_pos_k;
  const unsigned blocks = (unsigned)((image_bytes / 2 + 255) / 256);
  k_bw_pack<<<blocks, 256, 0, st>>>(S, image_bytes, view, net.f16_bwd, net.f32 + (view ? net.o_rgb_w : net.o_out_w), net.bw_wrgb);
  NM_CHECK_LAUNCH(ctx);
  net.bwd_packed = true;
  return NM_OK;
}

int nm_tc_backward(nm_ctx* ctx, NmNet& net, const float* d_raw, const float* scale, int64_t n, const __half* st_v,
                   const uint32_t* st_m, __half* g_pre, __half* g_f, __half* g_v, cudaStream_t st) {
  if (!net.bwd_packed) {
    int rc = nm_tc_pack_bwd(ctx, net, st);
    if (rc != NM_OK) return rc;
  }
  BwParams P;
  P.wimg = reinterpret_cast<const uint8_t*>(net.f16_bwd);
  P.d_raw = d_raw; P.scale = scale;
  const bool view = net.kind != NM_NET_NOVIEW;
  P.w_alpha = net.f32 + net.o_alpha_w;
  P.w_rgb = net.bw_wrgb;
  P.st_m = st_m;
  P.n = n;
  P.n_tiles = (n + 127) / 128;
  if (n >= (int64_t)0x7fff0000) NM_FAIL(ctx, NM_ERR_INVALID, "nm_mlp_backward: n too large for one call");
  memset(&P.map_f, 0, 2 * sizeof(CUtensorMap));
  if (tc_make_store_map(&P.map_pre, g_pre, 8, (uint64_t)n, 256) ||
      (view && (tc_make_store_map(&P.map_f, g_f, 1, (uint64_t)n, 256) || tc_make_store_map(&P.map_v, g_v, 1, (uint64_t)n, 128))))
    NM_FAIL(ctx, NM_ERR_CUDA, "nm_mlp_backward: cuTensorMapEncodeTiled failed");
  long long ctas = ctx->sm_count;
  if (P.n_tiles < ctas) ctas = P.n_tiles > 0 ? P.n_tiles : 1;
  if (view) {
    NM_SET_SMEM_ONCE(ctx, k_mlp_tc_bwd, BwCfg<true>::SMEM_BYTES);
    k_mlp_tc_bwd<<<(unsigned)ctas, BwCfg<true>::THREADS, BwCfg<true>::SMEM_BYTES, st>>>(P);
  } else {
    NM_SET_SMEM_ONCE(ctx, k_mlp_tc_bwd_noview, BwCfg<false>::SMEM_BYTES);
    k_mlp_tc_bwd_noview<<<(unsigned)ctas, BwCfg<false>::THREADS, BwCfg<false>::SMEM_BYTES, st>>>(P);
  }
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

// Tensor-core implementation of Joiner.forward (positional encoding + 8x256 NeRF MLP,
// models/vanilla.py:82-92,:120-152,:162-166) for sm_90a: wgmma (fp16 operands, fp32 accumulators in registers),
// weights streamed by bulk-TMA (cp.async.bulk) through a shared-memory ring, activations kept in registers between
// layers, persistent CTAs.
//
// fp16 operands carry the same 11-bit significand as TF32, at twice the tensor rate; accumulation,
// bias, ReLU, the alpha head and the encodings are fp32 (DESIGN.md "Numerics").
//
// Work decomposition
//   tile      = 128 consecutive samples per CTA, 64 per consumer warpgroup (wgmma M = 64).  The two warpgroups
//               share every weight slab; each has its own activations and encodings.
//   step      = one GEMM of the network: 0: L0 (K=64 PE) | 1-4: L1-4 | 5: L5 (PE block + 4 act
//               blocks, "input first", :131) | 6,7: L6,L7 (+alpha head in the epilogue of 7, :135) |
//               8: feature (:136) | 9: views layer (4 feature blocks + dir-PE block, N=128, :137-141) |
//               10: rgb (N=16, 3 used, :143).
//   slab      = one 64-wide K block of one step's weights: [N rows][128 B], 128B-swizzled, K-major -- the GMMA
//               canonical layout, pre-packed in HBM so one cp.async.bulk moves it.  Slabs flow through a
//               TcCfg::NSLOT-deep ring (tc_common.cuh: TcRing): 4 slots, 6 in the view-independent render kernel.
//   epilogue  : accumulator registers -> ReLU -> cvt to f16x2 -> `a`, the A register fragments of the next step's
//               MMAs (the accumulator layout of 16 columns is the A fragment layout of one K = 16 slice).  The
//               training forward writes the swizzled activation block in shared memory instead, the source of the
//               stash's TMA stores.  One step loop for both: a step's k-blocks are the position encoding from shared
//               memory (steps 0 and 5), the activation k-blocks (from `a`, or in training from the activation block),
//               then one from shared memory (bias slab, direction encoding or time slab), in this order in every
//               kernel: the order of the fp32 sums is part of the results.
#include "nm_internal.cuh"
#include "nm_pe.cuh"
#include "tc_common.cuh"
#include <string.h>
// ---------------------------------------------------------------------------------------------
// Plan: which slabs a step consumes, where they live in the packed image.
// ---------------------------------------------------------------------------------------------
#define TC_MAX_SLABS 64
struct TcPlan {
  uint32_t slab_off[TC_STEPS][6];   // byte offset inside the image
  uint32_t slab_bytes[TC_STEPS];    // bytes per slab of this step
  uint32_t image_bytes;             // size of the image
  uint32_t lin_off[TC_MAX_SLABS + 1];   // offset of the j-th slab in consumption order (= image order); [slabs] = image_bytes
};

// Every layer's bias rides in the MMAs.  The last channel of each encoding is the constant 1 (channel 63 of the position
// encoding, 27 of the direction encoding) and the weight column that multiplies it holds the bias (fp16, like every other
// weight): steps 0, 5 and 9 read an encoding block anyway, so there the bias costs nothing.  The K = 256 steps (1-4, 6-8)
// get one extra k-block, a "bias slab" that is zero except for column 63, consumed by ONE K = 16 MMA against the last K
// slice (channels 48..63) of the position encoding: channels 48..62 meet zero weights, channel 63 is 1.  The epilogue then
// has no bias loads and no adds at all; the extra MMA costs 1/16 of a layer's tensor time.
// `v` selects the net kind: true = view-dependent (steps 0-10 above), false = view-independent (use_viewdirs=False,
// models/vanilla.py:145-146): steps 0-7 as above, then step 8 = output_linear (N = 16, 4 used, K = 256 over the layer-7
// activation block, :146); no alpha, feature, views or rgb step, no direction encoding.
// `t` selects a NeRF-T net (view-dependent, position input (x, y, z, t), train.py:254-256): the 21 time channels t, sin(f_k t),
// cos(f_k t) sit in channels 32..52 of the direction-encoding block (the views step reads only its channels 0..31), and steps
// 0 and 5 get one more k-block, a "time slab" (last k-block of the step) consumed by two K = 16 MMAs on K slices 2..3 of that
// block, like the bias slab.
__host__ __device__ constexpr int tc_steps(bool v) { return v ? TC_STEPS : 9; }
__host__ __device__ constexpr int step_nkb(int s, bool v = true, bool t = false) {
  return s == 0 ? (t ? 2 : 1) : (s == 10 ? 2 : (!v && s == 8 ? 4 : (t && s == 5 ? 6 : 5)));
}
__host__ __device__ constexpr bool kb_is_bias(int s, int kb, bool v = true) {
  return kb == 4 && s != 5 && s != 9 && s >= 1 && (v ? s <= 8 : s <= 7);
}
__host__ __device__ constexpr bool kb_is_time(int s, int kb, bool t) { return t && ((s == 0 && kb == 1) || (s == 5 && kb == 5)); }
__host__ __device__ constexpr int step_N(int s, bool v = true) { return s <= 7 || (v && s == 8) ? 256 : (v && s == 9 ? 128 : 16); }
// k-block kb of step s reads the direction encoding
__host__ __device__ constexpr bool kb_is_dir(int s, int kb, bool v = true) { return v && s == 9 && kb == 4; }
__host__ __device__ constexpr int tc_slabs_per_tile(bool v = true, bool t = false) {
  int n = 0;
  for (int s = 0; s < tc_steps(v); ++s) n += step_nkb(s, v, t);
  return n;
}
static_assert(tc_slabs_per_tile(true, true) <= TC_MAX_SLABS && tc_slabs_per_tile(true) <= TC_MAX_SLABS, "slab table too small");

// Shared memory.  The render kernels keep activations in registers only and have no activation blocks, which the
// training forward keeps as the source of its stash stores.  Ring depth: 4 slots, measured 1-2 % faster than 6 in
// k_mlp_tc<false>; 6 in the view-independent render kernel, which spills 32 B with 4 (DESIGN.md §4).
template <bool kTrain, bool kView>
struct TcCfg {
  static constexpr int THREADS = 256;                  // two consumer warpgroups
  static constexpr int NSLOT = kTrain || kView ? 4 : 6;   // depth of the weight ring
  // per warpgroup: [act[4 k-blocks], kTrain only] | position encoding | direction encoding
  static constexpr int OFF_POS = kTrain ? 4 * TC_KB_BYTES : 0;
  static constexpr int OFF_DIR = OFF_POS + TC_KB_BYTES;
  static constexpr int WG_BYTES = OFF_DIR + TC_KB_BYTES;
  static constexpr int OFF_RING = 2 * WG_BYTES;
  static constexpr int OFF_BAR = OFF_RING + NSLOT * TC_SLAB_BYTES;  // full barriers (8 B), then release counters (4 B)
  static constexpr int OFF_CONST = OFF_BAR + 16 * NSLOT;            // the constant table (k_tc_consts), fp32
  static constexpr int SMEM_USED = OFF_CONST + 4 * TC_CONST_FLOATS;
  static constexpr int SMEM_BYTES = SMEM_USED + 1024;               // + alignment slack of the 1024-byte swizzle atoms
};
static_assert(TcCfg<false, false>::SMEM_BYTES <= 232448 && TcCfg<false, true>::SMEM_BYTES <= 232448 &&
              TcCfg<true, false>::SMEM_BYTES <= 232448 && TcCfg<true, true>::SMEM_BYTES <= 232448,
              "shared memory of the forward kernel exceeds 227 KB");

// constant table of the epilogue: [0, 256) alpha_linear.weight | 256..258 rgb bias | 259 alpha bias
// (view-independent nets: [0, 256) unused | 256..259 output_linear.bias)
#define TC_CONST_ALPHA 0
#define TC_CONST_OUT 256

struct TcParams {
  const uint8_t* wimg;      // packed slabs
  TcPlan plan;
  NmMlpInput in;
  NmPeSpec pos_pe, dir_pe;
  float* raw;
  const float* consts;      // device constant table (TC_CONST_FLOATS)
  long long n_tiles;        // number of 128-sample tiles
  int32_t* range_flag;      // device word: bit 0 is set when an activation reached the fp16 range limit (saturated)
  int range_phase;          // sampled range check: the rounds r with r % 64 == range_phase % 64 are checked
  // training forward (kTrain): fp16 activation stash for the backward pass, planes of n rows each
  __half* st_x;             // [8][n][256] post-ReLU outputs of layers 0..7
  __half* st_f;             // [n][256]    feature_linear output (view-dependent nets only)
  __half* st_v;             // [n][128]    views layer post-ReLU (view-dependent nets only)
  uint32_t* st_m;           // [9][n][8]   sign words, 16 bits per 16 columns: bit j = [col 2j > 0], bit 8+j = [col 2j+1 > 0];
                            //             planes 0..7 = pts_linears, plane 8 = views layer (words 0..3 used; view-independent
                            //             nets: [8][n][8], no plane 8)
  CUtensorMap map_x, map_f, map_v;   // TMA store maps of st_x / st_f / st_v (kTrain only)
};

// sin/cos of 2*pi*f (f in cycles).  The operands of the tensor-core path are fp16 (quantisation 2.4e-4 on a
// [-1,1] value), so the encodings only need ~1e-5: range reduction is done exactly in "cycles" with a
// two-float 1/(2*pi) scale (error-free products via fma), then MUFU sin/cos on [-pi, pi] (abs err ~4e-7).
__device__ __forceinline__ void sincos_cycles(float f, float& s, float& c) {
  f = f - rintf(f);
  const float a = f * 6.283185307179586f;
  s = __sinf(a);
  c = __cosf(a);
}

// Encodes x (3) into 64 f16 channels packed as 32 x f16x2; unused channels are zero.
// pe.table for this path: posenc [n_freqs][2] = (hi, lo) of f_k/(2*pi); rotate [3 n_freqs][6] = (hi[3], lo[3])
// of bvals[q]/(2*pi)  (api.cu: pe_cycles_table).
__device__ __forceinline__ void encode_f16(const NmPeSpec& pe, const float x[3], uint32_t (&out)[32], int nq) {
  float ch[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) ch[i] = 0.f;
  ch[0] = x[0]; ch[1] = x[1]; ch[2] = x[2];
  if (pe.kind == NM_PE_ROTATE) {
#pragma unroll
    for (int q = 0; q < 30; ++q) {
      if (q < nq) {
        const float* b = pe.table + 6 * q;
        float frac = 0.f, low = 0.f;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const float bh = __ldg(b + i), bl = __ldg(b + 3 + i);
          const float pr = x[i] * bh;
          low += fmaf(x[i], bl, fmaf(x[i], bh, -pr));        // exact product residual + low part
          frac += pr - rintf(pr);                            // exact
        }
        float s, c;
        sincos_cycles(frac + low, s, c);
        if (nq == 30) { ch[3 + q] = s; ch[33 + q] = c; }
        else { ch[3 + q] = s; ch[15 + q] = c; }
      }
    }
  } else {
#pragma unroll
    for (int k = 0; k < 10; ++k) {
      if (3 * k < nq) {
        const float fh = __ldg(pe.table + 2 * k), fl = __ldg(pe.table + 2 * k + 1);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          const float pr = x[d] * fh;
          const float low = fmaf(x[d], fl, fmaf(x[d], fh, -pr));
          float s, c;
          sincos_cycles((pr - rintf(pr)) + low, s, c);
          ch[3 + 6 * k + d] = s; ch[6 + 6 * k + d] = c;
        }
      }
    }
  }
  ch[nq == 30 ? 63 : 27] = 1.f;          // the constant channel that multiplies the bias column of the weight slabs
#pragma unroll
  for (int i = 0; i < 32; ++i) out[i] = pack_f16x2(ch[2 * i], ch[2 * i + 1], false);
}

// Encodes the time t of a NeRF-T net into channels 32..52 of a direction-encoding row (out[16..26]): channel 32 = t,
// 33 + 2k = sin(f_k t), 34 + 2k = cos(f_k t), with the position encoding's frequencies (posenc table, as encode_f16).
__device__ __forceinline__ void encode_time_f16(const NmPeSpec& pe, float t, uint32_t (&out)[32]) {
  float ch[22];
  ch[0] = t; ch[21] = 0.f;
#pragma unroll
  for (int k = 0; k < 10; ++k) {
    const float fh = __ldg(pe.table + 2 * k), fl = __ldg(pe.table + 2 * k + 1);
    const float pr = t * fh;
    const float low = fmaf(t, fl, fmaf(t, fh, -pr));
    sincos_cycles((pr - rintf(pr)) + low, ch[1 + 2 * k], ch[2 + 2 * k]);
  }
#pragma unroll
  for (int i = 0; i < 11; ++i) out[16 + i] = pack_f16x2(ch[2 * i], ch[2 * i + 1], false);
}

// write 8 * nchunks f16 of one 128-byte row of a K block with the 128B swizzle
__device__ __forceinline__ void store_row_swizzled(uint8_t* blk, int row, const uint32_t* v, int nchunks) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (j < nchunks) {
      uint4 q = make_uint4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
      *reinterpret_cast<uint4*>(blk + row * 128 + ((j ^ (row & 7)) << 4)) = q;
    }
  }
}

template <bool RELU>
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  uint32_t d;
  if (RELU) asm("cvt.rn.satfinite.relu.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  else asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}

// running maximum of |activation| as packed halves (range flag)
template <bool RELU>
__device__ __forceinline__ void track_range(uint32_t& rng, uint32_t packed) {
  __half2 h = *reinterpret_cast<const __half2*>(&packed);
  if (!RELU) h = __habs2(h);
  const __half2 m = __hmax2(*reinterpret_cast<const __half2*>(&rng), h);
  rng = *reinterpret_cast<const uint32_t*>(&m);
}

// ---------------------------------------------------------------------------------------------
// Epilogue of NC accumulator columns of this thread's two rows rA, rA + 8 (columns 8j + 2q, +1: tc_common.cuh):
// the alpha head on step 7 (fp32 FFMAs on the ReLU of the unrounded accumulators), ReLU, saturating f16x2 pack into
// the next step's A operand: `a`, its register fragments (a[2j] / a[2j + 1]: rows rA / rA + 8 of columns 8j + 2q, +1;
// K slice k of the next step reads a[4k..4k+3]), or with SMEM swizzled 4-byte stores into the activation block, and the ReLU sign words
// (word w = columns 32w..32w+31; bits 0-7 / 8-15: even / odd columns of the first 16, bits 16-31 the same for the
// next 16) as this thread's share, OR-reduced over the quad afterwards.
// ---------------------------------------------------------------------------------------------
template <int NC, bool RELU, bool ALPHA, bool SIGNS, bool SMEM>
__device__ __forceinline__ void fwd_epi(const float (&d)[128], uint32_t (&a)[64], uint8_t* act, int rA, int q,
                                        const float* s_walpha, float (&alpha)[2], uint32_t (&wA)[8], uint32_t (&wB)[8],
                                        bool track, uint32_t& rng) {
  const int rB = rA + 8;
#pragma unroll
  for (int j = 0; j < NC / 8; ++j) {
    const int c = 8 * j + 2 * q;
    const float x0 = d[4 * j], x1 = d[4 * j + 1], y0 = d[4 * j + 2], y1 = d[4 * j + 3];
    if (ALPHA) {                                // alpha_linear on the fp32 ReLU output (:135)
      const float2 w = *reinterpret_cast<const float2*>(s_walpha + c);
      alpha[0] = fmaf(fmaxf(x0, 0.f), w.x, fmaf(fmaxf(x1, 0.f), w.y, alpha[0]));
      alpha[1] = fmaf(fmaxf(y0, 0.f), w.x, fmaf(fmaxf(y1, 0.f), w.y, alpha[1]));
    }
    const uint32_t pA = pack2<RELU>(x0, x1), pB = pack2<RELU>(y0, y1);
    if (SMEM) {
      uint8_t* blk = act + (j >> 3) * TC_KB_BYTES;
      *reinterpret_cast<uint32_t*>(blk + swz_off(rA, c)) = pA;
      *reinterpret_cast<uint32_t*>(blk + swz_off(rB, c)) = pB;
    } else {
      a[2 * j] = pA;
      a[2 * j + 1] = pB;
    }
    if (track) { track_range<RELU>(rng, pA); track_range<RELU>(rng, pB); }
    if (SIGNS) {
      const __half2 zero2 = __float2half2_rn(0.f);
      const uint32_t mA = __hgt2_mask(*reinterpret_cast<const __half2*>(&pA), zero2);
      const uint32_t mB = __hgt2_mask(*reinterpret_cast<const __half2*>(&pB), zero2);
      const int bit = 16 * ((j >> 1) & 1) + 4 * (j & 1) + q;
      wA[j >> 2] |= ((mA & 1u) << bit) | ((mA >> 16 & 1u) << (bit + 8));
      wB[j >> 2] |= ((mB & 1u) << bit) | ((mB >> 16 & 1u) << (bit + 8));
    }
  }
}

// OR of the sign words over the four threads of a quad (they hold the same rows, different columns)
__device__ __forceinline__ void quad_or(uint32_t (&w)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    w[i] |= __shfl_xor_sync(0xffffffffu, w[i], 1);
    w[i] |= __shfl_xor_sync(0xffffffffu, w[i], 2);
  }
}

// ---------------------------------------------------------------------------------------------
// The kernel body, shared by the view-dependent (kView) and view-independent nets: same tile loop, same ring, same steps 0-7
// ---------------------------------------------------------------------------------------------
template <bool kTrain, bool kView, bool kTime = false>
__device__ __forceinline__ void mlp_tc_body(const TcParams& P) {
  static_assert(!kTime || kView, "NeRF-T nets are view-dependent");
  using C = TcCfg<kTrain, kView>;
  constexpr int SLABS = tc_slabs_per_tile(kView, kTime);
  constexpr int STEPS = tc_steps(kView);
  constexpr int LAST = STEPS - 1;                       // the output step: rgb (N = 16) or output_linear (N = 16)
  extern __shared__ uint8_t smem_dyn[];
  const uint32_t pad = (1024 - (smem_u32(smem_dyn) & 1023)) & 1023;     // SWIZZLE_128B atoms: 1024-byte aligned base
  uint8_t* smem = smem_dyn + pad;
  const uint32_t sbase = smem_u32(smem);
  const int wg = threadIdx.x >> 7, wtid = threadIdx.x & 127;
  const int lane = threadIdx.x & 31, q = lane & 3;
  const int rA = 16 * (wtid >> 5) + (lane >> 2);        // first of this thread's two accumulator rows (rA, rA + 8)
  uint8_t* wbuf = smem + wg * C::WG_BYTES;
  const uint32_t wbase = sbase + wg * C::WG_BYTES;
  float* s_const = reinterpret_cast<float*>(smem + C::OFF_CONST);
  const TcRing<C::NSLOT> R{sbase + C::OFF_RING, sbase + C::OFF_BAR};

  for (int i = threadIdx.x; i < TC_CONST_FLOATS; i += C::THREADS) s_const[i] = __ldg(P.consts + i);
  const long long my_tiles = blockIdx.x < P.n_tiles ? (P.n_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
  const uint32_t total = (uint32_t)(my_tiles * SLABS);
  auto fill = [&](uint32_t qq) {                        // the slab of fill qq, in consumption order
    const uint32_t j = qq % SLABS, off = P.plan.lin_off[j], bytes = P.plan.lin_off[j + 1] - off;
    mbar_arrive_expect_tx(R.full(qq), bytes);
    bulk_g2s(R.slot(qq), P.wimg + off, bytes, R.full(qq));
  };
  if (threadIdx.x == 0) R.init(total, fill);
  __syncthreads();

  const float4 ob = *reinterpret_cast<const float4*>(s_const + TC_CONST_OUT);
  float d[128];
  float d16[8];
  uint32_t a[64];                                       // the previous step's output: A fragments of 16 K slices
  uint32_t rng = 0;
  uint32_t qbase = 0;
  const long long rperiod = my_tiles < 64 ? my_tiles : 64;
  for (long long it = 0; it < my_tiles; ++it) {
    const long long tile = blockIdx.x + it * gridDim.x;
    const long long row0 = tile * 128 + wg * TC_WG_ROWS;          // first sample of this warpgroup
    // view-independent nets check every tile: with the sampled (data-dependent) check ptxas serialises the wgmma of their
    // training variant (C7520); the epilogue has the ALU time to spare without the alpha head
    const bool track = !kView || (it % rperiod) == (P.range_phase % rperiod);
    // ---- encodings (Embedder.forward, models/vanilla.py:82-92): threads 0-63 position, 64-127 direction of row wtid % 64 ----
    {
      // Ray / view row of sample row0 + r: one 64-bit division per tile, then a 32-bit one per thread.  A per-thread
      // 64-bit division compiles to a call on a path that depends on the thread's operands; with such a call in the
      // tile loop ptxas serialises every wgmma of the kernel (warning C7520; tests/test_tc_sass.py).
      const int r = wtid & 63;
      const int group = P.in.group;
      long long g0 = 0;
      uint32_t g0r = 0;
      if (group > 0) { g0 = tile * 128 / group; g0r = (uint32_t)(tile * 128 - g0 * group); }
      const uint32_t off = wg * TC_WG_ROWS + r;            // row0 + r - tile * 128
      const long long g = group > 0 ? g0 + (g0r + off) / (uint32_t)group : row0 + r;
      float p[3] = {0.f, 0.f, 0.f}, v[3] = {0.f, 0.f, 0.f};
      float t = 0.f;
      if (row0 + r < P.in.n) {
        nm_fetch_sample_at<kTime ? 4 : 3>(P.in, row0 + r, g, p, v);
        if (kTime) t = nm_fetch_time(P.in, row0 + r);
      }
      // rendering: the previous tile's last MMAs on the encoding blocks (the bias slab of step 8 / 7, the direction
      // k-block of step 9) must have retired in all four warps before the blocks are overwritten (in the training
      // forward the barrier before the epilogue of step 9 / 7 orders them)
      if (!kTrain && it > 0) wg_sync(wg);
      uint32_t e[32];
      if (wtid < 64) {
        encode_f16(P.pos_pe, p, e, 30);
        store_row_swizzled(wbuf + C::OFF_POS, r, e, 8);
      } else if (kView) {
        encode_f16(P.dir_pe, v, e, 12);
        if (kTime) encode_time_f16(P.pos_pe, t, e);
        store_row_swizzled(wbuf + C::OFF_DIR, r, e, kTime ? 8 : 4);
      }
      if (track && (kView || wtid < 64)) { track_range<false>(rng, e[0]); track_range<false>(rng, e[1]); }   // raw x, y, z (+ one sine)
      if (kTime && track && wtid >= 64) track_range<false>(rng, e[16]);                                       // t, sin(f_0 t)
      fence_async_smem();
      wg_sync(wg);
    }
    float alpha[2] = {0.f, 0.f};
    // rendering: unrolled, so each step's k-blocks and epilogue touch a fixed part of `a` and only that part is live (the
    // training kernels do not hold `a`: the unrolled loop makes them spill)
#pragma unroll (kTrain ? 1 : STEPS)
    for (int s = 0; s < STEPS; ++s) {
      const int nkb = step_nkb(s, kView, kTime);
      const bool wide = s <= (kView ? 8 : 7), views = kView && s == 9;     // N = 256 / 128 (views) / 16 (output)
      wgmma_fence();
      int kb = 0;
      // one k-block: wait for its slab, issue its MMAs (`issue(b_desc, first k-block of the step)`), commit, and
      // release the previous k-block's slab once its MMAs have retired
      auto kblock = [&](auto&& issue) {
        const uint32_t qq = qbase + kb;
        R.wait_full(qq);
        issue(gmma_desc_k(R.slot(qq)), kb == 0);
        wgmma_commit();
        if (kb > 0) { wgmma_wait<1>(); R.release(qq - 1, total, fill); }
        ++kb;
      };
      // a k-block whose A operand is a block in shared memory, K slices k0..k1-1.  K advances by 32 B (= 2 in descriptor
      // address units) inside the 128-byte swizzle atom.
      auto smem_kblock = [&](uint32_t a_addr, int k0, int k1) {
        kblock([&](uint64_t b_desc, bool first) {
          const uint64_t a_desc = gmma_desc_k(a_addr);
          for (int k = k0; k < k1; ++k) {
            const uint32_t acc = !first || k > k0;
            if (wide) wgmma_n256(d, a_desc + 2 * k, b_desc + 2 * k, acc);
            else if (views) wgmma_n128(d, a_desc + 2 * k, b_desc + 2 * k, acc);
            else wgmma_n16(d16, a_desc + 2 * k, b_desc + 2 * k, acc);
          }
        });
      };
      if (s == 0 || s == 5) smem_kblock(wbase + C::OFF_POS, 0, 4);       // position encoding (step 5: "input first", :131)
      if (s > 0) {
        const int nact = kView && s == LAST ? 2 : 4;                      // rgb reads the 128 columns of the views layer
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (j < nact) {
            // training: the activation block in shared memory (the source of the stash's stores); rendering: `a`
            if constexpr (kTrain) smem_kblock(wbase + j * TC_KB_BYTES, 0, 4);
            else kblock([&](uint64_t b_desc, bool first) {
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const uint32_t* f = a + 16 * j + 4 * k;
                const uint32_t acc = !first || k > 0;
                if (wide) wgmma_n256_rs(d, f[0], f[1], f[2], f[3], b_desc + 2 * k, acc);
                else if (views) wgmma_n128_rs(d, f[0], f[1], f[2], f[3], b_desc + 2 * k, acc);
                else wgmma_n16_rs(d16, f[0], f[1], f[2], f[3], b_desc + 2 * k, acc);
              }
            });
          }
        }
      }
      // the trailing k-block: a bias slab is one K = 16 MMA on the last K slice (channels 48..63 of the position
      // encoding x columns 48..63 of the slab), the direction encoding two on K slices 0..1, a time slab two on K
      // slices 2..3 (channels 32..63 of the direction block)
      if (kb < nkb) {
        if (kb_is_bias(s, kb, kView)) smem_kblock(wbase + C::OFF_POS, 3, 4);
        else if (kb_is_dir(s, kb, kView)) smem_kblock(wbase + C::OFF_DIR, 0, 2);
        else smem_kblock(wbase + C::OFF_DIR, 2, 4);
      }
      wgmma_wait<0>();
      wgmma_fence_regs(d);
      wgmma_fence_regs(d16);
      R.release(qbase + nkb - 1, total, fill);
      qbase += nkb;
      if (s < LAST) {
        // training forward: the MMAs of this step read the activation blocks, the stash stores of the previous step
        // still may: both must be done before the epilogue overwrites them
        if (kTrain) {
          if (wtid == 0) tma_store_wait_read();
          wg_sync(wg);
        }
        uint32_t wA[8] = {0, 0, 0, 0, 0, 0, 0, 0}, wB[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const float* s_walpha = s_const + TC_CONST_ALPHA;
        if (s == 7) fwd_epi<256, true, kView, kTrain, kTrain>(d, a, wbuf, rA, q, s_walpha, alpha, wA, wB, track, rng);
        else if (kView && s == 8) fwd_epi<256, false, false, false, kTrain>(d, a, wbuf, rA, q, s_walpha, alpha, wA, wB, track, rng);
        else if (s == 9) fwd_epi<128, true, false, kTrain, kTrain>(d, a, wbuf, rA, q, s_walpha, alpha, wA, wB, track, rng);
        else fwd_epi<256, true, false, kTrain, kTrain>(d, a, wbuf, rA, q, s_walpha, alpha, wA, wB, track, rng);
        if (kTrain) {
          fence_async_smem();
          wg_sync(wg);
          if (wtid == 0) {
            if (!kView || s < 8) tma_store_rows(&P.map_x, wbase, 0, 4, row0, s);
            else if (s == 8) tma_store_rows(&P.map_f, wbase, 0, 4, row0, 0);
            else tma_store_rows(&P.map_v, wbase, 0, 2, row0, 0);
          }
          if (!kView || s != 8) {
            quad_or(wA);
            quad_or(wB);
            const long long iA = row0 + rA, iB = iA + 8;
            if (!kView || s < 8) {
              uint32_t* m = P.st_m + (size_t)s * P.in.n * 8;
              if (iA < P.in.n) reinterpret_cast<uint2*>(m + iA * 8)[q] = make_uint2(wA[2 * q], wA[2 * q + 1]);
              if (iB < P.in.n) reinterpret_cast<uint2*>(m + iB * 8)[q] = make_uint2(wB[2 * q], wB[2 * q + 1]);
            } else {
              uint32_t* m = P.st_m + (size_t)8 * P.in.n * 8;
              if (iA < P.in.n) m[iA * 8 + q] = wA[q];
              if (iB < P.in.n) m[iB * 8 + q] = wB[q];
            }
          }
        }
        if (kView && s == 7) {
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            alpha[r] += __shfl_xor_sync(0xffffffffu, alpha[r], 1);
            alpha[r] += __shfl_xor_sync(0xffffffffu, alpha[r], 2);
          }
        }
      } else if (kView) {
        // rgb (columns 0..2: lane q = 0 holds 0, 1; lane q = 1 holds 2) and the alpha head -> raw [r, g, b, sigma] (:144)
        const float bA = __shfl_down_sync(0xffffffffu, d16[0], 1), bB = __shfl_down_sync(0xffffffffu, d16[2], 1);
        const long long iA = row0 + rA, iB = iA + 8;
        if (q == 0 && iA < P.in.n)
          reinterpret_cast<float4*>(P.raw)[iA] = make_float4(d16[0] + ob.x, d16[1] + ob.y, bA + ob.z, alpha[0] + ob.w);
        if (q == 0 && iB < P.in.n)
          reinterpret_cast<float4*>(P.raw)[iB] = make_float4(d16[2] + ob.x, d16[3] + ob.y, bB + ob.z, alpha[1] + ob.w);
      } else {
        // output_linear (:146): columns 0..3 = raw [r, g, b, sigma]; lane q = 0 holds 0, 1, lane q = 1 holds 2, 3
        const float cA = __shfl_down_sync(0xffffffffu, d16[0], 1), dA = __shfl_down_sync(0xffffffffu, d16[1], 1);
        const float cB = __shfl_down_sync(0xffffffffu, d16[2], 1), dB = __shfl_down_sync(0xffffffffu, d16[3], 1);
        const long long iA = row0 + rA, iB = iA + 8;
        if (q == 0 && iA < P.in.n)
          reinterpret_cast<float4*>(P.raw)[iA] = make_float4(d16[0] + ob.x, d16[1] + ob.y, cA + ob.z, dA + ob.w);
        if (q == 0 && iB < P.in.n)
          reinterpret_cast<float4*>(P.raw)[iB] = make_float4(d16[2] + ob.x, d16[3] + ob.y, cB + ob.z, dB + ob.w);
      }
    }
  }
  if (((rng & 0xFFFFu) >= 0x7BFFu) || ((rng >> 16) >= 0x7BFFu)) atomicOr(P.range_flag, 1);
  if (kTrain && wtid == 0) tma_store_wait_all();
}

// view-dependent nets (use_viewdirs=True): render (kTrain = false) and training forward
template <bool kTrain>
__global__ void __launch_bounds__(TcCfg<kTrain, true>::THREADS, 1) k_mlp_tc(const __grid_constant__ TcParams P) {
  mlp_tc_body<kTrain, true>(P);
}
// view-independent nets (use_viewdirs=False): no direction input, output_linear head
template <bool kTrain>
__global__ void __launch_bounds__(TcCfg<kTrain, false>::THREADS, 1) k_mlp_tc_noview(const __grid_constant__ TcParams P) {
  mlp_tc_body<kTrain, false>(P);
}
// NeRF-T nets (view-dependent, position input (x, y, z, t)): render (kTrain = false) and training forward
template <bool kTrain>
__global__ void __launch_bounds__(TcCfg<kTrain, true>::THREADS, 1) k_mlp_tc_nerft(const __grid_constant__ TcParams P) {
  mlp_tc_body<kTrain, true, true>(P);
}

// ---------------------------------------------------------------------------------------------
// Packing: fp32 nn.Linear weights -> fp16 slabs in the swizzled GMMA layout.
// ---------------------------------------------------------------------------------------------
struct PackSrc {
  const float* w[8]; const float* feat; const float* views; const float* rgb;
  const float* b[8]; const float* feat_b; const float* views_b;      // biases: they ride in the slabs (column of the constant-1 channel)
  const float* out_t;                                                 // output_linear.weight as [256][4] (view-independent nets)
};

// Column of a NeRF-T net's 84-wide encoding (the reference's order [x, y, z, t, sin(f_0 xyzt), cos(f_0 xyzt), ...],
// models/vanilla.py:69-75 with input_dims = 4) that feeds channel kk of the kernel's position block (kk < 63: x, y, z, then
// sin / cos of x, y, z per frequency as encode_f16 lays them out) or of its time channels (time = true, kk in 32..52);
// -1 for a channel no column feeds.
__device__ __forceinline__ int nerft_col(int kk, bool time) {
  if (time) {
    if (kk == 32) return 3;
    if (kk < 33 || kk > 52) return -1;
    const int k = (kk - 33) >> 1;
    return ((kk - 33) & 1) ? 11 + 8 * k : 7 + 8 * k;
  }
  if (kk < 3) return kk;
  const int i = kk - 3, k = i / 6, r = i - 6 * k;
  return r < 3 ? 4 + 8 * k + r : 8 + 8 * k + (r - 3);
}

// weight of (step s, output n, k-block kb, kk in [0,64)) or 0 for padding; `view`, `time` = the net kind (step tables above)
__device__ __forceinline__ float src_weight(const PackSrc& S, int s, int n, int kb, int kk, bool view, bool time) {
  if (!view && s == 8) return n < 4 ? S.out_t[(size_t)(kb * 64 + kk) * 4 + n] : 0.f;   // output_linear, N padded 4 -> 16
  if (kb_is_bias(s, kb, view)) {                 // bias slab of a K = 256 step: only the column of PE channel 63 is non-zero
    if (kk != 63) return 0.f;
    return s == 8 ? S.feat_b[n] : S.b[s][n];
  }
  if (time && (s == 0 || s == 5)) {              // pts_linears.0 [256,84] / .5 [256,340]: columns in the reference's order
    const int ld = s == 0 ? NM_POS_PE_T : NM_POS_PE_T + 256;
    const float* w = S.w[s] + (size_t)n * ld;
    if (kb_is_time(s, kb, true)) {
      const int c = nerft_col(kk, true);
      return c < 0 ? 0.f : w[c];
    }
    if (kb == 0) return kk < NM_POS_PE ? w[nerft_col(kk, false)] : S.b[s][n];                 // kk == 63: bias
    return w[NM_POS_PE_T + (kb - 1) * 64 + kk];
  }
  if (s == 0) return kk < NM_POS_PE ? S.w[0][(size_t)n * NM_POS_PE + kk] : S.b[0][n];           // kk == 63: bias
  if (s >= 1 && s <= 7 && s != 5) return S.w[s][(size_t)n * 256 + kb * 64 + kk];
  if (s == 5) {
    const int ld = NM_POS_PE + 256;
    if (kb == 0) return kk < NM_POS_PE ? S.w[5][(size_t)n * ld + kk] : S.b[5][n];
    return S.w[5][(size_t)n * ld + NM_POS_PE + (kb - 1) * 64 + kk];
  }
  if (s == 8) return S.feat[(size_t)n * 256 + kb * 64 + kk];
  if (s == 9) {
    const int ld = 256 + NM_DIR_PE;
    if (kb < 4) return S.views[(size_t)n * ld + kb * 64 + kk];
    return kk < NM_DIR_PE ? S.views[(size_t)n * ld + 256 + kk] : (kk == NM_DIR_PE ? S.views_b[n] : 0.f);    // kk == 27: bias
  }
  // s == 10: rgb, N padded 3 -> 16 (its bias is added with the alpha bias when the output is written)
  return n < 3 ? S.rgb[(size_t)n * 128 + kb * 64 + kk] : 0.f;
}

__global__ void k_tc_pack(PackSrc S, TcPlan plan, bool view, bool time, __half* __restrict__ out) {
  // one thread per packed element of the image
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;      // half index inside the image
  if (e * 2 >= plan.image_bytes) return;
  const uint32_t byte = (uint32_t)(e * 2);
  // locate (s, kb)
  int s = 0, kb = 0;
  for (int ss = 0; ss < tc_steps(view); ++ss)
    for (int k = 0; k < step_nkb(ss, view, time); ++k)
      if (byte >= plan.slab_off[ss][k]) { s = ss; kb = k; }
  const uint32_t in_slab = byte - plan.slab_off[s][kb];
  const int n = in_slab >> 7;
  const int chunk_phys = (in_slab & 127) >> 4;
  const int chunk = chunk_phys ^ (n & 7);                               // undo the 128B swizzle
  const int kk = chunk * 8 + ((in_slab & 15) >> 1);
  out[e] = __float2half_rn(src_weight(S, s, n, kb, kk, view, time));
}

// the constant table of the epilogue (layout: TC_CONST_ALPHA / TC_CONST_OUT)
__global__ void k_tc_consts(const float* rgb_b, const float* alpha_w, const float* alpha_b, float* __restrict__ out) {
  const int i = threadIdx.x;      // 256 threads
  out[TC_CONST_ALPHA + i] = alpha_w[i];
  if (i < TC_CONST_FLOATS - TC_CONST_OUT) out[TC_CONST_OUT + i] = i < 3 ? rgb_b[i] : (i == 3 ? alpha_b[0] : 0.f);
}
// ... of a view-independent net: no alpha weights, output_linear.bias at TC_CONST_OUT
__global__ void k_tc_consts_noview(const float* out_b, float* __restrict__ out) {
  const int i = threadIdx.x;      // 256 threads
  out[TC_CONST_ALPHA + i] = 0.f;
  if (i < TC_CONST_FLOATS - TC_CONST_OUT) out[TC_CONST_OUT + i] = i < 4 ? out_b[i] : 0.f;
}

// ---------------------------------------------------------------------------------------------
// The encodings as the tensor-core kernel feeds them to the MMAs (same code, same fp16 values), written out as
// planes for the weight-gradient GEMMs of the training step: [n][64] (position, channel 63 = 1.0) or [n][32]
// (direction, channel 27 = 1.0).  The constant channel multiplies a zero weight in the forward and returns the bias
// gradient as an extra column of  g^T @ plane.  One thread per sample; 10-20 us per step, cheaper than stashing the
// encodings from inside the MLP kernel (per-thread 128-byte rows from the epilogue warps: ~10 % of that kernel).
// ---------------------------------------------------------------------------------------------
__global__ void k_encode_f16(NmPeSpec pe, int which, const float* __restrict__ x, long long group, long long n,
                             __half* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long xi = group > 0 ? i / group : i;
  const float xv[3] = {x[3 * xi], x[3 * xi + 1], x[3 * xi + 2]};
  uint32_t e[32];
  encode_f16(pe, xv, e, which == 0 ? 30 : 12);
  if (which == 0) {
    e[31] |= 0x3C000000u;                                                  // channel 63 := 1.0
    uint4* dst = reinterpret_cast<uint4*>(out + (size_t)i * 64);
#pragma unroll
    for (int j = 0; j < 8; ++j) dst[j] = make_uint4(e[4 * j], e[4 * j + 1], e[4 * j + 2], e[4 * j + 3]);
  } else {
    e[13] |= 0x3C000000u;                                                  // channel 27 := 1.0
    uint4* dst = reinterpret_cast<uint4*>(out + (size_t)i * 32);
#pragma unroll
    for (int j = 0; j < 4; ++j) dst[j] = make_uint4(e[4 * j], e[4 * j + 1], e[4 * j + 2], e[4 * j + 3]);
  }
}

// The position encoding of a NeRF-T net as the forward kernel feeds it to the MMAs (the same fp16 values: encode_f16 /
// encode_time_f16 arithmetic), laid out in the reference's column order [x, y, z, t, sin(f_0 xyzt), cos(f_0 xyzt), ...]
// (84 channels), then 1.0 at channel 84 and zeros to 95: [n][96].  g^T @ plane gives pts_linears.0's weight gradient in
// the reference's layout and its bias gradient as column 84, so the kernel's channel permutation stays in this file.
__global__ void k_encode_f16_nerft(NmPeSpec pe, const float* __restrict__ x, long long group, long long n,
                                   __half* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long xi = group > 0 ? i / group : i;
  float ch[96];
#pragma unroll
  for (int c = 0; c < 96; ++c) ch[c] = 0.f;
#pragma unroll
  for (int d = 0; d < 4; ++d) ch[d] = x[4 * xi + d];
#pragma unroll
  for (int k = 0; k < 10; ++k) {
    const float fh = __ldg(pe.table + 2 * k), fl = __ldg(pe.table + 2 * k + 1);
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      const float v = ch[d];
      const float pr = v * fh;
      const float low = fmaf(v, fl, fmaf(v, fh, -pr));
      sincos_cycles((pr - rintf(pr)) + low, ch[4 + 8 * k + d], ch[8 + 8 * k + d]);
    }
  }
  ch[NM_POS_PE_T] = 1.f;
  uint4* dst = reinterpret_cast<uint4*>(out + (size_t)i * 96);
#pragma unroll
  for (int j = 0; j < 12; ++j)
    dst[j] = make_uint4(pack_f16x2(ch[8 * j], ch[8 * j + 1], false), pack_f16x2(ch[8 * j + 2], ch[8 * j + 3], false),
                        pack_f16x2(ch[8 * j + 4], ch[8 * j + 5], false), pack_f16x2(ch[8 * j + 6], ch[8 * j + 7], false));
}

int nm_tc_encode(nm_ctx* ctx, const NmNet& net, int which, const float* x, int64_t group, int64_t n, __half* out, cudaStream_t st) {
  NmPeSpec pe = which == 0 ? NmPeSpec{net.desc.pos_pe_kind, net.desc.pos_n_freqs, net.f32 + net.o_pos_cyc}
                           : NmPeSpec{net.desc.dir_pe_kind, net.desc.dir_n_freqs, net.f32 + net.o_dir_cyc};
  if (which == 0 && net.kind == NM_NET_NERFT)
    k_encode_f16_nerft<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(pe, x, group, n, out);
  else
    k_encode_f16<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(pe, which, x, group, n, out);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

static TcPlan make_plan(bool view, bool time) {
  TcPlan p{};
  uint32_t off = 0;
  int j = 0;
  for (int s = 0; s < tc_steps(view); ++s) {
    p.slab_bytes[s] = (uint32_t)step_N(s, view) * 128u;
    for (int kb = 0; kb < step_nkb(s, view, time); ++kb) {
      p.slab_off[s][kb] = p.lin_off[j++] = off;
      off += p.slab_bytes[s];
    }
  }
  p.lin_off[j] = p.image_bytes = off;
  return p;
}

int nm_tc_pack(nm_ctx* ctx, NmNet& net, cudaStream_t st) {
  const bool view = net.kind != NM_NET_NOVIEW, time = net.kind == NM_NET_NERFT;
  TcPlan plan = make_plan(view, time);
  const size_t halfs = plan.image_bytes / 2;
  if (!net.f16 || net.f16_halfs != halfs) {
    if (net.f16) { NM_CHECK_CUDA(ctx, cudaDeviceSynchronize()); NM_CHECK_CUDA(ctx, cudaFree(net.f16)); net.f16 = nullptr; }
    NM_CHECK_CUDA(ctx, cudaMalloc(&net.f16, halfs * sizeof(__half)));
    net.f16_halfs = halfs;
  }
  if (!net.tc_bias) NM_CHECK_CUDA(ctx, cudaMalloc(&net.tc_bias, TC_CONST_FLOATS * sizeof(float)));
  const nm_nerf_desc& d = net.desc;
  PackSrc S;
  for (int l = 0; l < 8; ++l) S.w[l] = d.pts_w[l];
  S.feat = d.feature_w; S.views = d.views_w; S.rgb = d.rgb_w;
  for (int l = 0; l < 8; ++l) S.b[l] = d.pts_b[l];
  S.feat_b = d.feature_b; S.views_b = d.views_b;
  S.out_t = net.f32 + net.o_out_w;
  k_tc_pack<<<(unsigned)((halfs + 255) / 256), 256, 0, st>>>(S, plan, view, time, net.f16);
  NM_CHECK_LAUNCH(ctx);
  if (view) k_tc_consts<<<1, 256, 0, st>>>(d.rgb_b, d.alpha_w, d.alpha_b, net.tc_bias);
  else k_tc_consts_noview<<<1, 256, 0, st>>>(net.f32 + net.o_out_b, net.tc_bias);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

template <bool kTrain, bool kView, bool kTime = false>
static int launch_tc(nm_ctx* ctx, const TcParams& P, cudaStream_t st) {
  void (*kernel)(const TcParams);
  if constexpr (kTime) kernel = k_mlp_tc_nerft<kTrain>;
  else kernel = kView ? k_mlp_tc<kTrain> : k_mlp_tc_noview<kTrain>;
  using C = TcCfg<kTrain, kView>;
  NM_SET_SMEM_ONCE(ctx, kernel, C::SMEM_BYTES);
  long long ctas = ctx->sm_count;
  if (P.n_tiles < ctas) ctas = P.n_tiles > 0 ? P.n_tiles : 1;
  kernel<<<(unsigned)ctas, C::THREADS, C::SMEM_BYTES, st>>>(P);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

int nm_tc_forward(nm_ctx* ctx, NmNet& net, const float* pts, const float* views, const float* origins,
                  const float* dirs, const float* z, int64_t n, int32_t group, float t, float* raw, cudaStream_t st,
                  const NmTrainStash* stash) {
  if (!net.f16 || !net.tc_bias) NM_FAIL(ctx, NM_ERR_STATE, "nm_tc_forward: weights not packed");
  const bool view = net.kind != NM_NET_NOVIEW, time = net.kind == NM_NET_NERFT;
  TcParams P;
  P.wimg = reinterpret_cast<const uint8_t*>(net.f16);
  P.plan = make_plan(view, time);
  P.in = NmMlpInput{pts, views, origins, dirs, z, (long long)n, group, t};
  P.pos_pe = NmPeSpec{net.desc.pos_pe_kind, net.desc.pos_n_freqs, net.f32 + net.o_pos_cyc};
  P.dir_pe = NmPeSpec{net.desc.dir_pe_kind, net.desc.dir_n_freqs, net.f32 + net.o_dir_cyc};
  P.raw = raw;
  P.consts = net.tc_bias;
  P.n_tiles = (n + 127) / 128;
  P.range_flag = ctx->d_counter + NM_RANGE_FLAG_WORD;
  P.range_phase = (int)(ctx->range_seq++ % 64);
  P.st_x = stash ? stash->x : nullptr; P.st_f = stash ? stash->f : nullptr; P.st_v = stash ? stash->v : nullptr;
  P.st_m = stash ? stash->m : nullptr;
  memset(&P.map_x, 0, 3 * sizeof(CUtensorMap));
  if (stash) {
    if (n >= (int64_t)0x7fff0000) NM_FAIL(ctx, NM_ERR_INVALID, "nm_mlp_forward_train: n too large for one call");
    if (tc_make_store_map(&P.map_x, stash->x, 8, (uint64_t)n, 256) ||
        (view && (tc_make_store_map(&P.map_f, stash->f, 1, (uint64_t)n, 256) || tc_make_store_map(&P.map_v, stash->v, 1, (uint64_t)n, 128))))
      NM_FAIL(ctx, NM_ERR_CUDA, "nm_mlp_forward_train: cuTensorMapEncodeTiled failed");
  }
  if (time) return stash ? launch_tc<true, true, true>(ctx, P, st) : launch_tc<false, true, true>(ctx, P, st);
  if (!view) return stash ? launch_tc<true, false>(ctx, P, st) : launch_tc<false, false>(ctx, P, st);
  return stash ? launch_tc<true, true>(ctx, P, st) : launch_tc<false, true>(ctx, P, st);
}

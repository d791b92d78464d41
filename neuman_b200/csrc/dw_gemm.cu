// Weight-gradient GEMMs of the training step at HBM rate:  dW = G^T @ X  with K = n samples,
//   G = fp16 gradient planes written by k_mlp_tc_bwd, X = fp16 activation planes written by the training forward
// (what torch autograd's  grad_output.t() @ input  computes for every nn.Linear of NeRF.forward,
// models/vanilla.py:120-152, inside trainers/vanilla_nerf_trainer.py:222 loss.backward()).
//
// Both operands are read straight from their row-major [n][width] planes:
//   TMA tensor loads bring 64-row x 64-column boxes into SWIZZLE_128B shared memory; a row-major [rows][64] box
//   is the canonical *MN-major* GMMA operand (rows = K, columns = M or N), so G serves as A (M = output channel)
//   and X as B (N = input channel) of wgmma without any transpose in memory.
//   A CTA owns 128 output channels (two warpgroups of M = 64) x 256 input channels of one GEMM; D[64 x 256] fp32 stays
//   in each warpgroup's registers while the CTA streams its row range; the epilogue reduces the partial results of the
//   CTAs with red.global.add.v2.f32 into the zero-initialised output.
// The nine 256-wide GEMMs of a step (pts_linears 1..7, feature_linear, views_linears.0's feature columns) are
// one launch: every pair of CTAs (the two output-channel halves) owns one (GEMM, row range) work item sized by its bytes.
// Bias gradients ride along: one extra N = 16 MMA per K step multiplies G^T with a block of ones, so every column of
// that accumulator holds sum_rows G[row][m] (rows past n are zero-filled by TMA and add nothing).
#include "nm_internal.cuh"
#include "tc_common.cuh"
#include <string.h>

#define DW_STAGES 4
#define DW_ROWS 64                          // K rows per pipeline stage
#define DW_BOX_BYTES (DW_ROWS * 128)        // one 64-column box
#define DW_STAGE_BYTES (6 * DW_BOX_BYTES)   // A: 2 boxes (this CTA's 128 M columns), B: 4 boxes (256 N columns)
#define DW_MAX_WORK 74
#define DW_ITEMS 9
#define DW_THREADS 256                      // two consumer warpgroups

struct DwWork {
  int a_map, a_plane, b_map, b_plane, out_idx, m_rows;
  long long row0, row1;                     // row0 and row1 multiples of DW_ROWS (row1 may be n)
};
struct DwParams {
  CUtensorMap maps[5];                      // 0: g_pre [8][n][256]  1: g_f [n][256]  2: g_v [n][128]  3: st_x [8][n][256]  4: st_f [n][256]
  DwWork work[DW_MAX_WORK];
  float* out;                               // [DW_ITEMS][256][256] fp32, zero-initialised
  float* bias_out;                          // [DW_ITEMS][256] fp32, zero-initialised: column sums of the item's G plane
  int n_work;
};

struct DwCfg {
  static constexpr int OFF_STAGE = 0;
  static constexpr int OFF_ONES = DW_STAGES * DW_STAGE_BYTES;     // one box of fp16 1.0 (any operand layout reads ones)
  static constexpr int OFF_BAR = OFF_ONES + DW_BOX_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 16 * DW_STAGES + 1024;  // + alignment slack
};
static_assert(DwCfg::SMEM_BYTES <= 232448, "shared memory of the weight-gradient kernel exceeds 227 KB");

__device__ __forceinline__ void tma_load_3d(uint32_t smem_dst, const CUtensorMap* map, int col, int row, int plane, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_dst),
      "l"(map), "r"(bar), "r"(col), "r"(row), "r"(plane) : "memory");
}

__global__ void __launch_bounds__(DW_THREADS, 1) k_dw_gemm(const __grid_constant__ DwParams P) {
  using C = DwCfg;
  extern __shared__ uint8_t smem_dyn[];
  const uint32_t pad = (1024 - (smem_u32(smem_dyn) & 1023)) & 1023;
  uint8_t* smem = smem_dyn + pad;
  const uint32_t sbase = smem_u32(smem);
  const int wg = threadIdx.x >> 7, wtid = threadIdx.x & 127;
  const int lane = threadIdx.x & 31, q = lane & 3;
  const int half = blockIdx.x & 1;                   // output channels [128 half, 128 half + 128) of the work item
  const int item = blockIdx.x >> 1;
  const TcRing<DW_STAGES, DW_STAGE_BYTES> R{sbase + C::OFF_STAGE, sbase + C::OFF_BAR};

  const DwWork W = P.work[item < P.n_work ? item : 0];
  const bool has_work = item < P.n_work && 128 * half < W.m_rows;
  const uint32_t n_stages = has_work ? (uint32_t)((W.row1 - W.row0 + DW_ROWS - 1) / DW_ROWS) : 0;

  for (int i = threadIdx.x; i < DW_BOX_BYTES / 4; i += DW_THREADS)
    reinterpret_cast<uint32_t*>(smem + C::OFF_ONES)[i] = 0x3C003C00u;      // fp16 {1.0, 1.0}
  fence_async_smem();                                                      // generic-proxy writes -> tensor-core reads
  auto fill = [&](uint32_t st) {                                           // stage st: rows row0 + 64 st ..
    mbar_arrive_expect_tx(R.full(st), DW_STAGE_BYTES);
    const uint32_t dst = R.slot(st);
    const int row = (int)(W.row0 + (long long)st * DW_ROWS);
    const CUtensorMap* ma = &P.maps[W.a_map];
    const CUtensorMap* mb = &P.maps[W.b_map];
    for (int b = 0; b < 2; ++b) tma_load_3d(dst + b * DW_BOX_BYTES, ma, 128 * half + 64 * b, row, W.a_plane, R.full(st));
    for (int b = 0; b < 4; ++b) tma_load_3d(dst + (2 + b) * DW_BOX_BYTES, mb, 64 * b, row, W.b_plane, R.full(st));
  };
  if (threadIdx.x == 0) R.init(n_stages, fill);
  __syncthreads();
  if (n_stages == 0) return;

  float d[128], db[8];
  const uint64_t ones_desc = gmma_desc_mn(sbase + C::OFF_ONES, DW_BOX_BYTES);
  for (uint32_t st = 0; st < n_stages; ++st) {
    R.wait_full(st);
    const uint32_t base = R.slot(st);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DW_ROWS / 16; ++kk) {       // 16 K rows = two 8-row groups = 2048 B
      const uint64_t a_desc = gmma_desc_mn(base + wg * DW_BOX_BYTES + kk * 2048, DW_BOX_BYTES);
      const uint64_t b_desc = gmma_desc_mn(base + 2 * DW_BOX_BYTES + kk * 2048, DW_BOX_BYTES);
      wgmma_n256_mn(d, a_desc, b_desc, (st | kk) != 0);
      wgmma_n16_mn(db, a_desc, ones_desc, (st | kk) != 0);
    }
    wgmma_commit();
    if (st > 0) { wgmma_wait<1>(); R.release(st - 1, n_stages, fill); }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(d);
  wgmma_fence_regs(db);

  // ---- epilogue: registers -> red.global.add (rows = output channels m, columns = input channels) ----
  const int mA = 128 * half + 64 * wg + 16 * (wtid >> 5) + (lane >> 2), mB = mA + 8;
  float* oA = P.out + ((size_t)W.out_idx * 256 + mA) * 256;
  float* oB = P.out + ((size_t)W.out_idx * 256 + mB) * 256;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c = 8 * j + 2 * q;
    if (mA < W.m_rows)
      asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(oA + c), "f"(d[4 * j]), "f"(d[4 * j + 1]) : "memory");
    if (mB < W.m_rows)
      asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(oB + c), "f"(d[4 * j + 2]), "f"(d[4 * j + 3]) : "memory");
  }
  if (q == 0) {                                                      // bias gradient: any of the 16 equal columns
    if (mA < W.m_rows) atomicAdd(P.bias_out + (size_t)W.out_idx * 256 + mA, db[0]);
    if (mB < W.m_rows) atomicAdd(P.bias_out + (size_t)W.out_idx * 256 + mB, db[2]);
  }
}

int nm_impl_dw_gemm(nm_ctx* ctx, const __half* g_pre, const __half* g_f, const __half* g_v, const __half* st_x,
                    const __half* st_f, int64_t n, float* out, float* bias_out, cudaStream_t st) {
  if (n >= (int64_t)0x7fff0000) NM_FAIL(ctx, NM_ERR_INVALID, "nm_dw_gemm: n too large for one call");
  NM_CHECK_CUDA(ctx, cudaMemsetAsync(out, 0, (size_t)DW_ITEMS * 256 * 256 * sizeof(float), st));
  NM_CHECK_CUDA(ctx, cudaMemsetAsync(bias_out, 0, (size_t)DW_ITEMS * 256 * sizeof(float), st));
  DwParams P;
  memset(&P, 0, sizeof(P));
  const CUtensorMapL2promotion l2 = CU_TENSOR_MAP_L2_PROMOTION_L2_128B;
  // a view-independent net (no feature / views layers: g_f, g_v, st_f null) has the seven trunk items 0..6 only
  const bool trunk_only = !g_f;
  const int n_items = trunk_only ? 7 : DW_ITEMS;
  if (tc_make_map(&P.maps[0], g_pre, 8, (uint64_t)n, 256, DW_ROWS, l2) || tc_make_map(&P.maps[3], st_x, 8, (uint64_t)n, 256, DW_ROWS, l2) ||
      (!trunk_only && (tc_make_map(&P.maps[1], g_f, 1, (uint64_t)n, 256, DW_ROWS, l2) ||
                       tc_make_map(&P.maps[2], g_v, 1, (uint64_t)n, 128, DW_ROWS, l2) ||
                       tc_make_map(&P.maps[4], st_f, 1, (uint64_t)n, 256, DW_ROWS, l2))))
    NM_FAIL(ctx, NM_ERR_CUDA, "nm_dw_gemm: cuTensorMapEncodeTiled failed");
  P.out = out;
  P.bias_out = bias_out;
  // work items (two CTAs each, one per half of the output channels): item k < 7 = pts_linears k+1 (G plane k+1, X plane k), 7 = feature_linear (g_f, X plane 7),
  // 8 = views_linears.0 feature columns (g_v: 128 output channels, st_f)
  int pairs_total = ctx->sm_count / 2;
  if (pairs_total > DW_MAX_WORK) pairs_total = DW_MAX_WORK;
  if (pairs_total < DW_ITEMS) NM_FAIL(ctx, NM_ERR_UNSUPPORTED, "nm_dw_gemm: needs at least 18 SMs");
  const long long blocks = (n + DW_ROWS - 1) / DW_ROWS;
  int pairs[DW_ITEMS];
  {
    const double wsum = trunk_only ? 7 * 1024.0 : 8 * 1024.0 + 768.0;
    int used = 0;
    for (int k = 0; k < n_items; ++k) {
      pairs[k] = (int)(pairs_total * (k < 8 ? 1024.0 : 768.0) / wsum);
      if (pairs[k] < 1) pairs[k] = 1;
      used += pairs[k];
    }
    for (int k = 0; used < pairs_total; k = (k + 1) % n_items) { ++pairs[k]; ++used; }
  }
  int w = 0;
  for (int k = 0; k < n_items; ++k) {
    for (int p = 0; p < pairs[k]; ++p, ++w) {
      DwWork& W = P.work[w];
      if (k < 7) { W.a_map = 0; W.a_plane = k + 1; W.b_map = 3; W.b_plane = k; W.m_rows = 256; }
      else if (k == 7) { W.a_map = 1; W.a_plane = 0; W.b_map = 3; W.b_plane = 7; W.m_rows = 256; }
      else { W.a_map = 2; W.a_plane = 0; W.b_map = 4; W.b_plane = 0; W.m_rows = 128; }
      W.out_idx = k;
      const long long b0 = blocks * p / pairs[k], b1 = blocks * (p + 1) / pairs[k];
      W.row0 = b0 * DW_ROWS;
      W.row1 = b1 * DW_ROWS < n ? b1 * DW_ROWS : n;
      if (W.row0 > W.row1) W.row0 = W.row1;
    }
  }
  P.n_work = w;
  NM_SET_SMEM_ONCE(ctx, (k_dw_gemm), DwCfg::SMEM_BYTES);
  k_dw_gemm<<<2 * w, DW_THREADS, DwCfg::SMEM_BYTES, st>>>(P);
  NM_CHECK_LAUNCH(ctx);
  return NM_OK;
}

// Stem convolutions (3 input channels, stride 2 along W) on Hopper (sm_90a) wgmma with ZERO-COPY im2col.
//
// The network input is stored NDHWC with 4 channels (f16) and the W padding written physically, so one input pixel
// is 8 bytes and an output pixel of a stride-2 convolution advances 16 bytes along the row.  A canonical NO-SWIZZLE
// K-major wgmma operand is made of core matrices of 8 rows x 16 bytes whose rows are 16 bytes apart; with
//     SBO (next 8-row group) = 128 B   and   LBO (next 16-byte K chunk) = 16 B
// the address of (row m, chunk j) is  start + 16 * (m + j):  row m of the A operand is the window of the RAW input row
// that starts at output pixel m - the im2col matrix of a (.., kw) filter row exists without being built.  So the A operand of a filter row (dt, dh) is just
// the input row (t + dt, 2 h + dh) copied once into shared memory by ONE bulk copy (cp.async.bulk, ~1.9 KB), instead
// of a 128-window tensor-map box per filter row (16 KB of overlapping 64-byte rows, one TMA request per window:
// the r01 "window mode", 330 us for the SlowFast Fast stem).
//
// One tile = one output row (up to 128 pixels along W) x all output channels; one pipeline stage = the kt * kh input
// rows of that tile; the packed weights stay resident in shared memory for the whole (persistent) CTA.  Warp roles
// (TMA producers, two wgmma consumer warpgroups) and the fused BN / activation epilogue are those of pv_igemm.cu.
#include "pv_common.cuh"
#include "pv_sm90.cuh"
#include "pv_epilogue.cuh"

#include <stdlib.h>
#include <string.h>

namespace pv {

using namespace sm90;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_fn();   // pv_igemm.cu

constexpr int ST_CONS_WARPS = 8;                                     // warps 0..7: two consumer warpgroups
constexpr int ST_PROD_WARPS = 3;                                     // warps 8..10: bulk-copy producers
constexpr int ST_THREADS = (ST_CONS_WARPS + ST_PROD_WARPS + 1) * 32; // 384, warp 11: epilogue DMA
constexpr int ST_DMA_WARP = ST_CONS_WARPS + ST_PROD_WARPS;
constexpr int ST_MAX_ROWS = 64;                                      // kt * kh filter rows per tile

struct StemParams {
  int N, Ti, Hi, To, Ho, Wo;
  int kt, kh, st, sh, pt, ph, dt, dh;
  int rows;                 // kt * kh input rows per tile
  int win;                  // window elements per filter row (16 | 32 | 64) = K of one filter row
  int wtiles;               // tiles along W (128 output pixels each)
  int n16;                  // output channels padded to 16: N extent of the packed weights
  int stages;
  unsigned seg_bytes;       // shared-memory bytes reserved per input row segment
  unsigned w_bytes;         // packed weights
  long long row_pitch;      // bytes between input rows (Wphys * 8)
  long long base_off;       // byte offset of the first window of a row (physical padding - conv padding - lead pixel)
  EpiParams epi;
};

// no-swizzle K-major descriptor: LBO = bytes between 16-byte K chunks, SBO = bytes between 8-row groups
template <int BN, int KS>   // KS = win / 16: k16 steps per filter row
__global__ void __launch_bounds__(ST_THREADS, 1)
conv3d_stem_rows_kernel(const __grid_constant__ StemParams P, const unsigned char* __restrict__ x,
                        const unsigned char* __restrict__ w, const unsigned char* __restrict__ zero_row,
                        const float* __restrict__ scale, const float* __restrict__ bias) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const int stages = P.stages;
  const uint32_t w_off = 0;                                                  // resident weights
  const uint32_t ring_off = (P.w_bytes + 1023u) & ~1023u;
  const uint32_t stage_bytes = (uint32_t)P.rows * P.seg_bytes + 2048u;       // + slack: the last windows read past a row
  const uint32_t staging_off = (ring_off + (uint32_t)stages * stage_bytes + 1023u) & ~1023u;
  const uint32_t staging = smem_base + staging_off;
  const uint32_t bar_base = staging + (uint32_t)(P.epi.nbuf * EPI_STAGING_BYTES);
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (stages + s); };
  const EpiSmem epi{staging, smem_gen + staging_off, bar_base + 8u * (2 * stages)};
  const uint32_t w_bar = epi.bars + 8u * EPI_BARS;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), ST_CONS_WARPS); }
    epi.init();
    mbar_init(w_bar, 1);
    prefetch_tmap(&P.epi.y_map);
    fence_mbar_init();
  }
  __syncthreads();
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  const int total_tiles = P.N * P.To * P.Ho * P.wtiles;
  auto tile_coords = [&](int tile, int& wt, int& ho, int& to, int& n) {
    wt = tile % P.wtiles; tile /= P.wtiles;
    ho = tile % P.Ho; tile /= P.Ho;
    to = tile % P.To; n = tile / P.To;
  };

  if (warp == ST_DMA_WARP) {
    epilogue_dma(P.epi, epi, total_tiles, [&](int tile, int& n0, int (&c)[4]) {
      n0 = 0;
      tile_coords(tile, c[0], c[1], c[2], c[3]);
      c[0] *= 128;
    });
  } else if (warp >= ST_CONS_WARPS) {
    // ================================ producers: one bulk copy per input row ================================
    const int pw = warp - ST_CONS_WARPS;
    if (pw == 0 && elect_one()) {          // the packed weights, once
      mbar_arrive_expect_tx(w_bar, P.w_bytes);
      for (uint32_t o = 0; o < P.w_bytes; o += 32768u)
        bulk_g2s(smem_base + w_off + o, w + o, min(32768u, P.w_bytes - o), w_bar);
    }
    int stage = 0;
    uint32_t phase = 0;
    const long long frame_pitch = P.row_pitch * P.Hi;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int wt, ho, to, n;
      tile_coords(tile, wt, ho, to, n);
      mbar_wait(empty_bar(stage), phase ^ 1u);
      const uint32_t st_base = smem_base + ring_off + (uint32_t)stage * stage_bytes;
      // bytes of a row this tile reads: 128 windows 16 B apart + the window itself, clipped to the physical row
      const long long col0 = P.base_off + (long long)wt * 128 * 16;
      long long want = 127ll * 16 + (long long)P.win * 2;          // a multiple of 16, like col0 and the row pitch
      if (col0 + want > P.row_pitch) want = P.row_pitch - col0;      // (windows of pixels >= Wo may then see stale bytes: their rows are never stored)
      const uint32_t nbytes = (uint32_t)want;
      if (elect_one()) {
        if (pw == 0) mbar_arrive_expect_tx(full_bar(stage), (uint32_t)P.rows * nbytes);
        for (int r = pw; r < P.rows; r += ST_PROD_WARPS) {
          const int fdt = r / P.kh, fdh = r - fdt * P.kh;
          const int ti = to * P.st - P.pt + fdt * P.dt, hi = ho * P.sh - P.ph + fdh * P.dh;
          const bool ok = (unsigned)ti < (unsigned)P.Ti && (unsigned)hi < (unsigned)P.Hi;
          const unsigned char* src = ok ? x + ((long long)n * P.Ti + ti) * frame_pitch + (long long)hi * P.row_pitch + col0
                                        : zero_row;                       // H / T padding: a row of zeros
          bulk_g2s(st_base + (uint32_t)r * P.seg_bytes, src, nbytes, full_bar(stage));
        }
      }
      __syncwarp();
      if (++stage == stages) { stage = 0; phase ^= 1u; }
    }
  } else {
    // ================================ consumers: wgmma + epilogue ===========================================
    // Warpgroup g computes output pixels [64 g, 64 g + 64) of the row: its windows start 64 x 16 B further on.
    // Weight columns >= n16 (BN rounded up to a wgmma width) read neighbouring K chunks: they are never stored.
    const int ctid = threadIdx.x;
    const uint32_t a_row_off = (uint32_t)(ctid >> 7) * 64u * 16u;
    const uint32_t b_lbo = (uint32_t)P.n16 * 16u;          // weights: [K / 8][n16][8] - all N rows of a K chunk contiguous
    int stage = 0, epi_buf = 0;
    uint32_t phase = 0, epi_phase = 0;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    mbar_wait(w_bar, 0);
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int wt, ho, to, n;
      tile_coords(tile, wt, ho, to, n);
      mbar_wait(full_bar(stage), phase);
      const uint32_t st_base = smem_base + ring_off + (uint32_t)stage * stage_bytes;
#pragma unroll 1
      for (int r = 0; r < P.rows; ++r) {
        // one wgmma group per filter row, one group kept in flight (the pattern of the conv main loop)
        acc_fence(acc);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
          // A: sliding windows over the raw row; B: K chunks (r * win + 16 ks) / 8 onwards
          const uint64_t a_desc = make_noswz_desc(st_base + (uint32_t)r * P.seg_bytes + (uint32_t)ks * 32u + a_row_off, 16u, 128u);
          const uint64_t b_desc = make_noswz_desc(smem_base + w_off + (uint32_t)((r * P.win + ks * 16) >> 3) * b_lbo, b_lbo, 128u);
          Wgmma<BN>::mma(acc, a_desc, b_desc, (r | ks) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        acc_fence(acc);
        wgmma_wait<1>();
      }
      wgmma_wait<0>();
      acc_fence(acc);
      mbar_arrive_if(empty_bar(stage), lane == 0);
      if (++stage == stages) { stage = 0; phase ^= 1u; }
      epilogue_tile<BN>(P.epi, epi, epi_buf, epi_phase, scale, bias, acc, ctid, 0, wt * 128, ho, to, n);
    }
  }
}

static int stem_window_lead(const pv_conv3d_desc* d) { return (((d->x_w_pad - d->pw) * d->Ci * 2) % 16) ? 1 : 0; }

}  // namespace pv

using namespace pv;

// Eligible: dense conv on the 4-channel, W-padded network input with stride 2 along W (16 bytes per output pixel),
// no residual, output channels <= 128.  The descriptor uses the window-mode conventions of pv_conv3d_desc
// (x_w_pad, x_w_phys, ci_pad64 = window length) but the weights are packed [K / 8][N16][8] (engine/packing.py).
extern "C" int pv_conv3d_stem_rows_supported(const pv_conv3d_desc* d) {
  if (!d || d->dtype != PV_F16 || d->groups != 1 || d->has_residual || !act_known(d->act)) return 0;
  if (conv3d_has_prologue(d)) return 0;
  if (d->Ci != 4 || d->sw != 2 || d->dw != 1 || d->x_w_pad <= 0 || d->x_row_stride != 4) return 0;
  if (d->x_w_pad < d->pw || (d->x_w_phys * 8) % 16) return 0;
  const int lead = stem_window_lead(d);
  const int run = (d->kw + lead) * 4;
  const int win = run <= 16 ? 16 : (run <= 32 ? 32 : 64);
  if (run > 64 || d->ci_pad64 != win) return 0;
  if (d->Co % 8 || d->Co > MAX_BN || d->y_row_stride % 8) return 0;
  if (d->kt * d->kh > ST_MAX_ROWS) return 0;
  if (!conv3d_addend_ok(d)) return 0;
  const long long base_off = (long long)(d->x_w_pad - d->pw - lead) * 8;
  if (base_off < 0 || base_off % 16) return 0;
  // every window of the last output pixel must lie inside the physical row
  if (base_off + (long long)(d->Wo - 1) * 16 + (long long)win * 2 > (long long)d->x_w_phys * 8) return 0;
  const int bn = (d->Co + 15) / 16 * 16;
  const long long wbytes = (long long)d->kt * d->kh * win * bn * 2;
  if (wbytes > 120 * 1024) return 0;
  return 1;
}

extern "C" int pv_conv3d_stem_rows_fwd(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                                       const float* bias, const void* zero_row, void* y, void* stream) {
  PV_CHECK_ARG(d && x && w && scale && bias && zero_row && y, "null argument");
  if (!pv_conv3d_stem_rows_supported(d)) { set_error("stem rows kernel: unsupported convolution"); return PV_ERR_UNSUPPORTED; }
  EncodeTiledFn encode = get_encode_fn();
  if (!encode) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return PV_ERR_CUDA; }
  const int sm_count = current_sm_count();
  if (sm_count <= 0) { set_error("cannot query the SM count"); return PV_ERR_CUDA; }
  StemParams P;
  memset(&P, 0, sizeof(P));
  P.N = d->N; P.Ti = d->Ti; P.Hi = d->Hi; P.To = d->To; P.Ho = d->Ho; P.Wo = d->Wo;
  P.kt = d->kt; P.kh = d->kh; P.st = d->st; P.sh = d->sh; P.pt = d->pt; P.ph = d->ph; P.dt = d->dt; P.dh = d->dh;
  P.rows = d->kt * d->kh;
  P.win = d->ci_pad64;
  P.wtiles = (int)cdiv(d->Wo, 128);
  P.n16 = (d->Co + 15) / 16 * 16;
  const int block_n = round_block_n(P.n16);
  P.row_pitch = (long long)d->x_w_phys * 8;
  P.base_off = (long long)(d->x_w_pad - d->pw - stem_window_lead(d)) * 8;
  P.w_bytes = (unsigned)((long long)P.rows * P.win * P.n16 * 2);
  P.seg_bytes = (unsigned)((127 * 16 + P.win * 2 + 127) & ~127);
  // everything but the stage ring: alignment slack, resident weights, ring alignment, epilogue staging and barriers,
  // ring and weight barriers (8 stages max).  With seg_bytes = 2176 for every window length, two staging buffers and
  // two ring stages fit when align1024(w_bytes) + 4352 * rows + 4096 <= 163656: every accepted shape with
  // kt * kh <= 9 filter rows (the ResNet, SlowFast, R(2+1)D and X3D stems have 3 or 7), and fewer as rows and weights
  // grow.  Otherwise one staging buffer, which fits wherever the single-buffered epilogue of earlier versions did.
  const unsigned stage_bytes = (unsigned)P.rows * P.seg_bytes + 2048u;
  size_t smem_fixed = 0;
  for (int nbuf = EPI_MAX_BUFS; nbuf >= 1; --nbuf) {
    P.epi.nbuf = nbuf;
    smem_fixed = 2048 + ((P.w_bytes + 1023) & ~1023u) + 1024 + epi_smem_bytes(nbuf) + 8 * (2 * 8 + 1) + 16;
    if (227 * 1024 - (long long)smem_fixed >= 2ll * stage_bytes) break;
  }
  {
    const long long budget = 227 * 1024 - (long long)smem_fixed;
    long long st = budget / stage_bytes;
    if (st > 8) st = 8;
    if (st < 2) { set_error("stem rows kernel: not enough shared memory for two stages"); return PV_ERR_UNSUPPORTED; }
    P.stages = (int)st;
  }
  const size_t smem_bytes = smem_fixed + (size_t)P.stages * stage_bytes;
  // ---- epilogue: output tile = box [64 ch, 128 px, 1, 1, 1] of y [Co, Wo, Ho, To, N]
  P.epi.block_n = block_n;
  P.epi.Co = d->Co;
  P.epi.rows = d->Wo < 128 ? d->Wo : 128;
  P.epi.act = d->act;
  P.epi.has_residual = 0;
  const long long ostr[4] = {1, d->Wo, (long long)d->Wo * d->Ho, (long long)d->Wo * d->Ho * d->To};
  const int O[4] = {d->Wo, d->Ho, d->To, d->N};
  const int box[4] = {P.epi.rows, 1, 1, 1};
  epi_set_addend(P.epi, d);
  for (int m = 0; m < 4; ++m) {
    P.epi.o_ext[m] = O[m];
    P.epi.o_box[m] = box[m];
    P.epi.o_pos[m] = (int)ostr[m];
  }
  {
    cuuint64_t gdim[5] = {(cuuint64_t)d->Co, (cuuint64_t)O[0], (cuuint64_t)O[1], (cuuint64_t)O[2], (cuuint64_t)O[3]};
    cuuint64_t gstr[4];
    cuuint32_t bx[5] = {64, (cuuint32_t)box[0], 1, 1, 1}, estr[5] = {1, 1, 1, 1, 1};
    for (int m = 0; m < 4; ++m) gstr[m] = (cuuint64_t)(ostr[m] * d->y_row_stride * 2);
    CUresult cr = encode(&P.epi.y_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, y, gdim, gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(stem Y) failed: %d", (int)cr); return PV_ERR_CUDA; }
  }
  const long long total_tiles = (long long)d->N * d->To * d->Ho * P.wtiles;
  if (total_tiles == 0) return PV_OK;
  PV_CHECK_ARG(total_tiles < (1ll << 31), "too many tiles");
  const int grid = (int)(total_tiles < sm_count ? total_tiles : sm_count);
  {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(ST_THREADS);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    const unsigned char *xb = (const unsigned char*)x, *wb = (const unsigned char*)w, *zb = (const unsigned char*)zero_row;
#define PV_ST_LAUNCH(BN, KS)                                                                              \
  if (block_n == BN && P.win == 16 * KS) {                                                                \
    PV_OPT_IN_SMEM((conv3d_stem_rows_kernel<BN, KS>), 227 * 1024);                                        \
    PV_CUDA_OK(cudaLaunchKernelEx(&cfg, conv3d_stem_rows_kernel<BN, KS>, P, xb, wb, zb, scale, bias));    \
    name = "conv3d_stem_rows_kernel<" #BN "," #KS ">";                                                     \
  }
    const char* name = nullptr;
    PV_ST_LAUNCH(16, 1) PV_ST_LAUNCH(16, 2) PV_ST_LAUNCH(16, 4)
    PV_ST_LAUNCH(32, 1) PV_ST_LAUNCH(32, 2) PV_ST_LAUNCH(32, 4)
    PV_ST_LAUNCH(64, 1) PV_ST_LAUNCH(64, 2) PV_ST_LAUNCH(64, 4)
    PV_ST_LAUNCH(128, 1) PV_ST_LAUNCH(128, 2) PV_ST_LAUNCH(128, 4)
#undef PV_ST_LAUNCH
    if (!name) { set_error("internal: no stem instance for BN=%d win=%d", block_n, P.win); return PV_ERR_INVALID; }
    PV_LAUNCH_OK(name);
  }
  return PV_OK;
}

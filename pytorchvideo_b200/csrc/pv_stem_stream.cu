// Temporal-streaming stem: a (KT, kh, kw) stem convolution with few output channels (the SlowFast Fast stem, 5x7x7,
// 3 -> 8) in ONE pass over the input, with the temporal taps summed on chip.
//
// The operand machinery is that of the stem-rows kernel (pv_stem.cu): the 4-channel, W-padded network input, one bulk
// copy per input row, no-swizzle A descriptors whose 16-byte K chunks overlap (LBO 16 B, SBO 128 B) so that row m of
// the A operand is the filter window of output pixel m, resident packed weights, two consumer warpgroups, three copy
// warps and the epilogue DMA warp.  What differs is the work unit: one output row (n, ho, 128-pixel W tile) walked
// over ALL input frames ti.  One pipeline stage holds the kh input rows of one frame; the consumers multiply them by
// the weights of all KT temporal taps at once (N = KT * 8 columns, column 8 j + c = tap j of output channel c).
//
// A wgmma fragment holds columns 8 i + 2 (lane % 4) + {0, 1}: one thread holds the same channel pair of EVERY tap for
// its two rows, so the temporal sum never leaves the thread.  Tap j of frame ti belongs to output frame
// to = ti + pt - j (stride and dilation 1); a ring of KT partial outputs in registers, rotated once per frame, takes
// them.  After frame ti the oldest slot (to = ti + pt - KT + 1) has received its last tap and is finished through
// the shared staging / TMA-store epilogue (pv_epilogue.cuh) as an n16 fragment; after the last frame the rest of the
// ring is.  Output frames therefore leave in increasing order, each once (pt < KT), and taps that would read frames
// outside [0, Ti) - the temporal zero padding - simply never arrive.  The taps are summed in fp32 and rounded to f16
// once, where the factored route (stem rows with KT * 8 channels + pv_temporal_tap_sum) rounds every tap's partial.
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

constexpr int SS_CONS_WARPS = 8;                                     // warps 0..7: two consumer warpgroups
constexpr int SS_PROD_WARPS = 3;                                     // warps 8..10: bulk-copy producers
constexpr int SS_THREADS = (SS_CONS_WARPS + SS_PROD_WARPS + 1) * 32; // 384, warp 11: epilogue DMA
constexpr int SS_DMA_WARP = SS_CONS_WARPS + SS_PROD_WARPS;
constexpr int SS_CO = 8;                                             // output channels

struct StreamParams {
  int N, Ti, Hi, To, Ho;
  int kh, sh, pt, ph, dh;
  int win;                  // window elements per filter row (16 | 32 | 64) = K of one filter row
  int wtiles;               // tiles along W (128 output pixels each)
  int stages;
  unsigned seg_bytes;       // shared-memory bytes reserved per input row segment
  unsigned w_bytes;         // packed weights [kh * win / 8][KT * 8][8]
  long long row_pitch;      // bytes between input rows (Wphys * 8)
  long long base_off;       // byte offset of the first window of a row (physical padding - conv padding - lead pixel)
  EpiParams epi;
};

template <int KT, int KS>   // KS = win / 16: k16 steps per filter row
__global__ void __launch_bounds__(SS_THREADS, 1)
conv3d_stem_stream_kernel(const __grid_constant__ StreamParams P, const unsigned char* __restrict__ x,
                          const unsigned char* __restrict__ w, const unsigned char* __restrict__ zero_row,
                          const float* __restrict__ scale, const float* __restrict__ bias) {
  constexpr int BN = KT * SS_CO;         // wgmma N: all taps of all channels
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const int stages = P.stages;
  const uint32_t ring_off = (P.w_bytes + 1023u) & ~1023u;                  // weights at 0
  const uint32_t stage_bytes = (uint32_t)P.kh * P.seg_bytes + 2048u;        // + slack: the last windows read past a row
  const uint32_t staging_off = (ring_off + (uint32_t)stages * stage_bytes + 1023u) & ~1023u;
  const uint32_t staging = smem_base + staging_off;
  const uint32_t bar_base = staging + (uint32_t)(P.epi.nbuf * EPI_STAGING_BYTES);
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (stages + s); };
  const EpiSmem epi{staging, smem_gen + staging_off, bar_base + 8u * (2 * stages)};
  const uint32_t w_bar = epi.bars + 8u * EPI_BARS;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), SS_CONS_WARPS); }
    epi.init();
    mbar_init(w_bar, 1);
    prefetch_tmap(&P.epi.y_map);
    fence_mbar_init();
  }
  __syncthreads();
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  const int units = P.N * P.Ho * P.wtiles;
  auto unit_coords = [&](int u, int& wt, int& ho, int& n) {
    wt = u % P.wtiles; u /= P.wtiles;
    ho = u % P.Ho; n = u / P.Ho;
  };

  if (warp == SS_DMA_WARP) {
    // ================================ epilogue DMA: one store per output frame ==============================
    // (epilogue_dma's protocol without a residual; the CTA's tiles are its units x every output frame, in order)
    if (!elect_one()) return;
    const int my_units = blockIdx.x < units ? (units - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const long long my_tiles = (long long)my_units * P.To;
    for (int b = 0; b < P.epi.nbuf; ++b)
      if (b < my_tiles) mbar_arrive(epi.ready(b));
    int b = 0;
    uint32_t phase = 0;
    long long k = 0;
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
      int wt, ho, n;
      unit_coords(u, wt, ho, n);
      for (int to = 0; to < P.To; ++to, ++k) {
        mbar_wait(epi.full(b), phase);
        tma_store_5d(&P.epi.y_map, epi.buf(b), 0, wt * 128, ho, to, n);
        tma_store_commit();
        tma_store_wait_read0();
        if (k + P.epi.nbuf < my_tiles) mbar_arrive(epi.ready(b));
        if (++b == P.epi.nbuf) { b = 0; phase ^= 1u; }
      }
    }
    tma_store_wait_all();
  } else if (warp >= SS_CONS_WARPS) {
    // ================================ producers: one bulk copy per input row of a frame =====================
    const int pw = warp - SS_CONS_WARPS;
    if (pw == 0 && elect_one()) {          // the packed weights, once
      mbar_arrive_expect_tx(w_bar, P.w_bytes);
      for (uint32_t o = 0; o < P.w_bytes; o += 32768u)
        bulk_g2s(smem_base + o, w + o, min(32768u, P.w_bytes - o), w_bar);
    }
    int stage = 0;
    uint32_t phase = 0;
    const long long frame_pitch = P.row_pitch * P.Hi;
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
      int wt, ho, n;
      unit_coords(u, wt, ho, n);
      // bytes of a row the tile reads: 128 windows 16 B apart + the window itself, clipped to the physical row
      const long long col0 = P.base_off + (long long)wt * 128 * 16;
      long long want = 127ll * 16 + (long long)P.win * 2;
      if (col0 + want > P.row_pitch) want = P.row_pitch - col0;     // (windows of pixels >= Wo are never stored)
      const uint32_t nbytes = (uint32_t)want;
      for (int ti = 0; ti < P.Ti; ++ti) {
        mbar_wait(empty_bar(stage), phase ^ 1u);
        const uint32_t st_base = smem_base + ring_off + (uint32_t)stage * stage_bytes;
        if (elect_one()) {
          if (pw == 0) mbar_arrive_expect_tx(full_bar(stage), (uint32_t)P.kh * nbytes);
          const unsigned char* frame = x + ((long long)n * P.Ti + ti) * frame_pitch + col0;
          for (int r = pw; r < P.kh; r += SS_PROD_WARPS) {
            const int hi = ho * P.sh - P.ph + r * P.dh;
            const unsigned char* src = (unsigned)hi < (unsigned)P.Hi ? frame + (long long)hi * P.row_pitch : zero_row;
            bulk_g2s(st_base + (uint32_t)r * P.seg_bytes, src, nbytes, full_bar(stage));
          }
        }
        __syncwarp();
        if (++stage == stages) { stage = 0; phase ^= 1u; }
      }
    }
  } else {
    // ================================ consumers: wgmma per frame, temporal ring, epilogue ===================
    // Warpgroup g computes output pixels [64 g, 64 g + 64) of the row: its windows start 64 x 16 B further on.
    const int ctid = threadIdx.x;
    const uint32_t a_row_off = (uint32_t)(ctid >> 7) * 64u * 16u;
    constexpr uint32_t b_lbo = (uint32_t)BN * 16u;          // weights: [K / 8][BN][8]
    int stage = 0, rstage = 0, epi_buf = 0;
    uint32_t phase = 0, epi_phase = 0;
    float acc[BN / 2];            // register 4 j + 2 i + e: tap j, row +8 i, channel 2 (lane % 4) + e
    float ring[KT][4];            // ring[s]: partial output frame ti + pt - s (after frame ti has been added)
    float frag[8];                // n16 fragment handed to the epilogue: channels 0..7 in registers 0..3
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
#pragma unroll
    for (int i = 4; i < 8; ++i) frag[i] = 0.f;
    mbar_wait(w_bar, 0);
    auto finish = [&](const float (&v)[4], int to, int wt, int ho, int n) {
#pragma unroll
      for (int i = 0; i < 4; ++i) frag[i] = v[i];
      epilogue_tile<16>(P.epi, epi, epi_buf, epi_phase, scale, bias, frag, ctid, 0, wt * 128, ho, to, n);
    };
    // all kh * KS products of the next frame in the ring as ONE commit group into `a`
    auto issue = [&](float (&a)[BN / 2]) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t st_base = smem_base + ring_off + (uint32_t)stage * stage_bytes;
      acc_fence(a);
      wgmma_fence();
#pragma unroll 1
      for (int r = 0; r < P.kh; ++r) {
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
          const uint64_t a_desc = make_noswz_desc(st_base + (uint32_t)r * P.seg_bytes + (uint32_t)ks * 32u + a_row_off, 16u, 128u);
          const uint64_t b_desc = make_noswz_desc(smem_base + (uint32_t)((r * P.win + ks * 16) >> 3) * b_lbo, b_lbo, 128u);
          Wgmma<BN>::mma(a, a_desc, b_desc, (r | ks) != 0 ? 1u : 0u);
        }
      }
      wgmma_commit();
      acc_fence(a);
      if (++stage == stages) { stage = 0; phase ^= 1u; }
    };
    // frame ti's products have landed in `a`: free its stage, add tap j to output frame ti + pt - j = ring slot j,
    // finish the slot that has all its taps and rotate the ring
    auto retire = [&](float (&a)[BN / 2], int ti, int wt, int ho, int n) {
      acc_fence(a);
      mbar_arrive_if(empty_bar(rstage), lane == 0);
      if (++rstage == stages) rstage = 0;
#pragma unroll
      for (int j = 0; j < KT; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) ring[j][i] += a[4 * j + i];
      const int done = ti + P.pt - (KT - 1);
      if ((unsigned)done < (unsigned)P.To) finish(ring[KT - 1], done, wt, ho, n);
#pragma unroll
      for (int s = KT - 1; s > 0; --s)
#pragma unroll
        for (int i = 0; i < 4; ++i) ring[s][i] = ring[s - 1][i];
#pragma unroll
      for (int i = 0; i < 4; ++i) ring[0][i] = 0.f;
    };
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
      int wt, ho, n;
      unit_coords(u, wt, ho, n);
#pragma unroll
      for (int s = 0; s < KT; ++s)
#pragma unroll
        for (int i = 0; i < 4; ++i) ring[s][i] = 0.f;
#pragma unroll 1
      for (int ti = 0; ti < P.Ti; ++ti) {
        issue(acc);
        wgmma_wait<0>();
        retire(acc, ti, wt, ho, n);
      }
      // frames past the clip are zero padding: the partials still in the ring are finished, oldest first
#pragma unroll
      for (int s = KT - 1; s > 0; --s) {
        const int to = P.Ti - 1 + P.pt - (s - 1);            // slot s now holds frame Ti + pt - s
        if ((unsigned)to < (unsigned)P.To) finish(ring[s], to, wt, ho, n);
      }
    }
  }
}

static int stream_window_lead(const pv_conv3d_desc* d) { return (((d->x_w_pad - d->pw) * d->Ci * 2) % 16) ? 1 : 0; }

}  // namespace pv

using namespace pv;

// Eligible: the stem-rows conditions (dense f16 conv on the 4-channel, W-padded network input, stride 2 along W, no
// residual) with KT = 5 temporal taps at stride and dilation 1, temporal padding < KT, 8 output channels, window 32
// (kw 5..7), and no addend.  Weights f16 [kh * win / 8][40][8] (engine/packing.py pack_stem_stream).
extern "C" int pv_conv3d_stem_stream_supported(const pv_conv3d_desc* d) {
  if (!d || d->dtype != PV_F16 || d->groups != 1 || d->has_residual || d->addend || !act_known(d->act)) return 0;
  if (conv3d_has_prologue(d)) return 0;
  if (d->Ci != 4 || d->sw != 2 || d->dw != 1 || d->x_w_pad <= 0 || d->x_row_stride != 4) return 0;
  if (d->x_w_pad < d->pw || (d->x_w_phys * 8) % 16) return 0;
  if (d->Co != SS_CO || d->kt != 5 || d->st != 1 || d->dt != 1 || d->pt < 0 || d->pt >= d->kt) return 0;
  if (d->To != d->Ti + 2 * d->pt - (d->kt - 1) || d->To <= 0 || d->Ti <= 0) return 0;
  if (d->kh < 1 || d->kh > 16 || d->y_row_stride % 8) return 0;
  const int lead = stream_window_lead(d);
  const int run = (d->kw + lead) * 4;
  const int win = run <= 16 ? 16 : (run <= 32 ? 32 : 64);
  if (win != 32 || d->ci_pad64 != win) return 0;
  const long long base_off = (long long)(d->x_w_pad - d->pw - lead) * 8;
  if (base_off < 0 || base_off % 16) return 0;
  // every window of the last output pixel must lie inside the physical row
  if (base_off + (long long)(d->Wo - 1) * 16 + (long long)win * 2 > (long long)d->x_w_phys * 8) return 0;
  return 1;
}

extern "C" int pv_conv3d_stem_stream_fwd(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                                         const float* bias, const void* zero_row, void* y, void* stream) {
  PV_CHECK_ARG(d && x && w && scale && bias && zero_row && y, "null argument");
  if (!pv_conv3d_stem_stream_supported(d)) { set_error("stem stream kernel: unsupported convolution"); return PV_ERR_UNSUPPORTED; }
  EncodeTiledFn encode = get_encode_fn();
  if (!encode) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return PV_ERR_CUDA; }
  const int sm_count = current_sm_count();
  if (sm_count <= 0) { set_error("cannot query the SM count"); return PV_ERR_CUDA; }
  StreamParams P;
  memset(&P, 0, sizeof(P));
  P.N = d->N; P.Ti = d->Ti; P.Hi = d->Hi; P.To = d->To; P.Ho = d->Ho;
  P.kh = d->kh; P.sh = d->sh; P.pt = d->pt; P.ph = d->ph; P.dh = d->dh;
  P.win = d->ci_pad64;
  P.wtiles = (int)cdiv(d->Wo, 128);
  P.row_pitch = (long long)d->x_w_phys * 8;
  P.base_off = (long long)(d->x_w_pad - d->pw - stream_window_lead(d)) * 8;
  P.w_bytes = (unsigned)((long long)d->kh * P.win * d->kt * SS_CO * 2);
  P.seg_bytes = (unsigned)((127 * 16 + P.win * 2 + 127) & ~127);
  // everything but the stage ring: alignment slack, resident weights, ring alignment, two epilogue staging buffers and
  // their barriers, ring and weight barriers (8 stages max); at kh = 7 (17 KB of weights) 8 ring stages fit
  const unsigned stage_bytes = (unsigned)P.kh * P.seg_bytes + 2048u;
  P.epi.nbuf = EPI_MAX_BUFS;
  const size_t smem_fixed = 2048 + ((P.w_bytes + 1023) & ~1023u) + 1024 + epi_smem_bytes(P.epi.nbuf) + 8 * (2 * 8 + 1) + 16;
  {
    long long st = (227 * 1024 - (long long)smem_fixed) / stage_bytes;
    if (st > 8) st = 8;
    if (st < 2) { set_error("stem stream kernel: not enough shared memory for two stages"); return PV_ERR_UNSUPPORTED; }
    P.stages = (int)st;
  }
  const size_t smem_bytes = smem_fixed + (size_t)P.stages * stage_bytes;
  // ---- epilogue: output tile = box [64 ch, 128 px, 1, 1, 1] of y [Co, Wo, Ho, To, N], clipped to Co = 8
  P.epi.block_n = 16;
  P.epi.Co = d->Co;
  P.epi.rows = d->Wo < 128 ? d->Wo : 128;
  P.epi.act = d->act;
  P.epi.has_residual = 0;
  epi_set_addend(P.epi, d);
  const long long ostr[4] = {1, d->Wo, (long long)d->Wo * d->Ho, (long long)d->Wo * d->Ho * d->To};
  const int O[4] = {d->Wo, d->Ho, d->To, d->N};
  const int box[4] = {P.epi.rows, 1, 1, 1};
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
    if (cr != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(stem stream Y) failed: %d", (int)cr); return PV_ERR_CUDA; }
  }
  const long long units = (long long)d->N * d->Ho * P.wtiles;
  if (units == 0) return PV_OK;
  PV_CHECK_ARG(units * d->To < (1ll << 31), "too many tiles");
  const int grid = (int)(units < sm_count ? units : sm_count);
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(SS_THREADS);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const unsigned char *xb = (const unsigned char*)x, *wb = (const unsigned char*)w, *zb = (const unsigned char*)zero_row;
  const char* name = nullptr;
#define PV_SS_LAUNCH(KT, KS)                                                                              \
  if (d->kt == KT && P.win == 16 * KS) {                                                                  \
    PV_OPT_IN_SMEM((conv3d_stem_stream_kernel<KT, KS>), 227 * 1024);                                      \
    PV_CUDA_OK(cudaLaunchKernelEx(&cfg, conv3d_stem_stream_kernel<KT, KS>, P, xb, wb, zb, scale, bias));  \
    name = "conv3d_stem_stream_kernel<" #KT "," #KS ">";                                                   \
  }
  PV_SS_LAUNCH(5, 2)
#undef PV_SS_LAUNCH
  if (!name) { set_error("internal: no stem stream instance for kt=%d win=%d", d->kt, P.win); return PV_ERR_INVALID; }
  PV_LAUNCH_OK(name);
  return PV_OK;
}

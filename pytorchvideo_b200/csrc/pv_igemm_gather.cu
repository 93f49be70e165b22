// Implicit-GEMM convolution for NARROW inputs (C_in < 64: the 3-channel stems, the SlowFast Fast
// pathway C=8..32, X3D's 24/48/56-wide tensors) on Hopper (sm_90a) tensor cores.
//
// With few input channels one filter tap is only 8..64 bytes of K, so a 64-channel TMA box per tap
// would be mostly zero fill.  Here the GEMM K axis is the flattened (tap, ci) index and the A tile
// (128 output positions x 64 K-elements, 128B-swizzled K-major) is assembled by up to 3 producer warps
// with coalesced 8/16-byte global loads (im2col gather, zero fill for padding) written straight to
// the swizzled shared-memory layout the wgmma descriptor expects; weights still arrive by TMA.
// The two consumer warpgroups (wgmma, register accumulators, fused epilogue) are those of pv_igemm.cu.
#include "pv_common.cuh"
#include "pv_sm90.cuh"
#include "pv_epilogue.cuh"

#include <mutex>
#include <stdlib.h>
#include <string.h>

namespace pv {

using namespace sm90;

constexpr int GG_BM = 128;
constexpr int GG_BK = 64;
constexpr int GG_A_BYTES = GG_BM * GG_BK * 2;
constexpr int GG_MAX_UNITS = 256;
constexpr int GG_CONS_WARPS = 8;          // warps 0..7: two consumer warpgroups
constexpr int GG_PROD_WARPS = 3;          // warps 8..10: gather producers
constexpr int GG_THREADS = (GG_CONS_WARPS + GG_PROD_WARPS + 1) * 32;   // 384, warp 11: epilogue DMA
constexpr int GG_DMA_WARP = GG_CONS_WARPS + GG_PROD_WARPS;

struct GatherParams {
  CUtensorMap b_map;
  int N, Ti, Hi, Wi, To, Ho, Wo;
  int st, sh, sw, pt, ph, pw;
  int gbytes;        // gather unit: 8 or 16 bytes
  int units_total;   // taps * (Ci*2/gbytes)
  int upk;           // units per 64-element k-block: 128 / gbytes
  int upt, taps;     // units per tap, taps (<= 64: one validity bit per tap)
  int num_kb;
  long long x_row_stride;
  long long M;
  int m_tiles, n_tiles, block_n, Co, stages;
  int nprod;   // active producer warps, <= stages (see the slot-ownership note in the kernel)
  EpiParams epi;
  int unit_off[GG_MAX_UNITS];        // element offset of the unit relative to the row's (t0,h0,w0) corner
  unsigned int unit_d[GG_MAX_UNITS];  // packed (dt | dh<<8 | dw<<16) tap displacement (dilation applied)
};

template <int BN>
__global__ void __launch_bounds__(GG_THREADS, 1)
conv3d_igemm_gather_kernel(const __grid_constant__ GatherParams P, const __half* __restrict__ x,
                           const float* __restrict__ scale, const float* __restrict__ bias) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const int stages = P.stages;
  const uint32_t b_bytes = (uint32_t)BN * GG_BK * 2;
  const uint32_t stage_bytes = GG_A_BYTES + b_bytes;
  const uint32_t staging_off = (uint32_t)((stages * stage_bytes + 1023u) & ~1023u);
  const uint32_t staging = smem_base + staging_off;
  const uint32_t bar_base = staging + (uint32_t)(P.epi.nbuf * EPI_STAGING_BYTES);
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (stages + s); };
  const EpiSmem epi{staging, smem_gen + staging_off, bar_base + 8u * (2 * stages)};

  __shared__ int s_off[GG_MAX_UNITS];
  __shared__ unsigned s_d[GG_MAX_UNITS];
  for (int i = threadIdx.x; i < GG_MAX_UNITS; i += blockDim.x) { s_off[i] = P.unit_off[i]; s_d[i] = P.unit_d[i]; }
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int PROD_WARP0 = GG_CONS_WARPS;

  if (threadIdx.x == 0) {
    prefetch_tmap(&P.b_map);
    prefetch_tmap(&P.epi.y_map);
    for (int s = 0; s < stages; ++s) {
      mbar_init(full_bar(s), 2);               // the owning producer warp's arrive + its expect_tx arrive
      mbar_init(empty_bar(s), GG_CONS_WARPS);  // one arrive per consumer warp
    }
    epi.init();
    fence_mbar_init();
  }
  __syncthreads();
  // Programmatic dependent launch: everything above (barrier init, descriptor prefetch) overlaps the tail of the
  // previous kernel in the stream / graph; its results are only touched below.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  const int total_tiles = P.n_tiles * P.m_tiles;

  if (warp == GG_DMA_WARP) {
    epilogue_dma(P.epi, epi, total_tiles, [&](int tile, int& n0, int (&c)[4]) {
      n0 = (tile % P.n_tiles) * BN;
      c[0] = (tile / P.n_tiles) * GG_BM;
      c[1] = c[2] = c[3] = 0;
    });
  } else if (warp >= PROD_WARP0) {
    // ================================ gather producers =======================================
    // Warp-per-k-block im2col gather.  Producer warp w owns k-blocks g = w, w+nprod, ... of this CTA's
    // (tile, k-block) sequence and fills the whole 128 x 64 A tile of that k-block alone: lane l
    // covers rows l, l+32, l+64, l+96, each unit is a zero-filling cp.async straight into the
    // swizzled layout.  All producer warps are in flight on different k-blocks, so the serial issue
    // latency of one thread (measured ~1000 clk per 4 copies when every warp worked on the SAME
    // k-block) no longer bounds the pipeline; a warp publishes its k-block (proxy fence + one
    // mbarrier arrive) when its own copies have landed.
    const int wprod = warp - PROD_WARP0;
    const int my_tiles = (total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int total_g = my_tiles * P.num_kb;
    int cur_seq = -1;
    const __half* xrow[4];
    unsigned long long vmask[4];     // bit `tap` set <=> row q's input position for that tap is inside the tensor
    int n_tile = 0;
    const unsigned Ti = (unsigned)P.Ti, Hi = (unsigned)P.Hi, Wi = (unsigned)P.Wi;
    const uint32_t rsw = (uint32_t)(lane & 7);           // (lane + 32q) & 7
    const uint32_t row_off = (uint32_t)lane * 128u;
    // Slot ownership: k-block g goes to slot g % stages and warp g % nprod, so when stages is not a multiple of
    // nprod consecutive fills of a slot come from different warps.  A parity wait must then not alias a completion
    // two phases back: the fill of g waits for the consumers to release g - stages, and the same warp's previous
    // fill, g - nprod, already waited for g - nprod - stages >= g - 2 stages (nprod <= stages) to be released, and
    // the consumers release in order.
    // ncu source view: the producers wait on their own cp.async data and on the empty barrier about equally.
    for (int g = wprod; wprod < P.nprod && g < total_g; g += P.nprod) {
      const int tile_seq = g / P.num_kb;
      const int kb = g - tile_seq * P.num_kb;
      const int stage = g % stages;
      const uint32_t phase = (uint32_t)((g / stages) & 1);
      if (tile_seq != cur_seq) {
        // Per tile: row corners + one validity bit per (row, tap).  Everything in the copy loop below is
        // then branch-free (the bounds tests used to compile into divergent short-circuit branches with a
        // constant-bank load each: ~4000 clk of exposed latency per k-block).
        cur_seq = tile_seq;
        const int tile = (int)blockIdx.x + tile_seq * (int)gridDim.x;
        n_tile = tile % P.n_tiles;
        const int m_tile = tile / P.n_tiles;
        int t0[4], h0[4], w0[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const long long m = (long long)m_tile * GG_BM + lane + 32 * q;
          const bool rok = m < P.M;
          const uint32_t mu = rok ? (uint32_t)m : 0u;
          uint32_t r = mu / (uint32_t)P.Wo;
          const int wo = (int)(mu - r * (uint32_t)P.Wo);
          uint32_t r2 = r / (uint32_t)P.Ho;
          const int ho = (int)(r - r2 * (uint32_t)P.Ho);
          const uint32_t n_u = r2 / (uint32_t)P.To;
          const int to = (int)(r2 - n_u * (uint32_t)P.To);
          t0[q] = to * P.st - P.pt; h0[q] = ho * P.sh - P.ph; w0[q] = wo * P.sw - P.pw;
          if (!rok) t0[q] = -100000;        // every tap out of range -> all-zero row
          xrow[q] = x + ((((long long)n_u * P.Ti + t0[q]) * P.Hi + h0[q]) * P.Wi + w0[q]) * P.x_row_stride;
          vmask[q] = 0ull;
        }
        for (int tap = 0; tap < P.taps; ++tap) {
          const unsigned dd = s_d[tap * P.upt];
          const int dt_ = (int)(dd & 0xffu), dh_ = (int)((dd >> 8) & 0xffu), dw_ = (int)((dd >> 16) & 0xffu);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const unsigned ok = (unsigned)((unsigned)(t0[q] + dt_) < Ti) & (unsigned)((unsigned)(h0[q] + dh_) < Hi) &
                                (unsigned)((unsigned)(w0[q] + dw_) < Wi);
            vmask[q] |= (unsigned long long)ok << tap;
          }
        }
      }
      mbar_wait(empty_bar(stage), phase ^ 1u);
      const uint32_t a_tile = smem_base + stage * stage_bytes;
      if (elect_one()) {
        mbar_arrive_expect_tx(full_bar(stage), b_bytes);
        tma_load_2d(a_tile + GG_A_BYTES, &P.b_map, full_bar(stage), kb * GG_BK, n_tile * BN);
      }
      __syncwarp();
      const int u_base = kb * P.upk;
      int units_here = P.units_total - u_base;
      if (units_here > P.upk) units_here = P.upk;
      // zero-fill the whole 64-element row: the consumers issue all four k16 steps of every k-block
      const int need = P.upk;
      const uint32_t rbase = a_tile + row_off;
      if (P.gbytes == 16) {
        for (int ui = 0; ui < need; ++ui) {
          const bool uok = ui < units_here;
          const int uu = uok ? u_base + ui : 0;
          const int off = s_off[uu];
          const unsigned tap = s_d[uu] >> 24;
          const uint32_t dst = rbase + (((uint32_t)ui ^ rsw) << 4);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const bool ok = uok && ((vmask[q] >> tap) & 1ull);
            const __half* src = ok ? xrow[q] + off : x;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + (uint32_t)q * 4096u), "l"(src),
                         "r"(ok ? 16u : 0u) : "memory");
          }
        }
      } else {
        for (int ui = 0; ui < need; ++ui) {
          const bool uok = ui < units_here;
          const int uu = uok ? u_base + ui : 0;
          const int off = s_off[uu];
          const unsigned tap = s_d[uu] >> 24;
          const uint32_t dst = rbase + ((((uint32_t)ui >> 1) ^ rsw) << 4) + (((uint32_t)ui & 1u) << 3);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const bool ok = uok && ((vmask[q] >> tap) & 1ull);
            const __half* src = ok ? xrow[q] + off : x;
            asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst + (uint32_t)q * 4096u), "l"(src),
                         "r"(ok ? 8u : 0u) : "memory");
          }
        }
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      fence_proxy_async_smem();
      __syncwarp();
      if (elect_one()) mbar_arrive(full_bar(stage));
    }
  } else if (warp < GG_CONS_WARPS) {
    // ================================ consumers: wgmma + epilogue ===========================
    const int ctid = threadIdx.x;
    const uint32_t a_row_off = (uint32_t)(ctid >> 7) * 64u * 128u;   // this warpgroup's 64 rows
    const int num_kb = P.num_kb;
    int stage = 0, epi_buf = 0;
    uint32_t phase = 0, epi_phase = 0;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int n_tile = tile % P.n_tiles;
      const int m_tile = tile / P.n_tiles;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t a_addr = smem_base + stage * stage_bytes;
        const uint64_t a_desc = make_kmajor_desc(a_addr + a_row_off, 128);
        const uint64_t b_desc = make_kmajor_desc(a_addr + GG_A_BYTES, 128);
        acc_fence(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GG_BK / 16; ++k)
          Wgmma<BN>::mma(acc, a_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k), (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        acc_fence(acc);
        wgmma_wait<1>();                          // the previous k-block's wgmma have retired: free its stage
        mbar_arrive_if(empty_bar(prev < 0 ? stage : prev), prev >= 0 && lane == 0);
        prev = stage;
        if (++stage == stages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      acc_fence(acc);
      mbar_arrive_if(empty_bar(prev < 0 ? stage : prev), prev >= 0 && lane == 0);
      epilogue_tile<BN>(P.epi, epi, epi_buf, epi_phase, scale, bias, acc, ctid, n_tile * BN, m_tile * GG_BM, 0, 0, 0);
    }
  }
}

// =============================================================================================
// Host side
// =============================================================================================
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_fn();   // pv_igemm.cu

int conv3d_gather_supported(const pv_conv3d_desc* d) {
  if (d->dtype != PV_F16 || d->groups != 1) return 0;
  if (!(d->Ci == 4 || (d->Ci % 8 == 0 && d->Ci < 64))) return 0;
  if (d->Co % 8) return 0;
  if (d->ci_pad64 != d->Ci) return 0;        // weights packed with the un-padded per-tap K extent
  const int gbytes = d->Ci == 4 ? 8 : 16;
  const int units = d->kt * d->kh * d->kw * (d->Ci * 2 / gbytes);
  if (units > GG_MAX_UNITS) return 0;
  if (d->x_row_stride % (gbytes / 2) || d->y_row_stride % 8 || (d->has_residual && d->res_row_stride % 8)) return 0;
  if (d->dt * (d->kt - 1) > 255 || d->dh * (d->kh - 1) > 255 || d->dw * (d->kw - 1) > 255) return 0;
  if (d->kt * d->kh * d->kw > 64) return 0;   // one validity bit per tap
  const long long M = (long long)d->N * d->To * d->Ho * d->Wo;
  if (M >= (1ll << 31)) return 0;
  return 1;
}

int conv3d_gather_launch(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                         const float* bias, const void* residual, void* y, cudaStream_t stream) {
  if (!conv3d_gather_supported(d)) {
    set_error("gather-fed implicit GEMM does not support this convolution");
    return PV_ERR_UNSUPPORTED;
  }
  EncodeTiledFn encode = get_encode_fn();
  if (!encode) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return PV_ERR_CUDA; }
  const int sm_count = current_sm_count();
  if (sm_count <= 0) { set_error("cannot query the SM count of the current device"); return PV_ERR_CUDA; }
  GatherParams P;
  memset(&P, 0, sizeof(P));
  P.N = d->N; P.Ti = d->Ti; P.Hi = d->Hi; P.Wi = d->Wi; P.To = d->To; P.Ho = d->Ho; P.Wo = d->Wo;
  P.st = d->st; P.sh = d->sh; P.sw = d->sw; P.pt = d->pt; P.ph = d->ph; P.pw = d->pw;
  P.gbytes = d->Ci == 4 ? 8 : 16;
  const int upt = d->Ci * 2 / P.gbytes;
  const int taps = d->kt * d->kh * d->kw;
  P.units_total = taps * upt;
  P.upt = upt; P.taps = taps;
  P.upk = 128 / P.gbytes;
  P.num_kb = (P.units_total + P.upk - 1) / P.upk;
  P.x_row_stride = d->x_row_stride;
  P.M = (long long)d->N * d->To * d->Ho * d->Wo;
  P.m_tiles = (int)cdiv(P.M, GG_BM);
  P.Co = d->Co;
  for (int it = 0; it < d->kt; ++it)
    for (int ih = 0; ih < d->kh; ++ih)
      for (int iw = 0; iw < d->kw; ++iw) {
        const int tap = (it * d->kh + ih) * d->kw + iw;
        const int dt = it * d->dt, dh = ih * d->dh, dw = iw * d->dw;
        const long long off = (((long long)dt * d->Hi + dh) * d->Wi + dw) * d->x_row_stride;
        for (int q = 0; q < upt; ++q) {
          const int u = tap * upt + q;
          const long long o = off + (long long)q * (P.gbytes / 2);
          if (o > 0x7fffffffll) { set_error("gather offset overflow"); return PV_ERR_UNSUPPORTED; }
          P.unit_off[u] = (int)o;
          P.unit_d[u] = (unsigned)dt | ((unsigned)dh << 8) | ((unsigned)dw << 16) | ((unsigned)tap << 24);
        }
      }
  {
    const int co16 = (int)cdiv(d->Co, 16) * 16;
    int bn = round_block_n(co16);   // a wgmma width, <= 128
    // keep a few hundred tiles in flight for small layers (several N tiles must be multiples of 64)
    while (bn > 64 && (long long)P.m_tiles * cdiv(d->Co, bn) < 2 * sm_count && (bn / 2) % 64 == 0) bn /= 2;
    P.block_n = bn;
    P.n_tiles = (int)cdiv(d->Co, bn);
  }
  P.epi.block_n = P.block_n;
  P.epi.Co = d->Co;
  P.epi.rows = GG_BM;
  P.epi.act = d->act;
  P.epi.has_residual = d->has_residual;
  P.epi.nbuf = EPI_MAX_BUFS;
  epi_set_addend(P.epi, d);
  for (int m = 0; m < 4; ++m) {      // output as [Co, M, 1, 1, 1]: a row's position is its GEMM row
    P.epi.o_ext[m] = m == 0 ? (int)P.M : 1;
    P.epi.o_box[m] = m == 0 ? GG_BM : 1;
    P.epi.o_pos[m] = m == 0 ? 1 : 0;
  }
  const int stage_bytes = GG_A_BYTES + P.block_n * GG_BK * 2;
  {
    int st = (227 * 1024 - 2048 - 2048 /*static tables*/ - epi_smem_bytes(P.epi.nbuf) - 512) / stage_bytes;
    if (st > 16) st = 16;
    if (st < 2) { set_error("gather: not enough smem stages"); return PV_ERR_UNSUPPORTED; }
    P.nprod = st < GG_PROD_WARPS ? st : GG_PROD_WARPS;
    P.stages = st;
  }
  const size_t smem_bytes = (size_t)P.stages * stage_bytes + 2048 + epi_smem_bytes(P.epi.nbuf) + 8 * (2 * P.stages) + 16;
  for (int pass = 0; pass < 2; ++pass) {     // output / residual as [Co, M, 1, 1, 1]
    if (pass == 1 && !d->has_residual) break;
    const long long rs = pass == 0 ? d->y_row_stride : d->res_row_stride;
    void* base = pass == 0 ? y : const_cast<void*>(residual);
    cuuint64_t gdim[5] = {(cuuint64_t)d->Co, (cuuint64_t)P.M, 1, 1, 1};
    cuuint64_t gstr[4] = {(cuuint64_t)rs * 2, (cuuint64_t)rs * 2 * (cuuint64_t)P.M, (cuuint64_t)rs * 2 * (cuuint64_t)P.M,
                          (cuuint64_t)rs * 2 * (cuuint64_t)P.M};
    cuuint32_t box[5] = {64, GG_BM, 1, 1, 1}, estr[5] = {1, 1, 1, 1, 1};
    CUresult cr = encode(pass == 0 ? &P.epi.y_map : &P.epi.r_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, base, gdim, gstr,
                         box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(gather %s) failed: %d", pass ? "R" : "Y", (int)cr); return PV_ERR_CUDA; }
  }
  {
    const long long kpad = (long long)cdiv((long long)taps * d->Ci, 64) * 64;
    cuuint64_t gdim[2] = {(cuuint64_t)kpad, (cuuint64_t)d->Co};
    cuuint64_t gstr[1] = {(cuuint64_t)kpad * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)P.block_n}, estr[2] = {1, 1};
    CUresult cr = encode(&P.b_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)w, gdim, gstr, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(B, gather) failed: %d", (int)cr); return PV_ERR_CUDA; }
  }
  const long long total_tiles = (long long)P.m_tiles * P.n_tiles;
  if (total_tiles == 0) return PV_OK;
  const int grid = (int)(total_tiles < sm_count ? total_tiles : sm_count);
  {
    // launched with the programmatic-stream-serialization attribute (PDL)
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(GG_THREADS);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    const __half* xh = (const __half*)x;
#define PV_GG_LAUNCH(BN)                                                                                 \
  PV_OPT_IN_SMEM(conv3d_igemm_gather_kernel<BN>, 225 * 1024);                                            \
  PV_CUDA_OK(cudaLaunchKernelEx(&cfg, conv3d_igemm_gather_kernel<BN>, P, xh, scale, bias));              \
  PV_LAUNCH_OK("conv3d_igemm_gather_kernel<" #BN ">");
    switch (P.block_n) {
      case 16: PV_GG_LAUNCH(16) break;
      case 32: PV_GG_LAUNCH(32) break;
      case 64: PV_GG_LAUNCH(64) break;
      default: PV_GG_LAUNCH(128) break;
    }
#undef PV_GG_LAUNCH
  }
  return PV_OK;
}

}  // namespace pv

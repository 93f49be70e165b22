// Fused epilogue shared by the implicit-GEMM kernels (TMA-fed, gather-fed, stem rows).
//
// Two consumer warpgroups (256 threads) hold a 128-row x BN tile of fp32 accumulators in wgmma fragments
// (warpgroup g: rows [64 g, 64 g + 64)) -> y = act(acc*scale+bias (+residual)) (+ addend[n][t][c]) -> f16 -> 128B-swizzled shared
// staging -> TMA tensor store.  The residual tile is brought in by a TMA tensor load into the SAME staging buffer
// (requested before the tile's main loop, so its latency hides behind the MMAs) and updated in place, so both the
// residual read and the output write are full-line bulk transfers issued by one thread, with the tile-edge and
// channel-tail clipping done by the TMA unit.  Staging is 32 KiB = two [128 rows x 64 f16] swizzled sub-tiles
// (BN <= 128).
#pragma once
#include "pv_common.cuh"
#include "pv_sm90.cuh"

namespace pv {
namespace sm90 {

constexpr int EPI_STAGING_BYTES = 2 * 128 * 128;
constexpr int EPI_THREADS = 256;       // two consumer warpgroups
constexpr int EPI_BAR_ID = 1;          // named barrier of the consumer warpgroups (0 is __syncthreads)
constexpr int MAX_BN = 128;

struct EpiParams {
  CUtensorMap y_map;    // output  [Co, d1, d2, d3, d4], box [64, b1, b2, b3, b4], SWIZZLE_128B
  CUtensorMap r_map;    // residual, same geometry
  int block_n, Co, rows, act, has_residual;
  // post-activation addend (pv_conv3d_desc.addend; nullptr = none): a[n * add_n + t * add_t + add_off + c]
  const __half* addend;
  long long add_n, add_t;
  int add_off;
  // y_map's outer dims d1..d4: extents, tile box and the flat output position (n, t, h, w) of one step along each;
  // a staged row -> its output position -> (n, t) = (pos / hw / To, pos / hw % To)
  int o_ext[4], o_box[4], o_pos[4];
  int hw, To;        // a conv output has fewer than 2^31 positions (checked by every launch that takes an addend)
};

// Host: fill the addend fields from the descriptor (o_ext / o_box / o_pos are set by the launch, which knows its map).
inline void epi_set_addend(EpiParams& E, const pv_conv3d_desc* d) {
  E.addend = static_cast<const __half*>(d->addend);
  E.add_n = d->add_n_stride;
  E.add_t = d->add_t_stride;
  E.add_off = d->add_ch_off;
  E.hw = d->Ho * d->Wo;
  E.To = d->To;
}

__device__ __forceinline__ void tma_store_5d(const void* tmap, uint32_t src, int c0, int c1, int c2, int c3,
                                             int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(tmap)),
      "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void epi_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

template <int ACT>
__device__ __forceinline__ float act_t(float x) {
  if (ACT == PV_ACT_RELU) return fmaxf(x, 0.f);
  if (ACT == PV_ACT_NONE) return x;
  return apply_act(x, ACT);
}

// Tile start (consumer thread 0 only): the staging buffer is free once the previous tile's bulk store has read it;
// then the residual tile of THIS tile is requested into it.  The named barrier in epilogue_tile publishes both.
__device__ __forceinline__ void epilogue_begin(const EpiParams& E, uint32_t staging, uint32_t res_bar, int n0, int c1,
                                               int c2, int c3, int c4) {
  tma_store_wait_read0();
  if (E.has_residual) {
    const int nsub = (E.block_n + 63) >> 6;
    mbar_arrive_expect_tx(res_bar, (uint32_t)(nsub * E.rows * 128));
    for (int s = 0; s < nsub; ++s)
      tma_load_5d(staging + (uint32_t)s * 16384u, &E.r_map, res_bar, n0 + s * 64, c1, c2, c3, c4);
  }
}

// wgmma m64nBN fragment of consumer thread `ctid` (0..255): register 4 j + 2 i + e holds row
// 64 (ctid / 128) + 16 ((ctid / 32) & 3) + (lane / 4) + 8 i, column 8 j + 2 (lane % 4) + e.
template <int BN, int ACT, bool RES>
__device__ __forceinline__ void epi_math(const float (&d)[BN / 2], uint8_t* stg, const float* __restrict__ scale,
                                         const float* __restrict__ bias, int Co, int n0, int ctid) {
  const int lane = ctid & 31;
  const int row0 = 64 * (ctid >> 7) + 16 * ((ctid >> 5) & 3) + (lane >> 2);
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = 8 * j + cq;
    const int c = n0 + col;
    float2 s = make_float2(0.f, 0.f), b = make_float2(0.f, 0.f);    // zeros beyond Co keep pad lanes at zero
    if (c < Co) {
      s = __ldg(reinterpret_cast<const float2*>(scale + c));
      b = __ldg(reinterpret_cast<const float2*>(bias + c));
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = row0 + 8 * i;
      // sub-tile (col / 64), row, swizzled 16-byte cell, 4-byte half2 inside the cell
      __half2* cell = reinterpret_cast<__half2*>(stg + (col >> 6) * 16384 + row * 128 +
                                                 ((((col & 63) >> 3) ^ (row & 7)) << 4) + cq * 2);
      float f0 = fmaf(d[4 * j + 2 * i], s.x, b.x), f1 = fmaf(d[4 * j + 2 * i + 1], s.y, b.y);
      if (RES) {
        const float2 r = __half22float2(*cell);
        f0 += r.x;
        f1 += r.y;
      }
      *cell = __floats2half2_rn(act_t<ACT>(f0), act_t<ACT>(f1));
    }
  }
}

template <int BN, int ACT>
__device__ __forceinline__ void epi_math_res(bool res, const float (&d)[BN / 2], uint8_t* stg, const float* scale,
                                             const float* bias, int Co, int n0, int ctid) {
  if (res) epi_math<BN, ACT, true>(d, stg, scale, bias, Co, n0, ctid);
  else epi_math<BN, ACT, false>(d, stg, scale, bias, Co, n0, ctid);
}

// Post-activation addend on the staged f16 tile: a second pass over the staging buffer once epi_math has written it,
// one 16-byte cell (8 channels of one row) per step.  It runs after the fragment math, so the accumulator-holding code
// and its register allocation are those of a launch without an addend.  Rows past the tensor edge (clipped by the TMA
// store) and cells at or past Co are skipped.
template <int BN>
__device__ __forceinline__ void epi_addend(const EpiParams& E, uint8_t* stg, int ctid, int n0, int c1, int c2, int c3,
                                           int c4) {
  constexpr int CELLS = BN / 8;                 // a thread keeps one 8-channel column and walks rows
  const int col = (ctid % CELLS) * 8;
  if (n0 + col >= E.Co) return;
  const __half* acol = E.addend + E.add_off + n0 + col;
#pragma unroll 1
  for (int row = ctid / CELLS; row < E.rows; row += EPI_THREADS / CELLS) {
    unsigned r = row, pos = 0;
    bool inside = true;
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const unsigned v = (unsigned)(m == 0 ? c1 : m == 1 ? c2 : m == 2 ? c3 : c4) + r % (unsigned)E.o_box[m];
      r /= (unsigned)E.o_box[m];
      inside &= v < (unsigned)E.o_ext[m];
      pos += v * (unsigned)E.o_pos[m];
    }
    if (!inside) continue;
    const unsigned nt = pos / (unsigned)E.hw;
    const unsigned n = nt / (unsigned)E.To, t = nt - n * (unsigned)E.To;
    const uint4 av = __ldg(reinterpret_cast<const uint4*>(acol + n * E.add_n + t * E.add_t));
    uint4* cell = reinterpret_cast<uint4*>(stg + (col >> 6) * 16384 + row * 128 + ((((col & 63) >> 3) ^ (row & 7)) << 4));
    uint4 sv = *cell;
    __half2* s2 = reinterpret_cast<__half2*>(&sv);
    const __half2* a2 = reinterpret_cast<const __half2*>(&av);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = __half22float2(s2[k]), g = __half22float2(a2[k]);
      s2[k] = __floats2half2_rn(f.x + g.x, f.y + g.y);
    }
    *cell = sv;
  }
}

// Called by the 256 consumer threads once the accumulators of the tile are complete (wgmma_wait<0>).
// (c1..c4): tile origin in the store tensor map's outer dims; n0: first output channel of the tile.
template <int BN>
__device__ __forceinline__ void epilogue_tile(const EpiParams& E, const float* __restrict__ scale,
                                              const float* __restrict__ bias, const float (&d)[BN / 2],
                                              uint32_t staging, uint8_t* staging_gen, uint32_t res_bar,
                                              uint32_t& res_phase, int ctid, int n0, int c1, int c2, int c3, int c4) {
  epi_bar_sync(EPI_BAR_ID, EPI_THREADS);     // staging free (thread 0 waited for the previous store's read)
  if (E.has_residual) {
    mbar_wait(res_bar, res_phase);
    res_phase ^= 1u;
  }
  switch (E.act) {
    case PV_ACT_RELU: epi_math_res<BN, PV_ACT_RELU>(E.has_residual, d, staging_gen, scale, bias, E.Co, n0, ctid); break;
    case PV_ACT_NONE: epi_math_res<BN, PV_ACT_NONE>(E.has_residual, d, staging_gen, scale, bias, E.Co, n0, ctid); break;
    case PV_ACT_SWISH: epi_math_res<BN, PV_ACT_SWISH>(E.has_residual, d, staging_gen, scale, bias, E.Co, n0, ctid); break;
    case PV_ACT_GELU: epi_math_res<BN, PV_ACT_GELU>(E.has_residual, d, staging_gen, scale, bias, E.Co, n0, ctid); break;
    default: epi_math_res<BN, PV_ACT_SIGMOID>(E.has_residual, d, staging_gen, scale, bias, E.Co, n0, ctid); break;
  }
  if (E.addend) {
    epi_bar_sync(EPI_BAR_ID, EPI_THREADS);   // the cells of a row were written by other threads
    epi_addend<BN>(E, staging_gen, ctid, n0, c1, c2, c3, c4);
  }
  // publish the staged tile to the async proxy and store it
  fence_proxy_async_smem();
  epi_bar_sync(EPI_BAR_ID, EPI_THREADS);
  if (ctid == 0) {
    const int nsub = (E.block_n + 63) >> 6;
    for (int s = 0; s < nsub; ++s) tma_store_5d(&E.y_map, staging + (uint32_t)s * 16384u, n0 + s * 64, c1, c2, c3, c4);
    tma_store_commit();
  }
}

// Tile widths with a wgmma instantiation; the host rounds the channel count up to one of them.
__host__ __device__ inline int round_block_n(int co) { return co <= 16 ? 16 : (co <= 32 ? 32 : (co <= 64 ? 64 : 128)); }

}  // namespace sm90
}  // namespace pv

// Fused epilogue shared by the implicit-GEMM kernels (TMA-fed, gather-fed, stem rows).
//
// Two consumer warpgroups (256 threads) hold a 128-row x BN tile of fp32 accumulators in wgmma fragments
// (warpgroup g: rows [64 g, 64 g + 64)) -> y = act(acc*scale+bias (+residual)) (+ addend[n][t][c]) -> f16 -> 128B-swizzled shared
// staging -> TMA tensor store.  The residual tile is brought in by a TMA tensor load into the staging buffer and
// updated in place, so both the residual read and the output write are full-line bulk transfers, with the tile-edge
// and channel-tail clipping done by the TMA unit.  One staging buffer is 32 KiB = two [128 rows x 64 f16] swizzled
// sub-tiles (BN <= 128).
//
// Pipelining: a CTA's k-th tile uses staging buffer S[k % nbuf] (nbuf = 2, or 1 where shared memory allows only
// one).  The consumers never touch the bulk-copy machinery; one elected lane of the epilogue DMA warp
// (epilogue_dma) issues every residual load and output store, and two mbarriers per buffer hand it back and forth:
//   epi_ready[b]  buffer free and its residual landed: the DMA warp's arrive (with expect_tx of the residual bytes)
//   epi_full[b]   tile staged: one arrive per consumer warp, after every thread's fence.proxy.async
// Per tile the DMA warp waits epi_full, stores, waits until the store has read the buffer out, then loads the
// residual of the tile nbuf further on into it.  So the store of tile k drains while the consumers compute tile
// k + 1, and each residual load is issued a whole tile ahead of its use.
#pragma once
#include "pv_common.cuh"
#include "pv_sm90.cuh"

namespace pv {
namespace sm90 {

constexpr int EPI_STAGING_BYTES = 2 * 128 * 128;   // one staging buffer
constexpr int EPI_MAX_BUFS = 2;
constexpr int EPI_BARS = 2 * EPI_MAX_BUFS;         // epi_ready[2], epi_full[2]
constexpr int EPI_THREADS = 256;       // two consumer warpgroups
constexpr int EPI_BAR_ID = 1;          // named barrier of the consumer warpgroups (0 is __syncthreads)
constexpr int MAX_BN = 128;

// Host: shared-memory bytes of the epilogue with `nbuf` staging buffers and its barriers.
constexpr int epi_smem_bytes(int nbuf) { return nbuf * EPI_STAGING_BYTES + 8 * EPI_BARS; }

struct EpiParams {
  CUtensorMap y_map;    // output  [Co, d1, d2, d3, d4], box [64, b1, b2, b3, b4], SWIZZLE_128B
  CUtensorMap r_map;    // residual, same geometry
  int block_n, Co, rows, act, has_residual;
  int nbuf;             // staging buffers (1 or 2)
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

// The fragment math has five instances: ReLU, none, Swish, GELU, and EPI_ACT_RARE for the rarely fused sigmoid and
// HardSwish, which picks between them at run time (act).  A sixth instance pushes the <128, *> kernels past their
// 168-register cap into spills (DESIGN.md section 1).
constexpr int EPI_ACT_RARE = -1;

template <int ACT>
__device__ __forceinline__ float act_t(float x, int act) {
  if (ACT == PV_ACT_RELU) return fmaxf(x, 0.f);
  if (ACT == PV_ACT_NONE) return x;
  if (ACT == EPI_ACT_RARE) return act == PV_ACT_HSWISH ? hswish(x) : apply_act(x, PV_ACT_SIGMOID);
  return apply_act(x, ACT);
}

// Staging buffers S[b] (1024-aligned, EPI_STAGING_BYTES apart) and the epilogue's mbarriers in shared memory.
struct EpiSmem {
  uint32_t staging;       // S[0]
  uint8_t* staging_gen;   // S[0], generic address
  uint32_t bars;          // epi_ready[0..1], epi_full[0..1]
  __device__ __forceinline__ uint32_t buf(int b) const { return staging + (uint32_t)b * EPI_STAGING_BYTES; }
  __device__ __forceinline__ uint8_t* buf_gen(int b) const { return staging_gen + b * EPI_STAGING_BYTES; }
  __device__ __forceinline__ uint32_t ready(int b) const { return bars + 8u * b; }
  __device__ __forceinline__ uint32_t full(int b) const { return bars + 8u * (EPI_MAX_BUFS + b); }
  __device__ __forceinline__ void init() const {   // one thread, before the kernel's fence_mbar_init
    for (int b = 0; b < EPI_MAX_BUFS; ++b) {
      mbar_init(ready(b), 1);                  // the DMA warp's (expect_tx) arrive
      mbar_init(full(b), EPI_THREADS / 32);    // one arrive per consumer warp
    }
  }
};

// The epilogue DMA warp: called by the whole warp after the kernel's griddepcontrol.wait (the residual may be
// written by the previous kernel).  coords(tile, n0, c) gives a tile's first output channel and its origin in the
// outer dims of the store / residual maps; the CTA's tiles are blockIdx.x, blockIdx.x + gridDim.x, ...
template <class Coords>
__device__ __forceinline__ void epilogue_dma(const EpiParams& E, const EpiSmem& S, int total_tiles, Coords coords) {
  if (!elect_one()) return;
  const int nbuf = E.nbuf;
  const int nsub = (E.block_n + 63) >> 6;
  auto fill = [&](int tile, int b) {   // buffer b is free: bring in the tile's residual (if any) and hand it over
    if (E.has_residual) {
      int n0, c[4];
      coords(tile, n0, c);
      mbar_arrive_expect_tx(S.ready(b), (uint32_t)(nsub * E.rows * 128));
      for (int s = 0; s < nsub; ++s)
        tma_load_5d(S.buf(b) + (uint32_t)s * 16384u, &E.r_map, S.ready(b), n0 + s * 64, c[0], c[1], c[2], c[3]);
    } else {
      mbar_arrive(S.ready(b));
    }
  };
  for (int b = 0; b < nbuf; ++b) {
    const int tile = (int)blockIdx.x + b * (int)gridDim.x;
    if (tile < total_tiles) fill(tile, b);
  }
  int b = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    mbar_wait(S.full(b), phase);
    int n0, c[4];
    coords(tile, n0, c);
    for (int s = 0; s < nsub; ++s)
      tma_store_5d(&E.y_map, S.buf(b) + (uint32_t)s * 16384u, n0 + s * 64, c[0], c[1], c[2], c[3]);
    tma_store_commit();
    tma_store_wait_read0();   // the store has read S[b]: it may be refilled while the write drains to HBM
    const long long next = (long long)tile + (long long)nbuf * gridDim.x;
    if (next < total_tiles) fill((int)next, b);
    if (++b == nbuf) { b = 0; phase ^= 1u; }
  }
  tma_store_wait_all();       // smem must outlive the bulk stores
}

// wgmma m64nBN fragment of consumer thread `ctid` (0..255): register 4 j + 2 i + e holds row
// 64 (ctid / 128) + 16 ((ctid / 32) & 3) + (lane / 4) + 8 i, column 8 j + 2 (lane % 4) + e.
template <int BN, int ACT, bool RES>
__device__ __forceinline__ void epi_math(const float (&d)[BN / 2], uint8_t* stg, const float* __restrict__ scale,
                                         const float* __restrict__ bias, int Co, int n0, int ctid, int act) {
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
      *cell = __floats2half2_rn(act_t<ACT>(f0, act), act_t<ACT>(f1, act));
    }
  }
}

template <int BN, int ACT>
__device__ __forceinline__ void epi_math_res(bool res, const float (&d)[BN / 2], uint8_t* stg, const float* scale,
                                             const float* bias, int Co, int n0, int ctid, int act) {
  if (res) epi_math<BN, ACT, true>(d, stg, scale, bias, Co, n0, ctid, act);
  else epi_math<BN, ACT, false>(d, stg, scale, bias, Co, n0, ctid, act);
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
// (buf, phase): the tile's staging buffer and the parity of its barriers, both start at 0 and are advanced here.
template <int BN>
__device__ __forceinline__ void epilogue_tile(const EpiParams& E, const EpiSmem& S, int& buf, uint32_t& phase,
                                              const float* __restrict__ scale, const float* __restrict__ bias,
                                              const float (&d)[BN / 2], int ctid, int n0, int c1, int c2, int c3,
                                              int c4) {
  mbar_wait(S.ready(buf), phase);            // buffer free, residual landed
  uint8_t* staging_gen = S.buf_gen(buf);
  switch (E.act) {
    case PV_ACT_RELU: epi_math_res<BN, PV_ACT_RELU>(E.has_residual, d, staging_gen, scale, bias, E.Co, n0, ctid, E.act); break;
    case PV_ACT_NONE: epi_math_res<BN, PV_ACT_NONE>(E.has_residual, d, staging_gen, scale, bias, E.Co, n0, ctid, E.act); break;
    case PV_ACT_SWISH: epi_math_res<BN, PV_ACT_SWISH>(E.has_residual, d, staging_gen, scale, bias, E.Co, n0, ctid, E.act); break;
    case PV_ACT_GELU: epi_math_res<BN, PV_ACT_GELU>(E.has_residual, d, staging_gen, scale, bias, E.Co, n0, ctid, E.act); break;
    // PV_ACT_SIGMOID, PV_ACT_HSWISH; the entry points reject every other code (act_known)
    default: epi_math_res<BN, EPI_ACT_RARE>(E.has_residual, d, staging_gen, scale, bias, E.Co, n0, ctid, E.act); break;
  }
  if (E.addend) {
    epi_bar_sync(EPI_BAR_ID, EPI_THREADS);   // the cells of a row were written by other threads
    epi_addend<BN>(E, staging_gen, ctid, n0, c1, c2, c3, c4);
  }
  // publish the staged tile to the async proxy and hand it to the DMA warp
  fence_proxy_async_smem();
  __syncwarp();
  mbar_arrive_if(S.full(buf), (ctid & 31) == 0);
  if (++buf == E.nbuf) { buf = 0; phase ^= 1u; }
}

// Tile widths with a wgmma instantiation; the host rounds the channel count up to one of them.
__host__ __device__ inline int round_block_n(int co) { return co <= 16 ? 16 : (co <= 32 ? 32 : (co <= 64 ? 64 : 128)); }

}  // namespace sm90
}  // namespace pv

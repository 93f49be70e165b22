// Implicit-GEMM 3-D convolution on Hopper (sm_90a) tensor cores.
//
//   D[m][co] = sum_{tap,ci} X[pos(m) + tap][ci] * Wt[co][tap][ci]        (fp32 accumulate in registers)
//   y        = act(D * scale[co] + bias[co] (+ residual))               (fused epilogue)
//
// * Activations are NDHWC f16.  The GEMM-M tile (128 rows) is a BOX of output positions
//   (b0 x b1 x b2 x b3 over the W/H/T/N-like dims, merged where the kernel is trivial), so for
//   every filter tap the A operand is ONE TMA tiled load of box [64 ch, b0, b1, b2, b3] at
//   shifted coordinates; TMA's out-of-bounds zero fill implements the convolution padding and
//   the channel tail (Ci % 64 != 0).  Strided convolutions use one tensor map per stride-parity
//   class (base pointer offset + multiplied global strides), so only documented tiled-mode
//   features are relied on.
// * B operand (packed weights, K-major rows of taps*ci_pad64) is a 2-D TMA load [64, BLOCK_N].
// * Both land in swizzled shared memory and feed wgmma (m64nBNk16) via shared-memory descriptors.
// * Warp-specialised persistent kernel: one producer warpgroup (TMA loads of the k-blocks dealt to up to 3 warps,
//   warp 11 the epilogue DMA warp) and two consumer warpgroups; consumer warpgroup g issues the wgmma of tile rows
//   [64 g, 64 g + 64), keeps their fp32 accumulators in registers and runs the fused epilogue on them.  smem ring of
//   `stages` {A,B} slots with full/empty mbarriers; one wgmma group stays in flight while the previous stage is
//   released.
#include "pv_common.cuh"
#include "pv_sm90.cuh"
#include "pv_epilogue.cuh"

#include <mutex>
#include <stdlib.h>
#include <string.h>

namespace pv {

using namespace sm90;

constexpr int IG_BM = 128;        // two consumer warpgroups x wgmma M = 64
constexpr int IG_MAX_TAPS = 64;
constexpr int IG_MAX_MAPS = 8;
constexpr int IG_PROD_WARPS = 4;   // warps 8..10: TMA loads (one elected lane each, k-blocks round-robin); 11: epilogue DMA
constexpr int IG_CONS_WARPS = 8;   // warps 0..7: two consumer warpgroups
constexpr int IG_THREADS = (IG_CONS_WARPS + IG_PROD_WARPS) * 32;   // 384
constexpr int IG_DMA_WARP = IG_CONS_WARPS + IG_PROD_WARPS - 1;

struct IgemmParams {
  CUtensorMap a_maps[IG_MAX_MAPS];
  CUtensorMap b_map;
  // tiling over the 4 merged output dims (0 = innermost)
  int O[4];        // output extents
  int box[4];      // tile box
  int nt[4];       // tiles per dim
  int rows;        // box[0]*box[1]*box[2]*box[3] (<= 128)
  int n_tiles, m_tiles;
  int block_n;
  int Co;
  int taps, num_kc;
  int kbytes;      // bytes of K per smem row and pipeline stage: 128 (64 ch, SW128) | 64 | 32 (window mode)
  int stages;
  int G, cpt;       // k-blocks per pipeline stage (chunk, 128 / kbytes: 64 K elements), chunks per tile
  int split_ab;     // producer warps that share the loads of a chunk (2 or 3)
  EpiParams epi;
  signed char tap_q[IG_MAX_TAPS][4];
  unsigned char tap_map[IG_MAX_TAPS];
};

// KB = kbytes.  A stage always holds 64 K elements (G = 128 / KB k-blocks, four k16 steps), so the wgmma sequence of a
// stage is unrolled at compile time: no branch between the wgmma of a stage keeps them asynchronous.  The last chunk of
// a tile is padded with k-blocks whose TMA loads lie entirely out of bounds (zero fill).
//
// GROUPED (grouped convolution, see conv3d_group_span): the output channels form spans of span_tiles N tiles, and the
// N tiles of span s read input channels [s * K_span, (s + 1) * K_span) with K_span = num_kc * 64, i.e. the A box of
// channel chunk kc starts at channel c0 + kc * 64 with c0 = (n_tile / span_tiles) * K_span.  The packed weights of a
// span are block-diagonal over its groups (zeros elsewhere), so the B operand, the epilogue and the stores are those of
// the dense kernel.  Grouped mode runs with 128-byte k-blocks only (G = 1): no padding k-block is ever loaded, whose
// channel coordinate num_kc * 64 would lie inside the next span.
template <int BN, int KB, bool GROUPED>
__device__ __forceinline__ void igemm_body(const IgemmParams& P, const float* __restrict__ scale,
                                           const float* __restrict__ bias, int span_tiles) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const int stages = P.stages;
  constexpr int G = 128 / KB, K16 = KB / 32;
  const uint32_t a_bytes = (uint32_t)IG_BM * KB;
  const uint32_t b_bytes = (uint32_t)BN * KB;
  const uint32_t stage_bytes = (uint32_t)G * (a_bytes + b_bytes);   // [G x A k-block][G x B k-block]
  constexpr int k_elems = KB / 2;
  // epilogue staging buffers (1024-aligned) and the barriers live after the tile ring
  const uint32_t staging_off = (uint32_t)((stages * stage_bytes + 1023u) & ~1023u);
  const uint32_t staging = smem_base + staging_off;
  const uint32_t bar_base = staging + (uint32_t)(P.epi.nbuf * EPI_STAGING_BYTES);
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (stages + s); };
  const EpiSmem epi{staging, smem_gen + staging_off, bar_base + 8u * (2 * stages)};

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    prefetch_tmap(&P.b_map);
    prefetch_tmap(&P.a_maps[0]);
    prefetch_tmap(&P.epi.y_map);
    for (int s = 0; s < stages; ++s) {
      mbar_init(full_bar(s), 1);                // producer warp 0's expect_tx arrive
      mbar_init(empty_bar(s), IG_CONS_WARPS);   // one arrive per consumer warp
    }
    epi.init();
    fence_mbar_init();
  }
  __syncthreads();
  // Programmatic dependent launch: everything above (barrier init, descriptor prefetch) overlaps the tail of
  // the previous kernel in the stream / graph; its results are only touched below.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  const int total_tiles = P.n_tiles * P.m_tiles;
  const int num_kb = P.taps * P.num_kc;
  // tile -> (n tile index, merged output coordinates of its 128-row box)
  auto tile_coords = [&](int tile, int& n_tile, int (&o)[4]) {
    n_tile = tile % P.n_tiles;
    int mt = tile / P.n_tiles;
#pragma unroll
    for (int i = 0; i < 4; ++i) { o[i] = (mt % P.nt[i]) * P.box[i]; mt /= P.nt[i]; }
  };

  if (warp == IG_DMA_WARP) {
    epilogue_dma(P.epi, epi, total_tiles, [&](int tile, int& n0, int (&c)[4]) {
      int n_tile;
      tile_coords(tile, n_tile, c);
      n0 = n_tile * BN;
    });
  } else if (warp >= IG_CONS_WARPS) {
    // ================================ TMA producers =========================================
    // The loads of a chunk (2 per k-block: A and B) are dealt round-robin to `nsplit` producer warps: one
    // issuing thread sustains only a limited rate of bulk-tensor loads.  Warp 0 of the group alone arrives on
    // the full barrier with the expected bytes of the WHOLE chunk; the other warps' loads may complete before
    // that arrive (the transaction count goes negative, the phase cannot complete without the arrive).
    const int pw = warp - IG_CONS_WARPS;
    const int nsplit = P.split_ab;
    if (pw < nsplit) {
      int stage = 0;
      uint32_t phase = 0;
      const uint32_t tx_bytes = (uint32_t)P.rows * KB + b_bytes;
      const int num_kc = P.num_kc, cpt = P.cpt;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int n_tile, o[4];
        tile_coords(tile, n_tile, o);
        const int n0 = n_tile * BN;
        const int c0 = GROUPED ? (n_tile / span_tiles) * num_kc * k_elems : 0;   // first input channel of the span
        int tap = 0, kc = 0;                  // (tap, channel chunk) of the next k-block, stepped without a divide
        for (int ch = 0; ch < cpt; ++ch) {
          const int kb0 = ch * G;
          const int nsub = min(G, num_kb - kb0);
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t st_base = smem_base + (uint32_t)stage * stage_bytes;
          if (elect_one()) {
            if (pw == 0) mbar_arrive_expect_tx(full_bar(stage), (uint32_t)G * tx_bytes);   // out-of-bounds boxes count in full
            int tp = tap, kk = kc;
            for (int j = 0; j < G; ++j) {
              const bool pad = j >= nsub;       // padding k-block: channel coordinate past the tensor -> zeros
              const int t = pad ? P.taps - 1 : tp;
              if ((2 * j) % nsplit == pw) {
                const void* amap = &P.a_maps[P.tap_map[t]];
                tma_load_5d(st_base + (uint32_t)j * a_bytes, amap, full_bar(stage),
                            (pad ? num_kc * k_elems : kk * k_elems) + c0,
                            o[0] + P.tap_q[t][0], o[1] + P.tap_q[t][1], o[2] + P.tap_q[t][2], o[3] + P.tap_q[t][3]);
              }
              if ((2 * j + 1) % nsplit == pw)
                tma_load_2d(st_base + (uint32_t)G * a_bytes + (uint32_t)j * b_bytes, &P.b_map, full_bar(stage),
                            (kb0 + j) * k_elems, n0);
              if (++kk == num_kc) { kk = 0; ++tp; }
            }
          }
          __syncwarp();
          for (int j = 0; j < nsub; ++j) { if (++kc == num_kc) { kc = 0; ++tap; } }
          if (++stage == stages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ================================ consumers: wgmma + epilogue ===========================
    const int ctid = threadIdx.x;
    const uint32_t a_row_off = (uint32_t)(ctid >> 7) * 64u * (uint32_t)KB;   // this warpgroup's 64 rows
    const int cpt = P.cpt;
    int stage = 0, epi_buf = 0;
    uint32_t phase = 0, epi_phase = 0;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int n_tile, o[4];
      tile_coords(tile, n_tile, o);
      int prev = -1;
      for (int ch = 0; ch < cpt; ++ch) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t st_base = smem_base + (uint32_t)stage * stage_bytes;
        acc_fence(acc);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < G; ++j) {
          const uint64_t a_desc = make_kmajor_desc(st_base + (uint32_t)j * a_bytes + a_row_off, KB);
          const uint64_t b_desc = make_kmajor_desc(st_base + (uint32_t)G * a_bytes + (uint32_t)j * b_bytes, KB);
#pragma unroll
          for (int k = 0; k < K16; ++k) {
            // advance 16 elements (32 B) along K inside the swizzle row: +2 in (addr>>4)
            Wgmma<BN>::mma(acc, a_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k), (ch | j | k) != 0 ? 1u : 0u);
          }
        }
        wgmma_commit();
        acc_fence(acc);
        wgmma_wait<1>();                          // the previous chunk's wgmma have retired: free its stage
        mbar_arrive_if(empty_bar(prev < 0 ? stage : prev), prev >= 0 && lane == 0);
        prev = stage;
        if (++stage == stages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      acc_fence(acc);
      mbar_arrive_if(empty_bar(prev < 0 ? stage : prev), prev >= 0 && lane == 0);
      epilogue_tile<BN>(P.epi, epi, epi_buf, epi_phase, scale, bias, acc, ctid, n_tile * BN, o[0], o[1], o[2], o[3]);
    }
  }
}

template <int BN, int KB>
__global__ void __launch_bounds__(IG_THREADS, 1)
conv3d_igemm_kernel(const __grid_constant__ IgemmParams P, const float* __restrict__ scale,
                    const float* __restrict__ bias) {
  igemm_body<BN, KB, false>(P, scale, bias, 1);
}

// span_tiles: N tiles per group span (N_span / BN)
template <int BN, int KB>
__global__ void __launch_bounds__(IG_THREADS, 1)
conv3d_igemm_grouped_kernel(const __grid_constant__ IgemmParams P, const float* __restrict__ scale,
                            const float* __restrict__ bias, int span_tiles) {
  igemm_body<BN, KB, true>(P, scale, bias, span_tiles);
}

// =============================================================================================
// Host side: problem reduction, tile search, tensor maps, launch
// =============================================================================================
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  });
  return fn;
}

struct Dim4 {      // one merged spatial dim
  long long I, O;  // input / output extent
  int k, s, p, dil;
  long long stride_bytes;   // byte distance of +1 input index in this dim
  bool nomerge;
};

struct IgemmPlan {
  Dim4 dim[4];
  int ndims;
  int orig2m[4];   // original dim (0=W,1=H,2=T,3=N) -> merged dim index
};

// Window mode (narrow C_in stems): the K axis of one pipeline stage is the contiguous run of
// kw*Ci input elements that one output pixel reads in one (dt,dh) filter row.  The TMA tensor map
// uses OVERLAPPING strides - dim0 = the run (padded to 16/32/64 elements), dim1 = output column
// with byte stride sw*Ci*2 - so one tiled load delivers 128 sliding windows.  The input rows carry
// x_w_pad physical zero pixels on the left (and enough on the right), written by the layout
// conversion, which implements the W padding; H/T padding is TMA out-of-bounds fill as usual.
static bool window_mode(const pv_conv3d_desc* d) { return d->x_w_pad > 0 && d->Ci <= 8; }
// Narrow TMA mode: C_in = 16 / 32 with the weights packed at the un-padded per-tap K extent.  One tap is a
// 32 / 64-byte box row (SWIZZLE_32B / 64B), one k-block per tap, several taps per pipeline stage - fewer
// barrier rounds and no SM instructions for the A operand, which beats the cp.async gather for these
// widths (the gather kernel keeps C_in = 4 / 8 / 24 / 40 / 48 / 56).
bool conv3d_tma_narrow(const pv_conv3d_desc* d) {
  return !window_mode(d) && (d->Ci == 16 || d->Ci == 32) && d->ci_pad64 == d->Ci;
}
// TMA needs a 16-byte aligned base: if the first tap of output column 0 sits at an odd pixel of a
// 4-channel row, the window starts one pixel earlier (the packed weights carry a zero pixel there).
static int window_lead(const pv_conv3d_desc* d) { return (((d->x_w_pad - d->pw) * d->Ci * 2) % 16) ? 1 : 0; }
static int window_elems(const pv_conv3d_desc* d) {
  const int run = (d->kw + window_lead(d)) * d->Ci;
  return run <= 16 ? 16 : (run <= 32 ? 32 : 64);
}

// Reduce (W,H,T,N) to <=4 merged dims: runs of adjacent trivial dims (k=1,s=1,p=0) collapse.
static void reduce_dims(const pv_conv3d_desc* d, IgemmPlan* pl) {
  const long long rs = d->x_row_stride * 2;   // bytes per position
  Dim4 raw[4];
  if (window_mode(d)) {
    const long long wp = d->x_w_phys;
    raw[0] = {d->Wo, d->Wo, 1, 1, 0, 1, (long long)d->sw * rs, true};
    raw[1] = {d->Hi, d->Ho, d->kh, d->sh, d->ph, d->dh, wp * rs, false};
    raw[2] = {d->Ti, d->To, d->kt, d->st, d->pt, d->dt, wp * d->Hi * rs, false};
    raw[3] = {d->N, d->N, 1, 1, 0, 1, wp * d->Hi * d->Ti * rs, false};
  } else {
    raw[0] = {d->Wi, d->Wo, d->kw, d->sw, d->pw, d->dw, rs, false};
    raw[1] = {d->Hi, d->Ho, d->kh, d->sh, d->ph, d->dh, (long long)d->Wi * rs, false};
    raw[2] = {d->Ti, d->To, d->kt, d->st, d->pt, d->dt, (long long)d->Wi * d->Hi * rs, false};
    raw[3] = {d->N, d->N, 1, 1, 0, 1, (long long)d->Wi * d->Hi * d->Ti * rs, false};
  }
  int n = 0;
  for (int i = 0; i < 4; ++i) {
    const bool triv = raw[i].k == 1 && raw[i].s == 1 && raw[i].p == 0 && !raw[i].nomerge;
    if (n > 0) {
      Dim4& prev = pl->dim[n - 1];
      const bool ptriv = prev.k == 1 && prev.s == 1 && prev.p == 0 && !prev.nomerge;
      if (triv && ptriv && prev.stride_bytes * prev.I == raw[i].stride_bytes) {
        prev.I *= raw[i].I;
        prev.O *= raw[i].O;
        pl->orig2m[i] = n - 1;
        continue;
      }
    }
    pl->orig2m[i] = n;
    pl->dim[n++] = raw[i];
  }
  pl->ndims = n;
  for (int i = n; i < 4; ++i)
    pl->dim[i] = {1, 1, 1, 1, 0, 1, pl->dim[n - 1].stride_bytes * pl->dim[n - 1].I, false};
}

static int floordiv(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }

// Group span of a grouped convolution: S = 64 / gcd(Cg_in, 64) consecutive groups, so that the span's K_span = S * Cg_in
// input channels fill whole 64-channel TMA boxes (no box reaches into the next span); N_span = S * Cg_out.  The last
// span may hold fewer groups: it ends at Ci, and TMA out-of-bounds fill covers its tail.  Returns 0 when groups does
// not divide both channel counts.
int conv3d_group_span(const pv_conv3d_desc* d, int* span_groups, int* span_k, int* span_n) {
  if (d->groups < 1 || d->Ci % d->groups || d->Co % d->groups) return 0;
  const int cgi = d->Ci / d->groups, cgo = d->Co / d->groups;
  int a = cgi, b = 64;
  while (b) { const int t = a % b; a = b; b = t; }   // gcd(Cg_in, 64)
  *span_groups = 64 / a;
  *span_k = *span_groups * cgi;
  *span_n = *span_groups * cgo;
  return 1;
}

int conv3d_tcgen05_supported(const pv_conv3d_desc* d, char* why, size_t why_len) {
#define NOPE(...)                          \
  do {                                     \
    if (why) snprintf(why, why_len, __VA_ARGS__); \
    return 0;                              \
  } while (0)
  if (d->dtype != PV_F16) NOPE("tcgen05 path needs f16 storage");
  if (!conv3d_addend_ok(d)) NOPE("addend layout (16-byte pointer, Co and strides multiples of 8, < 2^31 positions)");
  const bool grouped = d->groups != 1;
  int span_g = 0, span_k = 0, span_n = 0;
  if (grouped) {
    // grouped mode: several spans, each a block-diagonal GEMM over whole 64-channel boxes of its own input channels
    if (!conv3d_group_span(d, &span_g, &span_k, &span_n))
      NOPE("groups=%d does not divide Ci=%d and Co=%d", d->groups, d->Ci, d->Co);
    if (d->groups >= d->Ci) NOPE("depthwise (groups=%d) runs on pv_dwconv3d_fwd", d->groups);
    if (d->Ci != d->Co) NOPE("grouped mode needs square groups (Ci=%d, Co=%d)", d->Ci, d->Co);
    if (d->groups <= span_g) NOPE("one group span (%d groups): run as a dense convolution", span_g);
    if (span_n % 64) NOPE("span output width %d is not a multiple of 64", span_n);
    if (d->x_w_pad > 0) NOPE("grouped mode has no window mode");
    if (d->ci_pad64 != span_k) NOPE("grouped mode: ci_pad64 must equal the span width %d", span_k);
  }
  if (window_mode(d)) {
    if (d->Ci != 4 && d->Ci != 8) NOPE("window mode needs Ci in {4,8}");
    if (d->Co % 8) NOPE("Co must be a multiple of 8");
    if (d->dw != 1) NOPE("window mode needs dilation_w == 1");
    if (d->x_row_stride != d->Ci) NOPE("window mode needs densely packed pixels");
    if ((d->sw * d->Ci * 2) % 16) NOPE("window stride must be a multiple of 16 bytes");
    if ((d->kw + window_lead(d)) * d->Ci > 64) NOPE("window run longer than 64 elements");
    if (d->x_w_pad < d->pw) NOPE("physical W padding smaller than the conv padding");
    if (d->x_w_phys < d->x_w_pad + d->Wi + (d->pw > 0 ? d->pw : 0) || (d->x_w_phys * d->Ci * 2) % 16)
      NOPE("bad physical row width");
    if (d->kt * d->kh > IG_MAX_TAPS) NOPE("too many (dt,dh) taps");
    if (d->st * d->sh > IG_MAX_MAPS) NOPE("stride product too large");
    if (d->ci_pad64 != window_elems(d)) NOPE("window mode: ci_pad64 must equal the window length %d", window_elems(d));
    if (d->y_row_stride % 8 || (d->has_residual && d->res_row_stride % 8)) NOPE("row strides %% 8");
    return 1;
  }
  if (d->Ci % 8 || d->Co % 8) NOPE("Ci/Co must be multiples of 8");
  if (d->x_row_stride % 8 || d->y_row_stride % 8 || (d->has_residual && d->res_row_stride % 8))
    NOPE("row strides must be multiples of 8 elements (16 B)");
  if (d->kt * d->kh * d->kw > IG_MAX_TAPS) NOPE("too many taps");
  if (d->st * d->sh * d->sw > IG_MAX_MAPS) NOPE("stride product > %d", IG_MAX_MAPS);
  if (!grouped && !conv3d_tma_narrow(d) && (d->ci_pad64 < d->Ci || d->ci_pad64 % 64))
    NOPE("ci_pad64 must be a multiple of 64 >= Ci");
  const long long M = (long long)d->N * d->To * d->Ho * d->Wo;
  if (M >= (1ll << 31)) NOPE("too many output positions");
  for (int off : {d->pt, d->ph, d->pw, d->dt * (d->kt - 1), d->dh * (d->kh - 1), d->dw * (d->kw - 1)})
    if (off > 100) NOPE("tap offset too large");
  return 1;
#undef NOPE
}

static double tile_cycles(int n) {   // crude per-k-block cost model (see DESIGN.md)
  double mma = 2.0 * n, smem = 128.0 + n;
  return mma > smem ? mma : smem;
}

int conv3d_tcgen05_launch(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                          const float* bias, const void* residual, void* y, cudaStream_t stream) {
  char why[160];
  if (!conv3d_tcgen05_supported(d, why, sizeof(why))) {
    set_error("PV_ALGO_TCGEN05 unsupported: %s", why);
    return PV_ERR_UNSUPPORTED;
  }
  EncodeTiledFn encode = get_encode_fn();
  if (!encode) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return PV_ERR_CUDA; }

  const int sm_count = current_sm_count();
  if (sm_count <= 0) { set_error("cannot query the SM count of the current device"); return PV_ERR_CUDA; }

  IgemmPlan pl;
  reduce_dims(d, &pl);
  IgemmParams P;
  memset(&P, 0, sizeof(P));

  // ---- tile box search: maximise useful rows per 128-row tile
  {
    long long O[4];
    for (int i = 0; i < 4; ++i) O[i] = pl.dim[i].O;
    double best = -1;
    int bb[4] = {1, 1, 1, 1};
    for (int b0 = 1; b0 <= 128 && b0 <= O[0]; ++b0) {
      for (int b1 = 1; b0 * b1 <= 128 && b1 <= O[1]; ++b1) {
        for (int b2 = 1; b0 * b1 * b2 <= 128 && b2 <= O[2]; ++b2) {
          int b3 = 128 / (b0 * b1 * b2);
          if (b3 > O[3]) b3 = (int)O[3];
          if (b3 < 1) b3 = 1;
          const double tiles = (double)cdiv(O[0], b0) * cdiv(O[1], b1) * cdiv(O[2], b2) * cdiv(O[3], b3);
          const double eff = (double)O[0] * O[1] * O[2] * O[3] / (tiles * 128.0);
          // prefer efficiency, then longer inner runs
          const double score = eff + 1e-6 * b0;
          if (score > best) { best = score; bb[0] = b0; bb[1] = b1; bb[2] = b2; bb[3] = b3; }
        }
      }
    }
    long long mt = 1;
    for (int i = 0; i < 4; ++i) {
      P.O[i] = (int)O[i];
      P.box[i] = bb[i];
      P.nt[i] = (int)cdiv(O[i], bb[i]);
      mt *= P.nt[i];
    }
    P.rows = bb[0] * bb[1] * bb[2] * bb[3];
    P.m_tiles = (int)mt;
  }

  // ---- BLOCK_N (a wgmma width, <= 128): minimise waves * per-tile cost
  const bool grouped = d->groups != 1;
  int span_g = 0, span_k = 0, span_n = 0;
  if (grouped) conv3d_group_span(d, &span_g, &span_k, &span_n);
  {
    const int co16 = (int)cdiv(d->Co, 16) * 16;
    const int cands[4] = {128, 64, 32, 16};
    double best = 1e30;
    int bn = 16;
    for (int c : cands) {
      if (grouped && (c < 64 || span_n % c)) continue;   // grouped: an N tile never straddles two spans
      if (c > round_block_n(co16)) continue;
      if (c < co16 && (c % 64)) continue;   // several N tiles: TMA-store sub-tiles are 64 channels wide
      const long long tiles = (long long)P.m_tiles * cdiv(d->Co, c);
      const double waves = (double)cdiv(tiles, sm_count);
      const double cost = waves * tile_cycles(c) + 1e-3 * cdiv(d->Co, c);
      if (cost < best) { best = cost; bn = c; }
    }
    P.block_n = bn;
    P.n_tiles = (int)cdiv(d->Co, bn);
  }
  const bool wmode = window_mode(d);
  const bool narrow = conv3d_tma_narrow(d);
  const int win = wmode ? window_elems(d) : (narrow ? d->Ci : 64);
  P.kbytes = 2 * win;
  P.Co = d->Co;
  P.taps = wmode ? d->kt * d->kh : d->kt * d->kh * d->kw;
  P.num_kc = (wmode || narrow) ? 1 : d->ci_pad64 / 64;
  P.epi.block_n = P.block_n;
  P.epi.Co = d->Co;
  P.epi.rows = P.rows;
  P.epi.act = d->act;
  P.epi.has_residual = d->has_residual;
  P.epi.nbuf = EPI_MAX_BUFS;
  epi_set_addend(P.epi, d);
  // k-blocks per pipeline stage: 64 K elements (the kernel's compile-time wgmma sequence, see conv3d_igemm_kernel)
  const int kb_bytes = (IG_BM + P.block_n) * P.kbytes;
  const size_t smem_fixed = 2048 /*align*/ + epi_smem_bytes(P.epi.nbuf) + 16;
  {
    const int num_kb = P.taps * P.num_kc;
    const int G = 128 / P.kbytes;
    const int budget = (int)(227 * 1024 - smem_fixed) - 8 * (2 * 24);   // barriers of up to 24 stages
    int st = budget / (G * kb_bytes);
    if (st > 24 / G) st = 24 / G > 2 ? 24 / G : 2;
    if (st < 2) st = 2;
    P.G = G;
    // 2 producer warps (A / B) for one k-block per stage, 3 for chunked stages (window / narrow modes: up to 8 loads)
    P.split_ab = G >= 2 ? 3 : 2;
    P.cpt = (num_kb + G - 1) / G;
    P.stages = st;
    // a padding k-block would load channel num_kc * 64 of the span, i.e. the next span's first channels
    if (grouped && (G != 1 || P.block_n > span_n || span_n % P.block_n)) {
      set_error("internal: grouped mode needs one k-block per stage and BLOCK_N | N_span (G=%d BN=%d N_span=%d)", G,
                P.block_n, span_n);
      return PV_ERR_INVALID;
    }
  }
  const int stage_bytes = P.G * kb_bytes;
  const size_t smem_bytes = (size_t)P.stages * stage_bytes + smem_fixed + 8 * (2 * P.stages);

  // ---- taps -> (parity map, coordinate shift); original dims order: tap index = (kt, kh, kw)
  // merged dims never merge a dim that has taps, so each non-trivial original dim maps to one
  // merged dim.  Build per-merged-dim lists.
  int ks[4], ss[4], ps[4], dls[4];
  for (int i = 0; i < 4; ++i) { ks[i] = pl.dim[i].k; ss[i] = pl.dim[i].s; ps[i] = pl.dim[i].p; dls[i] = pl.dim[i].dil; }
  const int* orig2m = pl.orig2m;
  unsigned used_maps = 0;
  const int kw_loop = wmode ? 1 : d->kw;
  for (int it = 0; it < d->kt; ++it)
    for (int ih = 0; ih < d->kh; ++ih)
      for (int iw = 0; iw < kw_loop; ++iw) {
        const int tap = (it * d->kh + ih) * kw_loop + iw;
        int q[4] = {0, 0, 0, 0}, r[4] = {0, 0, 0, 0};
        // window mode: the W taps live inside the window and the W padding is physical
        const int offs[3] = {wmode ? 0 : iw * d->dw - d->pw, ih * d->dh - d->ph, it * d->dt - d->pt};
        const int strd[3] = {wmode ? 1 : d->sw, d->sh, d->st};
        for (int o = 0; o < 3; ++o) {
          const int m = orig2m[o];
          if (strd[o] == 1 && offs[o] == 0) continue;
          const int qq = floordiv(offs[o], strd[o]);
          q[m] = qq;
          r[m] = offs[o] - qq * strd[o];
        }
        int cls = 0, mul = 1;
        for (int m = 0; m < 4; ++m) { cls += r[m] * mul; mul *= ss[m]; }
        if (cls >= IG_MAX_MAPS) { set_error("internal: parity class %d", cls); return PV_ERR_INVALID; }
        P.tap_map[tap] = (unsigned char)cls;
        for (int m = 0; m < 4; ++m) P.tap_q[tap][m] = (signed char)q[m];
        used_maps |= 1u << cls;
      }

  // ---- tensor maps
  for (int cls = 0; cls < IG_MAX_MAPS; ++cls) {
    if (!(used_maps & (1u << cls))) continue;
    int r[4], c = cls;
    for (int m = 0; m < 4; ++m) { r[m] = c % ss[m]; c /= ss[m]; }
    long long base_off = wmode ? (long long)(d->x_w_pad - d->pw - window_lead(d)) * d->Ci * 2 : 0;   // bytes
    cuuint64_t gdim[5], gstr[4];
    cuuint32_t box[5], estr[5] = {1, 1, 1, 1, 1};
    gdim[0] = (cuuint64_t)(wmode ? win : d->Ci);
    box[0] = (cuuint32_t)win;
    for (int m = 0; m < 4; ++m) {
      const long long cnt = (pl.dim[m].I - r[m] + ss[m] - 1) / ss[m];
      gdim[m + 1] = (cuuint64_t)(cnt > 0 ? cnt : 1);
      gstr[m] = (cuuint64_t)(pl.dim[m].stride_bytes * ss[m]);
      box[m + 1] = (cuuint32_t)P.box[m];
      base_off += (long long)r[m] * pl.dim[m].stride_bytes;
    }
    void* gptr = (void*)((const char*)x + base_off);
    const CUtensorMapSwizzle swz = P.kbytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                   : (P.kbytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
    CUresult cr = encode(&P.a_maps[cls], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, gptr, gdim, gstr, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled(A, class %d) failed: %d (Ci=%d dims=%llu,%llu,%llu,%llu box=%u,%u,%u,%u)",
                cls, (int)cr, d->Ci, (unsigned long long)gdim[1], (unsigned long long)gdim[2],
                (unsigned long long)gdim[3], (unsigned long long)gdim[4], box[1], box[2], box[3], box[4]);
      return PV_ERR_CUDA;
    }
  }
  {
    const long long krow = (long long)P.taps * d->ci_pad64;     // window mode: ci_pad64 == window length
    const long long kpitch = narrow ? (krow + 63) / 64 * 64 : krow;   // narrow mode shares the gather packing (row end padded to 64)
    cuuint64_t gdim[2] = {(cuuint64_t)krow, (cuuint64_t)d->Co};
    cuuint64_t gstr[1] = {(cuuint64_t)kpitch * 2};
    cuuint32_t box[2] = {(cuuint32_t)win, (cuuint32_t)P.block_n}, estr[2] = {1, 1};
    const CUtensorMapSwizzle swz = P.kbytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                   : (P.kbytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
    CUresult cr = encode(&P.b_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)w, gdim, gstr, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(B) failed: %d", (int)cr); return PV_ERR_CUDA; }
  }

  // ---- output / residual tensor maps (merged OUTPUT dims follow the input merge pattern)
  {
    const long long ostr_orig[4] = {1, d->Wo, (long long)d->Wo * d->Ho, (long long)d->Wo * d->Ho * d->To};
    long long ostr[4] = {0, 0, 0, 0};
    bool seen[4] = {false, false, false, false};
    for (int o = 0; o < 4; ++o) {
      const int m = pl.orig2m[o];
      if (!seen[m]) { seen[m] = true; ostr[m] = ostr_orig[o]; }
    }
    for (int m = 0; m < 4; ++m) {
      P.epi.o_ext[m] = P.O[m];
      P.epi.o_box[m] = P.box[m];
      P.epi.o_pos[m] = seen[m] ? (int)ostr[m] : 0;
    }
    for (int pass = 0; pass < 2; ++pass) {
      if (pass == 1 && !d->has_residual) break;
      const long long rs = pass == 0 ? d->y_row_stride : d->res_row_stride;
      void* base = pass == 0 ? y : const_cast<void*>(residual);
      cuuint64_t gdim[5], gstr[4];
      cuuint32_t box[5], estr[5] = {1, 1, 1, 1, 1};
      gdim[0] = (cuuint64_t)d->Co;
      box[0] = 64;
      long long prev = rs * 2;      // byte extent covered so far (for filler dims)
      for (int m = 0; m < 4; ++m) {
        gdim[m + 1] = (cuuint64_t)P.O[m];
        const long long sb = seen[m] ? ostr[m] * rs * 2 : prev;
        gstr[m] = (cuuint64_t)sb;
        prev = sb * (long long)P.O[m];
        box[m + 1] = (cuuint32_t)P.box[m];
      }
      CUresult cr = encode(pass == 0 ? &P.epi.y_map : &P.epi.r_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, base, gdim,
                           gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (cr != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled(%s) failed: %d", pass == 0 ? "Y" : "R", (int)cr);
        return PV_ERR_CUDA;
      }
    }
  }

  const long long total_tiles = (long long)P.m_tiles * P.n_tiles;
  if (total_tiles == 0) return PV_OK;
  const int grid = (int)(total_tiles < sm_count ? total_tiles : sm_count);
  {
    // launched with the programmatic-stream-serialization attribute (PDL): the prologue overlaps the previous kernel
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(IG_THREADS);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
#define PV_IG_LAUNCH(BN, KB)                                                                   \
  if (P.block_n == BN && P.kbytes == KB) {                                                     \
    PV_OPT_IN_SMEM((conv3d_igemm_kernel<BN, KB>), 227 * 1024);                                 \
    PV_CUDA_OK(cudaLaunchKernelEx(&cfg, conv3d_igemm_kernel<BN, KB>, P, scale, bias));         \
    name = "conv3d_igemm_kernel<" #BN "," #KB ">";                                              \
  }
    const char* name = nullptr;
    if (grouped) {
      const int span_tiles = span_n / P.block_n;
#define PV_IG_GROUPED_LAUNCH(BN, KB)                                                                     \
  if (P.block_n == BN && P.kbytes == KB) {                                                               \
    PV_OPT_IN_SMEM((conv3d_igemm_grouped_kernel<BN, KB>), 227 * 1024);                                   \
    PV_CUDA_OK(cudaLaunchKernelEx(&cfg, conv3d_igemm_grouped_kernel<BN, KB>, P, scale, bias, span_tiles)); \
    name = "conv3d_igemm_grouped_kernel<" #BN "," #KB ">";                                               \
  }
      PV_IG_GROUPED_LAUNCH(64, 128) PV_IG_GROUPED_LAUNCH(128, 128)
#undef PV_IG_GROUPED_LAUNCH
      if (!name) { set_error("internal: no grouped igemm instance for BN=%d kbytes=%d", P.block_n, P.kbytes); return PV_ERR_INVALID; }
      PV_LAUNCH_OK(name);
      return PV_OK;
    }
    PV_IG_LAUNCH(16, 32) PV_IG_LAUNCH(16, 64) PV_IG_LAUNCH(16, 128)
    PV_IG_LAUNCH(32, 32) PV_IG_LAUNCH(32, 64) PV_IG_LAUNCH(32, 128)
    PV_IG_LAUNCH(64, 32) PV_IG_LAUNCH(64, 64) PV_IG_LAUNCH(64, 128)
    PV_IG_LAUNCH(128, 32) PV_IG_LAUNCH(128, 64) PV_IG_LAUNCH(128, 128)
#undef PV_IG_LAUNCH
    if (!name) { set_error("internal: no igemm instance for BN=%d kbytes=%d", P.block_n, P.kbytes); return PV_ERR_INVALID; }
    PV_LAUNCH_OK(name);
  }
  return PV_OK;
}

}  // namespace pv

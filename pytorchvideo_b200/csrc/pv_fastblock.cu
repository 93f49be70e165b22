// Fused bottleneck block for NARROW pathways (SlowFast Fast pathway res2 / res3: C_inner = 8 / 16):
//
//   a = relu(bn_a(conv_a(x)))      conv_a: (kt,1,1) temporal, C_in -> C_mid            (resnet.py:1345-1365)
//   b = relu(bn_b(conv_b(a)))      conv_b: (1,3,3) spatial stride (1,s,s), C_mid -> C_mid
//   y = act(bn_c(conv_c(b)) + sc)  conv_c: 1x1x1, C_mid -> C_out; sc = x or bn_1(conv_1(x)) stride (1,s,s) (resnet.py:1179-1189)
//
// Unfused, every one of these is a launch whose tensors (a, b: 8..32 channels) round-trip through L2 and whose
// tiles are far too thin for the warp-specialised implicit-GEMM pipeline (a 128-row tile is mostly pipeline latency).
// Here ONE CTA walks the frames of
// one spatial tile of one clip: the x frames t-1, t, t+1 live in a shared-memory ring (each frame tile is read from
// L2 exactly once, zero-filled outside the clip = the padding of conv_a), a and b never leave shared memory, and
// the residual comes from the x tile that is already there.  The three GEMMs are tiny (K <= 384, N <= 128) and run
// on mma.sync m16n8k16 with ldmatrix-fed A fragments gathered straight from the position-major tiles (the im2col
// of conv_b is just a different row address per lane); the block is bound by its x read + y write.
//
// Layouts: activations NDHWC f16 (row stride >= C); weights packed [n][k] f16 with k = (tap, ci), K padded to 16;
// folded BatchNorm as fp32 (scale, bias) per output channel, applied on the fp32 accumulator like everywhere else.
#include "pv_common.cuh"

#include <stdlib.h>
#include <string.h>

namespace pv {

struct FbParams {
  int N, T, H, W, Ho, Wo;
  int Cin, Cout;
  int kt, sb, has_sc, act;
  int TH, TW, TC;            // output tile (rows, cols) and frames per CTA
  int RH, RW;                // halo tile of x / a in input resolution: (TH-1)*sb+3, (TW-1)*sb+3
  int tiles_h, tiles_w, tchunks;
  int KA, KB, KC, KS;        // padded K extents (multiples of 16)
  int ldwa, ldwb, ldwc, ldws;  // shared-memory row pitches of the weight matrices (elements, K + 8: conflict-free B loads)
  long long xrs, yrs;        // row strides (elements)
  // shared memory carve-up (byte offsets)
  unsigned off_x, x_slot_bytes, off_a, off_b, off_y, off_wa, off_wb, off_wc, off_ws, off_sb, off_tab;
};

__device__ __forceinline__ unsigned fb_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

// 16-byte chunk swizzle inside a position row of `row_bytes` (power of two >= 16): keeps the 8 row addresses of an
// ldmatrix phase on distinct banks for 32 / 64 / >= 128-byte rows (16-byte rows are contiguous already).
__device__ __forceinline__ unsigned fb_swz(unsigned row, unsigned chunk, unsigned row_bytes) {
  if (row_bytes >= 128u) return chunk ^ (row & 7u);
  if (row_bytes == 64u) return chunk ^ ((row >> 1) & 3u);
  if (row_bytes == 32u) return chunk ^ ((row >> 2) & 1u);
  return chunk;
}

__device__ __forceinline__ void ldmatrix_x4(unsigned addr, unsigned (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float (&c)[4], const unsigned (&a)[4], unsigned b0, unsigned b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(unsigned dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16u : 0u) : "memory");
}

constexpr int FB_WARPS = 8;
constexpr int FB_THREADS = FB_WARPS * 32;
constexpr int FB_SLOTS = 4;      // frame ring: t-1, t, t+1 in use, t+2 in flight
constexpr int FB_MT = 2;         // m-tiles (16 rows) per warp and phase: tiles are chosen with <= 256 rows
constexpr unsigned FB_SKIP = 0xffffffffu;

template <unsigned ROW_BYTES>
__device__ __forceinline__ unsigned fb_swz_c(unsigned row, unsigned chunk) {   // fb_swz with a compile-time row size
  if (ROW_BYTES >= 128u) return chunk ^ (row & 7u);
  if (ROW_BYTES == 64u) return chunk ^ ((row >> 1) & 3u);
  if (ROW_BYTES == 32u) return chunk ^ ((row >> 2) & 1u);
  return chunk;
}
__device__ __forceinline__ int fb_lane_row(int lane) { return (lane & 7) + ((lane >> 3) & 1) * 8; }
__device__ __forceinline__ unsigned fb_lds32(unsigned addr) {
  unsigned v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void fb_sts32(unsigned addr, unsigned v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned fb_pack(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const unsigned*>(&h);
}

// The instruction diet (ncu, first version: 2340 warp-instructions per warp and frame at IPC 2.1, tensor pipe 5 %
// busy - issue-bound on address arithmetic): every shape is a template parameter, so all K loops unroll and the
// weight-fragment loads use immediate offsets; everything that depends on the POSITION a lane works on (ldmatrix
// row addresses, image-border flags, residual and output offsets) is the same for every frame and is computed once
// per CTA, before the frame loop.
template <int CIN, int CMID, int KT, int SB, bool HAS_SC>
__global__ void __launch_bounds__(FB_THREADS)
bottleneck_fused_kernel(const __grid_constant__ FbParams P, const __half* __restrict__ x, const __half* __restrict__ wa,
                        const __half* __restrict__ wb, const __half* __restrict__ wc, const __half* __restrict__ wsc,
                        const float* __restrict__ sa, const float* __restrict__ ba, const float* __restrict__ sb_,
                        const float* __restrict__ bb, const float* __restrict__ sc, const float* __restrict__ bc,
                        const float* __restrict__ ssc, const float* __restrict__ bsc, __half* __restrict__ y) {
  constexpr int NTM = CMID / 8;                          // n-tiles of the inner width
  constexpr int COUT = 4 * CMID;
  constexpr int NG = COUT / 32;                          // 32-channel output groups of phase C
  constexpr int KA = (KT * CIN + 15) / 16 * 16, KB = (9 * CMID + 15) / 16 * 16, KC = (CMID + 15) / 16 * 16, KS = (CIN + 15) / 16 * 16;
  constexpr int LDWA = KA + 8, LDWB = KB + 8, LDWC = KC + 8, LDWS = KS + 8;
  constexpr unsigned XROW = CIN * 2, AROW = CMID * 2, YROW = COUT * 2;
  constexpr int XCH = XROW / 16;
  constexpr int PAD_T = KT / 2;
  extern __shared__ __align__(128) unsigned char fb_smem[];
  const unsigned sbase = fb_smem_u32(fb_smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, q = lane & 3, hi = lane >> 4;

  // ---- which tile
  int bid = blockIdx.x;
  const int tw = bid % P.tiles_w; bid /= P.tiles_w;
  const int th = bid % P.tiles_h; bid /= P.tiles_h;
  const int tch = bid % P.tchunks;
  const int n = bid / P.tchunks;
  const int oy0 = th * P.TH, ox0 = tw * P.TW;                 // output tile origin
  const int iy0 = oy0 * SB - 1, ix0 = ox0 * SB - 1;           // halo tile origin in the input (may be -1)
  const int t_begin = tch * P.TC, t_end = min(P.T, t_begin + P.TC);
  const int npos_in = P.RH * P.RW, npos_out = P.TH * P.TW;

  // ---- weights, folded BN and the per-position source table into shared memory (once per CTA)
  __half* s_wa = reinterpret_cast<__half*>(fb_smem + P.off_wa);
  __half* s_wb = reinterpret_cast<__half*>(fb_smem + P.off_wb);
  __half* s_wc = reinterpret_cast<__half*>(fb_smem + P.off_wc);
  __half* s_ws = reinterpret_cast<__half*>(fb_smem + P.off_ws);
  float* s_sb = reinterpret_cast<float*>(fb_smem + P.off_sb);       // [sa ba sb bb](CMID each) [sc bc ssc bsc](COUT each)
  int* s_src = reinterpret_cast<int*>(fb_smem + P.off_tab);          // element offset of the position inside a frame, -1 outside
  for (int i = tid; i < CMID * (KA / 8); i += FB_THREADS) {
    const int r = i / (KA / 8), c = (i - r * (KA / 8)) * 8;
    *reinterpret_cast<uint4*>(s_wa + r * LDWA + c) = *reinterpret_cast<const uint4*>(wa + (size_t)r * KA + c);
  }
  for (int i = tid; i < CMID * (KB / 8); i += FB_THREADS) {
    const int r = i / (KB / 8), c = (i - r * (KB / 8)) * 8;
    *reinterpret_cast<uint4*>(s_wb + r * LDWB + c) = *reinterpret_cast<const uint4*>(wb + (size_t)r * KB + c);
  }
  for (int i = tid; i < COUT * (KC / 8); i += FB_THREADS) {
    const int r = i / (KC / 8), c = (i - r * (KC / 8)) * 8;
    *reinterpret_cast<uint4*>(s_wc + r * LDWC + c) = *reinterpret_cast<const uint4*>(wc + (size_t)r * KC + c);
  }
  if (HAS_SC)
    for (int i = tid; i < COUT * (KS / 8); i += FB_THREADS) {
      const int r = i / (KS / 8), c = (i - r * (KS / 8)) * 8;
      *reinterpret_cast<uint4*>(s_ws + r * LDWS + c) = *reinterpret_cast<const uint4*>(wsc + (size_t)r * KS + c);
    }
  for (int i = tid; i < CMID; i += FB_THREADS) {
    s_sb[i] = sa[i]; s_sb[CMID + i] = ba[i]; s_sb[2 * CMID + i] = sb_[i]; s_sb[3 * CMID + i] = bb[i];
  }
  for (int i = tid; i < COUT; i += FB_THREADS) {
    float* o = s_sb + 4 * CMID;
    o[i] = sc[i]; o[COUT + i] = bc[i];
    o[2 * COUT + i] = HAS_SC ? ssc[i] : 0.f; o[3 * COUT + i] = HAS_SC ? bsc[i] : 0.f;
  }
  for (int pos = tid; pos < npos_in; pos += FB_THREADS) {
    const int py = pos / P.RW, px = pos - py * P.RW;
    const int iy = iy0 + py, ix = ix0 + px;
    const bool ok = (unsigned)iy < (unsigned)P.H && (unsigned)ix < (unsigned)P.W;
    s_src[pos] = ok ? (int)(((long long)iy * P.W + ix) * P.xrs) : -1;
  }
  for (int opos = tid; opos < npos_out; opos += FB_THREADS) {       // output position -> element offset inside a y frame
    const int qy = opos / P.TW, qx = opos - qy * P.TW;
    const int oy = oy0 + qy, ox = ox0 + qx;
    s_src[256 + opos] = (oy < P.Ho && ox < P.Wo) ? (int)(((long long)oy * P.Wo + ox) * P.yrs) : -1;
  }
  const float* s_c = s_sb + 4 * CMID;

  // ---- frame loader: halo tile of frame f -> ring slot (f + 8) & 3, zero-filled outside the clip
  const __half* xn = x + (size_t)n * P.T * P.H * P.W * P.xrs;
  const size_t frame_elems = (size_t)P.H * P.W * P.xrs;
  auto load_frame = [&](int f) {
    const unsigned dst0 = sbase + P.off_x + ((unsigned)(f + 8) & (FB_SLOTS - 1)) * P.x_slot_bytes;
    const bool f_ok = f >= 0 && f < P.T;
    const __half* xf = xn + (f_ok ? (size_t)f * frame_elems : 0);
    for (int i = tid; i < npos_in * XCH; i += FB_THREADS) {
      const unsigned pos = (unsigned)i / XCH, ch = (unsigned)i % XCH;
      const int so = s_src[pos];
      const bool ok = f_ok && so >= 0;
      cp_async16(dst0 + pos * XROW + (fb_swz_c<XROW>(pos, ch) << 4), ok ? xf + so + ch * 8 : x, ok);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  __syncthreads();                                             // s_src is read by the loader
  for (int f = t_begin - PAD_T; f <= t_begin + PAD_T; ++f) load_frame(f);

  // ---- per-lane, frame-invariant offsets (FB_MT m-tiles per warp and phase: m-tile = warp + 8 * i)
  const int mt_in = (npos_in + 15) >> 4, mt_out = (npos_out + 15) >> 4;
  const unsigned a_base = sbase + P.off_a, b_base = sbase + P.off_b, y_base = sbase + P.off_y;
  unsigned A_ld[FB_MT], A_xor[FB_MT], A_st[FB_MT][2];          // phase A: ldmatrix row offset in a slot, swizzle phase, a-tile store
  unsigned B_pos[FB_MT], B_st[FB_MT][2];                        // phase B: window corner position in the a tile, b-tile store
  unsigned C_ld[FB_MT], C_x[FB_MT], C_res[FB_MT][2], C_y[FB_MT][2];   // phase C: b row, x centre row (ldmatrix / residual), y-tile store
#pragma unroll
  for (int i = 0; i < FB_MT; ++i) {
    const int mt = warp + FB_WARPS * i;
    {
      const unsigned pos = (unsigned)min(mt * 16 + fb_lane_row(lane), npos_in - 1);
      A_ld[i] = pos * XROW;
      A_xor[i] = fb_swz_c<XROW>(pos, 0);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int p2 = mt * 16 + g + 8 * h;
        A_st[i][h] = FB_SKIP;
        if (mt < mt_in && p2 < npos_in) {
          // bit 31 marks a position outside the image: a = 0 there (the zero padding of conv_b), not relu(bn(0))
          A_st[i][h] = ((unsigned)p2 * AROW + (unsigned)(2 * q) * 2u) | (s_src[p2] < 0 ? 0x80000000u : 0u);
        }
      }
    }
    {
      const int opos = min(mt * 16 + fb_lane_row(lane), npos_out - 1);
      const int qy = opos / P.TW, qx = opos - qy * P.TW;
      B_pos[i] = (unsigned)(qy * SB * P.RW + qx * SB);
      C_ld[i] = (unsigned)opos;
      C_x[i] = (unsigned)((qy * SB + 1) * P.RW + qx * SB + 1);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int o2 = mt * 16 + g + 8 * h;
        B_st[i][h] = FB_SKIP; C_res[i][h] = 0; C_y[i][h] = FB_SKIP;
        if (mt < mt_out && o2 < npos_out) {
          const int q2y = o2 / P.TW, q2x = o2 - q2y * P.TW;
          B_st[i][h] = (unsigned)o2;
          C_res[i][h] = (unsigned)((q2y * SB + 1) * P.RW + q2x * SB + 1);
          C_y[i][h] = (unsigned)o2 * YROW + (unsigned)(2 * q) * 2u;
        }
      }
    }
  }
  // lane's weight-fragment bases: row g of each n-tile, k = 2q (+8 for the second register)
  const unsigned wa_l = fb_smem_u32(s_wa) + (unsigned)(g * LDWA + 2 * q) * 2u;
  const unsigned wb_l = fb_smem_u32(s_wb) + (unsigned)(g * LDWB + 2 * q) * 2u;
  const unsigned wc_l = fb_smem_u32(s_wc) + (unsigned)(g * LDWC + 2 * q) * 2u;
  const unsigned ws_l = fb_smem_u32(s_ws) + (unsigned)(g * LDWS + 2 * q) * 2u;

  for (int t = t_begin; t < t_end; ++t) {
    load_frame(t + PAD_T + 1);                                 // into the slot frame t - PAD_T - 1 no longer needs
    asm volatile("cp.async.wait_group 1;" ::: "memory");      // everything but the frame just requested has landed
    __syncthreads();                                           // (also: weights / tables visible on the first step; s_y drained)
    unsigned slot_base[KT];
#pragma unroll
    for (int dt = 0; dt < KT; ++dt)
      slot_base[dt] = sbase + P.off_x + ((unsigned)(t + dt - PAD_T + 8) & (FB_SLOTS - 1)) * P.x_slot_bytes;

    // ================= phase A: a = relu(bn_a(conv_a(x))) on the halo tile, 0 outside the image =================
#pragma unroll
    for (int i = 0; i < FB_MT; ++i) {
      if (warp + FB_WARPS * i >= mt_in) break;
      float acc[NTM][4];
#pragma unroll
      for (int j = 0; j < NTM; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }
#pragma unroll
      for (int ks = 0; ks < KA / 16; ++ks) {
        // this lane's 8-wide K half: k = 16 ks + 8 hi = dt * CIN + ci  (K padding: zero weights, any finite data)
        int dt, ci;
        if (CIN == 8) { dt = min(2 * ks + hi, KT - 1); ci = 0; }
        else { dt = min((16 * ks) / CIN, KT - 1); ci = (16 * ks) % CIN + 8 * hi; }
        unsigned sb0 = slot_base[0];
#pragma unroll
        for (int d2 = 1; d2 < KT; ++d2) sb0 = dt == d2 ? slot_base[d2] : sb0;
        unsigned a[4];
        ldmatrix_x4(sb0 + A_ld[i] + ((((unsigned)ci >> 3) ^ A_xor[i]) << 4), a);
#pragma unroll
        for (int nt = 0; nt < NTM; ++nt) {
          const unsigned wofs = (unsigned)((nt * 8) * LDWA + ks * 16) * 2u;
          mma_16816(acc[nt], a, fb_lds32(wa_l + wofs), fb_lds32(wa_l + wofs + 16u));
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const unsigned st = A_st[i][h];
        if (st != FB_SKIP) {
          const bool inside = (st & 0x80000000u) == 0u;
          const unsigned off = st & 0x7fffffffu;
          const unsigned pos = off / AROW;
#pragma unroll
          for (int nt = 0; nt < NTM; ++nt) {
            const int c = nt * 8 + 2 * q;
            float v0 = fmaxf(fmaf(acc[nt][2 * h], s_sb[c], s_sb[CMID + c]), 0.f);
            float v1 = fmaxf(fmaf(acc[nt][2 * h + 1], s_sb[c + 1], s_sb[CMID + c + 1]), 0.f);
            if (!inside) { v0 = 0.f; v1 = 0.f; }
            fb_sts32(a_base + pos * AROW + (fb_swz_c<AROW>(pos, (unsigned)nt) << 4) + (unsigned)(2 * q) * 2u, fb_pack(v0, v1));
          }
        }
      }
    }
    __syncthreads();

    // ================= phase B: b = relu(bn_b(conv_b(a))), 3x3 window of the a tile ============================
#pragma unroll
    for (int i = 0; i < FB_MT; ++i) {
      if (warp + FB_WARPS * i >= mt_out) break;
      float acc[NTM][4];
#pragma unroll
      for (int j = 0; j < NTM; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }
#pragma unroll
      for (int ks = 0; ks < KB / 16; ++ks) {
        // k = 16 ks + 8 hi = (dh * 3 + dw) * CMID + ci
        int tap, ci;
        if (CMID == 8) { tap = min(2 * ks + hi, 8); ci = 0; }
        else { tap = min((16 * ks) / CMID, 8); ci = (16 * ks) % CMID + 8 * hi; }
        const int dh = (tap * 11) >> 5, dw = tap - dh * 3;
        const unsigned pos = B_pos[i] + (unsigned)(dh * P.RW + dw);
        unsigned a[4];
        ldmatrix_x4(a_base + pos * AROW + (fb_swz_c<AROW>(pos, (unsigned)ci >> 3) << 4), a);
#pragma unroll
        for (int nt = 0; nt < NTM; ++nt) {
          const unsigned wofs = (unsigned)((nt * 8) * LDWB + ks * 16) * 2u;
          mma_16816(acc[nt], a, fb_lds32(wb_l + wofs), fb_lds32(wb_l + wofs + 16u));
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const unsigned opos = B_st[i][h];
        if (opos != FB_SKIP) {
#pragma unroll
          for (int nt = 0; nt < NTM; ++nt) {
            const int c = nt * 8 + 2 * q;
            const float v0 = fmaxf(fmaf(acc[nt][2 * h], s_sb[2 * CMID + c], s_sb[3 * CMID + c]), 0.f);
            const float v1 = fmaxf(fmaf(acc[nt][2 * h + 1], s_sb[2 * CMID + c + 1], s_sb[3 * CMID + c + 1]), 0.f);
            fb_sts32(b_base + opos * AROW + (fb_swz_c<AROW>(opos, (unsigned)nt) << 4) + (unsigned)(2 * q) * 2u, fb_pack(v0, v1));
          }
        }
      }
    }
    __syncthreads();

    // ================= phase C: y = act(bn_c(conv_c(b)) + shortcut), 32 output channels per pass ================
    const unsigned xslot_t = slot_base[PAD_T];
#pragma unroll
    for (int i = 0; i < FB_MT; ++i) {
      if (warp + FB_WARPS * i >= mt_out) break;
      // A fragments of this m-tile: b rows (conv_c) and x centre rows (projection shortcut), loaded once for all groups
      unsigned fa[KC / 16][4];
#pragma unroll
      for (int ks = 0; ks < KC / 16; ++ks) {
        const int ci = min(16 * ks + 8 * hi, CMID - 8);          // K padding (CMID = 8): zero weights
        ldmatrix_x4(b_base + C_ld[i] * AROW + (fb_swz_c<AROW>(C_ld[i], (unsigned)ci >> 3) << 4), fa[ks]);
      }
#pragma unroll 1
      for (int ng = 0; ng < NG; ++ng) {
        float acc[4][4], acs[4][4];
#pragma unroll
        for (int j = 0; j < 4; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; acs[j][0] = acs[j][1] = acs[j][2] = acs[j][3] = 0.f; }
#pragma unroll
        for (int ks = 0; ks < KC / 16; ++ks)
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            const unsigned wofs = (unsigned)((ng * 32 + nt * 8) * LDWC + ks * 16) * 2u;
            mma_16816(acc[nt], fa[ks], fb_lds32(wc_l + wofs), fb_lds32(wc_l + wofs + 16u));
          }
        if (HAS_SC) {
#pragma unroll
          for (int ks = 0; ks < KS / 16; ++ks) {
            const int ci = min(16 * ks + 8 * hi, CIN - 8);
            unsigned a[4];
            ldmatrix_x4(xslot_t + C_x[i] * XROW + (fb_swz_c<XROW>(C_x[i], (unsigned)ci >> 3) << 4), a);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
              const unsigned wofs = (unsigned)((ng * 32 + nt * 8) * LDWS + ks * 16) * 2u;
              mma_16816(acs[nt], a, fb_lds32(ws_l + wofs), fb_lds32(ws_l + wofs + 16u));
            }
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (C_y[i][h] != FB_SKIP) {
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
              const int c = ng * 32 + nt * 8 + 2 * q;
              float v0 = fmaf(acc[nt][2 * h], s_c[c], s_c[COUT + c]);
              float v1 = fmaf(acc[nt][2 * h + 1], s_c[c + 1], s_c[COUT + c + 1]);
              if (HAS_SC) {
                v0 += fmaf(acs[nt][2 * h], s_c[2 * COUT + c], s_c[3 * COUT + c]);
                v1 += fmaf(acs[nt][2 * h + 1], s_c[2 * COUT + c + 1], s_c[3 * COUT + c + 1]);
              } else {                                           // identity shortcut: CIN == COUT, same channel
                const unsigned rp = C_res[i][h];
                const unsigned rv = fb_lds32(xslot_t + rp * XROW + (fb_swz_c<XROW>(rp, (unsigned)(c >> 3)) << 4) + (unsigned)(2 * q) * 2u);
                const float2 rf = __half22float2(*reinterpret_cast<const __half2*>(&rv));
                v0 += rf.x; v1 += rf.y;
              }
              if (P.act == PV_ACT_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
              fb_sts32(y_base + C_y[i][h] + (unsigned)(ng * 32 + nt * 8) * 2u, fb_pack(v0, v1));
            }
          }
        }
      }
    }
    __syncthreads();

    // ================= store the y tile: 16-byte coalesced rows ================================================
    {
      constexpr int YCH = YROW / 16;
      __half* yt = y + ((size_t)n * P.T + t) * P.Ho * P.Wo * P.yrs;
      const int* s_dst = s_src + 256;
      for (int i = tid; i < npos_out * YCH; i += FB_THREADS) {
        const unsigned opos = (unsigned)i / YCH, ch = (unsigned)i % YCH;
        const int dofs = s_dst[opos];
        if (dofs >= 0) {
          uint4 v;
          asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(y_base + opos * YROW + ch * 16u));
          *reinterpret_cast<uint4*>(yt + dofs + ch * 8) = v;
        }
      }
    }
    // (the next iteration's first __syncthreads orders these shared-memory reads before s_y / s_a are rewritten)
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}

static int fb_pad16(int k) { return (k + 15) / 16 * 16; }

}  // namespace pv

using namespace pv;

namespace {
struct FbCombo { int cin, cmid, kt, sb, sc; };
// the instantiated shapes: SlowFast Fast pathway res2 / res3 / res4 (first block with its projection shortcut, the
// following blocks with the identity), plus a pointwise-conv_a variant
const FbCombo kCombos[] = {
    {8, 8, 3, 1, 1},   {32, 8, 3, 1, 0},   {32, 8, 1, 1, 0},
    {32, 16, 3, 2, 1}, {32, 16, 3, 1, 1},  {64, 16, 3, 1, 0},
    // C_mid = 32 (res4: 14 x 14 planes, 170 registers -> one CTA per SM) measured SLOWER than the three implicit-GEMM launches
    // per block: not instantiated
};
bool fb_has_combo(int cin, int cmid, int kt, int sb, int sc) {
  for (const FbCombo& c : kCombos)
    if (c.cin == cin && c.cmid == cmid && c.kt == kt && c.sb == sb && c.sc == sc) return true;
  return false;
}
}  // namespace

extern "C" int pv_bottleneck_fused_supported(const pv_bottleneck_desc* d) {
  if (!d) return 0;
  if (d->Cout != 4 * d->Cmid) return 0;
  if (!fb_has_combo(d->Cin, d->Cmid, d->kt, d->sb, d->has_shortcut ? 1 : 0)) return 0;
  if (!d->has_shortcut && (d->Cin != d->Cout || d->sb != 1)) return 0;
  if (!(d->act == PV_ACT_RELU || d->act == PV_ACT_NONE)) return 0;
  if (d->x_row_stride % 8 || d->y_row_stride % 8 || d->x_row_stride < d->Cin || d->y_row_stride < d->Cout) return 0;
  if (d->N < 0 || d->T <= 0 || d->H <= 0 || d->W <= 0) return 0;       // (T = 0 would divide by zero below)
  // the kernel keeps in-frame element offsets of x and y in 32-bit tables
  if ((long long)d->H * d->W * d->x_row_stride >= (1ll << 31)) return 0;
  const long long Ho = (d->H - 1) / d->sb + 1, Wo = (d->W - 1) / d->sb + 1;
  if (Ho * Wo * d->y_row_stride >= (1ll << 31)) return 0;
  return 1;
}

namespace {
// The launch geometry of a supported descriptor on a device with sm_count SMs: tile, frame chunk, shared-memory
// carve-up.  Host-only; pv_bottleneck_fused_fwd and pv_bottleneck_fused_tiling both use it.
int fb_plan(const pv_bottleneck_desc* d, int sm_count, FbParams& P, size_t& smem_bytes) {
  memset(&P, 0, sizeof(P));
  P.N = d->N; P.T = d->T; P.H = d->H; P.W = d->W;
  P.Ho = (d->H + 2 - 3) / d->sb + 1; P.Wo = (d->W + 2 - 3) / d->sb + 1;
  P.Cin = d->Cin; P.Cout = d->Cout; P.kt = d->kt; P.sb = d->sb; P.has_sc = d->has_shortcut; P.act = d->act;
  P.xrs = d->x_row_stride; P.yrs = d->y_row_stride;
  P.KA = fb_pad16(d->kt * d->Cin); P.KB = fb_pad16(9 * d->Cmid); P.KC = fb_pad16(d->Cmid); P.KS = fb_pad16(d->Cin);
  P.ldwa = P.KA + 8; P.ldwb = P.KB + 8; P.ldwc = P.KC + 8; P.ldws = P.KS + 8;
  // ---- tile search: efficient tiles (little halo / m-tile padding) that still give every SM a few CTAs
  const size_t w_bytes = ((size_t)d->Cmid * P.ldwa + (size_t)d->Cmid * P.ldwb + (size_t)d->Cout * P.ldwc +
                          (d->has_shortcut ? (size_t)d->Cout * P.ldws : 0)) * 2;
  const size_t sb_bytes = (size_t)(4 * d->Cmid + 4 * d->Cout) * 4;
  const size_t budget = 200 * 1024;
  int best_th = 0, best_tw = 0, best_tc = 0;
  double best_score = -1;
  for (int th = 2; th <= 16; ++th)
    for (int tw = 2; tw <= 16; ++tw) {
      if (th > P.Ho + 1 || tw > P.Wo + 1) continue;
      const int rh = (th - 1) * d->sb + 3, rw = (tw - 1) * d->sb + 3;
      if (rh * rw > 16 * FB_MT * FB_WARPS || th * tw > 16 * FB_MT * FB_WARPS) continue;       // FB_MT m-tiles per warp
      const size_t xs = (size_t)rh * rw * d->Cin * 2;
      const size_t need = FB_SLOTS * ((xs + 127) & ~(size_t)127) + (((size_t)rh * rw * d->Cmid * 2 + 127) & ~(size_t)127) +
                          (((size_t)th * tw * d->Cmid * 2 + 127) & ~(size_t)127) + (((size_t)th * tw * d->Cout * 2 + 127) & ~(size_t)127) +
                          ((w_bytes + 127) & ~(size_t)127) + sb_bytes + 2048 + 512;
      if (need > budget) continue;
      const long long spatial = (long long)d->N * cdiv(P.Ho, th) * cdiv(P.Wo, tw);
      const int per_sm = (int)(budget / need) > 4 ? 4 : (int)(budget / need);                  // resident CTAs per SM
      int tchunks = 1;
      while (spatial * tchunks < (long long)2 * per_sm * sm_count && d->T / (tchunks + 1) >= 4) ++tchunks;
      const int tc = (int)cdiv(d->T, tchunks);
      const double ctas = (double)spatial * (double)cdiv(d->T, tc);
      const double cover = (double)P.Ho * P.Wo / ((double)cdiv(P.Ho, th) * th * cdiv(P.Wo, tw) * tw);   // edge waste
      const double reuse = (double)(th * tw) * d->sb * d->sb / (double)(rh * rw);                        // spatial halo
      const double mtile = (double)(th * tw) / (double)(cdiv(th * tw, 16) * 16) * (double)(rh * rw) / (double)(cdiv(rh * rw, 16) * 16);
      const double thalo = (double)tc / (double)(tc + 2 * (d->kt / 2));                                  // temporal halo frames
      const double fill = ctas >= (double)per_sm * sm_count ? 1.0 : ctas / ((double)per_sm * sm_count);  // machine filled?
      const double score = cover * reuse * mtile * thalo * fill;
      if (score > best_score) { best_score = score; best_th = th; best_tw = tw; best_tc = tc; }
    }
  if (best_score < 0) { set_error("fused bottleneck: no tile fits in shared memory"); return PV_ERR_UNSUPPORTED; }
  P.TH = best_th; P.TW = best_tw; P.TC = best_tc;
  P.RH = (P.TH - 1) * d->sb + 3; P.RW = (P.TW - 1) * d->sb + 3;
  P.tiles_h = (int)cdiv(P.Ho, P.TH); P.tiles_w = (int)cdiv(P.Wo, P.TW);
  P.tchunks = (int)cdiv(d->T, P.TC);
  {
    unsigned off = 0;
    auto take = [&](size_t bytes) { const unsigned o = off; off += (unsigned)((bytes + 127) & ~(size_t)127); return o; };
    P.x_slot_bytes = (unsigned)(((size_t)P.RH * P.RW * d->Cin * 2 + 127) & ~(size_t)127);
    P.off_x = take((size_t)FB_SLOTS * P.x_slot_bytes);
    P.off_a = take((size_t)P.RH * P.RW * d->Cmid * 2);
    P.off_b = take((size_t)P.TH * P.TW * d->Cmid * 2);
    P.off_y = take((size_t)P.TH * P.TW * d->Cout * 2);
    P.off_wa = take((size_t)d->Cmid * P.ldwa * 2);
    P.off_wb = take((size_t)d->Cmid * P.ldwb * 2);
    P.off_wc = take((size_t)d->Cout * P.ldwc * 2);
    P.off_ws = take(d->has_shortcut ? (size_t)d->Cout * P.ldws * 2 : 16);
    P.off_sb = take(sb_bytes);
    P.off_tab = take(512 * sizeof(int));
    smem_bytes = off;
  }
  return PV_OK;
}

bool fb_aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }
}  // namespace

extern "C" int pv_bottleneck_fused_tiling(const pv_bottleneck_desc* d, int sm_count, int* tile_h, int* tile_w,
                                          int* frames_per_cta, long long* smem_bytes) {
  PV_CHECK_ARG(d && sm_count > 0, "null descriptor or sm_count <= 0");
  if (!pv_bottleneck_fused_supported(d)) { set_error("fused bottleneck: unsupported configuration"); return PV_ERR_UNSUPPORTED; }
  FbParams P;
  size_t smem = 0;
  const int rc = fb_plan(d, sm_count, P, smem);
  if (rc != PV_OK) return rc;
  if (tile_h) *tile_h = P.TH;
  if (tile_w) *tile_w = P.TW;
  if (frames_per_cta) *frames_per_cta = P.TC;
  if (smem_bytes) *smem_bytes = (long long)smem;
  return PV_OK;
}

extern "C" int pv_bottleneck_fused_fwd(const pv_bottleneck_desc* d, const void* x, const void* wa, const void* wb,
                                       const void* wc, const void* wsc, const float* sa, const float* ba,
                                       const float* sb_, const float* bb, const float* sc, const float* bc,
                                       const float* ssc, const float* bsc, void* y, void* stream) {
  PV_CHECK_ARG(d && x && wa && wb && wc && sa && ba && sb_ && bb && sc && bc && y, "null argument");
  if (!pv_bottleneck_fused_supported(d)) { set_error("fused bottleneck: unsupported configuration"); return PV_ERR_UNSUPPORTED; }
  PV_CHECK_ARG(!d->has_shortcut || (wsc && ssc && bsc), "shortcut weights missing");
  // x is read with 16-byte cp.async, y written and the weights loaded as uint4
  PV_CHECK_ARG(fb_aligned16(x) && fb_aligned16(y) && fb_aligned16(wa) && fb_aligned16(wb) && fb_aligned16(wc) &&
                   (!d->has_shortcut || fb_aligned16(wsc)),
               "fused bottleneck: x, y and the weights must be 16-byte aligned");
  const int sm_count = current_sm_count();
  if (sm_count <= 0) { set_error("cannot query the SM count"); return PV_ERR_CUDA; }
  FbParams P;
  size_t smem_bytes = 0;
  const int rc = fb_plan(d, sm_count, P, smem_bytes);
  if (rc != PV_OK) return rc;
  const long long grid = (long long)d->N * P.tchunks * P.tiles_h * P.tiles_w;
  if (grid <= 0) return PV_OK;
  PV_CHECK_ARG(grid < (1ll << 31), "grid too large");
  cudaStream_t s = (cudaStream_t)stream;
#define PV_FB(CI, CM, KT_, SB_, SC_)                                                                                \
  if (d->Cin == CI && d->Cmid == CM && d->kt == KT_ && d->sb == SB_ && (d->has_shortcut ? 1 : 0) == SC_) {          \
    PV_OPT_IN_SMEM((bottleneck_fused_kernel<CI, CM, KT_, SB_, (SC_ != 0)>), 208 * 1024);                            \
    bottleneck_fused_kernel<CI, CM, KT_, SB_, (SC_ != 0)><<<(unsigned)grid, FB_THREADS, smem_bytes, s>>>(           \
        P, (const __half*)x, (const __half*)wa, (const __half*)wb, (const __half*)wc, (const __half*)wsc, sa, ba,   \
        sb_, bb, sc, bc, ssc, bsc, (__half*)y);                                                                     \
    PV_LAUNCH_OK("bottleneck_fused_kernel<" #CI "," #CM "," #KT_ "," #SB_ "," #SC_ ">");                            \
    return PV_OK;                                                                                                   \
  }
  PV_FB(8, 8, 3, 1, 1) PV_FB(32, 8, 3, 1, 0) PV_FB(32, 8, 1, 1, 0)
  PV_FB(32, 16, 3, 2, 1) PV_FB(32, 16, 3, 1, 1) PV_FB(64, 16, 3, 1, 0)
#undef PV_FB
  set_error("fused bottleneck: shape not instantiated");
  return PV_ERR_UNSUPPORTED;
}

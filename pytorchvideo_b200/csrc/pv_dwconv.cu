// Depthwise 3-D convolution as a shared-memory stencil fed by TMA (f16 storage, fp32 accumulate).
//
// One CTA = one box of output positions (bt x bh x bw) x up to 64 channels.  The input halo box
// ((bt-1)*st + (kt-1)*dt + 1, ...) x channels arrives with ONE TMA tiled load; out-of-bounds zero
// fill IS the convolution padding, and an arbitrary per-sample stride covers MViT token tensors
// (cls row in front of every sample).  Every input element therefore leaves L2 once per CTA
// instead of once per tap; the stencil then runs out of shared memory with 4-wide register tiling
// along W (each column converted once per filter row).  Epilogue: folded BN scale/bias, activation,
// optional per-(sample, channel) sums for Squeeze-Excitation (block reduce + one atomic per channel).
// Replaces the depthwise nn.Conv3d of X3D (models/x3d.py:180-189, 74-82), CSN (models/csn.py:169)
// and the MViT pooling convs (layers/attention.py:364-403).
#include "pv_common.cuh"
#include "pv_sm90.cuh"
#include <string.h>

namespace pv {

using namespace sm90;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_fn();   // pv_igemm.cu
int conv3d_check(const pv_conv3d_desc* d);
int conv3d_direct_launch(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                         const float* bias, const void* residual, void* y, cudaStream_t s);
int dwconv3d_lane_launch(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                         const float* bias, void* y, float* se_sums, cudaStream_t stream);   // pv_dwlane.cu

struct DwParams {
  CUtensorMap x_map;          // [Cc(chunk) .. C, W, H, T, N] f16, box [cc, ww, hh, tt, 1], no swizzle
  int C, cc;                  // total (padded) channels, channels per CTA chunk (<= 64, multiple of 8)
  int To, Ho, Wo;
  int bt, bh, bw;             // output box
  int tt, hh, ww;             // input halo box
  int nt_t, nt_h, nt_w;       // tiles per dim
  int kt, kh, st, sh, pt, ph, pw, dt, dh;
  int act;
  long long y_row_stride, y_batch_stride;
  int Ti, Hi, Wi;             // input extent (bounds of the prologue)
  const float* pre_scale;     // PRE: pre-activation prologue (pv_conv3d_desc.pre_*)
  const float* pre_bias;
  int pre_act;
};

// PRE: the pre-activation prologue runs once over the landed halo box (in-bounds positions only), before the stencil.
template <int KW, int SW, bool PRE>
__global__ void __launch_bounds__(256)
dwconv3d_tile_kernel(const __grid_constant__ DwParams P, const __half* __restrict__ w,
                     const float* __restrict__ scale, const float* __restrict__ bias,
                     __half* __restrict__ y, float* __restrict__ se_sums) {
  constexpr int WT = 4;
  constexpr int NCOL = (WT - 1) * SW + KW;
  extern __shared__ __align__(128) uint8_t dw_smem[];
  __shared__ __align__(8) uint64_t bar;
  __shared__ float se_acc[256][8];     // per-thread SE partial sums (one channel group per thread, see the item loop)
  const int cc = P.cc;
  const int halo_elems = P.tt * P.hh * P.ww * cc;
  __half* xs = reinterpret_cast<__half*>(dw_smem);                       // [tt][hh][ww][cc]
  __half* ws = xs + ((halo_elems + 63) & ~63);                           // [kt*kh*KW][cc]

  // ---- tile coordinates
  int tile = blockIdx.x;
  const int tw = tile % P.nt_w; tile /= P.nt_w;
  const int th = tile % P.nt_h; tile /= P.nt_h;
  const int ttile = tile % P.nt_t;
  const int n = tile / P.nt_t;
  const int c0 = blockIdx.y * cc;
  const int to0 = ttile * P.bt, ho0 = th * P.bh, wo0 = tw * P.bw;

  const uint32_t bar_a = smem_u32(&bar);
  if (threadIdx.x == 0) {
    mbar_init(bar_a, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(bar_a, (uint32_t)halo_elems * 2u);
    tma_load_5d(smem_u32(xs), &P.x_map, bar_a, c0, wo0 * SW - P.pw, ho0 * P.sh - P.ph, to0 * P.st - P.pt, n);
  }
  // weights of this channel chunk (overlaps the TMA flight)
  const int taps = P.kt * P.kh * KW;
  for (int i = threadIdx.x; i < taps * (cc >> 3); i += blockDim.x) {
    const int tap = i / (cc >> 3), g8 = (i - tap * (cc >> 3)) * 8;
    *reinterpret_cast<uint4*>(ws + tap * cc + g8) = *reinterpret_cast<const uint4*>(w + (long long)tap * P.C + c0 + g8);
  }
  __syncthreads();
  mbar_wait(bar_a, 0);
  if constexpr (PRE) {
    halo_prologue(xs, 1, P.tt, P.hh, P.ww, cc, c0, P.C, to0 * P.st - P.pt, ho0 * P.sh - P.ph, wo0 * SW - P.pw, P.Ti,
                  P.Hi, P.Wi, P.pre_scale, P.pre_bias, P.pre_act);
    __syncthreads();
  }

  const int G = cc >> 3;
  const int wq_n = (P.bw + WT - 1) / WT;
  const int items = P.bt * P.bh * wq_n * G;
  // The item stride is a multiple of G, so a thread keeps ONE channel group for all its items: the SE
  // partial sums stay in registers and are combined once per CTA without shared-memory atomics.
  const int stride = ((int)blockDim.x / G) * G;
  float se_reg[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) se_reg[i] = 0.f;
  for (int it = threadIdx.x; it < items && (int)threadIdx.x < stride; it += stride) {
    int r = it;
    const int cg = r % G; r /= G;
    const int wq = r % wq_n; r /= wq_n;
    const int h = r % P.bh;
    const int t = r / P.bh;
    const int c = cg * 8;
    const int wl0 = wq * WT;                       // first local output column of this item
    float acc[WT][8];
#pragma unroll
    for (int o = 0; o < WT; ++o)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[o][i] = 0.f;
    for (int kt_ = 0; kt_ < P.kt; ++kt_) {
      const int tz = t * P.st + kt_ * P.dt;
      for (int kh_ = 0; kh_ < P.kh; ++kh_) {
        const int hz = h * P.sh + kh_ * P.dh;
        const __half* row = xs + ((tz * P.hh + hz) * P.ww + wl0 * SW) * cc + c;
        const __half* wr = ws + ((kt_ * P.kh + kh_) * KW) * cc + c;
        float wv[KW][8];
#pragma unroll
        for (int k = 0; k < KW; ++k) ld8<__half>(wr + k * cc, wv[k]);
#pragma unroll
        for (int j = 0; j < NCOL; ++j) {
          float xv[8];
          ld8<__half>(row + j * cc, xv);
#pragma unroll
          for (int o = 0; o < WT; ++o) {
            const int k = j - o * SW;
            if (k >= 0 && k < KW) {
#pragma unroll
              for (int i = 0; i < 8; ++i) acc[o][i] = fmaf(xv[i], wv[k][i], acc[o][i]);
            }
          }
        }
      }
    }
    const int to = to0 + t, ho = ho0 + h;
    if (to >= P.To || ho >= P.Ho) continue;
    float sc[8], bi[8], ssum[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { sc[i] = __ldg(scale + c0 + c + i); bi[i] = __ldg(bias + c0 + c + i); ssum[i] = 0.f; }
#pragma unroll
    for (int o = 0; o < WT; ++o) {
      const int wo = wo0 + wl0 + o;
      if (wo >= P.Wo) break;
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float pre = acc[o][i] * sc[i] + bi[i];
        ssum[i] += pre;
        v[i] = apply_act(pre, P.act);
      }
      st8<__half>(y + (long long)n * P.y_batch_stride + (((long long)to * P.Ho + ho) * P.Wo + wo) * P.y_row_stride + c0 + c, v);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) se_reg[i] += ssum[i];
  }
  if (se_sums) {
#pragma unroll
    for (int i = 0; i < 8; ++i) se_acc[threadIdx.x][i] = se_reg[i];
    __syncthreads();
    if ((int)threadIdx.x < cc) {        // channel c of this chunk: threads t = (c >> 3) + k G hold its partials
      const int cgc = (int)threadIdx.x >> 3, ci = (int)threadIdx.x & 7;
      float tot = 0.f;
      for (int t = cgc; t < stride; t += G) tot += se_acc[t][ci];
      se_sum_add(se_sums, (long long)n * P.C + c0 + threadIdx.x, tot);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Temporal depthwise conv (kt x 1 x 1, stride 1): the X3D stem's conv_xy after the spatial conv (models/x3d.py:74-82;
// layers/convolutions.py:191-237 Conv2plus1d with a depthwise temporal half).  Pure streaming: a thread owns one
// (position, 8-channel group) column and slides a KT-frame register window along T, so every input element is read
// exactly once (16-byte coalesced vectors) and every output written once: (in + out) * 2 B per element, HBM-bound.
// The halo-tile kernel above re-reads the KT-1 overlapping frames of each box through shared memory and ran this layer
// at 1.1 TB/s (X3D-M B=32: 553 us for 617 MB).
// ---------------------------------------------------------------------------------------------------------------
template <int KT>
__global__ void __launch_bounds__(128)
dwconv_temporal_kernel(const __half* __restrict__ x, const __half* __restrict__ w, const float* __restrict__ scale,
                       const float* __restrict__ bias, __half* __restrict__ y, int T, long long hw, int G, int C,
                       long long x_row_stride, long long y_row_stride, long long x_batch_stride,
                       long long y_batch_stride, int act) {
  constexpr int PT = KT / 2;
  // taps and folded BN as fp32 in shared memory (read per use: keeps them out of the register file, see the ring below)
  extern __shared__ __align__(16) float tw_smem[];          // [KT][C] taps, [C] scale, [C] bias
  float* ws = tw_smem;
  float* scs = tw_smem + KT * C;
  float* bis = scs + C;
  for (int i = threadIdx.x; i < KT * C; i += blockDim.x) ws[i] = __half2float(w[i]);
  for (int i = threadIdx.x; i < C; i += blockDim.x) { scs[i] = __ldg(scale + i); bis[i] = __ldg(bias + i); }
  __syncthreads();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= hw * G) return;
  const long long pos = idx / G;
  const int c = (int)(idx - pos * G) * 8;
  const int n = blockIdx.y;
  const __half* xp = x + (long long)n * x_batch_stride + pos * x_row_stride + c;
  __half* yp = y + (long long)n * y_batch_stride + pos * y_row_stride + c;
  const long long xf = hw * x_row_stride, yf = hw * y_row_stride;      // frame strides
  // Ring of 8 raw 16-byte frames: slot f & 7 holds frame f; frames t-PT .. t+PT are the window, the rest is read-ahead
  // (PF = 8 - KT frames in flight per thread).  Everything stays packed f16 until it is used: ~90 registers, so 5 CTAs
  // of 128 threads per SM keep ~30 KB of loads outstanding per SM.
  constexpr int R = 8, PF = R - KT;
  static_assert(KT <= 5, "ring too small");
  uint4 ring[R];
  const uint4 z4 = make_uint4(0, 0, 0, 0);
#pragma unroll
  for (int s = 0; s < R; ++s) ring[s] = z4;
#pragma unroll
  for (int f = 0; f < R - PT; ++f)           // the ring holds frames t-PT .. t-PT+R-1 (frames < 0 stay zero: the padding)
    ring[f & (R - 1)] = f < T ? __ldg(reinterpret_cast<const uint4*>(xp + (long long)f * xf)) : z4;
  for (int t0 = 0; t0 < T; t0 += R) {
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const int t = t0 + j;                  // t & 7 == j: ring slots are compile-time
      if (t >= T) break;
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = 0.f;
#pragma unroll
      for (int k = 0; k < KT; ++k) {
        const __half2* xh = reinterpret_cast<const __half2*>(&ring[(j + k - PT + R) & (R - 1)]);
        const float4 w0 = *reinterpret_cast<const float4*>(ws + k * C + c), w1 = *reinterpret_cast<const float4*>(ws + k * C + c + 4);
        const float wf[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 xf2 = __half22float2(xh[i]);
          v[2 * i] = fmaf(xf2.x, wf[2 * i], v[2 * i]);
          v[2 * i + 1] = fmaf(xf2.y, wf[2 * i + 1], v[2 * i + 1]);
        }
      }
      // frame t-PT leaves the window: its slot takes frame t + PT + PF + 1 - ... = t - PT + R
      const int nf = t - PT + R;
      ring[(j - PT + R) & (R - 1)] = nf < T ? __ldg(reinterpret_cast<const uint4*>(xp + (long long)nf * xf)) : z4;
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = apply_act(v[i] * scs[c + i] + bis[c + i], act);
      st8<__half>(yp + (long long)t * yf, v);
    }
  }
}

int dwconv3d_temporal_launch(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                             const float* bias, void* y, float* se_sums, cudaStream_t stream) {
  if (se_sums || d->dtype != PV_F16 || d->groups != d->Ci || d->Ci != d->Co || d->has_residual) return PV_ERR_UNSUPPORTED;
  if (conv3d_has_prologue(d)) return PV_ERR_UNSUPPORTED;      // the tile kernel and the stencils take the prologue
  if (d->kh != 1 || d->kw != 1 || !(d->kt == 3 || d->kt == 5) || d->st != 1 || d->sh != 1 || d->sw != 1 || d->dt != 1)
    return PV_ERR_UNSUPPORTED;
  if (d->pt != d->kt / 2 || d->ph != 0 || d->pw != 0 || d->Co % 8 || d->x_row_stride % 8 || d->y_row_stride % 8)
    return PV_ERR_UNSUPPORTED;
  const long long hw = (long long)d->Ho * d->Wo;
  const int G = d->Co / 8;
  const long long xbs = d->x_batch_stride ? d->x_batch_stride : (long long)d->Ti * d->Hi * d->Wi * d->x_row_stride;
  const long long ybs = d->y_batch_stride ? d->y_batch_stride : (long long)d->To * d->Ho * d->Wo * d->y_row_stride;
  const long long blocks = (hw * G + 127) / 128;
  if (blocks > 0x7fffffffll || d->N > 65535) return PV_ERR_UNSUPPORTED;
  dim3 grid((unsigned)blocks, (unsigned)d->N), block(128);
  const size_t smem = (size_t)(d->kt + 2) * d->Co * sizeof(float);
  if (smem > 40 * 1024) return PV_ERR_UNSUPPORTED;
  if (d->kt == 5) {
    dwconv_temporal_kernel<5><<<grid, block, smem, stream>>>((const __half*)x, (const __half*)w, scale, bias, (__half*)y, d->To, hw,
                                                        G, d->Co, d->x_row_stride, d->y_row_stride, xbs, ybs, d->act);
    PV_LAUNCH_OK("dwconv_temporal_kernel<5>");
  } else {
    dwconv_temporal_kernel<3><<<grid, block, smem, stream>>>((const __half*)x, (const __half*)w, scale, bias, (__half*)y, d->To, hw,
                                                        G, d->Co, d->x_row_stride, d->y_row_stride, xbs, ybs, d->act);
    PV_LAUNCH_OK("dwconv_temporal_kernel<3>");
  }
  return PV_OK;
}

// Host: returns PV_ERR_UNSUPPORTED when the shape does not qualify (caller falls back).
int dwconv3d_tile_launch(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                         const float* bias, void* y, float* se_sums, cudaStream_t stream) {
  if (d->dtype != PV_F16 || d->groups != d->Ci || d->Ci != d->Co || d->has_residual) return PV_ERR_UNSUPPORTED;
  if (d->dw != 1 || !(d->kw == 3 || d->kw == 1) || !(d->sw == 1 || d->sw == 2)) return PV_ERR_UNSUPPORTED;
  if (d->Co % 8 || d->x_row_stride % 8 || d->y_row_stride % 8) return PV_ERR_UNSUPPORTED;
  EncodeTiledFn encode = get_encode_fn();
  if (!encode) return PV_ERR_UNSUPPORTED;
  DwParams P;
  memset(&P, 0, sizeof(P));
  P.C = d->Co;
  // channel chunk: largest multiple of 8 <= 64 that divides C evenly into equal chunks
  int chunks = (d->Co + 63) / 64;
  while ((d->Co % (chunks * 8)) != 0 && chunks < d->Co / 8) ++chunks;
  P.cc = d->Co / chunks;
  if (P.cc % 8 || P.cc > 64) return PV_ERR_UNSUPPORTED;
  P.To = d->To; P.Ho = d->Ho; P.Wo = d->Wo;
  P.kt = d->kt; P.kh = d->kh; P.st = d->st; P.sh = d->sh; P.pt = d->pt; P.ph = d->ph; P.pw = d->pw;
  P.dt = d->dt; P.dh = d->dh; P.act = d->act;
  P.Ti = d->Ti; P.Hi = d->Hi; P.Wi = d->Wi;
  P.pre_scale = d->pre_scale; P.pre_bias = d->pre_bias; P.pre_act = d->pre_act;
  const bool pre = d->pre_scale != nullptr;
  P.y_row_stride = d->y_row_stride;
  P.y_batch_stride = d->y_batch_stride ? d->y_batch_stride : (long long)d->To * d->Ho * d->Wo * d->y_row_stride;
  // ---- output box search: maximise outputs per halo byte under a 96 KiB halo budget
  const int budget = 96 * 1024;
  double best = -1;
  for (int bw = 4; bw <= 32; bw += 4) {
    if (bw > ((d->Wo + 3) / 4) * 4) break;
    for (int bh = 1; bh <= 16; ++bh) {
      if (bh > d->Ho) break;
      for (int bt = 1; bt <= 16; ++bt) {
        if (bt > d->To) break;
        const int ww = (bw - 1) * d->sw + d->kw, hh = (bh - 1) * d->sh + (d->kh - 1) * d->dh + 1;
        const int tt = (bt - 1) * d->st + (d->kt - 1) * d->dt + 1;
        if (ww > 256 || hh > 256 || tt > 256) continue;
        const long long halo = (long long)tt * hh * ww * P.cc * 2;
        if (halo > budget) continue;
        const int outs = bt * bh * bw;
        if (outs * (P.cc / 8) / 4 < 128) continue;             // keep the CTA busy
        const double waste_w = (double)d->Wo / (((d->Wo + bw - 1) / bw) * bw);
        const double waste_h = (double)d->Ho / (((d->Ho + bh - 1) / bh) * bh);
        const double waste_t = (double)d->To / (((d->To + bt - 1) / bt) * bt);
        const double score = (double)outs / (double)(tt * hh * ww) * waste_w * waste_h * waste_t;
        if (score > best) { best = score; P.bt = bt; P.bh = bh; P.bw = bw; P.tt = tt; P.hh = hh; P.ww = ww; }
      }
    }
  }
  if (best < 0) return PV_ERR_UNSUPPORTED;
  P.nt_t = (d->To + P.bt - 1) / P.bt; P.nt_h = (d->Ho + P.bh - 1) / P.bh; P.nt_w = (d->Wo + P.bw - 1) / P.bw;
  const long long tiles = (long long)d->N * P.nt_t * P.nt_h * P.nt_w;
  if (tiles > 0x7fffffffll || chunks > 65535) return PV_ERR_UNSUPPORTED;
  {
    const long long rs = d->x_row_stride * 2;
    const long long xbs = (d->x_batch_stride ? d->x_batch_stride : (long long)d->Ti * d->Hi * d->Wi * d->x_row_stride) * 2;
    cuuint64_t gdim[5] = {(cuuint64_t)d->Ci, (cuuint64_t)d->Wi, (cuuint64_t)d->Hi, (cuuint64_t)d->Ti, (cuuint64_t)d->N};
    cuuint64_t gstr[4] = {(cuuint64_t)rs, (cuuint64_t)rs * d->Wi, (cuuint64_t)rs * d->Wi * d->Hi, (cuuint64_t)xbs};
    cuuint32_t box[5] = {(cuuint32_t)P.cc, (cuuint32_t)P.ww, (cuuint32_t)P.hh, (cuuint32_t)P.tt, 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult cr = encode(&P.x_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(x), gdim, gstr, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) return PV_ERR_UNSUPPORTED;
  }
  const int halo_elems = P.tt * P.hh * P.ww * P.cc;
  const size_t smem = (size_t)(((halo_elems + 63) & ~63) + d->kt * d->kh * d->kw * P.cc) * 2 + 128;
  dim3 grid((unsigned)tiles, (unsigned)chunks), block(256);
#define PV_DWT2(KW_, SW_, PRE_)                                                                               \
  do {                                                                                                        \
    PV_OPT_IN_SMEM((dwconv3d_tile_kernel<KW_, SW_, PRE_>), 110 * 1024);                                       \
    dwconv3d_tile_kernel<KW_, SW_, PRE_><<<grid, block, smem, stream>>>(P, (const __half*)w, scale, bias, (__half*)y, \
                                                                        se_sums);                             \
    if (PRE_) PV_LAUNCH_OK("dwconv3d_tile_kernel<" #KW_ "," #SW_ ",pre>");                                    \
    else PV_LAUNCH_OK("dwconv3d_tile_kernel<" #KW_ "," #SW_ ">");                                             \
  } while (0)
#define PV_DWT(KW_, SW_)                                                                                      \
  do {                                                                                                        \
    if (pre) PV_DWT2(KW_, SW_, true); else PV_DWT2(KW_, SW_, false);                                          \
  } while (0)
  if (d->kw == 3 && d->sw == 1) PV_DWT(3, 1);
  else if (d->kw == 3) PV_DWT(3, 2);
  else if (d->sw == 1) PV_DWT(1, 1);
  else PV_DWT(1, 2);
#undef PV_DWT
#undef PV_DWT2
  return PV_OK;
}

}  // namespace pv

// Depthwise conv with optional fused Squeeze-Excitation channel sums (se_sums[n][C] += sum over
// positions of the pre-activation output; must be zeroed by the caller).  Falls through to the
// generic CUDA-core stencil when the TMA-tiled kernel does not apply (f32 storage, dilated W, ...).
extern "C" int pv_dwconv3d_fwd(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                               const float* bias, void* y, float* se_sums, void* stream) {
  PV_CHECK_ARG(d && x && w && scale && bias && y, "null pointer");
  PV_CHECK_ARG(d->groups == d->Ci && d->Ci == d->Co, "pv_dwconv3d_fwd is depthwise only");
  PV_CHECK_ARG(!d->has_residual, "pv_dwconv3d_fwd has no residual input");
  PV_CHECK_ARG(!d->addend, "pv_dwconv3d_fwd has no addend input");
  int rc = pv::conv3d_check(d);
  if (rc != PV_OK) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  // 3x3x3: lane-per-channel-pair register stencil (pv_dwlane.cu)
  rc = pv::dwconv3d_lane_launch(d, x, w, scale, bias, y, se_sums, s);
  if (rc != PV_ERR_UNSUPPORTED) return rc;
  // kt x 1 x 1: streaming register window
  rc = pv::dwconv3d_temporal_launch(d, x, w, scale, bias, y, se_sums, s);
  if (rc != PV_ERR_UNSUPPORTED) return rc;
  rc = pv::dwconv3d_tile_launch(d, x, w, scale, bias, y, se_sums, s);
  if (rc != PV_ERR_UNSUPPORTED) return rc;
  // generic path: stencil kernel, then (if requested) a separate channel-sum pass
  int rc2 = pv::conv3d_direct_launch(d, x, w, scale, bias, nullptr, y, s);
  if (rc2 != PV_OK || !se_sums) return rc2;
  if (d->act != PV_ACT_NONE) { pv::set_error("fused SE sums need act == none on the generic path"); return PV_ERR_UNSUPPORTED; }
  return pv_channel_sum(y, d->dtype, d->y_row_stride, d->N, (long long)d->To * d->Ho * d->Wo, d->Co, se_sums, stream);
}

// Depthwise 3x3 convolution over a single-frame token plane (kt = 1, T = 1): the attention pools of the image MViT
// (layers/attention.py:364-403 with kernel (1,3,3), strides (1,1,1), (1,2,2) and (1,4,4)).
//
// Same scheme as the 3x3x3 lane kernel (pv_dwlane.cu): a warp covers the <= 32 channel PAIRS of a chunk (lane = pair:
// one warp-wide read of an input position is one conflict-free 128-byte shared-memory row) and a thread owns a PH x PW
// patch of outputs of its pair.  The 9 taps of the pair stay in registers as fp32; each input position of the patch's
// halo is read once and feeds every output that uses it.  Accumulation is fp32, the output is rounded to f16 once after the
// folded scale and bias (no activation: the pools feed a LayerNorm or the attention core).
//
// A CTA loads its halo box [bn][hh][ww][cc] with ONE 5-D TMA tiled load (the T extent is 1; out-of-bounds fill = the
// zero padding; the batch stride steps over the cls row in front of every sample).  Small planes (7x7, 14x14) take
// several samples per CTA so a CTA still has a patch for every warp.  At stride 4 no input position feeds two outputs
// and a quarter of the halo's rows and columns feed none, so there each lane loads its 9 taps per output straight from
// global memory (one coalesced 128-byte row per warp and tap) instead of staging a halo box.
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

struct DwPlaneParams {
  CUtensorMap x_map;          // [C, W, H, 1, N] f16, box [cc, ww, hh, 1, bn], no swizzle
  int C, cc, N;               // real (padded-to-8) channels, channels per CTA chunk (<= 64, multiple of 8), samples
  int Ho, Wo;
  int bn, bh, bw;             // output box (bh % PH == 0, bw % PW == 0)
  int hh, ww;                 // input halo box
  int nt_n, nt_h, nt_w;       // tiles per dim
  int ph, pw;
  long long y_row_stride, y_batch_stride;
  const __half* x;            // stride 4 only: x read straight from global memory
  int Hi, Wi;
  long long x_row_stride, x_batch_stride;
  const float* pre_scale;     // PRE: pre-activation prologue (pv_conv3d_desc.pre_*)
  const float* pre_bias;
  int pre_act;
};

constexpr int kPlaneWarps = 4;

// PRE: the pre-activation prologue, once per input element: over the landed halo box (in-bounds positions only), or at
// stride 4, where every input position feeds at most one output, on each tap as it is loaded.
template <int S, int PH, int PW, bool PRE>
__global__ void __launch_bounds__(kPlaneWarps * 32, 4)
dwconv_plane_kernel(const __grid_constant__ DwPlaneParams P, const __half* __restrict__ w,
                    const float* __restrict__ scale, const float* __restrict__ bias, __half* __restrict__ y) {
  constexpr int IH = (PH - 1) * S + 3, IW = (PW - 1) * S + 3;
  extern __shared__ __align__(128) uint8_t dwp_smem[];
  __shared__ __align__(8) uint64_t bar;
  const __half* xs = reinterpret_cast<const __half*>(dwp_smem);          // [bn][hh][ww][cc]
  const int cc = P.cc;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  int tile = blockIdx.x;
  const int tw = tile % P.nt_w; tile /= P.nt_w;
  const int th = tile % P.nt_h;
  const int tn = tile / P.nt_h;
  const int c0 = blockIdx.y * cc;
  const int n0 = tn * P.bn, ho0 = th * P.bh, wo0 = tw * P.bw;

  const uint32_t bar_a = smem_u32(&bar);
  if (S != 4 && threadIdx.x == 0) {
    mbar_init(bar_a, 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(bar_a, (uint32_t)(P.bn * P.hh * P.ww * cc) * 2u);
    tma_load_5d(smem_u32(dwp_smem), &P.x_map, bar_a, c0, wo0 * S - P.pw, ho0 * S - P.ph, 0, n0);
  }
  // this lane's channel pair: filter taps, folded scale / bias (overlaps the TMA flight)
  const int ch = c0 + 2 * lane;
  const bool live = (2 * lane < cc) && (ch < P.C);
  float2 wr[9];
#pragma unroll
  for (int t = 0; t < 9; ++t)
    wr[t] = live ? __half22float2(*reinterpret_cast<const __half2*>(w + (long long)t * P.C + ch)) : make_float2(0.f, 0.f);
  const float2 sc = live ? make_float2(__ldg(scale + ch), __ldg(scale + ch + 1)) : make_float2(0.f, 0.f);
  const float2 bi = live ? make_float2(__ldg(bias + ch), __ldg(bias + ch + 1)) : make_float2(0.f, 0.f);
  const int lane_off = live ? 2 * lane : 0;
  if constexpr (S != 4) {
    __syncthreads();          // barrier initialised before anyone waits on it
    mbar_wait(bar_a, 0);
    if constexpr (PRE) {
      halo_prologue(reinterpret_cast<__half*>(dwp_smem), P.bn, 1, P.hh, P.ww, cc, c0, P.C, 0, ho0 * S - P.ph,
                    wo0 * S - P.pw, 1, P.Hi, P.Wi, P.pre_scale, P.pre_bias, P.pre_act);
      __syncthreads();
    }
  }
  float2 pps = make_float2(1.f, 1.f), ppb = make_float2(0.f, 0.f);
  if (PRE && S == 4 && live) {
    pps = make_float2(__ldg(P.pre_scale + ch), __ldg(P.pre_scale + ch + 1));
    ppb = make_float2(__ldg(P.pre_bias + ch), __ldg(P.pre_bias + ch + 1));
  }

  const int npw = P.bw / PW, nph = P.bh / PH;
  const int total = P.bn * nph * npw;
  const int row_e = P.ww * cc;                       // elements per halo row
  for (int p = warp; p < total; p += kPlaneWarps) {
    const int pwi = p % npw;
    const int r = p / npw;
    const int phi = r % nph, nb = r / nph;
    float2 acc[PH][PW];
#pragma unroll
    for (int a = 0; a < PH; ++a)
#pragma unroll
      for (int b = 0; b < PW; ++b) acc[a][b] = make_float2(0.f, 0.f);
    if constexpr (S == 4) {
      // stride 4: no input position feeds two outputs, so there is nothing to share through shared memory and a halo
      // box would also carry the quarter of rows and columns no tap reads; each lane loads exactly its 9 taps
      const int n = n0 + nb;
      if (n < P.N && live) {
        const __half* xn = P.x + (long long)n * P.x_batch_stride + ch;
#pragma unroll
        for (int a = 0; a < PH; ++a) {
#pragma unroll
          for (int kh = 0; kh < 3; ++kh) {
            const int h = (ho0 + phi * PH + a) * 4 - P.ph + kh;
            if (h < 0 || h >= P.Hi) continue;
#pragma unroll
            for (int b = 0; b < PW; ++b) {
#pragma unroll
              for (int kw = 0; kw < 3; ++kw) {
                const int wi = (wo0 + pwi * PW + b) * 4 - P.pw + kw;
                if (wi < 0 || wi >= P.Wi) continue;
                float2 xv = __half22float2(
                    __ldg(reinterpret_cast<const __half2*>(xn + ((long long)h * P.Wi + wi) * P.x_row_stride)));
                if constexpr (PRE) {
                  xv.x = pre_u(xv.x, pps.x, ppb.x, P.pre_act);
                  xv.y = pre_u(xv.y, pps.y, ppb.y, P.pre_act);
                }
                acc[a][b].x = fmaf(xv.x, wr[kh * 3 + kw].x, acc[a][b].x);
                acc[a][b].y = fmaf(xv.y, wr[kh * 3 + kw].y, acc[a][b].y);
              }
            }
          }
        }
      }
    } else {
      const __half* base = xs + ((nb * P.hh + phi * PH * S) * P.ww + pwi * PW * S) * cc + lane_off;
#pragma unroll
      for (int i = 0; i < IH; ++i) {
#pragma unroll
        for (int j = 0; j < IW; ++j) {
          const float2 xv = __half22float2(*reinterpret_cast<const __half2*>(base + i * row_e + j * cc));
#pragma unroll
          for (int kh = 0; kh < 3; ++kh) {
            if (i - kh < 0 || (i - kh) % S != 0 || (i - kh) / S >= PH) continue;
#pragma unroll
            for (int kw = 0; kw < 3; ++kw) {
              if (j - kw < 0 || (j - kw) % S != 0 || (j - kw) / S >= PW) continue;
              float2& a = acc[(i - kh) / S][(j - kw) / S];
              const float2 wv = wr[kh * 3 + kw];
              a.x = fmaf(xv.x, wv.x, a.x);
              a.y = fmaf(xv.y, wv.y, a.y);
            }
          }
        }
      }
    }
    const int n = n0 + nb;
    if (!live || n >= P.N) continue;
    const int ho_b = ho0 + phi * PH, wo_b = wo0 + pwi * PW;
    __half* yrow = y + (long long)n * P.y_batch_stride + ch + ((long long)ho_b * P.Wo + wo_b) * P.y_row_stride;
    const long long y_hstep = (long long)P.Wo * P.y_row_stride;
#pragma unroll
    for (int a = 0; a < PH; ++a) {
      if (ho_b + a >= P.Ho) break;
      __half* yp = yrow + a * y_hstep;
#pragma unroll
      for (int b = 0; b < PW; ++b) {
        if (wo_b + b >= P.Wo) break;
        *reinterpret_cast<__half2*>(yp) = __floats2half2_rn(acc[a][b].x * sc.x + bi.x, acc[a][b].y * sc.y + bi.y);
        yp += P.y_row_stride;
      }
    }
  }
}

// Host-side shape rules of the plane kernel (see pv_dwplane_supported in pv_b200.h).
static bool dwplane_takes(const pv_conv3d_desc* d) {
  if (d->dtype != PV_F16 || d->groups != d->Ci || d->Ci != d->Co || d->has_residual || d->addend) return false;
  if (d->act != PV_ACT_NONE) return false;
  if (d->Ti != 1 || d->To != 1 || d->kt != 1 || d->st != 1 || d->pt != 0) return false;
  if (d->kh != 3 || d->kw != 3 || d->dt != 1 || d->dh != 1 || d->dw != 1) return false;
  if (d->sh != d->sw || !(d->sw == 1 || d->sw == 2 || d->sw == 4)) return false;
  if (d->ph < 0 || d->ph > 2 || d->pw < 0 || d->pw > 2) return false;
  if (d->Co % 8 || d->x_row_stride % 8 || d->y_row_stride % 2 || d->x_batch_stride % 8) return false;
  if (d->N < 1 || d->Hi < 1 || d->Wi < 1 || d->Ho < 1 || d->Wo < 1) return false;
  if (d->Ho != (d->Hi + 2 * d->ph - 3) / d->sh + 1 || d->Wo != (d->Wi + 2 * d->pw - 3) / d->sw + 1) return false;
  return true;
}

}  // namespace pv

extern "C" int pv_dwplane_supported(const pv_conv3d_desc* d) {
  return d && pv::dwplane_takes(d) ? 1 : 0;
}

extern "C" int pv_dwplane_fwd(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                              const float* bias, void* y, void* stream) {
  using namespace pv;
  PV_CHECK_ARG(d && x && w && scale && bias && y, "null pointer");
  PV_CHECK_ARG(((uintptr_t)x & 15) == 0 && ((uintptr_t)y & 3) == 0 && ((uintptr_t)w & 3) == 0,
               "pv_dwplane_fwd: x must be 16-byte and y, w 4-byte aligned");
  PV_CHECK_ARG(conv3d_prologue_ok(d), "prologue: pre_scale and pre_bias both set, pre_act a known activation code");
  if (!dwplane_takes(d)) {
    set_error("pv_dwplane_fwd: f16 depthwise (1,3,3) on a one-frame plane, sh == sw in {1, 2, 4}, padding <= 2, "
              "no activation, channels and row / batch strides multiples of 8 (got k=(%d,%d,%d) s=(%d,%d,%d) T=%d)",
              d->kt, d->kh, d->kw, d->st, d->sh, d->sw, d->Ti);
    return PV_ERR_UNSUPPORTED;
  }
  EncodeTiledFn encode = get_encode_fn();
  if (!encode) { set_error("pv_dwplane_fwd: cuTensorMapEncodeTiled is unavailable"); return PV_ERR_CUDA; }
  const int S = d->sw;
  DwPlaneParams P;
  memset(&P, 0, sizeof(P));
  P.C = d->Co;
  P.N = d->N;
  const int chunks = (d->Co + 63) / 64;
  P.cc = (((d->Co + chunks - 1) / chunks) + 7) & ~7;       // near-equal chunks; the last one may run past C (TMA zero fill)
  P.Ho = d->Ho; P.Wo = d->Wo;
  P.ph = d->ph; P.pw = d->pw;
  P.y_row_stride = d->y_row_stride;
  P.y_batch_stride = d->y_batch_stride ? d->y_batch_stride : (long long)d->Ho * d->Wo * d->y_row_stride;
  P.x = (const __half*)x; P.Hi = d->Hi; P.Wi = d->Wi;
  P.x_row_stride = d->x_row_stride;
  P.x_batch_stride = d->x_batch_stride ? d->x_batch_stride : (long long)d->Hi * d->Wi * d->x_row_stride;
  P.pre_scale = d->pre_scale; P.pre_bias = d->pre_bias; P.pre_act = d->pre_act;
  const bool pre = d->pre_scale != nullptr;
  // patch shape: 4x4 unless the plane is a multiple of 7 wide but not of 4 (14x14, 7x7 planes): 2x7
  // stride 4 (loads straight from global memory): 1x2 patches, so enough warps are in flight to hide the latency
  const bool p27 = (d->Wo % 4 != 0) && (d->Wo % 7 == 0);
  const int PH = S == 4 ? 1 : p27 ? 2 : 4, PW = S == 4 ? 2 : p27 ? 7 : 4;
  // ---- output box: every warp busy, little padding waste, then halo reuse; 50 KB keeps four CTAs per SM
  const int budget = 50 * 1024;
  double best = -1;
  for (int bw = PW; bw <= 56; bw += PW) {
    if (bw - PW >= d->Wo) break;
    for (int bh = PH; bh <= 32; bh += PH) {
      if (bh - PH >= d->Ho) break;
      for (int bn = 1; bn <= 16; ++bn) {
        if (bn > d->N) break;
        const int ww = (bw - 1) * S + 3, hh = (bh - 1) * S + 3;
        if (ww > 256 || hh > 256) continue;
        const long long halo = (long long)bn * hh * ww * P.cc * 2;
        if (S != 4 && halo > budget) continue;
        const int patches = bn * (bh / PH) * (bw / PW);
        const double warp_eff = (double)patches / (double)(((patches + kPlaneWarps - 1) / kPlaneWarps) * kPlaneWarps);
        const double cov_w = (double)d->Wo / (((d->Wo + bw - 1) / bw) * bw);
        const double cov_h = (double)d->Ho / (((d->Ho + bh - 1) / bh) * bh);
        const double cov_n = (double)d->N / (((d->N + bn - 1) / bn) * bn);
        const double reuse = (double)(bh * bw) / (double)(hh * ww);
        const double score = warp_eff * cov_w * cov_h * cov_n * (0.75 + 0.25 * reuse) *
                             (patches >= 2 * kPlaneWarps ? 1.0 : 0.9);
        if (score > best) { best = score; P.bn = bn; P.bh = bh; P.bw = bw; P.hh = hh; P.ww = ww; }
      }
    }
  }
  if (best < 0) { set_error("pv_dwplane_fwd: no output box fits"); return PV_ERR_UNSUPPORTED; }
  P.nt_n = (d->N + P.bn - 1) / P.bn; P.nt_h = (d->Ho + P.bh - 1) / P.bh; P.nt_w = (d->Wo + P.bw - 1) / P.bw;
  const long long tiles = (long long)P.nt_n * P.nt_h * P.nt_w;
  if (tiles > 0x7fffffffll || chunks > 65535) { set_error("pv_dwplane_fwd: grid too large"); return PV_ERR_UNSUPPORTED; }
  // stride 4 reads x straight from global memory: no tensor map (its box, sized without the shared-memory budget, can
  // be one the driver rejects, as for the image MViT's 56x56 K/V pool at batch 3)
  if (S != 4) {
    const long long rs = d->x_row_stride * 2;
    const long long xbs = (d->x_batch_stride ? d->x_batch_stride : (long long)d->Hi * d->Wi * d->x_row_stride) * 2;
    cuuint64_t gdim[5] = {(cuuint64_t)d->Ci, (cuuint64_t)d->Wi, (cuuint64_t)d->Hi, 1, (cuuint64_t)d->N};
    cuuint64_t gstr[4] = {(cuuint64_t)rs, (cuuint64_t)rs * d->Wi, (cuuint64_t)rs * d->Wi * d->Hi, (cuuint64_t)xbs};
    cuuint32_t box[5] = {(cuuint32_t)P.cc, (cuuint32_t)P.ww, (cuuint32_t)P.hh, 1, (cuuint32_t)P.bn};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult cr = encode(&P.x_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(x), gdim, gstr, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) { set_error("pv_dwplane_fwd: tensor map rejected (%d)", (int)cr); return PV_ERR_CUDA; }
  }
  const size_t smem = S == 4 ? 256 : (size_t)P.bn * P.hh * P.ww * P.cc * 2 + 256;
  dim3 grid((unsigned)tiles, (unsigned)chunks), block(kPlaneWarps * 32);
  cudaStream_t s = (cudaStream_t)stream;
#define PV_DWP2(S_, PH_, PW_, PRE_)                                                                           \
  do {                                                                                                        \
    PV_OPT_IN_SMEM((dwconv_plane_kernel<S_, PH_, PW_, PRE_>), 52 * 1024);                                     \
    dwconv_plane_kernel<S_, PH_, PW_, PRE_><<<grid, block, smem, s>>>(P, (const __half*)w, scale, bias,        \
                                                                      (__half*)y);                            \
    if (PRE_) PV_LAUNCH_OK("dwconv_plane_kernel<" #S_ "," #PH_ "," #PW_ ",pre>");                             \
    else PV_LAUNCH_OK("dwconv_plane_kernel<" #S_ "," #PH_ "," #PW_ ">");                                      \
  } while (0)
#define PV_DWP(S_, PH_, PW_)                                                                                  \
  do {                                                                                                        \
    if (pre) PV_DWP2(S_, PH_, PW_, true); else PV_DWP2(S_, PH_, PW_, false);                                  \
  } while (0)
  if (S == 1 && !p27) PV_DWP(1, 4, 4);
  else if (S == 1) PV_DWP(1, 2, 7);
  else if (S == 2 && !p27) PV_DWP(2, 4, 4);
  else if (S == 2) PV_DWP(2, 2, 7);
  else PV_DWP(4, 1, 2);
#undef PV_DWP
#undef PV_DWP2
  return PV_OK;
}

// Depthwise 3x3x3 convolution, "one lane = one channel pair" register-tiled stencil (round 2).
//
// The first TMA-halo stencil (pv_dwconv.cu) gives a thread 4 outputs x 8 channels: every filter row re-reads and
// re-converts 3 weight vectors and 6 input vectors from shared memory, so only ~31 % of its issue slots are FFMA and its
// shared-memory traffic (one 16-byte LDS per 24 FMA) is as much a limit as the issue rate: 1.0 TB/s of 6.6 on X3D-M.
// Here a warp covers the <= 32 channel PAIRS of a chunk (lane = pair, so a warp-wide shared-memory read of one input
// position is one conflict-free 128-byte row) and a thread owns a PH x PW patch of outputs of its pair:
//   * the 27 filter taps of the pair live in registers as fp32 for the whole CTA (54 registers);
//   * per filter frame the (PH-1)*S+3 x (PW-1)*S+3 input patch is read ONCE (one 4-byte LDS + one half2->float2 convert
//     per input position) and every value feeds up to 9 outputs x 2 channels: 16 FMA per LDS at S = 1;
//   * accumulators stay in registers over the three filter frames; folded BN, activation, the optional
//     Squeeze-Excitation channel sums (pre-activation, models/x3d.py:190-208) and the f16 store follow.
// The halo box still arrives by ONE 5-D TMA tiled load per CTA (out-of-bounds fill = the convolution padding; the batch
// stride covers MViT's cls row).  Bound: fp32 FMA pipe (27 FMA per output); X3D-M B=32 needs 22 GFMA = 0.61 ms at
// 128 FMA/clk/SM, HBM 3.2 GB = 0.49 ms.
// Replaces depthwise nn.Conv3d 3x3x3 of X3D (models/x3d.py:180-189), CSN (models/csn.py:169) and the MViT pooling
// convs (layers/attention.py:364-403).
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

struct DwLaneParams {
  CUtensorMap x_map;          // [C, W, H, T, N] f16, box [cc, ww, hh, tt, 1], no swizzle
  int C, cc;                  // real (padded-to-8) channels, channels per CTA chunk (<= 64, multiple of 8)
  int To, Ho, Wo;
  int bt, bh, bw;             // output box (bh % PH == 0, bw % PW == 0)
  int tt, hh, ww;             // input halo box
  int nt_t, nt_h, nt_w;       // tiles per dim
  int st, pt, ph, pw;         // temporal stride, paddings
  int act;
  long long y_row_stride, y_batch_stride;
  int Ti, Hi, Wi;             // input extent (bounds of the prologue)
  const float* pre_scale;     // PRE: pre-activation prologue (pv_conv3d_desc.pre_*)
  const float* pre_bias;
  int pre_act;
};


// Four warps and at most 50 KB of halo per CTA: four CTAs per SM, whose TMA waits stagger.
constexpr int DWL_WARPS = 4;
constexpr int DWL_SMEM_BUDGET = 50 * 1024;

// PRE: the pre-activation prologue runs once over the landed halo box (in-bounds positions only), before the stencil.
template <int S, int PH, int PW, bool PRE>
__global__ void __launch_bounds__(DWL_WARPS * 32, 16 / DWL_WARPS)
dwconv3d_lane_kernel(const __grid_constant__ DwLaneParams P, const __half* __restrict__ w,
                     const float* __restrict__ scale, const float* __restrict__ bias,
                     __half* __restrict__ y, float* __restrict__ se_sums) {
  constexpr int IH = (PH - 1) * S + 3, IW = (PW - 1) * S + 3;
  extern __shared__ __align__(128) uint8_t dwl_smem[];
  __shared__ __align__(8) uint64_t bar;
  __shared__ float2 se_part[DWL_WARPS][32];
  const __half* xs = reinterpret_cast<const __half*>(dwl_smem);          // [tt][hh][ww][cc]
  const int cc = P.cc;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

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
    mbar_arrive_expect_tx(bar_a, (uint32_t)(P.tt * P.hh * P.ww * cc) * 2u);
    tma_load_5d(smem_u32(dwl_smem), &P.x_map, bar_a, c0, wo0 * S - P.pw, ho0 * S - P.ph, to0 * P.st - P.pt, n);
  }
  // this lane's channel pair: filter taps, folded BN (overlaps the TMA flight)
  const int ch = c0 + 2 * lane;
  const bool live = (2 * lane < cc) && (ch < P.C);
  float2 wr[27];
#pragma unroll
  for (int t = 0; t < 27; ++t)
    wr[t] = live ? __half22float2(*reinterpret_cast<const __half2*>(w + (long long)t * P.C + ch)) : make_float2(0.f, 0.f);
  const float2 sc = live ? make_float2(__ldg(scale + ch), __ldg(scale + ch + 1)) : make_float2(0.f, 0.f);
  const float2 bi = live ? make_float2(__ldg(bias + ch), __ldg(bias + ch + 1)) : make_float2(0.f, 0.f);
  const int lane_off = live ? 2 * lane : 0;
  __syncthreads();          // barrier initialised before anyone waits on it
  mbar_wait(bar_a, 0);
  if constexpr (PRE) {
    halo_prologue(reinterpret_cast<__half*>(dwl_smem), 1, P.tt, P.hh, P.ww, cc, c0, P.C, to0 * P.st - P.pt,
                  ho0 * S - P.ph, wo0 * S - P.pw, P.Ti, P.Hi, P.Wi, P.pre_scale, P.pre_bias, P.pre_act);
    __syncthreads();
  }

  const int npw = P.bw / PW, nph = P.bh / PH;
  const int total = P.bt * nph * npw;
  const int row_e = P.ww * cc;                       // elements per halo row
  float2 se = make_float2(0.f, 0.f);
  for (int p = warp; p < total; p += DWL_WARPS) {
    const int pwi = p % npw;
    const int r = p / npw;
    const int phi = r % nph, t = r / nph;
    float2 acc[PH][PW];
#pragma unroll
    for (int a = 0; a < PH; ++a)
#pragma unroll
      for (int b = 0; b < PW; ++b) acc[a][b] = make_float2(0.f, 0.f);
#pragma unroll
    for (int kt = 0; kt < 3; ++kt) {
      const __half* base = xs + (((t * P.st + kt) * P.hh + phi * PH * S) * P.ww + pwi * PW * S) * cc + lane_off;
#pragma unroll
      for (int i = 0; i < IH; ++i) {
        const __half* rp = base + i * row_e;
#pragma unroll
        for (int j = 0; j < IW; ++j) {
          const float2 xv = __half22float2(*reinterpret_cast<const __half2*>(rp));
          rp += cc;
#pragma unroll
          for (int kh = 0; kh < 3; ++kh) {
            if (i - kh < 0 || (i - kh) % S != 0 || (i - kh) / S >= PH) continue;
#pragma unroll
            for (int kw = 0; kw < 3; ++kw) {
              if (j - kw < 0 || (j - kw) % S != 0 || (j - kw) / S >= PW) continue;
              float2& a = acc[(i - kh) / S][(j - kw) / S];
              const float2 wv = wr[(kt * 3 + kh) * 3 + kw];
              a.x = fmaf(xv.x, wv.x, a.x);     // the lane's two channels: Hopper has no packed fp32 FMA
              a.y = fmaf(xv.y, wv.y, a.y);
            }
          }
        }
      }
    }
    const int to = to0 + t;
    if (!live || to >= P.To) continue;
    const int ho_b = ho0 + phi * PH, wo_b = wo0 + pwi * PW;
    __half* yrow = y + (long long)n * P.y_batch_stride + ch + (((long long)to * P.Ho + ho_b) * P.Wo + wo_b) * P.y_row_stride;
    const long long y_hstep = (long long)P.Wo * P.y_row_stride;
    // the activation is CTA-uniform: branch once around the whole patch, not per value
    auto store_patch = [&](auto actf) {
#pragma unroll
      for (int a = 0; a < PH; ++a) {
        if (ho_b + a >= P.Ho) break;
        __half* yp = yrow + a * y_hstep;
#pragma unroll
        for (int b = 0; b < PW; ++b) {
          if (wo_b + b >= P.Wo) break;
          const float px = acc[a][b].x * sc.x + bi.x, py = acc[a][b].y * sc.y + bi.y;
          se.x += px; se.y += py;
          *reinterpret_cast<__half2*>(yp) = __floats2half2_rn(actf(px), actf(py));
          yp += P.y_row_stride;
        }
      }
    };
    if (P.act == PV_ACT_NONE) store_patch([](float v) { return v; });
    else if (P.act == PV_ACT_RELU) store_patch([](float v) { return fmaxf(v, 0.f); });
    else if (P.act == PV_ACT_SWISH) store_patch([](float v) { return __fdividef(v, 1.f + __expf(-v)); });
    else store_patch([&](float v) { return apply_act(v, P.act); });
  }
  if (se_sums) {
    se_part[warp][lane] = se;
    __syncthreads();
    if (warp == 0 && live) {
      float2 tot = make_float2(0.f, 0.f);
#pragma unroll
      for (int k = 0; k < DWL_WARPS; ++k) { tot.x += se_part[k][lane].x; tot.y += se_part[k][lane].y; }
      se_sum_add(se_sums, (long long)n * P.C + ch, tot.x);
      se_sum_add(se_sums, (long long)n * P.C + ch + 1, tot.y);
    }
  }
}

// Host: returns PV_ERR_UNSUPPORTED when the shape does not qualify (caller falls back to the generic tile kernel).
int dwconv3d_lane_launch(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                         const float* bias, void* y, float* se_sums, cudaStream_t stream) {
  if (d->dtype != PV_F16 || d->groups != d->Ci || d->Ci != d->Co || d->has_residual) return PV_ERR_UNSUPPORTED;
  if (d->kt != 3 || d->kh != 3 || d->kw != 3 || d->dt != 1 || d->dh != 1 || d->dw != 1) return PV_ERR_UNSUPPORTED;
  if (d->sh != d->sw || !(d->sw == 1 || d->sw == 2) || d->st < 1 || d->st > 2) return PV_ERR_UNSUPPORTED;
  if (d->Co % 8 || d->x_row_stride % 8 || d->y_row_stride % 2) return PV_ERR_UNSUPPORTED;
  EncodeTiledFn encode = get_encode_fn();
  if (!encode) return PV_ERR_UNSUPPORTED;
  const int S = d->sw;
  DwLaneParams P;
  memset(&P, 0, sizeof(P));
  P.C = d->Co;
  const int chunks = (d->Co + 63) / 64;
  P.cc = (((d->Co + chunks - 1) / chunks) + 7) & ~7;       // near-equal chunks; the last one may run past C (TMA zero fill)
  if (P.cc > 64) return PV_ERR_UNSUPPORTED;
  P.To = d->To; P.Ho = d->Ho; P.Wo = d->Wo;
  P.st = d->st; P.pt = d->pt; P.ph = d->ph; P.pw = d->pw; P.act = d->act;
  P.y_row_stride = d->y_row_stride;
  P.y_batch_stride = d->y_batch_stride ? d->y_batch_stride : (long long)d->To * d->Ho * d->Wo * d->y_row_stride;
  P.Ti = d->Ti; P.Hi = d->Hi; P.Wi = d->Wi;
  P.pre_scale = d->pre_scale; P.pre_bias = d->pre_bias; P.pre_act = d->pre_act;
  const bool pre = d->pre_scale != nullptr;
  // patch shape: 4x4 unless the plane is a multiple of 7 wide but not of 4 (14x14, 7x7 planes): 2x7
  const bool p27 = (d->Wo % 4 != 0) && (d->Wo % 7 == 0);
  const int PH = p27 ? 2 : 4, PW = p27 ? 7 : 4;
  // ---- output box: maximise useful outputs per halo byte under a budget that keeps 16 / DWL_WARPS CTAs per SM
  constexpr int nw = DWL_WARPS;
  double best = -1;
  for (int bw = PW; bw <= 56; bw += PW) {
    if (bw - PW >= d->Wo) break;
    for (int bh = PH; bh <= 32; bh += PH) {
      if (bh - PH >= d->Ho) break;
      for (int bt = 1; bt <= 16; ++bt) {
        if (bt > d->To) break;
        const int ww = (bw - 1) * S + 3, hh = (bh - 1) * S + 3, tt = (bt - 1) * d->st + 3;
        if (ww > 256 || hh > 256 || tt > 256) continue;
        const long long halo = (long long)tt * hh * ww * P.cc * 2;
        if (halo > DWL_SMEM_BUDGET) continue;
        const int patches = bt * (bh / PH) * (bw / PW);
        const double warp_eff = (double)patches / (double)(((patches + nw - 1) / nw) * nw);
        const double cov_w = (double)d->Wo / (((d->Wo + bw - 1) / bw) * bw);
        const double cov_h = (double)d->Ho / (((d->Ho + bh - 1) / bh) * bh);
        const double cov_t = (double)d->To / (((d->To + bt - 1) / bt) * bt);
        const double reuse = (double)(bt * bh * bw) / (double)(tt * hh * ww);
        // compute efficiency dominates (FMA-bound); halo reuse breaks ties towards less L2 traffic
        const double score = warp_eff * cov_w * cov_h * cov_t * (0.75 + 0.25 * reuse) * (patches >= 2 * nw ? 1.0 : 0.9);
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
  const size_t smem = (size_t)P.tt * P.hh * P.ww * P.cc * 2 + 256;
  dim3 grid((unsigned)tiles, (unsigned)chunks), block(DWL_WARPS * 32);
#define PV_DWL2(S_, PH_, PW_, PRE_)                                                                            \
  do {                                                                                                        \
    PV_OPT_IN_SMEM((dwconv3d_lane_kernel<S_, PH_, PW_, PRE_>), 110 * 1024);                                   \
    dwconv3d_lane_kernel<S_, PH_, PW_, PRE_><<<grid, block, smem, stream>>>(P, (const __half*)w, scale, bias, \
                                                                           (__half*)y, se_sums);             \
    PV_LAUNCH_OK(PV_PRE_NAME("dwconv3d_lane_kernel<" #S_ "," #PH_ "," #PW_, PRE_));                           \
  } while (0)
#define PV_DWL(S_, PH_, PW_)                                                                                  \
  do {                                                                                                        \
    if (pre) PV_DWL2(S_, PH_, PW_, true); else PV_DWL2(S_, PH_, PW_, false);                                  \
  } while (0)
  if (S == 1 && !p27) PV_DWL(1, 4, 4);
  else if (S == 1) PV_DWL(1, 2, 7);
  else if (!p27) PV_DWL(2, 4, 4);
  else PV_DWL(2, 2, 7);
#undef PV_DWL
#undef PV_DWL2
  return PV_OK;
}

}  // namespace pv

// CUDA-core kernels: layout conversion, tiled direct convolution (dense), depthwise stencils,
// pooling, squeeze-excitation, head reduction, LayerNorm.  All are HBM-bound or serve shapes the
// tensor-core implicit-GEMM path does not take (3-channel stems, fp32 "parity" storage).
#include "pv_common.cuh"

namespace pv {

// =============================================================================================
// NCDHW <-> NDHWC
// =============================================================================================
template <typename SrcT, typename DstT>
__global__ void ncdhw_to_ndhwc_kernel(const SrcT* __restrict__ src, DstT* __restrict__ dst, int C,
                                      long long thw, int c_pad, long long dst_row_stride,
                                      long long total_pos) {
  long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total_pos) return;
  long long n = p / thw, r = p - n * thw;
  const SrcT* s = src + n * C * thw + r;
  DstT* o = dst + p * dst_row_stride;
  for (int c = 0; c < c_pad; ++c) {
    float v = (c < C) ? Elem<SrcT>::ld(s + (long long)c * thw) : 0.f;
    Elem<DstT>::st(o + c, v);
  }
}

// NCDHW -> NDHWC with physical zero padding along W (stem layout for the windowed-TMA conv)
template <typename SrcT, typename DstT>
__global__ void ncdhw_to_ndhwc_padw_kernel(const SrcT* __restrict__ src, DstT* __restrict__ dst, int C,
                                           int T, int H, int W, int c_pad, int w_pad, int w_phys,
                                           long long total_phys) {
  long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // physical pixel index
  if (p >= total_phys) return;
  const int wp = (int)(p % w_phys);
  long long r = p / w_phys;            // (n*T + t)*H + h
  const int w = wp - w_pad;
  DstT* o = dst + p * c_pad;
  if (w < 0 || w >= W) {
    for (int c = 0; c < c_pad; ++c) Elem<DstT>::st(o + c, 0.f);
    return;
  }
  const int h = (int)(r % H); r /= H;
  const int t = (int)(r % T); const long long n = r / T;
  const long long thw = (long long)T * H * W;
  const SrcT* s = src + n * C * thw + ((long long)t * H + h) * W + w;
  for (int c = 0; c < c_pad; ++c) {
    float v = (c < C) ? Elem<SrcT>::ld(s + (long long)c * thw) : 0.f;
    Elem<DstT>::st(o + c, v);
  }
}

// f32 NCDHW -> f16 NDHWC4 with W padding, 4 consecutive pixels per thread (16-byte reads per channel
// plane, one 32-byte write).  Requires W % 4 == 0, w_pad % 4 == 0, w_phys % 4 == 0, C <= 4, c_pad == 4.
__global__ void __launch_bounds__(256)
ncdhw_f32_to_ndhwc4_padw_kernel(const float* __restrict__ src, __half* __restrict__ dst, int C, int T, int H,
                                int W, int w_pad, int w_phys, long long total_quads) {
  long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // quad of 4 physical pixels
  if (q >= total_quads) return;
  const int qpr = w_phys >> 2;
  const int wq = (int)(q % qpr);
  long long r = q / qpr;                 // (n*T + t)*H + h
  const int w = wq * 4 - w_pad;
  uint4 o0 = make_uint4(0u, 0u, 0u, 0u), o1 = make_uint4(0u, 0u, 0u, 0u);
  if (w >= 0 && w < W) {
    const int h = (int)(r % H); long long r2 = r / H;
    const int t = (int)(r2 % T); const long long n = r2 / T;
    const long long thw = (long long)T * H * W;
    const float* s = src + n * C * thw + ((long long)t * H + h) * W + w;
    float4 c0 = *reinterpret_cast<const float4*>(s);
    float4 c1 = C > 1 ? *reinterpret_cast<const float4*>(s + thw) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 c2 = C > 2 ? *reinterpret_cast<const float4*>(s + 2 * thw) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 c3 = C > 3 ? *reinterpret_cast<const float4*>(s + 3 * thw) : make_float4(0.f, 0.f, 0.f, 0.f);
    __half2* p0 = reinterpret_cast<__half2*>(&o0);
    __half2* p1 = reinterpret_cast<__half2*>(&o1);
    p0[0] = __floats2half2_rn(c0.x, c1.x); p0[1] = __floats2half2_rn(c2.x, c3.x);
    p0[2] = __floats2half2_rn(c0.y, c1.y); p0[3] = __floats2half2_rn(c2.y, c3.y);
    p1[0] = __floats2half2_rn(c0.z, c1.z); p1[1] = __floats2half2_rn(c2.z, c3.z);
    p1[2] = __floats2half2_rn(c0.w, c1.w); p1[3] = __floats2half2_rn(c2.w, c3.w);
  }
  uint4* o = reinterpret_cast<uint4*>(dst + q * 16);
  o[0] = o0;
  o[1] = o1;
}

template <typename SrcT>
__global__ void ndhwc_to_ncdhw_kernel(const SrcT* __restrict__ src, long long src_row_stride,
                                      float* __restrict__ dst, int C, long long thw,
                                      long long total) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // over N*C*thw (dst order)
  if (i >= total) return;
  long long r = i % thw;
  long long nc = i / thw;
  int c = (int)(nc % C);
  long long n = nc / C;
  dst[i] = Elem<SrcT>::ld(src + (n * thw + r) * src_row_stride + c);
}

// =============================================================================================
// Dense direct convolution, tiled 64 positions x 64 output channels per CTA, K = (tap, ci)
// flattened and consumed in chunks of 16.  fp32 accumulation regardless of storage type.
// Requires Ci % 4 == 0, Co % 4 == 0.
// =============================================================================================
constexpr int DC_BM = 64, DC_BN = 64, DC_BK = 16;

template <typename T>
__global__ void __launch_bounds__(256)
conv3d_direct_kernel(pv_conv3d_desc d, const T* __restrict__ x, const T* __restrict__ w,
                     const float* __restrict__ scale, const float* __restrict__ bias,
                     const T* __restrict__ res, T* __restrict__ y, long long M) {
  __shared__ float As[DC_BK][DC_BM + 4];
  __shared__ float Bs[DC_BK][DC_BN + 4];
  __shared__ int pos_n[DC_BM], pos_t[DC_BM], pos_h[DC_BM], pos_w[DC_BM];

  const int tid = threadIdx.x;
  const long long m0 = (long long)blockIdx.x * DC_BM;
  const int n0 = blockIdx.y * DC_BN;

  if (tid < DC_BM) {
    long long m = m0 + tid;
    if (m < M) {
      int wo = (int)(m % d.Wo); long long r = m / d.Wo;
      int ho = (int)(r % d.Ho); r /= d.Ho;
      int to = (int)(r % d.To); int n = (int)(r / d.To);
      pos_n[tid] = n; pos_t[tid] = to * d.st - d.pt; pos_h[tid] = ho * d.sh - d.ph;
      pos_w[tid] = wo * d.sw - d.pw;
    } else {
      pos_n[tid] = -1; pos_t[tid] = 0; pos_h[tid] = 0; pos_w[tid] = 0;
    }
  }
  __syncthreads();

  const int K = d.kt * d.kh * d.kw * d.Ci;
  // A loader: thread -> (position a_m, 4 consecutive k starting at a_k)
  const int a_m = tid >> 2, a_k = (tid & 3) * 4;
  // B loader: thread -> (k row b_k, 4 consecutive co starting at b_n)
  const int b_k = tid >> 4, b_n = (tid & 15) * 4;
  const int tm = (tid >> 4) * 4, tn = (tid & 15) * 4;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int an = pos_n[a_m], at = pos_t[a_m], ah = pos_h[a_m], aw = pos_w[a_m];

  for (int k0 = 0; k0 < K; k0 += DC_BK) {
    // ---- A tile
    {
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      int k = k0 + a_k;
      if (an >= 0 && k < K) {
        int tap = k / d.Ci, ci = k - tap * d.Ci;
        int kw_ = tap % d.kw; int r = tap / d.kw; int kh_ = r % d.kh; int kt_ = r / d.kh;
        int ti = at + kt_ * d.dt, hi = ah + kh_ * d.dh, wi = aw + kw_ * d.dw;
        if ((unsigned)ti < (unsigned)d.Ti && (unsigned)hi < (unsigned)d.Hi &&
            (unsigned)wi < (unsigned)d.Wi) {
          const T* p = x + ((((long long)an * d.Ti + ti) * d.Hi + hi) * d.Wi + wi) * d.x_row_stride + ci;
          ld4<T>(p, v);
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) As[a_k + i][a_m] = v[i];
    }
    // ---- B tile
    {
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      int k = k0 + b_k, co = n0 + b_n;
      if (k < K && co < d.Co) ld4<T>(w + (long long)k * d.Co + co, v);
#pragma unroll
      for (int i = 0; i < 4; ++i) Bs[b_k][b_n + i] = v[i];
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < DC_BK; ++kk) {
      float a[4], b[4];
      *reinterpret_cast<float4*>(a) = *reinterpret_cast<const float4*>(&As[kk][tm]);
      *reinterpret_cast<float4*>(b) = *reinterpret_cast<const float4*>(&Bs[kk][tn]);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

  const int co = n0 + tn;
  if (co >= d.Co) return;
  float sc[4], bi[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) { sc[j] = __ldg(scale + co + j); bi[j] = __ldg(bias + co + j); }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    long long m = m0 + tm + i;
    if (m >= M) continue;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = acc[i][j] * sc[j] + bi[j];
    if (d.has_residual) {
      float r[4];
      ld4<T>(res + m * d.res_row_stride + co, r);
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] += r[j];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = apply_act(v[j], d.act);
    if (d.addend) {     // post-activation addend of output sample n, frame t (constant over h, w)
      const long long nt = m / ((long long)d.Ho * d.Wo);
      const long long n = nt / d.To, t = nt - n * d.To;
      float a[4];
      ld4<T>(static_cast<const T*>(d.addend) + n * d.add_n_stride + t * d.add_t_stride + d.add_ch_off + co, a);
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] += a[j];
    }
    st4<T>(y + m * d.y_row_stride + co, v);
  }
}

// =============================================================================================
// Depthwise convolution stencil (groups == C).  One thread = one output position x 8 channels;
// consecutive lanes walk the channel groups of a position, then the next position, so every
// warp-level load is a run of consecutive 16-byte vectors (coalesced in NDHWC).
// =============================================================================================
// PRE: pv_conv3d_desc's pre-activation prologue on every in-bounds input value as it is loaded (kept in fp32).
template <typename T, bool PRE>
__global__ void __launch_bounds__(256)
dwconv3d_kernel(pv_conv3d_desc d, const T* __restrict__ x, const T* __restrict__ w,
                const float* __restrict__ scale, const float* __restrict__ bias,
                const T* __restrict__ res, T* __restrict__ y, long long total) {
  long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int G = d.Co >> 3;
  const int cg = (int)(e % G);
  long long m = e / G;
  const int c = cg * 8;
  int wo = (int)(m % d.Wo); long long r = m / d.Wo;
  int ho = (int)(r % d.Ho); r /= d.Ho;
  int to = (int)(r % d.To); int n = (int)(r / d.To);
  const int t0 = to * d.st - d.pt, h0 = ho * d.sh - d.ph, w0 = wo * d.sw - d.pw;
  const long long xbs = d.x_batch_stride ? d.x_batch_stride : (long long)d.Ti * d.Hi * d.Wi * d.x_row_stride;
  const long long ybs = d.y_batch_stride ? d.y_batch_stride : (long long)d.To * d.Ho * d.Wo * d.y_row_stride;
  const long long mo = (((long long)to) * d.Ho + ho) * d.Wo + wo;   // position inside the sample

  float acc[8], ps[8], pb[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    acc[i] = 0.f;
    ps[i] = PRE ? __ldg(d.pre_scale + c + i) : 1.f;
    pb[i] = PRE ? __ldg(d.pre_bias + c + i) : 0.f;
  }

  for (int kt_ = 0; kt_ < d.kt; ++kt_) {
    const int ti = t0 + kt_ * d.dt;
    if ((unsigned)ti >= (unsigned)d.Ti) continue;
    for (int kh_ = 0; kh_ < d.kh; ++kh_) {
      const int hi = h0 + kh_ * d.dh;
      if ((unsigned)hi >= (unsigned)d.Hi) continue;
      const T* row = x + (long long)n * xbs + (((long long)ti) * d.Hi + hi) * d.Wi * d.x_row_stride + c;
      const T* wrow = w + (long long)((kt_ * d.kh + kh_) * d.kw) * d.Co + c;
      for (int kw_ = 0; kw_ < d.kw; ++kw_) {
        const int wi = w0 + kw_ * d.dw;
        if ((unsigned)wi >= (unsigned)d.Wi) continue;
        float xv[8], wv[8];
        ld8<T>(row + (long long)wi * d.x_row_stride, xv);
        ld8<T>(wrow + (long long)kw_ * d.Co, wv);
        if constexpr (PRE) {
#pragma unroll
          for (int i = 0; i < 8; ++i) xv[i] = pre_u(xv[i], ps[i], pb[i], d.pre_act);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(xv[i], wv[i], acc[i]);
      }
    }
  }
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = acc[i] * __ldg(scale + c + i) + __ldg(bias + c + i);
  if (d.has_residual) {
    float rr[8];
    ld8<T>(res + m * d.res_row_stride + c, rr);
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] += rr[i];
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = apply_act(v[i], d.act);
  st8<T>(y + (long long)n * ybs + mo * d.y_row_stride + c, v);
}

// Register-tiled depthwise stencil: one thread = 4 consecutive output columns x 8 channels.  For each
// (kt,kh) filter row the KW weight vectors are converted once and every input column is loaded and
// converted once and used by all outputs it feeds - 2.7x fewer loads and half the instructions of the
// one-output-per-thread kernel for the 3x3x3 / stride-1 case (X3D, CSN, MViT pooling).
// PRE: the pre-activation prologue on every in-bounds input column as it is loaded (once per column and filter row,
// kept in fp32).
template <typename T, int KW, int SW, bool PRE>
__global__ void __launch_bounds__(128)
dwconv3d_w4_kernel(pv_conv3d_desc d, const T* __restrict__ x, const T* __restrict__ w,
                   const float* __restrict__ scale, const float* __restrict__ bias, T* __restrict__ y,
                   long long total, int wo4) {
  constexpr int WT = 4;
  constexpr int NCOL = (WT - 1) * SW + KW;
  long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int G = d.Co >> 3;
  const int c = (int)(e % G) * 8;
  long long m = e / G;
  const int wq = (int)(m % wo4); long long r = m / wo4;
  const int ho = (int)(r % d.Ho); r /= d.Ho;
  const int to = (int)(r % d.To); const int n = (int)(r / d.To);
  const int wo0 = wq * WT;
  const int t0 = to * d.st - d.pt, h0 = ho * d.sh - d.ph, w0 = wo0 * SW - d.pw;
  const long long xbs = d.x_batch_stride ? d.x_batch_stride : (long long)d.Ti * d.Hi * d.Wi * d.x_row_stride;
  const long long ybs = d.y_batch_stride ? d.y_batch_stride : (long long)d.To * d.Ho * d.Wo * d.y_row_stride;
  float acc[WT][8], ps[8], pb[8];
#pragma unroll
  for (int o = 0; o < WT; ++o)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[o][i] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    ps[i] = PRE ? __ldg(d.pre_scale + c + i) : 1.f;
    pb[i] = PRE ? __ldg(d.pre_bias + c + i) : 0.f;
  }
  for (int kt_ = 0; kt_ < d.kt; ++kt_) {
    const int ti = t0 + kt_ * d.dt;
    if ((unsigned)ti >= (unsigned)d.Ti) continue;
    for (int kh_ = 0; kh_ < d.kh; ++kh_) {
      const int hi = h0 + kh_ * d.dh;
      if ((unsigned)hi >= (unsigned)d.Hi) continue;
      const T* row = x + (long long)n * xbs + (((long long)ti) * d.Hi + hi) * d.Wi * d.x_row_stride + c;
      const T* wrow = w + (long long)((kt_ * d.kh + kh_) * KW) * d.Co + c;
      float wv[KW][8];
#pragma unroll
      for (int k = 0; k < KW; ++k) ld8<T>(wrow + (long long)k * d.Co, wv[k]);
#pragma unroll
      for (int j = 0; j < NCOL; ++j) {
        const int wi = w0 + j;
        if ((unsigned)wi >= (unsigned)d.Wi) continue;
        float xv[8];
        ld8<T>(row + (long long)wi * d.x_row_stride, xv);
        if constexpr (PRE) {
#pragma unroll
          for (int i = 0; i < 8; ++i) xv[i] = pre_u(xv[i], ps[i], pb[i], d.pre_act);
        }
#pragma unroll
        for (int o = 0; o < WT; ++o) {
          const int k = j - o * SW;          // tap index this column has for output o (compile-time)
          if (k >= 0 && k < KW) {
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[o][i] = fmaf(xv[i], wv[k][i], acc[o][i]);
          }
        }
      }
    }
  }
  float sc[8], bi[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { sc[i] = __ldg(scale + c + i); bi[i] = __ldg(bias + c + i); }
#pragma unroll
  for (int o = 0; o < WT; ++o) {
    if (wo0 + o >= d.Wo) break;
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = apply_act(acc[o][i] * sc[i] + bi[i], d.act);
    st8<T>(y + (long long)n * ybs + ((((long long)to) * d.Ho + ho) * d.Wo + wo0 + o) * d.y_row_stride + c, v);
  }
}

// =============================================================================================
// Pooling (max / avg), NDHWC, one thread = one output position x 8 channels.
// =============================================================================================
template <typename T>
__global__ void __launch_bounds__(256)
pool3d_kernel(pv_pool3d_desc d, const T* __restrict__ x, T* __restrict__ y, long long total) {
  long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int G = d.C >> 3;
  const int c = (int)(e % G) * 8;
  long long m = e / G;
  int wo = (int)(m % d.Wo); long long r = m / d.Wo;
  int ho = (int)(r % d.Ho); r /= d.Ho;
  int to = (int)(r % d.To); int n = (int)(r / d.To);
  const int t0 = to * d.st - d.pt, h0 = ho * d.sh - d.ph, w0 = wo * d.sw - d.pw;
  const bool is_max = d.mode == PV_POOL_MAX;
  const long long xbs = d.x_batch_stride ? d.x_batch_stride : (long long)d.Ti * d.Hi * d.Wi * d.x_row_stride;
  const long long ybs = d.y_batch_stride ? d.y_batch_stride : (long long)d.To * d.Ho * d.Wo * d.y_row_stride;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = is_max ? -INFINITY : 0.f;
  for (int kt_ = 0; kt_ < d.kt; ++kt_) {
    const int ti = t0 + kt_;
    if ((unsigned)ti >= (unsigned)d.Ti) continue;
    for (int kh_ = 0; kh_ < d.kh; ++kh_) {
      const int hi = h0 + kh_;
      if ((unsigned)hi >= (unsigned)d.Hi) continue;
      const T* row = x + (long long)n * xbs + (((long long)ti) * d.Hi + hi) * d.Wi * d.x_row_stride + c;
      for (int kw_ = 0; kw_ < d.kw; ++kw_) {
        const int wi = w0 + kw_;
        if ((unsigned)wi >= (unsigned)d.Wi) continue;
        float v[8];
        ld8<T>(row + (long long)wi * d.x_row_stride, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = is_max ? fmaxf(acc[i], v[i]) : acc[i] + v[i];
      }
    }
  }
  if (!is_max) {
    const float inv = 1.f / (float)(d.kt * d.kh * d.kw);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] *= inv;
  }
  st8<T>(y + (long long)n * ybs + ((((long long)to) * d.Ho + ho) * d.Wo + wo) * d.y_row_stride + c, acc);
}

// Global pooling (kernel == whole T x H x W extent, the head pools): one CTA per (sample, 64-channel
// slab); 8 channel-group lanes x 32 position lanes, 128-byte coalesced reads, smem tree reduce.
template <typename T>
__global__ void __launch_bounds__(256)
global_pool_kernel(const T* __restrict__ x, T* __restrict__ y, long long x_row_stride,
                   long long y_row_stride, long long npos, int C, int is_max) {
  __shared__ float red[32][64 + 1];
  const int n = blockIdx.y;
  const int c0 = blockIdx.x * 64;
  const int cg = threadIdx.x & 7, pl = threadIdx.x >> 3;
  const int c = c0 + cg * 8;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = is_max ? -INFINITY : 0.f;
  if (c < C) {
    for (long long p = pl; p < npos; p += 32) {
      float v[8];
      ld8<T>(x + ((long long)n * npos + p) * x_row_stride + c, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = is_max ? fmaxf(acc[i], v[i]) : acc[i] + v[i];
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) red[pl][cg * 8 + i] = acc[i];
  __syncthreads();
  if (threadIdx.x < 64) {
    float r = red[0][threadIdx.x];
    for (int j = 1; j < 32; ++j) r = is_max ? fmaxf(r, red[j][threadIdx.x]) : r + red[j][threadIdx.x];
    if (!is_max) r *= 1.f / (float)npos;
    if (c0 + (int)threadIdx.x < C) Elem<T>::st(y + (long long)n * y_row_stride + c0 + threadIdx.x, r);
  }
}

// =============================================================================================
// Squeeze-Excitation helpers
// =============================================================================================
// grid = (chunks, N); each CTA reduces `chunk` positions of one sample for all channels and
// adds its partial sums with one atomic per channel (64-bit fixed point, se_sum_add: order-independent).
template <typename T>
__global__ void __launch_bounds__(256)
channel_sum_kernel(const T* __restrict__ x, long long row_stride, long long npos, int C,
                   long long chunk, float* __restrict__ sums) {
  extern __shared__ unsigned long long sh_fix[];   // [C], fixed point
  const int n = blockIdx.y;
  for (int c = threadIdx.x; c < C; c += blockDim.x) sh_fix[c] = 0ull;
  __syncthreads();
  const int G = C >> 3;
  const long long p0 = (long long)blockIdx.x * chunk;
  const long long p1 = min(p0 + chunk, npos);
  const int lanes_per_pos = G;
  const int pos_per_iter = blockDim.x / lanes_per_pos;
  if (pos_per_iter > 0) {
    const int cg = threadIdx.x % lanes_per_pos, pl = threadIdx.x / lanes_per_pos;
    if (pl < pos_per_iter) {
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
      for (long long p = p0 + pl; p < p1; p += pos_per_iter) {
        float v[8];
        ld8<T>(x + ((long long)n * npos + p) * row_stride + cg * 8, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += v[i];
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) atomicAdd(&sh_fix[cg * 8 + i], (unsigned long long)se_fix(acc[i]));
    }
  } else {   // more channel groups than threads
    for (int cg = threadIdx.x; cg < G; cg += blockDim.x) {
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
      for (long long p = p0; p < p1; ++p) {
        float v[8];
        ld8<T>(x + ((long long)n * npos + p) * row_stride + cg * 8, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += v[i];
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) sh_fix[cg * 8 + i] = (unsigned long long)se_fix(acc[i]);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) atomicAdd(reinterpret_cast<unsigned long long*>(sums) + (long long)n * C + c, sh_fix[c]);
}

// one CTA per sample; Cr <= 256
__global__ void se_gate_kernel(const float* __restrict__ sums, float inv_npos, int C, int Cr,
                               const float* __restrict__ w1, const float* __restrict__ b1,
                               const float* __restrict__ w2, const float* __restrict__ b2,
                               int c_stride_w, float* __restrict__ gate) {
  extern __shared__ float sh[];   // mean[C] + hidden[Cr]
  float* mean = sh;
  float* hid = sh + C;
  const int n = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) mean[c] = se_sum_get(sums, (long long)n * C + c) * inv_npos;
  __syncthreads();
  for (int j = threadIdx.x; j < Cr; j += blockDim.x) {
    float a = b1[j];
    for (int c = 0; c < C; ++c) a = fmaf(w1[(long long)j * c_stride_w + c], mean[c], a);
    hid[j] = fmaxf(a, 0.f);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = b2[c];
    for (int j = 0; j < Cr; ++j) a = fmaf(w2[(long long)c * Cr + j], hid[j], a);
    gate[(long long)n * C + c] = 1.f / (1.f + __expf(-a));
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
scale_act_kernel(const T* __restrict__ x, T* __restrict__ y, long long x_row_stride,
                 long long y_row_stride, long long npos, int C, const float* __restrict__ gate,
                 int act, long long total) {
  long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int G = C >> 3;
  int c;
  long long m, n;
  if (total < 0x7fffffffll) {        // 32-bit index math (64-bit divides cost more than the memory traffic here)
    const unsigned eu = (unsigned)e, mu = eu / (unsigned)G;
    c = (int)(eu - mu * (unsigned)G) * 8;
    m = mu;
    n = mu / (unsigned)npos;
  } else {
    c = (int)(e % G) * 8;
    m = e / G;
    n = m / npos;
  }
  float v[8];
  ld8<T>(x + m * x_row_stride + c, v);
  if (gate) {
    const float* gp = gate + n * C + c;     // C % 8 == 0 and cudaMalloc alignment: 32-byte aligned
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gp)), g1 = __ldg(reinterpret_cast<const float4*>(gp + 4));
    v[0] *= g0.x; v[1] *= g0.y; v[2] *= g0.z; v[3] *= g0.w; v[4] *= g1.x; v[5] *= g1.y; v[6] *= g1.z; v[7] *= g1.w;
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = apply_act(v[i], act);
  st8<T>(y + m * y_row_stride + c, v);
}

// =============================================================================================
// Head tail: optional per-position softmax over channels, then mean over positions -> f32.
// one CTA per sample, blockDim = 256.
// =============================================================================================
template <typename T>
__global__ void head_reduce_kernel(const T* __restrict__ x, long long row_stride, long long npos,
                                   int C, int softmax, float* __restrict__ out) {
  extern __shared__ float sh[];   // acc[C] + red[32]
  float* acc = sh;
  float* red = sh + C;
  const int n = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) acc[c] = 0.f;
  __syncthreads();
  for (long long p = 0; p < npos; ++p) {
    const T* row = x + ((long long)n * npos + p) * row_stride;
    if (!softmax) {
      for (int c = threadIdx.x; c < C; c += blockDim.x) acc[c] += Elem<T>::ld(row + c);
    } else {
      float mx = -INFINITY;
      for (int c = threadIdx.x; c < C; c += blockDim.x) mx = fmaxf(mx, Elem<T>::ld(row + c));
      for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
      __syncthreads();
      mx = red[0];
      for (int i = 1; i < (int)(blockDim.x >> 5); ++i) mx = fmaxf(mx, red[i]);
      __syncthreads();
      float sm = 0.f;
      for (int c = threadIdx.x; c < C; c += blockDim.x) sm += expf(Elem<T>::ld(row + c) - mx);
      for (int o = 16; o; o >>= 1) sm += __shfl_xor_sync(0xffffffffu, sm, o);
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sm;
      __syncthreads();
      sm = 0.f;
      for (int i = 0; i < (int)(blockDim.x >> 5); ++i) sm += red[i];
      __syncthreads();
      const float inv = 1.f / sm;
      for (int c = threadIdx.x; c < C; c += blockDim.x)
        acc[c] += expf(Elem<T>::ld(row + c) - mx) * inv;
    }
  }
  __syncthreads();
  const float inv = 1.f / (float)npos;
  for (int c = threadIdx.x; c < C; c += blockDim.x) out[(long long)n * C + c] = acc[c] * inv;
}

// =============================================================================================
// LayerNorm over the last dim, one warp per row, fp32 statistics (two-pass, like ATen).
// =============================================================================================
// Extras of pv_layernorm_sets: several (gamma, beta) sets (group g uses set g / groups_per_set - the pooled K and V
// of one MViT block are normalised by ONE launch with norm_k | norm_v) and rows whose input comes from another tensor
// (every npos-th row = the cls token that by-passes the pooling conv, layers/attention.py:184-205: no copy launch).
struct LnExtra {
  int groups_per_set;
  const void* cls_src;
  long long cls_batch_stride, npos;
};
template <typename T>
__global__ void __launch_bounds__(256)
layernorm_kernel(const T* __restrict__ x, T* __restrict__ y, long long rows, int groups, int C,
                 long long x_row_stride, long long y_row_stride, const float* __restrict__ gamma,
                 const float* __restrict__ beta, float eps, LnExtra X) {
  const long long rg = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);   // (row, group)
  if (rg >= rows * groups) return;
  const long long row = rg / groups;
  const int grp = (int)(rg - row * groups);
  const int lane = threadIdx.x & 31;
  const T* xr = x + row * x_row_stride + (long long)grp * C;
  if (X.cls_src != nullptr && row % X.npos == 0)
    xr = reinterpret_cast<const T*>(X.cls_src) + (row / X.npos) * X.cls_batch_stride + (long long)grp * C;
  gamma += (grp / X.groups_per_set) * C;
  beta += (grp / X.groups_per_set) * C;
  float s = 0.f;
  for (int c = lane * 8; c < C; c += 256) {
    float v[8];
    ld8<T>(xr + c, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) s += v[i];
  }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  float q = 0.f;
  for (int c = lane * 8; c < C; c += 256) {
    float v[8];
    ld8<T>(xr + c, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) { float dlt = v[i] - mean; q = fmaf(dlt, dlt, q); }
  }
  for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)C + eps);
  T* yr = y + row * y_row_stride + (long long)grp * C;
  for (int c = lane * 8; c < C; c += 256) {
    float v[8];
    ld8<T>(xr + c, v);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      v[i] = (v[i] - mean) * rstd * __ldg(gamma + c + i) + __ldg(beta + c + i);
    st8<T>(yr + c, v);
  }
}

// Row-in-registers LayerNorm for C <= 768: a row is read ONCE (8 channels per 16-byte load, up to NCH
// loads per lane), `lpr` lanes cooperate on a row (power of two >= ceil(C/8), so a 96-wide MViT row
// uses 16 lanes and a warp normalises two rows), mean and centred variance are reduced with sub-warp
// shuffles.  (The generic kernel below re-reads the row three times and keeps 12 of 32 lanes busy at C=96.)
template <typename T, int NCH>
__global__ void __launch_bounds__(256)
layernorm_reg_kernel(const T* __restrict__ x, T* __restrict__ y, long long rows, int groups, int C,
                     long long x_row_stride, long long y_row_stride, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float eps, int lpr_log2, LnExtra X) {
  const int lane = threadIdx.x & 31;
  const int lpr = 1 << lpr_log2;
  const int sub = lane >> lpr_log2, sl = lane & (lpr - 1);
  const long long total = rows * groups;
  long long rg = (((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) << (5 - lpr_log2)) + sub;
  const bool ok = rg < total;
  if (!ok) rg = 0;
  const long long row = rg / groups;
  const int grp = (int)(rg - row * groups);
  const T* xr = x + row * x_row_stride + (long long)grp * C;
  if (X.cls_src != nullptr && row % X.npos == 0)
    xr = reinterpret_cast<const T*>(X.cls_src) + (row / X.npos) * X.cls_batch_stride + (long long)grp * C;
  gamma += (grp / X.groups_per_set) * C;
  beta += (grp / X.groups_per_set) * C;
  float v[NCH][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = (sl + i * lpr) * 8;
    if (ok && c < C) {
      ld8<T>(xr + c, v[i]);
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[i][e] = 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) s += v[i][e];
  }
  for (int o = lpr >> 1; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = (sl + i * lpr) * 8;
    if (c < C) {
#pragma unroll
      for (int e = 0; e < 8; ++e) { const float dlt = v[i][e] - mean; q = fmaf(dlt, dlt, q); }
    }
  }
  for (int o = lpr >> 1; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)C + eps);
  T* yr = y + row * y_row_stride + (long long)grp * C;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = (sl + i * lpr) * 8;
    if (ok && c < C) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c + 4));
      float o8[8];
      o8[0] = (v[i][0] - mean) * rstd * g0.x + b0.x; o8[1] = (v[i][1] - mean) * rstd * g0.y + b0.y;
      o8[2] = (v[i][2] - mean) * rstd * g0.z + b0.z; o8[3] = (v[i][3] - mean) * rstd * g0.w + b0.w;
      o8[4] = (v[i][4] - mean) * rstd * g1.x + b1.x; o8[5] = (v[i][5] - mean) * rstd * g1.y + b1.y;
      o8[6] = (v[i][6] - mean) * rstd * g1.z + b1.z; o8[7] = (v[i][7] - mean) * rstd * g1.w + b1.w;
      st8<T>(yr + c, o8);
    }
  }
}

// Residual add + LayerNorm on an fp32 trunk (MViT token stream, layers/attention.py:746-757: x = x_res + x_block;
// x_norm = norm2(x); ... x = x + x_mlp; next block's norm1).  s = a + b in fp32 (a: f16 | f32, b: f16 branch or none);
// s is stored as fp32 (the residual trunk never takes an f16 rounding), y = LN(s) is stored as f16 (the next GEMM's
// A operand).  Same row-in-registers scheme as layernorm_reg_kernel; sum / y may each be null.
template <typename TA, bool HAS_B, int NCH>
__global__ void __launch_bounds__(256)
add_layernorm_kernel(const TA* __restrict__ a, const __half* __restrict__ b, float* __restrict__ sum,
                     __half* __restrict__ y, long long rows, int C, long long a_rs, long long b_rs, long long s_rs,
                     long long y_rs, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                     int lpr_log2) {
  const int lane = threadIdx.x & 31;
  const int lpr = 1 << lpr_log2;
  const int sub = lane >> lpr_log2, sl = lane & (lpr - 1);
  long long row = (((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) << (5 - lpr_log2)) + sub;
  const bool ok = row < rows;
  if (!ok) row = 0;
  float v[NCH][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = (sl + i * lpr) * 8;
    if (ok && c < C) {
      ld8<TA>(a + row * a_rs + c, v[i]);
      if (HAS_B) {
        float w[8];
        ld8<__half>(b + row * b_rs + c, w);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[i][e] += w[e];
      }
      if (sum != nullptr) st8<float>(sum + row * s_rs + c, v[i]);
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[i][e] = 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) s += v[i][e];
  }
  if (y == nullptr) return;
  for (int o = lpr >> 1; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = (sl + i * lpr) * 8;
    if (c < C) {
#pragma unroll
      for (int e = 0; e < 8; ++e) { const float dlt = v[i][e] - mean; q = fmaf(dlt, dlt, q); }
    }
  }
  for (int o = lpr >> 1; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)C + eps);
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = (sl + i * lpr) * 8;
    if (ok && c < C) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c + 4));
      float o8[8];
      o8[0] = (v[i][0] - mean) * rstd * g0.x + b0.x; o8[1] = (v[i][1] - mean) * rstd * g0.y + b0.y;
      o8[2] = (v[i][2] - mean) * rstd * g0.z + b0.z; o8[3] = (v[i][3] - mean) * rstd * g0.w + b0.w;
      o8[4] = (v[i][4] - mean) * rstd * g1.x + b1.x; o8[5] = (v[i][5] - mean) * rstd * g1.y + b1.y;
      o8[6] = (v[i][6] - mean) * rstd * g1.z + b1.z; o8[7] = (v[i][7] - mean) * rstd * g1.w + b1.w;
      st8<__half>(y + row * y_rs + c, o8);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
temporal_tap_sum_kernel(const T* __restrict__ yk, T* __restrict__ y, int Ti, int To, long long hw, int Co, int kt,
                        int st, int pt, int dil, const float* __restrict__ scale, const float* __restrict__ bias,
                        int act, long long irs, long long ors, long long total) {
  long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int G = Co >> 3;
  const int c = (int)(e % G) * 8;
  long long r = e / G;                      // (n*To + t)*hw + p
  const long long p = r % hw; r /= hw;
  const int t = (int)(r % To); const long long n = r / To;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int dt = 0; dt < kt; ++dt) {
    const int ti = t * st + dt * dil - pt;
    if ((unsigned)ti >= (unsigned)Ti) continue;
    float v[8];
    ld8<T>(yk + ((n * Ti + ti) * hw + p) * irs + (long long)dt * Co + c, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] += v[i];
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = apply_act(acc[i] * __ldg(scale + c + i) + __ldg(bias + c + i), act);
  st8<T>(y + ((n * To + t) * hw + p) * ors + c, acc);
}

template <typename T>
__global__ void copy_rows_kernel(const T* __restrict__ src, T* __restrict__ dst, long long rows, int C,
                                 long long ss, long long ds) {
  long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int G = C >> 3;
  if (e >= rows * G) return;
  const long long r = e / G;
  const int c = (int)(e - r * G) * 8;
  float v[8];
  ld8<T>(src + r * ss + c, v);
  st8<T>(dst + r * ds + c, v);
}

template <typename T, typename TO>
__global__ void add_pos_cls_kernel(const T* __restrict__ x, TO* __restrict__ y, long long n_patch, int C,
                                   long long x_row_stride, const float* __restrict__ pos, int has_cls,
                                   long long total) {
  long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int G = C >> 3;
  const int c = (int)(e % G) * 8;
  long long r = e / G;                         // output row over B * (has_cls + n_patch)
  const long long nrow = n_patch + has_cls;
  const long long b = r / nrow, i = r - b * nrow;
  float v[8];
  if (has_cls && i == 0) {
#pragma unroll
    for (int q = 0; q < 8; ++q) v[q] = __ldg(pos + c + q);
  } else {
    ld8<T>(x + (b * n_patch + (i - has_cls)) * x_row_stride + c, v);
#pragma unroll
    for (int q = 0; q < 8; ++q) v[q] += __ldg(pos + i * C + c + q);
  }
  st8<TO>(y + r * C + c, v);
}

}  // namespace pv

// =============================================================================================
// C ABI
// =============================================================================================
using namespace pv;

extern "C" int pv_ncdhw_to_ndhwc(const void* src, int src_dtype, void* dst, int dst_dtype, int N,
                                 int C, int T, int H, int W, int c_pad,
                                 long long dst_row_stride, void* stream) {
  PV_CHECK_ARG(src && dst, "null pointer");
  PV_CHECK_ARG(c_pad >= C && dst_row_stride >= c_pad, "bad padding");
  const long long thw = (long long)T * H * W, total = (long long)N * thw;
  if (total == 0) return PV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid((unsigned)cdiv(total, 256)), block(256);
#define PV_CASE(ST, DT)                                                                          \
  ncdhw_to_ndhwc_kernel<ST, DT><<<grid, block, 0, s>>>((const ST*)src, (DT*)dst, C, thw, c_pad, \
                                                     dst_row_stride, total)
  if (src_dtype == PV_F32 && dst_dtype == PV_F16) PV_CASE(float, __half);
  else if (src_dtype == PV_F32 && dst_dtype == PV_F32) PV_CASE(float, float);
  else if (src_dtype == PV_F16 && dst_dtype == PV_F16) PV_CASE(__half, __half);
  else if (src_dtype == PV_F16 && dst_dtype == PV_F32) PV_CASE(__half, float);
  else { set_error("unsupported dtype pair %d->%d", src_dtype, dst_dtype); return PV_ERR_INVALID; }
#undef PV_CASE
  PV_LAUNCH_OK("ncdhw_to_ndhwc_kernel");
  return PV_OK;
}

extern "C" int pv_ncdhw_to_ndhwc_padw(const void* src, int src_dtype, void* dst, int dst_dtype, int N,
                                      int C, int T, int H, int W, int c_pad, int w_pad, int w_phys,
                                      void* stream) {
  PV_CHECK_ARG(src && dst, "null pointer");
  PV_CHECK_ARG(c_pad >= C && w_pad >= 0 && w_phys >= w_pad + W, "bad padding");
  const long long total = (long long)N * T * H * w_phys;
  if (total == 0) return PV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  if (src_dtype == PV_F32 && dst_dtype == PV_F16 && c_pad == 4 && C <= 4 && W % 4 == 0 && w_pad % 4 == 0 &&
      w_phys % 4 == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
    const long long quads = total / 4;
    ncdhw_f32_to_ndhwc4_padw_kernel<<<(unsigned)cdiv(quads, 256), 256, 0, s>>>((const float*)src, (__half*)dst, C, T, H,
                                                                              W, w_pad, w_phys, quads);
    PV_LAUNCH_OK("ncdhw_f32_to_ndhwc4_padw_kernel");
    return PV_OK;
  }
  dim3 grid((unsigned)cdiv(total, 256)), block(256);
#define PV_CASE(ST, DT)                                                                         \
  ncdhw_to_ndhwc_padw_kernel<ST, DT><<<grid, block, 0, s>>>((const ST*)src, (DT*)dst, C, T, H, W, c_pad, \
                                                          w_pad, w_phys, total)
  if (src_dtype == PV_F32 && dst_dtype == PV_F16) PV_CASE(float, __half);
  else if (src_dtype == PV_F32 && dst_dtype == PV_F32) PV_CASE(float, float);
  else if (src_dtype == PV_F16 && dst_dtype == PV_F16) PV_CASE(__half, __half);
  else if (src_dtype == PV_F16 && dst_dtype == PV_F32) PV_CASE(__half, float);
  else { set_error("unsupported dtype pair %d->%d", src_dtype, dst_dtype); return PV_ERR_INVALID; }
#undef PV_CASE
  PV_LAUNCH_OK("ncdhw_to_ndhwc_padw_kernel");
  return PV_OK;
}

extern "C" int pv_temporal_tap_sum(const void* yk, void* y, int dtype, int N, int Ti, int To, long long hw,
                                   int Co, int kt, int st, int pt, int dil, const float* scale,
                                   const float* bias, int act, long long in_row_stride,
                                   long long out_row_stride, void* stream) {
  PV_CHECK_ARG(yk && y && scale && bias, "null pointer");
  PV_CHECK_ARG(act_known(act), "activation code %d unsupported", act);
  PV_CHECK_ARG(Co % 8 == 0 && in_row_stride % 8 == 0 && out_row_stride % 8 == 0, "Co/strides %% 8");
  PV_CHECK_ARG(in_row_stride >= (long long)kt * Co && out_row_stride >= Co, "row stride too small");
  const long long total = (long long)N * To * hw * (Co / 8);
  if (total == 0) return PV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid((unsigned)cdiv(total, 256)), block(256);
  if (dtype == PV_F16)
    temporal_tap_sum_kernel<__half><<<grid, block, 0, s>>>((const __half*)yk, (__half*)y, Ti, To, hw, Co, kt, st, pt, dil,
                                                        scale, bias, act, in_row_stride, out_row_stride, total);
  else if (dtype == PV_F32)
    temporal_tap_sum_kernel<float><<<grid, block, 0, s>>>((const float*)yk, (float*)y, Ti, To, hw, Co, kt, st, pt, dil,
                                                       scale, bias, act, in_row_stride, out_row_stride, total);
  else { set_error("unsupported dtype %d", dtype); return PV_ERR_INVALID; }
  PV_LAUNCH_OK("temporal_tap_sum_kernel");
  return PV_OK;
}

extern "C" int pv_copy_rows(const void* src, void* dst, int dtype, long long rows, int C,
                            long long src_row_stride, long long dst_row_stride, void* stream) {
  PV_CHECK_ARG(src && dst, "null pointer");
  PV_CHECK_ARG(C % 8 == 0 && src_row_stride % 8 == 0 && dst_row_stride % 8 == 0, "C/strides %% 8");
  const long long total = rows * (C / 8);
  if (total == 0) return PV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid((unsigned)cdiv(total, 256)), block(256);
  if (dtype == PV_F16)
    copy_rows_kernel<__half><<<grid, block, 0, s>>>((const __half*)src, (__half*)dst, rows, C, src_row_stride, dst_row_stride);
  else if (dtype == PV_F32)
    copy_rows_kernel<float><<<grid, block, 0, s>>>((const float*)src, (float*)dst, rows, C, src_row_stride, dst_row_stride);
  else { set_error("unsupported dtype %d", dtype); return PV_ERR_INVALID; }
  PV_LAUNCH_OK("copy_rows_kernel");
  return PV_OK;
}

extern "C" int pv_add_pos_cls_to(const void* x, int x_dtype, void* y, int y_dtype, int B, long long n_patch, int C,
                                 long long x_row_stride, const float* pos, int has_cls, void* stream) {
  PV_CHECK_ARG(x && y && pos, "null pointer");
  PV_CHECK_ARG(C % 8 == 0 && x_row_stride % 8 == 0, "C/strides %% 8");
  const long long total = (long long)B * (n_patch + (has_cls ? 1 : 0)) * (C / 8);
  if (total == 0) return PV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid((unsigned)cdiv(total, 256)), block(256);
  const int hc = has_cls ? 1 : 0;
  if (x_dtype == PV_F16 && y_dtype == PV_F16)
    add_pos_cls_kernel<__half, __half><<<grid, block, 0, s>>>((const __half*)x, (__half*)y, n_patch, C, x_row_stride, pos, hc, total);
  else if (x_dtype == PV_F16 && y_dtype == PV_F32)
    add_pos_cls_kernel<__half, float><<<grid, block, 0, s>>>((const __half*)x, (float*)y, n_patch, C, x_row_stride, pos, hc, total);
  else if (x_dtype == PV_F32 && y_dtype == PV_F32)
    add_pos_cls_kernel<float, float><<<grid, block, 0, s>>>((const float*)x, (float*)y, n_patch, C, x_row_stride, pos, hc, total);
  else { set_error("unsupported dtypes %d -> %d", x_dtype, y_dtype); return PV_ERR_INVALID; }
  PV_LAUNCH_OK("add_pos_cls_kernel");
  return PV_OK;
}

extern "C" int pv_add_pos_cls(const void* x, void* y, int dtype, int B, long long n_patch, int C,
                              long long x_row_stride, const float* pos, int has_cls, void* stream) {
  return pv_add_pos_cls_to(x, dtype, y, dtype, B, n_patch, C, x_row_stride, pos, has_cls, stream);
}

extern "C" int pv_add_layernorm(const void* a, int a_dtype, long long a_row_stride, const void* b,
                                long long b_row_stride, float* sum, long long sum_row_stride, void* y,
                                long long y_row_stride, long long rows, int C, const float* gamma,
                                const float* beta, float eps, void* stream) {
  PV_CHECK_ARG(a && (sum || y), "null pointer");
  PV_CHECK_ARG(!y || (gamma && beta), "LayerNorm output without gamma / beta");
  PV_CHECK_ARG(a_dtype == PV_F16 || a_dtype == PV_F32, "a must be f16 or f32");
  PV_CHECK_ARG(C % 8 == 0 && a_row_stride % 8 == 0 && b_row_stride % 8 == 0 && sum_row_stride % 8 == 0 &&
               y_row_stride % 8 == 0, "C/strides %% 8");
  PV_CHECK_ARG(a_row_stride >= C && (!b || b_row_stride >= C) && (!sum || sum_row_stride >= C) &&
               (!y || y_row_stride >= C), "row stride < C");
  PV_CHECK_ARG(!y || ((((uintptr_t)gamma | (uintptr_t)beta) & 15) == 0), "gamma / beta must be 16-byte aligned");
  if (rows == 0) return PV_OK;
  const int chunks = C / 8;
  int lpr_log2 = 2;
  while ((1 << lpr_log2) < chunks && lpr_log2 < 5) ++lpr_log2;
  const int nch = (chunks + (1 << lpr_log2) - 1) >> lpr_log2;
  if (nch > 3) { set_error("pv_add_layernorm: C = %d > 768 unsupported", C); return PV_ERR_UNSUPPORTED; }
  cudaStream_t s = (cudaStream_t)stream;
  const long long per_block = 8ll << (5 - lpr_log2);
  dim3 grid((unsigned)cdiv(rows, per_block)), block(256);
#define PV_ALN(TA, HB, N_) add_layernorm_kernel<TA, HB, N_><<<grid, block, 0, s>>>((const TA*)a, (const __half*)b, sum, (__half*)y, \
    rows, C, a_row_stride, b_row_stride, sum_row_stride, y_row_stride, gamma, beta, eps, lpr_log2)
#define PV_ALN_N(TA, HB) do { if (nch == 1) PV_ALN(TA, HB, 1); else if (nch == 2) PV_ALN(TA, HB, 2); else PV_ALN(TA, HB, 3); } while (0)
  if (a_dtype == PV_F16) { if (b) PV_ALN_N(__half, true); else PV_ALN_N(__half, false); }
  else { if (b) PV_ALN_N(float, true); else PV_ALN_N(float, false); }
#undef PV_ALN_N
#undef PV_ALN
  PV_LAUNCH_OK("add_layernorm_kernel");
  return PV_OK;
}

extern "C" int pv_zero_f32(float* dst, long long n, void* stream) {
  PV_CHECK_ARG(dst || n == 0, "null pointer");
  if (n > 0) PV_CUDA_OK(cudaMemsetAsync(dst, 0, (size_t)n * sizeof(float), (cudaStream_t)stream));
  return PV_OK;
}

extern "C" int pv_ndhwc_to_ncdhw(const void* src, int src_dtype, long long src_row_stride,
                                 float* dst, int N, int C, int T, int H, int W, void* stream) {
  PV_CHECK_ARG(src && dst, "null pointer");
  const long long thw = (long long)T * H * W, total = (long long)N * C * thw;
  if (total == 0) return PV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid((unsigned)cdiv(total, 256)), block(256);
  if (src_dtype == PV_F16)
    ndhwc_to_ncdhw_kernel<__half><<<grid, block, 0, s>>>((const __half*)src, src_row_stride, dst, C, thw, total);
  else if (src_dtype == PV_F32)
    ndhwc_to_ncdhw_kernel<float><<<grid, block, 0, s>>>((const float*)src, src_row_stride, dst, C, thw, total);
  else { set_error("unsupported dtype %d", src_dtype); return PV_ERR_INVALID; }
  PV_LAUNCH_OK("ndhwc_to_ncdhw_kernel");
  return PV_OK;
}

namespace pv {
int conv3d_check(const pv_conv3d_desc* d) {
  PV_CHECK_ARG(d, "null descriptor");
  PV_CHECK_ARG(d->dtype == PV_F16 || d->dtype == PV_F32, "conv dtype must be f16|f32");
  PV_CHECK_ARG(act_known(d->act), "activation code %d unsupported", d->act);
  PV_CHECK_ARG(d->N >= 0 && d->Ci > 0 && d->Co > 0, "bad sizes");
  PV_CHECK_ARG(d->kt > 0 && d->kh > 0 && d->kw > 0 && d->st > 0 && d->sh > 0 && d->sw > 0 &&
                   d->dt > 0 && d->dh > 0 && d->dw > 0, "bad kernel/stride/dilation");
  const int to = (d->Ti + 2 * d->pt - d->dt * (d->kt - 1) - 1) / d->st + 1;
  const int ho = (d->Hi + 2 * d->ph - d->dh * (d->kh - 1) - 1) / d->sh + 1;
  const int wo = (d->Wi + 2 * d->pw - d->dw * (d->kw - 1) - 1) / d->sw + 1;
  PV_CHECK_ARG(to == d->To && ho == d->Ho && wo == d->Wo,
               "output dims (%d,%d,%d) inconsistent with conv arithmetic (%d,%d,%d)", d->To, d->Ho,
               d->Wo, to, ho, wo);
  PV_CHECK_ARG(d->groups >= 1 && d->Ci % d->groups == 0 && d->Co % d->groups == 0,
               "groups must divide Ci and Co; got groups=%d Ci=%d Co=%d", d->groups, d->Ci, d->Co);
  PV_CHECK_ARG(d->x_row_stride >= d->Ci && d->y_row_stride >= d->Co, "row stride < channels");
  PV_CHECK_ARG(!d->has_residual || d->res_row_stride >= d->Co, "residual row stride < Co");
  PV_CHECK_ARG(conv3d_addend_ok(d), "addend: 16-byte aligned pointer and non-negative strides / channel offset that "
               "are multiples of 8 elements required");
  PV_CHECK_ARG(conv3d_prologue_ok(d), "prologue: pre_scale and pre_bias both set, pre_act a known activation code");
  return PV_OK;
}

int dwconv3d_tile_launch(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                         const float* bias, void* y, float* se_sums, cudaStream_t stream);   // pv_dwconv.cu

int conv3d_direct_launch(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                         const float* bias, const void* residual, void* y, cudaStream_t s) {
  const long long M = (long long)d->N * d->To * d->Ho * d->Wo;
  if (M == 0) return PV_OK;
  const int esz = d->dtype == PV_F16 ? 2 : 4;
  if (d->groups == 1) {
    if (conv3d_has_prologue(d)) {
      set_error("the pre-activation prologue is taken by depthwise convolutions only");
      return PV_ERR_UNSUPPORTED;
    }
    PV_CHECK_ARG(d->Ci % 4 == 0 && d->Co % 4 == 0, "direct conv needs Ci%%4==0 && Co%%4==0");
    PV_CHECK_ARG((d->x_row_stride * esz) % (4 * esz) == 0 && (d->y_row_stride % 4) == 0,
                 "row strides must be multiples of 4 elements");
    dim3 grid((unsigned)cdiv(M, DC_BM), (unsigned)cdiv(d->Co, DC_BN)), block(256);
    if (d->dtype == PV_F16) {
      conv3d_direct_kernel<__half><<<grid, block, 0, s>>>(*d, (const __half*)x, (const __half*)w, scale, bias,
                                                       (const __half*)residual, (__half*)y, M);
      PV_LAUNCH_OK("conv3d_direct_kernel<__half>");
    } else {
      conv3d_direct_kernel<float><<<grid, block, 0, s>>>(*d, (const float*)x, (const float*)w, scale, bias,
                                                      (const float*)residual, (float*)y, M);
      PV_LAUNCH_OK("conv3d_direct_kernel<float>");
    }
  } else {
    if (d->addend) {
      set_error("depthwise convolutions take no addend");
      return PV_ERR_UNSUPPORTED;
    }
    if (d->groups != d->Ci || d->Ci != d->Co) {
      set_error("PV_ALGO_DIRECT runs dense (groups=1) and depthwise (groups==Ci==Co) convolutions only; got groups=%d "
                "Ci=%d Co=%d", d->groups, d->Ci, d->Co);
      return PV_ERR_UNSUPPORTED;
    }
    PV_CHECK_ARG(d->Co % 8 == 0, "depthwise conv needs C%%8==0");
    const bool pre = d->pre_scale != nullptr;
    PV_CHECK_ARG(d->x_row_stride % 8 == 0 && d->y_row_stride % 8 == 0, "row strides must be multiples of 8");
    // TMA-fed shared-memory stencil (pv_dwconv.cu) whenever it applies
    if (!d->has_residual && d->dtype == PV_F16) {
      const int rc = dwconv3d_tile_launch(d, x, w, scale, bias, y, nullptr, s);
      if (rc != PV_ERR_UNSUPPORTED) return rc;
    }
    // register-tiled variant for the common stencils (dilation_w 1, kw in {1,3}, stride_w in {1,2}, no residual)
    if (!d->has_residual && d->dw == 1 && (d->kw == 3 || d->kw == 1) && (d->sw == 1 || d->sw == 2) && d->Wo >= 4) {
      const int wo4 = (d->Wo + 3) / 4;
      const long long tot4 = (long long)d->N * d->To * d->Ho * wo4 * (d->Co / 8);
      dim3 g4((unsigned)cdiv(tot4, 128)), b4(128);
#define PV_DW2(TT, KW_, SW_, PRE_)                                                                                     \
  do {                                                                                                                 \
    dwconv3d_w4_kernel<TT, KW_, SW_, PRE_><<<g4, b4, 0, s>>>(*d, (const TT*)x, (const TT*)w, scale, bias, (TT*)y, tot4, \
                                                             wo4);                                                     \
    PV_LAUNCH_OK(PV_PRE_NAME("dwconv3d_w4_kernel<" #TT "," #KW_ "," #SW_, PRE_));                                      \
  } while (0)
#define PV_DW(TT, KW_, SW_)                                                                                            \
  do {                                                                                                                 \
    if (pre) PV_DW2(TT, KW_, SW_, true); else PV_DW2(TT, KW_, SW_, false);                                             \
  } while (0)
      if (d->dtype == PV_F16) {
        if (d->kw == 3 && d->sw == 1) PV_DW(__half, 3, 1); else if (d->kw == 3) PV_DW(__half, 3, 2);
        else if (d->sw == 1) PV_DW(__half, 1, 1); else PV_DW(__half, 1, 2);
      } else {
        if (d->kw == 3 && d->sw == 1) PV_DW(float, 3, 1); else if (d->kw == 3) PV_DW(float, 3, 2);
        else if (d->sw == 1) PV_DW(float, 1, 1); else PV_DW(float, 1, 2);
      }
#undef PV_DW
#undef PV_DW2
      return PV_OK;
    }
    const long long total = M * (d->Co / 8);
    dim3 grid((unsigned)cdiv(total, 256)), block(256);
#define PV_DWG(TT, PRE_)                                                                                               \
  do {                                                                                                                 \
    dwconv3d_kernel<TT, PRE_><<<grid, block, 0, s>>>(*d, (const TT*)x, (const TT*)w, scale, bias, (const TT*)residual, \
                                                     (TT*)y, total);                                                   \
    PV_LAUNCH_OK(PV_PRE_NAME("dwconv3d_kernel<" #TT, PRE_));                                                           \
  } while (0)
    if (d->dtype == PV_F16) {
      if (pre) PV_DWG(__half, true); else PV_DWG(__half, false);
    } else {
      if (pre) PV_DWG(float, true); else PV_DWG(float, false);
    }
#undef PV_DWG
  }
  return PV_OK;
}
}  // namespace pv

extern "C" int pv_pool3d_fwd(const pv_pool3d_desc* d, const void* x, void* y, void* stream) {
  PV_CHECK_ARG(d && x && y, "null argument");
  PV_CHECK_ARG(d->dtype == PV_F16 || d->dtype == PV_F32, "pool dtype must be f16|f32");
  PV_CHECK_ARG(d->C % 8 == 0 && d->x_row_stride % 8 == 0 && d->y_row_stride % 8 == 0,
               "pool needs C and row strides %% 8 == 0");
  PV_CHECK_ARG(d->mode == PV_POOL_MAX || d->mode == PV_POOL_AVG, "bad pool mode");
  const int to = (d->Ti + 2 * d->pt - d->kt) / d->st + 1;
  const int ho = (d->Hi + 2 * d->ph - d->kh) / d->sh + 1;
  const int wo = (d->Wi + 2 * d->pw - d->kw) / d->sw + 1;
  PV_CHECK_ARG(to == d->To && ho == d->Ho && wo == d->Wo, "pool output dims inconsistent");
  const long long total = (long long)d->N * d->To * d->Ho * d->Wo * (d->C / 8);
  if (total == 0) return PV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  if (to == 1 && ho == 1 && wo == 1 && d->kt == d->Ti && d->kh == d->Hi && d->kw == d->Wi && d->pt == 0 &&
      d->ph == 0 && d->pw == 0 && d->N <= 65535 && d->x_batch_stride == 0 && d->y_batch_stride == 0) {
    const long long npos = (long long)d->Ti * d->Hi * d->Wi;
    dim3 grid((unsigned)cdiv(d->C, 64), d->N), block(256);
    if (d->dtype == PV_F16)
      global_pool_kernel<__half><<<grid, block, 0, s>>>((const __half*)x, (__half*)y, d->x_row_stride,
                                                      d->y_row_stride, npos, d->C, d->mode == PV_POOL_MAX);
    else
      global_pool_kernel<float><<<grid, block, 0, s>>>((const float*)x, (float*)y, d->x_row_stride,
                                                     d->y_row_stride, npos, d->C, d->mode == PV_POOL_MAX);
    PV_LAUNCH_OK("global_pool_kernel");
    return PV_OK;
  }
  dim3 grid((unsigned)cdiv(total, 256)), block(256);
  if (d->dtype == PV_F16)
    pool3d_kernel<__half><<<grid, block, 0, s>>>(*d, (const __half*)x, (__half*)y, total);
  else
    pool3d_kernel<float><<<grid, block, 0, s>>>(*d, (const float*)x, (float*)y, total);
  PV_LAUNCH_OK("pool3d_kernel");
  return PV_OK;
}

extern "C" int pv_channel_sum(const void* x, int dtype, long long row_stride, int N,
                              long long npos, int C, float* sums, void* stream) {
  PV_CHECK_ARG(x && sums, "null pointer");
  PV_CHECK_ARG(C % 8 == 0 && row_stride % 8 == 0, "C and row stride must be multiples of 8");
  if (N == 0 || npos == 0) return PV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  long long chunks = cdiv(npos, 2048);
  if (chunks > 1024) chunks = 1024;
  const long long chunk = cdiv(npos, chunks);
  chunks = cdiv(npos, chunk);
  dim3 grid((unsigned)chunks, N), block(256);
  size_t smem = (size_t)C * sizeof(unsigned long long);
  if (dtype == PV_F16)
    channel_sum_kernel<__half><<<grid, block, smem, s>>>((const __half*)x, row_stride, npos, C, chunk, sums);
  else if (dtype == PV_F32)
    channel_sum_kernel<float><<<grid, block, smem, s>>>((const float*)x, row_stride, npos, C, chunk, sums);
  else { set_error("unsupported dtype %d", dtype); return PV_ERR_INVALID; }
  PV_LAUNCH_OK("channel_sum_kernel");
  return PV_OK;
}

extern "C" int pv_se_gate(const float* sums, long long npos, int N, int C, int Cr, const float* w1,
                          const float* b1, const float* w2, const float* b2, int c_stride_w,
                          float* gate, void* stream) {
  PV_CHECK_ARG(sums && w1 && b1 && w2 && b2 && gate, "null pointer");
  PV_CHECK_ARG(npos > 0 && C > 0 && Cr > 0, "bad sizes");
  if (N == 0) return PV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  size_t smem = (size_t)(C + Cr) * sizeof(float);
  se_gate_kernel<<<N, 256, smem, s>>>(sums, 1.f / (float)npos, C, Cr, w1, b1, w2, b2, c_stride_w, gate);
  PV_LAUNCH_OK("se_gate_kernel");
  return PV_OK;
}

extern "C" int pv_scale_act(const void* x, void* y, int dtype, long long x_row_stride,
                            long long y_row_stride, int N, long long npos, int C,
                            const float* gate, int act, void* stream) {
  PV_CHECK_ARG(x && y, "null pointer");
  PV_CHECK_ARG(act_known(act), "activation code %d unsupported", act);
  PV_CHECK_ARG(C % 8 == 0 && x_row_stride % 8 == 0 && y_row_stride % 8 == 0, "C/strides %% 8");
  const long long total = (long long)N * npos * (C / 8);
  if (total == 0) return PV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid((unsigned)cdiv(total, 256)), block(256);
  if (dtype == PV_F16)
    scale_act_kernel<__half><<<grid, block, 0, s>>>((const __half*)x, (__half*)y, x_row_stride, y_row_stride,
                                                 npos, C, gate, act, total);
  else if (dtype == PV_F32)
    scale_act_kernel<float><<<grid, block, 0, s>>>((const float*)x, (float*)y, x_row_stride, y_row_stride,
                                                npos, C, gate, act, total);
  else { set_error("unsupported dtype %d", dtype); return PV_ERR_INVALID; }
  PV_LAUNCH_OK("scale_act_kernel");
  return PV_OK;
}

extern "C" int pv_head_reduce(const void* x, int dtype, long long row_stride, int N,
                              long long npos, int C_valid, int softmax, float* out, void* stream) {
  PV_CHECK_ARG(x && out, "null pointer");
  PV_CHECK_ARG(C_valid > 0 && npos > 0, "bad sizes");
  if (N == 0) return PV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  size_t smem = (size_t)(C_valid + 32) * sizeof(float);
  if (dtype == PV_F16)
    head_reduce_kernel<__half><<<N, 256, smem, s>>>((const __half*)x, row_stride, npos, C_valid, softmax, out);
  else if (dtype == PV_F32)
    head_reduce_kernel<float><<<N, 256, smem, s>>>((const float*)x, row_stride, npos, C_valid, softmax, out);
  else { set_error("unsupported dtype %d", dtype); return PV_ERR_INVALID; }
  PV_LAUNCH_OK("head_reduce_kernel");
  return PV_OK;
}

extern "C" int pv_layernorm_sets(const void* x, void* y, int dtype, long long rows, int groups, int C,
                                 long long x_row_stride, long long y_row_stride, const float* gamma,
                                 const float* beta, int groups_per_set, const void* cls_src,
                                 long long cls_batch_stride, long long npos, float eps, void* stream) {
  PV_CHECK_ARG(x && y && gamma && beta, "null pointer");
  PV_CHECK_ARG(groups_per_set >= 1 && groups % groups_per_set == 0, "groups %% groups_per_set");
  PV_CHECK_ARG(!cls_src || (npos >= 1 && rows % npos == 0 && cls_batch_stride % 8 == 0), "cls rows: rows %% npos, stride %% 8");
  pv::LnExtra X;
  X.groups_per_set = groups_per_set; X.cls_src = cls_src; X.cls_batch_stride = cls_batch_stride; X.npos = npos > 0 ? npos : 1;
  PV_CHECK_ARG(groups >= 1 && C % 8 == 0 && x_row_stride % 8 == 0 && y_row_stride % 8 == 0, "C/strides %% 8");
  PV_CHECK_ARG(x_row_stride >= (long long)groups * C && y_row_stride >= (long long)groups * C, "row stride < groups*C");
  if (rows == 0) return PV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const int chunks = (C + 7) / 8;
  int lpr_log2 = 2;
  while ((1 << lpr_log2) < chunks && lpr_log2 < 5) ++lpr_log2;
  const int nch = (chunks + (1 << lpr_log2) - 1) >> lpr_log2;
  const bool aligned16 = (((uintptr_t)gamma | (uintptr_t)beta) & 15) == 0;
  if (nch <= 3 && aligned16 && (dtype == PV_F16 || dtype == PV_F32)) {
    const long long per_block = 8ll << (5 - lpr_log2);     // rows per 256-thread block
    dim3 grid((unsigned)cdiv(rows * groups, per_block)), block(256);
#define PV_LN(TT, N_) layernorm_reg_kernel<TT, N_><<<grid, block, 0, s>>>((const TT*)x, (TT*)y, rows, groups, C, x_row_stride, y_row_stride, gamma, beta, eps, lpr_log2, X)
    if (dtype == PV_F16) { if (nch == 1) PV_LN(__half, 1); else if (nch == 2) PV_LN(__half, 2); else PV_LN(__half, 3); }
    else { if (nch == 1) PV_LN(float, 1); else if (nch == 2) PV_LN(float, 2); else PV_LN(float, 3); }
#undef PV_LN
    PV_LAUNCH_OK("layernorm_reg_kernel");
    return PV_OK;
  }
  dim3 grid((unsigned)cdiv(rows * groups, 8)), block(256);
  if (dtype == PV_F16)
    layernorm_kernel<__half><<<grid, block, 0, s>>>((const __half*)x, (__half*)y, rows, groups, C, x_row_stride,
                                                 y_row_stride, gamma, beta, eps, X);
  else if (dtype == PV_F32)
    layernorm_kernel<float><<<grid, block, 0, s>>>((const float*)x, (float*)y, rows, groups, C, x_row_stride,
                                                y_row_stride, gamma, beta, eps, X);
  else { set_error("unsupported dtype %d", dtype); return PV_ERR_INVALID; }
  PV_LAUNCH_OK("layernorm_kernel");
  return PV_OK;
}

extern "C" int pv_layernorm(const void* x, void* y, int dtype, long long rows, int groups, int C,
                            long long x_row_stride, long long y_row_stride, const float* gamma,
                            const float* beta, float eps, void* stream) {
  return pv_layernorm_sets(x, y, dtype, rows, groups, C, x_row_stride, y_row_stride, gamma, beta, groups > 0 ? groups : 1,
                           nullptr, 0, 1, eps, stream);
}

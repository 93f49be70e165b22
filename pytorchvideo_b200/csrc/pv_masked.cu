// Masked sequence ops of models/masked_multistream.py and layers/fusion.py: masked temporal pooling, the learned
// default of rows without a valid step, the forced first mask column of the attention modules, and the elementwise
// reduce fusion.  Token rows [B][T][C] with C % 8 == 0 (8-channel vectors, fp32 maths); masks are u8 [B][T].
#include "pv_common.cuh"

namespace pv {

// one thread per (row b, 8-channel group): the T steps are walked in order, so the sums are deterministic
template <typename T, int MODE>
__global__ void __launch_bounds__(256)
masked_pool_kernel(const T* __restrict__ x, long long xrs, int B, int Tn, int C, const unsigned char* __restrict__ mask,
                   T* __restrict__ y, long long yrs) {
  const int G = C >> 3;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)B * G) return;
  const int b = (int)(e / G), c = (int)(e - (long long)b * G) * 8;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = MODE == 0 ? -INFINITY : 0.f;
  int cnt = 0;
  for (int t = 0; t < Tn; ++t) {
    if (mask && !mask[(long long)b * Tn + t]) continue;
    ++cnt;
    float v[8];
    ld8<T>(x + ((long long)b * Tn + t) * xrs + c, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = MODE == 0 ? fmaxf(acc[i], v[i]) : acc[i] + v[i];
  }
  if (MODE == 0 && cnt == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;      // a row with no valid step pools to 0
  }
  if (MODE == 1) {
    const float n = (float)(cnt > 0 ? cnt : 1);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = acc[i] / n;
  }
  st8<T>(y + (long long)b * yrs + c, acc);
}

template <typename T>
__global__ void __launch_bounds__(256)
masked_default_kernel(const T* __restrict__ x, long long xrs, int B, int C, const unsigned char* __restrict__ mask,
                      int Tn, const float* __restrict__ def, T* __restrict__ y, long long yrs) {
  const int G = C >> 3;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)B * G) return;
  const int b = (int)(e / G), c = (int)(e - (long long)b * G) * 8;
  bool any = mask == nullptr;
  for (int t = 0; t < Tn && !any; ++t) any = mask[(long long)b * Tn + t] != 0;
  const float a = any ? 1.f : 0.f;
  float v[8];
  ld8<T>(x + (long long)b * xrs + c, v);
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = v[i] * a + __ldg(def + c + i) * (1.f - a);   // the reference's formula, in fp32
  st8<T>(y + (long long)b * yrs + c, v);
}

__global__ void mask_force_first_kernel(const unsigned char* __restrict__ src, unsigned char* __restrict__ dst,
                                        long long total, int Tn) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  dst[e] = (e % Tn) == 0 ? (unsigned char)1 : src[e];
}

struct ReduceSrcs {
  const void* x[8];
  long long rs[8];
};

template <typename T, int OP>
__global__ void __launch_bounds__(256)
reduce_fusion_kernel(ReduceSrcs S, int P, long long rows, int C, T* __restrict__ y, long long yrs) {
  const int G = C >> 3;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= rows * G) return;
  const long long r = e / G;
  const int c = (int)(e - r * G) * 8;
  float acc[8];
  ld8<T>((const T*)S.x[0] + r * S.rs[0] + c, acc);
  for (int p = 1; p < P; ++p) {
    float v[8];
    ld8<T>((const T*)S.x[p] + r * S.rs[p] + c, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = OP == 0 ? fmaxf(acc[i], v[i]) : (OP == 1 ? acc[i] + v[i] : acc[i] * v[i]);
  }
  st8<T>(y + r * yrs + c, acc);
}

}  // namespace pv

using namespace pv;

extern "C" int pv_masked_pool(const void* x, int dtype, long long x_row_stride, int B, int T, int C,
                              const unsigned char* mask, int mode, void* y, long long y_row_stride, void* stream) {
  PV_CHECK_ARG(x && y, "null pointer");
  PV_CHECK_ARG(B > 0 && T > 0 && C > 0 && C % 8 == 0, "bad shape B=%d T=%d C=%d (C %% 8 == 0)", B, T, C);
  PV_CHECK_ARG(x_row_stride % 8 == 0 && y_row_stride % 8 == 0 && x_row_stride >= C && y_row_stride >= C,
               "row strides must be multiples of 8 and >= C");
  PV_CHECK_ARG(mode >= 0 && mode <= 2, "pool mode %d (0 max, 1 avg, 2 sum)", mode);
  const long long total = (long long)B * (C / 8);
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = (unsigned)cdiv(total, 256);
#define PV_MP(TT, MODE_)                                                                                        \
  {                                                                                                             \
    masked_pool_kernel<TT, MODE_><<<grid, 256, 0, s>>>((const TT*)x, x_row_stride, B, T, C, mask, (TT*)y,       \
                                                       y_row_stride);                                           \
    PV_LAUNCH_OK("masked_pool_kernel<" #TT "," #MODE_ ">");                                                     \
    return PV_OK;                                                                                               \
  }
  if (dtype == PV_F16) {
    if (mode == 0) PV_MP(__half, 0)
    if (mode == 1) PV_MP(__half, 1)
    PV_MP(__half, 2)
  }
  if (dtype == PV_F32) {
    if (mode == 0) PV_MP(float, 0)
    if (mode == 1) PV_MP(float, 1)
    PV_MP(float, 2)
  }
#undef PV_MP
  set_error("unsupported dtype %d", dtype);
  return PV_ERR_INVALID;
}

extern "C" int pv_masked_default(const void* x, int dtype, long long x_row_stride, int B, int C,
                                 const unsigned char* mask, int T, const float* def, void* y, long long y_row_stride,
                                 void* stream) {
  PV_CHECK_ARG(x && y && def, "null pointer");
  PV_CHECK_ARG(B > 0 && C > 0 && C % 8 == 0 && (mask == nullptr || T > 0), "bad shape B=%d C=%d T=%d", B, C, T);
  PV_CHECK_ARG(x_row_stride % 8 == 0 && y_row_stride % 8 == 0 && x_row_stride >= C && y_row_stride >= C,
               "row strides must be multiples of 8 and >= C");
  const long long total = (long long)B * (C / 8);
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = (unsigned)cdiv(total, 256);
  if (dtype == PV_F16) {
    masked_default_kernel<__half><<<grid, 256, 0, s>>>((const __half*)x, x_row_stride, B, C, mask, T, def, (__half*)y,
                                                       y_row_stride);
    PV_LAUNCH_OK("masked_default_kernel<__half>");
  } else if (dtype == PV_F32) {
    masked_default_kernel<float><<<grid, 256, 0, s>>>((const float*)x, x_row_stride, B, C, mask, T, def, (float*)y,
                                                      y_row_stride);
    PV_LAUNCH_OK("masked_default_kernel<float>");
  } else {
    set_error("unsupported dtype %d", dtype);
    return PV_ERR_INVALID;
  }
  return PV_OK;
}

extern "C" int pv_mask_force_first(const unsigned char* src, unsigned char* dst, int B, int T, void* stream) {
  PV_CHECK_ARG(src && dst, "null pointer");
  PV_CHECK_ARG(B > 0 && T > 0, "bad shape B=%d T=%d", B, T);
  const long long total = (long long)B * T;
  mask_force_first_kernel<<<(unsigned)cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(src, dst, total, T);
  PV_LAUNCH_OK("mask_force_first_kernel");
  return PV_OK;
}

extern "C" int pv_reduce_fusion(const void* const* xs, const long long* x_row_strides, int P, int dtype, long long rows,
                                int C, int op, void* y, long long y_row_stride, void* stream) {
  PV_CHECK_ARG(xs && x_row_strides && y, "null pointer");
  PV_CHECK_ARG(P >= 1 && P <= 8, "reduce fusion takes 1 to 8 inputs, got %d", P);
  PV_CHECK_ARG(rows > 0 && C > 0 && C % 8 == 0 && y_row_stride % 8 == 0 && y_row_stride >= C, "bad shape");
  PV_CHECK_ARG(op >= 0 && op <= 2, "reduce op %d (0 max, 1 sum, 2 prod)", op);
  ReduceSrcs S;
  for (int p = 0; p < 8; ++p) {
    S.x[p] = p < P ? xs[p] : nullptr;
    S.rs[p] = p < P ? x_row_strides[p] : 0;
    if (p < P) PV_CHECK_ARG(xs[p] && S.rs[p] % 8 == 0 && S.rs[p] >= C, "input %d: null or bad row stride", p);
  }
  const long long total = rows * (C / 8);
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = (unsigned)cdiv(total, 256);
#define PV_RF(TT, OP_)                                                                                \
  {                                                                                                   \
    reduce_fusion_kernel<TT, OP_><<<grid, 256, 0, s>>>(S, P, rows, C, (TT*)y, y_row_stride);          \
    PV_LAUNCH_OK("reduce_fusion_kernel<" #TT "," #OP_ ">");                                           \
    return PV_OK;                                                                                     \
  }
  if (dtype == PV_F16) {
    if (op == 0) PV_RF(__half, 0)
    if (op == 1) PV_RF(__half, 1)
    PV_RF(__half, 2)
  }
  if (dtype == PV_F32) {
    if (op == 0) PV_RF(float, 0)
    if (op == 1) PV_RF(float, 1)
    PV_RF(float, 2)
  }
#undef PV_RF
  set_error("unsupported dtype %d", dtype);
  return PV_ERR_INVALID;
}

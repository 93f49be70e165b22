// Shared helpers for libpvb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/pv_b200.h"

namespace pv {

// ---- error plumbing -------------------------------------------------------------------------
void set_error(const char* fmt, ...);
// Counts one launch of `name`, a string literal naming the kernel with its template arguments
// ("conv3d_igemm_kernel<64,128>"); read back with pv_kernel_counts.
void count_launch(const char* name);

#define PV_CHECK_ARG(cond, ...)            \
  do {                                     \
    if (!(cond)) {                         \
      pv::set_error(__VA_ARGS__);          \
      return PV_ERR_INVALID;               \
    }                                      \
  } while (0)

#define PV_CUDA_OK(expr)                                                                   \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      pv::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,      \
                    __LINE__);                                                             \
      return PV_ERR_CUDA;                                                                  \
    }                                                                                      \
  } while (0)

#define PV_LAUNCH_OK(name)                                                                 \
  do {                                                                                     \
    cudaError_t _e = cudaPeekAtLastError();                                                \
    if (_e != cudaSuccess) {                                                               \
      pv::set_error("launch of %s failed: %s", name, cudaGetErrorString(_e));              \
      (void)cudaGetLastError();                                                            \
      return PV_ERR_CUDA;                                                                  \
    }                                                                                      \
    pv::count_launch(name);                                                                \
  } while (0)

static inline long long cdiv(long long a, long long b) { return (a + b - 1) / b; }

// Layout rules of pv_conv3d_desc.addend (16-byte vectors of 8 channels on every path that takes it, so Co % 8 == 0:
// the last vector of a row must not reach past the Co channels of the addend slice).
static inline bool conv3d_addend_ok(const pv_conv3d_desc* d) {
  return !d->addend || ((uintptr_t)d->addend % 16 == 0 && d->Co % 8 == 0 && d->add_n_stride >= 0 && d->add_t_stride >= 0 &&
                        d->add_ch_off >= 0 && d->add_n_stride % 8 == 0 && d->add_t_stride % 8 == 0 &&
                        d->add_ch_off % 8 == 0 && (long long)d->N * d->To * d->Ho * d->Wo < (1ll << 31));
}

// ---- per-device launch state -------------------------------------------------------------------
// Function attributes (opt-in dynamic shared memory) and the SM count are PER DEVICE: a process that runs a
// plan on cuda:0 and later on cuda:1 must opt in again on the second device.  One flag word per launch site,
// one bit per device ordinal (devices >= 64 simply re-set the attribute on every launch).
struct DeviceOnce {
  unsigned long long done = 0ull;
  // true exactly once per (site, current device)
  bool first(int dev) {
    if (dev < 0 || dev >= 64) return true;
    const unsigned long long bit = 1ull << dev;
    if (done & bit) return false;
    done |= bit;
    return true;
  }
};
static inline int current_device() {
  int dev = 0;
  return cudaGetDevice(&dev) == cudaSuccess ? dev : -1;
}
// SM count of the CURRENT device (cached per ordinal)
static inline int current_sm_count() {
  static int cache[64] = {0};
  const int dev = current_device();
  if (dev >= 0 && dev < 64 && cache[dev] > 0) return cache[dev];
  int n = 0;
  if (dev < 0 || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 0;
  if (dev < 64) cache[dev] = n;
  return n;
}
#define PV_OPT_IN_SMEM(kernel, bytes)                                                                   \
  do {                                                                                                  \
    static pv::DeviceOnce _once;                                                                        \
    if (_once.first(pv::current_device()))                                                              \
      PV_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))); \
  } while (0)

// ---- element helpers ------------------------------------------------------------------------
template <typename T> struct Elem;
template <> struct Elem<__half> {
  static __device__ __forceinline__ float ld(const __half* p) { return __half2float(*p); }
  static __device__ __forceinline__ void st(__half* p, float v) { *p = __float2half_rn(v); }
};
template <> struct Elem<float> {
  static __device__ __forceinline__ float ld(const float* p) { return *p; }
  static __device__ __forceinline__ void st(float* p, float v) { *p = v; }
};

// 4-element vector load / store with fp32 maths
template <typename T> __device__ __forceinline__ void ld4(const T* p, float (&v)[4]);
template <> __device__ __forceinline__ void ld4<__half>(const __half* p, float (&v)[4]) {
  uint2 r = *reinterpret_cast<const uint2*>(p);
  __half2 a = *reinterpret_cast<__half2*>(&r.x), b = *reinterpret_cast<__half2*>(&r.y);
  float2 fa = __half22float2(a), fb = __half22float2(b);
  v[0] = fa.x; v[1] = fa.y; v[2] = fb.x; v[3] = fb.y;
}
template <> __device__ __forceinline__ void ld4<float>(const float* p, float (&v)[4]) {
  float4 r = *reinterpret_cast<const float4*>(p);
  v[0] = r.x; v[1] = r.y; v[2] = r.z; v[3] = r.w;
}
template <typename T> __device__ __forceinline__ void st4(T* p, const float (&v)[4]);
template <> __device__ __forceinline__ void st4<__half>(__half* p, const float (&v)[4]) {
  __half2 a = __floats2half2_rn(v[0], v[1]), b = __floats2half2_rn(v[2], v[3]);
  uint2 r;
  r.x = *reinterpret_cast<uint32_t*>(&a);
  r.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = r;
}
template <> __device__ __forceinline__ void st4<float>(float* p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}

// 8-element vector load / store
template <typename T> __device__ __forceinline__ void ld8(const T* p, float (&v)[8]);
template <> __device__ __forceinline__ void ld8<__half>(const __half* p, float (&v)[8]) {
  uint4 r = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f = __half22float2(h[i]);
    v[2 * i] = f.x; v[2 * i + 1] = f.y;
  }
}
template <> __device__ __forceinline__ void ld8<float>(const float* p, float (&v)[8]) {
  float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <typename T> __device__ __forceinline__ void st8(T* p, const float (&v)[8]);
template <> __device__ __forceinline__ void st8<__half>(__half* p, const float (&v)[8]) {
  uint4 r;
  __half2* h = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = r;
}
template <> __device__ __forceinline__ void st8<float>(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}

// Squeeze-Excitation sums ([N][C] per-channel sums over positions) are accumulated as 64-bit fixed point with a
// resolution of 2^-24: integer atomics commute, so the sums do not depend on the order in which blocks add their
// partials.  The buffer holds one int64 per (sample, channel) (2 * N * C floats of storage).
__device__ __forceinline__ long long se_fix(float v) { return __float2ll_rn(v * 16777216.f); }
__device__ __forceinline__ void se_sum_add(float* sums, long long idx, float v) {
  atomicAdd(reinterpret_cast<unsigned long long*>(sums) + idx, (unsigned long long)se_fix(v));
}
__device__ __forceinline__ float se_sum_get(const float* sums, long long idx) {
  return (float)((double)reinterpret_cast<const long long*>(sums)[idx] * (1.0 / 16777216.0));
}

// torch.nn.Hardswish in fp32, in torch's order: x * min(max(x + 3, 0), 6) / 6 (a true division, not a multiply by 1/6)
__device__ __forceinline__ float hswish(float x) { return x * fminf(fmaxf(x + 3.f, 0.f), 6.f) / 6.f; }

__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case PV_ACT_RELU: return fmaxf(x, 0.f);
    case PV_ACT_SWISH: return x / (1.f + __expf(-x));
    case PV_ACT_GELU: return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f));
    case PV_ACT_SIGMOID: return 1.f / (1.f + __expf(-x));
    case PV_ACT_HSWISH: return hswish(x);
    default: return x;
  }
}

// The activation codes the library implements; entry points reject every other code (pv_b200.h pv_act), so no
// kernel ever sees one.
inline bool act_known(int act) { return act >= PV_ACT_NONE && act <= PV_ACT_HSWISH; }

// ---- pre-activation prologue of the depthwise kernels (pv_conv3d_desc.pre_scale / pre_bias / pre_act) -------------
inline bool conv3d_has_prologue(const pv_conv3d_desc* d) { return d->pre_scale || d->pre_bias || d->pre_act; }
inline bool conv3d_prologue_ok(const pv_conv3d_desc* d) {
  return !conv3d_has_prologue(d) || (d->pre_scale && d->pre_bias && act_known(d->pre_act));
}
// Launch-ledger name of a kernel instance with / without the prologue: "<base>>" or "<base>,pre>".
#define PV_PRE_NAME(base, pre) ((pre) ? base ",pre>" : base ">")

__device__ __forceinline__ float pre_u(float x, float s, float b, int act) { return apply_act(fmaf(s, x, b), act); }

// The prologue in place on a landed f16 halo box [outer][tt][hh][ww][cc]: element (t, h, w, c) of every outer slice is
// input position (t0 + t, h0 + h, w0 + w), channel c0 + c.  Only in-bounds positions of channels < C are transformed:
// the rest is the TMA zero fill, i.e. the convolution's zero padding, which must stay 0 although u(0) != 0.  A thread
// keeps one channel pair (its prologue constants in registers) and walks whole halo rows, so the index arithmetic is
// paid once per row; consecutive threads touch consecutive 4-byte words.  Each element is transformed once and rounded
// to f16; the caller synchronises the CTA before the stencil reads the box.
__device__ __forceinline__ void halo_prologue(__half* xs, int outer, int tt, int hh, int ww, int cc, int c0, int C,
                                              int t0, int h0, int w0, int Ti, int Hi, int Wi,
                                              const float* __restrict__ ps, const float* __restrict__ pb, int act) {
  const int cp = cc >> 1;
  const int nrow = blockDim.x / cp;
  const int ci = threadIdx.x % cp, r0 = threadIdx.x / cp;
  const int ch = c0 + 2 * ci;
  if (r0 >= nrow || ch >= C) return;
  const float s0 = __ldg(ps + ch), s1 = __ldg(ps + ch + 1), b0 = __ldg(pb + ch), b1 = __ldg(pb + ch + 1);
  const int wlo = max(0, -w0), whi = min(ww, Wi - w0);
  __half2* x2 = reinterpret_cast<__half2*>(xs) + ci;
  const int rows = outer * tt * hh;
  for (int r = r0; r < rows; r += nrow) {
    const int h = r % hh, t = (r / hh) % tt;
    if ((unsigned)(t0 + t) >= (unsigned)Ti || (unsigned)(h0 + h) >= (unsigned)Hi) continue;
    __half2* row = x2 + r * ww * cp;
    for (int w = wlo; w < whi; ++w) {
      const float2 v = __half22float2(row[w * cp]);
      row[w * cp] = __floats2half2_rn(pre_u(v.x, s0, b0, act), pre_u(v.y, s1, b1, act));
    }
  }
}

}  // namespace pv

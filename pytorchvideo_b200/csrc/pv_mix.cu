// Batch mixing (transforms/mix.py: MixUp, CutMix, MixVideo) in place on a batch of clips, and the mixed soft labels.
//
// Clip b pairs with clip B-1-b (the reference's x.flip(0)).  One thread owns one element of both clips of a pair, reads
// both values and writes both results, so the batch is mixed in place without a temporary.  MixUp restates the
// reference's eager sequence flip(0).mul_(1 - lam), mul_(lam), add_ with one rounding to the element type per op; the
// products are fp32 (ATen multiplies a float16 tensor by the float32 scalar in fp32) and __fmul_rn / __fadd_rn keep
// nvcc from contracting them into an FMA the CPU does not do.
#include "pv_common.cuh"

namespace pv {
namespace mix {

constexpr int THREADS = 256;

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

// T(T(a * lam) + T(b * oml)), every intermediate rounded to T as the eager ops store it
template <typename T> __device__ __forceinline__ T mix1(T a, T b, float lam, float oml) {
  const float pa = to_f(from_f<T>(__fmul_rn(to_f(a), lam)));
  const float pb = to_f(from_f<T>(__fmul_rn(to_f(b), oml)));
  return from_f<T>(__fadd_rn(pa, pb));
}

// ---- MixUp, any strides: blockIdx.y is the pair, x runs over the elements of one clip ------------------------------
template <typename T>
__global__ void __launch_bounds__(THREADS)
mixup_kernel(pv_mix_desc d, T* __restrict__ x, float lam, float oml) {
  const long long n = d.size[0] * d.size[1] * d.size[2] * d.size[3];
  const long long e = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (e >= n) return;
  long long r = e, off = 0;
#pragma unroll
  for (int i = 3; i > 0; --i) {
    const long long q = r / d.size[i];
    off += (r - q * d.size[i]) * d.stride[i];
    r = q;
  }
  off += r * d.stride[0];
  const int p = blockIdx.y, q = d.B - 1 - p;
  T* xp = x + (long long)p * d.s_batch + off;
  T* xq = x + (long long)q * d.s_batch + off;
  const T a = *xp, b = *xq;
  *xp = mix1<T>(a, b, lam, oml);
  if (q != p) *xq = mix1<T>(b, a, lam, oml);
}

// ---- MixUp on clips whose elements fill one dense block: 16-byte vectors ------------------------------------------
template <typename T>
__global__ void __launch_bounds__(THREADS)
mixup_vec_kernel(pv_mix_desc d, T* __restrict__ x, long long n_vec, float lam, float oml) {
  constexpr int V = 16 / sizeof(T);
  const long long v = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (v >= n_vec) return;
  const int p = blockIdx.y, q = d.B - 1 - p;
  uint4* xp = reinterpret_cast<uint4*>(x + (long long)p * d.s_batch) + v;
  uint4* xq = reinterpret_cast<uint4*>(x + (long long)q * d.s_batch) + v;
  uint4 ra = *xp, rb = *xq, oa, ob;
  const T* a = reinterpret_cast<const T*>(&ra);
  const T* b = reinterpret_cast<const T*>(&rb);
  T* ya = reinterpret_cast<T*>(&oa);
  T* yb = reinterpret_cast<T*>(&ob);
#pragma unroll
  for (int i = 0; i < V; ++i) {
    ya[i] = mix1<T>(a[i], b[i], lam, oml);
    yb[i] = mix1<T>(b[i], a[i], lam, oml);
  }
  *xp = oa;
  if (q != p) *xq = ob;
}

// ---- CutMix: swap the box of clips p and B-1-p across the outer dims; element size ES bytes -------------------------
template <int ES> struct Word;
template <> struct Word<1> { typedef uint8_t type; };
template <> struct Word<2> { typedef uint16_t type; };
template <> struct Word<4> { typedef uint32_t type; };

template <int ES>
__global__ void __launch_bounds__(THREADS)
cutmix_kernel(pv_mix_desc d, typename Word<ES>::type* __restrict__ x, int yl, int xl, int bh, int bw) {
  const long long n = d.size[0] * d.size[1] * bh * bw;
  const long long e = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (e >= n) return;
  const long long row = e / bw;
  const int xi = (int)(e - row * bw);
  const long long plane = row / bh;
  const int yi = (int)(row - plane * bh);
  const long long c = plane / d.size[1], t = plane - c * d.size[1];
  const long long off = c * d.stride[0] + t * d.stride[1] + (long long)(yl + yi) * d.stride[2] +
                        (long long)(xl + xi) * d.stride[3];
  const int p = blockIdx.y, q = d.B - 1 - p;
  typename Word<ES>::type* xp = x + (long long)p * d.s_batch + off;
  typename Word<ES>::type* xq = x + (long long)q * d.s_batch + off;
  const typename Word<ES>::type a = *xp;
  *xp = *xq;
  *xq = a;
}

// ---- labels: one thread per (b, k) of the (B, K) output -------------------------------------------------------------
template <bool ONE_HOT>
__global__ void __launch_bounds__(THREADS)
mix_labels_kernel(pv_mix_label_desc d, const void* __restrict__ labels, void* __restrict__ out, int* __restrict__ flag) {
  const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (i >= (long long)d.B * d.K) return;
  const int b = (int)(i / d.K), k = (int)(i - (long long)b * d.K), b2 = d.B - 1 - b;
  float l1, l2;
  if (ONE_HOT) {
    const float* lab = static_cast<const float*>(labels);
    l1 = lab[(long long)b * d.s_row + (long long)k * d.s_col];
    l2 = lab[(long long)b2 * d.s_row + (long long)k * d.s_col];
  } else {
    const long long* lab = static_cast<const long long*>(labels);
    const long long c1 = lab[(long long)b * d.s_row], c2 = lab[(long long)b2 * d.s_row];
    if (k == 0 && (c1 >= d.K || c1 < 0)) atomicOr(flag, c1 < 0 ? 2 : 1);
    l1 = c1 == k ? d.on : d.off;
    l2 = c2 == k ? d.on : d.off;
  }
  if (d.mode == 2) {
    static_cast<long long*>(out)[i] = (long long)l1;
  } else if (d.mode == 1) {
    static_cast<float*>(out)[i] = l1;
  } else {
    static_cast<float*>(out)[i] = __fadd_rn(__fmul_rn(l1, d.lam), __fmul_rn(l2, d.oml));
  }
}

}  // namespace mix
}  // namespace pv

static int check_mix_desc(const pv_mix_desc* d, const void* x) {
  PV_CHECK_ARG(d != nullptr && x != nullptr, "null argument");
  PV_CHECK_ARG(d->B >= 2 && d->B <= 2 * 65535, "mixing needs 2 .. 131070 clips (got %d)", d->B);
  for (int i = 0; i < 4; ++i) PV_CHECK_ARG(d->size[i] >= 1 && d->stride[i] >= 0, "bad clip dim %d", i);
  PV_CHECK_ARG(d->s_batch >= 0, "bad batch stride");
  return PV_OK;
}

// The clip's dims collapse into one unit-stride run of n elements when some order of them is dense.
static bool dense_clip(const pv_mix_desc* d, long long* n) {
  long long sizes[4], strides[4];
  int m = 0;
  for (int i = 0; i < 4; ++i)
    if (d->size[i] > 1) { sizes[m] = d->size[i]; strides[m] = d->stride[i]; ++m; }
  for (int i = 1; i < m; ++i)          // insertion sort by stride, innermost first
    for (int j = i; j > 0 && strides[j] < strides[j - 1]; --j) {
      long long t = strides[j]; strides[j] = strides[j - 1]; strides[j - 1] = t;
      t = sizes[j]; sizes[j] = sizes[j - 1]; sizes[j - 1] = t;
    }
  long long expect = 1;
  for (int i = 0; i < m; ++i) {
    if (strides[i] != expect) return false;
    expect *= sizes[i];
  }
  *n = expect;
  return true;
}

extern "C" int pv_mixup(const pv_mix_desc* d, void* x, float lam, float oml, void* stream) {
  const int rc = check_mix_desc(d, x);
  if (rc != PV_OK) return rc;
  PV_CHECK_ARG(d->dtype == PV_F32 || d->dtype == PV_F16, "MixUp takes float32 or float16 clips");
  const int es = d->dtype == PV_F32 ? 4 : 2;
  const unsigned pairs = (unsigned)((d->B + 1) / 2);
  cudaStream_t s = (cudaStream_t)stream;
  long long n = 0;
  const bool dense = dense_clip(d, &n);
  if (dense && (n * es) % 16 == 0 && (d->s_batch * es) % 16 == 0 && (uintptr_t)x % 16 == 0) {
    const long long n_vec = n * es / 16;
    const dim3 grid((unsigned)pv::cdiv(n_vec, pv::mix::THREADS), pairs);
    if (d->dtype == PV_F32) {
      pv::mix::mixup_vec_kernel<float><<<grid, pv::mix::THREADS, 0, s>>>(*d, (float*)x, n_vec, lam, oml);
      PV_LAUNCH_OK("mixup_vec_kernel<float>");
    } else {
      pv::mix::mixup_vec_kernel<__half><<<grid, pv::mix::THREADS, 0, s>>>(*d, (__half*)x, n_vec, lam, oml);
      PV_LAUNCH_OK("mixup_vec_kernel<__half>");
    }
    return PV_OK;
  }
  pv_mix_desc g = *d;
  if (dense) {                         // one unit-stride run: skip the per-dim index split
    g.size[0] = g.size[1] = g.size[2] = 1;
    g.size[3] = n;
    g.stride[0] = g.stride[1] = g.stride[2] = 0;
    g.stride[3] = 1;
  }
  const long long total = g.size[0] * g.size[1] * g.size[2] * g.size[3];
  const dim3 grid((unsigned)pv::cdiv(total, pv::mix::THREADS), pairs);
  if (d->dtype == PV_F32) {
    pv::mix::mixup_kernel<float><<<grid, pv::mix::THREADS, 0, s>>>(g, (float*)x, lam, oml);
    PV_LAUNCH_OK("mixup_kernel<float>");
  } else {
    pv::mix::mixup_kernel<__half><<<grid, pv::mix::THREADS, 0, s>>>(g, (__half*)x, lam, oml);
    PV_LAUNCH_OK("mixup_kernel<__half>");
  }
  return PV_OK;
}

extern "C" int pv_cutmix(const pv_mix_desc* d, void* x, int yl, int yh, int xl, int xh, void* stream) {
  const int rc = check_mix_desc(d, x);
  if (rc != PV_OK) return rc;
  PV_CHECK_ARG(0 <= yl && yl <= yh && yh <= d->size[2] && 0 <= xl && xl <= xh && xh <= d->size[3],
               "box [%d:%d, %d:%d] outside the %lld x %lld frame", yl, yh, xl, xh, d->size[2], d->size[3]);
  if (yh == yl || xh == xl) return PV_OK;            // empty box: nothing to swap
  const int bh = yh - yl, bw = xh - xl;
  const long long total = d->size[0] * d->size[1] * bh * bw;
  const dim3 grid((unsigned)pv::cdiv(total, pv::mix::THREADS), (unsigned)(d->B / 2));
  cudaStream_t s = (cudaStream_t)stream;
  switch (d->dtype) {
    case PV_U8:
      pv::mix::cutmix_kernel<1><<<grid, pv::mix::THREADS, 0, s>>>(*d, (uint8_t*)x, yl, xl, bh, bw);
      PV_LAUNCH_OK("cutmix_kernel<1>");
      break;
    case PV_F16:
      pv::mix::cutmix_kernel<2><<<grid, pv::mix::THREADS, 0, s>>>(*d, (uint16_t*)x, yl, xl, bh, bw);
      PV_LAUNCH_OK("cutmix_kernel<2>");
      break;
    case PV_F32:
      pv::mix::cutmix_kernel<4><<<grid, pv::mix::THREADS, 0, s>>>(*d, (uint32_t*)x, yl, xl, bh, bw);
      PV_LAUNCH_OK("cutmix_kernel<4>");
      break;
    default:
      PV_CHECK_ARG(false, "CutMix takes uint8, float16 or float32 clips");
  }
  return PV_OK;
}

extern "C" int pv_mix_labels(const pv_mix_label_desc* d, const void* labels, void* out, int* flag, void* stream) {
  PV_CHECK_ARG(d != nullptr && labels != nullptr && out != nullptr, "null argument");
  PV_CHECK_ARG(d->B >= 1 && d->K >= 1, "empty labels");
  PV_CHECK_ARG(d->mode >= 0 && d->mode <= 2, "bad mode %d", d->mode);
  PV_CHECK_ARG(!d->one_hot || d->mode == 0, "one-hot rows are only mixed");
  PV_CHECK_ARG(d->one_hot || flag != nullptr, "index labels need the range flag");
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = (unsigned)pv::cdiv((long long)d->B * d->K, pv::mix::THREADS);
  if (d->one_hot) {
    pv::mix::mix_labels_kernel<true><<<grid, pv::mix::THREADS, 0, s>>>(*d, labels, out, flag);
    PV_LAUNCH_OK("mix_labels_kernel<onehot>");
  } else {
    PV_CUDA_OK(cudaMemsetAsync(flag, 0, sizeof(int), s));
    pv::mix::mix_labels_kernel<false><<<grid, pv::mix::THREADS, 0, s>>>(*d, labels, out, flag);
    PV_LAUNCH_OK("mix_labels_kernel<index>");
  }
  return PV_OK;
}

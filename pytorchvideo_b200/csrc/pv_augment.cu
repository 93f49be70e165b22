// Video augmentation (RandAugment / AugMix op set, transforms/augmentations.py) on a batch of (T, 3, H, W) clips.
//
// Every op is torchvision's tensor implementation restated per pixel, with torchvision's fp32 operation order and one
// explicit rounding per eager op (__fmul_rn / __fadd_rn, so nvcc cannot contract a multiply-add the CPU does not).
// uint8 clips go through the same float arithmetic as torchvision's uint8 path and end with its cast (truncation
// after _blend, round-half-even after a grid transform).  Ops that need whole-frame statistics (AutoContrast's
// min / max, Equalize's histogram table, AdjustContrast's grayscale mean) read them from augment_stats_kernel.
#include <type_traits>

#include "pv_common.cuh"

namespace pv {
namespace aug {

constexpr int APPLY_THREADS = 256;
constexpr int STATS_THREADS = 512;

template <typename T> __device__ __forceinline__ float ld(const T* p);
template <> __device__ __forceinline__ float ld<uint8_t>(const uint8_t* p) { return (float)__ldg(p); }
template <> __device__ __forceinline__ float ld<float>(const float* p) { return __ldg(p); }

template <typename T> __device__ __forceinline__ void st(T* p, float v);
template <> __device__ __forceinline__ void st<uint8_t>(uint8_t* p, float v) { *p = (uint8_t)(int)v; }
template <> __device__ __forceinline__ void st<float>(float* p, float v) { *p = v; }

// (x * 255).to(torch.uint8) of the reference's float Equalize / Posterize: truncation, low byte
__device__ __forceinline__ int u8_of_unit(float v) { return ((int)__fmul_rn(v, 255.f)) & 0xFF; }

// torchvision rgb_to_grayscale: (0.2989 * r + 0.587 * g + 0.114 * b).to(img.dtype), three eager fp32 ops
template <bool U8> __device__ __forceinline__ float gray(float r, float g, float b) {
  const float l = __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, r), __fmul_rn(0.587f, g)), __fmul_rn(0.114f, b));
  return U8 ? (float)(int)l : l;
}

// torchvision _blend: (ratio * img1 + (1.0 - ratio) * img2).clamp(0, bound).to(img1.dtype)
template <bool U8> __device__ __forceinline__ float blend(float a, float b, float ratio, float omr) {
  float v = __fadd_rn(__fmul_rn(ratio, a), __fmul_rn(omr, b));
  v = fminf(fmaxf(v, 0.f), U8 ? 255.f : 1.f);
  return U8 ? (float)(int)v : v;
}

// ---- statistics: one block per (clip, frame) --------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(STATS_THREADS)
augment_stats_kernel(pv_augment_desc d, const T* __restrict__ src, pv_aug_frame_stats* __restrict__ stats) {
  constexpr bool U8 = std::is_same<T, uint8_t>::value;
  __shared__ int hist[3][256];
  __shared__ float red_mn[3][STATS_THREADS / 32], red_mx[3][STATS_THREADS / 32];
  __shared__ double red_sum[STATS_THREADS / 32];
  const int clip = blockIdx.x / d.T, t = blockIdx.x - clip * d.T;
  for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) (&hist[0][0])[i] = 0;
  __syncthreads();
  const T* base = src + (long long)(clip / d.src_div) * d.s_clip + (long long)t * d.st;
  const int hw = d.H * d.W;
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  double sum = 0.0;
  for (int p = threadIdx.x; p < hw; p += blockDim.x) {
    const int y = p / d.W, x = p - y * d.W;
    const long long off = (long long)y * d.sh + (long long)x * d.sw;
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      v[c] = ld<T>(base + off + c * d.sc);
      mn[c] = fminf(mn[c], v[c]);
      mx[c] = fmaxf(mx[c], v[c]);
      atomicAdd(&hist[c][U8 ? (int)v[c] : u8_of_unit(v[c])], 1);   // integer atomics: order-free
    }
    sum += (double)gray<U8>(v[0], v[1], v[2]);
  }
  // fixed-order reduction: warp butterfly, then warp 0 over the warps' partials
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      mn[c] = fminf(mn[c], __shfl_xor_sync(0xffffffffu, mn[c], o));
      mx[c] = fmaxf(mx[c], __shfl_xor_sync(0xffffffffu, mx[c], o));
    }
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
  }
  if (lane == 0) {
#pragma unroll
    for (int c = 0; c < 3; ++c) { red_mn[c][warp] = mn[c]; red_mx[c][warp] = mx[c]; }
    red_sum[warp] = sum;
  }
  __syncthreads();
  pv_aug_frame_stats* s = stats + blockIdx.x;
  if (threadIdx.x == 0) {
    double total = 0.0;
    for (int w = 0; w < n_warps; ++w) total += red_sum[w];
    s->gray_sum = total;
  }
  if (threadIdx.x < 3) {
    const int c = threadIdx.x;
    float a = INFINITY, b = -INFINITY;
    for (int w = 0; w < n_warps; ++w) { a = fminf(a, red_mn[c][w]); b = fmaxf(b, red_mx[c][w]); }
    s->mn[c] = a;
    s->mx[c] = b;
    // torchvision _scale_channel: step = sum(nonzero_hist[:-1]) // 255; lut = (cumsum + step // 2) // step shifted
    // right by one, clamped to [0, 255]; step == 0 leaves the channel unchanged
    int last = 0;
    for (int i = 0; i < 256; ++i) if (hist[c][i] != 0) last = hist[c][i];
    const int step = (hw - last) / 255;
    if (step == 0) {
      for (int i = 0; i < 256; ++i) s->lut[c][i] = (unsigned char)i;
    } else {
      int cum = 0;
      s->lut[c][0] = 0;
      for (int i = 0; i < 255; ++i) {
        cum += hist[c][i];
        s->lut[c][i + 1] = (unsigned char)min((cum + step / 2) / step, 255);
      }
    }
  }
}

// ---- one op per clip: one thread per pixel, all three channels ----------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(APPLY_THREADS)
augment_apply_kernel(pv_augment_desc d, const T* __restrict__ src, const pv_aug_op* __restrict__ ops,
                     const pv_aug_frame_stats* __restrict__ stats, T* __restrict__ dst) {
  constexpr bool U8 = std::is_same<T, uint8_t>::value;
  constexpr float bound = U8 ? 255.f : 1.f;
  const int hw = d.H * d.W;
  const int p = blockIdx.x * APPLY_THREADS + threadIdx.x;
  if (p >= hw) return;
  const int clip = blockIdx.y / d.T, t = blockIdx.y - clip * d.T;
  const int y = p / d.W, x = p - y * d.W;
  const T* base = src + (long long)(clip / d.src_div) * d.s_clip + (long long)t * d.st;
  T* out = dst + (long long)blockIdx.y * 3 * hw + p;
  const pv_aug_op op = ops[clip];
  auto at = [&](int c, int yy, int xx) { return ld<T>(base + (long long)yy * d.sh + (long long)xx * d.sw + c * d.sc); };
  float v[3], r[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = at(c, y, x);

  switch (op.kind) {
    case PV_AUG_BRIGHTNESS:
#pragma unroll
      for (int c = 0; c < 3; ++c) r[c] = blend<U8>(v[c], 0.f, op.ratio, op.omr);
      break;
    case PV_AUG_CONTRAST: {
      const float mean = (float)(stats[blockIdx.y].gray_sum / (double)hw);
#pragma unroll
      for (int c = 0; c < 3; ++c) r[c] = blend<U8>(v[c], mean, op.ratio, op.omr);
      break;
    }
    case PV_AUG_SATURATION: {
      const float g = gray<U8>(v[0], v[1], v[2]);
#pragma unroll
      for (int c = 0; c < 3; ++c) r[c] = blend<U8>(v[c], g, op.ratio, op.omr);
      break;
    }
    case PV_AUG_SHARPNESS: {
      // 3x3 kernel [[1,1,1],[1,5,1],[1,1,1]] / 13 on interior pixels, border pixels keep their value
      const bool inner = y > 0 && y < d.H - 1 && x > 0 && x < d.W - 1;
      const float k1 = __fdiv_rn(1.f, 13.f), k5 = __fdiv_rn(5.f, 13.f);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float b = v[c];
        if (inner) {
          b = 0.f;
          for (int dy = -1; dy <= 1; ++dy)
            for (int dx = -1; dx <= 1; ++dx)
              b = __fadd_rn(b, __fmul_rn(dy == 0 && dx == 0 ? k5 : k1, dy == 0 && dx == 0 ? v[c] : at(c, y + dy, x + dx)));
          if (U8) b = rintf(b);
        }
        r[c] = blend<U8>(v[c], b, op.ratio, op.omr);
      }
      break;
    }
    case PV_AUG_AUTOCONTRAST: {
      const pv_aug_frame_stats& s = stats[blockIdx.y];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        // torchvision's `bound / (maximum - minimum)` is a scalar over a tensor, which torch evaluates as
        // reciprocal() * bound: two roundings.  One division differs in the last bit for 46 of the 255 uint8 ranges
        // and then maps the frame's maximum to 255.00002 instead of 254.99998 (255 instead of torchvision's 254).
        float lo = s.mn[c], sc = __fmul_rn(__frcp_rn(__fsub_rn(s.mx[c], lo)), bound);
        if (!isfinite(sc)) { lo = 0.f; sc = 1.f; }
        const float q = fminf(fmaxf(__fmul_rn(__fsub_rn(v[c], lo), sc), 0.f), bound);
        r[c] = U8 ? (float)(int)q : q;
      }
      break;
    }
    case PV_AUG_EQUALIZE: {
      const pv_aug_frame_stats& s = stats[blockIdx.y];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float e = (float)s.lut[c][U8 ? (int)v[c] : u8_of_unit(v[c])];
        r[c] = U8 ? e : __fdiv_rn(e, 255.f);
      }
      break;
    }
    case PV_AUG_INVERT:
#pragma unroll
      for (int c = 0; c < 3; ++c) r[c] = __fsub_rn(bound, v[c]);
      break;
    case PV_AUG_POSTERIZE:
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float e = (float)((U8 ? (int)v[c] : u8_of_unit(v[c])) & op.ival);
        r[c] = U8 ? e : __fdiv_rn(e, 255.f);
      }
      break;
    case PV_AUG_SOLARIZE:
#pragma unroll
      for (int c = 0; c < 3; ++c)
        r[c] = (U8 ? v[c] >= (float)op.ival : v[c] >= op.ratio) ? __fsub_rn(bound, v[c]) : v[c];
      break;
    case PV_AUG_AFFINE: {
      // _gen_affine_grid: base (x - W/2 + 0.5, y - H/2 + 0.5, 1) times the rescaled matrix; grid_sample bilinear,
      // zero padding, align_corners=False: ix = (gx + 1) * (W / 2) - 0.5; the appended ones-channel gives the mask
      const float bx = (float)x + (0.5f - 0.5f * (float)d.W), by = (float)y + (0.5f - 0.5f * (float)d.H);
      const float gx = __fadd_rn(__fadd_rn(__fmul_rn(bx, op.theta[0]), __fmul_rn(by, op.theta[1])), op.theta[2]);
      const float gy = __fadd_rn(__fadd_rn(__fmul_rn(bx, op.theta[3]), __fmul_rn(by, op.theta[4])), op.theta[5]);
      const float ix = __fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), 0.5f * (float)d.W), 0.5f);
      const float iy = __fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), 0.5f * (float)d.H), 0.5f);
      float acc[3] = {0.f, 0.f, 0.f}, mask = 0.f;
      if (ix > -1.f && ix < (float)d.W && iy > -1.f && iy < (float)d.H) {   // otherwise no tap is inside
        const float fx = floorf(ix), fy = floorf(iy);
        const int x0 = (int)fx, y0 = (int)fy;
        const float tx = __fsub_rn(ix, fx), ty = __fsub_rn(iy, fy);
        const float ex = __fsub_rn(1.f, tx), sy = __fsub_rn(1.f, ty);
        const float wt[4] = {__fmul_rn(sy, ex), __fmul_rn(sy, tx), __fmul_rn(ty, ex), __fmul_rn(ty, tx)};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int xx = x0 + (k & 1), yy = y0 + (k >> 1);
          const bool in = xx >= 0 && xx < d.W && yy >= 0 && yy < d.H;
#pragma unroll
          for (int c = 0; c < 3; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(in ? at(c, yy, xx) : 0.f, wt[k]));
          mask = __fadd_rn(mask, __fmul_rn(in ? 1.f : 0.f, wt[k]));
        }
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float q = __fadd_rn(__fmul_rn(acc[c], mask), __fmul_rn(__fsub_rn(1.f, mask), op.fill[c]));
        r[c] = U8 ? rintf(q) : q;
      }
      break;
    }
    default:
#pragma unroll
      for (int c = 0; c < 3; ++c) r[c] = v[c];
      break;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) st<T>(out + (long long)c * hw, r[c]);
}

// ---- AugMix: m * x + (1 - m) * sum_k w_k * chain_k, accumulated in chain order ------------------------------------
template <typename T>
__global__ void __launch_bounds__(APPLY_THREADS)
augment_mix_kernel(pv_augment_desc d, const T* __restrict__ src, const T* __restrict__ chains, int width,
                   const float* __restrict__ mix, T* __restrict__ dst) {
  const int hw = d.H * d.W;
  const int e = blockIdx.x * APPLY_THREADS + threadIdx.x;
  if (e >= 3 * hw) return;
  const int clip = blockIdx.y / d.T, t = blockIdx.y - clip * d.T;
  const int c = e / hw, p = e - c * hw, y = p / d.W, x = p - y * d.W;
  const float xv = ld<T>(src + (long long)clip * d.s_clip + (long long)t * d.st + (long long)c * d.sc +
                         (long long)y * d.sh + (long long)x * d.sw);
  const float* w = mix + clip * (width + 2);
  const long long frame = (long long)d.T * 3 * hw;
  float mixed = 0.f;
  for (int k = 0; k < width; ++k)
    mixed = __fadd_rn(mixed, __fmul_rn(__ldg(w + k), ld<T>(chains + (clip * width + k) * frame + (long long)t * 3 * hw + e)));
  const float q = __fadd_rn(__fmul_rn(__ldg(w + width), xv), __fmul_rn(__ldg(w + width + 1), mixed));
  st<T>(dst + (long long)blockIdx.y * 3 * hw + e, q);   // uint8: the reference's truncating .type(torch.uint8)
}

}  // namespace aug
}  // namespace pv

static int check_aug_desc(const pv_augment_desc* d) {
  PV_CHECK_ARG(d != nullptr, "null descriptor");
  PV_CHECK_ARG(d->C == 3, "augmentation needs 3-channel frames (got C=%d)", d->C);
  PV_CHECK_ARG(d->n_clips >= 1 && d->src_div >= 1 && d->T >= 1 && d->H >= 1 && d->W >= 1, "empty clip");
  PV_CHECK_ARG(d->dtype == PV_U8 || d->dtype == PV_F32, "augmentation takes uint8 or float32 clips");
  PV_CHECK_ARG((long long)d->n_clips * d->T <= 65535, "too many frames per launch");
  PV_CHECK_ARG((long long)d->H * d->W * 3 < (1ll << 31), "frame too large");
  return PV_OK;
}

extern "C" int pv_augment_stats(const pv_augment_desc* d, const void* src, pv_aug_frame_stats* stats, void* stream) {
  const int rc = check_aug_desc(d);
  if (rc != PV_OK) return rc;
  PV_CHECK_ARG(src && stats, "null argument");
  const unsigned grid = (unsigned)(d->n_clips * d->T);
  cudaStream_t s = (cudaStream_t)stream;
  if (d->dtype == PV_U8) {
    pv::aug::augment_stats_kernel<uint8_t><<<grid, pv::aug::STATS_THREADS, 0, s>>>(*d, (const uint8_t*)src, stats);
    PV_LAUNCH_OK("augment_stats_kernel<uint8_t>");
  } else {
    pv::aug::augment_stats_kernel<float><<<grid, pv::aug::STATS_THREADS, 0, s>>>(*d, (const float*)src, stats);
    PV_LAUNCH_OK("augment_stats_kernel<float>");
  }
  return PV_OK;
}

extern "C" int pv_augment_apply(const pv_augment_desc* d, const void* src, const pv_aug_op* ops,
                                const pv_aug_frame_stats* stats, void* dst, void* stream) {
  const int rc = check_aug_desc(d);
  if (rc != PV_OK) return rc;
  PV_CHECK_ARG(src && ops && dst, "null argument");
  const dim3 grid((unsigned)pv::cdiv((long long)d->H * d->W, pv::aug::APPLY_THREADS), (unsigned)(d->n_clips * d->T));
  cudaStream_t s = (cudaStream_t)stream;
  if (d->dtype == PV_U8) {
    pv::aug::augment_apply_kernel<uint8_t><<<grid, pv::aug::APPLY_THREADS, 0, s>>>(*d, (const uint8_t*)src, ops, stats,
                                                                                   (uint8_t*)dst);
    PV_LAUNCH_OK("augment_apply_kernel<uint8_t>");
  } else {
    pv::aug::augment_apply_kernel<float><<<grid, pv::aug::APPLY_THREADS, 0, s>>>(*d, (const float*)src, ops, stats,
                                                                                 (float*)dst);
    PV_LAUNCH_OK("augment_apply_kernel<float>");
  }
  return PV_OK;
}

extern "C" int pv_augment_mix(const pv_augment_desc* d, const void* src, const void* chains, int width, const float* mix,
                              void* dst, void* stream) {
  const int rc = check_aug_desc(d);
  if (rc != PV_OK) return rc;
  PV_CHECK_ARG(src && chains && mix && dst && width >= 1, "null argument or width < 1");
  PV_CHECK_ARG(d->src_div == 1, "the mix reads one source clip per output clip");
  const dim3 grid((unsigned)pv::cdiv(3ll * d->H * d->W, pv::aug::APPLY_THREADS), (unsigned)(d->n_clips * d->T));
  cudaStream_t s = (cudaStream_t)stream;
  if (d->dtype == PV_U8) {
    pv::aug::augment_mix_kernel<uint8_t><<<grid, pv::aug::APPLY_THREADS, 0, s>>>(
        *d, (const uint8_t*)src, (const uint8_t*)chains, width, mix, (uint8_t*)dst);
    PV_LAUNCH_OK("augment_mix_kernel<uint8_t>");
  } else {
    pv::aug::augment_mix_kernel<float><<<grid, pv::aug::APPLY_THREADS, 0, s>>>(
        *d, (const float*)src, (const float*)chains, width, mix, (float*)dst);
    PV_LAUNCH_OK("augment_mix_kernel<float>");
  }
  return PV_OK;
}

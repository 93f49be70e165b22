// Contrastive view colour augmentation: ColorJitterVideoSSl of the trainer (torchvision's PIL ColorJitter,
// RandomGrayscale and Pillow's GaussianBlur on the clip stacked into one tall (n_t*H, W) RGB image), for every view of a
// batch in a fixed set of three launches.
//
// The arithmetic is Pillow's, operation by operation, so the bytes are Pillow's:
//   blend (Blend.c)       d + alpha * (x - d) in C float, clipped to [0, 255], truncated; every product and sum is
//                         rounded once (__fmul_rn / __fadd_rn: nvcc may not contract what the CPU computes in two steps)
//   luma (Convert.c)      (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16
//   RGB <-> HSV           rgb2hsv_row / hsv2rgb with their float and double steps (__d*_rn, round half away from zero)
//   box blur (BoxBlur.c)  window sum * ww + the two pixels just outside * fw + 2^23 >> 24 in unsigned 32-bit, edge
//                         pixels repeated; PV_CJ_BLUR_PASSES passes along x, then along the stacked y
// Contrast's degenerate grey is int(mean + 0.5) of the luma of the whole stacked clip as it stands when Contrast runs;
// colorjitter_stats_kernel sums it in integers (order free, so deterministic) and the apply kernel divides in double.
#include "pv_common.cuh"

namespace pv {
namespace cj {

constexpr int STATS_THREADS = 256;
constexpr int STATS_PER_THREAD = 16;
constexpr int APPLY_THREADS = 128;
constexpr int VBLUR_THREADS = 256;
constexpr int VBLUR_SMEM_TARGET = 96 * 1024;    // two strip buffers; the strip narrows until they fit
constexpr int VBLUR_SMEM_MAX = 200 * 1024;

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
__device__ __forceinline__ int clip8(int v) { return v <= 0 ? 0 : (v < 256 ? v : 255); }

// One source element as the byte Pillow sees (ToPILImage truncates in fp32).
template <typename T> __device__ __forceinline__ int src_byte(const T* p, int scale);
template <> __device__ __forceinline__ int src_byte<uint8_t>(const uint8_t* p, int) { return __ldg(p); }
template <> __device__ __forceinline__ int src_byte<float>(const float* p, int scale) {
  float x = __ldg(p);
  if (scale) x = __fdiv_rn(x, 255.f);      // Div255 of a 0..255 float clip
  const float v = __fmul_rn(x, 255.f);
  return v <= 0.f ? 0 : (v >= 255.f ? 255 : (int)v);
}

__device__ __forceinline__ int luma(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

__device__ __forceinline__ int blend(int d, int x, float a) {
  const float v = __fadd_rn((float)d, __fmul_rn(a, (float)(x - d)));
  return (int)fminf(fmaxf(v, 0.f), 255.f);
}

__device__ __forceinline__ void rgb_to_hsv(int r, int g, int b, int& h8, int& s8, int& v8) {
  const int maxc = max(r, max(g, b)), minc = min(r, min(g, b));
  v8 = maxc;
  if (maxc == minc) {
    h8 = 0;
    s8 = 0;
    return;
  }
  const float cr = (float)(maxc - minc);
  const float s = __fdiv_rn(cr, (float)maxc);
  const float rc = __fdiv_rn((float)(maxc - r), cr), gc = __fdiv_rn((float)(maxc - g), cr),
              bc = __fdiv_rn((float)(maxc - b), cr);
  float h;
  if (r == maxc) h = __fadd_rn(bc, -gc);
  else if (g == maxc) h = __double2float_rn(__dadd_rn(__dadd_rn(2.0, (double)rc), -(double)bc));
  else h = __double2float_rn(__dadd_rn(__dadd_rn(4.0, (double)gc), -(double)rc));
  h = __double2float_rn(fmod(__dadd_rn(__ddiv_rn((double)h, 6.0), 1.0), 1.0));
  h8 = clip8((int)__dmul_rn((double)h, 255.0));
  s8 = clip8((int)__dmul_rn((double)s, 255.0));
}

__device__ __forceinline__ void hsv_to_rgb(int h, int s, int v, int& r, int& g, int& b) {
  if (s == 0) {
    r = g = b = v;
    return;
  }
  const double hd = __ddiv_rn(__dmul_rn((double)h, 6.0), 255.0);
  const int i = (int)floor(hd);
  const float f = __double2float_rn(__dadd_rn(hd, -(double)(float)i));
  const float fs = __double2float_rn(__ddiv_rn((double)s, 255.0));
  const double vd = (double)v;
  const int p = clip8((int)round(__dmul_rn(vd, __dadd_rn(1.0, -(double)fs))));
  const int q = clip8((int)round(__dmul_rn(vd, __dadd_rn(1.0, -(double)__fmul_rn(fs, f)))));
  const int t = clip8((int)round(__dmul_rn(vd, __dadd_rn(1.0, -__dmul_rn((double)fs, __dadd_rn(1.0, -(double)f))))));
  switch (i % 6) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

// The view's op ids packed two bits each, first op lowest, so the op loop indexes no local array.
__device__ __forceinline__ unsigned op_code(const pv_cj_view& vw) {
  unsigned code = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) code |= (unsigned)(vw.ops[i] & 3) << (2 * i);
  return code;
}

// The first `stop` ops of `code` on one pixel; `mean` is Contrast's grey level.
__device__ __forceinline__ void jitter_px(int& r, int& g, int& b, const pv_cj_view& vw, unsigned code, int stop,
                                          int mean) {
  for (int i = 0; i < stop; ++i, code >>= 2) {
    const int op = code & 3;
    if (op == 0) {
      const float a = vw.factor[0];
      r = blend(0, r, a); g = blend(0, g, a); b = blend(0, b, a);
    } else if (op == 1) {
      const float a = vw.factor[1];
      r = blend(mean, r, a); g = blend(mean, g, a); b = blend(mean, b, a);
    } else if (op == 2) {
      const float a = vw.factor[2];
      const int l = luma(r, g, b);
      r = blend(l, r, a); g = blend(l, g, a); b = blend(l, b, a);
    } else {
      int h, s, v;
      rgb_to_hsv(r, g, b, h, s, v);
      hsv_to_rgb((h + vw.hue_shift) & 0xFF, s, v, r, g, b);
    }
  }
}

__device__ __forceinline__ int contrast_pos(const pv_cj_view& vw) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (i < vw.n_ops && vw.ops[i] == 1) return i;
  return -1;
}

// One output pixel of a box pass over n samples spaced `stride` bytes apart, edges repeated.
__device__ __forceinline__ uint8_t box_px(const uint8_t* a, int stride, int n, int i, int r, unsigned ww, unsigned fw) {
  unsigned acc = 0;
  for (int k = -r; k <= r; ++k) acc += a[clampi(i + k, 0, n - 1) * stride];
  const unsigned edge = (unsigned)a[clampi(i - r - 1, 0, n - 1) * stride] + a[clampi(i + r + 1, 0, n - 1) * stride];
  return (uint8_t)((acc * ww + edge * fw + (1u << 23)) >> 24);
}

// ---- Contrast's luma sums: blockIdx.y = view, blockIdx.x = a chunk of the stacked clip's pixels -------------------
template <typename T>
__global__ void __launch_bounds__(STATS_THREADS)
colorjitter_stats_kernel(pv_colorjitter_desc d, const T* __restrict__ src, const int32_t* __restrict__ frame_idx,
                         const pv_cj_view* __restrict__ views, unsigned long long* __restrict__ sums) {
  const int k = blockIdx.y;
  const pv_cj_view vw = views[k];
  const int stop = contrast_pos(vw);
  if (stop < 0) return;
  const unsigned code = op_code(vw);
  const long long n_px = (long long)d.n_t * d.H * d.W;
  const T* base = src + (long long)vw.clip * d.s_clip;
  unsigned part = 0;
  const long long p0 = (long long)blockIdx.x * STATS_THREADS * STATS_PER_THREAD + threadIdx.x;
#pragma unroll 4
  for (int j = 0; j < STATS_PER_THREAD; ++j) {
    const long long p = p0 + (long long)j * STATS_THREADS;
    if (p >= n_px) break;
    const int row = (int)(p / d.W), x = (int)(p - (long long)row * d.W);
    const int t = row / d.H, y = row - t * d.H;
    const T* px = base + (long long)__ldg(frame_idx + t) * d.st + (long long)y * d.sh + (long long)x * d.sw;
    int r = src_byte<T>(px, d.src_scale), g = src_byte<T>(px + d.sc, d.src_scale),
        b = src_byte<T>(px + 2 * d.sc, d.src_scale);
    jitter_px(r, g, b, vw, code, stop, 0);
    part += (unsigned)luma(r, g, b);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  __shared__ unsigned warp_sum[STATS_THREADS / 32];
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long s = 0;
    for (int w = 0; w < STATS_THREADS / 32; ++w) s += warp_sum[w];
    if (s) atomicAdd(sums + k, s);      // integer adds: the total does not depend on the order
  }
}

// ---- jitter + grayscale (+ the horizontal blur passes): blockIdx.x = stacked row, blockIdx.y = view ---------------
template <typename T>
__global__ void __launch_bounds__(APPLY_THREADS)
colorjitter_apply_kernel(pv_colorjitter_desc d, const T* __restrict__ src, const int32_t* __restrict__ frame_idx,
                         const pv_cj_view* __restrict__ views, const unsigned long long* __restrict__ sums,
                         uint8_t* __restrict__ dst) {
  extern __shared__ uint8_t row_buf[];      // 2 x [3][W] when the view is blurred
  const int k = blockIdx.y, row = blockIdx.x, W = d.W;
  const pv_cj_view vw = views[k];
  const int t = row / d.H, y = row - t * d.H;
  const long long n_px = (long long)d.n_t * d.H * W;
  int mean = 0;
  if (contrast_pos(vw) >= 0)    // int(ImageStat mean + 0.5): the integer sum divided in double
    mean = (int)__dadd_rn(__ddiv_rn((double)sums[k], (double)n_px), 0.5);
  const T* base = src + (long long)vw.clip * d.s_clip + (long long)__ldg(frame_idx + t) * d.st + (long long)y * d.sh;
  const long long plane = n_px;
  uint8_t* out = dst + (long long)k * 3 * plane + (long long)row * W;
  const bool blur = vw.blur_r >= 0;
  const unsigned code = op_code(vw);
  for (int x = threadIdx.x; x < W; x += APPLY_THREADS) {
    const T* px = base + (long long)x * d.sw;
    int r = src_byte<T>(px, d.src_scale), g = src_byte<T>(px + d.sc, d.src_scale),
        b = src_byte<T>(px + 2 * d.sc, d.src_scale);
    jitter_px(r, g, b, vw, code, vw.n_ops, mean);
    if (vw.gray) r = g = b = luma(r, g, b);
    if (blur) {
      row_buf[x] = (uint8_t)r;
      row_buf[W + x] = (uint8_t)g;
      row_buf[2 * W + x] = (uint8_t)b;
    } else {
      out[x] = (uint8_t)r;
      out[plane + x] = (uint8_t)g;
      out[2 * plane + x] = (uint8_t)b;
    }
  }
  if (!blur) return;
  uint8_t* a = row_buf;
  uint8_t* o = row_buf + 3 * W;
  for (int pass = 0; pass < PV_CJ_BLUR_PASSES; ++pass) {
    __syncthreads();
    for (int e = threadIdx.x; e < 3 * W; e += APPLY_THREADS) {
      const int c = e / W, x = e - c * W;
      o[e] = box_px(a + c * W, 1, W, x, vw.blur_r, vw.blur_ww, vw.blur_fw);
    }
    uint8_t* tmp = a;
    a = o;
    o = tmp;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < 3 * W; e += APPLY_THREADS) {
    const int c = e / W, x = e - c * W;
    out[c * plane + x] = a[e];
  }
}

// ---- vertical blur passes: blockIdx.x = strip of `strip` columns, blockIdx.y = channel, blockIdx.z = view ----------
__global__ void __launch_bounds__(VBLUR_THREADS)
colorjitter_vblur_kernel(pv_colorjitter_desc d, const pv_cj_view* __restrict__ views, int strip,
                         uint8_t* __restrict__ dst) {
  extern __shared__ uint8_t col_buf[];      // 2 x [rows][strip]
  const int k = blockIdx.z;
  const pv_cj_view vw = views[k];
  if (vw.blur_r < 0) return;
  const int rows = d.n_t * d.H, W = d.W;
  const int x0 = blockIdx.x * strip, cols = min(strip, W - x0);
  uint8_t* plane = dst + ((long long)k * 3 + blockIdx.y) * rows * W + x0;
  const int n = rows * strip;
  for (int e = threadIdx.x; e < n; e += VBLUR_THREADS) {
    const int yy = e / strip, c = e - yy * strip;
    if (c < cols) col_buf[e] = plane[(long long)yy * W + c];
  }
  uint8_t* a = col_buf;
  uint8_t* o = col_buf + n;
  for (int pass = 0; pass < PV_CJ_BLUR_PASSES; ++pass) {
    __syncthreads();
    for (int e = threadIdx.x; e < n; e += VBLUR_THREADS) {
      const int yy = e / strip, c = e - yy * strip;
      if (c < cols) o[e] = box_px(a + c, strip, rows, yy, vw.blur_r, vw.blur_ww, vw.blur_fw);
    }
    uint8_t* tmp = a;
    a = o;
    o = tmp;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < n; e += VBLUR_THREADS) {
    const int yy = e / strip, c = e - yy * strip;
    if (c < cols) plane[(long long)yy * W + c] = a[e];
  }
}

// Widest power-of-two strip (<= 32 columns) whose two buffers fit the target; one column may use up to the maximum.
static int vblur_strip(int rows) {
  int s = 32;
  while (s > 1 && 2ll * s * rows > VBLUR_SMEM_TARGET) s >>= 1;
  return s;
}

}  // namespace cj
}  // namespace pv

static int check_cj_desc(const pv_colorjitter_desc* d) {
  PV_CHECK_ARG(d != nullptr, "null descriptor");
  PV_CHECK_ARG(d->n_views >= 1 && d->n_views <= 65535, "n_views must be in 1..65535 (got %d)", d ? d->n_views : 0);
  PV_CHECK_ARG(d->n_t >= 1 && d->H >= 1 && d->W >= 1, "empty clip");
  PV_CHECK_ARG(d->src_dtype == PV_U8 || d->src_dtype == PV_F32, "colour jitter reads uint8 or float32 clips");
  PV_CHECK_ARG(d->src_scale == 0 || d->src_scale == 1, "src_scale must be 0 or 1");
  PV_CHECK_ARG((long long)d->n_t * d->H <= 0x7fffffffll && 6ll * d->W <= 48 * 1024,
               "frame width %d too large for the row buffers", d->W);
  PV_CHECK_ARG((long long)d->n_t * d->H * d->W * 255ll < (1ll << 53), "clip too large");
  return PV_OK;
}

extern "C" int pv_colorjitter_stats(const pv_colorjitter_desc* d, const void* src, const int32_t* frame_idx,
                                    const pv_cj_view* views, unsigned long long* sums, void* stream) {
  const int rc = check_cj_desc(d);
  if (rc != PV_OK) return rc;
  PV_CHECK_ARG(src && frame_idx && views && sums, "null argument");
  cudaStream_t s = (cudaStream_t)stream;
  PV_CUDA_OK(cudaMemsetAsync(sums, 0, sizeof(unsigned long long) * d->n_views, s));
  const long long n_px = (long long)d->n_t * d->H * d->W;
  const long long chunks = pv::cdiv(n_px, (long long)pv::cj::STATS_THREADS * pv::cj::STATS_PER_THREAD);
  PV_CHECK_ARG(chunks <= 0x7fffffffll, "clip too large");
  const dim3 grid((unsigned)chunks, (unsigned)d->n_views);
  if (d->src_dtype == PV_U8) {
    pv::cj::colorjitter_stats_kernel<uint8_t><<<grid, pv::cj::STATS_THREADS, 0, s>>>(*d, (const uint8_t*)src, frame_idx,
                                                                                      views, sums);
    PV_LAUNCH_OK("colorjitter_stats_kernel<uint8_t>");
  } else {
    pv::cj::colorjitter_stats_kernel<float><<<grid, pv::cj::STATS_THREADS, 0, s>>>(*d, (const float*)src, frame_idx,
                                                                                    views, sums);
    PV_LAUNCH_OK("colorjitter_stats_kernel<float>");
  }
  return PV_OK;
}

extern "C" int pv_colorjitter_apply(const pv_colorjitter_desc* d, const void* src, const int32_t* frame_idx,
                                    const pv_cj_view* views, const unsigned long long* sums, uint8_t* dst,
                                    void* stream) {
  const int rc = check_cj_desc(d);
  if (rc != PV_OK) return rc;
  PV_CHECK_ARG(src && frame_idx && views && sums && dst, "null argument");
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid((unsigned)(d->n_t * d->H), (unsigned)d->n_views);
  const size_t smem = 6 * (size_t)d->W;
  if (d->src_dtype == PV_U8) {
    pv::cj::colorjitter_apply_kernel<uint8_t><<<grid, pv::cj::APPLY_THREADS, smem, s>>>(
        *d, (const uint8_t*)src, frame_idx, views, sums, dst);
    PV_LAUNCH_OK("colorjitter_apply_kernel<uint8_t>");
  } else {
    pv::cj::colorjitter_apply_kernel<float><<<grid, pv::cj::APPLY_THREADS, smem, s>>>(
        *d, (const float*)src, frame_idx, views, sums, dst);
    PV_LAUNCH_OK("colorjitter_apply_kernel<float>");
  }
  return PV_OK;
}

extern "C" int pv_colorjitter_vblur(const pv_colorjitter_desc* d, const pv_cj_view* views, uint8_t* dst, void* stream) {
  const int rc = check_cj_desc(d);
  if (rc != PV_OK) return rc;
  PV_CHECK_ARG(views && dst, "null argument");
  const int rows = d->n_t * d->H;
  const int strip = pv::cj::vblur_strip(rows);
  const long long smem = 2ll * strip * rows;
  PV_CHECK_ARG(smem <= pv::cj::VBLUR_SMEM_MAX, "stacked clip of %d rows too tall for the vertical blur", rows);
  if (smem > 48 * 1024)
    PV_CUDA_OK(cudaFuncSetAttribute(pv::cj::colorjitter_vblur_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)smem));
  const dim3 grid((unsigned)pv::cdiv(d->W, strip), 3u, (unsigned)d->n_views);
  pv::cj::colorjitter_vblur_kernel<<<grid, pv::cj::VBLUR_THREADS, (size_t)smem, (cudaStream_t)stream>>>(*d, views, strip,
                                                                                                       dst);
  PV_LAUNCH_OK("colorjitter_vblur_kernel");
  return PV_OK;
}

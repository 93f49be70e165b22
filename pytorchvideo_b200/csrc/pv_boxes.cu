// Box arithmetic of the detection input transforms (transforms/functional.py:195-445: short_side_scale_with_boxes,
// random_crop_with_boxes, uniform_crop_with_boxes, horizontal_flip_with_boxes, clip_boxes_to_image, crop_boxes) on a
// batch of clips with ragged box lists, and the [K, 5] RoI rows the detection heads read.
//
// One thread owns one box.  Every step repeats the reference's expression with one rounding to the boxes' own type T
// per operation, as the eager ops store it: the __*_rn intrinsics keep nvcc from contracting the scale and the crop
// offset into an FMA the CPU does not do.  Clipping is numpy's maximum / minimum (a NaN propagates; max(0, -0) is +0
// here, while numpy leaves that zero's sign to its build).
#include "pv_common.cuh"

namespace pv {
namespace boxes {

constexpr int THREADS = 128;

__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }

// np.minimum(hi, np.maximum(0.0, x)); hi = size - 1.0 is exact in either type
template <typename T> __device__ __forceinline__ T clip1(T x, T hi) {
  if (x != x) return x;
  const T m = (T)0 >= x ? (T)0 : x;
  return hi <= m ? hi : m;
}

template <typename T>
__global__ void __launch_bounds__(THREADS)
clip_boxes_kernel(pv_boxes_desc d, const T* in, const int32_t* __restrict__ box_start,
                  const int32_t* __restrict__ geom, T* out, float* __restrict__ rois) {
  // in == out is allowed (short_side_scale_with_boxes scales in place): each thread reads its box before writing it
  const int k = blockIdx.x * THREADS + threadIdx.x;
  if (k >= d.n_boxes) return;
  int lo = 0, hi = d.n_clips - 1;            // the clip b with box_start[b] <= k < box_start[b + 1]
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(box_start + mid) <= k) lo = mid; else hi = mid - 1;
  }
  const int b = lo;
  int new_h = d.new_h, new_w = d.new_w, top = d.top, left = d.left, hflip = d.hflip;
  if (geom != nullptr) {
    const int32_t* g = geom + b * 6;
    new_h = g[0]; new_w = g[1]; top = g[2]; left = g[3]; hflip = g[4];
  }
  T x1 = in[4 * (long long)k + 0], y1 = in[4 * (long long)k + 1];
  T x2 = in[4 * (long long)k + 2], y2 = in[4 * (long long)k + 3];
  if (d.steps & PV_BOX_CLIP_SRC) {
    const T wm = (T)(d.in_w - 1), hm = (T)(d.in_h - 1);
    x1 = clip1(x1, wm); x2 = clip1(x2, wm); y1 = clip1(y1, hm); y2 = clip1(y2, hm);
  }
  if (d.steps & PV_BOX_SCALE) {
    // boxes *= float(new_h) / h  (w < h) else float(new_w) / w: a double quotient, rounded once to T
    const double f = d.in_w < d.in_h ? (double)new_h / (double)d.in_h : (double)new_w / (double)d.in_w;
    const T ft = (T)f;
    x1 = mul_rn(x1, ft); y1 = mul_rn(y1, ft); x2 = mul_rn(x2, ft); y2 = mul_rn(y2, ft);
  }
  if (d.steps & PV_BOX_CROP) {
    const T ox = (T)left, oy = (T)top;
    x1 = sub_rn(x1, ox); x2 = sub_rn(x2, ox); y1 = sub_rn(y1, oy); y2 = sub_rn(y2, oy);
  }
  const T wm = (T)(d.out_w - 1), hm = (T)(d.out_h - 1);
  if (d.steps & PV_BOX_CLIP_CROP) {
    x1 = clip1(x1, wm); x2 = clip1(x2, wm); y1 = clip1(y1, hm); y2 = clip1(y2, hm);
  }
  if ((d.steps & PV_BOX_FLIP) && hflip) {
    // x1' = width - x2 - 1, x2' = width - x1 - 1: two roundings each, as the reference evaluates them
    const T w = (T)d.out_w, one = (T)1;
    const T nx1 = sub_rn(sub_rn(w, x2), one), nx2 = sub_rn(sub_rn(w, x1), one);
    x1 = nx1; x2 = nx2;
  }
  if (d.steps & PV_BOX_CLIP_OUT) {
    x1 = clip1(x1, wm); x2 = clip1(x2, wm); y1 = clip1(y1, hm); y2 = clip1(y2, hm);
  }
  out[4 * (long long)k + 0] = x1; out[4 * (long long)k + 1] = y1;
  out[4 * (long long)k + 2] = x2; out[4 * (long long)k + 3] = y2;
  if (rois != nullptr) {
    float* r = rois + 5 * (long long)k;
    r[0] = (float)b; r[1] = (float)x1; r[2] = (float)y1; r[3] = (float)x2; r[4] = (float)y2;
  }
}

}  // namespace boxes
}  // namespace pv

extern "C" int pv_clip_boxes_transform(const pv_boxes_desc* d, const void* boxes_in, const int32_t* box_start,
                                       const int32_t* geom, void* boxes_out, float* rois_out, void* stream) {
  PV_CHECK_ARG(d != nullptr, "null descriptor");
  PV_CHECK_ARG(d->n_clips >= 1 && d->n_boxes >= 0, "bad clip / box count (%d clips, %d boxes)", d->n_clips, d->n_boxes);
  PV_CHECK_ARG(d->dtype == PV_BOX_F32 || d->dtype == PV_BOX_F64, "boxes must be float32 or float64 (got %d)", d->dtype);
  PV_CHECK_ARG((d->steps & ~PV_BOX_ALL_STEPS) == 0, "unknown step bits 0x%x", d->steps);
  PV_CHECK_ARG(!(d->steps & (PV_BOX_CLIP_SRC | PV_BOX_SCALE)) || (d->in_h >= 1 && d->in_w >= 1), "bad source frame");
  PV_CHECK_ARG(!(d->steps & (PV_BOX_CLIP_CROP | PV_BOX_FLIP | PV_BOX_CLIP_OUT)) || (d->out_h >= 1 && d->out_w >= 1),
               "bad output frame");
  if (d->n_boxes == 0) return PV_OK;                    // nothing to transform: no launch
  PV_CHECK_ARG(boxes_in != nullptr && box_start != nullptr && boxes_out != nullptr, "null argument");
  const unsigned grid = (unsigned)pv::cdiv(d->n_boxes, pv::boxes::THREADS);
  cudaStream_t s = (cudaStream_t)stream;
  if (d->dtype == PV_BOX_F32) {
    pv::boxes::clip_boxes_kernel<float><<<grid, pv::boxes::THREADS, 0, s>>>(
        *d, (const float*)boxes_in, box_start, geom, (float*)boxes_out, rois_out);
    PV_LAUNCH_OK("clip_boxes_kernel<float>");
  } else {
    pv::boxes::clip_boxes_kernel<double><<<grid, pv::boxes::THREADS, 0, s>>>(
        *d, (const double*)boxes_in, box_start, geom, (double*)boxes_out, rois_out);
    PV_LAUNCH_OK("clip_boxes_kernel<double>");
  }
  return PV_OK;
}

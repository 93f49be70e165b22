// The per-box body shared by clip_boxes_kernel (pv_boxes.cu) and clip_boxes_ragged_kernel (pv_boxes_ragged.cu).
//
// Every step repeats the reference's expression with one rounding to the boxes' own type T per operation, as the
// eager ops store it: the __*_rn intrinsics keep nvcc from contracting the scale and the crop offset into an FMA the
// CPU does not do.  Clipping is numpy's maximum / minimum (a NaN propagates; max(0, -0) is +0 here, while numpy leaves
// that zero's sign to its build).
#pragma once
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

// the clip b with box_start[b] <= k < box_start[b + 1]
__device__ __forceinline__ int clip_of_box(const int32_t* __restrict__ box_start, int n_clips, int k) {
  int lo = 0, hi = n_clips - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(box_start + mid) <= k) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// One clip's geometry as the box steps read it.
struct BoxGeom {
  int in_h, in_w, new_h, new_w, top, left, hflip;
};

// Steps PV_BOX_CLIP_SRC .. PV_BOX_CLIP_OUT of `steps` on one box, in that order.
template <typename T>
__device__ __forceinline__ void box_steps(int steps, const BoxGeom& g, int out_h, int out_w, T& x1, T& y1, T& x2, T& y2) {
  if (steps & PV_BOX_CLIP_SRC) {
    const T wm = (T)(g.in_w - 1), hm = (T)(g.in_h - 1);
    x1 = clip1(x1, wm); x2 = clip1(x2, wm); y1 = clip1(y1, hm); y2 = clip1(y2, hm);
  }
  if (steps & PV_BOX_SCALE) {
    // boxes *= float(new_h) / h  (w < h) else float(new_w) / w: a double quotient, rounded once to T
    const double f = g.in_w < g.in_h ? (double)g.new_h / (double)g.in_h : (double)g.new_w / (double)g.in_w;
    const T ft = (T)f;
    x1 = mul_rn(x1, ft); y1 = mul_rn(y1, ft); x2 = mul_rn(x2, ft); y2 = mul_rn(y2, ft);
  }
  if (steps & PV_BOX_CROP) {
    const T ox = (T)g.left, oy = (T)g.top;
    x1 = sub_rn(x1, ox); x2 = sub_rn(x2, ox); y1 = sub_rn(y1, oy); y2 = sub_rn(y2, oy);
  }
  const T wm = (T)(out_w - 1), hm = (T)(out_h - 1);
  if (steps & PV_BOX_CLIP_CROP) {
    x1 = clip1(x1, wm); x2 = clip1(x2, wm); y1 = clip1(y1, hm); y2 = clip1(y2, hm);
  }
  if ((steps & PV_BOX_FLIP) && g.hflip) {
    // x1' = width - x2 - 1, x2' = width - x1 - 1: two roundings each, as the reference evaluates them
    const T w = (T)out_w, one = (T)1;
    const T nx1 = sub_rn(sub_rn(w, x2), one), nx2 = sub_rn(sub_rn(w, x1), one);
    x1 = nx1; x2 = nx2;
  }
  if (steps & PV_BOX_CLIP_OUT) {
    x1 = clip1(x1, wm); x2 = clip1(x2, wm); y1 = clip1(y1, hm); y2 = clip1(y2, hm);
  }
}

// Box k to out in T and, when rois is set, its fp32 RoI row (b, x1, y1, x2, y2).
template <typename T>
__device__ __forceinline__ void store_box(int k, int b, T x1, T y1, T x2, T y2, T* out, float* __restrict__ rois) {
  out[4 * (long long)k + 0] = x1; out[4 * (long long)k + 1] = y1;
  out[4 * (long long)k + 2] = x2; out[4 * (long long)k + 3] = y2;
  if (rois != nullptr) {
    float* r = rois + 5 * (long long)k;
    r[0] = (float)b; r[1] = (float)x1; r[2] = (float)y1; r[3] = (float)x2; r[4] = (float)y2;
  }
}

}  // namespace boxes
}  // namespace pv

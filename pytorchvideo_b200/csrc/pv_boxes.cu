// Box arithmetic of the detection input transforms (transforms/functional.py:195-445: short_side_scale_with_boxes,
// random_crop_with_boxes, uniform_crop_with_boxes, horizontal_flip_with_boxes, clip_boxes_to_image, crop_boxes) on a
// batch of clips with ragged box lists, and the [K, 5] RoI rows the detection heads read.
//
// One thread owns one box; the per-box steps are box_steps of pv_boxes.cuh.
#include "pv_boxes.cuh"

namespace pv {
namespace boxes {

template <typename T>
__global__ void __launch_bounds__(THREADS)
clip_boxes_kernel(pv_boxes_desc d, const T* in, const int32_t* __restrict__ box_start,
                  const int32_t* __restrict__ geom, T* out, float* __restrict__ rois) {
  // in == out is allowed (short_side_scale_with_boxes scales in place): each thread reads its box before writing it
  const int k = blockIdx.x * THREADS + threadIdx.x;
  if (k >= d.n_boxes) return;
  const int b = clip_of_box(box_start, d.n_clips, k);
  BoxGeom g{d.in_h, d.in_w, d.new_h, d.new_w, d.top, d.left, d.hflip};
  if (geom != nullptr) {
    const int32_t* r = geom + b * 6;
    g.new_h = r[0]; g.new_w = r[1]; g.top = r[2]; g.left = r[3]; g.hflip = r[4];
  }
  T x1 = in[4 * (long long)k + 0], y1 = in[4 * (long long)k + 1];
  T x2 = in[4 * (long long)k + 2], y2 = in[4 * (long long)k + 3];
  box_steps(d.steps, g, d.out_h, d.out_w, x1, y1, x2, y2);
  store_box(k, b, x1, y1, x2, y2, out, rois);
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

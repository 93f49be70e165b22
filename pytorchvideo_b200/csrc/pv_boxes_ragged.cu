// Ragged mode of the box transform (pv_clip_boxes_transform_ragged): every clip of the batch has its own source frame.
// The geometry is the {in_h, in_w, new_h, new_w, top, left, hflip} table pv_clip_transform_ragged reads, so a loader
// uploads one table for a clip launch and a box launch and the two cannot disagree.  One thread owns one box and runs
// PV_BOX_DENORM, then box_steps of pv_boxes.cuh with its clip's source size.
#include "pv_boxes.cuh"

namespace pv {
namespace boxes {

constexpr int RAGGED_GEOM = 7;              // ints per clip row of the ragged geometry table

template <typename T>
__global__ void __launch_bounds__(THREADS)
clip_boxes_ragged_kernel(pv_boxes_desc d, const T* in, const int32_t* __restrict__ box_start,
                         const int32_t* __restrict__ geom, T* out, float* __restrict__ rois) {
  const int k = blockIdx.x * THREADS + threadIdx.x;
  if (k >= d.n_boxes) return;
  const int b = clip_of_box(box_start, d.n_clips, k);
  const int32_t* r = geom + b * RAGGED_GEOM;
  const BoxGeom g{__ldg(r + 0), __ldg(r + 1), __ldg(r + 2), __ldg(r + 3), __ldg(r + 4), __ldg(r + 5), __ldg(r + 6)};
  T x1 = in[4 * (long long)k + 0], y1 = in[4 * (long long)k + 1];
  T x2 = in[4 * (long long)k + 2], y2 = in[4 * (long long)k + 3];
  if (d.steps & PV_BOX_DENORM) {
    // [0, 1] coordinates to source pixels: boxes * tensor([W, H, W, H]), one rounding each
    const T w = (T)g.in_w, h = (T)g.in_h;
    x1 = mul_rn(x1, w); y1 = mul_rn(y1, h); x2 = mul_rn(x2, w); y2 = mul_rn(y2, h);
  }
  box_steps(d.steps, g, d.out_h, d.out_w, x1, y1, x2, y2);
  store_box(k, b, x1, y1, x2, y2, out, rois);
}

}  // namespace boxes
}  // namespace pv

extern "C" int pv_clip_boxes_transform_ragged(const pv_boxes_desc* d, const void* boxes_in, const int32_t* box_start,
                                              const int32_t* geom, const int32_t* geom_host, void* boxes_out,
                                              float* rois_out, void* stream) {
  PV_CHECK_ARG(d != nullptr && geom != nullptr && geom_host != nullptr, "null argument");
  PV_CHECK_ARG(d->n_clips >= 1 && d->n_boxes >= 0, "bad clip / box count (%d clips, %d boxes)", d->n_clips, d->n_boxes);
  PV_CHECK_ARG(d->dtype == PV_BOX_F32 || d->dtype == PV_BOX_F64, "boxes must be float32 or float64 (got %d)", d->dtype);
  PV_CHECK_ARG((d->steps & ~(PV_BOX_ALL_STEPS | PV_BOX_DENORM)) == 0, "unknown step bits 0x%x", d->steps);
  PV_CHECK_ARG(d->out_h >= 1 && d->out_w >= 1, "bad output frame");
  for (int b = 0; b < d->n_clips; ++b) {
    const int32_t* g = geom_host + pv::boxes::RAGGED_GEOM * b;
    PV_CHECK_ARG(g[0] >= 1 && g[1] >= 1 && g[2] >= 1 && g[3] >= 1, "clip %d: bad frame size", b);
    PV_CHECK_ARG(g[4] >= 0 && g[5] >= 0 && (long long)g[4] + d->out_h <= g[2] && (long long)g[5] + d->out_w <= g[3],
                 "clip %d: crop window outside the resized frame", b);
  }
  if (d->n_boxes == 0) return PV_OK;                    // nothing to transform: no launch
  PV_CHECK_ARG(boxes_in != nullptr && box_start != nullptr && boxes_out != nullptr, "null argument");
  const unsigned grid = (unsigned)pv::cdiv(d->n_boxes, pv::boxes::THREADS);
  cudaStream_t s = (cudaStream_t)stream;
  if (d->dtype == PV_BOX_F32) {
    pv::boxes::clip_boxes_ragged_kernel<float><<<grid, pv::boxes::THREADS, 0, s>>>(
        *d, (const float*)boxes_in, box_start, geom, (float*)boxes_out, rois_out);
    PV_LAUNCH_OK("clip_boxes_ragged_kernel<float>");
  } else {
    pv::boxes::clip_boxes_ragged_kernel<double><<<grid, pv::boxes::THREADS, 0, s>>>(
        *d, (const double*)boxes_in, box_start, geom, (double*)boxes_out, rois_out);
    PV_LAUNCH_OK("clip_boxes_ragged_kernel<double>");
  }
  return PV_OK;
}

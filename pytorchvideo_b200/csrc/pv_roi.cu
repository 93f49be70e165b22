// RoIAlign on channels-last feature maps for the detection heads (models/head.py:441-482 ResNetRoIHead:
// pool -> squeeze T -> roi_layer(x, bboxes) -> pool_spatial -> ... ; the reference's roi_layer is
// torchvision.ops.RoIAlign(output_size, spatial_scale, sampling_ratio), aligned=False).
//
// HBM/L2-bound gather: one CTA per (roi, output bin), threads over channel groups of 8 (one 16-byte vector per tap).
// The sampling grid, the bilinear weights and their boundary rules follow torchvision's roi_align exactly
// (csrc/ops/cpu/roi_align_common.h pre_calc_for_bilinear_interpolate):
//   roi_start = box * spatial_scale;  roi_size = max(roi_end - roi_start, 1);  bin = roi_size / pooled
//   grid = sampling_ratio > 0 ? sampling_ratio : ceil(roi_size / pooled);  count = max(grid_h * grid_w, 1)
//   sample (iy, ix): y = roi_start_h + ph * bin_h + (iy + .5) * bin_h / grid_h  (x alike)
//   outside [-1, H] x [-1, W] -> contributes 0;  y <= 0 -> 0;  y_low >= H-1 -> y_low = y_high = H-1, y = y_low
//   value = w1*v1 + w2*v2 + w3*v3 + w4*v4 summed in sample order (iy outer, ix inner), divided by count
// all in fp32 (the stored result is rounded once to the plan's storage type).
// The geometry (roi sizes, bin sizes, grid counts, sample positions) is written with explicitly rounded intrinsics:
// nvcc would otherwise contract `end * scale - start` and `start + ph * bin` into FMAs, which moves a sample by an
// ulp - enough to switch it across the -1 / H cutoffs or change ceil(roi / pooled) at a non-power-of-two scale.
// With the intrinsics the positions, indices and weights are bit-identical to torchvision's fp32 arithmetic.
#include "pv_common.cuh"

namespace pv {

template <typename T>
__global__ void __launch_bounds__(256)
roi_align_kernel(const T* __restrict__ x, const float* __restrict__ rois, T* __restrict__ y, int N, int H, int W,
                 int C, long long x_row_stride, long long y_row_stride, int K, int ph_n, int pw_n,
                 float spatial_scale, int sampling_ratio) {
  const int bin = blockIdx.x;                 // (roi, ph, pw)
  const int pw = bin % pw_n;
  const int ph = (bin / pw_n) % ph_n;
  const int k = bin / (pw_n * ph_n);
  const float* r = rois + (long long)k * 5;
  const int n = (int)__ldg(r);
  const float roi_start_w = __fmul_rn(__ldg(r + 1), spatial_scale), roi_start_h = __fmul_rn(__ldg(r + 2), spatial_scale);
  const float roi_end_w = __fmul_rn(__ldg(r + 3), spatial_scale), roi_end_h = __fmul_rn(__ldg(r + 4), spatial_scale);
  const float roi_w = fmaxf(__fsub_rn(roi_end_w, roi_start_w), 1.f), roi_h = fmaxf(__fsub_rn(roi_end_h, roi_start_h), 1.f);
  const float bin_h = __fdiv_rn(roi_h, (float)ph_n), bin_w = __fdiv_rn(roi_w, (float)pw_n);
  const int grid_h = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(__fdiv_rn(roi_h, (float)ph_n));
  const int grid_w = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(__fdiv_rn(roi_w, (float)pw_n));
  const float start_y = __fadd_rn(roi_start_h, __fmul_rn((float)ph, bin_h));   // torchvision: start + ph * bin
  const float start_x = __fadd_rn(roi_start_w, __fmul_rn((float)pw, bin_w));
  const float count = (float)max(grid_h * grid_w, 1);
  const bool valid_n = n >= 0 && n < N;
  const T* xn = x + (long long)(valid_n ? n : 0) * H * W * x_row_stride;
  T* yo = y + (long long)bin * y_row_stride;
  for (int c = threadIdx.x * 8; c < C; c += blockDim.x * 8) {
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int iy = 0; iy < grid_h; ++iy) {
      const float yy0 = __fadd_rn(start_y, __fdiv_rn(__fmul_rn((float)iy + .5f, bin_h), (float)grid_h));
      for (int ix = 0; ix < grid_w; ++ix) {
        const float xx0 = __fadd_rn(start_x, __fdiv_rn(__fmul_rn((float)ix + .5f, bin_w), (float)grid_w));
        float yy = yy0, xx = xx0;
        if (!valid_n || yy < -1.f || yy > (float)H || xx < -1.f || xx > (float)W) continue;   // zero weights
        if (yy <= 0.f) yy = 0.f;
        if (xx <= 0.f) xx = 0.f;
        int y_low = (int)yy, x_low = (int)xx, y_high, x_high;
        if (y_low >= H - 1) { y_high = y_low = H - 1; yy = (float)y_low; } else y_high = y_low + 1;
        if (x_low >= W - 1) { x_high = x_low = W - 1; xx = (float)x_low; } else x_high = x_low + 1;
        const float ly = yy - (float)y_low, lx = xx - (float)x_low, hy = 1.f - ly, hx = 1.f - lx;
        const float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
        float v1[8], v2[8], v3[8], v4[8];
        ld8<T>(xn + ((long long)y_low * W + x_low) * x_row_stride + c, v1);
        ld8<T>(xn + ((long long)y_low * W + x_high) * x_row_stride + c, v2);
        ld8<T>(xn + ((long long)y_high * W + x_low) * x_row_stride + c, v3);
        ld8<T>(xn + ((long long)y_high * W + x_high) * x_row_stride + c, v4);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += w1 * v1[i] + w2 * v2[i] + w3 * v3[i] + w4 * v4[i];
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = acc[i] / count;
    st8<T>(yo + c, acc);
  }
}

}  // namespace pv

// x: NDHWC features with T == 1, i.e. [N][H][W][C] rows of x_row_stride elements (C % 8 == 0, padded lanes zero);
// rois: DEVICE fp32 [K][5] = (batch index, x1, y1, x2, y2) in input-image pixels (torchvision's Tensor[K,5] format);
// y: [K][pooled_h][pooled_w][C] rows of y_row_stride elements.
extern "C" int pv_roi_align_fwd(const void* x, int dtype, long long x_row_stride, int N, int H, int W, int C,
                                const float* rois, int K, int pooled_h, int pooled_w, float spatial_scale,
                                int sampling_ratio, void* y, long long y_row_stride, void* stream) {
  PV_CHECK_ARG(x && rois && y, "null argument");
  PV_CHECK_ARG(dtype == PV_F16 || dtype == PV_F32, "dtype must be f16|f32");
  PV_CHECK_ARG(N >= 1 && H >= 1 && W >= 1 && C >= 8 && C % 8 == 0, "bad feature map (C must be a multiple of 8)");
  PV_CHECK_ARG(K >= 1 && pooled_h >= 1 && pooled_w >= 1, "empty output");
  PV_CHECK_ARG(x_row_stride >= C && y_row_stride >= C && x_row_stride % 8 == 0 && y_row_stride % 8 == 0, "bad row strides");
  PV_CHECK_ARG((long long)K * pooled_h * pooled_w <= 0x7fffffffll, "too many bins");
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned bins = (unsigned)((long long)K * pooled_h * pooled_w);
  int threads = ((C / 8 + 31) / 32) * 32;
  if (threads > 256) threads = 256;
  if (dtype == PV_F16) {
    pv::roi_align_kernel<__half><<<bins, threads, 0, s>>>((const __half*)x, rois, (__half*)y, N, H, W, C, x_row_stride,
                                                         y_row_stride, K, pooled_h, pooled_w, spatial_scale, sampling_ratio);
    PV_LAUNCH_OK("roi_align_kernel<__half>");
  } else {
    pv::roi_align_kernel<float><<<bins, threads, 0, s>>>((const float*)x, rois, (float*)y, N, H, W, C, x_row_stride,
                                                        y_row_stride, K, pooled_h, pooled_w, spatial_scale, sampling_ratio);
    PV_LAUNCH_OK("roi_align_kernel<float>");
  }
  return PV_OK;
}

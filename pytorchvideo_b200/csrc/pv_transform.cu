// Fused clip transform: temporal gather + /255 + normalize + bilinear resize + crop in ONE pass.
// HBM-bound byte work: every output pixel reads exactly its 2x2 uint8 taps and writes one
// f16/f32 value; nothing full-resolution is ever materialised (the reference materialises two
// fp32 full-resolution copies, transforms/functional.py:604-615 and transforms.py:187-195).
#include "pv_common.cuh"

namespace pv {

// One thread produces PX horizontally adjacent outputs of one (c, frame, row).
// grid = (ceil(out_w / (PX*128)), out_h, C * n_t);   block = 128
template <typename T> __device__ __forceinline__ float ld_src(const T* p);
template <> __device__ __forceinline__ float ld_src<uint8_t>(const uint8_t* p) { return (float)__ldg(p); }
template <> __device__ __forceinline__ float ld_src<float>(const float* p) { return __ldg(p); }
template <> __device__ __forceinline__ float ld_src<__half>(const __half* p) { return __half2float(__ldg(p)); }

template <typename SrcT, typename OutT, int PX>
__global__ void __launch_bounds__(128)
clip_transform_kernel(pv_clip_transform_desc d, const SrcT* __restrict__ src,
                      const int32_t* __restrict__ idx_t, const int32_t* __restrict__ y0t,
                      const int32_t* __restrict__ y1t, const float* __restrict__ lyt,
                      const int32_t* __restrict__ x0t, const int32_t* __restrict__ x1t,
                      const float* __restrict__ lxt, OutT* __restrict__ dst) {
  const int y = blockIdx.y;
  const int ct = blockIdx.z;
  const int c = ct / d.n_t, j = ct - c * d.n_t;
  const int xb = (blockIdx.x * blockDim.x + threadIdx.x) * PX;
  if (xb >= d.out_w) return;

  const long long frame = (long long)c * d.sc + (long long)__ldg(idx_t + j) * d.st;
  const SrcT* r0 = src + frame + (long long)__ldg(y0t + y) * d.sh;
  const SrcT* r1 = src + frame + (long long)__ldg(y1t + y) * d.sh;
  const float ly1 = __ldg(lyt + y), ly0 = 1.f - ly1;
  const float mean = d.mean[c], stdv = d.stdv[c];

  float out[PX];
#pragma unroll
  for (int i = 0; i < PX; ++i) {
    const int x = min(xb + i, d.out_w - 1);
    const long long xa = (long long)__ldg(x0t + x) * d.sw, xc = (long long)__ldg(x1t + x) * d.sw;
    const float lx1 = __ldg(lxt + x), lx0 = 1.f - lx1;
    float v00 = ld_src<SrcT>(r0 + xa), v01 = ld_src<SrcT>(r0 + xc);
    float v10 = ld_src<SrcT>(r1 + xa), v11 = ld_src<SrcT>(r1 + xc);
    if (d.div255) {   // same op order as the reference: x/255.0 then (x-mean)/std, all fp32
      v00 = v00 / 255.0f; v01 = v01 / 255.0f; v10 = v10 / 255.0f; v11 = v11 / 255.0f;
    }
    v00 = (v00 - mean) / stdv; v01 = (v01 - mean) / stdv;
    v10 = (v10 - mean) / stdv; v11 = (v11 - mean) / stdv;
    // ATen upsample_bilinear2d: l_h0*(l_w0*v00 + l_w1*v01) + l_h1*(l_w0*v10 + l_w1*v11)
    out[i] = ly0 * (lx0 * v00 + lx1 * v01) + ly1 * (lx0 * v10 + lx1 * v11);
  }
  OutT* o = dst + (((long long)ct * d.out_h + y) * d.out_w + xb);
  if (PX == 2 && xb + 1 < d.out_w && ((reinterpret_cast<uintptr_t>(o) & (2 * sizeof(OutT) - 1)) == 0)) {
    if constexpr (sizeof(OutT) == 2) {
      *reinterpret_cast<__half2*>(o) = __floats2half2_rn(out[0], out[PX - 1]);
    } else {
      *reinterpret_cast<float2*>(o) = make_float2(out[0], out[PX - 1]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < PX; ++i)
      if (xb + i < d.out_w) Elem<OutT>::st(o + i, out[i]);
  }
}


// ---------------------------------------------------------------------------------------------------------------
// Batched chain (pv_clip_transform_batch): ONE launch over a batch of clips, no tap tables.
//   * the bilinear taps are computed in the kernel with ATen's own arithmetic
//       scale = float(in) / float(out);  src = fma(scale, dst + 0.5, -0.5);  src = max(src, 0)
//       i0 = min(floor(src), in - 1);  l1 = clamp(src - i0, 0, 1);  i1 = i0 + (i0 < in - 1)
//     (area_pixel_compute_source_index / guard_index_and_lambda; bit-equal to the host tables of the
//     single-clip entry point, tests/test_gpu_transforms.py), so a thread has no dependent table loads;
//   * a thread produces PX = 2 adjacent output columns of one (clip, frame, row) for ALL channels: up to
//     24 independent byte loads in flight, the tap arithmetic shared by the channels;
//   * optional per-clip geometry (random short side, crop window, horizontal flip: the train chain on a batch;
//     plus a first-frame offset: the 3 spatial x K temporal test-time views of ONE video are a batch whose
//     clip stride is 0);
//   * optional second output = the SlowFast slow pathway (frames slow_pos[j] >= 0 of the kept frames,
//     pytorchvideo_trainer datamodule/transforms.py:129-136), written from the same registers;
//   * uint8 destination for pure frame selection / cropping (UniformTemporalSubsample keeps the dtype).
// grid = (1, ceil(out_h / TB_ROWS), n_clips * n_t);  block = (min(out_w/2, 256), 256 / that)
// ---------------------------------------------------------------------------------------------------------------
struct TapXY {
  int i0, i1;
  float l1;
};
__device__ __forceinline__ float bilinear_scale(int in_size, int out_size) {
  return __fdiv_rn((float)in_size, (float)out_size);
}
__device__ __forceinline__ TapXY bilinear_tap(int dst, int in_size, float scale) {
  float src = __fmaf_rn(scale, (float)dst + 0.5f, -0.5f);
  src = fmaxf(src, 0.f);
  TapXY t;
  t.i0 = min((int)floorf(src), in_size - 1);
  t.l1 = fminf(fmaxf(src - (float)t.i0, 0.f), 1.f);
  t.i1 = t.i0 + (t.i0 < in_size - 1 ? 1 : 0);
  return t;
}
template <typename T> __device__ __forceinline__ void st_out(T* p, float v);
template <> __device__ __forceinline__ void st_out<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void st_out<__half>(__half* p, float v) { *p = __float2half_rn(v); }
template <> __device__ __forceinline__ void st_out<uint8_t>(uint8_t* p, float v) { *p = (uint8_t)v; }   // pass-through only
// two adjacent outputs: one vector store when the address allows it
template <typename T> __device__ __forceinline__ void st_out2(T* p, float a, float b, bool two) {
  if (two && (reinterpret_cast<uintptr_t>(p) & (2 * sizeof(T) - 1)) == 0) {
    if constexpr (sizeof(T) == 2) *reinterpret_cast<__half2*>(p) = __floats2half2_rn(a, b);
    else if constexpr (sizeof(T) == 4) *reinterpret_cast<float2*>(p) = make_float2(a, b);
    else *reinterpret_cast<uchar2*>(p) = make_uchar2((unsigned char)a, (unsigned char)b);
  } else {
    st_out<T>(p, a);
    if (two) st_out<T>(p + 1, b);
  }
}

// Round-2 rework after the ncu capture showed the first version ISSUE-bound, not HBM-bound (48 IEEE fp32 divisions per
// thread for `x/255` and `(x-mean)/std`): a uint8 source has only 256 possible values per channel, so a block first
// builds the value table lut[c][u] = ((float)u / 255 - mean[c]) / std[c] in shared memory with the reference's own
// operations (bit-exact by construction) and a tap becomes one LDS.  A block of 256 threads covers TB_ROWS output
// rows of one (clip, frame) so the table costs ~0.4 divisions per output instead of 8.
constexpr int TB_ROWS = 8;
constexpr int TB_THREADS = 256;

// RRC (RandomResizedCrop mode, pv_clip_transform_rrc): geom holds one {top, left, h, w, hflip} source window per
// (clip, kept frame); the taps are ATen's for an h x w -> out_h x out_w resize, offset by the window origin.
// Ragged mode (pv_clip_transform_ragged), selected at run time by a non-null frame_off: kept frame j of clip b is a
// packed HWC frame at src + frame_off[b * n_t + j], and geom holds {in_h, in_w, new_h, new_w, top, left, hflip} per clip.
template <typename SrcT, typename OutT, int NC, bool LUT, bool RRC>
__device__ __forceinline__ void
clip_transform_batch_body(const pv_clip_batch_desc& d, const SrcT* __restrict__ src, const int32_t* __restrict__ idx_t,
                          const int32_t* __restrict__ slow_pos, const int32_t* __restrict__ geom,
                          const long long* __restrict__ frame_off, OutT* __restrict__ dst, OutT* __restrict__ dst_slow) {
  constexpr int PX = 2;
  __shared__ float lut[LUT ? NC * 256 : 1];
  if constexpr (LUT) {
    for (int e = threadIdx.y * blockDim.x + threadIdx.x; e < NC * 256; e += blockDim.x * blockDim.y) {
      const int c = e >> 8;
      float v = (float)(e & 255);
      if (d.div255) v = v / 255.0f;                        // reference op order, fp32
      if (d.normalize) v = (v - d.mean[c]) / d.stdv[c];
      lut[e] = v;
    }
    __syncthreads();
  }
  const int clip = blockIdx.z / d.n_t, j = blockIdx.z - clip * d.n_t;
  int new_h = d.new_h, new_w = d.new_w, top = d.top, left = d.left, flip = d.hflip;
  int t_off = 0;
  int win_h = 0, win_w = 0;                 // RRC source window size
  int in_h = d.in_h, in_w = d.in_w;
  unsigned sh = (unsigned)d.sh, sw = (unsigned)d.sw;
  if constexpr (RRC) {          // per-(clip, frame) source window
    const int32_t* g = geom + 5 * blockIdx.z;
    top = __ldg(g); left = __ldg(g + 1); win_h = __ldg(g + 2); win_w = __ldg(g + 3); flip = __ldg(g + 4);
    new_h = d.out_h; new_w = d.out_w;
  } else if (frame_off != nullptr) {   // ragged: per-clip source size and geometry, packed HWC frames
    const int32_t* g = geom + 7 * clip;
    in_h = __ldg(g); in_w = __ldg(g + 1); new_h = __ldg(g + 2); new_w = __ldg(g + 3);
    top = __ldg(g + 4); left = __ldg(g + 5); flip = __ldg(g + 6);
    sw = NC; sh = (unsigned)(NC * in_w);
  } else if (geom != nullptr) {        // per-clip (new_h, new_w, top, left, hflip, first frame)
    const int32_t* g = geom + 6 * clip;
    new_h = __ldg(g); new_w = __ldg(g + 1); top = __ldg(g + 2); left = __ldg(g + 3); flip = __ldg(g + 4);
    t_off = __ldg(g + 5);
  }
  // block-uniform channel planes of this (clip, frame); everything per thread below is a 32-bit offset into them
  // (the host checks in_h*|sh| + in_w*|sw| < 2^31, and in_h*in_w*NC < 2^31 for a ragged frame)
  const SrcT* cbase[NC];
  const SrcT* fbase = frame_off != nullptr ? src + __ldg(frame_off + blockIdx.z)
                                           : src + (long long)clip * d.s_clip + (long long)(__ldg(idx_t + j) + t_off) * d.st;
#pragma unroll
  for (int c = 0; c < NC; ++c) cbase[c] = fbase + (frame_off != nullptr ? (long long)c : (long long)c * d.sc);
  const int sp = slow_pos != nullptr ? __ldg(slow_pos + j) : -1;
  const int half_w = (d.out_w + PX - 1) / PX;
  const int y_base = blockIdx.y * TB_ROWS;
  const int n_rows = min(TB_ROWS, d.out_h - y_base);
  const int plane = d.out_h * d.out_w;                 // host checks C*n_t*plane < 2^31
  const float scale_y = RRC ? bilinear_scale(win_h, new_h) : bilinear_scale(in_h, new_h);
  const float scale_x = RRC ? bilinear_scale(win_w, new_w) : bilinear_scale(in_w, new_w);
  OutT* const dclip = dst + (long long)clip * d.d_clip + (long long)j * plane;
  OutT* const sclip = sp >= 0 ? dst_slow + (long long)clip * d.d_slow_clip + (long long)sp * plane : nullptr;
  const int cstep = d.n_t * plane, cstep_slow = d.n_slow * plane;

  // blockDim = (bx, by): x pairs along threadIdx.x, rows interleaved along threadIdx.y; the column taps are
  // computed once per thread and reused by its rows
  for (int xi = threadIdx.x; xi < half_w; xi += blockDim.x) {
    const int xb = xi * PX;
    unsigned xo0[PX], xo1[PX];
    float lx0[PX], lx1[PX];
#pragma unroll
    for (int i = 0; i < PX; ++i) {
      const int xo = min(xb + i, d.out_w - 1);
      if constexpr (RRC) {      // taps relative to the window, then its origin
        const TapXY t = bilinear_tap(flip ? d.out_w - 1 - xo : xo, win_w, scale_x);
        xo0[i] = (left + t.i0) * sw; xo1[i] = (left + t.i1) * sw;
        lx1[i] = t.l1; lx0[i] = 1.f - t.l1;
        continue;
      }
      const TapXY t = bilinear_tap(left + (flip ? d.out_w - 1 - xo : xo), in_w, scale_x);
      xo0[i] = t.i0 * sw; xo1[i] = t.i1 * sw;
      lx1[i] = t.l1; lx0[i] = 1.f - t.l1;
    }
    const bool two = (xb + 1 < d.out_w);
    for (int r = threadIdx.y; r < n_rows; r += blockDim.y) {
      const int y = y_base + r;
      const TapXY ty = RRC ? bilinear_tap(y, win_h, scale_y) : bilinear_tap(top + y, in_h, scale_y);
      const float ly1 = ty.l1, ly0 = 1.f - ly1;
      const unsigned ro0 = ((RRC ? top : 0) + ty.i0) * sh, ro1 = ((RRC ? top : 0) + ty.i1) * sh;
      unsigned off[PX][4];
#pragma unroll
      for (int i = 0; i < PX; ++i) {
        off[i][0] = ro0 + xo0[i]; off[i][1] = ro0 + xo1[i];
        off[i][2] = ro1 + xo0[i]; off[i][3] = ro1 + xo1[i];
      }
      // all loads first (independent), then the arithmetic
      float v[NC][PX][4];
      if constexpr (LUT) {
        unsigned u[NC][PX][4];
#pragma unroll
        for (int c = 0; c < NC; ++c)
#pragma unroll
          for (int i = 0; i < PX; ++i)
#pragma unroll
            for (int k = 0; k < 4; ++k) u[c][i][k] = __ldg(cbase[c] + off[i][k]);
#pragma unroll
        for (int c = 0; c < NC; ++c)
#pragma unroll
          for (int i = 0; i < PX; ++i)
#pragma unroll
            for (int k = 0; k < 4; ++k) v[c][i][k] = lut[c * 256 + u[c][i][k]];
      } else {
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          const float mean = d.mean[c], stdv = d.stdv[c];
#pragma unroll
          for (int i = 0; i < PX; ++i)
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              float t = ld_src<SrcT>(cbase[c] + off[i][k]);
              if (d.div255) t = t / 255.0f;
              if (d.normalize) t = (t - mean) / stdv;
              v[c][i][k] = t;
            }
        }
      }
      const int pix = y * d.out_w + xb;
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        float out[PX];
#pragma unroll
        for (int i = 0; i < PX; ++i)
          out[i] = ly0 * (lx0[i] * v[c][i][0] + lx1[i] * v[c][i][1]) + ly1 * (lx0[i] * v[c][i][2] + lx1[i] * v[c][i][3]);
        st_out2<OutT>(dclip + (c * cstep + pix), out[0], out[1], two);
        if (sp >= 0) st_out2<OutT>(sclip + (c * cstep_slow + pix), out[0], out[1], two);
      }
    }
  }
}

template <typename SrcT, typename OutT, int NC, bool LUT>
__global__ void __launch_bounds__(TB_THREADS)
clip_transform_batch_kernel(pv_clip_batch_desc d, const SrcT* __restrict__ src, const int32_t* __restrict__ idx_t,
                            const int32_t* __restrict__ slow_pos, const int32_t* __restrict__ geom,
                            const long long* __restrict__ frame_off, OutT* __restrict__ dst, OutT* __restrict__ dst_slow) {
  clip_transform_batch_body<SrcT, OutT, NC, LUT, false>(d, src, idx_t, slow_pos, geom, frame_off, dst, dst_slow);
}

template <typename SrcT, typename OutT, bool LUT>
__global__ void __launch_bounds__(TB_THREADS)
clip_transform_rrc_kernel(pv_clip_batch_desc d, const SrcT* __restrict__ src, const int32_t* __restrict__ idx_t,
                          const int32_t* __restrict__ boxes, OutT* __restrict__ dst) {
  clip_transform_batch_body<SrcT, OutT, 3, LUT, true>(d, src, idx_t, nullptr, boxes, nullptr, dst, nullptr);
}

}  // namespace pv

extern "C" int pv_clip_transform_fwd(const pv_clip_transform_desc* d, const void* src,
                                     const int32_t* idx_t, const int32_t* y0, const int32_t* y1,
                                     const float* ly, const int32_t* x0, const int32_t* x1,
                                     const float* lx, void* dst, void* stream) {
  PV_CHECK_ARG(d && src && idx_t && y0 && y1 && ly && x0 && x1 && lx && dst, "null argument");
  PV_CHECK_ARG(d->C >= 1 && d->C <= 4, "C must be in 1..4 (got %d)", d->C);
  PV_CHECK_ARG(d->n_t >= 1 && d->out_h >= 1 && d->out_w >= 1, "empty output");
  PV_CHECK_ARG(d->out_h <= 65535 && (long long)d->C * d->n_t <= 65535, "grid too large");
  PV_CHECK_ARG(d->dst_dtype == PV_F16 || d->dst_dtype == PV_F32, "dst dtype must be f16|f32");
  cudaStream_t s = (cudaStream_t)stream;
  constexpr int PX = 2;
  dim3 grid((unsigned)pv::cdiv(d->out_w, PX * 128), d->out_h, d->C * d->n_t), block(128);
#define PV_TR(ST, OT)                                                                                     \
  do {                                                                                                    \
    pv::clip_transform_kernel<ST, OT, PX><<<grid, block, 0, s>>>(*d, (const ST*)src, idx_t, y0, y1, ly,   \
                                                                x0, x1, lx, (OT*)dst);                    \
    PV_LAUNCH_OK("clip_transform_kernel<" #ST "," #OT ">");                                               \
  } while (0)
  const bool h = d->dst_dtype == PV_F16;
  switch (d->src_dtype) {
    case PV_U8: if (h) PV_TR(uint8_t, __half); else PV_TR(uint8_t, float); break;
    case PV_F32: if (h) PV_TR(float, __half); else PV_TR(float, float); break;
    case PV_F16: if (h) PV_TR(__half, __half); else PV_TR(__half, float); break;
    default: pv::set_error("src dtype %d unsupported", d->src_dtype); return PV_ERR_INVALID;
  }
#undef PV_TR
  return PV_OK;
}


namespace pv {
// Test-time ensembling over the views of a video (pytorchvideo_trainer module/video_classification.py:290-311:
// per-video accumulation of the per-clip predictions, "sum" or "max", then division by the clip count):
// out[v][k] = reduce_{i < n_views} preds[(v*n_views + i)][k];  mode 0 = sum, 1 = mean (sum / n_views), 2 = max.
// Both accumulators are the reference's: they start from torch.zeros, and "max" folds with torch.max, so it is
// max(0, max_i p_i) and a NaN in any view propagates (fmaxf would drop it).
__global__ void view_reduce_kernel(const float* __restrict__ preds, float* __restrict__ out, int n_videos, int n_views,
                                   int K, int mode) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_videos * K) return;
  const int v = i / K, k = i - v * K;
  const float* p = preds + (long long)v * n_views * K + k;
  float acc = 0.f;
  for (int j = 0; j < n_views; ++j) {
    const float x = p[(long long)j * K];
    if (mode != 2) acc = acc + x;
    else if (acc == acc) acc = (x != x || x > acc) ? x : acc;   // torch.max: NaN wins, else the larger
  }
  out[i] = mode == 1 ? acc / (float)n_views : acc;
}
}  // namespace pv

extern "C" int pv_view_reduce(const float* preds, float* out, int n_videos, int n_views, int K, int mode, void* stream) {
  PV_CHECK_ARG(preds && out, "null argument");
  PV_CHECK_ARG(n_videos >= 1 && n_views >= 1 && K >= 1 && mode >= 0 && mode <= 2, "bad sizes / mode");
  const int total = n_videos * K;
  pv::view_reduce_kernel<<<(unsigned)pv::cdiv(total, 128), 128, 0, (cudaStream_t)stream>>>(preds, out, n_videos, n_views, K, mode);
  PV_LAUNCH_OK("view_reduce_kernel");
  return PV_OK;
}

namespace pv {
static int launch_clip_batch(const pv_clip_batch_desc* d, const void* src, const int32_t* idx_t, const int32_t* slow_pos,
                             const int32_t* geom, const long long* frame_off, void* dst, void* dst_slow, cudaStream_t s);
}  // namespace pv

extern "C" int pv_clip_transform_batch(const pv_clip_batch_desc* d, const void* src, const int32_t* idx_t,
                                       const int32_t* slow_pos, const int32_t* geom, void* dst, void* dst_slow,
                                       void* stream) {
  PV_CHECK_ARG(d && src && idx_t && dst, "null argument");
  PV_CHECK_ARG(d->C >= 1 && d->C <= 4, "C must be in 1..4 (got %d)", d->C);
  PV_CHECK_ARG(d->n_clips >= 1 && d->n_t >= 1 && d->out_h >= 1 && d->out_w >= 1, "empty output");
  PV_CHECK_ARG((long long)d->n_clips * d->n_t <= 65535, "grid too large");
  PV_CHECK_ARG(d->in_h >= 1 && d->in_w >= 1 && d->new_h >= 1 && d->new_w >= 1, "bad frame size");
  PV_CHECK_ARG(geom != nullptr || (d->top >= 0 && d->left >= 0 && d->top + d->out_h <= d->new_h && d->left + d->out_w <= d->new_w),
               "crop window outside the resized frame");
  PV_CHECK_ARG((slow_pos == nullptr) == (dst_slow == nullptr) && (slow_pos == nullptr || d->n_slow >= 1), "slow pathway arguments");
  const bool pass = d->dst_dtype == PV_U8;
  PV_CHECK_ARG(!pass || (d->src_dtype == PV_U8 && !d->div255 && !d->normalize && geom == nullptr && d->new_h == d->in_h && d->new_w == d->in_w),
               "uint8 output is a pure frame selection / crop (no resize, no arithmetic)");
  auto absll = [](long long v) { return v < 0 ? -v : v; };
  PV_CHECK_ARG((long long)d->in_h * absll(d->sh) + (long long)d->in_w * absll(d->sw) < (1ll << 31) && d->sh >= 0 && d->sw >= 0,
               "frame too large for 32-bit in-plane offsets");
  PV_CHECK_ARG((long long)d->C * (d->n_t > d->n_slow ? d->n_t : d->n_slow) * d->out_h * d->out_w < (1ll << 31),
               "output clip too large for 32-bit offsets");
  return pv::launch_clip_batch(d, src, idx_t, slow_pos, geom, nullptr, dst, dst_slow, (cudaStream_t)stream);
}

namespace pv {
// grid and instance selection shared by the per-batch and ragged entry points; frame_off selects the ragged mode
static int launch_clip_batch(const pv_clip_batch_desc* d, const void* src, const int32_t* idx_t, const int32_t* slow_pos,
                             const int32_t* geom, const long long* frame_off, void* dst, void* dst_slow, cudaStream_t s) {
  const int half_w = (d->out_w + 1) / 2;
  const unsigned bx = (unsigned)(half_w >= pv::TB_THREADS ? pv::TB_THREADS : half_w);
  const unsigned by = (unsigned)(pv::TB_THREADS / bx >= pv::TB_ROWS ? pv::TB_ROWS : (pv::TB_THREADS / bx < 1 ? 1 : pv::TB_THREADS / bx));
  dim3 grid(1, (unsigned)pv::cdiv(d->out_h, pv::TB_ROWS), d->n_clips * d->n_t), block(bx, by);
  PV_CHECK_ARG(grid.y <= 65535, "grid too large");
  const bool arith = d->div255 || d->normalize;
  // LUT instances exist only for a uint8 source with a float destination (the uint8 pass-through has no arithmetic)
#define PV_TB_LAUNCH(ST, OT, NC, LUT)                                                                                  \
  do {                                                                                                                 \
    pv::clip_transform_batch_kernel<ST, OT, NC, LUT><<<grid, block, 0, s>>>(*d, (const ST*)src, idx_t, slow_pos, geom, \
                                                                           frame_off, (OT*)dst, (OT*)dst_slow);        \
    PV_LAUNCH_OK("clip_transform_batch_kernel<" #ST "," #OT "," #NC "," #LUT ">");                                    \
  } while (0)
#define PV_TB(ST, OT, NC)                                                                                              \
  do {                                                                                                                 \
    if constexpr (std::is_same<ST, uint8_t>::value && !std::is_same<OT, uint8_t>::value) {                             \
      if (arith) PV_TB_LAUNCH(ST, OT, NC, true);                                                                       \
      else PV_TB_LAUNCH(ST, OT, NC, false);                                                                            \
    } else {                                                                                                           \
      PV_TB_LAUNCH(ST, OT, NC, false);                                                                                 \
    }                                                                                                                  \
  } while (0)
#define PV_TBC(ST, OT)                                                          \
  do {                                                                          \
    switch (d->C) {                                                             \
      case 1: PV_TB(ST, OT, 1); break;                                          \
      case 2: PV_TB(ST, OT, 2); break;                                          \
      case 3: PV_TB(ST, OT, 3); break;                                          \
      default: PV_TB(ST, OT, 4); break;                                         \
    }                                                                           \
  } while (0)
  const int od = d->dst_dtype;
  switch (d->src_dtype) {
    case PV_U8:
      if (od == PV_F16) PV_TBC(uint8_t, __half); else if (od == PV_F32) PV_TBC(uint8_t, float); else PV_TBC(uint8_t, uint8_t);
      break;
    case PV_F32:
      if (od == PV_F16) PV_TBC(float, __half); else if (od == PV_F32) PV_TBC(float, float);
      else { pv::set_error("f32 source needs an f16|f32 destination"); return PV_ERR_INVALID; }
      break;
    case PV_F16:
      if (od == PV_F16) PV_TBC(__half, __half); else if (od == PV_F32) PV_TBC(__half, float);
      else { pv::set_error("f16 source needs an f16|f32 destination"); return PV_ERR_INVALID; }
      break;
    default: pv::set_error("src dtype %d unsupported", d->src_dtype); return PV_ERR_INVALID;
  }
#undef PV_TBC
#undef PV_TB
#undef PV_TB_LAUNCH
  return PV_OK;
}
}  // namespace pv

extern "C" int pv_clip_transform_ragged(const pv_clip_batch_desc* d, const void* src, const long long* frame_off,
                                        const int32_t* geom, const int32_t* geom_host, const int32_t* slow_pos,
                                        void* dst, void* dst_slow, void* stream) {
  PV_CHECK_ARG(d && src && frame_off && geom && geom_host && dst, "null argument");
  PV_CHECK_ARG(d->C == 3, "ragged mode needs 3 channels (got %d)", d->C);
  PV_CHECK_ARG(d->n_clips >= 1 && d->n_t >= 1 && d->out_h >= 1 && d->out_w >= 1, "empty batch");
  PV_CHECK_ARG((long long)d->n_clips * d->n_t <= 65535, "grid too large");
  PV_CHECK_ARG(d->src_dtype == PV_U8 || d->src_dtype == PV_F32, "ragged mode reads uint8 or f32 frames");
  PV_CHECK_ARG(d->dst_dtype == PV_F16 || d->dst_dtype == PV_F32, "ragged mode writes f16 or f32");
  PV_CHECK_ARG((slow_pos == nullptr) == (dst_slow == nullptr) && (slow_pos == nullptr || d->n_slow >= 1), "slow pathway arguments");
  PV_CHECK_ARG((long long)d->C * (d->n_t > d->n_slow ? d->n_t : d->n_slow) * d->out_h * d->out_w < (1ll << 31),
               "output clip too large for 32-bit offsets");
  for (int b = 0; b < d->n_clips; ++b) {
    const int32_t* g = geom_host + 7 * b;
    PV_CHECK_ARG(g[0] >= 1 && g[1] >= 1 && g[2] >= 1 && g[3] >= 1, "clip %d: bad frame size", b);
    PV_CHECK_ARG((long long)g[0] * g[1] * d->C < (1ll << 31), "clip %d: %dx%d frame too large for 32-bit in-frame offsets",
                 b, g[1], g[0]);
    PV_CHECK_ARG(g[4] >= 0 && g[5] >= 0 && (long long)g[4] + d->out_h <= g[2] && (long long)g[5] + d->out_w <= g[3],
                 "clip %d: crop window outside the resized frame", b);
  }
  return pv::launch_clip_batch(d, src, nullptr, slow_pos, geom, frame_off, dst, dst_slow, (cudaStream_t)stream);
}

extern "C" int pv_clip_transform_rrc(const pv_clip_batch_desc* d, const void* src, const int32_t* idx_t,
                                     const int32_t* boxes, void* dst, void* stream) {
  PV_CHECK_ARG(d && src && idx_t && boxes && dst, "null argument");
  PV_CHECK_ARG(d->C == 3, "RandomResizedCrop mode needs 3 channels (got %d)", d->C);
  PV_CHECK_ARG(d->n_clips >= 1 && d->n_t >= 1 && d->out_h >= 1 && d->out_w >= 1, "empty output");
  PV_CHECK_ARG((long long)d->n_clips * d->n_t <= 65535, "grid too large");
  PV_CHECK_ARG(d->in_h >= 1 && d->in_w >= 1, "bad frame size");
  PV_CHECK_ARG(d->src_dtype == PV_U8 || d->src_dtype == PV_F32, "RandomResizedCrop mode reads uint8 or f32 clips");
  PV_CHECK_ARG(d->dst_dtype == PV_F16 || d->dst_dtype == PV_F32, "RandomResizedCrop mode writes f16 or f32");
  auto absll = [](long long v) { return v < 0 ? -v : v; };
  PV_CHECK_ARG((long long)d->in_h * absll(d->sh) + (long long)d->in_w * absll(d->sw) < (1ll << 31) && d->sh >= 0 && d->sw >= 0,
               "frame too large for 32-bit in-plane offsets");
  PV_CHECK_ARG(3ll * d->n_t * d->out_h * d->out_w < (1ll << 31), "output clip too large for 32-bit offsets");
  const int half_w = (d->out_w + 1) / 2;
  const unsigned bx = (unsigned)(half_w >= pv::TB_THREADS ? pv::TB_THREADS : half_w);
  const unsigned by = (unsigned)(pv::TB_THREADS / bx >= pv::TB_ROWS ? pv::TB_ROWS : (pv::TB_THREADS / bx < 1 ? 1 : pv::TB_THREADS / bx));
  dim3 grid(1, (unsigned)pv::cdiv(d->out_h, pv::TB_ROWS), d->n_clips * d->n_t), block(bx, by);
  PV_CHECK_ARG(grid.y <= 65535, "grid too large");
  cudaStream_t s = (cudaStream_t)stream;
  const bool h = d->dst_dtype == PV_F16;
#define PV_RRC(ST, OT, LUT_)                                                                                         \
  do {                                                                                                               \
    pv::clip_transform_rrc_kernel<ST, OT, LUT_><<<grid, block, 0, s>>>(*d, (const ST*)src, idx_t, boxes, (OT*)dst); \
    PV_LAUNCH_OK("clip_transform_rrc_kernel<" #ST "," #OT ">");                                                      \
  } while (0)
  if (d->src_dtype == PV_U8) {
    if (h) PV_RRC(uint8_t, __half, true); else PV_RRC(uint8_t, float, true);
  } else {
    if (h) PV_RRC(float, __half, false); else PV_RRC(float, float, false);
  }
#undef PV_RRC
  return PV_OK;
}

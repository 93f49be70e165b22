/*
 * pv_b200.h - C ABI of libpvb200.so, the H100 (sm_90a) forward-path engine for the
 * PyTorchVideo hot path.
 *
 * Every entry point takes plain device pointers + sizes + an explicit cudaStream_t (passed as
 * void* so that the header needs no CUDA include), allocates nothing, never throws, and returns
 * 0 on success or a negative pv_status.  pv_last_error() returns a thread-local message.
 *
 * Activations are "NDHWC" (channels-last-3d): element (n,t,h,w,c) of a tensor lives at
 *   base + (((n*T + t)*H + h)*W + w) * row_stride + c
 * where row_stride >= C is the distance (in elements) between consecutive positions; a tensor
 * may therefore be a channel slice of a wider buffer (this is how torch.cat(dim=1) is fused
 * away).  Channel counts of internal activations are padded to a multiple of 8 and the pad
 * lanes are kept at exactly zero.
 *
 * Each function cites the reference call site(s) (facebookresearch/pytorchvideo @ f3142bb,
 * paths relative to the reference root) whose arithmetic it replaces.
 */
#ifndef PV_B200_H_
#define PV_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PV_ABI_VERSION 1

typedef enum pv_status {
  PV_OK = 0,
  PV_ERR_INVALID = -1,     /* bad argument / unsupported shape                       */
  PV_ERR_CUDA = -2,        /* a CUDA runtime / driver call failed                    */
  PV_ERR_UNSUPPORTED = -3, /* no kernel for this configuration (never falls back)    */
  PV_ERR_NO_DEVICE = -4    /* no sm_90 device visible                                */
} pv_status;

typedef enum pv_dtype { PV_F16 = 0, PV_F32 = 1, PV_U8 = 2, PV_I64 = 3 /* pv_soft_target_ce targets only */ } pv_dtype;

typedef enum pv_act {
  PV_ACT_NONE = 0,
  PV_ACT_RELU = 1,
  PV_ACT_SWISH = 2,   /* x*sigmoid(x)        reference layers/swish.py:25-28     */
  PV_ACT_GELU = 3,    /* exact erf GELU      reference layers/attention.py:74   */
  PV_ACT_SIGMOID = 4,
  PV_ACT_HSWISH = 5   /* x*clamp(x+3,0,6)/6  torch.nn.Hardswish; the mobile efficient blocks' "hswish"
                       * Every entry point that takes an activation rejects a code outside 0..5 with
                       * PV_ERR_INVALID (PV_ERR_UNSUPPORTED where a kernel family implements fewer
                       * codes), and every *_supported probe answers 0 for it. */
} pv_act;

typedef enum pv_conv_algo {
  PV_ALGO_AUTO = 0,
  PV_ALGO_DIRECT = 1,   /* CUDA-core tiled direct convolution (any shape, f16 or f32 storage) */
  PV_ALGO_TCGEN05 = 2   /* TMA + wgmma implicit GEMM (f16 storage, fp32 register accum)      */
} pv_conv_algo;

typedef enum pv_pool_mode { PV_POOL_MAX = 0, PV_POOL_AVG = 1 } pv_pool_mode;

/* ---------------------------------------------------------------------------------------------
 * Library / device
 * ------------------------------------------------------------------------------------------- */
int pv_abi_version(void);
const char* pv_last_error(void);
/* Fills sm_count / cc (major*10+minor); returns PV_ERR_NO_DEVICE when no GPU is visible. */
int pv_device_info(int* sm_count, int* cc);
/* Number of kernels launched by this library since load (bench.py "gpu_launches"). */
long long pv_launch_count(void);
/* Launches per kernel instance since load, one "name count\n" line per instance in name order, where the
 * name carries the template arguments that select the instance (e.g. "conv3d_igemm_kernel<64,128>").
 * Writes the NUL-terminated text to buf when it fits in len bytes (else buf[0] = 0) and returns its
 * length without the NUL.  CUDA-graph replays are not counted. */
int pv_kernel_counts(char* buf, int len);

/* ---------------------------------------------------------------------------------------------
 * Clip transform chain, fused (one kernel):
 *   UniformTemporalSubsample -> Div255 -> Normalize -> ShortSideScale(bilinear) -> crop
 * Replaces: transforms/functional.py:19-41 (uniform_temporal_subsample: idx_t is computed on the
 * host with torch.linspace exactly as functional.py:39-40 and passed in), functional.py:604-615
 * (div_255), transforms/transforms.py:177-195 (Normalize), functional.py:92-131
 * (short_side_scale -> F.interpolate bilinear, align_corners=False), torchvision CenterCrop /
 * RandomCrop / functional.py:302-347 (uniform_crop) window selection.
 *
 * src is a uint8 (or f32/f16) clip addressed as src[c*sc + t*st + h*sh + w*sw], so both the
 * CTHW-contiguous layout and the decoder's THWC-interleaved layout (data/utils.py:26-31) work.
 * The bilinear taps are host-computed tables (bit-exact w.r.t. ATen's index/lambda math):
 *   for output row y:  rows y0[y], y1[y], weight ly[y] of row y1   (already offset by the crop)
 *   for output col x:  cols x0[x], x1[x], weight lx[x] of col x1
 * out[c][j][y][x] = ly0*(lx0*v00 + lx1*v01) + ly1*(lx0*v10 + lx1*v11),
 *   v = (float(src)/255 - mean[c]) / std[c], taken from frame idx_t[j];  dst is [C,n_t,oh,ow].
 * With identity tables / mean 0 / std 1 / div255 0 the same kernel is each single transform
 * (UniformTemporalSubsample, Div255, Normalize, ShortSideScale, crop) on its own.
 * ------------------------------------------------------------------------------------------- */
typedef struct pv_clip_transform_desc {
  int C, n_t, out_h, out_w;
  long long sc, st, sh, sw;   /* source strides in ELEMENTS of the source dtype    */
  float mean[4], stdv[4];     /* per channel (C <= 4)                             */
  int src_dtype;              /* PV_U8 (decoder frames), PV_F32 or PV_F16         */
  int dst_dtype;              /* PV_F16 or PV_F32                                 */
  int div255;                 /* 1: v = src/255 first (Div255); 0: v = src        */
} pv_clip_transform_desc;

int pv_clip_transform_fwd(const pv_clip_transform_desc* d, const void* src,
                          const int32_t* idx_t,
                          const int32_t* y0, const int32_t* y1, const float* ly,
                          const int32_t* x0, const int32_t* x1, const float* lx,
                          void* dst, void* stream);

/* Batched chain: n_clips clips per launch (same source geometry), taps computed in the kernel with ATen's
 * arithmetic (no tables), optional per-clip geometry for the train chain, optional SECOND output = the SlowFast
 * slow pathway (pytorchvideo_trainer/datamodule/transforms.py:99-138 SlowFastPackPathway), uint8 pass-through
 * for pure frame selection (transforms/functional.py:19-41 keeps the dtype; :134-160 _repeated).
 *   src[clip*s_clip + c*sc + idx_t[j]*st + h*sh + w*sw]  ->  dst[clip*d_clip + ((c*n_t + j)*out_h + y)*out_w + x]
 *   slow_pos[j] >= 0: the same pixel is also written to dst_slow[clip*d_slow_clip + ((c*n_slow + slow_pos[j])*out_h + y)*out_w + x]
 *   geom (device, optional): per clip {new_h, new_w, top, left, hflip, first_frame} overriding the descriptor's
 *   values; first_frame is added to every idx_t[j] (temporal views of one video: s_clip = 0)
 * idx_t / slow_pos / geom are DEVICE int32 arrays; src/dst device pointers (src may be pinned host memory
 * mapped into the device address space: decoder frames are read exactly once).                            */
typedef struct pv_clip_batch_desc {
  int C, n_clips, n_t, n_slow;
  int in_h, in_w, new_h, new_w;     /* source frame, resize target (== source for no resize)      */
  int top, left, out_h, out_w;      /* crop window inside the resized frame                       */
  int hflip;                        /* mirror the cropped output along W                          */
  long long sc, st, sh, sw, s_clip; /* source strides in ELEMENTS (channel, frame, row, col, clip) */
  long long d_clip, d_slow_clip;    /* destination strides between clips, in elements             */
  float mean[4], stdv[4];
  int div255, normalize;            /* 1: x/255 first; 1: (x-mean)/std                             */
  int src_dtype, dst_dtype;         /* src: PV_U8|PV_F32|PV_F16, dst: PV_F16|PV_F32|PV_U8 (pass-through) */
} pv_clip_batch_desc;

int pv_clip_transform_batch(const pv_clip_batch_desc* d, const void* src, const int32_t* idx_t,
                            const int32_t* slow_pos, const int32_t* geom, void* dst, void* dst_slow,
                            void* stream);

/* RandomResizedCrop mode of the batched chain (transforms/functional.py random_resized_crop): every kept frame j of
 * clip b reads its own source window boxes[(b*n_t + j)*5 + {0..4}] = {top, left, h, w, hflip} of the in_h x in_w frame
 * and resizes it to out_h x out_w with ATen's bilinear taps relative to the window, after the optional /255 and
 * normalisation of the descriptor.  new_h/new_w/top/left/hflip/n_slow/d_slow_clip of the descriptor are ignored.
 * C must be 3; src PV_U8 or PV_F32, dst PV_F16 or PV_F32.  boxes is a DEVICE int32 array; the caller keeps every
 * window inside the frame.                                                                                            */
int pv_clip_transform_rrc(const pv_clip_batch_desc* d, const void* src, const int32_t* idx_t, const int32_t* boxes,
                          void* dst, void* stream);

/* Ragged mode of the batched chain: the output of pv_clip_transform_batch, but every clip reads its own frames, of
 * its own size (a batch of frame-folder videos of mixed resolutions, decoded by pv_jpeg_decode into one buffer).
 * Kept frame j of clip b is a packed HWC frame of C channels, in_h[b] x in_w[b], starting at element
 * frame_off[b * n_t + j] of src (temporal selection is done in frame_off; an entry may repeat).  geom is a DEVICE int32
 * array of {in_h, in_w, new_h, new_w, top, left, hflip} per clip and geom_host the same table in host memory, which the
 * call validates; frame_off is a DEVICE int64 array whose frames the caller keeps inside src.  slow_pos / dst_slow,
 * mean / stdv / div255 / normalize, out_h / out_w, n_slow, d_clip and d_slow_clip are read as pv_clip_transform_batch
 * reads them; in_h / in_w / new_h / new_w / top / left / hflip and the source strides of the descriptor are ignored.
 * C must be 3; src PV_U8 or PV_F32, dst PV_F16 or PV_F32.  PV_ERR_INVALID for an empty batch, a frame of
 * in_h * in_w * C >= 2^31 elements, or a window outside its resized frame.  One launch.                        */
int pv_clip_transform_ragged(const pv_clip_batch_desc* d, const void* src, const long long* frame_off,
                             const int32_t* geom, const int32_t* geom_host, const int32_t* slow_pos, void* dst,
                             void* dst_slow, void* stream);

/* Detection boxes of the batched chain (transforms/functional.py:195-445: short_side_scale_with_boxes,
 * random_crop_with_boxes, uniform_crop_with_boxes, horizontal_flip_with_boxes, clip_boxes_to_image, crop_boxes).
 * Clip b owns boxes box_start[b] .. box_start[b+1]-1 of the (n_boxes, 4) array of (x1, y1, x2, y2); box_start is a
 * DEVICE int32 array of n_clips + 1 non-decreasing offsets with box_start[n_clips] == n_boxes.  geom is the per-clip
 * {new_h, new_w, top, left, hflip, first_frame} array pv_clip_transform_batch reads (or NULL: the descriptor's
 * values for every clip), so a clip and its boxes share one crop and one flip.  The set bits of steps run in order:
 *   PV_BOX_CLIP_SRC   x = min(in_w - 1, max(0, x)), likewise y with in_h   (clip_boxes_to_image, source frame)
 *   PV_BOX_SCALE      x *= T(double(new_h) / in_h) if in_w < in_h, else T(double(new_w) / in_w)
 *   PV_BOX_CROP       x -= left, y -= top
 *   PV_BOX_CLIP_CROP  clip to out_h x out_w                                  (the crops' clip_boxes_to_image)
 *   PV_BOX_FLIP       when the clip's hflip is set: x1' = (out_w - x2) - 1, x2' = (out_w - x1) - 1
 *   PV_BOX_CLIP_OUT   clip to out_h x out_w                                  (clip_boxes_to_image, output frame)
 * Each operation rounds once to the boxes' type T (float32 or float64), as the reference's eager ops do.  The boxes
 * are written to boxes_out in T (boxes_out == boxes_in is allowed); rois_out, when not NULL, also receives the fp32
 * (n_boxes, 5) rows (b, x1, y1, x2, y2) that pv_roi_align_fwd reads.  One launch; n_boxes == 0 launches nothing.  */
#define PV_BOX_F32 1
#define PV_BOX_F64 3
#define PV_BOX_CLIP_SRC 1
#define PV_BOX_SCALE 2
#define PV_BOX_CROP 4
#define PV_BOX_CLIP_CROP 8
#define PV_BOX_FLIP 16
#define PV_BOX_CLIP_OUT 32
#define PV_BOX_ALL_STEPS 63

typedef struct pv_boxes_desc {
  int n_clips, n_boxes;             /* B clips, K boxes in all                                    */
  int steps;                        /* PV_BOX_* step mask                                         */
  int dtype;                        /* PV_BOX_F32 | PV_BOX_F64                                    */
  int in_h, in_w;                   /* source frame                                               */
  int new_h, new_w, top, left, hflip;  /* every clip's geometry when geom is NULL                  */
  int out_h, out_w;                 /* crop / output frame                                        */
} pv_boxes_desc;

int pv_clip_boxes_transform(const pv_boxes_desc* d, const void* boxes_in, const int32_t* box_start,
                            const int32_t* geom, void* boxes_out, float* rois_out, void* stream);

/* Ragged mode of the box transform: the boxes of a batch whose clips come from frames of their own sizes (the
 * companion of pv_clip_transform_ragged).  geom is the DEVICE int32 table pv_clip_transform_ragged reads, one row
 * {in_h, in_w, new_h, new_w, top, left, hflip} per clip, and geom_host the same table in host memory, which the call
 * validates (every size >= 1, the out_h x out_w window at (top, left) inside new_h x new_w).  Each clip takes its own
 * in_h / in_w for PV_BOX_CLIP_SRC and PV_BOX_SCALE (the scale's in_w < in_h test is made per clip); the descriptor's
 * in_*, new_*, top, left and hflip are ignored, and out_h / out_w (both >= 1) are read from it.  One more step bit,
 * accepted only here, runs before all the others:
 *   PV_BOX_DENORM     x = x * T(in_w), y = y * T(in_h), one rounding each   ([0, 1] coordinates to source pixels)
 * box_start, boxes_out == boxes_in, rois_out and the rounding are as in pv_clip_boxes_transform.  One launch;
 * n_boxes == 0 launches nothing.                                                                                */
#define PV_BOX_DENORM 64

int pv_clip_boxes_transform_ragged(const pv_boxes_desc* d, const void* boxes_in, const int32_t* box_start,
                                   const int32_t* geom, const int32_t* geom_host,
                                   void* boxes_out, float* rois_out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Video augmentation (transforms/augmentations.py, rand_augment.py, augmix.py): a batch of clips of (T, 3, H, W)
 * frames, each clip with its own op per layer step.
 *   src[(clip / src_div)*s_clip + t*st + c*sc + h*sh + w*sw]  (any strides; src_div > 1 feeds several AugMix chains
 *   from one clip)  ->  dst contiguous [n_clips][T][3][H][W] of the same dtype (PV_U8 or PV_F32).
 * pv_augment_stats fills one pv_aug_frame_stats per (clip, frame): per-channel min / max, the Equalize table and the
 * grayscale sum of AdjustContrast; integer histogram atomics and a fixed-order reduction make it deterministic.
 * pv_augment_apply runs ops[clip] on every clip (ops and stats are DEVICE arrays; stats may be NULL when no op needs it).
 * pv_augment_mix: dst[b] = m*x[b] + (1-m)*sum_k w_k*chains[b*width + k] with mix[b*(width+2)] = {w_0.., m, 1-m}.    */
typedef enum pv_aug_kind {
  PV_AUG_NONE = 0, PV_AUG_BRIGHTNESS = 1, PV_AUG_CONTRAST = 2, PV_AUG_SATURATION = 3, PV_AUG_SHARPNESS = 4,
  PV_AUG_AUTOCONTRAST = 5, PV_AUG_EQUALIZE = 6, PV_AUG_INVERT = 7, PV_AUG_POSTERIZE = 8, PV_AUG_SOLARIZE = 9,
  PV_AUG_AFFINE = 10
} pv_aug_kind;

typedef struct pv_aug_op {
  int kind;        /* pv_aug_kind                                                                      */
  int ival;        /* Posterize: bit mask; Solarize on uint8: threshold                                */
  float ratio;     /* _blend ratio (Brightness/Contrast/Saturation/Sharpness); Solarize on f32: threshold */
  float omr;       /* _blend: float(1 - ratio) rounded once from the double, as torchvision's scalar   */
  float theta[6];  /* Affine: the grid matrix already divided by (W/2, H/2), row-major 2x3             */
  float fill[3];   /* Affine: fill colour                                                              */
} pv_aug_op;

typedef struct pv_aug_frame_stats {
  float mn[3], mx[3];
  double gray_sum;
  unsigned char lut[3][256];
} pv_aug_frame_stats;

typedef struct pv_augment_desc {
  int n_clips, src_div, T, C, H, W;
  long long s_clip, st, sc, sh, sw;  /* source strides in elements */
  int dtype;                         /* PV_U8 | PV_F32             */
} pv_augment_desc;

int pv_augment_stats(const pv_augment_desc* d, const void* src, pv_aug_frame_stats* stats, void* stream);
int pv_augment_apply(const pv_augment_desc* d, const void* src, const pv_aug_op* ops, const pv_aug_frame_stats* stats,
                     void* dst, void* stream);
int pv_augment_mix(const pv_augment_desc* d, const void* src, const void* chains, int width, const float* mix,
                   void* dst, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Batch mixing (transforms/mix.py: MixUp, CutMix, MixVideo), in place on a batch of B clips.  Clip b pairs with clip
 * B-1-b.  Element e of clip b sits at x[b*s_batch + sum_i idx_i*stride[i]] over the per-clip dims size[0..3]
 * (outermost first, padded with 1 at the front); any strides, but no two elements may share memory.
 * pv_mixup: x[b] = T(T(x[b]*lam) + T(x[B-1-b]*oml)) for every b at once (the middle clip of an odd B mixes with
 *   itself), one rounding to the element type T (PV_F32 | PV_F16) per product and per sum; fp32 products.
 * pv_cutmix: swaps x[b][..., yl:yh, xl:xh] with x[B-1-b][..., yl:yh, xl:xh]; size[2], size[3] are H, W.  Any element
 *   size (PV_U8 | PV_F16 | PV_F32).  An empty box launches nothing.
 * pv_mix_labels: the (B, K) float32 label mix out[b] = f(f(l1*lam) + f(l2*oml)), l1 / l2 the label rows of clips b and
 *   B-1-b: one-hot rows (on at the class, off elsewhere) built from int64 indices, or float32 rows given (one_hot).
 *   mode 1 / 2 writes the one-hot row of clip b alone, as float32 / int64 (convert_to_one_hot).  Indices are checked:
 *   *flag |= 1 for an index >= K, |= 2 for a negative one (flag is zeroed first, on the stream).                      */
typedef struct pv_mix_desc {
  int B;                  /* clips in the batch                  */
  int dtype;              /* PV_F32 | PV_F16 | PV_U8             */
  long long size[4];      /* per-clip dims, outermost first      */
  long long stride[4];    /* their strides in elements           */
  long long s_batch;      /* stride between clips in elements    */
} pv_mix_desc;

typedef struct pv_mix_label_desc {
  int B, K;
  int one_hot;            /* labels are float32 (B, K) rows, not int64 indices             */
  int mode;               /* 0: mix; 1: one-hot rows as float32; 2: one-hot rows as int64   */
  float lam, oml;         /* the two weights, each already rounded to float32              */
  float on, off;          /* one-hot values: 1 - ls + ls/K and ls/K, rounded from double   */
  long long s_row, s_col; /* label strides in elements (s_col unused for indices)          */
} pv_mix_label_desc;

int pv_mixup(const pv_mix_desc* d, void* x, float lam, float oml, void* stream);
int pv_cutmix(const pv_mix_desc* d, void* x, int yl, int yh, int xl, int xh, void* stream);
int pv_mix_labels(const pv_mix_label_desc* d, const void* labels, void* out, int* flag, void* stream);

/* Test-time multi-view ensembling (pytorchvideo_trainer/module/video_classification.py:290-311, docs model_zoo.md:63
 * "3 spatial x 10 temporal views"): out[v][k] = reduce over the n_views consecutive rows of video v;
 * mode 0 = sum, 1 = mean (sum / clip count), 2 = max.  preds: [n_videos * n_views][K] f32.                    */
int pv_view_reduce(const float* preds, float* out, int n_videos, int n_views, int K, int mode, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Layout / dtype conversion at the API boundary.
 * NCDHW (reference model input, models/net.py:41-44) -> NDHWC with C padded to c_pad (zeros).
 * src dtype f32 or f16; dst dtype f16 or f32.
 * ------------------------------------------------------------------------------------------- */
int pv_ncdhw_to_ndhwc(const void* src, int src_dtype, void* dst, int dst_dtype,
                      int N, int C, int T, int H, int W, int c_pad, long long dst_row_stride,
                      void* stream);
/* Same, but every output row is x_w_phys pixels wide with w_pad zero pixels on the left and zeros
 * on the right (dst holds N*T*H*w_phys*c_pad + c_pad*8 elements): the stem layout of window mode. */
int pv_ncdhw_to_ndhwc_padw(const void* src, int src_dtype, void* dst, int dst_dtype,
                           int N, int C, int T, int H, int W, int c_pad, int w_pad, int w_phys,
                           void* stream);
/* Clears n floats (SE accumulators) with a stream-ordered memset. */
int pv_zero_f32(float* dst, long long n, void* stream);
/* NDHWC -> NCDHW f32 (for handing feature maps back to torch when a model has no head). */
int pv_ndhwc_to_ncdhw(const void* src, int src_dtype, long long src_row_stride, float* dst,
                      int N, int C, int T, int H, int W, void* stream);

/* ---------------------------------------------------------------------------------------------
 * 3-D convolution + folded BatchNorm(eval) scale/bias + optional residual + activation.
 * Replaces nn.Conv3d -> nn.BatchNorm3d(eval) -> activation chains built at
 * models/resnet.py:98-132 (conv_a/b/c), :422-438 (branch1), models/stem.py:80-87,
 * models/slowfast.py:672-679 (FuseFastToSlow), models/x3d.py:66-88,160-217, models/csn.py:169,
 * layers/convolutions.py:191-237 (Conv2plus1d), models/stem.py:330-337 (PatchEmbed) and the
 * residual add + ReLU of models/resnet.py:1179-1189.
 *   y = act( conv(x, w) * scale[co] + bias[co] (+ residual) )
 * groups must divide Ci and Co.  groups == 1 is dense, groups == Ci == Co depthwise (PV_ALGO_DIRECT or
 * pv_dwconv3d_fwd).  Other group counts (models/resnet.py conv_b_num_groups, models/csn.py width per group) run
 * only in the grouped mode of PV_ALGO_TCGEN05: f16, 1 < groups < Ci, Ci == Co, Ci % 8 == 0, more than one group
 * span (see pv_conv3d_group_span), the dense limits on taps, strides, offsets and row strides, and ci_pad64 equal to
 * the span width span_k.  PV_ALGO_DIRECT returns PV_ERR_UNSUPPORTED for them; a caller runs what grouped mode does
 * not take as the dense convolution with block-diagonal weights.
 *
 * Packed weights (host-side, see pytorchvideo_b200/engine/packing.py):
 *   PV_ALGO_DIRECT, dense : w[tap][ci][co]        (storage dtype, Ci/Co padded)
 *   depthwise (any algo)  : w[tap][c]             (storage dtype)
 *   PV_ALGO_TCGEN05       : w[co][tap][ci_pad64]  (f16, K-major rows of length taps*ci_pad64;
 *                           C_in < 64: ci_pad64 = Ci, row padded to a multiple of 64;
 *                           window mode: w[co][kt*kh][win] with win = 16|32|64 >= kw*Ci;
 *                           grouped mode: ci_pad64 = span_k, row co holds the weights of its group
 *                           g = co / Cg at offset (g mod span_groups) * Cg of every tap's span_k block,
 *                           zeros elsewhere)
 * ------------------------------------------------------------------------------------------- */
typedef struct pv_conv3d_desc {
  int dtype;                 /* storage dtype of x, y, residual, w: PV_F16 | PV_F32          */
  int N, Ti, Hi, Wi, Ci;     /* Ci, Co: padded channel counts                               */
  int To, Ho, Wo, Co;
  int kt, kh, kw;
  int st, sh, sw;
  int pt, ph, pw;
  int dt, dh, dw;            /* dilation                                                    */
  int groups;
  int act;                   /* pv_act applied last                                         */
  int has_residual;
  long long x_row_stride, y_row_stride, res_row_stride;
  int ci_pad64;              /* PV_ALGO_TCGEN05 only: per-tap K extent of the packed weights */
  /* "window mode" for 3/4-channel stems on the tensor cores: the input rows physically carry
   * x_w_pad zero pixels on the left (>= pw) and are x_w_phys pixels wide in memory (written that
   * way by pv_ncdhw_to_ndhwc_padw); Wi stays the logical width.  0 = ordinary layout.           */
  int x_w_pad, x_w_phys;
  /* Depthwise path only: element distance between consecutive samples of x / y when a sample is
   * not T*H*W*row_stride apart (MViT token tensors carry a cls row in front of every sample's
   * T*H*W patch tokens).  0 = densely packed.                                                   */
  long long x_batch_stride, y_batch_stride;
  /* Post-activation addend, constant over (h, w) (the audio fusion add of FuseAudioToFastSlow,
   * models/audio_visual_slowfast.py:406-418):
   *   y[n][t][h][w][c] = act(conv * scale + bias (+ residual)) + addend[n * add_n_stride + t * add_t_stride + add_ch_off + c]
   * for output sample n and frame t; add_t_stride = 0 broadcasts one row over every frame.  Storage dtype of y,
   * Co elements from add_ch_off on.  Co, add_n_stride, add_t_stride and add_ch_off are multiples of 8 elements, the
   * pointer is 16-byte aligned and the output has fewer than 2^31 positions (else PV_ERR_INVALID from
   * pv_conv3d_fwd; pv_conv3d_tcgen05_supported and pv_conv3d_stem_rows_supported return 0).  Dense (PV_ALGO_DIRECT, PV_ALGO_TCGEN05 incl. grouped mode) and stem-rows
   * convolutions take it; depthwise convolutions return PV_ERR_UNSUPPORTED.  On the tensor cores the addend is
   * added to the f16 result in the staged output tile (one more f16 rounding); PV_ALGO_DIRECT adds it in fp32.
   * NULL = no addend (a zero-initialised descriptor behaves as without these fields).                     */
  const void* addend;
  long long add_n_stride, add_t_stride;
  int add_ch_off;
  /* Pre-activation prologue of the depthwise entry points (the BatchNorm3d + GELU that MViT's attention pools apply
   * before a depthwise pooling conv, layers/attention.py:189-197):
   *   y[c] = scale[c] * sum_taps w[tap][c] * u(x_tap) + bias[c],  u(x) = act(pre_act, pre_scale[c] * x + pre_bias[c])
   * for in-bounds taps and u = 0 for padded taps (normalise, activate, then zero-pad).  fp32 vectors of Co values.  Set
   * by pre_scale != NULL; pre_bias must then be non-NULL too, and pre_act is a pv_act code applied to every in-bounds
   * input once.  pv_dwconv3d_fwd and pv_dwplane_fwd honour it on every kernel they dispatch to; pv_conv3d_fwd and the
   * stem entry points return PV_ERR_UNSUPPORTED when it is set.  NULL = no prologue (a zero-initialised descriptor
   * behaves as without these fields).                                                                              */
  const float* pre_scale;
  const float* pre_bias;
  int pre_act;
} pv_conv3d_desc;

/* Temporal tap reduction used to factor a (kt,kh,kw) stem convolution with few output channels into
 * a (1,kh,kw) convolution producing kt*Co channels (one group of Co per temporal tap, all taps in ONE
 * tensor-core pass over the input) followed by this sum:
 *   y[n][t][p][co] = act(scale[co] * sum_dt Yk[n][t*st + dt*dil - pt][p][dt*Co + co] + bias[co])
 * (frames outside [0,Ti) contribute zero = the temporal zero padding).  Same arithmetic as the
 * direct convolution up to one f16 rounding of the per-tap partial sums.                          */
int pv_temporal_tap_sum(const void* yk, void* y, int dtype, int N, int Ti, int To, long long hw, int Co,
                        int kt, int st, int pt, int dil, const float* scale, const float* bias, int act,
                        long long in_row_stride, long long out_row_stride, void* stream);

int pv_conv3d_fwd(const pv_conv3d_desc* d, int algo, const void* x, const void* w,
                  const float* scale, const float* bias, const void* residual, void* y,
                  void* stream);
/* Depthwise convolution (groups == Ci == Co) + folded BN + activation with optional fused
 * Squeeze-Excitation statistics: when se_sums != NULL, se_sums[n][c] += sum over output positions
 * of the PRE-activation value (caller zeroes it; feeds pv_se_gate).  f16 storage runs as a TMA-fed
 * shared-memory stencil; other cases take the generic CUDA-core stencil (+ pv_channel_sum).
 * Replaces conv_b -> norm_b -> SE-pool of models/x3d.py:180-198, the X3D stem conv_xy
 * (models/x3d.py:74-82), CSN's conv_b (models/csn.py:169) and MViT's pooling convs
 * (layers/attention.py:364-403).  w: [tap][C]. */
int pv_dwconv3d_fwd(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                    const float* bias, void* y, float* se_sums, void* stream);
/* Depthwise 3x3 convolution over a one-frame token plane: the (1,3,3) attention pools of the image MViT
 * (layers/attention.py:364-403, models/vision_transformers.py use_2d_patch=True).
 *   y[n][h][w][c] = scale[c] * sum_{i,j} x[n][h*sh + i - ph][w*sw + j - pw][c] * w[i*3 + j][c] + bias[c]
 * fp32 accumulation, one f16 rounding; no activation.  Takes f16, groups == Ci == Co, Ti == To == 1, kernel (1,3,3),
 * no temporal stride or padding, sh == sw in {1, 2, 4}, ph, pw <= 2, no dilation, residual or addend, Co and
 * x_row_stride and x_batch_stride multiples of 8, y_row_stride even, x 16-byte aligned; else PV_ERR_UNSUPPORTED.
 * x_batch_stride / y_batch_stride step over MViT's cls row as in pv_dwconv3d_fwd.  w: [tap][C].
 * pv_dwplane_supported answers 1 exactly for the descriptors pv_dwplane_fwd takes (host only, no GPU). */
int pv_dwplane_supported(const pv_conv3d_desc* d);
int pv_dwplane_fwd(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                   const float* bias, void* y, void* stream);

/* 1 if PV_ALGO_TCGEN05 supports this descriptor (pure host-side check, no GPU needed). */
int pv_conv3d_tcgen05_supported(const pv_conv3d_desc* d);
/* Group span of a grouped convolution (host only): span_groups = 64 / gcd(Cg, 64) consecutive groups of
 * Cg = Ci / groups channels, whose span_k = span_groups * Cg input channels fill whole 64-channel boxes;
 * span_n = span_groups * (Co / groups).  The last span may hold fewer groups.  Each output tile of grouped mode
 * reads the input channels of its own span, so it does taps * span_k * Co multiply-adds per output position, 1/spans
 * of the dense convolution of the same width.  Returns 1 when grouped mode takes the descriptor with its weights
 * packed at ci_pad64 = span_k (whatever d->ci_pad64 holds), else 0.  The outputs are filled whenever groups > 1
 * divides Ci and Co, and are 0 otherwise. */
int pv_conv3d_group_span(const pv_conv3d_desc* d, int* span_groups, int* span_k, int* span_n);

/* Stem convolutions (ResNetBasicStem.forward models/stem.py:252-260 conv; X3D stem conv_t models/x3d.py:83-88) on the
 * 4-channel, W-padded network input, stride 2 along W: zero-copy im2col - the A operand of a filter row is the RAW
 * input row in shared memory, addressed by a no-swizzle wgmma descriptor with a 16-byte K-chunk stride (csrc/pv_stem.cu).
 * Descriptor: window-mode conventions of pv_conv3d_desc (x_w_pad, x_w_phys, ci_pad64 = window length 16|32|64).
 * w: f16 [K / 8][pad16(Co)][8], K = (dt * kh + dh) * window + (lead + dw) * 4 + c;  zero_row: >= 4 KiB of zeros. */
int pv_conv3d_stem_rows_supported(const pv_conv3d_desc* d);
int pv_conv3d_stem_rows_fwd(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                            const float* bias, const void* zero_row, void* y, void* stream);

/* Temporal-streaming stem (the SlowFast Fast stem, csrc/pv_stem_stream.cu): the stem-rows input and descriptor
 * conventions, with kt = 5 temporal taps at stride / dilation 1 (pt < kt), Co = 8, window 32 and no addend.  One pass
 * over the input frames: all 5 taps in one wgmma (N = 40) per frame, summed in fp32 registers, rounded to f16 once.
 * w: f16 [kh * 32 / 8][40][8], column 8 j + c = temporal tap j of output channel c;  zero_row: >= 4 KiB of zeros. */
int pv_conv3d_stem_stream_supported(const pv_conv3d_desc* d);
int pv_conv3d_stem_stream_fwd(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                              const float* bias, const void* zero_row, void* y, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fused bottleneck block for narrow pathways (SlowFast Fast pathway), ONE launch:
 *   a = relu(bn_a(conv_a(x)))  (kt,1,1) C_in -> C_mid;   b = relu(bn_b(conv_b(a)))  (1,3,3) stride (1,sb,sb), pad 1
 *   y = act(bn_c(conv_c(b)) + shortcut),  shortcut = x (identity) or bn_1(conv_1(x)), 1x1x1 stride (1,sb,sb)
 * Replaces BottleneckBlock.forward (models/resnet.py:1345-1365) + ResBlock.forward (resnet.py:1179-1189) for
 * C_mid in {8, 16, 32}: a and b stay in shared memory, x is read once, the residual comes from the resident x tile.
 * x, y: NDHWC f16; weights f16 packed [n][k], k = tap * C + ci, K zero-padded to a multiple of 16:
 *   wa [Cmid][pad16(kt*Cin)], wb [Cmid][pad16(9*Cmid)], wc [Cout][pad16(Cmid)], wsc [Cout][pad16(Cin)] (or NULL);
 * folded BatchNorm (scale, bias) fp32 per output channel for each of the four convolutions.
 * Supported: the instantiated (Cin, Cmid, kt, sb, shortcut) combinations, row strides that are multiples of 8, and
 * H*W*x_row_stride and Ho*Wo*y_row_stride below 2^31 (in-frame offsets are 32-bit).  pv_bottleneck_fused_fwd also
 * requires 16-byte aligned x, y, wa, wb, wc and (with a projection shortcut) wsc, else PV_ERR_INVALID.
 * pv_bottleneck_fused_tiling is the host-only tile search pv_bottleneck_fused_fwd itself uses: for a device with
 * sm_count SMs, each CTA computes a tile_h x tile_w output tile of frames_per_cta consecutive frames of one clip
 * (the last frame chunk of a clip may be shorter) with smem_bytes of dynamic shared memory.
 * ------------------------------------------------------------------------------------------- */
typedef struct pv_bottleneck_desc {
  int N, T, H, W;            /* input extents; output (T, (H-1)/sb+1, (W-1)/sb+1)                 */
  int Cin, Cmid, Cout;       /* padded channel counts (multiples of 8; Cin a power of two)        */
  int kt, sb;                /* temporal taps of conv_a (1|3, padding kt/2); spatial stride of conv_b (1|2) */
  int has_shortcut;          /* 1: projection shortcut conv_1 + bn_1; 0: identity (Cin == Cout, sb == 1)    */
  int act;                   /* PV_ACT_RELU | PV_ACT_NONE after the residual add                  */
  long long x_row_stride, y_row_stride;
} pv_bottleneck_desc;
int pv_bottleneck_fused_supported(const pv_bottleneck_desc* d);
int pv_bottleneck_fused_fwd(const pv_bottleneck_desc* d, const void* x, const void* wa, const void* wb,
                            const void* wc, const void* wsc, const float* sa, const float* ba,
                            const float* sb, const float* bb, const float* sc, const float* bc,
                            const float* ssc, const float* bsc, void* y, void* stream);
int pv_bottleneck_fused_tiling(const pv_bottleneck_desc* d, int sm_count, int* tile_h, int* tile_w,
                               int* frames_per_cta, long long* smem_bytes);

/* ---------------------------------------------------------------------------------------------
 * Pooling. nn.MaxPool3d stem pool (models/stem.py:94-100), nn.AvgPool3d head pools
 * (models/head.py:116-118, models/slowfast.py:333-341, models/x3d.py:490), MViT skip-path
 * MaxPool3d (layers/attention.py:677-679).  AvgPool divides by the full kernel volume
 * (count_include_pad=True, the torch default); MaxPool pads with -inf.
 * ------------------------------------------------------------------------------------------- */
typedef struct pv_pool3d_desc {
  int dtype, mode;
  int N, Ti, Hi, Wi, C;
  int To, Ho, Wo;
  int kt, kh, kw, st, sh, sw, pt, ph, pw;
  long long x_row_stride, y_row_stride;
  long long x_batch_stride, y_batch_stride;   /* 0 = densely packed (see pv_conv3d_desc) */
} pv_pool3d_desc;
int pv_pool3d_fwd(const pv_pool3d_desc* d, const void* x, void* y, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Squeeze-Excitation (fvcore SqueezeExcitation as used at models/x3d.py:190-198):
 *   pv_channel_sum : sums[n][c] += sum over positions of x        (sums must be zeroed)
 *   pv_se_gate     : gate[n][c] = sigmoid(W2 relu(W1 (sums/npos) + b1) + b2)   (f32 weights)
 *   pv_scale_act   : y = act(x * gate[n][c])   in place allowed
 * ------------------------------------------------------------------------------------------- */
int pv_channel_sum(const void* x, int dtype, long long row_stride, int N, long long npos, int C,
                   float* sums, void* stream);
int pv_se_gate(const float* sums, long long npos, int N, int C, int Cr,
               const float* w1, const float* b1, const float* w2, const float* b2,
               int c_stride_w, float* gate, void* stream);
int pv_scale_act(const void* x, void* y, int dtype, long long x_row_stride,
                 long long y_row_stride, int N, long long npos, int C, const float* gate,
                 int act, void* stream);

/* RoIAlign for the detection heads (pytorchvideo/models/head.py:441-482 ResNetRoIHead.forward: pool -> squeeze T ->
 * roi_layer(x, bboxes) -> pool_spatial ...; roi_layer = torchvision.ops.RoIAlign(output_size, spatial_scale,
 * sampling_ratio), aligned=False, head.py:209-227).  x: NDHWC features with T == 1 ([N][H][W][C], rows of
 * x_row_stride elements, C % 8 == 0); rois: DEVICE fp32 [K][5] = (batch index, x1, y1, x2, y2) in input pixels;
 * y: [K][pooled_h][pooled_w][C].  Sampling grid, bilinear weights and boundary rules are torchvision's.          */
int pv_roi_align_fwd(const void* x, int dtype, long long x_row_stride, int N, int H, int W, int C,
                     const float* rois, int K, int pooled_h, int pooled_w, float spatial_scale,
                     int sampling_ratio, void* y, long long y_row_stride, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Head tail (models/head.py:371-391): optional softmax over channels per position
 * (activation applied BEFORE the global average, head.py:383-390), then mean over positions,
 * un-pad and cast to f32:  out[n][c] = mean_p act(x[n][p][c]),  c < C_valid.
 * ------------------------------------------------------------------------------------------- */
int pv_head_reduce(const void* x, int dtype, long long row_stride, int N, long long npos,
                   int C_valid, int softmax, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * MViT pieces (layers/attention.py).
 * pv_layernorm : y = (x-mean)/sqrt(var+eps)*gamma+beta over C channels (f32 statistics); every row
 *                holds `groups` consecutive groups of C channels normalised independently with the
 *                same gamma/beta (groups = heads for the per-head norm_q/k/v, attention.py:200-205)
 *                nn.LayerNorm(eps=1e-6) at attention.py:655,703 / vision_transformers.py:333.
 * nn.Linear    : (attention.py:93-95,315-320,541,716) has NO entry point of its own: y = act(x W^T + b) (+ residual) on a
 *                token tensor [B*N, C] is pv_conv3d_fwd with a 1x1x1 filter (N = B, T = H = 1, W = tokens).
 * pv_attention : o = softmax((q*scale) k^T) v (+ q)    attention.py:531-539, flash-style, the
 *                N_q x N_k matrix is never materialised.  q/k/v/o are [B][N][H][D] with
 *                explicit row strides (elements between consecutive tokens), D = head dim.
 *                f16: wgmma + TMA kernel for head dims 32/64/96 (csrc/pv_attention_wgmma.cu), the mma.sync flash
 *                kernel for D = 128 (csrc/pv_attention_mma.cu), both only with 16-byte aligned q/k/v pointers,
 *                row and batch strides and 4-byte aligned o / even o strides, q/k/v rows of at least H*D elements,
 *                batch strides (B > 1) of at least N rows and all strides below 2^40 bytes; everything else (and
 *                f32) runs the CUDA-core flash kernel.  pv_attention_kernel_for tells which one a call would launch;
 *                should the driver still refuse a tensor map, pv_attention_fwd returns PV_ERR_CUDA.
 *                Wide heads and the linear mode (Non-local block, layers/nonlocal_net.py:55-94): normalize = 1
 *                replaces the softmax by o = ((q k^T) * scale / Nk) v (the "dot_product" instantiation; no q
 *                residual, PV_ERR_INVALID otherwise).  Head dims 256 / 512 (either mode) and 64 / 128 with
 *                normalize = 1 run csrc/pv_attention_wide.cu: the f16 wgmma + TMA kernel (PV_ATTN_WIDE) under the
 *                alignment rules above, its CUDA-core twin for f32 and everything else.  normalize = 0 keeps the
 *                routing and results of the head dims 32-128 unchanged; other head dims are PV_ERR_UNSUPPORTED.
 * ------------------------------------------------------------------------------------------- */
int pv_layernorm(const void* x, void* y, int dtype, long long rows, int groups, int C,
                 long long x_row_stride, long long y_row_stride, const float* gamma,
                 const float* beta, float eps, void* stream);
/* pv_layernorm with (a) several (gamma, beta) sets: group g of a row uses set g / groups_per_set (gamma / beta hold
 * groups / groups_per_set sets of C floats) - the pooled K and V of one block, adjacent channel slices of one buffer, are
 * normalised by ONE launch with norm_k | norm_v (attention.py:200-205); (b) an optional second source for every
 * npos-th row (row % npos == 0, read from cls_src + (row / npos) * cls_batch_stride): the cls token by-passes the
 * pooling conv (attention.py:184-186, 196-197) and is normalised with the pooled rows without a copy launch.     */
int pv_layernorm_sets(const void* x, void* y, int dtype, long long rows, int groups, int C,
                      long long x_row_stride, long long y_row_stride, const float* gamma, const float* beta,
                      int groups_per_set, const void* cls_src, long long cls_batch_stride, long long npos,
                      float eps, void* stream);
/* Strided row copy dst[r][0:C] = src[r][0:C] (cls-token rows around the pooling ops). */
int pv_copy_rows(const void* src, void* dst, int dtype, long long rows, int C,
                 long long src_row_stride, long long dst_row_stride, void* stream);
/* MViT cls token + positional encoding (layers/positional_encoding.py:112-136):
 *   y[b][0][:]   = pos[0][:]                      (pos[0] = cls_token + pos_embed_class, f32)
 *   y[b][1+i][:] = x[b][i][:] + pos[1+i][:]       (pos[1+i] = spatial[i %% HW] + temporal[i / HW])
 * x: [B][n_patch][C] (row stride x_row_stride), y: [B][1+n_patch][C] dense.                     */
int pv_add_pos_cls(const void* x, void* y, int dtype, int B, long long n_patch, int C,
                   long long x_row_stride, const float* pos, int has_cls, void* stream);
/* Same with separate dtypes: x f16 -> y f32 starts the fp32 residual trunk of the f16 engine (see pv_add_layernorm). */
int pv_add_pos_cls_to(const void* x, int x_dtype, void* y, int y_dtype, int B, long long n_patch, int C,
                      long long x_row_stride, const float* pos, int has_cls, void* stream);
/* Residual add + LayerNorm of MultiScaleBlock.forward (layers/attention.py:746-757: x = x_res + x_block; norm2(x); ...
 * x = x + x_mlp; the next block's norm1 at :730 / the model's norm_embed, models/vision_transformers.py:177) on an
 * fp32 trunk:  s = a + b in fp32 (a: a_dtype f16|f32, row stride a_row_stride; b: f16 branch output or NULL),
 *   sum[r][:] = s (fp32, optional - the residual stream never takes an f16 rounding),
 *   y[r][:]   = LayerNorm(s) * gamma + beta as f16 (optional - the A operand of the next GEMM), fp32 statistics.
 * C % 8 == 0, C <= 768; gamma / beta fp32, 16-byte aligned.                                                    */
int pv_add_layernorm(const void* a, int a_dtype, long long a_row_stride, const void* b, long long b_row_stride,
                     float* sum, long long sum_row_stride, void* y, long long y_row_stride, long long rows, int C,
                     const float* gamma, const float* beta, float eps, void* stream);
typedef struct pv_attention_desc {
  int dtype;
  int B, H, Nq, Nk, D;
  long long q_row_stride, k_row_stride, v_row_stride, o_row_stride; /* per token           */
  long long q_batch_stride, k_batch_stride, v_batch_stride, o_batch_stride;
  float scale;
  int add_q_residual;   /* residual_pool=True: o += q (cls row included, attention.py:535-536) */
  int normalize;        /* 0 = softmax (today's behaviour), 1 = divide by Nk */
} pv_attention_desc;
int pv_attention_fwd(const pv_attention_desc* d, const void* q, const void* k, const void* v,
                     void* o, void* stream);
/* Host-only routing query, the predicate pv_attention_fwd itself uses: which kernel it would launch for these
 * arguments (the pointers are only inspected for alignment), or a negative pv_status when it would refuse them. */
typedef enum pv_attention_kernel {
  PV_ATTN_WGMMA = 1,    /* f16 wgmma + TMA flash kernel                */
  PV_ATTN_MMA = 2,      /* f16 mma.sync flash kernel                   */
  PV_ATTN_SIMT = 3,     /* CUDA-core flash kernel (f16 or f32 storage) */
  PV_ATTN_WIDE = 4      /* f16 wgmma + TMA kernel for wide heads / the linear mode */
} pv_attention_kernel;
int pv_attention_kernel_for(const pv_attention_desc* d, const void* q, const void* k, const void* v, const void* o);
/* Key-masked softmax attention (models/masked_multistream.py:137-151, nn.MultiheadAttention with a key_padding_mask):
 * pv_attention_fwd with key j of sample b taking part only where key_valid[b * Nk + j] != 0 (u8 [B][Nk]).  A row whose
 * keys are all masked gets o = 0 and lse = -inf.  lse_out (optional, fp32 [B][H][Nq]) receives the log-sum-exp of the
 * scaled scores, max + log(sum), for pv_attention_weights.  Same routing as pv_attention_fwd (pv_attention_kernel_for
 * answers for both), head dims 32 / 64 / 96 / 128, softmax mode only (normalize = 1 or a q residual: PV_ERR_INVALID,
 * other head dims: PV_ERR_UNSUPPORTED).  The masked instances are their own kernels; the unmasked ones are unchanged.
 * pv_attention_weights: the head-averaged softmax nn.MultiheadAttention returns with need_weights=True,
 *   w[b][i][j] = mean_h exp(scale * q_bhi . k_bhj - lse[b][h][i])  for valid keys, 0 for masked ones (fp32 [B][Nq][Nk]),
 * recomputed from q / k and the lse of the forward (CUDA cores, fp32 maths).                                           */
int pv_attention_masked_fwd(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o,
                            const unsigned char* key_valid, float* lse_out, void* stream);
int pv_attention_weights(const pv_attention_desc* d, const void* q, const void* k, const unsigned char* key_valid,
                         const float* lse, float* w, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Masked sequence ops (models/masked_multistream.py, layers/fusion.py).  x: token rows [B][T][C] (row stride
 * x_row_stride, C % 8 == 0), mask: u8 [B][T] (non-zero = valid) or NULL = every step valid.
 * pv_masked_pool     : MaskedTemporalPooling (:35-93), fp32 accumulation, y [B][C]:
 *                      mode 0 max  (invalid steps -inf; a row with no valid step gives 0),
 *                      mode 1 avg  (masked sum / max(valid count, 1)), mode 2 sum (masked sum).
 * pv_masked_default  : LearnMaskedDefault (:170-190): y = x * any + def * (1 - any) in fp32, any = any(mask[b]);
 *                      x, y [B][C], def fp32 [C].
 * pv_mask_force_first: dst = src with column 0 set (mask[:, 0] = True of :137-141 / :309-313), u8 [B][T].
 * pv_reduce_fusion   : ReduceFusion (layers/fusion.py:104-141) y = max | sum | prod (op 0 | 1 | 2) over P <= 8
 *                      same-shaped row sets xs[p] (row strides x_row_strides[p]), fp32 maths, `rows` rows of C.
 * ------------------------------------------------------------------------------------------- */
int pv_masked_pool(const void* x, int dtype, long long x_row_stride, int B, int T, int C, const unsigned char* mask,
                   int mode, void* y, long long y_row_stride, void* stream);
int pv_masked_default(const void* x, int dtype, long long x_row_stride, int B, int C, const unsigned char* mask, int T,
                      const float* def, void* y, long long y_row_stride, void* stream);
int pv_mask_force_first(const unsigned char* src, unsigned char* dst, int B, int T, void* stream);
int pv_reduce_fusion(const void* const* xs, const long long* x_row_strides, int P, int dtype, long long rows, int C,
                     int op, void* y, long long y_row_stride, void* stream);
/* Masked LSTM recurrence (models/masked_multistream.py:193-256), all T steps of ndir (1 | 2) directions in one launch.
 * G: gate pre-activations x W_ih^T + b_ih + b_hh, [B][T] rows of g_row_stride elements, direction d at columns
 * d * 4H + gate * H + j (gate order i, f, g, o); w_hh_t: W_hh^T per direction, fp32 [ndir][H][4H]; mask: u8 [B][T] or
 * NULL.  Row b runs its first len_b = clamp(popcount(mask[b]), 1, T) steps (the reverse direction from len_b - 1 down
 * to 0) from h = c = 0 and writes y[b][d * H + j] = h_n; gates and c in fp32.  H <= 512, else PV_ERR_UNSUPPORTED.
 * f16 with H a multiple of 32: one thread-block cluster per (direction, 32-row batch slice), W_hh resident in shared
 * memory as f16 and a wgmma product per step with h as the f16 B operand (cluster size: the smallest S <= 16 with H / S
 * a multiple of 32, at most 128, and 8 H^2 / S bytes of weights within 128 KiB); other H and f32 read W_hh from global
 * memory every step and multiply on the CUDA cores.                                                               */
int pv_lstm_recurrence(const void* G, int dtype, long long g_row_stride, const float* w_hh_t, const unsigned char* mask,
                       int B, int T, int H, int ndir, void* y, long long y_row_stride, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Self-supervised objectives (models/simclr.py, byol.py, memory_bank.py) and the soft-target cross entropy
 * (losses/soft_target_cross_entropy.py), csrc/pv_contrastive.cu.  Embeddings, logits and losses are fp32; every
 * reduction runs in a fixed order (no atomics on values), so repeated calls are bitwise identical.  Row strides are in
 * elements.  row_loss is a caller-owned fp32 [rows] workspace that receives the per-row terms; loss one fp32.
 * pv_rows_l2_normalize : y[r] = x[r] / max(||x[r]||_2, 1e-12) (F.normalize(x, p=2, dim=1), simclr.py:43,48,
 *                        byol.py:112,122, memory_bank.py:90); x f16 | f32, y fp32.
 * pv_contrastive_ce    : mode 0 (SimCLR, simclr.py:51-65): logits q_n . k_m / temperature for the M <= 16384 key rows
 *                        (fp32 FMA, kept in shared memory), row_loss[n] = logsumexp_m - logit[n][row_offset + n],
 *                        loss = mean.  mode 1 (BYOL, byol.py:68-77): M == N, loss = -mean_n(q_n . k_n).
 * pv_memory_bank_ce    : memory_bank.py:92-103 for B samples: logits[b][j] = memory[idx[b][j]] . x[b] / temperature
 *                        over the K1 = neg_size + 1 indices of row b (int64 [B][K1], dense fp32 bank of bank_rows x dim,
 *                        64-bit offsets), row_loss[b] = logsumexp_j - logits[b][0], loss = mean.  logits is an fp32
 *                        [B][K1] workspace.  An index outside [0, bank_rows) sets *flag (device int, cleared by the
 *                        call) and its row is never read; the caller raises.  dim <= 12288.
 * pv_soft_target_ce    : soft_target_cross_entropy.py:66-81: t = target (t / (eps + sum t) with normalize),
 *                        row_loss[n] = sum_c -t_c * log_softmax(x[n])_c, and with reduce_mean loss = mean_n.
 *                        x f16 | f32, target f16 | f32 | PV_I64 (one-hot rows of int64).
 * pv_ema_update        : byol.py:93-101 over many tensors in one launch: dst[t][i] = dst[t][i] * mmt + src[t][i] *
 *                        one_minus_mmt, each product and the sum rounded once (no FMA).  dst / src / numel are DEVICE
 *                        arrays of the fp32 tensors; chunks[b] = (t << 40) | start names the 4096 elements of tensor t
 *                        from `start` that block b updates.
 * ------------------------------------------------------------------------------------------- */
int pv_rows_l2_normalize(const void* x, int dtype, long long x_row_stride, float* y, long long y_row_stride, int rows,
                         int C, void* stream);
int pv_contrastive_ce(const float* q, long long q_row_stride, const float* k, long long k_row_stride, int N, int M, int C,
                      float temperature, long long row_offset, int mode, float* row_loss, float* loss, void* stream);
int pv_memory_bank_ce(const float* x, long long x_row_stride, const float* memory, long long bank_rows, int dim,
                      const long long* idx, int B, int K1, float temperature, float* logits, float* row_loss, float* loss,
                      int* flag, void* stream);
int pv_soft_target_ce(const void* x, int x_dtype, long long x_row_stride, const void* target, int t_dtype,
                      long long t_row_stride, int N, int C, int normalize, float eps, int reduce_mean, float* row_loss,
                      float* loss, void* stream);
int pv_ema_update(float* const* dst, const float* const* src, const long long* numel, const long long* chunks,
                  int n_chunks, float mmt, float one_minus_mmt, void* stream);
/* pv_weights_refresh (byol.py:93-101 without a recompile: BYOL's momentum plan after pv_ema_update): rewrites a compiled
 * plan's constants in place, so a captured CUDA graph stays valid.  Gather: gather_jobs holds 5 int64 per constant
 * (dst pointer, PV_F16 | PV_F32, n elements, offset into map, source slot); dst[i] = map[off + i] < 0 ? 0 :
 * srcs[slot][map[off + i]] (fp32 sources, stored with one round to nearest even); gather_chunks[b] = (job << 40) | start
 * names the 4096 elements block b writes.  Fold: fold_jobs holds 9 int64 per BatchNorm fold (scale dst, bias dst, c_out,
 * conv_bias, gamma, beta, running_mean, running_var as device pointers or 0, eps as the bits of a double) and computes
 * packing.fold_bn in fp64, each operation correctly rounded, then fp32: the bytes of a fresh compile.  All tables are
 * DEVICE arrays.                                                                                                   */
int pv_weights_refresh(const long long* gather_jobs, const long long* gather_chunks, int n_gather_chunks, const int* map,
                       const float* const* srcs, const long long* fold_jobs, int n_fold_jobs, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Bank scans (csrc/pv_bank.cu): fp32 query rows q [N][dim] (row stride q_row_stride) against a dense fp32 bank
 * [M][dim] with 64-bit offsets.  Similarities are q . m with the dim terms summed in ascending order by fmaf; the
 * (N, M) matrix is never stored.  Repeated calls are bitwise identical.
 * pv_bank_workspace : bytes of the device workspace of pv_bank_topk (op 0) or pv_queue_ce (op 1) for N queries, an
 *                     M-row bank and k neighbours (pass k = 1 for op 1).  Host only.
 * pv_bank_topk      : ssl_helper.py:288-311 (KnnMemory.eval_knn): per query the k largest similarities, descending,
 *                     equal similarities by ascending bank index (-0 equals +0, NaN above +inf), into sim_out [N][k]
 *                     and idx_out [N][k] (int64); then preds [N][n_classes] = sum_i onehot(labels[idx_i]) *
 *                     exp(sim_i / temperature) in that order, each product and sum rounded once (a weight of +inf
 *                     makes the other classes NaN, as 0 * inf).  labels: int64 [M]; one outside [0, n_classes) sets
 *                     *flag (cleared by the call).  1 <= k <= min(1024, M), 1 <= dim <= 2048, M < 2^31.
 * pv_bank_update    : ssl_helper.py:245-250 (KnnMemory.update): memory[ind[n]] = v / max(|v|, 1e-12) elementwise with
 *                     v = x[n] * momentum + memory[ind[n]] * one_minus_momentum (two products and a sum, each rounded
 *                     once), from the rows as they were before the call; of repeated indices the last occurrence
 *                     wins.  An index outside [0, M) sets *flag (cleared by the call) and nothing is written.
 * pv_queue_ce       : cross entropy against target 0 (losses.py:125-134), row_loss and with reduce_mean its mean.
 *                     With logits == NULL, MoCo's objective (moco_v2.py:312-323): keys holds n_views blocks of N rows;
 *                     for every block v != skip_view (-1: none), in order, row (j, n) has the logits
 *                     [q_n . key_v,n, q_n . queue_0 .. q_n . queue_K-1] / temperature; the queue part of each query's
 *                     logsumexp is one streamed pass over queue [K][dim].  With logits != NULL: N materialised rows
 *                     of L logits, divided by temperature.                                                       */
int pv_bank_workspace(int op, int N, long long M, int k, long long* bytes);
int pv_bank_topk(const float* q, long long q_row_stride, int N, const float* memory, long long M, int dim, int k,
                 const long long* labels, int n_classes, float temperature, void* workspace, long long workspace_bytes,
                 float* sim_out, long long* idx_out, float* preds, int* flag, void* stream);
int pv_bank_update(const float* x, long long x_row_stride, int N, const long long* ind, float* memory, long long M,
                   int dim, float momentum, float one_minus_momentum, int* flag, void* stream);
int pv_queue_ce(const float* q, long long q_row_stride, int N, int dim, const float* queue, long long K,
                const float* keys, long long key_row_stride, int n_views, int skip_view, const float* logits,
                long long logits_row_stride, int L, float temperature, void* workspace, long long workspace_bytes,
                int reduce_mean, float* row_loss, float* loss, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Contrastive view colour augmentation (pytorchvideo_trainer datamodule/transforms.py ColorJitterVideoSSl): torchvision's
 * PIL ColorJitter, RandomGrayscale and Pillow's GaussianBlur on each clip stacked into one tall (n_t*H, W) RGB image,
 * in Pillow's integer and float arithmetic (blend in C float, RGB<->HSV with its double steps, 16-bit fixed-point luma,
 * 24-bit fixed-point box blur).  Every view k of the table reads the kept frames frame_idx[0..n_t) of source clip
 * views[k].clip at src[clip*s_clip + c*sc + frame*st + y*sh + x*sw] and is written as uint8 to
 * dst[k][3][n_t][H][W] (contiguous).  A source byte is the uint8 value itself (PV_U8), or for PV_F32 the truncation of
 * x*255 (src_scale 0: x in [0, 1], torchvision's ToPILImage) or of (x/255)*255 (src_scale 1: 0..255 values after
 * Div255), each step in fp32.
 *   pv_colorjitter_stats   zeroes sums[0..n_views) and adds, for each view whose ops include Contrast, the integer sum
 *                          of the luma over its stacked clip with the ops before Contrast applied (Contrast's mean).
 *   pv_colorjitter_apply   one thread per pixel: the view's ops in order, then grayscale, then the horizontal box-blur
 *                          passes of a blurred view on its rows in shared memory.
 *   pv_colorjitter_vblur   the vertical passes of the blurred views over the stacked image, in column strips kept in
 *                          shared memory, in place on dst.  Only the clip's first and last rows are image edges.
 * views and sums are DEVICE arrays; each entry point is one launch whatever the number of views.                 */
#define PV_CJ_BLUR_PASSES 3

typedef struct pv_cj_view {
  int clip;                          /* source clip                                                      */
  int n_ops;                         /* ColorJitter ops applied, 0..4                                    */
  int ops[4];                        /* in application order: 0 brightness, 1 contrast, 2 saturation, 3 hue */
  float factor[3];                   /* blend factors of brightness, contrast, saturation (Pillow's C float) */
  int hue_shift;                     /* byte added to H modulo 256                                       */
  int gray;                          /* RandomGrayscale: luma to all three channels                     */
  int blur_r;                        /* integer box radius; -1 = no blur                                 */
  unsigned int blur_ww, blur_fw;     /* box weights of the window and of its two edge pixels, in 2^-24    */
} pv_cj_view;

typedef struct pv_colorjitter_desc {
  int n_views, n_t, H, W;
  long long s_clip, sc, st, sh, sw;  /* source strides in elements                                       */
  int src_dtype;                     /* PV_U8 | PV_F32                                                   */
  int src_scale;                     /* PV_F32: 0 = values in [0, 1], 1 = values 0..255                  */
} pv_colorjitter_desc;

int pv_colorjitter_stats(const pv_colorjitter_desc* d, const void* src, const int32_t* frame_idx,
                         const pv_cj_view* views, unsigned long long* sums, void* stream);
int pv_colorjitter_apply(const pv_colorjitter_desc* d, const void* src, const int32_t* frame_idx,
                         const pv_cj_view* views, const unsigned long long* sums, uint8_t* dst, void* stream);
int pv_colorjitter_vblur(const pv_colorjitter_desc* d, const pv_cj_view* views, uint8_t* dst, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Baseline JPEG decode (csrc/pv_jpeg.cu), data/frame_video.py:242-245 (cv2.imdecode(IMREAD_COLOR) + BGR2RGB): the
 * bytes libjpeg's default decode gives - ISLOW integer IDCT with its range-limit table and 10-bit wrap, fancy
 * (triangle) upsampling with replicated edge rows / columns (plain replication when the chroma plane is at most 2
 * samples wide, as libjpeg does), integer YCbCr->RGB tables, grayscale replicated to three channels.
 *
 * pv_jpeg_parse  : host only.  Parses one stream (SOI, DQT, SOF0/SOF1 8-bit, DHT, SOS, DRI; APPn/COM and fill bytes
 *                  skipped), builds its Huffman lookup tables and appends it to *batch: frame->data_off is where the
 *                  caller must place the stream in the batch's data buffer, frame->out_off where its (H, W, 3) output
 *                  goes in out (elements), and the byte ranges [begin, end) of its sequential segments (restart
 *                  intervals, or the whole scan) are written as uint32 pairs, stream-relative, to
 *                  segs[2 * batch->n_segments ...] (capacity seg_cap pairs).  On error nothing of *batch changes.
 *                  Rejects with its own code each class below; malformed or truncated headers and a scan that runs
 *                  off the buffer are PV_ERR_INVALID.  PV_ERR_UNSUPPORTED: Huffman table slots 2 and 3 (SOF1 allows
 *                  four; baseline files use 0 and 1), and frames of more than 2^31 - 1 pixels.
 * pv_jpeg_decode : three launches on `stream` for every frame of the batch: entropy decode (one single-warp CTA per
 *                  segment, int16 coefficients in natural order), dequantise + ISLOW IDCT into per-component uint8 planes,
 *                  and upsample + YCbCr->RGB into out (uint8 or fp32, (H, W, 3) per frame at frames[i].out_off), one
 *                  launch per sampling mode present.  frames, segs, data and status are DEVICE arrays (frames and
 *                  segs as parse wrote them, data holding each stream at its data_off); batch is the host struct.
 *                  status[i] is zeroed by the call and set to PV_JPEG_BAD_* bits when frame i's entropy data is
 *                  corrupt (its output is then unspecified, but every read and write stays inside its ranges).
 *                  workspace: batch->ws_bytes bytes, 16-byte aligned.                                            */
typedef enum pv_jpeg_error {
  PV_JPEG_ERR_PROGRESSIVE = -20,
  PV_JPEG_ERR_ARITHMETIC = -21,
  PV_JPEG_ERR_LOSSLESS = -22,
  PV_JPEG_ERR_HIERARCHICAL = -23,
  PV_JPEG_ERR_PRECISION = -24,     /* sample precision other than 8 bits                                       */
  PV_JPEG_ERR_COMPONENTS = -25,    /* 2 or more than 4 components                                               */
  PV_JPEG_ERR_COLORSPACE = -26,    /* CMYK / YCCK (4 components), an Adobe transform other than YCbCr, RGB ids */
  PV_JPEG_ERR_ORIENTATION = -27,   /* EXIF orientation other than 1 (IMREAD_COLOR would rotate)                */
  PV_JPEG_ERR_MULTISCAN = -28,     /* more than one scan                                                       */
  PV_JPEG_ERR_DNL = -29,           /* height given by a DNL marker                                             */
  PV_JPEG_ERR_SAMPLING = -30       /* chroma sampling other than 1x1, 2x1, 1x2, 2x2 of the luma grid           */
} pv_jpeg_error;

#define PV_JPEG_BAD_CODE 1       /* status bit: a Huffman code absent from its table, or an AC run past 63     */
#define PV_JPEG_BAD_OVERRUN 2    /* status bit: a segment's codes need more bits than it holds                */
#define PV_JPEG_BAD_RESTART 4    /* status bit: RSTn out of sequence                                          */

typedef enum pv_jpeg_mode { PV_JPEG_GRAY = 0, PV_JPEG_H1V1 = 1, PV_JPEG_H2V1 = 2, PV_JPEG_H1V2 = 3, PV_JPEG_H2V2 = 4 } pv_jpeg_mode;

typedef struct pv_jpeg_huff {
  uint16_t look[512];                /* (length << 8) | symbol of every code of <= 9 bits by its 9-bit prefix, else 0 */
  int32_t maxcode[18];               /* largest code of each length, -1 if none; [17] is a sentinel                  */
  int32_t valoff[18];                /* symbol index minus code, per length                                          */
  uint8_t val[256];
} pv_jpeg_huff;

typedef struct pv_jpeg_frame {
  int width, height, ncomp, mode;    /* mode: pv_jpeg_mode                                                       */
  int mcus_x, mcus_y, restart_interval, n_segments;
  int n_blocks;                      /* 8x8 blocks of all components (padded to whole MCUs)                      */
  int scan_comp[3];                  /* SOF index of the scan's components, in scan order                         */
  int h[3], v[3];                    /* sampling factors, SOF order (1 for a grayscale frame)                      */
  int bw[3], bh[3];                  /* block grid of each component                                               */
  int dw[3], dh[3];                  /* real sample width / height of each component                               */
  int block_off[3];                  /* first block of each component within the frame                             */
  int dc_tbl[3], ac_tbl[3];          /* Huffman table slot of each component (0 | 1)                               */
  long long data_off;                /* the stream's first byte in the batch data buffer                          */
  long long seg_base;                /* first segment pair in segs                                                 */
  long long block_base;              /* first block in the workspace                                               */
  long long out_off;                 /* first output element                                                       */
  uint16_t qt[3][64];                /* quantisation table of each component, natural order                        */
  pv_jpeg_huff dc[2], ac[2];
} pv_jpeg_frame;

typedef struct pv_jpeg_batch {
  int n_frames;
  int mode_mask;                     /* 1 << pv_jpeg_mode of every frame                                         */
  int max_blocks, max_pixels;        /* largest n_blocks, largest width * height                                   */
  long long n_segments, n_blocks;
  long long data_bytes;              /* bytes of all streams                                                       */
  long long out_elems;               /* 3 * sum of width * height                                                  */
  long long ws_bytes;                /* workspace of pv_jpeg_decode: 192 bytes per block                           */
} pv_jpeg_batch;

int pv_jpeg_parse(const uint8_t* data, long long len, pv_jpeg_batch* batch, pv_jpeg_frame* frame, uint32_t* segs,
                  long long seg_cap);
int pv_jpeg_decode(const pv_jpeg_batch* batch, const pv_jpeg_frame* frames, const uint32_t* segs, const uint8_t* data,
                   void* workspace, long long workspace_bytes, void* out, int out_dtype, int* status, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PV_B200_H_ */

// MViT pooled attention, flash style: o = softmax((q*scale) k^T) v (+ q); the N_q x N_k score
// matrix never reaches HBM (reference layers/attention.py:531-539 materialises it).
//
// Generic CUDA-core kernel (f16 or f32 storage, fp32 maths, any head dim D <= 128 with D%32==0).
// A CTA owns ATT_BQ query rows of one (batch, head); K/V stream through shared memory in tiles
// of 32 keys; online softmax state (running max / sum / output) stays in registers.
#include "pv_common.cuh"

namespace pv {

constexpr int ATT_WARPS = 8;
constexpr int ATT_QPW = 4;                     // queries per warp
constexpr int ATT_BQ = ATT_WARPS * ATT_QPW;    // 32 queries per CTA
constexpr int ATT_BK = 32;                     // keys per tile

// MASKED: key j of sample b counts only where kv_valid[b * Nk + j] != 0; lse (optional) receives max + log(sum) per row.
template <typename T, int D, bool MASKED = false>
__global__ void __launch_bounds__(ATT_WARPS * 32)
attention_kernel(pv_attention_desc d, const T* __restrict__ q, const T* __restrict__ k,
                 const T* __restrict__ v, T* __restrict__ o,
                 const unsigned char* __restrict__ kv_valid = nullptr, float* __restrict__ lse = nullptr) {
  constexpr int DS = D + 1;            // padded smem row stride (floats)
  constexpr int NC = D / 32;           // output columns per lane
  extern __shared__ float sh[];
  float* Qs = sh;                      // [ATT_BQ][DS]
  float* Ks = Qs + ATT_BQ * DS;        // [ATT_BK][DS]
  float* Vs = Ks + ATT_BK * DS;        // [ATT_BK][DS]
  float* Ps = Vs + ATT_BK * DS;        // [ATT_WARPS][ATT_QPW][32]

  const int bh = blockIdx.y;
  const int b = bh / d.H, h = bh - b * d.H;
  const int q0 = blockIdx.x * ATT_BQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  const T* qb = q + (long long)b * d.q_batch_stride + (long long)h * D;
  const T* kb = k + (long long)b * d.k_batch_stride + (long long)h * D;
  const T* vb = v + (long long)b * d.v_batch_stride + (long long)h * D;
  T* ob = o + (long long)b * d.o_batch_stride + (long long)h * D;

  // stage the query tile (unscaled copy kept for the residual; scaled used for the scores)
  for (int e = threadIdx.x; e < ATT_BQ * D; e += blockDim.x) {
    const int r = e / D, c = e - r * D;
    const int qi = q0 + r;
    Qs[r * DS + c] = qi < d.Nq ? Elem<T>::ld(qb + (long long)qi * d.q_row_stride + c) : 0.f;
  }

  float m[ATT_QPW], l[ATT_QPW], acc[ATT_QPW][NC];
#pragma unroll
  for (int i = 0; i < ATT_QPW; ++i) {
    m[i] = -INFINITY; l[i] = 0.f;
#pragma unroll
    for (int c = 0; c < NC; ++c) acc[i][c] = 0.f;
  }

  for (int k0 = 0; k0 < d.Nk; k0 += ATT_BK) {
    __syncthreads();   // previous tile fully consumed (also covers the Q staging above)
    for (int e = threadIdx.x; e < ATT_BK * D; e += blockDim.x) {
      const int r = e / D, c = e - r * D;
      const int ki = k0 + r;
      float kv = 0.f, vv = 0.f;
      if (ki < d.Nk) {
        kv = Elem<T>::ld(kb + (long long)ki * d.k_row_stride + c);
        vv = Elem<T>::ld(vb + (long long)ki * d.v_row_stride + c);
      }
      Ks[r * DS + c] = kv;
      Vs[r * DS + c] = vv;
    }
    __syncthreads();
    bool key_ok = (k0 + lane) < d.Nk;
    if constexpr (MASKED) key_ok = key_ok && kv_valid[(long long)b * d.Nk + k0 + lane] != 0;
#pragma unroll
    for (int i = 0; i < ATT_QPW; ++i) {
      const float* qrow = Qs + (warp * ATT_QPW + i) * DS;
      const float* krow = Ks + lane * DS;
      float s = 0.f;
#pragma unroll 8
      for (int c = 0; c < D; ++c) s = fmaf(qrow[c] * d.scale, krow[c], s);
      s = key_ok ? s : -INFINITY;
      float mx = s;
      for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      const float m_new = fmaxf(m[i], mx);     // masked: -inf while no valid key was seen; p stays 0 then
      const float p = key_ok ? __expf(s - m_new) : 0.f;
      float ps = p;
      for (int off = 16; off; off >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, off);
      const float corr = (m[i] == -INFINITY) ? 0.f : __expf(m[i] - m_new);
      l[i] = l[i] * corr + ps;
      m[i] = m_new;
      float* prow = Ps + (warp * ATT_QPW + i) * 32;
      prow[lane] = p;
      __syncwarp();
#pragma unroll
      for (int c = 0; c < NC; ++c) acc[i][c] *= corr;
#pragma unroll 8
      for (int j = 0; j < ATT_BK; ++j) {
        const float pj = prow[j];
#pragma unroll
        for (int c = 0; c < NC; ++c) acc[i][c] = fmaf(pj, Vs[j * DS + lane + 32 * c], acc[i][c]);
      }
      __syncwarp();
    }
  }

#pragma unroll
  for (int i = 0; i < ATT_QPW; ++i) {
    const int qi = q0 + warp * ATT_QPW + i;
    if (qi >= d.Nq) continue;
    float inv = 1.f / l[i];
    if constexpr (MASKED) {          // a row without a valid key: o = 0, lse = -inf
      inv = l[i] > 0.f ? inv : 0.f;
      if (lse && lane == 0) lse[(long long)bh * d.Nq + qi] = l[i] > 0.f ? m[i] + logf(l[i]) : -INFINITY;
    }
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      float val = acc[i][c] * inv;
      if (d.add_q_residual) val += Qs[(warp * ATT_QPW + i) * DS + lane + 32 * c];
      Elem<T>::st(ob + (long long)qi * d.o_row_stride + lane + 32 * c, val);
    }
  }
}

template <typename T, int D, bool MASKED = false>
static int launch_attention(const pv_attention_desc* d, const void* q, const void* k, const void* v,
                            void* o, cudaStream_t s, const char* name, const unsigned char* kv_valid = nullptr,
                            float* lse = nullptr) {
  const size_t smem = (size_t)((ATT_BQ + 2 * ATT_BK) * (D + 1) + ATT_WARPS * ATT_QPW * 32) * sizeof(float);
  PV_OPT_IN_SMEM((attention_kernel<T, D, MASKED>), smem);
  dim3 grid((unsigned)cdiv(d->Nq, ATT_BQ), (unsigned)(d->B * d->H)), block(ATT_WARPS * 32);
  attention_kernel<T, D, MASKED><<<grid, block, smem, s>>>(*d, (const T*)q, (const T*)k, (const T*)v, (T*)o, kv_valid, lse);
  PV_LAUNCH_OK(name);
  return PV_OK;
}

int attention_wgmma_launch(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o,
                          cudaStream_t s);   // pv_attention_wgmma.cu
int attention_mma_launch(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o,
                         cudaStream_t s);    // pv_attention_mma.cu
int attention_wide_launch(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o,
                          cudaStream_t s);   // pv_attention_wide.cu
int attention_wide_simt_launch(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o,
                               cudaStream_t s);   // pv_attention_wide.cu
int attention_wgmma_masked_launch(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o,
                                  const unsigned char* kv_valid, float* lse, cudaStream_t s);   // pv_attention_wgmma.cu
int attention_mma_masked_launch(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o,
                                const unsigned char* kv_valid, float* lse, cudaStream_t s);     // pv_attention_mma.cu

// Head-averaged softmax weights of the masked forward: one CTA per (query i, sample b) stages the scaled query row and
// its lse per head; a thread per key recomputes the scores in fp32 from q / k and normalises them with the lse.  `vec`:
// 16-byte aligned k rows, read 8 elements at a time.
template <typename T>
__global__ void __launch_bounds__(128)
attention_weights_kernel(pv_attention_desc d, const T* __restrict__ q, const T* __restrict__ k,
                         const unsigned char* __restrict__ kv_valid, const float* __restrict__ lse,
                         float* __restrict__ w, int vec) {
  extern __shared__ float aw_q[];                      // [H * D] scaled query row, then [H] lse
  const int i = blockIdx.x, b = blockIdx.y;
  const int HD = d.H * d.D;
  float* ls = aw_q + HD;
  const T* qr = q + (long long)b * d.q_batch_stride + (long long)i * d.q_row_stride;
  for (int e = threadIdx.x; e < HD; e += blockDim.x) aw_q[e] = Elem<T>::ld(qr + e) * d.scale;
  for (int h = threadIdx.x; h < d.H; h += blockDim.x) ls[h] = lse[((long long)b * d.H + h) * d.Nq + i];
  __syncthreads();
  for (int j = threadIdx.x; j < d.Nk; j += blockDim.x) {
    float acc = 0.f;
    if (!kv_valid || kv_valid[(long long)b * d.Nk + j]) {
      const T* kr = k + (long long)b * d.k_batch_stride + (long long)j * d.k_row_stride;
      for (int h = 0; h < d.H; ++h) {
        if (ls[h] == -INFINITY) continue;
        const float* qh = aw_q + h * d.D;
        float s = 0.f;
        if (vec) {
          for (int c = 0; c < d.D; c += 8) {
            float v[8];
            ld8<T>(kr + h * d.D + c, v);
#pragma unroll
            for (int e = 0; e < 8; ++e) s = fmaf(qh[c + e], v[e], s);
          }
        } else {
          for (int c = 0; c < d.D; ++c) s = fmaf(qh[c], Elem<T>::ld(kr + h * d.D + c), s);
        }
        acc += __expf(s - ls[h]);
      }
    }
    w[((long long)b * d.Nq + i) * d.Nk + j] = acc / (float)d.H;
  }
}
// Calls the kernels of pv_attention_wide.cu take: head dims 256 / 512 in either mode, and the linear mode
// (normalize = 1) at 64 / 128.
static bool wide_family(const pv_attention_desc* d) {
  return d->D == 256 || d->D == 512 || d->normalize != 0;
}

// The f16 tensor-core kernels read q / k / v with 16-byte cp.async / TMA and 4-byte fragment loads from every batch,
// head and row start, and store o as __half2: pointers, row strides and batch strides must keep that alignment.  The
// wgmma kernel also describes q / k / v as [B][N][H*D] tensor maps, whose strides must be non-zero, must not make rows
// or samples overlap and must stay below 2^40 bytes; both tensor-core kernels share this rule, so every call it admits
// can be encoded.  With B == 1 the batch strides are never used and are not checked.
static bool tc_strides_ok(long long rs, long long bs, int n, const pv_attention_desc* d) {
  const long long limit = (1ll << 39);               // elements: 2^40 bytes of f16
  if (rs % 8 || rs < (long long)d->H * d->D || rs >= limit) return false;
  if (d->B == 1) return true;
  return bs % 8 == 0 && bs >= rs * n && bs < limit;
}
static bool tensor_core_aligned(const pv_attention_desc* d, const void* q, const void* k, const void* v, const void* o) {
  if (!tc_strides_ok(d->q_row_stride, d->q_batch_stride, d->Nq, d) || !tc_strides_ok(d->k_row_stride, d->k_batch_stride, d->Nk, d) ||
      !tc_strides_ok(d->v_row_stride, d->v_batch_stride, d->Nk, d))
    return false;
  if (d->o_row_stride % 2 || (d->B > 1 && d->o_batch_stride % 2)) return false;
  if ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v)) & 15) return false;
  return (reinterpret_cast<uintptr_t>(o) & 3) == 0;
}

}  // namespace pv

extern "C" int pv_attention_kernel_for(const pv_attention_desc* d, const void* q, const void* k, const void* v,
                                       const void* o) {
  PV_CHECK_ARG(d && q && k && v && o, "null argument");
  PV_CHECK_ARG(d->dtype == PV_F16 || d->dtype == PV_F32, "attention dtype must be f16|f32");
  PV_CHECK_ARG(d->B > 0 && d->H > 0 && d->Nq > 0 && d->Nk > 0, "empty attention problem");
  PV_CHECK_ARG((long long)d->B * d->H <= 65535, "B*H too large");
  PV_CHECK_ARG(d->normalize == 0 || d->normalize == 1, "attention normalize must be 0 (softmax) or 1 (divide by Nk)");
  PV_CHECK_ARG(!(d->normalize && d->add_q_residual), "attention normalize = 1 takes no q residual");
  if (d->D != 32 && d->D != 64 && d->D != 96 && d->D != 128 && d->D != 256 && d->D != 512) {
    pv::set_error("attention head dim %d unsupported (32/64/96/128/256/512)", d->D);
    return PV_ERR_UNSUPPORTED;
  }
  if (d->normalize && d->D != 64 && d->D != 128 && d->D != 256 && d->D != 512) {
    pv::set_error("linear attention (normalize = 1) head dim %d unsupported (64/128/256/512)", d->D);
    return PV_ERR_UNSUPPORTED;
  }
  const bool tc = d->dtype == PV_F16 && pv::tensor_core_aligned(d, q, k, v, o);
  if (pv::wide_family(d)) return tc ? PV_ATTN_WIDE : PV_ATTN_SIMT;
  if (tc) return d->D == 128 ? PV_ATTN_MMA : PV_ATTN_WGMMA;
  return PV_ATTN_SIMT;
}

extern "C" int pv_attention_fwd(const pv_attention_desc* d, const void* q, const void* k,
                                const void* v, void* o, void* stream) {
  const int kernel = pv_attention_kernel_for(d, q, k, v, o);
  if (kernel < 0) return kernel;
  cudaStream_t s = (cudaStream_t)stream;
  if (kernel == PV_ATTN_WGMMA) return pv::attention_wgmma_launch(d, q, k, v, o, s);
  if (kernel == PV_ATTN_MMA) return pv::attention_mma_launch(d, q, k, v, o, s);
  if (kernel == PV_ATTN_WIDE) return pv::attention_wide_launch(d, q, k, v, o, s);
  if (pv::wide_family(d)) return pv::attention_wide_simt_launch(d, q, k, v, o, s);
#define PV_ATT(DD)                                                                                         \
  if (d->D == DD)                                                                                           \
    return d->dtype == PV_F16                                                                               \
               ? pv::launch_attention<__half, DD>(d, q, k, v, o, s, "attention_kernel<__half," #DD ">")     \
               : pv::launch_attention<float, DD>(d, q, k, v, o, s, "attention_kernel<float," #DD ">");
  PV_ATT(32)
  PV_ATT(64)
  PV_ATT(96)
  PV_ATT(128)
#undef PV_ATT
  pv::set_error("internal: attention head dim %d", d->D);
  return PV_ERR_INVALID;
}

extern "C" int pv_attention_masked_fwd(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o,
                                       const unsigned char* key_valid, float* lse_out, void* stream) {
  PV_CHECK_ARG(key_valid, "null key mask");
  const int kernel = pv_attention_kernel_for(d, q, k, v, o);
  if (kernel < 0) return kernel;
  PV_CHECK_ARG(d->normalize == 0 && d->add_q_residual == 0, "masked attention is softmax only, without a q residual");
  if (pv::wide_family(d)) {
    pv::set_error("masked attention head dim %d unsupported (32/64/96/128)", d->D);
    return PV_ERR_UNSUPPORTED;
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (kernel == PV_ATTN_WGMMA) return pv::attention_wgmma_masked_launch(d, q, k, v, o, key_valid, lse_out, s);
  if (kernel == PV_ATTN_MMA) return pv::attention_mma_masked_launch(d, q, k, v, o, key_valid, lse_out, s);
#define PV_ATTM(DD)                                                                                              \
  if (d->D == DD)                                                                                                \
    return d->dtype == PV_F16                                                                                    \
               ? pv::launch_attention<__half, DD, true>(d, q, k, v, o, s, "attention_masked_kernel<__half," #DD ">", \
                                                        key_valid, lse_out)                                      \
               : pv::launch_attention<float, DD, true>(d, q, k, v, o, s, "attention_masked_kernel<float," #DD ">",   \
                                                       key_valid, lse_out);
  PV_ATTM(32)
  PV_ATTM(64)
  PV_ATTM(96)
  PV_ATTM(128)
#undef PV_ATTM
  pv::set_error("internal: masked attention head dim %d", d->D);
  return PV_ERR_INVALID;
}

extern "C" int pv_attention_weights(const pv_attention_desc* d, const void* q, const void* k, const unsigned char* key_valid,
                                    const float* lse, float* w, void* stream) {
  PV_CHECK_ARG(d && q && k && lse && w, "null argument");
  PV_CHECK_ARG(d->dtype == PV_F16 || d->dtype == PV_F32, "attention dtype must be f16|f32");
  PV_CHECK_ARG(d->B > 0 && d->H > 0 && d->Nq > 0 && d->Nk > 0 && d->D > 0, "empty attention problem");
  PV_CHECK_ARG(d->B <= 65535 && (long long)d->H * d->D <= 8192, "attention weights: B <= 65535, H * D <= 8192");
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid((unsigned)d->Nq, (unsigned)d->B);
  const size_t smem = (size_t)(d->H * d->D + d->H) * sizeof(float);
  const int vec = d->D % 8 == 0 && d->k_row_stride % 8 == 0 && (d->B == 1 || d->k_batch_stride % 8 == 0) &&
                  (reinterpret_cast<uintptr_t>(k) & 15) == 0;
  if (d->dtype == PV_F16) {
    pv::attention_weights_kernel<__half><<<grid, 128, smem, s>>>(*d, (const __half*)q, (const __half*)k, key_valid, lse, w,
                                                                 vec);
    PV_LAUNCH_OK("attention_weights_kernel<__half>");
  } else {
    pv::attention_weights_kernel<float><<<grid, 128, smem, s>>>(*d, (const float*)q, (const float*)k, key_valid, lse, w,
                                                                vec);
    PV_LAUNCH_OK("attention_weights_kernel<float>");
  }
  return PV_OK;
}

// Single-head attention with wide heads, the core of the Non-local block (reference layers/nonlocal_net.py:55-94):
//   softmax mode (normalize = 0):  o = softmax((q*scale) k^T) v (+ q)
//   linear mode  (normalize = 1):  o = ((q k^T) * scale / Nk) v           ("dot_product" instantiation, no softmax)
// The N_q x N_k score matrix never reaches memory.  Two kernels:
//
// attention_wide_kernel<D, DO, NWG, BK> (f16 storage, Hopper wgmma + TMA).  A CTA is NWG consumer warpgroups of 64
// query rows each, all sharing K / V tiles of BK keys that arrive by TMA (3-D tensor maps over [B][N][H*D], 32-dim
// chunks of 64 B, SWIZZLE_64B; rows past N are zero-filled) into a double buffer.  S = Q K^T is one m64nBK wgmma per
// 16 dims over the full head width D; the online softmax (or the linear scaling) runs on the S fragments in fp32
// registers; P is re-packed to f16 and O += P V takes it straight from registers (register-A wgmma) with V MN-major
// from shared memory.  The fp32 output accumulator of a thread holds DO / 2 values, so the output columns a CTA
// computes are limited to DO = 256 (128 registers): at D = 512 grid.z = 2 CTAs each own one half of the output
// columns and both compute S over the full D (1.5x the ideal tensor FLOPs, DESIGN.md section 2).
//
// attention_wide_simt_kernel<T, D> (f16 or f32 storage, fp32 maths on CUDA cores): the parity / fallback path for the
// same widths and for the linear mode, one warp per 4 queries, K / V tiles of 32 keys in shared memory.
#include "pv_common.cuh"
#include "pv_sm90.cuh"

#include <string.h>

namespace pv {

using namespace sm90;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_fn();   // pv_igemm.cu

struct AttnWideParams {
  CUtensorMap q_map, k_map, v_map;
  pv_attention_desc d;
};

__device__ __forceinline__ uint32_t awd_pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

template <int D, int DO, int NWG, int BK>
constexpr size_t wide_smem_bytes() {
  // 1 KB alignment slack + Q (NWG x 64 rows x D) + K (2 x BK x D) + V (2 x BK x DO) + 3 mbarriers
  return 1024 + (size_t)NWG * 64 * D * 2 + 2 * (size_t)BK * D * 2 + 2 * (size_t)BK * DO * 2 + 64;
}

template <int D, int DO, int NWG, int BK>
__global__ void __launch_bounds__(128 * NWG, 1)
attention_wide_kernel(const __grid_constant__ AttnWideParams P, const __half* __restrict__ q, __half* __restrict__ o) {
  static_assert(D % 32 == 0 && DO % 32 == 0 && D % DO == 0 && DO <= 256, "head / output width");
  static_assert(BK == 32 || BK == 64, "key tile");
  constexpr int NCD = D / 32, NCO = DO / 32;          // 32-dim chunks of the q.k width and of the output width
  constexpr uint32_t QCH = 64 * 64, KCH = BK * 64;     // bytes of one chunk: [64 | BK rows x 32 f16], swizzle 64 B
  constexpr uint32_t QT = NCD * QCH, KT = NCD * KCH, VT = NCO * KCH;
  constexpr int NS = BK / 2;                           // S fragment registers (m64nBK)
  extern __shared__ uint8_t awd_smem[];
  const uint32_t base = (smem_u32(awd_smem) + 1023u) & ~1023u;
  const uint32_t q_s = base, k_s = q_s + NWG * QT, v_s = k_s + 2 * KT;
  const uint32_t bar = v_s + 2 * VT;                   // qbar, kvbar[2]
  const pv_attention_desc& d = P.d;

  const int bh = blockIdx.y;
  const int b = bh / d.H, h = bh - b * d.H;
  const int q0 = blockIdx.x * (64 * NWG);
  const int vo = blockIdx.z * DO;                      // first output column of this CTA
  const int wg = threadIdx.x >> 7;
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int ntiles = (d.Nk + BK - 1) / BK;
  const bool linear = d.normalize != 0;
  const float smul = linear ? d.scale / (float)d.Nk : d.scale;

  auto load_kv = [&](int kt, int buf) {
    const uint32_t bb = bar + 8u * (1 + buf);
    mbar_arrive_expect_tx(bb, KT + VT);
    for (int c = 0; c < NCD; ++c) tma_load_3d(k_s + buf * KT + c * KCH, &P.k_map, bb, h * D + c * 32, kt * BK, b);
    for (int c = 0; c < NCO; ++c) tma_load_3d(v_s + buf * VT + c * KCH, &P.v_map, bb, h * D + vo + c * 32, kt * BK, b);
  };
  if (threadIdx.x == 0) {
    prefetch_tmap(&P.q_map); prefetch_tmap(&P.k_map); prefetch_tmap(&P.v_map);
    for (int i = 0; i < 3; ++i) mbar_init(bar + 8u * i, 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(bar, NWG * QT);
    for (int w = 0; w < NWG; ++w)
      for (int c = 0; c < NCD; ++c) tma_load_3d(q_s + w * QT + c * QCH, &P.q_map, bar, h * D + c * 32, q0 + 64 * w, b);
    load_kv(0, 0);
  }
  __syncthreads();

  float sacc[NS];                                      // S: 64 x BK, wgmma fragment (row warp*16 + g (+8), col 8j + 2t (+1))
  float oacc[NCO][16];                                 // O: per 32-dim output chunk, 64 x 32
#pragma unroll
  for (int c = 0; c < NCO; ++c)
#pragma unroll
    for (int i = 0; i < 16; ++i) oacc[c][i] = 0.f;
#pragma unroll
  for (int i = 0; i < NS; ++i) sacc[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows g and g+8 (l: per-thread partial)
  const uint32_t my_q = q_s + wg * QT;

  mbar_wait(bar, 0);
  for (int kt = 0; kt < ntiles; ++kt) {
    const int buf = kt & 1;
    if (threadIdx.x == 0 && kt + 1 < ntiles) load_kv(kt + 1, buf ^ 1);   // buf ^ 1 was released by the barrier below
    mbar_wait(bar + 8u * (1 + buf), (uint32_t)((kt >> 1) & 1));

    // ---- S = Q K^T over the full width D
    acc_fence(sacc);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < NCD; ++c) {
      const uint64_t qd = make_kmajor_desc(my_q + c * QCH, 64);
      const uint64_t kd = make_kmajor_desc(k_s + buf * KT + c * KCH, 64);
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) Wgmma<BK>::mma(sacc, qd + (uint64_t)(2 * ks), kd + (uint64_t)(2 * ks), (c | ks) != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(sacc);

    // ---- scale, mask the key tail; softmax: online max / correction; linear: p = s * scale / Nk
    const int kbase = kt * BK + 2 * t;
    float c0 = 1.f, c1 = 1.f;
    if (linear) {
#pragma unroll
      for (int nt = 0; nt < BK / 8; ++nt) {
        const int key = kbase + nt * 8;
#pragma unroll
        for (int e = 0; e < 4; ++e) sacc[4 * nt + e] = (key + (e & 1)) < d.Nk ? sacc[4 * nt + e] * smul : 0.f;
      }
    } else {
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < BK / 8; ++nt) {
        const int key = kbase + nt * 8;
#pragma unroll
        for (int e = 0; e < 4; ++e) sacc[4 * nt + e] = (key + (e & 1)) < d.Nk ? sacc[4 * nt + e] * smul : -INFINITY;
        mx0 = fmaxf(mx0, fmaxf(sacc[4 * nt], sacc[4 * nt + 1]));
        mx1 = fmaxf(mx1, fmaxf(sacc[4 * nt + 2], sacc[4 * nt + 3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);     // finite: every tile has >= 1 valid key
      c0 = (m0 == -INFINITY) ? 0.f : __expf(m0 - mn0);
      c1 = (m1 == -INFINITY) ? 0.f : __expf(m1 - mn1);
      m0 = mn0; m1 = mn1;
      float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
      for (int nt = 0; nt < BK / 8; ++nt) {
        sacc[4 * nt] = __expf(sacc[4 * nt] - mn0); sacc[4 * nt + 1] = __expf(sacc[4 * nt + 1] - mn0);
        sacc[4 * nt + 2] = __expf(sacc[4 * nt + 2] - mn1); sacc[4 * nt + 3] = __expf(sacc[4 * nt + 3] - mn1);
        ps0 += sacc[4 * nt] + sacc[4 * nt + 1];
        ps1 += sacc[4 * nt + 2] + sacc[4 * nt + 3];
      }
      l0 = l0 * c0 + ps0;
      l1 = l1 * c1 + ps1;
#pragma unroll
      for (int c = 0; c < NCO; ++c)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          oacc[c][4 * j] *= c0; oacc[c][4 * j + 1] *= c0; oacc[c][4 * j + 2] *= c1; oacc[c][4 * j + 3] *= c1;
        }
    }

    // ---- O += P V: P (f16) from registers, V MN-major (8-key groups 512 B apart inside a 32-dim chunk)
    uint32_t pa[BK / 16][4];
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) {
      pa[kk][0] = awd_pack_h2(sacc[8 * kk], sacc[8 * kk + 1]);
      pa[kk][1] = awd_pack_h2(sacc[8 * kk + 2], sacc[8 * kk + 3]);
      pa[kk][2] = awd_pack_h2(sacc[8 * kk + 4], sacc[8 * kk + 5]);
      pa[kk][3] = awd_pack_h2(sacc[8 * kk + 6], sacc[8 * kk + 7]);
    }
#pragma unroll
    for (int c = 0; c < NCO; ++c) acc_fence(oacc[c]);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < NCO; ++c)
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk) {
        const uint32_t vaddr = v_s + buf * VT + c * KCH + (uint32_t)kk * 16u * 64u;
        WgmmaRS<32, 1>::mma(oacc[c], pa[kk], make_noswz_desc(vaddr, 512u, 512u) | (2ull << 62), 1u);
      }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < NCO; ++c) acc_fence(oacc[c]);
    __syncthreads();     // every warp is done with `buf` before thread 0 refills it next iteration
  }

  // ---- finalise: softmax row sums across the 4 lanes of a row, normalise, (+q), store
  float i0 = 1.f, i1 = 1.f;
  if (!linear) {
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    i0 = 1.f / l0; i1 = 1.f / l1;
  }
  const int qa = q0 + wg * 64 + warp * 16 + g, qb8 = qa + 8;
  const __half* qb = q + (long long)b * d.q_batch_stride + (long long)h * D + vo;
  __half* ob = o + (long long)b * d.o_batch_stride + (long long)h * D + vo;
#pragma unroll
  for (int c = 0; c < NCO; ++c)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int col = c * 32 + j * 8 + 2 * t;
      if (qa < d.Nq) {
        float x0 = oacc[c][4 * j] * i0, x1 = oacc[c][4 * j + 1] * i0;
        if (d.add_q_residual) {
          const float2 r = __half22float2(*reinterpret_cast<const __half2*>(qb + (long long)qa * d.q_row_stride + col));
          x0 += r.x; x1 += r.y;
        }
        *reinterpret_cast<__half2*>(ob + (long long)qa * d.o_row_stride + col) = __floats2half2_rn(x0, x1);
      }
      if (qb8 < d.Nq) {
        float x2 = oacc[c][4 * j + 2] * i1, x3 = oacc[c][4 * j + 3] * i1;
        if (d.add_q_residual) {
          const float2 r = __half22float2(*reinterpret_cast<const __half2*>(qb + (long long)qb8 * d.q_row_stride + col));
          x2 += r.x; x3 += r.y;
        }
        *reinterpret_cast<__half2*>(ob + (long long)qb8 * d.o_row_stride + col) = __floats2half2_rn(x2, x3);
      }
    }
}

// [B][N][H*D] f16 with the given row / batch strides (elements) -> 3-D map, box [32 dims, rows, 1], SWIZZLE_64B
static bool awd_encode(EncodeTiledFn encode, CUtensorMap* m, const void* p, const pv_attention_desc* d, int n, long long rs,
                       long long bs, uint32_t rows) {
  cuuint64_t gdim[3] = {(cuuint64_t)d->H * d->D, (cuuint64_t)n, (cuuint64_t)d->B};
  // one sample: the batch stride is never stepped over, give the map a valid one
  cuuint64_t gstr[2] = {(cuuint64_t)rs * 2, (cuuint64_t)(d->B == 1 ? rs * n : bs) * 2};
  cuuint32_t box[3] = {32, rows, 1}, estr[3] = {1, 1, 1};
  return encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(p), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int D, int DO, int NWG, int BK>
static int launch_attention_wide(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o, cudaStream_t s,
                                 const char* name) {
  EncodeTiledFn encode = get_encode_fn();
  if (!encode) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return PV_ERR_CUDA; }
  AttnWideParams P;
  memset(&P, 0, sizeof(P));
  P.d = *d;
  if (!awd_encode(encode, &P.q_map, q, d, d->Nq, d->q_row_stride, d->q_batch_stride, 64) ||
      !awd_encode(encode, &P.k_map, k, d, d->Nk, d->k_row_stride, d->k_batch_stride, BK) ||
      !awd_encode(encode, &P.v_map, v, d, d->Nk, d->v_row_stride, d->v_batch_stride, BK)) {
    set_error("cuTensorMapEncodeTiled(wide attention q/k/v) failed");
    return PV_ERR_CUDA;
  }
  constexpr size_t smem = wide_smem_bytes<D, DO, NWG, BK>();
  static_assert(smem <= 227 * 1024, "shared memory");
  PV_OPT_IN_SMEM((attention_wide_kernel<D, DO, NWG, BK>), smem);
  dim3 grid((unsigned)cdiv(d->Nq, 64 * NWG), (unsigned)(d->B * d->H), (unsigned)(D / DO)), block(128 * NWG);
  attention_wide_kernel<D, DO, NWG, BK><<<grid, block, smem, s>>>(P, (const __half*)q, (__half*)o);
  PV_LAUNCH_OK(name);
  return PV_OK;
}

// ---- CUDA-core kernel -----------------------------------------------------------------------------------------
constexpr int AWS_WARPS = 8;
constexpr int AWS_QPW = 4;                       // queries per warp
constexpr int AWS_BQ = AWS_WARPS * AWS_QPW;      // 32 queries per CTA
constexpr int AWS_BK = 32;                       // keys per tile

template <typename T, int D>
__global__ void __launch_bounds__(AWS_WARPS * 32)
attention_wide_simt_kernel(pv_attention_desc d, const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v,
                           T* __restrict__ o) {
  constexpr int DS = D + 1;            // padded smem row stride (floats)
  constexpr int NC = D / 32;           // output columns per lane
  extern __shared__ float aws_sh[];
  float* Qs = aws_sh;                  // [AWS_BQ][DS]
  float* Ks = Qs + AWS_BQ * DS;        // [AWS_BK][DS]
  float* Vs = Ks + AWS_BK * DS;        // [AWS_BK][DS]
  float* Ps = Vs + AWS_BK * DS;        // [AWS_WARPS][AWS_QPW][32]

  const int bh = blockIdx.y;
  const int b = bh / d.H, h = bh - b * d.H;
  const int q0 = blockIdx.x * AWS_BQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool linear = d.normalize != 0;
  const float smul = linear ? d.scale / (float)d.Nk : d.scale;

  const T* qb = q + (long long)b * d.q_batch_stride + (long long)h * D;
  const T* kb = k + (long long)b * d.k_batch_stride + (long long)h * D;
  const T* vb = v + (long long)b * d.v_batch_stride + (long long)h * D;
  T* ob = o + (long long)b * d.o_batch_stride + (long long)h * D;

  for (int e = threadIdx.x; e < AWS_BQ * D; e += blockDim.x) {
    const int r = e / D, c = e - r * D;
    const int qi = q0 + r;
    Qs[r * DS + c] = qi < d.Nq ? Elem<T>::ld(qb + (long long)qi * d.q_row_stride + c) : 0.f;
  }

  float m[AWS_QPW], l[AWS_QPW], acc[AWS_QPW][NC];
#pragma unroll
  for (int i = 0; i < AWS_QPW; ++i) {
    m[i] = -INFINITY; l[i] = 0.f;
#pragma unroll
    for (int c = 0; c < NC; ++c) acc[i][c] = 0.f;
  }

  for (int k0 = 0; k0 < d.Nk; k0 += AWS_BK) {
    __syncthreads();   // previous tile fully consumed (also covers the Q staging above)
    for (int e = threadIdx.x; e < AWS_BK * D; e += blockDim.x) {
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
    const bool key_ok = (k0 + lane) < d.Nk;
#pragma unroll
    for (int i = 0; i < AWS_QPW; ++i) {
      const float* qrow = Qs + (warp * AWS_QPW + i) * DS;
      const float* krow = Ks + lane * DS;
      float s = 0.f;
#pragma unroll 8
      for (int c = 0; c < D; ++c) s = fmaf(qrow[c], krow[c], s);
      s *= smul;
      float p, corr = 1.f;
      if (linear) {
        p = key_ok ? s : 0.f;
      } else {
        s = key_ok ? s : -INFINITY;
        float mx = s;
        for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
        const float m_new = fmaxf(m[i], mx);
        p = key_ok ? __expf(s - m_new) : 0.f;
        float ps = p;
        for (int off = 16; off; off >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, off);
        corr = (m[i] == -INFINITY) ? 0.f : __expf(m[i] - m_new);
        l[i] = l[i] * corr + ps;
        m[i] = m_new;
      }
      float* prow = Ps + (warp * AWS_QPW + i) * 32;
      prow[lane] = p;
      __syncwarp();
#pragma unroll
      for (int c = 0; c < NC; ++c) acc[i][c] *= corr;
#pragma unroll 8
      for (int j = 0; j < AWS_BK; ++j) {
        const float pj = prow[j];
#pragma unroll
        for (int c = 0; c < NC; ++c) acc[i][c] = fmaf(pj, Vs[j * DS + lane + 32 * c], acc[i][c]);
      }
      __syncwarp();
    }
  }

#pragma unroll
  for (int i = 0; i < AWS_QPW; ++i) {
    const int qi = q0 + warp * AWS_QPW + i;
    if (qi >= d.Nq) continue;
    const float inv = linear ? 1.f : 1.f / l[i];
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      float val = acc[i][c] * inv;
      if (d.add_q_residual) val += Qs[(warp * AWS_QPW + i) * DS + lane + 32 * c];
      Elem<T>::st(ob + (long long)qi * d.o_row_stride + lane + 32 * c, val);
    }
  }
}

template <typename T, int D>
static int launch_attention_wide_simt(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o,
                                      cudaStream_t s, const char* name) {
  constexpr size_t smem = (size_t)((AWS_BQ + 2 * AWS_BK) * (D + 1) + AWS_WARPS * AWS_QPW * 32) * sizeof(float);
  static_assert(smem <= 227 * 1024, "shared memory");
  PV_OPT_IN_SMEM((attention_wide_simt_kernel<T, D>), smem);
  dim3 grid((unsigned)cdiv(d->Nq, AWS_BQ), (unsigned)(d->B * d->H)), block(AWS_WARPS * 32);
  attention_wide_simt_kernel<T, D><<<grid, block, smem, s>>>(*d, (const T*)q, (const T*)k, (const T*)v, (T*)o);
  PV_LAUNCH_OK(name);
  return PV_OK;
}

// f16 tensor-core path for head dims 256 / 512 (either mode) and 64 / 128 (linear mode); pv_attention_fwd
// (pv_attention.cu) has checked the alignment of pointers and strides.
int attention_wide_launch(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o, cudaStream_t s) {
#define PV_AWIDE(DD, DO, NWG, BK)                                                                                   \
  if (d->D == DD)                                                                                                  \
    return launch_attention_wide<DD, DO, NWG, BK>(d, q, k, v, o, s, "attention_wide_kernel<" #DD "," #DO ">");
  PV_AWIDE(64, 64, 2, 64)
  PV_AWIDE(128, 128, 2, 64)
  PV_AWIDE(256, 256, 2, 64)
  PV_AWIDE(512, 256, 2, 32)
#undef PV_AWIDE
  set_error("internal: wide attention head dim %d", d->D);
  return PV_ERR_INVALID;
}

// CUDA-core path for the same widths and modes: f32 storage, and f16 calls the tensor-core kernel cannot take.
int attention_wide_simt_launch(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o,
                               cudaStream_t s) {
#define PV_AWS(DD)                                                                                                   \
  if (d->D == DD)                                                                                                    \
    return d->dtype == PV_F16                                                                                        \
               ? launch_attention_wide_simt<__half, DD>(d, q, k, v, o, s, "attention_wide_simt_kernel<__half," #DD ">") \
               : launch_attention_wide_simt<float, DD>(d, q, k, v, o, s, "attention_wide_simt_kernel<float," #DD ">");
  PV_AWS(64)
  PV_AWS(128)
  PV_AWS(256)
  PV_AWS(512)
#undef PV_AWS
  set_error("internal: wide attention head dim %d", d->D);
  return PV_ERR_INVALID;
}

}  // namespace pv

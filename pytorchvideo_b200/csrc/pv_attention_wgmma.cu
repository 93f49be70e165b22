// Flash-style pooled attention of MViT (layers/attention.py:531-539) on Hopper wgmma, f16 storage:
//   o = softmax((q*scale) k^T) v (+ q)
// One CTA = one warpgroup = 64 query rows of one (batch, head).  Q and double-buffered 64-key K / V tiles arrive by
// TMA (3-D tensor maps over [B][N][H*D], 32-dim chunks of 64 B, SWIZZLE_64B; rows past N are zero-filled) on
// mbarriers.  S = Q K^T is one m64n64 wgmma per 16 dims (both operands K-major in shared memory); the online softmax
// runs on the S fragments in registers; O += P V takes P straight from registers (register-A wgmma, the P fragment is
// the S accumulator layout re-packed to f16) and V MN-major from shared memory as it lies in memory, one m64n32 wgmma
// per 32-dim chunk and 16 keys.  Head dims 32 / 64 / 96; D = 128 uses the mma.sync kernel (pv_attention_mma.cu).
#include "pv_common.cuh"
#include "pv_sm90.cuh"

#include <string.h>

namespace pv {

using namespace sm90;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_fn();   // pv_igemm.cu

constexpr int AW_BQ = 64, AW_BK = 64;
constexpr uint32_t AW_CHUNK = 64 * 64;      // [64 rows x 32 f16] swizzle-64B chunk

struct AttnWgParams {
  CUtensorMap q_map, k_map, v_map;
  pv_attention_desc d;
};

__device__ __forceinline__ uint32_t aw_pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// MASKED: key j of sample b counts only where kv_valid[b * Nk + j] != 0; lse (optional) receives max + log(sum) per row.
template <int D, bool MASKED = false>
__global__ void __launch_bounds__(128, 1)
attention_wgmma_kernel(const __grid_constant__ AttnWgParams P, const __half* __restrict__ q, __half* __restrict__ o,
                       const unsigned char* __restrict__ kv_valid = nullptr, float* __restrict__ lse = nullptr) {
  constexpr int NC = D / 32;                          // 32-dim chunks
  constexpr uint32_t TILE = NC * AW_CHUNK;            // one Q / K / V tile
  extern __shared__ uint8_t aw_smem[];
  const uint32_t base = (smem_u32(aw_smem) + 1023u) & ~1023u;
  const uint32_t q_s = base, k_s = base + TILE, v_s = base + 3 * TILE;   // K / V: two buffers each
  const uint32_t bar = base + 5 * TILE;               // qbar, kvbar[2]
  const pv_attention_desc& d = P.d;

  const int bh = blockIdx.y;
  const int b = bh / d.H, h = bh - b * d.H;
  const int q0 = blockIdx.x * AW_BQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int ntiles = (d.Nk + AW_BK - 1) / AW_BK;

  auto load_kv = [&](int kt, int buf) {
    const uint32_t bb = bar + 8u * (1 + buf);
    mbar_arrive_expect_tx(bb, 2 * TILE);
    for (int c = 0; c < NC; ++c) {
      tma_load_3d(k_s + buf * TILE + c * AW_CHUNK, &P.k_map, bb, h * D + c * 32, kt * AW_BK, b);
      tma_load_3d(v_s + buf * TILE + c * AW_CHUNK, &P.v_map, bb, h * D + c * 32, kt * AW_BK, b);
    }
  };
  if (threadIdx.x == 0) {
    prefetch_tmap(&P.q_map); prefetch_tmap(&P.k_map); prefetch_tmap(&P.v_map);
    for (int i = 0; i < 3; ++i) mbar_init(bar + 8u * i, 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(bar, TILE);
    for (int c = 0; c < NC; ++c) tma_load_3d(q_s + c * AW_CHUNK, &P.q_map, bar, h * D + c * 32, q0, b);
    load_kv(0, 0);
  }
  __syncthreads();

  float sacc[32];                                      // S: 64 x 64, wgmma fragment (row warp*16 + g (+8), col 8j + 2t (+1))
  float oacc[NC][16];                                  // O: per 32-dim chunk, 64 x 32
#pragma unroll
  for (int c = 0; c < NC; ++c)
#pragma unroll
    for (int i = 0; i < 16; ++i) oacc[c][i] = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) sacc[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows g and g+8 (l: per-thread partial)

  mbar_wait(bar, 0);
  for (int kt = 0; kt < ntiles; ++kt) {
    const int buf = kt & 1;
    if (threadIdx.x == 0 && kt + 1 < ntiles) load_kv(kt + 1, buf ^ 1);   // buf ^ 1 was released by the barrier below
    mbar_wait(bar + 8u * (1 + buf), (uint32_t)((kt >> 1) & 1));

    // ---- S = Q K^T
    acc_fence(sacc);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const uint64_t qd = make_kmajor_desc(q_s + c * AW_CHUNK, 64);
      const uint64_t kd = make_kmajor_desc(k_s + buf * TILE + c * AW_CHUNK, 64);
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) Wgmma<64>::mma(sacc, qd + (uint64_t)(2 * ks), kd + (uint64_t)(2 * ks), (c | ks) != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(sacc);

    // ---- scale, mask the key tail, online softmax
    const int kbase = kt * AW_BK + 2 * t;
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int key = kbase + nt * 8;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        bool ok = (key + (e & 1)) < d.Nk;
        if constexpr (MASKED) ok = ok && kv_valid[(long long)b * d.Nk + key + (e & 1)] != 0;
        sacc[4 * nt + e] = ok ? sacc[4 * nt + e] * d.scale : -INFINITY;
      }
      mx0 = fmaxf(mx0, fmaxf(sacc[4 * nt], sacc[4 * nt + 1]));
      mx1 = fmaxf(mx1, fmaxf(sacc[4 * nt + 2], sacc[4 * nt + 3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);     // unmasked: finite, every tile has >= 1 valid key
    const float c0 = (m0 == -INFINITY) ? 0.f : __expf(m0 - mn0);
    const float c1 = (m1 == -INFINITY) ? 0.f : __expf(m1 - mn1);
    m0 = mn0; m1 = mn1;
    // masked: no valid key so far leaves the maximum at -inf; subtract 0 then, never -inf - -inf
    const float e0 = (MASKED && mn0 == -INFINITY) ? 0.f : mn0, e1 = (MASKED && mn1 == -INFINITY) ? 0.f : mn1;
    float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      sacc[4 * nt] = __expf(sacc[4 * nt] - e0); sacc[4 * nt + 1] = __expf(sacc[4 * nt + 1] - e0);
      sacc[4 * nt + 2] = __expf(sacc[4 * nt + 2] - e1); sacc[4 * nt + 3] = __expf(sacc[4 * nt + 3] - e1);
      ps0 += sacc[4 * nt] + sacc[4 * nt + 1];
      ps1 += sacc[4 * nt + 2] + sacc[4 * nt + 3];
    }
    l0 = l0 * c0 + ps0;
    l1 = l1 * c1 + ps1;
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        oacc[c][4 * j] *= c0; oacc[c][4 * j + 1] *= c0; oacc[c][4 * j + 2] *= c1; oacc[c][4 * j + 3] *= c1;
      }

    // ---- O += P V: P (f16) from registers, V MN-major (8-key groups 512 B apart inside a 32-dim chunk)
    uint32_t pa[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      pa[kk][0] = aw_pack_h2(sacc[8 * kk], sacc[8 * kk + 1]);
      pa[kk][1] = aw_pack_h2(sacc[8 * kk + 2], sacc[8 * kk + 3]);
      pa[kk][2] = aw_pack_h2(sacc[8 * kk + 4], sacc[8 * kk + 5]);
      pa[kk][3] = aw_pack_h2(sacc[8 * kk + 6], sacc[8 * kk + 7]);
    }
#pragma unroll
    for (int c = 0; c < NC; ++c) acc_fence(oacc[c]);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t vaddr = v_s + buf * TILE + c * AW_CHUNK + (uint32_t)kk * 16u * 64u;
        WgmmaRS<32, 1>::mma(oacc[c], pa[kk], make_noswz_desc(vaddr, 512u, 512u) | (2ull << 62), 1u);
      }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < NC; ++c) acc_fence(oacc[c]);
    __syncthreads();     // every warp is done with `buf` before thread 0 refills it next iteration
  }

  // ---- finalise: row sums across the 4 lanes of a row, normalise, (+q), store
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  float i0 = 1.f / l0, i1 = 1.f / l1;
  const int qa = q0 + warp * 16 + g, qb8 = qa + 8;
  if constexpr (MASKED) {          // a row without a valid key: o = 0, lse = -inf
    i0 = l0 > 0.f ? i0 : 0.f;
    i1 = l1 > 0.f ? i1 : 0.f;
    if (lse && t == 0) {
      float* lr = lse + (long long)bh * d.Nq;
      if (qa < d.Nq) lr[qa] = l0 > 0.f ? m0 + logf(l0) : -INFINITY;
      if (qb8 < d.Nq) lr[qb8] = l1 > 0.f ? m1 + logf(l1) : -INFINITY;
    }
  }
  const __half* qb = q + (long long)b * d.q_batch_stride + (long long)h * D;
  __half* ob = o + (long long)b * d.o_batch_stride + (long long)h * D;
#pragma unroll
  for (int c = 0; c < NC; ++c)
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

// [B][N][H*D] f16 with the given row / batch strides (elements) -> 3-D map, box [32 dims, 64 rows, 1], SWIZZLE_64B
static bool aw_encode(EncodeTiledFn encode, CUtensorMap* m, const void* p, const pv_attention_desc* d, int n, long long rs, long long bs) {
  cuuint64_t gdim[3] = {(cuuint64_t)d->H * d->D, (cuuint64_t)n, (cuuint64_t)d->B};
  // one sample: the batch stride is never stepped over, give the map a valid one
  cuuint64_t gstr[2] = {(cuuint64_t)rs * 2, (cuuint64_t)(d->B == 1 ? rs * n : bs) * 2};
  cuuint32_t box[3] = {32, 64, 1}, estr[3] = {1, 1, 1};
  return encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(p), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int D, bool MASKED = false>
static int launch_attention_wgmma(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o, cudaStream_t s,
                                  const char* name, const unsigned char* kv_valid = nullptr, float* lse = nullptr) {
  EncodeTiledFn encode = get_encode_fn();
  if (!encode) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return PV_ERR_CUDA; }
  AttnWgParams P;
  memset(&P, 0, sizeof(P));
  P.d = *d;
  if (!aw_encode(encode, &P.q_map, q, d, d->Nq, d->q_row_stride, d->q_batch_stride) ||
      !aw_encode(encode, &P.k_map, k, d, d->Nk, d->k_row_stride, d->k_batch_stride) ||
      !aw_encode(encode, &P.v_map, v, d, d->Nk, d->v_row_stride, d->v_batch_stride)) {
    set_error("cuTensorMapEncodeTiled(attention q/k/v) failed");
    return PV_ERR_CUDA;
  }
  constexpr size_t smem = 1024 + 5 * (size_t)(D / 32) * AW_CHUNK + 64;
  PV_OPT_IN_SMEM((attention_wgmma_kernel<D, MASKED>), smem);
  dim3 grid((unsigned)cdiv(d->Nq, AW_BQ), (unsigned)(d->B * d->H)), block(128);
  attention_wgmma_kernel<D, MASKED><<<grid, block, smem, s>>>(P, (const __half*)q, (__half*)o, kv_valid, lse);
  PV_LAUNCH_OK(name);
  return PV_OK;
}

// f16 wgmma path for head dims 32 / 64 / 96; pv_attention_fwd (pv_attention.cu) has checked the alignment of pointers
// and strides (16-byte tensor-map bases and strides, 4-byte output stores).
int attention_wgmma_launch(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o, cudaStream_t s) {
#define PV_AW(DD) \
  case DD: return launch_attention_wgmma<DD>(d, q, k, v, o, s, "attention_wgmma_kernel<" #DD ">");
  switch (d->D) {
    PV_AW(32) PV_AW(64) PV_AW(96)
    default: set_error("internal: wgmma attention head dim %d", d->D); return PV_ERR_INVALID;
  }
#undef PV_AW
}

// Key-masked twin (pv_attention_masked_fwd); same alignment rules and head dims.
int attention_wgmma_masked_launch(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o,
                                  const unsigned char* kv_valid, float* lse, cudaStream_t s) {
#define PV_AWM(DD) \
  case DD: return launch_attention_wgmma<DD, true>(d, q, k, v, o, s, "attention_wgmma_masked_kernel<" #DD ">", kv_valid, lse);
  switch (d->D) {
    PV_AWM(32) PV_AWM(64) PV_AWM(96)
    default: set_error("internal: masked wgmma attention head dim %d", d->D); return PV_ERR_INVALID;
  }
#undef PV_AWM
}

}  // namespace pv

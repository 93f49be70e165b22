// Flash-style pooled attention on the tensor cores (f16 storage, fp32 softmax / accumulation).
//   o = softmax((q*scale) k^T) v (+ q)        reference layers/attention.py:531-539
// One CTA = 64 query rows of one (batch, head): 4 warps x 16 rows.  K/V stream through shared memory
// in 64-key tiles (cp.async, double buffered); S = Q K^T and O += P V run on mma.sync m16n8k16 with
// the online-softmax state in registers, so the N_q x N_k score matrix never exists in memory.
// (The CUDA-core kernel remains the f32 "parity mode" path.)
#include "pv_common.cuh"

namespace pv {

constexpr int FA_BQ = 64, FA_BK = 64, FA_WARPS = 4;

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// MASKED: key j of sample b counts only where kv_valid[b * Nk + j] != 0; lse (optional) receives max + log(sum) per row.
template <int D, bool MASKED = false>
__global__ void __launch_bounds__(FA_WARPS * 32)
attention_mma_kernel(pv_attention_desc d, const __half* __restrict__ q, const __half* __restrict__ k,
                     const __half* __restrict__ v, __half* __restrict__ o,
                     const unsigned char* __restrict__ kv_valid = nullptr, float* __restrict__ lse = nullptr) {
  constexpr int DS = D + 8;                 // padded smem row (halves): conflict-free fragment loads
  constexpr int KS = D / 16;                // k-steps of the QK^T product
  constexpr int ND = D / 8;                 // n-tiles of the PV product
  constexpr int NT = FA_BK / 8;             // n-tiles (8 keys) of one key tile
  constexpr int CH = D / 8;                 // 16-byte chunks per row
  extern __shared__ __align__(16) uint8_t fa_smem[];
  __half* Ks = reinterpret_cast<__half*>(fa_smem);            // [2][FA_BK][DS]
  __half* Vs = Ks + 2 * FA_BK * DS;                           // [2][FA_BK][DS]

  const int bh = blockIdx.y;
  const int b = bh / d.H, h = bh - b * d.H;
  const int q0 = blockIdx.x * FA_BQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;

  const __half* qb = q + (long long)b * d.q_batch_stride + (long long)h * D;
  const __half* kb = k + (long long)b * d.k_batch_stride + (long long)h * D;
  const __half* vb = v + (long long)b * d.v_batch_stride + (long long)h * D;
  __half* ob = o + (long long)b * d.o_batch_stride + (long long)h * D;

  // ---- stage K/V tile `kt` into buffer `buf` (zero fill beyond Nk)
  auto load_tile = [&](int kt, int buf) {
    const int k0 = kt * FA_BK;
    __half* kd = Ks + buf * FA_BK * DS;
    __half* vd = Vs + buf * FA_BK * DS;
    for (int c = threadIdx.x; c < FA_BK * CH; c += FA_WARPS * 32) {
      const int r = c / CH, cc = c - r * CH;
      const int key = k0 + r;
      const bool ok = key < d.Nk;
      const __half* ks = ok ? kb + (long long)key * d.k_row_stride + cc * 8 : kb;
      const __half* vs = ok ? vb + (long long)key * d.v_row_stride + cc * 8 : vb;
      const uint32_t kdst = (uint32_t)__cvta_generic_to_shared(kd + r * DS + cc * 8);
      const uint32_t vdst = (uint32_t)__cvta_generic_to_shared(vd + r * DS + cc * 8);
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(kdst), "l"(ks), "r"(ok ? 16u : 0u) : "memory");
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(vdst), "l"(vs), "r"(ok ? 16u : 0u) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  // ---- Q fragments (A operand), rows r0+g and r0+g+8 of this warp
  const int r0 = q0 + warp * 16;
  const int qa = r0 + g, qb8 = r0 + g + 8;
  uint32_t aq[KS][4];
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    const __half* p0 = qb + (long long)qa * d.q_row_stride + ks * 16 + 2 * t;
    const __half* p1 = qb + (long long)qb8 * d.q_row_stride + ks * 16 + 2 * t;
    aq[ks][0] = qa < d.Nq ? *reinterpret_cast<const uint32_t*>(p0) : 0u;
    aq[ks][1] = qb8 < d.Nq ? *reinterpret_cast<const uint32_t*>(p1) : 0u;
    aq[ks][2] = qa < d.Nq ? *reinterpret_cast<const uint32_t*>(p0 + 8) : 0u;
    aq[ks][3] = qb8 < d.Nq ? *reinterpret_cast<const uint32_t*>(p1 + 8) : 0u;
  }

  float oacc[ND][4];
#pragma unroll
  for (int i = 0; i < ND; ++i) { oacc[i][0] = oacc[i][1] = oacc[i][2] = oacc[i][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows g and g+8 (l: per-thread partial)

  const int ntiles = (d.Nk + FA_BK - 1) / FA_BK;
  load_tile(0, 0);
  for (int kt = 0; kt < ntiles; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < ntiles) {
      load_tile(kt + 1, buf ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const __half* kt_s = Ks + buf * FA_BK * DS;
    const __half* vt_s = Vs + buf * FA_BK * DS;

    // ---- S = Q K^T  (16 x 64 per warp)
    float s[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) { s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const __half* kr = kt_s + (nt * 8 + g) * DS + ks * 16 + 2 * t;
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(kr);
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(kr + 8);
        mma16816(s[nt], aq[ks], b0, b1);
      }
    }
    // ---- scale, mask the key tail, online softmax
    const int kbase = kt * FA_BK + 2 * t;
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int key = kbase + nt * 8;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        bool ok = (key + (e & 1)) < d.Nk;
        if constexpr (MASKED) ok = ok && kv_valid[(long long)b * d.Nk + key + (e & 1)] != 0;
        s[nt][e] = ok ? s[nt][e] * d.scale : -INFINITY;
      }
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
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
    for (int nt = 0; nt < NT; ++nt) {
      s[nt][0] = __expf(s[nt][0] - e0); s[nt][1] = __expf(s[nt][1] - e0);
      s[nt][2] = __expf(s[nt][2] - e1); s[nt][3] = __expf(s[nt][3] - e1);
      ps0 += s[nt][0] + s[nt][1];
      ps1 += s[nt][2] + s[nt][3];
    }
    l0 = l0 * c0 + ps0;
    l1 = l1 * c1 + ps1;
#pragma unroll
    for (int nd = 0; nd < ND; ++nd) { oacc[nd][0] *= c0; oacc[nd][1] *= c0; oacc[nd][2] *= c1; oacc[nd][3] *= c1; }

    // ---- O += P V   (P from the S accumulators, V fragments via ldmatrix.trans)
#pragma unroll
    for (int kk = 0; kk < FA_BK / 16; ++kk) {
      uint32_t pa[4];
      pa[0] = pack_h2(s[2 * kk][0], s[2 * kk][1]);
      pa[1] = pack_h2(s[2 * kk][2], s[2 * kk][3]);
      pa[2] = pack_h2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      pa[3] = pack_h2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
      // lanes 0-7: keys kk*16+0..7 of dims nd*8.., lanes 8-15: keys kk*16+8..15, lanes 16-31: the next n-tile
      const int vrow = kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
      for (int nd = 0; nd < ND; nd += 2) {
        const int vcol = (nd + (lane >> 4)) * 8;
        const uint32_t addr = (uint32_t)__cvta_generic_to_shared(vt_s + vrow * DS + vcol);
        uint32_t b0, b1, b2, b3;
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                     : "=r"(b0), "=r"(b1), "=r"(b2), "=r"(b3) : "r"(addr));
        mma16816(oacc[nd], pa, b0, b1);
        mma16816(oacc[nd + 1], pa, b2, b3);
      }
    }
    __syncthreads();     // everyone is done with `buf` before it is refilled two iterations later
  }

  // ---- finalise: row sums across the 4 lanes of a row, normalise, (+q), store
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  float i0 = 1.f / l0, i1 = 1.f / l1;
  if constexpr (MASKED) {          // a row without a valid key: o = 0, lse = -inf
    i0 = l0 > 0.f ? i0 : 0.f;
    i1 = l1 > 0.f ? i1 : 0.f;
    if (lse && t == 0) {
      float* lr = lse + (long long)bh * d.Nq;
      if (qa < d.Nq) lr[qa] = l0 > 0.f ? m0 + logf(l0) : -INFINITY;
      if (qb8 < d.Nq) lr[qb8] = l1 > 0.f ? m1 + logf(l1) : -INFINITY;
    }
  }
#pragma unroll
  for (int nd = 0; nd < ND; ++nd) {
    const int col = nd * 8 + 2 * t;
    if (qa < d.Nq) {
      float x0 = oacc[nd][0] * i0, x1 = oacc[nd][1] * i0;
      if (d.add_q_residual) {
        const float2 r = __half22float2(*reinterpret_cast<const __half2*>(qb + (long long)qa * d.q_row_stride + col));
        x0 += r.x; x1 += r.y;
      }
      *reinterpret_cast<__half2*>(ob + (long long)qa * d.o_row_stride + col) = __floats2half2_rn(x0, x1);
    }
    if (qb8 < d.Nq) {
      float x2 = oacc[nd][2] * i1, x3 = oacc[nd][3] * i1;
      if (d.add_q_residual) {
        const float2 r = __half22float2(*reinterpret_cast<const __half2*>(qb + (long long)qb8 * d.q_row_stride + col));
        x2 += r.x; x3 += r.y;
      }
      *reinterpret_cast<__half2*>(ob + (long long)qb8 * d.o_row_stride + col) = __floats2half2_rn(x2, x3);
    }
  }
}

template <int D, bool MASKED = false>
static int launch_attention_mma(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o,
                                cudaStream_t s, const char* name, const unsigned char* kv_valid = nullptr,
                                float* lse = nullptr) {
  const size_t smem = (size_t)4 * FA_BK * (D + 8) * sizeof(__half);
  PV_OPT_IN_SMEM((attention_mma_kernel<D, MASKED>), smem);
  dim3 grid((unsigned)cdiv(d->Nq, FA_BQ), (unsigned)(d->B * d->H)), block(FA_WARPS * 32);
  attention_mma_kernel<D, MASKED><<<grid, block, smem, s>>>(*d, (const __half*)q, (const __half*)k, (const __half*)v,
                                                           (__half*)o, kv_valid, lse);
  PV_LAUNCH_OK(name);
  return PV_OK;
}

// f16 tensor-core path; pv_attention_fwd (pv_attention.cu) has checked the alignment of pointers and strides.
// Only D = 128 is routed here: the wgmma kernel takes 32 / 64 / 96 under the same alignment rules.
int attention_mma_launch(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o, cudaStream_t s) {
#define PV_AM(DD) \
  case DD: return launch_attention_mma<DD>(d, q, k, v, o, s, "attention_mma_kernel<" #DD ">");
  switch (d->D) {
    PV_AM(128)
    default: set_error("internal: mma attention head dim %d", d->D); return PV_ERR_INVALID;
  }
#undef PV_AM
}

// Key-masked twin (pv_attention_masked_fwd); same alignment rules.  Only D = 128 is routed here.
int attention_mma_masked_launch(const pv_attention_desc* d, const void* q, const void* k, const void* v, void* o,
                                const unsigned char* kv_valid, float* lse, cudaStream_t s) {
#define PV_AMM(DD) \
  case DD: return launch_attention_mma<DD, true>(d, q, k, v, o, s, "attention_mma_masked_kernel<" #DD ">", kv_valid, lse);
  switch (d->D) {
    PV_AMM(128)
    default: set_error("internal: masked mma attention head dim %d", d->D); return PV_ERR_INVALID;
  }
#undef PV_AMM
}

}  // namespace pv

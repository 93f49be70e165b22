// Objectives of the self-supervised models (models/simclr.py, byol.py, memory_bank.py) and the soft-target cross
// entropy (losses/soft_target_cross_entropy.py), plus BYOL's momentum (EMA) parameter update.
//
// Every reduction runs in a fixed order: a thread sums a fixed strided subset of its row, then a fixed xor-shuffle tree
// combines the lanes and a fixed tree the warps.  No atomics touch a value, so repeated calls are bitwise identical.
// Embeddings, logits and losses are fp32 throughout: at a temperature of 0.07 every logit error is multiplied by 14.
#include "pv_common.cuh"

namespace pv {
namespace ssl {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// Block-wide sum / max in a fixed order; every thread gets the result.  `red` holds WARPS floats.
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < WARPS; ++w) s += red[w];
  return s;
}
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = -INFINITY;
#pragma unroll
  for (int w = 0; w < WARPS; ++w) s = fmaxf(s, red[w]);
  return s;
}

template <typename T> __device__ __forceinline__ float ldf(const T* p);
template <> __device__ __forceinline__ float ldf<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ldf<__half>(const __half* p) { return __half2float(*p); }
template <> __device__ __forceinline__ float ldf<long long>(const long long* p) { return (float)*p; }

// ---- F.normalize(x, p=2, dim=1): y = x / max(||x||_2, 1e-12), one block per row ----------------------------------------
template <typename T>
__global__ void __launch_bounds__(THREADS)
l2_normalize_kernel(const T* __restrict__ x, long long xs, float* __restrict__ y, long long ys, int C) {
  __shared__ float red[WARPS];
  const T* xr = x + (long long)blockIdx.x * xs;
  float ss = 0.f;
  for (int c = threadIdx.x; c < C; c += THREADS) {
    const float v = ldf<T>(xr + c);
    ss = fmaf(v, v, ss);
  }
  const float nrm = fmaxf(__fsqrt_rn(block_sum(ss, red)), 1e-12f);
  float* yr = y + (long long)blockIdx.x * ys;
  for (int c = threadIdx.x; c < C; c += THREADS) yr[c] = __fdiv_rn(ldf<T>(xr + c), nrm);
}

// Dot product of two fp32 rows of C elements by one warp: lane l sums elements l, l + 32, ... in order, then the
// fixed shuffle tree.  Every lane returns the same value.
__device__ __forceinline__ float warp_dot(const float* __restrict__ a, const float* __restrict__ b, int C) {
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s = fmaf(a[c], b[c], s);
  return warp_sum(s);
}

// Row logsumexp over n values in shared memory, fixed order: max, then sum of expf(v - max).
__device__ __forceinline__ float block_lse(const float* v, int n, float* red) {
  float m = -INFINITY;
  for (int i = threadIdx.x; i < n; i += THREADS) m = fmaxf(m, v[i]);
  m = block_max(m, red);
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += THREADS) s += expf(v[i] - m);
  s = block_sum(s, red);
  return m + logf(s);
}

// ---- SimCLR: row n of q against every key row: logits (q_n . k_m) / T in shared memory, CE against key
//      row_offset + n.  BYOL: q_n . k_n.  One block per query row writes row[n]; the mean is a separate launch. ---------
__global__ void __launch_bounds__(THREADS)
contrastive_rows_kernel(const float* __restrict__ q, long long qs, const float* __restrict__ k, long long ks, int M, int C,
                        float temperature, long long row_offset, int mode, float* __restrict__ row) {
  extern __shared__ float logit[];
  __shared__ float red[WARPS];
  const int n = blockIdx.x;
  const float* qn = q + (long long)n * qs;
  const int warp = threadIdx.x >> 5;
  if (mode == 1) {                                       // BYOL: the similarity of row n with key row n
    if (warp == 0) {
      const float d = warp_dot(qn, k + (long long)n * ks, C);
      if (threadIdx.x == 0) row[n] = d;
    }
    return;
  }
  for (int m = warp; m < M; m += WARPS) {
    const float d = warp_dot(qn, k + (long long)m * ks, C);
    if ((threadIdx.x & 31) == 0) logit[m] = __fdiv_rn(d, temperature);
  }
  __syncthreads();
  const float lse = block_lse(logit, M, red);
  if (threadIdx.x == 0) row[n] = lse - logit[row_offset + n];
}

// ---- loss = scale * sum(row[0..n)) / n in a fixed order (one block) ---------------------------------------------------
__global__ void __launch_bounds__(THREADS)
mean_kernel(const float* __restrict__ row, int n, float sign, float* __restrict__ out) {
  __shared__ float red[WARPS];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += THREADS) s += row[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) *out = sign * __fdiv_rn(s, (float)n);
}

// ---- memory bank: logits[b][j] = (memory[idx[b][j]] . x_b) / T for the K1 = neg_size + 1 rows of sample b ----------
// The gather is the hot loop: it reads B * K1 * dim * 4 bytes of scattered bank rows.  One warp owns four rows at a
// time and issues the four rows' 16-byte loads together, so that enough bytes are in flight to stream at HBM rate
// even for short rows.  An index outside [0, bank_rows) sets *flag and is never dereferenced.
constexpr int MB_ROWS = 4;                   // rows per warp iteration
constexpr int MB_WARP_ROWS = 16;             // rows per warp per block (4 iterations)

template <bool VEC>
__global__ void __launch_bounds__(THREADS)
memory_bank_logits_kernel(const float* __restrict__ x, long long xs, const float* __restrict__ memory, long long bank_rows,
                          int dim, const long long* __restrict__ idx, int K1, float temperature,
                          float* __restrict__ logits, int* __restrict__ flag) {
  extern __shared__ float xsh[];
  const int b = blockIdx.y;
  const float* xb = x + (long long)b * xs;
  for (int c = threadIdx.x; c < dim; c += THREADS) xsh[c] = xb[c];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long* ib = idx + (long long)b * K1;
  float* lb = logits + (long long)b * K1;
  const int j0 = (blockIdx.x * WARPS + warp) * MB_WARP_ROWS;
  for (int jj = 0; jj < MB_WARP_ROWS; jj += MB_ROWS) {
    const float* rp[MB_ROWS];
    bool ok[MB_ROWS];
#pragma unroll
    for (int r = 0; r < MB_ROWS; ++r) {
      const int j = j0 + jj + r;
      const long long id = j < K1 ? __ldg(ib + j) : 0;
      ok[r] = j < K1 && id >= 0 && id < bank_rows;
      if (j < K1 && !ok[r] && lane == 0) atomicOr(flag, 1);
      rp[r] = memory + (ok[r] ? id : 0) * (long long)dim;     // 64-bit byte offsets
    }
    float s[MB_ROWS];
#pragma unroll
    for (int r = 0; r < MB_ROWS; ++r) s[r] = 0.f;
    if (VEC) {
      const float4* x4 = reinterpret_cast<const float4*>(xsh);
      for (int c = lane; c < dim / 4; c += 32) {
        float4 m[MB_ROWS];
#pragma unroll
        for (int r = 0; r < MB_ROWS; ++r)
          m[r] = ok[r] ? __ldcs(reinterpret_cast<const float4*>(rp[r]) + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 xv = x4[c];
#pragma unroll
        for (int r = 0; r < MB_ROWS; ++r) {
          s[r] = fmaf(m[r].x, xv.x, s[r]);
          s[r] = fmaf(m[r].y, xv.y, s[r]);
          s[r] = fmaf(m[r].z, xv.z, s[r]);
          s[r] = fmaf(m[r].w, xv.w, s[r]);
        }
      }
    } else {
      for (int c = lane; c < dim; c += 32) {
        const float xv = xsh[c];
#pragma unroll
        for (int r = 0; r < MB_ROWS; ++r)
          if (ok[r]) s[r] = fmaf(__ldcs(rp[r] + c), xv, s[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < MB_ROWS; ++r) {
      const float d = warp_sum(s[r]);
      const int j = j0 + jj + r;
      if (lane == 0 && j < K1) lb[j] = __fdiv_rn(d, temperature);
    }
  }
}

// row[b] = logsumexp(logits[b][0..K1)) - logits[b][0]: cross entropy against target 0 (memory_bank.py:102-103)
__global__ void __launch_bounds__(THREADS)
lse_target0_kernel(const float* __restrict__ logits, int K1, float* __restrict__ row) {
  __shared__ float red[WARPS];
  const float* lb = logits + (long long)blockIdx.x * K1;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < K1; i += THREADS) m = fmaxf(m, lb[i]);
  m = block_max(m, red);
  float s = 0.f;
  for (int i = threadIdx.x; i < K1; i += THREADS) s += expf(lb[i] - m);
  s = block_sum(s, red);
  if (threadIdx.x == 0) row[blockIdx.x] = m + logf(s) - lb[0];
}

// ---- soft-target cross entropy, one block per sample (soft_target_cross_entropy.py:66-71):
//      t = target (/ (eps + sum t) when normalising); row[n] = sum_c -t_c * log_softmax(x)_c ---------------------------
template <typename T, typename U>
__global__ void __launch_bounds__(THREADS)
soft_target_rows_kernel(const T* __restrict__ x, long long xs, const U* __restrict__ t, long long ts, int C, int normalize,
                        float eps, float* __restrict__ row) {
  __shared__ float red[WARPS];
  const T* xr = x + (long long)blockIdx.x * xs;
  const U* tr = t + (long long)blockIdx.x * ts;
  float m = -INFINITY, tsum = 0.f;
  for (int c = threadIdx.x; c < C; c += THREADS) {
    m = fmaxf(m, ldf<T>(xr + c));
    tsum += ldf<U>(tr + c);
  }
  m = block_max(m, red);
  float se = 0.f;
  for (int c = threadIdx.x; c < C; c += THREADS) se += expf(ldf<T>(xr + c) - m);
  se = block_sum(se, red);
  const float lz = logf(se);
  const float den = normalize ? block_sum(tsum, red) + eps : 1.f;
  float acc = 0.f;
  for (int c = threadIdx.x; c < C; c += THREADS) {
    float tv = ldf<U>(tr + c);
    if (normalize) tv = __fdiv_rn(tv, den);
    const float ls = (ldf<T>(xr + c) - m) - lz;
    acc = fmaf(-tv, ls, acc);
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) row[blockIdx.x] = acc;
}

// ---- BYOL momentum update, every parameter of the backbone in one launch: p_m = p_m * mmt + p * (1 - mmt) with each
//      product and the sum rounded once (the reference's three eager fp32 ops; no FMA contraction) -----------------------
constexpr int EMA_CHUNK = 4096;              // elements per block
__global__ void __launch_bounds__(THREADS)
ema_update_kernel(float* const* __restrict__ dst, const float* const* __restrict__ src, const long long* __restrict__ numel,
                  const long long* __restrict__ chunks, float mmt, float omm) {
  const long long e = chunks[blockIdx.x];
  const int t = (int)(e >> 40);                       // tensor index in the high bits, chunk start in the low 40
  const long long start = e & ((1ll << 40) - 1);
  const long long n = numel[t];
  float* d = dst[t];
  const float* s = src[t];
  const long long end = min(n, start + (long long)EMA_CHUNK);
  for (long long i = start + threadIdx.x; i < end; i += THREADS) d[i] = __fadd_rn(__fmul_rn(d[i], mmt), __fmul_rn(s[i], omm));
}

}  // namespace ssl
}  // namespace pv

using namespace pv::ssl;

extern "C" int pv_rows_l2_normalize(const void* x, int dtype, long long x_row_stride, float* y, long long y_row_stride,
                                    int rows, int C, void* stream) {
  PV_CHECK_ARG(x != nullptr && y != nullptr, "null argument");
  PV_CHECK_ARG(rows >= 1 && rows <= 2147483647 && C >= 1, "bad shape rows=%d C=%d", rows, C);
  PV_CHECK_ARG(x_row_stride >= C && y_row_stride >= C, "row strides must cover C");
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == PV_F32) {
    l2_normalize_kernel<float><<<rows, THREADS, 0, s>>>((const float*)x, x_row_stride, y, y_row_stride, C);
    PV_LAUNCH_OK("l2_normalize_kernel<float>");
  } else {
    PV_CHECK_ARG(dtype == PV_F16, "rows must be float16 or float32");
    l2_normalize_kernel<__half><<<rows, THREADS, 0, s>>>((const __half*)x, x_row_stride, y, y_row_stride, C);
    PV_LAUNCH_OK("l2_normalize_kernel<__half>");
  }
  return PV_OK;
}

extern "C" int pv_contrastive_ce(const float* q, long long q_row_stride, const float* k, long long k_row_stride, int N,
                                 int M, int C, float temperature, long long row_offset, int mode, float* row_loss,
                                 float* loss, void* stream) {
  PV_CHECK_ARG(q != nullptr && k != nullptr && row_loss != nullptr && loss != nullptr, "null argument");
  PV_CHECK_ARG(N >= 1 && M >= 1 && C >= 1, "bad shape N=%d M=%d C=%d", N, M, C);
  PV_CHECK_ARG(q_row_stride >= C && k_row_stride >= C, "row strides must cover C");
  PV_CHECK_ARG(mode == 0 || mode == 1, "mode must be 0 (SimCLR) or 1 (BYOL)");
  cudaStream_t s = (cudaStream_t)stream;
  if (mode == 0) {
    PV_CHECK_ARG(M <= 16384, "at most 16384 keys (got %d)", M);
    PV_CHECK_ARG(row_offset >= 0 && row_offset + N <= M, "targets %lld .. %lld outside the %d keys", row_offset,
                 row_offset + N - 1, M);
    const size_t smem = (size_t)M * sizeof(float);
    if (smem > 48 * 1024) PV_OPT_IN_SMEM(contrastive_rows_kernel, 16384 * sizeof(float));
    contrastive_rows_kernel<<<N, THREADS, smem, s>>>(q, q_row_stride, k, k_row_stride, M, C, temperature, row_offset, 0,
                                                     row_loss);
    PV_LAUNCH_OK("contrastive_rows_kernel<simclr>");
  } else {
    PV_CHECK_ARG(M == N, "BYOL pairs query row n with key row n (N=%d, M=%d)", N, M);
    contrastive_rows_kernel<<<N, THREADS, 0, s>>>(q, q_row_stride, k, k_row_stride, M, C, temperature, 0, 1, row_loss);
    PV_LAUNCH_OK("contrastive_rows_kernel<byol>");
  }
  mean_kernel<<<1, THREADS, 0, s>>>(row_loss, N, mode == 0 ? 1.f : -1.f, loss);
  PV_LAUNCH_OK("mean_kernel");
  return PV_OK;
}

extern "C" int pv_memory_bank_ce(const float* x, long long x_row_stride, const float* memory, long long bank_rows, int dim,
                                 const long long* idx, int B, int K1, float temperature, float* logits, float* row_loss,
                                 float* loss, int* flag, void* stream) {
  PV_CHECK_ARG(x != nullptr && memory != nullptr && idx != nullptr && logits != nullptr && row_loss != nullptr &&
               loss != nullptr && flag != nullptr, "null argument");
  PV_CHECK_ARG(B >= 1 && B <= 65535 && K1 >= 1 && dim >= 1 && bank_rows >= 1, "bad shape B=%d K1=%d dim=%d", B, K1, dim);
  PV_CHECK_ARG(dim <= 12 * 1024, "dim %d above 12288 (the sample row lives in shared memory)", dim);
  PV_CHECK_ARG(x_row_stride >= dim, "row stride must cover dim");
  cudaStream_t s = (cudaStream_t)stream;
  PV_CUDA_OK(cudaMemsetAsync(flag, 0, sizeof(int), s));
  const int rows_per_block = WARPS * MB_WARP_ROWS;
  const dim3 grid((unsigned)pv::cdiv(K1, rows_per_block), (unsigned)B);
  const size_t smem = (size_t)pv::cdiv(dim, 4) * 4 * sizeof(float);
  const bool vec = dim % 4 == 0 && (uintptr_t)memory % 16 == 0;
  if (vec) {
    if (smem > 48 * 1024) PV_OPT_IN_SMEM(memory_bank_logits_kernel<true>, 12 * 1024 * sizeof(float));
    memory_bank_logits_kernel<true><<<grid, THREADS, smem, s>>>(x, x_row_stride, memory, bank_rows, dim, idx, K1,
                                                                temperature, logits, flag);
    PV_LAUNCH_OK("memory_bank_logits_kernel<vec4>");
  } else {
    if (smem > 48 * 1024) PV_OPT_IN_SMEM(memory_bank_logits_kernel<false>, 12 * 1024 * sizeof(float));
    memory_bank_logits_kernel<false><<<grid, THREADS, smem, s>>>(x, x_row_stride, memory, bank_rows, dim, idx, K1,
                                                                 temperature, logits, flag);
    PV_LAUNCH_OK("memory_bank_logits_kernel<scalar>");
  }
  lse_target0_kernel<<<B, THREADS, 0, s>>>(logits, K1, row_loss);
  PV_LAUNCH_OK("lse_target0_kernel");
  mean_kernel<<<1, THREADS, 0, s>>>(row_loss, B, 1.f, loss);
  PV_LAUNCH_OK("mean_kernel");
  return PV_OK;
}

extern "C" int pv_soft_target_ce(const void* x, int x_dtype, long long x_row_stride, const void* target, int t_dtype,
                                 long long t_row_stride, int N, int C, int normalize, float eps, int reduce_mean,
                                 float* row_loss, float* loss, void* stream) {
  PV_CHECK_ARG(x != nullptr && target != nullptr && row_loss != nullptr, "null argument");
  PV_CHECK_ARG(!reduce_mean || loss != nullptr, "the mean needs its output");
  PV_CHECK_ARG(N >= 1 && N <= 2147483647 && C >= 1, "bad shape N=%d C=%d", N, C);
  PV_CHECK_ARG(x_row_stride >= C && t_row_stride >= C, "row strides must cover C");
  PV_CHECK_ARG(x_dtype == PV_F32 || x_dtype == PV_F16, "logits must be float16 or float32");
  PV_CHECK_ARG(t_dtype == PV_F32 || t_dtype == PV_F16 || t_dtype == PV_I64, "targets must be float or int64");
  cudaStream_t s = (cudaStream_t)stream;
#define PV_SOFT_CE(T, U, NAME)                                                                                  \
  soft_target_rows_kernel<T, U><<<N, THREADS, 0, s>>>((const T*)x, x_row_stride, (const U*)target, t_row_stride, C, \
                                                      normalize, eps, row_loss);                               \
  PV_LAUNCH_OK(NAME)
  if (x_dtype == PV_F32) {
    if (t_dtype == PV_F32) { PV_SOFT_CE(float, float, "soft_target_rows_kernel<float,float>"); }
    else if (t_dtype == PV_F16) { PV_SOFT_CE(float, __half, "soft_target_rows_kernel<float,__half>"); }
    else { PV_SOFT_CE(float, long long, "soft_target_rows_kernel<float,int64>"); }
  } else {
    if (t_dtype == PV_F32) { PV_SOFT_CE(__half, float, "soft_target_rows_kernel<__half,float>"); }
    else if (t_dtype == PV_F16) { PV_SOFT_CE(__half, __half, "soft_target_rows_kernel<__half,__half>"); }
    else { PV_SOFT_CE(__half, long long, "soft_target_rows_kernel<__half,int64>"); }
  }
#undef PV_SOFT_CE
  if (reduce_mean) {
    mean_kernel<<<1, THREADS, 0, s>>>(row_loss, N, 1.f, loss);
    PV_LAUNCH_OK("mean_kernel");
  }
  return PV_OK;
}

extern "C" int pv_ema_update(float* const* dst, const float* const* src, const long long* numel, const long long* chunks,
                             int n_chunks, float mmt, float one_minus_mmt, void* stream) {
  PV_CHECK_ARG(dst != nullptr && src != nullptr && numel != nullptr && chunks != nullptr, "null argument");
  PV_CHECK_ARG(n_chunks >= 0 && n_chunks <= 2147483647, "bad chunk count %d", n_chunks);
  if (n_chunks == 0) return PV_OK;
  ema_update_kernel<<<n_chunks, THREADS, 0, (cudaStream_t)stream>>>(dst, src, numel, chunks, mmt, one_minus_mmt);
  PV_LAUNCH_OK("ema_update_kernel");
  return PV_OK;
}

// ---- in-place weight refresh of a compiled plan (engine/refresh.py) ---------------------------------------------------
// Gather jobs: dst[i] = map[map_off + i] < 0 ? 0 : src[slot][map[map_off + i]], stored as f16 (round to nearest even,
// as torch's .to(float16)) or f32: the plan's packed weights re-derived from the module's fp32 parameters with the
// layout recorded when the plan was built.  Fold jobs: the BatchNorm fold of packing.fold_bn in fp64 - s = gamma /
// sqrt(var + eps), b = (conv_bias - mean) * s + beta, one correctly rounded double operation each (no FMA), then
// rounded to fp32 - so the refreshed bytes equal those of a fresh compile.
namespace pv {
namespace ssl {

constexpr int REFRESH_CHUNK = 4096;

__global__ void __launch_bounds__(THREADS)
refresh_gather_kernel(const long long* __restrict__ jobs, const long long* __restrict__ chunks,
                      const int* __restrict__ map, const float* const* __restrict__ srcs) {
  const long long e = chunks[blockIdx.x];
  const long long* job = jobs + (e >> 40) * 5;
  const long long start = e & ((1ll << 40) - 1);
  const long long n = job[2];
  const float* src = srcs[job[4]];
  const int* m = map + job[3];
  const long long end = min(n, start + (long long)REFRESH_CHUNK);
  if (job[1] == PV_F16) {
    __half* dst = reinterpret_cast<__half*>(job[0]);
    for (long long i = start + threadIdx.x; i < end; i += THREADS) {
      const int k = m[i];
      dst[i] = __float2half_rn(k < 0 ? 0.f : src[k]);
    }
  } else {
    float* dst = reinterpret_cast<float*>(job[0]);
    for (long long i = start + threadIdx.x; i < end; i += THREADS) {
      const int k = m[i];
      dst[i] = k < 0 ? 0.f : src[k];
    }
  }
}

// fold job: scale dst, bias dst, c_out, conv_bias, gamma, beta, mean, var (device pointers or 0), eps (double bits)
__global__ void __launch_bounds__(THREADS)
refresh_fold_kernel(const long long* __restrict__ jobs) {
  const long long* j = jobs + (long long)blockIdx.x * 9;
  float* sd = reinterpret_cast<float*>(j[0]);
  float* bd = reinterpret_cast<float*>(j[1]);
  const int c_out = (int)j[2];
  const float* cb = reinterpret_cast<const float*>(j[3]);
  const float* gamma = reinterpret_cast<const float*>(j[4]);
  const float* beta = reinterpret_cast<const float*>(j[5]);
  const float* mean = reinterpret_cast<const float*>(j[6]);
  const float* var = reinterpret_cast<const float*>(j[7]);
  const double eps = __longlong_as_double(j[8]);
  for (int c = threadIdx.x; c < c_out; c += THREADS) {
    double s = 1.0, b = cb ? (double)cb[c] : 0.0;
    if (var) {
      const double g = gamma ? (double)gamma[c] : 1.0;
      s = __ddiv_rn(g, __dsqrt_rn(__dadd_rn((double)var[c], eps)));
      b = __dadd_rn(__dmul_rn(__dsub_rn(b, (double)mean[c]), s), beta ? (double)beta[c] : 0.0);
    }
    sd[c] = __double2float_rn(s);
    bd[c] = __double2float_rn(b);
  }
}

}  // namespace ssl
}  // namespace pv

extern "C" int pv_weights_refresh(const long long* gather_jobs, const long long* gather_chunks, int n_gather_chunks,
                                  const int* map, const float* const* srcs, const long long* fold_jobs, int n_fold_jobs,
                                  void* stream) {
  PV_CHECK_ARG(n_gather_chunks >= 0 && n_fold_jobs >= 0, "negative job count");
  PV_CHECK_ARG(n_gather_chunks == 0 || (gather_jobs && gather_chunks && map && srcs), "null gather table");
  PV_CHECK_ARG(n_fold_jobs == 0 || fold_jobs, "null fold table");
  cudaStream_t s = (cudaStream_t)stream;
  if (n_gather_chunks > 0) {
    refresh_gather_kernel<<<n_gather_chunks, THREADS, 0, s>>>(gather_jobs, gather_chunks, map, srcs);
    PV_LAUNCH_OK("refresh_gather_kernel");
  }
  if (n_fold_jobs > 0) {
    refresh_fold_kernel<<<n_fold_jobs, THREADS, 0, s>>>(fold_jobs);
    PV_LAUNCH_OK("refresh_fold_kernel");
  }
  return PV_OK;
}

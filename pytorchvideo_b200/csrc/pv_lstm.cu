// Masked LSTM recurrence (models/masked_multistream.py:193-256: nn.LSTM over pack_padded_sequence, output h_n).
//
// The input projection of every step and both directions is one token GEMM on the convolution path before this
// launch (gate pre-activations G[b][t][dir * 4H + gate * H + j], gate order i, f, g, o, with b_ih + b_hh folded into
// its bias).  This file runs all T steps of both directions in ONE persistent launch: a CTA owns one direction and a
// slice of LSTM_NB batch rows, thread j owns hidden unit j of every row of the slice, so the cell update is local to
// the thread; c stays in registers, h_{t-1} of the slice sits in shared memory (double-buffered, one barrier per
// step).  W_hh is read from global memory every step as W^T [dir][k][4H] fp32 - coalesced across the units, resident
// in L2 - and each weight feeds the LSTM_NB rows of the slice.  fp32 maths throughout.  That kernel is the f32 parity
// mode (and takes f16 hidden sizes the cluster kernel below cannot split); f16 runs lstm_cluster_kernel.
//
// Row b runs its first len_b = clamp(popcount(mask[b]), 1, T) steps whatever their mask bits (pack_padded_sequence
// takes a count of valid steps, not the position of the last one); the reverse direction runs them backwards from
// step len_b - 1.  Rows past their length keep their state.  The lengths come from the device mask in the prologue,
// so nothing syncs with the host and one captured graph serves every mask.
#include "pv_common.cuh"
#include "pv_sm90.cuh"

namespace pv {

constexpr int LSTM_NB = 8;        // batch rows per CTA
constexpr int LSTM_MAX_H = 512;   // one thread per hidden unit

__device__ __forceinline__ float lstm_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

template <typename T>
__global__ void __launch_bounds__(512)
lstm_recurrence_kernel(const T* __restrict__ G, long long g_row_stride, const float* __restrict__ Wt,
                       const unsigned char* __restrict__ mask, int B, int Tn, int H, int ndir, T* __restrict__ y,
                       long long y_row_stride) {
  extern __shared__ float lstm_h[];                     // [2][LSTM_NB][H]
  __shared__ int len[LSTM_NB];
  const int dir = blockIdx.x, b0 = blockIdx.y * LSTM_NB;
  const int j = threadIdx.x;
  const int nb = min(LSTM_NB, B - b0);
  if (threadIdx.x < LSTM_NB) {
    int n = Tn;
    if (mask && (int)threadIdx.x < nb) {
      n = 0;
      const unsigned char* m = mask + (long long)(b0 + threadIdx.x) * Tn;
      for (int t = 0; t < Tn; ++t) n += m[t] != 0;
    }
    len[threadIdx.x] = (int)threadIdx.x < nb ? min(max(n, 1), Tn) : 0;
  }
  for (int e = threadIdx.x; e < 2 * LSTM_NB * H; e += blockDim.x) lstm_h[e] = 0.f;
  __syncthreads();
  int steps = 0;
#pragma unroll
  for (int r = 0; r < LSTM_NB; ++r) steps = max(steps, len[r]);

  const float* W = Wt + (long long)dir * H * 4 * H;
  const bool own = j < H;
  float c[LSTM_NB], h[LSTM_NB];
#pragma unroll
  for (int r = 0; r < LSTM_NB; ++r) c[r] = h[r] = 0.f;

  for (int s = 0; s < steps; ++s) {
    const float* hp = lstm_h + (s & 1) * LSTM_NB * H;
    float* hn = lstm_h + ((s + 1) & 1) * LSTM_NB * H;
    if (own) {
      float acc[4][LSTM_NB];
#pragma unroll
      for (int r = 0; r < LSTM_NB; ++r) {
        const int L = len[r];
        const int t = dir == 0 ? s : L - 1 - s;
        const T* g = G + ((long long)(b0 + r) * Tn + (t < 0 ? 0 : t)) * g_row_stride + (long long)dir * 4 * H + j;
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[q][r] = s < L ? Elem<T>::ld(g + q * H) : 0.f;
      }
      for (int k = 0; k < H; ++k) {
        const float* wk = W + (long long)k * 4 * H + j;
        const float w0 = __ldg(wk), w1 = __ldg(wk + H), w2 = __ldg(wk + 2 * H), w3 = __ldg(wk + 3 * H);
#pragma unroll
        for (int r = 0; r < LSTM_NB; ++r) {
          const float hv = hp[r * H + k];
          acc[0][r] = fmaf(w0, hv, acc[0][r]);
          acc[1][r] = fmaf(w1, hv, acc[1][r]);
          acc[2][r] = fmaf(w2, hv, acc[2][r]);
          acc[3][r] = fmaf(w3, hv, acc[3][r]);
        }
      }
#pragma unroll
      for (int r = 0; r < LSTM_NB; ++r) {
        if (s < len[r]) {
          const float ig = lstm_sigmoid(acc[0][r]), fg = lstm_sigmoid(acc[1][r]);
          const float gg = tanhf(acc[2][r]), og = lstm_sigmoid(acc[3][r]);
          c[r] = fg * c[r] + ig * gg;
          h[r] = og * tanhf(c[r]);
        }
        hn[r * H + j] = h[r];
      }
    }
    __syncthreads();
  }
  if (own)
    for (int r = 0; r < nb; ++r) Elem<T>::st(y + (long long)(b0 + r) * y_row_stride + (long long)dir * H + j, h[r]);
}

// ---- f16 mode: one thread-block cluster per (direction, LSTM_CNB-row batch slice) ---------------------------------------
// CTA `rank` of a cluster of S CTAs owns hs = H / S hidden units with all four of their gates, so the cell update stays
// in the CTA, and keeps their 4 * hs rows of W_hh in shared memory as f16 for the whole sequence.  Every step is one
// wgmma product per CTA: gates[4hs x 32] = W_hh_slice[4hs x H] . h_{t-1}^T[H x 32] (M = 4 hs, N = the 32-row batch
// slice, K = H), both operands K-major in the no-swizzle core-matrix layout, fp32 accumulators in registers.  The A rows
// are ordered so that the four gates of a unit land in one thread: warpgroup wg issues two m64 tiles, and tile mt, warp
// w, fragment row half / g hold gate 2 mt + half of unit 32 wg + 8 w + g, so a thread owns one unit for 8 batch rows
// (columns 8j + 2t (+1)).  c stays in fp32 registers.  The new h (f16, the B operand of the next step) goes into every
// CTA of the cluster through distributed shared memory, two units per 32-bit store, double-buffered, and one cluster
// barrier (arrive.release / wait.acquire) per step publishes it; a proxy fence then hands it to the tensor cores.
// Cluster size S: the smallest S <= 16 with hs a multiple of 32, hs <= 128 and 8 H^2 / S <= 128 KiB of weights
// (H = 512: 16 CTAs, non-portable; 384: 12; 256: 4; H <= 128: 1).  Other H run lstm_recurrence_kernel<__half>.
constexpr int LSTM_CNB = 32;           // batch rows per cluster: the wgmma N
constexpr int LSTM_W_SMEM = 128 * 1024;

__device__ __forceinline__ uint32_t lstm_cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void lstm_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// address of the same shared-memory location in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t lstm_map_rank(uint32_t smem_addr, uint32_t rank) {
  uint32_t out;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(out) : "r"(smem_addr), "r"(rank));
  return out;
}
__device__ __forceinline__ void lstm_st_cluster_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared::cluster.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// element (r, k) of a [rows][K] f16 operand in the K-major no-swizzle layout: 8 x 8 core matrices of 128 contiguous
// bytes, K-adjacent core matrices 128 B apart (LBO), row-group-adjacent ones K * 16 B apart (SBO)
__device__ __forceinline__ int lstm_cm(int r, int k, int K) {
  return ((r >> 3) * (K >> 3) + (k >> 3)) * 64 + (r & 7) * 8 + (k & 7);
}

__global__ void __launch_bounds__(512, 1)
lstm_cluster_kernel(const __half* __restrict__ G, long long g_row_stride, const float* __restrict__ Wt,
                    const unsigned char* __restrict__ mask, int B, int Tn, int H, int CS, __half* __restrict__ y,
                    long long y_row_stride) {
  using namespace sm90;
  extern __shared__ __align__(128) uint8_t lstm_cs[];
  const int hs = H / CS;
  __half* Ws = reinterpret_cast<__half*>(lstm_cs);                                      // A: [4 hs][H]
  __half* hb = reinterpret_cast<__half*>(lstm_cs + (size_t)4 * hs * H * sizeof(__half));   // B: [2][32][H]
  __shared__ int len[LSTM_CNB];
  const uint32_t rank = lstm_cluster_rank();
  const int dir = blockIdx.x / CS, b0 = blockIdx.y * LSTM_CNB;
  const int nb = min(LSTM_CNB, B - b0);
  const int wg = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int u = 32 * wg + 8 * w + g;                 // this thread's unit
  const int j = (int)rank * hs + u;                  // global hidden unit

  // prologue: this CTA's gate rows of W_hh (A row of gate q, unit v: 128 (v / 32) + 64 (q / 2) + 16 ((v % 32) / 8) +
  // 8 (q % 2) + v % 8), the lengths, h = 0
  const float* W = Wt + (long long)dir * H * 4 * H;
  for (int e = threadIdx.x; e < H * 4 * hs; e += blockDim.x) {
    const int k = e / (4 * hs), cq = e - k * 4 * hs, q = cq / hs, v = cq - q * hs;
    const int row = 128 * (v >> 5) + 64 * (q >> 1) + 16 * ((v & 31) >> 3) + 8 * (q & 1) + (v & 7);
    Ws[lstm_cm(row, k, H)] = __float2half_rn(W[(long long)k * 4 * H + q * H + (int)rank * hs + v]);
  }
  if (threadIdx.x < LSTM_CNB) {
    int n = Tn;
    if (mask && (int)threadIdx.x < nb) {
      n = 0;
      const unsigned char* m = mask + (long long)(b0 + threadIdx.x) * Tn;
      for (int tt = 0; tt < Tn; ++tt) n += m[tt] != 0;
    }
    len[threadIdx.x] = (int)threadIdx.x < nb ? min(max(n, 1), Tn) : 0;
  }
  for (int e = threadIdx.x; e < 2 * LSTM_CNB * H; e += blockDim.x) hb[e] = __float2half_rn(0.f);
  __syncthreads();
  lstm_cluster_sync();          // every CTA's h buffers are zeroed before anyone pushes into them
  int steps = 0;
  for (int r = 0; r < LSTM_CNB; ++r) steps = max(steps, len[r]);

  const uint32_t ws_addr = (uint32_t)__cvta_generic_to_shared(Ws), hb_addr = (uint32_t)__cvta_generic_to_shared(hb);
  const uint32_t sbo = (uint32_t)H * 16u;
  float c[8], h[8];                                  // rows n = 8 jj + 2 t + e1, index 2 jj + e1
#pragma unroll
  for (int i = 0; i < 8; ++i) c[i] = h[i] = 0.f;
  float acc[2][16];
  for (int s = 0; s < steps; ++s) {
    const int cur = s & 1;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // h written by the generic proxy -> tensor cores
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) acc_fence(acc[mt]);
    wgmma_fence();
    const uint32_t a0 = ws_addr + (uint32_t)(128 * wg) * (uint32_t)H * 2u;      // row 128 wg
    const uint32_t bb = hb_addr + (uint32_t)cur * LSTM_CNB * (uint32_t)H * 2u;
    for (int ks = 0; ks < H / 16; ++ks) {
      const uint64_t bd = make_noswz_desc(bb + (uint32_t)ks * 256u, 128u, sbo);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const uint64_t ad = make_noswz_desc(a0 + (uint32_t)(64 * mt) * (uint32_t)H * 2u + (uint32_t)ks * 256u, 128u, sbo);
        Wgmma<32>::mma(acc[mt], ad, bd, ks > 0 ? 1u : 0u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) acc_fence(acc[mt]);
    const uint32_t nxt = hb_addr + (uint32_t)(cur ^ 1) * LSTM_CNB * (uint32_t)H * 2u;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
#pragma unroll
      for (int e1 = 0; e1 < 2; ++e1) {
        const int n = 8 * jj + 2 * t + e1, i = 2 * jj + e1;
        const int L = len[n];
        if (s < L) {
          const int tt = dir == 0 ? s : L - 1 - s;
          const __half* gp = G + ((long long)(b0 + n) * Tn + tt) * g_row_stride + (long long)dir * 4 * H + j;
          const float zi = acc[0][4 * jj + e1] + __half2float(gp[0]);
          const float zf = acc[0][4 * jj + 2 + e1] + __half2float(gp[H]);
          const float zg = acc[1][4 * jj + e1] + __half2float(gp[2 * H]);
          const float zo = acc[1][4 * jj + 2 + e1] + __half2float(gp[3 * H]);
          c[i] = lstm_sigmoid(zf) * c[i] + lstm_sigmoid(zi) * tanhf(zg);
          h[i] = lstm_sigmoid(zo) * tanhf(c[i]);
        }
        // units u and u ^ 1 sit in lanes 4 apart: the even unit's lane stores the pair of e1 = 0 rows, the odd unit's
        // lane the pair of e1 = 1 rows, as one 32-bit store per cluster CTA
        const float other = __shfl_xor_sync(0xffffffffu, h[i], 4);
        if ((g & 1) == e1) {
          const __half2 pair = (g & 1) ? __floats2half2_rn(other, h[i]) : __floats2half2_rn(h[i], other);
          const uint32_t off = nxt + (uint32_t)lstm_cm(n, j & ~1, H) * 2u;
          const uint32_t v = *reinterpret_cast<const uint32_t*>(&pair);
          for (int q = 0; q < CS; ++q) lstm_st_cluster_b32(lstm_map_rank(off, (uint32_t)q), v);
        }
      }
    }
    lstm_cluster_sync();
  }
#pragma unroll
  for (int jj = 0; jj < 4; ++jj)
#pragma unroll
    for (int e1 = 0; e1 < 2; ++e1) {
      const int n = 8 * jj + 2 * t + e1;
      if (n < nb) y[(long long)(b0 + n) * y_row_stride + (long long)dir * H + j] = __float2half_rn(h[2 * jj + e1]);
    }
}

// cluster size of the f16 kernel for hidden size H, 0 when it takes no such H
static int lstm_cluster_size(int H) {
  if (H % 32) return 0;
  for (int cs = 1; cs <= 16; ++cs) {
    const int hs = H / cs;
    if (H % cs || hs % 32 || hs > 128 || (long long)8 * H * H / cs > LSTM_W_SMEM) continue;
    return cs;
  }
  return 0;
}

}  // namespace pv

using namespace pv;

extern "C" int pv_lstm_recurrence(const void* G, int dtype, long long g_row_stride, const float* w_hh_t,
                                  const unsigned char* mask, int B, int T, int H, int ndir, void* y,
                                  long long y_row_stride, void* stream) {
  PV_CHECK_ARG(G && w_hh_t && y, "null pointer");
  PV_CHECK_ARG(B > 0 && T > 0 && H > 0 && (ndir == 1 || ndir == 2), "bad shape B=%d T=%d H=%d ndir=%d", B, T, H, ndir);
  PV_CHECK_ARG(g_row_stride >= (long long)ndir * 4 * H && y_row_stride >= (long long)ndir * H, "row strides too small");
  if (H > LSTM_MAX_H) {
    set_error("LSTM hidden size %d unsupported (at most %d)", H, LSTM_MAX_H);
    return PV_ERR_UNSUPPORTED;
  }
  const size_t smem = (size_t)2 * LSTM_NB * H * sizeof(float);   // at most 32 KiB: no opt-in needed
  const dim3 grid((unsigned)ndir, (unsigned)cdiv(B, LSTM_NB));
  const unsigned block = (unsigned)((H + 31) / 32 * 32);
  cudaStream_t s = (cudaStream_t)stream;
  const int cs = dtype == PV_F16 ? lstm_cluster_size(H) : 0;
  if (cs > 0) {
    const int hs = H / cs;
    const size_t csmem = (size_t)H * 4 * hs * sizeof(__half) + (size_t)2 * LSTM_CNB * H * sizeof(__half);
    {
      static DeviceOnce once;
      if (once.first(current_device())) {
        PV_CUDA_OK(cudaFuncSetAttribute(lstm_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        LSTM_W_SMEM + 2 * LSTM_CNB * LSTM_MAX_H * (int)sizeof(__half)));
        PV_CUDA_OK(cudaFuncSetAttribute(lstm_cluster_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
      }
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(cs * ndir), (unsigned)cdiv(B, LSTM_CNB));
    cfg.blockDim = dim3((unsigned)(hs / 32 * 128));
    cfg.dynamicSmemBytes = csmem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)cs;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int clusters = 0;
    PV_CUDA_OK(cudaOccupancyMaxActiveClusters(&clusters, lstm_cluster_kernel, &cfg));
    if (clusters < 1) {
      set_error("LSTM: a cluster of %d CTAs with %zu B of shared memory each does not fit on this device", cs, csmem);
      return PV_ERR_UNSUPPORTED;
    }
    PV_CUDA_OK(cudaLaunchKernelEx(&cfg, lstm_cluster_kernel, (const __half*)G, g_row_stride, w_hh_t, mask, B, T, H, cs,
                                  (__half*)y, y_row_stride));
    PV_LAUNCH_OK("lstm_cluster_kernel");
    return PV_OK;
  }
  // f32 parity mode, and f16 hidden sizes without a cluster split (H not a multiple of the cluster size)
  if (dtype == PV_F16) {
    lstm_recurrence_kernel<__half><<<grid, block, smem, s>>>((const __half*)G, g_row_stride, w_hh_t, mask, B, T, H, ndir,
                                                             (__half*)y, y_row_stride);
    PV_LAUNCH_OK("lstm_recurrence_kernel<__half>");
  } else if (dtype == PV_F32) {
    lstm_recurrence_kernel<float><<<grid, block, smem, s>>>((const float*)G, g_row_stride, w_hh_t, mask, B, T, H, ndir,
                                                            (float*)y, y_row_stride);
    PV_LAUNCH_OK("lstm_recurrence_kernel<float>");
  } else {
    set_error("unsupported dtype %d", dtype);
    return PV_ERR_INVALID;
  }
  return PV_OK;
}

// Scoring a batch of fp32 query rows against a large fp32 bank (models/knn_memory.py, contrastive.py,
// losses/contrastive_loss.py): the kNN top-k and vote of KnnMemory.eval_knn, KnnMemory.update, and MoCo's queue
// cross entropy.  DESIGN.md section 2i.
//
// bank_score_kernel is one tiled fp32 FFMA product of a query tile (QT = 8 * TQ rows) with a slab of bank rows.  The
// bank streams through a two-stage cp.async ring in chunks of CHUNK rows x DK columns and is read once per query tile;
// every dot product sums its columns in ascending order with fmaf, so a similarity does not depend on the tiling.  The
// (N, M) similarities stay in registers.  What the chunk epilogue keeps depends on the mode:
//   TOPK: per query, a candidate list in shared memory.  A similarity enters when its order-preserving key reaches the
//         query's threshold; when the list could overflow it is cut to its best k by radix select and the threshold
//         becomes the k-th key.  Each CTA writes its slab's best min(k, slab rows) per query; bank_merge_vote_kernel
//         selects the best k of all slabs, sorts them and votes.
//   LSE:  per query, a running max and sum of exp over the slab's logits (MoCo's queue part of the logsumexp), combined
//         chunk by chunk in a fixed order; queue_ce_rows_kernel combines the slabs and each positive.
// Order: larger similarity first, and at equal similarity the lower bank index first (-0 equals +0; NaN ranks above
// +inf, as torch.topk).  Every reduction has a fixed order and no atomic touches a value, so repeated calls are
// bitwise identical.  Tensor cores are not used: TF32 would reorder neighbours against fp32 similarities.
#include <algorithm>

#include "pv_common.cuh"

namespace pv {
namespace bank {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int CHUNK = 256;                   // bank rows per chunk: 8 warps x 4 row groups x 8 rows
constexpr int DK = 32;                       // columns per stage (8 pieces of 16 bytes)
constexpr int MAX_SLABS = 1024;
constexpr int MODE_TOPK = 0, MODE_LSE = 1;
constexpr int HIST = 264;                    // words of one radix_select group: 256 counters and 4 results

template <int TQ> struct Cfg {
  static constexpr int QT = 8 * TQ;                          // queries per tile
  static constexpr int CAP = TQ == 4 ? 512 : 2048;           // candidate slots per query (TOPK)
  static constexpr int KMAX = CAP - CHUNK;                   // largest k
  static constexpr size_t STAGE_FLOATS = (size_t)CHUNK * DK + (size_t)QT * DK;
  static constexpr size_t SMEM_TOPK = 2 * STAGE_FLOATS * 4 + (size_t)QT * CAP * 8 + WARPS * HIST * 4 + QT * 4;
  static constexpr size_t SMEM_LSE = 2 * STAGE_FLOATS * 4 + (size_t)2 * WARPS * QT * 4 + QT * 8;
};

// order-preserving key of an fp32 similarity: -0 is +0, every NaN is the largest key
__device__ __forceinline__ uint32_t f2key(float f) {
  if (f != f) return 0xffffffffu;
  uint32_t b = __float_as_uint(f + 0.f);                     // -0 + 0 = +0
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
  if (k == 0xffffffffu) return __uint_as_float(0x7fc00000u);
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__device__ __forceinline__ void cp_async16(float* dst, const float* src, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async4(float* dst, const float* src, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(src), "r"(valid ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Rows of 32 floats; the 16-byte piece p of row r sits at piece p ^ ((r / group) & 7), so the rows one LDS.128 reads
// fall on different banks.
__device__ __forceinline__ int swz(int r, int piece, int group) { return r * DK + ((piece ^ ((r / group) & 7)) << 2); }

// One stage: bank rows [row0, row0 + CHUNK) x columns [c0, c0 + DK) and the query tile's same columns, zero-filled
// outside the bank, the queries and dim.
template <int TQ, bool VEC>
__device__ __forceinline__ void load_stage(float* bs, float* qs, const float* __restrict__ memory, long long row0,
                                           long long row_end, const float* __restrict__ q, long long qs_stride,
                                           int q0, int N, int dim, int c0) {
  constexpr int QT = Cfg<TQ>::QT;
  const int t = threadIdx.x;
  if (VEC) {
#pragma unroll
    for (int u = 0; u < CHUNK * 8 / THREADS; ++u) {
      const int p = t + u * THREADS, r = p >> 3, piece = p & 7, c = c0 + piece * 4;
      const long long row = row0 + r;
      const bool ok = row < row_end && c < dim;
      cp_async16(bs + swz(r, piece, 8), ok ? memory + row * (long long)dim + c : memory, ok);
    }
    if (t < QT * 8) {
      const int r = t >> 3, piece = t & 7, c = c0 + piece * 4;
      const bool ok = q0 + r < N && c < dim;
      cp_async16(qs + swz(r, piece, TQ), ok ? q + (long long)(q0 + r) * qs_stride + c : q, ok);
    }
  } else {
#pragma unroll 4
    for (int u = 0; u < CHUNK * DK / THREADS; ++u) {
      const int e = t + u * THREADS, r = e >> 5, c = e & 31;
      const long long row = row0 + r;
      const bool ok = row < row_end && c0 + c < dim;
      cp_async4(bs + swz(r, c >> 2, 8) + (c & 3), ok ? memory + row * (long long)dim + c0 + c : memory, ok);
    }
    for (int e = t; e < QT * DK; e += THREADS) {
      const int r = e >> 5, c = e & 31;
      const bool ok = q0 + r < N && c0 + c < dim;
      cp_async4(qs + swz(r, c >> 2, TQ) + (c & 3), ok ? q + (long long)(q0 + r) * qs_stride + c0 + c : q, ok);
    }
  }
}

// ---- radix select over a candidate list: the k-th largest (key, ~idx) pair --------------------------------------------
// G threads (a warp, or the whole block) select over n pairs at keys[i], idx[i] (shared or global memory).  Returns in
// (*tk, *ti) the key and the ~index of the k-th largest pair (k <= n); exactly k pairs have (key, ~idx) >= (tk, ti).
// hist: HIST words of this group in shared memory (256 counters, then the results of each pass).
template <int G>
__device__ __forceinline__ void group_sync() {
  if (G == 32) __syncwarp(); else __syncthreads();
}

template <int G>
__device__ void radix_select(const uint32_t* keys, const uint32_t* idx, int n, int k, uint32_t* hist,
                             uint32_t* tk, uint32_t* ti) {
  const int t = G == 32 ? (threadIdx.x & 31) : threadIdx.x;
  uint32_t prefix = 0, mask = 0, remaining = (uint32_t)k, kkey = 0;
  // pass 0 .. 3 select the key; pass 4 .. 7 the ~index among pairs whose key equals it (only when not all of them fit)
  for (int pass = 0; pass < 8; ++pass) {
    const bool on_idx = pass >= 4;
    const int shift = 24 - 8 * (pass & 3);
    if (pass == 4) {
      if (hist[256] == remaining) {                  // every pair with the k-th key is kept
        *tk = kkey;
        *ti = 0;
        return;
      }
      prefix = 0;
      mask = 0;
    }
    for (int b = t; b < 256; b += G) hist[b] = 0;
    group_sync<G>();
    for (int i = t; i < n; i += G) {
      const uint32_t kk = keys[i];
      const uint32_t v = on_idx ? ~idx[i] : kk;
      if ((!on_idx || kk == kkey) && (v & mask) == prefix) atomicAdd(&hist[(v >> shift) & 255], 1u);
    }
    group_sync<G>();
    if (t < 32) {                                    // the first warp of the group finds the digit
      const int lane = t;
      uint32_t c[8], s = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        c[j] = hist[255 - (lane * 8 + j)];
        s += c[j];
      }
      uint32_t incl = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
      }
      const uint32_t excl = incl - s;
      const bool here = excl < remaining && remaining <= incl;
      if (here) {
        uint32_t before = excl;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (before + c[j] >= remaining) {
            hist[257] = 255 - (lane * 8 + j);
            hist[258] = remaining - before;
            hist[259] = c[j];
            break;
          }
          before += c[j];
        }
      }
    }
    group_sync<G>();
    const uint32_t digit = hist[257];
    remaining = hist[258];
    const uint32_t bin = hist[259];
    prefix |= digit << shift;
    mask |= 255u << shift;
    if (pass == 3) {
      kkey = prefix;
      group_sync<G>();
      if (t == 0) hist[256] = bin;                   // pairs with the k-th key
      group_sync<G>();
    }
    group_sync<G>();
  }
  *tk = kkey;
  *ti = prefix;
}

// Keeps, in place and in their order, the pairs (key, ~idx) >= (tk, ti) of one warp's list; returns their number.
__device__ int warp_compact(uint32_t* keys, uint32_t* idx, int n, uint32_t tk, uint32_t ti) {
  const int lane = threadIdx.x & 31;
  int out = 0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    uint32_t kk = 0, ii = 0;
    bool keep = false;
    if (i < n) {
      kk = keys[i];
      ii = idx[i];
      keep = kk > tk || (kk == tk && ~ii >= ti);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    __syncwarp();
    if (keep) {
      const int pos = out + __popc(bal & ((1u << lane) - 1u));
      keys[pos] = kk;
      idx[pos] = ii;
    }
    out += __popc(bal);
    __syncwarp();
  }
  return out;
}

// ---- the scoring kernel ----------------------------------------------------------------------------------------------
// grid (slabs, query tiles).  Thread (warp w, lane): row group rg = lane >> 3 and query group qg = lane & 7; it owns the
// 8 rows w * 32 + rg * 8 + i of each chunk and the TQ queries qg * TQ + j of the tile.
// TOPK writes the slab's list to cand_key / cand_idx [N][slabs][k] (slots it leaves empty keep the caller's key 0);
// LSE writes part[N][slabs][2] = (max, sum).
template <int TQ, bool VEC, int MODE>
__global__ void __launch_bounds__(THREADS, 1)
bank_score_kernel(const float* __restrict__ q, long long q_stride, int N, const float* __restrict__ memory, long long M,
                  int dim, long long slab_rows, int k, float temperature, uint32_t* __restrict__ cand_key,
                  uint32_t* __restrict__ cand_idx, float* __restrict__ part) {
  using CF = Cfg<TQ>;
  constexpr int QT = CF::QT;
  extern __shared__ __align__(16) float smem[];
  float* stage[2] = {smem, smem + CF::STAGE_FLOATS};
  float* after = smem + 2 * CF::STAGE_FLOATS;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, rg = lane >> 3, qg = lane & 7;
  const int slab = blockIdx.x, n_slabs = gridDim.x, q0 = blockIdx.y * QT;
  const long long row_begin = (long long)slab * slab_rows;
  const long long row_end = min(M, row_begin + slab_rows);
  const int n_chunks = (int)((row_end - row_begin + CHUNK - 1) / CHUNK);
  const int nk = (dim + DK - 1) / DK;
  const int n_iter = n_chunks * nk;

  // TOPK state
  uint32_t* bkey = reinterpret_cast<uint32_t*>(after);
  uint32_t* bidx = bkey + (size_t)QT * CF::CAP;
  uint32_t* hist = bidx + (size_t)QT * CF::CAP;              // WARPS x HIST
  int* cnt = reinterpret_cast<int*>(hist + WARPS * HIST);
  __shared__ unsigned long long thr[32];                     // per query: the smallest key a list admits
  // LSE state
  float* red_m = after;
  float* red_s = red_m + WARPS * QT;
  float* run_m = red_s + WARPS * QT;
  float* run_s = run_m + QT;
  if (MODE == MODE_TOPK) {
    if (threadIdx.x < QT) {
      cnt[threadIdx.x] = 0;
      thr[threadIdx.x] = 0;                           // admit every key until a list holds k
    }
  } else if (threadIdx.x < QT) {
    run_m[threadIdx.x] = -INFINITY;
    run_s[threadIdx.x] = 0.f;
  }

  float acc[8][TQ];
  if (n_iter > 0) {
    load_stage<TQ, VEC>(stage[0], stage[0] + CHUNK * DK, memory, row_begin, row_end, q, q_stride, q0, N, dim, 0);
  }
  cp_commit();
  for (int it = 0; it < n_iter; ++it) {
    const int chunk = it / nk, ks = it % nk;
    if (it + 1 < n_iter) {
      const int c2 = (it + 1) / nk, k2 = (it + 1) % nk;
      float* s2 = stage[(it + 1) & 1];
      load_stage<TQ, VEC>(s2, s2 + CHUNK * DK, memory, row_begin + (long long)c2 * CHUNK, row_end, q, q_stride, q0, N,
                          dim, k2 * DK);
    }
    cp_commit();
    cp_wait<1>();
    __syncthreads();
    if (ks == 0) {
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TQ; ++j) acc[i][j] = 0.f;
    }
    const float* bs = stage[it & 1];
    const float* qs = bs + CHUNK * DK;
    const int rbase = w * 32 + rg * 8;
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      float4 qv[TQ];
#pragma unroll
      for (int j = 0; j < TQ; ++j) qv[j] = *reinterpret_cast<const float4*>(qs + swz(qg * TQ + j, p, TQ));
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 bv = *reinterpret_cast<const float4*>(bs + swz(rbase + i, p, 8));
#pragma unroll
        for (int j = 0; j < TQ; ++j) {
          acc[i][j] = fmaf(bv.x, qv[j].x, acc[i][j]);
          acc[i][j] = fmaf(bv.y, qv[j].y, acc[i][j]);
          acc[i][j] = fmaf(bv.z, qv[j].z, acc[i][j]);
          acc[i][j] = fmaf(bv.w, qv[j].w, acc[i][j]);
        }
      }
    }
    __syncthreads();                                   // the stage is free for the load of iteration it + 2
    if (ks != nk - 1) continue;

    const long long crow = row_begin + (long long)chunk * CHUNK + rbase;
    if (MODE == MODE_TOPK) {
#pragma unroll
      for (int j = 0; j < TQ; ++j) {
        const int ql = qg * TQ + j;
        if (q0 + ql >= N) continue;
        const unsigned long long th = thr[ql];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const uint32_t key = f2key(acc[i][j]);
          if (crow + i < row_end && (unsigned long long)key >= th) {
            const int pos = atomicAdd(&cnt[ql], 1);
            bkey[(size_t)ql * CF::CAP + pos] = key;
            bidx[(size_t)ql * CF::CAP + pos] = (uint32_t)(crow + i);
          }
        }
      }
      __syncthreads();
      const bool last = chunk == n_chunks - 1;
      for (int ql = w; ql < QT; ql += WARPS) {         // one warp cuts each list that could overflow (or ends)
        const int n = cnt[ql];
        if (n > k && (last || n > CF::CAP - CHUNK)) {
          uint32_t* hw = hist + w * HIST;
          uint32_t tk, ti;
          radix_select<32>(bkey + (size_t)ql * CF::CAP, bidx + (size_t)ql * CF::CAP, n, k, hw, &tk, &ti);
          const int kept = warp_compact(bkey + (size_t)ql * CF::CAP, bidx + (size_t)ql * CF::CAP, n, tk, ti);
          if (lane == 0) {
            cnt[ql] = kept;
            // later rows have larger indices, so they lose a tie with the k-th pair: admit keys above it only
            thr[ql] = (unsigned long long)tk + 1ull;
          }
        }
      }
      __syncthreads();
    } else {
      float m[TQ], s[TQ];
#pragma unroll
      for (int j = 0; j < TQ; ++j) {
        m[j] = -INFINITY;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          acc[i][j] = __fdiv_rn(acc[i][j], temperature);
          if (crow + i < row_end) m[j] = fmaxf(m[j], acc[i][j]);
        }
        m[j] = fmaxf(m[j], __shfl_xor_sync(0xffffffffu, m[j], 8));
        m[j] = fmaxf(m[j], __shfl_xor_sync(0xffffffffu, m[j], 16));
        if (rg == 0) red_m[w * QT + qg * TQ + j] = m[j];
      }
      __syncthreads();
#pragma unroll
      for (int j = 0; j < TQ; ++j) {
        const int ql = qg * TQ + j;
        float mc = -INFINITY;
        for (int ww = 0; ww < WARPS; ++ww) mc = fmaxf(mc, red_m[ww * QT + ql]);
        m[j] = mc;
        s[j] = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (crow + i < row_end) s[j] += expf(acc[i][j] - mc);
        s[j] += __shfl_xor_sync(0xffffffffu, s[j], 8);
        s[j] += __shfl_xor_sync(0xffffffffu, s[j], 16);
        if (rg == 0) red_s[w * QT + ql] = s[j];
      }
      __syncthreads();
      if (w == 0 && rg == 0) {
#pragma unroll
        for (int j = 0; j < TQ; ++j) {
          const int ql = qg * TQ + j;
          float sc = 0.f;
          for (int ww = 0; ww < WARPS; ++ww) sc += red_s[ww * QT + ql];
          const float mc = m[j], mo = run_m[ql];
          const float mn = fmaxf(mo, mc);
          if (mn == -INFINITY) continue;
          run_s[ql] = (mo == -INFINITY ? 0.f : run_s[ql] * expf(mo - mn)) + sc * expf(mc - mn);
          run_m[ql] = mn;
        }
      }
      __syncthreads();
    }
  }
  cp_wait<0>();

  if (MODE == MODE_TOPK) {
    for (int ql = w; ql < QT; ql += WARPS) {
      const int qn = q0 + ql;
      if (qn >= N) continue;
      const int n = cnt[ql];
      const size_t o = ((size_t)qn * n_slabs + slab) * (size_t)k;
      for (int i = lane; i < n; i += 32) {
        cand_key[o + i] = bkey[(size_t)ql * CF::CAP + i];
        cand_idx[o + i] = bidx[(size_t)ql * CF::CAP + i];
      }
    }
  } else if (threadIdx.x < QT && q0 + (int)threadIdx.x < N) {
    float* pp = part + ((size_t)(q0 + threadIdx.x) * n_slabs + slab) * 2;
    pp[0] = run_m[threadIdx.x];
    pp[1] = run_s[threadIdx.x];
  }
}

}  // namespace bank
}  // namespace pv

namespace pv {
namespace bank {

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

// ---- kNN: the best k of every slab's list, sorted, and the vote (ssl_helper.py:295-311), one block per query ---------
// preds[n][c] = sum_i onehot(label[idx_i])[c] * exp(sim_i / T) over the k neighbours in descending order, each product
// and sum rounded once: a weight of +inf gives 0 * inf = NaN in the other classes, as the reference's one-hot product.
constexpr int KMAX_ALL = 1024;
__global__ void __launch_bounds__(THREADS)
bank_merge_vote_kernel(const uint32_t* __restrict__ cand_key, const uint32_t* __restrict__ cand_idx, int n_slabs, int k,
                       const long long* __restrict__ labels, int n_classes, float temperature,
                       float* __restrict__ sim_out, long long* __restrict__ idx_out, float* __restrict__ preds,
                       int* __restrict__ flag) {
  __shared__ uint32_t hist[HIST];
  __shared__ unsigned long long sel[KMAX_ALL];
  __shared__ int lab[KMAX_ALL];
  __shared__ float wgt[KMAX_ALL];
  __shared__ int n_sel;
  const int n = blockIdx.x, t = threadIdx.x;
  const size_t base = (size_t)n * n_slabs * k;
  const int total = n_slabs * k;
  uint32_t tk, ti;
  radix_select<THREADS>(cand_key + base, cand_idx + base, total, k, hist, &tk, &ti);
  if (t == 0) n_sel = 0;
  int kp = 1;
  while (kp < k) kp <<= 1;
  for (int i = t; i < kp; i += THREADS) sel[i] = 0ull;
  __syncthreads();
  for (int i = t; i < total; i += THREADS) {
    const uint32_t kk = cand_key[base + i], ii = cand_idx[base + i];
    if (kk > tk || (kk == tk && ~ii >= ti)) sel[atomicAdd(&n_sel, 1)] = ((unsigned long long)kk << 32) | (~ii);
  }
  __syncthreads();
  for (int size = 2; size <= kp; size <<= 1) {         // bitonic sort, descending (key, then ascending index)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = t; i < kp; i += THREADS) {
        const int j = i ^ stride;
        if (j > i) {
          const bool desc = (i & size) == 0;
          const unsigned long long a = sel[i], b = sel[j];
          if ((a < b) == desc) {
            sel[i] = b;
            sel[j] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int i = t; i < k; i += THREADS) {
    const unsigned long long e = sel[i];
    const float sim = key2f((uint32_t)(e >> 32));
    const uint32_t idx = ~(uint32_t)e;
    sim_out[(size_t)n * k + i] = sim;
    idx_out[(size_t)n * k + i] = idx;
    const long long l = labels[idx];
    if (l < 0 || l >= n_classes) atomicOr(flag, 1);
    lab[i] = (int)l;
    wgt[i] = expf(__fdiv_rn(sim, temperature));
  }
  __syncthreads();
  for (int c = t; c < n_classes; c += THREADS) {
    float s = 0.f;
    for (int i = 0; i < k; ++i) s = __fadd_rn(s, __fmul_rn(lab[i] == c ? 1.f : 0.f, wgt[i]));
    preds[(size_t)n * n_classes + c] = s;
  }
}

// ---- MoCo rows (moco_v2.py:312-323, losses.py:131-133): row (j, n) has logits [q_n . key_j,n, q_n . Q_0 .. Q_K-1] / T
//      and target 0.  One warp per row: the positive's dot product, the slabs' (max, sum) in slab order, then
//      row = m + log(S e^(M - m) + e^(p - m)) - p with m = max(M, p). -------------------------------------------------
__global__ void __launch_bounds__(THREADS)
queue_ce_rows_kernel(const float* __restrict__ q, long long q_stride, int N, int dim, const float* __restrict__ keys,
                     long long key_stride, int skip_view, int n_rows, const float* __restrict__ part, int n_slabs,
                     float temperature, float* __restrict__ row_loss) {
  const int r = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= n_rows) return;
  const int j = r / N, n = r % N;
  const int v = (skip_view >= 0 && j >= skip_view) ? j + 1 : j;
  const float* qn = q + (long long)n * q_stride;
  const float* kn = keys + ((long long)v * N + n) * key_stride;
  float s = 0.f;
  for (int c = lane; c < dim; c += 32) s = fmaf(qn[c], kn[c], s);
  const float p = __fdiv_rn(warp_sum(s), temperature);
  if (lane == 0) {
    const float* pp = part + (size_t)n * n_slabs * 2;
    float M = -INFINITY;
    for (int i = 0; i < n_slabs; ++i) M = fmaxf(M, pp[2 * i]);
    float S = 0.f;
    for (int i = 0; i < n_slabs; ++i)
      if (pp[2 * i] != -INFINITY) S += pp[2 * i + 1] * expf(pp[2 * i] - M);
    const float m = fmaxf(M, p);
    const float tot = (M == -INFINITY ? 0.f : S * expf(M - m)) + expf(p - m);
    row_loss[r] = m + logf(tot) - p;
  }
}

// ---- ContrastiveLoss on materialised logits (losses.py:131-133): row = logsumexp(x / T) - x_0 / T, one block per row
__global__ void __launch_bounds__(THREADS)
logits_ce_rows_kernel(const float* __restrict__ x, long long x_stride, int L, float temperature,
                      float* __restrict__ row_loss) {
  __shared__ float red[WARPS];
  const float* xr = x + (long long)blockIdx.x * x_stride;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < L; i += THREADS) m = fmaxf(m, __fdiv_rn(xr[i], temperature));
  m = block_max(m, red);
  float s = 0.f;
  for (int i = threadIdx.x; i < L; i += THREADS) s += expf(__fdiv_rn(xr[i], temperature) - m);
  s = block_sum(s, red);
  if (threadIdx.x == 0) row_loss[blockIdx.x] = m + logf(s) - __fdiv_rn(xr[0], temperature);
}

// loss = sum(row[0..n)) / n in a fixed order (one block)
__global__ void __launch_bounds__(THREADS)
bank_mean_kernel(const float* __restrict__ row, int n, float* __restrict__ out) {
  __shared__ float red[WARPS];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += THREADS) s += row[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) *out = __fdiv_rn(s, (float)n);
}

// ---- KnnMemory.update (ssl_helper.py:245-250), one block per input row n: memory[ind[n]] =
//      normalize(x_n * m + memory[ind[n]] * (1 - m)) with the normalisation over a size-1 axis, v / max(|v|, 1e-12).
//      Only the last occurrence of an index writes, from the row as it was before the call; every block first scans
//      all indices, so an index outside [0, M) sets *flag and no block writes. --------------------------------------
__global__ void __launch_bounds__(THREADS)
bank_update_kernel(const float* __restrict__ x, long long x_stride, int N, const long long* __restrict__ ind,
                   float* __restrict__ memory, long long M, int dim, float mmt, float omm, int* __restrict__ flag) {
  const int n = blockIdx.x;
  const long long id = ind[n];
  bool bad = false, later = false;
  for (int j = threadIdx.x; j < N; j += THREADS) {
    const long long v = ind[j];
    bad |= v < 0 || v >= M;
    later |= j > n && v == id;
  }
  bad = __syncthreads_or(bad);
  later = __syncthreads_or(later);
  if (bad) {
    if (n == 0 && threadIdx.x == 0) atomicOr(flag, 1);
    return;
  }
  if (later) return;
  const float* xr = x + (long long)n * x_stride;
  float* mr = memory + id * (long long)dim;
  for (int c = threadIdx.x; c < dim; c += THREADS) {
    const float v = __fadd_rn(__fmul_rn(xr[c], mmt), __fmul_rn(mr[c], omm));
    mr[c] = __fdiv_rn(v, fmaxf(fabsf(v), 1e-12f));
  }
}

// Slabs of a launch: one wave of one CTA per SM, whole query tiles (the TOPK kernel's candidate lists take 208 KB of
// shared memory, and 242-255 registers per thread leave room for one CTA of 256 threads in either mode).  The grid is
// floor(SMs / tiles) slabs per tile, so no partial wave trails it; slabs need not be whole chunks.
struct Plan {
  int tq, n_qt, n_slabs;
  long long slab_rows;
};
static Plan make_plan(int op, int N, long long M, int k) {
  Plan p;
  p.tq = (op == 0 && k > Cfg<4>::KMAX) ? 1 : 4;
  const int qt = 8 * p.tq;
  p.n_qt = (int)pv::cdiv(N, qt);
  const int sms = pv::current_sm_count() > 0 ? pv::current_sm_count() : 132;
  long long ns = (long long)sms / p.n_qt;
  ns = std::max(1ll, std::min(ns, std::min((long long)MAX_SLABS, pv::cdiv(M, CHUNK))));
  p.slab_rows = pv::cdiv(M, ns);
  p.n_slabs = (int)pv::cdiv(M, p.slab_rows);
  return p;
}

}  // namespace bank
}  // namespace pv

using namespace pv::bank;

extern "C" int pv_bank_workspace(int op, int N, long long M, int k, long long* bytes) {
  PV_CHECK_ARG(bytes != nullptr, "null argument");
  PV_CHECK_ARG(op == 0 || op == 1, "op must be 0 (pv_bank_topk) or 1 (pv_queue_ce)");
  PV_CHECK_ARG(N >= 1 && M >= 1 && k >= 1, "bad shape N=%d M=%lld k=%d", N, M, k);
  const Plan p = make_plan(op, N, M, k);
  *bytes = op == 0 ? (long long)N * p.n_slabs * k * 8 : (long long)N * p.n_slabs * 2 * 4;
  return PV_OK;
}

extern "C" int pv_bank_topk(const float* q, long long q_row_stride, int N, const float* memory, long long M, int dim,
                            int k, const long long* labels, int n_classes, float temperature, void* workspace,
                            long long workspace_bytes, float* sim_out, long long* idx_out, float* preds, int* flag,
                            void* stream) {
  PV_CHECK_ARG(q && memory && labels && workspace && sim_out && idx_out && preds && flag, "null argument");
  PV_CHECK_ARG(N >= 1 && N <= 65535 * 8 && M >= 1 && M <= 2147483647ll && n_classes >= 1, "bad shape N=%d M=%lld C=%d",
               N, M, n_classes);
  PV_CHECK_ARG(dim >= 1 && dim <= 2048, "dim %d outside [1, 2048]", dim);
  PV_CHECK_ARG(k >= 1 && k <= 1024 && k <= M, "k %d outside [1, min(1024, M = %lld)]", k, M);
  PV_CHECK_ARG(q_row_stride >= dim, "row stride must cover dim");
  long long need = 0;
  pv_bank_workspace(0, N, M, k, &need);
  PV_CHECK_ARG(workspace_bytes >= need, "workspace of %lld bytes, %lld needed", workspace_bytes, need);
  const Plan p = make_plan(0, N, M, k);
  cudaStream_t s = (cudaStream_t)stream;
  PV_CUDA_OK(cudaMemsetAsync(flag, 0, sizeof(int), s));
  uint32_t* ck = (uint32_t*)workspace;
  uint32_t* ci = ck + (size_t)N * p.n_slabs * k;
  // slots a slab leaves empty hold key 0, below every real key (f2key never returns 0)
  PV_CUDA_OK(cudaMemsetAsync(ck, 0, (size_t)N * p.n_slabs * k * 4, s));
  const dim3 grid((unsigned)p.n_slabs, (unsigned)p.n_qt);
  const bool vec = dim % 4 == 0 && (uintptr_t)memory % 16 == 0 && (uintptr_t)q % 16 == 0 && q_row_stride % 4 == 0;
#define PV_TOPK(TQ, VEC, NAME)                                                                                       \
  do {                                                                                                               \
    PV_OPT_IN_SMEM((bank_score_kernel<TQ, VEC, MODE_TOPK>), Cfg<TQ>::SMEM_TOPK);                                     \
    bank_score_kernel<TQ, VEC, MODE_TOPK><<<grid, THREADS, Cfg<TQ>::SMEM_TOPK, s>>>(                                 \
        q, q_row_stride, N, memory, M, dim, p.slab_rows, k, temperature, ck, ci, nullptr);                  \
    PV_LAUNCH_OK(NAME);                                                                                              \
  } while (0)
  if (p.tq == 4) {
    if (vec) PV_TOPK(4, true, "bank_score_kernel<topk,32,vec4>");
    else PV_TOPK(4, false, "bank_score_kernel<topk,32,scalar>");
  } else {
    if (vec) PV_TOPK(1, true, "bank_score_kernel<topk,8,vec4>");
    else PV_TOPK(1, false, "bank_score_kernel<topk,8,scalar>");
  }
#undef PV_TOPK
  bank_merge_vote_kernel<<<N, THREADS, 0, s>>>(ck, ci, p.n_slabs, k, labels, n_classes, temperature, sim_out, idx_out,
                                               preds, flag);
  PV_LAUNCH_OK("bank_merge_vote_kernel");
  return PV_OK;
}

extern "C" int pv_bank_update(const float* x, long long x_row_stride, int N, const long long* ind, float* memory,
                              long long M, int dim, float momentum, float one_minus_momentum, int* flag, void* stream) {
  PV_CHECK_ARG(x && ind && memory && flag, "null argument");
  PV_CHECK_ARG(N >= 1 && N <= 2147483647 && M >= 1 && dim >= 1, "bad shape N=%d M=%lld dim=%d", N, M, dim);
  PV_CHECK_ARG(x_row_stride >= dim, "row stride must cover dim");
  cudaStream_t s = (cudaStream_t)stream;
  PV_CUDA_OK(cudaMemsetAsync(flag, 0, sizeof(int), s));
  bank_update_kernel<<<N, THREADS, 0, s>>>(x, x_row_stride, N, ind, memory, M, dim, momentum, one_minus_momentum, flag);
  PV_LAUNCH_OK("bank_update_kernel");
  return PV_OK;
}

extern "C" int pv_queue_ce(const float* q, long long q_row_stride, int N, int dim, const float* queue, long long K,
                           const float* keys, long long key_row_stride, int n_views, int skip_view, const float* logits,
                           long long logits_row_stride, int L, float temperature, void* workspace,
                           long long workspace_bytes, int reduce_mean, float* row_loss, float* loss, void* stream) {
  PV_CHECK_ARG(row_loss != nullptr && (!reduce_mean || loss != nullptr), "null argument");
  cudaStream_t s = (cudaStream_t)stream;
  int rows = N;
  if (logits != nullptr) {
    PV_CHECK_ARG(N >= 1 && N <= 2147483647 && L >= 1 && logits_row_stride >= L, "bad logits shape R=%d L=%d", N, L);
    logits_ce_rows_kernel<<<N, THREADS, 0, s>>>(logits, logits_row_stride, L, temperature, row_loss);
    PV_LAUNCH_OK("logits_ce_rows_kernel");
  } else {
    PV_CHECK_ARG(q && queue && keys && workspace, "null argument");
    PV_CHECK_ARG(N >= 1 && N <= 65535 * 8 && K >= 1 && K <= 2147483647ll && dim >= 1 && dim <= 2048,
                 "bad shape N=%d K=%lld dim=%d", N, K, dim);
    PV_CHECK_ARG(n_views >= 1 && skip_view >= -1 && skip_view < n_views, "bad views n_views=%d skip=%d", n_views,
                 skip_view);
    const int n_pos = n_views - (skip_view >= 0 ? 1 : 0);
    PV_CHECK_ARG(n_pos >= 1 && (long long)n_pos * N <= 2147483647ll, "no positive key block");
    PV_CHECK_ARG(q_row_stride >= dim && key_row_stride >= dim, "row strides must cover dim");
    long long need = 0;
    pv_bank_workspace(1, N, K, 1, &need);
    PV_CHECK_ARG(workspace_bytes >= need, "workspace of %lld bytes, %lld needed", workspace_bytes, need);
    const Plan p = make_plan(1, N, K, 1);
    float* part = (float*)workspace;
    const dim3 grid((unsigned)p.n_slabs, (unsigned)p.n_qt);
    const bool vec = dim % 4 == 0 && (uintptr_t)queue % 16 == 0 && (uintptr_t)q % 16 == 0 && q_row_stride % 4 == 0;
    if (vec) {
      PV_OPT_IN_SMEM((bank_score_kernel<4, true, MODE_LSE>), Cfg<4>::SMEM_LSE);
      bank_score_kernel<4, true, MODE_LSE><<<grid, THREADS, Cfg<4>::SMEM_LSE, s>>>(
          q, q_row_stride, N, queue, K, dim, p.slab_rows, 1, temperature, nullptr, nullptr, part);
      PV_LAUNCH_OK("bank_score_kernel<lse,32,vec4>");
    } else {
      PV_OPT_IN_SMEM((bank_score_kernel<4, false, MODE_LSE>), Cfg<4>::SMEM_LSE);
      bank_score_kernel<4, false, MODE_LSE><<<grid, THREADS, Cfg<4>::SMEM_LSE, s>>>(
          q, q_row_stride, N, queue, K, dim, p.slab_rows, 1, temperature, nullptr, nullptr, part);
      PV_LAUNCH_OK("bank_score_kernel<lse,32,scalar>");
    }
    rows = n_pos * N;
    queue_ce_rows_kernel<<<(unsigned)pv::cdiv(rows, WARPS), THREADS, 0, s>>>(
        q, q_row_stride, N, dim, keys, key_row_stride, skip_view, rows, part, p.n_slabs, temperature, row_loss);
    PV_LAUNCH_OK("queue_ce_rows_kernel");
  }
  if (reduce_mean) {
    bank_mean_kernel<<<1, THREADS, 0, s>>>(row_loss, rows, loss);
    PV_LAUNCH_OK("bank_mean_kernel");
  }
  return PV_OK;
}

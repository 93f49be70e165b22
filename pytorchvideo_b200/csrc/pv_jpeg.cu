// Baseline JPEG decode for frame-folder videos (data/frame_video.py): the bytes of libjpeg's default decode, as
// cv2.imdecode(IMREAD_COLOR) returns them, for a batch of streams in three launches.
//
//   host    pv_jpeg_parse: markers, Huffman lookup tables, geometry, segment byte ranges (restart intervals)
//   launch  jpeg_huffman_kernel: one single-warp CTA per sequential segment -> int16 coefficients, natural order
//   launch  jpeg_idct_islow_kernel: dequantise + ISLOW IDCT, 8 threads per block -> uint8 component planes
//   launch  jpeg_ycc_rgb_kernel<mode,T>: fancy upsampling + YCbCr->RGB, one thread per output pixel
//
// The per-element routines are __host__ __device__ so that they can be checked on a CPU against libjpeg.
#include "pv_common.cuh"

#include <stddef.h>
#include <string.h>

namespace pv {
namespace jpeg {

#define PV_HD __host__ __device__ __forceinline__

// zigzag index -> natural (row-major) index; entries past 63 are never used (a run past 63 is an error)
__constant__ unsigned char kNaturalOrder[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
static const unsigned char kNaturalOrderHost[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ---- entropy decoding ------------------------------------------------------------------------------------------
// MSB-first bit buffer over [p, end) with 0xFF00 unstuffing.  Past the end it shifts in zeros, as libjpeg does at a
// marker, and counts them: a segment whose codes consume more bits than it holds is an overrun.
struct BitReader {
  const uint8_t* p;
  const uint8_t* end;
  unsigned long long buf;
  int nbits;
  long long fed, used;   // real bits loaded, bits consumed
  PV_HD void fill() {
    while (nbits <= 56) {
      unsigned long long b = 0;
      if (p < end) {
        b = *p++;
        if (b == 0xFF) {
          if (p < end && *p == 0) ++p;
          else p = end;          // a marker inside the range: the host never makes such a range from valid data
        }
        fed += 8;
      }
      buf |= b << (56 - nbits);
      nbits += 8;
    }
  }
  PV_HD void skip(int n) { buf <<= n; nbits -= n; used += n; }
  PV_HD int bits(int n) {   // n <= 16, after a fill() that left at least n bits
    if (n == 0) return 0;
    const int v = (int)(buf >> (64 - n));
    skip(n);
    return v;
  }
};

// one Huffman symbol, or -1 for a code absent from the table
PV_HD int huff_decode(BitReader& br, const pv_jpeg_huff& t) {
  br.fill();
  const int look = t.look[br.buf >> 55];
  if (look) {
    br.skip(look >> 8);
    return look & 0xFF;
  }
  const int code16 = (int)(br.buf >> 48);
  for (int l = 10; l <= 16; ++l) {
    const int c = code16 >> (16 - l);
    if (c <= t.maxcode[l]) {
      const int i = c + t.valoff[l];
      if (i < 0 || i > 255) return -1;
      br.skip(l);
      return t.val[i];
    }
  }
  return -1;
}

PV_HD int huff_extend(int r, int s) { return r < (1 << (s - 1)) ? r + (-1 << s) + 1 : r; }

// one block: DC difference added to *pred, then the AC run/size codes; coefficients into blk (natural order, zeroed
// by the caller).  Returns 0 or PV_JPEG_BAD_CODE.
PV_HD int decode_block(BitReader& br, const pv_jpeg_huff& dc, const pv_jpeg_huff& ac, int* pred, int16_t* blk,
                       const unsigned char* natural) {
  int s = huff_decode(br, dc);
  if (s < 0 || s > 15) return PV_JPEG_BAD_CODE;
  if (s) {
    br.fill();
    s = huff_extend(br.bits(s), s);
  }
  *pred += s;
  blk[0] = (int16_t)*pred;
  for (int k = 1; k < 64; ++k) {
    const int rs = huff_decode(br, ac);
    if (rs < 0) return PV_JPEG_BAD_CODE;
    const int r = rs >> 4, sz = rs & 15;
    if (sz) {
      k += r;
      if (k > 63) return PV_JPEG_BAD_CODE;
      br.fill();
      blk[natural[k]] = (int16_t)huff_extend(br.bits(sz), sz);
    } else {
      if (r != 15) break;
      k += 15;
    }
  }
  return 0;
}

// Decodes segment `seg` of frame f into coef (the workspace's coefficient region, 16-byte aligned) with the frame's
// DC / AC tables dc[2], ac[2] (f.dc / f.ac or a copy of them).  blk is 64 int16 of 16-byte aligned scratch; blocks
// are zeroed and stored as 16-byte vectors.
PV_HD int decode_segment(const pv_jpeg_frame& f, const pv_jpeg_huff* dc, const pv_jpeg_huff* ac, const uint32_t* segs,
                         const uint8_t* data, int seg, int16_t* coef, int16_t* blk, const unsigned char* natural) {
  const long long total = (long long)f.mcus_x * f.mcus_y;
  const long long first = f.restart_interval ? (long long)seg * f.restart_interval : 0;
  const long long n_mcu = f.restart_interval ? (total - first < f.restart_interval ? total - first : f.restart_interval)
                                             : total;
  const uint8_t* stream = data + f.data_off;
  const uint32_t begin = segs[2 * (f.seg_base + seg)], end = segs[2 * (f.seg_base + seg) + 1];
  if (seg > 0 && stream[begin - 1] != 0xD0 + ((seg - 1) & 7)) return PV_JPEG_BAD_RESTART;
  BitReader br{stream + begin, stream + end, 0ull, 0, 0, 0};
  int pred[3] = {0, 0, 0};
  const int ns = f.ncomp;
  for (long long m = first; m < first + n_mcu; ++m) {
    const int mx = (int)(m % f.mcus_x), my = (int)(m / f.mcus_x);
    for (int sc = 0; sc < ns; ++sc) {
      const int c = f.scan_comp[sc];
      const int H = ns == 1 ? 1 : f.h[c], V = ns == 1 ? 1 : f.v[c];
      for (int yy = 0; yy < V; ++yy)
        for (int xx = 0; xx < H; ++xx) {
          int4* b4 = reinterpret_cast<int4*>(blk);
          for (int i = 0; i < 8; ++i) b4[i] = make_int4(0, 0, 0, 0);
          const int rc = decode_block(br, dc[f.dc_tbl[c]], ac[f.ac_tbl[c]], &pred[sc], blk, natural);
          if (rc) return rc;
          if (br.used > br.fed) return PV_JPEG_BAD_OVERRUN;
          const int by = my * V + yy, bx = mx * H + xx;
          int4* dst = reinterpret_cast<int4*>(coef + (f.block_base + f.block_off[c] + (long long)by * f.bw[c] + bx) * 64);
          for (int i = 0; i < 8; ++i) dst[i] = b4[i];
        }
    }
  }
  return 0;
}

// ---- ISLOW IDCT (the published jidctint.c integer algorithm) ----------------------------------------------------
enum : long long {
  F_0_298 = 2446, F_0_390 = 3196, F_0_541 = 4433, F_0_765 = 6270, F_0_899 = 7373, F_1_175 = 9633,
  F_1_501 = 12299, F_1_847 = 15137, F_1_961 = 16069, F_2_053 = 16819, F_2_562 = 20995, F_3_072 = 25172
};
constexpr int CONST_BITS = 13, PASS1_BITS = 2;

PV_HD long long descale(long long x, int n) { return (x + (1ll << (n - 1))) >> n; }

// the 1-D 8-point butterfly on in[0..7] (already scaled), outputs before the final descale
PV_HD void idct_1d(const long long* in, long long* out) {
  long long z2 = in[2], z3 = in[6];
  long long z1 = (z2 + z3) * F_0_541;
  const long long tmp2e = z1 + z3 * (-F_1_847);
  const long long tmp3e = z1 + z2 * F_0_765;
  z2 = in[0];
  z3 = in[4];
  const long long tmp0e = (z2 + z3) * (1ll << CONST_BITS);
  const long long tmp1e = (z2 - z3) * (1ll << CONST_BITS);
  const long long tmp10 = tmp0e + tmp3e, tmp13 = tmp0e - tmp3e, tmp11 = tmp1e + tmp2e, tmp12 = tmp1e - tmp2e;
  long long tmp0 = in[7], tmp1 = in[5], tmp2 = in[3], tmp3 = in[1];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  long long z4 = tmp1 + tmp3;
  const long long z5 = (z3 + z4) * F_1_175;
  tmp0 *= F_0_298;
  tmp1 *= F_2_053;
  tmp2 *= F_3_072;
  tmp3 *= F_1_501;
  z1 *= -F_0_899;
  z2 *= -F_2_562;
  z3 *= -F_1_961;
  z4 *= -F_0_390;
  z3 += z5;
  z4 += z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  out[0] = tmp10 + tmp3;
  out[7] = tmp10 - tmp3;
  out[1] = tmp11 + tmp2;
  out[6] = tmp11 - tmp2;
  out[2] = tmp12 + tmp1;
  out[5] = tmp12 - tmp1;
  out[3] = tmp13 + tmp0;
  out[4] = tmp13 - tmp0;
}

// libjpeg's post-IDCT range limit: x + 128 clamped to [0, 255], on the low 10 bits of x (RANGE_MASK), so values far
// out of range wrap exactly as the table lookup does
PV_HD uint8_t idct_range_limit(long long x) {
  const int t = (int)(x & 1023);
  return t < 128 ? (uint8_t)(t + 128) : t < 512 ? (uint8_t)255 : t < 896 ? (uint8_t)0 : (uint8_t)(t - 896);
}

// pass 1: column `col` of the dequantised block into ws (int32 [64], row-major)
PV_HD void idct_col(const int16_t* blk, const uint16_t* q, int col, int* ws) {
  long long in[8], out[8];
  for (int k = 0; k < 8; ++k) in[k] = (long long)blk[k * 8 + col] * q[k * 8 + col];
  idct_1d(in, out);
  for (int k = 0; k < 8; ++k) ws[k * 8 + col] = (int)descale(out[k], CONST_BITS - PASS1_BITS);
}

// pass 2: row `row` of ws into 8 samples
PV_HD void idct_row(const int* ws, int row, uint8_t* dst) {
  long long in[8], out[8];
  for (int k = 0; k < 8; ++k) in[k] = ws[row * 8 + k];
  idct_1d(in, out);
  for (int k = 0; k < 8; ++k) dst[k] = idct_range_limit(descale(out[k], CONST_BITS + PASS1_BITS + 3));
}

// ---- upsampling and colour conversion ------------------------------------------------------------------------------
PV_HD int clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

// chroma sample of output pixel (x, y) from plane p (row stride ps, real size dw x dh), libjpeg's fancy upsampling:
// h2: (3*near + far + 1 | 2) >> 2 by column parity, edge columns replicated; v2: the same with rows, edge rows
// replicated; h2v2: the 3:1 column sums of the two rows, then (3*near + far + 8 | 7) >> 4.  A plane at most 2 samples
// wide is replicated instead (libjpeg's fancy h2 paths need 3 columns).
template <int MODE>
PV_HD int chroma_at(const uint8_t* p, int ps, int dw, int dh, int x, int y) {
  if (MODE == PV_JPEG_H1V1) return p[(long long)y * ps + x];
  if (MODE == PV_JPEG_H2V1) {
    const uint8_t* r = p + (long long)y * ps;
    const int i = x >> 1;
    if (dw <= 2) return r[i];
    if ((x & 1) == 0) return i == 0 ? r[0] : (3 * r[i] + r[i - 1] + 1) >> 2;
    return i == dw - 1 ? r[i] : (3 * r[i] + r[i + 1] + 2) >> 2;
  }
  if (MODE == PV_JPEG_H1V2) {
    const int i = y >> 1;
    const int nb = clampi((y & 1) ? i + 1 : i - 1, 0, dh - 1);
    return (3 * p[(long long)i * ps + x] + p[(long long)nb * ps + x] + ((y & 1) ? 2 : 1)) >> 2;
  }
  // H2V2
  const int i = y >> 1, j = x >> 1;
  if (dw <= 2) return p[(long long)i * ps + j];
  const int nb = clampi((y & 1) ? i + 1 : i - 1, 0, dh - 1);
  const uint8_t* r0 = p + (long long)i * ps;
  const uint8_t* r1 = p + (long long)nb * ps;
  const int cs = 3 * r0[j] + r1[j];
  if ((x & 1) == 0) return j == 0 ? (cs * 4 + 8) >> 4 : (3 * cs + 3 * r0[j - 1] + r1[j - 1] + 8) >> 4;
  return j == dw - 1 ? (cs * 4 + 7) >> 4 : (3 * cs + 3 * r0[j + 1] + r1[j + 1] + 7) >> 4;
}

// jdcolor.c's integer tables, computed in place: FIX(x) = round(x * 2^16)
PV_HD void ycc_rgb(int y, int cb, int cr, uint8_t* rgb) {
  cb -= 128;
  cr -= 128;
  const long long r = y + ((91881ll * cr + 32768) >> 16);
  const long long g = y + ((-22554ll * cb + 32768 - 46802ll * cr) >> 16);
  const long long b = y + ((116130ll * cb + 32768) >> 16);
  rgb[0] = (uint8_t)(r < 0 ? 0 : r > 255 ? 255 : r);
  rgb[1] = (uint8_t)(g < 0 ? 0 : g > 255 ? 255 : g);
  rgb[2] = (uint8_t)(b < 0 ? 0 : b > 255 ? 255 : b);
}

template <int MODE>
PV_HD void pixel_rgb(const pv_jpeg_frame& f, const uint8_t* planes, int x, int y, uint8_t* rgb) {
  const uint8_t* py = planes + (f.block_base + f.block_off[0]) * 64;
  const int yv = py[(long long)y * f.bw[0] * 8 + x];
  if (MODE == PV_JPEG_GRAY) {
    rgb[0] = rgb[1] = rgb[2] = (uint8_t)yv;
    return;
  }
  const uint8_t* pb = planes + (f.block_base + f.block_off[1]) * 64;
  const uint8_t* pr = planes + (f.block_base + f.block_off[2]) * 64;
  const int cb = chroma_at<MODE>(pb, f.bw[1] * 8, f.dw[1], f.dh[1], x, y);
  const int cr = chroma_at<MODE>(pr, f.bw[2] * 8, f.dw[2], f.dh[2], x, y);
  ycc_rgb(yv, cb, cr, rgb);
}

// ---- kernels -----------------------------------------------------------------------------------------------------
constexpr int IDCT_BLOCKS = 32;            // 8x8 blocks per CTA, 8 threads each
constexpr int RGB_THREADS = 256;

// One single-warp CTA per segment (blockIdx.x): the segments spread over every SM and no warp mixes bit streams, whose
// data-dependent branches would serialise.  The warp stages the frame's four Huffman tables in shared memory, then
// lane 0 decodes the segment.
__global__ void __launch_bounds__(32)
jpeg_huffman_kernel(const pv_jpeg_frame* __restrict__ frames, int n_frames, const uint32_t* __restrict__ segs,
                    const uint8_t* __restrict__ data, int16_t* coef, int* status) {
  __shared__ pv_jpeg_huff tabs[4];                  // dc[0], dc[1], ac[0], ac[1]
  __shared__ __align__(16) int16_t blk[64];
  const long long g = blockIdx.x;
  int lo = 0, hi = n_frames - 1;   // the frame whose segments contain g
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (frames[mid].seg_base <= g) lo = mid;
    else hi = mid - 1;
  }
  const pv_jpeg_frame& f = frames[lo];
  static_assert(sizeof(pv_jpeg_huff) % 4 == 0 && offsetof(pv_jpeg_frame, ac) == offsetof(pv_jpeg_frame, dc) +
                2 * sizeof(pv_jpeg_huff), "dc and ac tables are copied as one run of words");
  const uint32_t* src = reinterpret_cast<const uint32_t*>(f.dc);
  uint32_t* dst = reinterpret_cast<uint32_t*>(tabs);
  for (int i = threadIdx.x; i < (int)(sizeof(tabs) / 4); i += 32) dst[i] = src[i];
  __syncwarp();
  if (threadIdx.x != 0) return;
  const int rc = decode_segment(f, tabs, tabs + 2, segs, data, (int)(g - f.seg_base), coef, blk, kNaturalOrder);
  if (rc) atomicOr(status + lo, rc);
}

__global__ void __launch_bounds__(IDCT_BLOCKS * 8)
jpeg_idct_islow_kernel(const pv_jpeg_frame* __restrict__ frames, const int16_t* __restrict__ coef, uint8_t* planes) {
  __shared__ int ws[IDCT_BLOCKS][64];
  const pv_jpeg_frame& f = frames[blockIdx.y];
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const int b = blockIdx.x * IDCT_BLOCKS + lb;
  const bool live = b < f.n_blocks;
  int c = 0, local = b;
  if (live) {
    c = b >= f.block_off[2] && f.ncomp == 3 ? 2 : b >= f.block_off[1] && f.ncomp == 3 ? 1 : 0;
    local = b - f.block_off[c];
    idct_col(coef + (f.block_base + b) * 64, f.qt[c], lane, ws[lb]);
  }
  __syncwarp();
  if (!live) return;
  const int by = local / f.bw[c], bx = local % f.bw[c];
  const long long stride = (long long)f.bw[c] * 8;
  uint8_t* dst = planes + (f.block_base + f.block_off[c]) * 64 + ((long long)by * 8 + lane) * stride + bx * 8;
  __align__(8) uint8_t row[8];
  idct_row(ws[lb], lane, row);
  *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<const uint2*>(row);
}

template <int MODE, typename T>
__global__ void __launch_bounds__(RGB_THREADS)
jpeg_ycc_rgb_kernel(const pv_jpeg_frame* __restrict__ frames, const uint8_t* __restrict__ planes, T* out) {
  const pv_jpeg_frame& f = frames[blockIdx.y];
  if (f.mode != MODE) return;
  const long long p = (long long)blockIdx.x * RGB_THREADS + threadIdx.x;
  if (p >= (long long)f.width * f.height) return;
  const int y = (int)(p / f.width), x = (int)(p % f.width);
  uint8_t rgb[3];
  pixel_rgb<MODE>(f, planes, x, y, rgb);
  T* o = out + f.out_off + p * 3;
  o[0] = (T)rgb[0];
  o[1] = (T)rgb[1];
  o[2] = (T)rgb[2];
}

// ---- host parser ---------------------------------------------------------------------------------------------------
struct Reader {
  const uint8_t* d;
  long long n, pos;
  bool ok;
  int u8() {
    if (pos >= n) { ok = false; return 0; }
    return d[pos++];
  }
  int u16() { const int a = u8(); return (a << 8) | u8(); }
};

// jdhuff.c's derived table: canonical codes from the 16 length counts, then the 9-bit lookahead
static int build_huff(const uint8_t* bits, const uint8_t* vals, int nsym, bool dc, pv_jpeg_huff* t) {
  memset(t, 0, sizeof(*t));
  int size[257], code[257];
  int p = 0;
  for (int l = 1; l <= 16; ++l)
    for (int i = 0; i < bits[l - 1]; ++i) size[p++] = l;
  size[p] = 0;
  int c = 0, si = size[0];
  p = 0;
  while (size[p]) {
    while (size[p] == si) code[p++] = c++;
    if (c >= (1 << si)) return PV_ERR_INVALID;   // over-subscribed lengths
    c <<= 1;
    ++si;
  }
  p = 0;
  for (int l = 1; l <= 16; ++l) {
    if (bits[l - 1]) {
      t->valoff[l] = p - code[p];
      p += bits[l - 1];
      t->maxcode[l] = code[p - 1];
    } else {
      t->maxcode[l] = -1;
    }
  }
  t->maxcode[0] = -1;
  t->maxcode[17] = 0xFFFFF;
  for (int i = 0; i < nsym; ++i) {
    if (dc && vals[i] > 15) return PV_ERR_INVALID;
    t->val[i] = vals[i];
  }
  p = 0;
  for (int l = 1; l <= 9; ++l)
    for (int i = 0; i < bits[l - 1]; ++i, ++p) {
      const int base = code[p] << (9 - l);
      for (int k = 0; k < (1 << (9 - l)); ++k) t->look[base + k] = (uint16_t)((l << 8) | vals[p]);
    }
  return PV_OK;
}

// EXIF orientation of an APP1 payload, 1 when absent or unreadable
static int exif_orientation(const uint8_t* a, long long n) {
  if (n < 14 || memcmp(a, "Exif\0\0", 6) != 0) return 1;
  const uint8_t* t = a + 6;
  const long long tn = n - 6;
  const bool le = t[0] == 'I' && t[1] == 'I';
  if (!le && !(t[0] == 'M' && t[1] == 'M')) return 1;
  auto r16 = [&](long long o) { return le ? t[o] | (t[o + 1] << 8) : (t[o] << 8) | t[o + 1]; };
  auto r32 = [&](long long o) {
    return le ? (long long)t[o] | ((long long)t[o + 1] << 8) | ((long long)t[o + 2] << 16) | ((long long)t[o + 3] << 24)
              : ((long long)t[o] << 24) | ((long long)t[o + 1] << 16) | ((long long)t[o + 2] << 8) | (long long)t[o + 3];
  };
  const long long ifd = r32(4);
  if (ifd < 8 || ifd + 2 > tn) return 1;
  const int count = r16(ifd);
  for (int i = 0; i < count; ++i) {
    const long long e = ifd + 2 + 12ll * i;
    if (e + 12 > tn) return 1;
    if (r16(e) == 0x0112) return r16(e + 8);
  }
  return 1;
}

static int reject(int code, const char* what) {
  set_error("jpeg: %s", what);
  return code;
}

static int parse(const uint8_t* data, long long len, const pv_jpeg_batch* batch, pv_jpeg_frame* f, uint32_t* segs,
                 long long seg_cap, int* n_seg_out) {
  Reader r{data, len, 0, true};
  if (r.u8() != 0xFF || r.u8() != 0xD8) return reject(PV_ERR_INVALID, "no SOI marker");
  memset(f, 0, sizeof(*f));
  uint16_t qt[4][64];
  bool qt_set[4] = {false, false, false, false};
  pv_jpeg_huff huff[2][2];   // [dc/ac][slot]
  bool huff_set[2][2] = {{false, false}, {false, false}};
  int comp_id[3] = {0, 0, 0}, comp_tq[3] = {0, 0, 0};
  bool have_sof = false, jfif = false, adobe = false;
  int adobe_transform = -1;
  while (true) {
    // next marker, skipping fill bytes
    int m = r.u8();
    if (!r.ok) return reject(PV_ERR_INVALID, "truncated before the scan");
    if (m != 0xFF) return reject(PV_ERR_INVALID, "marker expected");
    do m = r.u8(); while (m == 0xFF && r.ok);
    if (!r.ok) return reject(PV_ERR_INVALID, "truncated before the scan");
    if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x01 || m == 0x00)
      return reject(PV_ERR_INVALID, "unexpected marker before the scan");
    const long long seg_len = r.u16();
    if (!r.ok || seg_len < 2 || r.pos + seg_len - 2 > len) return reject(PV_ERR_INVALID, "truncated marker segment");
    const long long seg_end = r.pos + seg_len - 2;
    if (m == 0xC2) return reject(PV_JPEG_ERR_PROGRESSIVE, "progressive frame");
    if (m == 0xC3) return reject(PV_JPEG_ERR_LOSSLESS, "lossless frame");
    if (m == 0xC5 || m == 0xC6 || m == 0xC7 || m == 0xDE) return reject(PV_JPEG_ERR_HIERARCHICAL, "hierarchical frame");
    if ((m >= 0xC9 && m <= 0xCB) || (m >= 0xCD && m <= 0xCF) || m == 0xCC)
      return reject(PV_JPEG_ERR_ARITHMETIC, "arithmetic-coded frame");
    if (m == 0xDC) return reject(PV_JPEG_ERR_DNL, "DNL marker");
    if (m == 0xC0 || m == 0xC1) {
      if (have_sof) return reject(PV_ERR_INVALID, "second SOF");
      have_sof = true;
      const int prec = r.u8();
      f->height = r.u16();
      f->width = r.u16();
      const int nc = r.u8();
      if (!r.ok) return reject(PV_ERR_INVALID, "truncated SOF");
      if (prec != 8) return reject(PV_JPEG_ERR_PRECISION, "sample precision other than 8 bits");
      if (f->height == 0) return reject(PV_JPEG_ERR_DNL, "height defined by a DNL marker");
      if (f->width == 0) return reject(PV_ERR_INVALID, "zero width");
      if ((long long)f->width * f->height > 0x7FFFFFFFll)
        return reject(PV_ERR_UNSUPPORTED, "frame of more than 2^31 - 1 pixels");
      if (nc == 4) return reject(PV_JPEG_ERR_COLORSPACE, "CMYK / YCCK frame");
      if (nc != 1 && nc != 3) return reject(PV_JPEG_ERR_COMPONENTS, "component count other than 1 or 3");
      if (seg_len != 8 + 3 * nc) return reject(PV_ERR_INVALID, "bad SOF length");
      f->ncomp = nc;
      for (int c = 0; c < nc; ++c) {
        comp_id[c] = r.u8();
        const int hv = r.u8();
        f->h[c] = hv >> 4;
        f->v[c] = hv & 15;
        comp_tq[c] = r.u8();
        if (f->h[c] < 1 || f->h[c] > 4 || f->v[c] < 1 || f->v[c] > 4 || comp_tq[c] > 3)
          return reject(PV_ERR_INVALID, "bad component parameters");
      }
    } else if (m == 0xC4) {
      while (r.pos < seg_end) {
        const int tc_th = r.u8();
        const int tc = tc_th >> 4, th = tc_th & 15;
        uint8_t bits[16];
        int nsym = 0;
        for (int i = 0; i < 16; ++i) nsym += bits[i] = (uint8_t)r.u8();
        if (!r.ok || tc > 1 || nsym > 256 || r.pos + nsym > seg_end) return reject(PV_ERR_INVALID, "bad DHT");
        if (th > 1) return reject(PV_ERR_UNSUPPORTED, "Huffman table slot above 1");
        if (build_huff(bits, data + r.pos, nsym, tc == 0, &huff[tc][th]) != PV_OK)
          return reject(PV_ERR_INVALID, "bad Huffman table");
        huff_set[tc][th] = true;
        r.pos += nsym;
      }
    } else if (m == 0xDB) {
      while (r.pos < seg_end) {
        const int pq_tq = r.u8();
        const int pq = pq_tq >> 4, tq = pq_tq & 15;
        if (pq > 1 || tq > 3 || r.pos + 64 * (pq + 1) > seg_end) return reject(PV_ERR_INVALID, "bad DQT");
        for (int i = 0; i < 64; ++i) qt[tq][kNaturalOrderHost[i]] = (uint16_t)(pq ? r.u16() : r.u8());
        qt_set[tq] = true;
      }
    } else if (m == 0xDD) {
      if (seg_len != 4) return reject(PV_ERR_INVALID, "bad DRI");
      f->restart_interval = r.u16();
    } else if (m == 0xE0) {
      if (seg_len >= 7 && memcmp(data + r.pos, "JFIF\0", 5) == 0) jfif = true;
    } else if (m == 0xE1) {
      if (exif_orientation(data + r.pos, seg_len - 2) != 1)
        return reject(PV_JPEG_ERR_ORIENTATION, "EXIF orientation other than 1");
    } else if (m == 0xEE) {
      if (seg_len >= 14 && memcmp(data + r.pos, "Adobe", 5) == 0) {
        adobe = true;
        adobe_transform = data[r.pos + 11];
      }
    } else if (m == 0xDA) {
      if (!have_sof) return reject(PV_ERR_INVALID, "SOS before SOF");
      const int ns = r.u8();
      if (!r.ok || ns < 1 || ns > f->ncomp || seg_len != 6 + 2 * ns) return reject(PV_ERR_INVALID, "bad SOS");
      if (ns != f->ncomp) return reject(PV_JPEG_ERR_MULTISCAN, "scan with a subset of the components");
      for (int s = 0; s < ns; ++s) {
        const int id = r.u8(), tt = r.u8();
        int c = 0;
        while (c < f->ncomp && comp_id[c] != id) ++c;
        if (c == f->ncomp) return reject(PV_ERR_INVALID, "SOS names an unknown component");
        for (int k = 0; k < s; ++k)
          if (f->scan_comp[k] == c) return reject(PV_ERR_INVALID, "SOS names a component twice");
        f->scan_comp[s] = c;
        f->dc_tbl[c] = tt >> 4;
        f->ac_tbl[c] = tt & 15;
        if (f->dc_tbl[c] > 1 || f->ac_tbl[c] > 1) return reject(PV_ERR_UNSUPPORTED, "Huffman table slot above 1");
        if (!huff_set[0][f->dc_tbl[c]] || !huff_set[1][f->ac_tbl[c]]) return reject(PV_ERR_INVALID, "undefined Huffman table");
      }
      const int ss = r.u8(), se = r.u8(), ahal = r.u8();
      if (!r.ok || ss != 0 || se != 63 || ahal != 0) return reject(PV_ERR_INVALID, "non-sequential scan parameters");
      break;
    }
    r.pos = seg_end;
  }

  // colour space (jdapimin.c default_decompress_parms): 3 components are YCbCr unless an Adobe marker says RGB /
  // the ids are 'R','G','B' without JFIF or Adobe markers
  if (f->ncomp == 3) {
    if (adobe && adobe_transform != 1) return reject(PV_JPEG_ERR_COLORSPACE, "Adobe transform other than YCbCr");
    if (!jfif && !adobe && comp_id[0] == 'R' && comp_id[1] == 'G' && comp_id[2] == 'B')
      return reject(PV_JPEG_ERR_COLORSPACE, "RGB component ids");
  }
  for (int c = 0; c < f->ncomp; ++c) {
    if (!qt_set[comp_tq[c]]) return reject(PV_ERR_INVALID, "undefined quantisation table");
    memcpy(f->qt[c], qt[comp_tq[c]], sizeof(f->qt[c]));
  }
  memcpy(f->dc, huff[0], sizeof(f->dc));
  memcpy(f->ac, huff[1], sizeof(f->ac));

  // geometry
  const int W = f->width, H = f->height;
  if (f->ncomp == 1) {
    f->h[0] = f->v[0] = 1;
    f->mode = PV_JPEG_GRAY;
    f->mcus_x = (W + 7) / 8;
    f->mcus_y = (H + 7) / 8;
    f->bw[0] = f->mcus_x;
    f->bh[0] = f->mcus_y;
    f->dw[0] = W;
    f->dh[0] = H;
  } else {
    int hmax = 1, vmax = 1, bpm = 0;
    for (int c = 0; c < 3; ++c) {
      hmax = f->h[c] > hmax ? f->h[c] : hmax;
      vmax = f->v[c] > vmax ? f->v[c] : vmax;
      bpm += f->h[c] * f->v[c];
    }
    if (bpm > 10) return reject(PV_ERR_INVALID, "more than 10 blocks per MCU");
    const int rh = hmax / f->h[1], rv = vmax / f->v[1];
    if (f->h[0] != hmax || f->v[0] != vmax || f->h[1] != f->h[2] || f->v[1] != f->v[2] || hmax % f->h[1] ||
        vmax % f->v[1] || rh > 2 || rv > 2)
      return reject(PV_JPEG_ERR_SAMPLING, "chroma sampling other than 1x1, 2x1, 1x2 or 2x2 of the luma grid");
    f->mode = rh == 1 ? (rv == 1 ? PV_JPEG_H1V1 : PV_JPEG_H1V2) : (rv == 1 ? PV_JPEG_H2V1 : PV_JPEG_H2V2);
    f->mcus_x = (W + 8 * hmax - 1) / (8 * hmax);
    f->mcus_y = (H + 8 * vmax - 1) / (8 * vmax);
    for (int c = 0; c < 3; ++c) {
      f->bw[c] = f->mcus_x * f->h[c];
      f->bh[c] = f->mcus_y * f->v[c];
      f->dw[c] = (int)(((long long)W * f->h[c] + hmax - 1) / hmax);
      f->dh[c] = (int)(((long long)H * f->v[c] + vmax - 1) / vmax);
    }
  }
  long long nb = 0;
  for (int c = 0; c < f->ncomp; ++c) {
    f->block_off[c] = (int)nb;
    nb += (long long)f->bw[c] * f->bh[c];
  }
  if (nb > (1ll << 30)) return reject(PV_ERR_INVALID, "frame too large");
  f->n_blocks = (int)nb;
  const long long total_mcu = (long long)f->mcus_x * f->mcus_y;
  f->n_segments = f->restart_interval ? (int)((total_mcu + f->restart_interval - 1) / f->restart_interval) : 1;

  // entropy-coded data: segment ranges up to the first marker that is not RSTn
  const long long base = 2 * batch->n_segments;
  int nseg = 0;
  long long begin = r.pos, p = r.pos, after = -1;
  while (true) {
    const void* q = p < len ? memchr(data + p, 0xFF, (size_t)(len - p)) : nullptr;
    if (!q) return reject(PV_ERR_INVALID, "entropy-coded data runs off the buffer");
    p = (const uint8_t*)q - data;
    long long mk = p + 1;
    if (mk < len && data[mk] == 0x00) {
      p += 2;
      continue;
    }
    while (mk < len && data[mk] == 0xFF) ++mk;
    if (mk >= len) return reject(PV_ERR_INVALID, "entropy-coded data runs off the buffer");
    const int b = data[mk];
    if (b == 0x00) return reject(PV_ERR_INVALID, "fill bytes before stuffed data");
    const bool rst = b >= 0xD0 && b <= 0xD7;
    if (rst && !f->restart_interval) return reject(PV_ERR_INVALID, "RST marker without DRI");
    if (nseg >= f->n_segments) return reject(PV_ERR_INVALID, "more restart intervals than MCUs");
    if (base / 2 + nseg >= seg_cap) return reject(PV_ERR_INVALID, "segment table too small");
    if (p > 0xFFFFFFFFll) return reject(PV_ERR_INVALID, "stream above 4 GiB");
    segs[base + 2 * nseg] = (uint32_t)begin;
    segs[base + 2 * nseg + 1] = (uint32_t)p;
    ++nseg;
    if (!rst) {
      after = mk + 1;
      if (b == 0xDC) return reject(PV_JPEG_ERR_DNL, "DNL marker");
      if (b == 0xDA) return reject(PV_JPEG_ERR_MULTISCAN, "more than one scan");
      break;
    }
    begin = p = mk + 1;
  }
  if (nseg != f->n_segments) return reject(PV_ERR_INVALID, "restart marker count does not match the image size");
  // after the scan: only tables, APPn/COM and EOI may follow; a second SOS is a multi-scan file
  r.pos = after - 2;
  while (true) {
    int m = r.u8();
    if (!r.ok || m != 0xFF) return reject(PV_ERR_INVALID, "truncated after the scan");
    do m = r.u8(); while (m == 0xFF && r.ok);
    if (!r.ok) return reject(PV_ERR_INVALID, "truncated after the scan");
    if (m == 0xD9) break;
    if (m == 0xDA) return reject(PV_JPEG_ERR_MULTISCAN, "more than one scan");
    if (m == 0xDC) return reject(PV_JPEG_ERR_DNL, "DNL marker");
    const long long sl = r.u16();
    if (!r.ok || sl < 2 || r.pos + sl - 2 > len) return reject(PV_ERR_INVALID, "truncated marker segment");
    r.pos += sl - 2;
  }
  *n_seg_out = nseg;
  return PV_OK;
}

}  // namespace jpeg
}  // namespace pv

extern "C" int pv_jpeg_parse(const uint8_t* data, long long len, pv_jpeg_batch* batch, pv_jpeg_frame* frame,
                             uint32_t* segs, long long seg_cap) {
  PV_CHECK_ARG(data && batch && frame && segs && len >= 0 && seg_cap >= 0, "null or negative argument");
  int nseg = 0;
  const int rc = pv::jpeg::parse(data, len, batch, frame, segs, seg_cap, &nseg);
  if (rc != PV_OK) return rc;
  frame->data_off = batch->data_bytes;
  frame->seg_base = batch->n_segments;
  frame->block_base = batch->n_blocks;
  frame->out_off = batch->out_elems;
  const long long pixels = (long long)frame->width * frame->height;
  batch->n_frames += 1;
  batch->mode_mask |= 1 << frame->mode;
  batch->max_blocks = frame->n_blocks > batch->max_blocks ? frame->n_blocks : batch->max_blocks;
  batch->max_pixels = (int)(pixels > batch->max_pixels ? pixels : batch->max_pixels);
  batch->n_segments += nseg;
  batch->n_blocks += frame->n_blocks;
  batch->data_bytes += len;
  batch->out_elems += 3 * pixels;
  batch->ws_bytes = batch->n_blocks * 192;
  return PV_OK;
}

extern "C" int pv_jpeg_decode(const pv_jpeg_batch* batch, const pv_jpeg_frame* frames, const uint32_t* segs,
                              const uint8_t* data, void* workspace, long long workspace_bytes, void* out, int out_dtype,
                              int* status, void* stream) {
  using namespace pv::jpeg;
  PV_CHECK_ARG(batch && frames && segs && data && workspace && out && status, "null argument");
  PV_CHECK_ARG(batch->n_frames > 0 && batch->n_frames <= 65535, "1 to 65535 frames per batch");
  PV_CHECK_ARG(batch->n_segments <= 0x7FFFFFFFll, "more than 2^31 - 1 segments in one batch");
  PV_CHECK_ARG(workspace_bytes >= batch->ws_bytes, "workspace of %lld bytes, %lld needed", workspace_bytes,
               batch->ws_bytes);
  PV_CHECK_ARG((uintptr_t)workspace % 16 == 0, "workspace must be 16-byte aligned");
  PV_CHECK_ARG(out_dtype == PV_U8 || out_dtype == PV_F32, "out_dtype must be PV_U8 or PV_F32");
  cudaStream_t s = (cudaStream_t)stream;
  int16_t* coef = (int16_t*)workspace;
  uint8_t* planes = (uint8_t*)workspace + batch->n_blocks * 128;
  const int nf = batch->n_frames;
  PV_CUDA_OK(cudaMemsetAsync(status, 0, sizeof(int) * nf, s));
  jpeg_huffman_kernel<<<(unsigned)batch->n_segments, 32, 0, s>>>(frames, nf, segs, data, coef, status);
  PV_LAUNCH_OK("jpeg_huffman_kernel");
  jpeg_idct_islow_kernel<<<dim3((unsigned)pv::cdiv(batch->max_blocks, IDCT_BLOCKS), nf), IDCT_BLOCKS * 8, 0, s>>>(
      frames, coef, planes);
  PV_LAUNCH_OK("jpeg_idct_islow_kernel");
  const dim3 grid((unsigned)pv::cdiv(batch->max_pixels, RGB_THREADS), nf);
#define PV_JPEG_RGB(MODE, NAME)                                                                                    \
  if (batch->mode_mask & (1 << MODE)) {                                                                            \
    if (out_dtype == PV_U8) {                                                                                      \
      jpeg_ycc_rgb_kernel<MODE, uint8_t><<<grid, RGB_THREADS, 0, s>>>(frames, planes, (uint8_t*)out);             \
      PV_LAUNCH_OK("jpeg_ycc_rgb_kernel<" NAME ",u8>");                                                           \
    } else {                                                                                                       \
      jpeg_ycc_rgb_kernel<MODE, float><<<grid, RGB_THREADS, 0, s>>>(frames, planes, (float*)out);                 \
      PV_LAUNCH_OK("jpeg_ycc_rgb_kernel<" NAME ",f32>");                                                          \
    }                                                                                                              \
  }
  PV_JPEG_RGB(PV_JPEG_GRAY, "gray")
  PV_JPEG_RGB(PV_JPEG_H1V1, "h1v1")
  PV_JPEG_RGB(PV_JPEG_H2V1, "h2v1")
  PV_JPEG_RGB(PV_JPEG_H1V2, "h1v2")
  PV_JPEG_RGB(PV_JPEG_H2V2, "h2v2")
#undef PV_JPEG_RGB
  return PV_OK;
}

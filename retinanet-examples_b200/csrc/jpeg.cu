// jpeg.cu -- baseline JPEG decode on the GPU (the Image.open(path).convert("RGB") of odtk/data.py:50), bit-exact to
// libjpeg(-turbo)'s defaults as Pillow uses them.  Written from ITU-T T.81 and libjpeg's documented arithmetic.
//   1. jpeg_restart_kernel   one block per image: finds the RSTn markers of the scan, writes each segment's byte range
//   2. jpeg_entropy_kernel   one thread per (image, restart segment): Huffman decode into int16 coefficient blocks
//   3. jpeg_idct_kernel      one thread per 8x8 block: dequantisation + JDCT_ISLOW IDCT into uint8 component planes
//   4. jpeg_color_kernel     one thread per pixel: fancy upsampling + YCbCr -> RGB into uint8 HWC images
// Every kernel reads its sizes from the device descriptor table (n is the only size argument), so one CUDA graph
// replays for any batch of n images that fits the buffers.
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "prof.cuh"

namespace {

constexpr int JPEG_SCAN_THREADS = 256;

__constant__ unsigned char c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                           12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                           35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                           58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct SegRange {
  int start, end;   // bytes of the scan, RSTn excluded
};

struct Geometry {   // per component c: blocks across / down of its plane, first block relative to the image
  int mcux, mcuy, bw[3], bh[3], base[3];
};

__device__ __forceinline__ Geometry geometry(const odtk_jpeg_image_t &im) {
  Geometry g;
  g.mcux = (im.width + 8 * im.hmax - 1) / (8 * im.hmax);
  g.mcuy = (im.height + 8 * im.vmax - 1) / (8 * im.vmax);
  int base = 0;
  for (int c = 0; c < 3; c++) {
    g.bw[c] = c == 0 ? g.mcux * im.hmax : g.mcux;
    g.bh[c] = c == 0 ? g.mcuy * im.vmax : g.mcuy;
    g.base[c] = base;
    if (c < im.ncomp) base += g.bw[c] * g.bh[c];
  }
  return g;
}

__device__ __forceinline__ long long image_blocks(const odtk_jpeg_image_t &im) {
  const Geometry g = geometry(im);
  return (long long)g.mcux * g.mcuy * (im.hmax * im.vmax + (im.ncomp == 3 ? 2 : 0));
}

// Workspace layout [SegRange[segments], 256-byte aligned | int16 coefficients, 128 B per block | uint8 planes, 64 B per
// block].  The kernels take the totals from the device descriptor table, never from the host call: a CUDA graph captured
// with one batch and replayed with another that fits the workspace then places each region where that batch needs it.
struct WsLayout {
  long long coef, planes;   // byte offsets in the workspace
};

__host__ __device__ __forceinline__ WsLayout ws_layout(long long segments, long long blocks) {
  const long long seg_bytes = (segments * (long long)sizeof(SegRange) + 255) / 256 * 256;
  return WsLayout{seg_bytes, seg_bytes + blocks * 128};
}

__device__ __forceinline__ WsLayout ws_layout(const odtk_jpeg_image_t *tab, int n) {
  const odtk_jpeg_image_t last = tab[n - 1];
  return ws_layout((long long)last.seg_base + last.nseg, last.blk_base + image_blocks(last));
}

// image of a flat item index: the last image whose base <= item (bases ascending)
template <typename F>
__device__ __forceinline__ int find_image(const odtk_jpeg_image_t *tab, int n, long long item, F base) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (base(tab[mid]) <= item) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---- 1. restart markers -------------------------------------------------------------------------------------------
// Each thread counts the markers (0xFF followed by 0xD0-0xD7; entropy-coded 0xFF bytes are always followed by 0x00) in
// its contiguous chunk, a block scan numbers them, and marker k ends segment k and starts segment k + 1.
__global__ void __launch_bounds__(JPEG_SCAN_THREADS) jpeg_restart_kernel(const unsigned char *__restrict__ in,
                                                                         const odtk_jpeg_image_t *__restrict__ tab,
                                                                         SegRange *__restrict__ segs, int *__restrict__ status) {
  __shared__ int s_cnt[JPEG_SCAN_THREADS];
  const odtk_jpeg_image_t im = tab[blockIdx.x];
  const unsigned char *d = in + im.scan_offset;
  const int len = im.scan_bytes, nseg = im.nseg;
  SegRange *seg = segs + im.seg_base;
  if (nseg == 1) {
    if (threadIdx.x == 0) {
      seg[0] = SegRange{0, len};
      status[blockIdx.x] = 0;
    }
    return;
  }
  for (int k = threadIdx.x; k < nseg; k += blockDim.x) seg[k] = SegRange{len, len};   // missing segments: empty
  const int chunk = (len + JPEG_SCAN_THREADS - 1) / JPEG_SCAN_THREADS;
  const int p0 = min(threadIdx.x * chunk, len), p1 = min(p0 + chunk, len);
  int cnt = 0;
  for (int p = p0; p < p1; p++)
    if (d[p] == 0xFF && p + 1 < len && (d[p + 1] & 0xF8) == 0xD0) cnt++;
  s_cnt[threadIdx.x] = cnt;
  __syncthreads();
  for (int off = 1; off < JPEG_SCAN_THREADS; off <<= 1) {     // inclusive Hillis-Steele scan
    const int v = threadIdx.x >= off ? s_cnt[threadIdx.x - off] : 0;
    __syncthreads();
    s_cnt[threadIdx.x] += v;
    __syncthreads();
  }
  int k = s_cnt[threadIdx.x] - cnt;
  for (int p = p0; p < p1 && cnt; p++) {
    if (d[p] == 0xFF && p + 1 < len && (d[p + 1] & 0xF8) == 0xD0) {
      if (k < nseg - 1) {
        seg[k].end = p;
        seg[k + 1].start = p + 2;
      }
      k++;
      cnt--;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    seg[0].start = 0;
    if (s_cnt[JPEG_SCAN_THREADS - 1] >= nseg - 1) seg[nseg - 1].end = len;
    status[blockIdx.x] = s_cnt[JPEG_SCAN_THREADS - 1] == nseg - 1 ? 0 : ODTK_JPEG_BAD_RESTART;
  }
}

// ---- 2. entropy decode --------------------------------------------------------------------------------------------
// Bit reader over one segment: `acc` holds `nbits` unread bits at its low end.  0xFF 0x00 is a 0xFF data byte; any other
// byte after 0xFF, or the end of the segment, ends the data and feeds zero bits that are counted in `pad`.  More bits
// consumed than real ones were loaded (nbits < pad) means the segment ran out of data.
struct BitReader {
  const unsigned char *d;
  int pos, end, nbits, pad;
  unsigned long long acc;

  __device__ __forceinline__ void fill() {
    while (nbits <= 56) {
      unsigned b = 0;
      if (pos < end) {
        b = __ldg(d + pos);
        if (b == 0xFF) {
          if (pos + 1 < end && __ldg(d + pos + 1) == 0) {
            pos += 2;
          } else {
            pos = end;
            b = 0;
            pad += 8;
          }
        } else {
          pos++;
        }
      } else {
        pad += 8;
      }
      acc = (acc << 8) | b;
      nbits += 8;
    }
  }
  __device__ __forceinline__ unsigned peek16() const { return (unsigned)(acc >> (nbits - 16)) & 0xFFFFu; }
  __device__ __forceinline__ int bits(int s) {   // 1 <= s <= 16, nbits >= s
    nbits -= s;
    return (int)(acc >> nbits) & ((1 << s) - 1);
  }
};

__device__ __forceinline__ int huff_extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

// One symbol: 8-bit lookahead, then the canonical maxcode walk for 9..16 bits.  -1: no such code.  Needs nbits >= 16.
__device__ __forceinline__ int huff_decode(BitReader &br, const odtk_jpeg_huff_t *__restrict__ t) {
  const unsigned p = br.peek16();
  const unsigned e = __ldg(&t->look[p >> 8]);
  if (e) {
    br.nbits -= (int)(e >> 8);
    return (int)(e & 0xFF);
  }
  int l = 9;
  while (l <= 16 && (int)(p >> (16 - l)) > __ldg(&t->maxcode[l])) l++;
  if (l > 16) return -1;
  br.nbits -= l;
  return __ldg(&t->val[((int)(p >> (16 - l)) + __ldg(&t->valoff[l])) & 0xFF]);
}

// One 8x8 block into blk (64 int16, row-major).  Returns 0 or an ODTK_JPEG_* bit.
__device__ __forceinline__ int decode_block(BitReader &br, const odtk_jpeg_huff_t *__restrict__ dct,
                                            const odtk_jpeg_huff_t *__restrict__ act, int &pred, short *__restrict__ blk) {
  uint4 *b4 = reinterpret_cast<uint4 *>(blk);
#pragma unroll
  for (int i = 0; i < 8; i++) b4[i] = make_uint4(0u, 0u, 0u, 0u);
  br.fill();
  int s = huff_decode(br, dct);
  if (s < 0 || s > 16) return ODTK_JPEG_BAD_CODE;
  if (s) {
    br.fill();
    pred += huff_extend(br.bits(s), s);
  }
  blk[0] = (short)pred;
  for (int k = 1; k < 64; k++) {
    br.fill();
    const int rs = huff_decode(br, act);
    if (rs < 0) return ODTK_JPEG_BAD_CODE;
    const int r = rs >> 4;
    s = rs & 15;
    if (s) {
      k += r;
      if (k > 63) return ODTK_JPEG_BAD_INDEX;
      blk[c_zigzag[k]] = (short)huff_extend(br.bits(s), s);
    } else if (r == 15) {
      k += 15;
    } else {
      break;
    }
  }
  return br.nbits < br.pad ? ODTK_JPEG_TRUNCATED : 0;
}

__global__ void jpeg_entropy_kernel(const unsigned char *__restrict__ in, const odtk_jpeg_image_t *__restrict__ tab, int n,
                                    unsigned char *__restrict__ ws, int *__restrict__ status) {
  const SegRange *segs = reinterpret_cast<const SegRange *>(ws);
  short *coef = reinterpret_cast<short *>(ws + ws_layout(tab, n).coef);
  const int total = tab[n - 1].seg_base + tab[n - 1].nseg;
  for (int sidx = blockIdx.x * blockDim.x + threadIdx.x; sidx < total; sidx += gridDim.x * blockDim.x) {
    const int i = find_image(tab, n, sidx, [](const odtk_jpeg_image_t &t) { return (long long)t.seg_base; });
    const odtk_jpeg_image_t im = tab[i];
    const Geometry g = geometry(im);
    const int k = sidx - im.seg_base;
    const int mcus = g.mcux * g.mcuy;
    const int ri = im.restart_interval ? im.restart_interval : mcus;
    const SegRange sr = segs[sidx];
    BitReader br;
    br.d = in + im.scan_offset;
    br.pos = max(sr.start, 0);
    br.end = min(sr.end, im.scan_bytes);
    br.nbits = 0;
    br.pad = 0;
    br.acc = 0;
    int pred[3] = {0, 0, 0};
    short *cbase = coef + im.blk_base * 64;
    const odtk_jpeg_huff_t *dct[3], *act[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
      dct[c] = reinterpret_cast<const odtk_jpeg_huff_t *>(in + im.dc[c]);
      act[c] = reinterpret_cast<const odtk_jpeg_huff_t *>(in + im.ac[c]);
    }
    int err = 0;
    const int m1 = min((long long)(k + 1) * ri, (long long)mcus);
    for (int m = k * ri; m < m1 && !err; m++) {
      const int ux = m % g.mcux, uy = m / g.mcux;
      for (int c = 0; c < im.ncomp && !err; c++) {
        const int h = c == 0 ? im.hmax : 1, v = c == 0 ? im.vmax : 1;
        for (int bv = 0; bv < v && !err; bv++)
          for (int bh = 0; bh < h && !err; bh++) {
            short *blk = cbase + ((long long)g.base[c] + (long long)(uy * v + bv) * g.bw[c] + ux * h + bh) * 64;
            err = decode_block(br, dct[c], act[c], pred[c], blk);
          }
      }
    }
    if (err) atomicOr(status + i, err);
  }
}

// ---- 3. dequantisation + islow IDCT ---------------------------------------------------------------------------------
// libjpeg's JDCT_ISLOW: 13-bit constants, the column pass keeps 2 extra bits, rounding right shifts; the row pass result
// goes through the range limit (wrap to 10 bits, + 128, clamp to [0, 255]).
constexpr int IDCT_CONST_BITS = 13, IDCT_PASS1_BITS = 2;

__device__ __forceinline__ void idct_1d(int (&d)[8], int shift) {
  int z2 = d[2], z3 = d[6];
  int z1 = (z2 + z3) * 4433;                      // FIX(0.541196100)
  const int tmp2 = z1 + z3 * -15137;              // FIX(1.847759065)
  const int tmp3 = z1 + z2 * 6270;                // FIX(0.765366865)
  const int tmp0 = (d[0] + d[4]) * (1 << IDCT_CONST_BITS);
  const int tmp1 = (d[0] - d[4]) * (1 << IDCT_CONST_BITS);
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int t0 = d[7], t1 = d[5], t2 = d[3], t3 = d[1];
  z1 = t0 + t3;
  z2 = t1 + t2;
  z3 = t0 + t2;
  int z4 = t1 + t3;
  const int z5 = (z3 + z4) * 9633;                // FIX(1.175875602)
  t0 *= 2446;                                     // FIX(0.298631336)
  t1 *= 16819;                                    // FIX(2.053119869)
  t2 *= 25172;                                    // FIX(3.072711026)
  t3 *= 12299;                                    // FIX(1.501321110)
  z1 *= -7373;                                    // FIX(0.899976223)
  z2 *= -20995;                                   // FIX(2.562915447)
  z3 = z3 * -16069 + z5;                          // FIX(1.961570560)
  z4 = z4 * -3196 + z5;                           // FIX(0.390180644)
  t0 += z1 + z3;
  t1 += z2 + z4;
  t2 += z2 + z3;
  t3 += z1 + z4;
  const int r = 1 << (shift - 1);
  d[0] = (t10 + t3 + r) >> shift;
  d[7] = (t10 - t3 + r) >> shift;
  d[1] = (t11 + t2 + r) >> shift;
  d[6] = (t11 - t2 + r) >> shift;
  d[2] = (t12 + t1 + r) >> shift;
  d[5] = (t12 - t1 + r) >> shift;
  d[3] = (t13 + t0 + r) >> shift;
  d[4] = (t13 - t0 + r) >> shift;
}

__device__ __forceinline__ unsigned range_limit(int v) { return (unsigned)min(max(((v + 512) & 1023) - 384, 0), 255); }

__global__ void __launch_bounds__(128) jpeg_idct_kernel(const unsigned char *__restrict__ in,
                                                        const odtk_jpeg_image_t *__restrict__ tab, int n,
                                                        unsigned char *__restrict__ ws) {
  const WsLayout lay = ws_layout(tab, n);
  const short *coef = reinterpret_cast<const short *>(ws + lay.coef);
  unsigned char *planes = ws + lay.planes;
  const long long total = tab[n - 1].blk_base + image_blocks(tab[n - 1]);
  for (long long b = blockIdx.x * (long long)blockDim.x + threadIdx.x; b < total; b += (long long)gridDim.x * blockDim.x) {
    const int i = find_image(tab, n, b, [](const odtk_jpeg_image_t &t) { return t.blk_base; });
    const odtk_jpeg_image_t im = tab[i];
    const Geometry g = geometry(im);
    const int local = (int)(b - im.blk_base);
    const int c = im.ncomp == 3 ? (local >= g.base[2] ? 2 : local >= g.base[1] ? 1 : 0) : 0;
    const int cbase = c == 0 ? 0 : c == 1 ? g.base[1] : g.base[2], cbw = c == 0 ? g.bw[0] : g.bw[1];
    const int j = local - cbase, by = j / cbw, bx = j % cbw;
    const uint4 *q4 = reinterpret_cast<const uint4 *>(in + (c == 0 ? im.quant[0] : c == 1 ? im.quant[1] : im.quant[2]));
    const uint4 *c4 = reinterpret_cast<const uint4 *>(coef + b * 64);
    int ws[8][8];
#pragma unroll
    for (int r = 0; r < 8; r++) {
      const uint4 cv = __ldg(c4 + r), qv = __ldg(q4 + r);
      const unsigned cw[4] = {cv.x, cv.y, cv.z, cv.w}, qw[4] = {qv.x, qv.y, qv.z, qv.w};
#pragma unroll
      for (int k = 0; k < 4; k++) {
        ws[r][2 * k] = (int)(short)(cw[k] & 0xFFFF) * (int)(qw[k] & 0xFFFF);
        ws[r][2 * k + 1] = (int)(short)(cw[k] >> 16) * (int)(qw[k] >> 16);
      }
    }
#pragma unroll
    for (int col = 0; col < 8; col++) {            // pass 1: columns
      int d[8];
#pragma unroll
      for (int r = 0; r < 8; r++) d[r] = ws[r][col];
      idct_1d(d, IDCT_CONST_BITS - IDCT_PASS1_BITS);
#pragma unroll
      for (int r = 0; r < 8; r++) ws[r][col] = d[r];
    }
    unsigned char *dst = planes + (im.blk_base + cbase) * 64 + ((long long)by * 8 * cbw + bx) * 8;
    const int pitch = cbw * 8;
#pragma unroll
    for (int r = 0; r < 8; r++) {                  // pass 2: rows, range limit, one 8-byte store per row
      int d[8];
#pragma unroll
      for (int k = 0; k < 8; k++) d[k] = ws[r][k];
      idct_1d(d, IDCT_CONST_BITS + IDCT_PASS1_BITS + 3);
      uint2 o;
      o.x = range_limit(d[0]) | range_limit(d[1]) << 8 | range_limit(d[2]) << 16 | range_limit(d[3]) << 24;
      o.y = range_limit(d[4]) | range_limit(d[5]) << 8 | range_limit(d[6]) << 16 | range_limit(d[7]) << 24;
      *reinterpret_cast<uint2 *>(dst + (long long)r * pitch) = o;
    }
  }
}

// ---- 4. upsampling + colour conversion ------------------------------------------------------------------------------
// Fancy upsampling: h2v1 is (3 nearer + further + 1 | 2) >> 2 for even | odd outputs; h2v2 first forms the column sums
// 3 nearer row + further row, then (3 nearer + further + 8 | 7) >> 4.  Samples past the plane's ceil(W / h) x
// ceil(H / v) edge replicate the last one; a plane at most 2 samples wide is replicated (libjpeg's plain upsampler).
__device__ __forceinline__ int chroma(const unsigned char *__restrict__ p, int pitch, int cw, int ch, int h, int v, int y, int x) {
  const int i = x / h, r = y / v;
  if ((h == 1 && v == 1) || cw <= 2) return __ldg(p + (long long)r * pitch + i);
  const int in = (x & 1) ? min(i + 1, cw - 1) : max(i - 1, 0);
  const unsigned char *row = p + (long long)r * pitch;
  if (v == 1) return (3 * __ldg(row + i) + __ldg(row + in) + ((x & 1) ? 2 : 1)) >> 2;
  const unsigned char *nrow = p + (long long)((y & 1) ? min(r + 1, ch - 1) : max(r - 1, 0)) * pitch;
  const int t = 3 * __ldg(row + i) + __ldg(nrow + i), tn = 3 * __ldg(row + in) + __ldg(nrow + in);
  return (3 * t + tn + ((x & 1) ? 7 : 8)) >> 4;
}

__device__ __forceinline__ unsigned char clamp8(int v) { return (unsigned char)min(max(v, 0), 255); }

__global__ void __launch_bounds__(256) jpeg_color_kernel(const odtk_jpeg_image_t *__restrict__ tab, int n,
                                                         const odtk_resize_image_t *__restrict__ outs,
                                                         const unsigned char *__restrict__ ws, unsigned char *__restrict__ y) {
  const unsigned char *planes = ws + ws_layout(tab, n).planes;
  const long long total = tab[n - 1].pix_base + (long long)tab[n - 1].height * tab[n - 1].width;
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < total; q += (long long)gridDim.x * blockDim.x) {
    const int i = find_image(tab, n, q, [](const odtk_jpeg_image_t &t) { return t.pix_base; });
    const odtk_jpeg_image_t im = tab[i];
    const Geometry g = geometry(im);
    const int local = (int)(q - im.pix_base), py = local / im.width, px = local % im.width;
    const unsigned char *pl = planes + im.blk_base * 64;
    const int Y = __ldg(pl + (long long)py * g.bw[0] * 8 + px);
    unsigned char *o = y + __ldg(&outs[i].offset) + (long long)local * 3;
    if (im.ncomp == 1) {
      o[0] = o[1] = o[2] = (unsigned char)Y;
      continue;
    }
    const int cw = (im.width + im.hmax - 1) / im.hmax, ch = (im.height + im.vmax - 1) / im.vmax, pitch = g.bw[1] * 8;
    const int cb = chroma(pl + (long long)g.base[1] * 64, pitch, cw, ch, im.hmax, im.vmax, py, px) - 128;
    const int cr = chroma(pl + (long long)g.base[2] * 64, pitch, cw, ch, im.hmax, im.vmax, py, px) - 128;
    // 16-bit fixed point: FIX(1.40200) = 91881, FIX(1.77200) = 116130, FIX(0.71414) = 46802, FIX(0.34414) = 22554
    o[0] = clamp8(Y + ((91881 * cr + 32768) >> 16));
    o[1] = clamp8(Y + ((-46802 * cr - 22554 * cb + 32768) >> 16));
    o[2] = clamp8(Y + ((116130 * cb + 32768) >> 16));
  }
}

int grid_for(long long items, int threads) {
  return (int)std::min<long long>(std::max<long long>((items + threads - 1) / threads, 1), 1 << 20);
}

}  // namespace

extern "C" long long odtk_decode_jpeg(const void *in, size_t in_bytes, const odtk_jpeg_image_t *images, int n,
                                      const odtk_resize_image_t *outs, const odtk_resize_image_t *outs_dev, void *workspace,
                                      size_t workspace_bytes, void *y, size_t y_bytes, int *status, odtk_stream_t stream_) {
  if (!images || !outs || n <= 0 || n > 65535) return ODTK_E_INVALID;
  long long seg = 0, blk = 0, pix = 0;
  auto table_ok = [&](long long off, long long bytes) { return off > 0 && off % 16 == 0 && (unsigned long long)(off + bytes) <= in_bytes; };
  for (int i = 0; i < n; i++) {
    const odtk_jpeg_image_t &im = images[i];
    if (im.ncomp != 1 && im.ncomp != 3) return ODTK_E_UNSUPPORTED;
    const bool samp = im.ncomp == 1 ? (im.hmax == 1 && im.vmax == 1)
                                    : ((im.hmax == 1 && im.vmax == 1) || (im.hmax == 2 && (im.vmax == 1 || im.vmax == 2)));
    if (!samp) return ODTK_E_UNSUPPORTED;
    if (im.height <= 0 || im.width <= 0 || im.height > 65535 || im.width > 65535 || im.scan_bytes <= 0 || im.restart_interval < 0)
      return ODTK_E_INVALID;
    if ((long long)im.height * im.width > INT32_MAX) return ODTK_E_UNSUPPORTED;   // pixel indices within an image are int
    const long long mcus = (long long)((im.width + 8 * im.hmax - 1) / (8 * im.hmax)) * ((im.height + 8 * im.vmax - 1) / (8 * im.vmax));
    const long long nseg = im.restart_interval ? (mcus + im.restart_interval - 1) / im.restart_interval : 1;
    if (im.nseg != nseg || im.seg_base != seg || im.blk_base != blk || im.pix_base != pix) return ODTK_E_INVALID;
    if (im.scan_offset < 0 || (unsigned long long)(im.scan_offset + im.scan_bytes) > in_bytes) return ODTK_E_INVALID;
    for (int c = 0; c < im.ncomp; c++)
      if (!table_ok(im.quant[c], 128) || !table_ok(im.dc[c], sizeof(odtk_jpeg_huff_t)) || !table_ok(im.ac[c], sizeof(odtk_jpeg_huff_t)))
        return ODTK_E_INVALID;
    const odtk_resize_image_t &o = outs[i];
    if (o.src_h != im.height || o.src_w != im.width || o.offset < 0 ||
        (unsigned long long)o.offset + (unsigned long long)im.height * im.width * 3 > y_bytes)
      return ODTK_E_INVALID;
    seg += nseg;
    blk += mcus * (im.hmax * im.vmax + (im.ncomp == 3 ? 2 : 0));
    pix += (long long)im.height * im.width;
    if (seg > INT32_MAX || pix > INT32_MAX * 64LL) return ODTK_E_UNSUPPORTED;
  }
  const long long need = ws_layout(seg, blk).planes + blk * 64;
  if (!workspace) return need;
  if ((long long)workspace_bytes < need) return ODTK_E_WORKSPACE;
  if (!in || !outs_dev || !y || !status) return ODTK_E_INVALID;
  cudaStream_t stream = (cudaStream_t)stream_;
  const unsigned char *src = (const unsigned char *)in;
  const odtk_jpeg_image_t *tab = (const odtk_jpeg_image_t *)in;
  unsigned char *ws = (unsigned char *)workspace;
  OdtkProfScope prof(ODTK_PROF_LAYER, stream);
  jpeg_restart_kernel<<<n, JPEG_SCAN_THREADS, 0, stream>>>(src, tab, (SegRange *)ws, status);
  jpeg_entropy_kernel<<<grid_for(seg, 64), 64, 0, stream>>>(src, tab, n, ws, status);
  jpeg_idct_kernel<<<grid_for(blk, 128), 128, 0, stream>>>(src, tab, n, ws);
  jpeg_color_kernel<<<grid_for(pix, 256), 256, 0, stream>>>(tab, n, outs_dev, ws, (unsigned char *)y);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

// The stages of the JPEG decode (ITU-T T.81), as __host__ __device__ functions over one item each: the
// unstuffing of one scan byte, the Huffman decode of one subsequence from a given state, libjpeg's ISLOW
// IDCT of one block, and libjpeg-turbo's fancy upsampling + YCbCr->RGB of one output pixel.  The kernels
// of jpeg_decode.cu run them in parallel; tests/c_host/jpeg_host.cpp runs the same functions serially on
// the CPU so that their arithmetic is checked against PIL without a GPU.
#pragma once
#include <stdint.h>

#include "../../include/acnn.h"

#ifdef __CUDACC__
#define JPEG_HD __host__ __device__ __forceinline__
#else
#define JPEG_HD inline
#endif

namespace acnn {
namespace jpeg {

// Bits per subsequence of the parallel Huffman decode.
constexpr int kSubBits = 1024;
// Zero bytes after each image's unstuffed scan: the bit reader loads up to 8 bytes past its position
// and a symbol ends at most 31 bits past the end of its subsequence.
constexpr int kBitsPad = 16;

// zigzag index -> natural index; 16 extra entries of 63 as libjpeg's jpeg_natural_order, so a
// corrupt run past the end of a block lands on coefficient 63 exactly as there.
#ifdef __CUDACC__
__host__ __device__
#endif
inline int natural_order(int k) {
  const uint8_t zz[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                          41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                          30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
  return zz[k < 63 ? k : 63];
}

// ------------------------------------------------------------------------------------ unstuffing
// What byte i of an entropy-coded segment e[0, n) becomes once the stuffing and the restart markers are
// removed: 0 = dropped, 1 = kept, 2 = dropped and the next kept byte starts a restart interval.  The
// parser guarantees that inside the segment 0xFF is followed by 0x00 or a restart marker.
JPEG_HD int unstuff_class(const uint8_t* e, int64_t i, int64_t n) {
  const uint8_t b = e[i];
  const uint8_t prev = i > 0 ? e[i - 1] : 0;
  if (prev == 0xFF) return (b >= 0xD0 && b <= 0xD7) ? 2 : 0;     // stuffed 0x00, or the RSTn code
  if (b == 0xFF && i + 1 < n && e[i + 1] >= 0xD0 && e[i + 1] <= 0xD7) return 0;   // the 0xFF of RSTn
  return 1;
}

// ------------------------------------------------------------------------------------ bit reader
struct BitReader {
  const uint8_t* d;
  int64_t q;     // next byte to load
  uint64_t acc;  // bits left-aligned
  int cnt;       // valid bits in acc

  JPEG_HD void seek(const uint8_t* data, int64_t bit) {
    d = data;
    q = bit >> 3;
    acc = 0;
    cnt = 0;
    fill();
    const int skip = (int)(bit & 7);
    acc <<= skip;
    cnt -= skip;
  }
  JPEG_HD void fill() {
    while (cnt <= 56) {
      acc |= (uint64_t)d[q++] << (56 - cnt);
      cnt += 8;
    }
  }
  JPEG_HD int64_t pos() const { return q * 8 - cnt; }
  JPEG_HD uint32_t peek(int n) const { return (uint32_t)(acc >> (64 - n)); }   // 1 <= n <= 32
  JPEG_HD void skip(int n) {
    acc <<= n;
    cnt -= n;
  }
};

// One symbol of table t at the reader (which holds >= 16 bits); -1 for a bit pattern that is no code.
JPEG_HD int huff_decode(const acnn_jpeg_huff* t, BitReader& br) {
  const uint32_t code16 = br.peek(16);
  const int lk = t->look[code16 >> 7];
  if (lk) {
    br.skip(lk >> 8);
    return lk & 0xFF;
  }
  for (int l = 10; l <= 16; ++l) {
    const int code = (int)(code16 >> (16 - l));
    if (code <= t->maxcode[l]) {
      const int idx = t->valoff[l] + code;
      if (idx < 0 || idx > 255) return -1;
      br.skip(l);
      return t->vals[idx];
    }
  }
  return -1;
}

// T.81 F.2.2.1 EXTEND of an s-bit magnitude r (s <= 15)
JPEG_HD int extend(int r, int s) { return r < (1 << (s - 1)) ? r - (1 << s) + 1 : r; }

// ------------------------------------------------------------------------------------ entropy decode
// State of the decode at a symbol boundary: bit position p in the unstuffed scan (-1: unknown), the
// block c inside the MCU and the zigzag index z inside the block; nb counts the blocks completed since
// the entry state.
struct State {
  int32_t p;
  int32_t cz;   // c | z << 8
  int32_t nb;
  int32_t err;  // ACNN_JPEG_ST_* bits met on the way
};
JPEG_HD bool same_entry(const State& a, const State& b) { return a.p == b.p && a.cz == b.cz; }
JPEG_HD bool same_state(const State& a, const State& b) { return a.p == b.p && a.cz == b.cz && a.nb == b.nb; }

// Component of block c of an MCU (the luma blocks first, then one block per chroma component).
JPEG_HD int block_comp(const acnn_jpeg_desc& d, int c) {
  const int nl = d.comp[0].h * d.comp[0].v;
  return c < nl ? 0 : 1 + (c - nl);
}

// Decode symbols from state `s` while they start before bit `end`; `iend` is the end of the restart
// interval (or of the scan).  When end == iend (the last subsequence of an interval) the decode stops at
// the fill bits: fewer than 8 bits left, all ones.  A symbol that would run past iend, or a bit pattern
// that is no code, stops the decode with the error bit set.  With WRITE, the coefficients go to block
// (blk0 + blocks completed) of `coef` (int16 [64] natural order per block; DC as the difference), for
// blocks below n_store.  dc/ac: the image's tables (global or shared memory).
template <bool WRITE>
#ifdef __CUDACC__
__host__ __device__
#endif
inline State decode_run(const acnn_jpeg_desc& d, const acnn_jpeg_huff* dc, const acnn_jpeg_huff* ac,
                        const uint8_t* bits, State s, int32_t end, int32_t iend, int16_t* coef, int64_t blk0,
                        int64_t n_store) {
  BitReader br;
  br.seek(bits, s.p);
  int c = s.cz & 0xFF, z = s.cz >> 8;
  int nb = 0;
  const int bpm = d.bpm;
  int ci = block_comp(d, c);
  int64_t p = s.p;
  while (p < end) {
    br.fill();
    if (end == iend && iend - p < 8) {
      const int k = (int)(iend - p);
      if (br.peek(k) == (1u << k) - 1) break;   // fill bits
    }
    if (z == 0) {
      const int t = huff_decode(&dc[d.comp[ci].td], br);
      if (t < 0) return State{(int32_t)p, c | z << 8, nb, ACNN_JPEG_ST_BAD_CODE};
      int v = 0;
      if (t) {
        v = extend((int)br.peek(t), t);
        br.skip(t);
      }
      if (WRITE) {
        const int64_t b = blk0 + nb;
        if (b >= 0 && b < n_store) coef[b * 64] = (int16_t)v;
      }
      z = 1;
    } else {
      const int rs = huff_decode(&ac[d.comp[ci].ta], br);
      if (rs < 0) return State{(int32_t)p, c | z << 8, nb, ACNN_JPEG_ST_BAD_CODE};
      const int r = rs >> 4, sz = rs & 15;
      if (sz) {
        z += r;
        const int v = extend((int)br.peek(sz), sz);
        br.skip(sz);
        if (WRITE) {
          const int64_t b = blk0 + nb;
          if (b >= 0 && b < n_store) coef[b * 64 + natural_order(z)] = (int16_t)v;
        }
        ++z;
      } else if (r == 15) {
        z += 16;
      } else {
        z = 64;   // EOB
      }
    }
    if (z >= 64) {
      z = 0;
      ++nb;
      c = c + 1 == bpm ? 0 : c + 1;
      ci = block_comp(d, c);
    }
    p = br.pos();
    if (p > iend) return State{(int32_t)p, c | z << 8, nb, ACNN_JPEG_ST_OUT_OF_BITS};
  }
  return State{(int32_t)p, c | z << 8, nb, 0};
}

// ------------------------------------------------------------------------------------ IDCT
// libjpeg's jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2) on coefficients times quant (both int16, the
// product in int as DEQUANTIZE), with its descale and range limit (idct_range_limit: the 10-bit wrap).
JPEG_HD uint8_t idct_range_limit(int64_t x) {
  int v = (int)(x & 1023);
  if (v >= 512) v -= 1024;
  v += 128;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

#ifdef __CUDACC__
__host__ __device__
#endif
inline void idct_islow(const int16_t* in, const int16_t* quant, uint8_t* out, int64_t stride) {
  constexpr int CB = 13, PB = 2;
  constexpr int64_t F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633,
                    F1501 = 12299, F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
  int ws[64];
  for (int col = 0; col < 8; ++col) {
    int dq[8];
    for (int r = 0; r < 8; ++r) dq[r] = (int)in[r * 8 + col] * (int)quant[r * 8 + col];
    if (!(dq[1] | dq[2] | dq[3] | dq[4] | dq[5] | dq[6] | dq[7])) {
      const int dc = (int)((uint32_t)dq[0] << PB);
      for (int r = 0; r < 8; ++r) ws[r * 8 + col] = dc;
      continue;
    }
    int64_t z2 = dq[2], z3 = dq[6];
    int64_t z1 = (z2 + z3) * F0541;
    int64_t tmp2 = z1 + z3 * -F1847;
    int64_t tmp3 = z1 + z2 * F0765;
    z2 = dq[0];
    z3 = dq[4];
    int64_t tmp0 = (z2 + z3) * (1 << CB);
    int64_t tmp1 = (z2 - z3) * (1 << CB);
    const int64_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = dq[7];
    tmp1 = dq[5];
    tmp2 = dq[3];
    tmp3 = dq[1];
    z1 = tmp0 + tmp3;
    z2 = tmp1 + tmp2;
    z3 = tmp0 + tmp2;
    int64_t z4 = tmp1 + tmp3;
    const int64_t z5 = (z3 + z4) * F1175;
    tmp0 *= F0298;
    tmp1 *= F2053;
    tmp2 *= F3072;
    tmp3 *= F1501;
    z1 *= -F0899;
    z2 *= -F2562;
    z3 *= -F1961;
    z4 *= -F0390;
    z3 += z5;
    z4 += z5;
    tmp0 += z1 + z3;
    tmp1 += z2 + z4;
    tmp2 += z2 + z3;
    tmp3 += z1 + z4;
    constexpr int sh = CB - PB;
    constexpr int64_t rnd = (int64_t)1 << (sh - 1);
    ws[0 * 8 + col] = (int)((tmp10 + tmp3 + rnd) >> sh);
    ws[7 * 8 + col] = (int)((tmp10 - tmp3 + rnd) >> sh);
    ws[1 * 8 + col] = (int)((tmp11 + tmp2 + rnd) >> sh);
    ws[6 * 8 + col] = (int)((tmp11 - tmp2 + rnd) >> sh);
    ws[2 * 8 + col] = (int)((tmp12 + tmp1 + rnd) >> sh);
    ws[5 * 8 + col] = (int)((tmp12 - tmp1 + rnd) >> sh);
    ws[3 * 8 + col] = (int)((tmp13 + tmp0 + rnd) >> sh);
    ws[4 * 8 + col] = (int)((tmp13 - tmp0 + rnd) >> sh);
  }
  for (int row = 0; row < 8; ++row) {
    const int* w = ws + row * 8;
    uint8_t* o = out + row * stride;
    if (!(w[1] | w[2] | w[3] | w[4] | w[5] | w[6] | w[7])) {
      const uint8_t v = idct_range_limit(((int64_t)w[0] + (1 << (PB + 2))) >> (PB + 3));
      for (int k = 0; k < 8; ++k) o[k] = v;
      continue;
    }
    int64_t z2 = w[2], z3 = w[6];
    int64_t z1 = (z2 + z3) * F0541;
    int64_t tmp2 = z1 + z3 * -F1847;
    int64_t tmp3 = z1 + z2 * F0765;
    int64_t tmp0 = ((int64_t)w[0] + w[4]) * (1 << CB);
    int64_t tmp1 = ((int64_t)w[0] - w[4]) * (1 << CB);
    const int64_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = w[7];
    tmp1 = w[5];
    tmp2 = w[3];
    tmp3 = w[1];
    z1 = tmp0 + tmp3;
    z2 = tmp1 + tmp2;
    z3 = tmp0 + tmp2;
    int64_t z4 = tmp1 + tmp3;
    const int64_t z5 = (z3 + z4) * F1175;
    tmp0 *= F0298;
    tmp1 *= F2053;
    tmp2 *= F3072;
    tmp3 *= F1501;
    z1 *= -F0899;
    z2 *= -F2562;
    z3 *= -F1961;
    z4 *= -F0390;
    z3 += z5;
    z4 += z5;
    tmp0 += z1 + z3;
    tmp1 += z2 + z4;
    tmp2 += z2 + z3;
    tmp3 += z1 + z4;
    constexpr int sh = CB + PB + 3;
    constexpr int64_t rnd = (int64_t)1 << (sh - 1);
    o[0] = idct_range_limit((tmp10 + tmp3 + rnd) >> sh);
    o[7] = idct_range_limit((tmp10 - tmp3 + rnd) >> sh);
    o[1] = idct_range_limit((tmp11 + tmp2 + rnd) >> sh);
    o[6] = idct_range_limit((tmp11 - tmp2 + rnd) >> sh);
    o[2] = idct_range_limit((tmp12 + tmp1 + rnd) >> sh);
    o[5] = idct_range_limit((tmp12 - tmp1 + rnd) >> sh);
    o[3] = idct_range_limit((tmp13 + tmp0 + rnd) >> sh);
    o[4] = idct_range_limit((tmp13 - tmp0 + rnd) >> sh);
  }
}

// ------------------------------------------------------------------------------------ pixels
// A component plane holding the IDCT output of MCU rows r0.. and columns c0.. of the image.
struct Plane {
  const uint8_t* p;
  int64_t pitch;
  int32_t y0, x0;   // component sample coordinates of p[0]
  int32_t dw, dh;   // the component's sample columns / rows (the upsampling edges)
  JPEG_HD int at(int y, int x) const { return p[(int64_t)(y - y0) * pitch + (x - x0)]; }
};

// Chroma sample of output pixel (y, x) (libjpeg-turbo jdsample.c): h2v1 / h2v2 fancy (triangular)
// upsampling when the plane is wider than 2 samples, else replication; h1v2 fancy always; the rows
// above the first and below the last are the edge rows, the columns likewise.
JPEG_HD int chroma_sample(const Plane& c, int hmax, int vmax, int y, int x) {
  if (hmax == 1 && vmax == 1) return c.at(y, x);
  if (hmax == 1) {   // h1v2
    const int cy = y >> 1;
    if (y & 1) return (3 * c.at(cy, x) + c.at(cy + 1 < c.dh ? cy + 1 : cy, x) + 2) >> 2;
    return (3 * c.at(cy, x) + c.at(cy > 0 ? cy - 1 : 0, x) + 1) >> 2;
  }
  const int cx = x >> 1;
  const int cy = vmax == 2 ? y >> 1 : y;
  if (c.dw <= 2) return c.at(cy, cx);
  const int nx = (x & 1) ? (cx + 1 < c.dw ? cx + 1 : cx) : (cx > 0 ? cx - 1 : 0);
  if (vmax == 1) {   // h2v1
    return (x & 1) ? (3 * c.at(cy, cx) + c.at(cy, nx) + 2) >> 2 : (3 * c.at(cy, cx) + c.at(cy, nx) + 1) >> 2;
  }
  const int ny = (y & 1) ? (cy + 1 < c.dh ? cy + 1 : cy) : (cy > 0 ? cy - 1 : 0);   // h2v2
  const int here = 3 * c.at(cy, cx) + c.at(ny, cx);
  const int next = 3 * c.at(cy, nx) + c.at(ny, nx);
  return (3 * here + next + ((x & 1) ? 7 : 8)) >> 4;
}

// libjpeg's ycc_rgb_convert (jdcolor.c): 16-bit fixed point tables, range limited.
JPEG_HD uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }
JPEG_HD void ycc_to_rgb(int y, int cb, int cr, uint8_t* o) {
  constexpr int64_t half = (int64_t)1 << 15;
  const int64_t xb = cb - 128, xr = cr - 128;
  const int r_off = (int)((91881 * xr + half) >> 16);
  const int b_off = (int)((116130 * xb + half) >> 16);
  const int g_off = (int)((-46802 * xr + (-22554 * xb + half)) >> 16);
  o[0] = clamp255(y + r_off);
  o[1] = clamp255(y + g_off);
  o[2] = clamp255(y + b_off);
}

// RGB of output pixel (y, x) of the image (grayscale replicated, as convert("RGB")).
JPEG_HD void pixel_rgb(const acnn_jpeg_desc& d, const Plane* pl, int y, int x, uint8_t* o) {
  const int Y = pl[0].at(y, x);
  if (d.ncomp == 1) {
    o[0] = o[1] = o[2] = (uint8_t)Y;
    return;
  }
  ycc_to_rgb(Y, chroma_sample(pl[1], d.hmax, d.vmax, y, x), chroma_sample(pl[2], d.hmax, d.vmax, y, x), o);
}

}  // namespace jpeg
}  // namespace acnn

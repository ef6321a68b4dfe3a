// Host side of the JPEG decoder: the header parser (ITU-T T.81 B.2, libjpeg's colour-space rules for
// 3-component frames) and the batch planner of acnn_jpeg_decode.  No CUDA call.
#include <string.h>

#include <algorithm>

#include "common.h"
#include "jpeg_stages.cuh"

namespace acnn {
namespace {

constexpr int64_t kMaxPixels = 89478485;   // PIL's Image.MAX_IMAGE_PIXELS
constexpr int64_t kMaxScan = (int64_t)1 << 27;

int be16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

struct Parser {
  const uint8_t* b;
  int64_t n;
  acnn_jpeg_desc* d;
  bool have_q[4] = {}, have_dc[2] = {}, have_ac[2] = {}, jfif = false, adobe = false, seen_sof = false;
  int adobe_transform = -1;
  int comp_id[3] = {};

  int fail(int reason) {
    d->supported = 0;
    d->reason = reason;
    return reason;
  }

  // T.81 C: the canonical code of every symbol, then the decoding form of acnn_jpeg_huff.  Returns
  // ACNN_JPEG_OK, MALFORMED (more codes than lengths allow, libjpeg's JERR_BAD_HUFF_TABLE; a DC symbol
  // above 15) or LAYOUT (an all-ones code, which T.81 reserves and the interval-end rule relies on).
  int build_huff(acnn_jpeg_huff* t, const uint8_t* counts, const uint8_t* vals, int nvals, bool is_dc) {
    memset(t, 0, sizeof(*t));
    memcpy(t->vals, vals, nvals);
    for (int i = 0; i < nvals; ++i)
      if (is_dc && vals[i] > 15) return ACNN_JPEG_MALFORMED;
    int64_t kraft = 0;   // more codes than the lengths allow (libjpeg's code overflow check)
    for (int l = 1; l <= 16; ++l) kraft += (int64_t)counts[l - 1] << (16 - l);
    if (kraft > (1 << 16)) return ACNN_JPEG_MALFORMED;
    int code = 0, k = 0;
    t->maxcode[0] = -1;
    for (int l = 1; l <= 16; ++l) {
      const int cnt = counts[l - 1];
      t->valoff[l] = k - code;
      for (int i = 0; i < cnt; ++i, ++k, ++code) {
        if (code >= (1 << l)) return ACNN_JPEG_MALFORMED;
        if (code == (1 << l) - 1) return ACNN_JPEG_LAYOUT;
        if (l <= 9) {
          const int lo = code << (9 - l), hi = (code + 1) << (9 - l);
          for (int e = lo; e < hi; ++e) t->look[e] = (uint16_t)((l << 8) | vals[k]);
        }
      }
      t->maxcode[l] = cnt ? code - 1 : -1;
      code <<= 1;
    }
    t->maxcode[17] = 0x7fffffff;
    return ACNN_JPEG_OK;
  }

  int dqt(const uint8_t* s, int len) {
    int i = 0;
    while (i < len) {
      const int pq = s[i] >> 4, tq = s[i] & 15;
      if (pq > 1 || tq > 3) return fail(ACNN_JPEG_MALFORMED);
      const int need = 1 + 64 * (pq + 1);
      if (i + need > len) return fail(ACNN_JPEG_MALFORMED);
      for (int k = 0; k < 64; ++k) {
        const int v = pq ? be16(s + i + 1 + 2 * k) : s[i + 1 + k];
        d->quant[tq][jpeg::natural_order(k)] = (int16_t)v;   // libjpeg's (ISLOW_MULT_TYPE) cast
      }
      have_q[tq] = true;
      i += need;
    }
    return ACNN_JPEG_OK;
  }

  int dht(const uint8_t* s, int len) {
    int i = 0;
    while (i < len) {
      if (i + 17 > len) return fail(ACNN_JPEG_MALFORMED);
      const int tc = s[i] >> 4, th = s[i] & 15;
      if (tc > 1 || th > 3) return fail(ACNN_JPEG_MALFORMED);
      int nvals = 0;
      for (int l = 0; l < 16; ++l) nvals += s[i + 1 + l];
      if (nvals > 256 || i + 17 + nvals > len) return fail(ACNN_JPEG_MALFORMED);
      if (th > 1) return fail(ACNN_JPEG_LAYOUT);
      const int r = build_huff(tc ? &d->ac[th] : &d->dc[th], s + i + 1, s + i + 17, nvals, tc == 0);
      if (r) return fail(r);
      (tc ? have_ac : have_dc)[th] = true;
      i += 17 + nvals;
    }
    return ACNN_JPEG_OK;
  }

  int sof(int marker, const uint8_t* s, int len) {
    if (seen_sof) return fail(ACNN_JPEG_LAYOUT);
    seen_sof = true;
    if (len < 6) return fail(ACNN_JPEG_MALFORMED);
    const int P = s[0], H = be16(s + 1), W = be16(s + 3), nf = s[5];
    if (len != 6 + 3 * nf || nf == 0) return fail(ACNN_JPEG_MALFORMED);
    d->height = H;
    d->width = W;
    if (marker != 0xC0 && marker != 0xC1) return fail(ACNN_JPEG_PROCESS);
    if (P != 8) return fail(ACNN_JPEG_PRECISION);
    if (W == 0) return fail(ACNN_JPEG_MALFORMED);
    if (H == 0) return fail(ACNN_JPEG_LAYOUT);   // DNL
    if (nf != 1 && nf != 3) return fail(ACNN_JPEG_COLOR);
    if ((int64_t)H * W > kMaxPixels) return fail(ACNN_JPEG_SIZE);
    d->ncomp = nf;
    for (int c = 0; c < nf; ++c) {
      const uint8_t* q = s + 6 + 3 * c;
      comp_id[c] = q[0];
      d->comp[c].h = q[1] >> 4;
      d->comp[c].v = q[1] & 15;
      d->comp[c].tq = q[2];
      if (d->comp[c].h < 1 || d->comp[c].h > 4 || d->comp[c].v < 1 || d->comp[c].v > 4 || q[2] > 3)
        return fail(ACNN_JPEG_MALFORMED);
      for (int e = 0; e < c; ++e)
        if (comp_id[e] == comp_id[c]) return fail(ACNN_JPEG_MALFORMED);
    }
    if (nf == 1) {
      // a single-component scan is not interleaved: one block per MCU whatever the sampling factors
      d->comp[0].h = d->comp[0].v = 1;
    } else {
      const int h0 = d->comp[0].h, v0 = d->comp[0].v;
      const bool luma_ok = (h0 == 1 || h0 == 2) && (v0 == 1 || v0 == 2);
      for (int c = 1; c < 3; ++c)
        if (d->comp[c].h != 1 || d->comp[c].v != 1) return fail(ACNN_JPEG_SAMPLING);
      if (!luma_ok) return fail(ACNN_JPEG_SAMPLING);
    }
    d->hmax = d->comp[0].h;
    d->vmax = d->comp[0].v;
    d->bpm = 0;
    for (int c = 0; c < nf; ++c) {
      d->comp[c].blk0 = d->bpm;
      d->bpm += d->comp[c].h * d->comp[c].v;
      d->comp[c].dw = (int)(((int64_t)W * d->comp[c].h + d->hmax - 1) / d->hmax);
      d->comp[c].dh = (int)(((int64_t)H * d->comp[c].v + d->vmax - 1) / d->vmax);
    }
    d->mcus_x = (W + 8 * d->hmax - 1) / (8 * d->hmax);
    d->mcus_y = (H + 8 * d->vmax - 1) / (8 * d->vmax);
    return ACNN_JPEG_OK;
  }

  int sos(const uint8_t* s, int len, int64_t ecs) {
    if (!seen_sof) return fail(ACNN_JPEG_MALFORMED);
    if (len < 1) return fail(ACNN_JPEG_MALFORMED);
    const int ns = s[0];
    if (len != 4 + 2 * ns || ns < 1 || ns > 4) return fail(ACNN_JPEG_MALFORMED);
    if (ns != d->ncomp) return fail(ACNN_JPEG_LAYOUT);   // not one interleaved scan of every component
    for (int i = 0; i < ns; ++i) {
      if (s[1 + 2 * i] != comp_id[i]) return fail(ACNN_JPEG_LAYOUT);
      const int td = s[2 + 2 * i] >> 4, ta = s[2 + 2 * i] & 15;
      if (td > 1 || ta > 1) return fail(ACNN_JPEG_LAYOUT);
      d->comp[i].td = td;
      d->comp[i].ta = ta;
      // libjpeg substitutes the T.81 K.3 tables for missing ones; that is left to it
      if (!have_dc[td] || !have_ac[ta]) return fail(ACNN_JPEG_LAYOUT);
      if (!have_q[d->comp[i].tq]) return fail(ACNN_JPEG_MALFORMED);
    }
    const int ss = s[1 + 2 * ns], se = s[2 + 2 * ns], ahl = s[3 + 2 * ns];
    if (ss != 0 || se != 63 || ahl != 0) return fail(ACNN_JPEG_MALFORMED);
    // libjpeg's default_decompress_parms: which 3-component frames are YCbCr
    if (d->ncomp == 3 && !jfif) {
      if (adobe ? adobe_transform == 0 : (comp_id[0] == 'R' && comp_id[1] == 'G' && comp_id[2] == 'B'))
        return fail(ACNN_JPEG_COLOR);
    }
    // the entropy-coded segment: up to the first marker other than RSTn; the restart markers must be
    // numbered in sequence and come only with a restart interval
    int64_t i = ecs;
    int rst = 0;
    const uint8_t* e = b;
    while (true) {
      const void* f = i < n ? memchr(e + i, 0xFF, (size_t)(n - i)) : nullptr;
      if (!f) {
        i = n;   // truncated: the decode reports it
        break;
      }
      i = (const uint8_t*)f - e;
      if (i + 1 >= n) break;   // a lone 0xFF at the end of the buffer
      const uint8_t m = e[i + 1];
      if (m == 0x00) {
        i += 2;
        continue;
      }
      if (m >= 0xD0 && m <= 0xD7) {
        if (d->restart_interval == 0 || m != 0xD0 + (rst & 7)) return fail(ACNN_JPEG_LAYOUT);
        ++rst;
        i += 2;
        continue;
      }
      if (m != 0xD9) return fail(ACNN_JPEG_LAYOUT);   // fill bytes, DNL, a second scan, ...
      break;
    }
    d->ecs_offset = ecs;
    d->ecs_length = i - ecs;
    d->n_intervals = rst + 1;
    if (d->ecs_length >= kMaxScan) return fail(ACNN_JPEG_SIZE);
    d->supported = 1;
    d->reason = ACNN_JPEG_OK;
    return ACNN_JPEG_OK;
  }

  int run() {
    if (n < 2 || b[0] != 0xFF || b[1] != 0xD8) return fail(ACNN_JPEG_NOT_JPEG);
    int64_t p = 2;
    while (true) {
      if (p >= n) return fail(ACNN_JPEG_TRUNCATED);
      if (b[p] != 0xFF) return fail(ACNN_JPEG_LAYOUT);   // bytes between segments (libjpeg skips them)
      while (p < n && b[p] == 0xFF) ++p;
      if (p >= n) return fail(ACNN_JPEG_TRUNCATED);
      const int m = b[p++];
      if (m == 0xD9) return fail(ACNN_JPEG_MALFORMED);   // EOI before any scan
      if (m == 0xD8 || m == 0x01 || (m >= 0xD0 && m <= 0xD7) || m == 0x00) return fail(ACNN_JPEG_LAYOUT);
      if (p + 2 > n) return fail(ACNN_JPEG_TRUNCATED);
      const int L = be16(b + p);
      if (L < 2) return fail(ACNN_JPEG_MALFORMED);
      if (p + L > n) return fail(ACNN_JPEG_TRUNCATED);
      const uint8_t* s = b + p + 2;
      const int len = L - 2;
      int r = ACNN_JPEG_OK;
      switch (m) {
        case 0xC0: case 0xC1: case 0xC2: case 0xC3: case 0xC5: case 0xC6: case 0xC7:
        case 0xC9: case 0xCA: case 0xCB: case 0xCD: case 0xCE: case 0xCF:
          r = sof(m, s, len);
          break;
        case 0xC4: r = dht(s, len); break;
        case 0xCC: r = fail(ACNN_JPEG_PROCESS); break;   // DAC: arithmetic coding
        case 0xDB: r = dqt(s, len); break;
        case 0xDD:
          if (len != 2) return fail(ACNN_JPEG_MALFORMED);
          d->restart_interval = be16(s);
          break;
        case 0xDA: return sos(s, len, p + L);
        case 0xE0:
          if (len >= 5 && !memcmp(s, "JFIF\0", 5)) jfif = true;
          break;
        case 0xEE:
          if (len >= 12 && !memcmp(s, "Adobe", 5)) {
            adobe = true;
            adobe_transform = s[11];
          }
          break;
        default:
          if (!((m >= 0xE1 && m <= 0xEF) || m == 0xFE)) return fail(ACNN_JPEG_LAYOUT);   // DNL, DHP, EXP, JPGn
      }
      if (r) return r;
      p += L;
    }
  }
};

}  // namespace
}  // namespace acnn

using namespace acnn;

extern "C" {

const char* acnn_jpeg_reason(int code) {
  switch (code) {
    case ACNN_JPEG_OK: return "supported";
    case ACNN_JPEG_NOT_JPEG: return "not a JPEG: no SOI marker";
    case ACNN_JPEG_TRUNCATED: return "the buffer ends inside the JPEG header";
    case ACNN_JPEG_MALFORMED: return "malformed JPEG header (a marker segment contradicts T.81)";
    case ACNN_JPEG_PROCESS: return "progressive, lossless, hierarchical or arithmetic-coded JPEG";
    case ACNN_JPEG_PRECISION: return "JPEG sample precision other than 8 bits";
    case ACNN_JPEG_COLOR: return "JPEG colour space other than grayscale or YCbCr";
    case ACNN_JPEG_SAMPLING: return "JPEG sampling factors other than 1x1/2x1/1x2/2x2 luma with 1x1 chroma";
    case ACNN_JPEG_LAYOUT: return "JPEG stream layout the device decoder does not handle";
    case ACNN_JPEG_SIZE: return "JPEG too large for the device decoder";
    default: return "unknown JPEG reason code";
  }
}

int acnn_jpeg_parse(const uint8_t* data, const int64_t* offsets, const int64_t* lengths, int n,
                    acnn_jpeg_desc* desc) {
  ACNN_REQUIRE(n >= 0, "acnn_jpeg_parse: n=%d < 0", n);
  if (n == 0) return ACNN_OK;
  ACNN_REQUIRE(data && offsets && lengths && desc, "acnn_jpeg_parse: null pointer");
  for (int i = 0; i < n; ++i) {
    memset(&desc[i], 0, sizeof(acnn_jpeg_desc));
    ACNN_REQUIRE(offsets[i] >= 0 && lengths[i] >= 0, "acnn_jpeg_parse: image %d: negative offset or length", i);
    Parser ps{data + offsets[i], lengths[i], &desc[i]};
    ps.run();
  }
  return ACNN_OK;
}

int acnn_jpeg_plan(const acnn_jpeg_desc* desc, const int64_t* offsets, const int32_t* windows, int n,
                   acnn_jpeg_job* jobs, acnn_jpeg_batch* batch) {
  ACNN_REQUIRE(desc && offsets && jobs && batch && n >= 1, "acnn_jpeg_plan: null pointer or n=%d < 1", n);
  auto al = [](int64_t x) { return (x + 255) & ~(int64_t)255; };
  memset(batch, 0, sizeof(*batch));
  batch->n = n;
  int64_t work = 0, out = 0, coef = 0;
  // the coefficient blocks of every image come first, in one span that one memset zeroes
  for (int i = 0; i < n; ++i) {
    const acnn_jpeg_desc& d = desc[i];
    acnn_jpeg_job& j = jobs[i];
    memset(&j, 0, sizeof(j));
    j.src = offsets[i];
    const bool whole = windows == nullptr;
    j.win_y = whole ? 0 : windows[4 * i];
    j.win_x = whole ? 0 : windows[4 * i + 1];
    j.win_h = whole ? d.height : windows[4 * i + 2];
    j.win_w = whole ? d.width : windows[4 * i + 3];
    j.active = d.supported == 1;
    if (!j.active) continue;
    ACNN_REQUIRE(j.win_y >= 0 && j.win_x >= 0 && j.win_h >= 1 && j.win_w >= 1 &&
                     (int64_t)j.win_y + j.win_h <= d.height && (int64_t)j.win_x + j.win_w <= d.width,
                 "acnn_jpeg_plan: image %d: window (%d, %d, %d, %d) outside its %dx%d pixels", i, j.win_y,
                 j.win_x, j.win_h, j.win_w, d.height, d.width);
    ACNN_REQUIRE(d.ncomp == 1 || d.ncomp == 3, "acnn_jpeg_plan: image %d: descriptor not from acnn_jpeg_parse", i);
    // MCU rows / columns holding the window's samples of every component, plus one for the upsampling
    // context of a subsampled direction
    const int mh = 8 * d.vmax, mw = 8 * d.hmax;
    const int ey = d.vmax > 1 ? 1 : 0, ex = d.hmax > 1 ? 1 : 0;
    j.mcu_r0 = std::max(0, j.win_y / mh - ey);
    j.mcu_r1 = std::min(d.mcus_y - 1, (j.win_y + j.win_h - 1) / mh + ey);
    j.mcu_c0 = std::max(0, j.win_x / mw - ex);
    j.mcu_c1 = std::min(d.mcus_x - 1, (j.win_x + j.win_w - 1) / mw + ex);
    j.stored_blocks = (j.mcu_r1 + 1) * d.mcus_x * d.bpm;
    j.idct_blocks = (j.mcu_r1 - j.mcu_r0 + 1) * (j.mcu_c1 - j.mcu_c0 + 1) * d.bpm;
    j.o_coef = coef;
    coef += al((int64_t)j.stored_blocks * 128);
  }
  batch->coef_begin = 0;
  batch->coef_end = coef;
  work = coef;
  for (int i = 0; i < n; ++i) {
    const acnn_jpeg_desc& d = desc[i];
    acnn_jpeg_job& j = jobs[i];
    if (!j.active) continue;
    j.max_sub = (int)((d.ecs_length * 8 + jpeg::kSubBits - 1) / jpeg::kSubBits) + d.n_intervals;
    j.o_bits = work;
    work += al(d.ecs_length + jpeg::kBitsPad);
    j.o_intervals = work;
    work += al(4 * ((int64_t)d.n_intervals + 2));   // interval starts (bits), the scan's end, the subsequence count
    j.o_subs = work;
    work += al(16 * (int64_t)j.max_sub);
    j.o_state = work;
    work += al(2 * 16 * (int64_t)j.max_sub);   // two generations of subsequence states
    j.o_dirty = work;
    work += al(j.max_sub);
    j.o_prefix = work;
    work += al(4 * ((int64_t)j.max_sub + 1));
    const int rows = j.mcu_r1 - j.mcu_r0 + 1, cols = j.mcu_c1 - j.mcu_c0 + 1;
    for (int c = 0; c < d.ncomp; ++c) {
      j.o_plane[c] = work;
      work += al((int64_t)rows * 8 * d.comp[c].v * cols * 8 * d.comp[c].h);
    }
    j.out = out;
    out += ((int64_t)j.win_h * j.win_w * 3 + 15) & ~(int64_t)15;
    batch->max_sub = std::max(batch->max_sub, j.max_sub);
    batch->max_idct_blocks = std::max(batch->max_idct_blocks, j.idct_blocks);
    const int64_t px = (int64_t)j.win_h * j.win_w;
    batch->max_pixels = (int)std::max<int64_t>(batch->max_pixels, px);
  }
  for (int i = 0; i < n; ++i)
    if (!jobs[i].active) jobs[i].out = out;   // unsupported images take no output bytes
  batch->work_bytes = std::max<int64_t>(work, 256);
  batch->out_bytes = std::max<int64_t>(out, 16);
  return ACNN_OK;
}

}  // extern "C"

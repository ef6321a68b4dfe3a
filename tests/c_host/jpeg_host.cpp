// The device JPEG decode of assembled_cnn_b200/csrc/jpeg_decode.cu run serially on the CPU: the same
// stage functions (csrc/jpeg_stages.cuh) in the same order -- unstuff, the two decode passes from guessed
// and from predecessor states, the synchronisation loop, the block prefix and its checks, the coefficient
// pass, the DC prefix, the IDCT and the pixel pass -- for one image and one planned window.  Built with
// g++ by tests/test_jpeg_cpu.py, which compares it with PIL.
#include <string.h>

#include <vector>

#include "../../assembled_cnn_b200/csrc/jpeg_stages.cuh"

using namespace acnn::jpeg;

namespace {
struct Sub {
  int32_t start, end, iend, first;
};
State run_sub(const acnn_jpeg_desc& d, const uint8_t* bits, const Sub& s, State in) {
  State r = decode_run<false>(d, d.dc, d.ac, bits, in, s.end, s.iend, nullptr, 0, 0);
  if (r.err) r.p = -1;
  return r;
}
State entry_of(const Sub& s, const State* prev) {
  if (s.first || prev->p < 0) return State{s.start, 0, 0, 0};
  return *prev;
}
}  // namespace

// Returns the ACNN_JPEG_ST_* status; out gets the window (win_h x win_w x 3) when it is 0.
extern "C" int jpeg_host_decode(const acnn_jpeg_desc* dp, const acnn_jpeg_job* jp, const uint8_t* img, uint8_t* out) {
  const acnn_jpeg_desc& d = *dp;
  const acnn_jpeg_job& j = *jp;
  if (!j.active) return ACNN_JPEG_ST_UNSUPPORTED;
  int status = 0;
  // unstuff
  const uint8_t* e = img + d.ecs_offset;
  const int64_t n = d.ecs_length;
  std::vector<uint8_t> bits(n + kBitsPad, 0);
  std::vector<int32_t> intervals(d.n_intervals + 1, 0);
  int64_t kept = 0;
  int r = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int c = unstuff_class(e, i, n);
    if (c == 1) bits[kept++] = e[i];
    else if (c == 2 && r + 1 < d.n_intervals) intervals[++r] = (int32_t)(kept * 8);
    else if (c == 2) ++r;
  }
  intervals[d.n_intervals] = (int32_t)(kept * 8);
  if (r != d.n_intervals - 1) status |= ACNN_JPEG_ST_MCU_COUNT;
  std::vector<Sub> subs;
  for (int k = 0; k < d.n_intervals; ++k) {
    const int a = intervals[k], b = intervals[k + 1];
    const int m = b > a ? (b - a + kSubBits - 1) / kSubBits : 1;
    for (int t = 0; t < m; ++t) {
      const int st = a + t * kSubBits;
      subs.push_back(Sub{st, st + kSubBits < b ? st + kSubBits : b, b, t == 0 ? k + 1 : 0});
    }
  }
  const int ns = (int)subs.size();
  if (ns > j.max_sub) return status | ACNN_JPEG_ST_MCU_COUNT;
  // pass 0, pass 1, synchronisation
  std::vector<State> st0(ns), st(ns);
  std::vector<uint8_t> dirty(ns + 1, 0);
  for (int t = 0; t < ns; ++t) st0[t] = run_sub(d, bits.data(), subs[t], State{subs[t].start, 0, 0, 0});
  for (int t = 0; t < ns; ++t) {
    State x = st0[t];
    if (!subs[t].first && st0[t - 1].p >= 0) x = run_sub(d, bits.data(), subs[t], st0[t - 1]);
    st[t] = x;
    if (t + 1 < ns) dirty[t + 1] = !same_entry(x, st0[t]) && !subs[t + 1].first;
  }
  for (bool any = true; any;) {
    any = false;
    for (int t = 0; t < ns; ++t) {
      if (!dirty[t]) continue;
      dirty[t] = 0;
      const State x = run_sub(d, bits.data(), subs[t], entry_of(subs[t], &st[t - 1]));
      const bool changed = !same_entry(x, st[t]);
      st[t] = x;
      if (changed && t + 1 < ns && !subs[t + 1].first) dirty[t + 1] = any = true;
    }
  }
  // prefix and checks
  std::vector<int32_t> prefix(ns);
  const int64_t per_interval = (int64_t)d.restart_interval * d.bpm;
  int64_t acc = 0;
  for (int t = 0; t < ns; ++t) {
    prefix[t] = (int32_t)acc;
    status |= st[t].err;
    if (subs[t].first && acc != (int64_t)(subs[t].first - 1) * per_interval) status |= ACNN_JPEG_ST_MCU_COUNT;
    const bool last = t + 1 == ns || subs[t + 1].first;
    if (last && (st[t].cz & 0xFFFF) != 0) status |= ACNN_JPEG_ST_MCU_COUNT;
    acc += st[t].nb;
  }
  if (acc != (int64_t)d.mcus_x * d.mcus_y * d.bpm) status |= ACNN_JPEG_ST_MCU_COUNT;
  if (status) return status;
  // coefficients
  std::vector<int16_t> coef((size_t)j.stored_blocks * 64, 0);
  for (int t = 0; t < ns; ++t) {
    if (prefix[t] >= j.stored_blocks) continue;
    decode_run<true>(d, d.dc, d.ac, bits.data(), entry_of(subs[t], t ? &st[t - 1] : nullptr), subs[t].end,
                     subs[t].iend, coef.data(), prefix[t], j.stored_blocks);
  }
  // DC prefix per component, reset at every restart interval
  for (int ci = 0; ci < d.ncomp; ++ci) {
    const int nbc = d.comp[ci].h * d.comp[ci].v;
    const int64_t T = (int64_t)(j.mcu_r1 + 1) * d.mcus_x * nbc;
    uint32_t run = 0;
    for (int64_t t = 0; t < T; ++t) {
      const int64_t m = t / nbc, u = t - m * nbc;
      const int64_t blk = m * d.bpm + d.comp[ci].blk0 + u;
      const bool first = t == 0 || (d.restart_interval > 0 && u == 0 && m % d.restart_interval == 0);
      const uint32_t v = (uint32_t)(int32_t)coef[blk * 64];
      run = first ? v : run + v;
      coef[blk * 64] = (int16_t)run;
    }
  }
  // IDCT of the window's MCU rows and columns
  const int rows = j.mcu_r1 - j.mcu_r0 + 1, cols = j.mcu_c1 - j.mcu_c0 + 1;
  std::vector<std::vector<uint8_t>> planes(d.ncomp);
  Plane pl[3];
  for (int ci = 0; ci < d.ncomp; ++ci) {
    const acnn_jpeg_comp& cp = d.comp[ci];
    const int64_t pitch = (int64_t)cols * 8 * cp.h;
    planes[ci].assign((size_t)rows * 8 * cp.v * pitch, 0);
    pl[ci] = Plane{planes[ci].data(), pitch, j.mcu_r0 * 8 * cp.v, j.mcu_c0 * 8 * cp.h, cp.dw, cp.dh};
  }
  for (int idx = 0; idx < j.idct_blocks; ++idx) {
    const int mcu = idx / d.bpm, c = idx - mcu * d.bpm;
    const int mr = j.mcu_r0 + mcu / cols, mc = j.mcu_c0 + mcu % cols;
    const int ci = block_comp(d, c);
    const acnn_jpeg_comp& cp = d.comp[ci];
    const int u = (c - cp.blk0) % cp.h, w = (c - cp.blk0) / cp.h;
    const int64_t pitch = pl[ci].pitch;
    uint8_t* o = planes[ci].data() + (int64_t)(((mr - j.mcu_r0) * cp.v + w) * 8) * pitch + ((mc - j.mcu_c0) * cp.h + u) * 8;
    idct_islow(coef.data() + ((int64_t)(mr * d.mcus_x + mc) * d.bpm + c) * 64, d.quant[cp.tq], o, pitch);
  }
  for (int y = 0; y < j.win_h; ++y)
    for (int x = 0; x < j.win_w; ++x) pixel_rgb(d, pl, j.win_y + y, j.win_x + x, out + ((int64_t)y * j.win_w + x) * 3);
  return 0;
}

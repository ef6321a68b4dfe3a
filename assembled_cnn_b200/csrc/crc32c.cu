// CRC-32C (Castagnoli) of host memory, the checksum of the TFRecord framing (acnn_crc32c, include/acnn.h).
// Host code only: the TFRecord writer checks and writes every record's checksums with it.
#include <stdint.h>
#include <string.h>

#include "common.h"

#if defined(__x86_64__)
#include <nmmintrin.h>

// SSE4.2's crc32 instruction computes the reflected CRC-32C step itself: 8 bytes per instruction after
// byte steps up to an 8-byte boundary.  The attribute enables the instruction for this function only.
__attribute__((target("sse4.2"))) static uint32_t crc32c_update(const uint8_t* p, size_t n, uint32_t c) {
  for (; n && (reinterpret_cast<uintptr_t>(p) & 7); --n) c = _mm_crc32_u8(c, *p++);
  for (; n >= 8; n -= 8, p += 8) {
    uint64_t v;
    memcpy(&v, p, 8);
    c = static_cast<uint32_t>(_mm_crc32_u64(c, v));
  }
  for (; n; --n) c = _mm_crc32_u8(c, *p++);
  return c;
}
#else
// Other hosts: one table step per byte (reflected polynomial 0x82F63B78).
struct Crc32cTable {
  uint32_t t[256];
  Crc32cTable() {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0x82F63B78u & (0u - (c & 1u)));
      t[i] = c;
    }
  }
};

static uint32_t crc32c_update(const uint8_t* p, size_t n, uint32_t c) {
  static const Crc32cTable table;   // built once, thread-safe (C++11 static initialisation)
  for (; n; --n) c = table.t[(c ^ *p++) & 0xFF] ^ (c >> 8);
  return c;
}
#endif

extern "C" uint32_t acnn_crc32c(const void* data, size_t n, uint32_t crc) {
  return ~crc32c_update(static_cast<const uint8_t*>(data), n, ~crc);
}

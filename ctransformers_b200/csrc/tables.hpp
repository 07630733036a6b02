// Host-side scalar functions behind the fp16 lookup tables (reference: ggml.c:3556-3558 gelu, 3610-3612 silu, table
// construction 4319-4333).  Written with explicit fmaf()/separate operations so the values do not depend on what the
// host compiler decides to contract: the reference BINARY fuses (GELU_COEF_A*x)*x + 1.0f into one FMA (checked in the
// disassembly of ggml_init) and nothing else in these expressions can be fused.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace ctb {

inline float host_silu(float x) { return x / (1.0f + expf(-x)); }

inline float host_gelu(float x) {
  const float t = 0.044715f * x;
  const float inner = fmaf(t, x, 1.0f);
  const float a = 0.79788456080286535587989211986876f * x;
  const float arg = a * inner;
  const float h = 0.5f * x;
  const float u = 1.0f + tanhf(arg);
  return h * u;
}

// fp16 <-> fp32 on the host through the F16C-equivalent software path (bit-identical to the device's and the reference's, NaN
// payloads included)
inline float host_h2f(uint16_t h) {
  uint32_t sign = (uint32_t)(h & 0x8000u) << 16, exp = (h >> 10) & 0x1f, man = h & 0x3ffu, bits;
  if (exp == 0) {
    if (!man) bits = sign;
    else { int e = -1; do { man <<= 1; e++; } while (!(man & 0x400u)); man &= 0x3ffu; bits = sign | ((uint32_t)(127 - 15 - e) << 23) | (man << 13); }
  } else if (exp == 31) bits = sign | 0x7f800000u | (man << 13);
  else bits = sign | ((exp + 112) << 23) | (man << 13);
  float f; memcpy(&f, &bits, 4); return f;
}
inline uint16_t host_f2h(float f) {
  uint32_t x; memcpy(&x, &f, 4);
  const uint32_t sign = (x >> 16) & 0x8000u, ax = x & 0x7fffffffu;
  if (ax >= 0x7f800000u) return (uint16_t)(sign | 0x7c00u | (ax > 0x7f800000u ? (0x200u | ((ax >> 13) & 0x3ffu)) : 0));
  if (ax >= 0x477ff000u) return (uint16_t)(sign | 0x7c00u);
  if (ax < 0x33000001u) return (uint16_t)sign;
  const int32_t e = (int32_t)(ax >> 23) - 127;
  const uint32_t m = (ax & 0x7fffffu) | 0x800000u;
  if (e < -14) {
    const uint32_t shift = (uint32_t)(13 + (-14 - e));
    uint32_t r = m >> shift; const uint32_t rem = m & ((1u << shift) - 1), half = 1u << (shift - 1);
    if (rem > half || (rem == half && (r & 1))) r++;
    return (uint16_t)(sign | r);
  }
  uint32_t hb = ((uint32_t)(e + 15) << 10) | ((m >> 13) & 0x3ffu);
  const uint32_t rem = m & 0x1fffu;
  if (rem > 0x1000u || (rem == 0x1000u && (hb & 1))) hb++;
  return (uint16_t)(sign | hb);
}

// the 65536-entry fp16 tables of SiLU, GELU and exp, indexed by the fp16 bit pattern of the input (ggml.c:4319-4333)
struct HostTables { std::vector<uint16_t> silu, gelu, ex; };
inline HostTables host_tables() {
  HostTables t{std::vector<uint16_t>(65536), std::vector<uint16_t>(65536), std::vector<uint16_t>(65536)};
  for (int i = 0; i < 65536; i++) {
    const float f = host_h2f((uint16_t)i);
    t.silu[i] = host_f2h(host_silu(f));
    t.gelu[i] = host_f2h(host_gelu(f));
    t.ex[i] = host_f2h(expf(f));
  }
  return t;
}

}  // namespace ctb

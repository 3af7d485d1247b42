#include "common/mxfp8.h"

#include <cmath>
#include <cstring>

namespace bb::mxfp8 {

float bf16_to_float(uint16_t v) noexcept {
  uint32_t u = static_cast<uint32_t>(v) << 16;
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}

uint16_t float_to_bf16(float f) noexcept {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  if ((u & 0x7FFFFFFFu) > 0x7F800000u) return static_cast<uint16_t>((u >> 16) | 0x40);  // quiet NaN
  const uint32_t lsb = (u >> 16) & 1u;
  u += 0x7FFFu + lsb;
  return static_cast<uint16_t>(u >> 16);
}

float f16_to_float(uint16_t v) noexcept {
  const uint32_t sign = static_cast<uint32_t>(v & 0x8000u) << 16;
  const uint32_t e = (v >> 10) & 0x1F, m = v & 0x3FFu;
  uint32_t u;
  if (e == 0) {  // zero or subnormal: m * 2^-24, exact in fp32
    const float f = std::ldexp(static_cast<float>(m), -24);
    std::memcpy(&u, &f, 4);
    u |= sign;
  } else if (e == 0x1F) {
    u = sign | 0x7F800000u | (m << 13);
  } else {
    u = sign | ((e + 112) << 23) | (m << 13);
  }
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}

uint16_t float_to_f16(float f) noexcept {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  const uint16_t sign = static_cast<uint16_t>((u >> 16) & 0x8000u);
  u &= 0x7FFFFFFFu;
  if (u > 0x7F800000u) return sign | 0x7E00;  // quiet NaN
  if (u >= 0x477FF000u) return sign | 0x7C00;  // >= 65520 (the tie above 65504) rounds to Inf
  if (u < 0x38800000u) {                       // below 2^-14: an fp16 subnormal, k * 2^-24 (k = 1024 is 2^-14 itself)
    float a;
    std::memcpy(&a, &u, 4);
    return sign | static_cast<uint16_t>(std::nearbyint(a * 16777216.0f));  // exact scaling, then RNE
  }
  // normal: rebias the exponent and round the 13 dropped significand bits to nearest even (a carry moves the exponent)
  return sign | static_cast<uint16_t>((u - 0x38000000u + 0xFFFu + ((u >> 13) & 1u)) >> 13);
}

uint8_t float_to_e4m3_sat(float x) noexcept {
  if (std::isnan(x)) return 0x7F;
  const uint8_t sign = std::signbit(x) ? 0x80 : 0x00;
  float a = std::fabs(x);
  if (a >= 448.0f) return sign | 0x7E;  // saturate to max finite (S.1111.110)
  if (a == 0.0f) return sign;
  int e;
  std::frexp(a, &e);  // a = m * 2^e, m in [0.5, 1)
  int exp = e - 1;    // a = (1.f) * 2^exp
  if (exp < -6) {     // subnormal range: value = k * 2^-9, k = 0..7
    const float k = a * 512.0f;
    float r = std::nearbyint(k);  // RNE under default rounding mode
    if (r >= 8.0f) return sign | 0x08;  // rounds up to the smallest normal
    return sign | static_cast<uint8_t>(r);
  }
  const float scaled = std::ldexp(a, -exp);  // in [1, 2)
  float mant = std::nearbyint((scaled - 1.0f) * 8.0f);
  if (mant >= 8.0f) {
    mant = 0.0f;
    ++exp;
  }
  if (exp > 8 || (exp == 8 && mant > 6.0f)) return sign | 0x7E;
  return sign | static_cast<uint8_t>(((exp + 7) << 3) | static_cast<int>(mant));
}

float e4m3_to_float(uint8_t v) noexcept {
  const float sign = (v & 0x80) ? -1.0f : 1.0f;
  const int e = (v >> 3) & 0xF;
  const int m = v & 7;
  if (e == 0xF && m == 7) return std::nanf("");
  if (e == 0) return sign * std::ldexp(static_cast<float>(m), -9);
  return sign * std::ldexp(1.0f + static_cast<float>(m) / 8.0f, e - 7);
}

uint8_t block_scale_e8m0(float amax) noexcept {
  if (!(amax > 0.0f) || std::isinf(amax) || std::isnan(amax)) return 127;
  uint32_t u;
  std::memcpy(&u, &amax, 4);
  int exp = static_cast<int>((u >> 23) & 0xFF) - 127;  // floor(log2(amax)) for normal floats
  if (((u >> 23) & 0xFF) == 0) exp = -127;              // subnormal amax: treat as tiny
  int e = exp - 8 + 127;
  if (e < 0) e = 0;
  if (e > 254) e = 254;
  return static_cast<uint8_t>(e);
}

float e8m0_to_float(uint8_t e) noexcept { return std::ldexp(1.0f, static_cast<int>(e) - 127); }

namespace {

float load_wide(const void* src, Wide w, size_t i) noexcept {
  switch (w) {
    case Wide::F16: return f16_to_float(static_cast<const uint16_t*>(src)[i]);
    case Wide::F32: return static_cast<const float*>(src)[i];
    default: return bf16_to_float(static_cast<const uint16_t*>(src)[i]);
  }
}

void store_wide(void* dst, Wide w, size_t i, float f) noexcept {
  switch (w) {
    case Wide::F16: static_cast<uint16_t*>(dst)[i] = float_to_f16(f); break;
    case Wide::F32: static_cast<float*>(dst)[i] = f; break;
    default: static_cast<uint16_t*>(dst)[i] = float_to_bf16(f); break;
  }
}

}  // namespace

void pack(const void* src, Wide w, size_t n, uint8_t* dst) noexcept {
  uint8_t* scales = dst + n;
  for (size_t b = 0; b < n / kBlock; ++b) {
    float amax = 0.0f;
    for (size_t i = 0; i < kBlock; ++i) {
      const float f = std::fabs(load_wide(src, w, b * kBlock + i));
      if (f > amax && !std::isnan(f)) amax = f;
    }
    const uint8_t e = block_scale_e8m0(amax);
    scales[b] = e;
    const float inv = std::ldexp(1.0f, 127 - static_cast<int>(e));
    for (size_t i = 0; i < kBlock; ++i) dst[b * kBlock + i] = float_to_e4m3_sat(load_wide(src, w, b * kBlock + i) * inv);
  }
}

void unpack(const uint8_t* packed, size_t n, Wide w, void* dst) noexcept {
  const uint8_t* scales = packed + n;
  for (size_t b = 0; b < n / kBlock; ++b) {
    const float s = e8m0_to_float(scales[b]);
    for (size_t i = 0; i < kBlock; ++i) store_wide(dst, w, b * kBlock + i, e4m3_to_float(packed[b * kBlock + i]) * s);
  }
}

void pack_bf16(const uint16_t* src, size_t n, uint8_t* dst) noexcept { pack(src, Wide::BF16, n, dst); }

void unpack_bf16(const uint8_t* packed, size_t n, uint16_t* dst) noexcept { unpack(packed, n, Wide::BF16, dst); }

}  // namespace bb::mxfp8

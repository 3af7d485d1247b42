// MXFP8 (OCP microscaling: 32-element blocks, E8M0 shared scale, E4M3 elements) — CPU reference.
// New capability required by BASELINE.json ("optional block-scaled fp8 pack/unpack"); the
// reference has no payload transforms at all (SURVEY K12).
//
// Packed object layout for n elements (n % 32 == 0):  [ n bytes E4M3 | n/32 bytes E8M0 ]
//   shared_exp(block) = floor(log2(amax(block))) - 8        (8 = emax of E4M3: 448 = 1.75 * 2^8)
//   E8M0 byte         = clamp(shared_exp + 127, 0, 254);  all-zero block -> 127 (scale 1)
//   element           = sat_e4m3( x * 2^-shared_exp ), round-to-nearest-even
// The pack never emits E8M0 0xFF (a finite bf16 block gives at most 246).  Given one, the unpacks (this one and the
// device codec, kernels/mxfp8.cuh) read it as 2^128, which overflows fp32: +-Inf, and NaN for a zero payload, not the
// OCP NaN scale.  tests/test_mxfp8_exhaustive.py checks every (payload, scale) pair against an exact model of this rule.
//
// The wide (unpacked) side is bf16, fp16 or fp32 (Wide).  The format has nothing of the wide type in it:
//   pack   applies the rule above to each element's exact fp32 value (every bf16, fp16 and fp32 is one), amax skipping
//          NaN; an fp16 subnormal amax is an fp32 normal and gets its true binade (scale bytes 95..104);
//   unpack computes e4m3(p) * 2^(s - 127) exactly in fp32 and rounds once, to nearest even, to the wide type (for fp32
//          that is no rounding, unless a scale byte of 247 or more overflows it to +-Inf).
// So a bf16-representable tensor packs to the same bytes from any wide type, and any packed object unpacks to any wide
// type: the object does not record its source type.
#pragma once
#include <cstddef>
#include <cstdint>

namespace bb::mxfp8 {

constexpr size_t kBlock = 32;
inline size_t packed_bytes(size_t n_elems) { return n_elems + n_elems / kBlock; }

// The wide (unpacked) element type of an MXFP8 transfer.
enum class Wide : uint8_t { BF16 = 0, F16 = 1, F32 = 2 };
constexpr uint32_t wide_bytes(Wide w) { return w == Wide::F32 ? 4u : 2u; }

uint8_t float_to_e4m3_sat(float x) noexcept;  // RNE, saturating to +-448, NaN -> 0x7F
float e4m3_to_float(uint8_t v) noexcept;
uint8_t block_scale_e8m0(float amax) noexcept;
float e8m0_to_float(uint8_t e) noexcept;

// src: n elements of type `w`, dst: packed_bytes(n).  n must be a multiple of 32.
void pack(const void* src, Wide w, size_t n, uint8_t* dst) noexcept;
void unpack(const uint8_t* packed, size_t n, Wide w, void* dst) noexcept;
// pack / unpack with Wide::BF16 (src / dst: raw bf16 bits).
void pack_bf16(const uint16_t* src, size_t n, uint8_t* dst) noexcept;
void unpack_bf16(const uint8_t* packed, size_t n, uint16_t* dst) noexcept;

float bf16_to_float(uint16_t v) noexcept;
uint16_t float_to_bf16(float f) noexcept;  // RNE
float f16_to_float(uint16_t v) noexcept;
uint16_t float_to_f16(float f) noexcept;   // RNE: +-Inf from 65520 on, subnormals below 2^-14

}  // namespace bb::mxfp8

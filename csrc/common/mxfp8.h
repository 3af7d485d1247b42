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
#pragma once
#include <cstddef>
#include <cstdint>

namespace bb::mxfp8 {

constexpr size_t kBlock = 32;
inline size_t packed_bytes(size_t n_elems) { return n_elems + n_elems / kBlock; }

uint8_t float_to_e4m3_sat(float x) noexcept;  // RNE, saturating to +-448, NaN -> 0x7F
float e4m3_to_float(uint8_t v) noexcept;
uint8_t block_scale_e8m0(float amax) noexcept;
float e8m0_to_float(uint8_t e) noexcept;

// src: n bf16 values (raw uint16), dst: packed_bytes(n).  n must be a multiple of 32.
void pack_bf16(const uint16_t* src, size_t n, uint8_t* dst) noexcept;
void unpack_bf16(const uint8_t* packed, size_t n, uint16_t* dst) noexcept;

float bf16_to_float(uint16_t v) noexcept;
uint16_t float_to_bf16(float f) noexcept;  // RNE

}  // namespace bb::mxfp8

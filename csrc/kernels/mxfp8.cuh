// The MXFP8 codec of the device kernels: bf16 / fp16 / fp32 <-> [E4M3 payload | E8M0 scale per 32 elements], one chunk
// of 8 elements per lane and 4 lanes per 32-element block.  Used by the stand-alone pack / unpack kernels (mxfp8.cu) and
// the fused transfer (xfer_mxfp8.cu), so both store the same bytes; the CPU reference is common/mxfp8.cpp.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <cstdint>

namespace bb::gpu {

__device__ __forceinline__ __nv_bfloat162 as_bf162(uint32_t v) { return *reinterpret_cast<const __nv_bfloat162*>(&v); }

// Packs this lane's chunk `v`.  The block max is a shuffle over the 4 lanes of the block: every lane of the warp must
// call this (a lane without data passes zeros and discards the result).  The math runs on packed bf16x2 max / paired
// E4M3 conversions, which halves the instruction count of the element-at-a-time form.
__device__ __forceinline__ void pack_chunk(const uint4 v, uint2* payload_out, uint8_t* scale_out, bool write_scale) {
  // |x| on bf16x2 = clear the sign bits; max on the magnitudes as *integers* (monotonic for non-negative bf16).
  // NaN magnitudes (> 0x7F80) are skipped, as the CPU reference skips NaN; an Inf (0x7F80) wins the max and then
  // selects the neutral scale below
  auto mag = [](uint32_t w) { return w & 0x7FFF7FFFu; };
  auto finite_max = [](uint32_t m, uint32_t cur) {
    const uint32_t lo = m & 0xFFFFu, hi = m >> 16;
    uint32_t r = cur;
    r = (lo <= 0x7F80u && lo > r) ? lo : r;
    r = (hi <= 0x7F80u && hi > r) ? hi : r;
    return r;
  };
  uint32_t am = 0;
  am = finite_max(mag(v.x), am);
  am = finite_max(mag(v.y), am);
  am = finite_max(mag(v.z), am);
  am = finite_max(mag(v.w), am);
  am = max(am, __shfl_xor_sync(0xffffffffu, am, 1));
  am = max(am, __shfl_xor_sync(0xffffffffu, am, 2));
  // am = bf16 bits of the block's largest finite magnitude; exponent field = bits 14..7
  int e = 127;
  if (am != 0 && am < 0x7F80u) {
    const int be = static_cast<int>(am >> 7);
    e = (be == 0 ? -127 : be - 127) - 8 + 127;
    e = max(0, min(254, e));
  }
  const float inv = __int_as_float((254 - e) << 23);
  auto cvt2 = [&](uint32_t w) -> uint32_t {
    const float2 f = __bfloat1622float2(as_bf162(w));
    return static_cast<uint32_t>(__nv_cvt_float2_to_fp8x2(make_float2(f.x * inv, f.y * inv), __NV_SATFINITE, __NV_E4M3));
  };
  const uint32_t lo = cvt2(v.x) | (cvt2(v.y) << 16);
  const uint32_t hi = cvt2(v.z) | (cvt2(v.w) << 16);
  *payload_out = make_uint2(lo, hi);
  if (write_scale) *scale_out = static_cast<uint8_t>(e);
}

// Unpacks one 8-byte payload chunk with its block's scale into 8 bf16.
__device__ __forceinline__ uint4 unpack_chunk(const uint2 p, uint8_t scale) {
  // 2^(e-127).  e == 0 is 2^-127, the fp32 subnormal 0x00400000: the build keeps subnormals (no -ftz, no fast math), so
  // the products below are exact and only the bf16 conversion rounds, as in the CPU reference.
  const float s = __int_as_float(scale ? static_cast<int>(scale) << 23 : 0x00400000);
  auto cvt2 = [&](uint32_t two) -> uint32_t {  // two E4M3 bytes -> bf16x2
    const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(two & 0xFFFFu), __NV_E4M3);
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hr));
    const __nv_bfloat162 h = __floats2bfloat162_rn(f.x * s, f.y * s);
    return *reinterpret_cast<const uint32_t*>(&h);
  };
  return make_uint4(cvt2(p.x), cvt2(p.x >> 16), cvt2(p.y), cvt2(p.y >> 16));
}

// ---- fp16 and fp32 wide types (mxfp8::Wide F16 / F32).  Their chunk is the same 8 elements: one uint4 of fp16, two
// uint4 of fp32.  The load side turns them into exact fp32 pairs, the core below is the rule of common/mxfp8.h on fp32
// values, and the store side rounds once from the exact fp32 product.  pack_chunk / unpack_chunk above stay the bf16
// codec, whose integer block max on raw bf16 bits cannot serve fp16: an fp16 subnormal amax is an fp32 normal, with a
// binade of its own.

__device__ __forceinline__ void load_f16_chunk(const uint4 v, float2 (&f)[4]) {
  f[0] = __half22float2(*reinterpret_cast<const __half2*>(&v.x));
  f[1] = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
  f[2] = __half22float2(*reinterpret_cast<const __half2*>(&v.z));
  f[3] = __half22float2(*reinterpret_cast<const __half2*>(&v.w));
}

__device__ __forceinline__ void load_f32_chunk(const uint4 a, const uint4 b, float2 (&f)[4]) {
  f[0] = make_float2(__uint_as_float(a.x), __uint_as_float(a.y));
  f[1] = make_float2(__uint_as_float(a.z), __uint_as_float(a.w));
  f[2] = make_float2(__uint_as_float(b.x), __uint_as_float(b.y));
  f[3] = make_float2(__uint_as_float(b.z), __uint_as_float(b.w));
}

// pack_chunk on 8 exact fp32 values, with the same lane contract.  fmaxf returns the other operand for a NaN, so the
// block max skips NaN as the CPU reference does; an Inf wins and selects the neutral scale.
__device__ __forceinline__ void pack_chunk_f32(const float2 (&f)[4], uint2* payload_out, uint8_t* scale_out, bool write_scale) {
  float am = 0.0f;
#pragma unroll
  for (int k = 0; k < 4; ++k) am = fmaxf(am, fmaxf(fabsf(f[k].x), fabsf(f[k].y)));
  am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, 1));
  am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, 2));
  const uint32_t ab = __float_as_uint(am);
  int e = 127;
  if (ab != 0 && ab < 0x7F800000u) {  // floor(log2 amax) from the fp32 exponent; an fp32 subnormal amax clamps to 0
    const int be = static_cast<int>(ab >> 23);
    e = (be == 0 ? -127 : be - 127) - 8 + 127;
    e = max(0, min(254, e));
  }
  // x * 2^(127-e) is exact whenever it is >= 2^-126, and anything smaller is +-0 in E4M3: one rounding, in the cvt
  const float inv = __int_as_float((254 - e) << 23);
  auto cvt2 = [&](float2 v) -> uint32_t {
    return static_cast<uint32_t>(__nv_cvt_float2_to_fp8x2(make_float2(v.x * inv, v.y * inv), __NV_SATFINITE, __NV_E4M3));
  };
  *payload_out = make_uint2(cvt2(f[0]) | (cvt2(f[1]) << 16), cvt2(f[2]) | (cvt2(f[3]) << 16));
  if (write_scale) *scale_out = static_cast<uint8_t>(e);
}

// The exact fp32 values e4m3(p) * 2^(scale-127) of one 8-byte payload chunk (see unpack_chunk for the scale).
__device__ __forceinline__ void unpack_chunk_f32(const uint2 p, uint8_t scale, float2 (&f)[4]) {
  const float s = __int_as_float(scale ? static_cast<int>(scale) << 23 : 0x00400000);
  auto cvt2 = [&](uint32_t two) -> float2 {
    const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(two & 0xFFFFu), __NV_E4M3);
    const float2 v = __half22float2(*reinterpret_cast<const __half2*>(&hr));
    return make_float2(v.x * s, v.y * s);
  };
  f[0] = cvt2(p.x);
  f[1] = cvt2(p.x >> 16);
  f[2] = cvt2(p.y);
  f[3] = cvt2(p.y >> 16);
}

// 8 fp16, each rounded once (RNE) from the exact product: +-Inf from 65520 on, fp16 subnormals below 2^-14.
__device__ __forceinline__ uint4 store_f16_chunk(const float2 (&f)[4]) {
  uint32_t w[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const __half2 h = __float22half2_rn(f[k]);
    w[k] = *reinterpret_cast<const uint32_t*>(&h);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

__device__ __forceinline__ void store_f32_chunk(const float2 (&f)[4], uint4* a, uint4* b) {
  *a = make_uint4(__float_as_uint(f[0].x), __float_as_uint(f[0].y), __float_as_uint(f[1].x), __float_as_uint(f[1].y));
  *b = make_uint4(__float_as_uint(f[2].x), __float_as_uint(f[2].y), __float_as_uint(f[3].x), __float_as_uint(f[3].y));
}

// Packs chunk c (8 elements) of a wide array of 16-byte words `in` (WB = wide bytes per element): bf16 (f16 false) or
// fp16 (f16 true) when WB == 2, fp32 when WB == 4.  `f16` must be warp-uniform.
template <uint32_t WB>
__device__ __forceinline__ void pack_wide_chunk(const uint4* in, uint32_t c, bool f16, uint2* payload_out, uint8_t* scale_out, bool write_scale) {
  if constexpr (WB == 4) {
    float2 f[4];
    load_f32_chunk(in[2 * c], in[2 * c + 1], f);
    pack_chunk_f32(f, payload_out, scale_out, write_scale);
  } else {
    if (f16) {
      float2 f[4];
      load_f16_chunk(in[c], f);
      pack_chunk_f32(f, payload_out, scale_out, write_scale);
    } else {
      pack_chunk(in[c], payload_out, scale_out, write_scale);
    }
  }
}

// Unpacks one payload chunk into chunk c of a wide array of 16-byte words `out`, as pack_wide_chunk.
template <uint32_t WB>
__device__ __forceinline__ void unpack_wide_chunk(const uint2 p, uint8_t scale, bool f16, uint4* out, uint32_t c) {
  if constexpr (WB == 4) {
    float2 f[4];
    unpack_chunk_f32(p, scale, f);
    store_f32_chunk(f, &out[2 * c], &out[2 * c + 1]);
  } else {
    if (f16) {
      float2 f[4];
      unpack_chunk_f32(p, scale, f);
      out[c] = store_f16_chunk(f);
    } else {
      out[c] = unpack_chunk(p, scale);
    }
  }
}

}  // namespace bb::gpu

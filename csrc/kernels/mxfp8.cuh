// The MXFP8 codec of the device kernels: bf16 <-> [E4M3 payload | E8M0 scale per 32 elements], one 16-byte chunk of
// 8 bf16 per lane and 4 lanes per 32-element block.  Used by the stand-alone pack / unpack kernels (mxfp8.cu) and the
// fused transfer (xfer_mxfp8.cu), so both store the same bytes; the CPU reference is common/mxfp8.cpp.
#pragma once
#include <cuda_bf16.h>
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

}  // namespace bb::gpu

// split16.cuh -- fp32 -> 16-bit hi / lo split of the 16-bit split-operand core (gemm_umma16.cuh), and the [hi | lo]
// operand planes that epilogues write beside an fp32 activation so that the next GEMM's producers copy its operand tiles
// instead of gathering and converting fp32.
//
//     x = hi + lo + e,   hi = rn16(x),  lo = rn16(x - hi)          (x - hi is exact in fp32)
#pragma once
#include "common.cuh"

namespace drl {
namespace umma16 {

struct BF16 {
  static constexpr uint32_t kFormat = 1;
  static constexpr bool kBf16 = true;
  __device__ static __forceinline__ uint32_t pack2(float lo_elem, float hi_elem) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));   // d = {a (upper), b (lower)}
    return r;
  }
  __device__ static __forceinline__ float2 unpack2(uint32_t p) {
    return make_float2(__uint_as_float(p << 16), __uint_as_float(p & 0xffff0000u));
  }
};
struct F16 {
  static constexpr uint32_t kFormat = 0;
  static constexpr bool kBf16 = false;
  __device__ static __forceinline__ uint32_t pack2(float lo_elem, float hi_elem) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
    return r;
  }
  __device__ static __forceinline__ float2 unpack2(uint32_t p) {
    float2 f;
    asm("{\n\t.reg .b16 l, h;\n\tmov.b32 {l, h}, %2;\n\tcvt.f32.f16 %0, l;\n\tcvt.f32.f16 %1, h;\n\t}"
        : "=f"(f.x), "=f"(f.y) : "r"(p));
    return f;
  }
};

// two consecutive fp32 values -> their hi pair and lo pair (element 0 in the low half of each word, memory order)
template <class F>
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& h, uint32_t& l) {
  h = F::pack2(x0, x1);
  const float2 hf = F::unpack2(h);
  l = F::pack2(x0 - hf.x, x1 - hf.y);
}
// 8 consecutive fp32 values -> 8 hi halves + 8 lo halves (element i in the low/high half of word i/2, memory order)
template <class F>
__device__ __forceinline__ void split8(const float4& a, const float4& b, uint4& hi, uint4& lo) {
  split2<F>(a.x, a.y, hi.x, lo.x);
  split2<F>(a.z, a.w, hi.y, lo.y);
  split2<F>(b.x, b.y, hi.z, lo.z);
  split2<F>(b.z, b.w, hi.w, lo.w);
}

}  // namespace umma16

// A bf16 [hi | lo] operand plane beside an fp32 buffer of `count` elements: element i's hi half at p[i], its lo half at
// p[count + i], split by umma16::split8<BF16> element by element -- the bits the producers of gemm_umma16.cuh would have
// made from the fp32 value.  An epilogue that writes the fp32 value writes the plane from the same register (p == nullptr:
// no plane).  In the plane, 8 consecutive elements of the fp32 buffer are one 16-byte chunk of a SWIZZLE_128B tile.
struct Plane16 {
  uint16_t* p = nullptr;
  size_t count = 0;
  // elements [i, i + 4), i a multiple of 4
  __device__ __forceinline__ void store4(size_t i, float x0, float x1, float x2, float x3) const {
    if (p == nullptr) return;
    uint2 h, l;
    umma16::split2<umma16::BF16>(x0, x1, h.x, l.x);
    umma16::split2<umma16::BF16>(x2, x3, h.y, l.y);
    *reinterpret_cast<uint2*>(p + i) = h;
    *reinterpret_cast<uint2*>(p + count + i) = l;
  }
  __device__ __forceinline__ void store1(size_t i, float x) const {
    if (p == nullptr) return;
    uint32_t h, l;
    umma16::split2<umma16::BF16>(x, 0.f, h, l);
    p[i] = (uint16_t)(h & 0xffffu);
    p[count + i] = (uint16_t)(l & 0xffffu);
  }
};

}  // namespace drl

// act_quant.cuh -- the reference's activation quantisers, written once for every kernel that quantises fp32 activations
// (act_quant_kernel / act_quant_plain_kernel in act_prep.cu, quantise_to_smem in gemv_ring_impl.cuh, act_quant_imma_kernel in
// gemm_imma.cu), and the layout facts of the int8 activation image they write:
//   NS_COMP_Q8_0    : quantize_row_q8_0 (neural_speed/vectors/cpu/quantize.h:447-560, x86 body: id = 127/amax, round-half-even)
//   NS_COMP_INT8    : quantize_fp_u8_colblock (bestla/bestla/kernel_ref.h:1825-1883): u8 codes with a zero point
//   NS_COMP_INT8_S8 : quantize_fp_s8_colblock (bestla/bestla/kernel_ref.h:1886-1928): s8 codes
// A kernel starts a block's range with range_start, folds its values in with range_fold, reduces the range over the lanes
// that share the block with range_reduce, and quantises with block_quant + quant_code.  Loads, the code sums and the stores
// stay in each kernel: their images differ.
#pragma once
#include "nsb.cuh"

namespace nsq {

// utils::cast<float,uint8_t> (bestla_utils.h:515-521)
__device__ __forceinline__ int cast_u8(float x) {
  if (x != x) return 0;  // NaN -> 0 as on x86 (see cast_s8)
  x += 0.5f;
  x = fminf(x, 255.f);
  x = fmaxf(x, 0.f);
  return (int)x;
}
// utils::cast<float,int8_t> (bestla_utils.h:507-513)
__device__ __forceinline__ int cast_s8(float x) {
  // all-zero block: scale is denormal, 1/scale = inf, 0*inf = NaN.  On the reference's x86 build the NaN survives
  // std::min/std::max and converts to 0 (cvttss2si -> INT_MIN -> int8 0); CUDA's fminf would return 127 instead.
  if (x != x) return 0;
  x = roundf(x);
  x = fminf(x, 127.f);
  x = fmaxf(x, -128.f);
  return (int)x;
}

// Start of a block's range (vmax; vmin always starts at 0).  quantize_row_q8_0 takes amax from 0.  The BesTLA quantisers start
// maxval / absmaxval at FLT_MIN (kernel_ref.h:1832, :1892, :1910), except quantize_fp_u8_colblock's partial last block, which
// starts at 0 (:1857-1858).  partial: the block ends past K.
template <int COMP>
__device__ __forceinline__ float range_start(bool partial) {
  if (COMP == NS_COMP_Q8_0 || (COMP == NS_COMP_INT8 && partial)) return 0.f;
  return 1.17549435e-38f;
}
// INT8 keeps the signed range (kernel_ref.h:1836-1837), Q8_0 and INT8_S8 the largest magnitude (kernel_ref.h:1895)
template <int COMP>
__device__ __forceinline__ void range_fold(float v, float& vmax, float& vmin) {
  if (COMP == NS_COMP_INT8) {
    vmax = fmaxf(v, vmax);
    vmin = fminf(v, vmin);
  } else {
    vmax = fmaxf(vmax, fabsf(v));
  }
}
// the range of a block held by `width` consecutive lanes (a power of two <= 32; every lane of the warp takes part)
template <int COMP>
__device__ __forceinline__ void range_reduce(float& vmax, float& vmin, int width) {
  for (int o = 1; o < width; o <<= 1) {
    vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    if (COMP == NS_COMP_INT8) vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, o));
  }
}

struct BlockQuant {
  float scale;   // the block's dequantisation scale, as the reference stores it
  float rscale;  // multiplier from values to codes
  int za;        // zero point (INT8), else 0
};
template <int COMP>
__device__ __forceinline__ BlockQuant block_quant(float vmax, float vmin) {
  BlockQuant b;
  b.za = 0;
  if (COMP == NS_COMP_Q8_0) {
    // d = amax/127 rounded to fp16 (block_q8_0.d); the multiplier is 127/amax (x86 body of quantize_row_q8_0)
    b.scale = __half2float(__float2half_rn(vmax / 127.f));
    b.rscale = vmax != 0.f ? 127.f / vmax : 0.f;
  } else if (COMP == NS_COMP_INT8) {
    b.scale = (vmax - vmin) / 255;  // kernel_ref.h:1839-1841
    b.za = cast_u8((0 - vmin) / b.scale);
    b.rscale = 1.f / b.scale;
  } else {
    b.scale = vmax / 127;  // kernel_ref.h:1897-1898
    b.rscale = 1.f / b.scale;
  }
  return b;
}
// the code of one value of the block; padding past K takes b.za instead, so that it contributes (a - za) == 0
template <int COMP>
__device__ __forceinline__ int quant_code(float v, const BlockQuant& b) {
  if (COMP == NS_COMP_Q8_0) return __float2int_rn(v * b.rscale);  // round-half-even like _mm256_round_ps(NEAREST)
  if (COMP == NS_COMP_INT8) return cast_u8((float)b.za + (float)(int)roundf(v * b.rscale));  // kernel_ref.h:1848-1850
  return cast_s8(v * b.rscale);                                                             // kernel_ref.h:1903
}

// ---- layout of the int8 activation image (nsb.cuh) --------------------------------------------------------------------
// Byte position of element e (0..7) inside its 8-group: the two words of a group hold (e0,e4,e1,e5) / (e2,e6,e3,e7), the
// order of the NSB4 nibbles, so that dp4a and the IMMA fragments pair each activation with its weight.  S8 weights keep
// natural order.
__device__ __forceinline__ int dp4a_pos(int e) { return ((e & 3) << 1) | (e >> 2); }
// Ring image (gemv_ring.cu): per super-block of 32 chunks, the first 16 bytes of every chunk, then the second 16 bytes, so
// that a warp reading 16 bytes of 32 consecutive chunks hits no bank twice.  Byte `byte` (0..31) of chunk c.
__device__ __forceinline__ uint32_t ring_offset(uint32_t c, uint32_t byte) {
  return (c >> 5) * 1024u + (byte >> 4) * 512u + (c & 31) * 16u + (byte & 15);
}
// meta word of a chunk: {a_scale bits, (Sa & 0xffff) | za << 16}, Sa the sum of the codes (per chunk, or per block for IMMA)
__device__ __forceinline__ int2 meta_word(float scale, int sa, int za) {
  return make_int2(__float_as_int(scale), (sa & 0xffff) | (za << 16));
}

}  // namespace nsq

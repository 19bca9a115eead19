// kv_cache.cuh -- the element formats of the KV cache, written once for the kernels that store or read it (attention.cu's RoPE
// append, decode and prompt attention, beam.cu's block copy) and for the allocation in llama.cu.
//
//   NS_KV_F16   one plane per cache: [unit][n_ctx][hd] fp16
//   NS_KV_Q8_0  two planes per cache: q [unit][n_ctx][hd] int8 codes and d [unit][kv_d_stride(n_ctx, hd)] fp16 scales, row p of
//               a unit's d at p * hd / 32.  Each row is cut into blocks of 32 and every block quantised by the activation quantiser
//               of act_quant.cuh (NS_COMP_Q8_0: d = fp16(amax / 127), codes round-half-even of x * 127 / amax).
// A unit is one (layer, block, kv head): the rows of a head are contiguous, so a range of positions is one copy per plane.  The
// d stride pads a unit to 16 bytes and kv_q8_d_bytes rounds a range's scale bytes up to 16, as bulk copies want; the rounded
// range never leaves its unit.
// A kernel reads a Q8_0 value as fp16(q * float(d)) (the product is exact in fp32: one rounding), so a Q8_0 cache C behaves
// exactly like an fp16 cache holding those values.
#pragma once
#include <cuda_fp16.h>

#include <cstdint>
#include <type_traits>

#include "act_quant.cuh"

constexpr int kKvQ8Block = 32;

// element of the value plane: the fp16 cache itself, or the Q8_0 codes
template <int KV>
using kv_elem_t = std::conditional_t<KV == NS_KV_Q8_0, int8_t, __half>;

// halves of one unit of a d plane
__host__ __device__ __forceinline__ size_t kv_d_stride(int n_ctx, int hd) { return ((size_t)n_ctx * (hd / kKvQ8Block) + 7) / 8 * 8; }
// bytes of `rows` rows of a d plane, rounded up to the 16 bytes of a bulk copy
__host__ __device__ __forceinline__ uint32_t kv_q8_d_bytes(int rows, int hd) { return ((uint32_t)rows * (hd / kKvQ8Block) * 2 + 15) / 16 * 16; }

// bytes of one cache (K or V) of `units` units: every plane of it
inline size_t kv_cache_bytes(int kv, size_t units, int n_ctx, int hd) {
  if (kv == NS_KV_Q8_0) return units * ((size_t)n_ctx * hd + kv_d_stride(n_ctx, hd) * 2);
  return units * (size_t)n_ctx * hd * 2;
}

// The caches of one layer as the launchers take them: k / v the value planes (fp16 or Q8_0 codes) from a unit on, kd / vd the
// Q8_0 scale planes from the same unit (null for fp16)
struct KvPtrs {
  int type = NS_KV_F16;
  void* k = nullptr;
  void* v = nullptr;
  __half* kd = nullptr;
  __half* vd = nullptr;
  // the same caches `units` units further on
  KvPtrs at(size_t units, int n_ctx, int hd) const {
    KvPtrs p = *this;
    if (type == NS_KV_Q8_0) {
      p.k = static_cast<int8_t*>(k) + units * n_ctx * hd;
      p.v = static_cast<int8_t*>(v) + units * n_ctx * hd;
      p.kd = kd + units * kv_d_stride(n_ctx, hd);
      p.vd = vd + units * kv_d_stride(n_ctx, hd);
    } else {
      p.k = static_cast<__half*>(k) + units * n_ctx * hd;
      p.v = static_cast<__half*>(v) + units * n_ctx * hd;
    }
    return p;
  }
};

// ---- store: one 32-block held as pairs (x0, x1) by 16 consecutive lanes ----------------------------------------------------
// Every lane of the warp takes part (the block's amax is a shuffle reduction over the 16 lanes).
struct KvQ8Pair {
  int q0, q1;
  float d;  // the block's scale, an fp16 value
};
__device__ __forceinline__ KvQ8Pair kv_q8_quant_pair(float x0, float x1) {
  float vmax = nsq::range_start<NS_COMP_Q8_0>(false), vmin = 0.f;
  nsq::range_fold<NS_COMP_Q8_0>(x0, vmax, vmin);
  nsq::range_fold<NS_COMP_Q8_0>(x1, vmax, vmin);
  nsq::range_reduce<NS_COMP_Q8_0>(vmax, vmin, kKvQ8Block / 2);
  const nsq::BlockQuant b = nsq::block_quant<NS_COMP_Q8_0>(vmax, vmin);
  return KvQ8Pair{nsq::quant_code<NS_COMP_Q8_0>(x0, b), nsq::quant_code<NS_COMP_Q8_0>(x1, b), b.scale};
}
// the value a kernel reads back: fp16(q * d)
__device__ __forceinline__ float kv_q8_value(int q, float d) { return __half2float(__float2half_rn((float)q * d)); }
// pair i of a row: q_row / d_row the row's codes and scales
__device__ __forceinline__ void kv_q8_store_pair(int8_t* q_row, __half* d_row, int i, const KvQ8Pair& a) {
  *reinterpret_cast<char2*>(q_row + 2 * i) = make_char2((signed char)a.q0, (signed char)a.q1);
  if (i % (kKvQ8Block / 2) == 0) d_row[i / (kKvQ8Block / 2)] = __float2half_rn(a.d);
}

// ---- load -------------------------------------------------------------------------------------------------------------------
// N (2, 4 or 8) consecutive values of one block, from codes q (N-byte aligned) and the block's scale d
template <int N>
__device__ __forceinline__ void kv_q8_load(const int8_t* q, __half d, float* dst) {
  const float df = __half2float(d);
  if constexpr (N == 8) {
    const int2 u = *reinterpret_cast<const int2*>(q);
    const char4 a = *reinterpret_cast<const char4*>(&u.x), b = *reinterpret_cast<const char4*>(&u.y);
    dst[0] = kv_q8_value(a.x, df), dst[1] = kv_q8_value(a.y, df), dst[2] = kv_q8_value(a.z, df), dst[3] = kv_q8_value(a.w, df);
    dst[4] = kv_q8_value(b.x, df), dst[5] = kv_q8_value(b.y, df), dst[6] = kv_q8_value(b.z, df), dst[7] = kv_q8_value(b.w, df);
  } else if constexpr (N == 4) {
    const char4 a = *reinterpret_cast<const char4*>(q);
    dst[0] = kv_q8_value(a.x, df), dst[1] = kv_q8_value(a.y, df), dst[2] = kv_q8_value(a.z, df), dst[3] = kv_q8_value(a.w, df);
  } else {
    static_assert(N == 2, "2, 4 or 8 values");
    const char2 a = *reinterpret_cast<const char2*>(q);
    dst[0] = kv_q8_value(a.x, df), dst[1] = kv_q8_value(a.y, df);
  }
}
// 8 consecutive values as fp16, packed as 16 bytes (one row chunk of a padded shared-memory tile)
__device__ __forceinline__ uint4 kv_q8_load8_h(const int8_t* q, __half d) {
  float f[8];
  kv_q8_load<8>(q, d, f);
  uint4 r;
  __half2 h[4] = {__floats2half2_rn(f[0], f[1]), __floats2half2_rn(f[2], f[3]), __floats2half2_rn(f[4], f[5]), __floats2half2_rn(f[6], f[7])};
  r.x = *reinterpret_cast<uint32_t*>(&h[0]);
  r.y = *reinterpret_cast<uint32_t*>(&h[1]);
  r.z = *reinterpret_cast<uint32_t*>(&h[2]);
  r.w = *reinterpret_cast<uint32_t*>(&h[3]);
  return r;
}

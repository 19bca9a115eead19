// repack.cu -- load-time conversion of the reference's weight formats into the device ("NSB") layout, on the GPU.
//
// Counterpart of bestla_device_load_storage / convertTransStorage in the reference's SYCL backend
// (neural_speed/core/layers/ne_bestla_sycl.cpp:94-150, bestla/bestla/bestla_prologue_b.h:129-150): the host blob is
// uploaded verbatim and one kernel rewrites it N-major with K-contiguous nibbles and transposed scales.
// Sources handled:
//   * ggml rows of block_q4_0 (core/data_types.h:79-83: fp16 d + 16 bytes; byte j = elem j | elem j+16 << 4)
//   * ggml rows of block_q8_0 (core/data_types.h:107-111: fp16 d + 32 int8 codes, element j in byte j)
//   * canonical container  q int8 [K][N], scales f32 [K/g][N], zp int8 [K/g][N]   (what BTLAGemmPackB takes)
//   * serialized BesTLA blob: QBuf nibbles in [N/NTile][KPad/PackRow][NTile][PackRow] order
//     (bestla_prologue_b.h:490-510 reorderWeight + kernel_ref.h:40-58 padding_interleave + :155 compress_s8_s4),
//     scales/zp [KPad/g][NPad] (bestla_storage.h:151-248)
// plus the inverse (dequantise to fp32) and the device Q4_0 quantiser (vectors/cpu/quantize.h:243-279).
#include "nsb.cuh"

namespace {

// nibble position p of a 32-bit word holds element nsb4_perm(p) = {0,2,4,6,1,3,5,7}
__host__ __device__ constexpr int nsb4_perm(int p) { return p < 4 ? 2 * p : 2 * (p - 4) + 1; }

// ---- ggml Q4_0 rows -> NSB -------------------------------------------------------------------------------------------
__global__ void repack_q4_0_kernel(const uint8_t* __restrict__ rows, size_t nb01, int n, int nblocks,
                                   uint8_t* __restrict__ q, size_t row_bytes, int sc_off) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * nblocks) return;
  const int row = (int)(idx / nblocks), b = (int)(idx - (size_t)row * nblocks);
  const unsigned short* src = reinterpret_cast<const unsigned short*>(rows + (size_t)row * nb01 + (size_t)b * 18);
  unsigned short h[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) h[i] = src[i];
  uint8_t e[32];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const unsigned byte = (h[1 + (j >> 1)] >> ((j & 1) * 8)) & 0xff;
    e[j] = byte & 0xf;
    e[j + 16] = byte >> 4;
  }
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t v = 0;
#pragma unroll
    for (int p = 0; p < 8; ++p) v |= (uint32_t)e[8 * i + nsb4_perm(p)] << (4 * p);
    w[i] = v;
  }
  *reinterpret_cast<uint4*>(q + (size_t)row * row_bytes + (size_t)b * 16) = make_uint4(w[0], w[1], w[2], w[3]);
  *reinterpret_cast<unsigned short*>(q + (size_t)row * row_bytes + sc_off + (size_t)b * 2) = h[0];
}

// ---- ggml Q8_0 rows -> NSB: one thread per block; the 32 codes keep their order, d goes to the scale array ------------
__global__ void repack_q8_0_kernel(const uint8_t* __restrict__ rows, size_t nb01, int n, int nblocks,
                                   uint8_t* __restrict__ q, size_t row_bytes, int sc_off) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * nblocks) return;
  const int row = (int)(idx / nblocks), b = (int)(idx - (size_t)row * nblocks);
  const unsigned short* src = reinterpret_cast<const unsigned short*>(rows + (size_t)row * nb01 + (size_t)b * 34);
  uint32_t w[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) w[i] = (uint32_t)src[1 + 2 * i] | ((uint32_t)src[2 + 2 * i] << 16);
  uint4* dst = reinterpret_cast<uint4*>(q + (size_t)row * row_bytes + (size_t)b * 32);
  dst[0] = make_uint4(w[0], w[1], w[2], w[3]);
  dst[1] = make_uint4(w[4], w[5], w[6], w[7]);
  *reinterpret_cast<unsigned short*>(q + (size_t)row * row_bytes + sc_off + (size_t)b * 2) = src[0];
}

// ---- generic element accessors ---------------------------------------------------------------------------------------
struct SrcCanonical {  // q int8 [K][N] holding VALUES (nibble-8 for s4, code for nf4, value for s8)
  const int8_t* q;
  int n;
  __device__ int get(int k, int nn) const { return q[(size_t)k * n + nn]; }
};
struct SrcBtlaS4 {  // packed nibbles, [N/NTile][KPad/PackRow][NTile][PackRow]; nibble u = value + 8 (ints) or code (f4)
  const uint8_t* q;
  int kpad_src, ntile, packrow;
  int is_float;
  __device__ int get(int k, int nn) const {
    const size_t e = (size_t)(nn / ntile) * kpad_src * ntile + (size_t)(k / packrow) * packrow * ntile +
                     (size_t)(nn % ntile) * packrow + (k % packrow);
    const int byte = q[e >> 1];
    const int u = (e & 1) ? (byte >> 4) : (byte & 0xf);
    return is_float ? u : u - 8;
  }
};
struct SrcBtlaS8 {
  const int8_t* q;
  int kpad_src, ntile, packrow;
  __device__ int get(int k, int nn) const {
    const size_t e = (size_t)(nn / ntile) * kpad_src * ntile + (size_t)(k / packrow) * packrow * ntile +
                     (size_t)(nn % ntile) * packrow + (k % packrow);
    return q[e];
  }
};

// one thread per (n, 8-group of k); n fastest for coalesced canonical reads
template <typename Src>
__global__ void repack_q_kernel(Src src, int n, int k, int kpad, int wfmt, uint8_t* __restrict__ q, size_t row_bytes) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int ngrp = kpad >> 3;
  if (idx >= (size_t)n * ngrp) return;
  const int nn = (int)(idx % n), g = (int)(idx / n);
  const int k0 = g * 8;
  if (wfmt == NS_W_S8) {
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int v0 = (k0 + e < k) ? src.get(k0 + e, nn) : 0;
      const int v1 = (k0 + 4 + e < k) ? src.get(k0 + 4 + e, nn) : 0;
      lo |= (uint32_t)(v0 & 0xff) << (8 * e);
      hi |= (uint32_t)(v1 & 0xff) << (8 * e);
    }
    *reinterpret_cast<uint2*>(q + (size_t)nn * row_bytes + k0) = make_uint2(lo, hi);
  } else {
    uint32_t v = 0;
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      const int kk = k0 + nsb4_perm(p);
      int u;
      if (kk < k) {
        const int val = src.get(kk, nn);
        u = (wfmt == NS_W_NF4) ? (val & 0xf) : ((val + 8) & 0xf);
      } else {
        u = (wfmt == NS_W_NF4) ? 0 : 8;  // zero-valued padding
      }
      v |= (uint32_t)u << (4 * p);
    }
    *reinterpret_cast<uint32_t*>(q + (size_t)nn * row_bytes + (size_t)g * 4) = v;
  }
}

// scales/zp: src [ngroups][ld_src] (f32 | bf16 | f16 by src_stype) -> into each NSB row at sc_off / zp_off
__global__ void repack_scales_kernel(const void* __restrict__ sc, int src_stype, const int8_t* __restrict__ zp,
                                     int ld_src, int n, int ngroups, uint8_t* __restrict__ rows, size_t pitch, int sc_off,
                                     int zp_off, int dst_stype, int has_zp) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * ngroups) return;
  const int nn = (int)(idx % n), g = (int)(idx / n);
  const size_t si = (size_t)g * ld_src + nn;
  uint8_t* row = rows + (size_t)nn * pitch;
  float v;
  if (src_stype == NS_S_F32) v = reinterpret_cast<const float*>(sc)[si];
  else if (src_stype == NS_S_F16) v = __half2float(__ushort_as_half(reinterpret_cast<const unsigned short*>(sc)[si]));
  else v = __uint_as_float((uint32_t) reinterpret_cast<const unsigned short*>(sc)[si] << 16);
  if (dst_stype == NS_S_F32) {
    reinterpret_cast<float*>(row + sc_off)[g] = v;
  } else if (src_stype == dst_stype) {
    reinterpret_cast<unsigned short*>(row + sc_off)[g] = reinterpret_cast<const unsigned short*>(sc)[si];  // bit copy
  } else if (dst_stype == NS_S_F16) {
    reinterpret_cast<__half*>(row + sc_off)[g] = __float2half_rn(v);
  } else {
    reinterpret_cast<__nv_bfloat16*>(row + sc_off)[g] = __float2bfloat16_rn(v);  // RNE, as bestla_utils.h:146-153
  }
  if (has_zp) row[zp_off + g] = zp ? (uint8_t)zp[si] : 0;
}

// ---- NSB -> fp32 [n][ld] ---------------------------------------------------------------------------------------------
__global__ void dequant_kernel(const uint8_t* __restrict__ rows, size_t pitch, int sc_off, int zp_off, int stype, int asym,
                               int n, int k, int group, int wfmt, int f4kind, float* __restrict__ dst, int ld) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * k) return;
  const int row = (int)(idx / k), kk = (int)(idx - (size_t)row * k);
  const uint8_t* r = rows + (size_t)row * pitch;
  const int gi = kk / group;
  const float s = ns_scale_at(r + sc_off, stype, gi);
  const int z = asym ? (int)(signed char)r[zp_off + gi] : 0;
  float v;
  if (wfmt == NS_W_S8 || wfmt == NS_W_Q8_0) {  // Q8_0: fp32(d) * q, dequantize_row_q8_0 (quantize.h:780)
    v = (float)((int)(signed char)r[kk] - z) * s;
  } else {
    const uint32_t w = *reinterpret_cast<const uint32_t*>(r + (size_t)(kk >> 3) * 4);
    const int e = kk & 7;
    const int sh = ((e >> 1) << 2) + ((e & 1) << 4);
    const int u = (w >> sh) & 0xf;
    v = (wfmt == NS_W_NF4) ? NS_F4_LUT[f4kind][u] * s : (float)(u - 8 - z) * s;
  }
  dst[(size_t)row * ld + kk] = v;
}

// ---- device Q4_0 quantiser: one thread per block of 32 ----------------------------------------------------------------
// quantize_row_q4_0_reference (quantize.h:243-279).  x*id + 8.5f is evaluated as ONE fma: the reference's default
// x86 build (-O3 -mfma, fp-contract=fast) contracts it, and oracle/_ref pins that form (tests/test_oracle_vs_ref.py).
__global__ void quantize_q4_0_kernel(const float* __restrict__ src, int n, int k, uint8_t* __restrict__ dst) {
  const int nblocks = k >> 5;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * nblocks) return;
  const float* x = src + idx * 32;
  float v[32];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 t = reinterpret_cast<const float4*>(x)[j];
    v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
  }
  float amax = 0.f, vmax = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j)
    if (fabsf(v[j]) > amax) { amax = fabsf(v[j]); vmax = v[j]; }
  const float d = __fdiv_rn(vmax, -8.f);
  const float id = d != 0.f ? __fdiv_rn(1.0f, d) : 0.0f;
  unsigned short out[9];
  out[0] = __half_as_ushort(__float2half_rn(d));
#pragma unroll
  for (int j = 0; j < 16; j += 2) {
    unsigned b[2];
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      int lo = (int)(signed char)(int)__fmaf_rn(v[j + t], id, 8.5f);       // truncation toward zero
      int hi = (int)(signed char)(int)__fmaf_rn(v[j + t + 16], id, 8.5f);
      lo = min(lo, 15);
      hi = min(hi, 15);
      b[t] = (unsigned)(lo | (hi << 4)) & 0xff;
    }
    out[1 + (j >> 1)] = (unsigned short)(b[0] | (b[1] << 8));
  }
  unsigned short* o = reinterpret_cast<unsigned short*>(dst + idx * 18);
#pragma unroll
  for (int i = 0; i < 9; ++i) o[i] = out[i];
}

}  // namespace

int ns_launch_repack_q4_0(const void* rows_dev, size_t nb01, ns_weight* w, cudaStream_t st) {
  const int nblocks = w->k / 32;
  const size_t total = (size_t)w->n * nblocks;
  repack_q4_0_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const uint8_t*)rows_dev, nb01, w->n, nblocks,
                                                                      w->rows, (size_t)w->pitch, w->sc_off);
  NS_CUDA_TRY(cudaGetLastError());
  ns_count_launch();
  return NS_OK;
}

int ns_launch_repack_q8_0(const void* rows_dev, size_t nb01, ns_weight* w, cudaStream_t st) {
  const int nblocks = w->k / 32;
  const size_t total = (size_t)w->n * nblocks;
  repack_q8_0_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const uint8_t*)rows_dev, nb01, w->n, nblocks,
                                                                      w->rows, (size_t)w->pitch, w->sc_off);
  NS_CUDA_TRY(cudaGetLastError());
  ns_count_launch();
  return NS_OK;
}

static int launch_scales(const void* sc, int src_stype, const int8_t* zp, int ld_src, ns_weight* w, cudaStream_t st) {
  const size_t total = (size_t)w->n * w->ngroups;
  repack_scales_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(sc, src_stype, zp, ld_src, w->n, w->ngroups,
                                                                        w->rows, (size_t)w->pitch, w->sc_off, w->zp_off,
                                                                        w->stype, w->asym);
  NS_CUDA_TRY(cudaGetLastError());
  ns_count_launch();
  return NS_OK;
}

int ns_launch_repack_canonical(const int8_t* q_kn_dev, const float* sc_dev, const int8_t* zp_dev, ns_weight* w,
                               cudaStream_t st) {
  const size_t total = (size_t)w->n * (w->kpad >> 3);
  SrcCanonical src{q_kn_dev, w->n};
  repack_q_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(src, w->n, w->k, w->kpad, w->wfmt, w->rows, (size_t)w->pitch);
  NS_CUDA_TRY(cudaGetLastError());
  ns_count_launch();
  return launch_scales(sc_dev, NS_S_F32, zp_dev, w->n, w, st);
}

// blob pieces already on the device: qbuf (packed), scales [ngroups_src][cstep], zp (or NULL)
int ns_launch_repack_btla(const void* qbuf_dev, const void* sc_dev, int src_stype, const int8_t* zp_dev, int cstep,
                          int kpad_src, int ntile, int packrow, int is_float, ns_weight* w, cudaStream_t st) {
  const size_t total = (size_t)w->n * (w->kpad >> 3);
  const unsigned blocks = (unsigned)((total + 255) / 256);
  if (w->wfmt == NS_W_S8) {
    SrcBtlaS8 src{(const int8_t*)qbuf_dev, kpad_src, ntile, packrow};
    repack_q_kernel<<<blocks, 256, 0, st>>>(src, w->n, w->k, w->kpad, w->wfmt, w->rows, (size_t)w->pitch);
  } else {
    SrcBtlaS4 src{(const uint8_t*)qbuf_dev, kpad_src, ntile, packrow, is_float};
    repack_q_kernel<<<blocks, 256, 0, st>>>(src, w->n, w->k, w->kpad, w->wfmt, w->rows, (size_t)w->pitch);
  }
  NS_CUDA_TRY(cudaGetLastError());
  ns_count_launch();
  return launch_scales(sc_dev, src_stype, zp_dev, cstep, w, st);
}

int ns_launch_dequant(const ns_weight* w, float* dst, int ld, cudaStream_t st) {
  const size_t total = (size_t)w->n * w->k;
  dequant_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(w->rows, (size_t)w->pitch, w->sc_off, w->zp_off,
                                                                  w->stype, w->asym, w->n, w->k, w->group, w->wfmt, w->f4kind, dst, ld);
  NS_CUDA_TRY(cudaGetLastError());
  ns_count_launch();
  return NS_OK;
}

extern "C" int ns_device_quantize_q4_0(const float* src_dev, void* dst_dev, int n, int k, void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (k % 32 != 0) {
    ns_set_error("ns_device_quantize_q4_0: k=%d not a multiple of 32", k);
    return NS_E_INVALID;
  }
  const size_t total = (size_t)n * (k / 32);
  quantize_q4_0_kernel<<<(unsigned)((total + 127) / 128), 128, 0, (cudaStream_t)queue>>>(src_dev, n, k, (uint8_t*)dst_dev);
  NS_CUDA_TRY(cudaGetLastError());
  ns_count_launch();
  return NS_OK;
}

// ---- synthetic weight image for benchmarks: random codes, scales ~ U[0.005, 0.02], zero points in [-4, 3] -------------------
namespace {
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}
__global__ void __launch_bounds__(256) random_weight_kernel(uint8_t* __restrict__ rows, int n, int pitch, int q_bytes, int sc_off, int zp_off,
                                                           int ngroups, int stype, int asym, uint32_t seed) {
  const int row = blockIdx.x;
  uint8_t* r = rows + (size_t)row * pitch;
  for (int i = threadIdx.x; i < q_bytes / 4; i += 256) reinterpret_cast<uint32_t*>(r)[i] = mix32(seed ^ (uint32_t)(row * 0x9e3779b9u) ^ (uint32_t)i * 0x85ebca6bu);
  for (int g = threadIdx.x; g < ngroups; g += 256) {
    const float sc = 0.005f + 0.015f * (float)(mix32(seed + 77u + (uint32_t)row * 131071u + (uint32_t)g) & 0xffff) * (1.f / 65536.f);
    if (stype == NS_S_F32) reinterpret_cast<float*>(r + sc_off)[g] = sc;
    else if (stype == NS_S_F16) reinterpret_cast<__half*>(r + sc_off)[g] = __float2half_rn(sc);
    else reinterpret_cast<__nv_bfloat16*>(r + sc_off)[g] = __float2bfloat16_rn(sc);
    if (asym) reinterpret_cast<int8_t*>(r + zp_off)[g] = (int8_t)((int)(mix32(seed + 991u + (uint32_t)row * 8191u + (uint32_t)g) & 7) - 4);
  }
}
}  // namespace

int ns_launch_random_weight(ns_weight* w, unsigned seed, cudaStream_t st) {
  random_weight_kernel<<<w->n, 256, 0, st>>>(w->rows, w->n, w->pitch, w->q_bytes, w->sc_off, w->zp_off, w->ngroups, w->stype, w->asym, seed);
  NS_CUDA_TRY(cudaGetLastError());
  ns_count_launch();
  return NS_OK;
}

// pack.cpp -- host side of the weight-packing API (offline path; no GPU involved, as in the reference).
//
// Mirrors core/layers/bestla_gemm.h:37-56 (BTLAGemmPackBSize / QuantPackB / PackB / UnPackB), which
// models/model_utils/quant_utils.cpp:226-400 (bestla_qpack / bestla_quantize) and the pybind entry points
// np_bestla_qpack / np_bestla_quantize (application/main_pybind.cpp:378,404) sit on.  The produced buffer is a
// serialized StorageWeightKBlockNInteger / NFloat (bestla/bestla/bestla_storage.h:697-860) laid out exactly as
// the reference's x86 cores expect, so a file quantised here loads in the reference and vice versa:
//   NE_COMP_INT8 -> AVX512_VNNI KBlock core  (NTile 48, PackRow 4, KTile 4,  COMP_INT8_US_FP32, reduce bf16)
//   NE_COMP_BF16 -> AMX_BF16 core            (NTile 48, PackRow 2, KTile 32, COMP_BF16_FP32)
//   NE_COMP_F16  -> AMX_FP16 core            (NTile 48, PackRow 2, KTile 32, COMP_FP16_FP32)
//   NE_COMP_F32  -> AVX512F core             (NTile 48, PackRow 1, KTile 1,  COMP_FP32)
// (bestla_defs.h:36-54; selection order as BTLAGemmPackBSizeLocal, bestla_gemm.cpp:248-300, for a CPU with all ISAs
// except that the AVX512_VNNI layout is preferred over AMX_INT8: same bytes, smaller K padding, loadable everywhere).
// Arithmetic follows bestla/bestla/kernel_ref.h:1608-1720 (RTN), :1802-1823 + :1373-1414 (NF4),
// bestla_utils.h:146-153 (bf16 RNE), bestla_prologue_b.h:244-335 (corrections), :455-470 + kernel_ref.h:2132 (reduce).
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/ns_b200.h"
#include "btla_blob.h"

void ns_set_error(const char* fmt, ...);  // abi.cu

namespace {

struct Core {
  int ntile, packrow, ktile;
  uint32_t comp;  // gemm::CompType
  uint32_t isa;   // BTLA_ISA
  bool is_int;
  uint64_t id() const { return (uint64_t)ntile | ((uint64_t)packrow << 8) | ((uint64_t)comp << 16) | ((uint64_t)isa << 32); }
};
const Core kCoreInt8{48, 4, 4, 4u | (3u << 4) | (0u << 8), 6, true};    // tAVX512_VNNI_KBlock, COMP_INT8_US_FP32
const Core kCoreBf16{48, 2, 32, 1u | (1u << 4) | (0u << 8), 9, false};  // tAMX_BF16
const Core kCoreFp16{48, 2, 32, 2u | (2u << 4) | (0u << 8), 11, false}; // tAMX_FP16
const Core kCoreFp32{48, 1, 1, 0u, 4, false};                           // tAVX512F

inline bool dtype_is_int(uint32_t t) { return ((t >> 8) & 0xff) == 1; }
inline int dtype_bits(uint32_t t) { return (int)(t & 0xff); }
inline size_t dtype_size(uint32_t t) { return (size_t)(dtype_bits(t) + 7) / 8; }
inline size_t pad_to(size_t a, size_t b) { return (a + b - 1) / b * b; }

const Core* pick_core(uint32_t qtype, size_t blk, bool asym, int comp) {
  const bool is_int = dtype_is_int(qtype);
  switch (comp) {
    case NS_NE_COMP_INT8:
      if (is_int && !(qtype == NS_BTLA_S8 && asym) && blk % kCoreInt8.ktile == 0) return &kCoreInt8;
      /* fallthrough */
    case NS_NE_COMP_BF16:
      if (blk % kCoreBf16.ktile == 0) return &kCoreBf16;
      /* fallthrough */
    case NS_NE_COMP_F16:
      if (blk % kCoreFp16.ktile == 0) return &kCoreFp16;
      /* fallthrough */
    case NS_NE_COMP_F32:
    case NS_NE_COMP_UNDEF:
      return &kCoreFp32;
    default:
      return nullptr;
  }
}

inline uint16_t bf16_rne(float v) {
  uint32_t u;
  memcpy(&u, &v, 4);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
inline float bf16_to_f32(uint16_t b) {
  uint32_t u = (uint32_t)b << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
inline uint16_t f16_rne(float f) {  // IEEE binary16, round-to-nearest-even
  uint32_t x;
  memcpy(&x, &f, 4);
  const uint32_t sign = (x >> 16) & 0x8000u, ax = x & 0x7fffffffu;
  if (ax >= 0x7f800000u) return (uint16_t)(sign | 0x7c00u | (ax > 0x7f800000u ? 0x200u : 0));
  if (ax >= 0x477ff000u) return (uint16_t)(sign | 0x7c00u);
  if (ax < 0x33000001u) return (uint16_t)sign;
  const int e = (int)(ax >> 23) - 127;
  uint32_t m = (ax & 0x7fffffu) | 0x800000u, base = 0;
  int shift = 13;
  if (e < -14) shift += -14 - e;
  else { base = (uint32_t)(e + 15) << 10; m &= 0x7fffffu; }
  uint32_t q = m >> shift;
  const uint32_t rem = m & ((1u << shift) - 1), half = 1u << (shift - 1);
  if (rem > half || (rem == half && (q & 1))) ++q;
  return (uint16_t)(sign | (base + q));
}
inline float f16_to_f32(uint16_t h) {
  const uint32_t sign = (uint32_t)(h & 0x8000u) << 16, exp = (h >> 10) & 0x1f;
  uint32_t man = h & 0x3ffu, bits;
  if (exp == 0) {
    if (!man) bits = sign;
    else {
      int e = -1;
      do { man <<= 1; ++e; } while (!(man & 0x400u));
      bits = sign | (uint32_t)(112 - e) << 23 | (man & 0x3ffu) << 13;
    }
  } else if (exp == 31) bits = sign | 0x7f800000u | man << 13;
  else bits = sign | (exp + 112) << 23 | man << 13;
  float f;
  memcpy(&f, &bits, 4);
  return f;
}

inline int round_away(float x) { return (int)roundf(x); }  // utils::cast<float,int>
inline int clampi(int v, int lo, int hi) { return std::min(std::max(v, lo), hi); }

const float kNf4Lut[16] = {0.f, -0.6961928009986877f, -0.5250730514526367f, -0.39491748809814453f, -0.28444138169288635f,
                           -0.18477343022823334f, -0.09105003625154495f, -1.f, 0.07958029955625534f, 0.16093020141124725f,
                           0.24611230194568634f, 0.33791524171829224f, 0.44070982933044434f, 0.5626170039176941f,
                           0.7229568362236023f, 1.0f};
// FP4 "BNB" and FP4 E2M1 codebooks (kernel_ref.h:1209-1230, :1300-1321): sign-magnitude, sign in bit 3
const float kBnbLut[8] = {0.f, 5.208333333e-03f, 0.66666667f, 1.f, 0.33333333f, 0.5f, 0.16666667f, 0.25f};
const float kE2m1Lut[8] = {0.f, 0.010416666666666666f, 0.16666666666666666f, 0.25f, 0.3333333333333333f, 0.5f, 0.6666666666666666f, 1.f};
inline float f4_level(uint32_t qtype, int u) {
  if (qtype == NS_BTLA_F4_BNB) return (u & 8) ? -kBnbLut[u & 7] : kBnbLut[u & 7];
  if (qtype == NS_BTLA_F4_E2M1) return (u & 8) ? -kE2m1Lut[u & 7] : kE2m1Lut[u & 7];
  return kNf4Lut[u];
}
inline int bnb_code(float x) {  // fp4_bnb_quantize, kernel_ref.h:1234-1256
  const int sign = x < 0 ? 8 : 0;
  x = std::fabs(x);
  if (x > 0.29166667f) {
    if (x > 0.583333f) return (x > 0.8333333f ? 3 : 2) + sign;
    return (x > 0.4166667f ? 5 : 4) + sign;
  }
  if (x > 0.0859375f) return (x > 0.20833333f ? 7 : 6) + sign;
  return (x > 0.00260417f ? 1 : 0) + sign;
}
inline int e2m1_code(float x) {  // fp4_e2m1_quantize, kernel_ref.h:1258-1298
  const int sign = x < 0 ? 8 : 0;
  x = std::fabs(x);
  if (x > 1.75f / 6) {
    if (x > 3.5f / 6) return (x > 5.f / 6 ? 7 : 6) + sign;
    return (x > 2.5f / 6 ? 5 : 4) + sign;
  }
  if (x > 0.53125f / 6) return (x > 1.25f / 6 ? 3 : 2) + sign;
  return (x > 0.03125f / 6 ? 1 : 0) + sign;
}
inline bool is_f4(uint32_t t) { return t == NS_BTLA_F4_NF4 || t == NS_BTLA_F4_BNB || t == NS_BTLA_F4_E2M1; }
inline int nf4_code(float x) {  // kernel_ref.h:1373-1414 as a sorted threshold walk
  static const float thr[15] = {-0.8480964004993439f, -0.6106329262256622f, -0.4599952697753906f, -0.33967943489551544f,
                                -0.23460740596055984f, -0.13791173323988914f, -0.045525018125772476f, 0.03979014977812767f,
                                0.1202552504837513f, 0.2035212516784668f, 0.2920137718319893f, 0.3893125355243683f,
                                0.5016634166240692f, 0.6427869200706482f, 0.8614784181118011f};
  static const int code[16] = {7, 1, 2, 3, 4, 5, 6, 0, 8, 9, 10, 11, 12, 13, 14, 15};
  int r = 0;
  while (r < 15 && x > thr[r]) ++r;
  return code[r];
}

// RTN quantisation of W[K][N] (row stride ldw) in K-blocks of g.  Outputs q [K][N], scales [nb][N], zps [nb][N].
void quantize_kn(const float* W, size_t ldw, int K, int N, int g, uint32_t qtype, bool asym, int8_t* q, float* scales,
                 int8_t* zps) {
  const bool nf4 = is_f4(qtype);  // any 4-bit float codebook: absmax scale, nearest level (quantize_f32_f4_rowblock, kernel_ref.h:1802)
  const int bits = dtype_bits(qtype);
  const int full = 1 << (bits - 1), symv = full - 1;
#pragma omp parallel for schedule(static)
  for (int n = 0; n < N; ++n) {
    for (int k0 = 0; k0 < K; k0 += g) {
      const int len = std::min(g, K - k0);
      const size_t sidx = (size_t)(k0 / g) * N + n;
      if (nf4) {
        float amax = FLT_MIN;
        for (int i = 0; i < len; ++i) amax = std::max(amax, std::fabs(W[(size_t)(k0 + i) * ldw + n]));
        scales[sidx] = amax;
        const float r = 1.f / amax;
        for (int i = 0; i < len; ++i) {
          const float x = W[(size_t)(k0 + i) * ldw + n] * r;
          q[(size_t)(k0 + i) * N + n] = (int8_t)(qtype == NS_BTLA_F4_BNB ? bnb_code(x) : qtype == NS_BTLA_F4_E2M1 ? e2m1_code(x) : nf4_code(x));
        }
      } else if (!asym) {
        float vmax = FLT_MIN, vmin = FLT_MAX, amax = 0.f;
        for (int i = 0; i < len; ++i) {
          const float v = W[(size_t)(k0 + i) * ldw + n];
          vmax = std::max(vmax, v);
          vmin = std::min(vmin, v);
          amax = std::max(amax, std::fabs(v));
        }
        float nval = (float)symv + 0.5f;
        const float sum = vmax + vmin;
        if (std::fabs(sum) >= amax / (float)full) nval = sum > 0.f ? (float)-full : (float)full;
        const float scale = amax / nval, rscale = 1.f / scale;
        scales[sidx] = scale;
        for (int i = 0; i < len; ++i) {
          float t = roundf(W[(size_t)(k0 + i) * ldw + n] * rscale);
          t = std::max(std::min(t, 127.f), -128.f);  // cast<float,int8_t>
          q[(size_t)(k0 + i) * N + n] = (int8_t)clampi((int)t, -full, symv);
        }
      } else {
        float vmax = 0.f, vmin = 0.f;
        for (int i = 0; i < len; ++i) {
          const float v = W[(size_t)(k0 + i) * ldw + n];
          vmax = std::max(vmax, v);
          vmin = std::min(vmin, v);
        }
        const float scale = (vmax - vmin) / (float)((1 << bits) - 1), rscale = 1.f / scale;
        scales[sidx] = scale;
        const int zp = clampi(round_away((0.f - vmin) * rscale) - full, -full, symv);
        zps[sidx] = (int8_t)zp;
        for (int i = 0; i < len; ++i)
          q[(size_t)(k0 + i) * N + n] = (int8_t)clampi(round_away(W[(size_t)(k0 + i) * ldw + n] * rscale) + zp, -full, symv);
      }
    }
  }
}

// ---- serialized layout ------------------------------------------------------------------------------------------------
// Bit planes: StorageWeightKBlockNInteger::resize (bestla_storage.h:724-745) sizes mQBuf as the SUM of power-of-two planes
// and compressBit{2,3,5,6,7}Weight (bestla_prologue_b.h:512-564) + compress_{2,3,5,6,7}bit (kernel_ref.h:178-345) fill
// them over the FLAT element index e of the tile-interleaved [NPad x KPad] buffer (the same order the 4-bit nibbles use):
//     code u = q + 2^(bits-1)                      (q = the signed integer the RTN quantiser produced)
//     bits 7:  4-bit plane @0 | 2-bit plane @E/2 | 1-bit plane @E/2+E/4      u = b4 | b2 << 4 | b1 << 6
//     bits 6:  4-bit plane @0 | 2-bit plane @E/2                             u = b4 | b2 << 4
//     bits 5:  4-bit plane @0 | 1-bit plane @E/2                             u = b4 | b1 << 4
//     bits 3:  2-bit plane @0 | 1-bit plane @E/4                             u = b2 | b1 << 2
//     bits 2:  2-bit plane @0
// inside a plane element e sits at bit (e % (8/w)) * w of byte e / (8/w) (utils::bit4x2 / bit2x4 / bit1x8 bit-fields, x86 order).
// Returns false, with L->n = 0, for the widths stored as nibbles (4) or bytes (8) and for widths BesTLA does not have.
bool plane_layout(int bits, size_t E, BlobPlanes* L) {
  static const int W[8][3] = {{0, 0, 0}, {1, 0, 0}, {2, 0, 0}, {2, 1, 0}, {0, 0, 0}, {4, 1, 0}, {4, 2, 0}, {4, 2, 1}};
  *L = BlobPlanes{};
  if (bits < 1 || bits > 7 || bits == 4) return false;
  for (int i = 0; i < 3 && W[bits][i]; ++i) {
    L->width[i] = W[bits][i];
    L->off[i] = L->bytes;
    L->bytes += (E * (size_t)W[bits][i] + 7) / 8;  // utils::updiv(KPad * NPad * w, 8)
    L->n = i + 1;
  }
  return true;
}

inline int plane_get(const uint8_t* q, const BlobPlanes& L, size_t e) {
  int u = 0, sh = 0;
  for (int i = 0; i < L.n; ++i) {
    const int w = L.width[i], per = 8 / w;
    u |= ((q[L.off[i] + e / per] >> ((e % per) * w)) & ((1 << w) - 1)) << sh;
    sh += w;
  }
  return u;
}

inline void plane_put(uint8_t* q, const BlobPlanes& L, size_t e, int u) {
  for (int i = 0; i < L.n; ++i) {
    const int w = L.width[i], per = 8 / w, mask = (1 << w) - 1;
    uint8_t& b = q[L.off[i] + e / per];
    b = (uint8_t)((b & ~(mask << ((e % per) * w))) | ((u & mask) << ((e % per) * w)));
    u >>= w;
  }
}

struct BlobLayoutIn {
  int N, K, blk;
  uint32_t qtype, stype;
  bool asym, has_reduce, has_shuffle, is_float;
  const Core* core;
};
struct BlobDims {
  int npad, kpad, nk_scale;
  size_t qbytes, sbytes, zbytes, rbytes, shbytes, total;
};

BlobDims blob_dims(const BlobLayoutIn& L) {
  BlobDims d{};
  d.npad = (int)pad_to(L.N, L.core->ntile);
  d.kpad = (int)pad_to(L.K, L.core->ktile);
  d.nk_scale = (int)((d.kpad + L.blk - 1) / L.blk);
  d.qbytes = ((size_t)d.npad * d.kpad * dtype_bits(L.qtype) + 7) / 8;
  BlobPlanes pl;
  if (plane_layout(dtype_bits(L.qtype), (size_t)d.npad * d.kpad, &pl)) d.qbytes = pl.bytes;
  const size_t csize = (size_t)d.nk_scale * d.npad;
  d.sbytes = csize * dtype_size(L.stype);
  d.zbytes = L.asym ? csize : 0;
  d.rbytes = L.has_reduce ? csize * 2 : 0;  // reduce dtype bf16 ("Reduce dtype set to bf16", bestla_gemm.cpp:244)
  d.shbytes = L.has_shuffle ? (size_t)L.K * 4 : 0;
  size_t t = 8 + 4 + 8 + 4 * 4 + 4 + 4 + 4;  // mSize, prologue, core id, NPad KPad N K, dtype, blocksize, dqblocksize
  t += 16 + d.qbytes + 64;
  t += 4 * 3 + 4 + 8;
  t += 16 + d.sbytes + 64;
  t += 1 + (d.zbytes ? 16 + d.zbytes + 64 : 0);
  t += 1 + (d.rbytes ? 16 + d.rbytes + 64 : 0);
  t += 1;  // double-quant buffer: absent
  // StorageWeightKBlockNFloat::resize leaves the shuffle object out of mSize (bestla_storage.h:836-860); the byte its
  // serializer still writes lands inside the 64-byte padding
  if (!L.is_float) t += 1 + (d.shbytes ? 16 + d.shbytes + 64 : 0);
  d.total = pad_to(t, 64);
  return d;
}

struct Writer {
  uint8_t* p;
  template <typename T>
  void put(T v) {
    memcpy(p, &v, sizeof(T));
    p += sizeof(T);
  }
  // ObjectAlignedBuffer<64>::serializeToBuffer: size, offset-to-64B-alignment (of the real address), pad, data
  uint8_t* aligned(size_t bytes) {
    put<size_t>(bytes);
    uint8_t* after = p + sizeof(size_t);
    const size_t off = (size_t)((64 - ((uintptr_t)after & 63)) & 63);
    put<size_t>(off);
    memset(p, 0, off);
    p += off;
    uint8_t* data = p;
    p += bytes;
    return data;
  }
  uint8_t* optional(size_t bytes) {
    put<uint8_t>(bytes ? 1 : 0);
    return bytes ? aligned(bytes) : nullptr;
  }
};

struct BlobPtrs {
  uint8_t *q, *scale, *zp, *red, *shuffle;
};

BlobPtrs write_header(void* buf, const BlobLayoutIn& L, const BlobDims& d) {
  memset(buf, 0, d.total);
  Writer w{(uint8_t*)buf};
  w.put<size_t>(d.total);
  w.put<uint32_t>(L.is_float ? 2u : 1u);
  w.put<uint64_t>(L.core->id());
  w.put<int>(d.npad);
  w.put<int>(d.kpad);
  w.put<int>(L.N);
  w.put<int>(L.K);
  w.put<uint32_t>(L.qtype);
  w.put<int>(L.blk);
  w.put<int>(0);
  BlobPtrs P{};
  P.q = w.aligned(d.qbytes);
  w.put<uint32_t>(L.stype);
  w.put<uint32_t>(L.is_float ? 0u : (uint32_t)NS_BTLA_S8);    // zp dtype (EleBitsUndef for float storage)
  w.put<uint32_t>(L.is_float ? 0u : (uint32_t)NS_BTLA_BF16);  // reduce dtype
  w.put<int>(d.npad);                                          // CStep
  w.put<size_t>((size_t)d.nk_scale * d.npad);                  // CSize
  P.scale = w.aligned(d.sbytes);
  P.zp = w.optional(d.zbytes);
  P.red = w.optional(d.rbytes);
  w.optional(0);
  P.shuffle = w.optional(d.shbytes);
  return P;
}

// reorderWeight + compressWeight: element (k, n) -> [n/NTile][k/PackRow][n%NTile][k%PackRow]; int4 nibble = q + 8,
// f4 nibble = code; element 2i in the low nibble (kernel_ref.h:155-165).  Padding holds value 0.
void pack_q(const int8_t* q, int N, int K, const BlobLayoutIn& L, const BlobDims& d, uint8_t* out) {
  const int nt = L.core->ntile, pr = L.core->packrow;
  const int bits = dtype_bits(L.qtype);
  const int bias = L.is_float ? 0 : 8;
  BlobPlanes pl;
  const bool planes = plane_layout(bits, (size_t)d.npad * d.kpad, &pl);
  // (a tile block is kpad * 48 consecutive elements: a multiple of 8, so no plane byte is shared between two threads)
#pragma omp parallel for schedule(static)
  for (int nb = 0; nb < d.npad / nt; ++nb) {
    for (int k = 0; k < d.kpad; ++k) {
      for (int j = 0; j < nt; ++j) {
        const int n = nb * nt + j;
        const int v = (n < N && k < K) ? q[(size_t)k * N + n] : 0;
        const size_t e = (size_t)nb * d.kpad * nt + (size_t)(k / pr) * pr * nt + (size_t)j * pr + (k % pr);
        if (bits == 8) {
          out[e] = (uint8_t)v;
        } else if (planes) {
          plane_put(out, pl, e, v + (1 << (bits - 1)));
        } else {
          const uint8_t u = (uint8_t)((v + bias) & 0xf);
          if (e & 1) out[e >> 1] = (uint8_t)((out[e >> 1] & 0x0f) | (u << 4));
          else out[e >> 1] = (uint8_t)((out[e >> 1] & 0xf0) | u);
        }
      }
    }
  }
}

// scales are read as f32, bf16, or (any other scale type) f16
float load_scale(const uint8_t* p, uint32_t stype, size_t i) {
  if (stype == NS_BTLA_F32) return ((const float*)p)[i];
  if (stype == NS_BTLA_BF16) return bf16_to_f32(((const uint16_t*)p)[i]);
  return f16_to_f32(((const uint16_t*)p)[i]);
}
inline size_t load_scale_bytes(uint32_t stype) { return stype == NS_BTLA_F32 ? 4 : 2; }

// fill scales / zp / reduce / shuffle of the blob from canonical inputs
void fill_corrections(const int8_t* q, const float* scales, const int8_t* zps, const int* shuffle, const BlobLayoutIn& L,
                      const BlobDims& d, const BlobPtrs& P) {
  const int raw_nb = (L.K + L.blk - 1) / L.blk;
  for (int b = 0; b < raw_nb; ++b)
    for (int n = 0; n < L.N; ++n) {
      const size_t di = (size_t)b * d.npad + n, si = (size_t)b * L.N + n;
      if (L.stype == NS_BTLA_F32) ((float*)P.scale)[di] = scales[si];
      else if (L.stype == NS_BTLA_BF16) ((uint16_t*)P.scale)[di] = bf16_rne(scales[si]);
      else ((uint16_t*)P.scale)[di] = f16_rne(scales[si]);
      if (P.zp) ((int8_t*)P.zp)[di] = zps ? zps[si] : 0;
    }
  if (P.red) {
    // reduceWeight (bestla_prologue_b.h:455-470): per K-block sum over k of the DEQUANTISED weight -- dequantised with the
    // scale as stored (bf16-rounded when scales are bf16) -- accumulated in fp32 in k order, stored as bf16
#pragma omp parallel for schedule(static)
    for (int n = 0; n < L.N; ++n)
      for (int b = 0; b < raw_nb; ++b) {
        const size_t di = (size_t)b * d.npad + n;
        const float s = load_scale(P.scale, L.stype, di);
        const int z = P.zp ? ((int8_t*)P.zp)[di] : 0;
        float acc = 0.f;
        const int kend = std::min(L.K, (b + 1) * L.blk);
        for (int k = b * L.blk; k < kend; ++k) acc += (float)(q[(size_t)k * L.N + n] - z) * s;
        ((uint16_t*)P.red)[di] = bf16_rne(acc);
      }
  }
  if (P.shuffle && shuffle) {
    // setShuffleIndices (bestla_prologue_b.h:337-356): group-sorted position -> original k
    int* out = (int*)P.shuffle;
    std::vector<int> count(raw_nb, 0);
    for (int k = 0; k < L.K; ++k) {
      const int g = shuffle[k];
      if (g >= 0 && g < raw_nb && count[g] < L.blk) out[(size_t)g * L.blk + count[g]++] = k;
    }
  }
}

bool make_layout(size_t N, size_t K, size_t blk, uint32_t qtype, uint32_t stype, bool asym, int comp, bool shuffle,
                 BlobLayoutIn* L) {
  if (!N || !K) return false;
  if (blk == 0 || blk > K) blk = K;
  const bool is_int = dtype_is_int(qtype);
  if (!(qtype == NS_BTLA_S4_CLIP || qtype == NS_BTLA_S8 || is_f4(qtype) || qtype == NS_BTLA_S2_CLIP ||
        qtype == NS_BTLA_S3_CLIP || qtype == NS_BTLA_S5_CLIP || qtype == NS_BTLA_S6_CLIP || qtype == NS_BTLA_S7_CLIP))
    return false;
  if (!(stype == NS_BTLA_F32 || stype == NS_BTLA_BF16 || stype == NS_BTLA_F16)) return false;
  const Core* c = pick_core(qtype, blk, asym, comp);
  if (!c) return false;
  L->N = (int)N;
  L->K = (int)K;
  L->blk = (int)blk;
  L->qtype = qtype;
  L->stype = stype;
  L->asym = is_int && asym;
  L->is_float = !is_int;
  L->core = c;
  L->has_reduce = is_int && c->is_int;
  L->has_shuffle = is_int && shuffle;
  return true;
}

struct Reader {
  const uint8_t* p;
  const uint8_t* end;
  bool ok = true;
  template <typename T>
  T get() {
    T v{};
    if (p + sizeof(T) > end) {
      ok = false;
      return v;
    }
    memcpy(&v, p, sizeof(T));
    p += sizeof(T);
    return v;
  }
  // ObjectAlignedBuffer<64>::deserializeBuffer (bestla_storage.h:98-110)
  void aligned_buf(const uint8_t** data, size_t* bytes) {
    const size_t sz = get<size_t>();
    const size_t off = get<size_t>();
    // sizes come from an untrusted file: compare against what is left instead of forming p + off + sz (which can wrap)
    if (!ok || off > (size_t)(end - p) || sz > (size_t)(end - p) - off) {
      ok = false;
      return;
    }
    p += off;
    *data = p;
    *bytes = sz;
    p += sz;
  }
  // ObjectOptionalBuffer<64> (bestla_storage.h:113-146): bool flag first
  void optional_buf(const uint8_t** data, size_t* bytes) {
    *data = nullptr;
    *bytes = 0;
    const uint8_t flag = get<uint8_t>();
    if (ok && flag) aligned_buf(data, bytes);
  }
};

}  // namespace

// ---- the reader ---------------------------------------------------------------------------------------------------------
size_t blob_size(const void* blob) {
  size_t msize;
  memcpy(&msize, blob, sizeof(size_t));
  return (msize >= 64 && msize <= ((size_t)1 << 40)) ? msize : 0;
}

bool parse_blob(const void* blob, BlobView* v, size_t avail) {
  if (!blob || (avail && avail < 64)) return false;
  memset(v, 0, sizeof(*v));
  const size_t msize = blob_size(blob);
  if (!msize || (avail && msize > avail)) {
    ns_set_error("blob: implausible size field (64 B .. 1 TiB, within the %zu readable bytes when that is known)", avail);
    return false;
  }
  Reader r{(const uint8_t*)blob, (const uint8_t*)blob + msize};
  v->size = r.get<size_t>();
  v->prologue = r.get<uint32_t>();
  v->core_id = r.get<uint64_t>();
  v->npad = r.get<int>();
  v->kpad = r.get<int>();
  v->n = r.get<int>();
  v->k = r.get<int>();
  v->dtype = r.get<uint32_t>();
  v->blocksize = r.get<int>();
  v->dqblocksize = r.get<int>();
  if (!r.ok || (v->prologue != 1 && v->prologue != 2)) {  // BTLA_PROLOGUEB_IDS (bestla.h:91-102)
    ns_set_error("blob: prologue id %u is not WeightKBlockNInteger/NFloat", v->prologue);
    return false;
  }
  r.aligned_buf(&v->qbuf, &v->qbytes);
  v->sca_t = r.get<uint32_t>();
  v->zp_t = r.get<uint32_t>();
  v->red_t = r.get<uint32_t>();
  v->cstep = r.get<int>();
  v->csize = r.get<size_t>();
  r.aligned_buf(&v->scale, &v->scale_bytes);
  r.optional_buf(&v->zp, &v->zp_bytes);
  r.optional_buf(&v->red, &v->red_bytes);
  r.optional_buf(&v->dq, &v->dq_bytes);
  const uint8_t* sh = nullptr;
  r.optional_buf(&sh, &v->shuffle_bytes);
  v->shuffle = (const int*)sh;
  if (!r.ok) {
    ns_set_error("blob: truncated or corrupt (size field %zu)", msize);
    return false;
  }
  // CoreAttr (bestla_gemm.h:83-125)
  v->ntile = (int)(v->core_id & 0xff);
  v->packrow = (int)((v->core_id >> 8) & 0xff);
  const unsigned comp = (unsigned)((v->core_id >> 16) & 0xffff);
  v->comp_a = comp & 0xf;
  v->comp_b = (comp >> 4) & 0xf;  // CompType B: tFP32=0 tBF16=1 tFP16=2 tS8=3 tU8=4 (bestla_gemm.h:22-83)
  v->ne_comp = v->comp_b == 0 ? NS_NE_COMP_F32 : v->comp_b == 1 ? NS_NE_COMP_BF16 : v->comp_b == 3 ? NS_NE_COMP_INT8 : NS_NE_COMP_UNDEF;
  v->bits = dtype_bits(v->dtype);
  if (v->n <= 0 || v->k <= 0 || v->npad < v->n || v->kpad < v->k || v->ntile <= 0 ||
      !(v->packrow == 1 || v->packrow == 2 || v->packrow == 4) || v->npad % v->ntile != 0 || v->kpad % v->packrow != 0 ||
      v->blocksize <= 0) {
    ns_set_error("blob: inconsistent header (N=%d K=%d NPad=%d KPad=%d NTile=%d PackRow=%d BlockSize=%d)", v->n, v->k, v->npad,
                 v->kpad, v->ntile, v->packrow, v->blocksize);
    return false;
  }
  // npad * kpad codes: bytes, nibbles or, for integer codes of any other width, bit planes
  const size_t E = (size_t)v->npad * v->kpad;
  const bool planes = v->prologue == 1 && plane_layout(v->bits, E, &v->planes);
  if (!planes && v->bits != 4 && v->bits != 8) {
    ns_set_error("blob: no layout for %d-bit codes in a prologue %u blob", v->bits, v->prologue);
    return false;
  }
  const size_t ngroups = ((size_t)v->kpad + v->blocksize - 1) / v->blocksize;
  if (v->qbytes < (planes ? v->planes.bytes : v->bits == 8 ? E : (E + 1) / 2) || v->cstep < v->n ||
      v->scale_bytes < ngroups * v->cstep * load_scale_bytes(v->sca_t) || (v->zp && v->zp_bytes < ngroups * v->cstep) ||
      (v->shuffle && v->shuffle_bytes < (size_t)v->k * 4)) {
    ns_set_error("blob: buffer sizes do not match the header");
    return false;
  }
  return true;
}

int blob_code(const BlobView& v, size_t e) {
  if (v.planes.n) return plane_get(v.qbuf, v.planes, e) - (1 << (v.bits - 1));
  if (v.bits == 8) return (int8_t)v.qbuf[e];
  const int u = (e & 1) ? (v.qbuf[e >> 1] >> 4) : (v.qbuf[e >> 1] & 0xf);
  return v.prologue == 2 ? u : u - 8;
}

extern "C" size_t BTLAGemmPackBSize(size_t N, size_t K, size_t BlkSize, uint32_t QuantType, uint32_t ScaleDtype, bool isAsym,
                                    int CompType, int* shuffle_indice) {
  BlobLayoutIn L;
  if (!make_layout(N, K, BlkSize, QuantType, ScaleDtype, isAsym, CompType, shuffle_indice != nullptr, &L)) return 0;
  return blob_dims(L).total;
}

extern "C" bool BTLAGemmPackB(void* PackedBuf, const int8_t* QData, const float* Scales, const int8_t* Zp, size_t N, size_t K,
                              size_t ldb, size_t BlkSize, uint32_t QuantType, uint32_t ScaleDtype, bool isAsym, int CompType,
                              int* shuffle_indice, void* ThreadPool) {
  (void)ThreadPool;
  BlobLayoutIn L;
  if (!PackedBuf || !QData || !Scales || !dtype_is_int(QuantType)) return false;  // float types: assert(0) in the reference
  if (!make_layout(N, K, BlkSize, QuantType, ScaleDtype, isAsym, CompType, shuffle_indice != nullptr, &L)) return false;
  if (L.asym && !Zp) return false;
  const BlobDims d = blob_dims(L);
  std::vector<int8_t> qc;
  const int8_t* q = QData;
  if (ldb != N) {  // compact rows
    qc.resize(N * K);
    for (size_t k = 0; k < K; ++k) memcpy(&qc[k * N], QData + k * ldb, N);
    q = qc.data();
  }
  const BlobPtrs P = write_header(PackedBuf, L, d);
  pack_q(q, (int)N, (int)K, L, d, P.q);
  fill_corrections(q, Scales, Zp, shuffle_indice, L, d, P);
  return true;
}

extern "C" bool BTLAGemmQuantPackB(void* PackedBuf, const float* FpData, size_t N, size_t K, size_t ldb, size_t BlkSize,
                                   uint32_t QuantType, uint32_t ScaleDtype, bool isAsym, int CompType, bool isTrans,
                                   void* ThreadPool) {
  (void)ThreadPool;
  BlobLayoutIn L;
  if (!PackedBuf || !FpData) return false;
  if (!make_layout(N, K, BlkSize, QuantType, ScaleDtype, isAsym, CompType, false, &L)) return false;
  const BlobDims d = blob_dims(L);
  // isTrans: FpData is the torch layout [N][K] (ldb = K); else [K][N] (quant_utils.cpp:344-347)
  std::vector<float> wt;
  const float* W = FpData;
  size_t ldw = ldb;
  if (isTrans) {
    wt.resize(N * K);
#pragma omp parallel for schedule(static)
    for (long long n = 0; n < (long long)N; ++n)
      for (size_t k = 0; k < K; ++k) wt[k * N + n] = FpData[n * ldb + k];
    W = wt.data();
    ldw = N;
  }
  const int nb = (int)((K + L.blk - 1) / L.blk);
  std::vector<int8_t> q(N * K), zp(L.asym ? (size_t)nb * N : 0);
  std::vector<float> sc((size_t)nb * N);
  quantize_kn(W, ldw, (int)K, (int)N, L.blk, QuantType, L.asym, q.data(), sc.data(), L.asym ? zp.data() : nullptr);
  const BlobPtrs P = write_header(PackedBuf, L, d);
  pack_q(q.data(), (int)N, (int)K, L, d, P.q);
  fill_corrections(q.data(), sc.data(), L.asym ? zp.data() : nullptr, nullptr, L, d, P);
  return true;
}

// FpData [K][ldb] <- dequantised weight (unpackWeight, bestla_prologue_b.h:212-242: "packed ... to KxN f32 weight")
extern "C" bool BTLAGemmUnPackB(float* FpData, const void* PackedBuf, size_t N, size_t K, size_t ldb, void* ThreadPool) {
  (void)ThreadPool;
  BlobView v;
  if (!FpData || !parse_blob(PackedBuf, &v) || (size_t)v.n != N || (size_t)v.k != K || ldb < N) return false;
  const int nt = v.ntile, pr = v.packrow;
  const bool f4 = v.prologue == 2 && v.bits == 4;
#pragma omp parallel for schedule(static)
  for (long long kk = 0; kk < (long long)K; ++kk)
    for (size_t nn = 0; nn < N; ++nn) {
      const size_t e = (size_t)(nn / nt) * v.kpad * nt + (size_t)(kk / pr) * pr * nt + (size_t)(nn % nt) * pr + (kk % pr);
      const size_t ci = (size_t)(kk / v.blocksize) * v.cstep + nn;
      const float s = load_scale(v.scale, v.sca_t, ci);
      const int c = blob_code(v, e);
      FpData[(size_t)kk * ldb + nn] = f4 ? f4_level(v.dtype, c) * s : (float)(c - (v.zp ? (int8_t)v.zp[ci] : 0)) * s;
    }
  return true;
}

// Re-quantise an fp32 [k][ld] matrix (n columns used) with the attributes (block size, dtype, scale type, asym, compute
// type) of a parsed blob (ne_bestla.cpp:79-112)
static bool quant_pack_like(const BlobView& v, void* dst, const float* f32, size_t n, size_t k, size_t ld) {
  return BTLAGemmQuantPackB(dst, f32, n, k, ld, (size_t)v.blocksize, v.dtype, v.sca_t, v.zp != nullptr, v.ne_comp, false, nullptr);
}

// Nothing is written when srcptr is not a k-block blob, as in the reference.
extern "C" void bestla_packweight_copyattr(const float* f32ptr, void* dstptr, int n, int k, int ld, void* srcptr) {
  BlobView v;
  if (!f32ptr || !dstptr || !parse_blob(srcptr, &v)) return;
  quant_pack_like(v, dstptr, f32ptr, (size_t)n, (size_t)k, (size_t)ld);
}

// Tensor-parallel shard of a blob (bestla_split_weight, models/model_utils/model_files.h:1538-1562): unpack to fp32
// [src_k][src_n], take the [dst_k][dst_n] block at (k_rank, n_rank) -- or, with qkv_fusion, the rank's third of each of the
// three N-concatenated projections -- and re-quantise it with the source blob's attributes.
extern "C" size_t ns_split_weight_size(const void* src, size_t dst_n, size_t dst_k) {
  BlobView v;
  if (!parse_blob(src, &v)) return 0;
  return BTLAGemmPackBSize(dst_n, dst_k, (size_t)v.blocksize, v.dtype, v.sca_t, v.zp != nullptr, v.ne_comp, nullptr);
}
extern "C" bool ns_split_weight(const void* src, void* dst, size_t src_n, size_t src_k, size_t dst_n, size_t dst_k, size_t n_rank,
                                size_t k_rank, bool qkv_fusion) {
  BlobView v;
  if (!dst || !parse_blob(src, &v) || (size_t)v.n != src_n || (size_t)v.k != src_k) return false;
  if ((n_rank + 1) * dst_n > src_n || (k_rank + 1) * dst_k > src_k || (qkv_fusion && (dst_n % 3 || src_n % 3))) return false;
  std::vector<float> fp(src_n * src_k);
  if (!BTLAGemmUnPackB(fp.data(), src, src_n, src_k, src_n, nullptr)) return false;
  if (qkv_fusion) {
    std::vector<float> part(dst_n * dst_k);
    for (size_t i = 0; i < dst_k; ++i)
      for (int j = 0; j < 3; ++j)
        memcpy(part.data() + dst_n * i + j * dst_n / 3, fp.data() + src_n * (k_rank * dst_k + i) + j * src_n / 3 + n_rank * dst_n / 3,
               dst_n / 3 * sizeof(float));
    return quant_pack_like(v, dst, part.data(), dst_n, dst_k, dst_n);
  }
  return quant_pack_like(v, dst, fp.data() + k_rank * dst_k * src_n + n_rank * dst_n, dst_n, dst_k, src_n);
}

// quantize_row_q4_0_reference (vectors/cpu/quantize.h:243-279); x*id + 8.5f as one fma, as the reference's default
// x86 build contracts it (see oracle/oracle_ggml.c).
extern "C" void ns_quantize_row_q4_0(const float* x, void* vy, int k) {
  uint8_t* y = (uint8_t*)vy;
  for (int b = 0; b < k / 32; ++b, y += 18) {
    const float* xb = x + b * 32;
    float amax = 0.f, vmax = 0.f;
    for (int j = 0; j < 32; ++j)
      if (std::fabs(xb[j]) > amax) {
        amax = std::fabs(xb[j]);
        vmax = xb[j];
      }
    const float d = vmax / -8.f;
    const float id = d != 0.f ? 1.0f / d : 0.0f;
    const uint16_t h = f16_rne(d);
    memcpy(y, &h, 2);
    for (int j = 0; j < 16; ++j) {
      const int lo = std::min(15, (int)(int8_t)fmaf(xb[j], id, 8.5f));
      const int hi = std::min(15, (int)(int8_t)fmaf(xb[j + 16], id, 8.5f));
      y[2 + j] = (uint8_t)(lo | (hi << 4));
    }
  }
}

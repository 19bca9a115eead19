// gemm_imma.cu -- batched decode (5..32 activation rows): 4-bit weights x int8 activations on the INTEGER tensor cores.
//
// Replaces, for 4 < M <= 32, what the reference runs through LauncherIntKBlock + the VNNI / AMX int8 GemmCores
// (bestla/bestla/bestla_wrapper.h:214-350, bestla_gemm.h "ICoreRowNAvx512vnniKBlock" etc.): u8 (or s8) activations quantised
// per K-block (kernel_ref.h:1825 / :1886; quantize_row_q8_0 for ggml weights), exact integer dot per K-block, then
// fp32 accumulation of  isum * a_scale * w_scale  -- the same arithmetic as the M <= 4 GEMV (gemv_ring.cu), so a batch of 8 or
// 32 sequences gets bit-for-bit the block sums a single sequence gets, and the weights are read from HBM ONCE per step
// (the GEMV tiles re-read them every 4 rows; the bf16 wgmma GEMM changes the numerics).
//
// Built on mma.sync m16n8k32 u8 x s8 (native on sm_90a: SASS IMMA.16832.U8.S8); wgmma's integer form (s8 / u8 only) would need
// the per-32 / per-128-block rescaling out of its accumulator registers every block, which mma.sync fragments give directly.
//
// Tiling.  CTA = 128 weight rows (8 consumer warps x 16 rows = the MMA's M) x all MT tokens (MMA N = 8 per instruction) x a
// K range (split-K fills the SMs when N/128 is small).  One producer warp feeds a shared-memory ring, a stage = 256 k:
//   * the nibbles of 128 rows x 128 bytes as ONE 2-D TMA box with the 128-byte swizzle (cp.async.bulk.tensor, SASS UTMALDG), so
//     ldmatrix over 8 rows is bank-conflict free;
//   * the activations of the stage -- [8 chunks][MT tokens][32 B codes] + [8][MT] {scale, sum|zero point} -- as one 1-D bulk
//     copy out of the image act_quant_imma_kernel wrote (bytes already in MMA B-fragment order).
// A word of packed nibbles (8 consecutive k) gives MMA k-slots 4t..4t+3 (low nibbles) and 16+4t..16+4t+3 (high nibbles) of
// thread t of a quad; the activation image stores the matching bytes (nsb.cuh: (e0,e4,e1,e5) / (e2,e6,e3,e7)), so no
// shuffling happens in the loop: ldmatrix, 4 LOP, one 8-byte shared load per 8 tokens, MMA.
// Scales and zero points of the CTA's rows / K range are staged once, before griddepcontrol.wait (weights are constant).
// Split-K: partial tiles go to a workspace; the last CTA of a tile (ticket) sums them in split order -- deterministic --
// and runs the epilogue (bias, GELU, residual, QKV layout, SiLU(gate) * up).
#include <cuda.h>

#include "nsb.cuh"
#include "quant_smem.cuh"

namespace {

constexpr int BN = 128;   // weight rows per CTA
constexpr int KS = 256;   // k per ring stage
constexpr int kCons = 8;  // consumer warps
constexpr int kThr = (kCons + 1) * 32;
constexpr int kQStage = BN * (KS / 2);  // 16 KB of nibbles

struct ImmaParams {
  const uint8_t* rows[3];
  int n[3];
  long long dst_off[3];
  int tile0[3];  // first tile of each weight (plain / concat)
  int nw, mode;
  int k, group, cpg, acpg;  // 32-chunks per weight group / per activation block (powers of two)
  int cpg_shift;
  int pitch, sc_off, zp_off;
  const uint8_t* act_img;
  float* dst;
  int ldo, m;
  const float* bias;
  int bias_bcast;
  const float* residual;
  int eltop;
  int tiles, ksplit, nslices;
  float* partial;     // [ksplit][tiles][MT][BN]
  unsigned* tickets;  // [tiles], zero on entry (act_quant_imma_kernel clears them), zero again on exit
  int sc_row;         // bytes per row of the staged scales (+ zero points)
  int sc_zp;          // offset of the zero points inside a staged row
  int stages;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void tma_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
               "l"(map), "r"(x), "r"(y), "r"(bar)
               : "memory");
}
__device__ __forceinline__ uint2 lds64(uint32_t a) {
  uint2 r;
  asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "r"(a));
  return r;
}
__device__ __forceinline__ uint4 lds128(uint32_t a) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a));
  return r;
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t a, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
template <bool ACT_U8>
__device__ __forceinline__ void imma(int (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if (ACT_U8)
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// the same with a zero accumulator input: d = a x b (block size 32: every chunk is flushed, nothing to carry)
template <bool ACT_U8>
__device__ __forceinline__ void imma0(int (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if (ACT_U8)
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
                 : "=r"(c[0]), "=r"(c[1]), "=r"(c[2]), "=r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "r"(0));
  else
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
                 : "=r"(c[0]), "=r"(c[1]), "=r"(c[2]), "=r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "r"(0));
}
// exact int -> float for |i| < 2^22 without the quarter-rate I2F: (float)(i + 0x4B400000 as float bits) - 12582912
__device__ __forceinline__ float i2f_small(int i) { return __int_as_float(i + 0x4B400000) - 12582912.f; }

// ---- activation image ------------------------------------------------------------------------------------------------
// One warp per (token, activation block).  Same arithmetic as act_quant_kernel<COMP> (act_prep.cu) -- bit-exact codes, scales,
// zero points -- different destination: per K-slice of 256, [8 chunks][MT tokens][32 B] codes then [8][MT] {scale, S|za<<16}
// where S is the sum of the codes of the WHOLE activation block (the matmul corrects per block, not per chunk).
// Tokens >= M and chunks past K are written as zeros (scale 0): they contribute nothing.  Block 0 also clears the tickets.
template <int COMP>
__global__ void __launch_bounds__(256) act_quant_imma_kernel(const float* __restrict__ A, int lda, int M, int K, int qg, int MT, int nslices,
                                                             uint8_t* __restrict__ img, unsigned* __restrict__ tickets, int ntickets) {
  pdl_launch_dependents();
  pdl_wait();
  if (blockIdx.x == 0)
    for (int i = threadIdx.x; i < ntickets; i += blockDim.x) tickets[i] = 0u;
  const int lane = threadIdx.x & 31;
  const int cpb = qg >> 5;                   // chunks per activation block
  const int nblk = nslices * 8 / cpb;        // blocks per token, padding included
  const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (gw >= MT * nblk) return;
  const int m = gw / nblk, b = gw - m * nblk;
  const int k0 = b * qg;
  const size_t slice_bytes = (size_t)MT * 320;
  const bool live = m < M && k0 < K;
  const float* row = A + (size_t)(live ? m : 0) * lda;
  const int kend = min(k0 + qg, K);

  float vmax = (COMP == NS_COMP_Q8_0) ? 0.f : 1.17549435e-38f, vmin = 0.f;
  if (COMP == NS_COMP_INT8 && live && k0 + qg > K) vmax = 0.f;  // partial block: as act_quant_kernel
  float v[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    v[c] = 0.f;
    if (c < cpb) {
      const int k = k0 + c * 32 + lane;
      if (live && k < kend) {
        v[c] = row[k];
        if (COMP == NS_COMP_INT8) {
          vmax = fmaxf(v[c], vmax);
          vmin = fminf(v[c], vmin);
        } else {
          vmax = fmaxf(vmax, fabsf(v[c]));
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    if (COMP == NS_COMP_INT8) vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, o));
  }
  float scale, rscale;
  int za = 0;
  if (COMP == NS_COMP_Q8_0) {
    scale = __half2float(__float2half_rn(vmax / 127.f));
    rscale = vmax != 0.f ? 127.f / vmax : 0.f;
  } else if (COMP == NS_COMP_INT8) {
    scale = (vmax - vmin) / 255;
    za = nsq::cast_u8((0 - vmin) / scale);
    rscale = 1.f / scale;
  } else {
    scale = vmax / 127;
    rscale = 1.f / scale;
  }
  int q[8], stot = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    q[c] = 0;
    if (c < cpb) {
      const int k = k0 + c * 32 + lane;
      if (live && k < kend) {
        if (COMP == NS_COMP_Q8_0) q[c] = __float2int_rn(v[c] * rscale);
        else if (COMP == NS_COMP_INT8) q[c] = nsq::cast_u8((float)za + (float)(int)roundf(v[c] * rscale));
        else q[c] = nsq::cast_s8(v[c] * rscale);
      } else if (live) {
        q[c] = za;  // padding inside a live block contributes (a - za) == 0
      }
      stot += q[c];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) stot += __shfl_xor_sync(0xffffffffu, stot, o);
  if (!live) {
    scale = 0.f;
    za = 0;
    stot = 0;
  }
  const int pos = (lane & ~7) | (((lane & 3) << 1) | ((lane & 7) >> 2));  // byte order of the dp4a / MMA operands (nsb.cuh)
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    if (c < cpb) {
      const int ch = b * cpb + c;  // global chunk
      uint8_t* sl = img + (size_t)(ch >> 3) * slice_bytes;
      const int j = ch & 7;
      sl[(size_t)j * MT * 32 + (size_t)m * 32 + pos] = (uint8_t)q[c];
      if (lane == 0)
        *reinterpret_cast<int2*>(sl + (size_t)MT * 256 + ((size_t)j * MT + m) * 8) =
            make_int2(__float_as_int(scale), (stot & 0xffff) | (za << 16));
    }
  }
}

// ---- the matmul ------------------------------------------------------------------------------------------------------
template <int STYPE>
__device__ __forceinline__ float lds_scale_b(uint32_t a) {  // a: byte address of the scale
  if (STYPE == NS_S_F32) {
    uint32_t r;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(a));
    return __uint_as_float(r);
  }
  unsigned short h;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(a));
  if (STYPE == NS_S_F16) return __half2float(__ushort_as_half(h));
  return __uint_as_float((uint32_t)h << 16);
}

// PER: 32-chunks per activation block, compile-time for the common cases (1: ggml Q8_0 / group 32, 4: group 128) so that the
// eight chunks of a stage are one straight-line schedule; 0: read from the parameters (groups 64 / 256)
template <bool ACT_U8, int MT, bool ASYM, int STYPE, int PER>
__global__ void __launch_bounds__(kThr, 2)
    gemm_imma_kernel(const __grid_constant__ CUtensorMap map0, const __grid_constant__ CUtensorMap map1,
                     const __grid_constant__ CUtensorMap map2, const ImmaParams P) {
  constexpr int NTB = MT / 8;
  constexpr int kActStage = MT * 320;
  constexpr int kStage = kQStage + ((kActStage + 1023) / 1024) * 1024;  // q boxes must stay 1024-B aligned (128B swizzle)
  constexpr int SS = (STYPE == NS_S_F32) ? 4 : 2;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  // 128B-swizzled TMA boxes need 1024-byte aligned destinations: align by hand (the launcher adds the slack)
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t base = smem_u32(smem);
  const int stages = P.stages;
  const uint32_t sc_s = base + (uint32_t)stages * kStage;           // staged scales (+zp): [BN][sc_row]
  const uint32_t full0 = sc_s + (uint32_t)BN * P.sc_row;            // 8-B aligned: sc_row is a multiple of 8
  const uint32_t empty0 = full0 + 8u * stages;
  __shared__ int s_last;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x / P.ksplit, split = blockIdx.x - tile * P.ksplit;
  const int sl0 = (int)((long long)P.nslices * split / P.ksplit), sl1 = (int)((long long)P.nslices * (split + 1) / P.ksplit);
  const int nsl = sl1 - sl0;
  const bool gate_up = P.mode == NS_GEMV_GATE_UP_SILU;
  // which rows: plain / concat -> one weight, BN consecutive rows; gate/up -> 64 rows of w1 then the same 64 rows of w3
  int wi = 0;
  if (!gate_up) {
    if (P.nw > 1 && tile >= P.tile0[1]) wi = 1;
    if (P.nw > 2 && tile >= P.tile0[2]) wi = 2;
  }
  const int r0 = gate_up ? tile * (BN / 2) : (tile - P.tile0[wi]) * BN;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, kCons);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kCons) {
    // ===================== producer =====================
    if (lane == 0) {
      const CUtensorMap* mp0 = gate_up ? &map0 : (wi == 0 ? &map0 : (wi == 1 ? &map1 : &map2));
      const CUtensorMap* mp1 = &map1;
      auto issue_w = [&](int i, int s) {
        const uint32_t dst = base + (uint32_t)s * kStage;
        mbar_expect_tx(full0 + 8 * s, (uint32_t)(kQStage + kActStage));
        const int x = (sl0 + i) * (KS / 2);
        if (gate_up) {
          tma_2d(dst, mp0, x, r0, full0 + 8 * s);
          tma_2d(dst + (BN / 2) * (KS / 2), mp1, x, r0, full0 + 8 * s);
        } else {
          tma_2d(dst, mp0, x, r0, full0 + 8 * s);
        }
      };
      auto issue_a = [&](int i, int s) {
        bulk_g2s(base + (uint32_t)s * kStage + kQStage, P.act_img + (size_t)(sl0 + i) * kActStage, (uint32_t)kActStage, full0 + 8 * s);
      };
      const int pre = nsl < stages ? nsl : stages;
      for (int i = 0; i < pre; ++i) issue_w(i, i);  // weights do not depend on the previous kernel
      pdl_wait();                                   // the activation image does
      for (int i = 0; i < pre; ++i) issue_a(i, i);
      int s = 0;
      uint32_t phase = 0;
      for (int i = pre; i < nsl; ++i) {
        mbar_wait(empty0 + 8 * s, phase);
        issue_w(i, s);
        issue_a(i, s);
        if (++s == stages) {
          s = 0;
          phase ^= 1u;
        }
      }
    }
    return;
  }

  // ===================== consumers =====================
  // stage the scales (+ zero points) of this CTA's rows and K range: constant data, read before the dependency wait.
  // 16-byte segments (the range starts wherever group g0 falls: keep its misalignment inside the staged row), all loads of a
  // thread issued before the first store -- a scalar loop here cost more than the whole matmul.
  const int g0 = (sl0 * 8) >> P.cpg_shift;                          // first weight group of the range
  const int ng = ((sl1 * 8 + P.cpg - 1) >> P.cpg_shift) - g0;       // groups in the range
  const int dsc = (SS * g0) & 15, dzp = g0 & 15;                    // sc_off and zp_off are 16-byte multiples
  const int nsc = (dsc + SS * ng + 15) >> 4, nzp = ASYM ? (dzp + ng + 15) >> 4 : 0;
  const int scb = P.sc_zp;                                          // byte offset of the zero-point area in a staged row
  {
    const int nseg = nsc + nzp;
    constexpr int U = 4;
    for (int i0 = threadIdx.x; i0 < BN * nseg; i0 += U * kCons * 32) {
      uint4 v[U];
      uint32_t d[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int idx = i0 + u * kCons * 32;
        d[u] = 0u;
        if (idx < BN * nseg) {
          const int r = idx / nseg, sg = idx - r * nseg;
          int row, w = wi;
          if (gate_up) {
            w = r >= BN / 2 ? 1 : 0;
            row = r0 + (r & (BN / 2 - 1));
          } else {
            row = r0 + r;
          }
          if (row >= P.n[w]) row = 0;  // overhang rows: any valid data, the epilogue masks them
          const uint8_t* src = P.rows[w] + (size_t)row * P.pitch;
          if (sg < nsc) {
            src += ((P.sc_off + SS * g0) & ~15) + 16 * sg;
            d[u] = sc_s + (uint32_t)r * P.sc_row + 16u * sg;
          } else {
            src += ((P.zp_off + g0) & ~15) + 16 * (sg - nsc);
            d[u] = sc_s + (uint32_t)r * P.sc_row + scb + 16u * (sg - nsc);
          }
          v[u] = __ldg(reinterpret_cast<const uint4*>(src));
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (d[u]) asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(d[u]), "r"(v[u].x), "r"(v[u].y), "r"(v[u].z), "r"(v[u].w) : "memory");
    }
  }
  asm volatile("bar.sync 1, %0;" ::"n"(kCons * 32) : "memory");

  const int g = lane >> 2, t = lane & 3;
  const int rA = warp * 16 + g, rB = rA + 8;  // rows of this thread inside the tile
  const uint32_t scA = sc_s + (uint32_t)rA * P.sc_row + dsc, scB = sc_s + (uint32_t)rB * P.sc_row + dsc;
  const uint32_t zpo = (uint32_t)(scb + dzp - dsc);
  // ldmatrix row address of this lane: matrices 0/1 = rows +0..7 / +8..15 of chunk j, matrices 2/3 = the same rows of chunk j+1
  const int lrow = warp * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
  const int lsel = lane >> 4;  // 0: chunk j, 1: chunk j + 1
  // 128B swizzle: 16-byte unit index ^ (row & 7).  chunk j2 + lsel with j2 even = j2 ^ lsel, so the per-thread part of the
  // address is fixed and the chunk pair enters as one XOR
  const uint32_t lthread = (uint32_t)lrow * 128u + ((uint32_t)(lsel ^ (lrow & 7)) << 4);

  float acc[NTB][4];
  int ci[NTB][4];
  int cs[4] = {0, 0, 0, 0};
#pragma unroll
  for (int tb = 0; tb < NTB; ++tb)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      acc[tb][i] = 0.f;
      ci[tb][i] = 0;
    }

  int s = 0;
  uint32_t phase = 0;
  constexpr bool P1 = PER == 1;
  const int period = PER ? PER : P.acpg;
  for (int i = 0; i < nsl; ++i) {
    const int gstage = (((sl0 + i) * 8) >> P.cpg_shift) - g0;  // first weight group of the stage (a stage holds whole groups)
    mbar_wait(full0 + 8 * s, phase);
    const uint32_t qs = base + (uint32_t)s * kStage;
    const uint32_t as = qs + kQStage;
    const uint32_t ms = as + MT * 256;
#pragma unroll
    for (int j2 = 0; j2 < 8; j2 += 2) {
      uint32_t w0, w1, w2, w3;
      ldmatrix_x4(qs + (lthread ^ ((uint32_t)j2 << 4)), w0, w1, w2, w3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int j = j2 + h;
        const uint32_t wa = h ? w2 : w0, wb = h ? w3 : w1;
        const uint32_t a[4] = {wa & 0x0F0F0F0Fu, wb & 0x0F0F0F0Fu, (wa >> 4) & 0x0F0F0F0Fu, (wb >> 4) & 0x0F0F0F0Fu};
#pragma unroll
        for (int tb = 0; tb < NTB; ++tb) {
          const uint2 b = lds64(as + (uint32_t)j * (MT * 32) + (uint32_t)(tb * 8 + g) * 32u + 8u * t);
          if (P1) imma0<ACT_U8>(ci[tb], a, b.x, b.y);
          else imma<ACT_U8>(ci[tb], a, b.x, b.y);
        }
        if (ACT_U8) {  // row sums of the weight codes (zero-point term)
          if (P1) imma0<true>(cs, a, 0x01010101u, 0x01010101u);
          else imma<true>(cs, a, 0x01010101u, 0x01010101u);
        }
        if (PER ? ((j + 1) % (PER ? PER : 1) == 0) : (((j + 1) & (period - 1)) == 0)) {
          // end of an activation block: exact integer block sums -> fp32
          const int gi = gstage + (PER == 1 ? j : (PER ? j / (PER ? PER : 1) : (j >> P.cpg_shift)));
          const float wsA = lds_scale_b<STYPE>(scA + SS * gi), wsB = lds_scale_b<STYPE>(scB + SS * gi);
          int offA = 8, offB = 8;
          if (ASYM) {
            int z;
            asm volatile("ld.shared.s8 %0, [%1];" : "=r"(z) : "r"(scA + zpo + gi));
            offA += z;
            asm volatile("ld.shared.s8 %0, [%1];" : "=r"(z) : "r"(scB + zpo + gi));
            offB += z;
          }
          const int nel = 32 * period;
#pragma unroll
          for (int tb = 0; tb < NTB; ++tb) {
            const uint4 mt = lds128(ms + (uint32_t)(j * MT + tb * 8 + 2 * t) * 8u);  // {scale, S|za} of tokens 2t, 2t+1
            const float as0 = __uint_as_float(mt.x), as1 = __uint_as_float(mt.z);
            const int sa0 = ACT_U8 ? (int)(mt.y & 0xffffu) : (int)(short)(mt.y & 0xffffu);
            const int sa1 = ACT_U8 ? (int)(mt.w & 0xffffu) : (int)(short)(mt.w & 0xffffu);
            int i0 = ci[tb][0] - offA * sa0, i1 = ci[tb][1] - offA * sa1;
            int i2 = ci[tb][2] - offB * sa0, i3 = ci[tb][3] - offB * sa1;
            if (ACT_U8) {
              const int za0 = (int)((mt.y >> 16) & 0xffu), za1 = (int)((mt.w >> 16) & 0xffu);
              const int uA = cs[0] - nel * offA, uB = cs[2] - nel * offB;
              i0 -= za0 * uA;
              i1 -= za1 * uA;
              i2 -= za0 * uB;
              i3 -= za1 * uB;
            }
            acc[tb][0] = fmaf(i2f_small(i0), as0 * wsA, acc[tb][0]);  // |block sum| < 2^22: 256 x 255 x 15 < 1e6
            acc[tb][1] = fmaf(i2f_small(i1), as1 * wsA, acc[tb][1]);
            acc[tb][2] = fmaf(i2f_small(i2), as0 * wsB, acc[tb][2]);
            acc[tb][3] = fmaf(i2f_small(i3), as1 * wsB, acc[tb][3]);
            if (!P1) ci[tb][0] = ci[tb][1] = ci[tb][2] = ci[tb][3] = 0;
          }
          if (!P1) cs[0] = cs[1] = cs[2] = cs[3] = 0;
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty0 + 8 * s);
    if (++s == stages) {
      s = 0;
      phase ^= 1u;
    }
  }

  // ---- epilogue: tile [MT][BN] through shared memory (the ring is drained: every issued stage was consumed) ----
  asm volatile("bar.sync 1, %0;" ::"n"(kCons * 32) : "memory");
  float* tb_s = reinterpret_cast<float*>(smem);
#pragma unroll
  for (int tb = 0; tb < NTB; ++tb) {
    tb_s[(tb * 8 + 2 * t) * BN + rA] = acc[tb][0];
    tb_s[(tb * 8 + 2 * t + 1) * BN + rA] = acc[tb][1];
    tb_s[(tb * 8 + 2 * t) * BN + rB] = acc[tb][2];
    tb_s[(tb * 8 + 2 * t + 1) * BN + rB] = acc[tb][3];
  }
  asm volatile("bar.sync 1, %0;" ::"n"(kCons * 32) : "memory");
  const int ctid = threadIdx.x;  // 0..255
  if (P.ksplit > 1) {
    float4* mine = reinterpret_cast<float4*>(P.partial + ((size_t)split * P.tiles + tile) * (MT * BN));
    for (int idx = ctid; idx < MT * BN / 4; idx += kCons * 32) mine[idx] = reinterpret_cast<const float4*>(tb_s)[idx];
    __threadfence();
    asm volatile("bar.sync 1, %0;" ::"n"(kCons * 32) : "memory");
    if (ctid == 0) {
      const unsigned old = atomicAdd(P.tickets + tile, 1u);
      s_last = (old == (unsigned)(P.ksplit - 1));
      if (s_last) P.tickets[tile] = 0u;  // ready for the next launch / graph replay
    }
    asm volatile("bar.sync 1, %0;" ::"n"(kCons * 32) : "memory");
    if (!s_last) return;
    __threadfence();
    for (int idx = ctid; idx < MT * BN / 4; idx += kCons * 32) {
      float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int sp = 0; sp < P.ksplit; ++sp) {  // fixed order: the result does not depend on which CTA came last
        const float4* src = reinterpret_cast<const float4*>(P.partial + ((size_t)sp * P.tiles + tile) * (MT * BN)) + idx;
        float4 v;
        asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(src));
        sum.x += v.x;
        sum.y += v.y;
        sum.z += v.z;
        sum.w += v.w;
      }
      reinterpret_cast<float4*>(tb_s)[idx] = sum;
    }
    asm volatile("bar.sync 1, %0;" ::"n"(kCons * 32) : "memory");
  }
  if (gate_up) {
    constexpr int H = BN / 2;
    for (int idx = ctid; idx < MT * H; idx += kCons * 32) {
      const int m = idx / H, r = idx - m * H;
      const int row = r0 + r;
      if (m < P.m && row < P.n[0]) {
        const float gt = tb_s[m * BN + r], up = tb_s[m * BN + H + r];
        const float sg = P.eltop == NS_ELT_GELU ? ns_gelu(gt) : ns_silu(gt);
        P.dst[(size_t)m * P.ldo + row] = sg * up;
      }
    }
  } else {
    for (int idx = ctid; idx < MT * BN; idx += kCons * 32) {
      const int m = idx / BN, r = idx - m * BN;
      const int row = r0 + r;
      if (m < P.m && row < P.n[wi]) {
        const long long out = P.dst_off[wi] + row;
        const size_t o = (size_t)m * P.ldo + out;
        float v = tb_s[idx];
        if (P.bias) v += P.bias_bcast ? P.bias[out] : P.bias[o];
        if (P.eltop == NS_ELT_GELU) v = ns_gelu(v);
        if (P.residual) v += P.residual[o];
        P.dst[o] = v;
      }
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

constexpr int kMaxPartialTiles = 640;  // tiles x ksplit when K is split
constexpr int kMaxTiles = 16384;

struct Plan {
  int mt, tiles, ksplit, nslices, stages, sc_row, sc_zp;
  size_t smem, img_bytes, partial_bytes, ticket_bytes;
};

int mt_of(int m) { return m <= 8 ? 8 : (m <= 16 ? 16 : 32); }

bool make_plan(const ns_weight* const* ws, int nw, int mode, int m, Plan* pl) {
  const ns_weight* w0 = ws[0];
  pl->mt = mt_of(m);
  pl->nslices = (w0->kpad + KS - 1) / KS;
  int tiles = 0;
  if (mode == NS_GEMV_GATE_UP_SILU) {
    tiles = (w0->n + BN / 2 - 1) / (BN / 2);
  } else {
    for (int i = 0; i < nw; ++i) tiles += (ws[i]->n + BN - 1) / BN;
  }
  pl->tiles = tiles;
  if (tiles > kMaxTiles) return false;
  const int ss = ns_stype_size(w0->stype);
  const int cpg = w0->group / 32;
  const int kact = pl->mt * 320;
  const int kstage = kQStage + (kact + 1023) / 1024 * 1024;
  // split K.  Two CTAs share an SM (16 consumer warps hide the MMA / shared-memory latencies; one CTA's prologue overlaps the
  // other's main loop), so a wave has 2 x SMs slots and a CTA gets half an SM's bandwidth: cost of a choice = waves x (2 x slices
  // per CTA + ramp).  The staged scales must fit beside a ring of >= 3 stages in half an SM's shared memory.
  static const int env_split = getenv("NS_IMMA_KSPLIT") ? atoi(getenv("NS_IMMA_KSPLIT")) : 0;
  static const int env_budget = getenv("NS_IMMA_SMEM_KB") ? atoi(getenv("NS_IMMA_SMEM_KB")) : 0;
  const int sms = ns_num_sms();
  const size_t budget = (size_t)(env_budget > 0 ? env_budget : 111) * 1024;
  const int per_sm = budget > 112 * 1024 ? 1 : 2;
  int ksplit = 0;
  long best = -1;
  for (int ks = 1; ks <= 16 && ks <= pl->nslices; ++ks) {
    if (env_split > 0 && ks != env_split && env_split <= pl->nslices) continue;
    if (ks > 1 && tiles * ks > kMaxPartialTiles) continue;
    const int max_sl = (pl->nslices + ks - 1) / ks;
    const int ng = ((max_sl + 1) * 8 + cpg - 1) / cpg + 1;
    const int sc_zp = (int)ns_round_up((size_t)15 + (size_t)ss * ng, 16);
    const int sc_row = sc_zp + (w0->asym ? (int)ns_round_up((size_t)15 + ng, 16) : 0);
    const size_t fixed = (size_t)BN * sc_row + 16 * 16 + 64 + 1024;
    const int need = max_sl < 3 ? max_sl : 3;
    if (fixed + (size_t)need * kstage > budget) continue;
    const long waves = ((long)tiles * ks + per_sm * sms - 1) / (per_sm * sms);
    const long cost = waves * (per_sm * max_sl + 2) * 16 + ks;  // ties: fewer splits
    if (best < 0 || cost < best) {
      best = cost;
      ksplit = ks;
      int stages = (int)((budget - fixed) / kstage);
      if (stages > 16) stages = 16;
      if (stages > max_sl) stages = max_sl;
      pl->stages = stages;
      pl->sc_row = sc_row;
      pl->sc_zp = sc_zp;
      pl->smem = (size_t)stages * kstage + (size_t)BN * sc_row + 16 * (size_t)stages + 64 + 1024;
    }
  }
  if (!ksplit) return false;
  pl->ksplit = ksplit;
  pl->img_bytes = ns_round_up((size_t)pl->nslices * kact, 256);
  pl->partial_bytes = ksplit > 1 ? ns_round_up((size_t)ksplit * tiles * pl->mt * BN * sizeof(float), 256) : 0;
  pl->ticket_bytes = ns_round_up((size_t)tiles * sizeof(unsigned), 256);
  return true;
}

template <bool ACT_U8, int MT, bool ASYM, int STYPE, int PER>
int launch_p(const CUtensorMap* maps, const ImmaParams& P, const Plan& pl, cudaStream_t st) {
  auto kern = gemm_imma_kernel<ACT_U8, MT, ASYM, STYPE, PER>;
  static bool attr = false;
  if (!attr) {
    NS_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
    attr = true;
  }
  NS_CUDA_TRY(ns_launch_pdl(kern, dim3((unsigned)(pl.tiles * pl.ksplit)), dim3(kThr), pl.smem, st, maps[0], maps[1], maps[2], P));
  ns_count_launch();
  return NS_OK;
}
template <bool ACT_U8, int MT, bool ASYM, int STYPE>
int launch_k(const CUtensorMap* maps, const ImmaParams& P, const Plan& pl, cudaStream_t st) {
  if (P.acpg == 1 && P.cpg == 1) return launch_p<ACT_U8, MT, ASYM, STYPE, 1>(maps, P, pl, st);
  if (P.acpg == 4 && P.cpg == 4) return launch_p<ACT_U8, MT, ASYM, STYPE, 4>(maps, P, pl, st);
  return launch_p<ACT_U8, MT, ASYM, STYPE, 0>(maps, P, pl, st);
}
template <bool ACT_U8, int MT, bool ASYM>
int launch_s(const CUtensorMap* maps, const ImmaParams& P, const Plan& pl, int stype, cudaStream_t st) {
  switch (stype) {
    case NS_S_F32: return launch_k<ACT_U8, MT, ASYM, NS_S_F32>(maps, P, pl, st);
    case NS_S_F16: return launch_k<ACT_U8, MT, ASYM, NS_S_F16>(maps, P, pl, st);
    default: return launch_k<ACT_U8, MT, ASYM, NS_S_BF16>(maps, P, pl, st);
  }
}
template <bool ACT_U8, bool ASYM>
int launch_m(const CUtensorMap* maps, const ImmaParams& P, const Plan& pl, int stype, cudaStream_t st) {
  switch (pl.mt) {
    case 8: return launch_s<ACT_U8, 8, ASYM>(maps, P, pl, stype, st);
    case 16: return launch_s<ACT_U8, 16, ASYM>(maps, P, pl, stype, st);
    default: return launch_s<ACT_U8, 32, ASYM>(maps, P, pl, stype, st);
  }
}

}  // namespace

// Can this (fused) matmul of m activation rows run on the integer tensor cores?
bool ns_gemm_imma_supported(const ns_weight* const* ws, int nw, int m) {
  static const bool off = getenv("NS_NO_IMMA") != nullptr;
  static const int min_m = getenv("NS_IMMA_MIN_M") ? atoi(getenv("NS_IMMA_MIN_M")) : 3;  // measured: the 4-row GEMV tile is slower already
  if (off || m < min_m || m > 32 || nw < 1 || nw > 3) return false;
  const ns_weight* w0 = ws[0];
  for (int i = 0; i < nw; ++i) {
    const ns_weight* w = ws[i];
    if (!w || w->wfmt != NS_W_S4 || w->shuffle) return false;
    if (w->k != w0->k || w->group != w0->group || w->stype != w0->stype || w->comp != w0->comp || w->asym != w0->asym) return false;
  }
  if (!(w0->comp == NS_COMP_Q8_0 || w0->comp == NS_COMP_INT8 || w0->comp == NS_COMP_INT8_S8)) return false;
  if (!(w0->group == 32 || w0->group == 64 || w0->group == 128 || w0->group == 256) || w0->k % w0->group) return false;
  if (w0->k % KS) return false;  // whole 256-k stages only (every model width is): no per-chunk tail checks in the loop
  if (w0->pitch % 16) return false;
  return true;
}

// Workspace = activation image + split-K partial tiles + tickets.  The planner keeps tiles x ksplit <= kMaxPartialTiles when it
// splits and refuses more than kMaxTiles row tiles, so the bound depends on (m, k) only.
size_t ns_gemm_imma_workspace_bound(int m, int kpad) {
  const int mt = mt_of(m);
  const size_t img = ns_round_up((size_t)((kpad + KS - 1) / KS) * mt * 320, 256);
  return img + (size_t)kMaxPartialTiles * mt * BN * sizeof(float) + (size_t)kMaxTiles * sizeof(unsigned) + 512;
}

// act: fp32 [m][lda] (device).  dst layout and epilogue arguments as ns_launch_gemv.
int ns_launch_gemm_imma(const ns_weight* const* ws, int nw, int mode, const float* act, int lda, float* dst, int ldo, int m,
                        const float* bias, int bias_bcast, const float* residual, int eltop, void* workspace, cudaStream_t st) {
  if (!ns_gemm_imma_supported(ws, nw, m)) {
    ns_set_error("integer tensor-core matmul: unsupported weight format or row count %d", m);
    return NS_E_UNSUPPORTED;
  }
  if (mode == NS_GEMV_GATE_UP_SILU && (nw != 2 || ws[0]->n != ws[1]->n)) {
    ns_set_error("gate/up fusion needs two weights with equal n");
    return NS_E_INVALID;
  }
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    ns_set_error("cuTensorMapEncodeTiled not available from the driver");
    return NS_E_CUDA;
  }
  const ns_weight* w0 = ws[0];
  Plan pl;
  if (!make_plan(ws, nw, mode, m, &pl)) {
    ns_set_error("integer tensor-core matmul: no shared-memory plan for k=%d group=%d", w0->k, w0->group);
    return NS_E_UNSUPPORTED;
  }
  uint8_t* img = (uint8_t*)workspace;
  float* partial = (float*)(img + pl.img_bytes);
  unsigned* tickets = (unsigned*)(img + pl.img_bytes + pl.partial_bytes);

  // 1. activation image (+ ticket reset)
  {
    const int qg = w0->comp == NS_COMP_Q8_0 ? 32 : w0->group;
    const int nblk = pl.nslices * 8 / (qg / 32);
    const int warps = pl.mt * nblk;
    const dim3 grid((unsigned)((warps + 7) / 8)), block(256);
    cudaError_t e;
    if (w0->comp == NS_COMP_Q8_0)
      e = ns_launch_pdl(act_quant_imma_kernel<NS_COMP_Q8_0>, grid, block, 0, st, act, lda, m, w0->k, qg, pl.mt, pl.nslices, img, tickets, pl.tiles);
    else if (w0->comp == NS_COMP_INT8)
      e = ns_launch_pdl(act_quant_imma_kernel<NS_COMP_INT8>, grid, block, 0, st, act, lda, m, w0->k, qg, pl.mt, pl.nslices, img, tickets, pl.tiles);
    else
      e = ns_launch_pdl(act_quant_imma_kernel<NS_COMP_INT8_S8>, grid, block, 0, st, act, lda, m, w0->k, qg, pl.mt, pl.nslices, img, tickets,
                        pl.tiles);
    NS_CUDA_TRY(e);
    ns_count_launch();
  }

  // 2. tensor maps over the nibble part of each weight: uint8 [n][q_bytes], row pitch `pitch`; box = 128 B x rows, 128B swizzle
  CUtensorMap maps[3];
  const bool gate_up = mode == NS_GEMV_GATE_UP_SILU;
  for (int i = 0; i < 3; ++i) {
    const ns_weight* w = ws[i < nw ? i : 0];
    cuuint64_t dims[2] = {(cuuint64_t)w->q_bytes, (cuuint64_t)w->n};
    cuuint64_t strides[1] = {(cuuint64_t)w->pitch};
    cuuint32_t box[2] = {(cuuint32_t)(KS / 2), (cuuint32_t)(gate_up ? BN / 2 : BN)};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(&maps[i], CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, (void*)w->rows, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      ns_set_error("cuTensorMapEncodeTiled(weights) failed: %d", (int)r);
      return NS_E_CUDA;
    }
  }

  ImmaParams P = {};
  int t0 = 0;
  for (int i = 0; i < nw; ++i) {
    P.rows[i] = ws[i]->rows;
    P.n[i] = ws[i]->n;
    P.dst_off[i] = (mode == NS_GEMV_CONCAT) ? (long long)i * m * ldo : 0;
    P.tile0[i] = t0;
    t0 += (ws[i]->n + BN - 1) / BN;
  }
  P.nw = nw;
  P.mode = mode;
  P.k = w0->k;
  P.group = w0->group;
  P.cpg = w0->group / 32;
  P.acpg = w0->comp == NS_COMP_Q8_0 ? 1 : P.cpg;
  P.cpg_shift = P.cpg == 1 ? 0 : (P.cpg == 2 ? 1 : (P.cpg == 4 ? 2 : 3));
  P.pitch = w0->pitch;
  P.sc_off = w0->sc_off;
  P.zp_off = w0->zp_off;
  P.act_img = img;
  P.dst = dst;
  P.ldo = ldo;
  P.m = m;
  P.bias = bias;
  P.bias_bcast = bias_bcast;
  P.residual = residual;
  P.eltop = eltop;
  P.tiles = pl.tiles;
  P.ksplit = pl.ksplit;
  P.nslices = pl.nslices;
  P.partial = partial;
  P.tickets = tickets;
  P.sc_row = pl.sc_row;
  P.sc_zp = pl.sc_zp;
  P.stages = pl.stages;
  static const bool dbg = getenv("NS_IMMA_DEBUG") != nullptr;
  if (dbg)
    fprintf(stderr, "gemm_imma: m=%d mt=%d k=%d g=%d tiles=%d ksplit=%d stages=%d smem=%zu sc_row=%d\n", m, pl.mt, w0->k, w0->group, pl.tiles,
            pl.ksplit, pl.stages, pl.smem, pl.sc_row);
  const bool asym = w0->asym != 0;
  if (w0->comp == NS_COMP_INT8)
    return asym ? launch_m<true, true>(maps, P, pl, w0->stype, st) : launch_m<true, false>(maps, P, pl, w0->stype, st);
  return asym ? launch_m<false, true>(maps, P, pl, w0->stype, st) : launch_m<false, false>(maps, P, pl, w0->stype, st);
}

// gemv_ring_impl.cuh -- the ring GEMV kernel template, its activation prologue and launcher (the plan: ns_gemv_ring_choose).  Included by gemv_ring.cu (two CTAs
// per SM, 7 consumer warps) and gemv_ring_wide.cu (one CTA per SM, 14 consumer warps): two translation units so that the ~170
// instantiations compile in parallel.  See gemv_ring.cu for the design notes.
#pragma once
#include "act_quant.cuh"
#include "async_copy.cuh"

namespace {

constexpr int kConsumers = 7;
constexpr int kThreads = (kConsumers + 1) * 32;

__device__ __forceinline__ uint32_t lds32(uint32_t a) {
  uint32_t r;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(a));
  return r;
}
__device__ __forceinline__ uint32_t lds16(uint32_t a) {
  unsigned short r;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(r) : "r"(a));
  return r;
}
__device__ __forceinline__ int lds8s(uint32_t a) {
  int r;
  asm volatile("ld.shared.s8 %0, [%1];" : "=r"(r) : "r"(a));
  return r;
}
template <int STYPE>
__device__ __forceinline__ float lds_scale(uint32_t base, int idx) {
  if (STYPE == NS_S_F32) return __uint_as_float(lds32(base + 4 * idx));
  if (STYPE == NS_S_F16) return __half2float(__ushort_as_half((unsigned short)lds16(base + 2 * idx)));
  return __uint_as_float(lds16(base + 2 * idx) << 16);
}

// ---- activation prologue: fp32 rows -> the int8 ring image in shared memory (the fused NE_TASK_INIT) ----------------------
// Codes, scales and zero points are act_quant.cuh's, bit-exact.  NORM (the fused-RMSNorm kernels): rows are normalised first
// when norm_w is set -- ne_rms_norm + ne_mul (models/llama/llama.cpp:205-210) with the arithmetic of rmsnorm_kernel (llama.cu,
// kernel_ref.h:2199-2225): y = x * (1 / sqrt(sum(x^2)/n + eps)) * w.
struct QuantIn {
  const float* in;      // [M][lda] fp32, global (read through L2: another SM may have just written it)
  const float* norm_w;  // NORM: [k] RMSNorm weight, or NULL: no normalisation
  float eps;
  int lda, k, kpad, group;             // group: the activation block (32 for Q8_0)
  int act_row, meta_off, meta_stride;  // image geometry (bytes, bytes, int2 units)
};

__device__ __forceinline__ void sts64(uint32_t a, uint32_t x, uint32_t y) {
  asm volatile("st.shared.v2.u32 [%0], {%1,%2};" ::"r"(a), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ float4 ldcg4(const float* p) {
  float4 r;
  asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ float ldcg1(const float* p) {
  float r;
  asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}
template <int BAR, int NT>
__device__ __forceinline__ void bar_sync() {
  asm volatile("bar.sync %0, %1;" ::"n"(BAR), "n"(NT) : "memory");
}

// The RMSNorm weights of the 8-groups thread `tid` owns in a single-pass row (kpad / 8 <= 3 * NT).  They are constants of the model:
// the caller fetches them BEFORE griddepcontrol.wait, so the L2 broadcast of the weight vector to every CTA overlaps the previous
// launch's tail instead of sitting between the wait and the first dp4a.
template <int NT>
__device__ __forceinline__ void prefetch_norm_w(const float* __restrict__ norm_w, int k, int kpad, int tid, float (&gw)[3][8]) {
  const int ngroups8 = kpad >> 3;
#pragma unroll
  for (int it = 0; it < 3; ++it) {
    const int e = it * NT + tid, k0 = e * 8;
    if (e < ngroups8 && k0 + 8 <= k) {
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(norm_w + k0)), w1 = __ldg(reinterpret_cast<const float4*>(norm_w + k0 + 4));
      gw[it][0] = w0.x; gw[it][1] = w0.y; gw[it][2] = w0.z; gw[it][3] = w0.w;
      gw[it][4] = w1.x; gw[it][5] = w1.y; gw[it][6] = w1.z; gw[it][7] = w1.w;
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) gw[it][i] = (e < ngroups8 && k0 + i < k) ? __ldg(norm_w + k0 + i) : 0.f;
    }
  }
}

// the fp32 activations of NI passes of NT threads from pass eb on, 8 per thread, zero past K (the loads are issued back to
// back: L2 latency ~0.5 us each would otherwise serialise)
template <int NI, int NT>
__device__ __forceinline__ void load_passes(const float* row, int eb, int tid, int ngroups8, int k, float (&vv)[NI][8]) {
#pragma unroll
  for (int it = 0; it < NI; ++it) {
    const int e = eb + it * NT + tid;
    const int k0 = e * 8;
    if (e < ngroups8 && k0 + 8 <= k) {
      const float4 x0 = ldcg4(row + k0), x1 = ldcg4(row + k0 + 4);
      vv[it][0] = x0.x; vv[it][1] = x0.y; vv[it][2] = x0.z; vv[it][3] = x0.w;
      vv[it][4] = x1.x; vv[it][5] = x1.y; vv[it][6] = x1.z; vv[it][7] = x1.w;
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) vv[it][i] = (e < ngroups8 && k0 + i < k) ? ldcg1(row + k0 + i) : 0.f;
    }
  }
}

// Called by the NT consumer threads (whole warps, named barrier 1).  A thread owns one 8-group (8 consecutive k); group/8
// consecutive threads own one quantisation block.  NORM: red is shared float[NT/32], gw prefetch_norm_w's registers or NULL.
// NAT: the codes keep natural order inside their chunk (8-bit weights, act_prep.cu's perm8 = 0), else the NSB4 pairing order.
template <int COMP, int NT, bool NORM, bool NAT = false>
__device__ __forceinline__ void quantise_to_smem(const QuantIn& P, int M, uint32_t smem_base, float* red, const float (*gw)[8]) {
  constexpr int NI = 3;  // load passes kept in registers (3 x 512 threads x 8 = 12288 elements)
  const int tpb = (COMP == NS_COMP_Q8_0 ? 32 : P.group) >> 3;  // threads per quantisation block (4..32, power of two)
  const int ngroups8 = P.kpad >> 3;
  const int tid = threadIdx.x;
  const bool single = ngroups8 <= NI * NT;
  const bool norm = NORM && P.norm_w != nullptr;
  for (int m = 0; m < M; ++m) {
    const float* row = P.in + (size_t)m * P.lda;
    const uint32_t img = smem_base + (uint32_t)m * P.act_row;
    const uint32_t meta = smem_base + P.meta_off + 8u * (uint32_t)(m * P.meta_stride);
    float vv[NI][8];
    auto sum_sq = [&](float ss) {
#pragma unroll
      for (int it = 0; it < NI; ++it)
#pragma unroll
        for (int i = 0; i < 8; ++i) ss = fmaf(vv[it][i], vv[it][i], ss);
      return ss;
    };
    if (NORM && single) load_passes<NI, NT>(row, 0, tid, ngroups8, P.k, vv);  // a single-pass row stays in registers from the sum of squares to the quantiser
    float inv = 1.f;
    if (norm) {
      float ss = 0.f;
      if (single) {
        ss = sum_sq(ss);
      } else {
        for (int eb = 0; eb < ngroups8; eb += NI * NT) {
          load_passes<NI, NT>(row, eb, tid, ngroups8, P.k, vv);
          ss = sum_sq(ss);
        }
      }
      ss = warp_sum(ss);
      bar_sync<1, NT>();  // red[] free (previous row / previous use)
      if ((tid & 31) == 0) red[tid >> 5] = ss;
      bar_sync<1, NT>();
      float tot = 0.f;
#pragma unroll
      for (int i = 0; i < NT / 32; ++i) tot += red[i];
      inv = 1.f / sqrtf(tot / (float)P.k + P.eps);
    }
    for (int eb = 0; eb < ngroups8; eb += NI * NT) {
      if (!(NORM && single)) load_passes<NI, NT>(row, eb, tid, ngroups8, P.k, vv);
#pragma unroll
      for (int it = 0; it < NI; ++it) {
        const int e0 = eb + it * NT;
        if (e0 >= ngroups8) break;  // uniform across the CTA
        const int e = e0 + tid;
        const bool live = e < ngroups8;
        const int k0 = e * 8;
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = vv[it][i];
        if (norm && gw != nullptr && single) {
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = v[i] * inv * gw[it][i];  // (padding lanes: gw = 0, v = 0)
        } else if (norm) {
          if (live && k0 + 8 <= P.k) {
            const float4 w0 = __ldg((const float4*)(P.norm_w + k0)), w1 = __ldg((const float4*)(P.norm_w + k0 + 4));
            v[0] = v[0] * inv * w0.x; v[1] = v[1] * inv * w0.y; v[2] = v[2] * inv * w0.z; v[3] = v[3] * inv * w0.w;
            v[4] = v[4] * inv * w1.x; v[5] = v[5] * inv * w1.y; v[6] = v[6] * inv * w1.z; v[7] = v[7] * inv * w1.w;
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = (live && k0 + i < P.k) ? v[i] * inv * __ldg(P.norm_w + k0 + i) : 0.f;
          }
        }
        // block range (all lanes of the warp take part in the shuffles); a block ends past K only for a partial last block
        float vmax = nsq::range_start<COMP>((k0 | (tpb * 8 - 1)) >= P.k), vmin = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) nsq::range_fold<COMP>(v[i], vmax, vmin);
        nsq::range_reduce<COMP>(vmax, vmin, tpb);
        const nsq::BlockQuant bq = nsq::block_quant<COMP>(vmax, vmin);
        int q[8], sa = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          q[i] = k0 + i < P.k ? nsq::quant_code<COMP>(v[i], bq) : bq.za;
          sa += q[i];
        }
        // chunk sum over the 4 threads of a 32-element chunk
        sa += __shfl_xor_sync(0xffffffffu, sa, 1);
        sa += __shfl_xor_sync(0xffffffffu, sa, 2);
        if (live) {
          uint32_t w[2] = {0u, 0u};
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int pos = NAT ? i : nsq::dp4a_pos(i);
            w[pos >> 2] |= (uint32_t)(q[i] & 0xff) << (8 * (pos & 3));
          }
          const int c = e >> 2, i = e & 3;
          sts64(img + nsq::ring_offset((uint32_t)c, (uint32_t)i * 8u), w[0], w[1]);
          if (i == 0) {
            const int2 mw = nsq::meta_word(bq.scale, sa, bq.za);
            sts64(meta + 8u * (uint32_t)c, (uint32_t)mw.x, (uint32_t)mw.y);
          }
        }
      }
    }
  }
}

struct PairSrc {
  const uint8_t* r0;
  const uint8_t* r1;
  long long out0, out1;
  bool valid1;
};

__device__ __forceinline__ PairSrc resolve_pair(const GemvParams& P, int p) {
  PairSrc s;
  if (P.mode == NS_GEMV_GATE_UP_SILU) {
    s.r0 = P.rows[0] + (size_t)p * P.pitch;
    s.r1 = P.rows[1] + (size_t)p * P.pitch;
    s.out0 = s.out1 = p;
    s.valid1 = true;
    return s;
  }
  int row = 2 * p, wi = 0;
  if (P.nw > 1 && row >= P.n[0]) {
    row -= P.n[0];
    wi = 1;
    if (P.nw > 2 && row >= P.n[1]) {
      row -= P.n[1];
      wi = 2;
    }
  }
  // every weight but the last has an even n (checked by the launcher), so a pair never straddles two weights
  s.valid1 = row + 1 < P.n[wi];
  s.r0 = P.rows[wi] + (size_t)row * P.pitch;
  s.r1 = s.valid1 ? s.r0 + P.pitch : s.r0;
  s.out0 = P.dst_off[wi] + row;
  s.out1 = s.out0 + 1;
  return s;
}

struct RingCfg {
  int ring_off;     // byte offset of the ring inside dynamic shared memory
  int stages;
  int units;        // row pairs (ROWS == 2) or rows (ROWS == 1) of this launch
  int active;       // consumer warps that own ring stages (<= kConsumers; `stages` is a multiple of it)
  int act_row;      // bytes per activation row in the staged image
  int red_off;      // byte offset of the RMSNorm reduction scratch (8 floats) inside the activation region, fused-norm launches only
  uint32_t cpg_magic;  // ceil(2^32 / cpg): gi = umulhi(c, magic)
};

// ROWS == 1: unit u is row u of the concatenated weights (long rows: a pair would leave one ring stage per consumer warp)
__device__ __forceinline__ PairSrc resolve_single(const GemvParams& P, int u) {
  PairSrc s;
  int row = u, wi = 0;
  if (P.nw > 1 && row >= P.n[0]) {
    row -= P.n[0];
    wi = 1;
    if (P.nw > 2 && row >= P.n[1]) {
      row -= P.n[1];
      wi = 2;
    }
  }
  s.r0 = s.r1 = P.rows[wi] + (size_t)row * P.pitch;
  s.out0 = s.out1 = P.dst_off[wi] + row;
  s.valid1 = false;
  return s;
}

// The consumer loop over one ring stage for 8-bit codes (ggml Q8_0: symmetric, one fp16 scale per 32-chunk).  A chunk is 32
// natural-order code bytes against the natural-order activation image (bytes 0..15 at nsq::ring_offset(c, 0), 16..31 at + 512),
// so isum_c = sum a*q is one chain of eight s8 x s8 dp4a -- no nibble expansion, no offset term -- and the accumulation is the
// 4-bit path's: acc = fmaf(isum_c, fp32(a_scale * w_scale), acc) over c = lane, lane + 32, ...
template <int M, int ROWS, int STYPE>
__device__ __forceinline__ void ring_chunks_w8(const GemvParams& P, const RingCfg& R, const uint32_t (&rb)[2], uint32_t smem_base,
                                               uint32_t meta_s, int nchunks, int lane, float (&acc)[ROWS][M]) {
#pragma unroll 2
  for (int c = lane; c < nchunks; c += 32) {
    uint4 wl[ROWS], wh[ROWS];
    float ws[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      wl[r] = lds128(rb[r] + 32 * c);
      wh[r] = lds128(rb[r] + 32 * c + 16);
      ws[r] = lds_scale<STYPE>(rb[r] + P.sc_off, c);
    }
    const uint32_t a_off = (uint32_t)(c >> 5) * 1024u + (uint32_t)(c & 31) * 16u;
#pragma unroll
    for (int m = 0; m < M; ++m) {
      const uint32_t ab = smem_base + (uint32_t)m * R.act_row + a_off;
      const uint4 a0 = lds128(ab), a1 = lds128(ab + 512);
      const float a_scale = __uint_as_float(lds64(meta_s + 8u * (uint32_t)(m * P.meta_stride + c)).x);
#pragma unroll
      for (int r = 0; r < ROWS; ++r) {
        int isum = dp4a_ss((int)wl[r].x, (int)a0.x, 0);
        isum = dp4a_ss((int)wl[r].y, (int)a0.y, isum);
        isum = dp4a_ss((int)wl[r].z, (int)a0.z, isum);
        isum = dp4a_ss((int)wl[r].w, (int)a0.w, isum);
        isum = dp4a_ss((int)wh[r].x, (int)a1.x, isum);
        isum = dp4a_ss((int)wh[r].y, (int)a1.y, isum);
        isum = dp4a_ss((int)wh[r].z, (int)a1.z, isum);
        isum = dp4a_ss((int)wh[r].w, (int)a1.w, isum);
        acc[r][m] = fmaf((float)isum, a_scale * ws[r], acc[r][m]);  // |isum| <= 32 * 128 * 127: exact in fp32
      }
    }
  }
}

// NORM: the fused-RMSNorm prologue is a separate instantiation, so the plain kernels (the headline path) keep the code and the
// register allocation they had without it
// NC consumer warps: 7 (+1 producer warp, two CTAs per SM) or 14 (+2 producer warps, ONE CTA per SM: the activation row is pulled
// through L2 and quantised once per SM instead of twice -- the 16-44 KB broadcast to every CTA is what separates the fused launch
// list from the pre-quantised one; the two producer warps take alternate ring stages)
// W8: 8-bit codes (ggml Q8_0; instantiated with A_S8, symmetric, fp16 scales only), ring_chunks_w8 instead of the nibble loop
template <int AMODE, int M, bool ASYM, int STYPE, int ROWS, bool NORM, int NC, bool W8 = false>
__global__ void __launch_bounds__((NC + (NC > kConsumers ? 2 : 1)) * 32, NC > kConsumers ? 1 : 2)
    gemv_ring_kernel(const GemvParams P, const RingCfg R) {
  constexpr int NP = NC > kConsumers ? 2 : 1;  // producer warps
  extern __shared__ __align__(128) unsigned char smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int stage_bytes = ROWS * P.pitch;
  const int stages = R.stages;
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t ring = smem_base + R.ring_off;
  const uint32_t full0 = ring + (uint32_t)stages * stage_bytes;
  const uint32_t empty0 = full0 + 8u * stages;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int first = blockIdx.x;
  const int gstride = (int)gridDim.x;
  const int my_units = first < R.units ? (R.units - first + gstride - 1) / gstride : 0;

  if (warp >= NC) {
    // ===================== producer(s): stream whole row pairs, never touch activations =====================
    // producer warp pw takes units pw, pw + NP, ...; unit j always lands in stage j % stages (`stages` is a multiple of NC: even)
    if (lane == 0) {
      int s = warp - NC;
      uint32_t phase = 0;
      for (int j = warp - NC; j < my_units; j += NP) {
        if (j >= stages) mbar_wait(empty0 + 8 * s, phase ^ 1);
        const PairSrc ps = ROWS == 2 ? resolve_pair(P, first + j * gstride) : resolve_single(P, first + j * gstride);
        const uint32_t dst = ring + (uint32_t)s * stage_bytes;
        mbar_expect_tx(full0 + 8 * s, (uint32_t)stage_bytes);
        bulk_g2s(dst, ps.r0, (uint32_t)P.pitch, full0 + 8 * s);
        if (ROWS == 2) bulk_g2s(dst + P.pitch, ps.r1, (uint32_t)P.pitch, full0 + 8 * s);
        s += NP;
        if (s >= stages) {
          s -= stages;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // ===================== consumers =====================
  // fused RMSNorm: the norm weights are model constants -- fetch this thread's share before the wait (single-pass rows)
  float gw[NORM ? 3 : 1][8];
  bool gw_pref = false;
  if constexpr (NORM) {
    gw_pref = P.norm_w != nullptr && (P.kpad >> 3) <= 3 * NC * 32;
    if (gw_pref) prefetch_norm_w<NC * 32>(P.norm_w, P.k, P.kpad, (int)threadIdx.x, gw);
  }
  pdl_wait();  // activations (and residual) come from earlier kernels
  if (P.act_f32) {
    // fused NE_TASK_INIT: quantise the fp32 rows straight into the shared-memory image (no separate kernel, no round trip).
    // NORM with norm_w set: fused ne_rms_norm + ne_mul -- every CTA already reads the whole fp32 row, the sum of squares costs one
    // more block reduction instead of a kernel boundary (a norm-capable image also serves plain nodes: see GemvParams::one_image)
    const QuantIn qi{P.act_f32, NORM ? P.norm_w : nullptr, P.norm_eps, P.lda, P.k, P.kpad, P.comp == NS_COMP_Q8_0 ? 32 : P.group,
                     R.act_row, P.meta_off, P.meta_stride};
    float* red = reinterpret_cast<float*>(smem + R.red_off);
    const float(*gwp)[8] = gw_pref ? gw : nullptr;
    if constexpr (W8) {
      quantise_to_smem<NS_COMP_Q8_0, NC * 32, NORM, true>(qi, P.m, smem_base, red, gwp);
    } else {
      if (AMODE == A_U8) quantise_to_smem<NS_COMP_INT8, NC * 32, NORM>(qi, P.m, smem_base, red, gwp);
      else if (P.comp == NS_COMP_Q8_0) quantise_to_smem<NS_COMP_Q8_0, NC * 32, NORM>(qi, P.m, smem_base, red, gwp);
      else quantise_to_smem<NS_COMP_INT8_S8, NC * 32, NORM>(qi, P.m, smem_base, red, gwp);
    }
  } else {
    const uint4* src = reinterpret_cast<const uint4*>(P.act);
    uint4* dstv = reinterpret_cast<uint4*>(smem);
    const int nvec = P.act_bytes >> 4;
    for (int i = threadIdx.x; i < nvec; i += NC * 32) dstv[i] = src[i];
  }
  asm volatile("bar.sync 1, %0;" ::"n"(NC * 32) : "memory");
  const uint32_t meta_s = smem_base + P.meta_off;
  const int nchunks = P.kpad >> 5;

  // This warp visits units warp, warp+active, ... .  `stages` is a multiple of `active` (launcher), so stage s is only ever
  // consumed by warp s % active: every mbarrier is waited on by ONE warp that observes all of its phases in order (mbar_wait).
  int s = warp;
  uint32_t phase = 0;

  const int active = R.active;  // long rows leave room for fewer stages than consumer warps: the surplus warps only helped quantise
  if (warp >= active) return;
  for (int j = warp; j < my_units; j += active) {
    const PairSrc ps = ROWS == 2 ? resolve_pair(P, first + j * gstride) : resolve_single(P, first + j * gstride);
    mbar_wait(full0 + 8 * s, phase);
    const uint32_t r0 = ring + (uint32_t)s * stage_bytes;
    const uint32_t r1 = ROWS == 2 ? r0 + P.pitch : r0;
    const uint32_t rb[2] = {r0, r1};

    float acc[ROWS][M];
#pragma unroll
    for (int r = 0; r < ROWS; ++r)
#pragma unroll
      for (int m = 0; m < M; ++m) acc[r][m] = 0.f;

    if constexpr (W8) {
      ring_chunks_w8<M, ROWS, STYPE>(P, R, rb, smem_base, meta_s, nchunks, lane, acc);
    } else {
#pragma unroll 2
      for (int c = lane; c < nchunks; c += 32) {
        const int gi = (P.cpg == 1) ? c : (int)__umulhi((uint32_t)c, R.cpg_magic);
        uint4 wv[ROWS];
        float ws[ROWS];
        int off[ROWS];
#pragma unroll
        for (int r = 0; r < ROWS; ++r) {
          wv[r] = lds128(rb[r] + 16 * c);
          ws[r] = lds_scale<STYPE>(rb[r] + P.sc_off, gi);
          off[r] = 8;
          if (ASYM) off[r] += lds8s(rb[r] + P.zp_off + gi);
        }
        // low nibbles as bytes, high nibbles as bytes * 16 (no shift): exact, divided out after the dot
        uint32_t lo[ROWS][4], hi[ROWS][4];
        int su[ROWS];
#pragma unroll
        for (int r = 0; r < ROWS; ++r) {
          su[r] = 0;
          const uint32_t ww[4] = {wv[r].x, wv[r].y, wv[r].z, wv[r].w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            lo[r][i] = ww[i] & 0x0F0F0F0Fu;
            hi[r][i] = ww[i] & 0xF0F0F0F0u;
          }
          if (AMODE == A_U8) {  // sum of the weight codes, needed for the activation zero point
            int sl = 0, sh = 0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              sl = dp4a_uu(lo[r][i], 0x01010101u, sl);
              sh = dp4a_uu(hi[r][i], 0x01010101u, sh);
            }
            su[r] = sl + (sh >> 4);
          }
        }
        // activation image: bytes 0..15 and 16..31 of chunk c at nsq::ring_offset(c, 0) and + 512 (act_quant.cuh)
        const uint32_t a_off = (uint32_t)(c >> 5) * 1024u + (uint32_t)(c & 31) * 16u;
#pragma unroll
        for (int m = 0; m < M; ++m) {
          const uint32_t ab = smem_base + (uint32_t)m * R.act_row + a_off;
          const uint4 a0 = lds128(ab), a1 = lds128(ab + 512);
          const uint2 mt = lds64(meta_s + 8u * (uint32_t)(m * P.meta_stride + c));
          const float a_scale = __uint_as_float(mt.x);
          const int sa = (int)(short)(mt.y & 0xffff);
#pragma unroll
          for (int r = 0; r < ROWS; ++r) {
            int pl = 0, ph = 0;
            // NSB4: word i pairs with activation words (Alo_i, Ahi_i) = ((a0,a4,a1,a5),(a2,a6,a3,a7)) of 8-group i
            if (AMODE == A_U8) {
              pl = dp4a_uu(a0.x, lo[r][0], pl); ph = dp4a_uu(a0.y, hi[r][0], ph);
              pl = dp4a_uu(a0.z, lo[r][1], pl); ph = dp4a_uu(a0.w, hi[r][1], ph);
              pl = dp4a_uu(a1.x, lo[r][2], pl); ph = dp4a_uu(a1.y, hi[r][2], ph);
              pl = dp4a_uu(a1.z, lo[r][3], pl); ph = dp4a_uu(a1.w, hi[r][3], ph);
            } else {  // signed activations x unsigned weight bytes
              pl = dp4a_us(lo[r][0], (int)a0.x, pl); ph = dp4a_us(hi[r][0], (int)a0.y, ph);
              pl = dp4a_us(lo[r][1], (int)a0.z, pl); ph = dp4a_us(hi[r][1], (int)a0.w, ph);
              pl = dp4a_us(lo[r][2], (int)a1.x, pl); ph = dp4a_us(hi[r][2], (int)a1.y, ph);
              pl = dp4a_us(lo[r][3], (int)a1.z, pl); ph = dp4a_us(hi[r][3], (int)a1.w, ph);
            }
            // sum (a - za)(u - off) = sum a*u - off*Sa - za*(Su - 32*off): one exact integer per 32-element chunk
            int isum = pl + (ph >> 4) - off[r] * sa;  // ph is an exact multiple of 16
            if (AMODE == A_U8) {
              const int za = (int)((mt.y >> 16) & 0xff);
              isum -= za * (su[r] - 32 * off[r]);
            }
            acc[r][m] = fmaf((float)isum, a_scale * ws[r], acc[r][m]);
          }
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty0 + 8 * s);  // slot may be refilled
    s += active;
    if (s >= stages) {
      s -= stages;
      phase ^= 1u;
    }

#pragma unroll
    for (int r = 0; r < ROWS; ++r)
#pragma unroll
      for (int m = 0; m < M; ++m) acc[r][m] = warp_sum(acc[r][m]);
    if (lane == 0) {
      if (ROWS == 2 && P.mode == NS_GEMV_GATE_UP_SILU) {
#pragma unroll
        for (int m = 0; m < M; ++m) {
          if (m < P.m) {
            const float g = acc[0][m], up = acc[ROWS - 1][m];
            const float sg = P.eltop == NS_ELT_GELU ? ns_gelu(g) : ns_silu(g);  // kernel_ref.h:1569-1576
            if (P.aux) P.aux[(size_t)m * P.ldo + ps.out0] = sg;
            P.dst[(size_t)m * P.ldo + ps.out0] = sg * up;
          }
        }
      } else {
#pragma unroll
        for (int r = 0; r < ROWS; ++r) {
          if (r == 1 && !ps.valid1) continue;
          const long long out = r ? ps.out1 : ps.out0;
#pragma unroll
          for (int m = 0; m < M; ++m) {
            if (m < P.m) {
              const size_t o = (size_t)m * P.ldo + out;
              float v = acc[r][m];
              if (P.bias) v += P.bias_bcast ? P.bias[out] : P.bias[o];
              if (P.eltop == NS_ELT_GELU) v = ns_gelu(v);
              if (P.residual) v += P.residual[o];
              P.dst[o] = v;
            }
          }
        }
      }
    }
  }
}

template <int AMODE, int M, bool ASYM, int STYPE, int ROWS, bool NORM, int NC = kConsumers, bool W8 = false>
int launch_rows(const GemvParams& P, const RingPlan& plan, size_t act_region, int act_row, int red_off, cudaStream_t st) {
  auto kern = gemv_ring_kernel<AMODE, M, ASYM, STYPE, ROWS, NORM, NC, W8>;
  constexpr int threads = (NC + (NC > kConsumers ? 2 : 1)) * 32;
  static bool attr_set = false;
  if (!attr_set) {
    NS_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  const int stage_bytes = ROWS * P.pitch;
  const size_t smem = act_region + (size_t)plan.stages * stage_bytes + (size_t)plan.stages * 16;
  static const int env_cps = getenv("NS_RING_CPS") ? atoi(getenv("NS_RING_CPS")) : 0;  // tuning aid
  const int ctas_per_sm = plan.ctas == 1 ? 1 : (env_cps > 0 ? env_cps : 2);
  RingCfg R;
  R.ring_off = (int)act_region;
  R.stages = plan.stages;
  R.active = plan.active;
  R.act_row = act_row;
  R.red_off = red_off;
  if (ROWS == 2) {
    R.units = P.npairs;
  } else {
    long long rows = 0;
    for (int i = 0; i < P.nw; ++i) rows += P.n[i];
    R.units = (int)rows;
  }
  R.cpg_magic = P.cpg > 1 ? (uint32_t)((0x100000000ull + (uint64_t)P.cpg - 1) / (uint64_t)P.cpg) : 0u;
  int grid = ns_num_sms() * ctas_per_sm;
  if (grid > R.units) grid = R.units;
  if (grid < 1) grid = 1;
  static const bool dbg = getenv("NS_RING_DEBUG") != nullptr;
  if (dbg)
    fprintf(stderr, "gemv_ring: k=%d pitch=%d rows/stage=%d stages=%d active=%d smem=%zu ctas/sm=%d\n", P.k, P.pitch, ROWS, plan.stages,
            plan.active, smem, ctas_per_sm);
  NS_CUDA_TRY(ns_launch_pdl(kern, dim3(grid), dim3(threads), smem, st, P, R));
  ns_count_launch();
  return NS_OK;
}

}  // namespace

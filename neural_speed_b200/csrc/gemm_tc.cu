// gemm_tc.cu -- prefill / batched weight-only matmul on the Hopper tensor cores (wgmma + TMA + mbarrier), M > 4 rows.
//
// Replaces the reference's blocked GEMM for int4 weights: LauncherBase::run_block / LauncherIntKBlock::run_block
// (bestla/bestla/bestla_wrapper.h:501,768) with WeightKBlockNInteger::getWeight + decompress_kblock_s4_fp
// (bestla_prologue_b.h:642-733, kernel_ref.h:1113) feeding the JIT AMX/AVX512 micro-kernels (bestla_gemm.h), and the
// ggml Q4_0 mul_mat for prompt batches (core/ne_layers.c:7085).  Numerics: weights are dequantised to bf16
// ((u - 8 - zp) exactly in bf16, times the bf16-rounded scale), activations rounded to bf16, fp32 accumulation in registers --
// the reference's own CompBf16 numerics (BF16 tolerance 2e-2 at K=4096, bestla_ut.h:80-94); logits stay within the
// north-star's 1e-2 relative bar of the CPU path (tests/test_gpu_gemm_tc.py).
//
// Orientation ("swap-AB"): the WEIGHT tile is the wgmma M operand (128 output channels = two warpgroups x 64 rows) and the
// token tile is the wgmma N operand (T = 32..128 columns), so small batches do not waste the 64-row MMA.  Per CTA and per
// 64-wide k block:
//   warp 12     TMA producer: packed nibbles [128 rows][32 B] (cp.async.bulk.tensor 2-D over the NSB rows, row pitch = pitch)
//               and bf16 activations [T][64] (128B-swizzled) into two mbarrier rings
//   warps 8-11  dequant: 1 thread = 1 weight row: 2 x LDS.128 of nibbles -> 64 bf16 via (w >> 4j) & 0x000F000F | 0x4300
//               (bf16 128+u), HSUB2 (exact), HMUL2 by the group scale -> 8 x STS.128 into the 128B-swizzled K-major tile,
//               fence.proxy.async, arrive
//   warps 0-7   two consumer warpgroups: 4 x wgmma.mma_async m64nTk16 (bf16, fp32 accumulate) per k block on their 64 weight
//               rows, one k block kept in flight (wgmma.wait_group 1) before the smem slots are released; then the epilogue
//               (+bias, +residual) straight from the accumulator registers to fp32 global stores
// T stops at 128: the m64n128 accumulator is 64 fp32 registers per thread, which with 416 threads leaves room for the rest
// (65536 registers / 416 threads = 157); a 256-token tile would need 128 and spill.  Larger M takes more CTAs on grid.y.
// Roofline: tensor (bf16, fp32 accumulate): flops = 2*M*N*K per launch.
#include "async_copy.cuh"
#include "nsb.cuh"

namespace {

constexpr int BLOCK_N = 128;  // weight rows per CTA (two wgmma M = 64 halves)
constexpr int BLOCK_K = 64;   // bf16 elements per k block (one 128-byte swizzle atom)
constexpr int WG_K = 16;      // k of one wgmma
constexpr int DEQ_TILE = BLOCK_N * BLOCK_K * 2;  // 16384: one 128-row k block as bf16
constexpr int kConsumerThreads = 256, kDequantThreads = 128, kThreads = kConsumerThreads + kDequantThreads + 32;

struct GemmParams {
  const uint8_t* rows;
  int wfmt, f4kind;
  int pitch, sc_off, zp_off, stype, asym, group, ngroups;
  int n, k, kpad, m;
  float* dst;
  int ldo;
  const float* bias;
  int bias_bcast;
  const float* residual;
  int kb_per_split;  // k blocks per grid.z slice (>= total: no split)
  int dbg;  // NS_TC_DEBUG: 1 = dequant warps skip the conversion, 2 = no MMAs issued, 4 = epilogue skipped (timing experiments)
};

// The kernel addresses its barriers and ring slots by pointer.  These forward to async_copy.cuh and take the shared address inside
// the call, after the other arguments: smem_u32(&bar) at the call sites reorders the consumers' wait arithmetic in the SASS, and
// that order measured 0.7-1.0 % slower at 2048 tokens (NVIDIA H100 80GB HBM3, 700 W power limit).
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) { ::mbar_init(smem_u32(bar), count); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { ::mbar_expect_tx(smem_u32(bar), bytes); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { ::mbar_arrive(smem_u32(bar)); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) { ::mbar_wait(smem_u32(bar), parity); }
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int x, int y, uint64_t* bar) {
  tma_2d(smem_u32(dst), map, x, y, smem_u32(bar));
}
// K-major, 128B-swizzled tile: 8-row groups 1024 B apart (SBO), LBO unused (=1), layout SWIZZLE_128B (sm_90 encoding: 1 at bit 62)
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// D[64 x N] += A[64 x 16] * B[N x 16]^T, both operands K-major in shared memory, bf16 inputs, fp32 accumulate (SASS: HGMMA)
__device__ __forceinline__ void wgmma_m64n32k16(float (&d)[16], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
      "}, %16, %17, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(1));
}
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(1));
}
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(1));
}

template <int T>
__device__ __forceinline__ void wgmma_k16(float (&d)[T / 2], uint64_t adesc, uint64_t bdesc) {
  if constexpr (T == 32) wgmma_m64n32k16(d, adesc, bdesc);
  else if constexpr (T == 64) wgmma_m64n64k16(d, adesc, bdesc);
  else wgmma_m64n128k16(d, adesc, bdesc);
}

// W8: int8 weights (64 packed bytes per row and k block instead of 32).
template <int T, bool W8 = false>
struct Smem {
  static constexpr int SP = 6;                   // packed-weight stages
  static constexpr int SD = 3;                   // dequantised-weight stages
  static constexpr int SA = T >= 128 ? 4 : 6;    // activation stages
  static constexpr int ROW_BYTES = W8 ? BLOCK_K : BLOCK_K / 2;  // packed bytes per weight row and k block
  static constexpr int PACKED_STAGE = BLOCK_N * ROW_BYTES;
  static constexpr int DEQ_STAGE = DEQ_TILE;
  static constexpr int ACT_STAGE = T * BLOCK_K * 2;
  static constexpr int off_deq = 0;
  static constexpr int off_act = off_deq + SD * DEQ_STAGE;
  static constexpr int off_packed = off_act + SA * ACT_STAGE;
  static constexpr int off_bar = off_packed + SP * PACKED_STAGE;
  static constexpr int num_bars = 2 * SP + 2 * SA + 2 * SD;
  static constexpr int total = off_bar + num_bars * 8 + 1024;  // + slack for manual 1024-B alignment
};

template <int T, bool W8>
__global__ void __launch_bounds__(kThreads, 1)
    gemm_w4_tc_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_a, const GemmParams P) {
  using L = Smem<T, W8>;
  constexpr int ROW_BYTES = L::ROW_BYTES;
  constexpr int SA = L::SA, SP = L::SP, SD = L::SD, PACKED_STAGE = L::PACKED_STAGE, DEQ_STAGE = L::DEQ_STAGE;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023);
  unsigned char* deq = smem + L::off_deq;
  unsigned char* act = smem + L::off_act;
  unsigned char* packed = smem + L::off_packed;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::off_bar);
  uint64_t* p_full = bars;
  uint64_t* p_empty = p_full + SP;
  uint64_t* a_full = p_empty + SP;
  uint64_t* a_empty = a_full + SA;
  uint64_t* d_full = a_empty + SA;
  uint64_t* d_empty = d_full + SD;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * BLOCK_N;
  const int t0 = blockIdx.y * T;
  // split-K (small M: too few output tiles to fill the SMs): this CTA owns k blocks [kb0, kb0 + num_kb) and adds its partial
  // tile to dst with fp32 atomics (dst zeroed by the launcher; bias / residual applied by split 0)
  const int total_kb = (P.kpad + BLOCK_K - 1) / BLOCK_K;
  const int kb0 = blockIdx.z * P.kb_per_split;
  const int num_kb = (total_kb - kb0 < P.kb_per_split) ? total_kb - kb0 : P.kb_per_split;

  __shared__ float nf4_lut[16];  // constant memory serialises divergent indices; shared memory broadcasts per bank
  if (threadIdx.x >= 32 && threadIdx.x < 48) nf4_lut[threadIdx.x - 32] = NS_F4_LUT[P.f4kind][threadIdx.x - 32];
  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    for (int i = 0; i < SP; ++i) {
      mbar_init(&p_full[i], 1);
      mbar_init(&p_empty[i], kDequantThreads / 32);
    }
    for (int i = 0; i < SA; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], kConsumerThreads / 128);
    }
    for (int i = 0; i < SD; ++i) {
      mbar_init(&d_full[i], kDequantThreads / 32);
      mbar_init(&d_empty[i], kConsumerThreads / 128);
    }
    fence_mbar_init();
  }
  if (warp == 12 && lane == 0) {
    prefetch_tensormap(&tmap_w);
    prefetch_tensormap(&tmap_a);
  }
  __syncthreads();

  if (warp == 12) {
    // ============================ TMA producer ============================
    if (lane == 0) {
      // packed weights never depend on the previous kernel: prefetch the first ring before griddepcontrol.wait
      const int pre = num_kb < SP ? num_kb : SP;
      for (int kb = 0; kb < pre; ++kb) {
        mbar_expect_tx(&p_full[kb], PACKED_STAGE);
        tma_load_2d(packed + kb * PACKED_STAGE, &tmap_w, (kb0 + kb) * ROW_BYTES, n0, &p_full[kb]);
      }
      pdl_wait();  // activations were written by the preceding kernel
      for (int kb = 0; kb < num_kb; ++kb) {
        const int sa = kb % SA;
        if (kb >= SA) mbar_wait(&a_empty[sa], ((kb / SA) - 1) & 1);
        mbar_expect_tx(&a_full[sa], L::ACT_STAGE);
        tma_load_2d(act + sa * L::ACT_STAGE, &tmap_a, (kb0 + kb) * BLOCK_K, t0, &a_full[sa]);
        const int kp = kb + SP;  // keep the packed ring SP blocks ahead
        if (kp < num_kb) {
          const int sp = kp % SP;
          mbar_wait(&p_empty[sp], ((kp / SP) - 1) & 1);
          mbar_expect_tx(&p_full[sp], PACKED_STAGE);
          tma_load_2d(packed + sp * PACKED_STAGE, &tmap_w, (kb0 + kp) * ROW_BYTES, n0, &p_full[sp]);
        }
      }
    }
  } else if (warp >= 8) {
    // ============================ dequant: one thread per weight row (128 rows) ============================
    const int r = threadIdx.x - kConsumerThreads;  // row inside the CTA's 128 rows; packed rows are ROW_BYTES apart
    int grow = n0 + r;
    if (grow >= P.n) grow = P.n - 1;  // rows past N are zero-filled by TMA; keep the scale loads in bounds
    const uint8_t* rowp = P.rows + (size_t)grow * P.pitch;
    const int swz = r & 7;
    for (int kb = 0; kb < num_kb; ++kb) {
      const int sp = kb % SP, sd = kb % SD;
      // group scale / zero point of the two 32-element halves of this k block
      int g0 = ((kb0 + kb) * BLOCK_K) / P.group, g1 = ((kb0 + kb) * BLOCK_K + 32) / P.group;
      if (g0 >= P.ngroups) g0 = P.ngroups - 1;
      if (g1 >= P.ngroups) g1 = P.ngroups - 1;
      const float sc0 = ns_scale_at(rowp + P.sc_off, P.stype, g0);
      const float sc1 = (g1 == g0) ? sc0 : ns_scale_at(rowp + P.sc_off, P.stype, g1);
      // offset subtracted in bf16 before the scale: 128 (bf16 magic) + 8 (nibble bias) [+ zero point] for packed int4,
      // the zero point alone for int8 weights (all exactly representable)
      float of0 = W8 ? 0.f : 136.f, of1 = of0;
      if (P.asym) {
        of0 += (float)(int)(signed char)rowp[P.zp_off + g0];
        of1 += (float)(int)(signed char)rowp[P.zp_off + g1];
      }
      const __nv_bfloat162 s2[2] = {__float2bfloat162_rn(sc0), __float2bfloat162_rn(sc1)};
      const __nv_bfloat162 o2[2] = {__float2bfloat162_rn(of0), __float2bfloat162_rn(of1)};

      mbar_wait(&p_full[sp], (kb / SP) & 1);
      const uint4* pk = reinterpret_cast<const uint4*>(packed + sp * PACKED_STAGE + r * ROW_BYTES);
      uint32_t words[W8 ? 16 : 8];
#pragma unroll
      for (int i = 0; i < (W8 ? 4 : 2); ++i) {
        const uint4 qv = pk[i];
        words[4 * i] = qv.x, words[4 * i + 1] = qv.y, words[4 * i + 2] = qv.z, words[4 * i + 3] = qv.w;
      }
      if (kb >= SD) mbar_wait(&d_empty[sd], ((kb / SD) - 1) & 1);
      unsigned char* drow_base = deq + sd * DEQ_STAGE + (r >> 3) * 1024 + swz * 128;
      if (!(P.dbg & 1))
#pragma unroll
      for (int c = 0; c < 8; ++c) {  // 16-byte chunk c of the bf16 row = k 8c..8c+7
        const int h = c >> 2;
        uint32_t o[4];
        if (W8) {
          // int8 weights, natural byte order: words[2c] = k 8c..8c+3, words[2c+1] = k 8c+4..8c+7
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const uint32_t wsrc = words[2 * c + (j >> 1)];
            const int b0 = (int)(signed char)((wsrc >> (16 * (j & 1))) & 0xffu), b1 = (int)(signed char)((wsrc >> (16 * (j & 1) + 8)) & 0xffu);
            __nv_bfloat162 v = __floats2bfloat162_rn((float)b0, (float)b1);
            v = __hmul2(__hsub2(v, o2[h]), s2[h]);
            o[j] = *reinterpret_cast<uint32_t*>(&v);
          }
        } else if (P.wfmt == NS_W_NF4) {
          // NF4 codes: level from the table (kernel_ref.h:1325-1368), rounded to bf16, times the bf16 scale
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float l0 = nf4_lut[(words[c] >> (4 * j)) & 0xFu], l1 = nf4_lut[(words[c] >> (4 * j + 16)) & 0xFu];
            __nv_bfloat162 v = __hmul2(__floats2bfloat162_rn(l0, l1), s2[h]);
            o[j] = *reinterpret_cast<uint32_t*>(&v);
          }
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            uint32_t t = ((words[c] >> (4 * j)) & 0x000F000Fu) | 0x43004300u;  // bf16x2 (128 + e(2j), 128 + e(2j+1))
            __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&t);
            v = __hmul2(__hsub2(v, o2[h]), s2[h]);
            o[j] = *reinterpret_cast<uint32_t*>(&v);
          }
        }
        *reinterpret_cast<uint4*>(drow_base + ((c ^ swz) << 4)) = make_uint4(o[0], o[1], o[2], o[3]);
      }
      fence_proxy_async();  // generic-proxy writes -> visible to the MMA
      __syncwarp();
      // The packed slot is released only now that every lane has consumed its words: released right after the loads were
      // issued, the producer's next TMA into the slot could land before a lane's LDS had read it, and int8 rows then took
      // bytes of block kb + SP (tests/test_gpu_gemm_tc.py, exact tier)
      if (lane == 0) {
        mbar_arrive(&p_empty[sp]);
        mbar_arrive(&d_full[sd]);
      }
    }
  } else {
    // ============================ consumers: warpgroup g owns weight rows [64g, 64g + 64) of the tile ============================
    const int g = warp >> 2;
    const bool leader = (threadIdx.x & 127) == 0;
    float acc[T / 2];
#pragma unroll
    for (int i = 0; i < T / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < num_kb; ++kb) {
      const int sd = kb % SD, sa = kb % SA;
      mbar_wait(&d_full[sd], (kb / SD) & 1);
      mbar_wait(&a_full[sa], (kb / SA) & 1);
      const uint32_t a_addr = smem_u32(deq + sd * DEQ_STAGE) + g * (64 * BLOCK_K * 2);
      const uint32_t b_addr = smem_u32(act + sa * L::ACT_STAGE);
      if (!(P.dbg & 2)) {
        wgmma_fence();
#pragma unroll
        for (int k4 = 0; k4 < BLOCK_K / WG_K; ++k4)
          wgmma_k16<T>(acc, make_desc_sw128(a_addr + k4 * WG_K * 2), make_desc_sw128(b_addr + k4 * WG_K * 2));
        wgmma_commit();
      }
      wgmma_wait<1>();  // the previous k block's MMAs have finished reading shared memory
      if (kb > 0 && leader) {
        mbar_arrive(&d_empty[(kb - 1) % SD]);
        mbar_arrive(&a_empty[(kb - 1) % SA]);
      }
    }
    wgmma_wait<0>();
    // ============================ epilogue: accumulator registers -> global ============================
    // d[4j + 2h + e] holds weight row 64g + 16(warp & 3) + lane / 4 + 8h and token 8j + 2(lane & 3) + e
    pdl_wait();  // dst / residual may still be in use by the preceding kernel
    if (!(P.dbg & 4)) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int nrow = n0 + g * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        if (nrow >= P.n) continue;
        const float bcast_bias = (P.bias && P.bias_bcast) ? P.bias[nrow] : 0.f;
#pragma unroll
        for (int j = 0; j < T / 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int t = t0 + 8 * j + 2 * (lane & 3) + e;
            if (t < P.m) {
              const size_t o = (size_t)t * P.ldo + nrow;
              float x = acc[4 * j + 2 * h + e];
              if (blockIdx.z == 0) {
                x += bcast_bias;
                if (P.bias && !P.bias_bcast) x += P.bias[o];
                if (P.residual) x += P.residual[o];
              }
              if (gridDim.z > 1) atomicAdd(P.dst + o, x);
              else P.dst[o] = x;
            }
          }
      }
    }
  }
}

// fp32 -> bf16 activations [m][kpad], zero padded, optional column gather
__global__ void __launch_bounds__(256) act_to_bf16_kernel(const float* __restrict__ A, int lda, int M, int K, int kpad,
                                                          const int* __restrict__ shuffle, __nv_bfloat16* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one thread per 2 elements
  const size_t total = (size_t)M * (kpad >> 1);
  if (idx >= total) return;
  const int m = (int)(idx / (kpad >> 1)), k = (int)(idx - (size_t)m * (kpad >> 1)) * 2;
  float a = 0.f, b = 0.f;
  if (k < K) a = A[(size_t)m * lda + (shuffle ? shuffle[k] : k)];
  if (k + 1 < K) b = A[(size_t)m * lda + (shuffle ? shuffle[k + 1] : k + 1)];
  reinterpret_cast<__nv_bfloat162*>(out)[idx] = __floats2bfloat162_rn(a, b);
}
// same, 8 elements per thread (2 x 16-byte loads, one 16-byte store): K % 8 == 0, K == kpad, lda % 4 == 0, no gather.
// The scalar version above moved 1.6 TB/s; a 2048-token prefill converts 0.35 GB per layer.
__global__ void __launch_bounds__(256) act_to_bf16_v8_kernel(const float* __restrict__ A, int lda, int M, int K,
                                                             __nv_bfloat16* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int k8 = K >> 3;
  const size_t total = (size_t)M * k8;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int m = (int)(idx / k8), c = (int)(idx - (size_t)m * k8);
    const float4* src = (const float4*)(A + (size_t)m * lda) + 2 * c;
    const float4 x = src[0], y = src[1];
    __nv_bfloat162 p0 = __floats2bfloat162_rn(x.x, x.y), p1 = __floats2bfloat162_rn(x.z, x.w);
    __nv_bfloat162 p2 = __floats2bfloat162_rn(y.x, y.y), p3 = __floats2bfloat162_rn(y.z, y.w);
    uint4 o;
    o.x = *(uint32_t*)&p0, o.y = *(uint32_t*)&p1, o.z = *(uint32_t*)&p2, o.w = *(uint32_t*)&p3;
    ((uint4*)out)[idx] = o;
  }
}

// One launch's token tile and k split.  Small M gives too few output tiles to fill the SMs, so the k blocks are cut into up to 16
// slices of >= 8 blocks (512 k) each, one CTA per tile and slice, their partial tiles added with fp32 atomics.  A residual or bias
// that aliases dst keeps one slice: dst is zeroed before a split launch.
struct TcPlan {
  int T, splits, kb_per_split;
};
TcPlan tc_plan(int m, int n, int kpad, bool dst_aliased) {
  TcPlan p;
  p.T = m <= 32 ? 32 : (m <= 64 ? 64 : 128);
  const int total_kb = (kpad + BLOCK_K - 1) / BLOCK_K;
  const int tiles = ((n + BLOCK_N - 1) / BLOCK_N) * ((m + p.T - 1) / p.T);
  int splits = 1;
  static const int env_splits = getenv("NS_TC_SPLITS") ? atoi(getenv("NS_TC_SPLITS")) : 0;  // tuning aid
  if (3 * tiles < 2 * ns_num_sms() && !dst_aliased) {
    splits = ns_num_sms() / tiles;  // floor: one CTA per SM is resident (416 threads, ~100-160 KB smem), a partial second wave doubles the time
    if (splits > total_kb / 8) splits = total_kb / 8;  // keep >= 8 k blocks (512 k) per slice
    if (splits > 16) splits = 16;
    if (splits < 1) splits = 1;
  }
  if (env_splits > 0) splits = env_splits;
  p.kb_per_split = (total_kb + splits - 1) / splits;
  p.splits = (total_kb + p.kb_per_split - 1) / p.kb_per_split;
  return p;
}

template <int T, bool W8>
int launch_t(const CUtensorMap& mw, const CUtensorMap& ma, const GemmParams& P, const TcPlan& plan, cudaStream_t st) {
  using L = Smem<T, W8>;
  auto kern = gemm_w4_tc_kernel<T, W8>;
  static bool attr_set = false;
  if (!attr_set) {
    NS_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::total));
    attr_set = true;
  }
  dim3 grid((P.n + BLOCK_N - 1) / BLOCK_N, (P.m + T - 1) / T, (unsigned)plan.splits);
  GemmParams Q = P;
  Q.kb_per_split = plan.kb_per_split;
  if (plan.splits > 1) NS_CUDA_TRY(cudaMemset2DAsync(P.dst, (size_t)P.ldo * 4, 0, (size_t)P.n * 4, (size_t)P.m, st));
  NS_CUDA_TRY(ns_launch_pdl(kern, grid, dim3(kThreads), (size_t)L::total, st, mw, ma, Q));
  ns_count_launch();
  return NS_OK;
}

}  // namespace

extern "C" int ns_gemm_tc_plan(int m, int n, int kpad, int residual_is_dst, int* out) {
  if (m < 1 || n < 1 || kpad < 32 || kpad % 32 || !out) {
    ns_set_error("ns_gemm_tc_plan: invalid arguments (m=%d n=%d kpad=%d)", m, n, kpad);
    return NS_E_INVALID;
  }
  const TcPlan p = tc_plan(m, n, kpad, residual_is_dst != 0);
  out[0] = p.T, out[1] = p.splits, out[2] = p.kb_per_split;
  return NS_OK;
}

size_t ns_gemm_tc_workspace_bytes(int m, int kpad) { return ns_round_up((size_t)m * kpad * 2, 256); }

bool ns_gemm_tc_supported(const ns_weight* w) {
  return (w->wfmt == NS_W_S4 || w->wfmt == NS_W_NF4 || w->wfmt == NS_W_S8 || w->wfmt == NS_W_Q8_0) && (w->group % 32 == 0 || w->group == w->k);
}

// phase 1: fp32 activations -> bf16 [m][kpad] in ws (ns_gemm_tc_workspace_bytes(m, kpad) bytes)
int ns_launch_act_bf16(const ns_weight* w, const float* act, int lda, int m, void* ws, cudaStream_t st) {
  if (!w->shuffle && w->k == w->kpad && (w->k & 7) == 0 && (lda & 3) == 0 && ((uintptr_t)act & 15) == 0) {
    const size_t total8 = (size_t)m * (w->k >> 3);
    size_t blocks = (total8 + 255) / 256;
    if (blocks > (size_t)ns_num_sms() * 16) blocks = (size_t)ns_num_sms() * 16;
    NS_CUDA_TRY(ns_launch_pdl(act_to_bf16_v8_kernel, dim3((unsigned)blocks), dim3(256), 0, st, act, lda, m, w->k, (__nv_bfloat16*)ws));
    ns_count_launch();
    return NS_OK;
  }
  const size_t total = (size_t)m * (w->kpad >> 1);
  NS_CUDA_TRY(ns_launch_pdl(act_to_bf16_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st, act, lda, m, w->k,
                            w->kpad, (const int*)w->shuffle, (__nv_bfloat16*)ws));
  ns_count_launch();
  return NS_OK;
}

// silu(gate) * up, elementwise (epilogues Swish alpha=-1 + Mul of ip_fusion_ffn.cpp:408-470, kernel_ref.h:1574); 4 elements per
// thread when the pointers and the count allow it
template <bool V4>
__global__ void __launch_bounds__(256) silu_mul_kernel(const float* __restrict__ g, const float* __restrict__ u,
                                                       float* __restrict__ out, float* __restrict__ aux, size_t total,
                                                       int eltop) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t n = V4 ? total >> 2 : total;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (V4) {
      const float4 x = ((const float4*)g)[i], y = ((const float4*)u)[i];
      float4 sg;
      sg.x = eltop == NS_ELT_GELU ? ns_gelu(x.x) : ns_silu(x.x);
      sg.y = eltop == NS_ELT_GELU ? ns_gelu(x.y) : ns_silu(x.y);
      sg.z = eltop == NS_ELT_GELU ? ns_gelu(x.z) : ns_silu(x.z);
      sg.w = eltop == NS_ELT_GELU ? ns_gelu(x.w) : ns_silu(x.w);
      if (aux) ((float4*)aux)[i] = sg;
      ((float4*)out)[i] = make_float4(sg.x * y.x, sg.y * y.y, sg.z * y.z, sg.w * y.w);
    } else {
      const float x = g[i];
      const float sg = eltop == NS_ELT_GELU ? ns_gelu(x) : ns_silu(x);
      if (aux) aux[i] = sg;
      out[i] = sg * u[i];
    }
  }
}
// silu(gate) * up written straight into the bf16 activation image of the down projection: the fp32 product (m x fmid, 90 MB at 2048
// tokens of Llama-2-7B) is neither stored nor read back.  Same values as silu_mul_kernel followed by act_to_bf16_v8_kernel (the product
// is formed in fp32 and rounded once).  Used when the caller does not look at the intermediate (the eval step).
__global__ void __launch_bounds__(256) silu_mul_bf16_kernel(const float* __restrict__ g, const float* __restrict__ u, size_t total8,
                                                            __nv_bfloat16* __restrict__ out, int eltop) {
  pdl_launch_dependents();
  pdl_wait();
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total8; idx += (size_t)gridDim.x * blockDim.x) {
    const float4 x0 = ((const float4*)g)[2 * idx], x1 = ((const float4*)g)[2 * idx + 1];
    const float4 y0 = ((const float4*)u)[2 * idx], y1 = ((const float4*)u)[2 * idx + 1];
    const float xs[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
    const float ys[8] = {y0.x, y0.y, y0.z, y0.w, y1.x, y1.y, y1.z, y1.w};
    float p[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) p[i] = (eltop == NS_ELT_GELU ? ns_gelu(xs[i]) : ns_silu(xs[i])) * ys[i];
    __nv_bfloat162 q0 = __floats2bfloat162_rn(p[0], p[1]), q1 = __floats2bfloat162_rn(p[2], p[3]);
    __nv_bfloat162 q2 = __floats2bfloat162_rn(p[4], p[5]), q3 = __floats2bfloat162_rn(p[6], p[7]);
    uint4 o;
    o.x = *(uint32_t*)&q0, o.y = *(uint32_t*)&q1, o.z = *(uint32_t*)&q2, o.w = *(uint32_t*)&q3;
    ((uint4*)out)[idx] = o;
  }
}
// g, u: [m][w2->k] fp32 contiguous.  false: the layout needs the general conversion kernel (act-order gather, padded K) -- the caller
// takes the two-step path
bool ns_launch_silu_mul_bf16(const ns_weight* w2, const float* g, const float* u, int m, void* ws, cudaStream_t st, int eltop, int* rc) {
  if (w2->shuffle || w2->k != w2->kpad || (w2->k & 7) || (((uintptr_t)g | (uintptr_t)u | (uintptr_t)ws) & 15)) return false;
  const size_t total8 = (size_t)m * (w2->k >> 3);
  size_t blocks = (total8 + 255) / 256;
  if (blocks > (size_t)ns_num_sms() * 16) blocks = (size_t)ns_num_sms() * 16;
  if (blocks < 1) blocks = 1;
  *rc = ns_cuda_ok(ns_launch_pdl(silu_mul_bf16_kernel, dim3((unsigned)blocks), dim3(256), 0, st, g, u, total8, (__nv_bfloat16*)ws, eltop),
                   "silu_mul_bf16_kernel")
            ? NS_OK
            : NS_E_CUDA;
  ns_count_launch();
  return true;
}
int ns_launch_silu_mul(const float* g, const float* u, float* out, float* aux, size_t total, cudaStream_t st, int eltop) {
  const bool v4 = (total & 3) == 0 && (((uintptr_t)g | (uintptr_t)u | (uintptr_t)out | (uintptr_t)aux) & 15) == 0;
  const size_t n = v4 ? total >> 2 : total;
  size_t blocks = (n + 255) / 256;
  if (blocks > (size_t)ns_num_sms() * 16) blocks = (size_t)ns_num_sms() * 16;
  if (blocks < 1) blocks = 1;
  if (v4)
    NS_CUDA_TRY(ns_launch_pdl(silu_mul_kernel<true>, dim3((unsigned)blocks), dim3(256), 0, st, g, u, out, aux, total, eltop));
  else
    NS_CUDA_TRY(ns_launch_pdl(silu_mul_kernel<false>, dim3((unsigned)blocks), dim3(256), 0, st, g, u, out, aux, total, eltop));
  ns_count_launch();
  return NS_OK;
}
__global__ void __launch_bounds__(256) gelu_kernel(float* __restrict__ x, size_t total) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) x[i] = ns_gelu(x[i]);
}
int ns_launch_gelu(float* x, size_t total, cudaStream_t st) {
  NS_CUDA_TRY(ns_launch_pdl(gelu_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st, x, total));
  ns_count_launch();
  return NS_OK;
}

// phase 2: weights x bf16 activations already in ws
int ns_launch_gemm_tc(const ns_weight* w, const void* ws, float* dst, int ldo, int m, const float* bias, int bias_bcast,
                      const float* residual, cudaStream_t st) {
  if (!ns_gemm_tc_supported(w)) {
    ns_set_error("tensor-core GEMM: int4 / NF4 / int8 / Q8_0 weights with 32-multiple groups are supported");
    return NS_E_UNSUPPORTED;
  }
  const __nv_bfloat16* abf = (const __nv_bfloat16*)ws;
  const TcPlan plan = tc_plan(m, w->n, w->kpad, residual == dst || bias == dst);
  const int T = plan.T;
  const bool w8 = w->wfmt == NS_W_S8 || w->wfmt == NS_W_Q8_0;  // natural-order int8 codes (ggml Q8_0: zero point 0, fp16 d)
  CUtensorMap mw, ma;
  // packed nibbles: uint8 [n][q_bytes] with row pitch `pitch`; box = 32 bytes (64 k) x 128 rows, no swizzle
  int rc = ns_tensor_map_2d(&mw, CU_TENSOR_MAP_DATA_TYPE_UINT8, w->rows, w->q_bytes, w->n, w->pitch, w8 ? BLOCK_K : BLOCK_K / 2, BLOCK_N,
                            CU_TENSOR_MAP_SWIZZLE_NONE, "weights");
  if (rc != NS_OK) return rc;
  rc = ns_tensor_map_2d(&ma, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, abf, w->kpad, m, (uint64_t)w->kpad * 2, BLOCK_K, T,
                        CU_TENSOR_MAP_SWIZZLE_128B, "activations");
  if (rc != NS_OK) return rc;
  GemmParams P;
  P.rows = w->rows;
  P.wfmt = w->wfmt;
  P.f4kind = w->f4kind;
  P.pitch = w->pitch;
  P.sc_off = w->sc_off;
  P.zp_off = w->zp_off;
  P.stype = w->stype;
  P.asym = w->asym;
  P.group = w->group;
  P.ngroups = w->ngroups;
  P.n = w->n;
  P.k = w->k;
  P.kpad = w->kpad;
  P.m = m;
  P.dst = dst;
  P.ldo = ldo;
  P.bias = bias;
  P.bias_bcast = bias_bcast;
  P.residual = residual;
  static const int dbg = getenv("NS_TC_DEBUG") ? atoi(getenv("NS_TC_DEBUG")) : 0;
  P.dbg = dbg;
  if (w8) {
    switch (T) {
      case 32: return launch_t<32, true>(mw, ma, P, plan, st);
      case 64: return launch_t<64, true>(mw, ma, P, plan, st);
      default: return launch_t<128, true>(mw, ma, P, plan, st);
    }
  }
  switch (T) {
    case 32: return launch_t<32, false>(mw, ma, P, plan, st);
    case 64: return launch_t<64, false>(mw, ma, P, plan, st);
    default: return launch_t<128, false>(mw, ma, P, plan, st);
  }
}

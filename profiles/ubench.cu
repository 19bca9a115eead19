// ubench.cu -- micro-measurements that size the persistent decode kernel (round 2): grid-barrier latency, broadcast L2 reads,
// issue rates of the dp4a/lop3 mix.  Standalone: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o profiles/ubench.bin profiles/ubench.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x)                                                                      \
  do {                                                                             \
    cudaError_t e = (x);                                                           \
    if (e != cudaSuccess) {                                                        \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
      exit(1);                                                                     \
    }                                                                              \
  } while (0)

__device__ __forceinline__ unsigned long long clk64() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%clock64;" : "=l"(t));
  return t;
}
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned ld_relaxed(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_release(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ---- T1: grid barrier variants.  Every round: all threads write one float (the "output"), CTA barrier, grid barrier.
// mode 0: threadfence + atomicAdd, thread 0 polls ld.acquire (program.cu r01)
// mode 1: red.release.gpu.add, thread 0 polls ld.acquire
// mode 2: per-CTA flag (st.release), threads 0..G-1 poll one flag each (ld.acquire), then CTA barrier
// mode 3: as 2 with ld.relaxed polling + one fence.acq_rel at the end
template <int MODE>
__global__ void barrier_kernel(unsigned* ctr, unsigned* flags, float* sink, int rounds, unsigned long long* out) {
  const int G = gridDim.x;
  unsigned long long t0 = 0;
  for (int r = 0; r < rounds; ++r) {
    if (r == 8 && threadIdx.x == 0) t0 = clk64();
    sink[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = (float)r;
    __syncthreads();
    if (MODE == 0) {
      if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(ctr + r, 1u);
        while (ld_acquire(ctr + r) < (unsigned)G) {
        }
      }
    } else if (MODE == 1) {
      if (threadIdx.x == 0) {
        red_release(ctr + r, 1u);
        while (ld_acquire(ctr + r) < (unsigned)G) {
        }
      }
    } else if (MODE == 2) {
      if (threadIdx.x == 0) st_release(flags + blockIdx.x, (unsigned)(r + 1));
      if (threadIdx.x < G) {
        while (ld_acquire(flags + threadIdx.x) < (unsigned)(r + 1)) {
        }
      }
    } else {
      if (threadIdx.x == 0) st_release(flags + blockIdx.x, (unsigned)(r + 1));
      if (threadIdx.x < G) {
        while (ld_relaxed(flags + threadIdx.x) < (unsigned)(r + 1)) {
        }
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = clk64() - t0;
}

// ---- T2: every CTA reads the same `bytes` of fp32 from L2 (ld.global.cg.v4) right after a grid barrier; cycles until the data is
// in registers of all threads (max over threads via the CTA barrier)
__global__ void bcast_kernel(const float* src, int nvec, unsigned* flags, float* sink, int rounds, unsigned long long* out) {
  const int G = gridDim.x;
  unsigned long long acc = 0;
  float s = 0.f;
  for (int r = 0; r < rounds; ++r) {
    if (threadIdx.x == 0) st_release(flags + blockIdx.x, (unsigned)(r + 1));
    if (threadIdx.x < G) {
      while (ld_acquire(flags + threadIdx.x) < (unsigned)(r + 1)) {
      }
    }
    __syncthreads();
    const unsigned long long t0 = clk64();
    float4 v[4];
    int n = 0;
    for (int i = threadIdx.x; i < nvec && n < 4; i += blockDim.x, ++n)
      asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v[n].x), "=f"(v[n].y), "=f"(v[n].z), "=f"(v[n].w) : "l"(src + 4 * (size_t)i));
    for (int j = 0; j < n; ++j) s += v[j].x + v[j].y + v[j].z + v[j].w;
    __syncthreads();
    if (r >= 4) acc += clk64() - t0;
  }
  if (s == 1234.5f) sink[0] = s;
  if (threadIdx.x == 0) out[blockIdx.x] = acc / (rounds - 4);
}

// ---- T3: issue rates.  WHAT 0: dp4a only, 1: lop3 only, 2: 1:1 mix, 3: imad, 4: ffma, 5: the row-chunk mix (8 lop, 8 dp4a, i2f, fmul, ffma, lea)
template <int WHAT>
__global__ void pipe_kernel(int iters, unsigned* sink, unsigned long long* out) {
  unsigned a0 = threadIdx.x, a1 = threadIdx.x * 3, a2 = 7, a3 = 11, b0 = blockIdx.x | 0x01010101u, b1 = 0x0f0f0f0fu ^ threadIdx.x;
  int c0 = 0, c1 = 0, c2 = 0, c3 = 0;
  int d0 = 0, d1 = 0, d2 = 0, d3 = 0, e0 = 0, e1 = 0, e2 = 0, e3 = 0, g0 = 0, g1 = 0, g2 = 0, g3 = 0;
  float f0 = 1.f, f1 = 2.f, f2 = 0.5f, f3 = 0.25f;
  __syncthreads();
  const unsigned long long t0 = clk64();
#pragma unroll 1
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      if (WHAT == 0) {
        asm volatile("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(c0) : "r"(a0), "r"(b0));
        asm volatile("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(c1) : "r"(a1), "r"(b1));
        asm volatile("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(c2) : "r"(a2), "r"(b0));
        asm volatile("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(c3) : "r"(a3), "r"(b1));
      } else if (WHAT == 1) {
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a0) : "r"(b0), "r"(b1));
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a1) : "r"(b0), "r"(b1));
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a2) : "r"(b0), "r"(b1));
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a3) : "r"(b0), "r"(b1));
      } else if (WHAT == 2) {
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a0) : "r"(b0), "r"(b1));
        asm volatile("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(c0) : "r"(a1), "r"(b0));
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a2) : "r"(b0), "r"(b1));
        asm volatile("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(c1) : "r"(a3), "r"(b1));
      } else if (WHAT == 3) {
        asm volatile("mad.lo.s32 %0, %1, %2, %0;" : "+r"(c0) : "r"(a0), "r"(b0));
        asm volatile("mad.lo.s32 %0, %1, %2, %0;" : "+r"(c1) : "r"(a1), "r"(b1));
        asm volatile("mad.lo.s32 %0, %1, %2, %0;" : "+r"(c2) : "r"(a2), "r"(b0));
        asm volatile("mad.lo.s32 %0, %1, %2, %0;" : "+r"(c3) : "r"(a3), "r"(b1));
      } else if (WHAT == 4) {
        asm volatile("fma.rn.f32 %0, %1, %2, %0;" : "+f"(f0) : "f"(f2), "f"(f3));
        asm volatile("fma.rn.f32 %0, %1, %2, %0;" : "+f"(f1) : "f"(f2), "f"(f3));
        asm volatile("fma.rn.f32 %0, %1, %2, %0;" : "+f"(f2) : "f"(f0), "f"(f3));
        asm volatile("fma.rn.f32 %0, %1, %2, %0;" : "+f"(f3) : "f"(f1), "f"(f0));
      } else if (WHAT == 6) {
        // integer tensor-core MMA through mma.sync: m16n8k32 u8 x s8 -> s32, four independent accumulators
        asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+r"(c0), "+r"(c1), "+r"(c2), "+r"(c3) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
        asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+r"(d0), "+r"(d1), "+r"(d2), "+r"(d3) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b1), "r"(b0));
        asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+r"(e0), "+r"(e1), "+r"(e2), "+r"(e3) : "r"(a1), "r"(a0), "r"(a3), "r"(a2), "r"(b0), "r"(b1));
        asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+r"(g0), "+r"(g1), "+r"(g2), "+r"(g3) : "r"(a1), "r"(a0), "r"(a3), "r"(a2), "r"(b1), "r"(b0));
      } else {
        // one row-chunk: 4 words -> 8 lop, 8 dp4a (two chains), lea.hi-like add, i2f, fmul, ffma
        unsigned w[4] = {a0 + u, a1 + u, a2 + u, a3 + u};
        int pl = c0, ph = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          unsigned lo, hi;
          asm volatile("and.b32 %0, %1, 0x0f0f0f0f;" : "=r"(lo) : "r"(w[i]));
          asm volatile("and.b32 %0, %1, 0xf0f0f0f0;" : "=r"(hi) : "r"(w[i]));
          asm volatile("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(pl) : "r"(lo), "r"(b0));
          asm volatile("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(ph) : "r"(hi), "r"(b1));
        }
        int isum = pl + (ph >> 4);
        float fs = (float)isum;
        f0 = fmaf(fs, f2 * f3, f0);
        c1 += isum & 1;
      }
    }
  }
  const unsigned long long t1 = clk64();
  if (threadIdx.x == 0) out[blockIdx.x] = t1 - t0;
  sink[blockIdx.x * blockDim.x + threadIdx.x] = a0 ^ a1 ^ a2 ^ a3 ^ c0 ^ c1 ^ c2 ^ c3 ^ d0 ^ d1 ^ d2 ^ d3 ^ e0 ^ e1 ^ e2 ^ e3 ^ g0 ^ g1 ^ g2 ^ g3 ^
                                                   __float_as_uint(f0 + f1 + f2 + f3);
}

// ---- T4: TMA 1-D bulk-copy streaming rate: one producer warp per CTA, `lanes` lanes each issuing copies of `bytes` bytes into a
// ring of `slots` slots (one mbarrier each); a consumer thread waits for each slot and frees it at once (no compute).
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__global__ void __launch_bounds__(64, 1) tma_stream_kernel(const unsigned char* src, size_t total_bytes, int bytes, int slots, int lanes,
                                                           unsigned long long* out) {
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t base = smem_u32(smem);
  const uint32_t full0 = base + (uint32_t)slots * bytes, empty0 = full0 + 8u * slots;
  if (threadIdx.x == 0) {
    for (int s = 0; s < slots; ++s) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(full0 + 8 * s));
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(empty0 + 8 * s));
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const size_t per_cta = total_bytes / gridDim.x / bytes * bytes;
  const int n = (int)(per_cta / bytes);
  const unsigned char* my = src + (size_t)blockIdx.x * per_cta;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned long long t0 = clk64();
  if (warp == 0) {
    for (int i0 = 0; i0 < n; i0 += lanes) {
      const int i = i0 + lane;
      if (lane < lanes && i < n) {
        const int s = i % slots, lap = i / slots;
        if (lap > 0) {
          uint32_t ok;
          do {
            asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(ok) : "r"(empty0 + 8 * s), "r"((uint32_t)(lap - 1) & 1u) : "memory");
          } while (!ok);
        }
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(full0 + 8 * s), "r"((uint32_t)bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(base + (uint32_t)s * bytes),
                     "l"(my + (size_t)i * bytes), "r"((uint32_t)bytes), "r"(full0 + 8 * s)
                     : "memory");
      }
      __syncwarp();
    }
  } else if (lane == 0) {
    for (int i = 0; i < n; ++i) {
      const int s = i % slots, lap = i / slots;
      uint32_t ok;
      do {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(ok) : "r"(full0 + 8 * s), "r"((uint32_t)lap & 1u) : "memory");
      } while (!ok);
      asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(empty0 + 8 * s) : "memory");
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) out[blockIdx.x] = clk64() - t0;
}

static double med(unsigned long long* v, int n) {
  double s = 0;
  unsigned long long mx = 0;
  for (int i = 0; i < n; ++i) {
    s += (double)v[i];
    if (v[i] > mx) mx = v[i];
  }
  return s / n;
}

int main(int argc, char** argv) {
  const bool only_t3b = argc > 1 && argv[1][0] == 'm';  // only the integer-MMA rate
  const bool only_t4 = argc > 1 && argv[1][0] == 't';
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  printf("device %s, %d SMs, clock %d kHz\n", prop.name, sms, prop.clockRate);
  unsigned *ctr, *flags, *usink;
  float* sink;
  unsigned long long *out, hout[1024];
  CK(cudaMalloc(&ctr, 4096 * 4));
  CK(cudaMalloc(&flags, 4096 * 4));
  CK(cudaMalloc(&sink, 1024 * 1024 * 4));
  CK(cudaMalloc(&usink, 1024 * 1024 * 4));
  CK(cudaMalloc(&out, 1024 * 8));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  const int rounds = 1000;
  for (int per = 1; per <= 2 && !only_t4 && !only_t3b; ++per) {
    const int G = sms * per;
    for (int mode = 0; mode < 4; ++mode) {
      for (int threads = 288; threads <= 544; threads += 256) {
        if (per == 2 && threads > 288) continue;
        if (mode >= 2 && threads < G) continue;
        CK(cudaMemset(ctr, 0, 4096 * 4));
        CK(cudaMemset(flags, 0, 4096 * 4));
        void* args[] = {&ctr, &flags, &sink, (void*)&rounds, &out};
        const void* k = mode == 0 ? (const void*)barrier_kernel<0> : mode == 1 ? (const void*)barrier_kernel<1> : mode == 2 ? (const void*)barrier_kernel<2> : (const void*)barrier_kernel<3>;
        CK(cudaEventRecord(e0));
        CK(cudaLaunchCooperativeKernel(k, dim3(G), dim3(threads), args, 0, 0));
        CK(cudaEventRecord(e1));
        CK(cudaDeviceSynchronize());
        float ms;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        CK(cudaMemcpy(hout, out, G * 8, cudaMemcpyDeviceToHost));
        printf("T1 barrier mode %d grid %d threads %d: %.3f us/round (events), %.0f cycles/round (clock64)\n", mode, G, threads,
               ms * 1e3 / rounds, med(hout, G) / (rounds - 8));
      }
    }
  }
  // T2
  float* src;
  CK(cudaMalloc(&src, 1 << 20));
  CK(cudaMemset(src, 0, 1 << 20));
  for (int per = 1; per <= 2 && !only_t4 && !only_t3b; ++per) {
    const int G = sms * per;
    const int threads = per == 1 ? 544 : 320;
    for (int bytes = 16384; bytes <= 65536; bytes *= 2) {
      int b = bytes == 32768 ? 44032 : bytes;
      if (b / 16 > threads * 4) continue;
      int nvec = b / 16, r2 = 200;
      CK(cudaMemset(flags, 0, 4096 * 4));
      void* args[] = {&src, &nvec, &flags, &sink, &r2, &out};
      CK(cudaLaunchCooperativeKernel((const void*)bcast_kernel, dim3(G), dim3(threads), args, 0, 0));
      CK(cudaDeviceSynchronize());
      CK(cudaMemcpy(hout, out, G * 8, cudaMemcpyDeviceToHost));
      printf("T2 broadcast read %d B by %d CTAs x %d thr: %.0f cycles avg\n", b, G, threads, med(hout, G));
    }
  }
  // T3
  for (int what = (only_t3b ? 6 : 0); what < 7 && !only_t4; ++what) {
    for (int warps = 4; warps <= 16; warps *= 2) {
      int iters = 2000;
      void* args[] = {&iters, &usink, &out};
      const void* k = what == 0 ? (const void*)pipe_kernel<0> : what == 1 ? (const void*)pipe_kernel<1> : what == 2 ? (const void*)pipe_kernel<2> : what == 3 ? (const void*)pipe_kernel<3> : what == 4 ? (const void*)pipe_kernel<4> : what == 5 ? (const void*)pipe_kernel<5> : (const void*)pipe_kernel<6>;
      CK(cudaLaunchKernel(k, dim3(sms), dim3(warps * 32), args, 0, 0));
      CK(cudaDeviceSynchronize());
      CK(cudaMemcpy(hout, out, sms * 8, cudaMemcpyDeviceToHost));
      const double cyc = med(hout, sms);
      const double instr_per_warp = (what == 5 ? 8.0 * 22 : 8.0 * 4) * iters;
      printf("T3 pipe what %d warps/SM %d: %.3f cycles per warp-instr per SMSP (%.2f warp-instr/clk/SM)\n", what, warps,
             cyc / (instr_per_warp * warps / 4.0), instr_per_warp * warps / cyc);
    }
  }
  // T4: TMA streaming
  if (!only_t3b) {
    const size_t total = (size_t)1 << 30;  // 1 GiB >> L2
    unsigned char* big;
    CK(cudaMalloc(&big, total));
    CK(cudaMemset(big, 1, total));
    CK(cudaFuncSetAttribute(tma_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    const int sizes[] = {1152, 2304, 4608, 9216, 23040};
    for (int per = 1; per <= 2; ++per)
      for (int si = 0; si < 5; ++si)
        for (int lanes = 1; lanes <= 16; lanes *= 4) {
          const int bytes = sizes[si];
          const int budget = (per == 1 ? 200 : 100) * 1024;
          int slots = budget / (bytes + 16);
          if (slots > 64) slots = 64;
          if (slots < lanes) continue;
          const size_t smem = (size_t)slots * bytes + 16 * slots;
          const int G = sms * per;
          void* args[] = {&big, (void*)&total, (void*)&bytes, &slots, &lanes, &out};
          for (int rep = 0; rep < 2; ++rep) {
            CK(cudaEventRecord(e0));
            CK(cudaLaunchKernel((const void*)tma_stream_kernel, dim3(G), dim3(64), args, smem, 0));
            CK(cudaEventRecord(e1));
            CK(cudaDeviceSynchronize());
          }
          float ms;
          CK(cudaEventElapsedTime(&ms, e0, e1));
          printf("T4 tma stream: %d CTA/SM, copy %5d B, %2d slots (%3zu KB), %2d issuing lanes: %.0f GB/s\n", per, bytes, slots, smem / 1024, lanes,
                 (double)(total / G / bytes * bytes) * G / (ms * 1e-3) / 1e9);
        }
  }
  return 0;
}

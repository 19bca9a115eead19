// select.cuh -- the device top-k selection shared by the sampler (sample.cu) and the beam-search candidates (beam.cu).
#pragma once
#include <stdint.h>

namespace {

// the kth largest (1-based) of a set of distinct 64-bit keys: eight passes of an 8-bit digit histogram over the keys that share
// the digits chosen so far.  each(fn) calls fn(key) for this thread's share of the keys.  All threads of the CTA call it.
template <class Each>
__device__ uint64_t radix_kth(Each each, int kth, unsigned* hist, uint64_t* s_prefix, int* s_rem) {
  uint64_t prefix = 0, mask = 0;
  int rem = kth;
  for (int shift = 56; shift >= 0; shift -= 8) {
    if (threadIdx.x == 0) {
      *s_prefix = prefix;
      *s_rem = rem;
    }
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    each([&](uint64_t key) {
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255], 1u);
    });
    __syncthreads();
    if (threadIdx.x < 32) {  // lane L: digits 255 - 8 L .. 248 - 8 L, counted from the top
      const int lane = threadIdx.x;
      unsigned c = 0;
      for (int j = 0; j < 8; ++j) c += hist[255 - 8 * lane - j];
      unsigned incl = c;
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      const unsigned excl = incl - c;
      if (excl < (unsigned)rem && (unsigned)rem <= incl) {
        unsigned acc = excl;
        for (int j = 0; j < 8; ++j) {
          const int b = 255 - 8 * lane - j;
          if (acc + hist[b] >= (unsigned)rem) {
            *s_prefix = prefix | ((uint64_t)b << shift);
            *s_rem = rem - (int)acc;
            break;
          }
          acc += hist[b];
        }
      }
    }
    __syncthreads();
    prefix = *s_prefix;
    rem = *s_rem;
    mask |= (uint64_t)255 << shift;
    __syncthreads();
  }
  return prefix;
}

}  // namespace

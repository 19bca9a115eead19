// vocab_slices.cuh -- the reduction of a [rows][n] block of logits in vocabulary slices, shared by argmax_kernel and
// logprob_kernel (logprob.cu), sample_kernel (sample.cu) and beam_candidates_kernel (beam.cu).
//
// Grid (kVocabSlices, rows): CTA s of a row reduces slice s of the row (vocab_slice), writes its partials to global scratch
// and takes the row's ticket (last_of_row); the row's last CTA merges the partials in slice order, so a row's result does not
// depend on the order in which its CTAs finish.  The slice reductions:
//   slice_argmax, slice_expsum       the slice's max and lowest id, and its sum of exp(x - max), in the order logprob.h states;
//                                    merge_slice_maxima and merge_slice_sums merge them (on the host too)
//   slice_top_keys, row_top_keys     the slice's top K keys into the partials; in the last CTA, the row's top K over them, sorted
#pragma once
#include <stdint.h>

#include "logprob.h"

constexpr int kVocabSlices = 32;  // CTAs per row

// slice s of [0, n): [s per, (s + 1) per) within [0, n), per = ceil(n / kVocabSlices); the last slices of a short row are empty
struct VocabSlice {
  int lo, hi;
};
NS_HD int vocab_slice_width(int n) { return (n + kVocabSlices - 1) / kVocabSlices; }
NS_HD VocabSlice vocab_slice(int n, int s) {
  const int per = vocab_slice_width(n), lo = s * per < n ? s * per : n;
  return {lo, lo + per < n ? lo + per : n};
}

// M, I of logprob.h from the slices' maxima m[s] and ids id[s], in slice order; I = 0 when no slice has an id
template <class PM, class PI>
NS_HD void merge_slice_maxima(PM m, PI id, float& M, int& idx) {
  M = -INFINITY;
  idx = 0x7fffffff;
  for (int s = 0; s < kVocabSlices; ++s) ns_logprob_argmax_merge(M, idx, m[s], id[s]);
  if (idx == 0x7fffffff) idx = 0;  // all NaN / -inf: the reference's loop keeps index 0
}
// S of logprob.h from the slices' sums S_s[s] and maxima m[s], in slice order
template <class PF>
NS_HD float merge_slice_sums(PF S_s, PF m, float M) {
  float S = 0.f;
  for (int s = 0; s < kVocabSlices; ++s) S = NS_FADD(S, ns_logprob_merge_term(S_s[s], m[s], M));
  return S;
}

namespace {

// the per-warp values of a block reduction; one instance per kernel, shared by slice_argmax and slice_expsum
template <int THREADS>
struct WarpPartials {
  float v[THREADS / 32];
  int id[THREADS / 32];
};
template <int THREADS>
__device__ __forceinline__ WarpPartials<THREADS>& warp_partials() {
  __shared__ WarpPartials<THREADS> w;
  return w;
}

// fn(x_i, i) for this thread's entries of x[lo, hi), i = lo + threadIdx.x + j THREADS ascending, with 4 loads in flight
template <int THREADS, class Fn>
__device__ __forceinline__ void slice_each(const float* __restrict__ x, int lo, int hi, Fn fn) {
  constexpr int U = 4;
  for (int i0 = lo + threadIdx.x; i0 < hi; i0 += THREADS * U) {
    float v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = (i0 + u * THREADS < hi) ? x[i0 + u * THREADS] : 0.f;
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (i0 + u * THREADS < hi) fn(v[u], i0 + u * THREADS);
  }
}

// the greedy pick of x[lo, hi): its largest value and the lowest id of that value (ns_logprob_argmax_merge: NaN never wins;
// -inf and id 0x7fffffff when the slice holds nothing but NaN, or nothing).  Each thread merges its entries in ascending order,
// the lanes of a warp merge by xor butterfly, thread 0 merges the warps in order.  Every thread calls it; the result is thread 0's.
template <int THREADS>
__device__ __forceinline__ void slice_argmax(const float* __restrict__ x, int lo, int hi, float& best, int& bi) {
  WarpPartials<THREADS>& w = warp_partials<THREADS>();
  best = -INFINITY;
  bi = 0x7fffffff;
  slice_each<THREADS>(x, lo, hi, [&](float v, int i) { ns_logprob_argmax_merge(best, bi, v, i); });
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    ns_logprob_argmax_merge(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
  if ((threadIdx.x & 31) == 0) {
    w.v[threadIdx.x >> 5] = best;
    w.id[threadIdx.x >> 5] = bi;
  }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int k = 1; k < THREADS / 32; ++k) ns_logprob_argmax_merge(best, bi, w.v[k], w.id[k]);
}

// S_s of logprob.h: the sum of ns_logprob_term(x_i, m) over x[lo, hi), m the slice's max as thread 0 holds it (slice_argmax's).
// Thread j adds x_{lo + j}, x_{lo + j + THREADS}, ... in ascending order, the lanes of a warp combine by xor butterfly, thread 0
// adds the warps in order.  Every thread calls it; the result is thread 0's.
template <int THREADS>
__device__ __forceinline__ float slice_expsum(const float* __restrict__ x, int lo, int hi, float m) {
  WarpPartials<THREADS>& w = warp_partials<THREADS>();
  if (threadIdx.x == 0) w.v[0] = m;  // thread 0 is the only reader of the warp partials
  __syncthreads();
  m = w.v[0];
  float acc = 0.f;
  slice_each<THREADS>(x, lo, hi, [&](float v, int) { acc = __fadd_rn(acc, ns_logprob_term(v, m)); });
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  __syncthreads();  // every thread has read m
  if ((threadIdx.x & 31) == 0) w.v[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int k = 1; k < THREADS / 32; ++k) acc = __fadd_rn(acc, w.v[k]);
  return acc;
}

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

// the selection's shared memory; one instance per kernel, shared by slice_top_keys and row_top_keys
struct TopKeysScratch {
  unsigned hist[256];
  uint64_t prefix;
  int rem, cnt, off[kVocabSlices + 1];
};
__device__ __forceinline__ TopKeysScratch& top_keys_scratch() {
  __shared__ TopKeysScratch t;
  return t;
}

// the top kth of the n keys each(...) enumerates (radix_kth), into out[0 .. kth) in no particular order; the scratch's cnt is 0
template <class Each, class Out>
__device__ __forceinline__ void top_keys(Each each, int n, int kth, Out* out) {
  TopKeysScratch& t = top_keys_scratch();
  const uint64_t thr = n > kth ? radix_kth(each, kth, t.hist, &t.prefix, &t.rem) : 0;
  each([&](uint64_t key) {
    if (key >= thr) {
      const int pos = atomicAdd(&t.cnt, 1);
      if (pos < kth) out[pos] = key;
    }
  });
}

// the slice's top min(K, len) keys: key(i) is the key of the slice's entry i, 0 <= i < len (distinct keys, larger first: as
// ns_sample_key).  Writes them to keys[0 .. min(K, len)) in no particular order, and their count to *count (thread 0).  Every
// thread calls it.
template <int THREADS, class Key>
__device__ __forceinline__ void slice_top_keys(Key key, int len, int K, unsigned long long* keys, int* count) {
  const int kk = min(K, len);
  if (threadIdx.x == 0) top_keys_scratch().cnt = 0;
  __syncthreads();
  top_keys([&](auto fn) { for (int i = threadIdx.x; i < len; i += THREADS) fn(key(i)); }, len, kk, keys);
  if (threadIdx.x == 0) *count = kk;
}

// in the row's last CTA: the row's top K keys over its slices' partials (slice s: count[s] keys at keys + s * per_slice), sorted
// descending into sk[0 .. K) by a bitonic sort over P entries, P the power of two >= K (sk[K .. P) end as 0, which no key is).
// sk: P entries of shared memory.  Every thread calls it; returns P.
template <int THREADS>
__device__ __forceinline__ int row_top_keys(const unsigned long long* keys, const int* count, int per_slice, int K, uint64_t* sk) {
  TopKeysScratch& t = top_keys_scratch();
  if (threadIdx.x == 0) {
    int n = 0;
    for (int s = 0; s < kVocabSlices; ++s) {
      t.off[s] = n;
      n += ((const volatile int*)count)[s];
    }
    t.off[kVocabSlices] = n;
    t.cnt = 0;
  }
  int P = 1;
  while (P < K) P <<= 1;
  for (int i = threadIdx.x; i < P; i += THREADS) sk[i] = 0;
  __syncthreads();
  const volatile unsigned long long* rk = keys;
  top_keys(
      [&](auto fn) {
        for (int s = 0; s < kVocabSlices; ++s) {
          const int c = t.off[s + 1] - t.off[s];
          for (int j = threadIdx.x; j < c; j += THREADS) fn((uint64_t)rk[(size_t)s * per_slice + j]);
        }
      },
      t.off[kVocabSlices], K, sk);
  __syncthreads();
  for (int size = 2; size <= P; size <<= 1)  // bitonic sort, descending
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int q = threadIdx.x; q < P / 2; q += THREADS) {
        const int i = (q / stride) * stride * 2 + q % stride, j = i + stride;
        const bool desc = (i & size) == 0;
        const uint64_t u = sk[i], v = sk[j];
        if ((u < v) == desc) {
          sk[i] = v;
          sk[j] = u;
        }
      }
      __syncthreads();
    }
  return P;
}

// the ticket of a row: every thread of each of the row's `ctas` CTAs calls it once the CTA's partials are written.  True in
// every thread of the row's last CTA, which then sees the other CTAs' partials (read them through volatile pointers).  The
// caller sets tickets[row] back to 0 once the partials are merged, for the next launch or graph replay.
__device__ __forceinline__ bool last_of_row(unsigned* tickets, int row, unsigned ctas = kVocabSlices) {
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&tickets[row], 1u) == ctas - 1;
  __syncthreads();
  if (last) __threadfence();
  return last;
}

}  // namespace

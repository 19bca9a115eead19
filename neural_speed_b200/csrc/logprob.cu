// logprob.cu -- the scoring pass's log-softmax and target gather (ns_llama_eval_all) in one launch per lm_head chunk, its host
// restatement, and the parity entry ns_llama_logprob.
//
// Grid (kLogprobSlices, rows), kLogprobThreads threads, in the style of argmax_kernel.  Each CTA reads its slice twice: once for
// the slice's max and lowest id, once (from L2) for the sum of exp(x - slice max).  It stores {max, id, sum} and takes a ticket;
// the row's last CTA merges the slices in slice order and writes the row's argmax and log-prob.  The arithmetic and the order of
// every sum are stated once in logprob.h.
#include "nsb.cuh"
#include "logprob.h"

#include <algorithm>

namespace {

__global__ void __launch_bounds__(kLogprobThreads) logprob_kernel(LogprobLaunch a) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.y, n = a.n_vocab;
  const float* x = a.logits + (size_t)row * n;
  const int per = (n + kLogprobSlices - 1) / kLogprobSlices;
  const int lo = blockIdx.x * per, hi = min(n, lo + per);
  __shared__ float sv[kLogprobThreads / 32];
  __shared__ int si[kLogprobThreads / 32];
  __shared__ float s_max;
  __shared__ bool last;
  // pass 1: the slice's max and its lowest id
  float best = -INFINITY;
  int bi = 0x7fffffff;
  constexpr int U = 4;
  for (int i0 = lo + threadIdx.x; i0 < hi; i0 += kLogprobThreads * U) {
    float v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = (i0 + u * kLogprobThreads < hi) ? x[i0 + u * kLogprobThreads] : -INFINITY;
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (i0 + u * kLogprobThreads < hi) ns_logprob_argmax_merge(best, bi, v[u], i0 + u * kLogprobThreads);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    ns_logprob_argmax_merge(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
  if ((threadIdx.x & 31) == 0) {
    sv[threadIdx.x >> 5] = best;
    si[threadIdx.x >> 5] = bi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kLogprobThreads / 32; ++w) ns_logprob_argmax_merge(best, bi, sv[w], si[w]);
    s_max = best;
  }
  __syncthreads();
  const int slot = row * kLogprobSlices + blockIdx.x;
  // pass 2: the slice's sum of exp(x - max), in the order logprob.h states
  if (a.targets) {
    const float m = s_max;
    float acc = 0.f;
    for (int i0 = lo + threadIdx.x; i0 < hi; i0 += kLogprobThreads * U) {
      float v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = (i0 + u * kLogprobThreads < hi) ? x[i0 + u * kLogprobThreads] : 0.f;
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (i0 + u * kLogprobThreads < hi) acc = __fadd_rn(acc, ns_logprob_term(v[u], m));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
    __syncthreads();  // sv is reused
    if ((threadIdx.x & 31) == 0) sv[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kLogprobThreads / 32; ++w) acc = __fadd_rn(acc, sv[w]);
      a.psum[slot] = acc;
    }
  }
  if (threadIdx.x == 0) {
    a.pmax[slot] = best;
    a.pidx[slot] = bi;
    __threadfence();
    last = atomicAdd(&a.tickets[row], 1u) == kLogprobSlices - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  const volatile float* pm = a.pmax + row * kLogprobSlices;
  const volatile int* pi = a.pidx + row * kLogprobSlices;
  float M = -INFINITY;
  int I = 0x7fffffff;
  for (int s = 0; s < kLogprobSlices; ++s) ns_logprob_argmax_merge(M, I, pm[s], pi[s]);
  if (I == 0x7fffffff) I = 0;
  a.tickets[row] = 0u;  // ready for the next launch
  if (a.argmax) a.argmax[row] = I;
  if (!a.targets) return;
  const volatile float* ps = a.psum + row * kLogprobSlices;
  float S = 0.f;
  for (int s = 0; s < kLogprobSlices; ++s) S = __fadd_rn(S, ns_logprob_merge_term(ps[s], pm[s], M));
  const int t = a.targets[row];  // checked by the callers; NaN rather than a read outside the row
  a.logprobs[row] = t >= 0 && t < n ? ns_logprob_final(x[t], M, S) : __int_as_float(0x7fc00000);
}

}  // namespace

int ns_launch_logprob(const LogprobLaunch& a, cudaStream_t st) {
  NS_CUDA_TRY(ns_launch_pdl(logprob_kernel, dim3((unsigned)kLogprobSlices, (unsigned)a.rows), dim3(kLogprobThreads), 0, st, a));
  ns_count_launch();
  return NS_OK;
}

// ---- host restatement ------------------------------------------------------------------------------------------------------
extern "C" int ns_logprob_row_host(const float* logits, int n_vocab, int32_t target, float* logprob, int32_t* argmax) {
  if (!logits || n_vocab < 1 || (logprob && (target < 0 || target >= n_vocab)) || (!logprob && !argmax)) {
    ns_set_error("ns_logprob_row_host: invalid arguments (n_vocab %d target %d, or no output)", n_vocab, target);
    return NS_E_INVALID;
  }
  const int per = (n_vocab + kLogprobSlices - 1) / kLogprobSlices;
  float m[kLogprobSlices], S_s[kLogprobSlices];
  int id[kLogprobSlices];
  float M = -INFINITY;
  int I = 0x7fffffff;
  for (int s = 0; s < kLogprobSlices; ++s) {
    const int lo = s * per, hi = std::min(n_vocab, lo + per);
    m[s] = -INFINITY;
    id[s] = 0x7fffffff;
    for (int i = lo; i < hi; ++i) ns_logprob_argmax_merge(m[s], id[s], logits[i], i);
    float lane[kLogprobThreads];
    for (int j = 0; j < kLogprobThreads; ++j) {
      lane[j] = 0.f;
      for (int i = lo + j; i < hi; i += kLogprobThreads) lane[j] = NS_FADD(lane[j], ns_logprob_term(logits[i], m[s]));
    }
    for (int w = 0; w < kLogprobThreads / 32; ++w) {
      float* v = lane + 32 * w;
      for (int o = 16; o > 0; o >>= 1) {
        float t[32];
        for (int L = 0; L < 32; ++L) t[L] = NS_FADD(v[L], v[L ^ o]);
        for (int L = 0; L < 32; ++L) v[L] = t[L];
      }
    }
    S_s[s] = lane[0];
    for (int w = 1; w < kLogprobThreads / 32; ++w) S_s[s] = NS_FADD(S_s[s], lane[32 * w]);
    ns_logprob_argmax_merge(M, I, m[s], id[s]);
  }
  if (argmax) *argmax = I == 0x7fffffff ? 0 : I;
  if (logprob) {
    float S = 0.f;
    for (int s = 0; s < kLogprobSlices; ++s) S = NS_FADD(S, ns_logprob_merge_term(S_s[s], m[s], M));
    *logprob = ns_logprob_final(logits[target], M, S);
  }
  return NS_OK;
}

// ---- parity entry --------------------------------------------------------------------------------------------------------
// workspace: tickets [kLogprobMaxRows] (the first 128 bytes for every n) | max | id | sum, each [n][kLogprobSlices]
extern "C" size_t ns_llama_logprob_workspace_bytes(int n, int n_vocab) {
  if (n < 1 || n > kLogprobMaxRows || n_vocab < 1) return 0;
  return (size_t)kLogprobMaxRows * 4 + (size_t)3 * n * kLogprobSlices * 4;
}

extern "C" int ns_llama_logprob(const float* logits, int n, int n_vocab, const int32_t* targets, float* logprobs, int32_t* argmax, void* ws,
                                void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!logits || !ws || n < 1 || n > kLogprobMaxRows || n_vocab < 1 || (!targets) != (!logprobs) || (!logprobs && !argmax)) {
    ns_set_error("ns_llama_logprob: invalid arguments (n %d n_vocab %d; targets and logprobs both or neither, one output at least)", n,
                 n_vocab);
    return NS_E_INVALID;
  }
  char* w = static_cast<char*>(ws);
  LogprobLaunch a{};
  a.logits = logits;
  a.n_vocab = n_vocab;
  a.rows = n;
  a.targets = targets;
  a.logprobs = logprobs;
  a.argmax = argmax;
  a.tickets = reinterpret_cast<unsigned*>(w);
  a.pmax = reinterpret_cast<float*>(w + (size_t)kLogprobMaxRows * 4);
  a.pidx = reinterpret_cast<int*>(a.pmax + (size_t)n * kLogprobSlices);
  a.psum = reinterpret_cast<float*>(a.pidx + (size_t)n * kLogprobSlices);
  return ns_launch_logprob(a, ns_stream_of(queue));
}

// logprob.cu -- the eval step's greedy pick (argmax_kernel) and the scoring pass's log-softmax and target gather
// (logprob_kernel, ns_llama_eval_all) in one launch per lm_head chunk, their host restatement, and the parity entry
// ns_llama_logprob.
//
// Both kernels reduce vocabulary slices as vocab_slices.cuh describes.  Each CTA takes its slice's max and lowest id
// (slice_argmax); logprob_kernel then re-reads the slice (from L2) for its sum of exp(x - slice max) (slice_expsum).  The row's
// last CTA merges the slices in slice order: argmax_kernel advances the eval step's device state with the row's pick,
// logprob_kernel writes the row's argmax and log-prob.  The arithmetic and the order of every sum are stated once in logprob.h.
#include "nsb.cuh"
#include "logprob.h"
#include "vocab_slices.cuh"

namespace {

// BATCH: grid row y (one per sequence) uses logits row y, state + 4 y, record + y rec_stride, its own partial slots and its own
// ticket; the single-sequence instantiation keeps row 0 at compile time
template <bool BATCH>
__global__ void __launch_bounds__(kLogprobThreads) argmax_kernel(const float* __restrict__ logits, int n, int* __restrict__ state,
                                                                 int n_tokens, int advance, int* __restrict__ record, int rec_stride,
                                                                 float* __restrict__ pval, int* __restrict__ pidx,
                                                                 unsigned* __restrict__ tickets) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = BATCH ? (int)blockIdx.y : 0;
  const VocabSlice sl = vocab_slice(n, blockIdx.x);
  pval += row * kVocabSlices;
  pidx += row * kVocabSlices;
  float best;
  int bi;
  slice_argmax<kLogprobThreads>(logits + (size_t)row * n, sl.lo, sl.hi, best, bi);
  if (threadIdx.x == 0) {
    pval[blockIdx.x] = best;
    pidx[blockIdx.x] = bi;
  }
  if (!last_of_row(tickets, row) || threadIdx.x != 0) return;
  merge_slice_maxima((const volatile float*)pval, (const volatile int*)pidx, best, bi);
  tickets[row] = 0u;  // ready for the next launch
  state += 4 * row;
  state[3] = bi;
  if (advance) {
    state[0] = bi;
    state[1] += n_tokens;
    if (record) record[(size_t)row * rec_stride + state[2]++] = bi;
  }
}

__global__ void __launch_bounds__(kLogprobThreads) logprob_kernel(LogprobLaunch a) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.y, n = a.n_vocab, slot = row * kVocabSlices + blockIdx.x;
  const float* x = a.logits + (size_t)row * n;
  const VocabSlice sl = vocab_slice(n, blockIdx.x);
  float best;
  int bi;
  slice_argmax<kLogprobThreads>(x, sl.lo, sl.hi, best, bi);
  if (a.targets) {
    const float sum = slice_expsum<kLogprobThreads>(x, sl.lo, sl.hi, best);
    if (threadIdx.x == 0) a.psum[slot] = sum;
  }
  if (threadIdx.x == 0) {
    a.pmax[slot] = best;
    a.pidx[slot] = bi;
  }
  if (!last_of_row(a.tickets, row) || threadIdx.x != 0) return;
  const volatile float* pm = a.pmax + row * kVocabSlices;
  float M;
  int I;
  merge_slice_maxima(pm, (const volatile int*)a.pidx + row * kVocabSlices, M, I);
  a.tickets[row] = 0u;  // ready for the next launch
  if (a.argmax) a.argmax[row] = I;
  if (!a.targets) return;
  const float S = merge_slice_sums((const volatile float*)a.psum + row * kVocabSlices, pm, M);
  const int t = a.targets[row];  // checked by the callers; NaN rather than a read outside the row
  a.logprobs[row] = t >= 0 && t < n ? ns_logprob_final(x[t], M, S) : __int_as_float(0x7fc00000);
}

}  // namespace

int ns_launch_argmax(const float* logits, int n_vocab, int rows, bool rowwise, int* state, int n_tokens, int advance, int* record,
                     int rec_stride, float* pmax, int* pidx, unsigned* tickets, cudaStream_t st) {
  NS_CUDA_TRY(ns_launch_pdl(rowwise ? argmax_kernel<true> : argmax_kernel<false>, dim3((unsigned)kVocabSlices, (unsigned)rows),
                            dim3(kLogprobThreads), 0, st, logits, n_vocab, state, n_tokens, advance, record, rec_stride, pmax, pidx,
                            tickets));
  ns_count_launch();
  return NS_OK;
}

int ns_launch_logprob(const LogprobLaunch& a, cudaStream_t st) {
  NS_CUDA_TRY(ns_launch_pdl(logprob_kernel, dim3((unsigned)kVocabSlices, (unsigned)a.rows), dim3(kLogprobThreads), 0, st, a));
  ns_count_launch();
  return NS_OK;
}

// ---- host restatement ------------------------------------------------------------------------------------------------------
void ns_logprob_stats_host(const float* x, int n, float* M, int* I, float* S) {
  float m[kVocabSlices], S_s[kVocabSlices];
  int id[kVocabSlices];
  for (int s = 0; s < kVocabSlices; ++s) {
    const VocabSlice sl = vocab_slice(n, s);
    m[s] = -INFINITY;
    id[s] = 0x7fffffff;
    for (int i = sl.lo; i < sl.hi; ++i) ns_logprob_argmax_merge(m[s], id[s], x[i], i);
    float lane[kLogprobThreads];
    for (int j = 0; j < kLogprobThreads; ++j) {
      lane[j] = 0.f;
      for (int i = sl.lo + j; i < sl.hi; i += kLogprobThreads) lane[j] = NS_FADD(lane[j], ns_logprob_term(x[i], m[s]));
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
  }
  merge_slice_maxima(m, id, *M, *I);
  *S = merge_slice_sums(S_s, m, *M);
}

extern "C" int ns_logprob_row_host(const float* logits, int n_vocab, int32_t target, float* logprob, int32_t* argmax) {
  if (!logits || n_vocab < 1 || (logprob && (target < 0 || target >= n_vocab)) || (!logprob && !argmax)) {
    ns_set_error("ns_logprob_row_host: invalid arguments (n_vocab %d target %d, or no output)", n_vocab, target);
    return NS_E_INVALID;
  }
  float M, S;
  int I;
  ns_logprob_stats_host(logits, n_vocab, &M, &I, &S);
  if (argmax) *argmax = I;
  if (logprob) *logprob = ns_logprob_final(logits[target], M, S);
  return NS_OK;
}

// ---- parity entry --------------------------------------------------------------------------------------------------------
// workspace: tickets [kLogprobMaxRows] (the first 128 bytes for every n) | max | id | sum, each [n][kVocabSlices]
extern "C" size_t ns_llama_logprob_workspace_bytes(int n, int n_vocab) {
  if (n < 1 || n > kLogprobMaxRows || n_vocab < 1) return 0;
  return (size_t)kLogprobMaxRows * 4 + (size_t)3 * n * kVocabSlices * 4;
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
  a.pidx = reinterpret_cast<int*>(a.pmax + (size_t)n * kVocabSlices);
  a.psum = reinterpret_cast<float*>(a.pidx + (size_t)n * kVocabSlices);
  return ns_launch_logprob(a, ns_stream_of(queue));
}

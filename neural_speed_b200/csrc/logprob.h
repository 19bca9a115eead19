// logprob.h -- the stated arithmetic of the eval step's scoring pass (ns_llama_eval_all: model_eval with logits_all,
// llama.cpp:743-747, scored as the reference's lm-eval adapter scores it), compiled once for the host and once for the device
// so ns_logprob_row_host and logprob_kernel (logprob.cu) run the same operations in the same order.
//
// One row x[0 .. n) with a target t:
//   slices     s = 0 .. kVocabSlices - 1, the slices of vocab_slices.cuh (vocab_slice)
//   max        m_s, i_s = the largest value of slice s and its lowest id (NaN never wins; -inf, id i_s, when it holds no
//              number above -inf; an empty slice or one of NaN only gives -inf and no id); M, I the same over the slices in
//              order; I = 0 when no slice has an id (argmax_kernel's rule, model_utils.cpp:2963-2985)
//   sum        S_s = sum of ns_logprob_term(x_i, m_s) over slice s: thread j of kLogprobThreads adds x_{lo + j}, x_{lo + j + 256},
//              ... in ascending order into 0, the 32 lanes of a warp then combine by xor butterfly (v_L += v_{L ^ o}, o = 16, 8,
//              4, 2, 1), and the 8 warps' values are added in warp order (slice_expsum);
//              S = sum over s = 0 .. 31 in order of ns_logprob_merge_term(S_s, m_s, M)
//   logprob    (x_t - M) - ns_logf(S)
// Every term is exp(x - m) <= 1 with one term equal to 1 in the slice (or row) of the max, so S_s and S lie in [1, n] whenever
// the row holds a finite max: ns_logf is exact to within an ulp of glibc's logf over [1, 2^17] (tests/test_logprob_cpu.py).
// Consequences of the arithmetic: a NaN anywhere in the row makes S and every log-prob of the row NaN (the argmax skips it);
// a -inf target logit in a row with a finite max gives -inf; a row with no number above -inf has no distribution (S = 0 or
// NaN, log-prob NaN, argmax its lowest -inf id or 0); a +inf logit makes S NaN.
#pragma once
#include "sample.h"

constexpr int kLogprobThreads = 256;  // threads per CTA, which fixes the order of S_s
constexpr int kLogprobMaxRows = 32;   // rows of one launch (the eval step's lm_head chunk)

// log(x) in IEEE fp32 operations (fdlibm's e_logf.c scheme): x = 2^k (1 + f) with 1 + f in [sqrt(2)/2, sqrt(2)), s = f / (2 + f),
// log(1 + f) = f - (hf - s (hf + R(s^2))) with hf = f^2 / 2 and R the Remez polynomial of degree 7 in s^2, plus k ln2 in a head
// (k * ln2_hi exact for |k| < 2^8) and a tail.  0 -> -inf, x < 0 or NaN -> NaN, +inf -> +inf; subnormals are scaled by 2^25 first.
NS_HD float ns_logf(float x) {
  if (x != x) return x;
  if (x == 0.f) return ns_bits_float(0xff800000u);
  if (x < 0.f) return ns_bits_float(0x7fc00000u);
  uint32_t u = ns_float_bits(x);
  if (u == 0x7f800000u) return x;
  int k = 0;
  if (u < 0x00800000u) {  // subnormal
    x = NS_FMUL(x, 33554432.f);
    u = ns_float_bits(x);
    k = -25;
  }
  k += (int)(u >> 23) - 127;
  u &= 0x007fffffu;
  if (u > 0x3504f3u) {  // mantissa above sqrt(2): take 1 + f = m / 2
    u |= 0x3f000000u;
    k += 1;
  } else {
    u |= 0x3f800000u;
  }
  const float f = NS_FSUB(ns_bits_float(u), 1.f);  // exact (Sterbenz)
  const float s = NS_FDIV(f, NS_FADD(2.f, f));
  const float z = NS_FMUL(s, s);
  const float w = NS_FMUL(z, z);
  const float t1 = NS_FMUL(w, NS_FADD(4.0000000596e-01f, NS_FMUL(w, NS_FADD(2.2222198546e-01f, NS_FMUL(w, 1.5313838422e-01f)))));
  const float t2 = NS_FMUL(z, NS_FADD(6.6666668653e-01f,
                                      NS_FMUL(w, NS_FADD(2.8571429849e-01f, NS_FMUL(w, NS_FADD(1.8183572590e-01f, NS_FMUL(w, 1.4798198640e-01f)))))));
  const float R = NS_FADD(t2, t1);
  const float hf = NS_FMUL(NS_FMUL(0.5f, f), f);
  const float dk = (float)k;
  const float ln2_hi = 6.9313812256e-01f, ln2_lo = 9.0580006145e-06f;
  // dk ln2_hi - ((hf - (s (hf + R) + dk ln2_lo)) - f)
  const float tail = NS_FADD(NS_FMUL(s, NS_FADD(hf, R)), NS_FMUL(dk, ln2_lo));
  return NS_FSUB(NS_FMUL(dk, ln2_hi), NS_FSUB(NS_FSUB(hf, tail), f));
}

// the element term of a slice's sum: exp(x - m), 0 for x = -inf (also when m = -inf: the slice holds nothing above -inf)
NS_HD float ns_logprob_term(float x, float m) {
  return x == -INFINITY ? 0.f : ns_sample_expf(NS_FSUB(x, m));
}
// a slice's sum rescaled to the row's max; a slice whose max is -inf contributes its sum as it is (0, or NaN from a NaN logit)
NS_HD float ns_logprob_merge_term(float s, float m, float M) {
  return m == -INFINITY ? s : NS_FMUL(s, ns_sample_expf(NS_FSUB(m, M)));
}
// greedy order: larger value first, lower id among equal values; NaN never wins
NS_HD void ns_logprob_argmax_merge(float& best, int& bi, float v, int i) {
  if (v > best || (v == best && i < bi)) {
    best = v;
    bi = i;
  }
}
NS_HD float ns_logprob_final(float xt, float M, float S) { return NS_FSUB(NS_FSUB(xt, M), ns_logf(S)); }

// the host restatement (logprob.cu) of one row's M, I and S
void ns_logprob_stats_host(const float* x, int n, float* M, int* I, float* S);

#ifdef __CUDACC__
// ---- the device kernels (logprob.cu), grid (kVocabSlices, rows) -------------------------------------------------------------
// logprob_kernel: one launch per lm_head chunk
struct LogprobLaunch {
  const float* logits;  // [rows][n_vocab]
  int n_vocab, rows;    // 1 <= rows <= kLogprobMaxRows
  const int* targets;   // [rows], nullable (then no sums and no log-probs)
  float* logprobs;      // [rows], non-null with targets
  int* argmax;          // [rows], nullable
  // scratch: per-slice max / id / sum [rows][kVocabSlices], tickets [rows] (zero, and zero again after the launch)
  float* pmax;
  int* pidx;
  float* psum;
  unsigned* tickets;
};
int ns_launch_logprob(const LogprobLaunch& a, cudaStream_t st);  // counts its launch
// argmax_kernel: the eval step's greedy pick, I of each row, with state[3] = I and, when `advance`, state[0] = I,
// state[1] += n_tokens, record[state[2]++] = I.  rowwise: row r uses state + 4 r and record + r rec_stride (a pass over several
// sequences); otherwise the single row uses state and record.  Scratch: max / id [rows][kVocabSlices], tickets [rows] (zero, and
// zero again after the launch).  Counts its launch.
int ns_launch_argmax(const float* logits, int n_vocab, int rows, bool rowwise, int* state, int n_tokens, int advance, int* record,
                     int rec_stride, float* pmax, int* pidx, unsigned* tickets, cudaStream_t st);
#endif

// sample.h -- the stated arithmetic of the eval step's sampler (steps 5-7 of model_post_sample_top_k_top_p_repeat,
// model_utils.cpp:2987-3032, and the draw of model_sample_token, :971-991), compiled once for the host and once for the device
// so ns_sample_row_host and sample_kernel (sample.cu) run the same operations in the same order.
//
// Every fp32 / fp64 operation whose rounding matters is spelled out (__fmul_rn / __fadd_rn / fmaf on the device, where nvcc
// would otherwise contract a * b + c; plain operators on the host, built without FMA contraction for x86-64).  The exp is ours,
// not CUDA's expf or ex2.approx: Cody-Waite reduction by ln 2, a degree-7 polynomial in Horner form via fmaf, scaling by
// exponent bits.  It is within 1 ulp of glibc's expf on every finite x <= 0 (tests/test_sampling_cpu.py).
#pragma once
#include <stdint.h>
#include <math.h>
#include <string.h>

#ifdef __CUDACC__
#define NS_HD __host__ __device__ __forceinline__
#else
#define NS_HD inline
#endif

#if defined(__CUDA_ARCH__)
#define NS_FMUL(a, b) __fmul_rn(a, b)
#define NS_FADD(a, b) __fadd_rn(a, b)
#define NS_FSUB(a, b) __fsub_rn(a, b)
#define NS_FDIV(a, b) __fdiv_rn(a, b)
#define NS_DMUL(a, b) __dmul_rn(a, b)
#define NS_DADD(a, b) __dadd_rn(a, b)
#define NS_DDIV(a, b) __ddiv_rn(a, b)
#else
#define NS_FMUL(a, b) ((float)(a) * (float)(b))
#define NS_FADD(a, b) ((float)(a) + (float)(b))
#define NS_FSUB(a, b) ((float)(a) - (float)(b))
#define NS_FDIV(a, b) ((float)(a) / (float)(b))
#define NS_DMUL(a, b) ((double)(a) * (double)(b))
#define NS_DADD(a, b) ((double)(a) + (double)(b))
#define NS_DDIV(a, b) ((double)(a) / (double)(b))
#endif

constexpr int kSampleMaxK = 1024;       // top_k limit of the device selection (its per-row merge sorts <= 1024 keys)
constexpr int kSampleMaxWindow = 256;   // repeat_last_n limit
constexpr int kMtWords = 625;           // std::mt19937: 624 state words + the index of the next one

NS_HD float ns_bits_float(uint32_t u) {
  float f;
  memcpy(&f, &u, 4);
  return f;
}
NS_HD uint32_t ns_float_bits(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}

// exp(x) in IEEE fp32 operations: x = n ln2 + r with n = rint(x log2 e) and |r| <= ln2 / 2 (ln2 split in a 16-bit head, so
// n * head is exact for every n that reaches here), exp(r) = 1 + (r + r^2 q(r)), q the Taylor series to r^5 / 7!, and 2^n applied
// to the exponent field -- through an exact multiply by 2^(n + 100) and one rounding multiply by 2^-100 for subnormal results.
NS_HD float ns_sample_expf(float x) {
  if (x != x) return x;
  if (x > 88.72283935546875f) return ns_bits_float(0x7f800000u);
  if (x < -103.972084045410156f) return 0.f;
  const float n = rintf(NS_FMUL(x, 1.44269502162933349609f));
  float r = fmaf(-n, 0.693145751953125f, x);
  r = fmaf(-n, 1.42860676533018704e-06f, r);
  float q = 1.98412698412698413e-4f;  // 1/5040
  q = fmaf(q, r, 1.38888888888888889e-3f);
  q = fmaf(q, r, 8.33333333333333333e-3f);
  q = fmaf(q, r, 4.16666666666666667e-2f);
  q = fmaf(q, r, 1.66666666666666667e-1f);
  q = fmaf(q, r, 0.5f);
  const float s = fmaf(NS_FMUL(q, r), r, r);
  const float p = NS_FADD(1.f, s);
  const int ni = (int)n;
  if (ni > 127) return NS_FMUL(NS_FMUL(p, ns_bits_float(254u << 23)), ns_bits_float((uint32_t)ni << 23));  // 2^127 2^(ni - 127)
  if (ni >= -126) return NS_FMUL(p, ns_bits_float((uint32_t)(ni + 127) << 23));
  return NS_FMUL(NS_FMUL(p, ns_bits_float((uint32_t)(ni + 100 + 127) << 23)), ns_bits_float((uint32_t)(-100 + 127) << 23));
}

// step 2, one candidate in the window: model_sample_repetition_penalty (model_utils.cpp:822-826)
NS_HD float ns_sample_penalize(float l, float penalty) { return l <= 0.f ? NS_FMUL(l, penalty) : NS_FDIV(l, penalty); }

// the selection order: logit descending, id ascending among equal logits (+0 and -0 are equal logits, as for operator>).
// One 64-bit key per candidate, larger = earlier; keys are never 0 (a free padding value).
NS_HD uint64_t ns_sample_key(float v, int id) {
  uint32_t u = ns_float_bits(v);
  if (u == 0x80000000u) u = 0;
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((uint64_t)u << 32) | (uint32_t)(0xffffffffu - (uint32_t)id);
}
NS_HD float ns_sample_key_value(uint64_t key) {
  uint32_t u = (uint32_t)(key >> 32);
  u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
  return ns_bits_float(u);
}
NS_HD int ns_sample_key_id(uint64_t key) { return (int)(0xffffffffu - (uint32_t)key); }

// model_sample_softmax (model_utils.cpp:533-542) on l[0 .. n), sorted descending: p = exp(l - l[0]) / sequential sum
NS_HD void ns_sample_softmax(const float* l, float* p, int n) {
  const float mx = l[0];
  float sum = 0.f;
  for (int i = 0; i < n; ++i) {
    p[i] = ns_sample_expf(NS_FSUB(l[i], mx));
    sum = NS_FADD(sum, p[i]);
  }
  for (int i = 0; i < n; ++i) p[i] = NS_FDIV(p[i], sum);
}

// steps 5-7 on the top-k list l[0 .. K) (logits after the penalty, in selection order): top-p (model_sample_top_p, :572-602,
// min_keep 1: the first i >= 1 whose running sum passes top_p is dropped with everything after it), temperature on the kept
// entries (:719-729), and model_sample_token's softmax (:974).  Returns the kept count n; l[0 .. n) ends divided by temp and
// p[0 .. n) holds the final probabilities.
NS_HD int ns_sample_tail(float* l, float* p, int K, float top_p, float temp) {
  int n = K;
  if (top_p < 1.f) {
    ns_sample_softmax(l, p, K);
    float cum = 0.f;
    for (int i = 0; i < K; ++i) {
      cum = NS_FADD(cum, p[i]);
      if (cum > top_p && i >= 1) {
        n = i;
        break;
      }
    }
  }
  for (int i = 0; i < n; ++i) l[i] = NS_FDIV(l[i], temp);
  ns_sample_softmax(l, p, n);
  return n;
}

// std::discrete_distribution<>(p, p + n) (GCC 13 libstdc++, bits/random.tcc _M_initialize): the probabilities as double, divided
// by their sequential sum, partial sums, the last set to 1.  Lists of fewer than two entries keep no table (cp untouched).
NS_HD void ns_sample_cumulative(const float* p, int n, double* cp) {
  if (n < 2) return;
  double sum = 0.0;
  for (int i = 0; i < n; ++i) sum = NS_DADD(sum, (double)p[i]);
  double acc = 0.0;
  for (int i = 0; i < n; ++i) {
    acc = NS_DADD(acc, NS_DDIV((double)p[i], sum));
    cp[i] = acc;
  }
  cp[n - 1] = 1.0;
}

// std::mt19937: seed (mersenne_twister_engine::seed), twist, tempered output; mt[624] is the index of the next word
NS_HD void ns_mt_seed(uint32_t seed, uint32_t* mt) {
  mt[0] = seed;
  for (uint32_t i = 1; i < 624; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + i;
  mt[624] = 624;
}
NS_HD uint32_t ns_mt_next(uint32_t* mt) {
  if (mt[624] >= 624) {
    for (int i = 0; i < 624; ++i) {
      const uint32_t y = (mt[i] & 0x80000000u) | (mt[i + 1 < 624 ? i + 1 : 0] & 0x7fffffffu);
      mt[i] = mt[i + 397 < 624 ? i + 397 : i + 397 - 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    mt[624] = 0;
  }
  uint32_t y = mt[mt[624]++];
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= y >> 18;
  return y;
}

// the draw of std::discrete_distribution::operator(): no table (n < 2) returns 0 without touching the generator; otherwise
// u = generate_canonical<double, 53> (two 32-bit outputs, (x0 + x1 2^32) / 2^64, 1 - 2^-53 if that rounds to 1) and the pick is
// lower_bound(cp, cp + n, u)
NS_HD int ns_sample_pick(const double* cp, int n, uint32_t* mt) {
  if (n < 2) return 0;
  const uint32_t x0 = ns_mt_next(mt);
  const uint32_t x1 = ns_mt_next(mt);
  const double s = NS_DADD((double)x0, NS_DMUL((double)x1, 4294967296.0));
  double u = NS_DMUL(s, 5.42101086242752217e-20);  // 2^-64, exact
  if (u >= 1.0) u = 0.99999999999999988898;          // nextafter(1.0, 0.0)
  int lo = 0, len = n;
  while (len > 0) {
    const int half = len >> 1;
    if (cp[lo + half] < u) {
      lo += half + 1;
      len -= half + 1;
    } else {
      len = half;
    }
  }
  return lo;
}

#ifdef __CUDACC__
// ---- the device sampler (sample.cu), one launch in place of the eval step's argmax ------------------------------------------
// one entry of the per-sequence sampler's parameter table; greedy is {1, 1, 1, 1, 0}: one candidate, no penalty, no window
struct SampleCfg {
  int k;            // top_k, 1 .. kSampleMaxK
  float top_p, temp, penalty;
  int W;            // window length (0: no penalty, no window kept)
};
struct SampleLaunch {  // grid (kVocabSlices, rows): each CTA selects the top k of one slice of the vocabulary
  const float* logits;  // [rows][n_vocab]
  int n_vocab, rows;
  int k;                // top_k, 1 .. kSampleMaxK
  float top_p, temp, penalty;
  int W;                // window length (0: no penalty)
  int* win;             // stored windows: slot s at win + s * win_stride, W ids, oldest first
  int win_stride;
  const int* toks;      // row r's tokens of this pass: toks[r * tok_stride + t], t < tok_len ...
  int tok_stride, tok_len;
  const int* last;      // ... or, when non-null, toks[first_r .. last[r]] with first_r = r ? last[r - 1] + 1 : 0
  const int* slot;      // window slot of row r: slot[r], or slot_const when null (r itself when slot_const < 0)
  int slot_const;
  const int* order;     // caller index i is row order[i] (null: i); rows draw in caller order
  int store;            // write the windows back (0: a pass that will be evaluated again)
  int draw;             // draw from the generator (0: take the first entry and leave the generator alone)
  uint32_t* mt;         // [kMtWords]
  // scratch: slice candidates [rows][kVocabSlices][k] and their counts, cumulative tables [rows][k], tickets [rows + 1] (zero)
  unsigned long long* pkeys;
  int* pcnt;
  double* cp;
  unsigned* tickets;
  int* kept;            // [rows]
  int* ids;             // [rows][k]
  float* probs;         // [rows][k]
  int* picks;           // nullable [rows]
  // as argmax_kernel: state (nullable) row r at state + 4 r when rowwise; state[3] = pick; when advance: state[0] = pick,
  // state[1] += n_tokens, record[r * rec_stride + state[2]++] = pick
  int* state;
  int rowwise, n_tokens, advance;
  int* record;
  int rec_stride;
  // non-null: the per-sequence sampler.  Row r's slot s (as its window's) selects its parameters cfg[s] and its generator
  // mt + s kMtWords; k, top_p, temp, penalty and W above are not read, k is the stride of the scratch rows (>= every cfg k)
  // and the window is the last cfg[s].W of the win_stride entries at win + s win_stride.  Each row draws in its own last CTA;
  // order is not read.
  const SampleCfg* cfg;
};
int ns_launch_sample(const SampleLaunch& a, cudaStream_t st);  // counts its launch
int ns_sample_check(const char* who, const struct ns_llama_sampling* s);
// the table entry of a checked config, its window min(repeat_last_n, max_window); greedy for null
SampleCfg ns_sample_cfg(const struct ns_llama_sampling* s, int max_window);
#endif

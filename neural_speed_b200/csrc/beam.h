// beam.h -- the stated arithmetic of beam search's per-row candidates (the reference's logits_info and vocab_top_k,
// model_utils.cpp:2139-2211, used by beam_top_k_next_tokens, :2312-2376), compiled once for the host and once for the device so
// ns_beam_candidates_row_host and beam_candidates_kernel (beam.cu) run the same operations in the same order; and the flow's
// interface to the engine.
//
// One row x[0 .. n) with a prior score `prev`, and `mask` set when the row's generated length is below min_new_tokens (never on the
// first step, whose min_new_tokens is the reference's input default 0):
//   M, S       the row's max and sum of exp(x - M) over the RAW logits: logprob.h's M and S (ns_logprob_stats_host; M and S are
//              taken before the mask, as logits_info's constructor runs before logits_processor::process, model_utils.cpp:2319-2326)
//   x'         x with x'[eos] = -FLT_MAX when mask (model_utils.cpp:2228, NEG_INF)
//   selection  the K = min(k, n) largest x', logit descending and id ascending among equal logits (ns_sample_key)
//   score      logf(norm * expf(x' - M)) + prev with norm = 1 / S, every operation in fp32 (log_probability_from_logit, :2180-2186)
// The deviations from the reference are the order of S (the reference sums sequentially), the exp and the log (ns_sample_expf,
// ns_logf: each within 1 ulp of glibc), and the tie rules (the reference's heap order among equal values is unspecified).
#pragma once
#include <float.h>

#include <vector>

#include "logprob.h"

constexpr int kBeamMaxBeams = 32;               // num_beams limit: every beam of every request has a KV block
constexpr int kBeamMaxRows = 32;                // rows of one candidates launch
constexpr int kBeamMaxK = 2 * kBeamMaxBeams;    // candidates per row (sample_scale 2)

struct BeamCand {  // one candidate of a row: token id and its score (log-probability plus the row's prior score)
  int32_t id;
  float score;
};

NS_HD float ns_beam_masked(float x, int id, int eos, int mask) { return mask && id == eos ? -FLT_MAX : x; }
NS_HD float ns_beam_score(float x, float M, float norm, float prev) {
  return NS_FADD(ns_logf(NS_FMUL(norm, ns_sample_expf(NS_FSUB(x, M)))), prev);
}

// the KV copy: pair j copies positions [p0[j], p1[j]) of block src[j] into block dst[j], every layer, K and V
struct KvCopyPairs {
  int n = 0;
  int src[kBeamMaxRows], dst[kBeamMaxRows], p0[kBeamMaxRows], p1[kBeamMaxRows];
};

#ifdef __CUDACC__
#include <cuda_fp16.h>

#include "kv_cache.cuh"
// ---- the device kernels (beam.cu) ------------------------------------------------------------------------------------------
struct BeamLaunch {  // beam_candidates_kernel: grid (kVocabSlices, rows), kLogprobThreads threads, one launch per beam step
  const float* logits;  // [rows][n_vocab]
  int n_vocab, rows;    // 1 <= rows <= kBeamMaxRows
  int k;                // 1 .. kBeamMaxK
  int eos;
  unsigned mask;        // bit r: row r's EOS logit is -FLT_MAX
  float prev[kBeamMaxRows];
  BeamCand* out;        // [rows][min(k, n_vocab)]
  // scratch: tickets [rows] (zero, and zero again after the launch) | max, sum, count [rows][slices] | keys [rows][slices][k]
  unsigned* tickets;
  float* pmax;
  float* psum;
  int* pcnt;
  unsigned long long* pkeys;
};
int ns_launch_beam_candidates(const BeamLaunch& a, cudaStream_t st);  // counts its launch
size_t ns_beam_scratch_bytes(int rows, int k);                          // the scratch after the tickets
void ns_beam_scratch(BeamLaunch& a, void* scratch, int rows, int k);    // points pmax .. pkeys into it
// one launch for all pairs; refuses (NS_E_INVALID, nothing launched) a pair list in which a destination is also a source or
// appears twice, a block outside [0, n_seq) or a range outside [0, n_ctx); counts its launch.  kv: the caches from layer 0, block 0
int ns_launch_kv_copy(const KvCopyPairs& a, const KvPtrs& kv, int n_layer, int n_seq, int n_head_kv, int n_ctx, int hd, cudaStream_t st);
#endif

// ---- the flow (beam.cu): beam_search_flow::loop restated over an engine ------------------------------------------------------
struct BeamRows {  // the rows of one pass, in order (requests ascending, beams ascending)
  int n = 0;
  int req[kBeamMaxRows], block[kBeamMaxRows], n_past[kBeamMaxRows];
  int32_t tok[kBeamMaxRows];                       // the token evaluated (a prompt's last token on the prompt pass)
  float prev[kBeamMaxRows];                        // the row's prior score
  int mask[kBeamMaxRows];                          // EOS forbidden on this row
  const std::vector<int32_t>* gen[kBeamMaxRows];   // the row's generated tokens, tok last (empty on the prompt pass)
};
struct BeamEngine {
  // the prompt pass (row r: request r into block r B): K candidates of each prompt's last row
  virtual int prompts(const BeamRows& rows, int K, BeamCand* out) = 0;
  // one decode pass over the running beams: K candidates per row
  virtual int step(const BeamRows& rows, int K, BeamCand* out) = 0;
  // KV copies, one launch
  virtual int copy(const KvCopyPairs& pairs) = 0;
  virtual ~BeamEngine() {}
};
// checks cfg and the prompt lengths against n_ctx / n_vocab / n_seq (NS_E_INVALID with the reason set), nothing else
int ns_beam_check(const char* who, const struct ns_llama_beams* cfg, int n, const int* n_tokens, int n_ctx, int n_vocab, int n_seq);
// the flow over n requests (prompt r: n_tokens[r] tokens at tokens + sum of the earlier lengths); outputs as ns_llama_beam_search
int ns_beam_flow(const struct ns_llama_beams& cfg, int n, const int* n_tokens, const int32_t* tokens, BeamEngine& eng,
                 int32_t* out_tokens, int* out_len, float* out_score);

// beam.cu -- beam search (the reference's beam_search_flow, model_utils.cpp:2139-2766): the per-row candidates kernel and its host
// restatement, the KV block copy, and the flow itself in host C++ over an engine (the device one is in llama.cu, a host one with a
// caller's logits here).
//
// beam_candidates_kernel: grid (kVocabSlices, rows), kLogprobThreads threads, on the slice reductions of vocab_slices.cuh.  Each
// CTA takes its slice's max and sum of exp(x - max) as logprob_kernel does (slice_argmax, slice_expsum) and its top K keys of the
// masked logits (masked logit descending, id ascending: ns_sample_key; slice_top_keys); the row's last CTA merges the slices' max
// and sums in slice order, takes the row's top K over the partials, sorted (row_top_keys), and writes {id, score}.  beam.h states
// the arithmetic.
//
// kv_copy_kernel: grid (chunks, layer x KV head x {K, V}, pairs); a (layer, head) range of positions is contiguous in the
// [layer][seq][kv head][n_ctx][hd] fp16 cache, copied in 16-byte vectors.  On a Q8_0 cache (kv_cache.cuh) grid y runs over
// layer x KV head x {K codes, V codes, K scales, V scales}: the codes in 16-byte vectors, the scales (hd / 32 halves per row,
// 4-byte aligned) in 4-byte words.
#include "nsb.cuh"
#include "beam.h"
#include "kv_cache.cuh"
#include "vocab_slices.cuh"

#include <algorithm>
#include <cmath>
#include <numeric>
#include <vector>

namespace {

__global__ void __launch_bounds__(kLogprobThreads) beam_candidates_kernel(const BeamLaunch a) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_max, s_norm;
  __shared__ uint64_t sk[kBeamMaxK];
  const int row = blockIdx.y, tid = threadIdx.x, n = a.n_vocab, slot = row * kVocabSlices + blockIdx.x;
  const VocabSlice sl = vocab_slice(n, blockIdx.x);
  const float* x = a.logits + (size_t)row * n;
  const int mask = (a.mask >> row) & 1, K = min(a.k, n);
  // the slice's max and sum of the raw logits (logprob_kernel's)
  float best;
  int bi;
  slice_argmax<kLogprobThreads>(x, sl.lo, sl.hi, best, bi);
  const float sum = slice_expsum<kLogprobThreads>(x, sl.lo, sl.hi, best);
  if (tid == 0) {
    a.pmax[slot] = best;
    a.psum[slot] = sum;
  }
  // the slice's top keys of the masked logits
  slice_top_keys<kLogprobThreads>(
      [&](int j) {
        const int i = sl.lo + j;
        return ns_sample_key(ns_beam_masked(x[i], i, a.eos, mask), i);
      },
      sl.hi - sl.lo, K, a.pkeys + (size_t)slot * a.k, a.pcnt + slot);
  if (!last_of_row(a.tickets, row)) return;

  // ---- the row's last CTA: M, S in slice order; the top K of the partials, sorted ----
  row_top_keys<kLogprobThreads>(a.pkeys + (size_t)row * kVocabSlices * a.k, a.pcnt + row * kVocabSlices, a.k, K, sk);
  if (tid == 0) {
    const volatile float* pm = a.pmax + row * kVocabSlices;
    float M = -INFINITY;
    for (int s = 0; s < kVocabSlices; ++s) M = pm[s] > M ? pm[s] : M;
    s_max = M;
    s_norm = __fdiv_rn(1.f, merge_slice_sums((const volatile float*)a.psum + row * kVocabSlices, pm, M));
    a.tickets[row] = 0u;  // ready for the next launch
  }
  __syncthreads();
  const float M = s_max, norm = s_norm, prev = a.prev[row];
  for (int i = tid; i < K; i += kLogprobThreads) {
    BeamCand c;
    c.id = ns_sample_key_id(sk[i]);
    c.score = ns_beam_score(ns_sample_key_value(sk[i]), M, norm, prev);
    a.out[(size_t)row * K + i] = c;
  }
}

template <int KV = NS_KV_F16>
__global__ void __launch_bounds__(256) kv_copy_kernel(const KvCopyPairs a, kv_elem_t<KV>* __restrict__ kc, kv_elem_t<KV>* __restrict__ vc,
                                                      int n_seq, int n_head_kv, int n_ctx, int hd, __half* __restrict__ kd,
                                                      __half* __restrict__ vd) {
  pdl_launch_dependents();
  pdl_wait();
  if constexpr (KV == NS_KV_Q8_0) {
    const int pr = blockIdx.z, lh = blockIdx.y >> 2, plane = blockIdx.y & 3, layer = lh / n_head_kv, h = lh % n_head_kv;
    const size_t us = ((size_t)layer * n_seq + a.src[pr]) * n_head_kv + h, ud = ((size_t)layer * n_seq + a.dst[pr]) * n_head_kv + h;
    const int p0 = a.p0[pr], rows = a.p1[pr] - a.p0[pr];
    if (plane < 2) {
      int8_t* base = plane ? vc : kc;
      const int4* src = reinterpret_cast<const int4*>(base + us * n_ctx * hd + (size_t)p0 * hd);
      int4* dst = reinterpret_cast<int4*>(base + ud * n_ctx * hd + (size_t)p0 * hd);
      const int n16 = rows * hd / 16;
      for (int i = blockIdx.x * 256 + threadIdx.x; i < n16; i += gridDim.x * 256) dst[i] = src[i];
    } else {
      __half* base = plane == 3 ? vd : kd;
      const size_t ds = kv_d_stride(n_ctx, hd);
      const uint32_t* src = reinterpret_cast<const uint32_t*>(base + us * ds + (size_t)p0 * (hd / kKvQ8Block));
      uint32_t* dst = reinterpret_cast<uint32_t*>(base + ud * ds + (size_t)p0 * (hd / kKvQ8Block));
      const int n4 = rows * (hd / kKvQ8Block) / 2;
      for (int i = blockIdx.x * 256 + threadIdx.x; i < n4; i += gridDim.x * 256) dst[i] = src[i];
    }
  } else {
  const int pr = blockIdx.z, lh = blockIdx.y >> 1, layer = lh / n_head_kv, h = lh % n_head_kv;
  __half* base = (blockIdx.y & 1) ? vc : kc;
  auto at = [&](int blk, int pos) { return base + (((size_t)layer * n_seq + blk) * n_head_kv + h) * n_ctx * hd + (size_t)pos * hd; };
  const int4* src = reinterpret_cast<const int4*>(at(a.src[pr], a.p0[pr]));
  int4* dst = reinterpret_cast<int4*>(at(a.dst[pr], a.p0[pr]));
  const int n16 = (a.p1[pr] - a.p0[pr]) * hd / 8;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < n16; i += gridDim.x * 256) dst[i] = src[i];
  }
}

}  // namespace

size_t ns_beam_scratch_bytes(int rows, int k) {
  return (size_t)rows * kVocabSlices * 12 + (size_t)rows * kVocabSlices * k * 8;
}

void ns_beam_scratch(BeamLaunch& a, void* scratch, int rows, int k) {
  char* w = static_cast<char*>(scratch);
  a.pkeys = reinterpret_cast<unsigned long long*>(w);  // 8-byte aligned first
  w += (size_t)rows * kVocabSlices * k * 8;
  a.pmax = reinterpret_cast<float*>(w);
  a.psum = a.pmax + (size_t)rows * kVocabSlices;
  a.pcnt = reinterpret_cast<int*>(a.psum + (size_t)rows * kVocabSlices);
}

int ns_launch_beam_candidates(const BeamLaunch& a, cudaStream_t st) {
  NS_CUDA_TRY(ns_launch_pdl(beam_candidates_kernel, dim3((unsigned)kVocabSlices, (unsigned)a.rows), dim3(kLogprobThreads), 0, st, a));
  ns_count_launch();
  return NS_OK;
}

int ns_launch_kv_copy(const KvCopyPairs& a, const KvPtrs& kv, int n_layer, int n_seq, int n_head_kv, int n_ctx, int hd, cudaStream_t st) {
  if (a.n < 1 || a.n > kBeamMaxRows || a.n > n_seq) {
    ns_set_error("ns_llama_kv_copy: %d pairs (1 .. %d)", a.n, std::min(n_seq, kBeamMaxRows));
    return NS_E_INVALID;
  }
  int longest = 0;
  for (int i = 0; i < a.n; ++i) {
    if (a.src[i] < 0 || a.src[i] >= n_seq || a.dst[i] < 0 || a.dst[i] >= n_seq || a.p0[i] < 0 || a.p0[i] > a.p1[i] || a.p1[i] > n_ctx) {
      ns_set_error("ns_llama_kv_copy: pair %d (block %d -> %d, positions [%d, %d)) outside %d blocks of %d positions", i, a.src[i], a.dst[i],
                   a.p0[i], a.p1[i], n_seq, n_ctx);
      return NS_E_INVALID;
    }
    for (int j = 0; j < a.n; ++j)
      if (a.dst[i] == a.src[j] || (j != i && a.dst[i] == a.dst[j])) {
        ns_set_error("ns_llama_kv_copy: block %d is written by pair %d and %s by pair %d (pairs run in parallel)", a.dst[i], i,
                     a.dst[i] == a.src[j] ? "read" : "written", j);
        return NS_E_INVALID;
      }
    longest = std::max(longest, a.p1[i] - a.p0[i]);
  }
  const int n16 = longest * hd / 8;
  if (n16 == 0) return NS_OK;  // nothing to copy
  const unsigned gx = (unsigned)std::min((n16 + 255) / 256, 16);
  if (kv.type == NS_KV_Q8_0)
    NS_CUDA_TRY(ns_launch_pdl(kv_copy_kernel<NS_KV_Q8_0>, dim3(gx, (unsigned)(n_layer * n_head_kv * 4), (unsigned)a.n), dim3(256), 0, st, a,
                              static_cast<int8_t*>(kv.k), static_cast<int8_t*>(kv.v), n_seq, n_head_kv, n_ctx, hd, kv.kd, kv.vd));
  else
    NS_CUDA_TRY(ns_launch_pdl(kv_copy_kernel<>, dim3(gx, (unsigned)(n_layer * n_head_kv * 2), (unsigned)a.n), dim3(256), 0, st, a,
                              static_cast<__half*>(kv.k), static_cast<__half*>(kv.v), n_seq, n_head_kv, n_ctx, hd, (__half*)nullptr,
                              (__half*)nullptr));
  ns_count_launch();
  return NS_OK;
}

// ---- host restatement ------------------------------------------------------------------------------------------------------
static void candidates_row_host(const float* x, int n, int k, float prev, int mask, int eos, BeamCand* out) {
  float M, S;
  int I;
  ns_logprob_stats_host(x, n, &M, &I, &S);
  const float norm = NS_FDIV(1.f, S);
  const int K = std::min(k, n);
  std::vector<uint64_t> key(n);
  for (int i = 0; i < n; ++i) key[i] = ns_sample_key(ns_beam_masked(x[i], i, eos, mask), i);
  std::partial_sort(key.begin(), key.begin() + K, key.end(), [](uint64_t u, uint64_t v) { return u > v; });
  for (int i = 0; i < K; ++i) {
    out[i].id = ns_sample_key_id(key[i]);
    out[i].score = ns_beam_score(ns_sample_key_value(key[i]), M, norm, prev);
  }
}

extern "C" int ns_beam_candidates_row_host(const float* logits, int n_vocab, int k, float prev, int mask, int32_t eos, int32_t* ids,
                                           float* scores) {
  if (!logits || !ids || !scores || n_vocab < 1 || k < 1 || k > kBeamMaxK) {
    ns_set_error("ns_beam_candidates_row_host: invalid arguments (n_vocab %d k %d, or a null pointer)", n_vocab, k);
    return NS_E_INVALID;
  }
  std::vector<BeamCand> c(std::min(k, n_vocab));
  candidates_row_host(logits, n_vocab, k, prev, mask, eos, c.data());
  for (size_t i = 0; i < c.size(); ++i) {
    ids[i] = c[i].id;
    scores[i] = c[i].score;
  }
  return NS_OK;
}

extern "C" float ns_logf_host(float x) { return ns_logf(x); }

// ---- parity entry --------------------------------------------------------------------------------------------------------
// workspace: tickets [kBeamMaxRows] (the first 128 bytes for every n and k) | scratch (ns_beam_scratch)
extern "C" size_t ns_llama_beam_candidates_workspace_bytes(int n, int k) {
  if (n < 1 || n > kBeamMaxRows || k < 1 || k > kBeamMaxK) return 0;
  return (size_t)kBeamMaxRows * 4 + ns_beam_scratch_bytes(n, k);
}

extern "C" int ns_llama_beam_candidates(const float* logits, int n, int n_vocab, int k, const float* prev, const int* mask, int32_t eos,
                                        void* out, void* ws, void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!logits || !prev || !mask || !out || !ws || n < 1 || n > kBeamMaxRows || n_vocab < 1 || k < 1 || k > kBeamMaxK) {
    ns_set_error("ns_llama_beam_candidates: invalid arguments (n %d n_vocab %d k %d, or a null pointer)", n, n_vocab, k);
    return NS_E_INVALID;
  }
  BeamLaunch a{};
  a.logits = logits;
  a.n_vocab = n_vocab;
  a.rows = n;
  a.k = k;
  a.eos = eos;
  for (int r = 0; r < n; ++r) {
    a.prev[r] = prev[r];
    if (mask[r]) a.mask |= 1u << r;
  }
  a.out = static_cast<BeamCand*>(out);
  a.tickets = static_cast<unsigned*>(ws);
  ns_beam_scratch(a, static_cast<char*>(ws) + kBeamMaxRows * 4, n, k);
  return ns_launch_beam_candidates(a, ns_stream_of(queue));
}

// ---- the flow ------------------------------------------------------------------------------------------------------------
int ns_beam_check(const char* who, const ns_llama_beams* cfg, int n, const int* n_tokens, int n_ctx, int n_vocab, int n_seq) {
  const int B = cfg->num_beams;
  if (B < 2 || B > kBeamMaxBeams || cfg->max_new_tokens < 1 || cfg->min_new_tokens < 0 || !std::isfinite(cfg->length_penalty) ||
      (cfg->early_stopping != 0 && cfg->early_stopping != 1) || cfg->eos_token_id < 0 || cfg->eos_token_id >= n_vocab || 2 * B > n_vocab) {
    ns_set_error("%s: num_beams %d max_new_tokens %d min_new_tokens %d length_penalty %g early_stopping %d eos %d: need 2 <= num_beams "
                 "<= %d, 2 num_beams <= n_vocab %d, max_new_tokens >= 1, min_new_tokens >= 0, a finite length_penalty, early_stopping "
                 "0 / 1 and eos in [0, n_vocab)",
                 who, B, cfg->max_new_tokens, cfg->min_new_tokens, cfg->length_penalty, cfg->early_stopping, cfg->eos_token_id,
                 kBeamMaxBeams, n_vocab);
    return NS_E_INVALID;
  }
  if (n < 1 || (long long)n * B > n_seq) {
    ns_set_error("%s: %d requests of %d beams need %lld KV blocks, %d available", who, n, B, (long long)n * B, n_seq);
    return NS_E_INVALID;
  }
  for (int r = 0; r < n; ++r)
    if (n_tokens[r] < 1 || (long long)n_tokens[r] + cfg->max_new_tokens - 1 > n_ctx) {
      ns_set_error("%s: prompt %d of %d tokens and %d new tokens: need 1 <= n_tokens and n_tokens + max_new_tokens - 1 <= n_ctx %d", who, r,
                   n_tokens[r], cfg->max_new_tokens, n_ctx);
      return NS_E_INVALID;
    }
  return NS_OK;
}

namespace {
struct Beam {
  std::vector<int32_t> tok;  // generated tokens
  float score;
  int block;
};
struct Hyp {
  std::vector<int32_t> tok;
  float score;
  long long seq;  // order of addition
};
struct Cand {
  int32_t id;
  float score;
  int beam;
};
// the tie rules: candidates by (score descending, beam ascending, id ascending); hypotheses by score, a later one first
bool cand_before(const Cand& a, const Cand& b) {
  if (a.score != b.score) return a.score > b.score;
  if (a.beam != b.beam) return a.beam < b.beam;
  return a.id < b.id;
}
bool hyp_above(const Hyp& a, const Hyp& b) { return a.score != b.score ? a.score > b.score : a.seq > b.seq; }
}  // namespace

int ns_beam_flow(const ns_llama_beams& cfg, int n, const int* n_tokens, const int32_t* tokens, BeamEngine& eng, int32_t* out_tokens,
                 int* out_len, float* out_score) {
  const int B = cfg.num_beams, K = 2 * B, T = cfg.max_new_tokens;
  const int32_t eos = cfg.eos_token_id;
  std::vector<int> off(n, 0);
  for (int r = 1; r < n; ++r) off[r] = off[r - 1] + n_tokens[r - 1];
  std::vector<std::vector<Beam>> beams(n);
  std::vector<std::vector<Hyp>> hyps(n);
  std::vector<char> done(n, 0);
  std::vector<KvCopyPairs> pend(n);  // each request's KV copies before its next pass
  std::vector<BeamCand> cand((size_t)kBeamMaxRows * kBeamMaxK);
  long long seq = 0;
  // beam_hypotheses::add (model_utils.h:339-368): score / cur_len ^ length_penalty in double (std::pow of an unsigned and a float),
  // rounded to float; the B best kept
  auto add = [&](int r, const std::vector<int32_t>& tok, float score) {
    const unsigned cur_len = !tok.empty() && tok.back() == eos ? (unsigned)tok.size() - 1 : (unsigned)tok.size();
    hyps[r].push_back(Hyp{tok, (float)((double)score / std::pow((double)cur_len, (double)cfg.length_penalty)), seq++});
    if ((int)hyps[r].size() > B)
      hyps[r].erase(std::min_element(hyps[r].begin(), hyps[r].end(), [](const Hyp& a, const Hyp& b) { return hyp_above(b, a); }));
  };
  auto is_done = [&](int r) { return (int)hyps[r].size() >= B && cfg.early_stopping; };
  // update_status and finalize (model_utils.cpp:2622-2674)
  auto update_status = [&]() {
    for (int r = 0; r < n; ++r) {
      if (done[r]) continue;
      if (!is_done(r) && (int)beams[r][0].tok.size() != T) continue;
      done[r] = 1;
      if (!is_done(r))
        for (const Beam& b : beams[r]) add(r, b.tok, b.score);
      const Hyp& top = *std::max_element(hyps[r].begin(), hyps[r].end(), [](const Hyp& a, const Hyp& b) { return hyp_above(b, a); });
      std::copy(top.tok.begin(), top.tok.end(), out_tokens + (size_t)r * T);
      out_len[r] = (int)top.tok.size();
      if (out_score) out_score[r] = top.score;
    }
  };
  static const std::vector<int32_t> none;
  // first step (loop, :2688-2731): the prompts, then the top B of each prompt's last row, prior score 0.  No EOS mask: this step's
  // logits_processor reads min_new_tokens from the caller's inputs (:2323 with next_inputs = inputs, :2679), which
  // Model::beam_generate builds without a gen_conf (application/main_pybind.cpp:528-538), so it is generation_config{}'s 0
  // (model_types.h:283); the later steps read ctx->generation_conf (:2410, :2691)
  BeamRows rows;
  rows.n = n;
  for (int r = 0; r < n; ++r) {
    rows.req[r] = r;
    rows.block[r] = r * B;
    rows.n_past[r] = 0;
    rows.tok[r] = tokens[off[r] + n_tokens[r] - 1];
    rows.prev[r] = 0.f;
    rows.mask[r] = 0;
    rows.gen[r] = &none;
  }
  if (int rc = eng.prompts(rows, B, cand.data())) return rc;
  for (int r = 0; r < n; ++r) {
    std::vector<Cand> c(B);
    for (int i = 0; i < B; ++i) c[i] = Cand{cand[(size_t)r * B + i].id, cand[(size_t)r * B + i].score, 0};
    std::sort(c.begin(), c.end(), cand_before);
    beams[r].resize(B);
    for (int i = 0; i < B; ++i) beams[r][i] = Beam{{c[i].id}, c[i].score, r * B + i};
    KvCopyPairs& p = pend[r];  // the prompt into the other beams' blocks (beam_search_kv_cache_reorder::update, :2253-2260)
    for (int i = 1; i < B; ++i) {
      p.src[p.n] = r * B;
      p.dst[p.n] = r * B + i;
      p.p0[p.n] = 0;
      p.p1[p.n++] = n_tokens[r];
    }
  }
  update_status();
  for (int step = 1; step < T; ++step) {
    // the copies of the running requests, one launch
    KvCopyPairs all;
    for (int r = 0; r < n; ++r) {
      if (!done[r])
        for (int j = 0; j < pend[r].n; ++j) {
          all.src[all.n] = pend[r].src[j];
          all.dst[all.n] = pend[r].dst[j];
          all.p0[all.n] = pend[r].p0[j];
          all.p1[all.n++] = pend[r].p1[j];
        }
      pend[r].n = 0;
    }
    if (std::find(done.begin(), done.end(), 0) == done.end()) break;
    if (all.n)
      if (int rc = eng.copy(all)) return rc;
    // fill_next_beams_by_top_scores (:2378-2436): one pass over every running beam
    rows.n = 0;
    for (int r = 0; r < n; ++r)
      for (int i = 0; i < B && !done[r]; ++i) {
        const int j = rows.n++;
        rows.req[j] = r;
        rows.block[j] = beams[r][i].block;
        rows.n_past[j] = n_tokens[r] + step - 1;
        rows.tok[j] = beams[r][i].tok.back();
        rows.prev[j] = beams[r][i].score;
        rows.mask[j] = step < cfg.min_new_tokens;
        rows.gen[j] = &beams[r][i].tok;
      }
    if (int rc = eng.step(rows, K, cand.data())) return rc;
    int row0 = 0;
    for (int r = 0; r < n; ++r) {
      if (done[r]) continue;
      // beam_top_k_next_tokens (:2312-2376): the top 2B of the request's B x 2B candidates
      std::vector<Cand> c;
      c.reserve((size_t)B * K);
      for (int i = 0; i < B; ++i)
        for (int j = 0; j < K; ++j) {
          const BeamCand& x = cand[(size_t)(row0 + i) * K + j];
          c.push_back(Cand{x.id, x.score, i});
        }
      row0 += B;
      std::partial_sort(c.begin(), c.begin() + K, c.end(), cand_before);
      // next_candidate_beams (:2460-2500)
      std::vector<Beam> next;
      std::vector<int> src;
      for (int nt = 0; nt < K && (int)next.size() < B; ++nt) {
        const Beam& from = beams[r][c[nt].beam];
        if (c[nt].id == eos) {
          if (nt < B) add(r, from.tok, c[nt].score);
          continue;
        }
        next.push_back(Beam{from.tok, c[nt].score, -1});
        next.back().tok.push_back(c[nt].id);
        src.push_back(c[nt].beam);
      }
      // ordered by source beam, stable (:2494-2497); the KV blocks: a source's first descendant keeps its block, the others take
      // the blocks of the sources that have none, in source order, and receive the source's generated positions
      std::vector<int> ord(B);
      std::iota(ord.begin(), ord.end(), 0);
      std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return src[a] < src[b]; });
      std::vector<char> kept(B, 0), has(B, 0);
      for (int s : src) has[s] = 1;
      std::vector<int> spare;
      for (int s = 0; s < B; ++s)
        if (!has[s]) spare.push_back(beams[r][s].block);
      std::vector<Beam> nb(B);
      size_t fi = 0;
      KvCopyPairs& p = pend[r];
      for (int i = 0; i < B; ++i) {
        const int s = src[ord[i]];
        nb[i] = std::move(next[ord[i]]);
        if (!kept[s]) {
          kept[s] = 1;
          nb[i].block = beams[r][s].block;
        } else {
          nb[i].block = spare[fi++];
          p.src[p.n] = beams[r][s].block;
          p.dst[p.n] = nb[i].block;
          p.p0[p.n] = n_tokens[r];
          p.p1[p.n++] = n_tokens[r] + step;
        }
      }
      beams[r] = std::move(nb);
    }
    update_status();
  }
  return NS_OK;
}

// ---- the flow without a device -------------------------------------------------------------------------------------------
namespace {
struct HostEngine : BeamEngine {
  int n_vocab;
  const int* n_tokens;
  const int32_t* tokens;
  std::vector<int> off;
  ns_beam_logits_fn fn;
  void* user;
  int eos;
  int run(const BeamRows& rows, int K, BeamCand* out) {
    std::vector<std::vector<int32_t>> h(rows.n);
    std::vector<const int32_t*> hp(rows.n);
    std::vector<int> hl(rows.n), req(rows.req, rows.req + rows.n);
    for (int i = 0; i < rows.n; ++i) {
      const int r = rows.req[i];
      h[i].assign(tokens + off[r], tokens + off[r] + n_tokens[r]);
      h[i].insert(h[i].end(), rows.gen[i]->begin(), rows.gen[i]->end());
      hp[i] = h[i].data();
      hl[i] = (int)h[i].size();
    }
    std::vector<float> lg((size_t)rows.n * n_vocab);
    if (int rc = fn(user, rows.n, req.data(), hp.data(), hl.data(), lg.data())) {
      ns_set_error("ns_beam_search_host: the logits callback returned %d", rc);
      return rc < 0 ? rc : NS_E_INVALID;
    }
    for (int i = 0; i < rows.n; ++i)
      candidates_row_host(lg.data() + (size_t)i * n_vocab, n_vocab, K, rows.prev[i], rows.mask[i], eos, out + (size_t)i * K);
    return NS_OK;
  }
  int prompts(const BeamRows& rows, int K, BeamCand* out) override { return run(rows, K, out); }
  int step(const BeamRows& rows, int K, BeamCand* out) override { return run(rows, K, out); }
  int copy(const KvCopyPairs&) override { return NS_OK; }
};
}  // namespace

extern "C" int ns_beam_search_host(int n_vocab, int n_ctx, int n, const int* n_tokens, const int32_t* tokens, const ns_llama_beams* cfg,
                                   ns_beam_logits_fn logits, void* user, int32_t* out_tokens, int* out_len, float* out_score) {
  const char* who = "ns_beam_search_host";
  if (!n_tokens || !tokens || !cfg || !logits || !out_tokens || !out_len || n_vocab < 1) {
    ns_set_error("%s: null pointer or n_vocab %d", who, n_vocab);
    return NS_E_INVALID;
  }
  if (int rc = ns_beam_check(who, cfg, n, n_tokens, n_ctx, n_vocab, kBeamMaxRows)) return rc;
  HostEngine e;
  e.n_vocab = n_vocab;
  e.n_tokens = n_tokens;
  e.tokens = tokens;
  e.off.assign(n, 0);
  for (int r = 1; r < n; ++r) e.off[r] = e.off[r - 1] + n_tokens[r - 1];
  e.fn = logits;
  e.user = user;
  e.eos = cfg->eos_token_id;
  return ns_beam_flow(*cfg, n, n_tokens, tokens, e, out_tokens, out_len, out_score);
}

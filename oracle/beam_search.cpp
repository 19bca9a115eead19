// beam_search.cpp -- a C++ restatement of the reference's beam search (beam_search -> beam_search_flow::loop,
// neural_speed/models/model_utils/model_utils.cpp:2139-2766 and 2939-2944, beam_hypotheses in model_utils.h:288-400), for
// tests/test_beam_cpu.py and tests/test_gpu_beam.py.  model_utils.cpp needs xbyak and the whole engine to compile, so this
// restatement is pinned by reading: it keeps the reference's structures (cur_beams / next_beams indexed request * beam_size + beam,
// beam_hypotheses, logits_info) and calls std::max_element / accumulate / make_heap / pop_heap / push_heap / sort where the
// reference does.  Where the reference's order among equal scores is unspecified (std::sort, heap order) the comparators carry
// the library's tie rules -- candidates by (score descending, beam ascending, id ascending), hypotheses by score with a later one
// first, and a stable sort by beam index -- so the outputs are defined.
//
// The model is a callback: logits(user, rows, req, hist, hist_len, out) gives the logits of each row's last token from its whole
// history (prompt, then generated tokens).  The KV cache reorder of the reference has no counterpart here: each row's history is
// its cache.
//
// Per-row arithmetic: `row` null is the reference's -- glibc expf / logf through std::exp / std::log, a sequential std::accumulate,
// the max and the sum taken before the EOS mask (logits_info's constructor runs before logits_processor::process, :2319-2326).
// `row` non-null is the library's ns_beam_candidates_row_host, whose top-k list replaces vocab_top_k and its scores.
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <limits>
#include <numeric>
#include <vector>

#define ORC_API extern "C" __attribute__((visibility("default")))

typedef int (*logits_fn)(void* user, int rows, const int* req, const int32_t* const* hist, const int* hist_len, float* out);
typedef int (*row_fn)(const float* logits, int n_vocab, int k, float prev, int mask, int32_t eos, int32_t* ids, float* scores);

namespace {

const float NEG_INF = -std::numeric_limits<float>::max();  // model_utils.h:289

struct beam_next_token {
  int32_t id = -1;
  float score = 0.0f;
  int beam_idx = -1;
};
// the tie rule of the candidates: a ranks before b
bool cand_before(const beam_next_token& a, const beam_next_token& b) {
  if (a.score != b.score) return a.score > b.score;
  if (a.beam_idx != b.beam_idx) return a.beam_idx < b.beam_idx;
  return a.id < b.id;
}

struct beam {
  std::vector<int32_t> token_ids;
  float score = 0.0f;
  int request_idx = -1;
  int beam_idx = -1;
  bool done = false;
  long long seq = 0;  // order of addition to the hypotheses (the tie rule)
  bool eos(int32_t eos_id) const { return !token_ids.empty() && token_ids.back() == eos_id; }
};

// model_utils.h:318-388
struct beam_hypotheses {
  int num_beams;
  float length_penalty;
  bool early_stopping;
  int32_t eos_id;
  long long* counter;
  std::vector<beam> beams;
  // a ranks above b: larger score, a later addition among equal scores
  static bool above(const beam& a, const beam& b) { return a.score != b.score ? a.score > b.score : a.seq > b.seq; }
  void add(beam b) {
    auto comp = [](const beam& a, const beam& b) { return above(a, b); };  // reference: a.score > b.score (a min-heap)
    uint32_t cur_len = b.eos(eos_id) ? b.token_ids.size() - 1 : b.token_ids.size();
    float score = b.score / std::pow(cur_len, length_penalty);  // unsigned and float: std::pow in double, the division too
    b.score = score;
    b.seq = (*counter)++;
    if ((int)beams.size() < num_beams) {
      beams.push_back(std::move(b));
      if ((int)beams.size() == num_beams) std::make_heap(beams.begin(), beams.end(), comp);
    } else {
      if (beams.front().score > b.score) return;
      std::pop_heap(beams.begin(), beams.end(), comp);
      beams.back() = b;
      std::push_heap(beams.begin(), beams.end(), comp);
    }
  }
  bool is_done() const { return (int)beams.size() >= num_beams && early_stopping; }
  const beam& top1() const { return *std::max_element(beams.begin(), beams.end(), [](const beam& a, const beam& b) { return above(b, a); }); }
};

struct flow {
  int n_vocab, beam_size, request_bs, max_new_tokens, min_new_tokens;
  int32_t eos_id;
  logits_fn model;
  void* user;
  row_fn row;
  std::vector<std::vector<int32_t>> prompts;
  std::vector<beam> cur_beams, next_beams;
  std::vector<beam_hypotheses> beam_hypos;
  std::vector<bool> requests_done;
  std::vector<std::vector<int32_t>> response;
  std::vector<float> response_score;
  long long counter = 0;
  int err = 0;

  // model_eval over the rows (request, generated tokens): the logits of each row's last token, [rows][n_vocab]
  std::vector<float> eval(const std::vector<int>& req, const std::vector<const std::vector<int32_t>*>& gen) {
    const int rows = (int)req.size();
    std::vector<std::vector<int32_t>> h(rows);
    std::vector<const int32_t*> hp(rows);
    std::vector<int> hl(rows);
    for (int i = 0; i < rows; ++i) {
      h[i] = prompts[req[i]];
      h[i].insert(h[i].end(), gen[i]->begin(), gen[i]->end());
      hp[i] = h[i].data();
      hl[i] = (int)h[i].size();
    }
    std::vector<float> lg((size_t)rows * n_vocab);
    if (!err) err = model(user, rows, req.data(), hp.data(), hl.data(), lg.data());
    return lg;
  }

  // logits_info (:2139-2211) with logits_processor (:2213-2229) and the scoring of beam_top_k_next_tokens (:2331-2336): the top
  // raw_k tokens of each row by logit, scored log_softmax + beams_score, in heap order.  min_new is the rows' gen_conf.min_new_tokens
  // (:2323): next_inputs[i].gen_conf
  std::vector<std::vector<beam_next_token>> row_top_k(std::vector<float>& logits, const std::vector<uint32_t>& cur_lens,
                                                      const std::vector<float>& beams_score, int raw_k, uint32_t min_new) {
    const int bs = (int)cur_lens.size();
    std::vector<std::vector<beam_next_token>> out(bs);
    for (int i = 0; i < bs; ++i) {
      float* l = logits.data() + (size_t)i * n_vocab;
      const int mask = min_new > cur_lens[i];
      if (row) {
        std::vector<int32_t> ids(raw_k);
        std::vector<float> sc(raw_k);
        row(l, n_vocab, raw_k, beams_score[i], mask, eos_id, ids.data(), sc.data());
        for (int j = 0; j < std::min(raw_k, n_vocab); ++j) out[i].push_back(beam_next_token{ids[j], sc[j], -1});
        continue;
      }
      const float max_l = *std::max_element(l, l + n_vocab);
      const float norm = 1.0f / std::accumulate(l, l + n_vocab, 0.0f, [&](float sum, float x) { return sum + std::exp(x - max_l); });
      if (mask) l[eos_id] = NEG_INF;
      // vocab_top_k (:2189-2210)
      std::vector<beam_next_token>& h = out[i];
      const int tk = std::min(raw_k, n_vocab);
      for (int t = 0; t < tk; ++t) h.push_back(beam_next_token{t, l[t], -1});
      auto comp = [](const beam_next_token& a, const beam_next_token& b) { return a.score > b.score; };
      std::make_heap(h.begin(), h.end(), comp);
      for (int t = tk; t < n_vocab; ++t)
        if (h.front().score < l[t]) {
          std::pop_heap(h.begin(), h.end(), comp);
          h.back().id = t;
          h.back().score = l[t];
          std::push_heap(h.begin(), h.end(), comp);
        }
      for (beam_next_token& r : h) r.score = std::log(norm * std::exp(r.score - max_l)) + beams_score[i];
    }
    return out;
  }

  // beam_top_k_next_tokens (:2312-2376) over the rows of the running requests, num_beams[rb] rows each
  std::vector<beam_next_token> top_k_next_tokens(const std::vector<std::vector<beam_next_token>>& raw_top_k,
                                                 const std::vector<int>& num_beams, const std::vector<int>& beam_indices,
                                                 int sample_scale) {
    const int raw_k = sample_scale * beam_size;
    std::vector<beam_next_token> res;
    size_t row_off = 0;
    auto comp = [](const beam_next_token& a, const beam_next_token& b) { return cand_before(a, b); };  // reference: a.score > b.score
    for (size_t i = 0; i < num_beams.size(); ++i) {
      const int num_beam = num_beams[i];
      const int sample_k = num_beam == 1 ? beam_size : sample_scale * num_beam;
      std::vector<beam_next_token> min_heap;
      for (int j = 0; j < num_beam; ++j) {
        int n = 0;
        if (j == 0) {
          for (; n < sample_k; ++n)
            min_heap.push_back(beam_next_token{raw_top_k[row_off + j][n].id, raw_top_k[row_off + j][n].score, beam_indices[row_off + j]});
          std::make_heap(min_heap.begin(), min_heap.end(), comp);
        }
        for (; n < raw_k; ++n) {
          beam_next_token nr{raw_top_k[row_off + j][n].id, raw_top_k[row_off + j][n].score, beam_indices[row_off + j]};
          if (cand_before(nr, min_heap.front())) {  // reference: min_heap.front().score < nr.score
            std::pop_heap(min_heap.begin(), min_heap.end(), comp);
            min_heap.back() = nr;
            std::push_heap(min_heap.begin(), min_heap.end(), comp);
          }
        }
      }
      row_off += num_beam;
      std::sort(min_heap.begin(), min_heap.end(), cand_before);
      res.insert(res.end(), min_heap.begin(), min_heap.end());
    }
    return res;
  }

  // fill_next_beams_by_top_scores (:2378-2436) and next_candidate_beams (:2438-2510)
  void fill_next_beams_by_top_scores() {
    std::vector<int> req, beam_indices, running;
    std::vector<const std::vector<int32_t>*> gen;
    std::vector<float> beams_score;
    std::vector<uint32_t> cur_lens;
    for (size_t i = 0; i < cur_beams.size(); ++i) {
      if (cur_beams[i].done) {
        next_beams[i].done = true;
        continue;
      }
      if (running.empty() || running.back() != cur_beams[i].request_idx) running.push_back(cur_beams[i].request_idx);
      req.push_back(cur_beams[i].request_idx);
      gen.push_back(&cur_beams[i].token_ids);
      beam_indices.push_back(cur_beams[i].beam_idx);
      beams_score.push_back(cur_beams[i].score);
      cur_lens.push_back((uint32_t)cur_beams[cur_beams[i].request_idx * beam_size].token_ids.size());
    }
    std::vector<float> logits = eval(req, gen);
    const int sample_scale = 2;
    std::vector<int> num_beams(running.size(), beam_size);
    std::vector<beam_next_token> next =
        top_k_next_tokens(row_top_k(logits, cur_lens, beams_score, sample_scale * beam_size, (uint32_t)min_new_tokens), num_beams,
                          beam_indices, sample_scale);
    int rb_off = 0;
    for (size_t rb = 0; rb < running.size(); ++rb) {
      const int r = running[rb];
      int record_push = 0;
      for (int nt = 0; nt < num_beams[rb] * sample_scale; ++nt) {
        const beam_next_token& t = next[rb_off + nt];
        const int cb_off = t.beam_idx + r * beam_size;
        if (t.id == eos_id) {
          if (nt >= beam_size) continue;
          cur_beams[cb_off].score = t.score;
          beam_hypos[r].add(cur_beams[cb_off]);
        } else {
          beam next_beam = cur_beams[cb_off];
          next_beam.token_ids.push_back(t.id);
          next_beam.score = t.score;
          next_beams[r * beam_size + record_push] = std::move(next_beam);
          record_push++;
        }
        if (record_push == beam_size) {
          std::stable_sort(next_beams.begin() + r * beam_size, next_beams.begin() + (r + 1) * beam_size,
                           [](const beam& a, const beam& b) { return a.beam_idx < b.beam_idx; });
          break;
        }
      }
      rb_off += num_beams[rb] * sample_scale;
      for (int i = 0; i < beam_size; ++i) next_beams[r * beam_size + i].beam_idx = i;  // update_kv_cache_reorder_indices (:2560)
    }
  }

  // update_status and finalize (:2622-2674)
  void update_status() {
    std::vector<int> next_done;
    for (int h = 0; h < request_bs; ++h) {
      if (requests_done[h]) continue;
      const bool enough = !cur_beams[h * beam_size].token_ids.empty() && (int)cur_beams[h * beam_size].token_ids.size() == max_new_tokens;
      if (beam_hypos[h].is_done() || enough) {
        requests_done[h] = true;
        next_done.push_back(h);
        for (int i = 0; i < beam_size; ++i) cur_beams[h * beam_size + i].done = next_beams[h * beam_size + i].done = true;
      }
    }
    for (int h : next_done) {
      if (!beam_hypos[h].is_done())
        for (int i = 0; i < beam_size; ++i) beam_hypos[h].add(cur_beams[h * beam_size + i]);
      const beam& top = beam_hypos[h].top1();
      response[h] = top.token_ids;
      response_score[h] = top.score;
    }
  }

  // loop (:2676-2766)
  void loop() {
    for (int n = 0; n < max_new_tokens && !err; ++n) {
      if (n == 0) {
        std::vector<int> req(request_bs);
        std::iota(req.begin(), req.end(), 0);
        std::vector<std::vector<int32_t>> none(request_bs);
        std::vector<const std::vector<int32_t>*> gen;
        for (auto& v : none) gen.push_back(&v);
        std::vector<float> logits = eval(req, gen);
        std::vector<float> beam_scores(request_bs, 0.0f);
        std::vector<int> num_beams(request_bs, 1), beam_indices(request_bs, 0);
        std::vector<uint32_t> cur_lens(request_bs, 0);  // cur_beams hold no tokens yet
        // next_inputs are the caller's inputs (:2679), built by Model::beam_generate without a gen_conf
        // (application/main_pybind.cpp:528-538): min_new_tokens is generation_config{}'s 0 (model_types.h:283) on this step only;
        // the later steps carry gen_confs[request] = ctx->generation_conf (:2410, :2691)
        std::vector<beam_next_token> next =
            top_k_next_tokens(row_top_k(logits, cur_lens, beam_scores, beam_size, 0), num_beams, beam_indices, 1);
        for (int rb = 0; rb < request_bs; ++rb)
          for (int i = 0; i < beam_size; ++i) {
            beam b;
            b.token_ids.push_back(next[i + rb * beam_size].id);
            b.score = next[i + rb * beam_size].score;
            b.beam_idx = i;
            b.request_idx = rb;
            cur_beams[rb * beam_size + i] = std::move(b);
          }
      } else {
        fill_next_beams_by_top_scores();
        cur_beams.swap(next_beams);
      }
      update_status();
      if (std::find(requests_done.begin(), requests_done.end(), false) == requests_done.end()) break;
    }
  }
};

}  // namespace

ORC_API int orc_beam_search(int n_vocab, int n, const int* n_tokens, const int32_t* tokens, int num_beams, int max_new_tokens,
                            int min_new_tokens, float length_penalty, int early_stopping, int32_t eos_id, logits_fn model, void* user,
                            row_fn row, int32_t* out_tokens, int* out_len, float* out_score) {
  flow f;
  f.n_vocab = n_vocab;
  f.beam_size = num_beams;
  f.request_bs = n;
  f.max_new_tokens = max_new_tokens;
  f.min_new_tokens = min_new_tokens;
  f.eos_id = eos_id;
  f.model = model;
  f.user = user;
  f.row = row;
  for (int r = 0, off = 0; r < n; off += n_tokens[r++]) f.prompts.emplace_back(tokens + off, tokens + off + n_tokens[r]);
  f.cur_beams.resize((size_t)n * num_beams);
  f.next_beams.resize((size_t)n * num_beams);
  for (int r = 0; r < n; ++r) f.beam_hypos.push_back(beam_hypotheses{num_beams, length_penalty, early_stopping != 0, eos_id, &f.counter, {}});
  f.requests_done.assign(n, false);
  f.response.resize(n);
  f.response_score.assign(n, 0.0f);
  f.loop();
  if (f.err) return f.err;
  for (int r = 0; r < n; ++r) {
    std::copy(f.response[r].begin(), f.response[r].end(), out_tokens + (size_t)r * max_new_tokens);
    out_len[r] = (int)f.response[r].size();
    out_score[r] = f.response_score[r];
  }
  return 0;
}

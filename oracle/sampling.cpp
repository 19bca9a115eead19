// oracle/sampling.cpp -- a C++ restatement of the reference's sampler, model_post_sample_top_k_top_p_repeat
// (neural_speed/models/model_utils/model_utils.cpp:2987-3032) and the helpers it calls, for one row at a time on one
// std::mt19937 that lives across calls (model_context.rng, :1024).  TEST INFRASTRUCTURE ONLY.
// Built on its own (a shared library of this one file, -ffp-contract=off) by tests/test_sampling_cpu.py.
//
// model_utils.cpp cannot be compiled here (it includes bestla_gemm.h, which needs xbyak), so this restatement is pinned by
// reading; it calls std::partial_sort, std::sort, std::mt19937 and std::discrete_distribution exactly where the reference does,
// so the library's behaviour is the reference build's.  exp_fn selects the exp: null = glibc expf (the reference), or a pointer
// to the library's ns_sample_expf_host (the stated arithmetic of the device sampler).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <random>
#include <sstream>
#include <thread>
#include <vector>

#define ORC_API extern "C" __attribute__((visibility("default")))

namespace {
struct TokenData {  // model_token_data
  int id;
  float logit;
  float p;
};
typedef float (*ExpFn)(float);

float exp_of(ExpFn f, float x) { return f ? f(x) : expf(x); }

// model_sample_softmax (:521-547)
void softmax(std::vector<TokenData>& c, bool& sorted, ExpFn ef) {
  if (!sorted) {
    std::sort(c.begin(), c.end(), [](const TokenData& a, const TokenData& b) { return a.logit > b.logit; });
    sorted = true;
  }
  const float max_l = c[0].logit;
  float cum_sum = 0.0f;
  for (auto& t : c) {
    t.p = exp_of(ef, t.logit - max_l);
    cum_sum += t.p;
  }
  for (auto& t : c) t.p /= cum_sum;
}
}  // namespace

ORC_API void* orc_mt_new(uint32_t seed) { return new std::mt19937(seed); }
ORC_API void orc_mt_free(void* g) { delete static_cast<std::mt19937*>(g); }
ORC_API uint32_t orc_mt_next(void* g) { return (*static_cast<std::mt19937*>(g))(); }
// the engine's state as libstdc++ writes it (operator<<): 624 words, then the index of the next one
ORC_API void orc_mt_state(void* g, uint32_t* out) {
  std::ostringstream os;
  os << *static_cast<std::mt19937*>(g);
  std::istringstream is(os.str());
  for (int i = 0; i < 625; ++i) is >> out[i];
}
// std::discrete_distribution<>(p, p + n)(rng), as model_sample_token draws (:983-985)
ORC_API int orc_discrete_draw(void* g, const float* p, int n) {
  std::discrete_distribution<> dist(p, p + n);
  return dist(*static_cast<std::mt19937*>(g));
}

// One row: steps 1-7 of model_post_sample_top_k_top_p_repeat.  window: the W = min(repeat_last_n, n_ctx) last entries of the
// sequence's history (:3013-3018).  Returns the pick; kept / ids [kept] / probs [kept] (nullable) are the final candidates.
ORC_API int orc_sample_row(void* g, const float* logits, int n_vocab, const int* window, int W, int top_k, float top_p, float temp,
                           float penalty, ExpFn ef, int* kept, int* ids, float* probs) {
  // 1. candidates: every logit in id order (:3003-3008)
  std::vector<TokenData> c;
  c.reserve(n_vocab);
  for (int id = 0; id < n_vocab; ++id) c.push_back(TokenData{id, logits[id], 0.0f});
  bool sorted = false;
  // 2. model_sample_repetition_penalty (:798-828)
  if (W != 0 && penalty != 1.0f) {
    for (auto& t : c) {
      if (std::find(window, window + W, t.id) == window + W) continue;
      if (t.logit <= 0) t.logit *= penalty;
      else t.logit /= penalty;
    }
    sorted = false;
  }
  // frequency / presence penalties with alpha 0 (:830-834): nothing
  // 3. model_sample_top_k, min_keep 1 (:549-570)
  int k = std::max(top_k, 1);
  k = std::min(k, (int)c.size());
  if (!sorted) {
    auto comp = [](const TokenData& a, const TokenData& b) { return a.logit > b.logit; };
    if (k == (int)c.size()) std::sort(c.begin(), c.end(), comp);
    else std::partial_sort(c.begin(), c.begin() + k, c.end(), comp);
    sorted = true;
  }
  c.resize(k);
  // 4. tail-free z = 1 and typical p = 1 return at once (:604-606, :656-661)
  // 5. model_sample_top_p, min_keep 1 (:572-602)
  if (top_p < 1.0f) {
    softmax(c, sorted, ef);
    float cum_sum = 0.0f;
    size_t last_idx = c.size();
    for (size_t i = 0; i < c.size(); ++i) {
      cum_sum += c[i].p;
      if (cum_sum > top_p && i >= 1) {
        last_idx = i;
        break;
      }
    }
    c.resize(last_idx);
  }
  // 6. model_sample_temperature (:719-729)
  for (auto& t : c) t.logit /= temp;
  // 7. model_sample_token (:971-991)
  softmax(c, sorted, ef);
  std::vector<float> pr;
  pr.reserve(c.size());
  for (auto& t : c) pr.push_back(t.p);
  std::discrete_distribution<> dist(pr.begin(), pr.end());
  const int idx = dist(*static_cast<std::mt19937*>(g));
  if (kept) *kept = (int)c.size();
  for (size_t i = 0; i < c.size(); ++i) {
    if (ids) ids[i] = c[i].id;
    if (probs) probs[i] = c[i].p;
  }
  return c[idx].id;
}

// exp_fn against glibc expf over every finite x <= 0 (and +0): largest difference in ulps, and how many differ
ORC_API void orc_expf_compare(ExpFn ef, int* max_ulp, long long* n_diff, long long* n_total) {
  // b = -1 stands for +0; b = 0 .. 0x7f7fffff for the bit patterns 0x80000000 | b (-0 .. -FLT_MAX), split over threads
  const long long lo = -1, hi = 0x7f800000LL;
  const int nth = (int)std::max(1u, std::min(64u, std::thread::hardware_concurrency()));
  std::vector<int> mx(nth, 0);
  std::vector<long long> nd(nth, 0), nt(nth, 0);
  std::vector<std::thread> pool;
  for (int t = 0; t < nth; ++t)
    pool.emplace_back([&, t] {
      const long long b0 = lo + (hi - lo) * t / nth, b1 = lo + (hi - lo) * (t + 1) / nth;
      for (long long b = b0; b < b1; ++b) {
        const uint32_t u = b < 0 ? 0u : (0x80000000u | (uint32_t)b);
        float x;
        memcpy(&x, &u, 4);
        const float r0 = expf(x), r1 = ef(x);
        uint32_t a0, a1;
        memcpy(&a0, &r0, 4);
        memcpy(&a1, &r1, 4);
        const long long d = (long long)a0 - (long long)a1;  // both non-negative finite: bit distance = ulp distance
        const int ad = (int)(d < 0 ? -d : d);
        if (ad) ++nd[t];
        if (ad > mx[t]) mx[t] = ad;
        ++nt[t];
      }
    });
  for (auto& th : pool) th.join();
  *max_ulp = *std::max_element(mx.begin(), mx.end());
  *n_diff = *n_total = 0;
  for (int t = 0; t < nth; ++t) {
    *n_diff += nd[t];
    *n_total += nt[t];
  }
}

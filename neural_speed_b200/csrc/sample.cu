// sample.cu -- the reference's sampler (model_post_sample_top_k_top_p_repeat, model_utils.cpp:2987-3032) on the device, in one
// launch that takes the argmax's place in the eval step; its host restatement; and the parity entries ns_llama_sample and
// ns_llama_sample_rows.
//
// Grid (kVocabSlices, rows), 512 threads, on the slice reductions of vocab_slices.cuh.  Each CTA loads one slice of its row's
// logits into shared memory, applies the repetition penalty to the slice's ids found in the row's window (stored window + this
// pass's tokens, each id once), and selects the slice's top k keys (logit descending, id ascending: ns_sample_key) into global
// scratch (slice_top_keys).  The last CTA of a row takes the row's top k over those partials, sorted (row_top_keys), runs steps
// 5-7 in one thread (sample.h: every sum in the reference's order), then stores the row's window.  Then the draw, in one of two
// instantiations: the context-wide sampler's last row to finish (a second ticket) walks the rows in caller order, draws from the
// context's one std::mt19937 and writes picks and state; the per-sequence sampler's row takes {top_k, top_p, temperature,
// penalty, window} from a device table entry and draws in its own last CTA from that entry's generator, so rows are independent
// and a captured launch reads whatever the table holds at replay.
#include "nsb.cuh"
#include "sample.h"
#include "vocab_slices.cuh"

#include <algorithm>
#include <vector>

namespace {

constexpr int kSampleThreads = 512;

// row r's window entry j (0 <= j < W): the last W of (stored window ++ this pass's tl tokens)
__device__ __forceinline__ int window_at(const int* wv, const int* tp, int tl, int W, int j) {
  return j + tl < W ? wv[j + tl] : tp[j + tl - W];
}

// row r's pick: picks, then as argmax_kernel the row state and its record
__device__ __forceinline__ void store_pick(const SampleLaunch& a, int r, int pick) {
  if (a.picks) a.picks[r] = pick;
  if (a.state) {
    int* st = a.state + (a.rowwise ? 4 * r : 0);
    st[3] = pick;
    if (a.advance) {
      st[0] = pick;
      st[1] += a.n_tokens;
      if (a.record) a.record[(size_t)r * a.rec_stride + st[2]++] = pick;
    }
  }
}

// PER_SEQ: the parameters and generator of each row's slot (a.cfg), and the draw in the row's last CTA
template <bool PER_SEQ>
__global__ void __launch_bounds__(kSampleThreads) sample_kernel(const SampleLaunch a) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int s_kept;
  const int row = blockIdx.y, tid = threadIdx.x, n = a.n_vocab, slot = row * kVocabSlices + blockIdx.x;
  const VocabSlice sl = vocab_slice(n, blockIdx.x);
  const int lo = sl.lo, hi = sl.hi, len = hi - lo;
  const float* lg = a.logits + (size_t)row * n;
  const int* tp;
  int tl;
  if (a.last) {
    const int t0 = row ? a.last[row - 1] + 1 : 0;
    tp = a.toks + t0;
    tl = a.last[row] - t0 + 1;
  } else {
    tp = a.toks ? a.toks + (size_t)row * a.tok_stride : nullptr;
    tl = a.toks ? a.tok_len : 0;
  }
  int* wv = a.win ? a.win + (size_t)(a.slot ? a.slot[row] : a.slot_const >= 0 ? a.slot_const : row) * a.win_stride : nullptr;
  // PER_SEQ: the row's slot's parameters; its window is the last cf->W entries of the slot
  const SampleCfg* cf = PER_SEQ ? a.cfg + (a.slot ? a.slot[row] : a.slot_const >= 0 ? a.slot_const : row) : nullptr;
  if constexpr (PER_SEQ)
    if (wv) wv += a.win_stride - cf->W;
  const int W = PER_SEQ ? cf->W : a.W, K = min(PER_SEQ ? cf->k : a.k, n);
  const bool pen = W > 0 && (PER_SEQ ? cf->penalty : a.penalty) != 1.f;

  // ---- slice: load, penalise each window id of the slice once, select the slice's top min(K, len) ----
  float* vals = reinterpret_cast<float*>(smem);
  unsigned char* flag = smem + (size_t)vocab_slice_width(n) * sizeof(float);
  for (int i = tid; i < len; i += blockDim.x) {
    vals[i] = lg[lo + i];
    flag[i] = 0;
  }
  __syncthreads();
  if (pen) {
    for (int j = tid; j < W; j += blockDim.x) {
      const int id = window_at(wv, tp, tl, W, j);
      if (id >= lo && id < hi) flag[id - lo] = 1;
    }
    __syncthreads();
    for (int i = tid; i < len; i += blockDim.x)
      if (flag[i]) vals[i] = ns_sample_penalize(vals[i], PER_SEQ ? cf->penalty : a.penalty);
    __syncthreads();
  }
  slice_top_keys<kSampleThreads>([&](int i) { return ns_sample_key(vals[i], lo + i); }, len, K, a.pkeys + (size_t)slot * a.k,
                                 a.pcnt + slot);
  if (!last_of_row(a.tickets, row)) return;

  // ---- the row's last CTA: top K of the partials, sorted (the slice's values are dead) ----
  uint64_t* sk = reinterpret_cast<uint64_t*>(smem);
  const int P = row_top_keys<kSampleThreads>(a.pkeys + (size_t)row * kVocabSlices * a.k, a.pcnt + row * kVocabSlices, a.k, K, sk);
  float* l = reinterpret_cast<float*>(sk + P);  // [K]
  float* p = l + K;                             // [K]
  int* rid = a.ids + (size_t)row * a.k;
  for (int i = tid; i < K; i += blockDim.x) {
    l[i] = ns_sample_key_value(sk[i]);
    rid[i] = ns_sample_key_id(sk[i]);
  }
  __syncthreads();
  // ---- steps 5-7 in one thread, in the reference's order ----
  if (tid == 0) {
    const int kept = ns_sample_tail(l, p, K, PER_SEQ ? cf->top_p : a.top_p, PER_SEQ ? cf->temp : a.temp);
    ns_sample_cumulative(p, kept, a.cp + (size_t)row * a.k);
    a.kept[row] = kept;
    s_kept = kept;
  }
  __syncthreads();
  float* rp = a.probs + (size_t)row * a.k;
  for (int i = tid; i < K; i += blockDim.x) rp[i] = i < s_kept ? p[i] : 0.f;
  // ---- the row's window: the last W of (stored ++ this pass's tokens) ----
  if (a.store && wv && tl > 0) {
    const int v = tid < W ? window_at(wv, tp, tl, W, tid) : 0;
    __syncthreads();
    if (tid < W) wv[tid] = v;
  }
  if constexpr (PER_SEQ) {
    // the row's own draw, on its slot's generator: after the window store, which may read this pass's token from the state
    // the pick overwrites
    if (tid == 0) {
      uint32_t* mt = a.mt + (size_t)(a.slot ? a.slot[row] : a.slot_const >= 0 ? a.slot_const : row) * kMtWords;
      store_pick(a, row, ns_sample_key_id(sk[a.draw ? ns_sample_pick(a.cp + (size_t)row * a.k, s_kept, mt) : 0]));
      a.tickets[row] = 0u;
    }
    return;
  }
  if (tid == 0) a.tickets[row] = 0u;
  // ids, probs, the window: visible to the drawing CTA and the next launch
  if (!last_of_row(a.tickets, a.rows, a.rows) || tid != 0) return;
  // ---- the last row: draws in caller order ----
  for (int i = 0; i < a.rows; ++i) {
    const int r = a.order ? a.order[i] : i;
    const int kept = ((volatile int*)a.kept)[r];
    int idx = 0;
    if (a.draw && kept >= 2 && kept <= a.k) {
      const double* cpr = a.cp + (size_t)r * a.k;
      idx = ns_sample_pick(cpr, kept, a.mt);  // cp was written by other CTAs before their ticket: fenced above
    }
    store_pick(a, r, ((volatile int*)a.ids)[(size_t)r * a.k + idx]);
  }
  a.tickets[a.rows] = 0u;
}

size_t sample_smem(int n_vocab, int k) {
  const size_t per = (size_t)vocab_slice_width(n_vocab);
  const int K = k < n_vocab ? k : n_vocab;
  size_t P = 1;
  while (P < (size_t)K) P <<= 1;
  return std::max(per * 5, P * 8 + (size_t)K * 8);
}

}  // namespace

int ns_sample_check(const char* who, const ns_llama_sampling* s) {
  if (!(s->top_k >= 1) || !(s->top_p > 0.f && s->top_p <= 1.f) || !(s->temperature > 0.f && isfinite(s->temperature)) ||
      !(s->repeat_penalty > 0.f && isfinite(s->repeat_penalty)) || s->repeat_last_n < 0 || s->repeat_last_n > kSampleMaxWindow) {
    ns_set_error("%s: top_k %d top_p %g temperature %g repeat_penalty %g repeat_last_n %d: need top_k >= 1, 0 < top_p <= 1, finite "
                 "temperature and repeat_penalty > 0, 0 <= repeat_last_n <= %d",
                 who, s->top_k, s->top_p, s->temperature, s->repeat_penalty, s->repeat_last_n, kSampleMaxWindow);
    return NS_E_INVALID;
  }
  if (s->top_k > kSampleMaxK) {
    ns_set_error("%s: top_k %d above %d (the device selection sorts at most %d candidates per row)", who, s->top_k, kSampleMaxK,
                 kSampleMaxK);
    return NS_E_UNSUPPORTED;
  }
  return NS_OK;
}

// the per-sequence sampler sizes its shared memory by a.k, the largest top_k any row may take: one captured launch serves any
// contents of its parameter table
int ns_launch_sample(const SampleLaunch& a, cudaStream_t st) {
  const size_t smem = sample_smem(a.n_vocab, a.k);
  auto* kern = a.cfg ? sample_kernel<true> : sample_kernel<false>;
  if (smem > 48 * 1024) {
    if (smem > 220 * 1024) {
      ns_set_error("sampler: n_vocab %d too large (a slice of %d logits must fit in shared memory)", a.n_vocab, a.n_vocab / kVocabSlices);
      return NS_E_UNSUPPORTED;
    }
    NS_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  NS_CUDA_TRY(ns_launch_pdl(kern, dim3((unsigned)kVocabSlices, (unsigned)a.rows), dim3(kSampleThreads), smem, st, a));
  ns_count_launch();
  return NS_OK;
}

SampleCfg ns_sample_cfg(const ns_llama_sampling* s, int max_window) {
  if (!s) return SampleCfg{1, 1.f, 1.f, 1.f, 0};
  return SampleCfg{s->top_k, s->top_p, s->temperature, s->repeat_penalty, std::min(s->repeat_last_n, max_window)};
}

// ---- host restatement ------------------------------------------------------------------------------------------------------

extern "C" void ns_sample_seed_host(uint32_t seed, uint32_t* state) {
  if (state) ns_mt_seed(seed, state);
}

extern "C" float ns_sample_expf_host(float x) { return ns_sample_expf(x); }

extern "C" int ns_sample_row_host(const float* logits, int n_vocab, const int32_t* window, int n_window, const ns_llama_sampling* s,
                                  uint32_t* state, int32_t* pick, int* kept, int32_t* ids, float* probs) {
  if (!logits || !s || !state || !pick || n_vocab < 1 || n_window < 0 || n_window > kSampleMaxWindow || (n_window && !window)) {
    ns_set_error("ns_sample_row_host: invalid arguments (n_vocab %d n_window %d)", n_vocab, n_window);
    return NS_E_INVALID;
  }
  if (int rc = ns_sample_check("ns_sample_row_host", s)) return rc;
  // step 2: each candidate whose id is in the window changed once (model_utils.cpp:798-828)
  std::vector<float> v(logits, logits + n_vocab);
  if (s->repeat_penalty != 1.f) {
    std::vector<char> hit(n_vocab, 0);
    for (int j = 0; j < n_window; ++j)
      if (window[j] >= 0 && window[j] < n_vocab) hit[window[j]] = 1;
    for (int i = 0; i < n_vocab; ++i)
      if (hit[i]) v[i] = ns_sample_penalize(v[i], s->repeat_penalty);
  }
  // step 3: the top K in selection order (:549-570)
  const int K = std::min(s->top_k, n_vocab);
  std::vector<uint64_t> key(n_vocab);
  for (int i = 0; i < n_vocab; ++i) key[i] = ns_sample_key(v[i], i);
  std::partial_sort(key.begin(), key.begin() + K, key.end(), [](uint64_t x, uint64_t y) { return x > y; });
  std::vector<float> l(K), p(K);
  std::vector<double> cp(K);
  for (int i = 0; i < K; ++i) l[i] = ns_sample_key_value(key[i]);
  // steps 5-7
  const int n = ns_sample_tail(l.data(), p.data(), K, s->top_p, s->temperature);
  ns_sample_cumulative(p.data(), n, cp.data());
  const int idx = ns_sample_pick(cp.data(), n, state);
  *pick = ns_sample_key_id(key[idx]);
  if (kept) *kept = n;
  for (int i = 0; i < K; ++i) {
    if (ids) ids[i] = ns_sample_key_id(key[i]);
    if (probs) probs[i] = i < n ? p[i] : 0.f;
  }
  return NS_OK;
}

// ---- parity entries ------------------------------------------------------------------------------------------------------
// workspace: tickets [kSampleMaxRows + 1] (at the same place for every n and k, so one zeroed workspace serves calls of any
// shape) | pcnt [n][slices] | kept [n], each padded to 16 bytes | cp [n][k] | ids [n][k] | probs [n][k] | pkeys [n][slices][k] |
// the per-row parameters of ns_llama_sample_rows [n]
constexpr int kSampleMaxRows = 32;
static size_t pad16(size_t b) { return (b + 15) / 16 * 16; }
extern "C" size_t ns_llama_sample_workspace_bytes(int n, int top_k) {
  if (n < 1 || top_k < 1) return 0;
  const size_t k = (size_t)std::min(top_k, kSampleMaxK);
  return pad16((size_t)(kSampleMaxRows + 1) * 4) + pad16((size_t)n * kVocabSlices * 4) + pad16((size_t)n * 4) + pad16((size_t)n * k * 8) +
         pad16((size_t)n * k * 4) * 2 + (size_t)n * kVocabSlices * k * 8 + (size_t)n * sizeof(SampleCfg);
}

// the arguments both entries check; nothing is launched
static int check_rows(const char* who, const float* logits, int n, int n_vocab, const int32_t* windows, int n_window, const void* s,
                      const void* mt, const int32_t* picks, const void* ws) {
  if (int rc = ns_ensure_device()) return rc;
  if (!logits || !s || !mt || !picks || !ws || n < 1 || n > kSampleMaxRows || n_vocab < 1 || n_window < 0 || n_window > kSampleMaxWindow ||
      (n_window && !windows)) {
    ns_set_error("%s: invalid arguments (n %d n_vocab %d n_window %d, or a null pointer)", who, n, n_vocab, n_window);
    return NS_E_INVALID;
  }
  return NS_OK;
}

// a launch of n rows of scratch stride k over the workspace, the caller's outputs where given; row r's window at
// windows + r n_window.  Returns the end of the scratch (the per-row parameters' place).
static char* rows_launch(SampleLaunch& a, const float* logits, int n, int n_vocab, const int32_t* windows, int n_window, int k,
                         int32_t* picks, int* kept, int32_t* ids, float* probs, void* ws) {
  char* w = static_cast<char*>(ws);
  a.tickets = reinterpret_cast<unsigned*>(w);
  w += pad16((size_t)(kSampleMaxRows + 1) * 4);
  a.pcnt = reinterpret_cast<int*>(w);
  w += pad16((size_t)n * kVocabSlices * 4);
  a.kept = reinterpret_cast<int*>(w);
  w += pad16((size_t)n * 4);
  a.cp = reinterpret_cast<double*>(w);
  w += pad16((size_t)n * k * 8);
  a.ids = reinterpret_cast<int*>(w);
  w += pad16((size_t)n * k * 4);
  a.probs = reinterpret_cast<float*>(w);
  w += pad16((size_t)n * k * 4);
  a.pkeys = reinterpret_cast<unsigned long long*>(w);
  w += (size_t)n * kVocabSlices * k * 8;
  if (kept) a.kept = kept;
  if (ids) a.ids = ids;
  if (probs) a.probs = probs;
  a.logits = logits;
  a.n_vocab = n_vocab;
  a.rows = n;
  a.k = k;
  a.W = n_window;
  a.win = const_cast<int*>(windows);
  a.win_stride = n_window;
  a.slot = nullptr;
  a.slot_const = -1;  // row r reads windows + r * n_window
  a.store = 0;
  a.draw = 1;
  a.picks = picks;
  return w;
}

extern "C" int ns_llama_sample(const float* logits, int n, int n_vocab, const int32_t* windows, int n_window, const ns_llama_sampling* s,
                               uint32_t* mt_state, int32_t* picks, int* kept, int32_t* ids, float* probs, void* ws, void* queue) {
  const char* who = "ns_llama_sample";
  if (int rc = check_rows(who, logits, n, n_vocab, windows, n_window, s, mt_state, picks, ws)) return rc;
  if (int rc = ns_sample_check(who, s)) return rc;
  SampleLaunch a{};
  rows_launch(a, logits, n, n_vocab, windows, n_window, s->top_k, picks, kept, ids, probs, ws);
  a.top_p = s->top_p;
  a.temp = s->temperature;
  a.penalty = s->repeat_penalty;
  a.mt = mt_state;
  return ns_launch_sample(a, ns_stream_of(queue));
}

extern "C" int ns_llama_sample_rows(const float* logits, int n, int n_vocab, const int32_t* windows, int n_window,
                                    const ns_llama_sampling* s, uint32_t* mt_states, int32_t* picks, int* kept, int32_t* ids,
                                    float* probs, void* ws, void* queue) {
  const char* who = "ns_llama_sample_rows";
  if (int rc = check_rows(who, logits, n, n_vocab, windows, n_window, s, mt_states, picks, ws)) return rc;
  SampleCfg cfg[kSampleMaxRows];
  int k = 1;
  for (int r = 0; r < n; ++r) {
    if (int rc = ns_sample_check(who, &s[r])) return rc;
    cfg[r] = ns_sample_cfg(&s[r], n_window);
    k = std::max(k, s[r].top_k);
  }
  SampleLaunch a{};
  SampleCfg* d_cfg = reinterpret_cast<SampleCfg*>(rows_launch(a, logits, n, n_vocab, windows, n_window, k, picks, kept, ids, probs, ws));
  a.cfg = d_cfg;
  a.mt = mt_states;
  cudaStream_t st = ns_stream_of(queue);
  NS_CUDA_TRY(cudaMemcpyAsync(d_cfg, cfg, (size_t)n * sizeof(SampleCfg), cudaMemcpyHostToDevice, st));
  return ns_launch_sample(a, st);
}

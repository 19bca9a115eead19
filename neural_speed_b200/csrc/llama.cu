// llama.cu -- device-resident decode/prefill step around the weight-only matmuls (SURVEY §8 f.1).
//
// Mirrors the Llama-family eval graph of the reference, models/llama/llama.cpp:190-720 (model_eval_internal):
//   inpL = get_rows(tok_embeddings, tokens)                                    :190
//   per layer: cur = rms_norm(inpL) * attn_norm                                :205-210
//              Q,K,V = mul_qkv / mul_mat                                       :212-240
//              rope(Q), rope(K) at position n_past + t (mode 0, pairs (2i,2i+1)) :351-355, ne_layers.c:9380-9396
//              K,V -> fp16 KV cache; attention = softmax(K Q / sqrt(hd)) V      :362-420 / :286-302 (ggml path)
//              inpFF = wo * attn + inpSA                                       :585-598
//              cur = rms_norm(inpFF) * ffn_norm ; cur = ffn_silu(cur) + inpFF  :601-698
//   logits = output * (rms_norm(inpL) * out_norm)                              :707-719
// Greedy sampling = argmax with the lowest index on ties (model_utils.cpp:2963-2985).
// ns_llama_set_sampling swaps the argmax's launch for sample_kernel (sample.cu): model_post_sample_top_k_top_p_repeat
// (model_utils.cpp:2987-3032) with its generator and the sequences' repetition windows in device memory.
// ns_llama_set_sequence_sampling swaps it for the per-sequence instantiation instead: each KV block's parameters and generator
// in device tables that the captured graphs read at replay, so changing a block's config recaptures nothing.
//
// One token (n_tokens == 1) is ONE CUDA graph: the token id and n_past live in device memory (`state`), so the same graph
// replays for every position; ns_llama_generate chains graph launches with the argmax feeding the next embedding
// lookup on the device -- no host round trip per token.  The attention kernels and the plan of a pass over token segments
// are in attention.cu.
//
// Element-wise numerics follow the reference's ggml path: fp16 KV cache, Q and the softmax probabilities rounded to fp16
// before the K.Q and V.P dot products (ne_compute_forward_mul_mat_f16_f32), exp taken on the fp16-rounded argument and
// rounded to fp16 (table_exp_f16, ne_layers.c:8933-8937); rms_norm as kernel_ref.h:2199-2225.
#include <cuda_fp16.h>

#include <algorithm>
#include <vector>

#include "nsb.cuh"
#include "sample.h"
#include "logprob.h"
#include "beam.h"
#include "attention.cuh"
#include "vocab_slices.cuh"

namespace {

struct Layer {
  const float* attn_norm = nullptr;
  const float* ffn_norm = nullptr;
  const ns_weight *wq = nullptr, *wk = nullptr, *wv = nullptr, *wo = nullptr, *w1 = nullptr, *w2 = nullptr, *w3 = nullptr;
  // Qwen2 / Phi-3: the context's P-order copies behind wq / wk (ns_llama_set_arch); Qwen2: the biases [b_q | b_k | b_v] (b_q, b_k
  // in P order)
  ns_weight *own_q = nullptr, *own_k = nullptr;
  float* bias = nullptr;
  int bias_set = 0;  // bit i: part i of `bias` set
};

// The interleaved order P of ns_llama_set_arch, which puts the NeoX pair (i, i + hd/2) at (2i, 2i + 1): dst row h hd + 2i is src row
// h hd + i, dst row h hd + 2i + 1 is src row h hd + hd/2 + i.  Rows are self-contained `pitch`-byte ranges in every weight format
// (nsb.cuh, q6k.cu).  One CTA per row.
__global__ void __launch_bounds__(128) interleave_rows_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int pitch16, int hd) {
  const int r = blockIdx.x, j = r % hd;
  const int s = r - j + ((j & 1) ? hd / 2 + j / 2 : j / 2);
  const uint4* a = src + (size_t)s * pitch16;
  uint4* b = dst + (size_t)r * pitch16;
  for (int i = threadIdx.x; i < pitch16; i += blockDim.x) b[i] = a[i];
}

// x[t][:] = table[token[t * TSTRIDE]][:]   (TSTRIDE 4: the token slot of each row's device state in a batched step)
template <int TSTRIDE>
__global__ void __launch_bounds__(256) embed_kernel(const float* __restrict__ table, const int* __restrict__ tokens, int n_embd,
                                                    int n_vocab, float* __restrict__ x) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.y;
  int tok = tokens[t * TSTRIDE];
  tok = tok < 0 ? 0 : (tok >= n_vocab ? n_vocab - 1 : tok);
  const float4* src = (const float4*)(table + (size_t)tok * n_embd);
  float4* dst = (float4*)(x + (size_t)t * n_embd);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_embd / 4; i += gridDim.x * blockDim.x) dst[i] = src[i];
}

// y = x / sqrt(mean(x^2) + eps) * w      (ne_rms_norm + ne_mul; kernel_ref.h:2199-2225 "simplified")
// One CTA per row; every thread issues ALL its loads (x and w, float4) before the first use, so the row costs one memory
// latency instead of one per loop trip (a single CTA is latency-bound, not bandwidth-bound).
template <int V4>  // float4 per thread: n <= 256 * 4 * V4
__global__ void __launch_bounds__(256) rmsnorm_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y,
                                                      int n, float eps) {
  pdl_launch_dependents();
  const int n4 = n >> 2;
  float4 wv[V4];
#pragma unroll
  for (int j = 0; j < V4; ++j) {  // the norm weights do not depend on the previous kernel: fetch them before the wait
    const int i = threadIdx.x + j * 256;
    wv[j] = i < n4 ? ((const float4*)w)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  pdl_wait();
  const float4* xr = (const float4*)(x + (size_t)blockIdx.x * n);
  float4* yr = (float4*)(y + (size_t)blockIdx.x * n);
  float4 xv[V4];
#pragma unroll
  for (int j = 0; j < V4; ++j) {
    const int i = threadIdx.x + j * 256;
    xv[j] = i < n4 ? xr[i] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float ss = 0.f;
#pragma unroll
  for (int j = 0; j < V4; ++j) {
    ss = fmaf(xv[j].x, xv[j].x, ss);
    ss = fmaf(xv[j].y, xv[j].y, ss);
    ss = fmaf(xv[j].z, xv[j].z, ss);
    ss = fmaf(xv[j].w, xv[j].w, ss);
  }
  __shared__ float red[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float inv = 1.f / sqrtf(tot / (float)n + eps);
#pragma unroll
  for (int j = 0; j < V4; ++j) {
    const int i = threadIdx.x + j * 256;
    if (i < n4) yr[i] = make_float4(xv[j].x * inv * wv[j].x, xv[j].y * inv * wv[j].y, xv[j].z * inv * wv[j].z, xv[j].w * inv * wv[j].w);
  }
}

// dst[j][:] = x[src[j]][:]   (the last row of each segment of ns_llama_eval_batch, gathered for the lm_head); grid (blocks, n)
__global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ x, const int* __restrict__ src, int n_embd,
                                                          float* __restrict__ dst) {
  pdl_launch_dependents();
  pdl_wait();
  const float4* s = (const float4*)(x + (size_t)src[blockIdx.y] * n_embd);
  float4* d = (float4*)(dst + (size_t)blockIdx.y * n_embd);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_embd / 4; i += gridDim.x * blockDim.x) d[i] = s[i];
}

}  // namespace

constexpr int kPlanTiles = kMaxBatchRows / kAttnMmaRows + kMaxSeq;  // tile entries of one mixed pass, at most
// device tables of a mixed pass: rows [kMaxBatchRows][2] | tiles [kPlanTiles][kTileInts] | last row of each segment [kMaxSeq] |
// KV block of each segment [kMaxSeq] | internal segment of each caller index [kMaxSeq] (the sampler's window slots and draw order)
constexpr int kPlanInts = 2 * kMaxBatchRows + kPlanTiles * kTileInts + 3 * kMaxSeq;
constexpr int kAllChunk = kLogprobMaxRows;  // rows of one lm_head launch of ns_llama_eval_all

struct Graph {
  cudaGraphExec_t exec = nullptr;
  cudaGraph_t graph = nullptr;
};

struct ns_llama {
  ns_llama_hparams hp;
  int arch = NS_LLAMA_ARCH_LLAMA;  // ns_llama_set_arch
  cudaStream_t st;
  std::vector<Layer> layers;
  float* tok_embd = nullptr;
  float* out_norm = nullptr;
  const ns_weight* output = nullptr;
  std::vector<void*> owned;  // device allocations freed with the context
  int n_seq = 0;             // KV blocks: ns_llama_set_sequences (1 from ns_llama_create)
  int kv_type = NS_KV_F16;              // ns_llama_set_kv_type
  void *kc = nullptr, *vc = nullptr;    // [n_layer][n_seq][n_head_kv][n_ctx][hd] fp16, or the Q8_0 codes (kv_cache.cuh)
  __half *kd = nullptr, *vd = nullptr;  // Q8_0: the scale planes [n_layer][n_seq][n_head_kv][kv_d_stride]

  int* state = nullptr;   // device: {token, n_past, n_recorded, last_pick}
  int* tokens = nullptr;  // device: prompt tokens of the current eval
  int tok_cap = 0;        // ... their capacity: n_ctx, grown to the rows of a larger ns_llama_eval_batch pass
  int* plan = nullptr;    // device, ns_llama_eval_batch: kPlanInts (allocated on first use)
  int* record = nullptr;  // device: generated tokens
  int* bstate = nullptr;  // device, batched steps: [kMaxSeq][4] row states as `state` | [kMaxSeq] KV block of each row
  int* brecord = nullptr;   // device, batched steps: [n_seq][n_ctx] picks of each row
  float* am_val = nullptr;  // argmax partials: [kMaxSeq][kVocabSlices]
  int* am_idx = nullptr;
  unsigned* am_ticket = nullptr;  // [kMaxSeq]
  int m_cap = 0;
  AttnAttr attn_attr;                   // dynamic shared memory already granted to the attention kernels on this context's device
  float* attn_part = nullptr;           // split-context decode attention: [n_seq][n_head][nsplit][hd + 2] partials
  unsigned* attn_tickets = nullptr;     // [n_seq][n_head]
  int attn_nsplit = 0;
  int exact_prefill = 0;               // ns_llama_set_exact_prefill
  bool streaming = false;              // ns_llama_set_streaming: ring.n_keep sink slots, ring.tab the shift table
  Ring ring{};
  int n_total = 0;                     // tokens evaluated so far (the n_past a continuation passes)
  bool wrapped = false;                // a ring step has run since the last restart: only continuations and restarts are valid
  float *x = nullptr, *xn = nullptr, *qkv = nullptr, *attn = nullptr, *tmp = nullptr, *logits = nullptr;
  void* ws = nullptr;
  size_t ws_bytes = 0;
  Graph graph[kMaxSeq + 1];  // captured on first use: [0] the decode step of block 0, [n] a batched step of n rows
  int* h_state = nullptr;  // pinned host staging
  int* h_bstate = nullptr;  // [kMaxSeq * 5]
  int* h_plan = nullptr;      // [kMaxBatchRows] tokens | kPlanInts tables, as `plan` (allocated with it)
  float* h_logits = nullptr;  // [n_seq][n_vocab]
  // ns_llama_set_sampling: the sampler takes the argmax's launch while `sampling`; its device state is allocated on first use
  bool sampling = false;
  ns_llama_sampling smp{};
  uint32_t* mt = nullptr;             // std::mt19937 [kMtWords]
  int* win = nullptr;                 // windows [kMaxSeq][kSampleMaxWindow], slot = KV block
  unsigned long long* s_keys = nullptr;  // [kMaxSeq][kVocabSlices][kSampleMaxK]
  int* s_pcnt = nullptr;              // [kMaxSeq][kVocabSlices]
  double* s_cp = nullptr;             // [kMaxSeq][kSampleMaxK]
  unsigned* s_tickets = nullptr;      // [kMaxSeq + 1]
  int* s_kept = nullptr;              // [kMaxSeq]
  int* s_ids = nullptr;               // [kMaxSeq][kSampleMaxK]
  float* s_probs = nullptr;           // [kMaxSeq][kSampleMaxK]
  // ns_llama_set_sequence_sampling: while `per_seq`, block b samples with seq_cfg[b] (greedy when !seq_on[b]) from its own
  // generator; its window is the last seq_cfg[b].W entries of its slot of `win`.  Allocated on first use.
  bool per_seq = false;
  bool seq_on[kMaxSeq] = {};
  SampleCfg* seq_cfg = nullptr;       // [kMaxSeq]
  uint32_t* seq_mt = nullptr;         // std::mt19937 [kMaxSeq][kMtWords]
  // ns_llama_eval_all (allocated on first use): the lm_head's logits of one chunk of rows, the log-prob kernel's tickets and
  // partials, the rows' targets / log-probs / picks in internal order, and pinned staging for those and two chunks of logits
  float* all_logits = nullptr;        // [kAllChunk][n_vocab]
  unsigned* lp_tickets = nullptr;     // [kAllChunk] | max, id, sum [kAllChunk][kVocabSlices]
  int* all_io = nullptr;              // [3][kMaxBatchRows]
  int* h_all = nullptr;               // [3][kMaxBatchRows] | [2][kAllChunk][n_vocab] floats
  cudaEvent_t all_ev[2] = {};
  // ns_llama_beam_search (allocated on first use): the candidates kernel's tickets and scratch, its output and pinned staging
  unsigned* beam_ws = nullptr;        // tickets [kBeamMaxRows] | ns_beam_scratch(kBeamMaxRows, kBeamMaxK)
  BeamCand* beam_out = nullptr;       // [kBeamMaxRows][kBeamMaxK]
  BeamCand* h_beam = nullptr;
};

static void* dev_alloc(ns_llama* c, size_t bytes) {
  void* p = nullptr;
  if (cudaMalloc(&p, bytes) != cudaSuccess) {
    ns_set_error("ns_llama: cudaMalloc(%zu) failed", bytes);
    return nullptr;
  }
  c->owned.push_back(p);
  return p;
}

// release one allocation of the context early (superseded activation buffers / tensors set twice)
static void dev_free(ns_llama* c, void* p) {
  if (!p) return;
  for (size_t i = 0; i < c->owned.size(); ++i)
    if (c->owned[i] == p) {
      c->owned.erase(c->owned.begin() + (long)i);
      cudaFree(p);
      return;
    }
}

// captured graphs hold pointers to the weights, norms, buffers and KV blocks: dropped whenever one of those changes
static void drop_graphs(ns_llama* c) {
  for (Graph& g : c->graph)
    if (g.exec) {
      cudaGraphExecDestroy(g.exec);
      cudaGraphDestroy(g.graph);
      g = Graph{};
    }
}

// (re)allocates everything sized by the number of KV blocks -- caches, logits, decode-attention partials and tickets, batch
// record -- and zeroes the caches and tickets.  On failure n_seq is 0 and every eval refuses to run.
static int alloc_sequences(ns_llama* c, int n_seq) {
  const ns_llama_hparams& hp = c->hp;
  const int hd = hp.n_embd / hp.n_head;
  void* old[8] = {c->kc, c->vc, c->kd, c->vd, c->logits, c->attn_part, c->attn_tickets, c->brecord};
  for (void* p : old) dev_free(c, p);
  c->kc = c->vc = nullptr;
  c->kd = c->vd = nullptr;
  c->logits = c->attn_part = nullptr;
  c->attn_tickets = nullptr;
  c->brecord = nullptr;
  if (c->h_logits) cudaFreeHost(c->h_logits);
  c->h_logits = nullptr;
  c->n_seq = 0;
  const size_t units = (size_t)n_seq * hp.n_layer * hp.n_head_kv;
  const size_t vbytes = units * hp.n_ctx * hd * (c->kv_type == NS_KV_Q8_0 ? 1 : 2);  // value plane (fp16 or Q8_0 codes)
  const size_t dbytes = c->kv_type == NS_KV_Q8_0 ? kv_cache_bytes(NS_KV_Q8_0, units, hp.n_ctx, hd) - vbytes : 0;  // Q8_0 scales
  c->attn_nsplit = attn_ranges(hp.n_ctx);
  c->kc = dev_alloc(c, vbytes);
  c->vc = dev_alloc(c, vbytes);
  if (dbytes) {
    c->kd = (__half*)dev_alloc(c, dbytes);
    c->vd = (__half*)dev_alloc(c, dbytes);
    if (!c->kd || !c->vd) return NS_E_CUDA;
    NS_CUDA_TRY(cudaMemsetAsync(c->kd, 0, dbytes, c->st));
    NS_CUDA_TRY(cudaMemsetAsync(c->vd, 0, dbytes, c->st));
  }
  c->logits = (float*)dev_alloc(c, (size_t)n_seq * hp.n_vocab * 4);
  c->attn_part = (float*)dev_alloc(c, (size_t)n_seq * hp.n_head * c->attn_nsplit * (hd + 2) * sizeof(float));
  c->attn_tickets = (unsigned*)dev_alloc(c, (size_t)n_seq * hp.n_head * sizeof(unsigned));
  c->brecord = (int*)dev_alloc(c, (size_t)n_seq * hp.n_ctx * sizeof(int));
  if (!c->kc || !c->vc || !c->logits || !c->attn_part || !c->attn_tickets || !c->brecord) return NS_E_CUDA;
  if (!ns_cuda_ok(cudaMallocHost((void**)&c->h_logits, (size_t)n_seq * hp.n_vocab * 4), "cudaMallocHost")) {
    c->h_logits = nullptr;
    return NS_E_CUDA;
  }
  NS_CUDA_TRY(cudaMemsetAsync(c->attn_tickets, 0, (size_t)n_seq * hp.n_head * sizeof(unsigned), c->st));
  NS_CUDA_TRY(cudaMemsetAsync(c->kc, 0, vbytes, c->st));
  NS_CUDA_TRY(cudaMemsetAsync(c->vc, 0, vbytes, c->st));
  c->n_seq = n_seq;
  return NS_OK;
}

extern "C" ns_llama* ns_llama_create(const ns_llama_hparams* hp, void* queue) {
  if (ns_ensure_device()) return nullptr;
  if (!hp || hp->n_vocab <= 0 || hp->n_embd <= 0 || hp->n_head <= 0 || hp->n_head_kv <= 0 || hp->n_layer <= 0 || hp->n_ff <= 0 ||
      hp->n_ctx <= 0 || hp->n_embd % hp->n_head || hp->n_head % hp->n_head_kv || (hp->n_embd / hp->n_head) % 2 || hp->n_embd % 4) {
    ns_set_error("ns_llama_create: invalid hyper-parameters");
    return nullptr;
  }
  ns_llama* c = new ns_llama();
  c->hp = *hp;
  if (c->hp.rope_theta <= 0.f) c->hp.rope_theta = 10000.f;
  if (c->hp.rope_scale <= 0.f) c->hp.rope_scale = 1.f;
  if (c->hp.norm_eps <= 0.f) c->hp.norm_eps = 1e-6f;
  c->st = ns_stream_of(queue);
  c->layers.resize(hp->n_layer);
  const int hd = hp->n_embd / hp->n_head;
  {  // the single-pass attention kernels keep one score per cached position in shared memory
    if (attn_rows_smem(hd, hp->n_ctx) > 220 * 1024) {
      ns_set_error("ns_llama_create: n_ctx %d too large for the single-pass attention kernel (limit %zu positions at head size %d)",
                   hp->n_ctx, (220 * 1024 - attn_rows_smem(hd, 0)) / sizeof(float), hd);
      delete c;
      return nullptr;
    }
  }
  c->state = (int*)dev_alloc(c, 4 * sizeof(int));
  c->tokens = (int*)dev_alloc(c, (size_t)hp->n_ctx * sizeof(int));
  c->tok_cap = hp->n_ctx;
  c->record = (int*)dev_alloc(c, (size_t)hp->n_ctx * sizeof(int));
  c->bstate = (int*)dev_alloc(c, (size_t)kMaxSeq * 5 * sizeof(int));
  c->am_val = (float*)dev_alloc(c, (size_t)kMaxSeq * kVocabSlices * sizeof(float));
  c->am_idx = (int*)dev_alloc(c, (size_t)kMaxSeq * kVocabSlices * sizeof(int));
  c->am_ticket = (unsigned*)dev_alloc(c, kMaxSeq * sizeof(unsigned));
  if (c->am_ticket) cudaMemsetAsync(c->am_ticket, 0, kMaxSeq * sizeof(unsigned), c->st);
  if (!c->state || !c->tokens || !c->record || !c->bstate || !c->am_val || !c->am_idx || !c->am_ticket ||
      cudaMallocHost((void**)&c->h_state, 4 * sizeof(int)) != cudaSuccess ||
      cudaMallocHost((void**)&c->h_bstate, (size_t)kMaxSeq * 5 * sizeof(int)) != cudaSuccess || alloc_sequences(c, 1)) {
    ns_llama_free(c);
    return nullptr;
  }
  cudaMemsetAsync(c->state, 0, 4 * sizeof(int), c->st);
  return c;
}

extern "C" void ns_llama_free(ns_llama* c) {
  if (!c) return;
  cudaStreamSynchronize(c->st);
  drop_graphs(c);
  for (void* p : c->owned) cudaFree(p);
  for (Layer& l : c->layers) {  // the P-order copies' device rows were in `owned`
    delete l.own_q;
    delete l.own_k;
  }
  if (c->h_state) cudaFreeHost(c->h_state);
  if (c->h_bstate) cudaFreeHost(c->h_bstate);
  if (c->h_plan) cudaFreeHost(c->h_plan);
  if (c->h_logits) cudaFreeHost(c->h_logits);
  if (c->h_all) cudaFreeHost(c->h_all);
  if (c->h_beam) cudaFreeHost(c->h_beam);
  for (cudaEvent_t e : c->all_ev)
    if (e) cudaEventDestroy(e);
  delete c;
}

// NeoX RoPE (Qwen2, Phi-3): the context holds W_q / W_k in the interleaved order P and runs the mode-0 kernels (ns_llama_set_arch)
static bool neox(const ns_llama* c) { return c->arch != NS_LLAMA_ARCH_LLAMA; }

// the interleaved head order P of ns_llama_set_arch, on the host: dst[h hd + 2i] = src[h hd + i], dst[h hd + 2i + 1] = src[h hd + hd/2 + i]
static void interleave_host(const float* src, float* dst, size_t n, int hd) {
  for (size_t r = 0; r < n; ++r) {
    const size_t j = r % hd;
    dst[r] = src[r - j + ((j & 1) ? hd / 2 + j / 2 : j / 2)];
  }
}

// b_q / b_k / b_v of a Qwen2 context: parts of the layer's one bias allocation [b_q | b_k | b_v], b_q and b_k in P order
static int set_bias(ns_llama* c, int tensor, int layer, const float* host, size_t count) {
  const ns_llama_hparams& hp = c->hp;
  const int hd = hp.n_embd / hp.n_head, kvd = hd * hp.n_head_kv, part = tensor - NS_LT_BQ;
  const size_t want = part == 0 ? (size_t)hp.n_embd : (size_t)kvd;
  if (c->arch != NS_LLAMA_ARCH_QWEN2 || count != want || layer < 0 || layer >= hp.n_layer) {
    ns_set_error("ns_llama_set_f32: bias %d layer %d count %zu (%s)", tensor, layer, count,
                 c->arch != NS_LLAMA_ARCH_QWEN2 ? "biases need a Qwen2 context" : "wrong layer or size");
    return NS_E_INVALID;
  }
  Layer& l = c->layers[layer];
  if (!l.bias) {
    l.bias = (float*)dev_alloc(c, ((size_t)hp.n_embd + 2 * (size_t)kvd) * 4);
    if (!l.bias) return NS_E_CUDA;
  }
  std::vector<float> b(host, host + want);
  if (part < 2) interleave_host(host, b.data(), want, hd);
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));  // nothing in flight reads the part rewritten below
  const size_t off = part == 0 ? 0 : part == 1 ? (size_t)hp.n_embd : (size_t)hp.n_embd + kvd;
  NS_CUDA_TRY(cudaMemcpyAsync(l.bias + off, b.data(), want * 4, cudaMemcpyHostToDevice, c->st));
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));
  l.bias_set |= 1 << part;
  return NS_OK;
}

extern "C" int ns_llama_set_f32(ns_llama* c, int tensor, int layer, const float* host, size_t count) {
  if (!c || !host) return NS_E_INVALID;
  if (tensor >= NS_LT_BQ && tensor <= NS_LT_BV) return set_bias(c, tensor, layer, host, count);
  const ns_llama_hparams& hp = c->hp;
  size_t want = 0;
  if (tensor == NS_LT_TOK_EMBD) want = (size_t)hp.n_vocab * hp.n_embd;
  else if (tensor == NS_LT_OUT_NORM || tensor == NS_LT_ATTN_NORM || tensor == NS_LT_FFN_NORM) want = hp.n_embd;
  if (!want || count != want || ((tensor == NS_LT_ATTN_NORM || tensor == NS_LT_FFN_NORM) && (layer < 0 || layer >= hp.n_layer))) {
    ns_set_error("ns_llama_set_f32: tensor %d layer %d count %zu", tensor, layer, count);
    return NS_E_INVALID;
  }
  float* d = (float*)dev_alloc(c, want * 4);
  if (!d) return NS_E_CUDA;
  NS_CUDA_TRY(cudaMemcpyAsync(d, host, want * 4, cudaMemcpyHostToDevice, c->st));
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));  // also: nothing in flight reads the tensor this call replaces
  const float** slot = tensor == NS_LT_TOK_EMBD   ? (const float**)&c->tok_embd
                       : tensor == NS_LT_OUT_NORM ? (const float**)&c->out_norm
                       : tensor == NS_LT_ATTN_NORM ? &c->layers[layer].attn_norm
                                                   : &c->layers[layer].ffn_norm;
  if (*slot) {  // set twice: the captured graphs hold the old pointer
    drop_graphs(c);
    dev_free(c, (void*)*slot);
  }
  *slot = d;
  return NS_OK;
}

// *out = a context-owned copy of w with its rows in P order per head (interleave_rows_kernel); w is read, never written
static int interleaved_copy(ns_llama* c, const ns_weight* w, ns_weight** out) {
  const int hd = c->hp.n_embd / c->hp.n_head;
  if (w->pitch % 16 || w->n % hd) {
    ns_set_error("ns_llama_set_weight: rows of %d bytes / %d rows cannot be interleaved per head of %d", w->pitch, w->n, hd);
    return NS_E_INVALID;
  }
  const size_t bytes = (size_t)w->n * w->pitch;
  uint8_t* rows = (uint8_t*)dev_alloc(c, bytes);
  if (!rows) return NS_E_CUDA;
  // the caller's weight may have been filled on another stream: a load-time call, so wait for the whole device
  bool ok = ns_cuda_ok(cudaDeviceSynchronize(), "cudaDeviceSynchronize");
  if (ok) {
    interleave_rows_kernel<<<(unsigned)w->n, 128, 0, c->st>>>((const uint4*)w->rows, (uint4*)rows, w->pitch / 16, hd);
    ok = ns_cuda_ok(cudaGetLastError(), "interleave_rows_kernel") && ns_cuda_ok(cudaStreamSynchronize(c->st), "cudaStreamSynchronize");
  }
  if (!ok) {
    dev_free(c, rows);
    return NS_E_CUDA;
  }
  ns_count_launch();
  ns_weight* cp = new ns_weight(*w);
  cp->rows = rows;
  cp->base = nullptr;  // the rows are the context's; act-order `shuffle` (per column) stays the caller's
  cp->external = 1;
  cp->total_bytes = bytes;
  *out = cp;
  return NS_OK;
}

extern "C" int ns_llama_set_weight(ns_llama* c, int tensor, int layer, const ns_weight* w) {
  if (!c || !w) return NS_E_INVALID;
  const ns_llama_hparams& hp = c->hp;
  const int hd = hp.n_embd / hp.n_head, kvd = hd * hp.n_head_kv;
  int n = 0, k = hp.n_embd;
  switch (tensor) {
    case NS_LT_OUTPUT: n = hp.n_vocab; break;
    case NS_LT_WQ: n = hp.n_embd; break;
    case NS_LT_WK: case NS_LT_WV: n = kvd; break;
    case NS_LT_WO: n = hp.n_embd; break;
    case NS_LT_W1: case NS_LT_W3: n = hp.n_ff; break;
    case NS_LT_W2: n = hp.n_embd; k = hp.n_ff; break;
    default: n = 0;
  }
  if (!n || w->n != n || w->k != k || (tensor != NS_LT_OUTPUT && (layer < 0 || layer >= hp.n_layer))) {
    ns_set_error("ns_llama_set_weight: tensor %d layer %d wants %dx%d, got %dx%d", tensor, layer, n, k, w->n, w->k);
    return NS_E_INVALID;
  }
  if (tensor == NS_LT_OUTPUT) {
    c->output = w;
  } else {
    Layer& l = c->layers[layer];
    const ns_weight** slot = tensor == NS_LT_WQ ? &l.wq : tensor == NS_LT_WK ? &l.wk : tensor == NS_LT_WV ? &l.wv
                           : tensor == NS_LT_WO ? &l.wo : tensor == NS_LT_W1 ? &l.w1 : tensor == NS_LT_W2 ? &l.w2 : &l.w3;
    if (neox(c) && (tensor == NS_LT_WQ || tensor == NS_LT_WK)) {
      ns_weight** own = tensor == NS_LT_WQ ? &l.own_q : &l.own_k;
      ns_weight* cp = nullptr;
      if (int rc = interleaved_copy(c, w, &cp)) return rc;
      drop_graphs(c);  // nothing in flight (interleaved_copy synchronised): the old copy and the graphs reading it go
      if (*own) {
        dev_free(c, (*own)->rows);
        delete *own;
      }
      *own = cp;
      w = cp;
    }
    *slot = w;
  }
  drop_graphs(c);  // weights changed: the captured graphs hold stale pointers
  return NS_OK;
}

extern "C" const ns_weight* ns_llama_weight(const ns_llama* c, int tensor, int layer) {
  if (!c) return nullptr;
  if (tensor == NS_LT_OUTPUT) return c->output;
  if (layer < 0 || layer >= c->hp.n_layer) return nullptr;
  const Layer& l = c->layers[layer];
  switch (tensor) {
    case NS_LT_WQ: return l.wq;
    case NS_LT_WK: return l.wk;
    case NS_LT_WV: return l.wv;
    case NS_LT_WO: return l.wo;
    case NS_LT_W1: return l.w1;
    case NS_LT_W2: return l.w2;
    case NS_LT_W3: return l.w3;
    default: return nullptr;
  }
}

// Qwen2 / Phi-3 (set on a context without matmul weights or biases): see ns_b200.h
extern "C" int ns_llama_set_arch(ns_llama* c, int arch) {
  if (!c || (arch != NS_LLAMA_ARCH_LLAMA && arch != NS_LLAMA_ARCH_QWEN2 && arch != NS_LLAMA_ARCH_PHI3)) {
    ns_set_error("ns_llama_set_arch: arch %d (NS_LLAMA_ARCH_LLAMA %d, NS_LLAMA_ARCH_QWEN2 %d or NS_LLAMA_ARCH_PHI3 %d)", arch,
                 NS_LLAMA_ARCH_LLAMA, NS_LLAMA_ARCH_QWEN2, NS_LLAMA_ARCH_PHI3);
    return NS_E_INVALID;
  }
  bool any = c->output != nullptr;
  for (const Layer& l : c->layers)
    any = any || l.wq || l.wk || l.wv || l.wo || l.w1 || l.w2 || l.w3 || l.bias_set;
  if (any) {
    ns_set_error("ns_llama_set_arch: matmul weights or biases are set already (choose the architecture first)");
    return NS_E_INVALID;
  }
  if (arch != NS_LLAMA_ARCH_LLAMA && c->hp.rope_scale != 1.f) {
    ns_set_error("ns_llama_set_arch: rope_scale %g != 1 (the reference's NeoX RoPE scales the angle twice)", c->hp.rope_scale);
    return NS_E_UNSUPPORTED;
  }
  if (arch != NS_LLAMA_ARCH_LLAMA && c->streaming) {
    ns_set_error("ns_llama_set_arch: streaming is on (the reference has no NeoX shift-RoPE-K, qwen.cpp:85, phi3.cpp:188)");
    return NS_E_UNSUPPORTED;
  }
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));
  drop_graphs(c);
  c->arch = arch;
  return NS_OK;
}

static int launch_rmsnorm(const float* x, const float* w, float* y, int rows, int n, float eps, cudaStream_t st) {
  if (n % 4 || n > 256 * 4 * 8) {
    ns_set_error("ns_llama: n_embd %d unsupported by the RMSNorm kernel (needs n %% 4 == 0, n <= 8192)", n);
    return NS_E_UNSUPPORTED;
  }
  const int v4 = (n / 4 + 255) / 256;
  auto kern = v4 <= 1 ? rmsnorm_kernel<1> : v4 <= 2 ? rmsnorm_kernel<2> : v4 <= 4 ? rmsnorm_kernel<4> : rmsnorm_kernel<8>;
  NS_CUDA_TRY(ns_launch_pdl(kern, dim3((unsigned)rows), dim3(256), 0, st, x, w, y, n, eps));
  ns_count_launch();
  return NS_OK;
}

static int ensure_buffers(ns_llama* c, int m) {
  if (m <= c->m_cap) return NS_OK;
  const ns_llama_hparams& hp = c->hp;
  const int hd = hp.n_embd / hp.n_head, kvd = hd * hp.n_head_kv;
  if (c->m_cap > 0) {  // growing: the smaller buffers are dead once the stream has drained
    NS_CUDA_TRY(cudaStreamSynchronize(c->st));
    void* old[6] = {c->x, c->xn, c->qkv, c->attn, c->tmp, c->ws};
    for (void* p : old) dev_free(c, p);
    c->x = c->xn = c->qkv = c->attn = c->tmp = nullptr;
    c->ws = nullptr;
    c->m_cap = 0;
  }
  c->x = (float*)dev_alloc(c, (size_t)m * hp.n_embd * 4);
  c->xn = (float*)dev_alloc(c, (size_t)m * hp.n_embd * 4);
  c->qkv = (float*)dev_alloc(c, (size_t)m * (hp.n_embd + 2 * kvd) * 4);
  c->attn = (float*)dev_alloc(c, (size_t)m * hp.n_embd * 4);
  c->tmp = (float*)dev_alloc(c, (size_t)2 * m * hp.n_ff * 4);
  const size_t wsb = ns_device_workspace_bytes(m, hp.n_ff > hp.n_embd ? hp.n_ff : hp.n_embd);
  c->ws = dev_alloc(c, wsb);
  c->ws_bytes = wsb;
  if (!c->x || !c->xn || !c->qkv || !c->attn || !c->tmp || !c->ws) return NS_E_CUDA;
  c->m_cap = m;
  drop_graphs(c);
  return NS_OK;
}

static int check_complete(const ns_llama* c) {
  if (c->n_seq < 1) {
    ns_set_error("ns_llama: no KV cache (a failed ns_llama_set_sequences)");
    return NS_E_INVALID;
  }
  if (!c->tok_embd || !c->out_norm || !c->output) {
    ns_set_error("ns_llama: tok_embeddings / output norm / output weight not set");
    return NS_E_INVALID;
  }
  for (size_t i = 0; i < c->layers.size(); ++i) {
    const Layer& l = c->layers[i];
    if (!l.attn_norm || !l.ffn_norm || !l.wq || !l.wk || !l.wv || !l.wo || !l.w1 || !l.w2 || !l.w3) {
      ns_set_error("ns_llama: layer %zu is missing tensors", i);
      return NS_E_INVALID;
    }
    if (c->arch == NS_LLAMA_ARCH_QWEN2 && l.bias_set != 7) {
      ns_set_error("ns_llama: layer %zu is missing q / k / v biases (Qwen2)", i);
      return NS_E_INVALID;
    }
  }
  return NS_OK;
}

// One forward pass of m rows, of one of two kinds:
//   one sequence (!segs): rows are the positions state[1] .. of KV block `seq`, attention through launch_attention (the ring
//     variant for a one-row step when `ring`); the logits of the last row, the pick in c->state.
//   segments (segs): rows 0 .. d - 1 are one-token segments, their row states and KV blocks in bstate (launch_attention_batch);
//     rows d .. m - 1 the longer segments, on the ragged tables rows / tiles (launch_attention_ragged); the logits of each
//     segment's last row, the picks in bstate.  d == m is a batched decode step: no ragged launch and no gather.
// advance: each pick becomes its row's next token at the next position, recorded at record (+ r n_ctx for row r).  sample (while
// sampling is on): 2 = store the windows and draw, 1 = store the windows and take each row's first candidate (a prompt piece whose
// pick is not returned), 0 = neither (the eager pass before a capture, evaluated again by the graph).
struct Pass {
  int m = 0;
  const int* toks = nullptr;  // device: row r's token id at toks[r * tok_stride] (embed_kernel<TSTRIDE>)
  int tok_stride = 1;
  bool segs = false;
  int seq = 0;                // one sequence: its KV block
  bool ring = false;          // one sequence: one-row steps rotate the StreamingLLM ring
  int n = 0, d = 0, n_tiles = 0;
  const int* rows = nullptr;   // device [m][2]: {position, KV block}
  const int* tiles = nullptr;  // device [n_tiles][kTileInts], rows counted from row d
  const int* last = nullptr;   // device [n]: last row of each segment (null when d == m: row r is segment r)
  const int* slot = nullptr;   // device [n]: KV block of each segment
  const int* draw = nullptr;   // device [n]: internal segment of caller index i (null: the identity)
  int advance = 0;
  int* record = nullptr;
  int sample = 2;
};

// the decode graph's pass: one row of block 0, token and position in c->state, every pick fed back and recorded
static Pass decode_pass(ns_llama* c) {
  Pass s;
  s.m = 1;
  s.toks = c->state;
  s.ring = c->streaming;
  s.advance = 1;
  s.record = c->record;
  return s;
}

// n one-token segments staged in bstate: ids read there too (stride 4), so that a graph replay feeds each pick back
static Pass rows_pass(ns_llama* c, int n) {
  Pass s;
  s.m = s.n = s.d = n;
  s.segs = true;
  s.toks = c->bstate;
  s.tok_stride = 4;
  s.slot = c->bstate + 4 * kMaxSeq;
  return s;
}

// the caches from unit 0 (layer 0, block 0, kv head 0) on
static KvPtrs kv_base(const ns_llama* c) {
  KvPtrs p;
  p.type = c->kv_type;
  p.k = c->kc;
  p.v = c->vc;
  p.kd = c->kd;
  p.vd = c->vd;
  return p;
}

// the embedding and every layer: leaves the last layer's output rows in c->x
static int enqueue_body(ns_llama* c, const Pass& p) {
  const ns_llama_hparams& hp = c->hp;
  cudaStream_t st = c->st;
  const int m = p.m, E = hp.n_embd, hd = E / hp.n_head, kvd = hd * hp.n_head_kv;
  float* q = c->qkv;
  float* k = q + (size_t)m * E;
  float* v = k + (size_t)m * kvd;
  NS_CUDA_TRY(ns_launch_pdl(p.tok_stride == 4 ? embed_kernel<4> : embed_kernel<1>, dim3((unsigned)((E / 4 + 255) / 256), (unsigned)m),
                            dim3(256), 0, st, (const float*)c->tok_embd, p.toks, E, hp.n_vocab, c->x));
  ns_count_launch();
  for (int il = 0; il < hp.n_layer; ++il) {
    const Layer& L = c->layers[il];
    const KvPtrs kv = kv_base(c).at(((size_t)il * c->n_seq + p.seq) * hp.n_head_kv, hp.n_ctx, hd);  // segments: block 0 of the layer
    // Decode rows: the attention RMSNorm (llama.cpp:205-210) rides in the activation quantiser of the Q/K/V launch(es) -- every
    // CTA reads the whole row anyway -- instead of a one-CTA kernel and a launch boundary of its own.
    const ns_weight* qkvw[3] = {L.wq, L.wk, L.wv};
    // one fused QKV node (llama.cpp:212-215) where the three weights form one, dst = [3][m][E] = q | k | v; else three matmuls.
    // Qwen2's biases ride in the epilogues: a QKV node takes them for one row or on the wgmma path (ns_qkv_bias_ok)
    const int qkv_path = hp.n_head == hp.n_head_kv ? ns_route(NS_NODE_QKV, qkvw, m, 0) : -1;
    const bool qkv_node = qkv_path >= 0 && (!L.bias || ns_qkv_bias_ok(qkv_path, m));
    const bool fold = qkv_node ? ns_rmsnorm_fusable(qkvw, 3, m)
                               : (hp.n_head != hp.n_head_kv || L.bias) && ns_rmsnorm_fusable(&qkvw[0], 1, m) &&
                                     ns_rmsnorm_fusable(&qkvw[1], 1, m) && ns_rmsnorm_fusable(&qkvw[2], 1, m);
    if (!fold)
      if (int rc = launch_rmsnorm(c->x, L.attn_norm, c->xn, m, E, hp.norm_eps, st)) return rc;
    const float* xq = fold ? c->x : c->xn;
    if (qkv_node) {
      if (int rc = ns_mul_qkv_norm(L.wq, L.wk, L.wv, xq, E, q, E, m, c->ws, (void*)st, fold ? L.attn_norm : nullptr, hp.norm_eps, L.bias))
        return rc;
    } else {
      float* dq[3] = {q, k, v};
      const float* bq[3] = {L.bias, L.bias ? L.bias + E : nullptr, L.bias ? L.bias + E + kvd : nullptr};
      for (int i = 0; i < 3; ++i)
        if (int rc = ns_mul_mat_bias(qkvw[i], xq, E, dq[i], i ? kvd : E, m, bq[i], c->ws, st, fold ? L.attn_norm : nullptr,
                                     fold ? hp.norm_eps : 0.f))
          return rc;
    }
    if (p.segs) {
      const int d = p.d;
      if (d > 0)
        if (int rc = launch_attention_batch(q, k, v, kv, c->bstate, c->bstate + 4 * kMaxSeq, c->attn, c->attn_part, c->attn_tickets, d,
                                            hp.n_head, hp.n_head_kv, hd, hp.n_ctx, hp.rope_theta, hp.rope_scale, c->attn_attr, st))
          return rc;
      if (d < m)
        if (int rc = launch_attention_ragged(q + (size_t)d * E, k + (size_t)d * kvd, v + (size_t)d * kvd, kv, p.rows + 2 * d, p.tiles,
                                             m - d, p.n_tiles, c->attn + (size_t)d * E, hp.n_head, hp.n_head_kv, hd, hp.n_ctx,
                                             hp.rope_theta, hp.rope_scale, st))
          return rc;
    } else {
      if (int rc = launch_attention(NS_ATTN_AUTO, q, k, v, kv, c->state, c->attn, c->attn_part, c->attn_tickets, hp.n_head, hp.n_head_kv,
                                    hd, hp.n_ctx, m, hp.rope_theta, hp.rope_scale, c->attn_attr, st, p.ring ? &c->ring : nullptr))
        return rc;
    }
    // inpFF = wo * attn + inpSA, written over x (every row is read by its own output only after the matmul finished)
    if (int rc = ns_mul_mat_engine(L.wo, c->attn, E, c->xn, E, m, c->x, c->ws, st, nullptr, 0.f)) return rc;
    // xn now holds inpFF; FFN + residual back into x, the FFN RMSNorm folded into the gate/up launch where that is a ring GEMV,
    // else normalised into attn (free again) first
    const ns_weight* guw[2] = {L.w1, L.w3};
    if (ns_rmsnorm_fusable(guw, 2, m)) {
      if (int rc = ns_ffn_silu_residual(L.w1, L.w2, L.w3, c->xn, E, c->tmp, c->x, E, m, c->xn, c->ws, st, L.ffn_norm, hp.norm_eps, 1)) return rc;
    } else {
      if (int rc = launch_rmsnorm(c->xn, L.ffn_norm, c->attn, m, E, hp.norm_eps, st)) return rc;
      if (int rc = ns_ffn_silu_residual(L.w1, L.w2, L.w3, c->attn, E, c->tmp, c->x, E, m, c->xn, c->ws, st, nullptr, 0.f, 1)) return rc;
    }
  }
  return NS_OK;
}

// logits = output * (rms_norm(x) * out_norm) over `rows` rows (llama.cpp:707-719): the final RMSNorm folded into the lm_head's
// launch when `fold`, else x is normalised already and goes through ns_mul_mat with `flags`
static int launch_lm_head(ns_llama* c, const float* x, int rows, bool fold, int flags, float* logits) {
  const ns_llama_hparams& hp = c->hp;
  return fold ? ns_rmsnorm_mul_mat(c->output, x, hp.n_embd, c->out_norm, hp.norm_eps, logits, hp.n_vocab, rows, nullptr, c->ws, (void*)c->st)
              : ns_mul_mat(c->output, x, hp.n_embd, logits, hp.n_vocab, rows, nullptr, nullptr, flags, c->ws, (void*)c->st);
}

// the body, then the logits and the pick of the last row (model_eval keeps the last row unless logits_all), or of each segment's
// last row (llama.cpp:745-758)
static int enqueue_forward(ns_llama* c, const Pass& p) {
  if (int rc = enqueue_body(c, p)) return rc;
  const ns_llama_hparams& hp = c->hp;
  cudaStream_t st = c->st;
  const int E = hp.n_embd;
  const int rows = p.segs ? p.n : 1;
  const float* xl = c->x + (size_t)(p.m - rows) * E;
  if (p.last) {  // each segment's last row, gathered into attn (free after the last layer)
    NS_CUDA_TRY(ns_launch_pdl(gather_rows_kernel, dim3((unsigned)((E / 4 + 255) / 256), (unsigned)rows), dim3(256), 0, st,
                              (const float*)c->x, p.last, E, c->attn));
    ns_count_launch();
    xl = c->attn;
  }
  const ns_weight* outw[1] = {c->output};
  const bool fold = ns_rmsnorm_fusable(outw, 1, rows);
  if (!fold) {
    if (int rc = launch_rmsnorm(xl, c->out_norm, c->xn, rows, E, hp.norm_eps, st)) return rc;
    xl = c->xn;
  }
  if (int rc = launch_lm_head(c, xl, rows, fold, 0, c->logits)) return rc;
  int* state = p.segs ? c->bstate : c->state;  // a segments pass: a pick per row
  const int n_tokens = p.segs ? 1 : p.m;
  if (c->sampling || c->per_seq) {
    SampleLaunch a{};
    a.logits = c->logits;
    a.n_vocab = hp.n_vocab;
    a.rows = rows;
    a.k = c->per_seq ? kSampleMaxK : c->smp.top_k;  // per block: the scratch stride, and the shared memory of any top_k
    a.top_p = c->smp.top_p;
    a.temp = c->smp.temperature;
    a.penalty = c->smp.repeat_penalty;
    a.W = c->smp.repeat_last_n < hp.n_ctx ? c->smp.repeat_last_n : hp.n_ctx;
    a.win = c->win;
    a.win_stride = kSampleMaxWindow;
    a.toks = p.toks;
    a.tok_stride = p.tok_stride;
    a.tok_len = n_tokens;
    a.last = p.last;
    a.slot = p.slot;
    a.slot_const = p.seq;
    a.order = p.draw;
    a.store = p.sample >= 1;
    a.draw = p.sample >= 2;
    a.mt = c->per_seq ? c->seq_mt : c->mt;
    a.cfg = c->per_seq ? c->seq_cfg : nullptr;
    a.pkeys = c->s_keys;
    a.pcnt = c->s_pcnt;
    a.cp = c->s_cp;
    a.tickets = c->s_tickets;
    a.kept = c->s_kept;
    a.ids = c->s_ids;
    a.probs = c->s_probs;
    a.state = state;
    a.rowwise = p.segs;
    a.n_tokens = n_tokens;
    a.advance = p.advance;
    a.record = p.record;
    a.rec_stride = hp.n_ctx;
    return ns_launch_sample(a, st);
  }
  return ns_launch_argmax(c->logits, hp.n_vocab, rows, p.segs, state, n_tokens, p.advance, p.record, hp.n_ctx, c->am_val, c->am_idx,
                          c->am_ticket, st);
}

// Captures pass p into slot g on first use.  One eager pass first sets kernel attributes and sizes every lazily grown buffer
// outside the capture.  It writes the K/V rows the captured pass rewrites with the same values, and nothing else that lasts: it
// does not advance, records nothing, leaves the windows and the generator alone, and runs the plain attention even while
// streaming -- a ring step rotates the cache, which must happen once; the plain kernel writes nothing once the cache is full.
static int capture(ns_llama* c, const Pass& p, Graph& g) {
  if (g.exec) return NS_OK;
  Pass warm = p;
  warm.ring = false;
  warm.advance = 0;
  warm.record = nullptr;
  warm.sample = 0;
  if (int rc = enqueue_forward(c, warm)) return rc;
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));
  NS_CUDA_TRY(cudaStreamBeginCapture(c->st, cudaStreamCaptureModeThreadLocal));
  int rc = enqueue_forward(c, p);
  cudaGraph_t graph = nullptr;
  cudaError_t e = cudaStreamEndCapture(c->st, &graph);
  if (rc) {
    if (graph) cudaGraphDestroy(graph);
    return rc;
  }
  if (!ns_cuda_ok(e, "cudaStreamEndCapture") || !graph) return NS_E_CUDA;
  if (!ns_cuda_ok(cudaGraphInstantiate(&g.exec, graph, 0), "cudaGraphInstantiate")) {
    cudaGraphDestroy(graph);
    return NS_E_CUDA;
  }
  g.graph = graph;
  return NS_OK;
}

// model_eval (models/model_utils/model_utils.h): evaluate n_tokens new tokens after n_past cached ones.
// logits_host (nullable): n_vocab floats of the LAST token; next_token (nullable): its greedy pick.
extern "C" int ns_llama_set_exact_prefill(ns_llama* c, int on) {
  if (!c) return NS_E_INVALID;
  c->exact_prefill = on ? 1 : 0;
  return NS_OK;
}

extern "C" int ns_llama_set_streaming(ns_llama* c, int n_keep) {
  if (!c || n_keep < -1 || n_keep >= c->hp.n_ctx) {
    ns_set_error("ns_llama_set_streaming: n_keep %d outside [-1, n_ctx)", n_keep);
    return NS_E_INVALID;
  }
  const int hd = c->hp.n_embd / c->hp.n_head;
  if (n_keep >= 0 && c->n_seq > 1) {
    ns_set_error("ns_llama_set_streaming: %d sequences (the ring serves one; llama.cpp:104 forbids the pair)", c->n_seq);
    return NS_E_UNSUPPORTED;
  }
  if (n_keep >= 0 && c->hp.rope_scale != 1.f) {
    ns_set_error("ns_llama_set_streaming: rope_scale %g != 1 (the reference's positions and shift table disagree)", c->hp.rope_scale);
    return NS_E_UNSUPPORTED;
  }
  if (n_keep >= 0 && hd != 64 && hd != 128) {
    ns_set_error("ns_llama_set_streaming: head size %d (the shift rides in the split decode attention: 64 or 128)", hd);
    return NS_E_UNSUPPORTED;
  }
  if (n_keep >= 0 && c->kv_type != NS_KV_F16) {
    ns_set_error("ns_llama_set_streaming: the KV cache is Q8_0 (the ring's shift would re-quantise every key on each wrap; set NS_KV_F16)");
    return NS_E_UNSUPPORTED;
  }
  if (n_keep >= 0 && neox(c)) {
    ns_set_error("ns_llama_set_streaming: a %s context (the reference has no NeoX shift-RoPE-K, qwen.cpp:85, phi3.cpp:188)",
                 c->arch == NS_LLAMA_ARCH_QWEN2 ? "Qwen2" : "Phi-3");
    return NS_E_UNSUPPORTED;
  }
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));  // nothing in flight replays the graph dropped below
  drop_graphs(c);
  c->streaming = n_keep >= 0;
  c->ring = Ring{n_keep, c->streaming ? shift_table(hd, c->hp.rope_theta) : ShiftTable{}};
  c->wrapped = false;
  return NS_OK;
}

// the sampler's generator, windows and scratch, allocated on first use
static int ensure_sampler(ns_llama* c) {
  if (!c->mt) {
    c->mt = (uint32_t*)dev_alloc(c, kMtWords * sizeof(uint32_t));
    c->win = (int*)dev_alloc(c, (size_t)kMaxSeq * kSampleMaxWindow * sizeof(int));
    c->s_keys = (unsigned long long*)dev_alloc(c, (size_t)kMaxSeq * kVocabSlices * kSampleMaxK * sizeof(unsigned long long));
    c->s_pcnt = (int*)dev_alloc(c, (size_t)kMaxSeq * kVocabSlices * sizeof(int));
    c->s_cp = (double*)dev_alloc(c, (size_t)kMaxSeq * kSampleMaxK * sizeof(double));
    c->s_tickets = (unsigned*)dev_alloc(c, (kMaxSeq + 1) * sizeof(unsigned));
    c->s_kept = (int*)dev_alloc(c, kMaxSeq * sizeof(int));
    c->s_ids = (int*)dev_alloc(c, (size_t)kMaxSeq * kSampleMaxK * sizeof(int));
    c->s_probs = (float*)dev_alloc(c, (size_t)kMaxSeq * kSampleMaxK * sizeof(float));
    if (!c->mt || !c->win || !c->s_keys || !c->s_pcnt || !c->s_cp || !c->s_tickets || !c->s_kept || !c->s_ids || !c->s_probs) {
      void* got[9] = {c->mt, c->win, c->s_keys, c->s_pcnt, c->s_cp, c->s_tickets, c->s_kept, c->s_ids, c->s_probs};
      for (void* p : got) dev_free(c, p);
      c->mt = nullptr;
      c->win = nullptr;
      c->s_keys = nullptr;
      c->s_pcnt = nullptr;
      c->s_cp = nullptr;
      c->s_tickets = nullptr;
      c->s_kept = nullptr;
      c->s_ids = nullptr;
      c->s_probs = nullptr;
      return NS_E_CUDA;
    }
    NS_CUDA_TRY(cudaMemsetAsync(c->s_tickets, 0, (kMaxSeq + 1) * sizeof(unsigned), c->st));
  }
  return NS_OK;
}

// Sampling in place of greedy (model_post_sample_top_k_top_p_repeat): the generator is reseeded and every window restarts;
// NULL returns to greedy.  Either way the context leaves per-sequence mode, and the captured graphs, which bake in the pick
// kernel and its parameters, are dropped.
extern "C" int ns_llama_set_sampling(ns_llama* c, const ns_llama_sampling* s) {
  if (!c) return NS_E_INVALID;
  if (s)
    if (int rc = ns_sample_check("ns_llama_set_sampling", s)) return rc;
  if (s)
    if (int rc = ensure_sampler(c)) return rc;
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));  // nothing in flight replays the graphs dropped below or reads the generator
  drop_graphs(c);
  c->per_seq = false;
  c->sampling = s != nullptr;
  if (!s) return NS_OK;
  c->smp = *s;
  uint32_t mt[kMtWords];
  ns_mt_seed(s->seed, mt);
  NS_CUDA_TRY(cudaMemcpy(c->mt, mt, sizeof(mt), cudaMemcpyHostToDevice));
  NS_CUDA_TRY(cudaMemsetAsync(c->win, 0, (size_t)kMaxSeq * kSampleMaxWindow * sizeof(int), c->st));
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));
  return NS_OK;
}

// per-sequence mode: every block greedy, every window zero (stream-ordered)
static int greedy_blocks(ns_llama* c) {
  SampleCfg g[kMaxSeq];
  for (int b = 0; b < kMaxSeq; ++b) {
    g[b] = ns_sample_cfg(nullptr, 0);
    c->seq_on[b] = false;
  }
  NS_CUDA_TRY(cudaMemcpyAsync(c->seq_cfg, g, sizeof(g), cudaMemcpyHostToDevice, c->st));
  NS_CUDA_TRY(cudaMemsetAsync(c->win, 0, (size_t)kMaxSeq * kSampleMaxWindow * sizeof(int), c->st));
  return NS_OK;
}

// Block seq samples with s from the next step on (its generator reseeded, its window restarted), or is greedy for s NULL.  The
// first call enters per-sequence mode and drops the graphs once; later calls only rewrite the block's table entry, generator and
// window, which the captured graphs read at replay.
extern "C" int ns_llama_set_sequence_sampling(ns_llama* c, int seq, const ns_llama_sampling* s) {
  const char* who = "ns_llama_set_sequence_sampling";
  if (!c) return NS_E_INVALID;
  if (seq < 0 || seq >= c->n_seq) {
    ns_set_error("%s: sequence id %d outside [0, %d)", who, seq, c->n_seq);
    return NS_E_INVALID;
  }
  if (s)
    if (int rc = ns_sample_check(who, s)) return rc;
  if (int rc = ensure_sampler(c)) return rc;
  if (!c->seq_cfg) {
    c->seq_cfg = (SampleCfg*)dev_alloc(c, kMaxSeq * sizeof(SampleCfg));
    c->seq_mt = (uint32_t*)dev_alloc(c, (size_t)kMaxSeq * kMtWords * sizeof(uint32_t));
    if (!c->seq_cfg || !c->seq_mt) {
      dev_free(c, c->seq_cfg);
      dev_free(c, c->seq_mt);
      c->seq_cfg = nullptr;
      c->seq_mt = nullptr;
      return NS_E_CUDA;
    }
  }
  cudaStream_t st = c->st;
  if (!c->per_seq) {
    NS_CUDA_TRY(cudaStreamSynchronize(st));  // nothing in flight replays the graphs dropped below
    drop_graphs(c);
    c->sampling = false;
    c->per_seq = true;
    if (int rc = greedy_blocks(c)) return rc;
  }
  const SampleCfg cfg = ns_sample_cfg(s, c->hp.n_ctx);
  NS_CUDA_TRY(cudaMemcpyAsync(c->seq_cfg + seq, &cfg, sizeof(cfg), cudaMemcpyHostToDevice, st));
  if (s) {
    uint32_t mt[kMtWords];
    ns_mt_seed(s->seed, mt);
    NS_CUDA_TRY(cudaMemcpyAsync(c->seq_mt + (size_t)seq * kMtWords, mt, sizeof(mt), cudaMemcpyHostToDevice, st));
  }
  NS_CUDA_TRY(cudaMemsetAsync(c->win + (size_t)seq * kSampleMaxWindow, 0, kSampleMaxWindow * sizeof(int), st));
  NS_CUDA_TRY(cudaStreamSynchronize(st));  // the host sources are consumed; the next step samples with the new config
  c->seq_on[seq] = s != nullptr;
  return NS_OK;
}

// a block samples: the context-wide sampler is on, or a block has its own config
static bool any_sampling(const ns_llama* c) {
  if (c->sampling) return true;
  for (int b = 0; c->per_seq && b < kMaxSeq; ++b)
    if (c->seq_on[b]) return true;
  return false;
}

// Positions of a streaming context: n_past is n_total.  Steps that reach past n_ctx take one token and continue the sequence;
// once such a step has run, only a continuation or a restart inside the sinks (n_past <= n_keep) is meaningful.
static int check_streaming(ns_llama* c, const char* who, int n_past, int n) {
  const int n_ctx = c->hp.n_ctx;
  if (!c->streaming) {
    if (n_past + n > n_ctx) {
      ns_set_error("%s: invalid arguments (n_tokens=%d n_past=%d n_ctx=%d)", who, n, n_past, n_ctx);
      return NS_E_INVALID;
    }
    return NS_OK;
  }
  const bool cont = n_past == c->n_total;
  if ((c->wrapped && !cont && n_past > c->ring.n_keep) || (n_past >= n_ctx && !cont)) {
    ns_set_error("%s: n_past %d is neither the next position %d nor a restart at <= n_keep %d of the full ring", who, n_past,
                 c->n_total, c->ring.n_keep);
    return NS_E_INVALID;
  }
  return NS_OK;
}

// the sequence position after a successful call
static void advance_position(ns_llama* c, int n_past, int n) {
  c->n_total = n_past + n;
  c->wrapped = c->streaming && ((c->wrapped && n_past > c->ring.n_keep) || n_past + n > c->hp.n_ctx);
}

// the sequences seq[i] evaluated at n_past[i] 0 restart their sampling windows as zeros (the reference's fresh history); nothing
// while greedy
static int reset_windows(ns_llama* c, int n, const int* seq, const int* n_past) {
  if (!c->sampling && !c->per_seq) return NS_OK;
  for (int i = 0; i < n; ++i)
    if (n_past[i] == 0) NS_CUDA_TRY(cudaMemsetAsync(c->win + (size_t)seq[i] * kSampleMaxWindow, 0, kSampleMaxWindow * sizeof(int), c->st));
  return NS_OK;
}

// c->state = {token, n_past, 0 recorded, 0} on KV block seq, whose sampling window restarts at n_past 0
static int stage_state(ns_llama* c, int seq, int token, int n_past) {
  if (int rc = reset_windows(c, 1, &seq, &n_past)) return rc;
  c->h_state[0] = token;
  c->h_state[1] = n_past;
  c->h_state[2] = 0;
  c->h_state[3] = 0;
  NS_CUDA_TRY(cudaMemcpyAsync(c->state, c->h_state, 4 * sizeof(int), cudaMemcpyHostToDevice, c->st));
  return NS_OK;
}

// ns_llama_eval on KV block `seq`: block 0 one-token steps replay the decode graph, every other step (prompts, and single
// tokens of the other blocks, whose graph would bake in the block) runs the same kernels eagerly
static int eval_block(ns_llama* c, int seq, const int32_t* tokens, int n_tokens, int n_past, float* logits_host, int32_t* next_token,
                      bool draw = true) {
  if (c->streaming && n_tokens > 1 && n_past + n_tokens > c->hp.n_ctx) {
    // the reference masks a multi-token step in slot order, which means nothing in ring order (llama.cpp:467, a TODO there)
    ns_set_error("ns_llama_eval: %d tokens past n_ctx %d: the ring takes one token per step", n_tokens, c->hp.n_ctx);
    return NS_E_UNSUPPORTED;
  }
  if (int rc = check_streaming(c, "ns_llama_eval", n_past, n_tokens)) return rc;
  if (c->exact_prefill && n_tokens > 32) {
    // parity mode: prompts go through in pieces of <= 32 tokens, which the matmuls run on the integer tensor cores with the
    // reference's exact block sums (causal attention over the fp16 KV cache makes the split invisible to the arithmetic)
    for (int t0 = 0; t0 < n_tokens; t0 += 32) {
      const int nt = n_tokens - t0 < 32 ? n_tokens - t0 : 32;
      const bool last = t0 + nt == n_tokens;
      if (int rc = eval_block(c, seq, tokens + t0, nt, n_past + t0, last ? logits_host : nullptr, last ? next_token : nullptr, last && draw))
        return rc;
    }
    return NS_OK;
  }
  if (int rc = check_complete(c)) return rc;
  if (int rc = ensure_buffers(c, n_tokens)) return rc;
  cudaStream_t st = c->st;
  if (int rc = stage_state(c, seq, tokens[0], n_past)) return rc;
  if (n_tokens == 1 && seq == 0 && draw) {
    if (int rc = capture(c, decode_pass(c), c->graph[0])) return rc;
    NS_CUDA_TRY(cudaGraphLaunch(c->graph[0].exec, st));
  } else {
    NS_CUDA_TRY(cudaMemcpyAsync(c->tokens, tokens, (size_t)n_tokens * sizeof(int), cudaMemcpyHostToDevice, st));
    Pass s;
    s.m = n_tokens;
    s.toks = c->tokens;
    s.seq = seq;
    s.advance = 1;
    s.sample = draw ? 2 : 1;
    if (int rc = enqueue_forward(c, s)) return rc;
  }
  if (logits_host) NS_CUDA_TRY(cudaMemcpyAsync(c->h_logits, c->logits, (size_t)c->hp.n_vocab * 4, cudaMemcpyDeviceToHost, st));
  NS_CUDA_TRY(cudaMemcpyAsync(c->h_state, c->state, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
  NS_CUDA_TRY(cudaStreamSynchronize(st));
  if (logits_host) memcpy(logits_host, c->h_logits, (size_t)c->hp.n_vocab * 4);
  if (next_token) *next_token = c->h_state[3];
  advance_position(c, n_past, n_tokens);
  return NS_OK;
}

extern "C" int ns_llama_eval(ns_llama* c, const int32_t* tokens, int n_tokens, int n_past, float* logits_host, int32_t* next_token) {
  if (int rc = ns_ensure_device()) return rc;
  if (!c || !tokens || n_tokens <= 0 || n_past < 0) {
    ns_set_error("ns_llama_eval: invalid arguments (n_tokens=%d n_past=%d n_ctx=%d)", n_tokens, n_past, c ? c->hp.n_ctx : 0);
    return NS_E_INVALID;
  }
  return eval_block(c, 0, tokens, n_tokens, n_past, logits_host, next_token);
}

extern "C" int ns_llama_eval_seq(ns_llama* c, int seq, const int32_t* tokens, int n_tokens, int n_past, float* logits_host,
                                 int32_t* next_token) {
  if (int rc = ns_ensure_device()) return rc;
  if (!c || !tokens || n_tokens <= 0 || n_past < 0) {
    ns_set_error("ns_llama_eval_seq: invalid arguments (n_tokens=%d n_past=%d n_ctx=%d)", n_tokens, n_past, c ? c->hp.n_ctx : 0);
    return NS_E_INVALID;
  }
  if (seq < 0 || seq >= c->n_seq) {
    ns_set_error("ns_llama_eval_seq: sequence id %d outside [0, %d)", seq, c->n_seq);
    return NS_E_INVALID;
  }
  return eval_block(c, seq, tokens, n_tokens, n_past, logits_host, next_token);
}

// 1 <= n_seq <= 32 KV blocks: every block restarts empty
extern "C" int ns_llama_set_sequences(ns_llama* c, int n_seq) {
  if (!c || n_seq < 1 || n_seq > kMaxSeq) {
    ns_set_error("ns_llama_set_sequences: n_seq %d outside [1, %d]", n_seq, kMaxSeq);
    return NS_E_INVALID;
  }
  const int hd = c->hp.n_embd / c->hp.n_head;
  if (n_seq > 1 && c->streaming) {
    ns_set_error("ns_llama_set_sequences: %d sequences with streaming on (llama.cpp:104 forbids the pair)", n_seq);
    return NS_E_UNSUPPORTED;
  }
  if (n_seq > 1 && !attn_fast_hd(hd)) {
    ns_set_error("ns_llama_set_sequences: head size %d (the batched decode attention takes 64, 96 or 128)", hd);
    return NS_E_UNSUPPORTED;
  }
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));  // nothing in flight uses the blocks or graphs released below
  drop_graphs(c);
  c->n_total = 0;
  c->wrapped = false;
  if (int rc = alloc_sequences(c, n_seq)) return rc;
  if (c->per_seq) return greedy_blocks(c);
  if (c->win) NS_CUDA_TRY(cudaMemsetAsync(c->win, 0, (size_t)kMaxSeq * kSampleMaxWindow * sizeof(int), c->st));
  return NS_OK;
}

// What a pass over several KV blocks needs of the context: head size 64, 96 or 128, streaming off, at most 32 rows in exact-prefill
// mode, every tensor set; then buffers for its rows.  Nothing is launched.  ragged: the error texts name the ragged attention too.
static int check_context(ns_llama* c, const char* who, int rows, bool ragged) {
  const int hd = c->hp.n_embd / c->hp.n_head;
  if (!attn_fast_hd(hd)) {
    ns_set_error("%s: head size %d (the batched decode %s 64, 96 or 128)", who, hd, ragged ? "and ragged prompt attention take" : "attention takes");
    return NS_E_UNSUPPORTED;
  }
  if (c->streaming) {
    ns_set_error("%s: streaming is on (the ring serves ns_llama_eval / ns_llama_generate only%s)", who, ragged ? "; llama.cpp:104" : "");
    return NS_E_UNSUPPORTED;
  }
  if (c->exact_prefill && rows > 32) {
    ns_set_error("%s: %d rows in exact-prefill mode (the integer block sums hold up to 32 rows)", who, rows);
    return NS_E_UNSUPPORTED;
  }
  if (int rc = check_complete(c)) return rc;
  return ensure_buffers(c, rows);
}

// bstate = the row states of a batched step: row j < d {tok[j], n_past[j * stride], 0, 0} of KV block block[j * stride], every
// other row zero
static int stage_rows(ns_llama* c, int d, const int32_t* tok, const int* n_past, const int* block, int stride) {
  for (int j = 0; j < kMaxSeq; ++j) {
    int* r = c->h_bstate + 4 * j;
    r[0] = j < d ? tok[j] : 0;
    r[1] = j < d ? n_past[j * stride] : 0;
    r[2] = r[3] = 0;
    c->h_bstate[4 * kMaxSeq + j] = j < d ? block[j * stride] : 0;
  }
  NS_CUDA_TRY(cudaMemcpyAsync(c->bstate, c->h_bstate, (size_t)kMaxSeq * 5 * sizeof(int), cudaMemcpyHostToDevice, c->st));
  return NS_OK;
}

// n one-token rows {tokens[i], n_past[i]} of KV blocks seq[i], staged as a batched step; that step's graph captured on first use
static int stage_batch(ns_llama* c, int n, const int* seq, const int32_t* tokens, const int* n_past) {
  if (int rc = reset_windows(c, n, seq, n_past)) return rc;
  if (int rc = stage_rows(c, n, tokens, n_past, seq, 1)) return rc;
  Pass s = rows_pass(c, n);
  s.advance = 1;
  s.record = c->brecord;
  return capture(c, s, c->graph[n]);
}

// the logits and picks of the n rows of the pass just enqueued, on the host: row j is caller index order[j] (the identity if null)
static int read_rows(ns_llama* c, int n, const int* order, float* logits_host, int32_t* next_tokens) {
  cudaStream_t st = c->st;
  const size_t nv = (size_t)c->hp.n_vocab;
  if (logits_host) NS_CUDA_TRY(cudaMemcpyAsync(c->h_logits, c->logits, n * nv * 4, cudaMemcpyDeviceToHost, st));
  NS_CUDA_TRY(cudaMemcpyAsync(c->h_bstate, c->bstate, (size_t)n * 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
  NS_CUDA_TRY(cudaStreamSynchronize(st));
  for (int j = 0; j < n; ++j) {
    const int i = order ? order[j] : j;
    if (logits_host) memcpy(logits_host + (size_t)i * nv, c->h_logits + (size_t)j * nv, nv * 4);
    if (next_tokens) next_tokens[i] = c->h_bstate[4 * j + 3];
  }
  return NS_OK;
}

// one batched decode step: staged, the graph of n rows replayed, logits and picks back in the rows' order
static int decode_step(ns_llama* c, int n, const int* seq, const int32_t* tokens, const int* n_past, float* logits_host,
                       int32_t* next_tokens) {
  if (int rc = stage_batch(c, n, seq, tokens, n_past)) return rc;
  NS_CUDA_TRY(cudaGraphLaunch(c->graph[n].exec, c->st));
  return read_rows(c, n, nullptr, logits_host, next_tokens);
}

// the argument rules of a batched decode call: n rows of distinct KV blocks, `steps` new positions each
static int check_steps(ns_llama* c, const char* who, int n, const int* seq, const int32_t* tokens, const int* n_past, int steps) {
  if (!c || !seq || !tokens || !n_past) {
    ns_set_error("%s: null pointer", who);
    return NS_E_INVALID;
  }
  if (steps <= 0) {
    ns_set_error("%s: %d steps", who, steps);
    return NS_E_INVALID;
  }
  if (int rc = check_rows(who, c->n_seq, n, seq, n_past, steps, c->hp.n_ctx)) return rc;
  return check_context(c, who, n, false);
}

extern "C" int ns_llama_decode_batch(ns_llama* c, int n, const int* seq, const int32_t* tokens, const int* n_past, float* logits_host,
                                     int32_t* next_tokens) {
  if (int rc = ns_ensure_device()) return rc;
  if (int rc = check_steps(c, "ns_llama_decode_batch", n, seq, tokens, n_past, 1)) return rc;
  return decode_step(c, n, seq, tokens, n_past, logits_host, next_tokens);
}

extern "C" int ns_llama_generate_batch(ns_llama* c, int n, const int* seq, const int32_t* first_tokens, const int* n_past, int n_new,
                                       int32_t* out_tokens) {
  if (int rc = ns_ensure_device()) return rc;
  if (!out_tokens) {
    ns_set_error("ns_llama_generate_batch: null pointer");
    return NS_E_INVALID;
  }
  if (int rc = check_steps(c, "ns_llama_generate_batch", n, seq, first_tokens, n_past, n_new)) return rc;
  if (int rc = stage_batch(c, n, seq, first_tokens, n_past)) return rc;
  cudaStream_t st = c->st;
  for (int i = 0; i < n_new; ++i) NS_CUDA_TRY(cudaGraphLaunch(c->graph[n].exec, st));
  // row r's picks: brecord[r][0 .. n_new) (n_past + n_new <= n_ctx)
  NS_CUDA_TRY(cudaMemcpy2DAsync(out_tokens, (size_t)n_new * sizeof(int), c->brecord, (size_t)c->hp.n_ctx * sizeof(int),
                                (size_t)n_new * sizeof(int), (size_t)n, cudaMemcpyDeviceToHost, st));
  NS_CUDA_TRY(cudaStreamSynchronize(st));
  return NS_OK;
}

// The device tables of a pass over the segments of plan p: ids in internal order, rows, tiles, each segment's last row, block and
// draw order, and the one-token rows' states as a batched step's.  *s describes the pass.
static int stage_segments(ns_llama* c, int n, const int* seq, const int* n_tokens, const int32_t* tokens, const int* n_past,
                          const BatchPlan& p, Pass* s) {
  cudaStream_t st = c->st;
  if (!c->plan) {
    c->plan = (int*)dev_alloc(c, (size_t)kPlanInts * sizeof(int));
    if (!c->plan) return NS_E_CUDA;
    if (!ns_cuda_ok(cudaMallocHost((void**)&c->h_plan, (size_t)(kMaxBatchRows + kPlanInts) * sizeof(int)), "cudaMallocHost")) {
      c->h_plan = nullptr;
      dev_free(c, c->plan);
      c->plan = nullptr;
      return NS_E_CUDA;
    }
  }
  if (p.T > c->tok_cap) {  // nothing captured reads c->tokens: only the eager passes in flight, drained first
    NS_CUDA_TRY(cudaStreamSynchronize(st));
    dev_free(c, c->tokens);
    c->tokens = (int*)dev_alloc(c, (size_t)p.T * sizeof(int));
    c->tok_cap = c->tokens ? p.T : 0;
    if (!c->tokens) return NS_E_CUDA;
  }
  // staging: ids in internal order | rows | tiles | last rows
  int* h_tok = c->h_plan;
  int* h_tab = c->h_plan + kMaxBatchRows;
  std::vector<int> off(n, 0);  // first id of segment i in `tokens` (caller's order)
  for (int i = 1; i < n; ++i) off[i] = off[i - 1] + n_tokens[i - 1];
  int* h_last = h_tab + 2 * kMaxBatchRows + kPlanTiles * kTileInts;
  for (int j = 0; j < n; ++j) {
    const int i = p.order[j];
    memcpy(h_tok + p.first[j], tokens + off[i], (size_t)n_tokens[i] * sizeof(int));
    h_last[j] = p.first[j] + n_tokens[i] - 1;
    h_last[kMaxSeq + j] = seq[i];
    h_last[2 * kMaxSeq + i] = j;
  }
  if (int rc = reset_windows(c, n, seq, n_past)) return rc;
  std::copy(p.rows.begin(), p.rows.end(), h_tab);
  std::copy(p.tiles.begin(), p.tiles.end(), h_tab + 2 * kMaxBatchRows);
  NS_CUDA_TRY(cudaMemcpyAsync(c->tokens, h_tok, (size_t)p.T * sizeof(int), cudaMemcpyHostToDevice, st));
  NS_CUDA_TRY(cudaMemcpyAsync(c->plan, h_tab, (size_t)kPlanInts * sizeof(int), cudaMemcpyHostToDevice, st));
  // the one-token segments come first: row j < d has its id at h_tok[j] and its position and block at p.rows[2 j ..]
  if (int rc = stage_rows(c, p.d, h_tok, &p.rows[0], &p.rows[1], 2)) return rc;
  *s = rows_pass(c, n);
  if (p.d == n) return NS_OK;
  const int* d_last = c->plan + 2 * kMaxBatchRows + kPlanTiles * kTileInts;
  s->m = p.T;  // ids from c->tokens, the last rows gathered
  s->toks = c->tokens;
  s->tok_stride = 1;
  s->d = p.d;
  s->n_tiles = (int)p.tiles.size() / kTileInts;
  s->rows = c->plan;
  s->tiles = c->plan + 2 * kMaxBatchRows;
  s->last = d_last;
  s->slot = d_last + kMaxSeq;
  s->draw = d_last + 2 * kMaxSeq;
  return NS_OK;
}

// model_eval over n inputs (llama.cpp:53-90, 329-460, 745-758): one pass over the token segments of n distinct sequences
extern "C" int ns_llama_eval_batch(ns_llama* c, int n, const int* seq, const int* n_tokens, const int32_t* tokens, const int* n_past,
                                   float* logits_host, int32_t* next_tokens) {
  const char* who = "ns_llama_eval_batch";
  if (int rc = ns_ensure_device()) return rc;
  if (!c || !tokens) {
    ns_set_error("%s: null pointer", who);
    return NS_E_INVALID;
  }
  BatchPlan p;
  if (int rc = plan_batch(who, c->n_seq, c->hp.n_ctx, n, seq, n_tokens, n_past, p)) return rc;
  if (int rc = check_context(c, who, p.T, true)) return rc;
  // one-token segments only: the captured batched step (the plan keeps those segments in the caller's order)
  if (p.d == n) return decode_step(c, n, seq, tokens, n_past, logits_host, next_tokens);
  Pass s;
  if (int rc = stage_segments(c, n, seq, n_tokens, tokens, n_past, p, &s)) return rc;
  if (int rc = enqueue_forward(c, s)) return rc;
  return read_rows(c, n, p.order.data(), logits_host, next_tokens);
}

static int ensure_all_rows(ns_llama* c) {
  if (c->all_logits) return NS_OK;
  const size_t V = (size_t)c->hp.n_vocab;
  float* lg = (float*)dev_alloc(c, (size_t)kAllChunk * V * 4);
  unsigned* tk = (unsigned*)dev_alloc(c, (size_t)kAllChunk * (1 + 3 * kVocabSlices) * 4);
  int* io = (int*)dev_alloc(c, (size_t)3 * kMaxBatchRows * 4);
  int* h = nullptr;
  cudaEvent_t ev[2] = {};
  bool ok = lg && tk && io && cudaMallocHost((void**)&h, ((size_t)3 * kMaxBatchRows + 2 * kAllChunk * V) * 4) == cudaSuccess;
  for (int i = 0; i < 2 && ok; ++i) ok = cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming) == cudaSuccess;
  ok = ok && cudaMemsetAsync(tk, 0, (size_t)kAllChunk * 4, c->st) == cudaSuccess;
  if (!ok) {
    ns_set_error("ns_llama_eval_all: allocation failed");
    for (void* q : {(void*)lg, (void*)tk, (void*)io}) dev_free(c, q);
    if (h) cudaFreeHost(h);
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);
    return NS_E_CUDA;
  }
  c->all_logits = lg;
  c->lp_tickets = tk;
  c->all_io = io;
  c->h_all = h;
  c->all_ev[0] = ev[0];
  c->all_ev[1] = ev[1];
  return NS_OK;
}

// model_eval with logits_all (llama.cpp:743-747) over the segments of ns_llama_eval_batch: the same body, then the final RMSNorm
// over all T rows (folded into the lm_head where enqueue_forward folds it: one chunk of a row count ns_rmsnorm_fusable takes) and,
// per chunk of <= kAllChunk rows, the lm_head on its own route -- never the bf16 GEMM -- and one log-prob launch
extern "C" int ns_llama_eval_all(ns_llama* c, int n, const int* seq, const int* n_tokens, const int32_t* tokens, const int* n_past,
                                 const int32_t* targets, float* logprobs, int32_t* argmax, float* logits_host) {
  const char* who = "ns_llama_eval_all";
  if (int rc = ns_ensure_device()) return rc;
  if (!c || !tokens) {
    ns_set_error("%s: null pointer", who);
    return NS_E_INVALID;
  }
  BatchPlan p;
  if (int rc = plan_batch(who, c->n_seq, c->hp.n_ctx, n, seq, n_tokens, n_past, p)) return rc;
  const int V = c->hp.n_vocab, E = c->hp.n_embd, T = p.T;
  if ((!targets) != (!logprobs) || (!logprobs && !argmax && !logits_host)) {
    ns_set_error("%s: targets and logprobs must be both null or both non-null, and one output at least non-null", who);
    return NS_E_INVALID;
  }
  if (targets)
    for (int r = 0; r < T; ++r)
      if (targets[r] < 0 || targets[r] >= V) {
        ns_set_error("%s: target %d of row %d outside [0, n_vocab %d)", who, targets[r], r, V);
        return NS_E_INVALID;
      }
  if (any_sampling(c)) {
    ns_set_error("%s: sampling is on (a scoring pass draws nothing; set greedy first)", who);
    return NS_E_UNSUPPORTED;
  }
  if (int rc = check_context(c, who, T, true)) return rc;
  if (int rc = ensure_all_rows(c)) return rc;
  cudaStream_t st = c->st;
  Pass s;
  if (int rc = stage_segments(c, n, seq, n_tokens, tokens, n_past, p, &s)) return rc;
  // caller row of each internal row; targets up in internal order
  std::vector<int> off(n, 0), dst(T);
  for (int i = 1; i < n; ++i) off[i] = off[i - 1] + n_tokens[i - 1];
  for (int j = 0; j < n; ++j)
    for (int t = 0; t < n_tokens[p.order[j]]; ++t) dst[p.first[j] + t] = off[p.order[j]] + t;
  int* h_tgt = c->h_all;
  float* h_lp = reinterpret_cast<float*>(c->h_all + kMaxBatchRows);
  int* h_am = c->h_all + 2 * kMaxBatchRows;
  float* h_stage = reinterpret_cast<float*>(c->h_all + 3 * kMaxBatchRows);
  if (targets) {
    for (int r = 0; r < T; ++r) h_tgt[r] = targets[dst[r]];
    NS_CUDA_TRY(cudaMemcpyAsync(c->all_io, h_tgt, (size_t)T * 4, cudaMemcpyHostToDevice, st));
  }
  if (int rc = enqueue_body(c, s)) return rc;
  const ns_weight* outw[1] = {c->output};
  const bool fold = T <= kAllChunk && ns_rmsnorm_fusable(outw, 1, T);
  if (!fold)
    if (int rc = launch_rmsnorm(c->x, c->out_norm, c->xn, T, E, c->hp.norm_eps, st)) return rc;
  const float* xh = fold ? c->x : c->xn;  // the lm_head's input rows
  LogprobLaunch a{};
  a.logits = c->all_logits;
  a.n_vocab = V;
  a.tickets = c->lp_tickets;
  a.pmax = reinterpret_cast<float*>(c->lp_tickets + kAllChunk);
  a.pidx = reinterpret_cast<int*>(a.pmax + kAllChunk * kVocabSlices);
  a.psum = reinterpret_cast<float*>(a.pidx + kAllChunk * kVocabSlices);
  int* d_lp = c->all_io + kMaxBatchRows;
  int* d_am = c->all_io + 2 * kMaxBatchRows;
  const size_t chunk_floats = (size_t)kAllChunk * V;
  auto scatter = [&](int k) {  // chunk k's logits, staged in buffer k & 1, to the caller's rows
    const float* src = h_stage + (size_t)(k & 1) * chunk_floats;
    const int r0 = k * kAllChunk, rows = std::min(kAllChunk, T - r0);
    for (int r = 0; r < rows; ++r) memcpy(logits_host + (size_t)dst[r0 + r] * V, src + (size_t)r * V, (size_t)V * 4);
  };
  for (int k = 0; k * kAllChunk < T; ++k) {
    const int r0 = k * kAllChunk, rows = std::min(kAllChunk, T - r0);
    // the lm_head never takes the bf16 GEMM: a chunk ns_route would send there takes GEMV tiles
    const int flags = ns_route(NS_NODE_PLAIN, outw, rows, 0) == NS_PATH_TC ? NS_MM_FORCE_GEMV : 0;
    if (int rc = launch_lm_head(c, xh + (size_t)r0 * E, rows, fold, flags, c->all_logits)) return rc;
    a.rows = rows;
    a.targets = targets ? c->all_io + r0 : nullptr;
    a.logprobs = targets ? reinterpret_cast<float*>(d_lp + r0) : nullptr;
    a.argmax = d_am + r0;
    if (int rc = ns_launch_logprob(a, st)) return rc;
    if (logits_host) {  // the host copies chunk k - 1 out while the device runs chunk k
      NS_CUDA_TRY(cudaMemcpyAsync(h_stage + (size_t)(k & 1) * chunk_floats, c->all_logits, (size_t)rows * V * 4, cudaMemcpyDeviceToHost, st));
      NS_CUDA_TRY(cudaEventRecord(c->all_ev[k & 1], st));
      if (k > 0) {
        NS_CUDA_TRY(cudaEventSynchronize(c->all_ev[(k - 1) & 1]));
        scatter(k - 1);
      }
    }
  }
  if (logprobs) NS_CUDA_TRY(cudaMemcpyAsync(h_lp, d_lp, (size_t)T * 4, cudaMemcpyDeviceToHost, st));
  if (argmax) NS_CUDA_TRY(cudaMemcpyAsync(h_am, d_am, (size_t)T * 4, cudaMemcpyDeviceToHost, st));
  NS_CUDA_TRY(cudaStreamSynchronize(st));
  if (logits_host) scatter((T - 1) / kAllChunk);
  for (int r = 0; r < T; ++r) {
    if (logprobs) logprobs[dst[r]] = h_lp[r];
    if (argmax) argmax[dst[r]] = h_am[r];
  }
  return NS_OK;
}

// greedy generation: token `first` at position n_past, then n_new - 1 more, each fed from the previous argmax on the
// device (one graph launch per token, no host synchronisation in between).  out_tokens[i] = pick after step i.
extern "C" int ns_llama_generate(ns_llama* c, int32_t first_token, int n_past, int n_new, int32_t* out_tokens) {
  if (int rc = ns_ensure_device()) return rc;
  if (!c || !out_tokens || n_new <= 0 || n_past < 0) {
    ns_set_error("ns_llama_generate: invalid arguments (n_past=%d n_new=%d n_ctx=%d)", n_past, n_new, c ? c->hp.n_ctx : 0);
    return NS_E_INVALID;
  }
  if (int rc = check_streaming(c, "ns_llama_generate", n_past, n_new)) return rc;
  if (int rc = check_complete(c)) return rc;
  if (int rc = ensure_buffers(c, 1)) return rc;
  if (int rc = capture(c, decode_pass(c), c->graph[0])) return rc;
  cudaStream_t st = c->st;
  if (int rc = stage_state(c, 0, first_token, n_past)) return rc;
  // the record buffer holds n_ctx picks: a streaming generation past n_ctx drains it in pieces (stream-ordered, no host wait)
  for (int i0 = 0; i0 < n_new; i0 += c->hp.n_ctx) {
    const int n = n_new - i0 < c->hp.n_ctx ? n_new - i0 : c->hp.n_ctx;
    if (i0) NS_CUDA_TRY(cudaMemsetAsync(c->state + 2, 0, sizeof(int), st));
    for (int i = 0; i < n; ++i) NS_CUDA_TRY(cudaGraphLaunch(c->graph[0].exec, st));
    NS_CUDA_TRY(cudaMemcpyAsync(out_tokens + i0, c->record, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
  }
  NS_CUDA_TRY(cudaStreamSynchronize(st));
  advance_position(c, n_past, n_new);
  return NS_OK;
}

// ---- beam search ------------------------------------------------------------------------------------------------------
// The engine of the flow in beam.cu: the prompt pass is ns_llama_eval_batch's, a step is ns_llama_decode_batch's captured step
// without its readback; each is followed by one candidates launch over the logits and one copy of the candidates to the host.
namespace {
struct DeviceBeams : BeamEngine {
  ns_llama* c;
  int n;
  const int* n_tokens;
  const int32_t* tokens;
  int eos;
  const BatchPlan* plan;
  // K candidates of the rows of the pass just enqueued: logits row j is caller row order[j] (the identity if null)
  int candidates(const BeamRows& rows, const int* order, int K, BeamCand* out) {
    BeamLaunch a{};
    a.logits = c->logits;
    a.n_vocab = c->hp.n_vocab;
    a.rows = rows.n;
    a.k = K;
    a.eos = eos;
    for (int j = 0; j < rows.n; ++j) {
      const int i = order ? order[j] : j;
      a.prev[j] = rows.prev[i];
      if (rows.mask[i]) a.mask |= 1u << j;
    }
    a.out = c->beam_out;
    a.tickets = c->beam_ws;
    ns_beam_scratch(a, c->beam_ws + kBeamMaxRows, rows.n, K);
    if (int rc = ns_launch_beam_candidates(a, c->st)) return rc;
    NS_CUDA_TRY(cudaMemcpyAsync(c->h_beam, c->beam_out, (size_t)rows.n * K * sizeof(BeamCand), cudaMemcpyDeviceToHost, c->st));
    NS_CUDA_TRY(cudaStreamSynchronize(c->st));
    for (int j = 0; j < rows.n; ++j) memcpy(out + (size_t)(order ? order[j] : j) * K, c->h_beam + (size_t)j * K, (size_t)K * sizeof(BeamCand));
    return NS_OK;
  }
  int prompts(const BeamRows& rows, int K, BeamCand* out) override {
    std::vector<int> seq(rows.block, rows.block + n), n_past(n, 0);
    if (plan->d == n) {  // one-token prompts: the captured batched step, as ns_llama_eval_batch takes it
      if (int rc = stage_batch(c, n, seq.data(), tokens, n_past.data())) return rc;
      NS_CUDA_TRY(cudaGraphLaunch(c->graph[n].exec, c->st));
      return candidates(rows, nullptr, K, out);
    }
    Pass s;
    if (int rc = stage_segments(c, n, seq.data(), n_tokens, tokens, n_past.data(), *plan, &s)) return rc;
    if (int rc = enqueue_forward(c, s)) return rc;
    return candidates(rows, plan->order.data(), K, out);
  }
  int step(const BeamRows& rows, int K, BeamCand* out) override {
    if (int rc = stage_batch(c, rows.n, rows.block, rows.tok, rows.n_past)) return rc;
    NS_CUDA_TRY(cudaGraphLaunch(c->graph[rows.n].exec, c->st));
    return candidates(rows, nullptr, K, out);
  }
  int copy(const KvCopyPairs& p) override {
    const ns_llama_hparams& hp = c->hp;
    return ns_launch_kv_copy(p, kv_base(c), hp.n_layer, c->n_seq, hp.n_head_kv, hp.n_ctx, hp.n_embd / hp.n_head, c->st);
  }
};
}  // namespace

static int ensure_beams(ns_llama* c) {
  if (c->beam_ws) return NS_OK;
  const size_t wsb = (size_t)kBeamMaxRows * 4 + ns_beam_scratch_bytes(kBeamMaxRows, kBeamMaxK);
  unsigned* ws = (unsigned*)dev_alloc(c, wsb);
  BeamCand* out = (BeamCand*)dev_alloc(c, (size_t)kBeamMaxRows * kBeamMaxK * sizeof(BeamCand));
  BeamCand* h = nullptr;
  bool ok = ws && out && cudaMallocHost((void**)&h, (size_t)kBeamMaxRows * kBeamMaxK * sizeof(BeamCand)) == cudaSuccess;
  ok = ok && cudaMemsetAsync(ws, 0, (size_t)kBeamMaxRows * 4, c->st) == cudaSuccess;
  if (!ok) {
    ns_set_error("ns_llama_beam_search: allocation failed");
    dev_free(c, ws);
    dev_free(c, out);
    if (h) cudaFreeHost(h);
    return NS_E_CUDA;
  }
  c->beam_ws = ws;
  c->beam_out = out;
  c->h_beam = h;
  return NS_OK;
}

extern "C" int ns_llama_beam_search(ns_llama* c, int n, const int* n_tokens, const int32_t* tokens, const ns_llama_beams* cfg,
                                    int32_t* out_tokens, int* out_len, float* out_score) {
  const char* who = "ns_llama_beam_search";
  if (int rc = ns_ensure_device()) return rc;
  if (!c || !n_tokens || !tokens || !cfg || !out_tokens || !out_len) {
    ns_set_error("%s: null pointer", who);
    return NS_E_INVALID;
  }
  const int hd = c->hp.n_embd / c->hp.n_head;
  if (any_sampling(c) || c->streaming || !attn_fast_hd(hd)) {
    ns_set_error("%s: %s", who, any_sampling(c) ? "sampling is on (the reference searches beams only with do_sample off)"
                                : c->streaming ? "streaming is on (the reference's beam search has no shifted cache, model_utils.cpp:2245)"
                                               : "head size other than 64 / 96 / 128 (the batched decode attention)");
    return NS_E_UNSUPPORTED;
  }
  if (int rc = ns_beam_check(who, cfg, n, n_tokens, c->hp.n_ctx, c->hp.n_vocab, c->n_seq)) return rc;
  const int B = cfg->num_beams;
  std::vector<int> seq(n), n_past(n, 0);
  for (int r = 0; r < n; ++r) seq[r] = r * B;
  BatchPlan p;
  if (int rc = plan_batch(who, c->n_seq, c->hp.n_ctx, n, seq.data(), n_tokens, n_past.data(), p)) return rc;
  if (int rc = check_context(c, who, std::max(p.T, n * B), true)) return rc;
  if (int rc = ensure_beams(c)) return rc;
  DeviceBeams e;
  e.c = c;
  e.n = n;
  e.n_tokens = n_tokens;
  e.tokens = tokens;
  e.eos = cfg->eos_token_id;
  e.plan = &p;
  return ns_beam_flow(*cfg, n, n_tokens, tokens, e, out_tokens, out_len, out_score);
}

extern "C" int ns_llama_kv_copy(ns_llama* c, int n, const int* src, const int* dst, int p0, int p1) {
  if (int rc = ns_ensure_device()) return rc;
  if (!c || !src || !dst || n < 1 || n > std::min(c->n_seq, kBeamMaxRows)) {
    ns_set_error("ns_llama_kv_copy: null pointer or %d pairs (1 .. %d)", n, c ? std::min(c->n_seq, kBeamMaxRows) : 0);
    return NS_E_INVALID;
  }
  KvCopyPairs a;
  a.n = n;
  for (int i = 0; i < n; ++i) {
    a.src[i] = src[i];
    a.dst[i] = dst[i];
    a.p0[i] = p0;
    a.p1[i] = p1;
  }
  const ns_llama_hparams& hp = c->hp;
  if (int rc = ns_launch_kv_copy(a, kv_base(c), hp.n_layer, c->n_seq, hp.n_head_kv, hp.n_ctx, hp.n_embd / hp.n_head, c->st)) return rc;
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));
  return NS_OK;
}

extern "C" int ns_llama_kv_cache(const ns_llama* c, void** k, void** v) {
  if (!c || !k || !v) return NS_E_INVALID;
  if (c->kv_type != NS_KV_F16) {
    ns_set_error("ns_llama_kv_cache: the KV cache is Q8_0 (ns_llama_kv_planes)");
    return NS_E_UNSUPPORTED;
  }
  *k = c->kc;
  *v = c->vc;
  return NS_OK;
}

extern "C" int ns_llama_kv_planes(const ns_llama* c, void** k, void** kd, void** v, void** vd) {
  if (!c || !k || !kd || !v || !vd) return NS_E_INVALID;
  *k = c->kc;
  *kd = c->kd;
  *v = c->vc;
  *vd = c->vd;
  return NS_OK;
}

extern "C" unsigned long long ns_llama_kv_bytes(const ns_llama* c) {
  if (!c) return 0;
  const size_t units = (size_t)c->n_seq * c->hp.n_layer * c->hp.n_head_kv;
  return (unsigned long long)2 * kv_cache_bytes(c->kv_type, units, c->hp.n_ctx, c->hp.n_embd / c->hp.n_head);
}

extern "C" int ns_llama_kv_type(const ns_llama* c) { return c ? c->kv_type : NS_E_INVALID; }

// every block reallocated in the new format and empty, the graphs dropped (as ns_llama_set_sequences)
extern "C" int ns_llama_set_kv_type(ns_llama* c, int type) {
  if (!c || (type != NS_KV_F16 && type != NS_KV_Q8_0)) {
    ns_set_error("ns_llama_set_kv_type: type %d (NS_KV_F16 %d or NS_KV_Q8_0 %d)", type, NS_KV_F16, NS_KV_Q8_0);
    return NS_E_INVALID;
  }
  const int hd = c->hp.n_embd / c->hp.n_head;
  if (type == NS_KV_Q8_0 && c->streaming) {
    ns_set_error("ns_llama_set_kv_type: streaming is on (the ring's shift would re-quantise every key on each wrap)");
    return NS_E_UNSUPPORTED;
  }
  if (type == NS_KV_Q8_0 && hd != 64 && hd != 128) {
    ns_set_error("ns_llama_set_kv_type: head size %d (the Q8_0 KV cache is read by the head size 64 / 128 kernels)", hd);
    return NS_E_UNSUPPORTED;
  }
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));  // nothing in flight uses the blocks or graphs released below
  drop_graphs(c);
  c->n_total = 0;
  c->wrapped = false;
  c->kv_type = type;
  if (int rc = alloc_sequences(c, c->n_seq > 0 ? c->n_seq : 1)) return rc;
  if (c->win) NS_CUDA_TRY(cudaMemsetAsync(c->win, 0, (size_t)kMaxSeq * kSampleMaxWindow * sizeof(int), c->st));
  return NS_OK;
}

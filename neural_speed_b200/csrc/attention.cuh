// attention.cuh -- what the eval step (llama.cu) calls in attention.cu: the attention launchers of one layer and the plan of a
// pass over the token segments of several sequences.
#pragma once
#include <cuda_fp16.h>

#include <vector>

#include "kv_cache.cuh"
#include "nsb.cuh"

constexpr int kMaxSeq = 32;  // KV blocks of one context (ns_llama_set_sequences)
constexpr int kMaxBatchRows = 4096;  // rows of one pass over segments; the caller chunks longer prompts
constexpr int kAttnMmaRows = 64, kAttnMmaKeys = 64;
constexpr int kTileInts = 5;  // ints per entry of the ragged tile table

// Head sizes of the split decode and tensor-core prompt attention with an fp16 KV cache: one-row steps, prompts, the batched decode
// and the ragged prompt attention, so every pass over several KV blocks and beam search.
constexpr bool attn_fast_hd(int hd) { return hd == 64 || hd == 96 || hd == 128; }
// Head sizes where attn_fast_kernel (NS_ATTN_ROWS), the streaming ring and the Q8_0 KV cache exist as well
constexpr bool attn_all_hd(int hd) { return hd == 64 || hd == 128; }

struct AttnAttr {  // dynamic shared memory already granted to each kernel (function attributes are per device)
  struct Grant {
    const void* kern;
    size_t smem;
  } granted[17];  // 17 attention kernels can ask for more than 48 KB
  int n = 0;
};
// {cos, sin} of the one-position back shift per rotary pair, fp16 (model_utils.cpp:165-192); passed by value
struct ShiftTable {
  __half2 cs[64];
};

int attn_ranges(int n_ctx);  // 256-position ranges of the split decode attention
size_t attn_rows_smem(int hd, int n_ctx);  // dynamic shared memory of attn_fast_kernel
ShiftTable shift_table(int hd, float freq_base);

// part: [n_head][attn_ranges(n_ctx)][hd + 2] floats, tickets: [n_head] zero words (both read by attn_decode_kernel only; the
// last CTA of a head leaves its ticket at zero again).  ring (nullable): one-token steps run the ring variant of the split decode
// attention with ring->n_keep sink slots; prompts (m > 1, which never reach past n_ctx) run the plain kernels.
struct Ring {
  int n_keep;
  ShiftTable tab;
};
// kv: the layer's caches of the sequence's block (kv_cache.cuh)
int launch_attention(int kind, float* q, const float* k, const float* v, const KvPtrs& kv, const int* state, float* out,
                     float* part, unsigned* tickets, int n_head, int n_head_kv, int hd, int n_ctx, int m, float rope_theta,
                     float rope_scale, AttnAttr& attr, cudaStream_t st, const Ring* ring);

// Batched decode attention: one new token for each of n sequences, one launch (attn_decode_kernel<HD, false, true>).  rstate:
// [n][4] row states (n_past in slot 1), seqs [n] KV block per row, caches from the layer's block 0 on, q / out
// [n][n_head * hd], k / v [n][n_head_kv * hd], part [n][n_head][ranges][hd + 2], tickets [n][n_head].  hd 64 / 96 / 128
// (attn_fast_hd), 96 with an fp16 cache only.
int launch_attention_batch(const float* q, const float* k, const float* v, const KvPtrs& kv, const int* rstate,
                           const int* seqs, float* out, float* part, unsigned* tickets, int n, int n_head, int n_head_kv, int hd,
                           int n_ctx, float rope_theta, float rope_scale, AttnAttr& attr, cudaStream_t st);

// Ragged prompt attention: RoPE + KV append of n_rows rows (rows [n_rows][2] = {position, block}), then attn_mma_kernel<RAGGED> over
// n_tiles tile entries.  q / out [n_rows][n_head * hd], k / v [n_rows][n_head_kv * hd], caches from the layer's block 0 on.
int launch_attention_ragged(float* q, const float* k, const float* v, const KvPtrs& kv, const int* rows, const int* tiles,
                            int n_rows, int n_tiles, float* out, int n_head, int n_head_kv, int hd, int n_ctx, float rope_theta,
                            float rope_scale, cudaStream_t st);

// Checks the rows of a batched call: 1 <= n <= n_seq, every id in [0, n_seq) and distinct, 0 <= n_past[i], n_past[i] + steps <= n_ctx
int check_rows(const char* who, int n_seq, int n, const int* seq, const int* n_past, int steps, int n_ctx);

// The plan of ns_llama_eval_batch: internal order = the one-token segments, then the longer ones, each group in the caller's order.
// Rows 0 .. d - 1 take the batched decode attention, rows d .. T - 1 the ragged prompt attention (tile rows counted from row d).
struct BatchPlan {
  int T = 0, d = 0;
  std::vector<int> order, first, rows, tiles;
};
int plan_batch(const char* who, int n_seq, int n_ctx, int n, const int* seq, const int* n_tokens, const int* n_past,
               BatchPlan& p);

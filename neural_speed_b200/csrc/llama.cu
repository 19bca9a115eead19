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
//
// One token (n_tokens == 1) is ONE CUDA graph: the token id and n_past live in device memory (`state`), so the same graph
// replays for every position; ns_llama_generate chains graph launches with the argmax feeding the next embedding
// lookup on the device -- no host round trip per token.
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

namespace {

struct Layer {
  const float* attn_norm = nullptr;
  const float* ffn_norm = nullptr;
  const ns_weight *wq = nullptr, *wk = nullptr, *wv = nullptr, *wo = nullptr, *w1 = nullptr, *w2 = nullptr, *w3 = nullptr;
};

constexpr int kAttnThreads = 128;

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

// rope (mode 0) on q and k of every new token + append k,v to the fp16 cache.
// grid (n_head + n_head_kv, n_tokens), hd/2 threads.  pos = state[1] + t.
// RAGGED: the rows belong to segments of several sequences (ns_llama_eval_batch); row t takes its position and its KV block
// ([n_seq][n_head_kv][n_ctx][hd]) from rows[2 t], rows[2 t + 1] instead.
template <bool RAGGED = false>
__global__ void rope_kv_kernel(float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk, const float* __restrict__ v, int ldv,
                               __half* __restrict__ kc, __half* __restrict__ vc, const int* __restrict__ state, int n_head, int n_head_kv,
                               int hd, int n_ctx, float theta_scale, float freq_scale, const int* __restrict__ rows) {
  pdl_launch_dependents();
  pdl_wait();
  const int h = blockIdx.x, t = blockIdx.y, i = threadIdx.x;  // pair index
  int pos;
  if (RAGGED) {
    pos = rows[2 * t];
    const size_t blk = (size_t)rows[2 * t + 1] * n_head_kv * n_ctx * hd;
    kc += blk;
    vc += blk;
  } else {
    pos = state[1] + t;
  }
  // theta_base = p; repeated `theta_base *= theta_scale` (ne_layers.c:9321,9385): keep the same sequence of roundings
  float theta = (float)pos;
  for (int j = 0; j < i; ++j) theta *= theta_scale;
  theta *= freq_scale;
  float sn, cs;
  sincosf(theta, &sn, &cs);
  if (h < n_head) {
    float* p = q + (size_t)t * ldq + (size_t)h * hd + 2 * i;
    const float x0 = p[0], x1 = p[1];
    p[0] = x0 * cs - x1 * sn;
    p[1] = x0 * sn + x1 * cs;
  } else {
    const int hk = h - n_head;
    const float* p = k + (size_t)t * ldk + (size_t)hk * hd + 2 * i;
    const float x0 = p[0], x1 = p[1];
    if (pos < n_ctx) {
      __half* kd = kc + ((size_t)hk * n_ctx + pos) * hd + 2 * i;
      kd[0] = __float2half_rn(x0 * cs - x1 * sn);
      kd[1] = __float2half_rn(x0 * sn + x1 * cs);
      const float* pv = v + (size_t)t * ldv + (size_t)hk * hd + 2 * i;
      __half* vd = vc + ((size_t)hk * n_ctx + pos) * hd + 2 * i;
      vd[0] = __float2half_rn(pv[0]);
      vd[1] = __float2half_rn(pv[1]);
    }
  }
}

// one CTA per (head, new token): two-pass softmax over positions 0 .. state[1] + t, scores in shared memory.
// out[t][h*hd + d] = sum_i fp16(p_i) * V[i][d]
__global__ void __launch_bounds__(kAttnThreads) attn_kernel(const float* __restrict__ q, int ldq, const __half* __restrict__ kc,
                                                            const __half* __restrict__ vc, const int* __restrict__ state, float* __restrict__ out,
                                                            int ldo, int n_head, int n_head_kv, int hd, int n_ctx, float scale) {
  extern __shared__ float sm[];  // [hd] q (fp16-rounded) | [n_ctx] scores
  pdl_launch_dependents();
  pdl_wait();
  const int h = blockIdx.x, t = blockIdx.y;
  const int hk = h / (n_head / n_head_kv);
  int len = state[1] + t + 1;
  len = len > n_ctx ? n_ctx : len;
  float* sq = sm;
  float* sc = sm + hd;
  const float* qr = q + (size_t)t * ldq + (size_t)h * hd;
  for (int d = threadIdx.x; d < hd; d += blockDim.x) sq[d] = __half2float(__float2half_rn(qr[d]));
  __syncthreads();
  const __half* kh = kc + (size_t)hk * n_ctx * hd;
  const __half* vh = vc + (size_t)hk * n_ctx * hd;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  // pass 1: scores (one warp per position)
  float lmax = -INFINITY;
  for (int i = warp; i < len; i += nw) {
    const __half2* kr = (const __half2*)(kh + (size_t)i * hd);
    float acc = 0.f;
    for (int d2 = lane; d2 < hd / 2; d2 += 32) {
      const float2 kv = __half22float2(kr[d2]);
      acc = fmaf(sq[2 * d2], kv.x, acc);
      acc = fmaf(sq[2 * d2 + 1], kv.y, acc);
    }
    acc = warp_sum(acc) * scale;
    if (lane == 0) sc[i] = acc;
    lmax = fmaxf(lmax, acc);
  }
  __shared__ float red[kAttnThreads / 32];
  __shared__ float bcast;
  if (lane == 0) red[warp] = lmax;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = red[0];
    for (int i = 1; i < nw; ++i) m = fmaxf(m, red[i]);
    bcast = m;
  }
  __syncthreads();
  const float mx = bcast;
  // exp on the fp16-rounded argument, result rounded to fp16 (table_exp_f16), sum in fp32
  float lsum = 0.f;
  for (int i = threadIdx.x; i < len; i += blockDim.x) {
    const float a = __half2float(__float2half_rn(sc[i] - mx));
    const float e = __half2float(__float2half_rn(expf(a)));
    sc[i] = e;
    lsum += e;
  }
  lsum = warp_sum(lsum);
  __syncthreads();
  if (lane == 0) red[warp] = lsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < nw; ++i) s += red[i];
    bcast = 1.f / s;
  }
  __syncthreads();
  const float inv = bcast;
  // pass 2: thread d accumulates sum_i fp16(p_i) * V[i][d]
  for (int d = threadIdx.x; d < hd; d += blockDim.x) {
    float acc = 0.f;
    for (int i = 0; i < len; ++i) {
      const float p = __half2float(__float2half_rn(sc[i] * inv));
      acc = fmaf(p, __half2float(vh[(size_t)i * hd + d]), acc);
    }
    out[(size_t)t * ldo + (size_t)h * hd + d] = acc;
  }
}

// Decode-shaped attention for head sizes 64 / 128: kAW warps per (head, token); a warp streams whole K/V rows (one 4- or 8-byte
// load per lane), four rows in flight; with FUSE (single new token) the kernel also applies RoPE to its q head and to the
// new k row and appends k,v to the cache, so rope_kv_kernel is not launched.
constexpr int kAW = 16;  // warps per CTA: the kernel is a chain of dependent cache-row loads, more warps = more rows in flight
template <int HD, bool FUSE>
__global__ void __launch_bounds__(kAW * 32) attn_fast_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ knew, int ldk,
                                                        const float* __restrict__ vnew, int ldv, __half* __restrict__ kc,
                                                        __half* __restrict__ vc, const int* __restrict__ state, float* __restrict__ out, int ldo,
                                                        int n_head, int n_head_kv, int n_ctx, float scale, float theta_scale,
                                                        float freq_scale) {
  constexpr int EPL = HD / 32;  // elements per lane
  extern __shared__ float sm[];  // [HD] q | [HD] new k | [HD] new v | [kAW][HD] partial out | [n_ctx] scores
  float* sq = sm;
  float* sk = sm + HD;
  float* sv = sm + 2 * HD;
  float* part = sm + 3 * HD;
  float* sc = sm + 3 * HD + kAW * HD;
  pdl_launch_dependents();
  pdl_wait();
  const int h = blockIdx.x, t = blockIdx.y;
  const int group = n_head / n_head_kv, hk = h / group;
  const int pos = state[1] + t;
  int len = pos + 1;
  len = len > n_ctx ? n_ctx : len;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __half* kh = kc + (size_t)hk * n_ctx * HD;
  __half* vh = vc + (size_t)hk * n_ctx * HD;
  const float* qr = q + (size_t)t * ldq + (size_t)h * HD;
  if (FUSE) {
    if (threadIdx.x < HD / 2) {
      const int i = threadIdx.x;
      float theta = (float)pos;
      for (int j = 0; j < i; ++j) theta *= theta_scale;  // ne_layers.c:9385: same sequence of roundings
      theta *= freq_scale;
      float sn, cs;
      sincosf(theta, &sn, &cs);
      const float q0 = qr[2 * i], q1 = qr[2 * i + 1];
      sq[2 * i] = __half2float(__float2half_rn(q0 * cs - q1 * sn));
      sq[2 * i + 1] = __half2float(__float2half_rn(q0 * sn + q1 * cs));
      const float* kr = knew + (size_t)t * ldk + (size_t)hk * HD;
      const float k0 = kr[2 * i], k1 = kr[2 * i + 1];
      const __half r0 = __float2half_rn(k0 * cs - k1 * sn), r1 = __float2half_rn(k0 * sn + k1 * cs);
      sk[2 * i] = __half2float(r0);
      sk[2 * i + 1] = __half2float(r1);
      const float* vr = vnew + (size_t)t * ldv + (size_t)hk * HD;
      const __half w0 = __float2half_rn(vr[2 * i]), w1 = __float2half_rn(vr[2 * i + 1]);
      sv[2 * i] = __half2float(w0);
      sv[2 * i + 1] = __half2float(w1);
      if (h % group == 0 && pos < n_ctx) {  // one CTA per kv head appends to the cache
        *(__half2*)(kh + (size_t)pos * HD + 2 * i) = __halves2half2(r0, r1);
        *(__half2*)(vh + (size_t)pos * HD + 2 * i) = __halves2half2(w0, w1);
      }
    }
  } else {
    for (int d = threadIdx.x; d < HD; d += blockDim.x) sq[d] = __half2float(__float2half_rn(qr[d]));
  }
  __syncthreads();
  float ql[EPL];
#pragma unroll
  for (int e = 0; e < EPL; ++e) ql[e] = sq[lane * EPL + e];
  const int ncache = FUSE ? len - 1 : len;  // rows read from the cache; the new row comes from shared memory when fused

  auto load_row = [&](const __half* base, int i, float* dst) {
    if (EPL == 4) {
      const uint2 u = *(const uint2*)(base + (size_t)i * HD + lane * 4);
      const float2 a = __half22float2(*(const __half2*)&u.x), b = __half22float2(*(const __half2*)&u.y);
      dst[0] = a.x, dst[1] = a.y, dst[2] = b.x, dst[3] = b.y;
    } else {
      const __half2 u = *(const __half2*)(base + (size_t)i * HD + lane * 2);
      const float2 a = __half22float2(u);
      dst[0] = a.x, dst[1] = a.y;
    }
  };
  // pass 1: scores
  for (int i0 = warp * 4; i0 < ncache; i0 += kAW * 4) {
    float kr[4][EPL];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (i0 + u < ncache) load_row(kh, i0 + u, kr[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (i0 + u < ncache) {  // warp-uniform
        float acc = 0.f;
#pragma unroll
        for (int e = 0; e < EPL; ++e) acc = fmaf(ql[e], kr[u][e], acc);
        acc = warp_sum(acc);
        if (lane == 0) sc[i0 + u] = acc * scale;
      }
    }
  }
  if (FUSE && warp == 0 && len - 1 == ncache) {
    float acc = 0.f;
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc = fmaf(ql[e], sk[lane * EPL + e], acc);
    acc = warp_sum(acc);
    if (lane == 0) sc[len - 1] = acc * scale;
  }
  __syncthreads();
  __shared__ float red[kAW];
  __shared__ float bcast;
  float lmax = -INFINITY;
  for (int i = threadIdx.x; i < len; i += blockDim.x) lmax = fmaxf(lmax, sc[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
  if (lane == 0) red[warp] = lmax;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = red[0];
    for (int i = 1; i < kAW; ++i) m = fmaxf(m, red[i]);
    bcast = m;
  }
  __syncthreads();
  const float mx = bcast;
  float lsum = 0.f;
  for (int i = threadIdx.x; i < len; i += blockDim.x) {
    const float a = __half2float(__float2half_rn(sc[i] - mx));
    const float e = __half2float(__float2half_rn(expf(a)));  // table_exp_f16 (ne_layers.c:8933-8937)
    sc[i] = e;
    lsum += e;
  }
  lsum = warp_sum(lsum);
  __syncthreads();
  if (lane == 0) red[warp] = lsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s2 = 0.f;
    for (int i = 0; i < kAW; ++i) s2 += red[i];
    bcast = 1.f / s2;
  }
  __syncthreads();
  const float inv = bcast;
  // pass 2: each warp accumulates its rows, lanes own EPL output elements; then the 8 partials are summed
  float acc[EPL];
#pragma unroll
  for (int e = 0; e < EPL; ++e) acc[e] = 0.f;
  for (int i0 = warp * 4; i0 < ncache; i0 += kAW * 4) {
    float vr[4][EPL];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (i0 + u < ncache) load_row(vh, i0 + u, vr[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (i0 + u < ncache) {
        const float p = __half2float(__float2half_rn(sc[i0 + u] * inv));
#pragma unroll
        for (int e = 0; e < EPL; ++e) acc[e] = fmaf(p, vr[u][e], acc[e]);
      }
  }
  if (FUSE && warp == 0 && len - 1 == ncache) {
    const float p = __half2float(__float2half_rn(sc[len - 1] * inv));
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc[e] = fmaf(p, sv[lane * EPL + e], acc[e]);
  }
#pragma unroll
  for (int e = 0; e < EPL; ++e) part[warp * HD + lane * EPL + e] = acc[e];
  __syncthreads();
  for (int d = threadIdx.x; d < HD; d += blockDim.x) {
    float s2 = 0.f;
#pragma unroll
    for (int w = 0; w < kAW; ++w) s2 += part[w * HD + d];
    out[(size_t)t * ldo + (size_t)h * HD + d] = s2;
  }
}

// ---- decode attention: K / V of the head staged by TMA, split over the context ---------------------------------------------------
// One new token (llama.cpp:286-302 with N = 1; RoPE of q and of the new k row and the KV append fused in, as attn_fast_kernel<FUSE>).
// grid (n_head, ceil(n_ctx / 256)); CTA (h, s) owns cached positions [256 s, 256 s + 256) of head h and returns at once when the
// sequence has not reached its range (the position lives in device memory: one CUDA graph serves every position).  The rows of a
// head are contiguous in the cache ([kv head][n_ctx][hd] fp16), so the CTA's whole K and V ranges arrive as TWO cp.async.bulk copies
// (<= 64 KB each) on one mbarrier: a single global-memory latency per launch instead of a chain of dependent row loads -- the old
// kernel spent 2-3 round trips per pass at 100-200 positions.  Scores, soft_max and P.V then run out of shared memory.
// One active range (<= 256 positions): exactly the reference arithmetic (global maximum, e = fp16(exp(fp16(s - max))),
// p = fp16(e / sum), fp32 sums).  Several: every CTA leaves {max, sum e, sum e V} of its range, the last one to arrive (ticket per
// head) merges them with exp(max_s - max) weights -- same values up to the fp16 rounding of p (measured: tests/test_gpu_attention.py).
// Bound: latency at short contexts; HBM (2 x len x hd x 2 B per kv head) at long ones, spread over n_head x ceil(len / 256) CTAs.
//
// RING = true: the StreamingLLM ring of the reference's shift-RoPE-K mode (llama.cpp:102-107, 351-354, 430-470), grid
// (n_head_kv, ranges).  One CTA per (kv head, range) serves every query head of its group from the one staged tile, so no two CTAs
// of a launch touch the same K row.  Until the cache is full (state[1] < n_ctx) each head's arithmetic is the RING = false
// kernel's.  Once it is full, with n_total = state[1]: q is rotated at n_ctx - 1, the new k at n_ctx (fp32, then fp16) and stored
// with v in slot n_keep + (n_total - n_ctx) mod (n_ctx - n_keep), inside whichever range holds it; then every staged K row at or
// past n_keep, the new one included, is rotated one position back with the fp16 shift table (ne_layers.c:9514-9526), scored
// and written back with one bulk store; attention covers all n_ctx slots with no mask.
//
// BATCH = true: one new token for each of n sequences (continuous batching, llama.cpp:414-489 run per request), grid
// (n_head, ranges, n).  CTA z serves row z: its position is state[4 z + 1] (the row's {token, n_past, n_recorded, pick}), its
// KV block seqs[z] ([n_seq][n_head_kv][n_ctx][hd] per layer), and its q / k / v / out rows, partials and tickets are row z's.
// Everything after those offsets is the RING = false kernel's code, so each row's arithmetic is the single-sequence step's.
constexpr int kSplitKeys = 256;
constexpr int kDW = 16;  // warps per CTA
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
template <int HD>
static constexpr size_t attn_decode_smem() {
  return (size_t)2 * kSplitKeys * HD * 2 + (size_t)(3 + kDW) * HD * 4 + (size_t)(kSplitKeys + 8) * 4 + 16;
}
// {cos, sin} of the one-position back shift per rotary pair, fp16 (model_utils.cpp:165-192); passed by value
struct ShiftTable {
  __half2 cs[64];
};
template <int HD, bool RING, bool BATCH = false>
__global__ void __launch_bounds__(kDW * 32) attn_decode_kernel(const float* __restrict__ q, const float* __restrict__ knew,
                                                            const float* __restrict__ vnew, __half* __restrict__ kc, __half* __restrict__ vc,
                                                            const int* __restrict__ state, float* __restrict__ out, float* __restrict__ part_ws,
                                                            unsigned* __restrict__ tickets, int n_head, int n_head_kv, int n_ctx, int nsplit,
                                                            float scale, float theta_scale, float freq_scale, int n_keep, const ShiftTable tab,
                                                            const int* __restrict__ seqs) {
  static_assert(!(RING && BATCH), "the ring serves one sequence");
  constexpr int EPL = HD / 32;
  extern __shared__ __align__(128) unsigned char smraw[];
  __half* Kt = reinterpret_cast<__half*>(smraw);  // [kSplitKeys][HD]
  __half* Vt = Kt + kSplitKeys * HD;
  float* sq = reinterpret_cast<float*>(Vt + kSplitKeys * HD);
  float* sk = sq + HD;
  float* sv = sk + HD;
  float* part = sv + HD;         // [kDW][HD]
  float* sc = part + kDW * HD;   // [kSplitKeys + 1]: scores of the range (+ the new row)
  unsigned long long* bar = reinterpret_cast<unsigned long long*>(sc + kSplitKeys + 8);
  __shared__ float red[kDW];
  __shared__ float bcast;
  __shared__ int last_flag;
  pdl_launch_dependents();
  // The position was written by the PREVIOUS token's argmax kernel (an earlier graph launch / an H2D copy ahead of this eval's
  // first kernel), never by a kernel of this token: it may be read before griddepcontrol.wait.  CTAs whose range the sequence
  // has not reached leave at once, without holding 141 KB of an SM until the Q/K/V launch in front of this one has drained.
  const int split = blockIdx.y;
  const int group = n_head / n_head_kv;
  const int hk = RING ? (int)blockIdx.x : (int)blockIdx.x / group;
  const int h0 = RING ? hk * group : (int)blockIdx.x;  // query heads h0 .. h0 + nh - 1
  const int nh = RING ? group : 1;
  const int row = BATCH ? (int)blockIdx.z : 0;
  const int pos = state[4 * row + 1];
  const bool wrapped = RING && pos >= n_ctx;
  const int len = min(pos + 1, n_ctx);
  const int nact = (len + kSplitKeys - 1) / kSplitKeys;
  if (split >= nact) return;
  if (BATCH) {  // the row's KV block, activations, partials and tickets (the sequence ids, like the positions, precede this step)
    const size_t blk = (size_t)seqs[row] * n_head_kv * n_ctx * HD;
    kc += blk;
    vc += blk;
    q += (size_t)row * n_head * HD;
    knew += (size_t)row * n_head_kv * HD;
    vnew += (size_t)row * n_head_kv * HD;
    out += (size_t)row * n_head * HD;
    part_ws += (size_t)row * n_head * nsplit * (HD + 2);
    tickets += (size_t)row * n_head;
  }
  const int i0 = split * kSplitKeys, i1 = min(len, i0 + kSplitKeys);
  const int slot = wrapped ? n_keep + (pos - n_ctx) % (n_ctx - n_keep) : pos;  // cache row of the token being evaluated
  const bool has_new = wrapped ? slot >= i0 && slot < i1 : (i1 == len) && pos < n_ctx;  // ... sits in this range
  const bool tail_new = has_new && !wrapped;  // ... after the staged rows, its k / v from registers (else staged over its slot)
  const int ncache = (tail_new ? i1 - 1 : i1) - i0;  // rows staged from the cache
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __half* kh = kc + (size_t)hk * n_ctx * HD;
  __half* vh = vc + (size_t)hk * n_ctx * HD;
  const uint32_t bar_a = smem_addr(bar);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar_a), "r"(1) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    // the cached rows of this range were written by earlier tokens' launches: their copies start before the wait as well and
    // overlap the tail of the Q/K/V launch.  In the ring, the rows this token rewrites (shifted K, the new K / V slot) were
    // likewise last written by this layer's launch of the previous token -- the launch whose appended row the plain step
    // already reads here -- so the same ordering covers them.
    if (ncache > 0) {
      const uint32_t bytes = (uint32_t)ncache * HD * 2;
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(2 * bytes) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(Kt)),
                   "l"(kh + (size_t)i0 * HD), "r"(bytes), "r"(bar_a)
                   : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(Vt)),
                   "l"(vh + (size_t)i0 * HD), "r"(bytes), "r"(bar_a)
                   : "memory");
    }
  }
  __syncthreads();
  pdl_wait();  // q, k, v of the new token come from the launch in front
  auto rope_angle = [&](int p, int i, float* sn, float* cs) {
    float theta = (float)p;
    for (int j = 0; j < i; ++j) theta *= theta_scale;  // ne_layers.c:9385: same sequence of roundings
    theta *= freq_scale;
    sincosf(theta, sn, cs);
  };
  auto wait_tiles = [&]() {
    uint32_t ok;
    do {
      asm volatile(
          "{\n"
          ".reg .pred p;\n"
          "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
          "selp.u32 %0, 1, 0, p;\n"
          "}\n"
          : "=r"(ok)
          : "r"(bar_a), "r"(0)
          : "memory");
    } while (!ok);
  };
  // RoPE of the new k row; KV append by one CTA per kv head -- while the copies fly
  float qsn = 0.f, qcs = 0.f;  // the queries' angle (thread i < HD / 2: pair i)
  __half2 knew_h = __float2half2_rn(0.f), vnew_h = knew_h;
  if (threadIdx.x < HD / 2) {
    const int i = threadIdx.x;
    rope_angle(wrapped ? n_ctx - 1 : pos, i, &qsn, &qcs);  // llama.cpp:351: q at max(n_cached - N, n_past)
    if (has_new) {
      float sn = qsn, cs = qcs;
      if (wrapped) rope_angle(n_ctx, i, &sn, &cs);  // llama.cpp:353-354: the new k enters at n_ctx, shifted back below
      const float* kr = knew + (size_t)hk * HD;
      const float k0 = kr[2 * i], k1 = kr[2 * i + 1];
      const __half r0 = __float2half_rn(k0 * cs - k1 * sn), r1 = __float2half_rn(k0 * sn + k1 * cs);
      sk[2 * i] = __half2float(r0);
      sk[2 * i + 1] = __half2float(r1);
      const float* vr = vnew + (size_t)hk * HD;
      const __half w0 = __float2half_rn(vr[2 * i]), w1 = __float2half_rn(vr[2 * i + 1]);
      sv[2 * i] = __half2float(w0);
      sv[2 * i + 1] = __half2float(w1);
      knew_h = __halves2half2(r0, r1);
      vnew_h = __halves2half2(w0, w1);
      if (!wrapped && (RING || h0 % group == 0)) {
        *reinterpret_cast<__half2*>(kh + (size_t)pos * HD + 2 * i) = knew_h;
        *reinterpret_cast<__half2*>(vh + (size_t)pos * HD + 2 * i) = vnew_h;
      }
    }
  }
  const int shift0 = wrapped ? min(max(n_keep - i0, 0), ncache) : ncache;  // staged rows [shift0, ncache) are shifted
  if (wrapped) {
    wait_tiles();
    if (has_new && threadIdx.x < HD / 2) {  // the new row goes over its slot (write before shift: llama.cpp:408-409, :443)
      reinterpret_cast<__half2*>(Kt + (size_t)(slot - i0) * HD)[threadIdx.x] = knew_h;
      reinterpret_cast<__half2*>(Vt + (size_t)(slot - i0) * HD)[threadIdx.x] = vnew_h;
      reinterpret_cast<__half2*>(vh + (size_t)slot * HD)[threadIdx.x] = vnew_h;
    }
    __syncthreads();
    // blockDim.x is a multiple of HD / 2: a thread always meets the same rotary pair
    const float2 t = __half22float2(tab.cs[threadIdx.x % (HD / 2)]);
    __half2* kt2 = reinterpret_cast<__half2*>(Kt);
    for (int e = shift0 * (HD / 2) + threadIdx.x; e < ncache * (HD / 2); e += blockDim.x) {
      const float2 x = __half22float2(kt2[e]);
      // x0*cos - x1*sin, x1*cos + x0*sin (ne_layers.c:9524-9525): the products of two fp16 values are exact in fp32, so this
      // form rounds once per output, as every contraction of the reference's expressions does
      kt2[e] = __floats2half2_rn(fmaf(x.x, t.x, -(x.y * t.y)), fmaf(x.y, t.x, x.x * t.y));
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the shifted rows, visible to the bulk store
    __syncthreads();
    if (threadIdx.x == 0 && shift0 < ncache) {
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(kh + (size_t)(i0 + shift0) * HD),
                   "r"(smem_addr(Kt + (size_t)shift0 * HD)), "r"((uint32_t)(ncache - shift0) * HD * 2)
                   : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
  }
  for (int hi = 0; hi < nh; ++hi) {
  const int h = h0 + hi;
  if (threadIdx.x < HD / 2) {  // RoPE of this head's q (every range needs it)
    const int i = threadIdx.x;
    const float sn = qsn, cs = qcs;
    const float* qr = q + (size_t)h * HD;
    const float q0 = qr[2 * i], q1 = qr[2 * i + 1];
    sq[2 * i] = __half2float(__float2half_rn(q0 * cs - q1 * sn));
    sq[2 * i + 1] = __half2float(__float2half_rn(q0 * sn + q1 * cs));
  }
  __syncthreads();
  float ql[EPL];
#pragma unroll
  for (int e = 0; e < EPL; ++e) ql[e] = sq[lane * EPL + e];
  if (ncache > 0) wait_tiles();
  auto row = [&](const __half* base, int r, float* dst) {
    if (EPL == 4) {
      const uint2 u = *reinterpret_cast<const uint2*>(base + (size_t)r * HD + lane * 4);
      const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
      dst[0] = a.x, dst[1] = a.y, dst[2] = b.x, dst[3] = b.y;
    } else {
      const float2 a = __half22float2(*reinterpret_cast<const __half2*>(base + (size_t)r * HD + lane * 2));
      dst[0] = a.x, dst[1] = a.y;
    }
  };
  // pass 1: scores of the range
  for (int r = warp; r < ncache; r += kDW) {
    float kr[EPL];
    row(Kt, r, kr);
    float acc = 0.f;
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc = fmaf(ql[e], kr[e], acc);
    acc = warp_sum(acc);
    if (lane == 0) sc[r] = acc * scale;
  }
  if (tail_new && warp == kDW - 1) {
    float acc = 0.f;
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc = fmaf(ql[e], sk[lane * EPL + e], acc);
    acc = warp_sum(acc);
    if (lane == 0) sc[ncache] = acc * scale;
  }
  __syncthreads();
  const int nloc = ncache + (tail_new ? 1 : 0);
  float lmax = -INFINITY;
  for (int i = threadIdx.x; i < nloc; i += blockDim.x) lmax = fmaxf(lmax, sc[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
  if (lane == 0) red[warp] = lmax;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = red[0];
    for (int i = 1; i < kDW; ++i) m = fmaxf(m, red[i]);
    bcast = m;
  }
  __syncthreads();
  const float mx = bcast;
  float lsum = 0.f;
  for (int i = threadIdx.x; i < nloc; i += blockDim.x) {
    const float a = __half2float(__float2half_rn(sc[i] - mx));
    const float e = __half2float(__float2half_rn(expf(a)));  // table_exp_f16 (ne_layers.c:8933-8937)
    sc[i] = e;
    lsum += e;
  }
  lsum = warp_sum(lsum);
  __syncthreads();
  if (lane == 0) red[warp] = lsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s2 = 0.f;
    for (int i = 0; i < kDW; ++i) s2 += red[i];
    bcast = s2;
  }
  __syncthreads();
  const float lrange = bcast;
  const bool single = nact == 1;
  const float inv = 1.f / lrange;
  // pass 2: sum p V over the range; warps own rows, lanes own EPL output elements
  float acc[EPL];
#pragma unroll
  for (int e = 0; e < EPL; ++e) acc[e] = 0.f;
  for (int r = warp; r < ncache; r += kDW) {
    float vr[EPL];
    row(Vt, r, vr);
    const float p = single ? __half2float(__float2half_rn(sc[r] * inv)) : sc[r];
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc[e] = fmaf(p, vr[e], acc[e]);
  }
  if (tail_new && warp == kDW - 1) {
    const float p = single ? __half2float(__float2half_rn(sc[ncache] * inv)) : sc[ncache];
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc[e] = fmaf(p, sv[lane * EPL + e], acc[e]);
  }
#pragma unroll
  for (int e = 0; e < EPL; ++e) part[warp * HD + lane * EPL + e] = acc[e];
  __syncthreads();
  float mine = 0.f;
  if (threadIdx.x < HD) {
#pragma unroll
    for (int w = 0; w < kDW; ++w) mine += part[w * HD + threadIdx.x];
  }
  if (single) {
    if (threadIdx.x < HD) out[(size_t)h * HD + threadIdx.x] = mine;
  } else {
  // several ranges: leave {sum e V, max, sum e}; the last CTA of the head merges
  float* mypart = part_ws + ((size_t)h * nsplit + split) * (HD + 2);
  if (threadIdx.x < HD) mypart[threadIdx.x] = mine;
  if (threadIdx.x == 0) {
    mypart[HD] = mx;
    mypart[HD + 1] = lrange;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last_flag = (atomicAdd(&tickets[h], 1u) == (unsigned)(nact - 1)) ? 1 : 0;
  __syncthreads();
  if (last_flag) {
  __threadfence();
  if (threadIdx.x < HD) {
    const float* base = part_ws + (size_t)h * nsplit * (HD + 2);
    float gm = -INFINITY;
    for (int s2 = 0; s2 < nact; ++s2) gm = fmaxf(gm, __ldcg(base + (size_t)s2 * (HD + 2) + HD));
    float num = 0.f, den = 0.f;
    for (int s2 = 0; s2 < nact; ++s2) {
      const float w = expf(__ldcg(base + (size_t)s2 * (HD + 2) + HD) - gm);
      num = fmaf(w, __ldcg(base + (size_t)s2 * (HD + 2) + threadIdx.x), num);
      den = fmaf(w, __ldcg(base + (size_t)s2 * (HD + 2) + HD + 1), den);
    }
    out[(size_t)h * HD + threadIdx.x] = num / den;
  }
  if (threadIdx.x == 0) tickets[h] = 0u;  // ready for the next launch (graph replay)
  }
  }
  if (RING) __syncthreads();  // sq, sc, part and the reduction slots serve the next query head
  }
  // the bulk store reads the shifted rows out of shared memory: it must be complete before the CTA exits
  if (wrapped && threadIdx.x == 0 && shift0 < ncache) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// ---- prompt attention on the tensor cores ------------------------------------------------------------------------------------
// The ggml attention of the reference for N > 1 new tokens (llama.cpp:286-302: KQ = mul_mat(K, Q) -> scale -> diag_mask_inf ->
// soft_max -> mul_mat(V, KQ_soft_max); ne_compute_forward_mul_mat_f16_f32 rounds Q and the probabilities to fp16 and sums the
// fp16 x fp16 products in fp32, ne_layers.c:6943-7083; soft_max rounds (s - max) and exp() to fp16, :8887-8954) as a causal
// two-pass kernel on mma.sync.m16n8k16 f16 -> f32 (the same operand types and accumulator as the reference's dot products):
//   pass A  S = Q K^T tile by tile, row maxima (the reference's soft_max uses the GLOBAL row maximum, not a running one)
//   pass B  S again, e = fp16(exp(fp16(s - max))), l += e, O += e V (e is an exact fp16 value: the products are exact), out = O / l
// (difference to the reference: it rounds e / l to fp16 before the V product; here the division happens once, in fp32, after it).
// CTA = 64 query rows of one head (4 warps x 16 rows); K / V tiles of 64 keys staged in shared memory with 16-byte padded rows
// (conflict-free 32-bit B-fragment loads for K, ldmatrix.trans for V); every q-tile of a head re-reads that head's K / V through L2.
// Bound: tensor pipe / shared-memory bandwidth (K and V of one head are 0.5 MB at 2048 positions -- L2 resident).
//
// RAGGED: the query rows are segments of several sequences (ns_llama_eval_batch, llama.cpp:414-489 run per input), grid
// (tiles, n_head).  CTA x reads tiles[5 x] = {segment's first row, its length, its n_past, its KV block, the tile's first query row
// inside the segment}, offsets q / out by the first row and kc / vc by the block, and takes pos0 = n_past, m = length.  Everything
// after those offsets is the single-sequence code, so each segment is bit-identical to a launch of its own.
constexpr int kAttnMmaRows = 64, kAttnMmaKeys = 64;
constexpr int kTileInts = 5;  // ints per entry of the ragged tile table
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ void mma_f16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <int HD, bool RAGGED = false>
__global__ void __launch_bounds__(128) attn_mma_kernel(const float* __restrict__ q, int ldq, const __half* __restrict__ kc,
                                                       const __half* __restrict__ vc, const int* __restrict__ state, float* __restrict__ out,
                                                       int ldo, int n_head, int n_head_kv, int n_ctx, int m, float scale,
                                                       const int* __restrict__ tiles) {
  constexpr int LD = HD + 8;  // halves per shared-memory row: 16 bytes of padding rotate the banks by 4 words per row
  constexpr int KS = HD / 16, NT = HD / 8;
  __shared__ __align__(16) __half Ks[kAttnMmaKeys * LD];
  __shared__ __align__(16) __half Vs[kAttnMmaKeys * LD];
  pdl_launch_dependents();
  pdl_wait();
  const int h = blockIdx.y, hk = h / (n_head / n_head_kv);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;
  int pos0, q0;
  if (RAGGED) {
    const int* tl = tiles + kTileInts * blockIdx.x;
    q += (size_t)tl[0] * ldq;
    out += (size_t)tl[0] * ldo;
    const size_t blk = (size_t)tl[3] * n_head_kv * n_ctx * HD;
    kc += blk;
    vc += blk;
    m = tl[1];
    pos0 = tl[2];
    q0 = tl[4];
  } else {
    pos0 = state[1];
    q0 = blockIdx.x * kAttnMmaRows;
  }
  const int row0 = q0 + warp * 16 + g, row1 = row0 + 8;  // this thread's two query rows (token indices of the batch)
  const int total = min(pos0 + m, n_ctx);                // keys that exist
  const __half* kh = kc + (size_t)hk * n_ctx * HD;
  const __half* vh = vc + (size_t)hk * n_ctx * HD;

  // Q A-fragments, rounded to fp16 as the reference's mul_mat does with src1 (rows past the batch: zeros)
  uint32_t qa[KS][4];
  {
    const float* q0p = q + (size_t)row0 * ldq + (size_t)h * HD;
    const float* q1p = q + (size_t)row1 * ldq + (size_t)h * HD;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      const int c = ks * 16 + 2 * t4;
      const float2 a0 = row0 < m ? *reinterpret_cast<const float2*>(q0p + c) : make_float2(0.f, 0.f);
      const float2 a1 = row1 < m ? *reinterpret_cast<const float2*>(q1p + c) : make_float2(0.f, 0.f);
      const float2 a2 = row0 < m ? *reinterpret_cast<const float2*>(q0p + c + 8) : make_float2(0.f, 0.f);
      const float2 a3 = row1 < m ? *reinterpret_cast<const float2*>(q1p + c + 8) : make_float2(0.f, 0.f);
      qa[ks][0] = pack_h2(a0.x, a0.y);
      qa[ks][1] = pack_h2(a1.x, a1.y);
      qa[ks][2] = pack_h2(a2.x, a2.y);
      qa[ks][3] = pack_h2(a3.x, a3.y);
    }
  }
  const int last_row = min(q0 + kAttnMmaRows, m) - 1;
  const int nkt = min(pos0 + last_row, total - 1) / kAttnMmaKeys + 1;  // key tiles this CTA needs
  const int warp_last_key = pos0 + q0 + warp * 16 + 15;                // beyond it every key is masked for the whole warp

  auto load_tile = [&](const __half* base, __half* dst, int key0) {
    constexpr int C16 = HD / 8;  // 16-byte chunks per row
#pragma unroll
    for (int i = 0; i < kAttnMmaKeys * C16 / 128; ++i) {
      const int idx = i * 128 + (int)threadIdx.x;
      const int r = idx / C16, c = idx % C16;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (key0 + r < total) v = *reinterpret_cast<const uint4*>(base + (size_t)(key0 + r) * HD + c * 8);
      *reinterpret_cast<uint4*>(dst + r * LD + c * 8) = v;
    }
  };
  auto scores = [&](float (&s)[8][4]) {
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int c = 0; c < 4; ++c) s[j][c] = 0.f;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const __half* kr = Ks + (j * 8 + g) * LD + ks * 16 + 2 * t4;
        mma_f16_16816(s[j], qa[ks], *reinterpret_cast<const uint32_t*>(kr), *reinterpret_cast<const uint32_t*>(kr + 8));
      }
  };

  // ---- pass A: row maxima of the masked, scaled scores
  float mx0 = -INFINITY, mx1 = -INFINITY;
  for (int kt = 0; kt < nkt; ++kt) {
    __syncthreads();
    load_tile(kh, Ks, kt * kAttnMmaKeys);
    __syncthreads();
    if (kt * kAttnMmaKeys > warp_last_key) continue;
    float s[8][4];
    scores(s);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int key = kt * kAttnMmaKeys + j * 8 + 2 * t4 + (c & 1);
        const int row = (c < 2) ? row0 : row1;
        if (key <= pos0 + row && key < total) {
          if (c < 2) mx0 = fmaxf(mx0, s[j][c] * scale);
          else mx1 = fmaxf(mx1, s[j][c] * scale);
        }
      }
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  if (row0 >= m) mx0 = 0.f;  // rows past the batch: nothing valid, nothing stored
  if (row1 >= m) mx1 = 0.f;

  // ---- pass B: e = fp16(exp(fp16(s - max))), l = sum e, O = sum e V
  float o[NT][4];
#pragma unroll
  for (int n = 0; n < NT; ++n)
#pragma unroll
    for (int c = 0; c < 4; ++c) o[n][c] = 0.f;
  float l0 = 0.f, l1 = 0.f;
  for (int kt = 0; kt < nkt; ++kt) {
    __syncthreads();
    load_tile(kh, Ks, kt * kAttnMmaKeys);
    load_tile(vh, Vs, kt * kAttnMmaKeys);
    __syncthreads();
    if (kt * kAttnMmaKeys > warp_last_key) continue;
    float s[8][4];
    scores(s);
    uint32_t pe[8][2];  // per 8-key tile: (row0: keys 2t4, 2t4+1), (row1: same keys) as fp16 pairs
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float e[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int key = kt * kAttnMmaKeys + j * 8 + 2 * t4 + (c & 1);
        const int row = (c < 2) ? row0 : row1;
        const bool valid = key <= pos0 + row && key < total && row < m;
        const float a = __half2float(__float2half_rn(s[j][c] * scale - (c < 2 ? mx0 : mx1)));
        e[c] = valid ? __half2float(__float2half_rn(expf(a))) : 0.f;  // table_exp_f16 (ne_layers.c:8933-8937)
      }
      l0 += e[0] + e[1];
      l1 += e[2] + e[3];
      pe[j][0] = pack_h2(e[0], e[1]);
      pe[j][1] = pack_h2(e[2], e[3]);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {  // 16 keys per step: P as the A operand straight from the score accumulators
      const uint32_t pa[4] = {pe[2 * kk][0], pe[2 * kk][1], pe[2 * kk + 1][0], pe[2 * kk + 1][1]};
      const __half* vrow = Vs + (kk * 16 + (lane & 7) + 8 * ((lane >> 3) & 1)) * LD + 8 * (lane >> 4);
#pragma unroll
      for (int n2 = 0; n2 < NT / 2; ++n2) {
        uint32_t b0, b1, b2, b3;
        const uint32_t addr = (uint32_t)__cvta_generic_to_shared(vrow + n2 * 16);
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(b0), "=r"(b1), "=r"(b2), "=r"(b3) : "r"(addr));
        mma_f16_16816(o[2 * n2], pa, b0, b1);
        mma_f16_16816(o[2 * n2 + 1], pa, b2, b3);
      }
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
  for (int n = 0; n < NT; ++n) {
    const int d = n * 8 + 2 * t4;
    if (row0 < m) *reinterpret_cast<float2*>(out + (size_t)row0 * ldo + (size_t)h * HD + d) = make_float2(o[n][0] * i0, o[n][1] * i0);
    if (row1 < m) *reinterpret_cast<float2*>(out + (size_t)row1 * ldo + (size_t)h * HD + d) = make_float2(o[n][2] * i1, o[n][3] * i1);
  }
}

// greedy pick: index of the maximum, lowest index on ties (model_utils.cpp:2963-2985); also advances the device-side
// position.  kArgmaxBlocks CTAs scan slices (all loads in flight at once); the last CTA to finish (ticket) merges the
// partial results.  state[3] = pick; when `advance`: state[0] = pick, state[1] += n_tokens, record[state[2]++] = pick.
// BATCH: grid row y (one per sequence) does the same for logits row y with state + 4 y, record + y * rec_stride, its own partial
// slots and its own ticket (the single-sequence instantiation keeps row 0 at compile time).
constexpr int kArgmaxBlocks = 32;
__device__ __forceinline__ void argmax_merge(float& best, int& bi, float ov, int oi) {
  if (ov > best || (ov == best && oi < bi)) {
    best = ov;
    bi = oi;
  }
}
template <bool BATCH>
__global__ void __launch_bounds__(256) argmax_kernel(const float* __restrict__ logits, int n, int* __restrict__ state, int n_tokens,
                                                     int advance, int* __restrict__ record, int rec_stride, float* __restrict__ pval,
                                                     int* __restrict__ pidx, unsigned* __restrict__ ticket) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = BATCH ? (int)blockIdx.y : 0;
  logits += (size_t)row * n;
  state += 4 * row;
  if (record) record += (size_t)row * rec_stride;
  pval += row * kArgmaxBlocks;
  pidx += row * kArgmaxBlocks;
  ticket += row;
  const int per = (n + kArgmaxBlocks - 1) / kArgmaxBlocks;
  const int lo = blockIdx.x * per, hi = min(n, lo + per);
  float best = -INFINITY;
  int bi = 0x7fffffff;
  constexpr int U = 4;
  for (int i0 = lo + threadIdx.x; i0 < hi; i0 += 256 * U) {
    float v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = (i0 + u * 256 < hi) ? logits[i0 + u * 256] : -INFINITY;
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (i0 + u * 256 < hi) argmax_merge(best, bi, v[u], i0 + u * 256);
  }
  __shared__ float sv[8];
  __shared__ int si[8];
  __shared__ bool last;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) argmax_merge(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
  if ((threadIdx.x & 31) == 0) {
    sv[threadIdx.x >> 5] = best;
    si[threadIdx.x >> 5] = bi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) argmax_merge(best, bi, sv[w], si[w]);
    pval[blockIdx.x] = best;
    pidx[blockIdx.x] = bi;
    __threadfence();
    last = atomicAdd(ticket, 1u) == kArgmaxBlocks - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  best = -INFINITY;
  bi = 0x7fffffff;
  for (int b2 = 0; b2 < kArgmaxBlocks; ++b2) argmax_merge(best, bi, ((volatile float*)pval)[b2], ((volatile int*)pidx)[b2]);
  if (bi == 0x7fffffff) bi = 0;  // all NaN / -inf: the reference's loop keeps index 0
  *ticket = 0u;                  // ready for the next launch
  state[3] = bi;
  if (advance) {
    state[0] = bi;
    state[1] += n_tokens;
    if (record) record[state[2]++] = bi;
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

// ---- one layer's attention: RoPE of q and of the m new k rows at positions state[1] + t, fp16 KV append, causal attention ------
// q [m][n_head * hd] (rotated in place unless a fused kernel rotates it in registers), k / v [m][n_head_kv * hd], cache
// [n_head_kv][n_ctx][hd] fp16, out [m][n_head * hd].  NS_ATTN_AUTO picks what the eval step has always run:
//   hd 64 / 128, one row    attn_decode_kernel (context split over 256-position ranges) while the context has <= 1024 ranges
//                           and NS_ATTN_OLD_DECODE is unset, else attn_fast_kernel<FUSE>
//   hd 64 / 128, >= 8 rows  rope_kv_kernel + attn_mma_kernel unless NS_ATTN_SCALAR is set
//   hd 64 / 128, otherwise  rope_kv_kernel + attn_fast_kernel
//   any other (even) hd     rope_kv_kernel + attn_kernel
struct AttnAttr {  // dynamic shared memory already granted to each kernel (function attributes are per device)
  size_t generic = 0, rows = 0;
  bool decode = false;
};

static size_t attn_generic_smem(int hd, int n_ctx) { return (size_t)(hd + n_ctx) * sizeof(float); }
static size_t attn_rows_smem(int hd, int n_ctx) { return (size_t)((3 + kAW) * hd + n_ctx) * sizeof(float); }
static int attn_ranges(int n_ctx) { return (n_ctx + kSplitKeys - 1) / kSplitKeys; }

// the kernel `kind` resolves to for this shape, or NS_E_UNSUPPORTED when a forced kernel cannot take it
static int attn_resolve(int kind, int hd, int m, int n_ctx) {
  const bool fast = hd == 128 || hd == 64;
  if (kind == NS_ATTN_AUTO) {
    // debugging aids, read per call (not per process) so that a test can compare kernels on one engine
    const bool old_decode = getenv("NS_ATTN_OLD_DECODE") != nullptr;  // decode attention: one CTA per head, dependent row loads
    const bool scalar_attn = getenv("NS_ATTN_SCALAR") != nullptr;    // prompt attention: one CTA per (head, token), no tensor cores
    if (!fast) kind = NS_ATTN_GENERIC;
    else if (m == 1) kind = attn_ranges(n_ctx) <= 1024 && !old_decode ? NS_ATTN_SPLIT_DECODE : NS_ATTN_ROWS;
    else kind = m >= 8 && !scalar_attn ? NS_ATTN_MMA : NS_ATTN_ROWS;
  }
  if (kind < NS_ATTN_SPLIT_DECODE || kind > NS_ATTN_GENERIC) {
    ns_set_error("ns_llama: unknown attention kernel %d", kind);
    return NS_E_INVALID;
  }
  if (kind != NS_ATTN_GENERIC && !fast) {
    ns_set_error("ns_llama: attention kernel %d needs head size 64 or 128, got %d", kind, hd);
    return NS_E_UNSUPPORTED;
  }
  if (kind == NS_ATTN_SPLIT_DECODE && m != 1) {
    ns_set_error("ns_llama: the split-context decode attention takes one row, got %d", m);
    return NS_E_UNSUPPORTED;
  }
  const size_t smem = kind == NS_ATTN_GENERIC ? attn_generic_smem(hd, n_ctx) : kind == NS_ATTN_ROWS ? attn_rows_smem(hd, n_ctx) : 0;
  if (smem > 220 * 1024) {
    ns_set_error("ns_llama: n_ctx %d too large for the single-pass attention kernel", n_ctx);
    return NS_E_UNSUPPORTED;
  }
  return kind;
}

// The fp16 table that shifts a cached key one position back (model_utils.cpp:165-192 with freq_scale 1): theta starts at -1 and
// is multiplied by freq_base^(-2 / hd) per pair in fp32; cos and sin come from the host libm, as in the reference.
static ShiftTable shift_table(int hd, float freq_base) {
  ShiftTable t{};
  const float theta_scale = std::pow(freq_base, -2.0f / hd);
  float theta = -1.0f;
  for (int i = 0; i < hd / 2; ++i) {
    t.cs[i] = __halves2half2(__float2half_rn(std::cos(theta)), __float2half_rn(std::sin(theta)));
    theta *= theta_scale;
  }
  return t;
}

// part: [n_head][attn_ranges(n_ctx)][hd + 2] floats, tickets: [n_head] zero words (both read by attn_decode_kernel only; the
// last CTA of a head leaves its ticket at zero again).  ring (nullable): one-token steps run the ring variant of the split decode
// attention with ring->n_keep sink slots; prompts (m > 1, which never reach past n_ctx) run the plain kernels.
struct Ring {
  int n_keep;
  ShiftTable tab;
};
static int grant_decode_smem(AttnAttr& attr) {
  if (attr.decode) return NS_OK;
  NS_CUDA_TRY(cudaFuncSetAttribute(attn_decode_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_decode_smem<128>()));
  NS_CUDA_TRY(cudaFuncSetAttribute(attn_decode_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_decode_smem<64>()));
  NS_CUDA_TRY(cudaFuncSetAttribute(attn_decode_kernel<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_decode_smem<128>()));
  NS_CUDA_TRY(cudaFuncSetAttribute(attn_decode_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_decode_smem<64>()));
  NS_CUDA_TRY(cudaFuncSetAttribute(attn_decode_kernel<128, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)attn_decode_smem<128>()));
  NS_CUDA_TRY(cudaFuncSetAttribute(attn_decode_kernel<64, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)attn_decode_smem<64>()));
  attr.decode = true;
  return NS_OK;
}

// Batched decode attention: one new token for each of n sequences, one launch (attn_decode_kernel<HD, false, true>).  rstate:
// [n][4] row states (n_past in slot 1), seqs [n] KV block per row, caches [n_seq][n_head_kv][n_ctx][hd] fp16, q / out
// [n][n_head * hd], k / v [n][n_head_kv * hd], part [n][n_head][ranges][hd + 2], tickets [n][n_head].  hd 64 / 128 only.
static int launch_attention_batch(const float* q, const float* k, const float* v, __half* kc, __half* vc, const int* rstate,
                                  const int* seqs, float* out, float* part, unsigned* tickets, int n, int n_head, int n_head_kv, int hd,
                                  int n_ctx, float rope_theta, float rope_scale, AttnAttr& attr, cudaStream_t st) {
  if (hd != 64 && hd != 128) {
    ns_set_error("ns_llama: the batched decode attention needs head size 64 or 128, got %d", hd);
    return NS_E_UNSUPPORTED;
  }
  if (int rc = grant_decode_smem(attr)) return rc;
  const float theta_scale = powf(rope_theta, -2.0f / (float)hd);  // as launch_attention
  const float freq_scale = 1.f / rope_scale;
  const float attn_scale = 1.0f / sqrtf((float)hd);
  const int nsplit = attn_ranges(n_ctx);
  auto kern = hd == 128 ? attn_decode_kernel<128, false, true> : attn_decode_kernel<64, false, true>;
  NS_CUDA_TRY(ns_launch_pdl(kern, dim3((unsigned)n_head, (unsigned)nsplit, (unsigned)n), dim3(kDW * 32),
                            hd == 128 ? attn_decode_smem<128>() : attn_decode_smem<64>(), st, q, k,
                            v, kc, vc, rstate, out, part, tickets, n_head, n_head_kv, n_ctx, nsplit, attn_scale, theta_scale, freq_scale,
                            -1, ShiftTable{}, seqs));
  ns_count_launch();
  return NS_OK;
}

static int launch_attention(int kind, float* q, const float* k, const float* v, __half* kc, __half* vc, const int* state, float* out,
                            float* part, unsigned* tickets, int n_head, int n_head_kv, int hd, int n_ctx, int m, float rope_theta,
                            float rope_scale, AttnAttr& attr, cudaStream_t st, const Ring* ring = nullptr) {
  if (ring && m == 1) kind = NS_ATTN_SPLIT_DECODE;  // the only kernel that carries the shift
  kind = attn_resolve(kind, hd, m, n_ctx);
  if (kind < 0) return kind;
  const int ldq = n_head * hd, ldk = n_head_kv * hd;
  const float theta_scale = powf(rope_theta, -2.0f / (float)hd);  // n_rot == head_size (llama.cpp:131)
  const float freq_scale = 1.f / rope_scale;  // the angle is divided by hparams.freq_scale (ne_layers.c:9263, 9207)
  const float attn_scale = 1.0f / sqrtf((float)hd);
  const size_t rows_smem = attn_rows_smem(hd, n_ctx);
  if (kind == NS_ATTN_ROWS && rows_smem > 48 * 1024 && rows_smem > attr.rows) {
    NS_CUDA_TRY(cudaFuncSetAttribute(attn_fast_kernel<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rows_smem));
    NS_CUDA_TRY(cudaFuncSetAttribute(attn_fast_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rows_smem));
    NS_CUDA_TRY(cudaFuncSetAttribute(attn_fast_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rows_smem));
    NS_CUDA_TRY(cudaFuncSetAttribute(attn_fast_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rows_smem));
    attr.rows = rows_smem;
  }
  if (kind == NS_ATTN_SPLIT_DECODE) {
    // rope + KV append + attention in one launch, K / V staged by TMA, the context split over CTAs
    if (int rc = grant_decode_smem(attr)) return rc;
    const int nsplit = attn_ranges(n_ctx);
    const size_t dsm = hd == 128 ? attn_decode_smem<128>() : attn_decode_smem<64>();
    auto kern = ring ? (hd == 128 ? attn_decode_kernel<128, true> : attn_decode_kernel<64, true>)
                     : (hd == 128 ? attn_decode_kernel<128, false> : attn_decode_kernel<64, false>);
    const unsigned gx = (unsigned)(ring ? n_head_kv : n_head);  // ring: one CTA per (kv head, range)
    NS_CUDA_TRY(ns_launch_pdl(kern, dim3(gx, (unsigned)nsplit), dim3(kDW * 32), dsm, st, (const float*)q, k, v, kc, vc, state, out, part,
                              tickets, n_head, n_head_kv, n_ctx, nsplit, attn_scale, theta_scale, freq_scale, ring ? ring->n_keep : -1,
                              ring ? ring->tab : ShiftTable{}, (const int*)nullptr));
    ns_count_launch();
    return NS_OK;
  }
  if (kind == NS_ATTN_ROWS && m == 1) {  // the same fused launch with dependent row loads (one CTA per head)
    auto kern = hd == 128 ? attn_fast_kernel<128, true> : attn_fast_kernel<64, true>;
    NS_CUDA_TRY(ns_launch_pdl(kern, dim3((unsigned)n_head, 1u), dim3(kAW * 32), rows_smem, st, (const float*)q, ldq, k, ldk, v, ldk, kc, vc,
                              state, out, ldq, n_head, n_head_kv, n_ctx, attn_scale, theta_scale, freq_scale));
    ns_count_launch();
    return NS_OK;
  }
  NS_CUDA_TRY(ns_launch_pdl(rope_kv_kernel<false>, dim3((unsigned)(n_head + n_head_kv), (unsigned)m), dim3((unsigned)(hd / 2)), 0, st, q,
                            ldq, k, ldk, v, ldk, kc, vc, state, n_head, n_head_kv, hd, n_ctx, theta_scale, freq_scale, (const int*)nullptr));
  ns_count_launch();
  if (kind == NS_ATTN_MMA) {  // causal attention on the tensor cores, 64 query rows per CTA
    auto kern = hd == 128 ? attn_mma_kernel<128> : attn_mma_kernel<64>;
    NS_CUDA_TRY(ns_launch_pdl(kern, dim3((unsigned)((m + kAttnMmaRows - 1) / kAttnMmaRows), (unsigned)n_head), dim3(128), 0, st,
                              (const float*)q, ldq, (const __half*)kc, (const __half*)vc, state, out, ldq, n_head, n_head_kv, n_ctx, m,
                              attn_scale, (const int*)nullptr));
  } else if (kind == NS_ATTN_ROWS) {
    auto kern = hd == 128 ? attn_fast_kernel<128, false> : attn_fast_kernel<64, false>;
    NS_CUDA_TRY(ns_launch_pdl(kern, dim3((unsigned)n_head, (unsigned)m), dim3(kAW * 32), rows_smem, st, (const float*)q, ldq, k, ldk, v, ldk,
                              kc, vc, state, out, ldq, n_head, n_head_kv, n_ctx, attn_scale, theta_scale, freq_scale));
  } else {
    const size_t smem = attn_generic_smem(hd, n_ctx);
    if (smem > 48 * 1024 && smem > attr.generic) {
      NS_CUDA_TRY(cudaFuncSetAttribute(attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      attr.generic = smem;
    }
    NS_CUDA_TRY(ns_launch_pdl(attn_kernel, dim3((unsigned)n_head, (unsigned)m), dim3(kAttnThreads), smem, st, (const float*)q, ldq,
                              (const __half*)kc, (const __half*)vc, state, out, ldq, n_head, n_head_kv, hd, n_ctx, attn_scale));
  }
  ns_count_launch();
  return NS_OK;
}

// Workspace of ns_llama_attention: int state[4] (state[1] = n_past) | unsigned tickets[n_head], padded to 16 bytes |
// float partials[n_head][ceil(n_ctx / 256)][hd + 2]
static size_t attn_ws_tickets_offset() { return 4 * sizeof(int); }
static size_t attn_ws_part_offset(int n_head) { return attn_ws_tickets_offset() + ((size_t)n_head * sizeof(unsigned) + 15) / 16 * 16; }

extern "C" size_t ns_llama_attention_workspace_bytes(int n_head, int hd, int n_ctx) {
  if (n_head <= 0 || hd <= 0 || n_ctx <= 0) return 0;
  return attn_ws_part_offset(n_head) + (size_t)n_head * attn_ranges(n_ctx) * (hd + 2) * sizeof(float);
}

extern "C" int ns_llama_attention(int kernel, float* q, const float* k, const float* v, void* kc, void* vc, int n_head, int n_head_kv,
                                  int hd, int n_ctx, int n_past, int m, float rope_theta, float rope_scale, float* out, void* ws,
                                  void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!q || !k || !v || !kc || !vc || !out || !ws || n_head <= 0 || n_head_kv <= 0 || n_head % n_head_kv || hd <= 0 || hd % 2 ||
      n_ctx <= 0 || m <= 0 || n_past < 0 || n_past + m > n_ctx || !(rope_theta > 0.f) || !(rope_scale > 0.f)) {
    ns_set_error("ns_llama_attention: invalid arguments (n_head=%d n_head_kv=%d hd=%d n_ctx=%d n_past=%d m=%d)", n_head, n_head_kv, hd,
                 n_ctx, n_past, m);
    return NS_E_INVALID;
  }
  if (int rc = attn_resolve(kernel, hd, m, n_ctx); rc < 0) return rc;
  cudaStream_t st = ns_stream_of(queue);
  char* w = static_cast<char*>(ws);
  const int state[4] = {0, n_past, 0, 0};
  NS_CUDA_TRY(cudaMemcpyAsync(w, state, sizeof(state), cudaMemcpyHostToDevice, st));  // pageable source: staged before the call returns
  AttnAttr attr;
  return launch_attention(kernel, q, k, v, static_cast<__half*>(kc), static_cast<__half*>(vc), reinterpret_cast<const int*>(w), out,
                          reinterpret_cast<float*>(w + attn_ws_part_offset(n_head)),
                          reinterpret_cast<unsigned*>(w + attn_ws_tickets_offset()), n_head, n_head_kv, hd, n_ctx, m, rope_theta,
                          rope_scale, attr, st);
}

extern "C" int ns_llama_attention_ring(float* q, const float* k, const float* v, void* kc, void* vc, int n_head, int n_head_kv, int hd,
                                       int n_ctx, int n_keep, int n_total, float rope_theta, float* out, void* ws, void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!q || !k || !v || !kc || !vc || !out || !ws || n_head <= 0 || n_head_kv <= 0 || n_head % n_head_kv || hd <= 0 || hd % 2 ||
      n_ctx <= 0 || n_keep < 0 || n_keep >= n_ctx || n_total < 0 || !(rope_theta > 0.f)) {
    ns_set_error("ns_llama_attention_ring: invalid arguments (n_head=%d n_head_kv=%d hd=%d n_ctx=%d n_keep=%d n_total=%d)", n_head,
                 n_head_kv, hd, n_ctx, n_keep, n_total);
    return NS_E_INVALID;
  }
  if (int rc = attn_resolve(NS_ATTN_SPLIT_DECODE, hd, 1, n_ctx); rc < 0) return rc;
  cudaStream_t st = ns_stream_of(queue);
  char* w = static_cast<char*>(ws);
  const int state[4] = {0, n_total, 0, 0};
  NS_CUDA_TRY(cudaMemcpyAsync(w, state, sizeof(state), cudaMemcpyHostToDevice, st));  // pageable source: staged before the call returns
  AttnAttr attr;
  const Ring ring{n_keep, shift_table(hd, rope_theta)};
  return launch_attention(NS_ATTN_SPLIT_DECODE, q, k, v, static_cast<__half*>(kc), static_cast<__half*>(vc), reinterpret_cast<const int*>(w),
                          out, reinterpret_cast<float*>(w + attn_ws_part_offset(n_head)),
                          reinterpret_cast<unsigned*>(w + attn_ws_tickets_offset()), n_head, n_head_kv, hd, n_ctx, 1, rope_theta, 1.f, attr,
                          st, &ring);
}

// Checks the rows of a batched call: 1 <= n <= n_seq, every id in [0, n_seq) and distinct, 0 <= n_past[i], n_past[i] + steps <= n_ctx
static int check_rows(const char* who, int n_seq, int n, const int* seq, const int* n_past, int steps, int n_ctx) {
  if (n < 1 || n > n_seq) {
    ns_set_error("%s: n %d outside [1, n_seq %d]", who, n, n_seq);
    return NS_E_INVALID;
  }
  unsigned long long seen = 0;  // n_seq <= 32
  for (int i = 0; i < n; ++i) {
    if (seq[i] < 0 || seq[i] >= n_seq) {
      ns_set_error("%s: sequence id %d outside [0, %d)", who, seq[i], n_seq);
      return NS_E_INVALID;
    }
    if (seen >> seq[i] & 1ull) {
      ns_set_error("%s: sequence id %d appears twice", who, seq[i]);
      return NS_E_INVALID;
    }
    seen |= 1ull << seq[i];
    if (n_past[i] < 0 || n_past[i] + steps > n_ctx) {
      ns_set_error("%s: sequence %d: n_past %d + %d steps outside n_ctx %d", who, seq[i], n_past[i], steps, n_ctx);
      return NS_E_INVALID;
    }
  }
  return NS_OK;
}

// Workspace of ns_llama_attention_batch: int rows[n][4] (slot 1 = n_past) | int seq[n], padded to 16 bytes | unsigned
// tickets[n][n_head], padded to 16 bytes | float partials[n][n_head][ceil(n_ctx / 256)][hd + 2]
static size_t attnb_ws_seq_offset(int n) { return (size_t)n * 4 * sizeof(int); }
static size_t attnb_ws_tickets_offset(int n) { return attnb_ws_seq_offset(n) + ((size_t)n * sizeof(int) + 15) / 16 * 16; }
static size_t attnb_ws_part_offset(int n, int n_head) {
  return attnb_ws_tickets_offset(n) + ((size_t)n * n_head * sizeof(unsigned) + 15) / 16 * 16;
}

extern "C" size_t ns_llama_attention_batch_workspace_bytes(int n, int n_head, int hd, int n_ctx) {
  if (n <= 0 || n_head <= 0 || hd <= 0 || n_ctx <= 0) return 0;
  return attnb_ws_part_offset(n, n_head) + (size_t)n * n_head * attn_ranges(n_ctx) * (hd + 2) * sizeof(float);
}

extern "C" int ns_llama_attention_batch(float* q, const float* k, const float* v, void* kc, void* vc, int n_seq, int n, const int* seq,
                                        const int* n_past, int n_head, int n_head_kv, int hd, int n_ctx, float rope_theta,
                                        float rope_scale, float* out, void* ws, void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!q || !k || !v || !kc || !vc || !seq || !n_past || !out || !ws || n_seq < 1 || n_seq > 32 || n_head <= 0 || n_head_kv <= 0 ||
      n_head % n_head_kv || hd <= 0 || hd % 2 || n_ctx <= 0 || !(rope_theta > 0.f) || !(rope_scale > 0.f)) {
    ns_set_error("ns_llama_attention_batch: invalid arguments (n_seq=%d n=%d n_head=%d n_head_kv=%d hd=%d n_ctx=%d)", n_seq, n, n_head,
                 n_head_kv, hd, n_ctx);
    return NS_E_INVALID;
  }
  if (int rc = check_rows("ns_llama_attention_batch", n_seq, n, seq, n_past, 1, n_ctx)) return rc;
  if (hd != 64 && hd != 128) {
    ns_set_error("ns_llama_attention_batch: head size %d (the batched decode attention takes 64 or 128)", hd);
    return NS_E_UNSUPPORTED;
  }
  cudaStream_t st = ns_stream_of(queue);
  char* w = static_cast<char*>(ws);
  std::vector<int> rows((size_t)n * 5, 0);
  for (int i = 0; i < n; ++i) {
    rows[(size_t)4 * i + 1] = n_past[i];
    rows[(size_t)4 * n + i] = seq[i];
  }
  NS_CUDA_TRY(cudaMemcpyAsync(w, rows.data(), rows.size() * sizeof(int), cudaMemcpyHostToDevice, st));  // pageable: staged now
  AttnAttr attr;
  return launch_attention_batch(q, k, v, static_cast<__half*>(kc), static_cast<__half*>(vc), reinterpret_cast<const int*>(w),
                                reinterpret_cast<const int*>(w + attnb_ws_seq_offset(n)), out,
                                reinterpret_cast<float*>(w + attnb_ws_part_offset(n, n_head)),
                                reinterpret_cast<unsigned*>(w + attnb_ws_tickets_offset(n)), n, n_head, n_head_kv, hd, n_ctx, rope_theta,
                                rope_scale, attr, st);
}

// ---- mixed batches: token segments of several sequences in one pass (ns_llama_eval_batch) ------------------------------------
constexpr int kMaxBatchRows = 4096;  // rows of one pass over segments; the caller chunks longer prompts

// Checks the segments of a ragged call: the ids and n_past as check_rows, then 1 <= n_tokens[i], n_past[i] + n_tokens[i] <= n_ctx
// and at most kMaxBatchRows rows in all.  *total = the number of rows.
static int check_segments(const char* who, int n_seq, int n_ctx, int n, const int* seq, const int* n_tokens, const int* n_past, int* total) {
  if (!seq || !n_tokens || !n_past) {
    ns_set_error("%s: null pointer", who);
    return NS_E_INVALID;
  }
  if (int rc = check_rows(who, n_seq, n, seq, n_past, 1, n_ctx)) return rc;
  long long rows = 0;
  for (int i = 0; i < n; ++i) {
    if (n_tokens[i] < 1) {
      ns_set_error("%s: segment %d: n_tokens %d < 1", who, i, n_tokens[i]);
      return NS_E_INVALID;
    }
    if (n_tokens[i] > n_ctx - n_past[i]) {
      ns_set_error("%s: sequence %d: n_past %d + %d tokens outside n_ctx %d", who, seq[i], n_past[i], n_tokens[i], n_ctx);
      return NS_E_INVALID;
    }
    rows += n_tokens[i];
  }
  if (rows > kMaxBatchRows) {
    ns_set_error("%s: %lld rows in one pass, at most %d (chunk longer prompts)", who, rows, kMaxBatchRows);
    return NS_E_INVALID;
  }
  *total = (int)rows;
  return NS_OK;
}

// Row layout of segments order[0 .. n) placed back to back: first[j] = first row of segment order[j], rows[2 r] / rows[2 r + 1] =
// position / KV block of row r; the segments from j0 on also get one tile entry per 64 query rows {first row counted from the
// first row of segment order[j0], length, n_past, block, the tile's first query row inside the segment} (attn_mma_kernel<RAGGED>).
static void lay_out_segments(const std::vector<int>& order, int j0, const int* seq, const int* n_tokens, const int* n_past,
                             std::vector<int>& first, std::vector<int>& rows, std::vector<int>& tiles) {
  first.assign(order.size(), 0);
  rows.clear();
  tiles.clear();
  int r = 0, r0 = 0;
  for (size_t j = 0; j < order.size(); ++j) {
    const int i = order[j];
    if ((int)j == j0) r0 = r;
    first[j] = r;
    for (int t = 0; t < n_tokens[i]; ++t) rows.insert(rows.end(), {n_past[i] + t, seq[i]});
    if ((int)j >= j0)
      for (int q0 = 0; q0 < n_tokens[i]; q0 += kAttnMmaRows) tiles.insert(tiles.end(), {r - r0, n_tokens[i], n_past[i], seq[i], q0});
    r += n_tokens[i];
  }
}

// The plan of ns_llama_eval_batch: internal order = the one-token segments, then the longer ones, each group in the caller's order.
// Rows 0 .. d - 1 take the batched decode attention, rows d .. T - 1 the ragged prompt attention (tile rows counted from row d).
struct BatchPlan {
  int T = 0, d = 0;
  std::vector<int> order, first, rows, tiles;
};

static int plan_batch(const char* who, int n_seq, int n_ctx, int n, const int* seq, const int* n_tokens, const int* n_past, BatchPlan& p) {
  if (int rc = check_segments(who, n_seq, n_ctx, n, seq, n_tokens, n_past, &p.T)) return rc;
  p.order.clear();
  for (int i = 0; i < n; ++i)
    if (n_tokens[i] == 1) p.order.push_back(i);
  p.d = (int)p.order.size();
  for (int i = 0; i < n; ++i)
    if (n_tokens[i] > 1) p.order.push_back(i);
  lay_out_segments(p.order, p.d, seq, n_tokens, n_past, p.first, p.rows, p.tiles);
  return NS_OK;
}

extern "C" int ns_llama_batch_plan(int n_seq, int n_ctx, int n, const int* seq, const int* n_tokens, const int* n_past, int* order,
                                   int* rows, int* tiles, int* counts) {
  if (!order || !rows || !tiles || !counts) {
    ns_set_error("ns_llama_batch_plan: null pointer");
    return NS_E_INVALID;
  }
  if (n_seq < 1 || n_seq > 32 || n_ctx <= 0) {
    ns_set_error("ns_llama_batch_plan: invalid arguments (n_seq=%d n_ctx=%d)", n_seq, n_ctx);
    return NS_E_INVALID;
  }
  BatchPlan p;
  if (int rc = plan_batch("ns_llama_batch_plan", n_seq, n_ctx, n, seq, n_tokens, n_past, p)) return rc;
  std::copy(p.order.begin(), p.order.end(), order);
  std::copy(p.rows.begin(), p.rows.end(), rows);
  std::copy(p.tiles.begin(), p.tiles.end(), tiles);
  counts[0] = p.T;
  counts[1] = p.d;
  counts[2] = (int)p.tiles.size() / kTileInts;
  return NS_OK;
}

// Ragged prompt attention: RoPE + KV append of n_rows rows (rows [n_rows][2] = {position, block}), then attn_mma_kernel<RAGGED> over
// n_tiles tile entries.  q / out [n_rows][n_head * hd], k / v [n_rows][n_head_kv * hd], caches [n_seq][n_head_kv][n_ctx][hd] fp16.
static int launch_attention_ragged(float* q, const float* k, const float* v, __half* kc, __half* vc, const int* rows, const int* tiles,
                                   int n_rows, int n_tiles, float* out, int n_head, int n_head_kv, int hd, int n_ctx, float rope_theta,
                                   float rope_scale, cudaStream_t st) {
  if (hd != 64 && hd != 128) {
    ns_set_error("ns_llama: the ragged prompt attention needs head size 64 or 128, got %d", hd);
    return NS_E_UNSUPPORTED;
  }
  const int ldq = n_head * hd, ldk = n_head_kv * hd;
  const float theta_scale = powf(rope_theta, -2.0f / (float)hd);  // as launch_attention
  const float freq_scale = 1.f / rope_scale;
  const float attn_scale = 1.0f / sqrtf((float)hd);
  NS_CUDA_TRY(ns_launch_pdl(rope_kv_kernel<true>, dim3((unsigned)(n_head + n_head_kv), (unsigned)n_rows), dim3((unsigned)(hd / 2)), 0, st,
                            q, ldq, k, ldk, v, ldk, kc, vc, (const int*)nullptr, n_head, n_head_kv, hd, n_ctx, theta_scale, freq_scale,
                            rows));
  ns_count_launch();
  auto kern = hd == 128 ? attn_mma_kernel<128, true> : attn_mma_kernel<64, true>;
  NS_CUDA_TRY(ns_launch_pdl(kern, dim3((unsigned)n_tiles, (unsigned)n_head), dim3(128), 0, st, (const float*)q, ldq, (const __half*)kc,
                            (const __half*)vc, (const int*)nullptr, out, ldq, n_head, n_head_kv, n_ctx, 0, attn_scale, tiles));
  ns_count_launch();
  return NS_OK;
}

// Workspace of ns_llama_attention_ragged: int rows[n_rows][2] | int tiles[n_rows / 64 + n][5]
extern "C" size_t ns_llama_attention_ragged_workspace_bytes(int n, int n_rows) {
  if (n <= 0 || n_rows <= 0) return 0;
  return ((size_t)2 * n_rows + (size_t)(n_rows / kAttnMmaRows + n) * kTileInts) * sizeof(int);
}

extern "C" int ns_llama_attention_ragged(float* q, const float* k, const float* v, void* kc, void* vc, int n_seq, int n, const int* seq,
                                         const int* n_tokens, const int* n_past, int n_head, int n_head_kv, int hd, int n_ctx,
                                         float rope_theta, float rope_scale, float* out, void* ws, void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!q || !k || !v || !kc || !vc || !out || !ws || n_seq < 1 || n_seq > 32 || n_head <= 0 || n_head_kv <= 0 || n_head % n_head_kv ||
      hd <= 0 || hd % 2 || n_ctx <= 0 || !(rope_theta > 0.f) || !(rope_scale > 0.f)) {
    ns_set_error("ns_llama_attention_ragged: invalid arguments (n_seq=%d n=%d n_head=%d n_head_kv=%d hd=%d n_ctx=%d)", n_seq, n, n_head,
                 n_head_kv, hd, n_ctx);
    return NS_E_INVALID;
  }
  int n_rows = 0;
  if (int rc = check_segments("ns_llama_attention_ragged", n_seq, n_ctx, n, seq, n_tokens, n_past, &n_rows)) return rc;
  if (hd != 64 && hd != 128) {
    ns_set_error("ns_llama_attention_ragged: head size %d (the ragged prompt attention takes 64 or 128)", hd);
    return NS_E_UNSUPPORTED;
  }
  std::vector<int> order(n), first, rows, tiles;
  for (int i = 0; i < n; ++i) order[i] = i;
  lay_out_segments(order, 0, seq, n_tokens, n_past, first, rows, tiles);
  cudaStream_t st = ns_stream_of(queue);
  char* w = static_cast<char*>(ws);
  // pageable sources: staged before the calls return
  NS_CUDA_TRY(cudaMemcpyAsync(w, rows.data(), rows.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  NS_CUDA_TRY(cudaMemcpyAsync(w + (size_t)2 * n_rows * sizeof(int), tiles.data(), tiles.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  return launch_attention_ragged(q, k, v, static_cast<__half*>(kc), static_cast<__half*>(vc), reinterpret_cast<const int*>(w),
                                 reinterpret_cast<const int*>(w + (size_t)2 * n_rows * sizeof(int)), n_rows, (int)tiles.size() / kTileInts,
                                 out, n_head, n_head_kv, hd, n_ctx, rope_theta, rope_scale, st);
}

constexpr int kMaxSeq = 32;  // KV blocks of one context (ns_llama_set_sequences)
constexpr int kPlanTiles = kMaxBatchRows / kAttnMmaRows + kMaxSeq;  // tile entries of one mixed pass, at most
// device tables of a mixed pass: rows [kMaxBatchRows][2] | tiles [kPlanTiles][kTileInts] | last row of each segment [kMaxSeq] |
// KV block of each segment [kMaxSeq] | internal segment of each caller index [kMaxSeq] (the sampler's window slots and draw order)
constexpr int kPlanInts = 2 * kMaxBatchRows + kPlanTiles * kTileInts + 3 * kMaxSeq;
constexpr int kAllChunk = kLogprobMaxRows;  // rows of one lm_head launch of ns_llama_eval_all

struct ns_llama {
  ns_llama_hparams hp;
  cudaStream_t st;
  std::vector<Layer> layers;
  float* tok_embd = nullptr;
  float* out_norm = nullptr;
  const ns_weight* output = nullptr;
  std::vector<void*> owned;  // device allocations freed with the context
  int n_seq = 0;             // KV blocks: ns_llama_set_sequences (1 from ns_llama_create)
  __half *kc = nullptr, *vc = nullptr;  // [n_layer][n_seq][n_head_kv][n_ctx][hd] fp16
  int* state = nullptr;   // device: {token, n_past, n_recorded, last_pick}
  int* tokens = nullptr;  // device: prompt tokens of the current eval
  int tok_cap = 0;        // ... their capacity: n_ctx, grown to the rows of a larger ns_llama_eval_batch pass
  int* plan = nullptr;    // device, ns_llama_eval_batch: kPlanInts (allocated on first use)
  int* record = nullptr;  // device: generated tokens
  int* bstate = nullptr;  // device, batched steps: [kMaxSeq][4] row states as `state` | [kMaxSeq] KV block of each row
  int* brecord = nullptr;   // device, batched steps: [n_seq][n_ctx] picks of each row
  float* am_val = nullptr;  // argmax partials: [kMaxSeq][kArgmaxBlocks]
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
  cudaGraphExec_t decode_exec = nullptr;
  cudaGraph_t decode_graph = nullptr;
  cudaGraphExec_t batch_exec[kMaxSeq + 1] = {};  // one batched step of n rows, captured on first use
  cudaGraph_t batch_graph[kMaxSeq + 1] = {};
  int* h_state = nullptr;  // pinned host staging
  int* h_bstate = nullptr;  // [kMaxSeq * 5]
  int* h_plan = nullptr;      // [kMaxBatchRows] tokens | kPlanInts tables, as `plan` (allocated with it)
  float* h_logits = nullptr;  // [n_seq][n_vocab]
  // ns_llama_set_sampling: the sampler takes the argmax's launch while `sampling`; its device state is allocated on first use
  bool sampling = false;
  ns_llama_sampling smp{};
  uint32_t* mt = nullptr;             // std::mt19937 [kMtWords]
  int* win = nullptr;                 // windows [kMaxSeq][kSampleMaxWindow], slot = KV block
  unsigned long long* s_keys = nullptr;  // [kMaxSeq][kSampleSlices][kSampleMaxK]
  int* s_pcnt = nullptr;              // [kMaxSeq][kSampleSlices]
  double* s_cp = nullptr;             // [kMaxSeq][kSampleMaxK]
  unsigned* s_tickets = nullptr;      // [kMaxSeq + 1]
  int* s_kept = nullptr;              // [kMaxSeq]
  int* s_ids = nullptr;               // [kMaxSeq][kSampleMaxK]
  float* s_probs = nullptr;           // [kMaxSeq][kSampleMaxK]
  // ns_llama_eval_all (allocated on first use): the lm_head's logits of one chunk of rows, the log-prob kernel's tickets and
  // partials, the rows' targets / log-probs / picks in internal order, and pinned staging for those and two chunks of logits
  float* all_logits = nullptr;        // [kAllChunk][n_vocab]
  unsigned* lp_tickets = nullptr;     // [kAllChunk] | max, id, sum [kAllChunk][kLogprobSlices]
  int* all_io = nullptr;              // [3][kMaxBatchRows]
  int* h_all = nullptr;               // [3][kMaxBatchRows] | [2][kAllChunk][n_vocab] floats
  cudaEvent_t all_ev[2] = {};
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
  if (c->decode_exec) {
    cudaGraphExecDestroy(c->decode_exec);
    cudaGraphDestroy(c->decode_graph);
    c->decode_exec = nullptr;
    c->decode_graph = nullptr;
  }
  for (int n = 0; n <= kMaxSeq; ++n)
    if (c->batch_exec[n]) {
      cudaGraphExecDestroy(c->batch_exec[n]);
      cudaGraphDestroy(c->batch_graph[n]);
      c->batch_exec[n] = nullptr;
      c->batch_graph[n] = nullptr;
    }
}

// (re)allocates everything sized by the number of KV blocks -- caches, logits, decode-attention partials and tickets, batch
// record -- and zeroes the caches and tickets.  On failure n_seq is 0 and every eval refuses to run.
static int alloc_sequences(ns_llama* c, int n_seq) {
  const ns_llama_hparams& hp = c->hp;
  const int hd = hp.n_embd / hp.n_head;
  void* old[6] = {c->kc, c->vc, c->logits, c->attn_part, c->attn_tickets, c->brecord};
  for (void* p : old) dev_free(c, p);
  c->kc = c->vc = nullptr;
  c->logits = c->attn_part = nullptr;
  c->attn_tickets = nullptr;
  c->brecord = nullptr;
  if (c->h_logits) cudaFreeHost(c->h_logits);
  c->h_logits = nullptr;
  c->n_seq = 0;
  const size_t kv_elems = (size_t)n_seq * hp.n_layer * hp.n_head_kv * hp.n_ctx * hd;
  c->attn_nsplit = attn_ranges(hp.n_ctx);
  c->kc = (__half*)dev_alloc(c, kv_elems * 2);
  c->vc = (__half*)dev_alloc(c, kv_elems * 2);
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
  NS_CUDA_TRY(cudaMemsetAsync(c->kc, 0, kv_elems * 2, c->st));
  NS_CUDA_TRY(cudaMemsetAsync(c->vc, 0, kv_elems * 2, c->st));
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
    const size_t need = (size_t)((3 + kAW) * hd + hp->n_ctx) * sizeof(float);
    if (need > 220 * 1024) {
      ns_set_error("ns_llama_create: n_ctx %d too large for the single-pass attention kernel (limit %zu positions at head size %d)",
                   hp->n_ctx, (size_t)(220 * 1024) / sizeof(float) - (size_t)(3 + kAW) * hd, hd);
      delete c;
      return nullptr;
    }
  }
  c->state = (int*)dev_alloc(c, 4 * sizeof(int));
  c->tokens = (int*)dev_alloc(c, (size_t)hp->n_ctx * sizeof(int));
  c->tok_cap = hp->n_ctx;
  c->record = (int*)dev_alloc(c, (size_t)hp->n_ctx * sizeof(int));
  c->bstate = (int*)dev_alloc(c, (size_t)kMaxSeq * 5 * sizeof(int));
  c->am_val = (float*)dev_alloc(c, (size_t)kMaxSeq * kArgmaxBlocks * sizeof(float));
  c->am_idx = (int*)dev_alloc(c, (size_t)kMaxSeq * kArgmaxBlocks * sizeof(int));
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
  if (c->h_state) cudaFreeHost(c->h_state);
  if (c->h_bstate) cudaFreeHost(c->h_bstate);
  if (c->h_plan) cudaFreeHost(c->h_plan);
  if (c->h_logits) cudaFreeHost(c->h_logits);
  if (c->h_all) cudaFreeHost(c->h_all);
  for (cudaEvent_t e : c->all_ev)
    if (e) cudaEventDestroy(e);
  delete c;
}

extern "C" int ns_llama_set_f32(ns_llama* c, int tensor, int layer, const float* host, size_t count) {
  if (!c || !host) return NS_E_INVALID;
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
    *slot = w;
  }
  drop_graphs(c);  // weights changed: the captured graphs hold stale pointers
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
  }
  return NS_OK;
}

// enqueue the whole forward pass for m new tokens (ids in c->tokens[0..m) or, when from_state, the single id in
// state[0]); position base = state[1]; KV block `seq`.  Leaves logits of the LAST token in c->logits and the greedy pick in
// state[3].  batch: m rows of m different sequences instead (row i: token and position in bstate[4 i ..], KV block
// bstate[4 kMaxSeq + i]), logits and argmax of every row, picks recorded in brecord [row][n_ctx].
// mix: m rows of mix->n segments of distinct sequences (ns_llama_eval_batch), ids in c->tokens; rows 0 .. d - 1 are one-token
// segments (token, position and block in bstate as a batched step), rows d .. m - 1 the longer ones (mix->rows / mix->tiles);
// logits and argmax (no advance) of each segment's last row, in internal order.
// sample (while sampling is on): 2 = store the windows and draw, 1 = store the windows and take each row's first candidate
// (a prompt piece whose pick is not returned), 0 = neither (the eager pass before a capture, evaluated again by the graph).
struct MixedPass {
  int n, d, n_tiles;
  const int* rows;   // device [m][2]: {position, KV block}
  const int* tiles;  // device [n_tiles][kTileInts], rows counted from row d
  const int* last;   // device [n]: last row of each segment
  const int* slot;   // device [n]: KV block of each segment
  const int* draw;   // device [n]: internal segment of caller index i
};
// the embedding and every layer: leaves the last layer's output rows in c->x
static int enqueue_body(ns_llama* c, int m, bool from_state, bool ring, int seq, bool batch, const MixedPass* mix) {
  const ns_llama_hparams& hp = c->hp;
  cudaStream_t st = c->st;
  const int E = hp.n_embd, hd = E / hp.n_head, kvd = hd * hp.n_head_kv;
  float* q = c->qkv;
  float* k = q + (size_t)m * E;
  float* v = k + (size_t)m * kvd;
  const int* toks = batch ? c->bstate : from_state ? c->state : c->tokens;
  NS_CUDA_TRY(ns_launch_pdl(batch ? embed_kernel<4> : embed_kernel<1>, dim3((unsigned)((E / 4 + 255) / 256), (unsigned)m), dim3(256), 0, st,
                            (const float*)c->tok_embd, toks, E, hp.n_vocab, c->x));
  ns_count_launch();
  const size_t blk = (size_t)hp.n_head_kv * hp.n_ctx * hd;  // one sequence's cache of one layer
  for (int il = 0; il < hp.n_layer; ++il) {
    const Layer& L = c->layers[il];
    __half* kc = c->kc + ((size_t)il * c->n_seq + (batch ? 0 : seq)) * blk;
    __half* vc = c->vc + ((size_t)il * c->n_seq + (batch ? 0 : seq)) * blk;
    // Decode rows: the attention RMSNorm (llama.cpp:205-210) rides in the activation quantiser of the Q/K/V launch(es) -- every
    // CTA reads the whole row anyway -- instead of a one-CTA kernel and a launch boundary of its own.
    const ns_weight* qkvw[3] = {L.wq, L.wk, L.wv};
    // one fused QKV node (llama.cpp:212-215) where the three weights form one, dst = [3][m][E] = q | k | v; else three matmuls
    const bool qkv_node = hp.n_head == hp.n_head_kv && ns_route(NS_NODE_QKV, qkvw, m, 0) >= 0;
    const bool fold = qkv_node ? ns_rmsnorm_fusable(qkvw, 3, m)
                               : hp.n_head != hp.n_head_kv && ns_rmsnorm_fusable(&qkvw[0], 1, m) && ns_rmsnorm_fusable(&qkvw[1], 1, m) &&
                                     ns_rmsnorm_fusable(&qkvw[2], 1, m);
    if (!fold)
      if (int rc = launch_rmsnorm(c->x, L.attn_norm, c->xn, m, E, hp.norm_eps, st)) return rc;
    const float* xq = fold ? c->x : c->xn;
    if (qkv_node) {
      if (int rc = ns_mul_qkv_norm(L.wq, L.wk, L.wv, xq, E, q, E, m, c->ws, (void*)st, fold ? L.attn_norm : nullptr, hp.norm_eps)) return rc;
    } else {
      float* dq[3] = {q, k, v};
      for (int i = 0; i < 3; ++i)
        if (int rc = fold ? ns_rmsnorm_mul_mat(qkvw[i], xq, E, L.attn_norm, hp.norm_eps, dq[i], i ? kvd : E, m, nullptr, c->ws, (void*)st)
                          : ns_mul_mat(qkvw[i], xq, E, dq[i], i ? kvd : E, m, nullptr, nullptr, 0, c->ws, (void*)st))
          return rc;
    }
    static const int dbg_skip = getenv("NS_LLAMA_DEBUG_SKIP") ? atoi(getenv("NS_LLAMA_DEBUG_SKIP")) : 0;  // timing experiments only
    if (mix) {  // kc / vc: block 0 of the layer
      const int d = mix->d;
      if (d > 0)
        if (int rc = launch_attention_batch(q, k, v, kc, vc, c->bstate, c->bstate + 4 * kMaxSeq, c->attn, c->attn_part, c->attn_tickets, d,
                                            hp.n_head, hp.n_head_kv, hd, hp.n_ctx, hp.rope_theta, hp.rope_scale, c->attn_attr, st))
          return rc;
      if (int rc = launch_attention_ragged(q + (size_t)d * E, k + (size_t)d * kvd, v + (size_t)d * kvd, kc, vc, mix->rows + 2 * d, mix->tiles,
                                           m - d, mix->n_tiles, c->attn + (size_t)d * E, hp.n_head, hp.n_head_kv, hd, hp.n_ctx,
                                           hp.rope_theta, hp.rope_scale, st))
        return rc;
    } else if (batch) {
      if (int rc = launch_attention_batch(q, k, v, kc, vc, c->bstate, c->bstate + 4 * kMaxSeq, c->attn, c->attn_part, c->attn_tickets, m,
                                          hp.n_head, hp.n_head_kv, hd, hp.n_ctx, hp.rope_theta, hp.rope_scale, c->attn_attr, st))
        return rc;
    } else if (!(m == 1 && (dbg_skip & 1))) {  // (else results are wrong: the attention launch is left out to measure what it costs)
      if (int rc = launch_attention(NS_ATTN_AUTO, q, k, v, kc, vc, c->state, c->attn, c->attn_part, c->attn_tickets, hp.n_head, hp.n_head_kv,
                                    hd, hp.n_ctx, m, hp.rope_theta, hp.rope_scale, c->attn_attr, st, ring ? &c->ring : nullptr))
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

static int enqueue_forward(ns_llama* c, int m, bool from_state, int advance, int* record, bool ring, int seq = 0, bool batch = false,
                           const MixedPass* mix = nullptr, int sample = 2) {
  if (int rc = enqueue_body(c, m, from_state, ring, seq, batch, mix)) return rc;
  const ns_llama_hparams& hp = c->hp;
  cudaStream_t st = c->st;
  const int E = hp.n_embd;
  const int* toks = batch ? c->bstate : from_state ? c->state : c->tokens;
  // logits of the last token only (model_eval keeps the last row unless logits_all); a batched step: of every row, each being
  // its sequence's last token (llama.cpp:745-758)
  const int rows = batch ? m : mix ? mix->n : 1;
  const float* xl = c->x + (size_t)(m - rows) * E;
  if (mix) {  // each segment's last row, gathered into attn (free after the last layer)
    NS_CUDA_TRY(ns_launch_pdl(gather_rows_kernel, dim3((unsigned)((E / 4 + 255) / 256), (unsigned)rows), dim3(256), 0, st,
                              (const float*)c->x, mix->last, E, c->attn));
    ns_count_launch();
    xl = c->attn;
  }
  const ns_weight* outw[1] = {c->output};
  if (ns_rmsnorm_fusable(outw, 1, rows)) {
    if (int rc = ns_rmsnorm_mul_mat(c->output, xl, E, c->out_norm, hp.norm_eps, c->logits, hp.n_vocab, rows, nullptr, c->ws, (void*)st))
      return rc;
  } else {
    if (int rc = launch_rmsnorm(xl, c->out_norm, c->xn, rows, E, hp.norm_eps, st)) return rc;
    if (int rc = ns_mul_mat(c->output, c->xn, E, c->logits, hp.n_vocab, rows, nullptr, nullptr, 0, c->ws, (void*)st)) return rc;
  }
  const bool rowwise = batch || mix;  // a pick per row, in bstate
  if (c->sampling) {
    SampleLaunch a{};
    a.logits = c->logits;
    a.n_vocab = hp.n_vocab;
    a.rows = rows;
    a.k = c->smp.top_k;
    a.top_p = c->smp.top_p;
    a.temp = c->smp.temperature;
    a.penalty = c->smp.repeat_penalty;
    a.W = c->smp.repeat_last_n < hp.n_ctx ? c->smp.repeat_last_n : hp.n_ctx;
    a.win = c->win;
    a.win_stride = kSampleMaxWindow;
    if (mix) {
      a.toks = c->tokens;
      a.last = mix->last;
      a.slot = mix->slot;
      a.order = mix->draw;
    } else if (batch) {
      a.toks = c->bstate;
      a.tok_stride = 4;
      a.tok_len = 1;
      a.slot = c->bstate + 4 * kMaxSeq;
    } else {
      a.toks = toks;
      a.tok_len = m;
      a.slot_const = seq;
    }
    a.store = sample >= 1;
    a.draw = sample >= 2;
    a.mt = c->mt;
    a.pkeys = c->s_keys;
    a.pcnt = c->s_pcnt;
    a.cp = c->s_cp;
    a.tickets = c->s_tickets;
    a.kept = c->s_kept;
    a.ids = c->s_ids;
    a.probs = c->s_probs;
    a.state = rowwise ? c->bstate : c->state;
    a.rowwise = rowwise;
    a.n_tokens = rowwise ? 1 : m;
    a.advance = advance;
    a.record = record;
    a.rec_stride = hp.n_ctx;
    return ns_launch_sample(a, st);
  }
  NS_CUDA_TRY(ns_launch_pdl(rowwise ? argmax_kernel<true> : argmax_kernel<false>, dim3((unsigned)kArgmaxBlocks, (unsigned)rows), dim3(256), 0, st, (const float*)c->logits,
                            hp.n_vocab, rowwise ? c->bstate : c->state, rowwise ? 1 : m, advance, record, hp.n_ctx, c->am_val, c->am_idx,
                            c->am_ticket));
  ns_count_launch();
  return NS_OK;
}

static int ensure_batch_graph(ns_llama* c, int n) {
  if (c->batch_exec[n]) return NS_OK;
  // as ensure_decode_graph: one eager pass that does not advance the rows (it writes the K/V rows the captured pass rewrites
  // with the same values), then the capture
  if (int rc = enqueue_forward(c, n, true, 0, nullptr, false, 0, true, nullptr, 0)) return rc;
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));
  NS_CUDA_TRY(cudaStreamBeginCapture(c->st, cudaStreamCaptureModeThreadLocal));
  int rc = enqueue_forward(c, n, true, 1, c->brecord, false, 0, true);
  cudaGraph_t g = nullptr;
  cudaError_t e = cudaStreamEndCapture(c->st, &g);
  if (rc) {
    if (g) cudaGraphDestroy(g);
    return rc;
  }
  if (!ns_cuda_ok(e, "cudaStreamEndCapture") || !g) return NS_E_CUDA;
  if (!ns_cuda_ok(cudaGraphInstantiate(&c->batch_exec[n], g, 0), "cudaGraphInstantiate")) {
    cudaGraphDestroy(g);
    return NS_E_CUDA;
  }
  c->batch_graph[n] = g;
  return NS_OK;
}

static int ensure_decode_graph(ns_llama* c) {
  if (c->decode_exec) return NS_OK;
  // one eager pass (no state advance; it writes the same K/V the real pass will) sets kernel attributes and sizes every
  // lazily-grown buffer outside the capture, then capture.  The eager pass runs the plain attention even when streaming: a
  // ring step rotates the cache, which must happen once; the plain kernel writes nothing once the cache is full.
  if (int rc = enqueue_forward(c, 1, true, 0, nullptr, false, 0, false, nullptr, 0)) return rc;
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));
  NS_CUDA_TRY(cudaStreamBeginCapture(c->st, cudaStreamCaptureModeThreadLocal));
  int rc = enqueue_forward(c, 1, true, 1, c->record, c->streaming);
  cudaGraph_t g = nullptr;
  cudaError_t e = cudaStreamEndCapture(c->st, &g);
  if (rc) {
    if (g) cudaGraphDestroy(g);
    return rc;
  }
  if (!ns_cuda_ok(e, "cudaStreamEndCapture") || !g) return NS_E_CUDA;
  if (!ns_cuda_ok(cudaGraphInstantiate(&c->decode_exec, g, 0), "cudaGraphInstantiate")) {
    cudaGraphDestroy(g);
    return NS_E_CUDA;
  }
  c->decode_graph = g;
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
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));  // nothing in flight replays the graph dropped below
  drop_graphs(c);
  c->streaming = n_keep >= 0;
  c->ring = Ring{n_keep, c->streaming ? shift_table(hd, c->hp.rope_theta) : ShiftTable{}};
  c->wrapped = false;
  return NS_OK;
}

// Sampling in place of greedy (model_post_sample_top_k_top_p_repeat): the generator is reseeded and every window restarts;
// NULL returns to greedy.  Either way the captured graphs, which bake in the pick kernel and its parameters, are dropped.
extern "C" int ns_llama_set_sampling(ns_llama* c, const ns_llama_sampling* s) {
  if (!c) return NS_E_INVALID;
  if (s)
    if (int rc = ns_sample_check("ns_llama_set_sampling", s)) return rc;
  if (s && !c->mt) {
    c->mt = (uint32_t*)dev_alloc(c, kMtWords * sizeof(uint32_t));
    c->win = (int*)dev_alloc(c, (size_t)kMaxSeq * kSampleMaxWindow * sizeof(int));
    c->s_keys = (unsigned long long*)dev_alloc(c, (size_t)kMaxSeq * kSampleSlices * kSampleMaxK * sizeof(unsigned long long));
    c->s_pcnt = (int*)dev_alloc(c, (size_t)kMaxSeq * kSampleSlices * sizeof(int));
    c->s_cp = (double*)dev_alloc(c, (size_t)kMaxSeq * kSampleMaxK * sizeof(double));
    c->s_tickets = (unsigned*)dev_alloc(c, (kMaxSeq + 1) * sizeof(unsigned));
    c->s_kept = (int*)dev_alloc(c, kMaxSeq * sizeof(int));
    c->s_ids = (int*)dev_alloc(c, (size_t)kMaxSeq * kSampleMaxK * sizeof(int));
    c->s_probs = (float*)dev_alloc(c, (size_t)kMaxSeq * kSampleMaxK * sizeof(float));
    if (!c->mt || !c->win || !c->s_keys || !c->s_pcnt || !c->s_cp || !c->s_tickets || !c->s_kept || !c->s_ids || !c->s_probs) {
      void* got[9] = {c->mt, c->win, c->s_keys, c->s_pcnt, c->s_cp, c->s_tickets, c->s_kept, c->s_ids, c->s_probs};
      for (void* p : got) dev_free(c, p);
      c->mt = nullptr;
      return NS_E_CUDA;
    }
    NS_CUDA_TRY(cudaMemsetAsync(c->s_tickets, 0, (kMaxSeq + 1) * sizeof(unsigned), c->st));
  }
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));  // nothing in flight replays the graphs dropped below or reads the generator
  drop_graphs(c);
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

// a sequence evaluated at n_past 0 restarts its sampling window as zeros (the reference's fresh history); nothing while greedy
static int reset_window(ns_llama* c, int slot) {
  if (!c->sampling) return NS_OK;
  NS_CUDA_TRY(cudaMemsetAsync(c->win + (size_t)slot * kSampleMaxWindow, 0, kSampleMaxWindow * sizeof(int), c->st));
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
  if (n_past == 0)
    if (int rc = reset_window(c, seq)) return rc;
  c->h_state[0] = tokens[0];
  c->h_state[1] = n_past;
  c->h_state[2] = 0;
  c->h_state[3] = 0;
  NS_CUDA_TRY(cudaMemcpyAsync(c->state, c->h_state, 4 * sizeof(int), cudaMemcpyHostToDevice, st));
  if (n_tokens == 1 && seq == 0 && draw) {
    if (int rc = ensure_decode_graph(c)) return rc;
    NS_CUDA_TRY(cudaGraphLaunch(c->decode_exec, st));
  } else {
    NS_CUDA_TRY(cudaMemcpyAsync(c->tokens, tokens, (size_t)n_tokens * sizeof(int), cudaMemcpyHostToDevice, st));
    if (int rc = enqueue_forward(c, n_tokens, false, 1, nullptr, false, seq, false, nullptr, draw ? 2 : 1)) return rc;
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
  if (n_seq > 1 && hd != 64 && hd != 128) {
    ns_set_error("ns_llama_set_sequences: head size %d (the batched decode attention takes 64 or 128)", hd);
    return NS_E_UNSUPPORTED;
  }
  NS_CUDA_TRY(cudaStreamSynchronize(c->st));  // nothing in flight uses the blocks or graphs released below
  drop_graphs(c);
  c->n_total = 0;
  c->wrapped = false;
  if (int rc = alloc_sequences(c, n_seq)) return rc;
  if (c->win) NS_CUDA_TRY(cudaMemsetAsync(c->win, 0, (size_t)kMaxSeq * kSampleMaxWindow * sizeof(int), c->st));
  return NS_OK;
}

// argument checks and the rows' device state of a batched call (no launch when the call is refused)
static int start_batch(ns_llama* c, const char* who, int n, const int* seq, const int32_t* tokens, const int* n_past, int steps) {
  if (!c || !seq || !tokens || !n_past) {
    ns_set_error("%s: null pointer", who);
    return NS_E_INVALID;
  }
  if (steps <= 0) {
    ns_set_error("%s: %d steps", who, steps);
    return NS_E_INVALID;
  }
  if (int rc = check_rows(who, c->n_seq, n, seq, n_past, steps, c->hp.n_ctx)) return rc;
  const int hd = c->hp.n_embd / c->hp.n_head;
  if (hd != 64 && hd != 128) {
    ns_set_error("%s: head size %d (the batched decode attention takes 64 or 128)", who, hd);
    return NS_E_UNSUPPORTED;
  }
  if (c->streaming) {
    ns_set_error("%s: streaming is on (the ring serves ns_llama_eval / ns_llama_generate only)", who);
    return NS_E_UNSUPPORTED;
  }
  if (int rc = check_complete(c)) return rc;
  if (int rc = ensure_buffers(c, n)) return rc;
  for (int i = 0; i < n; ++i)
    if (n_past[i] == 0)
      if (int rc = reset_window(c, seq[i])) return rc;
  for (int i = 0; i < kMaxSeq; ++i) {
    int* r = c->h_bstate + 4 * i;
    r[0] = i < n ? tokens[i] : 0;
    r[1] = i < n ? n_past[i] : 0;
    r[2] = r[3] = 0;
    c->h_bstate[4 * kMaxSeq + i] = i < n ? seq[i] : 0;
  }
  NS_CUDA_TRY(cudaMemcpyAsync(c->bstate, c->h_bstate, (size_t)kMaxSeq * 5 * sizeof(int), cudaMemcpyHostToDevice, c->st));
  return ensure_batch_graph(c, n);
}

extern "C" int ns_llama_decode_batch(ns_llama* c, int n, const int* seq, const int32_t* tokens, const int* n_past, float* logits_host,
                                     int32_t* next_tokens) {
  if (int rc = ns_ensure_device()) return rc;
  if (int rc = start_batch(c, "ns_llama_decode_batch", n, seq, tokens, n_past, 1)) return rc;
  cudaStream_t st = c->st;
  const size_t nl = (size_t)n * c->hp.n_vocab;
  NS_CUDA_TRY(cudaGraphLaunch(c->batch_exec[n], st));
  if (logits_host) NS_CUDA_TRY(cudaMemcpyAsync(c->h_logits, c->logits, nl * 4, cudaMemcpyDeviceToHost, st));
  NS_CUDA_TRY(cudaMemcpyAsync(c->h_bstate, c->bstate, (size_t)n * 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
  NS_CUDA_TRY(cudaStreamSynchronize(st));
  if (logits_host) memcpy(logits_host, c->h_logits, nl * 4);
  if (next_tokens)
    for (int i = 0; i < n; ++i) next_tokens[i] = c->h_bstate[4 * i + 3];
  return NS_OK;
}

extern "C" int ns_llama_generate_batch(ns_llama* c, int n, const int* seq, const int32_t* first_tokens, const int* n_past, int n_new,
                                       int32_t* out_tokens) {
  if (int rc = ns_ensure_device()) return rc;
  if (!out_tokens) {
    ns_set_error("ns_llama_generate_batch: null pointer");
    return NS_E_INVALID;
  }
  if (int rc = start_batch(c, "ns_llama_generate_batch", n, seq, first_tokens, n_past, n_new)) return rc;
  cudaStream_t st = c->st;
  for (int i = 0; i < n_new; ++i) NS_CUDA_TRY(cudaGraphLaunch(c->batch_exec[n], st));
  // row r's picks: brecord[r][0 .. n_new) (n_past + n_new <= n_ctx)
  NS_CUDA_TRY(cudaMemcpy2DAsync(out_tokens, (size_t)n_new * sizeof(int), c->brecord, (size_t)c->hp.n_ctx * sizeof(int),
                                (size_t)n_new * sizeof(int), (size_t)n, cudaMemcpyDeviceToHost, st));
  NS_CUDA_TRY(cudaStreamSynchronize(st));
  return NS_OK;
}

// the argument rules of a pass over segments (ns_llama_eval_batch, ns_llama_eval_all); nothing is launched
static int check_pass(ns_llama* c, const char* who, int n, const int* seq, const int* n_tokens, const int32_t* tokens, const int* n_past,
                      BatchPlan& p) {
  if (!c || !tokens) {
    ns_set_error("%s: null pointer", who);
    return NS_E_INVALID;
  }
  if (int rc = plan_batch(who, c->n_seq, c->hp.n_ctx, n, seq, n_tokens, n_past, p)) return rc;
  const int hd = c->hp.n_embd / c->hp.n_head;
  if (hd != 64 && hd != 128) {
    ns_set_error("%s: head size %d (the batched decode and ragged prompt attention take 64 or 128)", who, hd);
    return NS_E_UNSUPPORTED;
  }
  if (c->streaming) {
    ns_set_error("%s: streaming is on (the ring serves ns_llama_eval / ns_llama_generate only; llama.cpp:104)", who);
    return NS_E_UNSUPPORTED;
  }
  if (c->exact_prefill && p.T > 32) {
    ns_set_error("%s: %d rows in exact-prefill mode (the integer block sums hold up to 32 rows)", who, p.T);
    return NS_E_UNSUPPORTED;
  }
  return NS_OK;
}

// The device tables of a pass over the segments of plan p: ids in internal order, rows, tiles, each segment's last row, block and
// draw order, and the one-token rows' states as a batched step's.  *mix describes the pass.
static int stage_segments(ns_llama* c, int n, const int* seq, const int* n_tokens, const int32_t* tokens, const int* n_past,
                          const BatchPlan& p, MixedPass* mix) {
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
  // staging: ids in internal order | rows | tiles | last rows; the one-token rows' states as a batched step's
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
  for (int i = 0; i < n; ++i)
    if (n_past[i] == 0)
      if (int rc = reset_window(c, seq[i])) return rc;
  std::copy(p.rows.begin(), p.rows.end(), h_tab);
  std::copy(p.tiles.begin(), p.tiles.end(), h_tab + 2 * kMaxBatchRows);
  for (int j = 0; j < kMaxSeq; ++j) {
    int* r = c->h_bstate + 4 * j;
    const int i = j < p.d ? p.order[j] : -1;
    r[0] = i >= 0 ? tokens[off[i]] : 0;
    r[1] = i >= 0 ? n_past[i] : 0;
    r[2] = r[3] = 0;
    c->h_bstate[4 * kMaxSeq + j] = i >= 0 ? seq[i] : 0;
  }
  NS_CUDA_TRY(cudaMemcpyAsync(c->tokens, h_tok, (size_t)p.T * sizeof(int), cudaMemcpyHostToDevice, st));
  NS_CUDA_TRY(cudaMemcpyAsync(c->plan, h_tab, (size_t)kPlanInts * sizeof(int), cudaMemcpyHostToDevice, st));
  NS_CUDA_TRY(cudaMemcpyAsync(c->bstate, c->h_bstate, (size_t)kMaxSeq * 5 * sizeof(int), cudaMemcpyHostToDevice, st));
  const int* d_last = c->plan + 2 * kMaxBatchRows + kPlanTiles * kTileInts;
  *mix = MixedPass{n, p.d, (int)p.tiles.size() / kTileInts, c->plan, c->plan + 2 * kMaxBatchRows, d_last, d_last + kMaxSeq,
                   d_last + 2 * kMaxSeq};
  return NS_OK;
}

// model_eval over n inputs (llama.cpp:53-90, 329-460, 745-758): one pass over the token segments of n distinct sequences
extern "C" int ns_llama_eval_batch(ns_llama* c, int n, const int* seq, const int* n_tokens, const int32_t* tokens, const int* n_past,
                                   float* logits_host, int32_t* next_tokens) {
  const char* who = "ns_llama_eval_batch";
  if (int rc = ns_ensure_device()) return rc;
  BatchPlan p;
  if (int rc = check_pass(c, who, n, seq, n_tokens, tokens, n_past, p)) return rc;
  if (p.d == n) return ns_llama_decode_batch(c, n, seq, tokens, n_past, logits_host, next_tokens);  // its captured graph
  if (int rc = check_complete(c)) return rc;
  if (int rc = ensure_buffers(c, p.T)) return rc;
  cudaStream_t st = c->st;
  MixedPass mix;
  if (int rc = stage_segments(c, n, seq, n_tokens, tokens, n_past, p, &mix)) return rc;
  if (int rc = enqueue_forward(c, p.T, false, 0, nullptr, false, 0, false, &mix)) return rc;
  const size_t nv = (size_t)c->hp.n_vocab;
  if (logits_host) NS_CUDA_TRY(cudaMemcpyAsync(c->h_logits, c->logits, n * nv * 4, cudaMemcpyDeviceToHost, st));
  NS_CUDA_TRY(cudaMemcpyAsync(c->h_bstate, c->bstate, (size_t)n * 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
  NS_CUDA_TRY(cudaStreamSynchronize(st));
  for (int j = 0; j < n; ++j) {  // back to the caller's order
    const int i = p.order[j];
    if (logits_host) memcpy(logits_host + (size_t)i * nv, c->h_logits + (size_t)j * nv, nv * 4);
    if (next_tokens) next_tokens[i] = c->h_bstate[4 * j + 3];
  }
  return NS_OK;
}

static int ensure_all_rows(ns_llama* c) {
  if (c->all_logits) return NS_OK;
  const size_t V = (size_t)c->hp.n_vocab;
  float* lg = (float*)dev_alloc(c, (size_t)kAllChunk * V * 4);
  unsigned* tk = (unsigned*)dev_alloc(c, (size_t)kAllChunk * (1 + 3 * kLogprobSlices) * 4);
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
  BatchPlan p;
  if (int rc = check_pass(c, who, n, seq, n_tokens, tokens, n_past, p)) return rc;
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
  if (c->sampling) {
    ns_set_error("%s: sampling is on (a scoring pass draws nothing; set greedy first)", who);
    return NS_E_UNSUPPORTED;
  }
  if (int rc = check_complete(c)) return rc;
  if (int rc = ensure_buffers(c, T)) return rc;
  if (int rc = ensure_all_rows(c)) return rc;
  cudaStream_t st = c->st;
  MixedPass mix;
  if (int rc = stage_segments(c, n, seq, n_tokens, tokens, n_past, p, &mix)) return rc;
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
  // one-token segments only: the kernels of ns_llama_decode_batch's graph, eagerly
  if (int rc = enqueue_body(c, T, false, false, 0, p.d == n, p.d == n ? nullptr : &mix)) return rc;
  const ns_weight* outw[1] = {c->output};
  const bool fold = T <= kAllChunk && ns_rmsnorm_fusable(outw, 1, T);
  if (!fold)
    if (int rc = launch_rmsnorm(c->x, c->out_norm, c->xn, T, E, c->hp.norm_eps, st)) return rc;
  LogprobLaunch a{};
  a.logits = c->all_logits;
  a.n_vocab = V;
  a.tickets = c->lp_tickets;
  a.pmax = reinterpret_cast<float*>(c->lp_tickets + kAllChunk);
  a.pidx = reinterpret_cast<int*>(a.pmax + kAllChunk * kLogprobSlices);
  a.psum = reinterpret_cast<float*>(a.pidx + kAllChunk * kLogprobSlices);
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
    if (int rc = fold ? ns_rmsnorm_mul_mat(c->output, c->x, E, c->out_norm, c->hp.norm_eps, c->all_logits, V, rows, nullptr, c->ws, (void*)st)
                      : ns_mul_mat(c->output, c->xn + (size_t)r0 * E, E, c->all_logits, V, rows, nullptr, nullptr, flags, c->ws, (void*)st))
      return rc;
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
  if (int rc = ensure_decode_graph(c)) return rc;
  cudaStream_t st = c->st;
  if (n_past == 0)
    if (int rc = reset_window(c, 0)) return rc;
  c->h_state[0] = first_token;
  c->h_state[1] = n_past;
  c->h_state[2] = 0;
  c->h_state[3] = 0;
  NS_CUDA_TRY(cudaMemcpyAsync(c->state, c->h_state, 4 * sizeof(int), cudaMemcpyHostToDevice, st));
  // the record buffer holds n_ctx picks: a streaming generation past n_ctx drains it in pieces (stream-ordered, no host wait)
  for (int i0 = 0; i0 < n_new; i0 += c->hp.n_ctx) {
    const int n = n_new - i0 < c->hp.n_ctx ? n_new - i0 : c->hp.n_ctx;
    if (i0) NS_CUDA_TRY(cudaMemsetAsync(c->state + 2, 0, sizeof(int), st));
    for (int i = 0; i < n; ++i) NS_CUDA_TRY(cudaGraphLaunch(c->decode_exec, st));
    NS_CUDA_TRY(cudaMemcpyAsync(out_tokens + i0, c->record, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
  }
  NS_CUDA_TRY(cudaStreamSynchronize(st));
  advance_position(c, n_past, n_new);
  return NS_OK;
}

extern "C" unsigned long long ns_llama_kv_bytes(const ns_llama* c) {
  if (!c) return 0;
  return (unsigned long long)2 * c->n_seq * c->hp.n_layer * c->hp.n_head_kv * c->hp.n_ctx * (c->hp.n_embd / c->hp.n_head) * 2;
}

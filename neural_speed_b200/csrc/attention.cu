// attention.cu -- one layer's RoPE, fp16 KV append and causal attention for the eval step (llama.cu, whose header states the
// numerics), the plan of a pass over token segments, and the standalone ns_llama_attention* entries.
#include <algorithm>

#include "async_copy.cuh"
#include "attention.cuh"
#include "kv_cache.cuh"

namespace {

constexpr int kAttnThreads = 128;

// rope (mode 0) on q and k of every new token + append k,v to the fp16 cache.
// grid (n_head + n_head_kv, n_tokens), hd/2 threads.  pos = state[1] + t.
// RAGGED: the rows belong to segments of several sequences (ns_llama_eval_batch); row t takes its position and its KV block
// ([n_seq][n_head_kv][n_ctx][hd]) from rows[2 t], rows[2 t + 1] instead.
// KV = NS_KV_Q8_0: kc / vc are the code planes, kd / vd the scale planes (kv_cache.cuh); the rotated k and the projected v rows are
// quantised in fp32, one 32-block per 16 threads.
template <bool RAGGED = false, int KV = NS_KV_F16>
__global__ void rope_kv_kernel(float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk, const float* __restrict__ v, int ldv,
                               kv_elem_t<KV>* __restrict__ kc, kv_elem_t<KV>* __restrict__ vc, const int* __restrict__ state, int n_head,
                               int n_head_kv, int hd, int n_ctx, float theta_scale, float freq_scale, const int* __restrict__ rows,
                               __half* __restrict__ kd, __half* __restrict__ vd) {
  constexpr bool Q8 = KV == NS_KV_Q8_0;
  pdl_launch_dependents();
  pdl_wait();
  const int h = blockIdx.x, t = blockIdx.y, i = threadIdx.x;  // pair index
  int pos;
  if (RAGGED) {
    pos = rows[2 * t];
    const size_t blk = (size_t)rows[2 * t + 1] * n_head_kv * n_ctx * hd;
    kc += blk;
    vc += blk;
    if constexpr (Q8) {
      kd += (size_t)rows[2 * t + 1] * n_head_kv * kv_d_stride(n_ctx, hd);
      vd += (size_t)rows[2 * t + 1] * n_head_kv * kv_d_stride(n_ctx, hd);
    }
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
      if constexpr (Q8) {  // whole warps: hd / 2 threads, the branch uniform over the CTA
        const float* pv = v + (size_t)t * ldv + (size_t)hk * hd + 2 * i;
        const size_t drow = (size_t)hk * kv_d_stride(n_ctx, hd) + (size_t)pos * (hd / kKvQ8Block);
        kv_q8_store_pair(kc + ((size_t)hk * n_ctx + pos) * hd, kd + drow, i, kv_q8_quant_pair(x0 * cs - x1 * sn, x0 * sn + x1 * cs));
        kv_q8_store_pair(vc + ((size_t)hk * n_ctx + pos) * hd, vd + drow, i, kv_q8_quant_pair(pv[0], pv[1]));
      } else {
        __half* kr = kc + ((size_t)hk * n_ctx + pos) * hd + 2 * i;
        kr[0] = __float2half_rn(x0 * cs - x1 * sn);
        kr[1] = __float2half_rn(x0 * sn + x1 * cs);
        const float* pv = v + (size_t)t * ldv + (size_t)hk * hd + 2 * i;
        __half* vr = vc + ((size_t)hk * n_ctx + pos) * hd + 2 * i;
        vr[0] = __float2half_rn(pv[0]);
        vr[1] = __float2half_rn(pv[1]);
      }
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

// Decode-shaped attention for head sizes 64 / 128 (attn_all_hd): kAW warps per (head, token); a warp streams whole K/V rows (one
// 4- or 8-byte load per lane), four rows in flight; with FUSE (single new token) the kernel also applies RoPE to its q head and to
// the new k row and appends k,v to the cache, so rope_kv_kernel is not launched.
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
// (<= 64 KB each; 48 KB at head size 96, whose rows of 192 B keep every range 16-byte aligned) on one mbarrier: a single
// global-memory latency per launch instead of a chain of dependent row loads -- the old kernel spent 2-3 round trips per pass at
// 100-200 positions.  Scores, soft_max and P.V then run out of shared memory.
// One active range (<= 256 positions): exactly the reference arithmetic (global maximum, e = fp16(exp(fp16(s - max))),
// p = fp16(e / sum), fp32 sums).  Several: every CTA leaves {max, sum e, sum e V} of its range, the last one to arrive (ticket per
// head) merges them with exp(max_s - max) weights -- same values up to the fp16 rounding of p (measured: tests/test_gpu_attention.py).
// Bound: latency at short contexts; HBM (2 x len x hd x 2 B per kv head) at long ones, spread over n_head x ceil(len / 256) CTAs.
// Head sizes 64 / 96 / 128 (attn_fast_hd): a lane owns EPL = hd / 32 consecutive elements of a row; 96 (fp16, RING = false only)
// reads its three with 2-byte loads.
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
//
// KV = NS_KV_Q8_0 (RING = false): kc / vc are the code planes, kd / vd the scale planes (kv_cache.cuh).  A range arrives as four
// bulk copies (codes and scales of K and V, the codes in the first half of the fp16 tile's space, the scales after them) and
// is dequantised on use.  The new k / v rows are quantised here (one 32-block per 16 threads) and the kernel scores and sums
// their dequantised values, as if read back from the cache.
constexpr int kSplitKeys = 256;
constexpr int kDW = 16;  // warps per CTA
template <int HD>
static constexpr size_t attn_decode_smem() {
  return (size_t)2 * kSplitKeys * HD * 2 + (size_t)(3 + kDW) * HD * 4 + (size_t)(kSplitKeys + 8) * 4 + 16;
}
template <int HD, bool RING, bool BATCH = false, int KV = NS_KV_F16>
__global__ void __launch_bounds__(kDW * 32) attn_decode_kernel(const float* __restrict__ q, const float* __restrict__ knew,
                                                            const float* __restrict__ vnew, kv_elem_t<KV>* __restrict__ kc,
                                                            kv_elem_t<KV>* __restrict__ vc, const int* __restrict__ state,
                                                            float* __restrict__ out, float* __restrict__ part_ws, unsigned* __restrict__ tickets,
                                                            int n_head, int n_head_kv, int n_ctx, int nsplit, float scale, float theta_scale,
                                                            float freq_scale, int n_keep, const ShiftTable tab, const int* __restrict__ seqs,
                                                            __half* __restrict__ kd, __half* __restrict__ vd) {
  static_assert(!(RING && BATCH), "the ring serves one sequence");
  constexpr bool Q8 = KV == NS_KV_Q8_0;
  static_assert(!(RING && Q8), "the ring shifts fp16 keys");
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
    if constexpr (Q8) {
      kd += (size_t)seqs[row] * n_head_kv * kv_d_stride(n_ctx, HD);
      vd += (size_t)seqs[row] * n_head_kv * kv_d_stride(n_ctx, HD);
    }
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
  kv_elem_t<KV>* kh = kc + (size_t)hk * n_ctx * HD;
  kv_elem_t<KV>* vh = vc + (size_t)hk * n_ctx * HD;
  __half* kdh = Q8 ? kd + (size_t)hk * kv_d_stride(n_ctx, HD) : nullptr;  // Q8_0: the head's scales
  __half* vdh = Q8 ? vd + (size_t)hk * kv_d_stride(n_ctx, HD) : nullptr;
  const uint32_t bar_a = smem_u32(bar);
  if (threadIdx.x == 0) {
    mbar_init(bar_a, 1);
    fence_mbar_init();
    // the cached rows of this range were written by earlier tokens' launches: their copies start before the wait as well and
    // overlap the tail of the Q/K/V launch.  In the ring, the rows this token rewrites (shifted K, the new K / V slot) were
    // likewise last written by this layer's launch of the previous token -- the launch whose appended row the plain step
    // already reads here -- so the same ordering covers them.
    if (ncache > 0) {
      if constexpr (Q8) {
        const uint32_t qbytes = (uint32_t)ncache * HD, dbytes = kv_q8_d_bytes(ncache, HD);
        mbar_expect_tx(bar_a, 2 * (qbytes + dbytes));
        bulk_g2s(smem_u32(Kt), kh + (size_t)i0 * HD, qbytes, bar_a);
        bulk_g2s(smem_u32(Kt) + kSplitKeys * HD, kdh + (size_t)i0 * (HD / kKvQ8Block), dbytes, bar_a);
        bulk_g2s(smem_u32(Vt), vh + (size_t)i0 * HD, qbytes, bar_a);
        bulk_g2s(smem_u32(Vt) + kSplitKeys * HD, vdh + (size_t)i0 * (HD / kKvQ8Block), dbytes, bar_a);
      } else {
        const uint32_t bytes = (uint32_t)ncache * HD * 2;
        mbar_expect_tx(bar_a, 2 * bytes);
        bulk_g2s(smem_u32(Kt), kh + (size_t)i0 * HD, bytes, bar_a);
        bulk_g2s(smem_u32(Vt), vh + (size_t)i0 * HD, bytes, bar_a);
      }
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
      if constexpr (Q8) {  // threads < HD / 2 are whole warps; has_new is uniform over the CTA
        const float* vr = vnew + (size_t)hk * HD;
        const KvQ8Pair a = kv_q8_quant_pair(k0 * cs - k1 * sn, k0 * sn + k1 * cs), b = kv_q8_quant_pair(vr[2 * i], vr[2 * i + 1]);
        sk[2 * i] = kv_q8_value(a.q0, a.d);
        sk[2 * i + 1] = kv_q8_value(a.q1, a.d);
        sv[2 * i] = kv_q8_value(b.q0, b.d);
        sv[2 * i + 1] = kv_q8_value(b.q1, b.d);
        if (h0 % group == 0) {
          kv_q8_store_pair(kh + (size_t)pos * HD, kdh + (size_t)pos * (HD / kKvQ8Block), i, a);
          kv_q8_store_pair(vh + (size_t)pos * HD, vdh + (size_t)pos * (HD / kKvQ8Block), i, b);
        }
      } else {
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
  }
  const int shift0 = wrapped ? min(max(n_keep - i0, 0), ncache) : ncache;  // staged rows [shift0, ncache) are shifted
  if (wrapped) {
    mbar_wait(bar_a, 0);
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
    fence_proxy_async();  // the shifted rows, visible to the bulk store
    __syncthreads();
    if (threadIdx.x == 0 && shift0 < ncache) {
      bulk_s2g(kh + (size_t)(i0 + shift0) * HD, smem_u32(Kt + (size_t)shift0 * HD), (uint32_t)(ncache - shift0) * HD * 2);
      bulk_commit();
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
  if (ncache > 0) mbar_wait(bar_a, 0);
  auto row = [&](const __half* base, int r, float* dst) {
    if constexpr (Q8) {  // base: the tile's space, codes [kSplitKeys][HD] then scales [kSplitKeys][HD / 32]
      const int8_t* qt = reinterpret_cast<const int8_t*>(base);
      const __half* dt = reinterpret_cast<const __half*>(qt + kSplitKeys * HD);
      kv_q8_load<EPL>(qt + (size_t)r * HD + lane * EPL, dt[r * (HD / kKvQ8Block) + lane * EPL / kKvQ8Block], dst);
    } else if (EPL == 4) {
      const uint2 u = *reinterpret_cast<const uint2*>(base + (size_t)r * HD + lane * 4);
      const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
      dst[0] = a.x, dst[1] = a.y, dst[2] = b.x, dst[3] = b.y;
    } else if (EPL == 2) {
      const float2 a = __half22float2(*reinterpret_cast<const __half2*>(base + (size_t)r * HD + lane * 2));
      dst[0] = a.x, dst[1] = a.y;
    } else {  // HD 96: three halves per lane, 6 bytes apart -- not aligned for a wider load (two lanes share a bank at most)
#pragma unroll
      for (int e = 0; e < EPL; ++e) dst[e] = __half2float(base[(size_t)r * HD + lane * EPL + e]);
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
  if (wrapped && threadIdx.x == 0 && shift0 < ncache) bulk_wait_all();
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
// (conflict-free 32-bit B-fragment loads for K, ldmatrix.trans for V; at HD 96 a row of 208 B rotates the banks by 20 words, still
// conflict-free); every q-tile of a head re-reads that head's K / V through L2.
// Bound: tensor pipe / shared-memory bandwidth (K and V of one head are 0.5 MB at 2048 positions -- L2 resident).
//
// RAGGED: the query rows are segments of several sequences (ns_llama_eval_batch, llama.cpp:414-489 run per input), grid
// (tiles, n_head).  CTA x reads tiles[5 x] = {segment's first row, its length, its n_past, its KV block, the tile's first query row
// inside the segment}, offsets q / out by the first row and kc / vc by the block, and takes pos0 = n_past, m = length.  Everything
// after those offsets is the single-sequence code, so each segment is bit-identical to a launch of its own.
//
// KV = NS_KV_Q8_0: kc / vc are the code planes, kd / vd the scale planes (kv_cache.cuh); the tile loads write the dequantised
// values fp16(q * d) into the same padded fp16 tiles, and everything after them is the fp16 kernel's.
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ void mma_f16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// At HD 96 ptxas, left to itself, caps the ragged form near 168 registers and spills; one CTA per SM as the floor gives it the
// registers it needs (the 64 / 128 forms keep the default bound).
template <int HD, bool RAGGED = false, int KV = NS_KV_F16>
__global__ void __launch_bounds__(128, HD == 96 ? 1 : 0)
    attn_mma_kernel(const float* __restrict__ q, int ldq, const kv_elem_t<KV>* __restrict__ kc, const kv_elem_t<KV>* __restrict__ vc,
                    const int* __restrict__ state, float* __restrict__ out, int ldo, int n_head, int n_head_kv, int n_ctx, int m,
                    float scale, const int* __restrict__ tiles, const __half* __restrict__ kd, const __half* __restrict__ vd) {
  constexpr bool Q8 = KV == NS_KV_Q8_0;
  constexpr int LD = HD + 8;  // halves per shared-memory row: 16 bytes of padding rotate the banks by 4 words per row
  constexpr int KS = HD / 16, NT = HD / 8;  // HD 96: 6 k-steps of Q K^T, 12 n-tiles (6 ldmatrix.x4) of P V
  static_assert(kAttnMmaKeys * (HD / 8) % 128 == 0, "load_tile: whole 16-byte chunks per thread");
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
    if constexpr (Q8) {
      kd += (size_t)tl[3] * n_head_kv * kv_d_stride(n_ctx, HD);
      vd += (size_t)tl[3] * n_head_kv * kv_d_stride(n_ctx, HD);
    }
    m = tl[1];
    pos0 = tl[2];
    q0 = tl[4];
  } else {
    pos0 = state[1];
    q0 = blockIdx.x * kAttnMmaRows;
  }
  const int row0 = q0 + warp * 16 + g, row1 = row0 + 8;  // this thread's two query rows (token indices of the batch)
  const int total = min(pos0 + m, n_ctx);                // keys that exist
  const kv_elem_t<KV>* kh = kc + (size_t)hk * n_ctx * HD;
  const kv_elem_t<KV>* vh = vc + (size_t)hk * n_ctx * HD;
  const __half* kdh = Q8 ? kd + (size_t)hk * kv_d_stride(n_ctx, HD) : nullptr;  // Q8_0: the head's scales
  const __half* vdh = Q8 ? vd + (size_t)hk * kv_d_stride(n_ctx, HD) : nullptr;

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

  auto load_tile = [&](const kv_elem_t<KV>* base, const __half* dbase, __half* dst, int key0) {
    constexpr int C16 = HD / 8;  // 16-byte chunks per row
#pragma unroll
    for (int i = 0; i < kAttnMmaKeys * C16 / 128; ++i) {
      const int idx = i * 128 + (int)threadIdx.x;
      const int r = idx / C16, c = idx % C16;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if constexpr (Q8) {
        if (key0 + r < total)
          v = kv_q8_load8_h(base + (size_t)(key0 + r) * HD + c * 8, dbase[(size_t)(key0 + r) * (HD / kKvQ8Block) + c * 8 / kKvQ8Block]);
      } else {
        if (key0 + r < total) v = *reinterpret_cast<const uint4*>(base + (size_t)(key0 + r) * HD + c * 8);
      }
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
    load_tile(kh, kdh, Ks, kt * kAttnMmaKeys);
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
    load_tile(kh, kdh, Ks, kt * kAttnMmaKeys);
    load_tile(vh, vdh, Vs, kt * kAttnMmaKeys);
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
        const uint32_t addr = smem_u32(vrow + n2 * 16);
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

}  // namespace

// ---- one layer's attention: RoPE of q and of the m new k rows at positions state[1] + t, KV append, causal attention ----------
// q [m][n_head * hd] (rotated in place unless a fused kernel rotates it in registers), k / v [m][n_head_kv * hd], cache
// [n_head_kv][n_ctx][hd] (kv_cache.cuh), out [m][n_head * hd].  NS_ATTN_AUTO picks:
//   hd 64 / 128, one row    attn_decode_kernel (context split over 256-position ranges) while the context has <= 1024 ranges
//                           and NS_ATTN_OLD_DECODE is unset, else attn_fast_kernel<FUSE>
//   hd 64 / 128, >= 8 rows  rope_kv_kernel + attn_mma_kernel unless NS_ATTN_SCALAR is set
//   hd 64 / 128, otherwise  rope_kv_kernel + attn_fast_kernel
//   hd 96                   attn_decode_kernel for one row, rope_kv_kernel + attn_mma_kernel for more (fp16 cache only)
//   any other (even) hd     rope_kv_kernel + attn_kernel
// A Q8_0 cache takes the split decode attention for one row and rope_kv_kernel + attn_mma_kernel for more, at head sizes 64 / 128;
// attn_fast_kernel and attn_kernel have no Q8_0 form.
// Each kernel has one launch function below; attn_dispatch turns (hd, cache format) into the template arguments they take.

static size_t attn_generic_smem(int hd, int n_ctx) { return (size_t)(hd + n_ctx) * sizeof(float); }
extern size_t attn_rows_smem(int hd, int n_ctx) { return (size_t)((3 + kAW) * hd + n_ctx) * sizeof(float); }
extern int attn_ranges(int n_ctx) { return (n_ctx + kSplitKeys - 1) / kSplitKeys; }

// the kernel `kind` resolves to for this shape and cache format, or NS_E_UNSUPPORTED when a forced kernel cannot take it
static int attn_resolve(int kind, int hd, int m, int n_ctx, int kv) {
  const bool all = attn_all_hd(hd), fast = attn_fast_hd(hd);
  const bool q8 = kv == NS_KV_Q8_0 && kind >= NS_ATTN_AUTO && kind <= NS_ATTN_GENERIC;
  if (q8 && !all) {
    ns_set_error("ns_llama: the Q8_0 KV cache needs head size 64 or 128, got %d", hd);
    return NS_E_UNSUPPORTED;
  }
  if (kind == NS_ATTN_AUTO) {
    // debugging aids, read per call (not per process) so that a test can compare kernels on one engine
    const bool old_decode = getenv("NS_ATTN_OLD_DECODE") != nullptr;  // decode attention: one CTA per head, dependent row loads
    const bool scalar_attn = getenv("NS_ATTN_SCALAR") != nullptr;    // prompt attention: one CTA per (head, token), no tensor cores
    if (q8 && (old_decode || scalar_attn)) {
      ns_set_error("ns_llama: NS_ATTN_OLD_DECODE / NS_ATTN_SCALAR select kernels without a Q8_0 KV form");
      return NS_E_UNSUPPORTED;
    }
    if (!fast) kind = NS_ATTN_GENERIC;
    else if (q8 || !all) kind = m == 1 ? NS_ATTN_SPLIT_DECODE : NS_ATTN_MMA;  // the two kernels with a Q8_0 form and a head size 96 form
    else if (m == 1) kind = attn_ranges(n_ctx) <= 1024 && !old_decode ? NS_ATTN_SPLIT_DECODE : NS_ATTN_ROWS;
    else kind = m >= 8 && !scalar_attn ? NS_ATTN_MMA : NS_ATTN_ROWS;
  }
  if (q8 && (kind == NS_ATTN_ROWS || kind == NS_ATTN_GENERIC)) {
    ns_set_error("ns_llama: attention kernel %d has no Q8_0 KV form (NS_ATTN_SPLIT_DECODE / NS_ATTN_MMA read Q8_0)", kind);
    return NS_E_UNSUPPORTED;
  }
  if ((q8 || (fast && !all)) && kind == NS_ATTN_SPLIT_DECODE && attn_ranges(n_ctx) > 1024) {
    ns_set_error("ns_llama: n_ctx %d too large for the split decode attention %s", n_ctx, q8 ? "over a Q8_0 KV cache" : "at head size 96");
    return NS_E_UNSUPPORTED;
  }
  if (kind < NS_ATTN_SPLIT_DECODE || kind > NS_ATTN_GENERIC) {
    ns_set_error("ns_llama: unknown attention kernel %d", kind);
    return NS_E_INVALID;
  }
  if (kind != NS_ATTN_GENERIC && !(kind == NS_ATTN_ROWS ? all : fast)) {
    ns_set_error("ns_llama: attention kernel %d needs head size %s, got %d", kind, kind == NS_ATTN_ROWS ? "64 or 128" : "64, 96 or 128", hd);
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
extern ShiftTable shift_table(int hd, float freq_base) {
  ShiftTable t{};
  const float theta_scale = std::pow(freq_base, -2.0f / hd);
  float theta = -1.0f;
  for (int i = 0; i < hd / 2; ++i) {
    t.cs[i] = __halves2half2(__float2half_rn(std::cos(theta)), __float2half_rn(std::sin(theta)));
    theta *= theta_scale;
  }
  return t;
}

// Runs f(HD, KV) with the head size and the cache format as compile-time constants (std::integral_constant): HD 64 or 128 with
// either cache format, the sizes every fast kernel is instantiated at, or 96 with an fp16 cache, where attn_decode_kernel and
// attn_mma_kernel are (f tests attn_all_hd(HD) before it names another kernel); `what` names the caller for any other pair.
template <class F>
static int attn_dispatch(const char* what, int hd, int kv, F&& f) {
  using F16 = std::integral_constant<int, NS_KV_F16>;
  using Q8 = std::integral_constant<int, NS_KV_Q8_0>;
  const auto at = [&](auto HD) { return kv == NS_KV_Q8_0 ? f(HD, Q8{}) : f(HD, F16{}); };
  if (hd == 128) return at(std::integral_constant<int, 128>{});
  if (hd == 64) return at(std::integral_constant<int, 64>{});
  if (hd == 96 && kv == NS_KV_F16) return f(std::integral_constant<int, 96>{}, F16{});
  ns_set_error("ns_llama: %s needs head size 64 or 128 (or 96 with an fp16 KV cache), got %d", what, hd);
  return NS_E_UNSUPPORTED;
}

// The launch constants of one layer's attention
struct AttnShape {
  int n_head, n_head_kv, hd, n_ctx, ldq, ldk, nsplit;
  float theta_scale, freq_scale, attn_scale;
};
static AttnShape attn_shape(int n_head, int n_head_kv, int hd, int n_ctx, float rope_theta, float rope_scale) {
  return AttnShape{n_head, n_head_kv, hd, n_ctx, n_head * hd, n_head_kv * hd, attn_ranges(n_ctx),
                   powf(rope_theta, -2.0f / (float)hd),  // n_rot == head_size (llama.cpp:131)
                   1.f / rope_scale,                     // the angle is divided by hparams.freq_scale (ne_layers.c:9263, 9207)
                   1.0f / sqrtf((float)hd)};
}

// Gives `kern` `smem` bytes of dynamic shared memory, once per context
template <class K>
static int grant_smem(AttnAttr& attr, K kern, size_t smem) {
  if (smem <= 48 * 1024) return NS_OK;
  const void* f = reinterpret_cast<const void*>(kern);
  int i = 0;
  while (i < attr.n && attr.granted[i].kern != f) ++i;
  if (i < attr.n && attr.granted[i].smem >= smem) return NS_OK;
  NS_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  if (i == attr.n) ++attr.n;
  attr.granted[i] = {f, smem};
  return NS_OK;
}

// RoPE + KV append of n_rows rows at positions state[1] + t, or (RAGGED) at the positions and blocks of rows[n_rows][2]
template <bool RAGGED, int KV>
static int launch_rope_kv(const AttnShape& s, float* q, const float* k, const float* v, const KvPtrs& kv, const int* state,
                          const int* rows, int n_rows, cudaStream_t st) {
  using T = kv_elem_t<KV>;
  NS_CUDA_TRY(ns_launch_pdl(rope_kv_kernel<RAGGED, KV>, dim3((unsigned)(s.n_head + s.n_head_kv), (unsigned)n_rows), dim3((unsigned)(s.hd / 2)),
                            0, st, q, s.ldq, k, s.ldk, v, s.ldk, static_cast<T*>(kv.k), static_cast<T*>(kv.v), state, s.n_head, s.n_head_kv,
                            s.hd, s.n_ctx, s.theta_scale, s.freq_scale, rows, kv.kd, kv.vd));
  ns_count_launch();
  return NS_OK;
}

// rope + KV append + attention of one new row in one launch, K / V staged by TMA, the context split over CTAs: one sequence, its
// ring form (one CTA per (kv head, range), n_keep sink slots, the shift table) or (BATCH) n_rows sequences
template <int HD, bool RING, bool BATCH, int KV>
static int launch_decode(const AttnShape& s, const float* q, const float* k, const float* v, const KvPtrs& kv, const int* state,
                         const int* seqs, float* out, float* part, unsigned* tickets, int n_rows, int n_keep, const ShiftTable& tab,
                         AttnAttr& attr, cudaStream_t st) {
  constexpr size_t smem = attn_decode_smem<HD>();
  if (int rc = grant_smem(attr, attn_decode_kernel<HD, RING, BATCH, KV>, smem)) return rc;
  // the eager pass before a capture runs this form where a streaming context's graph runs the ring form
  if constexpr (!RING && !BATCH && KV == NS_KV_F16 && attn_all_hd(HD))
    if (int rc = grant_smem(attr, attn_decode_kernel<HD, true>, smem)) return rc;
  using T = kv_elem_t<KV>;
  const dim3 grid((unsigned)(RING ? s.n_head_kv : s.n_head), (unsigned)s.nsplit, (unsigned)n_rows);
  NS_CUDA_TRY(ns_launch_pdl(attn_decode_kernel<HD, RING, BATCH, KV>, grid, dim3(kDW * 32), smem, st, q, k, v, static_cast<T*>(kv.k),
                            static_cast<T*>(kv.v), state, out, part, tickets, s.n_head, s.n_head_kv, s.n_ctx, s.nsplit, s.attn_scale,
                            s.theta_scale, s.freq_scale, n_keep, tab, seqs, kv.kd, kv.vd));
  ns_count_launch();
  return NS_OK;
}

// causal attention on the tensor cores, 64 query rows per CTA: grid_x tiles of m rows, or (RAGGED) of the tile table `tiles`
template <int HD, bool RAGGED, int KV>
static int launch_mma(const AttnShape& s, const float* q, const KvPtrs& kv, const int* state, const int* tiles, float* out, int m,
                      int grid_x, cudaStream_t st) {
  using T = kv_elem_t<KV>;
  NS_CUDA_TRY(ns_launch_pdl(attn_mma_kernel<HD, RAGGED, KV>, dim3((unsigned)grid_x, (unsigned)s.n_head), dim3(128), 0, st, q, s.ldq,
                            static_cast<const T*>(kv.k), static_cast<const T*>(kv.v), state, out, s.ldq, s.n_head, s.n_head_kv, s.n_ctx,
                            m, s.attn_scale, tiles, (const __half*)kv.kd, (const __half*)kv.vd));
  ns_count_launch();
  return NS_OK;
}

// one CTA per (head, row) with dependent row loads; FUSE (one row) also rotates and appends, as launch_decode
template <int HD, bool FUSE>
static int launch_fast(const AttnShape& s, const float* q, const float* k, const float* v, const KvPtrs& kv, const int* state,
                       float* out, int m, AttnAttr& attr, cudaStream_t st) {
  const size_t smem = attn_rows_smem(s.hd, s.n_ctx);
  if (int rc = grant_smem(attr, attn_fast_kernel<HD, FUSE>, smem)) return rc;
  NS_CUDA_TRY(ns_launch_pdl(attn_fast_kernel<HD, FUSE>, dim3((unsigned)s.n_head, (unsigned)m), dim3(kAW * 32), smem, st, q, s.ldq, k,
                            s.ldk, v, s.ldk, static_cast<__half*>(kv.k), static_cast<__half*>(kv.v), state, out, s.ldq, s.n_head,
                            s.n_head_kv, s.n_ctx, s.attn_scale, s.theta_scale, s.freq_scale));
  ns_count_launch();
  return NS_OK;
}

// one CTA per (head, row) at any even head size
static int launch_generic(const AttnShape& s, const float* q, const KvPtrs& kv, const int* state, float* out, int m, AttnAttr& attr,
                          cudaStream_t st) {
  const size_t smem = attn_generic_smem(s.hd, s.n_ctx);
  if (int rc = grant_smem(attr, attn_kernel, smem)) return rc;
  NS_CUDA_TRY(ns_launch_pdl(attn_kernel, dim3((unsigned)s.n_head, (unsigned)m), dim3(kAttnThreads), smem, st, q, s.ldq,
                            static_cast<const __half*>(kv.k), static_cast<const __half*>(kv.v), state, out, s.ldq, s.n_head, s.n_head_kv,
                            s.hd, s.n_ctx, s.attn_scale));
  ns_count_launch();
  return NS_OK;
}

extern int launch_attention_batch(const float* q, const float* k, const float* v, const KvPtrs& kv, const int* rstate,
                                  const int* seqs, float* out, float* part, unsigned* tickets, int n, int n_head, int n_head_kv, int hd,
                                  int n_ctx, float rope_theta, float rope_scale, AttnAttr& attr, cudaStream_t st) {
  const AttnShape s = attn_shape(n_head, n_head_kv, hd, n_ctx, rope_theta, rope_scale);
  return attn_dispatch("the batched decode attention", hd, kv.type, [&](auto HD, auto KV) {
    return launch_decode<HD, false, true, KV>(s, q, k, v, kv, rstate, seqs, out, part, tickets, n, -1, ShiftTable{}, attr, st);
  });
}

extern int launch_attention(int kind, float* q, const float* k, const float* v, const KvPtrs& kv, const int* state, float* out,
                            float* part, unsigned* tickets, int n_head, int n_head_kv, int hd, int n_ctx, int m, float rope_theta,
                            float rope_scale, AttnAttr& attr, cudaStream_t st, const Ring* ring = nullptr) {
  if (ring && kv.type != NS_KV_F16) {
    ns_set_error("ns_llama: the streaming ring shifts an fp16 KV cache only");
    return NS_E_UNSUPPORTED;
  }
  if (ring && !attn_all_hd(hd)) {
    ns_set_error("ns_llama: the streaming ring needs head size 64 or 128, got %d", hd);
    return NS_E_UNSUPPORTED;
  }
  if (ring && m == 1) kind = NS_ATTN_SPLIT_DECODE;  // the only kernel that carries the shift
  kind = attn_resolve(kind, hd, m, n_ctx, kv.type);
  if (kind < 0) return kind;
  const AttnShape s = attn_shape(n_head, n_head_kv, hd, n_ctx, rope_theta, rope_scale);
  if (kind == NS_ATTN_GENERIC) {  // any even head size, fp16 cache (attn_resolve)
    if (int rc = launch_rope_kv<false, NS_KV_F16>(s, q, k, v, kv, state, nullptr, m, st)) return rc;
    return launch_generic(s, q, kv, state, out, m, attr, st);
  }
  return attn_dispatch("attention kernel", hd, kv.type, [&](auto HD, auto KV) {  // attn_resolve left NS_ATTN_SPLIT_DECODE / MMA for Q8_0
    constexpr bool f16 = KV == NS_KV_F16, rows = f16 && attn_all_hd(HD);  // rows: the ring and attn_fast_kernel exist
    if (kind == NS_ATTN_SPLIT_DECODE) {
      if constexpr (rows)
        if (ring) return launch_decode<HD, true, false, KV>(s, q, k, v, kv, state, nullptr, out, part, tickets, 1, ring->n_keep, ring->tab, attr, st);
      return launch_decode<HD, false, false, KV>(s, q, k, v, kv, state, nullptr, out, part, tickets, 1, -1, ShiftTable{}, attr, st);
    }
    if constexpr (rows)
      if (kind == NS_ATTN_ROWS && m == 1) return launch_fast<HD, true>(s, q, k, v, kv, state, out, 1, attr, st);
    if (int rc = launch_rope_kv<false, KV>(s, q, k, v, kv, state, nullptr, m, st)) return rc;
    if constexpr (rows)
      if (kind == NS_ATTN_ROWS) return launch_fast<HD, false>(s, q, k, v, kv, state, out, m, attr, st);
    return launch_mma<HD, false, KV>(s, q, kv, state, nullptr, out, m, (m + kAttnMmaRows - 1) / kAttnMmaRows, st);
  });
}

// Workspace of ns_llama_attention: int state[4] (state[1] = n_past) | unsigned tickets[n_head], padded to 16 bytes |
// float partials[n_head][ceil(n_ctx / 256)][hd + 2]
static size_t attn_ws_tickets_offset() { return 4 * sizeof(int); }
static size_t attn_ws_part_offset(int n_head) { return attn_ws_tickets_offset() + ((size_t)n_head * sizeof(unsigned) + 15) / 16 * 16; }

extern "C" size_t ns_llama_attention_workspace_bytes(int n_head, int hd, int n_ctx) {
  if (n_head <= 0 || hd <= 0 || n_ctx <= 0) return 0;
  return attn_ws_part_offset(n_head) + (size_t)n_head * attn_ranges(n_ctx) * (hd + 2) * sizeof(float);
}

// the arguments every parity entry takes: pointers, the planes of the cache format, head counts, an even head size, the rope parameters
static bool attn_args_ok(const float* q, const float* k, const float* v, const KvPtrs& kv, const float* out, const void* ws, int n_head,
                         int n_head_kv, int hd, int n_ctx, float rope_theta, float rope_scale) {
  return q && k && v && kv.k && kv.v && (kv.type != NS_KV_Q8_0 || (kv.kd && kv.vd)) && out && ws && n_head > 0 && n_head_kv > 0 &&
         n_head % n_head_kv == 0 && hd > 0 && hd % 2 == 0 && n_ctx > 0 && rope_theta > 0.f && rope_scale > 0.f;
}

static int attention_entry(const char* who, int kernel, float* q, const float* k, const float* v, const KvPtrs& kv, int n_head,
                           int n_head_kv, int hd, int n_ctx, int n_past, int m, float rope_theta, float rope_scale, float* out, void* ws,
                           void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!attn_args_ok(q, k, v, kv, out, ws, n_head, n_head_kv, hd, n_ctx, rope_theta, rope_scale) || m <= 0 || n_past < 0 ||
      n_past + m > n_ctx) {
    ns_set_error("%s: invalid arguments (n_head=%d n_head_kv=%d hd=%d n_ctx=%d n_past=%d m=%d)", who, n_head, n_head_kv, hd, n_ctx, n_past, m);
    return NS_E_INVALID;
  }
  if (int rc = attn_resolve(kernel, hd, m, n_ctx, kv.type); rc < 0) return rc;
  cudaStream_t st = ns_stream_of(queue);
  char* w = static_cast<char*>(ws);
  const int state[4] = {0, n_past, 0, 0};
  NS_CUDA_TRY(cudaMemcpyAsync(w, state, sizeof(state), cudaMemcpyHostToDevice, st));  // pageable source: staged before the call returns
  AttnAttr attr;
  return launch_attention(kernel, q, k, v, kv, reinterpret_cast<const int*>(w), out, reinterpret_cast<float*>(w + attn_ws_part_offset(n_head)),
                          reinterpret_cast<unsigned*>(w + attn_ws_tickets_offset()), n_head, n_head_kv, hd, n_ctx, m, rope_theta,
                          rope_scale, attr, st);
}

static KvPtrs f16_planes(void* kc, void* vc) { return KvPtrs{NS_KV_F16, kc, vc}; }
static KvPtrs q8_planes(void* kq, void* kd, void* vq, void* vd) {
  return KvPtrs{NS_KV_Q8_0, kq, vq, static_cast<__half*>(kd), static_cast<__half*>(vd)};
}

extern "C" int ns_llama_attention(int kernel, float* q, const float* k, const float* v, void* kc, void* vc, int n_head, int n_head_kv,
                                  int hd, int n_ctx, int n_past, int m, float rope_theta, float rope_scale, float* out, void* ws,
                                  void* queue) {
  return attention_entry("ns_llama_attention", kernel, q, k, v, f16_planes(kc, vc), n_head, n_head_kv, hd, n_ctx, n_past, m, rope_theta,
                         rope_scale, out, ws, queue);
}

extern "C" int ns_llama_attention_q8_0(int kernel, float* q, const float* k, const float* v, void* kq, void* kd, void* vq, void* vd,
                                       int n_head, int n_head_kv, int hd, int n_ctx, int n_past, int m, float rope_theta, float rope_scale,
                                       float* out, void* ws, void* queue) {
  return attention_entry("ns_llama_attention_q8_0", kernel, q, k, v, q8_planes(kq, kd, vq, vd), n_head, n_head_kv, hd, n_ctx, n_past, m,
                         rope_theta, rope_scale, out, ws, queue);
}

extern "C" int ns_llama_attention_ring(float* q, const float* k, const float* v, void* kc, void* vc, int n_head, int n_head_kv, int hd,
                                       int n_ctx, int n_keep, int n_total, float rope_theta, float* out, void* ws, void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  const KvPtrs kv = f16_planes(kc, vc);
  if (!attn_args_ok(q, k, v, kv, out, ws, n_head, n_head_kv, hd, n_ctx, rope_theta, 1.f) || n_keep < 0 || n_keep >= n_ctx || n_total < 0) {
    ns_set_error("ns_llama_attention_ring: invalid arguments (n_head=%d n_head_kv=%d hd=%d n_ctx=%d n_keep=%d n_total=%d)", n_head,
                 n_head_kv, hd, n_ctx, n_keep, n_total);
    return NS_E_INVALID;
  }
  if (int rc = attn_resolve(NS_ATTN_SPLIT_DECODE, hd, 1, n_ctx, NS_KV_F16); rc < 0) return rc;
  cudaStream_t st = ns_stream_of(queue);
  char* w = static_cast<char*>(ws);
  const int state[4] = {0, n_total, 0, 0};
  NS_CUDA_TRY(cudaMemcpyAsync(w, state, sizeof(state), cudaMemcpyHostToDevice, st));  // pageable source: staged before the call returns
  AttnAttr attr;
  const Ring ring{n_keep, shift_table(hd, rope_theta)};
  return launch_attention(NS_ATTN_SPLIT_DECODE, q, k, v, kv, reinterpret_cast<const int*>(w), out, reinterpret_cast<float*>(w + attn_ws_part_offset(n_head)),
                          reinterpret_cast<unsigned*>(w + attn_ws_tickets_offset()), n_head, n_head_kv, hd, n_ctx, 1, rope_theta, 1.f, attr,
                          st, &ring);
}

extern int check_rows(const char* who, int n_seq, int n, const int* seq, const int* n_past, int steps, int n_ctx) {
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

static int attention_batch_entry(const char* who, float* q, const float* k, const float* v, const KvPtrs& kv, int n_seq, int n,
                                 const int* seq, const int* n_past, int n_head, int n_head_kv, int hd, int n_ctx, float rope_theta,
                                 float rope_scale, float* out, void* ws, void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!attn_args_ok(q, k, v, kv, out, ws, n_head, n_head_kv, hd, n_ctx, rope_theta, rope_scale) || !seq || !n_past || n_seq < 1 ||
      n_seq > 32) {
    ns_set_error("%s: invalid arguments (n_seq=%d n=%d n_head=%d n_head_kv=%d hd=%d n_ctx=%d)", who, n_seq, n, n_head, n_head_kv, hd, n_ctx);
    return NS_E_INVALID;
  }
  if (int rc = check_rows(who, n_seq, n, seq, n_past, 1, n_ctx)) return rc;
  if (!attn_fast_hd(hd)) {
    ns_set_error("%s: head size %d (the batched decode attention takes 64, 96 or 128)", who, hd);
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
  return launch_attention_batch(q, k, v, kv, reinterpret_cast<const int*>(w), reinterpret_cast<const int*>(w + attnb_ws_seq_offset(n)), out,
                                reinterpret_cast<float*>(w + attnb_ws_part_offset(n, n_head)),
                                reinterpret_cast<unsigned*>(w + attnb_ws_tickets_offset(n)), n, n_head, n_head_kv, hd, n_ctx, rope_theta,
                                rope_scale, attr, st);
}

extern "C" int ns_llama_attention_batch(float* q, const float* k, const float* v, void* kc, void* vc, int n_seq, int n, const int* seq,
                                        const int* n_past, int n_head, int n_head_kv, int hd, int n_ctx, float rope_theta,
                                        float rope_scale, float* out, void* ws, void* queue) {
  return attention_batch_entry("ns_llama_attention_batch", q, k, v, f16_planes(kc, vc), n_seq, n, seq, n_past, n_head, n_head_kv, hd, n_ctx,
                               rope_theta, rope_scale, out, ws, queue);
}

extern "C" int ns_llama_attention_batch_q8_0(float* q, const float* k, const float* v, void* kq, void* kd, void* vq, void* vd, int n_seq,
                                             int n, const int* seq, const int* n_past, int n_head, int n_head_kv, int hd, int n_ctx,
                                             float rope_theta, float rope_scale, float* out, void* ws, void* queue) {
  return attention_batch_entry("ns_llama_attention_batch_q8_0", q, k, v, q8_planes(kq, kd, vq, vd), n_seq, n, seq, n_past, n_head, n_head_kv,
                               hd, n_ctx, rope_theta, rope_scale, out, ws, queue);
}

// ---- mixed batches: token segments of several sequences in one pass (ns_llama_eval_batch) ------------------------------------

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


extern int plan_batch(const char* who, int n_seq, int n_ctx, int n, const int* seq, const int* n_tokens, const int* n_past, BatchPlan& p) {
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

extern int launch_attention_ragged(float* q, const float* k, const float* v, const KvPtrs& kv, const int* rows, const int* tiles,
                                   int n_rows, int n_tiles, float* out, int n_head, int n_head_kv, int hd, int n_ctx, float rope_theta,
                                   float rope_scale, cudaStream_t st) {
  const AttnShape s = attn_shape(n_head, n_head_kv, hd, n_ctx, rope_theta, rope_scale);
  return attn_dispatch("the ragged prompt attention", hd, kv.type, [&](auto HD, auto KV) {
    if (int rc = launch_rope_kv<true, KV>(s, q, k, v, kv, nullptr, rows, n_rows, st)) return rc;
    return launch_mma<HD, true, KV>(s, q, kv, nullptr, tiles, out, 0, n_tiles, st);
  });
}

// Workspace of ns_llama_attention_ragged: int rows[n_rows][2] | int tiles[n_rows / 64 + n][5]
extern "C" size_t ns_llama_attention_ragged_workspace_bytes(int n, int n_rows) {
  if (n <= 0 || n_rows <= 0) return 0;
  return ((size_t)2 * n_rows + (size_t)(n_rows / kAttnMmaRows + n) * kTileInts) * sizeof(int);
}

static int attention_ragged_entry(const char* who, float* q, const float* k, const float* v, const KvPtrs& kv, int n_seq, int n,
                                  const int* seq, const int* n_tokens, const int* n_past, int n_head, int n_head_kv, int hd, int n_ctx,
                                  float rope_theta, float rope_scale, float* out, void* ws, void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!attn_args_ok(q, k, v, kv, out, ws, n_head, n_head_kv, hd, n_ctx, rope_theta, rope_scale) || n_seq < 1 || n_seq > 32) {
    ns_set_error("%s: invalid arguments (n_seq=%d n=%d n_head=%d n_head_kv=%d hd=%d n_ctx=%d)", who, n_seq, n, n_head, n_head_kv, hd, n_ctx);
    return NS_E_INVALID;
  }
  int n_rows = 0;
  if (int rc = check_segments(who, n_seq, n_ctx, n, seq, n_tokens, n_past, &n_rows)) return rc;
  if (!attn_fast_hd(hd)) {
    ns_set_error("%s: head size %d (the ragged prompt attention takes 64, 96 or 128)", who, hd);
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
  return launch_attention_ragged(q, k, v, kv, reinterpret_cast<const int*>(w), reinterpret_cast<const int*>(w + (size_t)2 * n_rows * sizeof(int)),
                                 n_rows, (int)tiles.size() / kTileInts, out, n_head, n_head_kv, hd, n_ctx, rope_theta, rope_scale, st);
}

extern "C" int ns_llama_attention_ragged(float* q, const float* k, const float* v, void* kc, void* vc, int n_seq, int n, const int* seq,
                                         const int* n_tokens, const int* n_past, int n_head, int n_head_kv, int hd, int n_ctx,
                                         float rope_theta, float rope_scale, float* out, void* ws, void* queue) {
  return attention_ragged_entry("ns_llama_attention_ragged", q, k, v, f16_planes(kc, vc), n_seq, n, seq, n_tokens, n_past, n_head, n_head_kv,
                                hd, n_ctx, rope_theta, rope_scale, out, ws, queue);
}

extern "C" int ns_llama_attention_ragged_q8_0(float* q, const float* k, const float* v, void* kq, void* kd, void* vq, void* vd, int n_seq,
                                              int n, const int* seq, const int* n_tokens, const int* n_past, int n_head, int n_head_kv,
                                              int hd, int n_ctx, float rope_theta, float rope_scale, float* out, void* ws, void* queue) {
  return attention_ragged_entry("ns_llama_attention_ragged_q8_0", q, k, v, q8_planes(kq, kd, vq, vd), n_seq, n, seq, n_tokens, n_past,
                                n_head, n_head_kv, hd, n_ctx, rope_theta, rope_scale, out, ws, queue);
}

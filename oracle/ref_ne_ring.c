/*
 * oracle/ref_ne_ring.c -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * The reference's graph engine as oracle/ref_ne.c builds it (core/ne_layers.c compiled where it lies, BesTLA entry points
 * stubbed), plus the graphs of the shift-RoPE-K ("StreamingLLM") mode, driven through the public ne_* API:
 *   ref_ne_rope_shift       ne_rope_shift_inplace on an fp16 K tensor (ne_layers.c:9495-9532)
 *   ref_ne_llama_eval_ring  the Llama eval graph of ref_ne_llama_eval with the ring of models/llama/llama.cpp:102-107, 351-354,
 *                           430-470: q / k positions, the K shift after the KV write, no mask for one new token
 * Built by Makefile.ring into oracle/_ref/libref_ne_ring.so; oracle/streaming.py loads it.
 */
#include "ref_ne.c"

/* The fp16 K shift as the engine builds it does not run: ne_rope_impl gives the node 5 + ne[3] integer parameters (ne_layers.c:3403,
 * n_past .. n_keep and one padding entry per batch row) while ne_compute_forward_rope_f16 asserts exactly 5 (:9437) and aborts.
 * The harness hands the node a view of the first 5 -- all the fp16 kernel reads -- which leaves its arithmetic as written. */
static struct ne_tensor* ref_ne_rope_shift_f16(struct ne_context* ctx, struct ne_tensor* a, int n_shift, int n_dims, int n_keep,
                                               struct ne_tensor* cossin, float freq_base, float freq_scale) {
  struct ne_tensor* r = ne_rope_shift_inplace(ctx, a, n_shift, n_dims, 0, 0, n_keep, cossin, freq_base, freq_scale);
  r->src1 = ne_view_1d(ctx, r->src1, 5, 0);
  return r;
}

/* k: [n_seq][n_head][hd] fp16, every row of seq index >= n_keep shifted one position back in place (the K shift of llama.cpp:443
 * with N = 1); cossin: [hd] fp16 table (cos, sin per pair) or NULL, in which case the op builds its own from freq_base / freq_scale */
REF_API void ref_ne_rope_shift(uint16_t* k, int hd, int n_head, int n_seq, int n_keep, const uint16_t* cossin, float freq_base,
                               float freq_scale) {
  struct ne_context* ctx = ref_ne_ctx((size_t)hd * n_head * n_seq * 4 + (16u << 20));
  struct ne_tensor* t = ne_new_tensor_4d(ctx, NE_TYPE_F16, hd, n_head, n_seq, 1, NE_SIZE_CALC, NE_BACKEND_CPU);
  memcpy(t->data, k, (size_t)hd * n_head * n_seq * 2);
  struct ne_tensor* cs = NULL;
  if (cossin) {
    cs = ne_new_tensor_1d(ctx, NE_TYPE_F16, hd, NE_SIZE_CALC, NE_BACKEND_CPU);
    memcpy(cs->data, cossin, (size_t)hd * 2);
  }
  struct ne_tensor* r = ref_ne_rope_shift_f16(ctx, t, -1, hd, n_keep, cs, freq_base, freq_scale);
  ref_ne_run(ctx, r);
  memcpy(k, t->data, (size_t)hd * n_head * n_seq * 2);
  ne_free(ctx);
}

/* ref_ne_llama_eval's graph (Q4_0 weights, the ggml attention path) in shift-RoPE-K mode with n_keep sink slots.  n_past and
 * n_total are those of application/main_run.cpp:474-494: n_past is the cache slot the new tokens go to, n_total the number of
 * tokens evaluated so far; cossin: kv_self.cossin ([hd] fp16) or NULL (the op builds its own table). */
REF_API void ref_ne_llama_eval_ring(ref_ne_llama* m, const int* tokens, int N, int n_past, int n_total, int n_keep,
                                    const uint16_t* cossin, float* logits_last) {
  const int n_embd = m->n_embd, n_head = m->n_head, n_head_kv = m->n_head_kv, hd = n_embd / n_head, n_ctx = m->n_ctx, n_ff = m->n_ff;
  const int kvd = hd * n_head_kv;
  struct ne_context* ctx0 = ref_ne_ctx((size_t)N * ((size_t)n_embd * 64 + (size_t)n_ff * 16 + (size_t)n_ctx * n_head * 16) * m->n_layer +
                                       (size_t)m->n_vocab * 8 + (256u << 20));
  struct ne_cgraph gf;
  memset(&gf, 0, sizeof(gf));
  gf.n_threads = m->n_threads;
  struct ne_tensor* embd = ne_new_tensor_1d(ctx0, NE_TYPE_I32, N, NE_SIZE_CALC, NE_BACKEND_CPU);
  memcpy(embd->data, tokens, (size_t)N * 4);
  struct ne_tensor* inpL = ne_get_rows(ctx0, m->tok, embd);
  const float attn_scale = 1.0f / sqrtf((float)hd);
  const size_t e16 = sizeof(ne_fp16_t);
  const int ring_full = n_total > n_past;                                         /* llama.cpp:106 */
  const int n_cached = n_total + N < n_ctx ? n_total + N : n_ctx;                 /* :107 */
  const int q_pos = n_cached - N > n_past ? n_cached - N : n_past;                /* :351 */
  for (int il = 0; il < m->n_layer; ++il) {
    struct ne_tensor** w = m->lw + il * 9;
    struct ne_tensor* inpSA = inpL;
    struct ne_tensor* cur = ne_rms_norm(ctx0, inpL, m->eps);
    cur = ne_mul(ctx0, cur, w[0]);
    struct ne_tensor* Qcur = ne_reshape_3d(ctx0, ne_mul_mat(ctx0, w[1], cur), hd, n_head, N);
    struct ne_tensor* Kcur = ne_reshape_3d(ctx0, ne_mul_mat(ctx0, w[2], cur), hd, n_head_kv, N);
    struct ne_tensor* Vcur = ne_mul_mat(ctx0, w[3], cur);
    Qcur = ne_rope_inplace(ctx0, Qcur, q_pos, hd, 0, 0, m->freq_base, m->freq_scale);
    Kcur = ne_rope_inplace(ctx0, Kcur, ring_full ? n_ctx : n_past, hd, 0, 0, m->freq_base, m->freq_scale); /* :353-354 */
    /* store key and value to the cache (llama.cpp:362-412) */
    struct ne_tensor* k_cache = ne_view_1d(ctx0, m->kc, (int64_t)n_ctx * kvd, (size_t)il * n_ctx * e16 * kvd);
    struct ne_tensor* v_cache = ne_view_1d(ctx0, m->vc, (int64_t)n_ctx * kvd, (size_t)il * n_ctx * e16 * kvd);
    struct ne_tensor* k_dst = ne_view_3d(ctx0, k_cache, hd, N, n_head_kv, e16 * hd, e16 * hd * n_ctx, (size_t)hd * n_past * e16);
    struct ne_tensor* v_dst = ne_view_3d(ctx0, v_cache, N, hd, n_head_kv, (size_t)n_ctx * e16, (size_t)n_ctx * e16 * hd, (size_t)n_past * e16);
    ne_build_forward_expand(&gf, ne_cpy(ctx0, ne_permute(ctx0, Kcur, 0, 2, 1, 3), k_dst));
    ne_build_forward_expand(&gf, ne_cpy(ctx0, ne_permute(ctx0, ne_reshape_3d(ctx0, Vcur, hd, n_head_kv, N), 1, 2, 0, 3), v_dst));
    struct ne_tensor* Q = ne_permute(ctx0, Qcur, 0, 2, 1, 3);
    struct ne_tensor* K = ne_view_3d(ctx0, k_cache, hd, n_cached, n_head_kv, e16 * hd, e16 * hd * n_ctx, 0);
    if (ring_full) { /* llama.cpp:437-446: every cached key at or past n_keep one position back, after the write above */
      struct ne_tensor* cs = NULL;
      if (cossin && N == 1) {
        cs = ne_new_tensor_1d(ctx0, NE_TYPE_F16, hd, NE_SIZE_CALC, NE_BACKEND_CPU);
        memcpy(cs->data, cossin, (size_t)hd * e16);
      }
      K = ne_permute(ctx0, K, 0, 2, 1, 3);
      K = ref_ne_rope_shift_f16(ctx0, K, -N, hd, n_keep, cs, m->freq_base, m->freq_scale);
      K = ne_permute(ctx0, K, 0, 2, 1, 3);
    }
    struct ne_tensor* KQ = ne_mul_mat(ctx0, K, Q);
    struct ne_tensor* KQ_scaled = ne_scale_inplace(ctx0, KQ, ne_new_f32(ctx0, attn_scale));
    if (N > 1 || n_total == 0) KQ_scaled = ne_diag_mask_inf_inplace(ctx0, KQ_scaled, n_past); /* :467 */
    struct ne_tensor* KQ_soft_max = ne_soft_max_inplace(ctx0, KQ_scaled);
    struct ne_tensor* V = ne_view_3d(ctx0, v_cache, n_cached, hd, n_head_kv, (size_t)n_ctx * e16, (size_t)n_ctx * e16 * hd, 0);
    struct ne_tensor* KQV = ne_mul_mat(ctx0, V, KQ_soft_max);
    struct ne_tensor* KQV_merged = ne_permute(ctx0, KQV, 0, 2, 1, 3);
    cur = ne_cpy(ctx0, KQV_merged, ne_new_tensor_2d(ctx0, NE_TYPE_F32, n_embd, N, NE_SIZE_CALC, NE_BACKEND_CPU));
    cur = ne_mul_mat(ctx0, w[4], cur);
    struct ne_tensor* inpFF = ne_add(ctx0, cur, inpSA);
    cur = ne_rms_norm(ctx0, inpFF, m->eps);
    cur = ne_mul(ctx0, cur, w[5]);
    struct ne_tensor* tmp = ne_mul_mat(ctx0, w[8], cur); /* ffn[2] = w3 (llama.cpp:615-620) */
    cur = ne_mul_mat(ctx0, w[6], cur);
    cur = ne_silu(ctx0, cur);
    cur = ne_mul(ctx0, cur, tmp);
    cur = ne_mul_mat(ctx0, w[7], cur);
    cur = ne_add(ctx0, cur, inpFF);
    inpL = cur;
  }
  inpL = ne_rms_norm(ctx0, inpL, m->eps);
  inpL = ne_mul(ctx0, inpL, m->out_norm);
  inpL = ne_mul_mat(ctx0, m->output, inpL);
  ne_build_forward_expand(&gf, inpL);
  ne_graph_compute(ctx0, &gf);
  memcpy(logits_last, (float*)inpL->data + (size_t)(N - 1) * m->n_vocab, (size_t)m->n_vocab * 4);
  ne_free(ctx0);
}

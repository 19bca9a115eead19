/*
 * oracle/ref_ne_qwen2.c -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * The reference's graph engine as oracle/ref_ne.c builds it (core/ne_layers.c compiled where it lies, BesTLA entry points
 * stubbed), plus the pieces of the qwen architecture's version-2 graph (models/qwen/qwen.cpp, Qwen1.5 / Qwen2 / Qwen2.5), driven
 * through the public ne_* API:
 *   ref_ne_rope_neox     ne_rope_inplace with mode 2: the NeoX rotation of the pairs (i, i + hd/2) (ne_layers.c:9396-9423)
 *   ref_ne_qwen2_*       the graph of qwen.cpp's version-2 branch on the Q4_0 model of ref_ne_llama_create: q / k / v biases added
 *                        with ne_add(ne_repeat(bias, cur), cur) after each projection (:193-203), mode-2 RoPE (:206-209), the
 *                        non-fused attention, qwen_ff's unfused FFN up * silu(gate) (:41-62)
 * Built by Makefile.qwen2 into oracle/_ref/libref_ne_qwen2.so; oracle/qwen2.py loads it.
 */
#include "ref_ne.c"

/* x: [n_tok][n_head][hd] fp32, rotated in place at positions n_past .. n_past + n_tok - 1 */
REF_API void ref_ne_rope_neox(float* x, int hd, int n_head, int n_tok, int n_past, float freq_base, float freq_scale) {
  struct ne_context* ctx = ref_ne_ctx((size_t)hd * n_head * n_tok * 8 + (16u << 20));
  struct ne_tensor* t = ne_new_tensor_4d(ctx, NE_TYPE_F32, hd, n_head, n_tok, 1, NE_SIZE_CALC, NE_BACKEND_CPU);
  memcpy(t->data, x, (size_t)hd * n_head * n_tok * 4);
  struct ne_tensor* r = ne_rope_inplace(ctx, t, n_past, hd, 2, 0, freq_base, freq_scale);
  ref_ne_run(ctx, r);
  memcpy(x, t->data, (size_t)hd * n_head * n_tok * 4);
  ne_free(ctx);
}

typedef struct ref_ne_qwen2 {
  ref_ne_llama* m;       /* weights, norms, embedding table and KV cache, set with ref_ne_llama_set */
  struct ne_tensor** lb; /* per layer: b_q, b_k, b_v */
} ref_ne_qwen2;

REF_API ref_ne_qwen2* ref_ne_qwen2_create(int n_vocab, int n_embd, int n_head, int n_head_kv, int n_layer, int n_ff, int n_ctx,
                                          float eps, float freq_base, float freq_scale) {
  ref_ne_qwen2* q = (ref_ne_qwen2*)calloc(1, sizeof(*q));
  q->m = ref_ne_llama_create(n_vocab, n_embd, n_head, n_head_kv, n_layer, n_ff, n_ctx, eps, freq_base, freq_scale);
  const int kvd = n_embd / n_head * n_head_kv;
  q->lb = (struct ne_tensor**)calloc((size_t)n_layer * 3, sizeof(struct ne_tensor*));
  for (int il = 0; il < n_layer; ++il)
    for (int j = 0; j < 3; ++j) q->lb[il * 3 + j] = ne_new_tensor_1d(q->m->wctx, NE_TYPE_F32, j ? kvd : n_embd, NE_SIZE_CALC, NE_BACKEND_CPU);
  return q;
}
/* which: as ref_ne_llama_set */
REF_API int ref_ne_qwen2_set(ref_ne_qwen2* q, int layer, int which, const void* data, size_t bytes) {
  return ref_ne_llama_set(q->m, layer, which, data, bytes);
}
/* which: 0 b_q, 1 b_k, 2 b_v (f32) */
REF_API int ref_ne_qwen2_set_bias(ref_ne_qwen2* q, int layer, int which, const float* data, size_t bytes) {
  if (which < 0 || which > 2 || layer < 0 || layer >= q->m->n_layer) return -1;
  struct ne_tensor* t = q->lb[layer * 3 + which];
  if (ne_nbytes(t) != bytes) return -1;
  memcpy(t->data, data, bytes);
  return 0;
}
REF_API void ref_ne_qwen2_free(ref_ne_qwen2* q) {
  ref_ne_llama_free(q->m);
  free(q->lb);
  free(q);
}

/* ref_ne_llama_eval's graph (ggml path, batch 1) with the version-2 qwen differences */
REF_API void ref_ne_qwen2_eval(ref_ne_qwen2* q, const int* tokens, int N, int n_past, float* logits_last) {
  ref_ne_llama* m = q->m;
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
  for (int il = 0; il < m->n_layer; ++il) {
    struct ne_tensor** w = m->lw + il * 9;
    struct ne_tensor** b = q->lb + il * 3;
    struct ne_tensor* cur = ne_rms_norm(ctx0, inpL, m->eps);
    cur = ne_mul(ctx0, cur, w[0]);
    struct ne_tensor* Qcur = ne_mul_mat(ctx0, w[1], cur);
    Qcur = ne_reshape_3d(ctx0, ne_add(ctx0, ne_repeat(ctx0, b[0], Qcur), Qcur), hd, n_head, N);
    struct ne_tensor* Kcur = ne_mul_mat(ctx0, w[2], cur);
    Kcur = ne_reshape_3d(ctx0, ne_add(ctx0, ne_repeat(ctx0, b[1], Kcur), Kcur), hd, n_head_kv, N);
    struct ne_tensor* Vcur = ne_mul_mat(ctx0, w[3], cur);
    Vcur = ne_add(ctx0, ne_repeat(ctx0, b[2], Vcur), Vcur);
    Qcur = ne_rope_inplace(ctx0, Qcur, n_past, hd, 2, 0, m->freq_base, m->freq_scale);
    Kcur = ne_rope_inplace(ctx0, Kcur, n_past, hd, 2, 0, m->freq_base, m->freq_scale);
    struct ne_tensor* k_cache = ne_view_1d(ctx0, m->kc, (int64_t)n_ctx * kvd, (size_t)il * n_ctx * e16 * kvd);
    struct ne_tensor* v_cache = ne_view_1d(ctx0, m->vc, (int64_t)n_ctx * kvd, (size_t)il * n_ctx * e16 * kvd);
    struct ne_tensor* k_dst = ne_view_3d(ctx0, k_cache, hd, N, n_head_kv, e16 * hd, e16 * hd * n_ctx, (size_t)hd * n_past * e16);
    struct ne_tensor* v_dst = ne_view_3d(ctx0, v_cache, N, hd, n_head_kv, (size_t)n_ctx * e16, (size_t)n_ctx * e16 * hd, (size_t)n_past * e16);
    ne_build_forward_expand(&gf, ne_cpy(ctx0, ne_permute(ctx0, Kcur, 0, 2, 1, 3), k_dst));
    ne_build_forward_expand(&gf, ne_cpy(ctx0, ne_permute(ctx0, ne_reshape_3d(ctx0, Vcur, hd, n_head_kv, N), 1, 2, 0, 3), v_dst));
    struct ne_tensor* Q = ne_permute(ctx0, Qcur, 0, 2, 1, 3);
    struct ne_tensor* K = ne_view_3d(ctx0, k_cache, hd, n_past + N, n_head_kv, e16 * hd, e16 * hd * n_ctx, 0);
    struct ne_tensor* KQ = ne_mul_mat(ctx0, K, Q);
    struct ne_tensor* KQ_scaled = ne_scale_inplace(ctx0, KQ, ne_new_f32(ctx0, attn_scale));
    struct ne_tensor* KQ_masked = ne_diag_mask_inf_inplace(ctx0, KQ_scaled, n_past);
    struct ne_tensor* KQ_soft_max = ne_soft_max_inplace(ctx0, KQ_masked);
    struct ne_tensor* V = ne_view_3d(ctx0, v_cache, n_past + N, hd, n_head_kv, (size_t)n_ctx * e16, (size_t)n_ctx * e16 * hd, 0);
    struct ne_tensor* KQV = ne_mul_mat(ctx0, V, KQ_soft_max);
    cur = ne_cpy(ctx0, ne_permute(ctx0, KQV, 0, 2, 1, 3), ne_new_tensor_2d(ctx0, NE_TYPE_F32, n_embd, N, NE_SIZE_CALC, NE_BACKEND_CPU));
    cur = ne_mul_mat(ctx0, w[4], cur);
    cur = ne_add(ctx0, cur, inpL); /* qwen.cpp: cur = ne_add(cur, inpL); inpL = cur */
    inpL = cur;
    cur = ne_rms_norm(ctx0, cur, m->eps);
    cur = ne_mul(ctx0, cur, w[5]);
    struct ne_tensor* up = ne_mul_mat(ctx0, w[8], cur);                /* qwen_ff: cur_1 = ffn[0] = up */
    struct ne_tensor* gate = ne_silu(ctx0, ne_mul_mat(ctx0, w[6], cur)); /* cur_2 = silu(ffn[1] = gate) */
    cur = ne_mul_mat(ctx0, w[7], ne_mul(ctx0, up, gate));
    inpL = ne_add(ctx0, cur, inpL);
  }
  inpL = ne_rms_norm(ctx0, inpL, m->eps);
  inpL = ne_mul(ctx0, inpL, m->out_norm);
  inpL = ne_mul_mat(ctx0, m->output, inpL);
  ne_build_forward_expand(&gf, inpL);
  ne_graph_compute(ctx0, &gf);
  memcpy(logits_last, (float*)inpL->data + (size_t)(N - 1) * m->n_vocab, (size_t)m->n_vocab * 4);
  ne_free(ctx0);
}

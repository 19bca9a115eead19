/*
 * oracle/ref_ne_harness.h -- TEST INFRASTRUCTURE ONLY.  Graphs driven through the reference engine's PUBLIC API (ne_init /
 * ne_new_tensor_* / ne_mul_mat / ne_mul_qkv / ne_ffn_silu / ne_graph_compute ...).  Included after "core/ne_layers.c" by
 *   ref_ne.c     the engine with the BesTLA entry points stubbed (every node takes ne_layers.c's own ggml path): the oracle pin
 */
/* ---- single ops through the public graph API ------------------------------------------------------------------------ */
static struct ne_context* ref_ne_ctx(size_t bytes) {
  struct ne_init_params ip = {bytes, NULL, false};
  return ne_init(ip);
}
static void ref_ne_run(struct ne_context* ctx, struct ne_tensor* t) {
  struct ne_cgraph gf = ne_build_forward(t);
  gf.n_threads = 1;
  ne_graph_compute(ctx, &gf);
}

/* x: [n_tok][n_head][hd] fp32, rotated in place at positions n_past .. n_past + n_tok - 1 (llama.cpp:351-355, mode 0) */
REF_API void ref_ne_rope(float* x, int hd, int n_head, int n_tok, int n_past, float freq_base, float freq_scale) {
  struct ne_context* ctx = ref_ne_ctx((size_t)hd * n_head * n_tok * 8 + (16u << 20));
  struct ne_tensor* t = ne_new_tensor_4d(ctx, NE_TYPE_F32, hd, n_head, n_tok, 1, NE_SIZE_CALC, NE_BACKEND_CPU);
  memcpy(t->data, x, (size_t)hd * n_head * n_tok * 4);
  struct ne_tensor* r = ne_rope_inplace(ctx, t, n_past, hd, 0, 0, freq_base, freq_scale);
  ref_ne_run(ctx, r);
  memcpy(x, t->data, (size_t)hd * n_head * n_tok * 4);
  ne_free(ctx);
}

/* rows x n, soft_max over n in place (ne_compute_forward_soft_max_f32, ne_layers.c:8887-8954) */
REF_API void ref_ne_soft_max(float* x, int n, int rows) {
  struct ne_context* ctx = ref_ne_ctx((size_t)n * rows * 8 + (16u << 20));
  struct ne_tensor* t = ne_new_tensor_2d(ctx, NE_TYPE_F32, n, rows, NE_SIZE_CALC, NE_BACKEND_CPU);
  memcpy(t->data, x, (size_t)n * rows * 4);
  struct ne_tensor* r = ne_soft_max_inplace(ctx, t);
  ref_ne_run(ctx, r);
  memcpy(x, t->data, (size_t)n * rows * 4);
  ne_free(ctx);
}

/* y = rms_norm(x) (no weight), rows x n (ne_rms_norm -> bestla_layernormalization, ne_layers.c:6588-6626) */
REF_API void ref_ne_rms_norm(const float* x, float* y, int n, int rows, float eps) {
  struct ne_context* ctx = ref_ne_ctx((size_t)n * rows * 12 + (16u << 20));
  struct ne_tensor* t = ne_new_tensor_2d(ctx, NE_TYPE_F32, n, rows, NE_SIZE_CALC, NE_BACKEND_CPU);
  memcpy(t->data, x, (size_t)n * rows * 4);
  struct ne_tensor* r = ne_rms_norm(ctx, t, eps);
  ref_ne_run(ctx, r);
  memcpy(y, r->data, (size_t)n * rows * 4);
  ne_free(ctx);
}

/* The ggml attention of llama.cpp:286-302 for ONE new token: q [n_head][hd] fp32 (already rotated), k cache [n_head][len][hd]
 * fp16, v cache [n_head][hd][len] fp16 (transposed, as the reference stores it), out [n_head][hd].
 * KQ = mul_mat(K, Q) -> scale -> soft_max -> KQV = mul_mat(V, KQ_soft_max). */
REF_API void ref_ne_attn_1tok(const float* q, const uint16_t* kc, const uint16_t* vc, float* out, int hd, int n_head, int len,
                              float scale) {
  struct ne_context* ctx = ref_ne_ctx((size_t)n_head * ((size_t)hd * len * 4 + (size_t)hd * 16 + (size_t)len * 16) + (32u << 20));
  struct ne_tensor* Q = ne_new_tensor_3d(ctx, NE_TYPE_F32, hd, 1, n_head, NE_SIZE_CALC, NE_BACKEND_CPU);
  struct ne_tensor* K = ne_new_tensor_3d(ctx, NE_TYPE_F16, hd, len, n_head, NE_SIZE_CALC, NE_BACKEND_CPU);
  struct ne_tensor* V = ne_new_tensor_3d(ctx, NE_TYPE_F16, len, hd, n_head, NE_SIZE_CALC, NE_BACKEND_CPU);
  memcpy(Q->data, q, (size_t)hd * n_head * 4);
  memcpy(K->data, kc, (size_t)hd * len * n_head * 2);
  memcpy(V->data, vc, (size_t)hd * len * n_head * 2);
  struct ne_tensor* KQ = ne_mul_mat(ctx, K, Q);
  struct ne_tensor* KQ_scaled = ne_scale_inplace(ctx, KQ, ne_new_f32(ctx, scale));
  struct ne_tensor* P = ne_soft_max_inplace(ctx, KQ_scaled);
  struct ne_tensor* KQV = ne_mul_mat(ctx, V, P);
  ref_ne_run(ctx, KQV);
  memcpy(out, KQV->data, (size_t)hd * n_head * 4);
  ne_free(ctx);
}


/* ---- a whole Llama eval through the reference's engine ----------------------------------------------------------------
 * The graph of models/llama/llama.cpp:190-720 for ggml-type weights, batch 1, n_head == n_head_kv, the non-fused attention
 * path (:362-420 KV append, :286-302 shape of the K.Q / soft_max / V.P chain), built node by node with the public API and
 * executed by ne_graph_compute.  n_head_kv < n_head (GQA) relies on ne_mul_mat's head broadcast (ne_can_mul_mat,
 * ne_layers.c:618-623: consecutive query heads share a KV head).  Weights are Q4_0 rows (NE_TYPE_Q4_0 tensors: the ggml mul_mat path of ne_layers.c:7085);
 * norms and the embedding table fp32; KV cache fp16, K as [hd, n_ctx, head], V transposed [n_ctx, hd, head]. */
typedef struct ref_ne_llama {
  int n_vocab, n_embd, n_head, n_head_kv, n_layer, n_ff, n_ctx;
  int wtype;  /* NE_TYPE_Q4_0 or NE_TYPE_BTLA */
  int fused;  /* BTLA only: ne_mul_qkv / ne_ffn_silu nodes when the *_support probes agree (llama.cpp:212-215,609-618) */
  int n_threads;
  float eps, freq_base, freq_scale;
  struct ne_context* wctx; /* weights + KV cache */
  struct ne_tensor *tok, *out_norm, *output, *kc, *vc;
  struct ne_tensor** lw; /* per layer: attn_norm, wq, wk, wv, wo, ffn_norm, w1, w2, w3 */
} ref_ne_llama;

/* matmul weight [n rows][k] of the model's weight type; BTLA tensors carry an explicit byte size (the serialized blob) */
static struct ne_tensor* ref_ne_weight(ref_ne_llama* m, int k, int n, size_t blob_bytes) {
  if (m->wtype == NE_TYPE_BTLA) return ne_new_tensor_2d(m->wctx, NE_TYPE_BTLA, k, n, blob_bytes, NE_BACKEND_CPU);
  return ne_new_tensor_2d(m->wctx, (enum ne_type)m->wtype, k, n, NE_SIZE_CALC, NE_BACKEND_CPU);
}

/* blob_bytes: NULL for ggml types; for BTLA the byte size of each matmul weight in the order output, then per layer wq wk wv wo
 * w1 w2 w3 */
REF_API ref_ne_llama* ref_ne_llama_create_ex(int n_vocab, int n_embd, int n_head, int n_head_kv, int n_layer, int n_ff, int n_ctx,
                                             float eps, float freq_base, float freq_scale, int wtype, const size_t* blob_bytes,
                                             int fused, int n_threads) {
  ref_ne_llama* m = (ref_ne_llama*)calloc(1, sizeof(*m));
  m->wtype = wtype, m->fused = fused, m->n_threads = n_threads > 0 ? n_threads : 1;
  m->n_vocab = n_vocab, m->n_embd = n_embd, m->n_head = n_head, m->n_head_kv = n_head_kv, m->n_layer = n_layer, m->n_ff = n_ff;
  m->n_ctx = n_ctx;
  const int kvd = n_embd / n_head * n_head_kv;
  m->eps = eps, m->freq_base = freq_base, m->freq_scale = freq_scale;
  size_t bytes = (size_t)n_vocab * n_embd * 4 + (size_t)n_vocab * n_embd + (size_t)n_layer * ((size_t)4 * n_embd * n_embd + (size_t)3 * n_embd * n_ff) +
                 (size_t)n_layer * n_ctx * n_embd * 4 + (64u << 20);
  if (blob_bytes)
    for (int i = 0; i < 1 + 7 * n_layer; ++i) bytes += blob_bytes[i] + 4096;
  m->wctx = ref_ne_ctx(bytes);
  m->tok = ne_new_tensor_2d(m->wctx, NE_TYPE_F32, n_embd, n_vocab, NE_SIZE_CALC, NE_BACKEND_CPU);
  m->out_norm = ne_new_tensor_1d(m->wctx, NE_TYPE_F32, n_embd, NE_SIZE_CALC, NE_BACKEND_CPU);
  m->output = ref_ne_weight(m, n_embd, n_vocab, blob_bytes ? blob_bytes[0] : 0);
  m->kc = ne_new_tensor_1d(m->wctx, NE_TYPE_F16, (int64_t)n_layer * n_ctx * kvd, NE_SIZE_CALC, NE_BACKEND_CPU);
  m->vc = ne_new_tensor_1d(m->wctx, NE_TYPE_F16, (int64_t)n_layer * n_ctx * kvd, NE_SIZE_CALC, NE_BACKEND_CPU);
  memset(m->kc->data, 0, ne_nbytes(m->kc));
  memset(m->vc->data, 0, ne_nbytes(m->vc));
  m->lw = (struct ne_tensor**)calloc((size_t)n_layer * 9, sizeof(struct ne_tensor*));
  for (int il = 0; il < n_layer; ++il) {
    struct ne_tensor** w = m->lw + il * 9;
    w[0] = ne_new_tensor_1d(m->wctx, NE_TYPE_F32, n_embd, NE_SIZE_CALC, NE_BACKEND_CPU);
    const size_t* bb = blob_bytes ? blob_bytes + 1 + 7 * il : NULL;
    for (int j = 1; j <= 4; ++j) w[j] = ref_ne_weight(m, n_embd, (j == 2 || j == 3) ? kvd : n_embd, bb ? bb[j - 1] : 0);
    w[5] = ne_new_tensor_1d(m->wctx, NE_TYPE_F32, n_embd, NE_SIZE_CALC, NE_BACKEND_CPU);
    w[6] = ref_ne_weight(m, n_embd, n_ff, bb ? bb[4] : 0);
    w[7] = ref_ne_weight(m, n_ff, n_embd, bb ? bb[5] : 0);
    w[8] = ref_ne_weight(m, n_embd, n_ff, bb ? bb[6] : 0);
  }
  return m;
}
REF_API ref_ne_llama* ref_ne_llama_create(int n_vocab, int n_embd, int n_head, int n_head_kv, int n_layer, int n_ff, int n_ctx,
                                          float eps, float freq_base, float freq_scale) {
  return ref_ne_llama_create_ex(n_vocab, n_embd, n_head, n_head_kv, n_layer, n_ff, n_ctx, eps, freq_base, freq_scale, NE_TYPE_Q4_0,
                                NULL, 0, 1);
}
/* which: -1 tok_embd (f32), -2 out_norm (f32), -3 output (q4_0 rows); 0..8 = the layer's tensors in the order above */
REF_API int ref_ne_llama_set(ref_ne_llama* m, int layer, int which, const void* data, size_t bytes) {
  struct ne_tensor* t = which == -1 ? m->tok : which == -2 ? m->out_norm : which == -3 ? m->output : m->lw[layer * 9 + which];
  /* a BTLA tensor's size counts the tensor struct as well (ne_new_tensor_impl, ne_layers.c:1078,1095): the blob must fit */
  if (t->type == NE_TYPE_BTLA ? bytes > ne_nbytes(t) : ne_nbytes(t) != bytes) return -1;
  memcpy(t->data, data, bytes);
  return 0;
}
REF_API void ref_ne_llama_free(ref_ne_llama* m) {
  ne_free(m->wctx);
  free(m->lw);
  free(m);
}

REF_API void ref_ne_llama_eval(ref_ne_llama* m, const int* tokens, int N, int n_past, float* logits_last) {
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
    struct ne_tensor* inpSA = inpL;
    struct ne_tensor* cur = ne_rms_norm(ctx0, inpL, m->eps);
    cur = ne_mul(ctx0, cur, w[0]);
    struct ne_tensor *Qcur, *Kcur, *Vcur;
    if (m->fused && m->wtype == NE_TYPE_BTLA && n_head == n_head_kv &&
        bestla_fusion_QKV_f32f32_support(w[1]->data, w[2]->data, w[3]->data, N, n_embd, n_embd)) {
      /* llama.cpp:212-222: one node, result [3][N][n_embd] */
      struct ne_tensor* QKVcur = ne_mul_qkv(ctx0, w[1], w[2], w[3], cur);
      Qcur = ne_reshape_3d(ctx0, ne_view_1d(ctx0, QKVcur, (int64_t)N * n_embd, 0 * N * n_embd * ne_element_size(QKVcur)), hd, n_head, N);
      Kcur = ne_reshape_3d(ctx0, ne_view_1d(ctx0, QKVcur, (int64_t)N * n_embd, 1 * N * n_embd * ne_element_size(QKVcur)), hd, n_head_kv, N);
      Vcur = ne_view_1d(ctx0, QKVcur, (int64_t)N * n_embd, 2 * N * n_embd * ne_element_size(QKVcur));
    } else {
      Qcur = ne_reshape_3d(ctx0, ne_mul_mat(ctx0, w[1], cur), hd, n_head, N);
      Kcur = ne_reshape_3d(ctx0, ne_mul_mat(ctx0, w[2], cur), hd, n_head_kv, N);
      Vcur = ne_mul_mat(ctx0, w[3], cur);
    }
    Qcur = ne_rope_inplace(ctx0, Qcur, n_past, hd, 0, 0, m->freq_base, m->freq_scale);
    Kcur = ne_rope_inplace(ctx0, Kcur, n_past, hd, 0, 0, m->freq_base, m->freq_scale);
    /* store key and value to the cache (llama.cpp:362-412) */
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
    if (N > 1) KQ_scaled = ne_diag_mask_inf_inplace(ctx0, KQ_scaled, n_past);
    struct ne_tensor* KQ_soft_max = ne_soft_max_inplace(ctx0, KQ_scaled);
    struct ne_tensor* V = ne_view_3d(ctx0, v_cache, n_past + N, hd, n_head_kv, (size_t)n_ctx * e16, (size_t)n_ctx * e16 * hd, 0);
    struct ne_tensor* KQV = ne_mul_mat(ctx0, V, KQ_soft_max);
    struct ne_tensor* KQV_merged = ne_permute(ctx0, KQV, 0, 2, 1, 3);
    cur = ne_cpy(ctx0, KQV_merged, ne_new_tensor_2d(ctx0, NE_TYPE_F32, n_embd, N, NE_SIZE_CALC, NE_BACKEND_CPU));
    cur = ne_mul_mat(ctx0, w[4], cur);
    struct ne_tensor* inpFF = ne_add(ctx0, cur, inpSA);
    cur = ne_rms_norm(ctx0, inpFF, m->eps);
    cur = ne_mul(ctx0, cur, w[5]);
    if (m->fused && m->wtype == NE_TYPE_BTLA &&
        bestla_fusion_FFN_SiLu_f32f32_support(w[6]->data, w[7]->data, w[8]->data, N, n_embd, n_ff, n_embd)) {
      cur = ne_ffn_silu(ctx0, w[6], w[7], w[8], cur); /* llama.cpp:609-612 */
    } else {
      struct ne_tensor* tmp = ne_mul_mat(ctx0, w[8], cur); /* ffn[2] = w3 (llama.cpp:615-620) */
      cur = ne_mul_mat(ctx0, w[6], cur);
      cur = ne_silu(ctx0, cur);
      cur = ne_mul(ctx0, cur, tmp);
      cur = ne_mul_mat(ctx0, w[7], cur);
    }
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

/* ---- expert-indexed nodes (mixture of experts) through the public graph API ----------------------------------------------
 * ne_mul_mat_id (ne_layers.c:2384): n_as experts [k x n] of type wtype (NE_TYPE_Q4_0 rows, or NE_TYPE_BTLA blobs of
 * expert_bytes[e] bytes), ids [n_used x n_tok] int32, slot `id`, b [k x n_tok] fp32 -> out [n x n_tok] fp32. */
REF_API void ref_ne_mul_mat_id(const void* const* experts, const size_t* expert_bytes, int wtype, int n_as, int n, int k,
                               const int32_t* ids, int n_used, int id, const float* b, int n_tok, float* out, int n_threads) {
  size_t bytes = (size_t)n_tok * ((size_t)k + n) * 8 + (size_t)n_tok * n_used * 4 + (64u << 20);
  for (int e = 0; e < n_as; ++e) bytes += expert_bytes[e] + 4096;
  struct ne_context* ctx = ref_ne_ctx(bytes);
  struct ne_tensor* as[8];
  if (n_as > 8) { fprintf(stderr, "ref_ne_mul_mat_id: n_as > 8\n"); abort(); }
  for (int e = 0; e < n_as; ++e) {
    as[e] = wtype == NE_TYPE_BTLA ? ne_new_tensor_2d(ctx, NE_TYPE_BTLA, k, n, expert_bytes[e], NE_BACKEND_CPU)
                                  : ne_new_tensor_2d(ctx, (enum ne_type)wtype, k, n, NE_SIZE_CALC, NE_BACKEND_CPU);
    memcpy(as[e]->data, experts[e], expert_bytes[e]);
  }
  struct ne_tensor* I = ne_new_tensor_2d(ctx, NE_TYPE_I32, n_used, n_tok, NE_SIZE_CALC, NE_BACKEND_CPU);
  memcpy(I->data, ids, (size_t)n_used * n_tok * 4);
  struct ne_tensor* B = ne_new_tensor_2d(ctx, NE_TYPE_F32, k, n_tok, NE_SIZE_CALC, NE_BACKEND_CPU);
  memcpy(B->data, b, (size_t)k * n_tok * 4);
  struct ne_tensor* r = ne_mul_mat_id(ctx, as, n_as, I, id, B);
  struct ne_cgraph gf = ne_build_forward(r);
  gf.n_threads = n_threads > 0 ? n_threads : 1;
  ne_graph_compute(ctx, &gf);
  memcpy(out, r->data, (size_t)n * n_tok * 4);
  ne_free(ctx);
}

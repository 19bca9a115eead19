/*
 * ns_b200.h -- C ABI of libns_b200.so: the H100-native (sm_90a) replacement for neural-speed's low-bit
 * weight-only matmul path.  Plain pointers and sizes only; no torch / C++ types cross this boundary.
 *
 * Every entry point names the reference interface it replaces (paths relative to /root/reference).
 * Three groups:
 *   1. bestla_*          host-buffer drop-ins with the exact signatures of neural_speed/core/ne_bestla.h:21-83.
 *                        `weiptr` is a serialized BesTLA blob in HOST memory (bestla/bestla/bestla_storage.h:697-834);
 *                        activations / outputs are HOST fp32.  The library uploads + repacks each blob once
 *                        (cached by address), runs the CUDA kernels, copies the result back.
 *   2. bestla_device_*   device-resident set modelled on the reference's NS_SYCL block, ne_bestla.h:85-112
 *                        (void* queue == cudaStream_t).  Activations / outputs are DEVICE fp32.
 *   3. ns_* / BTLAGemm*  ggml Q4_0 path (ne_compute_forward_mul_mat_q_f32, core/ne_layers.c:7085), the weight
 *                        packing API (core/layers/bestla_gemm.h:30-58, models/model_utils/quant_utils.cpp:226-400)
 *                        and handles for fused / graph-captured decode.
 *
 * Error convention (mirrors the reference, SURVEY.md 8b): *_support() are pure probes returning bool;
 * *_forward() print "Err: ..." and abort() on invalid input or when no CUDA device / kernel image is usable
 * (there is NO CPU fallback in this library); pack functions return false / 0 on failure;
 * ns_* functions return 0 on success and a negative NS_E_* code otherwise (message via ns_last_error()).
 */
#ifndef NS_B200_H
#define NS_B200_H
#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#include "ns_ne_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

#define NS_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------------ enums */
/* weight element formats in the device ("NSB") layout */
enum ns_wfmt {
  NS_W_S4 = 0,
  NS_W_S8 = 1,
  NS_W_NF4 = 2,
  NS_W_Q6K = 3, /* ggml block_q6_K, only via ns_weight_from_q6_K */
  NS_W_Q8_0 = 4 /* ggml block_q8_0, only via ns_weight_from_q8_0: int8 codes in natural order, fp16 scale per 32, NS_COMP_Q8_0 */
};
/* scale storage */
enum ns_stype { NS_S_F32 = 0, NS_S_BF16 = 1, NS_S_F16 = 2 };
/* activation numerics ("compute type"): which reference arithmetic the kernel reproduces
 *   NS_COMP_F32     fp32 activations, w = (q-zp)*scale in fp32, fp32 FMA      (BesTLA CompFp32, kernel_ref.h:2490)
 *   NS_COMP_BF16    activations and dequantised weights rounded to bf16, fp32 accumulate (BesTLA CompBf16)
 *   NS_COMP_INT8    u8-asym per-K-block activations x int weights, exact integer block dots
 *                   (BesTLA CompInt8, kernel_ref.h:1825 + :2372)
 *   NS_COMP_Q8_0    ggml: s8 activations per 32, fp16 scales, round-half-even (quantize.h:447, vec_dot.h:131)
 *   NS_COMP_INT8_S8 s8-sym per-K-block activations (kernel_ref.h:1886 + :2432)
 */
enum ns_comp { NS_COMP_F32 = 0, NS_COMP_BF16 = 1, NS_COMP_INT8 = 2, NS_COMP_Q8_0 = 3, NS_COMP_INT8_S8 = 4 };
/* ne_comp_type, neural_speed/core/data_types.h:55-62 */
enum ns_ne_comp_type { NS_NE_COMP_UNDEF = 0, NS_NE_COMP_F32 = 1, NS_NE_COMP_BF16 = 2, NS_NE_COMP_F16 = 3, NS_NE_COMP_INT8 = 4 };
/* BTLA_DTYPE raw values, bestla/bestla/bestla.h:38-87 */
#define NS_BTLA_F32 32u
#define NS_BTLA_BF16 (16u | (1u << 16))
#define NS_BTLA_F16 16u
#define NS_BTLA_S8 (8u | (1u << 8))
#define NS_BTLA_S4_CLIP (4u | (1u << 8))
#define NS_BTLA_F4_NF4 (4u | (2u << 16))
#define NS_BTLA_F4_BNB (4u | (1u << 16)) /* 4-bit float codebooks of bestla.h:82-84, kernel_ref.h:1209-1321 */
#define NS_BTLA_F4_E2M1 4u
/* bit-plane integer types (bestla.h:75-81, storage bestla_storage.h:724-745): held on the device in the 4-bit (2, 3 bits) or
 * 8-bit (5, 6, 7 bits) container, same integers, same scales and zero points */
#define NS_BTLA_S2_CLIP (2u | (1u << 8))
#define NS_BTLA_S3_CLIP (3u | (1u << 8))
#define NS_BTLA_S5_CLIP (5u | (1u << 8))
#define NS_BTLA_S6_CLIP (6u | (1u << 8))
#define NS_BTLA_S7_CLIP (7u | (1u << 8))

#define NS_OK 0
#define NS_E_INVALID (-1)
#define NS_E_NODEVICE (-2)
#define NS_E_CUDA (-3)
#define NS_E_UNSUPPORTED (-4)

NS_API const char* ns_last_error(void);
NS_API const char* ns_version(void);
/* number of kernels this library has launched since load (bench.py's gpu_launches) */
NS_API unsigned long long ns_launch_count(void);

/* ------------------------------------------------------------------ 1. ne_bestla.h host-buffer drop-ins */
/* ne_bestla.h:33 / core/layers/ne_bestla.cpp:19.  Selects cuda:0 lazily; aborts later if none. */
NS_API void bestla_init(void);
/* ne_bestla.h:25-27.  Host threads are irrelevant on the GPU path; kept for ABI compatibility. */
NS_API int bestla_set_threads(int nth);
NS_API void* bestla_get_thread_handle(void);
NS_API void bestla_timer(bool init);

/* ne_bestla.h:35 / core/layers/inner_product.cpp:20 -- M * pad128(K) * 4 bytes, as the reference */
NS_API unsigned long long bestla_f32f32_get_workspace_size(int m, int n, int k, void* wptr);
/* ne_bestla.h:37 / inner_product.cpp:28 -- C[m][n] = A[m][k] . dequant(W)  (lda is ignored, K is used: bestla_gemm.cpp:44) */
NS_API void bestla_f32f32_forward(float* activation, void* weiptr, float* output, int m, int n, int k, int lda, int ldo,
                                  void* workspace);
/* ne_bestla.h:40-42 / inner_product.cpp:113,132 -- bias epilogue */
NS_API bool bestla_fusion_add_f32f32_support(void* weiptr, int m, int n, int k);
NS_API void bestla_fusion_add_f32f32_forward(float* activation, void* weiptr, float* bias, float* output, int m, int n,
                                             int k, int lda, int ldo, bool boardcast_bias, void* workspace);
/* ne_bestla.h:44-51 / core/layers/ip_fusion_qkv.cpp:155,163,194 -- out = [3][M][N] */
NS_API unsigned long long bestla_fusion_QKV_f32f32_get_workspace_size(int m, int n, int k, void* w1ptr);
NS_API bool bestla_fusion_QKV_f32f32_support(void* wqptr, void* wkptr, void* wvptr, int m, int n, int k);
NS_API void bestla_fusion_QKV_f32f32_forward(float* activation, void* wqptr, void* wkptr, void* wvptr, float* output,
                                             int m, int n, int k, int lda, int ldo, void* workspace);
/* ne_bestla.h:53-66 / core/layers/ip_fusion_ffn.cpp:20,724-740 -- out = (silu(x W1) * (x W3)) W2 */
NS_API unsigned long long bestla_fusion_FFN_f32f32_get_workspace_size(int seq, int fin, int fmid, int fout, void* w1ptr,
                                                                      void* w2ptr);
NS_API bool bestla_fusion_FFN_SiLu_f32f32_support(void* w1ptr, void* w2ptr, void* w3ptr, int seq, int fin, int fmid,
                                                  int fout);
NS_API void bestla_fusion_FFN_SiLu_f32f32_forward(float* activation, void* w1ptr, void* w2ptr, void* w3ptr, float* tmp1,
                                                  float* tmp2, float* output, int seq, int fin, int fmid, int fout,
                                                  void* workspace);
/* ne_bestla.h:75 / ne_bestla.cpp:74 -- dequantise a blob to fp32 [n][ld] (ld >= k) */
/* GELU feed-forward nodes of the non-Llama architectures (ne_bestla.h:53-73, ip_fusion_ffn.cpp:729-779);
 * tanh-GELU of kernel_ref.h:1570.  Gelu_Mul: tmp2 = gelu(x W1) * (x W3); GeLu: tmp1 = gelu(x W1); Add_GeLu adds b1/b2. */
NS_API bool bestla_fusion_FFN_Gelu_Mul_f32f32_support(void* w1ptr, void* w2ptr, void* w3ptr, int seq, int fin, int fmid,
                                                      int fout);
NS_API void bestla_fusion_FFN_Gelu_Mul_f32f32_forward(float* activation, void* w1ptr, void* w2ptr, void* w3ptr, float* tmp1,
                                                      float* tmp2, float* output, int seq, int fin, int fmid, int fout,
                                                      void* workspace);
NS_API bool bestla_fusion_FFN_GeLu_f32f32_support(void* w1ptr, void* w2ptr, int seq, int fin, int fmid, int fout);
NS_API void bestla_fusion_FFN_GeLu_f32f32_forward(float* activation, void* w1ptr, void* w2ptr, float* tmp1, float* output,
                                                  int seq, int fin, int fmid, int fout, void* workspace);
NS_API bool bestla_fusion_FFN_Add_GeLu_f32f32_support(void* w1ptr, void* w2ptr, int seq, int fin, int fmid, int fout);
NS_API void bestla_fusion_FFN_Add_GeLu_f32f32_forward(float* activation, void* w1ptr, void* w2ptr, float* b1ptr, float* b2ptr,
                                                      float* tmp1, float* output, int seq, int fin, int fmid, int fout,
                                                      bool boardcast_bias, void* workspace);
NS_API void bestla_unpackweight_fp32(void* wptr, int n, int k, float* fp32data, int ld);
/* ne_bestla.h:77: quantise f32 [n][ld] into dstptr with the attributes of the blob srcptr (host only) */
NS_API void bestla_packweight_copyattr(const float* f32ptr, void* dstptr, int n, int k, int ld, void* srcptr);

/* The entry points that take the graph engine's own structs (ne_bestla.h:24-32,85; core/layers/ne_bestla.cpp:42,114-166,176,205).
 * The struct layouts are restated in ns_ne_abi.h (struct ns_ne_tensor == struct ne_tensor, ne.h:161-206); with these exported,
 * the reference's ne_graph_compute (ne_layers.c:11915) links against this library unchanged.
 *   bestla_support           which nodes the library takes (BesTLA matmuls, fused QKV / FFN, contiguous add / mul / norms), host
 *                            work-buffer size, n_tasks = 1
 *   bestla_backend_support   every result lives on the host (NE_BACKEND_CPU) outside the device-resident route
 *   bestla_parallel_for      INIT / COMPUTE / FINALIZE over the node's tasks (host threads for the engine's own ggml nodes)
 *   bestla_mul / _add / _layernormalization  host-buffer element-wise ops ne_layers.c:4622,5677,6541,6625 call directly (CUDA
 *                            kernels behind host staging, like the matmul drop-ins) */
NS_API bool bestla_support(struct ns_ne_tensor* node, int n_threads, size_t* workspace, size_t* dev_workspace);
NS_API int bestla_backend_support(struct ns_ne_tensor* src0, struct ns_ne_tensor* src1, int op);
NS_API void bestla_parallel_for(ns_forward_compute_fptr fcomp, struct ns_ne_compute_params* mainparams, struct ns_ne_tensor* node);
NS_API void bestla_mul(int batch, int vsize, const float* tensor, const float* vector, int vstep, float* out);
NS_API void bestla_add(int batch, int vsize, const float* tensor, const float* vector, int vstep, float* out);
NS_API void bestla_layernormalization(int norm_count, int norm_size, bool isrms, float epsilon, const float* FpIn, float* FpOut);

/* ------------------------------------------------------------------ 2. device-resident set (NS_SYCL analogue) */
/* ne_bestla.h:86-95.  device = opaque context owning one CUDA stream on cuda:<current>; queue = cudaStream_t */
NS_API void* bestla_create_device(bool profile);
NS_API void* bestla_get_device_queue(void* device);
NS_API void bestla_release_device(void* device);
NS_API size_t bestla_device_gmem_size(void* device);
NS_API void* bestla_device_malloc(size_t size, void* queue);
NS_API void bestla_device_free(void* ptr, void* queue);
NS_API void bestla_device_memcpy(void* dstptr, const void* srcptr, size_t size, void* queue);
NS_API void bestla_device_memcpy_sync(void* dstptr, const void* srcptr, size_t size, void* queue);
NS_API void bestla_device_sync(void* queue);
/* ne_bestla.h:96-97 / ne_bestla_sycl.cpp:94.  hoststor = serialized blob (host); devstor = host descriptor of
 * bestla_device_storage_size() bytes filled by the call; deviceptr = device buffer of at least
 * ns_device_storage_bytes(hoststor) bytes that receives the repacked weight. */
NS_API size_t bestla_device_storage_size(void);
NS_API size_t ns_device_storage_bytes(const void* hoststor);
NS_API void bestla_device_load_storage(void* hoststor, void* devstor, void* deviceptr, void* queue);
/* ne_bestla.h:98-99 / ne_bestla_sycl.cpp:152.  activation/output are DEVICE fp32; weiptr = devstor descriptor.
 * workspace: device scratch of >= ns_device_workspace_bytes(m, k) bytes (or NULL: library-owned scratch). */
NS_API size_t ns_device_workspace_bytes(int m, int k);
NS_API void bestla_device_f32f32_forward(float* activation, void* weiptr, float* output, int m, int n, int k, int lda,
                                         int ldo, void* workspace, void* queue);

/* ------------------------------------------------------------------ 3a. weight handles (device resident) */
typedef struct ns_weight ns_weight; /* opaque: repacked weight in HBM + metadata */

/* ggml rows: src0 of ne_compute_forward_mul_mat_q_f32 (ne_layers.c:7085): n rows of k/32 block_q4_0
 * (data_types.h:79-83), row stride nb01 bytes.  `rows` may be a host or a device pointer (rows_on_device).  The blocks are read
 * as 16-bit words: nb01 must be even and device rows 2-byte aligned (NULL, message via ns_last_error, otherwise; as for Q8_0). */
NS_API ns_weight* ns_weight_from_q4_0(const void* rows, int n, int k, size_t nb01, int rows_on_device, void* queue);
/* serialized BesTLA blob (host memory), StorageWeightKBlockNInteger / NFloat */
/* N rows of K/256 block_q6_K (core/data_types.h:133-138, 210 bytes each), row stride nb01: the type of output.weight in
 * llama.cpp "Q4_0" GGUF files.  ns_mul_mat on it reproduces quantize_row_q8_K + ggml_vec_dot_q6_K_q8_K
 * (vectors/cpu/quantize.h:1020, core/layers/vec_dot.h:907) bit for bit; plain matmul only (no fused QKV/FFN). */
NS_API ns_weight* ns_weight_from_q6_K(const void* rows, int n, int k, size_t nb01, int rows_on_device, void* queue);
/* N rows of K/32 block_q8_0 (core/data_types.h:107-111, 34 bytes each: fp16 d + 32 int8 codes), row stride nb01: the type of every
 * 2-D tensor of llama.cpp "Q8_0" GGUF files.  k % 32 == 0, nb01 even.  Repacked once on the GPU into the NSB int8 row (kpad codes in natural
 * order, then k/32 fp16 scales); compute type NS_COMP_Q8_0 (activations quantised by quantize_row_q8_0, exact integer block dots,
 * ne_vec_dot_q8_0_q8_0 of core/layers/vec_dot.h:594).  Routed like Q4_0: the ring GEMV (<= 2 rows, and tiles of <= 4), the integer
 * tensor cores (3..32 rows), the bf16 wgmma GEMM (longer prompts). */
NS_API ns_weight* ns_weight_from_q8_0(const void* rows, int n, int k, size_t nb01, int rows_on_device, void* queue);
NS_API ns_weight* ns_weight_from_btla_blob(const void* blob, void* queue);
/* same, with the number of bytes readable at `blob` (file-backed blobs: the parser never reads past it) */
NS_API ns_weight* ns_weight_from_btla_blob_n(const void* blob, size_t nbytes, void* queue);
/* canonical unpacked container as BTLAGemmPackB takes it (bestla_gemm.h:46-50): q int8 [k][n] (values, e.g.
 * nibble-8), scales f32 [k/g][n], zp int8 [k/g][n] or NULL, shuffle int[k] or NULL.  Host pointers. */
NS_API ns_weight* ns_weight_from_unpacked(const int8_t* q, const float* scales, const int8_t* zp, const int* shuffle, int n,
                                          int k, int group, int wfmt, int stype, int comp, void* queue);
NS_API void ns_weight_free(ns_weight* w);
NS_API int ns_weight_info(const ns_weight* w, int* n, int* k, int* group, int* wfmt, int* stype, int* comp, int* asym);
NS_API int ns_weight_set_comp(ns_weight* w, int comp);
/* packed bytes one GEMV must read from HBM for this weight (roofline numerator, SURVEY.md 8d) */
NS_API size_t ns_weight_algorithmic_bytes(const ns_weight* w);
/* benchmark aid: device weight of the given geometry with random codes, scales in [0.005, 0.02] and zero points (no host data) */
NS_API ns_weight* ns_weight_random(int n, int k, int group, int wfmt, int stype, int comp, int asym, unsigned seed, void* queue);
/* dequantise to device fp32 [n][ld] (debug / parity; replaces bestla_unpackweight_fp32 on device) */
NS_API int ns_weight_dequant_f32(const ns_weight* w, float* dst_dev, int ld, void* queue);

/* ------------------------------------------------------------------ 3b. device matmuls on handles */
/* dst[m][n] (ldo) = act[m][k] (lda) . W^T ; act/dst device fp32.  flags: NS_MM_* ; bias/residual may be NULL. */
#define NS_MM_BIAS_BCAST 1   /* bias is [n] broadcast over m (else [m][ldo]) */
#define NS_MM_FORCE_GEMV 2   /* always use the dp4a/FMA GEMV path (exact-integer numerics) regardless of m */
#define NS_MM_FORCE_TC 4     /* always use the wgmma tensor-core path (bf16 numerics) */
NS_API int ns_mul_mat(const ns_weight* w, const float* act, int lda, float* dst, int ldo, int m, const float* bias,
                      const float* residual, int flags, void* workspace, void* queue);
/* three weights sharing one activation (ne_mul_qkv): dst = [3][m][ldo], weights may differ in n */
NS_API int ns_mul_qkv(const ns_weight* wq, const ns_weight* wk, const ns_weight* wv, const float* act, int lda, float* dst,
                      int ldo, int m, void* workspace, void* queue);
/* ne_ffn_silu: tmp = silu(act.W1^T) * (act.W3^T) [m][fmid];  dst = tmp.W2^T [m][fout] */
/* GELU variants on device buffers: w3 != NULL -> Gelu_Mul (b1/b2 must be NULL); w3 == NULL -> (Add_)GeLu with optional biases */
NS_API int ns_ffn_gelu(const ns_weight* w1, const ns_weight* w2, const ns_weight* w3, const float* b1, const float* b2,
                       int bias_bcast, const float* act, int lda, float* tmp, float* dst, int ldo, int m, void* workspace,
                       void* queue);
NS_API int ns_ffn_silu(const ns_weight* w1, const ns_weight* w2, const ns_weight* w3, const float* act, int lda, float* tmp,
                       float* dst, int ldo, int m, void* workspace, void* queue);

/* The RMSNorm in front of a matmul node folded into the node's launch: ne_rms_norm + ne_mul(norm weight) + ne_mul_mat /
 * ne_mul_qkv / ne_ffn_silu (models/llama/llama.cpp:205-215, :601-612, :703-712) as ONE kernel -- every CTA of the decode GEMV
 * reads the whole activation row for the fused NE_TASK_INIT quantiser anyway, so the sum of squares costs a block reduction
 * instead of a one-CTA kernel and a launch boundary.  Decode rows only (m <= 2, int4 weights with an integer compute type, or Q8_0):
 * ns_rmsnorm_fusable says whether a set of 1..3 weights qualifies; the calls return NS_E_UNSUPPORTED otherwise.
 *   ns_rmsnorm_mul_mat   dst = W (rms_norm(act) * norm_w) [+ residual]
 *   ns_rmsnorm_mul_qkv   dst[3][m][ldo] as ns_mul_qkv
 *   ns_rmsnorm_ffn_silu  dst = W2 (silu(W1 xn) * (W3 xn)) [+ residual],  xn = rms_norm(act) * norm_w */
NS_API int ns_rmsnorm_fusable(const ns_weight* const* weights, int nw, int m);
NS_API int ns_rmsnorm_mul_mat(const ns_weight* w, const float* act, int lda, const float* norm_w, float norm_eps, float* dst, int ldo,
                              int m, const float* residual, void* workspace, void* queue);
NS_API int ns_rmsnorm_mul_qkv(const ns_weight* wq, const ns_weight* wk, const ns_weight* wv, const float* act, int lda,
                              const float* norm_w, float norm_eps, float* dst, int ldo, int m, void* workspace, void* queue);
NS_API int ns_rmsnorm_ffn_silu(const ns_weight* w1, const ns_weight* w2, const ns_weight* w3, const float* act, int lda,
                               const float* norm_w, float norm_eps, float* tmp, float* dst, int ldo, int m, const float* residual,
                               void* workspace, void* queue);

/* Expert-indexed nodes of mixture-of-experts models: ne_mul_mat_id and ne_mul_id_ffn_silu / _gelu
 * (core/ne_layers.c:2384-2460; ne_compute_forward_mul_mat_id_q_f32 :7345-7498, _q_f32_bestla :7783-7916, dispatch :7918-7943,
 * ne_compute_forward_ffn_id_silu / _gelu :8053-8111).  dst[t] = W[e_t] . act[t] with e_t = ids[t * ids_stride + id]
 * (ids = the int32 top-k selection [n_tokens][n_used], id = which of the n_used slots this node serves, ids_stride >= n_used).
 * The reference walks the tokens of every expert one by one; here tokens are grouped by expert and every expert's weights are
 * read once per node.  ids may live on the host (ids_on_device = 0, what ne_graph_compute has) or on the device (one small
 * D2H + stream sync per node: the host sizes the per-expert launches).  Expert ids outside [0, n_as) -> NS_E_INVALID.
 * flags: NS_MM_* of ns_mul_mat (e.g. NS_MM_FORCE_GEMV keeps the exact-integer path whatever the group size).
 * ns_ffn_id: gelu = 0 SiLU(gate) * up (Mixtral), 1 GELU(gate) * up; tmp [2][m][fmid] floats.
 * ns_mul_mat_id_q4_0_f32_host: the ggml-type host-buffer drop-in (expert_rows[e] = dst->opt[e]->data, ids = ids->data). */
NS_API int ns_mul_mat_id(const ns_weight* const* experts, int n_as, const int32_t* ids, int ids_stride, int id, int ids_on_device,
                         const float* act, int lda, float* dst, int ldo, int m, int flags, void* queue);
NS_API int ns_ffn_id(const ns_weight* const* gate, const ns_weight* const* down, const ns_weight* const* up, int n_as, int gelu,
                     const int32_t* ids, int ids_stride, int id, int ids_on_device, const float* act, int lda, float* tmp, float* dst,
                     int ldo, int m, void* queue);
/* the host-side grouping ns_mul_mat_id / ns_ffn_id perform, on its own (no device): order[m] = token indices sorted stably by expert
 * (the matrix_rows lists of ne_layers.c:7440-7449, flattened), span[2 * n_as] = per expert [begin, end) inside order.  Returns 1 when
 * the tokens already lie grouped (no gather / scatter needed), 0 otherwise, NS_E_INVALID on an expert id outside [0, n_as). */
NS_API int ns_moe_plan(const int32_t* ids, int ids_stride, int id, int m, int n_as, int* order, int* span);
NS_API int ns_mul_mat_id_q4_0_f32_host(const void* const* expert_rows, int n_as, size_t nb01, const int32_t* ids, int ids_stride,
                                       int id, const float* src1, float* dst, int ne00, int ne01, int ne11);

/* The two phases of a reference matmul node, separately (ne_compute_forward_mul_mat_q_f32: NE_TASK_INIT quantises src1
 * into wdata, NE_TASK_COMPUTE runs the dots; core/ne_layers.c:7143-7203):
 *   ns_prepare_activation  act[m][k] (device fp32) -> activation image in `workspace` (m <= 4 rows per image)
 *   ns_matmul_prepared     runs 1..3 weights against a prepared image.  mode: 0 plain, 1 concat ([nw][m][ldo] output,
 *                          ne_mul_qkv), 2 gate/up + SiLU*mul (ne_ffn_silu first half; aux may receive silu(gate)). */
NS_API int ns_prepare_activation(const ns_weight* w, const float* act, int lda, int m, void* workspace, void* queue);
NS_API int ns_matmul_prepared(const ns_weight* const* weights, int nw, int mode, const void* workspace, float* dst, int ldo,
                              int m, const float* bias, int bias_bcast, const float* residual, float* aux, void* queue);

/* The decode GEMV's launch plan on its own, for parity tests (no device needed): how ns_mul_mat & co. run one launch of m <= 4
 * activation rows of int4 weights with an integer compute type (k, group, stype, asym, comp as ns_weight_from_unpacked; Q4_0:
 * group 32, NS_S_F16, asym 0, NS_COMP_Q8_0) in mode 0 / 1 / 2 of ns_matmul_prepared.  fused: the kernel quantises fp32
 * activations itself (the ns_mul_mat path for groups of 32..256 dividing k), else it reads an ns_prepare_activation image;
 * norm: a folded RMSNorm (fused, m <= 2).  out[5] = {wide (1: one CTA per SM with 14 consumer warps, 0: the 7-warp kernel),
 * weight rows per ring stage (2 or 1), ring stages, stage-owning consumer warps, CTAs per SM}.  Returns 1 when the launch has
 * a plan, 0 when none fits shared memory (the matmul calls then refuse the node with NS_E_UNSUPPORTED before launching
 * anything), NS_E_INVALID for a launch the ring does not run. */
NS_API int ns_gemv_ring_plan(int k, int group, int stype, int asym, int comp, int mode, int m, int fused, int norm, int* out);
/* the same plan for a ggml Q8_0 weight of row length k (8-bit codes: a row is about twice the Q4_0 pitch, so fewer ring stages fit) */
NS_API int ns_gemv_ring_plan_q8_0(int k, int mode, int m, int fused, int norm, int* out);
/* ns_mul_mat as the eval step runs its GEMV nodes, for parity tests: on the kernel image that can fold an RMSNorm, without one
 * (one image for every node of a token); no bias, optional residual */
NS_API int ns_mul_mat_engine_image(const ns_weight* w, const float* act, int lda, float* dst, int ldo, int m, const float* residual,
                                   void* workspace, void* queue);
/* ns_ffn_silu as the eval step runs its prompt FFN nodes, for parity tests: dst = W2 (silu(W1 act) * (W3 act)) [+ residual].  On the
 * wgmma GEMM path silu(gate) * up goes straight into the down projection's bf16 activation image (the same values the two-step
 * ns_ffn_silu rounds from its fp32 product) and tmp [2][m][fmid] keeps only the gate and up outputs. */
NS_API int ns_ffn_silu_engine_image(const ns_weight* w1, const ns_weight* w2, const ns_weight* w3, const float* act, int lda, float* tmp,
                                    float* dst, int ldo, int m, const float* residual, void* workspace, void* queue);
/* The wgmma GEMM's launch plan for an m x n output over kpad (k rounded up to 32) inputs, for tests: out[3] = {token tile T,
 * k slices, k blocks of 64 per slice}.  Slices above 1 add fp32 partial tiles into a zeroed dst with atomics; residual_is_dst
 * (a residual or bias aliasing dst) keeps one.  Uses the SM count of the current device.  NS_E_INVALID on bad arguments. */
NS_API int ns_gemm_tc_plan(int m, int n, int kpad, int residual_is_dst, int* out);

/* CUDA-graph capture of a sequence of calls on one queue (replaces the reference's per-token graph rebuild +
 * ne_graph_compute, models/llama/llama.cpp:136-143 / core/ne_layers.c:11915): begin, issue ns_* device calls with
 * caller-provided workspaces (no allocation may happen while capturing), end -> executable graph handle. */
typedef struct ns_graph ns_graph;
NS_API int ns_graph_begin(void* queue);
NS_API ns_graph* ns_graph_end(void* queue);
NS_API int ns_graph_launch(ns_graph* g, void* queue);
NS_API void ns_graph_free(ns_graph* g);

/* The host drop-ins (bestla_*_forward, ns_mul_mat_*_host) upload and repack a host weight once and cache the device copy by
 * host address + a checksum sampled over the whole payload.  ns_host_cache_clear() releases every cached copy (call it when the
 * model context that owned the host weights is freed: the reference frees its weights with the context, model_files.h:1490-1499). */
NS_API void ns_host_cache_clear(void);
NS_API size_t ns_host_cache_entries(void);

/* ggml drop-in with HOST buffers: ne_compute_forward_mul_mat_q_f32 (ne_layers.c:7085) for NE_TYPE_Q4_0:
 * dst[ne11][ne01] = src1[ne11][ne00] x src0 rows.  src0 is uploaded/repacked once and cached by address. */
NS_API int ns_mul_mat_q4_0_f32_host(const void* src0_rows, size_t nb01, const float* src1, float* dst, int ne00, int ne01,
                                    int ne11);

/* ------------------------------------------------------------------ 3c. quantisers / packing API */
/* device RTN->Q4_0 (quantize_row_q4_0_reference, quantize.h:243): src f32 [n][k] device -> dst block_q4_0 rows device */
/* same for NE_TYPE_Q6_K weights (ne_layers.c:320-327) */
NS_API int ns_mul_mat_q6_K_f32_host(const void* src0_rows, size_t nb01, const float* src1, float* dst, int ne00, int ne01,
                                    int ne11);
/* same for NE_TYPE_Q8_0 weights (ne_layers.c:302-310: vec_dot_q = ne_vec_dot_q8_0_q8_0) */
NS_API int ns_mul_mat_q8_0_f32_host(const void* src0_rows, size_t nb01, const float* src1, float* dst, int ne00, int ne01,
                                    int ne11);
NS_API int ns_device_quantize_q4_0(const float* src_dev, void* dst_dev, int n, int k, void* queue);
/* device activation quantiser exposed for parity tests: one of ns_comp; outputs are device buffers
 * q: [m][k] (int8/uint8), scale: [m][k/g] f32, zp: [m][k/g] int32 (u8 mode, else untouched) */
NS_API int ns_device_quantize_act(const float* act_dev, int lda, int m, int k, int group, int comp, void* q_dev,
                                  float* scale_dev, int* zp_dev, void* queue);

/* ---- device-resident Llama-family eval step (SURVEY 8 f.1) ----------------------------------------------------------
 * Mirrors model_eval for the llama architecture (models/llama/llama.cpp:190-720): embedding lookup, RMSNorm, fused
 * QKV / three matmuls (GQA), RoPE mode 0, fp16 KV cache, softmax attention, o-proj + residual, RMSNorm, SiLU FFN + residual,
 * final RMSNorm, lm_head, greedy argmax (lowest index on ties, model_utils.cpp:2963-2985).  Weights are ns_weight handles
 * (borrowed: they must outlive the context); norms and the embedding table are fp32 host arrays copied to the device.
 * One-token evals replay one CUDA graph; ns_llama_generate feeds each argmax to the next step on the device. */
typedef struct ns_llama ns_llama;
typedef struct ns_llama_hparams {
  int n_vocab, n_embd, n_head, n_head_kv, n_layer, n_ff, n_ctx;
  float norm_eps;   /* hparams.norm_eps   (<= 0: 1e-6)  */
  float rope_theta; /* hparams.freq_base  (<= 0: 10000) */
  float rope_scale; /* hparams.freq_scale (<= 0: 1): divides the RoPE angle, as ne_rope does */
} ns_llama_hparams;
enum ns_llama_tensor {
  NS_LT_TOK_EMBD = 0, /* others[0]  [n_vocab][n_embd] f32 */
  NS_LT_OUT_NORM = 1, /* others[1]  [n_embd] f32          */
  NS_LT_OUTPUT = 2,   /* others[2]  n_vocab x n_embd weight (any ns_weight format, incl. Q6_K) */
  NS_LT_ATTN_NORM = 3, NS_LT_WQ = 4, NS_LT_WK = 5, NS_LT_WV = 6, NS_LT_WO = 7, /* layers[il].norm[0], attn[0..3] */
  NS_LT_FFN_NORM = 8, NS_LT_W1 = 9, NS_LT_W2 = 10, NS_LT_W3 = 11,              /* layers[il].norm[1], ffn[0..2]  */
  NS_LT_BQ = 12, NS_LT_BK = 13, NS_LT_BV = 14  /* Qwen2 only: q / k / v biases, f32 [n_embd] / [kvd] / [kvd] (ns_llama_set_f32) */
};
NS_API ns_llama* ns_llama_create(const ns_llama_hparams* hp, void* queue);
NS_API void ns_llama_free(ns_llama* ctx);
NS_API int ns_llama_set_f32(ns_llama* ctx, int tensor, int layer, const float* host, size_t count);
NS_API int ns_llama_set_weight(ns_llama* ctx, int tensor, int layer, const ns_weight* w);
/* ---- architecture ----------------------------------------------------------------------------------------------------------
 *   NS_LLAMA_ARCH_LLAMA  (default) the graph above
 *   NS_LLAMA_ARCH_QWEN2  Qwen1.5 / Qwen2 / Qwen2.5 (models/qwen/qwen.cpp, version 2): Llama's graph with q / k / v biases
 *                        (Q = W_q x + b_q, ...) and NeoX RoPE (ne_rope_inplace mode 2: pairs (i, i + hd/2)).
 *   NS_LLAMA_ARCH_PHI3   Phi-3 (models/phi/phi3.cpp): Llama's graph with NeoX RoPE and no biases.  Phi-3-mini's head size 96
 *                        runs on the split decode and tensor-core prompt attention like 64 / 128 (fp16 KV cache only).
 * The NeoX rotation runs as the mode-0 rotation on an interleaved head order: within each head, P maps dim i -> 2i and
 * i + hd/2 -> 2i + 1 (i < hd/2; at hd 96: i -> 2i, i + 48 -> 2i + 1), and rope_mode0(P x) == P rope_neox(x) bit for bit at
 * rope_scale 1.  ns_llama_set_weight(WQ | WK) on a Qwen2 or Phi-3 context therefore makes a context-owned device copy of the weight with its rows in P order per head (the caller's
 * handle stays borrowed and unmodified; the copy is freed when the slot is set again and by ns_llama_free), and b_q / b_k are
 * stored in P order.  q.k sums the same products, V is not permuted, so everything after attention is unchanged.  The K cache
 * (ns_llama_kv_cache / ns_llama_kv_planes) holds each head's keys in P order.
 * Allowed only before any matmul weight or bias is set (NS_E_INVALID otherwise).  NS_E_UNSUPPORTED for rope_scale != 1 (the
 * reference's NeoX branch scales the angle twice) and with streaming on; ns_llama_set_streaming refuses n_keep >= 0 on a Qwen2
 * or Phi-3 context (the reference has no NeoX shift-RoPE-K).  On a Qwen2 context every eval entry point returns NS_E_INVALID
 * until each layer has its three biases; NS_LT_BQ / BK / BV on a Llama or Phi-3 context are NS_E_INVALID. */
#define NS_LLAMA_ARCH_LLAMA 0
#define NS_LLAMA_ARCH_QWEN2 1
#define NS_LLAMA_ARCH_PHI3 2
NS_API int ns_llama_set_arch(ns_llama* ctx, int arch);
/* The weight a context runs for matmul tensor `tensor` of layer `layer` (for tests): the caller's handle, or on a Qwen2 / Phi-3 context
 * the P-order copy for NS_LT_WQ / NS_LT_WK; NULL when unset or for a tensor id that is no matmul weight. */
NS_API const ns_weight* ns_llama_weight(const ns_llama* ctx, int tensor, int layer);
/* evaluate n_tokens new tokens after n_past cached ones; logits_host (nullable) gets the n_vocab logits of the LAST token,
 * next_token (nullable) its greedy pick.  Synchronous (host buffers). */
NS_API int ns_llama_eval(ns_llama* ctx, const int32_t* tokens, int n_tokens, int n_past, float* logits_host, int32_t* next_token);
/* greedy generation of n_new tokens starting with first_token at position n_past; out_tokens[i] = pick after step i */
NS_API int ns_llama_generate(ns_llama* ctx, int32_t first_token, int n_past, int n_new, int32_t* out_tokens);
/* Numerics of prompt evaluation.  Matmuls of up to 32 new tokens reproduce the reference's exact integer block sums (GEMV /
 * integer tensor cores); longer prompts run the bf16 wgmma GEMM (measured logit deviation <= 4e-2 of max|logit| on the toy
 * models of tests/test_gpu_llama.py, KV cache entries differ at bf16 precision).  on = 1 evaluates long prompts in pieces of 32
 * tokens instead: reference numerics for the whole prompt at about 1/6 of the prefill throughput. */
NS_API int ns_llama_set_exact_prefill(ns_llama* ctx, int on);
/* Generation past n_ctx: the StreamingLLM ring of the reference's shift-RoPE-K mode (model_context.shift_roped_k / n_keep,
 * models/llama/llama.cpp:102-107, 351-354, 430-470).  0 <= n_keep < n_ctx enables it with n_keep attention-sink slots, -1
 * disables it.  With it on, n_past is the number of tokens evaluated so far (the reference's n_total) and may reach or pass n_ctx
 * for one-token steps (ns_llama_eval with n_tokens = 1, ns_llama_generate for any n_new).  Once the cache is full, the new token's
 * K / V go to slot n_keep + (n_total - n_ctx) mod (n_ctx - n_keep) -- the sinks are never overwritten -- every cached key at or
 * past n_keep is rotated one position back in the fp16 cache (the reference's fp16 arithmetic, rounding included), and attention
 * covers all n_ctx slots without a mask.  Steps that stay inside n_ctx are bit-identical to a context without streaming.
 *   NS_E_UNSUPPORTED  rope_scale != 1 (the reference divides positions by freq_scale but builds its shift table from freq_scale
 *                     undivided, so the two disagree), or a head size other than 64 / 128
 *   ns_llama_eval then returns NS_E_UNSUPPORTED for n_tokens > 1 with n_past + n_tokens > n_ctx (the reference's mask is
 *   meaningless in ring order, llama.cpp:467), and, once a step has passed n_ctx, NS_E_INVALID for any n_past other than the next
 *   position or a restart at n_past <= n_keep.  Enabling or disabling drops the captured decode graph. */
NS_API int ns_llama_set_streaming(ns_llama* ctx, int n_keep);
/* ---- continuous batching (the reference's model_eval over an array of model_input, models/llama/llama.cpp:53-90) ----------
 * The KV cache holds n_seq blocks, one per sequence ([n_layer][n_seq][n_head_kv][n_ctx][hd] fp16; kv_n_ctx_block =
 * max_request_num, model_utils.cpp:1027-1036).  A batched step takes one new token of each of n distinct sequences through one
 * forward pass of n rows: every matmul runs on all n rows at once (the weights are read once), K / V go to each row's block at
 * its own position (llama.cpp:370-411), attention runs per row (:414-489), and every row's logits are returned (:745-758).
 * Each row's arithmetic per matmul node is what a prompt of n rows gets (GEMV for n <= 2, the integer tensor cores for 3 .. 32
 * rows of int4 weights with an integer compute type); the attention of each row is the one-token step's, bit for bit.
 *
 * 1 <= n_seq <= 32 KV blocks (default 1).  Reallocates and zeroes the cache; every sequence restarts at n_past 0; drops the
 * captured graphs.  NS_E_UNSUPPORTED for n_seq > 1 with streaming on (llama.cpp:104 forbids the pair) or a head size other
 * than 64 / 96 / 128.  ns_llama_set_streaming returns NS_E_UNSUPPORTED for n_keep >= 0 while n_seq > 1.  ns_llama_eval and
 * ns_llama_generate serve sequence 0. */
NS_API int ns_llama_set_sequences(ns_llama* ctx, int n_seq);
/* ns_llama_eval on KV block `seq` (prompts, exact-prefill mode and all argument rules as ns_llama_eval) */
NS_API int ns_llama_eval_seq(ns_llama* ctx, int seq, const int32_t* tokens, int n_tokens, int n_past, float* logits_host,
                             int32_t* next_token);
/* one new token for each of n DISTINCT sequences in one forward pass of n rows; logits_host (nullable) [n][n_vocab],
 * next_tokens (nullable) [n] greedy picks; n_past[i] + 1 <= n_ctx.  One CUDA graph per n (captured on first use) serves any
 * set of sequences at any positions.  NS_E_INVALID (nothing launched) for n outside [1, n_seq], a sequence id outside
 * [0, n_seq) or given twice, n_past[i] < 0 or past the context, null pointers; NS_E_UNSUPPORTED with streaming on or a head
 * size other than 64 / 96 / 128. */
NS_API int ns_llama_decode_batch(ns_llama* ctx, int n, const int* seq, const int32_t* tokens, const int* n_past,
                                 float* logits_host, int32_t* next_tokens);
/* greedy generation for n distinct sequences, each pick fed back on the device; out_tokens [n][n_new];
 * n_past[i] + n_new <= n_ctx; argument rules as ns_llama_decode_batch */
NS_API int ns_llama_generate_batch(ns_llama* ctx, int n, const int* seq, const int32_t* first_tokens, const int* n_past,
                                   int n_new, int32_t* out_tokens);
/* One forward pass over n segments of n DISTINCT sequences (model_eval with n_input inputs, llama.cpp:53-90, 329-460, 745-758).
 * Segment i is n_tokens[i] >= 1 tokens of sequence seq[i], appended at positions n_past[i] ..; tokens holds all segments back to
 * back (T = sum n_tokens rows).  logits_host (nullable) [n][n_vocab]: each segment's LAST token, in the caller's order;
 * next_tokens (nullable) [n]: greedy picks.  New prompts, prompt chunks at n_past > 0 and the decode tokens of running
 * sequences share one pass: every matmul reads its weights once for all T rows.
 * Every matmul node is routed by ns_route at T rows, as a prompt of T tokens is (so a decode token in a pass of T > 32 rows takes
 * the bf16 wgmma GEMM for that step); the one-token segments' attention is ns_llama_decode_batch's, each longer segment's is
 * the tensor-core prompt attention (NS_ATTN_MMA) on its block, bit for bit -- also for 2 .. 7 tokens, where ns_llama_eval_seq
 * takes NS_ATTN_ROWS at head sizes 64 / 128.  When every segment has one token the call is ns_llama_decode_batch (its captured graph); other passes
 * run eagerly.  NS_E_INVALID (nothing launched) for n outside [1, n_seq], a sequence id outside [0, n_seq) or given twice,
 * n_tokens[i] < 1, n_past[i] < 0 or n_past[i] + n_tokens[i] > n_ctx, T > 4096 rows (a fixed cap per call: chunk longer
 * prompts), null pointers; NS_E_UNSUPPORTED with streaming on, a head size other than 64 / 96 / 128, or exact-prefill mode with
 * T > 32 (its integer block sums hold up to 32 rows). */
NS_API int ns_llama_eval_batch(ns_llama* ctx, int n, const int* seq, const int* n_tokens, const int32_t* tokens,
                               const int* n_past, float* logits_host, int32_t* next_tokens);
/* The host plan of ns_llama_eval_batch on its own (no device needed): the argument rules above that return NS_E_INVALID, for a
 * context of n_seq KV blocks of n_ctx positions, and the layout of the pass.  Internal order: the one-token segments first,
 * then the longer ones, each group in the caller's order.  order [n]: caller index of internal segment j; rows [T][2]:
 * {position, KV block} of internal row r; tiles [>= T / 64 + n][5]: one entry per 64 query rows of each multi-token segment,
 * {segment's first row counted from internal row d, its length, its n_past, its block, the tile's first query row inside the
 * segment}; counts [3] = {T, d = number of one-token segments, number of tile entries}. */
NS_API int ns_llama_batch_plan(int n_seq, int n_ctx, int n, const int* seq, const int* n_tokens, const int* n_past, int* order,
                               int* rows, int* tiles, int* counts);
/* model_eval with logits_all (llama.cpp:743-747; Model.__call__(logits_all=True) -> model.evaluate) over the segments of
 * ns_llama_eval_batch: every input token's row, scored on the device.  Rows are the T = sum n_tokens input tokens in the caller's
 * order (segments back to back, as `tokens`).  Outputs, each nullable, at least one non-null:
 *   logprobs [T]              log softmax(logits of row r)[targets[r]] (targets and logprobs both null or both non-null; every
 *                             target in [0, n_vocab))
 *   argmax [T]                the greedy pick of row r (lowest id on ties, as ns_llama_eval_batch's picks)
 *   logits_host [T][n_vocab]  the raw logits of every row
 * The body is ns_llama_eval_batch's pass on the same segments (run eagerly also when every segment has one token) and appends
 * the same K/V.  Then the final RMSNorm of all T rows, and per chunk of <= 32 rows the lm_head at the chunk's row count through
 * ns_route -- GEMV tiles where the route would take the bf16 GEMM, so integer formats keep their exact block sums on every row --
 * and one log-prob launch (the arithmetic of ns_logprob_row_host).  Device memory for logits is one chunk; logits_host fills
 * through pinned staging.  Argument rules and codes as ns_llama_eval_batch; also NS_E_INVALID for a target outside
 * [0, n_vocab), targets / logprobs not paired, or no output; NS_E_UNSUPPORTED while sampling is on (a scoring pass draws nothing).
 * A refused call launches nothing. */
NS_API int ns_llama_eval_all(ns_llama* ctx, int n, const int* seq, const int* n_tokens, const int32_t* tokens, const int* n_past,
                             const int32_t* targets, float* logprobs, int32_t* argmax, float* logits_host);
/* The log-prob kernel on its own, for parity tests: one launch over device logits [n][n_vocab] (1 <= n <= 32); device targets /
 * logprobs [n] (both or neither) and argmax [n] (nullable; one output at least).  ws: device workspace of
 * ns_llama_logprob_workspace_bytes(n, n_vocab) bytes, zeroed once by the caller: its tickets lie in the first 128 bytes for every
 * n and are zero again after every call.  A target outside [0, n_vocab) gives a NaN log-prob. */
NS_API size_t ns_llama_logprob_workspace_bytes(int n, int n_vocab);
NS_API int ns_llama_logprob(const float* logits, int n, int n_vocab, const int32_t* targets, float* logprobs, int32_t* argmax,
                            void* ws, void* queue);
/* Host restatement of one row (no device needed), bit for bit what the kernel computes (neural_speed_b200/csrc/logprob.h states
 * the order of every sum): max M and argmax over 32 slices, S = sum of exp(x - M) with the library's exp (ns_sample_expf_host),
 * logprob = (x[target] - M) - log(S) with the library's log (within 1 ulp of glibc's logf).  A NaN logit makes the row's log-probs
 * NaN; a -inf target logit gives -inf when the row has a finite max; a row with nothing above -inf gives NaN.  logprob or argmax
 * nullable (one at least); target read only with logprob. */
NS_API int ns_logprob_row_host(const float* logits, int n_vocab, int32_t target, float* logprob, int32_t* argmax);
/* ---- sampling (the reference's Model.generate(do_sample=True): model_post_sample_top_k_top_p_repeat, model_utils.cpp:2987-3032)
 * Per row, in this order: the repetition penalty on every candidate whose id occurs in the sequence's window (once per id:
 * logit <= 0 ? logit * penalty : logit / penalty), the top_k largest logits (ties: lower id first), top-p on their fp32 softmax
 * (the first i >= 1 whose running sum passes top_p is dropped with everything after it), logits / temperature, an fp32 softmax,
 * and a draw of std::discrete_distribution on one std::mt19937(seed) for the whole context (GCC libstdc++'s arithmetic; a list
 * of one candidate takes it without drawing).  Rows of a batch draw in the caller's order.  In per-sequence mode
 * (ns_llama_set_sequence_sampling) each KV block has its own parameters, generator and window instead.  The exp is the library's own
 * (ns_sample_expf_host), within 1 ulp of glibc's expf.
 * Window of a sequence: its last W = min(repeat_last_n, n_ctx) evaluated tokens, preceded by zeros (the reference's history
 * starts as n_ctx zeros, application/main_pybind.cpp:460-474), including every token of the pass that samples.  Windows are kept
 * only while sampling is on: tokens evaluated with sampling off are in no window.  A sequence's window restarts as zeros when one
 * of its segments is evaluated at n_past == 0, and every window does on ns_llama_set_sampling and ns_llama_set_sequences. */
typedef struct ns_llama_sampling {
  int top_k;            /* 1 .. 1024 (NS_E_UNSUPPORTED above: the limit of the device selection) */
  float top_p;          /* (0, 1]; 1 = off */
  float temperature;    /* finite, > 0 */
  float repeat_penalty; /* finite, > 0; 1 = off */
  int repeat_last_n;    /* 0 .. 256 (the reference uses 64) */
  uint32_t seed;        /* std::mt19937(seed); a time-based seed is the caller's choice */
} ns_llama_sampling;
/* s non-null: sample from now on -- reseeds the generator and restarts every window; NULL: greedy (the default).  Either drops
 * the captured graphs.  Picks returned and fed back by ns_llama_eval, ns_llama_eval_seq, ns_llama_generate (also past n_ctx on
 * the streaming ring), ns_llama_decode_batch, ns_llama_generate_batch and ns_llama_eval_batch are then sampled; returned
 * logits stay the raw logits.  The sampler takes the argmax's launch, so every step launches as many kernels as greedy.
 * NS_E_INVALID (mode unchanged) for a field out of range; NS_E_UNSUPPORTED for top_k > 1024.  Either call also leaves
 * per-sequence mode (below): from then on the context picks exactly as one that never entered it. */
NS_API int ns_llama_set_sampling(ns_llama* ctx, const ns_llama_sampling* s);
/* Per-sequence sampling: each KV block its own parameters, generator and window, so greedy and sampled requests with any
 * settings share a batch and a request's draws depend on nothing but its own seed and logits.
 *   - The first call puts the context in per-sequence mode, where every block is greedy until it is given a config; entering
 *     the mode drops the captured graphs, once.
 *   - s non-null: block seq samples with s (the per-row arithmetic above) from its own std::mt19937(s->seed); its window
 *     restarts as zeros and holds W = min(s->repeat_last_n, n_ctx) tokens.  s NULL: block seq is greedy again and keeps no
 *     window.  A greedy block picks the argmax (lowest id on ties) and draws nothing.
 *   - A change after entering drops and recaptures no graph: each block's parameters, generator and window live in device
 *     tables that the captured steps read at replay.  The call synchronises the context's stream, so the change applies
 *     exactly from the next step.
 *   - Every entry point that picks -- ns_llama_eval, ns_llama_eval_seq, ns_llama_generate (block 0, also on the streaming
 *     ring), ns_llama_decode_batch, ns_llama_generate_batch and ns_llama_eval_batch -- samples each row with its block's
 *     config and draws from its block's generator, in whichever order the rows come; a row left with one candidate does
 *     not draw.  A segment evaluated at n_past == 0 restarts its block's window.  Every step launches as many kernels as
 *     greedy.
 *   - ns_llama_set_sequences makes every block greedy again and stays in the mode; ns_llama_set_sampling leaves it.
 *     ns_llama_eval_all and ns_llama_beam_search return NS_E_UNSUPPORTED while any block has a config.
 * NS_E_INVALID for seq outside [0, n_seq) or a field out of range; NS_E_UNSUPPORTED for top_k > 1024.  A refused call changes
 * nothing. */
NS_API int ns_llama_set_sequence_sampling(ns_llama* ctx, int seq, const ns_llama_sampling* s);
/* The sampler on its own, for parity tests: one launch over device logits [n][n_vocab] (1 <= n <= 32), device windows
 * [n][n_window] (0 <= n_window <= 256; every entry counts, repeat_last_n is not read) and a device generator mt_state[625] (as
 * ns_sample_seed_host writes it; advanced by the call).  picks [n] device; kept [n], ids [n][top_k] (the top_k list in selection
 * order) and probs [n][top_k] (the final probabilities of the kept entries, 0 after them), device and nullable.  ws: device
 * workspace of ns_llama_sample_workspace_bytes(n, top_k) bytes, zeroed once by the caller: its tickets lie in the first 144
 * bytes for every n and top_k and are zero again after every call.  NS_E_INVALID / NS_E_UNSUPPORTED as ns_llama_set_sampling, and for bad sizes or null pointers; a refused call
 * launches nothing. */
NS_API size_t ns_llama_sample_workspace_bytes(int n, int top_k);
NS_API int ns_llama_sample(const float* logits, int n, int n_vocab, const int32_t* windows, int n_window, const ns_llama_sampling* s,
                           uint32_t* mt_state, int32_t* picks, int* kept, int32_t* ids, float* probs, void* ws, void* queue);
/* The per-sequence sampler on its own, for parity tests: one launch as ns_llama_sample, but row r samples with its own config
 * s[r] (s: host [n]) and draws from its own generator mt_states + 625 r (device [n][625], each advanced by its row's draw
 * only).  Row r's window is the last min(s[r].repeat_last_n, n_window) entries of windows[r].  ids and probs are
 * [n][max top_k]; ws holds ns_llama_sample_workspace_bytes(n, max top_k) bytes, zeroed once, its tickets where
 * ns_llama_sample keeps them.  Codes as ns_llama_sample (the first refused row's); a refused call launches nothing and writes
 * nothing. */
NS_API int ns_llama_sample_rows(const float* logits, int n, int n_vocab, const int32_t* windows, int n_window,
                                const ns_llama_sampling* s, uint32_t* mt_states, int32_t* picks, int* kept, int32_t* ids,
                                float* probs, void* ws, void* queue);
/* Host restatements (no device needed): std::mt19937(seed) as 625 words; steps 2-7 for one row of n_vocab logits with the window
 * window[0 .. n_window) -- pick, kept count, ids [top_k] and probs [top_k] as ns_llama_sample writes them -- advancing `state`;
 * and the sampler's exp. */
NS_API void ns_sample_seed_host(uint32_t seed, uint32_t* state);
NS_API int ns_sample_row_host(const float* logits, int n_vocab, const int32_t* window, int n_window, const ns_llama_sampling* s,
                              uint32_t* state, int32_t* pick, int* kept, int32_t* ids, float* probs);
/* ---- beam search (the reference's Model.generate(num_beams > 1, do_sample=False): beam_search -> beam_search_flow::loop,
 * model_utils.cpp:2302-2766, 2939-2944) over n requests of B = num_beams beams each.  Request r owns KV blocks r B .. r B + B - 1
 * (their contents afterwards are unspecified); blocks from n B up are not touched.  Per step:
 *   candidates  each running beam's top 2B tokens by logit (B of beam 0 on the first step), scored log softmax + the beam's score
 *               (neural_speed_b200/csrc/beam.h states the arithmetic; on steps after the first, EOS is forbidden while fewer than
 *               min_new_tokens were generated: the reference's first step reads the inputs' default min_new_tokens, 0)
 *   selection   per request the top 2B candidates of all its beams; an EOS candidate ranked below B is dropped, one above scores its
 *               beam into the hypotheses (score / generated length ^ length_penalty, in double); the first B others become the
 *               next beams.  Ties: candidates by (score descending, beam ascending, id ascending); hypotheses by score, a later one
 *               above an earlier one.
 *   end         a request is done with max_new_tokens tokens, or with early_stopping once B hypotheses exist; then every current
 *               beam is scored into the hypotheses (unless done by early stopping) and the best one is the response.
 * The first step evaluates the prompts in one ns_llama_eval_batch pass; every later one replays the captured batched decode step
 * of the running beams, one candidates launch, one device-to-host copy of the candidates and at most one KV copy launch (a beam
 * that is not its source's first descendant takes a dropped beam's block and its source's generated positions). */
typedef struct ns_llama_beams {
  int num_beams;          /* 2 .. 32, with n * num_beams <= n_seq and 2 * num_beams <= n_vocab */
  int max_new_tokens;     /* >= 1 (the reference's n_predict) */
  int min_new_tokens;     /* >= 0: EOS forbidden before this many generated tokens, from the second step on */
  float length_penalty;   /* finite */
  int early_stopping;     /* 0 / 1 */
  int32_t eos_token_id;   /* [0, n_vocab) */
} ns_llama_beams;
/* prompts: n_tokens[r] >= 1 tokens each, back to back in `tokens`, with n_tokens[r] + max_new_tokens - 1 <= n_ctx (the last pick
 * is never evaluated).  out_tokens [n][max_new_tokens]: request r's response in out_tokens[r][0 .. out_len[r]); out_score [n]
 * (nullable): its length-penalised score.  NS_E_UNSUPPORTED while sampling or streaming is on, for a head size other than
 * 64 / 96 / 128, or in exact-prefill mode for prompts of more than 32 tokens in all (the prompt pass is ns_llama_eval_batch's); NS_E_INVALID for a field or length out of range or a null pointer.  A refused call launches nothing. */
NS_API int ns_llama_beam_search(ns_llama* ctx, int n, const int* n_tokens, const int32_t* tokens, const ns_llama_beams* cfg,
                                int32_t* out_tokens, int* out_len, float* out_score);
/* model_kv_cache_seq_cpy (model_utils.cpp:2058-2064) in one launch: positions [p0, p1) of KV block src[i] into block dst[i] for
 * i < n, every layer, K and V.  NS_E_INVALID (nothing launched) for a block outside [0, n_seq), a destination that is also a
 * source or appears twice, n outside [1, n_seq], or 0 <= p0 <= p1 <= n_ctx not holding. */
NS_API int ns_llama_kv_copy(ns_llama* ctx, int n, const int* src, const int* dst, int p0, int p1);
/* The candidates kernel on its own, for parity tests: one launch over device logits [n][n_vocab] (1 <= n <= 32), k in 1 .. 64;
 * prev [n] and mask [n] host arrays (mask[r]: row r's EOS logit is -FLT_MAX).  out: device [n][min(k, n_vocab)] {int32 id,
 * float score}.  ws: device workspace of ns_llama_beam_candidates_workspace_bytes(n, k) bytes, zeroed once by the caller: its
 * tickets lie in the first 128 bytes and are zero again after every call. */
NS_API size_t ns_llama_beam_candidates_workspace_bytes(int n, int k);
NS_API int ns_llama_beam_candidates(const float* logits, int n, int n_vocab, int k, const float* prev, const int* mask, int32_t eos,
                                    void* out, void* ws, void* queue);
/* Host restatement of one row (no device needed), bit for bit what the kernel computes: ids [min(k, n_vocab)] and scores. */
NS_API int ns_beam_candidates_row_host(const float* logits, int n_vocab, int k, float prev, int mask, int32_t eos, int32_t* ids,
                                       float* scores);
/* The library's log (ns_logf), for tests. */
NS_API float ns_logf_host(float x);
/* The flow of ns_llama_beam_search without a device: logits(user, rows, req, hist, hist_len, out) fills out [rows][n_vocab] with
 * the logits of each row's last token, row i being request req[i] with the token history hist[i][0 .. hist_len[i]) (prompt then
 * generated tokens); it returns 0 or an error that ends the search.  The first call holds the n prompts. */
typedef int (*ns_beam_logits_fn)(void* user, int rows, const int* req, const int32_t* const* hist, const int* hist_len, float* out);
NS_API int ns_beam_search_host(int n_vocab, int n_ctx, int n, const int* n_tokens, const int32_t* tokens, const ns_llama_beams* cfg,
                               ns_beam_logits_fn logits, void* user, int32_t* out_tokens, int* out_len, float* out_score);
NS_API float ns_sample_expf_host(float x);
NS_API unsigned long long ns_llama_kv_bytes(const ns_llama* ctx); /* all n_seq blocks, every plane: the device allocation */
/* The device pointers of the fp16 KV cache, [n_layer][n_seq][n_head_kv][n_ctx][head size] each for K and V (for tests).
 * NS_E_UNSUPPORTED while the cache is Q8_0 (ns_llama_kv_planes). */
NS_API int ns_llama_kv_cache(const ns_llama* ctx, void** k, void** v);
/* ---- KV cache element format ------------------------------------------------------------------------------------------------
 *   NS_KV_F16   (default) fp16 K / V, the reference's ggml cache
 *   NS_KV_Q8_0  K / V rows stored as ggml Q8_0 blocks of 32: K after RoPE and V as projected are quantised in fp32 by the
 *               activation quantiser of the NS_COMP_Q8_0 matmuls (d = fp16(amax / 127), codes round-half-even of x * 127 / amax);
 *               each unit (layer, block, kv head) has a code plane [n_ctx][hd] int8 and a scale plane of hd / 32 fp16 per row,
 *               n_ctx * hd / 32 halves padded to a multiple of 8.  Attention reads fp16(q * d) wherever it read an fp16 cache value,
 *               and the decode step's own new row likewise, so a Q8_0 cache C attends exactly as an fp16 cache holding those values.
 *               About 0.53x the bytes of fp16 at head size 128 (136 B against 256 B per row).
 * ns_llama_set_kv_type reallocates and zeroes every block (every sequence restarts at n_past 0) and drops the captured graphs, like
 * ns_llama_set_sequences.  NS_E_INVALID for another type; NS_E_UNSUPPORTED (nothing changed) for Q8_0 with streaming on (either
 * order: ns_llama_set_streaming refuses n_keep >= 0 on a Q8_0 cache) or a head size other than 64 / 128.  Under Q8_0 one-row steps
 * take the split decode attention and every longer step the tensor-core prompt attention (also 2 .. 7 rows of ns_llama_eval_seq);
 * NS_ATTN_ROWS / NS_ATTN_GENERIC (and the NS_ATTN_OLD_DECODE / NS_ATTN_SCALAR switches) have no Q8_0 form: NS_E_UNSUPPORTED. */
#define NS_KV_F16 0
#define NS_KV_Q8_0 1
NS_API int ns_llama_set_kv_type(ns_llama* ctx, int type);
NS_API int ns_llama_kv_type(const ns_llama* ctx);
/* The device planes of the KV cache (for tests): fp16 -- k / v as ns_llama_kv_cache, kd / vd null; Q8_0 -- k / v the codes
 * [n_layer][n_seq][n_head_kv][n_ctx][hd] int8, kd / vd the scales [n_layer][n_seq][n_head_kv][stride] fp16, stride = n_ctx * hd / 32
 * rounded up to a multiple of 8, row p of a unit at p * hd / 32. */
NS_API int ns_llama_kv_planes(const ns_llama* ctx, void** k, void** kd, void** v, void** vd);
/* One layer's attention of the eval step on its own, for parity tests: RoPE (mode 0, angle = p * rope_theta^(-2i/hd) / rope_scale)
 * of q [m][n_head * hd] in place and of the m new rows k [m][n_head_kv * hd] at positions n_past .. n_past + m - 1, k and v appended
 * to the fp16 caches kc / vc [n_head_kv][n_ctx][hd], out [m][n_head * hd] = causal softmax(K q / sqrt(hd)) V (llama.cpp:286-302).
 * All pointers are device memory.  kernel: NS_ATTN_AUTO (what ns_llama_eval runs for this shape) or one kernel forced:
 *   NS_ATTN_SPLIT_DECODE  m = 1, hd 64 / 96 / 128: context split over 256-position ranges, per-range results merged
 *   NS_ATTN_ROWS          hd 64 / 128: one CTA per (head, row); RoPE and the KV append fused in when m = 1
 *   NS_ATTN_MMA           hd 64 / 96 / 128: causal prompt attention on mma.sync tensor cores
 *   NS_ATTN_GENERIC       any even hd: one CTA per (head, row) after a separate RoPE + KV-append launch
 * NS_ATTN_AUTO at hd 96 takes NS_ATTN_SPLIT_DECODE for m = 1 and NS_ATTN_MMA otherwise.
 * A forced kernel that cannot take the shape returns NS_E_UNSUPPORTED without launching anything.
 * ws: device workspace of ns_llama_attention_workspace_bytes(n_head, hd, n_ctx) bytes, zeroed once by the caller:
 *   int state[4] (the call writes n_past to state[1]) | unsigned tickets[n_head] (zero again after every call), padded to 16 bytes |
 *   float partials[n_head][ceil(n_ctx / 256)][hd + 2] (split decode scratch, no value carried between calls) */
#define NS_ATTN_AUTO 0
#define NS_ATTN_SPLIT_DECODE 1
#define NS_ATTN_ROWS 2
#define NS_ATTN_MMA 3
#define NS_ATTN_GENERIC 4
NS_API size_t ns_llama_attention_workspace_bytes(int n_head, int hd, int n_ctx);
NS_API int ns_llama_attention(int kernel, float* q, const float* k, const float* v, void* kc, void* vc, int n_head, int n_head_kv,
                              int hd, int n_ctx, int n_past, int m, float rope_theta, float rope_scale, float* out, void* ws,
                              void* queue);
/* One layer's single-token step of the streaming ring (ns_llama_set_streaming) on its own, for parity tests: n_total tokens
 * evaluated before this one, n_keep sink slots, rope_scale 1.  While n_total < n_ctx it is the one-row step of ns_llama_attention;
 * after that q is rotated at n_ctx - 1, the new k at n_ctx, k / v stored in the ring slot, every cached key at or past n_keep
 * shifted one position back in place, and out covers all n_ctx slots.  Same workspace and argument rules as ns_llama_attention;
 * NS_E_UNSUPPORTED (nothing launched) for head sizes other than 64 / 128. */
NS_API int ns_llama_attention_ring(float* q, const float* k, const float* v, void* kc, void* vc, int n_head, int n_head_kv, int hd,
                                   int n_ctx, int n_keep, int n_total, float rope_theta, float* out, void* ws, void* queue);
/* One layer's batched decode attention on its own, for parity tests (as ns_llama_attention with NS_ATTN_SPLIT_DECODE, row by row):
 * q [n][n_head * hd] (rotated in registers only), k / v [n][n_head_kv * hd], caches [n_seq][n_head_kv][n_ctx][hd] fp16; row i
 * appends to block seq[i] at position n_past[i] and attends to positions 0 .. n_past[i] of that block; out [n][n_head * hd].
 * seq / n_past are host arrays of n entries (distinct ids in [0, n_seq), 0 <= n_past[i] < n_ctx, else NS_E_INVALID); hd 64 / 96 /
 * 128 (else NS_E_UNSUPPORTED); nothing is launched on a refused call.  ws: ns_llama_attention_batch_workspace_bytes(n, n_head, hd,
 * n_ctx) bytes, zeroed once by the caller: int rows[n][4] (n_past in slot 1) | int seq[n], padded to 16 bytes | unsigned
 * tickets[n][n_head] (zero again after every call), padded to 16 bytes | float partials[n][n_head][ceil(n_ctx / 256)][hd + 2]. */
NS_API size_t ns_llama_attention_batch_workspace_bytes(int n, int n_head, int hd, int n_ctx);
NS_API int ns_llama_attention_batch(float* q, const float* k, const float* v, void* kc, void* vc, int n_seq, int n,
                                    const int* seq, const int* n_past, int n_head, int n_head_kv, int hd, int n_ctx,
                                    float rope_theta, float rope_scale, float* out, void* ws, void* queue);
/* One layer's ragged prompt attention on its own, for parity tests (as one ns_llama_attention(NS_ATTN_MMA) call per segment on
 * that segment's block): segment i is n_tokens[i] >= 1 rows of sequence seq[i] at positions n_past[i] .., the segments back to
 * back in the caller's order (T = sum n_tokens rows).  q [T][n_head * hd] is rotated in place, k / v [T][n_head_kv * hd] are
 * rotated / appended to the caches [n_seq][n_head_kv][n_ctx][hd] fp16, out [T][n_head * hd].  Argument rules of
 * ns_llama_eval_batch (NS_E_INVALID, nothing launched), hd 64 / 96 / 128 (else NS_E_UNSUPPORTED).  ws: device workspace of
 * ns_llama_attention_ragged_workspace_bytes(n, T) bytes: int rows[T][2] | int tiles[T / 64 + n][5], written by the call. */
NS_API size_t ns_llama_attention_ragged_workspace_bytes(int n, int n_rows);
NS_API int ns_llama_attention_ragged(float* q, const float* k, const float* v, void* kc, void* vc, int n_seq, int n, const int* seq,
                                     const int* n_tokens, const int* n_past, int n_head, int n_head_kv, int hd, int n_ctx,
                                     float rope_theta, float rope_scale, float* out, void* ws, void* queue);
/* The three entries above on a Q8_0 cache (NS_KV_Q8_0): kq / vq the code planes, kd / vd the scale planes of the same units
 * (ns_llama_kv_planes' layout with n_layer = 1).  Same workspaces and argument rules; NS_E_UNSUPPORTED (nothing launched) for head
 * sizes other than 64 / 128 and for NS_ATTN_ROWS / NS_ATTN_GENERIC; NS_ATTN_AUTO takes NS_ATTN_SPLIT_DECODE for m = 1, NS_ATTN_MMA
 * otherwise. */
NS_API int ns_llama_attention_q8_0(int kernel, float* q, const float* k, const float* v, void* kq, void* kd, void* vq, void* vd,
                                   int n_head, int n_head_kv, int hd, int n_ctx, int n_past, int m, float rope_theta, float rope_scale,
                                   float* out, void* ws, void* queue);
NS_API int ns_llama_attention_batch_q8_0(float* q, const float* k, const float* v, void* kq, void* kd, void* vq, void* vd, int n_seq,
                                         int n, const int* seq, const int* n_past, int n_head, int n_head_kv, int hd, int n_ctx,
                                         float rope_theta, float rope_scale, float* out, void* ws, void* queue);
NS_API int ns_llama_attention_ragged_q8_0(float* q, const float* k, const float* v, void* kq, void* kd, void* vq, void* vd, int n_seq,
                                          int n, const int* seq, const int* n_tokens, const int* n_past, int n_head, int n_head_kv,
                                          int hd, int n_ctx, float rope_theta, float rope_scale, float* out, void* ws, void* queue);

/* ---- tensor-parallel exchange step over NVLink peer memory (SURVEY 8e) --------------------------------------------
 * One-shot sum all-reduce replacing reduce_add / ne_all_reduce (core/parallel_context.cpp:47, ne_layers.c:5466) for the
 * [M, n_embd] fp32 partials after o-proj / down-proj (llama.cpp:592,693).  One process per GPU: each creates a context,
 * the hosts exchange the ns_comm_get_handle blobs (e.g. torch.distributed all_gather) and call ns_comm_open_peers.
 * Every rank gets bit-identical sums (fixed rank order).  max_elems bounds n of later calls. */
typedef struct ns_comm ns_comm;
/* several ranks' communicators inside ONE process (loopback on one device, or one host process driving peer-enabled GPUs): wire
 * them by plain device pointers instead of cudaIpc handles; comms[r] is rank r */
NS_API int ns_comm_link_local(ns_comm* const* comms, int world);
NS_API size_t ns_comm_handle_bytes(void);
NS_API ns_comm* ns_comm_create(int rank, int world, size_t max_elems, void* queue);
NS_API int ns_comm_get_handle(ns_comm* c, void* handle_out);
NS_API int ns_comm_open_peers(ns_comm* c, const void* all_handles);
NS_API int ns_comm_all_reduce_f32(ns_comm* c, float* data, size_t n, const float* residual, void* queue);
NS_API int ns_comm_status(ns_comm* c);
NS_API void ns_comm_free(ns_comm* c);

/* core/layers/bestla_gemm.h:37-56 (C++ in the reference; same names/argument meaning, extern "C" here).
 * QuantType/ScaleDtype are raw BTLA_DTYPE values, CompType an ne_comp_type.  ThreadPool is ignored. */
NS_API size_t BTLAGemmPackBSize(size_t N, size_t K, size_t BlkSize, uint32_t QuantType, uint32_t ScaleDtype, bool isAsym,
                                int CompType, int* shuffle_indice);
NS_API bool BTLAGemmQuantPackB(void* PackedBuf, const float* FpData, size_t N, size_t K, size_t ldb, size_t BlkSize,
                               uint32_t QuantType, uint32_t ScaleDtype, bool isAsym, int CompType, bool isTrans,
                               void* ThreadPool);
NS_API bool BTLAGemmPackB(void* PackedBuf, const int8_t* QData, const float* Scales, const int8_t* Zp, size_t N, size_t K,
                          size_t ldb, size_t BlkSize, uint32_t QuantType, uint32_t ScaleDtype, bool isAsym, int CompType,
                          int* shuffle_indice, void* ThreadPool);
NS_API bool BTLAGemmUnPackB(float* FpData, const void* PackedBuf, size_t N, size_t K, size_t ldb, void* ThreadPool);
/* Tensor-parallel shard of a blob: bestla_split_weight (models/model_utils/model_files.h:1538-1562) -- unpack, slice the
 * [dst_k][dst_n] block at (k_rank, n_rank) (or the rank's third of each fused Q/K/V projection), re-quantise with the source
 * blob's attributes.  ns_split_weight_size gives the bytes `dst` must hold (0 = unsupported). Host only. */
NS_API size_t ns_split_weight_size(const void* src, size_t dst_n, size_t dst_k);
NS_API bool ns_split_weight(const void* src, void* dst, size_t src_n, size_t src_k, size_t dst_n, size_t dst_k, size_t n_rank,
                            size_t k_rank, bool qkv_fusion);
/* host Q4_0 row quantiser (ne_quantize_q4_0 path; quantize.h:243) for the weight-packing API */
NS_API void ns_quantize_row_q4_0(const float* x, void* y, int k);

#ifdef __cplusplus
}
#endif
#endif /* NS_B200_H */

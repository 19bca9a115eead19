// nsb.cuh -- internal definitions shared by the CUDA sources of libns_b200.so (sm_90a only).
//
// Device ("NSB") weight layout (see DESIGN.md "Data layout in HBM"):
//   N self-contained rows of `pitch` bytes (16-B multiple), row n at rows + n*pitch:
//     [ q      : q_bytes = kpad/2 (4-bit) or kpad (8-bit), kpad = roundup(K, 32)           ]
//     [ scales : ngroups x {f32|bf16|f16}, ngroups = ceil(K/group)  (at sc_off = q_bytes)  ]
//     [ zp     : ngroups x int8, asymmetric only       (at zp_off, 16-B aligned)           ]
//   Everything one output row needs is ONE contiguous byte range, so the decode GEMV streams whole rows with
//   cp.async.bulk (TMA 1-D) into a shared-memory ring, and the prefill GEMM sees the q part as a 2-D tensor of pitch
//   `pitch` for cp.async.bulk.tensor.
//   4-bit q: every 32-bit word holds 8 consecutive k (k0..k0+7); nibble position p (bits 4p..4p+3) holds element
//   k0 + {0,2,4,6,1,3,5,7}[p].  Hence (w >> 4j) & 0x000F000F yields elements (2j, 2j+1) in the (low, high) half-words
//   -- one op per bf16x2 pair for the tensor-core dequant -- and w & 0x0F0F0F0F / (w>>4) & 0x0F0F0F0F yield bytes
//   (e0,e4,e1,e5) / (e2,e6,e3,e7) for dp4a against activations stored in the same permuted order.
//   Stored nibble u = q + 8 (ints) or the NF4 code; value semantics w = (u - 8 - zp) * scale.
//   shuffle [K] int32 (GPTQ desc_act): activation column gather applied before activation quantisation.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/ns_b200.h"

struct ns_weight {
  int n, k, kpad;
  int group, ngroups;
  int wfmt, stype, comp, asym;
  uint8_t* rows;  // device: n * pitch bytes
  int pitch, q_bytes, sc_off, zp_off;
  int* shuffle;
  void* base;          // allocation owning rows/shuffle (NULL if external)
  size_t total_bytes;  // bytes of the device image
  int external;        // 1: memory supplied by caller (bestla_device_load_storage)
  int f4kind;          // NS_W_NF4 weights: which 16-level codebook the codes index (NS_F4_NF4 / _BNB / _E2M1)
};
enum { NS_F4_NF4 = 0, NS_F4_BNB = 1, NS_F4_E2M1 = 2 };

static inline size_t ns_round_up(size_t a, size_t b) { return (a + b - 1) / b * b; }
static inline int ns_stype_size(int stype) { return stype == NS_S_F32 ? 4 : 2; }

// fills kpad/group/ngroups/pitch/offsets from n,k,group,wfmt,stype,asym
static inline void ns_weight_layout(ns_weight* w) {
  w->kpad = (int)ns_round_up((size_t)w->k, 32);
  if (w->group <= 0 || w->group > w->k) w->group = w->k;
  w->ngroups = (w->k + w->group - 1) / w->group;
  w->q_bytes = (w->wfmt == NS_W_S8) ? w->kpad : w->kpad / 2;
  w->sc_off = w->q_bytes;
  w->zp_off = (int)ns_round_up((size_t)w->sc_off + (size_t)w->ngroups * ns_stype_size(w->stype), 16);  // TMA-copyable
  w->pitch = (int)ns_round_up((size_t)w->zp_off + (w->asym ? w->ngroups : 0), 16);
}

// ---- error handling -------------------------------------------------------------------------------------------------
void ns_set_error(const char* fmt, ...);
[[noreturn]] void ns_fatal(const char* fmt, ...);
bool ns_cuda_ok(cudaError_t e, const char* what);
int ns_ensure_device();  // 0 ok, <0 NS_E_*
void ns_count_launch(int n = 1);
int ns_num_sms();
cudaStream_t ns_stream_of(void* queue);  // NULL -> the library's default stream

#define NS_CUDA_TRY(expr)                             \
  do {                                                \
    if (!ns_cuda_ok((expr), #expr)) return NS_E_CUDA; \
  } while (0)

// ---- activation workspace layout (device scratch between act_prep and the matmul kernels) ----------------------------
// int8 modes : aq  [m][kpad] bytes (16-B padded)  then  meta [m][meta_stride] int2 {a_scale bits, (Sa & 0xffff) | za << 16}
// fp32 modes : af  [m][kpad] float
size_t ns_act_workspace_bytes(int m, int kpad);
static inline int ns_meta_stride(int kpad) { return (int)ns_round_up((size_t)(kpad >> 5), 2); }

// launchers implemented in the .cu files
int ns_launch_act_prep(const float* act, int lda, int m, const ns_weight* w, void* ws, cudaStream_t st);
int ns_gemv_tile_rows(const ns_weight* w);
int ns_launch_gemv(const ns_weight* const* ws_, int nw, int mode, const void* act_ws, float* dst, int ldo, int m,
                   int m_total, const float* bias, int bias_bcast, const float* residual, float* aux, cudaStream_t st,
                   const float* act_f32 = nullptr, int lda = 0, int eltop = 0, const float* norm_w = nullptr, float norm_eps = 0.f,
                   int one_image = 0);
bool ns_gemv_fused_quant_ok(const ns_weight* w);  // can the GEMV quantise the activations itself (one launch)?
// can RMSNorm(x) * norm_w be folded into that quantiser for m rows (m <= 2: the rows the ring GEMV takes before IMMA does)?
bool ns_gemv_fused_norm_ok(const ns_weight* const* ws, int nw, int m);
int ns_launch_repack_q4_0(const void* rows_dev, size_t nb01, ns_weight* w, cudaStream_t st);
int ns_launch_repack_canonical(const int8_t* q_kn_dev, const float* sc_dev, const int8_t* zp_dev, ns_weight* w,
                               cudaStream_t st);
int ns_launch_repack_btla(const void* qbuf_dev, const void* sc_dev, int src_stype, const int8_t* zp_dev, int cstep,
                          int kpad_src, int ntile, int packrow, int is_float, ns_weight* w, cudaStream_t st);
int ns_launch_dequant(const ns_weight* w, float* dst, int ld, cudaStream_t st);
int ns_launch_random_weight(ns_weight* w, unsigned seed, cudaStream_t st);  // synthetic image for benchmarks

// ggml Q6_K x Q8_K (q6k.cu)
void ns_q6k_layout(ns_weight* w);
int ns_launch_repack_q6k(const void* rows_dev, size_t nb01, ns_weight* w, cudaStream_t st);
size_t ns_q6k_workspace_bytes(int m, int k);
int ns_launch_dequant_q6k(const ns_weight* w, float* dst, int ld, cudaStream_t st);
int ns_launch_mul_mat_q6k(const ns_weight* w, const float* act, int lda, float* dst, int ldo, int m, const float* bias,
                          int bias_bcast, const float* residual, void* ws, cudaStream_t st);

// abi.cu: fused FFN with the residual add folded into the down projection (used by the decode engine, llama.cu)
int ns_ffn_silu_residual(const ns_weight* w1, const ns_weight* w2, const ns_weight* w3, const float* act, int lda, float* tmp,
                         float* dst, int ldo, int m, const float* residual, void* workspace, cudaStream_t st,
                         const float* norm_w = nullptr, float norm_eps = 0.f, int one_image = 0);
// abi.cu: plain matmul node of the decode engine (one_image: see GemvParams)
int ns_mul_mat_engine(const ns_weight* w, const float* act, int lda, float* dst, int ldo, int m, const float* residual, void* workspace,
                      cudaStream_t st, const float* norm_w, float norm_eps);
// abi.cu: fused QKV with the attention RMSNorm folded into the activation quantiser (norm_w may be NULL: plain ns_mul_qkv)
int ns_mul_qkv_norm(const ns_weight* wq, const ns_weight* wk, const ns_weight* wv, const float* act, int lda, float* dst, int ldo,
                    int m, void* workspace, void* queue, const float* norm_w, float norm_eps);

// moe.cu: dst[i] = src[idx[i]] (gather) or dst[idx[i]] = src[i] (scatter), rows of `cols` floats
int ns_launch_move_rows(bool gather, const float* src, int ld_src, const int* idx_dev, float* dst, int ld_dst, int rows, int cols,
                        cudaStream_t st);

// tensor-core path (gemm_tc.cu)
size_t ns_gemm_tc_workspace_bytes(int m, int kpad);
bool ns_gemm_tc_supported(const ns_weight* w);
int ns_launch_act_bf16(const ns_weight* w, const float* act, int lda, int m, void* ws, cudaStream_t st);
int ns_launch_gemm_tc(const ns_weight* w, const void* ws, float* dst, int ldo, int m, const float* bias, int bias_bcast,
                      const float* residual, cudaStream_t st);
int ns_launch_silu_mul(const float* g, const float* u, float* out, float* aux, size_t total, cudaStream_t st, int eltop = 0);
int ns_launch_gelu(float* x, size_t total, cudaStream_t st);
bool ns_launch_silu_mul_bf16(const ns_weight* w2, const float* g, const float* u, int m, void* ws, cudaStream_t st, int eltop, int* rc);

// integer tensor-core path for 5..32 activation rows (gemm_imma.cu); modes and epilogue arguments as ns_launch_gemv
bool ns_gemm_imma_supported(const ns_weight* const* ws, int nw, int m);
size_t ns_gemm_imma_workspace_bound(int m, int kpad);  // enough for any weight shape the launcher accepts
int ns_launch_gemm_imma(const ns_weight* const* ws, int nw, int mode, const float* act, int lda, float* dst, int ldo, int m,
                        const float* bias, int bias_bcast, const float* residual, int eltop, void* workspace, cudaStream_t st);

enum { NS_GEMV_PLAIN = 0, NS_GEMV_CONCAT = 1, NS_GEMV_GATE_UP_SILU = 2 };
// element-wise epilogue op (bestla.h:89 BTLA_ELTWISEOP): DEFAULT = Swish(alpha=-1) in gate/up mode, nothing otherwise
enum { NS_ELT_DEFAULT = 0, NS_ELT_GELU = 1 };
enum { A_S8 = 0, A_U8 = 1, A_F32 = 2 };

// shared by both GEMV kernels
struct GemvParams {
  const uint8_t* rows[3];  // row base of each weight
  int n[3];
  long long dst_off[3];
  int nw, mode;
  int k, kpad, group, ngroups, stype;
  int cpg;  // 32-element chunks per scale group
  int pitch, q_bytes, sc_off, zp_off;
  const void* act;  // prepared activation image (device), or NULL when act_f32 is given
  const float* act_f32;  // raw fp32 activations [m][lda]: quantised inside the kernel (fused NE_TASK_INIT)
  int lda, comp;
  int act_bytes;    // bytes to stage in shared memory
  int meta_off;     // byte offset of the meta array inside the image (int8 modes)
  int meta_stride;  // int2 per activation row
  float* dst;
  int ldo, m;
  const float* bias;
  int bias_bcast;
  const float* residual;
  float* aux;
  int npairs;
  int eltop;  // NS_ELT_*
  int f4kind;           // NS_W_NF4 weights: codebook
  const float* norm_w;  // fused ne_rms_norm + ne_mul in front of the activation quantiser (llama.cpp:205-210), or NULL
  float norm_eps;
  int one_image;  // decode engine: run this node on the norm-capable kernel image even without a norm, so that ALL the GEMV nodes of
                  // a token share ONE code image (two alternating images cost ~70 us per token in instruction fetch, measured: 736 -> 776 tok/s)
};
int ns_launch_gemv_ring(const GemvParams& P, int amode, bool asym, int mt, cudaStream_t st);  // gemv_ring.cu
int ns_launch_gemv_ring_wide(const GemvParams& P, int amode, bool asym, size_t act_region, int act_row, int red_off, cudaStream_t st,
                             bool* taken);  // gemv_ring_wide.cu

template <typename... Args>
static inline cudaError_t ns_launch_pdl(void (*kern)(Args...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                        Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  static const bool no_pdl = getenv("NS_NO_PDL") != nullptr;  // debugging aid: plain stream order
  cfg.attrs = attr;
  cfg.numAttrs = no_pdl ? 0 : 1;
  return cudaLaunchKernelEx(&cfg, kern, args...);
}

// ---- small device helpers --------------------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
// epilogue element-wise ops (kernel_ref.h:1569-1576: tanh-GELU and Swish alpha=-1)
__device__ __forceinline__ float ns_gelu(float x) {
  return 0.5f * x * (1.f + tanhf(0.7978845834732056f * (x + 0.044714998453855515f * x * x * x)));
}
__device__ __forceinline__ float ns_silu(float x) { return x / (1.f + expf(-x)); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// scale idx of a row whose scale array starts at `s` (global or shared memory, generic pointer)
__device__ __forceinline__ float ns_scale_at(const void* s, int stype, int idx) {
  if (stype == NS_S_F32) return reinterpret_cast<const float*>(s)[idx];
  if (stype == NS_S_F16) return __half2float(__ushort_as_half(reinterpret_cast<const unsigned short*>(s)[idx]));
  return __uint_as_float(static_cast<uint32_t>(reinterpret_cast<const unsigned short*>(s)[idx]) << 16);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int dp4a_uu(unsigned a, unsigned b, int c) {
  int d;
  asm("dp4a.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
__device__ __forceinline__ int dp4a_ss(int a, int b, int c) {
  int d;
  asm("dp4a.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
__device__ __forceinline__ int dp4a_us(unsigned a, int b, int c) {
  int d;
  asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
// 4-bit float codebooks by the reference's codes: NF4 (kernel_ref.h:1325-1368; code 0 <-> 0.0, code 7 <-> -1.0), FP4 "BNB"
// (:1209-1230) and FP4 E2M1 (:1300-1321), both sign-magnitude with the sign in bit 3
static __device__ __constant__ const float NS_F4_LUT[3][16] = {
    {0.f, -0.6961928009986877f, -0.5250730514526367f, -0.39491748809814453f, -0.28444138169288635f, -0.18477343022823334f, -0.09105003625154495f, -1.f, 0.07958029955625534f, 0.16093020141124725f, 0.24611230194568634f, 0.33791524171829224f, 0.44070982933044434f, 0.5626170039176941f, 0.7229568362236023f, 1.0f},
    {0.f, 5.208333333e-03f, 0.66666667f, 1.f, 0.33333333f, 0.5f, 0.16666667f, 0.25f,
     -0.f, -5.208333333e-03f, -0.66666667f, -1.f, -0.33333333f, -0.5f, -0.16666667f, -0.25f},
    {0.f, 0.010416666666666666f, 0.16666666666666666f, 0.25f, 0.3333333333333333f, 0.5f, 0.6666666666666666f, 1.f,
     -0.f, -0.010416666666666666f, -0.16666666666666666f, -0.25f, -0.3333333333333333f, -0.5f, -0.6666666666666666f, -1.f}};
#endif

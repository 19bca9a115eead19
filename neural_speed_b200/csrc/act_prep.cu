// act_prep.cu -- activation preparation kernels: the device counterpart of the reference's activation prologues
//   ggml  : quantize_row_q8_0                 (neural_speed/vectors/cpu/quantize.h:447-560, x86 body: id = 127/amax, RNE)
//   BesTLA: ActivationKBlockQuantize          (bestla/bestla/bestla_prologue_a.h:105-214) =
//           quantize_fp_u8_colblock / _s8_    (bestla/bestla/kernel_ref.h:1825 / :1886)
//           ShuffleActivationKBlock*          (bestla_prologue_a.h:299-424): column gather by g_idx before quantisation
// Output goes to a small device workspace in exactly the byte image the matmul kernels copy into shared memory.  The
// quantiser arithmetic and the image's byte order and ring offsets are those of act_quant.cuh.
#include "act_quant.cuh"

namespace {

// One warp per (row m, quantisation block b).  COMP: NS_COMP_Q8_0 | NS_COMP_INT8 (u8 asym) | NS_COMP_INT8_S8.
template <int COMP>
__global__ void __launch_bounds__(256) act_quant_kernel(const float* __restrict__ A, int lda, int M, int K, int kpad,
                                                        int group, int ngroups, const int* __restrict__ shuffle,
                                                        int perm8, uint8_t* __restrict__ aq, int2* __restrict__ meta,
                                                        int meta_stride, int act_row, int ring_layout) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (gw >= M * ngroups) return;
  const int m = gw / ngroups, b = gw - m * ngroups;
  const int k0 = b * group;
  const int kend = min(k0 + group, K);
  const int kend_pad = (b == ngroups - 1) ? kpad : kend;  // last block also owns the zero padding up to kpad
  const float* row = A + (size_t)m * lda;

  // pass 1: range
  float vmax = nsq::range_start<COMP>(k0 + group > K), vmin = 0.f;
  for (int k = k0 + lane; k < kend; k += 32) nsq::range_fold<COMP>(row[shuffle ? shuffle[k] : k], vmax, vmin);
  nsq::range_reduce<COMP>(vmax, vmin, 32);
  const nsq::BlockQuant bq = nsq::block_quant<COMP>(vmax, vmin);

  // pass 2: quantise 32 elements (one chunk) per iteration, emit permuted bytes + chunk meta
  uint8_t* qrow = aq + (size_t)m * act_row;
  for (int kc = k0; kc < kend_pad; kc += 32) {
    const int k = kc + lane;
    const int q = k < kend ? nsq::quant_code<COMP>(row[shuffle ? shuffle[k] : k], bq) : bq.za;
    int sa = q;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sa += __shfl_xor_sync(0xffffffffu, sa, o);
    const int pos = perm8 ? ((lane & ~7) | nsq::dp4a_pos(lane & 7)) : lane;
    qrow[ring_layout ? nsq::ring_offset((uint32_t)kc >> 5, (uint32_t)pos) : (uint32_t)(kc + pos)] = (uint8_t)q;
    if (lane == 0) meta[(size_t)m * meta_stride + (kc >> 5)] = nsq::meta_word(bq.scale, sa, bq.za);
  }
}

// fp32 / bf16-rounded activations, natural order, zero padded to kpad
__global__ void __launch_bounds__(256) act_copy_kernel(const float* __restrict__ A, int lda, int M, int K, int kpad,
                                                       const int* __restrict__ shuffle, int round_bf16,
                                                       float* __restrict__ af) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)M * kpad) return;
  const int m = (int)(idx / kpad), k = (int)(idx - (size_t)m * kpad);
  float v = 0.f;
  if (k < K) v = A[(size_t)m * lda + (shuffle ? shuffle[k] : k)];
  if (round_bf16) v = __bfloat162float(__float2bfloat16_rn(v));
  af[idx] = v;
}

// plain quantiser with un-permuted, un-fused outputs: the parity-test view of the same arithmetic
template <int COMP>
__global__ void act_quant_plain_kernel(const float* __restrict__ A, int lda, int M, int K, int group, int ngroups,
                                       uint8_t* __restrict__ q, float* __restrict__ scales, int* __restrict__ zps) {
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (gw >= M * ngroups) return;
  const int m = gw / ngroups, b = gw - m * ngroups;
  const int k0 = b * group, kend = min(k0 + group, K);
  const float* row = A + (size_t)m * lda;
  float vmax = nsq::range_start<COMP>(k0 + group > K), vmin = 0.f;
  for (int k = k0 + lane; k < kend; k += 32) nsq::range_fold<COMP>(row[k], vmax, vmin);
  nsq::range_reduce<COMP>(vmax, vmin, 32);
  const nsq::BlockQuant bq = nsq::block_quant<COMP>(vmax, vmin);
  for (int k = k0 + lane; k < kend; k += 32) q[(size_t)m * K + k] = (uint8_t)nsq::quant_code<COMP>(row[k], bq);
  if (lane == 0) {
    scales[(size_t)m * ngroups + b] = bq.scale;
    if (COMP == NS_COMP_INT8 && zps) zps[(size_t)m * ngroups + b] = bq.za;
  }
}

}  // namespace

size_t ns_act_workspace_bytes(int m, int kpad) {
  const size_t i8 = (size_t)m * ns_round_up((size_t)kpad, 1024) + (size_t)m * ns_meta_stride(kpad) * sizeof(int2);
  const size_t f32 = (size_t)m * kpad * sizeof(float);
  return ns_round_up(i8 > f32 ? i8 : f32, 256);
}

int ns_launch_act_prep(const float* act, int lda, int m, const ns_weight* w, void* ws, cudaStream_t st) {
  const int kpad = w->kpad;
  if (w->comp == NS_COMP_F32 || w->comp == NS_COMP_BF16) {
    const size_t total = (size_t)m * kpad;
    const int blocks = (int)((total + 255) / 256);
    NS_CUDA_TRY(ns_launch_pdl(act_copy_kernel, dim3(blocks), dim3(256), 0, st, act, lda, m, w->k, kpad,
                              (const int*)w->shuffle, (int)(w->comp == NS_COMP_BF16), (float*)ws));
    ns_count_launch();
    return NS_OK;
  }
  uint8_t* aq = (uint8_t*)ws;
  const int ring_layout = (w->wfmt == NS_W_S4 || w->wfmt == NS_W_Q8_0) ? 1 : 0;  // consumed by gemv_ring.cu; other formats use natural rows
  const int act_row = ring_layout ? (int)ns_round_up((size_t)kpad, 1024) : kpad;
  int2* meta = (int2*)((char*)ws + ns_round_up((size_t)m * act_row, 16));
  const int ms = ns_meta_stride(kpad);
  // activation blocks: ggml Q8_0 is always 32; BesTLA uses the weight's K-block (bestla_prologue_a.h:133)
  const int group = (w->comp == NS_COMP_Q8_0) ? 32 : w->group;
  const int ngroups = (w->k + group - 1) / group;
  const int warps = m * ngroups;
  const int blocks = (warps + 7) / 8;
  const int perm8 = (w->wfmt == NS_W_S8 || w->wfmt == NS_W_Q8_0) ? 0 : 1;  // 8-bit codes keep natural order (nsb.cuh)
  cudaError_t e;
  if (w->comp == NS_COMP_Q8_0)
    e = ns_launch_pdl(act_quant_kernel<NS_COMP_Q8_0>, dim3(blocks), dim3(256), 0, st, act, lda, m, w->k, kpad, group,
                      ngroups, (const int*)w->shuffle, perm8, aq, meta, ms, act_row, ring_layout);
  else if (w->comp == NS_COMP_INT8)
    e = ns_launch_pdl(act_quant_kernel<NS_COMP_INT8>, dim3(blocks), dim3(256), 0, st, act, lda, m, w->k, kpad, group,
                      ngroups, (const int*)w->shuffle, perm8, aq, meta, ms, act_row, ring_layout);
  else
    e = ns_launch_pdl(act_quant_kernel<NS_COMP_INT8_S8>, dim3(blocks), dim3(256), 0, st, act, lda, m, w->k, kpad, group,
                      ngroups, (const int*)w->shuffle, perm8, aq, meta, ms, act_row, ring_layout);
  NS_CUDA_TRY(e);
  ns_count_launch();
  return NS_OK;
}

extern "C" int ns_device_quantize_act(const float* act_dev, int lda, int m, int k, int group, int comp, void* q_dev,
                                      float* scale_dev, int* zp_dev, void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  cudaStream_t st = (cudaStream_t)queue;
  if (comp == NS_COMP_Q8_0) group = 32;
  if (group <= 0) group = k;
  const int ngroups = (k + group - 1) / group;
  const int blocks = (m * ngroups + 7) / 8;
  if (comp == NS_COMP_Q8_0)
    act_quant_plain_kernel<NS_COMP_Q8_0><<<blocks, 256, 0, st>>>(act_dev, lda, m, k, group, ngroups, (uint8_t*)q_dev, scale_dev, zp_dev);
  else if (comp == NS_COMP_INT8)
    act_quant_plain_kernel<NS_COMP_INT8><<<blocks, 256, 0, st>>>(act_dev, lda, m, k, group, ngroups, (uint8_t*)q_dev, scale_dev, zp_dev);
  else if (comp == NS_COMP_INT8_S8)
    act_quant_plain_kernel<NS_COMP_INT8_S8><<<blocks, 256, 0, st>>>(act_dev, lda, m, k, group, ngroups, (uint8_t*)q_dev, scale_dev, zp_dev);
  else {
    ns_set_error("ns_device_quantize_act: unsupported comp %d", comp);
    return NS_E_INVALID;
  }
  NS_CUDA_TRY(cudaGetLastError());
  ns_count_launch();
  return NS_OK;
}

// gemv_ring.cu -- the decode GEMV for 4-bit integer weights with 8-bit integer activations (ggml Q4_0 x Q8_0 and BesTLA
// int4 CompInt8): HBM -> shared-memory ring via TMA bulk copies, dp4a out of shared memory.
//
// Replaces the same reference functions as gemv.cu (ne_vec_dot_q4_0_q8_0, core/layers/vec_dot.h:131; gemv_4bit_u8s8_fp32 /
// gemv_4bit_s8s8_fp32, bestla/bestla/kernel_ref.h:2372/2432) for M <= 4.
//
// Why a ring: at 3.35 TB/s each of the 132 SMs of an H100 must keep >= ~25-50 KB of loads in flight (Little's law, ~1-2 us
// loaded HBM latency); register-staged loads cap that at occupancy x 128 B per thread.  Here one elected producer thread per CTA
// issues cp.async.bulk (UBLKCP) copies of whole weight-row PAIRS -- a row of the NSB layout is one contiguous
// [nibbles | scales | zero-points] byte range -- into a ring of slots guarded by full/empty mbarriers.  Each consumer warp
// owns a whole stage at a time (two rows): no cross-warp reduction, rows dealt round-robin over CTAs (balanced at any N).
// 7 consumer warps + 1 producer warp per CTA, 2 CTAs per SM (~105 KB ring each = 3 slots per consumer warp for K=4096).
// The producer streams BEFORE griddepcontrol.wait, so under programmatic dependent launch a CTA starts filling its ring the
// moment it becomes resident.
// Roofline: HBM.  Algorithmic bytes per launch = sum over weights of N*K/2 + N*ceil(K/g)*(scale_bytes [+1 if asym]).
#include "gemv_ring_impl.cuh"

namespace {

template <int AMODE, int M, bool ASYM, int STYPE>
int launch_one(const GemvParams& P, int mt, cudaStream_t st) {
  const int act_row = (int)ns_round_up((size_t)P.kpad, 1024);
  const size_t img_end = (size_t)mt * act_row + (size_t)mt * P.meta_stride * 8;
  const int red_off = (int)ns_round_up(img_end, 16);  // one float per consumer warp (<= 14) of reduction scratch behind the image
  const size_t act_region = ns_round_up(P.norm_w ? (size_t)red_off + 64 : img_end, 128);
  // Single-row launches that quantise their activations themselves run on the one-CTA-per-SM kernel with 14 consumer warps
  // (gemv_ring_wide.cu: the activation row is read and quantised once per SM); pre-quantised images stay on the two-CTA kernel.
  // NS_RING_WIDE=0 / 1 forces the choice.
  static const int env_wide = getenv("NS_RING_WIDE") ? atoi(getenv("NS_RING_WIDE")) : -1;
  if constexpr (M == 1) {
    if (env_wide == 1 || (env_wide < 0 && P.act_f32 != nullptr)) {
      bool taken = false;
      const int rc = ns_launch_gemv_ring_wide(P, AMODE, ASYM, act_region, act_row, red_off, st, &taken);
      if (taken) return rc;
    }
  }
  const RingPlan plan = plan_ring(P, act_region, false);
  if (plan.stages < 1) {
    ns_set_error("gemv_ring: row pitch %d too large for shared memory", P.pitch);
    return NS_E_UNSUPPORTED;
  }
  if constexpr (M <= 2) {  // the norm is only ever folded into launches of <= 2 rows (ns_gemv_fused_norm_ok)
    if ((P.norm_w || P.one_image) && P.act_f32) {
      if (plan.rows == 2) return launch_rows<AMODE, M, ASYM, STYPE, 2, true>(P, plan, act_region, act_row, red_off, st);
      return launch_rows<AMODE, M, ASYM, STYPE, 1, true>(P, plan, act_region, act_row, red_off, st);
    }
  }
  if (P.norm_w) {  // (one_image without fp32 activations or with 4 rows simply takes the plain kernel)
    ns_set_error("gemv_ring: fused RMSNorm needs fp32 activations and <= 2 rows");
    return NS_E_INVALID;
  }
  if (plan.rows == 2) return launch_rows<AMODE, M, ASYM, STYPE, 2, false>(P, plan, act_region, act_row, red_off, st);
  return launch_rows<AMODE, M, ASYM, STYPE, 1, false>(P, plan, act_region, act_row, red_off, st);
}

template <int AMODE, bool ASYM, int STYPE>
int launch_m(const GemvParams& P, int mt, cudaStream_t st) {
  switch (mt) {
    case 1: return launch_one<AMODE, 1, ASYM, STYPE>(P, mt, st);
    case 2: return launch_one<AMODE, 2, ASYM, STYPE>(P, mt, st);
    default: return launch_one<AMODE, 4, ASYM, STYPE>(P, mt, st);
  }
}

template <int AMODE, bool ASYM>
int launch_s(const GemvParams& P, int mt, cudaStream_t st) {
  switch (P.stype) {
    case NS_S_F32: return launch_m<AMODE, ASYM, NS_S_F32>(P, mt, st);
    case NS_S_F16: return launch_m<AMODE, ASYM, NS_S_F16>(P, mt, st);
    default: return launch_m<AMODE, ASYM, NS_S_BF16>(P, mt, st);
  }
}

}  // namespace

int ns_launch_gemv_ring(const GemvParams& P, int amode, bool asym, int mt, cudaStream_t st) {
  if (amode == A_U8) return asym ? launch_s<A_U8, true>(P, mt, st) : launch_s<A_U8, false>(P, mt, st);
  return asym ? launch_s<A_S8, true>(P, mt, st) : launch_s<A_S8, false>(P, mt, st);
}

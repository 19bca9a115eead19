// gemv_ring_wide.cu -- the decode GEMV on ONE CTA per SM: 14 consumer warps + 2 producer warps (alternate ring stages).
//
// Same kernel template as gemv_ring.cu (gemv_ring_impl.cuh), NC = 14.  Every CTA of the ring GEMV pulls the whole fp32 activation row
// (16-44 KB) through L2 and quantises it (fused NE_TASK_INIT: quantize_row_q8_0, vectors/cpu/quantize.h:447; quantize_fp_u8/s8_colblock,
// bestla/bestla/kernel_ref.h:1825/1886) before its first dp4a; with one CTA per SM the row is read and quantised once per SM
// instead of twice.  Used for single-row launches that quantise their
// own activations (the decode path); pre-quantised images and 2..4-row launches stay on the two-CTA shape.
#include "gemv_ring_impl.cuh"

namespace {

template <int AMODE, bool ASYM, int STYPE>
int wide_launch(const GemvParams& P, size_t act_region, int act_row, int red_off, cudaStream_t st, bool* taken) {
  const RingPlan wp = plan_ring(P, act_region, true);
  // two producer warps on alternate stages need an even ring; a ring too short for two consumer warps is not worth the SM
  if (!(wp.stages >= 2 && wp.stages % 2 == 0 && wp.active >= 2)) return NS_OK;
  *taken = true;
  if (P.norm_w && !P.act_f32) {
    ns_set_error("gemv_ring: fused RMSNorm needs fp32 activations");
    return NS_E_INVALID;
  }
  const bool nrm = (P.norm_w || P.one_image) && P.act_f32;
  constexpr int NC = 2 * kConsumers;
  if (wp.rows == 2)
    return nrm ? launch_rows<AMODE, 1, ASYM, STYPE, 2, true, NC>(P, wp, act_region, act_row, red_off, st)
               : launch_rows<AMODE, 1, ASYM, STYPE, 2, false, NC>(P, wp, act_region, act_row, red_off, st);
  return nrm ? launch_rows<AMODE, 1, ASYM, STYPE, 1, true, NC>(P, wp, act_region, act_row, red_off, st)
             : launch_rows<AMODE, 1, ASYM, STYPE, 1, false, NC>(P, wp, act_region, act_row, red_off, st);
}

template <int AMODE, bool ASYM>
int wide_s(const GemvParams& P, size_t act_region, int act_row, int red_off, cudaStream_t st, bool* taken) {
  switch (P.stype) {
    case NS_S_F32: return wide_launch<AMODE, ASYM, NS_S_F32>(P, act_region, act_row, red_off, st, taken);
    case NS_S_F16: return wide_launch<AMODE, ASYM, NS_S_F16>(P, act_region, act_row, red_off, st, taken);
    default: return wide_launch<AMODE, ASYM, NS_S_BF16>(P, act_region, act_row, red_off, st, taken);
  }
}

}  // namespace

// *taken = false: no plan for this shape on the wide kernel, the caller launches the two-CTA kernel
int ns_launch_gemv_ring_wide(const GemvParams& P, int amode, bool asym, size_t act_region, int act_row, int red_off, cudaStream_t st,
                             bool* taken) {
  *taken = false;
  if (amode == A_U8) return asym ? wide_s<A_U8, true>(P, act_region, act_row, red_off, st, taken) : wide_s<A_U8, false>(P, act_region, act_row, red_off, st, taken);
  return asym ? wide_s<A_S8, true>(P, act_region, act_row, red_off, st, taken) : wide_s<A_S8, false>(P, act_region, act_row, red_off, st, taken);
}

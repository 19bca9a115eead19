// gemv_ring.cu -- the decode GEMV for 4-bit integer weights with 8-bit integer activations (ggml Q4_0 x Q8_0 and BesTLA
// int4 CompInt8) and for ggml Q8_0 weights: HBM -> shared-memory ring via TMA bulk copies, dp4a out of shared memory.
//
// Replaces the same reference functions as gemv.cu (ne_vec_dot_q4_0_q8_0, core/layers/vec_dot.h:131; gemv_4bit_u8s8_fp32 /
// gemv_4bit_s8s8_fp32, bestla/bestla/kernel_ref.h:2372/2432) and ne_vec_dot_q8_0_q8_0 (vec_dot.h:594) for M <= 4.
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

// Shared-memory plan.  Candidates: row pairs or single rows per stage, half an SM (two CTAs per SM) or a whole SM.  The score
// is the number of consumer warps per SM that own a stage; pairs share the activation loads between two rows (measured:
// K = 11008 with 7 pair stages beats 14 single-row stages, 950 vs 937 tok/s), so single rows are only taken when pairs would
// leave consumer warps without a stage (K >= ~14000).  Ties go to the deeper ring.
RingPlan plan_ring(int pitch, int mode, size_t act_region, bool wide) {
  static const int env_budget = getenv("NS_RING_BUDGET_KB") ? atoi(getenv("NS_RING_BUDGET_KB")) : 0;  // tuning aids
  static const int env_rows = getenv("NS_RING_ROWS") ? atoi(getenv("NS_RING_ROWS")) : 0;
  const size_t budgets[2] = {(size_t)(env_budget > 0 ? env_budget : 113) * 1024, 200 * 1024};
  RingPlan best = {0, 0, 0, 0, 0, -1.0};
  for (int rows = 2; rows >= 1; --rows) {
    if (rows == 1 && mode == NS_GEMV_GATE_UP_SILU) continue;  // the gate/up epilogue needs both rows in one warp
    if (env_rows && rows != env_rows && !(env_rows == 1 && mode == NS_GEMV_GATE_UP_SILU)) continue;
    const int stage_bytes = rows * pitch;
    for (int i = 0; i < 2; ++i) {
      if (wide && i == 0) continue;  // the 14-consumer-warp kernel owns the SM
      const int kc = (wide && i == 1) ? 2 * kConsumers : kConsumers;
      int raw = 0;
      if (budgets[i] > act_region + 64) raw = (int)((budgets[i] - act_region - 64) / (stage_bytes + 16));
      if (raw > (wide ? 56 : 32)) raw = wide ? 56 : 32;
      const int ac = raw < kc ? raw : kc;
      if (ac < 1) continue;
      const int st = raw - raw % ac;  // one consumer warp per stage residue class (see kernel)
      const int ctas = i == 0 ? 2 : 1;
      const double score = ctas * ac * (rows == 2 ? 1.1 : 1.0) + 0.001 * st;
      if (score > best.score) best = RingPlan{rows, st, ac, ctas, budgets[i], score};
    }
  }
  return best;
}

}  // namespace

// The one place that decides how a ring launch runs (see nsb.cuh); the launchers below and ns_route both ask it.
bool ns_gemv_ring_choose(int kpad, int pitch, int mode, int mt, bool fused, bool norm, RingChoice* c) {
  c->act_row = (int)ns_round_up((size_t)kpad, 1024);
  const size_t img_end = (size_t)mt * c->act_row + (size_t)mt * ns_meta_stride(kpad) * 8;
  c->red_off = (int)ns_round_up(img_end, 16);  // one float per consumer warp (<= 14) of reduction scratch behind the image
  c->act_region = ns_round_up(norm ? (size_t)c->red_off + 64 : img_end, 128);
  // Single-row launches that quantise their activations themselves run on the one-CTA-per-SM kernel with 14 consumer warps
  // (gemv_ring_wide.cu: the activation row is read and quantised once per SM); pre-quantised images stay on the two-CTA kernel.
  // NS_RING_WIDE=0 / 1 forces the choice.
  static const int env_wide = getenv("NS_RING_WIDE") ? atoi(getenv("NS_RING_WIDE")) : -1;
  if (mt == 1 && (env_wide == 1 || (env_wide < 0 && fused))) {
    c->plan = plan_ring(pitch, mode, c->act_region, true);
    // two producer warps on alternate stages need an even ring; a ring too short for two consumer warps is not worth the SM
    c->wide = c->plan.stages >= 2 && c->plan.stages % 2 == 0 && c->plan.active >= 2;
    if (c->wide) return true;
  }
  c->wide = false;
  c->plan = plan_ring(pitch, mode, c->act_region, false);
  return c->plan.stages >= 1;
}

namespace {

template <int AMODE, int M, bool ASYM, int STYPE, bool W8 = false>
int launch_one(const GemvParams& P, int mt, cudaStream_t st) {
  RingChoice c;
  if (!ns_gemv_ring_choose(P.kpad, P.pitch, P.mode, mt, P.act_f32 != nullptr, P.norm_w != nullptr, &c)) {
    ns_set_error("gemv_ring: row pitch %d too large for shared memory", P.pitch);
    return NS_E_UNSUPPORTED;
  }
  if constexpr (M == 1) {
    if (c.wide) return W8 ? ns_launch_gemv_ring_wide_q8_0(P, c, st) : ns_launch_gemv_ring_wide(P, AMODE, ASYM, c, st);
  }
  const RingPlan& plan = c.plan;
  const size_t act_region = c.act_region;
  const int act_row = c.act_row, red_off = c.red_off;
  if constexpr (M <= 2) {  // the norm is only ever folded into launches of <= 2 rows (norm_foldable, abi.cu)
    if ((P.norm_w || P.one_image) && P.act_f32) {
      if (plan.rows == 2) return launch_rows<AMODE, M, ASYM, STYPE, 2, true, kConsumers, W8>(P, plan, act_region, act_row, red_off, st);
      return launch_rows<AMODE, M, ASYM, STYPE, 1, true, kConsumers, W8>(P, plan, act_region, act_row, red_off, st);
    }
  }
  if (P.norm_w) {  // (one_image without fp32 activations or with 4 rows simply takes the plain kernel)
    ns_set_error("gemv_ring: fused RMSNorm needs fp32 activations and <= 2 rows");
    return NS_E_INVALID;
  }
  if (plan.rows == 2) return launch_rows<AMODE, M, ASYM, STYPE, 2, false, kConsumers, W8>(P, plan, act_region, act_row, red_off, st);
  return launch_rows<AMODE, M, ASYM, STYPE, 1, false, kConsumers, W8>(P, plan, act_region, act_row, red_off, st);
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

// ggml Q8_0: one combination only (s8 activations, symmetric, fp16 scales), 1-, 2- and 4-row templates
int ns_launch_gemv_ring_q8_0(const GemvParams& P, int mt, cudaStream_t st) {
  switch (mt) {
    case 1: return launch_one<A_S8, 1, false, NS_S_F16, true>(P, mt, st);
    case 2: return launch_one<A_S8, 2, false, NS_S_F16, true>(P, mt, st);
    default: return launch_one<A_S8, 4, false, NS_S_F16, true>(P, mt, st);
  }
}

// gemv.cu -- decode-shape (M <= 4) weight-only matmul: launcher + the register-staged GEMV used for the formats the
// TMA-ring kernel (gemv_ring.cu) does not cover: fp32/bf16 compute (BesTLA CompFp32/CompBf16), NF4 and BesTLA 8-bit weights.
//
// Replaces, for M <= 4 (the reference's own GEMV cut-off, bestla_wrapper.h:283/568 "M<=4"):
//   ggml   ne_compute_forward_mul_mat_q_f32 + ne_vec_dot_q4_0_q8_0   (core/ne_layers.c:7085, core/layers/vec_dot.h:131)
//   BesTLA LauncherIntKBlock::run -> GEMVWrapper::gemv -> gemv_4bit_u8s8_fp32 / _s8s8_ / _fp32_fp32
//          (bestla/bestla/bestla_wrapper.h:568-729, bestla/bestla/kernel_ref.h:2372-2531)
//   and the fused callers ne_mul_qkv / ne_ffn_silu (core/layers/ip_fusion_qkv.cpp:194, ip_fusion_ffn.cpp:734).
//
// This kernel: one warp owns a PAIR of weight rows at a time; lanes stride K in 32-element chunks (16 B of nibbles,
// ld.global.nc.L1::no_allocate.v4), 2 rows x U=4 chunks in flight per lane; activations staged once per CTA in shared
// memory in the byte image act_prep.cu produced.  fp32 modes: w = (float)(q - zp) * scale (or lut[q] * scale), FMA.
// Roofline: HBM.  Algorithmic bytes per launch = N*K*bits/8 + N*ceil(K/g)*(scale_bytes [+1 if asym]).
#include "nsb.cuh"

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int U = 4;                        // chunks per row per lane per batch
constexpr size_t kSmemMax = 200 * 1024;     // dynamic shared memory the kernels are set up for (launch_one)

template <int WFMT>
struct WChunk {  // one 32-element chunk of one row
  uint4 a;
};
template <>
struct WChunk<NS_W_S8> {
  uint4 a, b;
};

template <int WFMT, bool ASYM>
struct Batch {
  WChunk<WFMT> w[2][U];
  float s[2][U];
  int z[2][U];
};

struct RowRef {
  const uint8_t* row;  // start of the NSB row
  long long out;       // element offset in dst for m == 0
  bool valid;
};

__device__ __forceinline__ void resolve_pair(const GemvParams& P, int p, RowRef rr[2]) {
  if (P.mode == NS_GEMV_GATE_UP_SILU) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      rr[r].row = P.rows[r] + (size_t)p * P.pitch;
      rr[r].out = (long long)p;
      rr[r].valid = true;
    }
    return;
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    int row = 2 * p + r;
    int wi = 0;
    if (P.nw > 1 && row >= P.n[0]) {
      row -= P.n[0];
      wi = 1;
      if (P.nw > 2 && row >= P.n[1]) {
        row -= P.n[1];
        wi = 2;
      }
    }
    const bool valid = row < P.n[wi];
    if (!valid) row = P.n[wi] - 1;
    rr[r].row = P.rows[wi] + (size_t)row * P.pitch;
    rr[r].out = P.dst_off[wi] + row;
    rr[r].valid = valid;
  }
}

template <int WFMT, bool ASYM>
__device__ __forceinline__ void load_batch(const GemvParams& P, const RowRef rr[2], int b, int lane, int nchunks,
                                           Batch<WFMT, ASYM>& B) {
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int c = lane + 32 * (b * U + u);
    const bool ok = c < nchunks;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      if (ok) {
        if constexpr (WFMT == NS_W_S8) {
          const uint4* src = reinterpret_cast<const uint4*>(rr[r].row) + 2 * c;
          B.w[r][u].a = ld_nc_v4(src);
          B.w[r][u].b = ld_nc_v4(src + 1);
        } else {
          B.w[r][u].a = ld_nc_v4(reinterpret_cast<const uint4*>(rr[r].row) + c);
        }
        const int gi = (P.cpg == 1) ? c : c / P.cpg;
        B.s[r][u] = ns_scale_at(rr[r].row + P.sc_off, P.stype, gi);
        if (ASYM) B.z[r][u] = (int)(signed char)rr[r].row[P.zp_off + gi];
      } else {
        B.w[r][u].a = make_uint4(0, 0, 0, 0);
        if constexpr (WFMT == NS_W_S8) B.w[r][u].b = make_uint4(0, 0, 0, 0);
        B.s[r][u] = 0.f;
        if (ASYM) B.z[r][u] = 0;
      }
    }
  }
}

__device__ __forceinline__ float dq_s4(uint32_t w, int idx, int off) {
  // element idx (0..7) of an NSB4 word: e(2j) = bits[4j..4j+3], e(2j+1) = bits[4j+16..4j+19]
  const int sh = ((idx >> 1) << 2) + ((idx & 1) << 4);
  return (float)((int)((w >> sh) & 0xF) - off);
}

template <int WFMT, int AMODE, int M, bool ASYM>
__global__ void __launch_bounds__(kThreads, 2) gemv_kernel(const GemvParams P) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ float lut_s[16];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nchunks = P.kpad >> 5;
  const int nbatches = (nchunks + 32 * U - 1) / (32 * U);
  const int warps_total = gridDim.x * kWarps;
  const int gw = blockIdx.x * kWarps + warp;

  pdl_launch_dependents();

  Batch<WFMT, ASYM> B;
  RowRef rr[2];
  int pair = gw;
  if (pair < P.npairs) {
    resolve_pair(P, pair, rr);
    load_batch<WFMT, ASYM>(P, rr, 0, lane, nchunks, B);  // weights do not depend on the previous kernel
  }

  pdl_wait();  // activations (and dst/residual) are produced by earlier kernels

  {
    const uint4* src = reinterpret_cast<const uint4*>(P.act);
    uint4* dstv = reinterpret_cast<uint4*>(smem);
    const int nvec = P.act_bytes >> 4;
    for (int i = threadIdx.x; i < nvec; i += kThreads) dstv[i] = src[i];
    if (WFMT == NS_W_NF4 && threadIdx.x < 16) lut_s[threadIdx.x] = NS_F4_LUT[P.f4kind][threadIdx.x];
  }
  __syncthreads();
  const int2* meta_s = reinterpret_cast<const int2*>(smem + P.meta_off);

  bool first = true;
  for (; pair < P.npairs; pair += warps_total) {
    if (!first) resolve_pair(P, pair, rr);
    float acc[2][M];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int m = 0; m < M; ++m) acc[r][m] = 0.f;

    for (int b = 0; b < nbatches; ++b) {
      if (!(first && b == 0)) load_batch<WFMT, ASYM>(P, rr, b, lane, nchunks, B);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int c = lane + 32 * (b * U + u);
        if (c >= nchunks) continue;
        if constexpr (AMODE != A_F32) {
          // ---------------- integer path: exact chunk dots via dp4a ----------------
          uint32_t lo[2][4], hi[2][4];
          int su[2] = {0, 0};
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            if constexpr (WFMT == NS_W_S8) {
              const WChunk<NS_W_S8>& wc = B.w[r][u];
              lo[r][0] = wc.a.x; lo[r][1] = wc.a.y; lo[r][2] = wc.a.z; lo[r][3] = wc.a.w;
              hi[r][0] = wc.b.x; hi[r][1] = wc.b.y; hi[r][2] = wc.b.z; hi[r][3] = wc.b.w;
            } else {
              const uint4 w = B.w[r][u].a;
              const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                lo[r][i] = ww[i] & 0x0F0F0F0Fu;
                hi[r][i] = (ww[i] >> 4) & 0x0F0F0F0Fu;
              }
            }
            if (AMODE == A_U8) {
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                su[r] = dp4a_ss(0x01010101, (int)lo[r][i], su[r]);
                su[r] = dp4a_ss(0x01010101, (int)hi[r][i], su[r]);
              }
            }
          }
#pragma unroll
          for (int m = 0; m < M; ++m) {
            const uint4* ap = reinterpret_cast<const uint4*>(smem + (size_t)m * P.kpad) + 2 * c;
            const uint4 a0 = ap[0], a1 = ap[1];
            const int2 mt = meta_s[m * P.meta_stride + c];
            const float a_scale = __int_as_float(mt.x);
            const int sa = (int)(short)(mt.y & 0xffff);
            const int za = (mt.y >> 16) & 0xff;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
              int ps = 0;
              if constexpr (WFMT == NS_W_S8) {
                // natural order: lo = k 0..15, hi = k 16..31
                if (AMODE == A_U8) {
                  ps = dp4a_us(a0.x, (int)lo[r][0], ps); ps = dp4a_us(a0.y, (int)lo[r][1], ps);
                  ps = dp4a_us(a0.z, (int)lo[r][2], ps); ps = dp4a_us(a0.w, (int)lo[r][3], ps);
                  ps = dp4a_us(a1.x, (int)hi[r][0], ps); ps = dp4a_us(a1.y, (int)hi[r][1], ps);
                  ps = dp4a_us(a1.z, (int)hi[r][2], ps); ps = dp4a_us(a1.w, (int)hi[r][3], ps);
                } else {
                  ps = dp4a_ss((int)a0.x, (int)lo[r][0], ps); ps = dp4a_ss((int)a0.y, (int)lo[r][1], ps);
                  ps = dp4a_ss((int)a0.z, (int)lo[r][2], ps); ps = dp4a_ss((int)a0.w, (int)lo[r][3], ps);
                  ps = dp4a_ss((int)a1.x, (int)hi[r][0], ps); ps = dp4a_ss((int)a1.y, (int)hi[r][1], ps);
                  ps = dp4a_ss((int)a1.z, (int)hi[r][2], ps); ps = dp4a_ss((int)a1.w, (int)hi[r][3], ps);
                }
              } else {
                // NSB4: word i pairs with activation words (Alo_i, Ahi_i) = ((a0,a4,a1,a5),(a2,a6,a3,a7)) of 8-group i
                if (AMODE == A_U8) {
                  ps = dp4a_uu(a0.x, lo[r][0], ps); ps = dp4a_uu(a0.y, hi[r][0], ps);
                  ps = dp4a_uu(a0.z, lo[r][1], ps); ps = dp4a_uu(a0.w, hi[r][1], ps);
                  ps = dp4a_uu(a1.x, lo[r][2], ps); ps = dp4a_uu(a1.y, hi[r][2], ps);
                  ps = dp4a_uu(a1.z, lo[r][3], ps); ps = dp4a_uu(a1.w, hi[r][3], ps);
                } else {
                  ps = dp4a_ss((int)a0.x, (int)lo[r][0], ps); ps = dp4a_ss((int)a0.y, (int)hi[r][0], ps);
                  ps = dp4a_ss((int)a0.z, (int)lo[r][1], ps); ps = dp4a_ss((int)a0.w, (int)hi[r][1], ps);
                  ps = dp4a_ss((int)a1.x, (int)lo[r][2], ps); ps = dp4a_ss((int)a1.y, (int)hi[r][2], ps);
                  ps = dp4a_ss((int)a1.z, (int)lo[r][3], ps); ps = dp4a_ss((int)a1.w, (int)hi[r][3], ps);
                }
              }
              // sum (a - za)(u - off) = sum a*u - off*Sa - za*(Su - 32*off);  off = 8 + zp (4-bit) or zp (8-bit)
              int off = (WFMT == NS_W_S8) ? 0 : 8;
              if (ASYM) off += B.z[r][u];
              int isum = ps - off * sa;
              if (AMODE == A_U8) isum -= za * (su[r] - 32 * off);
              acc[r][m] = fmaf((float)isum, a_scale * B.s[r][u], acc[r][m]);
            }
          }
        } else {
          // ---------------- fp32 path: w = (float)(q - zp) * scale (or lut[q] * scale), fp32 FMA ----------------
#pragma unroll
          for (int i = 0; i < 4; ++i) {  // 8 elements per step
            float wv[2][8];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
              const float s = B.s[r][u];
              if constexpr (WFMT == NS_W_S8) {
                const WChunk<NS_W_S8>& wc = B.w[r][u];
                const uint32_t w0 = (i == 0) ? wc.a.x : (i == 1) ? wc.a.z : (i == 2) ? wc.b.x : wc.b.z;
                const uint32_t w1 = (i == 0) ? wc.a.y : (i == 1) ? wc.a.w : (i == 2) ? wc.b.y : wc.b.w;
                const int zz = ASYM ? B.z[r][u] : 0;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  wv[r][e] = (float)((int)(signed char)((w0 >> (8 * e)) & 0xff) - zz) * s;
                  wv[r][4 + e] = (float)((int)(signed char)((w1 >> (8 * e)) & 0xff) - zz) * s;
                }
              } else {
                const uint4 w = B.w[r][u].a;
                const uint32_t ww = (i == 0) ? w.x : (i == 1) ? w.y : (i == 2) ? w.z : w.w;
                if (WFMT == NS_W_NF4) {
#pragma unroll
                  for (int e = 0; e < 8; ++e) {
                    const int sh = ((e >> 1) << 2) + ((e & 1) << 4);
                    wv[r][e] = lut_s[(ww >> sh) & 0xF] * s;
                  }
                } else {
                  const int off = 8 + (ASYM ? B.z[r][u] : 0);
#pragma unroll
                  for (int e = 0; e < 8; ++e) wv[r][e] = dq_s4(ww, e, off) * s;
                }
              }
            }
#pragma unroll
            for (int m = 0; m < M; ++m) {
              const float4* ap = reinterpret_cast<const float4*>(smem) + ((size_t)m * P.kpad + (size_t)c * 32 + i * 8) / 4;
              const float4 x0 = ap[0], x1 = ap[1];
              const float xa[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
              for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int e = 0; e < 8; ++e) acc[r][m] = fmaf(xa[e], wv[r][e], acc[r][m]);
            }
          }
        }
      }
    }
    first = false;

#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int m = 0; m < M; ++m) acc[r][m] = warp_sum(acc[r][m]);
    if (lane == 0) {
      if (P.mode == NS_GEMV_GATE_UP_SILU) {
#pragma unroll
        for (int m = 0; m < M; ++m) {
          if (m < P.m) {
            const float g = acc[0][m], up = acc[1][m];
            const float sg = P.eltop == NS_ELT_GELU ? ns_gelu(g) : ns_silu(g);  // kernel_ref.h:1569-1576
            if (P.aux) P.aux[(size_t)m * P.ldo + rr[0].out] = sg;
            P.dst[(size_t)m * P.ldo + rr[0].out] = sg * up;
          }
        }
      } else {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          if (!rr[r].valid) continue;
#pragma unroll
          for (int m = 0; m < M; ++m) {
            if (m < P.m) {
              const size_t o = (size_t)m * P.ldo + rr[r].out;
              float v = acc[r][m];
              if (P.bias) v += P.bias_bcast ? P.bias[rr[r].out] : P.bias[o];
              if (P.eltop == NS_ELT_GELU) v = ns_gelu(v);
              if (P.residual) v += P.residual[o];
              P.dst[o] = v;
            }
          }
        }
      }
    }
  }
}

template <int WFMT, int AMODE, int M, bool ASYM>
int launch_one(const GemvParams& P, size_t smem, cudaStream_t st) {
  auto kern = gemv_kernel<WFMT, AMODE, M, ASYM>;
  static bool attr_set = false;
  if (!attr_set) {
    NS_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemMax));
    attr_set = true;
  }
  const int need = (P.npairs + kWarps - 1) / kWarps;
  const int ctas_per_sm = smem > 100 * 1024 ? 1 : 2;
  int grid = ns_num_sms() * ctas_per_sm;
  if (grid > need) grid = need;
  if (grid < 1) grid = 1;
  NS_CUDA_TRY(ns_launch_pdl(kern, dim3(grid), dim3(kThreads), smem, st, P));
  ns_count_launch();
  return NS_OK;
}

template <int WFMT, int AMODE, bool ASYM>
int launch_m(const GemvParams& P, int mt, size_t smem, cudaStream_t st) {
  switch (mt) {
    case 1: return launch_one<WFMT, AMODE, 1, ASYM>(P, smem, st);
    case 2: return launch_one<WFMT, AMODE, 2, ASYM>(P, smem, st);
    default: return launch_one<WFMT, AMODE, 4, ASYM>(P, smem, st);
  }
}

template <int WFMT, int AMODE>
int launch_asym(const GemvParams& P, bool asym, int mt, size_t smem, cudaStream_t st) {
  return asym ? launch_m<WFMT, AMODE, true>(P, mt, smem, st) : launch_m<WFMT, AMODE, false>(P, mt, smem, st);
}

// Bytes of one activation row in the register GEMV's shared-memory image (fp32 values, or int8 codes + chunk meta)
size_t act_row_bytes(const ns_weight* w) {
  return (w->wfmt == NS_W_S4 || w->wfmt == NS_W_Q8_0) ? ns_round_up((size_t)w->kpad, 1024) : (size_t)w->kpad;
}
bool float_mode(const ns_weight* w) { return w->comp == NS_COMP_F32 || w->comp == NS_COMP_BF16; }
// Dynamic shared memory of a register-GEMV launch with an mt-row kernel template
size_t gemv_smem(const ns_weight* w, int mt) {
  const size_t s = float_mode(w) ? (size_t)mt * w->kpad * 4
                                 : ns_round_up((size_t)mt * act_row_bytes(w), 16) + (size_t)mt * ns_meta_stride(w->kpad) * 8;
  return ns_round_up(s, 16);
}

}  // namespace

// Largest activation-row tile one GEMV launch can take for this weight (bounded by shared memory).
int ns_gemv_tile_rows(const ns_weight* w) {
  const bool fmode = (w->comp == NS_COMP_F32 || w->comp == NS_COMP_BF16);
  const size_t per_row =
      fmode ? (size_t)w->kpad * 4 : ns_round_up((size_t)w->kpad, 1024) + (size_t)ns_meta_stride(w->kpad) * 8;
  int mt = 4;
  // int8 activations of 4 rows must leave room for a useful ring next to them (two CTAs per SM)
  const size_t cap = fmode ? 96 * 1024 : 64 * 1024;
  while (mt > 1 && per_row * mt > cap) mt >>= 1;
  return mt;
}

// One tile: m <= ns_gemv_tile_rows(w).  act_ws is the image ns_launch_act_prep produced for exactly these m rows.
// dst points at the tile's first output row; m_total is the full M (only used for the [nw][M][ldo] QKV layout).
bool ns_gemv_fused_quant_ok(const ns_weight* w) {
  if (!(w->wfmt == NS_W_S4 || w->wfmt == NS_W_Q8_0) || w->shuffle) return false;
  if (!(w->comp == NS_COMP_Q8_0 || w->comp == NS_COMP_INT8 || w->comp == NS_COMP_INT8_S8)) return false;
  const int qg = w->comp == NS_COMP_Q8_0 ? 32 : w->group;  // one activation block must sit inside one warp
  return (qg == 32 || qg == 64 || qg == 128 || qg == 256) && w->k % qg == 0;
}

int ns_gemv_check(const ns_weight* const* ws_, int nw, int mode) {
  const ns_weight* w0 = ws_[0];
  for (int i = 1; i < nw; ++i) {
    const ns_weight* wi = ws_[i];
    if (wi->k != w0->k || wi->group != w0->group || wi->wfmt != w0->wfmt || wi->stype != w0->stype ||
        wi->comp != w0->comp || wi->asym != w0->asym || wi->f4kind != w0->f4kind || wi->shuffle != nullptr || w0->shuffle != nullptr) {
      ns_set_error("fused matmul: weights differ in format (or use act-order shuffles)");
      return NS_E_UNSUPPORTED;
    }
  }
  if (w0->wfmt == NS_W_Q6K) {
    ns_set_error("Q6_K weights support the plain matmul only");
    return NS_E_UNSUPPORTED;
  }
  if (mode == NS_GEMV_GATE_UP_SILU && (nw != 2 || ws_[0]->n != ws_[1]->n)) {
    ns_set_error("gate/up fusion needs two weights with equal n");
    return NS_E_INVALID;
  }
  if (w0->group % 32 != 0 && w0->group != w0->k) {
    ns_set_error("group size %d is not a multiple of 32", w0->group);
    return NS_E_UNSUPPORTED;
  }
  if (w0->wfmt == NS_W_NF4 && !(w0->comp == NS_COMP_F32 || w0->comp == NS_COMP_BF16)) {
    ns_set_error("NF4 weights need a float compute type");
    return NS_E_UNSUPPORTED;
  }
  for (int i = 0; mode == NS_GEMV_CONCAT && i + 1 < nw; ++i)
    if (ws_[i]->n & 1) {
      ns_set_error("fused matmul: every weight but the last needs an even n");
      return NS_E_UNSUPPORTED;
    }
  // the register GEMV stages a whole activation row in shared memory: fp32 compute takes K <= 51200
  if (!ns_ring_format(w0) && gemv_smem(w0, 1) > kSmemMax) {
    ns_set_error("GEMV: one activation row of k=%d needs %zu B of shared memory, more than the %zu B the kernel has", w0->k,
                 gemv_smem(w0, 1), kSmemMax);
    return NS_E_UNSUPPORTED;
  }
  return NS_OK;
}

int ns_gemv_planned(const ns_weight* const* ws, int nw, int mode, int m, bool norm) {
  const ns_weight* w0 = ws[0];
  (void)nw;
  if (!ns_ring_format(w0)) return NS_OK;  // the register GEMV: ns_gemv_check has sized its launch
  const int tile = ns_gemv_tile_rows(w0);
  const bool fused = ns_gemv_fused_quant_ok(w0);
  const int rows[2] = {m < tile ? m : tile, m % tile};  // the full tiles and the last one
  for (int t : rows) {
    if (t < 1) continue;
    RingChoice c;
    if (!ns_gemv_ring_choose(w0->kpad, w0->pitch, mode, t >= 3 ? 4 : t, fused, norm && fused, &c)) {
      ns_set_error("ring GEMV: no shared-memory plan for a %d-row tile of k=%d (row pitch %d B%s)", t, w0->k, w0->pitch,
                   mode == NS_GEMV_GATE_UP_SILU ? ", gate/up row pairs" : "");
      return NS_E_UNSUPPORTED;
    }
  }
  return NS_OK;
}

int ns_launch_gemv(const ns_weight* const* ws_, int nw, int mode, const void* act_ws, float* dst, int ldo, int m,
                   int m_total, const float* bias, int bias_bcast, const float* residual, float* aux, cudaStream_t st,
                   const float* act_f32, int lda, int eltop, const float* norm_w, float norm_eps, int one_image) {
  if (int rc = ns_gemv_check(ws_, nw, mode)) return rc;
  const ns_weight* w0 = ws_[0];
  if (m < 1 || m > ns_gemv_tile_rows(w0)) {
    ns_set_error("internal: GEMV tile of %d rows", m);
    return NS_E_INVALID;
  }
  const int kpad = w0->kpad;
  const bool fmode = float_mode(w0);
  const int amode = fmode ? A_F32 : (w0->comp == NS_COMP_INT8 ? A_U8 : A_S8);
  const int meta_stride = ns_meta_stride(kpad);

  GemvParams P = {};
  long long ntot = 0;
  for (int i = 0; i < nw; ++i) {
    P.rows[i] = ws_[i]->rows;
    P.n[i] = ws_[i]->n;
    // QKV convention of the reference: dst = [nw][M][ldo] (ip_fusion_qkv.cpp:84-86)
    P.dst_off[i] = (mode == NS_GEMV_CONCAT) ? (long long)i * m_total * ldo : 0;
    ntot += ws_[i]->n;
  }
  P.nw = nw;
  P.mode = mode;
  P.k = w0->k;
  P.kpad = kpad;
  P.group = w0->group;
  P.ngroups = w0->ngroups;
  P.stype = w0->stype;
  P.cpg = (w0->group + 31) / 32;
  P.pitch = w0->pitch;
  P.q_bytes = w0->q_bytes;
  P.sc_off = w0->sc_off;
  P.zp_off = w0->zp_off;
  P.dst = dst;
  P.ldo = ldo;
  P.m = m;
  P.bias = bias;
  P.bias_bcast = bias_bcast;
  P.residual = residual;
  P.aux = aux;
  P.npairs = (mode == NS_GEMV_GATE_UP_SILU) ? w0->n : (int)((ntot + 1) / 2);
  P.act = act_ws;
  P.act_f32 = act_f32;
  P.lda = lda;
  P.eltop = eltop;
  P.comp = w0->comp;
  P.f4kind = w0->f4kind;
  P.norm_w = norm_w;
  P.norm_eps = norm_eps;
  P.one_image = one_image;
  if (norm_w && !(act_f32 && ns_gemv_fused_quant_ok(w0))) {
    ns_set_error("internal: fused RMSNorm needs the fused activation quantiser");
    return NS_E_INVALID;
  }
  if (act_f32 && !(ns_gemv_fused_quant_ok(w0))) {
    ns_set_error("internal: fused activation quantisation not available for this weight");
    return NS_E_INVALID;
  }

  const int mt = m >= 3 ? 4 : m;  // kernel template rows (1, 2, 4)
  if (fmode) {
    P.act_bytes = (int)((size_t)m * kpad * 4);
    P.meta_off = 0;
    P.meta_stride = 0;
  } else {
    // int8 image: [m][act_row] bytes then [m][meta_stride] int2; 4-bit weights use the ring layout (act_prep.cu)
    P.meta_off = (int)ns_round_up((size_t)m * act_row_bytes(w0), 16);
    P.meta_stride = meta_stride;
    P.act_bytes = (int)(P.meta_off + (size_t)m * meta_stride * 8);
  }
  const size_t smem = gemv_smem(w0, mt);
  const bool asym = w0->asym != 0;
  if (w0->wfmt == NS_W_S4 && !fmode) return ns_launch_gemv_ring(P, amode, asym, mt, st);  // the hot decode path
  if (w0->wfmt == NS_W_Q8_0) return ns_launch_gemv_ring_q8_0(P, mt, st);                    // its 8-bit-code form
  if (w0->wfmt == NS_W_S4) return launch_asym<NS_W_S4, A_F32>(P, asym, mt, smem, st);
  if (w0->wfmt == NS_W_S8) {
    return amode == A_F32  ? launch_asym<NS_W_S8, A_F32>(P, asym, mt, smem, st)
           : amode == A_U8 ? launch_asym<NS_W_S8, A_U8>(P, asym, mt, smem, st)
                           : launch_asym<NS_W_S8, A_S8>(P, asym, mt, smem, st);
  }
  return launch_m<NS_W_NF4, A_F32, false>(P, mt, smem, st);
}

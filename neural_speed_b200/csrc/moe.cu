// moe.cu -- row gather / scatter around the expert-indexed matmul (ns_mul_mat_id, abi.cu).
//
// Reference: ne_compute_forward_mul_mat_id_q_f32 / _q_f32_bestla (core/ne_layers.c:7345-7498, :7783-7916) build per-expert
// row lists (matrix_rows[n_as][ne11]) on the host and then walk the tokens of every expert ONE AT A TIME (vec_dot per row,
// or bestla_f32f32_forward with m = 1): each token re-reads its expert's weights.  Here the tokens are sorted by expert
// once, the activation rows are gathered into that order, every expert runs ONE matmul over its contiguous slice (GEMV ring,
// integer tensor cores or wgmma by slice height -- the expert's weights are read once per node), and the result rows are
// scattered back.  Both kernels are plain coalesced row copies: HBM-bound, 2 x m x cols x 4 bytes.
#include "nsb.cuh"

namespace {

// dst[i][:] = src[idx[i]][:]   (GATHER)      dst[idx[i]][:] = src[i][:]   (!GATHER)
template <bool GATHER>
__global__ void __launch_bounds__(256) move_rows_kernel(const float* __restrict__ src, int ld_src, const int* __restrict__ idx,
                                                        float* __restrict__ dst, int ld_dst, int cols) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x;  // row (grid.x: up to 2^31 - 1 rows)
  const int t = idx[i];
  const float* s = src + (size_t)(GATHER ? t : i) * ld_src;
  float* d = dst + (size_t)(GATHER ? i : t) * ld_dst;
  const bool v4 = !(cols & 3) && !(ld_src & 3) && !(ld_dst & 3) && !((size_t)src & 15) && !((size_t)dst & 15);
  if (v4) {
    const int c4 = cols >> 2;
    for (int c = blockIdx.y * blockDim.x + threadIdx.x; c < c4; c += gridDim.y * blockDim.x)
      reinterpret_cast<float4*>(d)[c] = reinterpret_cast<const float4*>(s)[c];
  } else {
    for (int c = blockIdx.y * blockDim.x + threadIdx.x; c < cols; c += gridDim.y * blockDim.x) d[c] = s[c];
  }
}

}  // namespace

int ns_launch_move_rows(bool gather, const float* src, int ld_src, const int* idx_dev, float* dst, int ld_dst, int rows, int cols,
                        cudaStream_t st) {
  if (rows <= 0 || cols <= 0) return NS_OK;
  int bx = (cols / 4 + 255) / 256;
  if (bx < 1) bx = 1;
  if (bx > 8) bx = 8;
  const dim3 grid((unsigned)rows, (unsigned)bx);
  if (gather) NS_CUDA_TRY(ns_launch_pdl(move_rows_kernel<true>, grid, dim3(256), 0, st, src, ld_src, idx_dev, dst, ld_dst, cols));
  else NS_CUDA_TRY(ns_launch_pdl(move_rows_kernel<false>, grid, dim3(256), 0, st, src, ld_src, idx_dev, dst, ld_dst, cols));
  ns_count_launch();
  return NS_OK;
}

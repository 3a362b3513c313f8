// The Gram product of two stacked sample sets that the latent-space evaluation entry points share
// (smd_latent_stats in latent_stats.cu, smd_latent_coverage in latent_coverage.cu).
//
//   Z = [x - mean x; y - mean y; mean x; mean y]   (bf16 hi + lo halves, rows padded to the GEMM tile, K to 64)
//   G = Z Z^T                                      (three wgmma launches: lo*hi, hi*lo, then hi*hi on top, fp32)
//
// plus diag[r] = G_rr for the n + m data rows and |mean x - mean y|^2 from the fp64 column means.
#pragma once
#include "plan.cuh"

namespace smd {

static constexpr int kLatentMaxRows = 16384;   // n + m: the fp32 Gram of the stacked sets is (n + m + 2)^2 floats

struct GramLayout {
  int R, Rp, Kp;                  // stacked rows n + m + 2, padded rows, padded K
  size_t z, z_lo, g, mean, diag, delta2, total;   // byte offsets; total: end of the Gram region (256-aligned)
};

inline size_t align256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

GramLayout gram_layout(int n, int m, int d);

// Fills the Gram region of ws (laid out by L = gram_layout(n, m, d)) on st.  SMD_OK or SMD_ERR_CUDA.
int latent_gram(const float* x, int n, const float* y, int m, int d, const GramLayout& L, uint8_t* ws,
                cudaStream_t st);

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// fixed-order block sum (every thread gets the result); red holds one double per warp
__device__ __forceinline__ double block_sum_f64(double v, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  v = warp_sum_f64(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double r = 0.0;
  for (int w = 0; w < nw; ++w) r += red[w];
  return r;
}

}  // namespace smd

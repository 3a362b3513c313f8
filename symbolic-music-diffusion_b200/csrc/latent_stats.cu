// Latent-space evaluation statistics (utils/metrics.py:24-77): everything the Frechet distance and the RBF / polynomial
// MMDs need from two sample sets x (n, d) and y (m, d), out of one Gram product.
//
//   Z = [x - mean x; y - mean y; mean x; mean y]   (bf16 hi + lo halves, rows padded to the GEMM tile, K to 64)
//   G = Z Z^T                                      (three wgmma launches: lo*hi, hi*lo, then hi*hi on top, fp32)
//
// Every inner product and squared distance between raw rows follows from G without subtracting large numbers:
// distances come from centred rows (plus the mean-difference terms for x-y pairs), raw inner products add the
// mean rows back.  The two kernels are evaluated and summed in fp64 with a fixed-order reduction, so repeated calls
// are bitwise equal.  The centred x-y block of G, (x - mean x)(y - mean y)^T, is what the trace term of the Frechet
// distance needs: tr sqrtm(S1 S2) is the nuclear norm of that block over sqrt((n - 1)(m - 1)).
#include <algorithm>
#include <climits>
#include <cmath>

#include "latent_gram.cuh"

namespace smd {

static constexpr int kLatentRowsPad = kBM;     // Gram rows / columns padded to the GEMM's 128-row tile
static constexpr int kMeanCols = 32, kMeanSlices = 32;

GramLayout gram_layout(int n, int m, int d) {
  GramLayout L;
  L.R = n + m + 2;
  L.Rp = (L.R + kLatentRowsPad - 1) / kLatentRowsPad * kLatentRowsPad;
  L.Kp = static_cast<int>((static_cast<long long>(d) + 63) / 64 * 64);
  const size_t zb = static_cast<size_t>(L.Rp) * L.Kp * sizeof(__nv_bfloat16);
  size_t off = 0;
  L.z = off; off = align256(off + zb);
  L.z_lo = off; off = align256(off + zb);
  L.g = off; off = align256(off + static_cast<size_t>(L.Rp) * L.Rp * sizeof(float));
  L.mean = off; off = align256(off + 2 * static_cast<size_t>(d) * sizeof(double));
  L.diag = off; off = align256(off + static_cast<size_t>(n + m) * sizeof(double));
  L.delta2 = off; off = align256(off + sizeof(double));
  L.total = off;
  return L;
}

// smd_latent_stats' workspace: the Gram region, then the per-row kernel-sum partials
struct LatentLayout {
  GramLayout gram;
  size_t part, total;
};

static LatentLayout latent_layout(int n, int m, int d) {
  LatentLayout L;
  L.gram = gram_layout(n, m, d);
  L.part = L.gram.total;
  L.total = align256(L.part + static_cast<size_t>(n + m) * 4 * sizeof(double));
  return L;
}

// column means of x (blockIdx.y = 0) and y (1) in fp64: 32 columns per block, 32 row slices summed in order
__global__ void __launch_bounds__(kMeanCols * kMeanSlices)
latent_mean_kernel(const float* __restrict__ x, int n, const float* __restrict__ y, int m, int d,
                   double* __restrict__ mean) {
  __shared__ double part[kMeanSlices][kMeanCols + 1];
  const float* src = blockIdx.y ? y : x;
  const int rows = blockIdx.y ? m : n;
  const int cl = threadIdx.x % kMeanCols, sl = threadIdx.x / kMeanCols;
  const int c = blockIdx.x * kMeanCols + cl;
  double s = 0.0;
  if (c < d)
    for (int r = sl; r < rows; r += kMeanSlices) s += src[static_cast<size_t>(r) * d + c];
  part[sl][cl] = s;
  __syncthreads();
  if (sl == 0 && c < d) {
    double t = 0.0;
    for (int k = 0; k < kMeanSlices; ++k) t += part[k][cl];
    mean[static_cast<size_t>(blockIdx.y) * d + c] = t / rows;
  }
}

// Z = [x - mean x; y - mean y; mean x; mean y; 0...] as bf16 hi / lo halves, [Rp][Kp], four columns per thread
__global__ void __launch_bounds__(256)
latent_split_kernel(const float* __restrict__ x, int n, const float* __restrict__ y, int m, int d,
                    const double* __restrict__ mean, int Rp, int Kp, __nv_bfloat16* __restrict__ hi,
                    __nv_bfloat16* __restrict__ lo) {
  const size_t quads = static_cast<size_t>(Rp) * (Kp / 4);
  for (size_t q = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; q < quads;
       q += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(q / (Kp / 4));
    const int c0 = static_cast<int>(q - static_cast<size_t>(r) * (Kp / 4)) * 4;
    __align__(8) __nv_bfloat16 h[4], l[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = c0 + k;
      double v = 0.0;
      if (c < d) {
        if (r < n) v = x[static_cast<size_t>(r) * d + c] - mean[c];
        else if (r < n + m) v = y[static_cast<size_t>(r - n) * d + c] - mean[static_cast<size_t>(d) + c];
        else if (r < n + m + 2) v = mean[static_cast<size_t>(r - n - m) * d + c];
      }
      const float f = static_cast<float>(v);
      h[k] = __float2bfloat16_rn(f);
      l[k] = bf16_lo_part(f);
    }
    const size_t o = static_cast<size_t>(r) * Kp + c0;
    *reinterpret_cast<uint2*>(hi + o) = *reinterpret_cast<const uint2*>(h);
    *reinterpret_cast<uint2*>(lo + o) = *reinterpret_cast<const uint2*>(l);
  }
}

// diag[r] = |z_r|^2 for the n + m data rows, and |mean x - mean y|^2 from the fp64 means (one block)
__global__ void __launch_bounds__(1024)
latent_diag_kernel(const float* __restrict__ G, int Rp, int rows, const double* __restrict__ mean, int d,
                   double* __restrict__ diag, double* __restrict__ delta2) {
  __shared__ double red[32];
  for (int r = threadIdx.x; r < rows; r += blockDim.x) diag[r] = G[static_cast<size_t>(r) * Rp + r];
  double s = 0.0;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    const double e = mean[c] - mean[static_cast<size_t>(d) + c];
    s += e * e;
  }
  s = block_sum_f64(s, red);
  if (threadIdx.x == 0) *delta2 = s;
}

__device__ __forceinline__ double ipow(double b, int e) {
  double r = 1.0;
  while (true) {
    if (e & 1) r *= b;
    e >>= 1;
    if (!e) return r;
    b *= b;
  }
}

// One block per data row a of the stacked sets: the sums over its same-set columns and (rows of x) its y columns of
// exp(-rbf_gamma |a - b|^2) and (poly_gamma <a, b> + poly_coef0)^degree, into part[a][0..3] =
// (rbf same, rbf x-y, poly same, poly x-y).  With c_r the centred rows and u / v the mean rows of Z:
//   |a - b|^2 = G_aa + G_bb - 2 G_ab                                          (same set)
//             = G_aa + G_bb - 2 G_ab + |u - v|^2 + 2 <c_a - c_b, u - v>          (a in x, b in y)
//   <a, b>    = G_ab + <c_a, mean(b)> + <c_b, mean(a)> + <mean(a), mean(b)>
// Squared distances are clamped at 0 (as sklearn's euclidean_distances).
__global__ void __launch_bounds__(256)
latent_kernel_sums_kernel(const float* __restrict__ G, int Rp, int n, int m, const double* __restrict__ diag,
                          const double* __restrict__ delta2_p, double rbf_gamma, int degree, double poly_gamma,
                          double poly_coef0, double* __restrict__ part) {
  __shared__ double red[8];
  const int a = blockIdx.x;
  const bool ax = a < n;
  const float* Ga = G + static_cast<size_t>(a) * Rp;
  const float* Gu = G + static_cast<size_t>(n + m) * Rp;       // row of mean x
  const float* Gv = Gu + Rp;                                    // row of mean y
  const double gaa = diag[a], dau = Gu[a], dav = Gv[a];
  const double guu = Gu[n + m], gvv = Gv[n + m + 1], guv = Gu[n + m + 1];
  const double delta2 = *delta2_p;
  // same set: columns [b0, b1) with the mean row mm of a's set
  const int b0 = ax ? 0 : n, b1 = ax ? n : n + m;
  const float* Gm = ax ? Gu : Gv;
  const double dam = ax ? dau : dav, gmm = ax ? guu : gvv;
  double rs = 0.0, ps = 0.0;
  for (int b = b0 + threadIdx.x; b < b1; b += blockDim.x) {
    const double g = Ga[b];
    const double dist = fmax(gaa + diag[b] - 2.0 * g, 0.0);
    const double ip = g + dam + static_cast<double>(Gm[b]) + gmm;
    rs += exp(-rbf_gamma * dist);
    ps += ipow(poly_gamma * ip + poly_coef0, degree);
  }
  double rc = 0.0, pc = 0.0;
  if (ax) {
    const double dad = dau - dav;                               // <c_a, u - v>
    for (int b = n + threadIdx.x; b < n + m; b += blockDim.x) {
      const double g = Ga[b], gbu = Gu[b], gbv = Gv[b];
      const double dist = fmax(gaa + diag[b] - 2.0 * g + delta2 + 2.0 * (dad - (gbu - gbv)), 0.0);
      const double ip = g + dav + gbu + guv;
      rc += exp(-rbf_gamma * dist);
      pc += ipow(poly_gamma * ip + poly_coef0, degree);
    }
  }
  double* out = part + static_cast<size_t>(a) * 4;
  rs = block_sum_f64(rs, red);
  ps = block_sum_f64(ps, red);
  rc = block_sum_f64(rc, red);
  pc = block_sum_f64(pc, red);
  if (threadIdx.x == 0) { out[0] = rs; out[1] = rc; out[2] = ps; out[3] = pc; }
}

// stats (see smd.h) from the per-row partials, the diagonal and |delta|^2, each sum in row order (one block)
__global__ void __launch_bounds__(1024)
latent_finish_kernel(const double* __restrict__ part, const double* __restrict__ diag,
                     const double* __restrict__ delta2, int n, int m, double* __restrict__ stats) {
  __shared__ double red[32];
  double s[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // x: tr, rbf xx, rbf xy, poly xx, poly xy; y: tr, rbf yy, poly yy
  for (int a = threadIdx.x; a < n + m; a += blockDim.x) {
    const double* p = part + static_cast<size_t>(a) * 4;
    if (a < n) { s[0] += diag[a]; s[1] += p[0]; s[2] += p[1]; s[3] += p[2]; s[4] += p[3]; }
    else { s[5] += diag[a]; s[6] += p[0]; s[7] += p[2]; }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) s[k] = block_sum_f64(s[k], red);
  if (threadIdx.x == 0) {
    const double dn = n, dm = m;
    stats[0] = *delta2;
    stats[1] = s[0] / (dn - 1.0);
    stats[2] = s[5] / (dm - 1.0);
    stats[3] = s[1] / (dn * dn);
    stats[4] = s[6] / (dm * dm);
    stats[5] = s[2] / (dn * dm);
    stats[6] = s[3] / (dn * dn);
    stats[7] = s[7] / (dm * dm);
    stats[8] = s[4] / (dn * dm);
  }
}

int latent_gram(const float* x, int n, const float* y, int m, int d, const GramLayout& L, uint8_t* ws,
                cudaStream_t st) {
  auto hi = reinterpret_cast<__nv_bfloat16*>(ws + L.z);
  auto lo = reinterpret_cast<__nv_bfloat16*>(ws + L.z_lo);
  float* G = reinterpret_cast<float*>(ws + L.g);
  double* mean = reinterpret_cast<double*>(ws + L.mean);
  double* diag = reinterpret_cast<double*>(ws + L.diag);
  double* delta2 = reinterpret_cast<double*>(ws + L.delta2);

  latent_mean_kernel<<<dim3((d + kMeanCols - 1) / kMeanCols, 2), kMeanCols * kMeanSlices, 0, st>>>(x, n, y, m, d, mean);
  CNT();
  const size_t quads = static_cast<size_t>(L.Rp) * (L.Kp / 4);
  const int split_blocks = static_cast<int>(std::min<size_t>((quads + 255) / 256, static_cast<size_t>(device_sm_count()) * 8));
  latent_split_kernel<<<split_blocks, 256, 0, st>>>(x, n, y, m, d, mean, L.Rp, L.Kp, hi, lo);
  CNT();
  SMD_LAUNCH_CHECK("latent_split");

  // G = Z Z^T in the strict (bf16x3) composition: G = lo hi^T; G += hi lo^T; G = hi hi^T + G
  GemmOp op;
  if (!make_gemm_op(&op, hi, static_cast<uint64_t>(L.Rp), hi, static_cast<uint64_t>(L.Rp), L.Rp, L.Kp, kBNMax, 0, 0,
                    0, 0, L.z_lo - L.z))
    return SMD_ERR_CUDA;
  GemmOp o1 = op; o1.tmA = op.tmA_lo;
  GemmEpilogue e = epi();
  e.out_f32 = G; e.ld_f32 = L.Rp;
  SMD_CUDA(launch_gemm(o1, L.Rp, e, st));
  GemmOp o2 = op; o2.tmB = op.tmB_lo;
  e.residual = G; e.ld_res = L.Rp;
  SMD_CUDA(launch_gemm(o2, L.Rp, e, st));
  SMD_CUDA(launch_gemm(op, L.Rp, e, st));

  latent_diag_kernel<<<1, 1024, 0, st>>>(G, L.Rp, n + m, mean, d, diag, delta2);
  CNT();
  SMD_LAUNCH_CHECK("latent_gram");
  return SMD_OK;
}

}  // namespace smd

using namespace smd;

extern "C" {

size_t smd_latent_stats_workspace_bytes(int n, int m, int d) {
  if (n < 2 || m < 2 || d < 1 || d > INT_MAX - 63 || n + m > kLatentMaxRows) return 0;
  return latent_layout(n, m, d).total;
}

int smd_latent_stats(const float* x, int n, const float* y, int m, int d, float rbf_gamma, int poly_degree,
                     float poly_gamma, float poly_coef0, void* workspace, size_t workspace_bytes, double* stats,
                     float* cross, smd_stream_t stream) {
  if (n < 2 || m < 2) { set_error("both sample sets need at least 2 rows"); return SMD_ERR_INVALID; }
  if (d < 1 || d > INT_MAX - 63) { set_error("d must be in [1, INT_MAX - 63]"); return SMD_ERR_INVALID; }
  if (poly_degree < 1) { set_error("poly_degree must be >= 1"); return SMD_ERR_INVALID; }
  if (n > kLatentMaxRows - m) {
    set_error("n + m must be <= " + std::to_string(kLatentMaxRows) + " (the Gram of the stacked sets)");
    return SMD_ERR_INVALID;
  }
  if (!x || !y || !workspace || !stats) { set_error("null argument"); return SMD_ERR_INVALID; }
  const LatentLayout L = latent_layout(n, m, d);
  if (workspace_bytes < L.total) {
    set_error("workspace too small: " + std::to_string(workspace_bytes) + " < " + std::to_string(L.total) + " bytes");
    return SMD_ERR_INVALID;
  }
  if (reinterpret_cast<uintptr_t>(workspace) & 255u) { set_error("workspace must be 256-byte aligned"); return SMD_ERR_INVALID; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const GramLayout& Lg = L.gram;
  if (const int rc = latent_gram(x, n, y, m, d, Lg, ws, st)) return rc;
  float* G = reinterpret_cast<float*>(ws + Lg.g);
  double* diag = reinterpret_cast<double*>(ws + Lg.diag);
  double* delta2 = reinterpret_cast<double*>(ws + Lg.delta2);
  double* part = reinterpret_cast<double*>(ws + L.part);
  latent_kernel_sums_kernel<<<n + m, 256, 0, st>>>(G, Lg.Rp, n, m, diag, delta2, rbf_gamma, poly_degree, poly_gamma,
                                                    poly_coef0, part);
  CNT();
  latent_finish_kernel<<<1, 1024, 0, st>>>(part, diag, delta2, n, m, stats);
  CNT();
  SMD_LAUNCH_CHECK("latent_stats");
  if (cross)
    SMD_CUDA(cudaMemcpy2DAsync(cross, static_cast<size_t>(m) * sizeof(float), G + n,
                               static_cast<size_t>(Lg.Rp) * sizeof(float), static_cast<size_t>(m) * sizeof(float), n,
                               cudaMemcpyDeviceToDevice, st));
  return SMD_OK;
}

}  // extern "C"

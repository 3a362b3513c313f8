// CUDA-core (SIMT) kernels of the DDPM hot path: everything that is not a large GEMM.
// All are HBM/latency-bound; they use coalesced vector access and warp-level reductions.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <cstdlib>
#include "ptx.cuh"

namespace smd {


// ---------------------------------------------------------------------------------------------------
// helpers
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// swish(v) = v * sigmoid(v) with sigmoid(v) = 0.5 + 0.5 * tanh(v / 2): one MUFU.TANH instead of exp + IEEE divide
// (abs error of tanh.approx ~5e-4; every consumer rounds the result to bf16 or feeds a bf16 GEMM operand)
__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float swishf(float v) {
  const float h = 0.5f * v;
  return fmaf(h, tanh_approx(h), h);
}
// Strict-precision mode (SMD precision = bf16x3): every bf16 tensor-core operand x is kept as the pair
// (hi = bf16(x), lo = bf16(x - hi)); lo lives `lo_delta` elements behind hi (0 = mode off) and the GEMMs add the
// hi*lo + lo*hi cross terms, so products carry ~16 mantissa bits.  Activations then use the accurate functions.
__device__ __forceinline__ __nv_bfloat16 bf16_lo_part(float x) {
  return __float2bfloat16_rn(x - __bfloat162float(__float2bfloat16_rn(x)));
}
__device__ __forceinline__ float swish_exact(float v) { return v / (1.0f + expf(-v)); }
__device__ __forceinline__ float swish_grad(float v) {  // d/dv [v * sigmoid(v)] = s * (1 + v * (1 - s))
  const float s = fmaf(0.5f, tanh_approx(0.5f * v), 0.5f);
  return s * fmaf(v, 1.0f - s, 1.0f);
}
// tf32 mma.sync helpers (attention forward / backward)
__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void mma_tf32_16x8x8(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float gelu_tanh_grad(float x) {
  const float c = 0.7978845608028654f;
  const float u = c * (x + 0.044715f * x * x * x);
  const float th = tanhf(u);
  return 0.5f * (1.0f + th) + 0.5f * x * (1.0f - th * th) * c * (1.0f + 3.0f * 0.044715f * x * x);
}

// threefry2x32 (20 rounds) -- jax.random's block function (jax 0.2.8; SURVEY Appendix B.3)
__device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
__device__ __forceinline__ void threefry2x32(uint32_t k0, uint32_t k1, uint32_t& x0, uint32_t& x1) {
  const uint32_t ks[3] = {k0, k1, k0 ^ k1 ^ 0x1BD11BDAu};
  x0 += ks[0]; x1 += ks[1];
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    if ((i & 1) == 0) {
      x0 += x1; x1 = rotl32(x1, 13); x1 ^= x0;
      x0 += x1; x1 = rotl32(x1, 15); x1 ^= x0;
      x0 += x1; x1 = rotl32(x1, 26); x1 ^= x0;
      x0 += x1; x1 = rotl32(x1, 6);  x1 ^= x0;
    } else {
      x0 += x1; x1 = rotl32(x1, 17); x1 ^= x0;
      x0 += x1; x1 = rotl32(x1, 29); x1 ^= x0;
      x0 += x1; x1 = rotl32(x1, 16); x1 ^= x0;
      x0 += x1; x1 = rotl32(x1, 24); x1 ^= x0;
    }
    x0 += ks[(i + 1) % 3];
    x1 += ks[(i + 2) % 3] + static_cast<uint32_t>(i + 1);
  }
}
// element `idx` of jax.random._random_bits(key, 32, (n,)): counters are split in halves (padded to even)
__device__ __forceinline__ uint32_t jax_random_bits(uint32_t k0, uint32_t k1, uint32_t idx, uint32_t n) {
  const uint32_t half = (n + 1u) >> 1;
  uint32_t x0, x1;
  if (idx < half) {
    x0 = idx; x1 = idx + half; if (x1 >= n) x1 = 0u;  // odd n: the pad counter is 0
    threefry2x32(k0, k1, x0, x1);
    return x0;
  }
  x0 = idx - half; x1 = idx;
  threefry2x32(k0, k1, x0, x1);
  return x1;
}
// XLA's float32 ErfInv (Giles) and jax.random.normal's transform
__device__ __forceinline__ float erfinv_giles(float x) {
  float w = -logf((1.0f - x) * (1.0f + x));
  float p;
  if (w < 5.0f) {
    w = w - 2.5f;
    p = 2.81022636e-08f;
    p = 3.43273939e-07f + p * w;
    p = -3.5233877e-06f + p * w;
    p = -4.39150654e-06f + p * w;
    p = 0.00021858087f + p * w;
    p = -0.00125372503f + p * w;
    p = -0.00417768164f + p * w;
    p = 0.246640727f + p * w;
    p = 1.50140941f + p * w;
  } else {
    w = sqrtf(w) - 3.0f;
    p = -0.000200214257f;
    p = 0.000100950558f + p * w;
    p = 0.00134934322f + p * w;
    p = -0.00367342844f + p * w;
    p = 0.00573950773f + p * w;
    p = -0.0076224613f + p * w;
    p = 0.00943887047f + p * w;
    p = 1.00167406f + p * w;
    p = 2.83297682f + p * w;
  }
  return p * x;
}
__device__ __forceinline__ float jax_normal_from_bits(uint32_t bits) {
  const float u01 = __uint_as_float((bits >> 9) | 0x3F800000u) - 1.0f;
  const float lo = -0.99999994f;                 // nextafter(-1, 0)
  float u = __fadd_rn(__fmul_rn(u01, __fsub_rn(1.0f, lo)), lo);  // u * (maxval - minval) + minval, unfused
  u = fmaxf(lo, u);
  return 1.41421356237f * erfinv_giles(u);
}

// Grid cap of the grid-stride kernels (256-thread CTAs): 8 CTAs per SM of a 148-SM part, which still covers every SM of
// an H100.  Every timing of these kernels was taken with this cap, so changing it is a performance change of its own.
static constexpr int kGridStrideMaxBlocks = 148 * 8;
inline int grid_stride_blocks(size_t n) {
  const size_t blocks = (n + 255) / 256;
  return static_cast<int>(blocks < kGridStrideMaxBlocks ? blocks : kGridStrideMaxBlocks);
}

// ---------------------------------------------------------------------------------------------------
// kernels (definitions in kernels.cu)
// ---------------------------------------------------------------------------------------------------
// x_t = sqrt(ua[b]) * x0 + sqrt(1 - ua[b]) * eps ; cond[b] = sqrt(ua[b])        (utils/losses.py:295-300)
void launch_q_sample(const float* x0, const float* eps, const float* used_alpha, float* xt, float* cond, int B,
                     int per_sample, cudaStream_t st, const float* const* ind = nullptr, int mode = 0);
// mode 1 (denoising score matching, utils/losses.py:163-165): xt = x0 + sigma[b] * eps ; cond[b] = sigma[b]

// h[m,:] = x[m,:] @ W_in + b_in + posenc[m % S,:]; a[m,:] = bf16(LN(h[m,:]; g, b))   (models/ncsn.py:155-160)
void launch_embed(const float* x, const float* W_in, const float* b_in, const float* posenc, const float* ln_g,
                  const float* ln_b, float* h, __nv_bfloat16* a, int M, int C, int S, cudaStream_t st,
                  long long lo_delta = 0);

// multi-head self-attention over S in {32, 64, 128} positions (flax.nn.SelfAttention core, models/ncsn.py:161)
// qkv fp32 [M][3E] -> o bf16 [M][E];  optionally saves the probabilities P [B][H][S][S] fp32 for backward.
// causal (S = 32 only; models/autoregressive.py:61, causal_mask=True): query i sees keys j <= i, masked P exactly 0.
// Returns cudaErrorInvalidValue (and launches nothing) for a length / mask combination without a kernel.
cudaError_t launch_attention(const float* qkv, __nv_bfloat16* o, float* probs_or_null, int B, int S, int H,
                             cudaStream_t st, long long lo_delta = 0, bool causal = false);

// out[m,:] = bf16( act( film( LN(u[m,:]; stats, g, b) ) ) )                        (models/shared.py:62-64,66-68)
// stats[m] = (sum, sumsq) over the N columns; scale/shift rows selected by m / S (or row 0 if film_bcast)
void launch_ln_film_act(const float* u, const float* stats, const float* g, const float* b, const float* scale,
                        const float* shift, int film_ld, int film_bcast, int act, __nv_bfloat16* out, int M, int N,
                        int S, cudaStream_t st, const int* film_row_dev = nullptr,
                        const __nv_bfloat16* u16 = nullptr,    // u16: the LayerNorm input stored as bf16 (u == null)
                        long long lo_delta = 0,
                        // part != null: the row statistics are the producing GEMM's per-tile partials
                        // part[(row * nslots + s) * 2], added here in slot order; the totals go to stats_out (or null)
                        const float* part = nullptr, int nslots = 0, float* stats_out = nullptr);

// enc[r, j] = sin((5000 t_r) f_j), enc[r, 64 + j] = cos(...)                          (models/ncsn.py:25-41)
void launch_noise_encoding(const float* t, const float* freqs, float* enc, int R, cudaStream_t st);

// y[r, n] = act(sum_k x[r,k] W[k,n] + b[n]), all fp32, small R (FiLM generator, models/ncsn.py:47-61)
void launch_small_linear(const float* x, const float* W, const float* b, float* y, int R, int K, int N, int act,
                         cudaStream_t st, float* pre_act_out = nullptr);

// tiled fp32 SGEMM (mode 0: A.B, 1: A.B^T, 2: A^T.B) with bias / pre-activation save / swish / * swish'(mul_pre)
void launch_sgemm_small(int mode, const float* A, const float* B, const float* bias, float* C, float* pre_out,
                        const float* mul_pre, int M, int N, int K, int act, cudaStream_t st);

// bf16 dst[r * ld + c] = src[r * cols + c] for c < cols (columns cols .. ld-1 are left as they are)
void launch_pad_cast_bf16(const float* src, __nv_bfloat16* dst, int rows, int cols, int ld, cudaStream_t st,
                          long long lo_delta = 0);
// bf16 dst[i] = src[i]
void launch_cast_bf16(const float* src, __nv_bfloat16* dst, size_t n, cudaStream_t st, long long lo_delta = 0);

struct ReverseStepArgs {
  const float* x;          // state (N, S, C)
  const float* eps_hat;    // model output
  const float* z;          // supplied N(0,1) noise or null -> threefry(key)
  uint32_t key0, key1;     // jax noise key of this step
  const uint32_t* key_tab; // optional device table [T][4] = (noise k0,k1, infill k0,k1) indexed by step t
  const float* coef;       // device table [T][8]: sqrt_recip, sqrt_m1, mu1, mu2, sigma, sqrt_ap, sqrt_1m_ap, alpha_prod
  const int* slot_tab;     // device table [T]: collection slot or -1 (or null)
  const int* t_ptr;        // device scalar: current t (graph-replayable), or null -> t
  int t;
  const float* infill_x;   // or null
  const float* infill_mask;
  const float* infill_z;   // supplied infill noise or null -> threefry(infill key)
  float* x_next;
  float* collection;       // (41, N, S, C) or null
  float* metrics;          // device [4][T] accumulators (grad_norm, step_norm, alpha_prod, noise_norm); slot = T-1-t
  int N, S, C, T;
  // sharded sampling: this call holds samples [rng_first / (S*C), ...) of a global batch of rng_total / (S*C) samples
  // and draws exactly that slice of the global threefry streams (0 / 0: the local batch is the whole batch)
  uint32_t rng_first, rng_total;
};
// One body of the reverse-diffusion scan after the network call (utils/ebm_utils.py:332-394)
void launch_reverse_step(const ReverseStepArgs& a, cudaStream_t st);
// *t_ptr -= 1 ; cond[0..n) = coef[t].sqrt_ap   (device-side step bookkeeping for graph replay)
void launch_step_advance(int* t_ptr, cudaStream_t st);
void launch_fill_cond(const float* coef, const int* t_ptr, float* cond, int n, cudaStream_t st);

// loss[b] = mean_{s,c} (eps - pred)^2 ; dpred = -2 (eps - pred) * gscale                (utils/losses.py:304-308)
void launch_ddpm_loss(const float* eps, const float* pred, float* loss_per_example, float* dpred_or_null,
                      float gscale, int B, int per_sample, cudaStream_t st, const float* dsm_sigma = nullptr);
// dsm_sigma != null: denoising score matching, loss[b] = 0.5 sum((pred + eps / sigma)^2) sigma^2 with pred = score

void launch_scale_rows(float* y, const float* sigma, int bcast, int B, int per, cudaStream_t st);

// ---- sliced score matching (utils/losses.py:182-247): tangent (Jacobian-vector product) pass of DenseNCSN ----
// d/dz swish(z) and d2/dz2 swish(z) with an exact sigmoid (s): s (1 + z (1 - s)) and s (1 - s) (2 + z (1 - 2 s))
__device__ __forceinline__ float sigmoid_exact(float z) { return 1.0f / (1.0f + expf(-z)); }
// NV sums over the CTA (blockDim.x a multiple of 32); every thread receives the totals
template <int NV>
__device__ __forceinline__ void block_sums(float (&v)[NV], float (&red)[NV][32]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    v[j] = warp_sum(v[j]);
    if (lane == 0) red[j][warp] = v[j];
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    float t = 0.f;
    for (int w = 0; w < nw; ++w) t += red[j][w];
    v[j] = t;
  }
  __syncthreads();
}
// Tangent of out = act(film(LN(x))) along xt: with xh = (x - mean) rstd from the PRIMAL row statistics (sum, sumsq),
//   xh' = rstd (xt - mean(xt) - xh mean(xh xt)),  y' = gamma xh',  z' = scale y',  out' = swish'(z) z'  (bf16).
// x: the primal LayerNorm input, fp32 (x32) or bf16 (x16); ss: FiLM [rows / S][film_ld] = [scale | shift] or null.
void launch_ln_film_tangent(const float* x32, const __nv_bfloat16* x16, const float* stats, const float* xt,
                            const float* g, const float* b, const float* ss, int film_ld, int act, __nv_bfloat16* out,
                            int M, int N, int S, cudaStream_t st, long long lo_delta);
// out = bf16(v) (+ lo halves); ind (graph replay) overrides v with ind[3]
void launch_tangent_input(const float* v, const float* const* ind, __nv_bfloat16* out, size_t n, cudaStream_t st,
                          long long lo_delta);
// Per example b (f = raw network output, ft its tangent along v, sg = sigma[b]):
//   loss[b] = 0.5 |f|^2 + sg v.ft  (= (0.5 |s|^2 + v.J_s v) sg^2 with s = f / sg);  score <- f / sg;  hvp[b] <- v.ft / sg.
// Training (df32 != null): the adjoint seeds df = f / global_batch (fp32 + bf16 padded to Cp) and dft = sg v / global_batch
// (bf16 padded), and loss_sum[0..1] as smd_ddpm_grads (summed in example order by the last block).
void launch_ssm_loss(const float* f, const float* ft, const float* v, const float* sigma, const float* const* ind,
                     float* loss, float* score, float* hvp, float* loss_sum, unsigned int* done_counter, float inv_gb,
                     float* df32, __nv_bfloat16* df16, __nv_bfloat16* dft16, int B, int C, int Cp, cudaStream_t st);

struct LangevinStepArgs {
  const float* x; const float* grad; const float* z;   // z: supplied N(0,1) or null -> threefry(key)
  uint32_t key0, key1, ikey0, ikey1;
  float alpha, noise_coef, infill_sigma;
  const float* infill_x; const float* infill_mask; const float* infill_z;
  float* x_next; float* collection_slot; float* metrics;   // metrics: 4 floats (accumulated; zero them first)
  int N, S, C;
};
void launch_langevin_step(const LangevinStepArgs& a, cudaStream_t st);

}  // namespace smd

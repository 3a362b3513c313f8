// Training-side pieces of libsmd: fused clip + Adam (+EMA), EMA update.
// (The backward pass itself lives in backward.cu.)
#include "plan.cuh"

namespace smd {

// ---------------------------------------------------------------------------------------------------
// fused global-norm clip + Adam (+ EMA)        (train_ncsn.py:284-287, flax.optim.Adam, train_utils.py:73-78)
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ g, long long n, float* __restrict__ out,
                                                    int vec_ok) {
  float s = 0.f;
  const long long n4 = vec_ok ? n / 4 : 0;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = g4[i];
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  for (long long i = n4 * 4 + blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    s += g[i] * g[i];
  __shared__ float red[8];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
    for (int j = 0; j < 8; ++j) v += red[j];
    out[1 + blockIdx.x] = v;   // per-block partial, no atomics: the total is summed in a fixed order by clip_adam_kernel,
  }                            // so every data-parallel rank derives bit-identical clip factors from identical gradients
}
static constexpr int kSumsqBlocks = 1023;   // partials live in scratch[1 .. 1023]; scratch[0] receives the total

__global__ void __launch_bounds__(256)
clip_adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                 float* __restrict__ ema, __nv_bfloat16* __restrict__ shadow, long long n, float lr, float max_norm, float b1, float b2, float eps,
                 float bc1, float bc2, float mu, float* __restrict__ sumsq, float* __restrict__ gnorm_out, int vec_ok) {
  __shared__ float nred[8];
  {
    float part = 0.f;
    for (int j = threadIdx.x; j < kSumsqBlocks; j += 256) part += sumsq[1 + j];   // fixed order in every block
    part = warp_sum(part);
    if ((threadIdx.x & 31) == 0) nred[threadIdx.x >> 5] = part;
    __syncthreads();
  }
  float total = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) total += nred[j];
  if (blockIdx.x == 0 && threadIdx.x == 0) sumsq[0] = total;
  const float norm = sqrtf(total);
  // jax.experimental.optimizers.clip_grads: g if norm < max else g * (max / norm)
  const float factor = (norm < max_norm) ? 1.0f : (max_norm / norm);
  if (blockIdx.x == 0 && threadIdx.x == 0 && gnorm_out) *gnorm_out = norm * factor;  // post-clip norm (train_ncsn.py:285)
  auto upd = [&](float gi, float& mi, float& vi, float& pi) {
    gi *= factor;
    mi = (1.0f - b1) * gi + b1 * mi;
    vi = (1.0f - b2) * gi * gi + b2 * vi;
    const float mh = mi / bc1, vh = vi / bc2;
    pi = pi - lr * mh / (sqrtf(vh) + eps);
  };
  // 16-byte accesses: five (six with EMA) independent streams per thread, the pass is HBM-bound
  const long long n4 = vec_ok ? n / 4 : 0;   // vec_ok: every arena is 16-byte aligned (8-byte for the bf16 shadow)
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 g4 = reinterpret_cast<const float4*>(g)[i];
    float4 m4 = reinterpret_cast<float4*>(m)[i], v4 = reinterpret_cast<float4*>(v)[i], p4 = reinterpret_cast<float4*>(p)[i];
    upd(g4.x, m4.x, v4.x, p4.x); upd(g4.y, m4.y, v4.y, p4.y); upd(g4.z, m4.z, v4.z, p4.z); upd(g4.w, m4.w, v4.w, p4.w);
    reinterpret_cast<float4*>(m)[i] = m4; reinterpret_cast<float4*>(v)[i] = v4; reinterpret_cast<float4*>(p)[i] = p4;
    if (shadow) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(p4.x, p4.y), hi = __floats2bfloat162_rn(p4.z, p4.w);
      uint2 pk;
      pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
      reinterpret_cast<uint2*>(shadow)[i] = pk;
    }
    if (ema) {
      float4 e4 = reinterpret_cast<float4*>(ema)[i];
      e4.x = e4.x * mu + p4.x * (1.0f - mu); e4.y = e4.y * mu + p4.y * (1.0f - mu);
      e4.z = e4.z * mu + p4.z * (1.0f - mu); e4.w = e4.w * mu + p4.w * (1.0f - mu);
      reinterpret_cast<float4*>(ema)[i] = e4;
    }
  }
  for (long long i = n4 * 4 + blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float mi = m[i], vi = v[i], pi = p[i];
    upd(g[i], mi, vi, pi);
    m[i] = mi; v[i] = vi; p[i] = pi;
    if (shadow) shadow[i] = __float2bfloat16_rn(pi);
    if (ema) ema[i] = ema[i] * mu + pi * (1.0f - mu);
  }
}

__global__ void ema_kernel(float* __restrict__ ema, const float* __restrict__ p, long long n, float mu) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    ema[i] = ema[i] * mu + p[i] * (1.0f - mu);
}

}  // namespace smd

using namespace smd;

extern "C" {

int smd_clip_adam(float* params, float* grads, float* adam_m, float* adam_v, float* ema_or_null,
                  void* bf16_shadow_or_null, long long n, float lr, int step, float max_norm, float beta1,
                  float beta2, float eps, float ema_mu, float* scratch, float* grad_norm_out, smd_stream_t stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n <= 0 || !scratch) { set_error("bad arguments"); return SMD_ERR_INVALID; }
  const int blocks = 148 * 8;
  auto al = [](const void* q, uintptr_t a) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) % a) == 0; };
  const int vec_ok = al(params, 16) && al(grads, 16) && al(adam_m, 16) && al(adam_v, 16) && al(ema_or_null, 16) &&
                     al(bf16_shadow_or_null, 8);
  sumsq_kernel<<<kSumsqBlocks, 256, 0, st>>>(grads, n, scratch, vec_ok);
  g_launches.fetch_add(1);
  const double t = static_cast<double>(step) + 1.0;
  const float bc1 = static_cast<float>(1.0 - pow(static_cast<double>(beta1), t));
  const float bc2 = static_cast<float>(1.0 - pow(static_cast<double>(beta2), t));
  clip_adam_kernel<<<blocks, 256, 0, st>>>(params, grads, adam_m, adam_v, ema_or_null,
                                           static_cast<__nv_bfloat16*>(bf16_shadow_or_null), n, lr, max_norm, beta1, beta2,
                                           eps, bc1, bc2, ema_mu, scratch, grad_norm_out, vec_ok);
  g_launches.fetch_add(1);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error(std::string("clip_adam: ") + cudaGetErrorString(e)); return SMD_ERR_CUDA; }
  return SMD_OK;
}

int smd_ema_update(float* ema, const float* params, long long n, float mu, smd_stream_t stream) {
  ema_kernel<<<148 * 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(ema, params, n, mu);
  g_launches.fetch_add(1);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error(std::string("ema: ") + cudaGetErrorString(e)); return SMD_ERR_CUDA; }
  return SMD_OK;
}

}  // extern "C"

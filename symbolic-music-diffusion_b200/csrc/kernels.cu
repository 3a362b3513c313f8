// SIMT kernels of the DDPM hot path (see kernels.cuh for the contract of each launcher).
#include <cstdlib>
#include "kernels.cuh"

namespace smd {

// ---------------------------------------------------------------------------------------------------
// q_sample (utils/losses.py:295-300)
// ---------------------------------------------------------------------------------------------------
// ind (optional): device table {x0, used_alpha, eps} that overrides the pointer arguments -- a captured CUDA graph of
// the train step reads its per-step inputs through it, so new input tensors do not force a re-capture
__global__ void q_sample_kernel(const float* __restrict__ x0, const float* __restrict__ eps,
                                const float* __restrict__ ua, float* __restrict__ xt, float* __restrict__ cond, int B,
                                int per_sample, const float* const* __restrict__ ind, int mode) {
  pdl_trigger();
  pdl_wait();
  if (ind) { x0 = ind[0]; ua = ind[1]; eps = ind[2]; }
  if (mode == 1) {
    // denoising score matching (utils/losses.py:163-165): x~ = x + sigma * eps, conditioned on sigma itself
    const size_t total1 = static_cast<size_t>(B) * per_sample;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total1;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
      const int b = static_cast<int>(i / per_sample);
      const float sg = ua[b];
      xt[i] = __fadd_rn(x0[i], __fmul_rn(sg, eps[i]));
      if (i % per_sample == 0) cond[b] = sg;
    }
    return;
  }
  const size_t total = static_cast<size_t>(B) * per_sample;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / per_sample);
    const float a = ua[b];
    const float sa = sqrtf(a), sb = sqrtf(1.0f - a);
    xt[i] = __fadd_rn(__fmul_rn(sa, x0[i]), __fmul_rn(sb, eps[i]));
    if (i % per_sample == 0) cond[b] = sa;
  }
}
void launch_q_sample(const float* x0, const float* eps, const float* used_alpha, float* xt, float* cond, int B,
                     int per_sample, cudaStream_t st, const float* const* ind, int mode) {
  const size_t total = static_cast<size_t>(B) * per_sample;
  q_sample_kernel<<<grid_stride_blocks(total), 256, 0, st>>>(x0, eps, used_alpha, xt, cond, B, per_sample, ind, mode);
}

// ---------------------------------------------------------------------------------------------------
// embed: C -> 128 projection + positional encoding + first LayerNorm (one warp per token)
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
embed_kernel(const float* __restrict__ x, const float* __restrict__ W, const float* __restrict__ bias,
             const float* __restrict__ posenc, const float* __restrict__ ln_g, const float* __restrict__ ln_b,
             float* __restrict__ h, __nv_bfloat16* __restrict__ a, int M, int C, int S, long long lo_delta) {
  pdl_trigger();
  pdl_wait();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= M) return;
  const int m = warp;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const float* xr = x + static_cast<size_t>(m) * C;
  for (int c0 = 0; c0 < C; c0 += 32) {
    const float xl = (c0 + lane < C) ? xr[c0 + lane] : 0.f;
    const int lim = min(32, C - c0);
    for (int cc = 0; cc < lim; ++cc) {
      const float xv = __shfl_sync(0xffffffffu, xl, cc);
      const float* wr = W + static_cast<size_t>(c0 + cc) * 128;
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = fmaf(xv, __ldg(wr + lane + 32 * j), acc[j]);
    }
  }
  const int s = m % S;
  float v[4];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int o = lane + 32 * j;
    v[j] = acc[j] + bias[o] + posenc[s * 128 + o];
    s1 += v[j]; s2 += v[j] * v[j];
    h[static_cast<size_t>(m) * 128 + o] = v[j];
  }
  s1 = warp_sum(s1); s2 = warp_sum(s2);
  const float mean = s1 * (1.0f / 128.0f);
  const float var = s2 * (1.0f / 128.0f) - mean * mean;
  const float rstd = rsqrtf(var + 1e-6f);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int o = lane + 32 * j;
    const float y = (v[j] - mean) * (rstd * ln_g[o]) + ln_b[o];
    a[static_cast<size_t>(m) * 128 + o] = __float2bfloat16_rn(y);
    if (lo_delta) a[static_cast<size_t>(m) * 128 + o + lo_delta] = bf16_lo_part(y);
  }
}
// Same arithmetic (channels accumulated in the same order -> bit-identical), but the projection matrix sits in shared
// memory and a warp carries 4 tokens at a time, so every weight read feeds 4 FMAs instead of 1 global load per FMA.
template <int TPW>
__global__ void __launch_bounds__(256)
embed_smem_kernel(const float* __restrict__ x, const float* __restrict__ W, const float* __restrict__ bias,
                  const float* __restrict__ posenc, const float* __restrict__ ln_g, const float* __restrict__ ln_b,
                  float* __restrict__ h, __nv_bfloat16* __restrict__ a, int M, int C, int S, long long lo_delta) {
  extern __shared__ __align__(16) float emb_w[];   // [C][128]
  pdl_trigger();
  // the weights are not written by the preceding kernel: stage them before waiting on it
  for (int i = threadIdx.x; i < C * 32; i += blockDim.x)
    reinterpret_cast<float4*>(emb_w)[i] = __ldg(reinterpret_cast<const float4*>(W) + i);
  pdl_wait();
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), nw = gridDim.x * (blockDim.x >> 5);
  float bo[4], go[4], eo[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) { bo[j] = bias[lane + 32 * j]; go[j] = ln_g[lane + 32 * j]; eo[j] = ln_b[lane + 32 * j]; }
  for (int m0 = gw * TPW; m0 < M; m0 += nw * TPW) {
    float acc[TPW][4];
#pragma unroll
    for (int t = 0; t < TPW; ++t)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[t][j] = 0.f;
    for (int c0 = 0; c0 < C; c0 += 32) {
      float xl[TPW];
#pragma unroll
      for (int t = 0; t < TPW; ++t)
        xl[t] = (c0 + lane < C && m0 + t < M) ? x[static_cast<size_t>(m0 + t) * C + c0 + lane] : 0.f;
      const int lim = min(32, C - c0);
      for (int cc = 0; cc < lim; ++cc) {
        const float* wr = emb_w + (c0 + cc) * 128 + lane;
        const float w0 = wr[0], w1 = wr[32], w2 = wr[64], w3 = wr[96];
#pragma unroll
        for (int t = 0; t < TPW; ++t) {
          const float xv = __shfl_sync(0xffffffffu, xl[t], cc);
          acc[t][0] = fmaf(xv, w0, acc[t][0]); acc[t][1] = fmaf(xv, w1, acc[t][1]);
          acc[t][2] = fmaf(xv, w2, acc[t][2]); acc[t][3] = fmaf(xv, w3, acc[t][3]);
        }
      }
    }
#pragma unroll
    for (int t = 0; t < TPW; ++t) {
      const int m = m0 + t;
      if (m >= M) break;
      const int s = m % S;
      float v[4];
      float s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int o = lane + 32 * j;
        v[j] = acc[t][j] + bo[j] + posenc[s * 128 + o];
        s1 += v[j]; s2 += v[j] * v[j];
        h[static_cast<size_t>(m) * 128 + o] = v[j];
      }
      s1 = warp_sum(s1); s2 = warp_sum(s2);
      const float mean = s1 * (1.0f / 128.0f);
      const float var = s2 * (1.0f / 128.0f) - mean * mean;
      const float rstd = rsqrtf(var + 1e-6f);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int o = lane + 32 * j;
        const float y = (v[j] - mean) * (rstd * go[j]) + eo[j];
        a[static_cast<size_t>(m) * 128 + o] = __float2bfloat16_rn(y);
        if (lo_delta) a[static_cast<size_t>(m) * 128 + o + lo_delta] = bf16_lo_part(y);
      }
    }
  }
}
void launch_embed(const float* x, const float* W_in, const float* b_in, const float* posenc, const float* ln_g,
                  const float* ln_b, float* h, __nv_bfloat16* a, int M, int C, int S, cudaStream_t st, long long lo_delta) {
  if (C <= 64 && (reinterpret_cast<uintptr_t>(W_in) & 15u) == 0) {
    int blocks = (M + 31) / 32;
    if (blocks > 148 * 4) blocks = 148 * 4;
    embed_smem_kernel<4><<<blocks, 256, static_cast<size_t>(C) * 128 * sizeof(float), st>>>(x, W_in, b_in, posenc, ln_g,
                                                                                          ln_b, h, a, M, C, S, lo_delta);
    return;
  }
  const int blocks = (M + 7) / 8;
  embed_kernel<<<blocks, 256, 0, st>>>(x, W_in, b_in, posenc, ln_g, ln_b, h, a, M, C, S, lo_delta);
}

// ---------------------------------------------------------------------------------------------------
// attention: one CTA per (sample, head group, 32-query block), one warp per head, lane = query position
// (S in {32, 64, 128}: the CTA stages all S rows of k and v and its 32 rows of q).
// CAUSAL: query i attends to keys j <= i only; the masked probabilities are exactly 0 (flax's -1e10 bias underflows
// to 0 in the softmax), so the stored-probability backward needs no change
// ---------------------------------------------------------------------------------------------------
template <int DH, int S, bool CAUSAL>
__device__ __forceinline__ void attention_simt(const float* __restrict__ qkv, __nv_bfloat16* __restrict__ o,
                                               float* __restrict__ probs, int B, int H, long long lo_delta) {
  pdl_trigger();
  pdl_wait();
  // a CTA owns HPB = blockDim.x / 32 heads of one sample (W = HPB * DH columns of k and v): small CTAs, several
  // resident per SM, so one CTA's global->shared fill overlaps another's math.  S = 32 keeps static tiles; longer
  // sequences stage S rows of k and v in dynamic shared memory (2 S W floats: over the 48 KB static limit at S = 128)
  __shared__ __align__(16) float sK32[S == 32 ? 32 * 128 : 1];
  __shared__ __align__(16) float sV32[S == 32 ? 32 * 128 : 1];
  extern __shared__ __align__(16) float att_kv[];
  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  const int HPB = blockDim.x >> 5, W = HPB * DH, W4 = W / 4;
  const int hb = blockIdx.y * HPB;
  const int q0 = S == 32 ? 0 : blockIdx.z * 32;   // first query row of this CTA
  float* sK = S == 32 ? sK32 : att_kv;
  float* sV = S == 32 ? sV32 : att_kv + S * W;
  const float* base = qkv + static_cast<size_t>(b) * S * 384;
  for (int i = tid; i < S * W4; i += blockDim.x) {
    const int row = i / W4, c4 = (i % W4) * 4, gc = hb * DH + c4;
    *reinterpret_cast<float4*>(&sK[row * W + c4]) = *reinterpret_cast<const float4*>(base + row * 384 + 128 + gc);
    *reinterpret_cast<float4*>(&sV[row * W + c4]) = *reinterpret_cast<const float4*>(base + row * 384 + 256 + gc);
  }
  __syncthreads();
  const int hl = tid >> 5, lane = tid & 31;
  const int h = hb + hl;
  if (h >= H) return;
  float q[DH];
  const float qs = rsqrtf(static_cast<float>(DH));
  const float* qr = base + (q0 + lane) * 384 + h * DH;
#pragma unroll
  for (int d = 0; d < DH; ++d) q[d] = qr[d] * qs;   // flax: query / sqrt(depth) before the dot
  float sc[S];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < S; ++j) {
    float s = 0.f;
    const float4* kr = reinterpret_cast<const float4*>(&sK[j * W + hl * DH]);
#pragma unroll
    for (int d4 = 0; d4 < DH / 4; ++d4) {
      const float4 k4 = kr[d4];   // one 16-byte broadcast read per 4 MACs
      s = fmaf(q[4 * d4], k4.x, s); s = fmaf(q[4 * d4 + 1], k4.y, s);
      s = fmaf(q[4 * d4 + 2], k4.z, s); s = fmaf(q[4 * d4 + 3], k4.w, s);
    }
    if (CAUSAL && j > q0 + lane) s = -INFINITY;
    sc[j] = s;
    mx = fmaxf(mx, s);
  }
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < S; ++j) { sc[j] = expf(sc[j] - mx); sum += sc[j]; }
  const float inv = 1.0f / sum;
  float acc[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) acc[d] = 0.f;
#pragma unroll
  for (int j = 0; j < S; ++j) {
    const float p = sc[j] * inv;
    sc[j] = p;
    const float4* vr = reinterpret_cast<const float4*>(&sV[j * W + hl * DH]);
#pragma unroll
    for (int d4 = 0; d4 < DH / 4; ++d4) {
      const float4 v4 = vr[d4];
      acc[4 * d4] = fmaf(p, v4.x, acc[4 * d4]); acc[4 * d4 + 1] = fmaf(p, v4.y, acc[4 * d4 + 1]);
      acc[4 * d4 + 2] = fmaf(p, v4.z, acc[4 * d4 + 2]); acc[4 * d4 + 3] = fmaf(p, v4.w, acc[4 * d4 + 3]);
    }
  }
  __nv_bfloat16* orow = o + (static_cast<size_t>(b) * S + q0 + lane) * 128 + h * DH;
#pragma unroll
  for (int d = 0; d < DH; d += 2) {
    *reinterpret_cast<__nv_bfloat162*>(orow + d) = __floats2bfloat162_rn(acc[d], acc[d + 1]);
    if (lo_delta) { orow[d + lo_delta] = bf16_lo_part(acc[d]); orow[d + 1 + lo_delta] = bf16_lo_part(acc[d + 1]); }
  }
  if (probs != nullptr) {
    float* pr = probs + ((static_cast<size_t>(b) * H + h) * S + q0 + lane) * S;
#pragma unroll
    for (int j = 0; j < S; j += 4) *reinterpret_cast<float4*>(pr + j) = make_float4(sc[j], sc[j + 1], sc[j + 2], sc[j + 3]);
  }
}
template <int DH, int S>
__global__ void attention_kernel(const float* __restrict__ qkv, __nv_bfloat16* __restrict__ o,
                                 float* __restrict__ probs, int B, int H, long long lo_delta) {
  attention_simt<DH, S, false>(qkv, o, probs, B, H, lo_delta);
}
template <int DH>
__global__ void causal_attention_kernel(const float* __restrict__ qkv, __nv_bfloat16* __restrict__ o,
                                        float* __restrict__ probs, int B, int H, long long lo_delta) {
  attention_simt<DH, 32, true>(qkv, o, probs, B, H, lo_delta);
}
// ---------------------------------------------------------------------------------------------------
// Tensor-core variant (DH % 8 == 0): same CTA / warp mapping, but Q K^T and P V run on mma.sync m16n8k8 tf32
// (a 32xSx16 problem per head is far below a wgmma tile; ~350 instructions per warp instead of ~2000 at S = 32):
// S / 8 n-tiles for Q K^T and S / 8 k-steps for P V.
// q, k, v are rounded to tf32 once while the CTA stages them in shared memory (row pitch = W + 4 words, so every
// fragment read is bank-conflict free); scores, softmax and the P V accumulation stay fp32.  The softmax output is
// fed to the second MMA straight from the accumulator registers: within each block of 8 keys, k-slot t holds key 2t
// and k-slot t+4 holds key 2t+1, and the V fragment is read with the same permutation (a sum over keys does not
// care about their order), so no shuffles are needed between the two products.
// ---------------------------------------------------------------------------------------------------
template <int DH, int S, bool CAUSAL>
__device__ __forceinline__ void attention_mma(const float* __restrict__ qkv, __nv_bfloat16* __restrict__ o,
                                              float* __restrict__ probs, int B, int H) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) uint32_t att_sm[];
  const int tid = threadIdx.x;
  const int HPB = blockDim.x >> 5, W = HPB * DH, W4 = W / 4, P = W + 4;
  uint32_t* sQ = att_sm;          // [32][P]: this CTA's query block
  uint32_t* sK = sQ + 32 * P;     // [S][P]
  uint32_t* sV = sK + S * P;      // [S][P]
  const int b = blockIdx.x, hb = blockIdx.y * HPB, q0 = S == 32 ? 0 : blockIdx.z * 32;
  const float qs = rsqrtf(static_cast<float>(DH));   // flax: query / sqrt(depth) before the dot
  const float* base = qkv + static_cast<size_t>(b) * S * 384;
  for (int i = tid; i < S * W4; i += blockDim.x) {
    const int row = i / W4, c4 = (i % W4) * 4, gc = hb * DH + c4;
    if (S == 32 || row < 32) {
      const float4 q4 = *reinterpret_cast<const float4*>(base + (q0 + row) * 384 + gc);
      *reinterpret_cast<uint4*>(&sQ[row * P + c4]) = make_uint4(to_tf32(q4.x * qs), to_tf32(q4.y * qs), to_tf32(q4.z * qs), to_tf32(q4.w * qs));
    }
    const float4 k4 = *reinterpret_cast<const float4*>(base + row * 384 + 128 + gc);
    const float4 v4 = *reinterpret_cast<const float4*>(base + row * 384 + 256 + gc);
    *reinterpret_cast<uint4*>(&sK[row * P + c4]) = make_uint4(to_tf32(k4.x), to_tf32(k4.y), to_tf32(k4.z), to_tf32(k4.w));
    *reinterpret_cast<uint4*>(&sV[row * P + c4]) = make_uint4(to_tf32(v4.x), to_tf32(v4.y), to_tf32(v4.z), to_tf32(v4.w));
  }
  __syncthreads();
  const int hl = tid >> 5, lane = tid & 31;
  const int h = hb + hl;
  if (h >= H) return;
  const int g = lane >> 2, t = lane & 3;
  const int hc = hl * DH;
  constexpr int NT = S / 8;   // key tiles
  // ---- scores = (Q / sqrt(dh)) K^T : 2 m-tiles x S / 8 n-tiles, DH / 8 k-steps
  float sc[2][NT][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) sc[mt][nt][i] = 0.f;
#pragma unroll
  for (int ks = 0; ks < DH / 8; ++ks) {
    uint32_t a[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const uint32_t* q0 = sQ + (16 * mt + g) * P + hc + 8 * ks + t;
      a[mt][0] = q0[0]; a[mt][1] = q0[8 * P]; a[mt][2] = q0[4]; a[mt][3] = q0[8 * P + 4];
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const uint32_t* k0 = sK + (8 * nt + g) * P + hc + 8 * ks + t;
      const uint32_t b0 = k0[0], b1 = k0[4];
      mma_tf32_16x8x8(sc[0][nt], a[0], b0, b1);
      mma_tf32_16x8x8(sc[1][nt], a[1], b0, b1);
    }
  }
  if (CAUSAL) {   // key 8 nt + 2 t (+1) against query q0 + 16 mt + g (+8): the diagonal key keeps every row finite
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (8 * nt + 2 * t + (i & 1) > q0 + 16 * mt + g + 8 * (i >> 1)) sc[mt][nt][i] = -INFINITY;
  }
  // ---- row softmax: a row lives in the 4 lanes of a quad (t = 0..3), S / 4 values per lane
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {   // hr = 0: row 16 mt + g (c0, c1); hr = 1: row 16 mt + g + 8 (c2, c3)
      float mx = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) mx = fmaxf(mx, fmaxf(sc[mt][nt][2 * hr], sc[mt][nt][2 * hr + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      float sum = 0.f;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const float e0 = expf(sc[mt][nt][2 * hr] - mx), e1 = expf(sc[mt][nt][2 * hr + 1] - mx);
        sc[mt][nt][2 * hr] = e0; sc[mt][nt][2 * hr + 1] = e1;
        sum += e0 + e1;
      }
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      const float inv = 1.0f / sum;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) { sc[mt][nt][2 * hr] *= inv; sc[mt][nt][2 * hr + 1] *= inv; }
    }
  }
  if (probs != nullptr) {
    float* pr = probs + ((static_cast<size_t>(b) * H + h) * S + q0) * S;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        *reinterpret_cast<float2*>(pr + (16 * mt + g) * S + 8 * nt + 2 * t) = make_float2(sc[mt][nt][0], sc[mt][nt][1]);
        *reinterpret_cast<float2*>(pr + (16 * mt + g + 8) * S + 8 * nt + 2 * t) = make_float2(sc[mt][nt][2], sc[mt][nt][3]);
      }
  }
  // ---- O = P V : 2 m-tiles x DH / 8 n-tiles, S / 8 k-steps (one per block of 8 keys, permuted as described above)
  float acc[2][DH / 8][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int n2 = 0; n2 < DH / 8; ++n2)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mt][n2][i] = 0.f;
#pragma unroll
  for (int kb = 0; kb < NT; ++kb) {
    uint32_t a[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      a[mt][0] = to_tf32(sc[mt][kb][0]);   // (row g,     slot t)     = key 2t
      a[mt][1] = to_tf32(sc[mt][kb][2]);   // (row g + 8, slot t)
      a[mt][2] = to_tf32(sc[mt][kb][1]);   // (row g,     slot t + 4) = key 2t + 1
      a[mt][3] = to_tf32(sc[mt][kb][3]);   // (row g + 8, slot t + 4)
    }
#pragma unroll
    for (int n2 = 0; n2 < DH / 8; ++n2) {
      const uint32_t* v0 = sV + (8 * kb + 2 * t) * P + hc + 8 * n2 + g;
      const uint32_t b0 = v0[0], b1 = v0[P];
      mma_tf32_16x8x8(acc[0][n2], a[0], b0, b1);
      mma_tf32_16x8x8(acc[1][n2], a[1], b0, b1);
    }
  }
  __nv_bfloat16* ob = o + (static_cast<size_t>(b) * S + q0) * 128 + h * DH;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int n2 = 0; n2 < DH / 8; ++n2) {
      *reinterpret_cast<__nv_bfloat162*>(ob + (16 * mt + g) * 128 + 8 * n2 + 2 * t) = __floats2bfloat162_rn(acc[mt][n2][0], acc[mt][n2][1]);
      *reinterpret_cast<__nv_bfloat162*>(ob + (16 * mt + g + 8) * 128 + 8 * n2 + 2 * t) = __floats2bfloat162_rn(acc[mt][n2][2], acc[mt][n2][3]);
    }
}
template <int DH, int S>
__global__ void __launch_bounds__(128)
attention_mma_kernel(const float* __restrict__ qkv, __nv_bfloat16* __restrict__ o, float* __restrict__ probs, int B, int H) {
  attention_mma<DH, S, false>(qkv, o, probs, B, H);
}
template <int DH>
__global__ void __launch_bounds__(128)
causal_attention_mma_kernel(const float* __restrict__ qkv, __nv_bfloat16* __restrict__ o, float* __restrict__ probs,
                            int B, int H) {
  attention_mma<DH, 32, true>(qkv, o, probs, B, H);
}
// the kernel a launch runs: the causal variants exist for S = 32 only
template <int DH, int S, bool CAUSAL>
constexpr auto attention_simt_fn() {
  if constexpr (CAUSAL) return &causal_attention_kernel<DH>; else return &attention_kernel<DH, S>;
}
template <int DH, int S, bool CAUSAL>
constexpr auto attention_mma_fn() {
  if constexpr (CAUSAL) return &causal_attention_mma_kernel<DH>; else return &attention_mma_kernel<DH, S>;
}

template <int S, bool CAUSAL>
static void launch_attention_s(const float* qkv, __nv_bfloat16* o, float* probs_or_null, int B, int H, cudaStream_t st,
                               long long lo_delta) {
  const int dh = 128 / H;
  int hpb = H;
  while (hpb > 4 && hpb % 2 == 0) hpb /= 2;
  const dim3 grid(B, H / hpb, S / 32);
  const int threads = hpb * 32;
  if (lo_delta == 0 && dh % 8 == 0 && dh <= 32) {   // (strict mode: fp32 SIMT attention, no tf32 rounding)
    const size_t smem = (32 + 2 * S) * static_cast<size_t>(hpb * dh + 4) * sizeof(uint32_t);
#define SMD_ATT_MMA(DHV)                                                                                          \
  {                                                                                                               \
    static bool attr = false;                                                                                     \
    if (!attr) {                                                                                                  \
      cudaFuncSetAttribute(attention_mma_fn<DHV, S, CAUSAL>(), cudaFuncAttributeMaxDynamicSharedMemorySize,       \
                           (32 + 2 * S) * 132 * 4);                                                               \
      attr = true;                                                                                                \
    }                                                                                                             \
    attention_mma_fn<DHV, S, CAUSAL>()<<<grid, threads, smem, st>>>(qkv, o, probs_or_null, B, H);                 \
  }
    if (dh == 16) SMD_ATT_MMA(16)
    else if (dh == 8) SMD_ATT_MMA(8)
    else SMD_ATT_MMA(32)
#undef SMD_ATT_MMA
    return;
  }
  // S = 32: static shared memory; longer sequences: k and v for S rows in dynamic shared memory
  const size_t smem = S == 32 ? 0 : 2 * S * static_cast<size_t>(hpb * dh) * sizeof(float);
#define SMD_ATT_SIMT(DHV)                                                                                         \
  {                                                                                                               \
    static bool attr = false;                                                                                     \
    if (S != 32 && !attr) {                                                                                       \
      cudaFuncSetAttribute(attention_simt_fn<DHV, S, CAUSAL>(), cudaFuncAttributeMaxDynamicSharedMemorySize,      \
                           2 * S * 128 * 4);                                                                      \
      attr = true;                                                                                                \
    }                                                                                                             \
    attention_simt_fn<DHV, S, CAUSAL>()<<<grid, threads, smem, st>>>(qkv, o, probs_or_null, B, H, lo_delta);      \
  }
  if (dh == 16) SMD_ATT_SIMT(16)
  else if (dh == 8) SMD_ATT_SIMT(8)
  else if (dh == 32) SMD_ATT_SIMT(32)
  else if (dh == 4) SMD_ATT_SIMT(4)
#undef SMD_ATT_SIMT
}

cudaError_t launch_attention(const float* qkv, __nv_bfloat16* o, float* probs_or_null, int B, int S, int H,
                             cudaStream_t st, long long lo_delta, bool causal) {
  if (causal) {
    if (S != 32) return cudaErrorInvalidValue;
    launch_attention_s<32, true>(qkv, o, probs_or_null, B, H, st, lo_delta);
  } else if (S == 32) launch_attention_s<32, false>(qkv, o, probs_or_null, B, H, st, lo_delta);
  else if (S == 64) launch_attention_s<64, false>(qkv, o, probs_or_null, B, H, st, lo_delta);
  else if (S == 128) launch_attention_s<128, false>(qkv, o, probs_or_null, B, H, st, lo_delta);
  else return cudaErrorInvalidValue;
  return cudaSuccess;
}

// ---------------------------------------------------------------------------------------------------
// LayerNorm-apply + FiLM + activation -> bf16.  HBM-bound: the CTA streams its 32 rows (inside one sample when 32 | S)
// through a double-buffered shared-memory ring with bulk async copies (cp.async.bulk + mbarrier), 4 rows = up to
// 32 KB per copy, so ~64 KB per CTA are in flight without tying up registers.  Column-stationary compute:
// blockDim.x = N / 4 threads, each owning one float4 column group whose gamma / beta / scale / shift stay in
// registers; the row statistics come from the producing GEMM's epilogue, so there is no reduction.
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t k_smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void k_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(k_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void k_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(k_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void k_mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t}"
        : "=r"(ok)
        : "r"(k_smem_u32(bar)), "r"(parity)
        : "memory");
  }
}
__device__ __forceinline__ void k_bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   k_smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(k_smem_u32(bar))
               : "memory");
}

template <int MAXT, bool IN_BF16>
__global__ void __launch_bounds__(MAXT)
ln_film_act_kernel(const void* __restrict__ uin, const float* __restrict__ stats, const float* __restrict__ g,
                   const float* __restrict__ bta, const float* __restrict__ scale, const float* __restrict__ shift,
                   int film_ld, int film_bcast, int act, __nv_bfloat16* __restrict__ out, int M, int N, int S,
                   const int* __restrict__ film_row_dev, long long lo_delta, const float* __restrict__ part, int nslots,
                   float* __restrict__ stats_out) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(128) uint8_t lsm[];
  __shared__ float2 row_mr[32];   // (mean, rstd) of this CTA's 32 rows
  constexpr int RPG = 4;                                   // rows per copy group
  constexpr int ES = IN_BF16 ? 2 : 4;
  const uint32_t row_bytes = static_cast<uint32_t>(N) * ES;
  uint8_t* buf[2] = {lsm, lsm + RPG * row_bytes};
  uint64_t* bar = reinterpret_cast<uint64_t*>(lsm + 2 * RPG * row_bytes);
  const int c = threadIdx.x * 4;
  const int r0 = blockIdx.x * 32;
  const int nrows = min(32, M - r0);
  const int ngroups = (nrows + RPG - 1) / RPG;
  const uint8_t* src = static_cast<const uint8_t*>(uin) + static_cast<size_t>(r0) * row_bytes;
  if (threadIdx.x == 0) {
    k_mbar_init(&bar[0], 1);
    k_mbar_init(&bar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](int grp) {
    const int rows = min(RPG, nrows - grp * RPG);
    const uint32_t bytes = static_cast<uint32_t>(rows) * row_bytes;
    k_mbar_expect_tx(&bar[grp & 1], bytes);
    k_bulk_g2s(buf[grp & 1], src + static_cast<size_t>(grp) * RPG * row_bytes, bytes, &bar[grp & 1]);
  };
  if (threadIdx.x == 0) {
    issue(0);
    if (ngroups > 1) issue(1);
  }
  const float inv_n = 1.0f / static_cast<float>(N);
  if (threadIdx.x < 32) {
    // row statistics: either the (sum, sumsq) totals, or the producing GEMM's per-tile partials added in slot order
    // (bit-reproducible; the totals are handed on to the backward pass through stats_out)
    const int row = r0 + static_cast<int>(threadIdx.x);
    float t1 = 0.f, t2 = 0.f;
    if (row < M) {
      if (part != nullptr) {
        const float2* pp = reinterpret_cast<const float2*>(part) + static_cast<size_t>(row) * nslots;
        for (int s = 0; s < nslots; ++s) { const float2 p2 = pp[s]; t1 += p2.x; t2 += p2.y; }
        if (stats_out != nullptr) *reinterpret_cast<float2*>(stats_out + 2 * static_cast<size_t>(row)) = make_float2(t1, t2);
      } else {
        const float2 st = *reinterpret_cast<const float2*>(stats + 2 * static_cast<size_t>(row));
        t1 = st.x; t2 = st.y;
      }
    }
    const float mean = t1 * inv_n;
    row_mr[threadIdx.x] = make_float2(mean, rsqrtf(t2 * inv_n - mean * mean + 1e-6f));
  }
  __syncthreads();
  const float4 g4 = *reinterpret_cast<const float4*>(g + c);
  const float4 b4 = *reinterpret_cast<const float4*>(bta + c);
  const bool film = scale != nullptr;
  // a 32-row block lies inside one sample when S is a multiple of 32: its FiLM row is r0 / S
  const bool row_const_film = film && (film_row_dev != nullptr || film_bcast || S % 32 == 0);
  float4 s4 = make_float4(1.f, 1.f, 1.f, 1.f), h4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (row_const_film) {
    const size_t frow = film_row_dev ? static_cast<size_t>(*film_row_dev) : (film_bcast ? 0 : static_cast<size_t>(r0 / S));
    s4 = *reinterpret_cast<const float4*>(scale + frow * film_ld + c);
    h4 = *reinterpret_cast<const float4*>(shift + frow * film_ld + c);
  }
  for (int grp = 0; grp < ngroups; ++grp) {
    k_mbar_wait(&bar[grp & 1], static_cast<uint32_t>((grp >> 1) & 1));
    const uint8_t* sb = buf[grp & 1];
#pragma unroll
    for (int q = 0; q < RPG; ++q) {
      const int row = r0 + grp * RPG + q;
      if (row >= M) continue;
      float4 x;
      if (IN_BF16) {
        const uint2 raw = *reinterpret_cast<const uint2*>(sb + static_cast<size_t>(q) * row_bytes + static_cast<size_t>(c) * 2);
        const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.x));
        const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.y));
        x = make_float4(lo.x, lo.y, hi.x, hi.y);
      } else {
        x = *reinterpret_cast<const float4*>(sb + static_cast<size_t>(q) * row_bytes + static_cast<size_t>(c) * 4);
      }
      const float2 mr = row_mr[row - r0];
      const float mean = mr.x, rstd = mr.y;
      if (film && !row_const_film) {
        const size_t frow = static_cast<size_t>(row / S);
        s4 = *reinterpret_cast<const float4*>(scale + frow * film_ld + c);
        h4 = *reinterpret_cast<const float4*>(shift + frow * film_ld + c);
      }
      float y[4] = {(x.x - mean) * (rstd * g4.x) + b4.x, (x.y - mean) * (rstd * g4.y) + b4.y,
                    (x.z - mean) * (rstd * g4.z) + b4.z, (x.w - mean) * (rstd * g4.w) + b4.w};
      if (film) {
        y[0] = s4.x * y[0] + h4.x; y[1] = s4.y * y[1] + h4.y; y[2] = s4.z * y[2] + h4.z; y[3] = s4.w * y[3] + h4.w;
      }
      if (act == 2) {
#pragma unroll
        for (int i = 0; i < 4; ++i) y[i] = lo_delta ? swish_exact(y[i]) : swishf(y[i]);
      }
      __nv_bfloat162 p0 = __floats2bfloat162_rn(y[0], y[1]);
      __nv_bfloat162 p1 = __floats2bfloat162_rn(y[2], y[3]);
      uint2 pk;
      pk.x = *reinterpret_cast<uint32_t*>(&p0);
      pk.y = *reinterpret_cast<uint32_t*>(&p1);
      *reinterpret_cast<uint2*>(out + static_cast<size_t>(row) * N + c) = pk;
      if (lo_delta) {
        __nv_bfloat16* lo = out + static_cast<size_t>(row) * N + c + lo_delta;
#pragma unroll
        for (int i = 0; i < 4; ++i) lo[i] = bf16_lo_part(y[i]);
      }
    }
    __syncthreads();                                   // everyone is done reading this buffer
    if (threadIdx.x == 0 && grp + 2 < ngroups) issue(grp + 2);
  }
}
void launch_ln_film_act(const float* u, const float* stats, const float* g, const float* b, const float* scale,
                        const float* shift, int film_ld, int film_bcast, int act, __nv_bfloat16* out, int M, int N,
                        int S, cudaStream_t st, const int* film_row_dev, const __nv_bfloat16* u16, long long lo_delta,
                        const float* part, int nslots, float* stats_out) {
  const int blocks = (M + 31) / 32;
  const int threads = N / 4;
  const bool bf = (u16 != nullptr);
  const size_t smem = static_cast<size_t>(2 * 4 * N * (bf ? 2 : 4) + 64);
  const void* in = bf ? static_cast<const void*>(u16) : static_cast<const void*>(u);
#define SMD_LN_LAUNCH(MAXT, BF)                                                                                  \
  {                                                                                                              \
    static bool attr = false;                                                                                    \
    if (!attr) {                                                                                                 \
      cudaFuncSetAttribute(ln_film_act_kernel<MAXT, BF>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 4 * 4096 * 4 + 64); \
      attr = true;                                                                                               \
    }                                                                                                            \
    ln_film_act_kernel<MAXT, BF><<<blocks, threads, smem, st>>>(in, stats, g, b, scale, shift, film_ld, film_bcast, act, \
                                                                out, M, N, S, film_row_dev, lo_delta, part, nslots, stats_out); \
  }
  if (threads <= 512) {
    if (bf) SMD_LN_LAUNCH(512, true) else SMD_LN_LAUNCH(512, false)
  } else {
    if (bf) SMD_LN_LAUNCH(1024, true) else SMD_LN_LAUNCH(1024, false)
  }
#undef SMD_LN_LAUNCH
}

// ---------------------------------------------------------------------------------------------------
// FiLM generator pieces
// ---------------------------------------------------------------------------------------------------
__global__ void noise_encoding_kernel(const float* __restrict__ t, const float* __restrict__ freqs,
                                      float* __restrict__ enc, int R) {
  pdl_trigger();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * 64) return;
  const int r = i / 64, j = i % 64;
  const float arg = __fmul_rn(__fmul_rn(5000.0f, t[r]), freqs[j]);  // (5000 * noise) * freq, in that order
  enc[r * 128 + j] = sinf(arg);
  enc[r * 128 + 64 + j] = cosf(arg);
}
void launch_noise_encoding(const float* t, const float* freqs, float* enc, int R, cudaStream_t st) {
  noise_encoding_kernel<<<(R * 64 + 127) / 128, 128, 0, st>>>(t, freqs, enc, R);
}

// Tiled fp32 SGEMM for the small FiLM-generator layers (forward and backward), 64x64 tile, 4x4 per thread.
//   MODE 0 (NN): C[M][N] = A[M][K] . B[K][N]          forward  y = x W
//   MODE 1 (NT): C[M][N] = A[M][K] . B[N][K]^T        input grad  dx = g W^T
//   MODE 2 (TN): C[M][N] = A[K][M]^T . B[K][N]        weight grad dW = x^T g
// Epilogue: + bias[n]; optional pre-activation copy; act (2 = swish); optional * swish'(mul_pre[m][n]).
template <int MODE>
__global__ void __launch_bounds__(256)
sgemm_small_kernel(const float* __restrict__ A, const float* __restrict__ B, const float* __restrict__ bias,
                   float* __restrict__ C, float* __restrict__ pre_out, const float* __restrict__ mul_pre, int M, int N,
                   int K, int act) {
  __shared__ float As[16][68];
  __shared__ float Bs[16][68];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  // register double-buffering: the global loads of chunk k0+16 are in flight while chunk k0 is multiplied
  float ra[4], rb[4];
  auto load_regs = [&](int k0) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = tid + 256 * j;
      if (MODE == 2) {  // A[K][M]: contiguous in m
        const int kk = i >> 6, m = i & 63;
        ra[j] = (k0 + kk < K && m0 + m < M) ? A[static_cast<size_t>(k0 + kk) * M + m0 + m] : 0.f;
      } else {          // A[M][K]: contiguous in k
        const int m = i >> 4, kk = i & 15;
        ra[j] = (k0 + kk < K && m0 + m < M) ? A[static_cast<size_t>(m0 + m) * K + k0 + kk] : 0.f;
      }
      if (MODE == 1) {  // B[N][K]: contiguous in k
        const int n = i >> 4, kk = i & 15;
        rb[j] = (k0 + kk < K && n0 + n < N) ? B[static_cast<size_t>(n0 + n) * K + k0 + kk] : 0.f;
      } else {          // B[K][N]: contiguous in n
        const int kk = i >> 6, n = i & 63;
        rb[j] = (k0 + kk < K && n0 + n < N) ? B[static_cast<size_t>(k0 + kk) * N + n0 + n] : 0.f;
      }
    }
  };
  auto store_regs = [&]() {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = tid + 256 * j;
      if (MODE == 2) As[i >> 6][i & 63] = ra[j]; else As[i & 15][i >> 4] = ra[j];
      if (MODE == 1) Bs[i & 15][i >> 4] = rb[j]; else Bs[i >> 6][i & 63] = rb[j];
    }
  };
  load_regs(0);
  for (int k0 = 0; k0 < K; k0 += 16) {
    store_regs();
    __syncthreads();
    if (k0 + 16 < K) load_regs(k0 + 16);
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      const float4 a4 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 b4 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float a[4] = {a4.x, a4.y, a4.z, a4.w};
      const float b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j] + (bias ? bias[n] : 0.f);
      const size_t o = static_cast<size_t>(m) * N + n;
      if (pre_out) pre_out[o] = v;
      if (act == 2) v = v / (1.0f + expf(-v));
      if (mul_pre) v *= swish_grad(mul_pre[o]);
      C[o] = v;
    }
  }
}
void launch_sgemm_small(int mode, const float* A, const float* B, const float* bias, float* C, float* pre_out,
                        const float* mul_pre, int M, int N, int K, int act, cudaStream_t st) {
  dim3 grid((N + 63) / 64, (M + 63) / 64);
  if (mode == 0) sgemm_small_kernel<0><<<grid, 256, 0, st>>>(A, B, bias, C, pre_out, mul_pre, M, N, K, act);
  else if (mode == 1) sgemm_small_kernel<1><<<grid, 256, 0, st>>>(A, B, bias, C, pre_out, mul_pre, M, N, K, act);
  else sgemm_small_kernel<2><<<grid, 256, 0, st>>>(A, B, bias, C, pre_out, mul_pre, M, N, K, act);
}
void launch_small_linear(const float* x, const float* W, const float* b, float* y, int R, int K, int N, int act,
                         cudaStream_t st, float* pre) {
  launch_sgemm_small(0, x, W, b, y, pre, nullptr, R, N, K, act, st);
}

__global__ void pad_cast_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int rows, int cols,
                                     int ld, long long lo_delta) {
  const int n = rows * cols;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const size_t o = static_cast<size_t>(i / cols) * ld + i % cols;
    dst[o] = __float2bfloat16_rn(src[i]);
    if (lo_delta) dst[o + lo_delta] = bf16_lo_part(src[i]);
  }
}
void launch_pad_cast_bf16(const float* src, __nv_bfloat16* dst, int rows, int cols, int ld, cudaStream_t st,
                          long long lo_delta) {
  pad_cast_bf16_kernel<<<(rows * cols + 255) / 256, 256, 0, st>>>(src, dst, rows, cols, ld, lo_delta);
}

__global__ void cast_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, size_t n,
                                 long long lo_delta) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    dst[i] = __float2bfloat16_rn(src[i]);
    if (lo_delta) dst[i + lo_delta] = bf16_lo_part(src[i]);
  }
}
void launch_cast_bf16(const float* src, __nv_bfloat16* dst, size_t n, cudaStream_t st, long long lo_delta) {
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > 148 * 16) blocks = 148 * 16;
  if (blocks < 1) blocks = 1;
  cast_bf16_kernel<<<blocks, 256, 0, st>>>(src, dst, n, lo_delta);
}

// ---------------------------------------------------------------------------------------------------
// Chain step bodies after the network call
// ---------------------------------------------------------------------------------------------------
// Block reduction of a chain step's per-column norms (m[0..2]: eps / grad, step, noise; 0 on lanes without a column)
// into the batch means over NC columns: metrics rows 0, 1 and 3 (`stride` floats apart) accumulate them, block 0
// writes `scalar` into row 2.  Every thread of the block calls it.
__device__ __forceinline__ void step_metrics(float* met, size_t stride, float (&m)[3], float scalar, int NC) {
  __shared__ float red[3][8];
  m[0] = warp_sum(m[0]); m[1] = warp_sum(m[1]); m[2] = warp_sum(m[2]);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red[0][w] = m[0]; red[1][w] = m[1]; red[2][w] = m[2]; }
  __syncthreads();
  if (threadIdx.x < 3) {
    float v = 0.f;
    for (int j = 0; j < (blockDim.x >> 5); ++j) v += red[threadIdx.x][j];
    const int row = (threadIdx.x == 0) ? 0 : (threadIdx.x == 1 ? 1 : 3);
    atomicAdd(met + row * stride, v / static_cast<float>(NC));
  }
  if (blockIdx.x == 0 && threadIdx.x == 3) met[2 * stride] = scalar;
}

// The reverse_step_kernel / ddim_step_kernel / dpm_step_kernel body: four adjacent lanes share one (sample, channel)
// column and take a quarter of its S positions each -- 4x the threads and a quarter of the serial threefry chain per
// thread.  Per element idx: z (when draw_noise: the supplied z, or threefry(k0, k1)), nx = update(x, eps_hat, z, noise,
// pos) with pos = s * N * C + (n * C + c) the element's position-major index (a permutation of idx under which the
// lanes of one warp step touch 4 runs of 8 consecutive floats whatever S and C are), the infill
// blend with y = infill_x, or sqrt_ap infill_x + sqrt_1m iz when draw_infill (iz: the supplied infill_z, or
// threefry(ik0, ik1)), the state and the collection row `slot` (< 0: none).  m receives the column norms
// sqrt(sum eps_hat^2 + 1e-10), of x - nx and of noise on the first lane of the column (two shuffles), 0 elsewhere.
template <typename Args, typename Update>
__device__ __forceinline__ void column_step(const Args& a, const float* z_in, const float* infill_z, uint32_t k0,
                                            uint32_t k1, uint32_t ik0, uint32_t ik1, bool draw_noise,
                                            bool draw_infill, float sqrt_ap, float sqrt_1m, int slot, Update update,
                                            float (&m)[3]) {
  const int NC = a.N * a.C;
  const uint32_t total = static_cast<uint32_t>(a.N) * a.S * a.C;
  const uint32_t rtotal = a.rng_total ? a.rng_total : total, rfirst = a.rng_total ? a.rng_first : 0u;
  constexpr int kSG = 4;
  const int gi = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = gi / kSG, sg = gi % kSG;
  float e2 = 0.f, st2 = 0.f, nz2 = 0.f;
  if (i < NC) {
    const int n = i / a.C, c = i % a.C;
    const int per = (a.S + kSG - 1) / kSG;
    const int s_end = min(a.S, (sg + 1) * per);
    for (int s = sg * per; s < s_end; ++s) {
      const uint32_t idx = (static_cast<uint32_t>(n) * a.S + s) * a.C + c;
      const float x = a.x[idx];
      const float eh = a.eps_hat[idx];
      float z = 0.f;
      if (draw_noise) z = z_in ? z_in[idx] : jax_normal_from_bits(jax_random_bits(k0, k1, rfirst + idx, rtotal));
      float noise;
      float nx = update(x, eh, z, noise, static_cast<uint32_t>(s) * NC + i);
      if (a.infill_mask) {
        const float mk = a.infill_mask[idx];
        const float ix = a.infill_x[idx];
        float y = ix;
        if (draw_infill) {
          const float iz = infill_z ? infill_z[idx] : jax_normal_from_bits(jax_random_bits(ik0, ik1, rfirst + idx, rtotal));
          y = sqrt_ap * ix + sqrt_1m * iz;
        }
        nx = nx * (1.0f - mk) + y * mk;
      }
      const float stp = x - nx;
      e2 += eh * eh; st2 += stp * stp; nz2 += noise * noise;
      a.x_next[idx] = nx;
      if (slot >= 0) a.collection[static_cast<size_t>(slot) * total + idx] = nx;
    }
  }
  e2 += __shfl_xor_sync(0xffffffffu, e2, 1); st2 += __shfl_xor_sync(0xffffffffu, st2, 1); nz2 += __shfl_xor_sync(0xffffffffu, nz2, 1);
  e2 += __shfl_xor_sync(0xffffffffu, e2, 2); st2 += __shfl_xor_sync(0xffffffffu, st2, 2); nz2 += __shfl_xor_sync(0xffffffffu, nz2, 2);
  m[0] = m[1] = m[2] = 0.f;
  if (i < NC && sg == 0) { m[0] = sqrtf(e2 + 1e-10f); m[1] = sqrtf(st2 + 1e-10f); m[2] = sqrtf(nz2 + 1e-10f); }
}

// reverse-diffusion step (utils/ebm_utils.py:332-394)
__global__ void __launch_bounds__(256)
reverse_step_kernel(const ReverseStepArgs a) {
  pdl_trigger();
  pdl_wait();
  const int t = a.t_ptr ? *a.t_ptr : a.t;
  const float* cf = a.coef + 8 * t;
  const float sqrt_recip = cf[0], sqrt_m1 = cf[1], mu1 = cf[2], mu2 = cf[3], sigma = cf[4];
  uint32_t k0 = a.key0, k1 = a.key1, ik0 = 0, ik1 = 0;
  if (a.key_tab) { k0 = a.key_tab[4 * t]; k1 = a.key_tab[4 * t + 1]; ik0 = a.key_tab[4 * t + 2]; ik1 = a.key_tab[4 * t + 3]; }
  const int slot = (a.slot_tab && a.collection) ? a.slot_tab[t] : -1;
  float m[3];
  column_step(a, a.z, a.infill_z, k0, k1, ik0, ik1, t > 0, t > 0, cf[5], cf[6], slot,
              [&](float x, float eh, float z, float& noise, uint32_t) {
                noise = z * sigma;
                float recon = __fsub_rn(__fmul_rn(sqrt_recip, x), __fmul_rn(sqrt_m1, eh));
                recon = fminf(fmaxf(recon, -1.0f), 1.0f);
                return __fadd_rn(__fadd_rn(__fmul_rn(mu1, recon), __fmul_rn(mu2, x)), noise);
              }, m);
  if (a.metrics) step_metrics(a.metrics + (a.T - 1 - t), a.T, m, cf[7], a.N * a.C);
}
void launch_reverse_step(const ReverseStepArgs& a, cudaStream_t st) {
  const int NC = a.N * a.C;
  reverse_step_kernel<<<(4 * NC + 255) / 256, 256, 0, st>>>(a);
}

// DDIM step (Song et al. 2021, eq. 12, with the reference's clipped x0 estimate)
__global__ void __launch_bounds__(256)
ddim_step_kernel(const DdimStepArgs a) {
  pdl_trigger();
  pdl_wait();
  const int si = *a.i_ptr;
  const float* cf = a.coef + 8 * si;
  const float sqrt_recip = cf[0], sqrt_m1 = cf[1], c_x0 = cf[2], c_dir = cf[3], sig = cf[4], sqrt_a = cf[5],
              sqrt_1m = cf[6];
  const uint32_t k0 = a.key_tab[4 * si], k1 = a.key_tab[4 * si + 1], ik0 = a.key_tab[4 * si + 2],
                 ik1 = a.key_tab[4 * si + 3];
  const bool t_pos = si > 0 || a.tau0 > 0;     // t = tau_i > 0
  const int slot = a.collection ? a.slot_tab[si] : -1;
  float m[3];
  // sig = 0 (eta = 0, or the last step) draws nothing: the deterministic chain needs no noise stream
  column_step(a, nullptr, nullptr, k0, k1, ik0, ik1, sig != 0.f, t_pos, sqrt_a, sqrt_1m, slot,
              [&](float x, float eh, float z, float& noise, uint32_t) {
                float x0 = __fsub_rn(__fmul_rn(sqrt_recip, x), __fmul_rn(sqrt_m1, eh));
                x0 = fminf(fmaxf(x0, -1.0f), 1.0f);
                const float dir = __fdiv_rn(__fsub_rn(x, __fmul_rn(sqrt_a, x0)), sqrt_1m);
                noise = sig != 0.f ? sig * z : 0.f;
                return __fadd_rn(__fadd_rn(__fmul_rn(c_x0, x0), __fmul_rn(c_dir, dir)), noise);
              }, m);
  if (a.metrics) step_metrics(a.metrics + (a.K - 1 - si), a.K, m, cf[7], a.N * a.C);
}
void launch_ddim_step(const DdimStepArgs& a, cudaStream_t st) {
  const int NC = a.N * a.C;
  ddim_step_kernel<<<(4 * NC + 255) / 256, 256, 0, st>>>(a);
}

// DPM-Solver++ multistep step (Lu et al. 2022, Algorithm 2 and its third-order form), linear in (x, m0, m1, m2)
__global__ void __launch_bounds__(256)
dpm_step_kernel(const DpmStepArgs a) {
  pdl_trigger();
  pdl_wait();
  const int si = *a.i_ptr;
  const float* cf = a.coef + 8 * si;
  const float sqrt_recip = cf[0], sqrt_m1 = cf[1], c_x = cf[2], c_0 = cf[3], c_1 = cf[4], sqrt_a = cf[5],
              c_2 = cf[6];
  // the infill template's sqrt(1-a): the DDPM chain's float32 value
  const float sqrt_1m = __fsqrt_rn(__fsub_rn(1.0f, cf[7]));
  const uint32_t ik0 = a.key_tab[4 * si + 2], ik1 = a.key_tab[4 * si + 3];
  const bool t_pos = si > 0 || a.tau0 > 0;     // t = tau_i > 0
  const int slot = a.collection ? a.slot_tab[si] : -1;
  float* h1 = a.history;
  float* h2 = a.history + static_cast<size_t>(a.N) * a.S * a.C;
  float m[3];
  column_step(a, nullptr, nullptr, 0u, 0u, ik0, ik1, false, t_pos, sqrt_a, sqrt_1m, slot,
              [&](float x, float eh, float, float& noise, uint32_t pos) {
                float m0 = __fsub_rn(__fmul_rn(sqrt_recip, x), __fmul_rn(sqrt_m1, eh));
                m0 = fminf(fmaxf(m0, -1.0f), 1.0f);
                float nx = __fadd_rn(__fmul_rn(c_x, x), __fmul_rn(c_0, m0));
                // a zero coefficient leaves its history unread: it is not written yet at the first steps
                float m1 = 0.f;
                if (c_1 != 0.f) { m1 = h1[pos]; nx = __fadd_rn(nx, __fmul_rn(c_1, m1)); }
                if (c_2 != 0.f) nx = __fadd_rn(nx, __fmul_rn(c_2, h2[pos]));
                if (a.hist_slots > 1 && c_1 != 0.f) h2[pos] = m1;
                if (a.hist_slots > 0) h1[pos] = m0;
                noise = 0.f;
                return nx;
              }, m);
  if (a.metrics) step_metrics(a.metrics + (a.K - 1 - si), a.K, m, cf[7], a.N * a.C);
}
void launch_dpm_step(const DpmStepArgs& a, cudaStream_t st) {
  const int NC = a.N * a.C;
  dpm_step_kernel<<<(4 * NC + 255) / 256, 256, 0, st>>>(a);
}

// ---------------------------------------------------------------------------------------------------
// DDIM encoder step (Song et al. 2021, sections 4.3 and 5.4): the eta = 0 update from data towards noise, with the x0
// estimate unclipped so that the decoder can invert it.  The ddim_step_kernel layout: four lanes per (sample, channel)
// column, a quarter of its S positions each
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ddim_encode_step_kernel(const DdimEncodeStepArgs a) {
  pdl_trigger();
  pdl_wait();
  const float* cf = a.coef + 8 * (*a.r_ptr);
  const float sqrt_recip = cf[0], sqrt_m1 = cf[1], c_x0 = cf[2], c_eps = cf[3];
  const int NC = a.N * a.C;
  constexpr int kSG = 4;
  const int gi = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = gi / kSG, sg = gi % kSG;
  if (i >= NC) return;
  const int n = i / a.C, c = i % a.C;
  const int per = (a.S + kSG - 1) / kSG;
  const int s_end = min(a.S, (sg + 1) * per);
  for (int s = sg * per; s < s_end; ++s) {
    const size_t idx = (static_cast<size_t>(n) * a.S + s) * a.C + c;
    const float x = a.x[idx];
    const float eh = a.eps_hat[idx];
    // at the first step (a = 1) the coefficients are 1 and 0, so x0 = x exactly
    const float x0 = __fsub_rn(__fmul_rn(sqrt_recip, x), __fmul_rn(sqrt_m1, eh));
    a.x_next[idx] = __fadd_rn(__fmul_rn(c_x0, x0), __fmul_rn(c_eps, eh));
  }
}
void launch_ddim_encode_step(const DdimEncodeStepArgs& a, cudaStream_t st) {
  const int NC = a.N * a.C;
  ddim_encode_step_kernel<<<(4 * NC + 255) / 256, 256, 0, st>>>(a);
}

__global__ void step_advance_kernel(int* t_ptr) { *t_ptr -= 1; }
void launch_step_advance(int* t_ptr, cudaStream_t st) { step_advance_kernel<<<1, 1, 0, st>>>(t_ptr); }
__global__ void fill_cond_kernel(const float* coef, int offset, const int* t_ptr, float* cond, int n) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) cond[i] = coef[8 * (*t_ptr) + offset];
}
void launch_fill_cond(const float* coef, int offset, const int* t_ptr, float* cond, int n, cudaStream_t st) {
  fill_cond_kernel<<<(n + 255) / 256, 256, 0, st>>>(coef, offset, t_ptr, cond, n);
}

// ---------------------------------------------------------------------------------------------------
// loss (utils/losses.py:304-308)
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ddpm_loss_kernel(const float* __restrict__ eps, const float* __restrict__ pred, float* __restrict__ loss,
                 float* __restrict__ dpred, float gscale, int per_sample, const float* __restrict__ sigma) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.x;
  const size_t base = static_cast<size_t>(b) * per_sample;
  float s = 0.f;
  if (sigma != nullptr) {
    // denoising score matching (utils/losses.py:166-177): target = -eps / sigma, loss = 0.5 sum((score - target)^2) sigma^2
    const float sg = sigma[b];
    for (int i = threadIdx.x; i < per_sample; i += blockDim.x) {
      const float d = __fmul_rn(__fadd_rn(pred[base + i], __fdiv_rn(eps[base + i], sg)), sg);   // (score - target) * sigma
      s += d * d;
    }
    s *= 0.5f * static_cast<float>(per_sample);     // (the common tail divides by per_sample)
  } else
  for (int i = threadIdx.x; i < per_sample; i += blockDim.x) {
    const float d = eps[base + i] - pred[base + i];
    s += d * d;
    if (dpred) dpred[base + i] = -2.0f * d * gscale;
  }
  __shared__ float red[8];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
    for (int j = 0; j < 8; ++j) v += red[j];
    loss[b] = v / static_cast<float>(per_sample);
  }
}
void launch_ddpm_loss(const float* eps, const float* pred, float* loss_per_example, float* dpred_or_null,
                      float gscale, int B, int per_sample, cudaStream_t st, const float* sigma) {
  ddpm_loss_kernel<<<B, 256, 0, st>>>(eps, pred, loss_per_example, dpred_or_null, gscale, per_sample, sigma);
}

// y[b, :] /= sigma[b]   (DenseNCSN: `output = x / sigmas`, models/ncsn.py:97)
__global__ void scale_rows_kernel(float* __restrict__ y, const float* __restrict__ sigma, int bcast, int B, int per) {
  const size_t total = static_cast<size_t>(B) * per;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    y[i] = __fdiv_rn(y[i], sigma[bcast ? 0 : i / per]);
}
void launch_scale_rows(float* y, const float* sigma, int bcast, int B, int per, cudaStream_t st) {
  const size_t total = static_cast<size_t>(B) * per;
  scale_rows_kernel<<<grid_stride_blocks(total), 256, 0, st>>>(y, sigma, bcast, B, per);
}

// ---------------------------------------------------------------------------------------------------
// sliced score matching: tangent pass and objective (utils/losses.py:182-247)
// ---------------------------------------------------------------------------------------------------
// one CTA per row, N / 4 threads, four columns each
__global__ void __launch_bounds__(1024)
ln_film_tangent_kernel(const float* __restrict__ x32, const __nv_bfloat16* __restrict__ x16,
                       const float* __restrict__ stats, const float* __restrict__ xt, const float* __restrict__ g,
                       const float* __restrict__ bta, const float* __restrict__ ss, int film_ld, int act,
                       __nv_bfloat16* __restrict__ out, int N, int S, long long lo_delta) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[2][32];
  const int row = blockIdx.x, c = threadIdx.x * 4;
  const size_t off = static_cast<size_t>(row) * N + c;
  const float inv_n = 1.0f / static_cast<float>(N);
  float x[4], d[4];
  if (x16) {
    const uint2 raw = *reinterpret_cast<const uint2*>(x16 + off);
    const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.x));
    const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.y));
    x[0] = lo.x; x[1] = lo.y; x[2] = hi.x; x[3] = hi.y;
  } else {
    const float4 q = *reinterpret_cast<const float4*>(x32 + off);
    x[0] = q.x; x[1] = q.y; x[2] = q.z; x[3] = q.w;
  }
  {
    const float4 q = *reinterpret_cast<const float4*>(xt + off);
    d[0] = q.x; d[1] = q.y; d[2] = q.z; d[3] = q.w;
  }
  const float mean = stats[2 * static_cast<size_t>(row)] * inv_n;
  const float rstd = rsqrtf(stats[2 * static_cast<size_t>(row) + 1] * inv_n - mean * mean + 1e-6f);
  float xh[4], s[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    xh[i] = (x[i] - mean) * rstd;
    s[0] += d[i];
    s[1] += xh[i] * d[i];
  }
  block_sums<2>(s, red);
  const float m1 = s[0] * inv_n, m2 = s[1] * inv_n;
  const float* sc = ss ? ss + static_cast<size_t>(row / S) * film_ld : nullptr;
  float o[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float gm = g[c + i];
    const float yd = gm * (rstd * (d[i] - m1 - xh[i] * m2));
    float z = fmaf(gm, xh[i], bta[c + i]), zd = yd;
    if (sc) { z = fmaf(sc[c + i], z, sc[N + c + i]); zd = sc[c + i] * yd; }
    if (act == 2) {
      const float sg = sigmoid_exact(z);
      zd *= sg * fmaf(z, 1.0f - sg, 1.0f);
    }
    o[i] = zd;
  }
  __nv_bfloat162 p0 = __floats2bfloat162_rn(o[0], o[1]);
  __nv_bfloat162 p1 = __floats2bfloat162_rn(o[2], o[3]);
  uint2 pk;
  pk.x = *reinterpret_cast<uint32_t*>(&p0);
  pk.y = *reinterpret_cast<uint32_t*>(&p1);
  *reinterpret_cast<uint2*>(out + off) = pk;
  if (lo_delta) {
#pragma unroll
    for (int i = 0; i < 4; ++i) out[off + i + lo_delta] = bf16_lo_part(o[i]);
  }
}
void launch_ln_film_tangent(const float* x32, const __nv_bfloat16* x16, const float* stats, const float* xt,
                            const float* g, const float* b, const float* ss, int film_ld, int act, __nv_bfloat16* out,
                            int M, int N, int S, cudaStream_t st, long long lo_delta) {
  ln_film_tangent_kernel<<<M, N / 4, 0, st>>>(x32, x16, stats, xt, g, b, ss, film_ld, act, out, N, S, lo_delta);
}

__global__ void tangent_input_kernel(const float* __restrict__ v, const float* const* __restrict__ ind,
                                     __nv_bfloat16* __restrict__ out, size_t n, long long lo_delta) {
  pdl_trigger();
  pdl_wait();
  if (ind) v = ind[3];
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    out[i] = __float2bfloat16_rn(v[i]);
    if (lo_delta) out[i + lo_delta] = bf16_lo_part(v[i]);
  }
}
void launch_tangent_input(const float* v, const float* const* ind, __nv_bfloat16* out, size_t n, cudaStream_t st,
                          long long lo_delta) {
  tangent_input_kernel<<<grid_stride_blocks(n), 256, 0, st>>>(v, ind, out, n, lo_delta);
}

__global__ void __launch_bounds__(256)
ssm_loss_kernel(const float* __restrict__ f, const float* __restrict__ ft, const float* __restrict__ v,
                const float* __restrict__ sigma, const float* const* __restrict__ ind, float* __restrict__ loss,
                float* __restrict__ score, float* __restrict__ hvp, float* __restrict__ loss_sum,
                unsigned int* __restrict__ done_counter, float inv_gb, float* __restrict__ df32,
                __nv_bfloat16* __restrict__ df16, __nv_bfloat16* __restrict__ dft16, int C, int Cp) {
  pdl_trigger();
  pdl_wait();
  if (ind) { sigma = ind[1]; v = ind[3]; }
  const int b = blockIdx.x;
  const size_t base = static_cast<size_t>(b) * C;
  const float sg = sigma[b];
  float s[2] = {0.f, 0.f};
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    const float fv = f[base + i], vv = v[base + i];
    s[0] += fv * fv;
    s[1] += vv * ft[base + i];
    if (score) score[base + i] = __fdiv_rn(fv, sg);
    if (df32) {
      const float gf = fv * inv_gb;
      df32[base + i] = gf;
      df16[static_cast<size_t>(b) * Cp + i] = __float2bfloat16_rn(gf);
      dft16[static_cast<size_t>(b) * Cp + i] = __float2bfloat16_rn(sg * vv * inv_gb);
    }
  }
  __shared__ float red[2][32];
  __shared__ bool last;
  block_sums<2>(s, red);
  if (threadIdx.x == 0) {
    loss[b] = fmaf(sg, s[1], 0.5f * s[0]);
    if (hvp) hvp[b] = __fdiv_rn(s[1], sg);
    last = false;
    if (loss_sum) {
      // as ddpm_loss_bwd_kernel: the last block adds the per-example losses in index order (bit-reproducible)
      __threadfence();
      last = atomicInc(done_counter, gridDim.x - 1) == gridDim.x - 1;
    }
  }
  __syncthreads();
  if (last && threadIdx.x < 32) {
    __threadfence();
    float acc = 0.f;
    for (int i = threadIdx.x; i < static_cast<int>(gridDim.x); i += 32) acc += __ldcg(loss + i);
    acc = warp_sum(acc);
    if (threadIdx.x == 0) { loss_sum[0] = acc; loss_sum[1] = acc * inv_gb; }
  }
}
void launch_ssm_loss(const float* f, const float* ft, const float* v, const float* sigma, const float* const* ind,
                     float* loss, float* score, float* hvp, float* loss_sum, unsigned int* done_counter, float inv_gb,
                     float* df32, __nv_bfloat16* df16, __nv_bfloat16* dft16, int B, int C, int Cp, cudaStream_t st) {
  ssm_loss_kernel<<<B, 256, 0, st>>>(f, ft, v, sigma, ind, loss, score, hvp, loss_sum, done_counter, inv_gb, df32,
                                     df16, dft16, C, Cp);
}

// One Langevin update after the network call (annealed: utils/ebm_utils.py:139-175; consistent: :231-253):
//   next = x + alpha * grad + noise_coef * z ;  infill blend with y = infill_x + infill_sigma * z_infill ;
//   metrics (mean over samples of sqrt(sum_axis1(.)^2 + 1e-10)): grad, alpha * grad, noise ; alpha itself.
// thread = (sample n, channel c) looping over the S positions (axis 1), like the DDPM step kernel.
// With a.state (graph replay of smd_langevin_sample) the per-step scalars, keys and output rows come from the device.
__global__ void __launch_bounds__(256) langevin_step_kernel(const LangevinStepArgs a) {
  const int NC = a.N * a.C;
  const uint32_t total = static_cast<uint32_t>(a.N) * a.S * a.C;
  const uint32_t rtotal = a.rng_total ? a.rng_total : total, rfirst = a.rng_total ? a.rng_first : 0u;
  float alpha = a.alpha, noise_coef = a.noise_coef, infill_sigma = a.infill_sigma;
  uint32_t k0 = a.key0, k1 = a.key1, ik0 = a.ikey0, ik1 = a.ikey1;
  float* coll = a.collection_slot;
  float* met = a.metrics;
  size_t mstride = 1;
  if (a.state) {
    const LangevinChainState* cs = a.state;
    const float* cf = a.coef + kLangevinCoef * cs->si;
    infill_sigma = cf[0]; alpha = cf[1]; noise_coef = cf[2];
    k0 = cs->skey[0]; k1 = cs->skey[1]; ik0 = cs->ikey[0]; ik1 = cs->ikey[1];
    coll = (coll && cs->slot >= 0) ? coll + static_cast<size_t>(cs->slot) * total : nullptr;
    if (met) { met += static_cast<size_t>(cs->si) * a.T + cs->i; mstride = static_cast<size_t>(a.L) * a.T; }
  }
  float m[3] = {0.f, 0.f, 0.f};   // grad_norm, step_norm, noise_norm (metrics rows 0, 1, 3; row 2: alpha)
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < NC) {
    const int n = i / a.C, c = i % a.C;
    float g2 = 0.f, s2 = 0.f, n2 = 0.f;
    for (int s = 0; s < a.S; ++s) {
      const uint32_t idx = (static_cast<uint32_t>(n) * a.S + s) * a.C + c;
      const float x = a.x[idx], g = a.grad[idx];
      const float z = a.z ? a.z[idx] : jax_normal_from_bits(jax_random_bits(k0, k1, rfirst + idx, rtotal));
      const float noise = __fmul_rn(noise_coef, z);
      const float stp = __fmul_rn(alpha, g);
      float nx = __fadd_rn(__fadd_rn(x, stp), noise);
      if (a.infill_mask) {
        const float iz = a.infill_z ? a.infill_z[idx] : jax_normal_from_bits(jax_random_bits(ik0, ik1, rfirst + idx, rtotal));
        const float y = __fadd_rn(a.infill_x[idx], __fmul_rn(infill_sigma, iz));
        const float mk = a.infill_mask[idx];
        nx = nx * (1.0f - mk) + y * mk;
      }
      g2 += g * g; s2 += stp * stp; n2 += noise * noise;
      a.x_next[idx] = nx;
      if (coll) coll[idx] = nx;
    }
    m[0] = sqrtf(g2 + 1e-10f); m[1] = sqrtf(s2 + 1e-10f); m[2] = sqrtf(n2 + 1e-10f);
  }
  if (met) step_metrics(met, mstride, m, alpha, NC);
}
void launch_langevin_step(const LangevinStepArgs& a, cudaStream_t st) {
  const int NC = a.N * a.C;
  langevin_step_kernel<<<(NC + 255) / 256, 256, 0, st>>>(a);
}

// jax.random.split(chain, nsplit) on the device: keys j = words (2j, 2j + 1) of threefry(chain, (i, nsplit + i))
__global__ void langevin_advance_kernel(LangevinChainState* s, const float* __restrict__ coef,
                                        const int* __restrict__ idx_tab, float* __restrict__ cond, int L, int T,
                                        int kind, int rows, int advance) {
  if (advance) s->step += 1;
  const int step = s->step;
  if (step >= L * T) return;   // after the last step: nothing left to prepare
  const int nsplit = kind == 0 ? 3 : 2;
  const uint32_t c0 = s->chain[0], c1 = s->chain[1];
  uint32_t flat[6] = {0u, 0u, 0u, 0u, 0u, 0u};
  for (int j = 0; j < nsplit; ++j) {
    uint32_t x0 = static_cast<uint32_t>(j), x1 = static_cast<uint32_t>(nsplit + j);
    threefry2x32(c0, c1, x0, x1);
    flat[j] = x0; flat[nsplit + j] = x1;
  }
  s->chain[0] = flat[0]; s->chain[1] = flat[1];
  s->skey[0] = flat[2]; s->skey[1] = flat[3];
  s->ikey[0] = flat[4]; s->ikey[1] = flat[5];   // zero for kind 1
  const int si = step / T;
  s->si = si;
  s->i = step % T;
  s->slot = idx_tab ? langevin_slot(idx_tab, step, rows) : -1;
  cond[0] = coef[kLangevinCoef * si];
}
void launch_langevin_advance(LangevinChainState* s, const float* coef, const int* idx_tab, float* cond, int L, int T,
                             int kind, int rows, int advance, cudaStream_t st) {
  langevin_advance_kernel<<<1, 1, 0, st>>>(s, coef, idx_tab, cond, L, T, kind, rows, advance);
}

}  // namespace smd

// Fused transformer sub-blocks for sm_90a, both ending in the next LayerNorm (models/ncsn.py:160-166):
//
//   ffn_fused_kernel : out = LayerNorm_next( gelu(a W1 + b1) W2 + b2 + residual )
//     128 tokens per tile, two consumer warpgroups (64 rows each).  The hidden dimension is processed in chunks of 128:
//       GEMM1_j : acc1 = A[64 x 128] . W1[:, chunk j]        (wgmma, both operands from shared memory, K = 128)
//       epi1_j  : + b1 -> gelu -> bf16, in registers.  The m64 x n128 accumulator fragment rounded to bf16 is exactly the
//                 register A-operand fragment of an m64 x k16 wgmma, so the hidden activation never leaves the
//                 registers
//       GEMM2_j : acc2 += H_j[64 x 128] . W2[chunk j, :]    (wgmma, A from registers, K = 128)
//
//   attn_block_kernel : h_mid = SelfAttention(a) + h_in ;  a2 = LayerNorm(h_mid)
//     64 tokens (two samples of 32 positions) per tile, one consumer warpgroup.
//       GEMM qkv : q | k | v = A[64 x 128] . Wqkv (three N = 128 wgmma products) + bias -> fp32 in shared memory
//       attention: one warp per head, lane = query, fp32 scores / max-subtracted softmax / P V (the same arithmetic as
//                  attention_kernel in kernels.cu) -> o as bf16, written in the K-major SWIZZLE_128B operand layout
//       GEMM out : O[64 x 128] . Wo (wgmma from shared memory)
//     q, k and v never leave the SM.
//
// Both: warp 0 is the TMA producer (activation tile once per tile, 32 KB weight blocks through a small mbarrier ring,
// re-read from L2 for every tile), the consumer warpgroups run the wgmma chains and the epilogues, and the final
// epilogue (+ bias + residual, full-row LayerNorm over the 128 columns) works on the accumulator fragments directly: a
// row's 128 columns sit in the four threads of a quad, so the row statistics need two shuffles.
#pragma once
#include "gemm_wgmma.cuh"

namespace smd {

// v = acc + bias + residual -> out_f32 ; (v - mean) * (rstd * gamma) + beta -> out_bf16  (flax LayerNorm:
// var = E[x^2] - E[x]^2, eps 1e-6).  `row` is this thread's first row (the second is row + 8); residual may alias
// out_f32 (every element is read by the thread that writes it, before the writes).
__device__ __forceinline__ void ln128_fragment_epilogue(float (&d)[64], int row, int M, const float* bias,
                                                        const float* residual, float* out_f32, const float* gamma,
                                                        const float* beta, __nv_bfloat16* out_bf16) {
  const int c = 2 * static_cast<int>(threadIdx.x & 3u);
  float s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 64; i += 2) {
    const int h = (i >> 1) & 1, col = 8 * (i >> 2) + c, r = row + 8 * h;
    const float2 b = __ldg(reinterpret_cast<const float2*>(bias + col));
    const float2 res = (r < M) ? *reinterpret_cast<const float2*>(residual + static_cast<size_t>(r) * 128 + col)
                               : make_float2(0.f, 0.f);
    d[i] = (d[i] + b.x) + res.x;
    d[i + 1] = (d[i + 1] + b.y) + res.y;
    s1[h] += d[i] + d[i + 1];
    s2[h] = fmaf(d[i], d[i], fmaf(d[i + 1], d[i + 1], s2[h]));
  }
  float mean[2], rstd[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    s1[h] += __shfl_xor_sync(0xffffffffu, s1[h], 1);
    s1[h] += __shfl_xor_sync(0xffffffffu, s1[h], 2);
    s2[h] += __shfl_xor_sync(0xffffffffu, s2[h], 1);
    s2[h] += __shfl_xor_sync(0xffffffffu, s2[h], 2);
    mean[h] = s1[h] * (1.0f / 128.0f);
    rstd[h] = rsqrtf(s2[h] * (1.0f / 128.0f) - mean[h] * mean[h] + 1e-6f);
  }
#pragma unroll
  for (int i = 0; i < 64; i += 2) {
    const int h = (i >> 1) & 1, col = 8 * (i >> 2) + c, r = row + 8 * h;
    if (r >= M) continue;
    *reinterpret_cast<float2*>(out_f32 + static_cast<size_t>(r) * 128 + col) = make_float2(d[i], d[i + 1]);
    const float2 g = __ldg(reinterpret_cast<const float2*>(gamma + col));
    const float2 b = __ldg(reinterpret_cast<const float2*>(beta + col));
    const float w0 = (d[i] - mean[h]) * (rstd[h] * g.x) + b.x;
    const float w1 = (d[i + 1] - mean[h]) * (rstd[h] * g.y) + b.y;
    *reinterpret_cast<uint32_t*>(out_bf16 + static_cast<size_t>(r) * 128 + col) = pack_bf16x2(w0, w1);
  }
}

// one 32 KB weight block [2 k-blocks][64 k][2 x 64 n] (MN-major, SWIZZLE_128B) of a row-major (K, N) matrix
__device__ __forceinline__ void tma_load_weight_block(const CUtensorMap* tm, uint64_t* bar, uint8_t* dst, int n0, int k0) {
  mbar_arrive_expect_tx(bar, 32768u);
#pragma unroll
  for (int kb = 0; kb < 2; ++kb)
#pragma unroll
    for (int nb = 0; nb < 2; ++nb) tma_load_2d(tm, bar, dst + kb * 16384 + nb * 8192, n0 + 64 * nb, k0 + 64 * kb);
}

// acc = A[64 x 128] . W[128 x 128], A K-major in shared memory (k-block stride a_kb bytes), W one weight block
__device__ __forceinline__ void wgmma_k128_ss(float (&acc)[64], uint32_t sA, uint32_t a_kb, uint32_t sW) {
  wgmma_fence();
#pragma unroll
  for (int kb = 0; kb < 2; ++kb)
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_m64n128k16_bf16<0, 1>(acc, make_smem_desc_sw128(sA + kb * a_kb + k * 32, 0u, 1024u),
                                  make_smem_desc_sw128(sW + kb * 16384 + k * 2048, 8192u, 1024u), (kb | k) != 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
}

// ---------------------------------------------------------------------------------------------------- fused FFN
struct FfnFusedArgs {
  const float* b1;               // [Md]
  const float* b2;               // [128]
  const float* residual;         // fp32 [M][128] (may alias out_f32)
  float* out_f32;                // fp32 [M][128]
  const float* ln_gamma;         // [128] LayerNorm applied to the new residual stream -> out_bf16
  const float* ln_beta;
  __nv_bfloat16* out_bf16;       // bf16 [M][128]
  int M, Md;
};

struct FfnSmem {
  static constexpr int kA = 32768;          // [2 k-blocks][128 rows][128 B]
  static constexpr int kW = 32768;          // one weight block
  static constexpr int kStages = 4;         // W1_j, W2_j, W1_j+1, ...
  static constexpr int offA = 0;
  static constexpr int offW = offA + kA;
  static constexpr int offBar = offW + kStages * kW;
  static constexpr int kBarBytes = 256;
  static constexpr int kTotal = offBar + kBarBytes + 1024;
  static constexpr int kThreads = 128 + 256;   // producer warpgroup (warp 0 works) + two consumer warpgroups
};

// kAct: the activation between the two GEMMs (ACT_GELU_TANH in the model).  A template parameter, like those of every
// kernel defined in a header that several translation units include.
template <int kAct>
__global__ void __launch_bounds__(FfnSmem::kThreads, 1)
ffn_fused_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW1,
                 const __grid_constant__ CUtensorMap tmW2, const FfnFusedArgs p) {
  using S = FfnSmem;
  extern __shared__ uint8_t ffn_smem_raw[];
  uint8_t* smem = ffn_smem_raw + ((1024u - (smem_u32(ffn_smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::offBar);
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + 1;
  uint64_t* w_full = bars + 2;                 // [kStages]
  uint64_t* w_empty = w_full + S::kStages;     // [kStages]
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = (p.M + 127) / 128;
  const int nchunks = p.Md / 128;

  pdl_trigger();
  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmW1);
    tma_prefetch_desc(&tmW2);
  }
  if (warp == 1 && elect_one()) {
    mbar_init(a_full, 1);
    mbar_init(a_empty, 8);                     // one arrival per consumer warp
    for (int i = 0; i < S::kStages; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == 0) {
    if (elect_one()) {
      int ws = 0; uint32_t wph = 0, it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
        mbar_wait(a_empty, (it & 1u) ^ 1u);
        mbar_arrive_expect_tx(a_full, static_cast<uint32_t>(S::kA));
        for (int kb = 0; kb < 2; ++kb) tma_load_2d(&tmA, a_full, smem + S::offA + kb * 16384, 64 * kb, tile * 128);
        for (int j = 0; j < nchunks; ++j) {
          for (int w = 0; w < 2; ++w) {
            mbar_wait(&w_empty[ws], wph ^ 1u);
            uint8_t* dst = smem + S::offW + ws * S::kW;
            if (w == 0) tma_load_weight_block(&tmW1, &w_full[ws], dst, 128 * j, 0);   // W1 (128, Md): columns of chunk j
            else tma_load_weight_block(&tmW2, &w_full[ws], dst, 0, 128 * j);          // W2 (Md, 128): rows of chunk j
            if (++ws == S::kStages) { ws = 0; wph ^= 1u; }
          }
        }
      }
    }
  } else if (warp >= 4) {
    const uint32_t wg = (warp - 4u) >> 2, wl = (warp - 4u) & 3u;
    const uint32_t sA = smem_u32(smem + S::offA) + wg * 8192u;
    int ws = 0; uint32_t wph = 0, it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int row = tile * 128 + static_cast<int>(wg * 64u + wl * 16u + (lane >> 2));
      const int c = 2 * static_cast<int>(lane & 3u);
      mbar_wait(a_full, it & 1u);
      float acc2[64];
      for (int j = 0; j < nchunks; ++j) {
        uint32_t hr[32];
        {
          float acc1[64];
          mbar_wait(&w_full[ws], wph);
          wgmma_k128_ss(acc1, sA, 16384u, smem_u32(smem + S::offW + ws * S::kW));
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(&w_empty[ws]);
            if (j == nchunks - 1) mbar_arrive(a_empty);
          }
          if (++ws == S::kStages) { ws = 0; wph ^= 1u; }
#pragma unroll
          for (int i = 0; i < 64; i += 2) {
            const int col = 128 * j + 8 * (i >> 2) + c;
            const float2 b = __ldg(reinterpret_cast<const float2*>(p.b1 + col));
            const float v0 = acc1[i] + b.x, v1 = acc1[i + 1] + b.y;
            hr[i >> 1] = pack_bf16x2(act_apply(v0, kAct), act_apply(v1, kAct));
          }
        }
        mbar_wait(&w_full[ws], wph);
        const uint32_t sW2 = smem_u32(smem + S::offW + ws * S::kW);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
          const uint32_t a[4] = {hr[4 * kk], hr[4 * kk + 1], hr[4 * kk + 2], hr[4 * kk + 3]};
          wgmma_m64n128k16_bf16_rs<1>(acc2, a, make_smem_desc_sw128(sW2 + (kk >> 2) * 16384 + (kk & 3) * 2048, 8192u, 1024u),
                                      (j | kk) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&w_empty[ws]);
        if (++ws == S::kStages) { ws = 0; wph ^= 1u; }
      }
      ln128_fragment_epilogue(acc2, row, p.M, p.b2, p.residual, p.out_f32, p.ln_gamma, p.ln_beta, p.out_bf16);
    }
  }
  __syncwarp();
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------- attention block
struct AttnBlockArgs {
  const float* b_qkv;            // [384] = bq | bk | bv
  const float* b_o;              // [128]
  const float* residual;         // fp32 [M][128] (may alias out_f32)
  float* out_f32;                // fp32 [M][128]
  const float* ln_gamma;         // [128] LayerNorm of the new residual stream -> out_bf16
  const float* ln_beta;
  __nv_bfloat16* out_bf16;       // bf16 [M][128]
  int M, H;                      // tokens (a multiple of S); heads (dh = 128 / H in {8, 16})
  int S;                         // sequence length: 32 (two samples per 64-row tile) or 64 (one)
};

struct AttnSmem {
  static constexpr int kA = 16384;                // [2 k-blocks][64 rows][128 B]
  static constexpr int kW = 32768;                // one weight block (q, k, v, o in turn)
  static constexpr int kStages = 2;
  static constexpr int kQkvPitch = 384 + 4;       // floats per q | k | v row
  static constexpr int kQkv = 64 * kQkvPitch * 4;
  static constexpr int kO = 16384;                // attention output as the out-projection's A operand
  static constexpr int offA = 0;
  static constexpr int offW = offA + kA;
  static constexpr int offQkv = offW + kStages * kW;
  static constexpr int offO = offQkv + kQkv;      // 1024-aligned (SWIZZLE_128B operand)
  static constexpr int offBar = offO + kO;
  static constexpr int kBarBytes = 256;
  static constexpr int kTotal = offBar + kBarBytes + 1024;
  static constexpr int kThreads = 128 + 128;      // producer warpgroup (warp 0 works) + one consumer warpgroup
  static_assert(offO % 1024 == 0, "O operand must be 1024-byte aligned");
};

template <int DH, int SEQ>
__global__ void __launch_bounds__(AttnSmem::kThreads, 1)
attn_block_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmWqkv,
                  const __grid_constant__ CUtensorMap tmWo, const AttnBlockArgs p) {
  using S = AttnSmem;
  extern __shared__ uint8_t attn_smem_raw[];
  uint8_t* smem = attn_smem_raw + ((1024u - (smem_u32(attn_smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::offBar);
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + 1;
  uint64_t* w_full = bars + 2;                 // [kStages]
  uint64_t* w_empty = w_full + S::kStages;     // [kStages]
  float* qkv_s = reinterpret_cast<float*>(smem + S::offQkv);
  uint8_t* o_s = smem + S::offO;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = (p.M + 63) / 64;

  pdl_trigger();
  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmWqkv);
    tma_prefetch_desc(&tmWo);
  }
  if (warp == 1 && elect_one()) {
    mbar_init(a_full, 1);
    mbar_init(a_empty, 4);
    for (int i = 0; i < S::kStages; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 4); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == 0) {
    if (elect_one()) {
      int ws = 0; uint32_t wph = 0, it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
        mbar_wait(a_empty, (it & 1u) ^ 1u);
        mbar_arrive_expect_tx(a_full, static_cast<uint32_t>(S::kA));
        for (int kb = 0; kb < 2; ++kb) tma_load_2d(&tmA, a_full, smem + S::offA + kb * 8192, 64 * kb, tile * 64);
        for (int w = 0; w < 4; ++w) {
          mbar_wait(&w_empty[ws], wph ^ 1u);
          uint8_t* dst = smem + S::offW + ws * S::kW;
          if (w < 3) tma_load_weight_block(&tmWqkv, &w_full[ws], dst, 128 * w, 0);
          else tma_load_weight_block(&tmWo, &w_full[ws], dst, 0, 0);
          if (++ws == S::kStages) { ws = 0; wph ^= 1u; }
        }
      }
    }
  } else if (warp >= 4) {
    const uint32_t wl = warp - 4u;
    const int lrow = static_cast<int>(wl * 16u + (lane >> 2));
    const int c = 2 * static_cast<int>(lane & 3u);
    int ws = 0; uint32_t wph = 0, it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int m0 = tile * 64;
      mbar_wait(a_full, it & 1u);
      // ---------------- q | k | v = A Wqkv + b  (fp32, shared memory) ----------------
      for (int w = 0; w < 3; ++w) {
        float acc[64];
        mbar_wait(&w_full[ws], wph);
        wgmma_k128_ss(acc, smem_u32(smem + S::offA), 8192u, smem_u32(smem + S::offW + ws * S::kW));
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&w_empty[ws]);
          if (w == 2) mbar_arrive(a_empty);
        }
        if (++ws == S::kStages) { ws = 0; wph ^= 1u; }
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
          const int col = 128 * w + 8 * (i >> 2) + c, lr = lrow + 8 * ((i >> 1) & 1);
          const float2 b = __ldg(reinterpret_cast<const float2*>(p.b_qkv + col));
          *reinterpret_cast<float2*>(qkv_s + lr * S::kQkvPitch + col) = make_float2(acc[i] + b.x, acc[i + 1] + b.y);
        }
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
      // ---------------- attention: warp = head, lane = query (attention_kernel's arithmetic) ----------------
      // the tile holds 64 / SEQ whole samples; a lane takes queries lane, lane + 32, ... of its sample
      for (int s = 0; s < 64 / SEQ; ++s) {
        const int smp = m0 / SEQ + s;
        if (smp * SEQ >= p.M) break;
        const float* base = qkv_s + (SEQ * s) * S::kQkvPitch;
        for (int h = static_cast<int>(wl); h < p.H; h += 4)
        for (int qh = 0; qh < SEQ / 32; ++qh) {
          const int qrow = 32 * qh + static_cast<int>(lane);
          float q[DH];
          const float qs = rsqrtf(static_cast<float>(DH));
#pragma unroll
          for (int d = 0; d < DH; ++d) q[d] = base[qrow * S::kQkvPitch + h * DH + d] * qs;   // flax: query / sqrt(depth)
          float sc[SEQ];
          float mx = -INFINITY;
#pragma unroll
          for (int j = 0; j < SEQ; ++j) {
            float sj = 0.f;
            const float4* kr = reinterpret_cast<const float4*>(base + j * S::kQkvPitch + 128 + h * DH);
#pragma unroll
            for (int d4 = 0; d4 < DH / 4; ++d4) {
              const float4 k4 = kr[d4];
              sj = fmaf(q[4 * d4], k4.x, sj); sj = fmaf(q[4 * d4 + 1], k4.y, sj);
              sj = fmaf(q[4 * d4 + 2], k4.z, sj); sj = fmaf(q[4 * d4 + 3], k4.w, sj);
            }
            sc[j] = sj;
            mx = fmaxf(mx, sj);
          }
          float sum = 0.f;
#pragma unroll
          for (int j = 0; j < SEQ; ++j) { sc[j] = expf(sc[j] - mx); sum += sc[j]; }
          const float inv = 1.0f / sum;
          float o[DH];
#pragma unroll
          for (int d = 0; d < DH; ++d) o[d] = 0.f;
#pragma unroll
          for (int j = 0; j < SEQ; ++j) {
            const float pj = sc[j] * inv;
            const float4* vr = reinterpret_cast<const float4*>(base + j * S::kQkvPitch + 256 + h * DH);
#pragma unroll
            for (int d4 = 0; d4 < DH / 4; ++d4) {
              const float4 v4 = vr[d4];
              o[4 * d4] = fmaf(pj, v4.x, o[4 * d4]); o[4 * d4 + 1] = fmaf(pj, v4.y, o[4 * d4 + 1]);
              o[4 * d4 + 2] = fmaf(pj, v4.z, o[4 * d4 + 2]); o[4 * d4 + 3] = fmaf(pj, v4.w, o[4 * d4 + 3]);
            }
          }
          const int orow = SEQ * s + qrow;
#pragma unroll
          for (int d = 0; d < DH; d += 2) {
            const int col = h * DH + d;
            // K-major SWIZZLE_128B: 16-byte chunk (col % 64) / 8 of row orow sits at chunk ^ (orow & 7)
            *reinterpret_cast<uint32_t*>(o_s + (col >> 6) * 8192 + orow * 128 + ((((col & 63) >> 3) ^ (orow & 7)) << 4) +
                                         (col & 7) * 2) = pack_bf16x2(o[d], o[d + 1]);
          }
        }
      }
      fence_proxy_async_smem();   // o (generic-proxy stores) -> the wgmma below reads it through the async proxy
      asm volatile("bar.sync 1, 128;" ::: "memory");
      // ---------------- out-projection + bias + residual + LayerNorm ----------------
      float acc[64];
      mbar_wait(&w_full[ws], wph);
      wgmma_k128_ss(acc, smem_u32(o_s), 8192u, smem_u32(smem + S::offW + ws * S::kW));
      __syncwarp();
      if (lane == 0) mbar_arrive(&w_empty[ws]);
      if (++ws == S::kStages) { ws = 0; wph ^= 1u; }
      ln128_fragment_epilogue(acc, m0 + lrow, p.M, p.b_o, p.residual, p.out_f32, p.ln_gamma, p.ln_beta, p.out_bf16);
    }
  }
  __syncwarp();
  __syncthreads();
}

}  // namespace smd

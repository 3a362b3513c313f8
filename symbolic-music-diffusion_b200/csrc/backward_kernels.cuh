// SIMT kernels of the hand-written backward pass (what jax.value_and_grad derives for train_ncsn.py:282-283;
// contract per op in SURVEY Appendix E).
#pragma once
#include <cstdlib>
#include <type_traits>
#include "kernels.cuh"

namespace smd {

// ---------------------------------------------------------------------------------------------------
// wide LayerNorm + FiLM + swish backward (models/shared.py:62-64 / 66-68), one CTA per 32 rows
// ---------------------------------------------------------------------------------------------------
struct LnFilmBwdArgs {
  const float* g;        // [M][N] gradient wrt the bf16 activation that fed the GEMM (fp32), or null ->
  const __nv_bfloat16* g16;  // the same gradient stored as bf16 (what the dX GEMM epilogue writes)
  const float* u;        // [M][N] LayerNorm input (fp32), or null ->
  const __nv_bfloat16* u16;  // the LayerNorm input stored as bf16
  const float* stats;    // [M][2] (sum, sumsq) of u rows
  const float* gamma;    // [N]
  const float* beta;     // [N]
  const float* ss;       // FiLM [nsamples][2N] = [scale | shift], or null (plain LayerNorm)
  int act;               // 2: swish, 0: none
  const float* dres;     // [M][N] residual-path gradient added to dx, or null (may alias dx32)
  float* dx32;           // [M][N], or null when only the bf16 copy / bias sums are needed
  __nv_bfloat16* dx16;   // [M][N] or null
  float* dgamma;         // [N] (atomics)
  float* dbeta;          // [N]
  float* dbias;          // [N] += column sums of the dx32 written here, or null
  float* dss;            // [nsamples][2N] gradient of [scale | shift], or null
  int dss_accum;         // 0: overwrite, 1: add (second use of the same FiLM pair).  The sequence fast path always
                         // ADDS: the caller zero-fills dss once per backward pass
  int M, N, S;           // rows per sample: 1, or a multiple of 32 (32, 64, 128)
};

// blockDim.x = N / 4 threads (N <= 4096): each thread owns one float4 column group; 4 rows per iteration so
// that 8 independent 16-byte loads per thread are in flight and one block reduction serves 4 rows.
template <int MAXT, bool G16, bool U16, bool RES>
__global__ void __launch_bounds__(MAXT)
ln_film_act_bwd_kernel(const LnFilmBwdArgs a) {
  pdl_trigger();
  constexpr int RPI = 4;
  __shared__ float red[2][32][2 * RPI];
  __shared__ float tot[2][2 * RPI];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nwarps = blockDim.x >> 5;
  const int r0 = blockIdx.x * 32;
  const int N = a.N;
  const int c = tid * 4;
  const float inv_n = 1.0f / static_cast<float>(N);
  const bool film = a.ss != nullptr;
  const bool per_block_sample = (a.S % 32 == 0);   // the CTA's 32 rows lie inside sample r0 / S
  float gam[4], bet[4], sc[4] = {1.f, 1.f, 1.f, 1.f}, sh[4] = {0.f, 0.f, 0.f, 0.f};
  float acc_dg[4] = {0, 0, 0, 0}, acc_db[4] = {0, 0, 0, 0}, acc_bias[4] = {0, 0, 0, 0};
  float acc_dsc[4] = {0, 0, 0, 0}, acc_dsh[4] = {0, 0, 0, 0};
  {
    const float4 g4 = *reinterpret_cast<const float4*>(a.gamma + c);
    const float4 b4 = *reinterpret_cast<const float4*>(a.beta + c);
    gam[0] = g4.x; gam[1] = g4.y; gam[2] = g4.z; gam[3] = g4.w;
    bet[0] = b4.x; bet[1] = b4.y; bet[2] = b4.z; bet[3] = b4.w;
  }
  if (film && per_block_sample && r0 < a.M) {
    const float* sp = a.ss + static_cast<size_t>(r0 / a.S) * 2 * N;
    const float4 s4 = *reinterpret_cast<const float4*>(sp + c);
    const float4 h4 = *reinterpret_cast<const float4*>(sp + N + c);
    sc[0] = s4.x; sc[1] = s4.y; sc[2] = s4.z; sc[3] = s4.w;
    sh[0] = h4.x; sh[1] = h4.y; sh[2] = h4.z; sh[3] = h4.w;
  }
  // Register software pipeline: the loads of row group r+RPI are issued before the math and the two block
  // reductions of group r, so ~80 KB per SM stays in flight instead of one exposed DRAM round trip per group.
  // Prefetched rows stay in their storage format (bf16 pairs as uint2) to keep the register budget under 128.
  using GRaw = typename std::conditional<G16, uint2, float4>::type;
  using URaw = typename std::conditional<U16, uint2, float4>::type;
  GRaw gn[RPI]; URaw un[RPI]; float4 dn[RES ? RPI : 1];
  auto unpack = [](const auto& raw) -> float4 {
    if constexpr (sizeof(raw) == 8) {
      const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.x));
      const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.y));
      return make_float4(lo.x, lo.y, hi.x, hi.y);
    } else {
      return raw;
    }
  };
  auto load_group = [&](int r) {
#pragma unroll
    for (int q = 0; q < RPI; ++q) {
      const int row = r0 + r + q;
      const size_t off = static_cast<size_t>(row) * N + c;
      if (row < a.M) {
        if constexpr (G16) gn[q] = *reinterpret_cast<const uint2*>(a.g16 + off);
        else gn[q] = *reinterpret_cast<const float4*>(a.g + off);
        if constexpr (U16) un[q] = *reinterpret_cast<const uint2*>(a.u16 + off);
        else un[q] = *reinterpret_cast<const float4*>(a.u + off);
        if constexpr (RES) dn[q] = *reinterpret_cast<const float4*>(a.dres + off);
      } else {
        gn[q] = GRaw{}; un[q] = URaw{};
        if constexpr (RES) dn[q] = make_float4(0, 0, 0, 0);
      }
    }
  };
  load_group(0);
  for (int r = 0; r < 32; r += RPI) {
    const int buf = (r / RPI) & 1;
    float dxh[RPI][4], xh[RPI][4], rstd[RPI], part[2 * RPI];
    float4 g4[RPI], u4[RPI], d4c[RES ? RPI : 1];
#pragma unroll
    for (int q = 0; q < RPI; ++q) {
      g4[q] = unpack(gn[q]); u4[q] = unpack(un[q]);
      if constexpr (RES) d4c[q] = dn[q];
    }
    if (r + RPI < 32) load_group(r + RPI);   // dres may alias dx32: rows r+RPI.. are not written before this read
#pragma unroll
    for (int q = 0; q < RPI; ++q) {
      const int row = r0 + r + q;
      part[2 * q] = 0.f; part[2 * q + 1] = 0.f; rstd[q] = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) { dxh[q][i] = 0.f; xh[q][i] = 0.f; }
      if (row < a.M) {
        const float s1 = a.stats[2 * static_cast<size_t>(row)], s2 = a.stats[2 * static_cast<size_t>(row) + 1];
        const float mean = s1 * inv_n;
        rstd[q] = rsqrtf(s2 * inv_n - mean * mean + 1e-6f);
        if (film && !per_block_sample) {
          const float* sp = a.ss + static_cast<size_t>(row / a.S) * 2 * N;
          const float4 s4 = *reinterpret_cast<const float4*>(sp + c);
          const float4 h4 = *reinterpret_cast<const float4*>(sp + N + c);
          sc[0] = s4.x; sc[1] = s4.y; sc[2] = s4.z; sc[3] = s4.w;
          sh[0] = h4.x; sh[1] = h4.y; sh[2] = h4.z; sh[3] = h4.w;
        }
        const float gg[4] = {g4[q].x, g4[q].y, g4[q].z, g4[q].w};
        const float uu[4] = {u4[q].x, u4[q].y, u4[q].z, u4[q].w};
        float dsc_row[4], dsh_row[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float x = (uu[i] - mean) * rstd[q];
          const float yln = x * gam[i] + bet[i];
          const float f = film ? (sc[i] * yln + sh[i]) : yln;
          const float dact = (a.act == 2) ? gg[i] * swish_grad(f) : gg[i];
          const float dyln = film ? dact * sc[i] : dact;
          dsh_row[i] = dact; dsc_row[i] = dact * yln;
          acc_db[i] += dyln;
          acc_dg[i] += dyln * x;
          const float d = dyln * gam[i];
          dxh[q][i] = d; xh[q][i] = x;
          part[2 * q] += d; part[2 * q + 1] += d * x;
        }
        if (film) {
          if (per_block_sample) {
#pragma unroll
            for (int i = 0; i < 4; ++i) { acc_dsc[i] += dsc_row[i]; acc_dsh[i] += dsh_row[i]; }
          } else if (a.dss) {
            float* dp = a.dss + static_cast<size_t>(row / a.S) * 2 * N;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              if (a.dss_accum) { dp[c + i] += dsc_row[i]; dp[N + c + i] += dsh_row[i]; }
              else { dp[c + i] = dsc_row[i]; dp[N + c + i] = dsh_row[i]; }
            }
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 2 * RPI; ++j) {
      const float v = warp_sum(part[j]);
      if (lane == 0) red[buf][warp][j] = v;
    }
    __syncthreads();
    if (warp == 0 && lane < 2 * RPI) {
      float t = 0.f;
      for (int w = 0; w < nwarps; ++w) t += red[buf][w][lane];
      tot[buf][lane] = t * inv_n;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < RPI; ++q) {
      const int row = r0 + r + q;
      if (row < a.M) {
        const float m1 = tot[buf][2 * q], m2 = tot[buf][2 * q + 1];
        float dx[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) dx[i] = rstd[q] * (dxh[q][i] - m1 - xh[q][i] * m2);
        if constexpr (RES) { dx[0] += d4c[q].x; dx[1] += d4c[q].y; dx[2] += d4c[q].z; dx[3] += d4c[q].w; }
#pragma unroll
        for (int i = 0; i < 4; ++i) acc_bias[i] += dx[i];
        if (a.dx32) *reinterpret_cast<float4*>(a.dx32 + static_cast<size_t>(row) * N + c) = make_float4(dx[0], dx[1], dx[2], dx[3]);
        if (a.dx16) {
          __nv_bfloat162 q0 = __floats2bfloat162_rn(dx[0], dx[1]);
          __nv_bfloat162 q1 = __floats2bfloat162_rn(dx[2], dx[3]);
          uint2 pk;
          pk.x = *reinterpret_cast<uint32_t*>(&q0);
          pk.y = *reinterpret_cast<uint32_t*>(&q1);
          *reinterpret_cast<uint2*>(a.dx16 + static_cast<size_t>(row) * N + c) = pk;
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    atomicAdd(a.dgamma + c + i, acc_dg[i]);
    atomicAdd(a.dbeta + c + i, acc_db[i]);
    if (a.dbias) atomicAdd(a.dbias + c + i, acc_bias[i]);
  }
  if (film && per_block_sample && a.dss && r0 < a.M) {
    float* dp = a.dss + static_cast<size_t>(r0 / a.S) * 2 * N;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (a.dss_accum) { dp[c + i] += acc_dsc[i]; dp[N + c + i] += acc_dsh[i]; }
      else { dp[c + i] = acc_dsc[i]; dp[N + c + i] = acc_dsh[i]; }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// Fast path of the same backward for the sequence model (a multiple of 32 rows per sample, all rows valid, bf16
// incoming gradient): 16 rows per CTA, all inside sample r0 / S, two CTAs resident per SM (<= 64 registers), two rows per iteration.  The FiLM pair is
// constant over the CTA, so per column only A1 = sum(dact) and A2 = sum(dact * xhat) are accumulated:
//   dbeta = sc A1, dgamma = sc A2, dshift = A1, dscale = gamma A2 + beta A1.
// Row reductions: 4 values per thread -> 6-shuffle multi-value butterfly -> [value][warp] smem -> one
// __syncthreads -> every warp folds the 16 partials itself (no second barrier; smem is double buffered).
// dss must be zero-initialised by the caller: the S / 16 CTAs of a sample add into it.
// ---------------------------------------------------------------------------------------------------
template <int BYTES>
__device__ __forceinline__ void cp_async_own(void* smem_dst, const void* gsrc) {   // per-thread LDGSTS, 8 or 16 bytes
  const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(d), "l"(gsrc), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ float4 unpack_bf16x4(const uint2 raw) {
  const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.x));
  const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.y));
  return make_float4(lo.x, lo.y, hi.x, hi.y);
}

template <bool U16, bool RES, bool FILM>
__global__ void __launch_bounds__(512, 2)
ln_film_bwd_fast_kernel(const LnFilmBwdArgs a) {
  pdl_trigger();
  pdl_wait();
  constexpr int RPB = 16;
  constexpr int UB = U16 ? 8 : 16;                 // bytes of one thread's 4 columns of u
  __shared__ float red[2][4][16];
  // Two-stage LDGSTS pipeline: every thread copies only its own 4 columns of the next two rows (g | u | dres)
  // into shared memory and later reads the same bytes back, so cp.async.wait_group is the only hand-off needed.
  extern __shared__ __align__(16) uint8_t stage_mem[];
  const int T = blockDim.x;
  const int stage_bytes = T * (16 + 2 * UB + (RES ? 32 : 0));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nwarps = blockDim.x >> 5;
  const int r0 = blockIdx.x * RPB;
  const int N = a.N;
  const int c = tid * 4;
  const float inv_n = 1.0f / static_cast<float>(N);
  float A[4], Bc[4], A1[4] = {0, 0, 0, 0}, A2[4] = {0, 0, 0, 0}, accb[4] = {0, 0, 0, 0};
  {
    const float4 g4 = *reinterpret_cast<const float4*>(a.gamma + c);
    A[0] = g4.x; A[1] = g4.y; A[2] = g4.z; A[3] = g4.w;
    if constexpr (FILM) {
      const float4 b4 = *reinterpret_cast<const float4*>(a.beta + c);
      const float* sp = a.ss + static_cast<size_t>(r0 / a.S) * 2 * N;
      const float4 s4 = *reinterpret_cast<const float4*>(sp + c);
      const float4 h4 = *reinterpret_cast<const float4*>(sp + N + c);
      Bc[0] = fmaf(b4.x, s4.x, h4.x); Bc[1] = fmaf(b4.y, s4.y, h4.y);
      Bc[2] = fmaf(b4.z, s4.z, h4.z); Bc[3] = fmaf(b4.w, s4.w, h4.w);
      A[0] *= s4.x; A[1] *= s4.y; A[2] *= s4.z; A[3] *= s4.w;     // A = gamma * scale
    } else {
      Bc[0] = Bc[1] = Bc[2] = Bc[3] = 0.f;
    }
  }
  const bool lo16 = (lane & 16) == 0, lo8 = (lane & 8) == 0;
  auto sg = [&](int stg, int q) { return stage_mem + stg * stage_bytes + (q * T + tid) * 8; };
  auto su = [&](int stg, int q) { return stage_mem + stg * stage_bytes + 16 * T + (q * T + tid) * UB; };
  auto sd = [&](int stg, int q) { return stage_mem + stg * stage_bytes + (16 + 2 * UB) * T + (q * T + tid) * 16; };
  auto issue = [&](int r, int stg) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const size_t off = static_cast<size_t>(r0 + r + q) * N + c;
      cp_async_own<8>(sg(stg, q), a.g16 + off);
      if constexpr (U16) cp_async_own<8>(su(stg, q), a.u16 + off);
      else cp_async_own<16>(su(stg, q), a.u + off);
      if constexpr (RES) cp_async_own<16>(sd(stg, q), a.dres + off);
    }
    cp_async_commit();
  };
  issue(0, 0);
  float4 st_next = *reinterpret_cast<const float4*>(a.stats + 2 * static_cast<size_t>(r0));
  for (int r = 0; r < RPB; r += 2) {
    const int buf = (r >> 1) & 1;
    const size_t off0 = static_cast<size_t>(r0 + r) * N + c, off1 = off0 + N;
    const float4 st = st_next;                     // (s1, s2) x 2 rows
    if (r + 2 < RPB) {
      issue(r + 2, buf ^ 1);                       // dres may alias dx32: rows r+2.. are not written before this
      st_next = *reinterpret_cast<const float4*>(a.stats + 2 * static_cast<size_t>(r0 + r + 2));
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    const uint2 graw0 = *reinterpret_cast<const uint2*>(sg(buf, 0));
    const uint2 graw1 = *reinterpret_cast<const uint2*>(sg(buf, 1));
    float4 u0, u1;
    if constexpr (U16) {
      u0 = unpack_bf16x4(*reinterpret_cast<const uint2*>(su(buf, 0)));
      u1 = unpack_bf16x4(*reinterpret_cast<const uint2*>(su(buf, 1)));
    } else {
      u0 = *reinterpret_cast<const float4*>(su(buf, 0));
      u1 = *reinterpret_cast<const float4*>(su(buf, 1));
    }
    const float mean0 = st.x * inv_n, mean1 = st.z * inv_n;
    const float rstd0 = rsqrtf(st.y * inv_n - mean0 * mean0 + 1e-6f);
    const float rstd1 = rsqrtf(st.w * inv_n - mean1 * mean1 + 1e-6f);
    const float4 g0 = unpack_bf16x4(graw0), g1 = unpack_bf16x4(graw1);
    float x[2][4], d[2][4];
    {
      const float uu0[4] = {u0.x, u0.y, u0.z, u0.w}, uu1[4] = {u1.x, u1.y, u1.z, u1.w};
      const float gg0[4] = {g0.x, g0.y, g0.z, g0.w}, gg1[4] = {g1.x, g1.y, g1.z, g1.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        x[0][i] = (uu0[i] - mean0) * rstd0;
        x[1][i] = (uu1[i] - mean1) * rstd1;
        float da0 = gg0[i], da1 = gg1[i];
        if constexpr (FILM) {
          da0 *= swish_grad(fmaf(x[0][i], A[i], Bc[i]));
          da1 *= swish_grad(fmaf(x[1][i], A[i], Bc[i]));
        }
        A1[i] += da0 + da1;
        A2[i] = fmaf(da0, x[0][i], fmaf(da1, x[1][i], A2[i]));
        d[0][i] = da0 * A[i];
        d[1][i] = da1 * A[i];
      }
    }
    float p0 = (d[0][0] + d[0][1]) + (d[0][2] + d[0][3]);
    float p1 = fmaf(d[0][0], x[0][0], fmaf(d[0][1], x[0][1], fmaf(d[0][2], x[0][2], d[0][3] * x[0][3])));
    float p2 = (d[1][0] + d[1][1]) + (d[1][2] + d[1][3]);
    float p3 = fmaf(d[1][0], x[1][0], fmaf(d[1][1], x[1][1], fmaf(d[1][2], x[1][2], d[1][3] * x[1][3])));
    {  // 4 values x 32 lanes -> lane (j * 8) holds the warp total of value j
      const float k0 = lo16 ? p0 : p2, s0 = lo16 ? p2 : p0;
      const float k1 = lo16 ? p1 : p3, s1 = lo16 ? p3 : p1;
      const float q0 = k0 + __shfl_xor_sync(0xffffffffu, s0, 16);
      const float q1 = k1 + __shfl_xor_sync(0xffffffffu, s1, 16);
      const float kk = lo8 ? q0 : q1, ss = lo8 ? q1 : q0;
      float v = kk + __shfl_xor_sync(0xffffffffu, ss, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      if ((lane & 7) == 0) red[buf][lane >> 3][warp] = v;   // value index = (bit4, bit3) of the lane
    }
    __syncthreads();
    float m[4];
    {
      const int w = lane & 15;
      float v0 = (w < nwarps) ? red[buf][lane >> 4][w] : 0.f;        // values 0 / 1
      float v1 = (w < nwarps) ? red[buf][2 + (lane >> 4)][w] : 0.f;  // values 2 / 3
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) {
        v0 += __shfl_xor_sync(0xffffffffu, v0, o);
        v1 += __shfl_xor_sync(0xffffffffu, v1, o);
      }
      m[0] = __shfl_sync(0xffffffffu, v0, 0) * inv_n;
      m[1] = __shfl_sync(0xffffffffu, v0, 16) * inv_n;
      m[2] = __shfl_sync(0xffffffffu, v1, 0) * inv_n;
      m[3] = __shfl_sync(0xffffffffu, v1, 16) * inv_n;
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const size_t off = q ? off1 : off0;
      const float rs = q ? rstd1 : rstd0;
      float dx[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) dx[i] = rs * (d[q][i] - m[2 * q] - x[q][i] * m[2 * q + 1]);
      if constexpr (RES) {
        const float4 d4 = *reinterpret_cast<const float4*>(sd(buf, q));
        dx[0] += d4.x; dx[1] += d4.y; dx[2] += d4.z; dx[3] += d4.w;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) accb[i] += dx[i];
      if (a.dx32) *reinterpret_cast<float4*>(a.dx32 + off) = make_float4(dx[0], dx[1], dx[2], dx[3]);
      if (a.dx16) {
        __nv_bfloat162 q0 = __floats2bfloat162_rn(dx[0], dx[1]);
        __nv_bfloat162 q1 = __floats2bfloat162_rn(dx[2], dx[3]);
        uint2 pk;
        pk.x = *reinterpret_cast<uint32_t*>(&q0);
        pk.y = *reinterpret_cast<uint32_t*>(&q1);
        *reinterpret_cast<uint2*>(a.dx16 + off) = pk;
      }
    }
  }
  // epilogue: column gradients (A currently holds gamma * scale)
  float sc[4] = {1.f, 1.f, 1.f, 1.f}, gam[4], bet[4] = {0.f, 0.f, 0.f, 0.f};
  {
    const float4 g4 = *reinterpret_cast<const float4*>(a.gamma + c);
    gam[0] = g4.x; gam[1] = g4.y; gam[2] = g4.z; gam[3] = g4.w;
    if constexpr (FILM) {
      const float4 b4 = *reinterpret_cast<const float4*>(a.beta + c);
      const float4 s4 = *reinterpret_cast<const float4*>(a.ss + static_cast<size_t>(r0 / a.S) * 2 * N + c);
      bet[0] = b4.x; bet[1] = b4.y; bet[2] = b4.z; bet[3] = b4.w;
      sc[0] = s4.x; sc[1] = s4.y; sc[2] = s4.z; sc[3] = s4.w;
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    atomicAdd(a.dgamma + c + i, sc[i] * A2[i]);
    atomicAdd(a.dbeta + c + i, sc[i] * A1[i]);
    if (a.dbias) atomicAdd(a.dbias + c + i, accb[i]);
  }
  if constexpr (FILM) {
    if (a.dss) {
      float* dp = a.dss + static_cast<size_t>(r0 / a.S) * 2 * N;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        atomicAdd(dp + c + i, fmaf(gam[i], A2[i], bet[i] * A1[i]));
        atomicAdd(dp + N + c + i, A1[i]);
      }
    }
  }
}

inline void launch_ln_film_act_bwd(const LnFilmBwdArgs& a, cudaStream_t st) {
  const int threads = a.N / 4;
  const bool film = a.ss != nullptr;
  if (a.S % 32 == 0 && a.g16 && !a.g && threads <= 512 && threads % 32 == 0 && a.M % 32 == 0 &&
      ((film && a.act == 2) || (!film && a.act == 0))) {
    const int fb = a.M / 16;
    const int key = (a.u16 ? 4 : 0) | (a.dres ? 2 : 0) | (film ? 1 : 0);
    const int smem = 2 * threads * (16 + 2 * (a.u16 ? 8 : 16) + (a.dres ? 32 : 0));   // <= 80 KB: two CTAs per SM
#define SMD_LNB_FAST(U, R, F)                                                                               \
  {                                                                                                          \
    cudaFuncSetAttribute(ln_film_bwd_fast_kernel<U, R, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); \
    ln_film_bwd_fast_kernel<U, R, F><<<fb, threads, smem, st>>>(a);                                          \
  }
    switch (key) {
      case 0: SMD_LNB_FAST(false, false, false) break;
      case 1: SMD_LNB_FAST(false, false, true) break;
      case 2: SMD_LNB_FAST(false, true, false) break;
      case 3: SMD_LNB_FAST(false, true, true) break;
      case 4: SMD_LNB_FAST(true, false, false) break;
      case 5: SMD_LNB_FAST(true, false, true) break;
      case 6: SMD_LNB_FAST(true, true, false) break;
      default: SMD_LNB_FAST(true, true, true) break;
    }
#undef SMD_LNB_FAST
    return;
  }
  const int blocks = (a.M + 31) / 32;
  auto go = [&](auto g16, auto u16, auto res) {
    constexpr bool G = decltype(g16)::value, U = decltype(u16)::value, R = decltype(res)::value;
    if (threads <= 512) ln_film_act_bwd_kernel<512, G, U, R><<<blocks, threads, 0, st>>>(a);
    else ln_film_act_bwd_kernel<1024, G, U, R><<<blocks, threads, 0, st>>>(a);
  };
  using T = std::true_type; using F = std::false_type;
  const int key = (a.g16 ? 4 : 0) | (a.u16 ? 2 : 0) | (a.dres ? 1 : 0);
  switch (key) {
    case 0: go(F{}, F{}, F{}); break;
    case 1: go(F{}, F{}, T{}); break;
    case 2: go(F{}, T{}, F{}); break;
    case 3: go(F{}, T{}, T{}); break;
    case 4: go(T{}, F{}, F{}); break;
    case 5: go(T{}, F{}, T{}); break;
    case 6: go(T{}, T{}, F{}); break;
    default: go(T{}, T{}, T{}); break;
  }
}

// ---------------------------------------------------------------------------------------------------
// sliced score matching: reverse pass through a wide LayerNorm + FiLM + swish AND its tangent (launch_ln_film_tangent).
// Per row, with xh = (x - mean) r, xc' = x' - mean(x'), q = r mean(xh x'), xh' = r xc' - xh q, z = s (gamma xh + beta) + h,
// z' = s gamma xh', out = swish(z), out' = swish'(z) z' and the incoming adjoints (g, g'):
//   gz = g swish'(z) + g' swish''(z) z',  gz' = g' swish'(z);   dscale += gz y + gz' y',  dshift += gz
//   tangent adjoint:  dx' = r (gxh' - mean(gxh') - xh mean(xh gxh'))          with gxh' = gamma s gz'
//   primal adjoint:   dx  = LN-backward(gxh - q gxh') - (r^2 xh / N) gr + (xc' / N) gP
//                     with gr = sum(gxh' xc') - 2 mean(xh x') sum(gxh' xh),  gP = -r^2 sum(gxh' xh)
// (the last two terms are the dependence of the tangent on x through r and mean(xh x')).  kSsmRows rows per CTA,
// the column sums (gamma, beta, bias) leave through one atomic per column and CTA.
// ---------------------------------------------------------------------------------------------------
struct SsmLnBwdArgs {
  const float* x32;           // [M][N] primal LayerNorm input (fp32), or null ->
  const __nv_bfloat16* x16;   // the same stored as bf16
  const float* xt;            // [M][N] its tangent (fp32)
  const float* stats;         // [M][2] (sum, sumsq) of the primal rows
  const float* gamma;
  const float* beta;
  const float* ss;            // FiLM [nsamples][2N] = [scale | shift], or null (plain LayerNorm)
  int act;                    // 2: swish, 0: none
  const __nv_bfloat16* g16;   // [M][N] adjoint of the primal output
  const __nv_bfloat16* gt16;  // [M][N] adjoint of the tangent output
  const float* dres;          // residual adjoints added to dx / dx' (may alias dx32 / dxt32), or null
  const float* dres_t;
  float* dx32; __nv_bfloat16* dx16;    // primal input adjoint (either may be null)
  float* dxt32; __nv_bfloat16* dxt16;  // tangent input adjoint
  float* dgamma; float* dbeta;         // [N] (atomics)
  float* dbias;                        // [N] += column sums of dx, or null
  float* dss;                          // [nsamples][2N] += gradient of [scale | shift] (zeroed by the caller)
  int M, N, S;
};
static constexpr int kSsmRows = 4;

__device__ __forceinline__ void store_bf16x4(__nv_bfloat16* p, const float (&v)[4]) {
  __nv_bfloat162 q0 = __floats2bfloat162_rn(v[0], v[1]);
  __nv_bfloat162 q1 = __floats2bfloat162_rn(v[2], v[3]);
  uint2 pk;
  pk.x = *reinterpret_cast<uint32_t*>(&q0);
  pk.y = *reinterpret_cast<uint32_t*>(&q1);
  *reinterpret_cast<uint2*>(p) = pk;
}

// CPT adjacent columns per thread, at most 512 threads (<= 128 registers, no spills): CPT = 4 up to N = 2048, 8 above
template <int CPT>
__global__ void __launch_bounds__(512) ssm_ln_bwd_kernel(const SsmLnBwdArgs a) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red2[2][32];
  __shared__ float red5[5][32];
  const int N = a.N, c = threadIdx.x * CPT;
  const float inv_n = 1.0f / static_cast<float>(N);
  float adg[CPT], adb[CPT], abias[CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) { adg[i] = 0.f; adb[i] = 0.f; abias[i] = 0.f; }
  auto ld4 = [](float* dst, const float4 v) { dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w; };
  for (int r = 0; r < kSsmRows; ++r) {
    const int row = blockIdx.x * kSsmRows + r;
    if (row >= a.M) break;   // uniform over the CTA
    const size_t off = static_cast<size_t>(row) * N + c;
    float x[CPT], d[CPT], g[CPT], gt[CPT];
#pragma unroll
    for (int j = 0; j < CPT; j += 4) {
      ld4(x + j, a.x16 ? unpack_bf16x4(*reinterpret_cast<const uint2*>(a.x16 + off + j))
                       : *reinterpret_cast<const float4*>(a.x32 + off + j));
      ld4(d + j, *reinterpret_cast<const float4*>(a.xt + off + j));
      ld4(g + j, unpack_bf16x4(*reinterpret_cast<const uint2*>(a.g16 + off + j)));
      ld4(gt + j, unpack_bf16x4(*reinterpret_cast<const uint2*>(a.gt16 + off + j)));
    }
    const float mean = a.stats[2 * static_cast<size_t>(row)] * inv_n;
    const float rstd = rsqrtf(a.stats[2 * static_cast<size_t>(row) + 1] * inv_n - mean * mean + 1e-6f);
    float xh[CPT], s2[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < CPT; ++i) {
      xh[i] = (x[i] - mean) * rstd;
      s2[0] += d[i];
      s2[1] += xh[i] * d[i];
    }
    block_sums<2>(s2, red2);
    const float m1 = s2[0] * inv_n, m2 = s2[1] * inv_n;
    const float q = rstd * m2;
    const float* sp = a.ss ? a.ss + static_cast<size_t>(row / a.S) * 2 * N : nullptr;
    float* dp = (sp && a.dss) ? a.dss + static_cast<size_t>(row / a.S) * 2 * N : nullptr;
    float* xc = d;   // d is dead once centred
    float gxd[CPT], h[CPT], s5[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < CPT; ++i) {
      const float gm = a.gamma[c + i];
      xc[i] = d[i] - m1;
      const float xhd = rstd * (xc[i] - xh[i] * m2);
      const float y = fmaf(gm, xh[i], a.beta[c + i]), yd = gm * xhd;
      const float sc = sp ? sp[c + i] : 1.0f;
      const float z = sp ? fmaf(sc, y, sp[N + c + i]) : y, zd = sc * yd;
      float gz = g[i], gzd = gt[i];
      if (a.act == 2) {
        const float sg = sigmoid_exact(z);
        const float d1 = sg * fmaf(z, 1.0f - sg, 1.0f);
        const float d2 = sg * (1.0f - sg) * fmaf(z, 1.0f - 2.0f * sg, 2.0f);
        gz = fmaf(g[i], d1, gt[i] * d2 * zd);
        gzd = gt[i] * d1;
      }
      if (dp) { dp[c + i] += fmaf(gz, y, gzd * yd); dp[N + c + i] += gz; }
      const float gy = gz * sc, gyd = gzd * sc;
      adg[i] += fmaf(gy, xh[i], gyd * xhd);
      adb[i] += gy;
      gxd[i] = gyd * gm;
      h[i] = fmaf(-q, gxd[i], gy * gm);
      s5[0] += gxd[i];
      s5[1] += xh[i] * gxd[i];
      s5[2] += gxd[i] * xc[i];
      s5[3] += h[i];
      s5[4] += xh[i] * h[i];
    }
    block_sums<5>(s5, red5);
    const float gr = s5[2] - 2.0f * m2 * s5[1];
    const float gP = -rstd * rstd * s5[1];
#pragma unroll
    for (int j = 0; j < CPT; j += 4) {
      float dx[4], dxt[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = j + u;
        dx[u] = rstd * (h[i] - s5[3] * inv_n - xh[i] * s5[4] * inv_n) - rstd * rstd * xh[i] * inv_n * gr +
                xc[i] * inv_n * gP;
        dxt[u] = rstd * (gxd[i] - s5[0] * inv_n - xh[i] * s5[1] * inv_n);
      }
      if (a.dres) {
        const float4 r4 = *reinterpret_cast<const float4*>(a.dres + off + j);
        dx[0] += r4.x; dx[1] += r4.y; dx[2] += r4.z; dx[3] += r4.w;
      }
      if (a.dres_t) {
        const float4 r4 = *reinterpret_cast<const float4*>(a.dres_t + off + j);
        dxt[0] += r4.x; dxt[1] += r4.y; dxt[2] += r4.z; dxt[3] += r4.w;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) abias[j + u] += dx[u];
      if (a.dx32) *reinterpret_cast<float4*>(a.dx32 + off + j) = make_float4(dx[0], dx[1], dx[2], dx[3]);
      if (a.dxt32) *reinterpret_cast<float4*>(a.dxt32 + off + j) = make_float4(dxt[0], dxt[1], dxt[2], dxt[3]);
      if (a.dx16) store_bf16x4(a.dx16 + off + j, dx);
      if (a.dxt16) store_bf16x4(a.dxt16 + off + j, dxt);
    }
  }
#pragma unroll
  for (int i = 0; i < CPT; ++i) {
    atomicAdd(a.dgamma + c + i, adg[i]);
    atomicAdd(a.dbeta + c + i, adb[i]);
    if (a.dbias) atomicAdd(a.dbias + c + i, abias[i]);
  }
}
inline void launch_ssm_ln_bwd(const SsmLnBwdArgs& a, cudaStream_t st) {
  const int blocks = (a.M + kSsmRows - 1) / kSsmRows;
  if (a.N <= 2048) ssm_ln_bwd_kernel<4><<<blocks, a.N / 4, 0, st>>>(a);
  else ssm_ln_bwd_kernel<8><<<blocks, a.N / 8, 0, st>>>(a);
}

// ---------------------------------------------------------------------------------------------------
// narrow (128-wide) LayerNorm backward, one warp per row; statistics recomputed from the saved input
// ---------------------------------------------------------------------------------------------------
struct Ln128BwdArgs {
  const float* g;       // [M][128] gradient wrt the LayerNorm output
  const float* h;      // [M][128] LayerNorm input
  const float* gamma;   // [128]
  const float* dres;    // [M][128] or null (may alias dx32)
  float* dx32;          // [M][128]
  __nv_bfloat16* dx16;  // [M][128] or null
  float* dgamma; float* dbeta;   // [128] atomics
  float* dbias;         // [128] += column sums of dx32, or null
  int M;
};

__global__ void __launch_bounds__(256) ln128_bwd_kernel(const Ln128BwdArgs a) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[3][8][128];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * 8 + warp, nw = gridDim.x * 8;
  const int c = lane * 4;
  const float4 gm = *reinterpret_cast<const float4*>(a.gamma + c);
  const float gam[4] = {gm.x, gm.y, gm.z, gm.w};
  float adg[4] = {0, 0, 0, 0}, adb[4] = {0, 0, 0, 0}, abias[4] = {0, 0, 0, 0};
  for (int row = gw; row < a.M; row += nw) {
    const float4 h4 = *reinterpret_cast<const float4*>(a.h + static_cast<size_t>(row) * 128 + c);
    const float4 g4 = *reinterpret_cast<const float4*>(a.g + static_cast<size_t>(row) * 128 + c);
    const float hh[4] = {h4.x, h4.y, h4.z, h4.w};
    const float gg[4] = {g4.x, g4.y, g4.z, g4.w};
    float s1 = hh[0] + hh[1] + hh[2] + hh[3];
    float s2 = hh[0] * hh[0] + hh[1] * hh[1] + hh[2] * hh[2] + hh[3] * hh[3];
    s1 = warp_sum(s1); s2 = warp_sum(s2);
    const float mean = s1 * (1.0f / 128.0f);
    const float rstd = rsqrtf(s2 * (1.0f / 128.0f) - mean * mean + 1e-6f);
    float xh[4], dxh[4], p1 = 0.f, p2 = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      xh[i] = (hh[i] - mean) * rstd;
      adb[i] += gg[i];
      adg[i] += gg[i] * xh[i];
      dxh[i] = gg[i] * gam[i];
      p1 += dxh[i]; p2 += dxh[i] * xh[i];
    }
    p1 = warp_sum(p1) * (1.0f / 128.0f); p2 = warp_sum(p2) * (1.0f / 128.0f);
    float dx[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) dx[i] = rstd * (dxh[i] - p1 - xh[i] * p2);
    if (a.dres) {
      const float4 d4 = *reinterpret_cast<const float4*>(a.dres + static_cast<size_t>(row) * 128 + c);
      dx[0] += d4.x; dx[1] += d4.y; dx[2] += d4.z; dx[3] += d4.w;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) abias[i] += dx[i];
    *reinterpret_cast<float4*>(a.dx32 + static_cast<size_t>(row) * 128 + c) = make_float4(dx[0], dx[1], dx[2], dx[3]);
    if (a.dx16) {
      __nv_bfloat162 q0 = __floats2bfloat162_rn(dx[0], dx[1]);
      __nv_bfloat162 q1 = __floats2bfloat162_rn(dx[2], dx[3]);
      uint2 pk;
      pk.x = *reinterpret_cast<uint32_t*>(&q0);
      pk.y = *reinterpret_cast<uint32_t*>(&q1);
      *reinterpret_cast<uint2*>(a.dx16 + static_cast<size_t>(row) * 128 + c) = pk;
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) { red[0][warp][c + i] = adg[i]; red[1][warp][c + i] = adb[i]; red[2][warp][c + i] = abias[i]; }
  __syncthreads();
  for (int idx = threadIdx.x; idx < 3 * 128; idx += blockDim.x) {
    const int k = idx / 128, col = idx % 128;
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += red[k][w][col];
    if (k == 0) atomicAdd(a.dgamma + col, v);
    else if (k == 1) atomicAdd(a.dbeta + col, v);
    else if (a.dbias) atomicAdd(a.dbias + col, v);
  }
}
inline void launch_ln128_bwd(const Ln128BwdArgs& a, cudaStream_t st) {
  int blocks = (a.M + 7) / 8;
  if (blocks > 148 * 2) blocks = 148 * 2;
  ln128_bwd_kernel<<<blocks, 256, 0, st>>>(a);
}

// ---------------------------------------------------------------------------------------------------
// column sums (bias gradients): out[n] += sum_m in[m][n]
// ---------------------------------------------------------------------------------------------------
// fp32: one column per thread; bf16: two adjacent columns per thread (4-byte loads); 64 rows per block
template <typename T>
__global__ void __launch_bounds__(128) colsum_kernel(const T* __restrict__ in, int ld, float* __restrict__ out, int M, int N) {
  pdl_trigger();
  const int m0 = blockIdx.y * 64, m1 = min(M, m0 + 64);
  if constexpr (sizeof(T) == 2) {
    const int n = (blockIdx.x * 128 + threadIdx.x) * 2;
    if (n >= N) return;
    float s0 = 0.f, s1 = 0.f;
    if (n + 1 < N && (ld & 1) == 0) {
#pragma unroll 8
      for (int m = m0; m < m1; ++m) {
        const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(in + static_cast<size_t>(m) * ld + n));
        s0 += f.x; s1 += f.y;
      }
      atomicAdd(out + n, s0); atomicAdd(out + n + 1, s1);
    } else {
      for (int m = m0; m < m1; ++m) s0 += __bfloat162float(in[static_cast<size_t>(m) * ld + n]);
      atomicAdd(out + n, s0);
      if (n + 1 < N) {
        for (int m = m0; m < m1; ++m) s1 += __bfloat162float(in[static_cast<size_t>(m) * ld + n + 1]);
        atomicAdd(out + n + 1, s1);
      }
    }
  } else {
    const int n = blockIdx.x * 128 + threadIdx.x;
    if (n >= N) return;
    float s = 0.f;
#pragma unroll 8
    for (int m = m0; m < m1; ++m) s += in[static_cast<size_t>(m) * ld + n];
    atomicAdd(out + n, s);
  }
}
template <typename T>
inline void launch_colsum(const T* in, int ld, float* out, int M, int N, cudaStream_t st) {
  const int cols_per_block = (sizeof(T) == 2) ? 256 : 128;
  dim3 grid((N + cols_per_block - 1) / cols_per_block, (M + 63) / 64);
  colsum_kernel<T><<<grid, 128, 0, st>>>(in, ld, out, M, N);
}

// ---------------------------------------------------------------------------------------------------
// attention backward at S = 32 (SURVEY Appendix E): one CTA per sample, one warp per head, lane = query / key index
// ---------------------------------------------------------------------------------------------------
template <int DH>
__global__ void attention_bwd_kernel(const float* __restrict__ qkv, const float* __restrict__ probs,
                                     const float* __restrict__ dO, __nv_bfloat16* __restrict__ dqkv16,
                                     float* __restrict__ dbias, int H) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) float sm[];
  // a CTA owns HPB = blockDim.x / 32 heads of one sample: W = HPB * DH columns of q, k, v and dO
  const int HPB = blockDim.x >> 5, W = HPB * DH, W4 = W / 4;
  const int hb = blockIdx.y * HPB;   // first head of this CTA
  float* sQ = sm;                  // [32][W] scaled q
  float* sK = sQ + 32 * W;
  float* sV = sK + 32 * W;
  float* sD = sV + 32 * W;         // dO
  float* scr = sD + 32 * W;        // [HPB][32][33]
  const int b = blockIdx.x, tid = threadIdx.x;
  const float qs = rsqrtf(static_cast<float>(DH));
  const float* base = qkv + static_cast<size_t>(b) * 32 * 384;
  const float* dob = dO + static_cast<size_t>(b) * 32 * 128;
  for (int i = tid; i < 32 * W4; i += blockDim.x) {
    const int row = i / W4, c4 = (i % W4) * 4, gc = hb * DH + c4;
    float4 q4 = *reinterpret_cast<const float4*>(base + row * 384 + gc);
    q4.x *= qs; q4.y *= qs; q4.z *= qs; q4.w *= qs;
    *reinterpret_cast<float4*>(&sQ[row * W + c4]) = q4;
    *reinterpret_cast<float4*>(&sK[row * W + c4]) = *reinterpret_cast<const float4*>(base + row * 384 + 128 + gc);
    *reinterpret_cast<float4*>(&sV[row * W + c4]) = *reinterpret_cast<const float4*>(base + row * 384 + 256 + gc);
    *reinterpret_cast<float4*>(&sD[row * W + c4]) = *reinterpret_cast<const float4*>(dob + row * 128 + gc);
  }
  __syncthreads();
  const int hl = tid >> 5, lane = tid & 31;
  const int h = hb + hl;
  if (h >= H) return;
  float* my = scr + hl * 32 * 33;
  const int hc = hl * DH;      // column offset inside the staged tiles
  const int gh = h * DH;       // column offset in global memory
  float P[32];
  const float* pr = probs + ((static_cast<size_t>(b) * H + h) * 32 + lane) * 32;
#pragma unroll
  for (int j = 0; j < 32; j += 4) {
    const float4 t = *reinterpret_cast<const float4*>(pr + j);
    P[j] = t.x; P[j + 1] = t.y; P[j + 2] = t.z; P[j + 3] = t.w;
  }
  float dO_i[DH];
#pragma unroll
  for (int d = 0; d < DH; d += 4) {
    const float4 t = *reinterpret_cast<const float4*>(&sD[lane * W + hc + d]);
    dO_i[d] = t.x; dO_i[d + 1] = t.y; dO_i[d + 2] = t.z; dO_i[d + 3] = t.w;
  }
  float dS[32];
  float rs = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < DH; d += 4) {   // broadcast 16-byte reads
      const float4 t = *reinterpret_cast<const float4*>(&sV[j * W + hc + d]);
      s = fmaf(dO_i[d], t.x, fmaf(dO_i[d + 1], t.y, fmaf(dO_i[d + 2], t.z, fmaf(dO_i[d + 3], t.w, s))));
    }
    dS[j] = s;
    rs = fmaf(s, P[j], rs);
  }
#pragma unroll
  for (int j = 0; j < 32; ++j) { my[lane * 33 + j] = P[j]; dS[j] = P[j] * (dS[j] - rs); }
  __syncwarp();
  // dv_j = sum_i P[i][j] dO_i    (lane = j)
  float dv[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) dv[d] = 0.f;
#pragma unroll 4
  for (int i = 0; i < 32; ++i) {
    const float p = my[i * 33 + lane];
#pragma unroll
    for (int d = 0; d < DH; d += 4) {
      const float4 t = *reinterpret_cast<const float4*>(&sD[i * W + hc + d]);
      dv[d] = fmaf(p, t.x, dv[d]); dv[d + 1] = fmaf(p, t.y, dv[d + 1]);
      dv[d + 2] = fmaf(p, t.z, dv[d + 2]); dv[d + 3] = fmaf(p, t.w, dv[d + 3]);
    }
  }
  __syncwarp();
  // dq_i = (sum_j dS[i][j] k_j) / sqrt(dh)   (lane = i)
  float dq[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) dq[d] = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    my[lane * 33 + j] = dS[j];
#pragma unroll
    for (int d = 0; d < DH; d += 4) {
      const float4 t = *reinterpret_cast<const float4*>(&sK[j * W + hc + d]);
      dq[d] = fmaf(dS[j], t.x, dq[d]); dq[d + 1] = fmaf(dS[j], t.y, dq[d + 1]);
      dq[d + 2] = fmaf(dS[j], t.z, dq[d + 2]); dq[d + 3] = fmaf(dS[j], t.w, dq[d + 3]);
    }
  }
#pragma unroll
  for (int d = 0; d < DH; ++d) dq[d] *= qs;
  __syncwarp();
  // dk_j = sum_i dS[i][j] q~_i   (lane = j)
  float dk[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) dk[d] = 0.f;
#pragma unroll 4
  for (int i = 0; i < 32; ++i) {
    const float s = my[i * 33 + lane];
#pragma unroll
    for (int d = 0; d < DH; d += 4) {
      const float4 t = *reinterpret_cast<const float4*>(&sQ[i * W + hc + d]);
      dk[d] = fmaf(s, t.x, dk[d]); dk[d + 1] = fmaf(s, t.y, dk[d + 1]);
      dk[d + 2] = fmaf(s, t.z, dk[d + 2]); dk[d + 3] = fmaf(s, t.w, dk[d + 3]);
    }
  }
  __nv_bfloat16* orow = dqkv16 + (static_cast<size_t>(b) * 32 + lane) * 384;
#pragma unroll
  for (int d = 0; d < DH; d += 2) {
    *reinterpret_cast<__nv_bfloat162*>(orow + gh + d) = __floats2bfloat162_rn(dq[d], dq[d + 1]);
    *reinterpret_cast<__nv_bfloat162*>(orow + 128 + gh + d) = __floats2bfloat162_rn(dk[d], dk[d + 1]);
    *reinterpret_cast<__nv_bfloat162*>(orow + 256 + gh + d) = __floats2bfloat162_rn(dv[d], dv[d + 1]);
  }
#pragma unroll
  for (int d = 0; d < DH; ++d) {
    const float a = warp_sum(dq[d]), bsum = warp_sum(dk[d]), c = warp_sum(dv[d]);
    if (lane == 0) {
      atomicAdd(dbias + gh + d, a);
      atomicAdd(dbias + 128 + gh + d, bsum);
      atomicAdd(dbias + 256 + gh + d, c);
    }
  }
}
// ---------------------------------------------------------------------------------------------------
// Tensor-core attention backward (DH % 8 == 0): the four 32x32x16-class products per head on mma.sync m16n8k8 tf32.
//   dP = dO V^T, dS = P (dP - rowsum(dP P)), dV = P^T dO, dQ = dS K / sqrt(dh), dK = dS^T Q~
// P and dS live in accumulator-layout registers; the products that need them as the A operand in the same
// orientation (dQ) take them straight from registers with the key permutation of the forward kernel, the transposed
// uses (dV, dK) go through a per-warp 32x36 shared tile read back as the transposed fragment (bank-conflict free
// with the same within-8 permutation applied to the B operand rows).
// ---------------------------------------------------------------------------------------------------
template <int DH>
__global__ void __launch_bounds__(128)
attention_bwd_mma_kernel(const float* __restrict__ qkv, const float* __restrict__ probs, const float* __restrict__ dO,
                         __nv_bfloat16* __restrict__ dqkv16, float* __restrict__ dbias, int H) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) uint32_t attb_sm[];
  constexpr int NT2 = DH / 8;
  const int tid = threadIdx.x;
  const int HPB = blockDim.x >> 5, W = HPB * DH, W4 = W / 4, PT = W + 4;
  uint32_t* sQ = attb_sm;             // [32][PT] tf32, q / sqrt(dh)
  uint32_t* sK = sQ + 32 * PT;
  uint32_t* sV = sK + 32 * PT;
  uint32_t* sD = sV + 32 * PT;        // dO
  uint32_t* sTall = sD + 32 * PT;     // [HPB][32][36]
  const int b = blockIdx.x, hb = blockIdx.y * HPB;
  const float qs = rsqrtf(static_cast<float>(DH));
  const float* base = qkv + static_cast<size_t>(b) * 32 * 384;
  const float* dob = dO + static_cast<size_t>(b) * 32 * 128;
  for (int i = tid; i < 32 * W4; i += blockDim.x) {
    const int row = i / W4, c4 = (i % W4) * 4, gc = hb * DH + c4;
    const float4 q4 = *reinterpret_cast<const float4*>(base + row * 384 + gc);
    const float4 k4 = *reinterpret_cast<const float4*>(base + row * 384 + 128 + gc);
    const float4 v4 = *reinterpret_cast<const float4*>(base + row * 384 + 256 + gc);
    const float4 d4 = *reinterpret_cast<const float4*>(dob + row * 128 + gc);
    *reinterpret_cast<uint4*>(&sQ[row * PT + c4]) = make_uint4(to_tf32(q4.x * qs), to_tf32(q4.y * qs), to_tf32(q4.z * qs), to_tf32(q4.w * qs));
    *reinterpret_cast<uint4*>(&sK[row * PT + c4]) = make_uint4(to_tf32(k4.x), to_tf32(k4.y), to_tf32(k4.z), to_tf32(k4.w));
    *reinterpret_cast<uint4*>(&sV[row * PT + c4]) = make_uint4(to_tf32(v4.x), to_tf32(v4.y), to_tf32(v4.z), to_tf32(v4.w));
    *reinterpret_cast<uint4*>(&sD[row * PT + c4]) = make_uint4(to_tf32(d4.x), to_tf32(d4.y), to_tf32(d4.z), to_tf32(d4.w));
  }
  __syncthreads();
  const int hl = tid >> 5, lane = tid & 31;
  const int h = hb + hl;
  if (h >= H) return;
  const int g = lane >> 2, t = lane & 3;
  const int hc = hl * DH, gh = h * DH;
  uint32_t* sT = sTall + hl * 32 * 36;

  // P in accumulator layout: [mt][nt] -> rows 16 mt + g (+8), keys 8 nt + 2t (+1)
  float pc[2][4][4];
  {
    const float* pr = probs + (static_cast<size_t>(b) * H + h) * 32 * 32;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const float2 lo = *reinterpret_cast<const float2*>(pr + (16 * mt + g) * 32 + 8 * nt + 2 * t);
        const float2 hi = *reinterpret_cast<const float2*>(pr + (16 * mt + g + 8) * 32 + 8 * nt + 2 * t);
        pc[mt][nt][0] = lo.x; pc[mt][nt][1] = lo.y; pc[mt][nt][2] = hi.x; pc[mt][nt][3] = hi.y;
      }
  }
  // ---- dP = dO V^T
  float ds[2][4][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) ds[mt][nt][i] = 0.f;
#pragma unroll
  for (int ks = 0; ks < NT2; ++ks) {
    uint32_t a[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const uint32_t* d0 = sD + (16 * mt + g) * PT + hc + 8 * ks + t;
      a[mt][0] = d0[0]; a[mt][1] = d0[8 * PT]; a[mt][2] = d0[4]; a[mt][3] = d0[8 * PT + 4];
    }
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const uint32_t* v0 = sV + (8 * nt + g) * PT + hc + 8 * ks + t;
      const uint32_t b0 = v0[0], b1 = v0[4];
      mma_tf32_16x8x8(ds[0][nt], a[0], b0, b1);
      mma_tf32_16x8x8(ds[1][nt], a[1], b0, b1);
    }
  }
  // ---- dS = P (dP - sum_j dP P)
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float rs = 0.f;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
        rs = fmaf(ds[mt][nt][2 * hr], pc[mt][nt][2 * hr], fmaf(ds[mt][nt][2 * hr + 1], pc[mt][nt][2 * hr + 1], rs));
      rs += __shfl_xor_sync(0xffffffffu, rs, 1);
      rs += __shfl_xor_sync(0xffffffffu, rs, 2);
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        ds[mt][nt][2 * hr] = pc[mt][nt][2 * hr] * (ds[mt][nt][2 * hr] - rs);
        ds[mt][nt][2 * hr + 1] = pc[mt][nt][2 * hr + 1] * (ds[mt][nt][2 * hr + 1] - rs);
      }
    }
  // stage an accumulator-layout [query][key] matrix in the warp's tile (tf32)
  auto stage = [&](const float (&m)[2][4][4]) {
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        *reinterpret_cast<uint2*>(&sT[(16 * mt + g) * 36 + 8 * nt + 2 * t]) = make_uint2(to_tf32(m[mt][nt][0]), to_tf32(m[mt][nt][1]));
        *reinterpret_cast<uint2*>(&sT[(16 * mt + g + 8) * 36 + 8 * nt + 2 * t]) = make_uint2(to_tf32(m[mt][nt][2]), to_tf32(m[mt][nt][3]));
      }
  };
  // out[key][dim] = sum_query T[query][key] * Bm[query][dim]; query slots of each 8-block permuted (t -> 2t, t+4 -> 2t+1)
  auto mma_transposed = [&](float (&out)[2][NT2][4], const uint32_t* Bm) {
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int n2 = 0; n2 < NT2; ++n2)
#pragma unroll
        for (int i = 0; i < 4; ++i) out[mt][n2][i] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      uint32_t a[2][4];
      const uint32_t* r0 = sT + (8 * ks + 2 * t) * 36;
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        a[mt][0] = r0[16 * mt + g];        // (key g,     query 2t)
        a[mt][1] = r0[16 * mt + g + 8];    // (key g + 8, query 2t)
        a[mt][2] = r0[36 + 16 * mt + g];   // (key g,     query 2t + 1)
        a[mt][3] = r0[36 + 16 * mt + g + 8];
      }
#pragma unroll
      for (int n2 = 0; n2 < NT2; ++n2) {
        const uint32_t* b0p = Bm + (8 * ks + 2 * t) * PT + hc + 8 * n2 + g;
        const uint32_t b0 = b0p[0], b1 = b0p[PT];
        mma_tf32_16x8x8(out[0][n2], a[0], b0, b1);
        mma_tf32_16x8x8(out[1][n2], a[1], b0, b1);
      }
    }
  };
  // ---- dV = P^T dO
  float dv[2][NT2][4];
  stage(pc);
  __syncwarp();
  mma_transposed(dv, sD);
  __syncwarp();
  // ---- dQ = dS K / sqrt(dh)  (A straight from registers, keys permuted as in the forward P V product)
  float dq[2][NT2][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int n2 = 0; n2 < NT2; ++n2)
#pragma unroll
      for (int i = 0; i < 4; ++i) dq[mt][n2][i] = 0.f;
#pragma unroll
  for (int kb = 0; kb < 4; ++kb) {
    uint32_t a[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      a[mt][0] = to_tf32(ds[mt][kb][0]); a[mt][1] = to_tf32(ds[mt][kb][2]);
      a[mt][2] = to_tf32(ds[mt][kb][1]); a[mt][3] = to_tf32(ds[mt][kb][3]);
    }
#pragma unroll
    for (int n2 = 0; n2 < NT2; ++n2) {
      const uint32_t* k0 = sK + (8 * kb + 2 * t) * PT + hc + 8 * n2 + g;
      const uint32_t b0 = k0[0], b1 = k0[PT];
      mma_tf32_16x8x8(dq[0][n2], a[0], b0, b1);
      mma_tf32_16x8x8(dq[1][n2], a[1], b0, b1);
    }
  }
  // ---- dK = dS^T Q~
  float dk[2][NT2][4];
  stage(ds);
  __syncwarp();
  mma_transposed(dk, sQ);
  // ---- outputs (bf16 GEMM operand) and bias gradients (column sums over the 32 rows)
  __nv_bfloat16* ob = dqkv16 + static_cast<size_t>(b) * 32 * 384 + gh;
  auto emit = [&](const float (&m)[2][NT2][4], int col_off, float scale) {
#pragma unroll
    for (int n2 = 0; n2 < NT2; ++n2) {
      float c0 = 0.f, c1 = 0.f;
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const float v0 = m[mt][n2][0] * scale, v1 = m[mt][n2][1] * scale, v2 = m[mt][n2][2] * scale, v3 = m[mt][n2][3] * scale;
        *reinterpret_cast<__nv_bfloat162*>(ob + (16 * mt + g) * 384 + col_off + 8 * n2 + 2 * t) = __floats2bfloat162_rn(v0, v1);
        *reinterpret_cast<__nv_bfloat162*>(ob + (16 * mt + g + 8) * 384 + col_off + 8 * n2 + 2 * t) = __floats2bfloat162_rn(v2, v3);
        c0 += v0 + v2; c1 += v1 + v3;
      }
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        c0 += __shfl_xor_sync(0xffffffffu, c0, o);
        c1 += __shfl_xor_sync(0xffffffffu, c1, o);
      }
      if (g == 0) {
        atomicAdd(dbias + col_off + gh + 8 * n2 + 2 * t, c0);
        atomicAdd(dbias + col_off + gh + 8 * n2 + 2 * t + 1, c1);
      }
    }
  };
  emit(dq, 0, qs);
  emit(dk, 128, 1.0f);
  emit(dv, 256, 1.0f);
}

// ---------------------------------------------------------------------------------------------------
// Attention backward for S in {64, 128} (any head dim): P and dS of 32 queries x S keys do not fit a warp's registers,
// so a CTA (one sample, HPB heads) walks the S / 32 query blocks of its sample and, inside each, the S / 32 key blocks.
//   query block qb (lane = query i):  rs_i = sum_j dP_ij P_ij ;  dS_ij = P_ij (dP_ij - rs_i) ;  dq_i = sum_j dS_ij k_j
//   per key block (lane = key j):     dv_j += sum_{i in qb} P_ij dO_i ;  dk_j += sum_{i in qb} dS_ij q~_i
// dP_ij = dO_i . v_j is recomputed in the second sweep instead of being kept.  dq is written once per query block;
// dk and dv accumulate in fp32 shared memory (a warp owns its head's columns) and are written once at the end.  The
// bias gradients are the same column sums, added with one atomic per column and block.
// ---------------------------------------------------------------------------------------------------
template <int DH, int S>
__global__ void __launch_bounds__(128)
attention_bwd_long_kernel(const float* __restrict__ qkv, const float* __restrict__ probs, const float* __restrict__ dO,
                          __nv_bfloat16* __restrict__ dqkv16, float* __restrict__ dbias, int H) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) float attl_sm[];
  const int HPB = blockDim.x >> 5, W = HPB * DH, W4 = W / 4;
  const int hb = blockIdx.y * HPB;
  float* sQ = attl_sm;             // [S][W] q / sqrt(dh)
  float* sK = sQ + S * W;
  float* sV = sK + S * W;
  float* sD = sV + S * W;          // dO
  float* sdK = sD + S * W;         // [S][W] fp32 accumulators
  float* sdV = sdK + S * W;
  float* scr = sdV + S * W;        // [HPB][2][32][33]: P and dS of one (query block, key block) tile
  const int b = blockIdx.x, tid = threadIdx.x;
  const float qs = rsqrtf(static_cast<float>(DH));
  const float* base = qkv + static_cast<size_t>(b) * S * 384;
  const float* dob = dO + static_cast<size_t>(b) * S * 128;
  for (int i = tid; i < S * W4; i += blockDim.x) {
    const int row = i / W4, c4 = (i % W4) * 4, gc = hb * DH + c4;
    float4 q4 = *reinterpret_cast<const float4*>(base + row * 384 + gc);
    q4.x *= qs; q4.y *= qs; q4.z *= qs; q4.w *= qs;
    *reinterpret_cast<float4*>(&sQ[row * W + c4]) = q4;
    *reinterpret_cast<float4*>(&sK[row * W + c4]) = *reinterpret_cast<const float4*>(base + row * 384 + 128 + gc);
    *reinterpret_cast<float4*>(&sV[row * W + c4]) = *reinterpret_cast<const float4*>(base + row * 384 + 256 + gc);
    *reinterpret_cast<float4*>(&sD[row * W + c4]) = *reinterpret_cast<const float4*>(dob + row * 128 + gc);
    *reinterpret_cast<float4*>(&sdK[row * W + c4]) = make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(&sdV[row * W + c4]) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __syncthreads();
  const int hl = tid >> 5, lane = tid & 31;
  const int h = hb + hl;
  if (h >= H) return;
  float* tP = scr + hl * 2 * 32 * 33;
  float* tS = tP + 32 * 33;
  const int hc = hl * DH;      // column offset inside the staged tiles
  const int gh = h * DH;       // column offset in global memory
  auto dot_dO_v = [&](const float (&d_i)[DH], int j) {
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < DH; d += 4) {   // broadcast 16-byte reads
      const float4 t = *reinterpret_cast<const float4*>(&sV[j * W + hc + d]);
      s = fmaf(d_i[d], t.x, fmaf(d_i[d + 1], t.y, fmaf(d_i[d + 2], t.z, fmaf(d_i[d + 3], t.w, s))));
    }
    return s;
  };
  for (int qb = 0; qb < S / 32; ++qb) {
    const int qi = qb * 32 + lane;
    const float* pr = probs + ((static_cast<size_t>(b) * H + h) * S + qi) * S;
    float dO_i[DH];
#pragma unroll
    for (int d = 0; d < DH; d += 4) {
      const float4 t = *reinterpret_cast<const float4*>(&sD[qi * W + hc + d]);
      dO_i[d] = t.x; dO_i[d + 1] = t.y; dO_i[d + 2] = t.z; dO_i[d + 3] = t.w;
    }
    float rs = 0.f;
    for (int j = 0; j < S; j += 4) {
      const float4 p4 = *reinterpret_cast<const float4*>(pr + j);
      rs = fmaf(dot_dO_v(dO_i, j), p4.x, rs); rs = fmaf(dot_dO_v(dO_i, j + 1), p4.y, rs);
      rs = fmaf(dot_dO_v(dO_i, j + 2), p4.z, rs); rs = fmaf(dot_dO_v(dO_i, j + 3), p4.w, rs);
    }
    float dq[DH];
#pragma unroll
    for (int d = 0; d < DH; ++d) dq[d] = 0.f;
    for (int kb = 0; kb < S / 32; ++kb) {
      // lane = query: this tile's P and dS rows, and dq
#pragma unroll 4
      for (int jj = 0; jj < 32; jj += 4) {
        const int j0 = kb * 32 + jj;
        const float4 p4 = *reinterpret_cast<const float4*>(pr + j0);
        const float pv[4] = {p4.x, p4.y, p4.z, p4.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int j = j0 + u;
          const float ds = pv[u] * (dot_dO_v(dO_i, j) - rs);
          tP[lane * 33 + jj + u] = pv[u];
          tS[lane * 33 + jj + u] = ds;
#pragma unroll
          for (int d = 0; d < DH; d += 4) {
            const float4 t = *reinterpret_cast<const float4*>(&sK[j * W + hc + d]);
            dq[d] = fmaf(ds, t.x, dq[d]); dq[d + 1] = fmaf(ds, t.y, dq[d + 1]);
            dq[d + 2] = fmaf(ds, t.z, dq[d + 2]); dq[d + 3] = fmaf(ds, t.w, dq[d + 3]);
          }
        }
      }
      __syncwarp();
      // lane = key kb * 32 + lane: contributions of this query block to dv and dk
      float dv[DH], dk[DH];
#pragma unroll
      for (int d = 0; d < DH; ++d) { dv[d] = 0.f; dk[d] = 0.f; }
#pragma unroll 4
      for (int i = 0; i < 32; ++i) {
        const float p = tP[i * 33 + lane], s = tS[i * 33 + lane];
        const int row = (qb * 32 + i) * W + hc;
#pragma unroll
        for (int d = 0; d < DH; d += 4) {
          const float4 td = *reinterpret_cast<const float4*>(&sD[row + d]);
          const float4 tq = *reinterpret_cast<const float4*>(&sQ[row + d]);
          dv[d] = fmaf(p, td.x, dv[d]); dv[d + 1] = fmaf(p, td.y, dv[d + 1]);
          dv[d + 2] = fmaf(p, td.z, dv[d + 2]); dv[d + 3] = fmaf(p, td.w, dv[d + 3]);
          dk[d] = fmaf(s, tq.x, dk[d]); dk[d + 1] = fmaf(s, tq.y, dk[d + 1]);
          dk[d + 2] = fmaf(s, tq.z, dk[d + 2]); dk[d + 3] = fmaf(s, tq.w, dk[d + 3]);
        }
      }
      const int krow = (kb * 32 + lane) * W + hc;
#pragma unroll
      for (int d = 0; d < DH; ++d) { sdV[krow + d] += dv[d]; sdK[krow + d] += dk[d]; }
      __syncwarp();
    }
    __nv_bfloat16* orow = dqkv16 + (static_cast<size_t>(b) * S + qi) * 384 + gh;
#pragma unroll
    for (int d = 0; d < DH; d += 2)
      *reinterpret_cast<__nv_bfloat162*>(orow + d) = __floats2bfloat162_rn(dq[d] * qs, dq[d + 1] * qs);
#pragma unroll
    for (int d = 0; d < DH; ++d) {
      const float v = warp_sum(dq[d] * qs);
      if (lane == 0) atomicAdd(dbias + gh + d, v);
    }
  }
  // dk, dv: lane = key, one pass per key block (the warp wrote these rows itself: __syncwarp suffices)
  for (int kb = 0; kb < S / 32; ++kb) {
    const int kj = kb * 32 + lane;
    __nv_bfloat16* orow = dqkv16 + (static_cast<size_t>(b) * S + kj) * 384 + gh;
#pragma unroll
    for (int d = 0; d < DH; d += 2) {
      const float k0 = sdK[kj * W + hc + d], k1 = sdK[kj * W + hc + d + 1];
      const float v0 = sdV[kj * W + hc + d], v1 = sdV[kj * W + hc + d + 1];
      *reinterpret_cast<__nv_bfloat162*>(orow + 128 + d) = __floats2bfloat162_rn(k0, k1);
      *reinterpret_cast<__nv_bfloat162*>(orow + 256 + d) = __floats2bfloat162_rn(v0, v1);
    }
#pragma unroll
    for (int d = 0; d < DH; ++d) {
      const float ksum = warp_sum(sdK[kj * W + hc + d]), vsum = warp_sum(sdV[kj * W + hc + d]);
      if (lane == 0) { atomicAdd(dbias + 128 + gh + d, ksum); atomicAdd(dbias + 256 + gh + d, vsum); }
    }
  }
}

template <int S>
inline cudaError_t launch_attention_bwd_long(const float* qkv, const float* probs, const float* dO,
                                             __nv_bfloat16* dqkv16, float* dbias, int B, int H, cudaStream_t st) {
  const int dh = 128 / H;
  int hpb = H;
  while (hpb > 4 && hpb % 2 == 0) hpb /= 2;
  while (hpb > 1 && hpb * dh * S > 4096) hpb /= 2;   // <= 4096 staged elements per tile: ~100 KB, two CTAs per SM
  const size_t smem = (6 * static_cast<size_t>(S) * hpb * dh + static_cast<size_t>(hpb) * 2 * 32 * 33) * sizeof(float);
  const dim3 grid(B, H / hpb);
#define SMD_ATT_BWD_LONG(DHV)                                                                                        \
  {                                                                                                                  \
    cudaError_t e = cudaFuncSetAttribute(attention_bwd_long_kernel<DHV, S>,                                          \
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));       \
    if (e != cudaSuccess) return e;                                                                                  \
    attention_bwd_long_kernel<DHV, S><<<grid, hpb * 32, smem, st>>>(qkv, probs, dO, dqkv16, dbias, H);               \
    return cudaPeekAtLastError();                                                                                    \
  }
  if (dh == 16) SMD_ATT_BWD_LONG(16)
  else if (dh == 8) SMD_ATT_BWD_LONG(8)
  else if (dh == 32) SMD_ATT_BWD_LONG(32)
  else SMD_ATT_BWD_LONG(4)
#undef SMD_ATT_BWD_LONG
}

inline cudaError_t launch_attention_bwd(const float* qkv, const float* probs, const float* dO, __nv_bfloat16* dqkv16,
                                        float* dbias, int B, int S, int H, cudaStream_t st) {
  if (S == 64) return launch_attention_bwd_long<64>(qkv, probs, dO, dqkv16, dbias, B, H, st);
  if (S == 128) return launch_attention_bwd_long<128>(qkv, probs, dO, dqkv16, dbias, B, H, st);
  const int dh = 128 / H;
  int hpb = H;                       // heads per CTA: <= 4 so that several CTAs are resident per SM
  while (hpb > 4 && hpb % 2 == 0) hpb /= 2;
  const size_t smem = (4 * 32 * static_cast<size_t>(hpb) * dh + static_cast<size_t>(hpb) * 32 * 33) * sizeof(float);
  const dim3 grid(B, H / hpb);
  if (dh % 8 == 0 && dh <= 32) {
    const size_t sm2 = (4 * 32 * static_cast<size_t>(hpb * dh + 4) + static_cast<size_t>(hpb) * 32 * 36) * sizeof(uint32_t);
#define SMD_ATT_BWD_MMA(DHV)                                                                                        \
  {                                                                                                                 \
    cudaError_t e = cudaFuncSetAttribute(attention_bwd_mma_kernel<DHV>, cudaFuncAttributeMaxDynamicSharedMemorySize,  \
                                         static_cast<int>(sm2));                                                    \
    if (e != cudaSuccess) return e;                                                                                 \
    attention_bwd_mma_kernel<DHV><<<grid, hpb * 32, sm2, st>>>(qkv, probs, dO, dqkv16, dbias, H);                   \
    return cudaPeekAtLastError();                                                                                   \
  }
    if (dh == 16) SMD_ATT_BWD_MMA(16)
    else if (dh == 8) SMD_ATT_BWD_MMA(8)
    else SMD_ATT_BWD_MMA(32)
#undef SMD_ATT_BWD_MMA
  }
#define SMD_ATT_BWD(DHV)                                                                                       \
  {                                                                                                            \
    cudaError_t e = cudaFuncSetAttribute(attention_bwd_kernel<DHV>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                         static_cast<int>(smem));                                              \
    if (e != cudaSuccess) return e;                                                                            \
    attention_bwd_kernel<DHV><<<grid, hpb * 32, smem, st>>>(qkv, probs, dO, dqkv16, dbias, H);                 \
  }
  if (dh == 16) SMD_ATT_BWD(16)
  else if (dh == 8) SMD_ATT_BWD(8)
  else if (dh == 32) SMD_ATT_BWD(32)
  else if (dh == 4) SMD_ATT_BWD(4)
#undef SMD_ATT_BWD
  return cudaSuccess;
}

// ---------------------------------------------------------------------------------------------------
// input projection backward: dW_in[c][o] += sum_m x[m][c] dh[m][o]
// ---------------------------------------------------------------------------------------------------
// One CTA per 128 tokens; thread (o, half) accumulates 32 input channels of output column o per 64-channel
// chunk, the x tile staged in shared memory (broadcast float4 reads), dh read once per chunk (coalesced).
__global__ void __launch_bounds__(256)
embed_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dh, float* __restrict__ dW, int M, int C) {
  pdl_trigger();
  pdl_wait();
  constexpr int ROWS = 128;
  __shared__ __align__(16) float xs[ROWS][64];
  const int tid = threadIdx.x, o = tid & 127, half = tid >> 7;
  const int m0 = blockIdx.x * ROWS;
  const int rows = min(ROWS, M - m0);
  for (int c0 = 0; c0 < C; c0 += 64) {
    for (int i = tid; i < ROWS * 64; i += 256) {
      const int r = i >> 6, j = i & 63;
      xs[r][j] = (r < rows && c0 + j < C) ? x[static_cast<size_t>(m0 + r) * C + c0 + j] : 0.f;
    }
    __syncthreads();
    float acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = 0.f;
    for (int rb = 0; rb < rows; rb += 8) {
      float d[8];
#pragma unroll
      for (int q = 0; q < 8; ++q)   // 8 independent loads in flight per thread
        d[q] = (rb + q < rows) ? dh[static_cast<size_t>(m0 + rb + q) * 128 + o] : 0.f;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4* xr = reinterpret_cast<const float4*>(&xs[rb + q][half * 32]);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 v = xr[j];
          acc[4 * j] = fmaf(v.x, d[q], acc[4 * j]);
          acc[4 * j + 1] = fmaf(v.y, d[q], acc[4 * j + 1]);
          acc[4 * j + 2] = fmaf(v.z, d[q], acc[4 * j + 2]);
          acc[4 * j + 3] = fmaf(v.w, d[q], acc[4 * j + 3]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int cc = c0 + half * 32 + j;
      if (cc < C) atomicAdd(dW + static_cast<size_t>(cc) * 128 + o, acc[j]);
    }
    __syncthreads();
  }
}
inline void launch_embed_bwd(const float* x, const float* dh, float* dW, int M, int C, cudaStream_t st) {
  embed_bwd_kernel<<<(M + 127) / 128, 256, 0, st>>>(x, dh, dW, M, C);
}

// small fp32 linear layers of the FiLM generator: weight gradient and input gradient (tiled SGEMM, kernels.cu)
inline void launch_small_linear_bwd_w(const float* x, const float* g, float* dW, int R, int K, int N, cudaStream_t st) {
  launch_sgemm_small(2, x, g, nullptr, dW, nullptr, nullptr, K, N, R, 0, st);   // dW[K][N] = x[R][K]^T g[R][N]
}
inline void launch_small_linear_bwd_x(const float* g, const float* W, const float* pre, float* dx, int R, int K, int N,
                                      cudaStream_t st) {
  launch_sgemm_small(1, g, W, nullptr, dx, nullptr, pre, R, K, N, 0, st);       // dx[R][K] = g[R][N] W[K][N]^T
}

// ---------------------------------------------------------------------------------------------------
// objective: per-example loss, d loss / d pred (fp32 + zero-padded bf16 operand), running loss sum
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ddpm_loss_bwd_kernel(const float* __restrict__ eps, const float* __restrict__ pred, float* __restrict__ loss,
                     float* __restrict__ loss_sum, unsigned int* __restrict__ done_counter, float inv_global_batch,
                     float* __restrict__ dpred32, __nv_bfloat16* __restrict__ dpred16, float gscale, int S, int C, int Cp,
                     const float* const* __restrict__ ind, int objective) {
  pdl_trigger();
  if (ind) eps = ind[2];
  const int b = blockIdx.x;
  const int per = S * C;
  const size_t base = static_cast<size_t>(b) * per;
  float s = 0.f;
  for (int i = threadIdx.x; i < per; i += blockDim.x) {
    // ddpm (utils/losses.py:304-306): (eps - pred)^2, d/dpred = -2 (eps - pred).  dsm (:166-177) with pred = the RAW network
    // output (score * sigma): 0.5 (pred + eps)^2 summed, d/dpred = pred + eps.
    const float d = objective == 1 ? pred[base + i] + eps[base + i] : eps[base + i] - pred[base + i];
    s += d * d;
    const float gval = (objective == 1 ? d : -2.0f * d) * gscale;
    dpred32[base + i] = gval;
    const int row = i / C, c = i % C;
    dpred16[(static_cast<size_t>(b) * S + row) * Cp + c] = __float2bfloat16_rn(gval);
  }
  __shared__ float red[8];
  __shared__ bool last;
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
    for (int j = 0; j < 8; ++j) v += red[j];
    v = objective == 1 ? 0.5f * v : v / static_cast<float>(per);
    loss[b] = v;
    last = false;
    if (loss_sum) {
      // the block that finishes last adds the per-example losses in index order: the reported loss is bit-reproducible
      // (an atomicAdd per block would make its summation order depend on block scheduling)
      __threadfence();
      last = atomicInc(done_counter, gridDim.x - 1) == gridDim.x - 1;   // wraps back to 0 for the next launch
    }
  }
  __syncthreads();
  if (last && threadIdx.x < 32) {
    __threadfence();
    float acc = 0.f;
    // fixed association: lane-strided partials, then the butterfly
    for (int i = threadIdx.x; i < static_cast<int>(gridDim.x); i += 32) acc += __ldcg(loss + i);
    acc = warp_sum(acc);
    if (threadIdx.x == 0) { loss_sum[0] = acc; loss_sum[1] = acc * inv_global_batch; }
  }
}

}  // namespace smd

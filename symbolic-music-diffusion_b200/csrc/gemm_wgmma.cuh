// Persistent, warp-specialised bf16 x bf16 -> fp32 GEMM for sm_90a:
//   TMA (cp.async.bulk.tensor, SWIZZLE_128B) -> shared-memory ring -> wgmma (two consumer warpgroups, 64 rows each,
//   fp32 accumulators in registers) -> accumulator tile staged row-major in shared memory -> epilogue fused with
//   bias / residual / activation / LayerNorm / row statistics.
//
//   D[M,N] = A[M,K] * B[N,K]^T     (both operands may independently be K-major or MN-major in global memory)
//
// One CTA per 128 x BN tile (BN <= 128).  Two thread layouts (kEW below):
//   * dedicated epilogue (kEW = 4, 512 threads): warpgroup 0 is the TMA producer, warpgroups 1 and 2 only run the K
//     loops and store their accumulators to `acc_tile`, warpgroup 3 runs the epilogue.  The accumulator hand-off goes
//     through two mbarriers (acc_full / acc_empty), so the MMA warps start tile i + 1 while the epilogue warps still
//     work on tile i: the tensor cores do not wait for the epilogue's HBM traffic.  setmaxnreg moves registers from
//     the producer and MMA warpgroups to the epilogue warpgroup.  Used for the long-K fp32 / bf16 kinds of launches
//     with more tiles than CTAs;
//   * shared (kEW = 8 or 12): the two wgmma warpgroups are also epilogue warps (plus a third, epilogue-only warpgroup
//     for kEW = 12).  While they run the epilogue of tile i, the TMA warp already streams the operands of tile i + 1
//     into the ring, but no MMA runs.  Single-round launches gain nothing from the overlap and keep the wider
//     epilogue; so do the short-K, LayerNorm, generic and strict kinds.
//
// This is the kernel behind every Dense layer on the hot path (reference: flax.nn.Dense call sites
// models/ncsn.py:155-178, models/shared.py:65,69).
#pragma once
#include <cuda.h>
#include <type_traits>
#include "ptx.cuh"

namespace smd {

enum : int { ACT_NONE = 0, ACT_GELU_TANH = 1, ACT_SWISH = 2 };

// Compile-time epilogue feature mask: the kernel is instantiated for a handful of feature sets so that each launch
// carries only the epilogue code it needs (the all-features build was ~23k SASS instructions and stalled on
// instruction fetch).  kEpiGeneric keeps every feature, the ragged / unaligned row-per-thread path included.
enum : uint32_t {
  F_BIAS = 1u, F_RES = 2u, F_F32 = 4u, F_BF16 = 8u, F_PRE = 16u, F_STATS = 32u, F_LN = 64u, F_GG = 128u,
  F_ATOMIC = 256u, F_ACT = 512u, F_RAGGED = 1024u, F_SCALE = 2048u, F_STRICT = 8192u
};
static constexpr uint32_t kEpiGeneric = 0xFFFu;
// strict-precision mode (bf16x3): the generic epilogue plus lo-half stores and exact activations.  A separate
// instantiation on purpose: carrying that code as a runtime branch in the specialised kinds cost the FFN-up / dX GEMMs
// a factor of 2.6 (register pressure and instruction fetch in the bf16 store path).
static constexpr uint32_t kEpiStrict = kEpiGeneric | F_STRICT;
static constexpr uint32_t kEpiF32 = F_BIAS | F_F32 | F_STATS;                     // qkv, post, res-block a, dX outputs
static constexpr uint32_t kEpiF32Res = F_BIAS | F_RES | F_F32 | F_STATS;          // res-block b
static constexpr uint32_t kEpiAct = F_BIAS | F_ACT | F_BF16 | F_PRE | F_STATS;    // FFN up (+GELU); res-block a (bf16 + row stats)
static constexpr uint32_t kEpiLn = F_BIAS | F_RES | F_F32 | F_LN | F_BF16;        // attention out / FFN down + LayerNorm
static constexpr uint32_t kEpiGG = F_GG | F_BF16;                                 // FFN backward (x gelu')
static constexpr uint32_t kEpiAtomic = F_F32 | F_ATOMIC;                          // split-K weight gradients

struct GemmEpilogue {
  const float* bias;            // [N] or null
  const float* residual;        // fp32 [M][ld_res] or null  (v = acc + bias + residual)
  int ld_res;
  float* out_f32;               // fp32 [M][ld_f32] <- v, or null
  int ld_f32;
  __nv_bfloat16* out_bf16;      // bf16 [M][ld_bf16] <- act(v)   (or LayerNorm(v) when ln_gamma != null), or null
  int ld_bf16;
  int act;                      // activation applied on the bf16 output path
  float* row_stats;             // [M][2] += (sum v, sum v^2) over this tile's columns (atomics), or null
  float* stats_part;            // if set (with row_stats): instead of atomics every (n-tile, column-group) pair stores its
                                // partial to stats_part[(row * nslots + n_tile * groups + group) * 2], groups =
                                // GemmSmem::kEpiGroups; the consumer (ln_film_act) adds the slots in a fixed order:
                                // bit-reproducible statistics
  const float* ln_gamma;        // full-row LayerNorm (requires N <= BN, a single n-tile): bf16 out = LN(v)*g+b
  const float* ln_beta;
  __nv_bfloat16* out_bf16_pre;  // bf16 [M][ld_bf16] <- v before the activation (training saves), or null
  float out_scale;              // v is multiplied by out_scale before everything else if != 0 (0 means 1)
  int atomic_out;               // out_f32 += v with atomics (split-K weight-gradient GEMMs; buffer pre-zeroed)
  const __nv_bfloat16* gelu_grad_of;  // v *= gelu_tanh'(gelu_grad_of[row][col]) (FFN backward), or null
  int ld_gg;
  // ---- strict-precision mode (bf16x3): every bf16 operand written through out_bf16 also gets its lo half at
  // out_bf16 + lo_delta (elements), and the activations use exact tanhf / expf.  0 = off.
  long long lo_delta;
};

struct GemmShape {
  int M, N, K;     // logical problem; K % 64 == 0
  int BN;          // n-tile width: multiple of 16, <= kBNMax
  int a_mn, b_mn;  // 0: operand is K-major ([rows][K], K contiguous); 1: MN-major ([K][rows], rows contiguous)
  int k_splits;    // >= 1: the K loop is cut into this many independent tiles (needs atomic_out when > 1)
};

static constexpr int kBM = 128;
static constexpr int kBK = 64;
static constexpr int kBNMax = 128;                 // widest n-tile: one m64n128 wgmma per consumer warpgroup
// floats per staged accumulator row: unpadded, the 16-byte chunks of each row are XOR-swizzled instead (acc_chunk), which
// leaves room in shared memory for a fourth operand stage in the 8-epilogue-warp kinds
static constexpr int kAccPitch = kBNMax;

// kEW = number of epilogue warps.  8: two per 32-row quadrant; 12: three, for epilogue-bound small-K GEMMs.  The first
// eight of them are the two wgmma warpgroups.  4: the dedicated-epilogue layout, one warp per quadrant in a warpgroup
// of its own, after the two wgmma warpgroups.
// Each tile's columns are split into kEpiGroups column groups (group g owns the 32-column chunks g, g + kEpiGroups,
// ...): one per warp of a quadrant in the shared layouts; a dedicated epilogue warp runs both groups of its quadrant
// one after the other, so its arithmetic and its statistics slots are those of the 8-warp layout.
// The pipeline depth is whatever fits next to the accumulator staging tile and the epilogue scratch in the 227 KB of
// shared memory.
static constexpr int epi_groups(int ew) { return ew == 4 ? 2 : ew / 4; }   // column groups per tile of layout ew
template <int kEW = 8>
struct GemmSmem {
  static constexpr int kABytes = kBM * kBK * 2;            // 16 KB
  static constexpr int kBBytes = kBNMax * kBK * 2;         // 16 KB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBarBytes = 256;
  static constexpr int kEpiWarps = kEW;
  static constexpr bool kDedicated = kEW == 4;
  static constexpr int kEpiGroups = epi_groups(kEW);
  static constexpr int kAccBytes = kBM * kAccPitch * 4;                    // 64 KB fp32 accumulator tile
  static constexpr int kScrPerWarp = 32 * 33;                              // floats of scratch per epilogue warp
  static constexpr int kScratchBytes = kEpiWarps * kScrPerWarp * 4;        // per-epilogue-warp transpose scratch
  static constexpr int kMaxSmem = 232448;                                  // 227 KB
  static constexpr int kStages = (kMaxSmem - 1024 - kBarBytes - kAccBytes - kScratchBytes) / kStageBytes;
  static constexpr int kTotal = kStages * kStageBytes + kBarBytes + kAccBytes + kScratchBytes + 1024;
  static constexpr int kThreads = kDedicated ? 512 : 128 + 32 * kEpiWarps;
  // dedicated layout: per-thread register budgets of the producer, MMA and epilogue warpgroups (setmaxnreg).  The CTA
  // starts with 128 per thread (512 threads, one CTA per SM), so the four warpgroups' budgets may add up to 4 x 128.
  static constexpr int kProdRegs = 40, kMmaRegs = 120, kEpiRegs = 232;
  static_assert(!kDedicated || kProdRegs + 2 * kMmaRegs + kEpiRegs <= 512, "register budgets exceed the CTA's file");
};
// the 8-epilogue-warp and dedicated-epilogue kinds (every res-block GEMM of the train step) keep four 32 KB stages in
// flight
static_assert(GemmSmem<8>::kStages == 4, "the 8-warp GEMM ring should hold four stages");
static_assert(GemmSmem<4>::kStages == 4, "the dedicated-epilogue GEMM ring should hold four stages");

// MUFU.TANH (abs error ~5e-4, far below the bf16 rounding of everything that consumes it)
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float gelu_tanh_grad_f(float x) {
  const float c = 0.7978845608028654f;
  const float u = c * (x + 0.044715f * x * x * x);
  const float th = tanh_fast(u);
  return 0.5f * (1.0f + th) + 0.5f * x * (1.0f - th * th) * c * (1.0f + 3.0f * 0.044715f * x * x);
}

// exact variants for the strict-precision mode (the tanh.approx forms above are good to ~5e-4 absolute)
__device__ __forceinline__ float act_apply_exact(float v, int act) {
  if (act == ACT_GELU_TANH) {
    const float c = 0.7978845608028654f;
    return 0.5f * v * (1.0f + tanhf(c * (v + 0.044715f * v * v * v)));
  } else if (act == ACT_SWISH) {
    return v / (1.0f + expf(-v));
  }
  return v;
}
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 p = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&p);
}
// lo halves of a pair: bf16(x - float(bf16(x)))
__device__ __forceinline__ uint32_t pack_bf16x2_lo(float a, float b) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const float2 hf = __bfloat1622float2(h);
  __nv_bfloat162 p = __floats2bfloat162_rn(a - hf.x, b - hf.y);
  return *reinterpret_cast<uint32_t*>(&p);
}

__device__ __forceinline__ float act_apply(float v, int act) {
  if (act == ACT_GELU_TANH) {
    const float c = 0.7978845608028654f;
    const float u = v * fmaf(v * v, 0.044715f * c, c);   // c (v + 0.044715 v^3)
    const float h = 0.5f * v;
    return fmaf(h, tanh_fast(u), h);
  } else if (act == ACT_SWISH) {
    const float h = 0.5f * v;
    return fmaf(h, tanh_fast(h), h);   // v * sigmoid(v), sigmoid(v) = 0.5 + 0.5 tanh(v/2)
  }
  return v;
}

// fp32 pairs kept in one 64-bit register pair; every lane op is the same round-to-nearest fp32 operation as the scalar
// form, so results are bit-identical to act_apply().
__device__ __forceinline__ uint64_t f32x2_pack(float a, float b) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ void f32x2_unpack(uint64_t v, float& a, float& b) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v));
}
__device__ __forceinline__ uint64_t f32x2_add(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  f32x2_unpack(a, a0, a1); f32x2_unpack(b, b0, b1);
  return f32x2_pack(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ uint64_t f32x2_mul(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  f32x2_unpack(a, a0, a1); f32x2_unpack(b, b0, b1);
  return f32x2_pack(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ uint64_t f32x2_fma(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  f32x2_unpack(a, a0, a1); f32x2_unpack(b, b0, b1); f32x2_unpack(c, c0, c1);
  return f32x2_pack(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
// tanh-GELU of the pair v (same operation order as act_apply(ACT_GELU_TANH))
__device__ __forceinline__ uint64_t gelu_tanh_x2(uint64_t v) {
  const float c = 0.7978845608028654f, cc = 0.044715f * c;
  const uint64_t t = f32x2_fma(f32x2_mul(v, v), f32x2_pack(cc, cc), f32x2_pack(c, c));
  float u0, u1;
  f32x2_unpack(f32x2_mul(v, t), u0, u1);
  const uint64_t h = f32x2_mul(v, f32x2_pack(0.5f, 0.5f));
  return f32x2_fma(h, f32x2_pack(tanh_fast(u0), tanh_fast(u1)), h);
}

// Staged accumulator tile [128][kAccPitch]: 16-byte chunk q of row r sits at chunk q ^ (r & 7) of the row, so that
// 16-byte row reads with one row per lane, and the wgmma fragment stores, are free of bank conflicts without padding.
__device__ __forceinline__ int acc_chunk(int q, int sw) { return q ^ sw; }
// the staged accumulator row `p` (row & 7 == sw) of this thread: 32 / 16 consecutive columns from column c0 (a multiple
// of 16), 16-byte shared accesses
__device__ __forceinline__ void acc_ld32(const float* p, int c0, int sw, uint32_t (&r)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 t = reinterpret_cast<const float4*>(p)[acc_chunk((c0 >> 2) + i, sw)];
    r[4 * i] = __float_as_uint(t.x); r[4 * i + 1] = __float_as_uint(t.y);
    r[4 * i + 2] = __float_as_uint(t.z); r[4 * i + 3] = __float_as_uint(t.w);
  }
}
__device__ __forceinline__ void acc_ld16(const float* p, int c0, int sw, uint32_t (&r)[16]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 t = reinterpret_cast<const float4*>(p)[acc_chunk((c0 >> 2) + i, sw)];
    r[4 * i] = __float_as_uint(t.x); r[4 * i + 1] = __float_as_uint(t.y);
    r[4 * i + 2] = __float_as_uint(t.z); r[4 * i + 3] = __float_as_uint(t.w);
  }
}
__device__ __forceinline__ void acc_st32(float* p, int c0, int sw, const uint32_t (&r)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
    reinterpret_cast<float4*>(p)[acc_chunk((c0 >> 2) + i, sw)] =
        make_float4(__uint_as_float(r[4 * i]), __uint_as_float(r[4 * i + 1]), __uint_as_float(r[4 * i + 2]),
                    __uint_as_float(r[4 * i + 3]));
}

// Epilogue chunk I/O.  A warp owns 32 rows of the tile (row_base, row_base + 32) and works on 32-column chunks: lane l
// holds row l of the chunk in v[32].  Global reads and writes go through a per-warp 32x33 scratch so that they are whole
// row segments: fp32 as 4 rows x 128 B per instruction, bf16 as 8 rows x 64 B.  Rows >= M are not written.
// fp32 transpose tile: 16-byte chunk j of row r at chunk slot r * 8 + (j ^ (r & 7)) -- 128-bit shared accesses,
// conflict-free for "lane = row" and "8 lanes = one row"
__device__ __forceinline__ float4* t4(float* scr, int r, int j) {
  return reinterpret_cast<float4*>(scr) + (r * 8 + (j ^ (r & 7)));
}
__device__ __forceinline__ void add_pair(float& a, float& b, float x, float y) {   // (a, b) += (x, y)
  f32x2_unpack(f32x2_add(f32x2_pack(a, b), f32x2_pack(x, y)), a, b);
}
// the residual chunk at columns [col, col + 32), rows >= M read as zero
__device__ __forceinline__ void res_load(float4 (&rp)[8], const float* res, int ld, int row_base, int M, int col,
                                         uint32_t lane) {
  const int f_r = static_cast<int>(lane >> 3), f_c = static_cast<int>(lane & 7u) * 4;
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int grow = row_base + it * 4 + f_r;
    rp[it] = (grow < M) ? *reinterpret_cast<const float4*>(res + static_cast<size_t>(grow) * ld + col + f_c)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}
// v += residual chunk: res_stage puts what res_load read into the transpose tile (rp may then be reloaded), res_add
// adds it row per lane
__device__ __forceinline__ void res_stage(float* scr, const float4 (&rp)[8], uint32_t lane) {
  const int f_r = static_cast<int>(lane >> 3), f_c = static_cast<int>(lane & 7u) * 4;
#pragma unroll
  for (int it = 0; it < 8; ++it) *t4(scr, it * 4 + f_r, f_c >> 2) = rp[it];
}
__device__ __forceinline__ void res_add(float (&v)[32], float* scr, uint32_t lane) {
  __syncwarp();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 t = *t4(scr, static_cast<int>(lane), i);
    add_pair(v[4 * i], v[4 * i + 1], t.x, t.y);
    add_pair(v[4 * i + 2], v[4 * i + 3], t.z, t.w);
  }
  __syncwarp();
}
__device__ __forceinline__ void bias_add(float (&v)[32], const float4 (&b)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    add_pair(v[4 * i], v[4 * i + 1], b[i].x, b[i].y);
    add_pair(v[4 * i + 2], v[4 * i + 3], b[i].z, b[i].w);
  }
}
// (s1, s2) += the chunk's (sum, sumsq), summed as column pairs
__device__ __forceinline__ void chunk_stats(const float (&v)[32], float& s1, float& s2) {
  uint64_t a1 = f32x2_pack(0.f, 0.f), a2 = f32x2_pack(0.f, 0.f);
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const uint64_t pv = f32x2_pack(v[2 * i], v[2 * i + 1]);
    a1 = f32x2_add(a1, pv);
    a2 = f32x2_fma(pv, pv, a2);
  }
  float lo, hi;
  f32x2_unpack(a1, lo, hi); s1 += lo + hi;
  f32x2_unpack(a2, lo, hi); s2 += lo + hi;
}
// out[row][col, col + 32) = v (or += with atomics)
__device__ __forceinline__ void store_f32_chunk(float* scr, const float (&v)[32], uint32_t lane, int row_base, int M,
                                                float* out, int ld, int col, bool atomic) {
  const int f_r = static_cast<int>(lane >> 3), f_c = static_cast<int>(lane & 7u) * 4;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    *t4(scr, static_cast<int>(lane), i) = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
  __syncwarp();
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int rr = it * 4 + f_r, grow = row_base + rr;
    if (grow < M) {
      float* op = out + static_cast<size_t>(grow) * ld + col + f_c;
      if (atomic) {
        const float4 sp = *t4(scr, rr, f_c >> 2);
        atomicAdd(op, sp.x); atomicAdd(op + 1, sp.y); atomicAdd(op + 2, sp.z); atomicAdd(op + 3, sp.w);
      } else {
        *reinterpret_cast<float4*>(op) = *t4(scr, rr, f_c >> 2);   // a 16-byte copy: one vector load, one vector store
      }
    }
  }
  __syncwarp();
}
// out[row][col, col + 32) = the 32 bf16 values each lane has put in its row of scrw (scrw[lane * 33 + j]: pair j)
__device__ __forceinline__ void store_bf16_chunk(const uint32_t* scrw, uint32_t lane, int row_base, int M,
                                                 __nv_bfloat16* out, int ld, int col) {
  const int h_r = static_cast<int>(lane >> 2), h_c = static_cast<int>(lane & 3u) * 8;
  __syncwarp();
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int rr = it * 8 + h_r, grow = row_base + rr;
    if (grow < M) {
      const uint32_t* sp = scrw + rr * 33 + (h_c >> 1);
      *reinterpret_cast<uint4*>(out + static_cast<size_t>(grow) * ld + col + h_c) = make_uint4(sp[0], sp[1], sp[2], sp[3]);
    }
  }
  __syncwarp();
}
// LayerNorm of the chunk with the row's (mean, rstd) as bf16 pairs into the lane's row of scrw (lo: the lo halves,
// strict mode)
__device__ __forceinline__ void ln_pack(const float (&v)[32], float mean, float rstd, const float* gamma,
                                        const float* beta, bool lo, uint32_t* scrw, uint32_t lane) {
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 g = __ldg(g4 + i), b = __ldg(b4 + i);
    const float w0 = (v[4 * i] - mean) * (rstd * g.x) + b.x;
    const float w1 = (v[4 * i + 1] - mean) * (rstd * g.y) + b.y;
    const float w2 = (v[4 * i + 2] - mean) * (rstd * g.z) + b.z;
    const float w3 = (v[4 * i + 3] - mean) * (rstd * g.w) + b.w;
    scrw[lane * 33 + 2 * i] = lo ? pack_bf16x2_lo(w0, w1) : pack_bf16x2(w0, w1);
    scrw[lane * 33 + 2 * i + 1] = lo ? pack_bf16x2_lo(w2, w3) : pack_bf16x2(w2, w3);
  }
}

// the K loop of one warpgroup: rows [64 wg, 64 wg + 64) of the tile, all kBNMax columns
template <int kTA, int kTB>
__device__ __forceinline__ void gemm_mainloop(float (&d)[64], uint8_t* smem, int stage_bytes, int a_bytes, int stages,
                                              uint64_t* full_bar, uint64_t* empty_bar, int& stage, uint32_t& phase,
                                              int nkb, uint32_t wg, bool releaser) {
  // per-k16 advance of the descriptor start address (bytes): 32 B inside a K-major row, two 8-row atoms MN-major
  const uint32_t a_kadv = kTA ? 2048u : 32u, b_kadv = kTB ? 2048u : 32u;
  const uint32_t a_lbo = kTA ? 8192u : 0u, b_lbo = kTB ? 8192u : 0u;
  int prev = -1;
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sA = smem_u32(smem + stage * stage_bytes) + wg * 8192u;   // 64 rows: 8 KB in either major order
    const uint32_t sB = smem_u32(smem + stage * stage_bytes + a_bytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k)
      wgmma_m64n128k16_bf16<kTA, kTB>(d, make_smem_desc_sw128(sA + k * a_kadv, a_lbo, 1024u),
                                      make_smem_desc_sw128(sB + k * b_kadv, b_lbo, 1024u), (kb | k) != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();                       // the previous k block's MMAs are done: its slot can be refilled
    if (prev >= 0 && releaser) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == stages) { stage = 0; phase ^= 1u; }
  }
  wgmma_wait<0>();
  if (prev >= 0 && releaser) mbar_arrive(&empty_bar[prev]);
}

// (ep is __grid_constant__ like the tensor maps: its fields are read in place from parameter space; without it ptxas
// allocates the 8- and 12-warp epilogue kinds with more spills)
template <uint32_t kF, int kEW = 8>
__global__ void __launch_bounds__(GemmSmem<kEW>::kThreads, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const GemmShape sh, const __grid_constant__ GemmEpilogue ep) {
  using SM = GemmSmem<kEW>;
  constexpr bool kDedicated = SM::kDedicated;
  constexpr int kGroups = SM::kEpiGroups;
  static_assert(SM::kStages >= 3, "pipeline too shallow");
  static_assert(!((kF & F_LN) && !(kF & F_RAGGED)) || kEW == 8, "the paired LayerNorm epilogue needs 8 epilogue warps");
  static_assert(!kDedicated || (kF & (F_LN | F_RAGGED | F_STRICT)) == 0,
                "the dedicated-epilogue layout runs the non-LayerNorm fast-path epilogue only");
  static_assert(2 * SM::kStages + 2 <= SM::kBarBytes / 8, "mbarriers do not fit their region");
  extern __shared__ uint8_t smem_raw[];
  // 1 KiB alignment by OFFSET from the __shared__ symbol (not by integer-casting the pointer): the compiler keeps the
  // shared address space, so the epilogue's staging accesses are LDS/STS instead of generic LD/ST.
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SM::kStages * SM::kStageBytes);
  uint64_t* full_bar = bars;                         // [kStages]
  uint64_t* empty_bar = bars + SM::kStages;          // [kStages]
  uint64_t* acc_full = bars + 2 * SM::kStages;       // dedicated layout: acc_tile holds a finished tile
  uint64_t* acc_empty = acc_full + 1;                // dedicated layout: the epilogue is done reading acc_tile
  float* acc_tile = reinterpret_cast<float*>(smem + SM::kStages * SM::kStageBytes + SM::kBarBytes);   // [128][kAccPitch]
  uint8_t* epi_smem = smem + SM::kStages * SM::kStageBytes + SM::kBarBytes + SM::kAccBytes;         // scratch

  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t lane = threadIdx.x & 31;

  const int BN = sh.BN;
  const int rows_per_tile = kBM;
  const int num_m = (sh.M + rows_per_tile - 1) / rows_per_tile;
  const int num_n = (sh.N + BN - 1) / BN;
  const int splits = sh.k_splits > 0 ? sh.k_splits : 1;
  const int num_tiles = num_m * num_n * splits;
  const int num_kb_total = sh.K / kBK;
  const int kb_per = (num_kb_total + splits - 1) / splits;
  const int group = blockIdx.x;
  const int num_groups = gridDim.x;
  const int b_rows = BN;  // B rows staged per k block

  pdl_trigger();   // the next kernel of the stream may start its own prologue now
  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  if (warp == 1 && elect_one()) {
    for (int i = 0; i < SM::kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);   // one arrival per MMA warp
    }
    if (kDedicated) {
      mbar_init(acc_full, 256);      // every MMA thread, after its fragment stores
      mbar_init(acc_empty, 128);     // every epilogue thread, after its last read of the tile
    }
    fence_barrier_init();
  }
  __syncthreads();
  // Everything above (barrier init, descriptor prefetch) touched no global data: under programmatic dependent launch
  // it overlaps the tail of the previous kernel.  From here on operands are read.
  pdl_wait();

  const uint32_t wg = (warp - 4u) >> 2;          // consumer warpgroup (0, 1: MMA; 2: epilogue only)
  int mma_stage = 0; uint32_t mma_phase = 0;
  // the K loop of one tile: this warpgroup's 64 rows, all kBNMax columns, into d
  auto mainloop = [&](int tile, float (&d)[64]) {
    const int split = tile % splits;
    const int kb0 = split * kb_per, kb1 = min(num_kb_total, kb0 + kb_per);
    const int nkb = kb1 - kb0;
    const bool rel = lane == 0;
    if (!sh.a_mn && !sh.b_mn) gemm_mainloop<0, 0>(d, smem, SM::kStageBytes, SM::kABytes, SM::kStages, full_bar, empty_bar, mma_stage, mma_phase, nkb, wg, rel);
    else if (!sh.a_mn) gemm_mainloop<0, 1>(d, smem, SM::kStageBytes, SM::kABytes, SM::kStages, full_bar, empty_bar, mma_stage, mma_phase, nkb, wg, rel);
    else if (!sh.b_mn) gemm_mainloop<1, 0>(d, smem, SM::kStageBytes, SM::kABytes, SM::kStages, full_bar, empty_bar, mma_stage, mma_phase, nkb, wg, rel);
    else gemm_mainloop<1, 1>(d, smem, SM::kStageBytes, SM::kABytes, SM::kStages, full_bar, empty_bar, mma_stage, mma_phase, nkb, wg, rel);
  };
  // the warpgroup's accumulator fragments -> acc_tile
  auto stage_acc = [&](const float (&d)[64]) {
    const int r0 = static_cast<int>(wg * 64u + ((warp - 4u) & 3u) * 16u + (lane >> 2));
    const int c = 2 * static_cast<int>(lane & 3u);
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int rr = r0 + 8 * ((i >> 1) & 1), cc = 8 * (i >> 2) + c;
      *reinterpret_cast<float2*>(acc_tile + rr * kAccPitch + acc_chunk(cc >> 2, rr & 7) * 4 + (cc & 3)) =
          make_float2(d[i], d[i + 1]);
    }
  };

  if (warp < 4) {
    // ===================== TMA producer (one lane of warp 0) =====================
    if constexpr (kDedicated) setmaxnreg_dec<SM::kProdRegs>();
    if (warp == 0 && elect_one()) {
      int stage = 0; uint32_t phase = 0;
      const uint32_t stage_tx = static_cast<uint32_t>((kBM + b_rows) * kBK * 2);
      for (int tile = group; tile < num_tiles; tile += num_groups) {
        const int mn = tile / splits, split = tile % splits;
        const int m_row0 = (mn / num_n) * rows_per_tile;
        const int n_row0 = (mn % num_n) * BN;
        const int kb0 = split * kb_per, kb1 = min(num_kb_total, kb0 + kb_per);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          uint8_t* sA = smem + stage * SM::kStageBytes;
          uint8_t* sB = sA + SM::kABytes;
          const int k0 = kb * kBK;
          mbar_arrive_expect_tx(&full_bar[stage], stage_tx);
          if (!sh.a_mn) tma_load_2d(&tmA, &full_bar[stage], sA, k0, m_row0);
          else
            for (int j = 0; j < kBM / 64; ++j) tma_load_2d(&tmA, &full_bar[stage], sA + j * 8192, m_row0 + 64 * j, k0);
          if (!sh.b_mn) tma_load_2d(&tmB, &full_bar[stage], sB, k0, n_row0);
          else
            for (int j = 0; j < b_rows / 64; ++j) tma_load_2d(&tmB, &full_bar[stage], sB + j * 8192, n_row0 + 64 * j, k0);
          if (++stage == SM::kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else if (kDedicated && wg < 2) {
    // ===================== dedicated layout: MMA warps =====================
    // Tile i's accumulators go to acc_tile as soon as the epilogue has released tile i - 1, then tile i + 1's K loop
    // starts while the epilogue warpgroup works on tile i.
    setmaxnreg_dec<SM::kMmaRegs>();
    uint32_t acc_phase = 0;
    for (int tile = group; tile < num_tiles; tile += num_groups) {
      float d[64];
      mainloop(tile, d);
      mbar_wait(acc_empty, acc_phase ^ 1u);
      stage_acc(d);
      mbar_arrive(acc_full);
      acc_phase ^= 1u;
    }
  } else {
    // ===================== epilogue warps (and, in the shared layouts, MMA warps) =====================
    // Per tile in the shared layouts: the two wgmma warpgroups (epilogue warps 0-7) run the K loop, every epilogue
    // warp waits until the previous tile's staged accumulators have been consumed, the warpgroups store theirs to
    // `acc_tile`.  In the dedicated layout the epilogue warps wait on acc_full instead.  Then each warp reads its 32
    // rows back one row per thread, exactly like the epilogue expects: every global tile access goes through a
    // per-warp 32x33 shared-memory scratch and is issued as whole 128-byte (fp32) / 64-byte (bf16) row segments.
    if constexpr (kDedicated) setmaxnreg_inc<SM::kEpiRegs>();
    auto epi_bar = [] { asm volatile("bar.sync 5, %0;" ::"n"(32 * kEW) : "memory"); };
    auto mma_tile = [&](int tile) {
      float d[64];
      const bool mma_warp = wg < 2;
      if (mma_warp) mainloop(tile, d);
      epi_bar();                                 // the previous tile's accumulators have been read by every warp
      if (mma_warp) stage_acc(d);
      epi_bar();
    };
    constexpr bool H_BIAS = (kF & F_BIAS) != 0, H_RES = (kF & F_RES) != 0, H_F32 = (kF & F_F32) != 0;
    constexpr bool H_BF16 = (kF & F_BF16) != 0, H_PRE = (kF & F_PRE) != 0, H_STATS = (kF & F_STATS) != 0;
    constexpr bool H_LN = (kF & F_LN) != 0, H_GG = (kF & F_GG) != 0, H_ATOMIC = (kF & F_ATOMIC) != 0;
    constexpr bool H_ACT = (kF & F_ACT) != 0, H_RAGGED = (kF & F_RAGGED) != 0, H_SCALE = (kF & F_SCALE) != 0;
    constexpr bool H_STRICT = (kF & F_STRICT) != 0;
    const long long lo_delta = H_STRICT ? ep.lo_delta : 0;
    const uint32_t q = warp & 3u;                      // 32-row quadrant of the tile this warp owns
    const int asw = static_cast<int>(lane & 7u);       // swizzle of this thread's staged row (q * 32 + lane)
    const uint32_t ew = warp - (kDedicated ? 12u : 4u);   // epilogue warp index
    // column group of this warp in the shared layouts: the warps of a quadrant split the chunks
    const int eg = static_cast<int>(ew) >> 2;
    float* scr = reinterpret_cast<float*>(epi_smem) + ew * SM::kScrPerWarp;
    uint32_t* scrw = reinterpret_cast<uint32_t*>(scr);
    const int f_r = static_cast<int>(lane >> 3), f_c = static_cast<int>(lane & 7u) * 4;  // fp32: 4 rows x 128 B / instr
    const int h_r = static_cast<int>(lane >> 2), h_c = static_cast<int>(lane & 3u) * 8;  // bf16: 8 rows x 64 B / instr
    const float oscale = (H_SCALE && ep.out_scale != 0.0f) ? ep.out_scale : 1.0f;
    const bool has_bias = H_BIAS && ep.bias != nullptr;
    const bool has_res = H_RES && ep.residual != nullptr;
    const bool has_f32 = H_F32 && ep.out_f32 != nullptr;
    const bool has_bf16 = H_BF16 && ep.out_bf16 != nullptr;
    const bool has_pre = H_PRE && ep.out_bf16_pre != nullptr;
    const bool has_stats = H_STATS && ep.row_stats != nullptr;
    const bool do_ln = H_LN && ep.ln_gamma != nullptr;
    const bool has_gg = H_GG && ep.gelu_grad_of != nullptr;
    const bool atomic_out = H_ATOMIC && ep.atomic_out != 0;
    const int act = H_ACT ? ep.act : ACT_NONE;
    const bool aligned_ok = !H_RAGGED ||
                            ((!has_res || (ep.ld_res & 3) == 0) && (!has_f32 || (ep.ld_f32 & 3) == 0) &&
                             ((!has_bf16 && !has_pre) || (ep.ld_bf16 & 7) == 0) && (!has_gg || (ep.ld_gg & 7) == 0));
    // Work items are (tile, column group) pairs: a shared-layout warp runs its own group `eg` of each of its tiles, a
    // dedicated epilogue warp both groups of each tile, one after the other.
    constexpr int kPer = kDedicated ? kGroups : 1;
    const int warp_eg = eg;
    uint32_t acc_phase = 0;
    for (int item = 0;; ++item) {
      const int tile = group + (item / kPer) * num_groups;
      if (tile >= num_tiles) break;
      const int eg = kDedicated ? item % kPer : warp_eg;
      if (item % kPer == 0) {
        if constexpr (kDedicated) mbar_wait(acc_full, acc_phase);
        else mma_tile(tile);
      }
      const int mn = tile / splits;
      const bool first_split = (tile % splits) == 0;
      const int row_base = (mn / num_n) * rows_per_tile + static_cast<int>(q * 32u);
      const int row = row_base + static_cast<int>(lane);
      const int n0 = (mn % num_n) * BN;
      const bool row_ok = row < sh.M;
      float* const arow = acc_tile + (q * 32u + lane) * kAccPitch;
      float s1 = 0.f, s2 = 0.f;
      // software prefetch of the residual / gelu-grad tiles of the NEXT chunk (their global latency would
      // otherwise be fully exposed: only two warps per SM sub-partition work on the epilogue)
      float4 rpre[H_RES ? 8 : 1];
      uint4 gpre[H_GG ? 4 : 1];
      const bool pre_res = has_res && first_split && aligned_ok;
      const bool pre_gg = has_gg && aligned_ok;
      auto prefetch = [&](int c) {
        const int colp = n0 + c;
        if constexpr (H_RES) {
          if (pre_res) res_load(rpre, ep.residual, ep.ld_res, row_base, sh.M, colp, lane);
        }
        if constexpr (H_GG) {
          if (pre_gg) {
#pragma unroll
            for (int it = 0; it < 4; ++it) {
              const int grow = row_base + it * 8 + h_r;
              gpre[it] = (grow < sh.M) ? *reinterpret_cast<const uint4*>(ep.gelu_grad_of + static_cast<size_t>(grow) * ep.ld_gg + colp + h_c)
                                       : make_uint4(0u, 0u, 0u, 0u);
            }
          }
        }
      };
      if constexpr (H_LN && !H_RAGGED) {
        // ---------- single-pass full-row LayerNorm (N == BN <= 128, so n0 == 0: attention out-proj, FFN down) ----------
        // The two warps of a row quadrant split the row's chunks, keep their values in registers, exchange the
        // per-row (sum, sumsq) partials through shared memory (named barrier of 64 threads) and each normalises
        // and stores its own chunks: no second pass over the staged tile, no global re-read.
        const float* scr_partner = reinterpret_cast<const float*>(epi_smem) + (ew ^ 4u) * SM::kScrPerWarp;
        const int nchunk = BN / 64;
        float vv[2][32];
        prefetch(eg * 32);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          if (j < nchunk) {
            const int c0 = eg * 32 + 64 * j;
            __syncwarp();
            uint32_t r[32];
            acc_ld32(arow, c0, asw, r);
#pragma unroll
            for (int i = 0; i < 32; ++i) vv[j][i] = __uint_as_float(r[i]);
            if (has_bias) {
              float4 bq[8];
              const float4* b4 = reinterpret_cast<const float4*>(ep.bias + c0);
#pragma unroll
              for (int i = 0; i < 8; ++i) bq[i] = __ldg(b4 + i);
              bias_add(vv[j], bq);
            }
            if (has_res) {
              res_stage(scr, rpre, lane);
              if (j + 1 < nchunk) prefetch(eg * 32 + 64 * (j + 1));
              res_add(vv[j], scr, lane);
            }
            chunk_stats(vv[j], s1, s2);
            if (has_f32) store_f32_chunk(scr, vv[j], lane, row_base, sh.M, ep.out_f32, ep.ld_f32, c0, false);
          }
        }
        // exchange the row partials with the partner warp of this quadrant
        scr[lane * 33] = s1; scr[lane * 33 + 1] = s2;
        asm volatile("bar.sync %0, 64;" ::"r"(1u + q) : "memory");
        const float t1 = s1 + scr_partner[lane * 33], t2 = s2 + scr_partner[lane * 33 + 1];
        asm volatile("bar.sync %0, 64;" ::"r"(1u + q) : "memory");
        const float inv_n = 1.0f / static_cast<float>(sh.N);
        const float mean = t1 * inv_n;
        const float rstd = rsqrtf(t2 * inv_n - mean * mean + 1e-6f);   // flax LayerNorm: E[x^2] - E[x]^2, eps 1e-6
        if (has_bf16) {
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            if (j < nchunk) {
              const int c0 = eg * 32 + 64 * j;
              ln_pack(vv[j], mean, rstd, ep.ln_gamma + c0, ep.ln_beta + c0, false, scrw, lane);
              store_bf16_chunk(scrw, lane, row_base, sh.M, ep.out_bf16, ep.ld_bf16, c0);
            }
          }
        }
      } else {
        float mean = 0.f, rstd = 0.f;
        const int npass = do_ln ? 2 : 1;
        // full-row LayerNorm needs one warp to see the whole row: group 1 sits those tiles out
        const int c_begin = do_ln ? (eg == 0 ? 0 : BN) : eg * 32;
        const int c_step = do_ln ? 32 : 32 * kGroups;
        auto chunk_fast = [&](int c) {
          return !H_RAGGED || ((BN - c) >= 32 && aligned_ok && (n0 + c + 32 <= sh.N));
        };
        if (c_begin < BN && chunk_fast(c_begin)) prefetch(c_begin);
        for (int pass = 0; pass < npass; ++pass) {
          for (int c0 = c_begin; c0 < BN; c0 += c_step) {
            __syncwarp();
            uint32_t r[32];
            bool half = false;
            if constexpr (H_RAGGED) half = (BN - c0) < 32;  // 16-column tail
            if (!half) {
              acc_ld32(arow, c0, asw, r);
            } else {
              uint32_t r16[16];
              acc_ld16(arow, c0, asw, r16);
#pragma unroll
              for (int i = 0; i < 16; ++i) { r[i] = r16[i]; r[16 + i] = 0u; }
            }
            const int col0 = n0 + c0;
            // the chunk's 32 bias values are fetched next to the staged-row load
            float4 bq[H_BIAS ? 8 : 1];
            if constexpr (H_BIAS) {
              if (has_bias && first_split && chunk_fast(c0)) {
                const float4* b4 = reinterpret_cast<const float4*>(ep.bias + col0);
#pragma unroll
                for (int i = 0; i < 8; ++i) bq[i] = __ldg(b4 + i);
              }
            }
            const int ncols = half ? 16 : 32;
            float v[32];
            if constexpr (H_SCALE) {
#pragma unroll
              for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]) * oscale;
            } else {
#pragma unroll
              for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]);
            }
            const bool reload = H_LN && (pass == 1) && has_f32;
            const bool write_bf16 = has_bf16 && (do_ln ? (pass == 1) : true);

            if (chunk_fast(c0)) {
              // ------------------------------ fast path: full 32-column chunk ------------------------------
              if (reload) {
                // LayerNorm pass 1: take v back from what this warp stored in pass 0 (the residual may alias the
                // output buffer, so it must not be re-added); __syncwarp orders the warp's own global writes
#pragma unroll
                for (int it = 0; it < 8; ++it) {
                  const int rr = it * 4 + f_r, grow = row_base + rr;
                  float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
                  if (grow < sh.M) t = *reinterpret_cast<const float4*>(ep.out_f32 + static_cast<size_t>(grow) * ep.ld_f32 + col0 + f_c);
                  float* d = scr + rr * 33 + f_c;
                  d[0] = t.x; d[1] = t.y; d[2] = t.z; d[3] = t.w;
                }
                __syncwarp();
#pragma unroll
                for (int i = 0; i < 32; ++i) v[i] = scr[lane * 33 + i];
                __syncwarp();
              } else {
                if constexpr (H_BIAS) {
                  if (has_bias && first_split) bias_add(v, bq);
                }
                uint4 gcur[H_GG ? 4 : 1];
                if constexpr (H_RES) {
                  if (pre_res) res_stage(scr, rpre, lane);
                }
                if constexpr (H_GG) {
                  if (pre_gg) {
#pragma unroll
                    for (int it = 0; it < 4; ++it) gcur[it] = gpre[it];
                  }
                }
                // issue the next chunk's global loads now: they complete while this chunk is processed
                if (pass == 0) {
                  const int cn = c0 + c_step;
                  if (cn < BN && chunk_fast(cn)) prefetch(cn);
                }
                if constexpr (H_RES) {
                  if (pre_res) res_add(v, scr, lane);
                }
                if constexpr (H_GG) {
                  if (pre_gg) {
#pragma unroll
                    for (int it = 0; it < 4; ++it) {
                      const __nv_bfloat162* hp = reinterpret_cast<const __nv_bfloat162*>(&gcur[it]);
                      float* d = scr + (it * 8 + h_r) * 33 + h_c;
#pragma unroll
                      for (int j = 0; j < 4; ++j) { const float2 f = __bfloat1622float2(hp[j]); d[2 * j] = f.x; d[2 * j + 1] = f.y; }
                    }
                    __syncwarp();
#pragma unroll
                    for (int i = 0; i < 32; ++i) v[i] *= gelu_tanh_grad_f(scr[lane * 33 + i]);
                    __syncwarp();
                  }
                }
              }
              if (pass == 0) {
                if constexpr (H_STATS || H_LN) {
                  if (has_stats || do_ln) chunk_stats(v, s1, s2);
                }
                if constexpr (H_F32) {
                  if (has_f32) store_f32_chunk(scr, v, lane, row_base, sh.M, ep.out_f32, ep.ld_f32, col0, H_ATOMIC && atomic_out);
                }
                if constexpr (H_PRE) {
                  if (has_pre) {
#pragma unroll
                    for (int j = 0; j < 16; ++j) scrw[lane * 33 + j] = pack_bf16x2(v[2 * j], v[2 * j + 1]);
                    store_bf16_chunk(scrw, lane, row_base, sh.M, ep.out_bf16_pre, ep.ld_bf16, col0);
                  }
                }
              }
              if constexpr (H_BF16) {
                if (write_bf16) {
                  for (int lo = 0; lo < ((H_STRICT && lo_delta) ? 2 : 1); ++lo) {   // strict mode: second sweep = lo halves
                    if (H_LN && do_ln) {
                      ln_pack(v, mean, rstd, ep.ln_gamma + col0, ep.ln_beta + col0, lo != 0, scrw, lane);
                    } else if (H_STRICT && lo_delta) {
#pragma unroll
                      for (int j = 0; j < 16; ++j) {
                        const float y0 = act_apply_exact(v[2 * j], act), y1 = act_apply_exact(v[2 * j + 1], act);
                        scrw[lane * 33 + j] = lo ? pack_bf16x2_lo(y0, y1) : pack_bf16x2(y0, y1);
                      }
                    } else {
#pragma unroll
                      for (int j = 0; j < 16; ++j) scrw[lane * 33 + j] = pack_bf16x2(act_apply(v[2 * j], act), act_apply(v[2 * j + 1], act));
                    }
                    store_bf16_chunk(scrw, lane, row_base, sh.M, ep.out_bf16 + (lo ? lo_delta : 0), ep.ld_bf16, col0);
                  }
                }
              }
              continue;
            }
            if constexpr (H_RAGGED) {
              // ------------------------------ slow path: ragged / unaligned chunk (row per thread) -------------
              if (!row_ok) continue;
              if (reload) {
                const float* op = ep.out_f32 + static_cast<size_t>(row) * ep.ld_f32 + col0;
#pragma unroll
                for (int i = 0; i < 32; ++i)
                  if (i < ncols && col0 + i < sh.N) v[i] = op[i];
              } else {
                if (has_bias && first_split) {
#pragma unroll
                  for (int i = 0; i < 32; ++i)
                    if (i < ncols && col0 + i < sh.N) v[i] += __ldg(ep.bias + col0 + i);
                }
                if (has_res && first_split) {
                  const float* rp = ep.residual + static_cast<size_t>(row) * ep.ld_res + col0;
#pragma unroll
                  for (int i = 0; i < 32; ++i)
                    if (i < ncols && col0 + i < sh.N) v[i] += rp[i];
                }
                if (has_gg) {
                  const __nv_bfloat16* gp = ep.gelu_grad_of + static_cast<size_t>(row) * ep.ld_gg + col0;
#pragma unroll
                  for (int i = 0; i < 32; ++i)
                    if (i < ncols && col0 + i < sh.N) v[i] *= gelu_tanh_grad_f(__bfloat162float(gp[i]));
                }
              }
              if (pass == 0) {
                if (has_stats || do_ln) {
#pragma unroll
                  for (int i = 0; i < 32; ++i)
                    if (i < ncols && col0 + i < sh.N) { s1 += v[i]; s2 += v[i] * v[i]; }
                }
                if (has_f32) {
                  float* op = ep.out_f32 + static_cast<size_t>(row) * ep.ld_f32 + col0;
#pragma unroll
                  for (int i = 0; i < 32; ++i) {
                    if (i < ncols && col0 + i < sh.N) {
                      if (atomic_out) atomicAdd(op + i, v[i]); else op[i] = v[i];
                    }
                  }
                }
                if (has_pre) {
                  __nv_bfloat16* op = ep.out_bf16_pre + static_cast<size_t>(row) * ep.ld_bf16 + col0;
#pragma unroll
                  for (int i = 0; i < 32; ++i)
                    if (i < ncols && col0 + i < sh.N) op[i] = __float2bfloat16_rn(v[i]);
                }
              }
              if (write_bf16) {
                __nv_bfloat16* op = ep.out_bf16 + static_cast<size_t>(row) * ep.ld_bf16 + col0;
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                  if (i < ncols && col0 + i < sh.N) {
                    float w;
                    if (do_ln) w = (v[i] - mean) * (rstd * __ldg(ep.ln_gamma + col0 + i)) + __ldg(ep.ln_beta + col0 + i);
                    else w = (H_STRICT && lo_delta) ? act_apply_exact(v[i], act) : act_apply(v[i], act);
                    op[i] = __float2bfloat16_rn(w);
                    if (H_STRICT && lo_delta) op[i + lo_delta] = __float2bfloat16_rn(w - __bfloat162float(__float2bfloat16_rn(w)));
                  }
                }
              }
            }
          }  // column chunks
          if (pass == 0 && do_ln) {
            // flax LayerNorm: var = E[x^2] - E[x]^2, eps = 1e-6
            const float inv_n = 1.0f / static_cast<float>(sh.N);
            mean = s1 * inv_n;
            const float var = s2 * inv_n - mean * mean;
            rstd = rsqrtf(var + 1e-6f);
          }
        }  // passes
      }
      if constexpr (H_STATS) {
        if (has_stats && row_ok) {
          if (ep.stats_part != nullptr && !do_ln) {
            float2* slot = reinterpret_cast<float2*>(ep.stats_part) +
                           static_cast<size_t>(row) * (num_n * kGroups) + ((mn % num_n) * kGroups + eg);
            *slot = make_float2(s1, s2);
          } else {
            atomicAdd(ep.row_stats + 2 * static_cast<size_t>(row), s1);
            atomicAdd(ep.row_stats + 2 * static_cast<size_t>(row) + 1, s2);
          }
        }
      }
      if (kDedicated && item % kPer == kPer - 1) {
        mbar_arrive(acc_empty);     // the staged tile may be overwritten
        acc_phase ^= 1u;
      }
    }
  }

  // ===================== teardown =====================
  __syncwarp();  // reconverge single-lane roles before the block barrier
  __syncthreads();
}

}  // namespace smd

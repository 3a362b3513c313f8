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
//     epilogue; so do the short-K, LayerNorm-fused, generic and strict kinds.
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
  F_ATOMIC = 256u, F_ACT = 512u, F_RAGGED = 1024u, F_SCALE = 2048u, F_LNF = 4096u, F_STRICT = 8192u
};
static constexpr uint32_t kEpiGeneric = 0xFFFu;
// strict-precision mode (bf16x3): the generic epilogue plus lo-half stores and exact activations.  A separate
// instantiation on purpose: carrying that code as a runtime branch in the specialised kinds cost the FFN-up / dX GEMMs
// a factor of 2.6 (register pressure and instruction fetch in the bf16 store path).
static constexpr uint32_t kEpiStrict = kEpiGeneric | F_STRICT;
// Two-pass epilogues that finish the NEXT layer's LayerNorm -> FiLM -> swish inside this GEMM (see the F_LNF branch):
static constexpr uint32_t kEpiLnfA = F_LNF | F_BIAS | F_BF16 | F_PRE | F_STATS;            // res-block a (+ bf16 pre-LN save)
static constexpr uint32_t kEpiLnfB = F_LNF | F_BIAS | F_RES | F_F32 | F_BF16 | F_STATS;    // res-block b / post / in
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
  long long split_stride;       // k_splits > 1 without atomics: split s stores its partial at out_f32 + s * split_stride
                                // (floats); the consumer adds the slabs in a fixed order (deterministic split-K)
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
  // ---- F_LNF: out_bf16 <- act2( film( LayerNorm(v; ln_gamma, ln_beta) ) ) over the FULL row of N columns, which
  // spans several n-tiles computed by different CTAs: every tile publishes its per-row (sum, sumsq) partial to
  // lnf_part and bumps the row group's counter; the tile stays parked in shared memory until the group's counter shows all
  // partials, then the same warps normalise it (models/shared.py:61-69).  row_stats (optional) gets the totals.
  float* lnf_part;              // [M_pad][lnf_slots][2] partial sums, slot = n_tile * 2 + column group
  uint32_t* lnf_cnt;            // [M_pad / 32] arrival counters, zeroed before the launch
  const float* film;            // scale at film[r * film_ld + c], shift at film[r * film_ld + N + c]; null = no FiLM
  int film_ld;                  // row pitch of the (scale | shift) table
  int film_bcast;               // 1: every row uses table row (*film_row_dev or 0); 0: row r uses table row r / 32
  const int* film_row_dev;
  int act2;                     // activation after the affine (ACT_SWISH / ACT_NONE)
  int lnf_nowait;               // measurement only (SMD_LNF_NOWAIT=1): skip the wait for the other tiles' partials
  // ---- strict-precision mode (bf16x3): every bf16 operand written through out_bf16 also gets its lo half at
  // out_bf16 + lo_delta (elements), and the activations use exact tanhf / expf.  0 = off.
  long long lo_delta;
};

struct GemmShape {
  int M, N, K;     // logical problem; K % 64 == 0
  int BN;          // n-tile width: multiple of 16, <= kBNMax
  int a_mn, b_mn;  // 0: operand is K-major ([rows][K], K contiguous); 1: MN-major ([K][rows], rows contiguous)
  int k_splits;    // >= 1: the K loop is cut into this many independent tiles (needs atomic_out or split_stride when > 1)
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
// kPark: the LN-fused epilogue (F_LNF) parks the tile as bf16 [128][128] in shared memory between its two passes.
template <int kEW = 8, bool kPark = false, int kScrFloats = 32 * 33>
struct GemmSmem {
  static constexpr int kABytes = kBM * kBK * 2;            // 16 KB
  static constexpr int kBBytes = kBNMax * kBK * 2;         // 16 KB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBarBytes = 256;
  static constexpr int kEpiWarps = kEW;
  static constexpr bool kDedicated = kEW == 4;
  static constexpr int kEpiGroups = kDedicated ? 2 : kEW / 4;
  static constexpr int kAccBytes = kBM * kAccPitch * 4;                    // 64 KB fp32 accumulator tile
  static constexpr int kScrPerWarp = kScrFloats;                           // floats of scratch per epilogue warp
  static constexpr int kScratchBytes = kEpiWarps * kScrFloats * 4;         // per-epilogue-warp transpose scratch
  static constexpr int kParkBytes = kPark ? kBM * kBNMax * 2 : 0;          // 32 KB
  static constexpr int kMaxSmem = 232448;                                  // 227 KB
  static constexpr int kStages = (kMaxSmem - 1024 - kBarBytes - kAccBytes - kScratchBytes - kParkBytes) / kStageBytes;
  static constexpr int kTotal = kStages * kStageBytes + kBarBytes + kAccBytes + kScratchBytes + kParkBytes + 1024;
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
static constexpr bool lnf_kind(uint32_t kF) { return (kF & F_LNF) != 0 && (kF & F_RAGGED) == 0; }
// LN-fused kinds without residual / fp32 output need no 32x33 transpose tile, only the staged coefficients
static constexpr int scr_floats(uint32_t kF) {
  return (lnf_kind(kF) && (kF & (F_RES | F_F32)) == 0) ? 384 : 32 * 33;
}

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

template <uint32_t kF, int kEW = 8>
__global__ void __launch_bounds__(GemmSmem<kEW>::kThreads, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const GemmShape sh, const GemmEpilogue ep) {
  using SM = GemmSmem<kEW, lnf_kind(kF), scr_floats(kF)>;
  constexpr bool kDedicated = SM::kDedicated;
  constexpr int kGroups = SM::kEpiGroups;
  // (the LN-fused kinds also hold a 32 KB parking buffer: two stages, each TMA load still overlaps one k block of MMAs)
  static_assert(SM::kStages >= (lnf_kind(kF) ? 2 : 3), "pipeline too shallow");
  static_assert(!((kF & F_LN) && !(kF & F_RAGGED)) || kEW == 8, "the paired LayerNorm epilogue needs 8 epilogue warps");
  static_assert(!kDedicated || (kF & (F_LN | F_LNF | F_RAGGED | F_STRICT)) == 0,
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
  uint8_t* epi_smem = smem + SM::kStages * SM::kStageBytes + SM::kBarBytes + SM::kAccBytes;         // scratch | park

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
    constexpr bool H_LNF = (kF & F_LNF) != 0 && !H_RAGGED;
    constexpr bool H_STRICT = (kF & F_STRICT) != 0;
    const long long lo_delta = H_STRICT ? ep.lo_delta : 0;
    const uint32_t q = warp & 3u;                      // 32-row quadrant of the tile this warp owns
    const int asw = static_cast<int>(lane & 7u);       // swizzle of this thread's staged row (q * 32 + lane)
    const uint32_t ew = warp - (kDedicated ? 12u : 4u);   // epilogue warp index
    // column group of this warp in the shared layouts: the warps of a quadrant split the chunks
    const int eg = static_cast<int>(ew) >> 2;
    float* scr = reinterpret_cast<float*>(epi_smem) + ew * SM::kScrPerWarp;
    uint32_t* scrw = reinterpret_cast<uint32_t*>(scr);
    // fp32 transpose tile addressing for the coalesced residual loads / fp32 stores: 16-byte chunk j of row r at chunk
    // slot r * 8 + (j ^ (r & 7)) -- 128-bit shared accesses, conflict-free for "lane = row" and "8 lanes = one row"
    auto t4 = [&](int r_, int j_) { return reinterpret_cast<float4*>(scr) + (r_ * 8 + (j_ ^ (r_ & 7))); };
    auto add_pair = [](float& a, float& b, float x, float y) {   // (a, b) += (x, y)
      f32x2_unpack(f32x2_add(f32x2_pack(a, b), f32x2_pack(x, y)), a, b);
    };
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
    if constexpr (H_LNF) {
      // ---------- epilogue that also finishes the NEXT LayerNorm -> FiLM -> activation over the FULL row ----------
      // The row (N = num_n * BN columns) spans num_n tiles computed by other CTAs in the same scheduling round (tiles
      // are m-major), so the row statistics are exchanged through global memory.
      //   pass 1: v = acc + bias (+ residual) -> fp32 out_f32 / bf16 out_bf16_pre stores as usual, per-row (sum, sumsq)
      //     of this warp's columns, and v parked as bf16 in shared memory (XOR-swizzled 16-byte chunks);
      //   exchange: the warp publishes its partial into its own slot, bumps the row group's counter and, while the
      //     other n-tiles arrive, stages the per-column affine (gamma * scale, beta * scale + shift) of its columns;
      //   pass 2: the slots are summed in a FIXED order (bit-reproducible, unlike atomics) and the parked tile becomes
      //     out_bf16 = act2(film(LN(v))) -- what the stand-alone ln_film_act kernel did with an HBM round trip and a
      //     launch of its own.  (Like that path's bf16 r1, the LayerNorm input is the bf16-rounded v; the statistics
      //     are those of the fp32 v.)
      // Deadlock freedom: tiles are visited in increasing index by co-resident persistent CTAs; a wait only targets
      // pass 1 of tiles of the same round, which never waits on anything (launch one such kernel at a time).
      constexpr int G = kEW / 4;          // epilogue warps per 32-row quadrant: they split the tile's 32-column chunks
      const int nslots = num_n * G;
      const float inv_n = 1.0f / static_cast<float>(sh.N);
      const int act2 = ep.act2;
      uint8_t* park = epi_smem + SM::kScratchBytes;   // [128 rows][256 B]
      // this warp's 32 rows; 16-byte chunk c of row r sits at chunk (c ^ (r & 7))
      auto park_ptr = [&](int rr, int chunk) {
        const int r = static_cast<int>(q) * 32 + rr;
        return park + r * 256 + ((chunk ^ (r & 7)) << 4);
      };
      float* coefA = scr;            // [128] gamma * scale of this warp's columns (chunk-major: 4 x 32)
      float* coefB = scr + 128;      // [128] beta * scale + shift
      float* rowst = scr + 256;      // [32][2] mean, rstd
      for (int tile = group; tile < num_tiles; tile += num_groups) {
        const int n_idx = tile % num_n;
        const int row_base = (tile / num_n) * rows_per_tile + static_cast<int>(q * 32u);
        const int row = row_base + static_cast<int>(lane);
        const int n0 = n_idx * BN;
        mma_tile(tile);
        float* const arow = acc_tile + (q * 32u + lane) * kAccPitch;
        float s1 = 0.f, s2 = 0.f;
        uint64_t s1p = f32x2_pack(0.f, 0.f), s2p = f32x2_pack(0.f, 0.f);
        auto tsw = [&](int r_, int j_) { return reinterpret_cast<float4*>(scr) + (r_ * 8 + (j_ ^ (r_ & 7))); };
        float4 rpre[H_RES ? 8 : 1];
        auto prefetch = [&](int c) {
          if constexpr (H_RES) {
#pragma unroll
            for (int it = 0; it < 8; ++it) {
              const int grow = row_base + it * 4 + f_r;
              rpre[it] = (has_res && grow < sh.M)
                             ? *reinterpret_cast<const float4*>(ep.residual + static_cast<size_t>(grow) * ep.ld_res + n0 + c + f_c)
                             : make_float4(0.f, 0.f, 0.f, 0.f);
            }
          }
        };
        prefetch(eg * 32);
        // ---------------- pass 1 ----------------
        for (int c0 = eg * 32; c0 < BN; c0 += 32 * G) {
          __syncwarp();
          uint32_t r[32];
          acc_ld32(arow, c0, asw, r);
          const int col0 = n0 + c0;
          float4 bq[8];
          if (has_bias) {
            const float4* b4 = reinterpret_cast<const float4*>(ep.bias + col0);
#pragma unroll
            for (int i = 0; i < 8; ++i) bq[i] = __ldg(b4 + i);
          }
          // fp32 pairs (two scalar round-to-nearest operations each)
          uint64_t v2[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) v2[i] = f32x2_pack(__uint_as_float(r[2 * i]), __uint_as_float(r[2 * i + 1]));
          if (has_bias) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              v2[2 * i] = f32x2_add(v2[2 * i], f32x2_pack(bq[i].x, bq[i].y));
              v2[2 * i + 1] = f32x2_add(v2[2 * i + 1], f32x2_pack(bq[i].z, bq[i].w));
            }
          }
          if constexpr (H_RES) {
            if (has_res) {
              // residual block -> 32 x 32 transpose tile (16-byte chunk j of row r at slot j ^ (r & 7)): 128-bit accesses
#pragma unroll
              for (int it = 0; it < 8; ++it) *tsw(it * 4 + f_r, f_c >> 2) = rpre[it];
              if (c0 + 32 * G < BN) prefetch(c0 + 32 * G);
              __syncwarp();
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float4 t = *tsw(static_cast<int>(lane), i);
                v2[2 * i] = f32x2_add(v2[2 * i], f32x2_pack(t.x, t.y));
                v2[2 * i + 1] = f32x2_add(v2[2 * i + 1], f32x2_pack(t.z, t.w));
              }
              __syncwarp();
            }
          }
#pragma unroll
          for (int i = 0; i < 16; ++i) { s1p = f32x2_add(s1p, v2[i]); s2p = f32x2_fma(v2[i], v2[i], s2p); }
          // park the row's 32 columns as bf16: four 16-byte chunks
          {
            uint32_t pk[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              float a, b;
              f32x2_unpack(v2[j], a, b);
              pk[j] = pack_bf16x2(a, b);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j)
              *reinterpret_cast<uint4*>(park_ptr(static_cast<int>(lane), (c0 >> 3) + j)) =
                  make_uint4(pk[4 * j], pk[4 * j + 1], pk[4 * j + 2], pk[4 * j + 3]);
          }
          if constexpr (H_F32) {
            if (has_f32) {
              // v goes back to the staged accumulator row: the fp32 store sweep runs AFTER the partials are published, so the fence of the
              // exchange does not have to drain 16 KB of tile stores per warp
#pragma unroll
              for (int i = 0; i < 16; ++i) {
                float a, b;
                f32x2_unpack(v2[i], a, b);
                r[2 * i] = __float_as_uint(a); r[2 * i + 1] = __float_as_uint(b);
              }
              acc_st32(arow, c0, asw, r);
            }
          }
        }
        {
          float a, b;
          f32x2_unpack(s1p, a, b); s1 = a + b;
          f32x2_unpack(s2p, a, b); s2 = a + b;
        }
        // ---------------- exchange ----------------
        uint32_t* cnt = ep.lnf_cnt + (row_base >> 5);
        {
          float2* slot = reinterpret_cast<float2*>(ep.lnf_part) + static_cast<size_t>(row) * nslots + (n_idx * G + eg);
          __stcg(slot, make_float2(s1, s2));
          __threadfence();
          __syncwarp();
          if (lane == 0) red_release_gpu_add(cnt, 1u);
        }
        if constexpr (H_F32) {
          if (has_f32) {
            for (int c0 = eg * 32; c0 < BN; c0 += 32 * G) {
              __syncwarp();
              uint32_t r[32];
              acc_ld32(arow, c0, asw, r);
#pragma unroll
              for (int i = 0; i < 8; ++i)
                *tsw(static_cast<int>(lane), i) = make_float4(__uint_as_float(r[4 * i]), __uint_as_float(r[4 * i + 1]),
                                                              __uint_as_float(r[4 * i + 2]), __uint_as_float(r[4 * i + 3]));
              __syncwarp();
#pragma unroll
              for (int it = 0; it < 8; ++it) {
                const int rr = it * 4 + f_r, grow = row_base + rr;
                if (grow < sh.M)
                  *reinterpret_cast<float4*>(ep.out_f32 + static_cast<size_t>(grow) * ep.ld_f32 + n0 + c0 + f_c) = *tsw(rr, f_c >> 2);
              }
            }
            __syncwarp();
          }
        }
        if constexpr (H_PRE) {
          if (has_pre) {
            // the pre-LayerNorm copy the backward pass wants (bf16 [M][N]) comes straight from the parked tile
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int c0 = (eg + G * j) * 32;
              const int chunk = (c0 >> 3) + static_cast<int>(lane & 3u);
#pragma unroll
              for (int it = 0; it < 4; ++it) {
                const int rr = it * 8 + h_r, grow = row_base + rr;
                if (c0 < BN && grow < sh.M)
                  *reinterpret_cast<uint4*>(ep.out_bf16_pre + static_cast<size_t>(grow) * ep.ld_bf16 + n0 + c0 + h_c) =
                      *reinterpret_cast<const uint4*>(park_ptr(rr, chunk));
              }
            }
          }
        }
        {
          // per-column affine of this warp's columns while the other n-tiles arrive: lane l owns 4 columns per chunk
          const float* film_row = nullptr;       // FiLM row of this warp's 32 rows (one sample when seq_len == 32)
          if (ep.film) {
            const int fr = ep.film_bcast ? (ep.film_row_dev ? *ep.film_row_dev : 0) : (row_base >> 5);
            film_row = ep.film + static_cast<size_t>(fr) * ep.film_ld;
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int c0 = (eg + G * j) * 32;
            if (c0 < BN) {
              const int col = n0 + c0 + 4 * static_cast<int>(lane & 7u);
              if (lane < 8) {
                float4 g = __ldg(reinterpret_cast<const float4*>(ep.ln_gamma + col));
                float4 b = __ldg(reinterpret_cast<const float4*>(ep.ln_beta + col));
                if (film_row) {
                  const float4 sc = __ldg(reinterpret_cast<const float4*>(film_row + col));
                  const float4 hf = __ldg(reinterpret_cast<const float4*>(film_row + sh.N + col));
                  b = make_float4(fmaf(b.x, sc.x, hf.x), fmaf(b.y, sc.y, hf.y), fmaf(b.z, sc.z, hf.z), fmaf(b.w, sc.w, hf.w));
                  g = make_float4(g.x * sc.x, g.y * sc.y, g.z * sc.z, g.w * sc.w);
                }
                *reinterpret_cast<float4*>(coefA + 32 * j + 4 * lane) = g;
                *reinterpret_cast<float4*>(coefB + 32 * j + 4 * lane) = b;
              }
            }
          }
        }
        if (lane == 0 && !ep.lnf_nowait) {
          uint32_t spins = 0;
          const unsigned long long t0 = global_timer_ns();
          while (ld_acquire_gpu(cnt) < static_cast<uint32_t>(nslots)) {
            if ((++spins & 0x3FFu) == 0 && global_timer_ns() - t0 > SMD_WAIT_LIMIT_NS) __trap();
          }
        }
        __syncwarp();
        {
          float t1 = 0.f, t2 = 0.f;
          const float2* pp = reinterpret_cast<const float2*>(ep.lnf_part) + static_cast<size_t>(row) * nslots;
          for (int s = 0; s < nslots; ++s) {         // fixed order: the statistics are bit-reproducible
            const float2 p = __ldcg(pp + s);
            t1 += p.x; t2 += p.y;
          }
          const float mean_l = t1 * inv_n;
          const float rstd_l = rsqrtf(t2 * inv_n - mean_l * mean_l + 1e-6f);   // flax LayerNorm: E[x^2] - E[x]^2, eps 1e-6
          if (has_stats && row < sh.M && n_idx == 0 && eg == 0)
            *reinterpret_cast<float2*>(ep.row_stats + 2 * static_cast<size_t>(row)) = make_float2(t1, t2);
          rowst[2 * lane] = mean_l; rowst[2 * lane + 1] = rstd_l;
        }
        __syncwarp();
        // ---------------- pass 2 ----------------
        auto pass2 = [&](auto swish_tag) {
        constexpr bool kSwish = decltype(swish_tag)::value;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c0 = (eg + G * j) * 32;
          if (c0 < BN) {
            const int col0 = n0 + c0;
            float A[8], Bc[8];
            {
              const float4 a0 = *reinterpret_cast<const float4*>(coefA + 32 * j + h_c), a1 = *reinterpret_cast<const float4*>(coefA + 32 * j + h_c + 4);
              const float4 b0 = *reinterpret_cast<const float4*>(coefB + 32 * j + h_c), b1 = *reinterpret_cast<const float4*>(coefB + 32 * j + h_c + 4);
              A[0] = a0.x; A[1] = a0.y; A[2] = a0.z; A[3] = a0.w; A[4] = a1.x; A[5] = a1.y; A[6] = a1.z; A[7] = a1.w;
              Bc[0] = b0.x; Bc[1] = b0.y; Bc[2] = b0.z; Bc[3] = b0.w; Bc[4] = b1.x; Bc[5] = b1.y; Bc[6] = b1.z; Bc[7] = b1.w;
            }
            const int chunk = (c0 >> 3) + static_cast<int>(lane & 3u);
#pragma unroll
            for (int it = 0; it < 4; ++it) {
              const int rr = it * 8 + h_r, grow = row_base + rr;
              const uint4 raw = *reinterpret_cast<const uint4*>(park_ptr(rr, chunk));
              const __nv_bfloat162* hp = reinterpret_cast<const __nv_bfloat162*>(&raw);
              const float mean = rowst[2 * rr], rstd = rowst[2 * rr + 1];
              const float nmr = -mean * rstd;
              const uint64_t rs2 = f32x2_pack(rstd, rstd), nm2 = f32x2_pack(nmr, nmr);
              uint32_t pk[4];
#pragma unroll
              for (int k2 = 0; k2 < 4; ++k2) {
                const float2 f = __bfloat1622float2(hp[k2]);
                // xhat = x rstd - mean rstd ; y = xhat (gamma scale) + (beta scale + shift) ; swish(y) = h + h tanh(h), h = y / 2
                uint64_t y = f32x2_fma(f32x2_fma(f32x2_pack(f.x, f.y), rs2, nm2), f32x2_pack(A[2 * k2], A[2 * k2 + 1]),
                                       f32x2_pack(Bc[2 * k2], Bc[2 * k2 + 1]));
                if constexpr (kSwish) {
                  const uint64_t h = f32x2_mul(y, f32x2_pack(0.5f, 0.5f));
                  float h0, h1;
                  f32x2_unpack(h, h0, h1);
                  y = f32x2_fma(h, f32x2_pack(tanh_fast(h0), tanh_fast(h1)), h);
                }
                float y0, y1;
                f32x2_unpack(y, y0, y1);
                pk[k2] = pack_bf16x2(y0, y1);
              }
              if (grow < sh.M)
                *reinterpret_cast<uint4*>(ep.out_bf16 + static_cast<size_t>(grow) * ep.ld_bf16 + col0 + h_c) =
                    make_uint4(pk[0], pk[1], pk[2], pk[3]);
            }
          }
        }
        };
        if (act2 == ACT_SWISH) pass2(std::true_type{}); else pass2(std::false_type{});
        __syncwarp();
      }
    } else if constexpr (H_LN && !H_RAGGED) {
      // ---------- single-pass full-row LayerNorm epilogue (N == BN <= 128: attention out-proj, FFN down) ----------
      // The two warps of a row quadrant split the row's chunks, keep their values in registers, exchange the
      // per-row (sum, sumsq) partials through shared memory (named barrier of 64 threads) and each normalises
      // and stores its own chunks: no second pass over the staged tile, no global re-read.
      float* scr_partner = reinterpret_cast<float*>(epi_smem) +
                           ((warp - 4u) ^ 4u) * (32 * 33);
      const int nchunk = BN / 64;
      const float inv_n = 1.0f / static_cast<float>(sh.N);
      for (int tile = group; tile < num_tiles; tile += num_groups) {
        const int row_base = (tile / num_n) * rows_per_tile + static_cast<int>(q * 32u);
        mma_tile(tile);
        float* const arow = acc_tile + (q * 32u + lane) * kAccPitch;
        float vv[2][32];
        float s1 = 0.f, s2 = 0.f;
        float4 rpre[8];
        auto prefetch = [&](int c) {
#pragma unroll
          for (int it = 0; it < 8; ++it) {
            const int grow = row_base + it * 4 + f_r;
            rpre[it] = (has_res && grow < sh.M)
                           ? *reinterpret_cast<const float4*>(ep.residual + static_cast<size_t>(grow) * ep.ld_res + c + f_c)
                           : make_float4(0.f, 0.f, 0.f, 0.f);
          }
        };
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
              const float4* b4 = reinterpret_cast<const float4*>(ep.bias + c0);
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float4 b = __ldg(b4 + i);
                add_pair(vv[j][4 * i], vv[j][4 * i + 1], b.x, b.y);
                add_pair(vv[j][4 * i + 2], vv[j][4 * i + 3], b.z, b.w);
              }
            }
            if (has_res) {
#pragma unroll
              for (int it = 0; it < 8; ++it) *t4(it * 4 + f_r, f_c >> 2) = rpre[it];
              if (j + 1 < nchunk) prefetch(eg * 32 + 64 * (j + 1));
              __syncwarp();
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float4 t = *t4(static_cast<int>(lane), i);
                add_pair(vv[j][4 * i], vv[j][4 * i + 1], t.x, t.y);
                add_pair(vv[j][4 * i + 2], vv[j][4 * i + 3], t.z, t.w);
              }
              __syncwarp();
            }
            {
              uint64_t a1 = f32x2_pack(0.f, 0.f), a2 = f32x2_pack(0.f, 0.f);
#pragma unroll
              for (int i = 0; i < 16; ++i) {
                const uint64_t pv = f32x2_pack(vv[j][2 * i], vv[j][2 * i + 1]);
                a1 = f32x2_add(a1, pv);
                a2 = f32x2_fma(pv, pv, a2);
              }
              float lo, hi;
              f32x2_unpack(a1, lo, hi); s1 += lo + hi;
              f32x2_unpack(a2, lo, hi); s2 += lo + hi;
            }
            if (has_f32) {
#pragma unroll
              for (int i = 0; i < 8; ++i)
                *t4(static_cast<int>(lane), i) = make_float4(vv[j][4 * i], vv[j][4 * i + 1], vv[j][4 * i + 2], vv[j][4 * i + 3]);
              __syncwarp();
#pragma unroll
              for (int it = 0; it < 8; ++it) {
                const int rr = it * 4 + f_r, grow = row_base + rr;
                if (grow < sh.M)
                  *reinterpret_cast<float4*>(ep.out_f32 + static_cast<size_t>(grow) * ep.ld_f32 + c0 + f_c) = *t4(rr, f_c >> 2);
              }
              __syncwarp();
            }
          }
        }
        // exchange the row partials with the partner warp of this quadrant
        scr[lane * 33] = s1; scr[lane * 33 + 1] = s2;
        asm volatile("bar.sync %0, 64;" ::"r"(1u + q) : "memory");
        const float t1 = s1 + scr_partner[lane * 33], t2 = s2 + scr_partner[lane * 33 + 1];
        asm volatile("bar.sync %0, 64;" ::"r"(1u + q) : "memory");
        const float mean = t1 * inv_n;
        const float rstd = rsqrtf(t2 * inv_n - mean * mean + 1e-6f);   // flax LayerNorm: E[x^2] - E[x]^2, eps 1e-6
        if (has_bf16) {
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            if (j < nchunk) {
              const int c0 = eg * 32 + 64 * j;
              const float4* g4 = reinterpret_cast<const float4*>(ep.ln_gamma + c0);
              const float4* b4 = reinterpret_cast<const float4*>(ep.ln_beta + c0);
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float4 g = __ldg(g4 + i), b = __ldg(b4 + i);
                const float w0 = (vv[j][4 * i] - mean) * (rstd * g.x) + b.x;
                const float w1 = (vv[j][4 * i + 1] - mean) * (rstd * g.y) + b.y;
                const float w2 = (vv[j][4 * i + 2] - mean) * (rstd * g.z) + b.z;
                const float w3 = (vv[j][4 * i + 3] - mean) * (rstd * g.w) + b.w;
                scrw[lane * 33 + 2 * i] = pack_bf16x2(w0, w1);
                scrw[lane * 33 + 2 * i + 1] = pack_bf16x2(w2, w3);
              }
              __syncwarp();
#pragma unroll
              for (int it = 0; it < 4; ++it) {
                const int rr = it * 8 + h_r, grow = row_base + rr;
                if (grow < sh.M) {
                  const uint32_t* sp = scrw + rr * 33 + (h_c >> 1);
                  *reinterpret_cast<uint4*>(ep.out_bf16 + static_cast<size_t>(grow) * ep.ld_bf16 + c0 + h_c) =
                      make_uint4(sp[0], sp[1], sp[2], sp[3]);
                }
              }
              __syncwarp();
            }
          }
        }
      }
    } else {
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
      float* const out_f32_s = ep.out_f32 ? ep.out_f32 + static_cast<long long>(tile % splits) * ep.split_stride : nullptr;
      const int row_base = (mn / num_n) * rows_per_tile + static_cast<int>(q * 32u);
      const int row = row_base + static_cast<int>(lane);
      const int n0 = (mn % num_n) * BN;
      const bool row_ok = row < sh.M;
      float* const arow = acc_tile + (q * 32u + lane) * kAccPitch;
      float s1 = 0.f, s2 = 0.f;
      float mean = 0.f, rstd = 0.f;
      const int npass = do_ln ? 2 : 1;
      // full-row LayerNorm needs one warp to see the whole row: group 1 sits those tiles out
      const int c_begin = do_ln ? (eg == 0 ? 0 : BN) : eg * 32;
      const int c_step = do_ln ? 32 : 32 * kGroups;
      // software prefetch of the residual / gelu-grad tiles of the NEXT chunk (their global latency would
      // otherwise be fully exposed: only two warps per SM sub-partition work on the epilogue)
      float4 rpre[H_RES ? 8 : 1];
      uint4 gpre[H_GG ? 4 : 1];
      const bool pre_res = has_res && first_split && aligned_ok;
      const bool pre_gg = has_gg && aligned_ok;
      auto chunk_fast = [&](int c) {
        return !H_RAGGED || ((BN - c) >= 32 && aligned_ok && (n0 + c + 32 <= sh.N));
      };
      auto prefetch = [&](int c) {
        const int colp = n0 + c;
        if constexpr (H_RES) {
          if (pre_res) {
#pragma unroll
            for (int it = 0; it < 8; ++it) {
              const int grow = row_base + it * 4 + f_r;
              rpre[it] = (grow < sh.M) ? *reinterpret_cast<const float4*>(ep.residual + static_cast<size_t>(grow) * ep.ld_res + colp + f_c)
                                       : make_float4(0.f, 0.f, 0.f, 0.f);
            }
          }
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
                if (grow < sh.M) t = *reinterpret_cast<const float4*>(out_f32_s + static_cast<size_t>(grow) * ep.ld_f32 + col0 + f_c);
                float* d = scr + rr * 33 + f_c;
                d[0] = t.x; d[1] = t.y; d[2] = t.z; d[3] = t.w;
              }
              __syncwarp();
#pragma unroll
              for (int i = 0; i < 32; ++i) v[i] = scr[lane * 33 + i];
              __syncwarp();
            } else {
              if constexpr (H_BIAS) {
                if (has_bias && first_split) {
#pragma unroll
                  for (int i = 0; i < 8; ++i) {
                    const float4 b = bq[i];
                    add_pair(v[4 * i], v[4 * i + 1], b.x, b.y);
                    add_pair(v[4 * i + 2], v[4 * i + 3], b.z, b.w);
                  }
                }
              }
              uint4 gcur[H_GG ? 4 : 1];
              if constexpr (H_RES) {
                if (pre_res) {
#pragma unroll
                  for (int it = 0; it < 8; ++it) *t4(it * 4 + f_r, f_c >> 2) = rpre[it];
                }
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
                if (pre_res) {
                  __syncwarp();
#pragma unroll
                  for (int i = 0; i < 8; ++i) {
                    const float4 t = *t4(static_cast<int>(lane), i);
                    add_pair(v[4 * i], v[4 * i + 1], t.x, t.y);
                    add_pair(v[4 * i + 2], v[4 * i + 3], t.z, t.w);
                  }
                  __syncwarp();
                }
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
                if (has_stats || do_ln) {
                  uint64_t a1 = f32x2_pack(0.f, 0.f), a2 = f32x2_pack(0.f, 0.f);   // paired partial sums
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
              }
              if constexpr (H_F32) {
                if (has_f32) {
#pragma unroll
                  for (int i = 0; i < 8; ++i)
                    *t4(static_cast<int>(lane), i) = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
                  __syncwarp();
#pragma unroll
                  for (int it = 0; it < 8; ++it) {
                    const int rr = it * 4 + f_r, grow = row_base + rr;
                    if (grow < sh.M) {
                      const float4 sp = *t4(rr, f_c >> 2);
                      float* op = out_f32_s + static_cast<size_t>(grow) * ep.ld_f32 + col0 + f_c;
                      if (H_ATOMIC && atomic_out) {
                        atomicAdd(op, sp.x); atomicAdd(op + 1, sp.y); atomicAdd(op + 2, sp.z); atomicAdd(op + 3, sp.w);
                      } else {
                        *reinterpret_cast<float4*>(op) = sp;
                      }
                    }
                  }
                  __syncwarp();
                }
              }
              if constexpr (H_PRE) {
                if (has_pre) {
#pragma unroll
                  for (int j = 0; j < 16; ++j) {
                    __nv_bfloat162 pk = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
                    scrw[lane * 33 + j] = *reinterpret_cast<uint32_t*>(&pk);
                  }
                  __syncwarp();
#pragma unroll
                  for (int it = 0; it < 4; ++it) {
                    const int rr = it * 8 + h_r, grow = row_base + rr;
                    if (grow < sh.M) {
                      const uint32_t* sp = scrw + rr * 33 + (h_c >> 1);
                      *reinterpret_cast<uint4*>(ep.out_bf16_pre + static_cast<size_t>(grow) * ep.ld_bf16 + col0 + h_c) =
                          make_uint4(sp[0], sp[1], sp[2], sp[3]);
                    }
                  }
                  __syncwarp();
                }
              }
            }
            if constexpr (H_BF16) {
              if (write_bf16) {
                for (int half = 0; half < ((H_STRICT && lo_delta) ? 2 : 1); ++half) {   // strict mode: second sweep = lo halves
                if (H_LN && do_ln) {
                  const float4* g4 = reinterpret_cast<const float4*>(ep.ln_gamma + col0);
                  const float4* b4 = reinterpret_cast<const float4*>(ep.ln_beta + col0);
#pragma unroll
                  for (int i = 0; i < 8; ++i) {
                    const float4 g = __ldg(g4 + i), b = __ldg(b4 + i);
                    const float w0 = (v[4 * i] - mean) * (rstd * g.x) + b.x;
                    const float w1 = (v[4 * i + 1] - mean) * (rstd * g.y) + b.y;
                    const float w2 = (v[4 * i + 2] - mean) * (rstd * g.z) + b.z;
                    const float w3 = (v[4 * i + 3] - mean) * (rstd * g.w) + b.w;
                    scrw[lane * 33 + 2 * i] = half ? pack_bf16x2_lo(w0, w1) : pack_bf16x2(w0, w1);
                    scrw[lane * 33 + 2 * i + 1] = half ? pack_bf16x2_lo(w2, w3) : pack_bf16x2(w2, w3);
                  }
                } else if (H_STRICT && lo_delta) {
#pragma unroll
                  for (int j = 0; j < 16; ++j) {
                    const float y0 = act_apply_exact(v[2 * j], act), y1 = act_apply_exact(v[2 * j + 1], act);
                    scrw[lane * 33 + j] = half ? pack_bf16x2_lo(y0, y1) : pack_bf16x2(y0, y1);
                  }
                } else {
#pragma unroll
                  for (int j = 0; j < 16; ++j) {
                    __nv_bfloat162 pk = __floats2bfloat162_rn(act_apply(v[2 * j], act), act_apply(v[2 * j + 1], act));
                    scrw[lane * 33 + j] = *reinterpret_cast<uint32_t*>(&pk);
                  }
                }
                __syncwarp();
#pragma unroll
                for (int it = 0; it < 4; ++it) {
                  const int rr = it * 8 + h_r, grow = row_base + rr;
                  if (grow < sh.M) {
                    const uint32_t* sp = scrw + rr * 33 + (h_c >> 1);
                    *reinterpret_cast<uint4*>(ep.out_bf16 + (half ? lo_delta : 0) + static_cast<size_t>(grow) * ep.ld_bf16 + col0 + h_c) =
                        make_uint4(sp[0], sp[1], sp[2], sp[3]);
                  }
                }
                __syncwarp();
                }
              }
            }
            continue;
          }

          if constexpr (H_RAGGED) {
            // ------------------------------ slow path: ragged / unaligned chunk (row per thread) -------------
            if (!row_ok) continue;
            if (reload) {
              const float* op = out_f32_s + static_cast<size_t>(row) * ep.ld_f32 + col0;
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
                float* op = out_f32_s + static_cast<size_t>(row) * ep.ld_f32 + col0;
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
  }

  // ===================== teardown =====================
  __syncwarp();  // reconverge single-lane roles before the block barrier
  __syncthreads();
}

}  // namespace smd

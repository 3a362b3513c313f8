// Row-resident, store-streaming wgmma GEMM for short K and wide N: the trunk's FFN up (+GELU, bf16 out and its bf16
// pre-activation), the FFN-up adjoint (x gelu'(pre-activation), bf16 out) and the post dense (fp32 out + row
// statistics), all with K = 128 and N = 2048.
//
// At K <= 128 the K loop is two k blocks; such a launch is an output stream (64 KB of bf16 / fp32 per 128 x 128 tile
// against 32 KB of operands).  Here a CTA owns one 128-row block and a run of n-tiles: it loads its A rows once with
// TMA and keeps them, the 128 x K weight tiles stream from L2 through a two-stage ring, and each tile's outputs leave
// through 1-D bulk stores (cp.async.bulk, one per output row) from shared-memory staging, so no warp waits on its
// global stores.
//
// 384 threads: warp 0 is the producer, warpgroups 1 and 2 own 64 rows of every tile each.  A consumer warpgroup keeps
// two accumulator sets: it issues tile j + 1's wgmma before it runs tile j's epilogue from the accumulator fragments.
// The epilogue goes out in 64-column half-tiles through a ring of three staging slots per warpgroup, each holding the
// half-tile of every output: while a warpgroup stages half-tile q, the bulk stores of q - 1 and q - 2 are still in
// flight, and only those of q - 3 (the slot's previous contents) must have read their source.  A single full-tile
// buffer would make each tile's staging wait for the previous tile's stores, and two of them do not fit next to the
// resident A rows and the weight ring.
//
// Every output is bit-identical to the 128 x 128 layouts': the same m64n128k16 sequence over K (same k-step order),
// then the same per-element epilogue arithmetic (bias add, act_apply's operations, gelu_tanh_grad_f, bf16 rounding).
// The row statistics go to the per-tile slots that stats_slots_for reports, three column groups per n-tile (group g
// sums the 32-column chunks g and g + 3 with chunk_stats, in that order, read back from the tile's two staged halves),
// so the totals ln_film_act forms are unchanged too.
#pragma once
#include "gemm_wgmma.cuh"

namespace smd {

// act_apply with the activation selected instead of branched on: the same operations, so the same bits.  ep.act is
// uniform, but a branch around every element's tanh keeps ptxas from overlapping one element's MUFU latency with the
// next element's arithmetic, which made the FFN-up staging latency-bound.
__device__ __forceinline__ float act_apply_select(float v, int act) {
  const float c = 0.7978845608028654f;
  const float h = 0.5f * v;
  const float u = act == ACT_GELU_TANH ? v * fmaf(v * v, 0.044715f * c, c) : h;
  const float y = fmaf(h, tanh_fast(u), h);
  return act == ACT_GELU_TANH || act == ACT_SWISH ? y : v;
}

template <uint32_t kF>
struct GemmSmemExpand {
  static constexpr bool kGG = kF == kEpiGG;
  static constexpr int kKMax = 128;                           // the whole K in one resident block
  static constexpr int kABytes = kBM * kKMax * 2;             // 32 KB: the CTA's A rows, two 64-wide k blocks
  static constexpr int kBBytes = kBNMax * kKMax * 2;          // 32 KB: one weight tile
  static constexpr int kStages = 2;
  static constexpr int kHPitch = kBNMax * 2 + 16;             // bytes per gelu_grad_of row (padded: conflict-free)
  static constexpr int kHBytes = kGG ? kBM * kHPitch : 0;     // the tile of gelu_grad_of, per stage
  // Staging ring, per consumer warpgroup: kSlots slots of one 64-row x 64-column half-tile of every output (fp32 out,
  // or bf16 out + the bf16 pre-activation for kEpiAct, or bf16 out), rows padded by 16 bytes (conflict-free), then
  // the half-tile's 64 bias values (kEpiAct, kEpiF32).
  static constexpr int kHalf = kBNMax / 2;
  static constexpr int kOuts = kF == kEpiAct ? 2 : 1;
  static constexpr int kSPitch = kHalf * (kF == kEpiF32 ? 4 : 2) + 16;
  static constexpr int kBiasOff = kOuts * 64 * kSPitch;
  static constexpr int kSlotBytes = kBiasOff + (kGG ? 0 : kHalf * 4);   // 18 688 (kEpiAct), 17 664 (kEpiF32), 9 216
  static constexpr int kSlots = 3;
  static constexpr int kBarBytes = 128;
  // 211 584 (kEpiAct), 205 440 (kEpiF32), 224 384 (kEpiGG) bytes
  static constexpr int kTotal = 1024 + kABytes + kStages * (kBBytes + kHBytes) + 2 * kSlots * kSlotBytes + kBarBytes;
  static constexpr int kThreads = 384;
  static constexpr int kEpiGroups = 3;                        // statistics slots per (row, n-tile)
  static constexpr int kProdRegs = 40, kMmaRegs = 232;
  static_assert(kProdRegs + 2 * kMmaRegs <= 3 * 170, "register budgets exceed the CTA's file");
  static_assert(kTotal <= GemmSmem<8>::kMaxSmem, "shared memory");
  static_assert(kSPitch % 16 == 0 && kSlotBytes % 16 == 0, "bulk-store sources must be 16-byte aligned");
  static_assert((1 + 2 * kStages + (kGG ? 2 * kStages : 0)) * 8 <= kBarBytes, "mbarriers do not fit their region");
};

// tmA: K-major A [M][128], 128-row boxes; tmB: the op's B map (kTB: 1 = MN-major [128][N]).  CTA c owns row block
// c / groups and the n-tiles [(c % groups) * tpc, + tpc), tpc = N / 128 / groups, an even number: the tile loop runs
// in pairs so that each accumulator set has a fixed role (a loop that may end after either set makes ptxas serialise
// the wgmma).
template <uint32_t kF, int kTB>
__global__ void __launch_bounds__(GemmSmemExpand<kF>::kThreads, 1)
gemm_bf16_wgmma_expand_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                              const GemmShape sh, const int tpc, const __grid_constant__ GemmEpilogue ep) {
  using SM = GemmSmemExpand<kF>;
  static_assert(kF == kEpiAct || kF == kEpiGG || kF == kEpiF32, "the expand layout runs kEpiAct / kEpiGG / kEpiF32");
  constexpr bool kGG = SM::kGG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = sA + SM::kABytes;                                   // [kStages][kBBytes]
  uint8_t* sH = sB + SM::kStages * SM::kBBytes;                     // [kStages][kHBytes]
  uint8_t* sOut = sH + SM::kStages * SM::kHBytes;                   // [2 warpgroups][kSlots][kSlotBytes]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sOut + 2 * SM::kSlots * SM::kSlotBytes);
  uint64_t* a_full = bars;
  uint64_t* b_full = bars + 1;                                      // [kStages]
  uint64_t* b_empty = b_full + SM::kStages;                         // [kStages]
  uint64_t* h_full = b_empty + SM::kStages;                         // [kStages] (kGG)
  uint64_t* h_empty = h_full + SM::kStages;                         // [kStages] (kGG)

  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t lane = threadIdx.x & 31;
  const int groups = (sh.N / kBNMax) / tpc;
  const int m0 = static_cast<int>(blockIdx.x) / groups * kBM;
  const int nt0 = static_cast<int>(blockIdx.x) % groups * tpc;      // first n-tile of this CTA
  constexpr int nkb = SM::kKMax / kBK;

  pdl_trigger();
  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  if (warp == 1 && elect_one()) {
    mbar_init(a_full, 1);
    for (int i = 0; i < SM::kStages; ++i) {
      mbar_init(&b_full[i], 1);
      mbar_init(&b_empty[i], 8);   // one arrival per MMA warp
      if (kGG) {
        mbar_init(&h_full[i], 1);
        mbar_init(&h_empty[i], 8);
      }
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp < 4) {
    // ===================== producer (warp 0) =====================
    setmaxnreg_dec<SM::kProdRegs>();
    if (warp != 0) return;
    if (elect_one()) {
      mbar_arrive_expect_tx(a_full, static_cast<uint32_t>(nkb * kBM * kBK * 2));
      for (int kb = 0; kb < nkb; ++kb) tma_load_2d(&tmA, a_full, sA + kb * (kBM * kBK * 2), kb * kBK, m0);
    }
    __syncwarp();
    const int rows = min(kBM, sh.M - m0);
    for (int i = 0; i < tpc; ++i) {
      const int s = i % SM::kStages;
      const uint32_t ph = static_cast<uint32_t>(i / SM::kStages) & 1u;
      const int n0 = (nt0 + i) * kBNMax;
      if (elect_one()) {
        mbar_wait(&b_empty[s], ph ^ 1u);
        uint8_t* b = sB + s * SM::kBBytes;
        mbar_arrive_expect_tx(&b_full[s], static_cast<uint32_t>(nkb * kBNMax * kBK * 2));
        for (int kb = 0; kb < nkb; ++kb) {
          uint8_t* bk = b + kb * (kBNMax * kBK * 2);
          if constexpr (!kTB) tma_load_2d(&tmB, &b_full[s], bk, kb * kBK, n0);
          else
            for (int j = 0; j < kBNMax / 64; ++j) tma_load_2d(&tmB, &b_full[s], bk + j * 8192, n0 + 64 * j, kb * kBK);
        }
      }
      __syncwarp();
      if constexpr (kGG) {
        // the tile's gelu_grad_of rows: one 256-byte bulk copy per row, spread over the warp
        mbar_wait(&h_empty[s], ph ^ 1u);
        if (lane == 0) mbar_arrive_expect_tx(&h_full[s], static_cast<uint32_t>(rows * kBNMax * 2));
        __syncwarp();
        uint8_t* h = sH + s * SM::kHBytes;
        for (int r = static_cast<int>(lane); r < rows; r += 32)
          bulk_load_1d(h + r * SM::kHPitch, ep.gelu_grad_of + static_cast<size_t>(m0 + r) * ep.ld_gg + n0,
                       kBNMax * 2, &h_full[s]);
        __syncwarp();
      }
    }
    return;
  }

  // ===================== consumer warpgroups: MMA, epilogue, bulk stores =====================
  setmaxnreg_inc<SM::kMmaRegs>();
  const uint32_t wg = (warp - 4u) >> 2;
  const uint32_t tid = threadIdx.x - 128u - wg * 128u;              // thread index inside the warpgroup
  auto wg_bar = [wg] { asm volatile("bar.sync %0, 128;" ::"r"(1u + wg) : "memory"); };
  uint8_t* ring = sOut + wg * (SM::kSlots * SM::kSlotBytes);
  // this thread's fragment: rows r_frag + 8 h of the warpgroup's 64, columns 8 j + c_frag + {0, 1} -> d[4 j + 2 h + e]
  const int r_frag = static_cast<int>(((warp - 4u) & 3u) * 16u + (lane >> 2));
  const int c_frag = 2 * static_cast<int>(lane & 3u);
  const int row0 = m0 + static_cast<int>(wg) * 64;                  // first row of this warpgroup
  // the half-tile's bulk stores, one per row and output, spread over all four warps: thread tid stores output
  // st_part of row st_row (kEpiAct), or row st_row from the even threads (one output)
  const int st_row = SM::kOuts == 2 ? static_cast<int>(tid & 63u) : static_cast<int>(tid >> 1);
  const int st_part = SM::kOuts == 2 ? static_cast<int>(tid >> 6) : static_cast<int>(tid & 1u);
  bool storer = row0 + st_row < sh.M;                               // rows >= M are never stored
  if constexpr (kF == kEpiAct) storer = storer && (st_part == 0 || ep.out_bf16_pre != nullptr);
  else storer = storer && st_part == 0;

  auto issue = [&](float (&d)[64], int i) {
    const int s = i % SM::kStages;
    mbar_wait(&b_full[s], static_cast<uint32_t>(i / SM::kStages) & 1u);
    const uint32_t a = smem_u32(sA) + wg * 8192u;
    const uint32_t b = smem_u32(sB + s * SM::kBBytes);
    // per-k16 advance of the weight descriptor: 32 B inside a K-major row, two 8-row atoms MN-major
    constexpr uint32_t b_kadv = kTB ? 2048u : 32u, b_lbo = kTB ? 8192u : 0u;
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < nkb; ++kb) {
#pragma unroll
      for (int k = 0; k < kBK / 16; ++k)
        wgmma_m64n128k16_bf16<0, kTB>(d, make_smem_desc_sw128(a + kb * 16384u + k * 32u, 0u, 1024u),
                                      make_smem_desc_sw128(b + kb * 16384u + k * b_kadv, b_lbo, 1024u),
                                      (kb | k) != 0 ? 1u : 0u);
    }
    wgmma_commit();
  };
  // tile i's MMAs are done: its weight stage may be refilled
  auto release_b = [&](int i) {
    if (lane == 0) mbar_arrive(&b_empty[i % SM::kStages]);
  };

  // Tile i leaves as half-tiles q = 2 i + h, staged in ring slot q % kSlots.  Every thread commits one bulk group per
  // half-tile (empty if it stores nothing), so waiting until kSlots - 1 groups remain means half-tile q - kSlots, the
  // slot's previous contents, has been read out.
  // The bias of half-tile q + 1 is read from global memory while half-tile q is staged: thread tid < 64 holds its
  // column tid and puts it into the slot before the slot's first barrier, so the staging reads it from shared memory.
  float bias_next = 0.f;
  auto load_bias = [&](int q) {
    if constexpr (!kGG) {
      if (ep.bias != nullptr && tid < 64u && q < 2 * tpc)
        bias_next = __ldg(ep.bias + (nt0 + q / 2) * kBNMax + SM::kHalf * (q % 2) + static_cast<int>(tid));
    }
  };
  load_bias(0);
  auto epilogue = [&](const float (&d)[64], int i) {
    const int n0 = (nt0 + i) * kBNMax;
    const int s = i % SM::kStages;
    if constexpr (kGG) mbar_wait(&h_full[s], static_cast<uint32_t>(i / SM::kStages) & 1u);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint8_t* slot = ring + ((2 * i + h) % SM::kSlots) * SM::kSlotBytes;
      const float* sbias = reinterpret_cast<const float*>(slot + SM::kBiasOff);
      if constexpr (!kGG) {
        // the slot's bias was last read while half-tile q - kSlots was staged, before this thread's later barriers
        if (ep.bias != nullptr && tid < 64u) reinterpret_cast<float*>(slot + SM::kBiasOff)[tid] = bias_next;
        load_bias(2 * i + h + 1);
      }
      bulk_wait_read<SM::kSlots - 1>();
      wg_bar();
#pragma unroll
      for (int jh = 0; jh < 8; ++jh) {
        const int j = 8 * h + jh;               // column octet of the tile
        const int col = 8 * jh + c_frag;        // column inside the half-tile
        float2 bj = make_float2(0.f, 0.f);
        if constexpr (kF != kEpiGG) {
          if (ep.bias != nullptr) bj = *reinterpret_cast<const float2*>(sbias + col);
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int r = r_frag + 8 * e;
          float v0 = d[4 * j + 2 * e], v1 = d[4 * j + 2 * e + 1];
          if constexpr (kF == kEpiF32) {
            if (ep.bias != nullptr) add_pair(v0, v1, bj.x, bj.y);
            *reinterpret_cast<float2*>(slot + r * SM::kSPitch + col * 4) = make_float2(v0, v1);
          } else if constexpr (kF == kEpiAct) {
            if (ep.bias != nullptr) add_pair(v0, v1, bj.x, bj.y);
            *reinterpret_cast<uint32_t*>(slot + r * SM::kSPitch + col * 2) =
                pack_bf16x2(act_apply_select(v0, ep.act), act_apply_select(v1, ep.act));
            *reinterpret_cast<uint32_t*>(slot + (64 + r) * SM::kSPitch + col * 2) = pack_bf16x2(v0, v1);
          } else {
            const uint8_t* hrow = sH + s * SM::kHBytes + (static_cast<int>(wg) * 64 + r) * SM::kHPitch;
            const float2 g =
                __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(hrow + (SM::kHalf * h + col) * 2));
            v0 *= gelu_tanh_grad_f(g.x);
            v1 *= gelu_tanh_grad_f(g.y);
            *reinterpret_cast<uint32_t*>(slot + r * SM::kSPitch + col * 2) = pack_bf16x2(v0, v1);
          }
        }
      }
      if constexpr (kGG) {
        if (h == 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&h_empty[s]);
        }
      }
      fence_proxy_async_smem();   // the staged half-tile is read by the bulk-copy (async) proxy
      wg_bar();
      if (storer) {
        const size_t row = static_cast<size_t>(row0 + st_row);
        const int c0 = n0 + SM::kHalf * h;
        if constexpr (kF == kEpiF32) {
          bulk_store_1d(ep.out_f32 + row * ep.ld_f32 + c0, slot + st_row * SM::kSPitch, SM::kHalf * 4);
        } else {
          __nv_bfloat16* dst = st_part == 0 ? ep.out_bf16 : ep.out_bf16_pre;
          bulk_store_1d(dst + row * ep.ld_bf16 + c0, slot + (64 * st_part + st_row) * SM::kSPitch, SM::kHalf * 2);
        }
      }
      bulk_commit();
    }
    if constexpr (kF == kEpiF32) {
      if (ep.row_stats != nullptr) {
        // From the tile's two staged halves, once the accumulators are dead (their slots are next written by
        // half-tiles 2 i + 3 and 2 i + 4, after barriers this thread has not reached yet).  Two threads per row: part 0
        // sums chunk 0, then chunk 3 (column group 0); part 1 sums chunk 1 (group 1), then chunk 2 (group 2).
        const int r = static_cast<int>(tid & 63u), part = static_cast<int>(tid >> 6);
        const int row = row0 + r;
        if (row < sh.M) {
          const size_t slot0 =
              static_cast<size_t>(row) * ((sh.N / kBNMax) * SM::kEpiGroups) + (nt0 + i) * SM::kEpiGroups;
          auto put = [&](int g, float s1, float s2) {
            if (ep.stats_part != nullptr) {
              reinterpret_cast<float2*>(ep.stats_part)[slot0 + g] = make_float2(s1, s2);
            } else {
              atomicAdd(ep.row_stats + 2 * static_cast<size_t>(row), s1);
              atomicAdd(ep.row_stats + 2 * static_cast<size_t>(row) + 1, s2);
            }
          };
          auto add_chunk = [&](int q, int half_chunk, float& s1, float& s2) {   // half-tile q, its chunk 0 or 1
            const float4* src = reinterpret_cast<const float4*>(ring + (q % SM::kSlots) * SM::kSlotBytes +
                                                                r * SM::kSPitch + half_chunk * 128);
            float v[32];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              const float4 t = src[k];
              v[4 * k] = t.x; v[4 * k + 1] = t.y; v[4 * k + 2] = t.z; v[4 * k + 3] = t.w;
            }
            chunk_stats(v, s1, s2);
          };
          float s1 = 0.f, s2 = 0.f;
          add_chunk(2 * i, part, s1, s2);
          if (part == 1) {
            put(1, s1, s2);
            s1 = 0.f;
            s2 = 0.f;
          }
          add_chunk(2 * i + 1, 1 - part, s1, s2);
          put(part == 0 ? 0 : 2, s1, s2);
        }
      }
    }
  };

  mbar_wait(a_full, 0);
  float da[64], db[64];
  issue(da, 0);
  for (int i = 0; i + 2 < tpc; i += 2) {
    issue(db, i + 1); wgmma_wait<1>(); release_b(i); epilogue(da, i);
    issue(da, i + 2); wgmma_wait<1>(); release_b(i + 1); epilogue(db, i + 1);
  }
  issue(db, tpc - 1); wgmma_wait<1>(); release_b(tpc - 2); epilogue(da, tpc - 2);
  wgmma_wait<0>(); release_b(tpc - 1); epilogue(db, tpc - 1);
  // the outputs are written before the CTA (and its staging ring) goes away
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

}  // namespace smd

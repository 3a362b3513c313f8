// Host side of the wgmma GEMM: tensor-map construction (cuTensorMapEncodeTiled through the runtime's
// driver-entry-point lookup, so libsmd.so has no link-time dependency on libcuda) and the launcher.
#pragma once
#include <cstdlib>
#include <cuda.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>
#include <atomic>
#include <string>
#include "gemm_wgmma.cuh"
#include "fused_wgmma.cuh"

namespace smd {

extern std::atomic<long long> g_launches;
void set_error(const std::string& msg);

inline PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || p == nullptr) return nullptr;
  fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  return fn;
}

// bf16 row-major matrix [rows][cols]; box = box_rows x 64 columns (128 bytes, SWIZZLE_128B).  pitch: row pitch in
// elements when the matrix is a column slice of a wider one (0: cols)
inline bool make_tmap_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows,
                           uint64_t pitch = 0) {
  auto fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)"); return false; }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {(pitch ? pitch : cols) * 2};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed: code " + std::to_string(static_cast<int>(r)) + " rows=" +
              std::to_string(rows) + " cols=" + std::to_string(cols) + " box_rows=" + std::to_string(box_rows));
    return false;
  }
  return true;
}

struct GemmOp {
  CUtensorMap tmA, tmB;
  CUtensorMap tmA_lo, tmB_lo;   // strict-precision mode: the lo halves of both operands (has_lo)
  bool has_lo = false;
  int N = 0, K = 0, BN = 0, a_mn = 0, b_mn = 0, k_splits = 1;
};

inline int choose_bn(int N) {
  if (N % kBNMax == 0 || N > kBNMax) return kBNMax;
  return ((N + 15) / 16) * 16;
}

// A: K-major [a_rows][K] (a_mn=0) or MN-major [K][a_rows] (a_mn=1); same for B with N rows.
// BN = kBNWide asks for the wide layout (GemmSmemWide).  It is kept for N % 256 == 0 and K > 256, where gemm_kind may
// run that layout; any other BN above kBNMax is lowered to kBNMax.  The tensor maps do not depend on the choice (B's
// box is at most 128 rows; the wide kernel loads its 256 rows as two boxes), so a launch that gemm_kind does not give
// the wide layout runs the same op with 128-wide tiles.
// b_pitch: row pitch (elements) of an MN-major B that is a column slice of a wider matrix (0: b_rows_total)
inline bool make_gemm_op(GemmOp* op, const void* A, uint64_t a_rows, const void* B, uint64_t b_rows_total, int N,
                         int K, int BN, int a_mn, int b_mn, uint64_t k_rows_a = 0, uint64_t k_rows_b = 0,
                         size_t lo_bytes = 0, uint64_t b_pitch = 0) {
  if (lo_bytes) {
    GemmOp lo;
    if (!make_gemm_op(&lo, static_cast<const uint8_t*>(A) + lo_bytes, a_rows, static_cast<const uint8_t*>(B) + lo_bytes,
                      b_rows_total, N, K, BN, a_mn, b_mn, k_rows_a, k_rows_b, 0, b_pitch)) return false;
    op->tmA_lo = lo.tmA; op->tmB_lo = lo.tmB; op->has_lo = true;
  }
  if (BN > kBNMax && !(BN == kBNWide && N % kBNWide == 0 && K > 256)) BN = kBNMax;
  op->N = N; op->K = K; op->BN = BN; op->a_mn = a_mn; op->b_mn = b_mn; op->k_splits = 1;
  if (K % 64 != 0) { set_error("GEMM K must be a multiple of 64"); return false; }
  if (BN % 16 != 0 || BN < 16) { set_error("bad BN " + std::to_string(BN)); return false; }
  if (b_mn && BN % 64 != 0) { set_error("MN-major B needs BN % 64 == 0"); return false; }
  bool ok;
  if (!a_mn) ok = make_tmap_bf16(&op->tmA, A, a_rows, static_cast<uint64_t>(K), 128);
  else ok = make_tmap_bf16(&op->tmA, A, k_rows_a ? k_rows_a : static_cast<uint64_t>(K), a_rows, 64);
  if (!ok) return false;
  if (!b_mn) ok = make_tmap_bf16(&op->tmB, B, b_rows_total, static_cast<uint64_t>(K), static_cast<uint32_t>(BN < kBNMax ? BN : kBNMax));
  else ok = make_tmap_bf16(&op->tmB, B, k_rows_b ? k_rows_b : static_cast<uint64_t>(K), b_rows_total, 64, b_pitch);
  return ok;
}

inline int device_sm_count() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}

// feature bits a launch needs, and whether it qualifies for a specialised (fast-path-only) instantiation
inline uint32_t epi_needs(const GemmEpilogue& e) {
  uint32_t f = 0;
  if (e.bias) f |= F_BIAS;
  if (e.residual) f |= F_RES;
  if (e.out_f32) f |= F_F32;
  if (e.out_bf16) f |= F_BF16;
  if (e.out_bf16_pre) f |= F_PRE;
  if (e.row_stats) f |= F_STATS;
  if (e.ln_gamma) f |= F_LN;
  if (e.gelu_grad_of) f |= F_GG;
  if (e.atomic_out) f |= F_ATOMIC;
  if (e.act != ACT_NONE) f |= F_ACT;
  if (e.out_scale != 0.0f && e.out_scale != 1.0f) f |= F_SCALE;
  return f;
}
// The fast epilogue kinds store every column of every n-tile: N must be a whole number of tiles.  (An N that is a
// multiple of 32 but not of BN -- the TransformerMDN head, 2 KCp + Kcp = 960 columns at 10 components -- would write
// the last tile's columns [N, BN-rounded N) into the next row of an output whose row pitch is N.)
inline bool epi_clean(const GemmOp& op, const GemmEpilogue& e) {
  auto a16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
  return (op.N % 32 == 0) && (op.BN % 32 == 0) && (op.N % op.BN == 0) && (!e.residual || ((e.ld_res & 3) == 0 && a16(e.residual))) &&
         (!e.out_f32 || ((e.ld_f32 & 3) == 0 && a16(e.out_f32))) &&
         ((!e.out_bf16 && !e.out_bf16_pre) || (e.ld_bf16 & 7) == 0) && (!e.out_bf16 || a16(e.out_bf16)) &&
         (!e.out_bf16_pre || a16(e.out_bf16_pre)) && (!e.gelu_grad_of || ((e.ld_gg & 7) == 0 && a16(e.gelu_grad_of))) &&
         (!e.bias || a16(e.bias)) && (!e.ln_gamma || (a16(e.ln_gamma) && a16(e.ln_beta)));
}

// the K-split count every split of which owns at least one 64-wide k block
inline int gemm_k_splits(const GemmOp& op) {
  const int num_kb = op.K / kBK;
  int splits = op.k_splits < 1 ? 1 : op.k_splits;
  if (splits > num_kb) splits = num_kb;
  const int per = (num_kb + splits - 1) / splits;
  return (num_kb + per - 1) / per;
}
inline int gemm_tiles(const GemmOp& op, int M) {
  return ((M + kBM - 1) / kBM) * ((op.N + op.BN - 1) / op.BN) * gemm_k_splits(op);
}

// SMD_PDL=0 launches the persistent kernels without programmatic dependent launch.  That is faster for the sampler's
// forward passes and slower for the train step, so it stays selectable until the code makes that choice itself.
inline bool pdl_enabled() {
  static const bool on = [] { const char* v = getenv("SMD_PDL"); return !(v && v[0] == '0'); }();
  return on;
}

// persistent grid of min(#SMs, tiles) CTAs, programmatic dependent launch unless SMD_PDL=0
template <typename Kern, typename... Args>
inline cudaError_t launch_persistent(Kern kern, int tiles, int threads, int smem, cudaStream_t st, const Args&... args) {
  int grid = device_sm_count();
  if (tiles < grid) grid = tiles;
  if (grid < 1) grid = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(grid));
  cfg.blockDim = dim3(static_cast<unsigned>(threads));
  cfg.dynamicSmemBytes = static_cast<size_t>(smem);
  cfg.stream = st;
  cudaLaunchAttribute attrs[1];
  attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attrs[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attrs;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return cudaLaunchKernelEx(&cfg, kern, args...);
}

// The GEMM instantiation a launch runs: epilogue feature set and thread layout (GemmSmem's kEW, or the wide layout).
struct GemmKind {
  uint32_t flags;
  int ew;
  bool wide = false;   // 128 x 256 tiles (GemmSmemWide); ew is then unused
};
// the 128-wide tiles a launch of an op built with BN = kBNWide runs when gemm_kind does not give it the wide layout
inline GemmOp narrow_op(const GemmOp& op) {
  GemmOp o = op;
  if (o.BN > kBNMax) o.BN = kBNMax;
  return o;
}
inline GemmKind gemm_kind(const GemmOp& op, int M, const GemmEpilogue& ep) {
  if (op.BN > kBNMax) {
    // Wide layout: ops built with BN = kBNWide (the res-block GEMMs), long K, one split, and a clean epilogue of one of
    // two kinds: fp32 out (dW) or bf16 out without activation (res-block a, dX).  Its epilogue runs on the MMA warps
    // from registers, not overlapped with MMA work.  The residual kind (res-block b) reads 128 KB of fp32 residual per
    // tile; in the wide layout that latency is exposed and costs more than the faster K loop gains, so it keeps the
    // dedicated-epilogue layout.  A launch whose 128-wide tiles fit in one round keeps them: halving the CTA count
    // would leave SMs idle.
    if (ep.lo_delta == 0 && op.K > 256 && op.N % kBNWide == 0 && gemm_k_splits(op) == 1 && epi_clean(op, ep) &&
        gemm_tiles(narrow_op(op), M) > device_sm_count()) {
      const uint32_t need = epi_needs(ep);
      for (const uint32_t kind : {kEpiF32, kEpiBf16})
        if ((need & ~kind) == 0) return {kind, 8, true};
    }
    return gemm_kind(narrow_op(op), M, ep);
  }
  if (ep.lo_delta != 0) return {kEpiStrict, 8};   // strict-precision mode (bf16x3)
  const uint32_t need = epi_needs(ep);
  if (epi_clean(op, ep)) {
    auto fits = [&](uint32_t kind) { return (need & ~kind) == 0; };
    // short-K GEMMs are epilogue-bound: give them a third epilogue warp per row quadrant
    const bool short_k = op.K <= 256;
    // long-K launches of several rounds: a dedicated epilogue warpgroup hides each tile's epilogue behind the next
    // tile's K loop.  A single round has no next tile to overlap with; its exposed epilogue keeps the 8-warp layout,
    // which runs it on twice as many warps.
    const bool overlap = !short_k && gemm_tiles(op, M) > device_sm_count();
    if (fits(kEpiF32)) return {kEpiF32, short_k ? 12 : overlap ? 4 : 8};
    if (fits(kEpiAtomic)) return {kEpiAtomic, 8};
    if (fits(kEpiF32Res)) return {kEpiF32Res, overlap ? 4 : 8};
    if (fits(kEpiAct)) return {kEpiAct, short_k ? 12 : overlap ? 4 : 8};
    if (fits(kEpiGG)) return {kEpiGG, 8};
    if ((need & F_LN) && fits(kEpiLn) && op.N == op.BN && op.BN <= 128 && op.BN % 64 == 0 && op.k_splits <= 1)
      return {kEpiLn, 8};
  }
  return {kEpiGeneric, 8};
}
// Slots per row of the per-tile statistics partials (GemmEpilogue::stats_part) the launch writes: one per n-tile and
// column group of its instantiation.
inline int stats_slots_for(const GemmOp& op, int M, const GemmEpilogue& ep) {
  const GemmKind k = gemm_kind(op, M, ep);
  if (k.wide) return (op.N / kBNWide) * GemmSmemWide::kEpiGroups;
  const GemmOp o = narrow_op(op);
  return ((o.N + o.BN - 1) / o.BN) * epi_groups(k.ew);
}

template <uint32_t kF, int kEW = 8>
inline cudaError_t launch_gemm_inst(const GemmOp& op, int M, const GemmEpilogue& ep, cudaStream_t st) {
  using SM = GemmSmem<kEW>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_wgmma_kernel<kF, kEW>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         SM::kTotal);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  GemmShape sh;
  sh.M = M; sh.N = op.N; sh.K = op.K; sh.BN = op.BN; sh.a_mn = op.a_mn; sh.b_mn = op.b_mn;
  sh.k_splits = gemm_k_splits(op);
  return launch_persistent(gemm_bf16_wgmma_kernel<kF, kEW>, gemm_tiles(op, M), SM::kThreads, SM::kTotal, st, op.tmA,
                           op.tmB, sh, ep);
}
// the kEpiF32 / kEpiAct kinds exist in all three layouts
template <uint32_t kF>
inline cudaError_t launch_gemm_ew(int ew, const GemmOp& op, int M, const GemmEpilogue& ep, cudaStream_t st) {
  return ew == 12 ? launch_gemm_inst<kF, 12>(op, M, ep, st)
                  : ew == 4 ? launch_gemm_inst<kF, 4>(op, M, ep, st) : launch_gemm_inst<kF, 8>(op, M, ep, st);
}

template <uint32_t kF>
inline cudaError_t launch_gemm_wide(const GemmOp& op, int M, const GemmEpilogue& ep, cudaStream_t st) {
  using SM = GemmSmemWide;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_wgmma_wide_kernel<kF>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         SM::kTotal);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  GemmShape sh;
  sh.M = M; sh.N = op.N; sh.K = op.K; sh.BN = kBNWide; sh.a_mn = op.a_mn; sh.b_mn = op.b_mn; sh.k_splits = 1;
  const int tiles = ((M + kBM - 1) / kBM) * (op.N / kBNWide);
  return launch_persistent(gemm_bf16_wgmma_wide_kernel<kF>, tiles, SM::kThreads, SM::kTotal, st, op.tmA, op.tmB, sh, ep);
}

inline cudaError_t launch_gemm(const GemmOp& wop, int M, const GemmEpilogue& ep, cudaStream_t st) {
  const GemmKind k = gemm_kind(wop, M, ep);
  if (k.wide) {
    return k.flags == kEpiF32 ? launch_gemm_wide<kEpiF32>(wop, M, ep, st) : launch_gemm_wide<kEpiBf16>(wop, M, ep, st);
  }
  const GemmOp op = narrow_op(wop);
  // full-row LayerNorm needs the whole row in one tile (N <= BN; BN is at most kBNMax)
  if (ep.ln_gamma != nullptr && op.N > op.BN) return cudaErrorInvalidValue;
  // the K splits of a tile add into the same output elements
  if (gemm_k_splits(op) > 1 && !ep.atomic_out) return cudaErrorInvalidValue;
  switch (k.flags) {
    case kEpiStrict: return launch_gemm_inst<kEpiStrict>(op, M, ep, st);
    case kEpiF32: return launch_gemm_ew<kEpiF32>(k.ew, op, M, ep, st);
    case kEpiAtomic: return launch_gemm_inst<kEpiAtomic>(op, M, ep, st);
    case kEpiF32Res:
      return k.ew == 4 ? launch_gemm_inst<kEpiF32Res, 4>(op, M, ep, st) : launch_gemm_inst<kEpiF32Res>(op, M, ep, st);
    case kEpiAct: return launch_gemm_ew<kEpiAct>(k.ew, op, M, ep, st);
    case kEpiGG: return launch_gemm_inst<kEpiGG>(op, M, ep, st);
    case kEpiLn: return launch_gemm_inst<kEpiLn>(op, M, ep, st);
    default: return launch_gemm_inst<kEpiGeneric>(op, M, ep, st);
  }
}

// ---------------------------------------------------------------------------------------------------
// fused FFN (fused_wgmma.cuh)
// ---------------------------------------------------------------------------------------------------
struct FfnOp {
  CUtensorMap tmA, tmW1, tmW2;
  bool ok = false;
};
// A: bf16 [rows][128] K-major; W1: bf16 (128, Md) row-major; W2: bf16 (Md, 128) row-major (both MN-major B operands)
inline bool make_ffn_op(FfnOp* op, const void* A, uint64_t rows, const void* W1, const void* W2, int Md) {
  op->ok = make_tmap_bf16(&op->tmA, A, rows, 128, 128) && make_tmap_bf16(&op->tmW1, W1, 128, static_cast<uint64_t>(Md), 64) &&
           make_tmap_bf16(&op->tmW2, W2, static_cast<uint64_t>(Md), 128, 64);
  return op->ok;
}
inline cudaError_t launch_ffn_fused(const FfnOp& op, const FfnFusedArgs& a, cudaStream_t st) {
  if (a.Md % 128 != 0) return cudaErrorInvalidValue;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(ffn_fused_kernel<ACT_GELU_TANH>, cudaFuncAttributeMaxDynamicSharedMemorySize, FfnSmem::kTotal);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const int tiles = (a.M + 127) / 128;
  return launch_persistent(ffn_fused_kernel<ACT_GELU_TANH>, tiles, FfnSmem::kThreads, FfnSmem::kTotal, st, op.tmA, op.tmW1, op.tmW2, a);
}


// ---------------------------------------------------------------------------------------------------
// fused attention block (fused_wgmma.cuh)
// ---------------------------------------------------------------------------------------------------
struct AttnOp {
  CUtensorMap tmA, tmWqkv, tmWo;
  bool ok = false;
};
// A: bf16 [rows][128] K-major (64-row tiles); Wqkv: bf16 (128, 384) row-major; Wo: bf16 (128, 128) row-major
inline bool make_attn_op(AttnOp* op, const void* A, uint64_t rows, const void* Wqkv, const void* Wo) {
  op->ok = make_tmap_bf16(&op->tmA, A, rows, 128, 64) && make_tmap_bf16(&op->tmWqkv, Wqkv, 128, 384, 64) &&
           make_tmap_bf16(&op->tmWo, Wo, 128, 128, 64);
  return op->ok;
}
inline cudaError_t launch_attn_block(const AttnOp& op, const AttnBlockArgs& a, cudaStream_t st) {
  const int dh = 128 / a.H;
  if ((dh != 8 && dh != 16) || (a.S != 32 && a.S != 64) || a.M % a.S != 0) return cudaErrorInvalidValue;
  static bool attr_set = false;
  if (!attr_set) {
    for (auto k : {attn_block_kernel<16, 32>, attn_block_kernel<8, 32>, attn_block_kernel<16, 64>, attn_block_kernel<8, 64>}) {
      const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnSmem::kTotal);
      if (e != cudaSuccess) return e;
    }
    attr_set = true;
  }
  const int tiles = (a.M + 63) / 64;
  const int T = AttnSmem::kThreads, B = AttnSmem::kTotal;
  auto kernel = a.S == 64 ? (dh == 16 ? attn_block_kernel<16, 64> : attn_block_kernel<8, 64>)
                          : (dh == 16 ? attn_block_kernel<16, 32> : attn_block_kernel<8, 32>);
  return launch_persistent(kernel, tiles, T, B, st, op.tmA, op.tmWqkv, op.tmWo, a);
}

}  // namespace smd

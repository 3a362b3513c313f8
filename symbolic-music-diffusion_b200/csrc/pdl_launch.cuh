// Host-side helper for programmatic dependent launch (device side: pdl_wait / pdl_trigger in ptx.cuh).
#pragma once
#include <cuda_runtime.h>
#include <cstdlib>

#ifndef SMD_PDL_SIMT_DEFAULT
#define SMD_PDL_SIMT_DEFAULT 0
#endif

namespace smd {

// SMD_PDL: 0 = programmatic dependent launch off, 1 (default) = tensor-core GEMM launches only, 2 = SIMT kernels
// too.  Early-resident SIMT CTAs can hold shared memory that the
// ~220 KB GEMM CTAs of the weight-gradient stream need, so level 2 stays opt-in (not re-measured on H100).
inline int pdl_level() {
  static const int lvl = [] { const char* v = getenv("SMD_PDL"); return (v && v[0] >= '0' && v[0] <= '2') ? v[0] - '0' : 1; }();
  return lvl;
}
inline bool pdl_enabled() { return pdl_level() >= 1; }
// SMD_PDL_SIMT: bit mask of SIMT kernel groups that also launch programmatically at level 1
// (1: ln128_bwd, 2: attention fwd / bwd, 4: LayerNorm-FiLM forward, 8: LayerNorm-FiLM backward, 16: the rest).
// Default mask 0 (no group measured to pay off; not re-measured on H100).
inline int pdl_simt_mask() {
  static const int m = [] { const char* v = getenv("SMD_PDL_SIMT"); return v ? atoi(v) : SMD_PDL_SIMT_DEFAULT; }();
  return m;
}
// Launch with programmatic stream serialization: the kernel may be scheduled while its in-stream predecessor is
// still running; every kernel launched this way calls pdl_wait() before its first global-memory access.
enum PdlGroup : int { kPdlLn128 = 1, kPdlAttention = 2, kPdlLnFilmFwd = 4, kPdlLnFilmBwd = 8, kPdlMisc = 16 };
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_g(int group, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (pdl_level() >= 2 || (pdl_level() >= 1 && (pdl_simt_mask() & group))) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_level() >= 2 ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace smd

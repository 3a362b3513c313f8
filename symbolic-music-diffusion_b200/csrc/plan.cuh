// Shared internals of libsmd: the plan object, error helpers and launch-count macros.
#pragma once
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/smd.h"
#include "gemm_host.cuh"
#include "kernels.cuh"
#include "train.cuh"

#define SMD_CUDA(expr)                                                                              \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess) {                                                                        \
      set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));                               \
      return SMD_ERR_CUDA;                                                                          \
    }                                                                                               \
  } while (0)
#define SMD_LAUNCH_CHECK(what)                                                                      \
  do {                                                                                              \
    cudaError_t _e = cudaGetLastError();                                                            \
    if (_e != cudaSuccess) {                                                                        \
      set_error(std::string(what) + ": " + cudaGetErrorString(_e));                                \
      return SMD_ERR_CUDA;                                                                          \
    }                                                                                               \
  } while (0)
#define CNT() g_launches.fetch_add(1, std::memory_order_relaxed)

namespace smd {
extern std::atomic<long long> g_launches;
void set_error(const std::string& msg);
const char* get_error();

struct TensorInfo {
  std::string name;
  long long offset;
  int shape[4];
  int ndim;
  long long size() const {
    long long n = 1;
    for (int i = 0; i < ndim; ++i) n *= shape[i];
    return n;
  }
};

static constexpr int kE = 128;       // embed_channels (models/ncsn.py:151)
static constexpr int kFilmEmb = 128; // DenseFiLM embedding_channels (models/ncsn.py:174)
static constexpr int kFilmHid = 512; // embedding_channels * 4
static constexpr int kMaxT = 8192;

}  // namespace smd

using namespace smd;

struct smd_plan {
  smd_config cfg;
  std::vector<TensorInfo> tensors;
  std::map<std::string, long long> off;
  long long arena = 0;
  int Mp = 0;  // padded token rows
  // strict-precision mode: the workspace is allocated twice; the lo half of a bf16 operand at byte offset o lives at
  // o + lo_bytes (lo_elems in bf16 elements; both 0 when the mode is off)
  size_t lo_bytes = 0;
  long long lo_elems = 0;
  int K = 0;   // number of FiLM res-blocks (num_mlp_layers, or num_layers for DenseDDPM)
  // ---- workspace carve (byte offsets) ----
  std::map<std::string, size_t> ws_off;
  size_t ws_bytes = 0;
  uint8_t* ws = nullptr;
  bool packed = false;
  std::vector<smd::PackJob> pack_jobs;
  std::vector<int> stat_slots;   // per wide LayerNorm: partial slots per row its producing GEMM wrote (0: atomics / totals)
  int pack_tiles = 0;
  // ---- GEMM ops ----
  std::vector<GemmOp> op_qkv, op_o, op_ffn1, op_ffn2, op_a, op_b;
  std::vector<FfnOp> op_ffn;   // fused FFN (mlp_dims % 128 == 0)
  std::vector<AttnOp> op_attn; // fused attention block (head dim 8 / 16)
  GemmOp op_post, op_out, op_in;
  // sampler
  int T = 0;
  int T_obj = 0;  // schedule length of the training objective
  int L_dsm = 0;  // length of the sigma schedule of the denoising-score-matching objective (smd_dsm_setup)
  // FiLM table of the sampler: [K][T][2*Md]; when film_tab_on, run_forward skips the generator and the tail reads
  // row film_row (host) or *film_row_dev (graph replay) of the table
  bool film_tab_ready = false, film_tab_on = false;
  int film_row = 0;
  const int* film_row_dev = nullptr;
  const float* film_tab_params = nullptr;
  bool sampler_ready = false;
  long long shard_first_row = 0, shard_total_rows = 0;   // smd_sampler_set_shard
  cudaGraphExec_t graph_exec = nullptr;
  int graph_n = -1;
  const float* graph_params = nullptr;
  float* graph_x = nullptr;
  const float* graph_infill_x = nullptr;
  const float* graph_infill_mask = nullptr;
  float* graph_collection = nullptr;
  float* graph_metrics = nullptr;
  long long graph_nodes = 0;
  cudaStream_t own_stream = nullptr;
  cudaEvent_t own_event = nullptr;
  // training: the FiLM generator (forward and backward) runs on a side stream, concurrently with the trunk
  cudaStream_t side_stream = nullptr;   // FiLM generator forward / backward
  cudaStream_t dw_stream = nullptr;     // trunk weight-gradient GEMMs (leaves of the backward graph)
  cudaEvent_t ev_fork = nullptr, ev_film = nullptr, ev_dss = nullptr, ev_join = nullptr, ev_dw = nullptr, ev_dwjoin = nullptr, ev_tail = nullptr, ev_dwtail = nullptr;
  smd::TrainState train;
  // graph replay of smd_ddpm_grads (backward.cu)
  cudaGraphExec_t tg_exec = nullptr;
  long long tg_nodes = 0;
  bool tg_valid = false, tg_warm = false;
  cudaEvent_t ev_gz = nullptr;      // gradient arena zeroed (on the weight-gradient stream)
  cudaEvent_t evx_join = nullptr;   // "FiLM generator gradients final", waitable from outside the graph
  const float* tg_params = nullptr;
  float* tg_grads = nullptr;
  float* tg_loss = nullptr;
  int tg_batch = 0, tg_global = 0, tg_objective = 0;

  template <typename Tp>
  Tp* buf(const std::string& n) const { return reinterpret_cast<Tp*>(ws + ws_off.at(n)); }
  const float* P(const float* params, const std::string& n) const { return params + off.at(n); }
};


namespace smd {
inline GemmEpilogue epi() {
  GemmEpilogue e;
  memset(&e, 0, sizeof(e));
  return e;
}
// raw_out: DenseNCSN only -- leave out the final division by sigma (the training path differentiates through it itself)
int run_forward(smd_plan* p, const float* params, const float* x, const float* t, int t_broadcast, int batch,
                float* y, cudaStream_t st, TrainState* save, bool raw_out = false);
int train_bind(smd_plan* p);
int ensure_side_stream(smd_plan* p);
void add_pack_job_ptr(smd_plan* p, const std::string& src, void* dst, int K, int N, int mode, int ld);
}  // namespace smd

// Shared internals of libsmd: the plan object, its parameter and workspace layouts, error helpers and launch-count macros.
#pragma once
#include <cstdint>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "../../include/smd.h"
#include "gemm_host.cuh"
#include "kernels.cuh"

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
// TransformerMDN: C + 2 Kc floats of dynamic shared memory per mixture-NLL row (48 KB less the kernel's static part)
static constexpr int kMdnMaxRowFloats = (48 * 1024 - 256) / 4;

// Parameter arena offsets (in floats).  The same offset indexes the fp32 parameters, the gradients and the bf16 shadow.
struct Dense { long long kernel = 0, bias = 0; };
struct Norm { long long scale = 0, bias = 0; };
struct LayerParams { Norm ln1; Dense qkv, out; Norm ln2; Dense ffn1, ffn2; };
struct FilmParams { Dense d1, d2, ss; };
struct BlockParams { FilmParams film; Norm ln_a; Dense a; Norm ln_b; Dense b; };   // TransformerMDN: no film
struct ParamLayout {
  Dense in;
  std::vector<LayerParams> layer;   // TransformerDDPM only
  Norm post_ln;                     // TransformerDDPM only
  Dense post;                       // TransformerDDPM only
  std::vector<BlockParams> block;   // FiLM'd residual blocks
  Norm out_ln;
  Dense out;                        // all but TransformerMDN
  Dense mdn_mu, mdn_log_sigma, mdn_pi;   // TransformerMDN: the mixture-density head (models/shared.py MDN)
};

// Workspace byte offsets of everything the forward pass, the objectives and the sampler use.
struct WorkspaceLayout {
  size_t wshadow = 0, out_pad = 0, xb = 0, stats = 0, stats_part = 0, tvec = 0, enc = 0, ss = 0, posenc = 0, freqs = 0;
  size_t xt = 0, eps_hat = 0, coef = 0, keys = 0, slots = 0, t_ptr = 0, abar = 0, sigmas = 0;
  size_t ftab_t = 0, ftab_enc = 0, ftab_e1 = 0, ftab_e2 = 0, ftab = 0;   // sampler FiLM table (sampler_T > 0)
  size_t x3_scratch = 0;                                                 // bf16x3 only
  // Forward activations by position: h[0..2L] (residual stream); a[2l] / a[2l+1] (LN1 / LN2 output of layer l),
  // a[2L] (post-LN output); qkv, o, hidden per layer; u[0..K] (tail residual stream); r1 per block; act[2k] / act[2k+1]
  // (LN-a / LN-b output of block k), act[2K] (out-LN output); e1, e2 per block.  A training plan has one region per
  // index (the backward pass reads them all); an inference plan gives every index of a family the same region.
  std::vector<size_t> h, a, qkv, o, hidden, u, r1, act, e1, e2;
  std::vector<size_t> hidden_pre, probs, e1pre;   // written by the training forward only; empty in an inference plan
  // DenseNCSN only -- tangent (Jacobian-vector product) pass of sliced score matching, same indexing as the primal
  // families: xbt (bf16 input tangent v), ut[0..K] (fp32), r1t per block (fp32), actt[0..2K] (bf16), yt (output tangent)
  size_t xbt = 0, yt = 0;
  std::vector<size_t> ut, r1t, actt;
  // TransformerMDN only: fp32 head output [Mp][Np] = [mu | log_sigma | pi] (each part padded to 64 columns) and the
  // matching padded fp32 bias [Np]; out_pad then holds the packed bf16 head weight [Md][Np]
  size_t head = 0, head_bias = 0;
  // TransformerMDN plans created with sampler_T > 0 (autoregressive decoding, smd_mdn_sample): per layer the fp32 q / k /
  // v rows of every decoded position, [max_batch][S][384] like qkv, and the fp32 input token of the step [max_batch][C]
  std::vector<size_t> kv;
  size_t tok = 0;
};

// Named workspace region, for smd_debug_buffer.
struct WsRegion { std::string name; size_t offset, bytes; };

// Backward-only state of a training plan: its workspace regions (byte offsets) and GEMM descriptors.
struct TrainState {
  size_t g16 = 0;                      // bf16 [Mp][Md]: output of the tail's dX GEMMs
  size_t du32 = 0;                     // fp32 [Mp][Md]: gradient wrt the tail's residual stream u
  // bf16 gradient operands of the tail, one buffer per use (their dW GEMMs run on the weight-gradient stream):
  std::vector<size_t> du16;            // bf16 [Mp][Md] x (K+1): gradient wrt the residual stream u_j entering block j
  std::vector<size_t> dr16t;           // bf16 [Mp][Md] x K: gradient wrt r1 (after LayerNorm-b backward)
  size_t dh = 0, dh2 = 0;              // fp32 [Mp][128]
  // per-layer bf16 gradient operands: the dW GEMMs that read them run on their own stream, so no buffer is
  // rewritten within one backward pass
  std::vector<size_t> dh16a;           // bf16 [Mp][128] x L: gradient entering layer l (from LN1 of l+1 / post-LN)
  std::vector<size_t> dh16b;           // bf16 [Mp][128] x L: gradient at the attention output (from LN2)
  std::vector<size_t> dr16;            // bf16 [Mp][Md]  x L: gradient at the FFN pre-activation
  std::vector<size_t> dqkv16;          // bf16 [Mp][384] x L
  size_t dpred16 = 0;                  // bf16 [Mp][Cp64] (TransformerMDN: dZ, the head-output gradient [Mp][Np])
  size_t dpred32 = 0;                  // fp32 [Mp][C]
  size_t dss = 0;                      // fp32 [K][B][2Md]
  size_t de = 0, de2 = 0;              // fp32 [B][512] x2
  size_t loss = 0;                     // fp32 [B] (TransformerMDN: [B][S], one loss per token)
  size_t loss_ctr = 0;                 // u32: block-completion counter of the loss kernel (zeroed at bind, self-resetting)
  size_t ind = 0;                      // device table {x0, used_alpha, eps} of the graph-replayed step
  size_t e2_16 = 0, dss16 = 0;         // bf16 [Bp][512], [Bp][2Md]
  std::vector<GemmOp> dWb, dXb, dWa, dXa, dWss, dXss;
  std::vector<GemmOp> dW2, dX2, dW1, dX1, dWo, dXo, dWqkv, dXqkv;
  GemmOp dWout, dXout, dWpost, dXpost, dWin;
  GemmOp dWmdn[3];                     // TransformerMDN: dW of the mu / log_sigma / pi column slices of dZ
  // DenseNCSN only -- adjoints of the tangent pass (sliced score matching): gt16 / dut32 mirror g16 / du32, dut16 /
  // drt16 / dpredt16 mirror du16 / dr16t / dpred16, and the t* GEMMs are the tangent halves of the dW / dX GEMMs
  size_t gt16 = 0, dut32 = 0, dpredt16 = 0;
  std::vector<size_t> dut16, drt16;
  std::vector<GemmOp> tdWb, tdXb, tdWa, tdXa;
  GemmOp tdWout, tdXout, tdWin;
};

// Training objectives of the grads entry points (backward.cu); the value is the `mode` / `objective` the q_sample and
// loss kernels receive.
enum Objective : int { kObjDdpm = 0, kObjDsm = 1, kObjSsm = 2, kObjMdn = 3 };

// The sampler chain whose tables (coef / keys / slots / t_ptr, the FiLM table) the workspace holds: the DDPM sampler,
// the Langevin chain, the DDIM chain, the DDIM encoder and the DPM-Solver++ chain share those regions, so at most one of
// them is set up at a time.
enum Chain : int { kChainNone = 0, kChainDdpm = 1, kChainLangevin = 2, kChainDdim = 3, kChainDdimEncode = 4,
                   kChainDpm = 5 };
// The chain set up in the workspace and the per-chain values its calls read back.
struct ChainSetup {
  Chain kind = kChainNone;
  int rows = 0;                 // rows of the coef and FiLM tables: T (DDPM), K (DDIM, encoder, DPM), L (Langevin)
  int steps = 1;                // Langevin: steps per level (1 for the consistent chain and for the other chains)
  int tau0 = 0;                 // DDIM, DPM: the first selected index tau_0
  int order = 0;                // DPM: the solver order (1, 2 or 3)
  int lv_kind = 0;              // Langevin: 0 annealed, 1 consistent
  uint32_t key[2] = {0u, 0u};   // Langevin: the chain key
  float sigma_last = 0.f;       // Langevin: sigma_L
};

// The legacy default stream cannot be captured into a CUDA graph.
inline bool capturable(cudaStream_t st) { return st != nullptr && st != cudaStreamLegacy && st != cudaStreamPerThread; }

// The call arguments (pointers and integers) a graph was captured with.
using GraphKey = std::vector<uintptr_t>;
template <typename T>
inline uintptr_t key_word(T* ptr) { return reinterpret_cast<uintptr_t>(ptr); }
inline uintptr_t key_word(long long v) { return static_cast<uintptr_t>(v); }
template <typename... A>
inline GraphKey graph_key(A... a) { return GraphKey{key_word(a)...}; }

// A launch sequence captured once and replayed as one CUDA graph.  g_launches counts the captured launches once per
// replay (launch), not at capture.
struct CapturedGraph {
  cudaGraphExec_t exec = nullptr;
  long long nodes = 0;   // launches recorded by the capture
  GraphKey key;          // the arguments of the capture

  // a replay is valid only for the arguments the graph was captured with
  bool replays(const GraphKey& k) const { return exec && key == k; }
  void drop() {
    if (exec) cudaGraphExecDestroy(exec);
    exec = nullptr;
    key.clear();
  }
  // Replaces the graph by what body() enqueues on st (a capturable stream) for the arguments `k`; returns body's error
  // code or SMD_ERR_CUDA, leaving no graph behind on failure.
  template <typename Body>
  int capture(cudaStream_t st, GraphKey k, Body&& body, const char* what) {
    drop();
    cudaGraph_t graph = nullptr;
    const long long before = g_launches.load();
    SMD_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    const int rc = body();
    cudaError_t ce = cudaStreamEndCapture(st, &graph);
    nodes = g_launches.load() - before;
    g_launches.store(before);
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (ce != cudaSuccess) { set_error(std::string(what) + " capture: " + cudaGetErrorString(ce)); return SMD_ERR_CUDA; }
    ce = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce == cudaSuccess) { key = std::move(k); return SMD_OK; }
    exec = nullptr;
    set_error(std::string(what) + " instantiate: " + cudaGetErrorString(ce));
    return SMD_ERR_CUDA;
  }
  int launch(cudaStream_t st) {
    SMD_CUDA(cudaGraphLaunch(exec, st));
    g_launches.fetch_add(nodes, std::memory_order_relaxed);
    return SMD_OK;
  }
};

}  // namespace smd

using namespace smd;

struct smd_plan {
  smd_config cfg;
  std::vector<TensorInfo> tensors;
  ParamLayout par;
  long long arena = 0;
  int Mp = 0;  // padded token rows
  // strict-precision mode: the workspace is allocated twice; the lo half of a bf16 operand at byte offset o lives at
  // o + lo_bytes (lo_elems in bf16 elements; both 0 when the mode is off)
  size_t lo_bytes = 0;
  long long lo_elems = 0;
  int L = 0;   // transformer layers (0 for the dense networks)
  int K = 0;   // number of (FiLM) res-blocks (num_mlp_layers, or num_layers for DenseDDPM)
  // output layer width: C (columns of out.kernel, padded to Cp for the bf16 copy), or for TransformerMDN the packed
  // head, Kc mixture components: [mu | log_sigma | pi] with parts of Kc C, Kc C and Kc columns, each padded to 64
  int Kc = 0;
  int KCp = 0, Kcp = 0;          // padded widths of the mu / log_sigma parts and of the pi part (TransformerMDN)
  int head_n = 0, head_ld = 0;   // valid columns of the output GEMM and the row pitch of its bf16 weight copy
  bool mdn() const { return cfg.arch == SMD_ARCH_TRANSFORMER_MDN; }
  // ---- workspace ----
  WorkspaceLayout reg;
  std::vector<WsRegion> regions;
  size_t ws_bytes = 0;
  uint8_t* ws = nullptr;
  bool packed = false;
  std::vector<int> stat_slots;   // per wide LayerNorm: partial slots per row its producing GEMM wrote (0: atomics / totals)
  // ---- GEMM ops ----
  std::vector<GemmOp> op_qkv, op_o, op_ffn1, op_ffn2, op_a, op_b;
  std::vector<FfnOp> op_ffn;   // fused FFN (mlp_dims % 128 == 0)
  std::vector<AttnOp> op_attn; // fused attention block (head dim 8 / 16)
  GemmOp op_post, op_out, op_in;
  std::vector<GemmOp> op_ta, op_tb;   // DenseNCSN tangent pass: same weights, tangent activations, no bias
  GemmOp op_tin, op_tout;
  // sampler
  int T_obj = 0;  // schedule length of the training objective
  int L_dsm = 0;  // length of the sigma schedule of the denoising-score-matching objective (smd_dsm_setup)
  // FiLM table of the sampler: [K][T][2*Md], built for the parameters film_tab_params (see FilmRows)
  bool film_tab_ready = false;
  const float* film_tab_params = nullptr;
  long long shard_first_row = 0, shard_total_rows = 0;   // smd_sampler_set_shard
  // The chain set up (smd_sampler_setup, smd_ddim_setup, smd_ddim_encode_setup, smd_dpm_setup or smd_langevin_setup),
  // and the graph replay of one step of it (smd_ddpm_sample, smd_ddim_sample, smd_ddim_encode, smd_dpm_sample or
  // smd_langevin_sample).
  smd::ChainSetup chain;
  smd::CapturedGraph chain_graph;
  cudaStream_t own_stream = nullptr;
  cudaEvent_t own_event = nullptr;
  // training: the FiLM generator (forward and backward) runs on a side stream, concurrently with the trunk
  cudaStream_t side_stream = nullptr;   // FiLM generator forward / backward
  cudaStream_t dw_stream = nullptr;     // trunk weight-gradient GEMMs (leaves of the backward graph)
  cudaEvent_t ev_fork = nullptr, ev_film = nullptr, ev_dss = nullptr, ev_join = nullptr, ev_dw = nullptr, ev_dwjoin = nullptr, ev_tail = nullptr, ev_dwtail = nullptr;
  smd::TrainState train;
  cudaEvent_t ev_gz = nullptr;      // gradient arena zeroed (on the weight-gradient stream)
  cudaEvent_t evx_join = nullptr;   // "FiLM generator gradients final", waitable from outside the graph
  // graph replay of the grads entry points (backward.cu), and the key (params, batch, objective) of the last call that
  // ran eagerly: the first call of a configuration runs eagerly, the next one captures
  smd::CapturedGraph train_graph;
  smd::GraphKey train_warm;

  template <typename Tp>
  Tp* at(size_t off) const { return reinterpret_cast<Tp*>(ws + off); }
  __nv_bfloat16* wsh(long long off) const { return at<__nv_bfloat16>(reg.wshadow) + off; }   // bf16 shadow of a tensor
};


namespace smd {
inline GemmEpilogue epi() {
  GemmEpilogue e;
  memset(&e, 0, sizeof(e));
  return e;
}
// Where the res-blocks' FiLM scale / shift rows come from.  table == nullptr: the FiLM generator runs on the
// conditioning values t.  Otherwise the sampler's FiLM table (reg.ftab, [K][T][2*Md]): row `row`, or *row_dev when
// row_dev is set (graph replay).
struct FilmRows { const float* table = nullptr; int row = 0; const int* row_dev = nullptr; };
// raw_out: DenseNCSN only -- leave out the final division by sigma (the training path differentiates through it itself)
// save: training forward -- keep the unfused kernels and write the save-only outputs the backward pass reads
// tangent: DenseNCSN only -- also push the tangent already cast into reg.xbt through the network (Jacobian-vector
// product, raw output tangent into reg.yt); it reads the primal row statistics of each LayerNorm
int run_forward(smd_plan* p, const float* params, const float* x, const float* t, int t_broadcast, int batch,
                float* y, cudaStream_t st, bool save, bool raw_out = false, bool tangent = false, FilmRows film = {});
int train_bind(smd_plan* p);
int ensure_side_stream(smd_plan* p);
// Every forward GEMM goes through here (bf16x3 passes, and the per-tile row statistics of wide LayerNorm `ln_slot`).
cudaError_t gemm(smd_plan* p, const GemmOp& op, int M, GemmEpilogue e, cudaStream_t st, int ln_slot = -1);
// The residual tail from u[0] (row statistics in stats[0]) through out_ln and the output GEMM into y, M rows.
int run_tail(smd_plan* p, const float* params, int M, int S, int t_broadcast, float* y, cudaStream_t st, bool tangent,
             FilmRows film = {});
// host threefry block function and jax.random.split (out: num x 2 words)
void h_threefry(uint32_t k0, uint32_t k1, uint32_t& x0, uint32_t& x1);
void h_split(const uint32_t key[2], int num, uint32_t* out);

// Pieces of the backward pass shared by the objectives (backward.cu).  bwd_begin zeroes the gradient arena (on the
// weight-gradient stream) and the reduction-tail rows of every MN-major gradient operand (with tangent, also those of
// the sliced-score-matching tangent adjoints); bwd_out_ln runs the output layer's dX GEMM (operand dpred16) and the
// out_ln backward; bwd_tail the (FiLM) res-blocks, then records the events of smd_wait_tail_grads; bwd_trunk the
// post / transformer layers / input projection (input reg.xt) and the joins.
int bwd_begin(smd_plan* p, int M, int batch, float* grads, cudaStream_t st, bool tangent = false);
int bwd_out_ln(smd_plan* p, const float* params, int M, float* grads, cudaStream_t st);
int bwd_tail(smd_plan* p, const float* params, int batch, float* grads, cudaStream_t st, bool capturing);
int bwd_trunk(smd_plan* p, const float* params, int batch, float* grads, cudaStream_t st);
cudaError_t fork_dw(smd_plan* p, cudaStream_t st);
// out[n] += sum_m in[m * ld + n] (bias gradients from a bf16 gradient operand)
void launch_colsum_bf16(const __nv_bfloat16* in, int ld, float* out, int M, int N, cudaStream_t st);
int pick_splits_side(int m_rows, int n_cols, int BN, int num_kb);
// op with its reduction length set to K and split `splits` ways (the dW GEMMs reduce over the batch's token rows)
cudaError_t gemm_k(const GemmOp& op0, int rows, int K, int splits, const GemmEpilogue& e, cudaStream_t st);

// TransformerMDN (mdn.cu): packed head refresh, backward GEMM descriptors, and the train step body
int mdn_pack_head(smd_plan* p, const float* params, cudaStream_t st);
int mdn_train_bind(smd_plan* p);
int mdn_grads_impl(smd_plan* p, const float* params, const float* x, const float* const* ind, int batch,
                   int global_batch, float* grads, float* loss_sum, cudaStream_t st, bool capturing);
}  // namespace smd

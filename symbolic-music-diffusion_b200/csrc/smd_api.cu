// libsmd C ABI implementation: plan / parameter arena / workspace carving, the score-network forward,
// objective, sampler, jax-compatible RNG helpers and test hooks.  See include/smd.h.
#include "../../include/smd.h"

#include <cmath>
#include <cstdio>
#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "plan.cuh"

namespace smd {

std::atomic<long long> g_launches{0};
static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
const char* get_error() { return g_err.c_str(); }

static void add_tensor(smd_plan* p, const std::string& name, std::initializer_list<int> shape) {
  TensorInfo t;
  t.name = name;
  t.ndim = static_cast<int>(shape.size());
  int i = 0;
  for (int s : shape) t.shape[i++] = s;
  for (; i < 4; ++i) t.shape[i] = 1;
  t.offset = p->arena;
  p->off[name] = t.offset;
  p->arena += (t.size() + 7) / 8 * 8;  // 32-byte aligned in fp32 => 16-byte aligned in the bf16 shadow arena (TMA)
  p->tensors.push_back(t);
}

static void add_film_resblock(smd_plan* p, const std::string& pre, int Mdim) {
  add_tensor(p, pre + "film.d1.kernel", {kFilmEmb, kFilmHid});
  add_tensor(p, pre + "film.d1.bias", {kFilmHid});
  add_tensor(p, pre + "film.d2.kernel", {kFilmHid, kFilmHid});
  add_tensor(p, pre + "film.d2.bias", {kFilmHid});
  add_tensor(p, pre + "film.ss.kernel", {kFilmHid, 2 * Mdim});
  add_tensor(p, pre + "film.ss.bias", {2 * Mdim});
  add_tensor(p, pre + "res.ln_a.scale", {Mdim});
  add_tensor(p, pre + "res.ln_a.bias", {Mdim});
  add_tensor(p, pre + "res.a.kernel", {Mdim, Mdim});
  add_tensor(p, pre + "res.a.bias", {Mdim});
  add_tensor(p, pre + "res.ln_b.scale", {Mdim});
  add_tensor(p, pre + "res.ln_b.bias", {Mdim});
  add_tensor(p, pre + "res.b.kernel", {Mdim, Mdim});
  add_tensor(p, pre + "res.b.bias", {Mdim});
}

static void build_layout(smd_plan* p) {
  const smd_config& c = p->cfg;
  const int C = c.channels, Md = c.mlp_dims;
  if (c.arch == SMD_ARCH_TRANSFORMER_DDPM) {
    add_tensor(p, "in.kernel", {C, kE});
    add_tensor(p, "in.bias", {kE});
    for (int l = 0; l < c.num_layers; ++l) {
      const std::string pre = "l" + std::to_string(l) + ".";
      add_tensor(p, pre + "ln1.scale", {kE});
      add_tensor(p, pre + "ln1.bias", {kE});
      add_tensor(p, pre + "attn.qkv.kernel", {kE, 3 * kE});
      add_tensor(p, pre + "attn.qkv.bias", {3 * kE});
      add_tensor(p, pre + "attn.out.kernel", {kE, kE});
      add_tensor(p, pre + "attn.out.bias", {kE});
      add_tensor(p, pre + "ln2.scale", {kE});
      add_tensor(p, pre + "ln2.bias", {kE});
      add_tensor(p, pre + "ffn1.kernel", {kE, Md});
      add_tensor(p, pre + "ffn1.bias", {Md});
      add_tensor(p, pre + "ffn2.kernel", {Md, kE});
      add_tensor(p, pre + "ffn2.bias", {kE});
    }
    add_tensor(p, "post_ln.scale", {kE});
    add_tensor(p, "post_ln.bias", {kE});
    add_tensor(p, "post.kernel", {kE, Md});
    add_tensor(p, "post.bias", {Md});
    p->K = c.num_mlp_layers;
  } else {
    add_tensor(p, "in.kernel", {C, Md});
    add_tensor(p, "in.bias", {Md});
    p->K = c.num_layers;
  }
  for (int k = 0; k < p->K; ++k) add_film_resblock(p, "k" + std::to_string(k) + ".", Md);
  add_tensor(p, "out_ln.scale", {Md});
  add_tensor(p, "out_ln.bias", {Md});
  add_tensor(p, "out.kernel", {Md, C});
  add_tensor(p, "out.bias", {C});
}

static size_t ws_add(smd_plan* p, const std::string& name, size_t bytes) {
  const size_t off = p->ws_bytes;
  p->ws_off[name] = off;
  p->ws_bytes += (bytes + 1023) / 1024 * 1024;
  return off;
}

static void build_workspace(smd_plan* p) {
  const smd_config& c = p->cfg;
  const size_t Mp = p->Mp, Md = c.mlp_dims, C = c.channels, B = c.max_batch, K = p->K;
  const bool tr = c.arch == SMD_ARCH_TRANSFORMER_DDPM;
  // bf16 shadow of the whole parameter arena (same offsets): every GEMM weight operand is read from it in place --
  // forward as an MN-major B operand ((in,out) = [K][N]), dX as a K-major B operand ([N=in][K=out]) -- so there
  // are no transposed copies and the optimizer refreshes it in the same pass that updates the fp32 masters.
  ws_add(p, "wshadow", static_cast<size_t>(p->arena) * 2);
  // out.kernel is (Md, C) with C = 42 / 146: its 2C-byte row pitch is not TMA-addressable, so it gets a copy
  // zero-padded to a multiple of 64 columns
  ws_add(p, "w.out_pad", Md * ((C + 63) / 64 * 64) * 2);
  // activations
  if (tr) {
    ws_add(p, "h", Mp * kE * 4);
    ws_add(p, "a", Mp * kE * 2);
    ws_add(p, "qkv", Mp * 3 * kE * 4);
    ws_add(p, "o", Mp * kE * 2);
    ws_add(p, "hidden", Mp * Md * 2);
  } else {
    ws_add(p, "xb", Mp * ((C + 63) / 64 * 64) * 2);
  }
  ws_add(p, "u", Mp * Md * 4);
  ws_add(p, "r1", Mp * Md * 4);
  ws_add(p, "act", Mp * Md * 2);
  // per-row LayerNorm (sum, sumsq) of the 2K+1 wide LayerNorms; zeroed once per forward
  ws_add(p, "stats", (2 * K + 1) * Mp * 2 * 4);
  // per-tile partial sums of the GEMM feeding the next wide LayerNorm: [row][n_tile * (2 or 3) + column group][2]
  ws_add(p, "stats_part", Mp * ((Md + kBNMax - 1) / kBNMax * 3) * 2 * 4);
  // FiLM generator
  ws_add(p, "tvec", B * 4);
  ws_add(p, "enc", B * kFilmEmb * 4);
  ws_add(p, "e1", B * kFilmHid * 4);
  ws_add(p, "e2", B * kFilmHid * 4);
  ws_add(p, "ss", K * B * 2 * Md * 4);
  ws_add(p, "posenc", static_cast<size_t>(c.seq_len) * kE * 4);
  ws_add(p, "freqs", 64 * 4);
  // objective / sampler scratch
  ws_add(p, "xt", B * c.seq_len * C * 4);
  ws_add(p, "eps_hat", B * c.seq_len * C * 4);
  ws_add(p, "coef", kMaxT * 8 * 4);
  ws_add(p, "keys", kMaxT * 4 * 4);
  ws_add(p, "slots", kMaxT * 4);
  ws_add(p, "t_ptr", 64);
  ws_add(p, "abar", (kMaxT + 1) * 4);
  ws_add(p, "sigmas", kMaxT * 4);
  ws_add(p, "packjobs", 256 * sizeof(PackJob));
  ws_add(p, "packmap", 65536 * 8);
  if (c.sampler_T > 0) {
    const size_t T = c.sampler_T;
    ws_add(p, "ftab.t", T * 4);
    ws_add(p, "ftab.enc", T * kFilmEmb * 4);
    ws_add(p, "ftab.e1", T * kFilmHid * 4);
    ws_add(p, "ftab.e2", T * kFilmHid * 4);
    ws_add(p, "ftab", K * T * 2 * Md * 4);
  }
  if (c.training) train_workspace(p->train, c, p->Mp, p->K, [&](const std::string& n, size_t b) { return ws_add(p, n, b); });
  if (c.precision == SMD_PRECISION_BF16X3) {
    ws_add(p, "x3.scratch", Mp * Md * 4);     // fp32 cross-term accumulator of the three-pass GEMMs
    p->lo_bytes = p->ws_bytes;                // second copy of the workspace: the lo halves, at the same offsets
    p->lo_elems = static_cast<long long>(p->lo_bytes / 2);
    p->ws_bytes *= 2;
  }
}

// sinusoid frequency table, float32 like jnp (models/ncsn.py:33-35, models/shared.py:41-43)
static void host_freqs(float* f) {
  const float emb = logf(10000.0f) / 63.0f;
  for (int j = 0; j < 64; ++j) f[j] = expf(static_cast<float>(j) * -emb);
}

static int build_ops(smd_plan* p) {
  const smd_config& c = p->cfg;
  const int Md = c.mlp_dims, C = c.channels;
  const int Cp = (C + 63) / 64 * 64;
  const uint64_t Mp = p->Mp;
  auto A = [&](const std::string& n) { return p->buf<void>(n); };
  auto Wsh = [&](const std::string& n) { return static_cast<const void*>(p->buf<__nv_bfloat16>("wshadow") + p->off.at(n)); };
  // forward GEMM: A K-major activations [Mp][K], B = (in,out) weight read MN-major ([K][N]) from the shadow arena
  auto fwd = [&](GemmOp* op, const std::string& a, const std::string& w, int K, int N, int BN) {
    return make_gemm_op(op, A(a), Mp, Wsh(w), static_cast<uint64_t>(N), N, K, BN, 0, 1, 0, 0, p->lo_bytes);
  };
  if (c.arch == SMD_ARCH_TRANSFORMER_DDPM) {
    p->op_qkv.resize(c.num_layers); p->op_o.resize(c.num_layers);
    p->op_ffn1.resize(c.num_layers); p->op_ffn2.resize(c.num_layers);
    p->op_ffn.resize(c.num_layers);
    p->op_attn.resize(c.num_layers);
    for (int l = 0; l < c.num_layers; ++l) {
      const std::string pre = "l" + std::to_string(l) + ".";
      if (!fwd(&p->op_qkv[l], "a", pre + "attn.qkv.kernel", kE, 3 * kE, 128)) return SMD_ERR_CUDA;
      if (!fwd(&p->op_o[l], "o", pre + "attn.out.kernel", kE, kE, 128)) return SMD_ERR_CUDA;
      if (!fwd(&p->op_ffn1[l], "a", pre + "ffn1.kernel", kE, Md, 256)) return SMD_ERR_CUDA;
      if (!fwd(&p->op_ffn2[l], "hidden", pre + "ffn2.kernel", Md, kE, 128)) return SMD_ERR_CUDA;
      if (Md % 128 == 0 &&
          !make_ffn_op(&p->op_ffn[l], A("a"), Mp, Wsh(pre + "ffn1.kernel"), Wsh(pre + "ffn2.kernel"), Md)) return SMD_ERR_CUDA;
      if ((c.num_heads == 8 || c.num_heads == 16) &&
          !make_attn_op(&p->op_attn[l], A("a"), Mp, Wsh(pre + "attn.qkv.kernel"), Wsh(pre + "attn.out.kernel"))) return SMD_ERR_CUDA;
    }
    if (!fwd(&p->op_post, "a", "post.kernel", kE, Md, 256)) return SMD_ERR_CUDA;
  } else {
    if (!fwd(&p->op_in, "xb", "in.kernel", C, Md, 256)) return SMD_ERR_CUDA;
  }
  p->op_a.resize(p->K); p->op_b.resize(p->K);
  for (int k = 0; k < p->K; ++k) {
    const std::string pre = "k" + std::to_string(k) + ".res.";
    if (!fwd(&p->op_a[k], "act", pre + "a.kernel", Md, Md, 256)) return SMD_ERR_CUDA;
    if (!fwd(&p->op_b[k], "act", pre + "b.kernel", Md, Md, 256)) return SMD_ERR_CUDA;
  }
  // output projection from the padded copy [Md][Cp]: N = C columns are valid, the tile is Cp (<= 256) wide
  {
    const int BN = Cp >= 256 ? 256 : Cp;
    if (!make_gemm_op(&p->op_out, A("act"), Mp, A("w.out_pad"), static_cast<uint64_t>(Cp), C, Md, BN, 0, 1, 0, 0,
                      p->lo_bytes))
      return SMD_ERR_CUDA;
  }
  return SMD_OK;
}

// Every forward GEMM goes through here.  Default precision: one launch.  bf16x3: the product of the (hi, lo) operand
// pairs as three launches -- scratch = A_lo B_hi (+ the layer's residual); scratch += A_hi B_lo; then the real launch
// A_hi B_hi with the layer's epilogue taking `scratch` as its residual -- all accumulated in fp32.
// ln_slot >= 0: this GEMM feeds wide LayerNorm `ln_slot` through a stand-alone ln_film_act launch: its row statistics
// go out as per-tile partials (added in a fixed order by the consumer) instead of atomics.
static cudaError_t gemm(smd_plan* p, const GemmOp& op, int M, GemmEpilogue e, cudaStream_t st, int ln_slot = -1) {
  auto arm_stats = [&](GemmEpilogue& ef) {
    if (ln_slot < 0 || ef.row_stats == nullptr) return;
    ef.stats_part = p->buf<float>("stats_part");
    p->stat_slots[ln_slot] = stats_slots_for(op, M, ef);
  };
  if (p->lo_bytes == 0) { arm_stats(e); return launch_gemm(op, M, e, st); }
  if (!op.has_lo) return cudaErrorInvalidValue;
  float* scratch = p->buf<float>("x3.scratch");
  GemmOp o1 = op; o1.tmA = op.tmA_lo;
  GemmEpilogue e1 = epi();
  e1.residual = e.residual; e1.ld_res = e.ld_res;
  e1.out_f32 = scratch; e1.ld_f32 = op.N;
  cudaError_t err = launch_gemm(o1, M, e1, st);
  if (err != cudaSuccess) return err;
  GemmOp o2 = op; o2.tmB = op.tmB_lo;
  GemmEpilogue e2 = epi();
  e2.residual = scratch; e2.ld_res = op.N;
  e2.out_f32 = scratch; e2.ld_f32 = op.N;
  err = launch_gemm(o2, M, e2, st);
  if (err != cudaSuccess) return err;
  e.residual = scratch; e.ld_res = op.N;
  e.lo_delta = p->lo_elems;
  arm_stats(e);
  return launch_gemm(op, M, e, st);
}
// ln_film_act arguments for the statistics of wide LayerNorm `ln_slot` (partials + slot count, or totals)
struct LnStats { const float* part; int nslots; float* totals; };
static LnStats ln_stats(smd_plan* p, int ln_slot) {
  float* totals = p->buf<float>("stats") + static_cast<size_t>(ln_slot) * p->Mp * 2;
  const int n = p->stat_slots[ln_slot];
  return n > 0 ? LnStats{p->buf<float>("stats_part"), n, totals} : LnStats{nullptr, 0, totals};
}

// FiLM generator for all K blocks: t (R values) -> ss[k][R][2*Md]   (models/ncsn.py:47-61)
static int run_film(smd_plan* p, const float* params, const float* t, int R, cudaStream_t st, TrainState* save) {
  const int Md = p->cfg.mlp_dims;
  float* enc = p->buf<float>("enc");
  float* ss = p->buf<float>("ss");
  launch_noise_encoding(t, p->buf<float>("freqs"), enc, R, st); CNT();
  for (int k = 0; k < p->K; ++k) {
    const std::string pre = "k" + std::to_string(k) + ".film.";
    float* e1 = save ? save->at<float>(p->ws, save->off_e1[k]) : p->buf<float>("e1");
    float* e2 = save ? save->at<float>(p->ws, save->off_e2[k]) : p->buf<float>("e2");
    float* e1pre = save ? save->at<float>(p->ws, save->off_e1pre[k]) : nullptr;
    launch_small_linear(enc, p->P(params, pre + "d1.kernel"), p->P(params, pre + "d1.bias"), e1, R, kFilmEmb, kFilmHid, 2, st, e1pre); CNT();
    launch_small_linear(e1, p->P(params, pre + "d2.kernel"), p->P(params, pre + "d2.bias"), e2, R, kFilmHid, kFilmHid, 0, st); CNT();
    launch_small_linear(e2, p->P(params, pre + "ss.kernel"), p->P(params, pre + "ss.bias"),
                        ss + static_cast<size_t>(k) * p->cfg.max_batch * 2 * Md, R, kFilmHid, 2 * Md, 0, st); CNT();
  }
  SMD_LAUNCH_CHECK("film");
  return SMD_OK;
}

int ensure_side_stream(smd_plan* p) {
  if (p->side_stream) return SMD_OK;
  SMD_CUDA(cudaStreamCreateWithFlags(&p->side_stream, cudaStreamNonBlocking));
  SMD_CUDA(cudaEventCreateWithFlags(&p->ev_fork, cudaEventDisableTiming));
  SMD_CUDA(cudaEventCreateWithFlags(&p->ev_film, cudaEventDisableTiming));
  SMD_CUDA(cudaEventCreateWithFlags(&p->ev_dss, cudaEventDisableTiming));
  SMD_CUDA(cudaEventCreateWithFlags(&p->ev_join, cudaEventDisableTiming));
  SMD_CUDA(cudaStreamCreateWithFlags(&p->dw_stream, cudaStreamNonBlocking));
  SMD_CUDA(cudaEventCreateWithFlags(&p->ev_dw, cudaEventDisableTiming));
  SMD_CUDA(cudaEventCreateWithFlags(&p->ev_dwjoin, cudaEventDisableTiming));
  SMD_CUDA(cudaEventCreateWithFlags(&p->ev_tail, cudaEventDisableTiming));
  SMD_CUDA(cudaEventCreateWithFlags(&p->ev_dwtail, cudaEventDisableTiming));
  SMD_CUDA(cudaEventCreateWithFlags(&p->evx_join, cudaEventDisableTiming));
  SMD_CUDA(cudaEventCreateWithFlags(&p->ev_gz, cudaEventDisableTiming));
  return SMD_OK;
}

// The FiLM'd residual tail shared by both architectures (models/ncsn.py:173-178, models/shared.py:61-75).
// On entry u (fp32 [M][Md]) and stats[0] hold the block input and its row statistics.
static int run_tail(smd_plan* p, const float* params, int M, int S, int t_broadcast, float* y, cudaStream_t st,
                    smd::TrainState* save) {
  const int Md = p->cfg.mlp_dims, C = p->cfg.channels;
  float* u = p->buf<float>("u");
  float* r1 = p->buf<float>("r1");
  __nv_bfloat16* act = p->buf<__nv_bfloat16>("act");
  float* stats = p->buf<float>("stats");
  const size_t sstride = static_cast<size_t>(p->Mp) * 2;
  float* ss = p->buf<float>("ss");
  for (int k = 0; k < p->K; ++k) {
    const std::string pre = "k" + std::to_string(k) + ".res.";
    const float* scale = ss + static_cast<size_t>(k) * p->cfg.max_batch * 2 * Md;
    const int* frow_dev = nullptr;
    if (p->film_tab_on) {
      scale = p->buf<float>("ftab") + static_cast<size_t>(k) * p->T * 2 * Md;
      if (p->film_row_dev) frow_dev = p->film_row_dev; else scale += static_cast<size_t>(p->film_row) * 2 * Md;
    }
    const float* shift = scale + Md;
    float* u_in = u;
    __nv_bfloat16* r1_out = reinterpret_cast<__nv_bfloat16*>(r1);   // r1 only feeds a LayerNorm: bf16 is enough
    __nv_bfloat16* act_a = act;
    __nv_bfloat16* act_b = act;
    float* u_out = u;
    if (save) {  // training keeps every block's tensors
      u_in = save->u(p->ws, k); r1_out = reinterpret_cast<__nv_bfloat16*>(save->r1(p->ws, k)); act_a = save->act_a(p->ws, k);
      act_b = save->act_b(p->ws, k); u_out = save->u(p->ws, k + 1);
    }
    const bool strict = p->lo_bytes != 0;
    LnStats ls = ln_stats(p, 2 * k);
    launch_ln_film_act(u_in, ls.totals, p->P(params, pre + "ln_a.scale"), p->P(params, pre + "ln_a.bias"),
                       scale, shift, 2 * Md, t_broadcast, 2, act_a, M, Md, S, st, frow_dev, nullptr, p->lo_elems,
                       ls.part, ls.nslots, ls.totals); CNT();
    GemmEpilogue e = epi();
    e.bias = p->P(params, pre + "a.bias");
    if (strict) { e.out_f32 = r1; e.ld_f32 = Md; }       // (strict mode keeps the pre-LayerNorm intermediate in fp32)
    else { e.out_bf16 = r1_out; e.ld_bf16 = Md; }
    e.row_stats = stats + (2 * k + 1) * sstride;
    GemmOp opa = p->op_a[k];
    GemmOp opb = p->op_b[k];
    if (save) { if (!retarget_a(&opa, act_a, p->Mp) || !retarget_a(&opb, act_b, p->Mp)) return SMD_ERR_CUDA; }
    SMD_CUDA(gemm(p, opa, M, e, st, 2 * k + 1));
    ls = ln_stats(p, 2 * k + 1);
    launch_ln_film_act(strict ? r1 : nullptr, ls.totals, p->P(params, pre + "ln_b.scale"),
                       p->P(params, pre + "ln_b.bias"), scale, shift, 2 * Md, t_broadcast, 2, act_b, M, Md, S, st, frow_dev,
                       strict ? nullptr : r1_out, p->lo_elems, ls.part, ls.nslots, ls.totals); CNT();
    e = epi();
    e.bias = p->P(params, pre + "b.bias");
    e.residual = u_in; e.ld_res = Md;
    e.out_f32 = u_out; e.ld_f32 = Md;
    e.row_stats = stats + (2 * k + 2) * sstride;
    SMD_CUDA(gemm(p, opb, M, e, st, 2 * k + 2));
  }
  float* u_last = save ? save->u(p->ws, p->K) : u;
  __nv_bfloat16* act_o = save ? save->act_out(p->ws) : act;
  const LnStats lo_ = ln_stats(p, 2 * p->K);
  launch_ln_film_act(u_last, lo_.totals, p->P(params, "out_ln.scale"), p->P(params, "out_ln.bias"),
                     nullptr, nullptr, 0, 0, 0, act_o, M, Md, S, st, nullptr, nullptr, p->lo_elems, lo_.part, lo_.nslots,
                     lo_.totals); CNT();
  GemmEpilogue e = epi();
  e.bias = p->P(params, "out.bias");
  e.out_f32 = y; e.ld_f32 = C;
  GemmOp opo = p->op_out;
  if (save) { if (!retarget_a(&opo, act_o, p->Mp)) return SMD_ERR_CUDA; }
  SMD_CUDA(gemm(p, opo, M, e, st));
  SMD_LAUNCH_CHECK("tail");
  return SMD_OK;
}

int run_forward(smd_plan* p, const float* params, const float* x, const float* t, int t_broadcast, int batch,
                float* y, cudaStream_t st, smd::TrainState* save, bool raw_out) {
  const smd_config& c = p->cfg;
  if (!p->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (!p->packed) { set_error("smd_pack_weights has not been called"); return SMD_ERR_STATE; }
  if (batch < 1 || batch > c.max_batch) { set_error("batch out of range"); return SMD_ERR_INVALID; }
  const int S = c.seq_len, C = c.channels, Md = c.mlp_dims;
  const int M = batch * S;
  float* stats = p->buf<float>("stats");
  p->stat_slots.assign(static_cast<size_t>(2 * p->K + 1), 0);
  SMD_CUDA(cudaMemsetAsync(stats, 0, static_cast<size_t>(2 * p->K + 1) * p->Mp * 2 * 4, st));
  int rc = SMD_OK;
  bool film_on_side = false;
  if (!p->film_tab_on) {
    if (save) {
      // training: the FiLM generator only feeds the tail, so it runs on a side stream next to the trunk
      rc = ensure_side_stream(p);
      if (rc) return rc;
      SMD_CUDA(cudaEventRecord(p->ev_fork, st));
      SMD_CUDA(cudaStreamWaitEvent(p->side_stream, p->ev_fork, 0));
      rc = run_film(p, params, t, batch, p->side_stream, save);
      if (rc) return rc;
      SMD_CUDA(cudaEventRecord(p->ev_film, p->side_stream));
      film_on_side = true;
    } else {
      rc = run_film(p, params, t, t_broadcast ? 1 : batch, st, save);
    }
  }
  if (rc) return rc;
  float* u0 = save ? save->u(p->ws, 0) : p->buf<float>("u");
  if (c.arch == SMD_ARCH_TRANSFORMER_DDPM) {
    float* h = p->buf<float>("h");
    __nv_bfloat16* a = p->buf<__nv_bfloat16>("a");
    float* qkv = p->buf<float>("qkv");
    __nv_bfloat16* o = p->buf<__nv_bfloat16>("o");
    __nv_bfloat16* hidden = p->buf<__nv_bfloat16>("hidden");
    if (save) { h = save->h(p->ws, 0); a = save->a1(p->ws, 0); }
    launch_embed(x, p->P(params, "in.kernel"), p->P(params, "in.bias"), p->buf<float>("posenc"),
                 p->P(params, "l0.ln1.scale"), p->P(params, "l0.ln1.bias"), h, a, M, C, S, st, p->lo_elems); CNT();
    for (int l = 0; l < c.num_layers; ++l) {
      const std::string pre = "l" + std::to_string(l) + ".";
      GemmOp oq = p->op_qkv[l], oo = p->op_o[l], o1 = p->op_ffn1[l], o2 = p->op_ffn2[l];
      float* h_in = h; float* h_mid = h; float* h_out = h;
      __nv_bfloat16* a1 = a; __nv_bfloat16* a2 = a; __nv_bfloat16* a_next = a;
      float* probs = nullptr;
      __nv_bfloat16* hid_pre = nullptr;
      if (save) {
        h_in = save->h(p->ws, 2 * l); h_mid = save->h(p->ws, 2 * l + 1); h_out = save->h(p->ws, 2 * l + 2);
        a1 = save->a1(p->ws, l); a2 = save->a2(p->ws, l);
        a_next = (l + 1 < c.num_layers) ? save->a1(p->ws, l + 1) : save->a_post(p->ws);
        qkv = save->qkv(p->ws, l); o = save->o(p->ws, l); hidden = save->hidden(p->ws, l);
        hid_pre = save->hidden_pre(p->ws, l); probs = save->probs(p->ws, l);
        if (!retarget_a(&oq, a1, p->Mp) || !retarget_a(&oo, o, p->Mp) || !retarget_a(&o1, a2, p->Mp) ||
            !retarget_a(&o2, hidden, p->Mp)) return SMD_ERR_CUDA;
      }
      GemmEpilogue e = epi();
      if (!save && p->op_attn[l].ok && p->lo_bytes == 0) {
        // QKV GEMM -> attention -> out-projection + residual + LayerNorm in ONE launch; q / k / v stay on chip
        AttnBlockArgs aa;
        aa.b_qkv = p->P(params, pre + "attn.qkv.bias"); aa.b_o = p->P(params, pre + "attn.out.bias");
        aa.residual = h_in; aa.out_f32 = h_mid;
        aa.ln_gamma = p->P(params, pre + "ln2.scale"); aa.ln_beta = p->P(params, pre + "ln2.bias");
        aa.out_bf16 = a2;
        aa.M = M; aa.H = c.num_heads;
        SMD_CUDA(launch_attn_block(p->op_attn[l], aa, st));
      } else {
      e.bias = p->P(params, pre + "attn.qkv.bias");
      e.out_f32 = qkv; e.ld_f32 = 3 * kE;
      SMD_CUDA(gemm(p, oq, M, e, st));
      launch_attention(qkv, o, probs, batch, c.num_heads, st, p->lo_elems); CNT();
      e = epi();
      e.bias = p->P(params, pre + "attn.out.bias");
      e.residual = h_in; e.ld_res = kE;
      e.out_f32 = h_mid; e.ld_f32 = kE;
      e.out_bf16 = a2; e.ld_bf16 = kE;
      e.ln_gamma = p->P(params, pre + "ln2.scale"); e.ln_beta = p->P(params, pre + "ln2.bias");
      SMD_CUDA(gemm(p, oo, M, e, st));
      }
      const std::string nl = (l + 1 < c.num_layers) ? ("l" + std::to_string(l + 1) + ".ln1.") : std::string("post_ln.");
      // worth it once the token count fills the machine; training keeps the two-GEMM path: it has to write the hidden
      // activations anyway
      if (!save && M >= 32 * 256 && p->op_ffn[l].ok && p->lo_bytes == 0) {
        // FFN up + GELU + FFN down + residual + next LayerNorm in one launch; the hidden activation stays on chip
        FfnFusedArgs fa;
        fa.b1 = p->P(params, pre + "ffn1.bias"); fa.b2 = p->P(params, pre + "ffn2.bias");
        fa.residual = h_mid; fa.out_f32 = h_out;
        fa.ln_gamma = p->P(params, nl + "scale"); fa.ln_beta = p->P(params, nl + "bias");
        fa.out_bf16 = a_next;
        fa.M = M; fa.Md = Md;
        SMD_CUDA(launch_ffn_fused(p->op_ffn[l], fa, st));
        continue;
      }
      e = epi();
      e.bias = p->P(params, pre + "ffn1.bias");
      e.out_bf16 = hidden; e.ld_bf16 = Md; e.act = ACT_GELU_TANH;
      e.out_bf16_pre = hid_pre;
      SMD_CUDA(gemm(p, o1, M, e, st));
      e = epi();
      e.bias = p->P(params, pre + "ffn2.bias");
      e.residual = h_mid; e.ld_res = kE;
      e.out_f32 = h_out; e.ld_f32 = kE;
      e.out_bf16 = a_next; e.ld_bf16 = kE;
      e.ln_gamma = p->P(params, nl + "scale"); e.ln_beta = p->P(params, nl + "bias");
      SMD_CUDA(gemm(p, o2, M, e, st));
    }
    GemmEpilogue e = epi();
    e.bias = p->P(params, "post.bias");
    e.out_f32 = u0; e.ld_f32 = Md;
    e.row_stats = stats;
    GemmOp op = p->op_post;
    if (save) { if (!retarget_a(&op, save->a_post(p->ws), p->Mp)) return SMD_ERR_CUDA; }
    SMD_CUDA(gemm(p, op, M, e, st, 0));
  } else {
    __nv_bfloat16* xb = p->buf<__nv_bfloat16>("xb");
    const int Cp = (C + 63) / 64 * 64;
    if (Cp != C) { set_error("DenseDDPM on the CUDA path needs channels % 64 == 0"); return SMD_ERR_INVALID; }
    launch_cast_bf16(x, xb, static_cast<size_t>(M) * C, st, p->lo_elems); CNT();
    GemmEpilogue e = epi();
    e.bias = p->P(params, "in.bias");
    e.out_f32 = u0; e.ld_f32 = Md;
    e.row_stats = stats;
    SMD_CUDA(gemm(p, p->op_in, M, e, st, 0));
  }
  SMD_LAUNCH_CHECK("trunk");
  if (film_on_side) SMD_CUDA(cudaStreamWaitEvent(st, p->ev_film, 0));
  rc = run_tail(p, params, M, S, t_broadcast, y, st, save);
  if (rc) return rc;
  if (c.arch == SMD_ARCH_DENSE_NCSN && !raw_out) {   // models/ncsn.py:97: output = x / sigmas
    launch_scale_rows(y, t, t_broadcast, batch, S * C, st); CNT();
    SMD_LAUNCH_CHECK("ncsn output scale");
  }
  return SMD_OK;
}

// host threefry (same block function as the device one)
static inline uint32_t h_rotl(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
static void h_threefry(uint32_t k0, uint32_t k1, uint32_t& x0, uint32_t& x1) {
  static const int R[2][4] = {{13, 15, 26, 6}, {17, 29, 16, 24}};
  const uint32_t ks[3] = {k0, k1, k0 ^ k1 ^ 0x1BD11BDAu};
  x0 += ks[0]; x1 += ks[1];
  for (int i = 0; i < 5; ++i) {
    for (int j = 0; j < 4; ++j) { x0 += x1; x1 = h_rotl(x1, R[i & 1][j]); x1 ^= x0; }
    x0 += ks[(i + 1) % 3];
    x1 += ks[(i + 2) % 3] + static_cast<uint32_t>(i + 1);
  }
}
static void h_split(const uint32_t key[2], int num, uint32_t* out) {
  // jax.random.split: threefry_2x32(key, iota(2*num)).reshape(num, 2); counters split in halves
  std::vector<uint32_t> flat(2 * num);
  for (int i = 0; i < num; ++i) {
    uint32_t a = static_cast<uint32_t>(i), b = static_cast<uint32_t>(num + i);
    h_threefry(key[0], key[1], a, b);
    flat[i] = a; flat[num + i] = b;
  }
  memcpy(out, flat.data(), sizeof(uint32_t) * 2 * num);
}

// labels = jax.random.randint(label_key, (B,), minlabel, T + minlabel); used = max(lo, u*(hi-lo)+lo) with
// lo = abar[l-1], hi = abar[l]   (utils/losses.py:272-286; minlabel = int(continuous_noise), and for label 0 the
// index -1 wraps to the last entry exactly as jnp indexing does).  Rows [first, first + n) of a GLOBAL batch of B
// examples: threefry is counter based, so a data-parallel rank generates exactly its slice of the global stream.
// (shared with denoising score matching, utils/losses.py:146-160: table = sigmas, span = L - int(continuous), and the
// uniform draw only when continuous -- otherwise used = table[label])
__global__ void draws_kernel(uint32_t lk0, uint32_t lk1, uint32_t nk0, uint32_t nk1, const float* __restrict__ abar,
                             int wrap_index, int span_i, int B, int first, int n, int minlabel, int continuous,
                             float* __restrict__ used, int* __restrict__ labels) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int i = first + j;
  // randint: k1,k2 = split(key); hi,lo bits; span = T; mult = (2^16 % span)^2 % span
  uint32_t a0 = 0, b0 = 2, a1 = 1, b1 = 3;
  threefry2x32(lk0, lk1, a0, b0);
  threefry2x32(lk0, lk1, a1, b1);
  const uint32_t k1_0 = a0, k1_1 = a1, k2_0 = b0, k2_1 = b1;
  const uint32_t hi = jax_random_bits(k1_0, k1_1, i, B);
  const uint32_t lo = jax_random_bits(k2_0, k2_1, i, B);
  const uint32_t span = static_cast<uint32_t>(span_i);
  uint32_t mult = 65536u % span;
  mult = static_cast<uint32_t>((static_cast<uint64_t>(mult) * mult) % span);
  const uint32_t off = static_cast<uint32_t>((static_cast<uint64_t>(hi % span) * mult + (lo % span)) % span);
  const int label = minlabel + static_cast<int>(off);
  if (labels) labels[j] = label;
  if (!continuous) { used[j] = abar[label]; return; }
  const float minv = abar[label > 0 ? label - 1 : wrap_index], maxv = abar[label];
  const uint32_t bits = jax_random_bits(nk0, nk1, i, B);
  const float u01 = __uint_as_float((bits >> 9) | 0x3F800000u) - 1.0f;
  used[j] = fmaxf(minv, __fadd_rn(__fmul_rn(u01, __fsub_rn(maxv, minv)), minv));
}

// jax.random.uniform (0.2.8): f = bitcast((bits >> 9) | 0x3F800000) - 1; max(minval, f * (maxval - minval) + minval)
__global__ void threefry_uniform_kernel(uint32_t k0, uint32_t k1, float* out, uint32_t n, float minv, float maxv) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t bits = jax_random_bits(k0, k1, i, n);
    const float u01 = __uint_as_float((bits >> 9) | 0x3F800000u) - 1.0f;
    out[i] = fmaxf(minv, __fadd_rn(__fmul_rn(u01, __fsub_rn(maxv, minv)), minv));
  }
}

// out[j] = element (first + j) of jax.random.normal(key, (total,))
__global__ void threefry_normal_kernel(uint32_t k0, uint32_t k1, float* out, uint32_t n, uint32_t first, uint32_t total) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    out[i] = jax_normal_from_bits(jax_random_bits(k0, k1, first + i, total));
}

void add_pack_job_ptr(smd_plan* p, const std::string& src, void* dst, int K, int N, int mode, int ld) {
  PackJob j;
  j.src_off = p->off.at(src); j.dst = dst; j.K = K; j.N = N; j.mode = mode; j.ld = ld;
  j.tiles_n = (N + 63) / 64;
  j.tile0 = p->pack_tiles;
  p->pack_tiles += ((K + 63) / 64) * j.tiles_n;
  p->pack_jobs.push_back(j);
}

// the only repack job left: out.kernel -> zero-padded [Md][Cp] copy (everything else is read from the bf16 shadow)
static int build_pack_jobs(smd_plan* plan) {
  const smd_config& c = plan->cfg;
  const int Md = c.mlp_dims, C = c.channels, Cp = (C + 63) / 64 * 64;
  plan->pack_jobs.clear();
  plan->pack_tiles = 0;
  add_pack_job_ptr(plan, "out.kernel", plan->buf<void>("w.out_pad"), Md, C, 1, Cp);
  SMD_CUDA(cudaMemcpy(plan->buf<PackJob>("packjobs"), plan->pack_jobs.data(), plan->pack_jobs.size() * sizeof(PackJob),
                      cudaMemcpyHostToDevice));
  std::vector<int> bm(static_cast<size_t>(plan->pack_tiles) * 2);
  for (size_t j = 0; j < plan->pack_jobs.size(); ++j) {
    const PackJob& pj = plan->pack_jobs[j];
    const int nt = ((pj.K + 63) / 64) * pj.tiles_n;
    for (int t = 0; t < nt; ++t) { bm[2 * (pj.tile0 + t)] = static_cast<int>(j); bm[2 * (pj.tile0 + t) + 1] = t; }
  }
  SMD_CUDA(cudaMemcpy(plan->buf<int>("packmap"), bm.data(), bm.size() * sizeof(int), cudaMemcpyHostToDevice));
  return SMD_OK;
}

}  // namespace smd

// =====================================================================================================
// C ABI
// =====================================================================================================
extern "C" {

const char* smd_last_error(void) { return get_error(); }
int smd_version(void) { return 100; }
long long smd_launch_count(void) { return g_launches.load(); }

int smd_plan_create(const smd_config* cfg, smd_plan** out) {
  if (!cfg || !out) { set_error("null argument"); return SMD_ERR_INVALID; }
  smd_config c = *cfg;
  if (c.arch != SMD_ARCH_TRANSFORMER_DDPM && c.arch != SMD_ARCH_DENSE_DDPM && c.arch != SMD_ARCH_DENSE_NCSN) { set_error("unknown arch"); return SMD_ERR_INVALID; }
  if (c.cta_group == 0) c.cta_group = 1;
  if (c.cta_group != 1 && c.cta_group != 2) { set_error("cta_group must be 1 or 2"); return SMD_ERR_INVALID; }
  if (c.mlp_dims < 256 || c.mlp_dims % 256 != 0 || c.mlp_dims > 4096) { set_error("mlp_dims must be a multiple of 256 in [256, 4096]"); return SMD_ERR_INVALID; }
  if (c.channels < 1 || c.max_batch < 1 || c.num_layers < 1) { set_error("bad sizes"); return SMD_ERR_INVALID; }
  if (c.precision != SMD_PRECISION_BF16 && c.precision != SMD_PRECISION_BF16X3) { set_error("unknown precision"); return SMD_ERR_INVALID; }
  if (c.precision == SMD_PRECISION_BF16X3 && c.training) { set_error("precision bf16x3 covers the forward pass / sampler only (training = 0)"); return SMD_ERR_INVALID; }
  if (c.arch == SMD_ARCH_TRANSFORMER_DDPM) {
    if (c.seq_len != 32) { set_error("TransformerDDPM CUDA path supports seq_len == 32 only (all reference configs)"); return SMD_ERR_INVALID; }
    if (c.num_heads != 4 && c.num_heads != 8 && c.num_heads != 16 && c.num_heads != 32) { set_error("num_heads must be 4, 8, 16 or 32"); return SMD_ERR_INVALID; }
    if (c.num_mlp_layers < 1) { set_error("num_mlp_layers must be >= 1"); return SMD_ERR_INVALID; }
  } else {
    c.seq_len = 1;
  }
  smd_plan* p = new smd_plan();
  p->cfg = c;
  p->Mp = (c.max_batch * c.seq_len + 255) / 256 * 256;
  build_layout(p);
  build_workspace(p);
  *out = p;
  return SMD_OK;
}

void smd_plan_destroy(smd_plan* plan) {
  if (!plan) return;
  if (plan->graph_exec) cudaGraphExecDestroy(plan->graph_exec);
  if (plan->tg_exec) cudaGraphExecDestroy(plan->tg_exec);
  if (plan->evx_join) cudaEventDestroy(plan->evx_join);
  if (plan->ev_gz) cudaEventDestroy(plan->ev_gz);
  if (plan->own_event) cudaEventDestroy(plan->own_event);
  if (plan->ev_fork) cudaEventDestroy(plan->ev_fork);
  if (plan->ev_film) cudaEventDestroy(plan->ev_film);
  if (plan->ev_dss) cudaEventDestroy(plan->ev_dss);
  if (plan->ev_join) cudaEventDestroy(plan->ev_join);
  if (plan->ev_dw) cudaEventDestroy(plan->ev_dw);
  if (plan->ev_dwjoin) cudaEventDestroy(plan->ev_dwjoin);
  if (plan->ev_tail) cudaEventDestroy(plan->ev_tail);
  if (plan->ev_dwtail) cudaEventDestroy(plan->ev_dwtail);
  if (plan->dw_stream) cudaStreamDestroy(plan->dw_stream);
  if (plan->side_stream) cudaStreamDestroy(plan->side_stream);
  if (plan->own_stream) cudaStreamDestroy(plan->own_stream);
  delete plan;
}

int smd_num_tensors(const smd_plan* plan) { return static_cast<int>(plan->tensors.size()); }
long long smd_arena_floats(const smd_plan* plan) { return plan->arena; }
int smd_tensor_info(const smd_plan* plan, int index, char* name, int name_cap, long long* offset, int* shape4,
                    int* ndim) {
  if (index < 0 || index >= static_cast<int>(plan->tensors.size())) { set_error("tensor index out of range"); return SMD_ERR_INVALID; }
  const TensorInfo& t = plan->tensors[index];
  if (name && name_cap > 0) { strncpy(name, t.name.c_str(), name_cap - 1); name[name_cap - 1] = 0; }
  if (offset) *offset = t.offset;
  if (shape4) for (int i = 0; i < 4; ++i) shape4[i] = t.shape[i];
  if (ndim) *ndim = t.ndim;
  return SMD_OK;
}
size_t smd_workspace_bytes(const smd_plan* plan) { return plan->ws_bytes; }

int smd_bind_workspace(smd_plan* plan, void* workspace, size_t bytes) {
  if (!workspace || bytes < plan->ws_bytes) { set_error("workspace too small"); return SMD_ERR_INVALID; }
  if (reinterpret_cast<uintptr_t>(workspace) % 1024 != 0) { set_error("workspace must be 1024-byte aligned"); return SMD_ERR_INVALID; }
  plan->ws = static_cast<uint8_t*>(workspace);
  SMD_CUDA(cudaMemset(workspace, 0, plan->ws_bytes));  // padded rows / columns of every operand start finite
  plan->packed = false;
  plan->sampler_ready = false;
  if (plan->tg_exec) { cudaGraphExecDestroy(plan->tg_exec); plan->tg_exec = nullptr; }
  plan->tg_valid = false; plan->tg_warm = false;
  int rc = build_ops(plan);
  if (rc) return rc;
  float f[64];
  host_freqs(f);
  SMD_CUDA(cudaMemcpy(plan->buf<float>("freqs"), f, sizeof(f), cudaMemcpyHostToDevice));
  // positional table (models/shared.py:33-48), float32 like jnp
  std::vector<float> pe(static_cast<size_t>(plan->cfg.seq_len) * kE);
  for (int s = 0; s < plan->cfg.seq_len; ++s)
    for (int j = 0; j < 64; ++j) {
      const float arg = static_cast<float>(s) * f[j];
      pe[s * kE + j] = sinf(arg);
      pe[s * kE + 64 + j] = cosf(arg);
    }
  SMD_CUDA(cudaMemcpy(plan->buf<float>("posenc"), pe.data(), pe.size() * 4, cudaMemcpyHostToDevice));
  if (plan->cfg.training) { rc = train_bind(plan); if (rc) return rc; }
  rc = build_pack_jobs(plan);
  if (rc) return rc;
  return SMD_OK;
}

static int refresh_operands(smd_plan* plan, const float* params, bool shadow_is_fresh, cudaStream_t st) {
  if (!plan->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (!shadow_is_fresh) {
    launch_cast_bf16(params, plan->buf<__nv_bfloat16>("wshadow"), static_cast<size_t>(plan->arena), st, plan->lo_elems); CNT();
  }
  launch_pack_multi(params, plan->buf<PackJob>("packjobs"), plan->buf<void>("packmap"), plan->pack_tiles, st, plan->lo_elems); CNT();
  SMD_LAUNCH_CHECK("pack_weights");
  plan->packed = true;
  plan->film_tab_ready = false;   // parameters changed
  return SMD_OK;
}

int smd_pack_weights(smd_plan* plan, const float* params, smd_stream_t stream) {
  return refresh_operands(plan, params, false, static_cast<cudaStream_t>(stream));
}

int smd_pack_weights_after_adam(smd_plan* plan, const float* params, smd_stream_t stream) {
  return refresh_operands(plan, params, true, static_cast<cudaStream_t>(stream));
}

void* smd_shadow_arena(smd_plan* plan) { return plan->ws ? plan->buf<void>("wshadow") : nullptr; }

int smd_grads_tail_range(const smd_plan* plan, long long* first_float, long long* num_floats) {
  if (!plan || !first_float || !num_floats) { set_error("null argument"); return SMD_ERR_INVALID; }
  auto it = plan->off.find("k0.film.d1.kernel");   // first tensor of the FiLM'd tail; out_ln / out follow it
  if (it == plan->off.end()) { set_error("plan has no FiLM'd residual tail"); return SMD_ERR_STATE; }
  *first_float = static_cast<long long>(it->second);
  *num_floats = static_cast<long long>(plan->arena) - *first_float;
  return SMD_OK;
}

int smd_wait_tail_grads(smd_plan* plan, smd_stream_t stream) {
  if (!plan || !plan->ev_tail || !plan->evx_join) { set_error("no smd_ddpm_grads call has been enqueued on this plan"); return SMD_ERR_STATE; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // (recorded by plain cudaEventRecord calls, or -- graph replay -- by external event-record nodes of the graph)
  SMD_CUDA(cudaStreamWaitEvent(st, plan->ev_tail, 0));   // tail + output-layer gradients (caller's stream)
  SMD_CUDA(cudaStreamWaitEvent(st, plan->evx_join, 0));  // FiLM generator gradients (side stream)
  SMD_CUDA(cudaStreamWaitEvent(st, plan->ev_dwtail, 0)); // res-block weight gradients (weight-gradient stream)
  return SMD_OK;
}

int smd_forward(smd_plan* plan, const float* params, const float* x, const float* t, int t_broadcast, int batch,
                float* y, smd_stream_t stream) {
  return run_forward(plan, params, x, t, t_broadcast, batch, y, static_cast<cudaStream_t>(stream), nullptr);
}

int smd_ddpm_loss(smd_plan* plan, const float* params, const float* x0, const float* used_alpha, const float* eps,
                  int batch, float* loss_per_example, float* pred_or_null, smd_stream_t stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!plan->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (batch < 1 || batch > plan->cfg.max_batch) { set_error("batch out of range"); return SMD_ERR_INVALID; }
  const int per = plan->cfg.seq_len * plan->cfg.channels;
  float* xt = plan->buf<float>("xt");
  float* cond = plan->buf<float>("tvec");
  float* pred = pred_or_null ? pred_or_null : plan->buf<float>("eps_hat");
  launch_q_sample(x0, eps, used_alpha, xt, cond, batch, per, st); CNT();
  int rc = run_forward(plan, params, xt, cond, 0, batch, pred, st, nullptr);
  if (rc) return rc;
  launch_ddpm_loss(eps, pred, loss_per_example, nullptr, 0.f, batch, per, st); CNT();
  SMD_LAUNCH_CHECK("ddpm_loss");
  return SMD_OK;
}

int smd_dsm_loss(smd_plan* plan, const float* params, const float* x0, const float* used_sigma, const float* eps,
                 int batch, float* loss_per_example, float* pred_or_null, smd_stream_t stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (plan->cfg.arch != SMD_ARCH_DENSE_NCSN) { set_error("smd_dsm_loss needs a score network (SMD_ARCH_DENSE_NCSN)"); return SMD_ERR_INVALID; }
  if (!plan->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (batch < 1 || batch > plan->cfg.max_batch) { set_error("batch out of range"); return SMD_ERR_INVALID; }
  const int per = plan->cfg.seq_len * plan->cfg.channels;
  float* xt = plan->buf<float>("xt");
  float* cond = plan->buf<float>("tvec");
  float* pred = pred_or_null ? pred_or_null : plan->buf<float>("eps_hat");
  launch_q_sample(x0, eps, used_sigma, xt, cond, batch, per, st, nullptr, 1); CNT();
  int rc = run_forward(plan, params, xt, cond, 0, batch, pred, st, nullptr);
  if (rc) return rc;
  launch_ddpm_loss(eps, pred, loss_per_example, nullptr, 0.f, batch, per, st, used_sigma); CNT();
  SMD_LAUNCH_CHECK("dsm_loss");
  return SMD_OK;
}

int smd_dsm_setup(smd_plan* plan, const float* host_sigmas, int L, smd_stream_t stream) {
  if (!plan->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (L < 2 || L > kMaxT) { set_error("schedule length out of range"); return SMD_ERR_INVALID; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SMD_CUDA(cudaMemcpyAsync(plan->buf<float>("sigmas"), host_sigmas, static_cast<size_t>(L) * 4, cudaMemcpyHostToDevice, st));
  SMD_CUDA(cudaStreamSynchronize(st));
  plan->L_dsm = L;
  return SMD_OK;
}

int smd_dsm_draws(smd_plan* plan, const uint32_t host_key[2], int global_batch, int first_row, int batch,
                  int continuous_noise, float* used_sigma, float* eps, int* labels_or_null, smd_stream_t stream) {
  if (plan->L_dsm <= 0) { set_error("smd_dsm_setup has not been called"); return SMD_ERR_STATE; }
  if (batch < 1 || first_row < 0 || global_batch < first_row + batch) { set_error("batch out of range"); return SMD_ERR_INVALID; }
  const long long per = static_cast<long long>(plan->cfg.seq_len) * plan->cfg.channels;
  if (static_cast<long long>(global_batch) * per > 0xFFFFFFFFll) { set_error("global batch too large"); return SMD_ERR_INVALID; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int L = plan->L_dsm, cn = continuous_noise ? 1 : 0;
  uint32_t k3[6], k2[4] = {0, 0, 0, 0};
  h_split(host_key, 3, k3);               // rng, label_rng, sample_rng          (utils/losses.py:146)
  if (cn) { const uint32_t rng[2] = {k3[0], k3[1]}; h_split(rng, 2, k2); }        // rng, noise_rng (:152-153)
  // labels = randint(label_rng, minval = int(continuous), maxval = L): span L - cn; table index label - 1 wraps for 0
  draws_kernel<<<(batch + 127) / 128, 128, 0, st>>>(k3[2], k3[3], k2[2], k2[3], plan->buf<float>("sigmas"), L - 1, L - cn,
                                                    global_batch, first_row, batch, cn, cn, used_sigma, labels_or_null);
  CNT();
  const long long n = static_cast<long long>(batch) * per;
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > 148 * 8) blocks = 148 * 8;
  threefry_normal_kernel<<<blocks, 256, 0, st>>>(k3[4], k3[5], eps, static_cast<uint32_t>(n),
                                                 static_cast<uint32_t>(first_row * per),
                                                 static_cast<uint32_t>(global_batch * per));
  CNT();
  SMD_LAUNCH_CHECK("dsm_draws");
  return SMD_OK;
}

int smd_langevin_step(smd_plan* plan, const float* x, const float* grad, int n, float alpha, float noise_coef,
                      const uint32_t step_key[2], const float* z, const float* infill_x, const float* infill_mask,
                      float infill_sigma, const uint32_t infill_key[2], const float* infill_z, float* x_next,
                      float* collection_slot, float* metrics4, smd_stream_t stream) {
  if (!plan || n < 1) { set_error("bad arguments"); return SMD_ERR_INVALID; }
  LangevinStepArgs a;
  memset(&a, 0, sizeof(a));
  a.x = x; a.grad = grad; a.z = z;
  if (step_key) { a.key0 = step_key[0]; a.key1 = step_key[1]; }
  if (infill_key) { a.ikey0 = infill_key[0]; a.ikey1 = infill_key[1]; }
  a.alpha = alpha; a.noise_coef = noise_coef; a.infill_sigma = infill_sigma;
  a.infill_x = infill_x; a.infill_mask = infill_mask; a.infill_z = infill_z;
  a.x_next = x_next; a.collection_slot = collection_slot; a.metrics = metrics4;
  a.N = n; a.S = plan->cfg.seq_len; a.C = plan->cfg.channels;
  if (plan->cfg.arch != SMD_ARCH_TRANSFORMER_DDPM) { a.S = plan->cfg.channels; a.C = 1; }   // (N, D) states: axis 1 = D
  launch_langevin_step(a, static_cast<cudaStream_t>(stream)); CNT();
  SMD_LAUNCH_CHECK("langevin_step");
  return SMD_OK;
}

int smd_objective_setup(smd_plan* plan, const float* host_betas, int T, smd_stream_t stream) {
  if (!plan->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (T < 1 || T > kMaxT) { set_error("T out of range"); return SMD_ERR_INVALID; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  std::vector<float> ap(T + 1);
  ap[0] = 1.0f;
  float run = 1.0f;
  for (int i = 0; i < T; ++i) { const float a = 1.0f - host_betas[i]; run = (i == 0) ? a : run * a; ap[i + 1] = run; }
  SMD_CUDA(cudaMemcpyAsync(plan->buf<float>("abar"), ap.data(), ap.size() * 4, cudaMemcpyHostToDevice, st));
  SMD_CUDA(cudaStreamSynchronize(st));
  plan->T_obj = T;
  return SMD_OK;
}

int smd_ddpm_draws_sharded(smd_plan* plan, const uint32_t host_key[2], int global_batch, int first_row, int batch,
                           int continuous_noise, float* used_alpha, float* eps, int* labels_or_null,
                           smd_stream_t stream) {
  if (plan->T_obj <= 0) { set_error("smd_objective_setup has not been called"); return SMD_ERR_STATE; }
  if (batch < 1 || first_row < 0 || global_batch < first_row + batch) { set_error("batch out of range"); return SMD_ERR_INVALID; }
  const long long per = static_cast<long long>(plan->cfg.seq_len) * plan->cfg.channels;
  if (static_cast<long long>(global_batch) * per > 0xFFFFFFFFll) { set_error("global batch too large"); return SMD_ERR_INVALID; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint32_t k3[6], k2[4];
  h_split(host_key, 3, k3);               // rng, label_rng, sample_rng
  const uint32_t rng[2] = {k3[0], k3[1]};
  h_split(rng, 2, k2);                    // rng, noise_rng
  // ddpm: labels = randint(int(continuous), T + int(continuous)) -> span T; alphas_prod has T + 1 entries (leading 1)
  draws_kernel<<<(batch + 127) / 128, 128, 0, st>>>(k3[2], k3[3], k2[2], k2[3], plan->buf<float>("abar"), plan->T_obj,
                                                    plan->T_obj, global_batch, first_row, batch, continuous_noise ? 1 : 0, 1,
                                                    used_alpha, labels_or_null);
  CNT();
  const long long n = static_cast<long long>(batch) * per;
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > 148 * 8) blocks = 148 * 8;
  threefry_normal_kernel<<<blocks, 256, 0, st>>>(k3[4], k3[5], eps, static_cast<uint32_t>(n),
                                                 static_cast<uint32_t>(first_row * per),
                                                 static_cast<uint32_t>(global_batch * per));
  CNT();
  SMD_LAUNCH_CHECK("ddpm_draws");
  return SMD_OK;
}

int smd_ddpm_draws(smd_plan* plan, const uint32_t host_key[2], int batch, float* used_alpha, float* eps,
                   int* labels_or_null, smd_stream_t stream) {
  return smd_ddpm_draws_sharded(plan, host_key, batch, 0, batch, 1, used_alpha, eps, labels_or_null, stream);
}

int smd_sampler_setup(smd_plan* plan, const float* host_betas, int T, const uint32_t host_key[2],
                      smd_stream_t stream) {
  if (!plan->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (T < 1 || T > kMaxT) { set_error("T out of range"); return SMD_ERR_INVALID; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // utils/ebm_utils.py:315-318, 332-357, 363-364 -- float32, same operation order
  std::vector<float> coef(static_cast<size_t>(T) * 8);
  std::vector<float> ap(T), app(T), al(T);
  float run = 1.0f;
  for (int i = 0; i < T; ++i) {
    al[i] = 1.0f - host_betas[i];
    run = (i == 0) ? al[0] : run * al[i];
    ap[i] = run;
    app[i] = (i == 0) ? 1.0f : ap[i - 1];
  }
  for (int i = 0; i < T; ++i) {
    const float beta = host_betas[i];
    const float sqrt_recip = sqrtf(1.0f / ap[i]);
    const float sqrt_m1 = sqrtf(1.0f - ap[i]) * sqrt_recip;
    const float mu1 = beta * sqrtf(app[i]) / (1.0f - ap[i]);
    const float mu2 = (1.0f - app[i]) * sqrtf(al[i]) / (1.0f - ap[i]);
    const float var = beta * (1.0f - app[i]) / (1.0f - ap[i]);
    const float logv = logf(fmaxf(var, 1e-20f));
    const float sigma = expf(0.5f * logv);
    float* c = &coef[static_cast<size_t>(i) * 8];
    c[0] = sqrt_recip; c[1] = sqrt_m1; c[2] = mu1; c[3] = mu2; c[4] = sigma;
    c[5] = sqrtf(ap[i]); c[6] = sqrtf(1.0f - ap[i]); c[7] = ap[i];
  }
  // keys: per scan step (t = T-1 .. 0): rng,key = split(rng); rng,infill = split(rng); rng,noise = split(rng)
  std::vector<uint32_t> keys(static_cast<size_t>(T) * 4);
  uint32_t rng[2] = {host_key[0], host_key[1]};
  for (int t = T - 1; t >= 0; --t) {
    uint32_t o[4];
    h_split(rng, 2, o); rng[0] = o[0]; rng[1] = o[1];
    h_split(rng, 2, o); rng[0] = o[0]; rng[1] = o[1];
    keys[4 * t + 2] = o[2]; keys[4 * t + 3] = o[3];
    h_split(rng, 2, o); rng[0] = o[0]; rng[1] = o[1];
    keys[4 * t + 0] = o[2]; keys[4 * t + 1] = o[3];
  }
  // collection slots (utils/ebm_utils.py:320-325, 387-394): collection_idx = linspace(1, T, 40).astype(int32)
  std::vector<int> slots(T, -1);
  int idx_tab[40];
  for (int j = 0; j < 40; ++j) {
    const float v = (40 > 1) ? (1.0f + static_cast<float>(j) * (static_cast<float>(T - 1) / 39.0f)) : 1.0f;
    idx_tab[j] = (j == 39) ? T : static_cast<int>(v);
  }
  for (int t = 0; t < T; ++t) {
    const int image_idx = T - t + 1;
    int sum = 0; bool any = false;
    for (int j = 0; j < 40; ++j) if (idx_tab[j] == image_idx) { sum += j; any = true; }
    if (any) slots[t] = sum + 1;
  }
  SMD_CUDA(cudaMemcpyAsync(plan->buf<float>("coef"), coef.data(), coef.size() * 4, cudaMemcpyHostToDevice, st));
  SMD_CUDA(cudaMemcpyAsync(plan->buf<uint32_t>("keys"), keys.data(), keys.size() * 4, cudaMemcpyHostToDevice, st));
  SMD_CUDA(cudaMemcpyAsync(plan->buf<int>("slots"), slots.data(), slots.size() * 4, cudaMemcpyHostToDevice, st));
  SMD_CUDA(cudaStreamSynchronize(st));  // host vectors go out of scope
  plan->T = T;
  plan->sampler_ready = true;
  plan->film_tab_ready = false;
  if (plan->graph_exec) { cudaGraphExecDestroy(plan->graph_exec); plan->graph_exec = nullptr; }
  return SMD_OK;
}

__global__ void gather_cond_kernel(const float* __restrict__ coef, float* __restrict__ tv, int T) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < T) tv[i] = coef[8 * i + 5];
}

// FiLM scale/shift for every step of the schedule (all samples share t, so this replaces 3K small launches per
// reverse step by one table lookup): ftab[k][t][:] = DenseFiLM_k(sqrt(alpha_bar_t))   (models/ncsn.py:44-61)
static int ensure_film_table(smd_plan* plan, const float* params, cudaStream_t st) {
  if (plan->cfg.sampler_T <= 0 || plan->T > plan->cfg.sampler_T) return SMD_OK;   // per-step generator instead
  if (plan->film_tab_ready && plan->film_tab_params == params) return SMD_OK;
  const int T = plan->T, Md = plan->cfg.mlp_dims;
  float* tv = plan->buf<float>("ftab.t");
  float* enc = plan->buf<float>("ftab.enc");
  float* e1 = plan->buf<float>("ftab.e1");
  float* e2 = plan->buf<float>("ftab.e2");
  float* tab = plan->buf<float>("ftab");
  gather_cond_kernel<<<(T + 255) / 256, 256, 0, st>>>(plan->buf<float>("coef"), tv, T); CNT();
  launch_noise_encoding(tv, plan->buf<float>("freqs"), enc, T, st); CNT();
  for (int k = 0; k < plan->K; ++k) {
    const std::string pre = "k" + std::to_string(k) + ".film.";
    launch_small_linear(enc, plan->P(params, pre + "d1.kernel"), plan->P(params, pre + "d1.bias"), e1, T, kFilmEmb, kFilmHid, 2, st); CNT();
    launch_small_linear(e1, plan->P(params, pre + "d2.kernel"), plan->P(params, pre + "d2.bias"), e2, T, kFilmHid, kFilmHid, 0, st); CNT();
    launch_small_linear(e2, plan->P(params, pre + "ss.kernel"), plan->P(params, pre + "ss.bias"),
                        tab + static_cast<size_t>(k) * T * 2 * Md, T, kFilmHid, 2 * Md, 0, st); CNT();
  }
  SMD_LAUNCH_CHECK("film table");
  plan->film_tab_ready = true;
  plan->film_tab_params = params;
  return SMD_OK;
}

// one reverse step; t < 0 means "read t from the device scalar t_ptr" (graph replay)
static int reverse_step_impl(smd_plan* plan, const float* params, const float* x, int n, int t, const float* z,
                             const float* infill_x, const float* infill_mask, const float* infill_z, float* x_next,
                             float* eps_hat, float* collection, float* metrics, cudaStream_t st) {
  float* tvec = plan->buf<float>("tvec");
  int* t_ptr = plan->buf<int>("t_ptr");
  const float* coef = plan->buf<float>("coef");
  const bool use_tab = plan->film_tab_ready && plan->film_tab_params == params;
  if (use_tab) {
    plan->film_tab_on = true;
    plan->film_row = (t >= 0) ? t : 0;
    plan->film_row_dev = (t >= 0) ? nullptr : t_ptr;
  } else if (t >= 0) {
    // conditioning value sqrt(alpha_prod_t), shared by every sample (utils/ebm_utils.py:367-369)
    SMD_CUDA(cudaMemcpyAsync(tvec, coef + 8 * t + 5, 4, cudaMemcpyDeviceToDevice, st));
  } else {
    launch_fill_cond(coef, t_ptr, tvec, 1, st); CNT();
  }
  float* eh = eps_hat ? eps_hat : plan->buf<float>("eps_hat");
  int rc = run_forward(plan, params, x, tvec, 1, n, eh, st, nullptr);
  plan->film_tab_on = false;
  plan->film_row_dev = nullptr;
  if (rc) return rc;
  ReverseStepArgs a;
  memset(&a, 0, sizeof(a));
  a.x = x; a.eps_hat = eh; a.z = z;
  a.key_tab = plan->buf<uint32_t>("keys");
  a.coef = coef;
  a.slot_tab = plan->buf<int>("slots");
  a.t_ptr = (t >= 0) ? nullptr : t_ptr;
  a.t = t;
  a.infill_x = infill_x; a.infill_mask = infill_mask; a.infill_z = infill_z;
  a.x_next = x_next; a.collection = collection; a.metrics = metrics;
  a.N = n; a.S = plan->cfg.seq_len; a.C = plan->cfg.channels; a.T = plan->T;
  // 2-D states (N, D) of the dense networks: the metrics' axis 1 (utils/ebm_utils.py:380-384) is D itself
  if (plan->cfg.arch != SMD_ARCH_TRANSFORMER_DDPM) { a.S = plan->cfg.channels; a.C = 1; }
  if (plan->shard_total_rows > 0) {
    const long long per = static_cast<long long>(a.S) * a.C;
    a.rng_first = static_cast<uint32_t>(plan->shard_first_row * per);
    a.rng_total = static_cast<uint32_t>(plan->shard_total_rows * per);
  }
  launch_reverse_step(a, st); CNT();
  SMD_LAUNCH_CHECK("reverse_step");
  return SMD_OK;
}

int smd_sampler_set_shard(smd_plan* plan, long long first_row, long long total_rows) {
  if (!plan) { set_error("null plan"); return SMD_ERR_INVALID; }
  if (total_rows < 0 || first_row < 0 || (total_rows > 0 && first_row >= total_rows) ||
      total_rows * plan->cfg.seq_len * plan->cfg.channels > 0xFFFFFFFFll) { set_error("bad shard"); return SMD_ERR_INVALID; }
  plan->shard_first_row = first_row;
  plan->shard_total_rows = total_rows;
  if (plan->graph_exec) { cudaGraphExecDestroy(plan->graph_exec); plan->graph_exec = nullptr; }  // kernel args changed
  return SMD_OK;
}

int smd_ddpm_reverse_step(smd_plan* plan, const float* params, const float* x, int n, int t, const float* z,
                          const float* infill_x, const float* infill_mask, const float* infill_z, float* x_next,
                          float* eps_hat_or_null, float* collection, float* metrics, smd_stream_t stream) {
  if (!plan->sampler_ready) { set_error("smd_sampler_setup has not been called"); return SMD_ERR_STATE; }
  if (t < 0 || t >= plan->T) { set_error("t out of range"); return SMD_ERR_INVALID; }
  if (n < 1 || n > plan->cfg.max_batch) { set_error("n out of range"); return SMD_ERR_INVALID; }
  int rc0 = ensure_film_table(plan, params, static_cast<cudaStream_t>(stream));
  if (rc0) return rc0;
  return reverse_step_impl(plan, params, x, n, t, z, infill_x, infill_mask, infill_z, x_next, eps_hat_or_null,
                           collection, metrics, static_cast<cudaStream_t>(stream));
}

int smd_ddpm_sample(smd_plan* plan, const float* params, float* x, int n, int steps, const float* infill_x,
                    const float* infill_mask, float* collection, float* metrics, int use_graph,
                    smd_stream_t stream) {
  if (!plan->sampler_ready) { set_error("smd_sampler_setup has not been called"); return SMD_ERR_STATE; }
  if (n < 1 || n > plan->cfg.max_batch) { set_error("n out of range"); return SMD_ERR_INVALID; }
  if (steps < 1 || steps > plan->T) { set_error("steps out of range"); return SMD_ERR_INVALID; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int T = plan->T;
  if (metrics) SMD_CUDA(cudaMemsetAsync(metrics, 0, sizeof(float) * 4 * T, st));
  { int rc0 = ensure_film_table(plan, params, st); if (rc0) return rc0; }
  if (!use_graph) {
    for (int i = 0; i < steps; ++i) {
      int rc = reverse_step_impl(plan, params, x, n, T - 1 - i, nullptr, infill_x, infill_mask, nullptr, x, nullptr,
                                 collection, metrics, st);
      if (rc) return rc;
    }
    return SMD_OK;
  }
  // the legacy default stream cannot be captured: run the replay loop on a private stream ordered after `st`
  cudaStream_t cs = st;
  if (st == nullptr || st == cudaStreamLegacy || st == cudaStreamPerThread) {
    if (!plan->own_stream) {
      SMD_CUDA(cudaStreamCreateWithFlags(&plan->own_stream, cudaStreamNonBlocking));
      SMD_CUDA(cudaEventCreateWithFlags(&plan->own_event, cudaEventDisableTiming));
    }
    SMD_CUDA(cudaEventRecord(plan->own_event, st));
    SMD_CUDA(cudaStreamWaitEvent(plan->own_stream, plan->own_event, 0));
    cs = plan->own_stream;
  }
  int* t_ptr = plan->buf<int>("t_ptr");
  const int t0 = T - 1;
  SMD_CUDA(cudaMemcpyAsync(t_ptr, &t0, sizeof(int), cudaMemcpyHostToDevice, cs));
  SMD_CUDA(cudaStreamSynchronize(cs));  // t0 is a stack variable
  const bool same = plan->graph_exec && plan->graph_n == n && plan->graph_params == params && plan->graph_x == x &&
                    plan->graph_infill_x == infill_x && plan->graph_infill_mask == infill_mask &&
                    plan->graph_collection == collection && plan->graph_metrics == metrics;
  if (!same) {
    if (plan->graph_exec) { cudaGraphExecDestroy(plan->graph_exec); plan->graph_exec = nullptr; }
    cudaGraph_t graph = nullptr;
    const long long before = g_launches.load();
    SMD_CUDA(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
    int rc = reverse_step_impl(plan, params, x, n, -1, nullptr, infill_x, infill_mask, nullptr, x, nullptr,
                               collection, metrics, cs);
    if (rc == SMD_OK) { launch_step_advance(t_ptr, cs); CNT(); }
    cudaError_t ce = cudaStreamEndCapture(cs, &graph);
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (ce != cudaSuccess) { set_error(std::string("graph capture: ") + cudaGetErrorString(ce)); return SMD_ERR_CUDA; }
    plan->graph_nodes = g_launches.load() - before;
    g_launches.store(before);  // captured launches are counted per replay below
    SMD_CUDA(cudaGraphInstantiate(&plan->graph_exec, graph, 0));
    cudaGraphDestroy(graph);
    plan->graph_n = n; plan->graph_params = params; plan->graph_x = x; plan->graph_infill_x = infill_x;
    plan->graph_infill_mask = infill_mask; plan->graph_collection = collection; plan->graph_metrics = metrics;
  }
  for (int i = 0; i < steps; ++i) {
    SMD_CUDA(cudaGraphLaunch(plan->graph_exec, cs));
    g_launches.fetch_add(plan->graph_nodes, std::memory_order_relaxed);
  }
  if (cs != st) {
    SMD_CUDA(cudaEventRecord(plan->own_event, cs));
    SMD_CUDA(cudaStreamWaitEvent(st, plan->own_event, 0));
  }
  return SMD_OK;
}

int smd_threefry_normal(const uint32_t host_key[2], float* out, long long n, smd_stream_t stream) {
  if (n < 0 || n > 0xFFFFFFFFll) { set_error("n out of range"); return SMD_ERR_INVALID; }
  if (n == 0) return SMD_OK;
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > 148 * 8) blocks = 148 * 8;
  threefry_normal_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(host_key[0], host_key[1], out,
                                                                                static_cast<uint32_t>(n), 0u,
                                                                                static_cast<uint32_t>(n));
  CNT();
  SMD_LAUNCH_CHECK("threefry_normal");
  return SMD_OK;
}
int smd_threefry_normal_slice(const uint32_t host_key[2], float* out, long long n, long long first, long long total,
                              smd_stream_t stream) {
  if (n < 0 || first < 0 || first + n > total || total > 0xFFFFFFFFll) { set_error("slice out of range"); return SMD_ERR_INVALID; }
  if (n == 0) return SMD_OK;
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > 148 * 8) blocks = 148 * 8;
  threefry_normal_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(host_key[0], host_key[1], out,
                                                                                static_cast<uint32_t>(n),
                                                                                static_cast<uint32_t>(first),
                                                                                static_cast<uint32_t>(total));
  CNT();
  SMD_LAUNCH_CHECK("threefry_normal_slice");
  return SMD_OK;
}
int smd_threefry_uniform(const uint32_t host_key[2], float* out, long long n, float minval, float maxval,
                         smd_stream_t stream) {
  if (n < 0 || n > 0xFFFFFFFFll) { set_error("n out of range"); return SMD_ERR_INVALID; }
  if (n == 0) return SMD_OK;
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > 148 * 8) blocks = 148 * 8;
  threefry_uniform_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(host_key[0], host_key[1], out,
                                                                                 static_cast<uint32_t>(n), minval, maxval);
  CNT();
  SMD_LAUNCH_CHECK("threefry_uniform");
  return SMD_OK;
}
int smd_threefry_split(const uint32_t host_key[2], int num, uint32_t* host_out_keys) {
  if (num < 1) { set_error("num must be >= 1"); return SMD_ERR_INVALID; }
  h_split(host_key, num, host_out_keys);
  return SMD_OK;
}

int smd_debug_forward_save(smd_plan* plan, const float* params, const float* x, const float* t, int batch, float* y,
                           smd_stream_t stream) {
  if (!plan->cfg.training) { set_error("plan was not created with training = 1"); return SMD_ERR_STATE; }
  return run_forward(plan, params, x, t, 0, batch, y, static_cast<cudaStream_t>(stream), &plan->train);
}

int smd_debug_buffer(smd_plan* plan, const char* name, void** dev_ptr, size_t* bytes) {
  if (!plan->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  auto it = plan->ws_off.find(name);
  if (it == plan->ws_off.end()) { set_error(std::string("no workspace region named ") + name); return SMD_ERR_INVALID; }
  size_t end = plan->ws_bytes;
  for (const auto& kv : plan->ws_off) if (kv.second > it->second && kv.second < end) end = kv.second;
  if (dev_ptr) *dev_ptr = plan->ws + it->second;
  if (bytes) *bytes = end - it->second;
  return SMD_OK;
}

int smd_gemm_bf16(const void* A, const void* B, int M, int N, int K, int a_mn, int b_mn, int BN, int cta_group,
                  const float* bias, const float* residual, int act, float* out_f32, void* out_bf16,
                  float* row_stats, const float* ln_gamma, const float* ln_beta, smd_stream_t stream) {
  if (cta_group != 1 && cta_group != 2) { set_error("cta_group must be 1 or 2"); return SMD_ERR_INVALID; }
  GemmOp op;
  if (BN <= 0) BN = choose_bn(N);
  if (!make_gemm_op(&op, A, static_cast<uint64_t>(M), B, static_cast<uint64_t>(N), N, K, BN, a_mn, b_mn))
    return SMD_ERR_CUDA;
  GemmEpilogue e = epi();
  e.bias = bias; e.residual = residual; e.ld_res = N; e.act = act;
  e.out_f32 = out_f32; e.ld_f32 = N;
  e.out_bf16 = static_cast<__nv_bfloat16*>(out_bf16); e.ld_bf16 = N;
  e.row_stats = row_stats; e.ln_gamma = ln_gamma; e.ln_beta = ln_beta;
  SMD_CUDA(launch_gemm(op, M, e, static_cast<cudaStream_t>(stream)));
  SMD_LAUNCH_CHECK("gemm");
  return SMD_OK;
}

}  // extern "C"

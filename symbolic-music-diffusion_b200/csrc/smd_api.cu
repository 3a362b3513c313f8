// libsmd C ABI implementation: plan / parameter arena / workspace carving, the score-network forward,
// objective, sampler, jax-compatible RNG helpers and test hooks.  See include/smd.h.
#include "../../include/smd.h"

#include <cmath>
#include <cstdio>
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "plan.cuh"

namespace smd {

std::atomic<long long> g_launches{0};
static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
const char* get_error() { return g_err.c_str(); }

static long long add_tensor(smd_plan* p, const std::string& name, std::initializer_list<int> shape) {
  TensorInfo t;
  t.name = name;
  t.ndim = static_cast<int>(shape.size());
  int i = 0;
  for (int s : shape) t.shape[i++] = s;
  for (; i < 4; ++i) t.shape[i] = 1;
  t.offset = p->arena;
  p->arena += (t.size() + 7) / 8 * 8;  // 32-byte aligned in fp32 => 16-byte aligned in the bf16 shadow arena (TMA)
  p->tensors.push_back(t);
  return t.offset;
}
static Dense add_dense(smd_plan* p, const std::string& pre, int in, int out) {
  Dense d;
  d.kernel = add_tensor(p, pre + "kernel", {in, out});
  d.bias = add_tensor(p, pre + "bias", {out});
  return d;
}
static Norm add_norm(smd_plan* p, const std::string& pre, int n) {
  Norm r;
  r.scale = add_tensor(p, pre + "scale", {n});
  r.bias = add_tensor(p, pre + "bias", {n});
  return r;
}

static void build_layout(smd_plan* p) {
  const smd_config& c = p->cfg;
  const int C = c.channels, Md = c.mlp_dims;
  ParamLayout& par = p->par;
  const bool film = !p->mdn();   // TransformerMDN's res-blocks are DenseResBlock(x, mlp_dims) with scale 1, shift 0
  if (c.arch == SMD_ARCH_TRANSFORMER_DDPM || p->mdn()) {
    par.in = add_dense(p, "in.", C, kE);
    p->L = c.num_layers;
    par.layer.resize(p->L);
    for (int l = 0; l < p->L; ++l) {
      const std::string pre = "l" + std::to_string(l) + ".";
      LayerParams& lp = par.layer[l];
      lp.ln1 = add_norm(p, pre + "ln1.", kE);
      lp.qkv = add_dense(p, pre + "attn.qkv.", kE, 3 * kE);
      lp.out = add_dense(p, pre + "attn.out.", kE, kE);
      lp.ln2 = add_norm(p, pre + "ln2.", kE);
      lp.ffn1 = add_dense(p, pre + "ffn1.", kE, Md);
      lp.ffn2 = add_dense(p, pre + "ffn2.", Md, kE);
    }
    par.post_ln = add_norm(p, "post_ln.", kE);
    par.post = add_dense(p, "post.", kE, Md);
    p->K = c.num_mlp_layers;
  } else {
    par.in = add_dense(p, "in.", C, Md);
    p->K = c.num_layers;
  }
  par.block.resize(p->K);
  for (int k = 0; k < p->K; ++k) {
    const std::string pre = "k" + std::to_string(k) + ".";
    BlockParams& bp = par.block[k];
    if (film) {
      bp.film.d1 = add_dense(p, pre + "film.d1.", kFilmEmb, kFilmHid);
      bp.film.d2 = add_dense(p, pre + "film.d2.", kFilmHid, kFilmHid);
      bp.film.ss = add_dense(p, pre + "film.ss.", kFilmHid, 2 * Md);
    }
    bp.ln_a = add_norm(p, pre + "res.ln_a.", Md);
    bp.a = add_dense(p, pre + "res.a.", Md, Md);
    bp.ln_b = add_norm(p, pre + "res.ln_b.", Md);
    bp.b = add_dense(p, pre + "res.b.", Md, Md);
  }
  par.out_ln = add_norm(p, "out_ln.", Md);
  if (p->mdn()) {   // models/shared.py MDN: three Dense layers, flax order mu, log_sigma, pi
    par.mdn_mu = add_dense(p, "mdn.mu.", Md, p->Kc * C);
    par.mdn_log_sigma = add_dense(p, "mdn.log_sigma.", Md, p->Kc * C);
    par.mdn_pi = add_dense(p, "mdn.pi.", Md, p->Kc);
  } else {
    par.out = add_dense(p, "out.", Md, C);
  }
}

// Reserves a 1024-byte aligned workspace region and returns its byte offset.
static size_t ws_add(smd_plan* p, std::string name, size_t bytes) {
  const size_t off = p->ws_bytes;
  bytes = (bytes + 1023) / 1024 * 1024;
  p->regions.push_back({std::move(name), off, bytes});
  p->ws_bytes += bytes;
  return off;
}

static void build_workspace(smd_plan* p) {
  const smd_config& c = p->cfg;
  const size_t Mp = p->Mp, Md = c.mlp_dims, C = c.channels, B = c.max_batch, K = p->K;
  const size_t Cp = (C + 63) / 64 * 64;
  const int L = p->L;
  const bool strict = c.precision == SMD_PRECISION_BF16X3;
  WorkspaceLayout& w = p->reg;
  // bf16 shadow of the whole parameter arena (same offsets): every GEMM weight operand is read from it in place --
  // forward as an MN-major B operand ((in,out) = [K][N]), dX as a K-major B operand ([N=in][K=out]) -- so there
  // are no transposed copies and the optimizer refreshes it in the same pass that updates the fp32 masters.
  w.wshadow = ws_add(p, "wshadow", static_cast<size_t>(p->arena) * 2);
  // out.kernel is (Md, C) with C = 42 / 146: its 2C-byte row pitch is not TMA-addressable, so it gets a copy
  // zero-padded to a multiple of 64 columns (TransformerMDN: the three head kernels packed into [Md][Np])
  const size_t Hp = p->head_ld;
  w.out_pad = ws_add(p, "w.out_pad", Md * Hp * 2);
  // forward activations, n indices per family: a training plan keeps every index for the backward pass, an inference
  // plan overwrites one region in place
  auto family = [&](int n, size_t bytes, auto name) {
    std::vector<size_t> v;
    for (int i = 0; i < n; ++i) v.push_back(i == 0 || c.training ? ws_add(p, name(i), bytes) : v[0]);
    return v;
  };
  auto idx = [](const char* base) { return [base](int i) { return base + std::to_string(i); }; };
  if (L > 0) {
    w.h = family(2 * L + 1, Mp * kE * 4, idx("t.h"));
    w.a = family(2 * L + 1, Mp * kE * 2, [L](int i) {
      return i == 2 * L ? std::string("t.a_post") : (i % 2 ? "t.a2_" : "t.a1_") + std::to_string(i / 2);
    });
    w.qkv = family(L, Mp * 3 * kE * 4, idx("t.qkv"));
    w.o = family(L, Mp * kE * 2, idx("t.o"));
    w.hidden = family(L, Mp * Md * 2, idx("t.hid"));
    if (c.training) {
      w.hidden_pre = family(L, Mp * Md * 2, idx("t.hpre"));
      w.probs = family(L, B * c.num_heads * c.seq_len * c.seq_len * 4, idx("t.probs"));   // [B][H][S][S]
    }
  } else {
    w.xb = ws_add(p, "xb", Mp * Cp * 2);
  }
  w.u = family(K + 1, Mp * Md * 4, idx("t.u"));
  w.r1 = family(K, Mp * Md * (strict ? 4 : 2), idx("t.r1_"));
  w.act = family(2 * K + 1, Mp * Md * 2, [K](int i) {
    return i == static_cast<int>(2 * K) ? std::string("t.act_out") : (i % 2 ? "t.actb" : "t.acta") + std::to_string(i / 2);
  });
  // per-row LayerNorm (sum, sumsq) of the 2K+1 wide LayerNorms; zeroed once per forward
  w.stats = ws_add(p, "stats", (2 * K + 1) * Mp * 2 * 4);
  // per-tile partial sums of the GEMM feeding the next wide LayerNorm: [row][n_tile * (2 or 3) + column group][2]
  w.stats_part = ws_add(p, "stats_part", Mp * ((Md + kBNMax - 1) / kBNMax * 3) * 2 * 4);
  // FiLM generator
  w.tvec = ws_add(p, "tvec", B * 4);
  w.enc = ws_add(p, "enc", B * kFilmEmb * 4);
  w.e1 = family(K, B * kFilmHid * 4, idx("t.e1_"));
  w.e2 = family(K, B * kFilmHid * 4, idx("t.e2_"));
  if (c.training) w.e1pre = family(K, B * kFilmHid * 4, idx("t.e1pre"));
  w.ss = ws_add(p, "ss", K * B * 2 * Md * 4);
  w.posenc = ws_add(p, "posenc", static_cast<size_t>(c.seq_len) * kE * 4);
  w.freqs = ws_add(p, "freqs", 64 * 4);
  // objective / sampler scratch
  w.xt = ws_add(p, "xt", B * c.seq_len * C * 4);
  w.eps_hat = ws_add(p, "eps_hat", B * c.seq_len * C * 4);
  w.coef = ws_add(p, "coef", kMaxT * 8 * 4);
  w.keys = ws_add(p, "keys", kMaxT * 4 * 4);
  w.slots = ws_add(p, "slots", kMaxT * 4);
  w.t_ptr = ws_add(p, "t_ptr", 64);
  w.abar = ws_add(p, "abar", (kMaxT + 1) * 4);
  w.sigmas = ws_add(p, "sigmas", kMaxT * 4);
  if (c.sampler_T > 0) {
    const size_t T = c.sampler_T;
    w.ftab_t = ws_add(p, "ftab.t", T * 4);
    w.ftab_enc = ws_add(p, "ftab.enc", T * kFilmEmb * 4);
    w.ftab_e1 = ws_add(p, "ftab.e1", T * kFilmHid * 4);
    w.ftab_e2 = ws_add(p, "ftab.e2", T * kFilmHid * 4);
    w.ftab = ws_add(p, "ftab", K * T * 2 * Md * 4);
  }
  if (c.training) {
    TrainState& t = p->train;
    t.g16 = ws_add(p, "t.g16", Mp * Md * 2);
    t.du32 = ws_add(p, "t.du32", Mp * Md * 4);
    t.du16 = family(K + 1, Mp * Md * 2, idx("t.du16_"));
    t.dr16t = family(K, Mp * Md * 2, idx("t.dr16t_"));
    t.dh = ws_add(p, "t.dh", Mp * kE * 4);
    t.dh2 = ws_add(p, "t.dh2", Mp * kE * 4);
    t.dh16a = family(L, Mp * kE * 2, idx("t.dh16a"));
    t.dh16b = family(L, Mp * kE * 2, idx("t.dh16b"));
    t.dr16 = family(L, Mp * Md * 2, idx("t.dr16_"));
    t.dqkv16 = family(L, Mp * 3 * kE * 2, idx("t.dqkv16_"));
    t.dpred16 = ws_add(p, "t.dpred16", Mp * Hp * 2);
    t.dpred32 = ws_add(p, "t.dpred32", Mp * C * 4);
    t.dss = ws_add(p, "t.dss", K * B * 2 * Md * 4);   // one [B][2Md] block per FiLM pair
    t.de = ws_add(p, "t.de", B * kFilmHid * 4);
    t.de2 = ws_add(p, "t.de2", B * kFilmHid * 4);
    t.loss = ws_add(p, "t.loss", B * (p->mdn() ? c.seq_len : 1) * 4);
    t.loss_ctr = ws_add(p, "t.loss_ctr", 64);
    t.ind = ws_add(p, "t.ind", 64);
    const size_t Bp = (B + 127) / 128 * 128;
    t.e2_16 = ws_add(p, "t.e2_16", Bp * kFilmHid * 2);
    t.dss16 = ws_add(p, "t.dss16", Bp * 2 * Md * 2);
  }
  if (c.arch == SMD_ARCH_DENSE_NCSN) {
    // tangent pass of sliced score matching, after every other region so the primal offsets stay where they are
    w.xbt = ws_add(p, "xbt", Mp * Cp * 2);
    w.ut = family(K + 1, Mp * Md * 4, idx("t.ut"));
    w.r1t = family(K, Mp * Md * 4, idx("t.r1t"));
    w.actt = family(2 * K + 1, Mp * Md * 2, idx("t.actt"));
    w.yt = ws_add(p, "yt", B * C * 4);
    if (c.training) {
      TrainState& t = p->train;
      t.gt16 = ws_add(p, "t.gt16", Mp * Md * 2);
      t.dut32 = ws_add(p, "t.dut32", Mp * Md * 4);
      t.dut16 = family(K + 1, Mp * Md * 2, idx("t.dut16_"));
      t.drt16 = family(K, Mp * Md * 2, idx("t.drt16_"));
      t.dpredt16 = ws_add(p, "t.dpredt16", Mp * Cp * 2);
    }
  }
  if (p->mdn()) {
    w.head = ws_add(p, "mdn.head", Mp * Hp * 4);
    w.head_bias = ws_add(p, "mdn.head_bias", Hp * 4);
  }
  if (strict) {
    w.x3_scratch = ws_add(p, "x3.scratch", Mp * Md * 4);   // fp32 cross-term accumulator of the three-pass GEMMs
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
  const WorkspaceLayout& w = p->reg;
  // forward GEMM: A K-major activations [Mp][K], B = (in,out) weight read MN-major ([K][N]) from the shadow arena; every
  // forward GEMM has N >= 128 and uses the widest tile
  auto fwd = [&](GemmOp* op, size_t a, long long wt, int K, int N) {
    return make_gemm_op(op, p->ws + a, Mp, p->wsh(wt), static_cast<uint64_t>(N), N, K, kBNMax, 0, 1, 0, 0, p->lo_bytes);
  };
  p->op_qkv.resize(p->L); p->op_o.resize(p->L);
  p->op_ffn1.resize(p->L); p->op_ffn2.resize(p->L);
  p->op_ffn.resize(p->L);
  p->op_attn.resize(p->L);
  for (int l = 0; l < p->L; ++l) {
    const LayerParams& lp = p->par.layer[l];
    const size_t a1 = w.a[2 * l], a2 = w.a[2 * l + 1];
    if (!fwd(&p->op_qkv[l], a1, lp.qkv.kernel, kE, 3 * kE)) return SMD_ERR_CUDA;
    if (!fwd(&p->op_o[l], w.o[l], lp.out.kernel, kE, kE)) return SMD_ERR_CUDA;
    if (!fwd(&p->op_ffn1[l], a2, lp.ffn1.kernel, kE, Md)) return SMD_ERR_CUDA;
    if (!fwd(&p->op_ffn2[l], w.hidden[l], lp.ffn2.kernel, Md, kE)) return SMD_ERR_CUDA;
    if (Md % 128 == 0 &&
        !make_ffn_op(&p->op_ffn[l], p->ws + a2, Mp, p->wsh(lp.ffn1.kernel), p->wsh(lp.ffn2.kernel), Md)) return SMD_ERR_CUDA;
    if ((c.num_heads == 8 || c.num_heads == 16) &&
        !make_attn_op(&p->op_attn[l], p->ws + a1, Mp, p->wsh(lp.qkv.kernel), p->wsh(lp.out.kernel))) return SMD_ERR_CUDA;
  }
  if (p->L > 0) {
    if (!fwd(&p->op_post, w.a[2 * p->L], p->par.post.kernel, kE, Md)) return SMD_ERR_CUDA;
  } else {
    if (!fwd(&p->op_in, w.xb, p->par.in.kernel, C, Md)) return SMD_ERR_CUDA;
  }
  p->op_a.resize(p->K); p->op_b.resize(p->K);
  for (int k = 0; k < p->K; ++k) {
    if (!fwd(&p->op_a[k], w.act[2 * k], p->par.block[k].a.kernel, Md, Md)) return SMD_ERR_CUDA;
    if (!fwd(&p->op_b[k], w.act[2 * k + 1], p->par.block[k].b.kernel, Md, Md)) return SMD_ERR_CUDA;
  }
  // output projection from the padded copy [Md][Cp]: N = C columns are valid (TransformerMDN: all Np of [Md][Np])
  if (!make_gemm_op(&p->op_out, p->ws + w.act[2 * p->K], Mp, p->ws + w.out_pad, static_cast<uint64_t>(p->head_ld),
                    p->head_n, Md, std::min(p->head_ld, kBNMax), 0, 1, 0, 0, p->lo_bytes))
    return SMD_ERR_CUDA;
  if (c.arch == SMD_ARCH_DENSE_NCSN) {
    if (!fwd(&p->op_tin, w.xbt, p->par.in.kernel, C, Md)) return SMD_ERR_CUDA;
    p->op_ta.resize(p->K); p->op_tb.resize(p->K);
    for (int k = 0; k < p->K; ++k) {
      if (!fwd(&p->op_ta[k], w.actt[2 * k], p->par.block[k].a.kernel, Md, Md)) return SMD_ERR_CUDA;
      if (!fwd(&p->op_tb[k], w.actt[2 * k + 1], p->par.block[k].b.kernel, Md, Md)) return SMD_ERR_CUDA;
    }
    if (!make_gemm_op(&p->op_tout, p->ws + w.actt[2 * p->K], Mp, p->ws + w.out_pad, static_cast<uint64_t>(Cp), C, Md,
                      std::min(Cp, kBNMax), 0, 1, 0, 0, p->lo_bytes))
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
    ef.stats_part = p->at<float>(p->reg.stats_part);
    p->stat_slots[ln_slot] = stats_slots_for(op, M, ef);
  };
  if (p->lo_bytes == 0) { arm_stats(e); return launch_gemm(op, M, e, st); }
  if (!op.has_lo) return cudaErrorInvalidValue;
  float* scratch = p->at<float>(p->reg.x3_scratch);
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
  float* totals = p->at<float>(p->reg.stats) + static_cast<size_t>(ln_slot) * p->Mp * 2;
  const int n = p->stat_slots[ln_slot];
  return n > 0 ? LnStats{p->at<float>(p->reg.stats_part), n, totals} : LnStats{nullptr, 0, totals};
}

// FiLM generator for all K blocks: t (R values) -> ss[k][R][2*Md]   (models/ncsn.py:47-61)
static int run_film(smd_plan* p, const float* params, const float* t, int R, cudaStream_t st, bool save) {
  const int Md = p->cfg.mlp_dims;
  const WorkspaceLayout& w = p->reg;
  float* enc = p->at<float>(w.enc);
  float* ss = p->at<float>(w.ss);
  launch_noise_encoding(t, p->at<float>(w.freqs), enc, R, st); CNT();
  for (int k = 0; k < p->K; ++k) {
    const FilmParams& f = p->par.block[k].film;
    float* e1 = p->at<float>(w.e1[k]);
    float* e2 = p->at<float>(w.e2[k]);
    float* e1pre = save ? p->at<float>(w.e1pre[k]) : nullptr;
    launch_small_linear(enc, params + f.d1.kernel, params + f.d1.bias, e1, R, kFilmEmb, kFilmHid, 2, st, e1pre); CNT();
    launch_small_linear(e1, params + f.d2.kernel, params + f.d2.bias, e2, R, kFilmHid, kFilmHid, 0, st); CNT();
    launch_small_linear(e2, params + f.ss.kernel, params + f.ss.bias,
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
// tangent: run the tangent pass next to it (ut[0] and the primal statistics are ready; see run_forward).
static int run_tail(smd_plan* p, const float* params, int M, int S, int t_broadcast, float* y, cudaStream_t st,
                    bool tangent) {
  const int Md = p->cfg.mlp_dims, C = p->cfg.channels;
  const WorkspaceLayout& w = p->reg;
  float* stats = p->at<float>(w.stats);
  const size_t sstride = static_cast<size_t>(p->Mp) * 2;
  float* ss = p->at<float>(w.ss);
  const bool strict = p->lo_bytes != 0;
  for (int k = 0; k < p->K; ++k) {
    const BlockParams& bp = p->par.block[k];
    const float* scale = p->mdn() ? nullptr : ss + static_cast<size_t>(k) * p->cfg.max_batch * 2 * Md;
    const int* frow_dev = nullptr;
    if (p->film_tab_on) {
      scale = p->at<float>(w.ftab) + static_cast<size_t>(k) * p->T * 2 * Md;
      if (p->film_row_dev) frow_dev = p->film_row_dev; else scale += static_cast<size_t>(p->film_row) * 2 * Md;
    }
    const float* shift = scale ? scale + Md : nullptr;
    float* u_in = p->at<float>(w.u[k]);
    float* u_out = p->at<float>(w.u[k + 1]);
    __nv_bfloat16* act_a = p->at<__nv_bfloat16>(w.act[2 * k]);
    __nv_bfloat16* act_b = p->at<__nv_bfloat16>(w.act[2 * k + 1]);
    LnStats ls = ln_stats(p, 2 * k);
    launch_ln_film_act(u_in, ls.totals, params + bp.ln_a.scale, params + bp.ln_a.bias,
                       scale, shift, 2 * Md, t_broadcast, 2, act_a, M, Md, S, st, frow_dev, nullptr, p->lo_elems,
                       ls.part, ls.nslots, ls.totals); CNT();
    if (tangent) {
      launch_ln_film_tangent(u_in, nullptr, ls.totals, p->at<float>(w.ut[k]), params + bp.ln_a.scale,
                             params + bp.ln_a.bias, scale, 2 * Md, 2, p->at<__nv_bfloat16>(w.actt[2 * k]), M, Md, S, st,
                             p->lo_elems); CNT();
    }
    GemmEpilogue e = epi();
    e.bias = params + bp.a.bias;
    // r1 only feeds a LayerNorm: bf16 is enough (strict mode keeps the pre-LayerNorm intermediate in fp32)
    float* r1 = strict ? p->at<float>(w.r1[k]) : nullptr;
    __nv_bfloat16* r1_16 = strict ? nullptr : p->at<__nv_bfloat16>(w.r1[k]);
    if (strict) { e.out_f32 = r1; e.ld_f32 = Md; }
    else { e.out_bf16 = r1_16; e.ld_bf16 = Md; }
    e.row_stats = stats + (2 * k + 1) * sstride;
    SMD_CUDA(gemm(p, p->op_a[k], M, e, st, 2 * k + 1));
    if (tangent) {
      e = epi();
      e.out_f32 = p->at<float>(w.r1t[k]); e.ld_f32 = Md;
      SMD_CUDA(gemm(p, p->op_ta[k], M, e, st));
    }
    ls = ln_stats(p, 2 * k + 1);
    launch_ln_film_act(r1, ls.totals, params + bp.ln_b.scale, params + bp.ln_b.bias, scale, shift, 2 * Md,
                       t_broadcast, 2, act_b, M, Md, S, st, frow_dev, r1_16, p->lo_elems, ls.part, ls.nslots,
                       ls.totals); CNT();
    if (tangent) {
      launch_ln_film_tangent(r1, r1_16, ls.totals, p->at<float>(w.r1t[k]), params + bp.ln_b.scale,
                             params + bp.ln_b.bias, scale, 2 * Md, 2, p->at<__nv_bfloat16>(w.actt[2 * k + 1]), M, Md, S,
                             st, p->lo_elems); CNT();
    }
    e = epi();
    e.bias = params + bp.b.bias;
    e.residual = u_in; e.ld_res = Md;
    e.out_f32 = u_out; e.ld_f32 = Md;
    e.row_stats = stats + (2 * k + 2) * sstride;
    SMD_CUDA(gemm(p, p->op_b[k], M, e, st, 2 * k + 2));
    if (tangent) {   // u' <- act_b' W_b + u'  (no bias)
      e = epi();
      e.residual = p->at<float>(w.ut[k]); e.ld_res = Md;
      e.out_f32 = p->at<float>(w.ut[k + 1]); e.ld_f32 = Md;
      SMD_CUDA(gemm(p, p->op_tb[k], M, e, st));
    }
  }
  const LnStats lo_ = ln_stats(p, 2 * p->K);
  launch_ln_film_act(p->at<float>(w.u[p->K]), lo_.totals, params + p->par.out_ln.scale, params + p->par.out_ln.bias,
                     nullptr, nullptr, 0, 0, 0, p->at<__nv_bfloat16>(w.act[2 * p->K]), M, Md, S, st, nullptr, nullptr,
                     p->lo_elems, lo_.part, lo_.nslots, lo_.totals); CNT();
  GemmEpilogue e = epi();
  e.bias = p->mdn() ? p->at<float>(w.head_bias) : params + p->par.out.bias;
  e.out_f32 = y; e.ld_f32 = p->mdn() ? p->head_ld : C;
  SMD_CUDA(gemm(p, p->op_out, M, e, st));
  if (tangent) {
    launch_ln_film_tangent(p->at<float>(w.u[p->K]), nullptr, lo_.totals, p->at<float>(w.ut[p->K]),
                           params + p->par.out_ln.scale, params + p->par.out_ln.bias, nullptr, 0, 0,
                           p->at<__nv_bfloat16>(w.actt[2 * p->K]), M, Md, S, st, p->lo_elems); CNT();
    e = epi();
    e.out_f32 = p->at<float>(w.yt); e.ld_f32 = C;
    SMD_CUDA(gemm(p, p->op_tout, M, e, st));
  }
  SMD_LAUNCH_CHECK("tail");
  return SMD_OK;
}

int run_forward(smd_plan* p, const float* params, const float* x, const float* t, int t_broadcast, int batch,
                float* y, cudaStream_t st, bool save, bool raw_out, bool tangent) {
  const smd_config& c = p->cfg;
  if (!p->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (!p->packed) { set_error("smd_pack_weights has not been called"); return SMD_ERR_STATE; }
  if (batch < 1 || batch > c.max_batch) { set_error("batch out of range"); return SMD_ERR_INVALID; }
  const int S = c.seq_len, C = c.channels, Md = c.mlp_dims;
  const int M = batch * S;
  const WorkspaceLayout& w = p->reg;
  float* stats = p->at<float>(w.stats);
  p->stat_slots.assign(static_cast<size_t>(2 * p->K + 1), 0);
  SMD_CUDA(cudaMemsetAsync(stats, 0, static_cast<size_t>(2 * p->K + 1) * p->Mp * 2 * 4, st));
  int rc = SMD_OK;
  bool film_on_side = false;
  if (!p->film_tab_on && !p->mdn()) {
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
  float* u0 = p->at<float>(w.u[0]);
  if (p->L > 0) {
    const ParamLayout& par = p->par;
    auto h = [&](int i) { return p->at<float>(w.h[i]); };
    auto a = [&](int i) { return p->at<__nv_bfloat16>(w.a[i]); };
    launch_embed(x, params + par.in.kernel, params + par.in.bias, p->at<float>(w.posenc),
                 params + par.layer[0].ln1.scale, params + par.layer[0].ln1.bias, h(0), a(0), M, C, S, st,
                 p->lo_elems); CNT();
    for (int l = 0; l < p->L; ++l) {
      const LayerParams& lp = par.layer[l];
      const Norm& next_ln = (l + 1 < p->L) ? par.layer[l + 1].ln1 : par.post_ln;
      float* h_in = h(2 * l); float* h_mid = h(2 * l + 1); float* h_out = h(2 * l + 2);
      __nv_bfloat16* a2 = a(2 * l + 1); __nv_bfloat16* a_next = a(2 * l + 2);
      GemmEpilogue e = epi();
      // the fused block's 64-row tile holds whole samples up to S = 64; S = 128 and causal attention take the
      // unfused path
      if (!save && S <= 64 && p->op_attn[l].ok && p->lo_bytes == 0 && !p->mdn()) {
        // QKV GEMM -> attention -> out-projection + residual + LayerNorm in ONE launch; q / k / v stay on chip
        AttnBlockArgs aa;
        aa.b_qkv = params + lp.qkv.bias; aa.b_o = params + lp.out.bias;
        aa.residual = h_in; aa.out_f32 = h_mid;
        aa.ln_gamma = params + lp.ln2.scale; aa.ln_beta = params + lp.ln2.bias;
        aa.out_bf16 = a2;
        aa.M = M; aa.H = c.num_heads; aa.S = S;
        SMD_CUDA(launch_attn_block(p->op_attn[l], aa, st));
      } else {
      float* qkv = p->at<float>(w.qkv[l]);
      e.bias = params + lp.qkv.bias;
      e.out_f32 = qkv; e.ld_f32 = 3 * kE;
      SMD_CUDA(gemm(p, p->op_qkv[l], M, e, st));
      SMD_CUDA(launch_attention(qkv, p->at<__nv_bfloat16>(w.o[l]), save ? p->at<float>(w.probs[l]) : nullptr, batch,
                                S, c.num_heads, st, p->lo_elems, /*causal=*/p->mdn())); CNT();
      e = epi();
      e.bias = params + lp.out.bias;
      e.residual = h_in; e.ld_res = kE;
      e.out_f32 = h_mid; e.ld_f32 = kE;
      e.out_bf16 = a2; e.ld_bf16 = kE;
      e.ln_gamma = params + lp.ln2.scale; e.ln_beta = params + lp.ln2.bias;
      SMD_CUDA(gemm(p, p->op_o[l], M, e, st));
      }
      // worth it once the token count fills the machine; training keeps the two-GEMM path: it has to write the hidden
      // activations anyway
      if (!save && M >= 32 * 256 && p->op_ffn[l].ok && p->lo_bytes == 0) {
        // FFN up + GELU + FFN down + residual + next LayerNorm in one launch; the hidden activation stays on chip
        FfnFusedArgs fa;
        fa.b1 = params + lp.ffn1.bias; fa.b2 = params + lp.ffn2.bias;
        fa.residual = h_mid; fa.out_f32 = h_out;
        fa.ln_gamma = params + next_ln.scale; fa.ln_beta = params + next_ln.bias;
        fa.out_bf16 = a_next;
        fa.M = M; fa.Md = Md;
        SMD_CUDA(launch_ffn_fused(p->op_ffn[l], fa, st));
        continue;
      }
      e = epi();
      e.bias = params + lp.ffn1.bias;
      e.out_bf16 = p->at<__nv_bfloat16>(w.hidden[l]); e.ld_bf16 = Md; e.act = ACT_GELU_TANH;
      e.out_bf16_pre = save ? p->at<__nv_bfloat16>(w.hidden_pre[l]) : nullptr;
      SMD_CUDA(gemm(p, p->op_ffn1[l], M, e, st));
      e = epi();
      e.bias = params + lp.ffn2.bias;
      e.residual = h_mid; e.ld_res = kE;
      e.out_f32 = h_out; e.ld_f32 = kE;
      e.out_bf16 = a_next; e.ld_bf16 = kE;
      e.ln_gamma = params + next_ln.scale; e.ln_beta = params + next_ln.bias;
      SMD_CUDA(gemm(p, p->op_ffn2[l], M, e, st));
    }
    GemmEpilogue e = epi();
    e.bias = params + par.post.bias;
    e.out_f32 = u0; e.ld_f32 = Md;
    e.row_stats = stats;
    SMD_CUDA(gemm(p, p->op_post, M, e, st, 0));
  } else {
    const int Cp = (C + 63) / 64 * 64;
    if (Cp != C) { set_error("DenseDDPM on the CUDA path needs channels % 64 == 0"); return SMD_ERR_INVALID; }
    launch_cast_bf16(x, p->at<__nv_bfloat16>(w.xb), static_cast<size_t>(M) * C, st, p->lo_elems); CNT();
    GemmEpilogue e = epi();
    e.bias = params + p->par.in.bias;
    e.out_f32 = u0; e.ld_f32 = Md;
    e.row_stats = stats;
    SMD_CUDA(gemm(p, p->op_in, M, e, st, 0));
    if (tangent) {   // u0' = v W_in (the caller cast v into xbt)
      e = epi();
      e.out_f32 = p->at<float>(w.ut[0]); e.ld_f32 = Md;
      SMD_CUDA(gemm(p, p->op_tin, M, e, st));
    }
  }
  SMD_LAUNCH_CHECK("trunk");
  if (film_on_side) SMD_CUDA(cudaStreamWaitEvent(st, p->ev_film, 0));
  rc = run_tail(p, params, M, S, t_broadcast, y, st, tangent);
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

// out[j] = element (first + j) of jax.random.rademacher(key, (total,)) as of jax 0.2.8: 2 bernoulli(key, 0.5) - 1 with
// bernoulli = uniform01 < 0.5, i.e. +1 exactly when the threefry word is below 2^31
__global__ void threefry_rademacher_kernel(uint32_t k0, uint32_t k1, float* out, uint32_t n, uint32_t first,
                                           uint32_t total) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    out[i] = jax_random_bits(k0, k1, first + i, total) < 0x80000000u ? 1.0f : -1.0f;
}

}  // namespace smd

// =====================================================================================================
// C ABI
// =====================================================================================================
extern "C" {

const char* smd_last_error(void) { return get_error(); }

// the score-network entry points have no meaning for the autoregressive baseline's plans
static bool reject_mdn(const smd_plan* plan, const char* fn) {
  if (!plan || !plan->mdn()) return false;
  set_error(std::string(fn) + " does not apply to a TransformerMDN plan (use the smd_mdn_* entry points)");
  return true;
}
int smd_version(void) { return 100; }
long long smd_launch_count(void) { return g_launches.load(); }

static int plan_create(const smd_config* cfg, int num_components, smd_plan** out) {
  if (!cfg || !out) { set_error("null argument"); return SMD_ERR_INVALID; }
  smd_config c = *cfg;
  const bool mdn = c.arch == SMD_ARCH_TRANSFORMER_MDN;
  if (c.arch != SMD_ARCH_TRANSFORMER_DDPM && c.arch != SMD_ARCH_DENSE_DDPM && c.arch != SMD_ARCH_DENSE_NCSN && !mdn) { set_error("unknown arch"); return SMD_ERR_INVALID; }
  if (c.cta_group == 0) c.cta_group = 1;
  if (c.cta_group != 1 && c.cta_group != 2) { set_error("cta_group must be 1 or 2"); return SMD_ERR_INVALID; }
  if (c.mlp_dims < 256 || c.mlp_dims % 256 != 0 || c.mlp_dims > 4096) { set_error("mlp_dims must be a multiple of 256 in [256, 4096]"); return SMD_ERR_INVALID; }
  if (c.channels < 1 || c.max_batch < 1 || c.num_layers < 1) { set_error("bad sizes"); return SMD_ERR_INVALID; }
  if (c.precision != SMD_PRECISION_BF16 && c.precision != SMD_PRECISION_BF16X3) { set_error("unknown precision"); return SMD_ERR_INVALID; }
  if (c.precision == SMD_PRECISION_BF16X3 && c.training) { set_error("precision bf16x3 covers the forward pass / sampler only (training = 0)"); return SMD_ERR_INVALID; }
  if (mdn) {
    if (c.seq_len != 32) { set_error("TransformerMDN CUDA path supports seq_len 32 only"); return SMD_ERR_INVALID; }
    if (c.precision != SMD_PRECISION_BF16) { set_error("TransformerMDN supports precision bf16 only"); return SMD_ERR_INVALID; }
    if (num_components < 1) { set_error("num_components must be >= 1"); return SMD_ERR_INVALID; }
    if (c.channels + 2LL * num_components > kMdnMaxRowFloats) { set_error("channels + 2 num_components must be <= " + std::to_string(kMdnMaxRowFloats)); return SMD_ERR_INVALID; }
  }
  if (c.arch == SMD_ARCH_TRANSFORMER_DDPM || mdn) {
    // each length divides the 128-row GEMM / LayerNorm tile and is a multiple of the 32-row blocks inside one sample
    if (c.seq_len != 32 && c.seq_len != 64 && c.seq_len != 128) { set_error("TransformerDDPM CUDA path supports seq_len in {32, 64, 128}"); return SMD_ERR_INVALID; }
    if (c.num_heads != 4 && c.num_heads != 8 && c.num_heads != 16 && c.num_heads != 32) { set_error("num_heads must be 4, 8, 16 or 32"); return SMD_ERR_INVALID; }
    if (c.num_mlp_layers < 1) { set_error("num_mlp_layers must be >= 1"); return SMD_ERR_INVALID; }
  } else {
    c.seq_len = 1;
  }
  smd_plan* p = new smd_plan();
  p->cfg = c;
  p->Mp = (c.max_batch * c.seq_len + 255) / 256 * 256;
  p->head_n = c.channels;
  p->head_ld = (c.channels + 63) / 64 * 64;
  if (mdn) {
    p->Kc = num_components;
    p->KCp = (num_components * c.channels + 63) / 64 * 64;
    p->Kcp = (num_components + 63) / 64 * 64;
    p->head_n = p->head_ld = 2 * p->KCp + p->Kcp;
  }
  build_layout(p);
  build_workspace(p);
  *out = p;
  return SMD_OK;
}

int smd_plan_create(const smd_config* cfg, smd_plan** out) {
  if (cfg && cfg->arch == SMD_ARCH_TRANSFORMER_MDN) {
    set_error("SMD_ARCH_TRANSFORMER_MDN plans are created with smd_mdn_plan_create (it takes the component count)");
    return SMD_ERR_INVALID;
  }
  return plan_create(cfg, 0, out);
}

int smd_mdn_plan_create(const smd_config* cfg, int num_components, smd_plan** out) {
  if (cfg && cfg->arch != SMD_ARCH_TRANSFORMER_MDN) { set_error("smd_mdn_plan_create needs arch SMD_ARCH_TRANSFORMER_MDN"); return SMD_ERR_INVALID; }
  return plan_create(cfg, num_components, out);
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
  SMD_CUDA(cudaMemcpy(plan->at<float>(plan->reg.freqs), f, sizeof(f), cudaMemcpyHostToDevice));
  // positional table (models/shared.py:33-48), float32 like jnp
  std::vector<float> pe(static_cast<size_t>(plan->cfg.seq_len) * kE);
  for (int s = 0; s < plan->cfg.seq_len; ++s)
    for (int j = 0; j < 64; ++j) {
      const float arg = static_cast<float>(s) * f[j];
      pe[s * kE + j] = sinf(arg);
      pe[s * kE + 64 + j] = cosf(arg);
    }
  SMD_CUDA(cudaMemcpy(plan->at<float>(plan->reg.posenc), pe.data(), pe.size() * 4, cudaMemcpyHostToDevice));
  if (plan->mdn() && plan->cfg.training) {
    // TransformerMDN's res-blocks are DenseResBlock with scale 1, shift 0: its backward passes these identity FiLM rows
    // ([max_batch][scale 1 | shift 0]) so the LayerNorm-swish backward takes its sequence fast path
    const size_t Md = plan->cfg.mlp_dims;
    std::vector<float> ident(plan->cfg.max_batch * 2 * Md, 0.0f);
    for (int b = 0; b < plan->cfg.max_batch; ++b) std::fill_n(ident.begin() + b * 2 * Md, Md, 1.0f);
    SMD_CUDA(cudaMemcpy(plan->at<float>(plan->reg.ss), ident.data(), ident.size() * 4, cudaMemcpyHostToDevice));
  }
  if (plan->cfg.training) { rc = train_bind(plan); if (rc) return rc; }
  return SMD_OK;
}

static int refresh_operands(smd_plan* plan, const float* params, bool shadow_is_fresh, cudaStream_t st) {
  if (!plan->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (!shadow_is_fresh) {
    launch_cast_bf16(params, plan->wsh(0), static_cast<size_t>(plan->arena), st, plan->lo_elems); CNT();
  }
  // out.kernel is the one GEMM weight not read from the shadow: its zero-padded copy (pad columns stay zero from bind)
  const int C = plan->cfg.channels;
  if (plan->mdn()) {
    const int rc = mdn_pack_head(plan, params, st);
    if (rc) return rc;
  } else {
    launch_pad_cast_bf16(params + plan->par.out.kernel, plan->at<__nv_bfloat16>(plan->reg.out_pad), plan->cfg.mlp_dims,
                         C, plan->head_ld, st, plan->lo_elems); CNT();
  }
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

void* smd_shadow_arena(smd_plan* plan) { return plan->ws ? plan->wsh(0) : nullptr; }

int smd_grads_tail_range(const smd_plan* plan, long long* first_float, long long* num_floats) {
  if (!plan || !first_float || !num_floats) { set_error("null argument"); return SMD_ERR_INVALID; }
  if (plan->par.block.empty()) { set_error("plan has no FiLM'd residual tail"); return SMD_ERR_STATE; }
  // first tensor of the residual tail; out_ln and the output layer (out, or mdn.*) follow it
  *first_float = plan->mdn() ? plan->par.block[0].ln_a.scale : plan->par.block[0].film.d1.kernel;
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
  if (reject_mdn(plan, "smd_forward")) return SMD_ERR_INVALID;
  return run_forward(plan, params, x, t, t_broadcast, batch, y, static_cast<cudaStream_t>(stream), false);
}

int smd_ddpm_loss(smd_plan* plan, const float* params, const float* x0, const float* used_alpha, const float* eps,
                  int batch, float* loss_per_example, float* pred_or_null, smd_stream_t stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (reject_mdn(plan, "smd_ddpm_loss")) return SMD_ERR_INVALID;
  if (!plan->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (batch < 1 || batch > plan->cfg.max_batch) { set_error("batch out of range"); return SMD_ERR_INVALID; }
  const int per = plan->cfg.seq_len * plan->cfg.channels;
  float* xt = plan->at<float>(plan->reg.xt);
  float* cond = plan->at<float>(plan->reg.tvec);
  float* pred = pred_or_null ? pred_or_null : plan->at<float>(plan->reg.eps_hat);
  launch_q_sample(x0, eps, used_alpha, xt, cond, batch, per, st); CNT();
  int rc = run_forward(plan, params, xt, cond, 0, batch, pred, st, false);
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
  float* xt = plan->at<float>(plan->reg.xt);
  float* cond = plan->at<float>(plan->reg.tvec);
  float* pred = pred_or_null ? pred_or_null : plan->at<float>(plan->reg.eps_hat);
  launch_q_sample(x0, eps, used_sigma, xt, cond, batch, per, st, nullptr, 1); CNT();
  int rc = run_forward(plan, params, xt, cond, 0, batch, pred, st, false);
  if (rc) return rc;
  launch_ddpm_loss(eps, pred, loss_per_example, nullptr, 0.f, batch, per, st, used_sigma); CNT();
  SMD_LAUNCH_CHECK("dsm_loss");
  return SMD_OK;
}

int smd_dsm_setup(smd_plan* plan, const float* host_sigmas, int L, smd_stream_t stream) {
  if (!plan->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (L < 2 || L > kMaxT) { set_error("schedule length out of range"); return SMD_ERR_INVALID; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SMD_CUDA(cudaMemcpyAsync(plan->at<float>(plan->reg.sigmas), host_sigmas, static_cast<size_t>(L) * 4, cudaMemcpyHostToDevice, st));
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
  draws_kernel<<<(batch + 127) / 128, 128, 0, st>>>(k3[2], k3[3], k2[2], k2[3], plan->at<float>(plan->reg.sigmas), L - 1, L - cn,
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

int smd_ssm_draws(smd_plan* plan, const uint32_t host_key[2], int global_batch, int first_row, int batch,
                  int continuous_noise, float* used_sigma, float* eps, float* v, int* labels_or_null,
                  smd_stream_t stream) {
  if (plan->cfg.arch != SMD_ARCH_DENSE_NCSN) { set_error("smd_ssm_draws needs a score network (SMD_ARCH_DENSE_NCSN)"); return SMD_ERR_INVALID; }
  if (plan->L_dsm <= 0) { set_error("smd_dsm_setup has not been called"); return SMD_ERR_STATE; }
  if (batch < 1 || first_row < 0 || global_batch < first_row + batch) { set_error("batch out of range"); return SMD_ERR_INVALID; }
  const long long per = static_cast<long long>(plan->cfg.seq_len) * plan->cfg.channels;
  if (static_cast<long long>(global_batch) * per > 0xFFFFFFFFll) { set_error("global batch too large"); return SMD_ERR_INVALID; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int L = plan->L_dsm, cn = continuous_noise ? 1 : 0;
  uint32_t k4[8], k2[4] = {0, 0, 0, 0};
  h_split(host_key, 4, k4);               // rng, label_rng, sample_rng, score_rng   (utils/losses.py:203)
  if (cn) { const uint32_t rng[2] = {k4[0], k4[1]}; h_split(rng, 2, k2); }        // rng, noise_rng (:210)
  draws_kernel<<<(batch + 127) / 128, 128, 0, st>>>(k4[2], k4[3], k2[2], k2[3], plan->at<float>(plan->reg.sigmas), L - 1, L - cn,
                                                    global_batch, first_row, batch, cn, cn, used_sigma, labels_or_null);
  CNT();
  const long long n = static_cast<long long>(batch) * per;
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > 148 * 8) blocks = 148 * 8;
  const uint32_t first = static_cast<uint32_t>(first_row * per), total = static_cast<uint32_t>(global_batch * per);
  threefry_normal_kernel<<<blocks, 256, 0, st>>>(k4[4], k4[5], eps, static_cast<uint32_t>(n), first, total);
  CNT();
  threefry_rademacher_kernel<<<blocks, 256, 0, st>>>(k4[6], k4[7], v, static_cast<uint32_t>(n), first, total);
  CNT();
  SMD_LAUNCH_CHECK("ssm_draws");
  return SMD_OK;
}

int smd_ssm_loss(smd_plan* plan, const float* params, const float* x0, const float* used_sigma, const float* eps,
                 const float* v, int batch, float* loss_per_example, float* score_or_null, float* hvp_or_null,
                 smd_stream_t stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (plan->cfg.arch != SMD_ARCH_DENSE_NCSN) { set_error("smd_ssm_loss needs a score network (SMD_ARCH_DENSE_NCSN)"); return SMD_ERR_INVALID; }
  if (!plan->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (batch < 1 || batch > plan->cfg.max_batch) { set_error("batch out of range"); return SMD_ERR_INVALID; }
  const int C = plan->cfg.channels;
  float* xt = plan->at<float>(plan->reg.xt);
  float* cond = plan->at<float>(plan->reg.tvec);
  float* f = plan->at<float>(plan->reg.eps_hat);
  launch_q_sample(x0, eps, used_sigma, xt, cond, batch, C, st, nullptr, 1); CNT();
  launch_tangent_input(v, nullptr, plan->at<__nv_bfloat16>(plan->reg.xbt), static_cast<size_t>(batch) * C, st,
                       plan->lo_elems); CNT();
  int rc = run_forward(plan, params, xt, cond, 0, batch, f, st, false, /*raw_out=*/true, /*tangent=*/true);
  if (rc) return rc;
  launch_ssm_loss(f, plan->at<float>(plan->reg.yt), v, used_sigma, nullptr, loss_per_example, score_or_null,
                  hvp_or_null, nullptr, nullptr, 1.0f, nullptr, nullptr, nullptr, batch, C, C, st); CNT();
  SMD_LAUNCH_CHECK("ssm_loss");
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
  SMD_CUDA(cudaMemcpyAsync(plan->at<float>(plan->reg.abar), ap.data(), ap.size() * 4, cudaMemcpyHostToDevice, st));
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
  draws_kernel<<<(batch + 127) / 128, 128, 0, st>>>(k3[2], k3[3], k2[2], k2[3], plan->at<float>(plan->reg.abar), plan->T_obj,
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
  if (reject_mdn(plan, "smd_sampler_setup")) return SMD_ERR_INVALID;
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
  SMD_CUDA(cudaMemcpyAsync(plan->at<float>(plan->reg.coef), coef.data(), coef.size() * 4, cudaMemcpyHostToDevice, st));
  SMD_CUDA(cudaMemcpyAsync(plan->at<uint32_t>(plan->reg.keys), keys.data(), keys.size() * 4, cudaMemcpyHostToDevice, st));
  SMD_CUDA(cudaMemcpyAsync(plan->at<int>(plan->reg.slots), slots.data(), slots.size() * 4, cudaMemcpyHostToDevice, st));
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
  float* tv = plan->at<float>(plan->reg.ftab_t);
  float* enc = plan->at<float>(plan->reg.ftab_enc);
  float* e1 = plan->at<float>(plan->reg.ftab_e1);
  float* e2 = plan->at<float>(plan->reg.ftab_e2);
  float* tab = plan->at<float>(plan->reg.ftab);
  gather_cond_kernel<<<(T + 255) / 256, 256, 0, st>>>(plan->at<float>(plan->reg.coef), tv, T); CNT();
  launch_noise_encoding(tv, plan->at<float>(plan->reg.freqs), enc, T, st); CNT();
  for (int k = 0; k < plan->K; ++k) {
    const FilmParams& f = plan->par.block[k].film;
    launch_small_linear(enc, params + f.d1.kernel, params + f.d1.bias, e1, T, kFilmEmb, kFilmHid, 2, st); CNT();
    launch_small_linear(e1, params + f.d2.kernel, params + f.d2.bias, e2, T, kFilmHid, kFilmHid, 0, st); CNT();
    launch_small_linear(e2, params + f.ss.kernel, params + f.ss.bias,
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
  float* tvec = plan->at<float>(plan->reg.tvec);
  int* t_ptr = plan->at<int>(plan->reg.t_ptr);
  const float* coef = plan->at<float>(plan->reg.coef);
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
  float* eh = eps_hat ? eps_hat : plan->at<float>(plan->reg.eps_hat);
  int rc = run_forward(plan, params, x, tvec, 1, n, eh, st, false);
  plan->film_tab_on = false;
  plan->film_row_dev = nullptr;
  if (rc) return rc;
  ReverseStepArgs a;
  memset(&a, 0, sizeof(a));
  a.x = x; a.eps_hat = eh; a.z = z;
  a.key_tab = plan->at<uint32_t>(plan->reg.keys);
  a.coef = coef;
  a.slot_tab = plan->at<int>(plan->reg.slots);
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
  if (reject_mdn(plan, "smd_ddpm_reverse_step")) return SMD_ERR_INVALID;
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
  if (reject_mdn(plan, "smd_ddpm_sample")) return SMD_ERR_INVALID;
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
  int* t_ptr = plan->at<int>(plan->reg.t_ptr);
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
  if (reject_mdn(plan, "smd_debug_forward_save")) return SMD_ERR_INVALID;
  if (!plan->cfg.training) { set_error("plan was not created with training = 1"); return SMD_ERR_STATE; }
  return run_forward(plan, params, x, t, 0, batch, y, static_cast<cudaStream_t>(stream), true);
}

int smd_debug_buffer(smd_plan* plan, const char* name, void** dev_ptr, size_t* bytes) {
  if (!plan->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  for (const WsRegion& r : plan->regions) {
    if (r.name != name) continue;
    if (dev_ptr) *dev_ptr = plan->ws + r.offset;
    if (bytes) *bytes = r.bytes;
    return SMD_OK;
  }
  set_error(std::string("no workspace region named ") + name);
  return SMD_ERR_INVALID;
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

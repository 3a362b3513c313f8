// Hand-written backward pass of the DDPM objective: what jax.value_and_grad(loss_fn) produces at
// train_ncsn.py:282-283 for diffusion_loss (utils/losses.py:250-308) over TransformerDDPM / DenseDDPM.
// Every matmul runs on the wgmma GEMM (dX: K-major operands, dW: MN-major operands reducing over tokens,
// split-K + atomics for the skinny ones); everything else is SIMT (backward_kernels.cuh).
#include "plan.cuh"
#include "backward_kernels.cuh"

namespace smd {

// Split count for a dW GEMM that runs beside the dX chain: ~48 CTAs, leaving two thirds of the SMs to `st`.
int pick_splits_side(int m_rows, int n_cols, int BN, int num_kb) {
  const int tiles = ((m_rows + 127) / 128) * ((n_cols + BN - 1) / BN);
  int s = 48 / tiles;
  if (s < 1) s = 1;
  if (s > num_kb) s = num_kb;
  return s;
}

// dW GEMM: A = X (MN-major [tokens][in]), B = G (MN-major [tokens][out]) -> out_f32 [in][out].  wide: ask for the
// 128 x 256 layout (the res-block GEMMs)
static bool make_dw(GemmOp* op, const void* X, int in_f, const void* G, int g_cols, int out_f, uint64_t rows,
                    bool wide = false) {
  const int BN = wide ? kBNWide : std::min((out_f + 63) / 64 * 64, kBNMax);
  return make_gemm_op(op, X, static_cast<uint64_t>(in_f), G, static_cast<uint64_t>(g_cols), out_f,
                      static_cast<int>(rows), BN, 1, 1);
}
// dX GEMM: A = G (K-major [tokens][out]), B = W plain (in,out) = [N=in][K=out] -> [tokens][in]
static bool make_dx(GemmOp* op, const void* G, int out_f, const void* W, int in_f, uint64_t rows, bool wide = false) {
  return make_gemm_op(op, G, rows, W, static_cast<uint64_t>(in_f), in_f, out_f, wide ? kBNWide : choose_bn(in_f), 0, 0);
}

int train_bind(smd_plan* p) {
  TrainState& ts = p->train;
  const WorkspaceLayout& w = p->reg;
  const ParamLayout& par = p->par;
  const smd_config& c = p->cfg;
  const int Md = c.mlp_dims, C = c.channels, K = p->K, L = p->L;
  const int Cp = (C + 63) / 64 * 64;
  const uint64_t Mp = p->Mp;
  auto B16 = [&](size_t off) { return p->at<__nv_bfloat16>(off); };
  ts.dWb.resize(K); ts.dXb.resize(K); ts.dWa.resize(K); ts.dXa.resize(K);
  ts.dWss.resize(K); ts.dXss.resize(K);
  const uint64_t Bp = (static_cast<uint64_t>(c.max_batch) + 127) / 128 * 128;
  for (int k = 0; k < K; ++k) {
    const BlockParams& bp = par.block[k];
    if (!make_dw(&ts.dWb[k], B16(w.act[2 * k + 1]), Md, B16(ts.du16[k + 1]), Md, Md, Mp, true)) return SMD_ERR_CUDA;
    if (!make_dx(&ts.dXb[k], B16(ts.du16[k + 1]), Md, p->wsh(bp.b.kernel), Md, Mp, true)) return SMD_ERR_CUDA;
    if (!make_dw(&ts.dWa[k], B16(w.act[2 * k]), Md, B16(ts.dr16t[k]), Md, Md, Mp, true)) return SMD_ERR_CUDA;
    if (!make_dx(&ts.dXa[k], B16(ts.dr16t[k]), Md, p->wsh(bp.a.kernel), Md, Mp, true)) return SMD_ERR_CUDA;
    if (p->mdn()) continue;   // no FiLM generator
    if (!make_dw(&ts.dWss[k], B16(ts.e2_16), 512, B16(ts.dss16), 2 * Md, 2 * Md, Bp)) return SMD_ERR_CUDA;
    if (!make_dx(&ts.dXss[k], B16(ts.dss16), 2 * Md, p->wsh(bp.film.ss.kernel), 512, Bp)) return SMD_ERR_CUDA;
  }
  // output projection: dpred16 is zero-padded to Cp columns; the plain weight copy is [Md][Cp] (TransformerMDN: dZ and
  // the packed head weight, both Np wide; its dW GEMMs are built by mdn_train_bind)
  if (!p->mdn() &&
      !make_gemm_op(&ts.dWout, B16(w.act[2 * K]), static_cast<uint64_t>(Md), B16(ts.dpred16), static_cast<uint64_t>(Cp),
                    C, static_cast<int>(Mp), std::min(Cp, kBNMax), 1, 1))
    return SMD_ERR_CUDA;
  if (!make_gemm_op(&ts.dXout, B16(ts.dpred16), Mp, B16(w.out_pad), static_cast<uint64_t>(Md), Md, p->head_ld,
                    choose_bn(Md), 0, 0)) return SMD_ERR_CUDA;
  if (L > 0) {
    if (!make_dw(&ts.dWpost, B16(w.a[2 * L]), 128, B16(ts.du16[0]), Md, Md, Mp)) return SMD_ERR_CUDA;
    if (!make_dx(&ts.dXpost, B16(ts.du16[0]), Md, p->wsh(par.post.kernel), 128, Mp)) return SMD_ERR_CUDA;
    ts.dW2.resize(L); ts.dX2.resize(L); ts.dW1.resize(L); ts.dX1.resize(L);
    ts.dWo.resize(L); ts.dXo.resize(L); ts.dWqkv.resize(L); ts.dXqkv.resize(L);
    for (int l = 0; l < L; ++l) {
      const LayerParams& lp = par.layer[l];
      if (!make_dw(&ts.dW2[l], B16(w.hidden[l]), Md, B16(ts.dh16a[l]), 128, 128, Mp)) return SMD_ERR_CUDA;
      if (!make_dx(&ts.dX2[l], B16(ts.dh16a[l]), 128, p->wsh(lp.ffn2.kernel), Md, Mp)) return SMD_ERR_CUDA;
      if (!make_dw(&ts.dW1[l], B16(w.a[2 * l + 1]), 128, B16(ts.dr16[l]), Md, Md, Mp)) return SMD_ERR_CUDA;
      if (!make_dx(&ts.dX1[l], B16(ts.dr16[l]), Md, p->wsh(lp.ffn1.kernel), 128, Mp)) return SMD_ERR_CUDA;
      if (!make_dw(&ts.dWo[l], B16(w.o[l]), 128, B16(ts.dh16b[l]), 128, 128, Mp)) return SMD_ERR_CUDA;
      if (!make_dx(&ts.dXo[l], B16(ts.dh16b[l]), 128, p->wsh(lp.out.kernel), 128, Mp)) return SMD_ERR_CUDA;
      if (!make_dw(&ts.dWqkv[l], B16(w.a[2 * l]), 128, B16(ts.dqkv16[l]), 384, 384, Mp)) return SMD_ERR_CUDA;
      if (!make_dx(&ts.dXqkv[l], B16(ts.dqkv16[l]), 384, p->wsh(lp.qkv.kernel), 128, Mp)) return SMD_ERR_CUDA;
    }
  } else {
    if (!make_dw(&ts.dWin, B16(w.xb), C, B16(ts.du16[0]), Md, Md, Mp)) return SMD_ERR_CUDA;
  }
  if (c.arch == SMD_ARCH_DENSE_NCSN) {   // tangent halves of the sliced-score-matching backward
    ts.tdWb.resize(K); ts.tdXb.resize(K); ts.tdWa.resize(K); ts.tdXa.resize(K);
    for (int k = 0; k < K; ++k) {
      const BlockParams& bp = par.block[k];
      if (!make_dw(&ts.tdWb[k], B16(w.actt[2 * k + 1]), Md, B16(ts.dut16[k + 1]), Md, Md, Mp, true)) return SMD_ERR_CUDA;
      if (!make_dx(&ts.tdXb[k], B16(ts.dut16[k + 1]), Md, p->wsh(bp.b.kernel), Md, Mp, true)) return SMD_ERR_CUDA;
      if (!make_dw(&ts.tdWa[k], B16(w.actt[2 * k]), Md, B16(ts.drt16[k]), Md, Md, Mp, true)) return SMD_ERR_CUDA;
      if (!make_dx(&ts.tdXa[k], B16(ts.drt16[k]), Md, p->wsh(bp.a.kernel), Md, Mp, true)) return SMD_ERR_CUDA;
    }
    if (!make_gemm_op(&ts.tdWout, B16(w.actt[2 * K]), static_cast<uint64_t>(Md), B16(ts.dpredt16), static_cast<uint64_t>(Cp),
                      C, static_cast<int>(Mp), std::min(Cp, kBNMax), 1, 1))
      return SMD_ERR_CUDA;
    if (!make_gemm_op(&ts.tdXout, B16(ts.dpredt16), Mp, B16(w.out_pad), static_cast<uint64_t>(Md), Md, Cp,
                      choose_bn(Md), 0, 0)) return SMD_ERR_CUDA;
    if (!make_dw(&ts.tdWin, B16(w.xbt), C, B16(ts.dut16[0]), Md, Md, Mp)) return SMD_ERR_CUDA;
  }
  if (p->mdn()) return mdn_train_bind(p);
  return SMD_OK;
}

cudaError_t gemm_k(const GemmOp& op0, int rows, int K, int splits, const GemmEpilogue& e, cudaStream_t st) {
  GemmOp op = op0;
  op.K = K;
  op.k_splits = splits;
  return launch_gemm(op, rows, e, st);
}

// FiLM generator backward of block k (models/ncsn.py:47-61); no gradient flows into t.  Independent of the rest of the
// backward pass: runs on the side stream once this block's dss (complete on `st`) is.
static cudaError_t film_generator_bwd(smd_plan* p, const float* params, int k, int batch, float* grads, cudaStream_t st) {
  TrainState& ts = p->train;
  const WorkspaceLayout& w = p->reg;
  const BlockParams& bp = p->par.block[k];
  const int Md = p->cfg.mlp_dims;
  const int Bk = (batch + 63) / 64 * 64;
  cudaStream_t side = p->side_stream;
  auto B16 = [&](size_t off) { return p->at<__nv_bfloat16>(off); };
  auto F32 = [&](size_t off) { return p->at<float>(off); };
  float* dss = F32(ts.dss) + static_cast<size_t>(k) * p->cfg.max_batch * 2 * Md;
  cudaError_t err = cudaEventRecord(p->ev_dss, st);
  if (err == cudaSuccess) err = cudaStreamWaitEvent(side, p->ev_dss, 0);
  if (err != cudaSuccess) return err;
  float* enc = F32(w.enc);
  float* e1pre = F32(w.e1pre[k]);
  float* e1 = F32(w.e1[k]);
  float* e2 = F32(w.e2[k]);
  float* de2 = F32(ts.de2);
  float* de1 = F32(ts.de);
  launch_colsum<float>(dss, 2 * Md, grads + bp.film.ss.bias, batch, 2 * Md, side); CNT();
  launch_cast_bf16(dss, B16(ts.dss16), static_cast<size_t>(batch) * 2 * Md, side); CNT();
  launch_cast_bf16(e2, B16(ts.e2_16), static_cast<size_t>(batch) * 512, side); CNT();
  GemmEpilogue e = epi();
  e.out_f32 = grads + bp.film.ss.kernel; e.ld_f32 = 2 * Md;
  err = gemm_k(ts.dWss[k], 512, Bk, 1, e, side);
  if (err != cudaSuccess) return err;
  e = epi();
  e.out_f32 = de2; e.ld_f32 = 512;
  err = launch_gemm(ts.dXss[k], batch, e, side);
  if (err != cudaSuccess) return err;
  launch_colsum<float>(de2, 512, grads + bp.film.d2.bias, batch, 512, side); CNT();
  launch_small_linear_bwd_w(e1, de2, grads + bp.film.d2.kernel, batch, 512, 512, side); CNT();
  launch_small_linear_bwd_x(de2, params + bp.film.d2.kernel, e1pre, de1, batch, 512, 512, side); CNT();
  launch_colsum<float>(de1, 512, grads + bp.film.d1.bias, batch, 512, side); CNT();
  launch_small_linear_bwd_w(enc, de1, grads + bp.film.d1.kernel, batch, 128, 512, side); CNT();
  return cudaSuccess;
}

void launch_colsum_bf16(const __nv_bfloat16* in, int ld, float* out, int M, int N, cudaStream_t st) {
  launch_colsum<__nv_bfloat16>(in, ld, out, M, N, st);
}

cudaError_t fork_dw(smd_plan* p, cudaStream_t st) {
  // Weight-gradient GEMMs are leaves of the backward graph: they run on dw_stream next to the dX chain; every gradient
  // operand they read has its own buffer, so nothing they read is rewritten within this backward pass.
  cudaError_t e1 = cudaEventRecord(p->ev_dw, st);
  if (e1 != cudaSuccess) return e1;
  return cudaStreamWaitEvent(p->dw_stream, p->ev_dw, 0);
}

int bwd_begin(smd_plan* p, int M, int batch, float* grads, cudaStream_t st, bool tangent) {
  TrainState& ts = p->train;
  const smd_config& c = p->cfg;
  const int Md = c.mlp_dims, K = p->K, L = p->L;
  const int Mk = (M + 63) / 64 * 64;           // reduction length of the dW GEMMs
  const int Bk = (batch + 63) / 64 * 64;
  auto B16 = [&](size_t off) { return p->at<__nv_bfloat16>(off); };
  // Zeroing the 100 MB gradient arena (~20 us) goes to the weight-gradient stream: the forward pass does not touch it
  // and every writer either runs on that stream or is ordered after ev_gz below.
  SMD_CUDA(fork_dw(p, st));
  SMD_CUDA(cudaMemsetAsync(grads, 0, sizeof(float) * p->arena, p->dw_stream));
  SMD_CUDA(cudaEventRecord(p->ev_gz, p->dw_stream));
  // FiLM (scale|shift) gradients are accumulated with atomics by the two CTAs of a sample and by both uses of a pair
  if (!p->mdn())
    SMD_CUDA(cudaMemsetAsync(p->at<float>(ts.dss), 0, sizeof(float) * static_cast<size_t>(K) * c.max_batch * 2 * Md, st));
  if (Mk != M) {  // zero the reduction-tail rows of every MN-major gradient operand
    const size_t tail = static_cast<size_t>(Mk - M);
    for (size_t off : ts.du16) SMD_CUDA(cudaMemsetAsync(B16(off) + static_cast<size_t>(M) * Md, 0, tail * Md * 2, st));
    for (size_t off : ts.dr16t) SMD_CUDA(cudaMemsetAsync(B16(off) + static_cast<size_t>(M) * Md, 0, tail * Md * 2, st));
    if (tangent) {
      for (size_t off : ts.dut16) SMD_CUDA(cudaMemsetAsync(B16(off) + static_cast<size_t>(M) * Md, 0, tail * Md * 2, st));
      for (size_t off : ts.drt16) SMD_CUDA(cudaMemsetAsync(B16(off) + static_cast<size_t>(M) * Md, 0, tail * Md * 2, st));
    }
    for (int l = 0; l < L; ++l) {
      SMD_CUDA(cudaMemsetAsync(B16(ts.dh16a[l]) + static_cast<size_t>(M) * 128, 0, tail * 128 * 2, st));
      SMD_CUDA(cudaMemsetAsync(B16(ts.dh16b[l]) + static_cast<size_t>(M) * 128, 0, tail * 128 * 2, st));
      SMD_CUDA(cudaMemsetAsync(B16(ts.dr16[l]) + static_cast<size_t>(M) * Md, 0, tail * Md * 2, st));
      SMD_CUDA(cudaMemsetAsync(B16(ts.dqkv16[l]) + static_cast<size_t>(M) * 384, 0, tail * 384 * 2, st));
    }
    SMD_CUDA(cudaMemsetAsync(B16(ts.dpred16) + static_cast<size_t>(M) * p->head_ld, 0, tail * p->head_ld * 2, st));
    if (tangent)
      SMD_CUDA(cudaMemsetAsync(B16(ts.dpredt16) + static_cast<size_t>(M) * p->head_ld, 0, tail * p->head_ld * 2, st));
  }
  if (Bk != batch && !p->mdn()) {
    SMD_CUDA(cudaMemsetAsync(B16(ts.dss16) + static_cast<size_t>(batch) * 2 * Md, 0,
                             static_cast<size_t>(Bk - batch) * 2 * Md * 2, st));
    SMD_CUDA(cudaMemsetAsync(B16(ts.e2_16) + static_cast<size_t>(batch) * 512, 0,
                             static_cast<size_t>(Bk - batch) * 512 * 2, st));
  }
  return SMD_OK;
}

int bwd_out_ln(smd_plan* p, const float* params, int M, float* grads, cudaStream_t st) {
  TrainState& ts = p->train;
  const ParamLayout& par = p->par;
  const int K = p->K;
  GemmEpilogue e = epi();
  e.out_bf16 = p->at<__nv_bfloat16>(ts.g16); e.ld_bf16 = p->cfg.mlp_dims;
  SMD_CUDA(launch_gemm(ts.dXout, M, e, st));
  LnFilmBwdArgs a;
  memset(&a, 0, sizeof(a));
  a.g16 = p->at<__nv_bfloat16>(ts.g16); a.u = p->at<float>(p->reg.u[K]);
  a.stats = p->at<float>(p->reg.stats) + (2 * K) * static_cast<size_t>(p->Mp) * 2;
  a.gamma = params + par.out_ln.scale; a.beta = params + par.out_ln.bias;
  a.dx32 = p->at<float>(ts.du32); a.dx16 = p->at<__nv_bfloat16>(ts.du16[K]);
  a.dgamma = grads + par.out_ln.scale; a.dbeta = grads + par.out_ln.bias;
  a.dbias = grads + par.block[K - 1].b.bias;
  a.M = M; a.N = p->cfg.mlp_dims; a.S = p->cfg.seq_len;
  launch_ln_film_act_bwd(a, st); CNT();
  return SMD_OK;
}

// Every k*. / out_ln / output-layer gradient is final once the three events recorded with `ext` have fired
// (smd_wait_tail_grads).  When the call is being captured into a CUDA graph they are EXTERNAL event nodes, so a stream
// outside the graph can wait on them.  Without a FiLM generator the side stream has no work of its own and joins here
// (a captured graph records events only on streams that take part in the capture).
static int bwd_tail_done(smd_plan* p, cudaStream_t st, bool capturing) {
  const unsigned ext = capturing ? cudaEventRecordExternal : cudaEventRecordDefault;
  if (p->mdn()) {
    SMD_CUDA(cudaEventRecord(p->ev_fork, st));
    SMD_CUDA(cudaStreamWaitEvent(p->side_stream, p->ev_fork, 0));
  }
  SMD_CUDA(cudaEventRecordWithFlags(p->evx_join, p->side_stream, ext));
  SMD_CUDA(cudaEventRecord(p->ev_join, p->side_stream));   // internal join marker (last node of the side stream: `st` waits on it)
  SMD_CUDA(cudaEventRecordWithFlags(p->ev_tail, st, ext));
  SMD_CUDA(cudaEventRecordWithFlags(p->ev_dwtail, p->dw_stream, ext));
  SMD_LAUNCH_CHECK("backward tail");
  return SMD_OK;
}

int bwd_tail(smd_plan* p, const float* params, int batch, float* grads, cudaStream_t st, bool capturing) {
  TrainState& ts = p->train;
  const smd_config& c = p->cfg;
  const int S = c.seq_len, Md = c.mlp_dims;
  const int M = batch * S;
  const int Mk = (M + 63) / 64 * 64;
  const WorkspaceLayout& w = p->reg;
  const ParamLayout& par = p->par;
  const int K = p->K, L = p->L;
  const bool film = !p->mdn();
  auto B16 = [&](size_t off) { return p->at<__nv_bfloat16>(off); };
  auto F32 = [&](size_t off) { return p->at<float>(off); };
  cudaStream_t dws = p->dw_stream;
  __nv_bfloat16* g16 = B16(ts.g16);
  float* du32 = F32(ts.du32);
  float* stats = F32(w.stats);
  const size_t sstride = static_cast<size_t>(p->Mp) * 2;
  float* ssbuf = F32(w.ss);
  float* dss_all = F32(ts.dss);
  for (int k = K - 1; k >= 0; --k) {
    const BlockParams& bp = par.block[k];
    // (TransformerMDN: the identity FiLM rows smd_bind_workspace wrote into block 0, no FiLM gradient)
    const float* ss_k = film ? ssbuf + static_cast<size_t>(k) * c.max_batch * 2 * Md : ssbuf;
    float* dss = film ? dss_all + static_cast<size_t>(k) * c.max_batch * 2 * Md : nullptr;
    SMD_CUDA(fork_dw(p, st));
    GemmEpilogue e = epi();
    e.out_f32 = grads + bp.b.kernel; e.ld_f32 = Md;
    SMD_CUDA(gemm_k(ts.dWb[k], Md, Mk, 1, e, dws));
    e = epi();
    e.out_bf16 = g16; e.ld_bf16 = Md;
    SMD_CUDA(launch_gemm(ts.dXb[k], M, e, st));
    LnFilmBwdArgs a;
    memset(&a, 0, sizeof(a));
    a.g16 = g16; a.u16 = B16(w.r1[k]); a.stats = stats + (2 * k + 1) * sstride;
    a.gamma = params + bp.ln_b.scale; a.beta = params + bp.ln_b.bias;
    a.ss = ss_k; a.act = 2;
    a.dx32 = nullptr; a.dx16 = B16(ts.dr16t[k]);   // dr1 is only consumed as a bf16 GEMM operand
    a.dgamma = grads + bp.ln_b.scale; a.dbeta = grads + bp.ln_b.bias;
    a.dbias = grads + bp.a.bias;
    a.dss = dss; a.dss_accum = 0;
    a.M = M; a.N = Md; a.S = S;
    launch_ln_film_act_bwd(a, st); CNT();
    SMD_CUDA(fork_dw(p, st));
    e = epi();
    e.out_f32 = grads + bp.a.kernel; e.ld_f32 = Md;
    SMD_CUDA(gemm_k(ts.dWa[k], Md, Mk, 1, e, dws));
    e = epi();
    e.out_bf16 = g16; e.ld_bf16 = Md;
    SMD_CUDA(launch_gemm(ts.dXa[k], M, e, st));
    memset(&a, 0, sizeof(a));
    a.g16 = g16; a.u = F32(w.u[k]); a.stats = stats + (2 * k) * sstride;
    a.gamma = params + bp.ln_a.scale; a.beta = params + bp.ln_a.bias;
    a.ss = ss_k; a.act = 2;
    a.dres = du32; a.dx32 = du32; a.dx16 = B16(ts.du16[k]);
    a.dgamma = grads + bp.ln_a.scale; a.dbeta = grads + bp.ln_a.bias;
    a.dbias = grads + (k > 0 ? par.block[k - 1].b.bias : L ? par.post.bias : par.in.bias);
    a.dss = dss; a.dss_accum = 1;
    a.M = M; a.N = Md; a.S = S;
    launch_ln_film_act_bwd(a, st); CNT();

    if (film) SMD_CUDA(film_generator_bwd(p, params, k, batch, grads, st));
  }
  return bwd_tail_done(p, st, capturing);
}

int bwd_trunk(smd_plan* p, const float* params, int batch, float* grads, cudaStream_t st) {
  TrainState& ts = p->train;
  const smd_config& c = p->cfg;
  const int S = c.seq_len, C = c.channels, Md = c.mlp_dims;
  const int M = batch * S;
  const int Mk = (M + 63) / 64 * 64;
  const int nkb = Mk / 64;
  const WorkspaceLayout& w = p->reg;
  const ParamLayout& par = p->par;
  const int L = p->L;
  auto B16 = [&](size_t off) { return p->at<__nv_bfloat16>(off); };
  auto F32 = [&](size_t off) { return p->at<float>(off); };
  cudaStream_t dws = p->dw_stream;
  // ---------------- post dense + post LayerNorm ----------------
  float* da32 = F32(ts.dh2);
  float* dh32 = F32(ts.dh);
  // (the trunk's weight-gradient GEMMs and bias column sums go to dw_stream as well, with a reduced CTA count, while
  // the dX chain -- the critical path, mostly 32-CTA launches -- keeps `st`)
  {
    GemmEpilogue e = epi();
    e.out_f32 = grads + par.post.kernel; e.ld_f32 = Md;
    const int sp = pick_splits_side(128, Md, ts.dWpost.BN, nkb);
    e.atomic_out = sp > 1;
    SMD_CUDA(fork_dw(p, st));
    SMD_CUDA(gemm_k(ts.dWpost, 128, Mk, sp, e, dws));
    e = epi();
    e.out_f32 = da32; e.ld_f32 = 128;
    SMD_CUDA(launch_gemm(ts.dXpost, M, e, st));
    Ln128BwdArgs a;
    memset(&a, 0, sizeof(a));
    a.g = da32; a.h = F32(w.h[2 * L]); a.gamma = params + par.post_ln.scale;
    a.dx32 = dh32; a.dx16 = B16(ts.dh16a[L - 1]);
    a.dgamma = grads + par.post_ln.scale; a.dbeta = grads + par.post_ln.bias;
    a.dbias = grads + par.layer[L - 1].ffn2.bias;
    a.M = M;
    launch_ln128_bwd(a, st); CNT();
  }

  // ---------------- transformer trunk ----------------
  for (int l = L - 1; l >= 0; --l) {
    const LayerParams& lp = par.layer[l];
    __nv_bfloat16* dr16l = B16(ts.dr16[l]);
    // FFN: h_out = gelu(a2 W1 + b1) W2 + b2 + h_mid
    GemmEpilogue e = epi();
    e.out_bf16 = dr16l; e.ld_bf16 = Md;
    e.gelu_grad_of = B16(w.hidden_pre[l]); e.ld_gg = Md;
    SMD_CUDA(launch_gemm(ts.dX2[l], M, e, st));
    SMD_CUDA(fork_dw(p, st));
    e = epi();
    e.out_f32 = grads + lp.ffn2.kernel; e.ld_f32 = 128;
    int sp = pick_splits_side(Md, 128, ts.dW2[l].BN, nkb);
    e.atomic_out = sp > 1;
    SMD_CUDA(gemm_k(ts.dW2[l], Md, Mk, sp, e, dws));
    launch_colsum<__nv_bfloat16>(dr16l, Md, grads + lp.ffn1.bias, M, Md, dws); CNT();
    e = epi();
    e.out_f32 = grads + lp.ffn1.kernel; e.ld_f32 = Md;
    sp = pick_splits_side(128, Md, ts.dW1[l].BN, nkb);
    e.atomic_out = sp > 1;
    SMD_CUDA(gemm_k(ts.dW1[l], 128, Mk, sp, e, dws));
    e = epi();
    e.out_f32 = da32; e.ld_f32 = 128;
    SMD_CUDA(launch_gemm(ts.dX1[l], M, e, st));
    Ln128BwdArgs a;
    memset(&a, 0, sizeof(a));
    a.g = da32;
    a.h = F32(w.h[2 * l + 1]); a.gamma = params + lp.ln2.scale;
    a.dres = dh32; a.dx32 = dh32; a.dx16 = B16(ts.dh16b[l]);
    a.dgamma = grads + lp.ln2.scale; a.dbeta = grads + lp.ln2.bias;
    a.dbias = grads + lp.out.bias;
    a.M = M;
    launch_ln128_bwd(a, st); CNT();
    // attention: h_mid = attn(a1) Wo + bo + h_in
    SMD_CUDA(fork_dw(p, st));
    e = epi();
    e.out_f32 = grads + lp.out.kernel; e.ld_f32 = 128;
    sp = pick_splits_side(128, 128, ts.dWo[l].BN, nkb);
    e.atomic_out = sp > 1;
    SMD_CUDA(gemm_k(ts.dWo[l], 128, Mk, sp, e, dws));
    e = epi();
    e.out_f32 = da32; e.ld_f32 = 128;
    SMD_CUDA(launch_gemm(ts.dXo[l], M, e, st));
    SMD_CUDA(launch_attention_bwd(F32(w.qkv[l]), F32(w.probs[l]), da32, B16(ts.dqkv16[l]), grads + lp.qkv.bias,
                                  batch, S, c.num_heads, st));
    CNT();
    SMD_CUDA(fork_dw(p, st));
    e = epi();
    e.out_f32 = grads + lp.qkv.kernel; e.ld_f32 = 384;
    sp = pick_splits_side(128, 384, ts.dWqkv[l].BN, nkb);
    e.atomic_out = sp > 1;
    SMD_CUDA(gemm_k(ts.dWqkv[l], 128, Mk, sp, e, dws));
    e = epi();
    e.out_f32 = da32; e.ld_f32 = 128;
    SMD_CUDA(launch_gemm(ts.dXqkv[l], M, e, st));
    memset(&a, 0, sizeof(a));
    a.g = da32; a.h = F32(w.h[2 * l]); a.gamma = params + lp.ln1.scale;
    a.dres = dh32; a.dx32 = dh32; a.dx16 = (l > 0) ? B16(ts.dh16a[l - 1]) : nullptr;
    a.dgamma = grads + lp.ln1.scale; a.dbeta = grads + lp.ln1.bias;
    a.dbias = grads + (l > 0 ? par.layer[l - 1].ffn2.bias : par.in.bias);
    a.M = M;
    launch_ln128_bwd(a, st); CNT();
  }
  SMD_CUDA(cudaEventRecord(p->ev_dwjoin, dws));
  // ---------------- input projection ----------------
  launch_embed_bwd(F32(w.xt), dh32, grads + par.in.kernel, M, C, st); CNT();
  SMD_CUDA(cudaStreamWaitEvent(st, p->ev_dwjoin, 0));
  SMD_CUDA(cudaStreamWaitEvent(st, p->ev_join, 0));
  SMD_LAUNCH_CHECK("backward trunk");
  return SMD_OK;
}

}  // namespace smd

using namespace smd;

// DenseDDPM / DenseNCSN (no trunk): the input projection's weight gradient (models/ncsn.py:129) -- with tangent, plus
// the product over the tangent rows x~ and v -- then the joins of the weight-gradient and side streams.
static int bwd_dense_in(smd_plan* p, int M, float* grads, cudaStream_t st, bool tangent) {
  const int Md = p->cfg.mlp_dims, C = p->cfg.channels;
  const int Mk = (M + 63) / 64 * 64;
  float* dw = grads + p->par.in.kernel;
  GemmEpilogue e = epi();
  e.out_f32 = dw; e.ld_f32 = Md;
  SMD_CUDA(gemm_k(p->train.dWin, C, Mk, 1, e, st));
  if (tangent) {
    e.residual = dw; e.ld_res = Md;
    SMD_CUDA(gemm_k(p->train.tdWin, C, Mk, 1, e, st));
  }
  SMD_CUDA(cudaEventRecord(p->ev_dwjoin, p->dw_stream));
  SMD_CUDA(cudaStreamWaitEvent(st, p->ev_dwjoin, 0));
  SMD_CUDA(cudaStreamWaitEvent(st, p->ev_join, 0));
  SMD_LAUNCH_CHECK("backward dense");
  return SMD_OK;
}

// DDPM or denoising score matching.  ind: device table {x0, used_alpha, eps} read by the kernels instead of the pointer
// arguments (graph replay), or null.
static int grads_impl(smd_plan* p, const float* params, const float* x0, const float* used_alpha, const float* eps,
                      const float* const* ind, int batch, int global_batch, float* grads, float* loss_sum,
                      cudaStream_t st, bool capturing, Objective objective) {
  TrainState& ts = p->train;
  const smd_config& c = p->cfg;
  const int S = c.seq_len, C = c.channels, Md = c.mlp_dims;
  const int Cp = (C + 63) / 64 * 64;
  const int M = batch * S;
  const int Mk = (M + 63) / 64 * 64;           // reduction length of the dW GEMMs
  const int per = S * C;
  const WorkspaceLayout& w = p->reg;
  const ParamLayout& par = p->par;
  const int L = p->L;
  auto B16 = [&](size_t off) { return p->at<__nv_bfloat16>(off); };
  auto F32 = [&](size_t off) { return p->at<float>(off); };

  { int rcs = ensure_side_stream(p); if (rcs) return rcs; }
  cudaStream_t dws = p->dw_stream;
  const int nkb = Mk / 64;
  float* xt = F32(w.xt);
  int rc = bwd_begin(p, M, batch, grads, st);
  if (rc) return rc;

  // ---------------- forward (keeps every activation) ----------------
  float* cond = F32(w.tvec);
  float* pred = F32(w.eps_hat);
  launch_q_sample(x0, eps, used_alpha, xt, cond, batch, per, st, ind, objective); CNT();
  rc = run_forward(p, params, xt, cond, 0, batch, pred, st, /*save=*/true, /*raw_out=*/true);
  if (rc) return rc;
  SMD_CUDA(cudaStreamWaitEvent(st, p->ev_gz, 0));   // gradient arena zeroed (long done by now)

  // ---------------- objective ----------------
  // ddpm: mean over (S, C) and the global batch; dsm: sum over (S, C) (x 0.5), mean over the global batch
  const float gscale = objective == kObjDsm ? 1.0f / static_cast<float>(global_batch)
                                           : 1.0f / (static_cast<float>(global_batch) * static_cast<float>(per));
  float* dpred32 = F32(ts.dpred32);
  __nv_bfloat16* dpred16 = B16(ts.dpred16);
  ddpm_loss_bwd_kernel<<<batch, 256, 0, st>>>(eps, pred, F32(ts.loss), loss_sum, p->at<unsigned int>(ts.loss_ctr),
                                              1.0f / static_cast<float>(global_batch), dpred32, dpred16, gscale, S, C, Cp,
                                              ind, objective);
  CNT();
  SMD_CUDA(fork_dw(p, st));
  launch_colsum<float>(dpred32, C, grads + par.out.bias, M, C, dws); CNT();

  // ---------------- output projection + final LayerNorm ----------------
  {
    GemmEpilogue e = epi();
    e.out_f32 = grads + par.out.kernel; e.ld_f32 = C;
    const int sp = pick_splits_side(Md, C, ts.dWout.BN, nkb);
    e.atomic_out = sp > 1;
    SMD_CUDA(gemm_k(ts.dWout, Md, Mk, sp, e, dws));
  }
  rc = bwd_out_ln(p, params, M, grads, st);
  if (rc) return rc;

  // ---------------- FiLM'd residual blocks ----------------
  rc = bwd_tail(p, params, batch, grads, st, capturing);
  if (rc) return rc;
  return L == 0 ? bwd_dense_in(p, M, grads, st, false) : bwd_trunk(p, params, batch, grads, st);
}

// Sliced score matching (utils/losses.py:182-247) on DenseNCSN: loss_b = 0.5 |f|^2 + sigma v.(J_f v) with f the raw
// network output.  The primal pass and its tangent along v (run_forward with tangent) are differentiated together in
// reverse mode ("reverse over forward"): every dX GEMM runs once on the primal and once on the tangent adjoint, every
// dW GEMM accumulates the primal and the tangent products, and the LayerNorm / FiLM / swish steps use ssm_ln_bwd.
// ind: device table {x0, used_sigma, eps, v} (graph replay) or null.
static int ssm_grads_impl(smd_plan* p, const float* params, const float* x0, const float* used_sigma, const float* eps,
                          const float* v, const float* const* ind, int batch, int global_batch, float* grads,
                          float* loss_sum, cudaStream_t st, bool capturing) {
  TrainState& ts = p->train;
  const smd_config& c = p->cfg;
  const int C = c.channels, Md = c.mlp_dims;
  const int Cp = (C + 63) / 64 * 64;
  const int M = batch;
  const int Mk = (M + 63) / 64 * 64;
  const WorkspaceLayout& w = p->reg;
  const ParamLayout& par = p->par;
  const int K = p->K;
  auto B16 = [&](size_t off) { return p->at<__nv_bfloat16>(off); };
  auto F32 = [&](size_t off) { return p->at<float>(off); };
  { int rcs = ensure_side_stream(p); if (rcs) return rcs; }
  cudaStream_t dws = p->dw_stream;
  // weight gradient = primal product + tangent product (reduction over both sets of rows), on the weight-gradient stream
  auto dw2 = [&](const GemmOp& op, const GemmOp& top, int rows, float* out, int ld) -> cudaError_t {
    GemmEpilogue e = epi();
    e.out_f32 = out; e.ld_f32 = ld;
    cudaError_t err = gemm_k(op, rows, Mk, 1, e, dws);
    if (err != cudaSuccess) return err;
    e.residual = out; e.ld_res = ld;
    return gemm_k(top, rows, Mk, 1, e, dws);
  };
  auto dx = [&](const GemmOp& op, __nv_bfloat16* out) -> cudaError_t {
    GemmEpilogue e = epi();
    e.out_bf16 = out; e.ld_bf16 = Md;
    return launch_gemm(op, M, e, st);
  };
  __nv_bfloat16* g16 = B16(ts.g16);
  __nv_bfloat16* gt16 = B16(ts.gt16);
  float* du32 = F32(ts.du32);
  float* dut32 = F32(ts.dut32);
  float* stats = F32(w.stats);
  const size_t sstride = static_cast<size_t>(p->Mp) * 2;
  int rc = bwd_begin(p, M, batch, grads, st, /*tangent=*/true);
  if (rc) return rc;

  // ---------------- forward: primal (keeps every activation) and tangent along v ----------------
  float* xt = F32(w.xt);
  float* cond = F32(w.tvec);
  float* f = F32(w.eps_hat);
  launch_q_sample(x0, eps, used_sigma, xt, cond, batch, C, st, ind, kObjDsm); CNT();   // x~ = x0 + sigma eps
  launch_tangent_input(v, ind, B16(w.xbt), static_cast<size_t>(M) * C, st, 0); CNT();
  rc = run_forward(p, params, xt, cond, 0, batch, f, st, /*save=*/true, /*raw_out=*/true, /*tangent=*/true);
  if (rc) return rc;
  SMD_CUDA(cudaStreamWaitEvent(st, p->ev_gz, 0));

  // ---------------- objective and its two adjoint seeds ----------------
  float* dpred32 = F32(ts.dpred32);
  launch_ssm_loss(f, F32(w.yt), v, used_sigma, ind, F32(ts.loss), nullptr, nullptr, loss_sum,
                  p->at<unsigned int>(ts.loss_ctr), 1.0f / static_cast<float>(global_batch), dpred32, B16(ts.dpred16),
                  B16(ts.dpredt16), batch, C, Cp, st); CNT();
  SMD_CUDA(fork_dw(p, st));
  launch_colsum<float>(dpred32, C, grads + par.out.bias, M, C, dws); CNT();

  // ---------------- output projection + final LayerNorm ----------------
  SMD_CUDA(dw2(ts.dWout, ts.tdWout, Md, grads + par.out.kernel, C));
  SMD_CUDA(dx(ts.dXout, g16));
  SMD_CUDA(dx(ts.tdXout, gt16));
  SsmLnBwdArgs a;
  memset(&a, 0, sizeof(a));
  a.x32 = F32(w.u[K]); a.xt = F32(w.ut[K]); a.stats = stats + (2 * K) * sstride;
  a.gamma = params + par.out_ln.scale; a.beta = params + par.out_ln.bias;
  a.g16 = g16; a.gt16 = gt16;
  a.dx32 = du32; a.dx16 = B16(ts.du16[K]); a.dxt32 = dut32; a.dxt16 = B16(ts.dut16[K]);
  a.dgamma = grads + par.out_ln.scale; a.dbeta = grads + par.out_ln.bias;
  a.dbias = grads + par.block[K - 1].b.bias;
  a.M = M; a.N = Md; a.S = 1;
  launch_ssm_ln_bwd(a, st); CNT();

  // ---------------- FiLM'd residual blocks ----------------
  for (int k = K - 1; k >= 0; --k) {
    const BlockParams& bp = par.block[k];
    const float* ss_k = F32(w.ss) + static_cast<size_t>(k) * c.max_batch * 2 * Md;
    float* dss = F32(ts.dss) + static_cast<size_t>(k) * c.max_batch * 2 * Md;
    SMD_CUDA(fork_dw(p, st));
    SMD_CUDA(dw2(ts.dWb[k], ts.tdWb[k], Md, grads + bp.b.kernel, Md));
    SMD_CUDA(dx(ts.dXb[k], g16));
    SMD_CUDA(dx(ts.tdXb[k], gt16));
    memset(&a, 0, sizeof(a));
    a.x16 = B16(w.r1[k]); a.xt = F32(w.r1t[k]); a.stats = stats + (2 * k + 1) * sstride;
    a.gamma = params + bp.ln_b.scale; a.beta = params + bp.ln_b.bias;
    a.ss = ss_k; a.act = 2;
    a.g16 = g16; a.gt16 = gt16;
    a.dx16 = B16(ts.dr16t[k]); a.dxt16 = B16(ts.drt16[k]);
    a.dgamma = grads + bp.ln_b.scale; a.dbeta = grads + bp.ln_b.bias;
    a.dbias = grads + bp.a.bias;
    a.dss = dss;
    a.M = M; a.N = Md; a.S = 1;
    launch_ssm_ln_bwd(a, st); CNT();
    SMD_CUDA(fork_dw(p, st));
    SMD_CUDA(dw2(ts.dWa[k], ts.tdWa[k], Md, grads + bp.a.kernel, Md));
    SMD_CUDA(dx(ts.dXa[k], g16));
    SMD_CUDA(dx(ts.tdXa[k], gt16));
    memset(&a, 0, sizeof(a));
    a.x32 = F32(w.u[k]); a.xt = F32(w.ut[k]); a.stats = stats + (2 * k) * sstride;
    a.gamma = params + bp.ln_a.scale; a.beta = params + bp.ln_a.bias;
    a.ss = ss_k; a.act = 2;
    a.g16 = g16; a.gt16 = gt16;
    a.dres = du32; a.dres_t = dut32;
    a.dx32 = du32; a.dx16 = B16(ts.du16[k]); a.dxt32 = dut32; a.dxt16 = B16(ts.dut16[k]);
    a.dgamma = grads + bp.ln_a.scale; a.dbeta = grads + bp.ln_a.bias;
    a.dbias = grads + (k > 0 ? par.block[k - 1].b.bias : par.in.bias);
    a.dss = dss;
    a.M = M; a.N = Md; a.S = 1;
    launch_ssm_ln_bwd(a, st); CNT();
    SMD_CUDA(film_generator_bwd(p, params, k, batch, grads, st));
  }
  rc = bwd_tail_done(p, st, capturing);
  if (rc) return rc;
  return bwd_dense_in(p, M, grads, st, /*tangent=*/true);
}

// v: the projection vectors of sliced score matching, else null.  TransformerMDN: x0 holds the sequences, used_alpha /
// eps are null.
static int grads_entry(smd_plan* p, const float* params, const float* x0, const float* used_alpha,
                       const float* eps, const float* v, int batch, int global_batch, float* grads, float* loss_sum,
                       smd_stream_t stream, Objective objective) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!p->cfg.training) { set_error("plan was not created with training = 1"); return SMD_ERR_STATE; }
  if (!p->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (batch < 1 || batch > p->cfg.max_batch || global_batch < batch) { set_error("batch out of range"); return SMD_ERR_INVALID; }
  auto impl = [&](const float* x0_, const float* ua_, const float* eps_, const float* v_, const float* const* ind_,
                  bool capturing) {
    if (objective == kObjSsm)
      return ssm_grads_impl(p, params, x0_, ua_, eps_, v_, ind_, batch, global_batch, grads, loss_sum, st, capturing);
    if (objective == kObjMdn) return mdn_grads_impl(p, params, x0_, ind_, batch, global_batch, grads, loss_sum, st, capturing);
    return grads_impl(p, params, x0_, ua_, eps_, ind_, batch, global_batch, grads, loss_sum, st, capturing, objective);
  };
  if (!capturable(st)) return impl(x0, used_alpha, eps, v, nullptr, false);
  // Graph replay: the pass's ~150 launches on three streams (dX chain, weight-gradient GEMMs, FiLM generator) are
  // captured once into one CUDA graph with the same fork / join structure.  The per-step inputs (x0, used_alpha, eps)
  // reach the kernels through a device pointer table, so new input tensors do not force a re-capture; the events a
  // data-parallel caller waits on (smd_wait_tail_grads) are external event-record nodes of the graph.
  const GraphKey key = graph_key(params, grads, loss_sum, batch, global_batch, objective);
  const float** ind = p->at<const float*>(p->train.ind);
  if (!p->train_graph.replays(key)) {
    p->train_graph.drop();
    const GraphKey warm = graph_key(params, batch, objective);
    if (p->train_warm != warm) {
      // first use of this configuration runs eagerly: lazy one-time calls (function attributes, stream / event
      // creation) stay out of the capture
      p->train_warm = warm;
      return impl(x0, used_alpha, eps, v, nullptr, false);
    }
    const int rc = p->train_graph.capture(
        st, key, [&] { return impl(nullptr, nullptr, nullptr, nullptr, ind, true); }, "train graph");
    if (rc) return rc;
  }
  // (pageable source: the driver stages these 32 bytes before returning, so the host array may die with this frame)
  const float* host_ind[4] = {x0, used_alpha, eps, v};
  SMD_CUDA(cudaMemcpyAsync(ind, host_ind, sizeof(host_ind), cudaMemcpyHostToDevice, st));
  return p->train_graph.launch(st);
}

extern "C" int smd_ddpm_grads(smd_plan* p, const float* params, const float* x0, const float* used_alpha,
                              const float* eps, int batch, int global_batch, float* grads, float* loss_sum,
                              smd_stream_t stream) {
  if (p->mdn()) { set_error("smd_ddpm_grads does not apply to a TransformerMDN plan (use smd_mdn_grads)"); return SMD_ERR_INVALID; }
  return grads_entry(p, params, x0, used_alpha, eps, nullptr, batch, global_batch, grads, loss_sum, stream, kObjDdpm);
}

// TransformerMDN (train_mdn.py:180-205): gradient of the mean token NLL; x is the only per-step input
extern "C" int smd_mdn_grads(smd_plan* p, const float* params, const float* x, int batch, int global_batch,
                             float* grads, float* loss_sum, smd_stream_t stream) {
  if (!p || !p->mdn()) { set_error("smd_mdn_grads needs a TransformerMDN plan (smd_mdn_plan_create)"); return SMD_ERR_INVALID; }
  return grads_entry(p, params, x, nullptr, nullptr, nullptr, batch, global_batch, grads, loss_sum, stream, kObjMdn);
}

// denoising score matching (utils/losses.py:129-179): the same pass with x~ = x0 + sigma eps, the network conditioned on
// sigma and the 0.5 (net + eps)^2 objective (for a network whose output is divided by sigma -- SMD_ARCH_DENSE_NCSN)
extern "C" int smd_dsm_grads(smd_plan* p, const float* params, const float* x0, const float* used_sigma,
                             const float* eps, int batch, int global_batch, float* grads, float* loss_sum,
                             smd_stream_t stream) {
  if (p->cfg.arch != SMD_ARCH_DENSE_NCSN) { set_error("smd_dsm_grads needs a score network (SMD_ARCH_DENSE_NCSN)"); return SMD_ERR_INVALID; }
  return grads_entry(p, params, x0, used_sigma, eps, nullptr, batch, global_batch, grads, loss_sum, stream, kObjDsm);
}

// sliced score matching (utils/losses.py:182-247) with the draws of smd_ssm_draws supplied (SMD_ARCH_DENSE_NCSN)
extern "C" int smd_ssm_grads(smd_plan* p, const float* params, const float* x0, const float* used_sigma,
                             const float* eps, const float* v, int batch, int global_batch, float* grads,
                             float* loss_sum, smd_stream_t stream) {
  if (p->cfg.arch != SMD_ARCH_DENSE_NCSN) { set_error("smd_ssm_grads needs a score network (SMD_ARCH_DENSE_NCSN)"); return SMD_ERR_INVALID; }
  return grads_entry(p, params, x0, used_sigma, eps, v, batch, global_batch, grads, loss_sum, stream, kObjSsm);
}

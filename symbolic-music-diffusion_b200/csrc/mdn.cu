// TransformerMDN, the reference's autoregressive baseline (models/autoregressive.py:37-82, train_mdn.py:100-205):
// the input shifted right by one position, the TransformerDDPM trunk with causal attention, res-blocks without FiLM
// (run_forward / the shared backward pieces) and a mixture-density head.  The head is one wgmma GEMM over the packed
// weight [mu | log_sigma | pi]; this file holds its packing, the mixture negative log-likelihood and its gradient, and
// the train-step body.
#include <cmath>

#include "plan.cuh"

namespace smd {

// xs[b][s] = x[b][s - 1], xs[b][0] = 0  (shift_right, models/autoregressive.py:25-33); ind (graph replay) overrides x
__global__ void mdn_shift_kernel(const float* __restrict__ x, const float* const* __restrict__ ind,
                                 float* __restrict__ xs, int B, int S, int C) {
  pdl_trigger();
  pdl_wait();
  if (ind) x = ind[0];
  const size_t per = static_cast<size_t>(S) * C, n = B * per;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    xs[i] = (i % per) < static_cast<size_t>(C) ? 0.0f : x[i - C];
}

struct MdnNllArgs {
  const float* pi; const float* mu; const float* ls;   // row r at pi + r * ld_pi, mu + r * ld_mu, ls + r * ld_ls
  int ld_pi, ld_mu, ld_ls;
  const float* x;              // targets [rows][C]
  const float* const* ind;     // graph replay: ind[0] overrides x
  int rows, C, Kc;
  float* loss;                 // [rows]
  // training (dz != null): dZ = d(sum of losses * gscale) / d(pi, mu, log_sigma) as bf16 into row r of dz at
  // columns off_mu + k C + c, off_ls + k C + c and off_pi + k; loss_sum as smd_ddpm_grads
  __nv_bfloat16* dz;
  int ld_dz, off_mu, off_ls, off_pi;
  float gscale;
  float* loss_sum;
  unsigned int* done_counter;
};

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float u = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, u) : v + u;
  }
  __syncthreads();   // red may still be read by the previous reduction
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = red[0];
  for (int w = 1; w < nw; ++w) r = is_max ? fmaxf(r, red[w]) : r + red[w];
  return r;
}

// Negative log-likelihood of MixtureSameFamily(Categorical(pi), MultivariateNormalDiag(mu, exp(log_sigma))) per row
// (train_mdn.py:100-133), one CTA per row, fp32 with accurate expf / logf:
//   lp_k = log_softmax(pi)_k + sum_c (-z^2 / 2 - log_sigma_kc) - (C / 2) log 2 pi,  z = (x_c - mu_kc) / sigma_kc
//   loss = -logsumexp_k lp_k;  with gamma = softmax(lp):  dmu = -gamma_k z / sigma,  dlog_sigma = gamma_k (1 - z^2),
//   dpi = softmax(pi) - gamma
__global__ void __launch_bounds__(256) mdn_nll_kernel(const MdnNllArgs a) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float mdn_sm[];
  float* xs = mdn_sm;          // [C] target row
  float* lp = xs + a.C;        // [Kc] component log densities (with the mixture weight)
  float* ep = lp + a.Kc;       // [Kc] exp(pi - max pi)
  __shared__ float red[32];
  __shared__ bool last;
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const int C = a.C, Kc = a.Kc;
  const float* x = (a.ind ? a.ind[0] : a.x) + static_cast<size_t>(r) * C;
  const float* pi = a.pi + static_cast<size_t>(r) * a.ld_pi;
  const float* mu = a.mu + static_cast<size_t>(r) * a.ld_mu;
  const float* ls = a.ls + static_cast<size_t>(r) * a.ld_ls;
  for (int c = tid; c < C; c += blockDim.x) xs[c] = x[c];
  float m = -INFINITY;
  for (int k = tid; k < Kc; k += blockDim.x) m = fmaxf(m, pi[k]);
  m = block_reduce(m, true, red);
  float se = 0.f;
  for (int k = tid; k < Kc; k += blockDim.x) { const float e = expf(pi[k] - m); ep[k] = e; se += e; }
  se = block_reduce(se, false, red);   // (its barriers also publish xs and ep)
  const float lse_pi = m + logf(se);
  const float norm = 0.5f * static_cast<float>(C) * 1.8378770664093453f;   // (C / 2) log(2 pi)
  for (int k = warp; k < Kc; k += nw) {
    float s = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float l = ls[static_cast<size_t>(k) * C + c];
      const float z = (xs[c] - mu[static_cast<size_t>(k) * C + c]) * expf(-l);
      s += -0.5f * z * z - l;
    }
    s = warp_sum(s);
    if (lane == 0) lp[k] = (pi[k] - lse_pi) + s - norm;
  }
  __syncthreads();
  float m2 = -INFINITY;
  for (int k = tid; k < Kc; k += blockDim.x) m2 = fmaxf(m2, lp[k]);
  m2 = block_reduce(m2, true, red);
  float s2 = 0.f;
  for (int k = tid; k < Kc; k += blockDim.x) s2 += expf(lp[k] - m2);
  s2 = block_reduce(s2, false, red);
  const float lse = m2 + logf(s2);
  if (tid == 0) a.loss[r] = -lse;
  if (a.dz) {
    __nv_bfloat16* dz = a.dz + static_cast<size_t>(r) * a.ld_dz;
    const float gs = a.gscale, inv_se = 1.0f / se;
    const int KC = Kc * C;
    for (int i = tid; i < KC; i += blockDim.x) {
      const int k = i / C, c = i - k * C;
      const float gam = expf(lp[k] - lse);
      const float inv_sig = expf(-ls[i]);
      const float z = (xs[c] - mu[i]) * inv_sig;
      dz[a.off_mu + i] = __float2bfloat16_rn(-gam * z * inv_sig * gs);
      dz[a.off_ls + i] = __float2bfloat16_rn(gam * (1.0f - z * z) * gs);
    }
    for (int k = tid; k < Kc; k += blockDim.x)
      dz[a.off_pi + k] = __float2bfloat16_rn((ep[k] * inv_se - expf(lp[k] - lse)) * gs);
  }
  if (!a.loss_sum) return;
  // as ddpm_loss_bwd_kernel: the block that finishes last adds the per-row losses in index order (bit-reproducible)
  if (tid == 0) {
    __threadfence();
    last = atomicInc(a.done_counter, gridDim.x - 1) == gridDim.x - 1;   // wraps back to 0 for the next launch
  }
  __syncthreads();
  if (last && tid < 32) {
    __threadfence();
    float acc = 0.f;
    for (int i = tid; i < static_cast<int>(gridDim.x); i += 32) acc += __ldcg(a.loss + i);
    acc = warp_sum(acc);
    if (tid == 0) { a.loss_sum[0] = acc; a.loss_sum[1] = acc * a.gscale; }
  }
}

static cudaError_t launch_mdn_nll(const MdnNllArgs& a, cudaStream_t st) {
  const size_t smem = static_cast<size_t>(a.C + 2 * a.Kc) * sizeof(float);
  mdn_nll_kernel<<<a.rows, 256, smem, st>>>(a); CNT();
  return cudaGetLastError();
}

static void launch_mdn_shift(const float* x, const float* const* ind, float* xs, int B, int S, int C, cudaStream_t st) {
  const size_t n = static_cast<size_t>(B) * S * C;
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > 148 * 8) blocks = 148 * 8;
  mdn_shift_kernel<<<blocks, 256, 0, st>>>(x, ind, xs, B, S, C); CNT();
}

// head-output columns of the three parts (offsets into the packed [mu | log_sigma | pi] width)
struct HeadParts { int off[3], cols[3]; const Dense* d[3]; };
static HeadParts head_parts(const smd_plan* p) {
  const int KC = p->Kc * p->cfg.channels;
  return HeadParts{{0, p->KCp, 2 * p->KCp}, {KC, KC, p->Kc},
                   {&p->par.mdn_mu, &p->par.mdn_log_sigma, &p->par.mdn_pi}};
}

// The bf16 head weight [Md][Np] and the fp32 bias [Np] from the three arena tensors (pad columns stay zero from bind).
int mdn_pack_head(smd_plan* p, const float* params, cudaStream_t st) {
  const HeadParts h = head_parts(p);
  __nv_bfloat16* w = p->at<__nv_bfloat16>(p->reg.out_pad);
  float* b = p->at<float>(p->reg.head_bias);
  for (int j = 0; j < 3; ++j) {
    launch_pad_cast_bf16(params + h.d[j]->kernel, w + h.off[j], p->cfg.mlp_dims, h.cols[j], p->head_ld, st); CNT();
    SMD_CUDA(cudaMemcpyAsync(b + h.off[j], params + h.d[j]->bias, static_cast<size_t>(h.cols[j]) * 4,
                             cudaMemcpyDeviceToDevice, st));
  }
  SMD_LAUNCH_CHECK("mdn pack head");
  return SMD_OK;
}

// dW of each part = act_out^T dZ[:, part]: B is a column slice of dZ, so its tensor map carries dZ's row pitch
int mdn_train_bind(smd_plan* p) {
  const HeadParts h = head_parts(p);
  const int Md = p->cfg.mlp_dims;
  const uint64_t Mp = p->Mp;
  __nv_bfloat16* act = p->at<__nv_bfloat16>(p->reg.act[2 * p->K]);
  __nv_bfloat16* dz = p->at<__nv_bfloat16>(p->train.dpred16);
  for (int j = 0; j < 3; ++j) {
    GemmOp& op = p->train.dWmdn[j];
    const int cols = h.cols[j];
    if (!make_gemm_op(&op, act, static_cast<uint64_t>(Md), dz + h.off[j], static_cast<uint64_t>(cols), cols,
                      static_cast<int>(Mp), std::min((cols + 63) / 64 * 64, kBNMax), 1, 1, 0, 0, 0,
                      static_cast<uint64_t>(p->head_ld)))
      return SMD_ERR_CUDA;
  }
  return SMD_OK;
}

static MdnNllArgs plan_nll_args(const smd_plan* p, const float* x, int rows, float* loss) {
  const HeadParts h = head_parts(p);
  const float* z = p->at<float>(p->reg.head);
  MdnNllArgs a;
  memset(&a, 0, sizeof(a));
  a.mu = z + h.off[0]; a.ls = z + h.off[1]; a.pi = z + h.off[2];
  a.ld_pi = a.ld_mu = a.ld_ls = p->head_ld;
  a.x = x; a.rows = rows; a.C = p->cfg.channels; a.Kc = p->Kc;
  a.loss = loss;
  return a;
}

static int mdn_check(const smd_plan* p, int batch, const char* fn) {
  if (!p || !p->mdn()) { set_error(std::string(fn) + " needs a TransformerMDN plan (smd_mdn_plan_create)"); return SMD_ERR_INVALID; }
  if (!p->ws) { set_error("workspace not bound"); return SMD_ERR_STATE; }
  if (batch < 1 || batch > p->cfg.max_batch) { set_error("batch out of range"); return SMD_ERR_INVALID; }
  return SMD_OK;
}

int mdn_grads_impl(smd_plan* p, const float* params, const float* x, const float* const* ind, int batch,
                   int global_batch, float* grads, float* loss_sum, cudaStream_t st, bool capturing) {
  TrainState& ts = p->train;
  const int S = p->cfg.seq_len, C = p->cfg.channels, Md = p->cfg.mlp_dims;
  const int M = batch * S;
  const int Mk = (M + 63) / 64 * 64;
  { int rcs = ensure_side_stream(p); if (rcs) return rcs; }
  int rc = bwd_begin(p, M, batch, grads, st);
  if (rc) return rc;
  // ---------------- forward on shift_right(x) (keeps every activation) ----------------
  float* xs = p->at<float>(p->reg.xt);
  launch_mdn_shift(x, ind, xs, batch, S, C, st);
  rc = run_forward(p, params, xs, nullptr, 0, batch, p->at<float>(p->reg.head), st, /*save=*/true);
  if (rc) return rc;
  SMD_CUDA(cudaStreamWaitEvent(st, p->ev_gz, 0));
  // ---------------- mixture NLL, its gradient dZ (bf16, scaled to the mean over the global tokens) ----------------
  const HeadParts h = head_parts(p);
  MdnNllArgs a = plan_nll_args(p, x, M, p->at<float>(ts.loss));
  a.ind = ind;
  a.dz = p->at<__nv_bfloat16>(ts.dpred16); a.ld_dz = p->head_ld;
  a.off_mu = h.off[0]; a.off_ls = h.off[1]; a.off_pi = h.off[2];
  a.gscale = 1.0f / (static_cast<float>(global_batch) * static_cast<float>(S));
  a.loss_sum = loss_sum; a.done_counter = p->at<unsigned int>(ts.loss_ctr);
  SMD_CUDA(launch_mdn_nll(a, st));
  // ---------------- head: bias = column sums of dZ, dW per part (weight-gradient stream), dX + out_ln ----------------
  SMD_CUDA(fork_dw(p, st));
  for (int j = 0; j < 3; ++j) {
    launch_colsum_bf16(a.dz + h.off[j], p->head_ld, grads + h.d[j]->bias, M, h.cols[j], p->dw_stream); CNT();
    GemmEpilogue e = epi();
    e.out_f32 = grads + h.d[j]->kernel; e.ld_f32 = h.cols[j];
    const int sp = pick_splits_side(Md, h.cols[j], ts.dWmdn[j].BN, Mk / 64);
    e.atomic_out = sp > 1;
    SMD_CUDA(gemm_k(ts.dWmdn[j], Md, Mk, sp, e, p->dw_stream));
  }
  rc = bwd_out_ln(p, params, M, grads, st);
  if (rc) return rc;
  // ---------------- res-blocks, then the causal trunk (the attention backward reads the saved probabilities,
  // exactly 0 above the diagonal, so the unmasked kernels apply) ----------------
  rc = bwd_tail(p, params, batch, grads, st, capturing);
  if (rc) return rc;
  return bwd_trunk(p, params, batch, grads, st);
}

}  // namespace smd

using namespace smd;

extern "C" {

int smd_mdn_forward(smd_plan* plan, const float* params, const float* x, int batch, int shift, float* pi, float* mu,
                    float* log_sigma, smd_stream_t stream) {
  int rc = mdn_check(plan, batch, "smd_mdn_forward");
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int S = plan->cfg.seq_len, C = plan->cfg.channels, M = batch * S;
  const float* xin = x;
  if (shift) {
    launch_mdn_shift(x, nullptr, plan->at<float>(plan->reg.xt), batch, S, C, st);
    xin = plan->at<float>(plan->reg.xt);
  }
  float* z = plan->at<float>(plan->reg.head);
  rc = run_forward(plan, params, xin, nullptr, 0, batch, z, st, false);
  if (rc) return rc;
  const HeadParts h = head_parts(plan);
  float* outs[3] = {mu, log_sigma, pi};
  for (int j = 0; j < 3; ++j)
    SMD_CUDA(cudaMemcpy2DAsync(outs[j], static_cast<size_t>(h.cols[j]) * 4, z + h.off[j],
                               static_cast<size_t>(plan->head_ld) * 4, static_cast<size_t>(h.cols[j]) * 4, M,
                               cudaMemcpyDeviceToDevice, st));
  SMD_LAUNCH_CHECK("mdn_forward");
  return SMD_OK;
}

int smd_mdn_nll(const float* pi, const float* mu, const float* log_sigma, const float* x, int rows, int C, int Kc,
                float* loss, smd_stream_t stream) {
  if (!pi || !mu || !log_sigma || !x || !loss) { set_error("null argument"); return SMD_ERR_INVALID; }
  if (rows < 1 || C < 1 || Kc < 1) { set_error("rows, C and Kc must be >= 1"); return SMD_ERR_INVALID; }
  if (static_cast<long long>(C) + 2LL * Kc > kMdnMaxRowFloats) { set_error("C + 2 Kc must be <= " + std::to_string(kMdnMaxRowFloats) + " (shared memory)"); return SMD_ERR_INVALID; }
  if (static_cast<long long>(Kc) * C > 0x7FFFFFFFll) { set_error("Kc * C too large"); return SMD_ERR_INVALID; }
  MdnNllArgs a;
  memset(&a, 0, sizeof(a));
  a.pi = pi; a.mu = mu; a.ls = log_sigma;
  a.ld_pi = Kc; a.ld_mu = a.ld_ls = Kc * C;
  a.x = x; a.rows = rows; a.C = C; a.Kc = Kc; a.loss = loss;
  SMD_CUDA(launch_mdn_nll(a, static_cast<cudaStream_t>(stream)));
  return SMD_OK;
}

int smd_mdn_loss(smd_plan* plan, const float* params, const float* x, int batch, float* loss_per_token,
                 smd_stream_t stream) {
  int rc = mdn_check(plan, batch, "smd_mdn_loss");
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int S = plan->cfg.seq_len, C = plan->cfg.channels;
  float* xs = plan->at<float>(plan->reg.xt);
  launch_mdn_shift(x, nullptr, xs, batch, S, C, st);
  rc = run_forward(plan, params, xs, nullptr, 0, batch, plan->at<float>(plan->reg.head), st, false);
  if (rc) return rc;
  SMD_CUDA(launch_mdn_nll(plan_nll_args(plan, x, batch * S, loss_per_token), st));
  return SMD_OK;
}

}  // extern "C"

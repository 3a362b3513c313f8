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

// ---------------------------------------------------------------------------------------------------------------------
// Autoregressive sampling (sample_mdn.py:54-119)
// ---------------------------------------------------------------------------------------------------------------------
static constexpr uint32_t kMixtureSalt = 0x916f26abu;   // int(sha512("MixtureSameFamily")) & 0xFFFFFFFF

// The keys of MixtureSameFamily(...).sample(seed=key), an assumption about tfp-nightly 0.12.0.dev20201127 on jax 0.2.8
// that cannot be checked against those packages (tests/mdn_reference.py restates it as mixture_sample_keys):
// MixtureSameFamily._sample_n takes components_seed, mix_seed = split_seed(seed, salt='MixtureSameFamily'), which is
// split(fold_in(seed, salt)), and jax 0.2.8's fold_in(k, d) is the threefry block of k on the counters (0, d).
static void mdn_mixture_keys(const uint32_t key[2], uint32_t comp[2], uint32_t mix[2]) {
  uint32_t f[2] = {0u, kMixtureSalt};
  h_threefry(key[0], key[1], f[0], f[1]);
  uint32_t s[4];
  h_split(f, 2, s);
  comp[0] = s[0]; comp[1] = s[1];
  mix[0] = s[2]; mix[1] = s[3];
}

struct MdnSampleArgs {
  const float* pi; const float* mu; const float* ls;   // local row j at pi + j * ld_pi, mu + j * ld_mu, ls + j * ld_ls
  int ld_pi, ld_mu, ld_ls;
  int rows, C, Kc;
  uint32_t comp0, comp1, mix0, mix1;   // normal draw of the components, Gumbel draw of the mixture
  uint32_t row0, row_step;             // local row j is row row0 + j * row_step of the draw ...
  uint32_t total_rows;                 // ... over total_rows rows (total_rows * Kc * C < 2^32)
  float* out; int ld_out;              // the sample of local row j at out + j * ld_out
  float* out2; int ld_out2;            // and (if not null) at out2 + j * ld_out2
  int* comp;                           // the chosen component per local row, or null
};

// One row of MixtureSameFamily(Categorical(logits=pi), MultivariateNormalDiag(mu, exp(log_sigma))).sample() per CTA.
// jax.random.categorical: k* = argmax_k(pi_k + g_k), g = -log(-log(uniform(mix_key, (R, Kc), tiny, 1))) (first index
// on ties); the value mu_k* + exp(log_sigma_k*) z with z = normal(comp_key, (R, Kc, C))[r, k*].  Threefry is counter
// based, so the CTA draws just the Kc + C elements its row uses.
__global__ void __launch_bounds__(128) mdn_mixture_sample_kernel(const MdnSampleArgs a) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red_v[4];
  __shared__ int red_k[4];
  const int j = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int C = a.C, Kc = a.Kc;
  const uint32_t r = a.row0 + static_cast<uint32_t>(j) * a.row_step;
  const uint32_t nu = a.total_rows * static_cast<uint32_t>(Kc);
  const float* pi = a.pi + static_cast<size_t>(j) * a.ld_pi;
  const float tiny = 1.17549435e-38f;   // jnp.finfo(float32).tiny
  float best = 0.f;
  int bk = -1;
  for (int k = tid; k < Kc; k += blockDim.x) {
    const uint32_t bits = jax_random_bits(a.mix0, a.mix1, r * static_cast<uint32_t>(Kc) + k, nu);
    const float u01 = __uint_as_float((bits >> 9) | 0x3F800000u) - 1.0f;
    const float u = fmaxf(tiny, __fadd_rn(__fmul_rn(u01, __fsub_rn(1.0f, tiny)), tiny));
    const float v = __fadd_rn(pi[k], -logf(-logf(u)));
    if (bk < 0 || v > best) { best = v; bk = k; }
  }
  // larger value wins, the lower index on ties
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
    if (ok >= 0 && (bk < 0 || ov > best || (ov == best && ok < bk))) { best = ov; bk = ok; }
  }
  if (lane == 0) { red_v[warp] = best; red_k[warp] = bk; }
  __syncthreads();
  best = red_v[0]; bk = red_k[0];
  for (int w = 1; w < static_cast<int>(blockDim.x >> 5); ++w)
    if (red_k[w] >= 0 && (bk < 0 || red_v[w] > best || (red_v[w] == best && red_k[w] < bk))) { best = red_v[w]; bk = red_k[w]; }
  const float* mu = a.mu + static_cast<size_t>(j) * a.ld_mu + static_cast<size_t>(bk) * C;
  const float* ls = a.ls + static_cast<size_t>(j) * a.ld_ls + static_cast<size_t>(bk) * C;
  const uint32_t nz = nu * static_cast<uint32_t>(C);
  const uint32_t z0 = (r * static_cast<uint32_t>(Kc) + static_cast<uint32_t>(bk)) * static_cast<uint32_t>(C);
  for (int c = tid; c < C; c += blockDim.x) {
    const float z = jax_normal_from_bits(jax_random_bits(a.comp0, a.comp1, z0 + c, nz));
    const float x = __fadd_rn(mu[c], __fmul_rn(expf(ls[c]), z));
    a.out[static_cast<size_t>(j) * a.ld_out + c] = x;
    if (a.out2) a.out2[static_cast<size_t>(j) * a.ld_out2 + c] = x;
  }
  if (a.comp && tid == 0) a.comp[j] = bk;
}

static cudaError_t launch_mdn_mixture_sample(const MdnSampleArgs& a, cudaStream_t st) {
  mdn_mixture_sample_kernel<<<a.rows, 128, 0, st>>>(a); CNT();
  return cudaGetLastError();
}

// Causal attention of decode step i: one query (position i) per (sample, head) against the cached keys / values 0..i of
// kv ([n][S][384] rows of q | k | v, as the full forward's qkv).  One thread per (sample, head), fp32 in
// causal_attention_kernel's order (q scaled by 1/sqrt(dh) before the dot, keys in ascending order, masked keys at
// -inf), so with the same kv rows its output is that kernel's row i.
template <int DH>
__global__ void __launch_bounds__(128) mdn_decode_attention_kernel(const float* __restrict__ kv,
                                                                   __nv_bfloat16* __restrict__ o, int n, int H, int i) {
  constexpr int S = 32;
  pdl_trigger();
  pdl_wait();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * H) return;
  const int b = t / H, h = t - b * H;
  const float* base = kv + static_cast<size_t>(b) * S * 384 + h * DH;
  const float qs = rsqrtf(static_cast<float>(DH));
  float q[DH];
#pragma unroll
  for (int d4 = 0; d4 < DH / 4; ++d4) {
    const float4 q4 = *reinterpret_cast<const float4*>(base + i * 384 + 4 * d4);
    q[4 * d4] = q4.x * qs; q[4 * d4 + 1] = q4.y * qs; q[4 * d4 + 2] = q4.z * qs; q[4 * d4 + 3] = q4.w * qs;
  }
  float sc[S];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < S; ++j) {
    float s = -INFINITY;
    if (j <= i) {
      s = 0.f;
      const float4* kr = reinterpret_cast<const float4*>(base + j * 384 + 128);
#pragma unroll
      for (int d4 = 0; d4 < DH / 4; ++d4) {
        const float4 k4 = kr[d4];
        s = fmaf(q[4 * d4], k4.x, s); s = fmaf(q[4 * d4 + 1], k4.y, s);
        s = fmaf(q[4 * d4 + 2], k4.z, s); s = fmaf(q[4 * d4 + 3], k4.w, s);
      }
    }
    sc[j] = s;
    mx = fmaxf(mx, s);
  }
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < S; ++j) { sc[j] = expf(sc[j] - mx); sum += sc[j]; }
  const float inv = 1.0f / sum;
  float acc[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) acc[d] = 0.f;
#pragma unroll
  for (int j = 0; j < S; ++j) {
    if (j > i) break;
    const float p = sc[j] * inv;
    const float4* vr = reinterpret_cast<const float4*>(base + j * 384 + 256);
#pragma unroll
    for (int d4 = 0; d4 < DH / 4; ++d4) {
      const float4 v4 = vr[d4];
      acc[4 * d4] = fmaf(p, v4.x, acc[4 * d4]); acc[4 * d4 + 1] = fmaf(p, v4.y, acc[4 * d4 + 1]);
      acc[4 * d4 + 2] = fmaf(p, v4.z, acc[4 * d4 + 2]); acc[4 * d4 + 3] = fmaf(p, v4.w, acc[4 * d4 + 3]);
    }
  }
  __nv_bfloat16* orow = o + static_cast<size_t>(b) * 128 + h * DH;
#pragma unroll
  for (int d = 0; d < DH; d += 2)
    *reinterpret_cast<__nv_bfloat162*>(orow + d) = __floats2bfloat162_rn(acc[d], acc[d + 1]);
}

static cudaError_t launch_mdn_decode_attention(const float* kv, __nv_bfloat16* o, int n, int H, int i, cudaStream_t st) {
  const int blocks = (n * H + 127) / 128;
  switch (128 / H) {
    case 4: mdn_decode_attention_kernel<4><<<blocks, 128, 0, st>>>(kv, o, n, H, i); break;
    case 8: mdn_decode_attention_kernel<8><<<blocks, 128, 0, st>>>(kv, o, n, H, i); break;
    case 16: mdn_decode_attention_kernel<16><<<blocks, 128, 0, st>>>(kv, o, n, H, i); break;
    case 32: mdn_decode_attention_kernel<32><<<blocks, 128, 0, st>>>(kv, o, n, H, i); break;
    default: return cudaErrorInvalidValue;
  }
  CNT();
  return cudaGetLastError();
}

// Decode step i < S - 1 on n samples: the network at position i only, fed the step's input token (mdn.tok).  The trunk
// runs one row per sample; its QKV GEMM appends the position's q / k / v to the cache and the attention reads keys and
// values 0..i from there, then the tail and the head write mdn.head rows [n].  Causal attention and per-token layers
// make this the full forward's output at position i.
static int mdn_decode_step(smd_plan* p, const float* params, int n, int i, cudaStream_t st) {
  const smd_config& c = p->cfg;
  const int S = c.seq_len, C = c.channels, Md = c.mlp_dims;
  const WorkspaceLayout& w = p->reg;
  const ParamLayout& par = p->par;
  p->stat_slots.assign(static_cast<size_t>(2 * p->K + 1), 0);
  SMD_CUDA(cudaMemsetAsync(p->at<float>(w.stats), 0, static_cast<size_t>(2 * p->K + 1) * p->Mp * 2 * 4, st));
  auto h = [&](int j) { return p->at<float>(w.h[j]); };
  auto a = [&](int j) { return p->at<__nv_bfloat16>(w.a[j]); };
  // one position per row: the embedding adds row (m % 1) of the table it is given, position i's encoding
  launch_embed(p->at<float>(w.tok), params + par.in.kernel, params + par.in.bias,
               p->at<float>(w.posenc) + static_cast<size_t>(i) * kE, params + par.layer[0].ln1.scale,
               params + par.layer[0].ln1.bias, h(0), a(0), n, C, 1, st); CNT();
  for (int l = 0; l < p->L; ++l) {
    const LayerParams& lp = par.layer[l];
    const Norm& next_ln = (l + 1 < p->L) ? par.layer[l + 1].ln1 : par.post_ln;
    float* kv = p->at<float>(w.kv[l]);
    GemmEpilogue e = epi();
    e.bias = params + lp.qkv.bias;
    e.out_f32 = kv + static_cast<size_t>(i) * 3 * kE; e.ld_f32 = S * 3 * kE;
    SMD_CUDA(gemm(p, p->op_qkv[l], n, e, st));
    SMD_CUDA(launch_mdn_decode_attention(kv, p->at<__nv_bfloat16>(w.o[l]), n, c.num_heads, i, st));
    e = epi();
    e.bias = params + lp.out.bias;
    e.residual = h(2 * l); e.ld_res = kE;
    e.out_f32 = h(2 * l + 1); e.ld_f32 = kE;
    e.out_bf16 = a(2 * l + 1); e.ld_bf16 = kE;
    e.ln_gamma = params + lp.ln2.scale; e.ln_beta = params + lp.ln2.bias;
    SMD_CUDA(gemm(p, p->op_o[l], n, e, st));
    e = epi();
    e.bias = params + lp.ffn1.bias;
    e.out_bf16 = p->at<__nv_bfloat16>(w.hidden[l]); e.ld_bf16 = Md; e.act = ACT_GELU_TANH;
    SMD_CUDA(gemm(p, p->op_ffn1[l], n, e, st));
    e = epi();
    e.bias = params + lp.ffn2.bias;
    e.residual = h(2 * l + 1); e.ld_res = kE;
    e.out_f32 = h(2 * l + 2); e.ld_f32 = kE;
    e.out_bf16 = a(2 * l + 2); e.ld_bf16 = kE;
    e.ln_gamma = params + next_ln.scale; e.ln_beta = params + next_ln.bias;
    SMD_CUDA(gemm(p, p->op_ffn2[l], n, e, st));
  }
  GemmEpilogue e = epi();
  e.bias = params + par.post.bias;
  e.out_f32 = p->at<float>(w.u[0]); e.ld_f32 = Md;
  e.row_stats = p->at<float>(w.stats);
  SMD_CUDA(gemm(p, p->op_post, n, e, st, 0));
  SMD_LAUNCH_CHECK("mdn decode trunk");
  return run_tail(p, params, n, 1, 0, p->at<float>(w.head), st, false);
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

int smd_mdn_mixture_sample(const float* pi, const float* mu, const float* log_sigma, int rows, int C, int Kc,
                           const uint32_t host_key[2], long long first_row, long long total_rows, float* out,
                           int* components_or_null, smd_stream_t stream) {
  if (!pi || !mu || !log_sigma || !host_key || !out) { set_error("null argument"); return SMD_ERR_INVALID; }
  if (rows < 1 || C < 1 || Kc < 1) { set_error("rows, C and Kc must be >= 1"); return SMD_ERR_INVALID; }
  if (total_rows == 0) total_rows = rows;
  if (first_row < 0 || first_row + rows > total_rows) { set_error("first_row + rows must be <= total_rows"); return SMD_ERR_INVALID; }
  if (total_rows * Kc * C > 0xFFFFFFFFll) { set_error("total_rows * Kc * C threefry counters exceed 2^32 - 1"); return SMD_ERR_INVALID; }
  MdnSampleArgs a;
  memset(&a, 0, sizeof(a));
  a.pi = pi; a.mu = mu; a.ls = log_sigma;
  a.ld_pi = Kc; a.ld_mu = a.ld_ls = Kc * C;
  a.rows = rows; a.C = C; a.Kc = Kc;
  uint32_t comp[2], mix[2];
  mdn_mixture_keys(host_key, comp, mix);
  a.comp0 = comp[0]; a.comp1 = comp[1]; a.mix0 = mix[0]; a.mix1 = mix[1];
  a.row0 = static_cast<uint32_t>(first_row); a.row_step = 1; a.total_rows = static_cast<uint32_t>(total_rows);
  a.out = out; a.ld_out = C;
  a.comp = components_or_null;
  SMD_CUDA(launch_mdn_mixture_sample(a, static_cast<cudaStream_t>(stream)));
  return SMD_OK;
}

int smd_mdn_sample(smd_plan* plan, const float* params, const uint32_t host_key[2], int n, long long first_row,
                   long long total_rows, float* out, float* chain_or_null, int* components_or_null,
                   smd_stream_t stream) {
  if (!plan || !plan->mdn()) { set_error("smd_mdn_sample needs a TransformerMDN plan (smd_mdn_plan_create)"); return SMD_ERR_INVALID; }
  if (plan->reg.kv.empty()) { set_error("smd_mdn_sample needs a plan created with sampler_T > 0 (decode state)"); return SMD_ERR_STATE; }
  int rc = mdn_check(plan, n, "smd_mdn_sample");
  if (rc) return rc;
  if (!plan->packed) { set_error("smd_pack_weights has not been called"); return SMD_ERR_STATE; }
  if (!params || !host_key || !out) { set_error("null argument"); return SMD_ERR_INVALID; }
  const int S = plan->cfg.seq_len, C = plan->cfg.channels, Kc = plan->Kc;
  if (total_rows == 0) total_rows = n;
  if (first_row < 0 || first_row + n > total_rows) { set_error("first_row + n must be <= total_rows"); return SMD_ERR_INVALID; }
  if (total_rows * S * Kc * C > 0xFFFFFFFFll) { set_error("total_rows * S * Kc * C threefry counters exceed 2^32 - 1"); return SMD_ERR_INVALID; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* xt = plan->at<float>(plan->reg.xt);   // the chain: position 0 zero, position i + 1 decoded at step i
  float* tok = plan->at<float>(plan->reg.tok);
  float* z = plan->at<float>(plan->reg.head);
  SMD_CUDA(cudaMemsetAsync(xt, 0, static_cast<size_t>(n) * S * C * 4, st));
  SMD_CUDA(cudaMemsetAsync(tok, 0, static_cast<size_t>(n) * C * 4, st));
  const HeadParts h = head_parts(plan);
  MdnSampleArgs a;
  memset(&a, 0, sizeof(a));
  a.mu = z + h.off[0]; a.ls = z + h.off[1]; a.pi = z + h.off[2];
  a.ld_pi = a.ld_mu = a.ld_ls = plan->head_ld;
  a.C = C; a.Kc = Kc;
  a.total_rows = static_cast<uint32_t>(total_rows * S);   // every step draws over all N * S rows (sample_mdn.py:110)
  uint32_t rng[2] = {host_key[0], host_key[1]};
  for (int i = 0; i < S; ++i) {
    uint32_t s4[4], comp[2], mix[2];
    h_split(rng, 2, s4);                                  // rng, embed_rng = split(rng)
    rng[0] = s4[0]; rng[1] = s4[1];
    mdn_mixture_keys(s4 + 2, comp, mix);
    a.comp0 = comp[0]; a.comp1 = comp[1]; a.mix0 = mix[0]; a.mix1 = mix[1];
    if (i < S - 1) {
      // tokens[:, i + 1] = next_tokens[:, i]: row b * S + i of the draw, into the chain and the next step's input
      rc = mdn_decode_step(plan, params, n, i, st);
      if (rc) return rc;
      a.rows = n; a.row0 = static_cast<uint32_t>(first_row * S + i); a.row_step = S;
      a.out = xt + static_cast<size_t>(i + 1) * C; a.ld_out = S * C;
      a.out2 = tok; a.ld_out2 = C;
    } else {
      // tokens = next_tokens: the last step keeps a fresh draw at every position of the full pass over the chain
      if (chain_or_null)
        SMD_CUDA(cudaMemcpyAsync(chain_or_null, xt, static_cast<size_t>(n) * S * C * 4, cudaMemcpyDeviceToDevice, st));
      rc = run_forward(plan, params, xt, nullptr, 0, n, z, st, false);
      if (rc) return rc;
      a.rows = n * S; a.row0 = static_cast<uint32_t>(first_row * S); a.row_step = 1;
      a.out = out; a.ld_out = C;
      a.out2 = nullptr;
      a.comp = components_or_null;
    }
    SMD_CUDA(launch_mdn_mixture_sample(a, st));
  }
  return SMD_OK;
}

}  // extern "C"

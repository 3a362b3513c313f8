/* libsmd -- C ABI of the native (sm_90a) DDPM noise-prediction hot path.
 *
 * The reference (magenta/symbolic-music-diffusion @ 469204d) has no FFI: its only host->device boundary is the
 * jax.jit boundary of three Python callables.  Each entry point below replaces one of them (or a piece of one)
 * and is what a ctypes binding in the reference's own files would call (see INTEGRATION.md):
 *
 *   smd_forward            <- model(inputs, t)               models/ncsn.py:141-179 (TransformerDDPM.apply),
 *                                                            models/ncsn.py:125-135 (DenseDDPM.apply)
 *   smd_ddpm_loss          <- diffusion_loss(...)            utils/losses.py:250-308   (eval_step, train_ncsn.py:206-221)
 *   smd_ddpm_grads + smd_clip_adam <- train_step(...)      train_ncsn.py:260-288 (value_and_grad, then clip + Adam)
 *   smd_ema_update         <- EMAHelper.update               utils/train_utils.py:73-78
 *   smd_ddpm_reverse_step  <- body of sample_with_beta       utils/ebm_utils.py:327-397
 *   smd_ddpm_sample        <- diffusion_dynamics(...)        utils/ebm_utils.py:274-405 (lax.scan over T steps)
 *   smd_threefry_*         <- jax.random.{split,normal,...}  (jax 0.2.8, call sites utils/losses.py:271-294,
 *                                                            utils/ebm_utils.py:329,342,360)
 *
 * Conventions: every pointer is a DEVICE pointer owned by the caller (PyTorch) unless named host_*; the library
 * allocates no device memory (the caller binds one workspace); all work is asynchronous on the given CUDA stream;
 * functions return 0 or a negative smd_status and smd_last_error() describes the failure (thread-local).
 * There is no CPU fallback anywhere behind this ABI.
 */
#ifndef SMD_H_
#define SMD_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct smd_plan smd_plan;
typedef void* smd_stream_t; /* cudaStream_t */

enum smd_status {
  SMD_OK = 0,
  SMD_ERR_INVALID = -1,   /* bad argument / unsupported configuration (Python raises ValueError) */
  SMD_ERR_CUDA = -2,      /* CUDA runtime / driver error */
  SMD_ERR_STATE = -3      /* call order (e.g. workspace not bound) */
};

enum smd_arch {
  SMD_ARCH_TRANSFORMER_DDPM = 0,
  SMD_ARCH_DENSE_DDPM = 1,
  /* models/ncsn.py:83-98 (DenseNCSN) with its undefined `t` read as `sigmas`: the DenseDDPM stack conditioned on sigma,
   * output divided by sigma (a score).  Same parameter layout as SMD_ARCH_DENSE_DDPM. */
  SMD_ARCH_DENSE_NCSN = 2,
  /* models/autoregressive.py:37-82 (TransformerMDN): the TransformerDDPM trunk on the input shifted right by one position,
   * causal self-attention, res-blocks without FiLM and a mixture-density head.  Created with smd_mdn_plan_create only
   * (seq_len 32, precision bf16). */
  SMD_ARCH_TRANSFORMER_MDN = 3
};

typedef struct smd_config {
  int arch;            /* smd_arch; TransformerDDPM4 (configs/ddpm-multi-32seq-512.cfg:1) == TransformerDDPM */
  int num_layers;      /* --num_layers   (train_ncsn.py:69)  trunk layers L, or DenseDDPM res-blocks */
  int num_heads;       /* --num_heads    (train_ncsn.py:70)  ignored by DenseDDPM */
  int num_mlp_layers;  /* --num_mlp_layers (train_ncsn.py:71) FiLM res-blocks K, ignored by DenseDDPM */
  int mlp_dims;        /* --mlp_dims     (train_ncsn.py:72) */
  int seq_len;         /* S: data_shape[0] for TransformerDDPM, one of 32, 64, 128 (else SMD_ERR_INVALID); 1 for DenseDDPM */
  int channels;        /* C: data_shape[-1] after --slice_ckpt (42 / 146 / 512) */
  int max_batch;       /* largest number of examples one call may pass */
  int cta_group;       /* 1 or 2 (accepted for compatibility; sm_90a GEMMs use one CTA per tile) */
  int training;        /* 1: reserve the saved-activation / gradient buffers of smd_ddpm_grads */
  int sampler_T;       /* > 0: reserve a (K, sampler_T, 2*mlp_dims) FiLM table so the sampler evaluates the FiLM
                          generator once per schedule instead of once per step (all samples share t) */
  int precision;       /* smd_precision.  SMD_PRECISION_BF16X3 (forward / sampling only, ~3x the GEMM time): every
                          tensor-core operand is split into bf16 hi + lo halves and the GEMMs add the cross terms
                          (hi*hi + hi*lo + lo*hi, fp32 accumulate), activations use exact tanhf / expf and attention runs
                          in fp32 -- the mode that shows the kernels reproduce the reference's fp32 arithmetic to ~1e-5
                          rather than to bf16 accuracy (tests/test_gpu_strict.py) */
} smd_config;
enum smd_precision { SMD_PRECISION_BF16 = 0, SMD_PRECISION_BF16X3 = 1 };

const char* smd_last_error(void);
int smd_version(void);

/* ---- plan / parameter arena ------------------------------------------------------------------------------- */
int smd_plan_create(const smd_config* cfg, smd_plan** out);
void smd_plan_destroy(smd_plan* plan);
/* fp32 parameter arena: `smd_num_tensors` named tensors laid out back to back (each start 16-byte aligned)
 * inside `smd_arena_floats` floats.  Names mirror the flax module tree. */
int smd_num_tensors(const smd_plan* plan);
long long smd_arena_floats(const smd_plan* plan);
int smd_tensor_info(const smd_plan* plan, int index, char* name, int name_cap, long long* offset, int* shape4,
                    int* ndim);
size_t smd_workspace_bytes(const smd_plan* plan);
int smd_bind_workspace(smd_plan* plan, void* workspace, size_t bytes);
/* Refresh the bf16 tensor-core operand copies from the fp32 arena (after init / restore / every optimizer step). */
int smd_pack_weights(smd_plan* plan, const float* params, smd_stream_t stream);
/* Same, when the bf16 shadow arena was already written by smd_clip_adam (only the padded out.kernel copy is rebuilt). */
int smd_pack_weights_after_adam(smd_plan* plan, const float* params, smd_stream_t stream);
/* Device pointer of the bf16 shadow of the parameter arena (same element offsets), NULL before the workspace is bound. */
void* smd_shadow_arena(smd_plan* plan);

/* ---- score network ---------------------------------------------------------------------------------------- */
/* eps_hat = model(x, t).  x: (batch, S, C) fp32; t: (batch) fp32 noise level sqrt(alpha_bar), or a single
 * value shared by the whole batch when t_broadcast != 0 (the sampler's case); y: (batch, S, C) fp32. */
int smd_forward(smd_plan* plan, const float* params, const float* x, const float* t, int t_broadcast, int batch,
                float* y, smd_stream_t stream);

/* ---- objective -------------------------------------------------------------------------------------------- */
/* diffusion_loss with the random draws supplied: x0 (batch,S,C), used_alpha (batch), eps (batch,S,C).
 * loss_per_example (batch) = mean_{S,C}((eps - pred)^2); pred_or_null receives the prediction. */
int smd_ddpm_loss(smd_plan* plan, const float* params, const float* x0, const float* used_alpha, const float* eps,
                  int batch, float* loss_per_example, float* pred_or_null, smd_stream_t stream);

/* One optimizer step of train_ncsn.py:260-288 on this rank's shard:
 *   grads <- d mean_{global batch}(loss) / d params   (scaled by 1/global_batch so a SUM all-reduce over ranks
 *   gives the gradient of the global mean);  loss_sum[0] = sum of this shard's per-example losses and
 *   loss_sum[1] = loss_sum[0] / global_batch (two floats, overwritten; summed in example order by the kernel's last
 *   block, so the reported loss is bit-reproducible; a SUM all-reduce of loss_sum[1] gives the global mean loss).
 * smd_ddpm_grads only produces grads (so the caller can all-reduce them with NCCL);
 * smd_clip_adam applies global-norm clipping (jax clip_grads), Adam (flax.optim.Adam) and optional EMA. */
int smd_ddpm_grads(smd_plan* plan, const float* params, const float* x0, const float* used_alpha, const float* eps,
                   int batch, int global_batch, float* grads, float* loss_sum, smd_stream_t stream);
/* Overlapping the data-parallel exchange with the backward pass (what jax.lax.pmean over the gradient pytree does at
 * train_ncsn.py:283-284, where XLA is free to schedule the collective early): the gradients of the FiLM'd residual
 * tail and the output layer -- the contiguous arena slice [*first_float, *first_float + *num_floats), ~85% of all
 * parameters -- are final long before the transformer trunk's.  After smd_ddpm_grads has been enqueued,
 * smd_wait_tail_grads makes `stream` (the caller's communication stream) wait until that slice is complete, so its
 * all-reduce runs under the trunk backward; the rest of the arena is reduced after smd_ddpm_grads' own stream. */
int smd_grads_tail_range(const smd_plan* plan, long long* first_float, long long* num_floats);
int smd_wait_tail_grads(smd_plan* plan, smd_stream_t stream);
/* scratch: >= 1024 floats (per-block partial sums of squares, combined in a fixed order so that all data-parallel
 * ranks compute bit-identical clip factors); grad_norm_out[0] = post-clip global L2 norm.
 * bf16_shadow_or_null: the plan's bf16 shadow arena (smd_shadow_arena): the updated parameters are also written
 * there in the same pass, after which smd_pack_weights_after_adam (not smd_pack_weights) completes the refresh. */
int smd_clip_adam(float* params, float* grads, float* adam_m, float* adam_v, float* ema_or_null,
                  void* bf16_shadow_or_null, long long n, float lr, int step, float max_norm, float beta1,
                  float beta2, float eps, float ema_mu, float* scratch, float* grad_norm_out, smd_stream_t stream);
int smd_ema_update(float* ema, const float* params, long long n, float mu, smd_stream_t stream);

/* Random draws of diffusion_loss (utils/losses.py:270-294) on device with jax 0.2.8 threefry semantics:
 * rng,label_rng,sample_rng = split(key,3); labels = randint(label_rng, 1, T+1); rng,noise_rng = split(rng);
 * used_alpha = uniform(noise_rng, minval=abar[labels-1], maxval=abar[labels]); eps = normal(sample_rng).
 * smd_objective_setup uploads abar = concat([1], cumprod(1-betas)) (host_betas: HOST pointer, T floats). */
int smd_objective_setup(smd_plan* plan, const float* host_betas, int T, smd_stream_t stream);
int smd_ddpm_draws(smd_plan* plan, const uint32_t host_key[2], int batch, float* used_alpha, float* eps,
                   int* labels_or_null, smd_stream_t stream);
/* The same draws for rows [first_row, first_row + batch) of a GLOBAL batch of global_batch examples (threefry is
 * counter based): a data-parallel rank consumes exactly its slice of the single-process stream, so a run on N GPUs
 * with seed s sees the noise of the 1-GPU run with seed s (SURVEY 8(e)).  continuous_noise == 0 follows the
 * reference's int(continuous_noise) label range (utils/losses.py:272-275): labels in [0, T), and for label 0 the
 * lower bound alphas_prod[-1] wraps to the last entry as jnp indexing does. */
int smd_ddpm_draws_sharded(smd_plan* plan, const uint32_t host_key[2], int global_batch, int first_row, int batch,
                           int continuous_noise, float* used_alpha, float* eps, int* labels_or_null,
                           smd_stream_t stream);

/* ---- NCSN family (SURVEY 8(f4)): denoising score matching + Langevin samplers ------------------------------- */
/* denoising_score_matching_loss (utils/losses.py:129-179) with the draws supplied: x~ = x0 + used_sigma * eps,
 * scores = model(x~, used_sigma), loss[b] = 0.5 * sum((scores + eps / sigma)^2) * sigma^2.  pred_or_null <- scores. */
int smd_dsm_loss(smd_plan* plan, const float* params, const float* x0, const float* used_sigma, const float* eps,
                 int batch, float* loss_per_example, float* pred_or_null, smd_stream_t stream);
/* gradients of mean_{global batch}(that loss); same contract as smd_ddpm_grads (loss_sum: 2 floats) */
int smd_dsm_grads(smd_plan* plan, const float* params, const float* x0, const float* used_sigma, const float* eps,
                  int batch, int global_batch, float* grads, float* loss_sum, smd_stream_t stream);
/* its random draws (utils/losses.py:146-164): labels = randint(int(continuous), L); used_sigma = uniform(sigmas[l-1],
 * sigmas[l]) (continuous) or sigmas[l]; eps = normal.  smd_dsm_setup uploads the schedule (host_sigmas: L floats). */
int smd_dsm_setup(smd_plan* plan, const float* host_sigmas, int L, smd_stream_t stream);
int smd_dsm_draws(smd_plan* plan, const uint32_t host_key[2], int global_batch, int first_row, int batch,
                  int continuous_noise, float* used_sigma, float* eps, int* labels_or_null, smd_stream_t stream);
/* sliced_score_matching_loss (utils/losses.py:182-247, one particle) with the draws supplied, SMD_ARCH_DENSE_NCSN only
 * (other plans: SMD_ERR_INVALID): x~ = x0 + used_sigma * eps, s = model(x~, used_sigma), v: (batch, C) of +-1,
 * loss[b] = (0.5 |s_b|^2 + v_b . (J_s v)_b) * sigma_b^2.  The Hessian term is a forward-mode Jacobian-vector product
 * through the network (a tangent pass next to the primal one).  score_or_null <- s; hvp_or_null (batch) <- v.J_s v.
 * A bf16x3 plan runs the tangent GEMMs in three passes as well. */
int smd_ssm_loss(smd_plan* plan, const float* params, const float* x0, const float* used_sigma, const float* eps,
                 const float* v, int batch, float* loss_per_example, float* score_or_null, float* hvp_or_null,
                 smd_stream_t stream);
/* gradients of mean_{global batch}(that loss) -- the primal and tangent passes differentiated together in reverse
 * mode; same contract as smd_dsm_grads (loss_sum: 2 floats) */
int smd_ssm_grads(smd_plan* plan, const float* params, const float* x0, const float* used_sigma, const float* eps,
                  const float* v, int batch, int global_batch, float* grads, float* loss_sum, smd_stream_t stream);
/* its random draws (utils/losses.py:203-223): rng, label_rng, sample_rng, score_rng = split(key, 4); labels and
 * used_sigma as smd_dsm_draws (noise_rng from split(rng) when continuous), eps = normal(sample_rng),
 * v = rademacher(score_rng) = +1 where the threefry word is < 2^31, else -1.  Schedule: smd_dsm_setup.  Rows
 * [first_row, first_row + batch) of a global batch, as smd_dsm_draws. */
int smd_ssm_draws(smd_plan* plan, const uint32_t host_key[2], int global_batch, int first_row, int batch,
                  int continuous_noise, float* used_sigma, float* eps, float* v, int* labels_or_null,
                  smd_stream_t stream);
/* One Langevin update after a network call (annealed_langevin_dynamics utils/ebm_utils.py:139-175, consistent_... :231-253):
 *   x_next = x + alpha * grad + noise_coef * z;  with a mask: x_next = x_next (1 - mask) + (infill_x + infill_sigma z') mask.
 * z / infill_z: supplied N(0,1) tensors or NULL -> jax.random.normal(step_key / infill_key).  metrics4 (device, 4 floats,
 * pre-zeroed) receives grad_norm, step_norm, alpha, noise_norm; collection_slot (n,S,C) or NULL gets a copy of x_next. */
int smd_langevin_step(smd_plan* plan, const float* x, const float* grad, int n, float alpha, float noise_coef,
                      const uint32_t step_key[2], const float* z, const float* infill_x, const float* infill_mask,
                      float infill_sigma, const uint32_t infill_key[2], const float* infill_z, float* x_next,
                      float* collection_slot, float* metrics4, smd_stream_t stream);

/* ---- sampler ---------------------------------------------------------------------------------------------- */
/* host_betas: HOST pointer, T floats.  Builds the per-step coefficient / key / slot tables in the workspace.
 * key = jax PRNG key (2 x uint32) that diffusion_dynamics receives as `rng`. */
int smd_sampler_setup(smd_plan* plan, const float* host_betas, int T, const uint32_t host_key[2],
                      smd_stream_t stream);
/* Sharded sampling (sample_size split over data-parallel ranks, SURVEY 8(e)): this plan's calls hold samples
 * [first_row, first_row + n) of a global batch of total_rows samples and draw exactly that slice of the chain's
 * threefry noise streams, so the gathered result equals the single-process chain.  total_rows = 0 switches it off. */
int smd_sampler_set_shard(smd_plan* plan, long long first_row, long long total_rows);
/* One reverse step at index t (T-1 .. 0) on state x (n,S,C), in place allowed (x_next == x).
 * z / infill_z: supplied N(0,1) tensors or NULL -> in-kernel threefry with the tables of smd_sampler_setup.
 * metrics: device (4, T) fp32 or NULL (column T-1-t accumulated: grad_norm, step_norm, alpha_prod, noise_norm).
 * collection: device (41, n, S, C) or NULL. */
int smd_ddpm_reverse_step(smd_plan* plan, const float* params, const float* x, int n, int t, const float* z,
                          const float* infill_x, const float* infill_mask, const float* infill_z, float* x_next,
                          float* eps_hat_or_null, float* collection, float* metrics, smd_stream_t stream);
/* Whole chain: `steps` reverse steps starting at t = T-1 (steps == T for the full chain), state updated in place.
 * use_graph != 0 captures one step into a CUDA graph and replays it. */
int smd_ddpm_sample(smd_plan* plan, const float* params, float* x, int n, int steps, const float* infill_x,
                    const float* infill_mask, float* collection, float* metrics, int use_graph,
                    smd_stream_t stream);

/* ---- autoregressive baseline (TransformerMDN, train_mdn.py) -------------------------------------------------- */
/* cfg->arch must be SMD_ARCH_TRANSFORMER_MDN; num_components = --mdn_components (Kc).  SMD_ERR_INVALID for
 * seq_len != 32, precision bf16x3 or num_components < 1.  Parameters: the TransformerDDPM trunk, k{i}.res.* without
 * film, out_ln, then mdn.mu / mdn.log_sigma (Md, Kc*C) and mdn.pi (Md, Kc); column k*C + c of mu / log_sigma is
 * component k, channel c.  smd_forward, the DDPM / NCSN objectives and the sampler return SMD_ERR_INVALID on such a
 * plan. */
int smd_mdn_plan_create(const smd_config* cfg, int num_components, smd_plan** out);
/* (pi, mu, log_sigma) = model(x, shift)   (models/autoregressive.py:40-82).  x: (batch, S, C) fp32; pi (batch, S, Kc),
 * mu and log_sigma (batch, S, Kc*C) fp32.  shift = 0 feeds x to the trunk as it is (autoregressive decoding). */
int smd_mdn_forward(smd_plan* plan, const float* params, const float* x, int batch, int shift, float* pi, float* mu,
                    float* log_sigma, smd_stream_t stream);
/* mdn_loss(pi, mu, log_sigma, x, 'none') (train_mdn.py:100-133), no plan needed: loss[r] = -log sum_k softmax(pi_r)_k
 * N(x_r; mu_rk, diag(exp(log_sigma_rk))^2) for rows r < rows; pi (rows, Kc), mu / log_sigma (rows, Kc*C), x (rows, C). */
int smd_mdn_nll(const float* pi, const float* mu, const float* log_sigma, const float* x, int rows, int C, int Kc,
                float* loss, smd_stream_t stream);
/* eval_step's loss (train_mdn.py:154-168): the model on shift_right(x), scored against x; one loss per token (batch*S). */
int smd_mdn_loss(smd_plan* plan, const float* params, const float* x, int batch, float* loss_per_token,
                 smd_stream_t stream);
/* gradients of the mean of that loss over global_batch * S tokens; same contract as smd_ddpm_grads (loss_sum[0] = this
 * shard's token-loss sum, loss_sum[1] = loss_sum[0] / (global_batch * S)), CUDA-graph replay and
 * smd_grads_tail_range / smd_wait_tail_grads (the k*, out_ln and mdn.* slice) included. */
int smd_mdn_grads(smd_plan* plan, const float* params, const float* x, int batch, int global_batch, float* grads,
                  float* loss_sum, smd_stream_t stream);

/* ---- jax.random (threefry2x32) on device ------------------------------------------------------------------ */
int smd_threefry_normal(const uint32_t host_key[2], float* out, long long n, smd_stream_t stream);
/* elements [first, first + n) of jax.random.normal(key, (total,)) (a rank's rows of the global initial state) */
int smd_threefry_normal_slice(const uint32_t host_key[2], float* out, long long n, long long first, long long total,
                              smd_stream_t stream);
/* jax.random.uniform(key, (n,), float32, minval, maxval) as of jax 0.2.8 (sample_ncsn.py:230: the infill initial state) */
int smd_threefry_uniform(const uint32_t host_key[2], float* out, long long n, float minval, float maxval,
                         smd_stream_t stream);
/* host-side split: out_keys = jax.random.split(key, num) (num x 2 uint32) */
int smd_threefry_split(const uint32_t host_key[2], int num, uint32_t* host_out_keys);

/* ---- test hooks (used by tests/ only) --------------------------------------------------------------------- */
/* D[M,N] = A * B^T with the production wgmma kernel.  A: bf16, K-major [M][K] or MN-major [K][M];
 * B: bf16, K-major [N][K] or MN-major [K][N].  Optional fused epilogue pieces (NULL to skip). */
int smd_gemm_bf16(const void* A, const void* B, int M, int N, int K, int a_mn, int b_mn, int BN, int cta_group,
                  const float* bias, const float* residual, int act, float* out_f32, void* out_bf16,
                  float* row_stats, const float* ln_gamma, const float* ln_beta, smd_stream_t stream);
/* forward pass that keeps every intermediate in the training save buffers (plan must have training = 1) */
int smd_debug_forward_save(smd_plan* plan, const float* params, const float* x, const float* t, int batch, float* y,
                           smd_stream_t stream);
/* device pointer / size of a named workspace region (names as allocated in smd_api.cu), for stage-by-stage parity */
int smd_debug_buffer(smd_plan* plan, const char* name, void** dev_ptr, size_t* bytes);
/* number of kernels this library has launched since load (bench.py's gpu_launches) */
long long smd_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* SMD_H_ */

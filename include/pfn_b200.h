/*
 * pfn_b200.h — C ABI of libpfn_b200.so, the sm_90a kernel library behind the PFN training hot path
 * (prior sample -> masked-attention transformer fwd+bwd -> BarDistribution NLL).
 *
 * The reference (automl/TransformersCanDoBayesianInference @ 9c20031) has no FFI of its own: its hot path is
 * Python calling torch.nn / gpytorch.  Each entry point below names the reference call it replaces
 * (file:line into the reference tree, or `torch:` for the library code the reference reaches).
 *
 * Conventions
 *   - all pointers are DEVICE pointers into caller-owned buffers (PyTorch CUDA tensors); nothing is allocated
 *     or retained by the library; `stream` is a cudaStream_t passed as void*; no call synchronises.
 *   - activations are sequence-first like the reference: token row = t*B + b, row-major [T*B, cols] with an
 *     explicit leading dimension (elements).
 *   - return 0 on success; non-zero on failure with a message in pfn_last_error() (thread-local).  No C++
 *     exception crosses this boundary.
 *   - dtype codes: PFN_F32 / PFN_BF16.  bf16 kernels accumulate and keep all statistics in fp32.
 */
#ifndef PFN_B200_H_
#define PFN_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PFN_B200_VERSION 1

enum { PFN_F32 = 0, PFN_BF16 = 1 };
enum { PFN_EPI_NONE = 0, PFN_EPI_GELU = 1, PFN_EPI_GELU_BWD = 2, PFN_EPI_ROWDOT = 3, PFN_EPI_MUL = 4 };
enum { PFN_KERNEL_RBF = 0, PFN_KERNEL_MATERN12 = 1, PFN_KERNEL_MATERN32 = 2, PFN_KERNEL_MATERN52 = 3 };

const char* pfn_last_error(void);
int pfn_version(void);
int pfn_num_sms(void);

/* ------------------------------------------------------------------------------------------------
 * GEMM:  C[M,N] (+)= epi( sum_k A(m,k) B(n,k) + bias[n] )  (+ aux[m,n] residual)
 *   K-major operand : element (i,k) at base + i*ld + k;   MN-major operand : element (i,k) at base + k*ld + i
 *   epilogue GELU      : C = gelu_erf(acc+bias), optional C2 = acc+bias (pre-activation, saved for backward)
 *   epilogue GELU_BWD  : C = acc * gelu_erf'(aux)
 *   epilogue MUL       : C = acc * aux   (tensor-core path only).  With GELU's c2_gelu_grad = 1 the forward stores gelu'(pre)
 *                        in C2 instead of the pre-activation, and the backward dgrad is this plain product: the ~14
 *                        instructions per element of gelu' leave the backward epilogue, whose cost is instruction issue.
 *   epilogue ROWDOT    : C = acc (+bias), and rowdot_out[m * ceil(N / rowdot_width) + n / rowdot_width] += sum over the
 *                        column group of C[m,n] * aux[m,n]   (fp32 atomics; aux is NOT added to C).  Used to produce
 *                        delta = rowsum(dO * O) per (token, head) in the out-projection dgrad (tensor-core path only).
 *   accumulate / k_splits>1 : atomic fp32 accumulation into C (weight gradients)
 * Replaces: nn.Linear / in_proj / out_proj / linear1 / linear2 / decoder GEMMs and their autograd backward
 *   (reference transformer.py:17-18,23,84-85; torch:nn/functional.py:6478; torch:nn/modules/transformer.py:980-982).
 * pfn_gemm_bf16_tc : TMA + wgmma path (bf16 operands; lda/ldb multiples of 8; 16-byte aligned bases).
 * pfn_gemm_simt    : fp32-FMA path for fp32 parity mode and shapes the tensor-core path does not take.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pfn_gemm_desc {
  int M, N, K;
  const void* A; int lda; int a_mn_major;
  const void* B; int ldb; int b_mn_major;
  void* C; int ldc; int c_dtype;
  const float* bias;
  const void* aux; int ld_aux;
  void* C2; int ldc2;
  int epilogue;
  int accumulate;
  int k_splits;
  int ab_dtype;            /* dtype of A, B, aux, C2 (simt path; the tc path is bf16 only) */
  float* rowdot_out;       /* epilogue ROWDOT: [M, ceil(N / rowdot_width)] fp32, accumulated (zero it first) */
  int rowdot_width;        /* columns per group (the head dimension); must be a multiple of 128 */
  int c2_gelu_grad;        /* epilogue GELU with C2, tensor-core path only: 1 = C2 receives gelu'(acc+bias) instead of acc+bias */
} pfn_gemm_desc;

int pfn_gemm_bf16_tc(const pfn_gemm_desc* d, void* stream);
int pfn_gemm_simt(const pfn_gemm_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Masked multi-head attention under the single_eval_pos mask (mask never materialised):
 *   keys(i) = {0..sep-1}  U  ({i} if i >= sep)          (reference transformer.py:35-41 generate_D_q_matrix)
 *   o_i = sum_j softmax_j(q_i.k_j * scale) v_j           (torch:nn/functional.py:6632-6690)
 * qkv : [T*B, 3*H*dh] packed in-projection output (q | k | v), head h = columns h*dh..(h+1)*dh of each third.
 * out : [T*B, H*dh];  lse : [B*H, T] fp32 natural-log-sum-exp of the scaled scores (saved for backward).
 * Backward writes dqkv [T*B, 3*H*dh] completely (no accumulation).
 * ---------------------------------------------------------------------------------------------- */
typedef struct pfn_attn_desc {
  int T, B, H, dh, sep;
  int dtype;
  float scale;
  const void* qkv; int ld_qkv;
  void* out; int ld_out;
  float* lse;
  const void* dout; int ld_dout;
  void* dqkv; int ld_dqkv;
  float* delta;            /* [B*H, T] fp32 scratch for backward: rowsum(dO * O) */
  int batch_major;         /* 0: token row = t*B + b (reference layout); 1: token row = b*T + t (tensor-core kernels only) */
  /* dropout on the attention probabilities (torch:nn/functional.py multi_head_attention_forward `dropout_p`; reference
   * train.py:22 default 0.2): drop_thr = round(256 p) in [0,255], 0 = off; the keep bit of (row i, key j) of head (b,h) is
   * pfn_dropout_keep_mask's bit for (row = (b*H + h)*T + i, col = j) under drop_seed. */
  uint32_t drop_seed;
  int drop_thr;
  /* backward, tensor-core kernels only, optional: dq_colsum[H*dh] += column sums of dQ (the q third of the in-projection bias
   * gradient), accumulated from the staged dQ tiles so that dqkv need not be re-read.  (The k third is zero in exact
   * arithmetic -- every row of dS sums to zero -- and the v third equals colsum(dO) = colsum(dz) W_out; see engine.py.) */
  float* dq_colsum;
  /* backward, tensor-core kernels only: 1 = `delta` already holds rowsum(dO * O) in TOKEN-major layout [T*B, H] (produced by the
   * ROWDOT epilogue of the out-projection dgrad GEMM); the kernels then skip their own delta pass.  0 = `delta` is [B*H, T]
   * scratch that the backward fills itself. */
  int delta_token_major;
} pfn_attn_desc;

int pfn_attention_fwd_simt(const pfn_attn_desc* d, void* stream);
int pfn_attention_bwd_simt(const pfn_attn_desc* d, void* stream);
int pfn_attention_fwd_tc(const pfn_attn_desc* d, void* stream);
int pfn_attention_bwd_tc(const pfn_attn_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Embedding stage (reference transformer.py:68-74):
 *   out[t,b,:] = x[t,b,:] Wx^T + bx + (t < sep ? y[t,b] wy + by : 0)
 * x [T*B, F] fp32, y [T*B] fp32, Wx [E,F], bx [E], wy [E], by [E] fp32; out [T*B, E] (out_dtype).
 * Backward accumulates (+=) into dWx, dbx, dwy, dby (fp32).
 * ---------------------------------------------------------------------------------------------- */
int pfn_embed_fwd(const float* x, const float* y, const float* Wx, const float* bx, const float* wy, const float* by,
                  void* out, int out_dtype, int T, int B, int F, int E, int sep, void* stream);
int pfn_embed_bwd(const void* dout, int dtype, const float* x, const float* y, float* dWx, float* dbx, float* dwy,
                  float* dby, int T, int B, int F, int E, int sep, void* stream);

/* ------------------------------------------------------------------------------------------------
 * LayerNorm over the last dim, eps inside the sqrt, biased variance (torch:nn/modules/transformer.py:951-956
 * norm1/norm2, eps 1e-5).  The residual add is done by the producing GEMM's epilogue, so z = x + sublayer(x).
 *   fwd : h = (z - mean) * rstd * gamma + beta ; saves mean, rstd (fp32 per row)
 *   bwd : dz = rstd * (g - mean(g) - xhat * mean(g*xhat)), g = dh*gamma ; dgamma += sum dh*xhat ; dbeta += sum dh
 *         optional colsum_out[E] += sum_rows dz   (bias gradient of the GEMM that produced z)
 * ---------------------------------------------------------------------------------------------- */
int pfn_layernorm_fwd(const void* z, int ldz, const float* gamma, const float* beta, void* h, int ldh, float* mean,
                      float* rstd, int rows, int E, float eps, int dtype, void* stream);
int pfn_layernorm_bwd(const void* dh, int lddh, const void* z, int ldz, const float* mean, const float* rstd,
                      const float* gamma, void* dz, int lddz, float* dgamma, float* dbeta, float* colsum_out, int rows,
                      int E, int dtype, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Elementwise dropout (+ residual) with a regenerated counter-based mask (csrc/dropout.cuh):
 *   out[r,c] = (keep(seed,r,c) ? x[r,c] * 256/(256-thr) : 0) + (residual ? residual[r,c] : 0)
 * in place when out == x.  Replaces torch:nn/modules/transformer.py:961-982 dropout1 / dropout / dropout2 of the encoder
 * layer in forward, and is applied to the incoming gradient with the same (seed, thr) in backward.  cols % 8 == 0.
 * pfn_dropout_keep_mask writes the keep bits (1/0) of a rows x cols site as bytes: the hook that lets a test's oracle
 * consume exactly the mask the kernels use (attention site: row = (b*H + h)*T + i, col = key j).
 * ---------------------------------------------------------------------------------------------- */
int pfn_dropout(const void* x, int ldx, const void* residual, int ldr, void* out, int ldo, int rows, int cols, int dtype,
                uint32_t seed, int thr, void* stream);
int pfn_dropout_keep_mask(uint8_t* out, int rows, int cols, uint32_t seed, int thr, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Optimizer step of the training inner loop (reference train.py:94-97):
 *     torch.nn.utils.clip_grad_norm_(model.parameters(), max_grad_norm);  optimizer.step()      [torch.optim.Adam]
 * over ALL parameter tensors in two launches.  `table` (DEVICE memory, n_tensors entries) names, per tensor, the fp32
 * parameter, its gradient, the two Adam moments and -- optionally -- a bf16 copy of the parameter that is rewritten with the
 * updated value (the operand the next step's GEMMs read).  `chunk_start` (DEVICE, n_tensors + 1 ints) holds the prefix sums
 * of ceil(n / pfn_adam_chunk_elems()) per tensor; n_chunks = chunk_start[n_tensors].  `step` is the 1-based step count of
 * the bias corrections; max_grad_norm <= 0 skips the clipping; weight_decay is torch.optim.Adam's L2 term.
 * norm_sq (DEVICE, 1 float) receives the squared total gradient norm BEFORE clipping.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pfn_adam_tensor {
  float* p;
  const float* g;
  float* m;
  float* v;
  void* p_bf16;            /* NULL = none */
  long long n;
} pfn_adam_tensor;
int pfn_adam_chunk_elems(void);
int pfn_adam_step(const pfn_adam_tensor* table, const int* chunk_start, int n_tensors, int n_chunks, float lr, float beta1,
                  float beta2, float eps, float weight_decay, float max_grad_norm, int step, float* norm_sq, void* stream);

/* column sums: out[n] += sum_m X[m,n]   (bias gradients; torch autograd of addmm bias) */
int pfn_colsum(const void* X, int ld, int dtype, float* out, int rows, int N, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Bar-distribution NLL (reference bar_distribution.py:19-33 BarDistribution, :83-108 FullSupport).
 *   idx  = searchsorted_left(borders, y) - 1 with the two edge fix-ups (:19-23)             -> int64, bit-exact
 *   nll  = logsumexp(z) - z[idx] + log(width[idx])  (+ half-normal tails when full_support)
 *   rows with idx outside [0, n_bars) are counted in *oob_count (the reference asserts, :27); FullSupport clamps.
 * bwd : dlogits[r,:] = g[r] * (softmax(z[r,:]) - onehot(idx[r]))
 * ---------------------------------------------------------------------------------------------- */
int pfn_bar_nll_fwd(const void* logits, int ld, int dtype, const float* y, const float* borders, int n_bars,
                    int full_support, float* nll, int64_t* idx, float* lse, int* oob_count, int rows, void* stream);
int pfn_bar_nll_bwd(const void* logits, int ld, int dtype, const int64_t* idx, const float* lse, const float* g,
                    void* dlogits, int ld_d, int d_dtype, int n_bars, int n_cols_pad, int rows, void* stream);
int pfn_bar_bucket_idx(const float* y, const float* borders, int n_bars, int64_t* idx, int rows, void* stream);

/* ------------------------------------------------------------------------------------------------
 * GP prior sample (reference priors/fast_gp.py:36-58, priors/fast_gp_mix.py:58-134):
 *   K_b = os_b * k(x_b, x_b; ls_b) + noise_b * I ;  L_b = chol(K_b) ;  y_b = L_b z_b
 * x [Bn, T, F] fp32, z [Bn, T] fp32, ls [Bn, F], os [Bn], noise [Bn] fp32, y [Bn, T] fp32,
 * work [Bn, T, ldw] fp32 scratch, ldw = T rounded up to 4; on return work[b][c][r] = L_b[r][c] (the factor, TRANSPOSED;
 * entries with r < c are unspecified), info [Bn] int (0 ok, k>0: pivot k not positive).
 * jitter is added to every diagonal (gpytorch psd_safe_cholesky retry semantics are driven by the host).
 * ---------------------------------------------------------------------------------------------- */
int pfn_gp_sample(const float* x, const float* z, const float* ls, const float* os, const float* noise, float jitter,
                  int kernel_type, float* y, float* work, int* info, int Bn, int T, int F, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fitted-hyperparameter GP baseline (reference priors/fast_gp_mix.py:24-55,156-169 with priors/fast_gp.py:88-120:
 * botorch SingleTaskGP + fit_gpytorch_model per prefix).  Problem p = i * B + b conditions on rows < ts[i] of dataset b and
 * minimises, by L-BFGS with a More-Thuente line search, the MAP objective in theta = (rho_1..F, rho_s, noise, mean):
 *   f = -(1/t) [ log N(y | mean 1, K) + sum_d log Gamma(ls_d; ls_conc, ls_rate) + log Gamma(s; os_conc, os_rate)
 *                + log Gamma(noise; noise_conc, noise_rate) ],   K = s k_nu(x, x; ls) + noise I,
 *   ls_d = softplus(rho_d), s = softplus(rho_s), noise >= noise_lb (projected), Gamma in rate form.
 * Then, where ts[i] < T, the latent predictive of row ts[i]: mean + k*^T K^-1 (y - mean) and s - k*^T K^-1 k*.
 * One CTA per problem holds the t x t matrix in fp64 shared memory: t <= T <= PFN_GP_FIT_MAX_T, F <= PFN_GP_FIT_MAX_F.
 * max_iter = 0 only evaluates f, its gradient and the predictive at the starting point.
 * x [B, T, F], y [B, T] fp32 (DEVICE); ts (HOST) [n_ts], 1 <= ts[i] <= T; theta0 (DEVICE, optional) [n_ts * B, F + 3];
 * outputs (DEVICE) indexed by problem p: theta [P, F + 3], f [P], grad [P, F + 3] (optional), mean / var [P] (optional; NaN where
 * no predictive is formed), iters / nevals / status [P] int (status: PFN_GP_FIT_*).  Each problem depends on its own inputs only.
 * ---------------------------------------------------------------------------------------------- */
enum { PFN_GP_FIT_MAX_T = 128, PFN_GP_FIT_MAX_F = 32 };
enum { PFN_GP_FIT_CONVERGED = 0, PFN_GP_FIT_MAX_ITER = 1, PFN_GP_FIT_LINE_SEARCH = 2, PFN_GP_FIT_NOT_PD = 3 };
typedef struct pfn_gp_fit_desc {
  int B, T, F;
  const float* x;
  const float* y;
  int n_ts;
  const int* ts;
  int kernel_type;                       /* PFN_KERNEL_MATERN12 / 32 / 52 (nu = 0.5 / 1.5 / 2.5) */
  double ls_conc, ls_rate, os_conc, os_rate, noise_conc, noise_rate;
  double noise_lb;                       /* lower bound of the noise */
  const double* theta0;                  /* NULL: rho = 0, noise = noise_init, mean = 0 */
  double noise_init;
  int max_iter, max_eval;                /* caps on accepted iterations and on objective evaluations */
  double ftol;                           /* stop when (f_old - f) <= ftol * max(|f_old|, |f|, 1) */
  double gtol;                           /* stop when the projected gradient's inf-norm <= gtol */
  double* theta;
  double* f;
  double* grad;
  double* mean;
  double* var;
  int* iters;
  int* nevals;
  int* status;
} pfn_gp_fit_desc;
int pfn_gp_fit(const pfn_gp_fit_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fully Bayesian GP baseline (reference priors/fast_gp_mix.py:171-268 get_mcmc_model / evaluate_: pyro NUTS over the Gamma
 * hyperpriors of the same SingleTaskGP, one chain per prefix).  Problem p = i * B + b samples the posterior of
 * u = log theta, theta = (ls_1..F, s, noise), given rows < ts[i] of dataset b, with the constant mean fixed at 0:
 *   U(u) = -log N(y | 0, s k_nu(x, x; ls) + noise I) - sum_k log Gamma(theta_k; a_k, b_k) - sum_k u_k
 * by NUTS with pyro 1.7's defaults (multinomial sampling, generalised no-U-turn criterion, divergence at an energy error
 * above 1000, step size found by doubling / halving and adapted by dual averaging to acceptance 0.8, diagonal mass matrix
 * adapted in Stan's windows, init u ~ U(-2, 2)).  A trial point whose K is not PD has U = +inf (a divergence).
 * Random numbers are counter-based hashes of (seed, b, ts[i], iteration, draw), never of the CTA index, so a chain is a
 * pure function of its inputs.  After sampling, the latent predictive of rows ts[i] .. ts[i] + n_pred - 1 (those < T) under
 * every sample, one factorisation per sample.
 * One CTA per problem, the limits of pfn_gp_fit: t <= T <= PFN_GP_FIT_MAX_T, F <= PFN_GP_FIT_MAX_F.
 * warmup_steps = num_samples = 0 with init given only evaluates U and its gradient at init (and the predictive there).
 * num_samples = 0 with warmup_steps > 0 runs the warmup only: the one output row is the state the warmup ended in
 * (samples = exp(u), log_samples = u), the predictive is formed at that state, and accept is NaN.
 * A chain without a finite starting point (init given with U = +inf, or none among 100 uniform draws) is not run: its
 * samples, predictive, step size, acceptance and gradient are NaN and its potential is +inf.
 * x [B, T, F], y [B, T] fp32 (DEVICE); ts (HOST) [n_ts]; init (DEVICE, optional) [P, F + 2] values of u.
 * Outputs (DEVICE), S' = max(num_samples, 1): samples [P, S', F + 2] natural values theta; log_samples (optional) the same
 * samples as u, exactly as sampled (an evaluate-only call at these u reproduces the predictive bit for bit); mean / var
 * [P, S', n_pred] (optional, NaN for rows >= T); potential [P] and grad [P, F + 2] (optional) U and dU/du at the chain's last state; step_size [P] (the
 * step size of the sampling phase); accept [P] mean acceptance statistic of the sampling phase; diag [P, PFN_GP_MCMC_NDIAG];
 * trace (optional) [P, warmup_steps + num_samples, F + 4]: per iteration, u after it, the step size it used and its tree depth.
 * ---------------------------------------------------------------------------------------------- */
enum { PFN_GP_MCMC_MAX_DEPTH = 10 };
enum {
  PFN_GP_MCMC_LEAPFROG = 0,        /* leapfrog steps of the NUTS trees (warmup and sampling) */
  PFN_GP_MCMC_EVALS = 1,           /* potential evaluations of all kinds (trees, step-size searches, init, predictive) */
  PFN_GP_MCMC_DIV_WARMUP = 2,      /* iterations ended by a divergence, warmup */
  PFN_GP_MCMC_DIV_SAMPLING = 3,    /* iterations ended by a divergence, sampling */
  PFN_GP_MCMC_MAX_DEPTH_HITS = 4,  /* iterations that reached max_tree_depth */
  PFN_GP_MCMC_NOT_PD = 5,          /* evaluations whose K was not positive definite */
  PFN_GP_MCMC_NDIAG = 6
};
typedef struct pfn_gp_mcmc_desc {
  int B, T, F;
  const float* x;
  const float* y;
  int n_ts;
  const int* ts;
  int kernel_type;                       /* PFN_KERNEL_MATERN12 / 32 / 52 */
  double ls_conc, ls_rate, os_conc, os_rate, noise_conc, noise_rate;
  int num_samples, warmup_steps;
  int max_tree_depth;                    /* 1 .. PFN_GP_MCMC_MAX_DEPTH */
  int n_pred;                            /* predictive rows after the prefix, 1 .. PFN_GP_FIT_MAX_T */
  uint32_t seed;
  const double* init;                    /* NULL: u ~ U(-2, 2) */
  double* samples;
  double* log_samples;
  double* mean;
  double* var;
  double* potential;
  double* grad;
  double* step_size;
  double* accept;
  int* diag;
  double* trace;
} pfn_gp_mcmc_desc;
int pfn_gp_mcmc(const pfn_gp_mcmc_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Stroke prior (reference priors/stroke.py:9-116): per dataset, C classes of 1..3 random strokes; per image, the strokes of
 * its class drawn with a random width, offset and end-point jitter like PIL's ImageDraw.line, ink filled with U{200..254},
 * ImageFilter.GaussianBlur(0.2), ToTensor (k / 255) and optionally per-image standardisation.
 * All ranges are inclusive integer ranges (random.randint), already scaled by the image side S (int(S * fraction)).
 * pfn_stroke_geometry : the rejection loop of every (dataset, class, stroke), capped at max_iters iterations (a capped stroke
 *   sets *cap_flag = 1 and keeps its last draw; the flag is never cleared here).  geom [B, C, strokes_max, 4] int32 receives
 *   (start x, start y, length, active) and turns [B, C, strokes_max] fp64 the direction as a fraction of a full turn
 *   (radians = 2 pi turns).
 * pfn_stroke_render : x [T, B, S*S] fp32 (sequence-first) for the class table cls [T, B] int32 (values in [0, C)).
 * Both draw their random numbers from counter-based hashes of `seed` (no device RNG state).
 * pfn_stroke_raster : the oracle hook.  Rasterises N images of side S, image i being the union of segs[i, 0..nseg[i]-1]
 *   (segs [N, K, 4] int32 end points x0, y0, x1, y1; x = column) at width widths[i]; mask [N, S*S] uint8 receives 1 on ink
 *   pixels, blurred [N, S*S] uint8 the GaussianBlur(0.2) of the image whose ink pixels hold fill [N, S*S] (NULL: 128).
 * S <= PFN_STROKE_MAX_SIDE, strokes per class and K <= PFN_STROKE_MAX_STROKES.
 * ---------------------------------------------------------------------------------------------- */
enum { PFN_STROKE_MAX_STROKES = 16, PFN_STROKE_MAX_SIDE = 112 };
typedef struct pfn_stroke_desc {
  int S;                           /* image side; an image has S*S pixels */
  int C;                           /* classes per dataset */
  int strokes_min, strokes_max;    /* strokes per class */
  int len_min, len_max;            /* stroke length */
  int start_min, start_max;        /* start point coordinate */
  int width_min, width_max;        /* line width per image */
  int offset_min, offset_max;      /* per-image offset of every start point */
  int jitter_min, jitter_max;      /* per-image, per-stroke integer jitter of each velocity component */
  int max_iters;                   /* rejection cap per stroke */
} pfn_stroke_desc;
int pfn_stroke_geometry(const pfn_stroke_desc* d, uint32_t seed, int B, int* geom, double* turns, int* cap_flag,
                        void* stream);
int pfn_stroke_render(const pfn_stroke_desc* d, uint32_t seed, const int* cls, const int* geom, const double* turns,
                      float* x, int T, int B, int normalize, void* stream);
int pfn_stroke_raster(const int* segs, const int* nseg, const int* widths, const uint8_t* fill, uint8_t* mask,
                      uint8_t* blurred, int N, int K, int S, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Omniglot few-shot episodes (reference priors/omniglot.py:36-72, datasets/omniglotNshot.py:16-77,172-230).
 * bank [n_classes, PFN_OMNIGLOT_IMAGES, S, S] uint8 holds the resized grey-level images (Pillow 'L', 255 = background);
 * pixel value v becomes (float)(1.0 - v / 255.0), the reference's float64 inversion cast to float32.
 * One CTA per episode b writes x [T, B, S*S] fp32, y [T, B] int64 (label of every position, the query's included) and
 * target_y [T, B] int64 (-100 except the last row, which equals y), T = n_way * k_shot + 1; the support rows come first
 * and the query is the last row.
 *   jonas = 0 (OmniglotNShot) : n_way distinct classes of pool_lo .. pool_lo + pool_n - 1, class j gets label j; per class
 *     k_shot + 1 distinct images (the last is the query image) and one rot90 turn shared by its images; support rows in a
 *     uniformly random order; the query is the image of a uniformly chosen class.
 *   jonas = 1 (OmniglotNShotJonas) : a uniform alphabet a < n_alpha; the classes are characters alpha_start[a] + 0..n_way-1
 *     in a random order, label = position; support class-major, no rotation.  train = 1: k_shot + 1 distinct images per
 *     class; train = 0: the support is images 0..k_shot-1 in a random order, the query image is uniform on k_shot..19.
 *     alpha_start (DEVICE, n_alpha ints) holds the first class of every alphabet of the split; every alphabet has at least
 *     alpha_min >= n_way characters.
 *   translate = 1 : every image is shifted by integer (tx, ty), uniform over the shifts that keep its ink (pixels != 255)
 *     inside the image, with NEAREST sampling and fill 0 (out[r][c] = in[r - ty][c - tx]); an image without ink is not shifted.
 * Random numbers are counter-based hashes of `seed`.  n_way <= PFN_OMNIGLOT_MAX_WAY, S <= PFN_OMNIGLOT_MAX_SIDE.
 * ---------------------------------------------------------------------------------------------- */
enum { PFN_OMNIGLOT_IMAGES = 20, PFN_OMNIGLOT_MAX_WAY = 64, PFN_OMNIGLOT_MAX_SIDE = 105 };
typedef struct pfn_omniglot_desc {
  int S;                           /* image side */
  int n_classes;                   /* classes in the bank */
  int B;                           /* episodes */
  int n_way, k_shot, T;            /* T = n_way * k_shot + 1 */
  int jonas, train, translate;
  int pool_lo, pool_n;             /* jonas = 0: the class pool */
  int n_alpha, alpha_min;          /* jonas = 1: alphabets of the split and the size of the smallest */
} pfn_omniglot_desc;
int pfn_omniglot_episodes(const pfn_omniglot_desc* d, uint32_t seed, const uint8_t* bank, const int* alpha_start, float* x,
                          int64_t* y, int64_t* target_y, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Bayesian-NN prior (reference priors/pyro.py:10-34 over mcmc_svi_transformer_on_bayesian.py:28-67 BayesianModel): per
 * dataset b, theta = (W1 [E, F], b1 [E], W2 [2, E], b2 [2]) ~ N(0, 1) (d = E F + 3 E + 2 values in that order), x [T, F] ~
 * N(0, 1), logits = W2 (W1 x + b1) + b2 (no nonlinearity between the layers, as in the reference), class ~ softmax(logits)
 * (class 0 when u < p_0 for u ~ U[0, 1)), then x standardised over the sequence axis per dataset and feature
 * ((x - mean) / (unbiased std + 1e-6)).  One CTA per dataset.  The normals are fp32 values; logits, softmax and the
 * statistics of the standardisation are formed from them in fp64.  Random numbers are counter-based hashes of
 * (seed, dataset_offset + b, counters): dataset b of a batch equals a one-dataset call with dataset_offset = b bit for bit.
 * x [T, B, F] fp32, y [T, B] fp32 (0. / 1.).  The oracle hook, all optional (NULL on the product path): weights [B, d] fp32,
 * x_raw [T, B, F] fp32 (x before the standardisation), u [T, B] fp64 (the uniform of every class draw).
 * d <= PFN_BNN_MAX_D; T * F fp32 values must fit in shared memory beside theta (an error otherwise).
 * ---------------------------------------------------------------------------------------------- */
enum { PFN_BNN_MAX_D = 1024 };
int pfn_bnn_prior(uint32_t seed, int dataset_offset, int B, int T, int F, int E, float* x, float* y, float* weights,
                  float* x_raw, double* u, void* stream);

/* ------------------------------------------------------------------------------------------------
 * NUTS baseline of the Bayesian NN (reference mcmc_svi_transformer_on_bayesian.py:249-267 eval_mcmc: one pyro NUTS chain per
 * dataset).  Chain b samples the posterior of theta (layout above, all sites N(0, 1), so unconstrained) given the n training
 * rows of dataset b:
 *   U(theta) = 1/2 |theta|^2 + d/2 log 2 pi - sum_r log softmax(W2 (W1 x_r + b1) + b2)[y_r]
 * with the algorithm, constants and random-number keys of pfn_gp_mcmc (keys (seed, b, n, iteration, draw)).  One CTA per
 * chain; every d-vector of the sampler (79 of them, the trial point always in shared memory: chain state, trajectory ends, the per-level stack of complete subtrees,
 * the mass-matrix accumulators) lives in dynamic shared memory when it fits and otherwise in `workspace`, which the caller
 * allocates: pfn_bnn_mcmc_workspace returns the doubles needed PER CHAIN (0 when shared memory holds the state, -1 for an
 * invalid descriptor); workspace then has N times that many doubles and need not be initialised.  All arithmetic is fp64.
 * After sampling, the class-1 probability of each of the n_test rows under every kept sample.
 * warmup_steps = num_samples = 0 with init given only evaluates U and its gradient (and the probabilities) at init.
 * num_samples = 0 with warmup_steps > 0 runs the warmup only: the one output row of samples (and of probs / obs) is the
 * state the warmup ended in, and accept is NaN.
 * A chain whose starting point has no finite potential is not run: its outputs are NaN and its potential +inf.
 * x_train [N, n, F], y_train [N, n] (0. / 1.), x_test [N, n_test, F] fp32 (DEVICE; x_test may be NULL when n_test = 0);
 * init (DEVICE, optional) [N, d].  Outputs (DEVICE), S' = max(num_samples, 1): samples [N, S', d]; probs (optional)
 * [N, S', n_test]; obs (optional) [N, S', n_test] fp32: one class (0. / 1.) drawn per sample and row from probs, with the
 * chain's keys at iteration warmup_steps + num_samples + 1 (what pyro's predictive returns as 'obs'); potential [N] and grad [N, d] (optional) at the chain's last state; step_size, accept [N];
 * diag [N, PFN_GP_MCMC_NDIAG] (the counters of pfn_gp_mcmc; NOT_PD counts evaluations whose U was not finite);
 * trace (optional) [N, warmup_steps + num_samples, d + 2]: per iteration theta after it, the step size used, the tree depth.
 * d <= PFN_BNN_MAX_D, n <= PFN_BNN_MAX_N.
 * ---------------------------------------------------------------------------------------------- */
enum { PFN_BNN_MAX_N = 1024, PFN_BNN_MCMC_VECTORS = 79 };
typedef struct pfn_bnn_mcmc_desc {
  int N, n, n_test, F, E;
  const float* x_train;
  const float* y_train;
  const float* x_test;
  int num_samples, warmup_steps;
  int max_tree_depth;                    /* 1 .. PFN_GP_MCMC_MAX_DEPTH */
  uint32_t seed;
  const double* init;                    /* NULL: theta ~ U(-2, 2) */
  double* samples;
  double* probs;
  float* obs;
  double* potential;
  double* grad;
  double* step_size;
  double* accept;
  int* diag;
  double* trace;
  double* workspace;                     /* [N, pfn_bnn_mcmc_workspace(d)] doubles; NULL when that is 0 */
} pfn_bnn_mcmc_desc;
int pfn_bnn_mcmc_workspace(const pfn_bnn_mcmc_desc* d);
int pfn_bnn_mcmc(const pfn_bnn_mcmc_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * KNN baseline of the tabular evaluation (reference tabular.py:350-369 knn_metric): for each of S problems,
 * GridSearchCV(KNeighborsClassifier(), {'n_neighbors': 1 .. K}, cv=StratifiedKFold(min(5, n // 2))) on its n training
 * rows, then the class-1 probability of its m test rows under the refit with the best k.  K = min(5, n - 2).  One CTA per
 * problem, all problems in one launch.  Neighbours: Euclidean in fp64 from direct differences, ordered by (distance, row);
 * vote ties predict class 0; the best k is the first maximal mean CV accuracy.
 * x [n + m, S, F] fp32 (rows 0 .. n-1 train, n .. n+m-1 test), y [n, S] fp32 labels (0. / 1.).  Outputs (DEVICE):
 * proba [m, S] fp64 (count of class-1 neighbours / k), k_best [S] int32, cv_mean [S, K] fp64 (NaN for a candidate larger
 * than some fold's training set), status [S] int32 (PFN_KNN_*; a problem that is not OK has NaN outputs and k_best 0).
 * 4 <= n <= PFN_KNN_MAX_N, F <= PFN_KNN_MAX_F.
 * ---------------------------------------------------------------------------------------------- */
enum { PFN_KNN_MAX_N = 1024, PFN_KNN_MAX_F = 1024, PFN_KNN_MAX_K = 5, PFN_KNN_MAX_SPLITS = 5 };
enum { PFN_KNN_OK = 0, PFN_KNN_BAD_LABEL = 1, PFN_KNN_FEW_MEMBERS = 2, PFN_KNN_ONE_CLASS = 3 };
typedef struct pfn_knn_cv_desc {
  int S, n, m, F;
  const float* x;
  const float* y;
  double* proba;
  int* k_best;
  double* cv_mean;
  int* status;
} pfn_knn_cv_desc;
int pfn_knn_cv(const pfn_knn_cv_desc* d, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PFN_B200_H_ */

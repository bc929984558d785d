/* cfm_b200.h -- C ABI of libcfm_b200.so (sm_90a kernels for torchcfm's two hot paths).
 *
 * The reference (atong01/conditional-flow-matching, torchcfm 1.0.7) is pure Python and
 * has no FFI of its own; the boundary below is what a binding for its hot path would
 * have to provide.  Each entry point names the reference interface it replaces
 * (paths relative to the reference root).  All pointers are DEVICE pointers unless the
 * name ends in `_host`; sizes are element counts unless stated; every call is
 * asynchronous on `stream` (a cudaStream_t passed as void*), allocates nothing and
 * keeps no state besides a per-thread error string.  Return value: 0 = ok, <0 = error
 * (see CFM_ERR_*; text via cfm_last_error()).  Numerical conditions are reported
 * through device-resident status words, never through the return value.
 */
#ifndef CFM_B200_H_
#define CFM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CFM_ABI_VERSION 2

#define CFM_OK 0
#define CFM_ERR_ARG (-1)   /* bad argument (shape, alignment, null pointer, workspace too small) */
#define CFM_ERR_CUDA (-2)  /* a CUDA runtime call failed */
#define CFM_ERR_ARCH (-3)  /* device is not sm_90 / kernel image missing */

/* status-word bit flags written by the solvers (device int32) */
#define CFM_FLAG_NONFINITE 1      /* optimal_transport.py:88-92  "p is not finite"            */
#define CFM_FLAG_ZERO_MASS 2      /* optimal_transport.py:93-96  uniform-plan fallback taken  */
#define CFM_FLAG_NOT_CONVERGED 4  /* POT "Sinkhorn did not converge" (numItermax reached)     */
#define CFM_FLAG_INFEASIBLE 8     /* exact assignment found no augmenting path (inf/nan cost) */

/* activations for cfm_mlp_forward_f32 */
#define CFM_ACT_SELU 0 /* torchcfm/models/models.py:12,14,16 (the reference MLP) */
#define CFM_ACT_SILU 1 /* notebook-local MLP2 variant named by BASELINE.json north_star */

/* ---- library ---------------------------------------------------------------- */
int cfm_abi_version(void);
const char* cfm_last_error(void);
/* sm count and compute capability (major*10+minor) of the current device */
int cfm_device_info(int* sm_count, int* cc);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
long long cfm_launch_count(void);

/* ---- (a3) cost matrix: M = torch.cdist(x0, x1) ** 2 --------------------------
 * replaces torchcfm/optimal_transport.py:84 (and :176, :297-299).
 * x0 (n0,d), x1 (n1,d) fp32 row-major contiguous; M (n0, n1) fp32 with row stride ldm.
 * M_ij = (sqrt(max(|x0_i|^2 + |x1_j|^2 - 2 x0_i.x1_j, 0)))^2 when squared != 0, the
 * un-squared distance otherwise (wasserstein power=1, :297).
 * cost_max (nullable, 1 float): receives max_ij M_ij (the M.max() of :86); must be
 * zeroed by the caller... it is zeroed by this call.
 * algo: 0 auto, 1 SIMT fp32 FMA, 3 wgmma fp16x3 (x = hi + lo 2^-11 in fp16, three fp16 wgmma MMAs into two
 * accumulators: fp32-grade accuracy; what auto picks for aligned shapes).  Any other value, 2 included (a
 * retired 3xTF32 path), fails with "unknown algo".
 */
size_t cfm_sqdist_workspace_bytes(int n0, int n1, int d, int algo);
int cfm_sqdist_f32(const float* x0, const float* x1, float* M, int n0, int n1, int d,
                   int64_t ldm, int squared, float* cost_max, int algo, void* workspace,
                   size_t workspace_bytes, void* stream);

/* ---- (a4) entropic plan: log-domain Sinkhorn on uniform marginals ---------------
 * replaces pot.sinkhorn(a, b, M, reg) as bound at optimal_transport.py:51 and called
 * at :87 (POT algorithm: ot/bregman/_sinkhorn.py::sinkhorn_log; a = b = pot.unif, :79).
 * M (n0,n1) fp32; if normalize != 0 the cost used is M / *cost_max (:85-86).
 * Iterates v then u (POT order), at most max_iters times; every `check_every`
 * iterations (POT: 10) the column-marginal L2 error is tested against stop_thr.
 * precise: 0 = fp32 exponent arithmetic (|M/reg| <~ 64), 1 = float64 potentials and
 * IEEE fp32 division for -M/reg exactly as NumPy forms it, -1 = choose on device from
 * *cost_max / reg, 2 = fp32 arithmetic forced onto the generic (L2-reuse) kernel, 3 = float64
 * potentials and exponent arguments with fp32 exponentials (terms good to ~1e-7).  In mode 3 (and in -1 when it
 * resolves to it) every term of a log-sum-exp is first screened in fp32 against (running maximum - 32): terms
 * more than ~30 units below the maximum (< 1e-13 of it) skip the float64 path; 4 = mode 3 without that
 * screening (cross-checks).
 * Outputs: log_u (n0), log_v (n1) float64 natural-log potentials with
 *   plan_ij = exp(-M_ij/reg + log_u_i + log_v_j);
 * stall_tol: 0 = POT's stopping rule only.  > 0 additionally stops at a check when the
 * error improved by less than this fraction since the previous check AND the RMS
 * relative column-marginal error is already < 1e-5 (fp32 fixed point reached; POT's
 * float64 loop would keep shaving an error our fp32 exponents cannot resolve).
 * status: int32[4] = {flags, iterations run, arithmetic used (0 fp32, 1 float64, 2 mode 3), kernel variant};
 * err: float64[1] last evaluated column-marginal L2 error.
 */
size_t cfm_sinkhorn_workspace_bytes(int n0, int n1);
int cfm_sinkhorn_log_f32(const float* M, int n0, int n1, int64_t ldm, float reg,
                         const float* cost_max, int normalize, int max_iters,
                         double stop_thr, int check_every, int precise, double stall_tol,
                         double* log_u, double* log_v, int32_t* status, double* err,
                         void* workspace, size_t workspace_bytes, void* stream);

/* materialise the float64 plan (what OTPlanSampler.get_map returns, :63-97) from the
 * potentials; also accumulates total mass into mass[0] (float64) and sets
 * CFM_FLAG_NONFINITE in *status when an entry is not finite. */
int cfm_plan_materialize_f64(const float* M, int n0, int n1, int64_t ldm, float reg,
                             const float* cost_max, int normalize, const double* log_u,
                             const double* log_v, double* plan, double* mass,
                             int32_t* status, void* stream);

/* <P, M> = sum_ij plan_ij * M_ij into out[0] (float64): the value pot.sinkhorn2 returns
 * (optimal_transport.py:288, called at :300 by wasserstein()). */
int cfm_plan_dot_cost(const float* M, int n0, int n1, int64_t ldm, float reg,
                      const float* cost_max, int normalize, const double* log_u,
                      const double* log_v, double* out, void* stream);

/* ---- (a6) pair sampling ---------------------------------------------------------
 * replaces OTPlanSampler.sample_map for replace=True (optimal_transport.py:116-121):
 * inverse-CDF draw over the row-major flattened plan for `n_draws` uniforms in [0,1)
 * (the caller draws them with np.random.random_sample to keep the reference's RNG
 * stream), returning row and column indices (int64, like np.divmod).
 * The plan is never materialised: entries are recomputed from (M, log_u, log_v).
 * workspace: cfm_plan_sample_workspace_bytes(n0).  If the total mass is < 1e-8 the
 * uniform plan is sampled instead and CFM_FLAG_ZERO_MASS is set (:93-96).
 * uniform_rows != 0: the potentials come from a solve whose last update was the row update
 * (always true for cfm_sinkhorn_log_f32), so every row has mass exactly 1/n0: the row-mass
 * pass is skipped and the within-row inversion weighs column j by pi_ij itself (exponent
 * -M_ij/reg + log_u_i + log_v_j <= 0: no under/overflow at any |M/reg|; formed in fp32 when
 * |M/reg| <= 64 and with float64 adds beyond, the rule cfm_sinkhorn_log_f32's auto mode uses).
 * A walk whose target lies past the weights' own sum is repeated against that sum, and the
 * row is totalled first when status[2] == 0 (fp32 solve) and |M/reg| > 64, so the draw is
 * never a column of weight 0.
 */
size_t cfm_plan_sample_workspace_bytes(int n0);
int cfm_plan_sample(const float* M, int n0, int n1, int64_t ldm, float reg,
                    const float* cost_max, int normalize, const double* log_u,
                    const double* log_v, int uniform_rows, const double* uniforms, int n_draws,
                    int64_t* i_out, int64_t* j_out, int32_t* status, void* workspace,
                    size_t workspace_bytes, void* stream);
/* row-conditional draw, replaces the per-sample loop of OTPlanSampler.sample_trajectory
 * (optimal_transport.py:239-248: np.random.choice(n1, p=pi[i] / pi[i].sum()) for i in rows):
 * j_out[k] = searchsorted(cumsum(pi[rows[k], :]) / sum(pi[rows[k], :]), uniforms[k], 'right') with
 * the plan row recomputed from (M, log_v).  log_u cancels in the row normalisation; it is used (when not
 * NULL) only to centre the exponents, -M_ij/reg + log_u_i + log_v_j = log pi_ij <= 0, so that no row can
 * under- or overflow at large |M/reg|; with log_u == NULL a row-maximum pass does the centring. */
int cfm_plan_sample_rows(const float* M, int n0, int n1, int64_t ldm, float reg,
                         const float* cost_max, int normalize, const double* log_u,
                         const double* log_v, const int64_t* rows, const double* uniforms,
                         int n_draws, int64_t* j_out, int32_t* status, void* stream);
/* same draw for a dense float64 plan already in device memory (staged parity test) */
int cfm_dense_plan_sample_f64(const double* plan, int n0, int n1, const double* uniforms,
                              int n_draws, int64_t* i_out, int64_t* j_out,
                              void* workspace, size_t workspace_bytes, void* stream);
/* exact-OT plan P_sigma/N: cdf is the N-step staircase `stairs` (float64, n entries,
 * the normalised sequential cumsum the reference forms); i = searchsorted(stairs, u,
 * 'right'), j = sigma[i]. */
int cfm_perm_plan_sample(const int32_t* sigma, const double* stairs, int n,
                         const double* uniforms, int n_draws, int64_t* i_out,
                         int64_t* j_out, void* stream);

/* ---- (a4, exact) optimal assignment on uniform marginals -------------------------
 * replaces pot.emd(a, b, M) as bound at optimal_transport.py:49 / called at :87, and
 * scipy.optimize.linear_sum_assignment at :179.  For a = b = 1/n the LP vertex is
 * P_sigma / n; this returns sigma (column of each row), solved by a shortest-
 * augmenting-path method in float64 on the fp32 costs (the reference casts M to
 * float64 too).  total_cost (float64[1]) = sum_i M[i, sigma_i] (emd2 * n, :300).
 * status: int32[3] = {flags, augmentations, Dijkstra steps}.
 */
size_t cfm_assign_workspace_bytes(int n);
int cfm_assign_exact_f32(const float* M, int n, int64_t ldm, const float* cost_max,
                         int normalize, int32_t* sigma, double* total_cost,
                         int32_t* status, void* workspace, size_t workspace_bytes,
                         void* stream);

/* ---- (a7) gather: out[k, :] = x[idx[k], :] ---------------------------------------
 * replaces x0[i], x1[j] at optimal_transport.py:145 / :213-218.  elem_bytes in {1,2,4,8}.
 */
int cfm_gather_rows(const void* x, int64_t row_elems, int elem_bytes, const int64_t* idx,
                    int64_t n_idx, void* out, void* stream);

/* ---- (a8, SURVEY 8 f-1) fused pair gather + path sample + conditional flow ------------
 * replaces x0[i], x1[j] (optimal_transport.py:145) followed by sample_xt /
 * compute_conditional_flow (conditional_flow_matching.py:104-154; overrides :329-394 target,
 * :429-478 Schrodinger bridge, :569-618 variance preserving) with one pass:
 *   reads x0[i_idx[r]], x1[j_idx[r]], eps[r]  ->  writes xt[r], ut[r]      (n rows of row_elems)
 * i_idx / j_idx NULL = identity pairing.  Per-row coefficient vectors (n floats, computed by the
 * caller with the reference's own expressions so results stay bit-identical):
 *   ICFM/OT : row_a = t, row_b = 1 - t                      sigma_t = `sigma`
 *   TARGET  : row_a = t, row_sigma = row_c = 1 - (1-sigma) t  konst = 1 - sigma
 *   SB      : row_a = t, row_b = 1 - t, row_sigma = sigma sqrt(t(1-t)), row_c = (1-2t)/(2t(1-t)+1e-8)
 *   VP      : row_a = cos(pi t / 2), row_b = sin(pi t / 2)    sigma_t = `sigma`, konst = pi / 2
 * row_sigma NULL = use the scalar `sigma`.  Every element op is an unfused, round-to-nearest fp32 op
 * in the reference's association order. */
#define CFM_FLOW_ICFM 0
#define CFM_FLOW_TARGET 1
#define CFM_FLOW_SB 2
#define CFM_FLOW_VP 3
int cfm_flow_pairs_f32(int kind, const float* x0, const float* x1, const int64_t* i_idx,
                       const int64_t* j_idx, const float* eps, const float* row_a, const float* row_b,
                       const float* row_sigma, const float* row_c, float sigma, float konst, float* xt,
                       float* ut, int64_t n, int64_t row_elems, void* stream);

/* ---- (a9/a10) MLP vector field ----------------------------------------------------
 * replaces torchcfm.models.MLP.forward (torchcfm/models/models.py:20-21) composed with
 * torch_wrapper.forward (torchcfm/utils.py:51-52): y = net(cat([x, t], 1)).
 * x (B, dim) fp32 contiguous.  Weights in torch.nn.Linear layout W_l (out_l, in_l),
 * b_l (out_l); `in_0 = dim + time_varying`.  When time_varying != 0, t is a scalar
 * shared by the batch and is folded into the first-layer bias; it is read from
 * *t_dev (device float) when t_dev != NULL, else t_host is used.
 * prepared: opaque device blob built once per weight set by cfm_mlp_prepare (split /
 * padded copies of the weights); workspace holds the two hidden activations.
 * algo: 0 auto (the tensor-core paths when cfm_mlp_tc_supported() accepts the shape and x, y and
 * the workspace are 16-byte aligned, SIMT fp32 otherwise), 1 SIMT fp32, 2 tensor cores (fails on a
 * shape or a pointer they cannot take).
 */
size_t cfm_mlp_prepared_bytes(int dim, int w, int out_dim, int time_varying);
int cfm_mlp_prepare(const float* W0, const float* b0, const float* W1, const float* b1,
                    const float* W2, const float* b2, const float* W3, const float* b3,
                    int dim, int w, int out_dim, int time_varying, void* prepared,
                    size_t prepared_bytes, void* stream);
size_t cfm_mlp_workspace_bytes(int batch, int dim, int w, int out_dim, int algo);
int cfm_mlp_forward_f32(const void* prepared, const float* x, int batch, int dim, int w,
                        int out_dim, int time_varying, const float* t_dev, float t_host,
                        int act, float* y, int algo, void* workspace,
                        size_t workspace_bytes, void* stream);

/* Same forward for an input that already exists as the tensor-core operand pair of the fp16x3 scheme
 * (fp16 arrays of B*dim elements: x_hi = fp16(x), x_lo = fp16((x - x_hi) * 2048), as written by
 * cfm_rk_stage_input); tensor-core paths only: ONE fused persistent launch for 256-wide hidden layers
 * (activations stay in shared memory), per-layer GEMM launches otherwise.  cfm_mlp_tc_supported() != 0
 * tells whether a shape runs on them.  Device-side gate: when *skip_if_nonzero != 0 (nullable) the fused kernel
 * returns at once.  The dopri5 driver passes &state->done, so that steps enqueued speculatively after the
 * integration has finished cost a launch, not a forward (the per-layer path ignores the gate: its result is simply
 * unused). */
int cfm_mlp_tc_supported(int batch, int dim, int w, int out_dim);
int cfm_mlp_forward_split_gated_f32(const void* prepared, const void* x_hi, const void* x_lo, int batch,
                                    int dim, int w, int out_dim, int time_varying, const float* t_dev,
                                    float t_host, int act, float* y, const int32_t* skip_if_nonzero,
                                    void* workspace, size_t workspace_bytes, void* stream);

/* ---- (a11) dopri5 lock-step driver pieces -------------------------------------------
 * replaces the arithmetic of torchdyn's NeuralODE(solver="dopri5").trajectory (call
 * sites: examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb:332-338;
 * torchdyn >= 1.0.6 is an un-vendored dependency, setup.py:13).  The batch advances in
 * lock-step with ONE scalar step size, so all step-control state lives in a device
 * struct and a whole step is enqueued without a host round trip.  Driver:
 * cfm_b200/ode.py.  Buffers are fp32 with numel = B*D elements: x, xnew, xs and
 * k = 7 contiguous stage derivatives k1..k7.
 */
typedef struct cfm_rk_state {
  float t, dt, t_end, atol, rtol;
  float dt_old;          /* step saved when a checkpoint clipped dt (also h0 during init) */
  float ratio;           /* last error ratio (hairer norm)                                */
  int32_t ckpt_flag;     /* dt was clipped to land on t_span[ckpt]                         */
  int32_t ckpt;          /* next t_span index to record                                    */
  int32_t n_span;        /* len(t_span)                                                    */
  int32_t commit;        /* last step accepted: cfm_rk_commit applies it                   */
  int32_t done;          /* t >= t_end                                                     */
  int32_t save_slot;     /* >= 0: commit also copies the new state into traj[save_slot]    */
  int32_t accepted, rejected, nfe;
  double err_acc;        /* sum((err/tol)^2) accumulated by cfm_rk_error_norm              */
} cfm_rk_state;

/* stage in 1..5: out = x + dt*sum_j a[stage][j]*k_j (input of stage+1's evaluation);
 * stage 6: the same with the 5th-order weights, i.e. out = xnew (and the FSAL input).
 * out (nullable) receives the fp32 value; out_hi/out_lo (nullable pair, fp16 arrays of numel elements)
 * receive its fp16x3 operand split, the form cfm_mlp_forward_split_gated_f32 consumes.  *t_stage (device
 * float, nullable) = t + c[stage]*dt.  err_partial (nullable, stage 6 only, numel floats): receives
 * sum_{j<=6} e_j k_j, the first six terms of the embedded error estimate -- stage 6 reads k1..k6 anyway, so
 * cfm_rk_error_norm can then read four arrays instead of eight. */
int cfm_rk_stage_input(const cfm_rk_state* st, const float* x, const float* k, float* out,
                       void* out_hi, void* out_lo, float* t_stage, float* err_partial, int64_t numel,
                       int stage, void* stream);
/* st->err_acc += sum((dt*sum_j e_j k_j / (atol + rtol*max(|x|,|xnew|)))^2); with err_partial (see above) the
 * sum over j is err_partial + e_7 k_7 */
int cfm_rk_error_norm(cfm_rk_state* st, const float* x, const float* xnew, const float* k,
                      const float* err_partial, int64_t numel, void* stream);
/* accept/reject, checkpoint bookkeeping, step-size adaptation, clipping of the next dt */
int cfm_rk_control(cfm_rk_state* st, const float* t_span, int64_t numel, void* stream);
/* if the step was accepted: x <- xnew, k1 <- k7 (FSAL), traj[save_slot] <- xnew */
int cfm_rk_commit(const cfm_rk_state* st, float* x, const float* xnew, float* k, float* traj,
                  int64_t numel, void* stream);
/* Hairer initial step (torchdyn init_step) around the f(t0+h0, x+h0*f0) evaluation, in four calls so that
 * row-sharded (lock-step) integration across ranks (SURVEY section 8e) can all-reduce between them:
 * cfm_rk_init_sums accumulates this shard's partial sums into scratch (4 doubles; phase 0: zeroes scratch, then
 * sum (x/scale)^2 and sum (f0/scale)^2; phase 1: sum ((f1-f0)/scale)^2); the driver all-reduces scratch over the
 * ranks; cfm_rk_init_probe (writes x_probe and *t_stage) and cfm_rk_init_finish (finishes dt and clips it) then
 * take the GLOBAL element count.  cfm_rk_control's numel is likewise the global count when st->err_acc has been
 * all-reduced. */
int cfm_rk_init_sums(const cfm_rk_state* st, const float* x, const float* f0, const float* f1,
                     double* scratch, int64_t numel, int phase, void* stream);
int cfm_rk_init_probe(cfm_rk_state* st, const float* x, const float* f0, float* x_probe, float* t_stage,
                      const double* scratch, int64_t numel, int64_t numel_global, void* stream);
int cfm_rk_init_finish(cfm_rk_state* st, const float* t_span, const double* scratch, int64_t numel_global,
                       void* stream);
/* x_out = x + h * k  (fixed-step Euler, torchdyn solver="euler") */
int cfm_axpy_f32(const float* x, const float* k, float h, float* x_out, int64_t numel,
                 void* stream);

/* ---- (f-2) whole-trajectory sampling for small vector-field MLPs, ONE launch -----------------
 * replaces torchdyn's NeuralODE(...).trajectory(x, t_span) loop for the reference's 2-D tutorial
 * models (examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb:332-338: MLP(dim=2,
 * w=64, time_varying=True), 1024 samples, 100 t_span points; runner/src/models/components/
 * solver.py:184-199), where a forward is microseconds and per-kernel launch latency dominates.
 * Weights are passed in torch.nn.Linear layout ([out][in], fp32; W0 is [w][dim + time_varying],
 * time is the LAST input column as torch_wrapper concatenates it, torchcfm/utils.py:51-52).
 * solver: 0 dopri5 (same controller semantics as the cfm_rk_* pieces above), 1 euler (one step per
 * t_span interval).  traj: [n_span][batch][dim].  state_out receives t, nfe, accepted, rejected,
 * done (done == 0 means the step budget ran out).  supported(): w in {32, 64, 128}, out_dim == dim
 * and the per-row state fits in shared memory.  workspace: cfm_ode_small_workspace_bytes(). */
int cfm_ode_small_supported(int64_t batch, int dim, int w, int out_dim);
size_t cfm_ode_small_workspace_bytes(int64_t batch, int dim, int w);
int cfm_ode_small_trajectory_f32(const float* W0, const float* b0, const float* W1, const float* b1,
                                 const float* W2, const float* b2, const float* W3, const float* b3,
                                 int dim, int w, int time_varying, int act, const float* x0,
                                 int64_t batch, const float* t_span, int n_span, float atol,
                                 float rtol, int solver, float* traj, cfm_rk_state* state_out,
                                 void* workspace, size_t workspace_bytes, void* stream);
/* Exact-likelihood (CNF) variant of the above: the state is [x, ll] with dim + 1 columns and the field is
 * [f(t, x), tr(df/dx)] (the log-density column LAST, with +div as its derivative), traced per row by forward-mode
 * tangents through the same MLP.  x0 is [batch][dim + 1], traj [n_span][batch][dim + 1]; every other argument,
 * the workspace and the state are as for cfm_ode_small_trajectory_f32, and the error norms cover all
 * batch * (dim + 1) elements.  supported(): w in {32, 64, 128}, dim <= 8 and the per-row state and tangent
 * buffers fit in shared memory. */
int cfm_ode_small_cnf_supported(int64_t batch, int dim, int w);
int cfm_ode_small_cnf_trajectory_f32(const float* W0, const float* b0, const float* W1, const float* b1,
                                     const float* W2, const float* b2, const float* W3, const float* b3,
                                     int dim, int w, int time_varying, int act, const float* x0,
                                     int64_t batch, const float* t_span, int n_span, float atol,
                                     float rtol, int solver, float* traj, cfm_rk_state* state_out,
                                     void* workspace, size_t workspace_bytes, void* stream);
/* Gradients through the CNF variant's Euler trajectory (solver = 1, time_varying = 1): given the trajectory traj
 * [n_span][batch][dim + 1] that cfm_ode_small_cnf_trajectory_f32 wrote for the same weights and t_span, and
 * grad_traj = dL/dtraj of the same shape, writes dL/dtheta for the eight parameters into grads (flat, in
 * parameters() order: W0 [w][dim + 1], b0, W1, b1, W2, b2, W3 [dim][w], b3) and, when grad_z is not null, dL/dx0
 * into grad_z [batch][dim + 1].  The exact gradient of the computed fp32 Euler trajectory (a discrete adjoint over
 * the stored states), in one cooperative launch with a deterministic fold: the same bits on every call.
 * supported(): w in {32, 64}, 1 <= dim <= 8 and a batch cfm_ode_small_cnf_supported accepts.  workspace:
 * cfm_ode_small_cnf_backward_workspace_bytes(). */
int cfm_ode_small_cnf_backward_supported(int64_t batch, int dim, int w);
size_t cfm_ode_small_cnf_backward_workspace_bytes(int64_t batch, int n_span, int dim, int w);
int cfm_ode_small_cnf_euler_backward_f32(const float* W0, const float* b0, const float* W1, const float* b1,
                                         const float* W2, const float* b2, const float* W3, const float* b3,
                                         int dim, int w, int act, const float* traj, int64_t batch,
                                         const float* t_span, int n_span, const float* grad_traj, float* grad_z,
                                         float* grads, void* workspace, size_t workspace_bytes, void* stream);
/* Gradient-field variant (action matching: torch_wrapper(GradModel(action)) of the 2-D tutorial): the field is
 * f(t, x) = grad_x s(t, x) of a scalar action s = MLP(dim, out_dim = 1, w, time_varying), evaluated per row by one
 * forward and one reverse pass through the same MLP.  W3 is [1][w] and b3 [1] (b3 does not enter the gradient);
 * x0 is [batch][dim] and traj [n_span][batch][dim]; every other argument, the workspace
 * (cfm_ode_small_workspace_bytes(batch, dim, w)) and the state are as for cfm_ode_small_trajectory_f32.
 * supported(): w in {32, 64}, dim <= 8 and the weights (W1 and W2 twice) plus the per-row state fit in shared
 * memory. */
int cfm_ode_small_grad_supported(int64_t batch, int dim, int w);
int cfm_ode_small_grad_trajectory_f32(const float* W0, const float* b0, const float* W1, const float* b1,
                                      const float* W2, const float* b2, const float* W3, const float* b3,
                                      int dim, int w, int time_varying, int act, const float* x0,
                                      int64_t batch, const float* t_span, int n_span, float atol,
                                      float rtol, int solver, float* traj, cfm_rk_state* state_out,
                                      void* workspace, size_t workspace_bytes, void* stream);

/* ---- Schrodinger-bridge SDE sampling for small MLPs, ONE launch -----------------------------------------------
 * replaces torchsde.sdeint(sde, y0, ts, method="euler") for the SDE class of the SF2M examples
 * (examples/2D_tutorials/SF2M_tutorial.ipynb cell 5, examples/single_cell/single-cell_example.ipynb cell 16):
 * dy = [drift(t, y) + score(t, y)] dt + sigma dW, Ito, diagonal noise, fixed-step Euler-Maruyama.
 * drift_host, score_host: HOST arrays of 8 device pointers {W0, b0, W1, b1, W2, b2, W3, b3} each, torch.nn.Linear
 * layout, both MLP(dim, w, time_varying=True) with out_dim == dim (time is the last input column).
 * grid: [n_steps + 1] step times; step n is y += h f(t_n, y) + sigma dW with h = grid[n + 1] - grid[n], evaluated
 * as fmaf(h, drift + score, y) + sigma * dW.  traj: [n_out][batch][dim]; traj[0] = x0, and output k >= 1 is
 * out_a[k] * y_before + out_b[k] * y_after of the step n with out_begin[n] <= k < out_begin[n + 1]
 * (out_begin: [n_steps + 1] ints).  increments (nullable): [n_steps][batch][dim] Brownian increments; when null
 * the kernel draws dW = sqrt(h) z with z from Philox4x32-10 (counter (c / 4, row lo, row hi, n), key (seed lo,
 * seed hi)) and Box-Muller, a function of (seed, n, row, column) only.  supported(): w in {32, 64} and the two
 * weight sets plus the per-row state fit in shared memory. */
int cfm_sde_small_supported(int64_t batch, int dim, int w);
int cfm_sde_small_euler_f32(const float* const* drift_host, const float* const* score_host, int dim, int w, int act,
                            float sigma, const float* x0, int64_t batch, const float* grid, int n_steps,
                            const int* out_begin, const float* out_a, const float* out_b, int n_out, uint64_t seed,
                            const float* increments, float* traj, void* stream);

/* ---- Schrodinger-bridge SDE sampling for WIDE MLPs, on the tensor cores -------------------------------------------
 * The same SDE, step grid, output interpolation, update expression and noise stream as cfm_sde_small_euler_f32, for
 * drift and score nets in the tensor-core class (e.g. the MNIST model MLP(784, w=256, time_varying=True)): a driver
 * (cfm_b200/sde.py) calls cfm_sde_tc_init once per trajectory and then, per step, cfm_mlp_pair_forward_split_f32 on
 * (y_hi, y_lo) with t_dev = &state->t followed by cfm_sde_tc_euler_step.  Every per-trajectory value the step needs
 * lives in the device state, so the two step calls can be captured once and replayed n_steps times.
 * supported(): exactly cfm_mlp_tc_supported(batch, dim, w, dim): batch >= 128, dim >= 32, dim and w multiples of 8,
 * w >= 32. */
typedef struct cfm_sde_state {
  uint64_t seed;            /* key of the device noise stream                                   */
  float* traj;              /* [n_out][batch][dim]                                              */
  const float* increments;  /* nullable: [n_steps][batch][dim] Brownian increments              */
  int32_t n;                /* next step                                                        */
  int32_t n_steps;
  float t;                  /* grid[n]: the time the forward of step n reads                    */
  uint32_t ticket;          /* CTAs of the running step that are done (0 between steps)         */
} cfm_sde_state;
int cfm_sde_tc_supported(int batch, int dim, int w);
/* Both nets (prepared_a, prepared_b: cfm_mlp_prepare blobs of one shape) on the same fp16x3 operand pair:
 * y_a = net_a(x), y_b = net_b(x), each with the bits cfm_mlp_forward_split_gated_f32 gives it.  For 256-wide hidden
 * layers and dim >= 64 this is ONE persistent launch over 2 ceil(batch / 128) slabs (net a's, then net b's);
 * otherwise the per-layer launches of each net in turn.  workspace: 2 * cfm_mlp_workspace_bytes(batch, dim, w,
 * out_dim, 2) bytes, 16-byte aligned.  Argument errors are reported before any CUDA call. */
int cfm_mlp_pair_forward_split_f32(const void* prepared_a, const void* prepared_b, const void* x_hi, const void* x_lo,
                                   int batch, int dim, int w, int out_dim, int time_varying, const float* t_dev,
                                   float t_host, int act, float* y_a, float* y_b, void* workspace,
                                   size_t workspace_bytes, void* stream);
/* state <- (seed, n = 0, t = grid[0], traj, increments); y = traj[0] = y0 (fp32 [batch][dim]) and (y_hi, y_lo) =
 * its fp16x3 operand split (fp16 [batch][dim] each, the split cfm_mlp_forward_f32 applies to an fp32 input).  Without
 * increments the step draws dW = sqrt(h) z with z from the stream of cfm_sde_small_euler_f32: a given (seed, step,
 * row, column) draws the same z in both classes. */
int cfm_sde_tc_init(cfm_sde_state* state, const float* y0, float* y, void* y_hi, void* y_lo, float* traj,
                    const float* increments, uint64_t seed, const float* grid, int n_steps, int batch, int dim,
                    void* stream);
/* Step n = state->n: y <- fmaf(h, drift + score, y) + sigma dW with h = grid[n + 1] - grid[n]; writes the outputs
 * out_begin[n] <= k < out_begin[n + 1] of traj, y and (y_hi, y_lo), then n += 1 and t = grid[n + 1].  drift and
 * score: [batch][dim] fp32 evaluated at (t, y).  A step enqueued after the last one does nothing.  All arrays
 * 16-byte aligned; argument errors are reported before any CUDA call. */
int cfm_sde_tc_euler_step(cfm_sde_state* state, float* y, const float* drift, const float* score, void* y_hi,
                          void* y_lo, const float* grid, const int* out_begin, const float* out_a, const float* out_b,
                          float sigma, int batch, int dim, void* stream);

/* ---- Hutchinson log-likelihood of WIDE MLP flows, on the tensor cores --------------------------------------------
 * replaces the field of cnf_wrapper(model, likelihood_estimator="hutch_gaussian" / "hutch_rademacher")
 * (examples/2D_tutorials/Maximum_likelihood_CNF_tutorial.ipynb, get_div_and_eps) for MLP(dim, w, time_varying=True)
 * with out_dim == dim in the tensor-core class: d/dt [x, ll] = [f(t, x), eps . (J eps)], J = df/dx at (t, x), with a
 * fresh probe eps per evaluation.  Entry (r, c) of probe n is the normal of the SDE noise stream (Philox4x32-10 counter
 * (c / 4, r lo, r hi, n), key (seed lo, seed hi), Box-Muller) or, for Rademacher, -1 where the top bit of Philox word
 * c % 4 of the same counter is set and +1 otherwise: a function of (seed, n, r, c) only.
 * supported(): exactly cfm_mlp_tc_supported(batch, dim, w, dim). */
#define CFM_HUTCH_GAUSSIAN 0
#define CFM_HUTCH_RADEMACHER 1
int cfm_cnf_tc_supported(int batch, int dim, int w);
size_t cfm_cnf_tc_workspace_bytes(int batch, int dim, int w);
/* One field evaluation at (t = *t_dev, x) for `batch` rows: f [batch][dim] (row stride dim) and div [batch], fp32,
 * any 4-byte alignment.  x is given either as fp32 [batch][dim] (x_hi = x_lo = NULL; split here) or as its fp16x3
 * operand pair (x = NULL), as cfm_rk_stage_input writes it.  The probe ordinal is *ordinal_dev + ordinal_offset and
 * the seed *seed_dev, both read on the device, so a captured evaluation replays with new values.  prepared: the
 * cfm_mlp_prepare blob (time_varying = 1, out_dim = dim).  Ten launches: probe (and x split), four primal and four
 * tangent GEMMs, the fold of the per-chunk float64 partials of eps . (J eps) in a fixed order (the same call gives the
 * same bits).  x, x_hi, x_lo and the workspace 16-byte aligned; argument errors are reported before any CUDA call. */
int cfm_cnf_tc_field_f32(const void* prepared, const float* x, const void* x_hi, const void* x_lo, int batch, int dim,
                         int w, int act, int estimator, const float* t_dev, const uint64_t* seed_dev,
                         const int32_t* ordinal_dev, int ordinal_offset, float* f, float* div, void* workspace,
                         size_t workspace_bytes, void* stream);
/* Euler driver state: step n evaluates the field at (t = t_span[n], x_n) with probe ordinal n (torchdyn's count). */
typedef struct cfm_cnf_tc_state {
  uint64_t seed;          /* key of the probe stream                                          */
  float* traj;            /* [n_span][batch][dim + 1]                                         */
  const float* t_span;    /* [n_span] fp32                                                    */
  int32_t n;              /* next step (and the probe ordinal of its evaluation)              */
  int32_t n_steps;        /* n_span - 1                                                       */
  float t;                /* t_span[n]: the time the evaluation of step n reads               */
  uint32_t ticket;        /* CTAs of the running step that are done (0 between steps)         */
} cfm_cnf_tc_state;
/* state <- (seed, traj, t_span, n = 0, t = t_span[0]); z0 [batch][dim + 1] -> x [batch][dim], ll [batch], traj[0] and
 * (x_hi, x_lo), the fp16x3 operand split of x.  x, x_hi, x_lo 16-byte aligned. */
int cfm_cnf_tc_euler_init(cfm_cnf_tc_state* state, const float* z0, float* x, float* ll, void* x_hi, void* x_lo,
                          float* traj, const float* t_span, int n_span, uint64_t seed, int batch, int dim,
                          void* stream);
/* Step n = state->n with h = (float)((double)t_span[n + 1] - (double)t_span[n]): x <- fmaf(h, f, x),
 * ll <- fmaf(h, div, ll), traj[n + 1], (x_hi, x_lo); then n += 1, t = t_span[n + 1].  A step enqueued after the last
 * one does nothing.  x, f, x_hi, x_lo 16-byte aligned. */
int cfm_cnf_tc_euler_step(cfm_cnf_tc_state* state, float* x, float* ll, const float* f, const float* div, void* x_hi,
                          void* x_lo, int batch, int dim, void* stream);

/* ---- the action-matching gradient field of WIDE scalar actions, on the tensor cores ------------------------------
 * replaces the field of torch_wrapper(GradModel(MLP(dim, out_dim=1, w, time_varying=True))) (action matching,
 * examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb cells 10-11) for actions in the tensor-core
 * class: v(t, x) = grad_x s(t, x) = W0x^T (D0 * W1^T (D1 * W2^T (D2 * W3[0, :]^T))), D_l = act'(pre_l).
 * supported(): B >= 128, dim >= 32, dim and w multiples of 8, w >= 32 (cfm_mlp_tc_supported(batch, dim, w, dim)).
 * Two blobs: mlp_prepared, the cfm_mlp_prepare blob of the action (out_dim = 1, time_varying = 1), and the blob of
 * cfm_grad_tc_prepare, the K-major transposed fp16x3 pairs of W0x, W1 and W2 built from it (one launch; rebuild both
 * when the weights change).  prepared_bytes() is 0 outside the class. */
int cfm_grad_tc_supported(int batch, int dim, int w);
size_t cfm_grad_tc_prepared_bytes(int dim, int w);
int cfm_grad_tc_prepare(const void* mlp_prepared, int dim, int w, void* prepared, size_t prepared_bytes, void* stream);
size_t cfm_grad_tc_workspace_bytes(int batch, int dim, int w);
/* One field evaluation at (t = *t_dev, x) for `batch` rows: v [batch][dim] fp32, row stride dim, any 4-byte
 * alignment.  x is given either as fp32 [batch][dim] (x_hi = x_lo = NULL; split here) or as its fp16x3 operand pair
 * (x = NULL), as cfm_rk_stage_input writes it.  Six launches (seven with an fp32 x): three primal and three reverse
 * GEMMs; no atomics, so the same call gives the same bits.  x, x_hi, x_lo, both blobs and the workspace 16-byte
 * aligned; argument errors are reported before any CUDA call. */
int cfm_grad_tc_field_f32(const void* mlp_prepared, const void* grad_prepared, const float* x, const void* x_hi,
                          const void* x_lo, int batch, int dim, int w, int act, const float* t_dev, float* v,
                          void* workspace, size_t workspace_bytes, void* stream);
/* Euler driver state: step n evaluates the field at (t = t_span[n], x_n). */
typedef struct cfm_grad_tc_state {
  float* traj;            /* [n_span][batch][dim]                                             */
  const float* t_span;    /* [n_span] fp32                                                    */
  int32_t n;              /* next step                                                        */
  int32_t n_steps;        /* n_span - 1                                                       */
  float t;                /* t_span[n]: the time the evaluation of step n reads               */
  uint32_t ticket;        /* CTAs of the running step that are done (0 between steps)         */
} cfm_grad_tc_state;
/* state <- (traj, t_span, n = 0, t = t_span[0]); x0 [batch][dim] -> x, traj[0] and (x_hi, x_lo), the fp16x3 operand
 * split of x.  x0, x, x_hi, x_lo and traj 16-byte aligned. */
int cfm_grad_tc_euler_init(cfm_grad_tc_state* state, const float* x0, float* x, void* x_hi, void* x_lo, float* traj,
                           const float* t_span, int n_span, int batch, int dim, void* stream);
/* Step n = state->n with h = (float)((double)t_span[n + 1] - (double)t_span[n]): x <- fmaf(h, v, x), traj[n + 1],
 * (x_hi, x_lo); then n += 1, t = t_span[n + 1].  A step enqueued after the last one does nothing.  x, v, x_hi, x_lo
 * 16-byte aligned. */
int cfm_grad_tc_euler_step(cfm_grad_tc_state* state, float* x, const float* v, void* x_hi, void* x_lo, int batch,
                           int dim, void* stream);

/* ---- training step of small vector-field MLPs: the regression loss and all parameter gradients, ONE launch ------
 * replaces the three lines every training cell of the 2-D tutorials repeats per step
 * (examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb raw lines 166-186, 310-330, 458-479, 602-623;
 * Flow_matching_tutorial.ipynb and SF2M_tutorial.ipynb likewise):
 *     vt = model(torch.cat([xt, t[:, None]], dim=-1)); loss = torch.mean((vt - ut) ** 2); loss.backward()
 * for model = MLP(dim, out_dim, w, time_varying=True).  Computes
 *     *loss = mean over [batch][out_dim] of (row_scale[r] * MLP([x_r, t_r]) - target[r])^2     (row_scale null: 1)
 * and, when with_grad != 0, d loss / d parameter into grads: W0 [w][dim + 1], b0 [w], W1 [w][w], b1, W2 [w][w], b2,
 * W3 [out_dim][w], b3 [out_dim], flat in that order (torch's parameters() order).  Weights are in torch.nn.Linear
 * layout ([out][in], fp32) with time as the LAST column of W0; x is [batch][dim], t [batch] (one time per row),
 * target [batch][out_dim], row_scale [batch].  No input gradients.  grads may be null iff with_grad == 0; the loss has
 * the same bits either way, and a call repeated on the same device gives the same bits (per-CTA partial sums folded
 * in CTA order, no atomics).  supported(): w in {32, 64}, 1 <= dim <= 8, 1 <= out_dim <= 8, batch >= 1; rows stream
 * from device memory, so the batch is not bounded by shared memory.  Argument errors are reported before any CUDA
 * call. */
int cfm_mlp_small_train_supported(int64_t batch, int dim, int w, int out_dim);
size_t cfm_mlp_small_train_workspace_bytes(int64_t batch, int dim, int w, int out_dim);
int cfm_mlp_small_mse_grad_f32(const float* W0, const float* b0, const float* W1, const float* b1,
                               const float* W2, const float* b2, const float* W3, const float* b3,
                               int dim, int w, int out_dim, int act, const float* x, const float* t,
                               const float* target, const float* row_scale, int64_t batch, int with_grad,
                               float* loss, float* grads, void* workspace, size_t workspace_bytes,
                               void* stream);

/* The action-matching loss of the 2-D tutorial (tutorial_training_8_gaussians_to_moons.ipynb, cell 11), which the
 * notebook differentiates with a double backward:
 *     loss = mean_r [ s(x0_r, 0) - s(x1_r, 1) + 1/2 sum_{d < dim} (d s / d x_d)(xt_r, t_r)^2 + (d s / d t)(xt_r, t_r) ]
 * for the scalar action s = MLP(dim, out_dim=1, w, time_varying=True).  When with_grad != 0, d loss / d parameter goes
 * to grads in the layout of cfm_mlp_small_mse_grad_f32 with out_dim = 1; the gradient of b3 is exactly 0 (b3 cancels
 * in s(x0) - s(x1) and does not enter grad s).  xt, x0, x1 are [batch][dim], t [batch].  The workspace is sized by
 * cfm_mlp_small_train_workspace_bytes(batch, dim, w, 1).  grads may be null iff with_grad == 0; the loss has the same
 * bits either way, and a call repeated on the same device gives the same bits.  Supported: w in {32, 64},
 * 1 <= dim <= 8, batch >= 1, SELU or SiLU.  Argument errors are reported before any CUDA call. */
int cfm_mlp_small_action_grad_f32(const float* W0, const float* b0, const float* W1, const float* b1,
                                  const float* W2, const float* b2, const float* W3, const float* b3,
                                  int dim, int w, int act, const float* xt, const float* t, const float* x0,
                                  const float* x1, int64_t batch, int with_grad, float* loss, float* grads,
                                  void* workspace, size_t workspace_bytes, void* stream);

/* The same loss, gradients, grads layout, row_scale and with_grad contract as cfm_mlp_small_mse_grad_f32 for WIDE
 * models, on the tensor cores (fp16x3 wgmma GEMMs, fp32-grade): the class the tensor-core forward samples,
 * cfm_mlp_tc_supported's shapes (dim >= 32, dim % 8 == 0, w >= 32, w % 8 == 0, out_dim % 4 == 0) with any
 * 1 <= batch <= 2^30, e.g. MLP(784, w=256, time_varying=True).  A fixed number of launches per call: 19 with
 * with_grad != 0, 8 without (DESIGN.md section 3.15).  The workspace (cfm_mlp_tc_train_workspace_bytes, 0 outside the
 * class) must be 16-byte aligned; the weights are split into it anew on every call.  A call repeated on the same
 * device gives the same bits, and the loss has the same bits with and without gradients.  Argument errors are
 * reported before any CUDA call. */
int cfm_mlp_tc_train_supported(int64_t batch, int dim, int w, int out_dim);
size_t cfm_mlp_tc_train_workspace_bytes(int64_t batch, int dim, int w, int out_dim);
int cfm_mlp_tc_mse_grad_f32(const float* W0, const float* b0, const float* W1, const float* b1,
                            const float* W2, const float* b2, const float* W3, const float* b3,
                            int dim, int w, int out_dim, int act, const float* x, const float* t,
                            const float* target, const float* row_scale, int64_t batch, int with_grad,
                            float* loss, float* grads, void* workspace, size_t workspace_bytes,
                            void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CFM_B200_H_ */

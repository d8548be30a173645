/*
 * ppsci_b200.h — C-ABI of the H100-native (sm_90a) PINN PDE-residual engine.
 *
 * The reference (PaddlePaddle/PaddleScience) has no FFI: its seam for this path is the
 * Python call  ExpressionSolver.train_forward(...)  followed by  total_loss.backward()
 *   (ppsci/utils/expression.py:60-131, ppsci/solver/train.py:117-158).
 * This header is the boundary a maintainer would bind *under* that seam (ctypes stub in
 * INTEGRATION.md).  Each entry point names the reference code it replaces.
 *
 * Conventions
 *   - plain pointers and sizes only; every device buffer is caller-owned
 *   - all work is enqueued on the caller's stream (cudaStream_t passed as void*)
 *   - every function returns 0 on success, non-zero on error; ppsci_b200_last_error()
 *     returns a thread-local human readable message
 *   - handles are not thread-safe
 */
#ifndef PPSCI_B200_H_
#define PPSCI_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PPSCI_MAX_IN 8      /* raw input columns (x, y, z, t, ...)                       */
#define PPSCI_MAX_FEAT 32   /* MLP input features after period embedding                 */
#define PPSCI_MAX_LAYERS 16 /* linear layers (hidden + last_fc)                          */
#define PPSCI_MAX_DIR 8     /* univariate Taylor directions                              */
#define PPSCI_MAX_ORDER 4   /* highest Taylor order per direction                        */
#define PPSCI_MAX_RES 16    /* residual (equation) outputs per call (one constraint, or a batch of them) */
#define PPSCI_MAX_REG 256   /* register file of the residual program                     */
#define PPSCI_MAX_PGRAD 32  /* (residual, learnable parameter) gradient terms per plan    */

/* dtype */
enum { PPSCI_F32 = 0, PPSCI_F64 = 1 };

/* activation of the hidden layers — ppsci/arch/activation.py:139-154 */
enum {
  PPSCI_ACT_TANH = 0,
  PPSCI_ACT_SIN = 1,
  PPSCI_ACT_COS = 2,
  PPSCI_ACT_SIGMOID = 3,
  PPSCI_ACT_SILU = 4, /* x*sigmoid(x): "silu" and "swish"(beta=1) */
  PPSCI_ACT_IDENTITY = 5,
  PPSCI_ACT_RELU = 6,
  PPSCI_ACT_GELU = 7, /* erf form (paddle nn.GELU default approximate=False) */
  PPSCI_ACT_ELU = 8,        /* nn.ELU(alpha = 1):  x > 0 ? x : exp(x) - 1 */
  PPSCI_ACT_SELU = 9,       /* nn.SELU: scale * (x > 0 ? x : alpha * (exp(x) - 1)), scale = 1.0507009873554805, alpha = 1.6732632423543772 */
  PPSCI_ACT_LEAKY_RELU = 10, /* nn.LeakyReLU(negative_slope = 0.01) */
  PPSCI_ACT_SIREN = 11,     /* Siren(w0 = 30): sin(30 x)  (activation.py:89-101) */
  /* Activations with a TRAINABLE parameter (plain MLP plans, CUDA-core kernels).  Their parameters sit behind every
   * other entry of the parameter / gradient buffers, hidden layer by hidden layer: */
  PPSCI_ACT_STAN = 12,      /* Stan (activation.py:28-46): tanh(x) (1 + beta x), one beta per unit (widths[l] values per layer), 1 at start */
  PPSCI_ACT_SWISH_B = 13,   /* Swish (activation.py:49-58): x sigmoid(beta x), one beta per layer, 1 at start */
  PPSCI_ACT_LAST = 13
};

/* input feature kinds — identity, or PeriodEmbedding (ppsci/arch/mlp.py:95-114) */
enum { PPSCI_FEAT_ID = 0, PPSCI_FEAT_COS = 1, PPSCI_FEAT_SIN = 2 };

/* residual program opcodes (register machine; see DESIGN.md "residual program") */
enum {
  PPSCI_OP_CONST = 0, /* dst = consts[a]            */
  PPSCI_OP_MOV = 1,   /* dst = r[a]                 */
  PPSCI_OP_ADD = 2,   /* dst = r[a] + r[b]          */
  PPSCI_OP_SUB = 3,
  PPSCI_OP_MUL = 4,
  PPSCI_OP_DIV = 5,
  PPSCI_OP_NEG = 6,
  PPSCI_OP_POWI = 7, /* dst = r[a] ** b (b = small signed int immediate) */
  PPSCI_OP_POW = 8,  /* dst = pow(r[a], r[b])      */
  PPSCI_OP_SIN = 9,
  PPSCI_OP_COS = 10,
  PPSCI_OP_TANH = 11,
  PPSCI_OP_EXP = 12,
  PPSCI_OP_LOG = 13,
  PPSCI_OP_SQRT = 14,
  PPSCI_OP_ABS = 15,
  PPSCI_OP_MAX = 16,
  PPSCI_OP_MIN = 17,
  PPSCI_OP_SIGN = 18,
  PPSCI_OP_FMA = 19, /* dst = r[a] * r[b] + r[dst]  (accumulate form) */
  PPSCI_OP_SINH = 20,
  PPSCI_OP_COSH = 21,
  PPSCI_OP_HEAVISIDE = 22,
};

/* MSELoss reduction — ppsci/loss/mse.py:82-106 */
enum { PPSCI_REDUCE_MEAN = 0, PPSCI_REDUCE_SUM = 1 };

/*
 * One compiled constraint: network + jet layout + residual program + loss.
 *
 * Jet layout.  Channel 0 is the value.  Direction d (d < n_dir) is the raw-input-space
 * vector dir_vec[d][0..n_in) and owns dir_order[d] channels holding the NORMALISED Taylor
 * coefficients  (1/k!) d^k/dt^k f(x + t v)|_{t=0},  k = 1..dir_order[d].
 * C = 1 + sum_d dir_order[d].  Channel index of (d, k) = 1 + sum_{e<d} dir_order[e] + (k-1).
 *
 * Residual program.  Register file r[0..n_reg).  Before the program runs, the engine loads
 *   r[c*n_out + j]                 = output-jet channel c of network output j
 *   r[C*n_out + i]                 = raw input column i          (i < n_in)
 *   r[C*n_out + n_in + a]          = auxiliary column a          (a < n_aux)
 * then executes prog (n_ops quads: op, dst, a, b).  Residual k is r[res_reg[k]].
 * grad_* lists the non-zero partials  d res[grad_res[g]] / d r[grad_in[g]]  (grad_in is an
 * output-jet register) found in r[grad_reg[g]] — produced by the same program.
 */
typedef struct ppsci_plan_spec {
  int32_t dtype;
  /* network — replaces ppsci/arch/mlp.py:281-315 (forward_tensor / forward) */
  int32_t n_in;
  int32_t n_feat;
  int32_t feat_src[PPSCI_MAX_FEAT];
  int32_t feat_kind[PPSCI_MAX_FEAT];
  double feat_omega[PPSCI_MAX_FEAT];
  int32_t n_layers;                     /* linear layers, >= 1                      */
  int32_t widths[PPSCI_MAX_LAYERS + 1]; /* widths[0] = n_feat ... widths[n_layers] = n_out */
  int32_t act;
  /* jets — replaces ppsci/autodiff/ad.py:56-160,196-303 (reverse-mode sweeps) */
  int32_t n_dir;
  int32_t dir_order[PPSCI_MAX_DIR];
  double dir_vec[PPSCI_MAX_DIR][PPSCI_MAX_IN];
  /* residual program — replaces ppsci/utils/symbolic.py:184-504 node execution */
  int32_t n_aux;
  int32_t n_reg;
  int32_t n_ops;
  const int32_t* prog; /* n_ops * 4 int32 (copied at plan_create) */
  int32_t n_consts;
  const double* consts; /* copied at plan_create */
  int32_t n_res;
  int32_t res_reg[PPSCI_MAX_RES];
  int32_t n_grad;
  const int32_t* grad_res; /* [n_grad] */
  const int32_t* grad_in;  /* [n_grad] register index < C*n_out */
  const int32_t* grad_reg; /* [n_grad] */
  /* loss — replaces ppsci/loss/mse.py:82-106 and ppsci/loss/mtl/sum.py:45-60 */
  int32_t reduction[PPSCI_MAX_RES];
  double loss_weight[PPSCI_MAX_RES];
  /* tuning */
  int32_t chunk_points; /* points per internal chunk (0 = default) */
  int32_t backend;      /* 0 = auto, 1 = force SIMT kernels, 2 = require the wgmma tensor-core kernels */
  /* Dense first-layer operand (DeepONet branch net, ppsci/arch/deeponet.py:96-106: MLP(input_dim=num_loc)):
   * when non-zero, n_in must be 1, x_cols[0] is a row-major [n_points][n_feat] matrix (n_feat up to 4096, the
   * feat_* arrays are ignored) and no input derivatives are available (n_dir must be 0). */
  int32_t dense_in;
  /* Activation applied to the output of the FIRST linear layer when it differs from `act` (PPSCI_ACT_* id), or -1:
   * FourierEmbedding (ppsci/arch/mlp.py:117-136, 298-315) is  [cos(x B), sin(x B)] = sin(x [B | B] + [pi/2 | 0]),
   * i.e. one more linear layer with tied weights whose activation is sin whatever the network's own activation is.
   * A plan with act_first != act runs on the CUDA-core kernels (the tensor-core kernels are specialised for one
   * activation across the layers they fuse). */
  int32_t act_first;
  /* Learnable scalar parameters of the equations — replaces ParameterNode (ppsci/utils/symbolic.py:471-485) and the
   * autograd path into PDE.learnable_parameters (ppsci/equation/pde/base.py:38, e.g. Vibration, pde/viv.py:41-60):
   * an auxiliary column flagged in aux_bcast is ONE device scalar (of the plan's dtype) read by every point, and the
   * n_pgrad triples (residual k, aux index, register holding d residual_k / d parameter) make the head kernel
   * accumulate dLoss/dparameter into the fp64 device scalar registered with ppsci_b200_plan_set_aux_grad. */
  int32_t aux_bcast[PPSCI_MAX_IN];
  int32_t n_pgrad;
  int32_t pgrad_res[PPSCI_MAX_PGRAD];
  int32_t pgrad_aux[PPSCI_MAX_PGRAD];
  int32_t pgrad_reg[PPSCI_MAX_PGRAD];
  /* Gated networks.  0: plain MLP.
   * 1 — ModifiedMLP.forward_tensor (ppsci/arch/mlp.py:488-506): two extra layers
   *       U = act(x Wu + bu),  V = act(x Wv + bv)            (embed_u / embed_v)
   *     and after every hidden layer  y <- y * U + (1 - y) * V  (a truncated Taylor product per jet direction).
   *     With act_first >= 0 (a Fourier embedding as layer 1) x is layer 1's stored output, otherwise the features.
   * 2 — PirateNet.forward_tensor over PirateNetBlock.forward (mlp.py:617-624, 800-809): layer 1 is the embedding
   *     (width = the blocks' width), then blocks of three layers: gate, gate, x <- alpha act(z3) + (1 - alpha) x
   *     with one trainable alpha per block; n_layers = 1 + 3 * blocks + 1.
   * Needs n_layers >= 2 (+1 with an embedding layer), equal widths of the gated layers, no dense_in.  Parameter /
   * gradient buffers: [W_1 | b_1 | ... | W_L | b_L | Wu | bu | Wv | bv | alpha_0 ... alpha_{B-1}].  Gated plans run on
   * the CUDA-core kernels (csrc/kernels_gate.cuh + the generic tile GEMMs); two-phase value calls are not offered. */
  int32_t gated;
} ppsci_plan_spec;

typedef struct ppsci_plan ppsci_plan;

/* Build a plan.  Validates the spec, copies the residual program to the device (five small buffers, freed by
 * plan_destroy); every other byte of device memory the calls touch is caller-owned workspace. */
int ppsci_b200_plan_create(const ppsci_plan_spec* spec, ppsci_plan** out);
void ppsci_b200_plan_destroy(ppsci_plan* plan);

/* Number of parameters in the flat buffer: for each layer l, W_l [in,out] row-major
 * (the reference's nn.Linear layout, ppsci/arch/mlp.py:246,274) followed by b_l [out]. */
int64_t ppsci_b200_plan_param_count(const ppsci_plan* plan);

/* Where the loss-and-gradient calls ACCUMULATE dLoss/d(aux parameter `aux_index`) (a device fp64 scalar owned by the
 * caller; NULL = do not accumulate).  Only meaningful for aux columns flagged in aux_bcast. */
int ppsci_b200_plan_set_aux_grad(ppsci_plan* plan, int32_t aux_index, double* grad_dev);
int32_t ppsci_b200_plan_channels(const ppsci_plan* plan);

/* Bytes of caller-provided device workspace needed for a call with n_points points. */
size_t ppsci_b200_plan_workspace_bytes(const ppsci_plan* plan, int64_t n_points);

/*
 * Forward jets + residuals + MSE + adjoint -> weight gradient.  One call per constraint per
 * step; replaces  ExpressionSolver.train_forward (ppsci/utils/expression.py:60-131)  +
 * total_loss.backward() (ppsci/solver/train.py:158)  for that constraint.
 *
 *   x_cols[i]      device pointer to raw input column i, n_points contiguous values
 *   aux_cols[a]    device pointer to auxiliary column a (may be NULL if n_aux == 0)
 *   label_cols[k]  label column of residual k, or NULL  -> label_const[k]
 *   weight_cols[k] per-point weight column of residual k, or NULL -> 1
 *   n_norm         denominator used by "mean" reductions (normally n_points)
 *   params         flat parameter buffer (see plan_param_count)
 *   grads          flat gradient buffer, ACCUMULATED in place (supports update_freq > 1,
 *                  ppsci/solver/train.py:141-164); may be NULL to skip the adjoint
 *   loss_out       n_res device scalars, OVERWRITTEN with the per-residual loss
 *   residual_out   optional: n_res device columns receiving the raw residual values
 */
int ppsci_b200_residual_loss_fwd_bwd(ppsci_plan* plan, const void* const* x_cols,
                                     const void* const* aux_cols,
                                     const void* const* label_cols,
                                     const double* label_const,
                                     const void* const* weight_cols, int64_t n_points,
                                     int64_t n_norm, const void* params, void* grads,
                                     void* loss_out, void* const* residual_out,
                                     void* workspace, size_t workspace_bytes, void* stream);

/*
 * Forward only: network outputs and/or output jets for eval / predict / lambdify parity.
 * Replaces Arch.forward (ppsci/arch/mlp.py:298-315) and ComposedNode.forward
 * (ppsci/utils/symbolic.py:498-504) without a loss.
 *   jets_out   optional device buffer [C][n_points][n_out] receiving NORMALISED Taylor
 *              coefficients per channel (channel 0 = network outputs)
 *   residual_out optional n_res device columns
 */
int ppsci_b200_residual_fwd(ppsci_plan* plan, const void* const* x_cols,
                            const void* const* aux_cols, int64_t n_points,
                            const void* params, void* jets_out, void* const* residual_out,
                            void* workspace, size_t workspace_bytes, void* stream);

/* Kernel launches enqueued by the most recent call on this plan (for bench accounting). */
int64_t ppsci_b200_plan_last_launches(const ppsci_plan* plan);

/* Test accessor: byte offset inside the (256-aligned) workspace of the jet planes of `layer`
 * ([C][min(n_points, chunk)][round4(width)]); layer == n_layers addresses the output jets. */
int64_t ppsci_b200_plan_stash_offset(const ppsci_plan* plan, int64_t n_points, int32_t layer);

/* Forward + adjoint of the network VALUES for caller-supplied output adjoints: runs the forward pass (stash), seeds
 * the value channel of the output adjoints with ybar[n_points][n_out] (row-major, dL/dy computed by the caller),
 * and accumulates dL/d(params) into grads.  No residual program, no loss.  This is how a model that combines
 * several MLPs outside the kernels (DeepONet: G = sum_i branch_i * act(trunk_i) + b, deeponet.py:129-154) gets its
 * weight gradients: the combination and the loss are elementwise work on [N, features] done by the caller. */
int ppsci_b200_values_fwd_bwd(ppsci_plan* plan, const void* const* x_cols, const void* const* aux_cols,
                              int64_t n_points, const void* params, void* grads, const void* ybar,
                              void* workspace, size_t workspace_bytes, void* stream);

/* Two-phase variant of values_fwd_bwd for callers whose output adjoints depend on the outputs (DeepONet: the product /
 * loss head sits between the forward and the adjoint of its two MLPs): values_fwd_keep runs the forward exactly as a
 * training call does (everything the adjoint reads stays in `workspace`) and writes the network outputs
 * y_out[n_points][n_out]; values_bwd_kept then runs ONLY the adjoint from that stash — the forward is not recomputed.
 * Both calls take at most plan_chunk_points points, the same inputs / params / workspace, and nothing else may use the
 * workspace in between.  In-place use (no copies): y_out may be NULL — the outputs are then read at
 * workspace + plan_stash_offset(plan, n_points, n_layers) as [n_points][ld], ld = n_out rounded up to a multiple of 4 —
 * and ybar may be workspace + plan_stash_offset(plan, n_points, 300) (same layout), written by the caller's head kernel. */
int32_t ppsci_b200_plan_chunk_points(const ppsci_plan* plan);
int ppsci_b200_values_fwd_keep(ppsci_plan* plan, const void* const* x_cols, const void* const* aux_cols,
                               int64_t n_points, const void* params, void* y_out, void* workspace,
                               size_t workspace_bytes, void* stream);
int ppsci_b200_values_bwd_kept(ppsci_plan* plan, const void* const* x_cols, const void* const* aux_cols,
                               int64_t n_points, const void* params, void* grads, const void* ybar,
                               void* workspace, size_t workspace_bytes, void* stream);

/* DeepONet head — replaces, for one batch, deeponet.py:141-149 (G = sum_i branch_i * act(trunk_i) + b), the MSE of
 * ppsci/loss/mse.py:82-106 on G and their derivatives (no framework autograd graph):
 *   b, t      [n][n_features] row-major branch / trunk features;  bias: device scalar or NULL
 *   g_out     optional [n] outputs
 *   loss_acc  optional device double, ACCUMULATES  coef * sum_p w_p (G_p - label_p)^2   (coef = loss weight / n_norm for "mean")
 *   bbar/tbar optional [n][n_features] adjoints dL/db, dL/dt (may alias b / t);  dbias: device scalar, accumulated
 * With bbar == tbar == NULL only g_out is produced (eval / predict). */
int ppsci_b200_deeponet_head(int32_t dtype, int32_t act, const void* b, const void* t, const void* bias,
                             const void* label, const void* weight, int64_t n, int32_t n_features, double coef,
                             void* g_out, double* loss_acc, void* bbar, void* tbar, void* dbias, void* stream);

/* Device-side collocation sampling — replaces, for axis-aligned boxes, the per-step numpy RNG + host-to-device copy of
 * ContinuousNamedArrayDataset.__iter__ (ppsci/data/dataset/array_dataset.py:208-228).  out_cols[d][i] = lo[d] +
 * (hi[d] - lo[d]) * U(seed; offset + i, d), U in [0, 1) from Philox4x32-10 (counter-based: the same (seed, offset)
 * reproduce the same points on any launch geometry).  Not numpy's stream: bit-exact reference sampling stays on the host
 * (geometry/*.py). */
int ppsci_b200_sample_uniform(int32_t dtype, uint64_t seed, uint64_t offset, int64_t n, int32_t ndim, const double* lo,
                              const double* hi, void* const* out_cols, void* stream);

/* Bench instrumentation: when on, every launch of the next calls is bracketed by CUDA events on
 * the caller's stream (no syncs).  get_profile returns, for the most recent call, the summed
 * device time [ms] and launch count per kernel class:
 *   0 forward-jet GEMM, 1 residual head, 2 dW GEMM, 3 dx GEMM (+activation adjoint), 4 misc,
 *   5 thin first/last-layer forward, 6 thin last-layer backward, 7 thin first-layer dW + bias gradients.
 * Both arrays have PPSCI_PROFILE_CLASSES (8) entries. */
#define PPSCI_PROFILE_CLASSES 8
int ppsci_b200_plan_set_profile(ppsci_plan* plan, int32_t on);
int ppsci_b200_plan_get_profile(ppsci_plan* plan, double* ms, int64_t* count);

/* 1 if the wgmma tensor-core kernels serve some pass (forward, dx or dW) of this plan's layers, else 0. */
int32_t ppsci_b200_plan_uses_tcgen05(const ppsci_plan* plan);

/* Fused Adam on flat buffers — replaces paddle.optimizer.Adam.step for this path
 * (ppsci/optimizer/optimizer.py:225-248, ppsci/solver/train.py:175).
 * grad_scale multiplies grads first (1/world for DP averaging).
 * weight_decay > 0: L2 regularisation folded into the gradient (paddle.optimizer.Adam(weight_decay=...));
 * weight_decay < 0: DECOUPLED decay with coefficient -weight_decay — paddle.optimizer.AdamW
 * (ppsci/optimizer/optimizer.py:386-496): params <- params (1 - lr coeff) before the Adam update. */
int ppsci_b200_adam_step(int32_t dtype, void* params, const void* grads, void* exp_avg,
                         void* exp_avg_sq, int64_t n, double lr, double beta1, double beta2,
                         double eps, double weight_decay, int64_t step, double grad_scale,
                         void* stream);

/* The same Adam update with the per-step scalars in DEVICE memory: hyper_dev[4] = {lr, 1 - beta1^t, 1 - beta2^t,
 * grad_scale}.  No argument of the launch changes from step to step, so the call can be recorded into a CUDA graph
 * together with ppsci_b200_residual_loss_fwd_bwd and replayed (the counterpart of the reference's
 * to_static=True, ppsci/solver/solver.py:487, 907-937: one captured launch train instead of a traced program).
 * zero_grads != 0 also clears the gradient buffer it consumed (optimizer.clear_grad, ppsci/solver/train.py:178). */
int ppsci_b200_adam_step_dev(int32_t dtype, void* params, void* grads, void* exp_avg, void* exp_avg_sq,
                             int64_t n, const double* hyper_dev, double beta1, double beta2, double eps,
                             double weight_decay, int32_t zero_grads, void* stream);

const char* ppsci_b200_last_error(void);
const char* ppsci_b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* PPSCI_B200_H_ */

// engine.cu — C-ABI implementation (include/ppsci_b200.h): plan validation, workspace carving
// and the per-chunk launch schedule
//     forward jets (layer by layer)  ->  residual program + MSE  ->  adjoint (dW, dx per layer).
// All device memory except the (tiny) residual program is caller-owned workspace.
#ifdef PPSCI_EMUL
#include "cuda_emul.h"
#endif

#include <stdio.h>
#include <stdlib.h>

#include <string>
#include <vector>

#include "kernels_simt.cuh"
#include "kernels_thin.cuh"
#include "kernels_wgmma.cuh"
#include "kernels_gate.cuh"

using namespace ppsci;

static thread_local std::string g_err;

static int fail(const std::string& msg) {
  g_err = msg;
  return 1;
}

// f(T()) for the element type T of dtype (PPSCI_F32 / PPSCI_F64); any other dtype fails as "<what>: bad dtype"
template <class F>
static int with_dtype(int dtype, const char* what, F f) {
  if (dtype == PPSCI_F64) return f(double());
  if (dtype == PPSCI_F32) return f(float());
  return fail(std::string(what) + ": bad dtype");
}

#define CK(call)                                                                              \
  do {                                                                                        \
    cudaError_t e_ = (call);                                                                  \
    if (e_ != cudaSuccess)                                                                    \
      return fail(std::string(#call) + " failed: " + cudaGetErrorString(e_) + " (" __FILE__ ":" + \
                  std::to_string(__LINE__) + ")");                                            \
  } while (0)

struct ppsci_plan {
  ppsci_plan_spec spec;
  std::vector<int32_t> prog, grad_res, grad_in, grad_reg;
  std::vector<double> consts;
  int C = 1;
  int kmax = 1;
  JetLayout J;
  int64_t w_off[PPSCI_MAX_LAYERS + 1];
  int64_t b_off[PPSCI_MAX_LAYERS + 1];
  int ld[PPSCI_MAX_LAYERS + 1];
  int64_t n_params = 0;
  int64_t gate_w_off[2] = {0, 0};  // gated plans: embed_u / embed_v weights and biases behind the layers
  int64_t gate_b_off[2] = {0, 0};
  int64_t alpha_off = 0;  // gated == 2: one residual weight per block behind the embeddings
  // trainable activation parameters (PPSCI_ACT_STAN: one beta per unit; PPSCI_ACT_SWISH_B: one per layer) of hidden
  // layer l, behind everything else; actp_stride 1 / 0, actp_off[l] < 0: layer l's activation has none
  int64_t actp_off[PPSCI_MAX_LAYERS + 1];
  int actp_stride = 0;
  int64_t omega_off = 0;  // spec.n_omega trainable frequencies, the last entries of the buffers
  int ld_hidden_max = 4;
  int chunk = 0;
  int num_sms = 132;
  bool use_wg = false;  // forward, dx and dW run on the wgmma kernels where the layer shapes allow (kernels_wgmma.cuh)
  // PPSCI_B200_TC_MASK (cross-checks): bit 0 forward, bit 1 dx, bit 2 dW of the eligible layers on the tensor cores;
  // the other bits are ignored
  int tc_mask = 7;
  // layer l's forward / dx / dW runs on the wgmma kernels; its forward (transposed) tf32 hi / lo weight image sits at
  // img_off[l] (imgT_off[l]) of the wimg workspace region, img_bytes long in all
  bool wg_fwd[PPSCI_MAX_LAYERS + 1] = {};
  bool wg_dx[PPSCI_MAX_LAYERS + 1] = {};
  bool wg_dw[PPSCI_MAX_LAYERS + 1] = {};
  size_t img_off[PPSCI_MAX_LAYERS + 1] = {};
  size_t imgT_off[PPSCI_MAX_LAYERS + 1] = {};
  size_t img_bytes = 0;
  // first / last layer on the thin kernels (kernels_thin.cuh); thin_vec: the vectorised ones (a jet layout of ThinLays)
  bool thin_first = false;
  bool thin_last = false;
  bool thin_vec = false;
  // PPSCI_B200_KEEP_ADJOINTS (tests): every hidden layer's Zbar gets a plane set of its own instead of the two ping-pong
  // sets, so that all of them survive a call; kernels and launches are the same
  bool keep_adj = false;
  // device copies of the residual program
  int* d_prog = nullptr;
  double* d_consts = nullptr;
  int* d_grad_res = nullptr;
  int* d_grad_in = nullptr;
  int* d_grad_reg = nullptr;
  double* aux_grad[PPSCI_MAX_IN] = {};  // ppsci_b200_plan_set_aux_grad
  int64_t launches = 0;
  bool attrs_set = false;
  // optional per-kernel-class timing (bench only; adds event records, no syncs)
  bool profile = false;
  std::vector<cudaEvent_t> ev_pool;
  size_t ev_used = 0;
  std::vector<int> ev_cls;  // class of event pair i (events 2i, 2i+1)
};

enum { CLS_FWD = 0, CLS_HEAD = 1, CLS_DW = 2, CLS_DX = 3, CLS_MISC = 4, CLS_THIN_FWD = 5, CLS_THIN_DX = 6, CLS_THIN_DW = 7, CLS_COUNT = 8 };

struct ProfScope {
  ppsci_plan* P;
  cudaStream_t st;
  bool on;
  ProfScope(ppsci_plan* P_, int cls, cudaStream_t st_) : P(P_), st(st_), on(P_->profile) {
    if (!on) return;
    if (P->ev_used + 2 > P->ev_pool.size()) {
      for (int i = 0; i < 64; ++i) {
        cudaEvent_t e;
        if (cudaEventCreate(&e) != cudaSuccess) { on = false; return; }
        P->ev_pool.push_back(e);
      }
    }
    P->ev_cls.push_back(cls);
    cudaEventRecord(P->ev_pool[P->ev_used], st);
  }
  ~ProfScope() {
    if (!on) return;
    cudaEventRecord(P->ev_pool[P->ev_used + 1], st);
    P->ev_used += 2;
  }
};

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static inline int round4(int x) { return (x + 3) / 4 * 4; }

struct Carve {
  size_t z[PPSCI_MAX_LAYERS + 1];  // z[l] for l = 1..n_layers-1 (hidden pre-activations)
  size_t y, ybar, zbar0, zbar1;
  size_t wt[PPSCI_MAX_LAYERS + 1];
  size_t loss_acc;
  size_t wimg;  // tf32 hi / lo weight images of the layers whose forward / dx run on the wgmma kernels
  // gated plans (ModifiedMLP): gated jets G_l per hidden layer, pre-activations of embed_u / embed_v and their adjoints
  size_t gt[PPSCI_MAX_LAYERS + 1];
  size_t zu, zv, zub, zvb;
  size_t xres, wtu, wtv;  // gated == 2: adjoint carried by the blocks' residual path; transposed embedding weights
  size_t omega_acc;       // fp64 dLoss/d omega accumulators of a call (n_omega)
  size_t zbl[PPSCI_MAX_LAYERS + 1];  // keep_adj: Zbar_l of hidden layer l (empty otherwise)
  size_t total;
};

// gated plans: 1 when layer 1 is an embedding layer whose stored output feeds the embed_u / embed_v layers and the
// first gated layer (PirateNet always; ModifiedMLP with a Fourier embedding, act_first >= 0), 0 when they read the seeds
static inline int gate_emb(const ppsci_plan_spec& s) { return (s.gated == 2 || (s.gated == 1 && s.act_first >= 0)) ? 1 : 0; }

// activation applied to the output of linear layer `lin` (1-based)
static inline int act_of_layer(const ppsci_plan_spec& s, int lin) { return (lin == 1 && s.act_first >= 0) ? s.act_first : s.act; }

static void carve(const ppsci_plan* P, int64_t nc, Carve* cv) {
  const size_t es = P->spec.dtype == PPSCI_F64 ? 8 : 4;
  const int L = P->spec.n_layers;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off = align_up(off + bytes, 256);
    return o;
  };
  for (int l = 1; l < L; ++l) cv->z[l] = take((size_t)P->C * nc * P->ld[l] * es);
  cv->y = take((size_t)P->C * nc * P->ld[L] * es);
  cv->ybar = take((size_t)P->C * nc * P->ld[L] * es);
  cv->zbar0 = take((size_t)P->C * nc * P->ld_hidden_max * es);
  cv->zbar1 = take((size_t)P->C * nc * P->ld_hidden_max * es);
  for (int l = 2; l <= L; ++l) cv->wt[l] = take((size_t)P->spec.widths[l] * P->spec.widths[l - 1] * es);
  cv->loss_acc = take(PPSCI_MAX_RES * sizeof(double));
  cv->wimg = take(P->img_bytes);
  const bool gated = P->spec.gated != 0;
  for (int l = 1; l < L; ++l) cv->gt[l] = take(gated ? (size_t)P->C * nc * P->ld[l] * es : 0);
  const int emb = gate_emb(P->spec);
  const int lg = (gated && emb + 1 <= L) ? emb + 1 : 1;  // first gated layer
  cv->zu = take(gated ? (size_t)P->C * nc * P->ld[lg] * es : 0);
  cv->zv = take(gated ? (size_t)P->C * nc * P->ld[lg] * es : 0);
  cv->zub = take(gated ? (size_t)P->C * nc * P->ld[lg] * es : 0);
  cv->zvb = take(gated ? (size_t)P->C * nc * P->ld[lg] * es : 0);
  const bool pirate = P->spec.gated == 2;
  cv->xres = take(pirate ? (size_t)P->C * nc * P->ld[1] * es : 0);
  cv->wtu = take(gated && emb ? (size_t)P->spec.widths[1] * P->spec.widths[lg] * es : 0);
  cv->wtv = take(gated && emb ? (size_t)P->spec.widths[1] * P->spec.widths[lg] * es : 0);
  cv->omega_acc = take((size_t)P->spec.n_omega * sizeof(double));
  for (int l = 1; l < L; ++l) cv->zbl[l] = take(P->keep_adj ? (size_t)P->C * nc * P->ld[l] * es : 0);
  cv->total = off;
}

extern "C" const char* ppsci_b200_last_error(void) { return g_err.c_str(); }
extern "C" const char* ppsci_b200_version(void) {
#ifdef PPSCI_EMUL
  return "ppsci_b200 0.1 (CPU emulation build: TEST ONLY)";
#else
  return "ppsci_b200 0.1 (sm_90a)";
#endif
}

static int op_arity(int op) {
  switch (op) {
    case PPSCI_OP_CONST: return 0;
    case PPSCI_OP_MOV: case PPSCI_OP_NEG: case PPSCI_OP_POWI: case PPSCI_OP_SIN: case PPSCI_OP_COS:
    case PPSCI_OP_TANH: case PPSCI_OP_EXP: case PPSCI_OP_LOG: case PPSCI_OP_SQRT: case PPSCI_OP_ABS:
    case PPSCI_OP_SIGN: case PPSCI_OP_SINH: case PPSCI_OP_COSH: case PPSCI_OP_HEAVISIDE:
      return 1;
    case PPSCI_OP_ADD: case PPSCI_OP_SUB: case PPSCI_OP_MUL: case PPSCI_OP_DIV: case PPSCI_OP_POW:
    case PPSCI_OP_MAX: case PPSCI_OP_MIN: case PPSCI_OP_FMA: case PPSCI_OP_EQ: case PPSCI_OP_SELECT:
      return 2;
    default: return -1;
  }
}

// registers, instructions, residual registers and the partials list of a residual program whose first n_inreg
// registers are loaded before it runs, n_grad_in of them output-jet registers (plan_create, deeponet_jet_head_create)
static int check_program(const std::string& what, int n_inreg, int n_grad_in, int n_reg, int n_ops, const int32_t* prog,
                         int n_consts, int n_res, const int32_t* res_reg, int n_grad, const int32_t* grad_res,
                         const int32_t* grad_in, const int32_t* grad_reg) {
  if (n_reg < n_inreg || n_reg > PPSCI_MAX_REG) return fail(what + ": n_reg out of range (max 256)");
  if (n_ops < 0 || (n_ops > 0 && !prog)) return fail(what + ": bad program");
  for (int i = 0; i < n_ops; ++i) {
    const int op = prog[4 * i], dst = prog[4 * i + 1], a = prog[4 * i + 2], b = prog[4 * i + 3];
    const int ar = op_arity(op);
    if (ar < 0) return fail(what + ": unknown opcode at op " + std::to_string(i));
    if (dst < 0 || dst >= n_reg) return fail(what + ": dst register out of range at op " + std::to_string(i));
    if (op == PPSCI_OP_CONST) {
      if (a < 0 || a >= n_consts) return fail(what + ": const index out of range at op " + std::to_string(i));
    } else {
      if (a < 0 || a >= n_reg) return fail(what + ": src register out of range at op " + std::to_string(i));
      if (ar == 2 && (b < 0 || b >= n_reg)) return fail(what + ": src register out of range at op " + std::to_string(i));
    }
  }
  for (int k = 0; k < n_res; ++k)
    if (res_reg[k] < 0 || res_reg[k] >= n_reg) return fail(what + ": res_reg out of range");
  if (n_grad < 0) return fail(what + ": n_grad < 0");
  if (n_grad > 0 && (!grad_res || !grad_in || !grad_reg)) return fail(what + ": null grad list");
  for (int g = 0; g < n_grad; ++g) {
    if (grad_res[g] < 0 || grad_res[g] >= n_res) return fail(what + ": grad_res out of range");
    if (grad_in[g] < 0 || grad_in[g] >= n_grad_in) return fail(what + ": grad_in out of range");
    if (grad_reg[g] < 0 || grad_reg[g] >= n_reg) return fail(what + ": grad_reg out of range");
    if (g > 0 && grad_in[g] < grad_in[g - 1]) return fail(what + ": grad list must be sorted by grad_in");
  }
  return 0;
}

extern "C" int ppsci_b200_plan_create(const ppsci_plan_spec* s, ppsci_plan** out) {
  if (!s || !out) return fail("plan_create: null argument");
  *out = nullptr;
  if (s->dtype != PPSCI_F32 && s->dtype != PPSCI_F64) return fail("plan_create: dtype must be f32 or f64");
  if (s->n_in < 1 || s->n_in > PPSCI_MAX_IN) return fail("plan_create: n_in out of range");
  if (s->dense_in) {  // dense [n_points][n_feat] first-layer operand (header: dense_in)
    if (s->n_in != 1) return fail("plan_create: dense_in needs n_in == 1 (one row-major matrix)");
    if (s->n_dir != 0) return fail("plan_create: dense_in has no input derivatives (n_dir must be 0)");
    if (s->n_feat < 1 || s->n_feat > 4096) return fail("plan_create: n_feat out of range");
  } else if (s->n_feat < 1 || s->n_feat > PPSCI_MAX_FEAT) {
    return fail("plan_create: n_feat out of range");
  }
  if (s->backend < 0 || s->backend > 2) return fail("plan_create: backend must be 0 (auto), 1 (SIMT) or 2 (tensor cores)");
  if (s->n_layers < 1 || s->n_layers > PPSCI_MAX_LAYERS) return fail("plan_create: n_layers out of range");
  if (s->widths[0] != s->n_feat) return fail("plan_create: widths[0] must equal n_feat");
  for (int l = 0; l <= s->n_layers; ++l)
    if (s->widths[l] < 1 || s->widths[l] > 4096) return fail("plan_create: layer width out of range");
  if (s->act < 0 || s->act > PPSCI_ACT_LAST) return fail("plan_create: unknown activation");
  if (s->act_first < -1 || s->act_first > PPSCI_ACT_LAST) return fail("plan_create: unknown first-layer activation");
  for (int f = 0; f < (s->dense_in ? 0 : s->n_feat); ++f) {
    if (s->feat_src[f] < 0 || s->feat_src[f] >= s->n_in) return fail("plan_create: feat_src out of range");
    if (s->feat_kind[f] < 0 || s->feat_kind[f] > PPSCI_FEAT_SIN) return fail("plan_create: bad feat_kind");
  }
  if (s->n_dir < 0 || s->n_dir > PPSCI_MAX_DIR) return fail("plan_create: n_dir out of range");
  if (s->act_first == PPSCI_ACT_STAN || s->act_first == PPSCI_ACT_SWISH_B)
    return fail("plan_create: act_first cannot be an activation with a trainable parameter");
  if ((s->act == PPSCI_ACT_STAN || s->act == PPSCI_ACT_SWISH_B) && s->gated)
    return fail("plan_create: activations with a trainable parameter (stan, swish) run on plain MLP plans, CUDA-core kernels");
  if (s->gated) {  // ModifiedMLP: the gate multiplies every hidden layer's output with the (same-width) embeddings
    if (s->n_layers < 2) return fail("plan_create: a gated network needs at least one hidden layer");
    if (s->gated != 1 && s->gated != 2) return fail("plan_create: gated must be 0, 1 (ModifiedMLP) or 2 (PirateNet)");
    if (s->dense_in) return fail("plan_create: gated networks do not take dense_in");
    if (s->gated == 2 && (s->n_layers < 5 || (s->n_layers - 2) % 3 != 0))
      return fail("plan_create: gated kind 2 needs 1 embedding layer + 3 layers per block + the output layer");
    const int emb = gate_emb(*s);
    if (s->n_layers < emb + 2) return fail("plan_create: a gated network needs a hidden layer behind its embedding layer");
    for (int l = emb + 2; l < s->n_layers; ++l)
      if (s->widths[l] != s->widths[emb + 1]) return fail("plan_create: a gated network needs equal hidden widths");
    if (s->gated == 2 && s->widths[1] != s->widths[2])
      return fail("plan_create: gated kind 2 adds a block's input to its output: the embedding layer needs the blocks' width");
  }
  int C = 1, kmax = 1;
  for (int d = 0; d < s->n_dir; ++d) {
    if (s->dir_order[d] < 1 || s->dir_order[d] > PPSCI_MAX_ORDER) return fail("plan_create: dir_order out of range");
    C += s->dir_order[d];
    if (s->dir_order[d] > kmax) kmax = s->dir_order[d];
  }
  if (C > RC) return fail("plan_create: too many jet channels (max 32)");
  const int n_out = s->widths[s->n_layers];
  if (s->n_aux < 0 || s->n_aux > PPSCI_MAX_IN) return fail("plan_create: n_aux out of range");
  // a plan without residual program (a sub-network whose outputs a caller's head reads) has no register file
  const int n_inreg = C * n_out + s->n_in + s->n_aux;
  if (s->n_res < 0 || s->n_res > PPSCI_MAX_RES) return fail("plan_create: n_res out of range");
  if ((s->n_ops != 0 || s->n_res != 0 || s->n_grad != 0) &&
      check_program("plan_create", n_inreg, C * n_out, s->n_reg, s->n_ops, s->prog, s->n_consts, s->n_res, s->res_reg,
                    s->n_grad, s->grad_res, s->grad_in, s->grad_reg))
    return 1;
  for (int k = 0; k < s->n_res; ++k)
    if (s->reduction[k] != PPSCI_REDUCE_MEAN && s->reduction[k] != PPSCI_REDUCE_SUM) return fail("plan_create: bad reduction");
  if (s->n_pgrad < 0 || s->n_pgrad > PPSCI_MAX_PGRAD) return fail("plan_create: n_pgrad out of range");
  for (int g = 0; g < s->n_pgrad; ++g) {
    if (s->pgrad_res[g] < 0 || s->pgrad_res[g] >= s->n_res) return fail("plan_create: pgrad_res out of range");
    if (s->pgrad_aux[g] < 0 || s->pgrad_aux[g] >= s->n_aux || !s->aux_bcast[s->pgrad_aux[g]])
      return fail("plan_create: pgrad_aux must name a learnable (aux_bcast) parameter");
    if (s->pgrad_reg[g] < 0 || s->pgrad_reg[g] >= s->n_reg) return fail("plan_create: pgrad_reg out of range");
  }
  if (s->n_omega < 0 || s->n_omega > PPSCI_MAX_FEAT) return fail("plan_create: n_omega out of range");
  if (s->n_omega > 0 && s->dense_in) return fail("plan_create: dense_in plans take no trainable frequencies");
  for (int f = 0; f < (s->n_omega > 0 ? s->n_feat : 0); ++f) {
    const int j = s->feat_omega_param[f];
    if (j < -1 || j >= s->n_omega) return fail("plan_create: feat_omega_param out of range");
    if (j >= 0 && s->feat_kind[f] == PPSCI_FEAT_ID) return fail("plan_create: only cos / sin features take a trainable frequency");
  }

  ppsci_plan* P = new ppsci_plan();
  P->spec = *s;
  P->prog.assign(s->prog, s->prog + 4 * (size_t)s->n_ops);
  P->consts.assign(s->consts, s->consts + (size_t)s->n_consts);
  P->grad_res.assign(s->grad_res, s->grad_res + (size_t)s->n_grad);
  P->grad_in.assign(s->grad_in, s->grad_in + (size_t)s->n_grad);
  P->grad_reg.assign(s->grad_reg, s->grad_reg + (size_t)s->n_grad);
  P->spec.prog = nullptr; P->spec.consts = nullptr;
  P->spec.grad_res = P->spec.grad_in = P->spec.grad_reg = nullptr;
  P->C = C;
  P->kmax = kmax;
  P->J.C = C;
  P->J.n_dir = s->n_dir;
  int base = 1;
  for (int d = 0; d < PPSCI_MAX_DIR; ++d) {
    P->J.dir_order[d] = d < s->n_dir ? s->dir_order[d] : 0;
    P->J.dir_base[d] = base;
    if (d < s->n_dir) base += s->dir_order[d];
  }
  int64_t off = 0;
  P->ld[0] = round4(s->widths[0]);
  for (int l = 1; l <= s->n_layers; ++l) {
    P->w_off[l] = off;
    off += (int64_t)s->widths[l - 1] * s->widths[l];
    P->b_off[l] = off;
    off += s->widths[l];
    P->ld[l] = round4(s->widths[l]);
    if (l < s->n_layers && P->ld[l] > P->ld_hidden_max) P->ld_hidden_max = P->ld[l];
  }
  if (s->gated) {
    for (int e = 0; e < 2; ++e) {
      P->gate_w_off[e] = off;
      const int emb = gate_emb(*s);  // 1: the embeddings read layer 1's output
      off += (int64_t)s->widths[emb] * s->widths[emb + 1];
      P->gate_b_off[e] = off;
      off += s->widths[emb + 1];
    }
    if (s->gated == 2) {
      P->alpha_off = off;
      off += (s->n_layers - 2) / 3;
    }
  }
  P->actp_stride = s->act == PPSCI_ACT_STAN ? 1 : 0;
  for (int l = 0; l <= PPSCI_MAX_LAYERS; ++l) P->actp_off[l] = -1;
  for (int l = 1; l < s->n_layers; ++l) {
    const int a_l = (l == 1 && s->act_first >= 0) ? s->act_first : s->act;
    if (a_l != PPSCI_ACT_STAN && a_l != PPSCI_ACT_SWISH_B) continue;
    P->actp_off[l] = off;
    off += a_l == PPSCI_ACT_STAN ? s->widths[l] : 1;
  }
  P->omega_off = off;
  off += s->n_omega;
  P->n_params = off;
  // default points per workspace chunk: large chunks amortise kernel prologues / tails and give the dW kernels long
  // reductions per split (measured on cfg3: 65,536 -> 77.7 ms/step, 262,144 -> 73.7 ms/step); capped below by memory
  P->chunk = s->chunk_points > 0 ? s->chunk_points : (s->dtype == PPSCI_F64 ? 32768 : 262144);
  if (s->chunk_points <= 0) {
    if (const char* m = getenv("PPSCI_B200_CHUNK_POINTS")) {  // tuning knob: points per workspace chunk
      const long long v = atoll(m);
      if (v >= 1024 && v <= (1 << 22)) P->chunk = (int)v;
    }
  }
  {  // the tensor-core dW kernels address a chunk's plane set with 32-bit element offsets
    long long ld_max = 4;
    for (int l = 0; l <= s->n_layers; ++l) ld_max = std::max<long long>(ld_max, (s->widths[l] + 3) / 4 * 4);
    while ((long long)C * P->chunk * ld_max >= (1LL << 32) && P->chunk > 1024) P->chunk /= 2;
  }

  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) == cudaSuccess && cudaGetDeviceProperties(&prop, dev) == cudaSuccess) {
    P->num_sms = prop.multiProcessorCount;
#ifndef PPSCI_EMUL
    if (prop.major != 9) {
      delete P;
      return fail("plan_create: this library is built for sm_90a (H100) only; found compute capability " +
                  std::to_string(prop.major) + "." + std::to_string(prop.minor));
    }
#endif
  } else {
    delete P;
    return fail("plan_create: no CUDA device available (the engine has no CPU fallback)");
  }
#ifndef PPSCI_EMUL
  if (const char* m = getenv("PPSCI_B200_TC_MASK")) P->tc_mask = atoi(m);
  const bool wg_plan = s->backend != 1 && wg_plan_ok(*s, P->J);
  for (int l = 2; l <= s->n_layers && wg_plan; ++l)
    if (((P->tc_mask & 1) && wg_fwd_ok(*s, l)) || ((P->tc_mask & 2) && wg_dx_ok(*s, l)) || ((P->tc_mask & 4) && wg_dw_ok(*s, l)))
      P->use_wg = true;
  for (int l = 1; l <= s->n_layers && P->use_wg; ++l) {  // use_wg also gates a dense first layer
    P->wg_fwd[l] = (P->tc_mask & 1) && wg_fwd_ok(*s, l);
    P->wg_dx[l] = (P->tc_mask & 2) && wg_dx_ok(*s, l);
    P->wg_dw[l] = (P->tc_mask & 4) && wg_dw_ok(*s, l);
  }
#endif
  for (int l = 1; l <= s->n_layers; ++l) {  // the forward images first; layer 1: contraction padded to the chunk width
    P->img_off[l] = P->img_bytes;
    if (P->wg_fwd[l]) P->img_bytes += (size_t)(l == 1 ? (s->widths[0] + 31) / 32 * 32 : s->widths[l - 1]) * s->widths[l] * 8;
  }
  for (int l = 1; l <= s->n_layers; ++l) {
    P->imgT_off[l] = P->img_bytes;
    if (P->wg_dx[l]) P->img_bytes += (size_t)s->widths[l - 1] * s->widths[l] * 8;
  }
  const bool thin_on = getenv("PPSCI_B200_NO_THIN") == nullptr;
  P->thin_first = thin_on && s->n_layers >= 2 && s->widths[0] <= THIN_MAXF && !s->dense_in && !s->gated;
  P->thin_last = thin_on && s->n_layers >= 2 && n_out <= THIN_MAXM && C * n_out <= THIN_MAXCM && !s->gated && !act_has_param(s->act);
  P->thin_vec = s->dtype == PPSCI_F32 && with_lay(ThinLays{}, P->J, [](auto) {}) && getenv("PPSCI_B200_NO_THINV") == nullptr;
  P->keep_adj = getenv("PPSCI_B200_KEEP_ADJOINTS") != nullptr;
  if (s->backend == 2 && !P->use_wg) {
    delete P;
    return fail("plan_create: backend=2 (tensor cores) requested but the plan is not eligible (needs f32, hidden widths that "
                "are multiples of 32 up to 256, and one of the compile-time jet layouts)");
  }

  auto up = [&](const void* src, size_t bytes, void** dst) -> cudaError_t {
    cudaError_t e = cudaMalloc(dst, bytes ? bytes : 16);
    if (e != cudaSuccess) return e;
    if (bytes) return cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice);
    return cudaSuccess;
  };
  cudaError_t e = cudaSuccess;
  if (e == cudaSuccess) e = up(P->prog.data(), P->prog.size() * 4, (void**)&P->d_prog);
  if (e == cudaSuccess) e = up(P->consts.data(), P->consts.size() * 8, (void**)&P->d_consts);
  if (e == cudaSuccess) e = up(P->grad_res.data(), P->grad_res.size() * 4, (void**)&P->d_grad_res);
  if (e == cudaSuccess) e = up(P->grad_in.data(), P->grad_in.size() * 4, (void**)&P->d_grad_in);
  if (e == cudaSuccess) e = up(P->grad_reg.data(), P->grad_reg.size() * 4, (void**)&P->d_grad_reg);
  if (e != cudaSuccess) {
    ppsci_b200_plan_destroy(P);
    return fail(std::string("plan_create: device upload of the residual program failed: ") + cudaGetErrorString(e));
  }
  if (s->chunk_points <= 0 && getenv("PPSCI_B200_CHUNK_POINTS") == nullptr) {
    // default chunk: keep one call's workspace under ~20 GB of the 80 GB of HBM
    for (;;) {
      Carve cv;
      carve(P, P->chunk, &cv);
      if (cv.total <= (size_t)20 << 30 || P->chunk <= 16384) break;
      P->chunk /= 2;
    }
  }
  *out = P;
  return 0;
}

extern "C" void ppsci_b200_plan_destroy(ppsci_plan* P) {
  if (!P) return;
  cudaFree(P->d_prog);
  cudaFree(P->d_consts);
  cudaFree(P->d_grad_res);
  cudaFree(P->d_grad_in);
  cudaFree(P->d_grad_reg);
  for (cudaEvent_t e : P->ev_pool) cudaEventDestroy(e);
  delete P;
}

extern "C" int64_t ppsci_b200_plan_param_count(const ppsci_plan* P) { return P ? P->n_params : -1; }
extern "C" int32_t ppsci_b200_plan_channels(const ppsci_plan* P) { return P ? P->C : -1; }
extern "C" int64_t ppsci_b200_plan_last_launches(const ppsci_plan* P) { return P ? P->launches : -1; }
extern "C" int ppsci_b200_plan_set_profile(ppsci_plan* P, int32_t on) {
  if (!P) return fail("null plan");
  P->profile = on != 0;
  return 0;
}
// ms[c] / count[c] for c in {fwd GEMM, head, dW GEMM, dx GEMM, misc} of the most recent call.
extern "C" int ppsci_b200_plan_get_profile(ppsci_plan* P, double* ms, int64_t* count) {
  if (!P || !ms || !count) return fail("null argument");
  for (int c = 0; c < CLS_COUNT; ++c) { ms[c] = 0.0; count[c] = 0; }
#ifndef PPSCI_EMUL
  for (size_t i = 0; i < P->ev_cls.size(); ++i) {
    float t = 0.f;
    CK(cudaEventSynchronize(P->ev_pool[2 * i + 1]));
    CK(cudaEventElapsedTime(&t, P->ev_pool[2 * i], P->ev_pool[2 * i + 1]));
    ms[P->ev_cls[i]] += t;
    count[P->ev_cls[i]] += 1;
  }
#endif
  return 0;
}
extern "C" int32_t ppsci_b200_plan_uses_tcgen05(const ppsci_plan* P) { return (P && P->use_wg) ? 1 : 0; }

// Debug / test accessor: byte offset (from the 256-aligned workspace base) of the jet planes of
// `layer` for a call with n_points points: layer in [1, n_layers) -> hidden pre-activations Z_l,
// layer == n_layers -> output jets Y.  Layout [C][min(n_points, chunk)][ld], ld = round4(width).
// 301 / 302 -> the Zbar ping-pong buffers zbar0 / zbar1 (the adjoint writes Zbar_l into buffer (L-1-l) mod 2).
// Gated plans: 400 + l -> G_l, the stored output of the gate or mix after hidden layer l; 310 / 311 -> Zu / Zv,
// 312 / 313 -> their adjoints Zubar / Zvbar (width of the first gated layer); 314 -> Xres (PirateNet, layer 1's width).
// 500 + l -> Zbar_l of hidden layer l when the plan was created with PPSCI_B200_KEEP_ADJOINTS set.
// -1 for a code whose buffer the plan does not carve.
extern "C" int64_t ppsci_b200_plan_stash_offset(const ppsci_plan* P, int64_t n_points, int32_t layer) {
  if (!P || n_points <= 0) return -1;
  const int64_t nc = n_points < P->chunk ? n_points : P->chunk;
  Carve cv;
  carve(P, nc, &cv);
  const int L = P->spec.n_layers;
  const bool gated = P->spec.gated != 0;
  if (layer == 300) return (int64_t)cv.ybar;  // output adjoints Ybar (values_bwd_kept accepts this address: no seeding copy)
  if (layer == 301) return (int64_t)cv.zbar0;
  if (layer == 302) return (int64_t)cv.zbar1;
  if (layer >= 310 && layer <= 313) return gated ? (int64_t)(layer == 310 ? cv.zu : layer == 311 ? cv.zv : layer == 312 ? cv.zub : cv.zvb) : -1;
  if (layer == 314) return P->spec.gated == 2 ? (int64_t)cv.xres : -1;
  if (layer > 400 && layer < 400 + L) return gated ? (int64_t)cv.gt[layer - 400] : -1;
  if (layer > 500 && layer < 500 + L) return P->keep_adj ? (int64_t)cv.zbl[layer - 500] : -1;
  if (layer < 1 || layer > L) return -1;
  return (int64_t)(layer < L ? cv.z[layer] : cv.y);
}

extern "C" size_t ppsci_b200_plan_workspace_bytes(const ppsci_plan* P, int64_t n_points) {
  if (!P || n_points <= 0) return 0;
  const int64_t nc = n_points < P->chunk ? n_points : P->chunk;
  Carve cv;
  carve(P, nc, &cv);
  return cv.total;
}

// ---------------------------------------------------------------------------------------------
template <typename T>
static void fill_seed(const ppsci_plan* P, const void* const* x_cols, int64_t x_off, const T* params, AOperand<T>* A) {
  const ppsci_plan_spec& s = P->spec;
  A->mode = A_SEED;
  A->act = s.act;
  A->Z = nullptr;
  A->ld = 0;
  A->plane = 0;
  A->x_off = x_off;
  SeedSpec& S = A->seed;
  S.n_in = s.n_in;
  S.n_feat = s.n_feat;
  for (int f = 0; f < PPSCI_MAX_FEAT; ++f) {
    S.feat_src[f] = f < s.n_feat ? s.feat_src[f] : 0;
    S.feat_kind[f] = f < s.n_feat ? s.feat_kind[f] : 0;
    S.feat_omega[f] = f < s.n_feat ? s.feat_omega[f] : 0.0;
    S.omega_idx[f] = (s.n_omega > 0 && f < s.n_feat) ? s.feat_omega_param[f] : -1;
  }
  S.omega = params + P->omega_off;
  for (int d = 0; d < PPSCI_MAX_DIR; ++d)
    for (int i = 0; i < PPSCI_MAX_IN; ++i) S.dir_vec[d][i] = (d < s.n_dir && i < s.n_in) ? s.dir_vec[d][i] : 0.0;
  for (int i = 0; i < PPSCI_MAX_IN; ++i) S.x_cols[i] = i < s.n_in ? x_cols[i] : nullptr;
}

template <typename T>
static void fill_act(const ppsci_plan* P, const T* Z, int ld, int64_t nc, int mode, AOperand<T>* A, int lin = 0) {
  A->mode = mode;
  A->act = act_of_layer(P->spec, lin);
  A->Z = Z;
  A->ld = ld;
  A->plane = (long long)nc * ld;
  A->x_off = 0;
  memset(&A->seed, 0, sizeof(SeedSpec));
}

// first-layer operand: input seeds, or (dense_in) the caller's row-major [n_points][n_feat] matrix as a plain operand
template <typename T>
static void fill_first(const ppsci_plan* P, const void* const* x_cols, int64_t x_off, int64_t nc, const T* params, AOperand<T>* A) {
  if (P->spec.dense_in) {
    const int nf = P->spec.n_feat;
    fill_act<T>(P, reinterpret_cast<const T*>(x_cols[0]) + x_off * nf, nf, nc, A_PLAIN, A);
  } else {
    fill_seed<T>(P, x_cols, x_off, params, A);
  }
}

struct CallArgs {
  const void* const* x_cols;
  const void* const* aux_cols;
  const void* const* label_cols;
  const double* label_const;
  const void* const* weight_cols;
  int64_t n_points;
  int64_t n_norm;
  const void* params;
  void* grads;
  void* loss_out;
  void* const* residual_out;
  void* jets_out;
  void* workspace;
  size_t workspace_bytes;
  void* stream;
  bool want_loss;
  const void* ybar_in = nullptr;  // values_fwd_bwd: caller-supplied dL/dy [n_points][n_out]
  int phase = 0;                  // 0: forward + adjoint; 1: forward only, stash kept for a later adjoint; 2: adjoint from the kept stash
};

// split of a dW GEMM along the points: `want` splits, clamped to [1, total_chunks], of chunks_per_split chunks each
struct DwSplit {
  int chunks_per_split;
  unsigned splits;
};
static DwSplit dw_split(long long want, long long total_chunks) {
  want = std::min(std::max(want, 1LL), total_chunks);
  const long long cps = (total_chunks + want - 1) / want;
  return {(int)cps, (unsigned)((total_chunks + cps - 1) / cps)};
}

template <typename T, int KMAX>
static int run(ppsci_plan* P, const CallArgs& a) {
  constexpr int TN = sizeof(T) == 8 ? 64 : 128;
  const ppsci_plan_spec& s = P->spec;
  const int L = s.n_layers;
  const int C = P->C;
  const int n_out = s.widths[L];
  auto kf = k_gemm_fwd<T, TN, KMAX>;
  auto kx = k_gemm_dx<T, TN, KMAX>;
  auto kw = k_gemm_dw<T, TN, KMAX>;
  const int smem_f = (KC * TMS + KC * TN) * (int)sizeof(T);
  const int smem_x = std::max(smem_f, TM * TN * (int)sizeof(T));
  const int smem_w = (RC * TMS + RC * TN) * (int)sizeof(T);
  if (!P->attrs_set) {
    CK(cudaFuncSetAttribute(kf, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_f));
    CK(cudaFuncSetAttribute(kx, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_x));
    CK(cudaFuncSetAttribute(kw, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_w));
    P->attrs_set = true;
  }
  const int64_t nc_max = a.n_points < P->chunk ? a.n_points : P->chunk;
  Carve cv;
  carve(P, nc_max, &cv);
  if (cv.total > a.workspace_bytes)
    return fail("workspace too small: need " + std::to_string(cv.total) + " bytes, got " + std::to_string(a.workspace_bytes));
  if ((reinterpret_cast<uintptr_t>(a.workspace) & 255) != 0) return fail("workspace must be 256-byte aligned");
  unsigned char* ws = reinterpret_cast<unsigned char*>(a.workspace);
  cudaStream_t st = (cudaStream_t)a.stream;
  const T* params = reinterpret_cast<const T*>(a.params);
  T* grads = reinterpret_cast<T*>(a.grads);
  double* loss_acc = reinterpret_cast<double*>(ws + cv.loss_acc);
  P->launches = 0;
  P->ev_used = 0;
  P->ev_cls.clear();

  // every launch of a call: timed in class cls when profiling, counted by plan_last_launches
  auto launch = [&](int cls, auto kernel, dim3 grid, dim3 block, int smem, auto... args) {
    ProfScope ps_(P, cls, st);
    PPSCI_LAUNCH(kernel, grid, block, smem, st, args...);
    P->launches++;
  };
  // Zbar_l: Ybar for l == L, otherwise ping-pong buffer (L - 1 - l) mod 2 (include/ppsci_b200.h), or with keep_adj
  // a plane set of its own
  auto zbar = [&](int l) {
    return reinterpret_cast<T*>(ws + (l == L ? cv.ybar : P->keep_adj ? cv.zbl[l] : (L - 1 - l) % 2 ? cv.zbar1 : cv.zbar0));
  };
  const int TP = TM / C;
  const int PT = RC / C;
  const bool gated = s.gated != 0;  // ModifiedMLP: generic tile GEMMs + the gate kernels (kernels_gate.cuh)
  if (gated && a.phase != 0) return fail("two-phase value calls are not offered for gated networks");
  const bool pirate = s.gated == 2;  // PirateNet: layer 1 = embedding, blocks of (gate, gate, adaptive residual)
  // what follows hidden layer l in a gated plan: 0 gate, 1 adaptive residual (end of a block), 2 plain activation
  const int emb = gated ? gate_emb(s) : 0;  // layer 1 is an embedding layer (its stored output feeds embed_u / embed_v)
  auto post_kind = [&](int l) -> int { return (emb && l == 1) ? 2 : ((pirate && (l - 2) % 3 == 2) ? 1 : 0); };
  auto fill_mix = [&](int l, int64_t nc, MixArgs<T>* ma) {
    memset(ma, 0, sizeof(*ma));
    ma->J = P->J;
    ma->act = act_of_layer(s, l);
    ma->Z = reinterpret_cast<const T*>(ws + cv.z[l]);
    if (post_kind(l) == 1) {
      ma->Xprev = reinterpret_cast<const T*>(ws + cv.gt[l - 3]);
      ma->alpha = params + P->alpha_off + (l - 2) / 3;
    }
    ma->ld = P->ld[l];
    ma->plane = (long long)nc_max * P->ld[l];
    ma->Np = nc;
    ma->H = s.widths[l];
  };
  auto fill_gate = [&](int l, int64_t nc, GateArgs<T>* ga) {  // gate of hidden layer l
    memset(ga, 0, sizeof(*ga));
    ga->J = P->J;
    ga->act = s.act;
    ga->Z = reinterpret_cast<const T*>(ws + cv.z[l]);
    ga->Zu = reinterpret_cast<const T*>(ws + cv.zu);
    ga->Zv = reinterpret_cast<const T*>(ws + cv.zv);
    ga->ld = P->ld[l];
    ga->plane = (long long)nc_max * P->ld[l];
    ga->Np = nc;
    ga->H = s.widths[l];
  };
  // A operand of linear layer l for the chunk at point c0: the network input (layer 1), the stored output G_{l-1} of
  // what follows layer l-1 in a gated plan, or act(Z_{l-1}) with the activation's trainable parameter if it has one
  auto operand = [&](int l, int64_t c0) {
    AOperand<T> A;
    memset(&A, 0, sizeof(A));
    if (l == 1) {
      fill_first<T>(P, a.x_cols, c0, nc_max, params, &A);
    } else if (gated) {
      fill_act<T>(P, reinterpret_cast<const T*>(ws + cv.gt[l - 1]), P->ld[l - 1], nc_max, A_PLAIN, &A);
    } else {
      fill_act<T>(P, reinterpret_cast<const T*>(ws + cv.z[l - 1]), P->ld[l - 1], nc_max, A_ACT, &A, l - 1);
      if (P->actp_off[l - 1] >= 0) {
        A.act_param = params + P->actp_off[l - 1];
        A.act_pstride = P->actp_stride;
      }
    }
    return A;
  };
#ifndef PPSCI_EMUL
  // k_wg_layer over a chunk of nc points (dx: Zbar_{l-1} from Zbar_l) with the weight image at img_off of the wimg
  // region, output in the pitch of layer lo; a persistent grid of at most one CTA per SM
  auto launch_wg = [&](int cls, bool dx, wg::WgArgs& w, size_t img_off, int lo, float* out, int64_t nc) -> int {
    w.J = P->J;
    w.Wimg = reinterpret_cast<const float*>(ws + cv.wimg + img_off);
    w.Out = out;
    w.ldo = P->ld[lo];
    w.oplane = (long long)nc_max * P->ld[lo];
    w.Np = nc;
    const unsigned tiles = (unsigned)((nc + wg::tile_points(C) - 1) / wg::tile_points(C));
    w.num_tiles = (int)tiles;
    const int smem = wg::fwd_smem_bytes(w.Nout);
    void (*k)(wg::WgArgs) = nullptr;
    with_lay(WgLays{}, P->J, [&](auto lay) {
      with_int<8>(w.Nout / 32, [&](auto nq) {
        k = dx ? wg::k_wg_layer<decltype(lay), nq, true> : wg::k_wg_layer<decltype(lay), nq, false>;
      });
    });
    CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    launch(cls, k, dim3(tiles < (unsigned)P->num_sms ? tiles : (unsigned)P->num_sms), dim3(wg::THREADS), smem, w);
    return 0;
  };
#endif

  if (a.want_loss) CK(cudaMemsetAsync(loss_acc, 0, PPSCI_MAX_RES * sizeof(double), st));
  double* omega_acc = reinterpret_cast<double*>(ws + cv.omega_acc);
  // phase 1 runs the forward exactly as a training call would (stash of everything the adjoint reads), phase 2 only the adjoint
  const bool do_bwd = ((a.want_loss || a.ybar_in) && grads != nullptr) || a.phase == 1;
  if (a.phase == 2 && a.n_points > nc_max)
    return fail("values_bwd_kept: the kept stash covers one workspace chunk (" + std::to_string(nc_max) + " points); got " +
                std::to_string(a.n_points));
  // dLoss/d omega of the trainable frequencies: fp64 sums over the call, added to grads at its end
  const bool omega_bwd = do_bwd && a.phase != 1 && s.n_omega > 0;
  if (omega_bwd) CK(cudaMemsetAsync(omega_acc, 0, (size_t)s.n_omega * sizeof(double), st));
  if (do_bwd) {  // W_l^T for l >= 2; the embeddings hand an adjoint back to layer 1's output: Wu^T, Wv^T (layer 2's shape)
    struct Transpose {
      int l;       // layer whose shape the weights have
      int64_t w;   // weights in params
      size_t wt;   // transpose in the workspace
    };
    std::vector<Transpose> tr;
    for (int l = 2; l <= L; ++l) tr.push_back({l, P->w_off[l], cv.wt[l]});
    for (int e = 0; e < (emb ? 2 : 0); ++e) tr.push_back({2, P->gate_w_off[e], e == 0 ? cv.wtu : cv.wtv});
    for (const Transpose& t : tr) {
      const int K = s.widths[t.l - 1], N = s.widths[t.l];
      launch(CLS_MISC, k_transpose<T>, dim3((unsigned)(((long long)K * N + 255) / 256)), dim3(256), 0, params + t.w,
             reinterpret_cast<T*>(ws + t.wt), K, N);
    }
  }

#ifndef PPSCI_EMUL
  for (int l = 1; l <= L; ++l) {  // tf32 hi / lo images of the weights of the wgmma-served layers, once per call
    const dim3 grid((unsigned)(((long long)s.widths[l - 1] * s.widths[l] + 255) / 256));
    const float* W = reinterpret_cast<const float*>(params) + P->w_off[l];
    if (P->wg_fwd[l] && a.phase != 2) {
      if (l == 1)  // zero rows beyond the dense first layer's contraction length
        CK(cudaMemsetAsync(ws + cv.wimg + P->img_off[1], 0, (size_t)wg_kpad(s.widths[0]) * s.widths[1] * 8, st));
      launch(CLS_MISC, wg::k_wg_prep_w, grid, dim3(256), 0, W, reinterpret_cast<float*>(ws + cv.wimg + P->img_off[l]),
             s.widths[l - 1], s.widths[l], 0);
    }
    if (P->wg_dx[l] && do_bwd)  // gemm K = fan-out, gemm N = fan-in
      launch(CLS_MISC, wg::k_wg_prep_w, grid, dim3(256), 0, W, reinterpret_cast<float*>(ws + cv.wimg + P->imgT_off[l]),
             s.widths[l], s.widths[l - 1], 1);
  }
#endif
  for (int64_t c0 = 0; c0 < a.n_points; c0 += nc_max) {
    const int64_t nc = (a.n_points - c0) < nc_max ? (a.n_points - c0) : nc_max;
    const unsigned ptiles = (unsigned)((nc + TP - 1) / TP);
    // ---------------- forward ----------------
    for (int l = (a.phase == 2 ? L + 1 : 1); l <= L; ++l) {
      if (l == 1 && P->thin_first) {
        FirstArgs<T> f;
        memset(&f, 0, sizeof(f));
        f.A = operand(1, c0);
        f.J = P->J;
        f.W = params + P->w_off[1];
        f.bias = params + P->b_off[1];
        f.nf = s.widths[0];
        f.N = s.widths[1];
        f.Out = reinterpret_cast<T*>(ws + cv.z[1]);
        f.ldo = P->ld[1];
        f.oplane = (long long)nc_max * P->ld[1];
        f.Np = nc;
        void (*k)(FirstArgs<T>) = k_first_fwd<T, KMAX>;
        dim3 grid((unsigned)((nc * f.N + 255) / 256));
        if constexpr (sizeof(T) == 4) {
          if (P->thin_vec && f.N % 4 == 0) {  // compile-time layout, 128-bit stores, seeds staged once per point
            with_lay(ThinLays{}, P->J, [&](auto lay) { k = thin::k_first_fwd_v<decltype(lay)>; });
            grid = dim3((unsigned)((nc + thin::PB - 1) / thin::PB));
          }
        }
        launch(CLS_THIN_FWD, k, grid, dim3(256), 0, f);
        continue;
      }
      if (l == L && P->thin_last) {
        LastArgs<T> f;
        memset(&f, 0, sizeof(f));
        f.A = operand(L, c0);
        f.J = P->J;
        f.W = params + P->w_off[L];
        f.bias = params + P->b_off[L];
        f.K = s.widths[L - 1];
        f.m = s.widths[L];
        f.Y = reinterpret_cast<T*>(ws + cv.y);
        f.ldy = P->ld[L];
        f.yplane = (long long)nc_max * P->ld[L];
        f.Np = nc;
        void (*k)(LastArgs<T>) = k_last_fwd<T, KMAX>;
        if constexpr (sizeof(T) == 4) {
          if (P->thin_vec && f.K % 4 == 0 && f.m <= 4)
            with_lay(ThinLays{}, P->J, [&](auto lay) { with_int<4>(f.m, [&](auto m) { k = thin::k_last_fwd_v<decltype(lay), m>; }); });
        }
        launch(CLS_THIN_FWD, k, dim3((unsigned)((nc + 7) / 8)), dim3(256), 0, f);
        continue;
      }
#ifndef PPSCI_EMUL
      if (P->wg_fwd[l]) {
        if constexpr (sizeof(T) == 4) {
          wg::WgArgs w;
          memset(&w, 0, sizeof(w));
          w.A = operand(l, c0);
          w.Kdim = s.widths[l - 1];
          if (l == 1) {  // dense first layer: the caller's [n_points][n_feat] matrix as is, columns beyond n_feat read as zero
            w.A.act = PPSCI_ACT_IDENTITY;
            w.Kdim = wg_kpad(s.widths[0]);
            w.Kvalid = s.widths[0];
          }
          w.Nout = s.widths[l];
          w.bias = params + P->b_off[l];
          // a wide output layer writes Y
          if (launch_wg(CLS_FWD, false, w, P->img_off[l], l, reinterpret_cast<T*>(ws + (l < L ? cv.z[l] : cv.y)), nc)) return 1;
        }
        continue;
      }
#endif
      GemmArgs<T> g;
      memset(&g, 0, sizeof(g));
      g.A = operand(l, c0);
      g.J = P->J;
      g.B = params + P->w_off[l];
      g.Kdim = s.widths[l - 1];
      g.Nout = s.widths[l];
      g.ldb = s.widths[l];
      g.bias = params + P->b_off[l];
      g.Out = reinterpret_cast<T*>(ws + (l < L ? cv.z[l] : cv.y));
      g.ldo = P->ld[l];
      g.oplane = (long long)nc_max * P->ld[l];
      g.Np = nc;
      g.TP = TP;
      launch(CLS_FWD, kf, dim3(ptiles, (unsigned)((g.Nout + TN - 1) / TN)), dim3(NTHREADS), smem_f, g);
      auto post_fwd = [&](int lay) {  // operand of layer lay + 1
        const dim3 grid((unsigned)(((long long)nc * s.widths[lay] + 127) / 128));
        if (post_kind(lay) == 0) {  // G = V + act(Z) (U - V)
          GateArgs<T> ga;
          fill_gate(lay, nc, &ga);
          ga.G = reinterpret_cast<T*>(ws + cv.gt[lay]);
          launch(CLS_MISC, k_gate_fwd<T, KMAX>, grid, dim3(128), 0, ga);
        } else {  // X = alpha act(Z) + (1 - alpha) X_block_in, or X = act(Z)
          MixArgs<T> ma;
          fill_mix(lay, nc, &ma);
          ma.X = reinterpret_cast<T*>(ws + cv.gt[lay]);
          launch(CLS_MISC, k_mix_fwd<T, KMAX>, grid, dim3(128), 0, ma);
        }
      };
      if (emb && l == 1) post_fwd(1);
      if (gated && l == 1) {  // embed_u / embed_v: two more layers from the seeds, or from the embedding layer's output
        g.A = operand(emb + 1, c0);
        g.Kdim = s.widths[emb];
        g.Nout = s.widths[emb + 1];
        g.ldb = s.widths[emb + 1];
        g.ldo = P->ld[emb + 1];
        g.oplane = (long long)nc_max * P->ld[emb + 1];
        for (int e = 0; e < 2; ++e) {
          g.B = params + P->gate_w_off[e];
          g.bias = params + P->gate_b_off[e];
          g.Out = reinterpret_cast<T*>(ws + (e == 0 ? cv.zu : cv.zv));
          launch(CLS_FWD, kf, dim3(ptiles, (unsigned)((g.Nout + TN - 1) / TN)), dim3(NTHREADS), smem_f, g);
        }
      }
      if (gated && l < L && !(emb && l == 1)) post_fwd(l);
    }
    // ---------------- residual program + loss + output adjoints ----------------
    if (a.jets_out) {
      const long long tot = (long long)C * nc * n_out;
      launch(CLS_MISC, k_copy_jets<T>, dim3((unsigned)((tot + 255) / 256)), dim3(256), 0,
             reinterpret_cast<const T*>(ws + cv.y), P->ld[L], (long long)nc_max * P->ld[L],
             reinterpret_cast<T*>(a.jets_out), (long long)a.n_points, (long long)c0, (long long)nc, C, n_out);
    }
    if (s.n_res > 0 && (a.want_loss || a.residual_out) && !a.ybar_in) {
      HeadArgs<T> h;
      memset(&h, 0, sizeof(h));
      h.P.prog = P->d_prog;
      h.P.consts = P->d_consts;
      h.P.n_ops = s.n_ops;
      h.P.n_reg = s.n_reg;
      h.P.n_res = s.n_res;
      for (int k = 0; k < PPSCI_MAX_RES; ++k) h.P.res_reg[k] = k < s.n_res ? s.res_reg[k] : 0;
      h.P.n_grad = s.n_grad;
      h.P.grad_res = P->d_grad_res;
      h.P.grad_in = P->d_grad_in;
      h.P.grad_reg = P->d_grad_reg;
      h.P.n_pgrad = s.n_pgrad;
      for (int g = 0; g < PPSCI_MAX_PGRAD; ++g) {
        h.P.pgrad_res[g] = g < s.n_pgrad ? s.pgrad_res[g] : 0;
        h.P.pgrad_aux[g] = g < s.n_pgrad ? s.pgrad_aux[g] : -1;
        h.P.pgrad_reg[g] = g < s.n_pgrad ? s.pgrad_reg[g] : 0;
      }
      for (int i = 0; i < PPSCI_MAX_IN; ++i) {
        h.aux_bcast[i] = i < s.n_aux ? s.aux_bcast[i] : 0;
        h.aux_grad[i] = (i < s.n_aux && s.aux_bcast[i] && do_bwd) ? P->aux_grad[i] : nullptr;
      }
      h.C = C;
      h.n_out = n_out;
      h.n_in = s.n_in;
      h.n_aux = s.n_aux;
      h.Y = reinterpret_cast<const T*>(ws + cv.y);
      h.ldy = P->ld[L];
      h.yplane = (long long)nc_max * P->ld[L];
      h.Ybar = do_bwd ? reinterpret_cast<T*>(ws + cv.ybar) : nullptr;
      for (int i = 0; i < s.n_in; ++i) h.x_cols[i] = a.x_cols[i];
      for (int i = 0; i < s.n_aux; ++i) h.aux_cols[i] = a.aux_cols ? a.aux_cols[i] : nullptr;
      h.x_off = c0;
      h.Np = nc;
      for (int k = 0; k < s.n_res; ++k) {
        h.label_cols[k] = a.label_cols ? a.label_cols[k] : nullptr;
        h.label_const[k] = a.label_const ? a.label_const[k] : 0.0;
        h.weight_cols[k] = a.weight_cols ? a.weight_cols[k] : nullptr;
        h.coef[k] = s.loss_weight[k] * (s.reduction[k] == PPSCI_REDUCE_MEAN ? 1.0 / (double)a.n_norm : 1.0);
        h.residual_out[k] = a.residual_out ? a.residual_out[k] : nullptr;
      }
      h.loss_acc = a.want_loss ? loss_acc : nullptr;
      launch(CLS_HEAD, k_head<T>, dim3((unsigned)((nc + HEAD_THREADS - 1) / HEAD_THREADS)), dim3(HEAD_THREADS), 0, h);
    }
    if (!do_bwd || a.phase == 1) continue;
    if (a.ybar_in && a.ybar_in != static_cast<const void*>(ws + cv.ybar)) {  // output adjoints from the caller (not already in place)
      const long long tot = (long long)nc * P->ld[L];
      launch(CLS_MISC, k_seed_ybar<T>, dim3((unsigned)((tot + 255) / 256)), dim3(256), 0, reinterpret_cast<const T*>(a.ybar_in),
             (long long)c0, (long long)nc, n_out, C, reinterpret_cast<T*>(ws + cv.ybar), P->ld[L], (long long)nc_max * P->ld[L]);
    }
    // ---------------- adjoint ----------------
    for (int l = L; l >= 1; --l) {
      if (l == L && P->thin_last) {  // dW_L, db_L and Zbar_{L-1} in one streaming pass
        LastArgs<T> f;
        memset(&f, 0, sizeof(f));
        f.A = operand(L, c0);
        f.J = P->J;
        f.W = params + P->w_off[L];
        f.K = s.widths[L - 1];
        f.m = s.widths[L];
        f.Ybar = zbar(L);
        f.ldy = P->ld[L];
        f.yplane = (long long)nc_max * P->ld[L];
        f.ZbarOut = zbar(L - 1);
        f.ldo = P->ld[L - 1];
        f.oplane = (long long)nc_max * P->ld[L - 1];
        f.dW = grads + P->w_off[L];
        f.db = grads + P->b_off[L];
        f.Np = nc;
        f.pts_per_block = 64;
        void (*k)(LastArgs<T>) = k_last_bwd<T, KMAX>;
        if constexpr (sizeof(T) == 4) {
          if (P->thin_vec && f.K % 4 == 0 && f.m <= 4) {
            f.pts_per_block = 128;
            with_lay(ThinLays{}, P->J, [&](auto lay) { with_int<4>(f.m, [&](auto m) { k = thin::k_last_bwd_v<decltype(lay), m>; }); });
          }
        }
        const dim3 grid((unsigned)((f.K + 255) / 256), (unsigned)((nc + f.pts_per_block - 1) / f.pts_per_block));
        launch(CLS_THIN_DX, k, grid, dim3(256), 0, f);
        continue;
      }
      if (l == 1 && P->thin_first) {
        FirstArgs<T> f;
        memset(&f, 0, sizeof(f));
        f.A = operand(1, c0);
        f.J = P->J;
        f.nf = s.widths[0];
        f.N = s.widths[1];
        f.Zbar = zbar(1);
        f.ldzb = P->ld[1];
        f.zbplane = (long long)nc_max * P->ld[1];
        f.dW = grads + P->w_off[1];
        f.db = grads + P->b_off[1];
        f.Np = nc;
        f.pts_per_block = 32;
        f.W = params + P->w_off[1];
        f.omega_grad = omega_acc;
        void (*k)(FirstArgs<T>) = omega_bwd ? k_first_dw<T, KMAX, true> : k_first_dw<T, KMAX>;
        if constexpr (sizeof(T) == 4) {
          if (P->thin_vec && f.N % 4 == 0) {
            f.pts_per_block = 256;
            with_lay(ThinLays{}, P->J, [&](auto lay) {
              k = omega_bwd ? thin::k_first_dw_v<decltype(lay), true> : thin::k_first_dw_v<decltype(lay)>;
            });
          }
        }
        const dim3 grid((unsigned)((f.N + 255) / 256), (unsigned)((nc + f.pts_per_block - 1) / f.pts_per_block));
        launch(CLS_THIN_DW, k, grid, dim3(256), 0, f);
        break;
      }
#ifndef PPSCI_EMUL
      if (P->wg_dw[l]) {  // dW_l and db_l on the tensor cores
        if constexpr (sizeof(T) == 4) {
          wg::WgDwArgs w;
          memset(&w, 0, sizeof(w));
          w.A = operand(l, c0);
          if (l == 1) w.A.act = PPSCI_ACT_IDENTITY;  // dense first layer: the caller's matrix is the operand
          w.J = P->J;
          w.Zbar = zbar(l);
          w.ldzb = P->ld[l];
          w.zbplane = (long long)nc_max * P->ld[l];
          w.Kdim = s.widths[l - 1];
          w.Nout = s.widths[l];
          w.dW = grads + P->w_off[l];
          w.db = grads + P->b_off[l];
          w.Np = nc;
          // column blocks of equal width (in units of 32) up to dw_maxq(C); fan-in blocks x column blocks fastest on the
          // grid, so the CTAs that read the same points run together and share them through L2
          const int nq = w.Nout / 32, ncb = (nq + wg::dw_maxq(C) - 1) / wg::dw_maxq(C), bnq = (nq + ncb - 1) / ncb;
          w.col_blocks = ncb;
          const unsigned tiles = (unsigned)((w.Kdim + wg::DW_TK - 1) / wg::DW_TK * ncb);
          const DwSplit sp = dw_split(P->num_sms / tiles, (nc + wg::dw_pch(C) - 1) / wg::dw_pch(C));
          w.chunks_per_split = sp.chunks_per_split;
          const int smem = wg::dw_smem_bytes(C, bnq);
          void (*k)(wg::WgDwArgs) = nullptr;
          with_lay(WgLays{}, P->J, [&](auto lay) {
            with_int<4>(bnq, [&](auto q) {  // bnq <= dw_maxq(C): the wider blocks of a layout are never instantiated
              if constexpr (q <= wg::dw_maxq(decltype(lay)::CS)) k = wg::k_wg_dw<decltype(lay), q>;
            });
          });
          CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
          launch(CLS_DW, k, dim3(tiles, sp.splits), dim3(wg::THREADS), smem, w);
        }
      } else
#endif
      {  // dW_l, db_l
        DwArgs<T> g;
        memset(&g, 0, sizeof(g));
        g.A = operand(l, c0);
        g.J = P->J;
        g.Zbar = zbar(l);
        g.ldzb = P->ld[l];
        g.zbplane = (long long)nc_max * P->ld[l];
        g.Kdim = s.widths[l - 1];
        g.Nout = s.widths[l];
        g.dW = grads + P->w_off[l];
        g.db = grads + P->b_off[l];
        g.Np = nc;
        g.PT = PT;
        const unsigned kt = (unsigned)((g.Kdim + TM - 1) / TM), nt = (unsigned)((g.Nout + TN - 1) / TN);
        const DwSplit sp = dw_split((4LL * P->num_sms + kt * nt - 1) / (kt * nt), (nc + PT - 1) / PT);
        g.chunks_per_split = sp.chunks_per_split;
        launch(CLS_DW, kw, dim3(kt, nt, sp.splits), dim3(NTHREADS), smem_w, g);
        if (gated && l == 1) {  // dWu, dbu, dWv, dbv from the adjoints the gates accumulated
          g.A = operand(emb + 1, c0);
          g.Kdim = s.widths[emb];
          g.Nout = s.widths[emb + 1];
          const dim3 grid_e((unsigned)((g.Kdim + TM - 1) / TM), (unsigned)((g.Nout + TN - 1) / TN), sp.splits);
          for (int e = 0; e < 2; ++e) {
            g.Zbar = reinterpret_cast<const T*>(ws + (e == 0 ? cv.zub : cv.zvb));
            g.ldzb = P->ld[emb + 1];
            g.zbplane = (long long)nc_max * P->ld[emb + 1];
            g.dW = grads + P->gate_w_off[e];
            g.db = grads + P->gate_b_off[e];
            launch(CLS_DW, kw, grid_e, dim3(NTHREADS), smem_w, g);
          }
        }
        if (l == 1 && omega_bwd) {  // dLoss/d omega from every GEMM that read the seeds
          OmegaArgs<T> o;
          memset(&o, 0, sizeof(o));
          o.A = operand(1, c0);
          o.J = P->J;
          o.nf = s.n_feat;
          auto cons = [&](const T* zb, int lo, int64_t w_off) {
            o.Zbar[o.n_cons] = zb;
            o.ldzb[o.n_cons] = P->ld[lo];
            o.zbplane[o.n_cons] = (long long)nc_max * P->ld[lo];
            o.W[o.n_cons] = params + w_off;
            o.N[o.n_cons] = s.widths[lo];
            o.n_cons++;
          };
          cons(zbar(1), 1, P->w_off[1]);
          if (gated && !emb) {  // ModifiedMLP without an embedding layer: embed_u / embed_v read the seeds too
            cons(reinterpret_cast<const T*>(ws + cv.zub), 1, P->gate_w_off[0]);
            cons(reinterpret_cast<const T*>(ws + cv.zvb), 1, P->gate_w_off[1]);
          }
          o.Np = nc;
          o.omega_grad = omega_acc;
          const long long want = (nc + 7) / 8, cap = 4LL * P->num_sms;
          launch(CLS_MISC, k_omega_grad<T, KMAX>, dim3((unsigned)(want < cap ? want : cap)), dim3(256), 0, o);
        }
      }
      if (l == 1) break;
#ifndef PPSCI_EMUL
      if (P->wg_dx[l]) {  // Zbar_{l-1} on the tensor cores
        if constexpr (sizeof(T) == 4) {
          wg::WgArgs w;
          memset(&w, 0, sizeof(w));
          fill_act<T>(P, zbar(l), P->ld[l], nc_max, A_PLAIN, &w.A);
          w.Kdim = s.widths[l];
          w.Nout = s.widths[l - 1];
          w.Zprev = reinterpret_cast<const T*>(ws + cv.z[l - 1]);
          w.ldz = P->ld[l - 1];
          w.zplane = (long long)nc_max * P->ld[l - 1];
          w.act = act_of_layer(s, l - 1);
          if (launch_wg(CLS_DX, true, w, P->imgT_off[l], l - 1, zbar(l - 1), nc)) return 1;
        }
        continue;
      }
#endif
      {  // Zbar_{l-1}
        GemmArgs<T> g;
        memset(&g, 0, sizeof(g));
        fill_act<T>(P, zbar(l), P->ld[l], nc_max, A_PLAIN, &g.A);
        g.J = P->J;
        g.B = reinterpret_cast<const T*>(ws + cv.wt[l]);  // [N_l][K_l]
        g.Kdim = s.widths[l];
        g.Nout = s.widths[l - 1];
        g.ldb = s.widths[l - 1];
        g.bias = nullptr;
        T* outp = zbar(l - 1);
        g.Out = outp;
        g.ldo = P->ld[l - 1];
        g.oplane = (long long)nc_max * P->ld[l - 1];
        g.Np = nc;
        g.TP = TP;
        g.Zprev = reinterpret_cast<const T*>(ws + cv.z[l - 1]);
        g.ldz = P->ld[l - 1];
        g.zplane = (long long)nc_max * P->ld[l - 1];
        g.act = gated ? (int)PPSCI_ACT_IDENTITY : act_of_layer(s, l - 1);  // gated: Gbar_{l-1}, the gate's adjoint follows
        if (!gated && P->actp_off[l - 1] >= 0) {  // trainable activation parameter: dLoss/dbeta comes out of this epilogue
          g.act_param = params + P->actp_off[l - 1];
          g.act_param_grad = grads + P->actp_off[l - 1];
          g.act_pstride = P->actp_stride;
        }
        const dim3 grid(ptiles, (unsigned)((g.Nout + TN - 1) / TN));
        launch(CLS_DX, kx, grid, dim3(NTHREADS), smem_x, g);
        if (gated && emb && l == 2) {  // layer 1's output also feeds the embeddings: += Zubar Wu^T + Zvbar Wv^T
          for (int e = 0; e < 2; ++e) {
            fill_act<T>(P, reinterpret_cast<const T*>(ws + (e == 0 ? cv.zub : cv.zvb)), P->ld[2], nc_max, A_PLAIN, &g.A);
            g.B = reinterpret_cast<const T*>(ws + (e == 0 ? cv.wtu : cv.wtv));
            g.accum = 1;
            launch(CLS_DX, kx, grid, dim3(NTHREADS), smem_x, g);
          }
        }
        if (gated) {  // adjoint of what follows layer l-1, in place: operand adjoint -> Zbar_{l-1}
          const long long tot = (long long)nc * s.widths[l - 1];
          if (post_kind(l - 1) == 0) {  // gate; the adjoints of the embeddings' pre-activations accumulate
            GateArgs<T> ga;
            fill_gate(l - 1, nc, &ga);
            ga.G = outp;
            ga.Zub = reinterpret_cast<T*>(ws + cv.zub);
            ga.Zvb = reinterpret_cast<T*>(ws + cv.zvb);
            ga.first = (l - 1 == (pirate ? L - 2 : L - 1)) ? 1 : 0;
            launch(CLS_MISC, k_gate_bwd<T, KMAX>, dim3((unsigned)((tot + 127) / 128)), dim3(128), 0, ga);
          } else {  // adaptive residual of a block (dLoss/dalpha reduced here), or the embedding layer's activation
            MixArgs<T> ma;
            fill_mix(l - 1, nc, &ma);
            ma.X = outp;
            ma.Xres = reinterpret_cast<T*>(ws + cv.xres);
            if (post_kind(l - 1) == 1) {
              ma.alpha_grad = grads + P->alpha_off + (l - 3) / 3;
              ma.use_res = (l - 1 != L - 1) ? 1 : 0;  // the last block's output feeds the output layer only
              ma.write_res = 1;
            } else {
              ma.use_res = pirate ? 1 : 0;  // block 0's residual path
            }
            const long long want = (tot + 127) / 128, cap = 8LL * P->num_sms;
            launch(CLS_MISC, k_mix_bwd<T, KMAX>, dim3((unsigned)(want < cap ? want : cap)), dim3(128), 0, ma);
          }
        }
      }
    }
  }
  if (omega_bwd)
    launch(CLS_MISC, k_omega_finish<T>, dim3((unsigned)((s.n_omega + 31) / 32)), dim3(32), 0, omega_acc, grads + P->omega_off,
           (int)s.n_omega);
  if (a.want_loss && a.loss_out && s.n_res > 0)
    launch(CLS_MISC, k_finalize_loss<T>, dim3(1), dim3(32), 0, loss_acc, reinterpret_cast<T*>(a.loss_out), s.n_res);
  CK(cudaGetLastError());
  return 0;
}

template <typename T>
static int dispatch_k(ppsci_plan* P, const CallArgs& a) {
  if (P->kmax <= 1) return run<T, 1>(P, a);
  if (P->kmax == 2) return run<T, 2>(P, a);
  return run<T, 4>(P, a);
}

static int dispatch(ppsci_plan* P, const CallArgs& a) {
  if (!P) return fail("null plan");
  if (a.n_points <= 0) return fail("n_points must be positive");
  if (!a.x_cols || !a.params || !a.workspace) return fail("null x_cols / params / workspace");
  for (int i = 0; i < P->spec.n_in; ++i)
    if (!a.x_cols[i]) return fail("null input column " + std::to_string(i));
  if (P->spec.n_aux > 0) {
    if (!a.aux_cols) return fail("plan needs aux columns but aux_cols is null");
    for (int i = 0; i < P->spec.n_aux; ++i)
      if (!a.aux_cols[i]) return fail("null aux column " + std::to_string(i));
  }
  return with_dtype(P->spec.dtype, "plan", [&](auto zero) { return dispatch_k<decltype(zero)>(P, a); });
}

extern "C" int ppsci_b200_plan_set_aux_grad(ppsci_plan* plan, int32_t aux_index, double* grad_dev) {
  if (!plan) return fail("null plan");
  if (aux_index < 0 || aux_index >= plan->spec.n_aux || !plan->spec.aux_bcast[aux_index])
    return fail("plan_set_aux_grad: aux_index is not a learnable (broadcast) parameter of this plan");
  plan->aux_grad[aux_index] = grad_dev;
  return 0;
}

extern "C" int ppsci_b200_values_fwd_bwd(ppsci_plan* plan, const void* const* x_cols, const void* const* aux_cols,
                                         int64_t n_points, const void* params, void* grads, const void* ybar,
                                         void* workspace, size_t workspace_bytes, void* stream) {
  if (!ybar || !grads) return fail("values_fwd_bwd: null ybar / grads");
  CallArgs a;
  memset(&a, 0, sizeof(a));
  a.x_cols = x_cols;
  a.aux_cols = aux_cols;
  a.n_points = n_points;
  a.n_norm = n_points;
  a.params = params;
  a.grads = grads;
  a.workspace = workspace;
  a.workspace_bytes = workspace_bytes;
  a.stream = stream;
  a.want_loss = false;
  a.ybar_in = ybar;
  return dispatch(plan, a);
}

extern "C" int ppsci_b200_residual_loss_fwd_bwd(ppsci_plan* plan, const void* const* x_cols,
                                                const void* const* aux_cols, const void* const* label_cols,
                                                const double* label_const, const void* const* weight_cols,
                                                int64_t n_points, int64_t n_norm, const void* params, void* grads,
                                                void* loss_out, void* const* residual_out, void* workspace,
                                                size_t workspace_bytes, void* stream) {
  if (plan && plan->spec.n_res < 1) return fail("residual_loss_fwd_bwd: plan has no residuals");
  if (!loss_out) return fail("residual_loss_fwd_bwd: loss_out is null");
  if (n_norm <= 0) return fail("residual_loss_fwd_bwd: n_norm must be positive");
  CallArgs a{x_cols, aux_cols, label_cols, label_const, weight_cols, n_points, n_norm, params, grads, loss_out,
             residual_out, nullptr, workspace, workspace_bytes, stream, true};
  return dispatch(plan, a);
}

extern "C" int ppsci_b200_residual_fwd(ppsci_plan* plan, const void* const* x_cols, const void* const* aux_cols,
                                       int64_t n_points, const void* params, void* jets_out,
                                       void* const* residual_out, void* workspace, size_t workspace_bytes,
                                       void* stream) {
  CallArgs a{x_cols, aux_cols, nullptr, nullptr, nullptr, n_points, 1, params, nullptr, nullptr,
             residual_out, jets_out, workspace, workspace_bytes, stream, false};
  return dispatch(plan, a);
}

extern "C" int32_t ppsci_b200_plan_chunk_points(const ppsci_plan* P) { return P ? P->chunk : -1; }

extern "C" int ppsci_b200_values_fwd_keep(ppsci_plan* plan, const void* const* x_cols, const void* const* aux_cols, int64_t n_points,
                                          const void* params, void* y_out, void* workspace, size_t workspace_bytes, void* stream) {
  // y_out may be NULL: the caller then reads the outputs in place, [n_points][ld] at plan_stash_offset(n_layers) of the
  // workspace (no copy; ld = n_out rounded up to a multiple of 4)
  if (plan && n_points > plan->chunk) return fail("values_fwd_keep: at most plan_chunk_points points per call");
  CallArgs a;
  memset(&a, 0, sizeof(a));
  a.x_cols = x_cols;
  a.aux_cols = aux_cols;
  a.n_points = n_points;
  a.n_norm = n_points;
  a.params = params;
  a.jets_out = y_out;  // C = 1: [n_points][n_out]
  a.workspace = workspace;
  a.workspace_bytes = workspace_bytes;
  a.stream = stream;
  a.phase = 1;
  if (plan && plan->C != 1) return fail("values_fwd_keep: the plan must have no input derivatives (C == 1)");
  return dispatch(plan, a);
}

extern "C" int ppsci_b200_values_bwd_kept(ppsci_plan* plan, const void* const* x_cols, const void* const* aux_cols, int64_t n_points,
                                          const void* params, void* grads, const void* ybar, void* workspace,
                                          size_t workspace_bytes, void* stream) {
  if (!ybar || !grads) return fail("values_bwd_kept: null ybar / grads");
  CallArgs a;
  memset(&a, 0, sizeof(a));
  a.x_cols = x_cols;
  a.aux_cols = aux_cols;
  a.n_points = n_points;
  a.n_norm = n_points;
  a.params = params;
  a.grads = grads;
  a.workspace = workspace;
  a.workspace_bytes = workspace_bytes;
  a.stream = stream;
  a.ybar_in = ybar;
  a.phase = 2;
  return dispatch(plan, a);
}

extern "C" int ppsci_b200_deeponet_head(int32_t dtype, int32_t act, const void* b, const void* t, const void* bias,
                                        const void* label, const void* weight, int64_t n, int32_t n_features, double coef,
                                        void* g_out, double* loss_acc, void* bbar, void* tbar, void* dbias, void* stream) {
  if (!b || !t || n <= 0 || n_features <= 0) return fail("deeponet_head: bad arguments");
  if ((bbar == nullptr) != (tbar == nullptr)) return fail("deeponet_head: bbar and tbar must both be given or both be null");
  if (act < 0 || act > PPSCI_ACT_LAST) return fail("deeponet_head: unknown activation");
  if (act_has_param(act)) return fail("deeponet_head: activations with a trainable parameter are not offered here");
  const long long warps = n < 132LL * 64 ? n : 132LL * 64;  // 8 warps per block
  const unsigned blocks = (unsigned)((warps + 7) / 8);
  return with_dtype(dtype, "deeponet_head", [&](auto zero) {
    using T = decltype(zero);
    PPSCI_LAUNCH(k_deeponet_head<T>, dim3(blocks), dim3(256), 0, stream, (const T*)b, (const T*)t, (const T*)bias, act,
                 (const T*)label, (const T*)weight, (long long)n, n_features, coef, (T*)g_out, loss_acc, (T*)bbar, (T*)tbar,
                 (T*)dbias);
    CK(cudaGetLastError());
    return 0;
  });
}

extern "C" int ppsci_b200_jets_fwd_keep(ppsci_plan* plan, const void* const* x_cols, const void* const* aux_cols, int64_t n_points,
                                        const void* params, void* workspace, size_t workspace_bytes, void* stream) {
  if (plan && n_points > plan->chunk) return fail("jets_fwd_keep: at most plan_chunk_points points per call");
  CallArgs a;
  memset(&a, 0, sizeof(a));
  a.x_cols = x_cols;
  a.aux_cols = aux_cols;
  a.n_points = n_points;
  a.n_norm = n_points;
  a.params = params;
  a.workspace = workspace;
  a.workspace_bytes = workspace_bytes;
  a.stream = stream;
  a.phase = 1;
  return dispatch(plan, a);
}

extern "C" int ppsci_b200_jets_bwd_kept(ppsci_plan* plan, const void* const* x_cols, const void* const* aux_cols, int64_t n_points,
                                        const void* params, void* grads, void* workspace, size_t workspace_bytes, void* stream) {
  if (!grads) return fail("jets_bwd_kept: null grads");
  if (!plan || !workspace || n_points <= 0) return fail("jets_bwd_kept: bad arguments");
  CallArgs a;
  memset(&a, 0, sizeof(a));
  a.x_cols = x_cols;
  a.aux_cols = aux_cols;
  a.n_points = n_points;
  a.n_norm = n_points;
  a.params = params;
  a.grads = grads;
  a.workspace = workspace;
  a.workspace_bytes = workspace_bytes;
  a.stream = stream;
  a.ybar_in = static_cast<unsigned char*>(workspace) + ppsci_b200_plan_stash_offset(plan, n_points, 300);  // in place: no seeding
  a.phase = 2;
  return dispatch(plan, a);
}

struct ppsci_deeponet_head {
  ppsci_deeponet_head_spec spec;
  JetLayout J;
  int cb = 2;  // channel bound of the kernel instance
  int* d_prog = nullptr;
  double* d_consts = nullptr;
  int* d_grad_res = nullptr;
  int* d_grad_in = nullptr;
  int* d_grad_reg = nullptr;
};

extern "C" void ppsci_b200_deeponet_jet_head_destroy(ppsci_deeponet_head* H) {
  if (!H) return;
  cudaFree(H->d_prog);
  cudaFree(H->d_consts);
  cudaFree(H->d_grad_res);
  cudaFree(H->d_grad_in);
  cudaFree(H->d_grad_reg);
  delete H;
}

extern "C" int ppsci_b200_deeponet_jet_head_create(const ppsci_deeponet_head_spec* s, ppsci_deeponet_head** out) {
  if (!s || !out) return fail("deeponet_jet_head_create: null argument");
  *out = nullptr;
  if (s->dtype != PPSCI_F32 && s->dtype != PPSCI_F64) return fail("deeponet_jet_head_create: dtype must be f32 or f64");
  if (s->act < 0 || s->act > PPSCI_ACT_LAST) return fail("deeponet_jet_head_create: unknown activation");
  if (act_has_param(s->act)) return fail("deeponet_jet_head_create: activations with a trainable parameter are not offered here");
  if (s->n_out < 1 || s->n_out > DEEPONET_MAX_OUT) return fail("deeponet_jet_head_create: n_out must be 1 .. 3");
  if (s->n_in < 1 || s->n_in > PPSCI_MAX_IN) return fail("deeponet_jet_head_create: n_in out of range");
  if (s->n_dir < 0 || s->n_dir > PPSCI_MAX_DIR) return fail("deeponet_jet_head_create: n_dir out of range");
  int C = 1;
  for (int d = 0; d < s->n_dir; ++d) {
    if (s->dir_order[d] < 1 || s->dir_order[d] > PPSCI_MAX_ORDER) return fail("deeponet_jet_head_create: dir_order out of range");
    C += s->dir_order[d];
  }
  if (C > DEEPONET_MAX_CHANNELS)
    return fail("deeponet_jet_head_create: " + std::to_string(C) + " jet channels; the largest head instance takes " +
                std::to_string(DEEPONET_MAX_CHANNELS));
  if (s->n_aux < 0 || s->n_aux > PPSCI_MAX_IN) return fail("deeponet_jet_head_create: n_aux out of range");
  if (s->n_res < 1 || s->n_res > PPSCI_MAX_RES) return fail("deeponet_jet_head_create: n_res out of range");
  if (check_program("deeponet_jet_head_create", C * s->n_out + s->n_in + s->n_aux, C * s->n_out, s->n_reg, s->n_ops, s->prog,
                    s->n_consts, s->n_res, s->res_reg, s->n_grad, s->grad_res, s->grad_in, s->grad_reg))
    return 1;
  ppsci_deeponet_head* H = new ppsci_deeponet_head();
  H->spec = *s;
  H->spec.prog = nullptr;
  H->spec.consts = nullptr;
  H->spec.grad_res = H->spec.grad_in = H->spec.grad_reg = nullptr;
  memset(&H->J, 0, sizeof(H->J));
  H->J.C = C;
  H->J.n_dir = s->n_dir;
  for (int d = 0, base = 1; d < s->n_dir; base += s->dir_order[d], ++d) {
    H->J.dir_order[d] = s->dir_order[d];
    H->J.dir_base[d] = base;
  }
  H->cb = C <= 2 ? 2 : C <= 3 ? 3 : C <= 5 ? 5 : DEEPONET_MAX_CHANNELS;
  auto up = [&](const void* src, size_t bytes, void** dst) -> cudaError_t {
    cudaError_t e = cudaMalloc(dst, bytes ? bytes : 16);
    if (e != cudaSuccess) return e;
    if (bytes) return cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice);
    return cudaSuccess;
  };
  cudaError_t e = cudaSuccess;
  if (e == cudaSuccess) e = up(s->prog, (size_t)s->n_ops * 16, (void**)&H->d_prog);
  if (e == cudaSuccess) e = up(s->consts, (size_t)s->n_consts * 8, (void**)&H->d_consts);
  if (e == cudaSuccess) e = up(s->grad_res, (size_t)s->n_grad * 4, (void**)&H->d_grad_res);
  if (e == cudaSuccess) e = up(s->grad_in, (size_t)s->n_grad * 4, (void**)&H->d_grad_in);
  if (e == cudaSuccess) e = up(s->grad_reg, (size_t)s->n_grad * 4, (void**)&H->d_grad_reg);
  if (e != cudaSuccess) {
    ppsci_b200_deeponet_jet_head_destroy(H);
    return fail(std::string("deeponet_jet_head_create: device upload of the residual program failed: ") + cudaGetErrorString(e));
  }
  *out = H;
  return 0;
}

extern "C" int ppsci_b200_deeponet_jet_head_run(const ppsci_deeponet_head* H, const ppsci_deeponet_jet_args* a, void* stream) {
  if (!H || !a) return fail("deeponet_jet_head_run: null argument");
  const ppsci_deeponet_head_spec& s = H->spec;
  if (!a->b || !a->t || a->n <= 0 || a->n_features <= 0 || a->x_off < 0) return fail("deeponet_jet_head_run: bad arguments");
  const long long width = (long long)s.n_out * a->n_features;
  if (a->ldb < width || a->ldt < width || (a->b2 && a->ldb2 < width) || (a->b3 && a->ldb3 < width) ||
      a->tplane < a->n * a->ldt)
    return fail("deeponet_jet_head_run: row pitch or plane stride smaller than n_out * n_features");
  if ((a->bbar == nullptr) != (a->tbar == nullptr)) return fail("deeponet_jet_head_run: bbar and tbar must both be given or both be null");
  if (a->b2bar && !a->b2) return fail("deeponet_jet_head_run: b2bar given without the second branch's features b2");
  if (a->b2 && a->bbar && !a->b2bar) return fail("deeponet_jet_head_run: the adjoint of a two-branch head needs b2bar");
  if (a->b3 && !a->b2) return fail("deeponet_jet_head_run: a third branch factor b3 needs the second one, b2");
  if ((a->b3bar != nullptr) != (a->b3 != nullptr && a->bbar != nullptr))
    return fail("deeponet_jet_head_run: b3bar must be given exactly when b3 and bbar are");
  for (int j = 0; j < s.n_in; ++j)
    if (!a->x_cols[j]) return fail("deeponet_jet_head_run: null trunk input column " + std::to_string(j));
  for (int i = 0; i < s.n_aux; ++i)
    if (!a->aux_cols[i]) return fail("deeponet_jet_head_run: null aux column " + std::to_string(i));
  return with_dtype(s.dtype, "deeponet_jet_head_run", [&](auto zero) {
    using T = decltype(zero);
    DeepONetJetArgs<T> h;
    memset(&h, 0, sizeof(h));
    h.P.prog = H->d_prog;
    h.P.consts = H->d_consts;
    h.P.n_ops = s.n_ops;
    h.P.n_reg = s.n_reg;
    h.P.n_res = s.n_res;
    for (int k = 0; k < s.n_res; ++k) h.P.res_reg[k] = s.res_reg[k];
    h.P.n_grad = s.n_grad;
    h.P.grad_res = H->d_grad_res;
    h.P.grad_in = H->d_grad_in;
    h.P.grad_reg = H->d_grad_reg;
    h.J = H->J;
    h.act = s.act;
    h.n_out = s.n_out;
    h.n_in = s.n_in;
    h.b = (const T*)a->b;
    h.ldb = a->ldb;
    h.b2 = (const T*)a->b2;
    h.ldb2 = a->ldb2;
    h.t = (const T*)a->t;
    h.ldt = a->ldt;
    h.tplane = a->tplane;
    h.n = a->n;
    h.F = a->n_features;
    h.bias = (const T*)a->bias;
    for (int j = 0; j < s.n_in; ++j) h.x_cols[j] = a->x_cols[j];
    for (int i = 0; i < s.n_aux; ++i) h.aux_cols[i] = a->aux_cols[i];
    h.n_aux = s.n_aux;
    h.x_off = a->x_off;
    for (int k = 0; k < s.n_res; ++k) {
      h.label_cols[k] = a->label_cols[k];
      h.label_const[k] = a->label_const[k];
      h.weight_cols[k] = a->weight_cols[k];
      h.coef[k] = a->coef[k];
      h.residual_out[k] = a->residual_out[k];
    }
    h.loss_acc = a->loss_acc;
    h.bbar = (T*)a->bbar;
    h.b2bar = (T*)a->b2bar;
    h.tbar = (T*)a->tbar;
    h.dbias = (T*)a->dbias;
    h.b3 = (const T*)a->b3;
    h.ldb3 = a->ldb3;
    h.b3bar = (T*)a->b3bar;
    const long long warps = a->n < 132LL * 64 ? a->n : 132LL * 64;  // 8 warps per block
    const unsigned blocks = (unsigned)((warps + 7) / 8);
    using K = void (*)(DeepONetJetArgs<T>);
    const K ks[2][4] = {{k_deeponet_jet_head<T, 2, false>, k_deeponet_jet_head<T, 3, false>, k_deeponet_jet_head<T, 5, false>,
                         k_deeponet_jet_head<T, DEEPONET_MAX_CHANNELS, false>},
                        {k_deeponet_jet_head<T, 2, true>, k_deeponet_jet_head<T, 3, true>, k_deeponet_jet_head<T, 5, true>,
                         k_deeponet_jet_head<T, DEEPONET_MAX_CHANNELS, true>}};
    const K k = ks[a->b3 != nullptr][H->cb == 2 ? 0 : H->cb == 3 ? 1 : H->cb == 5 ? 2 : 3];
    PPSCI_LAUNCH(k, dim3(blocks), dim3(256), 0, stream, h);
    CK(cudaGetLastError());
    return 0;
  });
}

extern "C" int ppsci_b200_sample_uniform(int32_t dtype, uint64_t seed, uint64_t offset, int64_t n, int32_t ndim, const double* lo,
                                         const double* hi, void* const* out_cols, void* stream) {
  if (n <= 0 || ndim < 1 || ndim > PPSCI_MAX_IN || !lo || !hi || !out_cols) return fail("sample_uniform: bad arguments");
  SampleArgs a;
  memset(&a, 0, sizeof(a));
  for (int d = 0; d < ndim; ++d) {
    if (!out_cols[d]) return fail("sample_uniform: null output column");
    a.cols[d] = out_cols[d];
    a.lo[d] = lo[d];
    a.hi[d] = hi[d];
  }
  a.ndim = ndim;
  a.n = n;
  a.seed = seed;
  a.offset = offset;
  const unsigned blocks = (unsigned)((n + 255) / 256);
  return with_dtype(dtype, "sample_uniform", [&](auto zero) {
    PPSCI_LAUNCH(k_sample_uniform<decltype(zero)>, dim3(blocks), dim3(256), 0, stream, a);
    CK(cudaGetLastError());
    return 0;
  });
}

extern "C" int ppsci_b200_adam_step(int32_t dtype, void* params, const void* grads, void* exp_avg, void* exp_avg_sq,
                                    int64_t n, double lr, double beta1, double beta2, double eps, double weight_decay,
                                    int64_t step, double grad_scale, void* stream) {
  if (!params || !grads || !exp_avg || !exp_avg_sq || n <= 0 || step < 1) return fail("adam_step: bad arguments");
  const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
  const unsigned blocks = (unsigned)((n + 255) / 256);
  return with_dtype(dtype, "adam_step", [&](auto zero) {
    using T = decltype(zero);
    PPSCI_LAUNCH(k_adam<T>, dim3(blocks), dim3(256), 0, stream, (T*)params, (const T*)grads, (T*)exp_avg, (T*)exp_avg_sq,
                 (long long)n, lr, beta1, beta2, eps, weight_decay, bc1, bc2, grad_scale);
    CK(cudaGetLastError());
    return 0;
  });
}

extern "C" int ppsci_b200_adam_step_dev(int32_t dtype, void* params, void* grads, void* exp_avg, void* exp_avg_sq,
                                        int64_t n, const double* hyper_dev, double beta1, double beta2, double eps,
                                        double weight_decay, int32_t zero_grads, void* stream) {
  if (!params || !grads || !exp_avg || !exp_avg_sq || !hyper_dev || n <= 0) return fail("adam_step_dev: bad arguments");
  const unsigned blocks = (unsigned)((n + 255) / 256);
  return with_dtype(dtype, "adam_step_dev", [&](auto zero) {
    using T = decltype(zero);
    PPSCI_LAUNCH(k_adam_dev<T>, dim3(blocks), dim3(256), 0, stream, (T*)params, (T*)grads, (T*)exp_avg, (T*)exp_avg_sq,
                 (long long)n, hyper_dev, beta1, beta2, eps, weight_decay, (int)zero_grads);
    CK(cudaGetLastError());
    return 0;
  });
}

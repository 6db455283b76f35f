// Learner: one PPO + adversarial minibatch update as a fixed schedule of kernels on one stream.
//   forward : RMS(train) -> style / actor / critic / disc (+enc) MLPs (GEMM + fused bias/activation epilogues)
//   heads   : ppo_head / disc_head / enc_head kernels produce d(loss)/d(head outputs) + all train_result sums
//   backward: dX GEMMs with the ReLU / tanh' mask fused in the epilogue, dW GEMMs (split-K, RED accumulation
//             into the flat gradient arena), bias column sums, analytic gradient-penalty double backward
//   Adam    : one fused kernel over the flat arena (separate entry point so NCCL can sit in between)
// Reference: learning/ase_agent.py:159-308, amp_agent.py:266-390,442-479, common_agent.py:353-435.
#include <new>
#include <string.h>
#include "common.cuh"
#include "kernels.h"

namespace ase {

struct Layer { int64_t w, b; int out, in; };   // float offsets into the arena: weight [out,in], bias [out]
struct TensorDesc { int64_t off; int rows, cols; };

struct Net {
  int n_style = 0; Layer style[ASE_MAX_LAYERS]; Layer style_dense;
  int n_actor = 0; Layer actor[ASE_MAX_LAYERS];
  int n_critic = 0; Layer critic[ASE_MAX_LAYERS];
  Layer value, mu;
  int n_disc = 0; Layer disc[ASE_MAX_LAYERS]; Layer logit, enc;
  int n_tensors = 0; TensorDesc desc[64];
  int64_t arena = 0;
};

static int build_net(const AseLearnerConfig& c, Net& n) {
  ASE_CHECK_ARG(c.kind >= ASE_KIND_PPO && c.kind <= ASE_KIND_ASE, "learner: bad kind %d", c.kind);
  ASE_CHECK_ARG(c.n_units >= 1 && c.n_units <= ASE_MAX_LAYERS, "learner: n_units %d", c.n_units);
  ASE_CHECK_ARG(c.obs_dim > 0 && c.act_dim > 0 && c.batch > 1, "learner: dims");
  const bool ase = c.kind == ASE_KIND_ASE, amp = c.kind != ASE_KIND_PPO;
  if (amp) ASE_CHECK_ARG(c.n_disc_units >= 1 && c.n_disc_units <= ASE_MAX_LAYERS && c.amp_dim > 0 && c.amp_batch > 1 && c.amp_batch <= c.batch,
                         "learner: disc config");
  if (ase) ASE_CHECK_ARG(c.n_style_units >= 1 && c.n_style_units <= ASE_MAX_LAYERS && c.latent_dim > 0, "learner: style config");
  int64_t off = 0;
  auto add = [&](int rows, int cols) -> int64_t {
    const int64_t o = off;
    n.desc[n.n_tensors++] = {o, rows, cols};
    off = align_up(off + (int64_t)rows * cols, 32);
    return o;
  };
  auto add_layer = [&](int out, int in) -> Layer {
    Layer l; l.out = out; l.in = in; l.w = add(out, in); l.b = add(1, out); return l;
  };
  if (ase) {
    int in = c.latent_dim;
    for (int k = 0; k < c.n_style_units; ++k) { n.style[k] = add_layer(c.style_units[k], in); in = c.style_units[k]; }
    n.n_style = c.n_style_units;
    n.style_dense = add_layer(c.latent_dim, in);
  }
  const int in0 = c.obs_dim + (ase ? c.latent_dim : 0);
  int in = in0;
  for (int k = 0; k < c.n_units; ++k) { n.actor[k] = add_layer(c.units[k], in); in = c.units[k]; }
  n.n_actor = c.n_units;
  in = in0;
  for (int k = 0; k < c.n_units; ++k) { n.critic[k] = add_layer(c.units[k], in); in = c.units[k]; }
  n.n_critic = c.n_units;
  n.value = add_layer(1, c.units[c.n_units - 1]);
  n.mu = add_layer(c.act_dim, c.units[c.n_units - 1]);
  if (amp) {
    in = c.amp_dim;
    for (int k = 0; k < c.n_disc_units; ++k) { n.disc[k] = add_layer(c.disc_units[k], in); in = c.disc_units[k]; }
    n.n_disc = c.n_disc_units;
    n.logit = add_layer(1, in);
    if (ase) n.enc = add_layer(c.latent_dim, in);
  }
  n.arena = off;
  return ASE_OK;
}

}  // namespace ase

using namespace ase;

struct AseLearner {
  AseLearnerConfig cfg;
  Net net;
  bool ase, amp, has_div;
  int B, Ba, Ra;            // Ra = actor rows (2B when the diversity pass is batched in)
  int sms;                  // SMs of the device the learner was created on (split-K planning of the dW GEMMs)
  int in0, ldx, amp_ld, maxw;
  int64_t gsz;              // floats of each gradient scratch buffer G0, G1
  // workspace
  float *Xa, *Xc, *Zc, *S[ASE_MAX_LAYERS], *H[ASE_MAX_LAYERS], *MU, *C[ASE_MAX_LAYERS], *V;
  float *Xd, *D[ASE_MAX_LAYERS], *LOGIT, *E;
  float *dMU, *dV, *dLOGIT, *dE, *G0, *G1, *U[ASE_MAX_LAYERS], *Gx;
  // ReLU activity bits of the stored activations (1 bit per element, row stride = ceil(cols / 32) words): the backward masks
  uint32_t *Sb[ASE_MAX_LAYERS], *Hb[ASE_MAX_LAYERS], *Cb[ASE_MAX_LAYERS], *Db[ASE_MAX_LAYERS];
  double* acc;
  void *rms_obs_scratch, *rms_amp_scratch;
  void* tc_ws; int64_t tc_ws_bytes;
  // operand planes (tensor-core backends): one hi/lo pair per registered activation buffer + one pair per weight
  PlaneRegistry* reg;
  float* act_planes; int64_t act_plane_floats;     // carved region for activation planes
  float* w_planes; int64_t w_plane_floats;         // carved region for weight planes
  const float* reg_params;                         // parameter arena the weight entries currently point at
  void* reg_dev;                                   // FP16 format: device amax / scale slots of the registry
  bool weights_split;                              // FP16 format: the weight planes are current (one batched split per optimizer step)
};

namespace ase {

struct Carver {
  char* base; int64_t off = 0;
  explicit Carver(void* b) : base((char*)b) {}
  template <typename T> T* take(int64_t count) {
    T* p = base ? (T*)(base + off) : nullptr;
    off = align_up(off + count * (int64_t)sizeof(T), 256);
    return p;
  }
};

static inline int64_t bits_ld(int cols) { return (cols + 31) / 32; }

static int64_t tc_ws_need(const AseLearner& L) {
  if (L.cfg.gemm_backend < 1) return 0;
  int64_t need = 0;
  auto upd = [&](int64_t M, int64_t N, int64_t K) { need = imax64(need, gemm_tc_workspace_bytes((int)M, (int)N, (int)K)); };
  const AseLearnerConfig& c = L.cfg;
  int in = L.in0;
  for (int k = 0; k < c.n_units; ++k) { upd(L.Ra, c.units[k], in); upd(L.Ra, in, c.units[k]); upd(c.units[k], in, L.Ra); in = c.units[k]; }
  upd(L.Ra, c.act_dim, in); upd(L.Ra, in, c.act_dim); upd(c.act_dim, in, L.Ra);
  upd(L.B, 1, in); upd(L.B, in, 1); upd(1, in, L.B);
  if (L.ase) {
    in = c.latent_dim;
    for (int k = 0; k < c.n_style_units; ++k) { upd(L.Ra, c.style_units[k], in); upd(L.Ra, in, c.style_units[k]); upd(c.style_units[k], in, L.Ra); in = c.style_units[k]; }
    upd(L.Ra, c.latent_dim, in); upd(L.Ra, in, c.latent_dim); upd(c.latent_dim, in, L.Ra);
  }
  if (L.amp) {
    in = c.amp_dim;
    for (int k = 0; k < c.n_disc_units; ++k) { upd(3 * L.Ba, c.disc_units[k], in); upd(3 * L.Ba, in, c.disc_units[k]); upd(c.disc_units[k], in, 3 * L.Ba); in = c.disc_units[k]; }
    upd(3 * L.Ba, c.latent_dim > 0 ? c.latent_dim : 1, in); upd(3 * L.Ba, in, c.latent_dim > 0 ? c.latent_dim : 1);
    upd(c.latent_dim > 0 ? c.latent_dim : 1, in, 3 * L.Ba); upd(L.Ba, c.amp_dim, c.disc_units[0]); upd(c.disc_units[0], c.amp_dim, L.Ba);
  }
  return need;
}

// Every buffer with operand planes on the tensor-core backends, as f(fp32 base, rows, cols, is_weight): the activation buffers, then
// every tensor of the parameter arena at `params` (null: base pointers not needed).  carve() sizes the plane regions with it and
// register_planes() registers the same list.
template <typename F>
static void for_each_plane_buf(const AseLearner& L, const float* params, F&& f) {
  const AseLearnerConfig& c = L.cfg;
  const int64_t Ra = L.Ra, B = L.B, Ba = L.Ba;
  f(L.Xa, Ra, L.ldx, false);
  if (L.ase) { f(L.Xc, B, L.ldx, false); f(L.Zc, Ra, c.latent_dim, false); for (int k = 0; k < c.n_style_units; ++k) f(L.S[k], Ra, c.style_units[k], false); }
  for (int k = 0; k < c.n_units; ++k) { f(L.H[k], Ra, c.units[k], false); f(L.C[k], B, c.units[k], false); }
  if (L.amp) {
    f(L.Xd, 3 * Ba, L.amp_ld, false);
    for (int k = 0; k < c.n_disc_units; ++k) { f(L.D[k], 3 * Ba, c.disc_units[k], false); f(L.U[k], Ba, c.disc_units[k], false); }
    f(L.Gx, Ba, L.amp_ld, false);
  }
  f(L.G0, 1, L.gsz, false); f(L.G1, 1, L.gsz, false);
  // head gradients (written by the loss kernels): split once for their dW and dX consumers
  f(L.dMU, Ra, c.act_dim, false); f(L.dV, B, 1, false);
  if (L.amp) { f(L.dLOGIT, 3 * Ba, 1, false); if (L.ase) f(L.dE, Ba, c.latent_dim, false); }
  for (int i = 0; i < L.net.n_tensors; ++i) {
    const TensorDesc& d = L.net.desc[i];
    f(params ? params + d.off : nullptr, d.rows, d.cols, true);
  }
}

static void carve(AseLearner& L, void* ws, int64_t* total) {
  const AseLearnerConfig& c = L.cfg;
  Carver cv(ws);
  const int64_t Ra = L.Ra, B = L.B, Ba = L.Ba;
  L.Xa = cv.take<float>(Ra * L.ldx);
  L.Xc = L.ase ? cv.take<float>(B * L.ldx) : L.Xa;
  L.Zc = L.ase ? cv.take<float>(Ra * c.latent_dim) : nullptr;
  for (int k = 0; k < c.n_style_units && L.ase; ++k) L.S[k] = cv.take<float>(Ra * c.style_units[k]);
  for (int k = 0; k < c.n_units; ++k) L.H[k] = cv.take<float>(Ra * c.units[k]);
  L.MU = cv.take<float>(Ra * c.act_dim);
  for (int k = 0; k < c.n_units; ++k) L.C[k] = cv.take<float>(B * c.units[k]);
  L.V = cv.take<float>(B);
  L.dMU = cv.take<float>(Ra * c.act_dim);
  L.dV = cv.take<float>(B);
  if (L.amp) {
    L.Xd = cv.take<float>(3 * Ba * L.amp_ld);
    for (int k = 0; k < c.n_disc_units; ++k) L.D[k] = cv.take<float>(3 * Ba * c.disc_units[k]);
    L.LOGIT = cv.take<float>(3 * Ba);
    L.dLOGIT = cv.take<float>(3 * Ba);
    if (L.ase) { L.E = cv.take<float>(3 * Ba * c.latent_dim); L.dE = cv.take<float>(Ba * c.latent_dim); }
    for (int k = 0; k < c.n_disc_units; ++k) L.U[k] = cv.take<float>(Ba * c.disc_units[k]);
    L.Gx = cv.take<float>(Ba * L.amp_ld);
  }
  L.G0 = cv.take<float>(L.gsz);
  L.G1 = cv.take<float>(L.gsz);
  L.acc = cv.take<double>(ACC_COUNT);
  for (int k = 0; k < c.n_style_units && L.ase; ++k) L.Sb[k] = cv.take<uint32_t>(Ra * bits_ld(c.style_units[k]));
  for (int k = 0; k < c.n_units; ++k) { L.Hb[k] = cv.take<uint32_t>(Ra * bits_ld(c.units[k])); L.Cb[k] = cv.take<uint32_t>(B * bits_ld(c.units[k])); }
  for (int k = 0; k < c.n_disc_units && L.amp; ++k) L.Db[k] = cv.take<uint32_t>(3 * Ba * bits_ld(c.disc_units[k]));
  L.rms_obs_scratch = cv.take<char>(rms_scratch_bytes(c.obs_dim, L.B, 1));
  L.rms_amp_scratch = L.amp ? cv.take<char>(rms_scratch_bytes(c.amp_dim, L.Ba, 3)) : nullptr;
  L.tc_ws_bytes = tc_ws_need(L);
  cv.off = align_up(cv.off, 1024);
  L.tc_ws = L.tc_ws_bytes ? cv.take<char>(L.tc_ws_bytes) : nullptr;
  L.reg_dev = (c.gemm_backend == 2) ? cv.take<char>(PlaneRegistry::device_bytes()) : nullptr;
  if (c.gemm_backend >= 1) {
    // one hi/lo plane pair per plane-backed buffer (ld padded to 4), registered lazily in register_planes()
    int64_t floats[2] = {0, 0};
    for_each_plane_buf(L, nullptr, [&](const float*, int64_t rows, int64_t cols, bool weight) { floats[weight] += rows * align_up(cols, 4); });
    L.act_plane_floats = floats[0];
    L.act_planes = cv.take<float>(2 * floats[0]);
    L.w_plane_floats = floats[1];
    L.w_planes = cv.take<float>(2 * floats[1]);
  }
  *total = cv.off;
}

// (Re)build the plane registry: activation buffers once, weight entries whenever the parameter arena pointer changes.
static void register_planes(AseLearner& L, const float* params) {
  if (L.cfg.gemm_backend < 1) return;
  if (!L.reg) { L.reg = new PlaneRegistry; if (L.cfg.gemm_backend == 2) { L.reg->f16 = true; L.reg->attach_device(L.reg_dev); } }
  if (L.reg->n > 0 && L.reg_params == params) return;
  PlaneRegistry& R = *L.reg;
  R.n = 0;
  int64_t off[2] = {0, 0};
  for_each_plane_buf(L, params, [&](const float* base, int64_t rows, int64_t cols, bool weight) {
    float* hi = weight ? L.w_planes : L.act_planes;
    float* lo = hi + (weight ? L.w_plane_floats : L.act_plane_floats);
    const int64_t cap = rows * align_up(cols, 4);
    R.add(base, rows * cols, hi + off[weight], lo + off[weight], cap);
    off[weight] += cap;
  });
  L.reg_params = params;
  L.weights_split = false;
}

// FP16 format: (re)split all weight matrices in one launch if the parameters changed since the last split.
// (desc[] alternates weight, bias per layer: even entries are the GEMM operands)
static int split_weights(AseLearner& L, const float* params, cudaStream_t st) {
  if (!L.reg || !L.reg->f16 || L.weights_split) return ASE_OK;
  const float* src[TcPrepBatch::MAX]; int rows[TcPrepBatch::MAX], cols[TcPrepBatch::MAX]; int n = 0;
  for (int i = 0; i < L.net.n_tensors && n < TcPrepBatch::MAX; i += 2) {
    const TensorDesc& d = L.net.desc[i];
    src[n] = params + d.off; rows[n] = d.rows; cols[n] = d.cols; ++n;
  }
  int rc = L.reg->prep_weights(src, rows, cols, n, st);
  if (rc) return rc;
  L.weights_split = true;
  return ASE_OK;
}

static int init_learner(AseLearner& L, const AseLearnerConfig& cfg) {
  L.cfg = cfg;
  int rc = build_net(cfg, L.net);
  if (rc) return rc;
  L.ase = cfg.kind == ASE_KIND_ASE; L.amp = cfg.kind != ASE_KIND_PPO;
  L.has_div = L.ase && cfg.amp_diversity_bonus != 0.0f;
  L.B = cfg.batch; L.Ba = L.amp ? cfg.amp_batch : 0; L.Ra = L.has_div ? 2 * cfg.batch : cfg.batch;
  L.in0 = cfg.obs_dim + (L.ase ? cfg.latent_dim : 0);
  L.ldx = (int)align_up(L.in0, 4);
  L.amp_ld = L.amp ? (int)align_up(cfg.amp_dim, 4) : 0;
  int mw = max(cfg.act_dim, L.in0);
  for (int k = 0; k < cfg.n_units; ++k) mw = max(mw, cfg.units[k]);
  if (L.ase) { for (int k = 0; k < cfg.n_style_units; ++k) mw = max(mw, cfg.style_units[k]); mw = max(mw, cfg.latent_dim); }
  L.maxw = mw;
  L.gsz = (int64_t)L.Ra * mw;
  for (int k = 0; k < cfg.n_disc_units && L.amp; ++k) L.gsz = imax64(L.gsz, 3 * (int64_t)L.Ba * cfg.disc_units[k]);
  return ASE_OK;
}

// ---- small GEMM helpers -------------------------------------------------------------------------------
#define RC(x) do { int _rc = (x); if (_rc) return _rc; } while (0)

struct G {
  AseLearner& L; cudaStream_t st; const float* P; float* GR;   // P = parameter arena, GR = gradient arena
  PlaneRegistry* reg() const { return L.reg; }
  void inval(const float* p) const { if (L.reg) L.reg->invalidate(p); }
  AseGemmParams base() const {
    AseGemmParams p; memset(&p, 0, sizeof(p));
    p.alpha = 1.0f; p.backend = L.cfg.gemm_backend; p.workspace = L.tc_ws; p.workspace_bytes = L.tc_ws_bytes;
    return p;
  }
  // Y[M,N] (ldc) = act(X[M,K] (lda) . W^T + b),  W = layer weight [N,K].  bits: ReLU activity of Y for the backward pass;
  // planes_only: Y is consumed only as a GEMM operand / through bits (its fp32 store may be elided)
  int fwd(const float* X, int64_t lda, int M, const Layer& l, float* Y, int64_t ldc, int act, uint32_t* bits = nullptr, bool planes_only = false) const {
    AseGemmParams p = base();
    p.A = X; p.lda = lda; p.B = P + l.w; p.ldb = l.in; p.C = Y; p.ldc = ldc; p.M = M; p.N = l.out; p.K = l.in;
    p.bias = P + l.b; p.act = act;
    p.relu_bits_out = bits; p.ldrb = bits_ld(l.out); p.c_planes_only = planes_only ? 1 : 0;
    return gemm_dispatch(p, st, reg());
  }
  // dX[M,ncols] (ldc) = (dZ[M,l.out] . W[:, col0:col0+ncols]) (*) mask;  mask_bits (row stride bits_ld(ncols)) replaces mask_src on the
  // tensor-core backends for mask_mode 1
  int dx(const float* dZ, int64_t ldz, int M, const Layer& l, int col0, int ncols, float* dX, int64_t ldc,
         const float* mask_src, int64_t ldm, int mask_mode, float* colsum = nullptr, const uint32_t* mask_bits = nullptr, bool planes_only = false) const {
    AseGemmParams p = base();
    p.colsum_out = colsum;
    p.A = dZ; p.lda = ldz; p.B = P + l.w + col0; p.ldb = l.in; p.b_trans = 1; p.C = dX; p.ldc = ldc; p.M = M; p.N = ncols; p.K = l.out;
    p.mask_src = mask_src; p.ldm = ldm; p.mask_mode = mask_src ? mask_mode : 0;
    p.mask_bits = (mask_mode == 1) ? mask_bits : nullptr; p.ldmb = bits_ld(ncols); p.c_planes_only = planes_only ? 1 : 0;
    return gemm_dispatch(p, st, reg());
  }
  // dW[l.out, l.in] += dZ[M,l.out]^T . X[M,l.in]
  int dw(const float* dZ, int64_t ldz, int M, const Layer& l, const float* X, int64_t ldx) const {
    AseGemmParams p = base();
    p.A = dZ; p.lda = ldz; p.a_trans = 1; p.B = X; p.ldb = ldx; p.b_trans = 1; p.C = GR + l.w; p.ldc = l.in;
    p.M = l.out; p.N = l.in; p.K = M; p.accumulate = 1;
    if (L.cfg.gemm_backend >= 1) {      // tile and split-K plan of the tensor-core kernel
      p.split_k = gemm_tc_plan(p.M, p.N, p.K, 1, TC_SPLIT_AUTO, L.sms, L.cfg.gemm_backend == 2).splits;
      return gemm_dispatch(p, st, reg());
    }
    // SIMT: split-K so that 128 x 128 tiles x splits fill whole waves of the SMs; every extra split adds one RED pass over dW
    const int tiles = ceil_div(l.out, 128) * ceil_div(l.in, 128);
    const int slots = L.sms;
    const int smax = max(1, min(16, M / 1024));
    int best = 1; double best_cost = 1e30;
    for (int s = 1; s <= smax; ++s) {
      const double waves = (double)ceil_div((int64_t)tiles * s, slots);
      const double cost = waves / s * (1.0 + 0.03 * s);
      if (cost < best_cost - 1e-9) { best_cost = cost; best = s; }
    }
    p.split_k = best;
    return gemm_dispatch(p, st, reg());
  }
  int db(const float* dZ, int64_t ldz, int M, const Layer& l) const { return launch_colsum(dZ, ldz, M, l.out, GR + l.b, st); }
  // Y = X . W^T (no bias), masked: used by the gradient-penalty backward chain
  int nt_masked(const float* X, int64_t lda, int M, const Layer& l, float* Y, const float* mask_src, int64_t ldm, const uint32_t* mask_bits,
                float* colsum = nullptr) const {
    AseGemmParams p = base();
    p.A = X; p.lda = lda; p.B = P + l.w; p.ldb = l.in; p.C = Y; p.ldc = l.out; p.M = M; p.N = l.out; p.K = l.in;
    p.mask_src = mask_src; p.ldm = ldm; p.mask_mode = 1; p.mask_bits = mask_bits; p.ldmb = bits_ld(l.out);
    p.colsum_out = colsum; p.c_planes_only = 1;       // consumed by the next dW / masked GEMM only (the last one by its fused column sum)
    return gemm_dispatch(p, st, reg());
  }
};

// Backward through a ReLU MLP trunk.  On entry *cur holds dZ of the LAST layer (already masked), [M, out_last].
// acts[k] = stored post-activation outputs, X0 (ld ldx0) = trunk input.  On exit *cur holds dZ of layer 0.
static int trunk_backward(const G& g, const Layer* layers, int n, float* const* acts, uint32_t* const* bits, const float* X0, int64_t ldx0, int M,
                          float** cur, float** other, bool have_db = false) {
  for (int k = n - 1; k >= 0; --k) {
    const Layer& l = layers[k];
    const float* Xin = (k == 0) ? X0 : acts[k - 1];
    const int64_t ldin = (k == 0) ? ldx0 : layers[k - 1].out;
    RC(g.dw(*cur, l.out, M, l, Xin, ldin));
    if (!have_db) RC(g.db(*cur, l.out, M, l));
    if (k > 0) {
      // the dX GEMM that produces dZ of layer k-1 also column-sums it into that layer's bias gradient; dZ is consumed by GEMMs only
      RC(g.dx(*cur, l.out, M, l, 0, l.in, *other, l.in, acts[k - 1], layers[k - 1].out, 1, g.GR + layers[k - 1].b, bits[k - 1], true));
      have_db = true;
      float* t = *cur; *cur = *other; *other = t;
    }
  }
  return ASE_OK;
}

__global__ void __launch_bounds__(256)
relu_mask_inplace_kernel(float* __restrict__ g, const float* __restrict__ h, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (!(h[i] > 0.0f)) g[i] = 0.0f;
}

static int forward_actor_critic(const G& g, int rows_a, int rows_c) {
  AseLearner& L = g.L; const Net& n = L.net; const AseLearnerConfig& c = L.cfg;
  if (L.ase && rows_a > 0) {   // style branch: tanh(dense(relu-mlp(z))) written next to the normalised obs (ase_network_builder.py:305-324)
    const float* x = L.Zc; int64_t ld = c.latent_dim;
    for (int k = 0; k < n.n_style; ++k) { RC(g.fwd(x, ld, rows_a, n.style[k], L.S[k], n.style[k].out, 1, L.Sb[k], true)); x = L.S[k]; ld = n.style[k].out; }
    RC(g.fwd(x, ld, rows_a, n.style_dense, L.Xa + c.obs_dim, L.ldx, 2));
  }
  if (rows_a > 0) {
    const float* x = L.Xa; int64_t ld = L.ldx;
    for (int k = 0; k < n.n_actor; ++k) { RC(g.fwd(x, ld, rows_a, n.actor[k], L.H[k], n.actor[k].out, 1, L.Hb[k], true)); x = L.H[k]; ld = n.actor[k].out; }
    RC(g.fwd(x, ld, rows_a, n.mu, L.MU, c.act_dim, c.mu_activation == 2 ? 2 : 0));
  }
  if (rows_c > 0) {
    const float* x = L.Xc; int64_t ld = L.ldx;
    for (int k = 0; k < n.n_critic; ++k) { RC(g.fwd(x, ld, rows_c, n.critic[k], L.C[k], n.critic[k].out, 1, L.Cb[k], true)); x = L.C[k]; ld = n.critic[k].out; }
    RC(g.fwd(x, ld, rows_c, n.value, L.V, 1, 0));
  }
  return ASE_OK;
}

static int forward_disc(const G& g, int rows, int enc_rows) {
  AseLearner& L = g.L; const Net& n = L.net; const AseLearnerConfig& c = L.cfg;
  const float* x = L.Xd; int64_t ld = L.amp_ld;
  // (the top disc layer keeps its fp32 copy: gp_u_last / relu_mask_inplace read it)
  for (int k = 0; k < n.n_disc; ++k) { RC(g.fwd(x, ld, rows, n.disc[k], L.D[k], n.disc[k].out, 1, L.Db[k], k < n.n_disc - 1)); x = L.D[k]; ld = n.disc[k].out; }
  RC(g.fwd(x, ld, rows, n.logit, L.LOGIT, 1, 0));
  if (L.ase && enc_rows > 0) RC(g.fwd(x, ld, enc_rows, n.enc, L.E, c.latent_dim, 0));
  return ASE_OK;
}

}  // namespace ase

// =================================================================================================== C ABI
extern "C" int ase_learner_num_params(const AseLearnerConfig* cfg) {
  Net n; if (!cfg || build_net(*cfg, n)) return ASE_ERR_INVALID;
  return n.n_tensors;
}
extern "C" int ase_learner_param_desc(const AseLearnerConfig* cfg, int index, int64_t* offset, int* rows, int* cols) {
  Net n; if (!cfg || build_net(*cfg, n)) return ASE_ERR_INVALID;
  ASE_CHECK_ARG(index >= 0 && index < n.n_tensors, "param index %d out of range", index);
  if (offset) *offset = n.desc[index].off;
  if (rows) *rows = n.desc[index].rows;
  if (cols) *cols = n.desc[index].cols;
  return ASE_OK;
}
extern "C" int64_t ase_learner_arena_floats(const AseLearnerConfig* cfg) {
  Net n; if (!cfg || build_net(*cfg, n)) return ASE_ERR_INVALID;
  return n.arena;
}
extern "C" int64_t ase_learner_workspace_bytes(const AseLearnerConfig* cfg) {
  if (!cfg) return ASE_ERR_INVALID;
  AseLearner L; memset(&L, 0, sizeof(L));
  if (init_learner(L, *cfg)) return ASE_ERR_INVALID;
  int64_t total = 0;
  carve(L, nullptr, &total);
  return total;
}
extern "C" int ase_learner_create(const AseLearnerConfig* cfg, void* workspace, int64_t workspace_bytes, AseLearner** out) {
  ASE_CHECK_ARG(cfg && workspace && out, "ase_learner_create: null pointer");
  ASE_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 1023) == 0, "ase_learner_create: workspace must be 1024-byte aligned");
  AseLearner* L = new (std::nothrow) AseLearner;
  ASE_CHECK_ARG(L != nullptr, "ase_learner_create: out of host memory");
  memset(L, 0, sizeof(*L));
  int rc = init_learner(*L, *cfg);
  if (rc) { delete L; return rc; }
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&L->sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || L->sms <= 0) {
    cudaGetLastError();
    L->sms = NUM_SMS;
  }
  int64_t total = 0;
  carve(*L, workspace, &total);
  if (total > workspace_bytes) {
    set_error("ase_learner_create: workspace %lld bytes < required %lld", (long long)workspace_bytes, (long long)total);
    delete L; return ASE_ERR_WORKSPACE;
  }
  // padding columns of the input buffers must be (and stay) zero
  cudaError_t e = cudaMemset(workspace, 0, (size_t)total);
  if (e != cudaSuccess) { set_error("cudaMemset(workspace): %s", cudaGetErrorString(e)); delete L; return ASE_ERR_CUDA; }
  *out = L;
  return ASE_OK;
}
extern "C" void ase_learner_destroy(AseLearner* l) { if (l) { delete l->reg; delete l; } }

extern "C" int ase_learner_params_changed(AseLearner* l) {
  ASE_CHECK_ARG(l != nullptr, "ase_learner_params_changed: null learner");
  if (l->reg && l->reg_params) l->reg->invalidate_range(l->reg_params, l->reg_params + l->net.arena);
  l->weights_split = false;
  if (l->reg) l->reg->forget_sites();     // new weights: the FP16 format recalibrates every scale exactly on the next call
  return ASE_OK;
}

extern "C" int ase_learner_plane_status(AseLearner* l, int* flags, void* stream) {
  ASE_CHECK_ARG(l && flags, "ase_learner_plane_status: null argument");
  *flags = 0;
  if (!l->reg || !l->reg->f16) return ASE_OK;
  unsigned f = 0;
  ASE_CUDA_OK(cudaMemcpyAsync(&f, l->reg->flag, sizeof(f), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  ASE_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
  *flags = (int)f;
  return ASE_OK;
}

namespace ase {
__global__ void plane_flag_to_kernel(const unsigned* __restrict__ flag, float* __restrict__ dst, int count, int64_t stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) dst[(int64_t)i * stride] = flag ? (float)(*flag) : 0.0f;
}
}  // namespace ase
extern "C" int ase_learner_plane_flag_to(AseLearner* l, float* dst, int count, int64_t stride, void* stream) {
  ASE_CHECK_ARG(l && dst && count >= 0, "ase_learner_plane_flag_to: bad argument");
  if (count == 0) return ASE_OK;
  const unsigned* f = (l->reg && l->reg->f16) ? l->reg->flag : nullptr;
  plane_flag_to_kernel<<<ceil_div(count, 128), 128, 0, (cudaStream_t)stream>>>(f, dst, count, stride);
  ASE_LAUNCH_OK();
  return ASE_OK;
}
extern "C" int ase_learner_plane_flag_clear(AseLearner* l, void* stream) {
  ASE_CHECK_ARG(l != nullptr, "ase_learner_plane_flag_clear: null learner");
  if (l->reg && l->reg->f16) ASE_CUDA_OK(cudaMemsetAsync(l->reg->flag, 0, sizeof(unsigned), (cudaStream_t)stream));
  return ASE_OK;
}

extern "C" int ase_learner_calc_gradients(AseLearner* lp, const AseLearnerState* s, const AseMinibatch* mb, const AseTrainResult* out,
                                          void* stream) {
  ASE_CHECK_ARG(lp && s && mb && out, "calc_gradients: null argument");
  AseLearner& L = *lp; const Net& n = L.net; const AseLearnerConfig& c = L.cfg;
  cudaStream_t st = (cudaStream_t)stream;
  ASE_CHECK_ARG(s->params && s->grads && s->logstd && s->obs_mean && s->obs_var && s->obs_count, "calc_gradients: state pointers");
  ASE_CHECK_ARG(mb->obs && mb->actions && mb->old_logp_actions && mb->advantages && mb->old_mu && mb->old_sigma && mb->returns,
                "calc_gradients: minibatch pointers");
  if (L.amp) ASE_CHECK_ARG(mb->amp_obs && mb->amp_obs_replay && mb->amp_obs_demo && s->amp_mean && s->amp_var && s->amp_count,
                           "calc_gradients: AMP pointers");
  if (L.ase) ASE_CHECK_ARG(mb->ase_latents && (!L.has_div || mb->new_latents), "calc_gradients: ASE latents");
  ASE_CHECK_ARG(out->scalars, "calc_gradients: scalars output");
  const int B = L.B, Ba = L.Ba, Ra = L.Ra, Z = c.latent_dim, A = c.act_dim;
  register_planes(L, s->params);
  if (L.reg) { RC(L.reg->begin_call(st, 0)); RC(split_weights(L, s->params, st)); }
  G g{L, st, s->params, s->grads};

  ASE_CUDA_OK(cudaMemsetAsync(L.acc, 0, ACC_COUNT * sizeof(double), st));
  ASE_CUDA_OK(cudaMemsetAsync(s->grads, 0, (size_t)n.arena * sizeof(float), st));
  RC(launch_mask_sum(L.amp ? mb->rand_action_mask : nullptr, B, L.acc, st));

  // ---- input normalisation (RunningMeanStd, train mode updates the stats first) -------------------------
  {
    RmsBatchList bl; bl.x[0] = mb->obs; bl.ld[0] = c.obs_dim; bl.rows = B;
    float *mf, *sf;
    RC(rms_update_batches(bl, 1, c.obs_dim, s->obs_mean, s->obs_var, s->obs_count, c.rms_eps, mb->update_rms, L.rms_obs_scratch, &mf, &sf, st));
    RmsDst d = {}; d.y[0] = L.Xa; d.ld[0] = L.ldx;
    if (L.has_div) { d.y[1] = L.Xa + (int64_t)B * L.ldx; d.ld[1] = L.ldx; }
    if (L.ase) { d.y[2] = L.Xc; d.ld[2] = L.ldx; }
    // the normalise pass also writes the operand planes of the network inputs (the style / latent columns follow below);
    // FP16 format: with the static scale -- the values are clamped to +-5
    PlaneRegistry* R = L.reg;
    PlaneBuf* pa = R ? R->declare(L.Xa, L.ldx, Ra, L.in0) : nullptr;
    PlaneBuf* pc = (R && L.ase) ? R->declare(L.Xc, L.ldx, B, L.in0) : nullptr;
    d.half = (R && R->f16) ? 1 : 0; d.pscale = PlaneRegistry::STATIC_SCALE;
    if (pa) { d.hi[0] = R->plane(pa, false, 0, 0); d.lo[0] = R->plane(pa, true, 0, 0); d.ldp[0] = pa->ldp; if (L.has_div) { d.hi[1] = R->plane(pa, false, B, 0); d.lo[1] = R->plane(pa, true, B, 0); d.ldp[1] = pa->ldp; } }
    if (pc) { d.hi[2] = R->plane(pc, false, 0, 0); d.lo[2] = R->plane(pc, true, 0, 0); d.ldp[2] = pc->ldp; }
    RC(rms_normalize(mb->obs, c.obs_dim, B, c.obs_dim, mf, sf, 0, d, st));
    if (!pa) g.inval(L.Xa);
    if (!pc) g.inval(L.Xc);
  }
  if (L.ase) {
    PlaneRegistry* R = L.reg;
    const int half = (R && R->f16) ? 1 : 0;
    unsigned* fl = R ? R->flag : nullptr;
    PlaneBuf* pc = R ? R->find(L.Xc) : nullptr;
    if (pc && !pc->valid) pc = nullptr;
    RC(copy_cols(mb->ase_latents, Z, B, Z, L.Xc + c.obs_dim, L.ldx, st, pc ? R->plane(pc, false, 0, c.obs_dim) : nullptr, pc ? R->plane(pc, true, 0, c.obs_dim) : nullptr,
                 pc ? pc->ldp : 0, half, PlaneRegistry::STATIC_SCALE, fl));
    if (!pc) g.inval(L.Xc);
    PlaneBuf* pz = R ? R->declare(L.Zc, Z, Ra, Z) : nullptr;
    RC(copy_cols(mb->ase_latents, Z, B, Z, L.Zc, Z, st, pz ? R->plane(pz, false, 0, 0) : nullptr, pz ? R->plane(pz, true, 0, 0) : nullptr, pz ? pz->ldp : 0, half,
                 PlaneRegistry::STATIC_SCALE, fl));
    if (L.has_div) RC(copy_cols(mb->new_latents, Z, B, Z, L.Zc + (int64_t)B * Z, Z, st, pz ? R->plane(pz, false, B, 0) : nullptr, pz ? R->plane(pz, true, B, 0) : nullptr,
                                pz ? pz->ldp : 0, half, PlaneRegistry::STATIC_SCALE, fl));
    if (!pz) g.inval(L.Zc);
  }
  if (L.amp) {
    // three sequential updates: agent, replay, demo -- each batch normalised with the stats after ITS update
    RmsBatchList bl; bl.x[0] = mb->amp_obs; bl.x[1] = mb->amp_obs_replay; bl.x[2] = mb->amp_obs_demo;
    bl.ld[0] = bl.ld[1] = bl.ld[2] = c.amp_dim; bl.rows = Ba;
    float *mf, *sf;
    RC(rms_update_batches(bl, 3, c.amp_dim, s->amp_mean, s->amp_var, s->amp_count, c.rms_eps, mb->update_rms, L.rms_amp_scratch, &mf, &sf, st));
    PlaneRegistry* R = L.reg;
    PlaneBuf* pd = R ? R->declare(L.Xd, L.amp_ld, 3 * Ba, c.amp_dim) : nullptr;
    for (int b = 0; b < 3; ++b) {
      RmsDst d = {}; d.y[0] = L.Xd + (int64_t)b * Ba * L.amp_ld; d.ld[0] = L.amp_ld;
      d.half = (R && R->f16) ? 1 : 0; d.pscale = PlaneRegistry::STATIC_SCALE;
      if (pd) { d.hi[0] = R->plane(pd, false, (int64_t)b * Ba, 0); d.lo[0] = R->plane(pd, true, (int64_t)b * Ba, 0); d.ldp[0] = pd->ldp; }
      RC(rms_normalize(bl.x[b], c.amp_dim, Ba, c.amp_dim, mf + (int64_t)b * c.amp_dim, sf + (int64_t)b * c.amp_dim, 0, d, st));
    }
    if (!pd) g.inval(L.Xd);
  }

  // ---- forward ------------------------------------------------------------------------------------------
  RC(forward_actor_critic(g, Ra, B));
  if (L.amp) RC(forward_disc(g, 3 * Ba, Ba));

  // ---- heads: losses + d(loss)/d(head outputs) ----------------------------------------------------------
  {
    PpoHeadArgs a; memset(&a, 0, sizeof(a));
    a.mu = L.MU; a.ld_mu = A; a.values = L.V; a.actions = mb->actions; a.old_logp = mb->old_logp_actions; a.adv = mb->advantages;
    a.old_mu = mb->old_mu; a.old_sigma = mb->old_sigma; a.returns = mb->returns; a.mask = L.amp ? mb->rand_action_mask : nullptr;
    a.logstd = s->logstd; a.z = mb->ase_latents; a.z2 = mb->new_latents; a.Z = Z; a.B = B; a.A = A; a.has_div = L.has_div ? 1 : 0;
    a.e_clip = c.e_clip; a.critic_coef = c.critic_coef; a.bounds_coef = c.bounds_loss_coef; a.div_bonus = c.amp_diversity_bonus;
    a.div_tar = c.amp_diversity_tar; a.dmu = L.dMU; a.dv = L.dV; a.acc = L.acc; a.mu_tanh = c.mu_activation == 2 ? 1 : 0;
    RC(launch_ppo_head(a, st));
    g.inval(L.dMU); g.inval(L.dV);
  }
  if (L.amp) { RC(launch_disc_head(L.LOGIT, Ba, c.disc_coef, L.dLOGIT, L.acc, out->disc_agent_logit, out->disc_demo_logit, st)); g.inval(L.dLOGIT); }
  if (L.ase) { RC(launch_enc_head(L.E, Ba, Z, mb->ase_latents, c.enc_coef, L.dE, nullptr, L.acc, st)); g.inval(L.dE); }

  // ---- backward: actor ----------------------------------------------------------------------------------
  float *cur = L.G0, *oth = L.G1;
  {
    const Layer& last = n.actor[n.n_actor - 1];
    RC(g.dw(L.dMU, A, Ra, n.mu, L.H[n.n_actor - 1], last.out));
    RC(g.db(L.dMU, A, Ra, n.mu));
    RC(g.dx(L.dMU, A, Ra, n.mu, 0, last.out, cur, last.out, L.H[n.n_actor - 1], last.out, 1, s->grads + last.b, L.Hb[n.n_actor - 1], true));
    RC(trunk_backward(g, n.actor, n.n_actor, L.H, L.Hb, L.Xa, L.ldx, Ra, &cur, &oth, true));
    if (L.ase) {
      // d(style pre-activation) = (dZ0 . W0[:, obs:obs+Z]) * (1 - style^2)
      const Layer& l0 = n.actor[0];
      RC(g.dx(cur, l0.out, Ra, l0, c.obs_dim, Z, oth, Z, L.Xa + c.obs_dim, L.ldx, 2, s->grads + n.style_dense.b, nullptr, true));
      { float* t = cur; cur = oth; oth = t; }
      const Layer& sd = n.style_dense; const Layer& sl = n.style[n.n_style - 1];
      RC(g.dw(cur, Z, Ra, sd, L.S[n.n_style - 1], sl.out));
      RC(g.dx(cur, Z, Ra, sd, 0, sl.out, oth, sl.out, L.S[n.n_style - 1], sl.out, 1, s->grads + sl.b, L.Sb[n.n_style - 1], true));
      { float* t = cur; cur = oth; oth = t; }
      RC(trunk_backward(g, n.style, n.n_style, L.S, L.Sb, L.Zc, Z, Ra, &cur, &oth, true));
    }
  }
  // ---- backward: critic ---------------------------------------------------------------------------------
  {
    const Layer& last = n.critic[n.n_critic - 1];
    RC(g.dw(L.dV, 1, B, n.value, L.C[n.n_critic - 1], last.out));
    RC(g.db(L.dV, 1, B, n.value));
    RC(g.dx(L.dV, 1, B, n.value, 0, last.out, cur, last.out, L.C[n.n_critic - 1], last.out, 1, s->grads + last.b, L.Cb[n.n_critic - 1], true));
    RC(trunk_backward(g, n.critic, n.n_critic, L.C, L.Cb, L.Xc, L.ldx, B, &cur, &oth, true));
  }
  // ---- backward: discriminator (+ encoder through the shared trunk) -------------------------------------
  if (L.amp) {
    const int nd = n.n_disc; const Layer& last = n.disc[nd - 1];
    const int R3 = 3 * Ba;
    RC(g.dw(L.dLOGIT, 1, R3, n.logit, L.D[nd - 1], last.out));
    RC(g.db(L.dLOGIT, 1, R3, n.logit));
    if (L.ase) {
      RC(g.dw(L.dE, Z, Ba, n.enc, L.D[nd - 1], last.out));
      RC(g.db(L.dE, Z, Ba, n.enc));
      RC(g.dx(L.dLOGIT, 1, R3, n.logit, 0, last.out, cur, last.out, nullptr, 0, 0));
      {   // rows [0,Ba): += dE . W_enc  (enc head sits on the agent rows of the shared trunk)
        AseGemmParams p = g.base();
        p.A = L.dE; p.lda = Z; p.B = s->params + n.enc.w; p.ldb = last.out; p.b_trans = 1; p.C = cur; p.ldc = last.out;
        p.M = Ba; p.N = last.out; p.K = Z; p.accumulate = 1; p.split_k = 1;
        RC(gemm_dispatch(p, st, g.reg()));
      }
      const int64_t tot = (int64_t)R3 * last.out;
      relu_mask_inplace_kernel<<<(int)imin64((tot + 255) / 256, NUM_SMS * 16), 256, 0, st>>>(cur, L.D[nd - 1], tot);
      ASE_LAUNCH_OK();
      g.inval(cur);
    } else {
      RC(g.dx(L.dLOGIT, 1, R3, n.logit, 0, last.out, cur, last.out, L.D[nd - 1], last.out, 1, s->grads + last.b, L.Db[nd - 1], true));
    }
    RC(trunk_backward(g, n.disc, nd, L.D, L.Db, L.Xd, L.amp_ld, R3, &cur, &oth, !L.ase));

    // ---- gradient penalty on the demo rows: analytic double backward (amp_agent.py:454-459) -------------
    const int64_t demo = (int64_t)2 * Ba;
    const float* wl = s->params + n.logit.w;
    RC(launch_gp_u_last(L.D[nd - 1] + demo * last.out, last.out, Ba, last.out, wl, L.U[nd - 1], st));
    g.inval(L.U[nd - 1]);
    for (int k = nd - 1; k >= 1; --k)   // U_{k-1} = D_{k-1} (*) (U_k . W_k)
      RC(g.dx(L.U[k], n.disc[k].out, Ba, n.disc[k], 0, n.disc[k].in, L.U[k - 1], n.disc[k].in,
              L.D[k - 1] + demo * n.disc[k - 1].out, n.disc[k - 1].out, 1, nullptr, L.Db[k - 1] + demo * bits_ld(n.disc[k - 1].out), true));
    RC(g.dx(L.U[0], n.disc[0].out, Ba, n.disc[0], 0, c.amp_dim, L.Gx, L.amp_ld, nullptr, 0, 0));     // G = U_0 . W_0
    // (padding columns of Gx are zero: they are never written)
    RC(launch_gp_scale(L.Gx, (int64_t)Ba * L.amp_ld, c.disc_coef * c.disc_grad_penalty * 2.0f / (float)Ba, L.acc, st));
    g.inval(L.Gx);
    RC(g.dw(L.U[0], n.disc[0].out, Ba, n.disc[0], L.Gx, L.amp_ld));                                   // dW_0 += U_0^T Gbar
    // (the last masked GEMM of the chain column-sums its output into d w_logit: d w_logit += sum_rows Ubar_last)
    RC(g.nt_masked(L.Gx, L.amp_ld, Ba, n.disc[0], cur, L.D[0] + demo * n.disc[0].out, n.disc[0].out, L.Db[0] + demo * bits_ld(n.disc[0].out),
                   nd == 1 ? s->grads + n.logit.w : nullptr));                                       // Ubar_0
    for (int k = 1; k < nd; ++k) {
      RC(g.dw(L.U[k], n.disc[k].out, Ba, n.disc[k], cur, n.disc[k].in));                              // dW_k += U_k^T Ubar_{k-1}
      RC(g.nt_masked(cur, n.disc[k].in, Ba, n.disc[k], oth, L.D[k] + demo * n.disc[k].out, n.disc[k].out, L.Db[k] + demo * bits_ld(n.disc[k].out),
                     k == nd - 1 ? s->grads + n.logit.w : nullptr));
      { float* t = cur; cur = oth; oth = t; }
    }

    // ---- logit-weight regulariser + weight decay (amp_agent.py:448-466) ---------------------------------
    for (int k = 0; k < nd; ++k)
      RC(launch_weight_reg(s->params + n.disc[k].w, s->grads + n.disc[k].w, (int64_t)n.disc[k].out * n.disc[k].in,
                           c.disc_coef * c.disc_weight_decay * 2.0f, L.acc, ACC_WDISC2, -1, st));
    RC(launch_weight_reg(wl, s->grads + n.logit.w, last.out, c.disc_coef * (c.disc_logit_reg + c.disc_weight_decay) * 2.0f, L.acc,
                         ACC_WLOGIT2, ACC_WDISC2, st));
  }

  // ---- train_result ---------------------------------------------------------------------------------------
  {
    FinalizeArgs f; memset(&f, 0, sizeof(f));
    f.acc = L.acc; f.out = out->scalars; f.logstd = s->logstd; f.kind = c.kind; f.B = B; f.Ba = Ba; f.A = A;
    f.critic_coef = c.critic_coef; f.entropy_coef = c.entropy_coef; f.bounds_coef = c.bounds_loss_coef; f.disc_coef = c.disc_coef;
    f.logit_reg = c.disc_logit_reg; f.gp_coef = c.disc_grad_penalty; f.weight_decay = c.disc_weight_decay; f.enc_coef = c.enc_coef;
    f.div_bonus = L.has_div ? c.amp_diversity_bonus : 0.0f;
    RC(launch_finalize(f, st));
  }
  if (out->mu) ASE_CUDA_OK(cudaMemcpyAsync(out->mu, L.MU, (size_t)B * A * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (out->values) ASE_CUDA_OK(cudaMemcpyAsync(out->values, L.V, (size_t)B * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return ASE_OK;
}

extern "C" int ase_learner_adam_step(AseLearner* lp, const AseLearnerState* s, int64_t step, float grad_scale, void* stream) {
  ASE_CHECK_ARG(lp && s && s->params && s->grads && s->exp_avg && s->exp_avg_sq && step >= 1, "adam_step: bad argument");
  const AseLearnerConfig& c = lp->cfg;
  if (lp->reg) lp->reg->invalidate_range(s->params, s->params + lp->net.arena);   // weight planes are stale after the update
  lp->weights_split = false;
  return launch_adam(s->params, s->grads, s->exp_avg, s->exp_avg_sq, lp->net.arena, grad_scale, c.beta1, c.beta2, c.lr, c.adam_eps, step,
                     (cudaStream_t)stream);
}

// allreduce (sum over the ranks, in place in every rank's peer-visible gradient arena) + Adam in ONE kernel over NVLink peer memory
// (peer.cu): replaces ase_grad_allreduce + ase_learner_adam_step.  s->grads must be the arena inside the rank's peer buffer (ase_peer_grads);
// params / exp_avg / exp_avg_sq must be readable 16 bytes at a time up to the arena rounded up to 4 floats.
extern "C" int ase_learner_peer_adam_step(AseLearner* lp, AsePeer* peer, const AseLearnerState* s, int64_t step, float grad_scale, void* stream) {
  ASE_CHECK_ARG(lp && peer && s && s->params && s->grads && s->exp_avg && s->exp_avg_sq && step >= 1, "peer_adam_step: bad argument");
  const AseLearnerConfig& c = lp->cfg;
  if (lp->reg) lp->reg->invalidate_range(s->params, s->params + lp->net.arena);   // weight planes are stale after the update
  lp->weights_split = false;
  return launch_peer_adam(peer, s->params, s->exp_avg, s->exp_avg_sq, grad_scale, c.beta1, c.beta2, c.lr, c.adam_eps, step,
                          lp->reg ? lp->reg->flag : nullptr, (cudaStream_t)stream);
}

extern "C" int ase_learner_eval_actor_critic(AseLearner* lp, const AseLearnerState* s, const float* obs, const float* latents, int rows,
                                             float* mu, float* value_normed, void* stream) {
  ASE_CHECK_ARG(lp && s && obs, "eval_actor_critic: null argument");
  AseLearner& L = *lp; const AseLearnerConfig& c = L.cfg;
  ASE_CHECK_ARG(rows > 0 && rows <= L.B, "eval_actor_critic: rows %d > minibatch %d", rows, L.B);
  ASE_CHECK_ARG(!L.ase || latents, "eval_actor_critic: latents required");
  cudaStream_t st = (cudaStream_t)stream;
  register_planes(L, s->params);
  if (L.reg) { RC(L.reg->begin_call(st, 600)); RC(split_weights(L, s->params, st)); }
  G g{L, st, s->params, s->grads};
  RC(rms_apply(obs, c.obs_dim, rows, c.obs_dim, s->obs_mean, s->obs_var, c.rms_eps, 0, L.Xa, L.ldx, st));
  g.inval(L.Xa); g.inval(L.Xc); g.inval(L.Zc);
  if (L.ase) {
    RC(copy_cols(L.Xa, L.ldx, rows, c.obs_dim, L.Xc, L.ldx, st));
    RC(copy_cols(latents, c.latent_dim, rows, c.latent_dim, L.Xc + c.obs_dim, L.ldx, st));
    RC(copy_cols(latents, c.latent_dim, rows, c.latent_dim, L.Zc, c.latent_dim, st));
  }
  RC(forward_actor_critic(g, mu ? rows : 0, value_normed ? rows : 0));
  if (mu) ASE_CUDA_OK(cudaMemcpyAsync(mu, L.MU, (size_t)rows * c.act_dim * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (value_normed) ASE_CUDA_OK(cudaMemcpyAsync(value_normed, L.V, (size_t)rows * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return ASE_OK;
}

extern "C" int ase_learner_eval_disc_enc(AseLearner* lp, const AseLearnerState* s, const float* amp_obs, int rows, float* disc_logits,
                                         float* enc_pred, void* stream) {
  ASE_CHECK_ARG(lp && s && amp_obs, "eval_disc_enc: null argument");
  AseLearner& L = *lp; const AseLearnerConfig& c = L.cfg;
  ASE_CHECK_ARG(L.amp, "eval_disc_enc: learner has no discriminator");
  ASE_CHECK_ARG(rows > 0 && rows <= 3 * L.Ba, "eval_disc_enc: rows %d > 3*amp_batch %d", rows, 3 * L.Ba);
  ASE_CHECK_ARG(!enc_pred || L.ase, "eval_disc_enc: enc_pred needs an ASE learner");
  cudaStream_t st = (cudaStream_t)stream;
  register_planes(L, s->params);
  if (L.reg) { RC(L.reg->begin_call(st, 800)); RC(split_weights(L, s->params, st)); }
  G g{L, st, s->params, s->grads};
  RC(rms_apply(amp_obs, c.amp_dim, rows, c.amp_dim, s->amp_mean, s->amp_var, c.rms_eps, 0, L.Xd, L.amp_ld, st));
  g.inval(L.Xd);
  RC(forward_disc(g, rows, enc_pred ? rows : 0));
  if (disc_logits) ASE_CUDA_OK(cudaMemcpyAsync(disc_logits, L.LOGIT, (size_t)rows * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (enc_pred) RC(launch_enc_head(L.E, rows, c.latent_dim, nullptr, 0.0f, nullptr, enc_pred, nullptr, st));
  return ASE_OK;
}

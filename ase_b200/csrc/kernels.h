// Internal (non-ABI) declarations shared by the .cu files of libase_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/ase_b200.h"

namespace ase {

// ------------------------------------------------------------------ RunningMeanStd
struct RmsBatchList { const float* x[3]; int64_t ld[3]; int rows; };
// optional operand planes per destination: fp32 words holding TF32 values, or (half != 0) halfs of y * pscale
struct RmsDst { float* y[3]; int64_t ld[3]; void* hi[3]; void* lo[3]; int64_t ldp[3]; int half; float pscale; };
int64_t rms_scratch_bytes(int cols, int rows, int nbatch);
int rms_update_batches(const RmsBatchList& bl, int nbatch, int cols, double* mean, double* var, double* count, float eps,
                       int update, void* scratch, float** meanf_out, float** stdf_out, cudaStream_t st);
int rms_normalize(const float* x, int64_t ldx, int rows, int cols, const float* meanf, const float* stdf, int unnorm,
                  const RmsDst& dst, cudaStream_t st);
int rms_apply(const float* x, int64_t ldx, int rows, int cols, const double* mean, const double* var, float eps, int unnorm,
              float* y, int64_t ldy, cudaStream_t st);
int copy_cols(const float* x, int64_t ldx, int rows, int cols, float* y, int64_t ldy, cudaStream_t st, void* hi = nullptr, void* lo = nullptr,
              int64_t ldp = 0, int half = 0, float pscale = 1.0f, unsigned* flag = nullptr);

// ------------------------------------------------------------------ GEMM backends
int gemm_simt(const AseGemmParams& p, cudaStream_t st);
// TF32 hi/lo operand planes kept next to registered fp32 buffers (gemm_tc.cu)
struct PlaneBuf {
  const float* base; int64_t capacity;          // fp32 buffer (floats)
  float* hi; float* lo; int64_t plane_capacity; // planes (floats each; the FP16 format stores halfs in the same space)
  int64_t ld; int rows, cols; int64_t ldp;      // geometry declared by the last full writer / first reader
  bool valid;
  // FP16 format
  const float* scale_ptr;                       // device [scale, 1/scale] the current planes were written with
  int amax_site;                                // site whose amax slot holds max |x| of the current fp32 contents (tracked by the GEMM that wrote them), -1 = unknown
  bool is_static;                               // planes written with the registry's static scale by a bounded non-GEMM writer
  bool fp32_stale;                              // the last producer skipped the fp32 store (c_planes_only): only the planes are current
  void drop() { valid = false; amax_site = -1; is_static = false; fp32_stale = false; }   // the buffer has no current planes
};
// FP16 format (backend 2): every tensor is multiplied by a power of two before the hi/lo split.  Scales live in device memory,
// one slot per SITE = (GEMM index within the top-level call, operand A / B / output C): the static kernel schedule of the learner
// puts the same logical tensor at the same site every call.  The first time a site is used its scale comes from an exact max pass
// (or from the max the producing GEMM tracked); afterwards the scale predicted from the previous call's max is used, which lets the
// producing GEMM's epilogue write the planes itself.  The predicted scale puts the previous call's max into [2^8, 2^9).  Overflow: a
// scaled value above 60000, i.e. growth by more than x117 .. x234 (never flagged at x64, always at x512), is flagged by the writer in
// the same call.  Underflow: a scaled max below 2^-6, i.e. shrinking by more than 2^14 .. 2^15 (never flagged at 2^-13, always at
// 2^-16), is flagged by tc_site_update_kernel at the start of the NEXT call.  Either raises a sticky device flag
// (ase_learner_plane_status), never a silent wrong result (tests/test_gpu_learner_shapes.py pins both edges).
// One tensor for the FP16 split pass: src[rows, cols] (ld) into zero-padded planes [rows_p, ldp]; its max slot, its site's
// [scale, 1/scale] and an optional copy of the scale the planes are written with.
struct TcPrepItem {
  const float* src; int64_t ld; int rows, cols, rows_p, ldp;
  void* hi; void* lo;
  unsigned* amax; float* scale; float* scale_copy;
};
template <int N> struct TcPrepList { static constexpr int MAX = N; TcPrepItem item[N]; };
using TcPrepBatch = TcPrepList<40>;   // the learner's weight tensors, split in one launch
struct PlaneRegistry {
  static constexpr int MAX = 160;
  static constexpr int WEIGHT_SITE0 = 960;      // fixed scale sites of the weight tensors (prep_weights)
  static constexpr int SITES = 1024;
  static constexpr float STATIC_SCALE = 64.0f;  // bounded writers (normalised observations clamp at 5, tanh outputs, unit latents)
  PlaneBuf b[MAX]; int n = 0;
  bool f16 = false;
  unsigned* amax = nullptr;       // [SITES] max |x| seen at the site during the current call (uint bits)
  float* scale = nullptr;         // [SITES][2] scale / inverse
  float* static_scale = nullptr;  // [2]
  float* bscale = nullptr;        // [MAX][2] copy of the scale a registered buffer's planes were SPLIT with by a prep pass: unlike the
                                  // site slots (re-predicted at every begin_call) it stays put, so weight planes survive across calls
  unsigned* flag = nullptr;       // [1] sticky: bit 0 overflow (|x * scale| > 60000), bit 1 underflow (max * scale < 2^-6, or a zero scale met data)
  bool known[SITES], touched[SITES];
  int call_base = 0, gemm_index = 0;
  static int64_t device_bytes() { return (int64_t)SITES * 4 + (int64_t)SITES * 8 + (int64_t)MAX * 8 + 64; }
  void attach_device(void* mem) {
    amax = (unsigned*)mem; scale = (float*)((char*)mem + SITES * 4); bscale = scale + 2 * SITES; static_scale = bscale + 2 * MAX; flag = (unsigned*)(static_scale + 2);
    for (int i = 0; i < SITES; ++i) known[i] = touched[i] = false;
  }
  int prep_weights(const float* const* src, const int* rows, const int* cols, int count, cudaStream_t st);
  int begin_call(cudaStream_t st, int base);    // start of one stream-ordered sequence of GEMMs (calc_gradients / eval_*)
  int site(int which) const { const int s = call_base + 3 * gemm_index + which; return s < SITES ? s : -1; }
  bool reset_pending = false;     // forget_sites(): the device slots are cleared at the next begin_call (stream-ordered)
  void forget_sites() { for (int i = 0; i < SITES; ++i) known[i] = touched[i] = false; reset_pending = true; }
  PlaneBuf* find(const float* p);
  // a non-GEMM kernel is about to write the whole buffer [rows, cols] (ld) INCLUDING its planes: returns the entry (valid) or null.
  // FP16 format: only bounded writers may call this (the planes get the static scale).
  PlaneBuf* declare(const float* base, int64_t ld, int rows, int cols);
  void* plane(const PlaneBuf* x, bool lo, int64_t r0, int64_t c0) const;   // element (r0, c0) of a plane, in either format
  void add(const float* base, int64_t capacity, float* hi, float* lo, int64_t plane_capacity);
  void invalidate(const float* p);
  void invalidate_range(const float* lo_, const float* hi_);
};
int gemm_tc(const AseGemmParams& p, cudaStream_t st, PlaneRegistry* reg = nullptr);   // wgmma 3xTF32 (backend 1) / 3xFP16-scaled (backend 2) (gemm_tc.cu)
int64_t gemm_tc_workspace_bytes(int M, int N, int K);
// tile plan of a tensor-core GEMM (gemm_tc.cu): tile height, tile width, K splits as launched
struct TcPlan { int bm, bn, splits; };
constexpr int TC_SPLIT_AUTO = -1;   // split_k for gemm_tc_plan: let the launch-time model choose the splits
TcPlan gemm_tc_plan(int M, int N, int K, int accumulate, int split_k, int sms, bool f16);
int gemm_dispatch(const AseGemmParams& p, cudaStream_t st, PlaneRegistry* reg = nullptr);    // checks p and runs the backend it names

// ------------------------------------------------------------------ loss-side accumulators (doubles)
enum {
  ACC_MSUM = 0, ACC_ALOSS, ACC_CLOSS, ACC_BLOSS, ACC_CLIPPED, ACC_KL, ACC_DIV,
  ACC_BCE_AGENT, ACC_BCE_DEMO, ACC_ACC_AGENT, ACC_ACC_DEMO, ACC_LOGIT_AGENT, ACC_LOGIT_DEMO,
  ACC_GP, ACC_WLOGIT2, ACC_WDISC2, ACC_ENC, ACC_COUNT = 24
};

struct PpoHeadArgs {
  const float* mu; int64_t ld_mu;      // [B or 2B, A]; rows B.. hold the diversity pass
  const float* values;                 // [B]
  const float* actions; const float* old_logp; const float* adv; const float* old_mu; const float* old_sigma;
  const float* returns; const float* mask; const float* logstd;
  const float* z; const float* z2; int Z;
  int B, A;
  int has_div;
  int mu_tanh;                         // mu = tanh(raw): gradients are taken to the pre-activation
  float e_clip, critic_coef, bounds_coef, div_bonus, div_tar;
  float* dmu;                          // same layout as mu
  float* dv;                           // [B]
  double* acc;
};

struct FinalizeArgs {
  const double* acc; float* out; const float* logstd;
  int kind, B, Ba, A;
  float critic_coef, entropy_coef, bounds_coef, disc_coef, logit_reg, gp_coef, weight_decay, enc_coef, div_bonus;
};

int launch_mask_sum(const float* mask, int rows, double* acc, cudaStream_t st);
int launch_ppo_head(const PpoHeadArgs& a, cudaStream_t st);
int launch_disc_head(const float* logit, int Ba, float disc_coef, float* dlogit, double* acc, float* out_agent, float* out_demo, cudaStream_t st);
int launch_enc_head(const float* e, int rows, int Z, const float* z, float enc_coef, float* de, float* enc_pred, double* acc, cudaStream_t st);
int launch_gp_u_last(const float* h, int64_t ldh, int rows, int cols, const float* w, float* u, cudaStream_t st);
int launch_gp_scale(float* g, int64_t total, float scale, double* acc, cudaStream_t st);
int launch_colsum(const float* dz, int64_t ld, int rows, int cols, float* db, cudaStream_t st);
int launch_weight_reg(const float* w, float* g, int64_t n, float coef, double* acc, int idx, int idx2, cudaStream_t st);
int launch_finalize(const FinalizeArgs& f, cudaStream_t st);
int launch_adam(float* p, const float* g, float* m, float* v, int64_t n, float grad_scale, float b1, float b2, float lr, float eps,
                int64_t step, cudaStream_t st);
// the fp32 constants torch.optim.Adam ends up with (evaluated in doubles from the decimal hyper-parameters, then rounded)
struct AdamConsts { float b1, b2, omb1, omb2, step_size, bc2_sqrt, eps; };
AdamConsts adam_consts(float b1, float b2, float lr, float eps, int64_t step);
}  // namespace ase
// allreduce + Adam over NVLink peer memory (peer.cu)
struct AsePeer;
namespace ase {
int launch_peer_adam(AsePeer* pr, float* p, float* m, float* v, float grad_scale, float b1, float b2, float lr, float eps, int64_t step,
                     unsigned* status, cudaStream_t st);

}  // namespace ase

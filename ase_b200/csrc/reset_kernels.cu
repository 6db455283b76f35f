// Episode resets of HumanoidAMP / HumanoidAMPGetup on the device, mask driven (no index lists, no host reads):
//   ase_amp_state_init   <- HumanoidAMP._reset_actors + _reset_default / _reset_ref_state_init / _reset_hybrid_state_init / _set_env_state
//                           (env/tasks/humanoid_amp.py:141-201,238-246), HumanoidAMPGetup._reset_actors + _reset_recovery_episode /
//                           _reset_fall_episode (env/tasks/humanoid_amp_getup.py:78-116), the zeroing of Humanoid._reset_env_tensors
//                           (env/tasks/humanoid.py:150-167)
//   ase_amp_history_init <- HumanoidAMP._init_amp_obs + _init_amp_obs_default / _init_amp_obs_ref (humanoid_amp.py:203-236), getup override
//                           (humanoid_amp_getup.py:123-129)
//   ase_recovery_step    <- HumanoidAMPGetup._update_recovery_count (humanoid_amp_getup.py:36-40,131-134) + its _compute_reset (:136-142).
//                           Run after the env's reset rule; decrementing at post-physics instead of pre_physics_step is equivalent because
//                           nothing reads the counter in between.
// Draws: Philox (philox.cuh) or injected outcomes; the layout is in include/ase_b200.h.
#include "common.cuh"
#include "kernels.h"
#include "motion_common.cuh"
#include "philox.cuh"

namespace ase {

struct StateInitArgs {
  AseStateInitParams p;
  const float* cdf;
  int M;
};

// one CTA of MOT_THREADS per env; unflagged envs exit at once (after writing kind NONE)
__global__ void __launch_bounds__(MOT_THREADS)
amp_state_init_kernel(MotionTablesDev mt, StateInitArgs a) {
  const AseStateInitParams& p = a.p;
  const int e = blockIdx.x;
  if (!p.reset_mask[e]) {
    if (threadIdx.x == 0) p.kind_out[e] = ASE_INIT_NONE;
    return;                                        // CTA-uniform
  }
  __shared__ int s_kind, s_row;
  __shared__ float s_blend;
  __shared__ int64_t s_f[2];
  if (threadIdx.x == 0) {
    bool rec, fall, hyb;
    float phase = 0.0f, uclip = 0.0f;
    int id = 0, row = 0;
    if (p.rng) {
      const uint4 w = philox_u4(p.rng, (uint32_t)p.stream_id, (uint32_t)e, 0u);
      rec = u01_open(w.x) < p.recovery_prob;
      fall = u01_open(w.y) < p.fall_prob;
      hyb = u01_open(w.z) < p.hybrid_prob;
      phase = u01_open(w.w);
      uclip = u01_open(philox_u4(p.rng, (uint32_t)p.stream_id, (uint32_t)e, 1u).x);
      row = (int)(philox_u4(p.rng, (uint32_t)p.stream_id + 1u, (uint32_t)e, 0xFFFFFFFEu).x % (uint32_t)max(1, p.num_fall_states));
    } else {
      rec = p.recovery_in && p.recovery_in[e] != 0;
      fall = p.fall_in && p.fall_in[e] != 0;
      hyb = p.hybrid_in && p.hybrid_in[e] != 0;
      if (p.phase_in) phase = p.phase_in[e];
      if (p.motion_id_in) id = p.motion_id_in[e];
      if (p.fall_row_in) row = p.fall_row_in[e];
    }
    rec = rec && p.terminate_buf[e] != 0;          // only a terminated episode may continue as a recovery episode
    int kind;
    if (rec) kind = ASE_INIT_RECOVERY;
    else if (fall) kind = ASE_INIT_FALL;
    else if (p.state_init == ASE_STATE_INIT_DEFAULT || (p.state_init == ASE_STATE_INIT_HYBRID && !hyb)) kind = ASE_INIT_DEFAULT;
    else kind = ASE_INIT_REF;
    float time = 0.0f;
    if (kind == ASE_INIT_REF) {
      if (p.rng) {                                 // inverse CDF: the first m with u < cdf[m] (cdf[M-1] == 1 > u)
        int lo = 0, hi = a.M - 1;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (uclip < a.cdf[mid]) hi = mid; else lo = mid + 1; }
        id = lo;
      }
      if (p.state_init != ASE_STATE_INIT_START) time = __fmul_rn(phase, mt.lengths[id]);     // sample_time: phase * motion_len
      int64_t f0l, f1l; float blend;
      frame_blend(mt, id, time, f0l, f1l, blend);
      s_f[0] = f0l; s_f[1] = f1l; s_blend = blend;
      p.motion_id_out[e] = id; p.motion_time_out[e] = time;
    }
    s_kind = kind; s_row = row;
    p.kind_out[e] = (uint8_t)kind;
    if (p.recovery_counter) p.recovery_counter[e] = (kind == ASE_INIT_RECOVERY || kind == ASE_INIT_FALL) ? p.recovery_steps : 0;
    p.progress[e] = 0; p.reset_buf[e] = 0; p.terminate_buf[e] = 0;
  }
  __syncthreads();
  const int kind = s_kind;
  if (kind == ASE_INIT_RECOVERY) return;
  const int D = mt.D;
  float* root = p.root_states + (int64_t)e * p.root_stride;
  float* dpos = p.dof_pos + (int64_t)e * p.dof_pos_stride;
  float* dvel = p.dof_vel + (int64_t)e * p.dof_vel_stride;
  if (kind != ASE_INIT_REF) {                      // copy rows: the env's initial state or a fall-bank row
    const bool df = kind == ASE_INIT_DEFAULT;
    const int64_t r = df ? e : s_row;
    const float* sr = (df ? p.init_root_states : p.fall_root_states) + r * 13;
    const float* sp = (df ? p.init_dof_pos : p.fall_dof_pos) + r * D;
    const float* sv = (df ? p.init_dof_vel : p.fall_dof_vel) + r * D;
    for (int i = threadIdx.x; i < 13 + 2 * D; i += MOT_THREADS) {
      if (i < 13) root[i] = sr[i];
      else if (i < 13 + D) dpos[(int64_t)(i - 13) * p.dof_pos_elem_stride] = sp[i - 13];
      else dvel[(int64_t)(i - 13 - D) * p.dof_vel_elem_stride] = sv[i - 13 - D];
    }
    return;
  }
  // reference state: get_motion_state (motion_lib.py:123-172) into _set_env_state's slots (humanoid_amp.py:238-246)
  const int64_t f0l = s_f[0], f1l = s_f[1];
  const float blend = s_blend;
  for (int item = threadIdx.x; item < 1 + mt.nj + D; item += MOT_THREADS) {
    if (item == 0) {
      const float* p0 = mt.gts + f0l * mt.J * 3; const float* p1 = mt.gts + f1l * mt.J * 3;
      for (int c = 0; c < 3; ++c) root[c] = (1.0f - blend) * p0[c] + blend * p1[c];
      const Quat rr = slerp(load_quat(mt.grs + f0l * mt.J * 4), load_quat(mt.grs + f1l * mt.J * 4), blend);
      root[3] = rr.x; root[4] = rr.y; root[5] = rr.z; root[6] = rr.w;
      for (int c = 0; c < 3; ++c) { root[7 + c] = mt.grvs[f0l * 3 + c]; root[10 + c] = mt.gravs[f0l * 3 + c]; }
    } else if (item < 1 + mt.nj) {
      const int j = item - 1;
      float dp[3];
      const int sz = joint_dof(mt, j, f0l, f1l, blend, dp);
      for (int c = 0; c < sz; ++c) dpos[(int64_t)(mt.dof_offsets[j] + c) * p.dof_pos_elem_stride] = dp[c];
    } else {
      const int d = item - 1 - mt.nj;
      dvel[(int64_t)d * p.dof_vel_elem_stride] = mt.dvs[f0l * D + d];
    }
  }
}

// grid (N, S - 1): CTA (e, k - 1) writes slot k of env e
__global__ void __launch_bounds__(MOT_THREADS)
amp_history_init_kernel(MotionTablesDev mt, const uint8_t* __restrict__ kind, const int32_t* __restrict__ ids, const float* __restrict__ times,
                        float sim_dt, int local_root_obs, int root_height_obs, float* __restrict__ amp_obs, int S, int F) {
  const int e = blockIdx.x, k = blockIdx.y + 1;
  const int kd = kind[e];
  float* row = amp_obs + (int64_t)e * S * F;
  if (kd == ASE_INIT_DEFAULT || kd == ASE_INIT_FALL) {
    for (int i = threadIdx.x; i < F; i += MOT_THREADS) row[(int64_t)k * F + i] = row[i];
  } else if (kd == ASE_INIT_REF) {
    // _init_amp_obs_ref: motion_times + (-dt * (arange + 1)), each product and sum rounded on its own
    const float t = __fadd_rn(times[e], __fmul_rn(-sim_dt, (float)k));
    amp_obs_frame(mt, ids[e], t, local_root_obs, root_height_obs, row + (int64_t)k * F);
  }
}

// one thread per env
__global__ void __launch_bounds__(256)
recovery_step_kernel(int32_t* __restrict__ counter, uint8_t* __restrict__ reset_buf, uint8_t* __restrict__ terminate_buf, int n) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int32_t c = max(counter[e] - 1, 0);
  counter[e] = c;
  if (c > 0) { reset_buf[e] = 0; terminate_buf[e] = 0; }
}

}  // namespace ase

using namespace ase;

extern "C" int ase_amp_state_init(const AseMotionLib* m, const float* motion_cdf, int num_motions, const AseStateInitParams* p, void* stream) {
  ASE_CHECK_ARG(p, "ase_amp_state_init: null params");
  MotionTablesDev t;
  int rc = fill_tables(m, t);
  if (rc) return rc;
  ASE_CHECK_ARG(p->state_init >= ASE_STATE_INIT_DEFAULT && p->state_init <= ASE_STATE_INIT_HYBRID, "ase_amp_state_init: unknown state_init %d",
                p->state_init);
  ASE_CHECK_ARG(p->reset_mask && p->root_states && p->dof_pos && p->dof_vel && p->progress && p->reset_buf && p->terminate_buf && p->kind_out &&
                p->motion_id_out && p->motion_time_out, "ase_amp_state_init: null pointer");
  ASE_CHECK_ARG(p->root_stride >= 13 && p->dof_pos_stride > 0 && p->dof_vel_stride > 0 && p->dof_pos_elem_stride > 0 && p->dof_vel_elem_stride > 0,
                "ase_amp_state_init: bad strides");
  const bool needs_default = p->state_init == ASE_STATE_INIT_DEFAULT || p->state_init == ASE_STATE_INIT_HYBRID;
  ASE_CHECK_ARG(!needs_default || (p->init_root_states && p->init_dof_pos && p->init_dof_vel), "ase_amp_state_init: initial state required");
  const bool may_fall = p->rng ? p->fall_prob > 0.0f : p->fall_in != nullptr;
  ASE_CHECK_ARG(!may_fall || (p->fall_root_states && p->fall_dof_pos && p->fall_dof_vel && p->num_fall_states > 0),
                "ase_amp_state_init: fall-state bank required");
  ASE_CHECK_ARG(p->recovery_steps >= 0, "ase_amp_state_init: recovery_steps < 0");
  if (p->state_init != ASE_STATE_INIT_DEFAULT) {
    ASE_CHECK_ARG(p->rng ? (motion_cdf && num_motions >= 1) : (p->motion_id_in && p->phase_in), "ase_amp_state_init: clip draws required");
  }
  ASE_CHECK_ARG(p->rng || !may_fall || p->fall_row_in, "ase_amp_state_init: fall_row_in required");
  if (p->num_envs <= 0) return ASE_OK;
  StateInitArgs a{*p, motion_cdf, num_motions};
  amp_state_init_kernel<<<p->num_envs, MOT_THREADS, 0, (cudaStream_t)stream>>>(t, a);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_amp_history_init(const AseMotionLib* m, const uint8_t* kind, const int32_t* motion_ids, const float* motion_times, int num_envs,
                                    float sim_dt, int local_root_obs, int root_height_obs, float* amp_obs, int hist_steps, void* stream) {
  MotionTablesDev t;
  int rc = fill_tables(m, t);
  if (rc) return rc;
  ASE_CHECK_ARG(kind && motion_ids && motion_times && amp_obs && hist_steps >= 1, "ase_amp_history_init: bad argument");
  if (num_envs <= 0 || hist_steps == 1) return ASE_OK;
  const int F = 13 + 6 * t.nj + t.D + 3 * t.nk;
  amp_history_init_kernel<<<dim3((unsigned)num_envs, (unsigned)(hist_steps - 1)), MOT_THREADS, 0, (cudaStream_t)stream>>>(
      t, kind, motion_ids, motion_times, sim_dt, local_root_obs, root_height_obs, amp_obs, hist_steps, F);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_recovery_step(int32_t* recovery_counter, uint8_t* reset_buf, uint8_t* terminate_buf, int num_envs, void* stream) {
  ASE_CHECK_ARG(recovery_counter && reset_buf && terminate_buf, "ase_recovery_step: null pointer");
  if (num_envs <= 0) return ASE_OK;
  recovery_step_kernel<<<ceil_div(num_envs, 256), 256, 0, (cudaStream_t)stream>>>(recovery_counter, reset_buf, terminate_buf, num_envs);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

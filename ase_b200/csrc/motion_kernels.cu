// Motion library on the device: (clip id, time) -> interpolated reference state -> demo AMP observations, fused.
//   ase_motion_state  <- MotionLib.get_motion_state           (utils/motion_lib.py:123-172,263-272,296-324)
//   ase_amp_obs_demo  <- HumanoidAMP.build_amp_obs_demo        (env/tasks/humanoid_amp.py:85-101) = get_motion_state on
//                        `steps` times going back by sim_dt + build_amp_observations (humanoid_amp.py:282-316)
// One CTA per (sample, step); gathers from the flat frame tables (~10 MB for the 87 shipped clips: L2 resident).
// The per-frame device code is in motion_common.cuh (shared with the reference-state resets of reset_kernels.cu).
#include "common.cuh"
#include "kernels.h"
#include "motion_common.cuh"

namespace ase {

// one CTA per (sample, step): out[(sample*steps + step) * F .. +F)
__global__ void __launch_bounds__(MOT_THREADS)
amp_obs_demo_kernel(MotionTablesDev mt, const int32_t* __restrict__ ids, const float* __restrict__ t0, int steps, float sim_dt,
                    int local_root_obs, int root_height_obs, float* __restrict__ out, int F) {
  const int sample = blockIdx.x / steps, step = blockIdx.x - sample * steps;
  const float time = t0[sample] - sim_dt * (float)step;
  amp_obs_frame(mt, ids[sample], time, local_root_obs, root_height_obs, out + (int64_t)blockIdx.x * F);
}

// one CTA per sample: the 7 tensors get_motion_state returns
__global__ void __launch_bounds__(MOT_THREADS)
motion_state_kernel(MotionTablesDev mt, const int32_t* __restrict__ ids, const float* __restrict__ times, float* __restrict__ root_pos,
                    float* __restrict__ root_rot, float* __restrict__ dof_pos, float* __restrict__ root_vel, float* __restrict__ root_ang_vel,
                    float* __restrict__ dof_vel, float* __restrict__ key_pos) {
  const int n = blockIdx.x, id = ids[n];
  int64_t f0l, f1l; float blend;
  frame_blend(mt, id, times[n], f0l, f1l, blend);
  for (int item = threadIdx.x; item < 1 + mt.nj + mt.D + mt.nk; item += MOT_THREADS) {
    if (item == 0) {
      const float* p0 = mt.gts + f0l * mt.J * 3; const float* p1 = mt.gts + f1l * mt.J * 3;
      for (int c = 0; c < 3; ++c) root_pos[n * 3 + c] = (1.0f - blend) * p0[c] + blend * p1[c];
      const Quat rr = slerp(load_quat(mt.grs + f0l * mt.J * 4), load_quat(mt.grs + f1l * mt.J * 4), blend);
      root_rot[n * 4 + 0] = rr.x; root_rot[n * 4 + 1] = rr.y; root_rot[n * 4 + 2] = rr.z; root_rot[n * 4 + 3] = rr.w;
      for (int c = 0; c < 3; ++c) { root_vel[n * 3 + c] = mt.grvs[f0l * 3 + c]; root_ang_vel[n * 3 + c] = mt.gravs[f0l * 3 + c]; }
    } else if (item < 1 + mt.nj) {
      const int j = item - 1;
      float dp[3];
      const int sz = joint_dof(mt, j, f0l, f1l, blend, dp);
      for (int c = 0; c < sz; ++c) dof_pos[(int64_t)n * mt.D + mt.dof_offsets[j] + c] = dp[c];
    } else if (item < 1 + mt.nj + mt.D) {
      const int d = item - 1 - mt.nj;
      dof_vel[(int64_t)n * mt.D + d] = mt.dvs[f0l * mt.D + d];
    } else {
      const int k = item - 1 - mt.nj - mt.D, body = mt.key_body_ids[k];
      const float* p0 = mt.gts + (f0l * mt.J + body) * 3; const float* p1 = mt.gts + (f1l * mt.J + body) * 3;
      for (int c = 0; c < 3; ++c) key_pos[((int64_t)n * mt.nk + k) * 3 + c] = (1.0f - blend) * p0[c] + blend * p1[c];
    }
  }
}

}  // namespace ase

using namespace ase;

extern "C" int ase_motion_state(const AseMotionLib* m, const int32_t* motion_ids, const float* motion_times, int n, float* root_pos,
                                float* root_rot, float* dof_pos, float* root_vel, float* root_ang_vel, float* dof_vel, float* key_pos,
                                void* stream) {
  MotionTablesDev t;
  int rc = fill_tables(m, t);
  if (rc) return rc;
  ASE_CHECK_ARG(motion_ids && motion_times && root_pos && root_rot && dof_pos && root_vel && root_ang_vel && dof_vel && key_pos,
                "ase_motion_state: null pointer");
  if (n <= 0) return ASE_OK;
  motion_state_kernel<<<n, MOT_THREADS, 0, (cudaStream_t)stream>>>(t, motion_ids, motion_times, root_pos, root_rot, dof_pos, root_vel,
                                                                    root_ang_vel, dof_vel, key_pos);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_amp_obs_demo(const AseMotionLib* m, const int32_t* motion_ids, const float* motion_times0, int n, float sim_dt,
                                int num_steps, int local_root_obs, int root_height_obs, float* amp_obs, void* stream) {
  MotionTablesDev t;
  int rc = fill_tables(m, t);
  if (rc) return rc;
  ASE_CHECK_ARG(motion_ids && motion_times0 && amp_obs && num_steps >= 1, "ase_amp_obs_demo: bad argument");
  if (n <= 0) return ASE_OK;
  const int F = 13 + 6 * t.nj + t.D + 3 * t.nk;
  amp_obs_demo_kernel<<<n * num_steps, MOT_THREADS, 0, (cudaStream_t)stream>>>(t, motion_ids, motion_times0, num_steps, sim_dt,
                                                                                 local_root_obs, root_height_obs, amp_obs, F);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

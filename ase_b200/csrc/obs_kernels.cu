// Per-env observation build (HBM-bound, coalesced through shared memory).
//   ase_obs_build      <- compute_humanoid_observations_max  (env/tasks/humanoid.py:591-635)
//   ase_amp_obs_build  <- build_amp_observations + dof_to_obs + history shift
//                         (env/tasks/humanoid_amp.py:248-316, env/tasks/humanoid.py:522-552)
// Algorithmic bytes (DESIGN.md): obs = (J*13 + obs_dim)*4 per env; amp = (13+2*dofs+3*keys + steps*step_dim)*4
// (+ (steps-1)*step_dim*4 re-read for the in-place shift).
#include "common.cuh"

namespace ase {

constexpr int OBS_ENVS_PER_BLOCK = 8;
constexpr int OBS_THREADS = 256;
constexpr int OBS_MAX_BODIES = 24;

__global__ void __launch_bounds__(OBS_THREADS)
obs_build_kernel(AseObsBuildParams p, int obs_dim) {
  extern __shared__ float smem[];
  const int J = p.num_bodies;
  const int in_per_env = J * 13;
  float* s_in = smem;                                      // [E][J*13]
  float* s_out = s_in + OBS_ENVS_PER_BLOCK * in_per_env;   // [E][obs_dim]
  float* s_hq = s_out + OBS_ENVS_PER_BLOCK * obs_dim;      // [E][4]
  const int count = p.env_ids ? p.num_env_ids : p.num_envs;
  const int e0 = blockIdx.x * OBS_ENVS_PER_BLOCK;
  const int ne = min(OBS_ENVS_PER_BLOCK, count - e0);

  // coalesced gather of the rigid-body rows (13 contiguous floats per body)
  for (int idx = threadIdx.x; idx < ne * in_per_env; idx += OBS_THREADS) {
    const int e = idx / in_per_env, r = idx - e * in_per_env;
    const int b = r / 13, c = r - b * 13;
    const int env = p.env_ids ? p.env_ids[e0 + e] : (e0 + e);
    s_in[idx] = p.body_state[(int64_t)env * p.env_stride + (int64_t)b * p.body_stride + c];
  }
  __syncthreads();
  if (threadIdx.x < ne) {
    const float* r = s_in + threadIdx.x * in_per_env;      // body 0 = root
    const Quat q = {r[3], r[4], r[5], r[6]};
    const Quat hq = calc_heading_quat_inv(q);
    float* o = s_hq + threadIdx.x * 4;
    o[0] = hq.x; o[1] = hq.y; o[2] = hq.z; o[3] = hq.w;
  }
  __syncthreads();
  const int off_p = 1, off_r = 1 + (J - 1) * 3, off_v = off_r + J * 6, off_w = off_v + J * 3;
  for (int item = threadIdx.x; item < ne * J; item += OBS_THREADS) {
    const int e = item / J, b = item - e * J;
    const float* root = s_in + e * in_per_env;
    const float* s = root + b * 13;
    float* o = s_out + e * obs_dim;
    const Quat hq = {s_hq[e * 4 + 0], s_hq[e * 4 + 1], s_hq[e * 4 + 2], s_hq[e * 4 + 3]};
    const Quat qb = {s[3], s[4], s[5], s[6]};
    if (b == 0) {
      o[0] = p.root_height_obs ? root[2] : 0.0f;
    } else {
      const Vec3 d = {s[0] - root[0], s[1] - root[1], s[2] - root[2]};
      const Vec3 lp = quat_rotate(hq, d);
      o[off_p + (b - 1) * 3 + 0] = lp.x; o[off_p + (b - 1) * 3 + 1] = lp.y; o[off_p + (b - 1) * 3 + 2] = lp.z;
    }
    // humanoid.py:622-624: with local_root_obs the root slot holds tan_norm of the GLOBAL root rotation
    const Quat qr = (b == 0 && p.local_root_obs) ? qb : quat_mul(hq, qb);
    quat_to_tan_norm(qr, o + off_r + b * 6);
    const Vec3 v = {s[7], s[8], s[9]}, w = {s[10], s[11], s[12]};
    const Vec3 lv = quat_rotate(hq, v), lw = quat_rotate(hq, w);
    o[off_v + b * 3 + 0] = lv.x; o[off_v + b * 3 + 1] = lv.y; o[off_v + b * 3 + 2] = lv.z;
    o[off_w + b * 3 + 0] = lw.x; o[off_w + b * 3 + 1] = lw.y; o[off_w + b * 3 + 2] = lw.z;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < ne * obs_dim; idx += OBS_THREADS) {
    const int e = idx / obs_dim, c = idx - e * obs_dim;
    const int env = p.env_ids ? p.env_ids[e0 + e] : (e0 + e);
    if (p.env_mask && !p.env_mask[env]) continue;          // masked reset path: only the flagged envs are rewritten
    p.obs[(int64_t)env * p.obs_ld + c] = s_out[idx];
  }
}

// ------------------------------------------------------------------------------------------------
constexpr int AMP_THREADS = 128;
constexpr int AMP_MAX_JOINTS = 32;
constexpr int AMP_MAX_KEYS = 16;

struct AmpTables {
  int dof_offsets[AMP_MAX_JOINTS + 1];
  int key_body_ids[AMP_MAX_KEYS];
};

// utils/torch_utils.py:68-91 exp_map_to_quat
__device__ __forceinline__ Quat exp_map_to_quat(float ex, float ey, float ez) {
  const float angle_raw = sqrtf(ex * ex + ey * ey + ez * ez);
  const float angle_n = atan2f(sinf(angle_raw), cosf(angle_raw));   // normalize_angle
  const bool ok = fabsf(angle_n) > 1e-5f;
  Vec3 axis = {0.0f, 0.0f, 1.0f};
  float angle = 0.0f;
  if (ok) { axis.x = ex / angle_raw; axis.y = ey / angle_raw; axis.z = ez / angle_raw; angle = angle_n; }
  return quat_from_angle_axis(angle, axis);
}

// one block per env: shift the 10-frame history by one slot and write the newest frame at slot 0
__global__ void __launch_bounds__(AMP_THREADS)
amp_obs_build_kernel(AseAmpObsBuildParams p, AmpTables tb) {
  extern __shared__ float smem[];
  const int F = p.step_dim, S = p.hist_steps;
  float* s_hist = smem;            // [(S-1)*F] old slots 0..S-2
  float* s_new = s_hist + (S - 1) * F;   // [F]
  __shared__ float s_hq[4];
  const int env = p.env_ids ? p.env_ids[blockIdx.x] : blockIdx.x;
  if (p.env_mask && !p.env_mask[env]) return;              // masked reset path (block-uniform)
  float* buf = p.amp_obs + (int64_t)env * S * F;
  if (p.shift_history) {
    for (int i = threadIdx.x; i < (S - 1) * F; i += AMP_THREADS) s_hist[i] = buf[i];
  }
  const float* root = p.body_state + (int64_t)env * p.env_stride;
  if (threadIdx.x == 0) {
    const Quat q = {root[3], root[4], root[5], root[6]};
    const Quat hq = calc_heading_quat_inv(q);
    s_hq[0] = hq.x; s_hq[1] = hq.y; s_hq[2] = hq.z; s_hq[3] = hq.w;
  }
  __syncthreads();
  const Quat hq = {s_hq[0], s_hq[1], s_hq[2], s_hq[3]};
  const int nj = p.num_joints, nd = p.num_dofs, nk = p.num_key_bodies;
  const int off_dof = 13, off_vel = 13 + 6 * nj, off_key = off_vel + nd;
  const int n_items = 1 + nj + nd + nk;
  for (int item = threadIdx.x; item < n_items; item += AMP_THREADS) {
    if (item == 0) {
      s_new[0] = p.root_height_obs ? root[2] : 0.0f;
      const Quat q = {root[3], root[4], root[5], root[6]};
      const Quat qr = p.local_root_obs ? quat_mul(hq, q) : q;
      quat_to_tan_norm(qr, s_new + 1);
      const Vec3 v = {root[7], root[8], root[9]}, w = {root[10], root[11], root[12]};
      const Vec3 lv = quat_rotate(hq, v), lw = quat_rotate(hq, w);
      s_new[7] = lv.x; s_new[8] = lv.y; s_new[9] = lv.z;
      s_new[10] = lw.x; s_new[11] = lw.y; s_new[12] = lw.z;
    } else if (item < 1 + nj) {
      const int j = item - 1;
      const int o = tb.dof_offsets[j], sz = tb.dof_offsets[j + 1] - o;
      const float* dp = p.dof_pos + (int64_t)env * p.dof_pos_ld + o;
      Quat q;
      if (sz == 3) {
        q = exp_map_to_quat(dp[0], dp[1], dp[2]);
      } else {   // 1-dof joint about y (humanoid.py:540-542)
        const Vec3 ay = {0.0f, 1.0f, 0.0f};
        q = quat_from_angle_axis(dp[0], ay);
      }
      quat_to_tan_norm(q, s_new + off_dof + j * 6);
    } else if (item < 1 + nj + nd) {
      const int d = item - 1 - nj;
      s_new[off_vel + d] = p.dof_vel[(int64_t)env * p.dof_vel_ld + d];
    } else {
      const int k = item - 1 - nj - nd;
      const float* kb = root + (int64_t)tb.key_body_ids[k] * p.body_stride;
      const Vec3 d = {kb[0] - root[0], kb[1] - root[1], kb[2] - root[2]};
      const Vec3 lp = quat_rotate(hq, d);
      s_new[off_key + k * 3 + 0] = lp.x; s_new[off_key + k * 3 + 1] = lp.y; s_new[off_key + k * 3 + 2] = lp.z;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < F; i += AMP_THREADS) buf[i] = s_new[i];
  if (p.fill_history) {       // reset (humanoid_amp.py:206-218 default-state path): the whole history := the current frame
    for (int i = threadIdx.x; i < (S - 1) * F; i += AMP_THREADS) buf[F + i] = s_new[i % F];
  } else if (p.shift_history) {
    for (int i = threadIdx.x; i < (S - 1) * F; i += AMP_THREADS) buf[F + i] = s_hist[i];
  }
}

// utils/torch_utils.py:130-141 heading quaternion (not inverted)
__device__ __forceinline__ Quat calc_heading_quat(const Quat q) {
  const Vec3 ex = {1.0f, 0.0f, 0.0f};
  const Vec3 d = quat_rotate(q, ex);
  const float heading = atan2f(d.y, d.x);
  const Vec3 ez = {0.0f, 0.0f, 1.0f};
  return quat_from_angle_axis(heading, ez);
}

// env/tasks/humanoid_heading.py:232-248
__global__ void __launch_bounds__(128)
heading_obs_kernel(const float* __restrict__ root, int64_t rs, const float* __restrict__ tar_dir, const float* __restrict__ tar_speed,
                   const float* __restrict__ face, int n, float* __restrict__ obs, int64_t ld, int col0) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float* r = root + (int64_t)e * rs;
  const Quat q = {r[3], r[4], r[5], r[6]};
  const Quat hq = calc_heading_quat_inv(q);
  const Vec3 td = {tar_dir[2 * e], tar_dir[2 * e + 1], 0.0f}, fd = {face[2 * e], face[2 * e + 1], 0.0f};
  const Vec3 ltd = quat_rotate(hq, td), lfd = quat_rotate(hq, fd);
  float* o = obs + (int64_t)e * ld + col0;
  o[0] = ltd.x; o[1] = ltd.y; o[2] = tar_speed[e]; o[3] = lfd.x; o[4] = lfd.y;
}

// env/tasks/humanoid_heading.py:250-285
__global__ void __launch_bounds__(128)
heading_reward_kernel(const float* __restrict__ pos, int64_t ps, const float* __restrict__ prev, int64_t pps, const float* __restrict__ rot,
                      int64_t rs, const float* __restrict__ tar_dir, const float* __restrict__ tar_speed, const float* __restrict__ face,
                      float dt, int n, float* __restrict__ reward) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float* p = pos + (int64_t)e * ps; const float* pp = prev + (int64_t)e * pps; const float* r = rot + (int64_t)e * rs;
  const float vx = (p[0] - pp[0]) / dt, vy = (p[1] - pp[1]) / dt;
  const float tx = tar_dir[2 * e], ty = tar_dir[2 * e + 1];
  const float tar_dir_speed = tx * vx + ty * vy;
  const float tangent_speed = (vx - tar_dir_speed * tx) + (vy - tar_dir_speed * ty);
  const float verr = tar_speed[e] - tar_dir_speed;
  float dir_reward = expf(-0.25f * (verr * verr + 0.1f * tangent_speed * tangent_speed));
  if (tar_dir_speed <= 0.0f) dir_reward = 0.0f;
  const Quat q = {r[0], r[1], r[2], r[3]};
  const Quat hq = calc_heading_quat(q);
  const Vec3 ex = {1.0f, 0.0f, 0.0f};
  const Vec3 fdir = quat_rotate(hq, ex);
  const float facing = fmaxf(face[2 * e] * fdir.x + face[2 * e + 1] * fdir.y, 0.0f);
  reward[e] = 0.7f * dir_reward + 0.3f * facing;
}

// F.normalize(tar_xy - root_xy) (eps 1e-12: a target exactly at the root gives a zero direction) and the velocity-toward-target term
// shared by compute_location_reward (humanoid_location.py:196-210) and compute_strike_reward (humanoid_strike.py:232-244)
__device__ __forceinline__ float toward_target_vel_reward(const float* p, const float* pp, float dx, float dy, float tar_speed, float dt,
                                                          float* tdx, float* tdy) {
  const float inv = 1.0f / fmaxf(sqrtf(dx * dx + dy * dy), 1e-12f);
  const float tx = dx * inv, ty = dy * inv;
  const float vx = (p[0] - pp[0]) / dt, vy = (p[1] - pp[1]) / dt;
  const float tar_dir_speed = tx * vx + ty * vy;
  const float err = fmaxf(tar_speed - tar_dir_speed, 0.0f);
  *tdx = tx; *tdy = ty;
  return tar_dir_speed <= 0.0f ? 0.0f : expf(-4.0f * (err * err));
}

// env/tasks/humanoid_location.py:169-182: 2-d target (z = 0) relative to the root, rotated by the inverse heading, xy kept
__global__ void __launch_bounds__(128)
location_obs_kernel(const float* __restrict__ root, int64_t rs, const float* __restrict__ tar, int n, float* __restrict__ obs, int64_t ld, int col0) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float* r = root + (int64_t)e * rs;
  const Quat hq = calc_heading_quat_inv({r[3], r[4], r[5], r[6]});
  const Vec3 d = {tar[2 * e] - r[0], tar[2 * e + 1] - r[1], 0.0f - r[2]};
  const Vec3 l = quat_rotate(hq, d);
  float* o = obs + (int64_t)e * ld + col0;
  o[0] = l.x; o[1] = l.y;
}

// env/tasks/humanoid_location.py:184-228
__global__ void __launch_bounds__(128)
location_reward_kernel(const float* __restrict__ root, int64_t rs, const float* __restrict__ prev, int64_t pps, const float* __restrict__ tar,
                       float tar_speed, float dt, int n, float* __restrict__ reward) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float* r = root + (int64_t)e * rs;
  const float dx = tar[2 * e] - r[0], dy = tar[2 * e + 1] - r[1];
  const float pos_err = dx * dx + dy * dy;
  const float pos_reward = expf(-0.5f * pos_err);
  float tx, ty;
  float vel_reward = toward_target_vel_reward(r, prev + (int64_t)e * pps, dx, dy, tar_speed, dt, &tx, &ty);
  const Quat hq = calc_heading_quat({r[3], r[4], r[5], r[6]});
  const Vec3 f = quat_rotate(hq, {1.0f, 0.0f, 0.0f});
  float facing_reward = fmaxf(tx * f.x + ty * f.y, 0.0f);
  if (pos_err < 0.5f) { facing_reward = 1.0f; vel_reward = 1.0f; }     // dist_mask
  reward[e] = 0.5f * pos_reward + 0.4f * vel_reward + 0.1f * facing_reward;
}

// env/tasks/humanoid_reach.py:174-182: the ABSOLUTE target rotated by the inverse heading (the root position is not subtracted, sic)
__global__ void __launch_bounds__(128)
reach_obs_kernel(const float* __restrict__ root, int64_t rs, const float* __restrict__ tar, int n, float* __restrict__ obs, int64_t ld, int col0) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float* r = root + (int64_t)e * rs;
  const Quat hq = calc_heading_quat_inv({r[3], r[4], r[5], r[6]});
  const Vec3 l = quat_rotate(hq, {tar[3 * e], tar[3 * e + 1], tar[3 * e + 2]});
  float* o = obs + (int64_t)e * ld + col0;
  o[0] = l.x; o[1] = l.y; o[2] = l.z;
}

// env/tasks/humanoid_reach.py:184-195: exp(-4 |tar - reach_body_pos|^2)
__global__ void __launch_bounds__(128)
reach_reward_kernel(const float* __restrict__ body, int64_t es, int64_t bs, int reach_body, const float* __restrict__ tar, int n,
                    float* __restrict__ reward) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float* b = body + (int64_t)e * es + (int64_t)reach_body * bs;
  const float dx = tar[3 * e] - b[0], dy = tar[3 * e + 1] - b[1], dz = tar[3 * e + 2] - b[2];
  reward[e] = expf(-4.0f * (dx * dx + dy * dy + dz * dz));
}

// env/tasks/humanoid_strike.py:193-216: local pos (z := the target's absolute z before the rotation, sic) | tan_norm | vel | ang vel
__global__ void __launch_bounds__(128)
strike_obs_kernel(const float* __restrict__ root, int64_t rs, const float* __restrict__ tar, int64_t ts, int n, float* __restrict__ obs,
                  int64_t ld, int col0) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float* r = root + (int64_t)e * rs;
  const float* t = tar + (int64_t)e * ts;
  const Quat hq = calc_heading_quat_inv({r[3], r[4], r[5], r[6]});
  const Vec3 lp = quat_rotate(hq, {t[0] - r[0], t[1] - r[1], t[2]});
  const Vec3 lv = quat_rotate(hq, {t[7], t[8], t[9]}), lw = quat_rotate(hq, {t[10], t[11], t[12]});
  float* o = obs + (int64_t)e * ld + col0;
  o[0] = lp.x; o[1] = lp.y; o[2] = lp.z;
  quat_to_tan_norm(quat_mul(hq, {t[3], t[4], t[5], t[6]}), o + 3);
  o[9] = lv.x; o[10] = lv.y; o[11] = lv.z;
  o[12] = lw.x; o[13] = lw.y; o[14] = lw.z;
}

// env/tasks/humanoid_strike.py:218-251 (strike_body_vel and near_dist are parameters there but unused)
__global__ void __launch_bounds__(128)
strike_reward_kernel(const float* __restrict__ tar, int64_t ts, const float* __restrict__ root, int64_t rs, const float* __restrict__ prev,
                     int64_t pps, float dt, int n, float* __restrict__ reward) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float* t = tar + (int64_t)e * ts;
  const float* r = root + (int64_t)e * rs;
  const Vec3 tar_up = quat_rotate({t[3], t[4], t[5], t[6]}, {0.0f, 0.0f, 1.0f});
  const float tar_rot_err = tar_up.z;
  const float tar_rot_r = fmaxf(1.0f - tar_rot_err, 0.0f);
  float tx, ty;
  const float vel_reward = toward_target_vel_reward(r, prev + (int64_t)e * pps, t[0] - r[0], t[1] - r[1], 1.0f, dt, &tx, &ty);
  const float rew = 0.6f * tar_rot_r + 0.4f * vel_reward;
  reward[e] = tar_rot_err < 0.2f ? 1.0f : rew;                         // succ
}

}  // namespace ase

using namespace ase;

extern "C" int ase_heading_obs(const float* root_states, int64_t root_stride, const float* tar_dir, const float* tar_speed,
                               const float* tar_face_dir, int num_envs, float* obs, int64_t obs_ld, int obs_col0, void* stream) {
  ASE_CHECK_ARG(root_states && tar_dir && tar_speed && tar_face_dir && obs, "ase_heading_obs: null pointer");
  if (num_envs <= 0) return ASE_OK;
  heading_obs_kernel<<<ceil_div(num_envs, 128), 128, 0, (cudaStream_t)stream>>>(root_states, root_stride, tar_dir, tar_speed, tar_face_dir,
                                                                                 num_envs, obs, obs_ld, obs_col0);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_heading_reward(const float* root_pos, int64_t root_pos_stride, const float* prev_root_pos, int64_t prev_stride,
                                  const float* root_rot, int64_t rot_stride, const float* tar_dir, const float* tar_speed,
                                  const float* tar_face_dir, float dt, int num_envs, float* reward, void* stream) {
  ASE_CHECK_ARG(root_pos && prev_root_pos && root_rot && tar_dir && tar_speed && tar_face_dir && reward, "ase_heading_reward: null pointer");
  if (num_envs <= 0) return ASE_OK;
  heading_reward_kernel<<<ceil_div(num_envs, 128), 128, 0, (cudaStream_t)stream>>>(root_pos, root_pos_stride, prev_root_pos, prev_stride,
                                                                                    root_rot, rot_stride, tar_dir, tar_speed, tar_face_dir, dt,
                                                                                    num_envs, reward);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_location_obs(const float* root_states, int64_t root_stride, const float* tar_pos, int num_envs, float* obs, int64_t obs_ld,
                                int obs_col0, void* stream) {
  ASE_CHECK_ARG(root_states && tar_pos && obs, "ase_location_obs: null pointer");
  if (num_envs <= 0) return ASE_OK;
  location_obs_kernel<<<ceil_div(num_envs, 128), 128, 0, (cudaStream_t)stream>>>(root_states, root_stride, tar_pos, num_envs, obs, obs_ld, obs_col0);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_location_reward(const float* root_states, int64_t root_stride, const float* prev_root_pos, int64_t prev_stride, const float* tar_pos,
                                   float tar_speed, float dt, int num_envs, float* reward, void* stream) {
  ASE_CHECK_ARG(root_states && prev_root_pos && tar_pos && reward, "ase_location_reward: null pointer");
  if (num_envs <= 0) return ASE_OK;
  location_reward_kernel<<<ceil_div(num_envs, 128), 128, 0, (cudaStream_t)stream>>>(root_states, root_stride, prev_root_pos, prev_stride, tar_pos,
                                                                                     tar_speed, dt, num_envs, reward);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_reach_obs(const float* root_states, int64_t root_stride, const float* tar_pos, int num_envs, float* obs, int64_t obs_ld,
                             int obs_col0, void* stream) {
  ASE_CHECK_ARG(root_states && tar_pos && obs, "ase_reach_obs: null pointer");
  if (num_envs <= 0) return ASE_OK;
  reach_obs_kernel<<<ceil_div(num_envs, 128), 128, 0, (cudaStream_t)stream>>>(root_states, root_stride, tar_pos, num_envs, obs, obs_ld, obs_col0);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_reach_reward(const float* body_state, int64_t env_stride, int64_t body_stride, int reach_body, const float* tar_pos, int num_envs,
                                float* reward, void* stream) {
  ASE_CHECK_ARG(body_state && tar_pos && reward && reach_body >= 0, "ase_reach_reward: bad argument");
  if (num_envs <= 0) return ASE_OK;
  reach_reward_kernel<<<ceil_div(num_envs, 128), 128, 0, (cudaStream_t)stream>>>(body_state, env_stride, body_stride, reach_body, tar_pos, num_envs,
                                                                                  reward);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_strike_obs(const float* root_states, int64_t root_stride, const float* tar_states, int64_t tar_stride, int num_envs, float* obs,
                              int64_t obs_ld, int obs_col0, void* stream) {
  ASE_CHECK_ARG(root_states && tar_states && obs, "ase_strike_obs: null pointer");
  if (num_envs <= 0) return ASE_OK;
  strike_obs_kernel<<<ceil_div(num_envs, 128), 128, 0, (cudaStream_t)stream>>>(root_states, root_stride, tar_states, tar_stride, num_envs, obs, obs_ld,
                                                                                obs_col0);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_strike_reward(const float* tar_states, int64_t tar_stride, const float* root_states, int64_t root_stride, const float* prev_root_pos,
                                 int64_t prev_stride, float dt, int num_envs, float* reward, void* stream) {
  ASE_CHECK_ARG(tar_states && root_states && prev_root_pos && reward, "ase_strike_reward: null pointer");
  if (num_envs <= 0) return ASE_OK;
  strike_reward_kernel<<<ceil_div(num_envs, 128), 128, 0, (cudaStream_t)stream>>>(tar_states, tar_stride, root_states, root_stride, prev_root_pos,
                                                                                   prev_stride, dt, num_envs, reward);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_obs_build(const AseObsBuildParams* p, void* stream) {
  ASE_CHECK_ARG(p && p->body_state && p->obs, "ase_obs_build: null pointer");
  ASE_CHECK_ARG(p->num_bodies >= 1 && p->num_bodies <= OBS_MAX_BODIES, "ase_obs_build: num_bodies %d out of range", p->num_bodies);
  const int J = p->num_bodies;
  const int obs_dim = 1 + (J - 1) * 3 + J * 6 + J * 3 + J * 3;
  ASE_CHECK_ARG(p->obs_ld >= obs_dim, "ase_obs_build: obs_ld %lld < %d", (long long)p->obs_ld, obs_dim);
  const int count = p->env_ids ? p->num_env_ids : p->num_envs;
  if (count <= 0) return ASE_OK;
  const size_t smem = (size_t)OBS_ENVS_PER_BLOCK * (J * 13 + obs_dim + 4) * sizeof(float);
  obs_build_kernel<<<ceil_div(count, OBS_ENVS_PER_BLOCK), OBS_THREADS, smem, (cudaStream_t)stream>>>(*p, obs_dim);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_amp_obs_build(const AseAmpObsBuildParams* p, void* stream) {
  ASE_CHECK_ARG(p && p->body_state && p->dof_pos && p->dof_vel && p->amp_obs && p->dof_offsets && p->key_body_ids,
                "ase_amp_obs_build: null pointer");
  ASE_CHECK_ARG(p->num_joints >= 1 && p->num_joints <= AMP_MAX_JOINTS && p->num_key_bodies >= 0 && p->num_key_bodies <= AMP_MAX_KEYS,
                "ase_amp_obs_build: joints/keys out of range");
  ASE_CHECK_ARG(p->step_dim == 13 + 6 * p->num_joints + p->num_dofs + 3 * p->num_key_bodies,
                "ase_amp_obs_build: step_dim %d inconsistent", p->step_dim);
  ASE_CHECK_ARG(p->hist_steps >= 1, "ase_amp_obs_build: hist_steps");
  ASE_CHECK_ARG(!(p->fill_history && p->shift_history), "ase_amp_obs_build: fill_history and shift_history exclude each other");
  AmpTables tb;
  for (int j = 0; j <= p->num_joints; ++j) tb.dof_offsets[j] = p->dof_offsets[j];
  for (int j = 0; j < p->num_joints; ++j) {
    const int sz = tb.dof_offsets[j + 1] - tb.dof_offsets[j];
    ASE_CHECK_ARG(sz == 1 || sz == 3, "ase_amp_obs_build: unsupported joint size %d (humanoid.py:543-545)", sz);
  }
  ASE_CHECK_ARG(tb.dof_offsets[p->num_joints] == p->num_dofs, "ase_amp_obs_build: dof_offsets[-1] != num_dofs");
  for (int k = 0; k < p->num_key_bodies; ++k) tb.key_body_ids[k] = p->key_body_ids[k];
  const int count = p->env_ids ? p->num_env_ids : p->num_envs;
  if (count <= 0) return ASE_OK;
  const size_t smem = (size_t)p->hist_steps * p->step_dim * sizeof(float);
  amp_obs_build_kernel<<<count, AMP_THREADS, smem, (cudaStream_t)stream>>>(*p, tb);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

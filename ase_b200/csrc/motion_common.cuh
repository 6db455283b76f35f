// Motion-library device code shared by motion_kernels.cu (ase_motion_state, ase_amp_obs_demo) and reset_kernels.cu (the reference-state
// episode init and its AMP history): frame blend, slerp, the joint dofs of a local rotation and the AMP observation of one (clip, time).
#pragma once
#include "common.cuh"

namespace ase {

constexpr int MOT_THREADS = 64;
constexpr int MOT_MAX_JOINTS = 32;
constexpr int MOT_MAX_KEYS = 16;

struct MotionTablesDev {
  const float *gts, *grs, *lrs, *grvs, *gravs, *dvs, *lengths, *dts;
  const int32_t *num_frames, *starts;
  int J, D, nj, nk;
  int dof_body_ids[MOT_MAX_JOINTS];
  int dof_offsets[MOT_MAX_JOINTS + 1];
  int key_body_ids[MOT_MAX_KEYS];
};

// utils/torch_utils.py:93-115 (component-wise, same select order)
__device__ __forceinline__ Quat slerp(Quat q0, Quat q1, float t) {
  float c = q0.x * q1.x + q0.y * q1.y + q0.z * q1.z + q0.w * q1.w;
  if (c < 0.0f) { q1.x = -q1.x; q1.y = -q1.y; q1.z = -q1.z; q1.w = -q1.w; }
  c = fabsf(c);
  const float half = acosf(c);
  const float s = sqrtf(1.0f - c * c);
  const float ra = sinf((1.0f - t) * half) / s, rb = sinf(t * half) / s;
  Quat r = {ra * q0.x + rb * q1.x, ra * q0.y + rb * q1.y, ra * q0.z + rb * q1.z, ra * q0.w + rb * q1.w};
  if (fabsf(s) < 0.001f) { r.x = 0.5f * q0.x + 0.5f * q1.x; r.y = 0.5f * q0.y + 0.5f * q1.y; r.z = 0.5f * q0.z + 0.5f * q1.z; r.w = 0.5f * q0.w + 0.5f * q1.w; }
  if (c >= 1.0f) r = q0;
  return r;
}

// utils/torch_utils.py:6-27
__device__ __forceinline__ void quat_to_angle_axis(const Quat q, float& angle, Vec3& axis) {
  const float st = sqrtf(1.0f - q.w * q.w);
  const float a = 2.0f * acosf(q.w);
  const float an = atan2f(sinf(a), cosf(a));
  const bool ok = fabsf(st) > 1e-5f;        // false for NaN (|w| > 1 after interpolation), like torch.where on the mask
  angle = ok ? an : 0.0f;
  axis.x = ok ? q.x / st : 0.0f; axis.y = ok ? q.y / st : 0.0f; axis.z = ok ? q.z / st : 1.0f;
}

// utils/motion_lib.py:263-272 _calc_frame_blend: the phase is clamped to [0, 1], the blend is not (a time before the clip start
// extrapolates with a negative blend, as the reference does)
__device__ __forceinline__ void frame_blend(const MotionTablesDev& mt, int id, float time, int64_t& f0l, int64_t& f1l, float& blend) {
  const float len = mt.lengths[id], dt = mt.dts[id];
  const int nf = mt.num_frames[id];
  float phase = time / len;
  phase = fminf(fmaxf(phase, 0.0f), 1.0f);
  const int f0 = (int)(phase * (float)(nf - 1));
  const int f1 = min(f0 + 1, nf - 1);
  blend = (time - (float)f0 * dt) / dt;
  f0l = (int64_t)f0 + mt.starts[id]; f1l = (int64_t)f1 + mt.starts[id];
}

__device__ __forceinline__ Quat load_quat(const float* p) { Quat q = {p[0], p[1], p[2], p[3]}; return q; }

// dof_pos of joint j from the interpolated local rotation (motion_lib.py:296-324); returns the joint size
__device__ __forceinline__ int joint_dof(const MotionTablesDev& mt, int j, int64_t f0l, int64_t f1l, float blend, float* out3) {
  const int body = mt.dof_body_ids[j], sz = mt.dof_offsets[j + 1] - mt.dof_offsets[j];
  const Quat q = slerp(load_quat(mt.lrs + (f0l * mt.J + body) * 4), load_quat(mt.lrs + (f1l * mt.J + body) * 4), blend);
  float angle; Vec3 axis;
  quat_to_angle_axis(q, angle, axis);
  if (sz == 3) { out3[0] = angle * axis.x; out3[1] = angle * axis.y; out3[2] = angle * axis.z; }
  else { const float th = angle * axis.y; out3[0] = atan2f(sinf(th), cosf(th)); }
  return sz;
}

// utils/torch_utils.py:68-91 exp_map_to_quat (same as obs_kernels.cu)
__device__ __forceinline__ Quat exp_map_to_quat_m(float ex, float ey, float ez) {
  const float angle_raw = sqrtf(ex * ex + ey * ey + ez * ez);
  const float angle_n = atan2f(sinf(angle_raw), cosf(angle_raw));
  const bool ok = fabsf(angle_n) > 1e-5f;
  Vec3 axis = {0.0f, 0.0f, 1.0f};
  float angle = 0.0f;
  if (ok) { axis.x = ex / angle_raw; axis.y = ey / angle_raw; axis.z = ez / angle_raw; angle = angle_n; }
  return quat_from_angle_axis(angle, axis);
}

// The AMP observation (build_amp_observations, humanoid_amp.py:282-316) of clip `id` at `time`, written to o[0 .. 13 + 6 nj + D + 3 nk) by
// the whole CTA (MOT_THREADS threads; contains __syncthreads, so every thread of the CTA must call it).
__device__ __forceinline__ void amp_obs_frame(const MotionTablesDev& mt, int id, float time, int local_root_obs, int root_height_obs,
                                              float* __restrict__ o) {
  __shared__ float s_root[8];     // root_pos(3), heading quat(4)
  __shared__ float s_blend;
  __shared__ int64_t s_f[2];
  if (threadIdx.x == 0) {
    int64_t f0l, f1l; float blend;
    frame_blend(mt, id, time, f0l, f1l, blend);
    s_f[0] = f0l; s_f[1] = f1l; s_blend = blend;
    const float* p0 = mt.gts + f0l * mt.J * 3; const float* p1 = mt.gts + f1l * mt.J * 3;
    const float rx = (1.0f - blend) * p0[0] + blend * p1[0], ry = (1.0f - blend) * p0[1] + blend * p1[1], rz = (1.0f - blend) * p0[2] + blend * p1[2];
    const Quat rr = slerp(load_quat(mt.grs + f0l * mt.J * 4), load_quat(mt.grs + f1l * mt.J * 4), blend);
    const Quat hq = calc_heading_quat_inv(rr);
    s_root[0] = rx; s_root[1] = ry; s_root[2] = rz; s_root[3] = hq.x; s_root[4] = hq.y; s_root[5] = hq.z; s_root[6] = hq.w;
    o[0] = root_height_obs ? rz : 0.0f;
    const Quat qr = local_root_obs ? quat_mul(hq, rr) : rr;
    quat_to_tan_norm(qr, o + 1);
    const float* v = mt.grvs + f0l * 3; const float* w = mt.gravs + f0l * 3;
    const Vec3 vv = {v[0], v[1], v[2]}, ww = {w[0], w[1], w[2]};
    const Vec3 lv = quat_rotate(hq, vv), lw = quat_rotate(hq, ww);
    o[7] = lv.x; o[8] = lv.y; o[9] = lv.z; o[10] = lw.x; o[11] = lw.y; o[12] = lw.z;
  }
  __syncthreads();
  const int64_t f0l = s_f[0], f1l = s_f[1];
  const float blend = s_blend;
  const Quat hq = {s_root[3], s_root[4], s_root[5], s_root[6]};
  const int off_dof = 13, off_vel = 13 + 6 * mt.nj, off_key = off_vel + mt.D;
  for (int item = threadIdx.x; item < mt.nj + mt.D + mt.nk; item += MOT_THREADS) {
    if (item < mt.nj) {
      float dp[3];
      const int sz = joint_dof(mt, item, f0l, f1l, blend, dp);
      Quat q;
      if (sz == 3) q = exp_map_to_quat_m(dp[0], dp[1], dp[2]);
      else { const Vec3 ay = {0.0f, 1.0f, 0.0f}; q = quat_from_angle_axis(dp[0], ay); }
      quat_to_tan_norm(q, o + off_dof + item * 6);
    } else if (item < mt.nj + mt.D) {
      const int d = item - mt.nj;
      o[off_vel + d] = mt.dvs[f0l * mt.D + d];
    } else {
      const int k = item - mt.nj - mt.D, body = mt.key_body_ids[k];
      const float* p0 = mt.gts + (f0l * mt.J + body) * 3; const float* p1 = mt.gts + (f1l * mt.J + body) * 3;
      const Vec3 d = {(1.0f - blend) * p0[0] + blend * p1[0] - s_root[0], (1.0f - blend) * p0[1] + blend * p1[1] - s_root[1],
                      (1.0f - blend) * p0[2] + blend * p1[2] - s_root[2]};
      const Vec3 lp = quat_rotate(hq, d);
      o[off_key + k * 3 + 0] = lp.x; o[off_key + k * 3 + 1] = lp.y; o[off_key + k * 3 + 2] = lp.z;
    }
  }
}

static inline int fill_tables(const AseMotionLib* m, MotionTablesDev& t) {
  ASE_CHECK_ARG(m && m->gts && m->grs && m->lrs && m->grvs && m->gravs && m->dvs && m->motion_lengths && m->motion_num_frames &&
                m->motion_dt && m->length_starts && m->dof_body_ids && m->dof_offsets && m->key_body_ids, "motion lib: null pointer");
  ASE_CHECK_ARG(m->num_joints >= 1 && m->num_joints <= MOT_MAX_JOINTS && m->num_key_bodies >= 0 && m->num_key_bodies <= MOT_MAX_KEYS,
                "motion lib: joints / key bodies out of range");
  t.gts = m->gts; t.grs = m->grs; t.lrs = m->lrs; t.grvs = m->grvs; t.gravs = m->gravs; t.dvs = m->dvs; t.lengths = m->motion_lengths;
  t.dts = m->motion_dt; t.num_frames = m->motion_num_frames; t.starts = m->length_starts;
  t.J = m->num_bodies; t.D = m->num_dofs; t.nj = m->num_joints; t.nk = m->num_key_bodies;
  for (int j = 0; j < m->num_joints; ++j) t.dof_body_ids[j] = m->dof_body_ids[j];
  for (int j = 0; j <= m->num_joints; ++j) t.dof_offsets[j] = m->dof_offsets[j];
  for (int j = 0; j < m->num_joints; ++j) {
    const int sz = t.dof_offsets[j + 1] - t.dof_offsets[j];
    ASE_CHECK_ARG(sz == 1 || sz == 3, "motion lib: unsupported joint size %d", sz);
  }
  ASE_CHECK_ARG(t.dof_offsets[m->num_joints] == m->num_dofs, "motion lib: dof_offsets[-1] != num_dofs");
  for (int k = 0; k < m->num_key_bodies; ++k) t.key_body_ids[k] = m->key_body_ids[k];
  return ASE_OK;
}

}  // namespace ase

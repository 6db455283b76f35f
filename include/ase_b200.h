/*
 * ase_b200.h -- C ABI of the H100-native (sm_90a) ASE/AMP training engine (libase_b200.so).
 *
 * The reference (nv-tlabs/ASE) is pure Python and has no FFI; each entry point below replaces a
 * Python/torch call site of the reference (cited as file:line relative to /root/reference/ase/).
 * Conventions
 *   - every pointer is a DEVICE pointer borrowed from the caller (PyTorch keeps ownership); the
 *     library never allocates or frees user-visible memory; the only internal memory is the
 *     caller-provided workspace handed to ase_learner_create;
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, no hidden host syncs;
 *   - matrices are row-major fp32 with an explicit leading dimension where noted; RunningMeanStd
 *     statistics are fp64 (rl_games checkpoint contract); dones are uint8;
 *   - return value: 0 on success, negative AseStatus on failure; ase_last_error() gives the text.
 */
#ifndef ASE_B200_H_
#define ASE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ASE_ABI_VERSION 4
#define ASE_MAX_LAYERS 4

typedef enum {
  ASE_OK = 0,
  ASE_ERR_INVALID = -1,     /* bad argument / unsupported shape */
  ASE_ERR_CUDA = -2,        /* a CUDA runtime / driver call failed */
  ASE_ERR_WORKSPACE = -3,   /* workspace too small or misaligned */
  ASE_ERR_UNSUPPORTED = -4  /* feature needs sm_90a hardware that is not present */
} AseStatus;

int ase_abi_version(void);
const char* ase_last_error(void);
/* number of kernels this library has launched since load (bench.py's gpu_launches counter) */
uint64_t ase_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Observation build (env side).  Replaces the TorchScript functions
 *   compute_humanoid_observations_max   env/tasks/humanoid.py:591-635  (+ _compute_humanoid_obs :395-409)
 *   build_amp_observations + dof_to_obs env/tasks/humanoid_amp.py:282-316, humanoid.py:522-552
 *   _update_hist_amp_obs                env/tasks/humanoid_amp.py:248-255
 * Rigid-body state is the Isaac Gym layout [N, bodies_per_env, 13] = pos3, quat xyzw 4, vel3, angvel3
 * (humanoid.py:82-89); strides are in floats so strided views are accepted.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const float* body_state;    /* [N, *, 13] */
  int64_t env_stride;         /* floats between envs */
  int64_t body_stride;        /* floats between bodies (13 for the native layout) */
  int num_envs;
  int num_bodies;             /* J (17 for amp_humanoid_sword_shield.xml) */
  int local_root_obs;         /* humanoid.py:622-624 quirk reproduced when non-zero */
  int root_height_obs;
  const int32_t* env_ids;     /* optional subset (reset path, humanoid.py:395-409); NULL = all */
  int num_env_ids;
  float* obs;                 /* [N, obs_ld]; row e (or env_ids[i]) is written */
  int64_t obs_ld;             /* >= 1 + (J-1)*3 + J*6 + J*3 + J*3 */
  const uint8_t* env_mask;    /* optional [N]: only envs with a non-zero flag are written (device-side reset without an index list) */
} AseObsBuildParams;
int ase_obs_build(const AseObsBuildParams* p, void* stream);

typedef struct {
  const float* body_state; int64_t env_stride; int64_t body_stride;
  const float* dof_pos; int64_t dof_pos_ld;   /* [N, num_dofs] */
  const float* dof_vel; int64_t dof_vel_ld;
  int num_envs;
  int num_dofs;                /* 31 */
  int num_joints;              /* 13 */
  const int32_t* dof_offsets;  /* HOST pointer, num_joints+1 entries (humanoid.py:192); joint size 1 or 3 */
  int num_key_bodies;          /* 6 */
  const int32_t* key_body_ids; /* HOST pointer */
  int local_root_obs; int root_height_obs;
  const int32_t* env_ids; int num_env_ids;  /* optional subset (reset path, humanoid_amp.py:257-275) */
  float* amp_obs;              /* [N, hist_steps, step_dim] contiguous (humanoid_amp.py:42-44) */
  int hist_steps;              /* 10 */
  int step_dim;                /* 13 + 6*num_joints + num_dofs + 3*num_key_bodies = 140 */
  int shift_history;           /* 1: slots i -> i+1 first (post_physics_step path, humanoid_amp.py:50-59) */
  const uint8_t* env_mask;     /* optional [N]: only envs with a non-zero flag are touched */
  int fill_history;            /* 1: every history slot := the current frame (reset, humanoid_amp.py:206-218 default-state path) */
} AseAmpObsBuildParams;
int ase_amp_obs_build(const AseAmpObsBuildParams* p, void* stream);

/* ------------------------------------------------------------------------------------------------
 * RunningMeanStd  (rl_games 1.1.4 algos_torch/running_mean_std.py; call sites common_agent.py:364,
 * amp_agent.py:535-538, ase_agent.py:118,170-181).  mean/var/count are fp64 device buffers
 * (count is a 1-element buffer).  scratch: >= ase_rms_scratch_bytes(rows, cols) bytes.
 * ---------------------------------------------------------------------------------------------- */
int64_t ase_rms_scratch_bytes(int rows, int cols);
/* train-mode forward: update stats with the unbiased batch moments of x[rows, cols], then (if y)
 * y = clamp((x-mean)/sqrt(var+eps), -5, 5) with the UPDATED stats. */
int ase_rms_update(const float* x, int64_t ldx, int rows, int cols,
                   double* mean, double* var, double* count, float eps,
                   float* y, int64_t ldy, void* scratch, void* stream);
/* eval-mode forward (unnorm=0) or value de-normalisation (unnorm=1: sqrt(var+eps)*clamp(x,+-5)+mean) */
int ase_rms_apply(const float* x, int64_t ldx, int rows, int cols,
                  const double* mean, const double* var, float eps, int unnorm,
                  float* y, int64_t ldy, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Rollout-side math
 * ---------------------------------------------------------------------------------------------- */
/* discount_values, learning/common_agent.py:437-449.  All inputs [H, N] (value_size 1), dones uint8.
 * Writes advs[H,N] and (if non-NULL) returns = advs + values. */
int ase_gae(const uint8_t* dones, const float* values, const float* rewards, const float* next_values,
            int horizon, int num_envs, float gamma, float tau, float* advs, float* returns, void* stream);
/* _calc_disc_rewards amp_agent.py:570-577, _calc_enc_rewards ase_agent.py:404-411,469-472,
 * _combine_rewards ase_agent.py:484-490.  enc_pred/latents may be NULL (AMP). */
int ase_amp_rewards(const float* disc_logits, const float* enc_pred, const float* latents, int latent_dim,
                    int rows, float disc_scale, float enc_scale,
                    const float* task_rewards, float task_w, float disc_w, float enc_w,
                    float* disc_r, float* enc_r, float* combined, void* stream);
/* ------------------------------------------------------------------------------------------------
 * Motion library (demo data for the discriminator).  Replaces MotionLib.get_motion_state (utils/motion_lib.py:123-172,
 * 263-272,296-324) and HumanoidAMP.build_amp_obs_demo (env/tasks/humanoid_amp.py:85-101).  The tables are the flat
 * per-frame device tensors MotionLib builds at load time (motion_lib.py:65-89): gts [F,J,3], grs/lrs [F,J,4] xyzw,
 * grvs/gravs [F,3], dvs [F,dofs]; per clip: length (s), frame count, frame dt, offset of its first frame.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const float *gts, *grs, *lrs, *grvs, *gravs, *dvs;
  const float* motion_lengths; const int32_t* motion_num_frames; const float* motion_dt; const int32_t* length_starts;
  int num_bodies, num_dofs;
  int num_joints; const int32_t* dof_body_ids; const int32_t* dof_offsets;   /* HOST pointers (humanoid.py:191-192) */
  int num_key_bodies; const int32_t* key_body_ids;                            /* HOST pointer */
} AseMotionLib;
/* outputs: root_pos [n,3], root_rot [n,4], dof_pos [n,dofs], root_vel [n,3], root_ang_vel [n,3], dof_vel [n,dofs], key_pos [n,keys,3] */
int ase_motion_state(const AseMotionLib* m, const int32_t* motion_ids, const float* motion_times, int n,
                     float* root_pos, float* root_rot, float* dof_pos, float* root_vel, float* root_ang_vel, float* dof_vel,
                     float* key_pos, void* stream);
/* amp_obs [n, num_steps * step_dim]: frame i is the AMP observation of the clip at motion_times0 - i * sim_dt */
int ase_amp_obs_demo(const AseMotionLib* m, const int32_t* motion_ids, const float* motion_times0, int n, float sim_dt,
                     int num_steps, int local_root_obs, int root_height_obs, float* amp_obs, void* stream);

/* HRL heading task (config 5): compute_heading_observations / compute_heading_reward, env/tasks/humanoid_heading.py:232-285.
 * root_states [N, 13] rows with stride root_stride; tar_dir / tar_face_dir [N,2]; tar_speed [N]; task_obs [N, 5] written at
 * obs + obs_col0 with row stride obs_ld (so it can land behind the 253 humanoid features, humanoid_amp_task.py:51-64). */
int ase_heading_obs(const float* root_states, int64_t root_stride, const float* tar_dir, const float* tar_speed,
                    const float* tar_face_dir, int num_envs, float* obs, int64_t obs_ld, int obs_col0, void* stream);
int ase_heading_reward(const float* root_pos, int64_t root_pos_stride, const float* prev_root_pos, int64_t prev_stride,
                       const float* root_rot, int64_t rot_stride, const float* tar_dir, const float* tar_speed,
                       const float* tar_face_dir, float dt, int num_envs, float* reward, void* stream);

/* HRL location / reach / strike tasks (the other three shipped high-level controllers).  Same conventions as the heading task: root_states and
 * tar_states are [N, 13] rows with an explicit stride (26 when both are views of Isaac Gym's _root_states with 2 actors per env), task obs are
 * written at obs + obs_col0 with row stride obs_ld.
 *   ase_location_obs    compute_location_observations  env/tasks/humanoid_location.py:169-182   tar_pos [N,2] (z = 0) -> 2 floats
 *   ase_location_reward compute_location_reward        env/tasks/humanoid_location.py:184-228   prev_root_pos [N,3] rows with prev_stride
 *   ase_reach_obs       compute_location_observations  env/tasks/humanoid_reach.py:174-182      tar_pos [N,3], absolute (not root-relative) -> 3
 *   ase_reach_reward    compute_reach_reward           env/tasks/humanoid_reach.py:184-195      reach body `reach_body` of the [N,J,13] rigid-body state
 *   ase_strike_obs      compute_strike_observations    env/tasks/humanoid_strike.py:193-216     -> 15 floats
 *   ase_strike_reward   compute_strike_reward          env/tasks/humanoid_strike.py:218-251     (strike_body_vel / near_dist are unused there) */
int ase_location_obs(const float* root_states, int64_t root_stride, const float* tar_pos, int num_envs, float* obs, int64_t obs_ld, int obs_col0,
                     void* stream);
int ase_location_reward(const float* root_states, int64_t root_stride, const float* prev_root_pos, int64_t prev_stride, const float* tar_pos,
                        float tar_speed, float dt, int num_envs, float* reward, void* stream);
int ase_reach_obs(const float* root_states, int64_t root_stride, const float* tar_pos, int num_envs, float* obs, int64_t obs_ld, int obs_col0,
                  void* stream);
int ase_reach_reward(const float* body_state, int64_t env_stride, int64_t body_stride, int reach_body, const float* tar_pos, int num_envs,
                     float* reward, void* stream);
int ase_strike_obs(const float* root_states, int64_t root_stride, const float* tar_states, int64_t tar_stride, int num_envs, float* obs,
                   int64_t obs_ld, int obs_col0, void* stream);
int ase_strike_reward(const float* tar_states, int64_t tar_stride, const float* root_states, int64_t root_stride, const float* prev_root_pos,
                      int64_t prev_stride, float dt, int num_envs, float* reward, void* stream);

/* Gaussian head in eval mode (rl_games ModelA2CContinuousLogStd.forward, is_train False) + the eps-greedy
 * override of get_action_values (amp_agent.py:164-167): a = mu + exp(logstd)*noise, neglogp(a); rows whose
 * rand_mask is 0 act deterministically (a := mu) but keep the sampled action's neglogp, as the reference does.
 * sigma_out (optional) receives exp(logstd) broadcast to [rows, act_dim]. */
int ase_policy_sample(const float* mu, const float* logstd, const float* noise, const float* rand_mask,
                      int rows, int act_dim, float* actions, float* neglogp, float* sigma_out, void* stream);
/* ---- rollout step without host round trips (learning/ase_agent.py:36-115,366-381; SURVEY.md 7.1 step 9) ---------------------------------
 * The reference draws action noise / the eps-greedy mask / fresh latents with eager torch calls and turns `dones` and
 * `_latent_reset_steps <= progress_buf` into index lists with nonzero() (a host sync per sim step).  These entry points run the same
 * arithmetic mask-driven, with a counter-based generator (Philox4x32-10) evaluated inside the kernels: `rng` is a 2-element device array
 * {seed, call counter}; ase_rollout_post_step advances the counter, so a whole rollout can be captured in a CUDA graph.  Each takes
 * optional injected draws (parity tests feed the reference's own draws).
 * Addressing: rng is read as uint64 (negative seeds wrap).  Words (x, y, z, w) of block (row, group) of stream sid are
 * Philox4x32-10(counter = (row, group, call lo, call hi), key = (seed lo, seed hi ^ sid * 0x9E3779B1)).  A 32-bit word x becomes
 * u = (fp32(x >> 8) + 0.5f) * 2^-24 in (0, 1] (the top code rounds to 1.0); Box-Muller normals (stream sid, group = column / 4,
 * (a cos, a sin, b cos, b sin) with radii from x and z, angles from y and w) take u as it is.  The Bernoulli draw (stream sid + 1, group
 * 0xFFFFFFFF, word x: u < p) and the task uniforms (stream sid, group 0, words x..w) take min(u, 1 - 2^-24), in (0, 1) like torch.rand,
 * so p = 1 always gives 1 and a target never reaches the top of its range.  Randints (stream sid + 1, group 0xFFFFFFFE, word x) are
 * min + x % max(1, max - min).  The episode resets (ase_amp_state_init) follow the same rules: their uniforms (stream sid, groups 0 and 1)
 * take min(u, 1 - 2^-24) and their fall-bank row is a randint (stream sid + 1, group 0xFFFFFFFE, word x).  oracle/philox_oracle.py restates
 * all of it (oracle/getup_oracle.py the reset draws). */
/* get_action_values' sampling half (rl_games ModelA2CContinuousLogStd eval + amp_agent.py:164-167): a = mu + exp(logstd) * noise,
 * rand_action_mask = bernoulli(rand_probs) (all ones when rand_probs is NULL), masked rows act deterministically. */
int ase_policy_sample_rng(const float* mu, const float* logstd, const float* rand_probs, int rows, int act_dim,
                          const uint64_t* rng, int stream_id, const float* noise_in, const float* mask_in,
                          float* actions, float* neglogp, float* sigma_out, float* mask_out, void* stream);
/* ASEAgent.env_reset's latent part (ase_agent.py:329-364) + _update_latents (:366-381): envs flagged in done_mask get a fresh latent and
 * reset_steps = randint(min, max); otherwise envs with reset_steps <= progress get a fresh latent and reset_steps += randint(min, max).
 * latent = normalize(randn(Z)) (ase_network_builder.py:221-225).  z_in [N, Z] (final latents) / steps_in [N] replace the draws. */
int ase_latent_update(float* latents, int latent_dim, int32_t* reset_steps, const int64_t* progress, const uint8_t* done_mask, int num_envs,
                      int steps_min, int steps_max, const uint64_t* rng, int stream_id, const float* z_in, const int32_t* steps_in, void* stream);
/* after env.step (ase_agent.py:66-92): next_values = value_mean_std^-1(v) * (1 - terminate); current_rewards / current_lengths bookkeeping with
 * the episode meters (meter[0..2] += sum of finished episodes' reward, length, count); rng[1] += 1.  next_values may be NULL. */
int ase_rollout_post_step(const float* rewards, const uint8_t* dones, const uint8_t* terminate, const float* v_next_normed,
                          const double* val_mean, const double* val_var, float eps, int num_envs, float* next_values,
                          float* cur_rewards, float* cur_lengths, float* meter, uint64_t* rng, void* stream);
/* ---- evaluation players (learning/common_player.py, amp_players.py, ase_players.py, hrl_players.py) ----------------------------------------
 * CommonPlayer.run reads `done.nonzero()` and two .item() sums back every step.  These entry points keep the step mask driven: the episode
 * statistics accumulate on the device in an AsePlayerStatus, and the host reads it once per window of steps.  Draws follow the addressing
 * above (rng / stream_id); the caller's ase_player_post_step advances rng[1] once per player step. */
typedef struct {
  double reward_sum;        /* run totals over the counted episodes: fp64 sums of their accumulated reward and step count */
  double steps_sum;
  int64_t games_played;     /* episodes counted so far */
  int32_t stopped;          /* sticky: set by the step that took games_played to >= n_games; later launches change nothing */
  uint32_t ticket;          /* block ticket of the running launch; 0 between launches */
} AsePlayerStatus;
/* ase_players.py:61-94: every env flagged in done_mask (_reset_latents(done_ids)), or every env when resample_all (_update_latents), gets
 * latent = normalize(randn(Z)) (the same device function as ase_latent_update).  z_in [N, Z] (final latents) replaces the draws. */
int ase_player_latents(float* latents, int latent_dim, const uint8_t* done_mask, int resample_all, int num_envs, const uint64_t* rng,
                       int stream_id, const float* z_in, void* stream);
/* ase_players.py:54-59, hrl_players.py:53-60,243-249: a = mu, or mu + exp(logstd) * eps when logstd is non-NULL (stochastic; eps from the
 * Philox stream or noise_in [rows, A]); a := clamp(a, -1, 1).  actions (optional) = rescale_actions(low, high, a) with per-component bounds
 * (a itself when low/high are NULL); unit_out (optional) = normalize(a), the HRL high-level step's latent for the LLC.  act_dim <= 128. */
int ase_player_act(const float* mu, const float* logstd, int rows, int act_dim, const float* low, const float* high, const uint64_t* rng,
                   int stream_id, const float* noise_in, float* actions, float* unit_out, void* stream);
/* bytes of the per-block partial sums ase_player_post_step needs for num_envs envs */
int ase_player_scratch_bytes(int num_envs);
/* CommonPlayer.run after env.step (common_player.py:73-117).  Sub-step mode (llc_steps > 1, HRLPlayer.env_step hrl_players.py:174-191):
 * sub_rewards / sub_dones accumulate r and d over sub_step = 0 .. llc_steps - 1; the last sub-step forms r = sum / llc_steps, d = count > 0
 * and runs the rest.  Per env: cr += r, steps += 1, done_out = d; for the done envs, record[0..2] = {count, sum of cr, sum of steps} (fp64,
 * reduced per block and then in block order by the last block to finish), added to the status totals, and their cr / steps zeroed.  A step
 * that takes games_played to >= n_games counts in full and sets status->stopped.  While stopped is set the launch changes nothing (record
 * included), so the caller zeroes the records it hands in.  Called with llc_steps == 1 and sub_step 0 outside HRL. */
int ase_player_post_step(const float* rewards, const uint8_t* dones, int num_envs, int sub_step, int llc_steps, float* sub_rewards,
                         float* sub_dones, float* cr, float* steps, uint8_t* done_out, int64_t n_games, AsePlayerStatus* status,
                         double* record, void* scratch, uint64_t* rng, void* stream);
/* compute_humanoid_reset, env/tasks/humanoid.py:645-670: contact forces [N, J, 3] (strides in floats), rigid-body state as in ase_obs_build,
 * is_contact_body [J] flags the bodies allowed to touch the ground (contact_body_ids), termination_heights [J]. */
int ase_humanoid_reset(const int64_t* progress, const float* contact, int64_t contact_env_stride, int64_t contact_body_stride,
                       const float* body_state, int64_t env_stride, int64_t body_stride, int num_bodies, const uint8_t* is_contact_body,
                       const float* termination_heights, float max_episode_length, int enable_early_termination, int num_envs,
                       uint8_t* reset_out, uint8_t* terminate_out, void* stream);
/* compute_humanoid_reset of the strike task, env/tasks/humanoid_strike.py:254-295: the base rule above, plus failure when the target's contact
 * force tar_contact [N,3] (rows with tar_contact_stride: body num_bodies of the net-contact tensor) exceeds 1.0 in x or y while a body that is
 * neither a contact body nor a strike body (is_strike_body [J]: sword, right_hand, right_lower_arm) has a force component above 1.0. */
int ase_strike_reset(const int64_t* progress, const float* contact, int64_t contact_env_stride, int64_t contact_body_stride,
                     const float* body_state, int64_t env_stride, int64_t body_stride, int num_bodies, const uint8_t* is_contact_body,
                     const uint8_t* is_strike_body, const float* termination_heights, const float* tar_contact, int64_t tar_contact_stride,
                     float max_episode_length, int enable_early_termination, int num_envs, uint8_t* reset_out, uint8_t* terminate_out, void* stream);

/* Task target resampling without host syncs: _update_task / _reset_task of env/tasks/humanoid_heading.py:147-174,
 * humanoid_location.py:107-125, humanoid_reach.py:111-130 and _reset_target of humanoid_strike.py:108-128.  The reference turns
 * `progress_buf >= change_steps` into an index list with nonzero() on every pre_physics_step; here one kernel is driven by a mask.
 *   reset_mask NULL (update mode): envs with progress >= change_steps resample (heading, location, reach; strike has no update);
 *   reset_mask [N] uint8 (reset mode): the flagged envs resample (progress is expected to be 0 already, as after _reset_env_tensors).
 * Targets: heading tar = tar_dir [N,2] (+ tar_speed [N], tar_face_dir [N,2]); location tar_pos [N,2]; reach tar_pos [N,3]; strike the [N,13]
 * target state.  tar rows are tar_stride floats apart.  change_steps [N] int64 := progress + randint(min, max) (not for strike).
 * Draws: rng / stream_id as ase_latent_update (streams stream_id and stream_id + 1; the caller advances rng[1] in a later launch), or injected
 * u_in [N,4] (uniform k of an env is its k-th draw in the reference's order) and steps_in [N] int64. */
typedef enum { ASE_TASK_HEADING = 0, ASE_TASK_LOCATION = 1, ASE_TASK_REACH = 2, ASE_TASK_STRIKE = 3 } AseTaskKind;
typedef struct {
  int kind;                                /* AseTaskKind */
  int change_steps_min, change_steps_max;  /* heading: headingChangeSteps{Min,Max}; location / reach: tarChangeSteps{Min,Max} */
  float speed_min, speed_max;              /* heading: tarSpeed{Min,Max} */
  int rand_heading;                        /* heading: enableRandHeading (0: both angles 0 and the speed is the first draw) */
  float dist_max;                          /* location / reach: tarDistMax; strike: far distance (10) */
  float height_min, height_max;            /* reach: tarHeight{Min,Max} */
  float dist_min, near_dist, near_prob;    /* strike: 0.5, 1.5, 0.5 */
  float target_height;                     /* strike: 0.9 */
} AseTaskParams;
int ase_task_resample(const AseTaskParams* p, const float* root_states, int64_t root_stride, const int64_t* progress, const uint8_t* reset_mask,
                      int num_envs, float* tar, int64_t tar_stride, float* tar_speed, float* tar_face_dir, int64_t* change_steps,
                      const uint64_t* rng, int stream_id, const float* u_in, const int64_t* steps_in, void* stream);

/* ---- episode resets of HumanoidAMP / HumanoidAMPGetup without host syncs -------------------------------------------------------------
 * The reference starts an episode with index lists (bernoulli -> env_ids[mask] -> len(...) > 0, multinomial for the clip ids): a host sync
 * per sim step.  Three mask-driven entry points replace it, in this order for a reset:
 *   ase_amp_state_init    HumanoidAMP._reset_actors / _reset_default / _reset_ref_state_init / _reset_hybrid_state_init / _set_env_state
 *                         (env/tasks/humanoid_amp.py:141-201,238-246), HumanoidAMPGetup._reset_actors / _reset_recovery_episode /
 *                         _reset_fall_episode (env/tasks/humanoid_amp_getup.py:78-116) and the buffer zeroing of
 *                         Humanoid._reset_env_tensors (env/tasks/humanoid.py:150-167);
 *   then ase_obs_build and ase_amp_obs_build (env_mask = reset_mask, no shift, no fill) rebuild the observation and AMP slot 0;
 *   ase_amp_history_init  HumanoidAMP._init_amp_obs / _init_amp_obs_default / _init_amp_obs_ref (humanoid_amp.py:203-236) and the getup
 *                         override (humanoid_amp_getup.py:123-129).
 * Every step, after the env's reset rule (ase_humanoid_reset):
 *   ase_recovery_step     HumanoidAMPGetup._update_recovery_count (pre_physics_step, humanoid_amp_getup.py:36-40,131-134) and its
 *                         _compute_reset override (:136-142).  The decrement runs at post-physics here; that is equivalent because nothing
 *                         reads the counter between pre_physics_step and _compute_reset.
 * Init kinds, decided per env flagged in reset_mask in the reference's order: recovery (bernoulli(recovery_prob) and terminate[env]: the state
 * is left as it is, counter := recovery_steps), else fall (bernoulli(fall_prob): root state, dof pos and dof vel := row randint(0, F) of the
 * fall-state bank, counter := recovery_steps), else by state_init: Default (the env's initial root state and dofs), Start (reference state at
 * time 0), Random (reference state at phase * motion_length), Hybrid (bernoulli(hybrid_prob): Random-style reference init, else Default);
 * counter := 0 in these cases.  The reference clip id is the first m with u < motion_cdf[m] (inverse CDF; motion_cdf [M] is the fp32 cumsum
 * of the normalised clip weights with the last entry 1.0, the role of torch.multinomial).  progress, reset and terminate := 0 for every
 * flagged env.  Unflagged envs, and the state of recovery envs, are not written.
 * Philox draws of env e (rng / stream_id as ase_latent_update; the caller advances rng[1] in a later launch): stream sid, group 0, words x, y,
 * z, w = the recovery, fall and hybrid Bernoulli uniforms and the phase; stream sid, group 1, word x = the clip-id uniform; all through
 * min(u, 1 - 2^-24) (so p = 1 always fires).  Fall row: stream sid + 1, group 0xFFFFFFFE, word x: x % max(1, F).
 * Injected draws (per env, the outcomes torch.bernoulli / torch.multinomial / torch.rand / torch.randint_like record in the reference):
 * recovery_in, fall_in, hybrid_in [N] uint8, motion_id_in [N] int32, phase_in [N] fp32, fall_row_in [N] int32. */
typedef enum { ASE_STATE_INIT_DEFAULT = 0, ASE_STATE_INIT_START = 1, ASE_STATE_INIT_RANDOM = 2, ASE_STATE_INIT_HYBRID = 3 } AseStateInit;
typedef enum { ASE_INIT_NONE = 0, ASE_INIT_DEFAULT = 1, ASE_INIT_REF = 2, ASE_INIT_FALL = 3, ASE_INIT_RECOVERY = 4 } AseInitKind;
typedef struct {
  int state_init;                          /* AseStateInit (stateInit) */
  float hybrid_prob;                       /* hybridInitProb */
  float recovery_prob, fall_prob;          /* recoveryEpisodeProb, fallInitProb (0 for plain HumanoidAMP) */
  int recovery_steps;                      /* recoverySteps */
  const uint8_t* reset_mask; int num_envs;
  /* env state, written in place: root rows [N, 13] (pos, quat xyzw, vel, ang vel) root_stride floats apart (26 for Isaac Gym's two-actor
   * _root_states); dof pos / vel [N, D] with row and element strides (Isaac Gym's [N, D, 2] _dof_state: row 2D, element 2) */
  float* root_states; int64_t root_stride;
  float* dof_pos; int64_t dof_pos_stride, dof_pos_elem_stride;
  float* dof_vel; int64_t dof_vel_stride, dof_vel_elem_stride;
  const float* init_root_states; const float* init_dof_pos; const float* init_dof_vel;    /* [N, 13], [N, D], [N, D] contiguous */
  const float* fall_root_states; const float* fall_dof_pos; const float* fall_dof_vel;    /* [F, 13], [F, D], [F, D] contiguous */
  int num_fall_states;                     /* F (0: no fall bank; fall_prob must then be 0) */
  int32_t* recovery_counter;               /* [N] or NULL (plain HumanoidAMP) */
  int64_t* progress; uint8_t* reset_buf; uint8_t* terminate_buf;                          /* [N]; terminate is read before it is cleared */
  uint8_t* kind_out; int32_t* motion_id_out; float* motion_time_out;                      /* [N]: AseInitKind of every env (NONE when not
                                                                                              flagged); clip id and time of REF envs */
  const uint64_t* rng; int stream_id;
  const uint8_t* recovery_in; const uint8_t* fall_in; const uint8_t* hybrid_in;
  const int32_t* motion_id_in; const float* phase_in; const int32_t* fall_row_in;
} AseStateInitParams;
int ase_amp_state_init(const AseMotionLib* m, const float* motion_cdf, int num_motions, const AseStateInitParams* p, void* stream);
/* After slot 0 of the flagged envs was rebuilt: DEFAULT and FALL envs get slots 1..S-1 := slot 0; REF envs get slot k := the AMP observation of
 * their clip at time + fp32(-sim_dt * k), k = 1..S-1 (bitwise what ase_amp_obs_demo gives for that time with one step; times before the clip
 * start extrapolate with a negative blend, as the reference does); NONE and RECOVERY envs are untouched.  amp_obs [N, S, step_dim]. */
int ase_amp_history_init(const AseMotionLib* m, const uint8_t* kind, const int32_t* motion_ids, const float* motion_times, int num_envs,
                         float sim_dt, int local_root_obs, int root_height_obs, float* amp_obs, int hist_steps, void* stream);
/* counter := max(counter - 1, 0); then reset := 0 and terminate := 0 wherever counter > 0. */
int ase_recovery_step(int32_t* recovery_counter, uint8_t* reset_buf, uint8_t* terminate_buf, int num_envs, void* stream);

/* _calc_advs amp_agent.py:551-561 (+ torch_ext.normalization_with_masks); mask NULL => plain
 * mean / unbiased std (common_agent.py:536-546).  scratch >= 64 bytes. */
int ase_adv_normalize(const float* returns, const float* values, const float* mask, int rows,
                      float* advs, void* scratch, void* stream);

/* Minibatch gather: dst_i[r, :] = src_i[idx_i[r], :] (idx NULL = identity) for up to ASE_GATHER_MAX fp32 tensors in one
 * launch.  Replaces the per-tensor advanced indexing of AMPDataset._get_item (learning/amp_datasets.py:14-27) and the demo /
 * replay row fetches (amp_agent.py:194-202, replay_buffer.py:27-69); idx are int64 device row indices as torch produces. */
#define ASE_GATHER_MAX 16
typedef struct { const float* src; float* dst; const int64_t* idx; int rows, cols; int64_t src_ld, dst_ld; } AseGatherItem;
typedef struct { int count; AseGatherItem item[ASE_GATHER_MAX]; } AseGatherBatch;
int ase_gather_rows(const AseGatherBatch* batch, void* stream);

/* ------------------------------------------------------------------------------------------------
 * GEMM primitives (exposed for tests / profiling; the learner drives them internally).
 *   C[M,N] = epilogue( alpha * op(A) . op(B) )          fp32 in, fp32 accumulate, fp32 out
 *   a_trans = 0: A is [M,K] row-major (lda);  1: A is [K,M] row-major
 *   b_trans = 0: B is [N,K] row-major (ldb) (torch Linear weight);  1: B is [K,N] row-major
 *   epilogue: + bias[N]; act 0 none / 1 relu / 2 tanh; mask_mode 1: *= (mask_src>0), 2: *= (1-mask_src^2);
 *   accumulate 1: C += result (atomic when split_k > 1)
 *   backend 0: SIMT fp32 FFMA kernel; 1: wgmma 3xTF32 tensor-core kernel (sm_90a; operands are
 *   split on the fly into TF32 hi/lo pairs -- see DESIGN.md "GEMM"); 2: wgmma 3xFP16 kernel (operands scaled by
 *   a per-tensor power of two and split into FP16 hi/lo pairs: same accuracy class, twice the MMA rate).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const float* A; int64_t lda; int a_trans;
  const float* B; int64_t ldb; int b_trans;
  float* C; int64_t ldc;
  int M, N, K;
  float alpha;
  const float* bias;
  int act;
  const float* mask_src; int64_t ldm; int mask_mode;
  int accumulate;
  int split_k;              /* 0/1 = none; < 0 with accumulate: the tensor-core backends choose (ase_gemm_tc_plan) */
  int backend;
  void* workspace; int64_t workspace_bytes;   /* backends 1, 2: >= ase_gemm_tc_workspace_bytes(), 1024-byte aligned */
  float* colsum_out;        /* optional [N]: colsum_out[n] += sum_m C[m,n] (not with accumulate) */
  /* tensor-core backends, optional (NULL / 0 = unused; the SIMT backend ignores them):
   *  relu_bits_out [M, ldrb words]: bit n%32 of word n/32 of row m := (C[m,n] > 0) -- the ReLU activity of a forward layer,
   *    1 bit instead of 32 for the backward pass;  mask_bits [M, ldmb words]: used INSTEAD of mask_src for mask_mode 1;
   *  c_planes_only: the caller promises that C is only ever consumed as a GEMM operand (through the learner's operand
   *    planes) or through relu_bits_out, so the fp32 store may be skipped whenever the planes are written. */
  uint32_t* relu_bits_out; int64_t ldrb;
  const uint32_t* mask_bits; int64_t ldmb;
  int c_planes_only;
} AseGemmParams;
int ase_gemm(const AseGemmParams* p, void* stream);
int64_t ase_gemm_tc_workspace_bytes(int M, int N, int K);
/* Tile plan the tensor-core backends (1, 2) use for an ase_gemm of this shape: output tile height (128 or 256) and width
 * (128 or 64), and the number of K splits as launched.  accumulate and split_k as in AseGemmParams; split_k < 0 (with
 * accumulate) is the plan the learner uses for its dW GEMMs: the splits are chosen by the kernel's launch-time model. */
int ase_gemm_tc_plan(int M, int N, int K, int accumulate, int split_k, int backend, int* tile_m, int* tile_n, int* splits);
/* Live timing of the tensor-core GEMM kernel (bench.py roofline): enable(1)/disable(0) resets the counters; while
 * enabled every launch is bracketed by CUDA events on its stream.  _read synchronises those events and returns the
 * summed kernel time, the launch count and the algorithmic FLOPs (2*M*N*Kpad per launch). */
int ase_gemm_tc_profile(int enable);
int ase_gemm_tc_profile_read(double* total_ms, int64_t* launches, double* flops);
/* The operand-plane registry the learner runs its tensor-core GEMMs through, exposed (for tests) behind an opaque handle: fp32
 * buffers registered with hi/lo planes in caller memory (TF32 words for backend 1, scaled FP16 halfs for backend 2, stored in the
 * same float space), per-call scale sites, weights split in one batched pass.  Each function maps onto one registry operation:
 *   create      backend 1 or 2; device_mem: >= ase_gemm_planes_device_bytes() (backend 2 only, zero-filled here; may be NULL for 1)
 *   add         register an fp32 buffer of capacity_floats and its planes (plane_capacity_floats floats each)
 *   begin_call  start of one stream-ordered sequence of GEMMs whose scale sites start at site_base (backend 2: re-predicts scales)
 *   forget      the parameters changed: every scale is re-derived exactly on the next call
 *   prep_weights  split each srcs[i] (contiguous [rows[i], cols[i]], registered) at weight site i, count <= 40
 *   gemm        ase_gemm through the registry (p->backend must match)
 *   info        out[6] = valid, fp32_stale, rows, cols, ld, ldp of the buffer registered at `base`; if the planes are valid (backend 2)
 *               and scale_dst is set, [scale, 1/scale] they were written with is copied to scale_dst (device, stream-ordered)
 *   status      the sticky scale-miss flag of backend 2 (bits as ase_learner_plane_status), one stream synchronisation; clear resets it */
typedef struct AseGemmPlanes AseGemmPlanes;
int64_t ase_gemm_planes_device_bytes(void);
int ase_gemm_planes_create(int backend, void* device_mem, AseGemmPlanes** out);
void ase_gemm_planes_destroy(AseGemmPlanes* h);
int ase_gemm_planes_add(AseGemmPlanes* h, const float* base, int64_t capacity_floats, float* hi, float* lo, int64_t plane_capacity_floats);
int ase_gemm_planes_begin_call(AseGemmPlanes* h, int site_base, void* stream);
int ase_gemm_planes_forget(AseGemmPlanes* h);
int ase_gemm_planes_prep_weights(AseGemmPlanes* h, const float* const* srcs, const int* rows, const int* cols, int count, void* stream);
int ase_gemm_planes_gemm(AseGemmPlanes* h, const AseGemmParams* p, void* stream);
int ase_gemm_planes_info(AseGemmPlanes* h, const float* base, int64_t* out, float* scale_dst, void* stream);
int ase_gemm_planes_status(AseGemmPlanes* h, int* flags, void* stream);
int ase_gemm_planes_clear(AseGemmPlanes* h, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Learner: one PPO + adversarial minibatch update.  Replaces
 *   ASEAgent.calc_gradients    learning/ase_agent.py:159-308   (kind ASE)
 *   AMPAgent.calc_gradients    learning/amp_agent.py:266-390   (kind AMP)
 *   CommonAgent.calc_gradients learning/common_agent.py:353-435 (kind PPO; HRL high-level policy)
 * including the networks of learning/{amp,ase}_network_builder.py, the Gaussian head of rl_games
 * ModelA2CContinuousLogStd, RunningMeanStd train-mode updates, every loss term and torch.optim.Adam
 * (common_agent.py:45).
 * ---------------------------------------------------------------------------------------------- */
typedef enum { ASE_KIND_PPO = 0, ASE_KIND_AMP = 1, ASE_KIND_ASE = 2 } AseKind;

typedef struct {
  int kind;
  int obs_dim, act_dim, amp_dim, latent_dim;
  int n_units;       int units[ASE_MAX_LAYERS];        /* actor / critic trunk (mlp.units) */
  int n_disc_units;  int disc_units[ASE_MAX_LAYERS];   /* disc (= enc) trunk (disc.units) */
  int n_style_units; int style_units[ASE_MAX_LAYERS];  /* [512,256] (ase_network_builder.py:160) */
  int batch;          /* minibatch_size */
  int amp_batch;      /* amp_minibatch_size */
  /* hyper-parameters (data/cfg/train/rlg/ase_humanoid.yaml:59-114) */
  float e_clip, critic_coef, entropy_coef, bounds_loss_coef;
  float disc_coef, disc_logit_reg, disc_grad_penalty, disc_weight_decay;
  float enc_coef, amp_diversity_bonus, amp_diversity_tar;
  float lr, beta1, beta2, adam_eps;
  float rms_eps;      /* 1e-5 */
  int gemm_backend;   /* 0 SIMT, 1 wgmma 3xTF32, 2 wgmma 3xFP16 (scaled planes) */
  int mu_activation;  /* 0 none (AMP/ASE), 2 tanh (HRL high-level policy, hrl_network_builder.py:26-29) */
} AseLearnerConfig;

/* Parameter arena: one flat fp32 buffer; tensor i (in the reference's model.parameters() order without
 * the frozen `sigma`, i.e. Adam state order) lives at float offset ase_learner_param_offset(i). */
typedef struct AseLearner AseLearner;

int ase_learner_num_params(const AseLearnerConfig* cfg);                      /* tensor count */
int ase_learner_param_desc(const AseLearnerConfig* cfg, int index, int64_t* offset, int* rows, int* cols);
int64_t ase_learner_arena_floats(const AseLearnerConfig* cfg);
int64_t ase_learner_workspace_bytes(const AseLearnerConfig* cfg);
int ase_learner_create(const AseLearnerConfig* cfg, void* workspace, int64_t workspace_bytes, AseLearner** out);
void ase_learner_destroy(AseLearner* l);

typedef struct {
  float* params; float* grads; float* exp_avg; float* exp_avg_sq;   /* arenas, ase_learner_arena_floats() each */
  const float* logstd;            /* [act_dim] frozen `sigma` parameter (-2.9) */
  double* obs_mean; double* obs_var; double* obs_count;             /* running_mean_std */
  double* amp_mean; double* amp_var; double* amp_count;             /* _amp_input_mean_std (NULL for PPO) */
} AseLearnerState;

typedef struct {
  /* minibatch, reference key names (ase_agent.py:162-186) */
  const float* obs;               /* [B, obs_dim] */
  const float* actions;           /* [B, act_dim] */
  const float* old_logp_actions;  /* [B] */
  const float* advantages;        /* [B] */
  const float* old_mu;            /* [B, act_dim] */
  const float* old_sigma;         /* [B, act_dim] */
  const float* returns;           /* [B] */
  const float* old_values;        /* [B] (unused: clip_value False) */
  const float* rand_action_mask;  /* [B]  (NULL for PPO) */
  const float* ase_latents;       /* [B, latent_dim] (ASE) */
  const float* new_latents;       /* [B, latent_dim] the z' of _diversity_loss (ase_agent.py:451) */
  const float* amp_obs;           /* [Ba, amp_dim] */
  const float* amp_obs_replay;    /* [Ba, amp_dim] */
  const float* amp_obs_demo;      /* [Ba, amp_dim] */
  int update_rms;                 /* 1 = train mode (reference behaviour) */
} AseMinibatch;

/* train_result (ase_agent.py:296-306, amp_agent.py:470-478): written as floats into `scalars` */
enum {
  ASE_TR_ACTOR_LOSS = 0, ASE_TR_CRITIC_LOSS, ASE_TR_B_LOSS, ASE_TR_ENTROPY, ASE_TR_CLIP_FRAC, ASE_TR_KL,
  ASE_TR_DISC_LOSS, ASE_TR_DISC_GRAD_PENALTY, ASE_TR_DISC_LOGIT_LOSS, ASE_TR_DISC_AGENT_ACC,
  ASE_TR_DISC_DEMO_ACC, ASE_TR_DISC_AGENT_LOGIT_MEAN, ASE_TR_DISC_DEMO_LOGIT_MEAN,
  ASE_TR_ENC_LOSS, ASE_TR_DIVERSITY_LOSS, ASE_TR_TOTAL_LOSS, ASE_TR_COUNT = 16
};

typedef struct {
  float* scalars;            /* [ASE_TR_COUNT] */
  float* disc_agent_logit;   /* optional [2*Ba] (agent then replay rows) */
  float* disc_demo_logit;    /* optional [Ba] */
  float* mu;                 /* optional [B, act_dim] current-policy means */
  float* values;             /* optional [B] */
} AseTrainResult;

/* Must be called after the parameter arena was modified by anything other than ase_learner_adam_step (checkpoint load,
 * initialisation, broadcast): the tensor-core backends cache hi/lo planes of the weights between calls. */
int ase_learner_params_changed(AseLearner* l);
/* gemm_backend 2 (scaled FP16 operand planes): sticky status of the per-tensor power-of-two scales, read with one
 * stream synchronisation.  0 = fine.  Bit 0: a value did not fit the scale predicted from the previous call (a tensor's max grew
 * by more than x117 .. x234 between two consecutive calls; x64 always fits); reported after the call that overflowed.  Bit 1: a
 * tensor's max shrank by more than 2^14 .. 2^15 between two calls (2^-13 always fits), so its split lost precision; this is
 * detected when the next call starts, so it is reported after the call FOLLOWING the one that shrank.  That lag is accepted: the
 * flag is sticky and the agent reads it once per epoch, and an underflowed split loses precision gradually (at the flagging edge
 * the max still keeps about 16 bits) instead of saturating as an overflow does.  Either bit means results since the last clear are
 * not fp32-accurate: the host mirror raises. */
int ase_learner_plane_status(AseLearner* l, int* flags, void* stream);
/* The same flag without a host round trip: dst[i * stride] = (float)flags for i < count, on the stream (the agent lets it ride in its
 * per-epoch train_result record); ..._clear resets it after the host has dealt with a miss. */
int ase_learner_plane_flag_to(AseLearner* l, float* dst, int count, int64_t stride, void* stream);
int ase_learner_plane_flag_clear(AseLearner* l, void* stream);

/* forward + losses + backward: fills state->grads (sum over local rows; no Adam) */
int ase_learner_calc_gradients(AseLearner* l, const AseLearnerState* st, const AseMinibatch* mb,
                               const AseTrainResult* out, void* stream);
/* Adam on the whole arena: grads are multiplied by grad_scale first (1/world after an NCCL sum-allreduce,
 * amp_agent.py:357-363 Horovod averaging); step is the 1-based Adam step count. */
int ase_learner_adam_step(AseLearner* l, const AseLearnerState* st, int64_t step, float grad_scale, void* stream);

/* Rollout-side inference with the same weights (eval mode, no RMS update):
 *   get_action_values ase_agent.py:117-148 / amp_agent.py:139-169; _eval_critic ase_agent.py:385-393;
 *   _eval_disc/_eval_enc ase_agent.py:395-411.  Any output pointer may be NULL (mu NULL skips the actor,
 *   value_normed NULL skips the critic).  rows <= batch (actor/critic), rows <= 3*amp_batch (disc/enc). */
int ase_learner_eval_actor_critic(AseLearner* l, const AseLearnerState* st, const float* obs, const float* latents,
                                  int rows, float* mu, float* value_normed, void* stream);
int ase_learner_eval_disc_enc(AseLearner* l, const AseLearnerState* st, const float* amp_obs, int rows,
                              float* disc_logits, float* enc_pred, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Multi-GPU: env-sharded data parallelism, ONE fp32 sum-allreduce of the flat gradient arena per minibatch over NCCL (NVLink / NVSwitch)
 * between calc_gradients and adam_step (learning/amp_agent.py:348-363: Horovod averages inside optimizer.step; 1/world goes into
 * ase_learner_adam_step's grad_scale).  The communicator is the library's own: rank 0 calls ase_comm_unique_id, the host ships the 128
 * bytes to the other ranks (torch.distributed's store in the Python mirror), every rank calls ase_comm_create.  libnccl.so.2 is resolved at
 * run time (ase_comm_load(path) or the default search path), never at link time.
 * ---------------------------------------------------------------------------------------------- */
typedef struct AseComm AseComm;
int ase_comm_load(const char* libnccl_path);
int ase_comm_unique_id(uint8_t* out128);
int ase_comm_create(const uint8_t* id128, int rank, int world, AseComm** out);
void ase_comm_destroy(AseComm* c);
int ase_grad_allreduce(AseComm* c, float* buf, int64_t count, void* stream);
int ase_comm_allreduce_f64(AseComm* c, double* buf, int64_t count, void* stream);   /* RunningMeanStd averaging once per epoch (hvd.sync_stats) */


/* ------------------------------------------------------------------------------------------------
 * Multi-GPU, one NVSwitch node: gradient allreduce + Adam as ONE kernel over NVLink peer memory (csrc/peer.cu) -- replaces the pair
 * ase_grad_allreduce + ase_learner_adam_step, i.e. Horovod's averaging inside optimizer.step (learning/amp_agent.py:348-363) plus
 * torch.optim.Adam (common_agent.py:45).  Each rank allocates its gradient arena with ase_peer_alloc (cudaMalloc + CUDA IPC handle), the
 * host gathers the 64-byte handles of all ranks in rank order, every rank calls ase_peer_open.  The learner then accumulates its gradients
 * straight into ase_peer_grads(local) and calls ase_learner_peer_adam_step once per minibatch: barrier, in-place reduce-scatter + all-gather
 * of the arena by direct peer loads / stores (rank r sums slice r in rank order 0..N-1: bit-identical results on every rank), barrier, Adam
 * over the full local arena (optimizer state stays replicated).  A peer that does not show up within ~15 s raises bit 2 of the status word
 * ase_learner_plane_status reports (and ase_peer_status): an error, never a hang.  2 <= world <= 8.
 * ---------------------------------------------------------------------------------------------- */
typedef struct AsePeer AsePeer;
int64_t ase_peer_buffer_bytes(int64_t arena_floats);
int ase_peer_alloc(int64_t arena_floats, void** local, uint8_t* handle64);
int ase_peer_open(const uint8_t* handles /* world x 64 bytes */, int world, int rank, void* local, int64_t arena_floats, AsePeer** out);
void ase_peer_close(AsePeer* p, int free_local);
float* ase_peer_grads(void* local);
int ase_peer_status(AsePeer* p, int* error, void* stream);
int ase_peer_debug(AsePeer* p, long long* out8);      /* clock64() stamps of block 0's phases in the last call: start, ready, reduced, fenced, done, end */
int ase_learner_peer_adam_step(AseLearner* l, AsePeer* p, const AseLearnerState* st, int64_t step, float grad_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif  /* ASE_B200_H_ */

"""ctypes binding of include/ase_b200.h (the C ABI of libase_b200.so).  No torch types cross the
boundary: tensors are passed as raw device pointers + sizes, the stream as a void*.
The library is REQUIRED: importing this module without the built .so raises (no CPU fallback)."""
import ctypes as C
import os

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'csrc', 'libase_b200.so')
ASE_MAX_LAYERS = 4
KIND_PPO, KIND_AMP, KIND_ASE = 0, 1, 2

TR_NAMES = ['actor_loss', 'critic_loss', 'b_loss', 'entropy', 'actor_clip_frac', 'kl', 'disc_loss', 'disc_grad_penalty',
            'disc_logit_loss', 'disc_agent_acc', 'disc_demo_acc', 'disc_agent_logit_mean', 'disc_demo_logit_mean',
            'enc_loss', 'amp_diversity_loss', 'total_loss']
TR_COUNT = 16

vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_int64, C.c_float


class ObsBuildParams(C.Structure):
    _fields_ = [('body_state', vp), ('env_stride', i64), ('body_stride', i64), ('num_envs', i32), ('num_bodies', i32),
                ('local_root_obs', i32), ('root_height_obs', i32), ('env_ids', vp), ('num_env_ids', i32),
                ('obs', vp), ('obs_ld', i64), ('env_mask', vp)]


class AmpObsBuildParams(C.Structure):
    _fields_ = [('body_state', vp), ('env_stride', i64), ('body_stride', i64),
                ('dof_pos', vp), ('dof_pos_ld', i64), ('dof_vel', vp), ('dof_vel_ld', i64),
                ('num_envs', i32), ('num_dofs', i32), ('num_joints', i32), ('dof_offsets', C.POINTER(C.c_int32)),
                ('num_key_bodies', i32), ('key_body_ids', C.POINTER(C.c_int32)),
                ('local_root_obs', i32), ('root_height_obs', i32), ('env_ids', vp), ('num_env_ids', i32),
                ('amp_obs', vp), ('hist_steps', i32), ('step_dim', i32), ('shift_history', i32), ('env_mask', vp), ('fill_history', i32)]


class MotionLibParams(C.Structure):
    _fields_ = [('gts', vp), ('grs', vp), ('lrs', vp), ('grvs', vp), ('gravs', vp), ('dvs', vp),
                ('motion_lengths', vp), ('motion_num_frames', vp), ('motion_dt', vp), ('length_starts', vp),
                ('num_bodies', i32), ('num_dofs', i32), ('num_joints', i32), ('dof_body_ids', C.POINTER(C.c_int32)),
                ('dof_offsets', C.POINTER(C.c_int32)), ('num_key_bodies', i32), ('key_body_ids', C.POINTER(C.c_int32))]


class GemmParams(C.Structure):
    _fields_ = [('A', vp), ('lda', i64), ('a_trans', i32), ('B', vp), ('ldb', i64), ('b_trans', i32),
                ('C', vp), ('ldc', i64), ('M', i32), ('N', i32), ('K', i32), ('alpha', f32), ('bias', vp), ('act', i32),
                ('mask_src', vp), ('ldm', i64), ('mask_mode', i32), ('accumulate', i32), ('split_k', i32), ('backend', i32),
                ('workspace', vp), ('workspace_bytes', i64), ('colsum_out', vp),
                ('relu_bits_out', vp), ('ldrb', i64), ('mask_bits', vp), ('ldmb', i64), ('c_planes_only', i32)]


ASE_GATHER_MAX = 16


class GatherItem(C.Structure):
    _fields_ = [('src', vp), ('dst', vp), ('idx', vp), ('rows', i32), ('cols', i32), ('src_ld', i64), ('dst_ld', i64)]


class GatherBatch(C.Structure):
    _fields_ = [('count', i32), ('item', GatherItem * ASE_GATHER_MAX)]


TASK_HEADING, TASK_LOCATION, TASK_REACH, TASK_STRIKE = 0, 1, 2, 3


class TaskParams(C.Structure):
    _fields_ = [('kind', i32), ('change_steps_min', i32), ('change_steps_max', i32), ('speed_min', f32), ('speed_max', f32), ('rand_heading', i32),
                ('dist_max', f32), ('height_min', f32), ('height_max', f32), ('dist_min', f32), ('near_dist', f32), ('near_prob', f32),
                ('target_height', f32)]


STATE_INIT = {'Default': 0, 'Start': 1, 'Random': 2, 'Hybrid': 3}                      # AseStateInit (HumanoidAMP.StateInit)
INIT_NONE, INIT_DEFAULT, INIT_REF, INIT_FALL, INIT_RECOVERY = 0, 1, 2, 3, 4            # AseInitKind


class StateInitParams(C.Structure):
    _fields_ = [('state_init', i32), ('hybrid_prob', f32), ('recovery_prob', f32), ('fall_prob', f32), ('recovery_steps', i32),
                ('reset_mask', vp), ('num_envs', i32), ('root_states', vp), ('root_stride', i64),
                ('dof_pos', vp), ('dof_pos_stride', i64), ('dof_pos_elem_stride', i64), ('dof_vel', vp), ('dof_vel_stride', i64),
                ('dof_vel_elem_stride', i64), ('init_root_states', vp), ('init_dof_pos', vp), ('init_dof_vel', vp),
                ('fall_root_states', vp), ('fall_dof_pos', vp), ('fall_dof_vel', vp), ('num_fall_states', i32),
                ('recovery_counter', vp), ('progress', vp), ('reset_buf', vp), ('terminate_buf', vp),
                ('kind_out', vp), ('motion_id_out', vp), ('motion_time_out', vp), ('rng', vp), ('stream_id', i32),
                ('recovery_in', vp), ('fall_in', vp), ('hybrid_in', vp), ('motion_id_in', vp), ('phase_in', vp), ('fall_row_in', vp)]


class LearnerConfig(C.Structure):
    _fields_ = [('kind', i32), ('obs_dim', i32), ('act_dim', i32), ('amp_dim', i32), ('latent_dim', i32),
                ('n_units', i32), ('units', i32 * ASE_MAX_LAYERS),
                ('n_disc_units', i32), ('disc_units', i32 * ASE_MAX_LAYERS),
                ('n_style_units', i32), ('style_units', i32 * ASE_MAX_LAYERS),
                ('batch', i32), ('amp_batch', i32),
                ('e_clip', f32), ('critic_coef', f32), ('entropy_coef', f32), ('bounds_loss_coef', f32),
                ('disc_coef', f32), ('disc_logit_reg', f32), ('disc_grad_penalty', f32), ('disc_weight_decay', f32),
                ('enc_coef', f32), ('amp_diversity_bonus', f32), ('amp_diversity_tar', f32),
                ('lr', f32), ('beta1', f32), ('beta2', f32), ('adam_eps', f32), ('rms_eps', f32), ('gemm_backend', i32), ('mu_activation', i32)]


class LearnerState(C.Structure):
    _fields_ = [('params', vp), ('grads', vp), ('exp_avg', vp), ('exp_avg_sq', vp), ('logstd', vp),
                ('obs_mean', vp), ('obs_var', vp), ('obs_count', vp), ('amp_mean', vp), ('amp_var', vp), ('amp_count', vp)]


class Minibatch(C.Structure):
    _fields_ = [('obs', vp), ('actions', vp), ('old_logp_actions', vp), ('advantages', vp), ('old_mu', vp), ('old_sigma', vp),
                ('returns', vp), ('old_values', vp), ('rand_action_mask', vp), ('ase_latents', vp), ('new_latents', vp),
                ('amp_obs', vp), ('amp_obs_replay', vp), ('amp_obs_demo', vp), ('update_rms', i32)]


class TrainResult(C.Structure):
    _fields_ = [('scalars', vp), ('disc_agent_logit', vp), ('disc_demo_logit', vp), ('mu', vp), ('values', vp)]


# every symbol declared in include/ase_b200.h (tests/test_abi.py checks the two lists agree)
EXPORTS = ['ase_abi_version', 'ase_last_error', 'ase_launch_count', 'ase_obs_build', 'ase_amp_obs_build',
           'ase_rms_scratch_bytes', 'ase_rms_update', 'ase_rms_apply', 'ase_gae', 'ase_amp_rewards', 'ase_heading_obs', 'ase_heading_reward', 'ase_location_obs', 'ase_location_reward', 'ase_reach_obs', 'ase_reach_reward', 'ase_strike_obs', 'ase_strike_reward', 'ase_motion_state', 'ase_amp_obs_demo', 'ase_policy_sample', 'ase_policy_sample_rng', 'ase_latent_update', 'ase_rollout_post_step', 'ase_player_latents', 'ase_player_act', 'ase_player_scratch_bytes', 'ase_player_post_step', 'ase_humanoid_reset', 'ase_strike_reset', 'ase_task_resample', 'ase_amp_state_init', 'ase_amp_history_init', 'ase_recovery_step', 'ase_adv_normalize', 'ase_gather_rows',
           'ase_gemm', 'ase_gemm_tc_workspace_bytes', 'ase_gemm_tc_plan', 'ase_gemm_tc_profile', 'ase_gemm_tc_profile_read', 'ase_learner_num_params', 'ase_learner_param_desc',
           'ase_learner_arena_floats', 'ase_learner_workspace_bytes', 'ase_learner_create', 'ase_learner_destroy', 'ase_learner_params_changed', 'ase_learner_plane_status', 'ase_learner_plane_flag_to', 'ase_learner_plane_flag_clear',
           'ase_learner_calc_gradients', 'ase_learner_adam_step', 'ase_learner_eval_actor_critic',
           'ase_learner_eval_disc_enc', 'ase_comm_load', 'ase_comm_unique_id', 'ase_comm_create', 'ase_comm_destroy', 'ase_grad_allreduce',
           'ase_comm_allreduce_f64', 'ase_peer_buffer_bytes', 'ase_peer_alloc', 'ase_peer_open', 'ase_peer_close', 'ase_peer_grads',
           'ase_peer_status', 'ase_peer_debug', 'ase_learner_peer_adam_step']


class AseError(RuntimeError):
    pass


def _load():
    if not os.path.exists(_LIB_PATH):
        raise ImportError(f"{_LIB_PATH} is missing: build it with `python -m ase_b200.build` "
                          "(ase_b200 has no CPU fallback; the CUDA library is the product)")
    lib = C.CDLL(_LIB_PATH)
    lib.ase_last_error.restype = C.c_char_p
    lib.ase_launch_count.restype = C.c_uint64
    for n in ('ase_rms_scratch_bytes', 'ase_gemm_tc_workspace_bytes', 'ase_learner_arena_floats', 'ase_learner_workspace_bytes'):
        getattr(lib, n).restype = C.c_int64
    lib.ase_learner_destroy.restype = None
    lib.ase_rms_scratch_bytes.argtypes = [i32, i32]
    lib.ase_rms_update.argtypes = [vp, i64, i32, i32, vp, vp, vp, f32, vp, i64, vp, vp]
    lib.ase_rms_apply.argtypes = [vp, i64, i32, i32, vp, vp, f32, i32, vp, i64, vp]
    lib.ase_gae.argtypes = [vp, vp, vp, vp, i32, i32, f32, f32, vp, vp, vp]
    lib.ase_amp_rewards.argtypes = [vp, vp, vp, i32, i32, f32, f32, vp, f32, f32, f32, vp, vp, vp, vp]
    lib.ase_heading_obs.argtypes = [vp, i64, vp, vp, vp, i32, vp, i64, i32, vp]
    lib.ase_heading_reward.argtypes = [vp, i64, vp, i64, vp, i64, vp, vp, vp, f32, i32, vp, vp]
    lib.ase_location_obs.argtypes = [vp, i64, vp, i32, vp, i64, i32, vp]
    lib.ase_location_reward.argtypes = [vp, i64, vp, i64, vp, f32, f32, i32, vp, vp]
    lib.ase_reach_obs.argtypes = [vp, i64, vp, i32, vp, i64, i32, vp]
    lib.ase_reach_reward.argtypes = [vp, i64, i64, i32, vp, i32, vp, vp]
    lib.ase_strike_obs.argtypes = [vp, i64, vp, i64, i32, vp, i64, i32, vp]
    lib.ase_strike_reward.argtypes = [vp, i64, vp, i64, vp, i64, f32, i32, vp, vp]
    lib.ase_motion_state.argtypes = [C.POINTER(MotionLibParams), vp, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.ase_amp_obs_demo.argtypes = [C.POINTER(MotionLibParams), vp, vp, i32, f32, i32, i32, i32, vp, vp]
    lib.ase_policy_sample.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, vp, vp]
    lib.ase_adv_normalize.argtypes = [vp, vp, vp, i32, vp, vp, vp]
    lib.ase_policy_sample_rng.argtypes = [vp, vp, vp, i32, i32, vp, i32, vp, vp, vp, vp, vp, vp, vp]
    lib.ase_latent_update.argtypes = [vp, i32, vp, vp, vp, i32, i32, i32, vp, i32, vp, vp, vp]
    lib.ase_rollout_post_step.argtypes = [vp, vp, vp, vp, vp, vp, f32, i32, vp, vp, vp, vp, vp, vp]
    lib.ase_player_latents.argtypes = [vp, i32, vp, i32, i32, vp, i32, vp, vp]
    lib.ase_player_act.argtypes = [vp, vp, i32, i32, vp, vp, vp, i32, vp, vp, vp, vp]
    lib.ase_player_scratch_bytes.argtypes = [i32]
    lib.ase_player_post_step.argtypes = [vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, i64, vp, vp, vp, vp, vp]
    lib.ase_humanoid_reset.argtypes = [vp, vp, i64, i64, vp, i64, i64, i32, vp, vp, f32, i32, i32, vp, vp, vp]
    lib.ase_strike_reset.argtypes = [vp, vp, i64, i64, vp, i64, i64, i32, vp, vp, vp, vp, i64, f32, i32, i32, vp, vp, vp]
    lib.ase_task_resample.argtypes = [C.POINTER(TaskParams), vp, i64, vp, vp, i32, vp, i64, vp, vp, vp, vp, i32, vp, vp, vp]
    lib.ase_amp_state_init.argtypes = [C.POINTER(MotionLibParams), vp, i32, C.POINTER(StateInitParams), vp]
    lib.ase_amp_history_init.argtypes = [C.POINTER(MotionLibParams), vp, vp, vp, i32, f32, i32, i32, vp, i32, vp]
    lib.ase_recovery_step.argtypes = [vp, vp, vp, i32, vp]
    lib.ase_learner_plane_flag_to.argtypes = [vp, vp, i32, i64, vp]
    lib.ase_learner_plane_flag_clear.argtypes = [vp, vp]
    lib.ase_gather_rows.argtypes = [C.POINTER(GatherBatch), vp]
    lib.ase_obs_build.argtypes = [C.POINTER(ObsBuildParams), vp]
    lib.ase_amp_obs_build.argtypes = [C.POINTER(AmpObsBuildParams), vp]
    lib.ase_gemm.argtypes = [C.POINTER(GemmParams), vp]
    lib.ase_gemm_tc_workspace_bytes.argtypes = [i32, i32, i32]
    lib.ase_gemm_tc_plan.argtypes = [i32, i32, i32, i32, i32, i32, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.ase_gemm_tc_profile.argtypes = [i32]
    lib.ase_gemm_tc_profile_read.argtypes = [C.POINTER(C.c_double), C.POINTER(i64), C.POINTER(C.c_double)]
    lib.ase_learner_num_params.argtypes = [C.POINTER(LearnerConfig)]
    lib.ase_learner_param_desc.argtypes = [C.POINTER(LearnerConfig), i32, C.POINTER(i64), C.POINTER(i32), C.POINTER(i32)]
    lib.ase_learner_arena_floats.argtypes = [C.POINTER(LearnerConfig)]
    lib.ase_learner_workspace_bytes.argtypes = [C.POINTER(LearnerConfig)]
    lib.ase_learner_create.argtypes = [C.POINTER(LearnerConfig), vp, i64, C.POINTER(vp)]
    lib.ase_learner_destroy.argtypes = [vp]
    lib.ase_learner_params_changed.argtypes = [vp]
    lib.ase_learner_plane_status.argtypes = [vp, C.POINTER(C.c_int), vp]
    lib.ase_learner_calc_gradients.argtypes = [vp, C.POINTER(LearnerState), C.POINTER(Minibatch), C.POINTER(TrainResult), vp]
    lib.ase_learner_adam_step.argtypes = [vp, C.POINTER(LearnerState), i64, f32, vp]
    lib.ase_learner_eval_actor_critic.argtypes = [vp, C.POINTER(LearnerState), vp, vp, i32, vp, vp, vp]
    lib.ase_learner_eval_disc_enc.argtypes = [vp, C.POINTER(LearnerState), vp, i32, vp, vp, vp]
    lib.ase_comm_load.argtypes = [C.c_char_p]
    lib.ase_comm_unique_id.argtypes = [vp]
    lib.ase_comm_create.argtypes = [vp, i32, i32, C.POINTER(vp)]
    lib.ase_comm_destroy.argtypes = [vp]
    lib.ase_comm_destroy.restype = None
    lib.ase_grad_allreduce.argtypes = [vp, vp, i64, vp]
    lib.ase_comm_allreduce_f64.argtypes = [vp, vp, i64, vp]
    lib.ase_peer_buffer_bytes.argtypes = [i64]; lib.ase_peer_buffer_bytes.restype = i64
    lib.ase_peer_alloc.argtypes = [i64, C.POINTER(vp), vp]
    lib.ase_peer_open.argtypes = [vp, i32, i32, vp, i64, C.POINTER(vp)]
    lib.ase_peer_close.argtypes = [vp, i32]; lib.ase_peer_close.restype = None
    lib.ase_peer_grads.argtypes = [vp]; lib.ase_peer_grads.restype = vp
    lib.ase_peer_status.argtypes = [vp, C.POINTER(i32), vp]
    lib.ase_peer_debug.argtypes = [vp, vp]
    lib.ase_learner_peer_adam_step.argtypes = [vp, vp, C.POINTER(LearnerState), i64, f32, vp]
    return lib


lib = _load()


def check(rc, what=''):
    if rc != 0:
        raise AseError(f"{what} failed with status {rc}: {lib.ase_last_error().decode()}")


def launch_count():
    return int(lib.ase_launch_count())

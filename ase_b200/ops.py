"""Host-side mirror of the reference's env/agent helper functions, each a thin call into the C ABI.
Tensors stay torch CUDA tensors (device memory + stream plumbing only); all arithmetic is in libase_b200.so."""
import ctypes as C

import torch

from . import lib as L
from .lib import lib, check

DOF_OFFSETS_SWORD_SHIELD = [0, 3, 6, 9, 10, 13, 16, 17, 20, 21, 24, 27, 28, 31]   # env/tasks/humanoid.py:192
KEY_BODY_IDS_SWORD_SHIELD = [5, 10, 13, 16, 6, 9]                                 # humanoid_ase_sword_shield_getup.yaml:20


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _f32c(t, name):
    if not (t.is_cuda and t.dtype == torch.float32):
        raise TypeError(f"{name}: expected a CUDA float32 tensor, got {t.device} {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


def _body_strides(body_state):
    """body_state [N, J, 13] (possibly a strided view of [N, bodies_per_env, 13]); inner dim must be contiguous."""
    if not (body_state.is_cuda and body_state.dtype == torch.float32 and body_state.dim() == 3 and body_state.shape[2] == 13
            and body_state.stride(2) == 1):
        raise TypeError("body_state must be a CUDA float32 [N, J, 13] tensor with contiguous last dim")
    return body_state.stride(0), body_state.stride(1)


def compute_humanoid_observations_max(body_state, local_root_obs, root_height_obs, out=None, env_ids=None, env_mask=None):
    """env/tasks/humanoid.py:591-635 on the packed rigid-body state [N, J, 13] (pos, quat xyzw, vel, angvel).
    env_ids (int32 CUDA tensor) restricts the update to a subset of rows (reset path, humanoid.py:395-409); env_mask (uint8 [N]) does the
    same without an index list (no host sync)."""
    n, j, _ = body_state.shape
    es, bs = _body_strides(body_state)
    obs_dim = 1 + (j - 1) * 3 + j * 6 + j * 3 + j * 3
    if out is None:
        out = torch.empty(n, obs_dim, device=body_state.device, dtype=torch.float32)
    p = L.ObsBuildParams(_p(body_state), es, bs, n, j, int(bool(local_root_obs)), int(bool(root_height_obs)),
                         _p(env_ids), 0 if env_ids is None else env_ids.numel(), _p(out), out.stride(0), _p(env_mask))
    check(lib.ase_obs_build(C.byref(p), _stream()), 'ase_obs_build')
    return out


def build_amp_observations(body_state, dof_pos, dof_vel, amp_obs_buf, local_root_obs, root_height_obs,
                           dof_offsets=DOF_OFFSETS_SWORD_SHIELD, key_body_ids=KEY_BODY_IDS_SWORD_SHIELD,
                           shift_history=True, env_ids=None, env_mask=None, fill_history=False):
    """env/tasks/humanoid_amp.py:248-316: (optionally) shift the [N, S, F] history and write the newest frame at slot 0.
    env_mask (uint8 [N]) restricts the update to flagged envs; fill_history sets every slot to the new frame (reset)."""
    n = body_state.shape[0]
    es, bs = _body_strides(body_state)
    dof_pos = _f32c(dof_pos, 'dof_pos'); dof_vel = _f32c(dof_vel, 'dof_vel')
    assert amp_obs_buf.is_contiguous() and amp_obs_buf.dim() == 3
    nj = len(dof_offsets) - 1
    offs = (C.c_int32 * (nj + 1))(*dof_offsets)
    keys = (C.c_int32 * len(key_body_ids))(*key_body_ids)
    p = L.AmpObsBuildParams(_p(body_state), es, bs, _p(dof_pos), dof_pos.stride(0), _p(dof_vel), dof_vel.stride(0),
                            n, dof_pos.shape[1], nj, offs, len(key_body_ids), keys,
                            int(bool(local_root_obs)), int(bool(root_height_obs)), _p(env_ids),
                            0 if env_ids is None else env_ids.numel(), _p(amp_obs_buf), amp_obs_buf.shape[1], amp_obs_buf.shape[2],
                            int(bool(shift_history)), _p(env_mask), int(bool(fill_history)))
    check(lib.ase_amp_obs_build(C.byref(p), _stream()), 'ase_amp_obs_build')
    return amp_obs_buf


class RunningMeanStd:
    """rl_games 1.1.4 RunningMeanStd: f64 buffers named as in the checkpoint (running_mean/running_var/count)."""

    def __init__(self, size, device, eps=1e-5):
        self.size = int(size)
        self.eps = eps
        self.running_mean = torch.zeros(self.size, dtype=torch.float64, device=device)
        self.running_var = torch.ones(self.size, dtype=torch.float64, device=device)
        self.count = torch.ones((), dtype=torch.float64, device=device)
        self.training = True
        self._scratch = None

    def train(self): self.training = True
    def eval(self): self.training = False

    def state_dict(self):
        return {'running_mean': self.running_mean, 'running_var': self.running_var, 'count': self.count}

    def load_state_dict(self, sd):
        self.running_mean.copy_(sd['running_mean']); self.running_var.copy_(sd['running_var']); self.count.copy_(sd['count'])

    def __call__(self, x, unnorm=False, out=None):
        shp = x.shape
        x2 = _f32c(x.reshape(-1, self.size), 'x')
        if out is not None:
            assert out.is_contiguous() and out.numel() == x2.numel() and out.dtype == torch.float32
        y = torch.empty_like(x2) if out is None else out.view(x2.shape)
        if self.training and not unnorm:
            need = lib.ase_rms_scratch_bytes(x2.shape[0], self.size)
            if self._scratch is None or self._scratch.numel() < need:
                self._scratch = torch.empty(need, dtype=torch.uint8, device=x.device)
            check(lib.ase_rms_update(_p(x2), x2.stride(0), x2.shape[0], self.size, _p(self.running_mean), _p(self.running_var),
                                     _p(self.count), self.eps, _p(y), y.stride(0), _p(self._scratch), _stream()), 'ase_rms_update')
        else:
            if self.training and unnorm:
                # rl_games quirk: train-mode forward with unnorm=True also updates; the reference never does that on this path
                raise NotImplementedError("unnorm in train mode is not on the reference's hot path")
            check(lib.ase_rms_apply(_p(x2), x2.stride(0), x2.shape[0], self.size, _p(self.running_mean), _p(self.running_var),
                                    self.eps, int(bool(unnorm)), _p(y), y.stride(0), _stream()), 'ase_rms_apply')
        return y.reshape(shp) if out is None else out


def policy_sample_rng(mu, logstd, rand_probs, rng, stream_id, out_actions, out_neglogp, out_sigma, out_mask, noise=None, mask=None):
    """get_action_values' sampling half with in-kernel Philox draws (or injected noise / mask), written straight into the given
    experience-buffer slices."""
    rows, a = mu.shape
    check(lib.ase_policy_sample_rng(_p(mu), _p(logstd), _p(rand_probs), rows, a, _p(rng), int(stream_id), _p(noise), _p(mask),
                                    _p(out_actions), _p(out_neglogp), _p(out_sigma), _p(out_mask), _stream()), 'ase_policy_sample_rng')


def latent_update(latents, reset_steps, progress, done_mask, steps_min, steps_max, rng, stream_id, z_in=None, steps_in=None):
    """ASEAgent.env_reset (latent part) + _update_latents, mask driven (ase_agent.py:329-381)."""
    n, z = latents.shape
    assert latents.is_contiguous() and reset_steps.dtype == torch.int32 and progress.dtype == torch.int64
    check(lib.ase_latent_update(_p(latents), z, _p(reset_steps), _p(progress), _p(done_mask), n, int(steps_min), int(steps_max),
                                _p(rng), int(stream_id), _p(z_in), _p(steps_in), _stream()), 'ase_latent_update')


def rollout_post_step(rewards, dones, terminate, v_next_normed, value_rms, next_values_out, cur_rewards, cur_lengths, meter, rng):
    """ase_agent.py:66-92 after env.step: next_values, episode bookkeeping, RNG call counter."""
    n = dones.shape[0]
    check(lib.ase_rollout_post_step(_p(rewards), _p(dones), _p(terminate), _p(v_next_normed),
                                    _p(value_rms.running_mean) if value_rms is not None else None,
                                    _p(value_rms.running_var) if value_rms is not None else None,
                                    value_rms.eps if value_rms is not None else 0.0, n, _p(next_values_out), _p(cur_rewards), _p(cur_lengths),
                                    _p(meter), _p(rng), _stream()), 'ase_rollout_post_step')


def player_latents(latents, done_mask, resample_all, rng, stream_id, z_in=None):
    """ASEPlayer._reset_latents(done ids) (done_mask) or of every env (resample_all), mask driven (ase_players.py:61-94)."""
    n, z = latents.shape
    assert latents.is_contiguous() and (done_mask is None or done_mask.dtype == torch.uint8)
    check(lib.ase_player_latents(_p(latents), z, _p(done_mask), int(bool(resample_all)), n, _p(rng), int(stream_id), _p(z_in), _stream()),
          'ase_player_latents')


def player_act(mu, logstd, low, high, rng, stream_id, actions=None, unit_out=None, noise=None):
    """A player's action from the head output mu: Normal.sample when logstd is given (else mu), clamp to [-1, 1], rescale_actions(low, high)
    into `actions` and / or the L2-normalised clamped action into `unit_out` (ase_players.py:54-59, hrl_players.py:53-60,243-249)."""
    rows, a = mu.shape
    mu = _f32c(mu, 'mu')
    check(lib.ase_player_act(_p(mu), _p(logstd), rows, a, _p(low), _p(high), _p(rng), int(stream_id), _p(noise), _p(actions), _p(unit_out),
                             _stream()), 'ase_player_act')


def player_post_step(rewards, dones, sub_step, llc_steps, sub_rewards, sub_dones, cr, steps, done_out, n_games, status, record, scratch, rng):
    """CommonPlayer.run's bookkeeping after env.step (common_player.py:73-117; HRL sub-steps hrl_players.py:174-191) into the device
    AsePlayerStatus `status` (a uint8 tensor of its 32 bytes) and this step's record (3 float64)."""
    n = cr.shape[0]
    rewards = _f32c(rewards.reshape(n), 'rewards')
    dones = dones.reshape(n)
    if dones.dtype != torch.uint8:
        dones = dones.to(torch.uint8)
    check(lib.ase_player_post_step(_p(rewards), _p(dones.contiguous()), n, int(sub_step), int(llc_steps), _p(sub_rewards), _p(sub_dones), _p(cr),
                                   _p(steps), _p(done_out), int(n_games), _p(status), _p(record), _p(scratch), _p(rng), _stream()),
          'ase_player_post_step')


def compute_humanoid_reset(progress_buf, contact_buf, is_contact_body, body_state, max_episode_length, enable_early_termination,
                           termination_heights, reset_out=None, terminate_out=None):
    """env/tasks/humanoid.py:645-670 -> (reset, terminated) uint8 [N].  contact_buf [N, J, 3]; body_state [N, J, 13];
    is_contact_body uint8 [J] (1 for the bodies in contact_body_ids)."""
    n, j, _ = body_state.shape
    es, bs = _body_strides(body_state)
    if reset_out is None:
        reset_out = torch.empty(n, dtype=torch.uint8, device=body_state.device)
    if terminate_out is None:
        terminate_out = torch.empty(n, dtype=torch.uint8, device=body_state.device)
    assert contact_buf.stride(2) == 1
    check(lib.ase_humanoid_reset(_p(progress_buf), _p(contact_buf), contact_buf.stride(0), contact_buf.stride(1), _p(body_state), es, bs, j,
                                 _p(is_contact_body), _p(termination_heights), float(max_episode_length), int(bool(enable_early_termination)), n,
                                 _p(reset_out), _p(terminate_out), _stream()), 'ase_humanoid_reset')
    return reset_out, terminate_out


def discount_values(dones, values, rewards, next_values, gamma, tau, want_returns=False):
    """learning/common_agent.py:437-449.  dones uint8 [H,N]; values/rewards/next_values [H,N,1] or [H,N]."""
    h, n = dones.shape[0], dones.shape[1]
    v = _f32c(values.reshape(h, n), 'values'); r = _f32c(rewards.reshape(h, n), 'rewards'); nv = _f32c(next_values.reshape(h, n), 'next_values')
    d = dones if dones.dtype == torch.uint8 else dones.to(torch.uint8)
    d = d.contiguous()
    advs = torch.empty(h, n, device=v.device, dtype=torch.float32)
    rets = torch.empty_like(advs) if want_returns else None
    check(lib.ase_gae(_p(d), _p(v), _p(r), _p(nv), h, n, gamma, tau, _p(advs), _p(rets), _stream()), 'ase_gae')
    advs = advs.reshape(values.shape)
    return (advs, rets.reshape(values.shape)) if want_returns else advs


def amp_rewards(disc_logits, enc_pred=None, latents=None, disc_scale=2.0, enc_scale=1.0, task_rewards=None,
                task_w=0.0, disc_w=0.5, enc_w=0.5):
    """amp_agent.py:570-577 + ase_agent.py:404-411,484-490 -> (disc_r, enc_r or None, combined), each [rows,1]."""
    rows = disc_logits.numel()
    lg = _f32c(disc_logits.reshape(rows), 'disc_logits')
    zdim = 0
    if enc_pred is not None:
        zdim = enc_pred.shape[-1]
        enc_pred = _f32c(enc_pred.reshape(rows, zdim), 'enc_pred'); latents = _f32c(latents.reshape(rows, zdim), 'latents')
    tr = None if task_rewards is None else _f32c(task_rewards.reshape(rows), 'task_rewards')
    dr = torch.empty(rows, 1, device=lg.device, dtype=torch.float32)
    er = torch.empty_like(dr) if enc_pred is not None else None
    comb = torch.empty_like(dr)
    check(lib.ase_amp_rewards(_p(lg), _p(enc_pred), _p(latents), zdim, rows, disc_scale, enc_scale, _p(tr), task_w, disc_w, enc_w,
                              _p(dr), _p(er), _p(comb), _stream()), 'ase_amp_rewards')
    return dr, er, comb


def compute_heading_observations(root_states, tar_dir, tar_speed, tar_face_dir, out=None, col0=0):
    """env/tasks/humanoid_heading.py:232-248 -> [N,5] (or written into out[:, col0:col0+5])."""
    n = root_states.shape[0]
    assert root_states.stride(1) == 1
    tar_dir = _f32c(tar_dir, 'tar_dir'); tar_speed = _f32c(tar_speed, 'tar_speed'); tar_face_dir = _f32c(tar_face_dir, 'tar_face_dir')
    if out is None:
        out = torch.empty(n, 5, device=root_states.device, dtype=torch.float32)
    check(lib.ase_heading_obs(_p(root_states), root_states.stride(0), _p(tar_dir), _p(tar_speed), _p(tar_face_dir), n, _p(out),
                              out.stride(0), col0, _stream()), 'ase_heading_obs')
    return out


def compute_heading_reward(root_pos, prev_root_pos, root_rot, tar_dir, tar_speed, tar_face_dir, dt):
    """env/tasks/humanoid_heading.py:250-285 -> [N]."""
    n = root_pos.shape[0]
    assert root_pos.stride(1) == 1 and prev_root_pos.stride(1) == 1 and root_rot.stride(1) == 1
    tar_dir = _f32c(tar_dir, 'tar_dir'); tar_speed = _f32c(tar_speed, 'tar_speed'); tar_face_dir = _f32c(tar_face_dir, 'tar_face_dir')
    r = torch.empty(n, device=root_pos.device, dtype=torch.float32)
    check(lib.ase_heading_reward(_p(root_pos), root_pos.stride(0), _p(prev_root_pos), prev_root_pos.stride(0), _p(root_rot), root_rot.stride(0),
                                 _p(tar_dir), _p(tar_speed), _p(tar_face_dir), float(dt), n, _p(r), _stream()), 'ase_heading_reward')
    return r


# ---- the other three HRL tasks (env/tasks/humanoid_{location,reach,strike}.py) and their target resampling -------------------------------
TASK_OBS_SIZE = {'heading': 5, 'location': 2, 'reach': 3, 'strike': 15}
REACH_BODY_SWORD_SHIELD = 6                       # reachBodyName: sword (humanoid_sword_shield_reach.yaml:29)
STRIKE_BODY_IDS_SWORD_SHIELD = [6, 5, 4]          # strikeBodyNames: sword, right_hand, right_lower_arm (humanoid_sword_shield_strike.yaml:22)
# the YAML constants of ase/data/cfg/humanoid_sword_shield_<task>.yaml and the strike task's hard-coded ones (humanoid_strike.py:19-22,117)
TASK_PARAMS = {
    'heading': dict(change_steps_min=100, change_steps_max=200, speed_min=1.5, speed_max=1.6, rand_heading=1),
    'location': dict(change_steps_min=100, change_steps_max=200, dist_max=10.0),
    'reach': dict(change_steps_min=50, change_steps_max=100, dist_max=1.0, height_min=0.2, height_max=2.0),
    'strike': dict(dist_max=10.0, dist_min=0.5, near_dist=1.5, near_prob=0.5, target_height=0.9),
}
_TASK_KIND = {'heading': L.TASK_HEADING, 'location': L.TASK_LOCATION, 'reach': L.TASK_REACH, 'strike': L.TASK_STRIKE}


def _rows(t, name):
    if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.stride(1) == 1):
        raise TypeError(f"{name}: expected CUDA float32 rows with a contiguous last dim")
    return t.stride(0)


def compute_location_observations(root_states, tar_pos, out=None, col0=0):
    """env/tasks/humanoid_location.py:169-182 -> [N,2] (or written into out[:, col0:col0+2])."""
    n = root_states.shape[0]
    rs = _rows(root_states, 'root_states'); tar_pos = _f32c(tar_pos, 'tar_pos')
    if out is None:
        out = torch.empty(n, 2, device=root_states.device, dtype=torch.float32)
    check(lib.ase_location_obs(_p(root_states), rs, _p(tar_pos), n, _p(out), out.stride(0), col0, _stream()), 'ase_location_obs')
    return out


def compute_location_reward(root_states, prev_root_pos, tar_pos, tar_speed, dt, out=None):
    """env/tasks/humanoid_location.py:184-228 -> [N]."""
    n = root_states.shape[0]
    rs = _rows(root_states, 'root_states'); ps = _rows(prev_root_pos, 'prev_root_pos'); tar_pos = _f32c(tar_pos, 'tar_pos')
    if out is None:
        out = torch.empty(n, device=root_states.device, dtype=torch.float32)
    check(lib.ase_location_reward(_p(root_states), rs, _p(prev_root_pos), ps, _p(tar_pos), float(tar_speed), float(dt), n, _p(out), _stream()),
          'ase_location_reward')
    return out


def compute_reach_observations(root_states, tar_pos, out=None, col0=0):
    """env/tasks/humanoid_reach.py:174-182 -> [N,3]: the absolute target rotated by the inverse heading."""
    n = root_states.shape[0]
    rs = _rows(root_states, 'root_states'); tar_pos = _f32c(tar_pos, 'tar_pos')
    if out is None:
        out = torch.empty(n, 3, device=root_states.device, dtype=torch.float32)
    check(lib.ase_reach_obs(_p(root_states), rs, _p(tar_pos), n, _p(out), out.stride(0), col0, _stream()), 'ase_reach_obs')
    return out


def compute_reach_reward(body_state, tar_pos, reach_body=REACH_BODY_SWORD_SHIELD, out=None):
    """env/tasks/humanoid_reach.py:184-195 on the rigid-body state [N, J, 13] -> [N]."""
    n = body_state.shape[0]
    es, bs = _body_strides(body_state); tar_pos = _f32c(tar_pos, 'tar_pos')
    if out is None:
        out = torch.empty(n, device=body_state.device, dtype=torch.float32)
    check(lib.ase_reach_reward(_p(body_state), es, bs, int(reach_body), _p(tar_pos), n, _p(out), _stream()), 'ase_reach_reward')
    return out


def compute_strike_observations(root_states, tar_states, out=None, col0=0):
    """env/tasks/humanoid_strike.py:193-216 -> [N,15]."""
    n = root_states.shape[0]
    rs = _rows(root_states, 'root_states'); ts = _rows(tar_states, 'tar_states')
    if out is None:
        out = torch.empty(n, 15, device=root_states.device, dtype=torch.float32)
    check(lib.ase_strike_obs(_p(root_states), rs, _p(tar_states), ts, n, _p(out), out.stride(0), col0, _stream()), 'ase_strike_obs')
    return out


def compute_strike_reward(tar_states, root_states, prev_root_pos, dt, out=None):
    """env/tasks/humanoid_strike.py:218-251 -> [N]."""
    n = root_states.shape[0]
    ts = _rows(tar_states, 'tar_states'); rs = _rows(root_states, 'root_states'); ps = _rows(prev_root_pos, 'prev_root_pos')
    if out is None:
        out = torch.empty(n, device=root_states.device, dtype=torch.float32)
    check(lib.ase_strike_reward(_p(tar_states), ts, _p(root_states), rs, _p(prev_root_pos), ps, float(dt), n, _p(out), _stream()), 'ase_strike_reward')
    return out


def compute_strike_reset(progress_buf, contact_buf, is_contact_body, is_strike_body, body_state, tar_contact_forces, max_episode_length,
                         enable_early_termination, termination_heights, reset_out=None, terminate_out=None):
    """env/tasks/humanoid_strike.py:254-295 -> (reset, terminated) uint8 [N].  contact_buf [N, J, 3]; tar_contact_forces [N, 3] rows;
    is_contact_body / is_strike_body uint8 [J]."""
    n, j, _ = body_state.shape
    es, bs = _body_strides(body_state)
    if reset_out is None:
        reset_out = torch.empty(n, dtype=torch.uint8, device=body_state.device)
    if terminate_out is None:
        terminate_out = torch.empty(n, dtype=torch.uint8, device=body_state.device)
    assert contact_buf.stride(2) == 1 and tar_contact_forces.stride(1) == 1
    check(lib.ase_strike_reset(_p(progress_buf), _p(contact_buf), contact_buf.stride(0), contact_buf.stride(1), _p(body_state), es, bs, j,
                               _p(is_contact_body), _p(is_strike_body), _p(termination_heights), _p(tar_contact_forces), tar_contact_forces.stride(0),
                               float(max_episode_length), int(bool(enable_early_termination)), n, _p(reset_out), _p(terminate_out), _stream()),
          'ase_strike_reset')
    return reset_out, terminate_out


def task_resample(task, tar, progress, root_states=None, reset_mask=None, tar_speed=None, tar_face_dir=None, change_steps=None, rng=None,
                  stream_id=0, u_in=None, steps_in=None, params=None):
    """_update_task (reset_mask None: envs with progress >= change_steps) / _reset_task / strike _reset_target (envs flagged in the uint8
    reset_mask) without nonzero().  tar: heading tar_dir [N,2], location tar_pos [N,2], reach tar_pos [N,3], strike target states [N,13] rows.
    params overrides entries of TASK_PARAMS[task].  Draws come from the Philox stream {rng, stream_id} or from u_in [N,4] / steps_in [N]."""
    kw = dict(TASK_PARAMS[task], **(params or {}))
    p = L.TaskParams(kind=_TASK_KIND[task], **kw)
    n = tar.shape[0]
    ts = _rows(tar, 'tar')
    rs = 0 if root_states is None else _rows(root_states, 'root_states')
    assert change_steps is None or change_steps.dtype == torch.int64
    assert progress is None or progress.dtype == torch.int64
    check(lib.ase_task_resample(C.byref(p), _p(root_states), rs, _p(progress), _p(reset_mask), n, _p(tar), ts, _p(tar_speed), _p(tar_face_dir),
                                _p(change_steps), _p(rng), int(stream_id), _p(u_in), _p(steps_in), _stream()), 'ase_task_resample')


def policy_sample(mu, logstd, noise, rand_mask=None):
    """Eval-mode Gaussian head + eps-greedy override (amp_agent.py:139-169) -> (actions, neglogpacs, sigmas)."""
    rows, a = mu.shape
    mu = _f32c(mu, 'mu'); noise = _f32c(noise, 'noise')
    actions = torch.empty_like(mu); sig = torch.empty_like(mu)
    nlp = torch.empty(rows, device=mu.device, dtype=torch.float32)
    check(lib.ase_policy_sample(_p(mu), _p(logstd), _p(noise), _p(rand_mask), rows, a, _p(actions), _p(nlp), _p(sig), _stream()),
          'ase_policy_sample')
    return actions, nlp, sig


def calc_advs(returns, values, mask=None):
    """amp_agent.py:551-561 / common_agent.py:536-546 (value_size 1)."""
    rows = returns.shape[0]
    r = _f32c(returns.reshape(rows), 'returns'); v = _f32c(values.reshape(rows), 'values')
    m = None if mask is None else _f32c(mask.reshape(rows), 'mask')
    out = torch.empty(rows, device=r.device, dtype=torch.float32)
    scratch = torch.empty(64, dtype=torch.uint8, device=r.device)
    check(lib.ase_adv_normalize(_p(r), _p(v), _p(m), rows, _p(out), _p(scratch), _stream()), 'ase_adv_normalize')
    return out


def gather_rows(items):
    """items: list of (src [n, ...] contiguous fp32, dst [rows, ...] contiguous fp32, idx int64 [rows] or None): dst[r] = src[idx[r]]
    for all of them in one launch (AMPDataset._get_item + demo / replay fetches, amp_datasets.py:14-27)."""
    for s0 in range(0, len(items), L.ASE_GATHER_MAX):
        chunk = items[s0:s0 + L.ASE_GATHER_MAX]
        b = L.GatherBatch()
        b.count = len(chunk)
        for i, (src, dst, idx) in enumerate(chunk):
            assert src.dtype == torch.float32 and dst.dtype == torch.float32 and src.is_contiguous() and dst.is_contiguous()
            assert idx is None or (idx.dtype == torch.int64 and idx.is_contiguous() and idx.numel() == dst.shape[0])
            cols = 1 if src.dim() == 1 else int(src[0].numel())
            assert (1 if dst.dim() == 1 else int(dst[0].numel())) == cols
            it = b.item[i]
            it.src, it.dst, it.idx = src.data_ptr(), dst.data_ptr(), None if idx is None else idx.data_ptr()
            it.rows, it.cols, it.src_ld, it.dst_ld = dst.shape[0], cols, cols, cols
        check(lib.ase_gather_rows(C.byref(b), _stream()), 'ase_gather_rows')


def gemm(A, B, a_trans=False, b_trans=False, bias=None, act=0, mask_src=None, mask_mode=0, out=None, accumulate=False,
         split_k=0, alpha=1.0, backend=0, colsum_out=None, relu_bits_out=None, mask_bits=None):
    """C = epi(alpha * op(A) . op(B)); see include/ase_b200.h (AseGemmParams)."""
    M = A.shape[1] if a_trans else A.shape[0]
    K = A.shape[0] if a_trans else A.shape[1]
    N = B.shape[1] if b_trans else B.shape[0]
    assert (B.shape[0] if b_trans else B.shape[1]) == K
    assert A.stride(1) == 1 and B.stride(1) == 1
    if out is None:
        out = torch.zeros(M, N, device=A.device, dtype=torch.float32)
    ws, wsb = None, 0
    if backend >= 1:
        wsb = lib.ase_gemm_tc_workspace_bytes(M, N, K)
        ws = torch.empty(wsb + 1024, dtype=torch.uint8, device=A.device)
        off = (-ws.data_ptr()) % 1024
        ws = ws[off:off + wsb]
    p = L.GemmParams(_p(A), A.stride(0), int(a_trans), _p(B), B.stride(0), int(b_trans), _p(out), out.stride(0), M, N, K, alpha,
                     _p(bias), act, _p(mask_src), 0 if mask_src is None else mask_src.stride(0), mask_mode, int(accumulate),
                     split_k, backend, _p(ws), wsb, _p(colsum_out), _p(relu_bits_out), 0 if relu_bits_out is None else relu_bits_out.stride(0),
                     _p(mask_bits), 0 if mask_bits is None else mask_bits.stride(0), 0)
    check(lib.ase_gemm(C.byref(p), _stream()), 'ase_gemm')
    return out


def gemm_tc_plan(M, N, K, accumulate=False, split_k=0, backend=2):
    """(tile rows, tile cols, K splits) the tensor-core backends launch for this ase_gemm shape (ase_gemm_tc_plan)."""
    bm, bn, s = C.c_int(), C.c_int(), C.c_int()
    check(lib.ase_gemm_tc_plan(M, N, K, int(accumulate), split_k, backend, C.byref(bm), C.byref(bn), C.byref(s)), 'ase_gemm_tc_plan')
    return bm.value, bn.value, s.value


# ---- episode resets of HumanoidAMP / HumanoidAMPGetup (env/tasks/humanoid_amp.py:141-246, humanoid_amp_getup.py) -----------------------
# the YAML constants: humanoid_ase_sword_shield_getup.yaml (ASE pre-training) and humanoid_sword_shield.yaml (AMP)
STATE_INIT_PARAMS = {
    'getup': dict(state_init='Hybrid', hybrid_prob=0.5, recovery_prob=0.2, recovery_steps=60, fall_prob=0.1),
    'amp': dict(state_init='Random', hybrid_prob=0.5, recovery_prob=0.0, recovery_steps=0, fall_prob=0.0),
}


def _dof_strides(t, name):
    if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 2):
        raise TypeError(f"{name}: expected a CUDA float32 [N, D] tensor (any strides)")
    return t.stride(0), t.stride(1)


def amp_state_init(motion_lib, reset_mask, root_states, dof_pos, dof_vel, progress, reset_buf, terminate_buf, kind_out, motion_id_out,
                   motion_time_out, state_init='Hybrid', hybrid_prob=0.5, recovery_prob=0.0, fall_prob=0.0, recovery_steps=0,
                   init_root_states=None, init_dof_pos=None, init_dof_vel=None, fall_root_states=None, fall_dof_pos=None, fall_dof_vel=None,
                   recovery_counter=None, rng=None, stream_id=0, recovery_in=None, fall_in=None, hybrid_in=None, motion_id_in=None,
                   phase_in=None, fall_row_in=None):
    """HumanoidAMP / HumanoidAMPGetup._reset_actors for the envs flagged in the uint8 reset_mask, without index lists.  root_states [N, 13] rows
    and dof_pos / dof_vel [N, D] may be strided views (Isaac Gym's _root_states with two actors, the interleaved [N, D, 2] _dof_state); they
    are written in place.  Draws come from the Philox stream {rng, stream_id} or from the injected per-env outcomes."""
    n = reset_mask.shape[0]
    rs = _rows(root_states, 'root_states')
    dps, dpe = _dof_strides(dof_pos, 'dof_pos'); dvs, dve = _dof_strides(dof_vel, 'dof_vel')
    assert progress.dtype == torch.int64 and reset_buf.dtype == torch.uint8 and terminate_buf.dtype == torch.uint8
    assert kind_out.dtype == torch.uint8 and motion_id_out.dtype == torch.int32 and motion_time_out.dtype == torch.float32
    assert recovery_counter is None or recovery_counter.dtype == torch.int32
    for t in (init_root_states, init_dof_pos, init_dof_vel, fall_root_states, fall_dof_pos, fall_dof_vel):
        assert t is None or (t.is_contiguous() and t.dtype == torch.float32)
    p = L.StateInitParams(L.STATE_INIT[state_init], float(hybrid_prob), float(recovery_prob), float(fall_prob), int(recovery_steps),
                          _p(reset_mask), n, _p(root_states), rs, _p(dof_pos), dps, dpe, _p(dof_vel), dvs, dve,
                          _p(init_root_states), _p(init_dof_pos), _p(init_dof_vel), _p(fall_root_states), _p(fall_dof_pos), _p(fall_dof_vel),
                          0 if fall_root_states is None else fall_root_states.shape[0], _p(recovery_counter), _p(progress), _p(reset_buf),
                          _p(terminate_buf), _p(kind_out), _p(motion_id_out), _p(motion_time_out), _p(rng), int(stream_id),
                          _p(recovery_in), _p(fall_in), _p(hybrid_in), _p(motion_id_in), _p(phase_in), _p(fall_row_in))
    mp = motion_lib._params()
    check(lib.ase_amp_state_init(C.byref(mp), _p(motion_lib._motion_cdf), motion_lib.num_motions(), C.byref(p), _stream()), 'ase_amp_state_init')


def amp_history_init(motion_lib, kind, motion_ids, motion_times, amp_obs_buf, sim_dt, local_root_obs=True, root_height_obs=True):
    """HumanoidAMP._init_amp_obs (+ the getup override) after slot 0 of the reset envs was rebuilt: default / fall envs repeat slot 0,
    reference-init envs get their clip's frames at time - k dt; amp_obs_buf [N, S, step_dim] contiguous."""
    assert amp_obs_buf.is_contiguous() and amp_obs_buf.dim() == 3
    n, s, _ = amp_obs_buf.shape
    mp = motion_lib._params()
    check(lib.ase_amp_history_init(C.byref(mp), _p(kind), _p(motion_ids), _p(motion_times), n, float(sim_dt), int(bool(local_root_obs)),
                                   int(bool(root_height_obs)), _p(amp_obs_buf), s, _stream()), 'ase_amp_history_init')


def recovery_step(recovery_counter, reset_buf, terminate_buf):
    """HumanoidAMPGetup._update_recovery_count + its _compute_reset override, after the env's reset rule."""
    assert recovery_counter.dtype == torch.int32 and reset_buf.dtype == torch.uint8 and terminate_buf.dtype == torch.uint8
    check(lib.ase_recovery_step(_p(recovery_counter), _p(reset_buf), _p(terminate_buf), recovery_counter.shape[0], _stream()), 'ase_recovery_step')

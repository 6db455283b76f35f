"""TEST INFRASTRUCTURE ONLY -- CPU (torch fp32/f64) restatement of the HRL tasks' jit functions and target resampling (nv-tlabs/ASE
@ 28952a3): the location, reach and strike task observations, rewards and strike termination, and the per-env arithmetic of the four
tasks' _reset_task / _reset_target.  The checker for the task kernels of ase_b200/csrc; pinned against the reference's own outputs
(tests/golden/task_*.pt, written by oracle/gen_golden_hrl_tasks.py).  All file:line citations are relative to the reference's ase/ directory."""
import math

import torch
import torch.nn.functional as F

from ase_oracle import calc_heading_quat, calc_heading_quat_inv, quat_from_angle_axis, quat_mul, quat_rotate, quat_to_tan_norm

# YAML constants of ase/data/cfg/humanoid_sword_shield_{heading,location,reach}.yaml and the strike task's hard-coded ones
# (humanoid_strike.py:19-22,117)
HRL_TASK_PARAMS = {
    'heading': dict(change_steps_min=100, change_steps_max=200, speed_min=1.5, speed_max=1.6, rand_heading=1),
    'location': dict(change_steps_min=100, change_steps_max=200, dist_max=10.0),
    'reach': dict(change_steps_min=50, change_steps_max=100, dist_max=1.0, height_min=0.2, height_max=2.0),
    'strike': dict(dist_max=10.0, dist_min=0.5, near_dist=1.5, near_prob=0.5, target_height=0.9),
}
STRIKE_BODY_IDS_SWORD_SHIELD = [6, 5, 4]      # strikeBodyNames: sword, right_hand, right_lower_arm


def _toward_target_vel_reward(tar_xy, root_pos, prev_root_pos, dt, tar_speed):
    """The velocity-toward-target term of compute_location_reward / compute_strike_reward -> (F.normalize'd tar_dir, vel_reward)."""
    tar_dir = F.normalize(tar_xy - root_pos[..., 0:2], dim=-1)          # eps 1e-12: a target at the root gives a zero direction
    root_vel = (root_pos - prev_root_pos) / dt
    tar_dir_speed = (tar_dir * root_vel[..., :2]).sum(-1)
    err = torch.clamp_min(tar_speed - tar_dir_speed, 0.0)
    vel_reward = torch.exp(-4.0 * (err * err))
    return tar_dir, torch.where(tar_dir_speed <= 0, torch.zeros_like(vel_reward), vel_reward)


def compute_location_observations(root_states, tar_pos):
    """env/tasks/humanoid_location.py:169-182 -> [N,2] (tar_pos is 2-d, z = 0)."""
    hq = calc_heading_quat_inv(root_states[:, 3:7])
    t3 = torch.cat([tar_pos, torch.zeros_like(tar_pos[..., 0:1])], dim=-1)
    return quat_rotate(hq, t3 - root_states[:, 0:3])[..., 0:2]


def compute_location_reward(root_pos, prev_root_pos, root_rot, tar_pos, tar_speed, dt):
    """env/tasks/humanoid_location.py:184-228."""
    pos_diff = tar_pos - root_pos[..., 0:2]
    pos_err = (pos_diff * pos_diff).sum(-1)
    pos_reward = torch.exp(-0.5 * pos_err)
    tar_dir, vel_reward = _toward_target_vel_reward(tar_pos, root_pos, prev_root_pos, dt, tar_speed)
    ex = torch.zeros_like(root_pos); ex[..., 0] = 1.0
    facing = quat_rotate(calc_heading_quat(root_rot), ex)
    facing_reward = torch.clamp_min((tar_dir * facing[..., 0:2]).sum(-1), 0.0)
    dist_mask = pos_err < 0.5
    facing_reward = torch.where(dist_mask, torch.ones_like(facing_reward), facing_reward)
    vel_reward = torch.where(dist_mask, torch.ones_like(vel_reward), vel_reward)
    return 0.5 * pos_reward + 0.4 * vel_reward + 0.1 * facing_reward


def compute_reach_observations(root_states, tar_pos):
    """env/tasks/humanoid_reach.py:174-182 -> [N,3]: the absolute target rotated by the inverse heading (no root subtraction, sic)."""
    return quat_rotate(calc_heading_quat_inv(root_states[:, 3:7]), tar_pos)


def compute_reach_reward(reach_body_pos, tar_pos):
    """env/tasks/humanoid_reach.py:184-195."""
    d = tar_pos - reach_body_pos
    return torch.exp(-4.0 * (d * d).sum(-1))


def compute_strike_observations(root_states, tar_states):
    """env/tasks/humanoid_strike.py:193-216 -> [N,15]; z of the local target position is the target's absolute z (sic)."""
    hq = calc_heading_quat_inv(root_states[:, 3:7])
    lp = tar_states[:, 0:3] - root_states[:, 0:3]
    lp = torch.cat([lp[:, 0:2], tar_states[:, 2:3]], dim=-1)
    return torch.cat([quat_rotate(hq, lp), quat_to_tan_norm(quat_mul(hq, tar_states[:, 3:7])), quat_rotate(hq, tar_states[:, 7:10]),
                      quat_rotate(hq, tar_states[:, 10:13])], dim=-1)


def compute_strike_reward(tar_pos, tar_rot, root_state, prev_root_pos, dt):
    """env/tasks/humanoid_strike.py:218-251 (the reference's unused strike_body_vel / near_dist parameters are dropped)."""
    up = torch.zeros_like(tar_pos); up[..., -1] = 1
    tar_rot_err = (up * quat_rotate(tar_rot, up)).sum(-1)
    tar_rot_r = torch.clamp_min(1.0 - tar_rot_err, 0.0)
    _, vel_reward = _toward_target_vel_reward(tar_pos[..., 0:2], root_state[..., 0:3], prev_root_pos, dt, 1.0)
    reward = 0.6 * tar_rot_r + 0.4 * vel_reward
    return torch.where(tar_rot_err < 0.2, torch.ones_like(reward), reward)


def compute_strike_reset(progress, contact, contact_body_ids, body_pos, tar_contact_forces, strike_body_ids, max_episode_length,
                         enable_early_termination, termination_heights):
    """env/tasks/humanoid_strike.py:254-295 -> (reset, terminated) as long tensors.  fall_contact is taken BEFORE the strike bodies are
    zeroed in the aliased masked buffer; the target contact looks at x and y only."""
    terminated = torch.zeros_like(progress)
    if enable_early_termination:
        masked = contact.clone()
        masked[:, contact_body_ids, :] = 0
        fall_contact = (masked.abs() > 0.1).any(-1).any(-1)
        fall_height = body_pos[..., 2] < termination_heights
        fall_height[:, contact_body_ids] = False
        has_fallen = fall_contact & fall_height.any(-1)
        tar_has_contact = (tar_contact_forces[..., 0:2].abs() > 1.0).any(-1)
        masked[:, strike_body_ids, :] = 0
        nonstrike = (masked.abs() > 1.0).any(-1).any(-1)
        has_failed = (has_fallen | (tar_has_contact & nonstrike)) & (progress > 1)
        terminated = torch.where(has_failed, torch.ones_like(progress), terminated)
    reset = torch.where(progress >= max_episode_length - 1, torch.ones_like(progress), terminated)
    return reset, terminated


def task_resample(task, params, u, steps, root_pos, progress):
    """The per-env arithmetic of _reset_task (heading humanoid_heading.py:154-174, location humanoid_location.py:114-125, reach
    humanoid_reach.py:118-130) and strike _reset_target (humanoid_strike.py:108-128) for the resampled rows, given their draws:
    u [n,4] (column k = the env's k-th uniform in the reference's draw order), steps [n] (the randint), root_pos [n,>=2], progress [n].
    -> dict of the new target tensors for those rows."""
    two_pi = 2 * math.pi
    if task == 'heading':
        if params['rand_heading']:
            th, thf, us = two_pi * u[:, 0] - math.pi, two_pi * u[:, 1] - math.pi, u[:, 2]
        else:
            th, thf, us = torch.zeros_like(u[:, 0]), torch.zeros_like(u[:, 0]), u[:, 0]
        return dict(tar_dir=torch.stack([torch.cos(th), torch.sin(th)], dim=-1),
                    tar_speed=(params['speed_max'] - params['speed_min']) * us + params['speed_min'],
                    tar_face_dir=torch.stack([torch.cos(thf), torch.sin(thf)], dim=-1), change_steps=progress + steps)
    if task == 'location':
        return dict(tar_pos=root_pos[:, 0:2] + params['dist_max'] * (2.0 * u[:, 0:2] - 1.0), change_steps=progress + steps)
    if task == 'reach':
        xy = params['dist_max'] * (2.0 * u[:, 0:2] - 1.0)
        z = (params['height_max'] - params['height_min']) * u[:, 2] + params['height_min']
        return dict(tar_pos=torch.cat([xy, z.unsqueeze(-1)], dim=-1), change_steps=progress + steps)
    assert task == 'strike'
    dmax = torch.where(u[:, 0] < params['near_prob'], torch.full_like(u[:, 0], params['near_dist']), torch.full_like(u[:, 0], params['dist_max']))
    dist = (dmax - params['dist_min']) * u[:, 1] + params['dist_min']
    th = two_pi * u[:, 2]
    st = torch.zeros(u.shape[0], 13, dtype=u.dtype, device=u.device)
    st[:, 0] = dist * torch.cos(th) + root_pos[:, 0]
    st[:, 1] = dist * torch.sin(th) + root_pos[:, 1]
    st[:, 2] = params['target_height']
    ez = torch.zeros(u.shape[0], 3, dtype=u.dtype, device=u.device); ez[:, 2] = 1.0
    st[:, 3:7] = quat_from_angle_axis(two_pi * u[:, 3], ez)
    return dict(tar_states=st)
